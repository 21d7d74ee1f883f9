"""LM-fused CTC prefix beam search on the GPU (sb_ctc_prefix_beam_lm, csrc/decode.cu).

- against the reference restatement tests/ctc_lm_ref.prefix_beam_search_lm: labels identical,
  float64 scores within 1e-9 relative (the device's log / exp may differ from libm's in the last
  bit).  The log-probabilities are taken on the host with np.log, as the reference does, so both
  sides search the same float32 inputs;
- with lm_weight = insertion_bonus = 0, bit for bit the LM-less search, on both routes;
- the forced shortlist route bit for bit the full scan with an LM;
- a strongly weighted LM changes an acoustically ambiguous decode;
- CTC.infer with an LM, default and exact-lengths modes.
"""
import ctypes

import numpy as np
import pytest
import torch

from ctc_lm_ref import prefix_beam_search_lm
from ngram_ref import ArpaLM
from speech_b200 import _lib
from speech_b200.lm import NGramLM
from speech_b200.models import ctc_decoder

pytestmark = pytest.mark.gpu


def _probs(rng, B, T, S, sharp=2.5):
    x = rng.randn(B, T, S) * sharp
    x[:, :, S - 1] += 1.5                                   # the blank is common, as in CTC
    p = np.exp(x - x.max(2, keepdims=True))
    return (p / p.sum(2, keepdims=True)).astype(np.float32)


def _lm(tmp_path, rng, S, order, n=200):
    """a trained LM over classes 0..S-2 (blank = S-1) and its reference reader"""
    seqs = [rng.randint(0, S - 1, rng.randint(1, 25)).tolist() for _ in range(n)]
    lm = NGramLM.train(seqs, order, S, S - 1)
    p = str(tmp_path / ("lm%d.arpa" % order))
    lm.to_arpa(p)
    return lm, ArpaLM(p, [str(c) for c in range(S - 1)], S - 1)


def _call(logp, lens, K, blank, lm=None, a=0.0, b=0.0, shortlist=False):
    """a C ABI entry point on host float32 log-probabilities -> [(labels, score)]"""
    lib = _lib.load()
    B, T, S = logp.shape
    lp = torch.from_numpy(np.ascontiguousarray(logp, np.float32)).cuda()
    ln = torch.tensor(lens, dtype=torch.int32, device="cuda")
    nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    lab = torch.empty(B, T, dtype=torch.int32, device="cuda")
    n = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = torch.empty(B, dtype=torch.float64, device="cuda")
    outs = (lab.data_ptr(), n.data_ptr(), sc.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr())
    if lm is None:
        fn = lib.sb_ctc_prefix_beam_shortlist if shortlist else lib.sb_ctc_prefix_beam
        st = fn(lp.data_ptr(), ln.data_ptr(), B, T, S, K, blank, *outs)
    else:
        fn = lib.sb_ctc_prefix_beam_lm_shortlist if shortlist else lib.sb_ctc_prefix_beam_lm
        tables, _ = lm.device_tables(lp.device)
        st = fn(lp.data_ptr(), ln.data_ptr(), B, T, S, K, blank, ctypes.byref(tables), a, b, *outs)
    _lib.check(st, fn.__name__)
    lab, n, sc = lab.cpu().numpy(), n.cpu().numpy(), sc.cpu().numpy()
    return [(tuple(int(v) for v in lab[i, :n[i]]), float(sc[i])) for i in range(B)]


def _host_log(probs):
    with np.errstate(divide="ignore"):
        return np.log(probs)


def _assert_oracle(res, probs, lens, K, blank, ref, a, b):
    for i, L in enumerate(lens):
        lab, sc = prefix_beam_search_lm(probs[i, :L], K, blank, ref, a, b)
        assert res[i][0] == tuple(lab), i
        assert abs(res[i][1] - sc) <= 1e-9 * max(1.0, abs(sc)), (i, res[i][1], sc)


@pytest.mark.parametrize("T,S,K,order,a,b", [
    (247, 29, 1, 3, 0.8, 1.0),
    (247, 29, 1, 8, 2.0, -1.0),
    (247, 29, 8, 5, 0.5, 0.5),
    (247, 29, 8, 1, 1.5, -0.3),
    (60, 29, 32, 3, 1.0, 2.0),
    (60, 29, 32, 8, 0.3, -2.0),
    (100, 62, 10, 5, 1.2, 0.0),
    (100, 62, 10, 1, 0.7, -0.7),
])
def test_lm_search_equals_oracle(tmp_path, T, S, K, order, a, b):
    rng = np.random.RandomState(T + S + K + order)
    lm, ref = _lm(tmp_path, rng, S, order)
    lens = [T, T - 17, T // 2]
    probs = _probs(rng, 3, T, S)
    res = _call(_host_log(probs), lens, K, S - 1, lm, a, b)
    _assert_oracle(res, probs, lens, K, S - 1, ref, a, b)
    if K > 1:
        assert _call(_host_log(probs), lens, K, S - 1, lm, a, b, shortlist=True) == res


@pytest.mark.parametrize("S,K", [(29, 1), (29, 8), (62, 32), (1000, 8)])
def test_zero_weights_are_the_plain_search(tmp_path, S, K):
    rng = np.random.RandomState(S + K)
    lm, _ = _lm(tmp_path, rng, S, 4)
    lens = [80, 61, 5]
    probs = _probs(rng, 3, 80, S)
    logp = _host_log(probs)
    for sl in (False, True):
        assert _call(logp, lens, K, S - 1, lm, 0.0, 0.0, sl) == _call(logp, lens, K, S - 1,
                                                                       shortlist=sl)
    pt = torch.from_numpy(probs).cuda()
    assert (ctc_decoder.decode_batch(pt, K, S - 1, lens, True, lm=lm)
            == ctc_decoder.decode_batch(pt, K, S - 1, lens, True))


@pytest.mark.parametrize("S,K,order,a,b", [(29, 4, 5, 1.0, 0.5), (29, 16, 3, 3.0, -1.0),
                                           (1000, 8, 3, 0.6, 1.0), (1000, 4, 2, 5.0, 0.0)])
def test_forced_shortlist_equals_full_scan(tmp_path, S, K, order, a, b):
    rng = np.random.RandomState(S * K + order)
    lm, _ = _lm(tmp_path, rng, S, order, n=400)
    lens = [120, 97, 33, 120]
    logp = _host_log(_probs(rng, 4, 120, S, sharp=1.5))
    full = _call(logp, lens, K, S - 1, lm, a, b)
    assert _call(logp, lens, K, S - 1, lm, a, b, shortlist=True) == full


def test_large_vocabulary_takes_the_shortlist_and_equals_oracle(tmp_path):
    rng = np.random.RandomState(7)
    S, K, T = 5001, 4, 10
    lm, ref = _lm(tmp_path, rng, S, 3, n=300)
    lens = [T, 7]
    probs = _probs(rng, 2, T, S, sharp=3.0)
    res = _call(_host_log(probs), lens, K, S - 1, lm, 0.7, 0.5)
    _assert_oracle(res, probs, lens, K, S - 1, ref, 0.7, 0.5)


def test_the_lm_decides_ambiguous_frames(tmp_path):
    # classes 0..3, blank 4.  Frame 1 says "0"; frame 3 is ambiguous between 1 and 2, slightly
    # for 2.  The LM has only ever seen "0 1".
    S, blank = 5, 4
    lm = NGramLM.train([[0, 1]] * 50 + [[3]], 2, S, blank)
    p = np.full((1, 4, S), 0.01, np.float32)
    p[0, 0, 0] = 0.96
    p[0, 1, blank] = 0.96
    p[0, 2, 1], p[0, 2, 2], p[0, 2, blank] = 0.47, 0.50, 0.01
    p[0, 3, blank] = 0.96
    p /= p.sum(2, keepdims=True)
    pt = torch.from_numpy(p).cuda()
    for K in (1, 4):
        assert ctc_decoder.decode_batch(pt, K, blank, lm=lm, lm_weight=0.0)[0] == (0, 2)
        assert ctc_decoder.decode_batch(pt, K, blank)[0] == (0, 2)
        assert ctc_decoder.decode_batch(pt, K, blank, lm=lm, lm_weight=2.0)[0] == (0, 1)
        lab, sc = ctc_decoder.decode(p[0], K, blank, lm=lm, lm_weight=2.0)
        assert lab == (0, 1) and np.isfinite(sc)


def test_decoder_checks_its_lm_arguments(tmp_path):
    rng = np.random.RandomState(0)
    lm, _ = _lm(tmp_path, rng, 29, 2)
    pt = torch.from_numpy(_probs(rng, 1, 10, 30)).cuda()
    with pytest.raises(ValueError):
        ctc_decoder.decode_batch(pt, 4, 29, lm=lm, lm_weight=0.5)          # 29 classes, not 30
    with pytest.raises(ValueError):
        ctc_decoder.decode_batch(pt, 4, 29, lm_weight=0.5)
    with pytest.raises(_lib.SpeechB200Error):
        ctc_decoder.decode_batch(pt[..., :29].contiguous(), 33, 28, lm=lm)  # beam > 32


@pytest.mark.parametrize("exact", [False, True])
def test_ctc_infer_with_lm_equals_oracle(tmp_path, exact):
    from speech_b200.models import CTC
    torch.manual_seed(0)
    rng = np.random.RandomState(1)
    V = 28
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                       "rnn": {"dim": 32, "bidirectional": True, "layers": 2}}}
    m = CTC(80, V, cfg).cuda()
    m.set_eval()
    inputs = [rng.randn(n, 80).astype(np.float32) for n in (150, 120, 96)]
    labels = [rng.randint(0, V, 9).tolist() for _ in range(3)]
    lm, ref = _lm(tmp_path, rng, V + 1, 4)
    _, _, x_lens, _ = m.collate(inputs, labels)
    with torch.no_grad():
        probs = torch.softmax(m((inputs, labels)), 2).cpu().numpy()
    lens = x_lens.tolist() if exact else [probs.shape[1]] * 3
    preds = m.infer((inputs, labels), beam_size=8, lm=lm, lm_weight=1.0, insertion_bonus=0.5)
    for i, L in enumerate(lens):
        lab, _ = prefix_beam_search_lm(probs[i, :L], 8, V, ref, 1.0, 0.5)
        assert tuple(preds[i]) == tuple(lab), i
    with pytest.raises(ValueError):
        m.infer((inputs, labels), beam_size=8, lm=NGramLM.train([[0]], 2, V, V - 1))
