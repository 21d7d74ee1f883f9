"""GPU tests of the Transducer's large-vocabulary decoding: the shortlist producer
(sb_rnnt_shortlist_rows, csrc/joint_vocab.cu) and the shortlist beam search
(sb_rnnt_decode_static_shortlist, csrc/tdecode.cu).

- producer: values and classes bit-identical to a stable sort of the slab path's lp_full rows;
- search: labels, lengths and float64 scores bit-identical to sb_rnnt_decode_static wherever that
  kernel runs, equal to the CPU oracle at V+1 = 20001, and the flag on a lattice built to need it;
- model: a 20000-label Transducer trains a step and infers without the full lattice, with the
  predictions of the oracle and of decode_static_batch on m(batch)."""
import math

import numpy as np
import pytest
import torch

from oracle import decode_static_ref as ref
from test_rnnt_shortlist_host import tie_lattice

pytestmark = pytest.mark.gpu


def _joint_case(B, T, U1, H, V1, blank, seed):
    """fx, fy, fc2 weight / bias and label matrix with exact ties between classes (duplicated fc2
    rows, some across the GEMM's 128- and 256-column tile edges) and -inf classes (bias -inf)."""
    rng = np.random.RandomState(seed)
    fx = torch.from_numpy(rng.randn(B, T, H).astype(np.float32) * 0.7).cuda()
    fy = torch.from_numpy(rng.randn(B, U1, H).astype(np.float32) * 0.7).cuda()
    w2 = rng.randn(V1, H).astype(np.float32) / np.sqrt(H)
    b2 = rng.randn(V1).astype(np.float32) * 0.1
    for a, c in ((1, 3), (127, 128), (255, 256), (300, 17), (V1 - 2, 5)):
        if a < V1 and c < V1 and blank not in (a, c):       # tied classes near the top of a row
            b2[a] = 1.5 + 0.1 * rng.rand()
            w2[c], b2[c] = w2[a], b2[a]
    for k in (2, 40, V1 // 2):
        if k != blank:
            b2[k] = -np.inf
    ymat = rng.randint(0, V1 - 1, size=(B, U1 - 1))
    ymat[ymat >= blank] += 1
    edges = [k for k in (127, 128, 255, 256, V1 - 2) if k < V1 and k != blank]
    ymat.flat[:len(edges)] = edges[:ymat.size]
    return fx, fy, torch.from_numpy(w2).cuda(), torch.from_numpy(b2).cuda(), torch.from_numpy(ymat)


def _sorted_reference(lp, kp, blank):
    """(values, classes, blank lp, beta) from a stable descending sort of the non-blank columns"""
    V1 = lp.shape[-1]
    cls = torch.tensor([k for k in range(V1) if k != blank], device=lp.device)
    s, o = torch.sort(lp[..., cls], dim=-1, descending=True, stable=True)
    n = min(kp, V1 - 1)
    beta = s[..., kp] if V1 - 1 > kp else torch.full_like(s[..., 0], -math.inf)
    return s[..., :n], cls[o[..., :n]].int(), lp[..., blank], beta


@pytest.mark.parametrize("V1,blank,kp", [(65, 64, 64), (65, 0, 8), (1000, 999, 4), (1000, 0, 33),
                                         (8192, 8191, 8), (32768, 32767, 64), (32768, 0, 1)])
def test_producer_is_a_stable_sort_of_lp_full(cuda_lib, V1, blank, kp):
    from speech_b200.functions.transducer import joint_log_probs, joint_shortlists
    from speech_b200.transducer_decoders import shortlists_of_lp
    B, T, U1, H = 2, 11, 5, 64
    fx, fy, w2, b2, ymat = _joint_case(B, T, U1, H, V1, blank, V1 + kp)

    class FC2:
        weight, bias = w2, b2
    lp = joint_log_probs(fx, fy, FC2, ymat, blank)
    val, idx, meta = joint_shortlists(fx, fy, FC2, ymat, blank, kp)
    wv, wi, wb, wbeta = _sorted_reference(lp, kp, blank)
    n = wv.shape[-1]
    assert torch.equal(idx[..., :n], wi)
    assert torch.equal(val[..., :n], wv)                   # bit for bit (-inf included)
    assert torch.equal(meta[..., 0], wb)
    assert torch.equal(meta[..., 1], wbeta)
    if n < kp:
        assert bool((idx[..., n:] == -1).all()) and bool((val[..., n:] == -math.inf).all())
    # the producer on the given tensor (batch-first rows, no lse) writes the same lists
    for a, b in zip(shortlists_of_lp(lp, kp, blank), (val, idx, meta)):
        assert torch.equal(a, b)


def _lattice(rng, kind, T, U, V, peak=0.0):
    if kind == "quantised":
        return -rng.randint(1, 5, size=(T, U, V)).astype(np.float32)
    x = rng.randn(T, U, V) * (3.0 if kind == "peaky" else 1.0)
    if peak:
        x[..., rng.randint(0, V)] += peak
    x = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    if kind == "neginf":
        x[rng.rand(T, U, V) < 0.3] = -np.inf
    return x


def _both(lp, tlens, ulens, K, blank):
    """full-lattice kernel and shortlist kernel (kp = K) on the same lattice, on the host"""
    from speech_b200.transducer_decoders import (_shortlist_search, decode_static_batch,
                                                 decode_static_fits, shortlists_of_lp)
    V = lp.shape[-1]
    assert decode_static_fits(K, V)
    full = decode_static_batch(lp, tlens, ulens, K, blank)
    sl = _shortlist_search(shortlists_of_lp(lp, K, blank), tlens, ulens, V, K, blank)
    return full, sl


def _same_score(a, b):
    return a == b or (math.isnan(a) and math.isnan(b))


@pytest.mark.parametrize("K,V", [(1, 29), (1, 1500), (4, 29), (4, 1000), (4, 6000), (8, 500),
                                 (8, 3000), (32, 200), (32, 790)])
@pytest.mark.parametrize("kind", ["random", "peaky", "quantised", "neginf"])
def test_shortlist_search_bit_identical_to_full(cuda_lib, K, V, kind):
    rng = np.random.RandomState(K * 7919 + V + len(kind))
    B, T, U1 = 6, 14, 7
    lp = torch.from_numpy(np.stack([_lattice(rng, kind, T, U1, V) for _ in range(B)])).cuda()
    tlens = [14, 9, 14, 3, 1, 14]                          # ragged batch
    ulens = [7, 7, 4, 2, 1, 6]
    for blank in (V - 1, 0):
        (fl, fs), (sl, ss, flags) = _both(lp, tlens, ulens, K, blank)
        assert flags == [0] * B, (blank, flags)
        assert sl == fl, blank
        assert all(_same_score(a, b) for a, b in zip(ss, fs)), (blank, ss, fs)


@pytest.mark.parametrize("beam", [1, 2, 4, 8])
@pytest.mark.parametrize("T,U,V,peak,seed", [(6, 4, 5, 0.0, 0), (20, 8, 11, 0.0, 1),
                                             (30, 12, 29, 3.0, 2), (48, 21, 11, 2.0, 3),
                                             (12, 3, 62, 0.0, 4)])
def test_decode_static_lattices(cuda_lib, beam, T, U, V, peak, seed):
    """the lattices of tests/test_decode_static.py"""
    rng = np.random.RandomState(seed)
    lat = torch.from_numpy(_lattice(rng, "random", T, U, V, peak)[None]).cuda()
    for blank in (V - 1, 0):
        (fl, fs), (sl, ss, flags) = _both(lat, [T], [U], beam, blank)
        assert flags == [0] and sl == fl and ss == fs, (beam, blank)


@pytest.mark.parametrize("beam,blank,seed", [(2, 20000, 0), (4, 0, 1), (4, 20000, 2)])
def test_large_vocabulary_equals_oracle(cuda_lib, beam, blank, seed):
    from speech_b200.transducer_decoders import decode_static, decode_static_fits
    V = 20001
    assert not decode_static_fits(beam, V)
    rng = np.random.RandomState(seed)
    lat = _lattice(rng, "peaky", 4, 3, V, peak=6.0)
    want, wscore = ref.decode_static(lat, beam, blank)
    got, gscore = decode_static(lat, beam, blank)
    assert got == want and gscore == wscore


def test_flag_on_merged_scores(cuda_lib):
    from speech_b200.transducer_decoders import (_shortlist_search, decode_static,
                                                 decode_static_fits, shortlists_of_lp)
    lat, blank = tie_lattice()
    V = lat.shape[-1]
    assert not decode_static_fits(2, V)
    lp = torch.from_numpy(lat[None]).cuda()
    labels, _, flags = _shortlist_search(shortlists_of_lp(lp, 2, blank), [2], [2], V, 2, blank)
    assert flags[0] > 0 and labels == [[5]]
    want, wscore = ref.decode_static(lat, 2, blank)
    assert decode_static(lat, 2, blank) == (want, wscore)


def _model(exact):
    from speech_b200.models import Transducer
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                       "rnn": {"dim": 64, "bidirectional": True, "layers": 1}},
           "decoder": {"embedding_dim": 32, "layers": 1}}
    return Transducer(80, 20000, cfg).cuda()


@pytest.mark.parametrize("exact", [False, True])
def test_model_infers_at_20000_labels(cuda_lib, exact):
    from speech_b200.optim import FlatSGD
    from speech_b200.transducer_decoders import decode_static_batch
    m = _model(exact)
    rng = np.random.RandomState(5)
    inputs = [rng.randn(n, 80).astype(np.float32) for n in (30, 26)]
    labels = [rng.randint(0, 20000, n).tolist() for n in (2, 1)]
    opt = FlatSGD(m, lr=1e-3)
    opt.zero_grad()
    loss = m.loss((inputs, labels))
    loss.backward()
    opt.step()
    assert math.isfinite(loss.item())
    with torch.no_grad():
        out = m((inputs, labels))
    T = out.shape[1]
    tlens = ([m.conv_out_size(i.shape[0], 0) for i in inputs] if exact
             else [min(i.shape[0], T) for i in inputs])
    ulens = [len(l) + 1 for l in labels]
    for beam in (4, 8):
        preds = m.infer((inputs, labels), beam_size=beam)
        batch_preds, _ = decode_static_batch(out, tlens, ulens, beam, m.blank)
        assert preds == batch_preds, beam
        for b in range(len(inputs)):
            want, _ = ref.decode_static(out[b, :tlens[b], :ulens[b]].cpu().numpy(), beam, m.blank)
            assert preds[b] == want, (beam, b)


def test_model_infer_never_holds_the_lattice(cuda_lib):
    from speech_b200.transducer_decoders import decode_static_batch
    m = _model(False)
    rng = np.random.RandomState(6)
    inputs = [rng.randn(n, 80).astype(np.float32) for n in (240, 200, 220)]
    labels = [rng.randint(0, 20000, n).tolist() for n in (9, 6, 7)]
    preds = m.infer((inputs, labels), beam_size=4)         # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    preds = m.infer((inputs, labels), beam_size=4)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    with torch.no_grad():
        out = m((inputs, labels))
    assert growth < out.numel() * 4 // 2, (growth, out.numel() * 4)
    T = out.shape[1]
    want, _ = decode_static_batch(out, [min(i.shape[0], T) for i in inputs],
                                  [len(l) + 1 for l in labels], 4, m.blank)
    assert preds == want
