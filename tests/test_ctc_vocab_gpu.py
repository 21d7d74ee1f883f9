"""CTC loss and prefix beam search at subword-sized vocabularies (csrc/ctc.cu compact path,
csrc/decode.cu shortlist search), against the CPU oracles and against the kernels they stand in for.

Tolerances are those of tests/test_ctc_gpu.py (1e-4 relative; gradients relative to the largest
|grad| of the utterance) and tests/test_decode_gpu.py (labels exact, scores 1e-5).  The shortlist
search must be bit-identical to the full scan: labels, lengths and float64 scores.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ctc_decoder_ref, ctc_ref

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def _labels(rng, V, blank, lens, repeats=False):
    out = []
    for L in lens:
        if repeats:
            l = rng.choice([3, 3, 5, V - 2, 0], size=L)
        else:
            l = rng.randint(0, V - 1, size=L)
        out.append(np.where(l == blank, 1, l).astype(np.int32))
    return np.concatenate(out) if out else np.zeros(0, np.int32)


def _ctc_call(entry, acts, flat, alen, llen, blank, need_grad=True):
    """sb_ctc_fwd_bwd or sb_ctc_fwd_bwd_compact through the C ABI."""
    from speech_b200 import _lib
    lib = _lib.load()
    B, T, V = acts.shape
    a = torch.from_numpy(acts).cuda()
    offs = np.zeros(B, np.int32)
    offs[1:] = np.cumsum(llen)[:-1]
    d = [torch.from_numpy(np.ascontiguousarray(v, np.int32)).cuda()
         for v in (flat if flat.size else np.zeros(1, np.int32), offs, llen, alen)]
    max_l = int(llen.max())
    n = ctypes.c_size_t(0)
    size_fn = lib.sb_ctc_compact_workspace_size if entry == "compact" else lib.sb_ctc_workspace_size
    _lib.check(size_fn(B, T, V, max_l, ctypes.byref(n)), "workspace size")
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    costs = torch.empty(B, device="cuda")
    grads = torch.full_like(a, float("nan")) if need_grad else None
    fn = lib.sb_ctc_fwd_bwd_compact if entry == "compact" else lib.sb_ctc_fwd_bwd
    _lib.check(fn(a.data_ptr(), _lib.ptr(grads), d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                  d[3].data_ptr(), B, T, V, blank, max_l, costs.data_ptr(), ws.data_ptr(), n.value,
                  _lib.stream_ptr()), entry)
    torch.cuda.synchronize()
    g = grads.cpu().numpy().astype(np.float64) if need_grad else None
    return costs.cpu().numpy().astype(np.float64), g


def _check(c, g, c_ref, g_ref):
    fin = np.isfinite(c_ref)
    assert np.array_equal(np.isfinite(c), fin)
    np.testing.assert_allclose(c[fin], c_ref[fin], rtol=RTOL)
    if g is None:
        return
    for b in range(g.shape[0]):
        denom = max(np.abs(g_ref[b]).max(), 1e-6)
        assert np.abs(g[b] - g_ref[b]).max() / denom < RTOL, "utt %d" % b


def _case(V, seed):
    """B=5: repeats, an infeasible utterance (labels longer than its frames), an empty label,
    ragged act_lens"""
    rng = np.random.RandomState(seed)
    B, T = 5, 24
    acts = (rng.randn(B, T, V) * 2.0).astype(np.float32)
    llen = np.array([9, 12, 0, 14, 5], np.int32)
    alen = np.array([24, 20, 17, 10, 24], np.int32)   # utterance 3: 14 labels in 10 frames
    blank = V - 1
    flat = _labels(rng, V, blank, llen[:1], repeats=True)
    flat = np.concatenate([flat, _labels(rng, V, blank, llen[1:])])
    return acts, flat, alen, llen, blank


@pytest.mark.parametrize("V", [20001, 32768])
def test_large_vocab_loss_matches_oracle(cuda_lib, V):
    from speech_b200.functions.ctc import ctc_costs_and_grads
    acts, flat, alen, llen, blank = _case(V, seed=V)
    c_ref, g_ref = ctc_ref.ctc_loss_and_grad(acts, flat, alen, llen, blank)
    assert np.isinf(c_ref[3]) and np.isfinite(c_ref[[0, 1, 2, 4]]).all()
    costs, grads = ctc_costs_and_grads(torch.from_numpy(acts).cuda(), torch.from_numpy(flat),
                                       torch.from_numpy(alen), torch.from_numpy(llen), blank=blank)
    c, g = costs.cpu().double().numpy(), grads.cpu().double().numpy()
    _check(c, g, c_ref, g_ref)
    assert np.all(g[3] == 0)
    for b in range(5):
        assert np.all(g[b, alen[b]:] == 0)
    costs2, none = ctc_costs_and_grads(torch.from_numpy(acts).cuda(), torch.from_numpy(flat),
                                       torch.from_numpy(alen), torch.from_numpy(llen), blank=blank,
                                       need_grad=False)
    assert none is None
    assert np.array_equal(costs2.cpu().double().numpy(), c)


def test_large_vocab_blank_first_and_label_equal_to_blank(cuda_lib):
    rng = np.random.RandomState(4)
    B, T, V = 3, 30, 20001
    acts = rng.randn(B, T, V).astype(np.float32)
    llen = np.array([6, 8, 4], np.int32)
    flat = rng.randint(1, V, size=int(llen.sum())).astype(np.int32)
    flat[2] = 0                                  # a label equal to the blank class
    alen = np.full(B, T, np.int32)
    c_ref, g_ref = ctc_ref.ctc_loss_and_grad(acts, flat, alen, llen, 0)
    c, g = _ctc_call("fused", acts, flat, alen, llen, 0)
    _check(c, g, c_ref, g_ref)


@pytest.mark.parametrize("V", [11, 29, 120, 1000])
def test_compact_matches_fused_and_oracle(cuda_lib, V):
    acts, flat, alen, llen, blank = _case(V, seed=V)
    c_ref, g_ref = ctc_ref.ctc_loss_and_grad(acts, flat, alen, llen, blank)
    c_f, g_f = _ctc_call("fused", acts, flat, alen, llen, blank)
    c_c, g_c = _ctc_call("compact", acts, flat, alen, llen, blank)
    _check(c_f, g_f, c_ref, g_ref)
    _check(c_c, g_c, c_ref, g_ref)
    _check(c_c, g_c, c_f, g_f)
    c_n, _ = _ctc_call("compact", acts, flat, alen, llen, blank, need_grad=False)
    assert np.array_equal(c_n, c_c)


def test_compact_label_set_covers_every_class(cuda_lib):
    # every class is the blank or a label: the rest column is empty (-inf)
    rng = np.random.RandomState(9)
    V, T = 11, 40
    acts = rng.randn(2, T, V).astype(np.float32)
    flat = np.concatenate([np.arange(10), rng.randint(0, 10, 6)]).astype(np.int32)
    llen = np.array([10, 6], np.int32)
    alen = np.full(2, T, np.int32)
    c_ref, g_ref = ctc_ref.ctc_loss_and_grad(acts, flat, alen, llen, 10)
    _check(*_ctc_call("compact", acts, flat, alen, llen, 10), c_ref, g_ref)


# ---------------------------------------------------------------------------------------------
# beam search
# ---------------------------------------------------------------------------------------------
def _probs(rng, B, T, S, kind):
    logits = rng.randn(B, T, S).astype(np.float32) * 3.0
    if kind == "ties":
        logits = np.round(logits)                   # many exactly equal probabilities
    p = torch.softmax(torch.from_numpy(logits), 2)
    if kind == "ties":
        p = torch.round(p * 64) / 64                # quantised, many zeros
    if kind == "inf":
        keep = torch.from_numpy(rng.rand(B, T, S) < 0.02)
        keep[..., S - 1] = True
        p = torch.where(keep, p, torch.zeros_like(p))   # mostly zero probability: -inf log
    return p.contiguous()


def _beam_call(entry, logp, lens, K, blank):
    from speech_b200 import _lib
    lib = _lib.load()
    B, T, S = logp.shape
    n = ctypes.c_size_t(0)
    _lib.check(lib.sb_ctc_prefix_beam_workspace_size(B, T, K, ctypes.byref(n)), "ws")
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    lab = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
    ln = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = torch.empty(B, dtype=torch.float64, device="cuda")
    fn = lib.sb_ctc_prefix_beam_shortlist if entry == "shortlist" else lib.sb_ctc_prefix_beam
    _lib.check(fn(logp.data_ptr(), lens.data_ptr(), B, T, S, K, blank, lab.data_ptr(),
                  ln.data_ptr(), sc.data_ptr(), ws.data_ptr(), n.value, _lib.stream_ptr()), entry)
    ln = ln.cpu().numpy()
    lab = lab.cpu().numpy()
    return [lab[b, :ln[b]].tolist() for b in range(B)], ln, sc.cpu().numpy()


@pytest.mark.parametrize("S", [29, 500, 1500])
@pytest.mark.parametrize("K", [1, 8, 32])
@pytest.mark.parametrize("kind", ["random", "ties", "inf"])
def test_shortlist_bit_identical_to_full_scan(cuda_lib, S, K, kind):
    rng = np.random.RandomState(S * 100 + K)
    B, T = 4, 40
    logp = torch.log(_probs(rng, B, T, S, kind)).cuda()
    lens = torch.tensor([T, T - 7, 1, T // 2], dtype=torch.int32, device="cuda")
    full = _beam_call("full", logp, lens, K, S - 1)
    short = _beam_call("shortlist", logp, lens, K, S - 1)
    assert full[0] == short[0]
    assert np.array_equal(full[1], short[1])
    assert np.array_equal(full[2].view(np.int64), short[2].view(np.int64))


@pytest.mark.parametrize("S,K", [(3000, 8), (2000, 10), (20000, 4)])
def test_large_vocab_decode_matches_oracle(cuda_lib, S, K):
    from speech_b200.models.ctc_decoder import decode, decode_batch
    rng = np.random.RandomState(S + K)
    B, T = 3, 36
    probs = _probs(rng, B, T, S, "random")
    pn = probs.numpy()
    lens = np.array([T, 30, 41 - 11], np.int32)
    res = decode_batch(probs.cuda(), beam_size=K, blank=S - 1, lens=lens, with_scores=True)
    for b in range(B):
        lab, sc = ctc_decoder_ref.prefix_beam_search(pn[b, :lens[b]], beam_size=K, blank=S - 1)
        assert tuple(lab) == res[b][0], b
        assert abs(sc - res[b][1]) < 1e-5 * max(1.0, abs(sc))
    lab, sc = decode(pn[0], beam_size=K, blank=S - 1)
    ref_lab, ref_sc = ctc_decoder_ref.prefix_beam_search(pn[0], beam_size=K, blank=S - 1)
    assert tuple(lab) == tuple(ref_lab)
    assert abs(sc - ref_sc) < 1e-5 * max(1.0, abs(ref_sc))


def test_ctc_model_32767_symbols(cuda_lib):
    """CTC over 32767 symbols: one FlatSGD step, the logits' gradient against float64
    F.ctc_loss, and infer(beam_size=8) against per-utterance decode()."""
    from speech_b200.models import CTC
    from speech_b200.models.ctc_decoder import decode
    from speech_b200.optim import FlatSGD
    torch.manual_seed(0)
    rng = np.random.RandomState(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                       "rnn": {"dim": 64, "bidirectional": True, "layers": 1}}}
    m = CTC(80, 32767, cfg).cuda()
    inputs = [rng.randn(100 - 6 * i, 80).astype(np.float32) for i in range(3)]
    labels = [rng.randint(0, 32767, 5 + 2 * i).tolist() for i in range(3)]
    x, y, x_lens, y_lens = m._collated((inputs, labels))
    out = m._forward_impl(x, None)
    out.retain_grad()
    loss = m.ctc_loss(out, y, x_lens, y_lens)
    loss.backward()
    a = out.detach().cpu().double().requires_grad_(True)
    ref = torch.nn.functional.ctc_loss(torch.log_softmax(a, 2).transpose(0, 1), y.long(),
                                       x_lens.long(), y_lens.long(), blank=32767,
                                       reduction="sum", zero_infinity=False)
    ref.backward()
    assert abs(loss.item() - ref.item()) < RTOL * abs(ref.item())
    g, g_ref = out.grad.cpu().double().numpy(), a.grad.numpy()
    for b in range(3):
        assert np.abs(g[b] - g_ref[b]).max() / np.abs(g_ref[b]).max() < RTOL
    opt = FlatSGD(m, lr=1e-3)
    opt.zero_grad()
    m.loss((inputs, labels)).backward()
    opt.step()
    torch.cuda.synchronize()
    assert all(torch.isfinite(p).all() for p in m.parameters())
    m.eval()
    preds = m.infer((inputs, labels), beam_size=8)
    with torch.no_grad():
        probs = m._forward_impl(x, None, softmax=True).cpu().numpy()
    for b in range(3):
        assert tuple(preds[b]) == decode(probs[b], beam_size=8, blank=32767)[0], b
