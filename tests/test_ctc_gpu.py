"""GPU parity: fused sm_90a CTC kernel (through the C ABI) vs the CPU oracle.

Tolerance: loss and gradients within 1e-4 relative (BASELINE.json north_star), fp32 kernel vs
float64 oracle.  Gradient tolerance is relative to the largest |grad| of the utterance (entries
are differences of probabilities, many are ~0).
"""
import numpy as np
import pytest
import torch

from oracle import ctc_ref

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def _make(B, T, V, Lmin, Lmax, seed, scale=1.0, repeats=False):
    rng = np.random.RandomState(seed)
    acts = (rng.randn(B, T, V) * scale).astype(np.float32)
    lens = rng.randint(Lmin, Lmax + 1, size=B)
    labels = []
    for L in lens:
        if repeats:
            l = rng.randint(0, 3, size=L)  # many repeated neighbours
        else:
            l = rng.randint(0, V - 1, size=L)
        labels.append(l.astype(np.int32))
    flat = np.concatenate(labels) if len(labels) else np.zeros(0, np.int32)
    return acts, flat, lens.astype(np.int32)


def _run_gpu(acts, flat, act_lens, label_lens, blank=None):
    from speech_b200.functions.ctc import ctc_costs_and_grads
    a = torch.from_numpy(acts).cuda()
    costs, grads = ctc_costs_and_grads(a, torch.from_numpy(flat), torch.from_numpy(act_lens),
                                       torch.from_numpy(label_lens), blank=blank)
    torch.cuda.synchronize()
    return costs.cpu().numpy().astype(np.float64), grads.cpu().numpy().astype(np.float64)


def _check(acts, flat, act_lens, label_lens, blank=None):
    c_ref, g_ref = ctc_ref.ctc_loss_and_grad(acts, flat, act_lens, label_lens, blank)
    c, g = _run_gpu(acts, flat, act_lens, label_lens, blank)
    fin = np.isfinite(c_ref)
    assert np.array_equal(np.isfinite(c), fin)
    np.testing.assert_allclose(c[fin], c_ref[fin], rtol=RTOL)
    for b in range(acts.shape[0]):
        denom = max(np.abs(g_ref[b]).max(), 1e-6)
        assert np.abs(g[b] - g_ref[b]).max() / denom < RTOL, "utt %d" % b


@pytest.mark.parametrize("B,T,V,Lmin,Lmax", [
    (4, 48, 11, 20, 20),     # tests/ctc_test.py shapes (SURVEY §4)
    (3, 1, 5, 0, 1),         # single frame; empty label
    (2, 7, 3, 3, 3),         # odd T
    (5, 33, 29, 0, 16),      # ragged labels incl. empty
    (2, 300, 29, 100, 140),  # S > 256 -> two lattice states per thread
])
def test_ctc_matches_oracle(cuda_lib, B, T, V, Lmin, Lmax):
    acts, flat, llen = _make(B, T, V, Lmin, Lmax, seed=B * 1000 + T)
    alen = np.full(B, T, np.int32)
    _check(acts, flat, alen, llen)


def test_ctc_repeated_labels_and_blank_first(cuda_lib):
    acts, flat, llen = _make(4, 40, 6, 5, 12, seed=7, repeats=True)
    alen = np.full(4, 40, np.int32)
    _check(acts, flat, alen, llen, blank=0 + 5)
    # blank = 0 variant: shift labels so they avoid class 0
    _check(acts, flat + 1, alen, llen, blank=0)


def test_ctc_ragged_act_lens(cuda_lib):
    acts, flat, llen = _make(4, 50, 9, 3, 10, seed=11)
    alen = np.array([50, 37, 21, 44], np.int32)
    _check(acts, flat, alen, llen)


def test_ctc_infeasible_alignment_gives_inf_cost_zero_grad(cuda_lib):
    # label longer than the number of frames -> no valid path
    acts = np.random.RandomState(0).randn(2, 4, 5).astype(np.float32)
    flat = np.array([0, 1, 2, 3, 0, 1, 1], np.int32)
    llen = np.array([6, 1], np.int32)
    flat = np.array([0, 1, 2, 3, 0, 1, 1], np.int32)
    alen = np.array([4, 4], np.int32)
    c, g = _run_gpu(acts, flat, alen, llen)
    assert np.isinf(c[0]) and np.isfinite(c[1])
    assert np.all(g[0] == 0)


def test_ctc_large_logit_range(cuda_lib):
    acts, flat, llen = _make(3, 60, 12, 5, 15, seed=3, scale=12.0)
    alen = np.full(3, 60, np.int32)
    _check(acts, flat, alen, llen)


def test_ctc_unstaged_path_large_vocab(cuda_lib):
    # T*V*4 > 220 KB forces the non-staged (global gather) variant
    acts, flat, llen = _make(2, 600, 120, 10, 30, seed=5)
    alen = np.array([600, 555], np.int32)
    c, g = _run_gpu(acts, flat, alen, llen)
    a = torch.from_numpy(acts).double().requires_grad_(True)
    lp = torch.log_softmax(a, 2).transpose(0, 1)
    loss = torch.nn.functional.ctc_loss(lp, torch.from_numpy(flat).long(), torch.from_numpy(alen).long(),
                                        torch.from_numpy(llen).long(), blank=119, reduction="none")
    loss.sum().backward()
    np.testing.assert_allclose(c, loss.detach().numpy(), rtol=RTOL)
    g_ref = a.grad.numpy()
    for b in range(2):
        assert np.abs(g[b] - g_ref[b]).max() / np.abs(g_ref[b]).max() < RTOL


def test_ctc_north_star_shape_vs_torch_cpu(cuda_lib):
    """B=64, T=1000, V=29 (SURVEY §8d standalone microbench shape) against torch's CPU CTC."""
    rng = np.random.RandomState(0)
    B, T, V = 64, 1000, 29
    acts = rng.randn(B, T, V).astype(np.float32)
    llen = rng.randint(40, 121, size=B).astype(np.int32)
    flat = np.concatenate([rng.randint(0, 28, size=L) for L in llen]).astype(np.int32)
    alen = np.full(B, T, np.int32)
    c, g = _run_gpu(acts, flat, alen, llen)
    a = torch.from_numpy(acts).double().requires_grad_(True)
    lp = torch.log_softmax(a, 2).transpose(0, 1)
    loss = torch.nn.functional.ctc_loss(lp, torch.from_numpy(flat).long(), torch.from_numpy(alen).long(),
                                        torch.from_numpy(llen).long(), blank=V - 1, reduction="none")
    loss.sum().backward()
    np.testing.assert_allclose(c, loss.detach().numpy(), rtol=RTOL)
    g_ref = a.grad.numpy()
    for b in range(B):
        assert np.abs(g[b] - g_ref[b]).max() / np.abs(g_ref[b]).max() < RTOL
    # size-independent property: every gradient row sums to ~0 (softmax minus a distribution)
    assert np.abs(g.sum(-1)).max() < 1e-4


def test_ctcloss_module_contract(cuda_lib):
    """functions.ctc.CTCLoss drop-in: zero-arg ctor, (1,)-shaped differentiable loss, CPU int tensors."""
    from speech_b200.functions.ctc import CTCLoss
    acts, flat, llen = _make(4, 48, 11, 20, 20, seed=1)
    a = torch.from_numpy(acts).cuda().requires_grad_(True)
    loss = CTCLoss()(a, torch.IntTensor(flat), torch.IntTensor([48] * 4), torch.IntTensor(llen))
    assert loss.shape == (1,)
    (2.0 * loss).backward()
    c_ref, g_ref = ctc_ref.ctc_loss_and_grad(acts, flat, [48] * 4, llen)
    assert abs(loss.item() - c_ref.sum()) / c_ref.sum() < RTOL
    assert np.abs(a.grad.cpu().numpy() - 2.0 * g_ref).max() < 2e-4
