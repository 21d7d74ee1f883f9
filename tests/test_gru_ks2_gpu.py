"""GPU tests of the K-split GRU forward recurrence kernel over 2-CTA clusters (gru_fwd_ks_kernel<2>).

Each CTA of a 2-CTA cluster contracts one half of h_{t-1} for the 32 units of its cluster; the two
partial products are exchanged through distributed shared memory and summed in rank order.  It is
what sb_gru_fwd runs for both directions of H = 1024 at <= 64 batch rows on a 132-SM H100, where
4-CTA clusters do not fit.  Developer flag 1024 forces it wherever it applies (H % 128 == 0, at
most 64 rows), flag 32 disables every K-split forward (the plain gru_fwd_kernel), and
sb_debug_gru_fwd_kernel says which forward kernel the last launch used.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

FORCE_KS2, NO_KSPLIT = 1024, 32


def _kernel(lib):
    return lib.sb_debug_gru_fwd_kernel().decode()


def _ref_and_ours(B, T, In, H, L, bidir, seed, lens=None, flags=FORCE_KS2):
    """nn.GRU in fp64 on the CPU vs ops.gru_stack under developer flags -> (..., forward kernel)"""
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    from speech_b200 import _lib
    from speech_b200.ops import gru_stack
    torch.manual_seed(seed)
    rnn = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=bidir)
    x = torch.randn(B, T, In)
    rnn64 = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=bidir).double()
    rnn64.load_state_dict({k: v.double() for k, v in rnn.state_dict().items()})
    x64 = x.double().requires_grad_(True)
    if lens is None:
        y64, _ = rnn64(x64)
    else:
        y64, _ = rnn64(pack_padded_sequence(x64, torch.tensor(lens), batch_first=True,
                                            enforce_sorted=False))
        y64, _ = pad_packed_sequence(y64, batch_first=True, total_length=T)
    w = torch.randn_like(y64)
    (y64 * w).sum().backward()
    rnn_c = rnn.cuda()
    xc = x.cuda().requires_grad_(True)
    lib = _lib.load()
    lib.sb_debug_gru_flags(flags)
    try:
        yc = gru_stack(xc, rnn_c, lens=lens)
        torch.cuda.synchronize()
        kernel = _kernel(lib)
        (yc * w.float().cuda()).sum().backward()
        torch.cuda.synchronize()
    finally:
        lib.sb_debug_gru_flags(0)
    return rnn64, x64, y64, rnn_c, xc, yc, kernel


def _check(rnn64, x64, y64, rnn_c, xc, yc, kernel, lens=None):
    """the bars of tests/test_gru_gpu.py"""
    assert kernel == "ks2", kernel
    for b in range(y64.shape[0]):
        L = y64.shape[1] if lens is None else lens[b]
        assert (yc[b, :L].detach().double().cpu() - y64[b, :L]).abs().max().item() < 2e-2, b
    gx = xc.grad.double().cpu()
    assert (gx - x64.grad).abs().max().item() < 3e-2 * x64.grad.abs().max().item() + 1e-4
    for (n, p64), (_, pc) in zip(rnn64.named_parameters(), rnn_c.named_parameters()):
        ref = p64.grad
        assert (pc.grad.double().cpu() - ref).abs().max().item() < \
            3e-2 * ref.abs().max().item() + 1e-4, n


@pytest.mark.parametrize("B,T,In,H,L,bidir", [
    (8, 247, 64, 1024, 1, True),      # the benchmark width and length, 8 / 32 / 64 rows
    (32, 247, 64, 1024, 1, True),
    (64, 247, 64, 1024, 1, True),
    (20, 11, 96, 512, 2, False),      # unidirectional
    (24, 9, 96, 256, 2, True),
    (12, 9, 64, 250, 1, True),        # runs at Hp = 256
])
def test_ks2_forced_matches_fp64(cuda_lib, B, T, In, H, L, bidir):
    _check(*_ref_and_ours(B, T, In, H, L, bidir, seed=B + H))


def test_ks2_exact_lengths_at_benchmark_width(cuda_lib):
    lens = [40, 13, 1, 29, 40, 22, 7, 35]
    out = _ref_and_ours(len(lens), max(lens), 64, 1024, 1, True, seed=11, lens=lens)
    _check(*out, lens=lens)
    xc, yc = out[4], out[5]
    for b, L in enumerate(lens):
        assert float(xc.grad[b, L:].abs().sum()) == 0.0, b
        assert float(yc[b, L:].detach().abs().sum()) == 0.0, b


def test_ks2_padded_width_at_benchmark_width(cuda_lib):
    """H = 1020 runs at Hp = 1024 on the 2-CTA K-split forward"""
    _check(*_ref_and_ours(16, 12, 64, 1020, 1, True, seed=1020))


# ---- direct sb_gru_fwd calls -------------------------------------------------------------------

def _fwd_inputs(T, Bp, H, ndir, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    gi = torch.randn(T * Bp, ndir * 3 * H, device="cuda", generator=g)
    # spectral radius about 0.5: the recurrence contracts, so one-bit differences stay small
    whh = (torch.randn(ndir, 3 * H, H, device="cuda", generator=g) * (0.5 / H ** 0.5)).to(
        torch.bfloat16)
    bhh = torch.randn(ndir, 3 * H, device="cuda", generator=g) * 0.1
    return gi, whh, bhh


def _run_fwd(lib, flags, T, Bp, H, ndir, inputs):
    """one sb_gru_fwd call under developer flags -> (y, xn, gates, forward kernel)"""
    from speech_b200 import _lib, ops
    gi, whh, bhh = inputs
    D = ndir * H
    y = torch.full((T * Bp, D), float("nan"), device="cuda")
    xn = torch.zeros(T * Bp, D, dtype=torch.bfloat16, device="cuda")
    gates = torch.full((T * Bp, ndir, 4, H), float("nan"), device="cuda")
    n = ctypes.c_size_t(0)
    _lib.check(lib.sb_gru_fwd_workspace_size(Bp, H, ndir, ctypes.byref(n)), "ws")
    ws = ops._workspace(n.value, "cuda")
    lib.sb_debug_gru_flags(flags)
    try:
        _lib.check(lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), y.data_ptr(),
                                  xn.data_ptr(), gates.data_ptr(), ws.data_ptr(), n.value,
                                  T, Bp, H, ndir, _lib.stream_ptr()), "sb_gru_fwd")
        torch.cuda.synchronize()
        kernel = _kernel(lib)
    finally:
        lib.sb_debug_gru_flags(0)
    return y, xn, gates, kernel


def _bf16_ulps(a, b):
    """distance in units in the last place between two bf16 tensors (bit patterns, sign-aware)"""
    def key(t):
        i = t.view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -32768 - i, i)     # monotone in the value
    return (key(a) - key(b)).abs()


@pytest.mark.parametrize("Bp", [24, 64])
def test_ks2_matches_ks4(cuda_lib, Bp):
    """bidirectional H = 512: both K splits fit; only the fp32 summation order differs.  At the
    first step that uses the recurrent product (dir 0: t = 1, dir 1: t = T - 2) both kernels see
    the same h_{t-1}, so xn differs in at most the last bf16 bit; later steps inherit those
    one-bit differences through W_hh, so y is compared to a small absolute tolerance."""
    T, H, ndir = 24, 512, 2
    inputs = _fwd_inputs(T, Bp, H, ndir, seed=Bp)
    y2, xn2, g2, k2 = _run_fwd(cuda_lib, FORCE_KS2, T, Bp, H, ndir, inputs)
    y4, xn4, g4, k4 = _run_fwd(cuda_lib, 0, T, Bp, H, ndir, inputs)
    assert (k2, k4) == ("ks2", "ks4")
    assert torch.isfinite(y2).all() and torch.isfinite(g2).all()
    # step 0 has no recurrent product: identical
    for d, t in ((0, 0), (1, T - 1)):
        rows = slice(t * Bp, (t + 1) * Bp)
        cols = slice(d * H, (d + 1) * H)
        assert torch.equal(y2[rows, cols], y4[rows, cols])
    for d, t in ((0, 1), (1, T - 2)):
        rows = slice(t * Bp, (t + 1) * Bp)
        cols = slice(d * H, (d + 1) * H)
        assert int(_bf16_ulps(xn2[rows, cols], xn4[rows, cols]).max()) <= 1
        assert (y2[rows, cols] - y4[rows, cols]).abs().max().item() < 1e-5
    assert (y2 - y4).abs().max().item() < 2e-3
    assert (g2 - g4).abs().max().item() < 2e-3


def test_ks2_is_repeatable(cuda_lib):
    """the receiving CTA sums the two halves in rank order: bitwise equal run to run"""
    T, Bp, H, ndir = 247, 64, 1024, 2
    inputs = _fwd_inputs(T, Bp, H, ndir, seed=3)
    a = _run_fwd(cuda_lib, FORCE_KS2, T, Bp, H, ndir, inputs)
    b = _run_fwd(cuda_lib, FORCE_KS2, T, Bp, H, ndir, inputs)
    assert a[3] == b[3] == "ks2"
    assert torch.isfinite(a[0]).all()
    for u, v in zip(a[:3], b[:3]):
        assert torch.equal(u, v)


def test_ks2_against_plain_kernel_at_benchmark_shape(cuda_lib):
    """the default selection vs the plain kernel (flag 32) on the same inputs"""
    T, Bp, H, ndir = 247, 64, 1024, 2
    inputs = _fwd_inputs(T, Bp, H, ndir, seed=4)
    new = _run_fwd(cuda_lib, FORCE_KS2, T, Bp, H, ndir, inputs)
    old = _run_fwd(cuda_lib, NO_KSPLIT, T, Bp, H, ndir, inputs)
    assert (new[3], old[3]) == ("ks2", "plain")
    assert (new[0] - old[0]).abs().max().item() < 2e-3
    assert (new[2] - old[2]).abs().max().item() < 2e-3


@pytest.mark.parametrize("Bp,H,flags,expect", [
    (64, 1024, 0, "ks2"),             # the benchmark shape: 4-CTA clusters do not fit
    (32, 1024, 0, "ks2"),
    (72, 1024, 0, "plain"),           # above 64 rows
    (64, 1024, NO_KSPLIT, "plain"),
    (64, 512, 0, "ks4"),              # 4-CTA clusters fit
    (64, 384, 0, "plain"),            # below H = 512 the 2-CTA split does not pay
    (64, 384, FORCE_KS2, "ks2"),
])
def test_forward_kernel_selection(cuda_lib, Bp, H, flags, expect):
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("selection figures are for a 132-SM H100")
    T, ndir = 6, 2
    out = _run_fwd(cuda_lib, flags, T, Bp, H, ndir, _fwd_inputs(T, Bp, H, ndir, seed=Bp + H))
    assert out[3] == expect
    assert torch.isfinite(out[0]).all()
