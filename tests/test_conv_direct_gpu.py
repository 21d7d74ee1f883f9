"""GPU parity of the direct-convolution kernels (sb_conv_fwd_direct, sb_conv_dgrad_direct,
sb_conv_wgrad_direct) that run the conv layers past the first without a patch matrix.

They stage their operands exactly as im2col does (ReLU, dropout, bf16), so against the im2col path
(SB_CONV_FLAGS=1, here ops._conv_flags = 1) the outputs may differ only by fp32 summation order and
the gradients by that plus the bf16 rounding of the backward operands it can flip.  They are also
held to the fp64 rounded-operand reference of test_conv_gpu.py, and their forward must be bitwise
independent of the batch and of the length (the streaming recognisers compare chunked and whole
runs of the conv stack)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _build(specs, in_c=1, p=0.0):
    layers = []
    for out_c, h, w, s in specs:
        layers += [torch.nn.Conv2d(in_c, out_c, (h, w), stride=(s, s)), torch.nn.ReLU()]
        if p > 0.0:
            layers.append(torch.nn.Dropout(p))
        in_c = out_c
    return torch.nn.Sequential(*layers)


def _run(ops, conv, x, wgt, flags, training=True, seed=7):
    """conv_stack forward + backward with SB_CONV_FLAGS = flags -> (y, grads, launched kernels)"""
    ops._ensure_knobs()
    old = ops._conv_flags
    ops._conv_flags = flags
    try:
        for q in conv.parameters():
            q.grad = None
        torch.manual_seed(seed)
        ops.profile_begin()
        y = ops.conv_stack(x, conv, training)
        (y * wgt).sum().backward()
        names = set(ops.profile_end())
    finally:
        ops._conv_flags = old
    return y.detach(), {n: q.grad.clone() for n, q in conv.named_parameters()}, names


DIRECT = {"conv_fwd_direct", "conv_dgrad_direct", "conv_wgrad_direct"}


@pytest.mark.parametrize("specs,B,T,F,p", [
    ([[32, 5, 8, 2], [32, 5, 8, 2]], 4, 1000, 80, 0.0),     # the benchmark's stack
    ([[16, 3, 4, 1], [8, 2, 3, 3]], 2, 33, 21, 0.0),         # stride 3, 2 x 3 taps, Co = 8
    ([[8, 5, 8, 2], [8, 5, 8, 2]], 3, 61, 80, 0.0),          # Ci = 8: k-chunks span two taps
    ([[8, 7, 12, 1], [8, 6, 11, 2]], 2, 40, 48, 0.0),        # 66 taps, odd K / 16
    ([[16, 5, 8, 2], [24, 3, 4, 1], [32, 3, 3, 2]], 2, 70, 40, 0.3),   # dropout, three layers
])
def test_direct_matches_im2col(cuda_lib, specs, B, T, F, p):
    from speech_b200 import ops
    torch.manual_seed(B + T + F)
    conv = _build(specs, p=p).cuda()
    x = torch.randn(B, T, F, device="cuda")
    y0, g0, n0 = _run(ops, conv, x, 1.0, 1)
    wgt = torch.randn_like(y0)
    y0, g0, n0 = _run(ops, conv, x, wgt, 1)
    y1, g1, n1 = _run(ops, conv, x, wgt, 0)
    assert not (n0 & DIRECT)
    assert DIRECT <= n1 and "conv_col2im_relu" not in n1
    # two layers: the direct layer's operands are bit-identical, only the fp32 order differs;
    # deeper, that reordering can flip the bf16 rounding of a later layer's operand
    scale = y0.abs().max().item()
    assert (y1 - y0).abs().max().item() <= (1e-5 if len(specs) == 2 else 1e-3) * scale
    for n in g0:
        ref = g0[n].double()
        err = (g1[n].double() - ref).abs().max().item()
        assert err <= 3e-2 * ref.abs().max().item() + 1e-4, (n, err, ref.abs().max().item())


@pytest.mark.parametrize("specs,B,T,F,p", [
    ([[32, 5, 8, 2], [32, 5, 8, 2]], 2, 90, 80, 0.0),
    ([[16, 3, 4, 1], [8, 2, 3, 3]], 2, 33, 21, 0.0),
    ([[8, 5, 8, 2], [16, 3, 4, 1]], 3, 61, 40, 0.4),
])
def test_direct_matches_rounded_fp64_reference(cuda_lib, specs, B, T, F, p):
    """test_conv_gpu.py's reference: torch conv2d in fp64 on operands rounded to bf16 where the
    kernels round them (straight-through gradients), dropout masks drawn in the same order."""
    from speech_b200 import ops
    torch.manual_seed(3 + B + T)
    conv = _build(specs, p=p).cuda()
    x = torch.randn(B, T, F, device="cuda")
    y, _, _ = _run(ops, conv, x, 1.0, 0, seed=99)
    wgt = torch.randn_like(y)
    y, got, names = _run(ops, conv, x, wgt, 0, seed=99)
    assert DIRECT <= names

    def rnd(t):
        return t + (t.detach().float().bfloat16().double() - t.detach())

    torch.manual_seed(99)
    params = {n: q.detach().double().requires_grad_(True) for n, q in conv.named_parameters()}
    mods = [(i, m) for i, m in enumerate(conv) if isinstance(m, torch.nn.Conv2d)]
    h = rnd(x.double().unsqueeze(1))
    for li, (i, m) in enumerate(mods):
        pre = torch.nn.functional.conv2d(h, rnd(params["%d.weight" % i]), params["%d.bias" % i],
                                         stride=m.stride)
        h = torch.relu(pre)
        if p > 0.0:
            b, c, t, f = pre.shape
            mask = (torch.rand(b * t * f, c, device="cuda") >= p).double() / (1.0 - p)
            h = h * mask.view(b, t, f, c).permute(0, 3, 1, 2)
        if li + 1 < len(mods):
            h = rnd(h)
    b, c, t, f = h.shape
    y64 = h.transpose(1, 2).reshape(b, t, c * f)
    (y64 * wgt.double()).sum().backward()
    if p > 0.0:
        assert (y == 0).float().mean().item() > p * 0.8
    scale = y64.abs().max().item()
    assert (y.double() - y64).abs().max().item() < 2e-3 * scale
    for n, q in params.items():
        err = (got[n].double() - q.grad).abs().max().item()
        assert err < 3e-2 * q.grad.abs().max().item() + 1e-4, (n, err)


def test_domain_and_fallback(cuda_lib):
    """The benchmark's second layer runs direct; the TIMIT recipe's [32, 5, 32, 1] second layer
    (32 x 5120 bf16 of weights, 320 KB) does not fit and stays on im2col + GEMM."""
    from speech_b200 import ops
    assert ops.conv_direct_ok(37, 32, 32, 5, 8, 2)
    assert not ops.conv_direct_ok(65, 32, 32, 5, 32, 1)
    torch.manual_seed(0)
    conv = _build([[32, 5, 32, 2], [32, 5, 32, 1]]).cuda()
    x = torch.randn(2, 60, 161, device="cuda")
    y, _, names = _run(ops, conv, x, 1.0, 0)
    assert not (names & DIRECT) and "conv_col2im_relu" in names


def test_forward_bitwise_invariant_to_batch_and_length(cuda_lib):
    from speech_b200 import ops
    torch.manual_seed(1)
    conv = _build([[32, 5, 8, 2], [32, 5, 8, 2]]).cuda()
    x = torch.randn(8, 400, 80, device="cuda")
    with torch.no_grad():
        y8 = ops.conv_stack(x, conv, False)
        y1 = ops.conv_stack(x[5:6].contiguous(), conv, False)
        ys = ops.conv_stack(x[:, :157].contiguous(), conv, False)
        again = ops.conv_stack(x, conv, False)
    assert torch.equal(y8, again)
    assert torch.equal(y8[5:6], y1)
    assert torch.equal(y8[:, :ys.shape[1]], ys)


def test_no_patch_matrix_allocated(cuda_lib):
    """One forward + backward at the benchmark's conv shape (B = 64, T = 1000): the direct path
    allocates neither the [237120][1280] bf16 patch matrix (607 MB) nor its fp32 gradient."""
    from speech_b200 import ops
    torch.manual_seed(2)
    conv = _build([[32, 5, 8, 2], [32, 5, 8, 2]]).cuda()
    x = torch.randn(64, 1000, 80, device="cuda")
    peaks = {}
    for flags in (1, 0):
        ops._ensure_knobs()
        old = ops._conv_flags
        ops._conv_flags = flags
        try:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            y = ops.conv_stack(x, conv, True)
            y.sum().backward()
            torch.cuda.synchronize()
            peaks[flags] = torch.cuda.max_memory_allocated() - base
            del y
        finally:
            ops._conv_flags = old
    assert peaks[1] - peaks[0] > 1.0e9, peaks
