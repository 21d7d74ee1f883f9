"""GPU parity of every GRU recurrence kernel with the rounding-faithful reference (tests/gru_ref.py).

sb_gru_fwd / sb_gru_bwd are called directly through the C ABI, each case pinned to the kernel
variant it must run (sb_debug_gru_fwd_kernel / sb_debug_gru_bwd_kernel), forced where needed with
the developer knobs.  The reference applies the kernels' bf16 roundings and is teacher-forced by
the kernels' own states, so what is compared is the fp32 error of one step, and the bars of
gru_ref (set by an fp32 emulation, two orders of magnitude under the smallest planted fault) are
100x tighter than those of the fp64 nn.GRU parity tests:
  forward   y and the saved gates within FWD_ABS; xn == bf16(y) bitwise; a second call on the
            same workspace gives the same bits;
  backward  fed the reference's y and gates and a random dy: dgi and dghn within one bf16 ulp of
            the reference plus BWD_FLOOR of the largest entry; the bias gradients, added to
            non-zero contents, within DB_REL of the largest entry.
Inputs: W_hh, b_hh ~ U(+-g/sqrt(H)) with gains 1 and 3 (3 saturates the gates), gi ~ N(0, 1) on
every row of the padded batch.  sb_gru_fwd_f32, the fp32 parity-mode recurrence, is held to the
unrounded reference within F32_ABS.
"""
import ctypes

import pytest
import torch

import gru_ref as R

gpu = pytest.mark.gpu

FWD_KERNELS = ("plain", "kt", "ks4", "ks2", "wide")
BWD_KERNELS = ("plain", "kt", "ks4", "ks_l2", "ks4_x2", "wide")
# developer flags of sb_debug_gru_flags
NO_KT, KT, NO_KS_FWD, L2RS, NO_L2RS, KS2, STREAM = 8, 16, 32, 256, 512, 1024, 2048

# id: (T, Bp, H, ndir, flags, K-split backward on, forward kernel, backward kernel, selection is
# that of a 132-SM H100).  H is the width the kernels run (gru_padded_width of the layer's).
CASES = {
    "t1_uni": (1, 8, 64, 1, 0, 1, "plain", "plain", False),
    "t1_bi": (1, 8, 256, 2, 0, 1, "kt", "ks4", False),
    "t2_uni": (2, 16, 128, 1, 0, 1, "plain", "plain", False),
    "t2_bi": (2, 24, 256, 2, 0, 1, "ks4", "ks4", False),
    "smallest_uni": (5, 8, 16, 1, 0, 1, "plain", "plain", False),
    "smallest_bi": (5, 8, 16, 2, 0, 1, "plain", "plain", False),
    "bp128": (9, 128, 256, 2, 0, 1, "plain", "ks4", False),
    "bp128_plain_bwd": (9, 128, 256, 2, 0, 0, "plain", "plain", False),
    "kt_bp8": (12, 8, 256, 2, KT, 1, "kt", "kt", False),
    "kt_bp24": (12, 24, 256, 2, KT, 1, "kt", "kt", False),
    "kt_bp56": (12, 56, 256, 2, KT, 1, "kt", "kt", False),
    "ks4_h512": (20, 64, 512, 2, 0, 1, "ks4", "ks4", False),
    "bench": (247, 64, 1024, 2, 0, 1, "ks2", "ks_l2", True),
    "bench_ks4_x2": (247, 64, 1024, 2, NO_L2RS, 1, "ks2", "ks4_x2", True),
    "ks_l2_h256": (15, 32, 256, 2, L2RS, 1, "ks4", "ks_l2", False),
    "ks_l2_h512": (15, 16, 512, 2, L2RS, 1, "kt", "ks_l2", False),
    "resident_ceiling": (8, 32, 1056, 2, 0, 1, "plain", "plain", True),
    "wide_h1152_bp128": (6, 128, 1152, 2, 0, 1, "wide", "wide", True),
    "wide_h1280_bp8": (6, 8, 1280, 2, 0, 1, "wide", "wide", True),
    "wide_uni_h2128": (6, 64, 2144, 1, 0, 1, "wide", "wide", True),   # H = 2128 runs at 2144
    "streamed_h256": (10, 64, 256, 2, STREAM, 1, "wide", "wide", False),
}


def test_cases_name_every_kernel():
    assert {c[6] for c in CASES.values()} >= set(FWD_KERNELS)
    assert {c[7] for c in CASES.values()} >= set(BWD_KERNELS)
    assert {c[6] for c in CASES.values()} <= set(FWD_KERNELS)
    assert {c[7] for c in CASES.values()} <= set(BWD_KERNELS)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(T, Bp, H, ndir, gain, seed):
    g = torch.Generator().manual_seed(seed)
    a = gain / H ** 0.5
    whh = ((torch.rand(ndir, 3 * H, H, generator=g) * 2 - 1) * a).to(torch.bfloat16)
    bhh = (torch.rand(ndir, 3 * H, generator=g) * 2 - 1) * a
    gi = torch.randn(T * Bp, ndir * 3 * H, generator=g)
    dy = torch.randn(T * Bp, ndir * H, generator=g)
    return gi, whh, bhh, dy


def _workspace(lib, query, Bp, H, ndir):
    from speech_b200 import _lib, ops
    n = ctypes.c_size_t(0)
    _lib.check(query(Bp, H, ndir, ctypes.byref(n)), "workspace size")
    return ops._workspace(n.value, "cuda"), n.value


def _run_fwd(lib, T, Bp, H, ndir, gi, whh, bhh, ws, nws):
    from speech_b200 import _lib
    D = ndir * H
    y = torch.full((T * Bp, D), float("nan"), device="cuda")
    xn = torch.zeros(T * Bp, D, dtype=torch.bfloat16, device="cuda")
    gates = torch.full((T * Bp, ndir, 4, H), float("nan"), device="cuda")
    _lib.check(lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), y.data_ptr(),
                              xn.data_ptr(), gates.data_ptr(), ws.data_ptr(), nws, T, Bp, H, ndir,
                              _lib.stream_ptr()), "sb_gru_fwd")
    torch.cuda.synchronize()
    return y, xn, gates


def _run_bwd(lib, T, Bp, H, ndir, dy, y, gates, whh, dbias, ws, nws):
    from speech_b200 import _lib
    dgi = torch.zeros(T * Bp, ndir * 3 * H, dtype=torch.bfloat16, device="cuda")
    dghn = torch.zeros(T * Bp, ndir * H, dtype=torch.bfloat16, device="cuda")
    dbih, dbhh = dbias[0].clone(), dbias[1].clone()
    _lib.check(lib.sb_gru_bwd(dy.data_ptr(), y.data_ptr(), gates.data_ptr(), whh.data_ptr(),
                              dgi.data_ptr(), dghn.data_ptr(), dbih.data_ptr(), dbhh.data_ptr(),
                              ws.data_ptr(), nws, T, Bp, H, ndir, _lib.stream_ptr()), "sb_gru_bwd")
    torch.cuda.synchronize()
    return dgi, dghn, dbih, dbhh


@gpu
@pytest.mark.parametrize("gain", [1, 3])
@pytest.mark.parametrize("case", list(CASES))
def test_kernel_matches_rounded_reference(cuda_lib, case, gain):
    T, Bp, H, ndir, flags, ksplit, fwd_kernel, bwd_kernel, h100 = CASES[case]
    if h100 and _sms() != 132:
        pytest.skip("selection figures are for a 132-SM H100")
    lib = cuda_lib
    gi, whh, bhh, dy = _inputs(T, Bp, H, ndir, gain, seed=T + Bp + H + gain)
    gi_c, whh_c, bhh_c, dy_c = gi.cuda(), whh.cuda(), bhh.cuda(), dy.cuda()
    g = torch.Generator().manual_seed(gain)
    prefill = [torch.randn(ndir * 3 * H, generator=g) for _ in range(2)]
    lib.sb_debug_gru_flags(flags)
    lib.sb_debug_gru_ksplit(ksplit)
    try:
        # the knobs change the workspace the selected kernels need
        fws, nf = _workspace(lib, lib.sb_gru_fwd_workspace_size, Bp, H, ndir)
        bws, nb = _workspace(lib, lib.sb_gru_bwd_workspace_size, Bp, H, ndir)
        y, xn, gates = _run_fwd(lib, T, Bp, H, ndir, gi_c, whh_c, bhh_c, fws, nf)
        assert lib.sb_debug_gru_fwd_kernel().decode() == fwd_kernel
        again = _run_fwd(lib, T, Bp, H, ndir, gi_c, whh_c, bhh_c, fws, nf)
        # the backward's inputs: the reference's own states (teacher-forced by the kernel's y)
        ry, rg, _ = R.gru_fwd(gi, whh, bhh, T, h_prev=y)
        ry32, rg32 = ry.float(), rg.float()
        pre = [p.cuda() for p in prefill]
        out = _run_bwd(lib, T, Bp, H, ndir, dy_c, ry32.cuda(), rg32.cuda(), whh_c, pre, bws, nb)
        assert lib.sb_debug_gru_bwd_kernel().decode() == bwd_kernel
        out2 = _run_bwd(lib, T, Bp, H, ndir, dy_c, ry32.cuda(), rg32.cuda(), whh_c, pre, bws, nb)
    finally:
        lib.sb_debug_gru_flags(0)
        lib.sb_debug_gru_ksplit(1)
    # forward
    assert torch.equal(xn, y.to(torch.bfloat16))
    for a, b in zip((y, xn, gates), again):
        assert torch.equal(a, b)
    err = R.fwd_err(y, gates, ry, rg)
    print("\n%s gain %d fwd %s: fwd_err %.2e (bar %.0e)" % (case, gain, fwd_kernel, err, R.FWD_ABS))
    assert err < R.FWD_ABS, err
    # backward
    assert torch.equal(out[0], out2[0]) and torch.equal(out[1], out2[1])
    got = (out[0].cpu(), out[1].cpu(), out[2].cpu().double() - prefill[0].double(),
           out[3].cpu().double() - prefill[1].double())
    ref = R.gru_bwd(dy, ry32, rg32, whh, T, xr=got[:2])
    elem, bias = R.bwd_errs(got, ref)
    print("%s gain %d bwd %s: dgi/dghn beyond 1 ulp %.2e (bar %.0e), bias %.2e (bar %.0e)"
          % (case, gain, bwd_kernel, elem, R.BWD_FLOOR, bias, R.DB_REL))
    assert elem < R.BWD_FLOOR, elem
    assert bias < R.DB_REL, bias


# ---- the fp32 parity-mode recurrence ----------------------------------------------------------------
@gpu
@pytest.mark.parametrize("T,Bp,H,ndir", [
    (9, 8, 20, 2),         # H % 8 != 0: the last CTA holds 4 units
    (9, 8, 20, 1),
    (7, 72, 64, 2),        # rows b and b + 64 in one thread, the second half partial
    (7, 128, 32, 1),
    (247, 64, 1024, 2),    # the benchmark's width and length
])
@pytest.mark.parametrize("gain", [1, 3])
def test_f32_recurrence_matches_unrounded_reference(cuda_lib, T, Bp, H, ndir, gain):
    from speech_b200 import _lib
    if (H + 7) // 8 > _sms():
        pytest.skip("one CTA of 8 units per SM")
    gi, whh, bhh, _ = _inputs(T, Bp, H, ndir, gain, seed=T + Bp + H + gain)
    whh = whh.float() + (torch.rand(whh.shape) - 0.5) * (gain / H ** 0.5) * 2 ** -8   # not bf16
    y = torch.full((T * Bp, ndir * H), float("nan"), device="cuda")
    barrier = torch.zeros(2, dtype=torch.int32, device="cuda")
    gi_c, w_c, b_c = gi.cuda(), whh.cuda(), bhh.cuda()
    _lib.check(cuda_lib.sb_gru_fwd_f32(gi_c.data_ptr(), w_c.data_ptr(), b_c.data_ptr(),
                                       y.data_ptr(), barrier.data_ptr(), T, Bp, H, ndir,
                                       _lib.stream_ptr()), "sb_gru_fwd_f32")
    torch.cuda.synchronize()
    ry, _, _ = R.gru_fwd(gi, whh, bhh, T, rounded=False, h_prev=y)
    err = (y.cpu().double() - ry).abs().max().item()
    print("\nf32 T %d Bp %d H %d ndir %d gain %d: %.2e (bar %.0e)" % (T, Bp, H, ndir, gain, err,
                                                                    R.F32_ABS))
    assert err < R.F32_ABS, err


# ---- the stack: ops.gru_stack, glue included ----------------------------------------------------------
@gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_stack_matches_rounded_reference(cuda_lib, seed):
    """2-layer biGRU at H = 250 (the kernels run Hp = 256 with zero units, pad_gru_layer) in the
    exact-lengths mode (the reverse direction on right-aligned frames, time_align), against
    gru_ref.gru_stack at the layer's own width: gi from bf16 X and W_ih, the dW_hh operands
    shifted by Bp rows (one way per direction), bf16 dgi / dghn into dW and dx."""
    from speech_b200 import ops
    torch.manual_seed(seed)
    lens = [24, 9, 1, 17, 24, 12, 5]
    B, T, In, H = len(lens), max(lens), 40, 250
    assert ops.gru_padded_width(8, H, 2) == 256
    rnn = torch.nn.GRU(In, H, 2, batch_first=True, bidirectional=True)
    x = torch.randn(B, T, In)
    dout = torch.randn(B, T, 2 * H)
    ry, rdx, rgrads = R.gru_stack(x, list(rnn.parameters()), 2, dout, lens)
    rnn_c = rnn.cuda()
    xc = x.cuda().requires_grad_(True)
    y = ops.gru_stack(xc, rnn_c, lens=lens)
    (y * dout.cuda()).sum().backward()
    torch.cuda.synchronize()
    ey = (y.detach().cpu().double() - ry).abs().max().item()
    errs = {"dx": R.rel_err(xc.grad, rdx)}
    errs.update({n: R.rel_err(p.grad, g) for (n, p), g in zip(rnn_c.named_parameters(), rgrads)})
    print("\nstack seed %d: y %.2e (bar %.0e), worst gradient %s %.2e (bar %.0e)"
          % (seed, ey, R.STACK_Y_ABS, max(errs, key=errs.get), max(errs.values()),
             R.STACK_GRAD_REL))
    assert ey < R.STACK_Y_ABS, ey
    for n, e in errs.items():
        assert e < R.STACK_GRAD_REL, (n, e)
