"""GPU tests of the staged epilogue of the 128 x 256 GEMM kernel over 2-CTA clusters.

By default gemm_bf16_tn_c2_kernel writes its output tiles through shared memory with TMA bulk
tensor stores (reduce-adds for accumulating launches with one writer per tile); developer flag 2
of sb_debug_gemm_flags makes it store straight from the registers, as every other path does.
Only the store changes, not the sums, so both must agree bit for bit wherever each output element
is written once.  sb_debug_gemm_epilogue says which epilogue the last launch used.
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REGS = 2
NO_STORES = 4


def _run(flags, fn):
    from speech_b200 import _lib
    lib = _lib.load()
    lib.sb_debug_gemm_flags(flags)
    try:
        out = fn()
        torch.cuda.synchronize()
        return out, lib.sb_debug_gemm_kernel().decode(), lib.sb_debug_gemm_epilogue().decode()
    finally:
        lib.sb_debug_gemm_flags(0)


def _operands(M, N, K, a_mn, b_mn, seed):
    """bf16 A [M][K], B [N][K] and, for MN-major operands, strided [K][MN] views of wider matrices
    holding the same values (as the weight-gradient call sites pass them)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    B = torch.randn(N, K, device="cuda", generator=g).bfloat16()
    a, b = A, B
    if a_mn:
        At = torch.zeros(K, (M + 7) // 8 * 8 + 16, device="cuda", dtype=torch.bfloat16)
        At[:, 8:8 + M] = A.t()
        a = At[:, 8:8 + M]
    if b_mn:
        Bt = torch.zeros(K, (N + 7) // 8 * 8 + 32, device="cuda", dtype=torch.bfloat16)
        Bt[:, 8:8 + N] = B.t()
        b = Bt[:, 8:8 + N]
    return A, B, a, b


@pytest.mark.parametrize("M,N,K,a_mn,b_mn,bias", [
    (15808, 6144, 2048, False, False, True),    # gi = X W_ih^T + b, layers 1-4
    (15808, 6144, 480, False, False, True),     # gi, layer 0 (K % 64 != 0)
    (15808, 2048, 6144, False, True, False),    # dX = dgi W_ih
    (15808, 480, 6144, False, True, False),     # dX, layer 0 (N % 32 == 0, N % 256 != 0)
    (15808, 2048, 32, False, False, False),     # fc dY
    (237120, 1280, 32, False, True, False),     # conv2 patch gradient dA
    (300, 200, 1000, False, False, True),       # odd M-tile count, N < 256, K % 64 != 0
    (300, 200, 1000, True, False, False),
    (300, 200, 1000, False, True, True),
    (300, 200, 1000, True, True, False),
    (640, 300, 72, True, True, True),           # 5 M tiles, 2 N tiles (the second mostly empty)
    (129, 130, 64, False, False, False),        # one row past a tile, two past 128 columns
    (200, 1001, 104, False, False, True),       # N odd: a ragged last staging box
])
def test_tma_store_bit_identical_to_register_epilogue(cuda_lib, M, N, K, a_mn, b_mn, bias):
    from speech_b200 import ops
    A, B, a, b = _operands(M, N, K, a_mn, b_mn, M + N + K)
    bvec = torch.randn(N, device="cuda") if bias else None
    # N odd leaves a row pitch the tensor map cannot take: give that case a padded output view
    pitch = (N + 3) // 4 * 4

    def go():
        out = torch.full((M, pitch), float("nan"), device="cuda")[:, :N]
        return ops.gemm_bf16_tn(a, b, out=out, bias=bvec, a_mn=a_mn, b_mn=b_mn)
    new, kn, en = _run(0, go)
    old, ko, eo = _run(REGS, go)
    assert (kn, en) == ("c2_128x256", "tma")
    assert (ko, eo) == ("c2_128x256", "regs")
    assert torch.equal(new, old)
    if M * N <= 1 << 26:
        f32 = A.float() @ B.float().t() + (0 if bvec is None else bvec)
        assert ((new - f32).abs().max() / f32.abs().max()).item() < 1e-4


@pytest.mark.parametrize("col_off,pitch_pad,epilogue", [
    (0, 4, "tma"),       # row pitch N + 4 floats: 16-byte multiple
    (4, 12, "tma"),      # view starting 16 bytes into the row
    (0, 3, "regs"),      # row pitch not a multiple of 16 bytes: register epilogue
    (1, 7, "regs"),      # base not 16-byte aligned: register epilogue
])
def test_strided_output_views(cuda_lib, col_off, pitch_pad, epilogue):
    """out is a column slice of a wider matrix; the columns around it stay untouched"""
    from speech_b200 import ops
    M, N, K = 700, 520, 200
    A, B, a, b = _operands(M, N, K, False, False, 11)
    bvec = torch.randn(N, device="cuda")
    outs = {}
    for flags in (0, REGS):
        big = torch.full((M, N + pitch_pad), -7.0, device="cuda")
        view = big[:, col_off:col_off + N]
        _, kn, en = _run(flags, lambda: ops.gemm_bf16_tn(a, b, out=view, bias=bvec))
        assert kn == "c2_128x256"
        assert en == (epilogue if flags == 0 else "regs")
        outs[flags] = big
    assert torch.equal(outs[0], outs[REGS])
    big = outs[0]
    assert (big[:, :col_off] == -7.0).all() and (big[:, col_off + N:] == -7.0).all()
    ref = A.float() @ B.float().t() + bvec
    assert ((big[:, col_off:col_off + N] - ref).abs().max() / ref.abs().max()).item() < 1e-4


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [
    (6144, 2048, 15808, True, True),    # dW_ih of both directions in one launch
    (4096, 2048, 256, True, True),
    (1024, 768, 512, False, False),
    (640, 300, 72, True, True),         # ragged N, odd M-tile count
])
def test_tma_reduce_bit_identical_to_atomics_one_writer_per_tile(cuda_lib, M, N, K, a_mn, b_mn):
    """accumulating launches the library runs without a K split: one add per element either way"""
    from speech_b200 import ops
    A, B, a, b = _operands(M, N, K, a_mn, b_mn, M + K)
    C0 = torch.randn(M, N, device="cuda")
    new, kn, en = _run(0, lambda: ops.gemm_bf16_tn(a, b, out=C0.clone(), accumulate=True,
                                                   a_mn=a_mn, b_mn=b_mn))
    old, _, eo = _run(REGS, lambda: ops.gemm_bf16_tn(a, b, out=C0.clone(), accumulate=True,
                                                     a_mn=a_mn, b_mn=b_mn))
    assert (kn, en, eo) == ("c2_128x256", "tma_reduce", "regs")
    assert torch.equal(new, old)
    ref = C0 + A.float() @ B.float().t()
    assert ((new - ref).abs().max() / ref.abs().max()).item() < 1e-4


def test_merged_dwih_into_flat_gradient_buffer(cuda_lib):
    """the two-direction dW_ih view into a flat gradient buffer (other parameters around it)"""
    from speech_b200 import ops
    M, K3, D = 15808, 3072, 2048
    g = torch.Generator(device="cuda").manual_seed(5)
    dgi = torch.randn(M, 2 * K3, device="cuda", generator=g).bfloat16()
    X = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    off = 4 * 1000 + 1024
    flat0 = torch.randn(off + 2 * K3 * D + 4096, device="cuda", generator=g)
    outs = {}
    for flags in (0, REGS):
        flat = flat0.clone()
        view = flat[off:off + 2 * K3 * D].view(2 * K3, D)
        _, _, e = _run(flags, lambda: ops.gemm_bf16_tn(dgi, X, out=view, accumulate=True,
                                                       a_mn=True, b_mn=True))
        assert e == ("tma_reduce" if flags == 0 else "regs")
        outs[flags] = flat
    assert torch.equal(outs[0], outs[REGS])
    assert torch.equal(outs[0][:off], flat0[:off])
    assert torch.equal(outs[0][off + 2 * K3 * D:], flat0[off + 2 * K3 * D:])


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [
    (3072, 2048, 15808, True, True),    # dW_ih per direction
    (2048, 1024, 15744, True, True),    # dW_hh (r,z rows)
    (600, 700, 5000, False, False),     # ragged M, N, K; odd M-tile count
])
def test_split_k_accumulate_matches_fp32_reference(cuda_lib, M, N, K, a_mn, b_mn):
    """split-K launches: several CTAs add into one tile, from the registers (atomic adds)"""
    from speech_b200 import ops
    A, B, a, b = _operands(M, N, K, a_mn, b_mn, M + K)
    C0 = torch.randn(M, N, device="cuda")
    C, kn, en = _run(0, lambda: ops.gemm_bf16_tn(a, b, out=C0.clone(), accumulate=True,
                                                 a_mn=a_mn, b_mn=b_mn))
    assert (kn, en) == ("c2_128x256", "regs")
    ref = C0 + A.float() @ B.float().t()
    assert ((C - ref).abs().max() / ref.abs().max()).item() < 1e-4


@pytest.mark.parametrize("case,flags,kernel,epilogue", [
    ("plain", 0, "c2_128x256", "tma"),
    ("plain", REGS, "c2_128x256", "regs"),
    ("plain", NO_STORES, "c2_128x256", "skipped"),
    ("plain", 1, "128x128", "regs"),
    ("narrow", 0, "128x128", "regs"),
    ("remap", 0, "c2_128x256", "regs"),
    ("acc", 0, "c2_128x256", "tma_reduce"),
    ("acc_split", 0, "c2_128x256", "regs"),
])
def test_epilogue_report(cuda_lib, case, flags, kernel, epilogue):
    from speech_b200 import ops
    N = 128 if case == "narrow" else 512
    K = 15808 if case == "acc_split" else 128
    _, _, a, b = _operands(512, N, K, False, False, 1)
    if case == "remap":
        fn = lambda: ops.gemm_bf16_tn(a, b, remap=(8, 64, 5))          # noqa: E731
    elif case.startswith("acc"):
        fn = lambda: ops.gemm_bf16_tn(a, b, out=torch.zeros(512, N, device="cuda"),  # noqa: E731
                                      accumulate=True)
    else:
        fn = lambda: ops.gemm_bf16_tn(a, b)                              # noqa: E731
    _, k, e = _run(flags, fn)
    assert (k, e) == (kernel, epilogue)


def test_northstar_forward_bit_identical_under_both_epilogues(cuda_lib):
    """the north-star CTC model at seed 0: logits and loss of one forward pass are bitwise equal"""
    sys.path.insert(0, ROOT)
    import bench
    from speech_b200.models import CTC
    torch.manual_seed(0)
    m = CTC(bench.F_IN, bench.VOCAB, bench.MODEL_CFG).cuda()
    m.set_eval()
    inputs, labels = bench.synth_batch(8)
    batch = (tuple(inputs), tuple(labels))
    out = {}
    for flags in (0, REGS):
        with torch.no_grad():
            out[flags] = _run(flags, lambda: (m(batch), m.loss(batch)))[0]
    assert torch.equal(out[0][0], out[REGS][0])
    assert torch.equal(out[0][1], out[REGS][1])
