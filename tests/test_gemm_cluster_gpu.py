"""GPU tests of the 128 x 256 GEMM kernel over 2-CTA clusters (gemm_bf16_tn_c2_kernel).

sb_gemm_bf16_tn runs every GEMM with N > 128 on it; developer flag 1 of sb_debug_gemm_flags
selects the 128 x 128 one-CTA kernel instead, and sb_debug_gemm_kernel says which kernel the last
launch used.  Both kernels give every output element the same fp32 sum (one accumulator, k-blocks
ascending, the same k16 wgmma steps), so non-accumulating launches must agree bit for bit.
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEGACY = 1


def _run(flags, fn):
    from speech_b200 import _lib
    lib = _lib.load()
    lib.sb_debug_gemm_flags(flags)
    try:
        out = fn()
        torch.cuda.synchronize()
        return out, lib.sb_debug_gemm_kernel().decode()
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
    (15808, 480, 6144, False, True, False),     # dX, layer 0 (N % 256 != 0)
    (3072, 2048, 15808, True, True, False),     # dW_ih shape, not accumulating
    (2048, 1024, 15744, True, True, False),     # dW_hh (r,z rows) shape
    (300, 200, 1000, False, False, True),       # odd M-tile count, N < 256, K % 64 != 0
    (300, 200, 1000, True, False, False),
    (300, 200, 1000, False, True, True),
    (300, 200, 1000, True, True, False),
    (640, 300, 72, True, True, True),           # 5 M tiles, 2 N tiles (the second mostly empty)
    (129, 130, 64, False, False, False),        # one row past a tile, two past 128 columns
])
def test_c2_bit_identical_to_legacy(cuda_lib, M, N, K, a_mn, b_mn, bias):
    from speech_b200 import ops
    A, B, a, b = _operands(M, N, K, a_mn, b_mn, M + N + K)
    bvec = torch.randn(N, device="cuda") if bias else None
    new, kn = _run(0, lambda: ops.gemm_bf16_tn(a, b, bias=bvec, a_mn=a_mn, b_mn=b_mn))
    old, ko = _run(LEGACY, lambda: ops.gemm_bf16_tn(a, b, bias=bvec, a_mn=a_mn, b_mn=b_mn))
    assert (kn, ko) == ("c2_128x256", "128x128")
    assert torch.equal(new, old)
    f32 = A.float() @ B.float().t() + (0 if bvec is None else bvec)
    assert ((new - f32).abs().max() / f32.abs().max()).item() < 1e-4


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)])
def test_c2_row_remap_bit_identical_to_legacy(cuda_lib, a_mn, b_mn):
    from speech_b200 import ops
    T, Bp, Bv, K, N = 37, 8, 5, 128, 300
    A, B, a, b = _operands(T * Bp, N, K, a_mn, b_mn, 7)
    bvec = torch.randn(N, device="cuda")

    def go():
        return ops.gemm_bf16_tn(a, b, bias=bvec, remap=(Bp, T, Bv), a_mn=a_mn, b_mn=b_mn)
    new, kn = _run(0, go)
    old, _ = _run(LEGACY, go)
    assert kn == "c2_128x256"
    assert torch.equal(new, old)
    ref = (A.float() @ B.float().t() + bvec).view(T, Bp, N)[:, :Bv].transpose(0, 1)
    assert (new - ref.reshape(Bv * T, N)).abs().max().item() < 2e-2


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [
    (3072, 2048, 15808, True, True),    # dW_ih per direction
    (6144, 2048, 15808, True, True),    # dW_ih of both directions in one launch
    (3072, 480, 15808, True, True),     # layer-0 dW_ih
    (2048, 1024, 15744, True, True),    # dW_hh (r,z rows)
    (1024, 1024, 15744, True, True),    # dW_hh (n rows)
    (600, 700, 5000, False, False),     # ragged M, N, K; odd M-tile count
])
def test_c2_accumulate_matches_fp32_reference(cuda_lib, M, N, K, a_mn, b_mn):
    from speech_b200 import ops
    A, B, a, b = _operands(M, N, K, a_mn, b_mn, M + K)
    C0 = torch.randn(M, N, device="cuda")
    C, kn = _run(0, lambda: ops.gemm_bf16_tn(a, b, out=C0.clone(), accumulate=True,
                                             a_mn=a_mn, b_mn=b_mn))
    assert kn == "c2_128x256"
    ref = C0 + A.float() @ B.float().t()
    assert ((C - ref).abs().max() / ref.abs().max()).item() < 1e-4


def test_merged_two_direction_dwih_matches_per_direction_launches(cuda_lib):
    """dW_ih of both directions as one [6144][2048] launch == two [3072][2048] launches"""
    from speech_b200 import ops
    M, K3, D = 15808, 3072, 2048
    g = torch.Generator(device="cuda").manual_seed(3)
    dgi = torch.randn(M, 2 * K3, device="cuda", generator=g).bfloat16()
    X = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    both = torch.zeros(2 * K3, D, device="cuda")
    ops.gemm_bf16_tn(dgi, X, out=both, accumulate=True, a_mn=True, b_mn=True)
    per = torch.zeros(2 * K3, D, device="cuda")
    for d in range(2):
        ops.gemm_bf16_tn(dgi[:, d * K3:(d + 1) * K3], X, out=per[d * K3:(d + 1) * K3],
                         accumulate=True, a_mn=True, b_mn=True)
    torch.cuda.synchronize()
    assert ((both - per).abs().max() / per.abs().max()).item() < 1e-4


def test_gru_backward_merges_dwih_into_flat_grad_buffer(cuda_lib):
    """With optim.FlatSGD the .grad of both directions' W_ih are adjacent: the GRU backward runs
    dW_ih as one launch per layer, and the gradients equal those of the per-direction path"""
    import numpy as np
    from speech_b200 import ops
    from speech_b200.models import CTC
    from speech_b200.optim import FlatSGD
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                       "rnn": {"dim": 256, "bidirectional": True, "layers": 2}}}
    rng = np.random.RandomState(0)
    inputs = [rng.randn(200 + 5 * i, 80).astype(np.float32) for i in range(8)]
    labels = [rng.randint(0, 28, 10 + i).tolist() for i in range(8)]
    torch.manual_seed(0)
    m = CTC(80, 28, cfg).cuda()
    opt = FlatSGD(m, lr=1e-3)
    names = [n for n, _ in m.named_parameters() if "weight_ih" in n]

    def grads(sink):
        opt.zero_grad()
        ops._grad_sink_enabled = sink
        old_detail = ops._prof_detail
        ops._prof_detail = True
        ops.profile_begin()
        try:
            m.loss((inputs, labels)).backward()
        finally:
            prof = ops.profile_end()
            ops._prof_detail = old_detail
            ops._grad_sink_enabled = True
        p = dict(m.named_parameters())
        return {n: p[n].grad.detach().clone() for n in names}, prof

    merged, prof_m = grads(True)
    per, prof_p = grads(False)
    assert any(k.startswith("gemm 1536x") and k.endswith("aT bT acc") for k in prof_m), prof_m
    assert not any(k.startswith("gemm 1536x") for k in prof_p), prof_p
    for n in names:
        ref = per[n]
        assert ((merged[n] - ref).abs().max() / ref.abs().max()).item() < 1e-4, n


@pytest.mark.parametrize("N,b_mn,flags,kernel", [
    (29, False, 0, "128x32"),
    (64, True, 0, "128x64"),
    (100, False, 0, "128x128"),
    (128, True, 0, "128x128"),
    (129, False, 0, "c2_128x256"),
    (6144, False, 0, "c2_128x256"),
    (6144, True, LEGACY, "128x128"),
    (64, False, LEGACY, "128x64"),
])
def test_kernel_selection(cuda_lib, N, b_mn, flags, kernel):
    from speech_b200 import ops
    _, _, a, b = _operands(256, N, 128, False, b_mn, 1)
    _, k = _run(flags, lambda: ops.gemm_bf16_tn(a, b, b_mn=b_mn))
    assert k == kernel


def test_northstar_forward_bit_identical_under_legacy_and_c2(cuda_lib):
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
    for flags in (0, LEGACY):
        with torch.no_grad():
            out[flags] = _run(flags, lambda: (m(batch), m.loss(batch)))[0]
    assert torch.equal(out[0][0], out[LEGACY][0])
    assert torch.equal(out[0][1], out[LEGACY][1])
