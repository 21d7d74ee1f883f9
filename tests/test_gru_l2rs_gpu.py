"""GPU tests of the L2 reduce-scatter mode of the K-split GRU backward recurrence kernel.

Without a thread-block cluster the four K-quarter partial products of a group of 4 CTAs are
exchanged through a staging area in global memory instead of distributed shared memory; every
owner still adds the four slices in the same order.  So the backward's dgi and dghn must be
BITWISE equal to the clustered launches (at H = 1024 on a 132-SM H100: the two one-direction
launches that developer flag 512 selects; at H = 256 / 512: the both-direction clustered launch).
The bias gradients are summed with atomics in both paths and are compared to 1e-6 relative.
The rest runs the backward with the mode forced (flag 256) at the fp64 `nn.GRU` bars of
test_gru_gpu.py.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

FORCE, DISABLE = 256, 512


def _bwd_inputs(T, Bp, H, ndir, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    D = ndir * H
    dy = torch.randn(T * Bp, D, device=dev, generator=g) * 0.1
    y = torch.rand(T * Bp, D, device=dev, generator=g) * 2 - 1
    gates = torch.rand(T * Bp, ndir, 4, H, device=dev, generator=g)
    gates[:, :, 2] = gates[:, :, 2] * 2 - 1                       # n in (-1, 1)
    gates[:, :, 3] = torch.randn(T * Bp, ndir, H, device=dev, generator=g)
    whh = (torch.randn(ndir, 3 * H, H, device=dev, generator=g) / H ** 0.5).to(torch.bfloat16)
    return dy, y, gates, whh


def _run_bwd(lib, flags, T, Bp, H, ndir, inputs):
    """one sb_gru_bwd call under developer flags -> (dgi, dghn, dbih, dbhh, cluster size used)"""
    from speech_b200 import _lib, ops
    dy, y, gates, whh = inputs
    dgi = torch.empty(T * Bp, ndir * 3 * H, dtype=torch.bfloat16, device="cuda")
    dghn = torch.empty(T * Bp, ndir * H, dtype=torch.bfloat16, device="cuda")
    dbih = torch.zeros(ndir * 3 * H, device="cuda")
    dbhh = torch.zeros(ndir * 3 * H, device="cuda")
    n = ctypes.c_size_t(0)
    _lib.check(lib.sb_gru_bwd_workspace_size(Bp, H, ndir, ctypes.byref(n)), "ws")
    ws = ops._workspace(n.value, "cuda")
    lib.sb_debug_gru_flags(flags)
    try:
        _lib.check(lib.sb_gru_bwd(dy.data_ptr(), y.data_ptr(), gates.data_ptr(), whh.data_ptr(),
                                  dgi.data_ptr(), dghn.data_ptr(), dbih.data_ptr(),
                                  dbhh.data_ptr(), ws.data_ptr(), n.value, T, Bp, H, ndir,
                                  _lib.stream_ptr()), "sb_gru_bwd")
        torch.cuda.synchronize()
        cs = lib.sb_debug_gru_cluster(0)
    finally:
        lib.sb_debug_gru_flags(0)
    return dgi, dghn, dbih, dbhh, cs


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("H,Bp,T,new_flags,old_flags", [
    (1024, 8, 247, 0, DISABLE),       # default selection at H = 1024 vs the two-launch path
    (1024, 32, 247, 0, DISABLE),
    (1024, 64, 247, 0, DISABLE),
    (256, 64, 40, FORCE, 0),          # forced vs the clustered both-direction launch
    (512, 24, 40, FORCE, 0),
])
def test_l2_reduce_scatter_backward_is_bit_identical(cuda_lib, H, Bp, T, new_flags, old_flags):
    inputs = _bwd_inputs(T, Bp, H, 2, seed=H + Bp)
    new = _run_bwd(cuda_lib, new_flags, T, Bp, H, 2, inputs)
    old = _run_bwd(cuda_lib, old_flags, T, Bp, H, 2, inputs)
    assert new[4] == 1 and old[4] == 4, (new[4], old[4])   # no cluster vs 4-CTA clusters
    assert torch.isfinite(new[0].float()).all()
    assert torch.equal(new[0], old[0])                     # dgi
    assert torch.equal(new[1], old[1])                     # dghn
    assert _rel(new[2], old[2]) < 1e-6                     # dbih
    assert _rel(new[3], old[3]) < 1e-6                     # dbhh


def _ref_and_ours_forced(B, T, In, H, L, seed, lens=None):
    """nn.GRU in fp64 on the CPU vs ops.gru_stack with the L2 mode forced (bidirectional)"""
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    from speech_b200 import _lib
    from speech_b200.ops import gru_stack
    torch.manual_seed(seed)
    rnn = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=True)
    x = torch.randn(B, T, In)
    rnn64 = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=True).double()
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
    lib.sb_debug_gru_flags(FORCE)
    try:
        yc = gru_stack(xc, rnn_c, lens=lens)
        (yc * w.float().cuda()).sum().backward()
        torch.cuda.synchronize()
    finally:
        lib.sb_debug_gru_flags(0)
    return rnn64, x64, y64, rnn_c, xc, yc


def _check(rnn64, x64, y64, rnn_c, xc, yc, lens=None):
    B = y64.shape[0]
    for b in range(B):
        L = y64.shape[1] if lens is None else lens[b]
        assert (yc[b, :L].detach().double().cpu() - y64[b, :L]).abs().max().item() < 2e-2, b
    gx = xc.grad.double().cpu()
    assert (gx - x64.grad).abs().max().item() < 3e-2 * x64.grad.abs().max().item() + 1e-4
    for (n, p64), (_, pc) in zip(rnn64.named_parameters(), rnn_c.named_parameters()):
        ref = p64.grad
        assert (pc.grad.double().cpu() - ref).abs().max().item() < \
            3e-2 * ref.abs().max().item() + 1e-4, n


@pytest.mark.parametrize("B", [8, 20, 33, 56, 64])
def test_l2_reduce_scatter_forced_matches_fp64(cuda_lib, B):
    """the shapes of test_gru_both_k_split_flavours, forward and backward in the L2 mode"""
    _check(*_ref_and_ours_forced(B, 7, 96, 256, 2, seed=B + 256))


def test_l2_reduce_scatter_forced_exact_lengths(cuda_lib):
    lens = [31, 9, 1, 24, 31, 17, 5]
    out = _ref_and_ours_forced(len(lens), max(lens), 48, 256, 2, seed=7, lens=lens)
    _check(*out, lens=lens)
    xc, yc = out[4], out[5]
    for b, L in enumerate(lens):
        assert float(xc.grad[b, L:].abs().sum()) == 0.0, b
        assert float(yc[b, L:].detach().abs().sum()) == 0.0, b


def test_l2_reduce_scatter_forced_padded_width(cuda_lib):
    """H = 250 runs at Hp = 256, inside the K-split domain"""
    _check(*_ref_and_ours_forced(12, 9, 64, 250, 1, seed=250))
