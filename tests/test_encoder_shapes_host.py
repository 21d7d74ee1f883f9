"""Host checks (no GPU) of the zero-padding that lets the kernels run GRU widths that are not a
multiple of 16 (up to the resident limit), any conv channel count and any joint width: the
padding helpers reproduce the unpadded modules exactly in fp64, and the joint's routing query
agrees with the fused kernel's shared-memory budget."""
import math

import pytest
import torch
import torch.nn.functional as F
from torch.func import functional_call


def _close(a, b):
    return (a - b).abs().max().item() <= 1e-12 * max(1.0, b.abs().max().item())


@pytest.mark.parametrize("H", [40, 200, 1000])
def test_padded_gru_reproduces_unpadded_gru(H):
    from speech_b200 import ops
    torch.manual_seed(H)
    B, T, In, L = 2, 5, 24, 2
    Hp = (H + 15) // 16 * 16
    rnn = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=True).double()
    wide = torch.nn.GRU(In, Hp, L, batch_first=True, bidirectional=True).double()
    x = torch.randn(B, T, In, dtype=torch.float64)
    w = torch.randn(B, T, 2 * H, dtype=torch.float64)
    y, _ = rnn(x)
    (y * w).sum().backward()
    src = {n: q.detach().clone().requires_grad_(True) for n, q in rnn.named_parameters()}
    padded = {}
    for l in range(L):
        for sfx in ("_l%d" % l, "_l%d_reverse" % l):
            names = [k + sfx for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
            for n, q in zip(names, ops.pad_gru_layer(*[src[n] for n in names], H, Hp,
                                                      2 if l else 0)):
                padded[n] = q
    yp, _ = functional_call(wide, padded, (x,))
    assert yp.shape == (B, T, 2 * Hp)
    assert torch.all(yp.view(B, T, 2, Hp)[..., H:] == 0)         # padded units stay exactly 0
    got = ops.unpad_blocks(yp, 2, 2, H, Hp)
    assert _close(got, y.detach())
    (got * w).sum().backward()
    for n, q in rnn.named_parameters():
        assert src[n].grad.shape == q.grad.shape
        assert _close(src[n].grad, q.grad), n


@pytest.mark.parametrize("C", [1, 4, 12])
def test_padded_conv_channels_reproduce_unpadded_stack(C):
    from speech_b200 import ops
    torch.manual_seed(C)
    specs = [(C, 5, 7, 2), (C, 3, 5, 1)]
    x = torch.randn(2, 30, 40, dtype=torch.float64)
    params, ci = [], 1
    for co, kh, kw, s in specs:
        params += [(torch.randn(co, ci, kh, kw, dtype=torch.float64) / math.sqrt(ci * kh * kw))
                   .requires_grad_(True), torch.randn(co, dtype=torch.float64).requires_grad_(True)]
        ci = co

    def run(pad):
        y, ci_p = x.unsqueeze(1), 1
        for l, (co, kh, kw, s) in enumerate(specs):
            wt, b = params[2 * l], params[2 * l + 1]
            cop = (co + 7) // 8 * 8 if pad else co
            wt = ops.pad_blocks(ops.pad_blocks(wt, 0, 1, co, cop), 1, 1, wt.shape[1], ci_p)
            b = ops.pad_blocks(b, 0, 1, co, cop)
            y, ci_p = torch.relu(F.conv2d(y, wt, b, stride=s)), cop
        b_, c_, t_, f_ = y.shape
        return y.transpose(1, 2).reshape(b_, t_, c_ * f_), f_   # channel-major features

    ref, f = run(False)
    wgt = torch.randn_like(ref)
    gref = torch.autograd.grad((ref * wgt).sum(), params)
    out, f = run(True)
    assert out.shape[2] == (C + 7) // 8 * 8 * f
    assert torch.all(out[:, :, C * f:] == 0)
    got = out[:, :, :C * f]
    assert _close(got, ref.detach())
    for g, r in zip(torch.autograd.grad((got * wgt).sum(), params), gref):
        assert _close(g, r)


def test_joint_routing_query_matches_the_fused_kernels_budget():
    """sb_rnnt_joint_resident answers from joint_launch's own shared-memory arithmetic: fc2 stays
    resident up to H = 1024 with 33..64 classes and up to H = 1792 with <= 32 classes."""
    from speech_b200 import _lib
    from speech_b200.functions import transducer
    lib = _lib.load()
    assert lib.sb_rnnt_joint_resident(1024, 64) == 1
    assert lib.sb_rnnt_joint_resident(1040, 40) == 0
    assert lib.sb_rnnt_joint_resident(1792, 29) == 1
    assert lib.sb_rnnt_joint_resident(1808, 29) == 0
    assert lib.sb_rnnt_joint_resident(100, 29) == 0          # H % 8 != 0
    assert lib.sb_rnnt_joint_resident(104, 29) == 1
    assert lib.sb_rnnt_joint_resident(256, 65) == 0
    assert not transducer.joint_uses_slabs(1024, 64)
    assert transducer.joint_uses_slabs(1280, 40)
    assert transducer.joint_uses_slabs(256, 65)

