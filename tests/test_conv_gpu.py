"""GPU parity: im2col + wgmma conv stack vs torch conv2d in fp64 on the CPU.

The kernels round the GEMM operands (inputs, weights, inter-layer activations) to bf16 and
accumulate in fp32.  A ReLU mask is discontinuous, so a reference computed from UN-rounded operands
flips the mask of the few pre-activations that lie within the rounding error of zero and its
gradient then differs by O(1) on those elements (measured: ~0.3 % of elements, 6 % of the largest
gradient entry under a white-noise upstream gradient) - that is a property of bf16 arithmetic, not
of the kernels.  The reference here therefore applies the SAME operand rounding (straight-through
in backward) and is otherwise exact (fp64): outputs must agree to 1e-3 of the output scale,
gradients to 3 % of the largest reference entry (bf16 rounding of the backward operands)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _build(specs, in_c=1):
    layers = []
    for out_c, h, w, s in specs:
        layers += [torch.nn.Conv2d(in_c, out_c, (h, w), stride=(s, s)), torch.nn.ReLU()]
        in_c = out_c
    return torch.nn.Sequential(*layers)


@pytest.mark.parametrize("specs,B,T,F", [
    ([[32, 5, 32, 2]], 4, 100, 40),                      # tests/shared.py tiny config
    ([[8, 5, 8, 2], [8, 5, 8, 2]], 3, 61, 80),          # golden 'bi' config
    ([[32, 5, 8, 2], [32, 5, 8, 2]], 2, 90, 80),        # north-star conv stack (WSJ)
    ([[16, 3, 4, 1], [8, 2, 3, 3]], 2, 33, 21),          # odd geometry, stride 1 and 3
    # the shipped TIMIT recipe (examples/timit/ctc_config.json: second layer [32, 5, 32, 1] =
    # 5 x 32 taps per input pixel -> the runtime-loop col2im gather; was a cuDNN fallback)
    ([[32, 5, 32, 2], [32, 5, 32, 1]], 2, 60, 161),
    ([[8, 7, 12, 1], [8, 6, 11, 2]], 2, 40, 48),         # > 5 x 8 taps per stride phase, stride 2
])
def test_conv_stack_forward_backward(cuda_lib, specs, B, T, F):
    from speech_b200 import ops
    torch.manual_seed(B + T + F)
    conv = _build(specs)
    x = torch.randn(B, T, F)
    conv64 = _build(specs).double()
    conv64.load_state_dict({k: v.double() for k, v in conv.state_dict().items()})

    def rnd(t):   # bf16 rounding with a straight-through gradient
        return t + (t.detach().float().bfloat16().double() - t.detach())

    h = rnd(x.double().unsqueeze(1))
    mods = [m for m in conv64 if isinstance(m, torch.nn.Conv2d)]
    for li, m in enumerate(mods):
        pre = torch.nn.functional.conv2d(h, rnd(m.weight), m.bias, stride=m.stride)
        h = torch.relu(pre)
        if li + 1 < len(mods):
            h = rnd(h)
    y64 = h
    b, c, t, f = y64.shape
    y64 = y64.transpose(1, 2).reshape(b, t, c * f)
    w = torch.randn_like(y64)
    (y64 * w).sum().backward()
    conv_c = conv.cuda()
    y = ops.conv_stack(x.cuda(), conv_c, True)
    assert y.shape == y64.shape
    (y * w.float().cuda()).sum().backward()
    scale = y64.abs().max().item()
    assert (y.double().cpu() - y64).abs().max().item() < 1e-3 * scale
    for (n, p64), (_, pc) in zip(conv64.named_parameters(), conv_c.named_parameters()):
        ref = p64.grad
        err = (pc.grad.double().cpu() - ref).abs().max().item()
        assert err < 3e-2 * ref.abs().max().item() + 1e-4, (n, err, ref.abs().max().item())


def test_conv_stack_dropout_matches_masked_reference(cuda_lib):
    """Training-time Dropout after each ReLU (model.py:25-26) runs inside our kernels: the masks
    are drawn with torch.rand in layer order, so re-seeding reproduces them for the reference."""
    from speech_b200 import ops
    specs, B, T, F, p = [[8, 5, 8, 2], [16, 3, 4, 1]], 3, 61, 40, 0.4
    torch.manual_seed(5)
    layers, in_c = [], 1
    for out_c, h, w, s in specs:
        layers += [torch.nn.Conv2d(in_c, out_c, (h, w), stride=(s, s)), torch.nn.ReLU(),
                   torch.nn.Dropout(p)]
        in_c = out_c
    conv = torch.nn.Sequential(*layers).cuda()
    x = torch.randn(B, T, F).cuda()

    torch.manual_seed(99)
    y = ops.conv_stack(x, conv, True)
    wgt = torch.randn_like(y)
    (y * wgt).sum().backward()
    got = {n: q.grad.clone() for n, q in conv.named_parameters()}

    def rnd(t):
        return t + (t.detach().float().bfloat16().double() - t.detach())

    torch.manual_seed(99)
    h = rnd(x.double().unsqueeze(1))
    params = {n: q.detach().double().requires_grad_(True) for n, q in conv.named_parameters()}
    mods = [m for m in conv if isinstance(m, torch.nn.Conv2d)]
    for li, m in enumerate(mods):
        pre = torch.nn.functional.conv2d(h, rnd(params["%d.weight" % (3 * li)]),
                                         params["%d.bias" % (3 * li)], stride=m.stride)
        b, c, t, f = pre.shape
        mask = (torch.rand(b * t * f, c, device="cuda") >= p).double() / (1.0 - p)
        mask = mask.view(b, t, f, c).permute(0, 3, 1, 2)
        h = torch.relu(pre) * mask
        if li + 1 < len(mods):
            h = rnd(h)
    b, c, t, f = h.shape
    y64 = h.transpose(1, 2).reshape(b, t, c * f)
    (y64 * wgt.double()).sum().backward()
    zero_frac = (y == 0).float().mean().item()
    assert zero_frac > p * 0.8                      # dropout really happened
    scale = y64.abs().max().item()
    assert (y.double() - y64).abs().max().item() < 2e-3 * scale
    for n, ref in params.items():
        err = (got[n].double() - ref.grad).abs().max().item()
        assert err < 3e-2 * ref.grad.abs().max().item() + 1e-4, (n, err)
    # eval mode: no dropout, deterministic
    y1 = ops.conv_stack(x, conv, False)
    y2 = ops.conv_stack(x, conv, False)
    assert torch.equal(y1, y2)
