"""CPU checks of tests/gru_ref.py, the rounding-faithful reference of the GRU recurrence kernels.

1. With rounded=False the reference is the GRU of torch.nn.GRU: forward, and the gradients with
   respect to the input projections, both biases and W_hh, to 1e-10 in fp64.
2. The bars have power in both directions: the fp32 emulation of the kernels' arithmetic passes
   every bar, and every planted fault of gru_ref.MUTATIONS fails at least one.
"""
import pytest
import torch

import gru_ref as R


def _inputs(T, Bp, H, ndir, gain, seed):
    g = torch.Generator().manual_seed(seed)
    a = gain / H ** 0.5
    whh = (torch.rand(ndir, 3 * H, H, generator=g) * 2 - 1) * a
    bhh = (torch.rand(ndir, 3 * H, generator=g) * 2 - 1) * a
    gi = torch.randn(T * Bp, ndir * 3 * H, generator=g)
    dy = torch.randn(T * Bp, ndir * H, generator=g)
    return gi, whh, bhh, dy


def _dwhh(dgi, dghn, y, T, ndir):
    """dW_hh = sum over steps with a predecessor of [dr | dz | dhn]^T h_{t-1}"""
    H = dghn.shape[1] // ndir
    dgi = dgi.view(T, -1, ndir, 3 * H)
    dghn = dghn.view(T, -1, ndir, H)
    y = y.view(T, -1, ndir, H)
    out = []
    for d in range(ndir):
        rows = torch.cat([dgi[:, :, d, :2 * H], dghn[:, :, d]], 2)
        cur, prev = (slice(1, T), slice(0, T - 1)) if d == 0 else (slice(0, T - 1), slice(1, T))
        out.append(torch.einsum("tbk,tbh->kh", rows[cur], y[prev, :, d]))
    return out


@pytest.mark.parametrize("ndir", [1, 2])
@pytest.mark.parametrize("T", [1, 2, 9])
def test_unrounded_reference_is_nn_gru(T, ndir):
    """gi enters nn.GRU as its input through W_ih = [I | 0] / [0 | I] and b_ih = 0, so the input
    gradient is the gradient w.r.t. gi."""
    Bp, H = 5, 12
    gi, whh, bhh, dy = [v.double() for v in _inputs(T, Bp, H, ndir, 2.0, T + ndir)]
    rnn = torch.nn.GRU(ndir * 3 * H, H, bidirectional=ndir == 2).double()
    eye = torch.eye(ndir * 3 * H, dtype=torch.float64)
    with torch.no_grad():
        for d in range(ndir):
            sfx = "_l0" + ("_reverse" if d else "")
            getattr(rnn, "weight_ih" + sfx).copy_(eye[d * 3 * H:(d + 1) * 3 * H])
            getattr(rnn, "bias_ih" + sfx).zero_()
            getattr(rnn, "weight_hh" + sfx).copy_(whh[d])
            getattr(rnn, "bias_hh" + sfx).copy_(bhh[d])
    x = gi.view(T, Bp, -1).clone().requires_grad_(True)
    y_nn, _ = rnn(x)
    (y_nn * dy.view(T, Bp, -1)).sum().backward()

    y, gates, xn = R.gru_fwd(gi, whh, bhh, T, rounded=False)
    assert (y - y_nn.detach().reshape(T * Bp, -1)).abs().max().item() < 1e-10
    assert torch.equal(xn, y.to(torch.bfloat16))
    dgi, dghn, dbih, dbhh = R.gru_bwd(dy, y, gates, whh, T, rounded=False)
    assert (dgi - x.grad.reshape(T * Bp, -1)).abs().max().item() < 1e-10
    for d, dw in enumerate(_dwhh(dgi, dghn, y, T, ndir)):
        sfx = "_l0" + ("_reverse" if d else "")
        K3 = slice(d * 3 * H, (d + 1) * 3 * H)
        assert (dbih[K3] - getattr(rnn, "bias_ih" + sfx).grad).abs().max().item() < 1e-10
        assert (dbhh[K3] - getattr(rnn, "bias_hh" + sfx).grad).abs().max().item() < 1e-10
        assert (dw - getattr(rnn, "weight_hh" + sfx).grad).abs().max().item() < 1e-10


def _emulated(T, Bp, H, ndir, gain, mutate):
    """(fwd_err, (dgi/dghn element error, bias error)) of the fp32 emulation of the kernels, with
    one planted fault or none, against the teacher-forced fp64 reference"""
    gi, whh, bhh, dy = _inputs(T, Bp, H, ndir, gain, 7 * T + H + gain)
    whh = whh.to(torch.bfloat16)
    fwd_fault = mutate if mutate in ("zh_bf16", "missing_chunk", "bhn_outside", "fwd_start") else None
    y, gates, _ = R.gru_fwd(gi, whh, bhh, T, dtype=torch.float32, mutate=fwd_fault)
    ry, rg, _ = R.gru_fwd(gi, whh, bhh, T, h_prev=y)
    fwd = R.fwd_err(y, gates, ry, rg)
    # the backward is fed the forward's y and gates (fp32), as the GPU tests feed the kernels
    yr, gr, _ = R.gru_fwd(gi, whh, bhh, T)
    yr, gr = yr.float(), gr.float()
    bwd_fault = None if mutate == fwd_fault else mutate
    e = R.gru_bwd(dy, yr, gr, whh, T, dtype=torch.float32, mutate=bwd_fault)
    out = (e[0].to(torch.bfloat16), e[1].to(torch.bfloat16), e[2], e[3])
    ref = R.gru_bwd(dy, yr, gr, whh, T, xr=out[:2])
    return fwd, R.bwd_errs(out, ref)


SHAPES = [(40, 16, 256, 1), (12, 24, 128, 2)]


@pytest.mark.parametrize("gain", [1, 3])
@pytest.mark.parametrize("T,Bp,H,ndir", SHAPES)
def test_fp32_emulation_passes_every_bar(T, Bp, H, ndir, gain):
    fwd, (elem, bias) = _emulated(T, Bp, H, ndir, gain, None)
    assert fwd < R.FWD_ABS / 20, fwd
    assert elem < R.BWD_FLOOR / 20, elem
    assert bias < R.DB_REL / 20, bias


@pytest.mark.parametrize("mutate", R.MUTATIONS)
@pytest.mark.parametrize("gain", [1, 3])
@pytest.mark.parametrize("T,Bp,H,ndir", SHAPES)
def test_every_planted_fault_fails_a_bar(T, Bp, H, ndir, gain, mutate):
    fwd, (elem, bias) = _emulated(T, Bp, H, ndir, gain, mutate)
    failed = fwd > R.FWD_ABS or elem > R.BWD_FLOOR or bias > R.DB_REL
    assert failed, (fwd, elem, bias)


def test_unrounded_stack_reference_is_packed_nn_gru():
    """gru_ref.gru_stack with rounded=False: nn.GRU over pack_padded_sequence, 2 layers, both
    directions, forward and every gradient"""
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    torch.manual_seed(0)
    lens = [11, 4, 1, 9, 11, 6]
    B, T, In, H = len(lens), max(lens), 20, 10
    rnn = torch.nn.GRU(In, H, 2, batch_first=True, bidirectional=True).double()
    x = torch.randn(B, T, In, dtype=torch.float64, requires_grad=True)
    out, _ = rnn(pack_padded_sequence(x, torch.tensor(lens), batch_first=True, enforce_sorted=False))
    out, _ = pad_packed_sequence(out, batch_first=True, total_length=T)
    dout = torch.randn_like(out)
    (out * dout).sum().backward()
    y, dx, grads = R.gru_stack(x, list(rnn.parameters()), 2, dout, lens, rounded=False)
    assert (y - out.detach()).abs().max().item() < 1e-10
    assert (dx - x.grad).abs().max().item() < 1e-10
    for (n, p), g in zip(rnn.named_parameters(), grads):
        assert (g - p.grad).abs().max().item() < 1e-10, n
