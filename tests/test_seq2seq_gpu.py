"""GPU parity of the attention decoder kernels (csrc/s2s.cu, functions/s2s.py).

Reference formulation = the per-token chain of Seq2Seq.decode (speech/models/seq2seq.py:78-112)
and NNAttention.forward (:344-360) restated here with stock torch modules in float64 on the CPU,
sharing the model's parameters: teacher-forced logits / alignments within 1e-4, every gradient
(encoder states and all decoder parameters) within 2 % of its largest entry (the time-batched
weight gradients use bf16 tensor-core operands, everything else is fp32).  Greedy decode and beam
search run device-resident and must return the hypotheses of the reference's host loops (restated
below over the SAME step kernels), on the model's own encoder states."""
import math
import random

import numpy as np
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu


def _cfg(H, layers=1, bidir=True, log_t=False, sample=0.0):
    return {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                        "rnn": {"dim": H, "bidirectional": bidir, "layers": layers}},
            "decoder": {"embedding_dim": H, "layers": 1, "log_t": log_t, "sample_prob": sample}}


def _eager_decode(m, x, y, flags):
    """seq2seq.py:78-112 + :344-360 in float64 on the CPU with the model's parameters."""
    emb = m.embedding.weight.detach().double().cpu().requires_grad_(True)
    cell = nn.GRUCell(emb.shape[1], x.shape[2]).double()
    cell.load_state_dict({k: v.detach().double().cpu() for k, v in m.dec_rnn.state_dict().items()})
    conv = nn.Conv1d(1, x.shape[2], m.attend.conv.kernel_size[0],
                     padding=m.attend.conv.padding[0]).double()
    conv.load_state_dict({k: v.detach().double().cpu() for k, v in m.attend.conv.state_dict().items()})
    lin = nn.Linear(x.shape[2], 1).double()
    lin.load_state_dict({k: v.detach().double().cpu() for k, v in m.attend.nn[1].fc.state_dict().items()})
    fc = nn.Linear(x.shape[2], m.fc.fc.out_features).double()
    fc.load_state_dict({k: v.detach().double().cpu() for k, v in m.fc.fc.state_dict().items()})
    x = x.detach().double().cpu().requires_grad_(True)
    y = y.cpu()
    hx = torch.zeros(x.shape[0], x.shape[2], dtype=torch.float64)
    ax = sx = None
    out, aligns = [], []
    for t in range(y.shape[1] - 1):
        if t > 0 and flags[t]:
            tok = torch.max(out[-1], dim=1)[1]
        else:
            tok = y[:, t]
        ix = emb[tok]
        if sx is not None:
            ix = ix + sx
        hx = cell(ix, hx)
        pax = x + hx.unsqueeze(1)
        if ax is not None:
            pax = pax + conv(ax.unsqueeze(1)).transpose(1, 2)
        pax = lin(torch.relu(pax)).squeeze(2)
        if m.attend.log_t:
            pax = math.log(pax.shape[1]) * pax
        ax = torch.softmax(pax, dim=1)
        sx = torch.sum(x * ax.unsqueeze(2), dim=1)
        aligns.append(ax)
        out.append(fc(hx + sx))
    params = {"embedding.weight": emb, "dec_rnn.weight_ih": cell.weight_ih,
              "dec_rnn.weight_hh": cell.weight_hh, "dec_rnn.bias_ih": cell.bias_ih,
              "dec_rnn.bias_hh": cell.bias_hh, "attend.conv.weight": conv.weight,
              "attend.conv.bias": conv.bias, "attend.nn.1.fc.weight": lin.weight,
              "attend.nn.1.fc.bias": lin.bias, "fc.fc.weight": fc.weight, "fc.fc.bias": fc.bias}
    return torch.stack(out, 1), torch.stack(aligns, 1), x, params


@pytest.mark.parametrize("B,T,H,V,U,log_t,sample", [
    (3, 19, 16, 9, 6, False, 0.0),
    (4, 37, 64, 12, 9, True, 0.0),
    (5, 50, 128, 30, 12, True, 0.5),      # scheduled sampling: arg-max tokens fed back
    (2, 33, 256, 30, 7, False, 0.0),
])
def test_teacher_forced_decode_forward_and_backward(cuda_lib, B, T, H, V, U, log_t, sample):
    from speech_b200.models import Seq2Seq
    from speech_b200.functions import s2s
    torch.manual_seed(B + T + H)
    m = Seq2Seq(40, V, _cfg(H, log_t=log_t)).cuda()
    x = (torch.randn(B, T, H) * 0.5).cuda().requires_grad_(True)
    y = torch.randint(0, V - 1, (B, U)).cuda()
    rng = random.Random(3)
    flags = [False] + [rng.random() < sample for _ in range(U - 2)]
    out, aligns = s2s.decode(m, x, y, flags)
    assert tuple(out.shape) == (B, U - 1, V - 1) and tuple(aligns.shape) == (B, U - 1, T)
    w = torch.randn_like(out)
    (out * w).sum().backward()
    ro, ra, rx, rp = _eager_decode(m, x, y, flags)
    (ro * w.double().cpu()).sum().backward()
    assert (out.double().cpu() - ro).abs().max().item() < 1e-4 * max(1.0, ro.abs().max().item())
    assert (aligns.double().cpu() - ra).abs().max().item() < 1e-5
    assert abs(aligns.sum(2) - 1).max().item() < 1e-5
    g = x.grad.double().cpu()
    assert (g - rx.grad).abs().max().item() < 2e-3 * rx.grad.abs().max().item() + 1e-6
    for name, p in m.named_parameters():
        if name not in rp:
            continue
        ref = rp[name].grad
        got = p.grad.double().cpu().reshape(ref.shape)
        # time-batched on the wgmma GEMM (bf16 operands): cell weights and the output projection
        tol = 2e-2 if name in ("dec_rnn.weight_ih", "dec_rnn.weight_hh", "fc.fc.weight") else 2e-3
        # the softmax is invariant to a shift of the scores, so d(attention bias) is EXACTLY zero:
        # what both sides hold is the rounding residue of sum_t d score_t (fp64: 1e-16, fp32: 1e-6)
        floor = 1e-5 if name == "attend.nn.1.fc.bias" else 1e-6
        assert (got - ref).abs().max().item() < tol * ref.abs().max().item() + floor, name


def test_decode_step_loop_equals_teacher_forced_decode(cuda_lib):
    """awni/speech tests/seq2seq_test.py:32-45 on the drop-in: rtol 1e-5 / atol 1e-7."""
    from speech_b200.models import Seq2Seq
    torch.manual_seed(1337)
    np.random.seed(1337)
    m = Seq2Seq(40, 11, _cfg(32)).cuda()
    m.set_eval()
    inputs = [np.random.randn(70, 40).astype(np.float32) for _ in range(4)]
    labels = [np.random.randint(0, 10, 9).tolist() for _ in range(4)]
    x, y = m.collate(inputs, labels)
    with torch.no_grad():
        x_enc = m.encode(x.cuda())
        y = y.cuda()
        out_t, _ = m.decode(x_enc, y)
        state, outs = None, []
        for t in range(y.shape[1] - 1):
            o, state = m.decode_step(x_enc, y[:, t:t + 1], state=state)
            outs.append(o)
    assert np.allclose(torch.stack(outs, 1).cpu().numpy(), out_t.cpu().numpy(), rtol=1e-5, atol=1e-7)


def _host_greedy(m, x_enc, y0, end_tok, max_len):
    y, state, toks = y0, None, [y0]
    for _ in range(max_len):
        out, state = m.decode_step(x_enc, y, state=state)
        y = torch.max(out, dim=1)[1].unsqueeze(1)
        toks.append(y)
        if bool((y == end_tok).all()):
            break
    return torch.cat(toks, 1).cpu().tolist()


def _host_beam(m, x_enc, start_tok, end_tok, beam_size, max_len):
    """seq2seq.py:180-227 (with the py3 list() fix) over decode_step."""
    y = torch.zeros(1, 1, dtype=torch.int64, device=x_enc.device)
    beam = [((start_tok,), 0, None)]
    complete = []
    for _ in range(max_len):
        new_beam = []
        for hyp, score, state in beam:
            y[0] = hyp[-1]
            out, state = m.decode_step(x_enc, y, state=state, softmax=True)
            for i, p in enumerate(out.cpu().numpy().squeeze(0).tolist()):
                new_beam.append((hyp + (i,), score + p, state))
        new_beam = sorted(new_beam, key=lambda c: c[1], reverse=True)
        for cand in new_beam[:beam_size]:
            if cand[0][-1] == end_tok:
                complete.append(cand)
        beam = [c for c in new_beam if c[0][-1] != end_tok][:beam_size]
        if len(beam) == 0:
            break
        if sum(c[1] > beam[0][1] for c in complete) >= beam_size:
            break
    complete = sorted(complete, key=lambda c: c[1], reverse=True)
    if len(complete) == 0:
        complete = beam
    return complete[0][0]


@pytest.mark.parametrize("wsj", [False, True])
def test_device_resident_greedy_and_beam_match_the_host_loops_on_own_encoder(cuda_lib, wsj):
    """Hypotheses on the model's OWN (bf16-kernel) encoder states: WSJ-shaped model (north-star
    conv stack, 3-layer biGRU-512, log_t) with beams 1 / 4 / 8, and a small model."""
    from speech_b200.models import Seq2Seq
    torch.manual_seed(11)
    np.random.seed(11)
    if wsj:
        cfg = {"dropout": 0.0, "encoder": {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
                                           "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
               "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True}}
        fdim, V, T = 80, 30, 300
    else:
        cfg, fdim, V, T = _cfg(32, layers=2), 40, 11, 90
    m = Seq2Seq(fdim, V, cfg).cuda()
    m.set_eval()
    with torch.no_grad():                 # make the decoder less uniform than at initialisation
        m.fc.fc.weight.mul_(8.0)
        m.embedding.weight.mul_(3.0)
    inputs = [np.random.randn(T - 7 * i, fdim).astype(np.float32) for i in range(3)]
    labels = [[V - 1] + np.random.randint(0, V - 2, 6).tolist() + [V - 2] for _ in range(3)]
    batch = (inputs, labels)
    x, y = m.collate(*batch)
    end_tok = int(y[0, -1])
    with torch.no_grad():
        x_enc = m.encode(x.cuda())
        want = _host_greedy(m, x_enc, y[:, 0:1].cuda(), end_tok, 25)
    got = m.infer(batch, max_len=25)
    assert got == want
    for e in range(2):
        one = ([inputs[e]], [labels[e]])
        with torch.no_grad():
            xe = m.encode(m.collate(*one)[0].cuda())
        for bs in (1, 4, 8):
            hyp = m.beam_search(one, beam_size=bs, max_len=20)[0]
            ref = _host_beam(m, xe, int(y[0, 0]), end_tok, bs, 20)
            assert tuple(hyp) == tuple(ref), (e, bs)
