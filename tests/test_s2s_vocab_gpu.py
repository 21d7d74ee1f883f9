"""The attention decoder at subword-sized vocabularies: the output projection over many CTAs
(sb_s2s_fc_rows / _logp), the split beam selection and the GEMM backward of the projection
(csrc/s2s_vocab.cu, csrc/s2s.cu, functions/s2s.py).

Reference formulation = the per-token chain of Seq2Seq.decode (speech/models/seq2seq.py:78-112)
and NNAttention.forward (:344-360), restated here with stock torch modules in float64 on the CPU.
Decoding runs device-resident and must return the hypotheses of the reference's host loops over
decode_step."""
import ctypes
import math
import random

import numpy as np
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu


def _cfg(H, layers=1, log_t=False, sample=0.0):
    return {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                        "rnn": {"dim": H, "bidirectional": True, "layers": layers}},
            "decoder": {"embedding_dim": H, "layers": 1, "log_t": log_t, "sample_prob": sample}}


def _eager_decode(m, x, y, flags, lens=None):
    """seq2seq.py:78-112 + :344-360 in float64 on the CPU with the model's parameters; lens: the
    frames each utterance attends over (softmax and log T over those only)."""
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
    B, T = x.shape[0], x.shape[1]
    if lens is None:
        mask, scale = None, torch.full((B, 1), math.log(T), dtype=torch.float64)
    else:
        ln = torch.as_tensor(lens)
        mask = torch.arange(T).unsqueeze(0) >= ln.unsqueeze(1)
        scale = torch.log(ln.double()).unsqueeze(1)
    hx = torch.zeros(B, x.shape[2], dtype=torch.float64)
    ax = sx = None
    out, aligns = [], []
    for t in range(y.shape[1] - 1):
        tok = torch.max(out[-1], dim=1)[1] if t > 0 and flags[t] else y[:, t]
        ix = emb[tok]
        if sx is not None:
            ix = ix + sx
        hx = cell(ix, hx)
        pax = x + hx.unsqueeze(1)
        if ax is not None:
            pax = pax + conv(ax.unsqueeze(1)).transpose(1, 2)
        pax = lin(torch.relu(pax)).squeeze(2)
        if m.attend.log_t:
            pax = scale * pax
        if mask is not None:
            pax = pax.masked_fill(mask, -math.inf)
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


@pytest.mark.parametrize("B,T,H,C,U,log_t,sample,use_lens", [
    (3, 19, 16, 200, 6, False, 0.0, False),        # many-CTA projection, sb_s2s_dout backward
    (4, 37, 64, 1000, 9, True, 0.0, False),
    (5, 50, 128, 4000, 8, True, 0.5, False),       # scheduled sampling: per-step projection
    (3, 25, 16, 9000, 5, False, 0.0, False),       # GEMM backward of the projection
    (1, 10, 1200, 8200, 4, False, 0.0, False),     # fused forward, GEMM backward
    (2, 20, 32, 32000, 4, False, 0.0, False),
    (3, 40, 64, 1000, 7, True, 0.0, True),         # exact-lengths attention
])
def test_teacher_forced_decode_forward_and_backward(cuda_lib, B, T, H, C, U, log_t, sample,
                                                    use_lens):
    from speech_b200.models import Seq2Seq
    from speech_b200.functions import s2s
    torch.manual_seed(B + T + H + C)
    m = Seq2Seq(40, C + 1, _cfg(H, log_t=log_t)).cuda()
    assert s2s.DecoderWeights(m).fused == (C <= 7 * H)
    x = (torch.randn(B, T, H) * 0.5).cuda().requires_grad_(True)
    y = torch.randint(0, C, (B, U)).cuda()
    rng = random.Random(3)
    flags = [False] + [rng.random() < sample for _ in range(U - 2)]
    lens = [T - 9 * b for b in range(B)] if use_lens else None
    out, aligns = s2s.decode(m, x, y, flags, lens)
    assert tuple(out.shape) == (B, U - 1, C) and tuple(aligns.shape) == (B, U - 1, T)
    w = torch.randn_like(out)
    (out * w).sum().backward()
    ro, ra, rx, rp = _eager_decode(m, x, y, flags, lens)
    (ro * w.double().cpu()).sum().backward()
    assert (out.double().cpu() - ro).abs().max().item() < 1e-4 * max(1.0, ro.abs().max().item())
    assert (aligns.double().cpu() - ra).abs().max().item() < 1e-5
    g = x.grad.double().cpu()
    assert (g - rx.grad).abs().max().item() < 2e-3 * rx.grad.abs().max().item() + 1e-6
    for name, p in m.named_parameters():
        if name not in rp:
            continue
        ref = rp[name].grad
        got = p.grad.double().cpu().reshape(ref.shape)
        tol = 2e-2 if name in ("dec_rnn.weight_ih", "dec_rnn.weight_hh", "fc.fc.weight") else 2e-3
        # d(attention bias) is exactly zero (softmax shift invariance): both sides hold the rounding
        # residue of sum_t d score_t, whose terms grow with the number of classes fed back (the
        # random output weights w: d o sums C of them)
        floor = 1e-5 * max(1.0, C / 1000.0) if name == "attend.nn.1.fc.bias" else 1e-6
        assert (got - ref).abs().max().item() < tol * ref.abs().max().item() + floor, name


def test_decode_step_loop_equals_teacher_forced_decode_on_the_many_cta_route(cuda_lib):
    """awni/speech tests/seq2seq_test.py:32-45 at C = 1000 > 7 H: rtol 1e-5 / atol 1e-7."""
    from speech_b200.models import Seq2Seq
    from speech_b200.functions import s2s
    torch.manual_seed(1337)
    np.random.seed(1337)
    m = Seq2Seq(40, 1001, _cfg(32)).cuda()
    m.set_eval()
    assert not s2s.DecoderWeights(m).fused
    inputs = [np.random.randn(70, 40).astype(np.float32) for _ in range(4)]
    labels = [np.random.randint(0, 1000, 9).tolist() for _ in range(4)]
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


def _decoder_model(H, V, seed):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(seed)
    np.random.seed(seed)
    m = Seq2Seq(40, V, _cfg(H)).cuda()
    m.set_eval()
    with torch.no_grad():                 # make the decoder less uniform than at initialisation
        m.fc.fc.weight.mul_(8.0)
        m.embedding.weight.mul_(3.0)
    return m


def _check_decoders_match_host_loops(m, V, beams, max_len=12):
    inputs = [np.random.randn(60 - 7 * i, 40).astype(np.float32) for i in range(3)]
    labels = [[V - 1] + np.random.randint(0, V - 2, 6).tolist() + [V - 2] for _ in range(3)]
    batch = (inputs, labels)
    x, y = m.collate(*batch)
    end_tok = int(y[0, -1])
    with torch.no_grad():
        x_enc = m.encode(x.cuda())
        want = _host_greedy(m, x_enc, y[:, 0:1].cuda(), end_tok, max_len)
    assert m.infer(batch, max_len=max_len) == want
    one = ([inputs[0]], [labels[0]])
    with torch.no_grad():
        xe = m.encode(m.collate(*one)[0].cuda())
    for bs in beams:
        hyp = m.beam_search(one, beam_size=bs, max_len=max_len)[0]
        ref = _host_beam(m, xe, int(y[0, 0]), end_tok, bs, max_len)
        assert tuple(hyp) == tuple(ref), bs


def test_device_greedy_and_beam_match_host_loops_at_5000_classes(cuda_lib):
    """C = 5000 at H = 64: the many-CTA projection; beams 8 and 32 take the split selection."""
    from speech_b200.functions import s2s
    m = _decoder_model(64, 5001, 21)
    assert not s2s.fc_fused(64, 5000)
    assert s2s.beam_select_fits(4, 5000) and not s2s.beam_select_fits(8, 5000)
    _check_decoders_match_host_loops(m, 5001, (1, 4, 8, 32), max_len=8)


def test_device_beam_matches_host_loop_fused_projection_split_selection(cuda_lib):
    """C = 3300 at H = 512: the fused projection, but beam 8 exceeds the single-CTA selection."""
    from speech_b200.functions import s2s
    m = _decoder_model(512, 3301, 22)
    assert s2s.fc_fused(512, 3300) and not s2s.beam_select_fits(8, 3300)
    _check_decoders_match_host_loops(m, 3301, (8,), max_len=8)


def test_forced_many_cta_route_matches_the_fused_route_at_small_vocab(cuda_lib, monkeypatch):
    from speech_b200.functions import s2s
    m = _decoder_model(64, 31, 23)
    assert s2s.fc_fused(64, 30)
    inputs = [np.random.randn(60 - 7 * i, 40).astype(np.float32) for i in range(3)]
    labels = [[30] + np.random.randint(0, 29, 6).tolist() + [29] for _ in range(3)]
    batch = (inputs, labels)
    one = ([inputs[0]], [labels[0]])
    x, y = m.collate(*batch)

    def run():
        with torch.no_grad():
            x_enc = m.encode(x.cuda())
            logits, _ = m.decode(x_enc, y.cuda())
            step, _ = m.decode_step(x_enc, y[:, :1].cuda(), softmax=True)
        return (logits, step, m.infer(batch, max_len=15),
                [m.beam_search(one, beam_size=bs, max_len=15)[0] for bs in (1, 4, 8)])

    fused = run()
    monkeypatch.setattr(s2s, "fc_fused", lambda H, C: False)
    monkeypatch.setattr(s2s, "beam_select_fits", lambda K, C: False)
    assert not s2s.DecoderWeights(m).fused
    split = run()
    for a, b in zip(fused[:2], split[:2]):
        assert (a - b).abs().max().item() <= 1e-5 * max(1.0, a.abs().max().item())
    assert fused[2] == split[2]
    assert [tuple(h) for h in fused[3]] == [tuple(h) for h in split[3]]


def _beam_buffers(lib, K, C, max_len, dev):
    n = ctypes.c_size_t(0)
    lib.sb_s2s_beam_state_size(ctypes.byref(n))
    node_cap, c_cap = 2 * K * (max_len + 1) + 2, K * (max_len + 1)
    return {"state": torch.zeros(n.value + 64, dtype=torch.uint8, device=dev),
            "nodes": torch.zeros(node_cap, 2, dtype=torch.int32, device=dev),
            "c_scores": torch.zeros(c_cap, dtype=torch.float64, device=dev),
            "parent": torch.zeros(K, dtype=torch.int32, device=dev),
            "tok": torch.zeros(K, dtype=torch.int32, device=dev),
            "out": torch.zeros(max_len + 2, dtype=torch.int32, device=dev),
            "node_cap": node_cap, "c_cap": c_cap}


@pytest.mark.parametrize("K,C,ties", [(4, 50, True), (8, 1000, False), (8, 1000, True),
                                      (32, 200, True), (3, 7, False)])
def test_split_selection_equals_single_cta_selection(cuda_lib, K, C, ties):
    """Same logp and state into both selections: same parent_row, tok_next, state bytes, nodes and
    complete scores after every step.  ties: logp on a coarse grid, so equal scores are common and
    (score desc, flat index asc) decides."""
    from speech_b200 import _lib
    from speech_b200.functions import s2s
    lib = _lib.load()
    dev = torch.device("cuda")
    assert s2s.beam_select_fits(K, C)
    max_len, end_tok = 7, C - 1
    g = torch.Generator().manual_seed(K * C)
    bufs = [_beam_buffers(lib, K, C, max_len, dev) for _ in range(2)]
    sp = _lib.stream_ptr()
    for b in bufs:
        _lib.check(lib.sb_s2s_beam_init(b["state"].data_ptr(), b["nodes"].data_ptr(),
                                        b["tok"].data_ptr(), 0, sp), "beam init")
    n = ctypes.c_size_t(0)
    lib.sb_s2s_beam_split_workspace_size(K, C, ctypes.byref(n))
    ws = torch.empty(n.value, dtype=torch.uint8, device=dev)
    for step in range(max_len):
        lp = torch.log_softmax(torch.randn(K, C, generator=g) * 2.0, 1)
        if ties:
            lp = torch.round(lp * 2.0) / 2.0
        lp = lp.float().to(dev).contiguous()
        a, b = bufs
        _lib.check(lib.sb_s2s_beam_select(
            lp.data_ptr(), a["state"].data_ptr(), a["c_scores"].data_ptr(), a["nodes"].data_ptr(),
            a["parent"].data_ptr(), a["tok"].data_ptr(), a["out"].data_ptr(), K, C, end_tok, step,
            max_len, a["node_cap"], a["c_cap"], sp), "beam select")
        _lib.check(lib.sb_s2s_beam_select_split(
            lp.data_ptr(), b["state"].data_ptr(), b["c_scores"].data_ptr(), b["nodes"].data_ptr(),
            b["parent"].data_ptr(), b["tok"].data_ptr(), b["out"].data_ptr(), K, C, end_tok, step,
            max_len, b["node_cap"], b["c_cap"], ws.data_ptr(), ws.numel(), sp), "beam split")
        torch.cuda.synchronize()
        for key in ("state", "nodes", "c_scores", "parent", "tok", "out"):
            assert torch.equal(a[key], b[key]), (step, key)


@pytest.mark.parametrize("split", [False, True])
def test_selection_breaks_ties_by_flat_index(cuda_lib, split):
    """The reference's stable descending sort over (beam row, class) candidates: equal float64
    scores keep ascending flat index r * C + c.  Integer logp make nearly every score a tie; no
    end token is ever selected, so every step keeps the K best candidates."""
    from speech_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda")
    K, C, max_len = 4, 6, 5
    g = torch.Generator().manual_seed(7)
    buf = _beam_buffers(lib, K, C, max_len, dev)
    sp = _lib.stream_ptr()
    _lib.check(lib.sb_s2s_beam_init(buf["state"].data_ptr(), buf["nodes"].data_ptr(),
                                    buf["tok"].data_ptr(), 0, sp), "beam init")
    n = ctypes.c_size_t(0)
    lib.sb_s2s_beam_split_workspace_size(K, C, ctypes.byref(n))
    ws = torch.empty(n.value, dtype=torch.uint8, device=dev)
    scores = [0.0]
    for step in range(max_len - 1):
        lp = torch.randint(-2, 1, (K, C), generator=g).float()
        lpd = lp.to(dev)
        args = (lpd.data_ptr(), buf["state"].data_ptr(), buf["c_scores"].data_ptr(),
                buf["nodes"].data_ptr(), buf["parent"].data_ptr(), buf["tok"].data_ptr(),
                buf["out"].data_ptr(), K, C, C, step, max_len, buf["node_cap"], buf["c_cap"])
        if split:
            _lib.check(lib.sb_s2s_beam_select_split(*args, ws.data_ptr(), ws.numel(), sp), "split")
        else:
            _lib.check(lib.sb_s2s_beam_select(*args, sp), "select")
        torch.cuda.synchronize()
        cand = sorted(((scores[r] + float(lp[r, c]), r * C + c) for r in range(len(scores))
                       for c in range(C)), key=lambda e: (-e[0], e[1]))[:K]
        assert buf["parent"].tolist() == [i // C for _, i in cand], step
        assert buf["tok"].tolist() == [i % C for _, i in cand], step
        scores = [s for s, _ in cand]


def test_public_class_end_to_end_at_4001_pieces(cuda_lib):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(5)
    np.random.seed(5)
    V = 4001
    m = Seq2Seq(40, V, _cfg(128)).cuda()
    inputs = [np.random.randn(80 - 9 * i, 40).astype(np.float32) for i in range(4)]
    labels = [[V - 1] + np.random.randint(0, V - 2, 7).tolist() + [V - 2] for _ in range(4)]
    batch = (inputs, labels)
    m.set_train()
    loss = m.loss(batch)
    loss.backward()
    assert torch.isfinite(loss).all()
    for name, p in m.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), name
    m.set_eval()
    hyps = m.infer(batch, max_len=10)
    assert len(hyps) == 4 and all(isinstance(t, int) for h in hyps for t in h)
    beam = m.beam_search(([inputs[0]], [labels[0]]), beam_size=8, max_len=10)
    assert len(beam) == 1 and all(isinstance(t, int) for t in beam[0])
