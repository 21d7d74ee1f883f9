"""GPU tests of the exact-lengths mode (`"exact_lengths": true`): every output of an utterance is
what the utterance gives alone in a batch of one.

Tolerances are the ones the existing parity tests use for the same quantities: encoder states
2e-2 absolute (test_encode_matches_reference_output), logits 3e-2 absolute and costs 2e-3 relative
(test_models_gpu).  Gradients of a mixed batch are compared with the sum of the per-utterance
gradients at 1e-2 relative L2 per parameter: both sides run the same bf16 kernels on the same
rows, so they differ only in fp32 accumulation order (atomic split-K weight gradients, GEMM
tiling), far below the 5e-2 that test_zz_northstar_grads_gpu allows against an fp32 reference.
The default (padded) mode must miss these bounds, so the comparison can fail.
"""
import numpy as np
import pytest
import torch

from exact_lengths_ref import packed_encode

pytestmark = pytest.mark.gpu

ENC = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                   "rnn": {"dim": 32, "bidirectional": True, "layers": 2}},
       "decoder": {"embedding_dim": 32, "layers": 1}}
LENS = [100, 40, 73, 58, 91, 47]          # input frames; 6 utterances, Bp = 8 padding rows


def _cfg(exact, bidirectional=True, dropout=0.0):
    c = {"dropout": dropout, "exact_lengths": exact,
         "encoder": {"conv": ENC["encoder"]["conv"],
                     "rnn": {"dim": 32, "bidirectional": bidirectional, "layers": 2}},
         "decoder": ENC["decoder"]}
    return c


def _batch(lens, F=40, V=10, seed=0):
    rng = np.random.RandomState(seed)
    inputs = [rng.randn(n, F).astype(np.float32) for n in lens]
    labels = [rng.randint(0, V, 2 + (i % 3)).tolist() for i in range(len(lens))]
    return inputs, labels


def _model(family, exact, seed=0, **kw):
    import speech_b200.models as models
    torch.manual_seed(seed)
    vocab = 12 if family == "Seq2Seq" else 10      # Seq2Seq: + start (11) and end (10) tokens
    return getattr(models, family)(40, vocab, _cfg(exact, **kw)).cuda()


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


# ---- 1. the alignment kernel ----------------------------------------------------------------
def _ref_align(a, lens, T, Bp, right):
    out = torch.zeros_like(a)
    A, O = a.view(T, Bp, -1), out.view(T, Bp, -1)
    for b in range(Bp):
        s = T - lens[b]
        if right:
            O[s:, b] = A[:T - s, b]
        else:
            O[:T - s, b] = A[s:, b]
    return out


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("cols,off", [(24, 0), (13, 3), (256, 8)])
def test_time_align_matches_indexing(cuda_lib, dtype, cols, off):
    from speech_b200 import ops
    T, B, Bp = 7, 5, 8
    lens = [1, 7, 3, 6, 2] + [T] * (Bp - B)               # len = 1, len = T, padding rows = T
    lens_dev = torch.tensor(lens, dtype=torch.int32, device="cuda")
    wide = torch.randn(T * Bp, cols + off + 8, device="cuda").to(dtype)   # 16-byte rows for (24, 0), (256, 8)
    src = wide[:, off:off + cols]                         # a column block of a wider matrix
    for right in (True, False):
        got = ops.time_align(src, lens_dev, T, Bp, right)
        assert torch.equal(got, _ref_align(src.contiguous(), lens, T, Bp, right))
    # out-of-place into a column block, then back: the valid rows round-trip exactly
    dst = torch.full((T * Bp, cols + 2), 7.0, device="cuda").to(dtype)
    ops.time_align(src, lens_dev, T, Bp, True, out=dst[:, 2:])
    assert bool((dst[:, :2] == 7.0).all())
    back = ops.time_align(dst[:, 2:], lens_dev, T, Bp, False)
    keep = (torch.arange(T, device="cuda")[:, None] < lens_dev[None, :]).reshape(T * Bp, 1)
    assert torch.equal(back, torch.where(keep, src, torch.zeros_like(src)))


# ---- 2. all lengths equal: the mode changes nothing --------------------------------------------
@pytest.mark.parametrize("family", ["CTC", "Transducer", "Seq2Seq"])
def test_equal_lengths_bit_identical_to_default(cuda_lib, family, monkeypatch):
    """Same code path (no alignment runs), so logits and loss are bit-identical.  Gradients are
    compared at fp32 reordering noise, because the default mode itself does not reproduce them
    bit for bit: accumulating GEMMs split K and add their partials with atomicAdd (csrc/gemm.cu,
    epilogue of SB_GEMM_ACCUMULATE; every weight gradient), and the joint network's fc2 bias
    gradient and the conv bias gradients are atomicAdd column sums (csrc/joint.cu, csrc/conv.cu),
    so the order of fp32 additions varies from run to run."""
    from speech_b200 import ops
    inputs, labels = _batch([80] * 5)
    if family == "Seq2Seq":
        labels = [[11] + l + [10] for l in labels]
    runs = []
    for exact in (False, True):
        if exact:
            def boom(*a, **k):
                raise AssertionError("alignment must be skipped when every len_b == T'")
            monkeypatch.setattr(ops, "time_align", boom)
        m = _model(family, exact)
        with torch.no_grad():
            out = m((inputs, labels))
        loss = m.loss((inputs, labels))
        loss.backward()
        runs.append((out, loss.detach(), _grads(m)))
    (o0, l0, g0), (oe, le, ge) = runs
    assert torch.equal(o0, oe) and torch.equal(l0, le)
    assert g0.keys() == ge.keys()
    for n in g0:
        assert (ge[n] - g0[n]).abs().max().item() <= 1e-5 * g0[n].abs().max().item() + 1e-7, n


# ---- 3. encoder against nn.GRU over pack_padded_sequence ---------------------------------------
@pytest.mark.parametrize("bidirectional", [False, True])
def test_encoder_matches_packed_oracle(cuda_lib, bidirectional):
    from oracle.model_ref import RefEncoder
    from speech_b200.models import Model
    torch.manual_seed(0)
    cfg = _cfg(True, bidirectional)
    m = Model(40, cfg)
    ref = RefEncoder(40, cfg).double()
    ref.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    m.cuda()
    inputs, labels = _batch(LENS + [64])                  # B = 7
    x, _, x_lens, _ = m.lattice_batch(inputs, labels)
    with torch.no_grad():
        y = m.encode(x, x_lens).cpu().double()
        r, lens = packed_encode(ref, x.cpu().double(), [len(i) for i in inputs])
    assert x_lens.tolist() == lens.tolist()
    for b, L in enumerate(lens.tolist()):
        assert (y[b, :L] - r[b, :L]).abs().max().item() < 2e-2, b
        assert float(y[b, L:].abs().sum()) == 0.0


@pytest.mark.parametrize("bidirectional,dropout", [(False, 0.0), (True, 0.0), (True, 0.3)])
def test_gru_stack_input_gradient(cuda_lib, bidirectional, dropout):
    """Input gradient of ops.gru_stack with lens: exactly zero at frames >= len_b (whatever
    arrives there from above), and the packed nn.GRU's gradient at the valid frames."""
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    from speech_b200 import ops
    torch.manual_seed(0)
    rnn = torch.nn.GRU(24, 32, 2, batch_first=True, bidirectional=bidirectional).cuda()
    lens = [31, 9, 1, 24, 31, 17, 5]
    B, T = len(lens), max(lens)
    x = torch.randn(B, T, 24, device="cuda", requires_grad=True)
    g = torch.randn(B, T, 32 * (2 if bidirectional else 1), device="cuda")
    y = ops.gru_stack(x, rnn, dropout=dropout, lens=lens)
    (y * g).sum().backward()
    assert torch.isfinite(x.grad).all()
    for b, L in enumerate(lens):
        assert float(x.grad[b, L:].abs().sum()) == 0.0, b
        assert float(y[b, L:].detach().abs().sum()) == 0.0, b
    if dropout:
        return
    r64 = torch.nn.GRU(24, 32, 2, batch_first=True, bidirectional=bidirectional).double()
    r64.load_state_dict({k: v.double().cpu() for k, v in rnn.state_dict().items()})
    x64 = x.detach().double().cpu().requires_grad_(True)
    out, _ = r64(pack_padded_sequence(x64, torch.tensor(lens), batch_first=True,
                                      enforce_sorted=False))
    out, _ = pad_packed_sequence(out, batch_first=True, total_length=T)
    (out * g.double().cpu()).sum().backward()
    for b, L in enumerate(lens):
        assert (y[b, :L].double().cpu() - out[b, :L]).abs().max().item() < 2e-2
    gx = x.grad.double().cpu()
    assert (gx - x64.grad).abs().max().item() < 3e-2 * x64.grad.abs().max().item() + 1e-4


# ---- 4. batch-composition invariance ----------------------------------------------------------
def _per_utterance(family, m, inputs, labels):
    """(logits / log-probs at the valid frames, cost) of every utterance, from one batch."""
    from speech_b200.functions import ctc, transducer
    x, y, x_lens, y_lens = m.collate(inputs, labels)
    with torch.no_grad():
        out = m((inputs, labels))
        if family == "CTC":
            costs, _ = ctc.ctc_costs_and_grads(out, y, x_lens, y_lens, need_grad=False)
        else:
            costs, _ = transducer.rnnt_costs_and_grads(out, y, x_lens, y_lens, blank=m.blank,
                                                       need_grad=False)
    res = []
    for b, L in enumerate(x_lens.tolist()):
        o = out[b, :L] if family == "CTC" else out[b, :L, :len(labels[b]) + 1]
        res.append((o.cpu(), float(costs[b])))
    return res


def _invariance_errors(family, exact):
    inputs, labels = _batch(LENS, seed=1)
    m = _model(family, exact)
    batch = _per_utterance(family, m, inputs, labels)
    m.zero_grad()
    m.loss((inputs, labels)).backward()
    gb = _grads(m)
    gsum = {}
    e_logit = e_cost = 0.0
    for b in range(len(inputs)):
        alone_in, alone_lab = [inputs[b]], [labels[b]]
        (o1, c1), = _per_utterance(family, m, alone_in, alone_lab)
        ob, cb = batch[b]
        L = min(o1.shape[0], ob.shape[0])
        e_logit = max(e_logit, (ob[:L] - o1[:L]).abs().max().item()
                      + (0.0 if ob.shape[0] == o1.shape[0] else float("inf")))
        e_cost = max(e_cost, abs(cb - c1) / abs(c1))
        m.zero_grad()
        m.loss((alone_in, alone_lab)).backward()
        for n, g in _grads(m).items():
            gsum[n] = gsum[n] + g if n in gsum else g
    e_grad = max(_rel(gb[n], gsum[n]) for n in gsum)
    return e_logit, e_cost, e_grad


@pytest.mark.parametrize("family", ["CTC", "Transducer"])
def test_batch_composition_invariance(cuda_lib, family):
    e_logit, e_cost, e_grad = _invariance_errors(family, exact=True)
    assert e_logit < 3e-2 and e_cost < 2e-3 and e_grad < 1e-2, (e_logit, e_cost, e_grad)
    d_logit, d_cost, d_grad = _invariance_errors(family, exact=False)
    print("%s: exact %.2e %.2e %.2e, default %.2e %.2e %.2e"
          % (family, e_logit, e_cost, e_grad, d_logit, d_cost, d_grad))
    assert d_cost > 2e-3 and d_grad > 1e-2, (d_logit, d_cost, d_grad)


# ---- 5. decoders -----------------------------------------------------------------------------
@pytest.mark.parametrize("beam", [1, 8])
def test_ctc_infer_decodes_each_utterance_over_its_frames(cuda_lib, beam):
    from oracle import ctc_decoder_ref
    m = _model("CTC", True)
    m.set_eval()
    inputs, labels = _batch(LENS, seed=2)
    _, _, x_lens, _ = m.collate(inputs, labels)
    with torch.no_grad():
        probs = torch.softmax(m((inputs, labels)), 2).cpu().numpy()
    preds = m.infer((inputs, labels), beam_size=beam)
    for b, L in enumerate(x_lens.tolist()):
        ref = ctc_decoder_ref.prefix_beam_search(probs[b, :L], beam, m.blank)[0]
        assert tuple(preds[b]) == tuple(ref), b


def test_transducer_infer_decodes_each_utterance_over_its_frames(cuda_lib):
    from oracle import decode_static_ref
    m = _model("Transducer", True)
    m.set_eval()
    inputs, labels = _batch(LENS, seed=3)
    _, _, x_lens, _ = m.collate(inputs, labels)
    with torch.no_grad():
        lp = m((inputs, labels)).cpu().numpy()
    preds = m.infer((inputs, labels), beam_size=4)
    for b, L in enumerate(x_lens.tolist()):
        ref = decode_static_ref.decode_static(lp[b, :L, :len(labels[b]) + 1], 4, m.blank)[0]
        assert list(preds[b]) == list(ref), b


# ---- 6. masked attention ----------------------------------------------------------------------
@pytest.mark.parametrize("log_t", [False, True])
def test_masked_attention_decode_matches_oracle(cuda_lib, log_t):
    """s2s.decode with lens (sb_s2s_attn_fwd / _bwd) on a padded batch against the masked
    float64 restatement, which equals each utterance run alone (test_exact_lengths_host); bounds
    of test_teacher_forced_decode_forward_and_backward.  Padded frames get exactly zero
    alignment and zero gradient."""
    from exact_lengths_ref import masked_decode_ref
    from speech_b200.functions import s2s
    from speech_b200.models import Seq2Seq
    torch.manual_seed(1)
    cfg = _cfg(True)
    cfg["decoder"] = {"embedding_dim": 64, "layers": 1, "log_t": log_t}
    cfg["encoder"]["rnn"]["dim"] = 64
    m = Seq2Seq(40, 12, cfg).cuda()
    lens = [61, 1, 24, 25, 48, 61]          # 24 frames per CTA: tiles wholly past len_b exit
    B, T, H, U = len(lens), max(lens), 64, 7
    x = (torch.randn(B, T, H) * 0.5).cuda()
    for b, L in enumerate(lens):
        x[b, L:] = 3.0                      # padding that would change every score if attended
    x.requires_grad_(True)
    y = torch.randint(0, 11, (B, U)).cuda()
    out, al = s2s.decode(m, x, y, [False] * U, lens)
    w = torch.randn_like(out)
    (out * w).sum().backward()
    ro, ra, rx, rp = masked_decode_ref(m, x, y, lens)
    (ro * w.double().cpu()).sum().backward()
    assert (out.double().cpu() - ro).abs().max().item() < 1e-4 * max(1.0, ro.abs().max().item())
    assert (al.double().cpu() - ra).abs().max().item() < 1e-5
    assert abs(al.sum(2) - 1).max().item() < 1e-5
    g = x.grad.double().cpu()
    assert (g - rx.grad).abs().max().item() < 2e-3 * rx.grad.abs().max().item() + 1e-6
    for b, L in enumerate(lens):
        assert float(al[b, :, L:].detach().abs().sum()) == 0.0
        assert float(x.grad[b, L:].abs().sum()) == 0.0
    for name, p in m.named_parameters():
        if name not in rp:
            continue
        ref = rp[name].grad
        got = p.grad.double().cpu().reshape(ref.shape)
        tol = 2e-2 if name in ("dec_rnn.weight_ih", "dec_rnn.weight_hh", "fc.fc.weight") else 2e-3
        floor = 1e-5 if name == "attend.nn.1.fc.bias" else 1e-6
        assert (got - ref).abs().max().item() < tol * ref.abs().max().item() + floor, name


@pytest.mark.parametrize("log_t", [False, True])
def test_masked_attn_step_matches_each_utterance_alone(cuda_lib, log_t):
    """NNAttention.forward with lens (sb_s2s_attn_fwd), first and later steps, against the
    unmasked kernel on each utterance alone; bound of test_attn_step_kernel_matches_reference_
    formulation."""
    from speech_b200.models.seq2seq import NNAttention
    torch.manual_seed(2)
    H, lens = 32, [50, 3, 24, 49]
    att = NNAttention(H, log_t=log_t).cuda()
    B, T = len(lens), max(lens)
    eh = torch.randn(B, T, H).cuda()
    dhx = torch.randn(B, 1, H).cuda()
    with torch.no_grad():
        sx0, ax0 = att(eh, dhx, None, lens)
        sx1, ax1 = att(eh, dhx, ax0, lens)
        for b, L in enumerate(lens):
            a0 = att(eh[b:b + 1, :L], dhx[b:b + 1], None)
            a1 = att(eh[b:b + 1, :L], dhx[b:b + 1], a0[1])
            for (s_ref, a_ref), s, a in ((a0, sx0, ax0), (a1, sx1, ax1)):
                assert (s[b] - s_ref[0]).abs().max().item() < 1e-4 * max(1.0, s_ref.abs().max().item())
                assert (a[b, :L] - a_ref[0]).abs().max().item() < 1e-4
                assert float(a[b, L:].abs().sum()) == 0.0


def test_seq2seq_mixed_batch_matches_each_utterance_alone(cuda_lib):
    """Loss and greedy hypotheses of a mixed-length batch against each utterance alone.  All label
    sequences have one length: the reference scores end-padding of labels (seq2seq.py:58-63),
    which is not what this mode is about."""
    m = _model("Seq2Seq", True)
    m.set_eval()
    inputs, labels = _batch(LENS, seed=5)
    labels = [[11] + np.random.RandomState(b).randint(0, 10, 4).tolist() + [10]
              for b in range(len(LENS))]
    with torch.no_grad():
        total = m.loss((inputs, labels)).item() * len(inputs)      # loss is the batch mean
        hyps = m.infer((inputs, labels), max_len=12)
        alone_loss = [m.loss(([inputs[b]], [labels[b]])).item() for b in range(len(inputs))]
        alone_hyp = [m.infer(([inputs[b]], [labels[b]]), max_len=12)[0]
                     for b in range(len(inputs))]
    assert abs(total - sum(alone_loss)) / sum(alone_loss) < 2e-3, (total, alone_loss)

    def upto_end(h):
        return h[:h.index(10) + 1] if 10 in h[1:] else h
    for b in range(len(inputs)):
        n = len(upto_end(alone_hyp[b]))
        assert upto_end(hyps[b])[:n] == upto_end(alone_hyp[b]), b


# ---- 7. training ---------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["CTC", "Transducer", "Seq2Seq"])
def test_training_in_exact_mode(cuda_lib, family):
    from speech_b200.optim import FlatSGD
    m = _model(family, True)
    opt = FlatSGD(m, lr=1e-2)
    inputs, labels = _batch(LENS, seed=4)
    if family == "Seq2Seq":
        labels = [[11] + l + [10] for l in labels]
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = m.loss((inputs, labels))
        loss.backward()
        assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)
        opt.step()
        losses.append(loss.item())
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
