"""GPU tests of the lookahead convolution (csrc/lookahead.cu, ops.GRUStackFunction, the models and
the streams).

  * kernels: sb_lookahead_fwd / _bwd against float64 autograd of F.conv1d over the right-padded,
    length-masked input, to fp32 rounding of their sums; rb == bf16(r); exact zeros past len_b;
    dW bit-identical across runs.
  * models: loss and every parameter's gradient against a float64 torch restatement of the encoder
    (conv2d + nn.GRU + conv1d + linear on the same weights), H not a multiple of 16.
  * exact lengths, FlatSGD / GradSync training, batches above one recurrence launch.
  * streams: CTC.stream after every push against decode_batch over the frames searched so far,
    and after finish() against the whole utterances, bit for bit; Transducer.stream after finish()
    against recognize, bit for bit.
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _la_ref(h, w, lens):
    """h (T, Bp, Hp) f64, w (tau+1, Hp) f64, lens (Bp) -> r (T, Bp, Hp): conv1d over h masked past
    len_b and padded by tau zero frames, zero past len_b"""
    T, Bp, Hp = h.shape
    tau = w.shape[0] - 1
    valid = (torch.arange(T, device=h.device)[:, None] < lens[None, :]).to(h.dtype)[:, :, None]
    x = (h * valid).permute(1, 2, 0)                                  # (Bp, Hp, T)
    r = F.conv1d(F.pad(x, (0, tau)), w.t().unsqueeze(1), groups=Hp)
    return r.permute(2, 0, 1) * valid


def _run(lib, h, w, lens, T, Bp, Hp, tau):
    from speech_b200 import _lib as L
    r = torch.full((T * Bp, Hp), float("nan"), device="cuda")
    rb = torch.zeros(T * Bp, Hp, dtype=torch.bfloat16, device="cuda")
    L.check(lib.sb_lookahead_fwd(h.data_ptr(), w.data_ptr(), L.ptr(lens), r.data_ptr(),
                                 rb.data_ptr(), T, Bp, Hp, tau, L.stream_ptr()), "fwd")
    return r, rb


def _bwd(lib, dr, h, w, lens, T, Bp, Hp, tau):
    from speech_b200 import _lib as L
    dh = torch.full((T * Bp, Hp), float("nan"), device="cuda")
    dw = torch.full((tau + 1, Hp), float("nan"), device="cuda")
    nb = L.workspace_size(lib.sb_lookahead_bwd_workspace_size, T, Bp, Hp, tau)
    ws = torch.full((nb,), 0xff, dtype=torch.uint8, device="cuda")
    L.check(lib.sb_lookahead_bwd(dr.data_ptr(), h.data_ptr(), w.data_ptr(), L.ptr(lens),
                                 dh.data_ptr(), dw.data_ptr(), ws.data_ptr(), nb, T, Bp, Hp, tau,
                                 L.stream_ptr()), "bwd")
    return dh, dw


@pytest.mark.parametrize("Bp", [8, 64, 128])
@pytest.mark.parametrize("Hp", [128, 1024])
@pytest.mark.parametrize("tau", [1, 5, 20, 32])
def test_kernels_match_float64_conv1d(cuda_lib, Bp, Hp, tau):
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(Bp * 7 + Hp + tau)
    for T in sorted({1, tau, 247}):
        for with_lens in (False, True):
            h = torch.randn(T * Bp, Hp, device="cuda", generator=g)
            w = torch.randn(tau + 1, Hp, device="cuda", generator=g) / (tau + 1) ** 0.5
            dr = torch.randn(T * Bp, Hp, device="cuda", generator=g)
            if with_lens:
                ln = torch.randint(0, T + 1, (Bp,), device="cuda", generator=g)
                ln[0] = 0
                ln[1] = min(T, max(0, tau - 1))
                ln[2] = T
                lens = ln.to(torch.int32)
            else:
                lens = None
            full = lens.long() if lens is not None else torch.full((Bp,), T, device="cuda")
            r, rb = _run(lib, h, w, lens, T, Bp, Hp, tau)
            assert torch.equal(rb, r.to(torch.bfloat16))
            past = (torch.arange(T, device="cuda")[:, None] >= full[None, :]).reshape(-1)
            assert torch.equal(r[past], torch.zeros_like(r[past]))
            h64 = h.double().view(T, Bp, Hp).requires_grad_(True)
            w64 = w.double().requires_grad_(True)
            ref = _la_ref(h64, w64, full)
            absref = _la_ref(h64.detach().abs(), w64.detach().abs(), full)
            err = (r.double().view(T, Bp, Hp) - ref.detach()).abs()
            assert bool((err <= 2 * (tau + 1) * U * absref + 1e-30).all()), (T, with_lens)
            ref.backward(dr.double().view(T, Bp, Hp))
            dh, dw = _bwd(lib, dr, h, w, lens, T, Bp, Hp, tau)
            assert torch.equal(dh[past], torch.zeros_like(dh[past]))
            # |dh| bound: the same chain over W and dr; |dW| bound: chains over a tile's frames
            # (at most 64) plus the reduction over the tiles x rows partials (at most their count)
            dr64 = dr.double().view(T, Bp, Hp)
            ha = h64.detach().abs().requires_grad_(True)
            wa = w64.detach().abs().requires_grad_(True)
            _la_ref(ha, wa, full).backward(dr64.abs())
            e_dh = (dh.double().view(T, Bp, Hp) - h64.grad).abs()
            assert bool((e_dh <= 2 * (tau + 1) * U * ha.grad + 1e-30).all()), (T, with_lens)
            parts = (T + 63) // 64 * Bp
            e_dw = (dw.double() - w64.grad).abs()
            assert bool((e_dw <= 2 * (64 + parts) * U * wa.grad + 1e-30).all()), (T, with_lens)
            _, dw2 = _bwd(lib, dr, h, w, lens, T, Bp, Hp, tau)
            assert torch.equal(dw.view(torch.int32), dw2.view(torch.int32))


# ---- models ------------------------------------------------------------------------------------
ENC = {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]], "rnn": {"dim": 40, "bidirectional": False,
                                                     "layers": 2}, "lookahead": 3}


def _family(kind, tau=3, exact=False):
    from speech_b200.models import CTC, Seq2Seq, Transducer
    enc = dict(ENC, lookahead=tau)
    cfg = {"dropout": 0.0, "exact_lengths": exact, "encoder": enc}
    if kind == "ctc":
        return CTC(80, 27, cfg)
    cfg["decoder"] = {"embedding_dim": 16, "layers": 1}
    return Transducer(80, 27, cfg) if kind == "rnnt" else Seq2Seq(80, 29, cfg)


def _ref_encode(m, x):
    """float64 restatement of the encoder with m's parameters (m on the CPU, float64)"""
    y = x.unsqueeze(1)
    for c in m.conv.children():
        if isinstance(c, torch.nn.Conv2d):
            y = torch.relu(F.conv2d(y, c.weight, c.bias, stride=c.stride))
    B, C, T, Fo = y.shape
    y = y.transpose(1, 2).reshape(B, T, C * Fo)
    h, _ = m.rnn(y)
    tau = m.lookahead.kernel_size[0] - 1
    return F.conv1d(F.pad(h.transpose(1, 2), (0, tau)), m.lookahead.weight,
                    groups=h.shape[2]).transpose(1, 2)


def _compare_grads(m, ref, names=None):
    for n, p in ref.named_parameters():
        if names is not None and not any(n.startswith(k) for k in names):
            continue
        g = dict(m.named_parameters())[n].grad
        assert g is not None, n
        g = g.double().cpu()
        r = p.grad
        rel = ((g - r).norm() / r.norm()).item()
        cos = (torch.dot(g.flatten(), r.flatten()) / (g.norm() * r.norm())).item()
        # the conv front-end's gradients arrive through every bf16 operand of the stack, and at
        # this size sum few, partly cancelling terms: they keep direction and size more loosely
        lo_cos, hi_rel = (0.995, 0.1) if n.startswith("conv.") else (0.999, 5e-2)
        assert cos > lo_cos and rel < hi_rel, (n, rel, cos)


def test_ctc_loss_and_gradients_match_float64(cuda_lib):
    torch.manual_seed(0)
    m = _family("ctc")
    ref = copy.deepcopy(m).double()
    m.cuda()
    rng = np.random.RandomState(0)
    B = 5
    inputs = [rng.randn(90, 80).astype(np.float32) for _ in range(B)]
    labels = [rng.randint(0, 27, 6).tolist() for _ in range(B)]
    loss = m.loss((inputs, labels))
    loss.backward()
    x = torch.from_numpy(np.stack(inputs)).double()
    logits = F.linear(_ref_encode(ref, x), ref.fc.fc.weight, ref.fc.fc.bias)
    T = logits.shape[1]
    lp = torch.log_softmax(logits, 2).transpose(0, 1)
    want = F.ctc_loss(lp, torch.tensor(sum(labels, [])), torch.full((B,), T),
                      torch.tensor([len(l) for l in labels]), blank=27, reduction="sum")
    want.backward()
    assert abs(loss.item() - want.item()) / want.item() < 5e-3, (loss.item(), want.item())
    _compare_grads(m, ref)
    assert m.lookahead.weight.grad.shape == (40, 1, 4)


@pytest.mark.parametrize("kind", ["rnnt", "s2s"])
def test_encoder_gradients_match_float64(cuda_lib, kind):
    torch.manual_seed(1)
    m = _family(kind)
    ref = copy.deepcopy(m).double()
    m.cuda()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(5, 90, 80, generator=g)
    enc = m.encode(x.cuda())
    want = _ref_encode(ref, x.double())
    assert enc.shape == want.shape
    assert (enc.detach().double().cpu() - want.detach()).abs().max().item() < 3e-2
    G = torch.randn(want.shape, generator=g)
    (enc * G.cuda()).sum().backward()
    (want * G.double()).sum().backward()
    _compare_grads(m, ref, names=("conv.", "rnn.", "lookahead."))


def test_exact_lengths_each_utterance_equals_itself_alone(cuda_lib):
    torch.manual_seed(3)
    m = _family("ctc", tau=4, exact=True).cuda()
    m.set_eval()
    rng = np.random.RandomState(3)
    lens = [30, 95, 61, 22, 80]
    inputs = [rng.randn(n, 80).astype(np.float32) for n in lens]
    labels = [[1]] * len(lens)
    out = m((inputs, labels))
    for b, n in enumerate(lens):
        t = m.conv_out_size(n, 0)
        alone = m(([inputs[b]], [[1]]))
        assert alone.shape[1] == t
        assert (out[b, :t] - alone[0]).abs().max().item() < 2e-3, b


def test_parity_mode_with_a_lookahead_is_not_implemented(cuda_lib):
    m = _family("ctc", tau=2).cuda()
    m.parity_mode = True
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="lookahead"):
            m.encode_logits(torch.zeros(2, 40, 80, device="cuda"))


def test_flat_sgd_lowers_the_loss_and_grad_sync_carries_the_gradient(cuda_lib):
    from speech_b200.optim import FlatSGD
    from speech_b200.parallel import GradSync
    torch.manual_seed(4)
    m = _family("ctc", tau=5).cuda()
    rng = np.random.RandomState(4)
    batch = ([rng.randn(70, 80).astype(np.float32) for _ in range(6)],
             [rng.randint(0, 27, 5).tolist() for _ in range(6)])
    opt = FlatSGD(m, lr=1e-3, momentum=0.9)
    w0 = m.lookahead.weight.detach().clone()
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss = m.loss(batch)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0], losses
    assert not torch.equal(m.lookahead.weight.detach(), w0)

    torch.manual_seed(5)
    m = _family("ctc", tau=5).cuda()
    want = torch.autograd.grad(m.loss(batch), [m.lookahead.weight])[0]
    sync = GradSync(m, 1)
    m.loss(batch).backward()
    sync.all_reduce()
    o0, o1 = sync.offsets[id(m.lookahead.weight)]
    assert torch.equal(sync.flat[o0:o1].view_as(want), want)
    assert want.abs().sum().item() > 0


def test_batches_above_one_launch_sum_their_chunks(cuda_lib):
    torch.manual_seed(6)
    m = _family("ctc", tau=2).cuda()
    rng = np.random.RandomState(6)
    B = 136
    inputs = [rng.randn(40, 80).astype(np.float32) for _ in range(B)]
    labels = [rng.randint(0, 27, 3).tolist() for _ in range(B)]
    got = torch.autograd.grad(m.loss((inputs, labels)), [m.lookahead.weight])[0]
    parts = [torch.autograd.grad(m.loss((inputs[i:i + 128], labels[i:i + 128])),
                                 [m.lookahead.weight])[0] for i in (0, 128)]
    assert torch.allclose(got, parts[0] + parts[1], rtol=1e-5, atol=1e-6)


# ---- streams -----------------------------------------------------------------------------------
def _ctc_stream_model(tau, seed):
    from speech_b200.models import CTC
    torch.manual_seed(seed)
    cfg = {"dropout": 0.0, "exact_lengths": True,
           "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                       "rnn": {"dim": 40, "bidirectional": False, "layers": 2}, "lookahead": tau}}
    m = CTC(80, 28, cfg).cuda()
    m.set_eval()
    return m


def _lm(S, order, seed):
    from speech_b200.lm import NGramLM
    rng = np.random.RandomState(seed)
    seqs = [rng.randint(0, S - 1, rng.randint(1, 12)).tolist() for _ in range(300)]
    return NGramLM.train(seqs, order, num_classes=S, blank=S - 1)


@pytest.mark.parametrize("tau", [1, 4])
@pytest.mark.parametrize("chunk", [1, 3, 0])
@pytest.mark.parametrize("order", [0, 3])
def test_ctc_stream_equals_offline(cuda_lib, tau, chunk, order):
    from speech_b200.models.ctc_decoder import decode_batch
    m = _ctc_stream_model(tau, seed=tau + chunk)
    rng = np.random.RandomState(tau * 10 + chunk + order)
    B, K = 4, 4
    lens = [23, 61, 40, 75]
    feats = [rng.randn(n, 80).astype(np.float32) for n in lens]
    kw = {} if order == 0 else {"lm": _lm(m.blank + 1, order, 1), "lm_weight": 0.5,
                                "insertion_bonus": 0.25}
    x, _, x_lens, _ = m.collate(feats, [[0]] * B)
    elens = m.exact_lens(x_lens)
    with torch.no_grad():
        probs = m._forward_impl(x, elens, softmax=True)
    want = decode_batch(probs, beam_size=K, blank=m.blank, lens=elens, with_scores=True, **kw)
    st = m.stream(B, beam_size=K, max_frames=100, **kw)
    pos = [0] * B
    done = set()
    while any(p < n for p, n in zip(pos, lens)):
        chunks = []
        for b in range(B):
            k = lens[b] if chunk == 0 else chunk
            chunks.append(feats[b][pos[b]:pos[b] + k])
            pos[b] = min(pos[b] + k, lens[b])
        st.push(chunks)
        for b in range(B):
            n = max(0, m.conv_out_size(pos[b], 0))
            held = 0 if b in done else min(tau, n)
            assert (st.frames[b], st.pending[b]) == (n - held, held), (b, pos[b])
        if min(st.frames) > 0:
            part = decode_batch(probs, beam_size=K, blank=m.blank,
                                lens=torch.tensor(st.frames, dtype=torch.int32),
                                with_scores=True, **kw)
            assert st.partial(return_scores=True) == part, pos
        # stream 0 ends first; the others go on
        if pos[0] == lens[0] and 0 not in done:
            st.finish([0])
            done.add(0)
            assert st.pending[0] == 0
            assert st.partial(return_scores=True)[0] == want[0]
    st.finish()
    assert st.pending == [0] * B
    assert st.frames == [m.conv_out_size(n, 0) for n in lens]
    assert st.partial(return_scores=True) == want


def test_transducer_stream_equals_recognize_after_finish(cuda_lib):
    from speech_b200.models import Transducer
    torch.manual_seed(7)
    cfg = {"dropout": 0.0, "exact_lengths": True,
           "encoder": {"conv": [[4, 5, 5, 2]], "rnn": {"dim": 24, "bidirectional": False,
                                                       "layers": 2}, "lookahead": 2},
           "decoder": {"embedding_dim": 16, "layers": 1}}
    m = Transducer(40, 28, cfg).cuda()
    for p in m.parameters():
        p.data.mul_(2.0)
    m.set_eval()
    rng = np.random.RandomState(7)
    B = 8
    lens = rng.randint(40, 120, size=B).tolist()
    feats = [rng.randn(n, 40).astype(np.float32) for n in lens]
    kw = dict(beam_size=4, max_symbols_per_frame=4)
    st = m.stream(B, max_frames=100, **kw)
    pos = [0] * B
    while any(p < n for p, n in zip(pos, lens)):
        chunks = []
        for b in range(B):
            k = int(rng.choice([0, 1, 2, 5, 8, 17]))
            chunks.append(feats[b][pos[b]:pos[b] + k])
            pos[b] = min(pos[b] + k, lens[b])
        st.push(chunks)
    assert st.pending == [min(2, m.conv_out_size(n, 0)) for n in lens]
    st.finish()
    labels, scores = m.recognize(feats, return_scores=True, **kw)
    assert st.partial(return_scores=True) == [(tuple(l), s) for l, s in zip(labels, scores)]


def test_push_after_finish_raises_until_reset(cuda_lib):
    m = _ctc_stream_model(2, seed=8)
    rng = np.random.RandomState(8)
    st = m.stream(2, beam_size=2)
    f = rng.randn(30, 80).astype(np.float32)
    st.push([f, f])
    st.finish([1])
    with pytest.raises(ValueError):
        st.push([f[:0], f[:5]])
    with pytest.raises(ValueError):
        st.push_audio([np.zeros(0, np.int16), np.ones(400, np.int16)])
    st.push([f[:5], f[:0]])              # the open stream goes on; an empty chunk is accepted
    st.reset(1)
    st.push([f[:0], f])
    st.finish()
    single = m.stream(1, beam_size=2)
    single.push([f])
    single.finish()
    assert st.frames[1] == single.frames[0]


def test_pickle_from_before_the_layer_runs_as_before(cuda_lib):
    """a model pickled before the lookahead existed (tests/golden) runs without the layer: its
    logits equal those of the same weights in a model built now without the key"""
    import os
    from speech_b200.models import CTC
    old = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                  "ctc_before_lookahead.pt"), weights_only=False).cuda()
    assert old.lookahead is None
    cfg = {"dropout": 0.0, "encoder": {"conv": [[4, 5, 8, 2]],
                                       "rnn": {"dim": 24, "bidirectional": False, "layers": 1}}}
    new = CTC(80, 27, cfg).cuda()
    new.load_state_dict(old.state_dict())
    rng = np.random.RandomState(9)
    batch = ([rng.randn(n, 80).astype(np.float32) for n in (60, 45, 80)], [[1], [2], [3]])
    old.set_eval()
    new.set_eval()
    assert torch.equal(old(batch), new(batch))
    assert old.infer(batch, beam_size=4) == new.infer(batch, beam_size=4)
