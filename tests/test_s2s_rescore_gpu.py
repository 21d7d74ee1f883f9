"""GPU tests of two-pass decoding of the attention model: the CTC head's prefix beam search gives
an N-best (sb_ctc_stream_nbest), the attention decoder scores each entry teacher-forced
(functions/s2s.py: score_batch -> sb_s2s_score_tokens), and the combination picks one
(Seq2Seq.recognize_two_pass, Seq2Seq.stream -> streaming.Seq2SeqStream).

- N-best: entry 0 after one whole-utterance step equals the offline search (ctc_decoder._run on
  the same float32 log-probabilities) bit for bit, at K = 1 / 4 / 10 / 32, lens < T, and at
  C = 5000 (the shortlist route); every entry equals the float64 reference beam of
  tests/s2s_rescore_ref.py (labels exact, c to 1e-12 relative); uneven chunks give the same bits.
- scoring: the teacher-forced score of recognize's own result (ctc_weight = 0) is recognize's
  score bit for bit, K = 1 / 4 / 10, both padding modes, and on the many-CTA projection; a_i
  against decode_step logits log-softmaxed in float64 (1e-5 per token); an empty hypothesis
  scores l(END | START).
- end to end: recognize_two_pass equals the reference combination over the GPU's c_i and a_i;
  w = 1 gives the first pass's best; each utterance's result is the one it gets alone.
- stream: after finish, rescored(return_scores=True) equals recognize_two_pass bit for bit
  (uneven chunks, a lookahead layer, push_audio, reset), and partial() equals the offline search
  over the frames searched so far.
"""
import numpy as np
import pytest
import torch

from s2s_rescore_ref import nbest_prefix_beam, select

pytestmark = pytest.mark.gpu


def _cfg(H=32, layers=1, exact=False, lookahead=0, bidirectional=False, w=0.3):
    enc = {"conv": [[8, 5, 8, 2]], "rnn": {"dim": H, "bidirectional": bidirectional,
                                           "layers": layers}}
    if lookahead:
        enc["lookahead"] = lookahead
    cfg = {"dropout": 0.0, "encoder": enc,
           "decoder": {"embedding_dim": H, "layers": 1, "ctc_weight": w}}
    if exact:
        cfg["exact_lengths"] = True
    return cfg


def _model(V, seed, F=40, sharpen=2.0, **kw):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(seed)
    m = Seq2Seq(F, V, _cfg(**kw)).cuda()
    m.set_eval()
    with torch.no_grad():
        m.fc.fc.weight.mul_(sharpen)
        m.embedding.weight.mul_(3.0)
        m.ctc_fc.fc.weight.mul_(4.0)
    return m


def _inputs(T, n=3, step=9, seed=0, F=40):
    rng = np.random.RandomState(seed)
    return [rng.randn(T - step * i, F).astype(np.float32) for i in range(n)]


def _encode(m, inputs):
    lens = m.input_lens(inputs)
    with torch.no_grad():
        x = m._encode(m.stage_inputs(inputs), lens)
        y = torch.log_softmax(m.ctc_fc(x).float(), dim=-1).contiguous()
    return x, y, lens


def _logp(B, T, C, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, C, generator=g) * scale
    return torch.log_softmax(x, -1).float().cuda().contiguous()


def _offline(logp, lens, K):
    from speech_b200.models import ctc_decoder
    C = logp.shape[2]
    return ctc_decoder._run(logp, torch.tensor(lens, dtype=torch.int32).cuda(), K, C - 1)


# ---- N-best ------------------------------------------------------------------------------------

@pytest.mark.parametrize("C", [12, 5000])
@pytest.mark.parametrize("K", [1, 4, 10, 32])
def test_nbest_entry_0_is_the_offline_search(cuda_lib, K, C):
    from speech_b200.functions import s2s
    B, T = 3, 30
    logp = _logp(B, T, C, K + C)
    lens = [T, T - 7, 13]
    labels, ln, c = s2s.ctc_first_pass(logp, lens, K)
    ref = _offline(logp, lens, K)
    ln, c, labels = ln.cpu(), c.cpu(), labels.cpu()
    for b in range(B):
        n = int(ln[b, 0])
        assert tuple(labels[b, 0, :n].tolist()) == tuple(ref[b][0]), (K, C, b)
        assert -c[b, 0].item() == ref[b][1], (K, C, b)


@pytest.mark.parametrize("K", [1, 4, 10, 32])
def test_nbest_equals_the_reference_beam(cuda_lib, K):
    from speech_b200.functions import s2s
    B, T, C = 3, 16, 6
    logp = _logp(B, T, C, 100 + K, scale=1.5)
    lens = [T, 11, 5]
    labels, ln, c = s2s.ctc_first_pass(logp, lens, K)
    labels, ln, c = labels.cpu(), ln.cpu(), c.cpu()
    lp = logp.cpu().double().numpy()
    for b in range(B):
        ref = nbest_prefix_beam(lp[b, :lens[b]], K, C - 1)
        for i in range(K):
            if i >= len(ref):
                assert int(ln[b, i]) == -1 and c[b, i].item() == -float("inf")
                continue
            n = int(ln[b, i])
            assert tuple(labels[b, i, :n].tolist()) == ref[i][0], (K, b, i)
            assert abs(c[b, i].item() - ref[i][1]) <= 1e-12 * abs(ref[i][1]), (K, b, i)


@pytest.mark.parametrize("C,K", [(12, 4), (12, 32), (5000, 4)])
def test_stream_search_nbest_of_uneven_chunks_is_the_same(cuda_lib, C, K):
    from speech_b200.functions import s2s
    from speech_b200.models.ctc_decoder import StreamSearch
    B, T = 3, 40
    logp = _logp(B, T, C, 7 + K)
    lens = [T, 29, 17]
    whole = s2s.ctc_first_pass(logp, lens, K)
    search = StreamSearch(B, T, K, C - 1, logp.device)
    rng = np.random.RandomState(K)
    pos = [0] * B
    while any(p < n for p, n in zip(pos, lens)):
        step = [min(int(rng.choice([0, 1, 3, 8])), n - p) for p, n in zip(pos, lens)]
        Tc = max(max(step), 1)
        chunk = torch.zeros(B, Tc, C, device="cuda")
        for b in range(B):
            chunk[b, :step[b]] = logp[b, pos[b]:pos[b] + step[b]]
        search.push(chunk.contiguous(), step)
        pos = [p + s for p, s in zip(pos, step)]
    got = search.nbest()
    ln = whole[1].cpu()
    assert torch.equal(got[1].cpu(), ln)
    assert torch.equal(got[2].cpu(), whole[2].cpu())
    for b in range(B):
        for i in range(K):
            n = int(ln[b, i])
            if n > 0:
                assert torch.equal(got[0][b, i, :n].cpu(), whole[0][b, i, :n].cpu())


# ---- scoring -----------------------------------------------------------------------------------

def _tokens(hyps, K, V):
    """(R, L + 2) token matrix and lens of B*K hypotheses (None: an empty slot)"""
    L = max([len(h) for h in hyps if h is not None] + [0])
    tok = torch.full((len(hyps), L + 2), V - 2, dtype=torch.int32)
    tok[:, 0] = V - 1
    lens = torch.full((len(hyps),), -1, dtype=torch.int32)
    for r, h in enumerate(hyps):
        if h is not None:
            tok[r, 1:1 + len(h)] = torch.tensor(h, dtype=torch.int32)
            lens[r] = len(h)
    return tok.cuda(), lens.cuda()


@pytest.mark.parametrize("V,H", [(11, 32), (5001, 64)])
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("K", [1, 4, 10])
def test_score_of_recognize_result_is_recognize_score(cuda_lib, K, exact, V, H):
    from speech_b200.functions import s2s
    m = _model(V, 40 + K, H=H, exact=exact, sharpen=2.0 if V < 100 else 1.0)
    if V > 100:
        assert not s2s.fc_fused(H, V - 1)
    inputs = _inputs(70, n=5, step=5, seed=K)
    bias = m.fc.fc.bias[V - 2].item()
    # raise END's bias until some hypothesis completes with labels within max_len; where none
    # does, the last bias's (empty) completions are still checked
    for extra in np.arange(-6.0, 6.01, 0.5):
        with torch.no_grad():
            m.fc.fc.bias[V - 2] = bias + float(extra)
        labels, scores = m.recognize(inputs, beam_size=K, max_len=60, return_scores=True)
        done = [lab[-1] == V - 2 for lab in labels]
        if any(d and len(lab) > 2 for d, lab in zip(done, labels)):
            break
    assert any(done), labels
    x, _, lens = _encode(m, inputs)
    hyps = []
    for d, lab in zip(done, labels):
        assert lab[0] == V - 1
        hyps += [lab[1:-1] if d else None] + [None] * (K - 1)
    tok, ln = _tokens(hyps, K, V)
    with torch.no_grad():
        a = s2s.score_batch(m, x, tok, ln, K, lens).cpu()
    for b in range(len(inputs)):
        if done[b]:
            assert a[b * K].item() == scores[b], (K, exact, V, b)
        assert all(a[b * K + i].item() == 0.0 for i in range(1, K))


def test_scores_follow_decode_step(cuda_lib):
    """an independent check of which tokens are gathered: decode_step logits of the forced
    prefix, log-softmaxed in float64 on the host and summed (1e-5 per token)"""
    from speech_b200.functions import s2s
    V, K = 11, 3
    m = _model(V, 50)
    inputs = _inputs(60, n=2, seed=5)
    x, _, _ = _encode(m, inputs)
    rng = np.random.RandomState(3)
    hyps = [rng.randint(0, V - 2, n).tolist() for n in (0, 4, 9, 2, 7, 1)]
    tok, ln = _tokens(hyps, K, V)
    with torch.no_grad():
        a = s2s.score_batch(m, x, tok, ln, K).cpu()
    for r, h in enumerate(hyps):
        eh = x[r // K:r // K + 1]
        state, ref = None, 0.0
        seq = [V - 1] + h + [V - 2]
        with torch.no_grad():
            for u in range(len(h) + 1):
                out, state = m.decode_step(eh, torch.tensor([[seq[u]]]).cuda(), state)
                lp = torch.log_softmax(out.double(), -1)[0]
                ref += lp[seq[u + 1]].item()
        assert abs(a[r].item() - ref) <= 1e-5 * (len(h) + 1), (r, a[r].item(), ref)


def test_empty_hypothesis_scores_end_after_start(cuda_lib):
    from speech_b200.functions import s2s
    V, K = 11, 2
    m = _model(V, 51)
    x, _, _ = _encode(m, _inputs(60, n=2, seed=6))
    tok, ln = _tokens([[], None, [], [3]], K, V)
    with torch.no_grad():
        a = s2s.score_batch(m, x, tok, ln, K).cpu()
        for b in range(2):
            lp, _ = m.decode_step(x[b:b + 1], torch.tensor([[V - 1]]).cuda(), None, softmax=True)
            assert abs(a[b * K].item() - lp[0, V - 2].item()) <= 1e-6
    assert a[1].item() == 0.0


# ---- end to end --------------------------------------------------------------------------------

@pytest.mark.parametrize("w", [0.0, 0.3, 0.5, 1.0])
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("K", [1, 4, 10])
def test_two_pass_equals_the_reference_combination(cuda_lib, K, exact, w):
    from speech_b200.functions import s2s
    V = 11
    m = _model(V, 60 + K, exact=exact)
    inputs = _inputs(80, n=3, seed=K + 1)
    labels, scores = m.recognize_two_pass(inputs, beam_size=K, ctc_weight=w, return_scores=True)
    x, y, lens = _encode(m, inputs)
    B, T, _ = y.shape
    frames = lens if lens is not None else [T] * B
    with torch.no_grad():
        nl, nn_, nc = s2s.ctc_first_pass(y, frames, K)
        hyps = [None if int(nn_[b, i]) < 0 else nl[b, i, :int(nn_[b, i])].tolist()
                for b in range(B) for i in range(K)]
        tok, ln = _tokens(hyps, K, V)
        a = s2s.score_batch(m, x, tok, ln, K, lens).cpu().view(B, K)
    c = nc.cpu()
    ref = _offline(y, frames, K)
    for b in range(B):
        n = sum(h is not None for h in hyps[b * K:(b + 1) * K])
        i, r = select(a[b, :n].tolist(), c[b, :n].tolist(), w)
        assert labels[b] == [V - 1] + hyps[b * K + i] + [V - 2], (K, w, b)
        assert scores[b] == r, (K, w, b)
        if w == 1.0:
            assert labels[b][1:-1] == list(ref[b][0]) and scores[b] == -ref[b][1]


@pytest.mark.parametrize("K", [1, 4])
def test_each_utterance_gets_its_own_result(cuda_lib, K):
    """exact-lengths mode: each utterance's result from its encoder states alone is the batch's"""
    from speech_b200.functions import s2s
    m = _model(11, 70, exact=True)
    inputs = _inputs(90, n=3, step=13, seed=9)
    x, y, lens = _encode(m, inputs)
    with torch.no_grad():
        batch = s2s.recognize_two_pass(m, x, y, lens, K, 0.4, True)
        for b, n in enumerate(lens):
            one = s2s.recognize_two_pass(m, x[b:b + 1, :n], y[b:b + 1, :n], [n], K, 0.4, True)
            assert one[0][0] == batch[0][b] and one[1][0] == batch[1][b], (K, b)


# ---- stream ------------------------------------------------------------------------------------

def _feed(st, inputs, rng, sizes=(0, 1, 5, 16, 33)):
    pos = [0] * len(inputs)
    while any(p < len(x) for p, x in zip(pos, inputs)):
        chunks = []
        for b, x in enumerate(inputs):
            k = min(int(rng.choice(sizes)), len(x) - pos[b])
            chunks.append(x[pos[b]:pos[b] + k])
            pos[b] += k
        st.push(chunks)


@pytest.mark.parametrize("tau", [0, 3])
@pytest.mark.parametrize("K", [1, 4, 10])
def test_stream_equals_two_pass(cuda_lib, K, tau):
    from speech_b200.models import ctc_decoder
    m = _model(11, 80 + K, exact=True, lookahead=tau)
    inputs = _inputs(200, n=3, step=31, seed=K)      # B * T' >= 128: ctc_fc on the GEMM
    want = m.recognize_two_pass(inputs, beam_size=K, ctc_weight=0.3, return_scores=True)
    _, y, lens = _encode(m, inputs)
    st = m.stream(3, beam_size=K, max_frames=200, ctc_weight=0.3)
    rng = np.random.RandomState(K + tau)
    half = [x[:len(x) // 2] for x in inputs]
    _feed(st, half, rng)
    f = st.frames
    got = st.partial(return_scores=True)
    ref = _offline(y[:, :max(f)].contiguous(), f, K)
    assert [g[0] for g in got] == [r[0] for r in ref]
    assert [g[1] for g in got] == [r[1] for r in ref]
    _feed(st, [x[len(x) // 2:] for x in inputs], rng)
    st.finish()
    assert st.frames == lens
    assert st.rescored(return_scores=True) == want
    got = st.partial(return_scores=True)
    ref = ctc_decoder._run(y, torch.tensor(lens, dtype=torch.int32).cuda(), K, 9)
    assert got == [(r[0], r[1]) for r in ref]


def test_stream_reset_isolates_a_stream(cuda_lib):
    m = _model(11, 90, exact=True, lookahead=2)
    inputs = _inputs(160, n=3, step=17, seed=4)
    other = _inputs(120, n=3, step=5, seed=5)
    want = m.recognize_two_pass([inputs[0], other[1], inputs[2]], beam_size=4,
                                return_scores=True)
    st = m.stream(3, beam_size=4, max_frames=160)
    rng = np.random.RandomState(1)
    _feed(st, inputs, rng)
    st.finish([1])
    st.reset(1)
    _feed(st, [np.zeros((0, 40), np.float32), other[1], np.zeros((0, 40), np.float32)], rng)
    st.finish()
    assert st.rescored(return_scores=True) == want


def test_stream_push_audio_equals_two_pass(cuda_lib):
    from speech_b200 import features
    m = _model(11, 91, F=161, exact=True, lookahead=2)
    rng = np.random.RandomState(2)
    audio = [(rng.randn(n) * 3000).astype(np.int16) for n in (16000, 12345, 9000)]
    whole, nf = features.log_specgram_batch(audio, 16000)
    want = m.recognize_two_pass([whole[b, :nf[b]].cpu().numpy() for b in range(3)],
                                beam_size=4, return_scores=True)
    st = m.stream(3, beam_size=4, max_frames=200)
    pos = [0] * 3
    while any(p < len(a) for p, a in zip(pos, audio)):
        pcm = []
        for b in range(3):
            k = int(rng.choice([0, 159, 160, 999, 3200]))
            pcm.append(audio[b][pos[b]:pos[b] + k])
            pos[b] += len(pcm[-1])
        st.push_audio(pcm)
    st.finish()
    assert st.rescored(return_scores=True) == want
