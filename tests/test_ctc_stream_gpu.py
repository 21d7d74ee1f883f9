"""GPU tests of streaming recognition: the GRU recurrence resumed from a state (sb_gru_fwd_h0), the
resumable CTC prefix beam search (sb_ctc_stream_*) and CTC.stream end to end.

Every equality here is bit for bit: a chunked run computes what one offline pass computes.
  * sb_gru_fwd_h0 on each forward kernel kind: frames [0, T1) with sb_gru_fwd, then the rest in
    chunks from the carried state, give sb_gru_fwd's y and xn over [0, T); from a random state the
    result is held to the rounding-faithful reference (tests/gru_ref.py).
  * the stream search: after every chunk, sb_ctc_stream_best equals sb_ctc_prefix_beam[_lm] over
    each stream's frames so far (labels, lengths, float64 scores), on both routes.
  * CTC.stream: the final partial(return_scores=True) equals decode_batch(with_scores=True) on the
    logits of the same B utterances in the exact-lengths mode.
"""
import ctypes

import numpy as np
import pytest
import torch

import gru_ref as R

gpu = pytest.mark.gpu

NO_KT, KT, NO_KS_FWD, KS2, STREAM = 8, 16, 32, 1024, 2048

# kind: (Bp, H, flags)
GRU_CASES = {
    "plain": (16, 128, 0),
    "kt": (8, 256, KT),
    "ks4": (24, 256, NO_KT),
    "ks2": (64, 512, NO_KT | KS2),
    "wide": (64, 256, STREAM),
}


def _lib():
    from speech_b200 import _lib
    return _lib


def _gru_ws(lib, Bp, H):
    from speech_b200 import ops
    n = ctypes.c_size_t(0)
    _lib().check(lib.sb_gru_fwd_workspace_size(Bp, H, 1, ctypes.byref(n)), "ws")
    return ops._workspace(n.value, "cuda"), n.value


def _fwd(lib, gi, whh, bhh, T, Bp, H, ws, nws):
    y = torch.full((T * Bp, H), float("nan"), device="cuda")
    xn = torch.zeros(T * Bp, H, dtype=torch.bfloat16, device="cuda")
    _lib().check(lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), y.data_ptr(),
                                xn.data_ptr(), None, ws.data_ptr(), nws, T, Bp, H, 1,
                                _lib().stream_ptr()), "sb_gru_fwd")
    return y, xn


def _fwd_h0(lib, gi, whh, bhh, h0, hb0, T, Bp, H, ws, nws, gates=None):
    y = torch.full(((T + 1) * Bp, H), float("nan"), device="cuda")
    xn = torch.zeros((T + 1) * Bp, H, dtype=torch.bfloat16, device="cuda")
    _lib().check(lib.sb_gru_fwd_h0(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), h0.data_ptr(),
                                   hb0.data_ptr(), y.data_ptr(), xn.data_ptr(),
                                   _lib().ptr(gates), ws.data_ptr(), nws, T, Bp, H, 1,
                                   _lib().stream_ptr()), "sb_gru_fwd_h0")
    return y, xn


@gpu
@pytest.mark.parametrize("kind", list(GRU_CASES))
def test_gru_h0_chunks_equal_one_pass(cuda_lib, kind):
    lib = cuda_lib
    Bp, H, flags = GRU_CASES[kind]
    T = 13
    g = torch.Generator().manual_seed(Bp + H)
    a = 1.0 / H ** 0.5
    whh = ((torch.rand(1, 3 * H, H, generator=g) * 2 - 1) * a).to(torch.bfloat16).cuda()
    bhh = ((torch.rand(1, 3 * H, generator=g) * 2 - 1) * a).cuda()
    gi = torch.randn(T * Bp, 3 * H, generator=g).cuda()
    lib.sb_debug_gru_flags(flags)
    try:
        ws, nws = _gru_ws(lib, Bp, H)
        y, xn = _fwd(lib, gi, whh, bhh, T, Bp, H, ws, nws)
        assert lib.sb_debug_gru_fwd_kernel().decode() == kind
        for cuts in ([1], [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12], [5, 6, 11]):
            y1, xn1 = _fwd(lib, gi[:cuts[0] * Bp], whh, bhh, cuts[0], Bp, H, ws, nws)
            ys, xns = [y1], [xn1]
            h, hb = y1[-Bp:], xn1[-Bp:]
            for t0, t1 in zip(cuts, cuts[1:] + [T]):
                yc, xc = _fwd_h0(lib, gi[t0 * Bp:t1 * Bp], whh, bhh, h, hb, t1 - t0, Bp, H, ws,
                                 nws)
                assert lib.sb_debug_gru_fwd_kernel().decode() == kind
                assert torch.equal(yc[:Bp], h) and torch.equal(xc[:Bp], hb)
                ys.append(yc[Bp:])
                xns.append(xc[Bp:])
                h, hb = yc[-Bp:], xc[-Bp:]
            assert torch.equal(torch.cat(ys), y), cuts
            assert torch.equal(torch.cat(xns), xn), cuts
        # from a random state: the rounding-faithful reference, teacher-forced by the kernel's y
        h0 = torch.randn(Bp, H, generator=g).tanh().cuda()
        gates = torch.full(((T + 1) * Bp, 1, 4, H), float("nan"), device="cuda")
        yr, xr = _fwd_h0(lib, gi, whh, bhh, h0, h0.to(torch.bfloat16), T, Bp, H, ws, nws, gates)
        assert lib.sb_debug_gru_fwd_kernel().decode() == kind
    finally:
        lib.sb_debug_gru_flags(0)
    gi0 = torch.cat([torch.zeros(Bp, 3 * H, device="cuda"), gi])
    ry, rg, _ = R.gru_fwd(gi0.cpu(), whh.cpu(), bhh.cpu(), T + 1, h_prev=yr)
    assert torch.equal(xr, yr.to(torch.bfloat16))
    err = R.fwd_err(yr[Bp:], gates[Bp:], ry[Bp:], rg[Bp:])
    assert err < R.FWD_ABS, err


# ---- the resumable search ---------------------------------------------------------------------
def _logp(B, T, S, seed, peaked=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, S, generator=g) * (4.0 if peaked else 1.5)
    return torch.log_softmax(x, -1).float().cuda()


def _offline(lib, logp, lens, K, blank, lm=None, shortlist=False):
    from speech_b200 import _lib as L
    B, T, S = logp.shape
    if lm is None:
        nb = L.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, K)
    else:
        nb = L.workspace_size(lib.sb_ctc_prefix_beam_lm_workspace_size, B, T, K, lm[0].order)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    lab = torch.empty(B, T, dtype=torch.int32, device="cuda")
    n = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = torch.empty(B, dtype=torch.float64, device="cuda")
    d_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    outs = (lab.data_ptr(), n.data_ptr(), sc.data_ptr(), ws.data_ptr(), nb, L.stream_ptr())
    if lm is None:
        fn = lib.sb_ctc_prefix_beam_shortlist if shortlist else lib.sb_ctc_prefix_beam
        L.check(fn(logp.data_ptr(), d_lens.data_ptr(), B, T, S, K, blank, *outs), "offline")
    else:
        fn = lib.sb_ctc_prefix_beam_lm_shortlist if shortlist else lib.sb_ctc_prefix_beam_lm
        tables, _ = lm[0].device_tables(logp.device)
        L.check(fn(logp.data_ptr(), d_lens.data_ptr(), B, T, S, K, blank, tables, lm[1], lm[2],
                   *outs), "offline lm")
    lab, n, sc = lab.cpu().numpy(), n.cpu().numpy(), sc.cpu().numpy()
    return [(tuple(lab[b, :n[b]].tolist()), float(sc[b])) for b in range(B)]


class _Search:
    """sb_ctc_stream_* over B streams, called through the C ABI"""

    def __init__(self, lib, B, K, max_frames, lm=None, shortlist=False):
        from speech_b200 import _lib as L
        self.lib, self.L, self.B, self.K, self.Tm, self.lm, self.sl = lib, L, B, K, max_frames, lm, \
            shortlist
        nb = L.workspace_size(lib.sb_ctc_stream_state_size, B, max_frames, K,
                              0 if lm is None else lm[0].order)
        self.state = torch.empty(nb, dtype=torch.uint8, device="cuda")
        self.reset(0, B)

    def reset(self, first, count):
        self.L.check(self.lib.sb_ctc_stream_reset(self.state.data_ptr(), self.B, self.Tm, self.K,
                                                  first, count, self.L.stream_ptr()), "reset")

    def step(self, logp, n, blank):
        lib, L = self.lib, self.L
        B, T, S = logp.shape
        nb = L.workspace_size(lib.sb_ctc_stream_workspace_size, B, T, self.K)
        ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
        d_n = torch.tensor(n, dtype=torch.int32, device="cuda")
        tail = (self.Tm, self.state.data_ptr(), ws.data_ptr(), nb, L.stream_ptr())
        if self.lm is None:
            fn = lib.sb_ctc_stream_step_shortlist if self.sl else lib.sb_ctc_stream_step
            L.check(fn(logp.data_ptr(), d_n.data_ptr(), B, T, S, self.K, blank, *tail), "step")
        else:
            fn = lib.sb_ctc_stream_step_lm_shortlist if self.sl else lib.sb_ctc_stream_step_lm
            tables, _ = self.lm[0].device_tables(logp.device)
            L.check(fn(logp.data_ptr(), d_n.data_ptr(), B, T, S, self.K, blank, tables,
                       self.lm[1], self.lm[2], *tail), "step lm")

    def best(self):
        B, Tm = self.B, self.Tm
        lab = torch.full((B, Tm), -7, dtype=torch.int32, device="cuda")
        n = torch.empty(B, dtype=torch.int32, device="cuda")
        sc = torch.empty(B, dtype=torch.float64, device="cuda")
        ovf = torch.empty(B, dtype=torch.int32, device="cuda")
        self.L.check(self.lib.sb_ctc_stream_best(self.state.data_ptr(), B, Tm, self.K,
                                                 lab.data_ptr(), n.data_ptr(), sc.data_ptr(),
                                                 ovf.data_ptr(), self.L.stream_ptr()), "best")
        lab, n, sc = lab.cpu().numpy(), n.cpu().numpy(), sc.cpu().numpy()
        return [(tuple(lab[b, :n[b]].tolist()), float(sc[b])) for b in range(B)], \
            ovf.cpu().numpy().tolist()


def _lm(S, order, seed):
    from speech_b200.lm import NGramLM
    rng = np.random.RandomState(seed)
    seqs = [rng.randint(0, S - 1, rng.randint(1, 12)).tolist() for _ in range(300)]
    return NGramLM.train(seqs, order, num_classes=S, blank=S - 1)


def _chunkings(rng, B, T):
    """per stream, a random split of [0, T) into chunks; some chunks empty"""
    out = []
    for _ in range(B):
        cuts = sorted(rng.choice(np.arange(0, T + 1), size=rng.randint(1, 6)).tolist())
        cuts = [0] + cuts + [T]
        out.append(list(zip(cuts[:-1], cuts[1:])))
    return out


SEARCH_CASES = [
    # (S, K, order, shortlist)
    (29, 1, 0, False), (29, 8, 0, False), (29, 32, 0, False), (29, 8, 0, True),
    (29, 8, 1, False), (29, 8, 3, False), (29, 32, 5, True), (29, 1, 3, True),
    (5000, 8, 0, False), (5000, 1, 0, False), (5000, 8, 3, False), (5000, 32, 0, False),
]


@gpu
@pytest.mark.parametrize("S,K,order,shortlist", SEARCH_CASES)
def test_stream_search_equals_offline_after_every_chunk(cuda_lib, S, K, order, shortlist):
    lib = cuda_lib
    B, T = 6, 40 if S == 29 else 24
    blank = S - 1
    rng = np.random.RandomState(S + K + order)
    logp = _logp(B, T, S, seed=K + order, peaked=(K == 1))
    lm = None if order == 0 else (_lm(S, order, order), 0.7, -0.3)
    st = _Search(lib, B, K, T, lm, shortlist)
    plan = _chunkings(rng, B, T)
    rounds = max(len(p) for p in plan)
    done = [0] * B
    for r in range(rounds):
        spans = [p[r] if r < len(p) else (done[b], done[b]) for b, p in enumerate(plan)]
        n = [e - s for s, e in spans]
        Tc = max(max(n), 1)
        chunk = torch.zeros(B, Tc, S, device="cuda")
        for b, (s, e) in enumerate(spans):
            chunk[b, :e - s] = logp[b, s:e]
        st.step(chunk, n, blank)
        done = [e for _, e in spans]
        got, ovf = st.best()
        want = _offline(lib, logp, done, K, blank, lm) if max(done) > 0 else None
        for b in range(B):
            if done[b] == 0:
                assert got[b] == ((), -0.0) or got[b] == ((), 0.0)
                continue
            assert got[b][0] == want[b][0], (r, b)
            assert got[b][1] == want[b][1], (r, b)
        assert ovf == [0] * B
    assert done == [T] * B
    # the forced shortlist route equals the full scan offline too
    assert got == _offline(lib, logp, [T] * B, K, blank, lm, shortlist=not shortlist)


@gpu
def test_stream_reset_one_slot_leaves_the_others(cuda_lib):
    lib = cuda_lib
    B, T, S, K = 4, 30, 29, 8
    logp = _logp(B, T, S, seed=3)
    st = _Search(lib, B, K, 2 * T)
    st.step(logp[:, :12].contiguous(), [12] * B, S - 1)
    st.reset(2, 1)
    st.step(logp[:, 12:].contiguous(), [T - 12] * B, S - 1)
    got, _ = st.best()
    want = _offline(lib, logp, [T] * B, K, S - 1)
    fresh = _offline(lib, logp[:, 12:].contiguous(), [T - 12] * B, K, S - 1)
    assert [got[b] for b in (0, 1, 3)] == [want[b] for b in (0, 1, 3)]
    assert got[2] == fresh[2]


@gpu
def test_stream_overflow_is_flagged_and_clamped(cuda_lib):
    lib = cuda_lib
    B, S, K, Tm = 3, 29, 8, 10
    logp = _logp(B, 16, S, seed=5)
    st = _Search(lib, B, K, Tm)
    # the state is followed by a guard region that must stay untouched
    guard = torch.randint(0, 255, (1 << 16,), dtype=torch.uint8, device="cuda")
    big = torch.cat([st.state, guard])
    st.state = big[:st.state.numel()]
    st.reset(0, B)
    st.step(logp[:, :8].contiguous(), [8, 8, 2], S - 1)
    st.step(logp[:, 8:].contiguous(), [8, 2, 8], S - 1)        # streams 0 and 2 pass Tm
    got, ovf = st.best()
    assert ovf == [1, 0, 0]
    want = _offline(lib, logp, [10, 10, 10], K, S - 1)
    assert got[0] == want[0] and got[1] == want[1]
    assert torch.equal(big[st.state.numel():], guard)


# ---- end to end -------------------------------------------------------------------------------
MODEL_CASES = {
    # name: (conv, GRU dim, layers, classes)
    "small": ([[8, 5, 8, 2], [8, 5, 8, 2]], 64, 2, 28),
    "wide": ([[8, 5, 8, 2], [8, 5, 8, 2]], 2128, 1, 28),
    "bench": ([[32, 5, 8, 2], [32, 5, 8, 2]], 1024, 2, 28),
}


def _model(name, seed):
    from speech_b200.models import CTC
    conv, dim, layers, V = MODEL_CASES[name]
    torch.manual_seed(seed)
    cfg = {"dropout": 0.0, "encoder": {"conv": conv, "rnn": {"dim": dim, "bidirectional": False,
                                                              "layers": layers}}}
    m = CTC(80, V, cfg).cuda()
    m.eval()
    return m


@gpu
@pytest.mark.parametrize("name,B,K,order", [
    ("small", 5, 1, 0), ("small", 5, 8, 3), ("wide", 3, 8, 0), ("bench", 16, 8, 0),
    ("bench", 4, 4, 2)])
def test_ctc_stream_equals_offline(cuda_lib, name, B, K, order):
    from speech_b200.models.ctc_decoder import decode_batch
    m = _model(name, seed=B + K)
    rng = np.random.RandomState(B + order)
    lens = rng.randint(20, 160, size=B).tolist()
    feats = [rng.randn(n, 80).astype(np.float32) for n in lens]
    lm = None if order == 0 else _lm(m.blank + 1, order, 1)
    kw = {} if lm is None else {"lm": lm, "lm_weight": 0.5, "insertion_bonus": 0.25}
    m.exact_lengths = True
    # offline: the same B utterances, exact-lengths mode
    x, _, x_lens, _ = m.collate(feats, [[0]] * B)
    elens = m.exact_lens(x_lens)
    with torch.no_grad():
        probs = m._forward_impl(x, elens, softmax=True)
    want = decode_batch(probs, beam_size=K, blank=m.blank, lens=elens, with_scores=True, **kw)
    st = m.stream(B, beam_size=K, max_frames=200, **kw)
    pos = [0] * B
    while any(p < n for p, n in zip(pos, lens)):
        chunks = []
        for b in range(B):
            k = int(rng.choice([0, 1, 1, 3, 8, 17, 40]))
            chunks.append(feats[b][pos[b]:pos[b] + k])
            pos[b] = min(pos[b] + k, lens[b])
        st.push(chunks)
    assert st.frames == [m.conv_out_size(n, 0) for n in lens]
    got = st.partial(return_scores=True)
    assert got == want
    assert st.partial() == [w[0] for w in want]


@gpu
def test_push_audio_features_equal_whole_utterance(cuda_lib):
    from speech_b200 import features
    from speech_b200.models import CTC
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                       "rnn": {"dim": 32, "bidirectional": False, "layers": 1}}}
    m = CTC(161, 28, cfg).cuda()
    m.eval()
    rng = np.random.RandomState(0)
    B = 3
    audio = [(rng.randn(n) * 3000).astype(np.int16) for n in (8000, 12345, 400)]
    whole, nf = features.log_specgram_batch(audio, 16000)
    st = m.stream(B)
    seen = [[] for _ in range(B)]
    push = st.push

    def spy(chunks):
        for b, c in enumerate(chunks):
            seen[b].append(torch.as_tensor(c).float().cpu())
        return push(chunks)
    st.push = spy
    pos = [0] * B
    while any(p < len(a) for p, a in zip(pos, audio)):
        pcm = []
        for b in range(B):
            k = int(rng.choice([0, 1, 159, 160, 161, 999, 3200]))
            pcm.append(audio[b][pos[b]:pos[b] + k])
            pos[b] += k
        st.push_audio(pcm)
    for b in range(B):
        got = torch.cat(seen[b])
        assert got.shape[0] == nf[b]
        assert torch.equal(got, whole[b, :nf[b]].cpu())
