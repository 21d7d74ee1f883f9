"""GPU tests of Transducer streaming (transducer_decoders.StreamSearch, streaming.TransducerStream).

- the search alone, over static lattices: after every push the stream's best hypothesis equals
  search_batch over each stream's frames so far, labels, lengths and float64 scores bit for bit,
  on both candidate routes (the stream's shortlist route reads 64-entry lists from the first
  frame), with and without an n-gram LM, and with chunkings that leave streams at different
  offsets, push zero frames, and push odd frame counts (the beam-block parity copy);
- the tie lattice, where the offline search reruns from 64-entry lists;
- reset of one slot mid-stream;
- end to end: Transducer.stream against Transducer.recognize in the exact-lengths mode with the
  same B, after every push where the offline fc1 runs on the GEMM (B * T' >= 128, or H not a
  multiple of 8); push_audio against the whole-utterance featuriser."""
import numpy as np
import pytest
import torch

from test_rnnt_lm_gpu import StaticRows
from test_rnnt_shortlist_host import tie_lattice

pytestmark = pytest.mark.gpu


class StreamRows:
    """row provider of a stream over a (B, T, U1, V1) lattice: the row of a slot at frame t of a
    push is lat[b, base_b + t, its length], base_b the frames stream b had before the push"""

    def __init__(self, lat, blank):
        self.lat, self.blank = lat, blank
        self.B, self.T, self.U1, self.V1 = lat.shape
        self.device = lat.device
        self.base = torch.zeros(self.B, dtype=torch.int64, device=self.device)

    def begin(self, slots):
        pass

    def rows(self, t, block, slots):
        from speech_b200.transducer_decoders import shortlists_of_lp
        u = slots.slot_lens.long().clamp(0, self.U1 - 1)
        f = (self.base + t).clamp(max=self.T - 1)
        rows = self.lat[torch.arange(self.B, device=self.device)[:, None], f[:, None], u]
        if slots.lp is not None:
            slots.lp.copy_(rows)
        if slots.sl is not None:
            for a, b in zip(slots.sl, shortlists_of_lp(rows[:, None].contiguous(), slots.kp,
                                                      self.blank)):
                a.copy_(b)

    def extend(self, src, dst, slots):
        pass

    def arenas(self):
        return None, 0, 0, None, 0


def _lattice(rng, B, T, U, V, scale=2.0):
    x = rng.randn(B, T, U, V).astype(np.float32) * scale
    x -= np.log(np.exp(x.astype(np.float64)).sum(-1, keepdims=True)).astype(np.float32)
    return torch.from_numpy(x)


def _lm(V1, order, seed):
    from speech_b200.lm import NGramLM
    rng = np.random.RandomState(seed)
    seqs = [rng.randint(0, V1 - 1, rng.randint(1, 15)).tolist() for _ in range(300)]
    return NGramLM.train(seqs, order, num_classes=V1, blank=V1 - 1)


def _schedule(rng, B, T, pushes):
    """per push, the frame count of every stream: zeros, ones and odd counts, streams apart"""
    left = [T] * B
    plan = []
    for r in range(pushes):
        counts = []
        for b in range(B):
            n = int(rng.choice([0, 1, 1, 2, 3, 5, 7])) if r < pushes - 1 else left[b]
            n = min(n, left[b])
            left[b] -= n
            counts.append(n)
        plan.append(counts)
    return plan


def _offline(lat, frames, K, blank, S, max_len, lm_args):
    from speech_b200.transducer_decoders import search_batch
    Tn = max(frames)
    lab, sc = search_batch(StaticRows(lat[:, :max(Tn, 1)].contiguous(), blank), frames, K, blank,
                           S, max_len, *lm_args)
    return lab, sc


SEARCH_CASES = [
    # V+1, K, S, LM order, max_len; routes: full at (29, *) and (1000, 4), shortlists otherwise
    (29, 1, 1, 0, None), (29, 4, 4, 0, None), (29, 8, 4, 1, None), (29, 32, 1, 3, None),
    (29, 4, 4, 5, 5), (1000, 4, 4, 0, None), (1000, 4, 1, 3, None), (1000, 32, 4, 0, None),
    (1000, 32, 1, 5, None), (1000, 32, 4, 1, 6), (20001, 8, 4, 0, None), (20001, 8, 1, 3, None),
]


@pytest.mark.parametrize("V1,K,S,order,max_len", SEARCH_CASES)
def test_stream_search_equals_offline_after_every_push(cuda_lib, V1, K, S, order, max_len):
    from speech_b200.transducer_decoders import StreamSearch, decode_static_fits
    rng = np.random.RandomState(V1 + K + S + order)
    B, T, U1 = (5, 24, 10) if V1 < 20000 else (3, 10, 6)
    blank = V1 - 1
    lat = _lattice(rng, B, T, U1, V1).cuda()
    lm_args = () if order == 0 else (_lm(V1, order, order), 0.6, -0.4)
    rows = StreamRows(lat, blank)
    st = StreamSearch(rows, K, S, T, blank, max_len, *lm_args)
    assert (st.kp is None) == decode_static_fits(K, V1)
    frames = [0] * B
    odd = False
    for counts in _schedule(rng, B, T, 7):
        rows.base = torch.tensor(frames, dtype=torch.int64, device="cuda")
        st.push(counts)
        odd |= any(n % 2 for n in counts)
        frames = [f + n for f, n in zip(frames, counts)]
        assert st.frames == frames
        want = _offline(lat, frames, K, blank, S, max_len, lm_args)
        got = st.best()
        assert got == want, (counts, frames)
    assert frames == [T] * B and odd


def test_tie_lattice_stream_gives_the_rerun_answer(cuda_lib):
    from speech_b200.transducer_decoders import StreamSearch, search_batch
    lat, blank = tie_lattice()
    lp = torch.from_numpy(lat[None]).cuda()
    want = search_batch(StaticRows(lp, blank), [2], 2, blank, 1, 1)
    for plan in ([[2]], [[1], [1]], [[0], [1], [0], [1]]):
        rows = StreamRows(lp, blank)
        st = StreamSearch(rows, 2, 1, 4, blank, 1)
        assert st.kp == 64
        done = 0
        for counts in plan:
            rows.base = torch.tensor([done], dtype=torch.int64, device="cuda")
            st.push(counts)
            done += counts[0]
        assert st.best() == want


@pytest.mark.parametrize("V1,K", [(29, 4), (1000, 32)])
def test_reset_one_slot_leaves_the_others(cuda_lib, V1, K):
    from speech_b200.transducer_decoders import StreamSearch
    rng = np.random.RandomState(V1)
    B, T, U1, S = 4, 20, 8, 2
    blank = V1 - 1
    lat = _lattice(rng, B, T, U1, V1).cuda()
    new = _lattice(rng, 1, T, U1, V1).cuda()
    rows = StreamRows(lat.clone(), blank)
    st = StreamSearch(rows, K, S, 2 * T, blank)
    st.push([7, 3, 5, 0])
    frames = [7, 3, 5, 0]
    st.reset(2)
    assert st.frames == [7, 3, 0, 0]
    rows.lat[2] = new[0]                           # slot 2 takes a new utterance from frame 0
    frames[2] = 0
    for counts in ([4, 1, 6, 3], [0, 9, 3, 2]):
        rows.base = torch.tensor(frames, dtype=torch.int64, device="cuda")
        st.push(counts)
        frames = [f + n for f, n in zip(frames, counts)]
    got = st.best()
    want = _offline(lat, frames, K, blank, S, None, ())
    fresh = _offline(new, frames[2:3], K, blank, S, None, ())
    for b in (0, 1, 3):
        assert (got[0][b], got[1][b]) == (want[0][b], want[1][b]), b
    assert (got[0][2], got[1][2]) == (fresh[0][0], fresh[1][0])


# ---- end to end -------------------------------------------------------------------------------
def _model(H, layers, E, V1, seed, F=40):
    from speech_b200.models import Transducer
    torch.manual_seed(seed)
    cfg = {"dropout": 0.0, "exact_lengths": True,
           "encoder": {"conv": [[4, 5, 5, 2]], "rnn": {"dim": H, "bidirectional": False,
                                                       "layers": 2}},
           "decoder": {"embedding_dim": E, "layers": layers}}
    m = Transducer(F, V1 - 1, cfg).cuda()
    for p in m.parameters():                        # peakier rows than the default init
        p.data.mul_(2.0)
    m.set_eval()
    return m


E2E_CASES = [
    # H, prediction layers, embedding, V+1, beam, S, LM order
    (20, 1, 16, 29, 4, 4, 0),          # fused joint, H not a multiple of 8
    (24, 2, 16, 29, 4, 2, 3),          # fused joint, offline fc1 on the GEMM where B*T' >= 128
    (20, 2, 24, 1024, 4, 3, 0),        # slab joint, full route
    (32, 1, 16, 1024, 4, 4, 2),
    (20, 1, 16, 5001, 8, 2, 0),        # slab joint, shortlist route (64-entry lists)
    (24, 2, 16, 5001, 8, 2, 3),
]


@pytest.mark.parametrize("H,layers,E,V1,K,S,order", E2E_CASES)
def test_transducer_stream_equals_recognize(cuda_lib, H, layers, E, V1, K, S, order):
    m = _model(H, layers, E, V1, seed=H + V1 + order)
    rng = np.random.RandomState(H + layers + order)
    B = 8
    lens = rng.randint(40, 120, size=B).tolist()
    feats = [rng.randn(n, 40).astype(np.float32) for n in lens]
    kw = dict(beam_size=K, max_symbols_per_frame=S)
    if order:
        kw.update(lm=_lm(V1, order, 7), lm_weight=0.5, insertion_bonus=0.25)
    st = m.stream(B, max_frames=100, **kw)
    pos = [0] * B
    checked = 0
    first = True
    while any(p < n for p, n in zip(pos, lens)):
        chunks = []
        for b in range(B):
            k = 9 if first else int(rng.choice([0, 1, 1, 2, 5, 8, 17]))
            chunks.append(feats[b][pos[b]:pos[b] + k])
            pos[b] = min(pos[b] + k, lens[b])
        first = False
        st.push(chunks)
        frames = st.frames
        assert frames == [max(0, m.conv_out_size(p, 0)) for p in pos]
        got = st.partial(return_scores=True)
        if B * max(frames) >= 128 or H % 8:
            labels, scores = m.recognize([f[:p] for f, p in zip(feats, pos)],
                                         return_scores=True, **kw)
            assert got == [(tuple(l), s) for l, s in zip(labels, scores)], pos
            checked += 1
    assert checked >= 3
    assert st.partial() == [g[0] for g in got]
    # one slot restarted mid-stream: its next utterance equals a fresh decode of it, and the
    # prediction state of the empty hypothesis is restored in its arena rows
    st.reset(3)
    assert st.frames[3] == 0 and st.partial()[3] == ()
    p = 0
    for k in (6, 0, 1, 30, 200):
        chunks = [f[:0] for f in feats]
        chunks[3] = feats[5][p:p + k]
        p += k
        st.push(chunks)
    inputs = list(feats)
    inputs[3] = feats[5]
    labels, scores = m.recognize(inputs, return_scores=True, **kw)
    want = [(tuple(l), s) for l, s in zip(labels, scores)]
    after = st.partial(return_scores=True)
    assert after == want
    assert after[:3] + after[4:] == got[:3] + got[4:]


def test_push_audio_features_equal_whole_utterance(cuda_lib):
    from speech_b200 import features
    m = _model(20, 1, 16, 29, seed=0, F=161)
    rng = np.random.RandomState(0)
    B = 3
    audio = [(rng.randn(n) * 3000).astype(np.int16) for n in (8000, 12345, 4000)]
    whole, nf = features.log_specgram_batch(audio, 16000)
    st = m.stream(B, beam_size=4)
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
    inputs = [whole[b, :nf[b]].cpu().numpy() for b in range(B)]
    labels, scores = m.recognize(inputs, beam_size=4, return_scores=True)
    assert st.partial(return_scores=True) == [(tuple(l), s) for l, s in zip(labels, scores)]
