"""GPU tests of the label-free transducer beam search (csrc/rnnt_search.cu,
transducer_decoders.search_batch, Transducer.recognize).

- search kernels: with static rows lat[t, len(h)] and S = max_len = U - 1 the device loop is
  sb_rnnt_decode_static bit for bit (labels, lengths, float64 scores), on both candidate routes;
- model: labels equal the rounding-faithful oracle (oracle/rnnt_search_ref.py) wherever its
  smallest selection gap exceeds 1e-4, scores to a relative 1e-5;
- with a zero embedding the prediction network ignores the labels, so recognize is `infer`'s
  search on the teacher-forced lattice."""
import math

import numpy as np
import pytest
import torch

from oracle import decode_static_ref, rnnt_search_ref as ref
from test_rnnt_shortlist_host import tie_lattice

pytestmark = pytest.mark.gpu


class StaticRows:
    """row provider of a (B, T, U1, V1) lattice: the row of a slot is lat[b, t, its length]"""

    def __init__(self, lat, blank):
        self.lat, self.blank = lat, blank
        self.B, self.T, self.U1, self.V1 = lat.shape
        self.device = lat.device

    def begin(self, slots):
        pass

    def rows(self, t, block, slots):
        from speech_b200.transducer_decoders import shortlists_of_lp
        u = slots.slot_lens.long().clamp(0, self.U1 - 1)
        rows = self.lat[torch.arange(self.B, device=self.device)[:, None], t, u]
        if slots.kp is None:
            slots.lp.copy_(rows)
        else:
            for a, b in zip(slots.sl, shortlists_of_lp(rows[:, None].contiguous(), slots.kp,
                                                      self.blank)):
                a.copy_(b)

    def extend(self, src, dst, slots):
        pass

    def arenas(self):
        return None, 0, 0, None, 0


def _lattice(rng, B, T, U, V, scale=1.0):
    x = rng.randn(B, T, U, V) * scale
    return torch.from_numpy((x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32))


def _static_both(lat, tlens, K, blank):
    from speech_b200.transducer_decoders import decode_static_batch, search_batch
    B, T, U1, V = lat.shape
    want = decode_static_batch(lat, tlens, [U1] * B, K, blank)
    got = search_batch(StaticRows(lat, blank), tlens, K, blank, U1 - 1, U1 - 1)
    return want, got


@pytest.mark.parametrize("K,V", [(1, 29), (4, 29), (32, 29), (4, 1000), (32, 1000), (8, 20001)])
def test_static_rows_bit_identical_to_decode_static(cuda_lib, K, V):
    from speech_b200.transducer_decoders import decode_static_fits
    rng = np.random.RandomState(K * 31 + V)
    B, T, U1 = 5, 9 if V > 5000 else 14, 5
    lat = _lattice(rng, B, T, U1, V, scale=2.0).cuda()
    tlens = [T, T - 3, 1, 0, T]
    for blank in (V - 1, 0):
        (wl, ws), (gl, gs) = _static_both(lat, tlens, K, blank)
        assert gl == wl and gs == ws, (blank, decode_static_fits(K, V))
    assert gl[3] == [] and gs[3] == 0.0                  # 0 frames: empty hypothesis, score 0


def test_static_rows_tie_lattice_reruns(cuda_lib):
    from speech_b200.transducer_decoders import search_batch
    lat, blank = tie_lattice()
    lp = torch.from_numpy(lat[None]).cuda()
    want = decode_static_ref.decode_static(lat, 2, blank)
    got = search_batch(StaticRows(lp, blank), [2], 2, blank, 1, 1)
    assert (got[0][0], got[1][0]) == want


def _model(H, bidir, layers, E, V, exact, seed=0):
    from speech_b200.models import Transducer
    torch.manual_seed(seed)
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": [[4, 5, 5, 2]], "rnn": {"dim": H, "bidirectional": bidir,
                                                       "layers": 1}},
           "decoder": {"embedding_dim": E, "layers": layers}}
    m = Transducer(40, V - 1, cfg).cuda()
    for p in m.parameters():                        # peakier rows than the default init
        p.data.mul_(2.0)
    m.set_eval()
    return m


def _inputs(rng, lens):
    return [rng.randn(n, 40).astype(np.float32) for n in lens]


CASES = [  # H, bidir, layers, E, V+1, beam, exact
    (24, True, 1, 16, 11, 1, False),
    (24, False, 2, 24, 11, 4, True),
    (20, True, 1, 12, 11, 8, False),
    (20, False, 2, 16, 300, 4, True),
    (24, True, 1, 16, 300, 32, False),
]


@pytest.mark.parametrize("H,bidir,layers,E,V1,beam,exact", CASES)
def test_model_equals_rounding_faithful_oracle(cuda_lib, H, bidir, layers, E, V1, beam, exact):
    from speech_b200.models.transducer_model import PredictionRows
    from speech_b200.transducer_decoders import search_batch
    m = _model(H, bidir, layers, E, V1, exact, seed=H + V1 + beam)
    rng = np.random.RandomState(beam)
    inputs = _inputs(rng, [40, 31, 36, 24])
    rows = PredictionRows(m, inputs)
    S = 2
    labels, scores = search_batch(rows, rows.tlens, beam, m.blank, S, None)
    assert labels == m.recognize(inputs, beam_size=beam, max_symbols_per_frame=S)
    decisive = 0
    for b in range(len(inputs)):
        oracle = ref.LabelFreeRows(m, rows.fxT[:, b])
        want, wscore, gap = ref.search(oracle, rows.tlens[b], beam, m.blank, S, 10 ** 9)
        assert abs(scores[b] - wscore) <= 1e-5 * abs(wscore) + 1e-6, (b, scores[b], wscore)
        if gap > 1e-4:
            decisive += 1
            assert labels[b] == want, b
    assert decisive >= len(inputs) // 2, decisive


def test_zero_embedding_is_infer_on_the_teacher_forced_lattice(cuda_lib):
    from speech_b200.transducer_decoders import decode_static_batch
    m = _model(24, True, 1, 16, 11, False, seed=7)
    m.embedding.weight.data.zero_()
    rng = np.random.RandomState(3)
    inputs = _inputs(rng, [40, 40, 40])
    U = 6
    dummy = [[0] * (U - 1) for _ in inputs]
    with torch.no_grad():
        out = m((inputs, dummy))
    T = out.shape[1]
    want, wscores = decode_static_batch(out, [T] * 3, [U] * 3, 4, m.blank)
    assert m.infer((inputs, dummy), beam_size=4) == want
    got, gscores = m.recognize(inputs, beam_size=4, max_symbols_per_frame=U - 1, max_len=U - 1,
                               return_scores=True)
    assert got == want
    # P runs in fp32 here and through the bf16 recurrence of ops.gru_stack in `forward`; fy is a
    # bf16-operand GEMM of P in both, so rows differ by about a bf16 ulp of the logits
    for a, b in zip(gscores, wscores):
        assert abs(a - b) <= 2e-2 * abs(b) + 1e-2, (a, b)


def test_batch_independence_in_exact_lengths_mode(cuda_lib):
    m = _model(24, False, 1, 16, 11, True, seed=11)
    rng = np.random.RandomState(4)
    inputs = _inputs(rng, [40, 17, 33, 9])
    together = m.recognize(inputs, beam_size=4, max_symbols_per_frame=2)
    for b, x in enumerate(inputs):
        assert m.recognize([x], beam_size=4, max_symbols_per_frame=2) == [together[b]], b


def test_edges(cuda_lib):
    m = _model(24, True, 1, 16, 11, False, seed=5)
    rng = np.random.RandomState(5)
    inputs = _inputs(rng, [40, 35])
    for n in (0, 1, 3):                              # max_len binds
        labels = m.recognize(inputs, beam_size=4, max_symbols_per_frame=3, max_len=n)
        assert all(len(l) <= n for l in labels)
    labels, scores = m.recognize(inputs, beam_size=12, max_symbols_per_frame=2,
                                 return_scores=True)  # beam >= V1 - 1
    assert all(math.isfinite(s) for s in scores)
    big = _inputs(rng, [40] * 40)                    # B*K = 320 prediction rows
    labels = m.recognize(big, beam_size=8, max_symbols_per_frame=2)
    alone = m.recognize(big[:1], beam_size=8, max_symbols_per_frame=2)
    assert labels[0] == alone[0]


def test_large_vocabulary_never_holds_the_lattice(cuda_lib):
    from speech_b200.models.transducer_model import PredictionRows
    from speech_b200.transducer_decoders import decode_static_fits, search_batch
    V1 = 20001
    m = _model(24, True, 1, 16, V1, False, seed=9)
    assert not decode_static_fits(4, V1)
    rng = np.random.RandomState(9)
    inputs = _inputs(rng, [40, 30])
    m.recognize(inputs, beam_size=4, max_symbols_per_frame=2)      # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    labels, scores = m.recognize(inputs, beam_size=4, max_symbols_per_frame=2, return_scores=True)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    rows = PredictionRows(m, inputs)
    lattice = rows.B * rows.T * 4 * V1 * 4            # (B, T', K, V+1) f32, never materialised
    assert growth < lattice // 2, (growth, lattice)
    for b in range(2):
        want, wscore, gap = ref.search(ref.LabelFreeRows(m, rows.fxT[:, b]), rows.tlens[b], 4,
                                       m.blank, 2, 10 ** 9)
        assert abs(scores[b] - wscore) <= 1e-5 * abs(wscore) + 1e-6
        if gap > 1e-4:
            assert labels[b] == want
