"""GPU tests of n-gram LM shallow fusion in the label-free transducer beam search
(csrc/rnnt_search.cu sb_rnnt_search_lm_rows / sb_rnnt_search_round_lm,
transducer_decoders.search_batch(lm=...), Transducer.recognize(lm=...)):

- identity: lm_weight = insertion_bonus = 0 gives the LM-less recognize bit for bit, on both
  candidate routes;
- static rows: the device search equals the fused restatement (tests/rnnt_lm_ref.py), and the full
  route, the forced shortlist route (kp = K) and kp = 64 agree bit for bit;
- model: labels equal LabelFreeRows + the fused restatement wherever its smallest gap exceeds 1e-4,
  scores to a relative 1e-5; exact-lengths mode; V+1 = 5001 without the lattice;
- an acoustic tie between two labels goes to the LM's label when lm_weight > 0."""
import numpy as np
import pytest
import torch

import rnnt_lm_ref as lref
from ngram_ref import ArpaLM
from oracle import rnnt_search_ref as ref
from speech_b200.lm import NGramLM

pytestmark = pytest.mark.gpu


class StaticRows:
    """row provider of a (B, T, U1, V1) lattice: the row of a slot is lat[b, t, its length]; fills
    slots.lp and / or slots.sl, whichever the search gives"""

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


def _lattice(rng, B, T, U, V, scale=1.0):
    x = rng.randn(B, T, U, V) * scale
    return torch.from_numpy((x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32))


def _lm(tmp_path, rng, V1, order, n=200, name="lm"):
    """a trained LM over labels 0..V1-2 (blank V1-1) and its ARPA reader"""
    seqs = [rng.randint(0, V1 - 1, rng.randint(1, 20)).tolist() for _ in range(n)]
    lm = NGramLM.train(seqs, order, V1, V1 - 1)
    p = str(tmp_path / ("%s%d_%d.arpa" % (name, order, V1)))
    lm.to_arpa(p)
    return lm, ArpaLM(p, [str(c) for c in range(V1 - 1)], V1 - 1)


def _force_shortlist(monkeypatch):
    from speech_b200 import transducer_decoders
    monkeypatch.setattr(transducer_decoders, "decode_static_fits", lambda K, V: False)


def _model(H, bidir, layers, E, V1, exact, seed=0):
    from speech_b200.models import Transducer
    torch.manual_seed(seed)
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": [[4, 5, 5, 2]], "rnn": {"dim": H, "bidirectional": bidir,
                                                       "layers": 1}},
           "decoder": {"embedding_dim": E, "layers": layers}}
    m = Transducer(40, V1 - 1, cfg).cuda()
    for p in m.parameters():                        # peakier rows than the default init
        p.data.mul_(2.0)
    m.set_eval()
    return m


def _inputs(rng, lens):
    return [rng.randn(n, 40).astype(np.float32) for n in lens]


# ---- identity at zero weights ---------------------------------------------------------------
@pytest.mark.parametrize("V1,beam,force", [(11, 1, False), (11, 4, False), (11, 8, False),
                                           (11, 32, False), (29, 1, False), (29, 4, False),
                                           (29, 8, False), (29, 32, False), (300, 32, True),
                                           (5001, 4, False), (5001, 8, False)])
def test_zero_weights_are_recognize_without_an_lm(cuda_lib, monkeypatch, V1, beam, force):
    from speech_b200 import transducer_decoders as td
    m = _model(24, True, 1, 16, V1, False, seed=V1 + beam)
    rng = np.random.RandomState(beam)
    inputs = _inputs(rng, [40, 31, 36])
    if force:
        _force_shortlist(monkeypatch)
    # full candidate lists up to 200 KB: V+1 = 5001 takes shortlists at beam 8, not at beam 4
    assert td.decode_static_fits(beam, V1) == (V1 * beam * 8 + 16 <= 200 * 1024 and not force)
    lm = NGramLM.train([rng.randint(0, V1 - 1, 8).tolist() for _ in range(50)], 3, V1, V1 - 1)
    want = m.recognize(inputs, beam_size=beam, max_symbols_per_frame=2, return_scores=True)
    got = m.recognize(inputs, beam_size=beam, max_symbols_per_frame=2, return_scores=True, lm=lm)
    assert got == want


# ---- static rows against the restatement ---------------------------------------------------
@pytest.mark.parametrize("V1,K,order,a,b,force", [(29, 4, 3, 0.5, 1.0, False),
                                                  (29, 8, 5, 1.0, -0.5, True),
                                                  (11, 2, 1, 0.8, 0.3, False),
                                                  (1000, 32, 3, 0.5, 1.0, False)])
def test_static_rows_equal_the_fused_restatement(cuda_lib, tmp_path, monkeypatch, V1, K, order, a,
                                                 b, force):
    from speech_b200.transducer_decoders import search_batch
    rng = np.random.RandomState(V1 + K)
    B, T, S = 3, 6, 2
    U1 = T * S + 1
    lat = _lattice(rng, B, T, U1, V1, scale=2.0).cuda()
    lm, arpa = _lm(tmp_path, rng, V1, order)
    if force:
        _force_shortlist(monkeypatch)
    tlens = [T, T - 2, 1]
    labels, scores = search_batch(StaticRows(lat, V1 - 1), tlens, K, V1 - 1, S, None, lm, a, b)
    host = lat.cpu().numpy()
    for i in range(B):
        want, ws, _ = lref.search(ref.static_rows(host[i]), tlens[i], K, V1 - 1, S, T * S, arpa,
                                  a, b)
        assert labels[i] == want, i
        assert abs(scores[i] - ws) <= 1e-9 * abs(ws), (i, scores[i], ws)


def test_forced_routes_agree_bit_for_bit(cuda_lib, tmp_path):
    from speech_b200 import transducer_decoders as td
    rng = np.random.RandomState(5)
    B, T, S, V1, K = 4, 8, 3, 100, 8
    lat = _lattice(rng, B, T, T * S + 1, V1, scale=1.5).cuda()
    lm, _ = _lm(tmp_path, rng, V1, 4)
    prov = StaticRows(lat, V1 - 1)
    tl = [T, T - 1, 3, 0]
    runs = [td._search_once(prov, tl, T, K, S, T * S, T * S, V1 - 1, kp, (lm, 0.7, 0.4))
            for kp in (None, K, 64)]
    full = runs[0][:2]
    for kp, (lab, sc, fl) in zip((K, 64), runs[1:]):
        if not any(fl):
            assert (lab, sc) == full, kp
    assert not any(runs[2][2])
    assert runs[2][:2] == full


# ---- the model against the oracle ----------------------------------------------------------
CASES = [  # H, bidir, layers, E, V+1, beam, exact, order, force
    (24, True, 1, 16, 11, 4, False, 1, False),
    (24, False, 2, 24, 11, 8, True, 3, False),
    (20, True, 1, 12, 29, 4, False, 5, False),
    (20, False, 2, 16, 300, 4, False, 3, True),
]


@pytest.mark.parametrize("H,bidir,layers,E,V1,beam,exact,order,force", CASES)
def test_model_equals_the_fused_oracle(cuda_lib, tmp_path, monkeypatch, H, bidir, layers, E, V1,
                                       beam, exact, order, force):
    from speech_b200.models.transducer_model import PredictionRows
    m = _model(H, bidir, layers, E, V1, exact, seed=H + V1 + beam)
    rng = np.random.RandomState(beam + order)
    inputs = _inputs(rng, [40, 31, 36, 24])
    lm, arpa = _lm(tmp_path, rng, V1, order)
    if force:
        _force_shortlist(monkeypatch)
    S, a, b = 2, 0.5, 1.0
    labels, scores = m.recognize(inputs, beam_size=beam, max_symbols_per_frame=S,
                                 return_scores=True, lm=lm, lm_weight=a, insertion_bonus=b)
    rows = PredictionRows(m, inputs)
    decisive = 0
    for i in range(len(inputs)):
        oracle = ref.LabelFreeRows(m, rows.fxT[:, i])
        want, ws, gap = lref.search(oracle, rows.tlens[i], beam, m.blank, S, 10 ** 9, arpa, a, b)
        assert abs(scores[i] - ws) <= 1e-5 * abs(ws) + 1e-6, (i, scores[i], ws)
        if gap > 1e-4:
            decisive += 1
            assert labels[i] == want, i
    assert decisive >= len(inputs) // 2, decisive


def test_batch_independence_in_exact_lengths_mode(cuda_lib, tmp_path):
    m = _model(24, False, 1, 16, 11, True, seed=11)
    rng = np.random.RandomState(4)
    inputs = _inputs(rng, [40, 17, 33, 9])
    lm, _ = _lm(tmp_path, rng, 11, 3)
    kw = dict(beam_size=4, max_symbols_per_frame=2, return_scores=True, lm=lm, lm_weight=0.6,
              insertion_bonus=0.5)
    together = m.recognize(inputs, **kw)
    for i, x in enumerate(inputs):
        alone = m.recognize([x], **kw)
        assert (alone[0][0], alone[1][0]) == (together[0][i], together[1][i]), i


def test_large_vocabulary_with_an_lm_never_holds_the_lattice(cuda_lib, tmp_path):
    from speech_b200.models.transducer_model import PredictionRows
    V1 = 5001
    m = _model(24, True, 1, 16, V1, False, seed=9)
    rng = np.random.RandomState(9)
    inputs = _inputs(rng, [40, 30])
    lm, arpa = _lm(tmp_path, rng, V1, 3, n=400)
    kw = dict(beam_size=4, max_symbols_per_frame=2, lm=lm, lm_weight=0.5, insertion_bonus=1.0)
    m.recognize(inputs, **kw)                                        # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    labels, scores = m.recognize(inputs, return_scores=True, **kw)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    rows = PredictionRows(m, inputs)
    lattice = rows.B * rows.T * 4 * V1 * 4            # (B, T', K, V+1) f32, never materialised
    assert growth < lattice // 2, (growth, lattice)
    for i in range(2):
        want, ws, gap = lref.search(ref.LabelFreeRows(m, rows.fxT[:, i]), rows.tlens[i], 4,
                                    m.blank, 2, 10 ** 9, arpa, 0.5, 1.0)
        assert abs(scores[i] - ws) <= 1e-5 * abs(ws) + 1e-6
        if gap > 1e-4:
            assert labels[i] == want


def test_an_acoustic_tie_goes_to_the_lms_label(cuda_lib):
    """labels 2 and 5 tie at every frame; the full search takes 2 (the lower class) without the
    LM, and the LM, trained on sequences of 5, turns it to 5"""
    from speech_b200.transducer_decoders import search_batch
    V1, T = 9, 3
    lat = np.full((1, T, T + 1, V1), -8.0, dtype=np.float32)
    lat[..., V1 - 1] = -0.5
    lat[0, :, :, 2] = -1.0
    lat[0, :, :, 5] = -1.0
    lat = torch.from_numpy(lat).cuda()
    lm = NGramLM.train([[5, 5, 5]] * 20 + [[1]], 2, V1, V1 - 1)
    plain, _ = search_batch(StaticRows(lat, V1 - 1), [T], 4, V1 - 1, 1, None)
    zero, _ = search_batch(StaticRows(lat, V1 - 1), [T], 4, V1 - 1, 1, None, lm, 0.0, 0.0)
    fused, _ = search_batch(StaticRows(lat, V1 - 1), [T], 4, V1 - 1, 1, None, lm, 0.3, 0.0)
    assert plain == zero and plain[0] and set(plain[0]) == {2}
    assert fused[0] and set(fused[0]) == {5}
