"""Host checks (no GPU) of n-gram LM shallow fusion in the label-free transducer beam search
(transducer_decoders.search_batch(lm=...), Transducer.recognize(lm=...)):

- the restated search (tests/rnnt_lm_ref.py) is oracle/rnnt_search_ref.search at zero weights,
  and with a beam that holds every hypothesis it is the fused enumeration (orders 1 / 3 / 5,
  negative insertion bonus included);
- the host mirror of the shortlist route over fused float64 values equals the full restatement,
  and flags the tie lattice, whose 2-entry lists cannot prove the full search's choice;
- every ValueError of recognize, and the C ABI's argument checks and bound symbols.
"""
import ctypes
import math

import numpy as np
import pytest

import rnnt_lm_ref as lref
from ngram_ref import ArpaLM
from oracle import rnnt_search_ref as ref
from speech_b200 import _lib
from speech_b200.lm import NGramLM
from test_rnnt_shortlist_host import tie_lattice


def _lm(tmp_path, rng, V1, order, n=120, name="lm"):
    """a trained LM over labels 0..V1-2 (blank V1-1) and its ARPA reader"""
    seqs = [rng.randint(0, V1 - 1, rng.randint(1, 12)).tolist() for _ in range(n)]
    lm = NGramLM.train(seqs, order, V1, V1 - 1)
    p = str(tmp_path / ("%s%d.arpa" % (name, order)))
    lm.to_arpa(p)
    return lm, ArpaLM(p, [str(c) for c in range(V1 - 1)], V1 - 1)


def _label_rows(V, seed, scale=2.0):
    """rows that depend on the whole hypothesis (a deterministic random log-softmax per (t, h))"""
    cache = {}

    def row(t, hyp):
        key = (t, hyp)
        if key not in cache:
            rng = np.random.RandomState(abs(hash((seed,) + key)) % (2 ** 31))
            x = rng.randn(V) * scale
            cache[key] = (x - np.log(np.exp(x).sum())).astype(np.float32)
        return cache[key]
    return row


@pytest.mark.parametrize("order", [1, 3])
@pytest.mark.parametrize("T,V,K,S,seed", [(6, 5, 1, 2, 0), (8, 7, 4, 3, 1), (5, 9, 8, 2, 2)])
def test_zero_weights_are_the_plain_search(tmp_path, order, T, V, K, S, seed):
    _, arpa = _lm(tmp_path, np.random.RandomState(seed), V, order)
    row = _label_rows(V, seed)
    want = ref.search(row, T, K, V - 1, S, 10 ** 9)
    got = lref.search(row, T, K, V - 1, S, 10 ** 9, arpa, 0.0, 0.0)
    assert got == want


@pytest.mark.parametrize("order,a,b", [(1, 0.7, 0.5), (3, 0.5, 1.0), (5, 1.5, -0.8),
                                       (3, 2.0, -2.0)])
@pytest.mark.parametrize("T,V,max_len,seed", [(2, 3, 2, 0), (3, 3, 3, 1), (3, 4, 2, 2)])
def test_exhaustive_beam_is_the_fused_argmax(tmp_path, order, a, b, T, V, max_len, seed):
    _, arpa = _lm(tmp_path, np.random.RandomState(seed + 10), V, order)
    row = _label_rows(V, seed)
    blank = V - 1
    want, ws = lref.best_by_enumeration(row, T, V, blank, max_len, arpa, a, b)
    n_hyps = sum((V - 1) ** n for n in range(max_len + 1))
    got, gs, _ = lref.search(row, T, n_hyps, blank, max_len, max_len, arpa, a, b)
    assert got == want
    assert abs(gs - ws) < 1e-9 * max(1.0, abs(ws))


def _shortlist_route(row, T, K, blank, S, max_len, arpa, a, b):
    """the route as search_batch runs it: kp = K lists, flagged searches again from 64"""
    got = lref.shortlist_search(row, T, K, blank, S, max_len, arpa, a, b, K)
    if got[2]:
        got = lref.shortlist_search(row, T, K, blank, S, max_len, arpa, a, b, 64)
        assert got[2] == 0
    return got


@pytest.mark.parametrize("order,a,b", [(1, 0.5, 1.0), (3, 0.5, 1.0), (5, 1.0, -0.5),
                                       (3, 0.0, 0.0)])
@pytest.mark.parametrize("T,V,K,S,seed", [(6, 12, 2, 2, 0), (7, 20, 4, 3, 1), (5, 40, 8, 2, 2)])
def test_shortlist_mirror_equals_the_full_restatement(tmp_path, order, a, b, T, V, K, S, seed):
    _, arpa = _lm(tmp_path, np.random.RandomState(seed + 20), V, order)
    row = _label_rows(V, seed, scale=1.0)
    want = lref.search(row, T, K, V - 1, S, 10 ** 9, arpa, a, b)
    got = _shortlist_route(row, T, K, V - 1, S, 10 ** 9, arpa, a, b)
    assert (got[0], got[1]) == (want[0], want[1])
    for kp in (K, K + 3, 64):                            # any list length that is not flagged
        lab, sc, fl = lref.shortlist_search(row, T, K, V - 1, S, 10 ** 9, arpa, a, b, kp)
        if not fl:
            assert (lab, sc) == (want[0], want[1]), kp


def test_shortlist_mirror_flags_the_tie_lattice(tmp_path):
    """fused values lp + 0.5 at a hypothesis score of -2^40: labels 0, 5 and 7 tie on score, the
    full search takes class 0 first, and 2-entry lists ([5, 7], beta = class 0's value) cannot
    show it"""
    lat, blank = tie_lattice(V=40)
    _, arpa = _lm(tmp_path, np.random.RandomState(0), 40, 2)
    row = ref.static_rows(lat)
    want = lref.search(row, 2, 2, blank, 1, 1, arpa, 0.0, 0.5)
    assert want[0] == [0]
    got, _, flags = lref.shortlist_search(row, 2, 2, blank, 1, 1, arpa, 0.0, 0.5, 2)
    assert flags > 0 and got == [5]
    got = _shortlist_route(row, 2, 2, blank, 1, 1, arpa, 0.0, 0.5)
    assert (got[0], got[1]) == (want[0], want[1])


# ---------------------------------------------------------------------------------------------
# Transducer.recognize argument checks (before any launch: the model here is on the CPU)
# ---------------------------------------------------------------------------------------------
def test_recognize_rejects_bad_fusion_arguments():
    from speech_b200.models import Transducer
    cfg = {"dropout": 0.0, "encoder": {"conv": [[4, 5, 5, 2]],
                                       "rnn": {"dim": 24, "bidirectional": True, "layers": 1}},
           "decoder": {"embedding_dim": 16, "layers": 1}}
    m = Transducer(40, 10, cfg)                          # V + 1 = 11 classes, blank 10
    lm = NGramLM.train([[0, 1, 2]], 2, 11, 10)
    bad = [
        dict(lm=None, lm_weight=0.5),                    # weights without an LM
        dict(lm=None, insertion_bonus=1.0),
        dict(lm=lm, lm_weight=-0.1),
        dict(lm=lm, lm_weight=math.inf),
        dict(lm=lm, lm_weight=math.nan),
        dict(lm=lm, lm_weight=0.5, insertion_bonus=math.inf),
        dict(lm=lm, lm_weight=0.5, insertion_bonus=math.nan),
        dict(lm=NGramLM.train([[0, 1]], 2, 12, 11)),     # class count
        dict(lm=NGramLM.train([[1, 2]], 2, 11, 0)),      # blank
        dict(lm=NGramLM.train([[0, 1, 9]], 2, 11, 10, end=9)),   # an end class
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            m.recognize([np.zeros((40, 40), np.float32)], **kw)
    with pytest.raises(ValueError, match="the Transducer search has no end class"):
        m.recognize([np.zeros((40, 40), np.float32)], lm=bad[-1]["lm"])


def test_ctc_check_keeps_its_message():
    from speech_b200.models.ctc_decoder import check_lm
    with pytest.raises(ValueError) as e:
        check_lm(NGramLM.train([[0, 1, 2]], 2, 4, 3, end=2), 0.5, 0.0, 4, 3)
    assert str(e.value) == "the LM reads class 2 as </s>; the CTC search has no end class"


# ---------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------
def test_rnnt_lm_symbols_are_bound():
    lib = _lib.load()
    for name in ("sb_rnnt_search_lm_rows", "sb_rnnt_search_round_lm"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


def _lm_struct(**kw):
    f = dict(keys=8, vals=8, logp=8, bow=8, tok=8, cap=64, order=3, num_classes=29, bos=29,
             blank=28, lm_upper=0.0, lm_abs=10.0)
    f.update(kw)
    return _lib.SbNgramLm(*[f[name] for name, _ in _lib.SbNgramLm._fields_])


B, T, S, K, V, BLANK = 2, 5, 2, 4, 29, 28
WS = 1 << 40                     # never dereferenced: every call below fails its checks first


def _rows(fused=8, sl=(None, None, None), kp=0, t=0, level=0, V_=V, blank=BLANK, K_=K):
    return (8, fused, *sl, kp, 8, t, level, B, T, S, V_, K_, blank)


@pytest.mark.parametrize("kw,weights,args,status", [
    ({}, (-0.5, 0.0), {}, 1),
    ({}, (math.nan, 0.0), {}, 1),
    ({}, (math.inf, 0.0), {}, 1),
    ({}, (0.5, math.inf), {}, 1),
    ({}, (0.5, math.nan), {}, 1),
    ({"num_classes": 28}, (0.5, 0.0), {}, 1),
    ({"lm_upper": math.inf}, (0.5, 0.0), {}, 1),
    ({"lm_abs": math.nan}, (0.5, 0.0), {}, 1),
    ({"keys": None}, (0.5, 0.0), {}, 1),
    ({"vals": None}, (0.5, 0.0), {}, 1),
    ({"logp": None}, (0.5, 0.0), {}, 1),
    ({"bow": None}, (0.5, 0.0), {}, 1),
    ({"tok": None}, (0.5, 0.0), {}, 1),
    ({"cap": 48}, (0.5, 0.0), {}, 1),
    ({"order": 0}, (0.5, 0.0), {}, 1),
    ({"blank": 3}, (0.5, 0.0), {}, 1),
    ({}, (0.5, 0.0), {"blank": V}, 1),                     # what sb_rnnt_search_round rejects
    ({}, (0.5, 0.0), {"t": T}, 1),
    ({}, (0.5, 0.0), {"level": S + 1}, 1),
    ({}, (0.5, 0.0), {"fused": None, "sl": (8, 8, None), "kp": K}, 1),
    ({}, (0.5, 0.0), {"fused": None, "sl": (8, 8, 8), "kp": K - 1}, 1),
    ({"order": 11}, (0.5, 0.0), {}, 3),
    ({}, (0.5, 0.0), {"fused": None, "sl": (8, 8, 8), "kp": 65}, 3),
])
def test_lm_rows_rejects_bad_arguments(kw, weights, args, status):
    lib = _lib.load()
    st = _lm_struct(**kw)
    assert lib.sb_rnnt_search_lm_rows(*_rows(**args), ctypes.byref(st), *weights, 256, WS,
                                      None) == status


def test_lm_rows_rejects_a_missing_lm_or_rows():
    lib = _lib.load()
    st = _lm_struct()
    assert lib.sb_rnnt_search_lm_rows(*_rows(), None, 0.5, 0.0, 256, WS, None) == 1
    args = list(_rows())
    args[0] = None                                         # no acoustic rows
    assert lib.sb_rnnt_search_lm_rows(*args, ctypes.byref(st), 0.5, 0.0, 256, WS, None) == 1
    args = list(_rows())
    args[6] = None                                         # no tlens
    assert lib.sb_rnnt_search_lm_rows(*args, ctypes.byref(st), 0.5, 0.0, 256, WS, None) == 1
    assert lib.sb_rnnt_search_lm_rows(*_rows(), ctypes.byref(st), 0.5, 0.0, None, WS, None) == 1
    assert lib.sb_rnnt_search_lm_rows(*_rows(), ctypes.byref(st), 0.5, 0.0, 256, 1, None) == 4
    assert lib.sb_rnnt_search_lm_rows(*_rows(K_=33), ctypes.byref(st), 0.5, 0.0, 256, WS,
                                      None) == 3


def _round(lp=8, sl=(None, None, None), kp=0, t=0, level=0, max_len=5, V_=V, blank=BLANK, K_=K):
    return (lp, *sl, kp, 8, t, level, max_len, 8, 8, 8, B, T, S, V_, K_, blank, 256, WS, None)


@pytest.mark.parametrize("args,status", [
    ({"blank": V}, 1),
    ({"blank": -1}, 1),
    ({"t": -1}, 1),
    ({"level": S + 1}, 1),
    ({"max_len": -1}, 1),
    ({"lp": None, "sl": (8, None, 8), "kp": K}, 1),
    ({"lp": None, "sl": (8, 8, 8), "kp": K - 1}, 1),
    ({"lp": None, "sl": (8, 8, 8), "kp": 65}, 3),
    ({"V_": 7000, "K_": 4}, 3),                            # K * V * 8 past 200 KB of candidates
    ({"K_": 33}, 3),
])
def test_round_lm_rejects_what_the_round_rejects(args, status):
    lib = _lib.load()
    assert lib.sb_rnnt_search_round_lm(*_round(**args)) == status
    assert lib.sb_rnnt_search_round(*_round(**args)) == status
