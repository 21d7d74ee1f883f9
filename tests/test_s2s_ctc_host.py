"""Host checks (no GPU) of joint CTC/attention training and decoding of the attention model:

- the float64 CTC prefix scorer of tests/s2s_ctc_ref.py against brute-force enumeration of CTC
  paths, END against the CTC oracle, and the decomposition psi(h) = lse_c psi(h + c);
- every ValueError of the config, of recognize and of the joint loss;
- the model's structure with and without the head, and head-less pickles;
- the C ABI: bound symbols, and every entry point's argument checks before any launch.
"""
import ctypes
import itertools
import math
import pickle

import numpy as np
import pytest
import torch

from s2s_ctc_ref import brute_force, lse, prefix_scores, vectors_of
from speech_b200 import _lib


def _y(rng, T, C):
    """float64 log-probabilities: the brute force and the decomposition assume rows normalised
    to float64 rounding"""
    x = rng.randn(T, C) * 1.5
    return x - np.log(np.exp(x).sum(1, keepdims=True))


def _hyps(L, n):
    return [h for k in range(n + 1) for h in itertools.product(range(L), repeat=k)]


@pytest.mark.parametrize("T", [1, 2, 4, 6])
def test_prefix_scorer_equals_brute_force(T):
    rng = np.random.RandomState(T)
    C = 4                                      # labels 0..2 (2 also stands for END) and blank 3
    y = _y(rng, T, C)
    for h in _hyps(3, 3):
        gn, gb = vectors_of(y, T, h)
        last = h[-1] if h else None
        for c in range(3):
            got = prefix_scores(y, gn, gb, last, [c], end=-1)[0]
            ref = brute_force(y, h + (c,))
            assert (got == ref == -math.inf) or abs(got - ref) <= 1e-12 * max(1.0, abs(ref)), \
                (h, c, got, ref)
        got = prefix_scores(y, gn, gb, last, [C - 1], end=C - 1)[0]
        ref = brute_force(y, h, end_only=True)
        assert (got == ref == -math.inf) or abs(got - ref) <= 1e-12 * max(1.0, abs(ref)), (h, got)


def test_end_equals_the_ctc_oracle():
    from oracle import ctc_ref
    rng = np.random.RandomState(3)
    T, C = 12, 6
    y = _y(rng, T, C)
    for h in [(), (0,), (1, 1), (2, 0, 4, 4, 1)]:
        gn, gb = vectors_of(y, T, h)
        psi = prefix_scores(y, gn, gb, h[-1] if h else None, [C - 1], end=C - 1)[0]
        loss = ctc_ref.ctc_single(y.astype(np.float64), list(h), C - 1)
        loss = loss[0] if isinstance(loss, tuple) else loss
        assert abs(psi + float(loss)) <= 1e-9 * max(1.0, abs(psi)), (h, psi, loss)


def test_prefix_scores_decompose_the_prefix_probability():
    """psi(h) = lse over c of psi(h + c), c over every label and END"""
    rng = np.random.RandomState(4)
    T, C = 9, 5
    y = _y(rng, T, C)
    for h in [(0,), (1, 1), (3, 0, 2), (2, 2, 2)]:
        gn, gb = vectors_of(y, T, h[:-1])
        psi_h = prefix_scores(y, gn, gb, h[-2] if len(h) > 1 else None, [h[-1]], end=C - 1)[0]
        gn, gb = vectors_of(y, T, h)
        parts = prefix_scores(y, gn, gb, h[-1], list(range(C)), end=C - 1)
        tot = -math.inf
        for v in parts:
            tot = float(lse(tot, v))
        assert abs(tot - psi_h) <= 1e-12 * max(1.0, abs(psi_h)), (h, tot, psi_h)


# ---------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------
def _cfg(**dec):
    d = {"embedding_dim": 16, "layers": 1}
    d.update(dec)
    return {"dropout": 0.0, "encoder": {"conv": [[4, 5, 8, 2]],
                                        "rnn": {"dim": 16, "bidirectional": True, "layers": 1}},
            "decoder": d}


def _build(seed=0, **dec):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(seed)
    return Seq2Seq(40, 9, _cfg(**dec))


@pytest.mark.parametrize("w", [-0.1, 1.0, 1.5, math.nan, math.inf, "0.3", True])
def test_config_rejects_a_bad_ctc_weight(w):
    with pytest.raises(ValueError):
        _build(ctc_weight=w)


def test_without_a_head_the_model_is_unchanged():
    base = _build(0).state_dict()
    for dec in ({"ctc_weight": 0}, {"ctc_weight": 0.0}):
        m = _build(0, **dec)
        sd = m.state_dict()
        assert list(sd) == list(base) and m.ctc_weight == 0.0 and not hasattr(m, "ctc_fc")
        assert all(torch.equal(sd[k], base[k]) for k in base)


def test_a_head_adds_exactly_its_projection():
    base = _build(0).state_dict()
    m = _build(0, ctc_weight=0.3)
    sd = m.state_dict()
    assert m.ctc_weight == 0.3
    assert set(sd) - set(base) == {"ctc_fc.fc.weight", "ctc_fc.fc.bias"}
    assert list(sd)[:len(base)] == list(base)
    assert all(torch.equal(sd[k], base[k]) for k in base)
    assert tuple(sd["ctc_fc.fc.weight"].shape) == (8, 16)


def test_a_headless_pickle_loads_with_no_ctc_weight():
    m = _build(0)
    assert "ctc_weight" not in m.__dict__        # as pickled before the head existed
    back = pickle.loads(pickle.dumps(m))
    assert back.ctc_weight == 0.0 and "ctc_weight" not in back.__dict__


def _utterances(n=2):
    rng = np.random.RandomState(0)
    return [rng.randn(60, 40).astype(np.float32) for _ in range(n)]


@pytest.mark.parametrize("kw", [dict(ctc_weight=-0.1), dict(ctc_weight=1.0),
                                dict(ctc_weight=math.nan), dict(ctc_weight=0.5, ctc_prebeam=0),
                                dict(ctc_weight=0.5, ctc_prebeam=9),
                                dict(ctc_weight=0.5, ctc_prebeam=2.5),
                                dict(ctc_weight=0.5, start_tok=0),
                                dict(ctc_weight=0.5, end_tok=0)])
def test_recognize_rejects_bad_joint_arguments(kw):
    """on a CPU model: the ValueError comes before anything touches a device"""
    m = _build(0, ctc_weight=0.3)
    with pytest.raises(ValueError):
        m.recognize(_utterances(), beam_size=4, max_len=5, **kw)


def test_recognize_needs_a_head_for_joint_decoding():
    with pytest.raises(ValueError):
        _build(0).recognize(_utterances(), beam_size=4, max_len=5, ctc_weight=0.5)


def test_the_default_prebeam():
    V = 9
    m = _build(0, ctc_weight=0.3)
    assert m._check_ctc(0.5, None, 4, V, V - 1, V - 2) == 6
    assert m._check_ctc(0.5, None, 10, V, V - 1, V - 2) == 8       # min(C, 3K // 2)
    assert m._check_ctc(0.5, None, 1, V, V - 1, V - 2) == 1
    assert m._check_ctc(0.5, 8, 4, V, V - 1, V - 2) == 8
    assert _build(0)._check_ctc(0.0, None, 4, V, 0, 1) == 6        # no joint decoding


@pytest.mark.parametrize("seq", [[0, 1, 7], [8, 0, 1], [8, 7, 7], [8, 0, 8, 7], [8], [8, 9, 7]])
def test_joint_loss_rejects_malformed_transcripts(seq):
    """on a CPU model: the ValueError comes before anything touches a device"""
    m = _build(0, ctc_weight=0.3)
    with pytest.raises(ValueError):
        m.loss((_utterances(), [[8, 0, 7], seq]))
    flat, lens = m._ctc_targets([[8, 0, 1, 7], [8, 7]])
    assert flat.tolist() == [0, 1] and lens.tolist() == [2, 0]


# ---------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------
NAMES = ("sb_s2s_ctc_state_size", "sb_s2s_ctc_init", "sb_s2s_ctc_candidates",
         "sb_s2s_ctc_select_batch")


def test_s2s_ctc_symbols_are_bound():
    lib = _lib.load()
    for name in NAMES:
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


def _lm_struct(**kw):
    f = dict(keys=8, vals=8, logp=8, bow=8, tok=8, cap=64, order=3, num_classes=31, bos=31,
             blank=30, lm_upper=0.0, lm_abs=10.0)
    f.update(kw)
    return _lib.SbNgramLm(*[f[name] for name, _ in _lib.SbNgramLm._fields_])


GOOD = dict(K=4, C=30, M=6, T=50, start=30, end=29, w=0.3, B=2, nbytes=1 << 30)


def _calls(lib, a, lm=None, lw=0.0, bonus=0.0):
    shape = (a["K"], a["C"], a["M"], a["T"], a["start"], a["end"], a["w"])
    return (
        lib.sb_s2s_ctc_init(8, None, 8, a["nbytes"], *shape, a["B"], None),
        lib.sb_s2s_ctc_candidates(8, 8, None, 8, 8, 100, 8, a["nbytes"], *shape, 0, 8, a["B"], lm,
                                  lw, bonus, None),
        lib.sb_s2s_ctc_select_batch(8, None, 8, a["nbytes"], 8, 8, 8, 8, 8, 8, *shape, 0, 10, 100,
                                    100, 8, a["B"], None))


@pytest.mark.parametrize("kw,status", [
    ({"K": 0}, 1), ({"K": 33}, 3), ({"M": 0}, 1), ({"M": 31}, 1), ({"C": 200, "M": 129,
                                                                      "start": 200, "end": 199}, 3),
    ({"w": 0.0}, 1), ({"w": 1.0}, 1), ({"w": math.nan}, 1), ({"w": -0.5}, 1), ({"T": 0}, 1),
    ({"end": 28}, 1), ({"start": 31}, 1), ({"C": 1, "M": 1, "start": 1, "end": 0}, 1),
    ({"B": 0}, 1), ({"nbytes": 64}, 4),
])
def test_s2s_ctc_entry_points_reject_bad_arguments(kw, status):
    """every check fails before any launch, so fake device pointers are never dereferenced"""
    lib = _lib.load()
    a = dict(GOOD, **kw)
    assert _calls(lib, a) == (status,) * 3


@pytest.mark.parametrize("kw,weights", [({}, (-0.5, 0.0)), ({}, (math.nan, 0.0)),
                                        ({}, (0.5, math.inf)), ({"num_classes": 29}, (0.5, 0.0)),
                                        ({"keys": None}, (0.5, 0.0)), ({"cap": 48}, (0.5, 0.0)),
                                        ({"blank": 3}, (0.5, 0.0))])
def test_s2s_ctc_candidates_checks_the_lm(kw, weights):
    lib = _lib.load()
    st = _lm_struct(**kw)
    assert _calls(lib, GOOD, ctypes.byref(st), *weights)[1] == 1
    assert _calls(lib, GOOD, None, 0.5, 0.0)[1] == 1           # weights without an LM
    st = _lm_struct(order=11)
    assert _calls(lib, GOOD, ctypes.byref(st), 0.5, 0.0)[1] == 3


def test_s2s_ctc_state_size():
    lib = _lib.load()
    n = _lib.workspace_size(lib.sb_s2s_ctc_state_size, 4, 6, 50, 2)
    R = 8
    assert n >= 8 * (R + 4 * R * 50 + 3 * R * 6) + 4 * R * 6
    n = ctypes.c_size_t(0)
    assert lib.sb_s2s_ctc_state_size(0, 6, 50, 2, ctypes.byref(n)) == 1
