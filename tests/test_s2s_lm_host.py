"""Host checks (no GPU) of the n-gram LM with an end class, behind the LM-fused attention beam
search (Seq2Seq.recognize(lm=...)):

- NGramLM with `end`: a Preprocessor-style symbol map, the ARPA round trip, Kneser-Ney training
  on encode() outputs, the stored </s> predictions, pickles from before `end` existed;
- the device lookup, mirrored in Python over the packed tables (tests/s2s_lm_ref.py), against the
  ARPA backoff lookup of tests/ngram_ref.py, </s> predictions included;
- every new ValueError, the CTC decoder's refusal of an LM with an end class, and the C ABI's
  argument checks and bound symbols.
"""
import ctypes
import itertools
import math
import pickle

import numpy as np
import pytest

from ngram_ref import KneserNey
from s2s_lm_ref import EndArpaLM, device_lookup
from speech_b200 import _lib
from speech_b200.lm import NGramLM


def _int_to_char(V):
    """the reference Preprocessor's layout: V - 2 characters, then </s> (END) and <s> (START)"""
    return dict(enumerate([chr(ord("a") + c) for c in range(V - 2)] + ["</s>", "<s>"]))


def _encoded(rng, n, V, max_len=10):
    """Preprocessor.encode outputs: START, characters, END"""
    return [[V - 1] + rng.randint(0, V - 2, rng.randint(0, max_len)).tolist() + [V - 2]
            for _ in range(n)]


def _contexts(V, L):
    return [pre for n in range(L + 1) for pre in itertools.product(range(V), repeat=n)]


def _random_arpa(path, rng, words, order):
    """random values; n-grams predicting </s> at every order, some contexts with no n-gram"""
    sec = {1: {(w,): None for w in words + ["</s>", "<s>"]}}
    for n in range(2, order + 1):
        sec[n] = {}
        for _ in range(6 * len(words)):
            g = tuple(rng.choice(words + ["</s>"], n).tolist())
            if rng.rand() < 0.5:
                g = ("<s>",) + g[1:]
            if "</s>" not in g[:-1]:
                sec[n][g] = None
    lines = ["\\data\\"] + ["ngram %d=%d" % (n, len(sec[n])) for n in sec]
    for n in sec:
        lines += ["", "\\%d-grams:" % n]
        for g in sec[n]:
            line = "%r\t%s" % (-99.0 if g == ("<s>",) else -rng.rand() * 3, " ".join(g))
            if n < order and rng.rand() < 0.7:
                line += "\t%r" % (rng.randn() * 0.8)
            lines.append(line)
    lines += ["", "\\end\\", ""]
    open(path, "w").write("\n".join(lines))


# ---------------------------------------------------------------------------------------------
# NGramLM with an end class
# ---------------------------------------------------------------------------------------------
def test_from_arpa_takes_the_preprocessor_symbol_map(tmp_path):
    V = 7
    p = str(tmp_path / "lm.arpa")
    _random_arpa(p, np.random.RandomState(0), [chr(ord("a") + c) for c in range(V - 2)], 3)
    lm = NGramLM.from_arpa(p, _int_to_char(V), blank=V - 1, end=V - 2)
    assert (lm.num_classes, lm.blank, lm.end, lm.order) == (V, V - 1, V - 2, 3)
    t = lm.host_tables()
    assert t["tok"][V - 2] == V + 1 and t["tok"][V - 1] == -1          # </s>, and START none
    assert list(t["tok"][:V - 2]) == list(range(V - 2))
    # without an end class the reserved symbols are refused, as before
    with pytest.raises(ValueError):
        NGramLM.from_arpa(p, _int_to_char(V), blank=V - 1)


@pytest.mark.parametrize("order", [1, 3, 5])
def test_arpa_round_trip_with_an_end_class_is_exact(tmp_path, order):
    V = 8
    lm = NGramLM.train(_encoded(np.random.RandomState(order), 40, V), order, V, V - 1, end=V - 2)
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p, _int_to_char(V))
    back = NGramLM.from_arpa(p, _int_to_char(V), blank=V - 1, end=V - 2)
    assert back._ngrams == lm._ngrams and back.end == V - 2
    for k in ("keys", "vals", "logp", "bow", "tok"):
        assert np.array_equal(back.host_tables()[k], lm.host_tables()[k])
    for k in ("cap", "order", "bos", "lm_upper", "lm_abs"):
        assert back.host_tables()[k] == lm.host_tables()[k]


@pytest.mark.parametrize("order", [1, 2, 3, 4])
def test_train_on_encoded_sequences_is_kneser_ney(tmp_path, order):
    """encode() outputs go straight in; </s> is the end class; the model is normalised over the
    characters and </s>, and equals KN from the counts (classes 0..V-3 and E = </s>)"""
    V = 5
    rng = np.random.RandomState(20 + order)
    enc = _encoded(rng, 30, V, max_len=8)
    lm = NGramLM.train(enc, order, V, V - 1, end=V - 2)
    # the same model from the bare character sequences, one class fewer (V - 2 is not seen)
    kn = KneserNey([s[1:-1] for s in enc], order, V - 1, V - 2)
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p, _int_to_char(V))
    ref = EndArpaLM(p, [_int_to_char(V)[c] for c in range(V)], V - 1, V - 2)
    for pre in _contexts(V - 2, min(order, 3)):
        h = ref.context(pre)
        hk = tuple("B" if w == "<s>" else ord(w) - ord("a") for w in h)
        total = 0.0
        for c in range(V - 1):                                   # the characters and END
            v = ref.score(pre, c)
            total += math.exp(v)
            direct = math.log(kn.prob(hk, "E" if c == V - 2 else c))
            assert abs(v - direct) <= 1e-12, (pre, c, v, direct)
        assert abs(total - 1.0) <= 1e-9, (pre, total)
    # a sequence without START / END is taken as it is
    assert NGramLM.train([s[1:-1] for s in enc], order, V, V - 1, end=V - 2)._ngrams == lm._ngrams


@pytest.mark.parametrize("order", [1, 2, 3, 5])
def test_device_lookup_of_end_equals_arpa_backoff(tmp_path, order):
    V = 6
    p = str(tmp_path / "lm.arpa")
    _random_arpa(p, np.random.RandomState(30 + order), [chr(ord("a") + c) for c in range(V - 2)],
                 order)
    lm = NGramLM.from_arpa(p, _int_to_char(V), blank=V - 1, end=V - 2)
    ref = EndArpaLM(p, [_int_to_char(V)[c] for c in range(V)], V - 1, V - 2)
    t = lm.host_tables()
    upper = -math.inf
    for pre in _contexts(V - 2, min(order + 1, 4)):
        for c in range(V - 1):                                   # the characters and END
            v = device_lookup(t, pre, c)
            assert v == ref.score(pre, c), (pre, c)
            upper = max(upper, v)
            assert abs(v) <= t["lm_abs"]
    assert upper <= t["lm_upper"]


def test_tables_without_an_end_class_hold_no_end_prediction(tmp_path):
    V = 6
    p = str(tmp_path / "lm.arpa")
    words = [chr(ord("a") + c) for c in range(V)]
    _random_arpa(p, np.random.RandomState(7), words, 3)
    plain = NGramLM.from_arpa(p, words)                          # CTC layout: blank = V
    t = plain.host_tables()
    eos = plain.num_classes + 1
    tokens = [(int(k) >> 1 & 0x7fffffff) - 1 for k, kind in
              ((k, int(k) & 1) for k in t["keys"] if int(k)) if kind == 1]
    assert tokens and eos not in tokens
    with_end = NGramLM.from_arpa(p, words + ["</s>", "<s>"], blank=V + 1, end=V)
    tokens_end = [(int(k) >> 1 & 0x7fffffff) - 1 for k in with_end.host_tables()["keys"]
                  if int(k) and int(k) & 1]
    assert with_end.num_classes + 1 in tokens_end


def test_pickle_from_before_the_end_class_loads_with_no_end():
    lm = NGramLM.train([[0, 1, 2]], 2, 4, 3)
    state = lm.__getstate__()
    del state["_end"]                      # as pickled before LMs had an end class
    old = NGramLM.__new__(NGramLM)
    old.__setstate__(state)
    assert old.end is None and np.array_equal(old.host_tables()["keys"], lm.host_tables()["keys"])
    back = pickle.loads(pickle.dumps(NGramLM.train([[3, 0, 1, 2]], 2, 4, 3, end=2)))
    assert back.end == 2


def test_end_class_errors(tmp_path):
    V = 6
    for end in (V - 1, V, -1):                   # the blank, and out of range
        with pytest.raises(ValueError):
            NGramLM.train([[0, 1]], 2, V, V - 1, end=end)
    for seq in ([V - 1, 0, V - 2, 1, V - 2], [0, V - 1, 1], [V - 1, V - 1, 0], [0, V - 2, V - 2]):
        with pytest.raises(ValueError):                          # START / END mid-sequence
            NGramLM.train([seq], 2, V, V - 1, end=V - 2)
    p = str(tmp_path / "lm.arpa")
    open(p, "w").write("\\data\\\nngram 1=3\n\n\\1-grams:\n-1.0\ta\n-1.0\tb\n-99\t<s>\n\n\\end\\\n")
    syms = {0: "a", 1: "b", 2: "</s>", 3: "<s>"}
    with pytest.raises(ValueError):                              # no </s> unigram
        NGramLM.from_arpa(p, syms, blank=3, end=2)
    for end in (3, 4):
        with pytest.raises(ValueError):
            NGramLM.from_arpa(p, syms, blank=3, end=end)


def test_ctc_decoder_refuses_an_lm_with_an_end_class():
    from speech_b200.models.ctc_decoder import check_lm
    plain = NGramLM.train([[0, 1]], 2, 4, 3)
    check_lm(plain, 0.5, 0.0, 4, 3)
    with pytest.raises(ValueError):
        check_lm(NGramLM.train([[0, 1]], 2, 4, 3, end=2), 0.5, 0.0, 4, 3)


def test_recognize_rejects_bad_fusion_arguments():
    """Seq2Seq._check_lm, which recognize runs before any launch"""
    from speech_b200.models import Seq2Seq
    V = 6
    lm = NGramLM.train([[V - 1, 0, 1, V - 2]], 2, V, V - 1, end=V - 2)
    Seq2Seq._check_lm(None, 0.0, 0.0, V, V - 1, V - 2)
    Seq2Seq._check_lm(lm, 0.5, -1.0, V, V - 1, V - 2)
    bad = [(None, 0.5, 0.0, V, V - 1, V - 2), (None, 0.0, 1.0, V, V - 1, V - 2),
           (lm, -0.1, 0.0, V, V - 1, V - 2), (lm, math.inf, 0.0, V, V - 1, V - 2),
           (lm, math.nan, 0.0, V, V - 1, V - 2), (lm, 0.5, math.inf, V, V - 1, V - 2),
           (lm, 0.5, 0.0, V + 1, V, V - 2),                        # class count
           (lm, 0.5, 0.0, V, V - 2, V - 2),                        # blank is not the start token
           (lm, 0.5, 0.0, V, V - 1, 0),                            # end is not the end token
           (NGramLM.train([[0, 1]], 2, V, V - 1), 0.5, 0.0, V, V - 1, V - 2)]   # no end class
    for args in bad:
        with pytest.raises(ValueError):
            Seq2Seq._check_lm(*args)
    lm_mid = NGramLM.train([[0, 1]], 2, V, 2, end=V - 2)
    with pytest.raises(ValueError):                              # START a predicted class
        Seq2Seq._check_lm(lm_mid, 0.5, 0.0, V, 2, V - 2)


# ---------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------
def test_s2s_lm_symbols_are_bound():
    lib = _lib.load()
    for name in ("sb_s2s_beam_select_lm_batch", "sb_s2s_beam_select_split_lm_batch"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


def _lm_struct(**kw):
    f = dict(keys=8, vals=8, logp=8, bow=8, tok=8, cap=64, order=3, num_classes=31, bos=31,
             blank=30, lm_upper=0.0, lm_abs=10.0)
    f.update(kw)
    return _lib.SbNgramLm(*[f[name] for name, _ in _lib.SbNgramLm._fields_])


@pytest.mark.parametrize("kw,weights,status", [
    ({}, (-0.5, 0.0), 1),
    ({}, (math.nan, 0.0), 1),
    ({}, (math.inf, 0.0), 1),
    ({}, (0.5, math.inf), 1),
    ({}, (0.5, math.nan), 1),
    ({"num_classes": 29}, (0.5, 0.0), 1),
    ({"lm_upper": math.inf}, (0.5, 0.0), 1),
    ({"lm_abs": math.nan}, (0.5, 0.0), 1),
    ({"keys": None}, (0.5, 0.0), 1),
    ({"tok": None}, (0.5, 0.0), 1),
    ({"cap": 48}, (0.5, 0.0), 1),
    ({"blank": 3}, (0.5, 0.0), 1),
    ({"order": 11}, (0.5, 0.0), 3),
])
def test_s2s_lm_entry_points_reject_bad_arguments(kw, weights, status):
    """every check fails before any launch, so fake device pointers are never dereferenced"""
    lib = _lib.load()
    st = _lm_struct(**kw)
    K, C = 4, 30
    common = (8, 8, 8, 8, 8, 8, 8, K, C, 28, 0, 10, 100, 100, 8, 1)
    assert lib.sb_s2s_beam_select_lm_batch(*common, ctypes.byref(st), *weights, None) == status
    assert lib.sb_s2s_beam_select_split_lm_batch(*common, 8, 1 << 30, ctypes.byref(st), *weights,
                                                 None) == status
    assert lib.sb_s2s_beam_select_lm_batch(*common, None, 0.5, 0.0, None) == 1     # no LM
