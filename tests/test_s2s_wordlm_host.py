"""Host checks (no GPU) of the word-LM attention beam search:

- speech_b200.lm.WordLM with an end class: ARPA round trip, training, the end's validation, and
  pickles from before the end class;
- Seq2Seq._check_lm's acceptance of such an LM and each refusal, and the CTC search's refusal;
- the reference's candidate values (tests/s2s_wordlm_ref.py) on hand-computed candidates of every
  row of the table in include/speech_b200.h;
- the refusals of the new C entry points (fake device pointers: every check precedes any launch),
  and their bindings.
"""
import ctypes
import math
import pickle

import pytest

from ctc_wordlm_ref import WordArpa
from s2s_wordlm_ref import WordPart
from speech_b200 import _lib
from speech_b200.lm import WordLM

# the attention model's layout: letters, the space (delimiter), END, START (the blank)
SYMBOLS = list("abcde") + [" ", "</s>", "<s>"]
DELIM, END, START = 5, 6, 7
V = 8
TEXTS = ["ab c", "c ab", "bad ab c", "ab ab", "c", "bad c ab"]
LN10 = math.log(10.0)

_ARPA = """\\data\\
ngram 1=6
ngram 2=3

\\1-grams:
-99 <s> -0.5
-0.7 </s>
-0.9 <unk>
-0.6 ab -0.3
-1.1 c -0.1
-1.3 bad

\\2-grams:
-0.2 <s> ab
-0.4 ab c
-0.3 c </s>

\\end\\
"""


def _arpa(tmp_path):
    p = str(tmp_path / "w.arpa")
    with open(p, "w") as f:
        f.write(_ARPA)
    return p


def _lm(tmp_path, **kw):
    return WordLM.from_arpa(_arpa(tmp_path), SYMBOLS, blank=START, end=END, **kw)


# ---------------------------------------------------------------------------------------------
# WordLM with an end class
# ---------------------------------------------------------------------------------------------
def test_arpa_round_trip_keeps_the_end_class(tmp_path):
    lm = _lm(tmp_path, oov_penalty=-1.5)
    assert (lm.end, lm.blank, lm.delimiter, lm.num_classes) == (END, START, DELIM, V)
    assert lm.words == ["ab", "bad", "c"]
    p = str(tmp_path / "again.arpa")
    lm.to_arpa(p)
    again = WordLM.from_arpa(p, SYMBOLS, blank=START, end=END, oov_penalty=-1.5)
    assert again.end == END and again.words == lm.words
    for k in ("keys", "vals", "logp", "bow", "lex_keys", "lex_vals", "lex_word"):
        assert (again.host_tables()[k] == lm.host_tables()[k]).all(), k
    # the end class spells nothing; the lexicon is the one the CTC layout spells
    assert lm.spell("ab") == (0, 1) and lm.spell("</s>") is None
    ctc = WordLM.from_arpa(_arpa(tmp_path), list("abcde") + [" "])
    assert ctc.end is None
    assert (ctc.host_tables()["lex_keys"] == lm.host_tables()["lex_keys"]).all()


def test_training_with_an_end_class(tmp_path):
    lm = WordLM.train(TEXTS, 3, SYMBOLS, blank=START, end=END)
    plain = WordLM.train(TEXTS, 3, SYMBOLS, blank=START)
    assert lm.end == END and plain.end is None
    assert lm.words == plain.words == ["ab", "bad", "c"]
    assert (lm.host_tables()["logp"] == plain.host_tables()["logp"]).all()


@pytest.mark.parametrize("end", [START, DELIM, V, -1, 2.0])
def test_a_bad_end_class_is_refused(tmp_path, end):
    with pytest.raises(ValueError):
        WordLM.from_arpa(_arpa(tmp_path), SYMBOLS, blank=START, end=end)
    with pytest.raises(ValueError):
        WordLM.train(TEXTS, 2, SYMBOLS, blank=START, end=end)


def test_a_pickle_from_before_the_end_class_loads_without_one(tmp_path):
    lm = WordLM.from_arpa(_arpa(tmp_path), list("abcde") + [" "])
    d = lm.__getstate__()
    del d["_end"]                          # the state WordLM pickled before it had an end class
    old = WordLM.__new__(WordLM)
    old.__setstate__(d)
    assert old.end is None
    assert pickle.loads(pickle.dumps(_lm(tmp_path))).end == END


# ---------------------------------------------------------------------------------------------
# the Python checks
# ---------------------------------------------------------------------------------------------
def test_seq2seq_accepts_a_word_lm_of_its_layout(tmp_path):
    from speech_b200.models.seq2seq import Seq2Seq
    lm = _lm(tmp_path)
    Seq2Seq._check_lm(lm, 0.8, 1.0, V, START, END)
    Seq2Seq._check_lm(lm, 0.0, 0.0, V, START, END)


@pytest.mark.parametrize("args", [
    (-0.1, 0.0, V, START, END),             # lm_weight < 0
    (math.inf, 0.0, V, START, END),
    (0.5, math.nan, V, START, END),         # insertion_bonus not finite
    (0.5, 0.0, V + 1, START, END),          # class count
    (0.5, 0.0, V, START - 1, END),          # the start token is not the LM's blank
    (0.5, 0.0, V, START, END - 1),          # the end token is not the LM's end class
])
def test_seq2seq_refuses_each_mismatch(tmp_path, args):
    from speech_b200.models.seq2seq import Seq2Seq
    with pytest.raises(ValueError):
        Seq2Seq._check_lm(_lm(tmp_path), *args)


def test_seq2seq_refuses_a_word_lm_without_an_end_class(tmp_path):
    from speech_b200.models.seq2seq import Seq2Seq
    lm = WordLM.from_arpa(_arpa(tmp_path), SYMBOLS, blank=START)
    with pytest.raises(ValueError):
        Seq2Seq._check_lm(lm, 0.5, 1.0, V, START, END)


def test_the_ctc_search_refuses_a_word_lm_with_an_end_class(tmp_path):
    from speech_b200.models.ctc_decoder import check_lm
    lm = _lm(tmp_path)
    with pytest.raises(ValueError):
        check_lm(lm, 0.5, 1.0, V, START)
    check_lm(WordLM.from_arpa(_arpa(tmp_path), SYMBOLS, blank=START), 0.5, 1.0, V, START)


# ---------------------------------------------------------------------------------------------
# the reference's table, by hand
# ---------------------------------------------------------------------------------------------
def test_every_row_of_the_candidate_table(tmp_path):
    lm = _lm(tmp_path, oov_penalty=-2.5)
    a, b, g = 0.8, 1.0, -2.5
    part = WordPart(WordArpa(_arpa(tmp_path), lm.spell, lm.delimiter), END, a, b, g)
    s, p = -3.25, -0.625
    A, B_, C_, D = 0, 1, 2, 3              # letters a b c d
    lp = {("<s>", "ab"): -0.2, ("ab", "c"): -0.4, ("c", "</s>"): -0.3}

    def uni(w):
        return {"</s>": -0.7, "<unk>": -0.9, "ab": -0.6, "c": -1.1, "bad": -1.3}[w] * LN10
    bow = {"<s>": -0.5 * LN10, "ab": -0.3 * LN10, "c": -0.1 * LN10}
    # the delimiter with an empty partial word: free, leading or repeated
    assert part.value(s, (), DELIM, p) == s + p
    assert part.value(s, (A, B_, DELIM), DELIM, p) == s + p
    # the delimiter ending a word of the lexicon: d = (a lm(ab | <s>) + b) + 0
    d = (a * (lp[("<s>", "ab")] * LN10) + b) + 0.0
    assert part.value(s, (A, B_), DELIM, p) == s + (p + d)
    # ... a lexicon prefix that is no word ("ba"): <unk>, charged gamma now
    d = (a * (bow["<s>"] + uni("<unk>")) + b) + g
    assert part.value(s, (B_, A), DELIM, p) == s + (p + d)
    # ... a word that left the lexicon ("aa", node -1): <unk>, gamma charged already
    d = (a * (bow["<s>"] + uni("<unk>")) + b) + 0.0
    assert part.value(s, (A, A), DELIM, p) == s + (p + d)
    # END after a completed word: e = 0.0, then lm(</s> | ab) backs off
    t = 0.0 + a * (bow["ab"] + uni("</s>"))
    assert part.value(s, (A, B_, DELIM), END, p) == s + (p + t)
    # END with a trailing word "c": its delimiter term, then lm(</s> | c)
    e = (a * (lp[("ab", "c")] * LN10) + b) + 0.0
    t = e + a * (lp[("c", "</s>")] * LN10)
    assert part.value(s, (A, B_, DELIM, C_), END, p) == s + (p + t)
    # END of the empty hypothesis: lm(</s> | <s>)
    assert part.value(s, (), END, p) == s + (p + (0.0 + a * (bow["<s>"] + uni("</s>"))))
    # a class with no lexicon child: gamma, once
    assert part.value(s, (A,), A, p) == s + (p + g)
    assert part.value(s, (), D, p) == s + (p + g)
    assert part.value(s, (A, A), B_, p) == s + p               # node -1 already
    # a class with a lexicon child
    assert part.value(s, (A,), B_, p) == s + p
    assert part.value(s, (A, B_, DELIM), C_, p) == s + p
    # zero weights add nothing anywhere
    zero = WordPart(part.arpa, END, 0.0, 0.0, 0.0)
    for hyp in [(), (A,), (A, B_), (B_, A), (A, A), (A, B_, DELIM)]:
        for c in range(V - 1):
            assert zero.value(s, hyp, c, p) == s + p, (hyp, c)


# ---------------------------------------------------------------------------------------------
# the C ABI
# ---------------------------------------------------------------------------------------------
def _wlm_struct(ng=None, **kw):
    f = dict(keys=8, vals=8, logp=8, bow=8, tok=8, cap=64, order=3, num_classes=10, bos=7,
             blank=-1, lm_upper=0.0, lm_abs=10.0)
    f.update(ng or {})
    ngram = _lib.SbNgramLm(*[f[name] for name, _ in _lib.SbNgramLm._fields_])
    # C = 29 scored classes, END 28, START 29 (the blank), the space 27
    w = dict(ngram=ngram, lex_keys=8, lex_vals=8, lex_word=8, lex_cap=64, num_words=7, has_unk=1,
             num_classes=30, blank=29, delimiter=27)
    w.update(kw)
    return _lib.SbWordLm(*[w[name] for name, _ in _lib.SbWordLm._fields_])


@pytest.mark.parametrize("ng,kw,weights,K,wn,status", [
    ({}, {}, (-0.5, 0.0, 0.0), 8, 8, 1),
    ({}, {}, (math.inf, 0.0, 0.0), 8, 8, 1),
    ({}, {}, (math.nan, 0.0, 0.0), 8, 8, 1),
    ({}, {}, (0.5, math.nan, 0.0), 8, 8, 1),
    ({}, {}, (0.5, -math.inf, 0.0), 8, 8, 1),
    ({}, {}, (0.5, 0.0, 0.5), 8, 8, 1),                # oov_penalty > 0
    ({}, {}, (0.5, 0.0, math.nan), 8, 8, 1),
    ({}, {"has_unk": 0}, (0.5, 0.0, -2.5), 8, 8, 1),   # no <unk>: oov_penalty must be -inf
    ({}, {"delimiter": 28}, (0.5, 0.0, 0.0), 8, 8, 1),  # END
    ({}, {"delimiter": 29}, (0.5, 0.0, 0.0), 8, 8, 1),  # outside [0, C)
    ({}, {"delimiter": -1}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({}, {"blank": 0}, (0.5, 0.0, 0.0), 8, 8, 1),      # a scored class
    ({}, {"blank": 28}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({}, {"num_classes": 28}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({}, {"lex_keys": None}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({}, {"lex_word": None}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({"keys": None}, {}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({}, {"lex_cap": 48}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({"cap": 48}, {}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({"order": 0}, {}, (0.5, 0.0, 0.0), 8, 8, 1),
    ({}, {}, (0.5, 0.0, 0.0), 8, None, 1),             # no word_nodes
    ({"order": 11}, {}, (0.5, 0.0, 0.0), 8, 8, 3),
    ({}, {}, (0.5, 0.0, 0.0), 33, 8, 3),
])
def test_wordlm_entry_points_reject_bad_arguments(ng, kw, weights, K, wn, status):
    """every check fails before any launch, so fake device pointers are never dereferenced"""
    lib = _lib.load()
    st = ctypes.byref(_wlm_struct(ng, **kw))
    C, end, start = 29, 28, 29
    sel = (8, 8, 8, 8, 8, 8, 8, K, C, end, 0, 20, 1000, 500, 8, 2)
    assert lib.sb_s2s_beam_select_wordlm_batch(*sel, st, *weights, wn, None) == status
    assert lib.sb_s2s_beam_select_split_wordlm_batch(*sel, 8, 1 << 30, st, *weights, wn,
                                                     None) == status
    assert lib.sb_s2s_ctc_candidates_wordlm(8, 8, None, 8, 8, 1000, 8, 1 << 30, K, C, 4, 10,
                                            start, end, 0.3, 0, 8, 2, st, *weights, wn,
                                            None) == status
    # a null table
    assert lib.sb_s2s_beam_select_wordlm_batch(*sel, None, *weights, wn, None) == 1
    assert lib.sb_s2s_ctc_candidates_wordlm(8, 8, None, 8, 8, 1000, 8, 1 << 30, 8, C, 4, 10,
                                            start, end, 0.3, 0, 8, 2, None, 0.5, 0.0, 0.0, 8,
                                            None) == 1


def test_s2s_wordlm_symbols_are_bound():
    lib = _lib.load()
    for name in ("sb_s2s_beam_select_wordlm_batch", "sb_s2s_beam_select_split_wordlm_batch",
                 "sb_s2s_ctc_candidates_wordlm"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name
