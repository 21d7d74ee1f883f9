"""Host checks (no GPU) of the word n-gram LM behind the word-LM CTC prefix beam search:

- speech_b200.lm.WordLM: ARPA round trip, Kneser-Ney training against a direct computation from
  the counts, normalisation, spelling and dropping, input validation;
- its packed device tables (word n-gram and lexicon), read by a Python mirror of csrc/decode.cu's
  lookups, against the plain ARPA word backoff of tests/ctc_wordlm_ref.py;
- the reference search's zero-weight and closed-vocabulary properties;
- the refusals of bad fusion arguments by every search, in Python and at the C ABI;
- compute_wer, and the new symbols.
"""
import ctypes
import itertools
import math

import numpy as np
import pytest

from ctc_wordlm_ref import WordArpa, prefix_beam_search_wordlm
from ngram_ref import KneserNey
from speech_b200 import _lib
from speech_b200.lm import WordLM

CHARS = "abcde"
SYMBOLS = list(CHARS) + [" "]          # classes 0..4 letters, 5 the space; blank 6
DELIM, BLANK = 5, 6


def _texts(rng, n, vocab, max_words=6):
    return [" ".join(rng.choice(vocab, rng.randint(1, max_words))) for _ in range(n)]


def _vocab(rng, n, max_len=4):
    words = set()
    while len(words) < n:
        words.add("".join(rng.choice(list(CHARS), rng.randint(1, max_len + 1))))
    return sorted(words)


def _ref(path, lm):
    return WordArpa(path, lm.spell, lm.delimiter)


# ---------------------------------------------------------------------------------------------
# WordLM
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2, 3, 5])
def test_arpa_round_trip_is_exact(tmp_path, order):
    rng = np.random.RandomState(order)
    lm = WordLM.train(_texts(rng, 40, _vocab(rng, 12)), order, SYMBOLS)
    p = str(tmp_path / "w.arpa")
    lm.to_arpa(p)
    back = WordLM.from_arpa(p, SYMBOLS)
    assert back.order == order and back.words == lm.words and back._ngrams == lm._ngrams
    assert back.dropped == 0 and back.num_classes == 7 and back.blank == BLANK
    assert back.delimiter == DELIM and back.num_words == lm.num_words
    for k in ("keys", "vals", "logp", "bow", "tok", "lex_keys", "lex_vals", "lex_word"):
        assert np.array_equal(back.host_tables()[k], lm.host_tables()[k]), k
    p2 = str(tmp_path / "w2.arpa")
    back.to_arpa(p2)
    assert open(p).read() == open(p2).read()


@pytest.mark.parametrize("order", [1, 2, 3, 4])
def test_trained_lm_is_normalised_and_is_kneser_ney(tmp_path, order):
    rng = np.random.RandomState(20 + order)
    vocab = _vocab(rng, 5)
    texts = _texts(rng, 30, vocab) + ["a zz b"]          # "zz" cannot be spelled: <unk>
    lm = WordLM.train(texts, order, SYMBOLS)
    W = lm.num_words
    assert "zz" not in lm.words and lm.has_unk
    p = str(tmp_path / "w.arpa")
    lm.to_arpa(p)
    ref = _ref(p, lm)
    tok = {w: t for t, w in enumerate(lm.words)}
    seqs = [[tok.get(w, W) for w in t.split()] for t in texts]
    kn = KneserNey(seqs, order, W + 2, W + 1)            # class W stands for <unk>
    names = lm.words + ["<unk>", "</s>"]
    for n in range(min(order, 3)):
        for h in itertools.product(lm.words + ["<unk>"], repeat=n):
            for start in ((), ("<s>",)):
                hh = (start + h)[-(order - 1):] if order > 1 else ()
                hk = tuple("B" if w == "<s>" else (W if w == "<unk>" else tok[w]) for w in hh)
                total = 0.0
                for w in names:
                    v = ref.logprob(hh, w)
                    total += math.exp(v)
                    direct = math.log(kn.prob(hk, "E" if w == "</s>" else
                                              (W if w == "<unk>" else tok[w])))
                    assert abs(v - direct) <= 1e-12, (hh, w, v, direct)
                assert abs(total - 1.0) <= 1e-9, (hh, total)


_ARPA = ("\\data\\\nngram 1=7\nngram 2=3\n\n\\1-grams:\n-1.0\tab\t-0.2\n-1.2\tabc\n-1.5\tdog\n"
         "-0.9\tb\t-0.3\n-0.5\t</s>\n-99\t<s>\t-0.1\n-2.0\t<unk>\n\n\\2-grams:\n-0.3\t<s> ab\n"
         "-0.4\tab dog\n-0.2\tab b\n\n\\end\\\n")


def _write(tmp_path, text):
    p = str(tmp_path / "lm.arpa")
    open(p, "w").write(text)
    return p


def test_spelling_and_dropping(tmp_path):
    lm = WordLM.from_arpa(_write(tmp_path, _ARPA), SYMBOLS)
    assert lm.words == ["ab", "abc", "b"] and lm.dropped == 2       # "dog" and "ab dog"
    assert lm.spell("abc") == (0, 1, 2) and lm.spell("dog") is None and lm.spell("") is None
    t = lm.host_tables()
    node = _child(t, _child(t, 0, 0), 1)
    assert t["lex_word"][node] == 0                                   # "ab"
    assert _child(t, node, 3) == -1 and t["lex_word"][_child(t, 0, 1)] == 2      # "b"
    # an int_to_char mapping, the blank inside the symbols, another delimiter
    m = WordLM.from_arpa(_write(tmp_path, _ARPA), dict(enumerate(["_"] + list(CHARS) + ["|"])),
                         delimiter="|", blank=0)
    assert m.words == lm.words and m.delimiter == 6 and m.blank == 0 and m.num_classes == 7


@pytest.mark.parametrize("text,kw", [
    (_ARPA.replace("ab", "AB").replace("abc", "ABC").replace("\tb", "\tB"), {}),   # case
    (_ARPA, {"oov_penalty": 0.5}),
    (_ARPA, {"oov_penalty": math.nan}),
    (_ARPA, {"delimiter": "_"}),                       # no class has it
    (_ARPA.replace("-0.5\t</s>\n", "-0.5\tb c\n"), {}),  # no </s>
    (_ARPA.replace("-2.0\t<unk>", "-2.0\tcab"), {}),   # no <unk>: needs oov_penalty = -inf
])
def test_bad_word_lms_raise(tmp_path, text, kw):
    with pytest.raises(ValueError):
        WordLM.from_arpa(_write(tmp_path, text), SYMBOLS, **kw)


def test_oov_penalty_is_settable_and_checked(tmp_path):
    lm = WordLM.from_arpa(_write(tmp_path, _ARPA), SYMBOLS, oov_penalty=-2.5)
    t = lm.host_tables()
    lm.oov_penalty = -math.inf
    assert lm.oov_penalty == -math.inf and lm.host_tables() is t
    for bad in (0.1, math.inf, math.nan):
        with pytest.raises(ValueError):
            lm.oov_penalty = bad
    no_unk = WordLM.from_arpa(_write(tmp_path, _ARPA.replace("-2.0\t<unk>", "-2.0\tcab")),
                              SYMBOLS, oov_penalty=-math.inf)
    assert not no_unk.has_unk
    with pytest.raises(ValueError):
        no_unk.oov_penalty = 0.0
    with pytest.raises(ValueError):
        WordLM.train(["ZZ YY"], 2, SYMBOLS)            # nothing spellable


# ---------------------------------------------------------------------------------------------
# device tables: a Python mirror of csrc/decode.cu's lookups
# ---------------------------------------------------------------------------------------------
def _find(keys, vals, cap, node, tok, kind):
    key = (node << 32) | ((tok + 1) << 1) | kind
    h = ((key * 0x9E3779B97F4A7C15) & ((1 << 64) - 1)) >> 32 & (cap - 1)
    while int(keys[h]) != 0:
        if int(keys[h]) == key:
            return int(vals[h])
        h = (h + 1) & (cap - 1)
    return -1


def _child(t, node, c):
    return _find(t["lex_keys"], t["lex_vals"], t["lex_cap"], node, c, 0)


def _word_lookup(t, hist, w):
    """lm_context over word tokens (most recent first, -1 = <s>), then lm_backoff"""
    ctx = [0]
    for h in hist[:t["order"] - 1]:
        nc = _find(t["keys"], t["vals"], t["cap"], ctx[-1],
                   t["bos"] if h < 0 else int(t["tok"][h]), 0)
        if nc < 0:
            break
        ctx.append(nc)
        if h < 0:
            break
    acc = 0.0
    for c in reversed(ctx):
        g = _find(t["keys"], t["vals"], t["cap"], c, w, 1)
        if g >= 0:
            return acc + float(t["logp"][g])
        acc += float(t["bow"][c])
    return acc


@pytest.mark.parametrize("order", [1, 2, 3, 4])
def test_device_tables_equal_arpa_word_backoff(tmp_path, order):
    rng = np.random.RandomState(40 + order)
    lm = WordLM.train(_texts(rng, 60, _vocab(rng, 8)), order, SYMBOLS)
    p = str(tmp_path / "w.arpa")
    lm.to_arpa(p)
    ref = _ref(p, lm)
    t = lm.host_tables()
    W = lm.num_words
    names = lm.words + ["<s>", "</s>", "<unk>"]
    assert np.array_equal(t["tok"], np.arange(W + 3)) and t["bos"] == W
    for w, word in enumerate(lm.words):                    # the lexicon spells every word
        node = 0
        for c in lm.spell(word):
            node = _child(t, node, c)
        assert node > 0 and t["lex_word"][node] == w
    toks = list(range(W)) + [W + 2]
    for n in range(min(order + 1, 3)):
        for words in itertools.product(toks, repeat=n):    # completed words, oldest first
            hist = list(words[::-1]) + [-1]                # most recent first, then <s>
            h = ref.context([names[x] for x in words])
            for w in toks + [W + 1]:
                assert _word_lookup(t, hist, w) == ref.logprob(h, names[w]), (words, w)


def test_zero_weights_reproduce_the_plain_search(tmp_path):
    from oracle.ctc_decoder_ref import prefix_beam_search
    rng = np.random.RandomState(2)
    lm = WordLM.train(_texts(rng, 20, _vocab(rng, 6)), 3, SYMBOLS)
    p = str(tmp_path / "w.arpa")
    lm.to_arpa(p)
    ref = _ref(p, lm)
    for K in (1, 4):
        x = rng.randn(12, 7) * 2.5
        probs = np.exp(x) / np.exp(x).sum(1, keepdims=True)
        assert prefix_beam_search_wordlm(probs, K, BLANK, ref, 0.0, 0.0, 0.0) == \
            prefix_beam_search(probs, K, BLANK)


def test_closed_vocabulary_keeps_to_the_lexicon(tmp_path):
    rng = np.random.RandomState(3)
    lm = WordLM.train(_texts(rng, 20, _vocab(rng, 5)), 2, SYMBOLS)
    p = str(tmp_path / "w.arpa")
    lm.to_arpa(p)
    ref = _ref(p, lm)
    for _ in range(4):
        x = rng.randn(20, 7) * 2.0
        probs = np.exp(x) / np.exp(x).sum(1, keepdims=True)
        lab, sc = prefix_beam_search_wordlm(probs, 8, BLANK, ref, 0.5, 1.0, -math.inf)
        words, partial = ref.split(lab)
        if math.isfinite(sc):
            assert all(w in lm.words for w in words) and (not partial or partial in ref.word_of)


# ---------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------
def test_other_searches_refuse_a_word_lm(tmp_path):
    from speech_b200.models.ctc_decoder import check_lm
    from speech_b200.models.seq2seq import Seq2Seq
    from speech_b200.transducer_decoders import check_stream_args
    lm = WordLM.from_arpa(_write(tmp_path, _ARPA), SYMBOLS)
    check_lm(lm, 0.5, 1.0, 7, BLANK)                                  # the CTC search
    for args in [(lm, -0.1, 0.0, 7, BLANK), (lm, math.inf, 0.0, 7, BLANK),
                 (lm, 0.5, math.nan, 7, BLANK), (lm, 0.5, 0.0, 8, BLANK),
                 (lm, 0.5, 0.0, 7, 0)]:
        with pytest.raises(ValueError):
            check_lm(*args)
    with pytest.raises(ValueError):
        check_lm(lm, 0.5, 1.0, 7, BLANK, search="Transducer")          # Transducer.recognize
    with pytest.raises(ValueError):
        check_stream_args(4, 4, 100, None, 7, BLANK, lm, 0.5, 1.0)     # Transducer.stream
    with pytest.raises(ValueError):
        Seq2Seq._check_lm(lm, 0.5, 1.0, 7, 6, 5)                       # Seq2Seq.recognize


def _wlm_struct(ng=None, **kw):
    f = dict(keys=8, vals=8, logp=8, bow=8, tok=8, cap=64, order=3, num_classes=10, bos=7,
             blank=-1, lm_upper=0.0, lm_abs=10.0)
    f.update(ng or {})
    ngram = _lib.SbNgramLm(*[f[name] for name, _ in _lib.SbNgramLm._fields_])
    w = dict(ngram=ngram, lex_keys=8, lex_vals=8, lex_word=8, lex_cap=64, num_words=7, has_unk=1,
             num_classes=29, blank=28, delimiter=27)
    w.update(kw)
    return _lib.SbWordLm(*[w[name] for name, _ in _lib.SbWordLm._fields_])


@pytest.mark.parametrize("ng,kw,weights,K,status", [
    ({}, {}, (-0.5, 0.0, 0.0), 8, 1),
    ({}, {}, (math.inf, 0.0, 0.0), 8, 1),
    ({}, {}, (0.5, math.nan, 0.0), 8, 1),
    ({}, {}, (0.5, 0.0, 0.5), 8, 1),                   # oov_penalty > 0
    ({}, {}, (0.5, 0.0, math.nan), 8, 1),
    ({}, {"has_unk": 0}, (0.5, 0.0, -2.5), 8, 1),      # no <unk>: oov_penalty must be -inf
    ({}, {"delimiter": 28}, (0.5, 0.0, 0.0), 8, 1),    # the blank
    ({}, {"delimiter": 29}, (0.5, 0.0, 0.0), 8, 1),    # outside [0, S)
    ({}, {"delimiter": -1}, (0.5, 0.0, 0.0), 8, 1),
    ({}, {"blank": 0}, (0.5, 0.0, 0.0), 8, 1),
    ({}, {"num_classes": 28}, (0.5, 0.0, 0.0), 8, 1),
    ({}, {"lex_keys": None}, (0.5, 0.0, 0.0), 8, 1),
    ({"keys": None}, {}, (0.5, 0.0, 0.0), 8, 1),
    ({}, {"lex_cap": 48}, (0.5, 0.0, 0.0), 8, 1),
    ({"order": 11}, {}, (0.5, 0.0, 0.0), 8, 3),
    ({}, {}, (0.5, 0.0, 0.0), 33, 3),
])
def test_wordlm_entry_points_reject_bad_arguments(ng, kw, weights, K, status):
    """every check fails before any launch, so fake device pointers are never dereferenced"""
    lib = _lib.load()
    st = _wlm_struct(ng, **kw)
    for fn in (lib.sb_ctc_prefix_beam_wordlm, lib.sb_ctc_prefix_beam_wordlm_shortlist):
        assert fn(8, 8, 2, 10, 29, K, 28, ctypes.byref(st), *weights, 8, 8, 8, 8, 1 << 30,
                  None) == status
    for fn in (lib.sb_ctc_stream_step_wordlm, lib.sb_ctc_stream_step_wordlm_shortlist):
        assert fn(8, 8, 2, 10, 29, K, 28, ctypes.byref(st), *weights, 100, 8, 8, 1 << 30,
                  None) == status
    # the stream's best takes S and the blank from the LM, so only the mismatches are no refusal
    if K <= 32 and not {"blank", "num_classes"} & set(kw):
        assert lib.sb_ctc_stream_best_wordlm(8, 2, 100, K, ctypes.byref(st), *weights, 8, 8, 8, 8,
                                             None) == status
    assert lib.sb_ctc_stream_best_wordlm(8, 2, 100, K, None, 0.5, 0.0, 0.0, 8, 8, 8, 8,
                                         None) == 1


def test_wordlm_symbols_are_bound():
    import speech_b200
    lib = _lib.load()
    for name in ("sb_ctc_prefix_beam_wordlm", "sb_ctc_prefix_beam_wordlm_shortlist",
                 "sb_ctc_stream_step_wordlm", "sb_ctc_stream_step_wordlm_shortlist",
                 "sb_ctc_stream_best_wordlm"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name
    assert speech_b200.compute_wer is not None and speech_b200.lm.WordLM is WordLM


# ---------------------------------------------------------------------------------------------
# compute_wer
# ---------------------------------------------------------------------------------------------
def test_compute_wer_by_hand():
    from speech_b200 import compute_wer
    from speech_b200.utils.score import compute_cer
    d = 0
    # "ab c" vs "ab c": 0 of 2
    assert compute_wer([((1, 2, d, 3), (1, 2, d, 3))], d) == 0.0
    # leading, trailing and repeated delimiters make no words
    assert compute_wer([((d, 1, 2, d, d, 3, d), (1, 2, d, 3))], d) == 0.0
    # one substitution ("c" -> "e") and one deletion over 3 + 1 reference words
    res = [((1, d, 2, d, 3), (1, d, 5)), ((4,), (4,))]
    assert compute_wer(res, d) == 2 / 4
    # an insertion: 1 error over 1 word
    assert compute_wer([((1, 2), (1, 2, d, 7))], d) == 1.0
    # a word is a whole run: "ab" vs "ac" is one error, not half
    assert compute_wer([((1, 2), (1, 3))], d) == 1.0
    assert compute_cer([((1, 2), (1, 3))]) == 0.5
