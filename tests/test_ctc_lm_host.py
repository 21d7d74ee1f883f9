"""Host checks (no GPU) of the n-gram LM behind the LM-fused CTC prefix beam search:

- speech_b200.lm.NGramLM: ARPA round trip, interpolated Kneser-Ney training against a direct
  computation from the counts, normalisation, input validation;
- its packed device tables, read by a Python mirror of csrc/decode.cu's context walk and lookup,
  against the ARPA backoff lookup of tests/ngram_ref.py;
- the LM-aware shortlist bound of csrc/decode.cu, restated in the reference's arithmetic, against
  the full LM-fused search (tests/ctc_lm_ref.py);
- the C ABI's argument checks, workspace query and bound symbols.
"""
import ctypes
import itertools
import math

import numpy as np
import pytest

from ctc_lm_ref import prefix_beam_search_lm
from ngram_ref import ArpaLM, KneserNey
from oracle.ctc_decoder_ref import NEG_INF, _lse
from speech_b200 import _lib
from speech_b200.lm import NGramLM


def _corpus(rng, n, V, max_len=12):
    return [rng.randint(0, V, rng.randint(0, max_len)).tolist() for _ in range(n)]


def _symbols(V):
    return [chr(ord("a") + c) for c in range(V)]


def _random_arpa(path, rng, V, order, unk=False, drop=()):
    """An ARPA model with random values: positive and negative backoffs, missing backoffs,
    n-grams whose context is not stored, optionally <unk> and classes left out (`drop`)."""
    words = [w for c, w in enumerate(_symbols(V)) if c not in drop] + (["<unk>"] if unk else [])
    sec = {1: {(w,): None for w in words + ["</s>", "<s>"]}}
    for n in range(2, order + 1):
        sec[n] = {}
        for _ in range(6 * V):
            g = tuple(rng.choice(words + ["</s>"], n).tolist())
            if rng.rand() < 0.5:
                g = ("<s>",) + g[1:]
            if "</s>" in g[:-1]:
                continue
            sec[n][g] = None
    lines = ["\\data\\"] + ["ngram %d=%d" % (n, len(sec[n])) for n in sec]
    for n in sec:
        lines += ["", "\\%d-grams:" % n]
        for g in sec[n]:
            p = -99.0 if g == ("<s>",) else -rng.rand() * 3
            line = "%r\t%s" % (p, " ".join(g))
            if n < order and rng.rand() < 0.7:
                line += "\t%r" % (rng.randn() * 0.8)
            lines.append(line)
    lines += ["", "\\end\\", ""]
    open(path, "w").write("\n".join(lines))


# ---------------------------------------------------------------------------------------------
# NGramLM
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 3, 6])
def test_arpa_round_trip_is_exact(tmp_path, order):
    rng = np.random.RandomState(order)
    V = 7
    lm = NGramLM.train(_corpus(rng, 40, V), order, V + 1, V)
    for symbols in (None, _symbols(V)):
        p = str(tmp_path / "lm.arpa")
        lm.to_arpa(p, symbols)
        back = NGramLM.from_arpa(p, symbols if symbols else [str(c) for c in range(V)])
        assert back.order == order and back.num_classes == V + 1
        assert back._ngrams == lm._ngrams
        for k in ("keys", "vals", "logp", "bow", "tok"):
            assert np.array_equal(back.host_tables()[k], lm.host_tables()[k])
        assert back.host_tables()["lm_upper"] == lm.host_tables()["lm_upper"]


def test_blank_inside_the_symbol_list(tmp_path):
    rng = np.random.RandomState(3)
    seqs = [[c + 1 for c in seq] for seq in _corpus(rng, 20, 5)]
    lm = NGramLM.train(seqs, 3, 6, 0)                            # blank = class 0
    p = str(tmp_path / "lm.arpa")
    symbols = ["_"] + _symbols(5)
    lm.to_arpa(p, symbols)
    back = NGramLM.from_arpa(p, symbols, blank=0)
    assert back.num_classes == 6 and back.blank == 0 and back._ngrams == lm._ngrams


def test_symbols_as_a_class_mapping(tmp_path):
    """the reference Preprocessor.int_to_char is a dict {class: char}"""
    rng = np.random.RandomState(4)
    V = 6
    lm = NGramLM.train(_corpus(rng, 20, V), 3, V + 1, V)
    int_to_char = dict(enumerate(_symbols(V)))
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p, int_to_char)
    back = NGramLM.from_arpa(p, int_to_char)
    assert back.num_classes == V + 1 and back.blank == V and back._ngrams == lm._ngrams
    assert NGramLM.from_arpa(p, _symbols(V))._ngrams == lm._ngrams
    with pytest.raises(ValueError):
        NGramLM.from_arpa(p, {c + 1: s for c, s in int_to_char.items()})


def _contexts(V, L):
    return [pre for n in range(L + 1) for pre in itertools.product(range(V), repeat=n)]


@pytest.mark.parametrize("order", [1, 2, 3, 4, 5, 6])
def test_trained_lm_is_normalised_and_is_kneser_ney(tmp_path, order):
    rng = np.random.RandomState(10 + order)
    V = 4
    seqs = _corpus(rng, 30, V - 1, max_len=9)          # class V - 1 is never seen
    lm = NGramLM.train(seqs, order, V + 1, V)
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p, _symbols(V))
    ref = ArpaLM(p, _symbols(V), V)
    kn = KneserNey(seqs, order, V + 1, V)
    seen = unseen = 0
    for pre in _contexts(V, min(order, 4)):
        h = ref.context(pre)
        hk = tuple("B" if w == "<s>" else ord(w) - ord("a") for w in h)
        seen_here = any(g[:-1] == hk for g in kn.count if len(g) == len(hk) + 1)
        seen += seen_here
        unseen += not seen_here
        total = 0.0
        for s in list(range(V)) + ["</s>"]:
            v = ref.score(pre, s)
            total += math.exp(v)
            direct = math.log(kn.prob(hk, "E" if s == "</s>" else s))
            assert abs(v - direct) <= 1e-12, (pre, s, v, direct)
        assert abs(total - 1.0) <= 1e-9, (pre, total)
    assert seen and (unseen or order == 1)


def test_every_class_gets_a_unigram():
    lm = NGramLM.train([[0, 0, 1]], 3, 10, 9)                   # classes 2..8 never seen
    uni = lm.host_tables()
    assert all(uni["tok"][c] == c for c in range(9)) and uni["tok"][9] == -1


# ---------------------------------------------------------------------------------------------
# device tables: a Python mirror of csrc/decode.cu's lookup
# ---------------------------------------------------------------------------------------------
def _find(t, node, tok, kind):
    key = (node << 32) | ((tok + 1) << 1) | kind
    cap = t["cap"]
    h = ((key * 0x9E3779B97F4A7C15) & ((1 << 64) - 1)) >> 32 & (cap - 1)
    while int(t["keys"][h]) != 0:
        if int(t["keys"][h]) == key:
            return int(t["vals"][h])
        h = (h + 1) & (cap - 1)
    return -1


def _device_lookup(t, prefix, s):
    """lm_resolve (most recent first, -1 = <s>) then LmFuse::lm_logp"""
    hist = ([-1] + list(prefix))[::-1][:t["order"] - 1]
    ctx = [0]
    for h in hist:
        nc = _find(t, ctx[-1], t["bos"] if h < 0 else int(t["tok"][h]), 0)
        if nc < 0:
            break
        ctx.append(nc)
        if h < 0:
            break
    acc = 0.0
    for c in reversed(ctx):
        g = _find(t, c, int(t["tok"][s]), 1)
        if g >= 0:
            return acc + float(t["logp"][g])
        acc += float(t["bow"][c])
    raise AssertionError("no unigram")


@pytest.mark.parametrize("order,unk,drop", [(1, False, ()), (2, False, ()), (3, True, (1, 4)),
                                            (5, True, (0,)), (4, False, ())])
def test_device_lookup_equals_arpa_backoff(tmp_path, order, unk, drop):
    rng = np.random.RandomState(order * 13 + len(drop))
    V = 5
    p = str(tmp_path / "lm.arpa")
    _random_arpa(p, rng, V, order, unk, drop)
    lm = NGramLM.from_arpa(p, _symbols(V))
    ref = ArpaLM(p, _symbols(V), V)
    t = lm.host_tables()
    upper = -math.inf
    for pre in _contexts(V, min(order + 1, 4)):
        for s in range(V):
            v = _device_lookup(t, pre, s)
            assert v == ref.score(pre, s), (pre, s)
            upper = max(upper, v)
            assert abs(v) <= t["lm_abs"]
    assert upper <= t["lm_upper"]


def test_trained_tables_equal_arpa_backoff(tmp_path):
    rng = np.random.RandomState(5)
    V = 6
    lm = NGramLM.train(_corpus(rng, 50, V), 4, V + 1, V)
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p, _symbols(V))
    ref = ArpaLM(p, _symbols(V), V)
    t = lm.host_tables()
    for pre in _contexts(V, 4):
        for s in range(V):
            assert _device_lookup(t, pre, s) == ref.score(pre, s)


# ---------------------------------------------------------------------------------------------
# the LM-aware shortlist search
# ---------------------------------------------------------------------------------------------
def _shortlist_search_lm(probs, K, blank, lm, a, b, lm_upper, lm_abs):
    """prefix_beam_search_lm scoring per frame only the 2K+1 most probable non-blank symbols, the
    blank and every entry's last symbol, with csrc/decode.cu's LM-aware check and fall-back"""
    T, S = probs.shape
    with np.errstate(divide="ignore"):
        logp = np.log(probs)
    L = min(2 * K + 1, S - 1)
    beam = [((), (0.0, NEG_INF))]
    rescans = 0
    for t in range(T):
        lp = logp[t]
        order = sorted((s for s in range(S) if s != blank), key=lambda s: (-float(lp[s]), s))
        short = order[:L]

        def step(symbols):
            cand = {}

            def slot(prefix):
                if prefix not in cand:
                    cand[prefix] = [NEG_INF, NEG_INF]
                return cand[prefix]

            for s in symbols:
                p = float(lp[s])
                for prefix, (p_b, p_nb) in beam:
                    if s == blank:
                        e = slot(prefix)
                        e[0] = _lse(e[0], p_b + p, p_nb + p)
                        continue
                    q = p + (a * lm.score(prefix, s) + b)
                    last = prefix[-1] if prefix else None
                    e = slot(prefix + (s,))
                    if s != last:
                        e[1] = _lse(e[1], p_b + q, p_nb + q)
                    else:
                        e[1] = _lse(e[1], p_b + q)
                        k = slot(prefix)
                        k[1] = _lse(k[1], p_nb + p)
            ranked = sorted(cand.items(), key=lambda kv: _lse(*kv[1]), reverse=True)
            return [(k, (v[0], v[1])) for k, v in ranked[:K]]

        if L == S - 1:
            beam = step(range(S))
            continue
        lasts = {pr[-1] for pr, _ in beam if pr}
        sel = step(sorted(set(short) | lasts | {blank}))
        pmin = float(lp[short[-1]])
        qmax = pmin + (a * lm_upper + b)
        U = max(_lse(pb + qmax, pnb + qmax) for _, (pb, pnb) in beam)
        kth = _lse(*sel[-1][1]) if len(sel) == K else NEG_INF
        mag = 1 + abs(U) + abs(pmin) + a * lm_abs + abs(b)
        ok = kth != NEG_INF and (U == NEG_INF or kth > U + 1e-12 * mag)
        if not ok:
            rescans += 1
            sel = step(range(S))
        beam = sel
    best = beam[0]
    return best[0], -_lse(*best[1]), rescans


def _lattice(rng, kind, T, S):
    x = rng.randn(T, S) * 2.5
    if kind == "zeros":
        x[rng.rand(T, S) < 0.7] = -np.inf
        x[:, S - 1] = np.maximum(x[:, S - 1], 0.0)
    p = np.exp(x - x.max(1, keepdims=True))
    return (p / p.sum(1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("K", [1, 2, 8])
@pytest.mark.parametrize("kind", ["random", "zeros"])
def test_lm_shortlist_search_equals_oracle(tmp_path, K, kind):
    rng = np.random.RandomState(K * 5 + len(kind))
    rescans = frames = 0
    for it in range(8):
        T = rng.randint(4, 10)
        S = rng.randint(2 * K + 3, 2 * K + 12)
        blank = S - 1
        order = [1, 2, 3, 5][it % 4]
        lm = NGramLM.train(_corpus(rng, 25, S - 1, 8), order, S, blank)
        p = str(tmp_path / "lm.arpa")
        lm.to_arpa(p)
        ref = ArpaLM(p, [str(c) for c in range(S - 1)], blank)
        t = lm.host_tables()
        a, b = [(0.0, 0.0), (0.5, 1.0), (2.0, -0.5), (1.0, 0.0)][it % 4]
        probs = _lattice(rng, kind, T, S)
        lab, sc, n = _shortlist_search_lm(probs, K, blank, ref, a, b, t["lm_upper"], t["lm_abs"])
        ref_lab, ref_sc = prefix_beam_search_lm(probs, K, blank, ref, a, b)
        assert tuple(lab) == tuple(ref_lab)
        assert sc == ref_sc or (math.isinf(sc) and math.isinf(ref_sc))
        rescans += n
        frames += T
    assert rescans > 0                                  # the fall-back is exercised
    assert rescans < frames or K == 8


def test_zero_weights_reproduce_the_plain_search(tmp_path):
    from oracle.ctc_decoder_ref import prefix_beam_search
    rng = np.random.RandomState(2)
    lm = NGramLM.train(_corpus(rng, 20, 9), 3, 10, 9)
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p)
    ref = ArpaLM(p, [str(c) for c in range(9)], 9)
    for K in (1, 4):
        probs = _lattice(rng, "random", 12, 10)
        assert prefix_beam_search_lm(probs, K, 9, ref, 0.0, 0.0) == prefix_beam_search(probs, K, 9)


# ---------------------------------------------------------------------------------------------
# validation
# ---------------------------------------------------------------------------------------------
def _write(tmp_path, text):
    p = str(tmp_path / "bad.arpa")
    open(p, "w").write(text)
    return p


_GOOD = "\\data\\\nngram 1=4\nngram 2=1\n\n\\1-grams:\n-1.0\ta\t-0.2\n-1.0\tb\n-0.5\t</s>\n" \
        "-99\t<s>\t-0.1\n\n\\2-grams:\n-0.3\t<s> a\n\n\\end\\\n"


def test_good_arpa_reads(tmp_path):
    lm = NGramLM.from_arpa(_write(tmp_path, _GOOD), ["a", "b"])
    assert lm.order == 2 and lm.num_classes == 3


@pytest.mark.parametrize("text", [
    _GOOD.replace("\\data\\\n", ""),                                  # no \data\
    _GOOD.replace("ngram 1=4", "ngram 1=5"),                          # wrong count
    _GOOD.replace("ngram 2=1", "ngram 2=2"),
    _GOOD.replace("ngram 2=1", "ngram 2=0"),
    _GOOD.replace("\\2-grams:", "\\3-grams:"),                        # missing section
    _GOOD.replace("\\end\\\n", ""),                                   # no \end\
    _GOOD.replace("-1.0\tb", "-1.0\tb c d"),                          # malformed line
    _GOOD.replace("-1.0\tb", "x\tb"),
    _GOOD.replace("-1.0\tb", "-inf\tb"),                              # non-finite
    _GOOD.replace("-1.0\tb", "nan\tb"),
    _GOOD.replace("-0.2", "inf"),
    _GOOD.replace("-1.0\tb", "-1.0\ta"),                              # duplicate n-gram
    _GOOD.replace("-1.0\tb\n", "-1.0\tz\n"),                          # class b absent, no <unk>
])
def test_bad_arpa_raises(tmp_path, text):
    with pytest.raises(ValueError):
        NGramLM.from_arpa(_write(tmp_path, text), ["a", "b"])


def test_unk_covers_absent_classes(tmp_path):
    text = _GOOD.replace("-1.0\tb\n", "-1.5\t<unk>\n")
    lm = NGramLM.from_arpa(_write(tmp_path, text), ["a", "b"])
    assert lm.host_tables()["tok"][1] == 3 + 2


def test_order_limits(tmp_path):
    text = "\\data\\\n" + "".join("ngram %d=0\n" % n for n in range(1, 12)) + "\\end\\\n"
    with pytest.raises(ValueError):
        NGramLM.from_arpa(_write(tmp_path, text), ["a"])
    for order in (0, 11):
        with pytest.raises(ValueError):
            NGramLM.train([[0]], order, 3, 2)


@pytest.mark.parametrize("symbols", [["a", "b c"], ["a", "a"], ["a", ""], ["a", "<s>"]])
def test_bad_symbols_raise(tmp_path, symbols):
    with pytest.raises(ValueError):
        NGramLM.from_arpa(_write(tmp_path, _GOOD), symbols)
    lm = NGramLM.train([[0, 1]], 2, 3, 2)
    with pytest.raises(ValueError):
        lm.to_arpa(str(tmp_path / "out.arpa"), symbols)


@pytest.mark.parametrize("seqs", [[[0, 5]], [[2]], [[-1]]])
def test_bad_training_labels_raise(seqs):
    with pytest.raises(ValueError):
        NGramLM.train(seqs, 3, 3, 2)


def test_decoder_rejects_bad_fusion_arguments():
    from speech_b200.models.ctc_decoder import check_lm
    lm = NGramLM.train([[0, 1]], 2, 3, 2)
    check_lm(None, 0.0, 0.0, 3, 0)
    check_lm(lm, 0.5, -1.0, 3, 2)
    for args in [(None, 0.5, 0.0, 3, 2), (None, 0.0, 1.0, 3, 2), (lm, 0.5, 0.0, 4, 2),
                 (lm, -0.1, 0.0, 3, 2), (lm, math.inf, 0.0, 3, 2), (lm, 0.1, math.nan, 3, 2),
                 (lm, 0.5, 0.0, 3, 0)]:                   # the LM's blank is 2, the search's 0
        with pytest.raises(ValueError):
            check_lm(*args)


# ---------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------
def test_lm_symbols_are_bound():
    lib = _lib.load()
    for name in ("sb_ctc_prefix_beam_lm_workspace_size", "sb_ctc_prefix_beam_lm",
                 "sb_ctc_prefix_beam_lm_shortlist"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


@pytest.mark.parametrize("B,T,K", [(1, 1, 1), (4, 247, 8), (64, 247, 32)])
def test_lm_workspace_equals_the_plain_search(B, T, K):
    lib = _lib.load()
    plain = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, K)
    for order in (1, 5, 10):
        assert _lib.workspace_size(lib.sb_ctc_prefix_beam_lm_workspace_size, B, T, K,
                                   order) == plain
    n = ctypes.c_size_t(0)
    assert lib.sb_ctc_prefix_beam_lm_workspace_size(B, T, K, 11, ctypes.byref(n)) == 3
    assert lib.sb_ctc_prefix_beam_lm_workspace_size(B, T, K, 0, ctypes.byref(n)) == 1


def _lm_struct(**kw):
    f = dict(keys=8, vals=8, logp=8, bow=8, tok=8, cap=64, order=3, num_classes=29, bos=29,
             blank=28, lm_upper=0.0, lm_abs=10.0)
    f.update(kw)
    return _lib.SbNgramLm(*[f[name] for name, _ in _lib.SbNgramLm._fields_])


@pytest.mark.parametrize("kw,weights,K,status", [
    ({}, (-0.5, 0.0), 8, 1),
    ({}, (math.nan, 0.0), 8, 1),
    ({}, (math.inf, 0.0), 8, 1),
    ({}, (0.5, math.inf), 8, 1),
    ({"num_classes": 28}, (0.5, 0.0), 8, 1),
    ({"lm_upper": math.inf}, (0.5, 0.0), 8, 1),
    ({"keys": None}, (0.5, 0.0), 8, 1),
    ({"blank": 0}, (0.5, 0.0), 8, 1),
    ({"order": 11}, (0.5, 0.0), 8, 3),
    ({}, (0.5, 0.0), 33, 3),
])
def test_lm_entry_points_reject_bad_arguments(kw, weights, K, status):
    """every check fails before any launch, so fake device pointers are never dereferenced"""
    lib = _lib.load()
    st = _lm_struct(**kw)
    for fn in (lib.sb_ctc_prefix_beam_lm, lib.sb_ctc_prefix_beam_lm_shortlist):
        assert fn(8, 8, 2, 10, 29, K, 28, ctypes.byref(st), weights[0], weights[1], 8, 8, 8, 8,
                  1 << 30, None) == status
