"""Word-LM CTC prefix beam search on the GPU (sb_ctc_prefix_beam_wordlm and the stream forms,
csrc/decode.cu) against the reference search tests/ctc_wordlm_ref.prefix_beam_search_wordlm:
labels identical, float64 scores within 1e-9 relative (the device's log / exp may differ from
libm's in the last bit), over several (K, order, weights) and oov_penalty in {0, -2.5, -inf}
with lens < T;
- the forced shortlist route bit for bit the full scan, and, at a vocabulary the full scan does
  not fit, the shortlist route against the reference;
- zero weights bit for bit the LM-less search; a closed vocabulary keeps every word in the
  lexicon; the word LM picks the in-vocabulary spelling of an ambiguous lattice;
- CTC.infer with a word LM in both padding modes, and CTC.stream after every push.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from ctc_wordlm_ref import WordArpa, prefix_beam_search_wordlm
from speech_b200 import _lib
from speech_b200.lm import WordLM
from speech_b200.models import ctc_decoder

pytestmark = pytest.mark.gpu

LETTERS = [chr(ord("a") + i) for i in range(26)]
SYMBOLS = LETTERS + [" "]                     # classes 0..25, the space 26; blank 27
S, DELIM, BLANK = 28, 26, 27
NEG = -math.inf


def _words(rng, n, lo=2, hi=6):
    out = set()
    while len(out) < n:
        out.add("".join(rng.choice(LETTERS[:12], rng.randint(lo, hi + 1))))
    return sorted(out)


def _wlm(tmp_path, rng, order, vocab, n=300, symbols=SYMBOLS, oov=0.0):
    texts = [" ".join(rng.choice(vocab, rng.randint(1, 8))) for _ in range(n)]
    lm = WordLM.train(texts, order, symbols, oov_penalty=oov)
    p = str(tmp_path / ("w%d.arpa" % order))
    lm.to_arpa(p)
    return lm, WordArpa(p, lm.spell, lm.delimiter)


def _posteriors(rng, vocab, B, T, S=S, delim=DELIM, spell=None, oov=0.2, sharp=2.0):
    """(B, T, S) float32 posteriors of spoken word text: each character on one or two frames
    between blanks, the space between words, some characters confused and some words OOV"""
    spell = spell or (lambda w: [ord(c) - ord("a") for c in w])
    x = rng.randn(B, T, S) * sharp
    for b in range(B):
        t = 0
        while True:
            w = rng.choice(vocab) if rng.rand() > oov else "".join(rng.choice(LETTERS, 3))
            labels = spell(w) + [delim]
            if t + 3 * len(labels) >= T:
                break
            for c in labels:
                for _ in range(rng.randint(1, 3)):
                    x[b, t, c] += 6.0
                    if rng.rand() < 0.3:                          # a confusable character
                        x[b, t, rng.randint(0, S - 1)] += 5.5
                    t += 1
                x[b, t, S - 1] += 5.0
                t += 1
        x[b, t:, S - 1] += 6.0
    p = np.exp(x - x.max(2, keepdims=True))
    return (p / p.sum(2, keepdims=True)).astype(np.float32)


def _call(logp, lens, K, blank, lm=None, w=(0.0, 0.0, 0.0), shortlist=False):
    """a C ABI entry point on host float32 log-probabilities -> [(labels, score)]"""
    lib = _lib.load()
    B, T, S_ = logp.shape
    lp = torch.from_numpy(np.ascontiguousarray(logp, np.float32)).cuda()
    ln = torch.tensor(lens, dtype=torch.int32, device="cuda")
    nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    lab = torch.empty(B, T, dtype=torch.int32, device="cuda")
    n = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = torch.empty(B, dtype=torch.float64, device="cuda")
    outs = (lab.data_ptr(), n.data_ptr(), sc.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr())
    if lm is None:
        fn = lib.sb_ctc_prefix_beam_shortlist if shortlist else lib.sb_ctc_prefix_beam
        st = fn(lp.data_ptr(), ln.data_ptr(), B, T, S_, K, blank, *outs)
    else:
        fn = lib.sb_ctc_prefix_beam_wordlm_shortlist if shortlist else lib.sb_ctc_prefix_beam_wordlm
        tables, _ = lm.device_tables(lp.device)
        st = fn(lp.data_ptr(), ln.data_ptr(), B, T, S_, K, blank, ctypes.byref(tables), *w, *outs)
    _lib.check(st, fn.__name__)
    lab, n, sc = lab.cpu().numpy(), n.cpu().numpy(), sc.cpu().numpy()
    return [(tuple(int(v) for v in lab[i, :n[i]]), float(sc[i])) for i in range(B)]


def _host_log(probs):
    with np.errstate(divide="ignore"):
        return np.log(probs)


def _same(got, want):
    (lab, sc), (ref_lab, ref_sc) = got, want
    assert lab == tuple(ref_lab), (lab, ref_lab)
    if math.isinf(ref_sc):
        assert sc == ref_sc
    else:
        assert abs(sc - ref_sc) <= 1e-9 * max(1.0, abs(ref_sc)), (sc, ref_sc)


@pytest.mark.parametrize("K,order,a,b,g", [
    (1, 3, 0.8, 1.0, 0.0),
    (8, 3, 0.5, 2.0, -2.5),
    (8, 2, 1.5, 0.5, NEG),
    (8, 1, 1.0, 0.0, 0.0),
    (4, 5, 2.0, -1.0, NEG),
    (32, 4, 0.8, 1.0, -2.5),
])
def test_search_equals_oracle(tmp_path, K, order, a, b, g):
    rng = np.random.RandomState(K * 10 + order)
    vocab = _words(rng, 40)
    lm, ref = _wlm(tmp_path, rng, order, vocab, oov=g)
    T = 40 if K == 32 else 70
    lens = [T, T - 13, T // 2]
    probs = _posteriors(rng, vocab, 3, T)
    logp = _host_log(probs)
    res = _call(logp, lens, K, BLANK, lm, (a, b, g))
    for i, L in enumerate(lens):
        _same(res[i], prefix_beam_search_wordlm(probs[i, :L], K, BLANK, ref, a, b, g))
    assert _call(logp, lens, K, BLANK, lm, (a, b, g), shortlist=True) == res


def test_large_vocabulary_takes_the_shortlist_and_equals_oracle(tmp_path):
    # 5000 distinct one-character symbols: K*(S+1)*13 bytes of candidates exceed the full scan's
    S_, K, T = 5001, 4, 14
    symbols = [chr(0x4e00 + i) for i in range(S_ - 2)] + [" "]
    delim, blank = S_ - 2, S_ - 1
    rng = np.random.RandomState(5)
    vocab = ["".join(symbols[c] for c in rng.randint(0, 12, rng.randint(2, 4)))
             for _ in range(30)]
    lm, ref = _wlm(tmp_path, rng, 3, sorted(set(vocab)), symbols=symbols)
    probs = _posteriors(rng, sorted(set(vocab)), 2, T, S=S_, delim=delim,
                        spell=lambda w: list(lm.spell(w) or rng.randint(0, 20, 3)), sharp=3.0)
    lens = [T, 9]
    res = _call(_host_log(probs), lens, K, blank, lm, (0.7, 0.5, -2.0))
    for i, L in enumerate(lens):
        _same(res[i], prefix_beam_search_wordlm(probs[i, :L], K, blank, ref, 0.7, 0.5, -2.0))
    assert res == _call(_host_log(probs), lens, K, blank, lm, (0.7, 0.5, -2.0), shortlist=True)


@pytest.mark.parametrize("K", [1, 8, 32])
def test_zero_weights_are_the_plain_search(tmp_path, K):
    rng = np.random.RandomState(K)
    vocab = _words(rng, 30)
    lm, _ = _wlm(tmp_path, rng, 3, vocab)
    lens = [80, 61, 5]
    probs = _posteriors(rng, vocab, 3, 80)
    logp = _host_log(probs)
    for sl in (False, True):
        assert _call(logp, lens, K, BLANK, lm, (0.0, 0.0, 0.0), sl) == _call(logp, lens, K, BLANK,
                                                                             shortlist=sl)
    pt = torch.from_numpy(probs).cuda()
    assert (ctc_decoder.decode_batch(pt, K, BLANK, lens, True, lm=lm)
            == ctc_decoder.decode_batch(pt, K, BLANK, lens, True))


def test_closed_vocabulary_keeps_to_the_lexicon(tmp_path):
    rng = np.random.RandomState(11)
    vocab = _words(rng, 25)
    lm, ref = _wlm(tmp_path, rng, 3, vocab, oov=NEG)
    probs = _posteriors(rng, vocab, 8, 120, oov=0.4)
    pt = torch.from_numpy(probs).cuda()
    for K in (4, 16):
        finite = 0
        for lab, sc in ctc_decoder.decode_batch(pt, K, BLANK, with_scores=True, lm=lm,
                                                lm_weight=0.5, insertion_bonus=1.0):
            text = "".join(SYMBOLS[c] for c in lab)
            # a finite result is made of lexicon words; where every final entry ends inside a
            # non-word (score +inf, the beam too narrow), its completed words still are
            words = text.split() if math.isfinite(sc) else text[:text.rfind(" ") + 1].split()
            assert all(w in lm.words for w in words), words
            finite += math.isfinite(sc)
        assert finite >= 6, finite


def test_the_word_lm_picks_the_in_vocabulary_spelling(tmp_path):
    # "c", then "a" or "s" (slightly for "s"), then "t": the LM-less search reads "cst"
    lm = WordLM.train(["cat dog", "dog cat", "cat"] * 20, 2, SYMBOLS, oov_penalty=-3.0)
    p = np.full((1, 7, S), 0.002, np.float32)
    for t, c in enumerate([2, BLANK, None, BLANK, 19, BLANK, BLANK]):
        if c is not None:
            p[0, t, c] = 0.96
    p[0, 2, 0], p[0, 2, 18] = 0.45, 0.50
    p /= p.sum(2, keepdims=True)
    pt = torch.from_numpy(p).cuda()
    for K in (1, 4):
        assert ctc_decoder.decode_batch(pt, K, BLANK)[0] == (2, 18, 19)
        lm.oov_penalty = 0.0
        assert ctc_decoder.decode_batch(pt, K, BLANK, lm=lm, lm_weight=0.0)[0] == (2, 18, 19)
        # the word's LM score arrives at its end (no look-ahead): only a beam that still holds
        # "ca" then can take it
        want = (2, 0, 19) if K > 1 else (2, 18, 19)
        assert ctc_decoder.decode_batch(pt, K, BLANK, lm=lm, lm_weight=1.0)[0] == want
        # the OOV penalty is charged where "cs" leaves the lexicon, so any beam avoids it
        lm.oov_penalty = -3.0
        assert ctc_decoder.decode_batch(pt, K, BLANK, lm=lm, lm_weight=0.0)[0] == (2, 0, 19)
        lab, sc = ctc_decoder.decode(p[0], K, BLANK, lm=lm, lm_weight=1.0, insertion_bonus=0.5)
        assert lab == (2, 0, 19) and np.isfinite(sc)


def _model(exact, bidirectional=True, seed=0):
    from speech_b200.models import CTC
    torch.manual_seed(seed)
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                       "rnn": {"dim": 64, "bidirectional": bidirectional, "layers": 2}}}
    m = CTC(80, S - 1, cfg).cuda()
    m.eval()
    return m


@pytest.mark.parametrize("exact", [False, True])
def test_ctc_infer_with_word_lm_equals_oracle(tmp_path, exact):
    rng = np.random.RandomState(1)
    m = _model(exact)
    m.set_eval()
    inputs = [rng.randn(n, 80).astype(np.float32) for n in (150, 120, 96)]
    labels = [rng.randint(0, S - 1, 9).tolist() for _ in range(3)]
    vocab = _words(rng, 30, 1, 3)
    lm, ref = _wlm(tmp_path, rng, 3, vocab, oov=-1.0)
    _, _, x_lens, _ = m.collate(inputs, labels)
    with torch.no_grad():
        probs = torch.softmax(m((inputs, labels)), 2).cpu().numpy()
    lens = x_lens.tolist() if exact else [probs.shape[1]] * 3
    preds = m.infer((inputs, labels), beam_size=8, lm=lm, lm_weight=1.0, insertion_bonus=0.5)
    for i, L in enumerate(lens):
        lab, _ = prefix_beam_search_wordlm(probs[i, :L], 8, BLANK, ref, 1.0, 0.5, -1.0)
        assert tuple(preds[i]) == tuple(lab), i


@pytest.mark.parametrize("K,order,g", [(4, 2, -1.5), (8, 3, NEG)])
def test_ctc_stream_with_word_lm(tmp_path, K, order, g):
    """after every push, partial equals the reference over the frames so far (the device's own
    log-probabilities of the same B utterances); the last equals infer's search bit for bit"""
    rng = np.random.RandomState(K + order)
    m = _model(True, bidirectional=False, seed=K)
    B = 3
    vocab = _words(rng, 30, 1, 3)
    lm, ref = _wlm(tmp_path, rng, order, vocab, oov=g)
    a, b = 0.8, 0.5
    kw = {"lm": lm, "lm_weight": a, "insertion_bonus": b}
    lens = rng.randint(40, 150, size=B).tolist()
    feats = [rng.randn(n, 80).astype(np.float32) for n in lens]
    x, _, x_lens, _ = m.collate(feats, [[0]] * B)
    elens = m.exact_lens(x_lens)
    with torch.no_grad():
        probs = m._forward_impl(x, elens, softmax=True)
    logp = torch.log(probs.float()).cpu().numpy().astype(np.float64)
    want = ctc_decoder.decode_batch(probs, beam_size=K, blank=m.blank, lens=elens,
                                    with_scores=True, **kw)
    for chunking in range(2):
        st = m.stream(B, beam_size=K, max_frames=200, **kw)
        pos = [0] * B
        while any(p < n for p, n in zip(pos, lens)):
            chunks = []
            for i in range(B):
                k = int(rng.choice([0, 1, 3, 8, 17, 40] if chunking else [5, 30]))
                chunks.append(feats[i][pos[i]:pos[i] + k])
                pos[i] = min(pos[i] + k, lens[i])
            st.push(chunks)
            got = st.partial(return_scores=True)
            for i, n in enumerate(st.frames):
                _same(got[i], prefix_beam_search_wordlm(logp[i, :n], K, m.blank, ref, a, b, g,
                                                        log_input=True))
        assert st.partial(return_scores=True) == want
