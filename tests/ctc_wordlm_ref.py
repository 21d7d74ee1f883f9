"""Reference word-LM CTC prefix beam search (test infrastructure, plain Python).

- WordArpa: an ARPA word LM read with tests/ngram_ref.read_arpa, its lexicon spelled in class
  ids, and the backoff lookup lm(w | h) accumulated as acc = 0, acc += bow per missed order from
  the longest context down, acc += prob (a word without a unigram ends with acc);
- prefix_beam_search_wordlm: tests/ctc_lm_ref.prefix_beam_search_lm with the word rule of
  include/speech_b200.h (SbWordLm): the word state of a prefix is recomputed from its labels, the
  LM term is added on the delimiter that ends a non-empty word, the OOV penalty where the partial
  word leaves the lexicon, and the end-of-utterance rule picks the result.
"""
import numpy as np

from ngram_ref import read_arpa
from oracle.ctc_decoder_ref import NEG_INF, _lse


class WordArpa:
    def __init__(self, path, spell, delimiter):
        """spell(word) -> class tuple, or None where the word cannot be spelled"""
        self.order, self.probs, self.bows = read_arpa(path)
        self.delim = delimiter
        self.word_of = {}
        for (w,) in (g for g in self.probs if len(g) == 1):
            if w in ("<s>", "</s>", "<unk>"):
                continue
            sp = spell(w)
            if sp is not None:
                self.word_of[sp] = w
        self.prefixes = {sp[:k] for sp in self.word_of for k in range(len(sp) + 1)}
        self._split = {}

    def logprob(self, h, w):
        acc = 0.0
        while True:
            if h + (w,) in self.probs:
                return acc + self.probs[h + (w,)]
            acc += self.bows.get(h, 0.0)
            if not h:
                return acc
            h = h[1:]

    def context(self, words):
        n = self.order - 1
        h = ("<s>",) + tuple(words)
        return h[max(0, len(h) - n):] if n else ()

    def split(self, prefix):
        """(completed words, partial word) of a label prefix; a word is its string or <unk>"""
        if prefix in self._split:
            return self._split[prefix]
        words, cur = [], []
        for c in prefix:
            if c == self.delim:
                if cur:
                    words.append(self.word_of.get(tuple(cur), "<unk>"))
                cur = []
            else:
                cur.append(c)
        self._split[prefix] = words, tuple(cur)
        return words, tuple(cur)

    def delim_term(self, words, partial, a, b, g):
        """(a * lm(w | words) + b) + g_i of the delimiter ending the non-empty `partial`"""
        w = self.word_of.get(partial, "<unk>")
        oov = g if (partial in self.prefixes and partial not in self.word_of) else 0.0
        return (a * self.logprob(self.context(words), w) + b) + oov

    def q(self, prefix, s, p, a, b, g):
        words, partial = self.split(prefix)
        if s == self.delim:
            return p if not partial else p + self.delim_term(words, partial, a, b, g)
        if partial in self.prefixes and partial + (s,) not in self.prefixes:
            return p + g
        return p

    def end_term(self, prefix, a, b, g):
        words, partial = self.split(prefix)
        if not partial:
            return 0.0 + a * self.logprob(self.context(words), "</s>")
        e = self.delim_term(words, partial, a, b, g)
        words = list(words) + [self.word_of.get(partial, "<unk>")]
        return e + a * self.logprob(self.context(words), "</s>")


def rescore(beam, lm, a, b, g):
    """(labels, score) of a final beam [(prefix, (p_b, p_nb))] under the end-of-utterance rule"""
    best, best_v = 0, None
    for i, (prefix, (pb, pnb)) in enumerate(beam):
        v = _lse(pb, pnb) + lm.end_term(prefix, a, b, g)
        if best_v is None or v > best_v:
            best, best_v = i, v
    return beam[best][0], -best_v


def prefix_beam_search_wordlm(probs, beam_size, blank, lm, a, b, g, log_input=False):
    """(labels, score) of the best prefix; probs (T, S), or log-probabilities with log_input"""
    probs = np.asarray(probs)
    T, S = probs.shape
    if log_input:
        logp = probs
    else:
        with np.errstate(divide="ignore"):
            logp = np.log(probs)
    beam = [((), (0.0, NEG_INF))]
    for t in range(T):
        cand = {}

        def slot(prefix):
            if prefix not in cand:
                cand[prefix] = [NEG_INF, NEG_INF]
            return cand[prefix]

        for s in range(S):
            p = float(logp[t, s])
            for prefix, (p_b, p_nb) in beam:
                if s == blank:
                    e = slot(prefix)
                    e[0] = _lse(e[0], p_b + p, p_nb + p)
                    continue
                q = lm.q(prefix, s, p, a, b, g)
                last = prefix[-1] if prefix else None
                e = slot(prefix + (s,))
                if s != last:
                    e[1] = _lse(e[1], p_b + q, p_nb + q)
                else:
                    e[1] = _lse(e[1], p_b + q)
                    k = slot(prefix)
                    k[1] = _lse(k[1], p_nb + p)
        ranked = sorted(cand.items(), key=lambda kv: _lse(*kv[1]), reverse=True)
        beam = [(k, (v[0], v[1])) for k, v in ranked[:beam_size]]
    return rescore(beam, lm, a, b, g)
