"""Reference n-gram LM for the LM-fused CTC search tests (test infrastructure, plain Python).

- read_arpa: an ARPA file into plain dicts of word tuples, values in natural log (v10 * log(10));
- ArpaLM.score: the backoff lookup lm(s | prefix) over class ids, with the context and <unk>
  rules of speech_b200.lm, accumulated as acc = 0, acc += bow per missed order from the longest
  context down, acc += prob;
- KneserNey: interpolated Kneser-Ney probabilities computed straight from the counts, recursively,
  without the backoff form, to check NGramLM.train.
"""
import math
from collections import Counter

LN10 = math.log(10.0)


def read_arpa(path):
    """-> (order, {word tuple: natural-log prob}, {word tuple: natural-log backoff})"""
    probs, bows = {}, {}
    order = 0
    section = None
    for line in open(path, encoding="utf-8"):
        f = line.split()
        if not f:
            continue
        if f[0].startswith("\\") and f[0].endswith("-grams:"):
            section = int(f[0][1:-7])
            order = max(order, section)
            continue
        if f[0] in ("\\data\\", "\\end\\") or f[0] == "ngram":
            section = None
            continue
        if section is None:
            continue
        g = tuple(f[1:section + 1])
        probs[g] = float(f[0]) * LN10
        if len(f) == section + 2:
            bows[g] = float(f[section + 1]) * LN10
    return order, probs, bows


class ArpaLM:
    def __init__(self, path, symbols, blank):
        self.order, self.probs, self.bows = read_arpa(path)
        self.words = {c: s for c, s in enumerate(symbols) if c != blank}

    def word(self, c):
        w = self.words[c]
        return w if (w,) in self.probs else "<unk>"

    def context(self, prefix):
        """the last order-1 tokens of <s> prefix"""
        n = self.order - 1
        h = ("<s>",) + tuple(self.word(c) for c in prefix)
        return h[max(0, len(h) - n):] if n else ()

    def logprob(self, h, w):
        acc = 0.0
        while True:
            if h + (w,) in self.probs:
                return acc + self.probs[h + (w,)]
            acc += self.bows.get(h, 0.0)
            h = h[1:]

    def score(self, prefix, s):
        """lm(s | prefix), s a class id or '</s>'"""
        return self.logprob(self.context(prefix), "</s>" if s == "</s>" else self.word(s))


class KneserNey:
    """Interpolated Kneser-Ney over class ids, from the counts (tokens: classes, 'B' = <s>,
    'E' = </s>)."""

    def __init__(self, sequences, order, num_classes, blank):
        self.N, self.C = order, num_classes
        self.vocab = [c for c in range(num_classes) if c != blank] + ["E"]
        grams = Counter()
        for seq in sequences:
            w = ["B"] + list(seq) + ["E"]
            for n in range(1, order + 1):
                for j in range(len(w) - n + 1):
                    grams[tuple(w[j:j + n])] += 1
        self.raw = grams
        self.count = {}
        for g, c in grams.items():
            n = len(g)
            if g == ("B",):
                continue
            if n == order or g[0] == "B":
                self.count[g] = c
            else:
                self.count[g] = sum(1 for x in grams if len(x) == n + 1 and x[1:] == g)
        self.D = {}
        for n in range(1, order + 1):
            cs = [c for g, c in self.count.items() if len(g) == n]
            n1, n2 = cs.count(1), cs.count(2)
            d = n1 / (n1 + 2 * n2) if n1 + 2 * n2 else 0.0
            self.D[n] = d if 0 < d < 1 else 0.5

    def prob(self, h, w):
        """P(w | h), len(h) <= order - 1"""
        n = len(h) + 1
        lower = self.prob(h[1:], w) if h else 1.0 / self.C
        ext = {g: c for g, c in self.count.items() if len(g) == n and g[:-1] == tuple(h)}
        total = sum(ext.values())
        if total == 0:
            return lower
        D = self.D[n]
        return (max(ext.get(tuple(h) + (w,), 0) - D, 0) / total
                + D * len(ext) / total * lower)
