"""Reference LM-fused label-free transducer beam search (test infrastructure).

oracle/rnnt_search_ref.search with shallow fusion: extending hypothesis h by label k != blank
scores score + (row[k] + (lm_weight * lm(k | h) + insertion_bonus)), evaluated in that order in
float64; a blank emission scores score + row[blank], unchanged.  Merging, the tie order (a stable
descending sort) and the frame structure are the oracle's.  `lm` is anything with score(prefix, k)
(tests/ngram_ref.ArpaLM); its values are cached per context.

Also:
- best_by_enumeration: the most probable label sequence under the fused score, acoustic
  sequence_log_prob + lm_weight * sum of lm + insertion_bonus * length, for tiny shapes;
- shortlist_search: a host mirror of the device's shortlist route over fused float64 values
  (csrc/rnnt_search.cu + tsearch.cuh's ts_expand_shortlist): per frontier entry the kp best
  classes by (f desc, k asc) and beta, the K-way merge, and the flag of selections a left-out
  class could tie with.
"""
import math

import numpy as np

from oracle import rnnt_search_ref as ref


def _lse(a, b):
    m = max(a, b)
    if m == -math.inf:
        return -math.inf
    return m + math.log(math.exp(a - m) + math.exp(b - m))


class Fused:
    """fused rows f (float64, f[blank] = row[blank]) of hypotheses under one LM and weights"""

    def __init__(self, lm, lm_weight, insertion_bonus, blank):
        self.lm, self.a, self.b, self.blank = lm, lm_weight, insertion_bonus, blank
        self._lm = {}

    def lm_row(self, hyp, V):
        key = (self.lm.context(hyp) if hasattr(self.lm, "context") else tuple(hyp), V)
        if key not in self._lm:
            self._lm[key] = [0.0 if k == self.blank else self.lm.score(hyp, k) for k in range(V)]
        return self._lm[key]

    def __call__(self, row, hyp):
        V = len(row)
        lms = self.lm_row(hyp, V)
        f = np.empty(V, dtype=np.float64)
        for k in range(V):
            x = float(row[k])
            f[k] = x if k == self.blank else x + (self.a * lms[k] + self.b)
        return f


def search(row_fn, T, beam_size, blank, max_symbols_per_frame, max_len, lm, lm_weight,
           insertion_bonus):
    """-> (labels, fused float64 score, smallest score gap at any cut or between the final beam's
    first two)"""
    fused = Fused(lm, lm_weight, insertion_bonus, blank)
    S = max_symbols_per_frame
    beam = {(): 0.0}
    gaps = []
    for t in range(T):
        done = {}
        frontier = dict(beam)
        for level in range(S + 1):
            nxt = {}
            for hyp, score in frontier.items():
                row = row_fn(t, hyp)
                b = score + float(row[blank])
                done[hyp] = _lse(done[hyp], b) if hyp in done else b
                if level < S and len(hyp) < max_len:
                    f = fused(row, hyp)
                    for k in range(len(row)):
                        if k != blank:
                            nxt[hyp + (k,)] = score + float(f[k])
            if not nxt:
                break
            frontier = ref._take(nxt.items(), beam_size, gaps)
        beam = ref._take(done.items(), beam_size, gaps)
    best = list(beam.items())
    if len(best) > 1:
        gaps.append(best[0][1] - best[1][1])
    return list(best[0][0]), best[0][1], (min(gaps) if gaps else math.inf)


def best_by_enumeration(row_fn, T, V, blank, max_len, lm, lm_weight, insertion_bonus):
    """arg-max of sequence_log_prob + lm_weight * sum lm + insertion_bonus * length over every
    label sequence of at most max_len labels (tiny shapes only)"""
    import itertools
    symbols = [k for k in range(V) if k != blank]
    best, best_s = None, -math.inf
    for n in range(max_len + 1):
        for seq in itertools.product(symbols, repeat=n):
            s = ref.sequence_log_prob(row_fn, T, list(seq), blank)
            s += lm_weight * sum(lm.score(seq[:u], seq[u]) for u in range(n))
            s += insertion_bonus * n
            if s > best_s:
                best, best_s = list(seq), s
    return best, best_s


def shortlist(f, kp, blank):
    """(values, classes, beta) of one fused row, as sb_rnnt_search_lm_rows writes them"""
    k = np.array([c for c in range(f.shape[0]) if c != blank], dtype=np.int64)
    order = k[np.lexsort((k, -f[k]))]                   # f desc, class asc
    beta = float(f[order[kp]]) if order.shape[0] > kp else -math.inf
    return f[order[:kp]], order[:kp], beta


def _next_down(x):
    return float(np.nextafter(x, -np.inf))


def shortlist_search(row_fn, T, beam_size, blank, max_symbols_per_frame, max_len, lm, lm_weight,
                     insertion_bonus, kp):
    """-> (labels, fused score, number of flagged selections)"""
    fused = Fused(lm, lm_weight, insertion_bonus, blank)
    S = max_symbols_per_frame
    flags = 0
    beam = [((), 0.0)]
    for t in range(T):
        done = {}
        frontier = beam
        for level in range(S + 1):
            rows = [fused(row_fn(t, hyp), hyp) for hyp, _ in frontier]
            for (hyp, score), f in zip(frontier, rows):
                b = score + float(f[blank])
                done[hyp] = _lse(done[hyp], b) if hyp in done else b
            if level == S:
                break
            live = [i for i, (hyp, _) in enumerate(frontier)
                    if len(hyp) < max_len and rows[i].shape[0] > 1]
            if not live:
                break
            V = rows[0].shape[0]
            lists = {i: shortlist(rows[i], kp, blank) for i in live}
            used = {i: set() for i in live}
            taken = {i: 0 for i in live}

            def head(i):
                fs = frontier[i][1]
                if fs == -math.inf:                       # ties on every class: index order
                    c = taken[i]
                    if c >= V - 1:
                        return None
                    return -math.inf, (c if c < blank else c + 1), None
                vals, idx, _ = lists[i]
                free = [q for q in range(len(vals)) if q not in used[i]]
                if not free:
                    return None
                q0 = free[0]
                s = fs + float(vals[q0])
                best_k, best_q = int(idx[q0]), q0
                for q in range(q0 + 1, len(vals)):
                    if fs + float(vals[q]) != s:
                        break
                    if q not in used[i] and int(idx[q]) < best_k:
                        best_k, best_q = int(idx[q]), q
                return s, best_k, best_q

            nxt = []
            for _ in range(beam_size):
                best = None
                for i in live:
                    h = head(i)
                    if h is not None and (best is None or h[0] > best[0]):
                        best = (h[0], i, h[1], h[2])
                if best is None:
                    break
                s, i, k, q = best
                hyp, fs = frontier[i]
                if q is None:
                    taken[i] += 1
                else:
                    used[i].add(q)
                    vals, _, beta = lists[i]
                    x = float(vals[q])
                    if fs + beta == s and (x != beta or (beta != -math.inf and
                                                         fs + _next_down(beta) == s)):
                        flags += 1
                nxt.append((hyp + (k,), s))
            frontier = nxt
        beam = sorted(done.items(), key=lambda kv: -kv[1])[:beam_size]
    return list(beam[0][0]), beam[0][1], flags
