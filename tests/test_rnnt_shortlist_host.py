"""The shortlist beam search of the transducer (csrc/tdecode.cu, sb_rnnt_decode_static_shortlist)
and its producer (csrc/joint_vocab.cu, sb_rnnt_shortlist_rows), restated in numpy / Python floats,
against the CPU oracle oracle/decode_static_ref.py: label for label and score for score.

The restatement keeps the kernel's rules: per node the kp best non-blank classes by (float32 lp
desc, class asc) and beta, the next value; a K-way merge whose head is the smallest unconsumed class
of the current equal-score run; a hypothesis scored -inf takes the non-blank classes in index order;
a selection is flagged when a class left out of the list could tie with it; flagged lattices are
searched again from 64-entry lists."""
import math

import numpy as np
import pytest

from oracle import decode_static_ref as ref

RERUN = 64


def _lse(a, b):
    m = max(a, b)
    return m + math.log(math.exp(a - m) + math.exp(b - m))


def shortlist(row, kp, blank):
    """(values, classes, blank lp, beta) of one node, as sb_rnnt_shortlist_rows writes them."""
    row = np.asarray(row, dtype=np.float32)
    k = np.array([c for c in range(row.shape[0]) if c != blank], dtype=np.int64)
    order = k[np.lexsort((k, -row[k]))]                 # lp desc, class asc
    beta = float(row[order[kp]]) if order.shape[0] > kp else -math.inf
    return row[order[:kp]], order[:kp], float(row[blank]), beta


def _next_down(x):
    return float(np.nextafter(np.float32(x), np.float32(-np.inf)))


def shortlist_search(lp, beam_size, blank, kp):
    """-> (labels, score, number of flagged selections)"""
    lat = np.asarray(lp, dtype=np.float32)
    T, U, V = lat.shape
    lists = {}

    def node(t, u):
        if (t, u) not in lists:
            lists[(t, u)] = shortlist(lat[t, u], kp, blank)
        return lists[(t, u)]

    flags = 0
    beam = [((), 0.0)]
    for t in range(T):
        done = {}
        frontier = beam
        for _ in range(U):
            for hyp, score in frontier:
                u = len(hyp)
                if u >= U:
                    continue
                b = score + node(t, u)[2]
                done[hyp] = _lse(done[hyp], b) if hyp in done else b
            live = [i for i, (hyp, _) in enumerate(frontier) if len(hyp) + 1 < U and V > 1]
            if not live:
                break
            used = {i: set() for i in live}
            taken = {i: 0 for i in live}

            def head(i):
                hyp, fs = frontier[i]
                if fs == -math.inf:                       # ties on every class: index order
                    c = taken[i]
                    if c >= V - 1:
                        return None
                    return -math.inf, (c if c < blank else c + 1), None
                vals, idx, _, _ = node(t, len(hyp))
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
                    vals, _, _, beta = node(t, len(hyp))
                    x = float(vals[q])
                    if fs + beta == s and (x != beta or (beta != -math.inf and
                                                         fs + _next_down(beta) == s)):
                        flags += 1
                nxt.append((hyp + (k,), s))
            frontier = nxt
        beam = sorted(done.items(), key=lambda kv: -kv[1])[:beam_size]
    best = max(beam, key=lambda kv: kv[1])
    return list(best[0]), best[1], flags


def decode(lp, beam_size, blank):
    """the host side of the route: kp = beam_size, flagged lattices again at kp = 64"""
    labels, score, flags = shortlist_search(lp, beam_size, blank, beam_size)
    if flags:
        labels, score, flags = shortlist_search(lp, beam_size, blank, RERUN)
        assert not flags
    return labels, score


def _lattice(rng, kind, T, U, V):
    if kind == "quantised":                 # many float32 ties, inside and across nodes
        return -rng.randint(1, 4, size=(T, U, V)).astype(np.float32)
    x = rng.randn(T, U, V) * 2.0
    x = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    if kind == "neginf":                    # -inf entries are live candidates
        x[rng.rand(T, U, V) < 0.4] = -np.inf
    return x


@pytest.mark.parametrize("kind", ["random", "quantised", "neginf"])
def test_shortlist_search_equals_oracle(kind):
    rng = np.random.RandomState({"random": 0, "quantised": 1, "neginf": 2}[kind])
    for n in range(110):
        T, U = rng.randint(1, 7), rng.randint(1, 6)       # ragged lattices
        V = rng.randint(2, 41)
        K = rng.randint(1, 9)
        blank = (0, V - 1)[n % 2]                          # blank first and last
        lat = _lattice(rng, kind, T, U, V)
        want, wscore = ref.decode_static(lat, K, blank)
        got, gscore, flags = shortlist_search(lat, K, blank, K)
        assert flags == 0, (n, kind)
        assert got == want, (n, kind, T, U, V, K, blank)
        # (merging two -inf scores gives NaN, in the oracle as in the kernels)
        assert gscore == wscore or (math.isnan(gscore) and math.isnan(wscore)), (n, kind)


def test_shortlist_is_the_head_of_the_stable_order():
    row = np.array([-1.0, -2.0, -1.0, -np.inf, -0.5, -1.0, -np.inf], dtype=np.float32)
    vals, idx, blp, beta = shortlist(row, 3, 4)
    assert idx.tolist() == [0, 2, 5] and vals.tolist() == [-1.0, -1.0, -1.0]
    assert blp == -0.5 and beta == -2.0
    vals, idx, _, beta = shortlist(row, 5, 4)
    assert idx.tolist() == [0, 2, 5, 1, 3] and beta == -np.inf
    vals, idx, _, beta = shortlist(row, 6, 4)
    assert idx.tolist() == [0, 2, 5, 1, 3, 6] and beta == -np.inf      # nothing left out


def tie_lattice(V=13000):
    """A lattice whose beam hypothesis scores -2^40 after the first frame: at that magnitude
    float64 ulps are 2^-12, so the labels 0 (lp -1 - 2^-23) and 5, 7 (lp -1) tie on score and the
    full search takes class 0 first - which 2-entry lists ([5, 7], beta = lp of class 0) cannot
    show.  Blank is the last class."""
    blank = V - 1
    lat = np.full((2, 2, V), -np.inf, dtype=np.float32)
    lat[0, 0, blank] = -2.0 ** 40
    lat[0, 1, blank] = 0.0
    lat[1, 0, :blank] = -50.0
    lat[1, 0, 0] = np.nextafter(np.float32(-1.0), np.float32(-2.0))
    lat[1, 0, 5] = -1.0
    lat[1, 0, 7] = -1.0
    lat[1, 0, blank] = -10.0
    lat[1, 1, blank] = 0.0
    return lat, blank


def test_merged_scores_raise_the_flag_and_the_rerun_equals_the_oracle():
    lat, blank = tie_lattice()
    assert float(lat[1, 0, 0]) != -1.0
    want, wscore = ref.decode_static(lat, 2, blank)
    assert want == [0]
    got, gscore, flags = shortlist_search(lat, 2, blank, 2)
    assert flags > 0 and got == [5]                   # the 2-entry lists would answer wrongly
    got, gscore, flags = shortlist_search(lat, 2, blank, RERUN)
    assert flags == 0 and got == want and gscore == wscore
    assert decode(lat, 2, blank) == (want, wscore)
