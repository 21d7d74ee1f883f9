"""float64 references of the Viterbi (forced) alignments of sb_ctc_viterbi and sb_rnnt_viterbi, with
their tie rules, and brute-force enumerations of every alignment that the host tests hold them to.

CTC: states of l' = (blank, y1, blank, ..., yL, blank); on equal scores the predecessor s wins
over s-1 and s-1 over s-2, and the path ends in S-1 rather than S-2.
Transducer: on equal scores the blank arc into (t, u) wins over the label arc."""
import itertools

import numpy as np

NEG_INF = -np.inf


def log_softmax(x, axis=-1):
    x = np.asarray(x, np.float64)
    m = x.max(axis=axis, keepdims=True)
    return x - (m + np.log(np.exp(x - m).sum(axis=axis, keepdims=True)))


def ctc_viterbi(lp, labels, blank):
    """lp (T, V) float64 log-probabilities -> (path (T,) int: label index or -1 for blank, score);
    (None, -inf) where no alignment exists.  T = 0 aligns only the empty transcript (score 0)."""
    T = lp.shape[0]
    L = len(labels)
    S = 2 * L + 1
    if T == 0:
        return (np.zeros(0, np.int64), 0.0) if L == 0 else (None, NEG_INF)
    cls = np.full(S, blank, np.int64)
    cls[1::2] = labels
    skip = np.zeros(S, bool)
    for s in range(3, S, 2):
        skip[s] = cls[s] != blank and cls[s] != cls[s - 2]
    d = np.full((T, S), NEG_INF)
    bp = np.zeros((T, S), np.int64)
    d[0, 0] = lp[0, blank]
    if S > 1:
        d[0, 1] = lp[0, cls[1]]
    for t in range(1, T):
        prev = np.concatenate([[NEG_INF, NEG_INF], d[t - 1]])
        cand = np.stack([prev[2:], prev[1:-1], np.where(skip, prev[:-2], NEG_INF)])
        bp[t] = np.argmax(cand, axis=0)            # the first of equal maxima: s, then s-1, s-2
        d[t] = cand[bp[t], np.arange(S)] + lp[t, cls]
    end = S - 1
    if S >= 2 and d[T - 1, S - 2] > d[T - 1, S - 1]:
        end = S - 2
    score = d[T - 1, end]
    if score == NEG_INF:
        return None, NEG_INF
    path = np.empty(T, np.int64)
    s = end
    for t in range(T - 1, -1, -1):
        path[t] = (s - 1) // 2 if s & 1 else -1
        s -= bp[t, s]
    return path, float(score)


def ctc_rescore(lp, labels, blank, path):
    """float64 log-probability of a frame-to-label path (path[t] = label index or -1)"""
    return float(sum(lp[t, blank if j < 0 else labels[j]] for t, j in enumerate(path)))


def ctc_path_errors(path, labels, T_b):
    """why `path` (length >= T_b, -2 past T_b) is not a CTC alignment of `labels`, or None"""
    path = list(path)
    if any(j != -2 for j in path[T_b:]):
        return "frames past T_b are not -2"
    seq = path[:T_b]
    prev = -1
    for t, j in enumerate(seq):
        if j < -1 or j >= len(labels):
            return "label index out of range at frame %d" % t
        if j >= 0:
            if j < prev or j > prev + 1:
                return "not monotone at frame %d" % t
            # a label equal to the one before must be separated by a blank
            if j == prev + 1 and j > 0 and t > 0 and seq[t - 1] == j - 1 and labels[j] == labels[j - 1]:
                return "repeat without a blank at frame %d" % t
            prev = j
    if prev != len(labels) - 1:
        return "not every label is covered"
    return None


def ctc_enumerate(lp, labels, blank):
    """every frame-symbol sequence over V classes that collapses to `labels`, as (score, states):
    score summed over frames in order, states the sequence's l' indices"""
    T, V = lp.shape
    out = []
    for pi in itertools.product(range(V), repeat=T):
        j, prev, states, seq = -1, None, [], []
        for c in pi:
            if c == blank:
                states.append(2 * (j + 1))
            elif c == prev:
                states.append(2 * j + 1)
            else:
                j += 1
                seq.append(c)
                states.append(2 * j + 1)
            prev = c
        if seq != list(labels):
            continue
        score = 0.0
        for t, c in enumerate(pi):
            score = score + lp[t, c]
        out.append((score, states))
    return out


def ctc_brute_force(lp, labels, blank):
    """best path by enumeration; among equal scores the tie rule is the largest state sequence
    read backwards from the last frame -> (path, score) or (None, -inf)"""
    paths = ctc_enumerate(lp, labels, blank)
    if not paths:
        return None, NEG_INF
    score, states = max(paths, key=lambda p: (p[0], p[1][::-1]))
    return np.array([(s - 1) // 2 if s & 1 else -1 for s in states]), score


def rnnt_viterbi(blank_lp, label_lp, T, U):
    """blank_lp / label_lp (>= T, >= U+1) float64 node values: blank(t, u) and label(t, u) of arc
    u -> u+1 -> (frames (U,) emission frame of each label, score); (None, -inf) for T = 0."""
    if T == 0:
        return None, NEG_INF
    a = np.full((T, U + 1), NEG_INF)
    lab = np.zeros((T, U + 1), bool)
    for d in range(T + U):
        u = np.arange(max(0, d - T + 1), min(U, d) + 1)
        t = d - u
        if d == 0:
            a[0, 0] = 0.0
            continue
        bl = np.where(t > 0, a[np.maximum(t - 1, 0), u] + blank_lp[np.maximum(t - 1, 0), u], NEG_INF)
        lb = np.where(u > 0, a[t, np.maximum(u - 1, 0)] + label_lp[t, np.maximum(u - 1, 0)], NEG_INF)
        lab[t, u] = lb > bl                          # ties take the blank arc
        a[t, u] = np.where(lab[t, u], lb, bl)
    score = a[T - 1, U] + blank_lp[T - 1, U]
    frames = np.full(U, -1, np.int64)
    t, u = T - 1, U
    while t > 0 or u > 0:
        if lab[t, u]:
            u -= 1
            frames[u] = t
        else:
            t -= 1
    return frames, float(score)


def rnnt_rescore(blank_lp, label_lp, T, frames):
    """float64 log-probability of the path that emits label u at frames[u] (non-decreasing)"""
    score, u = 0.0, 0
    for t in range(T):
        while u < len(frames) and frames[u] == t:
            score = score + label_lp[t, u]
            u += 1
        score = score + blank_lp[t, u]
    return float(score)


def rnnt_brute_force(blank_lp, label_lp, T, U):
    """best path by enumeration of every arrangement of U label arcs among the frames; among
    equal scores the tie rule is the smallest arc sequence (label = 1) read backwards from the end
    -> (frames, score)"""
    if T == 0:
        return None, NEG_INF
    best = None
    for pos in itertools.combinations(range(T - 1 + U), U):
        arcs = np.zeros(T - 1 + U, np.int64)
        arcs[list(pos)] = 1
        t = u = 0
        score = 0.0
        frames = []
        for k in arcs:
            if k:
                score = score + label_lp[t, u]
                frames.append(t)
                u += 1
            else:
                score = score + blank_lp[t, u]
                t += 1
        score = score + blank_lp[t, u]
        key = (score, tuple(-arcs[::-1]))
        if best is None or key > best[0]:
            best = (key, np.array(frames, np.int64), score)
    return best[1], best[2]
