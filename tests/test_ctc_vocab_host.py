"""Host checks (no GPU) of the two reductions behind large-vocabulary CTC:

- the compact loss problem of csrc/ctc.cu: each frame reduced to (blank, distinct label classes,
  log-sum-exp of the rest) gives the full problem's costs, and the expanded gradient (softmax
  outside the label set, compact gradient inside) gives the full gradient (float64 torch);
- the shortlist beam search of csrc/decode.cu, restated in the reference's own arithmetic: scoring
  only each frame's 2K+1 most probable non-blank symbols plus every entry's last symbol, with the
  per-frame bound check and its fall-back to a full scan, returns the oracle's labels and scores
  exactly.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ctc_decoder_ref

NEG_INF = -float("inf")


# ---------------------------------------------------------------------------------------------
# loss: compact problem
# ---------------------------------------------------------------------------------------------
def _ctc(acts, labels, alen, llen, blank):
    """float64 costs (inf where infeasible) and d(sum of finite costs)/d acts"""
    a = torch.from_numpy(acts).double().requires_grad_(True)
    lp = torch.log_softmax(a, 2).transpose(0, 1)
    args = (torch.from_numpy(labels).long(), torch.from_numpy(alen).long(),
            torch.from_numpy(llen).long())
    costs = F.ctc_loss(lp, *args, blank=blank, reduction="none").detach().numpy()
    F.ctc_loss(lp, *args, blank=blank, reduction="sum", zero_infinity=True).backward()
    return costs, a.grad.numpy()


def _compact(acts, labels, llen, blank):
    """the compact rows, remapped labels and column classes of csrc/ctc.cu (float64)"""
    B, T, V = acts.shape
    Vc = int(llen.max()) + 2
    out = np.full((B, T, Vc), NEG_INF)
    lab_c, cols = [], []
    off = 0
    for b in range(B):
        lab = labels[off:off + llen[b]]
        off += llen[b]
        cls = [blank]
        for c in lab:
            if c != blank and c not in cls:
                cls.append(int(c))
        lab_c += [cls.index(int(c)) for c in lab]
        rest = np.ones(V, bool)
        rest[cls] = False
        x = acts[b].astype(np.float64)
        out[b, :, :len(cls)] = x[:, cls]
        if rest.any():
            m = x[:, rest].max(1)
            out[b, :, len(cls)] = m + np.log(np.exp(x[:, rest] - m[:, None]).sum(1))
        cols.append(cls)
    return out, np.array(lab_c, np.int64), cols


def _expand(acts, g_c, cols, costs, alen):
    B, T, V = acts.shape
    x = acts.astype(np.float64)
    m = x.max(2, keepdims=True)
    soft = np.exp(x - m) / np.exp(x - m).sum(2, keepdims=True)
    g = soft.copy()
    for b in range(B):
        g[b][:, cols[b]] = g_c[b][:, :len(cols[b])]
        if not np.isfinite(costs[b]):
            g[b] = 0.0
        g[b, alen[b]:] = 0.0
    return g


@pytest.mark.parametrize("case", ["repeats", "label_is_blank", "empty", "infeasible", "ragged",
                                  "covers_all"])
def test_compact_loss_equals_full(case):
    rng = np.random.RandomState(len(case) * 31 + ord(case[0]))
    B, T, V = 4, 20, 37
    blank = V - 1
    llen = np.array([6, 9, 4, 7], np.int64)
    alen = np.full(B, T, np.int64)
    labels = [rng.randint(0, V - 1, n) for n in llen]
    if case == "repeats":
        labels[0] = np.array([3, 3, 3, 5, 5, 3])
    if case == "label_is_blank":
        labels[1][2] = blank
    if case == "empty":
        llen[2] = 0
        labels[2] = labels[2][:0]
    if case == "infeasible":
        alen[3] = 5
    if case == "ragged":
        alen[:] = [20, 13, 7, 17]
    if case == "covers_all":
        V, blank = 8, 7
        llen[0] = 9
        labels = [np.array([0, 1, 2, 3, 4, 5, 6, 6, 1])] + [rng.randint(0, 7, n) for n in llen[1:]]
    acts = (rng.randn(B, T, V) * 2).astype(np.float32)
    flat = np.concatenate(labels).astype(np.int64)
    c_full, g_full = _ctc(acts, flat, alen, llen, blank)
    a_c, lab_c, cols = _compact(acts, flat, llen, blank)
    if case == "covers_all":
        assert len(cols[0]) == V and np.all(a_c[0, :, V] == NEG_INF)
    # torch's CTC backward turns -inf log-probabilities into NaN; -1e30 has the same softmax
    # (exp underflows to exactly 0), so it stands in for the empty columns here
    c_c, g_c = _ctc(np.where(a_c == NEG_INF, -1e30, a_c), lab_c, alen, llen, 0)
    fin = np.isfinite(c_full)
    assert np.array_equal(np.isfinite(c_c), fin)
    if case == "infeasible":
        assert not fin[3]
    np.testing.assert_allclose(c_c[fin], c_full[fin], rtol=1e-10)
    g = _expand(acts, g_c, cols, c_c, alen)
    np.testing.assert_allclose(g, g_full, rtol=1e-10, atol=1e-12)


# ---------------------------------------------------------------------------------------------
# decode: shortlist search
# ---------------------------------------------------------------------------------------------
_lse = ctc_decoder_ref._lse


def _shortlist_search(probs, K, blank):
    """the oracle's search (same arithmetic and first-touch order), scoring per frame only the
    shortlisted symbols, the blank and every entry's last symbol, with csrc/decode.cu's check"""
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
                    last = prefix[-1] if prefix else None
                    e = slot(prefix + (s,))
                    if s != last:
                        e[1] = _lse(e[1], p_b + p, p_nb + p)
                    else:
                        e[1] = _lse(e[1], p_b + p)
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
        U = max(_lse(pb + pmin, pnb + pmin) for _, (pb, pnb) in beam)
        kth = _lse(*sel[-1][1]) if len(sel) == K else NEG_INF
        ok = kth != NEG_INF and (U == NEG_INF or kth > U + 1e-12 * (1 + abs(U)))
        if not ok:
            rescans += 1
            sel = step(range(S))
        beam = sel
    best = beam[0]
    return best[0], -_lse(*best[1]), rescans


def _lattice(rng, kind, T, S):
    x = rng.randn(T, S) * 2.5
    if kind == "quantised":
        p = np.exp(x) / np.exp(x).sum(1, keepdims=True)
        p = np.round(p * 16) / 16                       # many exact ties and zeros
        p[p.sum(1) == 0, 0] = 1.0
        return p.astype(np.float32)
    if kind == "zeros":
        x[rng.rand(T, S) < 0.7] = -np.inf               # many zero probabilities
        x[:, S - 1] = np.maximum(x[:, S - 1], 0.0)
    p = np.exp(x - x.max(1, keepdims=True))
    return (p / p.sum(1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("K", [1, 2, 8, 10])
@pytest.mark.parametrize("kind", ["random", "quantised", "zeros"])
def test_shortlist_search_equals_oracle(K, kind):
    rng = np.random.RandomState(K * 7 + len(kind))
    rescans = 0
    for _ in range(25):
        T = rng.randint(4, 12)
        S = rng.randint(2 * K + 3, 2 * K + 16)
        blank = int(rng.choice([0, S - 1]))
        probs = _lattice(rng, kind, T, S)
        lab, sc, n = _shortlist_search(probs, K, blank)
        ref_lab, ref_sc = ctc_decoder_ref.prefix_beam_search(probs, K, blank)
        assert tuple(lab) == tuple(ref_lab)
        assert sc == ref_sc or (math.isinf(sc) and math.isinf(ref_sc))
        rescans += n
    if kind != "random" and K >= 8:
        assert rescans > 0                              # the fall-back is exercised
