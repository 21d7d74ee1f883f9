"""Reference joint CTC/attention decoding (test infrastructure).

The CTC prefix scorer of Watanabe et al. 2017 ("Hybrid CTC/Attention Architecture for End-to-End
Speech Recognition", Algorithm 2) in float64 numpy, in the log domain, over float32 CTC
log-probabilities y (T, C) with blank C - 1; brute-force enumeration of CTC paths to hold it to;
and the attention beam search loop (seq2seq.py:180-227 with the py3 list() fix) restated over
decode_step with the CTC pre-beam and candidate value of csrc/s2s_ctc.cu:
    P(c) = (1 - w) logp[c] (+ (alpha lm(c | h) + beta_c)),   value = (A + P(c)) + w psi(h + c).
"""
import itertools
import math

import numpy as np
import torch

NEG = -math.inf


def lse(a, b):
    """max + log1p(exp(min - max)) elementwise, -inf where both are -inf"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    mx, mn = np.maximum(a, b), np.minimum(a, b)
    with np.errstate(invalid="ignore"):
        out = mx + np.log1p(np.exp(mn - mx))
    return np.where(mx == NEG, NEG, out)


def root_vectors(y, Tb):
    """(gn, gb) of the empty hypothesis over frames 0..Tb-1"""
    gb = np.cumsum(y[:Tb, -1].astype(np.float64))
    return np.full(Tb, NEG), gb


def extend(y, gn_h, gb_h, c, last):
    """(gn, gb) of h + c from those of h; last: h's last label, None at the root"""
    Tb = len(gn_h)
    yd = y[:Tb].astype(np.float64)
    gn, gb = np.full(Tb, NEG), np.full(Tb, NEG)
    gn[0] = yd[0, c] if last is None else NEG
    for t in range(1, Tb):
        phi = gb_h[t - 1] if c == last else lse(gb_h[t - 1], gn_h[t - 1])
        gn[t] = lse(gn[t - 1], phi) + yd[t, c]
        gb[t] = lse(gb[t - 1], gn[t - 1]) + yd[t, -1]
    return gn, gb


def prefix_scores(y, gn_h, gb_h, last, classes, end):
    """psi(h + c) for each c of classes; c == end: the full CTC probability of h"""
    Tb = len(gn_h)
    yd = y[:Tb].astype(np.float64)
    out = []
    for c in classes:
        if c == end:
            out.append(float(lse(gn_h[Tb - 1], gb_h[Tb - 1])))
            continue
        gn = yd[0, c] if last is None else NEG
        gb = NEG
        psi = gn
        for t in range(1, Tb):
            phi = gb_h[t - 1] if c == last else float(lse(gb_h[t - 1], gn_h[t - 1]))
            ngn = float(lse(gn, phi)) + yd[t, c]
            gb = float(lse(gb, gn)) + yd[t, -1]
            psi = float(lse(psi, phi + yd[t, c]))
            gn = ngn
        out.append(psi)
    return out


def vectors_of(y, Tb, hyp):
    """(gn, gb) of a label sequence"""
    gn, gb = root_vectors(y, Tb)
    last = None
    for c in hyp:
        gn, gb = extend(y, gn, gb, c, last)
        last = c
    return gn, gb


def brute_force(y, h, end_only=False):
    """log sum of P(path) over the CTC paths of len(y) frames (blank C - 1) whose collapse starts
    with h (end_only: equals h)"""
    T, C = y.shape
    yd = y.astype(np.float64)
    tot = NEG
    for path in itertools.product(range(C), repeat=T):
        col, prev = [], None
        for s in path:
            if s != C - 1 and s != prev:
                col.append(s)
            prev = s
        ok = col == list(h) if end_only else col[:len(h)] == list(h)
        if ok:
            tot = float(lse(tot, sum(yd[t, s] for t, s in enumerate(path))))
    return tot


def beam_search_ctc(m, x_enc, y, Tb, start_tok, end_tok, beam_size, max_len, ctc_weight, prebeam,
                    lm=None, lm_weight=0.0, insertion_bonus=0.0, lens=None):
    """one utterance (x_enc (1, T, H), y (T, C) float32 numpy) -> (token tuple, float64 score)"""
    w = float(ctc_weight)
    ydev = torch.zeros(1, 1, dtype=torch.int64, device=x_enc.device)
    gn0, gb0 = root_vectors(y, Tb)
    # (hyp, A, S, decoder state, gn, gb)
    beam = [((start_tok,), 0.0, 0.0, None, gn0, gb0)]
    complete = []
    for _ in range(max_len):
        new_beam = []
        for hyp, A, S, state, gn, gb in beam:
            ydev[0] = hyp[-1]
            out, state = m.decode_step(x_enc, ydev, state=state, softmax=True, lens=lens)
            logp = out.cpu().numpy().squeeze(0).tolist()
            P = []
            for c, p in enumerate(logp):
                v = (1.0 - w) * p
                if lm is not None:
                    l = lm.score(hyp[1:], c)
                    v = v + (lm_weight * l + (0.0 if c == end_tok else insertion_bonus))
                P.append(v)
            top = sorted(sorted(range(len(P)), key=lambda c: P[c], reverse=True)[:prebeam])
            last = None if len(hyp) == 1 else hyp[-1]
            psi = prefix_scores(y, gn, gb, last, top, end_tok)
            for c, ps in zip(top, psi):
                a = A + P[c]
                new_beam.append((hyp + (c,), a + w * ps, a, state, gn, gb, last))
        new_beam = sorted(new_beam, key=lambda h: h[1], reverse=True)
        for cand in new_beam[:beam_size]:
            if cand[0][-1] == end_tok:
                complete.append(cand)
        live = [h for h in new_beam if h[0][-1] != end_tok][:beam_size]
        beam = []
        for hyp, S, a, state, gn, gb, last in live:
            ngn, ngb = extend(y, gn, gb, hyp[-1], last)
            beam.append((hyp, a, S, state, ngn, ngb))
        if len(beam) == 0:
            break
        if sum(h[1] > beam[0][2] for h in complete) >= beam_size:
            break
    complete = sorted(complete, key=lambda h: h[1], reverse=True)
    if len(complete) == 0:
        return beam[0][0], beam[0][2]
    return complete[0][0], complete[0][1]
