"""CPU oracle of the label-free transducer beam search (TEST INFRASTRUCTURE - never imported by
speech_b200/).

`search` is decode_static_ref.decode_static with three changes: the row of hypothesis h at frame t
comes from row_fn(t, h) instead of lat[t, len(h)]; a frame runs S + 1 rounds (S =
max_symbols_per_frame) and extends on the first S only; a hypothesis with max_len labels is not
extended.  Merging, tie order (a stable descending sort) and float64 scores are decode_static's, so
with row_fn = lat[t, len(h)] and S = max_len = U - 1 it IS decode_static.

`LabelFreeRows` restates Transducer's rows for one hypothesis (speech/models/transducer_model.py
:59-76 on the hypothesis's own labels) in float64, rounding to bf16 exactly the operands the GPU
rounds: the fc1 GEMM of the prediction rows (both operands), z = relu(fx + fy) and fc2's weight.
The prediction GRU runs in fp32 on the GPU and unrounded here.  fx is the GPU's.

`best_by_enumeration` pins `search`: with S >= max_len and a beam that holds every hypothesis the
search is exact, so it returns the most probable label sequence, computed here by the forward
algorithm over the rows of each sequence's own prefixes.
"""
import itertools
import math

import numpy as np
import torch


def _lse(a, b):
    m = max(a, b)
    if m == -math.inf:
        return -math.inf
    return m + math.log(math.exp(a - m) + math.exp(b - m))


def _take(items, k, gaps):
    """stable descending sort, first k; records the score gap at the cut"""
    order = sorted(items, key=lambda kv: -kv[1])
    if len(order) > k:
        gaps.append(order[k - 1][1] - order[k][1])
    return dict(order[:k])


def search(row_fn, T, beam_size, blank, max_symbols_per_frame, max_len):
    """-> (labels, float64 log-probability, smallest score gap at any cut of a selection or between
    the final beam's first two)"""
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
                    for k in range(len(row)):
                        if k != blank:
                            nxt[hyp + (k,)] = score + float(row[k])
            if not nxt:
                break
            frontier = _take(nxt.items(), beam_size, gaps)
        beam = _take(done.items(), beam_size, gaps)
    best = list(beam.items())
    if len(best) > 1:
        gaps.append(best[0][1] - best[1][1])
    return list(best[0][0]), best[0][1], (min(gaps) if gaps else math.inf)


def static_rows(lat):
    """row_fn of a static (T, U, V) lattice: lat[t, len(h)]"""
    lat = np.asarray(lat, dtype=np.float32)
    return lambda t, hyp: lat[t, len(hyp)]


def _bf16(x):
    return torch.as_tensor(x, dtype=torch.float64).to(torch.bfloat16).to(torch.float64)


class LabelFreeRows:
    """row_fn(t, hyp) of one utterance: model (a Transducer, its fp32 weights read once), fx the
    GPU's fc1(encoder) rows (T', Hj) of that utterance."""

    def __init__(self, model, fx):
        d = lambda p: p.detach().cpu().double()
        rnn = model.dec_rnn
        self.emb = d(model.embedding.weight)
        self.gru = [tuple(d(getattr(rnn, "%s_l%d" % (n, l)))
                          for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
                    for l in range(rnn.num_layers)]
        H = model.fc1.fc.out_features
        self.fx = torch.as_tensor(fx).detach().cpu().double()
        Hj = self.fx.shape[1]
        w1 = torch.zeros(Hj, H, dtype=torch.float64)
        w1[:H] = d(model.fc1.fc.weight)
        self.w1 = _bf16(w1)
        self.b1 = torch.zeros(Hj, dtype=torch.float64)
        self.b1[:H] = d(model.fc1.fc.bias)
        w2 = torch.zeros(model.fc2.fc.out_features, Hj, dtype=torch.float64)
        w2[:, :H] = d(model.fc2.fc.weight)
        self.w2 = _bf16(w2)
        self.b2 = d(model.fc2.fc.bias)
        self._fy = {}

    def _gru(self, x, h, w):
        w_ih, w_hh, b_ih, b_hh = w
        gi = w_ih @ x + b_ih
        gh = w_hh @ h + b_hh
        Hh = h.shape[0]
        r = torch.sigmoid(gi[:Hh] + gh[:Hh])
        z = torch.sigmoid(gi[Hh:2 * Hh] + gh[Hh:2 * Hh])
        n = torch.tanh(gi[2 * Hh:] + r * gh[2 * Hh:])
        return (1 - z) * n + z * h

    def _states(self, hyp):
        """per-layer GRU states after the start vector and the labels of hyp"""
        if hyp in self._fy:
            return self._fy[hyp][0]
        if not hyp:
            hs = [torch.zeros(w[1].shape[1], dtype=torch.float64) for w in self.gru]
            x = torch.zeros(self.emb.shape[1], dtype=torch.float64)
        else:
            hs = self._states(hyp[:-1])
            x = self.emb[hyp[-1]]
        out = []
        for h, w in zip(hs, self.gru):
            x = self._gru(x, h, w)
            out.append(x)
        fy = _bf16(out[-1]) @ self.w1.T + self.b1
        self._fy[hyp] = (out, fy)
        return out

    def __call__(self, t, hyp):
        self._states(hyp)
        fy = self._fy[hyp][1]
        z = _bf16(torch.relu(self.fx[t] + fy))
        logits = self.w2 @ z + self.b2
        return torch.log_softmax(logits, 0).numpy()


def sequence_log_prob(row_fn, T, labels, blank):
    """log of the total probability of emitting exactly `labels` in T frames, rows per prefix"""
    U = len(labels)
    rows = [[row_fn(t, tuple(labels[:u])) for u in range(U + 1)] for t in range(T)]
    alpha = np.full((T, U + 1), -np.inf)
    for t in range(T):
        for u in range(U + 1):
            if t == 0 and u == 0:
                alpha[t, u] = 0.0
                continue
            a = alpha[t - 1, u] + rows[t - 1][u][blank] if t > 0 else -np.inf
            c = alpha[t, u - 1] + rows[t][u - 1][labels[u - 1]] if u > 0 else -np.inf
            alpha[t, u] = np.logaddexp(a, c)
    return alpha[T - 1, U] + rows[T - 1][U][blank]


def best_by_enumeration(row_fn, T, V, blank, max_len):
    """arg-max over every label sequence of at most max_len labels: tiny T, V, max_len only"""
    symbols = [k for k in range(V) if k != blank]
    best, best_lp = None, -np.inf
    for n in range(max_len + 1):
        for seq in itertools.product(symbols, repeat=n):
            s = sequence_log_prob(row_fn, T, list(seq), blank)
            if s > best_lp:
                best, best_lp = list(seq), s
    return best, best_lp
