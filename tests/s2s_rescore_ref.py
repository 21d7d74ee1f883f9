"""Float64 CPU restatement of two-pass decoding (Seq2Seq.recognize_two_pass), for the tests:

- nbest_prefix_beam: the CTC prefix beam search of oracle/ctc_decoder_ref.py over log-probabilities
  (no log taken here), returning the whole final beam of <= K entries in its order - the stable
  descending sort by lse(p_b, p_nb), ties in first-touch order - with each entry's c = lse(p_b,
  p_nb);
- combine / select: r = (1 - w) a + w c with both products rounded and then added (Python floats
  are float64 and never contracted), and the first index of the largest r.
"""
import math

NEG_INF = -float("inf")


def _lse(*xs):
    if all(x == NEG_INF for x in xs):
        return NEG_INF
    m = max(xs)
    return m + math.log(sum(math.exp(x - m) for x in xs))


def nbest_prefix_beam(logp, beam_size, blank):
    """logp (T, S) log-probabilities (any float array; each value is used as a float64) -> list
    of (label tuple, c) of the final beam, best first"""
    T, S = len(logp), len(logp[0]) if len(logp) else 0
    beam = [((), (0.0, NEG_INF))]
    for t in range(T):
        cand = {}

        def slot(prefix):
            if prefix not in cand:
                cand[prefix] = [NEG_INF, NEG_INF]
            return cand[prefix]

        for s in range(S):
            p = float(logp[t][s])
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
        beam = [(k, (v[0], v[1])) for k, v in ranked[:beam_size]]
    return [(k, _lse(*v)) for k, v in beam]


def combine(a, c, w):
    """r = (1 - w) a + w c in float64"""
    return (1.0 - w) * a + w * c


def select(a, c, w):
    """index of the largest r over the entries (a_i, c_i), ties to the lowest index; -> (i, r_i)"""
    best, rb = -1, NEG_INF
    for i, (ai, ci) in enumerate(zip(a, c)):
        r = combine(ai, ci, w)
        if best < 0 or r > rb:
            best, rb = i, r
    return best, rb
