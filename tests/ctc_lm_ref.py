"""Reference LM-fused CTC prefix beam search (test infrastructure).

oracle/ctc_decoder_ref.prefix_beam_search with shallow fusion: extending a prefix by a non-blank
symbol s uses q = p_s + (lm_weight * lm(s | prefix) + insertion_bonus) in every term of that
extension, including a repeated symbol's extension from the blank-ending mass.  Blank terms and
the repeated symbol that keeps the prefix use p_s.  Float64, first-touch order and the stable
sort are the oracle's.  `lm` is anything with score(prefix, s) (tests/ngram_ref.ArpaLM).
"""
import numpy as np

from oracle.ctc_decoder_ref import NEG_INF, _lse


def prefix_beam_search_lm(probs, beam_size, blank, lm, lm_weight, insertion_bonus):
    probs = np.asarray(probs)
    T, S = probs.shape
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
                q = p + (lm_weight * lm.score(prefix, s) + insertion_bonus)
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
    best = beam[0]
    return best[0], -_lse(*best[1])
