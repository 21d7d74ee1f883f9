"""Reference LM-fused attention beam search (test infrastructure).

The reference's Seq2Seq.beam_search loop (seq2seq.py:180-227, with the py3 list() fix), restated
over decode_step with the fused candidate value
    score + (logp[c] + (lm_weight * lm(c | hyp) + beta_c)),   beta_c = insertion_bonus, 0 for END,
evaluated in that order in float64.  hyp's LM context is its tokens after the start token, preceded
by <s>; lm(END | hyp) is lm(</s> | hyp).  `lm` is anything with score(prefix, c) (EndArpaLM:
tests/ngram_ref.ArpaLM reading the end class as </s>).  Also a Python mirror of the device lookup
(csrc/ngram.cuh) over NGramLM.host_tables(), with the context read from a hypothesis as the attention
search reads it.
"""
import torch

from ngram_ref import ArpaLM


class EndArpaLM(ArpaLM):
    """ArpaLM over a vocabulary with an end class: class `end` is scored as </s> and, like the
    blank, is never a word of the context"""

    def __init__(self, path, symbols, blank, end):
        super().__init__(path, symbols, blank)
        self.words.pop(end, None)
        self.end = end

    def score(self, prefix, s):
        return super().score(prefix, "</s>" if s == self.end else s)


def _find(t, node, tok, kind):
    key = (node << 32) | ((tok + 1) << 1) | kind
    cap = t["cap"]
    h = ((key * 0x9E3779B97F4A7C15) & ((1 << 64) - 1)) >> 32 & (cap - 1)
    while int(t["keys"][h]) != 0:
        if int(t["keys"][h]) == key:
            return int(t["vals"][h])
        h = (h + 1) & (cap - 1)
    return -1


def device_lookup(t, prefix, c):
    """lm(c | <s> prefix) as the attention search computes it: lm_context over the prefix read
    most recent first (the root reads as <s>, -1), then lm_backoff with token tok[c]"""
    hist = ([-1] + list(prefix))[::-1][:t["order"] - 1]
    ctx = [0]
    for h in hist:
        nc = _find(t, ctx[-1], t["bos"] if h < 0 else int(t["tok"][h]), 0)
        if nc < 0:
            break
        ctx.append(nc)
        if h < 0:
            break
    acc = 0.0
    for node in reversed(ctx):
        g = _find(t, node, int(t["tok"][c]), 1)
        if g >= 0:
            return acc + float(t["logp"][g])
        acc += float(t["bow"][node])
    raise AssertionError("no unigram")


def fused(score, p, l, c, end_tok, lm_weight, insertion_bonus):
    return score + (p + (lm_weight * l + (0.0 if c == end_tok else insertion_bonus)))


def beam_search_lm(m, x_enc, start_tok, end_tok, beam_size, max_len, lm, lm_weight,
                   insertion_bonus):
    """one utterance (x_enc (1, T, H)) -> (token tuple, fused float64 score)"""
    y = torch.zeros(1, 1, dtype=torch.int64, device=x_enc.device)
    beam = [((start_tok,), 0.0, None)]
    complete = []
    for _ in range(max_len):
        new_beam = []
        for hyp, score, state in beam:
            y[0] = hyp[-1]
            out, state = m.decode_step(x_enc, y, state=state, softmax=True)
            for c, p in enumerate(out.cpu().numpy().squeeze(0).tolist()):
                l = lm.score(hyp[1:], c)
                new_beam.append((hyp + (c,), fused(score, p, l, c, end_tok, lm_weight,
                                                   insertion_bonus), state))
        new_beam = sorted(new_beam, key=lambda h: h[1], reverse=True)
        for cand in new_beam[:beam_size]:
            if cand[0][-1] == end_tok:
                complete.append(cand)
        beam = [h for h in new_beam if h[0][-1] != end_tok][:beam_size]
        if len(beam) == 0:
            break
        if sum(h[1] > beam[0][1] for h in complete) >= beam_size:
            break
    complete = sorted(complete, key=lambda h: h[1], reverse=True)
    if len(complete) == 0:
        complete = beam
    return complete[0][0], complete[0][1]
