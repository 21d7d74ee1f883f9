"""Reference word-LM attention beam search (test infrastructure, float64 on the host).

The candidate table of include/speech_b200.h (sb_s2s_beam_select_wordlm_batch) over the terms of
tests/ctc_wordlm_ref.WordArpa: candidate c of a hypothesis h (its classes after the start token)
scores score + (p + term(h, c)), or score + p where the table adds nothing:
    c the delimiter ending a non-empty partial word:   the delimiter term d
    c = END:                                           the end term t (trailing word and </s>)
    c taking the partial word out of the lexicon:      gamma
WordPart.score(h, c) is that term (0.0 where there is none), so the LM loops of tests/s2s_lm_ref.py
and tests/s2s_ctc_ref.py run the word LM as an `lm` at lm_weight = 1, insertion_bonus = 0:
score + (p + (1.0 * l + 0.0)) and (1 - w) p + (1.0 * l + 0.0) are those values to the bit.
"""
from s2s_ctc_ref import beam_search_ctc
from s2s_lm_ref import beam_search_lm


class WordPart:
    """the LM part of each candidate under a WordArpa `arpa`, end class `end`, weights a, b, g"""

    def __init__(self, arpa, end, a, b, g):
        self.arpa, self.end, self.a, self.b, self.g = arpa, end, a, b, g

    def term(self, hyp, c):
        """the table's term of candidate (hyp, c), or None where it adds nothing"""
        w = self.arpa
        hyp = tuple(hyp)
        if c == self.end:
            return w.end_term(hyp, self.a, self.b, self.g)
        words, partial = w.split(hyp)
        if c == w.delim:
            return w.delim_term(words, partial, self.a, self.b, self.g) if partial else None
        if partial in w.prefixes and partial + (c,) not in w.prefixes:
            return self.g
        return None

    def score(self, hyp, c):
        t = self.term(hyp, c)
        return 0.0 if t is None else t

    def value(self, score, hyp, c, p):
        """the fused candidate value, written as the table writes it"""
        t = self.term(hyp, c)
        return score + p if t is None else score + (p + t)


def beam_search_wordlm(m, x_enc, start_tok, end_tok, beam_size, max_len, part):
    """one utterance (x_enc (1, T, H)) -> (token tuple, fused float64 score)"""
    return beam_search_lm(m, x_enc, start_tok, end_tok, beam_size, max_len, part, 1.0, 0.0)


def beam_search_ctc_wordlm(m, x_enc, y, Tb, start_tok, end_tok, beam_size, max_len, ctc_weight,
                           prebeam, part, lens=None):
    """joint CTC/attention (tests/s2s_ctc_ref.beam_search_ctc) with the word LM's part"""
    return beam_search_ctc(m, x_enc, y, Tb, start_tok, end_tok, beam_size, max_len, ctc_weight,
                           prebeam, part, 1.0, 0.0, lens)
