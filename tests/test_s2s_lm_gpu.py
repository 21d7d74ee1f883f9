"""Seq2Seq.recognize with an n-gram LM: shallow fusion inside the batched attention beam search
(functions/s2s.py: beam_search_batch -> sb_s2s_beam_select{,_split}_lm_batch, csrc/s2s.cu).

- lm_weight = insertion_bonus = 0 gives the LM-less search bit for bit (tokens, float64 scores);
- each utterance of a batch gets its own B = 1 LM search bit for bit;
- tokens equal the reference loop over decode_step with the fused value (tests/s2s_lm_ref.py and
  the ARPA lookup of tests/ngram_ref.py), scores to 1e-9 relative, at orders 1 / 3 / 5;
- the split selection, forced and at V = 5001, and the exact-lengths mode;
- the LM decides where the acoustic rows do not: uniform rows give the LM's sentence, and an
  acoustic tie flips with the LM weight.
"""
import math

import numpy as np
import pytest
import torch

from s2s_lm_ref import EndArpaLM, beam_search_lm
from speech_b200.lm import NGramLM

pytestmark = pytest.mark.gpu


def _small_cfg(H=32, layers=2):
    return {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                        "rnn": {"dim": H, "bidirectional": True, "layers": layers}},
            "decoder": {"embedding_dim": H, "layers": 1}}


WSJ_CFG = {"dropout": 0.0, "encoder": {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
                                       "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True}}


def _model(cfg, fdim, V, seed, exact=False, sharpen=8.0):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(seed)
    np.random.seed(seed)
    if exact:
        cfg = dict(cfg, exact_lengths=True)
    m = Seq2Seq(fdim, V, cfg).cuda()
    m.set_eval()
    with torch.no_grad():
        m.fc.fc.weight.mul_(sharpen)
        m.embedding.weight.mul_(3.0)
    return m


def _inputs(fdim, T, n=5, step=13, seed=0):
    rng = np.random.RandomState(seed)
    return [rng.randn(T - step * i, fdim).astype(np.float32) for i in range(n)]


def _encode(m, inputs):
    lens = m.input_lens(inputs)
    with torch.no_grad():
        return m._encode(m.stage_inputs(inputs), lens), lens


def _symbols(V):
    """Preprocessor.int_to_char layout: V - 2 symbols, </s> (END), <s> (START)"""
    return {c: ("w%d" % c if c < V - 2 else ("</s>", "<s>")[c - V + 2]) for c in range(V)}


def _lm(V, order, seed, n=60, max_len=12, sentences=None):
    rng = np.random.RandomState(seed)
    if sentences is None:
        sentences = [[V - 1] + rng.randint(0, V - 2, rng.randint(0, max_len)).tolist() + [V - 2]
                     for _ in range(n)]
    return NGramLM.train(sentences, order, V, V - 1, end=V - 2)


def _arpa(lm, V, tmp_path):
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p, _symbols(V))
    return EndArpaLM(p, [_symbols(V)[c] for c in range(V)], V - 1, V - 2)


def _single_lm(m, x_enc, b, K, max_len, lm, a, bonus, frames=None):
    from speech_b200.functions import s2s
    V = m.embedding.num_embeddings
    eh = x_enc[b:b + 1] if frames is None else x_enc[b:b + 1, :frames]
    with torch.no_grad():
        (toks, score, _), = s2s.beam_search_batch(m, eh, V - 1, V - 2, K, max_len, None, lm, a,
                                                  bonus)
    return list(toks), score


@pytest.mark.parametrize("K", [1, 4, 8, 32])
@pytest.mark.parametrize("wsj", [False, True])
def test_zero_weights_give_the_plain_search_bit_for_bit(cuda_lib, wsj, K):
    if wsj:
        V, m, inputs = 30, _model(WSJ_CFG, 80, 30, 11), _inputs(80, 300, step=23)
    else:
        V, m, inputs = 11, _model(_small_cfg(), 40, 11, 12), _inputs(40, 90, step=9)
    lm = _lm(V, 4, 1)
    plain = m.recognize(inputs, beam_size=K, max_len=20, return_scores=True)
    fused = m.recognize(inputs, beam_size=K, max_len=20, return_scores=True, lm=lm,
                        lm_weight=0.0, insertion_bonus=0.0)
    assert fused == plain
    # and a nonzero weight changes the search (the LM is live on this path)
    other = m.recognize(inputs, beam_size=K, max_len=20, return_scores=True, lm=lm,
                        lm_weight=0.7, insertion_bonus=0.3)
    assert other[1] != plain[1]


@pytest.mark.parametrize("K", [1, 4, 8])
def test_batch_equals_single_utterance_lm_search(cuda_lib, K):
    V = 11
    m, inputs = _model(_small_cfg(), 40, V, 13), _inputs(40, 90, step=9, seed=1)
    lm = _lm(V, 3, 2)
    x_enc, _ = _encode(m, inputs)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, lm=lm,
                                 lm_weight=0.6, insertion_bonus=0.4)
    for b in range(5):
        assert (labels[b], scores[b]) == _single_lm(m, x_enc, b, K, 15, lm, 0.6, 0.4), (K, b)


@pytest.mark.parametrize("order,a,bonus", [(1, 0.5, 0.0), (3, 0.8, 0.5), (3, 1.5, -0.7),
                                           (5, 0.4, 1.0), (5, 2.0, -0.3)])
def test_lm_search_equals_the_fused_reference_loop(cuda_lib, tmp_path, order, a, bonus):
    V = 11
    m, inputs = _model(_small_cfg(), 40, V, 14, sharpen=2.0), _inputs(40, 80, n=3, step=9, seed=2)
    lm = _lm(V, order, 3 + order)
    ref_lm = _arpa(lm, V, tmp_path)
    x_enc, _ = _encode(m, inputs)
    for K in (1, 4):
        labels, scores = m.recognize(inputs, beam_size=K, max_len=12, return_scores=True, lm=lm,
                                     lm_weight=a, insertion_bonus=bonus)
        for b in range(len(inputs)):
            ref, ref_score = beam_search_lm(m, x_enc[b:b + 1], V - 1, V - 2, K, 12, ref_lm, a,
                                            bonus)
            assert labels[b] == list(ref), (K, b)
            assert abs(scores[b] - ref_score) <= 1e-9 * max(1.0, abs(ref_score)), (K, b)


def test_forced_split_selection_equals_single_cta_selection_with_lm(cuda_lib, monkeypatch):
    from speech_b200.functions import s2s
    V = 31
    m = _model(_small_cfg(), 40, V, 23)
    inputs = _inputs(40, 80, step=9, seed=3)
    lm = _lm(V, 4, 4)
    assert s2s.beam_select_fits(8, V - 1)
    runs = []
    for forced in (False, True):
        if forced:
            monkeypatch.setattr(s2s, "beam_select_fits", lambda K, C: False)
        runs.append([m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, lm=lm,
                                 lm_weight=0.9, insertion_bonus=0.2) for K in (1, 4, 8)])
    assert runs[0] == runs[1]


def test_large_vocabulary_split_selection_matches_the_reference(cuda_lib, tmp_path):
    from speech_b200.functions import s2s
    V = 5001
    m = _model(_small_cfg(64, layers=1), 40, V, 21, sharpen=1.0)
    assert not s2s.fc_fused(64, V - 1) and not s2s.beam_select_fits(8, V - 1)
    lm = _lm(V, 3, 5, n=400, max_len=8)
    ref_lm = _arpa(lm, V, tmp_path)
    inputs = _inputs(40, 60, n=2, step=7, seed=4)
    x_enc, _ = _encode(m, inputs)
    labels, scores = m.recognize(inputs, beam_size=8, max_len=5, return_scores=True, lm=lm,
                                 lm_weight=0.5, insertion_bonus=0.5)
    for b in range(len(inputs)):
        ref, ref_score = beam_search_lm(m, x_enc[b:b + 1], V - 1, V - 2, 8, 5, ref_lm, 0.5, 0.5)
        assert labels[b] == list(ref), b
        assert abs(scores[b] - ref_score) <= 1e-9 * max(1.0, abs(ref_score)), b


@pytest.mark.parametrize("K", [1, 4, 8])
def test_exact_lengths_with_lm(cuda_lib, K):
    V = 11
    m = _model(_small_cfg(), 40, V, 15, exact=True)
    inputs = _inputs(40, 100, step=15, seed=5)
    lm = _lm(V, 3, 6)
    x_enc, lens = _encode(m, inputs)
    assert len(set(lens)) == len(lens)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, lm=lm,
                                 lm_weight=0.5, insertion_bonus=0.5)
    for b in range(len(inputs)):
        assert (labels[b], scores[b]) == _single_lm(m, x_enc, b, K, 15, lm, 0.5, 0.5,
                                                    frames=lens[b]), (K, b)


@pytest.mark.parametrize("K", [1, 4])
def test_uniform_acoustics_give_the_lm_sentence(cuda_lib, K):
    V = 12
    m = _model(_small_cfg(), 40, V, 16)
    with torch.no_grad():
        m.fc.fc.weight.zero_()
        m.fc.fc.bias.zero_()
    sentence = [3, 7, 1, 1, 8, 0, 5]
    lm = _lm(V, 4, 0, sentences=[[V - 1] + sentence + [V - 2]])
    # the bonus cancels the uniform rows' log(1 / C) on every token but END
    labels = m.recognize(_inputs(40, 90, n=3, step=9, seed=6), beam_size=K, max_len=20, lm=lm,
                         lm_weight=1.0, insertion_bonus=math.log(V - 1))
    assert labels == [[V - 1] + sentence + [V - 2]] * 3


def test_an_acoustic_tie_flips_with_the_lm_weight(cuda_lib):
    V = 12
    m = _model(_small_cfg(), 40, V, 17)
    with torch.no_grad():
        m.fc.fc.weight.zero_()
        m.fc.fc.bias.fill_(-5.0)
        m.fc.fc.bias[2] = m.fc.fc.bias[6] = 5.0               # classes 2 and 6 tie
        m.fc.fc.bias[V - 2] = -30.0                           # END stays out of the top K
    lm = _lm(V, 2, 0, sentences=[[V - 1, 6, V - 2]] * 3 + [[V - 1, 2, V - 2]])
    inputs = _inputs(40, 90, n=2, step=9, seed=7)
    for K in (1, 4):
        tie = m.recognize(inputs, beam_size=K, max_len=1)
        assert tie == m.recognize(inputs, beam_size=K, max_len=1, lm=lm, lm_weight=0.0)
        assert tie == [[V - 1, 2]] * 2                             # the lower index wins a tie
        assert m.recognize(inputs, beam_size=K, max_len=1, lm=lm,
                           lm_weight=0.5) == [[V - 1, 6]] * 2
