"""Seq2Seq.recognize with a word n-gram LM: each word scored at its delimiter and the trailing word
with </s> at END, inside the batched attention beam search (functions/s2s.py: beam_search_batch ->
sb_s2s_beam_select{,_split}_wordlm_batch / sb_s2s_ctc_candidates_wordlm, csrc/s2s_beam.cuh).

- zero weights give the LM-less search bit for bit, small and WSJ-shaped; nonzero weights change it;
- each utterance of a batch gets its own single-utterance search bit for bit;
- tokens equal the reference loop (tests/s2s_wordlm_ref.py) and scores match to 1e-9 relative, at
  orders 1 to 4, with oov_penalty = 0, finite and -inf;
- the split selection, forced and at a ~6000-class vocabulary, and the exact-lengths mode;
- joint CTC/attention with a word LM against its reference, and at zero weights against the joint
  search without an LM;
- the LM decides where the acoustics do not: uniform rows give the LM's sentence, an acoustic tie
  goes to the lexicon's spelling, and a closed vocabulary decodes lexicon words only.
"""
import math

import numpy as np
import pytest
import torch

from ctc_wordlm_ref import WordArpa
from s2s_wordlm_ref import WordPart, beam_search_ctc_wordlm, beam_search_wordlm
from speech_b200.lm import WordLM

pytestmark = pytest.mark.gpu

LETTERS = "abcde"


def _symbols(letters):
    """Preprocessor.int_to_char layout: letters, the space, </s> (END), <s> (START)"""
    return list(letters) + [" ", "</s>", "<s>"]


def _cfg(H=32, layers=2, ctc_weight=None):
    dec = {"embedding_dim": H, "layers": 1}
    if ctc_weight:
        dec["ctc_weight"] = ctc_weight
    return {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                        "rnn": {"dim": H, "bidirectional": True, "layers": layers}},
            "decoder": dec}


WSJ_CFG = {"dropout": 0.0, "encoder": {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
                                       "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True}}


def _model(cfg, fdim, V, seed, exact=False, sharpen=2.0):
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
        if m.ctc_weight > 0:
            m.ctc_fc.fc.weight.mul_(4.0)
    return m


def _inputs(fdim, T, n=3, step=9, seed=0):
    rng = np.random.RandomState(seed)
    return [rng.randn(T - step * i, fdim).astype(np.float32) for i in range(n)]


def _encode(m, inputs):
    lens = m.input_lens(inputs)
    with torch.no_grad():
        return m._encode(m.stage_inputs(inputs), lens), lens


def _texts(letters, seed, n_words=8, n=40, max_len=3):
    rng = np.random.RandomState(seed)
    vocab = sorted({"".join(rng.choice(list(letters), rng.randint(1, max_len + 1)))
                    for _ in range(n_words)})
    return [" ".join(rng.choice(vocab, rng.randint(1, 5))) for _ in range(n)]


def _wlm(order, seed, g=-2.0, letters=LETTERS, texts=None):
    syms = _symbols(letters)
    V = len(syms)
    texts = _texts(letters, seed) if texts is None else texts
    return WordLM.train(texts, order, syms, blank=V - 1, end=V - 2, oov_penalty=g)


def _part(lm, tmp_path, a, b):
    p = str(tmp_path / "w.arpa")
    lm.to_arpa(p)
    return WordPart(WordArpa(p, lm.spell, lm.delimiter), lm.end, a, b, lm.oov_penalty)


def _close(got, ref):
    return got == ref or abs(got - ref) <= 1e-9 * max(1.0, abs(ref))


def _single(m, x_enc, b, K, max_len, lm, a, bonus, frames=None):
    from speech_b200.functions import s2s
    V = m.embedding.num_embeddings
    eh = x_enc[b:b + 1] if frames is None else x_enc[b:b + 1, :frames]
    with torch.no_grad():
        (toks, score, _), = s2s.beam_search_batch(m, eh, V - 1, V - 2, K, max_len, None, lm, a,
                                                  bonus)
    return list(toks), score


WSJ_LETTERS = "abcdefghijklmnopqrstuvwxyz'.-"     # V = 32 with the space, END and START


@pytest.mark.parametrize("K", [1, 4, 8, 32])
@pytest.mark.parametrize("wsj", [False, True])
def test_zero_weights_give_the_plain_search_bit_for_bit(cuda_lib, wsj, K):
    if wsj:
        letters = WSJ_LETTERS
        V, m, inputs = 32, _model(WSJ_CFG, 80, 32, 11, sharpen=8.0), _inputs(80, 300, n=5, step=23)
    else:
        letters = LETTERS
        V, m, inputs = 8, _model(_cfg(), 40, 8, 12, sharpen=8.0), _inputs(40, 90, n=5)
    lm = _wlm(3, 1, g=0.0, letters=letters)
    assert lm.num_classes == V
    plain = m.recognize(inputs, beam_size=K, max_len=20, return_scores=True)
    fused = m.recognize(inputs, beam_size=K, max_len=20, return_scores=True, lm=lm,
                        lm_weight=0.0, insertion_bonus=0.0)
    assert fused == plain
    # nonzero weights change the search (the LM is live on this path)
    lm.oov_penalty = -1.0
    other = m.recognize(inputs, beam_size=K, max_len=20, return_scores=True, lm=lm,
                        lm_weight=0.7, insertion_bonus=0.3)
    assert other[1] != plain[1]


@pytest.mark.parametrize("K", [1, 4, 8])
def test_batch_equals_single_utterance_search(cuda_lib, K):
    m, inputs = _model(_cfg(), 40, 8, 13), _inputs(40, 90, n=5, seed=1)
    lm = _wlm(3, 2, g=-1.5)
    x_enc, _ = _encode(m, inputs)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, lm=lm,
                                 lm_weight=0.6, insertion_bonus=0.4)
    for b in range(len(inputs)):
        assert (labels[b], scores[b]) == _single(m, x_enc, b, K, 15, lm, 0.6, 0.4), (K, b)


@pytest.mark.parametrize("order,a,bonus,g", [(1, 0.5, 0.5, 0.0), (2, 0.8, 1.0, -2.0),
                                             (3, 1.5, -0.5, -math.inf), (4, 0.6, 0.3, -1.0),
                                             (3, 2.0, 2.0, -0.5)])
def test_search_equals_the_reference_loop(cuda_lib, tmp_path, order, a, bonus, g):
    V = 8
    m, inputs = _model(_cfg(), 40, V, 14), _inputs(40, 80, seed=2)
    lm = _wlm(order, 3 + order, g=g)
    part = _part(lm, tmp_path, a, bonus)
    x_enc, _ = _encode(m, inputs)
    for K in (1, 4):
        labels, scores = m.recognize(inputs, beam_size=K, max_len=12, return_scores=True, lm=lm,
                                     lm_weight=a, insertion_bonus=bonus)
        for b in range(len(inputs)):
            ref, ref_score = beam_search_wordlm(m, x_enc[b:b + 1], V - 1, V - 2, K, 12, part)
            assert labels[b] == list(ref), (K, b, labels[b], ref)
            assert _close(scores[b], ref_score), (K, b, scores[b], ref_score)


def test_forced_split_selection_equals_single_cta_selection(cuda_lib, monkeypatch):
    from speech_b200.functions import s2s
    m, inputs = _model(_cfg(), 40, 8, 23), _inputs(40, 80, n=4, seed=3)
    lm = _wlm(4, 4, g=-1.0)
    assert s2s.beam_select_fits(8, 7)
    runs = []
    for forced in (False, True):
        if forced:
            monkeypatch.setattr(s2s, "beam_select_fits", lambda K, C: False)
        runs.append([m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, lm=lm,
                                 lm_weight=0.9, insertion_bonus=0.2) for K in (1, 4, 8)])
    assert runs[0] == runs[1]


def test_large_vocabulary_split_selection_matches_the_reference(cuda_lib, tmp_path):
    from speech_b200.functions import s2s
    letters = "".join(chr(0x4E00 + i) for i in range(6000))
    V = len(letters) + 3
    m = _model(_cfg(64, layers=1), 40, V, 21, sharpen=1.0)
    assert not s2s.fc_fused(64, V - 1) and not s2s.beam_select_fits(8, V - 1)
    lm = WordLM.train(_texts(letters[:12], 5, n_words=20), 3, _symbols(letters), blank=V - 1,
                      end=V - 2, oov_penalty=-2.5)
    part = _part(lm, tmp_path, 0.5, 0.5)
    inputs = _inputs(40, 60, n=2, step=7, seed=4)
    x_enc, _ = _encode(m, inputs)
    labels, scores = m.recognize(inputs, beam_size=8, max_len=5, return_scores=True, lm=lm,
                                 lm_weight=0.5, insertion_bonus=0.5)
    for b in range(len(inputs)):
        ref, ref_score = beam_search_wordlm(m, x_enc[b:b + 1], V - 1, V - 2, 8, 5, part)
        assert labels[b] == list(ref), b
        assert _close(scores[b], ref_score), b


@pytest.mark.parametrize("K", [1, 4, 8])
def test_exact_lengths_with_a_word_lm(cuda_lib, K):
    m = _model(_cfg(), 40, 8, 15, exact=True)
    inputs = _inputs(40, 100, n=5, step=15, seed=5)
    lm = _wlm(3, 6, g=-1.0)
    x_enc, lens = _encode(m, inputs)
    assert len(set(lens)) == len(lens)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, lm=lm,
                                 lm_weight=0.5, insertion_bonus=0.5)
    for b in range(len(inputs)):
        assert (labels[b], scores[b]) == _single(m, x_enc, b, K, 15, lm, 0.5, 0.5,
                                                 frames=lens[b]), (K, b)


@pytest.mark.parametrize("K,M,g", [(1, None, -1.0), (4, None, -math.inf), (4, 7, -2.0)])
def test_joint_ctc_with_a_word_lm_equals_the_reference_loop(cuda_lib, tmp_path, K, M, g):
    V, w, a, bonus = 8, 0.4, 0.6, 0.3
    m = _model(_cfg(ctc_weight=0.3), 40, V, 31)
    inputs = _inputs(40, 80, seed=6)
    lm = _wlm(3, 8, g=g)
    part = _part(lm, tmp_path, a, bonus)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=12, return_scores=True, lm=lm,
                                 lm_weight=a, insertion_bonus=bonus, ctc_weight=w, ctc_prebeam=M)
    x, _ = _encode(m, inputs)
    with torch.no_grad():
        y = torch.log_softmax(m.ctc_fc(x).float(), dim=-1).cpu().numpy()
    Mr = min(V - 1, 3 * K // 2) if M is None else M
    for b in range(len(inputs)):
        ref, ref_score = beam_search_ctc_wordlm(m, x[b:b + 1], y[b], y.shape[1], V - 1, V - 2, K,
                                                12, w, Mr, part)
        assert labels[b] == list(ref), (K, M, b, labels[b], ref)
        assert _close(scores[b], ref_score), (K, M, b)


@pytest.mark.parametrize("K", [1, 4, 8])
def test_joint_ctc_at_zero_weights_is_the_joint_search_without_an_lm(cuda_lib, K):
    m = _model(_cfg(ctc_weight=0.3), 40, 8, 32)
    inputs = _inputs(40, 90, n=4, seed=7)
    lm = _wlm(3, 9, g=0.0)
    plain = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, ctc_weight=0.5)
    fused = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True, lm=lm,
                        lm_weight=0.0, insertion_bonus=0.0, ctc_weight=0.5)
    assert fused == plain


@pytest.mark.parametrize("K", [16, 32])
def test_uniform_acoustics_give_the_lm_sentence(cuda_lib, K):
    V = 8
    m = _model(_cfg(), 40, V, 16)
    with torch.no_grad():
        m.fc.fc.weight.zero_()
        m.fc.fc.bias.zero_()
    lm = _wlm(3, 0, g=-math.inf, texts=["ab c"])
    # a, b, space, c: the LM's words and </s> outweigh the acoustic cost of the longer sentence.
    # The word LM scores nothing inside a word, so the letters that start the next word tie and a
    # narrow beam keeps the lower-indexed "ab ab .." (the reference loop agrees); 16 entries keep c.
    labels = m.recognize(_inputs(40, 90, seed=8), beam_size=K, max_len=20, lm=lm, lm_weight=8.0,
                         insertion_bonus=1.0)
    assert labels == [[V - 1, 0, 1, 5, 2, V - 2]] * 3


def test_an_acoustic_tie_goes_to_the_lexicon_spelling(cuda_lib):
    V = 8
    m = _model(_cfg(), 40, V, 17)
    with torch.no_grad():
        m.fc.fc.weight.zero_()
        m.fc.fc.bias.fill_(-5.0)
        m.fc.fc.bias[2] = m.fc.fc.bias[3] = 5.0               # c and d tie
        m.fc.fc.bias[V - 2] = -30.0                           # END stays out of the top K
    lm = _wlm(2, 0, g=0.0, texts=["da", "de da"])             # no word starts with c
    inputs = _inputs(40, 90, n=2, seed=9)
    for K in (1, 4):
        tie = m.recognize(inputs, beam_size=K, max_len=1)
        assert tie == [[V - 1, 2]] * 2                        # the lower index wins a tie
        assert m.recognize(inputs, beam_size=K, max_len=1, lm=lm, lm_weight=0.5) == tie
        lm.oov_penalty = -2.0
        assert m.recognize(inputs, beam_size=K, max_len=1, lm=lm,
                           lm_weight=0.5) == [[V - 1, 3]] * 2
        lm.oov_penalty = 0.0


@pytest.mark.parametrize("K", [1, 4, 8])
def test_a_closed_vocabulary_decodes_lexicon_words_only(cuda_lib, K):
    V = 8
    m, inputs = _model(_cfg(), 40, V, 18), _inputs(40, 90, n=5, seed=10)
    lm = _wlm(3, 11, g=-math.inf)
    words = set(lm.words)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=30, return_scores=True, lm=lm,
                                 lm_weight=0.5, insertion_bonus=0.5)
    checked = 0
    for toks, s in zip(labels, scores):
        if not math.isfinite(s):
            continue
        body = toks[1:]
        ended = bool(body) and body[-1] == V - 2
        text = "".join(" " if c == 5 else LETTERS[c] for c in (body[:-1] if ended else body))
        parts = text.split(" ")
        done = parts if ended else parts[:-1]               # a live result's partial word aside
        assert all(w in words for w in done if w), (toks, words)
        checked += 1
    assert checked > 0
