"""Seq2Seq.recognize: beam search of a whole minibatch in one device-resident call
(functions/s2s.py: beam_search_batch -> csrc/s2s.cu).

Every utterance of the batch must get, bit for bit (tokens and float64 score), the search it gets
alone - the single-utterance device search (`s2s.beam_search`'s path, B = 1) on its own slice of
the same encoder output - and the tokens of the reference's host loop (seq2seq.py:180-227,
restated below over decode_step).  Covered: small and WSJ-shaped decoders at beams 1 / 4 / 8 / 32,
the many-CTA projection with the split selection at V = 5001, the split selection forced at a
small vocabulary, the exact-lengths mode, and utterances that stop at different steps."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _small_cfg(H=32, layers=2):
    return {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                        "rnn": {"dim": H, "bidirectional": True, "layers": layers}},
            "decoder": {"embedding_dim": H, "layers": 1}}


WSJ_CFG = {"dropout": 0.0, "encoder": {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
                                       "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True}}


def _model(cfg, fdim, V, seed, exact=False):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(seed)
    np.random.seed(seed)
    if exact:
        cfg = dict(cfg, exact_lengths=True)
    m = Seq2Seq(fdim, V, cfg).cuda()
    m.set_eval()
    with torch.no_grad():                 # make the decoder far from uniform
        m.fc.fc.weight.mul_(8.0)
        m.embedding.weight.mul_(3.0)
    return m


def _inputs(fdim, T, n=5, step=13, seed=0):
    rng = np.random.RandomState(seed)
    return [rng.randn(T - step * i, fdim).astype(np.float32) for i in range(n)]


def _encode(m, inputs):
    lens = m.input_lens(inputs)
    with torch.no_grad():
        return m._encode(m.stage_inputs(inputs), lens), lens


def _single(m, x_enc, b, start, end, K, max_len, frames=None):
    """the single-utterance device search on utterance b's slice of the batch's encoder output"""
    from speech_b200.functions import s2s
    eh = x_enc[b:b + 1] if frames is None else x_enc[b:b + 1, :frames]
    with torch.no_grad():
        (toks, score, steps), = s2s.beam_search_batch(m, eh, start, end, K, max_len)
        assert s2s.beam_search(m, eh, start, end, K, max_len) == toks
    return toks, score, steps


def _check_against_single(m, inputs, K, max_len, exact=False):
    V = m.embedding.num_embeddings
    start, end = V - 1, V - 2
    x_enc, lens = _encode(m, inputs)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=max_len, return_scores=True)
    assert len(labels) == len(scores) == len(inputs)
    for b in range(len(inputs)):
        toks, score, _ = _single(m, x_enc, b, start, end, K, max_len,
                                 frames=lens[b] if exact else None)
        assert labels[b] == list(toks), (K, b)
        assert scores[b] == score, (K, b)                    # float64, bit for bit
        assert labels[b][0] == start
        assert isinstance(scores[b], float)
    return labels, scores


def _host_beam(m, x_enc, start_tok, end_tok, beam_size, max_len):
    """seq2seq.py:180-227 (with the py3 list() fix) over decode_step, one utterance."""
    y = torch.zeros(1, 1, dtype=torch.int64, device=x_enc.device)
    beam = [((start_tok,), 0, None)]
    complete = []
    for _ in range(max_len):
        new_beam = []
        for hyp, score, state in beam:
            y[0] = hyp[-1]
            out, state = m.decode_step(x_enc, y, state=state, softmax=True)
            for i, p in enumerate(out.cpu().numpy().squeeze(0).tolist()):
                new_beam.append((hyp + (i,), score + p, state))
        new_beam = sorted(new_beam, key=lambda c: c[1], reverse=True)
        for cand in new_beam[:beam_size]:
            if cand[0][-1] == end_tok:
                complete.append(cand)
        beam = [c for c in new_beam if c[0][-1] != end_tok][:beam_size]
        if len(beam) == 0:
            break
        if sum(c[1] > beam[0][1] for c in complete) >= beam_size:
            break
    complete = sorted(complete, key=lambda c: c[1], reverse=True)
    if len(complete) == 0:
        complete = beam
    return complete[0][0], complete[0][1]


@pytest.mark.parametrize("K", [1, 4, 8, 32])
@pytest.mark.parametrize("wsj", [False, True])
def test_batch_equals_single_utterance_search_bit_for_bit(cuda_lib, wsj, K):
    if wsj:
        m, inputs = _model(WSJ_CFG, 80, 30, 11), _inputs(80, 300, step=23)
    else:
        m, inputs = _model(_small_cfg(), 40, 11, 12), _inputs(40, 90, step=9)
    _check_against_single(m, inputs, K, max_len=20)


@pytest.mark.parametrize("K", [1, 4, 8])
def test_batch_equals_the_reference_host_loop(cuda_lib, K):
    m, inputs = _model(_small_cfg(), 40, 11, 13), _inputs(40, 80, step=9, seed=1)
    V = 11
    x_enc, _ = _encode(m, inputs)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=12, return_scores=True)
    for b in range(len(inputs)):
        ref, ref_score = _host_beam(m, x_enc[b:b + 1], V - 1, V - 2, K, 12)
        assert labels[b] == list(ref), (K, b)
        assert abs(scores[b] - ref_score) <= 1e-9 * max(1.0, abs(ref_score)), (K, b)


def test_large_vocabulary_many_cta_projection_and_split_selection(cuda_lib):
    from speech_b200.functions import s2s
    m = _model(_small_cfg(64, layers=1), 40, 5001, 21)
    assert not s2s.fc_fused(64, 5000) and not s2s.beam_select_fits(8, 5000)
    _check_against_single(m, _inputs(40, 60, step=7, seed=2), 8, max_len=8)


def test_forced_split_selection_equals_single_cta_selection(cuda_lib, monkeypatch):
    from speech_b200.functions import s2s
    m = _model(_small_cfg(), 40, 31, 23)
    inputs = _inputs(40, 80, step=9, seed=3)
    assert s2s.beam_select_fits(8, 30)
    runs = []
    for forced in (False, True):
        if forced:
            monkeypatch.setattr(s2s, "beam_select_fits", lambda K, C: False)
        runs.append([m.recognize(inputs, beam_size=K, max_len=15, return_scores=True)
                     for K in (1, 4, 8)])
    assert runs[0] == runs[1]


@pytest.mark.parametrize("K", [1, 4, 8])
def test_exact_lengths_each_utterance_searches_its_own_frames(cuda_lib, K):
    m = _model(_small_cfg(), 40, 11, 14, exact=True)
    inputs = _inputs(40, 100, step=15, seed=4)
    lens = m.input_lens(inputs)
    assert len(set(lens)) == len(lens)
    _check_against_single(m, inputs, K, max_len=15, exact=True)


def test_utterances_that_stop_at_different_steps(cuda_lib):
    """A batch in which some searches stop early on their own and at least one runs to max_len:
    every result is still its single-utterance search; and max_len = 1."""
    from speech_b200.functions import s2s
    m = _model(_small_cfg(), 40, 11, 15)
    inputs = _inputs(40, 90, n=5, step=11, seed=5)
    x_enc, _ = _encode(m, inputs)
    K, end = 4, 9
    # raise the END logit until the natural stop steps (max_len = 60) spread out
    found = None
    for bias in (0.0, 1.0, 2.0, 3.0, 4.0, 6.0, 8.0):
        with torch.no_grad():
            m.fc.fc.bias[end] += bias - (found or 0.0)
        found = bias
        with torch.no_grad():
            steps = [r[2] for r in s2s.beam_search_batch(m, x_enc, 10, end, K, 60)]
        if min(steps) < max(steps) - 1:
            break
    assert min(steps) < max(steps) - 1, steps
    max_len = max(steps) - 1
    with torch.no_grad():
        res = s2s.beam_search_batch(m, x_enc, 10, end, K, max_len)
    early = [b for b in range(5) if res[b][2] < max_len]
    full = [b for b in range(5) if res[b][2] == max_len]
    assert early and full, [r[2] for r in res]
    for b in range(5):
        assert res[b] == _single(m, x_enc, b, 10, end, K, max_len), b
    # the batch API agrees, and at max_len = 1 every search stops after its first step
    assert m.recognize(inputs, beam_size=K, max_len=max_len) == [list(r[0]) for r in res]
    for K1 in (1, 4):
        one = m.recognize(inputs, beam_size=K1, max_len=1, return_scores=True)
        for b in range(5):
            toks, score, steps1 = _single(m, x_enc, b, 10, end, K1, 1)
            assert steps1 == 1
            assert one[0][b] == list(toks) and one[1][b] == score
            assert len(toks) == 2
