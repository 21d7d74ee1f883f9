"""Host checks (no GPU) of two-pass decoding of the attention model (Seq2Seq.recognize_two_pass,
Seq2Seq.stream -> streaming.Seq2SeqStream):

- the C ABI: the new symbols are bound, and every status of sb_ctc_stream_nbest and
  sb_s2s_score_tokens from null or out-of-range arguments, before any launch;
- every ValueError of recognize_two_pass, stream and Seq2SeqStream, raised before the CUDA check;
- the selection rule (functions/s2s.py: two_pass_select) on hand-made (a, c) arrays, ties, empty
  slots, w = 0 and w = 1, against the float64 reference of tests/s2s_rescore_ref.py.
"""
import math

import numpy as np
import pytest
import torch

from s2s_rescore_ref import combine, nbest_prefix_beam, select
from speech_b200 import _lib

INVALID, UNSUPPORTED = 1, 3


def _cfg(w=0.3, bidirectional=False, lookahead=0):
    enc = {"conv": [[8, 5, 8, 2]], "rnn": {"dim": 32, "bidirectional": bidirectional, "layers": 1}}
    if lookahead:
        enc["lookahead"] = lookahead
    return {"dropout": 0.0, "encoder": enc,
            "decoder": {"embedding_dim": 32, "layers": 1, "ctc_weight": w}}


def _model(w=0.3, **kw):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(0)
    return Seq2Seq(40, 9, _cfg(w, **kw))


def test_two_pass_symbols_are_bound():
    lib = _lib.load()
    for name in ("sb_ctc_stream_nbest", "sb_s2s_score_tokens"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


@pytest.mark.parametrize("args,status", [
    ((None, 2, 10, 4, 8, 8, 8, 8), INVALID),
    ((8, 2, 10, 4, None, 8, 8, 8), INVALID),
    ((8, 2, 10, 4, 8, None, 8, 8), INVALID),
    ((8, 2, 10, 4, 8, 8, None, 8), INVALID),
    ((8, 2, 10, 4, 8, 8, 8, None), INVALID),
    ((8, 0, 10, 4, 8, 8, 8, 8), INVALID),
    ((8, 2, 0, 4, 8, 8, 8, 8), INVALID),
    ((8, 2, 10, 0, 8, 8, 8, 8), INVALID),
    ((8, 2, 10, 33, 8, 8, 8, 8), UNSUPPORTED),
])
def test_nbest_refuses_bad_arguments(args, status):
    """statuses as sb_ctc_stream_best's, before any launch: fake pointers are never read"""
    lib = _lib.load()
    assert lib.sb_ctc_stream_nbest(*args, None) == status


@pytest.mark.parametrize("args", [
    (None, 4, 9, 8, 3, 8, 0, 7, 8),
    (8, 4, 9, None, 3, 8, 0, 7, 8),
    (8, 4, 9, 8, 3, None, 0, 7, 8),
    (8, 4, 9, 8, 3, 8, 0, 7, None),
    (8, 0, 9, 8, 3, 8, 0, 7, 8),         # R
    (8, -1, 9, 8, 3, 8, 0, 7, 8),
    (8, 4, 0, 8, 3, 8, 0, 7, 8),         # C
    (8, 4, 9, 8, 0, 8, 0, 7, 8),         # ld
    (8, 4, 9, 8, 3, 8, -1, 7, 8),        # u
    (8, 4, 9, 8, 3, 8, 0, 9, 8),         # end_tok outside [0, C)
    (8, 4, 9, 8, 3, 8, 0, -1, 8),
])
def test_score_tokens_refuses_bad_arguments(args):
    lib = _lib.load()
    assert lib.sb_s2s_score_tokens(*args, None) == INVALID


def test_score_tokens_refuses_more_rows_than_a_grid_holds():
    lib = _lib.load()
    assert lib.sb_s2s_score_tokens(8, 1 << 40, 9, 8, 3, 8, 0, 7, 8, None) == UNSUPPORTED


# ---- ValueErrors, all before the model's CUDA check (the models here live on the CPU) ----------

def _inputs():
    return [np.zeros((40, 40), np.float32)]


def test_recognize_two_pass_needs_a_ctc_head():
    from speech_b200.models import Seq2Seq
    m = Seq2Seq(40, 9, dict(_cfg(), decoder={"embedding_dim": 32, "layers": 1}))
    with pytest.raises(ValueError, match="CTC head"):
        m.recognize_two_pass(_inputs())
    with pytest.raises(ValueError, match="CTC head"):
        m.stream(2)


@pytest.mark.parametrize("K", [0, 33, -1, 2.5, True])
def test_recognize_two_pass_refuses_a_beam_size(K):
    m = _model()
    with pytest.raises(ValueError, match="beam_size"):
        m.recognize_two_pass(_inputs(), beam_size=K)
    with pytest.raises(ValueError, match="beam_size"):
        m.stream(2, beam_size=K)


@pytest.mark.parametrize("w", [-0.1, 1.5, math.nan, math.inf, "0.5", None, True])
def test_recognize_two_pass_refuses_a_ctc_weight(w):
    m = _model()
    with pytest.raises(ValueError, match="ctc_weight"):
        m.recognize_two_pass(_inputs(), ctc_weight=w)
    with pytest.raises(ValueError, match="ctc_weight"):
        m.stream(2, ctc_weight=w)


def test_recognize_two_pass_refuses_an_empty_batch():
    with pytest.raises(ValueError, match="at least one"):
        _model().recognize_two_pass([])


def test_stream_keeps_the_ctc_stream_refusals():
    m = _model()
    with pytest.raises(ValueError, match="num_streams"):
        m.stream(0)
    with pytest.raises(ValueError, match="max_frames"):
        m.stream(2, max_frames=0)
    with pytest.raises(ValueError, match="bidirectional"):
        _model(bidirectional=True).stream(2)


def test_stream_needs_a_cuda_model_after_its_checks():
    """the arguments pass; the CPU model is then refused by the CUDA check"""
    with pytest.raises(_lib.SpeechB200Error, match="CUDA"):
        _model(lookahead=2).stream(2, beam_size=4, ctc_weight=1.0)


# ---- the selection rule --------------------------------------------------------------------

def _select(a, c, valid, w):
    from speech_b200.functions import s2s
    a = torch.tensor(a, dtype=torch.float64)
    c = torch.tensor(c, dtype=torch.float64)
    best, r = s2s.two_pass_select(a, c, torch.tensor(valid), w)
    return best.tolist(), r


def test_selection_equals_the_reference_bit_for_bit():
    rng = np.random.RandomState(1)
    for w in [0.0, 0.1, 0.3, 0.5, 0.7, 1.0, 1.0 / 3.0]:
        a = (rng.randn(6, 10) * 7).tolist()
        c = (rng.randn(6, 10) * 7).tolist()
        best, r = _select(a, c, [[True] * 10] * 6, w)
        for b in range(6):
            i, rb = select(a[b], c[b], w)
            assert best[b] == i
            assert r[b, i].item() == rb
            for k in range(10):
                assert r[b, k].item() == combine(a[b][k], c[b][k], w)


def test_selection_ties_go_to_the_lower_index():
    a = [[-1.0, -2.0, -1.0, -0.5], [-3.0, -3.0, -3.0, -3.0]]
    c = [[-2.0, -1.0, -2.0, -2.5], [-1.0, -1.0, -1.0, -1.0]]
    best, _ = _select(a, c, [[True] * 4] * 2, 0.5)     # r = -1.5 -1.5 -1.5 -1.5 / all -2
    assert best == [0, 0]
    best, _ = _select([[-1.0, 0.0, 0.0]], [[0.0, -5.0, -5.0]], [[True] * 3], 0.0)
    assert best == [1]


def test_selection_at_w_0_and_w_1():
    a = [[-9.0, -1.0, -4.0]]
    c = [[-1.0, -2.0, -3.0]]
    assert _select(a, c, [[True] * 3], 1.0)[0] == [0]     # the first pass's best
    assert _select(a, c, [[True] * 3], 0.0)[0] == [1]     # the attention's choice
    assert _select(a, c, [[True] * 3], 1.0)[1][0, 0].item() == -1.0


def test_selection_skips_empty_slots():
    """an empty slot (c = -inf, a = 0) never wins, also at w = 0 where 0 * -inf would be NaN"""
    a = [[-5.0, 0.0, 0.0]]
    c = [[-1.0, -math.inf, -math.inf]]
    for w in [0.0, 0.5, 1.0]:
        best, r = _select(a, c, [[True, False, False]], w)
        assert best == [0]
        assert r[0, 1].item() == -math.inf


def test_reference_nbest_keeps_the_beam_order():
    """the reference's final beam is sorted by c, best first, with the offline oracle's best"""
    from oracle import ctc_decoder_ref
    rng = np.random.RandomState(2)
    x = rng.randn(12, 5)
    probs = np.exp(x) / np.exp(x).sum(1, keepdims=True)
    logp = np.log(probs)
    beam = nbest_prefix_beam(logp, 6, 4)
    assert len(beam) == 6
    cs = [c for _, c in beam]
    assert cs == sorted(cs, reverse=True)
    best, score = ctc_decoder_ref.prefix_beam_search(probs, 6, 4)
    assert beam[0][0] == tuple(best) and beam[0][1] == -score
