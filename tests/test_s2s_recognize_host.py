"""Seq2Seq.recognize without a GPU: its argument checks (all before any launch), and the batched
beam-search entry points of the C ABI (csrc/s2s.cu) - their workspace arithmetic and the
arguments they refuse before launching anything."""
import ctypes

import numpy as np
import pytest

from speech_b200 import _lib
from speech_b200.functions import s2s

ERR_INVALID = 1


def _model(V=11):
    from speech_b200.models import Seq2Seq
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                       "rnn": {"dim": 32, "bidirectional": True, "layers": 1}},
           "decoder": {"embedding_dim": 32, "layers": 1}}
    return Seq2Seq(40, V, cfg)


def _inputs():
    return [np.zeros((60, 40), np.float32), np.zeros((50, 40), np.float32)]


@pytest.mark.parametrize("kw", [
    {"beam_size": 0}, {"beam_size": 33}, {"beam_size": -1},
    {"max_len": 0}, {"max_len": -5},
    {"start_tok": 11}, {"start_tok": -1},
    {"end_tok": 10}, {"end_tok": -1}, {"end_tok": 11},
])
def test_recognize_rejects_bad_arguments_before_any_launch(kw):
    # a CPU model: anything past the checks would fail on the missing device, not with ValueError
    with pytest.raises(ValueError):
        _model().recognize(_inputs(), **kw)


def test_recognize_rejects_an_empty_batch():
    with pytest.raises(ValueError):
        _model().recognize([])


def test_beam_width_limit_is_the_kernels():
    assert s2s.BEAM_MAX_WIDTH == 32
    assert s2s.beam_select_fits(32, 10) and not s2s.beam_select_fits(33, 10)


def test_batched_symbols_are_bound():
    lib = _lib.load()
    for name in ("sb_s2s_beam_init_batch", "sb_s2s_beam_select_batch",
                 "sb_s2s_beam_select_split_batch", "sb_s2s_beam_split_workspace_size_batch",
                 "sb_s2s_beam_gather_batch"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


@pytest.mark.parametrize("K,C", [(1, 7), (4, 50), (8, 5000), (32, 200), (8, 32000)])
@pytest.mark.parametrize("B", [1, 2, 5, 16, 1000])
def test_batched_split_workspace_is_B_times_one_utterance(K, C, B):
    lib = _lib.load()
    one, many = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert lib.sb_s2s_beam_split_workspace_size(K, C, ctypes.byref(one)) == 0
    assert lib.sb_s2s_beam_split_workspace_size_batch(K, C, B, ctypes.byref(many)) == 0
    assert many.value == B * one.value
    # what the carve needs: [B][tiles][2K] float64 + int32, [B][tiles] int32
    tiles = -(-K * C // 4096)
    assert many.value >= B * tiles * (2 * K * 12 + 4)


@pytest.mark.parametrize("B", [0, -1])
def test_batched_entry_points_reject_empty_batches(B):
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_s2s_beam_split_workspace_size_batch(8, 100, B, ctypes.byref(n)) == ERR_INVALID
    p = 256                     # never dereferenced: the checks return before any launch
    assert lib.sb_s2s_beam_init_batch(p, p, 10, p, 4, 0, p, B, None) == ERR_INVALID
    assert lib.sb_s2s_beam_select_batch(p, p, p, p, p, p, p, 4, 10, 9, 0, 5, 50, 30, p, B,
                                        None) == ERR_INVALID
    assert lib.sb_s2s_beam_select_split_batch(p, p, p, p, p, p, p, 4, 10, 9, 0, 5, 50, 30, p, B,
                                              p, 1 << 20, None) == ERR_INVALID
    assert lib.sb_s2s_beam_gather_batch(p, p, p, p, p, p, p, p, 4, 32, 40, B, None) == ERR_INVALID


def test_batched_entry_points_need_the_stop_words():
    lib = _lib.load()
    p = 256
    assert lib.sb_s2s_beam_init_batch(p, p, 10, p, 4, 0, None, 2, None) == ERR_INVALID
    assert lib.sb_s2s_beam_select_batch(p, p, p, p, p, p, p, 4, 10, 9, 0, 5, 50, 30, None, 2,
                                        None) == ERR_INVALID
    assert lib.sb_s2s_beam_select_split_batch(p, p, p, p, p, p, p, 4, 10, 9, 0, 5, 50, 30, None,
                                              2, p, 1 << 20, None) == ERR_INVALID


def test_beam_state_ends_in_the_final_score():
    # done (int32) at 0, out_len (int32) at 4, the float64 score in the last 8 bytes
    n = _lib.workspace_size(_lib.load().sb_s2s_beam_state_size)
    assert n % 8 == 0 and n >= 8 + 32 * 8 + 8
