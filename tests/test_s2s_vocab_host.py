"""Routing of the attention decoder's output projection and beam selection by shape
(functions/s2s.py, csrc/s2s_vocab.cu): the predicates the package routes by (the C ABI's, pure
host arithmetic, no GPU needed) against their formulas at and around the boundaries."""
import pytest

from speech_b200.functions import s2s


@pytest.mark.parametrize("H", [4, 16, 64, 128, 512, 1200, 1664])
def test_fc_fused_boundary_is_seven_H(H):
    assert s2s.fc_fused(H, 1)
    assert s2s.fc_fused(H, 7 * H)
    assert not s2s.fc_fused(H, 7 * H + 1)
    assert not s2s.fc_fused(H, 0)
    for C in (1, 7 * H - 1, 7 * H, 7 * H + 1, 8192, 8193, 32000):
        assert s2s.fc_fused(H, C) == (C <= 7 * H), (H, C)


def test_dout_boundary_is_8192_classes():
    assert s2s.dout_fits(8192)
    assert not s2s.dout_fits(8193)


@pytest.mark.parametrize("K", [1, 2, 4, 8, 16, 25, 32])
def test_beam_select_fits_boundary_is_200_kb_of_candidates(K):
    cmax = 200 * 1024 // (8 * K)                  # the most classes whose K*C float64 fit
    assert s2s.beam_select_fits(K, cmax)
    assert not s2s.beam_select_fits(K, cmax + 1)
    assert K * cmax * 8 <= 200 * 1024 < K * (cmax + 1) * 8
    for C in (1, cmax - 1, cmax, cmax + 1, 5000):
        assert s2s.beam_select_fits(K, C) == (K * C * 8 <= 200 * 1024), (K, C)


def test_beam_select_fits_rejects_beams_past_32():
    assert not s2s.beam_select_fits(33, 10)
    assert not s2s.beam_select_fits(0, 10)
    cmax = 200 * 1024 // (8 * 33)
    for C in (1, cmax - 1, cmax, cmax + 1, 5000):
        assert not s2s.beam_select_fits(33, C), C


def test_workspace_queries_of_the_large_vocabulary_kernels():
    import ctypes
    from speech_b200 import _lib
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_s2s_fc_workspace_size(16, 32000, ctypes.byref(n)) == 0
    small = n.value
    assert lib.sb_s2s_fc_workspace_size(1600, 32000, ctypes.byref(n)) == 0
    assert n.value > small >= 16 * 1000 * 12
    assert lib.sb_s2s_fc_workspace_size(0, 10, ctypes.byref(n)) != 0
    assert lib.sb_s2s_beam_split_workspace_size(8, 5000, ctypes.byref(n)) == 0
    assert n.value >= 10 * 16 * 12
    assert lib.sb_s2s_beam_split_workspace_size(8, 0, ctypes.byref(n)) != 0
