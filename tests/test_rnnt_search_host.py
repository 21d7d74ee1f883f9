"""CPU tests of the label-free transducer search's oracle (oracle/rnnt_search_ref.py) and of the
workspace query of its kernels (csrc/rnnt_search.cu)."""
import ctypes

import numpy as np
import pytest

from oracle import decode_static_ref, rnnt_search_ref as ref
from test_rnnt_shortlist_host import tie_lattice


def _lattice(rng, T, U, V, scale=1.0):
    x = rng.randn(T, U, V) * scale
    return (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)


@pytest.mark.parametrize("beam", [1, 2, 4, 8])
@pytest.mark.parametrize("T,U,V,seed", [(6, 4, 5, 0), (12, 6, 9, 1), (20, 8, 11, 2), (5, 1, 7, 3),
                                        (9, 3, 29, 4)])
def test_static_rows_are_decode_static(beam, T, U, V, seed):
    lat = _lattice(np.random.RandomState(seed), T, U, V, scale=2.0)
    for blank in (V - 1, 0):
        want = decode_static_ref.decode_static(lat, beam, blank)
        got = ref.search(ref.static_rows(lat), T, beam, blank, U - 1 if U > 1 else 1, U - 1)
        assert (got[0], got[1]) == want, (blank, got, want)


def test_static_rows_on_the_tie_lattice():
    lat, blank = tie_lattice(V=40)
    for beam in (1, 2, 4):
        want = decode_static_ref.decode_static(lat, beam, blank)
        got = ref.search(ref.static_rows(lat), 2, beam, blank, 1, 1)
        assert (got[0], got[1]) == want, beam


def _label_rows(V, seed):
    """rows that depend on the whole hypothesis (a deterministic random log-softmax per (t, h))"""
    cache = {}

    def row(t, hyp):
        key = (t, hyp)
        if key not in cache:
            rng = np.random.RandomState(abs(hash((seed,) + key)) % (2 ** 31))
            x = rng.randn(V) * 2.0
            cache[key] = (x - np.log(np.exp(x).sum())).astype(np.float32)
        return cache[key]
    return row


@pytest.mark.parametrize("T,V,max_len,seed", [(2, 3, 2, 0), (3, 3, 3, 1), (3, 4, 2, 2),
                                              (4, 3, 3, 3), (1, 5, 2, 4)])
def test_exhaustive_beam_is_the_most_probable_sequence(T, V, max_len, seed):
    row = _label_rows(V, seed)
    blank = V - 1
    want, wlp = ref.best_by_enumeration(row, T, V, blank, max_len)
    n_hyps = sum((V - 1) ** n for n in range(max_len + 1))
    got, glp, _ = ref.search(row, T, n_hyps, blank, max_len, max_len)
    assert got == want
    assert abs(glp - wlp) < 1e-9


def test_per_frame_and_length_caps():
    V, blank = 4, 3
    lat = np.full((3, 8, V), -20.0, dtype=np.float32)
    lat[:, :, 0] = 5.0                         # rows need not be normalised: label 0 pays
    lat[:, :, blank] = -1.0                    # for itself, so more labels score higher
    got, _, _ = ref.search(ref.static_rows(lat), 3, 2, blank, 2, 100)
    assert got == [0] * 6                      # at most 2 per frame
    got, _, _ = ref.search(ref.static_rows(lat), 3, 2, blank, 2, 4)
    assert got == [0] * 4                      # max_len binds


def _pow2(need):
    cap = 64
    while cap < need:
        cap <<= 1
    return cap


@pytest.mark.parametrize("B,T,S,K", [(1, 1, 1, 1), (3, 17, 4, 4), (32, 247, 4, 8), (40, 9, 2, 32)])
def test_workspace_size_query(B, T, S, K):
    from speech_b200 import _lib
    lib = _lib.load()
    n = T * S * K + 2
    c = _pow2(2 * n)
    d = K * (S + 1) + 1
    want = 1024 + 4096 + B * (1184 + 8 * n + 12 * c + 20 * d)
    assert _lib.workspace_size(lib.sb_rnnt_search_workspace_size, B, T, S, K) == want
    out = ctypes.c_size_t(0)
    assert lib.sb_rnnt_search_workspace_size(0, T, S, K, ctypes.byref(out)) != 0
    assert lib.sb_rnnt_search_workspace_size(B, T, 0, K, ctypes.byref(out)) != 0
