"""Host checks (no GPU) of the Viterbi (forced) alignments:

- the float64 references of tests/align_ref.py against brute-force enumeration of every alignment
  on tiny lattices: the best score and the path the tie rule picks;
- the log-sum-exp over the CTC enumeration against the loss oracle, which ties the reference to
  the lattice the loss sums over;
- the C ABI: bound symbols, argument checks (before any launch, with fake pointers) and the
  workspace queries.
"""
import ctypes

import numpy as np
import pytest

import align_ref
from speech_b200 import _lib


def _lse(x):
    x = np.asarray(x, np.float64)
    m = x.max()
    return m + np.log(np.exp(x - m).sum())


@pytest.mark.parametrize("seed", range(12))
def test_ctc_reference_equals_enumeration(seed):
    rng = np.random.RandomState(seed)
    V, blank = 3, 2
    T = rng.randint(1, 7)
    L = rng.randint(0, 4)
    labels = rng.randint(0, 2, L).tolist()
    acts = rng.randn(T, V) * 2
    if seed % 3 == 0:                                  # tie lattice: every value equal
        acts[:] = 0.0
    lp = align_ref.log_softmax(acts)
    path, score = align_ref.ctc_viterbi(lp, labels, blank)
    bpath, bscore = align_ref.ctc_brute_force(lp, labels, blank)
    if bpath is None:
        assert path is None and score == -np.inf
        return
    assert score == bscore
    np.testing.assert_array_equal(path, bpath)
    assert align_ref.ctc_path_errors(path, labels, T) is None
    assert align_ref.ctc_rescore(lp, labels, blank, path) == score


@pytest.mark.parametrize("seed", range(6))
def test_ctc_enumeration_sums_to_the_loss_oracle(seed):
    from oracle import build
    rng = np.random.RandomState(100 + seed)
    V, blank, T = 3, 2, 6
    labels = [rng.randint(0, 2, rng.randint(1, 4)).tolist() for _ in range(3)]
    acts = rng.randn(3, T, V).astype(np.float32)
    costs, _ = build.ctc(acts, np.concatenate(labels), [len(l) for l in labels], [T] * 3, blank,
                         need_grad=False)
    for b in range(3):
        lp = align_ref.log_softmax(acts[b])
        paths = align_ref.ctc_enumerate(lp, labels[b], blank)
        assert abs(_lse([p[0] for p in paths]) + costs[b]) < 1e-5
        assert align_ref.ctc_viterbi(lp, labels[b], blank)[1] <= -costs[b]


def test_ctc_reference_edge_cases():
    lp = align_ref.log_softmax(np.zeros((4, 3)))
    path, score = align_ref.ctc_viterbi(lp, [], 2)
    np.testing.assert_array_equal(path, [-1] * 4)
    assert score == pytest.approx(4 * np.log(1 / 3))
    # two equal labels need a blank between them: 3 frames, not 2
    assert align_ref.ctc_viterbi(lp[:2], [0, 0], 2) == (None, -np.inf)
    path, _ = align_ref.ctc_viterbi(lp[:3], [0, 0], 2)
    np.testing.assert_array_equal(path, [0, -1, 1])
    # on a tie lattice the path stays where it is: labels as early as possible
    path, _ = align_ref.ctc_viterbi(lp, [0, 1], 2)
    np.testing.assert_array_equal(path, [0, 1, -1, -1])
    assert align_ref.ctc_path_errors([0, 1, -1, -2], [0, 1], 3) is None
    assert align_ref.ctc_path_errors([0, 1], [0, 0], 2) is not None
    assert align_ref.ctc_path_errors([1, 0], [0, 1], 2) is not None


@pytest.mark.parametrize("seed", range(12))
def test_rnnt_reference_equals_enumeration(seed):
    rng = np.random.RandomState(seed)
    T = rng.randint(1, 6)
    U = rng.randint(0, 4)
    blank_lp = np.log(rng.uniform(0.05, 1.0, (T, U + 1)))
    label_lp = np.log(rng.uniform(0.05, 1.0, (T, U + 1)))
    if seed % 3 == 0:                                  # tie lattice
        blank_lp[:] = label_lp[:] = np.log(0.25)
    frames, score = align_ref.rnnt_viterbi(blank_lp, label_lp, T, U)
    bframes, bscore = align_ref.rnnt_brute_force(blank_lp, label_lp, T, U)
    assert score == bscore
    np.testing.assert_array_equal(frames, bframes)
    assert align_ref.rnnt_rescore(blank_lp, label_lp, T, frames) == score
    if seed % 3 == 0:                                  # ties emit every label at frame 0
        np.testing.assert_array_equal(frames, [0] * U)


def test_rnnt_enumeration_sums_to_the_loss_oracle():
    """the log-sum-exp over every path equals minus the loss oracle's cost"""
    import itertools
    from oracle import rnnt_ref
    rng = np.random.RandomState(7)
    T, U, V = 4, 3, 5
    lp = align_ref.log_softmax(rng.randn(T, U + 1, V))
    labels = rng.randint(0, V - 1, U)
    cost = rnnt_ref.rnnt_single(lp, labels, V - 1)[0]
    blank_lp = lp[:, :, V - 1]
    label_lp = np.zeros((T, U + 1))
    label_lp[:, :U] = lp[:, np.arange(U), labels]
    scores = []
    for pos in itertools.combinations(range(T - 1 + U), U):
        frames, t = [], 0
        for k in range(T - 1 + U):
            if k in pos:
                frames.append(t)
            else:
                t += 1
        scores.append(align_ref.rnnt_rescore(blank_lp, label_lp, T, frames))
    assert abs(_lse(scores) + cost) < 1e-9
    assert align_ref.rnnt_viterbi(blank_lp, label_lp, T, U)[1] == max(scores)


# ---------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------
def test_align_symbols_are_bound():
    lib = _lib.load()
    for name in ("sb_ctc_viterbi_workspace_size", "sb_ctc_viterbi",
                 "sb_rnnt_viterbi_workspace_size", "sb_rnnt_viterbi"):
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


F = 8   # a fake device pointer: every check below fails before any launch


@pytest.mark.parametrize("change,status", [
    ({"acts": None}, 1), ({"labels": None}, 1), ({"offs": None}, 1), ({"llen": None}, 1),
    ({"alen": None}, 1), ({"path": None}, 1), ({"scores": None}, 1), ({"ws": None}, 1),
    ({"B": 0}, 1), ({"T": 0}, 1), ({"V": 0}, 1), ({"blank": -1}, 1), ({"blank": 29}, 1),
    ({"L": -1}, 1), ({"L": 1024}, 3), ({"nbytes": 0}, 4),
])
def test_ctc_viterbi_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(acts=F, labels=F, offs=F, llen=F, alen=F, B=4, T=50, V=29, blank=28, L=10, path=F,
             scores=F, ws=F, nbytes=1 << 40)
    a.update(change)
    assert lib.sb_ctc_viterbi(a["acts"], a["labels"], a["offs"], a["llen"], a["alen"], a["B"],
                              a["T"], a["V"], a["blank"], a["L"], a["path"], a["scores"], a["ws"],
                              a["nbytes"], None) == status


@pytest.mark.parametrize("change,status", [
    ({"lat": None}, 1), ({"labels": None}, 1), ({"offs": None}, 1), ({"llen": None}, 1),
    ({"alen": None}, 1), ({"frames": None}, 1), ({"scores": None}, 1), ({"ws": None}, 1),
    ({"B": 0}, 1), ({"T": 0}, 1), ({"U1": 0}, 1), ({"U1": 1025}, 3), ({"nbytes": 0}, 4),
])
def test_rnnt_viterbi_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(lat=F, labels=F, offs=F, llen=F, alen=F, B=4, T=50, U1=20, frames=F, scores=F, ws=F,
             nbytes=1 << 40)
    a.update(change)
    assert lib.sb_rnnt_viterbi(a["lat"], a["labels"], a["offs"], a["llen"], a["alen"], a["B"],
                               a["T"], a["U1"], a["frames"], a["scores"], a["ws"], a["nbytes"],
                               None) == status


def _size(fn, *args):
    n = ctypes.c_size_t(0)
    rc = fn(*args, ctypes.byref(n))
    return rc, n.value


def test_viterbi_workspace_sizes():
    lib = _lib.load()
    c = lib.sb_ctc_viterbi_workspace_size
    r = lib.sb_rnnt_viterbi_workspace_size
    assert c(0, 10, 29, 5, ctypes.byref(ctypes.c_size_t())) == 1
    assert c(2, 10, 0, 5, ctypes.byref(ctypes.c_size_t())) == 1
    assert c(2, 10, 29, -1, ctypes.byref(ctypes.c_size_t())) == 1
    assert c(2, 10, 29, 1024, ctypes.byref(ctypes.c_size_t())) == 3
    assert c(2, 10, 29, 5, None) == 1
    assert r(0, 10, 5, ctypes.byref(ctypes.c_size_t())) == 1
    assert r(2, 0, 5, ctypes.byref(ctypes.c_size_t())) == 1
    assert r(2, 10, 0, ctypes.byref(ctypes.c_size_t())) == 1
    assert r(2, 10, 1025, ctypes.byref(ctypes.c_size_t())) == 3
    base = _size(c, 4, 100, 29, 50)[1]
    for args in ((8, 100, 29, 50), (4, 200, 29, 50), (4, 100, 29, 51), (4, 100, 29, 200)):
        assert _size(c, *args) == (0, _size(c, *args)[1]) and _size(c, *args)[1] > base
    prev = 0
    for L in (0, 1, 127, 128, 255, 256, 511, 512, 1023):
        n = _size(c, 4, 100, 29, L)[1]
        assert n >= prev
        prev = n
    base = _size(r, 4, 100, 50)[1]
    for args in ((8, 100, 50), (4, 200, 50), (4, 100, 51), (4, 100, 300)):
        assert _size(r, *args)[0] == 0 and _size(r, *args)[1] > base
    prev = 0
    for U1 in (1, 256, 257, 512, 513, 1024):
        n = _size(r, 4, 100, U1)[1]
        assert n >= prev
        prev = n
