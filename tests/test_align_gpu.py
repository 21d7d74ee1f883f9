"""GPU checks of the Viterbi (forced) alignments against the float64 references of
tests/align_ref.py: CTC (sb_ctc_viterbi) at V+1 = 29 and 5000, the Transducer (sb_rnnt_viterbi) on
the resident joint (V+1 = 29) and the slab path (V+1 = 1024), at the benchmarks' shapes and small
ones, then CTC.align / Transducer.align end to end."""
import numpy as np
import pytest
import torch

import align_ref
from speech_b200.functions import ctc as ctc_fn
from speech_b200.functions import transducer as rnnt_fn

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------
# CTC
# ---------------------------------------------------------------------------------------------
def _ctc_case(rng, B, T, V, lo, hi, mixed=True):
    """labels with repeats, an empty transcript, an infeasible utterance, mixed act_lens"""
    blank = V - 1
    labels = [rng.randint(0, min(V - 1, 6) if b % 4 == 1 else V - 1, rng.randint(lo, hi + 1)).tolist()
              for b in range(B)]
    labels[0] = []
    act = [T] * B
    if mixed:
        act = [int(rng.randint(max(1, T // 2), T + 1)) for _ in range(B)]
        act[0] = T
    # infeasible: fewer frames than labels + adjacent repeats
    labels[-1] = [1, 1, 2, 2, 3]
    act[-1] = 6
    return labels, act, blank


def _run_ctc(acts, labels, act, blank):
    flat = torch.tensor([c for l in labels for c in l], dtype=torch.int32)
    llen = torch.tensor([len(l) for l in labels], dtype=torch.int32)
    alen = torch.tensor(act, dtype=torch.int32)
    path, scores = ctc_fn.ctc_viterbi(acts, flat, alen, llen, blank)
    costs, _ = ctc_fn.ctc_costs_and_grads(acts, flat, alen, llen, blank, need_grad=False)
    return path.cpu().numpy(), scores.cpu().numpy(), costs.cpu().numpy()


def _check_ctc(acts, labels, act, blank, exact_paths):
    path, scores, costs = _run_ctc(acts, labels, act, blank)
    path2, scores2, _ = _run_ctc(acts, labels, act, blank)
    np.testing.assert_array_equal(path, path2)                # two calls are bit-identical
    np.testing.assert_array_equal(scores, scores2)
    lp_all = align_ref.log_softmax(acts.double().cpu().numpy())
    T = acts.shape[1]
    for b, lab in enumerate(labels):
        lp = lp_all[b, :act[b]]
        rpath, rscore = align_ref.ctc_viterbi(lp, lab, blank)
        if rpath is None:
            assert scores[b] == -np.inf, b
            assert (path[b] == -2).all(), b
            continue
        assert align_ref.ctc_path_errors(path[b], lab, act[b]) is None, b
        assert (path[b, act[b]:] == -2).all() and path.shape[1] == T
        rescored = align_ref.ctc_rescore(lp, lab, blank, path[b, :act[b]])
        assert abs(rescored - rscore) < 1e-3, (b, rescored, rscore)
        assert abs(scores[b] - rscore) < 1e-3, (b, scores[b], rscore)
        assert scores[b] <= -costs[b] + 1e-3 * max(1.0, abs(costs[b])), b
        if exact_paths:
            np.testing.assert_array_equal(path[b, :act[b]], rpath, err_msg=str(b))
    return path, scores


# long transcripts: S = 2L+1 states over 256 threads, 2, 4 and 8 states per thread
CTC_LONG = [(29, 5, 500, 150, 250), (29, 5, 900, 300, 450), (29, 5, 2500, 600, 1023)]


@pytest.mark.parametrize("V,B,T,lo,hi", [(29, 6, 40, 1, 12), (29, 64, 247, 40, 120),
                                         (5000, 6, 40, 1, 12), (5000, 64, 247, 40, 120),
                                         (5000, 5, 900, 300, 450)] + CTC_LONG)
def test_ctc_viterbi_random(cuda_lib, V, B, T, lo, hi):
    rng = np.random.RandomState(V + T)
    labels, act, blank = _ctc_case(rng, B, T, V, lo, hi)
    acts = torch.from_numpy(rng.randn(B, T, V).astype(np.float32) * 2).cuda()
    _check_ctc(acts, labels, act, blank, exact_paths=False)


@pytest.mark.parametrize("V,B,T,lo,hi", [(29, 8, 60, 1, 12), (29, 64, 247, 40, 120),
                                         (5000, 64, 247, 40, 120)] + CTC_LONG)
def test_ctc_viterbi_peaked_paths_equal_the_reference(cuda_lib, V, B, T, lo, hi):
    """logits peaked along a random alignment of each transcript"""
    rng = np.random.RandomState(7 + V)
    labels, act, blank = _ctc_case(rng, B, T, V, lo, hi)
    x = rng.randn(B, T, V).astype(np.float32)
    for b, lab in enumerate(labels):
        if not lab or len(lab) > act[b] // 2:
            continue
        cuts = np.sort(rng.choice(np.arange(1, act[b]), len(lab), replace=False))
        for j, c in enumerate(lab):
            x[b, cuts[j]:cuts[j] + 1, c] += 8.0
    acts = torch.from_numpy(x).cuda()
    _check_ctc(acts, labels, act, blank, exact_paths=True)


@pytest.mark.parametrize("V,B,T,lo,hi", [(29, 8, 40, 1, 12), (29, 64, 247, 40, 120),
                                         (5000, 16, 247, 40, 120)] + CTC_LONG)
def test_ctc_viterbi_tie_lattice(cuda_lib, V, B, T, lo, hi):
    """all-zero logits: every path sums the same values in the same order, so scores tie exactly
    and only the tie rule picks the path"""
    rng = np.random.RandomState(11)
    labels, act, blank = _ctc_case(rng, B, T, V, lo, hi)
    acts = torch.zeros(B, T, V, device="cuda")
    path, scores = _check_ctc(acts, labels, act, blank, exact_paths=True)
    by_len = {}
    for b in range(B):
        if scores[b] != -np.inf:
            by_len.setdefault(act[b], set()).add(float(scores[b]))
    assert all(len(v) == 1 for v in by_len.values()), by_len


# ---------------------------------------------------------------------------------------------
# Transducer
# ---------------------------------------------------------------------------------------------
def _rnnt_case(rng, B, T, H, V1, lo, hi, scale=1.0, zero_fc2=False):
    blank = V1 - 1
    labels = [rng.randint(0, V1 - 1, rng.randint(lo, hi + 1)).tolist() for _ in range(B)]
    labels[1] = []
    U1 = max(len(l) for l in labels) + 1
    ymat = np.zeros((B, U1 - 1), np.int64)
    for b, l in enumerate(labels):
        ymat[b, :len(l)] = l
    fx = torch.from_numpy(rng.randn(B, T, H).astype(np.float32) * scale).cuda()
    fy = torch.from_numpy(rng.randn(B, U1, H).astype(np.float32) * scale).cuda()
    fc2 = torch.nn.Linear(H, V1).cuda()
    with torch.no_grad():
        fc2.weight.copy_(torch.from_numpy(rng.randn(V1, H).astype(np.float32) / np.sqrt(H)))
        fc2.bias.copy_(torch.from_numpy(rng.randn(V1).astype(np.float32)))
        if zero_fc2:
            fc2.weight.zero_()
            fc2.bias.zero_()
    x_lens = [int(rng.randint(max(1, T // 2), T + 1)) for _ in range(B)]
    x_lens[0] = T
    return labels, torch.from_numpy(ymat), fx, fy, fc2, x_lens, blank


def _check_rnnt(labels, ymat, fx, fy, fc2, x_lens, blank, exact_paths):
    B = fx.shape[0]
    flat = torch.tensor([c for l in labels for c in l], dtype=torch.int32)
    ylen = torch.tensor([len(l) for l in labels], dtype=torch.int32)
    xlen = torch.tensor(x_lens, dtype=torch.int32)
    frames, scores = rnnt_fn.rnnt_viterbi(fx, fy, fc2, ymat, flat, xlen, ylen, blank)
    frames2, scores2 = rnnt_fn.rnnt_viterbi(fx, fy, fc2, ymat, flat, xlen, ylen, blank)
    assert torch.equal(frames, frames2) and torch.equal(scores, scores2)
    with torch.no_grad():
        lp = rnnt_fn.joint_log_probs(fx, fy, fc2, ymat.cuda(), blank)     # (B, T, U1, V1)
        blank_lp = lp[..., blank].double().cpu().numpy()
        U1 = lp.shape[2]
        idx = torch.cat([ymat.cuda(), ymat.new_zeros(B, 1).cuda()], 1)
        label_lp = torch.gather(lp, 3, idx[:, None, :, None].expand(B, lp.shape[1], U1, 1))
        label_lp = label_lp[..., 0].double().cpu().numpy()
        costs, _ = rnnt_fn.rnnt_costs_and_grads(lp, flat, xlen, ylen, blank, need_grad=False)
    del lp
    frames, scores, costs = frames.cpu().numpy(), scores.cpu().numpy(), costs.cpu().numpy()
    for b, lab in enumerate(labels):
        T, U = x_lens[b], len(lab)
        rframes, rscore = align_ref.rnnt_viterbi(blank_lp[b], label_lp[b], T, U)
        f = frames[b, :U]
        assert (frames[b, U:] == -1).all(), b
        assert (np.diff(f) >= 0).all() and (f >= 0).all() and (f < T).all(), b
        rescored = align_ref.rnnt_rescore(blank_lp[b], label_lp[b], T, f)
        assert abs(rescored - rscore) < 1e-3, (b, rescored, rscore)
        assert abs(scores[b] - rscore) < 1e-3, (b, scores[b], rscore)
        assert scores[b] <= -costs[b] + 1e-3 * max(1.0, abs(costs[b])), b
        if exact_paths:
            np.testing.assert_array_equal(f, rframes, err_msg=str(b))
    return frames, scores


RNNT_SHAPES = [(29, 6, 30, 64, 1, 10), (29, 32, 247, 256, 40, 100),
               (1024, 6, 30, 64, 1, 10), (1024, 32, 247, 256, 40, 100),
               # long transcripts: U+1 columns over 256 threads, 2 and 4 columns per thread
               (29, 4, 400, 64, 280, 320), (29, 3, 300, 64, 600, 1000),
               (1024, 2, 200, 64, 280, 320)]


@pytest.mark.parametrize("V1,B,T,H,lo,hi", RNNT_SHAPES)
def test_rnnt_viterbi_random(cuda_lib, V1, B, T, H, lo, hi):
    rng = np.random.RandomState(V1 + T)
    _check_rnnt(*_rnnt_case(rng, B, T, H, V1, lo, hi), exact_paths=False)


@pytest.mark.parametrize("V1,B,T,H,lo,hi", RNNT_SHAPES)
def test_rnnt_viterbi_peaked_paths_equal_the_reference(cuda_lib, V1, B, T, H, lo, hi):
    rng = np.random.RandomState(3 + V1)
    _check_rnnt(*_rnnt_case(rng, B, T, H, V1, lo, hi, scale=6.0), exact_paths=True)


@pytest.mark.parametrize("V1,B,T,H,lo,hi", RNNT_SHAPES)
def test_rnnt_viterbi_tie_lattice(cuda_lib, V1, B, T, H, lo, hi):
    """zero fc2: every node holds the same two values, so every path of an utterance sums the same
    sequence; ties take the blank arc, which emits every label at frame 0"""
    rng = np.random.RandomState(5)
    case = _rnnt_case(rng, B, T, H, V1, lo, hi, zero_fc2=True)
    frames, scores = _check_rnnt(*case, exact_paths=True)
    labels = case[0]
    for b, lab in enumerate(labels):
        assert (frames[b, :len(lab)] == 0).all()


def test_rnnt_viterbi_without_frames(cuda_lib):
    rng = np.random.RandomState(1)
    labels, ymat, fx, fy, fc2, x_lens, blank = _rnnt_case(rng, 3, 10, 64, 29, 1, 4)
    x_lens[2] = 0
    flat = torch.tensor([c for l in labels for c in l], dtype=torch.int32)
    frames, scores = rnnt_fn.rnnt_viterbi(fx, fy, fc2, ymat, flat,
                                          torch.tensor(x_lens, dtype=torch.int32),
                                          torch.tensor([len(l) for l in labels], dtype=torch.int32),
                                          blank)
    assert scores[2].item() == -np.inf and (frames[2] == -1).all()
    assert np.isfinite(scores[:2].cpu().numpy()).all()


# ---------------------------------------------------------------------------------------------
# the models
# ---------------------------------------------------------------------------------------------
def _ctc_model(exact):
    from speech_b200.models import CTC
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                       "rnn": {"dim": 32, "bidirectional": True, "layers": 2}}}
    m = CTC(40, 28, cfg).cuda()
    m.set_eval()
    return m


def _spans_ok(spans, n, frames):
    assert len(spans) == n
    prev = -1
    for first, last in spans:
        assert prev < first <= last < frames
        prev = last


@pytest.mark.parametrize("exact", [False, True])
def test_ctc_align(cuda_lib, exact):
    m = _ctc_model(exact)
    rng = np.random.RandomState(2)
    lens = [200, 120, 160, 90]
    inputs = [rng.randn(n, 40).astype(np.float32) for n in lens]
    labels = [rng.randint(0, 28, 12).tolist(), [], [3, 3, 3, 4], [5] * 40]
    spans, scores = m.align((inputs, labels), return_scores=True)
    x, y, x_lens, y_lens = m.collate(inputs, labels)
    with torch.no_grad():
        out = m((inputs, labels))
    lp = align_ref.log_softmax(out.double().cpu().numpy())
    for b, lab in enumerate(labels):
        T_b = int(x_lens[b])
        assert T_b == (m.conv_out_size(lens[b], 0) if exact else out.shape[1])
        _, rscore = align_ref.ctc_viterbi(lp[b, :T_b], lab, m.blank)
        if rscore == -np.inf:
            assert spans[b] is None and scores[b] == -np.inf
            continue
        _spans_ok(spans[b], len(lab), T_b)
        assert abs(scores[b] - rscore) < 1e-3
    assert spans[3] is None                     # 40 equal labels need 79 frames
    assert spans[1] == []
    assert m.align(([inputs[1]], [[]])) == [[]]
    # timestamps of a hypothesis: align over the decoder's output
    hyps = m.infer((inputs, labels))
    spans = m.align((inputs, hyps))
    for b, h in enumerate(hyps):
        _spans_ok(spans[b], len(h), int(x_lens[b]))


def _rnnt_model(exact, V1):
    from speech_b200.models import Transducer
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": [[4, 5, 5, 2]], "rnn": {"dim": 64, "bidirectional": True,
                                                      "layers": 1}},
           "decoder": {"embedding_dim": 16, "layers": 1}}
    m = Transducer(40, V1 - 1, cfg).cuda()
    m.set_eval()
    return m


@pytest.mark.parametrize("exact,V1", [(False, 29), (True, 29), (True, 1024)])
def test_transducer_align(cuda_lib, exact, V1):
    m = _rnnt_model(exact, V1)
    rng = np.random.RandomState(4)
    lens = [150, 60, 110]
    inputs = [rng.randn(n, 40).astype(np.float32) for n in lens]
    labels = [rng.randint(0, V1 - 1, 20).tolist(), [], rng.randint(0, V1 - 1, 7).tolist()]
    frames, scores = m.align((inputs, labels), return_scores=True)
    x, y, x_lens, y_lens = m.collate(inputs, labels)
    for b, lab in enumerate(labels):
        T_b = int(x_lens[b])
        f = np.array(frames[b])
        assert len(f) == len(lab) and np.isfinite(scores[b])
        assert (np.diff(f) >= 0).all() and ((f >= 0) & (f < T_b)).all()
    # in the exact-lengths mode an utterance aligns alone as it does in its batch
    if exact:
        for b in range(3):
            fb, sb = m.align(([inputs[b]], [labels[b]]), return_scores=True)
            # the encoder's GEMMs may round a row differently in a smaller batch
            assert len(fb[0]) == len(labels[b])
            assert abs(sb[0] - scores[b]) < 1e-3 + 1e-4 * abs(scores[b])
    hyps = m.recognize(inputs, beam_size=2)
    hframes = m.align((inputs, hyps))
    for b, h in enumerate(hyps):
        f = np.array(hframes[b])
        assert len(f) == len(h) and (np.diff(f) >= 0).all() and ((f >= 0) & (f < int(x_lens[b]))).all()
