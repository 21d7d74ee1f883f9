"""Host tests of streaming recognition: the C ABI's argument checks (every refusal comes before any
CUDA call), CTC.stream's refusals, and the conv front-end's carry bookkeeping against a float64
CPU convolution of the whole utterance."""
import numpy as np
import pytest
import torch

from speech_b200 import _lib
from speech_b200.models import CTC
from speech_b200.streaming import CTCStream

F = 8   # a fake device pointer: every check below fails before any launch

STREAM_SYMBOLS = ("sb_gru_fwd_h0", "sb_ctc_stream_state_size", "sb_ctc_stream_workspace_size",
                  "sb_ctc_stream_reset", "sb_ctc_stream_step", "sb_ctc_stream_step_shortlist",
                  "sb_ctc_stream_step_lm", "sb_ctc_stream_step_lm_shortlist",
                  "sb_ctc_stream_best")


def test_stream_symbols_are_bound():
    lib = _lib.load()
    for name in STREAM_SYMBOLS:
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


@pytest.mark.parametrize("change,status", [
    ({"ndir": 2}, 3), ({"h0": None}, 1), ({"hb0": None}, 1), ({"gi": None}, 1), ({"y": None}, 1),
    ({"xn": None}, 1), ({"ws": None}, 1), ({"T": 0}, 1), ({"Bp": 12}, 3), ({"Bp": 136}, 3),
    ({"H": 40}, 3), ({"ndir": 3}, 1)])
def test_gru_fwd_h0_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(gi=F, whh=F, bhh=F, h0=F, hb0=F, y=F, xn=F, ws=F, T=5, Bp=8, H=64, ndir=1)
    a.update(change)
    assert lib.sb_gru_fwd_h0(a["gi"], a["whh"], a["bhh"], a["h0"], a["hb0"], a["y"], a["xn"],
                             None, a["ws"], 1 << 20, a["T"], a["Bp"], a["H"], a["ndir"],
                             None) == status


def test_stream_sizes():
    import ctypes
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_ctc_stream_state_size(4, 100, 8, 0, ctypes.byref(n)) == 0
    small = n.value
    assert lib.sb_ctc_stream_state_size(4, 200, 8, 3, ctypes.byref(n)) == 0 and n.value > small
    for args, status in [((0, 100, 8, 0), 1), ((4, 0, 8, 0), 1), ((4, 100, 0, 0), 1),
                         ((4, 100, 33, 0), 3), ((4, 100, 8, -1), 1), ((4, 100, 8, 11), 3)]:
        assert lib.sb_ctc_stream_state_size(*args, ctypes.byref(n)) == status, args
    assert lib.sb_ctc_stream_state_size(4, 100, 8, 0, None) == 1
    assert lib.sb_ctc_stream_workspace_size(4, 10, 8, ctypes.byref(n)) == 0
    assert n.value == 4 * 10 * 17 * 4
    for args in [(0, 10, 8), (4, 0, 8), (4, 10, 0)]:
        assert lib.sb_ctc_stream_workspace_size(*args, ctypes.byref(n)) == 1


@pytest.mark.parametrize("change,status", [
    ({"state": None}, 1), ({"B": 0}, 1), ({"Tm": 0}, 1), ({"K": 0}, 1), ({"K": 33}, 3),
    ({"first": -1}, 1), ({"count": 0}, 1), ({"first": 3, "count": 2}, 1)])
def test_stream_reset_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(state=F, B=4, Tm=100, K=8, first=0, count=4)
    a.update(change)
    assert lib.sb_ctc_stream_reset(a["state"], a["B"], a["Tm"], a["K"], a["first"], a["count"],
                                   None) == status


@pytest.mark.parametrize("change,status", [
    ({"state": None}, 1), ({"labels": None}, 1), ({"lens": None}, 1), ({"scores": None}, 1),
    ({"ovf": None}, 1), ({"B": 0}, 1), ({"Tm": 0}, 1), ({"K": 33}, 3)])
def test_stream_best_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(state=F, B=4, Tm=100, K=8, labels=F, lens=F, scores=F, ovf=F)
    a.update(change)
    assert lib.sb_ctc_stream_best(a["state"], a["B"], a["Tm"], a["K"], a["labels"], a["lens"],
                                  a["scores"], a["ovf"], None) == status


STEP_CHANGES = [
    ({"logp": None}, 1), ({"n": None}, 1), ({"state": None}, 1), ({"ws": None}, 1), ({"B": 0}, 1),
    ({"T": 0}, 1), ({"S": 0}, 1), ({"K": 0}, 1), ({"K": 33}, 3), ({"blank": -1}, 1),
    ({"blank": 29}, 1), ({"Tm": 0}, 1), ({"nbytes": 0}, 4)]


def _fake_lm(**kw):
    d = dict(keys=F, vals=F, logp=F, bow=F, tok=F, cap=64, order=3, num_classes=29, bos=0,
             blank=28, lm_upper=0.0, lm_abs=1.0)
    d.update(kw)
    return _lib.SbNgramLm(**d)


@pytest.mark.parametrize("shortlist", [False, True])
@pytest.mark.parametrize("change,status", STEP_CHANGES)
def test_stream_step_rejects_bad_arguments(change, status, shortlist):
    lib = _lib.load()
    a = dict(logp=F, n=F, B=4, T=10, S=29, K=8, blank=28, Tm=100, state=F, ws=F, nbytes=1 << 40)
    a.update(change)
    fn = lib.sb_ctc_stream_step_shortlist if shortlist else lib.sb_ctc_stream_step
    assert fn(a["logp"], a["n"], a["B"], a["T"], a["S"], a["K"], a["blank"], a["Tm"], a["state"],
              a["ws"], a["nbytes"], None) == status
    fn = lib.sb_ctc_stream_step_lm_shortlist if shortlist else lib.sb_ctc_stream_step_lm
    lm = _fake_lm()
    assert fn(a["logp"], a["n"], a["B"], a["T"], a["S"], a["K"], a["blank"], lm, 0.5, 1.0,
              a["Tm"], a["state"], a["ws"], a["nbytes"], None) == status


@pytest.mark.parametrize("lm_change,w,bonus,status", [
    ({"keys": None}, 0.5, 0.0, 1), ({"tok": None}, 0.5, 0.0, 1), ({}, -1.0, 0.0, 1),
    ({}, float("inf"), 0.0, 1), ({}, 0.5, float("nan"), 1), ({"num_classes": 20}, 0.5, 0.0, 1),
    ({"blank": 3}, 0.5, 0.0, 1), ({"cap": 63}, 0.5, 0.0, 1), ({"order": 0}, 0.5, 0.0, 1),
    ({"order": 11}, 0.5, 0.0, 3), ({"lm_upper": float("inf")}, 0.5, 0.0, 1)])
def test_stream_step_lm_rejects_bad_lm(lm_change, w, bonus, status):
    lib = _lib.load()
    lm = _fake_lm(**lm_change)
    for fn in (lib.sb_ctc_stream_step_lm, lib.sb_ctc_stream_step_lm_shortlist):
        assert fn(F, F, 4, 10, 29, 8, 28, lm, w, bonus, 100, F, F, 1 << 40, None) == status
    assert lib.sb_ctc_stream_step_lm(F, F, 4, 10, 29, 8, 28, None, 0.5, 0.0, 100, F, F, 1 << 40,
                                     None) == 1


# ---- CTC.stream -------------------------------------------------------------------------------
def _model(bidirectional=False, conv=([8, 5, 8, 2], [8, 5, 8, 2])):
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [list(c) for c in conv],
                                       "rnn": {"dim": 16, "bidirectional": bidirectional,
                                               "layers": 1}}}
    return CTC(80, 28, cfg)


def test_stream_refusals():
    from speech_b200.lm import NGramLM
    m = _model()
    with pytest.raises(ValueError, match="num_streams"):
        m.stream(129)
    with pytest.raises(ValueError, match="num_streams"):
        m.stream(0)
    with pytest.raises(ValueError, match="bidirectional"):
        _model(bidirectional=True).stream(2)
    m.parity_mode = True
    with pytest.raises(ValueError, match="parity_mode"):
        m.stream(2)
    m.parity_mode = False
    with pytest.raises(ValueError, match="beam_size"):
        m.stream(2, beam_size=33)
    with pytest.raises(ValueError, match="max_frames"):
        m.stream(2, max_frames=0)
    with pytest.raises(ValueError, match="need an lm"):
        m.stream(2, lm_weight=0.5)
    lm = NGramLM.train([[1, 2, 3]] * 5, 2, num_classes=29, blank=28)
    with pytest.raises(ValueError, match="lm_weight"):
        m.stream(2, lm=lm, lm_weight=-1.0)
    with pytest.raises(ValueError, match="classes"):
        m.stream(2, lm=NGramLM.train([[1, 2, 3]] * 5, 2, num_classes=30, blank=28))


def _host_stream(m, B, max_frames=10 ** 6):
    """a CTCStream with just the conv bookkeeping's state, on the CPU"""
    st = CTCStream.__new__(CTCStream)
    st.model, st.B, st.max_frames, st.dev = m, B, max_frames, torch.device("cpu")
    st.stride = int(np.prod([c.stride[0] for c in m.conv.children()
                             if isinstance(c, torch.nn.Conv2d)]))
    st.carry, st.next = [None] * B, [0] * B
    return st


def _conv64(m, x):
    """the conv stack in float64 on the CPU: (T, F) -> (T', C*F') channel-major"""
    h = x.double()[None, None]
    for c in m.conv.children():
        if isinstance(c, torch.nn.Conv2d):
            h = torch.relu(torch.nn.functional.conv2d(h, c.weight.double(), c.bias.double(),
                                                      stride=c.stride))
    return h[0].transpose(0, 1).reshape(h.shape[2], -1).detach()


@pytest.mark.parametrize("conv", [([8, 5, 8, 2], [8, 5, 8, 2]), ([4, 3, 8, 1], [4, 7, 8, 3]),
                                  ([4, 5, 8, 2],)])
@pytest.mark.parametrize("seed", range(4))
def test_conv_carry_reproduces_whole_utterance(conv, seed):
    m = _model(conv=conv)
    rng = np.random.RandomState(seed)
    B = 3
    lens = rng.randint(0, 90, size=B).tolist()
    feats = [torch.from_numpy(rng.randn(n, 80).astype(np.float32)) for n in lens]
    st = _host_stream(m, B)
    got = [[] for _ in range(B)]
    pos = [0] * B
    while any(p < n for p, n in zip(pos, lens)) or pos == [0] * B:
        chunks = []
        for b in range(B):
            k = int(rng.choice([0, 1, 2, 5, 13]))
            chunks.append(feats[b][pos[b]:pos[b] + k])
            pos[b] = min(pos[b] + k, lens[b])
        xs, counts = st._conv_inputs(chunks)
        for b in range(B):
            if counts[b]:
                got[b].append(_conv64(m, xs[b]).detach()[:counts[b]])
            else:
                assert m.conv_out_size(xs[b].shape[0], 0) <= 0
        st._advance(xs, counts)
        if all(p == n for p, n in zip(pos, lens)):
            break
    for b in range(B):
        total = max(0, m.conv_out_size(lens[b], 0))
        assert st.next[b] == total
        if total:
            # float64 sums over different lengths may group differently: exact up to rounding
            torch.testing.assert_close(torch.cat(got[b]), _conv64(m, feats[b]), rtol=0,
                                       atol=1e-12)


def test_push_past_max_frames_is_refused():
    m = _model()
    st = _host_stream(m, 2, max_frames=5)
    xs, counts = st._conv_inputs([torch.zeros(31, 80), torch.zeros(3, 80)])
    assert counts == [5, 0]
    st._advance(xs, counts)
    with pytest.raises(ValueError, match="max_frames"):
        st._conv_inputs([torch.zeros(4, 80), torch.zeros(0, 80)])
    assert st.next == [5, 0]
    with pytest.raises(ValueError, match="one chunk per stream"):
        st._conv_inputs([torch.zeros(4, 80)])
