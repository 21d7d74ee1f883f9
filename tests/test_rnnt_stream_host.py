"""Host tests of Transducer streaming: sb_rnnt_search_reset's argument checks (every refusal comes
before any CUDA call), Transducer.stream's refusals (all before the CUDA check), the refusal of a
push past max_frames, and the end-of-push copy of odd streams' beam states into block 0 against a
per-stream loop."""
import numpy as np
import pytest
import torch

from speech_b200 import _lib
from speech_b200.models import Transducer
from speech_b200.streaming import TransducerStream
from speech_b200.transducer_decoders import StreamSearch, settle_beams

F = 8   # a fake device pointer: every check below fails before any launch


def test_reset_symbol_is_bound():
    lib = _lib.load()
    assert "sb_rnnt_search_reset" in _lib.SIGNATURES
    assert lib.sb_rnnt_search_reset.argtypes == _lib.SIGNATURES["sb_rnnt_search_reset"][1]


@pytest.mark.parametrize("change,status", [
    ({"slot_lens": None}, 1), ({"ws": None}, 1), ({"B": 0}, 1), ({"T": 0}, 1), ({"S": 0}, 1),
    ({"K": 0}, 1), ({"first": -1}, 1), ({"count": 0}, 1), ({"count": -1}, 1),
    ({"first": 3, "count": 2}, 1), ({"first": 4, "count": 1}, 1), ({"nbytes": 1024}, 4),
    ({"K": 33}, 3)])
def test_reset_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(slot_lens=F, B=4, T=100, S=4, K=8, first=0, count=4, ws=F, nbytes=1 << 40)
    a.update(change)
    assert lib.sb_rnnt_search_reset(a["slot_lens"], a["B"], a["T"], a["S"], a["K"], a["first"],
                                    a["count"], a["ws"], a["nbytes"], None) == status


def test_reset_accepts_the_exact_workspace_size():
    import ctypes
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_rnnt_search_workspace_size(4, 3000, 4, 8, ctypes.byref(n)) == 0
    # the header's formula: 5120 + B * (1184 + 8 n + 12 c + 20 d)
    nodes = 3000 * 4 * 8 + 2
    c = 64
    while c < 2 * nodes:
        c *= 2
    assert n.value == 5120 + 4 * (1184 + 8 * nodes + 12 * c + 20 * (8 * 5 + 1)) == \
        5120 + 4 * 3915748
    # one byte short is refused before the (null-stream) launch
    assert lib.sb_rnnt_search_reset(F, 4, 3000, 4, 8, 1, 2, F, n.value - 1, None) == 4


# ---- Transducer.stream ------------------------------------------------------------------------
def _model(bidirectional=False, V=28):
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                       "rnn": {"dim": 16, "bidirectional": bidirectional,
                                               "layers": 1}},
           "decoder": {"embedding_dim": 8, "layers": 1}}
    return Transducer(80, V, cfg)


def test_stream_refusals_come_before_the_cuda_check():
    from speech_b200.lm import NGramLM
    m = _model()                                     # on the CPU: a valid call raises after these
    for kw, match in [(dict(num_streams=129), "num_streams"), (dict(num_streams=0), "num_streams"),
                      (dict(beam_size=0), "beam_size"), (dict(beam_size=33), "beam_size"),
                      (dict(max_symbols_per_frame=0), "max_symbols_per_frame"),
                      (dict(max_frames=0), "max_frames"), (dict(max_len=0), "max_len"),
                      (dict(lm_weight=0.5), "need an lm")]:
        args = dict(num_streams=2)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            m.stream(**args)
    with pytest.raises(ValueError, match="bidirectional"):
        _model(bidirectional=True).stream(2)
    lm = NGramLM.train([[1, 2, 3]] * 5, 2, num_classes=29, blank=28)
    with pytest.raises(ValueError, match="lm_weight"):
        m.stream(2, lm=lm, lm_weight=-1.0)
    with pytest.raises(ValueError, match="classes"):
        m.stream(2, lm=NGramLM.train([[1, 2, 3]] * 5, 2, num_classes=30, blank=28))
    with pytest.raises(_lib.SpeechB200Error, match="CUDA"):
        m.stream(2, lm=lm, lm_weight=0.5, max_len=7)


def _host_stream(m, B, max_frames=10 ** 6):
    """a TransducerStream with just the conv bookkeeping's state, on the CPU"""
    st = TransducerStream.__new__(TransducerStream)
    st.model, st.B, st.max_frames, st.dev = m, B, max_frames, torch.device("cpu")
    st.stride = int(np.prod([c.stride[0] for c in m.conv.children()
                             if isinstance(c, torch.nn.Conv2d)]))
    st.carry, st.next = [None] * B, [0] * B
    return st


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
    with pytest.raises(ValueError, match="frames, features"):
        st._conv_inputs([torch.zeros(4), torch.zeros(0, 80)])
    # the search refuses on its own too, before any launch
    s = StreamSearch.__new__(StreamSearch)
    s.B, s.Tm, s.frames = 2, 5, [5, 0]
    with pytest.raises(ValueError, match="max_frames"):
        s.push([1, 0])
    with pytest.raises(ValueError, match="one frame count per stream"):
        s.push([1])
    assert s.frames == [5, 0]


@pytest.mark.parametrize("B,K,S,layers", [(1, 1, 1, 1), (5, 4, 2, 2), (3, 8, 4, 1)])
def test_settle_beams_equals_a_per_stream_copy(B, K, S, layers):
    g = torch.Generator().manual_seed(B * 100 + K)
    H, Hj, R = 6, 8, B * K
    hid = torch.randn(S + 2, layers, R, H, generator=g)
    fy = torch.randn(S + 2, R, Hj, generator=g)
    counts = torch.randint(0, 5, (B,), generator=g, dtype=torch.int32)
    counts[0] = 3                                    # at least one odd stream
    want_hid, want_fy = hid.clone(), fy.clone()
    for b in range(B):
        if int(counts[b]) % 2:
            rows = slice(b * K, (b + 1) * K)
            want_hid[0, :, rows] = hid[S + 1, :, rows]
            want_fy[0, rows] = fy[S + 1, rows]
    settle_beams((hid, None, fy), counts, K)
    assert torch.equal(hid, want_hid) and torch.equal(fy, want_fy)
