"""Host tests of the lookahead convolution: the C ABI's bindings and argument checks (every refusal
comes before any CUDA call), the model's configuration, parameters and pickles, and the streams'
emitted and pending frame counts against a closed-form restatement."""
import ctypes
import os
import pickle

import numpy as np
import pytest
import torch

from speech_b200 import _lib
from speech_b200.models import CTC, Seq2Seq, Transducer
from speech_b200.streaming import lookahead_counts

F = 8   # a fake device pointer: every check below fails before any launch

SYMBOLS = ("sb_lookahead_fwd", "sb_lookahead_bwd_workspace_size", "sb_lookahead_bwd")


def test_symbols_are_bound():
    lib = _lib.load()
    for name in SYMBOLS:
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1], name


BAD_SHAPES = [({"T": 0}, 1), ({"tau": 0}, 3), ({"tau": 33}, 3), ({"Bp": 12}, 3), ({"Bp": 136}, 3),
              ({"Bp": 0}, 3), ({"Hp": 12}, 3), ({"Hp": 0}, 3)]


@pytest.mark.parametrize("change,status", BAD_SHAPES + [
    ({"h": None}, 1), ({"w": None}, 1), ({"r": None, "rb": None}, 1)])
def test_fwd_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(h=F, w=F, r=F, rb=F, T=5, Bp=8, Hp=64, tau=3)
    a.update(change)
    assert lib.sb_lookahead_fwd(a["h"], a["w"], None, a["r"], a["rb"], a["T"], a["Bp"], a["Hp"],
                                a["tau"], None) == status


@pytest.mark.parametrize("change,status", BAD_SHAPES + [
    ({"dr": None}, 1), ({"h": None}, 1), ({"w": None}, 1), ({"dh": None}, 1), ({"dw": None}, 1),
    ({"ws": None}, 1), ({"nbytes": -1}, 4)])
def test_bwd_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(dr=F, h=F, w=F, dh=F, dw=F, ws=F, T=5, Bp=8, Hp=64, tau=3, nbytes=0)
    a.update(change)
    if a["nbytes"] == 0:
        a["nbytes"] = 1 << 30
    elif a["nbytes"] == -1:
        a["nbytes"] = _lib.workspace_size(lib.sb_lookahead_bwd_workspace_size, 5, 8, 64, 3) - 1
    assert lib.sb_lookahead_bwd(a["dr"], a["h"], a["w"], None, a["dh"], a["dw"], a["ws"],
                                a["nbytes"], a["T"], a["Bp"], a["Hp"], a["tau"], None) == status


@pytest.mark.parametrize("change,status", BAD_SHAPES)
def test_workspace_size_rejects_bad_arguments(change, status):
    lib = _lib.load()
    a = dict(T=5, Bp=8, Hp=64, tau=3)
    a.update(change)
    n = ctypes.c_size_t(0)
    assert lib.sb_lookahead_bwd_workspace_size(a["T"], a["Bp"], a["Hp"], a["tau"],
                                               ctypes.byref(n)) == status
    assert lib.sb_lookahead_bwd_workspace_size(5, 8, 64, 3, None) == 1


def test_workspace_size_grows_with_the_shape():
    lib = _lib.load()
    q = lib.sb_lookahead_bwd_workspace_size
    n = _lib.workspace_size(q, 247, 64, 1024, 5)
    assert n > 0
    assert _lib.workspace_size(q, 247, 64, 1024, 20) > n
    assert _lib.workspace_size(q, 500, 64, 1024, 5) > n


# ---- models ------------------------------------------------------------------------------------
def _cfg(tau=None, bidirectional=False, dim=40):
    enc = {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
           "rnn": {"dim": dim, "bidirectional": bidirectional, "layers": 2}}
    if tau is not None:
        enc["lookahead"] = tau
    return {"dropout": 0.0, "encoder": enc,
            "decoder": {"embedding_dim": 16, "layers": 1, "ctc_weight": 0.3}}


FAMILIES = {"ctc": lambda c: CTC(80, 27, c), "rnnt": lambda c: Transducer(80, 27, c),
            "s2s": lambda c: Seq2Seq(80, 29, c)}


@pytest.mark.parametrize("tau", [-1, 33, 2.0, True, "3"])
def test_lookahead_out_of_range_is_refused(tau):
    with pytest.raises(ValueError, match="lookahead"):
        CTC(80, 27, _cfg(tau))


@pytest.mark.parametrize("family", list(FAMILIES))
def test_lookahead_with_a_bidirectional_encoder_is_refused(family):
    with pytest.raises(ValueError, match="unidirectional"):
        FAMILIES[family](_cfg(2, bidirectional=True))
    FAMILIES[family](_cfg(0, bidirectional=True))          # 0: no layer, nothing to refuse


@pytest.mark.parametrize("family", list(FAMILIES))
def test_no_key_keeps_the_state_dict(family):
    torch.manual_seed(0)
    a = FAMILIES[family](_cfg())
    torch.manual_seed(0)
    b = FAMILIES[family](_cfg(0))
    assert a.lookahead is None and b.lookahead is None
    assert list(a.state_dict()) == list(b.state_dict())
    assert not any(k.startswith("lookahead") for k in a.state_dict())
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("tau", [1, 5])
def test_lookahead_leaves_every_other_parameter_as_it_was(family, tau):
    torch.manual_seed(3)
    plain = FAMILIES[family](_cfg())
    torch.manual_seed(3)
    la = FAMILIES[family](_cfg(tau))
    sd_plain, sd_la = plain.state_dict(), la.state_dict()
    assert list(sd_la) == list(sd_plain) + ["lookahead.weight"]
    for k, v in sd_plain.items():
        assert torch.equal(v, sd_la[k]), k
    assert sd_la["lookahead.weight"].shape == (40, 1, tau + 1)
    conv = la.lookahead
    assert conv.groups == 40 and conv.bias is None and conv.kernel_size == (tau + 1,)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                      "ctc_before_lookahead.pt")


def _load_old():
    """a CTC model (unidirectional, GRU-24) pickled whole by torch.save before the lookahead
    existed: no `lookahead` module, no lookahead configuration"""
    return torch.load(GOLDEN, weights_only=False)


def test_pickle_from_before_the_layer_loads_with_no_lookahead():
    m = _load_old()
    assert m.lookahead is None
    assert "lookahead" not in dict(m.named_modules())
    assert sorted(m.state_dict()) == ["conv.0.bias", "conv.0.weight", "fc.fc.bias",
                                      "fc.fc.weight", "rnn.bias_hh_l0", "rnn.bias_ih_l0",
                                      "rnn.weight_hh_l0", "rnn.weight_ih_l0"]
    la = CTC(80, 27, _cfg(4))
    la2 = pickle.loads(pickle.dumps(la))
    assert la2.lookahead is not None
    assert torch.equal(la2.lookahead.weight, la.lookahead.weight)


def test_pickle_from_before_the_layer_encodes_without_one(monkeypatch):
    """the old model's forward reaches the GRU stack with lookahead=None (the device work itself
    is replaced: there is no CPU path)"""
    from speech_b200 import ops
    seen = []
    monkeypatch.setattr(_lib, "require_cuda", lambda t, name: None)
    monkeypatch.setattr(ops, "conv_stack", lambda x, conv, training: x)
    monkeypatch.setattr(ops, "gru_stack_logits",
                        lambda x, rnn, fc, dropout=0.0, lens=None, lookahead=None:
                        seen.append(("logits", lookahead)) or x)
    monkeypatch.setattr(ops, "gru_stack", lambda x, rnn, dropout=0.0, lens=None, lookahead=None:
                        seen.append(("stack", lookahead)) or x)
    m = _load_old()
    x = torch.zeros(1, 4, 8)
    m.encode_logits(x)
    m.encode(x)
    assert seen == [("logits", None), ("stack", None)]


def test_the_layer_can_be_removed():
    m = CTC(80, 27, _cfg(3))
    m.lookahead = None
    assert m.lookahead is None and "lookahead.weight" not in m.state_dict()
    plain = CTC(80, 27, _cfg())
    plain.lookahead = None                 # nothing to remove: still no layer
    assert plain.lookahead is None
    with pytest.raises(TypeError):
        plain.lookahead = 3


# ---- stream bookkeeping ------------------------------------------------------------------------
def _restated(total, tau, ended):
    """frames searched and held back once a stream has produced `total` encoder frames"""
    if ended:
        return total, 0
    held = min(tau, total)
    return total - held, held


@pytest.mark.parametrize("tau", [1, 2, 5, 32])
@pytest.mark.parametrize("seed", range(4))
def test_emitted_and_pending_counts(tau, seed):
    rng = np.random.RandomState(seed)
    B = 4
    pending, searched, total = [0] * B, [0] * B, [0] * B
    ended = set()
    for step in range(60):
        counts = [0 if b in ended else int(rng.choice([0, 0, 1, 2, tau - 1 if tau > 1 else 0,
                                                       tau, 3 * tau]))
                  for b in range(B)]
        ends = set()
        if step % 17 == 16:
            ends = {int(rng.randint(B))} - ended
            counts = [0] * B
        emit, pending = lookahead_counts(pending, counts, tau, ends)
        ended |= ends
        for b in range(B):
            total[b] += counts[b]
            searched[b] += emit[b]
            assert 0 <= pending[b] <= (0 if b in ended else tau)
            assert (searched[b], pending[b]) == _restated(total[b], tau, b in ended), (b, step)
    emit, pending = lookahead_counts(pending, [0] * B, tau, set(range(B)))
    for b in range(B):
        searched[b] += emit[b]
    assert searched == total and pending == [0] * B
