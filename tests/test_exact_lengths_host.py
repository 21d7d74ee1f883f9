"""Host-side pieces of the exact-lengths mode (no GPU): the switch, the lengths the models hand to
the losses and decoders, and the length-aware CPU oracle the GPU tests compare against."""
import pickle

import numpy as np
import pytest
import torch

from exact_lengths_ref import packed_ctc_costs, packed_encode

CFG = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                   "rnn": {"dim": 16, "bidirectional": True, "layers": 2}},
       "decoder": {"embedding_dim": 16, "layers": 1}}


def _cfg(exact):
    c = dict(CFG)
    c["exact_lengths"] = exact
    return c


def _batch(lens, F=40, seed=0):
    rng = np.random.RandomState(seed)
    inputs = [rng.randn(n, F).astype(np.float32) for n in lens]
    labels = [rng.randint(0, 10, 3 + i).tolist() for i in range(len(lens))]
    return inputs, labels


@pytest.mark.parametrize("family", ["CTC", "Transducer"])
def test_collate_lengths(family):
    import speech_b200.models as models
    lens = [77, 40, 63, 91]
    inputs, labels = _batch(lens)
    m = getattr(models, family)(40, 10, _cfg(True))
    x, y, x_lens, y_lens = m.collate(inputs, labels)
    assert x_lens.dtype == torch.int32
    assert x_lens.tolist() == [m.conv_out_size(n, 0) for n in lens]
    assert x.shape[1] == 91 and y_lens.tolist() == [len(l) for l in labels]
    d = getattr(models, family)(40, 10, _cfg(False))
    xd, yd, xl_d, yl_d = d.collate(inputs, labels)
    assert xl_d.tolist() == [d.conv_out_size(91, 0)] * 4          # the reference's padded T'
    assert torch.equal(xd, x) and torch.equal(yd, y) and torch.equal(yl_d, y_lens)


def test_switch_config_pickle_and_state_dict():
    from speech_b200.models import CTC, Seq2Seq, Transducer
    for cls in (CTC, Transducer, Seq2Seq):
        assert cls(40, 10, CFG).exact_lengths is False
        m = cls(40, 10, _cfg(True))
        assert m.exact_lengths is True
        assert list(m.state_dict()) == list(cls(40, 10, CFG).state_dict())
        assert pickle.loads(pickle.dumps(m)).exact_lengths is True
        # a model pickled before the attribute existed
        del m.__dict__["exact_lengths"]
        old = pickle.loads(pickle.dumps(m))
        assert "exact_lengths" not in old.__dict__ and old.exact_lengths is False
        old.exact_lengths = True                   # settable on a loaded checkpoint
        assert old.exact_lengths is True


def test_seq2seq_input_lens():
    from speech_b200.models import Seq2Seq
    inputs, _ = _batch([50, 60, 44])
    m = Seq2Seq(40, 12, _cfg(True))
    assert m.input_lens(inputs) == [m.conv_out_size(n, 0) for n in (50, 60, 44)]
    assert Seq2Seq(40, 12, CFG).input_lens(inputs) is None


@pytest.mark.parametrize("log_t", [False, True])
def test_masked_attention_oracle_equals_each_utterance_alone(log_t):
    from speech_b200.models import Seq2Seq
    from exact_lengths_ref import masked_decode_ref
    torch.manual_seed(0)
    cfg = _cfg(True)
    cfg["decoder"] = {"embedding_dim": 16, "layers": 1, "log_t": log_t}
    m = Seq2Seq(40, 12, cfg)
    lens = [23, 9, 17, 1]
    x = torch.randn(4, 23, 16, dtype=torch.float64)
    y = torch.randint(0, 11, (4, 6))
    out, al, xl, _ = masked_decode_ref(m, x, y, lens)
    out.sum().backward()
    for b, L in enumerate(lens):
        o1, a1, x1, _ = masked_decode_ref(m, x[b:b + 1, :L], y[b:b + 1], [L])
        o1.sum().backward()
        assert (out[b] - o1[0]).abs().max().item() < 1e-10
        assert (al[b, :, :L] - a1[0]).abs().max().item() < 1e-10
        assert float(al[b, :, L:].abs().sum()) == 0.0
        assert (xl.grad[b, :L] - x1.grad[0]).abs().max().item() < 1e-10
        assert float(xl.grad[b, L:].abs().sum()) == 0.0


def test_batch_chunks_slice_lens():
    from speech_b200 import ops
    seen = []

    def fn(xc, lc):
        seen.append((xc.shape[0], list(lc)))
        return xc

    x = torch.zeros(300, 2, 1)
    lens = list(range(300))
    ops._batch_chunks(x, lens, fn)
    assert seen == [(128, lens[:128]), (128, lens[128:256]), (44, lens[256:])]


@pytest.mark.parametrize("bidirectional", [False, True])
def test_packed_oracle_equals_each_utterance_alone(bidirectional):
    from oracle.model_ref import RefCTC
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                       "rnn": {"dim": 16, "bidirectional": bidirectional,
                                               "layers": 2}}}
    ref = RefCTC(40, 10, cfg).double()
    in_lens = [100, 40, 73, 58, 100, 41]
    x = torch.zeros(len(in_lens), max(in_lens), 40, dtype=torch.float64)
    for b, n in enumerate(in_lens):
        x[b, :n] = torch.randn(n, 40, dtype=torch.float64)
    rng = np.random.RandomState(1)
    labels = [torch.tensor(rng.randint(0, 10, 2 + b)) for b in range(len(in_lens))]
    with torch.no_grad():
        h, lens = packed_encode(ref.enc, x, in_lens)
        logits = ref.fc(h)
        costs = packed_ctc_costs(logits, lens, torch.cat(labels),
                                 [len(l) for l in labels], ref.blank)
        for b, n in enumerate(in_lens):
            L = int(lens[b])
            alone = ref.enc(x[b:b + 1, :n])
            assert alone.shape[1] == L
            assert (h[b, :L] - alone[0]).abs().max().item() < 1e-10
            assert float(h[b, L:].abs().sum()) == 0.0
            c1 = ref.loss(x[b:b + 1, :n], labels[b], torch.tensor([len(labels[b])]))
            assert abs(costs[b].item() - c1.item()) < 1e-10 * max(1.0, abs(c1.item()))
        if bidirectional:
            # padding changes the plain (unpacked) result: the oracle has something to catch
            plain = ref.enc(x)
            b = int(np.argmin(in_lens))
            L = int(lens[b])
            assert (plain[b, :L] - h[b, :L]).abs().max().item() > 1e-6
