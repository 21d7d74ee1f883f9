"""GPU parity of the shapes the kernels reach through zero-padding: GRU widths that are not a
multiple of 16, conv stacks with any out_channels, and the Transducer joint at any width (slab
routing where fc2 does not fit the fused kernel, fc1 padded to a multiple of 8).

Bars as in tests/test_gru_gpu.py: outputs within 2e-2 of the fp64 reference, gradients within 3%
of the largest reference entry."""
import numpy as np
import pytest
import torch

from exact_lengths_ref import packed_encode

pytestmark = pytest.mark.gpu


def _grad_ok(got, ref):
    return (got - ref).abs().max().item() < 3e-2 * ref.abs().max().item() + 1e-4


def _model_grad_ok(got, ref):
    """Whole-model bars of tests/test_zz_northstar_grads_gpu.py: the bottom conv layer's gradient
    has passed through every bf16 layer above it, so it keeps direction and size, not entries."""
    rel = ((got - ref).norm() / ref.norm()).item()
    cos = (torch.dot(got.flatten(), ref.flatten()) / (got.norm() * ref.norm())).item()
    return rel < 5e-2 and cos > 0.999


@pytest.mark.parametrize("B,T,In,H,L,bidir", [
    (4, 9, 40, 40, 2, False),      # uni, 2 layers: padded input columns of layer 1
    (8, 12, 64, 200, 2, True),
    (16, 6, 96, 1000, 1, True),    # 2 x 63 CTAs
    (128, 4, 64, 1000, 1, True),   # two m64 blocks of batch rows
    (6, 60, 32, 200, 1, True),     # long run
])
def test_padded_gru_widths_match_fp64(cuda_lib, B, T, In, H, L, bidir):
    from speech_b200.ops import gru_stack
    torch.manual_seed(B + T + H)
    rnn = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=bidir)
    x = torch.randn(B, T, In)
    rnn64 = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=bidir).double()
    rnn64.load_state_dict({k: v.double() for k, v in rnn.state_dict().items()})
    x64 = x.double().requires_grad_(True)
    y64, _ = rnn64(x64)
    w = torch.randn_like(y64)
    (y64 * w).sum().backward()
    rnn_c = rnn.cuda()
    xc = x.cuda().requires_grad_(True)
    yc = gru_stack(xc, rnn_c)
    (yc * w.float().cuda()).sum().backward()
    assert yc.shape == y64.shape
    assert (yc.double().cpu() - y64).abs().max().item() < 2e-2
    assert _grad_ok(xc.grad.double().cpu(), x64.grad)
    for (n, p64), (_, pc) in zip(rnn64.named_parameters(), rnn_c.named_parameters()):
        assert pc.grad.shape == p64.grad.shape
        assert _grad_ok(pc.grad.double().cpu(), p64.grad), n


def test_gru_plan_covers_every_width_up_to_the_resident_limit(cuda_lib):
    """sb_gru_plan rounds H up to whole CTAs of 16 units, for every width whose padded grid the
    resident kernels hold (one CTA per SM), and the padded width runs in both passes."""
    from speech_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for H, ndir, want in ((1000, 2, 1008), (1024, 2, 1024), (40, 1, 48), (100, 2, 112),
                          (250, 1, 256)):
        assert ops.gru_padded_width(64, H, ndir) == want
    widest_bi = sms // 2 * 16
    assert ops.gru_padded_width(64, widest_bi - 5, 2) == widest_bi
    assert ops.gru_padded_width(64, sms * 16 - 9, 1) == sms * 16
    rnn = torch.nn.GRU(16, widest_bi - 5, 1, batch_first=True, bidirectional=True).cuda()
    x = torch.randn(8, 3, 16, device="cuda", requires_grad=True)
    ops.gru_stack(x, rnn).sum().backward()
    assert torch.isfinite(x.grad).all()


def test_padded_layer_dropout_matches_masked_reference(cuda_lib):
    """The inter-layer dropout masks of a padded layer are drawn over the H real units, so the
    restatement of test_gru_inter_layer_dropout_matches_masked_reference applies unchanged."""
    from speech_b200.ops import gru_stack
    B, T, In, H, L, p = 6, 11, 40, 40, 2, 0.3
    torch.manual_seed(B + T)
    rnn = torch.nn.GRU(In, H, L, batch_first=True, bidirectional=True, dropout=p).cuda()
    x = torch.randn(B, T, In).cuda().requires_grad_(True)
    torch.manual_seed(1234)
    y = gru_stack(x, rnn, dropout=p)
    w = torch.randn_like(y)
    (y * w).sum().backward()
    got = {n: q.grad.double().cpu() for n, q in rnn.named_parameters()}
    Bp = (B + 7) // 8 * 8
    torch.manual_seed(1234)
    masks = [(torch.rand(T * Bp, 2 * H, device="cuda") >= p).double().cpu() / (1.0 - p)
             for _ in range(L - 1)]
    h = x.detach().double().cpu().requires_grad_(True)
    x64 = h
    layers = []
    for l in range(L):
        g = torch.nn.GRU(In if l == 0 else 2 * H, H, 1, batch_first=True,
                         bidirectional=True).double()
        g.load_state_dict({k.replace("_l%d" % l, "_l0"): v.double().cpu()
                           for k, v in rnn.state_dict().items() if "_l%d" % l in k})
        layers.append(g)
        h, _ = g(h)
        if l + 1 < L:
            h = h * masks[l].view(T, Bp, 2 * H)[:, :B].transpose(0, 1)
    (h * w.double().cpu()).sum().backward()
    assert (y.double().cpu() - h.detach()).abs().max().item() < 3e-2
    assert _grad_ok(x.grad.double().cpu(), x64.grad)
    for l, g in enumerate(layers):
        for k, q in g.named_parameters():
            name = k.replace("_l0", "_l%d" % l)
            assert _grad_ok(got[name], q.grad), name


CFG = {"dropout": 0.0, "encoder": {"conv": [[4, 5, 7, 2], [12, 3, 5, 1]],
                                   "rnn": {"dim": 1000, "bidirectional": True, "layers": 1}}}


def test_padded_encoder_exact_lengths_matches_packed_reference(cuda_lib):
    from oracle.model_ref import RefEncoder
    from speech_b200.models import Model
    torch.manual_seed(0)
    cfg = dict(CFG, exact_lengths=True)
    cfg["encoder"] = {"conv": CFG["encoder"]["conv"],
                      "rnn": {"dim": 200, "bidirectional": True, "layers": 2}}
    m = Model(40, cfg)
    ref = RefEncoder(40, cfg).double()
    ref.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    m.cuda()
    rng = np.random.RandomState(0)
    inputs = [rng.randn(n, 40).astype(np.float32) for n in (60, 31, 47, 52, 39)]
    x, _, x_lens, _ = m.lattice_batch(inputs, [[1, 2]] * len(inputs))
    with torch.no_grad():
        y = m.encode(x, x_lens).cpu().double()
        r, lens = packed_encode(ref, x.cpu().double(), [len(i) for i in inputs])
    assert x_lens.tolist() == lens.tolist()
    for b, n in enumerate(lens.tolist()):
        assert (y[b, :n] - r[b, :n]).abs().max().item() < 2e-2, b
        assert float(y[b, n:].abs().sum()) == 0.0


def _ctc_batch(B=4, T=40, V=10, seed=0):
    rng = np.random.RandomState(seed)
    inputs = [rng.randn(T, 40).astype(np.float32) for _ in range(B)]
    labels = [rng.randint(0, V, 6).tolist() for _ in range(B)]
    return inputs, labels


def test_ctc_dim_1000_with_4_and_12_channels_matches_reference_model(cuda_lib):
    """Logits, loss and the GRU / output-layer gradients against the fp64 reference model; the
    conv gradients are pinned by the zero-embedded comparison below."""
    from oracle.model_ref import RefCTC
    from speech_b200.models import CTC
    torch.manual_seed(1)
    m = CTC(40, 10, CFG)
    ref = RefCTC(40, 10, CFG).double()
    ref.load_from_dropin({k: v.double() for k, v in m.state_dict().items()})
    m.cuda()
    batch = _ctc_batch()
    x, y, _, y_lens = m.collate(*batch)
    with torch.no_grad():
        logits = m.forward_impl(x).double().cpu()
    loss = m.loss(batch)
    loss.backward()
    x64 = x.cpu().double()
    ref_logits = ref.logits(x64)
    assert logits.shape == ref_logits.shape
    assert (logits - ref_logits.detach()).abs().max().item() < 2e-2
    ref_loss = ref.loss(x64, y, y_lens)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) / ref_loss.item() < 1e-2
    mine = dict(m.named_parameters())
    for n, q in ref.named_parameters():
        if n.startswith("enc.conv."):
            continue
        key = n[len("enc."):] if n.startswith("enc.") else "fc.fc." + n[len("fc."):]
        assert _model_grad_ok(mine[key].grad.double().cpu(), q.grad), n


def test_padded_model_equals_zero_embedded_wider_model(cuda_lib):
    """CTC with conv channels 4, 12 and GRU width 1000 against CTC with 8, 16 and 1008 whose extra
    filters and units are explicitly zero (the kernels' own widths, no padding inside): same
    logits, loss and gradients of the real blocks up to float summation order."""
    from speech_b200 import ops
    from speech_b200.models import CTC
    torch.manual_seed(4)
    m = CTC(40, 10, CFG)
    wcfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 7, 2], [16, 3, 5, 1]],
                                        "rnn": {"dim": 1008, "bidirectional": True, "layers": 1}}}
    w = CTC(40, 10, wcfg)
    sd = m.state_dict()
    F1 = m.conv_out_size(40, 1)
    wsd = {"conv.0.weight": ops.pad_blocks(sd["conv.0.weight"], 0, 1, 4, 8),
           "conv.0.bias": ops.pad_blocks(sd["conv.0.bias"], 0, 1, 4, 8),
           "conv.2.weight": ops.pad_blocks(ops.pad_blocks(sd["conv.2.weight"], 0, 1, 12, 16),
                                           1, 1, 4, 8),
           "conv.2.bias": ops.pad_blocks(sd["conv.2.bias"], 0, 1, 12, 16),
           "fc.fc.weight": ops.pad_blocks(sd["fc.fc.weight"], 1, 1, 1000, 1008),
           "fc.fc.bias": sd["fc.fc.bias"]}
    for s_ in ("_l0", "_l0_reverse"):
        names = ["rnn." + k + s_ for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        q = list(ops.pad_gru_layer(*[sd[n] for n in names], 1000, 1008, 0))
        q[0] = ops.pad_blocks(q[0], 1, 1, 12 * F1, 16 * F1)
        wsd.update(zip(names, q))
    w.load_state_dict(wsd)
    m.cuda()
    w.cuda()
    batch = _ctc_batch(seed=5)
    x, _, _, _ = m.collate(*batch)
    with torch.no_grad():
        assert (m.forward_impl(x) - w.forward_impl(x)).abs().max().item() < 1e-4
    lm, lw = m.loss(batch), w.loss(batch)
    assert abs(lm.item() - lw.item()) < 1e-4 * abs(lw.item())
    lm.backward()
    lw.backward()
    gw = dict(w.named_parameters())
    real = {"conv.0.weight": (slice(0, 4),), "conv.0.bias": (slice(0, 4),),
            "conv.2.weight": (slice(0, 12), slice(0, 4)), "conv.2.bias": (slice(0, 12),),
            "fc.fc.weight": (slice(None), slice(0, 1000)), "fc.fc.bias": (slice(None),)}
    for n, p in m.named_parameters():
        if n in real:
            g = gw[n].grad[real[n]]
        else:
            g = ops.unpad_blocks(gw[n].grad, 0, 3, 1000, 1008)
            if "weight_hh" in n:
                g = g[:, :1000]
            elif "weight_ih" in n:
                g = g[:, :12 * F1]
        assert g.shape == p.grad.shape, n
        assert (p.grad - g).abs().max().item() < 1e-3 * g.abs().max().item() + 1e-6, n


def test_flat_sgd_gradient_of_padded_model_equals_autograd(cuda_lib):
    """The padded GRU layer computes into temporaries and adds the real block into FlatSGD's flat
    gradient buffer: same values as plain autograd, and the layer is announced once."""
    from speech_b200 import ops
    from speech_b200.models import CTC
    from speech_b200.optim import FlatSGD
    torch.manual_seed(2)
    cfg = dict(CFG)
    cfg["encoder"] = {"conv": CFG["encoder"]["conv"],
                      "rnn": {"dim": 200, "bidirectional": True, "layers": 2}}
    ma, mb = CTC(40, 10, cfg).cuda(), CTC(40, 10, cfg).cuda()
    mb.load_state_dict(ma.state_dict())
    batch = _ctc_batch(seed=3)
    ma.loss(batch).backward()
    opt = FlatSGD(mb, lr=0.0)
    announced = []
    ops.set_grad_ready_hook(lambda ps: announced.append([id(p) for p in ps]))
    try:
        opt.zero_grad()
        mb.loss(batch).backward()
    finally:
        ops.set_grad_ready_hook(None)
    for (n, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
        assert torch.allclose(pb.grad, pa.grad, rtol=1e-5, atol=1e-6), n
    layers = [[id(getattr(mb.rnn, k + "_l%d%s" % (l, s)))
               for s in ("", "_reverse") for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
              for l in range(2)]
    assert sorted(map(sorted, announced)) == sorted(map(sorted, layers))


def test_joint_slab_routing_at_width_1280(cuda_lib):
    """V+1 = 40 at H = 1280: fc2 does not fit the fused kernel, the slab path runs."""
    from speech_b200.functions import transducer
    from test_joint_vocab_gpu import _case, _ours, _reference
    B, T, U1, H, V1 = 2, 9, 5, 1280, 40
    assert transducer.joint_uses_slabs(H, V1)
    fx, fy, w2, b2, ymat, flat, xlen, ylen = _case(B, T, U1, H, V1, V1 - 1, 8)
    cost, ref_grads, ref_lp = _reference(fx, fy, w2, b2, flat, xlen, ylen, V1 - 1)
    loss, grads, full = _ours(fx, fy, w2, b2, ymat, flat, xlen, ylen, V1 - 1)
    assert abs(loss - cost) / cost < 1e-4, (loss, cost)
    for name, a, r in zip(("fx", "fy", "w2", "b2"), grads, ref_grads):
        assert (a - r).abs().max().item() < 2e-2 * r.abs().max().item() + 1e-6, name
    assert (full - ref_lp).abs().max().item() < 2e-3


def test_transducer_width_100_matches_fp64_restatement(cuda_lib):
    """H = 100: the GRUs run at 112 units, fc1 at 104 outputs with fc2's zero columns."""
    import torch.nn.functional as F
    from oracle import rnnt_ref
    from oracle.model_ref import RefEncoder
    from speech_b200.models import Transducer
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 32, 2]],
                                       "rnn": {"dim": 100, "bidirectional": True, "layers": 1}},
           "decoder": {"embedding_dim": 24, "layers": 1}}
    m = Transducer(40, 10, cfg)
    sd = {k: v.double() for k, v in m.state_dict().items()}
    enc = RefEncoder(40, cfg).double()
    enc.load_state_dict({k: v for k, v in sd.items() if k.startswith(("conv.", "rnn."))})
    dec = torch.nn.GRU(24, 100, 1, batch_first=True).double()
    dec.load_state_dict({k[len("dec_rnn."):]: v for k, v in sd.items() if k.startswith("dec_rnn.")})
    m.cuda()
    rng = np.random.RandomState(0)
    inputs = [rng.randn(60, 40).astype(np.float32) for _ in range(3)]
    labels = [rng.randint(0, 10, n).tolist() for n in (5, 7, 3)]
    batch = (inputs, labels)
    with torch.no_grad():
        out = m(batch).double().cpu()
    loss = m.loss(batch)
    loss.backward()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())
    # fp64 restatement of transducer_model.py:54-77
    x, _, _, _ = m.collate(*batch)
    ymat = m.label_collate(labels)
    xe = enc(x.cpu().double())
    emb = F.embedding(ymat, sd["embedding.weight"])
    pred, _ = dec(torch.cat([torch.zeros(3, 1, 24, dtype=torch.float64), emb], 1))
    fx = F.linear(xe, sd["fc1.fc.weight"], sd["fc1.fc.bias"])
    fy = F.linear(pred, sd["fc1.fc.weight"], sd["fc1.fc.bias"])
    lp = torch.log_softmax(F.linear(torch.relu(fx[:, :, None] + fy[:, None]),
                                    sd["fc2.fc.weight"], sd["fc2.fc.bias"]), 3)
    assert out.shape == lp.shape
    assert (out - lp.detach()).abs().max().item() < 2e-2
    flat = np.concatenate(labels).astype(np.int32)
    T = out.shape[1]
    c_ours, _ = rnnt_ref.rnnt_loss_and_grad(out.numpy(), flat, [T] * 3, [len(l) for l in labels])
    assert abs(loss.item() - c_ours.sum()) / c_ours.sum() < 1e-4
    c_ref, _ = rnnt_ref.rnnt_loss_and_grad(lp.detach().numpy(), flat, [T] * 3, [len(l) for l in labels])
    assert abs(loss.item() - c_ref.sum()) / c_ref.sum() < 1e-2
