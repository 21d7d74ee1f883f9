"""GPU parity of the large-vocabulary RNN-T joint (V+1 > 64: csrc/joint_vocab.cu row kernels between
the slab GEMMs) against the reference's formulation restated on the CPU in float64, with the same
bf16 operand rounding as tests/test_joint_gpu.py:

    lp = log_softmax(fc2(relu(fx[:, :, None] + fy[:, None])), 3)      transducer_model.py:71-76
    loss = TransducerLoss(lp, labels, x_lens, y_lens)                  (oracle/rnnt_ref.py)

Bars: loss within 1e-4 relative, every gradient within 2 % of its largest entry, the full
log-probability tensor within 2e-3 absolute and its rows normalised to 1e-5."""
import numpy as np
import pytest
import torch

from oracle import rnnt_ref

pytestmark = pytest.mark.gpu


def _rnd(t):     # bf16 rounding with a straight-through gradient
    return t + (t.detach().float().bfloat16().double() - t.detach())


def _case(B, T, U1, H, V1, blank, seed, w2_scale=1.0):
    rng = np.random.RandomState(seed)
    fx = torch.from_numpy(rng.randn(B, T, H) * 0.7)
    fy = torch.from_numpy(rng.randn(B, U1, H) * 0.7)
    w2 = torch.from_numpy(rng.randn(V1, H) / np.sqrt(H) * w2_scale)
    b2 = torch.from_numpy(rng.randn(V1) * 0.1)
    ylen = rng.randint(max(0, U1 - 4), U1, size=B).astype(np.int32)
    ylen[0] = U1 - 1
    xlen = np.full(B, T, np.int32)
    labels = np.array([k for k in range(V1) if k != blank])
    ymat = labels[rng.randint(0, V1 - 1, size=(B, U1 - 1))].astype(np.int64)
    # labels on the edges of the GEMM's column tiles and at the last non-blank class
    edges = [k for k in (63, 64, 127, 128, V1 - 2) if k < V1 and k != blank]
    for i, k in enumerate(edges):
        ymat[i % B, (i // B) % (U1 - 1)] = k
    flat = np.concatenate([ymat[b, :ylen[b]] for b in range(B)]).astype(np.int32)
    return fx, fy, w2, b2, ymat, flat, xlen, ylen


def _reference(fx, fy, w2, b2, flat, xlen, ylen, blank):
    rf = [t.clone().requires_grad_(True) for t in (fx, fy, w2, b2)]
    z = _rnd(torch.relu(rf[0][:, :, None, :] + rf[1][:, None, :, :]))
    lp = torch.log_softmax(z @ _rnd(rf[2]).t() + rf[3], 3)
    costs, g = rnnt_ref.rnnt_loss_and_grad(lp.detach().numpy(), flat, xlen, ylen, blank)
    lp.backward(torch.from_numpy(g))
    return costs.sum(), [r.grad for r in rf], lp.detach()


def _ours(fx, fy, w2, b2, ymat, flat, xlen, ylen, blank):
    from speech_b200.functions.transducer import JointTransducerLoss, joint_log_probs
    mine = [t.float().cuda().requires_grad_(True) for t in (fx, fy, w2, b2)]
    loss = JointTransducerLoss(blank=blank)(mine[0], mine[1], mine[2], mine[3],
                                            torch.from_numpy(ymat), torch.from_numpy(flat),
                                            torch.from_numpy(xlen), torch.from_numpy(ylen))
    assert loss.shape == (1,)
    loss.backward()

    class FC2:
        weight, bias = mine[2].detach(), mine[3].detach()
    full = joint_log_probs(mine[0].detach(), mine[1].detach(), FC2, torch.from_numpy(ymat), blank)
    torch.cuda.synchronize()
    return loss.item(), [m.grad.double().cpu() for m in mine], full.double().cpu()


@pytest.mark.parametrize("B,T,U1,H,V1,blank,seed", [
    (2, 5, 4, 16, 65, 64, 0),          # one class over the resident kernel's limit
    (3, 23, 9, 96, 130, 0, 1),         # blank first, H not a multiple of 64, several slabs
    (2, 17, 6, 256, 257, 256, 2),      # V1 not a multiple of 8
    (2, 9, 5, 1024, 1024, 1023, 3),
    (1, 4, 3, 64, 4096, 4095, 4),      # rows wider than one CTA's column chunk
])
def test_large_vocab_joint_matches_reference_formulation(cuda_lib, B, T, U1, H, V1, blank, seed):
    fx, fy, w2, b2, ymat, flat, xlen, ylen = _case(B, T, U1, H, V1, blank, seed)
    cost, ref_grads, ref_lp = _reference(fx, fy, w2, b2, flat, xlen, ylen, blank)
    loss, grads, full = _ours(fx, fy, w2, b2, ymat, flat, xlen, ylen, blank)
    assert abs(loss - cost) / cost < 1e-4, (loss, cost)
    for name, a, r in zip(("fx", "fy", "w2", "b2"), grads, ref_grads):
        err = (a - r).abs().max().item()
        assert err < 2e-2 * r.abs().max().item() + 1e-6, (name, err, r.abs().max().item())
    assert tuple(full.shape) == (B, T, U1, V1)
    assert (full - ref_lp).abs().max().item() < 2e-3
    assert np.allclose(np.exp(full.numpy()).sum(-1), 1.0, atol=1e-5)


def test_large_vocab_joint_is_max_subtracted(cuda_lib):
    """Logits spanning about +-200: exp() of an un-shifted logit would overflow fp32."""
    B, T, U1, H, V1 = 2, 9, 5, 128, 300
    fx, fy, w2, b2, ymat, flat, xlen, ylen = _case(B, T, U1, H, V1, V1 - 1, 5)
    z = _rnd(torch.relu(fx[:, :, None, :] + fy[:, None, :, :]))
    w2 = w2 * (200.0 / (z @ _rnd(w2).t()).abs().max().item())
    cost, _, ref_lp = _reference(fx, fy, w2, b2, flat, xlen, ylen, V1 - 1)
    assert (z @ _rnd(w2).t()).abs().max().item() > 150
    loss, grads, full = _ours(fx, fy, w2, b2, ymat, flat, xlen, ylen, V1 - 1)
    assert np.isfinite(loss) and all(torch.isfinite(g).all() for g in grads)
    assert abs(loss - cost) / cost < 1e-4, (loss, cost)
    assert np.allclose(np.exp(full.numpy()).sum(-1), 1.0, atol=1e-5)


@pytest.mark.parametrize("V1", [33, 64])
def test_slab_path_matches_resident_kernel(cuda_lib, monkeypatch, V1):
    """Both implementations on the same small vocabulary: lattice and full log-probabilities within
    1e-4; gradients within 1e-3 of each one's largest entry (both round dlogits to bf16, their fp32
    accumulation orders differ)."""
    from speech_b200.functions import transducer
    B, T, U1, H = 3, 21, 7, 192
    blank = V1 - 1
    fx, fy, w2, b2, ymat, flat, xlen, ylen = _case(B, T, U1, H, V1, blank, 6)
    loss_r, grads_r, full_r = _ours(fx, fy, w2, b2, ymat, flat, xlen, ylen, blank)
    # slab path, called directly
    fxc, fyc = fx.float().cuda(), fy.float().cuda()
    w2b, b2c = w2.float().cuda().bfloat16(), b2.float().cuda()
    ym = torch.from_numpy(ymat).to("cuda", torch.int32)
    full_s = torch.empty(B, T, U1, V1, dtype=torch.float32, device="cuda")
    lat, lse = transducer.joint_vocab_forward(fxc, fyc, w2b, b2c, ym, blank, lp_full=full_s)
    torch.cuda.synchronize()
    assert (full_s.double().cpu() - full_r).abs().max().item() < 1e-4
    # lat[(t*B + b)*U1 + u] = {lp[blank], lp[label of arc u]} of the resident kernel's tensor
    lat = lat.double().cpu().reshape(T, B, U1, 2).permute(1, 0, 2, 3)
    assert (lat[..., 0] - full_r[..., blank]).abs().max().item() < 1e-4
    lab = torch.from_numpy(ymat)[:, None, :, None].expand(B, T, U1 - 1, 1)
    ref_l = full_r[:, :, :U1 - 1].gather(3, lab)[..., 0]
    assert (lat[:, :, :U1 - 1, 1] - ref_l).abs().max().item() < 1e-4
    assert torch.isneginf(lat[:, :, U1 - 1, 1]).all()
    assert torch.isfinite(lse).all()
    # slab path through the autograd function
    monkeypatch.setattr(transducer, "JOINT_RESIDENT_MAX_CLASSES", 0)
    loss_s, grads_s, _ = _ours(fx, fy, w2, b2, ymat, flat, xlen, ylen, blank)
    assert abs(loss_s - loss_r) / abs(loss_r) < 1e-5, (loss_s, loss_r)
    for name, a, r in zip(("fx", "fy", "w2", "b2"), grads_s, grads_r):
        err = (a - r).abs().max().item()
        assert err < 1e-3 * r.abs().max().item() + 1e-7, (name, err, r.abs().max().item())


def test_large_vocab_joint_memory_stays_within_slabs(cuda_lib):
    """loss + backward at V1 = 2048 allocate far less than one full (nodes x V1) fp32 logits tensor."""
    from speech_b200.functions.transducer import JointTransducerLoss
    B, T, U1, H, V1 = 4, 64, 40, 256, 2048
    rng = np.random.RandomState(7)
    dev = "cuda"
    fx = torch.from_numpy(rng.randn(B, T, H).astype(np.float32) * 0.7).to(dev).requires_grad_(True)
    fy = torch.from_numpy(rng.randn(B, U1, H).astype(np.float32) * 0.7).to(dev).requires_grad_(True)
    w2 = torch.from_numpy((rng.randn(V1, H) / np.sqrt(H)).astype(np.float32)).to(dev).requires_grad_(True)
    b2 = torch.zeros(V1, device=dev, requires_grad=True)
    ylen = np.full(B, U1 - 1, np.int32)
    ymat = rng.randint(0, V1 - 1, size=(B, U1 - 1))
    flat = torch.from_numpy(ymat.reshape(-1).astype(np.int32))
    xlen = torch.full((B,), T, dtype=torch.int32)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss = JointTransducerLoss()(fx, fy, w2, b2, torch.from_numpy(ymat), flat, xlen,
                                 torch.from_numpy(ylen))
    loss.backward()
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    full_logits = T * B * U1 * V1 * 4
    assert torch.isfinite(loss).all()
    assert growth < full_logits / 2, (growth, full_logits)


def test_transducer_model_trains_with_a_large_vocabulary(cuda_lib):
    """Transducer with 300 labels (V+1 = 301): finite loss, every parameter receives a gradient, the
    loss equals the reference formulation on the model's own full log-probabilities, and `infer`
    equals the beam search run on them."""
    from speech_b200.models import Transducer
    from speech_b200.transducer_decoders import decode_static_batch
    torch.manual_seed(0)
    np.random.seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                       "rnn": {"dim": 32, "bidirectional": True, "layers": 1}},
           "decoder": {"embedding_dim": 16, "layers": 1}}
    m = Transducer(40, 300, cfg).cuda()
    inputs = [np.random.randn(60, 40).astype(np.float32) for _ in range(3)]
    labels = [np.random.randint(0, 300, n).tolist() for n in (5, 3, 4)]
    batch = (inputs, labels)
    loss = m.loss(batch)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    for n, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        assert p.grad.abs().sum() > 0, n
    with torch.no_grad():
        lp = m(batch)                                     # (B, T', U+1, V+1)
    assert lp.shape[-1] == 301
    x, y, x_lens, y_lens = m.collate(*batch)
    costs, _ = rnnt_ref.rnnt_loss_and_grad(lp.double().cpu().numpy(), y.numpy(), x_lens.numpy(),
                                           y_lens.numpy(), m.blank)
    assert abs(loss.item() - costs.sum()) / costs.sum() < 1e-4
    preds = m.infer(batch)
    tlens = [min(i.shape[0], lp.shape[1]) for i in inputs]
    expect, _ = decode_static_batch(lp, tlens, [len(l) + 1 for l in labels], 4, m.blank)
    assert preds == expect
