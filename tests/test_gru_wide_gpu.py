"""GPU tests of the wide GRU recurrence kernels (gru_fwd_wide_kernel / gru_bwd_wide_kernel).

A layer whose W_hh slices do not fit one CTA of 16 units per SM runs U = 16 or 32 units per CTA
with the head of each CTA's weight slice resident in shared memory and the tail streamed from L2
every step.  sb_gru_plan rounds such widths up to a multiple of U; every width the resident
kernels took keeps its answer and its kernels.  Parity bars are those of test_gru_gpu.py: outputs
within 2e-2 of fp64 nn.GRU, gradients within 3% of the largest reference entry.  Developer flag
2048 forces the wide kernels with no resident chunks, so the weight stream runs at small widths,
where the sums are those of the plain resident kernels (same chunk order, same MMA shape).
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

FORCE_STREAM = 2048
PLAIN = 32            # no K-split forward: gru_fwd_kernel where it fits


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _plan(lib, backward):
    out = (ctypes.c_int * 3)()
    assert lib.sb_debug_gru_plan(backward, out) == 0
    return tuple(out)


def _units(H, Hp, ndir):
    """units per CTA the wide plan uses for a padded width Hp"""
    return 16 if ndir * Hp // 16 <= _sms() else 32


# ---- 1. plan ------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,ndir,Bp", [
    (H, 2, Bp) for H in (1072, 1152, 1280, 1536, 2048) for Bp in (8, 64, 128)
] + [(2128, 1, Bp) for Bp in (8, 64, 128)] + [(2048, 1, 128)])
def test_plan_past_the_resident_limit(cuda_lib, H, ndir, Bp):
    from speech_b200 import ops
    Hp = ops.gru_padded_width(Bp, H, ndir)
    U = _units(H, Hp, ndir)
    assert 0 <= Hp - H < U and Hp % U == 0 and ndir * Hp // U <= _sms()
    _run_passes(cuda_lib, 3, Bp, Hp, ndir, 0, seed=H + Bp)
    assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == "wide"
    # unidirectional 2048 at 128 rows: only the forward's ring misses; the backward stays resident
    bwd_wide = not (ndir == 1 and H == 2048)
    assert cuda_lib.sb_debug_gru_bwd_kernel().decode() == ("wide" if bwd_wide else "plain")
    for backward in ((0, 1) if bwd_wide else (0,)):
        u, r, s = _plan(cuda_lib, backward)
        assert u == U and r + s == ((3 if backward else 1) * Hp + 63) // 64


@pytest.mark.parametrize("Bp", [8, 64, 128])
def test_plan_unchanged_up_to_the_resident_limit(cuda_lib, Bp):
    """Every width up to ndir * H / 16 = SM count keeps H rounded up to 16; at 128 rows the
    unidirectional widths above 1920, which the resident forward never took, do so too (their
    wide forward runs U = 16)."""
    from speech_b200 import ops
    sms = _sms()
    for ndir in (1, 2):
        for H in range(16, sms // ndir * 16 + 1, 16):
            assert ops.gru_padded_width(Bp, H, ndir) == H
            assert ops.gru_padded_width(Bp, H - 7, ndir) == H


def test_plan_ceiling(cuda_lib):
    from speech_b200 import ops, _lib
    sms = _sms()
    for ndir in (1, 2):
        top = sms // ndir * 32
        assert ops.gru_padded_width(64, top, ndir) == top
        with pytest.raises(_lib.SpeechB200Error):
            ops.gru_padded_width(64, top + 1, ndir)


# ---- 2. selection -------------------------------------------------------------------------------
def test_selection_unchanged_at_1024(cuda_lib):
    for Bp, want in ((64, "ks2"), (128, "plain")):
        _run_passes(cuda_lib, 3, Bp, 1024, 2, 0, seed=Bp)
        assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == want
        assert cuda_lib.sb_debug_gru_bwd_kernel().decode() != "wide"
        assert _plan(cuda_lib, 0) == (0, 0, 0) and _plan(cuda_lib, 1) == (0, 0, 0)


# ---- 3. parity with fp64 nn.GRU through ops.gru_stack --------------------------------------------
def _parity(B, T, In, H, L, bidir, seed):
    from speech_b200.ops import gru_stack
    torch.manual_seed(seed)
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
    torch.cuda.synchronize()
    assert (yc.double().cpu() - y64).abs().max().item() < 2e-2
    gx = xc.grad.double().cpu()
    assert (gx - x64.grad).abs().max().item() < 3e-2 * x64.grad.abs().max().item() + 1e-4
    for (n, p64), (_, pc) in zip(rnn64.named_parameters(), rnn_c.named_parameters()):
        ref = p64.grad
        err = (pc.grad.double().cpu() - ref).abs().max().item()
        assert err < 3e-2 * ref.abs().max().item() + 1e-4, (n, err, ref.abs().max().item())


@pytest.mark.parametrize("B,T,In,H,L,bidir", [
    (8, 12, 64, 1280, 1, True),
    (64, 6, 64, 1536, 1, True),
    (128, 4, 64, 1152, 1, True),     # two m64 blocks, two epilogue passes
    (4, 10, 48, 2048, 2, True),      # a wide layer input
    (16, 8, 64, 2200, 1, False),
    (8, 9, 40, 1100, 1, True),       # a padded width
])
def test_wide_layer_matches_fp64(cuda_lib, B, T, In, H, L, bidir):
    _parity(B, T, In, H, L, bidir, seed=B + T + H)
    assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == "wide"
    assert cuda_lib.sb_debug_gru_bwd_kernel().decode() == "wide"


# ---- 4. the weight stream at small widths ---------------------------------------------------------
def _inputs(T, Bp, H, ndir, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = ndir * H
    gi = torch.randn(T * Bp, ndir * 3 * H, device="cuda", generator=g)
    whh = (torch.randn(ndir, 3 * H, H, device="cuda", generator=g) / H ** 0.5).to(torch.bfloat16)
    bhh = torch.randn(ndir, 3 * H, device="cuda", generator=g) * 0.1
    dy = torch.randn(T * Bp, D, device="cuda", generator=g) * 0.1
    return gi, whh, bhh, dy


def _run_passes(lib, T, Bp, H, ndir, flags, seed):
    """sb_gru_fwd then sb_gru_bwd on its outputs, under developer flags"""
    from speech_b200 import _lib, ops
    gi, whh, bhh, dy = _inputs(T, Bp, H, ndir, seed)
    D = ndir * H
    y = torch.empty(T * Bp, D, device="cuda")
    xn = torch.empty(T * Bp, D, dtype=torch.bfloat16, device="cuda")
    gates = torch.empty(T * Bp, ndir, 4, H, device="cuda")
    dgi = torch.empty(T * Bp, ndir * 3 * H, dtype=torch.bfloat16, device="cuda")
    dghn = torch.empty(T * Bp, D, dtype=torch.bfloat16, device="cuda")
    dbih = torch.zeros(ndir * 3 * H, device="cuda")
    dbhh = torch.zeros(ndir * 3 * H, device="cuda")
    lib.sb_debug_gru_flags(flags)
    try:
        nf, nb = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.check(lib.sb_gru_fwd_workspace_size(Bp, H, ndir, ctypes.byref(nf)), "ws")
        _lib.check(lib.sb_gru_bwd_workspace_size(Bp, H, ndir, ctypes.byref(nb)), "ws")
        wf, wb = ops._workspace(nf.value, "cuda"), ops._workspace(nb.value, "cuda")
        sp = _lib.stream_ptr()
        _lib.check(lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), y.data_ptr(),
                                  xn.data_ptr(), gates.data_ptr(), wf.data_ptr(), nf.value,
                                  T, Bp, H, ndir, sp), "sb_gru_fwd")
        _lib.check(lib.sb_gru_bwd(dy.data_ptr(), y.data_ptr(), gates.data_ptr(), whh.data_ptr(),
                                  dgi.data_ptr(), dghn.data_ptr(), dbih.data_ptr(),
                                  dbhh.data_ptr(), wb.data_ptr(), nb.value, T, Bp, H, ndir, sp),
                   "sb_gru_bwd")
        torch.cuda.synchronize()
    finally:
        lib.sb_debug_gru_flags(0)
        lib.sb_debug_gru_ksplit(1)
    return y, xn, gates, dgi, dghn, dbih, dbhh


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("Bp", [8, 64])
@pytest.mark.parametrize("H", [256, 512])
def test_streamed_weights_match_resident_kernels(cuda_lib, H, Bp):
    """rg = 0: every chunk of W_hh streams through the weight ring each step.  Against the plain
    resident kernels (K-split kernels disabled), the sums are the same: bitwise equal outputs
    and exchange operands, bias gradients (atomics) within 1e-6."""
    T, ndir = 20, 2
    cuda_lib.sb_debug_gru_ksplit(0)
    ref = _run_passes(cuda_lib, T, Bp, H, ndir, PLAIN | 8, seed=H + Bp)
    assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == "plain"
    assert cuda_lib.sb_debug_gru_bwd_kernel().decode() == "plain"
    got = _run_passes(cuda_lib, T, Bp, H, ndir, FORCE_STREAM, seed=H + Bp)
    assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == "wide"
    assert cuda_lib.sb_debug_gru_bwd_kernel().decode() == "wide"
    assert _plan(cuda_lib, 0) == (16, 0, H // 64)
    assert _plan(cuda_lib, 1) == (16, 0, 3 * H // 64)
    for name, a, b in zip(("y", "xn", "gates", "dgi", "dghn"), got[:5], ref[:5]):
        assert torch.equal(a, b), (name, _rel(a, b))
    for name, a, b in zip(("dbih", "dbhh"), got[5:], ref[5:]):
        assert _rel(a, b) < 1e-6, name


# ---- 5. exact-lengths mode ------------------------------------------------------------------------
def test_exact_lengths_at_1280(cuda_lib):
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    from speech_b200 import ops
    torch.manual_seed(0)
    H = 1280
    rnn = torch.nn.GRU(32, H, 1, batch_first=True, bidirectional=True).cuda()
    lens = [11, 4, 1, 9, 11, 6]
    B, T = len(lens), max(lens)
    x = torch.randn(B, T, 32, device="cuda", requires_grad=True)
    g = torch.randn(B, T, 2 * H, device="cuda")
    y = ops.gru_stack(x, rnn, lens=lens)
    (y * g).sum().backward()
    assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == "wide"
    for b, L in enumerate(lens):
        assert float(x.grad[b, L:].abs().sum()) == 0.0, b
        assert float(y[b, L:].detach().abs().sum()) == 0.0, b
    r64 = torch.nn.GRU(32, H, 1, batch_first=True, bidirectional=True).double()
    r64.load_state_dict({k: v.double().cpu() for k, v in rnn.state_dict().items()})
    x64 = x.detach().double().cpu().requires_grad_(True)
    out, _ = r64(pack_padded_sequence(x64, torch.tensor(lens), batch_first=True,
                                      enforce_sorted=False))
    out, _ = pad_packed_sequence(out, batch_first=True, total_length=T)
    (out * g.double().cpu()).sum().backward()
    for b, L in enumerate(lens):
        assert (y[b, :L].double().cpu() - out[b, :L]).abs().max().item() < 2e-2
    gx = x.grad.double().cpu()
    assert (gx - x64.grad).abs().max().item() < 3e-2 * x64.grad.abs().max().item() + 1e-4
    for (n, p64), (_, pc) in zip(r64.named_parameters(), rnn.named_parameters()):
        ref = p64.grad
        assert (pc.grad.double().cpu() - ref).abs().max().item() < \
            3e-2 * ref.abs().max().item() + 1e-4, n


# ---- 6. models at wide widths ---------------------------------------------------------------------
WIDE_CTC = {"dropout": 0.0, "encoder": {"conv": [[4, 5, 7, 2], [12, 3, 5, 1]],
                                        "rnn": {"dim": 1280, "bidirectional": True, "layers": 2}}}


def test_ctc_2_layer_bigru_1280_matches_reference_model(cuda_lib):
    """Logits, loss and the GRU / output-layer gradients against the fp64 reference model, with
    the whole-model bars of test_encoder_shapes_gpu.py."""
    from oracle.model_ref import RefCTC
    from speech_b200.models import CTC
    from test_encoder_shapes_gpu import _ctc_batch, _model_grad_ok
    torch.manual_seed(1)
    m = CTC(40, 10, WIDE_CTC)
    ref = RefCTC(40, 10, WIDE_CTC).double()
    ref.load_from_dropin({k: v.double() for k, v in m.state_dict().items()})
    m.cuda()
    batch = _ctc_batch()
    x, y, _, y_lens = m.collate(*batch)
    with torch.no_grad():
        logits = m.forward_impl(x).double().cpu()
    assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == "wide"
    loss = m.loss(batch)
    loss.backward()
    assert cuda_lib.sb_debug_gru_bwd_kernel().decode() == "wide"
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


def test_ctc_bigru_1280_flat_sgd_gradient_equals_autograd(cuda_lib):
    """FlatSGD's in-place gradient sinks (the merged two-direction dW_ih included) at a wide
    width: the same gradients as plain autograd, up to the split-K GEMMs' summation order."""
    from speech_b200.models import CTC
    from speech_b200.optim import FlatSGD
    from test_encoder_shapes_gpu import _ctc_batch
    torch.manual_seed(2)
    ma, mb = CTC(40, 10, WIDE_CTC).cuda(), CTC(40, 10, WIDE_CTC).cuda()
    mb.load_state_dict(ma.state_dict())
    batch = _ctc_batch(seed=3)
    ma.loss(batch).backward()
    opt = FlatSGD(mb, lr=0.0)
    opt.zero_grad()
    mb.loss(batch).backward()
    for (n, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
        assert (pb.grad - pa.grad).abs().max().item() < 1e-4 * pa.grad.abs().max().item() + 1e-6, n


def test_transducer_width_1152_matches_fp64_restatement(cuda_lib):
    """Encoder biGRU-1152 on the wide kernels; the restatement of
    test_transducer_width_100_matches_fp64_restatement."""
    import numpy as np
    import torch.nn.functional as F
    from oracle import rnnt_ref
    from oracle.model_ref import RefEncoder
    from speech_b200.models import Transducer
    torch.manual_seed(0)
    H = 1152
    cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 32, 2]],
                                       "rnn": {"dim": H, "bidirectional": True, "layers": 1}},
           "decoder": {"embedding_dim": 24, "layers": 1}}
    m = Transducer(40, 10, cfg)
    sd = {k: v.double() for k, v in m.state_dict().items()}
    enc = RefEncoder(40, cfg).double()
    enc.load_state_dict({k: v for k, v in sd.items() if k.startswith(("conv.", "rnn."))})
    dec = torch.nn.GRU(24, H, 1, batch_first=True).double()
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


def test_seq2seq_dim_1280_trains_and_decodes(cuda_lib):
    import numpy as np
    from speech_b200.models import Seq2Seq
    from test_seq2seq_gpu import _cfg
    torch.manual_seed(3)
    V = 11
    m = Seq2Seq(40, V, _cfg(1280)).cuda()
    rng = np.random.RandomState(3)
    inputs = [rng.randn(60 - 5 * i, 40).astype(np.float32) for i in range(3)]
    labels = [[V - 1] + rng.randint(0, V - 2, 5).tolist() + [V - 2] for _ in range(3)]
    batch = (inputs, labels)
    loss = m.loss(batch)
    loss.backward()
    assert cuda_lib.sb_debug_gru_fwd_kernel().decode() == "wide"
    assert torch.isfinite(loss).item()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)
    m.set_eval()
    hyps = m.infer(batch, max_len=10)
    assert len(hyps) == 3
