"""Drop-in for `transducer.functions.transducer` of awni/transducer, which the reference imports at
speech/models/transducer_model.py:11 (call site :46-52; dependency cloned by Makefile:10-12).

    loss = TransducerLoss()(log_probs, labels, x_lens, y_lens)      # 1-element tensor

    log_probs  (B, T, U+1, V+1) log-softmax on the CUDA device (the reference applies log_softmax
               itself, transducer_model.py:76); gradient flows to it
    labels     IntTensor flat (sum(y_lens),);  x_lens, y_lens IntTensor (B,)   (CPU or CUDA)
Blank = last class (transducer_model.py:28); reduction = sum over the minibatch.  Both are
constructor keywords because the un-vendored dependency could not be inspected.
"""
import torch

from .. import _lib, ops


def rnnt_costs_and_grads(log_probs, labels, x_lens, y_lens, blank=None, need_grad=True):
    _lib.require_cuda(log_probs, "log_probs")
    lib = _lib.load()
    lp = log_probs.float().contiguous()
    B, T, U1, V = lp.shape
    if blank is None:
        blank = V - 1
    dev = lp.device
    (lab, offs, ylen, xlen), _ = _lib.pack_labels(labels, y_lens, x_lens, B, dev, lattice_rows=U1)
    nbytes = _lib.workspace_size(lib.sb_rnnt_workspace_size, B, T, U1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    grads = torch.empty_like(lp) if need_grad else None
    with torch.cuda.device(dev):
        sp = _lib.stream_ptr()
        ops._launch("rnnt_fwd_bwd", 0.0,
                    lambda: lib.sb_rnnt_fwd_bwd(lp.data_ptr(), _lib.ptr(grads), lab.data_ptr(),
                                                offs.data_ptr(), ylen.data_ptr(), xlen.data_ptr(),
                                                B, T, U1, V, int(blank), costs.data_ptr(),
                                                ws.data_ptr(), nbytes, sp))
    return costs, grads


class _RNNTFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, log_probs, labels, x_lens, y_lens, blank, size_average):
        costs, grads = rnnt_costs_and_grads(log_probs, labels, x_lens, y_lens, blank,
                                            log_probs.requires_grad)
        loss = costs.sum().reshape(1)
        if size_average:
            loss = loss / log_probs.shape[0]
            if grads is not None:
                grads = grads / log_probs.shape[0]
        ctx.grads = grads
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        g = ctx.grads
        if g is None:
            return (None,) * 6
        return (g * grad_out.reshape(1, 1, 1, 1),) + (None,) * 5


class TransducerLoss(torch.nn.Module):
    def __init__(self, blank=None, size_average=False):
        super().__init__()
        self.blank = blank
        self.size_average = size_average

    def forward(self, log_probs, labels, x_lens, y_lens):
        return _RNNTFunction.apply(log_probs, labels, x_lens, y_lens, self.blank,
                                   self.size_average)


# ------------------------------------------------------------------------------------------------
# Fused joint network + loss: the (B, T', U+1, H) and (B, T', U+1, V+1) tensors of the reference
# (transducer_model.py:71-76) never exist on the training path.
# ------------------------------------------------------------------------------------------------
JOINT_SLAB_FRAMES = 8     # frames whose hidden activations are materialised at a time in backward
JOINT_RESIDENT_MAX_CLASSES = 64   # V+1 up to which fc2's weight can stay resident in the fused kernel
# Cap on one slab's fp32 logits in the large-vocabulary path.  Measured on an H100 80GB HBM3 at a
# 700 W power limit (tools/joint_vocab_bench.py, B=32, T'=247, U+1=100, H=1024), forward + backward:
#   V+1 = 1024: Tc = 1, 2, 4, 8 -> 40.8, 32.5, 27.0, 24.4 ms (host enqueue 30.5, 16.0, 8.1, 5.9 ms)
#   V+1 = 4096: Tc = 1, 2, 4, 8 -> 100.6, 91.8, 84.8, 81.8 ms
# (the same order on a card limited to 400 W: 40.8, 37.9, 32.6, 29.5 ms at V+1 = 1024).
# Keeping a slab's logits in the 50 MB L2 (Tc <= 2 at V+1 = 1024) loses to the larger GEMMs and the
# fewer launches of bigger slabs, so the cap only bounds memory: Tc = 8 up to V+1 = 5120 there.
JOINT_VOCAB_SLAB_BYTES = 512 << 20


def _round_up(x, m):
    return (x + m - 1) // m * m


def joint_uses_slabs(H, V1):
    """True if the joint of width H over V1 classes runs a slab of frames at a time: whenever the
    fused kernel cannot keep fc2's weight in shared memory (V1 > 64, or H too wide for V1, as
    sb_rnnt_joint_resident decides)."""
    return V1 > JOINT_RESIDENT_MAX_CLASSES or not _lib.load().sb_rnnt_joint_resident(H, V1)


def joint_vocab_slab_frames(B, U1, V1, budget=None):
    """Frames per slab of the large-vocabulary joint (forward and backward): as many as keep one
    slab's fp32 logits within `budget` bytes, at most JOINT_SLAB_FRAMES (the limit of
    sb_rnnt_joint_reduce_slab); one frame when a single frame alone exceeds the budget."""
    budget = JOINT_VOCAB_SLAB_BYTES if budget is None else budget
    frame = B * U1 * _round_up(V1, 8) * 4
    return max(1, min(JOINT_SLAB_FRAMES, budget // frame))


def joint_vocab_forward(fxc, fyc, w2b, b2c, ym, blank, lp_full=None, shortlists=None):
    """Joint + log-softmax for any V1 (used for V1 > 64), a slab of frames at a time:
    z = relu(fx + fy) (bf16) -> logits = z W2^T + b2 (f32, GEMM) -> per-row log-sum-exp.
    fxc (B,T,H) f32, fyc (B,U1,H) f32, w2b (V1,H) bf16, b2c (V1,) f32, ym (B,U1-1) int32, all
    contiguous on the device.  Fills lp_full (B,T,U1,V1) f32 if given, and the batch-first
    shortlists (val, idx, meta) of sb_rnnt_shortlist_rows if given (kp = val.shape[3]).
    -> lat (nodes, 2) {log p(blank), log p(label)}, lse (nodes,) log-sum-exp of every node."""
    lib = _lib.load()
    B, T, H = fxc.shape
    U1 = fyc.shape[1]
    V1 = w2b.shape[0]
    dev = fxc.device
    ld = _round_up(V1, 8)
    Tc = min(joint_vocab_slab_frames(B, U1, V1), T)
    lat = torch.empty(T * B * U1, 2, dtype=torch.float32, device=dev)
    lse = torch.empty(T * B * U1, dtype=torch.float32, device=dev)
    z = torch.empty(Tc * B * U1, H, dtype=torch.bfloat16, device=dev)
    logits = torch.empty(Tc * B * U1, ld, dtype=torch.float32, device=dev)
    sp = _lib.stream_ptr()
    for t0 in range(0, T, Tc):
        tc = min(Tc, T - t0)
        ops._launch("rnnt_joint_slab", 0.0,
                    lambda: lib.sb_rnnt_joint_build_slab(fxc.data_ptr(), fyc.data_ptr(),
                                                         z.data_ptr(), B, T, U1, H, t0, tc, sp))
        ops.gemm_bf16_tn(z[:tc * B * U1], w2b, out=logits, bias=b2c)
        ops._launch("rnnt_joint_rows", 0.0,
                    lambda: lib.sb_rnnt_joint_vocab_fwd_rows(logits.data_ptr(), ld, ym.data_ptr(),
                                                             lat.data_ptr(), lse.data_ptr(),
                                                             _lib.ptr(lp_full), B, T, U1, V1,
                                                             int(blank), t0, tc, sp))
        if shortlists is not None:
            val, idx, meta = shortlists
            ops._launch("rnnt_shortlist_rows", 0.0,
                        lambda: lib.sb_rnnt_shortlist_rows(logits.data_ptr(), ld, lse.data_ptr(), B,
                                                           T, U1, V1, int(blank), val.shape[3], t0,
                                                           tc, 1, val.data_ptr(), idx.data_ptr(),
                                                           meta.data_ptr(), sp))
    return lat, lse


def joint_vocab_backward(fxc, fyc, w2b, b2c, ym, garc, lse, blank):
    """Backward of joint_vocab_forward from garc (nodes, 2), the gradient w.r.t. lat, and the
    forward's lse.  Per slab: z, the logits again (same GEMM), dlogits (bf16) and db2 from the row
    kernel, dW2 += dlogits^T z, dz = dlogits W2, then dz is reduced into dfx / dfy.
    -> dfx (B,T,H), dfy (B,U1,H), dw2 (V1,H), db2 (V1,), all f32."""
    lib = _lib.load()
    B, T, H = fxc.shape
    U1 = fyc.shape[1]
    V1 = w2b.shape[0]
    dev = fxc.device
    ld = _round_up(V1, 8)
    Tc = min(joint_vocab_slab_frames(B, U1, V1), T)
    rows_max = Tc * B * U1
    z = torch.empty(rows_max, H, dtype=torch.bfloat16, device=dev)
    logits = torch.empty(rows_max, ld, dtype=torch.float32, device=dev)
    dl = torch.empty(rows_max, ld, dtype=torch.bfloat16, device=dev)
    dz = torch.empty(rows_max, H, dtype=torch.float32, device=dev)
    dw2 = torch.zeros(V1, H, dtype=torch.float32, device=dev)
    db2 = torch.zeros(V1, dtype=torch.float32, device=dev)
    dfx = torch.empty(B, T, H, dtype=torch.float32, device=dev)
    dfy = torch.zeros(B, U1, H, dtype=torch.float32, device=dev)
    sp = _lib.stream_ptr()
    for t0 in range(0, T, Tc):
        tc = min(Tc, T - t0)
        rows = tc * B * U1
        ops._launch("rnnt_joint_slab", 0.0,
                    lambda: lib.sb_rnnt_joint_build_slab(fxc.data_ptr(), fyc.data_ptr(),
                                                         z.data_ptr(), B, T, U1, H, t0, tc, sp))
        ops.gemm_bf16_tn(z[:rows], w2b, out=logits, bias=b2c)
        ops._launch("rnnt_joint_rows", 0.0,
                    lambda: lib.sb_rnnt_joint_vocab_bwd_rows(logits.data_ptr(), ld, lse.data_ptr(),
                                                             garc.data_ptr(), ym.data_ptr(),
                                                             dl.data_ptr(), ld, db2.data_ptr(), B, T,
                                                             U1, V1, int(blank), t0, tc, sp))
        dlv = dl[:rows, :V1]
        # dW2 (V1 x H) += dlogits^T z   (token-major operands, MN-major wgmma)
        ops.gemm_bf16_tn(dlv, z[:rows], out=dw2, accumulate=True, a_mn=True, b_mn=True)
        # dz (rows x H) = dlogits W2    (W2 is the [K][N] form of the B operand)
        ops.gemm_bf16_tn(dlv, w2b, out=dz[:rows], b_mn=True)
        ops._launch("rnnt_joint_slab", 0.0,
                    lambda: lib.sb_rnnt_joint_reduce_slab(dz.data_ptr(), z.data_ptr(),
                                                          dfx.data_ptr(), dfy.data_ptr(), B, T,
                                                          U1, H, t0, tc, sp))
    return dfx, dfy, dw2, db2


def _joint_operands(fx, fy, fc2, ymat):
    """fx, fy (f32), fc2's weight (bf16, zero columns up to fx's width), bias (f32) and the label
    matrix (int32), contiguous on fx's device, as the joint kernels take them."""
    H = fx.shape[2]
    fxc, fyc = fx.detach().float().contiguous(), fy.detach().float().contiguous()
    w2 = fc2.weight.detach().to(torch.bfloat16)
    w2 = ops.pad_blocks(w2, 1, 1, w2.shape[1], H).contiguous()
    b2 = fc2.bias.detach().float().contiguous()
    ym = ymat.detach().to(fx.device, torch.int32).contiguous()
    return fxc, fyc, w2, b2, ym


def joint_log_probs(fx, fy, fc2, ymat, blank):
    """Full (B, T, U1, V1) log-probabilities of the joint network (what `Transducer.infer` hands
    to the beam search), from fx = fc1(x) (B,T,H), fy = fc1(pred) (B,U1,H); no autograd.
    fx / fy may carry zero units past fc2's input width (see Transducer.joint_inputs): fc2's
    weight gets zero columns for them."""
    _lib.require_cuda(fx, "fx")
    lib = _lib.load()
    B, T, H = fx.shape
    U1 = fy.shape[1]
    V1 = fc2.weight.shape[0]
    fxc, fyc, w2, b2, ym = _joint_operands(fx, fy, fc2, ymat)
    if joint_uses_slabs(H, V1):
        out = torch.empty(B, T, U1, V1, dtype=torch.float32, device=fx.device)
        joint_vocab_forward(fxc, fyc, w2, b2, ym, blank, lp_full=out)
        return out
    lat = torch.empty(T * B * U1, 2, dtype=torch.float32, device=fx.device)
    out = torch.empty(B, T, U1, V1, dtype=torch.float32, device=fx.device)
    sp = _lib.stream_ptr()
    ops._launch("rnnt_joint", 2.0 * B * T * U1 * H * V1,
                lambda: lib.sb_rnnt_joint_fwd(fxc.data_ptr(), fyc.data_ptr(), w2.data_ptr(),
                                              b2.data_ptr(), ym.data_ptr(), lat.data_ptr(),
                                              out.data_ptr(), B, T, U1, H, V1, int(blank), sp))
    return out


def joint_shortlists(fx, fy, fc2, ymat, blank, kp):
    """Shortlists of the joint's log-probabilities (transducer_decoders.alloc_shortlists' layout,
    kp entries per node) for the beam search where the full lattice is too large to hold: the
    slabs of joint_vocab_forward, so the values are joint_log_probs' entries bit for bit, without
    ever materialising the (B, T, U1, V1) tensor.  Arguments as joint_log_probs."""
    from ..transducer_decoders import alloc_shortlists, shortlists_of_lp
    _lib.require_cuda(fx, "fx")
    B, T, H = fx.shape
    U1 = fy.shape[1]
    V1 = fc2.weight.shape[0]
    if not joint_uses_slabs(H, V1):     # fc2 resident: a lattice small enough to write in full
        return shortlists_of_lp(joint_log_probs(fx, fy, fc2, ymat, blank), kp, blank)
    fxc, fyc, w2, b2, ym = _joint_operands(fx, fy, fc2, ymat)
    sl = alloc_shortlists(B, T, U1, kp, fx.device)
    joint_vocab_forward(fxc, fyc, w2, b2, ym, blank, shortlists=sl)
    return sl


def compact_lattice(fxc, fyc, w2b, b2c, ym, blank):
    """The compact (T, B, U1, 2) lattice {log p(blank), log p(label)} the loss and the Viterbi
    alignment read, from the joint's operands (as _joint_operands returns them): the fused joint
    where fc2 stays resident, else the slab path.  -> lat (nodes, 2), and the slab path's per-node
    log-sum-exp (None from the fused joint)."""
    lib = _lib.load()
    B, T, H = fxc.shape
    U1 = fyc.shape[1]
    V1 = w2b.shape[0]
    if joint_uses_slabs(H, V1):
        return joint_vocab_forward(fxc, fyc, w2b, b2c, ym, blank)
    nodes = T * B * U1
    lat = torch.empty(nodes, 2, dtype=torch.float32, device=fxc.device)
    sp = _lib.stream_ptr()
    ops._launch("rnnt_joint", 2.0 * nodes * H * V1,
                lambda: lib.sb_rnnt_joint_fwd(fxc.data_ptr(), fyc.data_ptr(), w2b.data_ptr(),
                                              b2c.data_ptr(), ym.data_ptr(), lat.data_ptr(), None,
                                              B, T, U1, H, V1, int(blank), sp))
    return lat, None


def rnnt_viterbi(fx, fy, fc2, ymat, labels, x_lens, y_lens, blank):
    """Viterbi (forced) alignment through the Transducer lattice of fx = fc1(x) (B,T,H) and
    fy = fc1(pred) (B,U1,H) (sb_rnnt_viterbi on the loss's compact lattice); no autograd.
    Returns, on the device, frames (B, U1-1) int32 -- the frame at which each label is emitted,
    -1 past y_lens[b] -- and scores (B,) float64, the path's log-probability (-inf where
    x_lens[b] = 0)."""
    _lib.require_cuda(fx, "fx")
    lib = _lib.load()
    B, T = fx.shape[0], fx.shape[1]
    U1 = fy.shape[1]
    dev = fx.device
    fxc, fyc, w2b, b2c, ym = _joint_operands(fx, fy, fc2, ymat)
    (lab, offs, ylen, xlen), _ = _lib.pack_labels(labels, y_lens, x_lens, B, dev, lattice_rows=U1)
    lat, _ = compact_lattice(fxc, fyc, w2b, b2c, ym, blank)
    nbytes = _lib.workspace_size(lib.sb_rnnt_viterbi_workspace_size, B, T, U1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    frames = torch.empty(B, max(U1 - 1, 1), dtype=torch.int32, device=dev)
    scores = torch.empty(B, dtype=torch.float64, device=dev)
    lab_ptr = lab.data_ptr() or offs.data_ptr()   # no labels in the batch: none is read
    sp = _lib.stream_ptr()
    ops._launch("rnnt_viterbi", 0.0,
                lambda: lib.sb_rnnt_viterbi(lat.data_ptr(), lab_ptr, offs.data_ptr(),
                                            ylen.data_ptr(), xlen.data_ptr(), B, T, U1,
                                            frames.data_ptr(), scores.data_ptr(), ws.data_ptr(),
                                            nbytes, sp))
    return frames[:, :U1 - 1], scores


class _JointLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fx, fy, w2, b2, ymat, labels, x_lens, y_lens, blank, size_average):
        _lib.require_cuda(fx, "fx")
        lib = _lib.load()
        B, T, H = fx.shape
        U1 = fy.shape[1]
        V1 = w2.shape[0]
        dev = fx.device
        fxc, fyc = fx.detach().float().contiguous(), fy.detach().float().contiguous()
        w2b = w2.detach().to(torch.bfloat16).contiguous()
        b2c = b2.detach().float().contiguous()
        ym = ymat.detach().to(dev, torch.int32).contiguous()
        (lab, offs, ylen, xlen), _ = _lib.pack_labels(labels, y_lens, x_lens, B, dev,
                                                      lattice_rows=U1)
        nodes = T * B * U1
        lat, lse = compact_lattice(fxc, fyc, w2b, b2c, ym, blank)
        sp = _lib.stream_ptr()
        need = any(ctx.needs_input_grad[:4])
        nbytes = _lib.workspace_size(lib.sb_rnnt_workspace_size, B, T, U1)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        costs = torch.empty(B, dtype=torch.float32, device=dev)
        garc = torch.empty(nodes, 2, dtype=torch.float32, device=dev) if need else None
        ops._launch("rnnt_fwd_bwd", 0.0,
                    lambda: lib.sb_rnnt_fwd_bwd_compact(lat.data_ptr(), _lib.ptr(garc),
                                                        lab.data_ptr(), offs.data_ptr(),
                                                        ylen.data_ptr(), xlen.data_ptr(), B, T, U1,
                                                        int(blank), costs.data_ptr(), ws.data_ptr(),
                                                        nbytes, sp))
        loss = costs.sum().reshape(1)
        scale = 1.0 / B if size_average else 1.0
        ctx.saved = (fxc, fyc, w2b, b2c, ym, garc)
        ctx.dims = (B, T, U1, H, V1, int(blank), scale)
        ctx.lse = lse
        return loss * scale

    @staticmethod
    def backward(ctx, grad_out):
        lib = _lib.load()
        fxc, fyc, w2b, b2c, ym, garc = ctx.saved
        B, T, U1, H, V1, blank, scale = ctx.dims
        dev = fxc.device
        if garc is None:
            return (None,) * 10
        garc = garc * (grad_out.reshape(1, 1).float() * scale)
        nodes = T * B * U1
        if ctx.lse is not None:                   # the forward ran the slab path
            dfx, dfy, dw2, db2 = joint_vocab_backward(fxc, fyc, w2b, b2c, ym, garc, ctx.lse, blank)
            return dfx, dfy, dw2, db2, None, None, None, None, None, None
        NV = 32 if V1 <= 32 else 64
        dlog = torch.empty(nodes, NV, dtype=torch.bfloat16, device=dev)
        db2 = torch.zeros(V1, dtype=torch.float32, device=dev)
        sp = _lib.stream_ptr()
        # recompute pass: logits -> softmax -> gradient w.r.t. the logits (bf16 rows)
        ops._launch("rnnt_joint", 2.0 * nodes * H * V1,
                    lambda: lib.sb_rnnt_joint_dlogits(fxc.data_ptr(), fyc.data_ptr(), w2b.data_ptr(),
                                                      b2c.data_ptr(), ym.data_ptr(), garc.data_ptr(),
                                                      dlog.data_ptr(), db2.data_ptr(), B, T, U1, H,
                                                      V1, blank, sp))
        # weight / input gradients, a slab of frames at a time: the hidden activations of Tc
        # frames (z, bf16) and their gradient (dz, f32) are the only (.., H)-wide temporaries
        Tc = max(1, min(JOINT_SLAB_FRAMES, T))
        rows_max = Tc * B * U1
        z = torch.empty(rows_max, H, dtype=torch.bfloat16, device=dev)
        dz = torch.empty(rows_max, H, dtype=torch.float32, device=dev)
        dw2 = torch.zeros(NV, H, dtype=torch.float32, device=dev)
        dfx = torch.empty(B, T, H, dtype=torch.float32, device=dev)
        dfy = torch.zeros(B, U1, H, dtype=torch.float32, device=dev)
        w2p = torch.zeros(NV, H, dtype=torch.bfloat16, device=dev)
        w2p[:V1] = w2b
        for t0 in range(0, T, Tc):
            tc = min(Tc, T - t0)
            rows = tc * B * U1
            dl = dlog[t0 * B * U1:t0 * B * U1 + rows]
            ops._launch("rnnt_joint_slab", 0.0,
                        lambda: lib.sb_rnnt_joint_build_slab(fxc.data_ptr(), fyc.data_ptr(),
                                                             z.data_ptr(), B, T, U1, H, t0, tc, sp))
            # dW2 (NV x H) += dlogits^T z   (token-major operands, MN-major UMMA)
            ops.gemm_bf16_tn(dl, z[:rows], out=dw2, accumulate=True, a_mn=True, b_mn=True)
            # dz (rows x H) = dlogits W2    (W2 is the [K][N] form of the B operand)
            ops.gemm_bf16_tn(dl, w2p, out=dz[:rows], b_mn=True)
            ops._launch("rnnt_joint_slab", 0.0,
                        lambda: lib.sb_rnnt_joint_reduce_slab(dz.data_ptr(), z.data_ptr(),
                                                              dfx.data_ptr(), dfy.data_ptr(), B, T,
                                                              U1, H, t0, tc, sp))
        return dfx, dfy, dw2[:V1], db2, None, None, None, None, None, None


class JointTransducerLoss(torch.nn.Module):
    """fc2 + log-softmax + transducer loss on fx = fc1(x), fy = fc1(pred) without the 4-D tensors:
    loss = JointTransducerLoss()(fx, fy, fc2.weight, fc2.bias, ymat, labels, x_lens, y_lens)."""

    def __init__(self, blank=None, size_average=False):
        super().__init__()
        self.blank = blank
        self.size_average = size_average

    def forward(self, fx, fy, w2, b2, ymat, labels, x_lens, y_lens):
        blank = w2.shape[0] - 1 if self.blank is None else self.blank
        return _JointLossFunction.apply(fx, fy, w2, b2, ymat, labels, x_lens, y_lens, blank,
                                        self.size_average)
