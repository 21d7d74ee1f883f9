"""Host-side operators over the C ABI: dense contraction and the (bi)GRU stack.

PyTorch is used here for device memory, streams and autograd plumbing only; the arithmetic of
the recurrence and of every projection runs in the hand-written sm_90a kernels of csrc/.
Internal activations are TIME-MAJOR with the batch padded to a multiple of 8 (row m = t*Bp + b).
"""
import ctypes

import torch

from . import _lib

GEMM_ACCUMULATE = 1
GEMM_ROW_REMAP = 2
GEMM_A_MN = 4
GEMM_B_MN = 8


def _round_up(x, m):
    return (x + m - 1) // m * m


def pad_blocks(t, dim, blocks, n, n_pad):
    """Dimension `dim` of t as `blocks` consecutive blocks of n entries -> blocks of n_pad, each
    block's new tail zero (autograd-aware; t itself when n_pad == n).  This is how GRU layers run
    at the kernels' width: gate blocks (r|z|n) of the weight rows and biases, direction blocks
    (fwd|rev) of the next layer's input columns, and the conv stack's channels."""
    if n_pad == n:
        return t
    dim %= t.dim()
    shape = tuple(t.shape)
    v = t.reshape(shape[:dim] + (blocks, n) + shape[dim + 1:])
    v = torch.nn.functional.pad(v, [0, 0] * (len(shape) - dim - 1) + [0, n_pad - n])
    return v.reshape(shape[:dim] + (blocks * n_pad,) + shape[dim + 1:])


def unpad_blocks(t, dim, blocks, n, n_pad):
    """Inverse of pad_blocks: the first n entries of each n_pad-block of dimension `dim`."""
    if n_pad == n:
        return t
    dim %= t.dim()
    shape = tuple(t.shape)
    v = t.reshape(shape[:dim] + (blocks, n_pad) + shape[dim + 1:]).narrow(dim + 1, 0, n)
    return v.reshape(shape[:dim] + (blocks * n,) + shape[dim + 1:])


def pad_gru_layer(w_ih, w_hh, b_ih, b_hh, H, Hp, in_dirs):
    """One direction's nn.GRU parameters of hidden size H as those of a GRU of size Hp whose
    units H..Hp-1 (per gate) are zero: exact, because a zero unit with h_0 = 0 stays 0
    (r = z = 1/2, n = tanh(0) = 0, h_t = h_{t-1} / 2) and its zero W_hh column never reaches a
    real unit.  in_dirs: 0 for the first layer (its input is not padded), else the number of
    directions of the layer below, whose outputs arrive as in_dirs blocks of Hp columns."""
    w_ih = pad_blocks(w_ih, 0, 3, H, Hp)
    if in_dirs:
        w_ih = pad_blocks(w_ih, 1, in_dirs, H, Hp)
    return (w_ih, pad_blocks(pad_blocks(w_hh, 0, 3, H, Hp), 1, 1, H, Hp),
            pad_blocks(b_ih, 0, 3, H, Hp), pad_blocks(b_hh, 0, 3, H, Hp))


def gru_padded_width(Bp, H, ndir):
    """The width the recurrence kernels run a layer of H units at (sb_gru_plan); raises if none."""
    hp = ctypes.c_int(0)
    _lib.check(_lib.load().sb_gru_plan(Bp, H, ndir, ctypes.byref(hp)),
               "sb_gru_plan (H = %d, %d direction(s), %d batch rows)" % (H, ndir, Bp))
    return hp.value


def _apply_env_knobs():
    """Developer knobs (profiling under ncu cannot replay clustered cooperative launches):
    SB_GRU_KSPLIT=0 disables the K-split backward kernel, SB_GRU_CLUSTER=<1|2|4|8> sets the
    preferred cluster size of the other GRU kernels, SB_GRU_FLAGS=<int> sets sb_debug_gru_flags
    (e.g. 512: no L2 reduce-scatter mode, the backward's two clustered one-direction launches at
    H = 1024; 256: that mode wherever the K-split backward kernel applies), SB_GEMM_FLAGS=<int>
    sets sb_debug_gemm_flags (bits: 1 = the 128 x 128 one-CTA GEMM kernel instead of the 128 x 256
    one over 2-CTA clusters; 2 = that kernel stores its output straight from the registers instead
    of through shared memory and TMA; 4 = it stores no output at all, for timing only),
    SB_CONV_FLAGS=1 runs every conv layer on im2col + GEMM (no direct-convolution kernels)."""
    import os
    global _conv_flags
    lib = _lib.load()
    _conv_flags = int(os.environ.get("SB_CONV_FLAGS", "0"))
    if os.environ.get("SB_GRU_KSPLIT") is not None:
        lib.sb_debug_gru_ksplit(int(os.environ["SB_GRU_KSPLIT"]))
    if os.environ.get("SB_GRU_CLUSTER") is not None:
        lib.sb_debug_gru_cluster(int(os.environ["SB_GRU_CLUSTER"]))
    if os.environ.get("SB_GRU_FLAGS") is not None:
        lib.sb_debug_gru_flags(int(os.environ["SB_GRU_FLAGS"]))
    if os.environ.get("SB_GEMM_FLAGS") is not None:
        lib.sb_debug_gemm_flags(int(os.environ["SB_GEMM_FLAGS"]))


_knobs_applied = False
_conv_flags = 0


def _ensure_knobs():
    global _knobs_applied
    if not _knobs_applied:
        _knobs_applied = True
        _apply_env_knobs()


# ---- optional per-kernel timing (CUDA events on the launching stream; used by bench.py) ----
_prof = None
_prof_detail = False      # developer: one profile class per GEMM shape (tools/debug_step.py)


def profile_begin():
    global _prof
    _prof = []


def profile_end():
    """-> {kernel class: (launches, total ms, total algorithmic FLOPs)}"""
    global _prof
    rec, _prof = _prof, None
    torch.cuda.synchronize()
    out = {}
    for name, flops, e0, e1 in rec or []:
        n, ms, fl = out.get(name, (0, 0.0, 0.0))
        out[name] = (n + 1, ms + e0.elapsed_time(e1), fl + flops)
    return out


def _launch(name, flops, fn):
    """Run one C-ABI launch; counts it and, when profiling, brackets it with CUDA events."""
    _ensure_knobs()
    _lib.launch_count += 1
    if _prof is None:
        return _lib.check(fn(), name)
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = fn()
    e1.record()
    _prof.append((name, flops, e0, e1))
    return _lib.check(rc, name)


def gemm_bf16_tn(A, B, out=None, bias=None, accumulate=False, split_k=1, remap=None,
                 a_mn=False, b_mn=False):
    """out[M,N] (f32) (+)= A[M,K] (bf16) @ B[N,K]^T (bf16) (+ bias).  A/B may be row-strided views.

    a_mn / b_mn: that operand is given as [K][M] / [K][N] (the contraction runs over its rows).
    remap=(Bp, T, valid_B): rows m = t*Bp + b are written batch-first to row b*T + t.
    """
    lib = _lib.load()
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    assert A.stride(1) == 1 and B.stride(1) == 1
    K, M = A.shape if a_mn else (A.shape[1], A.shape[0])
    Kb, N = B.shape if b_mn else (B.shape[1], B.shape[0])
    assert K == Kb
    flags = (GEMM_A_MN if a_mn else 0) | (GEMM_B_MN if b_mn else 0)
    rB = rT = vB = 0
    if remap is not None:
        rB, rT, vB = remap
        flags |= GEMM_ROW_REMAP
        rows = vB * rT
    else:
        rows = M
    if out is None:
        assert not accumulate
        out = torch.empty(rows, N, dtype=torch.float32, device=A.device)
    assert out.dtype == torch.float32 and out.stride(1) == 1 and out.shape[0] >= rows
    if accumulate:
        flags |= GEMM_ACCUMULATE
    sp = _lib.stream_ptr()
    name = "gemm_bf16_tn"
    if _prof_detail:
        name = "gemm %dx%dx%d%s%s%s" % (M, N, K, " aT" if a_mn else "", " bT" if b_mn else "",
                                       " acc" if accumulate else "")
    _launch(name, 2.0 * M * N * K,
            lambda: lib.sb_gemm_bf16_tn(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0),
                                        out.data_ptr(), out.stride(0), _lib.ptr(bias), M, N, K,
                                        flags, split_k, rB, rT, vB, sp))
    return out


# ------------------------------------------------------------------------------------------------
# "Parity mode" (SURVEY.md section 7): the forward pass of the encoder in reference precision, to
# measure the bf16 tensor-core path against.  Dense contractions run as 3-pass split-bf16 GEMMs
# (x = hi + lo with hi = bf16(x), lo = bf16(x - hi): hi*hi + hi*lo + lo*hi on the tensor cores,
# relative error ~2^-16), the recurrence in plain fp32 (csrc/gru_f32.cu).  No autograd.
# ------------------------------------------------------------------------------------------------
def _split_bf16(t, Kp):
    t = t.detach().float()
    hi = t.to(torch.bfloat16)
    lo = (t - hi.float()).to(torch.bfloat16)
    if Kp != t.shape[1]:
        hi = torch.nn.functional.pad(hi, (0, Kp - t.shape[1]))
        lo = torch.nn.functional.pad(lo, (0, Kp - t.shape[1]))
    return hi.contiguous(), lo.contiguous()


def gemm_split(A, B, bias=None, remap=None):
    """A (M,K) f32 @ B (N,K)^T f32 -> (M,N) f32 with split-bf16 operands (3 tensor-core passes)."""
    Kp = _round_up(A.shape[1], 8)
    a_hi, a_lo = _split_bf16(A, Kp)
    b_hi, b_lo = _split_bf16(B, Kp)
    out = gemm_bf16_tn(a_hi, b_hi, bias=bias, remap=remap)
    gemm_bf16_tn(a_hi, b_lo, out=out, accumulate=True, remap=remap)
    gemm_bf16_tn(a_lo, b_hi, out=out, accumulate=True, remap=remap)
    return out


def encode_logits_parity(x, conv, rnn, fc):
    """Reference-precision forward of conv stack -> GRU stack -> halves-sum -> fc (no grad):
    x (B,T,F) -> logits (B,T',V).  Same kernels' layouts, split-bf16 GEMMs, fp32 recurrence."""
    _lib.require_cuda(x, "x")
    lib = _lib.load()
    dev = x.device
    B, Ti, Fi = x.shape
    sp = _lib.stream_ptr()
    cur = x.detach().float().contiguous()              # (B, Ti, Fi, Ci) channels-last, Ci = 1
    Ci = 1
    for l, c in enumerate(m for m in conv.children() if isinstance(m, torch.nn.Conv2d)):
        kh, kw, s_ = c.kernel_size[0], c.kernel_size[1], c.stride[0]
        Co = c.out_channels
        K = kh * kw * Ci
        Kp = _round_up(K, 8)
        To, Fo = (Ti - kh) // s_ + 1, (Fi - kw) // s_ + 1
        M = B * To * Fo
        r = cur if l == 0 else torch.relu(cur)
        r_hi = r.to(torch.bfloat16).float()
        parts = []
        for src in (r_hi, r - r_hi):                   # im2col of the hi and lo halves (exact)
            A = torch.empty(M, Kp, dtype=torch.bfloat16, device=dev)
            _launch("conv_im2col", 0.0,
                    lambda: lib.sb_conv_im2col(src.data_ptr(), None, 1.0, A.data_ptr(), B, Ti, Fi,
                                               Ci, kh, kw, s_, Kp, 0, sp))
            parts.append(A)
        W = torch.zeros(Co, Kp, dtype=torch.float32, device=dev)
        W[:, :K] = c.weight.detach().float().permute(0, 2, 3, 1).reshape(Co, K)
        w_hi, w_lo = _split_bf16(W, Kp)
        C = gemm_bf16_tn(parts[0], w_hi, bias=c.bias.detach().float().contiguous())
        gemm_bf16_tn(parts[0], w_lo, out=C, accumulate=True)
        gemm_bf16_tn(parts[1], w_hi, out=C, accumulate=True)
        cur, Ti, Fi, Ci = C, To, Fo, Co
    feats = torch.empty(B, Ti, Ci * Fi, dtype=torch.float32, device=dev)
    _launch("conv_relu_to_bct", 0.0,
            lambda: lib.sb_conv_relu_to_bct(cur.data_ptr(), None, 1.0, feats.data_ptr(), B, Ti, Fi,
                                            Ci, sp))
    ndir, weights = _gru_weights(rnn)
    H = rnn.hidden_size
    T = Ti
    Bp = _round_up(B, 8)
    M = T * Bp
    X = torch.zeros(T, Bp, feats.shape[2], dtype=torch.float32, device=dev)
    X[:, :B] = feats.transpose(0, 1)
    X = X.view(M, -1)
    barrier = torch.zeros(2, dtype=torch.int32, device=dev)
    for l in range(rnn.num_layers):
        wl = weights[l * 4 * ndir:(l + 1) * 4 * ndir]
        w_ih = torch.cat([wl[d * 4].detach().float() for d in range(ndir)])
        b_ih = torch.cat([wl[d * 4 + 2].detach().float() for d in range(ndir)]).contiguous()
        w_hh = torch.stack([wl[d * 4 + 1].detach().float() for d in range(ndir)]).contiguous()
        b_hh = torch.stack([wl[d * 4 + 3].detach().float() for d in range(ndir)]).contiguous()
        gi = gemm_split(X, w_ih, bias=b_ih)
        y = torch.empty(M, ndir * H, dtype=torch.float32, device=dev)
        _launch("gru_fwd_f32", 2.0 * M * 3 * H * H * ndir,
                lambda: lib.sb_gru_fwd_f32(gi.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(),
                                           y.data_ptr(), barrier.data_ptr(), T, Bp, H, ndir, sp))
        X = y
    w = fc.weight.detach().float()
    wcat = torch.cat([w, w], 1) if ndir == 2 else w
    V = w.shape[0]
    return gemm_split(X, wcat, bias=fc.bias.detach().float().contiguous(),
                      remap=(Bp, T, B)).view(B, T, V)


class LinearFunction(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM (bf16 operands, fp32 accumulate), forward and backward:
    the arithmetic behind the reference's LinearND / nn.Linear (model.py:115-133).
    x (N, K) f32, W (O, K), b (O) -> (N, O) f32."""

    @staticmethod
    def forward(ctx, x, w, b):
        _lib.require_cuda(x, "x")
        N, K = x.shape
        Kp = _round_up(K, 8)
        xb = x.detach().to(torch.bfloat16)
        wb = w.detach().to(torch.bfloat16)
        if Kp != K:
            xb = torch.nn.functional.pad(xb, (0, Kp - K))
            wb = torch.nn.functional.pad(wb, (0, Kp - K))
        xb, wb = xb.contiguous(), wb.contiguous()
        ctx.save_for_backward(xb, wb)
        ctx.K = K
        ctx.has_bias = b is not None
        return gemm_bf16_tn(xb, wb, bias=None if b is None else b.detach().float().contiguous())

    @staticmethod
    def backward(ctx, dy):
        xb, wb = ctx.saved_tensors
        K = ctx.K
        O = wb.shape[0]
        Op = _round_up(O, 8)
        dyb = dy.detach().to(torch.bfloat16)
        if Op != O:
            dyb = torch.nn.functional.pad(dyb, (0, Op - O))
            wb = torch.nn.functional.pad(wb, (0, 0, 0, Op - O))
        dyb, wb = dyb.contiguous(), wb.contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = gemm_bf16_tn(dyb, wb, b_mn=True)[:, :K]          # dY W: W is the [K][N] form
        if ctx.needs_input_grad[1]:
            dw = torch.zeros(Op, xb.shape[1], dtype=torch.float32, device=dy.device)
            gemm_bf16_tn(dyb, xb, out=dw, accumulate=True, a_mn=True, b_mn=True)   # dY^T X
            dw = dw[:O, :K]
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum(0)
        return dx, dw, db


def linear(x, w, b=None):
    """nn.Linear semantics over the last dimension of an N-D CUDA tensor, on the wgmma GEMM."""
    lead = x.shape[:-1]
    out = LinearFunction.apply(x.reshape(-1, x.shape[-1]).float(), w, b)
    return out.view(*lead, out.shape[-1])


_gru_operands = {}


def register_gru_operands(first_w_ih, entry):
    """optim.FlatSGD: operands of one GRU layer as views of its flat buffers (see there)."""
    _gru_operands[id(first_w_ih)] = entry


def _cached_gru_operands(w_ih0, Kl):
    e = _gru_operands.get(id(w_ih0))
    if e is None or e["wih"].shape[1] != Kl or e["params"][0] is not w_ih0:
        return None
    if any(q._version != v for q, v in zip(e["params"], e["versions"])):
        return None          # modified outside FlatSGD.step(): fall back to casting the fp32 values
    return e


_grad_ready_hook = None
_announce = True
_grad_sink_enabled = False


def set_grad_sink(enabled):
    """Opt-in (optim.FlatSGD): let the weight-gradient GEMMs of GRUStackFunction.backward
    accumulate straight into the parameters' existing .grad buffers and return None to autograd
    for them.  Off by default, so that torch.autograd.grad, gradcheck, tensor hooks and gradient
    accumulation see ordinary returned gradients."""
    global _grad_sink_enabled
    _grad_sink_enabled = bool(enabled)


_grad_guard = None


def set_grad_ready_hook(fn, guard=None):
    """fn(list_of_parameters) is called from inside GRUStackFunction.backward as soon as the
    gradients of one layer's parameters are final in their .grad buffers (all producing kernels
    enqueued on the current stream).  Used by optim.FlatSGD to start that layer's all-reduce
    while the layers below are still being differentiated.  None disables.
    guard(parameters) (optional) runs at the START of every announcing backward of a GRU stack,
    before any gradient buffer is touched: it raises if gradients of these parameters were
    already announced in this step (a second backward pass would add local gradients into
    slices that are being all-reduced)."""
    global _grad_ready_hook, _grad_guard
    _grad_ready_hook = fn
    _grad_guard = guard if fn is not None else None


def _bias_sink(param):
    if not _grad_sink_enabled:
        return None
    g = getattr(param, "grad", None)
    if g is None or not g.is_cuda or g.dtype != torch.float32:
        return None
    return g


def _grad_sink(param, rows=None):
    """The parameter's existing .grad (optionally a row slice) if the weight-gradient GEMM can
    accumulate straight into it (fp32, contiguous, 16-byte aligned rows), else None.  Writing
    dW with the GEMM's reduce-add epilogue into .grad replaces a zero-filled temporary plus
    autograd's separate `grad += dW` pass (the gradient-accumulation fusion used by large-model
    trainers); the Function then returns None for that parameter."""
    if not _grad_sink_enabled:
        return None
    g = getattr(param, "grad", None)
    if g is None or not g.is_cuda or g.dtype != torch.float32 or not g.is_contiguous():
        return None
    if g.dim() != 2 or (g.stride(0) % 4) != 0 or (g.data_ptr() % 16) != 0:
        return None
    return g if rows is None else g[rows[0]:rows[1]]


def time_align(src, lens_dev, T, Bp, right, out=None):
    """Per-utterance shift of the rows of a time-major [T*Bp][cols] matrix (row m = t*Bp + b):
    right=True moves row (t, b) to (t + T - len_b, b), right=False moves it back; vacated rows are
    zero.  src / out may be column blocks of wider matrices; lens_dev: (Bp,) int32 on the device."""
    lib = _lib.load()
    M, cols = src.shape
    assert M == T * Bp and src.stride(1) == 1 and src.dtype in (torch.bfloat16, torch.float32)
    if out is None:
        out = torch.empty(M, cols, dtype=src.dtype, device=src.device)
    assert out.shape == src.shape and out.dtype == src.dtype and out.stride(1) == 1
    sp = _lib.stream_ptr()
    _launch("time_align", 0.0,
            lambda: lib.sb_time_align(src.data_ptr(), src.stride(0), out.data_ptr(), out.stride(0),
                                      lens_dev.data_ptr(), T, Bp, cols, src.element_size(),
                                      1 if right else 0, sp))
    return out


def _align_reverse(a, lens_dev, T, Bp, half, right):
    """[M][2*half] with its reverse-direction half (columns half..) aligned (see time_align)."""
    out = torch.empty_like(a)
    out[:, :half].copy_(a[:, :half])
    time_align(a[:, half:], lens_dev, T, Bp, right, out=out[:, half:])
    return out


def _lens_operands(lens, B, T, Bp, dev):
    """Exact-lengths mode of the GRU stack: (Bp,) int32 device lengths (padding rows of the batch
    count as full length) and the (B, T, 1) f32 mask of valid frames, or None when every utterance
    fills the padded T (nothing to align or mask)."""
    if lens is None:
        return None
    ln = torch.as_tensor(lens).detach().to("cpu", torch.int64).reshape(-1)
    if ln.numel() != B:
        raise ValueError("lens must have one entry per utterance (%d), got %d" % (B, ln.numel()))
    if B and (int(ln.min()) < 0 or int(ln.max()) > T):
        raise ValueError("lens must lie in [0, T] (T = %d)" % T)
    if bool((ln == T).all()):
        return None
    full = torch.full((Bp,), T, dtype=torch.int32)
    full[:B] = ln.to(torch.int32)
    lens_dev = full.pin_memory().to(dev, non_blocking=True)
    valid = (torch.arange(T, device=dev)[None, :] < lens_dev[:B, None].long())
    return lens_dev, valid.unsqueeze(2).float()


def _workspace(nbytes, dev):
    """1024-byte aligned scratch for one recurrence launch (counters + exchange tiles)"""
    buf = torch.empty(nbytes + 1024, dtype=torch.uint8, device=dev)
    off = (-buf.data_ptr()) % 1024
    return buf[off:off + nbytes]


def gru_layer_operands(wl, l, Kl, ndir, H, Hp, dev):
    """The recurrence's operands of GRU layer l at width Hp from its nn.GRU parameters wl (w_ih,
    w_hh, b_ih, b_hh per direction) and an input of Kl columns: (wih_cat [ndir*3Hp][Kl] bf16,
    whh [ndir][3Hp][Hp] bf16, bih_cat [ndir*3Hp] f32, bhh [ndir][3Hp] f32)."""
    K3 = 3 * Hp
    cached = _cached_gru_operands(wl[0], Kl) if Hp == H else None
    if cached is not None:
        # views of the optimizer's flat buffers (bf16 shadow written by sgd_clip_step)
        return cached["wih"], cached["whh"], cached["bih"], cached["bhh"]
    # (w_ih, w_hh, b_ih, b_hh) of each direction at the kernels' width
    lw = [pad_gru_layer(*[q.detach() for q in wl[d * 4:d * 4 + 4]], H, Hp,
                        ndir if l > 0 else 0) for d in range(ndir)]
    In_l = lw[0][0].shape[1]
    # bf16 operand copies of the master weights: one fused cast+copy per matrix
    wih_cat = (torch.empty if Kl == In_l else torch.zeros)(
        ndir * K3, Kl, dtype=torch.bfloat16, device=dev)
    whh = torch.empty(ndir, K3, Hp, dtype=torch.bfloat16, device=dev)
    for d in range(ndir):
        wih_cat[d * K3:(d + 1) * K3, :In_l].copy_(lw[d][0])
        whh[d].copy_(lw[d][1])
    bih_cat = torch.cat([q[2] for q in lw]).float().contiguous()
    bhh = torch.stack([q[3] for q in lw]).float().contiguous()
    return wih_cat, whh, bih_cat, bhh


def fc_operand(fc_w, ndir, H, Hp):
    """[W | W] (one W per direction) bf16 at the layer width Hp: the B operand of the output
    projection fused with the sum of the direction halves."""
    wcat = fc_w.detach().to(torch.bfloat16)
    if ndir == 2:
        wcat = torch.cat([wcat, wcat], 1)
    return pad_blocks(wcat, 1, ndir, H, Hp).contiguous()


class GRUStackFunction(torch.autograd.Function):
    """Multi-layer (bi)directional GRU, semantics of nn.GRU(batch_first=True) with h0 = 0.

    forward(x (B,T,In) f32 cuda, ndir, H, train, *weights) -> (B,T,ndir*H) f32
    weights: per layer, per direction: w_ih (3H,In_l), w_hh (3H,H), b_ih (3H), b_hh (3H)
    (the parameter order of nn.GRU: weight_ih_l{k}[_reverse], weight_hh_..., bias_ih_..., bias_hh_...)

    lens (optional, B ints): valid frames per utterance, the semantics of nn.GRU over
    pack_padded_sequence.  The reverse direction runs on right-aligned operands (time_align), so
    it starts at each utterance's own last frame; its gates and states stay in those aligned
    coordinates for the backward pass, and its half of each layer output is left-aligned again.
    The gradient arriving at output frames >= len_b is ignored (and without the fused projection
    those output rows are zero), so frames >= len_b of x receive exactly zero gradient.

    Every layer runs at the kernels' width Hp = gru_padded_width(Bp, H, ndir) >= H: when Hp > H
    the bf16 operands are built with zero units (pad_gru_layer), all internal activations carry
    ndir blocks of Hp columns, and the outputs and gradients are sliced back to H.
    """

    @staticmethod
    def forward(ctx, x, ndir, H, dropout, fc_w, fc_b, lens, la_w, *weights):
        """fc_w/fc_b (optional): fuse `LinearND(sum of direction halves)` (reference
        model.py:75-77 + ctc_model.py:29) as ONE contraction on the bf16 top-layer output:
        (h_f + h_b) W^T = [h_f | h_b] [W | W]^T, written batch-first by the GEMM epilogue.
        la_w (optional, ndir = 1 only): the (H, 1, tau + 1) weight of a lookahead convolution
        over the top layer's output (sb_lookahead_fwd, exact-lengths `lens` honoured); the fused
        projection then reads its bf16 output, and the unfused path returns its fp32 output."""
        _lib.require_cuda(x, "x")
        lib = _lib.load()
        B, T, In = x.shape
        dev = x.device
        L = len(weights) // (4 * ndir)
        Bp = _round_up(B, 8)
        if Bp > 128:
            raise _lib.SpeechB200Error("per-GPU batch > 128 not supported by the GRU kernel yet")
        M = T * Bp
        Hp = gru_padded_width(Bp, H, ndir)
        D = ndir * Hp
        K3 = 3 * Hp
        need_grad = any(ctx.needs_input_grad)     # all False under torch.no_grad()
        lo = _lens_operands(lens, B, T, Bp, dev)
        al, valid = lo if lo is not None else (None, None)
        la_lens = al
        if ndir == 1:
            al = None                             # the forward direction is causal

        # layer-0 operand: time-major, batch padded, K padded to a multiple of 8, bf16
        Inp = _round_up(In, 8)
        if B == Bp and In == Inp:
            X = x.detach().transpose(0, 1).to(torch.bfloat16).reshape(M, Inp)
        else:
            X = torch.zeros(T, Bp, Inp, dtype=torch.bfloat16, device=dev)
            X[:, :B, :In] = x.transpose(0, 1)
            X = X.view(M, Inp)
        nbytes = _lib.workspace_size(lib.sb_gru_fwd_workspace_size, Bp, Hp, ndir)
        ws = _workspace(nbytes, dev)
        saved = []
        y = None
        for l in range(L):
            wl = weights[l * 4 * ndir:(l + 1) * 4 * ndir]
            wih_cat, whh, bih_cat, bhh = gru_layer_operands(wl, l, X.shape[1], ndir, H, Hp, dev)
            if al is None:
                gi = gemm_bf16_tn(X, wih_cat, bias=bih_cat)
            else:
                # the reverse projection reads the right-aligned layer input
                gi = torch.empty(M, 2 * K3, dtype=torch.float32, device=dev)
                gemm_bf16_tn(X, wih_cat[:K3], out=gi[:, :K3], bias=bih_cat[:K3])
                gemm_bf16_tn(time_align(X, al, T, Bp, right=True), wih_cat[K3:], out=gi[:, K3:],
                             bias=bih_cat[K3:])
            y = torch.empty(M, D, dtype=torch.float32, device=dev)
            xn = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
            gates = None
            if need_grad:
                gates = torch.empty(M, ndir, 4, Hp, dtype=torch.float32, device=dev)
            sp = _lib.stream_ptr()
            _launch("gru_fwd", 2.0 * M * 3 * Hp * Hp * ndir,
                    lambda: lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(),
                                           y.data_ptr(), xn.data_ptr(), _lib.ptr(gates),
                                           ws.data_ptr(), nbytes, T, Bp, Hp, ndir, sp))
            mask = None
            hb = xn                                     # bf16 h_t (un-masked): dW_hh operand
            y_rec = y                                   # as the recurrence wrote it (backward)
            if al is not None:
                xn = _align_reverse(xn, al, T, Bp, Hp, right=False)
                if (dropout > 0.0 and l + 1 < L) or (l + 1 == L and fc_w is None):
                    y = _align_reverse(y, al, T, Bp, Hp, right=False)
            if dropout > 0.0 and l + 1 < L:
                # inter-layer dropout of nn.GRU(dropout=p): applied to every layer output but the
                # last; drawn over the H real units, so padding does not change the masks
                mask = (torch.rand(M, ndir * H, device=dev) >= dropout).float() * \
                    (1.0 / (1.0 - dropout))
                mask = pad_blocks(mask, 1, ndir, H, Hp)
                # the next layer's operand stays bf16 (bf16 * f32 would promote to f32): mask the
                # fp32 state and round once
                xn = (y * mask).to(torch.bfloat16)
            if need_grad:
                saved.append((X, y_rec, gates, mask, wih_cat, whh, hb))
            X = xn
        ctx.la = None
        if la_w is not None:
            # r over the top layer's fp32 states as the recurrence wrote them; frames >= len_b
            # of each utterance are never read
            tau = la_w.shape[2] - 1
            taps = lookahead_taps(la_w, H, Hp)
            r = None if fc_w is not None else torch.empty(M, Hp, dtype=torch.float32, device=dev)
            rb = torch.empty(M, Hp, dtype=torch.bfloat16, device=dev) if fc_w is not None else None
            lookahead_fwd(y_rec, taps, la_lens, r, rb, T, Bp, Hp, tau)
            if need_grad:
                ctx.la = (la_w, taps, la_lens, y_rec, tau)
            if fc_w is not None:
                X = rb
            else:
                y = r
        ctx.saved = saved
        ctx.announce = _announce
        ctx.weights = weights
        ctx.dims = (B, T, In, Bp, H, Hp, ndir, L)
        ctx.lens = (al, valid)
        ctx.fc = None
        if fc_w is not None:
            V = fc_w.shape[0]
            wcat = fc_operand(fc_w, ndir, H, Hp)
            out = gemm_bf16_tn(X, wcat, bias=fc_b.detach().float().contiguous(),
                               remap=(Bp, T, B)).view(B, T, V)
            ctx.fc = (fc_w, X)
            return out
        out = unpad_blocks(y.view(T, Bp, D)[:, :B], 2, ndir, H, Hp).transpose(0, 1).contiguous()
        if valid is not None:
            out.mul_(valid)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = _lib.load()
        B, T, In, Bp, H, Hp, ndir, L = ctx.dims
        weights = ctx.weights
        if _grad_ready_hook is not None and ctx.announce and _grad_guard is not None:
            _grad_guard(list(weights))
        dev = dout.device
        M = T * Bp
        D = ndir * Hp
        K3 = 3 * Hp
        padded = Hp != H
        al, valid = ctx.lens
        if valid is not None:
            dout = dout * valid
        dfc_w = dfc_b = None
        if ctx.fc is not None:
            fc_w, Xtop = ctx.fc
            V = fc_w.shape[0]
            Vp = _round_up(V, 8)
            dl = torch.zeros(T, Bp, Vp, dtype=torch.bfloat16, device=dev)
            dl[:, :B, :V] = dout.transpose(0, 1)
            dl = dl.view(M, Vp)
            w = fc_w.detach().to(torch.bfloat16)
            wT = torch.zeros(D, Vp, dtype=torch.bfloat16, device=dev)      # [D][Vp] = [W | W]^T
            for d in range(ndir):
                wT[d * Hp:d * Hp + H, :V] = w.t()
            dY = gemm_bf16_tn(dl, wT)                                         # [M][D] f32
            dw2 = torch.zeros(Vp, D, dtype=torch.float32, device=dev)
            # dW (Vp x D) = dl^T Xtop, both operands read token-major (MN-major UMMA)
            gemm_bf16_tn(dl, Xtop, out=dw2, accumulate=True, a_mn=True, b_mn=True)
            dfc_w = dw2[:V, :H] if ndir == 1 else dw2[:V, :H] + dw2[:V, Hp:Hp + H]
            dfc_b = dout.sum((0, 1))
        elif B == Bp and not padded:
            # (dout may be an expanded stride-0 tensor, e.g. from y.sum(): force a real copy)
            dY = dout.transpose(0, 1).float().contiguous().view(M, D)
        else:
            dY = torch.zeros(T, Bp, D, dtype=torch.float32, device=dev)
            dY[:, :B] = pad_blocks(dout.transpose(0, 1), 2, ndir, H, Hp)
            dY = dY.view(M, D)
        dla = None
        if ctx.la is not None:
            la_w, taps, la_lens, h_top, tau = ctx.la
            dY, dla = lookahead_bwd(dY.contiguous(), h_top, taps, la_lens, T, Bp, Hp, tau)
            dla = dla[:, :H].t().reshape(la_w.shape)
            ctx.la = None
        nbytes = _lib.workspace_size(lib.sb_gru_bwd_workspace_size, Bp, Hp, ndir)
        ws = _workspace(nbytes, dev)
        grads = [None] * len(weights)
        for l in reversed(range(L)):
            X, y, gates, mask, wih_cat, whh, hb = ctx.saved[l]
            if mask is not None:
                dY = dY * mask
            if al is not None:
                dY = _align_reverse(dY, al, T, Bp, Hp, right=True)
            wl = weights[l * 4 * ndir:(l + 1) * 4 * ndir]
            Kl = X.shape[1]
            In_l = wl[0].shape[1] if l == 0 else D     # input columns at the kernels' width
            dgi = torch.empty(M, ndir * K3, dtype=torch.bfloat16, device=dev)
            dghn = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
            dbih = torch.zeros(ndir * K3, dtype=torch.float32, device=dev)
            dbhh = torch.zeros(ndir * K3, dtype=torch.float32, device=dev)
            sp = _lib.stream_ptr()
            _launch("gru_bwd", 2.0 * M * 3 * Hp * Hp * ndir,
                    lambda dY=dY: lib.sb_gru_bwd(dY.data_ptr(), y.data_ptr(), gates.data_ptr(),
                                                 whh.data_ptr(), dgi.data_ptr(), dghn.data_ptr(),
                                                 dbih.data_ptr(), dbhh.data_ptr(), ws.data_ptr(),
                                                 nbytes, T, Bp, Hp, ndir, sp))
            base = l * 4 * ndir
            # dW_hh pairs dgi with the states in the recurrence's coordinates; dW_ih and dX pair
            # it with the layer input, where the reverse half is left-aligned
            dgi_x = dgi if al is None else _align_reverse(dgi, al, T, Bp, K3, right=False)
            # ---- weight gradients: contract the token-major operands over their rows ----
            Ms = M - Bp                      # tokens that have a predecessor in the recurrence
            # When the .grad of both directions' W_ih lie back to back (optim.FlatSGD's flat
            # gradient buffer), dW_ih of both is one [2*3H][In_l] GEMM into that block: one
            # wave-filling launch instead of two.
            both = None
            if ndir == 2 and not padded and al is None:
                s0, s1 = _grad_sink(wl[0]), _grad_sink(wl[4])
                if (s0 is not None and s1 is not None and s0.shape == (K3, In_l)
                        and s1.shape == s0.shape
                        and s1.untyped_storage().data_ptr() == s0.untyped_storage().data_ptr()
                        and s1.data_ptr() == s0.data_ptr() + s0.numel() * s0.element_size()):
                    both = s0.as_strided((2 * K3, In_l), (In_l, 1))
                    gemm_bf16_tn(dgi_x, X[:, :In_l], out=both, accumulate=True,
                                 a_mn=True, b_mn=True)
            for d in range(ndir):
                # dW_ih[d] (3H x In_l) = dgi[:, d]^T X.  A padded layer computes the padded
                # gradients into temporaries and hands on (or adds into the sink) the real block.
                sink = None if padded else _grad_sink(wl[d * 4])
                dwih = sink if sink is not None else \
                    torch.zeros(K3, In_l, dtype=torch.float32, device=dev)
                if both is None:
                    gemm_bf16_tn(dgi_x[:, d * K3:(d + 1) * K3], X[:, :In_l], out=dwih,
                                 accumulate=True, a_mn=True, b_mn=True)
                # dW_hh[d] = [dgi_r | dgi_z | dghn]^T h_prev: h_prev of token (t, b) is token
                # (t-1, b) in the forward direction and (t+1, b) in the reverse one, so the
                # shift is a row offset of Bp on one of the two operands
                sink_hh = None if padded else _grad_sink(wl[d * 4 + 1])
                dwhh = sink_hh if sink_hh is not None else \
                    torch.zeros(K3, Hp, dtype=torch.float32, device=dev)
                if Ms > 0:
                    ga, hp = (slice(Bp, M), slice(0, Ms)) if d == 0 else \
                        (slice(0, Ms), slice(Bp, M))
                    gemm_bf16_tn(dgi[ga, d * K3:d * K3 + 2 * Hp], hb[hp, d * Hp:(d + 1) * Hp],
                                 out=dwhh[:2 * Hp], accumulate=True, a_mn=True, b_mn=True)
                    gemm_bf16_tn(dghn[ga, d * Hp:(d + 1) * Hp], hb[hp, d * Hp:(d + 1) * Hp],
                                 out=dwhh[2 * Hp:], accumulate=True, a_mn=True, b_mn=True)
                dbi, dbh = dbih[d * K3:(d + 1) * K3], dbhh[d * K3:(d + 1) * K3]
                if padded:
                    dwih = unpad_blocks(dwih, 0, 3, H, Hp)
                    if l > 0:
                        dwih = unpad_blocks(dwih, 1, ndir, H, Hp)
                    dwhh = unpad_blocks(unpad_blocks(dwhh, 0, 3, H, Hp), 1, 1, H, Hp)
                    dbi, dbh = unpad_blocks(dbi, 0, 3, H, Hp), unpad_blocks(dbh, 0, 3, H, Hp)
                    sink, sink_hh = _grad_sink(wl[d * 4]), _grad_sink(wl[d * 4 + 1])
                    for s, g in ((sink, dwih), (sink_hh, dwhh)):
                        if s is not None:
                            s.add_(g)
                grads[base + d * 4 + 0] = None if sink is not None else dwih
                grads[base + d * 4 + 1] = None if sink_hh is not None else dwhh
                grads[base + d * 4 + 2] = dbi
                grads[base + d * 4 + 3] = dbh
            if _grad_ready_hook is not None and ctx.announce:
                base = l * 4 * ndir
                if all(grads[base + d * 4 + k] is None for d in range(ndir) for k in (0, 1)):
                    # weights already sit in .grad; add the biases there too, then announce
                    ok = True
                    for d in range(ndir):
                        for k in (2, 3):
                            sink = _bias_sink(wl[d * 4 + k])
                            if sink is None:
                                ok = False
                                continue
                            sink.add_(grads[base + d * 4 + k])
                            grads[base + d * 4 + k] = None
                    if ok:
                        _grad_ready_hook(list(wl))
            # ---- gradient w.r.t. the layer input ----
            if l > 0 or ctx.needs_input_grad[0]:
                # dX = dgi W_ih: W_ih (3H x In) is the [K][N] form of the B operand
                dY = gemm_bf16_tn(dgi_x, wih_cat, b_mn=True)              # [M][Kl] f32
        dx = None
        if ctx.needs_input_grad[0]:
            dx = dY.view(T, Bp, -1)[:, :B, :In].transpose(0, 1).contiguous()
        ctx.saved = None
        return (dx, None, None, None, dfc_w, dfc_b, None, dla) + tuple(grads)


def lookahead_taps(la_w, H, Hp):
    """(H, 1, tau + 1) lookahead weight -> the kernels' [tau + 1][Hp] f32 taps (padded units 0)"""
    taps = la_w.detach().float().reshape(H, -1).t()
    return pad_blocks(taps, 1, 1, H, Hp).contiguous()


def lookahead_fwd(h, taps, lens_dev, r, rb, T, Bp, Hp, tau):
    """sb_lookahead_fwd of the time-major [T*Bp][Hp] f32 h into r (f32) and / or rb (bf16)"""
    lib = _lib.load()
    sp = _lib.stream_ptr()
    _launch("lookahead_fwd", 2.0 * T * Bp * Hp * (tau + 1),
            lambda: lib.sb_lookahead_fwd(h.data_ptr(), taps.data_ptr(), _lib.ptr(lens_dev),
                                         _lib.ptr(r), _lib.ptr(rb), T, Bp, Hp, tau, sp))


def lookahead_bwd(dr, h, taps, lens_dev, T, Bp, Hp, tau):
    """sb_lookahead_bwd: -> (dh [T*Bp][Hp] f32, dW [tau + 1][Hp] f32)"""
    lib = _lib.load()
    dev = dr.device
    dh = torch.empty(T * Bp, Hp, dtype=torch.float32, device=dev)
    dw = torch.empty(tau + 1, Hp, dtype=torch.float32, device=dev)
    nbytes = _lib.workspace_size(lib.sb_lookahead_bwd_workspace_size, T, Bp, Hp, tau)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    sp = _lib.stream_ptr()
    _launch("lookahead_bwd", 4.0 * T * Bp * Hp * (tau + 1),
            lambda: lib.sb_lookahead_bwd(dr.data_ptr(), h.data_ptr(), taps.data_ptr(),
                                         _lib.ptr(lens_dev), dh.data_ptr(), dw.data_ptr(),
                                         ws.data_ptr(), nbytes, T, Bp, Hp, tau, sp))
    return dh, dw


def _lookahead_weight(rnn, lookahead):
    if lookahead is None:
        return None
    if rnn.bidirectional:
        raise ValueError("a lookahead convolution needs a unidirectional GRU stack")
    return lookahead.weight


def _gru_weights(rnn):
    ndir = 2 if rnn.bidirectional else 1
    weights = []
    for l in range(rnn.num_layers):
        for d in range(ndir):
            sfx = "_l%d%s" % (l, "_reverse" if d == 1 else "")
            if not rnn.bias:
                raise _lib.SpeechB200Error("GRU without bias is not supported")
            weights += [getattr(rnn, "weight_ih" + sfx), getattr(rnn, "weight_hh" + sfx),
                        getattr(rnn, "bias_ih" + sfx), getattr(rnn, "bias_hh" + sfx)]
    return ndir, weights


GRU_MAX_BATCH = 128   # rows one recurrence launch keeps resident (gru.cu)


def _batch_chunks(x, lens, fn):
    """The recurrence is independent across utterances, so a minibatch larger than one launch
    holds is run as consecutive chunks of <= GRU_MAX_BATCH rows (exact, autograd sees a cat);
    `lens` (optional) is sliced with the batch."""
    global _announce
    if x.shape[0] <= GRU_MAX_BATCH:
        return fn(x, lens)
    _announce = False     # several backward passes add into the same .grad: none of them is final
    try:
        return torch.cat([fn(x[i:i + GRU_MAX_BATCH],
                             None if lens is None else lens[i:i + GRU_MAX_BATCH])
                          for i in range(0, x.shape[0], GRU_MAX_BATCH)], 0)
    finally:
        _announce = True


def gru_stack_logits(x, rnn, fc, dropout=0.0, lens=None, lookahead=None):
    """GRU stack + sum of direction halves + output projection `fc` (an nn.Linear), fused:
    returns logits (B, T, V) - the encoder tail of CTC.forward_impl (ctc_model.py:25-32).
    lens (optional): valid frames per utterance (GRUStackFunction); logits are exact at frames
    < lens[b].  lookahead (optional, unidirectional rnn): the model's lookahead nn.Conv1d, run
    between the top layer and fc."""
    ndir, weights = _gru_weights(rnn)
    la_w = _lookahead_weight(rnn, lookahead)
    return _batch_chunks(x, lens, lambda xc, lc: GRUStackFunction.apply(
        xc, ndir, rnn.hidden_size, float(dropout), fc.weight, fc.bias, lc, la_w, *weights))


def gru_stack(x, rnn, dropout=0.0, lens=None, lookahead=None):
    """Run the sm_90a GRU stack with the parameters of an nn.GRU module (batch_first, h0 = 0).
    lens (optional): valid frames per utterance, as nn.GRU over pack_padded_sequence followed by
    pad_packed_sequence (GRUStackFunction).  lookahead (optional, unidirectional rnn): an
    nn.Conv1d(H, H, tau + 1, groups=H, bias=False) over the top layer's output, zero-padded by
    tau frames on the right (by lens[b] frames' end in the exact-lengths mode)."""
    ndir, weights = _gru_weights(rnn)
    la_w = _lookahead_weight(rnn, lookahead)
    return _batch_chunks(x, lens, lambda xc, lc: GRUStackFunction.apply(
        xc, ndir, rnn.hidden_size, float(dropout), None, None, lc, la_w, *weights))


_direct_ok = {}


def conv_direct_ok(Fi, Ci, Co, kh, kw, s):
    """True when a conv layer past the first (input width Fi, Ci -> Co channels, kernel kh x kw,
    stride s; channel counts as the kernels run them, multiples of 8) runs on the direct
    convolution kernels: Co <= 32, and its resident weights and input footprint fit in shared
    memory.  Every other layer runs on im2col + GEMM."""
    key = (Fi, Ci, Co, kh, kw, s)
    if key not in _direct_ok:
        _direct_ok[key] = bool(_lib.load().sb_conv_direct_ok(*key))
    return _direct_ok[key]


class ConvStackFunction(torch.autograd.Function):
    """Conv2d+ReLU stack (csrc/conv.cu, csrc/gemm.cu): the first layer (one input channel) and any
    layer outside conv_direct_ok as im2col + wgmma GEMM, the others as direct convolutions that
    read their input activations straight from the previous layer's output (no patch matrix).

    forward(x (B,T,F) f32, specs ((kh,kw,s),...), w0, b0, w1, b1, ...) -> (B, T', C*F') f32 with
    the reference's channel-major feature order (model.py:66-71)."""

    @staticmethod
    def forward(ctx, x, specs, dropout, *params):
        """dropout > 0: nn.Dropout(p) after every ReLU (model.py:25-26) as a keep-byte mask
        (scaled by 1/(1-p)) in the activations' own layout, applied by the kernels that read them."""
        _lib.require_cuda(x, "x")
        lib = _lib.load()
        dev = x.device
        B, Ti, Fi = x.shape
        Ci = 1
        cur = x.detach().float().contiguous()
        saved = []
        masks = []
        mscale = 1.0 / (1.0 - dropout) if dropout > 0.0 else 1.0
        need_grad = any(ctx.needs_input_grad)
        sp = _lib.stream_ptr()
        _ensure_knobs()
        for l, (kh, kw, s_) in enumerate(specs):
            co_r, ci_r = params[2 * l].shape[:2]
            # zero filters up to the GEMM's multiple of 8 channels: a padded channel is
            # ReLU(0) = 0 everywhere, and the next layer's weights for it are zero
            Co = _round_up(co_r, 8)
            w = pad_blocks(pad_blocks(params[2 * l].detach(), 0, 1, co_r, Co), 1, 1, ci_r, Ci)
            b = pad_blocks(params[2 * l + 1].detach(), 0, 1, co_r, Co)
            K = kh * kw * Ci
            Kp = _round_up(K, 8)
            To, Fo = (Ti - kh) // s_ + 1, (Fi - kw) // s_ + 1
            M = B * To * Fo
            src = cur
            mprev = masks[l - 1] if l > 0 else None
            Wp = torch.zeros(Co, Kp, dtype=torch.bfloat16, device=dev)
            Wp[:, :K] = w.detach().permute(0, 2, 3, 1).reshape(Co, K)
            bias = b.detach().float().contiguous()
            if l > 0 and _conv_flags != 1 and conv_direct_ok(Fi, Ci, Co, kh, kw, s_):
                A = None          # the backward re-reads the activations themselves
                C = torch.empty(M, Co, dtype=torch.float32, device=dev)
                _launch("conv_fwd_direct", 2.0 * M * Co * K,
                        lambda: lib.sb_conv_fwd_direct(src.data_ptr(), _lib.ptr(mprev), mscale,
                                                       Wp.data_ptr(), Kp, bias.data_ptr(),
                                                       C.data_ptr(), B, Ti, Fi, Ci, Co, kh, kw,
                                                       s_, sp))
            else:
                A = torch.empty(M, Kp, dtype=torch.bfloat16, device=dev)
                _launch("conv_im2col", 0.0,
                        lambda: lib.sb_conv_im2col(src.data_ptr(), _lib.ptr(mprev), mscale,
                                                   A.data_ptr(), B, Ti, Fi, Ci, kh, kw, s_, Kp,
                                                   1 if l > 0 else 0, sp))
                C = gemm_bf16_tn(A, Wp, bias=bias)
            mask = None
            if dropout > 0.0:
                mask = (torch.rand(M, Co, device=dev) >= dropout).to(torch.uint8)
            masks.append(mask)
            if need_grad:
                saved.append((A, cur, C, Wp,
                              (Ti, Fi, Ci, kh, kw, s_, To, Fo, Co, K, Kp, co_r, ci_r)))
            cur, Ti, Fi, Ci = C, To, Fo, Co
        out = torch.empty(B, Ti, Ci * Fi, dtype=torch.float32, device=dev)
        _launch("conv_relu_to_bct", 0.0,
                lambda: lib.sb_conv_relu_to_bct(cur.data_ptr(), _lib.ptr(masks[-1]), mscale,
                                                out.data_ptr(),
                                                B, Ti, Fi, Ci, sp))
        ctx.saved = saved
        ctx.masks = masks
        ctx.mscale = mscale
        ctx.B = B
        ctx.nl = len(specs)
        # channel-major features: the real channels 0..co_r-1 are the leading co_r*F' columns
        ctx.pad_cols = (Ci - co_r) * Fi
        return out[:, :, :co_r * Fi] if ctx.pad_cols else out

    @staticmethod
    def backward(ctx, dY):
        lib = _lib.load()
        dev = dY.device
        B = ctx.B
        sp = _lib.stream_ptr()
        grads = [None] * (2 * ctx.nl)
        dY = dY.contiguous().float()
        if ctx.pad_cols:
            dY = torch.nn.functional.pad(dY, (0, ctx.pad_cols))
        dC = None
        for l in reversed(range(ctx.nl)):
            A, Pprev, C, Wp, (Ti, Fi, Ci, kh, kw, s_, To, Fo, Co, K, Kp, co_r, ci_r) = ctx.saved[l]
            M = B * To * Fo
            if dC is None:
                dC = torch.empty(M, Co, dtype=torch.bfloat16, device=dev)
                db = torch.zeros(Co, dtype=torch.float32, device=dev)
                dCl = dC
                _launch("conv_dtop", 0.0,
                        lambda: lib.sb_conv_dtop(dY.data_ptr(), C.data_ptr(),
                                                 _lib.ptr(ctx.masks[l]), ctx.mscale,
                                                 dCl.data_ptr(),
                                                 db.data_ptr(), B, To, Fo, Co, sp))
            grads[2 * l + 1] = db[:co_r]
            # weight gradient: contraction over the M = B*To*Fo patch rows (split-K over all SMs)
            # dWp^T [Kp][Co] = A^T dC with both operands read token-major (MN-major UMMA)
            dWpT = torch.zeros(Kp, Co, dtype=torch.float32, device=dev)
            mprev = ctx.masks[l - 1] if l > 0 else None
            if A is None:
                dCw = dC
                _launch("conv_wgrad_direct", 2.0 * M * Co * K,
                        lambda: lib.sb_conv_wgrad_direct(Pprev.data_ptr(), _lib.ptr(mprev),
                                                         ctx.mscale, dCw.data_ptr(),
                                                         dWpT.data_ptr(), B, Ti, Fi, Ci, Co, kh,
                                                         kw, s_, sp))
            else:
                gemm_bf16_tn(A, dC, out=dWpT, accumulate=True, a_mn=True, b_mn=True)
            dWp = dWpT.t()
            grads[2 * l] = dWp[:co_r, :K].reshape(co_r, kh, kw, Ci).permute(0, 3, 1, 2)[:, :ci_r] \
                .contiguous()
            if l > 0 and A is None:
                Mp = B * Ti * Fi
                dCp = torch.empty(Mp, Ci, dtype=torch.bfloat16, device=dev)
                db = torch.zeros(Ci, dtype=torch.float32, device=dev)
                dCd = dC
                _launch("conv_dgrad_direct", 2.0 * M * Co * K,
                        lambda: lib.sb_conv_dgrad_direct(dCd.data_ptr(), Wp.data_ptr(), Kp,
                                                         Pprev.data_ptr(), _lib.ptr(mprev),
                                                         ctx.mscale, dCp.data_ptr(),
                                                         db.data_ptr(), B, Ti, Fi, Ci, Co, kh,
                                                         kw, s_, sp))
                dC = dCp
            elif l > 0:
                dA = gemm_bf16_tn(dC, Wp, b_mn=True)            # [M][Kp] f32 patch gradient
                Mp = B * Ti * Fi
                dCp = torch.empty(Mp, Ci, dtype=torch.bfloat16, device=dev)
                db = torch.zeros(Ci, dtype=torch.float32, device=dev)
                _launch("conv_col2im_relu", 0.0,
                        lambda: lib.sb_conv_col2im_relu(dA.data_ptr(), dA.stride(0),
                                                        Pprev.data_ptr(),
                                                        _lib.ptr(ctx.masks[l - 1]), ctx.mscale,
                                                        dCp.data_ptr(),
                                                        db.data_ptr(), B, Ti, Fi, Ci, kh, kw, s_,
                                                        sp))
                dC = dCp
        ctx.saved = None
        ctx.masks = None
        return (None, None, None) + tuple(grads)


def conv_stack(x, conv, training):
    """Conv2d+ReLU(+Dropout) front-end of the encoder (reference model.py:19-29,60-71).

    x (B, T, F) -> (B, T', C*F') with the reference's channel-major feature flattening
    (transpose(1,2) of (B,C,T',F') then view, model.py:66-71).  Runs on our im2col + wgmma
    kernels and, for the layers conv_direct_ok takes, on the direct-convolution kernels,
    including the Dropout after each ReLU when training, for every stack the reference
    can express (model.py:21-23: square stride, no padding, dilation or groups, bias, one dropout
    rate); any other stack raises, there is no library fallback.  Any out_channels runs: a layer
    whose count is not a multiple of 8 gets zero filters up to the next multiple (exact: such a
    channel is 0 after the ReLU, and the next layer's weights for it are zero), its dropout mask
    covers the padded channels too, and the real features are the leading C*F' columns.
    """
    mods = list(conv.children())
    convs = [m for m in mods if isinstance(m, torch.nn.Conv2d)]
    ps = [m.p for m in mods if isinstance(m, torch.nn.Dropout)]
    p_drop = (ps[0] if ps else 0.0) if training else 0.0
    drop = len(set(ps)) > 1
    simple = all(c.stride[0] == c.stride[1] and c.padding == (0, 0) and c.dilation == (1, 1)
                 and c.groups == 1 and c.bias is not None for c in convs)
    if not (convs and simple and not drop):
        raise _lib.SpeechB200Error(
            "conv_stack: unsupported convolution stack (needs square stride, no padding / "
            "dilation / groups, bias, one dropout rate); this package has no cuDNN fallback")
    specs = tuple((c.kernel_size[0], c.kernel_size[1], c.stride[0]) for c in convs)
    params = []
    for c in convs:
        params += [c.weight, c.bias]
    return ConvStackFunction.apply(x, specs, float(p_drop), *params)
