"""Attention-decoder operators over the C ABI (csrc/s2s.cu): the per-token step of
Seq2Seq.decode / decode_step / infer / beam_search (speech/models/seq2seq.py:78-227) and
NNAttention.forward (:344-360) as two kernels per token (GRU cell; attention + output projection),
with a hand-written backward (three kernels per token, the output-projection backward of all
steps in one launch, the weight gradients time-batched on the wgmma GEMM), a greedy loop and a
beam search that never leave the device: the host only enqueues kernels and reads the final
hypothesis back once.
"""
import ctypes

import torch

from .. import _lib


def _f(t):
    return t.detach().float().contiguous()


class DecoderWeights:
    """fp32 contiguous views of the decoder parameters, in the layout the kernels take."""

    def __init__(self, m):
        self.emb = _f(m.embedding.weight)
        self.w_ih, self.w_hh = _f(m.dec_rnn.weight_ih), _f(m.dec_rnn.weight_hh)
        self.b_ih, self.b_hh = _f(m.dec_rnn.bias_ih), _f(m.dec_rnn.bias_hh)
        conv, lin = m.attend.conv, m.attend.nn[1].fc
        self.conv_wT = _f(conv.weight).reshape(conv.weight.shape[0], -1).t().contiguous()  # (Kc, H)
        self.conv_b = _f(conv.bias)
        self.lin_w = _f(lin.weight).reshape(-1)
        self.lin_b = float(lin.bias.detach().float().item()) if lin.bias is not None else 0.0
        self.fc_w, self.fc_b = _f(m.fc.fc.weight), _f(m.fc.fc.bias)
        self.log_t = 1 if m.attend.log_t else 0
        self.H = self.w_hh.shape[1]
        self.Kc = self.conv_wT.shape[0]
        self.C = self.fc_w.shape[0]
        if self.emb.shape[1] != self.H:
            raise _lib.SpeechB200Error("Seq2Seq: embedding_dim must equal the encoder dim (ix + sx)")
        # device addresses, looked up once: the per-token loops only do integer arithmetic
        for n in ("emb", "w_ih", "w_hh", "b_ih", "b_hh", "conv_wT", "conv_b", "lin_w", "fc_w",
                  "fc_b"):
            setattr(self, "p_" + n, getattr(self, n).data_ptr())


def attn_workspace(lib, B, T, H, dev):
    """zeroed scratch of the attention kernels (per-CTA softmax partials + ticket counters); one
    buffer serves every step of a decode on the same stream"""
    n = ctypes.c_size_t(0)
    _lib.check(lib.sb_s2s_workspace_size(B, T, H, ctypes.byref(n)), "s2s workspace")
    return torch.zeros(n.value, dtype=torch.uint8, device=dev)


def _a(x):
    """device address of a tensor; ints (addresses computed by the caller) and None pass through"""
    return x if x is None or isinstance(x, int) else x.data_ptr()


def _cell_fwd(lib, w, tok, tok_stride, sx_prev, hx_prev, hx, ix_save, gates_save, done, B, sp):
    from .. import ops
    ops._launch("s2s_cell_fwd", 0.0,
                lambda: lib.sb_s2s_cell_fwd(w.p_emb, tok, tok_stride, _a(sx_prev), _a(hx_prev),
                                            w.p_w_ih, w.p_w_hh, w.p_b_ih, w.p_b_hh, _a(hx),
                                            _a(ix_save), _a(gates_save), done, B, w.H, sp))


def _attn_fwd(lib, w, ws, eh, bcast, hx, ax_prev, sx, ax, B, T, sp, logits=None, logit_stride=0,
              logp=None, argmax=None, history=None, hist_stride=0, hist_col=0, end_count=None,
              end_tok=-1, done=None, with_fc=True):
    from .. import ops
    ops._launch("s2s_attn_fwd", 0.0,
                lambda: lib.sb_s2s_attn_fwd(_a(eh), bcast, _a(hx), _a(ax_prev), w.p_conv_wT,
                                            w.p_conv_b, w.p_lin_w, w.lin_b, w.log_t, B, T, w.H,
                                            w.Kc, _a(sx), _a(ax),
                                            w.p_fc_w if with_fc else None,
                                            w.p_fc_b if with_fc else None, w.C,
                                            logits, logit_stride, _a(logp), _a(argmax),
                                            history, hist_stride, hist_col, end_count, end_tok,
                                            done, _a(ws), ws.numel(), sp))


class DecodeFunction(torch.autograd.Function):
    """Teacher-forced decode (seq2seq.py:78-112): eh (B,T,H), tokens (B,U) -> logits (B,U-1,C),
    alignments (B,U-1,T).  sample_flags[u] (host bools, drawn by the caller from Python's `random`
    exactly as the reference does, :94): feed the arg-max of the previous step instead of the
    label."""

    @staticmethod
    def forward(ctx, eh, tokens, sample_flags, w, emb_w, w_ih, w_hh, b_ih, b_hh, conv_w, conv_b,
                lin_w, lin_b, fc_w, fc_b):
        _lib.require_cuda(eh, "encoder states")
        lib = _lib.load()
        ehc = _f(eh)
        B, T, H = ehc.shape
        U = tokens.shape[1]
        steps = U - 1
        dev = ehc.device
        tok = tokens.detach().to(dev, torch.int32).contiguous()
        need = any(ctx.needs_input_grad)
        hx_all = torch.zeros(steps + 1, B, H, dtype=torch.float32, device=dev)
        sx_all = torch.empty(steps, B, H, dtype=torch.float32, device=dev)
        ax_all = torch.empty(steps, B, T, dtype=torch.float32, device=dev)
        ix_all = torch.empty(steps, B, H, dtype=torch.float32, device=dev) if need else None
        gates_all = torch.empty(steps, B, 4, H, dtype=torch.float32, device=dev) if need else None
        logits = torch.empty(B, steps, w.C, dtype=torch.float32, device=dev)
        sampling = any(sample_flags[1:steps]) if steps > 1 else False
        amax = torch.zeros(B, dtype=torch.int32, device=dev) if sampling else None
        used = tok[:, :steps].t().contiguous() if need else None          # (steps, B) tokens fed
        sp = _lib.stream_ptr()
        ws = attn_workspace(lib, B, T, H, dev)
        # per-token launches: addresses by integer arithmetic (no tensor slicing in the loop)
        BH, BT = 4 * B * H, 4 * B * T
        p_hx, p_sx, p_ax = hx_all.data_ptr(), sx_all.data_ptr(), ax_all.data_ptr()
        p_ix = ix_all.data_ptr() if need else None
        p_gt = gates_all.data_ptr() if need else None
        p_tok, p_logits = tok.data_ptr(), logits.data_ptr()
        p_amax = amax.data_ptr() if sampling else None
        for u in range(steps):
            if u > 0 and sample_flags[u]:
                if need:
                    used[u].copy_(amax)
                tk, ts = p_amax, 1
            else:
                tk, ts = p_tok + 4 * u, U
            _cell_fwd(lib, w, tk, ts, p_sx + (u - 1) * BH if u > 0 else None, p_hx + u * BH,
                      p_hx + (u + 1) * BH, p_ix + u * BH if need else None,
                      p_gt + 4 * u * BH if need else None, None, B, sp)
            _attn_fwd(lib, w, ws, ehc, 0, p_hx + (u + 1) * BH, p_ax + (u - 1) * BT if u > 0 else None,
                      p_sx + u * BH, p_ax + u * BT, B, T, sp, logits=p_logits + 4 * u * w.C,
                      logit_stride=steps * w.C, argmax=p_amax)
        ctx.w = w
        ctx.saved = (ehc, hx_all, sx_all, ax_all, ix_all, gates_all, used)
        ctx.dims = (B, T, H, steps)
        ctx.vocab = emb_w.shape[0]
        ctx.conv_shape = conv_w.shape
        ctx.lin_shape = lin_w.shape
        ctx.has_lin_b = lin_b is not None
        return logits, ax_all.permute(1, 0, 2)

    @staticmethod
    def backward(ctx, dlogits, daligns):
        from .. import ops
        lib = _lib.load()
        w = ctx.w
        ehc, hx_all, sx_all, ax_all, ix_all, gates_all, used = ctx.saved
        B, T, H, steps = ctx.dims
        C, Kc = w.C, w.Kc
        dev = ehc.device
        dl = dlogits.detach().float().permute(1, 0, 2).contiguous()        # (steps, B, C)
        da_ext = None
        if daligns is not None and bool((daligns != 0).any()):
            da_ext = daligns.detach().float().permute(1, 0, 2).contiguous()   # (steps, B, T)
        d_eh = torch.zeros(B, T, H, dtype=torch.float32, device=dev)
        d_gi = torch.empty(steps, B, 3 * H, dtype=torch.float32, device=dev)
        d_gh = torch.empty(steps, B, 3 * H, dtype=torch.float32, device=dev)
        d_ix = torch.empty(steps, B, H, dtype=torch.float32, device=dev)
        o_all = torch.empty(steps, B, H, dtype=torch.float32, device=dev)
        d_hx_direct = torch.empty(B, H, dtype=torch.float32, device=dev)
        d_hx_prev = torch.empty(B, H, dtype=torch.float32, device=dev)
        d_o = torch.empty(steps, B, H, dtype=torch.float32, device=dev)
        d_ax = [torch.zeros(B, T, dtype=torch.float32, device=dev) for _ in range(2)]
        TS = (T + 23) // 24                                  # CTAs per utterance (csrc/s2s.cu)
        g_conv_wT = torch.zeros(B, TS, Kc, H, dtype=torch.float32, device=dev)
        g_conv_b = torch.zeros(B, H, dtype=torch.float32, device=dev)
        g_lin_w = torch.zeros(B, H, dtype=torch.float32, device=dev)
        g_lin_b = torch.zeros(B, dtype=torch.float32, device=dev)
        sp = _lib.stream_ptr()
        ws = attn_workspace(lib, B, T, H, dev)
        w_ihT, w_hhT = w.w_ih.t().contiguous(), w.w_hh.t().contiguous()
        ops._launch("s2s_dout", 0.0, lambda: lib.sb_s2s_dout(
            dl.data_ptr(), w.fc_w.data_ptr(), hx_all[1:].data_ptr(), sx_all.data_ptr(),
            d_o.data_ptr(), o_all.data_ptr(), steps * B, C, H, sp))
        BH, BT = 4 * B * H, 4 * B * T
        p_eh, p_hx, p_ax = ehc.data_ptr(), hx_all.data_ptr(), ax_all.data_ptr()
        p_gt, p_do, p_dix = gates_all.data_ptr(), d_o.data_ptr(), d_ix.data_ptr()
        p_dgi, p_dgh = d_gi.data_ptr(), d_gh.data_ptr()
        p_dax = (d_ax[0].data_ptr(), d_ax[1].data_ptr())
        p_dhd, p_dhp, p_deh = d_hx_direct.data_ptr(), d_hx_prev.data_ptr(), d_eh.data_ptr()
        p_gcw, p_gcb = g_conv_wT.data_ptr(), g_conv_b.data_ptr()
        p_glw, p_glb = g_lin_w.data_ptr(), g_lin_b.data_ptr()
        p_wihT, p_whhT, p_ws, n_ws = w_ihT.data_ptr(), w_hhT.data_ptr(), ws.data_ptr(), ws.numel()
        for u in reversed(range(steps)):
            last = (u == steps - 1)
            d_ax_next = None if last else p_dax[(u + 1) & 1]
            if da_ext is not None:
                if last:
                    d_ax_next = da_ext[u].data_ptr()
                else:
                    d_ax[(u + 1) & 1].add_(da_ext[u])
            ops._launch("s2s_attn_bwd", 0.0, lambda: lib.sb_s2s_attn_bwd(
                p_eh, p_hx + (u + 1) * BH, p_hx + u * BH, p_ax + (u - 1) * BT if u > 0 else None,
                p_ax + u * BT, w.p_conv_wT, w.p_conv_b, w.p_lin_w, p_do + u * BH,
                None if last else p_dix + (u + 1) * BH, d_ax_next, None if last else p_dhp,
                p_gt + 4 * u * BH, p_deh, p_dax[u & 1], p_dgi + 3 * u * BH, p_dgh + 3 * u * BH,
                p_dhd, p_gcw, p_gcb, p_glw, p_glb, w.log_t, B, T, H, Kc, p_ws, n_ws, sp))
            ops._launch("s2s_cell_bwd", 0.0, lambda: lib.sb_s2s_cell_bwd(
                p_dgi + 3 * u * BH, p_dgh + 3 * u * BH, p_dhd, p_wihT, p_whhT, p_dix + u * BH,
                p_dhp, B, H, sp))
        # ---- time-batched weight gradients: contractions over all (u, b) rows on the wgmma GEMM
        R = steps * B

        def wgrad(dy, x):          # dy (R, O) f32, x (R, K) f32 -> dy^T x  (O, K) f32
            O, K = dy.shape[1], x.shape[1]
            Op, Kp = (O + 7) // 8 * 8, (K + 7) // 8 * 8
            a = torch.zeros(R, Op, dtype=torch.bfloat16, device=dev)
            a[:, :O] = dy
            b = torch.zeros(R, Kp, dtype=torch.bfloat16, device=dev)
            b[:, :K] = x
            out = torch.zeros(Op, Kp, dtype=torch.float32, device=dev)
            ops.gemm_bf16_tn(a, b, out=out, accumulate=True, a_mn=True, b_mn=True)
            return out[:O, :K]

        d_w_ih = wgrad(d_gi.view(R, 3 * H), ix_all.view(R, H))
        d_w_hh = wgrad(d_gh.view(R, 3 * H), hx_all[:steps].reshape(R, H))
        d_fc_w = wgrad(dl.view(R, C), o_all.view(R, H))
        d_b_ih = d_gi.sum((0, 1))
        d_b_hh = d_gh.sum((0, 1))
        d_fc_b = dl.sum((0, 1))
        d_emb = torch.zeros(ctx.vocab, H, dtype=torch.float32, device=dev)
        d_emb.index_add_(0, used.reshape(-1).long(), d_ix.view(R, H))
        d_conv_w = g_conv_wT.sum((0, 1)).t().reshape(ctx.conv_shape)
        d_conv_b = g_conv_b.sum(0)
        d_lin_w = g_lin_w.sum(0).reshape(ctx.lin_shape)
        d_lin_b = g_lin_b.sum().reshape(1) if ctx.has_lin_b else None
        return (d_eh, None, None, None, d_emb, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_conv_w, d_conv_b,
                d_lin_w, d_lin_b, d_fc_w, d_fc_b)


def decode(m, eh, tokens, sample_flags):
    """logits (B, U-1, C), alignments (B, U-1, T) with autograd through the kernels above."""
    w = DecoderWeights(m)
    lin = m.attend.nn[1].fc
    return DecodeFunction.apply(eh, tokens, sample_flags, w, m.embedding.weight,
                                m.dec_rnn.weight_ih, m.dec_rnn.weight_hh, m.dec_rnn.bias_ih,
                                m.dec_rnn.bias_hh, m.attend.conv.weight, m.attend.conv.bias,
                                lin.weight, lin.bias, m.fc.fc.weight, m.fc.fc.bias)


def decode_step(m, eh, y, state, softmax):
    """One step (seq2seq.py:114-137), no autograd: y (B,1) tokens -> (out (B,C), (hx, ax, sx))."""
    lib = _lib.load()
    w = DecoderWeights(m)
    ehc = _f(eh)
    B, T, H = ehc.shape
    dev = ehc.device
    if state is None:
        hx_prev = torch.zeros(B, H, dtype=torch.float32, device=dev)
        ax_prev = sx_prev = None
    else:
        hx_prev, ax_prev, sx_prev = state
        hx_prev = _f(hx_prev)
        ax_prev = _f(ax_prev)
        sx_prev = _f(sx_prev).reshape(B, H)
    tok = y.detach().to(dev, torch.int32).reshape(B).contiguous()
    hx = torch.empty(B, H, dtype=torch.float32, device=dev)
    sx = torch.empty(B, H, dtype=torch.float32, device=dev)
    ax = torch.empty(B, T, dtype=torch.float32, device=dev)
    out = torch.empty(B, w.C, dtype=torch.float32, device=dev)
    logp = torch.empty(B, w.C, dtype=torch.float32, device=dev) if softmax else None
    sp = _lib.stream_ptr()
    ws = attn_workspace(lib, B, T, H, dev)
    _cell_fwd(lib, w, tok.data_ptr(), 1, sx_prev, hx_prev, hx, None, None, None, B, sp)
    _attn_fwd(lib, w, ws, ehc, 0, hx, ax_prev, sx, ax, B, T, sp, logits=out.data_ptr(),
              logit_stride=w.C, logp=logp)
    return (logp if softmax else out), (hx, ax, sx.unsqueeze(1))


def greedy(m, eh, start, end_tok, max_len):
    """Greedy decode (seq2seq.py:145-178) without leaving the device: every kernel of every step
    is enqueued up front, kernels after the stop condition (all rows emitted end_tok in the same
    step, :155-156) are no-ops, ONE device->host copy returns the tokens.  -> (B, steps+1) list."""
    lib = _lib.load()
    w = DecoderWeights(m)
    ehc = _f(eh)
    B, T, H = ehc.shape
    dev = ehc.device
    hist = torch.zeros(B, max_len + 1, dtype=torch.int32, device=dev)
    hist[:, 0] = start.to(dev, torch.int32).reshape(B)
    ctl = torch.zeros(max_len + 2, dtype=torch.int32, device=dev)    # end counts | done | nsteps
    done, nsteps = ctl[max_len:max_len + 1], ctl[max_len + 1:]
    hx = [torch.zeros(B, H, dtype=torch.float32, device=dev) for _ in range(2)]
    sx = [torch.empty(B, H, dtype=torch.float32, device=dev) for _ in range(2)]
    ax = [torch.empty(B, T, dtype=torch.float32, device=dev) for _ in range(2)]
    sp = _lib.stream_ptr()
    ws = attn_workspace(lib, B, T, H, dev)
    from .. import ops
    for e in range(max_len):
        cur, prv = e & 1, (e & 1) ^ 1
        _cell_fwd(lib, w, hist.data_ptr() + 4 * e, max_len + 1, sx[prv] if e > 0 else None,
                  hx[prv], hx[cur], None, None, done.data_ptr(), B, sp)
        _attn_fwd(lib, w, ws, ehc, 0, hx[cur], ax[prv] if e > 0 else None, sx[cur], ax[cur], B, T, sp,
                  history=hist.data_ptr(), hist_stride=max_len + 1, hist_col=e + 1,
                  end_count=ctl.data_ptr() + 4 * e, end_tok=int(end_tok), done=done.data_ptr())
        ops._launch("s2s_check_done", 0.0,
                    lambda: lib.sb_s2s_check_done(ctl.data_ptr() + 4 * e, B, done.data_ptr(),
                                                  nsteps.data_ptr(), e + 1, sp))
    n = int(nsteps.item())                      # the one synchronisation of the whole decode
    return hist[:, :n + 1].cpu().tolist()


def beam_search(m, eh, start_tok, end_tok, beam_size, max_len):
    """Seq2Seq.beam_search for one utterance (seq2seq.py:180-227), device-resident: the beam
    entries are the rows of the step kernels, expand/prune/complete/stop run in one bookkeeping
    kernel per step (csrc/s2s.cu), the hypothesis is back-tracked on the device."""
    from .. import ops
    lib = _lib.load()
    w = DecoderWeights(m)
    ehc = _f(eh)[:1].contiguous()
    _, T, H = ehc.shape
    K, C = int(beam_size), w.C
    dev = ehc.device
    nbytes = ctypes.c_size_t(0)
    _lib.check(lib.sb_s2s_beam_state_size(ctypes.byref(nbytes)), "beam state")
    state = torch.zeros(nbytes.value + 64, dtype=torch.uint8, device=dev)
    node_cap = 2 * K * (max_len + 1) + 2
    nodes = torch.zeros(node_cap, 2, dtype=torch.int32, device=dev)
    c_cap = K * (max_len + 1)
    c_scores = torch.zeros(c_cap, dtype=torch.float64, device=dev)
    parent = torch.zeros(K, dtype=torch.int32, device=dev)
    tok = torch.zeros(K, dtype=torch.int32, device=dev)
    out_tokens = torch.zeros(max_len + 2, dtype=torch.int32, device=dev)
    hx = [torch.zeros(K, H, dtype=torch.float32, device=dev) for _ in range(3)]
    sx = [torch.zeros(K, H, dtype=torch.float32, device=dev) for _ in range(3)]
    ax = [torch.zeros(K, T, dtype=torch.float32, device=dev) for _ in range(3)]
    logp = torch.empty(K, C, dtype=torch.float32, device=dev)
    sp = _lib.stream_ptr()
    ws = attn_workspace(lib, K, T, H, dev)
    _lib.check(lib.sb_s2s_beam_init(state.data_ptr(), nodes.data_ptr(), tok.data_ptr(),
                                    int(start_tok), sp), "beam init")
    # the `done` word of the state struct doubles as the no-op flag of the step kernels
    done_ptr = state.data_ptr() + _beam_done_offset()
    # buffers: [0] = state entering the step (gathered), [1] = state produced by the step
    for e in range(max_len):
        _cell_fwd(lib, w, tok.data_ptr(), 1, sx[0] if e > 0 else None, hx[0], hx[1], None, None,
                  done_ptr, K, sp)
        _attn_fwd(lib, w, ws, ehc, 1, hx[1], ax[0] if e > 0 else None, sx[1], ax[1], K, T, sp,
                  logp=logp, done=done_ptr)
        ops._launch("s2s_beam_select", 0.0, lambda: lib.sb_s2s_beam_select(
            logp.data_ptr(), state.data_ptr(), c_scores.data_ptr(), nodes.data_ptr(),
            parent.data_ptr(), tok.data_ptr(), out_tokens.data_ptr(), K, C, int(end_tok), e,
            max_len, node_cap, c_cap, sp))
        ops._launch("s2s_beam_gather", 0.0, lambda: lib.sb_s2s_beam_gather(
            hx[1].data_ptr(), sx[1].data_ptr(), ax[1].data_ptr(), hx[0].data_ptr(),
            sx[0].data_ptr(), ax[0].data_ptr(), parent.data_ptr(), state.data_ptr(), K, H, T, sp))
    n = int(state[_beam_outlen_offset():_beam_outlen_offset() + 4].view(torch.int32).item())
    return tuple(out_tokens[:n].cpu().tolist())


def _beam_done_offset():
    # struct BeamState { double score[32]; int node[32]; int token[32]; int nlive; int ncomplete;
    #                    double best_c_score; int best_c_node; int have_complete; int done; ... }
    return 32 * 8 + 32 * 4 + 32 * 4 + 4 + 4 + 8 + 4 + 4


def _beam_outlen_offset():
    return _beam_done_offset() + 4 + 4
