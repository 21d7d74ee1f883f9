"""Attention-decoder operators over the C ABI (csrc/s2s.cu): the per-token step of
Seq2Seq.decode / decode_step / infer / beam_search (speech/models/seq2seq.py:78-227) and
NNAttention.forward (:344-360) as two kernels per token (GRU cell; attention + output projection),
with a hand-written backward (three kernels per token, the output-projection backward of all
steps in one launch, the weight gradients time-batched on the wgmma GEMM), a greedy loop and a
beam search over a whole batch that never leave the device: the host only enqueues kernels and
reads the final hypotheses back once.
"""
import torch

from .. import _lib, ops
from ..lm import NGramLM, WordLM, fusion_args, fusion_kind
from ..models.ctc_decoder import StreamSearch


def _f(t):
    return t.detach().float().contiguous()


# Routes by shape.  The attention kernel runs the output projection in one CTA per utterance,
# which holds all C logits next to its 8 H-float tiles: C <= 7 H (sb_s2s_fc_fused).  Larger
# vocabularies project over many CTAs (sb_s2s_fc_rows, csrc/s2s_vocab.cu).  sb_s2s_dout holds one
# row of dlogits in shared memory (C <= 8192); past that d_o runs on the GEMM.  The single-CTA beam
# selection holds all K*C float64 candidates (<= 200 KB, sb_s2s_beam_select_fits); past that it
# runs split over many CTAs.
DOUT_MAX_CLASSES = 8192
# byte offsets of `done` and of the final hypothesis' length in the beam state (speech_b200.h); the
# hypothesis' float64 score is the state's last 8 bytes
BEAM_DONE_OFFSET = 0
BEAM_OUT_LEN_OFFSET = 4
BEAM_MAX_WIDTH = 32
# the beam search's per-step entry point by route and LM kind: (ops._launch name, symbol).  On the
# joint CTC/attention route it builds the candidates, and sb_s2s_ctc_select_batch selects.
_SELECT = {
    ("single", None): ("s2s_beam_select", "sb_s2s_beam_select_batch"),
    ("single", NGramLM): ("s2s_beam_select_lm", "sb_s2s_beam_select_lm_batch"),
    ("single", WordLM): ("s2s_beam_select_wordlm", "sb_s2s_beam_select_wordlm_batch"),
    ("split", None): ("s2s_beam_select_split", "sb_s2s_beam_select_split_batch"),
    ("split", NGramLM): ("s2s_beam_select_split_lm", "sb_s2s_beam_select_split_lm_batch"),
    ("split", WordLM): ("s2s_beam_select_split_wordlm", "sb_s2s_beam_select_split_wordlm_batch"),
    ("ctc", None): ("s2s_ctc_candidates", "sb_s2s_ctc_candidates"),
    ("ctc", NGramLM): ("s2s_ctc_candidates", "sb_s2s_ctc_candidates"),
    ("ctc", WordLM): ("s2s_ctc_candidates", "sb_s2s_ctc_candidates_wordlm"),
}


def fc_fused(H, C):
    """True where the attention kernel computes the logits itself (sb_s2s_fc_fused(H, C))."""
    return bool(_lib.load().sb_s2s_fc_fused(int(H), int(C)))


def dout_fits(C):
    """True where sb_s2s_dout runs the backward of the projection; else it runs on the GEMM."""
    return 0 < C <= DOUT_MAX_CLASSES


def beam_select_fits(K, C):
    """True where the single-CTA beam selection runs (sb_s2s_beam_select_fits(K, C))."""
    return bool(_lib.load().sb_s2s_beam_select_fits(int(K), int(C)))


class AttentionWeights:
    """fp32 contiguous views of NNAttention's parameters, in the layout the attention kernel takes,
    and their device addresses (looked up once: the per-token loops only do integer arithmetic)."""

    def __init__(self, attend):
        conv, lin = attend.conv, attend.nn[1].fc
        self.conv_wT = _f(conv.weight).reshape(conv.weight.shape[0], -1).t().contiguous()  # (Kc, H)
        self.conv_b = _f(conv.bias)
        self.lin_w = _f(lin.weight).reshape(-1)
        self.lin_b = float(lin.bias.detach().float().item()) if lin.bias is not None else 0.0
        self.log_t = 1 if attend.log_t else 0
        self.Kc, self.H = self.conv_wT.shape
        self._addresses("conv_wT", "conv_b", "lin_w")

    def _addresses(self, *names):
        for n in names:
            setattr(self, "p_" + n, getattr(self, n).data_ptr())


class DecoderWeights(AttentionWeights):
    """fp32 contiguous views of the decoder parameters, in the layout the kernels take.  `fused`:
    the attention kernel runs the output projection (fc_fused), else sb_s2s_fc_rows does."""

    def __init__(self, m):
        super().__init__(m.attend)
        self.emb = _f(m.embedding.weight)
        self.w_ih, self.w_hh = _f(m.dec_rnn.weight_ih), _f(m.dec_rnn.weight_hh)
        self.b_ih, self.b_hh = _f(m.dec_rnn.bias_ih), _f(m.dec_rnn.bias_hh)
        self.fc_w, self.fc_b = _f(m.fc.fc.weight), _f(m.fc.fc.bias)
        self.H = self.w_hh.shape[1]
        self.C = self.fc_w.shape[0]
        if self.emb.shape[1] != self.H:
            raise _lib.SpeechB200Error("Seq2Seq: embedding_dim must equal the encoder dim (ix + sx)")
        self.fused = fc_fused(self.H, self.C)
        self._addresses("emb", "w_ih", "w_hh", "b_ih", "b_hh", "fc_w", "fc_b")


def attn_workspace(lib, B, T, H, dev):
    """zeroed scratch of the attention kernels (per-CTA softmax partials + ticket counters); one
    buffer serves every step of a decode on the same stream"""
    n = _lib.workspace_size(lib.sb_s2s_workspace_size, B, T, H)
    return torch.zeros(n, dtype=torch.uint8, device=dev)


def _a(x):
    """device address of a tensor; ints (addresses computed by the caller) and None pass through"""
    return x if x is None or isinstance(x, int) else x.data_ptr()


def _cell_fwd(lib, w, tok, tok_stride, sx_prev, hx_prev, hx, ix_save, gates_save, done, B, sp):
    ops._launch("s2s_cell_fwd", 0.0,
                lambda: lib.sb_s2s_cell_fwd(w.p_emb, tok, tok_stride, _a(sx_prev), _a(hx_prev),
                                            w.p_w_ih, w.p_w_hh, w.p_b_ih, w.p_b_hh, _a(hx),
                                            _a(ix_save), _a(gates_save), done, B, w.H, sp))


def _attn_fwd(lib, w, ws, eh, group, hx, ax_prev, sx, ax, B, T, sp, logits=None, logit_stride=0,
              logp=None, argmax=None, history=None, hist_stride=0, hist_col=0, end_count=None,
              end_tok=-1, done=None, with_fc=True, lens=None):
    """the attention step of B rows, row b over utterance b // group of eh; with_fc: also the
    output projection (w: DecoderWeights), else the attention alone (w may be AttentionWeights)"""
    fc_w, fc_b, C = (w.p_fc_w, w.p_fc_b, w.C) if with_fc else (None, None, 0)
    ops._launch("s2s_attn_fwd", 0.0,
                lambda: lib.sb_s2s_attn_fwd(_a(eh), group, _a(hx), _a(ax_prev), w.p_conv_wT,
                                            w.p_conv_b, w.p_lin_w, w.lin_b, w.log_t, B, T, w.H,
                                            w.Kc, _a(sx), _a(ax), fc_w, fc_b, C, logits,
                                            logit_stride, _a(logp), _a(argmax), history,
                                            hist_stride, hist_col, end_count, end_tok, done,
                                            _a(lens), _a(ws), ws.numel(), sp))


def fc_workspace(lib, R, C, dev):
    """zeroed scratch of sb_s2s_fc_rows / _logp for R rows (tile partials, log-sum-exp, tickets)"""
    n = _lib.workspace_size(lib.sb_s2s_fc_workspace_size, R, C)
    return torch.zeros(n, dtype=torch.uint8, device=dev)


def _fc_rows(lib, w, ws, hx, sx, R, sp, logits=None, group=0, ld0=0, ld1=0, argmax=None,
             history=None, hist_stride=0, hist_col=0, end_count=None, end_tok=-1, done=None):
    """logits of R rows o = hx + sx over many CTAs; row r at logits + (r % group) * ld0 +
    (r / group) * ld1 (default: dense (R, C)), with the row reductions of the same launch."""
    group = group or R
    ld0 = ld0 or w.C
    ops._launch("s2s_fc_rows", 2.0 * R * w.C * w.H,
                lambda: lib.sb_s2s_fc_rows(_a(hx), _a(sx), w.p_fc_w, w.p_fc_b, R, w.H, w.C,
                                           _a(logits), group, ld0, ld1, _a(argmax), _a(history),
                                           hist_stride, hist_col, _a(end_count), end_tok, _a(done),
                                           _a(ws), ws.numel(), sp))


def _fc_logp(lib, w, ws, logits, logp, R, sp, done=None):
    """logp (R, C) = logits (dense (R, C)) - the log-sum-exp the last _fc_rows left in ws"""
    ops._launch("s2s_fc_logp", 0.0,
                lambda: lib.sb_s2s_fc_logp(_a(logits), R, w.C, 0, _a(logp), R, w.C, _a(done),
                                           _a(ws), ws.numel(), sp))


def _dout_gemm(dl, fc_w, d_o):
    """d_o (R, H) = dl (R, C) @ fc_w (C, H) for C past sb_s2s_dout: 3-pass split-bf16 on the wgmma
    GEMM (hi*hi + hi*lo + lo*hi, relative error ~2^-16, as ops.gemm_split), fc_w read as [K][N]."""
    R, C = dl.shape
    H = fc_w.shape[1]
    Cp, Hp = (C + 7) // 8 * 8, (H + 7) // 8 * 8
    a_hi, a_lo = ops._split_bf16(dl, Cp)
    wp = fc_w
    if Cp != C:
        wp = torch.zeros(Cp, H, dtype=torch.float32, device=dl.device)
        wp[:C] = fc_w
    b_hi, b_lo = ops._split_bf16(wp, Hp)
    out = torch.empty(R, Hp, dtype=torch.float32, device=dl.device)
    ops.gemm_bf16_tn(a_hi, b_hi, out=out, b_mn=True)
    ops.gemm_bf16_tn(a_hi, b_lo, out=out, accumulate=True, b_mn=True)
    ops.gemm_bf16_tn(a_lo, b_hi, out=out, accumulate=True, b_mn=True)
    d_o.copy_(out[:, :H])


def attn_lens(lens, B, T, dev):
    """(B,) int32 device frames per utterance for the length-masked attention kernels, or None
    (every utterance attends over all T frames)."""
    if lens is None:
        return None
    ln = torch.as_tensor(lens).detach().to("cpu", torch.int64).reshape(-1)
    if ln.numel() != B:
        raise ValueError("lens must have one entry per utterance (%d), got %d" % (B, ln.numel()))
    if B and (int(ln.min()) < 1 or int(ln.max()) > T):
        raise ValueError("attention lens must lie in [1, T] (T = %d)" % T)
    if bool((ln == T).all()):
        return None
    return ln.to(torch.int32).to(dev)


def attn_step(attend, eh, dhx, ax_prev, lens=None):
    """NNAttention.forward on the decode path (no autograd): eh (B,T,H), dhx (B,1,H) or (B,H),
    ax_prev (B,T) or None; lens (optional): frames each utterance attends over (ax is 0 past
    them).  Returns (sx (B,1,H), ax (B,T)) like the reference module."""
    _lib.require_cuda(eh, "eh")
    lib = _lib.load()
    w = AttentionWeights(attend)
    eh = _f(eh)
    B, T, H = eh.shape
    d = dhx.detach().float().reshape(B, H).contiguous()
    axp = None if ax_prev is None else _f(ax_prev)
    sx = torch.empty(B, H, dtype=torch.float32, device=eh.device)
    ax = torch.empty(B, T, dtype=torch.float32, device=eh.device)
    ws = attn_workspace(lib, B, T, H, eh.device)
    ld = attn_lens(lens, B, T, eh.device)
    _attn_fwd(lib, w, ws, eh, 1, d, axp, sx, ax, B, T, _lib.stream_ptr(), with_fc=False, lens=ld)
    return sx.unsqueeze(1), ax


class DecodeFunction(torch.autograd.Function):
    """Teacher-forced decode (seq2seq.py:78-112): eh (B,T,H), tokens (B,U) -> logits (B,U-1,C),
    alignments (B,U-1,T).  sample_flags[u] (host bools, drawn by the caller from Python's `random`
    exactly as the reference does, :94): feed the arg-max of the previous step instead of the
    label.  lens (optional, (B,) int32 device): frames each utterance attends over."""

    @staticmethod
    def forward(ctx, eh, tokens, sample_flags, w, lens, emb_w, w_ih, w_hh, b_ih, b_hh, conv_w,
                conv_b, lin_w, lin_b, fc_w, fc_b):
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
        # large vocabularies: the attention without fc, the logits over many CTAs - per step when
        # the arg-max feeds the next step, else once over all steps*B rows after the loop
        fc_ws = None
        if not w.fused and steps > 0:
            fc_ws = fc_workspace(lib, B if sampling else steps * B, w.C, dev)
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
            if w.fused:
                _attn_fwd(lib, w, ws, ehc, 1, p_hx + (u + 1) * BH,
                          p_ax + (u - 1) * BT if u > 0 else None, p_sx + u * BH, p_ax + u * BT, B,
                          T, sp, logits=p_logits + 4 * u * w.C, logit_stride=steps * w.C,
                          argmax=p_amax, lens=lens)
                continue
            _attn_fwd(lib, w, ws, ehc, 1, p_hx + (u + 1) * BH,
                      p_ax + (u - 1) * BT if u > 0 else None, p_sx + u * BH, p_ax + u * BT, B, T,
                      sp, with_fc=False, lens=lens)
            if sampling:
                _fc_rows(lib, w, fc_ws, p_hx + (u + 1) * BH, p_sx + u * BH, B, sp,
                         logits=p_logits + 4 * u * w.C, ld0=steps * w.C, argmax=p_amax)
        if not w.fused and not sampling and steps > 0:
            # row r = u*B + b of (hx_all[1:], sx_all) -> logits[b, u]
            _fc_rows(lib, w, fc_ws, p_hx + BH, p_sx, steps * B, sp, logits=p_logits, group=B,
                     ld0=steps * w.C, ld1=w.C)
        ctx.w = w
        ctx.lens = lens
        ctx.saved = (ehc, hx_all, sx_all, ax_all, ix_all, gates_all, used)
        ctx.dims = (B, T, H, steps)
        ctx.vocab = emb_w.shape[0]
        ctx.conv_shape = conv_w.shape
        ctx.lin_shape = lin_w.shape
        ctx.has_lin_b = lin_b is not None
        return logits, ax_all.permute(1, 0, 2)

    @staticmethod
    def backward(ctx, dlogits, daligns):
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
        if dout_fits(C):
            ops._launch("s2s_dout", 0.0, lambda: lib.sb_s2s_dout(
                dl.data_ptr(), w.fc_w.data_ptr(), hx_all[1:].data_ptr(), sx_all.data_ptr(),
                d_o.data_ptr(), o_all.data_ptr(), steps * B, C, H, sp))
        else:
            torch.add(hx_all[1:], sx_all, out=o_all)
            _dout_gemm(dl.view(steps * B, C), w.fc_w, d_o.view(steps * B, H))
        BH, BT = 4 * B * H, 4 * B * T
        p_eh, p_hx, p_ax = ehc.data_ptr(), hx_all.data_ptr(), ax_all.data_ptr()
        p_gt, p_do, p_dix = gates_all.data_ptr(), d_o.data_ptr(), d_ix.data_ptr()
        p_dgi, p_dgh = d_gi.data_ptr(), d_gh.data_ptr()
        p_dax = (d_ax[0].data_ptr(), d_ax[1].data_ptr())
        p_dhd, p_dhp, p_deh = d_hx_direct.data_ptr(), d_hx_prev.data_ptr(), d_eh.data_ptr()
        p_gcw, p_gcb = g_conv_wT.data_ptr(), g_conv_b.data_ptr()
        p_glw, p_glb = g_lin_w.data_ptr(), g_lin_b.data_ptr()
        p_wihT, p_whhT, p_ws, n_ws = w_ihT.data_ptr(), w_hhT.data_ptr(), ws.data_ptr(), ws.numel()
        p_lens = _a(ctx.lens)
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
                p_dhd, p_gcw, p_gcb, p_glw, p_glb, w.log_t, B, T, H, Kc, p_lens, p_ws, n_ws, sp))
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
        return (d_eh, None, None, None, None, d_emb, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_conv_w, d_conv_b,
                d_lin_w, d_lin_b, d_fc_w, d_fc_b)


def decode(m, eh, tokens, sample_flags, lens=None):
    """logits (B, U-1, C), alignments (B, U-1, T) with autograd through the kernels above.
    lens (optional): frames each utterance attends over (alignments are 0 past them)."""
    w = DecoderWeights(m)
    lin = m.attend.nn[1].fc
    ld = attn_lens(lens, eh.shape[0], eh.shape[1], eh.device)
    return DecodeFunction.apply(eh, tokens, sample_flags, w, ld, m.embedding.weight,
                                m.dec_rnn.weight_ih, m.dec_rnn.weight_hh, m.dec_rnn.bias_ih,
                                m.dec_rnn.bias_hh, m.attend.conv.weight, m.attend.conv.bias,
                                lin.weight, lin.bias, m.fc.fc.weight, m.fc.fc.bias)


def decode_step(m, eh, y, state, softmax, lens=None):
    """One step (seq2seq.py:114-137), no autograd: y (B,1) tokens -> (out (B,C), (hx, ax, sx)).
    lens (optional): frames each utterance attends over."""
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
    ld = attn_lens(lens, B, T, dev)
    _cell_fwd(lib, w, tok.data_ptr(), 1, sx_prev, hx_prev, hx, None, None, None, B, sp)
    if w.fused:
        _attn_fwd(lib, w, ws, ehc, 1, hx, ax_prev, sx, ax, B, T, sp, logits=out.data_ptr(),
                  logit_stride=w.C, logp=logp, lens=ld)
    else:
        _attn_fwd(lib, w, ws, ehc, 1, hx, ax_prev, sx, ax, B, T, sp, with_fc=False, lens=ld)
        fc_ws = fc_workspace(lib, B, w.C, dev)
        _fc_rows(lib, w, fc_ws, hx, sx, B, sp, logits=out)
        if softmax:
            _fc_logp(lib, w, fc_ws, out, logp, B, sp)
    return (logp if softmax else out), (hx, ax, sx.unsqueeze(1))


def greedy(m, eh, start, end_tok, max_len, lens=None):
    """Greedy decode (seq2seq.py:145-178) without leaving the device: every kernel of every step
    is enqueued up front, kernels after the stop condition (all rows emitted end_tok in the same
    step, :155-156) are no-ops, ONE device->host copy returns the tokens.  -> (B, steps+1) list.
    lens (optional): frames each utterance attends over."""
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
    ld = attn_lens(lens, B, T, dev)
    fc_ws = None if w.fused else fc_workspace(lib, B, w.C, dev)
    for e in range(max_len):
        cur, prv = e & 1, (e & 1) ^ 1
        _cell_fwd(lib, w, hist.data_ptr() + 4 * e, max_len + 1, sx[prv] if e > 0 else None,
                  hx[prv], hx[cur], None, None, done.data_ptr(), B, sp)
        if w.fused:
            _attn_fwd(lib, w, ws, ehc, 1, hx[cur], ax[prv] if e > 0 else None, sx[cur], ax[cur], B,
                      T, sp, history=hist.data_ptr(), hist_stride=max_len + 1, hist_col=e + 1,
                      end_count=ctl.data_ptr() + 4 * e, end_tok=int(end_tok),
                      done=done.data_ptr(), lens=ld)
        else:
            _attn_fwd(lib, w, ws, ehc, 1, hx[cur], ax[prv] if e > 0 else None, sx[cur], ax[cur], B,
                      T, sp, done=done.data_ptr(), with_fc=False, lens=ld)
            _fc_rows(lib, w, fc_ws, hx[cur], sx[cur], B, sp, history=hist.data_ptr(),
                     hist_stride=max_len + 1, hist_col=e + 1, end_count=ctl.data_ptr() + 4 * e,
                     end_tok=int(end_tok), done=done.data_ptr())
        ops._launch("s2s_check_done", 0.0,
                    lambda: lib.sb_s2s_check_done(ctl.data_ptr() + 4 * e, B, done.data_ptr(),
                                                  nsteps.data_ptr(), e + 1, sp))
    n = int(nsteps.item())                      # the one synchronisation of the whole decode
    return hist[:, :n + 1].cpu().tolist()


def beam_search(m, eh, start_tok, end_tok, beam_size, max_len):
    """Seq2Seq.beam_search for one utterance (seq2seq.py:180-227): beam_search_batch on the first
    utterance of eh.  -> token tuple."""
    return beam_search_batch(m, _f(eh)[:1], start_tok, end_tok, beam_size, max_len)[0][0]


def beam_search_batch(m, eh, start_tok, end_tok, beam_size, max_len, lens=None, lm=None,
                      lm_weight=0.0, insertion_bonus=0.0, ctc=None):
    """Seq2Seq.beam_search (seq2seq.py:180-227) for each of the B utterances of eh (B, T, H) at
    once, device-resident.  Utterance b's K beam entries are rows b*K .. b*K+K-1 of the step
    kernels, which run over all B*K rows until every utterance has stopped; expand / prune /
    complete / stop run in one bookkeeping CTA per utterance and step (csrc/s2s.cu), and the
    hypotheses are back-tracked on the device.  Each utterance's search is the one it gets alone,
    bit for bit.  The host enqueues every step up front and reads all B results back in ONE copy.
    lens (optional): frames each utterance attends over.  lm (optional): an NGramLM whose classes
    are the vocabulary, blank the start token and end the end token (the caller checks), fused
    into every candidate as logp + (lm_weight * lm + insertion_bonus, no bonus for the end token);
    the scores are then the fused ones.  lm may instead be a WordLM with the same layout and a
    delimiter class: the word-LM entry points (csrc/s2s_beam.cuh, S2sWordLmFuse) score each word
    at its delimiter and the trailing word with </s> at the end token, insertion_bonus per word and
    lm.oov_penalty per word that leaves the lexicon, with each node's word state in a
    [B][node_cap][3] arena beside the hypothesis nodes.  ctc (optional): (y, ctc_weight,
    prebeam), joint CTC/attention decoding (csrc/s2s_ctc.cu) with y the float32 CTC
    log-probabilities (B, T, C), blank C - 1 = end_tok, start_tok = C: candidate c of row r is
    one of the row's `prebeam` classes with the largest P = (1 - ctc_weight) logp[c] (+ the LM
    part), valued (A_r + P) + ctc_weight * psi(h_r + c), psi the CTC prefix log-probability; the
    scores are then A + ctc_weight * psi.  -> list of B (token tuple, float64 score of that hypothesis, steps that
    utterance's search ran)."""
    lib = _lib.load()
    w = DecoderWeights(m)
    ehc = _f(eh)
    B, T, H = ehc.shape
    K, C = int(beam_size), w.C
    R = B * K
    dev = ehc.device
    ld = attn_lens(lens, B, T, dev)
    ctc_ld = ld
    if ld is not None:
        ld = ld.repeat_interleave(K)
    S = _lib.workspace_size(lib.sb_s2s_beam_state_size)
    out_cap = max_len + 2
    # the B states, then the B final hypotheses: the buffer the one device->host copy reads
    res = torch.zeros(B * S + 4 * B * out_cap, dtype=torch.uint8, device=dev)
    state, out_tokens = res[:B * S], res[B * S:].view(torch.int32)
    node_cap = 2 * K * (max_len + 1) + 2
    nodes = torch.zeros(B, node_cap, 2, dtype=torch.int32, device=dev)
    c_cap = K * (max_len + 1)
    c_scores = torch.zeros(B, c_cap, dtype=torch.float64, device=dev)
    parent = torch.zeros(R, dtype=torch.int32, device=dev)
    tok = torch.zeros(R, dtype=torch.int32, device=dev)
    stop = torch.zeros(2, dtype=torch.int32, device=dev)        # stopped utterances | batch done
    hx = [torch.zeros(R, H, dtype=torch.float32, device=dev) for _ in range(2)]
    sx = [torch.zeros(R, H, dtype=torch.float32, device=dev) for _ in range(2)]
    ax = [torch.zeros(R, T, dtype=torch.float32, device=dev) for _ in range(2)]
    logp = torch.empty(R, C, dtype=torch.float32, device=dev)
    sp = _lib.stream_ptr()
    ws = attn_workspace(lib, R, T, H, dev)
    _lib.check(lib.sb_s2s_beam_init_batch(state.data_ptr(), nodes.data_ptr(), node_cap,
                                          tok.data_ptr(), K, int(start_tok), stop.data_ptr(), B,
                                          sp), "beam init")
    done_ptr = stop.data_ptr() + 4              # the no-op flag of the step kernels
    fc_ws = None if w.fused else fc_workspace(lib, R, C, dev)
    split = ctc is None and not beam_select_fits(K, C)
    if split:
        sel_ws = torch.empty(_lib.workspace_size(lib.sb_s2s_beam_split_workspace_size_batch, K, C,
                                                 B), dtype=torch.uint8, device=dev)
    p_state, p_c, p_nodes = state.data_ptr(), c_scores.data_ptr(), nodes.data_ptr()
    p_par, p_tok, p_out = parent.data_ptr(), tok.data_ptr(), out_tokens.data_ptr()
    p_stop = stop.data_ptr()
    kind = fusion_kind(lm)
    fusion = fusion_args(lm, lm_weight, insertion_bonus, dev)
    if kind is WordLM:
        word_nodes = torch.empty(B, node_cap, 3, dtype=torch.int32, device=dev)
        fusion += (word_nodes.data_ptr(),)
    if ctc is not None:
        y, lam, M = ctc
        if tuple(y.shape) != (B, T, C) or y.dtype != torch.float32 or y.device != ehc.device:
            raise ValueError("ctc log-probabilities must be float32 (%d, %d, %d) on the encoder's "
                             "device, got %s %s" % (B, T, C, y.dtype, tuple(y.shape)))
        y = y.contiguous()
        lam, M = float(lam), int(M)
        cbuf = torch.empty(_lib.workspace_size(lib.sb_s2s_ctc_state_size, K, M, T, B),
                           dtype=torch.uint8, device=dev)
        cargs = (y.data_ptr(), _a(ctc_ld), cbuf.data_ptr(), cbuf.numel())
        shape = (K, C, M, T, int(start_tok), int(end_tok), lam)
        _lib.check(lib.sb_s2s_ctc_init(*cargs, *shape, B, sp), "ctc init")
        # the joint candidates take a null LM where there is none
        head = (cargs[0], cargs[1], p_state, p_nodes, node_cap, cargs[2], cargs[3], *shape)
        tail = (p_stop, B, *(fusion or (None, 0.0, 0.0)))
    else:
        head = (p_state, p_c, p_nodes, p_par, p_tok, p_out, K, C, int(end_tok))
        tail = (max_len, node_cap, c_cap, p_stop, B,
                *((sel_ws.data_ptr(), sel_ws.numel()) if split else ()), *fusion)
    name, symbol = _SELECT["ctc" if ctc is not None else "split" if split else "single", kind]
    select = getattr(lib, symbol)
    # buffers: [0] = state entering the step (gathered), [1] = state produced by the step
    for e in range(max_len):
        _cell_fwd(lib, w, p_tok, 1, sx[0] if e > 0 else None, hx[0], hx[1], None, None, done_ptr,
                  R, sp)
        if w.fused:
            _attn_fwd(lib, w, ws, ehc, K, hx[1], ax[0] if e > 0 else None, sx[1], ax[1], R, T, sp,
                      logp=logp, done=done_ptr, lens=ld)
        else:
            _attn_fwd(lib, w, ws, ehc, K, hx[1], ax[0] if e > 0 else None, sx[1], ax[1], R, T, sp,
                      done=done_ptr, with_fc=False, lens=ld)
            _fc_rows(lib, w, fc_ws, hx[1], sx[1], R, sp, logits=logp, done=done_ptr)
            _fc_logp(lib, w, fc_ws, logp, logp, R, sp, done=done_ptr)
        ops._launch(name, 0.0, lambda: select(logp.data_ptr(), *head, e, *tail, sp))
        if ctc is not None:
            ops._launch("s2s_ctc_select", 0.0, lambda: lib.sb_s2s_ctc_select_batch(
                *cargs, p_state, p_c, p_nodes, p_par, p_tok, p_out, *shape, e, max_len, node_cap,
                c_cap, p_stop, B, sp))
        ops._launch("s2s_beam_gather", 0.0, lambda: lib.sb_s2s_beam_gather_batch(
            hx[1].data_ptr(), sx[1].data_ptr(), ax[1].data_ptr(), hx[0].data_ptr(),
            sx[0].data_ptr(), ax[0].data_ptr(), p_par, p_state, K, H, T, B, sp))
    host = res.cpu()                            # the one synchronisation of the whole search
    st = host[:B * S].view(B, S)
    steps = st[:, BEAM_DONE_OFFSET:BEAM_DONE_OFFSET + 4].contiguous().view(torch.int32).reshape(B)
    n = st[:, BEAM_OUT_LEN_OFFSET:BEAM_OUT_LEN_OFFSET + 4].contiguous().view(torch.int32).reshape(B)
    score = st[:, S - 8:].contiguous().view(torch.float64).reshape(B)
    toks = host[B * S:].view(torch.int32).view(B, out_cap)
    return [(tuple(toks[b, :int(n[b])].tolist()), float(score[b]), int(steps[b]))
            for b in range(B)]


# ---- two-pass decoding: CTC prefix beam search N-best, then attention rescoring ----------------

def ctc_first_pass(y, frames, K):
    """The first pass over whole utterances: y (B, T, C) float32 CTC log-probabilities (blank
    C - 1), frames[b] <= T the frames of utterance b.  One reset, one step over all T frames and
    one N-best read: the streaming path, whose entry 0 is sb_ctc_prefix_beam's result.
    -> ctc_decoder.StreamSearch.nbest's (labels, lens, c)."""
    B, T, C = y.shape
    search = StreamSearch(B, T, K, C - 1, y.device)
    search.push(y, frames)
    return search.nbest()


def score_batch(m, eh, tokens, lens, K, frame_lens=None):
    """Teacher-forced attention scores of R = B*K hypotheses, K per utterance of eh (B, T, H):
    tokens (R, ld) int32 on the device, row r START then its lens[r] labels (lens (R) int32 on the
    device, -1 for a row that scores nothing); frame_lens (optional): frames each utterance
    attends over.  Runs recognize's step sequence over the R rows (row r attends over utterance
    r // K) for ld - 1 steps, sb_s2s_score_tokens after each step's log-softmax, with nothing
    copied to the host.  -> a (R,) float64: sum over u = 0..lens[r] of the float32 log-probability
    of the forced token (the next label, then END), as recognize's selection adds them."""
    lib = _lib.load()
    w = DecoderWeights(m)
    ehc = _f(eh)
    B, T, H = ehc.shape
    R, ld = tokens.shape
    C = w.C
    dev = ehc.device
    if R != B * K or tuple(lens.shape) != (R,):
        raise ValueError("score_batch needs %d rows of tokens and lens, got %s / %s"
                         % (B * K, tuple(tokens.shape), tuple(lens.shape)))
    end_tok = m.embedding.num_embeddings - 2
    tok = tokens.to(dev, torch.int32).contiguous()
    ln = lens.to(dev, torch.int32).contiguous()
    al = attn_lens(frame_lens, B, T, dev)
    if al is not None:
        al = al.repeat_interleave(K)
    acc = torch.zeros(R, dtype=torch.float64, device=dev)
    hx = [torch.zeros(R, H, dtype=torch.float32, device=dev) for _ in range(2)]
    sx = [torch.empty(R, H, dtype=torch.float32, device=dev) for _ in range(2)]
    ax = [torch.empty(R, T, dtype=torch.float32, device=dev) for _ in range(2)]
    logp = torch.empty(R, C, dtype=torch.float32, device=dev)
    sp = _lib.stream_ptr()
    ws = attn_workspace(lib, R, T, H, dev)
    fc_ws = None if w.fused else fc_workspace(lib, R, C, dev)
    p_tok, p_ln, p_acc, p_logp = tok.data_ptr(), ln.data_ptr(), acc.data_ptr(), logp.data_ptr()
    for u in range(ld - 1):
        cur, prv = u & 1, (u & 1) ^ 1
        _cell_fwd(lib, w, p_tok + 4 * u, ld, sx[prv] if u > 0 else None, hx[prv], hx[cur], None,
                  None, None, R, sp)
        if w.fused:
            _attn_fwd(lib, w, ws, ehc, K, hx[cur], ax[prv] if u > 0 else None, sx[cur], ax[cur],
                      R, T, sp, logp=logp, lens=al)
        else:
            _attn_fwd(lib, w, ws, ehc, K, hx[cur], ax[prv] if u > 0 else None, sx[cur], ax[cur],
                      R, T, sp, with_fc=False, lens=al)
            _fc_rows(lib, w, fc_ws, hx[cur], sx[cur], R, sp, logits=logp)
            _fc_logp(lib, w, fc_ws, logp, logp, R, sp)
        ops._launch("s2s_score_tokens", 0.0, lambda: lib.sb_s2s_score_tokens(
            p_logp, R, C, p_tok, ld, p_ln, u, end_tok, p_acc, sp))
    return acc


def two_pass_select(a, c, valid, ctc_weight):
    """The combination r = (1 - w) a + w c in float64 (both products rounded, then added) of the
    (B, K) attention scores a and CTC log-probabilities c; slots where `valid` is False (empty
    beam slots) get -inf.  -> (index of the largest r per row, the first on ties; r)."""
    w = float(ctc_weight)
    r = torch.mul(a, 1.0 - w).add_(torch.mul(c, w))
    r = torch.where(valid, r, torch.full_like(r, -float("inf")))
    return torch.argmax(r, dim=1), r


def rescore(m, eh, nbest, frame_lens, K, ctc_weight, return_scores):
    """The second pass over a first pass's N-best (StreamSearch.nbest's output, utterance b's
    entries over eh[b]) and the selection: -> B token lists [START] + y + [END] (and their float64
    scores r).
    Reads the longest hypothesis's length before the step loop and the chosen hypotheses once at
    the end: two device-to-host copies per call."""
    labels, lens, c = nbest
    B, _, Lcap = labels.shape
    dev = labels.device
    V = m.embedding.num_embeddings
    start, end = V - 1, V - 2
    L = max(0, int(lens.max()))
    R = B * K
    col = torch.arange(L, device=dev, dtype=torch.int32)
    body = torch.where(col < lens.view(R, 1), labels.view(R, Lcap)[:, :L],
                       torch.full((1, 1), end, dtype=torch.int32, device=dev))
    tokens = torch.cat([torch.full((R, 1), start, dtype=torch.int32, device=dev), body,
                        torch.full((R, 1), end, dtype=torch.int32, device=dev)], 1)
    a = score_batch(m, eh, tokens, lens.view(R), K, frame_lens).view(B, K)
    best, r = two_pass_select(a, c, lens >= 0, ctc_weight)
    rows = torch.arange(B, device=dev) * K + best
    # [B float64 scores | B lengths | B rows of L labels] as int32, the scores 8-byte aligned
    out = torch.cat([r.gather(1, best.view(B, 1)).view(torch.int32).reshape(-1),
                     lens.view(R)[rows], body[rows].reshape(-1)])
    host = out.cpu()                            # the chosen hypotheses, in one copy
    score = host[:2 * B].view(torch.float64).tolist()
    n = host[2 * B:3 * B].tolist()
    lab = host[3 * B:].view(B, L)
    res = [[start] + lab[b, :n[b]].tolist() + [end] for b in range(B)]
    return (res, score) if return_scores else res


def recognize_two_pass(m, eh, y, frame_lens, K, ctc_weight, return_scores):
    """Two-pass decoding of whole utterances: eh (B, T, H) encoder states, y (B, T, C) float32
    CTC log-probabilities; frame_lens (optional) the frames of each utterance (default T)."""
    B, T, _ = y.shape
    frames = [T] * B if frame_lens is None else [int(f) for f in frame_lens]
    nbest = ctc_first_pass(y.contiguous(), frames, K)
    return rescore(m, eh, nbest, frame_lens, K, ctc_weight, return_scores)
