"""Rounding-faithful CPU reference of the GRU recurrence kernels (test infrastructure, never
imported by speech_b200/): sb_gru_fwd / sb_gru_bwd restated in plain torch, fp64 by default, with
the bf16 roundings the kernels apply at the points where they apply them, so that what is left
between a kernel and this reference is fp32 arithmetic alone.

Layouts are those of the C ABI (time-major, row m = t * Bp + b):
  gi    [T*Bp][ndir*3H]   input projections, b_ih included
  whh   [ndir][3H][H]     W_hh (rows r | z | n)
  bhh   [ndir][3H]
  y     [T*Bp][ndir*H]    h_t
  gates [T*Bp][ndir][4][H] r, z, n, hn = W_hn h_{t-1} + b_hn
Direction 0 runs t = 0 .. T-1, direction 1 t = T-1 .. 0, each from h = 0.

Where the kernels round (gru.cu, every variant):
  forward   the product W_hh h_{t-1} takes bf16 W_hh and bf16 h_{t-1} (the xn rows the CTAs
            exchange) and accumulates in fp32; the gate math and h_t = (1-z) n + z h_{t-1} use the
            fp32 h_{t-1} each thread keeps in registers; xn = bf16(h_t).
  backward  the recurrent product W_hh^T [dr | dz | dhn] takes the bf16 exchange row; the direct
            path g z, the gate gradients and the bias sums stay fp32; dgi and dghn are stored
            as bf16.
The K-split and wide variants (ks4, ks2, kt, ks_l2, ks4_x2, wide) split the contraction over CTAs
or stream W_hh through L2, but every partial product they exchange (DSMEM, the L2 staging area,
the transposed staging slices) is fp32, and the bf16 operands are the same rows: they change the
fp32 summation order and nothing else, so one reference serves all eleven.
"""
import torch

# ---- bars ---------------------------------------------------------------------------------------
# The comparisons are teacher-forced (h_prev / xr below): each step of the reference starts from
# the kernel's own previous state, so a bar bounds the error of one step, and a one-bit flip of a
# bf16 operand is not carried into the steps after it (free-running, the recurrence amplifies
# such flips to 3e-4 at gain 1 and 5e-3 at gain 3 by T = 60: as much as some of the faults below).
# Calibration: the fp32 emulation of the kernels' arithmetic (gru_fwd / gru_bwd with
# dtype=float32, every rounding point above), teacher-forced against this fp64 reference, weights
# U(+-g/sqrt(H)) with gains 1 and 3, gi ~ N(0, 1), at T = 60 H = 256, T = 20 H = 128 (both
# directions) and T = 247 H = 1024:
#   forward  fwd_err: emulation <= 7.1e-7; the mutations of MUTATIONS >= 1.9e-3 (z h on bf16 h)
#   backward bias sums, rel_err: emulation <= 2.3e-7; mutations >= 9.3e-4 (g z rounded to bf16)
#   backward dgi / dghn, bwd_elem_err (beyond one bf16 ulp): emulation <= 2.4e-8; mutations
#            >= 1.0e-3 (g z rounded to bf16), the missing K chunk >= 2.6e-3
# The bars sit about 20x below the smallest fault and leave the kernels' tensor-core accumulation
# and fast exp / divide two orders of magnitude above the emulation.  Measured on an H100 80GB
# HBM3 (700 W power limit), every case of tests/test_gru_rounded_gpu.py at gains 1 and 3:
# forward <= 6.0e-6 (wide, H = 2144, gain 3; ks2 at the benchmark shape 1.8e-6), dgi / dghn
# beyond one ulp <= 7.1e-7, bias sums <= 2.4e-6.
FWD_ABS = 5e-5
DB_REL = 1e-4
BWD_FLOOR = 1e-4
# sb_gru_fwd_f32 (fp32 weights and state, expf / tanhf) against rounded=False, teacher-forced;
# measured on the same H100: <= 1.6e-6 (T = 247, H = 1024, gain 3)
F32_ABS = 1e-5
# ops.gru_stack against gru_stack below, which cannot be teacher-forced: free-running, one flipped
# bf16 operand of a layer input or of dgi moves a weight-gradient entry by up to 2e-3 of the
# largest.  The fp32 emulation of a 2-layer biGRU-250 at T = 24 and 40 with ragged lengths, nn.GRU
# initialisation: y <= 2.0e-4 absolute, dx and every weight / bias gradient <= 2.1e-3 of the
# largest entry (against 2e-2 and 3e-2 in the fp64 nn.GRU parity tests); measured on the same
# H100: y <= 1.9e-4, gradients <= 2.0e-3.
STACK_Y_ABS = 1e-3
STACK_GRAD_REL = 6e-3

MUTATIONS = (
    "zh_bf16",         # forward: z * h_{t-1} on the bf16 h_{t-1} instead of the fp32 one
    "missing_chunk",   # forward: units 0..15 miss the product of K chunk 1 (h columns 64..127)
    "bhn_outside",     # forward: n = tanh(gi_n + r * (W_hn h) + b_hn), b_hn outside the reset gate
    "fwd_start",       # forward: step 1 of each direction also runs without the recurrent product
    "bwd_missing_chunk",  # backward: units 0..15 miss rows 64..127 of W_hh^T [dr | dz | dhn]
    "gz_bf16",         # backward: the direct path g * z rounded to bf16
    "bwd_start",       # backward: h_{t-1} = 0 one step past the direction's first step
)


def bf16(x):
    """x rounded to bf16 (round to nearest even), in x's dtype"""
    return x.to(torch.bfloat16).to(x.dtype)


def _order(T, d):
    """forward time order of direction d"""
    return list(range(T)) if d == 0 else list(range(T - 1, -1, -1))


def _check_mutation(mutate):
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError("unknown mutation %r" % (mutate,))


def _fwd_product(hb, W, mutate):
    """W_hh h_{t-1} of one direction: hb [..., H] (already rounded), W [3H][H] -> [..., 3, H]"""
    H = W.shape[1]
    acc = (hb @ W.t()).unflatten(-1, (3, H))
    if mutate == "missing_chunk" and H > 64:
        part = (hb[..., 64:128] @ W[:, 64:128].t()).unflatten(-1, (3, H))
        acc[..., :16] -= part[..., :16]
    return acc


def _fwd_cell(g, acc, bh, h, mutate):
    """g [..., 3, H] input projections, acc [..., 3, H] the product, bh [3, H] b_hh, h = h_{t-1}
    -> h_t, gates [..., 4, H]"""
    r = torch.sigmoid(g[..., 0, :] + acc[..., 0, :] + bh[0])
    z = torch.sigmoid(g[..., 1, :] + acc[..., 1, :] + bh[1])
    hn = acc[..., 2, :] + bh[2]
    if mutate == "bhn_outside":
        n = torch.tanh(g[..., 2, :] + r * acc[..., 2, :] + bh[2])
    else:
        n = torch.tanh(g[..., 2, :] + r * hn)
    hz = bf16(h) if mutate == "zh_bf16" else h
    return (1 - z) * n + z * hz, torch.stack([r, z, n, hn], -2)


def gru_fwd(gi, whh, bhh, T, rounded=True, dtype=torch.float64, mutate=None, h_prev=None):
    """-> y [T*Bp][ndir*H], gates [T*Bp][ndir][4][H], xn = bf16(y) (torch.bfloat16), on the CPU.
    rounded=False: plain GRU math in `dtype` (nn.GRU's recurrence, h_{-1} = 0).
    h_prev (optional, [T*Bp][ndir*H]): a kernel's y.  Each step then starts from that y at the
    direction's previous step instead of the reference's own state (teacher forcing, see the bars);
    the steps are then independent and computed all at once."""
    _check_mutation(mutate)
    rnd = bf16 if rounded else (lambda v: v)
    ndir, H3, H = whh.shape
    gi = gi.detach().cpu().to(dtype).view(T, -1, ndir, 3, H)
    Bp = gi.shape[1]
    W = rnd(whh.detach().cpu().to(dtype))
    bh = bhh.detach().cpu().to(dtype).view(ndir, 3, H)
    y = torch.zeros(T, Bp, ndir, H, dtype=dtype)
    gates = torch.zeros(T, Bp, ndir, 4, H, dtype=dtype)
    for d in range(ndir):
        order = _order(T, d)
        if h_prev is not None:
            hk = h_prev.detach().cpu().to(dtype).view(T, Bp, ndir, H)[:, :, d]
            hp = torch.zeros(T, Bp, H, dtype=dtype)            # in this direction's step order
            hp[1:] = hk[order[:-1]]
            acc = _fwd_product(rnd(hp), W[d], mutate)
            acc[0] = 0
            if mutate == "fwd_start" and T > 1:
                acc[1] = 0
            h, g = _fwd_cell(gi[order, :, d], acc, bh[d], hp, mutate)
            y[order, :, d] = h
            gates[order, :, d] = g
            continue
        h = torch.zeros(Bp, H, dtype=dtype)
        for step, t in enumerate(order):
            acc = _fwd_product(rnd(h), W[d], mutate)
            if step == 0 or (mutate == "fwd_start" and step == 1):
                acc = torch.zeros_like(acc)
            h, gates[t, :, d] = _fwd_cell(gi[t, :, d], acc, bh[d], h, mutate)
            y[t, :, d] = h
    y = y.view(T * Bp, ndir * H)
    return y, gates.view(T * Bp, ndir, 4, H), y.to(torch.bfloat16)


def gru_bwd(dy, y, gates, whh, T, rounded=True, dtype=torch.float64, mutate=None, xr=None):
    """Backward recurrence fed the forward's y and gates (any source) and dL/dy.
    -> dgi [T*Bp][ndir*3H] = (dr, dz, dn), dghn [T*Bp][ndir*H] = dn * r, both UNROUNDED (the
    kernels store bf16 of these), and the bias gradients dbih = sum (dr, dz, dn),
    dbhh = sum (dr, dz, dhn) over t and every row [ndir*3H].
    xr (optional): a kernel's bf16 (dgi, dghn).  The recurrent product of each step then takes
    that step's stored bf16 dr, dz and dhn, the exchange row the kernel multiplied, instead of the
    reference's own rounding of them (teacher forcing, see the bars)."""
    _check_mutation(mutate)
    rnd = bf16 if rounded else (lambda v: v)
    ndir, H3, H = whh.shape
    dy = dy.detach().cpu().to(dtype).view(T, -1, ndir, H)
    Bp = dy.shape[1]
    y = y.detach().cpu().to(dtype).view(T, Bp, ndir, H)
    gates = gates.detach().cpu().to(dtype).view(T, Bp, ndir, 4, H)
    W = rnd(whh.detach().cpu().to(dtype))
    dgi = torch.zeros(T, Bp, ndir, 3, H, dtype=dtype)
    dghn = torch.zeros(T, Bp, ndir, H, dtype=dtype)
    prods = None
    for d in range(ndir):
        if xr is not None:
            rows = torch.cat([xr[0].detach().cpu().to(dtype).view(T, Bp, ndir, 3 * H)[:, :, d, :2 * H],
                              xr[1].detach().cpu().to(dtype).view(T, Bp, ndir, H)[:, :, d]], 2)
            prods = rows @ W[d]
            if mutate == "bwd_missing_chunk" and 3 * H > 64:
                prods[..., :16] -= (rows[..., 64:128] @ W[d][64:128])[..., :16]
        dh_rec = torch.zeros(Bp, H, dtype=dtype)
        order = _order(T, d)
        for step, t in enumerate(order[::-1]):
            r, z, n, hn = gates[t, :, d].unbind(1)
            first = step == T - 1 or (mutate == "bwd_start" and step == T - 2)
            hp = torch.zeros(Bp, H, dtype=dtype) if first else y[t - 1 if d == 0 else t + 1, :, d]
            g = dy[t, :, d] + dh_rec
            dn = g * (1 - z) * (1 - n * n)
            dz = g * (hp - n) * z * (1 - z)
            dr = dn * hn * r * (1 - r)
            dhn = dn * r
            dgi[t, :, d] = torch.stack([dr, dz, dn], 1)
            dghn[t, :, d] = dhn
            if prods is not None:
                prod = prods[t]
            else:
                row = torch.cat([rnd(dr), rnd(dz), rnd(dhn)], 1)
                prod = row @ W[d]
                if mutate == "bwd_missing_chunk" and 3 * H > 64:
                    prod[:, :16] -= (row[:, 64:128] @ W[d][64:128])[:, :16]
            gz = g * z
            dh_rec = (bf16(gz) if mutate == "gz_bf16" else gz) + prod
    dbih = dgi.sum((0, 1)).reshape(ndir * 3 * H)
    dbhh = torch.cat([dgi[..., :2, :], dghn.unsqueeze(3)], 3).sum((0, 1)).reshape(ndir * 3 * H)
    return dgi.view(T * Bp, ndir * 3 * H), dghn.view(T * Bp, ndir * H), dbih, dbhh


# ---- comparisons --------------------------------------------------------------------------------
def fwd_err(y, gates, y_ref, gates_ref):
    """max abs error of y and of r, z, n, and of hn relative to max(1, |hn|max)"""
    y, gates = y.double().cpu(), gates.double().cpu()
    y_ref, gates_ref = y_ref.double().cpu(), gates_ref.double().cpu()
    e = (y - y_ref).abs().max().item()
    e = max(e, (gates[:, :, :3] - gates_ref[:, :, :3]).abs().max().item())
    hn_scale = max(1.0, gates_ref[:, :, 3].abs().max().item())
    return max(e, (gates[:, :, 3] - gates_ref[:, :, 3]).abs().max().item() / hn_scale)


def bf16_ulp(x):
    """the spacing of bf16 numbers at |x| (8 significant bits), elementwise, in float64"""
    x = x.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(x)) - 7)


def bwd_elem_err(got, ref):
    """max over elements of |got - ref| - (one bf16 ulp of ref), relative to max |ref|: <= BWD_FLOOR
    when every element of the bf16 output is within one ulp plus BWD_FLOOR * max |ref|"""
    got, ref = got.double().cpu(), ref.double().cpu()
    excess = ((got - ref).abs() - bf16_ulp(ref)).max().item()
    return excess / max(ref.abs().max().item(), 1e-30)


def rel_err(got, ref):
    """max |got - ref| / max |ref|"""
    got, ref = got.double().cpu(), ref.double().cpu()
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def bwd_errs(out, ref):
    """(dgi, dghn, dbih, dbhh) against the reference's -> (dgi/dghn element error, bias error)"""
    return (max(bwd_elem_err(out[0], ref[0]), bwd_elem_err(out[1], ref[1])),
            max(rel_err(out[2], ref[2]), rel_err(out[3], ref[3])))


# ---- the GRU stack (speech_b200.ops.GRUStackFunction) ---------------------------------------------
def _align(a, lens, right):
    """time_align of a [T][Bp][cols]: right=True moves frame t of row b to t + T - lens[b]"""
    T = a.shape[0]
    out = torch.zeros_like(a)
    for b, n in enumerate(lens):
        if right:
            out[T - n:, b] = a[:n, b]
        else:
            out[:n, b] = a[T - n:, b]
    return out


def gru_stack(x, weights, ndir, dout, lens=None, rounded=True, dtype=torch.float64):
    """Forward and backward of ops.gru_stack (batch_first, h0 = 0, no dropout) with the glue's
    rounding points: bf16 layer inputs and W_ih into an fp32 gi, the recurrence of gru_fwd /
    gru_bwd, bf16 dgi and dghn into the weight-gradient and dX contractions, bf16 h_{t-1} for
    dW_hh (rounded=False: none of them).  The reverse direction of an utterance shorter than T
    runs on right-aligned frames.
    Runs at the layer's own width (no padded units: a zero unit is exact).
    weights: nn.GRU's parameters in its order; dout (B, T, ndir*H) dL/dy.
    -> y (B, T, ndir*H) zero past lens, dx (B, T, In), [gradient of each weight]."""
    rnd = bf16 if rounded else (lambda v: v)
    B, T, In = x.shape
    Bp = (B + 7) // 8 * 8
    lens = [T] * Bp if lens is None else list(lens) + [T] * (Bp - B)
    L = len(weights) // (4 * ndir)
    w = [q.detach().cpu().to(dtype) for q in weights]
    H = w[1].shape[1]
    valid = (torch.arange(T)[:, None] < torch.tensor(lens)[None, :]).to(dtype)   # [T][Bp]
    X = torch.zeros(T, Bp, In, dtype=dtype)
    X[:, :B] = rnd(x.detach().cpu().to(dtype)).transpose(0, 1)
    saved = []
    for l in range(L):
        wl = w[l * 4 * ndir:(l + 1) * 4 * ndir]
        gi = torch.cat([(_align(X, lens, True) if d else X) @ rnd(wl[4 * d]).t() + wl[4 * d + 2]
                        for d in range(ndir)], 2)
        whh = rnd(torch.stack([wl[4 * d + 1] for d in range(ndir)]))
        bhh = torch.stack([wl[4 * d + 3] for d in range(ndir)])
        y, gates, _ = gru_fwd(gi.reshape(T * Bp, -1), whh, bhh, T, rounded, dtype)
        y = y.view(T, Bp, ndir, H)
        saved.append((X, y, gates, whh))
        if ndir == 2:
            y = torch.stack([y[:, :, 0], _align(y[:, :, 1], lens, False)], 2)
        X = rnd(y.reshape(T, Bp, ndir * H))
    out = y.reshape(T, Bp, ndir * H) * valid[:, :, None]
    dY = torch.zeros(T, Bp, ndir * H, dtype=dtype)
    dY[:, :B] = dout.detach().cpu().to(dtype).transpose(0, 1)
    dY = dY * valid[:, :, None]
    grads = [None] * len(w)
    for l in reversed(range(L)):
        X, y, gates, whh = saved[l]
        dY = dY.view(T, Bp, ndir, H)
        if ndir == 2:
            dY = torch.stack([dY[:, :, 0], _align(dY[:, :, 1], lens, True)], 2)
        dgi, dghn, dbih, dbhh = gru_bwd(dY.reshape(T * Bp, -1), y.reshape(T * Bp, -1), gates, whh,
                                        T, rounded, dtype)
        dgi = rnd(dgi).view(T, Bp, ndir, 3 * H)
        dghn = rnd(dghn).view(T, Bp, ndir, H)
        hb = rnd(y)
        dX = torch.zeros(T, Bp, X.shape[2], dtype=dtype)
        for d in range(ndir):
            base = (l * ndir + d) * 4
            rows = torch.cat([dgi[:, :, d, :2 * H], dghn[:, :, d]], 2)
            cur, prev = (slice(1, T), slice(0, T - 1)) if d == 0 else (slice(0, T - 1), slice(1, T))
            grads[base + 1] = torch.einsum("tbk,tbh->kh", rows[cur], hb[prev, :, d])
            grads[base + 2] = dbih[d * 3 * H:(d + 1) * 3 * H]
            grads[base + 3] = dbhh[d * 3 * H:(d + 1) * 3 * H]
            dgx = _align(dgi[:, :, d], lens, False) if d else dgi[:, :, d]
            grads[base] = torch.einsum("tbk,tbi->ki", dgx, X)
            dX = dX + dgx @ rnd(w[base])
        dY = dX
    return out[:, :B].transpose(0, 1), dY[:, :B].transpose(0, 1), grads
