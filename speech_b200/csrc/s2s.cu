// Attention decoder step of the sequence-to-sequence model: forward and backward kernels.
//
// Replaces, for Seq2Seq.decode / decode_step (speech/models/seq2seq.py:78-137) and
// NNAttention.forward (:344-360), the per-token chain of small library calls the reference runs
// (nn.Embedding, nn.GRUCell -> cuBLAS, Conv1d -> cuDNN, broadcast add / ReLU / Linear / softmax /
// weighted sum -> ATen, LinearND -> cuBLAS; ~8 launches and a (B,T,H) temporary per token):
//   step u:  ix = emb[y_u] + sx_{u-1}                                   (:84,:100-101)
//            hx_u = GRUCell(ix, hx_{u-1})                               (:103)
//            score_t = w . relu(eh_t + hx_u + conv1d(ax_{u-1})_t) + b   (:345-353)
//            ax_u = softmax_t(score [* log T]);  sx_u = sum_t ax_u[t] eh_t   (:354-359)
//            out_u = fc(hx_u + sx_u)                                    (:108)
// as two kernels per token forward and three backward:
//   s2s_cell_fwd      embedding gather + context add + GRU cell in fp32 on CUDA cores: one warp
//                     per hidden unit, lanes over K, 16 batch rows in registers (every weight is
//                     read once per token: 6 H^2 floats from L2, FMA-bound);
//   s2s_attn_fwd      grid (T/24, B): every CTA scores 24 frames of one utterance with ONE pass
//                     over its encoder states (online softmax; the reference reads them twice and
//                     materialises a (B,T,H) temporary); the utterance's last CTA (ticket counter)
//                     combines the partials in a fixed order and runs the output projection and,
//                     for the decode path, the arg-max token / log-softmax of the step, so that
//                     greedy and beam decoding never leave the device;
//   s2s_attn_bwd_a/b  gradient of the step's attention on the same grid (the softmax Jacobian
//                     needs sum_t a_t da_t over all frames: kernel A; everything else: kernel B),
//                     accumulates d eh in place, emits d ax_{u-1}, the parameter gradients of the
//                     attention, and the gate pre-activation gradients of the cell (so the cell's
//                     backward is a pure matrix product);
//   s2s_cell_bwd      d ix = d gi W_ih, d hx_{u-1} = d gh W_hh + z * d hx_u on transposed weights.
// The output-projection backward (d o = dlogits W_fc) of ALL steps is one launch before the loop
// (s2s_dout); the weight gradients of the cell, the embedding and fc are time-batched contractions
// over all (u, b) rows and run once per sequence on the wgmma GEMM (SB_GEMM_A_MN | SB_GEMM_B_MN).
// Everything is fp32 (the reference's arithmetic); roofline: L2 bandwidth on eh and the cell
// weights per token (B*T*H*4 bytes forward, 3x that backward, + 24 H^2), in practice launch-bound.
#include "s2s_beam.cuh"
#include <math.h>
#include <stddef.h>
#include <string.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int CELL_WARPS = 4;     // warps per CTA of the cell kernels
static constexpr int CELL_NB = 8;        // batch rows per CTA (accumulators live in registers)
static constexpr int ATT_THREADS = 256;
static constexpr int ATT_NW = ATT_THREADS / 32;
static constexpr int ATT_FG = 3;                        // consecutive frames per warp
static constexpr int ATT_TT = ATT_NW * ATT_FG;          // frames per CTA
static constexpr int ATT_KMAX = 16;                     // taps of the location conv: odd, <= 15
static constexpr int ATT_WIN = ATT_FG + ATT_KMAX - 1;   // alignment window of one frame group
static constexpr int ATT_MAX_TS = 256;                  // CTAs per utterance (T <= 6144)

SB_DEVINL float dot4(const float4 a, const float4 b) {
  return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
}
SB_DEVINL float4 add4(const float4 a, const float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
// a * s + c
SB_DEVINL float4 fma4(const float4 a, const float s, const float4 c) {
  return make_float4(fmaf(a.x, s, c.x), fmaf(a.y, s, c.y), fmaf(a.z, s, c.z), fmaf(a.w, s, c.w));
}

// ------------------------------------------------------------------------------------------------
// cell forward.  The (B x 2H) x (2H x 3H) product of one token is 0.1 GFLOP, but on a cold chain
// of L2 round trips (~1 us each): the kernel is built to have as few of them as possible.  One
// warp per hidden unit: its six weight rows (r, z, n of W_ih and W_hh), one K chunk of 512 at a
// time, are loaded into REGISTERS up front (24 independent 16-byte loads per lane, one round
// trip) while the CTA stages the 8 batch rows of ix = emb[tok] + sx and of hx in shared memory;
// the products then run from registers and shared memory only.
// ------------------------------------------------------------------------------------------------
static constexpr int CELL_KC = 512;      // K chunk of the forward cell (weights in registers)
static constexpr int CELL_KCB = 768;     // K chunk of the backward cell

struct CellFwdParams {
  const float* emb;       // [Vocab][H]
  const int* tok;         // token of row b at tok[b * tok_stride]
  int tok_stride;
  const float* sx_prev;   // [B][H] or null (first step)
  const float* hx_prev;   // [B][H]
  const float* w_ih;      // [3H][H]
  const float* w_hh;      // [3H][H]
  const float* b_ih;      // [3H]
  const float* b_hh;      // [3H]
  float* hx;              // [B][H]
  float* ix_save;         // [B][H] or null
  float* gates_save;      // [B][4][H] (r, z, n, hn) or null
  const int* done;        // device flag: != 0 -> the decode has finished, do nothing (or null)
  int B, H;
};

__global__ void __launch_bounds__(32 * CELL_WARPS) s2s_cell_fwd_kernel(const CellFwdParams p) {
  extern __shared__ float4 cell_smem[];
  if (p.done && *p.done) return;
  const int H = p.H, B = p.B;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int j = min(blockIdx.x * CELL_WARPS + warp, H - 1);   // (clamped: every warp takes part in the barriers)
  const bool owner = blockIdx.x * CELL_WARPS + warp < H;
  const int b0 = blockIdx.y * CELL_NB;
  const int nb = min(CELL_NB, B - b0);
  float4* xs = cell_smem;                                // [NB][KC/4] ix chunk
  float4* hs = cell_smem + CELL_NB * (CELL_KC / 4);      // [NB][KC/4] hx_prev chunk
  float acc[CELL_NB][6];
#pragma unroll
  for (int b = 0; b < CELL_NB; ++b)
#pragma unroll
    for (int d = 0; d < 6; ++d) acc[b][d] = 0.f;
  const long long gstr = (long long)H * H / 4;          // float4s between the gates' rows
  for (int kc0 = 0; kc0 < H; kc0 += CELL_KC) {
    const int nk4 = min(CELL_KC, H - kc0) / 4;
    const float4* wi = reinterpret_cast<const float4*>(p.w_ih + (long long)j * H + kc0);
    const float4* wh = reinterpret_cast<const float4*>(p.w_hh + (long long)j * H + kc0);
    float4 w[6][CELL_KC / 128];
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
      for (int i = 0; i < CELL_KC / 128; ++i) {
        const int idx = lane + 32 * i;
        w[g][i] = idx < nk4 ? __ldg(wi + g * gstr + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
        w[3 + g][i] = idx < nk4 ? __ldg(wh + g * gstr + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    __syncthreads();                                     // the previous chunk has been consumed
    for (int e = tid; e < CELL_NB * nk4; e += 32 * CELL_WARPS) {
      const int r = e / nk4, c4 = e - r * nk4;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f), h = x;
      if (r < nb) {
        const long long ro = (long long)(b0 + r) * H + kc0;
        const long long tk = p.tok[(long long)(b0 + r) * p.tok_stride];
        x = __ldg(reinterpret_cast<const float4*>(p.emb + tk * H + kc0) + c4);
        if (p.sx_prev) {
          const float4 sv = __ldg(reinterpret_cast<const float4*>(p.sx_prev + ro) + c4);
          x.x += sv.x; x.y += sv.y; x.z += sv.z; x.w += sv.w;
        }
        h = __ldg(reinterpret_cast<const float4*>(p.hx_prev + ro) + c4);
        if (p.ix_save && blockIdx.x == 0) reinterpret_cast<float4*>(p.ix_save + ro)[c4] = x;
      }
      xs[r * (CELL_KC / 4) + c4] = x;
      hs[r * (CELL_KC / 4) + c4] = h;
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < CELL_NB; ++b) {
      if (b < nb) {
#pragma unroll
        for (int i = 0; i < CELL_KC / 128; ++i) {
          const int idx = lane + 32 * i;
          if (idx < nk4) {
            const float4 x = xs[b * (CELL_KC / 4) + idx], h = hs[b * (CELL_KC / 4) + idx];
#pragma unroll
            for (int g = 0; g < 3; ++g) {
              acc[b][g] += dot4(w[g][i], x);
              acc[b][3 + g] += dot4(w[3 + g][i], h);
            }
          }
        }
      }
    }
  }
  float mine[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int b = 0; b < CELL_NB; ++b) {
    if (b < nb) {
#pragma unroll
      for (int d = 0; d < 6; ++d) {
        const float v = warp_sum(acc[b][d]);
        if (lane == b) mine[d] = v;
      }
    }
  }
  if (owner && lane < nb) {
    const int b = b0 + lane;
    const float gir = mine[0] + p.b_ih[j], giz = mine[1] + p.b_ih[H + j], gin = mine[2] + p.b_ih[2 * H + j];
    const float ghr = mine[3] + p.b_hh[j], ghz = mine[4] + p.b_hh[H + j], ghn = mine[5] + p.b_hh[2 * H + j];
    const float r = 1.f / (1.f + expf(-(gir + ghr)));
    const float z = 1.f / (1.f + expf(-(giz + ghz)));
    const float n = tanhf(gin + r * ghn);
    const float hp = p.hx_prev[(long long)b * H + j];
    p.hx[(long long)b * H + j] = (1.f - z) * n + z * hp;
    if (p.gates_save) {
      float* g = p.gates_save + (long long)b * 4 * H + j;
      g[0] = r; g[H] = z; g[2 * H] = n; g[3 * H] = ghn;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// attention + output projection forward.
//
// Grid (ceil(T/24), B): a CTA owns 24 consecutive frames of one utterance, a warp 3 of them.  The
// warp keeps the 3+14 alignment values its location-conv window needs in registers, walks over
// h with lanes (coalesced reads of eh, of the TRANSPOSED conv weights [Kc][H] and of the
// query), and produces 3 scores; an online-softmax partial (max, sum, weighted eh sum) per warp
// is combined per CTA and written to the workspace.  The LAST CTA of the utterance to finish (a
// ticket counter) combines the partials in a fixed order - bit-reproducible - normalises the
// alignment, and runs the output projection / arg-max / log-softmax of the step.
// ------------------------------------------------------------------------------------------------
struct AttnWs {
  float* score;        // [B][T]
  float* m;            // [B][TS]
  float* l;            // [B][TS]
  float* acc;          // [B][TS][H]
  float* aux;          // [B][TS][H]   (backward: second per-CTA partial)
  float* s;            // [B][TS]      (backward: per-CTA scalars)
  float* s2;           // [B][TS]
  unsigned int* cnt;   // [B] tickets, zero between launches
};

static size_t attn_ws_bytes(int B, int T, int H) {
  const size_t TS = (size_t)(T + ATT_TT - 1) / ATT_TT;
  return sizeof(float) * ((size_t)B * T + 4 * (size_t)B * TS + 2 * (size_t)B * TS * H) +
         sizeof(unsigned int) * (size_t)B + 64;
}
static AttnWs attn_ws_carve(void* ws, int B, int T, int H) {
  const size_t TS = (size_t)(T + ATT_TT - 1) / ATT_TT;
  AttnWs w;
  w.cnt = reinterpret_cast<unsigned int*>(ws);           // first: the caller zeroes B words once
  float* f = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + (((size_t)B * 4 + 63) & ~(size_t)63));
  w.score = f; f += (size_t)B * T;
  w.m = f; f += (size_t)B * TS;
  w.l = f; f += (size_t)B * TS;
  w.s = f; f += (size_t)B * TS;
  w.s2 = f; f += (size_t)B * TS;
  w.acc = f; f += (size_t)B * TS * H;
  w.aux = f;
  return w;
}

struct AttnFwdParams {
  const float* eh;        // (B / eh_group, T, H) encoder states
  int eh_group;           // row b attends over utterance b / eh_group (1: its own; K: K beam rows each)
  const float* hx;        // (B, H) decoder state of this step
  const float* ax_prev;   // (B, T) or null
  const float* conv_wT;   // (Kc, H)  transposed location-conv weights
  const float* conv_b;    // (H)
  const float* lin_w;     // (H)
  float lin_b;
  float* sx;              // (B, H)
  float* ax;              // (B, T)
  // output projection (optional): logits[b*logit_stride + c] = fc_b[c] + fc_w[c,:] . (hx + sx)
  const float* fc_w;      // (C, H) or null
  const float* fc_b;      // (C)
  float* logits;
  long long logit_stride;
  float* logp;            // (B, C) log-softmax of the logits or null
  int* argmax;            // (B) arg-max class (first maximum) or null
  int* history;           // greedy decode: history[b * hist_stride + hist_col] = arg-max (or null)
  int hist_stride, hist_col;
  int* end_count;         // += 1 when this row's arg-max == end_tok (or null)
  int end_tok;
  const int* done;        // device flag: != 0 -> do nothing
  const int* lens;        // (B) frames each row attends over, or null (all T)
  AttnWs ws;
  int B, T, H, Kc, C, log_t;
};

// Frames row b attends over: lens[b] clamped to [1, T], or T.  Frames >= this are left out of the
// softmax (a_t = 0) and of the location conv's input, log_t scales by its log, and CTAs whose
// frame tile lies wholly past it do nothing (they also stay out of the ticket count).
SB_DEVINL int attn_frames(const int* lens, int b, int T) {
  return lens ? min(max(__ldg(lens + b), 1), T) : T;
}

// the warp's alignment window: a[i] = ax_prev[tw + i - pad] (zero outside [0, T))
SB_DEVINL void load_window(const float* ax_prev_b, int tw, int pad, int T, int Kc,
                           float (&a)[ATT_WIN]) {
#pragma unroll
  for (int i = 0; i < ATT_WIN; ++i) {
    const int tt = tw + i - pad;
    a[i] = (ax_prev_b && i < ATT_FG + Kc - 1 && tt >= 0 && tt < T) ? __ldg(ax_prev_b + tt) : 0.f;
  }
}

__global__ void __launch_bounds__(ATT_THREADS) s2s_attn_fwd_kernel(const AttnFwdParams p) {
  extern __shared__ float att_smem[];
  __shared__ int s_last;
  if (p.done && *p.done) return;
  const int b = blockIdx.y, ts = blockIdx.x, TS = gridDim.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = p.T, H = p.H, Kc = p.Kc, pad = (Kc - 1) / 2;
  const int Tb = attn_frames(p.lens, b, T), TSb = (Tb + ATT_TT - 1) / ATT_TT;
  if (ts >= TSb) return;
  float* wacc = att_smem;                      // [NW][H] per-warp weighted sums; later o, logits
  float* wst = wacc + ATT_NW * H;              // [NW][2] per-warp (max, sum)
  float* sct = wst + 2 * ATT_NW;               // [TS] scale of each CTA partial (final combine)
  const bool has_prev = p.ax_prev != nullptr;
  const float tscale = p.log_t ? logf((float)Tb) : 1.0f;
  const float* eh = p.eh + (size_t)(b / p.eh_group) * T * H;
  const int tw = ts * ATT_TT + warp * ATT_FG;
  const int nf = max(0, min(ATT_FG, Tb - tw));

  float a[ATT_WIN];
  load_window(has_prev ? p.ax_prev + (size_t)b * T : nullptr, tw, pad, Tb, Kc, a);
  // lanes over h in groups of four (16-byte loads): the h loop is a chain of L2 round trips, so it
  // has to be short - H/128 iterations
  const int H4 = H >> 2;
  const float4* eh4 = reinterpret_cast<const float4*>(eh);
  float part[ATT_FG];
#pragma unroll
  for (int f = 0; f < ATT_FG; ++f) part[f] = 0.f;
  if (nf > 0) {
    for (int h4 = lane; h4 < H4; h4 += 32) {
      float4 dch = reinterpret_cast<const float4*>(p.hx + (size_t)b * H)[h4];
      if (has_prev) dch = add4(dch, __ldg(reinterpret_cast<const float4*>(p.conv_b) + h4));
      const float4 lwh = __ldg(reinterpret_cast<const float4*>(p.lin_w) + h4);
      float4 c[ATT_KMAX];
#pragma unroll
      for (int k = 0; k < ATT_KMAX; ++k)
        c[k] = (has_prev && k < Kc) ? __ldg(reinterpret_cast<const float4*>(p.conv_wT) + (size_t)k * H4 + h4)
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 e[ATT_FG];
#pragma unroll
      for (int f = 0; f < ATT_FG; ++f)
        e[f] = f < nf ? __ldg(eh4 + (size_t)(tw + f) * H4 + h4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int f = 0; f < ATT_FG; ++f) {
        if (f < nf) {
          float4 v = add4(e[f], dch);
          if (has_prev) {
            float4 sacc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < ATT_KMAX; ++k) sacc = fma4(c[k], a[f + k], sacc);
            v = add4(v, sacc);
          }
          part[f] += lwh.x * fmaxf(v.x, 0.f) + lwh.y * fmaxf(v.y, 0.f) + lwh.z * fmaxf(v.z, 0.f) +
                     lwh.w * fmaxf(v.w, 0.f);
        }
      }
    }
  }
  float sc[ATT_FG], m_w = -INFINITY;
#pragma unroll
  for (int f = 0; f < ATT_FG; ++f) {
    sc[f] = -INFINITY;
    if (f < nf) {
      sc[f] = (warp_sum(part[f]) + p.lin_b) * tscale;
      m_w = fmaxf(m_w, sc[f]);
      if (lane == 0) p.ws.score[(size_t)b * T + tw + f] = sc[f];
    }
  }
  float w[ATT_FG], l_w = 0.f;
#pragma unroll
  for (int f = 0; f < ATT_FG; ++f) {
    w[f] = f < nf ? __expf(sc[f] - m_w) : 0.f;
    l_w += w[f];
  }
  for (int h4 = lane; h4 < H4; h4 += 32) {
    float4 sacc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int f = 0; f < ATT_FG; ++f)
      if (f < nf) sacc = fma4(__ldg(eh4 + (size_t)(tw + f) * H4 + h4), w[f], sacc);
    reinterpret_cast<float4*>(wacc + warp * H)[h4] = sacc;
  }
  if (lane == 0) { wst[warp * 2] = m_w; wst[warp * 2 + 1] = l_w; }
  __syncthreads();
  // ---- CTA partial ----
  float m_c = -INFINITY;
#pragma unroll
  for (int q = 0; q < ATT_NW; ++q) m_c = fmaxf(m_c, wst[q * 2]);
  float scl[ATT_NW], l_c = 0.f;
#pragma unroll
  for (int q = 0; q < ATT_NW; ++q) {
    scl[q] = wst[q * 2] == -INFINITY ? 0.f : __expf(wst[q * 2] - m_c);
    l_c += wst[q * 2 + 1] * scl[q];
  }
  const size_t slot = (size_t)b * TS + ts;
  for (int h = tid; h < H; h += ATT_THREADS) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < ATT_NW; ++q) s += wacc[q * H + h] * scl[q];
    p.ws.acc[slot * H + h] = s;
  }
  if (tid == 0) { p.ws.m[slot] = m_c; p.ws.l[slot] = l_c; }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(p.ws.cnt + b, 1u) == (unsigned int)(TSb - 1));
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- the utterance's last CTA: combine the TSb partials in index order ----
  float m = -INFINITY;
  for (int q = 0; q < TSb; ++q) m = fmaxf(m, __ldcg(p.ws.m + (size_t)b * TS + q));
  for (int q = tid; q < TSb; q += ATT_THREADS) sct[q] = __expf(__ldcg(p.ws.m + (size_t)b * TS + q) - m);
  __syncthreads();
  float l = 0.f;
  for (int q = 0; q < TSb; ++q) l += __ldcg(p.ws.l + (size_t)b * TS + q) * sct[q];
  const float inv = 1.0f / l;
  float* o = wacc;                 // [H]   hx + sx
  float* lg = wacc + H;            // [C]
  for (int h = tid; h < H; h += ATT_THREADS) {
    float s = 0.f;
    for (int q = 0; q < TSb; ++q) s += __ldcg(p.ws.acc + ((size_t)b * TS + q) * H + h) * sct[q];
    s *= inv;
    p.sx[(size_t)b * H + h] = s;
    o[h] = p.hx[(size_t)b * H + h] + s;
  }
  for (int t = tid; t < T; t += ATT_THREADS)
    p.ax[(size_t)b * T + t] = t < Tb ? __expf(__ldcg(p.ws.score + (size_t)b * T + t) - m) * inv : 0.f;
  if (tid == 0) p.ws.cnt[b] = 0u;
  if (!p.fc_w) return;
  // ---- output projection on o = hx + sx (seq2seq.py:108,131-132) ----
  __syncthreads();
  for (int c = warp; c < p.C; c += ATT_NW) {
    const float* wr = p.fc_w + (size_t)c * H;
    float s = 0.f;
    for (int h = lane; h < H; h += 32) s += __ldg(wr + h) * o[h];
    s = warp_sum(s);
    if (lane == 0) {
      s += p.fc_b[c];
      lg[c] = s;
      if (p.logits) p.logits[(size_t)b * p.logit_stride + c] = s;
    }
  }
  __syncthreads();
  if (warp == 0 && (p.logp || p.argmax || p.history || p.end_count)) {
    float mx = -INFINITY;
    int am = 0x7fffffff;
    for (int c = lane; c < p.C; c += 32)
      if (lg[c] > mx) { mx = lg[c]; am = c; }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, off);
      const int oa = __shfl_xor_sync(0xffffffffu, am, off);
      if (om > mx || (om == mx && oa < am)) { mx = om; am = oa; }
    }
    if (p.logp) {
      float se = 0.f;
      for (int c = lane; c < p.C; c += 32) se += expf(lg[c] - mx);
      se = warp_sum(se);
      const float lse = mx + logf(se);
      for (int c = lane; c < p.C; c += 32) p.logp[(size_t)b * p.C + c] = lg[c] - lse;
    }
    if (lane == 0) {
      if (p.argmax) p.argmax[b] = am;
      if (p.history) p.history[(size_t)b * p.hist_stride + p.hist_col] = am;
      if (p.end_count && am == p.end_tok) atomicAdd(p.end_count, 1);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward of the output projection for ALL steps at once (no dependence on the recurrence):
//   d_o[r, :] = dlogits[r, :] W_fc,   o[r, :] = hx[r, :] + sx[r, :]      r = (step, utterance)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) s2s_dout_kernel(const float* __restrict__ dl,
                                                       const float* __restrict__ fc_w,
                                                       const float* __restrict__ hx,
                                                       const float* __restrict__ sx,
                                                       float* __restrict__ d_o,
                                                       float* __restrict__ o_all, int C, int H) {
  extern __shared__ float dl_s[];
  const size_t r = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += 256) dl_s[c] = dl[r * C + c];
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += 256) {
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += dl_s[c] * __ldg(fc_w + (size_t)c * H + h);
    d_o[r * H + h] = s;
    o_all[r * H + h] = hx[r * H + h] + sx[r * H + h];
  }
}

// ------------------------------------------------------------------------------------------------
// attention backward of one step, same (frames, utterance) grid as the forward, two kernels
// (the softmax Jacobian needs S = sum_t a_t da_t over ALL frames before anything else):
//   A  da_t = eh_t . d sx + d ax_next[t]; per-CTA partial of S; zeroes d ax_prev
//   B  d score_t = tscale a_t (da_t - S), back through linear / ReLU / location conv:
//      d eh += a_t d sx + d pre_t (in place), d ax_prev (window sums; neighbouring CTAs overlap in
//      at most two contributions per element, so the atomic adds are order-independent), per-CTA
//      partials of the conv-weight gradient (accumulated over the steps in the CTA's own slot),
//      of d lin_w and of sum_t d pre_t; the utterance's last CTA (ticket) adds the partials in
//      index order and emits the gate pre-activation gradients of the cell.
// ------------------------------------------------------------------------------------------------
struct AttnBwdParams {
  const float* eh;         // (B, T, H)
  const float* hx;         // (B, H) decoder state of this step
  const float* hx_prev;    // (B, H)
  const float* ax_prev;    // (B, T) or null (first step)
  const float* ax;         // (B, T) this step's alignment (saved by forward)
  const float* conv_wT;    // (Kc, H)
  const float* conv_b; const float* lin_w;
  const float* d_o;        // (B, H) gradient w.r.t. o = hx + sx of this step (s2s_dout_kernel)
  const float* d_ix_next;  // (B, H) gradient w.r.t. the NEXT step's ix (= d sx through ix = emb + sx); null at the last step
  const float* d_ax_next;  // (B, T) gradient w.r.t. ax from the next step's conv; null at the last step
  const float* d_hx_next;  // (B, H) gradient w.r.t. hx from the next step's cell; null at the last step
  const float* gates;      // (B, 4, H) r, z, n, hn saved by the cell
  float* d_eh;             // (B, T, H) +=
  float* d_ax_prev;        // (B, T) out (gradient w.r.t. the previous alignment), unused at the first step
  float* d_gi;             // (B, 3H) out: gate pre-activation gradients of the cell (input side)
  float* d_gh;             // (B, 3H) out: (hidden side: the n entry carries r)
  float* d_hx_direct;      // (B, H) out: z * d hx (direct path to hx_prev)
  // parameter gradients accumulated over the steps, reduced over their leading dims by the caller
  float* g_conv_wT;        // (B, TS, Kc, H) +=
  float* g_conv_b;         // (B, H) +=
  float* g_lin_w;          // (B, H) +=
  float* g_lin_b;          // (B) +=
  const int* lens;         // (B) frames of each utterance, or null (all T)
  AttnWs ws;
  int B, T, H, Kc, log_t;
};

__global__ void __launch_bounds__(ATT_THREADS) s2s_attn_bwd_a_kernel(const AttnBwdParams p) {
  extern __shared__ float bwa_smem[];
  const int b = blockIdx.y, ts = blockIdx.x, TS = gridDim.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = p.T, H = p.H;
  const int Tb = attn_frames(p.lens, b, T);
  if (ts * ATT_TT >= Tb) return;
  float* dsx = bwa_smem;             // [H]
  float* red = dsx + H;              // [NW]
  for (int h = tid; h < H; h += ATT_THREADS)
    dsx[h] = p.d_o[(size_t)b * H + h] + (p.d_ix_next ? p.d_ix_next[(size_t)b * H + h] : 0.f);
  __syncthreads();
  const float* eh = p.eh + (size_t)b * T * H;
  const int tw = ts * ATT_TT + warp * ATT_FG;
  const int nf = max(0, min(ATT_FG, Tb - tw));
  float part[ATT_FG];
#pragma unroll
  for (int f = 0; f < ATT_FG; ++f) part[f] = 0.f;
  const int H4 = H >> 2;
  const float4* eh4 = reinterpret_cast<const float4*>(eh);
  for (int h4 = lane; h4 < H4; h4 += 32) {
    const float4 d = reinterpret_cast<const float4*>(dsx)[h4];
#pragma unroll
    for (int f = 0; f < ATT_FG; ++f)
      if (f < nf) part[f] += dot4(__ldg(eh4 + (size_t)(tw + f) * H4 + h4), d);
  }
  float spart = 0.f;
#pragma unroll
  for (int f = 0; f < ATT_FG; ++f) {
    if (f < nf) {
      const size_t ix = (size_t)b * T + tw + f;
      const float da = warp_sum(part[f]) + (p.d_ax_next ? p.d_ax_next[ix] : 0.f);
      spart += p.ax[ix] * da;
      if (lane == 0) {
        p.ws.score[ix] = da;
        if (p.ax_prev) p.d_ax_prev[ix] = 0.f;
      }
    }
  }
  if (lane == 0) red[warp] = spart;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < ATT_NW; ++q) s += red[q];
    p.ws.s[(size_t)b * TS + ts] = s;
  }
}

__global__ void __launch_bounds__(ATT_THREADS) s2s_attn_bwd_b_kernel(const AttnBwdParams p) {
  extern __shared__ float bwb_smem[];
  __shared__ int s_last;
  const int b = blockIdx.y, ts = blockIdx.x, TS = gridDim.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = p.T, H = p.H, Kc = p.Kc, pad = (Kc - 1) / 2;
  const int Tb = attn_frames(p.lens, b, T), TSb = (Tb + ATT_TT - 1) / ATT_TT;
  if (ts >= TSb) return;
  float* dsx = bwb_smem;                         // [H]
  float* dpre_s = dsx + H;                       // [TT][H]  d pre of the CTA's frames
  float* glw_w = dpre_s + ATT_TT * H;            // [NW][H]  per-warp d lin_w
  float* win_s = glw_w + ATT_NW * H;             // [NW][WIN] per-warp d alignment windows
  float* axc = win_s + ATT_NW * ATT_WIN;         // [TT + KMAX - 1] the CTA's alignment window
  float* red = axc + ATT_TT + ATT_KMAX - 1;      // [NW]
  const bool has_prev = p.ax_prev != nullptr;
  const float tscale = p.log_t ? logf((float)Tb) : 1.0f;
  const float* eh = p.eh + (size_t)b * T * H;
  float* deh = p.d_eh + (size_t)b * T * H;
  const int t0 = ts * ATT_TT;
  const int tw = t0 + warp * ATT_FG;
  const int nf = max(0, min(ATT_FG, Tb - tw));
  for (int h = tid; h < H; h += ATT_THREADS)
    dsx[h] = p.d_o[(size_t)b * H + h] + (p.d_ix_next ? p.d_ix_next[(size_t)b * H + h] : 0.f);
  for (int j = tid; j < ATT_TT + ATT_KMAX - 1; j += ATT_THREADS) {
    const int tt = t0 - pad + j;
    axc[j] = (has_prev && tt >= 0 && tt < Tb) ? p.ax_prev[(size_t)b * T + tt] : 0.f;
  }
  float S = 0.f;
  for (int q = 0; q < TSb; ++q) S += p.ws.s[(size_t)b * TS + q];
  __syncthreads();
  // ---- (i) warp per frame group ----
  float ds[ATT_FG], at[ATT_FG];
  float glb = 0.f;
#pragma unroll
  for (int f = 0; f < ATT_FG; ++f) {
    ds[f] = 0.f; at[f] = 0.f;
    if (f < nf) {
      const size_t ix = (size_t)b * T + tw + f;
      at[f] = p.ax[ix];
      ds[f] = tscale * at[f] * (p.ws.score[ix] - S);
      glb += ds[f];
    }
  }
  float a[ATT_WIN];
  load_window(has_prev ? p.ax_prev + (size_t)b * T : nullptr, tw, pad, Tb, Kc, a);
  float dwin[ATT_WIN];
#pragma unroll
  for (int i = 0; i < ATT_WIN; ++i) dwin[i] = 0.f;
  const int H4 = H >> 2;
  const float4* eh4 = reinterpret_cast<const float4*>(eh);
  float4* deh4 = reinterpret_cast<float4*>(deh);
  for (int h4 = lane; h4 < H4; h4 += 32) {
    float4 dch = reinterpret_cast<const float4*>(p.hx + (size_t)b * H)[h4];
    if (has_prev) dch = add4(dch, __ldg(reinterpret_cast<const float4*>(p.conv_b) + h4));
    const float4 lwh = __ldg(reinterpret_cast<const float4*>(p.lin_w) + h4);
    const float4 dsxh = reinterpret_cast<const float4*>(dsx)[h4];
    float4 c[ATT_KMAX];
#pragma unroll
    for (int k = 0; k < ATT_KMAX; ++k)
      c[k] = (has_prev && k < Kc) ? __ldg(reinterpret_cast<const float4*>(p.conv_wT) + (size_t)k * H4 + h4)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 e[ATT_FG], dold[ATT_FG];
#pragma unroll
    for (int f = 0; f < ATT_FG; ++f) {
      e[f] = dold[f] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < nf) {
        e[f] = __ldg(eh4 + (size_t)(tw + f) * H4 + h4);
        dold[f] = deh4[(size_t)(tw + f) * H4 + h4];
      }
    }
    float4 glw = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int f = 0; f < ATT_FG; ++f) {
      float4 dpre = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < nf) {
        float4 v = add4(e[f], dch);
        if (has_prev) {
          float4 sacc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int k = 0; k < ATT_KMAX; ++k) sacc = fma4(c[k], a[f + k], sacc);
          v = add4(v, sacc);
        }
        dpre.x = v.x > 0.f ? ds[f] * lwh.x : 0.f;
        dpre.y = v.y > 0.f ? ds[f] * lwh.y : 0.f;
        dpre.z = v.z > 0.f ? ds[f] * lwh.z : 0.f;
        dpre.w = v.w > 0.f ? ds[f] * lwh.w : 0.f;
        glw.x += ds[f] * fmaxf(v.x, 0.f); glw.y += ds[f] * fmaxf(v.y, 0.f);
        glw.z += ds[f] * fmaxf(v.z, 0.f); glw.w += ds[f] * fmaxf(v.w, 0.f);
        deh4[(size_t)(tw + f) * H4 + h4] = add4(dold[f], fma4(dsxh, at[f], dpre));
        if (has_prev) {
#pragma unroll
          for (int k = 0; k < ATT_KMAX; ++k) dwin[f + k] += dot4(dpre, c[k]);
        }
      }
      reinterpret_cast<float4*>(dpre_s + (warp * ATT_FG + f) * H)[h4] = dpre;
    }
    reinterpret_cast<float4*>(glw_w + warp * H)[h4] = glw;
  }
  if (has_prev) {
#pragma unroll
    for (int i = 0; i < ATT_WIN; ++i) {
      const float s = warp_sum(dwin[i]);
      if (lane == 0) win_s[warp * ATT_WIN + i] = s;
    }
  }
  if (lane == 0) red[warp] = glb;
  __syncthreads();
  // ---- (ii) d ax_prev of the CTA's window: the warps' windows added in warp order ----
  if (has_prev) {
    for (int j = tid; j < ATT_TT + Kc - 1; j += ATT_THREADS) {
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < ATT_NW; ++q) {
        const int i = j - q * ATT_FG;
        if (i >= 0 && i < ATT_FG + Kc - 1) s += win_s[q * ATT_WIN + i];
      }
      const int tt = t0 - pad + j;
      if (tt >= 0 && tt < Tb) atomicAdd(p.d_ax_prev + (size_t)b * T + tt, s);
    }
  }
  // ---- (iii) thread per h over the CTA's frames: partial sums, conv weight gradient ----
  const size_t slot = (size_t)b * TS + ts;
  for (int h = tid; h < H; h += ATT_THREADS) {
    float gdh = 0.f, glw = 0.f;
#pragma unroll
    for (int q = 0; q < ATT_NW; ++q) glw += glw_w[q * H + h];
    float g[ATT_KMAX];
#pragma unroll
    for (int k = 0; k < ATT_KMAX; ++k) g[k] = 0.f;
#pragma unroll 1
    for (int q = 0; q < ATT_NW; ++q) {
      float aw[ATT_WIN];
#pragma unroll
      for (int i = 0; i < ATT_WIN; ++i) aw[i] = axc[q * ATT_FG + i < ATT_TT + ATT_KMAX - 1 ? q * ATT_FG + i : 0];
#pragma unroll
      for (int f = 0; f < ATT_FG; ++f) {
        const float d = dpre_s[(q * ATT_FG + f) * H + h];
        gdh += d;
#pragma unroll
        for (int k = 0; k < ATT_KMAX; ++k) g[k] += d * aw[f + k];
      }
    }
    p.ws.acc[slot * H + h] = gdh;
    p.ws.aux[slot * H + h] = glw;
    if (has_prev) {
      float* gw = p.g_conv_wT + slot * (size_t)Kc * H + h;
#pragma unroll
      for (int k = 0; k < ATT_KMAX; ++k)
        if (k < Kc) gw[(size_t)k * H] += g[k];
    }
  }
  if (tid == 0) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < ATT_NW; ++q) s += red[q];
    p.ws.s2[slot] = s;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(p.ws.cnt + b, 1u) == (unsigned int)(TSb - 1));
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- the utterance's last CTA: totals in index order, gate gradients of the cell ----
  if (tid == 0) {
    float s = 0.f;
    for (int q = 0; q < TSb; ++q) s += __ldcg(p.ws.s2 + (size_t)b * TS + q);
    p.g_lin_b[b] += s;
    p.ws.cnt[b] = 0u;
  }
  const float* gt = p.gates + (size_t)b * 4 * H;
  for (int h = tid; h < H; h += ATT_THREADS) {
    float gdh = 0.f, glw = 0.f;
    for (int q = 0; q < TSb; ++q) {
      gdh += __ldcg(p.ws.acc + ((size_t)b * TS + q) * H + h);
      glw += __ldcg(p.ws.aux + ((size_t)b * TS + q) * H + h);
    }
    p.g_lin_w[(size_t)b * H + h] += glw;
    if (has_prev) p.g_conv_b[(size_t)b * H + h] += gdh;
    // total gradient w.r.t. hx_u: output projection + attention query + next step's cell
    const float dh = p.d_o[(size_t)b * H + h] + gdh +
                     (p.d_hx_next ? p.d_hx_next[(size_t)b * H + h] : 0.f);
    const float r = gt[h], z = gt[H + h], n = gt[2 * H + h], hn = gt[3 * H + h];
    const float hp = p.hx_prev[(size_t)b * H + h];
    const float dn = dh * (1.f - z) * (1.f - n * n);
    const float dz = dh * (hp - n) * z * (1.f - z);
    const float dr = dn * hn * r * (1.f - r);
    float* gi = p.d_gi + (size_t)b * 3 * H;
    float* gh = p.d_gh + (size_t)b * 3 * H;
    gi[h] = dr; gi[H + h] = dz; gi[2 * H + h] = dn;
    gh[h] = dr; gh[H + h] = dz; gh[2 * H + h] = dn * r;
    p.d_hx_direct[(size_t)b * H + h] = dh * z;
  }
}

// ------------------------------------------------------------------------------------------------
// cell backward: d ix = d gi W_ih ; d hx_prev = d gh W_hh + d_hx_direct.  Same structure as the
// forward on TRANSPOSED weights (W^T [H][3H], made once per backward by the caller): one warp per
// two output columns, their four weight rows of one 768-wide K chunk in registers, the 8 batch
// rows of d gi / d gh staged in shared memory.
// ------------------------------------------------------------------------------------------------
struct CellBwdParams {
  const float* d_gi;        // (B, 3H)
  const float* d_gh;        // (B, 3H)
  const float* d_hx_direct; // (B, H)
  const float* w_ihT;       // [H][3H]
  const float* w_hhT;       // [H][3H]
  float* d_ix;              // (B, H) out
  float* d_hx_prev;         // (B, H) out
  int B, H;
};

__global__ void __launch_bounds__(32 * CELL_WARPS) s2s_cell_bwd_kernel(const CellBwdParams p) {
  extern __shared__ float4 cell_smem[];
  const int H = p.H, B = p.B, N3 = 3 * H;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int kraw = (blockIdx.x * CELL_WARPS + warp) * 2;  // this warp's two output columns
  const bool owner = kraw < H;
  const int k0 = owner ? kraw : 0;
  const bool two = k0 + 1 < H;
  const int b0 = blockIdx.y * CELL_NB;
  const int nb = min(CELL_NB, B - b0);
  float4* gis = cell_smem;                                 // [NB][KCB/4] d gi chunk
  float4* ghs = cell_smem + CELL_NB * (CELL_KCB / 4);      // [NB][KCB/4] d gh chunk
  float acc[CELL_NB][4];
#pragma unroll
  for (int b = 0; b < CELL_NB; ++b)
#pragma unroll
    for (int d = 0; d < 4; ++d) acc[b][d] = 0.f;
  const int row4 = N3 / 4;
  for (int n0 = 0; n0 < N3; n0 += CELL_KCB) {
    const int nk4 = min(CELL_KCB, N3 - n0) / 4;
    const float4* wi = reinterpret_cast<const float4*>(p.w_ihT + (long long)k0 * N3 + n0);
    const float4* wh = reinterpret_cast<const float4*>(p.w_hhT + (long long)k0 * N3 + n0);
    float4 w[4][CELL_KCB / 128];
#pragma unroll
    for (int i = 0; i < CELL_KCB / 128; ++i) {
      const int idx = lane + 32 * i;
      const bool ok = idx < nk4;
      const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
      w[0][i] = ok ? __ldg(wi + idx) : zero;
      w[1][i] = ok ? __ldg(wh + idx) : zero;
      w[2][i] = ok && two ? __ldg(wi + row4 + idx) : zero;
      w[3][i] = ok && two ? __ldg(wh + row4 + idx) : zero;
    }
    __syncthreads();
    for (int e = tid; e < CELL_NB * nk4; e += 32 * CELL_WARPS) {
      const int r = e / nk4, c4 = e - r * nk4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), c = a;
      if (r < nb) {
        a = __ldg(reinterpret_cast<const float4*>(p.d_gi + (long long)(b0 + r) * N3 + n0) + c4);
        c = __ldg(reinterpret_cast<const float4*>(p.d_gh + (long long)(b0 + r) * N3 + n0) + c4);
      }
      gis[r * (CELL_KCB / 4) + c4] = a;
      ghs[r * (CELL_KCB / 4) + c4] = c;
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < CELL_NB; ++b) {
      if (b < nb) {
#pragma unroll
        for (int i = 0; i < CELL_KCB / 128; ++i) {
          const int idx = lane + 32 * i;
          if (idx < nk4) {
            const float4 gi = gis[b * (CELL_KCB / 4) + idx], gh = ghs[b * (CELL_KCB / 4) + idx];
            acc[b][0] += dot4(w[0][i], gi); acc[b][1] += dot4(w[1][i], gh);
            acc[b][2] += dot4(w[2][i], gi); acc[b][3] += dot4(w[3][i], gh);
          }
        }
      }
    }
  }
  float mine[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int b = 0; b < CELL_NB; ++b) {
    if (b < nb) {
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        const float v = warp_sum(acc[b][d]);
        if (lane == b) mine[d] = v;
      }
    }
  }
  if (owner && lane < nb) {
    const long long o = (long long)(b0 + lane) * H + k0;
    p.d_ix[o] = mine[0];
    p.d_hx_prev[o] = mine[1] + p.d_hx_direct[o];
    if (two) {
      p.d_ix[o + 1] = mine[2];
      p.d_hx_prev[o + 1] = mine[3] + p.d_hx_direct[o + 1];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Shallow fusion.  The selection is written once over a policy that gives the value of candidate
// (r, c), live row r extended by class c:
//   S2sNoFuse  score_r + logp[r][c] (the LM-less search, its arithmetic untouched);
//   S2sLmFuse  score_r + ((double)logp[r][c] + (alpha * lm(c | h_r) + beta_c)), lm the backoff
//              lookup of SbNgramLm (ngram.cuh), beta_c = beta but 0 for end_tok, whose LM token is
//              </s>; with alpha = beta = 0 this is the LM-less value bit for bit.
// h_r is row r's last order-1 tokens, read from its node up the parent links of the arena; the
// root (the start token) reads as <s>.  Once per step each CTA resolves every live row's context
// nodes into shared memory (resolve), so a candidate's lookup is at most `order` probes.  The
// fused value is the hypothesis score everywhere after: selection, completion, stop rule, result.
//   S2sWordLmFuse  the word LM of SbWordLm: the LM term on the delimiter that ends a non-empty
//              word and on end_tok, an OOV penalty where a word leaves the lexicon.
// The beam state, the bookkeeping, S2sLmFuse and S2sWordLmFuse are in s2s_beam.cuh.
// ------------------------------------------------------------------------------------------------
struct S2sNoFuse {
  static constexpr bool kLm = false;
  SB_DEVINL void resolve(const BeamParams&, const BeamState*, int) const {}
  SB_DEVINL double value(const BeamParams& p, const BeamState* st, int r, int c) const {
    return st->score[r] + (double)p.logp[(size_t)r * p.C + c];
  }
};

// grid B: CTA b selects for utterance b
template <class Fuse>
__global__ void __launch_bounds__(256) s2s_beam_select_kernel(const BeamParams pb, const Fuse fu) {
  extern __shared__ unsigned char bm_smem[];
  const BeamParams p = pb.of(blockIdx.x);
  double* sc = reinterpret_cast<double*>(bm_smem);       // [K * C]
  __shared__ int sel_idx[2 * BM_MAXK];
  __shared__ double sel_sc[2 * BM_MAXK];
  const int tid = threadIdx.x;
  BeamState* st = p.st;
  if (st->done) return;
  const int K = p.K, C = p.C, nl = st->nlive;
  if constexpr (Fuse::kLm) {
    fu.resolve(p, st, nl);
    __syncthreads();
  }
  for (int i = tid; i < K * C; i += 256) {
    const int r = i / C, c = i - r * C;
    sc[i] = r < nl ? fu.value(p, st, r, c) : nan("");
  }
  __syncthreads();
  const int want = min(2 * K, nl * C);
  for (int q = 0; q < want; ++q) {
    double bs;
    const int bi = beam_take_first<256>(sc, K * C, bs);
    if (tid == 0) { sel_idx[q] = bi; sel_sc[q] = bs; }
  }
  if (tid != 0) return;
  beam_bookkeep(p, sel_idx, sel_sc, want, p.C);
}

// ------------------------------------------------------------------------------------------------
// split beam selection, for K*C candidates that do not fit one CTA's shared memory:
//   stage 1 (s2s_beam_tiles): grid (tiles, B), CTA per tile of BM_TILE flat indices i*C + c of the
//           utterance's live rows; each keeps its own top min(2K, n) candidates by (score desc,
//           index asc), in that order.
//   stage 2 (s2s_beam_merge): grid B, a CTA per utterance merges its tiles' sorted lists (a head
//           per tile) into the first min(2K, nl*C) and runs the same bookkeeping.
// The union of the top K and the first K non-ended candidates lies in the global top 2K (at most
// K of the top K end in end_tok), so the 2K per tile lose nothing.  The argument holds for any
// candidate values, so for the fused ones too; with an LM every tile CTA resolves the live rows'
// contexts itself (a few probes per row, next to the tile's 4096 lookups).
// ------------------------------------------------------------------------------------------------
static constexpr int BM_PER_THREAD = 16;
static constexpr int BM_TILE = 256 * BM_PER_THREAD;

// t_sc / t_idx [B][tiles][2K], t_cnt [B][tiles]
template <class Fuse>
__global__ void __launch_bounds__(256) s2s_beam_tiles_kernel(const BeamParams pb, double* t_sc,
                                                             int* t_idx, int* t_cnt,
                                                             const Fuse fu) {
  const BeamParams p = pb.of(blockIdx.y);
  const BeamState* st = p.st;
  if (st->done) return;
  const int tid = threadIdx.x, tile = blockIdx.x, K2 = 2 * p.K, C = p.C;
  const size_t u0 = (size_t)blockIdx.y * gridDim.x;      // the utterance's first tile slot
  t_sc += u0 * K2;
  t_idx += u0 * K2;
  t_cnt += u0;
  const int n = st->nlive * C;
  if constexpr (Fuse::kLm) {
    fu.resolve(p, st, st->nlive);
    __syncthreads();
  }
  double v[BM_PER_THREAD];
#pragma unroll
  for (int j = 0; j < BM_PER_THREAD; ++j) {
    const int i = tile * BM_TILE + j * 256 + tid;
    v[j] = nan("");
    if (i < n) {
      const int r = i / C, c = i - r * C;
      v[j] = fu.value(p, st, r, c);
    }
  }
  int q = 0;
  for (; q < K2; ++q) {
    double bs = 0.0;
    int bi = -1;
#pragma unroll
    for (int j = 0; j < BM_PER_THREAD; ++j)
      beam_scan_step(v[j], tile * BM_TILE + j * 256 + tid, bs, bi);
    beam_block_first<256>(bs, bi);
    if (bi < 0) break;
    if (tid == 0) { t_sc[(size_t)tile * K2 + q] = bs; t_idx[(size_t)tile * K2 + q] = bi; }
#pragma unroll
    for (int j = 0; j < BM_PER_THREAD; ++j)
      if (tile * BM_TILE + j * 256 + tid == bi) v[j] = nan("");
  }
  if (tid == 0) t_cnt[tile] = q;
}

__global__ void __launch_bounds__(256) s2s_beam_merge_kernel(const BeamParams pb,
                                                             const double* t_sc, const int* t_idx,
                                                             const int* t_cnt, int ntiles) {
  extern __shared__ int bmm_head[];                  // [ntiles] next entry of each tile's list
  __shared__ int sel_idx[2 * BM_MAXK];
  __shared__ double sel_sc[2 * BM_MAXK];
  const BeamParams p = pb.of(blockIdx.x);
  BeamState* st = p.st;
  if (st->done) return;
  const int tid = threadIdx.x, K2 = 2 * p.K;
  const size_t u0 = (size_t)blockIdx.x * ntiles;
  t_sc += u0 * K2;
  t_idx += u0 * K2;
  t_cnt += u0;
  const int want = min(K2, st->nlive * p.C);
  for (int t = tid; t < ntiles; t += 256) bmm_head[t] = 0;
  __syncthreads();
  for (int q = 0; q < want; ++q) {
    double bs = 0.0;
    int bi = -1;
    for (int t = tid; t < ntiles; t += 256) {
      const int h = bmm_head[t];
      if (h < t_cnt[t]) {
        const double s = t_sc[(size_t)t * K2 + h];
        const int i = t_idx[(size_t)t * K2 + h];
        if (beam_before(s, i, bs, bi)) { bs = s; bi = i; }
      }
    }
    beam_block_first<256>(bs, bi);
    if (tid == 0) {
      sel_idx[q] = bi;
      sel_sc[q] = bs;
      if (bi >= 0) bmm_head[bi / BM_TILE] += 1;
    }
    __syncthreads();
  }
  if (tid != 0) return;
  beam_bookkeep(p, sel_idx, sel_sc, want, p.C);
}

// rows of the next beam continue rows parent_row[] of the previous one: gather hx / sx / ax.
// Grid B*K: CTA b*K + r fills row r of utterance b from row parent_row[b*K + r] of the same one.
__global__ void __launch_bounds__(256)
s2s_beam_gather_kernel(const float* __restrict__ hx_in, const float* __restrict__ sx_in,
                       const float* __restrict__ ax_in, float* __restrict__ hx_out,
                       float* __restrict__ sx_out, float* __restrict__ ax_out,
                       const int* __restrict__ parent_row, const BeamState* st, int K, int H,
                       int T) {
  const int b = blockIdx.x / K, r = blockIdx.x - b * K;
  if (st[b].done || r >= st[b].nlive) return;
  const size_t dst = blockIdx.x, src = (size_t)b * K + parent_row[dst];
  for (int h = threadIdx.x; h < H; h += 256) {
    hx_out[dst * H + h] = hx_in[src * H + h];
    sx_out[dst * H + h] = sx_in[src * H + h];
  }
  for (int t = threadIdx.x; t < T; t += 256) ax_out[dst * T + t] = ax_in[src * T + t];
}

// grid B: utterance b's state (the root alone), its root node and the token of its first row
__global__ void s2s_beam_init_kernel(BeamState* st, int* nodes, int node_cap, int* tok_next, int K,
                                     int start_tok, int* stop) {
  const int b = blockIdx.x;
  int* w = reinterpret_cast<int*>(st + b);
  for (int i = threadIdx.x; i < (int)(sizeof(BeamState) / sizeof(int)); i += blockDim.x) w[i] = 0;
  __syncthreads();
  if (threadIdx.x != 0) return;
  BeamState* s = st + b;
  s->score[0] = 0.0; s->node[0] = 0; s->token[0] = start_tok; s->nlive = 1; s->nodes_used = 1;
  nodes[(size_t)b * 2 * node_cap] = -1;
  nodes[(size_t)b * 2 * node_cap + 1] = start_tok;
  tok_next[(size_t)b * K] = start_tok;
  if (stop && b == 0) { stop[0] = 0; stop[1] = 0; }
}

// greedy decode: stop when EVERY row emitted end_tok at this step (seq2seq.py:162-178, :155-156)
__global__ void s2s_check_done_kernel(const int* end_count, int B, int* done, int* nsteps, int step1) {
  if (*done) return;
  *nsteps = step1;
  if (*end_count == B) *done = 1;
}

}  // namespace sb

using namespace sb;

extern "C" int sb_s2s_workspace_size(int B, int T, int H, size_t* bytes) {
  if (!bytes || B <= 0 || T <= 0 || H <= 0) return SB_ERR_INVALID;
  *bytes = attn_ws_bytes(B, T, H);
  return SB_OK;
}

extern "C" int sb_s2s_cell_fwd(const float* emb, const int* tok, int tok_stride, const float* sx_prev,
                               const float* hx_prev, const float* w_ih, const float* w_hh,
                               const float* b_ih, const float* b_hh, float* hx, float* ix_save,
                               float* gates_save, const int* done, int B, int H, void* stream_) {
  if (!emb || !tok || !hx_prev || !w_ih || !w_hh || !b_ih || !b_hh || !hx || B <= 0 || H <= 0)
    return SB_ERR_INVALID;
  if (H % 4 != 0) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CellFwdParams p;
  p.emb = emb; p.tok = tok; p.tok_stride = tok_stride; p.sx_prev = sx_prev; p.hx_prev = hx_prev;
  p.w_ih = w_ih; p.w_hh = w_hh; p.b_ih = b_ih; p.b_hh = b_hh; p.hx = hx; p.ix_save = ix_save;
  p.gates_save = gates_save; p.done = done; p.B = B; p.H = H;
  const dim3 grid((H + CELL_WARPS - 1) / CELL_WARPS, (B + CELL_NB - 1) / CELL_NB);
  const size_t smem = (size_t)2 * CELL_NB * CELL_KC * sizeof(float);
  s2s_cell_fwd_kernel<<<grid, 32 * CELL_WARPS, smem, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

static int attn_dims_ok(int B, int T, int H, int Kc) {
  if (B <= 0 || T <= 0 || H <= 0 || Kc <= 0 || (Kc & 1) == 0) return SB_ERR_INVALID;
  if (Kc >= ATT_KMAX || (T + ATT_TT - 1) / ATT_TT > ATT_MAX_TS || B > 65535)
    return SB_ERR_UNSUPPORTED;
  return SB_OK;
}

extern "C" int sb_s2s_attn_fwd(const float* eh, int eh_group, const float* hx, const float* ax_prev,
                               const float* conv_wT, const float* conv_b, const float* lin_w,
                               float lin_b, int log_t, int B, int T, int H, int Kc, float* sx,
                               float* ax, const float* fc_w, const float* fc_b, int C,
                               float* logits, long long logit_stride, float* logp, int* argmax,
                               int* history, int hist_stride, int hist_col, int* end_count,
                               int end_tok, const int* done, const int* lens, void* workspace,
                               size_t workspace_bytes, void* stream_) {
  if (!eh || eh_group < 1 || !hx || !conv_wT || !conv_b || !lin_w || !sx || !ax || !workspace)
    return SB_ERR_INVALID;
  int rc = attn_dims_ok(B, T, H, Kc);
  if (rc != SB_OK) return rc;
  if (workspace_bytes < attn_ws_bytes(B, T, H)) return SB_ERR_WORKSPACE;
  if (fc_w && (!fc_b || C <= 0 || C > (ATT_NW - 1) * H)) return SB_ERR_INVALID;
  const size_t smem = sizeof(float) * ((size_t)ATT_NW * H + 2 * ATT_NW + ATT_MAX_TS);
  if (smem > 220 * 1024) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (smem > 40 * 1024 &&
      cudaFuncSetAttribute(s2s_attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)smem) != cudaSuccess)
    return SB_ERR_CUDA;
  AttnFwdParams p;
  p.eh = eh; p.eh_group = eh_group; p.hx = hx; p.ax_prev = ax_prev; p.conv_wT = conv_wT;
  p.conv_b = conv_b; p.lin_w = lin_w; p.lin_b = lin_b; p.sx = sx; p.ax = ax; p.fc_w = fc_w;
  p.fc_b = fc_b; p.logits = logits; p.logit_stride = logit_stride; p.logp = logp;
  p.argmax = argmax; p.history = history; p.hist_stride = hist_stride; p.hist_col = hist_col;
  p.end_count = end_count; p.end_tok = end_tok; p.done = done; p.lens = lens;
  p.ws = attn_ws_carve(workspace, B, T, H);
  p.B = B; p.T = T; p.H = H; p.Kc = Kc; p.C = C; p.log_t = log_t;
  s2s_attn_fwd_kernel<<<dim3((T + ATT_TT - 1) / ATT_TT, B), ATT_THREADS, smem, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_dout(const float* dlogits, const float* fc_w, const float* hx, const float* sx,
                           float* d_o, float* o_all, long long rows, int C, int H, void* stream_) {
  if (!dlogits || !fc_w || !hx || !sx || !d_o || !o_all || rows <= 0 || C <= 0 || H <= 0)
    return SB_ERR_INVALID;
  if (rows > 0x7fffffffLL || C > 8192) return SB_ERR_UNSUPPORTED;
  s2s_dout_kernel<<<(unsigned int)rows, 256, C * sizeof(float),
                    reinterpret_cast<cudaStream_t>(stream_)>>>(dlogits, fc_w, hx, sx, d_o, o_all, C, H);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_attn_bwd(const float* eh, const float* hx, const float* hx_prev,
                               const float* ax_prev, const float* ax, const float* conv_wT,
                               const float* conv_b, const float* lin_w, const float* d_o,
                               const float* d_ix_next, const float* d_ax_next,
                               const float* d_hx_next, const float* gates, float* d_eh,
                               float* d_ax_prev, float* d_gi, float* d_gh, float* d_hx_direct,
                               float* g_conv_wT, float* g_conv_b, float* g_lin_w, float* g_lin_b,
                               int log_t, int B, int T, int H, int Kc, const int* lens,
                               void* workspace, size_t workspace_bytes, void* stream_) {
  if (!eh || !hx || !hx_prev || !ax || !conv_wT || !conv_b || !lin_w || !d_o || !gates || !d_eh ||
      !d_ax_prev || !d_gi || !d_gh || !d_hx_direct || !g_conv_wT || !g_conv_b || !g_lin_w ||
      !g_lin_b || !workspace)
    return SB_ERR_INVALID;
  int rc = attn_dims_ok(B, T, H, Kc);
  if (rc != SB_OK) return rc;
  if (workspace_bytes < attn_ws_bytes(B, T, H)) return SB_ERR_WORKSPACE;
  const size_t smem_a = sizeof(float) * ((size_t)H + ATT_NW);
  const size_t smem_b = sizeof(float) * ((size_t)H * (1 + ATT_TT + ATT_NW) + ATT_NW * ATT_WIN +
                                         ATT_TT + ATT_KMAX - 1 + ATT_NW);
  if (smem_b > 220 * 1024) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (smem_b > 40 * 1024 &&
      cudaFuncSetAttribute(s2s_attn_bwd_b_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)smem_b) != cudaSuccess)
    return SB_ERR_CUDA;
  AttnBwdParams p;
  p.eh = eh; p.hx = hx; p.hx_prev = hx_prev; p.ax_prev = ax_prev; p.ax = ax;
  p.conv_wT = conv_wT; p.conv_b = conv_b; p.lin_w = lin_w; p.d_o = d_o;
  p.d_ix_next = d_ix_next; p.d_ax_next = d_ax_next;
  p.d_hx_next = d_hx_next; p.gates = gates; p.d_eh = d_eh; p.d_ax_prev = d_ax_prev; p.d_gi = d_gi;
  p.d_gh = d_gh; p.d_hx_direct = d_hx_direct; p.g_conv_wT = g_conv_wT;
  p.g_conv_b = g_conv_b; p.g_lin_w = g_lin_w; p.g_lin_b = g_lin_b; p.lens = lens;
  p.ws = attn_ws_carve(workspace, B, T, H);
  p.B = B; p.T = T; p.H = H; p.Kc = Kc; p.log_t = log_t;
  const dim3 grid((T + ATT_TT - 1) / ATT_TT, B);
  s2s_attn_bwd_a_kernel<<<grid, ATT_THREADS, smem_a, stream>>>(p);
  s2s_attn_bwd_b_kernel<<<grid, ATT_THREADS, smem_b, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_cell_bwd(const float* d_gi, const float* d_gh, const float* d_hx_direct,
                               const float* w_ihT, const float* w_hhT, float* d_ix,
                               float* d_hx_prev, int B, int H, void* stream_) {
  if (!d_gi || !d_gh || !d_hx_direct || !w_ihT || !w_hhT || !d_ix || !d_hx_prev || B <= 0 || H <= 0)
    return SB_ERR_INVALID;
  if ((3 * H) % 4 != 0) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CellBwdParams p;
  p.d_gi = d_gi; p.d_gh = d_gh; p.d_hx_direct = d_hx_direct; p.w_ihT = w_ihT; p.w_hhT = w_hhT;
  p.d_ix = d_ix; p.d_hx_prev = d_hx_prev; p.B = B; p.H = H;
  const int cols = (H + 1) / 2;
  const dim3 grid((cols + CELL_WARPS - 1) / CELL_WARPS, (B + CELL_NB - 1) / CELL_NB);
  const size_t smem = (size_t)2 * CELL_NB * CELL_KCB * sizeof(float);
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(s2s_cell_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem) != cudaSuccess)
      return SB_ERR_CUDA;
    attr = true;
  }
  s2s_cell_bwd_kernel<<<grid, 32 * CELL_WARPS, smem, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_check_done(const int* end_count, int B, int* done, int* nsteps, int step1,
                                 void* stream_) {
  if (!end_count || !done || !nsteps) return SB_ERR_INVALID;
  s2s_check_done_kernel<<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(end_count, B, done,
                                                                               nsteps, step1);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_beam_state_size(size_t* bytes) {
  if (!bytes) return SB_ERR_INVALID;
  *bytes = sizeof(sb::BeamState);
  return SB_OK;
}

// The single-utterance entry points below are the batched ones at B = 1 without a stop counter:
// the utterance's own `done` is then the no-op flag of the step kernels.
static int beam_batch_ok(int B) {
  return B <= 0 ? SB_ERR_INVALID : (B > 65535 ? SB_ERR_UNSUPPORTED : SB_OK);
}

// utterance b: state zero but score[0] = 0, node[0] = root node id 0 (its nodes[0] = {-1, start
// token}), token[0] = start token, nlive = 1, nodes_used = 1; tok_next[b*K] = start token
static int beam_init(void* state, int* nodes, int node_cap, int* tok_next, int K, int start_tok,
                     int* stop, int B, void* stream_) {
  if (!state || !nodes || !tok_next || K <= 0 || node_cap <= 0) return SB_ERR_INVALID;
  const int rc = beam_batch_ok(B);
  if (rc != SB_OK) return rc;
  sb::s2s_beam_init_kernel<<<B, 32, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<sb::BeamState*>(state), nodes, node_cap, tok_next, K, start_tok, stop);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_beam_init(void* state, int* nodes, int* tok_next, int start_tok,
                                void* stream_) {
  return beam_init(state, nodes, 1, tok_next, 1, start_tok, nullptr, 1, stream_);
}

extern "C" int sb_s2s_beam_init_batch(void* state, int* nodes, int node_cap, int* tok_next, int K,
                                      int start_tok, int* stop, int B, void* stream_) {
  if (!stop) return SB_ERR_INVALID;
  return beam_init(state, nodes, node_cap, tok_next, K, start_tok, stop, B, stream_);
}

// checks and fill-in shared by the single-CTA and the split selection
static int beam_params(sb::BeamParams* p, const float* logp, void* state, double* c_scores,
                       int* nodes, int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                       int end_tok, int step, int max_len, int node_cap, int c_cap, int* stop,
                       int B) {
  if (!logp || !state || !c_scores || !nodes || !parent_row || !tok_next || !out_tokens)
    return SB_ERR_INVALID;
  const int rc = beam_batch_ok(B);
  if (rc != SB_OK) return rc;
  if (K <= 0 || K > sb::BM_MAXK || C <= 0) return SB_ERR_UNSUPPORTED;
  p->logp = logp; p->st = reinterpret_cast<sb::BeamState*>(state); p->c_scores = c_scores;
  p->nodes = nodes; p->parent_row = parent_row; p->tok_next = tok_next; p->out_tokens = out_tokens;
  p->stop = stop;
  p->K = K; p->C = C; p->end_tok = end_tok; p->step = step; p->max_len = max_len;
  p->node_cap = node_cap; p->c_cap = c_cap; p->B = B;
  return SB_OK;
}

template <class Fuse>
static int beam_select(const float* logp, void* state, double* c_scores, int* nodes,
                       int* parent_row, int* tok_next, int* out_tokens, int K, int C, int end_tok,
                       int step, int max_len, int node_cap, int c_cap, int* stop, int B,
                       void* stream_, const Fuse& fu) {
  sb::BeamParams p;
  const int rc = beam_params(&p, logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K,
                             C, end_tok, step, max_len, node_cap, c_cap, stop, B);
  if (rc != SB_OK) return rc;
  const size_t smem = (size_t)K * C * sizeof(double);
  if (smem > 200 * 1024) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (smem > 40 * 1024 &&
      cudaFuncSetAttribute(sb::s2s_beam_select_kernel<Fuse>,
                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return SB_ERR_CUDA;
  sb::s2s_beam_select_kernel<Fuse><<<B, 256, smem, stream>>>(p, fu);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_beam_select(const float* logp, void* state, double* c_scores, int* nodes,
                                  int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                                  int end_tok, int step, int max_len, int node_cap, int c_cap,
                                  void* stream_) {
  return beam_select(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C, end_tok,
                     step, max_len, node_cap, c_cap, nullptr, 1, stream_, sb::S2sNoFuse{});
}

extern "C" int sb_s2s_beam_select_batch(const float* logp, void* state, double* c_scores,
                                        int* nodes, int* parent_row, int* tok_next,
                                        int* out_tokens, int K, int C, int end_tok, int step,
                                        int max_len, int node_cap, int c_cap, int* stop, int B,
                                        void* stream_) {
  if (!stop) return SB_ERR_INVALID;
  return beam_select(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C, end_tok,
                     step, max_len, node_cap, c_cap, stop, B, stream_, sb::S2sNoFuse{});
}

extern "C" int sb_s2s_beam_select_fits(int K, int C) {
  return (K > 0 && K <= sb::BM_MAXK && C > 0 && (long long)K * C * 8 <= 200 * 1024) ? 1 : 0;
}

static int beam_split_tiles(int K, int C) {
  return (int)(((long long)K * C + sb::BM_TILE - 1) / sb::BM_TILE);
}

// B utterances: B times the bytes of one; carved as [B][tiles][2K] scores | [B][tiles][2K]
// indices | [B][tiles] counts, which needs less than that
extern "C" int sb_s2s_beam_split_workspace_size_batch(int K, int C, int B, size_t* bytes) {
  if (!bytes || K <= 0 || C <= 0 || B <= 0) return SB_ERR_INVALID;
  const size_t nt = (size_t)beam_split_tiles(K, C);
  *bytes = (size_t)B * (nt * 2 * K * (sizeof(double) + sizeof(int)) + nt * sizeof(int) + 64);
  return SB_OK;
}

extern "C" int sb_s2s_beam_split_workspace_size(int K, int C, size_t* bytes) {
  return sb_s2s_beam_split_workspace_size_batch(K, C, 1, bytes);
}

template <class Fuse>
static int beam_select_split(const float* logp, void* state, double* c_scores, int* nodes,
                             int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                             int end_tok, int step, int max_len, int node_cap, int c_cap,
                             int* stop, int B, void* workspace, size_t workspace_bytes,
                             void* stream_, const Fuse& fu) {
  if (!workspace) return SB_ERR_INVALID;
  sb::BeamParams p;
  const int rc = beam_params(&p, logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K,
                             C, end_tok, step, max_len, node_cap, c_cap, stop, B);
  if (rc != SB_OK) return rc;
  if ((long long)K * C > 0x7fffffffLL) return SB_ERR_UNSUPPORTED;
  size_t need = 0;
  sb_s2s_beam_split_workspace_size_batch(K, C, B, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  const int nt = beam_split_tiles(K, C);
  const size_t smem = (size_t)nt * sizeof(int);
  if (smem > 200 * 1024) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (smem > 40 * 1024 &&
      cudaFuncSetAttribute(sb::s2s_beam_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)smem) != cudaSuccess)
    return SB_ERR_CUDA;
  const size_t slots = (size_t)B * nt * 2 * K;
  double* t_sc = reinterpret_cast<double*>(workspace);
  int* t_idx = reinterpret_cast<int*>(t_sc + slots);
  int* t_cnt = t_idx + slots;
  sb::s2s_beam_tiles_kernel<Fuse><<<dim3(nt, B), 256, 0, stream>>>(p, t_sc, t_idx, t_cnt, fu);
  sb::s2s_beam_merge_kernel<<<B, 256, smem, stream>>>(p, t_sc, t_idx, t_cnt, nt);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_beam_select_split(const float* logp, void* state, double* c_scores,
                                        int* nodes, int* parent_row, int* tok_next,
                                        int* out_tokens, int K, int C, int end_tok, int step,
                                        int max_len, int node_cap, int c_cap, void* workspace,
                                        size_t workspace_bytes, void* stream_) {
  return beam_select_split(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C,
                           end_tok, step, max_len, node_cap, c_cap, nullptr, 1, workspace,
                           workspace_bytes, stream_, sb::S2sNoFuse{});
}

extern "C" int sb_s2s_beam_select_split_batch(const float* logp, void* state, double* c_scores,
                                              int* nodes, int* parent_row, int* tok_next,
                                              int* out_tokens, int K, int C, int end_tok,
                                              int step, int max_len, int node_cap, int c_cap,
                                              int* stop, int B, void* workspace,
                                              size_t workspace_bytes, void* stream_) {
  if (!stop) return SB_ERR_INVALID;
  return beam_select_split(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C,
                           end_tok, step, max_len, node_cap, c_cap, stop, B, workspace,
                           workspace_bytes, stream_, sb::S2sNoFuse{});
}

extern "C" int sb_s2s_beam_select_lm_batch(const float* logp, void* state, double* c_scores,
                                           int* nodes, int* parent_row, int* tok_next,
                                           int* out_tokens, int K, int C, int end_tok, int step,
                                           int max_len, int node_cap, int c_cap, int* stop, int B,
                                           const SbNgramLm* lm, double lm_weight,
                                           double insertion_bonus, void* stream_) {
  if (!stop) return SB_ERR_INVALID;
  sb::S2sLmFuse fu;
  const int rc = beam_lm_fuse(lm, lm_weight, insertion_bonus, C, &fu);
  if (rc != SB_OK) return rc;
  return beam_select(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C, end_tok,
                     step, max_len, node_cap, c_cap, stop, B, stream_, fu);
}

extern "C" int sb_s2s_beam_select_split_lm_batch(const float* logp, void* state,
                                                 double* c_scores, int* nodes, int* parent_row,
                                                 int* tok_next, int* out_tokens, int K, int C,
                                                 int end_tok, int step, int max_len, int node_cap,
                                                 int c_cap, int* stop, int B, void* workspace,
                                                 size_t workspace_bytes, const SbNgramLm* lm,
                                                 double lm_weight, double insertion_bonus,
                                                 void* stream_) {
  if (!stop) return SB_ERR_INVALID;
  sb::S2sLmFuse fu;
  const int rc = beam_lm_fuse(lm, lm_weight, insertion_bonus, C, &fu);
  if (rc != SB_OK) return rc;
  return beam_select_split(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C,
                           end_tok, step, max_len, node_cap, c_cap, stop, B, workspace,
                           workspace_bytes, stream_, fu);
}

extern "C" int sb_s2s_beam_select_wordlm_batch(const float* logp, void* state, double* c_scores,
                                               int* nodes, int* parent_row, int* tok_next,
                                               int* out_tokens, int K, int C, int end_tok,
                                               int step, int max_len, int node_cap, int c_cap,
                                               int* stop, int B, const SbWordLm* lm,
                                               double lm_weight, double insertion_bonus,
                                               double oov_penalty, int* word_nodes,
                                               void* stream_) {
  if (!stop) return SB_ERR_INVALID;
  sb::S2sWordLmFuse fu;
  const int rc = beam_wordlm_fuse(lm, lm_weight, insertion_bonus, oov_penalty, C, end_tok,
                                  word_nodes, nodes, &fu);
  if (rc != SB_OK) return rc;
  return beam_select(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C, end_tok,
                     step, max_len, node_cap, c_cap, stop, B, stream_, fu);
}

extern "C" int sb_s2s_beam_select_split_wordlm_batch(
    const float* logp, void* state, double* c_scores, int* nodes, int* parent_row, int* tok_next,
    int* out_tokens, int K, int C, int end_tok, int step, int max_len, int node_cap, int c_cap,
    int* stop, int B, void* workspace, size_t workspace_bytes, const SbWordLm* lm,
    double lm_weight, double insertion_bonus, double oov_penalty, int* word_nodes,
    void* stream_) {
  if (!stop) return SB_ERR_INVALID;
  sb::S2sWordLmFuse fu;
  const int rc = beam_wordlm_fuse(lm, lm_weight, insertion_bonus, oov_penalty, C, end_tok,
                                  word_nodes, nodes, &fu);
  if (rc != SB_OK) return rc;
  return beam_select_split(logp, state, c_scores, nodes, parent_row, tok_next, out_tokens, K, C,
                           end_tok, step, max_len, node_cap, c_cap, stop, B, workspace,
                           workspace_bytes, stream_, fu);
}

extern "C" int sb_s2s_beam_gather_batch(const float* hx_in, const float* sx_in,
                                        const float* ax_in, float* hx_out, float* sx_out,
                                        float* ax_out, const int* parent_row, const void* state,
                                        int K, int H, int T, int B, void* stream_) {
  if (!hx_in || !sx_in || !ax_in || !hx_out || !sx_out || !ax_out || !parent_row || !state ||
      K <= 0)
    return SB_ERR_INVALID;
  const int rc = beam_batch_ok(B);
  if (rc != SB_OK) return rc;
  sb::s2s_beam_gather_kernel<<<B * K, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      hx_in, sx_in, ax_in, hx_out, sx_out, ax_out, parent_row,
      reinterpret_cast<const sb::BeamState*>(state), K, H, T);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_beam_gather(const float* hx_in, const float* sx_in, const float* ax_in,
                                  float* hx_out, float* sx_out, float* ax_out,
                                  const int* parent_row, const void* state, int K, int H, int T,
                                  void* stream_) {
  return sb_s2s_beam_gather_batch(hx_in, sx_in, ax_in, hx_out, sx_out, ax_out, parent_row, state,
                                  K, H, T, 1, stream_);
}
