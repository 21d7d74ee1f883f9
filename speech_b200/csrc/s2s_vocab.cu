// Output projection of the attention decoder over many CTAs: the route for vocabularies the fused
// attention kernel cannot hold (C > 7 H, see sb_s2s_fc_fused).
//
//   logits[r, c] = fc_b[c] + sum_h fc_w[c, h] o[r, h],   o = hx + sx          (seq2seq.py:108,131)
//
// s2s_fc_rows     grid (C/32 class tiles, R/64 row blocks).  A CTA stages 16 rows of o at a time in
//                 shared memory; each warp owns 4 classes and keeps 4 x 16 accumulators in
//                 registers, lanes over h in float4 steps.  The sum of every logit runs in one
//                 order that depends on H only (lane-strided fmaf chain, then a butterfly), so a
//                 row gives bit-identical logits whether it is projected alone (decode_step,
//                 greedy, beam) or with all steps*B rows of a teacher-forced decode.  Each CTA then
//                 writes per-row partials of its tile (max, first arg-max, sum exp(l - max)); the
//                 last CTA of a row block (ticket, reset in-kernel) combines them in a fixed order
//                 into the arg-max, the greedy history / end count and the log-sum-exp.
// s2s_fc_logp     logp = logit - lse, elementwise (in place allowed).
// Both honour the `done` word of the decode loops.  fp32 throughout, like the fused kernel.
#include "common.cuh"
#include <limits.h>
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int FC_THREADS = 256;
static constexpr int FC_NW = FC_THREADS / 32;
static constexpr int FC_CPW = 4;                     // classes per warp
static constexpr int FC_CT = FC_NW * FC_CPW;         // classes per CTA tile
static constexpr int FC_RB = 16;                     // rows per chunk (register accumulators)
static constexpr int FC_RPB = 4 * FC_RB;             // rows per CTA (row block)
static constexpr int FC_ATT_NW = 8;                  // warps of s2s_attn_fwd (csrc/s2s.cu)
static_assert(FC_CT == 32, "a warp computes the tile partials of one row, one class per lane");

struct FcWs {
  unsigned int* cnt;   // [NRB] tickets, zero between launches
  float* lse;          // [R]
  float* pm;           // [R][NT] tile max
  float* ps;           // [R][NT] tile sum exp(l - max)
  int* pa;             // [R][NT] tile first arg-max
};

static size_t fc_ws_bytes(long long R, int C) {
  const size_t NT = (size_t)(C + FC_CT - 1) / FC_CT, NRB = (size_t)(R + FC_RPB - 1) / FC_RPB;
  return ((NRB * 4 + 255) & ~(size_t)255) + 4 * (size_t)R * (1 + 3 * NT) + 64;
}
static FcWs fc_ws_carve(void* ws, long long R, int C) {
  const size_t NT = (size_t)(C + FC_CT - 1) / FC_CT, NRB = (size_t)(R + FC_RPB - 1) / FC_RPB;
  FcWs w;
  w.cnt = reinterpret_cast<unsigned int*>(ws);      // first: the caller zeroes the buffer once
  float* f = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + ((NRB * 4 + 255) & ~(size_t)255));
  w.lse = f; f += R;
  w.pm = f; f += (size_t)R * NT;
  w.ps = f; f += (size_t)R * NT;
  w.pa = reinterpret_cast<int*>(f);
  return w;
}

struct FcParams {
  const float* hx;        // (R, H)
  const float* sx;        // (R, H) or null (o = hx)
  const float* fc_w;      // (C, H)
  const float* fc_b;      // (C)
  float* logits;          // row r at logits + (r % group) * ld0 + (r / group) * ld1, or null
  long long ld0, ld1;
  int group;
  int* argmax;            // (R) or null
  int* history;           // history[r * hist_stride + hist_col] = arg-max, or null
  int hist_stride, hist_col;
  int* end_count;         // += 1 per row whose arg-max == end_tok, or null
  int end_tok;
  const int* done;        // != 0 -> no-op, or null
  FcWs ws;
  int R, H, C;
};

SB_DEVINL long long fc_row_off(long long r, int group, long long ld0, long long ld1) {
  return (r % group) * ld0 + (r / group) * ld1;
}

// (m, a, s) <- (m, a, s) (+) (m2, a2, s2): max, first arg-max, sum exp(l - max).  Symmetric in its
// two arguments, so a butterfly gives every lane the same bits.
SB_DEVINL void lse_combine(float& m, int& a, float& s, float m2, int a2, float s2) {
  const float mn = fmaxf(m, m2);
  const float t1 = m == -INFINITY ? 0.f : s * expf(m - mn);
  const float t2 = m2 == -INFINITY ? 0.f : s2 * expf(m2 - mn);
  if (m2 > m || (m2 == m && a2 < a)) a = a2;
  m = mn;
  s = t1 + t2;
}

SB_DEVINL float fc_fma4(const float4 w, const float4 o, float acc) {
  acc = fmaf(w.x, o.x, acc);
  acc = fmaf(w.y, o.y, acc);
  acc = fmaf(w.z, o.z, acc);
  return fmaf(w.w, o.w, acc);
}

__global__ void __launch_bounds__(FC_THREADS) s2s_fc_rows_kernel(const FcParams p) {
  extern __shared__ float4 fc_smem[];              // [RB][H/4] o rows of the chunk
  __shared__ float lg[FC_RB][FC_CT + 1];
  __shared__ int s_last;
  if (p.done && *p.done) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = p.H, H4 = H >> 2, C = p.C;
  const int tile = blockIdx.x, NT = gridDim.x, rb = blockIdx.y;
  const int c0 = tile * FC_CT;
  const long long r_begin = (long long)rb * FC_RPB;
  const long long r_end = min((long long)p.R, r_begin + FC_RPB);
  const float4* wr[FC_CPW];
#pragma unroll
  for (int k = 0; k < FC_CPW; ++k)     // (clamped: classes past C compute and are dropped)
    wr[k] = reinterpret_cast<const float4*>(p.fc_w + (size_t)min(c0 + warp * FC_CPW + k, C - 1) * H);
  for (long long r0 = r_begin; r0 < r_end; r0 += FC_RB) {
    const int nr = (int)min((long long)FC_RB, r_end - r0);
    __syncthreads();                               // the previous chunk has been consumed
    for (int e = tid; e < FC_RB * H4; e += FC_THREADS) {
      const int r = e / H4, h4 = e - r * H4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < nr) {
        const size_t ro = (size_t)(r0 + r) * H;
        v = __ldg(reinterpret_cast<const float4*>(p.hx + ro) + h4);
        if (p.sx) {
          const float4 s = __ldg(reinterpret_cast<const float4*>(p.sx + ro) + h4);
          v.x += s.x; v.y += s.y; v.z += s.z; v.w += s.w;
        }
      }
      fc_smem[e] = v;
    }
    __syncthreads();
    float acc[FC_CPW][FC_RB];
#pragma unroll
    for (int k = 0; k < FC_CPW; ++k)
#pragma unroll
      for (int r = 0; r < FC_RB; ++r) acc[k][r] = 0.f;
    for (int h4 = lane; h4 < H4; h4 += 32) {
      float4 wv[FC_CPW];
#pragma unroll
      for (int k = 0; k < FC_CPW; ++k) wv[k] = __ldg(wr[k] + h4);
#pragma unroll
      for (int r = 0; r < FC_RB; ++r) {
        const float4 o = fc_smem[r * H4 + h4];
#pragma unroll
        for (int k = 0; k < FC_CPW; ++k) acc[k][r] = fc_fma4(wv[k], o, acc[k][r]);
      }
    }
#pragma unroll
    for (int k = 0; k < FC_CPW; ++k) {
      const int c = min(c0 + warp * FC_CPW + k, C - 1);
      const float bias = __ldg(p.fc_b + c);
#pragma unroll
      for (int r = 0; r < FC_RB; ++r) {
        const float v = warp_sum(acc[k][r]);
        if (lane == 0) lg[r][warp * FC_CPW + k] = v + bias;
      }
    }
    __syncthreads();
    // ---- the tile's partials of each row: a warp per row, a lane per class ----
    for (int r = warp; r < nr; r += FC_NW) {
      const long long row = r0 + r;
      const int c = c0 + lane;
      const bool ok = c < C;
      const float v = ok ? lg[r][lane] : -INFINITY;
      if (ok && p.logits) p.logits[fc_row_off(row, p.group, p.ld0, p.ld1) + c] = v;
      float mx = v;
      int am = ok ? c : INT_MAX;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mx, off);
        const int oa = __shfl_xor_sync(0xffffffffu, am, off);
        if (om > mx || (om == mx && oa < am)) { mx = om; am = oa; }
      }
      const float se = warp_sum(ok ? expf(v - mx) : 0.f);
      if (lane == 0) {
        const size_t q = (size_t)row * NT + tile;
        p.ws.pm[q] = mx; p.ws.ps[q] = se; p.ws.pa[q] = am;
      }
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(p.ws.cnt + rb, 1u) == (unsigned int)(NT - 1));
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- the row block's last CTA: every row's tiles, lane-strided in tile order, then a butterfly
  for (long long row = r_begin + warp; row < r_end; row += FC_NW) {
    float m = -INFINITY, s = 0.f;
    int a = INT_MAX;
    for (int t = lane; t < NT; t += 32) {
      const size_t q = (size_t)row * NT + t;
      lse_combine(m, a, s, __ldcg(p.ws.pm + q), __ldcg(p.ws.pa + q), __ldcg(p.ws.ps + q));
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, off);
      const int oa = __shfl_xor_sync(0xffffffffu, a, off);
      const float os = __shfl_xor_sync(0xffffffffu, s, off);
      lse_combine(m, a, s, om, oa, os);
    }
    if (lane == 0) {
      p.ws.lse[row] = m + logf(s);
      if (p.argmax) p.argmax[row] = a;
      if (p.history) p.history[(size_t)row * p.hist_stride + p.hist_col] = a;
      if (p.end_count && a == p.end_tok) atomicAdd(p.end_count, 1);
    }
  }
  if (tid == 0) p.ws.cnt[rb] = 0u;
}

__global__ void __launch_bounds__(256) s2s_fc_logp_kernel(const float* logits, int group,
                                                          long long ld0, long long ld1,
                                                          const float* __restrict__ lse,
                                                          float* logp, int C, const int* done) {
  if (done && *done) return;
  const long long r = blockIdx.y;
  const float* src = logits + fc_row_off(r, group, ld0, ld1);
  const float l = lse[r];
  for (int c = blockIdx.x * 1024 + threadIdx.x; c < min(C, (int)(blockIdx.x + 1) * 1024); c += 256)
    logp[(size_t)r * C + c] = src[c] - l;
}

}  // namespace sb

using namespace sb;

extern "C" int sb_s2s_fc_fused(int H, int C) {
  return (H > 0 && C > 0 && (long long)C <= (long long)(FC_ATT_NW - 1) * H) ? 1 : 0;
}

extern "C" int sb_s2s_fc_workspace_size(long long R, int C, size_t* bytes) {
  if (!bytes || R <= 0 || C <= 0) return SB_ERR_INVALID;
  *bytes = fc_ws_bytes(R, C);
  return SB_OK;
}

extern "C" int sb_s2s_fc_rows(const float* hx, const float* sx, const float* fc_w,
                              const float* fc_b, long long R, int H, int C, float* logits,
                              int row_group, long long ld0, long long ld1, int* argmax,
                              int* history, int hist_stride, int hist_col, int* end_count,
                              int end_tok, const int* done, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  if (!hx || !fc_w || !fc_b || !workspace || R <= 0 || H <= 0 || C <= 0 || row_group <= 0)
    return SB_ERR_INVALID;
  if (H % 4 != 0 || (R + FC_RPB - 1) / FC_RPB > 65535) return SB_ERR_UNSUPPORTED;
  if (workspace_bytes < fc_ws_bytes(R, C)) return SB_ERR_WORKSPACE;
  const size_t smem = sizeof(float) * (size_t)FC_RB * H;
  if (smem > 200 * 1024) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (smem > 40 * 1024 &&
      cudaFuncSetAttribute(s2s_fc_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)smem) != cudaSuccess)
    return SB_ERR_CUDA;
  FcParams p;
  p.hx = hx; p.sx = sx; p.fc_w = fc_w; p.fc_b = fc_b; p.logits = logits; p.ld0 = ld0; p.ld1 = ld1;
  p.group = row_group; p.argmax = argmax; p.history = history; p.hist_stride = hist_stride;
  p.hist_col = hist_col; p.end_count = end_count; p.end_tok = end_tok; p.done = done;
  p.ws = fc_ws_carve(workspace, R, C);
  p.R = (int)R; p.H = H; p.C = C;
  const dim3 grid((C + FC_CT - 1) / FC_CT, (unsigned int)((R + FC_RPB - 1) / FC_RPB));
  s2s_fc_rows_kernel<<<grid, FC_THREADS, smem, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_s2s_fc_logp(const float* logits, int row_group, long long ld0, long long ld1,
                              float* logp, long long R, int C, const int* done,
                              const void* workspace, size_t workspace_bytes, void* stream_) {
  if (!logits || !logp || !workspace || R <= 0 || C <= 0 || row_group <= 0) return SB_ERR_INVALID;
  if (R > 65535) return SB_ERR_UNSUPPORTED;
  if (workspace_bytes < fc_ws_bytes(R, C)) return SB_ERR_WORKSPACE;
  const FcWs w = fc_ws_carve(const_cast<void*>(workspace), R, C);
  const dim3 grid((C + 1023) / 1024, (unsigned int)R);
  s2s_fc_logp_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      logits, row_group, ld0, ld1, w.lse, logp, C, done);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
