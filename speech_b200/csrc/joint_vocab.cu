// Row kernels of the large-vocabulary RNN-T joint (V1 = V+1 > 64 classes, where fc2's weight no
// longer fits the shared memory of the fused kernel in joint.cu).
//
// The lattice is processed a slab of Tc frames at a time (nodes are TIME-major, n = (t*B + b)*U1 + u,
// so a slab is the contiguous row range n0 = t0*B*U1 .. n0 + Tc*B*U1):
//   1. sb_rnnt_joint_build_slab        z = relu(fx + fy)            bf16 [rows][H]
//   2. sb_gemm_bf16_tn                 logits = z W2^T + b2         f32  [rows][ld], ld >= V1
//   3. forward : sb_rnnt_joint_vocab_fwd_rows   max / log-sum-exp per row -> lat, lse (and lp_full)
//      backward: sb_rnnt_joint_vocab_bwd_rows   dlogits = g_b [k = blank] + g_l [k = label]
//                                                          - (g_b + g_l) exp(v_k - lse)  (bf16)
//                                                db2 += column sums of dlogits
//   4. decoding: sb_rnnt_shortlist_rows   per node the blank's log-prob, the kp best non-blank
//                                          classes and the next value, for the beam search of
//                                          csrc/tdecode.cu (also run on a given lp tensor)
// Neither the (nodes x V1) logits nor their gradient ever exist in full, only one slab of each.
// Roofline of the row kernels: memory bandwidth (one fp32 read per logit, plus one bf16 write per
// logit in the backward pass); the slab is read back from L2 when it fits there.
#include "common.cuh"
#include "shortlist.cuh"
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

typedef __nv_bfloat16 bf16;

// (b, t, u) of node n and the label of its arc (u -> u+1), -1 at the last label position
SB_DEVINL void vocab_node(long long n, int B, int U1, const int* ymat, int* b, int* t, int* u,
                          int* lab) {
  const long long tb = n / U1;
  *u = (int)(n - tb * U1);
  *b = (int)(tb % B);
  *t = (int)(tb / B);
  *lab = (*u < U1 - 1) ? ymat[(long long)*b * (U1 - 1) + *u] : -1;
}

// ---- forward: one warp per row.  Online max / sum of exp over float4 groups of the row, then a
// warp-level merge of the (max, sum) pairs. ----
__global__ void __launch_bounds__(256)
joint_vocab_fwd_rows_kernel(const float* __restrict__ logits, long long ld,
                            const int* __restrict__ ymat, float* __restrict__ lat,
                            float* __restrict__ lse_out, float* __restrict__ lp_full, int B, int T,
                            int U1, int V1, int blank, long long n0, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long r = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* v = logits + r * ld;
  float m = -INFINITY, s = 0.f;
  for (int j = lane * 4; j < V1; j += 128) {
    const float4 q = *reinterpret_cast<const float4*>(v + j);   // j + 3 < ld (ld % 8 == 0)
    const float x0 = q.x;
    const float x1 = j + 1 < V1 ? q.y : -INFINITY;
    const float x2 = j + 2 < V1 ? q.z : -INFINITY;
    const float x3 = j + 3 < V1 ? q.w : -INFINITY;
    const float cm = fmaxf(fmaxf(x0, x1), fmaxf(x2, x3));
    if (cm > m) {
      s *= __expf(m - cm);
      m = cm;
    }
    s += __expf(x0 - m) + __expf(x1 - m) + __expf(x2 - m) + __expf(x3 - m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, m, o);
    const float so = __shfl_xor_sync(0xffffffffu, s, o);
    const float mm = fmaxf(m, mo);
    // a lane that saw no class has (m, s) = (-inf, 0) and contributes nothing
    s = (m == -INFINITY ? 0.f : s * __expf(m - mm)) + (mo == -INFINITY ? 0.f : so * __expf(mo - mm));
    m = mm;
  }
  const float lse = m + __logf(s);
  const long long n = n0 + r;
  int b, t, u, lab;
  vocab_node(n, B, U1, ymat, &b, &t, &u, &lab);
  if (lane == 0) {
    const float ll = (lab >= 0 && lab < V1) ? v[lab] - lse : -INFINITY;
    *reinterpret_cast<float2*>(lat + n * 2) = make_float2(v[blank] - lse, ll);
    lse_out[n] = lse;
  }
  if (lp_full) {
    float* o = lp_full + (((long long)b * T + t) * U1 + u) * V1;   // batch-first
    for (int j = lane; j < V1; j += 32) o[j] = v[j] - lse;
  }
}

// ---- backward: a row is covered by TPR threads of 4 columns each (TPR = 32..256, the smallest
// that spans the row or 256), the CTA takes 256 / TPR rows at a time and walks a strided set of
// rows; grid.y splits rows wider than 1024 columns.  Column sums of dlogits are kept per thread in
// registers, merged in shared memory and added to db2 once per CTA. ----
__global__ void __launch_bounds__(256)
joint_vocab_bwd_rows_kernel(const float* __restrict__ logits, long long ld,
                            const float* __restrict__ lse, const float* __restrict__ garc,
                            const int* __restrict__ ymat, bf16* __restrict__ dl, long long ldd,
                            float* __restrict__ db2, int B, int U1, int V1, int blank, int tpr,
                            long long n0, long long rows) {
  __shared__ float db_s[1024];
  const int tid = threadIdx.x;
  const int slot = tid / tpr, rpi = 256 / tpr;
  const int c = blockIdx.y * (4 * tpr) + (tid - slot * tpr) * 4;
  for (int k = tid; k < 4 * tpr; k += 256) db_s[k] = 0.f;
  __syncthreads();
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (c < ldd) {
    for (long long r = blockIdx.x * (long long)rpi + slot; r < rows; r += (long long)gridDim.x * rpi) {
      const long long n = n0 + r;
      int b, t, u, lab;
      vocab_node(n, B, U1, ymat, &b, &t, &u, &lab);
      const float2 g = *reinterpret_cast<const float2*>(garc + n * 2);
      const float gs = g.x + g.y, l = lse[n];
      float d[4] = {0.f, 0.f, 0.f, 0.f};
      if (c < V1) {
        const float4 q = __ldcs(reinterpret_cast<const float4*>(logits + r * ld + c));
        const float x[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (c + i < V1)
            d[i] = (c + i == blank ? g.x : 0.f) + (c + i == lab ? g.y : 0.f) - gs * __expf(x[i] - l);
      }
      a0 += d[0]; a1 += d[1]; a2 += d[2]; a3 += d[3];
      *reinterpret_cast<uint2*>(dl + r * ldd + c) = make_uint2(pack_bf16x2(d[0], d[1]),
                                                               pack_bf16x2(d[2], d[3]));
    }
  }
  const int lc = c - blockIdx.y * (4 * tpr);
  atomicAdd(&db_s[lc], a0);
  atomicAdd(&db_s[lc + 1], a1);
  atomicAdd(&db_s[lc + 2], a2);
  atomicAdd(&db_s[lc + 3], a3);
  __syncthreads();
  for (int k = tid; k < 4 * tpr; k += 256) {
    const int col = blockIdx.y * (4 * tpr) + k;
    if (col < V1) atomicAdd(db2 + col, db_s[k]);
  }
}

// ---- shortlist rows: one warp per row.  lp_k = v_k - lse is formed with the same fp32 expression
// as the lp_full rows of joint_vocab_fwd_rows_kernel (or read as is when lse is NULL), so every
// shortlisted value is bit-identical to the full tensor's entry.  The row streams through the
// warp's top-P selection (shortlist.cuh, P = kp + 1), ranking on the ROUNDED lp, since v - lse can
// map distinct logits to equal log-probs. ----
__global__ void __launch_bounds__(256)
rnnt_shortlist_rows_kernel(const float* __restrict__ v, long long ld, const float* __restrict__ lse,
                           int B, int T, int U1, int V1, int blank, int kp, long long n0,
                           long long rows, int time_major, float* __restrict__ sl_val,
                           int* __restrict__ sl_idx, float* __restrict__ sl_meta) {
  __shared__ float buf_v[8][SL_CAP];
  __shared__ int buf_i[8][SL_CAP];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long r = blockIdx.x * 8LL + w;
  if (r >= rows) return;                   // whole warps: only __syncwarp below
  float* bv = buf_v[w];
  int* bi = buf_i[w];
  const long long n = n0 + r;
  const float* row = v + r * ld;
  const float l = lse ? lse[n] : 0.f;
  long long o = n;                         // batch-first output node
  if (time_major) {
    const long long tb = n / U1;
    const int u = (int)(n - tb * U1);
    o = ((tb % B) * T + tb / B) * U1 + u;
  }
  const int P = kp + 1;
  int cnt = 0;
  bool thr = false;
  float tv = 0.f;
  int tk = 0;
  for (int base = 0; base < V1; base += 128) {
    float x[4];
    bool q[4];
    bool anyq = false;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = base + e * 32 + lane;
      q[e] = j < V1 && j != blank;
      x[e] = 0.f;
      if (q[e]) {
        x[e] = lse ? row[j] - l : row[j];
        q[e] = !thr || sl_better(x[e], j, tv, tk);
      }
      anyq |= q[e];
    }
    if (!__any_sync(0xffffffffu, anyq)) continue;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = base + e * 32 + lane;
      unsigned m = __ballot_sync(0xffffffffu, q[e]);
      if (!m) continue;
      if (cnt + __popc(m) > SL_CAP) {      // cut the buffer to its P best, raise the threshold
        sl_sort(bv, bi, cnt, lane);
        cnt = P;
        thr = true;
        tv = bv[P - 1];
        tk = bi[P - 1];
        __syncwarp();
        q[e] = q[e] && sl_better(x[e], j, tv, tk);
        m = __ballot_sync(0xffffffffu, q[e]);
      }
      if (q[e]) {
        const int pos = cnt + __popc(m & ((1u << lane) - 1u));
        bv[pos] = x[e];
        bi[pos] = j;
      }
      cnt += __popc(m);
      __syncwarp();
    }
  }
  sl_sort(bv, bi, cnt, lane);
  for (int e = lane; e < kp; e += 32) {
    sl_val[o * kp + e] = e < cnt ? bv[e] : -INFINITY;
    sl_idx[o * kp + e] = e < cnt ? bi[e] : -1;
  }
  if (lane == 0) {
    const float bl = lse ? row[blank] - l : row[blank];
    *reinterpret_cast<float2*>(sl_meta + o * 2) = make_float2(bl, cnt > kp ? bv[kp] : -INFINITY);
  }
}

// argument checks shared by both entry points: the leading dimension of a row is a multiple of 8
// elements (16-byte aligned float4 / bf16x4 accesses), the slab lies within [0, T)
static int vocab_check(long long ld, int B, int T, int U1, int V1, int blank, int t0, int Tc) {
  if (B <= 0 || T <= 0 || U1 <= 0 || V1 <= 0 || Tc <= 0) return SB_ERR_INVALID;
  if (blank < 0 || blank >= V1 || t0 < 0 || t0 + Tc > T) return SB_ERR_INVALID;
  if (ld < V1 || ld % 8 != 0) return SB_ERR_INVALID;
  return SB_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace sb

using namespace sb;

extern "C" int sb_rnnt_joint_vocab_fwd_rows(const float* logits, long long ld, const int* ymat,
                                            float* lat, float* lse, float* lp_full, int B, int T,
                                            int U1, int V1, int blank, int t0, int Tc,
                                            void* stream_) {
  if (!logits || !ymat || !lat || !lse || !aligned16(logits)) return SB_ERR_INVALID;
  const int rc = vocab_check(ld, B, T, U1, V1, blank, t0, Tc);
  if (rc != SB_OK) return rc;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long rows = (long long)Tc * B * U1;
  const long long n0 = (long long)t0 * B * U1;
  const long long grid = (rows + 7) / 8;
  if (grid > 0x7fffffffLL) return SB_ERR_UNSUPPORTED;
  joint_vocab_fwd_rows_kernel<<<(unsigned)grid, 256, 0, stream>>>(logits, ld, ymat, lat, lse, lp_full,
                                                                  B, T, U1, V1, blank, n0, rows);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_shortlist_rows(const float* v, long long ld, const float* lse, int B, int T,
                                      int U1, int V1, int blank, int kp, int t0, int Tc,
                                      int time_major, float* sl_val, int* sl_idx, float* sl_meta,
                                      void* stream_) {
  if (!v || !sl_val || !sl_idx || !sl_meta || ld < V1) return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || U1 <= 0 || V1 <= 0 || Tc <= 0 || t0 < 0 || t0 + Tc > T)
    return SB_ERR_INVALID;
  if (blank < 0 || blank >= V1 || kp < 1 || (!time_major && (t0 != 0 || Tc != T)))
    return SB_ERR_INVALID;
  if (kp > SL_MAX_KP) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long rows = (long long)Tc * B * U1;
  const long long n0 = (long long)t0 * B * U1;
  const long long grid = (rows + 7) / 8;
  if (grid > 0x7fffffffLL) return SB_ERR_UNSUPPORTED;
  rnnt_shortlist_rows_kernel<<<(unsigned)grid, 256, 0, stream>>>(
      v, ld, lse, B, T, U1, V1, blank, kp, n0, rows, time_major, sl_val, sl_idx, sl_meta);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_joint_vocab_bwd_rows(const float* logits, long long ld, const float* lse,
                                            const float* garc, const int* ymat, void* dlogits_bf16,
                                            long long ldd, float* db2, int B, int T, int U1, int V1,
                                            int blank, int t0, int Tc, void* stream_) {
  if (!logits || !lse || !garc || !ymat || !dlogits_bf16 || !db2 || !aligned16(logits) ||
      !aligned16(dlogits_bf16))
    return SB_ERR_INVALID;
  int rc = vocab_check(ld, B, T, U1, V1, blank, t0, Tc);
  if (rc != SB_OK) return rc;
  rc = vocab_check(ldd, B, T, U1, V1, blank, t0, Tc);
  if (rc != SB_OK) return rc;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long rows = (long long)Tc * B * U1;
  const long long n0 = (long long)t0 * B * U1;
  int tpr = 32;
  while (tpr < 256 && 4 * tpr < ldd) tpr *= 2;
  const long long gy = (ldd + 4 * tpr - 1) / (4 * tpr);
  if (gy > 65535) return SB_ERR_UNSUPPORTED;
  const int rpi = 256 / tpr;
  long long gx = (rows + rpi - 1) / rpi;
  const long long cap = (long long)device_sm_count() * 8 / gy + 1;   // ~8 CTAs per SM in all
  if (gx > cap) gx = cap;
  joint_vocab_bwd_rows_kernel<<<dim3((unsigned)gx, (unsigned)gy), 256, 0, stream>>>(
      logits, ld, lse, garc, ymat, reinterpret_cast<bf16*>(dlogits_bf16), ldd, db2, B, U1, V1,
      blank, tpr, n0, rows);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
