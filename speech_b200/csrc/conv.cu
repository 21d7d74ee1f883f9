// Conv2d(+ReLU) front-end of the encoder as im2col + tensor-core GEMM.
//
// Replaces the cuDNN convolutions behind nn.Conv2d in Model.__init__/encode
// (speech/models/model.py:19-29,60-71): valid (padding 0) 2-D convolution over (time, freq) with
// kernel (kh, kw) and stride s in both dims, followed by ReLU; the stack's output is flattened
// channel-major to (B, T', C*F') (model.py:66-71).
//
// Layouts (all row-major):
//   activations between layers: "pixel-major channels-last"  P[(b*To + t)*Fo + f][c]  f32 =
//       exactly the C matrix of the GEMM; ReLU is applied by whoever READS it (so the
//       pre-activation sign is available to the backward mask);
//   im2col matrix A[m][(i*kw + j)*Ci + ci] bf16 (K padded to a multiple of 8 with zeros); the
//       weights are permuted to the same K order on the host side (40 K elements);
//   conv = sb_gemm_bf16_tn(A, Wp) + bias  on the wgmma GEMM.
// Backward: dC (pre-activation grad, bf16) -> dW = dC^T A (GEMM on transposed copies, split-K),
//   dA = dC Wp (GEMM), col2im as a GATHER (each input pixel sums its <= ceil(kh/s)*ceil(kw/s)
//   taps; no atomics) fused with the ReLU mask of the layer below.
// All kernels here are HBM-bound elementwise/gather kernels (algorithmic bytes = one read of the
// source + one write of the destination); the FLOPs run in gemm.cu.  The layers past the first
// that fit the direct-convolution kernels at the end of this file skip im2col, the GEMMs and
// col2im altogether.
#include "common.cuh"

#include "../../include/speech_b200.h"

namespace sb {

typedef __nv_bfloat16 bf16;

// ---- im2col ------------------------------------------------------------------------------------
// src: P[(b*Ti + ti)*Fi + fi][Ci] f32 (relu on read if `relu`), dst: A[M][Kp] bf16.
// One thread produces 8 consecutive K entries (one 16-byte store).  For Ci % 8 == 0 these are 8
// channels of one tap (two float4 loads); otherwise the scalar path is used per element.
__global__ void __launch_bounds__(256)
im2col_kernel(const float* __restrict__ src, const unsigned char* __restrict__ mask,
              float mscale, bf16* __restrict__ dst, int B, int Ti, int Fi, int Ci,
              int kh, int kw, int s, int To, int Fo, int Kp, int relu) {
  const int K = kh * kw * Ci;
  const int kvec = Kp >> 3;                       // 8-wide groups per row
  const long long M = (long long)B * To * Fo;
  const long long total = M * kvec;
  const bool vec = (Ci & 7) == 0;
  for (long long idx = blockIdx.x * 256LL + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * 256) {
    const long long m = idx / kvec;
    const int k0 = (int)(idx - m * kvec) << 3;
    const int f = (int)(m % Fo);
    const int bt = (int)(m / Fo);
    const int t = bt % To;
    const int b = bt / To;
    float v[8];
    if (vec && k0 < K) {
      const int ci = k0 % Ci;
      const int ij = k0 / Ci;
      const int j = ij % kw, i = ij / kw;
      const long long off = (((long long)b * Ti + (s * t + i)) * Fi + (s * f + j)) * Ci + ci;
      const float4* p = reinterpret_cast<const float4*>(src + off);
      const float4 a = __ldg(p), c = __ldg(p + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
      if (relu) {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], 0.f);
      }
      if (mask) {   // dropout of the layer below: keep-byte per element, same layout as src
        const uint2 mk = __ldg(reinterpret_cast<const uint2*>(mask + off));
        const unsigned char* mb = reinterpret_cast<const unsigned char*>(&mk);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = mb[e] ? v[e] * mscale : 0.f;
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int k = k0 + e;
        v[e] = 0.f;
        if (k < K) {
          const int ci = k % Ci;
          const int ij = k / Ci;
          const int j = ij % kw, i = ij / kw;
          const long long off = (((long long)b * Ti + (s * t + i)) * Fi + (s * f + j)) * Ci + ci;
          v[e] = __ldg(src + off);
          if (relu) v[e] = fmaxf(v[e], 0.f);
          if (mask) v[e] = mask[off] ? v[e] * mscale : 0.f;
        }
      }
    }
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
    o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(dst + m * Kp + k0) = o;
  }
}

// ---- final relayout: C[(b*To+t)*Fo+f][c] -> out[b][t][c*Fo + f] with ReLU ------------------------
__global__ void __launch_bounds__(256)
relu_to_bct_kernel(const float* __restrict__ C, const unsigned char* __restrict__ mask,
                   float mscale, float* __restrict__ out, int B, int To, int Fo, int Co) {
  const long long total = (long long)B * To * Fo * Co;
  for (long long idx = blockIdx.x * 256LL + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * 256) {
    // idx enumerates the OUTPUT (f fastest) so that writes are coalesced
    const int f = (int)(idx % Fo);
    long long r = idx / Fo;
    const int c = (int)(r % Co);
    r /= Co;                       // r = b*To + t
    const long long src = (r * Fo + f) * Co + c;
    float v = fmaxf(__ldg(C + src), 0.f);
    if (mask) v = mask[src] ? v * mscale : 0.f;
    out[idx] = v;
  }
}

// ---- top of backward: dY[b][t][c*Fo+f] * (C > 0) -> dC[(b*To+t)*Fo+f][c] bf16, db[c] += ----------
__global__ void __launch_bounds__(256)
dconv_top_kernel(const float* __restrict__ dY, const float* __restrict__ C,
                 const unsigned char* __restrict__ mask, float mscale, bf16* __restrict__ dC,
                 float* __restrict__ db, int B, int To, int Fo, int Co) {
  extern __shared__ float dbs[];
  for (int c = threadIdx.x; c < Co; c += 256) dbs[c] = 0.f;
  __syncthreads();
  const long long total = (long long)B * To * Fo * Co;
  for (long long idx = blockIdx.x * 256LL + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * 256) {
    const int c = (int)(idx % Co);     // idx enumerates dC (c fastest)
    const long long m = idx / Co;
    const int f = (int)(m % Fo);
    const long long r = m / Fo;
    float g = __ldg(dY + (r * Co + c) * Fo + f);
    if (__ldg(C + idx) <= 0.f) g = 0.f;
    else if (mask) g = mask[idx] ? g * mscale : 0.f;
    dC[idx] = __float2bfloat16_rn(g);
    if (g != 0.f) atomicAdd(&dbs[c], g);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Co; c += 256)
    if (dbs[c] != 0.f) atomicAdd(db + c, dbs[c]);
}

// ---- col2im as a gather, fused with the ReLU mask of the layer below -----------------------------
// dA[m][(i*kw+j)*Ci + ci] f32 (ld = ldA) -> dCprev[(b*Ti+ti)*Fi+fi][ci] bf16 (masked by Pprev > 0)
// Each input pixel receives at most ceil(kh/s)*ceil(kw/s) taps.  All tap loads of a thread are
// issued before any is consumed (a loop with data-dependent `continue`s left ONE load in flight
// per thread and ran at 0.9 TB/s).
template <int MAXI, int MAXJ>
__global__ void __launch_bounds__(256)
col2im_relu_kernel(const float* __restrict__ dA, long long ldA, const float* __restrict__ Pprev,
                   const unsigned char* __restrict__ maskprev, float mscale,
                   bf16* __restrict__ dCprev, float* __restrict__ db, int B, int Ti, int Fi,
                   int Ci, int kh, int kw, int s, int To, int Fo) {
  extern __shared__ float dbs[];
  for (int c = threadIdx.x; c < Ci; c += 256) dbs[c] = 0.f;
  __syncthreads();
  const long long total = (long long)B * Ti * Fi * Ci;
  for (long long idx = blockIdx.x * 256LL + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * 256) {
    const int ci = (int)(idx % Ci);
    const int px = (int)(idx / Ci);
    const int fi = px % Fi;
    const int bt = px / Fi;
    const int ti = bt % Ti;
    const int b = bt / Ti;
    const float mask = __ldg(Pprev + idx);
    float v[MAXI * MAXJ];
#pragma unroll
    for (int a = 0; a < MAXI; ++a) {
      const int i = ti % s + a * s;
      const int t = (ti - i) / s;
      const bool okt = (i < kh) && (ti - i >= 0) && (t < To);
#pragma unroll
      for (int c = 0; c < MAXJ; ++c) {
        const int j = fi % s + c * s;
        const int f = (fi - j) / s;
        const bool ok = okt && (j < kw) && (fi - j >= 0) && (f < Fo);
        v[a * MAXJ + c] = 0.f;
        if (ok)
          v[a * MAXJ + c] =
              __ldcs(dA + (((long long)b * To + t) * Fo + f) * ldA + (i * kw + j) * Ci + ci);
      }
    }
    float g = 0.f;
#pragma unroll
    for (int e = 0; e < MAXI * MAXJ; ++e) g += v[e];
    if (mask <= 0.f) g = 0.f;
    else if (maskprev) g = maskprev[idx] ? g * mscale : 0.f;
    dCprev[idx] = __float2bfloat16_rn(g);
    if (g != 0.f) atomicAdd(&dbs[ci], g);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Ci; c += 256)
    if (dbs[c] != 0.f) atomicAdd(db + c, dbs[c]);
}

// Same gather with FOUR channels per thread (Ci % 4 == 0): 16-byte tap loads, a quarter of the
// index arithmetic per element (the scalar kernel was instruction-bound: 0.70 ms at 1.9 TB/s).
template <int MAXI, int MAXJ>
__global__ void __launch_bounds__(256)
col2im_relu_v4_kernel(const float* __restrict__ dA, long long ldA, const float* __restrict__ Pprev,
                      const unsigned char* __restrict__ maskprev, float mscale,
                      bf16* __restrict__ dCprev, float* __restrict__ db, int B, int Ti, int Fi,
                      int Ci, int kh, int kw, int s, int To, int Fo) {
  extern __shared__ float dbs[];
  for (int c = threadIdx.x; c < Ci; c += 256) dbs[c] = 0.f;
  __syncthreads();
  const int C4 = Ci >> 2;
  const long long total = (long long)B * Ti * Fi * C4;
  for (long long idx = blockIdx.x * 256LL + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * 256) {
    const int c4 = (int)(idx % C4);
    const int px = (int)(idx / C4);
    const int fi = px % Fi;
    const int bt = px / Fi;
    const int ti = bt % Ti;
    const int b = bt / Ti;
    const float4 mask = __ldg(reinterpret_cast<const float4*>(Pprev) + idx);
    float4 v[MAXI * MAXJ];
#pragma unroll
    for (int a = 0; a < MAXI; ++a) {
      const int i = ti % s + a * s;
      const int t = (ti - i) / s;
      const bool okt = (i < kh) && (ti - i >= 0) && (t < To);
#pragma unroll
      for (int c = 0; c < MAXJ; ++c) {
        const int j = fi % s + c * s;
        const int f = (fi - j) / s;
        const bool ok = okt && (j < kw) && (fi - j >= 0) && (f < Fo);
        v[a * MAXJ + c] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok)
          v[a * MAXJ + c] = __ldcs(reinterpret_cast<const float4*>(
              dA + (((long long)b * To + t) * Fo + f) * ldA + (i * kw + j) * Ci + c4 * 4));
      }
    }
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int e = 0; e < MAXI * MAXJ; ++e) { g.x += v[e].x; g.y += v[e].y; g.z += v[e].z; g.w += v[e].w; }
    if (mask.x <= 0.f) g.x = 0.f;
    if (mask.y <= 0.f) g.y = 0.f;
    if (mask.z <= 0.f) g.z = 0.f;
    if (mask.w <= 0.f) g.w = 0.f;
    if (maskprev) {
      const uchar4 mk = reinterpret_cast<const uchar4*>(maskprev)[idx];
      g.x = mk.x ? g.x * mscale : 0.f; g.y = mk.y ? g.y * mscale : 0.f;
      g.z = mk.z ? g.z * mscale : 0.f; g.w = mk.w ? g.w * mscale : 0.f;
    }
    reinterpret_cast<uint2*>(dCprev)[idx] = make_uint2(pack_bf16x2(g.x, g.y), pack_bf16x2(g.z, g.w));
    if (g.x != 0.f) atomicAdd(&dbs[c4 * 4], g.x);
    if (g.y != 0.f) atomicAdd(&dbs[c4 * 4 + 1], g.y);
    if (g.z != 0.f) atomicAdd(&dbs[c4 * 4 + 2], g.z);
    if (g.w != 0.f) atomicAdd(&dbs[c4 * 4 + 3], g.w);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Ci; c += 256)
    if (dbs[c] != 0.f) atomicAdd(db + c, dbs[c]);
}

// Any tap count (runtime loops): the TIMIT recipes' second layer [*, 5, 32, 1] has 5 x 32 taps per
// input pixel, far beyond the unrolled instantiations above.  The inner loop over j is unrolled by
// 4 with the loads issued before their use, so 4 loads are in flight per thread.
__global__ void __launch_bounds__(256)
col2im_relu_generic_kernel(const float* __restrict__ dA, long long ldA,
                           const float* __restrict__ Pprev,
                           const unsigned char* __restrict__ maskprev, float mscale,
                           bf16* __restrict__ dCprev, float* __restrict__ db, int B, int Ti, int Fi,
                           int Ci, int kh, int kw, int s, int To, int Fo) {
  extern __shared__ float dbs[];
  for (int c = threadIdx.x; c < Ci; c += 256) dbs[c] = 0.f;
  __syncthreads();
  const long long total = (long long)B * Ti * Fi * Ci;
  for (long long idx = blockIdx.x * 256LL + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * 256) {
    const int ci = (int)(idx % Ci);
    const int px = (int)(idx / Ci);
    const int fi = px % Fi;
    const int bt = px / Fi;
    const int ti = bt % Ti;
    const int b = bt / Ti;
    const float mask = __ldg(Pprev + idx);
    float g = 0.f;
    if (mask > 0.f) {
      for (int i = ti % s; i < kh && i <= ti; i += s) {
        const int t = (ti - i) / s;
        if (t >= To) continue;
        const float* rowp = dA + ((long long)b * To + t) * Fo * ldA + (long long)i * kw * Ci + ci;
        int j = fi % s;
        for (; j + 3 * s < kw && j + 3 * s <= fi; j += 4 * s) {
          float v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int f = (fi - j - u * s) / s;
            v[u] = f < Fo ? __ldcs(rowp + (long long)f * ldA + (j + u * s) * Ci) : 0.f;
          }
          g += (v[0] + v[1]) + (v[2] + v[3]);
        }
        for (; j < kw && j <= fi; j += s) {
          const int f = (fi - j) / s;
          if (f < Fo) g += __ldcs(rowp + (long long)f * ldA + j * Ci);
        }
      }
      if (maskprev) g = maskprev[idx] ? g * mscale : 0.f;
    }
    dCprev[idx] = __float2bfloat16_rn(g);
    if (g != 0.f) atomicAdd(&dbs[ci], g);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Ci; c += 256)
    if (dbs[c] != 0.f) atomicAdd(db + c, dbs[c]);
}

static int grid_for(long long total) {
  long long g = (total + 255) / 256;
  const long long cap = (long long)device_sm_count() * 16;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace sb

using namespace sb;

extern "C" int sb_conv_im2col(const float* src, const void* mask_u8, float mscale,
                              void* dst_bf16, int B,
                              int Ti, int Fi, int Ci, int kh, int kw, int stride, int Kp,
                              int relu, void* stream_) {
  if (!src || !dst_bf16 || B <= 0 || Ci <= 0 || kh <= 0 || kw <= 0 || stride <= 0)
    return SB_ERR_INVALID;
  const int To = (Ti - kh) / stride + 1, Fo = (Fi - kw) / stride + 1;
  if (To <= 0 || Fo <= 0 || Kp < kh * kw * Ci) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long total = (long long)B * To * Fo * (Kp / 8);
  im2col_kernel<<<grid_for(total), 256, 0, stream>>>(
      src, reinterpret_cast<const unsigned char*>(mask_u8), mscale,
      reinterpret_cast<bf16*>(dst_bf16), B, Ti, Fi,
      Ci, kh, kw, stride, To, Fo, Kp, relu);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_conv_relu_to_bct(const float* C, const void* mask_u8, float mscale,
                                   float* out, int B,
                                   int To, int Fo, int Co, void* stream_) {
  if (!C || !out || B <= 0 || To <= 0 || Fo <= 0 || Co <= 0) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  relu_to_bct_kernel<<<grid_for((long long)B * To * Fo * Co), 256, 0, stream>>>(
      C, reinterpret_cast<const unsigned char*>(mask_u8), mscale, out, B, To, Fo, Co);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_conv_dtop(const float* dY, const float* C, const void* mask_u8, float mscale,
                            void* dC_bf16,
                            float* db, int B, int To, int Fo, int Co, void* stream_) {
  if (!dY || !C || !dC_bf16 || !db || B <= 0 || To <= 0 || Fo <= 0 || Co <= 0)
    return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  dconv_top_kernel<<<grid_for((long long)B * To * Fo * Co), 256, Co * sizeof(float), stream>>>(
      dY, C, reinterpret_cast<const unsigned char*>(mask_u8), mscale,
      reinterpret_cast<bf16*>(dC_bf16), db, B, To, Fo, Co);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_conv_col2im_relu(const float* dA, long long ldA, const float* Pprev,
                                   const void* maskprev_u8, float mscale, void* dCprev_bf16,
                                   float* db, int B,
                                   int Ti, int Fi, int Ci, int kh, int kw, int stride,
                                   void* stream_) {
  if (!dA || !Pprev || !dCprev_bf16 || !db || B <= 0) return SB_ERR_INVALID;
  const int To = (Ti - kh) / stride + 1, Fo = (Fi - kw) / stride + 1;
  if (To <= 0 || Fo <= 0) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int ni = (kh + stride - 1) / stride, nj = (kw + stride - 1) / stride;
  const int g = grid_for((long long)B * Ti * Fi * Ci);
  bf16* out = reinterpret_cast<bf16*>(dCprev_bf16);
  const size_t sm = Ci * sizeof(float);
  if ((long long)B * Ti * Fi >= (1LL << 31)) return SB_ERR_UNSUPPORTED;
#define SB_C2I(I, J)                                                                              \
  col2im_relu_kernel<I, J><<<g, 256, sm, stream>>>(                                                \
      dA, ldA, Pprev, reinterpret_cast<const unsigned char*>(maskprev_u8), mscale, out, db, B, Ti,  \
      Fi, Ci, kh, kw,                                                                                 \
      stride, To, Fo)
  // four channels per thread when the layout allows 16-byte tap loads
  const bool v4 = (Ci % 4 == 0) && (ldA % 4 == 0) && ((reinterpret_cast<uintptr_t>(dA) & 15) == 0) &&
                  ((reinterpret_cast<uintptr_t>(Pprev) & 15) == 0) &&
                  ((reinterpret_cast<uintptr_t>(dCprev_bf16) & 7) == 0) &&
                  (!maskprev_u8 || (reinterpret_cast<uintptr_t>(maskprev_u8) & 3) == 0);
  const int g4 = grid_for((long long)B * Ti * Fi * (Ci / 4));
#define SB_C2I4(I, J)                                                                             \
  col2im_relu_v4_kernel<I, J><<<g4, 256, sm, stream>>>(                                            \
      dA, ldA, Pprev, reinterpret_cast<const unsigned char*>(maskprev_u8), mscale, out, db, B, Ti,  \
      Fi, Ci, kh, kw, stride, To, Fo)
  if (v4 && ni <= 2 && nj <= 2) SB_C2I4(2, 2);
  else if (v4 && ni <= 3 && nj <= 4) SB_C2I4(3, 4);
  else if (ni <= 2 && nj <= 2) SB_C2I(2, 2);
  else if (ni <= 3 && nj <= 4) SB_C2I(3, 4);
  else if (ni <= 5 && nj <= 8) SB_C2I(5, 8);
  else
    col2im_relu_generic_kernel<<<g, 256, sm, stream>>>(
        dA, ldA, Pprev, reinterpret_cast<const unsigned char*>(maskprev_u8), mscale, out, db, B, Ti,
        Fi, Ci, kh, kw, stride, To, Fo);
#undef SB_C2I
#undef SB_C2I4
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

// ================================================================================================
// Direct convolution of the layers past the first: no patch matrix, no patch gradient in HBM.
//
// Each CTA stages the input footprint of its tile in shared memory and runs the contraction on
// mma.sync.m16n8k16 (bf16 in, fp32 accumulate), each tap (i, j) being an address offset into the
// footprint.  N = Co (or Ci) is a few dozen channels, far too narrow for wgmma, and every pass is
// bound by HBM bytes, not by the tensor pipe.
//   sb_conv_fwd_direct     C[m][co] = bias + sum_(i,j,ci) act * W     (W resident in smem)
//   sb_conv_dgrad_direct   dCprev = mask(sum over the taps of each stride phase of dC * W),
//                          fused with the ReLU / dropout masks of the layer below and its db
//   sb_conv_wgrad_direct   dW^T[(i,j,ci)][co] += sum_pixels act * dC  (split over pixel tiles,
//                          fp32 atomics across CTAs, as the split-K GEMM does)
// Activations are staged exactly as im2col_kernel makes A (ReLU, then the dropout keep-byte times
// mscale, then bf16 rounding), so the operands are bit-identical to the im2col path's; only the
// fp32 summation order differs.  Every output element is summed in one fixed order (the k-chunk
// loop below), independent of the batch, the length and the pixel's place in the tile.
// ================================================================================================
namespace sb {

static constexpr int kFwdThreads = 512;        // forward: 16 warps, one CTA per SM
static constexpr int kWgradThreads = 256;      // weight gradient: 8 warps, one CTA per SM
static constexpr int kDgradThreads = 256;      // data gradient: two CTAs per SM
static constexpr int kWgradChunks = 10;        // 16-row k-chunks of dW^T per warp (wgrad)
static constexpr int kSmemTwoPerSM = 110 * 1024;
static constexpr int kSmemMax = 227 * 1024;

SB_DEVINL void ldsm_x4(uint32_t (&r)[4], const bf16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
SB_DEVINL void ldsm_x4_t(uint32_t (&r)[4], const bf16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
SB_DEVINL void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 "
               "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// 16-byte async copy; src_bytes = 0 fills the 16 bytes with zeros
SB_DEVINL void cp_async16(void* dst, const void* src, int src_bytes = 16) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n"
               ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
SB_DEVINL void cp_async4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
SB_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
SB_DEVINL void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// Geometry of one layer and of its tiles; a tile is TT output rows (all Fo columns) of one
// utterance, so its pixels are the contiguous rows [(b*To + t0)*Fo, +TT*Fo) of C.
struct DirectGeom {
  int B, Ti, Fi, Ci, Co, kh, kw, s, To, Fo;
  int K, nkc;            // K = kh*kw*Ci, nkc = ceil(K / 16)
  int CiS, CoS;          // smem pixel strides (bf16): 16-byte rows for ldmatrix
  int Fu;                // footprint columns (s*(Fo-1) + kw)
  int FuS;               // smem positions per footprint row: s phases of ceil(Fu/s) columns
  int TT, R, npix;       // forward / wgrad tile: output rows, footprint rows, pixels
  int TQ, namax, ncmax, NR, NCOL, Qf, nkcp;   // dgrad tile (see conv_dgrad_direct_kernel)
};

// The activation footprint of output rows [t0, t0+TT) of utterance b is input rows s*t0 ..
// s*t0+R-1 (those < Ti), columns 0 .. Fu-1: each row one contiguous run of Fu*Ci floats.  It is
// copied raw (f32, and the keep-bytes) with cp.async while the previous tile computes, then
// converted in shared memory as im2col_kernel converts A (ReLU, dropout, bf16).  Each converted
// row stores its columns by stride phase (column u at (u % s)*ceil(Fu/s) + u/s), so that the
// pixels of consecutive output columns, which ldmatrix reads together, are adjacent
// (CiS*2 = 16 bytes times an odd number apart: no bank conflicts).
SB_DEVINL int act_rows(const DirectGeom& g, int t0) { return min(g.R, g.Ti - g.s * t0); }

SB_DEVINL void issue_act(float* raw, unsigned char* rawm, const float* __restrict__ P,
                         const unsigned char* __restrict__ mask, const DirectGeom& g, int b,
                         int t0) {
  const int run4 = g.Fu * g.Ci >> 2;                  // 16-byte pieces per footprint row
  const int rows = act_rows(g, t0);
  const long long row0 = ((long long)b * g.Ti + (long long)g.s * t0) * g.Fi * g.Ci;
  for (int e = threadIdx.x; e < run4; e += blockDim.x)
    for (int r = 0; r < rows; ++r) {
      const long long off = row0 + (long long)r * g.Fi * g.Ci + 4 * e;
      cp_async16(raw + 4 * (r * run4 + e), P + off);
      if (mask) cp_async4(rawm + 4 * (r * run4 + e), mask + off);
    }
}

SB_DEVINL void convert_act(bf16* fp, const float* raw, const unsigned char* rawm, bool masked,
                           float mscale, const DirectGeom& g, int t0) {
  const int c4n = g.Ci >> 2, run4 = g.Fu * c4n;
  const int rows = act_rows(g, t0);
  for (int e = threadIdx.x; e < run4; e += blockDim.x) {
    const int u = e / c4n, c4 = e - u * c4n;          // column, channel quad
    const int q = u / g.s;
    const int dst = ((u - q * g.s) * (g.FuS / g.s) + q) * g.CiS + c4 * 4;
    for (int r = 0; r < rows; ++r) {
      const int idx = r * run4 + e;
      const float4 v = reinterpret_cast<const float4*>(raw)[idx];
      float x[4] = {fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f)};
      if (masked) {
        const uint32_t mk = reinterpret_cast<const uint32_t*>(rawm)[idx];
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = ((mk >> (8 * k)) & 0xff) ? x[k] * mscale : 0.f;
      }
      *reinterpret_cast<uint2*>(fp + r * g.FuS * g.CiS + dst) =
          make_uint2(pack_bf16x2(x[0], x[1]), pack_bf16x2(x[2], x[3]));
    }
  }
}

// Footprint offsets of the two 8-wide halves of k-chunk kc (K order (i, j, ci), Ci % 8 == 0);
// a half past K points at offset 0 (finite data; the weights there are zero / it is skipped).
SB_DEVINL int2 act_chunk_offsets(const DirectGeom& g, int kc) {
  int o[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = kc * 16 + 8 * h;
    o[h] = 0;
    if (k < g.K) {
      const int tap = k / g.Ci, ci = k - tap * g.Ci;
      const int i = tap / g.kw, j = tap - i * g.kw;
      o[h] = (i * g.FuS + (j % g.s) * (g.FuS / g.s) + j / g.s) * g.CiS + ci;
    }
  }
  return make_int2(o[0], o[1]);
}

// Footprint offset of output pixel p (< npix) of the tile.
SB_DEVINL int act_pixel_base(const DirectGeom& g, int p) {
  const int tl = p / g.Fo, f = p - tl * g.Fo;
  return (tl * g.s * g.FuS + f) * g.CiS;
}

// ---- forward ------------------------------------------------------------------------------------
// smem: W [Co][nkc*16 + 8] bf16 | footprint [R][FuS][CiS] bf16 | raw footprint [R][Fu*Ci] f32 |
//       k-chunk offsets [nkc] int2 | raw keep-bytes [R][Fu*Ci]
__global__ void __launch_bounds__(kFwdThreads, 1)
conv_fwd_direct_kernel(const float* __restrict__ P, const unsigned char* __restrict__ mask,
                       float mscale, const bf16* __restrict__ Wp, int ldw,
                       const float* __restrict__ bias, float* __restrict__ C, DirectGeom g) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int kWarps = kFwdThreads / 32;
  const int KS = g.nkc * 16 + 8;
  bf16* Ws = reinterpret_cast<bf16*>(smem);
  bf16* fp = Ws + (size_t)g.Co * KS;
  float* raw = reinterpret_cast<float*>(fp + (size_t)g.R * g.FuS * g.CiS);
  int2* tab = reinterpret_cast<int2*>(raw + (size_t)g.R * g.Fu * g.Ci);
  unsigned char* rawm = reinterpret_cast<unsigned char*>(tab + ((g.nkc + 1) & ~1));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ntt = (g.To + g.TT - 1) / g.TT, ntiles = g.B * ntt;
  int tile = blockIdx.x;
  if (tile < ntiles) issue_act(raw, rawm, P, mask, g, tile / ntt, (tile % ntt) * g.TT);
  cp_async_commit();
  // resident weights, zero past K
  const int k8n = KS >> 3, K8 = g.K >> 3;
  for (int idx = threadIdx.x; idx < g.Co * k8n; idx += kFwdThreads) {
    const int co = idx / k8n, k8 = idx - co * k8n;
    uint4 w = make_uint4(0, 0, 0, 0);
    if (k8 < K8) w = __ldg(reinterpret_cast<const uint4*>(Wp + (size_t)co * ldw) + k8);
    reinterpret_cast<uint4*>(Ws + (size_t)co * KS)[k8] = w;
  }
  for (int kc = threadIdx.x; kc < g.nkc; kc += kFwdThreads) tab[kc] = act_chunk_offsets(g, kc);

  const int MT2 = (g.npix + 31) >> 5, NQ = (g.Co + 31) >> 5;
  const int g8 = lane >> 2, t4 = lane & 3;
  for (; tile < ntiles; tile += gridDim.x) {
    const int b = tile / ntt, t0 = (tile - b * ntt) * g.TT;
    cp_async_wait_all();
    __syncthreads();                       // raw footprint landed; the last tile's reads are done
    convert_act(fp, raw, rawm, mask != nullptr, mscale, g, t0);
    __syncthreads();
    const int next = tile + gridDim.x;     // the next footprint streams in while this one computes
    if (next < ntiles) issue_act(raw, rawm, P, mask, g, next / ntt, (next % ntt) * g.TT);
    cp_async_commit();
    const int npv = min(g.TT, g.To - t0) * g.Fo;      // valid pixels of this tile
    // warp item: 32 pixels (two m16 tiles) x 32 channels (four n8 tiles); the fragments of
    // chunk kc+1 are loaded while chunk kc multiplies
    for (int item = warp; item < MT2 * NQ; item += kWarps) {
      const int mp = item / NQ, nq = item - mp * NQ;
      const bf16* arow[2];
#pragma unroll
      for (int m = 0; m < 2; ++m)
        arow[m] = fp + act_pixel_base(
            g, min(mp * 32 + m * 16 + (lane & 7) + 8 * ((lane >> 3) & 1), npv - 1));
      const int ahalf = lane >> 4;
      const bf16* brow[2];
#pragma unroll
      for (int n = 0; n < 2; ++n)
        brow[n] = Ws + (size_t)min(nq * 32 + n * 16 + (lane & 7) + 8 * (lane >> 4), g.Co - 1) * KS +
                  8 * ((lane >> 3) & 1);
      float acc[2][4][4] = {};
      uint32_t af[2][2][4], bfr[2][2][4];
      auto load = [&](int buf, int kc) {
        const int2 o = tab[kc];
        const int off = ahalf ? o.y : o.x;
        ldsm_x4(af[buf][0], arow[0] + off);
        ldsm_x4(af[buf][1], arow[1] + off);
        ldsm_x4(bfr[buf][0], brow[0] + kc * 16);
        ldsm_x4(bfr[buf][1], brow[1] + kc * 16);
      };
      auto mma8 = [&](int buf) {
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int n = 0; n < 4; ++n)
            mma_bf16(acc[m][n], af[buf][m], bfr[buf][n >> 1][2 * (n & 1)],
                     bfr[buf][n >> 1][2 * (n & 1) + 1]);
      };
      load(0, 0);
      int kc = 0;
      for (; kc + 2 <= g.nkc; kc += 2) {
        load(1, kc + 1);
        mma8(0);
        if (kc + 2 < g.nkc) load(0, kc + 2);
        mma8(1);
      }
      if (kc < g.nkc) mma8(0);
      float* crow = C + ((long long)b * g.To + t0) * g.Fo * g.Co;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const int co = nq * 32 + n * 8 + 2 * t4;
        if (co >= g.Co) continue;
        const float b0 = __ldg(bias + co), b1 = __ldg(bias + co + 1);
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int p = mp * 32 + m * 16 + g8 + 8 * h;
            if (p < npv)
              *reinterpret_cast<float2*>(crow + (long long)p * g.Co + co) =
                  make_float2(acc[m][n][2 * h] + b0, acc[m][n][2 * h + 1] + b1);
          }
      }
    }
  }
  cp_async_wait_all();
}

// ---- weight gradient ----------------------------------------------------------------------------
// dW^T[k][co] += sum_p act[p][k] dC[p][co]: the M dimension of the mma is k (16-row chunks), N is
// co, and the contraction runs over the tile's pixels, both operands read with ldmatrix.trans.
// Warp w of k-group blockIdx.y owns chunks (blockIdx.y*8 + w)*10 + u and keeps them in registers
// across all its tiles.
// smem: footprint | raw footprint | raw dC rows [np16*16][Co] | dC rows [np16*16][CoS] bf16 |
//       raw keep-bytes
__global__ void __launch_bounds__(kWgradThreads, 1)
conv_wgrad_direct_kernel(const float* __restrict__ P, const unsigned char* __restrict__ mask,
                         float mscale, const bf16* __restrict__ dC, float* __restrict__ dWT,
                         DirectGeom g) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int kWarps = kWgradThreads / 32;
  const int np16 = (g.npix + 15) >> 4;
  bf16* fp = reinterpret_cast<bf16*>(smem);
  float* raw = reinterpret_cast<float*>(fp + (size_t)g.R * g.FuS * g.CiS);
  bf16* rawdc = reinterpret_cast<bf16*>(raw + (size_t)g.R * g.Fu * g.Ci);
  bf16* ds = rawdc + (size_t)np16 * 16 * g.Co;
  unsigned char* rawm = reinterpret_cast<unsigned char*>(ds + (size_t)np16 * 16 * g.CoS);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ntt = (g.To + g.TT - 1) / g.TT, ntiles = g.B * ntt;
  const int c8n = g.Co >> 3;
  // raw copies of a tile: the footprint and its dC rows (contiguous: npv*Co bf16)
  auto issue = [&](int t) {
    const int b = t / ntt, t0 = (t - b * ntt) * g.TT;
    issue_act(raw, rawm, P, mask, g, b, t0);
    const int npv = min(g.TT, g.To - t0) * g.Fo;
    const bf16* src = dC + ((long long)b * g.To + t0) * g.Fo * g.Co;
    for (int idx = threadIdx.x; idx < npv * c8n; idx += kWgradThreads)
      cp_async16(rawdc + 8 * idx, src + 8 * idx);
  };
  int tile = blockIdx.x;
  if (tile < ntiles) issue(tile);
  cp_async_commit();
  const int kc0 = (blockIdx.y * kWarps + warp) * kWgradChunks;
  const int ahalf = (lane >> 3) & 1;
  int aoff[kWgradChunks];                          // this lane's footprint offset of each chunk
#pragma unroll
  for (int u = 0; u < kWgradChunks; ++u) {
    const int2 o = act_chunk_offsets(g, min(kc0 + u, g.nkc - 1));
    aoff[u] = ahalf ? o.y : o.x;
  }
  const int NT = g.Co >> 3;
  float acc[kWgradChunks][4][4] = {};
  for (; tile < ntiles; tile += gridDim.x) {
    const int b = tile / ntt, t0 = (tile - b * ntt) * g.TT;
    cp_async_wait_all();
    __syncthreads();
    convert_act(fp, raw, rawm, mask != nullptr, mscale, g, t0);
    const int npv = min(g.TT, g.To - t0) * g.Fo;
    for (int idx = threadIdx.x; idx < np16 * 16 * c8n; idx += kWgradThreads) {
      const int p = idx / c8n, c8 = idx - p * c8n;
      uint4 v = make_uint4(0, 0, 0, 0);                // pixels past the tile contribute 0
      if (p < npv) v = reinterpret_cast<const uint4*>(rawdc)[idx];
      *reinterpret_cast<uint4*>(ds + p * g.CoS + c8 * 8) = v;
    }
    __syncthreads();
    if (tile + gridDim.x < ntiles) issue(tile + gridDim.x);
    cp_async_commit();
    if (kc0 >= g.nkc) continue;
    for (int pc = 0; pc < np16; ++pc) {
      // B fragments of every n-tile: dC rows pc*16 .. +15
      uint32_t bf[2][4];
      const int pb = pc * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        const int co = min(np * 16 + 8 * (lane >> 4), g.Co - 8);
        if (np * 16 < g.Co) ldsm_x4_t(bf[np], ds + pb * g.CoS + co);
      }
      const int pa = min(pc * 16 + (lane & 7) + 8 * (lane >> 4), npv - 1);
      const bf16* arow = fp + act_pixel_base(g, pa);
      uint32_t a[2][4];
      ldsm_x4_t(a[0], arow + aoff[0]);
#pragma unroll
      for (int u = 0; u < kWgradChunks; ++u) {     // chunks past nkc repeat the last; unused
        if (u + 1 < kWgradChunks) ldsm_x4_t(a[(u + 1) & 1], arow + aoff[u + 1]);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
          if (nt < NT)
            mma_bf16(acc[u][nt], a[u & 1], bf[nt >> 1][2 * (nt & 1)], bf[nt >> 1][2 * (nt & 1) + 1]);
      }
    }
  }
  cp_async_wait_all();
  const int g8 = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int u = 0; u < kWgradChunks; ++u) {
    const int kc = kc0 + u;
    if (kc >= g.nkc) break;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      if (nt >= NT) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = kc * 16 + g8 + 8 * h;
        if (k >= g.K) continue;
        float* d = dWT + (long long)k * g.Co + nt * 8 + 2 * t4;
        atomicAdd(d, acc[u][nt][2 * h]);
        atomicAdd(d + 1, acc[u][nt][2 * h + 1]);
      }
    }
  }
}

// ---- data gradient ------------------------------------------------------------------------------
// Input pixel (ti, fi) = (s*qt + pi, s*qf + pj) of stride phase (pi, pj) receives the taps
// i = pi + a*s, j = pj + c*s from output pixel (qt - a, qf - c): per phase a dense contraction
// over K = na*nc*Co, K order (a, c, co), A = the staged dC footprint, B = W transposed to
// [ci][(i, j, co)] in smem.  A tile is TQ quotient rows qt (s*TQ input rows, all columns); each
// input pixel is written by exactly one thread, no atomics on dCprev.
// smem: W^T [Ci][kh*kw*Co + 8] bf16 | dC [NR][NCOL][CoS] bf16 (zero outside the map) |
//       per-phase chunk offsets [s*s][nkcp] int4 (A half 0, A half 1, B half 0, B half 1) | db [Ci]
__global__ void __launch_bounds__(kDgradThreads, 2)
conv_dgrad_direct_kernel(const bf16* __restrict__ dC, const bf16* __restrict__ Wp, int ldw,
                         const float* __restrict__ Pprev, const unsigned char* __restrict__ maskprev,
                         float mscale, bf16* __restrict__ dCp, float* __restrict__ db, DirectGeom g) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int kWarps = kDgradThreads / 32;
  const int K2 = g.kh * g.kw * g.Co, KS = K2 + 8;
  bf16* Wt = reinterpret_cast<bf16*>(smem);
  bf16* ds = Wt + (size_t)g.Ci * KS;
  int4* tab = reinterpret_cast<int4*>(ds + (size_t)g.NR * g.NCOL * g.CoS);
  float* dbs = reinterpret_cast<float*>(tab + g.s * g.s * g.nkcp);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s = g.s;
  for (int idx = threadIdx.x; idx < g.Co * g.K; idx += kDgradThreads) {
    const int co = idx / g.K, k = idx - co * g.K;
    const int tap = k / g.Ci, ci = k - tap * g.Ci;
    Wt[(size_t)ci * KS + tap * g.Co + co] = Wp[(size_t)co * ldw + k];
  }
  for (int idx = threadIdx.x; idx < g.Ci * 8; idx += kDgradThreads)
    Wt[(size_t)(idx >> 3) * KS + K2 + (idx & 7)] = __float2bfloat16_rn(0.f);
  for (int idx = threadIdx.x; idx < s * s * g.nkcp; idx += kDgradThreads) {
    const int ph = idx / g.nkcp, kc = idx - ph * g.nkcp;
    const int pi = ph / s, pj = ph - pi * s;
    const int na = pi < g.kh ? (g.kh - pi + s - 1) / s : 0;
    const int nc = pj < g.kw ? (g.kw - pj + s - 1) / s : 0;
    int o[4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = kc * 16 + 8 * h;
      o[h] = 0;
      o[2 + h] = K2;                                   // zero weights
      if (k < na * nc * g.Co) {
        const int ac = k / g.Co, co = k - ac * g.Co;
        const int a = ac / nc, c = ac - a * nc;
        o[h] = -(a * g.NCOL + c) * g.CoS + co;
        o[2 + h] = ((pi + a * s) * g.kw + pj + c * s) * g.Co + co;
      }
    }
    tab[idx] = make_int4(o[0], o[1], o[2], o[3]);
  }
  for (int c = threadIdx.x; c < g.Ci; c += kDgradThreads) dbs[c] = 0.f;

  const int nqt = (g.Ti + s - 1) / s;                  // quotient rows qt of the input
  const int ntq = (nqt + g.TQ - 1) / g.TQ;
  const int NQ = (g.Ci + 31) >> 5;
  const int c8n = g.Co >> 3;
  const int g8 = lane >> 2, t4 = lane & 3;
  for (int tile = blockIdx.x; tile < g.B * ntq; tile += gridDim.x) {
    const int b = tile / ntq, q0 = (tile - b * ntq) * g.TQ;
    __syncthreads();
    const int tlo = q0 - (g.namax - 1), flo = -(g.ncmax - 1);
    for (int e = threadIdx.x; e < g.NCOL * c8n; e += kDgradThreads) {
      const int col = e / c8n, c8 = e - col * c8n;
      const int f = flo + col;
      for (int r = 0; r < g.NR; ++r) {
        const int t = tlo + r;
        const bool in = t >= 0 && t < g.To && f >= 0 && f < g.Fo;
        cp_async16(ds + (r * g.NCOL + col) * g.CoS + c8 * 8,
                   in ? dC + (((long long)b * g.To + t) * g.Fo + f) * g.Co + c8 * 8 : dC,
                   in ? 16 : 0);
      }
    }
    cp_async_wait_all();
    __syncthreads();
    // work items: (phase, 16-pixel tile, 32 channels), enumerated phase by phase
    int first = 0;
    for (int ph = 0; ph < s * s; ++ph) {
      const int pi = ph / s, pj = ph - pi * s;
      const int nqf = (g.Fi - pj + s - 1) / s;
      const int npx = g.TQ * nqf;
      const int nitems = ((npx + 15) >> 4) * NQ;
      const int4* ptab = tab + ph * g.nkcp;
      const int na = pi < g.kh ? (g.kh - pi + s - 1) / s : 0;
      const int nc = pj < g.kw ? (g.kw - pj + s - 1) / s : 0;
      const int nkc = (na * nc * g.Co + 15) >> 4;
      for (int item = (warp - first % kWarps + kWarps) % kWarps; item < nitems; item += kWarps) {
        const int mt = item / NQ, nq = item - mt * NQ;
        // the epilogue's operands (ReLU and dropout masks of the layer below) are loaded first,
        // so that their latency hides behind the contraction
        long long eidx[2];
        float2 pv[2][4];
        uint32_t mk[2][4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int p = mt * 16 + g8 + 8 * h;
          const int tq = p / nqf, qf = p - tq * nqf;
          const int ti = (q0 + tq) * s + pi, fi = qf * s + pj;
          eidx[h] = (p < npx && ti < g.Ti) ? (((long long)b * g.Ti + ti) * g.Fi + fi) * g.Ci : -1;
#pragma unroll
          for (int n = 0; n < 4; ++n) {
            const int ci = nq * 32 + n * 8 + 2 * t4;
            pv[h][n] = make_float2(0.f, 0.f);
            mk[h][n] = 0x0101u;
            if (eidx[h] >= 0 && ci < g.Ci) {
              pv[h][n] = __ldg(reinterpret_cast<const float2*>(Pprev + eidx[h] + ci));
              if (maskprev)
                mk[h][n] = __ldg(reinterpret_cast<const unsigned short*>(maskprev + eidx[h] + ci));
            }
          }
        }
        const int pa = min(mt * 16 + (lane & 7) + 8 * ((lane >> 3) & 1), npx - 1);
        const int tqa = pa / nqf, qfa = pa - tqa * nqf;
        const bf16* arow = ds + ((tqa + g.namax - 1) * g.NCOL + qfa + g.ncmax - 1) * g.CoS;
        const int ahalf = lane >> 4;
        const bf16* brow[2];
#pragma unroll
        for (int n = 0; n < 2; ++n)
          brow[n] = Wt + (size_t)min(nq * 32 + n * 16 + (lane & 7) + 8 * (lane >> 4), g.Ci - 1) * KS;
        const int bhalf = (lane >> 3) & 1;
        float acc[4][4] = {};
        uint32_t af[2][4], bfr[2][2][4];
        auto load = [&](int buf, int kc) {
          const int4 o = ptab[kc];
          ldsm_x4(af[buf], arow + (ahalf ? o.y : o.x));
          const int bo = bhalf ? o.w : o.z;
          ldsm_x4(bfr[buf][0], brow[0] + bo);
          ldsm_x4(bfr[buf][1], brow[1] + bo);
        };
        auto mma4 = [&](int buf) {
#pragma unroll
          for (int n = 0; n < 4; ++n)
            mma_bf16(acc[n], af[buf], bfr[buf][n >> 1][2 * (n & 1)], bfr[buf][n >> 1][2 * (n & 1) + 1]);
        };
        if (nkc > 0) load(0, 0);
        int kc = 0;
        for (; kc + 2 <= nkc; kc += 2) {
          load(1, kc + 1);
          mma4(0);
          if (kc + 2 < nkc) load(0, kc + 2);
          mma4(1);
        }
        if (kc < nkc) mma4(0);
        // epilogue of col2im_relu: ReLU mask (Pprev > 0), dropout of the layer below, bf16, db
        float dsum[4][2] = {};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (eidx[h] < 0) continue;
#pragma unroll
          for (int n = 0; n < 4; ++n) {
            const int ci = nq * 32 + n * 8 + 2 * t4;
            if (ci >= g.Ci) continue;
            float v0 = acc[n][2 * h], v1 = acc[n][2 * h + 1];
            if (pv[h][n].x <= 0.f) v0 = 0.f;
            else if (maskprev) v0 = (mk[h][n] & 0xff) ? v0 * mscale : 0.f;
            if (pv[h][n].y <= 0.f) v1 = 0.f;
            else if (maskprev) v1 = (mk[h][n] >> 8) ? v1 * mscale : 0.f;
            *reinterpret_cast<uint32_t*>(dCp + eidx[h] + ci) = pack_bf16x2(v0, v1);
            dsum[n][0] += v0;
            dsum[n][1] += v1;
          }
        }
#pragma unroll
        for (int n = 0; n < 4; ++n)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v = dsum[n][e];
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            const int ci = nq * 32 + n * 8 + 2 * t4 + e;
            if (g8 == 0 && ci < g.Ci && v != 0.f) atomicAdd(&dbs[ci], v);
          }
      }
      first += nitems;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < g.Ci; c += kDgradThreads)
    if (dbs[c] != 0.f) atomicAdd(db + c, dbs[c]);
}

// ---- plans: tile sizes and shared memory; false outside the direct kernels' domain ----------------
static bool direct_geom(DirectGeom& g, int B, int Ti, int Fi, int Ci, int Co, int kh, int kw, int s) {
  g = DirectGeom{};
  g.B = B; g.Ti = Ti; g.Fi = Fi; g.Ci = Ci; g.Co = Co; g.kh = kh; g.kw = kw; g.s = s;
  if (Ci < 8 || Ci % 8 || Co < 8 || Co % 8 || Co > 32 || kh <= 0 || kw <= 0 || s <= 0 ||
      Ti < kh || Fi < kw)
    return false;
  g.To = (Ti - kh) / s + 1;
  g.Fo = (Fi - kw) / s + 1;
  g.K = kh * kw * Ci;
  g.nkc = (g.K + 15) / 16;
  g.CiS = Ci + 8;
  g.CoS = Co + 8;
  g.Fu = s * (g.Fo - 1) + kw;
  g.FuS = s * ((g.Fu + s - 1) / s);
  g.namax = (kh + s - 1) / s;
  g.ncmax = (kw + s - 1) / s;
  g.Qf = (Fi - 1) / s + 1;
  g.NCOL = g.Qf + g.ncmax - 1;
  g.nkcp = (g.namax * g.ncmax * Co + 15) / 16;
  return true;
}

// footprint (bf16), its raw copy (f32 and keep-bytes) and the k-chunk offsets
static size_t act_smem(const DirectGeom& g, int TT) {
  const size_t R = (size_t)((TT - 1) * g.s + g.kh);
  return R * g.FuS * g.CiS * 2 + R * g.Fu * g.Ci * 5 + (size_t)((g.nkc + 1) & ~1) * 8;
}
static size_t fwd_smem(const DirectGeom& g, int TT) {
  return (size_t)g.Co * (g.nkc * 16 + 8) * 2 + act_smem(g, TT);
}
static size_t wgrad_smem(const DirectGeom& g, int TT) {   // (it keeps its offsets in registers)
  return act_smem(g, TT) + (size_t)((TT * g.Fo + 15) / 16) * 16 * (g.Co + g.CoS) * 2;
}
static size_t dgrad_smem(const DirectGeom& g, int TQ) {
  return (size_t)g.Ci * (g.kh * g.kw * g.Co + 8) * 2 +
         (size_t)(TQ + g.namax - 1) * g.NCOL * g.CoS * 2 + (size_t)g.s * g.s * g.nkcp * 16 +
         (size_t)g.Ci * 4;
}

// Largest tile of at most `cap` rows within `lim` bytes of shared memory, else within one CTA's
// maximum; 0 if none fits.
template <class F>
static int pick_tile(F smem, int cap, int lim) {
  for (int l : {lim, kSmemMax})
    for (int t = cap; t >= 1; --t)
      if (smem(t) <= (size_t)l) return t;
  return 0;
}

static bool direct_plan(DirectGeom& g, int B, int Ti, int Fi, int Ci, int Co, int kh, int kw, int s,
                        int pass) {
  if (!direct_geom(g, B, Ti, Fi, Ci, Co, kh, kw, s)) return false;
  const int cap = min(8, g.To);
  if (pass == 0) g.TT = pick_tile([&](int t) { return fwd_smem(g, t); }, cap, kSmemMax);
  if (pass == 2) g.TT = pick_tile([&](int t) { return wgrad_smem(g, t); }, cap, kSmemMax);
  if (pass == 1) {
    g.TQ = pick_tile([&](int t) { return dgrad_smem(g, t); }, min(8, (Ti + s - 1) / s),
                     kSmemTwoPerSM);
    g.NR = g.TQ + g.namax - 1;
    return g.TQ > 0;
  }
  g.R = (g.TT - 1) * s + kh;
  g.npix = g.TT * g.Fo;
  return g.TT > 0;
}

// Persistent grid: as many CTAs as fit on the device at once (per k-group), at most one per tile.
template <class K>
static int launch_direct(K kernel, int threads, int groups, long long tiles, size_t smem, int& gx) {
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return SB_ERR_CUDA;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) !=
          cudaSuccess || per_sm < 1)
    return SB_ERR_CUDA;
  const long long cap = std::max(1LL, (long long)device_sm_count() * per_sm / groups);
  gx = (int)std::max(1LL, std::min(tiles, cap));
  return SB_OK;
}

}  // namespace sb

extern "C" int sb_conv_direct_ok(int Fi, int Ci, int Co, int kh, int kw, int stride) {
  DirectGeom g;
  const int Ti = kh + 7 * stride;   // the tile sizes cap at 8 rows: a longer input changes nothing
  for (int pass = 0; pass < 3; ++pass)
    if (!direct_plan(g, 1, Ti, Fi, Ci, Co, kh, kw, stride, pass)) return 0;
  return 1;
}

extern "C" int sb_conv_fwd_direct(const float* P, const void* mask_u8, float mscale,
                                  const void* Wp_bf16, int ldw, const float* bias, float* C, int B,
                                  int Ti, int Fi, int Ci, int Co, int kh, int kw, int stride,
                                  void* stream_) {
  DirectGeom g;
  if (!P || !Wp_bf16 || !bias || !C || B <= 0) return SB_ERR_INVALID;
  if (!direct_plan(g, B, Ti, Fi, Ci, Co, kh, kw, stride, 0)) return SB_ERR_UNSUPPORTED;
  if (ldw < g.K || ldw % 8 || (reinterpret_cast<uintptr_t>(Wp_bf16) & 15) ||
      (reinterpret_cast<uintptr_t>(P) & 15) || (reinterpret_cast<uintptr_t>(mask_u8) & 3))
    return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const size_t smem = fwd_smem(g, g.TT);
  const long long tiles = (long long)B * ((g.To + g.TT - 1) / g.TT);
  int gx = 0;
  const int rc = launch_direct(conv_fwd_direct_kernel, kFwdThreads, 1, tiles, smem, gx);
  if (rc != SB_OK) return rc;
  conv_fwd_direct_kernel<<<gx, kFwdThreads, smem, stream>>>(
      P, reinterpret_cast<const unsigned char*>(mask_u8), mscale,
      reinterpret_cast<const bf16*>(Wp_bf16), ldw, bias, C, g);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_conv_wgrad_direct(const float* P, const void* mask_u8, float mscale,
                                    const void* dC_bf16, float* dWT, int B, int Ti, int Fi, int Ci,
                                    int Co, int kh, int kw, int stride, void* stream_) {
  DirectGeom g;
  if (!P || !dC_bf16 || !dWT || B <= 0) return SB_ERR_INVALID;
  if (!direct_plan(g, B, Ti, Fi, Ci, Co, kh, kw, stride, 2)) return SB_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(P) & 15) || (reinterpret_cast<uintptr_t>(dC_bf16) & 15) ||
      (reinterpret_cast<uintptr_t>(mask_u8) & 3))
    return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const size_t smem = wgrad_smem(g, g.TT);
  const long long tiles = (long long)B * ((g.To + g.TT - 1) / g.TT);
  const int per_cta = (kWgradThreads / 32) * kWgradChunks;
  const int gy = (g.nkc + per_cta - 1) / per_cta;
  int gx = 0;
  const int rc = launch_direct(conv_wgrad_direct_kernel, kWgradThreads, gy, tiles, smem, gx);
  if (rc != SB_OK) return rc;
  conv_wgrad_direct_kernel<<<dim3(gx, gy), kWgradThreads, smem, stream>>>(
      P, reinterpret_cast<const unsigned char*>(mask_u8), mscale,
      reinterpret_cast<const bf16*>(dC_bf16), dWT, g);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_conv_dgrad_direct(const void* dC_bf16, const void* Wp_bf16, int ldw,
                                    const float* Pprev, const void* maskprev_u8, float mscale,
                                    void* dCprev_bf16, float* db, int B, int Ti, int Fi, int Ci,
                                    int Co, int kh, int kw, int stride, void* stream_) {
  DirectGeom g;
  if (!dC_bf16 || !Wp_bf16 || !Pprev || !dCprev_bf16 || !db || B <= 0) return SB_ERR_INVALID;
  if (!direct_plan(g, B, Ti, Fi, Ci, Co, kh, kw, stride, 1)) return SB_ERR_UNSUPPORTED;
  if (ldw < g.K || (reinterpret_cast<uintptr_t>(dC_bf16) & 15) ||
      (reinterpret_cast<uintptr_t>(Pprev) & 7) || (reinterpret_cast<uintptr_t>(dCprev_bf16) & 3) ||
      (reinterpret_cast<uintptr_t>(maskprev_u8) & 1))
    return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const size_t smem = dgrad_smem(g, g.TQ);
  const long long tiles = (long long)B * (((Ti + stride - 1) / stride + g.TQ - 1) / g.TQ);
  int gx = 0;
  const int rc = launch_direct(conv_dgrad_direct_kernel, kDgradThreads, 1, tiles, smem, gx);
  if (rc != SB_OK) return rc;
  conv_dgrad_direct_kernel<<<gx, kDgradThreads, smem, stream>>>(
      reinterpret_cast<const bf16*>(dC_bf16), reinterpret_cast<const bf16*>(Wp_bf16), ldw, Pprev,
      reinterpret_cast<const unsigned char*>(maskprev_u8), mscale,
      reinterpret_cast<bf16*>(dCprev_bf16), db, g);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
