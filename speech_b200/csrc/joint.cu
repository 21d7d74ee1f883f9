// Fused RNN-T joint: relu(fc1(x)[b,t] + fc1(pred)[b,u]) -> fc2 -> log-softmax for every lattice
// node, WITHOUT materialising the (B, T', U+1, H) intermediate.
//
// Replaces the broadcast add + ReLU + LinearND + log_softmax of Transducer.decode
// (speech/models/transducer_model.py:71-76; fc1 is shared by both streams, :73).  The reference
// builds a (B, T', U+1, H) tensor (3.2 GB at B=32, T'=247, U+1=100, H=1024) and a
// (B, T', U+1, V+1) log-probability tensor; the transducer loss reads only two entries per node
// (blank and the next label), so the training path here writes a COMPACT lattice
// lat[node] = {log p(blank), log p(label_u)} (8 bytes per node) and the hidden tensor only ever
// exists as 16 KB operand tiles in shared memory:
//   * 3 x 4 producer warps (thread = node row; the groups take the k-blocks in turn) build
//     A tiles [128 nodes x 64] bf16 of relu(fx[b,t,:] + fy[b,u,:]) straight into the wgmma
//     K-major SWIZZLE_128B layout (fx, fy: fp32 outputs of the fc1 GEMMs, L2 resident: 7.9 K
//     and 3.2 K rows);
//   * fc2's weight (V+1 <= 64 rows x H, bf16) stays resident in shared memory;
//   * one consumer warpgroup issues wgmma  D[128 x NV] += A * W2^T  (two m64 halves, fp32
//     accumulators in registers), parks the tile in shared memory and re-reads it as thread = node;
//   * the same 4 warps (thread = node) add the bias, take the log-softmax over the V+1 classes
//     in registers and write either the compact lattice (+ optionally the full log-probabilities,
//     which `infer` needs for the beam search), or - in the backward recompute pass - the
//     gradient w.r.t. the logits as bf16 rows [node][NV] from the per-arc gradients of the
//     lattice kernel:  dlogit_k = g_blank ([k = blank] - p_k) + g_label ([k = label] - p_k).
// Roofline: tensor work (2 * nodes * H * (V+1) FLOPs), in practice bound by the producers'
// shared-memory tile construction (16 KB per 64 MMA cycles).
#include "common.cuh"
#include <math.h>
#include <string.h>

#include "../../include/speech_b200.h"

namespace sb {

typedef __nv_bfloat16 bf16;

// producer groups of 4 warps: 3 for the 32-class kernel, 2 for the 64-class one (whose epilogue
// keeps 2 x 64 values per thread and would spill under the register cap of 16 warps).  The
// 64-class kernel keeps 4 ring stages so that fc2's weight (128 KB at H = 1024), the ring and the
// accumulator tile fit in the 227 KB of shared memory of one block.
template <int NV> struct JtCfg {
  static constexpr int kGroups = NV <= 32 ? 3 : 2;
  static constexpr int kPW = 4 * kGroups;              // producer warps
  static constexpr int kThreads = 32 * (kPW + 4);      // producers | consumer warpgroup
  static constexpr int kStages = NV <= 32 ? 6 : 4;
  static constexpr int kAccPitch = NV + 1;             // floats per node row of the parked tile
};

struct JointParams {
  const float* fx;      // [B*T][H]   fc1(encoder states)   (bias included)
  const float* fy;      // [B*U1][H]  fc1(prediction net)   (bias included)
  const bf16* w2;       // [V1][H]    fc2 weight
  const float* b2;      // [V1]
  const int* ymat;      // [B][U1-1]  label matrix (end-padded), label of arc (u -> u+1)
  float* lat;           // [nodes][2] {log p(blank), log p(label)}, node = (t*B + b)*U1 + u  (mode 0)
  float* lp_full;       // (B, T, U1, V1) full log-probabilities, batch-first, or null  (mode 0)
  const float* garc;    // [nodes][2] gradient w.r.t. lat                      (mode 1)
  bf16* dlogits;        // [nodes][NV] gradient w.r.t. the logits, bf16        (mode 1)
  float* db2;           // [V1] += sum over nodes of dlogits                   (mode 1)
  long long nodes;
  int B, T, U1, H, V1, blank, mode;
};

template <int NV>
__global__ void __launch_bounds__(JtCfg<NV>::kThreads, 1) joint_kernel(const JointParams p) {
  constexpr int JT_GROUPS = JtCfg<NV>::kGroups, JT_PW = JtCfg<NV>::kPW, JT_THREADS = JtCfg<NV>::kThreads;
  constexpr int JT_STAGES = JtCfg<NV>::kStages, ACC_LD = JtCfg<NV>::kAccPitch;
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H;
  const int nkb = (H + 63) / 64;
  constexpr int A_BYTES = 128 * 128;          // [128 rows][64 bf16]
  constexpr int WCHUNK = NV * 128;            // [NV rows][64 bf16]
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* a_ring = base;
  uint8_t* wtile = a_ring + JT_STAGES * A_BYTES;
  float* acc_s = reinterpret_cast<float*>(wtile + (size_t)nkb * WCHUNK);   // [128][ACC_LD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(acc_s + 128 * ACC_LD + 2);
  uint64_t* full = bars;                    // [JT_STAGES]  4 producer-warp arrivals
  uint64_t* empty = bars + JT_STAGES;       // [JT_STAGES]  1 consumer arrival
  float* bias_s = reinterpret_cast<float*>(empty + JT_STAGES);   // [NV]
  float* db_s = bias_s + NV;                                  // [NV]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // ---- one-time: fc2 weight -> shared memory (wgmma K-major SWIZZLE_128B chunks), bias ----
  for (int k = tid; k < nkb * WCHUNK / 16; k += JT_THREADS)
    reinterpret_cast<uint4*>(wtile)[k] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    const int pieces = nkb * 8;
    for (int k = tid; k < p.V1 * pieces; k += JT_THREADS) {
      const int r = k / pieces, pc = k % pieces;
      const int col = pc * 8;
      if (col < H)   // (H % 8 == 0)
        *reinterpret_cast<uint4*>(wtile + (pc >> 3) * WCHUNK + sw128_offset(r, pc & 7)) =
            *reinterpret_cast<const uint4*>(p.w2 + (long long)r * H + col);
    }
    if (tid < NV) {
      bias_s[tid] = tid < p.V1 ? p.b2[tid] : 0.f;
      db_s[tid] = 0.f;
    }
  }
  if (tid == 0) {
    for (int s = 0; s < JT_STAGES; ++s) {
      mbar_init(&full[s], 4);
      mbar_init(&empty[s], 1);
    }
    mbar_fence_init();
  }
  fence_proxy_async_smem();
  __syncthreads();
  const long long ntiles = (p.nodes + 127) / 128;

  if (warp < JT_PW) {
    // ===================== producers: thread = node row of the tile =====================
    // The groups of 4 warps take k-blocks in turn (item i = running (tile, k-block) index goes to
    // group i % JT_GROUPS, ring stage i % JT_STAGES): a k-block is one L2 round trip (128 rows x
    // 256 B of fy), so JT_GROUPS of them are in flight per CTA.  Measured: 2.36 ms per pass with
    // one group, 1.05 ms with two, against an L2-ingest floor of 0.73 ms (3.3 GB of fy rows at
    // ~30 GB/s per SM).
    const int grp = warp >> 2;
    const int rowt = tid & 127;
    long long item = 0;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const long long n = tile * 128 + rowt;
      const bool ok = n < p.nodes;
      // nodes are TIME-major: n = (t * B + b) * U1 + u (a range of frames is a contiguous slab)
      const long long tb = ok ? n / p.U1 : 0;
      const int u = ok ? (int)(n - tb * p.U1) : 0;
      const int b = (int)(tb % p.B);
      const int t = (int)(tb / p.B);
      const float* xr = p.fx + ((long long)b * p.T + t) * H;
      const float* yr = p.fy + ((long long)b * p.U1 + u) * H;
      for (int kb = 0; kb < nkb; ++kb, ++item) {
        if ((int)(item % JT_GROUPS) != grp) continue;
        const int stage = (int)(item % JT_STAGES);
        const uint32_t phase = (uint32_t)((item / JT_STAGES) & 1);
        if (lane == 0) mbar_wait(&empty[stage], phase ^ 1);
        __syncwarp();
        uint8_t* a = a_ring + stage * A_BYTES;
#pragma unroll
        for (int c16 = 0; c16 < 8; ++c16) {
          const int k0 = kb * 64 + c16 * 8;
          uint4 o = make_uint4(0, 0, 0, 0);
          if (ok && k0 < H) {
            const float4 x0 = __ldg(reinterpret_cast<const float4*>(xr + k0));
            const float4 x1 = __ldg(reinterpret_cast<const float4*>(xr + k0) + 1);
            const float4 y0 = __ldg(reinterpret_cast<const float4*>(yr + k0));
            const float4 y1 = __ldg(reinterpret_cast<const float4*>(yr + k0) + 1);
            o.x = pack_bf16x2(fmaxf(x0.x + y0.x, 0.f), fmaxf(x0.y + y0.y, 0.f));
            o.y = pack_bf16x2(fmaxf(x0.z + y0.z, 0.f), fmaxf(x0.w + y0.w, 0.f));
            o.z = pack_bf16x2(fmaxf(x1.x + y1.x, 0.f), fmaxf(x1.y + y1.y, 0.f));
            o.w = pack_bf16x2(fmaxf(x1.z + y1.z, 0.f), fmaxf(x1.w + y1.w, 0.f));
          }
          *reinterpret_cast<uint4*>(a + sw128_offset((uint32_t)rowt, (uint32_t)c16)) = o;
        }
        fence_proxy_async_smem();     // generic st.shared -> wgmma (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[stage]);
      }
    }
  } else {
    // ===================== consumer warpgroup: wgmma, then thread = node =====================
    const int row = tid - 32 * JT_PW;          // 0..127
    int stage = 0;
    uint32_t phase = 0;
    float dbacc[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) dbacc[j] = 0.f;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const long long n = tile * 128 + row;
      const bool ok = n < p.nodes;
      float d0[NV / 2], d1[NV / 2];            // node rows 0..63 | 64..127 of the tile
#pragma unroll
      for (int j = 0; j < NV / 2; ++j) { d0[j] = 0.f; d1[j] = 0.f; }
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(a_ring + stage * A_BYTES);
        const uint64_t da0 = gmma_desc_sw128_kmajor(sa);
        const uint64_t da1 = gmma_desc_sw128_kmajor(sa + 64 * 128);
        const uint64_t db = gmma_desc_sw128_kmajor(smem_u32(wtile + kb * WCHUNK));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint32_t accum = (kb > 0 || kk > 0) ? 1u : 0u;
          wgmma_bf16<NV>(d0, da0 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), accum);
          wgmma_bf16<NV>(d1, da1 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), accum);
        }
        wgmma_commit();
        wgmma_wait<1>();                       // the previous k-block's group has retired
        if (prev >= 0 && row == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == JT_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d0);
      wgmma_fence_regs(d1);
      if (prev >= 0 && row == 0) mbar_arrive(&empty[prev]);
      // fragment layout -> thread = node row
      wg_store_rows<NV>(d0, acc_s, ACC_LD, 0, 128);
      wg_store_rows<NV>(d1, acc_s, ACC_LD, 64, 128);
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float v[NV];
#pragma unroll
      for (int j = 0; j < NV; ++j) v[j] = acc_s[row * ACC_LD + j];
      asm volatile("bar.sync 1, 128;" ::: "memory");   // the next tile may overwrite acc_s
      if (!ok) continue;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        v[j] = j < p.V1 ? v[j] + bias_s[j] : -INFINITY;
        mx = fmaxf(mx, v[j]);
      }
      float se = 0.f;
#pragma unroll
      for (int j = 0; j < NV; ++j) se += j < p.V1 ? __expf(v[j] - mx) : 0.f;
      const float lse = mx + __logf(se);
      const long long tb = n / p.U1;
      const int u = (int)(n - tb * p.U1);
      const int b = (int)(tb % p.B);
      const int t = (int)(tb / p.B);
      const int lab = (u < p.U1 - 1) ? p.ymat[(long long)b * (p.U1 - 1) + u] : -1;
      if (p.mode == 0) {
        float lb = 0.f, ll = -INFINITY;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          if (j == p.blank) lb = v[j] - lse;
          if (j == lab) ll = v[j] - lse;
        }
        *reinterpret_cast<float2*>(p.lat + n * 2) = make_float2(lb, ll);
        if (p.lp_full) {
          float* o = p.lp_full + (((long long)b * p.T + t) * p.U1 + u) * p.V1;   // batch-first
#pragma unroll
          for (int j = 0; j < NV; ++j)
            if (j < p.V1) o[j] = v[j] - lse;
        }
      } else {
        const float2 g = *reinterpret_cast<const float2*>(p.garc + n * 2);
        const float gs = g.x + g.y;
        uint32_t packed[NV / 2];
#pragma unroll
        for (int j = 0; j < NV; j += 2) {
          float d0 = 0.f, d1 = 0.f;
          if (j < p.V1)
            d0 = (j == p.blank ? g.x : 0.f) + (j == lab ? g.y : 0.f) - gs * __expf(v[j] - lse);
          if (j + 1 < p.V1)
            d1 = (j + 1 == p.blank ? g.x : 0.f) + (j + 1 == lab ? g.y : 0.f) -
                 gs * __expf(v[j + 1] - lse);
          dbacc[j] += d0;
          dbacc[j + 1] += d1;
          packed[j / 2] = pack_bf16x2(d0, d1);
        }
        uint4* o = reinterpret_cast<uint4*>(p.dlogits + n * NV);
#pragma unroll
        for (int q = 0; q < NV / 8; ++q)
          o[q] = make_uint4(packed[4 * q], packed[4 * q + 1], packed[4 * q + 2], packed[4 * q + 3]);
      }
    }
    if (p.mode == 1) {
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const float s = warp_sum(dbacc[j]);
        if (lane == 0 && j < p.V1) atomicAdd(&db_s[j], s);
      }
    }
  }

  __syncthreads();
  if (p.mode == 1 && tid < p.V1) atomicAdd(p.db2 + tid, db_s[tid]);
}

// ---- slab kernels of the backward pass -------------------------------------------------------
// Z slab: rows r = ((tt * B + b) * U1 + u) = nodes of frames t0 .. t0+Tc-1 in node order,
// z[r][h] = relu(fx[b, t0+tt, h] + fy[b, u, h]) bf16
__global__ void __launch_bounds__(256)
joint_build_slab_kernel(const float* __restrict__ fx, const float* __restrict__ fy,
                        bf16* __restrict__ z, int B, int T, int U1, int H, int t0, int Tc) {
  const long long total = (long long)B * Tc * U1 * (H / 8);
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int h8 = (int)(i % (H / 8));
    long long r = i / (H / 8);
    const int u = (int)(r % U1);
    r /= U1;
    const int b = (int)(r % B);
    const int tt = (int)(r / B);
    const float4* x = reinterpret_cast<const float4*>(fx + ((long long)b * T + t0 + tt) * H + h8 * 8);
    const float4* y = reinterpret_cast<const float4*>(fy + ((long long)b * U1 + u) * H + h8 * 8);
    const float4 x0 = __ldg(x), x1 = __ldg(x + 1), y0 = __ldg(y), y1 = __ldg(y + 1);
    uint4 o;
    o.x = pack_bf16x2(fmaxf(x0.x + y0.x, 0.f), fmaxf(x0.y + y0.y, 0.f));
    o.y = pack_bf16x2(fmaxf(x0.z + y0.z, 0.f), fmaxf(x0.w + y0.w, 0.f));
    o.z = pack_bf16x2(fmaxf(x1.x + y1.x, 0.f), fmaxf(x1.y + y1.y, 0.f));
    o.w = pack_bf16x2(fmaxf(x1.z + y1.z, 0.f), fmaxf(x1.w + y1.w, 0.f));
    reinterpret_cast<uint4*>(z)[i] = o;
  }
}

// dZ slab (fp32 [rows][H]) masked by z > 0 and summed over u (-> dfx of the slab's frames) and
// over the slab's frames (-> += dfy).  CTA = (utterance, 128 columns of h): lanes over h in float4
// groups, the 8 warps take u = warp, warp+8, ...; every thread walks only ~U1/8 label positions
// (the walk is a chain of L2 round trips: with one thread per (b, h) walking all of them the
// kernel ran 300 us per slab at 0.5 TB/s).  dfy has exactly one writer per element; the 8
// per-warp partial sums of dfx are added in warp order through shared memory (no atomics).
static constexpr int JT_MAX_TC = 8;
__global__ void __launch_bounds__(256)
joint_reduce_slab_kernel(const float* __restrict__ dz, const bf16* __restrict__ z,
                         float* __restrict__ dfx, float* __restrict__ dfy, int B, int T, int U1,
                         int H, int t0, int Tc) {
  __shared__ float4 fxs[8][JT_MAX_TC][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int H4 = H >> 2;
  const int h4 = blockIdx.x * 32 + lane;
  const int b = blockIdx.y;
  const bool ok = h4 < H4;
  const float4* dz4 = reinterpret_cast<const float4*>(dz);
  const uint2* z4 = reinterpret_cast<const uint2*>(z);
  float4* dfy4 = reinterpret_cast<float4*>(dfy);
  float4 fxacc[JT_MAX_TC];
#pragma unroll
  for (int tt = 0; tt < JT_MAX_TC; ++tt) fxacc[tt] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ok) {
#pragma unroll 1
    for (int u = warp; u < U1; u += 8) {
      float4 g[JT_MAX_TC];
      uint2 zz[JT_MAX_TC];
#pragma unroll
      for (int tt = 0; tt < JT_MAX_TC; ++tt) {
        if (tt < Tc) {
          const long long row = ((long long)tt * B + b) * U1 + u;
          g[tt] = __ldcs(dz4 + row * H4 + h4);
          zz[tt] = __ldcs(z4 + row * H4 + h4);
        }
      }
      float4* yo = dfy4 + ((long long)b * U1 + u) * H4 + h4;
      float4 sy = *yo;
#pragma unroll
      for (int tt = 0; tt < JT_MAX_TC; ++tt) {
        if (tt < Tc) {
          // a bf16 is positive iff its sign bit is clear and it is not zero
          const float gx = (zz[tt].x & 0x7fffu) != 0u && !(zz[tt].x & 0x8000u) ? g[tt].x : 0.f;
          const float gy = (zz[tt].x & 0x7fff0000u) != 0u && !(zz[tt].x & 0x80000000u) ? g[tt].y : 0.f;
          const float gz = (zz[tt].y & 0x7fffu) != 0u && !(zz[tt].y & 0x8000u) ? g[tt].z : 0.f;
          const float gw = (zz[tt].y & 0x7fff0000u) != 0u && !(zz[tt].y & 0x80000000u) ? g[tt].w : 0.f;
          sy.x += gx; sy.y += gy; sy.z += gz; sy.w += gw;
          fxacc[tt].x += gx; fxacc[tt].y += gy; fxacc[tt].z += gz; fxacc[tt].w += gw;
        }
      }
      *yo = sy;
    }
  }
#pragma unroll
  for (int tt = 0; tt < JT_MAX_TC; ++tt) fxs[warp][tt][lane] = fxacc[tt];
  __syncthreads();
  if (ok && warp < Tc) {
    float4 s = fxs[0][warp][lane];
#pragma unroll
    for (int q = 1; q < 8; ++q) {
      const float4 v = fxs[q][warp][lane];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    reinterpret_cast<float4*>(dfx)[((long long)b * T + t0 + warp) * H4 + h4] = s;
  }
}

}  // namespace sb

using namespace sb;

// shared memory of the fused kernel for (H, V1): ring | fc2 weight | parked accumulator tile |
// barriers, bias, bias gradient
static size_t joint_smem_bytes(int H, int V1) {
  const int nv = V1 <= 32 ? 32 : 64;
  const int nkb = (H + 63) / 64;
  const int stages = nv == 32 ? JtCfg<32>::kStages : JtCfg<64>::kStages;
  return (size_t)stages * 128 * 128 + (size_t)nkb * nv * 128 + (size_t)128 * (nv + 1) * 4 + 8 +
         1024 + 16 * stages + 8 * nv;
}

// 1 if the fused kernel (fc2 resident in shared memory) runs (H, V1), else 0
extern "C" int sb_rnnt_joint_resident(int H, int V1) {
  return H > 0 && H % 8 == 0 && V1 > 0 && V1 <= 64 && joint_smem_bytes(H, V1) <= 227 * 1024;
}

static int joint_launch(JointParams& p, void* stream_) {
  if (!sb_rnnt_joint_resident(p.H, p.V1) || p.blank < 0 || p.blank >= p.V1)
    return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int nv = p.V1 <= 32 ? 32 : 64;
  const size_t smem = joint_smem_bytes(p.H, p.V1);
  const long long ntiles = (p.nodes + 127) / 128;
  int grid = device_sm_count();
  if (grid > ntiles) grid = (int)ntiles;
  cudaError_t e;
  if (nv == 32) {
    e = cudaFuncSetAttribute(joint_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return SB_ERR_CUDA;
    joint_kernel<32><<<grid, JtCfg<32>::kThreads, smem, stream>>>(p);
  } else {
    e = cudaFuncSetAttribute(joint_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return SB_ERR_CUDA;
    joint_kernel<64><<<grid, JtCfg<64>::kThreads, smem, stream>>>(p);
  }
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_joint_fwd(const float* fx, const float* fy, const void* w2_bf16,
                                 const float* b2, const int* ymat, float* lat, float* lp_full,
                                 int B, int T, int U1, int H, int V1, int blank, void* stream) {
  if (!fx || !fy || !w2_bf16 || !b2 || !ymat || !lat || B <= 0 || T <= 0 || U1 <= 0)
    return SB_ERR_INVALID;
  JointParams p;
  memset(&p, 0, sizeof(p));
  p.fx = fx; p.fy = fy; p.w2 = reinterpret_cast<const bf16*>(w2_bf16); p.b2 = b2; p.ymat = ymat;
  p.lat = lat; p.lp_full = lp_full; p.nodes = (long long)B * T * U1;
  p.B = B; p.T = T; p.U1 = U1; p.H = H; p.V1 = V1; p.blank = blank; p.mode = 0;
  return joint_launch(p, stream);
}

extern "C" int sb_rnnt_joint_dlogits(const float* fx, const float* fy, const void* w2_bf16,
                                     const float* b2, const int* ymat, const float* garc,
                                     void* dlogits_bf16, float* db2, int B, int T, int U1, int H,
                                     int V1, int blank, void* stream) {
  if (!fx || !fy || !w2_bf16 || !b2 || !ymat || !garc || !dlogits_bf16 || !db2 || B <= 0 ||
      T <= 0 || U1 <= 0)
    return SB_ERR_INVALID;
  JointParams p;
  memset(&p, 0, sizeof(p));
  p.fx = fx; p.fy = fy; p.w2 = reinterpret_cast<const bf16*>(w2_bf16); p.b2 = b2; p.ymat = ymat;
  p.garc = garc; p.dlogits = reinterpret_cast<bf16*>(dlogits_bf16); p.db2 = db2;
  p.nodes = (long long)B * T * U1;
  p.B = B; p.T = T; p.U1 = U1; p.H = H; p.V1 = V1; p.blank = blank; p.mode = 1;
  return joint_launch(p, stream);
}

extern "C" int sb_rnnt_joint_build_slab(const float* fx, const float* fy, void* z_bf16, int B, int T,
                                        int U1, int H, int t0, int Tc, void* stream_) {
  if (!fx || !fy || !z_bf16 || H % 8 != 0 || t0 < 0 || t0 + Tc > T) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long total = (long long)B * Tc * U1 * (H / 8);
  long long g = (total + 255) / 256;
  const long long cap = (long long)device_sm_count() * 16;
  joint_build_slab_kernel<<<(int)(g < cap ? g : cap), 256, 0, stream>>>(
      fx, fy, reinterpret_cast<bf16*>(z_bf16), B, T, U1, H, t0, Tc);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_joint_reduce_slab(const float* dz, const void* z_bf16, float* dfx, float* dfy,
                                         int B, int T, int U1, int H, int t0, int Tc,
                                         void* stream_) {
  if (!dz || !z_bf16 || !dfx || !dfy || t0 < 0 || t0 + Tc > T || Tc > JT_MAX_TC)
    return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (H % 4 != 0 || B > 65535) return SB_ERR_UNSUPPORTED;
  const dim3 grid((H / 4 + 31) / 32, B);
  joint_reduce_slab_kernel<<<grid, 256, 0, stream>>>(
      dz, reinterpret_cast<const bf16*>(z_bf16), dfx, dfy, B, T, U1, H, t0, Tc);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
