// sb_gemm_bf16_tn: C[M,N] (f32) (+)= A[M,K] (bf16, K-major) * B[N,K]^T (bf16, K-major) (+ bias[N])
//
// Hand-written sm_90a GEMM used for every dense contraction on the encoder path
// (GRU input projections X*W_ih^T, their dgrad/wgrad, the output projection and its grads;
//  reference: nn.GRU / LinearND in speech/models/model.py:35-39,115-133, which reach cuDNN/cuBLAS).
//
//   * persistent grid (one CTA per SM), static tile schedule, N-fastest rasterisation so the
//     A row-panel is served from L2 to the CTAs working on its N tiles
//   * warp 0   : TMA producer (cp.async.bulk.tensor, SWIZZLE_128B boxes of 64 bf16 along K)
//   * warpgroups 1, 2: wgmma consumers, 64 rows of the 128 x BN tile each, fp32 accumulators in
//     registers; each releases a ring slot as soon as the wgmma group that read it has retired
//     (one group kept in flight), then stores its rows straight from the registers
//   * smem ring of kStages {A 128x64, B BNx64} tiles, full/empty mbarriers
//
// Roofline: tensor (bf16 dense).  Algorithmic FLOPs = 2*M*N*K per launch.
#include "common.cuh"
#include <cuda.h>
#include <stdio.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int BM = 128;
static constexpr int BK = 64;  // 64 bf16 = 128 bytes = one SWIZZLE_128B row
static constexpr int GEMM_THREADS = 384;

struct GemmParams {
  float* C;
  const float* bias;
  long long ldc;
  int M, N, K;
  int k_blocks_total;   // ceil(K / 64)
  int split_k;          // >= 1
  int flags;            // SB_GEMM_ACCUMULATE | SB_GEMM_ROW_REMAP
  int remap_B, remap_T, valid_B;
  int m_tiles, n_tiles;
};

// MN-major operand tiles: the contraction runs over the ROWS of the global matrix ([K][MN], MN
// contiguous), which is how activations [tokens][features] look to a weight-gradient GEMM.  A TMA
// box {64 MN (inner, 128 B), 64 K rows} with SWIZZLE_128B lands as one 8 KB block that is exactly
// the canonical MN-major SWIZZLE_128B layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units:
// 8 K-rows of 128 B per swizzle atom (SBO = 1024 B between atoms), the next 64 MN at
// LBO = 8192 B (the next box).  One MMA (K = 16) spans two atoms; the next MMA starts 2048 B on.
static constexpr int MN_BOX_BYTES = 64 * 64 * 2;
static int g_mn_lbo = MN_BOX_BYTES, g_mn_sbo = 1024, g_mn_kadv = 2048;   // developer knobs

struct MnDesc { uint32_t lbo, sbo, kadv; };

template <int BN>
struct GemmCfg {
  static constexpr int kStageBytes = (BM + BN) * BK * 2;
  static constexpr int kStagesRaw = (200 * 1024) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/;
};

template <int BN, int TA, int TB>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmap_a,
                    const __grid_constant__ CUtensorMap tmap_b, const GemmParams p,
                    const MnDesc mn) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte aligned tile ring (SWIZZLE_128B requirement)
  uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                              ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(tiles + kStages * Cfg::kStageBytes);
  uint64_t* full_bar = bars;                  // [kStages]
  uint64_t* empty_bar = bars + kStages;       // [kStages]  one arrive per consumer warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    mbar_fence_init();
  }
  __syncthreads();

  const int tiles_mn = p.m_tiles * p.n_tiles;
  const int total_work = tiles_mn * p.split_k;
  const int kb_per_split = (p.k_blocks_total + p.split_k - 1) / p.split_k;

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        const int split = w / tiles_mn;
        const int t = w - split * tiles_mn;
        const int m_blk = t / p.n_tiles;
        const int n_blk = t - m_blk * p.n_tiles;
        const int kb0 = split * kb_per_split;
        int kb1 = kb0 + kb_per_split;
        if (kb1 > p.k_blocks_total) kb1 = p.k_blocks_total;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = tiles + stage * Cfg::kStageBytes;
          uint8_t* sb_ = sa + BM * BK * 2;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (TA) {
#pragma unroll
            for (int b = 0; b < BM / 64; ++b)
              tma_load_2d(sa + b * MN_BOX_BYTES, &tmap_a, &full_bar[stage], m_blk * BM + b * 64,
                          kb * BK);
          } else {
            tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BK, m_blk * BM);
          }
          if (TB) {
#pragma unroll
            for (int b = 0; b < (BN + 63) / 64; ++b)
              tma_load_2d(sb_ + b * MN_BOX_BYTES, &tmap_b, &full_bar[stage], n_blk * BN + b * 64,
                          kb * BK);
          } else {
            tma_load_2d(sb_, &tmap_b, &full_bar[stage], kb * BK, n_blk * BN);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup 1 -> rows 0..63, 2 -> rows 64..127 ==========
    const int half = (warp >> 2) - 1;
    const int t = threadIdx.x & 127;
    const bool leader = t == 0;
    const uint64_t a_step = TA ? (uint64_t)(mn.kadv >> 4) : 2u;
    const uint64_t b_step = TB ? (uint64_t)(mn.kadv >> 4) : 2u;
    const bool vec_ok = ((p.ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
      const int split = w / tiles_mn;
      const int tt = w - split * tiles_mn;
      const int m_blk = tt / p.n_tiles;
      const int n_blk = tt - m_blk * p.n_tiles;
      const int kb0 = split * kb_per_split;
      int kb1 = kb0 + kb_per_split;
      if (kb1 > p.k_blocks_total) kb1 = p.k_blocks_total;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(tiles + stage * Cfg::kStageBytes);
        const uint32_t sb_ = sa + BM * BK * 2;
        // K-major A: rows 64*half.. start 8 KB on; MN-major A: the half-th 64-wide box
        const uint64_t da = TA ? gmma_desc_sw128_mnmajor(sa + half * MN_BOX_BYTES, mn.lbo, mn.sbo)
                               : gmma_desc_sw128_kmajor(sa + half * 64 * 128);
        const uint64_t db = TB ? gmma_desc_sw128_mnmajor(sb_, mn.lbo, mn.sbo)
                               : gmma_desc_sw128_kmajor(sb_);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_bf16<BN, TA, TB>(acc, da + a_step * k, db + b_step * k, (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                 // the group of the previous k-block has retired
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
      if (kb1 <= kb0) continue;          // empty K range (over-split K): nothing accumulated

      // ---- epilogue straight from the registers: rows r, r + 8; column pairs every 8 ----
      const bool add_bias = (p.bias != nullptr) && (split == 0);
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        const int m = m_blk * BM + half * 64 + ((t >> 5) << 4) + ((t & 31) >> 2) + rh * 8;
        bool row_ok = m < p.M;
        long long out_row = m;
        if (p.flags & SB_GEMM_ROW_REMAP) {
          const int b = m % p.remap_B;
          const int tm = m / p.remap_B;
          row_ok = row_ok && (b < p.valid_B);
          out_row = (long long)b * p.remap_T + tm;
        }
        if (!row_ok) continue;
        float* crow = p.C + out_row * p.ldc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n_blk * BN + j * 8 + ((t & 3) << 1);
          float x0 = acc[4 * j + 2 * rh], x1 = acc[4 * j + 2 * rh + 1];
          if (n >= p.N) continue;
          const bool two = n + 1 < p.N;
          if (add_bias) {
            x0 += __ldg(p.bias + n);
            if (two) x1 += __ldg(p.bias + n + 1);
          }
          if (p.flags & SB_GEMM_ACCUMULATE) {
            atomicAdd(crow + n, x0);
            if (two) atomicAdd(crow + n + 1, x1);
          } else if (two && vec_ok) {
            *reinterpret_cast<float2*>(crow + n) = make_float2(x0, x1);
          } else {
            crow[n] = x0;
            if (two) crow[n + 1] = x1;
          }
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess) return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  return fn;
}

// 2-D bf16 tensor map over a row-major [rows, cols] matrix with leading dimension ld (elements);
// box = 64 columns x box_rows rows, SWIZZLE_128B, out-of-bounds reads return zero.
int make_tmap_bf16_2d(CUtensorMap* map, const void* base, long long rows, long long cols,
                      long long ld, int box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return SB_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || ((ld * 2) & 15) != 0) return SB_ERR_INVALID;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? SB_OK : SB_ERR_CUDA;
}

int device_sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

// K split of an ACCUMULATING GEMM (the caller's value is only a hint).  Work items = tiles x
// splits are dealt round-robin to `units` CTAs, so the launch takes ceil(tiles*split/units)
// rounds of (k-blocks per item + E) each, E ~ the epilogue / reduce-add pass of an item expressed
// in k-block times.  The minimum of that product fills whole waves while every wave still walks
// K in lockstep, which keeps the operand panels in L2.
static int pick_wave_filling_split(long long tiles, int units, int k_blocks) {
  const long long kEpilogue = 4;
  int best_split = 1;
  long long best = -1;
  for (int sp = 1; sp <= 512; ++sp) {
    if (sp > 1 && k_blocks / sp < 8) break;
    const long long rounds = (tiles * sp + units - 1) / units;
    const long long cost = rounds * ((k_blocks + sp - 1) / sp + kEpilogue);
    if (best < 0 || cost < best) { best = cost; best_split = sp; }   // ties: fewer splits
  }
  return best_split;
}

template <int BN, int TA, int TB>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, GemmParams p,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_tn_kernel<BN, TA, TB>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) return SB_ERR_CUDA;
    attr_set = true;
  }
  p.n_tiles = (p.N + BN - 1) / BN;
  const int total = p.m_tiles * p.n_tiles * p.split_k;
  int grid = device_sm_count();
  if (grid > total) grid = total;
  const MnDesc mn = {(uint32_t)g_mn_lbo, (uint32_t)g_mn_sbo, (uint32_t)g_mn_kadv};
  gemm_bf16_tn_kernel<BN, TA, TB><<<grid, GEMM_THREADS, Cfg::kSmemBytes, stream>>>(ta, tb, p, mn);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

template <int BN>
static int launch_gemm_bn(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          bool a_mn, bool b_mn, cudaStream_t stream) {
  if (a_mn) return b_mn ? launch_gemm<BN, 1, 1>(ta, tb, p, stream) : launch_gemm<BN, 1, 0>(ta, tb, p, stream);
  return b_mn ? launch_gemm<BN, 0, 1>(ta, tb, p, stream) : launch_gemm<BN, 0, 0>(ta, tb, p, stream);
}

}  // namespace sb

using namespace sb;

// developer hook: override the MN-major descriptor fields (bytes); 0 keeps a field
extern "C" int sb_debug_umma_mn(int lbo, int sbo, int kadv) {
  if (lbo > 0) sb::g_mn_lbo = lbo;
  if (sbo > 0) sb::g_mn_sbo = sbo;
  if (kadv > 0) sb::g_mn_kadv = kadv;
  return SB_OK;
}

extern "C" int sb_gemm_bf16_tn(const void* A, long long lda, const void* B, long long ldb, float* C,
                               long long ldc, const float* bias, int M, int N, int K, int flags,
                               int split_k, int remap_B, int remap_T, int valid_B,
                               void* stream_) {
  if (!A || !B || !C || M <= 0 || N <= 0 || K <= 0) return SB_ERR_INVALID;
  if (split_k < 1) split_k = 1;
  if (split_k > 1 && !(flags & SB_GEMM_ACCUMULATE)) return SB_ERR_INVALID;
  if ((flags & SB_GEMM_ROW_REMAP) && (remap_B <= 0 || remap_T <= 0)) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GemmParams p;
  p.C = C; p.bias = bias; p.ldc = ldc; p.M = M; p.N = N; p.K = K;
  p.k_blocks_total = (K + BK - 1) / BK;
  if (split_k > p.k_blocks_total) split_k = p.k_blocks_total;
  p.split_k = split_k; p.flags = flags;
  p.remap_B = remap_B; p.remap_T = remap_T; p.valid_B = valid_B;
  p.m_tiles = (M + BM - 1) / BM;
  p.n_tiles = 0;
  const bool a_mn = (flags & SB_GEMM_A_MN) != 0;
  const bool b_mn = (flags & SB_GEMM_B_MN) != 0;
  // tile-N choice: 128 x 128 tiles keep the 64 accumulator registers per consumer thread below the
  // register cap of a 3-warpgroup CTA; narrow GEMMs take narrower tiles (an MN-major B tile is
  // made of 64-wide boxes)
  int bn;
  if (N <= 32 && !b_mn) bn = 32;
  else if (N <= 64) bn = 64;
  else bn = 128;
  if (flags & SB_GEMM_ACCUMULATE)
    p.split_k = pick_wave_filling_split((long long)p.m_tiles * ((N + bn - 1) / bn),
                                        device_sm_count(), p.k_blocks_total);
  // tensor maps: K-major operands are [rows][K] with box {64 K, rows}; MN-major operands are
  // [K][rows] with box {64 rows, 64 K}
  CUtensorMap ta, tb;
  int rc = a_mn ? make_tmap_bf16_2d(&ta, A, K, M, lda, 64) : make_tmap_bf16_2d(&ta, A, M, K, lda, BM);
  if (rc != SB_OK) return rc;
  rc = b_mn ? make_tmap_bf16_2d(&tb, B, K, N, ldb, 64) : make_tmap_bf16_2d(&tb, B, N, K, ldb, bn);
  if (rc != SB_OK) return rc;
  switch (bn) {
    case 32: return launch_gemm_bn<32>(ta, tb, p, a_mn, b_mn, stream);
    case 64: return launch_gemm_bn<64>(ta, tb, p, a_mn, b_mn, stream);
    default: return launch_gemm_bn<128>(ta, tb, p, a_mn, b_mn, stream);
  }
}
