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
// GEMMs with N > 128 run gemm_bf16_tn_c2_kernel instead: 128 x 256 tiles over 2-CTA clusters that
// share the B tile by TMA multicast (see there).
//
// Roofline: tensor (bf16 dense).  Algorithmic FLOPs = 2*M*N*K per launch.
#include "common.cuh"
#include <cuda.h>
#include <stdio.h>
#include <string.h>

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
  int m_pairs;          // gemm_bf16_tn_c2_kernel: ceil(m_tiles / 2)
  int epi;              // gemm_bf16_tn_c2_kernel: C2Epilogue
};

// How gemm_bf16_tn_c2_kernel writes its output tiles
enum C2Epilogue : int {
  C2_EPI_REGS = 0,        // straight from the registers (st.global / atomicAdd per element pair)
  C2_EPI_TMA = 1,         // staged through shared memory, TMA bulk tensor stores
  C2_EPI_TMA_REDUCE = 2,  // staged through shared memory, TMA bulk tensor reduce-add
  C2_EPI_NONE = 3,        // timing only: no output at all
};

// MN-major operand tiles: the contraction runs over the ROWS of the global matrix ([K][MN], MN
// contiguous), which is how activations [tokens][features] look to a weight-gradient GEMM.  A TMA
// box {64 MN (inner, 128 B), 64 K rows} with SWIZZLE_128B lands as one 8 KB block that is exactly
// the canonical MN-major SWIZZLE_128B layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units:
// 8 K-rows of 128 B per swizzle atom (SBO = 1024 B between atoms), the next 64 MN at
// LBO = 8192 B (the next box).  One MMA (K = 16) spans two atoms; the next MMA starts 2048 B on.
static constexpr int MN_BOX_BYTES = 64 * 64 * 2;
static constexpr uint32_t MN_LBO = MN_BOX_BYTES, MN_SBO = 1024, MN_KADV = 2048;

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
                    const __grid_constant__ CUtensorMap tmap_b, const GemmParams p) {
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
    const uint64_t a_step = TA ? (uint64_t)(MN_KADV >> 4) : 2u;
    const uint64_t b_step = TB ? (uint64_t)(MN_KADV >> 4) : 2u;
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
        const uint64_t da = TA ? gmma_desc_sw128_mnmajor(sa + half * MN_BOX_BYTES, MN_LBO, MN_SBO)
                               : gmma_desc_sw128_kmajor(sa + half * 64 * 128);
        const uint64_t db = TB ? gmma_desc_sw128_mnmajor(sb_, MN_LBO, MN_SBO)
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
// gemm_bf16_tn_c2_kernel: 128 x 256 tiles over 2-CTA clusters, for N > 128.
//
//   * the two CTAs of a cluster take M tiles 2i and 2i + 1 of the same N tile; each loads its own
//     A tile (128 x 64) and HALF of the shared B tile (128 of the 256 rows) with a TMA multicast
//     into both CTAs: 32 KB of L2 -> SM traffic per CTA per k-block for 4.2 MFLOP (7.8 B/kFLOP,
//     half the 15.6 of the 128 x 128 kernel above)
//   * register reallocation: the producer warpgroup drops to 40 registers, the two consumer
//     warpgroups rise to 232, enough for one 64 x 256 fp32 accumulator (128 registers) each
//   * a ring slot holds data written by both CTAs' TMA, so it is refilled only after the
//     consumers of BOTH CTAs have released it: each consumer warpgroup arrives on the empty
//     barrier of both CTAs (count 4)
//   * an unpaired last M tile runs on rank 0; rank 1 loads a box past M (zero fill) so that the
//     shared B stays in lockstep, and stores nothing
//   * epilogue (C2_EPI_TMA / C2_EPI_TMA_REDUCE): each consumer warpgroup writes its 64 x 256 fp32
//     rows, bias added, into a shared-memory box of 64 rows x 32 columns (128 B rows, SWIZZLE_128B
//     so the st.shared are free of bank conflicts), and one thread hands the box to the TMA unit as
//     a bulk tensor store (reduce-add for accumulating launches).  C2_EPI_BUFS boxes per
//     warpgroup take turns; a box is rewritten only after the TMA has read it, so the global
//     writes of a tile drain while the warpgroup fills the next boxes and runs the next tile's
//     MMAs.  The tensor map of C clips rows >= M and columns >= N.  C2_EPI_REGS stores straight
//     from the registers (row remap, C not 16-byte aligned, split-K accumulation).
// Every output element has the same sum as in gemm_bf16_tn_kernel (one fp32 accumulator,
// k-blocks ascending, the same k16 wgmma steps), so non-accumulating results are bit-identical.
// ----------------------------------------------------------------------------------------------
static constexpr int C2_BN = 256;
static constexpr int C2_STAGES = 4;
static constexpr int C2_A_BYTES = BM * BK * 2;                  // 16 KB
static constexpr int C2_STAGE_BYTES = (BM + C2_BN) * BK * 2;    // 48 KB
static constexpr int C2_EPI_COLS = 32;                          // fp32 columns of a staging box
static constexpr int C2_EPI_BOX_BYTES = 64 * C2_EPI_COLS * 4;   // 8 KB: 64 rows of 128 B
static constexpr int C2_EPI_BUFS = 2;                           // staging boxes per warpgroup
static constexpr int C2_EPI_BYTES = 2 /*warpgroups*/ * C2_EPI_BUFS * C2_EPI_BOX_BYTES;
static constexpr int C2_SMEM_BYTES = C2_STAGES * C2_STAGE_BYTES + C2_EPI_BYTES + 1024 /*align*/ +
                                     256 /*barriers*/;

template <int TA, int TB>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_tn_c2_kernel(const __grid_constant__ CUtensorMap tmap_a,
                       const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_c, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                              ~static_cast<uintptr_t>(1023));
  uint8_t* epi_boxes = tiles + C2_STAGES * C2_STAGE_BYTES;     // [warpgroup][C2_EPI_BUFS] boxes
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_boxes + C2_EPI_BYTES);
  uint64_t* full_bar = bars;                  // [C2_STAGES]
  uint64_t* empty_bar = bars + C2_STAGES;     // [C2_STAGES]  one arrive per consumer warpgroup
                                              //              of each CTA of the cluster
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int rank = (int)cluster_rank();

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.epi == C2_EPI_TMA || p.epi == C2_EPI_TMA_REDUCE) tma_prefetch_desc(&tmap_c);
    for (int s = 0; s < C2_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    mbar_fence_init();
  }
  cluster_sync_all();   // the peer's barriers are initialised before anyone signals them

  const int pair_tiles = p.m_pairs * p.n_tiles;
  const int total_work = pair_tiles * p.split_k;
  const int kb_per_split = (p.k_blocks_total + p.split_k - 1) / p.split_k;
  const int cluster_id = blockIdx.x >> 1;
  const int n_clusters = gridDim.x >> 1;

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = cluster_id; w < total_work; w += n_clusters) {
        const int split = w / pair_tiles;
        const int t = w - split * pair_tiles;
        const int m_pair = t / p.n_tiles;
        const int n_blk = t - m_pair * p.n_tiles;
        const int m_blk = 2 * m_pair + rank;
        const int kb0 = split * kb_per_split;
        int kb1 = kb0 + kb_per_split;
        if (kb1 > p.k_blocks_total) kb1 = p.k_blocks_total;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = tiles + stage * C2_STAGE_BYTES;
          uint8_t* sb_ = sa + C2_A_BYTES;
          mbar_expect_tx(&full_bar[stage], C2_STAGE_BYTES);   // own A + both halves of B
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
            for (int b = 2 * rank; b < 2 * rank + 2; ++b)
              tma_load_2d_mc(sb_ + b * MN_BOX_BYTES, &tmap_b, &full_bar[stage],
                             n_blk * C2_BN + b * 64, kb * BK, 0x3);
          } else {
            tma_load_2d_mc(sb_ + rank * (C2_BN / 2) * BK * 2, &tmap_b, &full_bar[stage], kb * BK,
                           n_blk * C2_BN + rank * (C2_BN / 2), 0x3);
          }
          if (++stage == C2_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers: warpgroup 1 -> rows 0..63, 2 -> rows 64..127 ==========
    setmaxnreg_inc<232>();
    const int half = (warp >> 2) - 1;
    const int t = threadIdx.x & 127;
    const bool leader = t == 0;
    const uint64_t a_step = TA ? (uint64_t)(MN_KADV >> 4) : 2u;
    const uint64_t b_step = TB ? (uint64_t)(MN_KADV >> 4) : 2u;
    const bool vec_ok = ((p.ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
    const uint32_t my_boxes = smem_u32(epi_boxes + half * C2_EPI_BUFS * C2_EPI_BOX_BYTES);
    uint32_t n_boxes = 0;                // boxes this warpgroup has staged (the next buffer follows)
    int stage = 0;
    uint32_t phase = 0;
    for (int w = cluster_id; w < total_work; w += n_clusters) {
      const int split = w / pair_tiles;
      const int tt = w - split * pair_tiles;
      const int m_pair = tt / p.n_tiles;
      const int n_blk = tt - m_pair * p.n_tiles;
      const int m_blk = 2 * m_pair + rank;
      const int kb0 = split * kb_per_split;
      int kb1 = kb0 + kb_per_split;
      if (kb1 > p.k_blocks_total) kb1 = p.k_blocks_total;
      float acc[C2_BN / 2];
#pragma unroll
      for (int i = 0; i < C2_BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(tiles + stage * C2_STAGE_BYTES);
        const uint32_t sb_ = sa + C2_A_BYTES;
        const uint64_t da = TA ? gmma_desc_sw128_mnmajor(sa + half * MN_BOX_BYTES, MN_LBO, MN_SBO)
                               : gmma_desc_sw128_kmajor(sa + half * 64 * 128);
        const uint64_t db = TB ? gmma_desc_sw128_mnmajor(sb_, MN_LBO, MN_SBO)
                               : gmma_desc_sw128_kmajor(sb_);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_bf16<C2_BN, TA, TB>(acc, da + a_step * k, db + b_step * k,
                                    (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                 // the group of the previous k-block has retired
        if (prev >= 0 && leader) { mbar_arrive_remote(&empty_bar[prev], 0); mbar_arrive_remote(&empty_bar[prev], 1); }
        prev = stage;
        if (++stage == C2_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && leader) { mbar_arrive_remote(&empty_bar[prev], 0); mbar_arrive_remote(&empty_bar[prev], 1); }
      if (kb1 <= kb0 || m_blk >= p.m_tiles) continue;   // empty K range / unpaired M tile
      if (p.epi == C2_EPI_NONE) continue;
      const bool add_bias = (p.bias != nullptr) && (split == 0);

      if (p.epi != C2_EPI_REGS) {
        // ---- staged epilogue: eight 64 x 32 boxes, TMA bulk store / reduce-add of each ----
        // Thread t holds rows r, r + 8 (r = 16 * warp + lane / 4) and, in box b, the column pairs
        // 8 jj + 2 (t & 3) (jj < 4): registers acc[4 (4b + jj) + 2 rh + {0, 1}].  Pair jj of row
        // r lies in 16-byte chunk 2 jj + (t & 3) / 2 of the 128-byte row, stored at chunk
        // position chunk ^ (r & 7) (SWIZZLE_128B; r & 7 = lane / 4).
        const int r0 = ((t >> 5) << 4) + ((t & 31) >> 2);
        const uint32_t sw = (uint32_t)((t & 31) >> 2);
        const int row0 = m_blk * BM + half * 64;
#pragma unroll
        for (int b = 0; b < C2_BN / C2_EPI_COLS; ++b) {
          const int col0 = n_blk * C2_BN + b * C2_EPI_COLS;
          if (col0 >= p.N) break;          // the rest of the tile lies past N (same for all)
          float bv[8];
          if (add_bias) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int n = col0 + (i >> 1) * 8 + ((t & 3) << 1) + (i & 1);
              bv[i] = n < p.N ? __ldg(p.bias + n) : 0.f;
            }
          }
          const uint32_t box = my_boxes + (n_boxes % C2_EPI_BUFS) * C2_EPI_BOX_BYTES;
          if (leader) bulk_wait_group_read<C2_EPI_BUFS - 1>();   // the TMA has read this buffer
          named_bar_sync(1 + half, 128);
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const uint32_t chunk = (uint32_t)(2 * jj + ((t & 3) >> 1));
            const uint32_t off = ((chunk ^ sw) << 4) + ((t & 1) << 3);
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
              float x0 = acc[4 * (4 * b + jj) + 2 * rh], x1 = acc[4 * (4 * b + jj) + 2 * rh + 1];
              if (add_bias) { x0 += bv[2 * jj]; x1 += bv[2 * jj + 1]; }
              st_shared_f2(box + (uint32_t)(r0 + 8 * rh) * 128u + off, x0, x1);
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(1 + half, 128);
          if (leader) {
            if (p.epi == C2_EPI_TMA_REDUCE) tma_reduce_add_2d(&tmap_c, box, col0, row0);
            else tma_store_2d(&tmap_c, box, col0, row0);
            bulk_commit_group();
          }
          ++n_boxes;
        }
        continue;
      }

      // ---- epilogue straight from the registers: rows r, r + 8; column pairs every 8 ----
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
        for (int j = 0; j < C2_BN / 8; ++j) {
          const int n = n_blk * C2_BN + j * 8 + ((t & 3) << 1);
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
    if (leader) bulk_wait_group<0>();    // the last boxes are written before the CTA exits
  }
  cluster_sync_all();   // no CTA leaves while its peer may still multicast into it or signal it
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

// 2-D fp32 tensor map over the row-major [rows, cols] output C (leading dimension ld elements) for
// the staged epilogue of gemm_bf16_tn_c2_kernel: box = C2_EPI_COLS columns (128 B) x 64 rows,
// SWIZZLE_128B; stores and reduce-adds outside [rows, cols] are dropped.
static int make_tmap_f32_c(CUtensorMap* map, const float* base, long long rows, long long cols,
                           long long ld) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return SB_ERR_CUDA;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)C2_EPI_COLS, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
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
  gemm_bf16_tn_kernel<BN, TA, TB><<<grid, GEMM_THREADS, Cfg::kSmemBytes, stream>>>(ta, tb, p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

// Clusters of gemm_bf16_tn_c2_kernel resident at once: the size of its persistent grid.  Every
// instantiation has the same block size, launch bounds and shared memory, so one query serves all.
static int c2_max_clusters() {
  static int n = -1;
  if (n >= 0) return n;
  auto kernel = gemm_bf16_tn_c2_kernel<0, 0>;
  n = 0;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C2_SMEM_BYTES) !=
      cudaSuccess) {
    cudaGetLastError();
    return n;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * (device_sm_count() / 2));
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = C2_SMEM_BYTES;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) {
    cudaGetLastError();
    n = 0;
  }
  return n;
}

template <int TA, int TB>
static int launch_gemm_c2(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                          GemmParams p, cudaStream_t stream) {
  auto kernel = gemm_bf16_tn_c2_kernel<TA, TB>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C2_SMEM_BYTES) !=
        cudaSuccess)
      return SB_ERR_CUDA;
    attr_set = true;
  }
  p.n_tiles = (p.N + C2_BN - 1) / C2_BN;
  p.m_pairs = (p.m_tiles + 1) / 2;
  const int total = p.m_pairs * p.n_tiles * p.split_k;
  int clusters = c2_max_clusters();
  if (clusters <= 0) return SB_ERR_UNSUPPORTED;
  if (clusters > total) clusters = total;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * clusters);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = C2_SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, ta, tb, tc, p) == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

template <int BN>
static int launch_gemm_bn(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          bool a_mn, bool b_mn, cudaStream_t stream) {
  if (a_mn) return b_mn ? launch_gemm<BN, 1, 1>(ta, tb, p, stream) : launch_gemm<BN, 1, 0>(ta, tb, p, stream);
  return b_mn ? launch_gemm<BN, 0, 1>(ta, tb, p, stream) : launch_gemm<BN, 0, 0>(ta, tb, p, stream);
}

// developer knob (sb_debug_gemm_flags): 1 = the 128 x BN kernel for every shape, 2 = the c2
// kernel stores from the registers, 4 = the c2 kernel stores nothing (timing only)
static int g_gemm_flags = 0;
// which kernel and which epilogue the last sb_gemm_bf16_tn launched (sb_debug_gemm_kernel / _epilogue)
static const char* g_gemm_last = "none";
static const char* g_gemm_epi_last = "none";

}  // namespace sb

using namespace sb;

extern "C" int sb_debug_gemm_flags(int flags) {
  sb::g_gemm_flags = flags;
  return SB_OK;
}
// "c2_128x256" (gemm_bf16_tn_c2_kernel), "128x128" / "128x64" / "128x32" (gemm_bf16_tn_kernel at
// that tile), "none" before the first launch
extern "C" const char* sb_debug_gemm_kernel(void) { return sb::g_gemm_last; }
// "tma" / "tma_reduce" (c2 kernel, tiles staged through shared memory and written by TMA bulk
// stores / reduce-adds), "regs" (stored straight from the registers: every other kernel, and the
// c2 kernel's fall-back), "skipped" (flag 4), "none" before the first launch
extern "C" const char* sb_debug_gemm_epilogue(void) { return sb::g_gemm_epi_last; }

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
  p.m_pairs = 0;
  p.epi = C2_EPI_REGS;
  const bool a_mn = (flags & SB_GEMM_A_MN) != 0;
  const bool b_mn = (flags & SB_GEMM_B_MN) != 0;
  // tile-N choice: N > 128 takes the 128 x 256 tiles of the 2-CTA cluster kernel; narrower GEMMs
  // take 128 x BN tiles of gemm_bf16_tn_kernel (an MN-major B tile is made of 64-wide boxes)
  int bn;
  if (N <= 32 && !b_mn) bn = 32;
  else if (N <= 64) bn = 64;
  else if (N <= 128 || (g_gemm_flags & 1)) bn = 128;
  else bn = C2_BN;
  if (flags & SB_GEMM_ACCUMULATE) {
    // the c2 kernel deals tile pairs to clusters
    const bool c2 = bn == C2_BN;
    const long long units = c2 ? (long long)((p.m_tiles + 1) / 2) * ((N + bn - 1) / bn)
                               : (long long)p.m_tiles * ((N + bn - 1) / bn);
    p.split_k = pick_wave_filling_split(units, c2 ? std::max(c2_max_clusters(), 1) : device_sm_count(),
                                        p.k_blocks_total);
  }
  // tensor maps: K-major operands are [rows][K] with box {64 K, rows}; MN-major operands are
  // [K][rows] with box {64 rows, 64 K}.  The c2 kernel loads half of its 256-row B tile per CTA.
  CUtensorMap ta, tb;
  int rc = a_mn ? make_tmap_bf16_2d(&ta, A, K, M, lda, 64) : make_tmap_bf16_2d(&ta, A, M, K, lda, BM);
  if (rc != SB_OK) return rc;
  rc = b_mn ? make_tmap_bf16_2d(&tb, B, K, N, ldb, 64)
            : make_tmap_bf16_2d(&tb, B, N, K, ldb, bn == C2_BN ? C2_BN / 2 : bn);
  if (rc != SB_OK) return rc;
  // output of the c2 kernel: staged through shared memory and written by TMA, except for a row
  // remap, a C the tensor map cannot describe (base or row pitch not a multiple of 16 bytes) and
  // split-K accumulation (several CTAs add into the same tile), which store from the registers
  CUtensorMap tc;
  memset(&tc, 0, sizeof(tc));
  if (bn == C2_BN) {
    const bool tma_ok = !(flags & SB_GEMM_ROW_REMAP) && (reinterpret_cast<uintptr_t>(C) & 15) == 0 &&
                        ((ldc * 4) & 15) == 0 && !(g_gemm_flags & 2);
    if (g_gemm_flags & 4) p.epi = C2_EPI_NONE;
    else if (tma_ok && !(flags & SB_GEMM_ACCUMULATE)) p.epi = C2_EPI_TMA;
    else if (tma_ok && p.split_k == 1) p.epi = C2_EPI_TMA_REDUCE;
    if (p.epi == C2_EPI_TMA || p.epi == C2_EPI_TMA_REDUCE) {
      rc = make_tmap_f32_c(&tc, C, M, N, ldc);
      if (rc != SB_OK) return rc;
    }
  }
  switch (bn) {
    case 32: g_gemm_last = "128x32"; g_gemm_epi_last = "regs"; return launch_gemm_bn<32>(ta, tb, p, a_mn, b_mn, stream);
    case 64: g_gemm_last = "128x64"; g_gemm_epi_last = "regs"; return launch_gemm_bn<64>(ta, tb, p, a_mn, b_mn, stream);
    case 128: g_gemm_last = "128x128"; g_gemm_epi_last = "regs"; return launch_gemm_bn<128>(ta, tb, p, a_mn, b_mn, stream);
    default:
      g_gemm_last = "c2_128x256";
      g_gemm_epi_last = p.epi == C2_EPI_TMA ? "tma" : p.epi == C2_EPI_TMA_REDUCE ? "tma_reduce"
                      : p.epi == C2_EPI_NONE ? "skipped" : "regs";
      if (a_mn) return b_mn ? launch_gemm_c2<1, 1>(ta, tb, tc, p, stream) : launch_gemm_c2<1, 0>(ta, tb, tc, p, stream);
      return b_mn ? launch_gemm_c2<0, 1>(ta, tb, tc, p, stream) : launch_gemm_c2<0, 0>(ta, tb, tc, p, stream);
  }
}
