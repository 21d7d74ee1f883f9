// Persistent GRU recurrence kernels (forward and backward in time) for sm_90a.
//
// Replaces the cuDNN RNN reached through nn.GRU in the reference encoder
// (speech/models/model.py:35-39 construction, :73 call; gate order r,z,n; bidirectional halves
// are summed by the caller, model.py:75-77) and the pred-net GRU of the transducer
// (speech/models/transducer_model.py:23-26,68).
//
// The time-batched input projection gi = X W_ih^T + b_ih is done for all T at once by
// sb_gemm_bf16_tn; these kernels run the T-serial part.  One cooperative launch per layer covers
// BOTH directions:
//   * CTA c of direction d owns 16 hidden units j0..j0+15: its 48 rows of W_hh (r,z,n) stay
//     resident in shared memory (bf16, wgmma K-major SWIZZLE_128B chunks) for all T steps;
//   * per step every CTA needs ALL of h_{t-1} (bf16, written by the CTAs of its direction in the
//     previous step).  CTAs form thread-block clusters of up to 8; each CTA fetches 1/CS of the
//     [Bp x 64] chunks with TMA and MULTICASTS them into the shared memory of all CTAs of its
//     cluster, so L2 is read once per cluster instead of once per CTA (the un-multicast version
//     was bound by 64 SMs hammering the same L2 lines: 4 us of a 13 us step);
//   * one warpgroup issues wgmma  D[batch x 48] += h_{t-1}[batch x 64] * Wslice[48 x 64]^T
//     (one m64 block per 64 batch rows) per chunk as its mbarrier completes, accumulates in
//     registers and parks the finished product in shared memory;
//   * 8 epilogue warps (thread = batch row, 8 hidden units each) read the product back, apply
//     the gate math in fp32 (h_{t-1} of the thread's own units
//     stays in registers across steps), publish the bf16 h_t, arrive on the per-direction grid
//     barrier, and only then write the fp32 state / transposed copy / saved gates;
//   * the grid barrier is one red.release.gpu + ld.acquire.gpu polling on a global counter.
// The backward kernel has the same structure with W_hh^T resident (16 rows x 3H) and the
// all-gather over the pre-activation gradients dgh_t (batch x 3H).
//
// Roofline: tensor work, but each step is bound by the all-gather + barrier latency
// (tools/gru_timeline.py prints the per-step timeline).
#include "common.cuh"
#include <cuda.h>
#include <string.h>
#include <algorithm>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int GRU_HC = 16;            // hidden units per CTA
static constexpr int GRU_UPT = 8;            // hidden units per epilogue thread
static constexpr int GRU_MAX_RING = 16;      // smem ring slots for the gathered operand
static constexpr int GRU_EPI = 256;          // warps 0..7: epilogue
static constexpr int GRU_MMA_WARP = 8;       // warps 8..11: the wgmma warpgroup
static constexpr int GRU_TMA_WARP = 12;      // warp 12: TMA producer
static constexpr int GRU_THREADS = GRU_EPI + 128 + 32;

typedef __nv_bfloat16 bf16;

struct GruFwdParams {
  const float* gi;     // [T*Bp][ndir*3H]  input projections (b_ih already added)
  const bf16* whh;     // [ndir][3H][H]    recurrent weights, bf16
  const float* bhh;    // [ndir][3H]
  float* y;            // [T*Bp][ndir*H]   h_t fp32
  bf16* xn;            // [T*Bp][ndir*H]   h_t bf16 (operand of the next projection)
  bf16* xnT;           // [ndir*H][(T+2)*Bp] h_t bf16 transposed, column (t+1)*Bp+b ; may be null
  float* gates;        // [T*Bp][ndir][4][H] saved r,z,n,hn for backward ; may be null
  unsigned int* barrier;  // [ndir] zero-initialised counters
  unsigned long long* dbg;  // optional timeline (CTA 0): [step][16] globaltimer stamps, or null
  int T, Bp, H, ndir, ring, gc;   // ring: slots (groups of gc chunks) in shared memory
  int ablate;          // developer knobs: see sb_debug_gru_flags
};

struct GruBwdParams {
  const float* dy;     // [T*Bp][ndir*H]   gradient w.r.t. this layer's output
  const float* y;      // [T*Bp][ndir*H]   forward h_t (fp32)
  const float* gates;  // [T*Bp][ndir][4][H]
  const bf16* whh;     // [ndir][3H][H]    W_hh as stored, bf16 (transposed while staging)
  bf16* dgi;           // [T*Bp][ndir*3H]  d(pre-activation) of the input projection, bf16
  bf16* dghn;          // [T*Bp][ndir*H]   dn_pre * r, token-major (wgrad of W_hn)
  bf16* xchg;          // [ndir][2][Bp][3H] per-step exchange of dgh_t (double-buffered)
  float* dbih;         // [ndir*3H] += sum_{t,b} dgi
  float* dbhh;         // [ndir*3H] += sum_{t,b} dgh
  unsigned int* barrier;  // [ndir]
  unsigned long long* dbg;
  int T, Bp, H, ndir, ring, gc;
  int dir0;            // direction of CTA 0 (gru_bwd_ks_kernel launched for one direction: 0 or 1)
  int ablate;          // developer knobs: see sb_debug_gru_flags
};

SB_DEVINL unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define GRU_STAMP(ev)                                                              \
  do {                                                                             \
    if (p.dbg && blockIdx.x == 0 && step < 64) p.dbg[step * 16 + (ev)] = gtime(); \
  } while (0)

// ---- per-direction grid barrier ------------------------------------------------------------
SB_DEVINL void grid_arrive(unsigned int* ctr) { red_release_gpu_add(ctr, 1u); }
// Polling modes of the grid barrier (developer knob sb_debug_gru_flags bits 64 / 128):
//   0   : ld.acquire.gpu per poll (its implied fence throttles the poll rate)
//   64  : ld.relaxed.gpu + nanosleep per poll, one fence.acq_rel.gpu when the count is complete
//   128 : ld.relaxed.gpu + nanosleep per poll, no fence (the TMA reads that follow go to L2)
// (Un-throttled relaxed polling was measured SLOWER, 7.8 vs 7.3 us/step: the tight spin of 128
// pollers on the counter's L2 line delays the arriving reductions.)
SB_DEVINL void grid_wait(const unsigned int* ctr, unsigned int target, int mode = 0) {
  unsigned int spins = 0;
  if (mode == 0) {
    while (ld_acquire_gpu(ctr) < target) {
      if (++spins > SB_SPIN_LIMIT) __trap();
    }
    return;
  }
  while (ld_relaxed_gpu(ctr) < target) {
    __nanosleep(64);
    if (++spins > SB_SPIN_LIMIT) __trap();
  }
  if (mode & 64) fence_acq_rel_gpu();
}
SB_DEVINL void epi_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(GRU_EPI) : "memory"); }

// ---- cluster helpers ---------------------------------------------------------------------------
SB_DEVINL uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
SB_DEVINL uint32_t cluster_size() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
SB_DEVINL void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// TMA box load multicast to every CTA in `mask` (same smem offset + same mbarrier offset in each)
SB_DEVINL void tma_load_2d_mc(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0,
                              int32_t c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      ".multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
// arrive on the mbarrier at this offset in each of the first `cs` CTAs of the cluster
SB_DEVINL void mbar_arrive_all_ctas(uint64_t* bar, uint32_t cs) {
  for (uint32_t r = 0; r < cs; ++r) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(bar)), "r"(r));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(ra) : "memory");
  }
}

struct GruSmem {
  uint8_t* ring;    // ring slots (stride = Bp*128 bytes), placed BEFORE the weights so that the
                    // 128-row MMA read of the last slot overruns into (finite) weight data
  uint8_t* wtile;   // resident weight chunks
  uint64_t* full;   // [GRU_MAX_RING]
  uint64_t* empty;  // [GRU_MAX_RING]
  uint64_t* accfull;
  float* scratch;   // [64]
  float* accbuf;    // [Bp][N + 4] the finished recurrent product, batch-major
};

SB_DEVINL GruSmem carve(uint8_t* raw, int ring_bytes, int wbytes) {
  GruSmem s;
  s.ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) &
                                      ~static_cast<uintptr_t>(1023));
  s.wtile = s.ring + ring_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s.wtile + wbytes);
  s.full = bars;
  s.empty = bars + GRU_MAX_RING;
  s.accfull = bars + 2 * GRU_MAX_RING;
  s.scratch = reinterpret_cast<float*>(bars + 2 * GRU_MAX_RING + 2);
  s.accbuf = s.scratch + 64;
  return s;
}

// The gathered operand of one step is `nchunks` [Bp x 64] boxes, handled in groups of `gc` chunks
// that share ONE full/empty mbarrier pair (an mbarrier wait costs ~100 ns even when it is already
// complete, so per-chunk barriers were 3 us of a 10 us step).  Group g uses ring slot g % ring and
// ngroups % ring == 0, so every slot is used upr = ngroups/ring times per step and the mbarrier
// phase of use (k, g) is k*upr + g/ring for both barriers of the slot.
//
// TMA producer (one thread per CTA).  Every CTA arms its own full barriers; chunk c is fetched
// by the CTA whose cluster rank is c % CS and multicast to the whole cluster.
SB_DEVINL void tma_gather(const GruSmem& s, const CUtensorMap* tm, int row0, int Bp, int nchunks,
                          int ring, int gc, int k, uint32_t rank, uint32_t cs) {
  const int stride = Bp * 128;
  const int ngroups = nchunks / gc;
  const int upr = ngroups / ring;
  const uint16_t mask = (uint16_t)((1u << cs) - 1u);
  for (int g = 0; g < ngroups; ++g) {
    const int slot = g % ring;
    const unsigned int P = (unsigned int)(k * upr + g / ring);
    if (g >= ring) mbar_wait(&s.empty[slot], (P - 1u) & 1u);   // released by ALL CTAs of the cluster
    mbar_expect_tx(&s.full[slot], (uint32_t)(stride * gc));
    for (int i = 0; i < gc; ++i) {
      const int c = g * gc + i;
      if ((uint32_t)c % cs != rank) continue;
      uint8_t* dst = s.ring + (slot * gc + i) * stride;
      if (cs > 1) tma_load_2d_mc(dst, tm, &s.full[slot], c * 64, row0, mask);
      else tma_load_2d(dst, tm, &s.full[slot], c * 64, row0);
    }
  }
}

// MMA warpgroup: consume the step's chunks against the resident weight chunks, one m64 block per
// 64 batch rows, then park D[Bp x N] in s.accbuf (pitch N + 4) and arrive on s.accfull (count 128).
// (TWO: Bp > 64, a second m64 block; a template parameter so that no wgmma sits under a branch.
// The scale-d = 0 first MMA initialises the accumulators.)
template <int N, bool TWO>
SB_DEVINL void mma_consume(const GruSmem& s, int nchunks, int wchunk_bytes, int Bp, int ring,
                           int gc, int k, uint32_t cs) {
  const int stride = Bp * 128;
  const int ngroups = nchunks / gc;
  const int upr = ngroups / ring;
  constexpr bool two = TWO;
  float d0[N / 2], d1[N / 2];
  for (int g = 0; g < ngroups; ++g) {
    const int slot = g % ring;
    const unsigned int P = (unsigned int)(k * upr + g / ring);
    mbar_wait(&s.full[slot], P & 1u);
    wgmma_fence();
    for (int i = 0; i < gc; ++i) {
      const int c = g * gc + i;
      const uint32_t sa = smem_u32(s.ring + (slot * gc + i) * stride);
      const uint64_t da0 = gmma_desc_sw128_kmajor(sa);
      const uint64_t da1 = gmma_desc_sw128_kmajor(sa + 64 * 128);
      const uint64_t db = gmma_desc_sw128_kmajor(smem_u32(s.wtile + c * wchunk_bytes));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t acc = (c > 0 || kk > 0) ? 1u : 0u;
        wgmma_bf16<N>(d0, da0 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), acc);
        if (two) wgmma_bf16<N>(d1, da1 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), acc);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (ring < ngroups && (threadIdx.x & 127) == 0) {
      if (cs > 1) mbar_arrive_all_ctas(&s.empty[slot], cs);   // the slot is free in every CTA
      else mbar_arrive(&s.empty[slot]);
    }
  }
  wgmma_fence_regs(d0);
  wgmma_fence_regs(d1);
  wg_store_rows<N>(d0, s.accbuf, N + 4, 0, Bp);
  if (two) wg_store_rows<N>(d1, s.accbuf, N + 4, 64, Bp);
  mbar_arrive(s.accfull);
}

SB_DEVINL float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
SB_DEVINL float fast_tanh(float x) {
  // 1 - 2/(exp(2x)+1), clamped so exp never overflows (__fdividef(2, inf) is not guaranteed 0)
  const float xc = fminf(fmaxf(x, -15.f), 15.f);
  return 1.0f - __fdividef(2.0f, __expf(2.0f * xc) + 1.0f);
}

// One-touch data (gi, saved gates, dy, fp32 state, GEMM operands written for later kernels) uses
// the streaming cache policy (.cs) so that it does not evict the latency-critical bf16 exchange
// buffers, which every CTA re-reads from L2 each step.
SB_DEVINL void ld8(const float* p, float (&v)[8]) {
  const float4 a = __ldcs(reinterpret_cast<const float4*>(p));
  const float4 b = __ldcs(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
SB_DEVINL void st8(float* p, const float (&v)[8]) {
  __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
  __stcs(reinterpret_cast<float4*>(p) + 1, make_float4(v[4], v[5], v[6], v[7]));
}
SB_DEVINL void st_stream_u4(void* p, uint4 v) { __stcs(reinterpret_cast<uint4*>(p), v); }
SB_DEVINL void st_stream_bf16(bf16* p, float v) {
  const unsigned short u = __bfloat16_as_ushort(__float2bfloat16_rn(v));
  asm volatile("st.global.cs.u16 [%0], %1;" ::"l"(p), "h"(u) : "memory");
}
SB_DEVINL uint4 pack8(const float (&v)[8]) {
  uint4 r;
  r.x = pack_bf16x2(v[0], v[1]); r.y = pack_bf16x2(v[2], v[3]);
  r.z = pack_bf16x2(v[4], v[5]); r.w = pack_bf16x2(v[6], v[7]);
  return r;
}

// =============================================================================================
// forward
// =============================================================================================
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_kernel(const __grid_constant__ CUtensorMap tm_d0, const __grid_constant__ CUtensorMap tm_d1,
               const GruFwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = blockIdx.x / nC;
  const int j0 = (blockIdx.x % nC) * GRU_HC;
  const int nchunks = (H + 63) / 64;
  constexpr int WCHUNK = 48 * 128;  // 48 rows x 64 bf16
  const int ring_bytes = p.ring * p.gc * Bp * 128;
  // the 128-row A read of the last ring slot overruns by (16 KB - stride) into this region
  const int wbytes = max(nchunks * WCHUNK, 16384 - Bp * 128);
  const GruSmem s = carve(smem_raw, ring_bytes, wbytes);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = p.ndir * H;
  const long long ldT = (long long)(T + 2) * Bp;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const uint32_t crank = cluster_rank(), csize = cluster_size();

  // ---- one-time setup: zero ring + weight region, stage the 48 weight rows, barriers ----
  for (int k = tid; k < (ring_bytes + wbytes) / 16; k += GRU_THREADS)
    reinterpret_cast<uint4*>(s.ring)[k] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    const int pieces_per_row = nchunks * 8;
    for (int k = tid; k < 48 * pieces_per_row; k += GRU_THREADS) {
      const int r = k / pieces_per_row, pc = k % pieces_per_row;
      const int g = r / GRU_HC, jj = r % GRU_HC;
      const int col = pc * 8;
      if (col < H) {
        const uint4 v = *reinterpret_cast<const uint4*>(
            p.whh + ((long long)dir * 3 * H + g * H + j0 + jj) * H + col);
        *reinterpret_cast<uint4*>(s.wtile + (pc >> 3) * WCHUNK + sw128_offset(r, pc & 7)) = v;
      }
    }
    if (tid < 48) {
      const int g = tid / GRU_HC, jj = tid % GRU_HC;
      s.scratch[tid] = p.bhh[dir * 3 * H + g * H + j0 + jj];
    }
  }
  if (tid == 0) {
    for (int i = 0; i < GRU_MAX_RING; ++i) {
      mbar_init(&s.full[i], 1);
      mbar_init(&s.empty[i], csize);
    }
    mbar_init(s.accfull, 128);
    mbar_fence_init();
    tma_prefetch_desc(tm);
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();   // peers' barriers are initialised before anyone multicasts into them
  unsigned int* ctr = p.barrier + dir * 32;   // one L2 line per direction

  if (warp == GRU_TMA_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      for (int step = 1; step < T; ++step) {
        const int t = dir == 0 ? step : (T - 1 - step);
        const int tp = dir == 0 ? t - 1 : t + 1;
        grid_wait(ctr, (unsigned int)nC * step);   // all CTAs published h_{tp}
        GRU_STAMP(0);
        // (the writers ran fence.proxy.async before their release; no reader-side proxy fence)
        tma_gather(s, tm, tp * Bp, Bp, nchunks, p.ring, p.gc, step - 1, crank, csize);
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    // ===================== MMA warpgroup =====================
    for (int step = 1; step < T; ++step) {
      if (Bp > 64) mma_consume<48, true>(s, nchunks, WCHUNK, Bp, p.ring, p.gc, step - 1, csize);
      else mma_consume<48, false>(s, nchunks, WCHUNK, Bp, p.ring, p.gc, step - 1, csize);
      if (tid == GRU_MMA_WARP * 32) GRU_STAMP(2);
    }
  } else {
    // ===================== epilogue: thread = (batch row, half of the 16 units) ==============
    const int row = (warp & 3) * 32 + lane;      // batch row
    const int uh = warp >> 2;                    // which 8 of the CTA's 16 units
    const int ju = j0 + uh * GRU_UPT;
    float hprev[GRU_UPT];
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) hprev[jj] = 0.f;
    float bias[3][GRU_UPT];
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
      for (int jj = 0; jj < GRU_UPT; ++jj) bias[g][jj] = s.scratch[g * 16 + uh * GRU_UPT + jj];
    const bool active = row < Bp;
    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? step : (T - 1 - step);
      // this step's input projections do not depend on the recurrence: fetch them first
      float gi[3][GRU_UPT];
      if (active) {
        const float* g = p.gi + ((long long)t * Bp + row) * (p.ndir * 3 * H) + dir * 3 * H + ju;
#pragma unroll
        for (int gg = 0; gg < 3; ++gg) ld8(g + gg * H, gi[gg]);
      }
      float acc[3][GRU_UPT];
      if (step > 0) {
        mbar_wait(s.accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        const float* ar = s.accbuf + row * (48 + 4) + uh * GRU_UPT;
#pragma unroll
        for (int gg = 0; gg < 3; ++gg)
#pragma unroll
          for (int jj = 0; jj < GRU_UPT; ++jj) acc[gg][jj] = active ? ar[gg * 16 + jj] : 0.f;
        if (tid == 0) GRU_STAMP(4);
      } else {
#pragma unroll
        for (int gg = 0; gg < 3; ++gg)
#pragma unroll
          for (int jj = 0; jj < GRU_UPT; ++jj) acc[gg][jj] = 0.f;
      }
      const long long m = (long long)t * Bp + row;
      float hn[GRU_UPT], rr[GRU_UPT], zz[GRU_UPT], nn[GRU_UPT];
      if (active) {
#pragma unroll
        for (int jj = 0; jj < GRU_UPT; ++jj) {
          rr[jj] = fast_sigmoid(gi[0][jj] + acc[0][jj] + bias[0][jj]);
          zz[jj] = fast_sigmoid(gi[1][jj] + acc[1][jj] + bias[1][jj]);
          hn[jj] = acc[2][jj] + bias[2][jj];
          nn[jj] = fast_tanh(gi[2][jj] + rr[jj] * hn[jj]);
          hprev[jj] = (1.f - zz[jj]) * nn[jj] + zz[jj] * hprev[jj];
        }
        // critical path: only the bf16 h_t that the other CTAs gather next step
        *reinterpret_cast<uint4*>(p.xn + m * D + dir * H + ju) = pack8(hprev);
        if (tid == 0) GRU_STAMP(5);
        if (!(p.ablate & 1)) fence_proxy_async_global();   // generic writes -> other CTAs' TMA reads
        if (tid == 0) GRU_STAMP(6);
      }
      epi_barrier();
      if (tid == 0) {
        GRU_STAMP(7);
        grid_arrive(ctr);          // release: cumulative over the CTA's writes ordered by bar.sync
        GRU_STAMP(9);
      }
      // off the critical path: fp32 state, transposed copy, saved gates
      if (active && !(p.ablate & 2)) {
        st8(p.y + m * D + dir * H + ju, hprev);
        if (p.xnT) {
          bf16* xt = p.xnT + (long long)(dir * H + ju) * ldT + (long long)(t + 1) * Bp + row;
#pragma unroll
          for (int jj = 0; jj < GRU_UPT; ++jj) st_stream_bf16(xt + jj * ldT, hprev[jj]);
        }
        if (p.gates) {
          float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
          st8(go, rr);
          st8(go + H, zz);
          st8(go + 2 * H, nn);
          st8(go + 3 * H, hn);
        }
      }
      if (tid == 0) GRU_STAMP(10);
    }
  }

  __syncthreads();
  cluster_sync_all();   // no CTA leaves while peers may still signal its barriers
}

// =============================================================================================
// backward (reverse of the forward time order of each direction)
// =============================================================================================
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_bwd_kernel(const __grid_constant__ CUtensorMap tm_d0, const __grid_constant__ CUtensorMap tm_d1,
               const GruBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = blockIdx.x / nC;
  const int j0 = (blockIdx.x % nC) * GRU_HC;
  const int K3 = 3 * H;
  const int nchunks = (K3 + 63) / 64;
  constexpr int WCHUNK = 16 * 128;  // 16 rows x 64 bf16
  const int ring_bytes = p.ring * p.gc * Bp * 128;
  const int wbytes = max(nchunks * WCHUNK, 16384 - Bp * 128);
  const GruSmem s = carve(smem_raw, ring_bytes, wbytes);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = p.ndir * H;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const uint32_t crank = cluster_rank(), csize = cluster_size();

  for (int k = tid; k < (ring_bytes + wbytes) / 16; k += GRU_THREADS)
    reinterpret_cast<uint4*>(s.ring)[k] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    // resident operand: rows = the 16 hidden units j0..j0+15 of W_hh^T, K = 3H.  W_hh is read as
    // stored ([3H][H]: 32 contiguous bytes per k) and transposed on the way into shared memory
    for (int k = tid; k < K3 * 2; k += GRU_THREADS) {
      const int kk = k >> 1, half = k & 1;
      const uint4 v = *reinterpret_cast<const uint4*>(
          p.whh + ((long long)dir * K3 + kk) * H + j0 + half * 8);
      const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
      uint8_t* chunk = s.wtile + (kk >> 6) * WCHUNK + (kk & 7) * 2;
#pragma unroll
      for (int q = 0; q < 8; ++q)
        *reinterpret_cast<unsigned short*>(
            chunk + sw128_offset((uint32_t)(half * 8 + q), (uint32_t)((kk & 63) >> 3))) = e[q];
    }
  }
  if (tid == 0) {
    for (int i = 0; i < GRU_MAX_RING; ++i) {
      mbar_init(&s.full[i], 1);
      mbar_init(&s.empty[i], csize);
    }
    mbar_init(s.accfull, 128);
    mbar_fence_init();
    tma_prefetch_desc(tm);
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();
  unsigned int* ctr = p.barrier + dir * 32;   // one L2 line per direction

  if (warp == GRU_TMA_WARP) {
    if (lane == 0) {
      // the recurrent product is needed for every step except the last one processed
      for (int step = 0; step + 1 < T; ++step) {
        grid_wait(ctr, (unsigned int)nC * (step + 1));   // dgh of this step is complete
        GRU_STAMP(0);
        tma_gather(s, tm, (step & 1) * Bp, Bp, nchunks, p.ring, p.gc, step, crank, csize);
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    for (int step = 0; step + 1 < T; ++step) {
      if (Bp > 64) mma_consume<16, true>(s, nchunks, WCHUNK, Bp, p.ring, p.gc, step, csize);
      else mma_consume<16, false>(s, nchunks, WCHUNK, Bp, p.ring, p.gc, step, csize);
      if (tid == GRU_MMA_WARP * 32) GRU_STAMP(2);
    }
  } else {
    const int row = (warp & 3) * 32 + lane;
    const int uh = warp >> 2;
    const int ju = j0 + uh * GRU_UPT;
    const bool active = row < Bp;
    float dh_rec[GRU_UPT];   // dL/dh_t arriving through the recurrence (own units)
    float db_r[GRU_UPT], db_z[GRU_UPT], db_n[GRU_UPT], db_hn[GRU_UPT];
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) {
      dh_rec[jj] = 0.f; db_r[jj] = 0.f; db_z[jj] = 0.f; db_n[jj] = 0.f; db_hn[jj] = 0.f;
    }

    for (int step = 0; step < T; ++step) {
      // forward order of dir 0 is t=0..T-1, so its backward order is T-1..0; dir 1 mirrored
      const int t = dir == 0 ? (T - 1 - step) : step;
      const int tp = dir == 0 ? t - 1 : t + 1;       // time index of h_{prev} in forward order
      const bool has_prev = dir == 0 ? (t > 0) : (t < T - 1);
      bf16* xb = p.xchg + ((long long)(dir * 2 + (step & 1)) * Bp) * K3;
      const long long m = (long long)t * Bp + row;
      // ---- saved activations of this step: independent of the recurrence, fetched first ----
      float rr[GRU_UPT], zz[GRU_UPT], nn[GRU_UPT], hn[GRU_UPT], dh[GRU_UPT], hp[GRU_UPT];
      if (active) {
        const float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
        ld8(go, rr);
        ld8(go + H, zz);
        ld8(go + 2 * H, nn);
        ld8(go + 3 * H, hn);
        ld8(p.dy + m * D + dir * H + ju, dh);
        if (has_prev) {
          ld8(p.y + ((long long)tp * Bp + row) * D + dir * H + ju, hp);
        } else {
#pragma unroll
          for (int jj = 0; jj < GRU_UPT; ++jj) hp[jj] = 0.f;
        }
      }
      // ---- recurrent part of dL/dh_t: product issued in the previous step ----
      if (step > 0) {
        mbar_wait(s.accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        const float* ar = s.accbuf + row * (16 + 4) + uh * GRU_UPT;
        if (tid == 0) GRU_STAMP(4);
#pragma unroll
        for (int jj = 0; jj < GRU_UPT; ++jj) dh_rec[jj] += active ? ar[jj] : 0.f;
      }
      float dr[GRU_UPT], dz[GRU_UPT], dn[GRU_UPT], dnr[GRU_UPT];
      if (active) {
#pragma unroll
        for (int jj = 0; jj < GRU_UPT; ++jj) {
          const float g = dh[jj] + dh_rec[jj];
          dn[jj] = g * (1.f - zz[jj]) * (1.f - nn[jj] * nn[jj]);
          dz[jj] = g * (hp[jj] - nn[jj]) * zz[jj] * (1.f - zz[jj]);
          dr[jj] = dn[jj] * hn[jj] * rr[jj] * (1.f - rr[jj]);
          dnr[jj] = dn[jj] * rr[jj];
          dh_rec[jj] = g * zz[jj];      // direct path h_{t-1} -> h_t; the W_hh path is added next step
          db_r[jj] += dr[jj];
          db_z[jj] += dz[jj];
          db_n[jj] += dn[jj];
          db_hn[jj] += dnr[jj];
        }
        // critical path: the exchange rows [dr | dz | dn*r] every CTA gathers for the product
        if (step + 1 < T) {
          bf16* x = xb + (long long)row * K3 + ju;
          *reinterpret_cast<uint4*>(x) = pack8(dr);
          *reinterpret_cast<uint4*>(x + H) = pack8(dz);
          *reinterpret_cast<uint4*>(x + 2 * H) = pack8(dnr);
          if (tid == 0) GRU_STAMP(5);
          fence_proxy_async_global();
          if (tid == 0) GRU_STAMP(6);
        }
      }
      if (step + 1 < T) {
        epi_barrier();
        if (tid == 0) {
          GRU_STAMP(7);
          grid_arrive(ctr);
          GRU_STAMP(9);
        }
      }
      // ---- off the critical path: operands of the dX / dW GEMMs ----
      if (active) {
        bf16* o = p.dgi + m * (p.ndir * K3) + dir * K3 + ju;
        st_stream_u4(o, pack8(dr));
        st_stream_u4(o + H, pack8(dz));
        st_stream_u4(o + 2 * H, pack8(dn));
        st_stream_u4(p.dghn + m * D + dir * H + ju, pack8(dnr));
      }
      if (tid == 0) GRU_STAMP(10);
    }
    // ---- bias gradients: reduce the per-batch-row partial sums over the CTA ----
    epi_barrier();
    float* red = s.scratch;  // [64]: r(16) z(16) n(16) hn(16)
    if (tid < 64) red[tid] = 0.f;
    epi_barrier();
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) {
      const float a = warp_sum(active ? db_r[jj] : 0.f);
      const float b = warp_sum(active ? db_z[jj] : 0.f);
      const float c = warp_sum(active ? db_n[jj] : 0.f);
      const float d = warp_sum(active ? db_hn[jj] : 0.f);
      if (lane == 0) {
        atomicAdd(&red[uh * GRU_UPT + jj], a);
        atomicAdd(&red[16 + uh * GRU_UPT + jj], b);
        atomicAdd(&red[32 + uh * GRU_UPT + jj], c);
        atomicAdd(&red[48 + uh * GRU_UPT + jj], d);
      }
    }
    epi_barrier();
    if (tid < 48) {
      const int g = tid / GRU_HC, jj = tid % GRU_HC;
      const int idx = dir * K3 + g * H + j0 + jj;
      atomicAdd(p.dbih + idx, red[tid]);
      atomicAdd(p.dbhh + idx, g < 2 ? red[tid] : red[48 + jj]);
    }
  }

  __syncthreads();
  cluster_sync_all();
}

// =============================================================================================
// backward, K-split variant: the 4 CTAs of a cluster jointly own 64 hidden units.
//
// The plain backward kernel makes every CTA gather ALL of dgh_t (Bp x 3H bf16 = 384 KB at the
// north-star size) every step; with 96 KB of weights resident only 128 KB can be in flight, so
// the gather alone costs ~9 us of the 15.8 us step.  Here CTA r of a cluster contracts only the
// r-th QUARTER of the K = 3H dimension, for all 64 units of its cluster:
//     D_r[batch x 64] = dgh_t[:, quarter r] * W_hh[quarter r, 64 units]          (96 KB gathered)
// and the four partial products are reduce-scattered through distributed shared memory: each
// epilogue thread pushes the three 8-float slices that belong to peer CTAs with st.shared::cluster
// and arrives (release.cluster) on the peer's mbarrier; the owner adds the three slices it received
// to its own.  12 KB of DSMEM traffic replaces 288 KB of L2 reads per CTA per step.
// Requires cluster size 4, H % 256 == 0.
// =============================================================================================
static constexpr int KS = 4;

SB_DEVINL uint32_t mapa_shared(uint32_t local_addr, uint32_t peer) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(peer));
  return r;
}
SB_DEVINL void st_cluster_f4(uint32_t raddr, float4 v) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(raddr), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
SB_DEVINL void mbar_arrive_remote_release(uint32_t raddr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(raddr)
               : "memory");
}
SB_DEVINL void mbar_wait_acquire_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0, ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (!ok && ++spins > SB_SPIN_LIMIT) __trap();
  }
}

// bulk copy from this CTA's shared memory into a PEER's shared memory (DSMEM through the copy
// engine), completing `bytes` on the peer's mbarrier.  Measured: pushing the reduce-scatter
// slices with per-thread st.shared::cluster took 4.1 us for 36 KB (~9 KB/us per SM).
SB_DEVINL void bulk_s2peer(uint32_t peer_dst, const void* local_src, uint32_t bytes,
                           uint32_t peer_bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(peer_dst), "r"(smem_u32(local_src)), "r"(bytes), "r"(peer_bar)
      : "memory");
}

__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_bwd_ks_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = p.dir0 + blockIdx.x / nC;
  const int cta_in_dir = blockIdx.x % nC;
  const int j0 = cta_in_dir * GRU_HC;                 // own 16 units (elementwise work)
  const uint32_t crank = cluster_rank();              // == cta_in_dir % 4
  const int k0c = (cta_in_dir / KS) * (KS * GRU_HC);  // first of the cluster's 64 units
  const int K3 = 3 * H;
  const int KQ = K3 / KS;                             // this CTA's share of the contraction
  const int nchunks = KQ / 64;
  constexpr int WCHUNK = 64 * 128;                    // 64 rows (units) x 64 bf16
  const int stride = Bp * 128;
  const int ring_bytes = nchunks * stride;            // the whole quarter is resident
  const int wbytes = nchunks * WCHUNK;
  // carve: ring | weights | recv | barriers
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* ring = base;
  uint8_t* wtile = ring + ring_bytes;
  float* recv = reinterpret_cast<float*>(wtile + wbytes);          // [KS][Bp][16] from peer src
  float* stage = recv + KS * Bp * 16;                              // [KS][Bp][16] for peer dst
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage + KS * Bp * 16);
  uint64_t* full = bars;          // [4] groups
  uint64_t* accfull = bars + 4;
  uint64_t* recvbar = bars + 5;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = p.ndir * H;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const int gc = (nchunks % 4 == 0) ? 4 : ((nchunks % 3 == 0) ? 3 : ((nchunks % 2 == 0) ? 2 : 1));
  const int ngroups = nchunks / gc;                   // <= 4 for H <= 1024 ... checked on host

  for (int k = tid; k < (ring_bytes + wbytes + 2 * KS * Bp * 64) / 16; k += GRU_THREADS)
    reinterpret_cast<uint4*>(base)[k] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    // resident operand: rows = the cluster's 64 units of W_hh^T, columns = this CTA's K quarter.
    // W_hh is read as stored ([3H][H]: the cluster's 64 units are 128 contiguous bytes of row k)
    // and transposed on the way into shared memory (once per launch)
    for (int k = tid; k < KQ * 8; k += GRU_THREADS) {
      const int kl = k >> 3, piece = k & 7;       // local k, 8-unit piece of the 64 units
      const uint4 v = *reinterpret_cast<const uint4*>(
          p.whh + ((long long)dir * K3 + (long long)crank * KQ + kl) * H + k0c + piece * 8);
      const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
      uint8_t* chunk = wtile + (kl >> 6) * WCHUNK + (kl & 7) * 2;
#pragma unroll
      for (int q = 0; q < 8; ++q)
        *reinterpret_cast<unsigned short*>(
            chunk + sw128_offset((uint32_t)(piece * 8 + q), (uint32_t)((kl & 63) >> 3))) = e[q];
    }
  }
  if (tid == 0) {
    for (int i = 0; i < 4; ++i) mbar_init(&full[i], 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);   // one local arrive.expect_tx per step; the peers' copies complete_tx
    mbar_fence_init();
    tma_prefetch_desc(tm);
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();
  unsigned int* ctr = p.barrier + dir * 32;   // one L2 line per direction

  if (warp == GRU_TMA_WARP) {
    if (lane == 0) {
      // step = the epilogue step that consumes the product (as in the forward kernels)
      for (int step = 1; step < T; ++step) {
        grid_wait(ctr, (unsigned int)nC * step, p.ablate & 192);   // dgh of step - 1 is complete
        GRU_STAMP(0);
        for (int g = 0; g < ngroups; ++g) {
          mbar_expect_tx(&full[g], (uint32_t)(stride * gc));
          for (int i = 0; i < gc; ++i) {
            const int c = g * gc + i;
            tma_load_2d(ring + c * stride, tm, &full[g], (int)crank * KQ + c * 64,
                        ((step - 1) & 1) * Bp);
          }
        }
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    // ===================== MMA warpgroup: D[Bp x 64 units] for this K quarter ===============
    // The product is written straight into the reduce-scatter buffers: the 16 columns of peer pr
    // into stage[pr], the CTA's own 16 columns into recv[crank] (which no peer writes).
    const int t = tid & 127;
    const bool two = Bp > 64;                 // batch rows 64..127: a second m64 block
    for (int step = 1; step < T; ++step) {
      float d[2][32];   // initialised by the scale-d = 0 first MMA (d[1] only used if two)
      for (int g = 0; g < ngroups; ++g) {
        mbar_wait(&full[g], (step - 1) & 1);
        wgmma_fence();
        for (int i = 0; i < gc; ++i) {
          const int c = g * gc + i;
          const uint32_t sa = smem_u32(ring + c * stride);
          const uint64_t da0 = gmma_desc_sw128_kmajor(sa);
          const uint64_t da1 = gmma_desc_sw128_kmajor(sa + 64 * 128);
          const uint64_t db = gmma_desc_sw128_kmajor(smem_u32(wtile + c * WCHUNK));
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint32_t acc = (c > 0 || kk > 0) ? 1u : 0u;
            wgmma_bf16<64>(d[0], da0 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), acc);
            if (two) wgmma_bf16<64>(d[1], da1 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), acc);
          }
        }
        wgmma_commit();
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d[0]);
      wgmma_fence_regs(d[1]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int r = h * 64 + wg_frag_row(t, i), col = wg_frag_col(t, i);
          const uint32_t pr = (uint32_t)(col >> 4);
          if (r < Bp)
            (pr == crank ? recv : stage)[((size_t)pr * Bp + r) * 16 + (col & 15)] = d[h][i];
        }
      }
      fence_proxy_async_smem();   // generic st.shared -> the bulk copies (async proxy) to the peers
      mbar_arrive(accfull);
      if (t == 0) GRU_STAMP(2);
    }
  } else {
    const int row = (warp & 3) * 32 + lane;
    const int uh = warp >> 2;
    const int ju = j0 + uh * GRU_UPT;
    const bool active = row < Bp;
    float dh_rec[GRU_UPT];
    float db_r[GRU_UPT], db_z[GRU_UPT], db_n[GRU_UPT], db_hn[GRU_UPT];
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) {
      dh_rec[jj] = 0.f; db_r[jj] = 0.f; db_z[jj] = 0.f; db_n[jj] = 0.f; db_hn[jj] = 0.f;
    }

    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? (T - 1 - step) : step;
      const int tp = dir == 0 ? t - 1 : t + 1;
      const bool has_prev = dir == 0 ? (t > 0) : (t < T - 1);
      bf16* xb = p.xchg + ((long long)(dir * 2 + (step & 1)) * Bp) * K3;
      const long long m = (long long)t * Bp + row;
      float rr[GRU_UPT], zz[GRU_UPT], nn[GRU_UPT], hn[GRU_UPT], dh[GRU_UPT], hp[GRU_UPT];
      if (active) {
        const float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
        ld8(go, rr);
        ld8(go + H, zz);
        ld8(go + 2 * H, nn);
        ld8(go + 3 * H, hn);
        ld8(p.dy + m * D + dir * H + ju, dh);
        if (has_prev) {
          ld8(p.y + ((long long)tp * Bp + row) * D + dir * H + ju, hp);
        } else {
#pragma unroll
          for (int jj = 0; jj < GRU_UPT; ++jj) hp[jj] = 0.f;
        }
      }
      // ---- recurrent part of dL/dh_t: reduce-scatter of the four partial products ----
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        // the MMA warpgroup staged the peers' slices: one bulk copy into each peer's receive
        // buffer; the own slice already sits in recv[crank]
        if (tid == 0) {
          mbar_expect_tx(recvbar, (uint32_t)((KS - 1) * Bp * 16 * 4));
          for (uint32_t q = 1; q < KS; ++q) {
            const uint32_t pr = (crank + q) % KS;
            bulk_s2peer(mapa_shared(smem_u32(recv + (size_t)crank * Bp * 16), pr),
                        stage + (size_t)pr * Bp * 16, (uint32_t)(Bp * 16 * 4),
                        mapa_shared(smem_u32(recvbar), pr));
          }
        }
        if (tid == 0) GRU_STAMP(4);
        mbar_wait(recvbar, (step - 1) & 1);
        if (active) {
#pragma unroll
          for (int src = 0; src < KS; ++src) {
            const float4* rp = reinterpret_cast<const float4*>(
                recv + ((size_t)src * Bp + row) * 16 + uh * GRU_UPT);
            const float4 a = rp[0], b = rp[1];
            dh_rec[0] += a.x; dh_rec[1] += a.y; dh_rec[2] += a.z; dh_rec[3] += a.w;
            dh_rec[4] += b.x; dh_rec[5] += b.y; dh_rec[6] += b.z; dh_rec[7] += b.w;
          }
        }
      }
      float dr[GRU_UPT], dz[GRU_UPT], dn[GRU_UPT], dnr[GRU_UPT];
      if (active) {
#pragma unroll
        for (int jj = 0; jj < GRU_UPT; ++jj) {
          const float g = dh[jj] + dh_rec[jj];
          dn[jj] = g * (1.f - zz[jj]) * (1.f - nn[jj] * nn[jj]);
          dz[jj] = g * (hp[jj] - nn[jj]) * zz[jj] * (1.f - zz[jj]);
          dr[jj] = dn[jj] * hn[jj] * rr[jj] * (1.f - rr[jj]);
          dnr[jj] = dn[jj] * rr[jj];
          dh_rec[jj] = g * zz[jj];
          db_r[jj] += dr[jj];
          db_z[jj] += dz[jj];
          db_n[jj] += dn[jj];
          db_hn[jj] += dnr[jj];
        }
        if (step + 1 < T) {
          bf16* x = xb + (long long)row * K3 + ju;
          *reinterpret_cast<uint4*>(x) = pack8(dr);
          *reinterpret_cast<uint4*>(x + H) = pack8(dz);
          *reinterpret_cast<uint4*>(x + 2 * H) = pack8(dnr);
          if (tid == 0) GRU_STAMP(5);
          if (!(p.ablate & 1)) fence_proxy_async_global();
          if (tid == 0) GRU_STAMP(6);
        }
      }
      if (step + 1 < T) {
        epi_barrier();
        if (tid == 0) {
          GRU_STAMP(7);
          grid_arrive(ctr);
          GRU_STAMP(9);
        }
      }
      if (active && !(p.ablate & 2)) {
        bf16* o = p.dgi + m * (p.ndir * K3) + dir * K3 + ju;
        st_stream_u4(o, pack8(dr));
        st_stream_u4(o + H, pack8(dz));
        st_stream_u4(o + 2 * H, pack8(dn));
        st_stream_u4(p.dghn + m * D + dir * H + ju, pack8(dnr));
      }
      if (tid == 0) GRU_STAMP(10);
    }
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) {
      const float a = warp_sum(active ? db_r[jj] : 0.f);
      const float b = warp_sum(active ? db_z[jj] : 0.f);
      const float c = warp_sum(active ? db_n[jj] : 0.f);
      const float d = warp_sum(active ? db_hn[jj] : 0.f);
      if (lane == 0) {
        const int bi = dir * K3 + ju + jj;
        atomicAdd(p.dbih + bi, a);
        atomicAdd(p.dbih + bi + H, b);
        atomicAdd(p.dbih + bi + 2 * H, c);
        atomicAdd(p.dbhh + bi, a);
        atomicAdd(p.dbhh + bi + H, b);
        atomicAdd(p.dbhh + bi + 2 * H, d);
      }
    }
  }

  __syncthreads();
  cluster_sync_all();
}

// =============================================================================================
// forward, K-split variant: the 4 CTAs of a cluster jointly own 64 hidden units.
//
// Measured on gru_fwd_kernel (globaltimer timeline, H = 1024, B = 64, 7.4 us/step): 3.5 us pass
// between "h_{t-1} is complete" and "all MMAs retired", for a gather of 128 KB per CTA - the same
// ~30 B/ns per SM whether it is fetched as tensor boxes or as contiguous bulk copies, with or
// without cluster multicast: 128 CTAs x 128 KB = 16 MB of L2->SM traffic per step is the bound,
// next to 480 KB of shared-memory traffic (TMA writes + MMA operand reads of a 128-row A tile).
// Here CTA r of a cluster contracts only the r-th QUARTER of K = H for all 64 units of its
// cluster and all three gates,
//     D_r[batch x 192] = h_{t-1}[:, quarter r] * W_hh[(r|z|n) x 64 units, quarter r]^T,
// i.e. it gathers 32 KB instead of 128 KB (the whole quarter stays resident: no ring) and issues
// 16 MMAs of N = 192 instead of 64 of N = 48; the four partial products are reduce-scattered
// through distributed shared memory exactly as in gru_bwd_ks_kernel (each CTA receives the
// 3 x 16 columns of its own units from its three peers: 36 KB per CTA and step).
// Requires cluster size 4, H % 256 == 0, Bp <= 64.
// =============================================================================================
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_ks_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruFwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = blockIdx.x / nC;
  const int cta_in_dir = blockIdx.x % nC;
  const int j0 = cta_in_dir * GRU_HC;                 // own 16 units (gate math, stores)
  const uint32_t crank = cluster_rank();              // == cta_in_dir % 4
  const int k0c = (cta_in_dir / KS) * (KS * GRU_HC);  // first of the cluster's 64 units
  const int KQ = H / KS;                              // this CTA's share of the contraction
  const int nchunks = KQ / 64;
  constexpr int NCOL = 3 * KS * GRU_HC;               // 192 accumulator columns: gate x 64 units
  constexpr int WCHUNK = NCOL * 128;                  // 192 rows x 64 bf16
  constexpr int RW = 3 * GRU_HC;                      // 48 floats received per row and peer
  const int stride = Bp * 128;
  const int ring_bytes = nchunks * stride;            // the whole quarter is resident
  const int wbytes = nchunks * WCHUNK;
  // carve: ring | weights | recv | barriers.  (The 128-row A read of the last chunk runs past the
  // ring into the weights: finite data, rows >= Bp are never used.)
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* ring = base;
  uint8_t* wtile = ring + ring_bytes;
  float* recv = reinterpret_cast<float*>(wtile + wbytes);          // [KS][Bp][48] from peer src
  float* stage = recv + KS * Bp * RW;                              // [KS][Bp][48] for peer dst
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage + KS * Bp * RW);
  uint64_t* full = bars;
  uint64_t* accfull = bars + 1;
  uint64_t* recvbar = bars + 2;
  float* bias_s = reinterpret_cast<float*>(bars + 4);             // [48]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = p.ndir * H;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;

  for (int k = tid; k < (ring_bytes + wbytes + 2 * KS * Bp * RW * 4) / 16; k += GRU_THREADS)
    reinterpret_cast<uint4*>(base)[k] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    // resident operand: rows = (gate, unit of the cluster), columns = this CTA's K quarter
    const int pieces_per_row = nchunks * 8;
    for (int k = tid; k < NCOL * pieces_per_row; k += GRU_THREADS) {
      const int r = k / pieces_per_row, pc = k % pieces_per_row;
      const int g = r / (KS * GRU_HC), u = r % (KS * GRU_HC);
      const uint4 v = *reinterpret_cast<const uint4*>(
          p.whh + ((long long)dir * 3 * H + (long long)g * H + k0c + u) * H + (long long)crank * KQ +
          pc * 8);
      *reinterpret_cast<uint4*>(wtile + (pc >> 3) * WCHUNK + sw128_offset(r, pc & 7)) = v;
    }
    if (tid < RW) {
      const int g = tid / GRU_HC, jj = tid % GRU_HC;
      bias_s[tid] = p.bhh[dir * 3 * H + g * H + j0 + jj];
    }
  }
  if (tid == 0) {
    mbar_init(full, 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);   // one local arrive.expect_tx per step; the peers' copies complete_tx
    mbar_fence_init();
    tma_prefetch_desc(tm);
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();
  unsigned int* ctr = p.barrier + dir * 32;   // one L2 line per direction

  if (warp == GRU_TMA_WARP) {
    // ===================== TMA producer: this CTA's K quarter of h_{t-1} =====================
    if (lane == 0) {
      for (int step = 1; step < T; ++step) {
        const int t = dir == 0 ? step : (T - 1 - step);
        const int tp = dir == 0 ? t - 1 : t + 1;
        grid_wait(ctr, (unsigned int)nC * step, p.ablate & 192);   // all CTAs published h_{tp}
        GRU_STAMP(0);
        if (p.dbg && step == 21) p.dbg[1024 + 256 + blockIdx.x] = gtime();   // skew probe
        mbar_expect_tx(full, (uint32_t)(stride * nchunks));
        for (int c = 0; c < nchunks; ++c)
          tma_load_2d(ring + c * stride, tm, full, (int)crank * KQ + c * 64, tp * Bp);
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    // ===================== MMA warpgroup: D[Bp x (gate, 64 units)] for this K quarter ========
    // Column gg*64 + pr*16 + u belongs to unit u of peer pr: it is written straight into
    // stage[pr] (row pitch RW = 48, gate-major), the CTA's own columns into recv[crank].
    const int t = tid & 127;
    for (int step = 1; step < T; ++step) {
      float d[NCOL / 2];   // initialised by the scale-d = 0 first MMA
      mbar_wait(full, (step - 1) & 1);
      wgmma_fence();
      for (int c = 0; c < nchunks; ++c) {
        const uint64_t da = gmma_desc_sw128_kmajor(smem_u32(ring + c * stride));
        const uint64_t db = gmma_desc_sw128_kmajor(smem_u32(wtile + c * WCHUNK));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_bf16<NCOL>(d, da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2),
                           (c > 0 || kk > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(d);
#pragma unroll
      for (int i = 0; i < NCOL / 2; ++i) {
        const int r = wg_frag_row(t, i), col = wg_frag_col(t, i);
        const int gg = col >> 6, u = col & 15;
        const uint32_t pr = (uint32_t)((col >> 4) & 3);
        if (r < Bp)
          (pr == crank ? recv : stage)[((size_t)pr * Bp + r) * RW + gg * GRU_HC + u] = d[i];
      }
      fence_proxy_async_smem();   // generic st.shared -> the bulk copies (async proxy) to the peers
      mbar_arrive(accfull);
      if (t == 0) GRU_STAMP(2);
    }
  } else {
    // ===================== epilogue: thread = (batch row, half of the CTA's 16 units) ==========
    const int row = (warp & 3) * 32 + lane;
    const int uh = warp >> 2;
    const int ju = j0 + uh * GRU_UPT;
    const bool active = row < Bp;
    float hprev[GRU_UPT];
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) hprev[jj] = 0.f;
    float bias[3][GRU_UPT];
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
      for (int jj = 0; jj < GRU_UPT; ++jj) bias[g][jj] = bias_s[g * GRU_HC + uh * GRU_UPT + jj];

    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? step : (T - 1 - step);
      float gi[3][GRU_UPT];
      if (active) {
        const float* g = p.gi + ((long long)t * Bp + row) * (p.ndir * 3 * H) + dir * 3 * H + ju;
#pragma unroll
        for (int gg = 0; gg < 3; ++gg) ld8(g + gg * H, gi[gg]);
      }
      float acc[3][GRU_UPT];
#pragma unroll
      for (int gg = 0; gg < 3; ++gg)
#pragma unroll
        for (int jj = 0; jj < GRU_UPT; ++jj) acc[gg][jj] = 0.f;
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        // ---- reduce-scatter of the four partial products: the MMA warpgroup staged the three
        // slices that belong to the peers, each leaves as ONE bulk copy into the peer's receive
        // buffer; the CTA's own slice already sits in recv[crank] ----
        if (tid == 0) {
          mbar_expect_tx(recvbar, (uint32_t)((KS - 1) * Bp * RW * 4));
          for (uint32_t q = 1; q < KS; ++q) {
            const uint32_t pr = (crank + q) % KS;
            bulk_s2peer(mapa_shared(smem_u32(recv + (size_t)crank * Bp * RW), pr),
                        stage + (size_t)pr * Bp * RW, (uint32_t)(Bp * RW * 4),
                        mapa_shared(smem_u32(recvbar), pr));
          }
        }
        if (tid == 0) GRU_STAMP(4);
        mbar_wait(recvbar, (step - 1) & 1);
        if (active) {
#pragma unroll
          for (int src = 0; src < KS; ++src) {
            const float* rp = recv + ((size_t)src * Bp + row) * RW + uh * GRU_UPT;
#pragma unroll
            for (int gg = 0; gg < 3; ++gg) {
              const float4 a = *reinterpret_cast<const float4*>(rp + gg * GRU_HC);
              const float4 b = *reinterpret_cast<const float4*>(rp + gg * GRU_HC + 4);
              acc[gg][0] += a.x; acc[gg][1] += a.y; acc[gg][2] += a.z; acc[gg][3] += a.w;
              acc[gg][4] += b.x; acc[gg][5] += b.y; acc[gg][6] += b.z; acc[gg][7] += b.w;
            }
          }
        }
      }
      const long long m = (long long)t * Bp + row;
      float hn[GRU_UPT], rr[GRU_UPT], zz[GRU_UPT], nn[GRU_UPT];
      if (active) {
#pragma unroll
        for (int jj = 0; jj < GRU_UPT; ++jj) {
          rr[jj] = fast_sigmoid(gi[0][jj] + acc[0][jj] + bias[0][jj]);
          zz[jj] = fast_sigmoid(gi[1][jj] + acc[1][jj] + bias[1][jj]);
          hn[jj] = acc[2][jj] + bias[2][jj];
          nn[jj] = fast_tanh(gi[2][jj] + rr[jj] * hn[jj]);
          hprev[jj] = (1.f - zz[jj]) * nn[jj] + zz[jj] * hprev[jj];
        }
        // critical path: only the bf16 h_t that the other CTAs gather next step
        *reinterpret_cast<uint4*>(p.xn + m * D + dir * H + ju) = pack8(hprev);
        if (tid == 0) GRU_STAMP(5);
        if (!(p.ablate & 1)) fence_proxy_async_global();   // generic writes -> other CTAs' TMA reads
        if (tid == 0) GRU_STAMP(6);
      }
      epi_barrier();
      if (tid == 0) {
        GRU_STAMP(7);
        if (p.dbg && step == 20) p.dbg[1024 + blockIdx.x] = gtime();         // skew probe
        grid_arrive(ctr);
        GRU_STAMP(9);
      }
      if (active && !(p.ablate & 2)) {
        st8(p.y + m * D + dir * H + ju, hprev);
        if (p.gates) {
          float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
          st8(go, rr);
          st8(go + H, zz);
          st8(go + 2 * H, nn);
          st8(go + 3 * H, hn);
        }
      }
      if (tid == 0) GRU_STAMP(10);
    }
  }

  __syncthreads();
  cluster_sync_all();
}

// =============================================================================================
// forward, K split with the accumulator TRANSPOSED: D^T[(gate, unit) x batch].
//
// Same partition as gru_fwd_ks_kernel (cluster of 4 owns 64 units, CTA r contracts K quarter r),
// but the resident weight slice is the M-side operand and h_{t-1} the N-side one:
//     D[192 x NB] = W[(r|z|n) x 64 units, quarter r] * h_{t-1}[:, quarter r]^T
// issued as three wgmma m64 blocks of weight rows with N = NB (the batch rounded up to 16).  The
// batch-major form needs M >= 64 batch rows per m64 block whatever the batch is, so at 8 rows it
// spends 8x the tensor work of this one (N = 192 on 64 mostly empty rows).  The weight rows are
// ordered by OWNER: rows 32q..32q+31 are the r and z rows of the 16 units CTA q of the cluster
// owns, rows 128+16q..128+16q+15 its n rows, so every accumulator row goes to exactly one peer:
// the MMA warpgroup writes it as one row of [48][Bp] (pitch Bp+4) into the staging slice for
// that peer, the three slices leave as one bulk copy each, and the gate math then runs on ALL 256
// epilogue threads (thread = batch row x UPT units) from the four received slices.
// Requires cluster size 4, H % 256 == 0, Bp <= 64 (Bp % 8 == 0 as everywhere).
// =============================================================================================
template <int UPT>
SB_DEVINL void ldu(const float* p, float (&v)[UPT]) {
  if constexpr (UPT == 4) {
    const float4 a = __ldcs(reinterpret_cast<const float4*>(p));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  } else if constexpr (UPT == 2) {
    const float2 a = __ldcs(reinterpret_cast<const float2*>(p));
    v[0] = a.x; v[1] = a.y;
  } else {
    v[0] = __ldcs(p);
  }
}
template <int UPT>
SB_DEVINL void stu(float* p, const float (&v)[UPT]) {
  if constexpr (UPT == 4) __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
  else if constexpr (UPT == 2) __stcs(reinterpret_cast<float2*>(p), make_float2(v[0], v[1]));
  else __stcs(p, v[0]);
}
template <int UPT>
SB_DEVINL void st_bf16u(bf16* p, const float (&v)[UPT]) {
  if constexpr (UPT == 4) {
    *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]));
  } else if constexpr (UPT == 2) {
    *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(v[0], v[1]);
  } else {
    *p = __float2bfloat16_rn(v[0]);
  }
}

// Owner-major staging of the transposed accumulators: slice of peer q (the own slice lives in
// recv[crank], the others in stage[(q - crank) mod KS - 1]), row srow, column = batch row.
SB_DEVINL float* kt_slice(float* recv, float* stage, int slice, uint32_t q, uint32_t crank) {
  const uint32_t q0 = (q + KS - crank) % KS;
  return q0 == 0 ? recv + (size_t)crank * slice : stage + (size_t)(q0 - 1) * slice;
}

// MMA warpgroup of gru_fwd_kt_kernel, one step per iteration: three m64 blocks of weight rows
// (r,z of the cluster's 64 units | n of them) x NB batch rows; the scale-d = 0 first MMA
// initialises the accumulators.
template <int NB>
SB_DEVINL void fwd_kt_mma(uint8_t* ring, uint8_t* wtile, float* recv, float* stage, uint64_t* full,
                          uint64_t* accfull, int nchunks, int stride, int Bp, int P, int slice,
                          uint32_t crank, int T) {
  constexpr int WCHUNK = 3 * KS * GRU_HC * 128;
  const int t = threadIdx.x & 127;
  for (int step = 1; step < T; ++step) {
    float d[3][NB / 2];
    mbar_wait(full, (step - 1) & 1);
    wgmma_fence();
    for (int c = 0; c < nchunks; ++c) {
      const uint32_t wa = smem_u32(wtile + c * WCHUNK);
      const uint64_t db = gmma_desc_sw128_kmajor(smem_u32(ring + c * stride));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t acc = (c > 0 || kk > 0) ? 1u : 0u;
#pragma unroll
        for (int j = 0; j < 3; ++j)
          wgmma_bf16<NB>(d[j], gmma_desc_sw128_kmajor(wa + j * 64 * 128) + (uint64_t)(kk * 2),
                         db + (uint64_t)(kk * 2), acc);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 3; ++j) wgmma_fence_regs(d[j]);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
#pragma unroll
      for (int i = 0; i < NB / 2; ++i) {
        const int r = j * 64 + wg_frag_row(t, i), b = wg_frag_col(t, i);
        const uint32_t q = r < 128 ? (uint32_t)(r >> 5) : (uint32_t)((r - 128) >> 4);
        const int srow = r < 128 ? (r & 31) : 2 * GRU_HC + (r & 15);
        if (b < Bp) kt_slice(recv, stage, slice, q, crank)[srow * P + b] = d[j][i];
      }
    }
    fence_proxy_async_smem();   // generic st.shared -> the bulk copies (async proxy) to the peers
    mbar_arrive(accfull);
  }
}

// MMA warpgroup of gru_bwd_kt_kernel: one m64 block (the cluster's 64 units) x NB batch rows
template <int NB>
SB_DEVINL void bwd_kt_mma(uint8_t* ring, uint8_t* wtile, float* recv, float* stage, uint64_t* full,
                          uint64_t* accfull, int ngroups, int gc, int stride, int Bp, int P,
                          int slice, uint32_t crank, int T) {
  constexpr int WCHUNK = 64 * 128;
  const int t = threadIdx.x & 127;
  for (int step = 0; step + 1 < T; ++step) {
    float d[NB / 2];
    for (int g = 0; g < ngroups; ++g) {
      mbar_wait(&full[g], step & 1);
      wgmma_fence();
      for (int i = 0; i < gc; ++i) {
        const int c = g * gc + i;
        const uint64_t da = gmma_desc_sw128_kmajor(smem_u32(wtile + c * WCHUNK));
        const uint64_t db = gmma_desc_sw128_kmajor(smem_u32(ring + c * stride));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_bf16<NB>(d, da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2),
                         (c > 0 || kk > 0) ? 1u : 0u);
      }
      wgmma_commit();
    }
    wgmma_wait<0>();
    wgmma_fence_regs(d);
#pragma unroll
    for (int i = 0; i < NB / 2; ++i) {
      const int r = wg_frag_row(t, i), b = wg_frag_col(t, i);
      if (b < Bp) kt_slice(recv, stage, slice, (uint32_t)(r >> 4), crank)[(r & 15) * P + b] = d[i];
    }
    fence_proxy_async_smem();
    mbar_arrive(accfull);
  }
}

template <int UPT>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_kt_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruFwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = blockIdx.x / nC;
  const int cta_in_dir = blockIdx.x % nC;
  const int j0 = cta_in_dir * GRU_HC;                 // own 16 units (gate math, stores)
  const uint32_t crank = cluster_rank();              // == cta_in_dir % 4
  const int k0c = (cta_in_dir / KS) * (KS * GRU_HC);  // first of the cluster's 64 units
  const int KQ = H / KS;                              // this CTA's share of the contraction
  const int nchunks = KQ / 64;
  constexpr int WROWS = 3 * KS * GRU_HC;              // 192 weight rows: 128 (r,z) + 64 (n)
  constexpr int WCHUNK = WROWS * 128;                 // 192 rows x 64 bf16
  constexpr int RW = 3 * GRU_HC;                      // 48 accumulator rows per owner
  const int P = Bp + 4;                               // pitch of a staged row (floats)
  const int slice = RW * P;                           // floats per (source, owner) slice
  const int NB = (Bp + 15) & ~15;                     // MMA N (rows of h read per chunk)
  const int stride = Bp * 128;
  const int ring_bytes = nchunks * stride;            // the whole quarter is resident
  const int wbytes = nchunks * WCHUNK;
  // carve: ring | weights | recv | stage | barriers.  The N-side read of the last chunk may run
  // up to 8 rows past the ring into the weights: it only feeds accumulator columns >= Bp, which
  // are never stored.
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* ring = base;
  uint8_t* wtile = ring + ring_bytes;
  float* recv = reinterpret_cast<float*>(wtile + wbytes);          // [KS src][48][P]
  float* stage = recv + KS * slice;                                // [KS-1 dst][48][P]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage + (KS - 1) * slice);
  uint64_t* full = bars;
  uint64_t* accfull = bars + 1;
  uint64_t* recvbar = bars + 2;
  float* bias_s = reinterpret_cast<float*>(bars + 4);             // [48]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = p.ndir * H;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;

  for (int k = tid; k < (ring_bytes + wbytes + (2 * KS - 1) * slice * 4) / 16; k += GRU_THREADS)
    reinterpret_cast<uint4*>(base)[k] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    // resident operand: rows ordered by owner (see above), columns = this CTA's K quarter
    const int pieces_per_row = nchunks * 8;
    for (int k = tid; k < WROWS * pieces_per_row; k += GRU_THREADS) {
      const int r = k / pieces_per_row, pc = k % pieces_per_row;
      int g, u;
      if (r < 128) { g = (r & 31) >> 4; u = (r >> 5) * GRU_HC + (r & 15); }
      else { g = 2; u = r - 128; }
      const uint4 v = *reinterpret_cast<const uint4*>(
          p.whh + ((long long)dir * 3 * H + (long long)g * H + k0c + u) * H + (long long)crank * KQ +
          pc * 8);
      *reinterpret_cast<uint4*>(wtile + (pc >> 3) * WCHUNK + sw128_offset(r, pc & 7)) = v;
    }
    if (tid < RW) {
      const int g = tid / GRU_HC, jj = tid % GRU_HC;
      bias_s[tid] = p.bhh[dir * 3 * H + g * H + j0 + jj];
    }
  }
  if (tid == 0) {
    mbar_init(full, 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);   // one local arrive.expect_tx per step; the peers' copies complete_tx
    mbar_fence_init();
    tma_prefetch_desc(tm);
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();
  unsigned int* ctr = p.barrier + dir * 32;   // one L2 line per direction

  if (warp == GRU_TMA_WARP) {
    // ===================== TMA producer: this CTA's K quarter of h_{t-1} =====================
    if (lane == 0) {
      for (int step = 1; step < T; ++step) {
        const int t = dir == 0 ? step : (T - 1 - step);
        const int tp = dir == 0 ? t - 1 : t + 1;
        grid_wait(ctr, (unsigned int)nC * step, p.ablate & 192);   // all CTAs published h_{tp}
        GRU_STAMP(0);
        if (p.dbg && step == 21) p.dbg[1024 + 256 + blockIdx.x] = gtime();   // skew probe
        mbar_expect_tx(full, (uint32_t)(stride * nchunks));
        for (int c = 0; c < nchunks; ++c)
          tma_load_2d(ring + c * stride, tm, full, (int)crank * KQ + c * 64, tp * Bp);
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    // ===================== MMA warpgroup =====================
    switch (NB) {
      case 16: fwd_kt_mma<16>(ring, wtile, recv, stage, full, accfull, nchunks, stride, Bp, P, slice, crank, T); break;
      case 32: fwd_kt_mma<32>(ring, wtile, recv, stage, full, accfull, nchunks, stride, Bp, P, slice, crank, T); break;
      case 48: fwd_kt_mma<48>(ring, wtile, recv, stage, full, accfull, nchunks, stride, Bp, P, slice, crank, T); break;
      default: fwd_kt_mma<64>(ring, wtile, recv, stage, full, accfull, nchunks, stride, Bp, P, slice, crank, T); break;
    }
  } else {
    // ===================== epilogue =====================
    // phase B (gate math): thread = (batch row b, UPT of the CTA's 16 units)
    const int b = tid % Bp, ug = tid / Bp;
    const bool active = ug * UPT < GRU_HC;
    const int u0 = ug * UPT;
    const int ju = j0 + u0;
    float hprev[UPT];
#pragma unroll
    for (int jj = 0; jj < UPT; ++jj) hprev[jj] = 0.f;
    float bias[3][UPT];
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
      for (int jj = 0; jj < UPT; ++jj) bias[g][jj] = active ? bias_s[g * GRU_HC + u0 + jj] : 0.f;

    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? step : (T - 1 - step);
      float gi[3][UPT];
      if (active) {
        const float* g = p.gi + ((long long)t * Bp + b) * (p.ndir * 3 * H) + dir * 3 * H + ju;
#pragma unroll
        for (int gg = 0; gg < 3; ++gg) ldu<UPT>(g + gg * H, gi[gg]);
      }
      float acc[3][UPT];
#pragma unroll
      for (int gg = 0; gg < 3; ++gg)
#pragma unroll
        for (int jj = 0; jj < UPT; ++jj) acc[gg][jj] = 0.f;
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        // the MMA warpgroup staged the three outgoing slices (and the own one in recv[crank])
        if (tid == 0) mbar_expect_tx(recvbar, (uint32_t)((KS - 1) * slice * 4));
        if (lane == 0 && warp >= 1 && warp <= KS - 1) {
          const uint32_t pr = (crank + (uint32_t)warp) % KS;
          bulk_s2peer(mapa_shared(smem_u32(recv + (size_t)crank * slice), pr),
                      stage + (size_t)(warp - 1) * slice, (uint32_t)(slice * 4),
                      mapa_shared(smem_u32(recvbar), pr));
        }
        if (tid == 0) GRU_STAMP(4);
        mbar_wait(recvbar, (step - 1) & 1);
        if (active) {
#pragma unroll
          for (int src = 0; src < KS; ++src) {
            const float* rp = recv + (size_t)src * slice + u0 * P + b;
#pragma unroll
            for (int gg = 0; gg < 3; ++gg)
#pragma unroll
              for (int jj = 0; jj < UPT; ++jj) acc[gg][jj] += rp[(gg * GRU_HC + jj) * P];
          }
        }
      }
      const long long m = (long long)t * Bp + b;
      float hn[UPT], rr[UPT], zz[UPT], nn[UPT];
      if (active) {
#pragma unroll
        for (int jj = 0; jj < UPT; ++jj) {
          rr[jj] = fast_sigmoid(gi[0][jj] + acc[0][jj] + bias[0][jj]);
          zz[jj] = fast_sigmoid(gi[1][jj] + acc[1][jj] + bias[1][jj]);
          hn[jj] = acc[2][jj] + bias[2][jj];
          nn[jj] = fast_tanh(gi[2][jj] + rr[jj] * hn[jj]);
          hprev[jj] = (1.f - zz[jj]) * nn[jj] + zz[jj] * hprev[jj];
        }
        // critical path: only the bf16 h_t that the other CTAs gather next step
        st_bf16u<UPT>(p.xn + m * D + dir * H + ju, hprev);
        if (tid == 0) GRU_STAMP(5);
        fence_proxy_async_global();   // generic writes -> other CTAs' TMA reads
        if (tid == 0) GRU_STAMP(6);
      }
      epi_barrier();
      if (tid == 0) {
        GRU_STAMP(7);
        if (p.dbg && step == 20) p.dbg[1024 + blockIdx.x] = gtime();         // skew probe
        grid_arrive(ctr);
        GRU_STAMP(9);
      }
      if (active) {
        stu<UPT>(p.y + m * D + dir * H + ju, hprev);
        if (p.gates) {
          float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
          stu<UPT>(go, rr);
          stu<UPT>(go + H, zz);
          stu<UPT>(go + 2 * H, nn);
          stu<UPT>(go + 3 * H, hn);
        }
      }
      if (tid == 0) GRU_STAMP(10);
    }
  }

  __syncthreads();
  cluster_sync_all();
}

// =============================================================================================
// backward, K split with the accumulator TRANSPOSED (see gru_fwd_kt_kernel):
//     D^T[64 units x Bp] = W_hh^T[64 units of the cluster, quarter r of 3H] * dgh[:, quarter r]^T
// issued as one wgmma m64 block of weight rows with N = NB.  The weight tile is the one of
// gru_bwd_ks_kernel (its 64 rows are already grouped by owner: rows 16q..16q+15 belong to CTA q
// of the cluster); an accumulator row is a unit, so its Bp partial sums go to exactly one peer, and the elementwise work runs on all 256
// epilogue threads (thread = batch row x UPT units).
// =============================================================================================
template <int UPT>
SB_DEVINL void st_stream_bf16u(bf16* p, const float (&v)[UPT]) {
  if constexpr (UPT == 4) {
    __stcs(reinterpret_cast<uint2*>(p), make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3])));
  } else if constexpr (UPT == 2) {
    __stcs(reinterpret_cast<unsigned int*>(p), pack_bf16x2(v[0], v[1]));
  } else {
    st_stream_bf16(p, v[0]);
  }
}

template <int UPT>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_bwd_kt_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = blockIdx.x / nC;
  const int cta_in_dir = blockIdx.x % nC;
  const int j0 = cta_in_dir * GRU_HC;                 // own 16 units (elementwise work)
  const uint32_t crank = cluster_rank();              // == cta_in_dir % 4
  const int k0c = (cta_in_dir / KS) * (KS * GRU_HC);  // first of the cluster's 64 units
  const int K3 = 3 * H;
  const int KQ = K3 / KS;                             // this CTA's share of the contraction
  const int nchunks = KQ / 64;
  constexpr int WCHUNK = 64 * 128;                    // 64 rows (units) x 64 bf16
  const int P = Bp + 4;                               // pitch of a staged row (floats)
  const int slice = GRU_HC * P;                       // floats per (source, owner) slice
  const int NB = (Bp + 15) & ~15;
  const int stride = Bp * 128;
  const int ring_bytes = nchunks * stride;            // the whole quarter is resident
  const int wbytes = nchunks * WCHUNK;
  // carve: ring | weights | recv | stage | barriers
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* ring = base;
  uint8_t* wtile = ring + ring_bytes;
  float* recv = reinterpret_cast<float*>(wtile + wbytes);          // [KS src][16][P]
  float* stage = recv + KS * slice;                                // [KS-1 dst][16][P]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage + (KS - 1) * slice);
  uint64_t* full = bars;          // [4] groups
  uint64_t* accfull = bars + 4;
  uint64_t* recvbar = bars + 5;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = p.ndir * H;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const int gc = (nchunks % 4 == 0) ? 4 : ((nchunks % 3 == 0) ? 3 : ((nchunks % 2 == 0) ? 2 : 1));
  const int ngroups = nchunks / gc;                   // <= 4 for H <= 1024 ... checked on host

  for (int k = tid; k < (ring_bytes + wbytes + (2 * KS - 1) * slice * 4) / 16;
       k += GRU_THREADS)
    reinterpret_cast<uint4*>(base)[k] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    // resident operand: see gru_bwd_ks_kernel
    for (int k = tid; k < KQ * 8; k += GRU_THREADS) {
      const int kl = k >> 3, piece = k & 7;       // local k, 8-unit piece of the 64 units
      const uint4 v = *reinterpret_cast<const uint4*>(
          p.whh + ((long long)dir * K3 + (long long)crank * KQ + kl) * H + k0c + piece * 8);
      const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
      uint8_t* chunk = wtile + (kl >> 6) * WCHUNK + (kl & 7) * 2;
#pragma unroll
      for (int q = 0; q < 8; ++q)
        *reinterpret_cast<unsigned short*>(
            chunk + sw128_offset((uint32_t)(piece * 8 + q), (uint32_t)((kl & 63) >> 3))) = e[q];
    }
  }
  if (tid == 0) {
    for (int i = 0; i < 4; ++i) mbar_init(&full[i], 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);
    mbar_fence_init();
    tma_prefetch_desc(tm);
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();
  unsigned int* ctr = p.barrier + dir * 32;   // one L2 line per direction

  if (warp == GRU_TMA_WARP) {
    if (lane == 0) {
      for (int step = 0; step + 1 < T; ++step) {
        grid_wait(ctr, (unsigned int)nC * (step + 1), p.ablate & 192);   // dgh of this step is complete
        GRU_STAMP(0);
        for (int g = 0; g < ngroups; ++g) {
          mbar_expect_tx(&full[g], (uint32_t)(stride * gc));
          for (int i = 0; i < gc; ++i) {
            const int c = g * gc + i;
            tma_load_2d(ring + c * stride, tm, &full[g], (int)crank * KQ + c * 64,
                        (step & 1) * Bp);
          }
        }
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    switch (NB) {
      case 16: bwd_kt_mma<16>(ring, wtile, recv, stage, full, accfull, ngroups, gc, stride, Bp, P, slice, crank, T); break;
      case 32: bwd_kt_mma<32>(ring, wtile, recv, stage, full, accfull, ngroups, gc, stride, Bp, P, slice, crank, T); break;
      case 48: bwd_kt_mma<48>(ring, wtile, recv, stage, full, accfull, ngroups, gc, stride, Bp, P, slice, crank, T); break;
      default: bwd_kt_mma<64>(ring, wtile, recv, stage, full, accfull, ngroups, gc, stride, Bp, P, slice, crank, T); break;
    }
  } else {
    // phase B: thread = (batch row b, UPT of the CTA's 16 units)
    const int b = tid % Bp, ug = tid / Bp;
    const bool active = ug * UPT < GRU_HC;
    const int u0 = ug * UPT;
    const int ju = j0 + u0;
    float dh_rec[UPT];
    float db_r[UPT], db_z[UPT], db_n[UPT], db_hn[UPT];
#pragma unroll
    for (int jj = 0; jj < UPT; ++jj) {
      dh_rec[jj] = 0.f; db_r[jj] = 0.f; db_z[jj] = 0.f; db_n[jj] = 0.f; db_hn[jj] = 0.f;
    }

    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? (T - 1 - step) : step;
      const int tp = dir == 0 ? t - 1 : t + 1;
      const bool has_prev = dir == 0 ? (t > 0) : (t < T - 1);
      bf16* xb = p.xchg + ((long long)(dir * 2 + (step & 1)) * Bp) * K3;
      const long long m = (long long)t * Bp + b;
      float rr[UPT], zz[UPT], nn[UPT], hn[UPT], dh[UPT], hp[UPT];
      if (active) {
        const float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
        ldu<UPT>(go, rr);
        ldu<UPT>(go + H, zz);
        ldu<UPT>(go + 2 * H, nn);
        ldu<UPT>(go + 3 * H, hn);
        ldu<UPT>(p.dy + m * D + dir * H + ju, dh);
        if (has_prev) {
          ldu<UPT>(p.y + ((long long)tp * Bp + b) * D + dir * H + ju, hp);
        } else {
#pragma unroll
          for (int jj = 0; jj < UPT; ++jj) hp[jj] = 0.f;
        }
      }
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        // the MMA warpgroup staged the three outgoing slices (and the own one in recv[crank])
        if (tid == 0) mbar_expect_tx(recvbar, (uint32_t)((KS - 1) * slice * 4));
        if (lane == 0 && warp >= 1 && warp <= KS - 1) {
          const uint32_t pr = (crank + (uint32_t)warp) % KS;
          bulk_s2peer(mapa_shared(smem_u32(recv + (size_t)crank * slice), pr),
                      stage + (size_t)(warp - 1) * slice, (uint32_t)(slice * 4),
                      mapa_shared(smem_u32(recvbar), pr));
        }
        if (tid == 0) GRU_STAMP(4);
        mbar_wait(recvbar, (step - 1) & 1);
        if (active) {
#pragma unroll
          for (int src = 0; src < KS; ++src) {
            const float* rp = recv + (size_t)src * slice + u0 * P + b;
#pragma unroll
            for (int jj = 0; jj < UPT; ++jj) dh_rec[jj] += rp[jj * P];
          }
        }
      }
      float dr[UPT], dz[UPT], dn[UPT], dnr[UPT];
      if (active) {
#pragma unroll
        for (int jj = 0; jj < UPT; ++jj) {
          const float g = dh[jj] + dh_rec[jj];
          dn[jj] = g * (1.f - zz[jj]) * (1.f - nn[jj] * nn[jj]);
          dz[jj] = g * (hp[jj] - nn[jj]) * zz[jj] * (1.f - zz[jj]);
          dr[jj] = dn[jj] * hn[jj] * rr[jj] * (1.f - rr[jj]);
          dnr[jj] = dn[jj] * rr[jj];
          dh_rec[jj] = g * zz[jj];
          db_r[jj] += dr[jj];
          db_z[jj] += dz[jj];
          db_n[jj] += dn[jj];
          db_hn[jj] += dnr[jj];
        }
        if (step + 1 < T) {
          bf16* x = xb + (long long)b * K3 + ju;
          st_bf16u<UPT>(x, dr);
          st_bf16u<UPT>(x + H, dz);
          st_bf16u<UPT>(x + 2 * H, dnr);
          if (tid == 0) GRU_STAMP(5);
          fence_proxy_async_global();
          if (tid == 0) GRU_STAMP(6);
        }
      }
      if (step + 1 < T) {
        epi_barrier();
        if (tid == 0) {
          GRU_STAMP(7);
          grid_arrive(ctr);
          GRU_STAMP(9);
        }
      }
      if (active) {
        bf16* o = p.dgi + m * (p.ndir * K3) + dir * K3 + ju;
        st_stream_bf16u<UPT>(o, dr);
        st_stream_bf16u<UPT>(o + H, dz);
        st_stream_bf16u<UPT>(o + 2 * H, dn);
        st_stream_bf16u<UPT>(p.dghn + m * D + dir * H + ju, dnr);
      }
      if (tid == 0) GRU_STAMP(10);
    }
    if (active) {
#pragma unroll
      for (int jj = 0; jj < UPT; ++jj) {
        const int bi = dir * K3 + ju + jj;
        atomicAdd(p.dbih + bi, db_r[jj]);
        atomicAdd(p.dbih + bi + H, db_z[jj]);
        atomicAdd(p.dbih + bi + 2 * H, db_n[jj]);
        atomicAdd(p.dbhh + bi, db_r[jj]);
        atomicAdd(p.dbhh + bi + H, db_z[jj]);
        atomicAdd(p.dbhh + bi + 2 * H, db_hn[jj]);
      }
    }
  }

  __syncthreads();
  cluster_sync_all();
}

int make_tmap_bf16_2d(CUtensorMap* map, const void* base, long long rows, long long cols,
                      long long ld, int box_rows);

// chunks are grouped gc per mbarrier pair (gc = largest of 4,3,2,1 dividing nchunks); ring = the
// largest divisor of ngroups (<= GRU_MAX_RING) whose slots fit next to the resident weights and
// the parked recurrent product of `acc_cols` columns
static int gru_ring_slots(int wbytes, int Bp, int nchunks, int acc_cols, int* gc_out,
                          size_t* smem_bytes) {
  int gc = 1;
  for (int g = 4; g >= 1; --g)
    if (nchunks % g == 0) { gc = g; break; }
  const int ngroups = nchunks / gc;
  const int slot = gc * Bp * 128;
  const int fixed = wbytes + 1024 /*align*/ + (2 * GRU_MAX_RING + 2) * 8 + 256 /*scratch*/ + 64 +
                    Bp * (acc_cols + 4) * 4;
  int fit = (227 * 1024 - fixed) / slot;
  if (fit > GRU_MAX_RING) fit = GRU_MAX_RING;
  int ring = -1;
  for (int r = fit; r >= 1; --r)
    if (ngroups % r == 0) { ring = r; break; }
  if (ring < 1) {
    if (gc == 1) return -1;
    // fall back to single-chunk groups
    gc = 1;
    fit = (227 * 1024 - fixed) / (Bp * 128);
    if (fit > GRU_MAX_RING) fit = GRU_MAX_RING;
    for (int r = fit; r >= 1; --r)
      if (nchunks % r == 0) { ring = r; break; }
    if (ring < 1) return -1;
  }
  *gc_out = gc;
  *smem_bytes = (size_t)fixed + (size_t)ring * gc * Bp * 128;
  return ring;
}

static int g_gru_cluster = 4;   // preferred cluster size (developer knob: sb_debug_gru_cluster)
static int g_gru_last_cluster = 0;

static int gru_cluster_size(int nC) {
  int cs = g_gru_cluster;
  while (cs > 1 && (nC % cs) != 0) cs >>= 1;
  return cs < 1 ? 1 : cs;
}

static int gru_launch(const void* kernel, int grid, int cs, size_t smem, void** args,
                      cudaStream_t stream) {
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return SB_ERR_CUDA;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GRU_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  attrs[0].id = cudaLaunchAttributeCooperative;
  attrs[0].val.cooperative = 1;
  attrs[1].id = cudaLaunchAttributeClusterDimension;
  attrs[1].val.clusterDim.x = cs;
  attrs[1].val.clusterDim.y = 1;
  attrs[1].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 2;
  // all CTAs must be co-resident (grid barrier): shrink the cluster until the grid fits
  if (cs > 1 &&
      cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 0) != cudaSuccess)
    cudaGetLastError();
  for (; cs >= 1; cs >>= 1) {
    attrs[1].val.clusterDim.x = cs;
    int nclusters = 0;
    if (cs > 1) {
      if (cudaOccupancyMaxActiveClusters(&nclusters, kernel, &cfg) != cudaSuccess) {
        cudaGetLastError();
        continue;
      }
      if (nclusters * cs < grid) continue;
    }
    if (cudaLaunchKernelExC(&cfg, kernel, args) == cudaSuccess) {
      g_gru_last_cluster = cs;
      return SB_OK;
    }
    cudaGetLastError();
  }
  return SB_ERR_CUDA;
}

static unsigned long long* g_gru_dbg = nullptr;
static int g_gru_ablate = 0;
static int g_gru_ksplit = 1;   // developer knob: 0 disables the K-split backward kernel

// Which K-split flavour: the transposed-accumulator kernels (gru_*_kt_kernel) spend tensor work
// in proportion to the batch (N = batch) instead of a whole m64 block of batch rows.
// An H100 holds 30 clusters of 4 one-CTA-per-SM blocks (120 CTAs), so at H = 1024 the two
// directions (128 CTAs) never fit as one K-split launch: the forward runs gru_fwd_kernel there
// and the backward gru_bwd_ks_kernel once per direction.  Measured on an H100 80GB HBM3 (400 W
// power limit), recurrence kernel alone, us per step at T = 247, ONE direction of H = 1024
// (kt | ks): forward 4.12 | 4.17 at 8 rows, 4.59 | 4.34 at 16, 7.73 | 5.46 at 32, 14.68 | 8.38 at
// 64; backward 3.17 | 4.28 at 8, 4.08 | 4.37 at 16, 6.09 | 5.12 at 32, 8.15 | 7.94 at 64.  Both
// directions at 64 rows: gru_fwd_kernel 11.7; backward 23.4 with gru_bwd_kernel, 15.5 with the
// two one-direction gru_bwd_ks_kernel launches.
// Developer knob (sb_debug_gru_flags): 16 forces them, 8 disables them.
static bool gru_use_kt(int Bp, bool backward) {
  if (g_gru_ablate & 8) return false;
  if (g_gru_ablate & 16) return true;
  return !backward && Bp <= 16;
}

// cooperative launch with EXACTLY the given cluster size; fails if the grid is not co-resident
static int gru_launch_exact(const void* kernel, int grid, int cs, size_t smem, void** args,
                            cudaStream_t stream) {
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess) {
    cudaGetLastError();
    return SB_ERR_CUDA;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GRU_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  // Clustered launches are NOT flagged cooperative: co-residency of the whole grid is established
  // by the occupancy query below (1 CTA per SM, grid <= resident capacity), every spin-wait in
  // the kernels is bounded, and Nsight Compute cannot replay cooperative+cluster launches.
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeClusterDimension;
  attrs[0].val.clusterDim.x = cs;
  attrs[0].val.clusterDim.y = 1;
  attrs[0].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  int nclusters = 0;
  if (cudaOccupancyMaxActiveClusters(&nclusters, kernel, &cfg) != cudaSuccess ||
      nclusters * cs < grid) {
    cudaGetLastError();
    return SB_ERR_UNSUPPORTED;
  }
  if (cudaLaunchKernelExC(&cfg, kernel, args) != cudaSuccess) {
    cudaGetLastError();
    return SB_ERR_CUDA;
  }
  g_gru_last_cluster = cs;
  return SB_OK;
}

}  // namespace sb

using namespace sb;

// developer hooks (not part of the drop-in surface)
extern "C" int sb_debug_gru_timeline(void* dev_buffer) {
  sb::g_gru_dbg = reinterpret_cast<unsigned long long*>(dev_buffer);
  return SB_OK;
}
// developer knobs: 1 / 2: gru_fwd_kernel and the gru_*_ks_kernel without the proxy fence / the
// off-path stores (timing only: results become wrong); 8 / 16: never / always use the
// transposed-accumulator K-split kernels (default: by batch size, see gru_use_kt); 32: disable
// the K-split forward kernels;
// 64 / 128: polling mode of the grid barrier in the K-split kernels (see grid_wait)
extern "C" int sb_debug_gru_flags(int flags) {
  sb::g_gru_ablate = flags;
  return SB_OK;
}
extern "C" int sb_debug_gru_ksplit(int enable) {
  sb::g_gru_ksplit = enable ? 1 : 0;
  return SB_OK;
}
extern "C" int sb_debug_gru_cluster(int cluster_size) {
  // cluster_size 0 queries: returns the cluster size the last GRU launch actually used
  if (cluster_size == 0) return sb::g_gru_last_cluster;
  if (cluster_size != 1 && cluster_size != 2 && cluster_size != 4 && cluster_size != 8)
    return -1;
  sb::g_gru_cluster = cluster_size;
  return sb::g_gru_last_cluster;
}

static int gru_check(int T, int Bp, int H, int ndir) {
  if (T <= 0 || Bp <= 0 || H <= 0 || (ndir != 1 && ndir != 2)) return SB_ERR_INVALID;
  if (H % GRU_HC != 0 || Bp % 8 != 0 || Bp > 128) return SB_ERR_UNSUPPORTED;
  if (ndir * (H / GRU_HC) > sb::device_sm_count()) return SB_ERR_UNSUPPORTED;
  return SB_OK;
}

// workspace of one recurrence launch: [0,1024) the per-direction grid-barrier words, then the
// exchange buffers of the backward kernels
static size_t gru_ws_counters_bytes(int ndir) {
  (void)ndir;
  return 1024;
}

extern "C" int sb_gru_fwd_workspace_size(int Bp, int H, int ndir, size_t* bytes) {
  if (!bytes || Bp <= 0 || H <= 0 || (ndir != 1 && ndir != 2)) return SB_ERR_INVALID;
  (void)Bp;
  *bytes = gru_ws_counters_bytes(ndir);      // the forward kernels exchange h_t through xn itself
  return SB_OK;
}

extern "C" int sb_gru_fwd(const float* gi, const void* whh_bf16, const float* bhh, float* y,
                          void* xn_bf16, float* gates, void* workspace, size_t workspace_bytes,
                          int T, int Bp, int H, int ndir, void* stream_) {
  int rc = gru_check(T, Bp, H, ndir);
  if (rc != SB_OK) return rc;
  if (!gi || !whh_bf16 || !bhh || !y || !xn_bf16 || !workspace) return SB_ERR_INVALID;
  size_t need = 0;
  sb_gru_fwd_workspace_size(Bp, H, ndir, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  if ((reinterpret_cast<uintptr_t>(workspace) & 1023) != 0) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int nchunks = (H + 63) / 64;
  const int nC = H / GRU_HC;
  if (cudaMemsetAsync(workspace, 0, need, stream) != cudaSuccess) return SB_ERR_CUDA;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  unsigned int* barrier = reinterpret_cast<unsigned int*>(ws);
  int gc = 1;
  size_t smem = 0;
  const int ring =
      gru_ring_slots(std::max(nchunks * 48 * 128, 16384 - Bp * 128), Bp, nchunks, 48, &gc, &smem);
  if (ring < 0) return SB_ERR_UNSUPPORTED;

  // ---- preferred: K-split over 4-CTA clusters (H % 256 == 0, batch rows <= 64) ----
  if (!(g_gru_ablate & 32) && H % 256 == 0 && nC % KS == 0 && Bp <= 64) {
    const int nq = H / KS / 64;
    const size_t ks_smem = (size_t)nq * Bp * 128 + (size_t)nq * 192 * 128 +
                           (size_t)2 * KS * Bp * 48 * 4 + 1024 + 512;
    if (ks_smem <= 227 * 1024) {
      GruFwdParams q;
      q.gi = gi; q.whh = reinterpret_cast<const bf16*>(whh_bf16); q.bhh = bhh; q.y = y;
      q.xn = reinterpret_cast<bf16*>(xn_bf16); q.xnT = nullptr; q.gates = gates;
      q.barrier = barrier; q.T = T; q.Bp = Bp; q.H = H; q.ndir = ndir;
      q.dbg = g_gru_dbg; q.ablate = g_gru_ablate & 195; q.ring = nq; q.gc = 1;
      CUtensorMap tq[2];
      for (int d = 0; d < 2; ++d) {
        const int dd = d < ndir ? d : 0;
        rc = make_tmap_bf16_2d(&tq[d], q.xn + (size_t)dd * H, (long long)T * Bp, H,
                               (long long)ndir * H, Bp);
        if (rc != SB_OK) return rc;
      }
      void* kargs[] = {(void*)&tq[0], (void*)&tq[1], (void*)&q};
      const size_t kt_smem = (size_t)nq * Bp * 128 + (size_t)nq * 192 * 128 +
                             (size_t)(2 * KS - 1) * 48 * (Bp + 4) * 4 + 1024 + 512;
      if (gru_use_kt(Bp, false) && kt_smem <= 227 * 1024) {
        const void* kt = Bp > 32   ? (const void*)gru_fwd_kt_kernel<4>
                         : Bp > 16 ? (const void*)gru_fwd_kt_kernel<2>
                                   : (const void*)gru_fwd_kt_kernel<1>;
        rc = gru_launch_exact(kt, ndir * nC, KS, kt_smem, kargs, stream);
        if (rc == SB_OK) return SB_OK;
      }
      rc = gru_launch_exact((const void*)gru_fwd_ks_kernel, ndir * nC, KS, ks_smem, kargs, stream);
      if (rc == SB_OK) return SB_OK;
    }
  }

  // ---- every other shape: each CTA gathers all of h_{t-1} (tensor-map TMA, cluster multicast) ----
  GruFwdParams p;
  p.gi = gi; p.whh = reinterpret_cast<const bf16*>(whh_bf16); p.bhh = bhh; p.y = y;
  p.xn = reinterpret_cast<bf16*>(xn_bf16); p.xnT = nullptr;
  p.gates = gates; p.barrier = barrier; p.T = T; p.Bp = Bp; p.H = H; p.ndir = ndir;
  p.dbg = g_gru_dbg;
  p.ablate = g_gru_ablate & 31;
  p.ring = ring; p.gc = gc;
  CUtensorMap tm[2];
  for (int d = 0; d < 2; ++d) {
    const int dd = d < ndir ? d : 0;
    rc = make_tmap_bf16_2d(&tm[d], p.xn + (size_t)dd * H, (long long)T * Bp, H,
                           (long long)ndir * H, Bp);
    if (rc != SB_OK) return rc;
  }
  void* args[] = {(void*)&tm[0], (void*)&tm[1], (void*)&p};
  return gru_launch((const void*)gru_fwd_kernel, ndir * nC, gru_cluster_size(nC), smem, args,
                    stream);
}

extern "C" int sb_gru_bwd_workspace_size(int Bp, int H, int ndir, size_t* bytes) {
  if (!bytes || Bp <= 0 || H <= 0 || (ndir != 1 && ndir != 2)) return SB_ERR_INVALID;
  // counters + the double-buffered exchange of dgh_t (Bp x 3H bf16 per direction and parity; the
  // tile-major form of the K-split kernel rounds 3H up to whole 64-column chunks)
  const size_t k3p = (size_t)((3 * H + 63) / 64) * 64;
  *bytes = gru_ws_counters_bytes(ndir) + (size_t)ndir * 2 * Bp * k3p * sizeof(bf16) + 1024;
  return SB_OK;
}

extern "C" int sb_gru_bwd(const float* dy, const float* y, const float* gates,
                          const void* whh_bf16, void* dgi_bf16, void* dghn_bf16, float* dbih,
                          float* dbhh, void* workspace, size_t workspace_bytes, int T, int Bp,
                          int H, int ndir, void* stream_) {
  int rc = gru_check(T, Bp, H, ndir);
  if (rc != SB_OK) return rc;
  if (!dy || !y || !gates || !whh_bf16 || !dgi_bf16 || !dghn_bf16 || !dbih || !dbhh ||
      !workspace)
    return SB_ERR_INVALID;
  size_t need = 0;
  sb_gru_bwd_workspace_size(Bp, H, ndir, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  if ((reinterpret_cast<uintptr_t>(workspace) & 1023) != 0) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  GruBwdParams p;
  p.dy = dy; p.y = y; p.gates = gates; p.whh = reinterpret_cast<const bf16*>(whh_bf16);
  p.dgi = reinterpret_cast<bf16*>(dgi_bf16);
  p.dghn = reinterpret_cast<bf16*>(dghn_bf16);
  p.barrier = reinterpret_cast<unsigned int*>(ws);
  p.xchg = reinterpret_cast<bf16*>(ws + gru_ws_counters_bytes(ndir));
  p.dbih = dbih; p.dbhh = dbhh; p.T = T; p.Bp = Bp; p.H = H; p.ndir = ndir;
  p.dbg = g_gru_dbg;
  p.dir0 = 0;
  p.ablate = g_gru_ablate & 195;
  const int K3 = 3 * H;
  const int nchunks = (K3 + 63) / 64;
  size_t smem = 0;
  const int nC_ = H / GRU_HC;
  // counters and barrier words start at zero; the exchange tiles too (columns past 3H of a
  // partial chunk are never written and must read as zero)
  if (cudaMemsetAsync(workspace, 0, need, stream) != cudaSuccess) return SB_ERR_CUDA;
  // ---- preferred: K-split over 4-CTA clusters ----
  if (g_gru_ksplit && H % 256 == 0 && nC_ % KS == 0 && (K3 / KS / 64) <= 16) {
    const int nq = K3 / KS / 64;
    const size_t ks_smem = (size_t)nq * Bp * 128 + (size_t)nq * 64 * 128 +
                           (size_t)2 * KS * Bp * 64 + 1024 + 256;
    if (ks_smem <= 227 * 1024) {
      CUtensorMap tq[2];
      for (int d = 0; d < 2; ++d) {
        const int dd = d < ndir ? d : 0;
        rc = make_tmap_bf16_2d(&tq[d], p.xchg + (size_t)dd * 2 * Bp * K3, 2LL * Bp, K3, K3, Bp);
        if (rc != SB_OK) return rc;
      }
      p.ring = nq; p.gc = 1;
      void* kargs[] = {(void*)&tq[0], (void*)&tq[1], (void*)&p};
      const size_t kt_smem = (size_t)nq * Bp * 128 + (size_t)nq * 64 * 128 +
                             (size_t)(2 * KS - 1) * GRU_HC * (Bp + 4) * 4 + 1024 + 256;
      if (gru_use_kt(Bp, true) && Bp <= 64 && kt_smem <= 227 * 1024) {
        const void* kt = Bp > 32   ? (const void*)gru_bwd_kt_kernel<4>
                         : Bp > 16 ? (const void*)gru_bwd_kt_kernel<2>
                                   : (const void*)gru_bwd_kt_kernel<1>;
        rc = gru_launch_exact(kt, ndir * nC_, KS, kt_smem, kargs, stream);
        if (rc == SB_OK) return SB_OK;
      }
      rc = gru_launch_exact((const void*)gru_bwd_ks_kernel, ndir * nC_, KS, ks_smem, kargs, stream);
      if (rc == SB_OK) return SB_OK;
      // Both directions do not fit as 4-CTA clusters (an H100 holds 30 of them, 120 CTAs, against
      // 128 at H = 1024): run the directions one after the other, each with its own barrier
      // counter.  Still faster than the plain kernel, whose every CTA gathers all of dgh_t.
      if (rc == SB_ERR_UNSUPPORTED && ndir == 2) {
        rc = gru_launch_exact((const void*)gru_bwd_ks_kernel, nC_, KS, ks_smem, kargs, stream);
        if (rc == SB_OK) {
          p.dir0 = 1;   // kernel parameters are copied at launch
          return gru_launch_exact((const void*)gru_bwd_ks_kernel, nC_, KS, ks_smem, kargs, stream);
        }
      }
    }
  }
  p.ring = gru_ring_slots(std::max(nchunks * 16 * 128, 16384 - Bp * 128), Bp, nchunks, 16, &p.gc,
                          &smem);
  if (p.ring < 0) return SB_ERR_UNSUPPORTED;
  // per direction: the two parity buffers stacked as [2*Bp rows][3H cols]
  CUtensorMap tm[2];
  for (int d = 0; d < 2; ++d) {
    const int dd = d < ndir ? d : 0;
    rc = make_tmap_bf16_2d(&tm[d], p.xchg + (size_t)dd * 2 * Bp * K3, 2LL * Bp, K3, K3, Bp);
    if (rc != SB_OK) return rc;
  }
  void* args[] = {(void*)&tm[0], (void*)&tm[1], (void*)&p};
  const int nC = H / GRU_HC;
  return gru_launch((const void*)gru_bwd_kernel, ndir * nC, gru_cluster_size(nC), smem, args,
                    stream);
}
