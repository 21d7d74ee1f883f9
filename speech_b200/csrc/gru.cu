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
  float* gates;        // [T*Bp][ndir][4][H] saved r,z,n,hn for backward ; may be null
  unsigned int* barrier;  // [ndir] zero-initialised counters
  unsigned long long* dbg;  // optional timeline (CTA 0): [step][16] globaltimer stamps, or null
  int T, Bp, H, ndir, ring, gc;   // ring: slots (groups of gc chunks) in shared memory
  int ablate;          // developer knobs: see sb_debug_gru_flags
  int rg, wr;          // wide kernels: resident weight groups, weight-ring slots
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
  float* rs;           // L2 reduce-scatter staging [ndir][H/64][2][4][4][Bp][16] (gru_bwd_ks_kernel<true>)
  unsigned int* rsctr; // its counters, [ndir][H/64] x 32 words (one L2 line each)
  int rg, wr;          // gru_bwd_wide_kernel: resident weight groups, weight-ring slots
  bf16* whhT;          // gru_bwd_wide_kernel: [ndir][H][3H] W_hh transposed (each CTA its rows)
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

// ---- vectors of UPT = 1, 2, 4 or 8 consecutive hidden units of one thread ----------------------
// One-touch data (gi, saved gates, dy, fp32 state, GEMM operands written for later kernels) uses
// the streaming cache policy (.cs) so that it does not evict the latency-critical bf16 exchange
// buffers, which every CTA re-reads from L2 each step.
template <int UPT>
SB_DEVINL void ld_stream(const float* p, float (&v)[UPT]) {
  if constexpr (UPT >= 4) {
#pragma unroll
    for (int i = 0; i < UPT; i += 4) {
      const float4 a = __ldcs(reinterpret_cast<const float4*>(p + i));
      v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
    }
  } else if constexpr (UPT == 2) {
    const float2 a = __ldcs(reinterpret_cast<const float2*>(p));
    v[0] = a.x; v[1] = a.y;
  } else {
    v[0] = __ldcs(p);
  }
}
template <int UPT>
SB_DEVINL void st_stream(float* p, const float (&v)[UPT]) {
  if constexpr (UPT >= 4) {
#pragma unroll
    for (int i = 0; i < UPT; i += 4)
      __stcs(reinterpret_cast<float4*>(p + i), make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]));
  } else if constexpr (UPT == 2) {
    __stcs(reinterpret_cast<float2*>(p), make_float2(v[0], v[1]));
  } else {
    __stcs(p, v[0]);
  }
}
// bf16 vectors are rounded once (to_bf16) and kept packed in pairs until stored: the backward
// stores each of its gradients twice, once on each side of the grid barrier, and packed halves
// the registers they hold across it.  UPT = 1 uses the low half of w[0].
template <int UPT>
struct Bf16Vec {
  uint32_t w[(UPT + 1) / 2];
};
template <int UPT>
SB_DEVINL Bf16Vec<UPT> to_bf16(const float (&v)[UPT]) {
  Bf16Vec<UPT> b;
  if constexpr (UPT == 1) {
    b.w[0] = __bfloat16_as_ushort(__float2bfloat16_rn(v[0]));
  } else {
#pragma unroll
    for (int i = 0; i < UPT / 2; ++i) b.w[i] = pack_bf16x2(v[2 * i], v[2 * i + 1]);
  }
  return b;
}
// the default policy (the exchange rows other CTAs read next) and the streaming one
template <int UPT>
SB_DEVINL void st_bf16(bf16* p, const Bf16Vec<UPT>& b) {
  if constexpr (UPT == 8) *reinterpret_cast<uint4*>(p) = make_uint4(b.w[0], b.w[1], b.w[2], b.w[3]);
  else if constexpr (UPT == 4) *reinterpret_cast<uint2*>(p) = make_uint2(b.w[0], b.w[1]);
  else if constexpr (UPT == 2) *reinterpret_cast<uint32_t*>(p) = b.w[0];
  else *reinterpret_cast<unsigned short*>(p) = (unsigned short)b.w[0];
}
template <int UPT>
SB_DEVINL void st_stream_bf16(bf16* p, const Bf16Vec<UPT>& b) {
  if constexpr (UPT == 8) {
    __stcs(reinterpret_cast<uint4*>(p), make_uint4(b.w[0], b.w[1], b.w[2], b.w[3]));
  } else if constexpr (UPT == 4) {
    __stcs(reinterpret_cast<uint2*>(p), make_uint2(b.w[0], b.w[1]));
  } else if constexpr (UPT == 2) {
    __stcs(reinterpret_cast<unsigned int*>(p), b.w[0]);
  } else {
    asm volatile("st.global.cs.u16 [%0], %1;" ::"l"(p), "h"((unsigned short)b.w[0]) : "memory");
  }
}

// ---- the GRU cell, shared by every recurrence kernel ------------------------------------------
// Four per-gate values of UPT units: the saved activations r, z, n, hn (= W_hn h_{t-1} + b_hn),
// their gradients dr, dz, dn, dn*r (the pre-activation gradients of the r, z and n gates, and of
// hn), or the bias partial sums of those.
template <int UPT>
struct GruGates {
  float r[UPT], z[UPT], n[UPT], hn[UPT];
};
template <int UPT>
struct GruGatesBf16 {
  Bf16Vec<UPT> r, z, n, hn;
};

// Forward step of one batch row: gi = the input projections (b_ih included), acc = the finished
// recurrent product W_hh h_{t-1}, bias = b_hh; h holds h_{t-1} and receives h_t.
template <int UPT>
SB_DEVINL void gru_cell_fwd(const float (&gi)[3][UPT], const float (&acc)[3][UPT],
                            const float (&bias)[3][UPT], float (&h)[UPT], GruGates<UPT>& g) {
#pragma unroll
  for (int jj = 0; jj < UPT; ++jj) {
    g.r[jj] = fast_sigmoid(gi[0][jj] + acc[0][jj] + bias[0][jj]);
    g.z[jj] = fast_sigmoid(gi[1][jj] + acc[1][jj] + bias[1][jj]);
    g.hn[jj] = acc[2][jj] + bias[2][jj];
    g.n[jj] = fast_tanh(gi[2][jj] + g.r[jj] * g.hn[jj]);
    h[jj] = (1.f - g.z[jj]) * g.n[jj] + g.z[jj] * h[jj];
  }
}

// Backward step of one batch row: dh = dL/dh_t from the layer output, dh_rec = its recurrent part
// (on return: the direct path h_{t-1} -> h_t; the W_hh path is added next step), s = the saved
// gates, hp = h_{t-1}.  Adds the pre-activation gradients to the bias sums db and returns them in
// bf16, the form every kernel stores.
template <int UPT>
SB_DEVINL GruGatesBf16<UPT> gru_cell_bwd(const float (&dh)[UPT], float (&dh_rec)[UPT],
                                         const GruGates<UPT>& s, const float (&hp)[UPT],
                                         GruGates<UPT>& db) {
  GruGates<UPT> d;
#pragma unroll
  for (int jj = 0; jj < UPT; ++jj) {
    const float g = dh[jj] + dh_rec[jj];
    d.n[jj] = g * (1.f - s.z[jj]) * (1.f - s.n[jj] * s.n[jj]);
    d.z[jj] = g * (hp[jj] - s.n[jj]) * s.z[jj] * (1.f - s.z[jj]);
    d.r[jj] = d.n[jj] * s.hn[jj] * s.r[jj] * (1.f - s.r[jj]);
    d.hn[jj] = d.n[jj] * s.r[jj];
    dh_rec[jj] = g * s.z[jj];
    db.r[jj] += d.r[jj];
    db.z[jj] += d.z[jj];
    db.n[jj] += d.n[jj];
    db.hn[jj] += d.hn[jj];
  }
  return {to_bf16(d.r), to_bf16(d.z), to_bf16(d.n), to_bf16(d.hn)};
}

// ---- per-step epilogue pieces -----------------------------------------------------------------
// This step's input projections of UPT units from ju of batch row `row`: they do not depend on
// the recurrence, so every kernel fetches them before it waits for the product.
template <int UPT>
SB_DEVINL void gru_load_gi(const GruFwdParams& p, int t, int row, int dir, int ju,
                           float (&gi)[3][UPT]) {
  const int H = p.H;
  const float* g = p.gi + ((long long)t * p.Bp + row) * (p.ndir * 3 * H) + dir * 3 * H + ju;
#pragma unroll
  for (int gg = 0; gg < 3; ++gg) ld_stream<UPT>(g + gg * H, gi[gg]);
}

// b_hh of the thread's units from shared memory (`pitch` floats per gate)
template <int UPT>
SB_DEVINL void gru_load_bias(const float* src, int pitch, float (&bias)[3][UPT]) {
#pragma unroll
  for (int g = 0; g < 3; ++g)
#pragma unroll
    for (int jj = 0; jj < UPT; ++jj) bias[g][jj] = src[g * pitch + jj];
}

// The saved activations of backward step t (forward time index): gates, dy and h_{t-1} (zero where
// the direction's sequence starts).  Independent of the recurrence: fetched first.
template <int UPT>
SB_DEVINL void gru_load_saved(const GruBwdParams& p, int t, int row, int dir, int ju,
                              GruGates<UPT>& s, float (&dh)[UPT], float (&hp)[UPT]) {
  const int H = p.H, Bp = p.Bp, D = p.ndir * H;
  const long long m = (long long)t * Bp + row;
  const float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
  ld_stream<UPT>(go, s.r);
  ld_stream<UPT>(go + H, s.z);
  ld_stream<UPT>(go + 2 * H, s.n);
  ld_stream<UPT>(go + 3 * H, s.hn);
  ld_stream<UPT>(p.dy + m * D + dir * H + ju, dh);
  const int tp = dir == 0 ? t - 1 : t + 1;
  if (dir == 0 ? (t > 0) : (t < p.T - 1)) {
    ld_stream<UPT>(p.y + ((long long)tp * Bp + row) * D + dir * H + ju, hp);
  } else {
#pragma unroll
    for (int jj = 0; jj < UPT; ++jj) hp[jj] = 0.f;
  }
}

// Critical path of the backward: the exchange row [dr | dz | dn*r] every CTA gathers next step
template <int UPT>
SB_DEVINL void gru_store_xchg(const GruBwdParams& p, int step, int row, int dir, int ju,
                              const GruGatesBf16<UPT>& d) {
  const int H = p.H;
  bf16* x = p.xchg + ((long long)(dir * 2 + (step & 1)) * p.Bp + row) * (3 * H) + ju;
  st_bf16<UPT>(x, d.r);
  st_bf16<UPT>(x + H, d.z);
  st_bf16<UPT>(x + 2 * H, d.hn);
}

// After the CTA's bf16 rows of the step are stored (wrote: by this thread): order them before the
// other CTAs' TMA reads (generic -> async proxy), then one release arrive per CTA on the
// direction's grid barrier once every epilogue thread is done.  skew_probe: the K-split forward
// kernels record the arrive of step 20 per CTA (tools/gru_timeline.py).
// Developer knob (sb_debug_gru_flags) 1 drops the fence: timing only, results become wrong.
template <class Params>
SB_DEVINL void gru_publish(const Params& p, unsigned int* ctr, int step, bool wrote,
                           bool skew_probe) {
  const bool lead = threadIdx.x == 0;
  if (lead) GRU_STAMP(5);
  if (wrote && !(p.ablate & 1)) fence_proxy_async_global();
  if (lead) GRU_STAMP(6);
  epi_barrier();
  if (lead) {
    GRU_STAMP(7);
    if (skew_probe && p.dbg && step == 20) p.dbg[1024 + blockIdx.x] = gtime();
    grid_arrive(ctr);   // release: cumulative over the CTA's writes ordered by bar.sync
    GRU_STAMP(9);
  }
}

// Off the critical path: the forward's fp32 h_t and saved gates, the backward's operands of the
// dX / dW GEMMs.  Developer knob 2 skips them (timing only).
template <int UPT>
SB_DEVINL void gru_store_fwd(const GruFwdParams& p, long long m, int dir, int ju,
                             const float (&h)[UPT], const GruGates<UPT>& g) {
  if (p.ablate & 2) return;
  const int H = p.H;
  st_stream<UPT>(p.y + m * (p.ndir * H) + dir * H + ju, h);
  if (p.gates) {
    float* go = p.gates + ((m * p.ndir + dir) * 4) * H + ju;
    st_stream<UPT>(go, g.r);
    st_stream<UPT>(go + H, g.z);
    st_stream<UPT>(go + 2 * H, g.n);
    st_stream<UPT>(go + 3 * H, g.hn);
  }
}
template <int UPT>
SB_DEVINL void gru_store_bwd(const GruBwdParams& p, long long m, int dir, int ju,
                             const GruGatesBf16<UPT>& d) {
  if (p.ablate & 2) return;
  const int H = p.H, K3 = 3 * H;
  bf16* o = p.dgi + m * (p.ndir * K3) + dir * K3 + ju;
  st_stream_bf16<UPT>(o, d.r);
  st_stream_bf16<UPT>(o + H, d.z);
  st_stream_bf16<UPT>(o + 2 * H, d.n);
  st_stream_bf16<UPT>(p.dghn + m * (p.ndir * H) + dir * H + ju, d.hn);
}

// Resumed forward (sb_gru_fwd_h0, one direction): step 0 publishes h_{-1}, which the caller put in
// frame 0 of y and xn, instead of computing a state, and step s >= 1 reads gi frame s - 1.
template <int UPT>
SB_DEVINL void gru_load_h0(const GruFwdParams& p, int row, int ju, float (&h)[UPT]) {
  ld_stream<UPT>(p.y + (long long)row * p.H + ju, h);
}

// ---- prologue pieces --------------------------------------------------------------------------
SB_DEVINL void smem_zero(uint8_t* base, int bytes) {
  for (int k = threadIdx.x; k < bytes / 16; k += GRU_THREADS)
    reinterpret_cast<uint4*>(base)[k] = make_uint4(0, 0, 0, 0);
}

// Forward weight layout: shared-memory row r <- row row_of(r) of one direction's W_hh ([3H][H],
// the row of gate g and unit u is g * H + u), columns k0 .. k0 + ncols, into K-major SWIZZLE_128B
// chunks of 64 columns (wchunk bytes each).  Pieces past ncols keep the zeroed contents.
template <class RowOf>
SB_DEVINL void stage_w_rows(uint8_t* wtile, int wchunk, const bf16* w, int H, int nrows, int k0,
                            int ncols, RowOf row_of) {
  const int pieces_per_row = (ncols + 63) / 64 * 8;
  for (int k = threadIdx.x; k < nrows * pieces_per_row; k += GRU_THREADS) {
    const int r = k / pieces_per_row, pc = k % pieces_per_row;
    if (pc * 8 < ncols) {
      const uint4 v =
          *reinterpret_cast<const uint4*>(w + (long long)row_of(r) * H + k0 + pc * 8);
      *reinterpret_cast<uint4*>(wtile + (pc >> 3) * wchunk + sw128_offset(r, pc & 7)) = v;
    }
  }
}

// Backward weight layout: rows = the NU units u0.. of one direction's W_hh^T, K = rows k0 .. k0 + nk
// of W_hh.  W_hh is read as stored (2 * NU contiguous bytes per k) and transposed on the way into
// K-major SWIZZLE_128B chunks of NU rows x 64.
template <int NU>
SB_DEVINL void stage_w_cols(uint8_t* wtile, const bf16* w, int H, int k0, int nk, int u0) {
  constexpr int PIECES = NU / 8;
  for (int k = threadIdx.x; k < nk * PIECES; k += GRU_THREADS) {
    const int kl = k / PIECES, piece = k % PIECES;
    const uint4 v = *reinterpret_cast<const uint4*>(w + (long long)(k0 + kl) * H + u0 + piece * 8);
    const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
    uint8_t* chunk = wtile + (kl >> 6) * (NU * 128) + (kl & 7) * 2;
#pragma unroll
    for (int q = 0; q < 8; ++q)
      *reinterpret_cast<unsigned short*>(
          chunk + sw128_offset((uint32_t)(piece * 8 + q), (uint32_t)((kl & 63) >> 3))) = e[q];
  }
}

// Thread 0 initialises the kernel's mbarriers (init) and prefetches the tensor-map descriptors
// (tw may be null); then the CTA syncs, and with `cluster` the cluster too, so that no peer
// multicasts into or signals a barrier before it is initialised.
template <class Init>
SB_DEVINL void gru_init_barriers(const CUtensorMap* tm, const CUtensorMap* tw, bool cluster,
                                 Init init) {
  if (threadIdx.x == 0) {
    init();
    mbar_fence_init();
    tma_prefetch_desc(tm);
    if (tw) tma_prefetch_desc(tw);
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (cluster) cluster_sync_all();
}
// the full / empty pairs of a gather ring whose slots every CTA of the cluster releases
SB_DEVINL void init_ring_bars(uint64_t* full, uint64_t* empty, uint32_t csize) {
  for (int i = 0; i < GRU_MAX_RING; ++i) {
    mbar_init(&full[i], 1);
    mbar_init(&empty[i], csize);
  }
}

// =============================================================================================
// forward
// =============================================================================================
template <bool H0>
SB_DEVINL void gru_fwd_body(const CUtensorMap& tm_d0, const CUtensorMap& tm_d1,
                            const GruFwdParams& p) {
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
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const uint32_t crank = cluster_rank(), csize = cluster_size();

  // ---- one-time setup: zero ring + weight region, stage the 48 weight rows, barriers ----
  smem_zero(s.ring, ring_bytes + wbytes);
  __syncthreads();
  stage_w_rows(s.wtile, WCHUNK, p.whh + (long long)dir * 3 * H * H, H, 48, 0, H,
               [=](int r) { return (r / GRU_HC) * H + j0 + r % GRU_HC; });
  if (tid < 48) s.scratch[tid] = p.bhh[dir * 3 * H + (tid / GRU_HC) * H + j0 + tid % GRU_HC];
  gru_init_barriers(tm, nullptr, true, [=] {
    init_ring_bars(s.full, s.empty, csize);
    mbar_init(s.accfull, 128);
  });
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
    // accbuf is made opaque to the compiler, which otherwise recomputes it from the carve before
    // each store of the parked product, on the critical path of every step.  Measured with and
    // without this line, same source otherwise (H100 80GB HBM3 at 700 W, both directions, us
    // per step): H = 1024 at 64 rows 11.2 with, 11.6 without; at 8 rows 3.3 with, 3.7 without;
    // H = 384 at 32 rows 4.0 with, 4.4 without.
    GruSmem sm = s;
    asm volatile("" : "+l"(sm.accbuf));
    for (int step = 1; step < T; ++step) {
      if (Bp > 64) mma_consume<48, true>(sm, nchunks, WCHUNK, Bp, p.ring, p.gc, step - 1, csize);
      else mma_consume<48, false>(sm, nchunks, WCHUNK, Bp, p.ring, p.gc, step - 1, csize);
      if (tid == GRU_MMA_WARP * 32) GRU_STAMP(2);
    }
  } else {
    // ===================== epilogue: thread = (batch row, half of the 16 units) ==============
    const int row = (warp & 3) * 32 + lane;      // batch row
    const int uh = warp >> 2;                    // which 8 of the CTA's 16 units
    const int ju = j0 + uh * GRU_UPT;
    float hprev[GRU_UPT] = {};
    float bias[3][GRU_UPT];
    gru_load_bias(s.scratch + uh * GRU_UPT, GRU_HC, bias);
    const bool active = row < Bp;
    int step0 = 0;
    if constexpr (H0) {
      if (active) gru_load_h0(p, row, ju, hprev);
      gru_publish(p, ctr, 0, false, false);
      step0 = 1;
    }
    for (int step = step0; step < T; ++step) {
      const int t = dir == 0 ? step : (T - 1 - step);
      float gi[3][GRU_UPT];
      if (active) gru_load_gi(p, t - step0, row, dir, ju, gi);
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
      GruGates<GRU_UPT> gt;
      if (active) {
        gru_cell_fwd(gi, acc, bias, hprev, gt);
        // critical path: only the bf16 h_t that the other CTAs gather next step
        st_bf16(p.xn + m * D + dir * H + ju, to_bf16(hprev));
      }
      gru_publish(p, ctr, step, active, false);
      if (active) gru_store_fwd(p, m, dir, ju, hprev, gt);
      if (tid == 0) GRU_STAMP(10);
    }
  }

  __syncthreads();
  cluster_sync_all();   // no CTA leaves while peers may still signal its barriers
}

__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_kernel(const __grid_constant__ CUtensorMap tm_d0, const __grid_constant__ CUtensorMap tm_d1,
               const GruFwdParams p) {
  gru_fwd_body<false>(tm_d0, tm_d1, p);
}
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_h0_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruFwdParams p) {
  gru_fwd_body<true>(tm_d0, tm_d1, p);
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
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const uint32_t crank = cluster_rank(), csize = cluster_size();

  smem_zero(s.ring, ring_bytes + wbytes);
  __syncthreads();
  // resident operand: rows = the 16 hidden units j0..j0+15 of W_hh^T, K = 3H
  stage_w_cols<GRU_HC>(s.wtile, p.whh + (long long)dir * K3 * H, H, 0, K3, j0);
  gru_init_barriers(tm, nullptr, true, [=] {
    init_ring_bars(s.full, s.empty, csize);
    mbar_init(s.accfull, 128);
  });
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
    float dh_rec[GRU_UPT] = {};   // dL/dh_t arriving through the recurrence (own units)
    GruGates<GRU_UPT> db = {};

    for (int step = 0; step < T; ++step) {
      // forward order of dir 0 is t=0..T-1, so its backward order is T-1..0; dir 1 mirrored
      const int t = dir == 0 ? (T - 1 - step) : step;
      const long long m = (long long)t * Bp + row;
      GruGates<GRU_UPT> sv;
      float dh[GRU_UPT], hp[GRU_UPT];
      if (active) gru_load_saved(p, t, row, dir, ju, sv, dh, hp);
      // ---- recurrent part of dL/dh_t: product issued in the previous step ----
      if (step > 0) {
        mbar_wait(s.accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        const float* ar = s.accbuf + row * (16 + 4) + uh * GRU_UPT;
        if (tid == 0) GRU_STAMP(4);
#pragma unroll
        for (int jj = 0; jj < GRU_UPT; ++jj) dh_rec[jj] += active ? ar[jj] : 0.f;
      }
      GruGatesBf16<GRU_UPT> d;
      if (active) {
        d = gru_cell_bwd(dh, dh_rec, sv, hp, db);
        if (step + 1 < T) gru_store_xchg(p, step, row, dir, ju, d);
      }
      if (step + 1 < T) gru_publish(p, ctr, step, active, false);
      if (active) gru_store_bwd(p, m, dir, ju, d);
      if (tid == 0) GRU_STAMP(10);
    }
    // ---- bias gradients: reduce the per-batch-row partial sums over the CTA ----
    epi_barrier();
    float* red = s.scratch;  // [64]: r(16) z(16) n(16) hn(16)
    if (tid < 64) red[tid] = 0.f;
    epi_barrier();
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) {
      const float a = warp_sum(active ? db.r[jj] : 0.f);
      const float b = warp_sum(active ? db.z[jj] : 0.f);
      const float c = warp_sum(active ? db.n[jj] : 0.f);
      const float d = warp_sum(active ? db.hn[jj] : 0.f);
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

// ---- reduce-scatter through L2 (gru_bwd_ks_kernel<true>) ---------------------------------------
// The cluster of the K-split backward kernel serves only the reduce-scatter.  4-CTA clusters cap
// the resident grid (an H100 holds 30 of them, 120 CTAs), so both directions of H = 1024 (128
// CTAs) do not fit as one clustered launch; without a cluster they fit as one ordinary cooperative
// launch of one CTA per SM.  In that mode the "cluster" is a group of 4 consecutive CTAs of a
// direction (group = cta_in_dir / 4, rank = cta_in_dir % 4) and each step's slices travel
// through a global staging area [dir][group][parity][dst][src][slice] instead of DSMEM:
//   * the producer (one epilogue thread) copies its three peer slices from shared memory to the
//     staging area with bulk copies, waits until those WRITES are complete (wait_group, not
//     .read), orders them for the generic proxy and arrives on the group's counter (release);
//   * it then polls the counter (acquire) until all 4 CTAs of the group published the step and
//     fetches the three slices addressed to it with bulk copies that complete on recvbar, exactly
//     where the DSMEM copies of the clustered launch complete.
// Two parities of the staging area are enough: a peer writes parity s & 1 again at step s + 2 at
// the earliest.  That needs its TMA gather of step s + 2, hence the grid barrier of step s + 1,
// which counts the owner's arrival after its epilogue of step s + 1; the owner arrives only after
// recvbar completed for step s + 1, i.e. long after its copies of step s finished reading.
// (The same mode for gru_fwd_ks_kernel<4>, whose slices are 3x larger, measured 11.22 us per step
// for both directions at 64 rows against 11.38 for gru_fwd_kernel, and 7.35 against 6.41 at 32
// rows, H100 80GB HBM3 at 400 W: too little to change the forward's summation order for.)
SB_DEVINL void bulk_s2g(void* gdst, const void* local_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               ::"l"(reinterpret_cast<uint64_t>(gdst)), "r"(smem_u32(local_src)), "r"(bytes)
               : "memory");
}
SB_DEVINL void bulk_g2s(void* dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// One step of the reduce-scatter, issued by one epilogue thread: stage[pr] holds the slice of
// `slice` floats that belongs to rank pr, recv[crank] already holds the CTA's own.  Arms recvbar
// for the three incoming slices, which land in recv[src].  L2RS: gslot is this group's staging
// area of the step's parity, gctr its counter; st (or null) receives two timeline stamps.
template <bool L2RS>
SB_DEVINL void ks_exchange(float* recv, const float* stage, uint64_t* recvbar, uint32_t crank,
                           int slice, float* gslot, unsigned int* gctr, int step,
                           unsigned long long* st) {
  const uint32_t bytes = (uint32_t)slice * 4u;
  mbar_expect_tx(recvbar, (KS - 1) * bytes);
  if (!L2RS) {
    for (uint32_t q = 1; q < KS; ++q) {
      const uint32_t pr = (crank + q) % KS;
      bulk_s2peer(mapa_shared(smem_u32(recv + (size_t)crank * slice), pr),
                  stage + (size_t)pr * slice, bytes, mapa_shared(smem_u32(recvbar), pr));
    }
    return;
  }
  for (uint32_t q = 1; q < KS; ++q) {
    const uint32_t pr = (crank + q) % KS;
    bulk_s2g(gslot + ((size_t)pr * KS + crank) * slice, stage + (size_t)pr * slice, bytes);
  }
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  fence_proxy_async_global();   // async-proxy writes -> the release below
  red_release_gpu_add(gctr, 1u);
  if (st) st[11] = gtime();
  unsigned int spins = 0;
  while (ld_acquire_gpu(gctr) < (unsigned int)(KS * step)) {
    if (++spins > SB_SPIN_LIMIT) __trap();
  }
  if (st) st[12] = gtime();
  for (uint32_t q = 1; q < KS; ++q) {
    const uint32_t src = (crank + q) % KS;
    bulk_g2s(recv + (size_t)src * slice, gslot + ((size_t)crank * KS + src) * slice, bytes,
             recvbar);
  }
}

// L2RS: launched without a cluster, the reduce-scatter goes through L2 (see ks_exchange).
template <bool L2RS>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_bwd_ks_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = p.dir0 + blockIdx.x / nC;
  const int cta_in_dir = blockIdx.x % nC;
  const int j0 = cta_in_dir * GRU_HC;                 // own 16 units (elementwise work)
  const uint32_t crank = L2RS ? (uint32_t)(cta_in_dir % KS) : cluster_rank();
  const int k0c = (cta_in_dir / KS) * (KS * GRU_HC);  // first of the cluster's 64 units
  const int rsg = dir * (nC / KS) + cta_in_dir / KS;  // L2RS: this group's staging area / counter
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
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const int gc = (nchunks % 4 == 0) ? 4 : ((nchunks % 3 == 0) ? 3 : ((nchunks % 2 == 0) ? 2 : 1));
  const int ngroups = nchunks / gc;                   // <= 4 for H <= 1024 ... checked on host

  smem_zero(base, ring_bytes + wbytes + 2 * KS * Bp * 64);
  __syncthreads();
  // resident operand: rows = the cluster's 64 units of W_hh^T, columns = this CTA's K quarter
  stage_w_cols<KS * GRU_HC>(wtile, p.whh + (long long)dir * K3 * H, H, (int)crank * KQ, KQ, k0c);
  gru_init_barriers(tm, nullptr, !L2RS, [=] {
    for (int i = 0; i < 4; ++i) mbar_init(&full[i], 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);   // one local arrive.expect_tx per step; the peers' copies complete_tx
  });
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
    float dh_rec[GRU_UPT] = {};
    GruGates<GRU_UPT> db = {};

    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? (T - 1 - step) : step;
      const long long m = (long long)t * Bp + row;
      GruGates<GRU_UPT> sv;
      float dh[GRU_UPT], hp[GRU_UPT];
      if (active) gru_load_saved(p, t, row, dir, ju, sv, dh, hp);
      // ---- recurrent part of dL/dh_t: reduce-scatter of the four partial products ----
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        // the MMA warpgroup staged the peers' slices: one bulk copy into each peer's receive
        // buffer; the own slice already sits in recv[crank]
        if (tid == 0)
          ks_exchange<L2RS>(recv, stage, recvbar, crank, Bp * 16,
                            p.rs + ((size_t)rsg * 2 + (step & 1)) * KS * KS * Bp * 16,
                            p.rsctr + rsg * 32, step,
                            (p.dbg && blockIdx.x == 0 && step < 64) ? p.dbg + step * 16 : nullptr);
        if (tid == 0) GRU_STAMP(4);
        mbar_wait(recvbar, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(13);
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
      GruGatesBf16<GRU_UPT> d;
      if (active) {
        d = gru_cell_bwd(dh, dh_rec, sv, hp, db);
        if (step + 1 < T) gru_store_xchg(p, step, row, dir, ju, d);
      }
      if (step + 1 < T) gru_publish(p, ctr, step, active, false);
      if (active) gru_store_bwd(p, m, dir, ju, d);
      if (tid == 0) GRU_STAMP(10);
    }
#pragma unroll
    for (int jj = 0; jj < GRU_UPT; ++jj) {
      const float a = warp_sum(active ? db.r[jj] : 0.f);
      const float b = warp_sum(active ? db.z[jj] : 0.f);
      const float c = warp_sum(active ? db.n[jj] : 0.f);
      const float d = warp_sum(active ? db.hn[jj] : 0.f);
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
  if (!L2RS) cluster_sync_all();
}

// =============================================================================================
// forward, K-split variant: the KS CTAs of a cluster (KS = 4 or 2) jointly own KS x 16 hidden
// units.
//
// Measured on gru_fwd_kernel (globaltimer timeline, H = 1024, B = 64, 7.4 us/step): 3.5 us pass
// between "h_{t-1} is complete" and "all MMAs retired", for a gather of 128 KB per CTA - the same
// ~30 B/ns per SM whether it is fetched as tensor boxes or as contiguous bulk copies, with or
// without cluster multicast: 128 CTAs x 128 KB = 16 MB of L2->SM traffic per step is the bound,
// next to 480 KB of shared-memory traffic (TMA writes + MMA operand reads of a 128-row A tile).
// Here CTA r of a cluster contracts only the r-th of KS slices of K = H, for all KS x 16 units of
// its cluster and all three gates (KS = 4: N = 192, quarters of K),
//     D_r[batch x 3*KS*16] = h_{t-1}[:, slice r] * W_hh[(r|z|n) x KS*16 units, slice r]^T,
// i.e. it gathers H/KS columns of h_{t-1} instead of all H (KS = 4: 32 KB instead of 128 KB at
// H = 1024, Bp = 64; the whole slice stays resident: no ring) and issues 4*H/(KS*64) MMAs of
// N = 3*KS*16 instead of H/16 of N = 48; the KS partial products are reduce-scattered through
// distributed shared memory exactly as in gru_bwd_ks_kernel (each CTA receives the 3 x 16 columns
// of its own units from each of its KS - 1 peers: 12 KB per peer at Bp = 64) and summed in rank
// order, so the result does not depend on arrival order.
// KS = 2 exists because an H100 holds at most 30 clusters of 4 such CTAs (120): both directions of
// H = 1024 (128 CTAs) do not fit with KS = 4, but fit as 64 clusters of 2, and each CTA still
// gathers half of h_{t-1} (64 KB at Bp = 64) instead of all of it.  Shared memory at Bp = 64,
// H = 1024 (operand + weights + recv/stage, plus 1.5 KB of barriers and alignment): KS = 4
// 32 + 96 + 96 KB, KS = 2 64 + 96 + 48 KB.  Measured on an H100 80GB HBM3 at 400 W, both
// directions of H = 1024, T = 247: 7.50 us per step at 64 rows and 5.10 at 32 with KS = 2,
// against 11.11 and 6.54 for gru_fwd_kernel.  The globaltimer timeline (tools/gru_timeline.py) of
// KS = 2 at 64 rows: 2.8 us from the CTA's own arrive until the grid barrier completes, 0.45 us to
// issue the gather, 1.5 us until the product is staged, 1.5-1.7 us for the exchange and gate math
// until h_t is stored, 1.0-1.25 us more until the arrive.
// Requires cluster size KS, H % (KS * 64) == 0, Bp <= 64.
// =============================================================================================
template <int KS, bool H0>
SB_DEVINL void gru_fwd_ks_body(const CUtensorMap& tm_d0, const CUtensorMap& tm_d1,
                               const GruFwdParams& p) {
  static_assert(KS == 2 || KS == 4, "gru_fwd_ks_kernel: K split 2 or 4 ways");
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / GRU_HC;
  const int dir = blockIdx.x / nC;
  const int cta_in_dir = blockIdx.x % nC;
  const int j0 = cta_in_dir * GRU_HC;                 // own 16 units (gate math, stores)
  const uint32_t crank = cluster_rank();              // == cta_in_dir % KS
  const int k0c = (cta_in_dir / KS) * (KS * GRU_HC);  // first of the cluster's KS*16 units
  const int KQ = H / KS;                              // this CTA's share of the contraction
  const int nchunks = KQ / 64;
  constexpr int NCOL = 3 * KS * GRU_HC;               // accumulator columns: gate x KS*16 units
  constexpr int WCHUNK = NCOL * 128;                  // NCOL rows x 64 bf16
  constexpr int RW = 3 * GRU_HC;                      // 48 floats received per row and peer
  const int stride = Bp * 128;
  const int ring_bytes = nchunks * stride;            // the whole K slice is resident
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

  smem_zero(base, ring_bytes + wbytes + 2 * KS * Bp * RW * 4);
  __syncthreads();
  // resident operand: rows = (gate, unit of the cluster), columns = this CTA's K slice
  stage_w_rows(wtile, WCHUNK, p.whh + (long long)dir * 3 * H * H, H, NCOL, (int)crank * KQ, KQ,
               [=](int r) { return (r / (KS * GRU_HC)) * H + k0c + r % (KS * GRU_HC); });
  if (tid < RW) bias_s[tid] = p.bhh[dir * 3 * H + (tid / GRU_HC) * H + j0 + tid % GRU_HC];
  gru_init_barriers(tm, nullptr, true, [=] {
    mbar_init(full, 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);   // one local arrive.expect_tx per step; the peers' copies complete_tx
  });
  unsigned int* ctr = p.barrier + dir * 32;   // one L2 line per direction

  if (warp == GRU_TMA_WARP) {
    // ===================== TMA producer: this CTA's K slice of h_{t-1} =======================
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
    // ===================== MMA warpgroup: D[Bp x (gate, KS*16 units)] for this K slice ========
    // Column gg*KS*16 + pr*16 + u belongs to unit u of peer pr: it is written straight into
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
        const int r = wg_frag_row(t, i), col = wg_frag_col(t, i);   // col >= 0
        const int gg = (uint32_t)col / (KS * GRU_HC), u = col & 15;
        const uint32_t pr = (uint32_t)(col >> 4) % KS;
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
    float hprev[GRU_UPT] = {};
    float bias[3][GRU_UPT];
    gru_load_bias(bias_s + uh * GRU_UPT, GRU_HC, bias);

    int step0 = 0;
    if constexpr (H0) {
      if (active) gru_load_h0(p, row, ju, hprev);
      gru_publish(p, ctr, 0, false, true);
      step0 = 1;
    }
    for (int step = step0; step < T; ++step) {
      const int t = dir == 0 ? step : (T - 1 - step);
      float gi[3][GRU_UPT];
      if (active) gru_load_gi(p, t - step0, row, dir, ju, gi);
      float acc[3][GRU_UPT] = {};
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        // ---- reduce-scatter of the KS partial products: the MMA warpgroup staged the KS - 1
        // slices that belong to the peers, each leaves as ONE bulk copy into the peer's receive
        // buffer; the CTA's own slice already sits in recv[crank].  The slices are summed in
        // rank order below, whatever order they arrived in ----
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
      GruGates<GRU_UPT> gt;
      if (active) {
        gru_cell_fwd(gi, acc, bias, hprev, gt);
        st_bf16(p.xn + m * D + dir * H + ju, to_bf16(hprev));
      }
      gru_publish(p, ctr, step, active, true);
      if (active) gru_store_fwd(p, m, dir, ju, hprev, gt);
      if (tid == 0) GRU_STAMP(10);
    }
  }

  __syncthreads();
  cluster_sync_all();
}

template <int KS>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_ks_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruFwdParams p) {
  gru_fwd_ks_body<KS, false>(tm_d0, tm_d1, p);
}
template <int KS>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_ks_h0_kernel(const __grid_constant__ CUtensorMap tm_d0,
                     const __grid_constant__ CUtensorMap tm_d1, const GruFwdParams p) {
  gru_fwd_ks_body<KS, true>(tm_d0, tm_d1, p);
}

// =============================================================================================
// forward, K split with the accumulator TRANSPOSED: D^T[(gate, unit) x batch].
//
// Same partition as gru_fwd_ks_kernel<4> (cluster of 4 owns 64 units, CTA r contracts K quarter r),
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
// Owner-major staging of the transposed accumulators: slice of peer q (the own slice lives in
// recv[crank], the others in stage[(q - crank) mod KS - 1]), row srow, column = batch row.
SB_DEVINL float* kt_slice(float* recv, float* stage, int slice, uint32_t q, uint32_t crank) {
  const uint32_t q0 = (q + KS - crank) % KS;
  return q0 == 0 ? recv + (size_t)crank * slice : stage + (size_t)(q0 - 1) * slice;
}

// Reduce-scatter of one step once the MMA warpgroup staged the three outgoing slices (and the own
// one in recv[crank]): thread 0 arms recvbar for the incoming ones, lane 0 of warp w = 1..3 sends
// the slice of peer crank + w as one bulk copy into its recv[crank].
SB_DEVINL void kt_exchange(float* recv, const float* stage, uint64_t* recvbar, uint32_t crank,
                           int slice) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) mbar_expect_tx(recvbar, (uint32_t)((KS - 1) * slice * 4));
  if (lane == 0 && warp >= 1 && warp <= KS - 1) {
    const uint32_t pr = (crank + (uint32_t)warp) % KS;
    bulk_s2peer(mapa_shared(smem_u32(recv + (size_t)crank * slice), pr),
                stage + (size_t)(warp - 1) * slice, (uint32_t)(slice * 4),
                mapa_shared(smem_u32(recvbar), pr));
  }
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

template <int UPT, bool H0>
SB_DEVINL void gru_fwd_kt_body(const CUtensorMap& tm_d0, const CUtensorMap& tm_d1,
                               const GruFwdParams& p) {
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

  smem_zero(base, ring_bytes + wbytes + (2 * KS - 1) * slice * 4);
  __syncthreads();
  // resident operand: rows ordered by owner (see above), columns = this CTA's K quarter
  stage_w_rows(wtile, WCHUNK, p.whh + (long long)dir * 3 * H * H, H, WROWS, (int)crank * KQ, KQ,
               [=](int r) {
                 return r < 128 ? ((r & 31) >> 4) * H + k0c + (r >> 5) * GRU_HC + (r & 15)
                                : 2 * H + k0c + r - 128;
               });
  if (tid < RW) bias_s[tid] = p.bhh[dir * 3 * H + (tid / GRU_HC) * H + j0 + tid % GRU_HC];
  gru_init_barriers(tm, nullptr, true, [=] {
    mbar_init(full, 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);   // one local arrive.expect_tx per step; the peers' copies complete_tx
  });
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
    float hprev[UPT] = {};
    float bias[3][UPT] = {};
    if (active) gru_load_bias(bias_s + u0, GRU_HC, bias);

    int step0 = 0;
    if constexpr (H0) {
      if (active) gru_load_h0(p, b, ju, hprev);
      gru_publish(p, ctr, 0, false, true);
      step0 = 1;
    }
    for (int step = step0; step < T; ++step) {
      const int t = dir == 0 ? step : (T - 1 - step);
      float gi[3][UPT];
      if (active) gru_load_gi(p, t - step0, b, dir, ju, gi);
      float acc[3][UPT] = {};
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        kt_exchange(recv, stage, recvbar, crank, slice);
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
      GruGates<UPT> gt;
      if (active) {
        gru_cell_fwd(gi, acc, bias, hprev, gt);
        st_bf16(p.xn + m * D + dir * H + ju, to_bf16(hprev));
      }
      gru_publish(p, ctr, step, active, true);
      if (active) gru_store_fwd(p, m, dir, ju, hprev, gt);
      if (tid == 0) GRU_STAMP(10);
    }
  }

  __syncthreads();
  cluster_sync_all();
}

template <int UPT>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_kt_kernel(const __grid_constant__ CUtensorMap tm_d0,
                  const __grid_constant__ CUtensorMap tm_d1, const GruFwdParams p) {
  gru_fwd_kt_body<UPT, false>(tm_d0, tm_d1, p);
}
template <int UPT>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_kt_h0_kernel(const __grid_constant__ CUtensorMap tm_d0,
                     const __grid_constant__ CUtensorMap tm_d1, const GruFwdParams p) {
  gru_fwd_kt_body<UPT, true>(tm_d0, tm_d1, p);
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
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const int gc = (nchunks % 4 == 0) ? 4 : ((nchunks % 3 == 0) ? 3 : ((nchunks % 2 == 0) ? 2 : 1));
  const int ngroups = nchunks / gc;                   // <= 4 for H <= 1024 ... checked on host

  smem_zero(base, ring_bytes + wbytes + (2 * KS - 1) * slice * 4);
  __syncthreads();
  // resident operand: see gru_bwd_ks_kernel
  stage_w_cols<KS * GRU_HC>(wtile, p.whh + (long long)dir * K3 * H, H, (int)crank * KQ, KQ, k0c);
  gru_init_barriers(tm, nullptr, true, [=] {
    for (int i = 0; i < 4; ++i) mbar_init(&full[i], 1);
    mbar_init(accfull, 128);
    mbar_init(recvbar, 1);
  });
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
    float dh_rec[UPT] = {};
    GruGates<UPT> db = {};

    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? (T - 1 - step) : step;
      const long long m = (long long)t * Bp + b;
      GruGates<UPT> sv;
      float dh[UPT], hp[UPT];
      if (active) gru_load_saved(p, t, b, dir, ju, sv, dh, hp);
      if (step > 0) {
        mbar_wait(accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
        kt_exchange(recv, stage, recvbar, crank, slice);
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
      GruGatesBf16<UPT> d;
      if (active) {
        d = gru_cell_bwd(dh, dh_rec, sv, hp, db);
        if (step + 1 < T) gru_store_xchg(p, step, b, dir, ju, d);
      }
      if (step + 1 < T) gru_publish(p, ctr, step, active, false);
      if (active) gru_store_bwd(p, m, dir, ju, d);
      if (tid == 0) GRU_STAMP(10);
    }
    if (active) {
#pragma unroll
      for (int jj = 0; jj < UPT; ++jj) {
        const int bi = dir * K3 + ju + jj;
        atomicAdd(p.dbih + bi, db.r[jj]);
        atomicAdd(p.dbih + bi + H, db.z[jj]);
        atomicAdd(p.dbih + bi + 2 * H, db.n[jj]);
        atomicAdd(p.dbhh + bi, db.r[jj]);
        atomicAdd(p.dbhh + bi + H, db.z[jj]);
        atomicAdd(p.dbhh + bi + 2 * H, db.hn[jj]);
      }
    }
  }

  __syncthreads();
  cluster_sync_all();
}

// =============================================================================================
// wide layers: W_hh no longer fits in the shared memory of one CTA per 16 units per SM.
//
// CTA c of direction d owns U = 16 or 32 hidden units (ndir * H / U <= SM count).  Its weight
// slice is NW = 3U rows of W_hh (forward) or U rows of W_hh^T (backward), cut into 64-wide K
// chunks handled in groups of gc chunks.  The first rg groups stay resident in shared memory; the
// remaining ones are streamed from L2 every step through a ring of wr slots of their own (TMA with
// an evict_last hint: the weights are the only operand every step re-reads).  The producer issues
// the first min(streamed, wr) weight groups of a step BEFORE it waits on the grid barrier, so that
// they travel during the wait; the rest follow the gather group they pair with.  Producer order
// never waits on something not yet issued: the gather slot of group g is released by group
// g - ring, the weight slot of streamed group g by streamed group g - wr, both issued earlier.
// The all-gather of h_{t-1} / dgh_t, the grid barrier, the .cs stores and the GRU_STAMP points are
// those of gru_fwd_kernel / gru_bwd_kernel.  The epilogue maps thread = (batch row, 8 units) with
// 2048 / U rows per pass of the 256 threads, so NQ = 2 passes at U = 32 above 64 rows.
// The backward reads its weight tiles K-major from a transposed copy W_hh^T in the workspace
// that each CTA writes for its own U rows in its prologue, so both passes share one tile format.
// Shared memory: gather ring | resident groups | weight ring (at least 16 KB - Bp*128 after the
// gather ring: the 64/128-row A read of the last slot runs past it) | barriers | bias | product.
// =============================================================================================
static constexpr int GRU_WIDE_MAX_WR = 8;
static constexpr int GRU_WIDE_GATHER_KB = 64;   // default gather-ring bytes / 1024 (see below)
static constexpr int GRU_FORCE_STREAM = 2048;   // sb_debug_gru_flags bit: wide kernels, rg = 0

SB_DEVINL uint64_t l2_evict_last_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
SB_DEVINL void tma_load_2d_hint(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0,
                                int32_t c1, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      ".L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1), "l"(pol)
      : "memory");
}

struct WideSmem {
  uint8_t* ring;     // gather ring
  uint8_t* wres;     // resident weight groups
  uint8_t* wring;    // streamed weight groups
  uint64_t *full, *empty, *wfull, *wempty, *accfull, *wresbar;
  float* scratch;    // [4 * U]: bias (forward) / bias-gradient reduction (backward)
  float* accbuf;     // [Bp][NW + 4]
};

__host__ __device__ inline int gru_wide_wbytes(int rg, int wr, int wgroup, int Bp) {
  const int w = (rg + wr) * wgroup;
  return w > 16384 - Bp * 128 ? w : 16384 - Bp * 128;
}

SB_DEVINL WideSmem wide_carve(uint8_t* raw, int ring_bytes, int rg, int wgroup, int wbytes, int U) {
  WideSmem s;
  s.ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) &
                                      ~static_cast<uintptr_t>(1023));
  s.wres = s.ring + ring_bytes;
  s.wring = s.wres + rg * wgroup;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s.wres + wbytes);
  s.full = bars;
  s.empty = bars + GRU_MAX_RING;
  s.wfull = bars + 2 * GRU_MAX_RING;
  s.wempty = s.wfull + GRU_WIDE_MAX_WR;
  s.accfull = s.wempty + GRU_WIDE_MAX_WR;
  s.wresbar = s.accfull + 1;
  s.scratch = reinterpret_cast<float*>(s.wresbar + 1);
  s.accbuf = s.scratch + 4 * U;
  return s;
}

// Weight group g into `dst` (gc chunks of NW rows = nbox boxes of U rows each; box b of chunk c
// comes from rows wrow0 + b * wstep, columns c * 64 of the weight tensor map).
SB_DEVINL void wide_load_wgroup(uint8_t* dst, const CUtensorMap* tw, uint64_t* bar, int g, int gc,
                                int U, int nbox, int wrow0, int wstep, uint64_t pol) {
  for (int i = 0; i < gc; ++i) {
    const int c = g * gc + i;
    for (int b = 0; b < nbox; ++b)
      tma_load_2d_hint(dst + (i * nbox + b) * U * 128, tw, bar, c * 64, wrow0 + b * wstep, pol);
  }
}

// streamed weight group g (rg <= g < ngroups) into weight-ring slot wn % wr; wn counts the
// streamed groups issued since the launch
SB_DEVINL void wide_issue_wgroup(const WideSmem& s, const CUtensorMap* tw, int g, int gc, int U,
                                 int nbox, int wr, unsigned int& wn, int wrow0, int wstep,
                                 uint64_t pol) {
  const int slot = (int)(wn % (unsigned int)wr);
  const unsigned int use = wn / (unsigned int)wr;
  if (use > 0) mbar_wait(&s.wempty[slot], (use - 1u) & 1u);
  mbar_expect_tx(&s.wfull[slot], (uint32_t)(gc * nbox * U * 128));
  wide_load_wgroup(s.wring + slot * gc * nbox * U * 128, tw, &s.wfull[slot], g, gc, U, nbox, wrow0,
                   wstep, pol);
  ++wn;
}

// TMA producer of one product: wide_prefetch_weights ahead of the grid barrier, wide_gather after
// it (the gather interleaved with the streamed weight groups the prefetch left out)
SB_DEVINL void wide_prefetch_weights(const WideSmem& s, const CUtensorMap* tw, int ngroups, int gc,
                                     int rg, int wr, int U, int nbox, int wrow0, int wstep,
                                     unsigned int& wn, uint64_t pol) {
  const int sg = ngroups - rg;
  const int pre = sg < wr ? sg : wr;
  for (int g = rg; g < rg + pre; ++g)
    wide_issue_wgroup(s, tw, g, gc, U, nbox, wr, wn, wrow0, wstep, pol);
}
// The gather ring of the wide kernels counts its uses across steps (gn), so any ring of >= 2
// slots works: every reuse waits for the slot's release, whatever the group count.
SB_DEVINL void wide_gather(const WideSmem& s, const CUtensorMap* tm, const CUtensorMap* tw,
                           int row0, int Bp, int ngroups, int ring, int gc, int rg, int wr, int U,
                           int nbox, int wrow0, int wstep, unsigned int& gn, unsigned int& wn,
                           uint64_t pol, uint32_t rank, uint32_t cs) {
  const int sg = ngroups - rg;
  const int pre = sg < wr ? sg : wr;
  const int stride = Bp * 128;
  const uint16_t mask = (uint16_t)((1u << cs) - 1u);
  for (int g = 0; g < ngroups; ++g, ++gn) {
    const int slot = (int)(gn % (unsigned int)ring);
    const unsigned int use = gn / (unsigned int)ring;
    if (use > 0) mbar_wait(&s.empty[slot], (use - 1u) & 1u);   // released by ALL CTAs of the cluster
    mbar_expect_tx(&s.full[slot], (uint32_t)(stride * gc));
    for (int i = 0; i < gc; ++i) {
      const int c = g * gc + i;
      if ((uint32_t)c % cs != rank) continue;
      uint8_t* dst = s.ring + (slot * gc + i) * stride;
      if (cs > 1) tma_load_2d_mc(dst, tm, &s.full[slot], c * 64, row0, mask);
      else tma_load_2d(dst, tm, &s.full[slot], c * 64, row0);
    }
    if (g >= rg + pre) wide_issue_wgroup(s, tw, g, gc, U, nbox, wr, wn, wrow0, wstep, pol);
  }
}

// MMA warpgroup, product k: D[Bp x NW] over all groups, resident or streamed; parks D in accbuf
// (pitch NW + 4) and arrives on accfull (count 128).  wn counts the streamed groups consumed.  One
// group's MMAs stay in flight while the next group's operands are awaited: a group's gather and
// weight slots are released once the following group has been issued and it has retired.
template <int NW, bool TWO>
SB_DEVINL void wide_mma(const WideSmem& s, int Bp, int ngroups, int ring, int gc, int rg, int wr,
                        unsigned int& gn, unsigned int& wn, uint32_t cs) {
  constexpr int WCHUNK = NW * 128;
  const int stride = Bp * 128;
  const bool leader = (threadIdx.x & 127) == 0;
  float d0[NW / 2], d1[NW / 2];
  int prev_slot = -1, prev_wslot = -1;
  auto release = [&](int slot, int wslot) {
    if (!leader || slot < 0) return;
    if (cs > 1) mbar_arrive_all_ctas(&s.empty[slot], cs);
    else mbar_arrive(&s.empty[slot]);
    if (wslot >= 0) mbar_arrive(&s.wempty[wslot]);
  };
  for (int g = 0; g < ngroups; ++g, ++gn) {
    const int slot = (int)(gn % (unsigned int)ring);
    mbar_wait(&s.full[slot], (gn / (unsigned int)ring) & 1u);
    int wslot = -1;
    const uint8_t* wsrc = s.wres + g * gc * WCHUNK;
    if (g >= rg) {
      wslot = (int)(wn % (unsigned int)wr);
      mbar_wait(&s.wfull[wslot], (wn / (unsigned int)wr) & 1u);
      wsrc = s.wring + wslot * gc * WCHUNK;
      ++wn;
    }
    wgmma_fence();
    for (int i = 0; i < gc; ++i) {
      const int c = g * gc + i;
      const uint32_t sa = smem_u32(s.ring + (slot * gc + i) * stride);
      const uint64_t da0 = gmma_desc_sw128_kmajor(sa);
      const uint64_t da1 = gmma_desc_sw128_kmajor(sa + 64 * 128);
      const uint64_t db = gmma_desc_sw128_kmajor(smem_u32(wsrc + i * WCHUNK));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t acc = (c > 0 || kk > 0) ? 1u : 0u;
        wgmma_bf16<NW>(d0, da0 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), acc);
        if constexpr (TWO) wgmma_bf16<NW>(d1, da1 + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), acc);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();          // the previous group's MMAs have retired
    release(prev_slot, prev_wslot);
    prev_slot = slot;
    prev_wslot = wslot;
  }
  wgmma_wait<0>();
  release(prev_slot, prev_wslot);
  wgmma_fence_regs(d0);
  wg_store_rows<NW>(d0, s.accbuf, NW + 4, 0, Bp);
  if constexpr (TWO) {
    wgmma_fence_regs(d1);
    wg_store_rows<NW>(d1, s.accbuf, NW + 4, 64, Bp);
  }
  mbar_arrive(s.accfull);
}

// one-time setup shared by both wide kernels: zero the operand regions, barriers, cluster sync
SB_DEVINL void wide_setup(const WideSmem& s, int ring_bytes, int wbytes, uint32_t csize,
                          const CUtensorMap* tm, const CUtensorMap* tw) {
  smem_zero(s.ring, ring_bytes + wbytes);
  gru_init_barriers(tm, tw, true, [=] {
    init_ring_bars(s.full, s.empty, csize);
    for (int i = 0; i < GRU_WIDE_MAX_WR; ++i) {
      mbar_init(&s.wfull[i], 1);
      mbar_init(&s.wempty[i], 1);
    }
    mbar_init(s.accfull, 128);
    mbar_init(s.wresbar, 1);
  });
}

template <int U, int NQ, bool H0>
SB_DEVINL void gru_fwd_wide_body(const CUtensorMap& tm_d0, const CUtensorMap& tm_d1,
                                 const CUtensorMap& tm_w, const GruFwdParams& p) {
  constexpr int NW = 3 * U;
  constexpr int WCHUNK = NW * 128;
  constexpr int RPT = 2048 / U;      // batch rows per pass of the 256 epilogue threads
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / U;
  const int dir = blockIdx.x / nC;
  const int j0 = (blockIdx.x % nC) * U;
  const int nchunks = (H + 63) / 64;
  const int gc = p.gc, ngroups = nchunks / gc, rg = p.rg, wr = p.wr;
  const int ring_bytes = p.ring * gc * Bp * 128;
  const int wbytes = gru_wide_wbytes(rg, wr, gc * WCHUNK, Bp);
  const WideSmem s = wide_carve(smem_raw, ring_bytes, rg, gc * WCHUNK, wbytes, U);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = p.ndir * H;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const uint32_t crank = cluster_rank(), csize = cluster_size();
  const int wrow0 = dir * 3 * H + j0;   // gate b of the slice: rows wrow0 + b * H of W_hh

  if (tid < NW) s.scratch[tid] = p.bhh[dir * 3 * H + (tid / U) * H + j0 + tid % U];
  wide_setup(s, ring_bytes, wbytes, csize, tm, &tm_w);
  unsigned int* ctr = p.barrier + dir * 32;

  if (warp == GRU_TMA_WARP) {
    if (lane == 0) {
      const uint64_t pol = l2_evict_last_policy();
      if (rg > 0) {
        mbar_expect_tx(s.wresbar, (uint32_t)(rg * gc * WCHUNK));
        for (int g = 0; g < rg; ++g)
          wide_load_wgroup(s.wres + g * gc * WCHUNK, &tm_w, s.wresbar, g, gc, U, 3, wrow0, H, pol);
      }
      unsigned int gn = 0, wn = 0;
      for (int step = 1; step < T; ++step) {
        const int t = dir == 0 ? step : (T - 1 - step);
        const int tp = dir == 0 ? t - 1 : t + 1;
        wide_prefetch_weights(s, &tm_w, ngroups, gc, rg, wr, U, 3, wrow0, H, wn, pol);
        grid_wait(ctr, (unsigned int)nC * step);   // all CTAs published h_{tp}
        GRU_STAMP(0);
        wide_gather(s, tm, &tm_w, tp * Bp, Bp, ngroups, p.ring, gc, rg, wr, U, 3, wrow0, H, gn,
                    wn, pol, crank, csize);
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    if (rg > 0) mbar_wait(s.wresbar, 0);
    unsigned int gn = 0, wn = 0;
    for (int step = 1; step < T; ++step) {
      if (Bp > 64) wide_mma<NW, true>(s, Bp, ngroups, p.ring, gc, rg, wr, gn, wn, csize);
      else wide_mma<NW, false>(s, Bp, ngroups, p.ring, gc, rg, wr, gn, wn, csize);
      if (tid == GRU_MMA_WARP * 32) GRU_STAMP(2);
    }
  } else {
    // ===================== epilogue: thread = (batch row, 8 of the CTA's U units) per pass =====
    const int rsub = tid % RPT;
    const int uo = (tid / RPT) * GRU_UPT;
    const int ju = j0 + uo;
    float hprev[NQ][GRU_UPT] = {};
    float bias[3][GRU_UPT];
    gru_load_bias(s.scratch + uo, U, bias);
    int step0 = 0;
    if constexpr (H0) {
#pragma unroll
      for (int q = 0; q < NQ; ++q)
        if (rsub + q * RPT < Bp) gru_load_h0(p, rsub + q * RPT, ju, hprev[q]);
      gru_publish(p, ctr, 0, false, false);
      step0 = 1;
    }
    for (int step = step0; step < T; ++step) {
      const int t = dir == 0 ? step : (T - 1 - step);
      float gi[NQ][3][GRU_UPT];
#pragma unroll
      for (int q = 0; q < NQ; ++q)
        if (rsub + q * RPT < Bp) gru_load_gi(p, t - step0, rsub + q * RPT, dir, ju, gi[q]);
      if (step > 0) {
        mbar_wait(s.accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
      }
      GruGates<GRU_UPT> gt[NQ];
      bool any = false;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int row = rsub + q * RPT;
        if (row >= Bp) continue;
        any = true;
        const float* ar = s.accbuf + row * (NW + 4) + uo;
        float acc[3][GRU_UPT];
#pragma unroll
        for (int gg = 0; gg < 3; ++gg)
#pragma unroll
          for (int jj = 0; jj < GRU_UPT; ++jj) acc[gg][jj] = step > 0 ? ar[gg * U + jj] : 0.f;
        gru_cell_fwd(gi[q], acc, bias, hprev[q], gt[q]);
        st_bf16(p.xn + ((long long)t * Bp + row) * D + dir * H + ju, to_bf16(hprev[q]));
      }
      gru_publish(p, ctr, step, any, false);
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int row = rsub + q * RPT;
        if (row < Bp) gru_store_fwd(p, (long long)t * Bp + row, dir, ju, hprev[q], gt[q]);
      }
      if (tid == 0) GRU_STAMP(10);
    }
  }

  __syncthreads();
  cluster_sync_all();
}

template <int U, int NQ>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_wide_kernel(const __grid_constant__ CUtensorMap tm_d0,
                    const __grid_constant__ CUtensorMap tm_d1,
                    const __grid_constant__ CUtensorMap tm_w, const GruFwdParams p) {
  gru_fwd_wide_body<U, NQ, false>(tm_d0, tm_d1, tm_w, p);
}
template <int U, int NQ>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_fwd_wide_h0_kernel(const __grid_constant__ CUtensorMap tm_d0,
                       const __grid_constant__ CUtensorMap tm_d1,
                       const __grid_constant__ CUtensorMap tm_w, const GruFwdParams p) {
  gru_fwd_wide_body<U, NQ, true>(tm_d0, tm_d1, tm_w, p);
}

template <int U, int NQ>
__global__ void __launch_bounds__(GRU_THREADS, 1)
gru_bwd_wide_kernel(const __grid_constant__ CUtensorMap tm_d0,
                    const __grid_constant__ CUtensorMap tm_d1,
                    const __grid_constant__ CUtensorMap tm_w, const GruBwdParams p) {
  constexpr int WCHUNK = U * 128;
  constexpr int RPT = 2048 / U;
  extern __shared__ uint8_t smem_raw[];
  const int H = p.H, Bp = p.Bp, T = p.T;
  const int nC = H / U;
  const int dir = blockIdx.x / nC;
  const int j0 = (blockIdx.x % nC) * U;
  const int K3 = 3 * H;
  const int nchunks = (K3 + 63) / 64;
  const int gc = p.gc, ngroups = nchunks / gc, rg = p.rg, wr = p.wr;
  const int ring_bytes = p.ring * gc * Bp * 128;
  const int wbytes = gru_wide_wbytes(rg, wr, gc * WCHUNK, Bp);
  const WideSmem s = wide_carve(smem_raw, ring_bytes, rg, gc * WCHUNK, wbytes, U);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const CUtensorMap* tm = dir == 0 ? &tm_d0 : &tm_d1;
  const uint32_t crank = cluster_rank(), csize = cluster_size();
  const int wrow0 = dir * H + j0;       // rows of W_hh^T: the CTA's units

  // this CTA's U rows of W_hh^T (read back by its own TMA only): thread = (k, 8 units)
  for (int k = tid; k < K3 * (U / 8); k += GRU_THREADS) {
    const int kk = k % K3, piece = k / K3;
    const uint4 v = *reinterpret_cast<const uint4*>(
        p.whh + ((long long)dir * K3 + kk) * H + j0 + piece * 8);
    const bf16* e = reinterpret_cast<const bf16*>(&v);
#pragma unroll
    for (int q = 0; q < 8; ++q) p.whhT[(long long)(wrow0 + piece * 8 + q) * K3 + kk] = e[q];
  }
  fence_proxy_async_global();   // generic writes -> this CTA's TMA reads
  wide_setup(s, ring_bytes, wbytes, csize, tm, &tm_w);
  unsigned int* ctr = p.barrier + dir * 32;

  if (warp == GRU_TMA_WARP) {
    if (lane == 0) {
      const uint64_t pol = l2_evict_last_policy();
      if (rg > 0) {
        mbar_expect_tx(s.wresbar, (uint32_t)(rg * gc * WCHUNK));
        for (int g = 0; g < rg; ++g)
          wide_load_wgroup(s.wres + g * gc * WCHUNK, &tm_w, s.wresbar, g, gc, U, 1, wrow0, 0, pol);
      }
      unsigned int gn = 0, wn = 0;
      for (int step = 0; step + 1 < T; ++step) {
        wide_prefetch_weights(s, &tm_w, ngroups, gc, rg, wr, U, 1, wrow0, 0, wn, pol);
        grid_wait(ctr, (unsigned int)nC * (step + 1));   // dgh of this step is complete
        GRU_STAMP(0);
        wide_gather(s, tm, &tm_w, (step & 1) * Bp, Bp, ngroups, p.ring, gc, rg, wr, U, 1, wrow0, 0,
                    gn, wn, pol, crank, csize);
        GRU_STAMP(1);
      }
    }
  } else if (warp >= GRU_MMA_WARP) {
    if (rg > 0) mbar_wait(s.wresbar, 0);
    unsigned int gn = 0, wn = 0;
    for (int step = 0; step + 1 < T; ++step) {
      if (Bp > 64) wide_mma<U, true>(s, Bp, ngroups, p.ring, gc, rg, wr, gn, wn, csize);
      else wide_mma<U, false>(s, Bp, ngroups, p.ring, gc, rg, wr, gn, wn, csize);
      if (tid == GRU_MMA_WARP * 32) GRU_STAMP(2);
    }
  } else {
    const int rsub = tid % RPT;
    const int uo = (tid / RPT) * GRU_UPT;
    const int ju = j0 + uo;
    float dh_rec[NQ][GRU_UPT] = {};
    GruGates<GRU_UPT> db[NQ] = {};

    for (int step = 0; step < T; ++step) {
      const int t = dir == 0 ? (T - 1 - step) : step;
      GruGates<GRU_UPT> sv[NQ];
      float dh[NQ][GRU_UPT], hp[NQ][GRU_UPT];
#pragma unroll
      for (int q = 0; q < NQ; ++q)
        if (rsub + q * RPT < Bp) gru_load_saved(p, t, rsub + q * RPT, dir, ju, sv[q], dh[q], hp[q]);
      if (step > 0) {
        mbar_wait(s.accfull, (step - 1) & 1);
        if (tid == 0) GRU_STAMP(3);
      }
      GruGatesBf16<GRU_UPT> d[NQ];
      bool any = false;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int row = rsub + q * RPT;
        if (row >= Bp) continue;
        any = true;
        const float* ar = s.accbuf + row * (U + 4) + uo;
        if (step > 0) {
#pragma unroll
          for (int jj = 0; jj < GRU_UPT; ++jj) dh_rec[q][jj] += ar[jj];
        }
        d[q] = gru_cell_bwd(dh[q], dh_rec[q], sv[q], hp[q], db[q]);
        if (step + 1 < T) gru_store_xchg(p, step, row, dir, ju, d[q]);
      }
      if (step + 1 < T) gru_publish(p, ctr, step, any, false);
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int row = rsub + q * RPT;
        if (row < Bp) gru_store_bwd(p, (long long)t * Bp + row, dir, ju, d[q]);
      }
      if (tid == 0) GRU_STAMP(10);
    }
    // ---- bias gradients: the warp's rows share its 8 units; reduce over the CTA ----
    epi_barrier();
    float* red = s.scratch;   // [4][U]: r z n hn
    for (int i = tid; i < 4 * U; i += GRU_EPI) red[i] = 0.f;
    epi_barrier();
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
      const bool active = rsub + q * RPT < Bp;
#pragma unroll
      for (int jj = 0; jj < GRU_UPT; ++jj) {
        const float a = warp_sum(active ? db[q].r[jj] : 0.f);
        const float b = warp_sum(active ? db[q].z[jj] : 0.f);
        const float c = warp_sum(active ? db[q].n[jj] : 0.f);
        const float d = warp_sum(active ? db[q].hn[jj] : 0.f);
        if (lane == 0) {
          atomicAdd(&red[uo + jj], a);
          atomicAdd(&red[U + uo + jj], b);
          atomicAdd(&red[2 * U + uo + jj], c);
          atomicAdd(&red[3 * U + uo + jj], d);
        }
      }
    }
    epi_barrier();
    if (tid < 3 * U) {
      const int g = tid / U, jj = tid % U;
      const int idx = dir * K3 + g * H + j0 + jj;
      atomicAdd(p.dbih + idx, red[tid]);
      atomicAdd(p.dbhh + idx, g < 2 ? red[tid] : red[3 * U + jj]);
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
// which forward recurrence kernel the last sb_gru_fwd launched (sb_debug_gru_fwd_kernel)
enum { GRU_FWD_NONE, GRU_FWD_PLAIN, GRU_FWD_KT, GRU_FWD_KS4, GRU_FWD_KS2, GRU_FWD_WIDE };
static int g_gru_last_fwd = GRU_FWD_NONE;
static int gru_fwd_launched(int kind) {
  g_gru_last_fwd = kind;
  return SB_OK;
}

static int gru_cluster_size(int nC) {
  int cs = g_gru_cluster;
  while (cs > 1 && (nC % cs) != 0) cs >>= 1;
  return cs < 1 ? 1 : cs;
}

// Launch configuration of a recurrence kernel: `grid` CTAs in clusters of cs.  Cooperative:
// attrs = {cooperative, cluster}; otherwise attrs = {cluster}.
static cudaLaunchConfig_t gru_launch_config(int grid, int cs, bool cooperative, size_t smem,
                                            cudaStream_t stream, cudaLaunchAttribute (&attrs)[2]) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GRU_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  int n = 0;
  if (cooperative) {
    attrs[n].id = cudaLaunchAttributeCooperative;
    attrs[n++].val.cooperative = 1;
  }
  attrs[n].id = cudaLaunchAttributeClusterDimension;
  attrs[n].val.clusterDim.x = cs;
  attrs[n].val.clusterDim.y = 1;
  attrs[n].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = n + 1;
  return cfg;
}

// cooperative launch over clusters of at most cs CTAs
static int gru_launch(const void* kernel, int grid, int cs, size_t smem, void** args,
                      cudaStream_t stream) {
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return SB_ERR_CUDA;
  cudaLaunchAttribute attrs[2];
  cudaLaunchConfig_t cfg = gru_launch_config(grid, cs, true, smem, stream, attrs);
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
// directions (128 CTAs) never fit as one 4-CTA clustered K-split launch: the forward runs
// gru_fwd_ks_kernel<2> over 2-CTA clusters there and the backward gru_bwd_ks_kernel in its L2
// reduce-scatter mode, both directions in one launch each.  Measured on an H100 80GB HBM3 (400 W
// power limit), recurrence kernel alone, us per step at T = 247, ONE direction of H = 1024
// (kt | ks): forward 4.12 | 4.17 at 8 rows, 4.59 | 4.34 at 16, 7.73 | 5.46 at 32, 14.68 | 8.38 at
// 64; backward 3.17 | 4.28 at 8, 4.08 | 4.37 at 16, 6.09 | 5.12 at 32, 8.15 | 7.94 at 64.  Both
// directions: forward 6.54 at 32 rows / 11.11 at 64 with gru_fwd_kernel against 5.10 / 7.50 with
// gru_fwd_ks_kernel<2> (tools/gru_fwd_ks2_bench.py, alternated); backward 23.4 at 64 rows with
// gru_bwd_kernel, and with gru_bwd_ks_kernel 7.29 at 32 rows / 10.25 at 64 in the L2 mode
// against 10.16 / 15.50 as two one-direction clustered launches (tools/gru_l2rs_bench.py).
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
  // Clustered launches are NOT flagged cooperative: co-residency of the whole grid is established
  // by the occupancy query below (1 CTA per SM, grid <= resident capacity), every spin-wait in
  // the kernels is bounded, and Nsight Compute cannot replay cooperative+cluster launches.
  cudaLaunchAttribute attrs[2];
  const cudaLaunchConfig_t cfg = gru_launch_config(grid, cs, false, smem, stream, attrs);
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

// ---- wide kernels: plan, selection, launch -----------------------------------------------------
enum { GRU_BWD_NONE, GRU_BWD_PLAIN, GRU_BWD_KT, GRU_BWD_KS4, GRU_BWD_KS_L2, GRU_BWD_KS4_X2,
       GRU_BWD_WIDE };
static int g_gru_last_bwd = GRU_BWD_NONE;
static int gru_bwd_launched(int kind) {
  g_gru_last_bwd = kind;
  return SB_OK;
}
// [pass][units per CTA, resident K chunks, streamed K chunks] of the last launch; zeros unless it
// ran a wide kernel
static int g_gru_last_plan[2][3];

struct GruWidePlan {
  int U, gc, ngroups, ring, rg, wr;
  size_t smem;
};

// Bytes of the wide kernels' gather ring (developer knob sb_debug_gru_wide_ring; the default was
// chosen by tools/gru_wide_bench.py --ring-sweep, see the comment of gru_fwd_wide_kernel).
static int g_gru_wide_gather_kb = GRU_WIDE_GATHER_KB;

// Shared memory of one wide pass over nchunks K chunks of nw weight rows.  Groups of gc = 2
// chunks where 2 divides nchunks; the gather ring holds g_gru_wide_gather_kb, at least 2 and at
// most GRU_MAX_RING slots (the MMA warpgroup holds two while one group is in flight); the rest
// holds as many resident groups as fit next to a weight ring of 2 slots, or every group.
// no_resident (GRU_FORCE_STREAM): rg = 0.
static bool gru_wide_layout(int Bp, int U, int nchunks, int nw, bool no_resident, GruWidePlan* w) {
  const int budget = 227 * 1024;
  w->U = U;
  w->gc = nchunks % 2 == 0 ? 2 : 1;
  w->ngroups = nchunks / w->gc;
  const int gslot = w->gc * Bp * 128, wslot = w->gc * nw * 128;
  const int fixed = 1024 /*align*/ + (2 * GRU_MAX_RING + 2 * GRU_WIDE_MAX_WR + 2) * 8 +
                    4 * U * 4 + Bp * (nw + 4) * 4;
  w->ring = std::min(std::max(g_gru_wide_gather_kb * 1024 / gslot, 2), GRU_MAX_RING);
  const int avail = budget - fixed - w->ring * gslot;
  if (!no_resident && avail >= w->ngroups * wslot) {
    w->rg = w->ngroups;
    w->wr = 0;
  } else {
    w->rg = no_resident ? 0 : std::min(w->ngroups - 1, std::max(0, avail / wslot - 2));
    w->wr = std::min(std::min(w->ngroups - w->rg, GRU_WIDE_MAX_WR), (avail - w->rg * wslot) / wslot);
    if (w->wr < std::min(w->ngroups - w->rg, 2)) return false;
  }
  w->smem = (size_t)fixed + (size_t)w->ring * gslot + gru_wide_wbytes(w->rg, w->wr, wslot, Bp);
  return w->smem <= (size_t)budget;
}

// Wide plan of one pass at width H: U = the smallest of 16, 32 that divides H, puts the grid of
// ndir * H / U CTAs on the SMs and whose shared memory fits.  Arithmetic only (workspace queries).
static bool gru_wide_plan(int Bp, int H, int ndir, bool backward, bool no_resident,
                          GruWidePlan* w) {
  if (Bp <= 0 || Bp % 8 != 0 || Bp > 128 || H <= 0 || (ndir != 1 && ndir != 2)) return false;
  for (int U = 16; U <= 32; U += 16) {
    if (H % U != 0 || ndir * (H / U) > sb::device_sm_count()) continue;
    const int nchunks = backward ? (3 * H + 63) / 64 : (H + 63) / 64;
    if (gru_wide_layout(Bp, U, nchunks, backward ? U : 3 * U, no_resident, w)) return true;
  }
  return false;
}

static const void* gru_wide_kernel_fn(const GruWidePlan& w, int Bp, bool backward,
                                      bool h0 = false) {
  if (h0)
    return w.U == 16 ? (const void*)gru_fwd_wide_h0_kernel<16, 1>
           : Bp > 64 ? (const void*)gru_fwd_wide_h0_kernel<32, 2>
                     : (const void*)gru_fwd_wide_h0_kernel<32, 1>;
  if (backward)
    return w.U == 16 ? (const void*)gru_bwd_wide_kernel<16, 1>
           : Bp > 64 ? (const void*)gru_bwd_wide_kernel<32, 2>
                     : (const void*)gru_bwd_wide_kernel<32, 1>;
  return w.U == 16 ? (const void*)gru_fwd_wide_kernel<16, 1>
         : Bp > 64 ? (const void*)gru_fwd_wide_kernel<32, 2>
                   : (const void*)gru_fwd_wide_kernel<32, 1>;
}

static void gru_record_plan(int pass, const GruWidePlan* w) {
  g_gru_last_plan[pass][0] = w ? w->U : 0;
  g_gru_last_plan[pass][1] = w ? w->rg * w->gc : 0;
  g_gru_last_plan[pass][2] = w ? (w->ngroups - w->rg) * w->gc : 0;
}

}  // namespace sb

using namespace sb;

// developer hooks (not part of the drop-in surface)
extern "C" int sb_debug_gru_timeline(void* dev_buffer) {
  sb::g_gru_dbg = reinterpret_cast<unsigned long long*>(dev_buffer);
  return SB_OK;
}
// developer knobs: 1 / 2: the recurrence kernels without the proxy fence / the off-path stores
// (timing only: results become wrong; see gru_publish, gru_store_fwd); 8 / 16: never / always
// use the transposed-accumulator K-split kernels (default: by batch size, see gru_use_kt); 32:
// disable the K-split forward kernels;
// 64 / 128: polling mode of the grid barrier in the K-split kernels (see grid_wait);
// 256 / 512: always (wherever the K-split backward kernel applies) / never use its L2
// reduce-scatter mode (see ks_exchange and sb_gru_bwd); 1024: the K-split forward over 2-CTA
// clusters wherever it applies (H % 128 == 0, batch rows <= 64), skipping the 4-CTA ones;
// 2048: the wide kernels with no resident weight chunks wherever they apply (tests the stream)
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
// which forward recurrence kernel the last sb_gru_fwd launched: "plain" (gru_fwd_kernel), "kt"
// (gru_fwd_kt_kernel), "ks4" / "ks2" (gru_fwd_ks_kernel<4> / <2>), "wide" (gru_fwd_wide_kernel);
// "none" before the first
extern "C" const char* sb_debug_gru_fwd_kernel(void) {
  static const char* const names[] = {"none", "plain", "kt", "ks4", "ks2", "wide"};
  return names[sb::g_gru_last_fwd];
}
// which backward recurrence kernel the last sb_gru_bwd launched: "plain" (gru_bwd_kernel), "kt"
// (gru_bwd_kt_kernel), "ks4" (gru_bwd_ks_kernel over 4-CTA clusters), "ks_l2" (its L2
// reduce-scatter mode), "ks4_x2" (one clustered launch per direction), "wide"
// (gru_bwd_wide_kernel); "none" before the first
extern "C" const char* sb_debug_gru_bwd_kernel(void) {
  static const char* const names[] = {"none", "plain", "kt", "ks4", "ks_l2", "ks4_x2", "wide"};
  return names[sb::g_gru_last_bwd];
}
// plan of the last sb_gru_fwd (backward = 0) / sb_gru_bwd (1) launch: out[0] units per CTA,
// out[1] resident and out[2] streamed W_hh chunks of 64 per CTA; all 0 unless it was "wide"
extern "C" int sb_debug_gru_plan(int backward, int* out) {
  if (!out || (backward != 0 && backward != 1)) return SB_ERR_INVALID;
  for (int i = 0; i < 3; ++i) out[i] = sb::g_gru_last_plan[backward][i];
  return SB_OK;
}

// developer knob: gather-ring bytes / 1024 of the wide kernels (> 0 sets; returns the value in use)
extern "C" int sb_debug_gru_wide_ring(int kb) {
  if (kb > 0) sb::g_gru_wide_gather_kb = kb;
  return sb::g_gru_wide_gather_kb;
}

static int gru_check_shape(int T, int Bp, int H, int ndir) {
  if (T <= 0 || Bp <= 0 || H <= 0 || (ndir != 1 && ndir != 2)) return SB_ERR_INVALID;
  if (H % GRU_HC != 0 || Bp % 8 != 0 || Bp > 128) return SB_ERR_UNSUPPORTED;
  return SB_OK;
}
// the resident kernels: one CTA of 16 units per SM
static int gru_check(int T, int Bp, int H, int ndir) {
  const int rc = gru_check_shape(T, Bp, H, ndir);
  if (rc != SB_OK) return rc;
  if (ndir * (H / GRU_HC) > sb::device_sm_count()) return SB_ERR_UNSUPPORTED;
  return SB_OK;
}

// Shared-memory ring of the plain (every-shape) kernels, forward and backward: -1 if the weight
// slice leaves no room for one slot.  sb_gru_fwd / sb_gru_bwd launch with exactly these values.
static int gru_fwd_ring(int Bp, int H, int* gc, size_t* smem) {
  const int nchunks = (H + 63) / 64;
  return gru_ring_slots(std::max(nchunks * 48 * 128, 16384 - Bp * 128), Bp, nchunks, 48, gc, smem);
}
static int gru_bwd_ring(int Bp, int H, int* gc, size_t* smem) {
  const int nchunks = (3 * H + 63) / 64;
  return gru_ring_slots(std::max(nchunks * 16 * 128, 16384 - Bp * 128), Bp, nchunks, 16, gc, smem);
}

// whether `grid` CTAs of `kernel` with `smem` bytes fit on the device at once (the cluster-size-1
// launch gru_launch falls back to; the preferred clustered kernels fall back to it in turn)
static bool gru_coresident(const void* kernel, int grid, size_t smem) {
  int per_sm = 0;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
          cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, GRU_THREADS, smem) !=
          cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return per_sm * sb::device_sm_count() >= grid;
}

// Whether a pass runs the wide kernel at width H (and its plan): where the resident kernels do
// not take the width (more CTAs of 16 units than SMs, or no ring next to the weight slice), or
// everywhere the wide kernel applies under the developer flag GRU_FORCE_STREAM.  Arithmetic only.
static bool gru_selects_wide(int Bp, int H, int ndir, bool backward, GruWidePlan* w) {
  const bool force = (g_gru_ablate & GRU_FORCE_STREAM) != 0;
  int gc = 1;
  size_t smem = 0;
  const bool resident = ndir * (H / GRU_HC) <= sb::device_sm_count() &&
                        (backward ? gru_bwd_ring(Bp, H, &gc, &smem) : gru_fwd_ring(Bp, H, &gc, &smem)) >= 0;
  return (force || !resident) && gru_wide_plan(Bp, H, ndir, backward, force, w);
}

// Width the recurrence kernels run a layer of H hidden units at.  First H rounded up to whole CTAs
// of GRU_HC units, provided both passes accept that width with the resident kernels: gru_check,
// the rings of the plain forward and backward kernels (the kernels every such shape falls back
// to) and their co-residency.  Otherwise the wide kernels' width: H rounded up to whole CTAs of
// U = 16 or 32 units (the smallest whose grid fits on the SMs), provided both wide passes fit in
// shared memory and are co-resident.  The caller pads the layer with zero units; such a unit stays
// exactly 0 (h_t = sigmoid(0) * h_{t-1} = 0) and its zero W_hh columns never reach a real unit.
extern "C" int sb_gru_plan(int Bp, int H, int ndir, int* Hp) {
  if (!Hp || H <= 0) return SB_ERR_INVALID;
  const int hp = (H + GRU_HC - 1) / GRU_HC * GRU_HC;
  const int rc = gru_check_shape(1, Bp, hp, ndir);
  if (rc != SB_OK) return rc;
  if (gru_check(1, Bp, hp, ndir) == SB_OK) {
    int gc = 1;
    size_t fsmem = 0, bsmem = 0;
    const int grid = ndir * (hp / GRU_HC);
    if (gru_fwd_ring(Bp, hp, &gc, &fsmem) >= 0 && gru_bwd_ring(Bp, hp, &gc, &bsmem) >= 0 &&
        gru_coresident((const void*)gru_fwd_kernel, grid, fsmem) &&
        gru_coresident((const void*)gru_bwd_kernel, grid, bsmem)) {
      *Hp = hp;
      return SB_OK;
    }
  }
  // each pass at hw: the kernel it will launch (wide, or resident where that pass still fits)
  // must be co-resident with its exact grid and shared memory
  auto pass_fits = [&](int hw, bool backward, int U) {
    GruWidePlan w;
    if (gru_selects_wide(Bp, hw, ndir, backward, &w))
      return w.U == U && gru_coresident(gru_wide_kernel_fn(w, Bp, backward), ndir * (hw / U), w.smem);
    int gc = 1;
    size_t smem = 0;
    if ((backward ? gru_bwd_ring(Bp, hw, &gc, &smem) : gru_fwd_ring(Bp, hw, &gc, &smem)) < 0 ||
        ndir * (hw / GRU_HC) > sb::device_sm_count())
      return false;
    return gru_coresident(backward ? (const void*)gru_bwd_kernel : (const void*)gru_fwd_kernel,
                          ndir * (hw / GRU_HC), smem);
  };
  for (int U = 16; U <= 32; U += 16) {
    const int hw = (H + U - 1) / U * U;
    if (pass_fits(hw, false, U) && pass_fits(hw, true, U)) {
      *Hp = hw;
      return SB_OK;
    }
  }
  return SB_ERR_UNSUPPORTED;
}

// workspace of one recurrence launch: [0,1024) the per-direction grid-barrier words (one L2 line
// each), then the exchange buffers of the backward kernels
static constexpr size_t GRU_WS_COUNTERS = 1024;

// The L2 reduce-scatter of the K-split backward kernel (ks_exchange), at the END of its
// workspace: one counter line per direction and group of 4 CTAs, then the staging area, two
// parities of [dst][src] slices of Bp x 16 floats.  Nothing outside the K-split domain.  Only the
// counters need zeroing: every slice is written before it is read.
static size_t gru_rs_groups(int H, int ndir) {
  return H % (KS * 64) == 0 ? (size_t)ndir * (H / (KS * GRU_HC)) : 0;
}
static size_t gru_rs_bytes(int Bp, int H, int ndir, size_t* zeroed) {
  *zeroed = gru_rs_groups(H, ndir) * 128;
  return *zeroed + gru_rs_groups(H, ndir) * 2 * KS * KS * (size_t)Bp * GRU_HC * sizeof(float);
}

// Dynamic shared memory of gru_fwd_ks_kernel<ks>: the K slice of h_{t-1} and of the weights,
// recv + stage ([ks][Bp][48] fp32 each), barriers and bias, alignment.
static size_t gru_fwd_ks_smem(int ks, int Bp, int H) {
  const size_t nq = (size_t)H / ks / 64;
  return nq * Bp * 128 + nq * (3 * ks * GRU_HC) * 128 + (size_t)2 * ks * Bp * 3 * GRU_HC * 4 +
         1024 + 512;
}
// gru_fwd_kt_kernel: the K quarter of h_{t-1} and of the 192 weight rows, recv + stage
// ([4 + 3][48][Bp + 4] fp32), barriers and bias, alignment.
static size_t gru_fwd_kt_smem(int Bp, int H) {
  const size_t nq = (size_t)H / KS / 64;
  return nq * Bp * 128 + nq * (3 * KS * GRU_HC) * 128 +
         (size_t)(2 * KS - 1) * 3 * GRU_HC * (Bp + 4) * 4 + 1024 + 512;
}
// gru_bwd_ks_kernel: the K quarter of dgh_t (3H / 4 columns) and of the 64 weight rows, recv +
// stage ([4][Bp][16] fp32 each), barriers, alignment.
static size_t gru_bwd_ks_smem(int Bp, int H) {
  const size_t nq = (size_t)3 * H / KS / 64;
  return nq * Bp * 128 + nq * (KS * GRU_HC) * 128 + (size_t)2 * KS * Bp * GRU_HC * 4 + 1024 + 256;
}
// gru_bwd_kt_kernel: as gru_bwd_ks_kernel, with recv + stage [4 + 3][16][Bp + 4] fp32.
static size_t gru_bwd_kt_smem(int Bp, int H) {
  const size_t nq = (size_t)3 * H / KS / 64;
  return nq * Bp * 128 + nq * (KS * GRU_HC) * 128 + (size_t)(2 * KS - 1) * GRU_HC * (Bp + 4) * 4 +
         1024 + 256;
}

// The two per-direction tensor maps of a gathered operand (boxes of Bp rows): direction d's
// [rows x cols] matrix (pitch ld) starts d * dir_stride elements after `base`; a one-direction
// layer maps direction 0 twice.
static int gru_dir_tmaps(CUtensorMap* tm, const bf16* base, size_t dir_stride, long long rows,
                         long long cols, long long ld, int ndir, int Bp) {
  for (int d = 0; d < 2; ++d) {
    const int rc = make_tmap_bf16_2d(&tm[d], base + (d < ndir ? d : 0) * dir_stride, rows, cols,
                                     ld, Bp);
    if (rc != SB_OK) return rc;
  }
  return SB_OK;
}

extern "C" int sb_gru_fwd_workspace_size(int Bp, int H, int ndir, size_t* bytes) {
  if (!bytes || Bp <= 0 || H <= 0 || (ndir != 1 && ndir != 2)) return SB_ERR_INVALID;
  *bytes = GRU_WS_COUNTERS;      // the forward kernels exchange h_t through xn itself
  return SB_OK;
}

// sb_gru_fwd, and with h0 (non-null) its resumed form sb_gru_fwd_h0, whose launch has T + 1 steps:
// step 0 publishes h0, copied to frame 0 of y and xn.  The kernel selection depends on (Bp, H,
// ndir) alone, so both forms of a shape run the same kernel.
static int gru_fwd_entry(const float* gi, const void* whh_bf16, const float* bhh, const float* h0f,
                         const void* h0_bf16, float* y, void* xn_bf16, float* gates,
                         void* workspace, size_t workspace_bytes, int T, int Bp, int H, int ndir,
                         void* stream_) {
  const bool h0 = h0f != nullptr;
  GruWidePlan w;
  const bool wide = gru_check_shape(T, Bp, H, ndir) == SB_OK &&
                    gru_selects_wide(Bp, H, ndir, false, &w);
  int rc = wide ? SB_OK : gru_check(T, Bp, H, ndir);
  if (rc != SB_OK) return rc;
  if (!gi || !whh_bf16 || !bhh || !y || !xn_bf16 || !workspace) return SB_ERR_INVALID;
  size_t need = 0;
  sb_gru_fwd_workspace_size(Bp, H, ndir, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  if ((reinterpret_cast<uintptr_t>(workspace) & 1023) != 0) return SB_ERR_INVALID;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int nC = H / GRU_HC;
  if (cudaMemsetAsync(workspace, 0, need, stream) != cudaSuccess) return SB_ERR_CUDA;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  unsigned int* barrier = reinterpret_cast<unsigned int*>(ws);
  gru_record_plan(0, nullptr);
  if (h0) {
    const size_t n = (size_t)Bp * H;
    if ((static_cast<const void*>(h0f) != y &&
         cudaMemcpyAsync(y, h0f, n * sizeof(float), cudaMemcpyDeviceToDevice, stream) !=
             cudaSuccess) ||
        (h0_bf16 != xn_bf16 && cudaMemcpyAsync(xn_bf16, h0_bf16, n * sizeof(bf16),
                                               cudaMemcpyDeviceToDevice, stream) != cudaSuccess))
      return SB_ERR_CUDA;
    ++T;
  }

  // ---- wide layers: U units per CTA, W_hh partly streamed from L2 (gru_fwd_wide_kernel) ----
  if (wide) {
    GruFwdParams p;
    memset(&p, 0, sizeof(p));
    p.gi = gi; p.whh = reinterpret_cast<const bf16*>(whh_bf16); p.bhh = bhh; p.y = y;
    p.xn = reinterpret_cast<bf16*>(xn_bf16); p.gates = gates; p.barrier = barrier;
    p.T = T; p.Bp = Bp; p.H = H; p.ndir = ndir; p.dbg = g_gru_dbg; p.ablate = g_gru_ablate & 3;
    p.ring = w.ring; p.gc = w.gc; p.rg = w.rg; p.wr = w.wr;
    CUtensorMap tm[3];
    rc = gru_dir_tmaps(tm, p.xn, H, (long long)T * Bp, H, (long long)ndir * H, ndir, Bp);
    if (rc != SB_OK) return rc;
    rc = make_tmap_bf16_2d(&tm[2], p.whh, (long long)ndir * 3 * H, H, H, w.U);
    if (rc != SB_OK) return rc;
    void* args[] = {(void*)&tm[0], (void*)&tm[1], (void*)&tm[2], (void*)&p};
    const int nCw = H / w.U;
    rc = gru_launch(gru_wide_kernel_fn(w, Bp, false, h0), ndir * nCw, gru_cluster_size(nCw),
                    w.smem, args, stream);
    if (rc != SB_OK) return rc;
    gru_record_plan(0, &w);
    return gru_fwd_launched(GRU_FWD_WIDE);
  }

  int gc = 1;
  size_t smem = 0;
  const int ring = gru_fwd_ring(Bp, H, &gc, &smem);
  if (ring < 0) return SB_ERR_UNSUPPORTED;

  // ---- preferred: K-split over clusters of KS CTAs (H % (KS * 64) == 0, batch rows <= 64) ----
  // Tried in this order, each where its grid of 1-CTA-per-SM clusters is co-resident: the
  // transposed-accumulator flavour (small batches, see gru_use_kt) and gru_fwd_ks_kernel<4> over
  // 4-CTA clusters, then gru_fwd_ks_kernel<2> over 2-CTA clusters from H = 512 up (both
  // directions of H = 1024 on a 132-SM H100: 128 CTAs fit as 2-CTA clusters, not as 4-CTA ones).
  // Developer knobs: 32 disables all of them, 1024 skips straight to KS = 2 at any width.
  if (!(g_gru_ablate & 32) && H % 128 == 0 && Bp <= 64) {
    GruFwdParams q;
    q.gi = gi; q.whh = reinterpret_cast<const bf16*>(whh_bf16); q.bhh = bhh; q.y = y;
    q.xn = reinterpret_cast<bf16*>(xn_bf16); q.gates = gates;
    q.barrier = barrier; q.T = T; q.Bp = Bp; q.H = H; q.ndir = ndir;
    q.dbg = g_gru_dbg; q.ablate = g_gru_ablate & 195; q.gc = 1;
    CUtensorMap tq[2];
    rc = gru_dir_tmaps(tq, q.xn, H, (long long)T * Bp, H, (long long)ndir * H, ndir, Bp);
    if (rc != SB_OK) return rc;
    void* kargs[] = {(void*)&tq[0], (void*)&tq[1], (void*)&q};   // q is copied at launch
    if (!(g_gru_ablate & 1024) && H % 256 == 0) {
      const size_t ks_smem = gru_fwd_ks_smem(KS, Bp, H);   // KS = 4
      q.ring = H / KS / 64;
      if (ks_smem <= 227 * 1024) {
        const size_t kt_smem = gru_fwd_kt_smem(Bp, H);
        if (gru_use_kt(Bp, false) && kt_smem <= 227 * 1024) {
          const void* kt = h0 ? (Bp > 32   ? (const void*)gru_fwd_kt_h0_kernel<4>
                                 : Bp > 16 ? (const void*)gru_fwd_kt_h0_kernel<2>
                                           : (const void*)gru_fwd_kt_h0_kernel<1>)
                              : (Bp > 32   ? (const void*)gru_fwd_kt_kernel<4>
                                 : Bp > 16 ? (const void*)gru_fwd_kt_kernel<2>
                                           : (const void*)gru_fwd_kt_kernel<1>);
          rc = gru_launch_exact(kt, ndir * nC, KS, kt_smem, kargs, stream);
          if (rc == SB_OK) return gru_fwd_launched(GRU_FWD_KT);
        }
        rc = gru_launch_exact(h0 ? (const void*)gru_fwd_ks_h0_kernel<KS>
                                 : (const void*)gru_fwd_ks_kernel<KS>,
                              ndir * nC, KS, ks_smem, kargs, stream);
        if (rc == SB_OK) return gru_fwd_launched(GRU_FWD_KS4);
      }
    }
    // KS = 2 by default only from H = 512 up: below, the exchange costs more than halving the
    // gather saves.  H100 80GB HBM3 at 400 W, T = 247, us per step, gru_fwd_kernel | KS = 2 at 64
    // rows: H = 128 one direction 3.86 | 4.24, both directions H = 384 4.80 | 5.11, H = 640
    // 6.44 | 5.74, H = 896 8.90 | 6.88, H = 1024 11.07 | 7.49 (tools/gru_fwd_ks2_bench.py).
    const size_t ks2_smem = gru_fwd_ks_smem(2, Bp, H);
    if (ks2_smem <= 227 * 1024 && (H >= 512 || (g_gru_ablate & 1024))) {
      q.ring = H / 2 / 64;
      rc = gru_launch_exact(h0 ? (const void*)gru_fwd_ks_h0_kernel<2>
                               : (const void*)gru_fwd_ks_kernel<2>,
                            ndir * nC, 2, ks2_smem, kargs, stream);
      if (rc == SB_OK) return gru_fwd_launched(GRU_FWD_KS2);
    }
  }

  // ---- every other shape: each CTA gathers all of h_{t-1} (tensor-map TMA, cluster multicast) ----
  GruFwdParams p;
  p.gi = gi; p.whh = reinterpret_cast<const bf16*>(whh_bf16); p.bhh = bhh; p.y = y;
  p.xn = reinterpret_cast<bf16*>(xn_bf16);
  p.gates = gates; p.barrier = barrier; p.T = T; p.Bp = Bp; p.H = H; p.ndir = ndir;
  p.dbg = g_gru_dbg;
  p.ablate = g_gru_ablate & 31;
  p.ring = ring; p.gc = gc;
  CUtensorMap tm[2];
  rc = gru_dir_tmaps(tm, p.xn, H, (long long)T * Bp, H, (long long)ndir * H, ndir, Bp);
  if (rc != SB_OK) return rc;
  void* args[] = {(void*)&tm[0], (void*)&tm[1], (void*)&p};
  rc = gru_launch(h0 ? (const void*)gru_fwd_h0_kernel : (const void*)gru_fwd_kernel, ndir * nC,
                  gru_cluster_size(nC), smem, args, stream);
  return rc == SB_OK ? gru_fwd_launched(GRU_FWD_PLAIN) : rc;
}

extern "C" int sb_gru_fwd(const float* gi, const void* whh_bf16, const float* bhh, float* y,
                          void* xn_bf16, float* gates, void* workspace, size_t workspace_bytes,
                          int T, int Bp, int H, int ndir, void* stream) {
  return gru_fwd_entry(gi, whh_bf16, bhh, nullptr, nullptr, y, xn_bf16, gates, workspace,
                       workspace_bytes, T, Bp, H, ndir, stream);
}

extern "C" int sb_gru_fwd_h0(const float* gi, const void* whh_bf16, const float* bhh,
                             const float* h0, const void* h0_bf16, float* y, void* xn_bf16,
                             float* gates, void* workspace, size_t workspace_bytes, int T, int Bp,
                             int H, int ndir, void* stream) {
  if (ndir == 2) return SB_ERR_UNSUPPORTED;
  if (!h0 || !h0_bf16) return SB_ERR_INVALID;
  return gru_fwd_entry(gi, whh_bf16, bhh, h0, h0_bf16, y, xn_bf16, gates, workspace,
                       workspace_bytes, T, Bp, H, ndir, stream);
}

// counters + the double-buffered exchange of dgh_t (Bp x 3H bf16 per direction and parity; the
// tile-major form of the K-split kernel rounds 3H up to whole 64-column chunks) + the L2
// reduce-scatter area; the wide kernel's W_hh^T ([ndir][H][3H] bf16) follows at this offset
static size_t gru_bwd_ws_base(int Bp, int H, int ndir) {
  const size_t k3p = (size_t)((3 * H + 63) / 64) * 64;
  size_t z = 0;
  return GRU_WS_COUNTERS + (size_t)ndir * 2 * Bp * k3p * sizeof(bf16) + 1024 +
         gru_rs_bytes(Bp, H, ndir, &z);
}

extern "C" int sb_gru_bwd_workspace_size(int Bp, int H, int ndir, size_t* bytes) {
  if (!bytes || Bp <= 0 || H <= 0 || (ndir != 1 && ndir != 2)) return SB_ERR_INVALID;
  *bytes = gru_bwd_ws_base(Bp, H, ndir);
  GruWidePlan w;
  if (gru_check_shape(1, Bp, H, ndir) == SB_OK && gru_selects_wide(Bp, H, ndir, true, &w))
    *bytes = (*bytes + 1023) / 1024 * 1024 + (size_t)ndir * 3 * H * H * sizeof(bf16);
  return SB_OK;
}

extern "C" int sb_gru_bwd(const float* dy, const float* y, const float* gates,
                          const void* whh_bf16, void* dgi_bf16, void* dghn_bf16, float* dbih,
                          float* dbhh, void* workspace, size_t workspace_bytes, int T, int Bp,
                          int H, int ndir, void* stream_) {
  GruWidePlan w;
  const bool wide = gru_check_shape(T, Bp, H, ndir) == SB_OK &&
                    gru_selects_wide(Bp, H, ndir, true, &w);
  int rc = wide ? SB_OK : gru_check(T, Bp, H, ndir);
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
  p.xchg = reinterpret_cast<bf16*>(ws + GRU_WS_COUNTERS);
  p.dbih = dbih; p.dbhh = dbhh; p.T = T; p.Bp = Bp; p.H = H; p.ndir = ndir;
  p.dbg = g_gru_dbg;
  p.dir0 = 0;
  p.ablate = g_gru_ablate & 195;
  const int K3 = 3 * H;
  size_t smem = 0;
  const int nC_ = H / GRU_HC;
  size_t rs_zeroed = 0;
  const size_t rs_at = gru_bwd_ws_base(Bp, H, ndir) - gru_rs_bytes(Bp, H, ndir, &rs_zeroed);
  p.rsctr = reinterpret_cast<unsigned int*>(ws + rs_at);
  p.rs = reinterpret_cast<float*>(ws + rs_at + rs_zeroed);
  // counters and barrier words start at zero; the exchange tiles too (columns past 3H of a
  // partial chunk are never written and must read as zero)
  if (cudaMemsetAsync(workspace, 0, rs_at + rs_zeroed, stream) != cudaSuccess) return SB_ERR_CUDA;
  gru_record_plan(1, nullptr);

  // ---- wide layers: U units per CTA, W_hh^T partly streamed from L2 (gru_bwd_wide_kernel) ----
  if (wide) {
    p.whhT = reinterpret_cast<bf16*>(ws + (gru_bwd_ws_base(Bp, H, ndir) + 1023) / 1024 * 1024);
    p.ring = w.ring; p.gc = w.gc; p.rg = w.rg; p.wr = w.wr;
    CUtensorMap tm[3];
    rc = gru_dir_tmaps(tm, p.xchg, (size_t)2 * Bp * K3, 2LL * Bp, K3, K3, ndir, Bp);
    if (rc != SB_OK) return rc;
    rc = make_tmap_bf16_2d(&tm[2], p.whhT, (long long)ndir * H, K3, K3, w.U);
    if (rc != SB_OK) return rc;
    void* args[] = {(void*)&tm[0], (void*)&tm[1], (void*)&tm[2], (void*)&p};
    const int nCw = H / w.U;
    rc = gru_launch(gru_wide_kernel_fn(w, Bp, true), ndir * nCw, gru_cluster_size(nCw), w.smem,
                    args, stream);
    if (rc != SB_OK) return rc;
    gru_record_plan(1, &w);
    return gru_bwd_launched(GRU_BWD_WIDE);
  }
  // ---- preferred: K-split over 4-CTA clusters ----
  if (g_gru_ksplit && H % 256 == 0 && nC_ % KS == 0 && (K3 / KS / 64) <= 16) {
    const size_t ks_smem = gru_bwd_ks_smem(Bp, H);
    if (ks_smem <= 227 * 1024) {
      CUtensorMap tq[2];
      rc = gru_dir_tmaps(tq, p.xchg, (size_t)2 * Bp * K3, 2LL * Bp, K3, K3, ndir, Bp);
      if (rc != SB_OK) return rc;
      p.ring = K3 / KS / 64; p.gc = 1;
      void* kargs[] = {(void*)&tq[0], (void*)&tq[1], (void*)&p};
      const size_t kt_smem = gru_bwd_kt_smem(Bp, H);
      if (gru_use_kt(Bp, true) && !(g_gru_ablate & 256) && Bp <= 64 && kt_smem <= 227 * 1024) {
        const void* kt = Bp > 32   ? (const void*)gru_bwd_kt_kernel<4>
                         : Bp > 16 ? (const void*)gru_bwd_kt_kernel<2>
                                   : (const void*)gru_bwd_kt_kernel<1>;
        rc = gru_launch_exact(kt, ndir * nC_, KS, kt_smem, kargs, stream);
        if (rc == SB_OK) return gru_bwd_launched(GRU_BWD_KT);
      }
      // 1. both directions as 4-CTA clusters, reduce-scattering through DSMEM
      const void* ks = (const void*)gru_bwd_ks_kernel<false>;
      const void* ks_l2 = (const void*)gru_bwd_ks_kernel<true>;
      rc = SB_ERR_UNSUPPORTED;
      if (!(g_gru_ablate & 256)) {
        rc = gru_launch_exact(ks, ndir * nC_, KS, ks_smem, kargs, stream);
        if (rc == SB_OK) return gru_bwd_launched(GRU_BWD_KS4);
      }
      // 2. Both directions do not fit as 4-CTA clusters (an H100 holds 30 of them, 120 CTAs,
      // against 128 at H = 1024), but fit without a cluster, one CTA per SM: the same kernel
      // reduce-scattering through L2, both directions in one cooperative launch
      // (sb_debug_gru_cluster(0) then reports 1).  Developer knobs: 256 forces it wherever the
      // K-split domain holds, 512 disables it.
      if (rc == SB_ERR_UNSUPPORTED && !(g_gru_ablate & 512) &&
          gru_coresident(ks_l2, ndir * nC_, ks_smem)) {
        rc = gru_launch(ks_l2, ndir * nC_, 1, ks_smem, kargs, stream);
        if (rc == SB_OK) return gru_bwd_launched(GRU_BWD_KS_L2);
      }
      // 3. Neither fits (fewer SMs than CTAs, e.g. a 114-SM part): the directions one after the
      // other as clustered launches, each with its own barrier counter.  Still faster than the
      // plain kernel, whose every CTA gathers all of dgh_t.
      if (rc == SB_ERR_UNSUPPORTED && ndir == 2) {
        rc = gru_launch_exact(ks, nC_, KS, ks_smem, kargs, stream);
        if (rc == SB_OK) {
          p.dir0 = 1;   // kernel parameters are copied at launch
          rc = gru_launch_exact(ks, nC_, KS, ks_smem, kargs, stream);
          return rc == SB_OK ? gru_bwd_launched(GRU_BWD_KS4_X2) : rc;
        }
      }
    }
  }
  p.ring = gru_bwd_ring(Bp, H, &p.gc, &smem);
  if (p.ring < 0) return SB_ERR_UNSUPPORTED;
  // per direction: the two parity buffers stacked as [2*Bp rows][3H cols]
  CUtensorMap tm[2];
  rc = gru_dir_tmaps(tm, p.xchg, (size_t)2 * Bp * K3, 2LL * Bp, K3, K3, ndir, Bp);
  if (rc != SB_OK) return rc;
  void* args[] = {(void*)&tm[0], (void*)&tm[1], (void*)&p};
  const int nC = H / GRU_HC;
  rc = gru_launch((const void*)gru_bwd_kernel, ndir * nC, gru_cluster_size(nC), smem, args,
                  stream);
  return rc == SB_OK ? gru_bwd_launched(GRU_BWD_PLAIN) : rc;
}
