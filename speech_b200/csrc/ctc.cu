// sb_ctc_fwd_bwd: CTC negative log-likelihood + gradient w.r.t. the UN-normalised activations.
//
// Replaces functions.ctc.CTCLoss (libs/warp-ctc binding; call site speech/models/ctc_model.py:34-40,
// un-vendored dependency Makefile:4-7).  Semantics: activations (B, T, V) batch-first raw logits,
// softmax is internal, blank index is a parameter (the reference uses the LAST class,
// ctc_model.py:18), labels are a flat int32 array, per-utterance costs are returned and the
// caller reduces them (sum over the minibatch by default).
//
// One CTA per utterance, 512 threads = two "sides" of 256:
//   side 0 runs the alpha recursion forward in time, side 1 runs the beta recursion backward in
//   time, CONCURRENTLY, so the serial dependency chain is T steps instead of 2T.  They meet in the
//   middle (t = T/2): log p(y|x) is formed there from alpha_t and beta_t, and each side then
//   continues into the half the other side already covered, fusing the gradient
//     dL/da[t,k] = softmax_t(k) - (1/p) * sum_{s: l'_s = k} alpha_t(s) beta_t(s) / softmax_t(k)
//   with its recursion.  Only half of each lattice is ever spilled (to an L2-resident workspace).
//   The (T x V) log-softmax of the utterance is staged ONCE in shared memory with coalesced
//   reads of the logits (116 KB at T=1000, V=29); lattice rows ping-pong in shared memory.
//
// Precision: the lattice recursion runs in float64 (see lse3d) and every row is stored relative to the maximum of the previous row (per-warp maxima are
// published before the step barrier, so this costs no extra synchronisation); the subtracted
// amounts accumulate in a per-side double.  fp32 log-space values therefore stay O(1) for any T
// and the 1e-4 parity bar holds for long utterances.
//
// Roofline: nominally HBM (read logits + write grads = 2*B*T*V*4 bytes), in practice bound by
// the T-step serial chain.
#include "common.cuh"
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int CTC_SIDE = 256;
#define CTC_NEG_INF (-INFINITY)

struct CtcParams {
  const float* acts;    // (B, T, V)
  float* grads;         // (B, T, V) or nullptr
  const int* labels;    // flat
  const int* label_off; // (B) exclusive prefix sum of label_lens
  const int* label_lens;
  const int* act_lens;
  float* costs;         // (B)
  float* ws;            // (B, T, S_stride) lattice spill (rows stored relative to offs)
  double* offs;         // (B, T) scalar offset of each spilled row
  int B, T, V, blank, S_stride;
};

SB_DEVINL float lse2(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == CTC_NEG_INF) return CTC_NEG_INF;
  return m + __logf(__expf(a - m) + __expf(b - m));
}
SB_DEVINL float lse3(float a, float b, float c) {
  // On the T-step chain exp and log must be the accurate ones: the fast intrinsics' ~1e-7 errors
  // are biased, differ between the alpha and beta recursions and accumulate linearly with T
  // (measured 1.4e-4 relative gradient error at the ends of a T=1000 utterance).
  const float m = fmaxf(fmaxf(a, b), c);
  if (m == CTC_NEG_INF) return CTC_NEG_INF;
  return m + logf(expf(a - m) + expf(b - m) + expf(c - m));
}

// log(exp(a)+exp(b)+exp(c)) in float64: the largest term contributes exp(0) = 1 exactly, so
// only the two smaller terms are exponentiated.  float32 here accumulates ~1e-4 relative
// gradient error over a T=1000 lattice (measured, and reproduced in numpy), float64 gives 2e-7.
SB_DEVINL double lse3d(double a, double b, double c) {
  const double hi = fmax(a, b), lo = fmin(a, b);
  const double m = fmax(hi, c);
  if (m == -INFINITY) return -INFINITY;
  const double o1 = (c > hi) ? hi : lo;
  const double o2 = (c > hi) ? lo : c;
  return m + log1p(exp(o1 - m) + exp(o2 - m));
}

SB_DEVINL void side_barrier(int side) {
  asm volatile("bar.sync %0, %1;" ::"r"(side + 1), "r"(CTC_SIDE) : "memory");
}

template <int NS, bool STAGED>
__global__ void __launch_bounds__(2 * CTC_SIDE, 1) ctc_fwd_bwd_kernel(const CtcParams p) {
  extern __shared__ double smem_d[];
  float* smem = reinterpret_cast<float*>(smem_d);
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int side = tid / CTC_SIDE;  // 0: alpha, 1: beta
  const int i = tid % CTC_SIDE;
  const int V = p.V;
  const int T = min(p.act_lens[b], p.T);
  const int L = p.label_lens[b];
  const int S = 2 * L + 1;
  const int* lab = p.labels + p.label_off[b];
  const float* acts = p.acts + (size_t)b * p.T * V;
  float* grads = p.grads ? p.grads + (size_t)b * p.T * V : nullptr;
  float* ws = p.ws + (size_t)b * p.T * p.S_stride;
  double* offs = p.offs + (size_t)b * p.T;

  // ---- shared memory carve-up ----
  constexpr int SP = NS * CTC_SIDE + 4;        // padded lattice row (2 pads each end)
  double* row_buf = reinterpret_cast<double*>(smem);   // [2 sides][2][SP]  float64 lattice rows
  float* occ = reinterpret_cast<float*>(row_buf + 4 * SP);  // [2 sides][2][V]
  float* red = occ + 4 * V;                     // [48] reduction scratch
  float* nred = red + 32;                       // [2 sides][2][8] per-warp row maxima
  float* lse_t = red + 64;                      // [T] (only !STAGED)
  float* lp = STAGED ? (red + 64) : nullptr;    // [T*V] (only STAGED)

  for (int k = tid; k < 4 * SP; k += 2 * CTC_SIDE) row_buf[k] = -INFINITY;
  for (int k = tid; k < 4 * V; k += 2 * CTC_SIDE) occ[k] = 0.f;

  // zero the gradient rows beyond this utterance's length
  if (grads) {
    for (int k = T * V + tid; k < p.T * V; k += 2 * CTC_SIDE) grads[k] = 0.f;
  }

  // ---- log-softmax of the whole utterance (coalesced read of the logits) ----
  const int warp = tid >> 5, lane = tid & 31;
  if (STAGED) {
    for (int k = tid; k < T * V; k += 2 * CTC_SIDE) lp[k] = __ldg(acts + k);
    __syncthreads();
    for (int t = warp; t < T; t += (2 * CTC_SIDE) / 32) {
      float m = CTC_NEG_INF;
      for (int k = lane; k < V; k += 32) m = fmaxf(m, lp[t * V + k]);
      m = warp_max(m);
      float s = 0.f;
      for (int k = lane; k < V; k += 32) s += __expf(lp[t * V + k] - m);
      s = warp_sum(s);
      const float lz = m + __logf(s);
      for (int k = lane; k < V; k += 32) lp[t * V + k] -= lz;
    }
  } else {
    for (int t = warp; t < T; t += (2 * CTC_SIDE) / 32) {
      float m = CTC_NEG_INF;
      for (int k = lane; k < V; k += 32) m = fmaxf(m, __ldg(acts + t * V + k));
      m = warp_max(m);
      float s = 0.f;
      for (int k = lane; k < V; k += 32) s += __expf(__ldg(acts + t * V + k) - m);
      s = warp_sum(s);
      if (lane == 0) lse_t[t] = m + __logf(s);
    }
  }
  __syncthreads();

  auto emit = [&](int t, int k) -> float {
    if (STAGED) return lp[t * V + k];
    return __ldg(acts + t * V + k) - lse_t[t];
  };

  // degenerate: no frames
  if (T <= 0) {
    if (tid == 0) p.costs[b] = (L == 0) ? 0.f : INFINITY;
    return;
  }

  // ---- per-thread lattice states: s = i + 256*q ----
  int cls[NS];      // class emitted in state s
  bool skip[NS];    // transition s-2 -> s allowed (alpha) ; for beta: s -> s+2 allowed
  bool valid[NS];
#pragma unroll
  for (int q = 0; q < NS; ++q) {
    const int s = i + CTC_SIDE * q;
    valid[q] = s < S;
    cls[q] = p.blank;
    skip[q] = false;
    if (valid[q] && (s & 1)) {
      const int li = (s - 1) >> 1;
      cls[q] = lab[li];
      if (side == 0) skip[q] = (li > 0) && (lab[li - 1] != cls[q]);
      else skip[q] = (li + 1 < L) && (lab[li + 1] != cls[q]);
    }
  }

  double* my_rows = row_buf + side * 2 * SP + 2;  // +2: leading pad so [s-2] is addressable
  float* my_occ = occ + side * 2 * V;
  float* my_nred = nred + side * 16;             // [2][8] warp maxima of the last two rows
  const int Th = T / 2;
  const int swarp = i >> 5;  // warp index inside the side
  double C = 0.0;            // offset of the newest row of this side: true value = stored + C

  // Row n of this side (time t) from row n-1 (smem ping-pong slot n&1).  The maximum of row n-1
  // (gathered from per-warp maxima published before the previous barrier) is subtracted, so
  // stored values stay O(1); the subtracted amounts accumulate in C (double).  One barrier per
  // row, issued by the caller.
  auto step_row = [&](int n, int t, double (&vals)[NS]) {
    double* cur = my_rows + (n & 1) * SP;
    const double* prev = my_rows + ((n & 1) ^ 1) * SP;
    float m_prev = 0.f;
    if (n > 0) {
      const float* w = my_nred + ((n - 1) & 1) * 8;
      m_prev = w[0];
#pragma unroll
      for (int k = 1; k < CTC_SIDE / 32; ++k) m_prev = fmaxf(m_prev, w[k]);
      if (m_prev == CTC_NEG_INF) m_prev = 0.f;
    }
    C += (double)m_prev;
    float wm = CTC_NEG_INF;
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int s = i + CTC_SIDE * q;
      double v = -INFINITY;
      if (valid[q]) {
        if (n == 0) {
          if (side == 0) { if (s <= 1) v = 0.0; }
          else { if (s >= S - 2) v = 0.0; }
        } else if (side == 0) {
          v = lse3d(prev[s], prev[s - 1], skip[q] ? prev[s - 2] : -INFINITY) - (double)m_prev;
        } else {
          v = lse3d(prev[s], prev[s + 1], skip[q] ? prev[s + 2] : -INFINITY) - (double)m_prev;
        }
        v += (double)emit(t, cls[q]);
        cur[s] = v;
        wm = fmaxf(wm, (float)v);
      }
      vals[q] = v;
    }
    wm = warp_max(wm);
    if (lane == 0) my_nred[(n & 1) * 8 + swarp] = wm;
  };

  // ------------------------------------------------------------------------------------------
  // phase 1: alpha rows [0, Th), beta rows [Th, T) ; each row is spilled to the workspace
  // ------------------------------------------------------------------------------------------
  {
    const int nsteps = side == 0 ? Th : (T - Th);
    for (int n = 0; n < nsteps; ++n) {
      const int t = side == 0 ? n : (T - 1 - n);
      double vals[NS];
      step_row(n, t, vals);
#pragma unroll
      for (int q = 0; q < NS; ++q)   // spilled once, consumed once: float32 is enough here
        if (valid[q]) ws[(size_t)t * p.S_stride + i + CTC_SIDE * q] = (float)vals[q];
      if (i == 0) offs[t] = C;
      side_barrier(side);
    }
  }
  __syncthreads();

  // ------------------------------------------------------------------------------------------
  // meet in the middle: alpha_Th (side 0) x beta_Th (spilled by side 1) -> log p(y|x)
  // ------------------------------------------------------------------------------------------
  double a_reg[NS];
  if (side == 0) {
    step_row(Th, Th, a_reg);
    float local_max = CTC_NEG_INF;
    float contrib[NS];
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int s = i + CTC_SIDE * q;
      contrib[q] = CTC_NEG_INF;
      if (valid[q]) {
        contrib[q] = (float)(a_reg[q] + (double)ld_cg_f(ws + (size_t)Th * p.S_stride + s) -
                             (double)emit(Th, cls[q]));
        local_max = fmaxf(local_max, contrib[q]);
      }
    }
    // block logsumexp over the 256 alpha-side threads
    float m = warp_max(local_max);
    if (lane == 0) red[warp] = m;
    side_barrier(0);
    m = red[0];
#pragma unroll
    for (int w = 1; w < CTC_SIDE / 32; ++w) m = fmaxf(m, red[w]);
    float sum = 0.f;
    if (m != CTC_NEG_INF) {
#pragma unroll
      for (int q = 0; q < NS; ++q) sum += __expf(contrib[q] - m);
    }
    sum = warp_sum(sum);
    if (lane == 0) red[8 + warp] = sum;
    side_barrier(0);
    if (tid == 0) {
      float tot = 0.f;
      for (int w = 0; w < CTC_SIDE / 32; ++w) tot += red[8 + w];
      double logp = -INFINITY;
      if (m != CTC_NEG_INF) logp = (double)m + (double)logf(tot) + C + offs[Th];
      reinterpret_cast<double*>(red + 16)[0] = logp;   // red is 8-byte aligned (see carve-up)
      p.costs[b] = (float)(-logp);
    }
  }
  __syncthreads();
  const double logp = reinterpret_cast<const double*>(red + 16)[0];
  if (grads == nullptr) return;
  if (logp == -INFINITY) {
    // infeasible alignment: cost = +inf, gradient defined as zero
    for (int k = tid; k < T * V; k += 2 * CTC_SIDE) grads[k] = 0.f;
    return;
  }

  // ------------------------------------------------------------------------------------------
  // phase 2: alpha continues over [Th, T) using spilled beta rows; beta continues over [0, Th)
  // using spilled alpha rows.  Gradient rows are produced on the fly.
  // ------------------------------------------------------------------------------------------
  {
    const int nsteps = side == 0 ? (T - Th) : Th;
    const int n0 = side == 0 ? Th : (T - Th);   // row index of this side at it == 0
    float other[NS];  // spilled row of the other lattice, prefetched one step ahead
    double other_off = 0.0;
    if (nsteps > 0) {
      const int t0 = side == 0 ? Th : (Th - 1);
#pragma unroll
      for (int q = 0; q < NS; ++q) {
        const int s = i + CTC_SIDE * q;
        other[q] = valid[q] ? ld_cg_f(ws + (size_t)t0 * p.S_stride + s) : CTC_NEG_INF;
      }
      other_off = offs[t0];
    }
    for (int it = 0; it < nsteps; ++it) {
      const int t = side == 0 ? (Th + it) : (Th - 1 - it);
      float* occ_t = my_occ + (it & 1) * V;
      float other_next[NS];
      double other_off_next = 0.0;
      const bool more = it + 1 < nsteps;
      const int tn = side == 0 ? (t + 1) : (t - 1);
#pragma unroll
      for (int q = 0; q < NS; ++q) {
        const int s = i + CTC_SIDE * q;
        other_next[q] = (more && valid[q]) ? ld_cg_f(ws + (size_t)tn * p.S_stride + s)
                                           : CTC_NEG_INF;
      }
      if (more) other_off_next = offs[tn];
      double vals[NS];
      if (side == 0 && it == 0) {
#pragma unroll
        for (int q = 0; q < NS; ++q) vals[q] = a_reg[q];   // row Th was formed at the meeting point
      } else {
        step_row(n0 + it, t, vals);
      }
      // scalar part of the exponent, formed in double: C_own + C_other(t) - log p
      const float delta = (float)(C + other_off - logp);
      float blank_sum = 0.f;
#pragma unroll
      for (int q = 0; q < NS; ++q) {
        const int s = i + CTC_SIDE * q;
        if (valid[q]) {
          const float g =
              __expf((float)(vals[q] + (double)other[q] - (double)emit(t, cls[q])) + delta);
          if (s & 1) atomicAdd(occ_t + cls[q], g);
          else blank_sum += g;
        }
      }
      // even threads own the blank states: one shared atomic per warp
      blank_sum = warp_sum(blank_sum);
      if (lane == 0 && blank_sum != 0.f) atomicAdd(occ_t + p.blank, blank_sum);
      side_barrier(side);
      for (int k = i; k < V; k += CTC_SIDE) {
        grads[t * V + k] = __expf(emit(t, k)) - occ_t[k];
        occ_t[k] = 0.f;
      }
#pragma unroll
      for (int q = 0; q < NS; ++q) other[q] = other_next[q];
      other_off = other_off_next;
    }
  }
}

template <int NS, bool STAGED>
static int launch_ctc(const CtcParams& p, size_t smem_bytes, cudaStream_t stream) {
  static size_t configured = 0;
  if (smem_bytes > configured) {
    if (cudaFuncSetAttribute(ctc_fwd_bwd_kernel<NS, STAGED>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem_bytes) != cudaSuccess)
      return SB_ERR_CUDA;
    configured = smem_bytes;
  }
  ctc_fwd_bwd_kernel<NS, STAGED><<<p.B, 2 * CTC_SIDE, smem_bytes, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

static int ctc_ns_for(int max_label_len) {
  const int S = 2 * max_label_len + 1;
  int ns = (S + CTC_SIDE - 1) / CTC_SIDE;
  if (ns <= 1) return 1;
  if (ns <= 2) return 2;
  if (ns <= 4) return 4;
  if (ns <= 8) return 8;
  return -1;
}

// Shared memory of the fused kernel: lattice rows, occupancies occ[4][V], reduction scratch, and
// either the staged (T x V) log-softmax or the per-frame log-sum-exp.
static constexpr size_t CTC_SMEM_LIMIT = 220 * 1024;
static size_t ctc_fixed_smem(int ns, int V) {
  return (size_t)(4 * (ns * CTC_SIDE + 4)) * sizeof(double) + (size_t)(4 * V + 64) * sizeof(float) + 8;
}
static bool ctc_staged(int ns, int T, int V) {
  return ctc_fixed_smem(ns, V) + (size_t)T * V * sizeof(float) <= CTC_SMEM_LIMIT;
}
// true where the fused kernel holds the shape (staged or not); every other shape takes the compact path
static bool ctc_fused_fits(int ns, int T, int V) {
  return ctc_staged(ns, T, V) || ctc_fixed_smem(ns, V) + (size_t)T * sizeof(float) <= CTC_SMEM_LIMIT;
}

static size_t ctc_fused_ws_bytes(int B, int T, int ns) {
  const size_t Tn = (size_t)(T > 0 ? T : 1);
  return (size_t)B * Tn * (size_t)(ns * CTC_SIDE) * sizeof(float) + (size_t)B * Tn * sizeof(double) + 512;
}

// the fused kernel at (B, T, p.V); p.offs / p.ws are carved from `workspace`
static int ctc_run_fused(CtcParams p, int ns, void* workspace, cudaStream_t stream) {
  const int B = p.B, T = p.T, V = p.V;
  p.offs = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  p.ws = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(p.offs + (size_t)B * T) + 255) & ~(uintptr_t)255);
  p.S_stride = ns * CTC_SIDE;
  if (!ctc_fused_fits(ns, T, V)) return SB_ERR_UNSUPPORTED;
  const bool staged = ctc_staged(ns, T, V);
  const size_t smem = ctc_fixed_smem(ns, V) + (size_t)T * (staged ? V : 1) * sizeof(float);

#define SB_CTC_CASE(NSV)                                                      \
  case NSV:                                                                   \
    return staged ? launch_ctc<NSV, true>(p, smem, stream)                    \
                  : launch_ctc<NSV, false>(p, smem, stream);
  switch (ns) {
    SB_CTC_CASE(1)
    SB_CTC_CASE(2)
    SB_CTC_CASE(4)
    SB_CTC_CASE(8)
  }
#undef SB_CTC_CASE
  return SB_ERR_UNSUPPORTED;
}

// ------------------------------------------------------------------------------------------------
// Compact path (any V).  The lattice of utterance b reads only the blank, its own label classes and
// each frame's log-sum-exp.  So each frame is reduced to Vc = max_label_len + 2 columns
//   0 = blank, 1..D_b = the D_b distinct non-blank label classes (order of first occurrence),
//   D_b + 1 = rest = log-sum-exp of the logits of every class outside that set (-inf if none),
//   D_b + 2 .. Vc - 1 = -inf (padding: no mass, zero gradient),
// whose log-softmax equals the full row's at the kept classes; the unchanged fused kernel then runs
// on the compact rows with blank = 0 and the labels remapped to columns.  The gradient of a class
// outside the set is its softmax (its occupancy is 0), that of a kept class the compact gradient of
// its column.  Labels equal to the blank class map to column 0, as the fused kernel treats them.
// ------------------------------------------------------------------------------------------------
static constexpr int CTC_CMP_THREADS = 256;
static constexpr int CTC_CMP_ROWS = 32;   // frames per CTA of the row kernels (one warp per frame)

struct CtcCompact {
  const float* acts;     // (B, T, V)
  float* grads;          // (B, T, V) or nullptr
  const int* labels;
  const int* label_off;
  const int* label_lens;
  const int* act_lens;
  const float* costs;    // (B) written by the fused kernel (read by the gradient expansion)
  float* acts_c;         // (B, T, Vc)
  const float* grads_c;  // (B, T, Vc)
  float* lse;            // (B, T) full-row log-sum-exp
  int* lab_c;            // (B, Lmax) labels as columns, utterance b at b * Lmax
  int* off_c;            // (B) = b * Lmax
  int* col_cls;          // (B, Vc) class of each column: >= 0 class, -1 rest, -2 padding
  int* ncols;            // (B) D_b
  int B, T, V, Vc, blank, Lmax;
};

// one CTA per utterance: dedupe the labels into columns (L <= 1023)
__global__ void __launch_bounds__(CTC_CMP_THREADS) ctc_colmap_kernel(const CtcCompact p) {
  __shared__ int first[1024];   // position of the first occurrence of label j's class
  __shared__ int colid[1024];   // column of a first occurrence
  const int b = blockIdx.x, tid = threadIdx.x;
  const int L = min(p.label_lens[b], p.Lmax);
  const int* lab = p.labels + p.label_off[b];
  for (int j = tid; j < L; j += CTC_CMP_THREADS) {
    const int c = lab[j];
    int f = j;
    for (int i = 0; i < j; ++i)
      if (lab[i] == c) { f = i; break; }
    first[j] = f;
  }
  __syncthreads();
  int* cls = p.col_cls + (size_t)b * p.Vc;
  if (tid == 0) {
    int d = 0;
    cls[0] = p.blank;
    for (int j = 0; j < L; ++j) {
      if (first[j] == j && lab[j] != p.blank) { colid[j] = ++d; cls[d] = lab[j]; }
    }
    for (int c = d + 1; c < p.Vc; ++c) cls[c] = (c == d + 1) ? -1 : -2;
    p.ncols[b] = d;
    p.off_c[b] = b * p.Lmax;
  }
  __syncthreads();
  int* out = p.lab_c + (size_t)b * p.Lmax;
  for (int j = tid; j < L; j += CTC_CMP_THREADS)
    out[j] = lab[j] == p.blank ? 0 : colid[first[j]];
}

// V-bit membership bitmap of {blank} + labels of utterance b in shared memory
SB_DEVINL void ctc_build_bitmap(const CtcCompact& p, int b, unsigned* bits) {
  const int words = (p.V + 31) >> 5;
  for (int w = threadIdx.x; w < words; w += blockDim.x) bits[w] = 0u;
  __syncthreads();
  const int L = min(p.label_lens[b], p.Lmax);
  const int* lab = p.labels + p.label_off[b];
  for (int j = threadIdx.x; j <= L; j += blockDim.x) {
    const int c = j < L ? lab[j] : p.blank;
    atomicOr(&bits[c >> 5], 1u << (c & 31));
  }
  __syncthreads();
}

// running (max, sum of exp(x - max)) of a stream of logits
SB_DEVINL void lse_push(float x, float& m, float& s) {
  if (x > m) {
    s = (m == CTC_NEG_INF ? 0.f : s * __expf(m - x)) + 1.f;
    m = x;
  } else if (x != CTC_NEG_INF) {
    s += __expf(x - m);
  }
}
SB_DEVINL float lse_warp(float m, float s) {
  const float M = warp_max(m);
  s = (M == CTC_NEG_INF || m == CTC_NEG_INF) ? 0.f : s * __expf(m - M);
  s = warp_sum(s);
  return s > 0.f ? M + __logf(s) : CTC_NEG_INF;
}

// grid (ceil(T / CTC_CMP_ROWS), B): compact rows and full-row log-sum-exp of the frames t < act_lens[b]
__global__ void __launch_bounds__(CTC_CMP_THREADS) ctc_compact_rows_kernel(const CtcCompact p) {
  extern __shared__ unsigned ctc_bits[];
  const int b = blockIdx.y;
  const int Tb = min(p.act_lens[b], p.T);
  const int t0 = blockIdx.x * CTC_CMP_ROWS;
  if (t0 >= Tb) return;
  ctc_build_bitmap(p, b, ctc_bits);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int V = p.V, Vc = p.Vc;
  const int* cls = p.col_cls + (size_t)b * Vc;
  for (int t = t0 + warp; t < min(t0 + CTC_CMP_ROWS, Tb); t += CTC_CMP_THREADS / 32) {
    const size_t row = (size_t)b * p.T + t;
    const float* a = p.acts + row * V;
    float mf = CTC_NEG_INF, sf = 0.f, mr = CTC_NEG_INF, sr = 0.f;
    for (int k = lane; k < V; k += 32) {
      const float x = __ldg(a + k);
      lse_push(x, mf, sf);
      if (!((ctc_bits[k >> 5] >> (k & 31)) & 1u)) lse_push(x, mr, sr);
    }
    const float lse_full = lse_warp(mf, sf);
    const float rest = lse_warp(mr, sr);
    if (lane == 0) p.lse[row] = lse_full;
    float* ac = p.acts_c + row * Vc;
    for (int c = lane; c < Vc; c += 32) {
      const int k = cls[c];
      ac[c] = k >= 0 ? __ldg(a + k) : (k == -1 ? rest : CTC_NEG_INF);
    }
  }
}

// grid (ceil(T / CTC_CMP_ROWS), B): every grads[b, t, k]
__global__ void __launch_bounds__(CTC_CMP_THREADS) ctc_expand_grads_kernel(const CtcCompact p) {
  extern __shared__ unsigned ctc_bits[];
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * CTC_CMP_ROWS;
  if (t0 >= p.T) return;
  const int Tb = p.costs[b] == INFINITY ? 0 : min(p.act_lens[b], p.T);
  const bool any = t0 < Tb;
  if (any) ctc_build_bitmap(p, b, ctc_bits);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int V = p.V, Vc = p.Vc;
  const int* cls = p.col_cls + (size_t)b * Vc;
  const int D = p.ncols[b];
  for (int t = t0 + warp; t < min(t0 + CTC_CMP_ROWS, p.T); t += CTC_CMP_THREADS / 32) {
    const size_t row = (size_t)b * p.T + t;
    float* g = p.grads + row * V;
    if (t >= Tb) {
      for (int k = lane; k < V; k += 32) g[k] = 0.f;
      continue;
    }
    const float* a = p.acts + row * V;
    const float lz = p.lse[row];
    for (int k = lane; k < V; k += 32)
      if (!((ctc_bits[k >> 5] >> (k & 31)) & 1u)) g[k] = __expf(__ldg(a + k) - lz);
    const float* gc = p.grads_c + row * Vc;
    for (int c = lane; c <= D; c += 32) g[cls[c]] = gc[c];
  }
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct CtcCompactLayout {
  size_t fused, acts_c, grads_c, lse, lab_c, off_c, col_cls, ncols, total;
};
static CtcCompactLayout ctc_compact_layout(int B, int T, int max_label_len, int ns) {
  const int Vc = max_label_len + 2;
  const size_t rows = (size_t)B * T;
  CtcCompactLayout l;
  size_t o = 256;   // slack for aligning the base pointer
  l.fused = o;   o += align256(ctc_fused_ws_bytes(B, T, ns));
  l.acts_c = o;  o += align256(rows * Vc * sizeof(float));
  l.grads_c = o; o += align256(rows * Vc * sizeof(float));
  l.lse = o;     o += align256(rows * sizeof(float));
  l.lab_c = o;   o += align256((size_t)B * (max_label_len > 0 ? max_label_len : 1) * sizeof(int));
  l.off_c = o;   o += align256((size_t)B * sizeof(int));
  l.col_cls = o; o += align256((size_t)B * Vc * sizeof(int));
  l.ncols = o;   o += align256((size_t)B * sizeof(int));
  l.total = o;
  return l;
}

template <typename K>
static int ctc_bitmap_kernel_attr(K kernel, size_t smem) {
  if (smem <= 48 * 1024) return SB_OK;
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) ==
                 cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

static int ctc_run_compact(const CtcParams& full, int max_label_len, int ns, void* workspace,
                           cudaStream_t stream) {
  const int B = full.B, T = full.T, V = full.V;
  const CtcCompactLayout l = ctc_compact_layout(B, T, max_label_len, ns);
  unsigned char* base = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255) - 256;
  CtcCompact c;
  c.acts = full.acts; c.grads = full.grads; c.labels = full.labels; c.label_off = full.label_off;
  c.label_lens = full.label_lens; c.act_lens = full.act_lens; c.costs = full.costs;
  c.acts_c = reinterpret_cast<float*>(base + l.acts_c);
  c.grads_c = reinterpret_cast<float*>(base + l.grads_c);
  c.lse = reinterpret_cast<float*>(base + l.lse);
  c.lab_c = reinterpret_cast<int*>(base + l.lab_c);
  c.off_c = reinterpret_cast<int*>(base + l.off_c);
  c.col_cls = reinterpret_cast<int*>(base + l.col_cls);
  c.ncols = reinterpret_cast<int*>(base + l.ncols);
  c.B = B; c.T = T; c.V = V; c.Vc = max_label_len + 2; c.blank = full.blank;
  c.Lmax = max_label_len > 0 ? max_label_len : 1;

  const size_t bits_smem = (size_t)((V + 31) / 32) * sizeof(unsigned);
  const dim3 rgrid((T + CTC_CMP_ROWS - 1) / CTC_CMP_ROWS, B);
  if (ctc_bitmap_kernel_attr(ctc_compact_rows_kernel, bits_smem) != SB_OK ||
      ctc_bitmap_kernel_attr(ctc_expand_grads_kernel, bits_smem) != SB_OK)
    return SB_ERR_CUDA;
  ctc_colmap_kernel<<<B, CTC_CMP_THREADS, 0, stream>>>(c);
  ctc_compact_rows_kernel<<<rgrid, CTC_CMP_THREADS, bits_smem, stream>>>(c);
  if (cudaGetLastError() != cudaSuccess) return SB_ERR_CUDA;

  CtcParams p = full;
  p.acts = c.acts_c;
  p.grads = full.grads ? const_cast<float*>(c.grads_c) : nullptr;
  p.labels = c.lab_c;
  p.label_off = c.off_c;
  p.V = c.Vc;
  p.blank = 0;
  const int rc = ctc_run_fused(p, ns, base + l.fused, stream);
  if (rc != SB_OK || !full.grads) return rc;
  ctc_expand_grads_kernel<<<rgrid, CTC_CMP_THREADS, bits_smem, stream>>>(c);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

// ------------------------------------------------------------------------------------------------
// Viterbi alignment (sb_ctc_viterbi).  The compact path's column map and row kernels reduce every
// frame first (any V); then one CTA of 256 threads per utterance runs the max-plus recursion over
// the extended labels, states s = i + 256*q, two float64 rows ping-ponged in shared memory, one
// barrier per frame.  Each warp packs its 32 states' 2-bit backpointers into one uint2 per frame
// with two ballots (bit 0 in .x, bit 1 in .y); warp 0 then walks them back, 32 frames per batch of
// loads: over 32 frames the state drops by at most 62, i.e. into the 3 words below and at its own.
// ------------------------------------------------------------------------------------------------
struct CtcViterbi {
  const float* acts_c;   // (B, T, Vc) compact rows
  const float* lse;      // (B, T) full-row log-sum-exp
  const int* lab_c;      // labels as columns, utterance b at b * Lstride
  const int* label_lens;
  const int* act_lens;
  uint2* bp;             // (B, T, NS * 8) backpointers
  int* path;             // (B, T)
  double* scores;        // (B)
  int B, T, Vc, Lmax, Lstride;
};

template <int NS>
__global__ void __launch_bounds__(CTC_SIDE) ctc_viterbi_kernel(const CtcViterbi p) {
  constexpr int NW = NS * CTC_SIDE / 32;   // backpointer words per frame
  __shared__ double rows[2][NS * CTC_SIDE + 2];
  __shared__ int s_end;
  const int b = blockIdx.x, i = threadIdx.x, warp = i >> 5, lane = i & 31;
  const int Tb = max(0, min(p.act_lens[b], p.T));
  const int L = max(0, min(p.label_lens[b], p.Lmax));
  const int S = 2 * L + 1;
  const int* lab = p.lab_c + (size_t)b * p.Lstride;
  const float* ac = p.acts_c + (size_t)b * p.T * p.Vc;
  const float* lz = p.lse + (size_t)b * p.T;
  uint2* bp = p.bp + (size_t)b * p.T * NW;
  int* path = p.path + (size_t)b * p.T;

  int col[NS];
  bool skip[NS], valid[NS];
#pragma unroll
  for (int q = 0; q < NS; ++q) {
    const int s = i + CTC_SIDE * q;
    valid[q] = s < S;
    col[q] = 0;
    skip[q] = false;
    if (valid[q] && (s & 1)) {
      const int j = (s - 1) >> 1;
      col[q] = lab[j];
      skip[q] = j > 0 && col[q] != 0 && lab[j - 1] != col[q];
    }
  }
  for (int k = i; k < 2 * (NS * CTC_SIDE + 2); k += CTC_SIDE) (&rows[0][0])[k] = -INFINITY;
  __syncthreads();

  // log-probability of this thread's states at frame t: compact column minus the full row's
  // log-sum-exp, in float32 as the compact loss path forms it
  auto emit = [&](int t, float (&e)[NS]) {
    const float z = __ldg(lz + t);
#pragma unroll
    for (int q = 0; q < NS; ++q) e[q] = valid[q] ? __ldg(ac + (size_t)t * p.Vc + col[q]) - z : 0.f;
  };
  float e[NS];
  if (Tb > 0) emit(0, e);
  for (int t = 0; t < Tb; ++t) {
    float en[NS];
    if (t + 1 < Tb) emit(t + 1, en);   // the next frame's loads overlap this frame's step
    double* cur = rows[t & 1] + 2;
    const double* prv = rows[(t & 1) ^ 1] + 2;
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int s = i + CTC_SIDE * q;
      unsigned code = 0;   // predecessor s - code; ties keep the smaller code
      if (valid[q]) {
        double v = -INFINITY;
        if (t == 0) {
          if (s <= 1) v = (double)e[q];
        } else {
          double best = prv[s];
          if (prv[s - 1] > best) { best = prv[s - 1]; code = 1; }
          if (skip[q] && prv[s - 2] > best) { best = prv[s - 2]; code = 2; }
          v = best + (double)e[q];
        }
        cur[s] = v;
      }
      const unsigned lo = __ballot_sync(0xffffffffu, code & 1u);
      const unsigned hi = __ballot_sync(0xffffffffu, code >> 1);
      if (lane == 0) bp[(size_t)t * NW + q * (CTC_SIDE / 32) + warp] = make_uint2(lo, hi);
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < NS; ++q) e[q] = en[q];
  }

  if (i == 0) {
    double sc = L == 0 ? 0.0 : -INFINITY;
    int end = -1;
    if (Tb > 0) {
      const double* last = rows[(Tb - 1) & 1] + 2;
      sc = last[S - 1];
      end = S - 1;
      if (S >= 2 && last[S - 2] > sc) { sc = last[S - 2]; end = S - 2; }
    }
    if (sc == -INFINITY) end = -1;
    p.scores[b] = sc;
    s_end = end;
  }
  __syncthreads();
  const int end = s_end;
  for (int t = (end < 0 ? 0 : Tb) + i; t < p.T; t += CTC_SIDE) path[t] = -2;
  if (end < 0 || warp != 0) return;

  int s = end;
  for (int t1 = Tb - 1; t1 >= 0; t1 -= 32) {
    const int w0 = s >> 5;
    const int tl = t1 - lane;
    uint2 wd[3] = {make_uint2(0u, 0u), make_uint2(0u, 0u), make_uint2(0u, 0u)};
    if (tl >= 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (w0 - k >= 0) wd[k] = __ldcg(bp + (size_t)tl * NW + w0 - k);
    }
    int mine = -2;
    const int n = min(32, t1 + 1);
    for (int k = 0; k < n; ++k) {
      const int dw = w0 - (s >> 5);
      const unsigned lo0 = __shfl_sync(0xffffffffu, wd[0].x, k), hi0 = __shfl_sync(0xffffffffu, wd[0].y, k);
      const unsigned lo1 = __shfl_sync(0xffffffffu, wd[1].x, k), hi1 = __shfl_sync(0xffffffffu, wd[1].y, k);
      const unsigned lo2 = __shfl_sync(0xffffffffu, wd[2].x, k), hi2 = __shfl_sync(0xffffffffu, wd[2].y, k);
      const unsigned lo = dw == 0 ? lo0 : (dw == 1 ? lo1 : lo2);
      const unsigned hi = dw == 0 ? hi0 : (dw == 1 ? hi1 : hi2);
      if (lane == k) mine = (s & 1) ? (s - 1) >> 1 : -1;
      s -= (int)(((lo >> (s & 31)) & 1u) | (((hi >> (s & 31)) & 1u) << 1));
    }
    if (lane < n) path[t1 - lane] = mine;
  }
}

struct CtcViterbiLayout {
  size_t acts_c, lse, lab_c, off_c, col_cls, ncols, bp, total;
};
static CtcViterbiLayout ctc_viterbi_layout(int B, int T, int max_label_len, int ns) {
  const int Vc = max_label_len + 2;
  const size_t rows = (size_t)B * T;
  CtcViterbiLayout l;
  size_t o = 256;   // slack for aligning the base pointer
  l.acts_c = o;  o += align256(rows * Vc * sizeof(float));
  l.lse = o;     o += align256(rows * sizeof(float));
  l.lab_c = o;   o += align256((size_t)B * (max_label_len > 0 ? max_label_len : 1) * sizeof(int));
  l.off_c = o;   o += align256((size_t)B * sizeof(int));
  l.col_cls = o; o += align256((size_t)B * Vc * sizeof(int));
  l.ncols = o;   o += align256((size_t)B * sizeof(int));
  l.bp = o;      o += align256(rows * (size_t)(ns * CTC_SIDE / 32) * sizeof(uint2));
  l.total = o;
  return l;
}

}  // namespace sb

using namespace sb;

extern "C" int sb_ctc_compact_workspace_size(int B, int T, int V, int max_label_len,
                                             size_t* bytes) {
  if (!bytes || B <= 0 || T < 0 || V <= 0 || max_label_len < 0) return SB_ERR_INVALID;
  const int ns = ctc_ns_for(max_label_len);
  if (ns < 0) return SB_ERR_UNSUPPORTED;
  *bytes = ctc_compact_layout(B, T > 0 ? T : 1, max_label_len, ns).total;
  return SB_OK;
}

extern "C" int sb_ctc_workspace_size(int B, int T, int V, int max_label_len, size_t* bytes) {
  if (!bytes || B <= 0 || T < 0 || V <= 0 || max_label_len < 0) return SB_ERR_INVALID;
  const int ns = ctc_ns_for(max_label_len);
  if (ns < 0) return SB_ERR_UNSUPPORTED;
  if (!ctc_fused_fits(ns, T, V)) return sb_ctc_compact_workspace_size(B, T, V, max_label_len, bytes);
  *bytes = ctc_fused_ws_bytes(B, T, ns);
  return SB_OK;
}

static int ctc_entry(const float* acts, float* grads, const int* labels_dev,
                     const int* label_offsets_dev, const int* label_lens_dev,
                     const int* act_lens_dev, int B, int T, int V, int blank, int max_label_len,
                     float* costs, void* workspace, size_t workspace_bytes, void* stream_,
                     bool compact) {
  if (!acts || !labels_dev || !label_offsets_dev || !label_lens_dev || !act_lens_dev || !costs ||
      !workspace)
    return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || V <= 0 || blank < 0 || blank >= V || max_label_len < 0)
    return SB_ERR_INVALID;
  const int ns = ctc_ns_for(max_label_len);
  if (ns < 0) return SB_ERR_UNSUPPORTED;
  compact = compact || !ctc_fused_fits(ns, T, V);
  size_t need = 0;
  int rc = compact ? sb_ctc_compact_workspace_size(B, T, V, max_label_len, &need)
                   : sb_ctc_workspace_size(B, T, V, max_label_len, &need);
  if (rc != SB_OK) return rc;
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);

  CtcParams p;
  p.acts = acts; p.grads = grads; p.labels = labels_dev; p.label_off = label_offsets_dev;
  p.label_lens = label_lens_dev; p.act_lens = act_lens_dev; p.costs = costs;
  p.offs = nullptr; p.ws = nullptr;
  p.B = B; p.T = T; p.V = V; p.blank = blank; p.S_stride = ns * CTC_SIDE;
  return compact ? ctc_run_compact(p, max_label_len, ns, workspace, stream)
                 : ctc_run_fused(p, ns, workspace, stream);
}

extern "C" int sb_ctc_fwd_bwd(const float* acts, float* grads, const int* labels_dev,
                              const int* label_offsets_dev, const int* label_lens_dev,
                              const int* act_lens_dev, int B, int T, int V, int blank,
                              int max_label_len, float* costs, void* workspace,
                              size_t workspace_bytes, void* stream) {
  return ctc_entry(acts, grads, labels_dev, label_offsets_dev, label_lens_dev, act_lens_dev, B, T,
                   V, blank, max_label_len, costs, workspace, workspace_bytes, stream, false);
}

extern "C" int sb_ctc_fwd_bwd_compact(const float* acts, float* grads, const int* labels_dev,
                                      const int* label_offsets_dev, const int* label_lens_dev,
                                      const int* act_lens_dev, int B, int T, int V, int blank,
                                      int max_label_len, float* costs, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  return ctc_entry(acts, grads, labels_dev, label_offsets_dev, label_lens_dev, act_lens_dev, B, T,
                   V, blank, max_label_len, costs, workspace, workspace_bytes, stream, true);
}

extern "C" int sb_ctc_viterbi_workspace_size(int B, int T, int V, int max_label_len,
                                             size_t* bytes) {
  if (!bytes || B <= 0 || T < 0 || V <= 0 || max_label_len < 0) return SB_ERR_INVALID;
  const int ns = ctc_ns_for(max_label_len);
  if (ns < 0) return SB_ERR_UNSUPPORTED;
  *bytes = ctc_viterbi_layout(B, T > 0 ? T : 1, max_label_len, ns).total;
  return SB_OK;
}

extern "C" int sb_ctc_viterbi(const float* acts, const int* labels_dev,
                              const int* label_offsets_dev, const int* label_lens_dev,
                              const int* act_lens_dev, int B, int T, int V, int blank,
                              int max_label_len, int* path, double* scores, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  if (!acts || !labels_dev || !label_offsets_dev || !label_lens_dev || !act_lens_dev || !path ||
      !scores || !workspace)
    return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || V <= 0 || blank < 0 || blank >= V || max_label_len < 0)
    return SB_ERR_INVALID;
  const int ns = ctc_ns_for(max_label_len);
  if (ns < 0) return SB_ERR_UNSUPPORTED;
  const CtcViterbiLayout l = ctc_viterbi_layout(B, T, max_label_len, ns);
  if (workspace_bytes < l.total) return SB_ERR_WORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  unsigned char* base = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255) - 256;

  CtcCompact c;
  c.acts = acts; c.grads = nullptr; c.labels = labels_dev; c.label_off = label_offsets_dev;
  c.label_lens = label_lens_dev; c.act_lens = act_lens_dev; c.costs = nullptr;
  c.acts_c = reinterpret_cast<float*>(base + l.acts_c);
  c.grads_c = nullptr;
  c.lse = reinterpret_cast<float*>(base + l.lse);
  c.lab_c = reinterpret_cast<int*>(base + l.lab_c);
  c.off_c = reinterpret_cast<int*>(base + l.off_c);
  c.col_cls = reinterpret_cast<int*>(base + l.col_cls);
  c.ncols = reinterpret_cast<int*>(base + l.ncols);
  c.B = B; c.T = T; c.V = V; c.Vc = max_label_len + 2; c.blank = blank;
  c.Lmax = max_label_len > 0 ? max_label_len : 1;

  const size_t bits_smem = (size_t)((V + 31) / 32) * sizeof(unsigned);
  if (ctc_bitmap_kernel_attr(ctc_compact_rows_kernel, bits_smem) != SB_OK) return SB_ERR_CUDA;
  ctc_colmap_kernel<<<B, CTC_CMP_THREADS, 0, stream>>>(c);
  ctc_compact_rows_kernel<<<dim3((T + CTC_CMP_ROWS - 1) / CTC_CMP_ROWS, B), CTC_CMP_THREADS,
                            bits_smem, stream>>>(c);

  CtcViterbi v;
  v.acts_c = c.acts_c; v.lse = c.lse; v.lab_c = c.lab_c;
  v.label_lens = label_lens_dev; v.act_lens = act_lens_dev;
  v.bp = reinterpret_cast<uint2*>(base + l.bp);
  v.path = path; v.scores = scores;
  v.B = B; v.T = T; v.Vc = c.Vc; v.Lmax = max_label_len; v.Lstride = c.Lmax;
  switch (ns) {
    case 1: ctc_viterbi_kernel<1><<<B, CTC_SIDE, 0, stream>>>(v); break;
    case 2: ctc_viterbi_kernel<2><<<B, CTC_SIDE, 0, stream>>>(v); break;
    case 4: ctc_viterbi_kernel<4><<<B, CTC_SIDE, 0, stream>>>(v); break;
    default: ctc_viterbi_kernel<8><<<B, CTC_SIDE, 0, stream>>>(v); break;
  }
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
