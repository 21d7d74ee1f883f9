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

}  // namespace sb

using namespace sb;

extern "C" int sb_ctc_workspace_size(int B, int T, int V, int max_label_len, size_t* bytes) {
  if (!bytes || B <= 0 || T < 0 || V <= 0 || max_label_len < 0) return SB_ERR_INVALID;
  const int ns = ctc_ns_for(max_label_len);
  if (ns < 0) return SB_ERR_UNSUPPORTED;
  const size_t Tn = (size_t)(T > 0 ? T : 1);
  *bytes = (size_t)B * Tn * (size_t)(ns * CTC_SIDE) * sizeof(float) + (size_t)B * Tn * sizeof(double) + 512;
  return SB_OK;
}

extern "C" int sb_ctc_fwd_bwd(const float* acts, float* grads, const int* labels_dev,
                              const int* label_offsets_dev, const int* label_lens_dev,
                              const int* act_lens_dev, int B, int T, int V, int blank,
                              int max_label_len, float* costs, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  if (!acts || !labels_dev || !label_offsets_dev || !label_lens_dev || !act_lens_dev || !costs ||
      !workspace)
    return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || V <= 0 || blank < 0 || blank >= V) return SB_ERR_INVALID;
  size_t need = 0;
  int rc = sb_ctc_workspace_size(B, T, V, max_label_len, &need);
  if (rc != SB_OK) return rc;
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  const int ns = ctc_ns_for(max_label_len);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);

  CtcParams p;
  p.acts = acts; p.grads = grads; p.labels = labels_dev; p.label_off = label_offsets_dev;
  p.label_lens = label_lens_dev; p.act_lens = act_lens_dev; p.costs = costs;
  p.offs = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  p.ws = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(p.offs + (size_t)B * T) + 255) & ~(uintptr_t)255);
  p.B = B; p.T = T; p.V = V; p.blank = blank; p.S_stride = ns * CTC_SIDE;

  const size_t fixed = (size_t)(4 * (ns * CTC_SIDE + 4)) * sizeof(double) +
                       (size_t)(4 * V + 64) * sizeof(float) + 8;
  const size_t staged_bytes = fixed + (size_t)T * V * sizeof(float);
  const size_t unstaged_bytes = fixed + (size_t)T * sizeof(float);
  const size_t limit = 220 * 1024;
  const bool staged = staged_bytes <= limit;
  if (!staged && unstaged_bytes > limit) return SB_ERR_UNSUPPORTED;
  const size_t smem = staged ? staged_bytes : unstaged_bytes;

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
