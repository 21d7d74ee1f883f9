// sb_rnnt_fwd_bwd: RNN-Transducer negative log-likelihood + gradient w.r.t. the LOG-PROBABILITIES.
//
// Replaces transducer.functions.transducer.TransducerLoss (libs/transducer, un-vendored,
// Makefile:10-12; call site speech/models/transducer_model.py:46-52): input is the
// (B, T, U+1, V+1) log-softmax tensor the reference builds itself (transducer_model.py:71-76),
// flat int32 labels, per-utterance frame / label counts; blank = last class (:28); the caller sums
// the per-utterance costs.  Arithmetic after Graves 2012: alpha(t,u) / beta(t,u) over the
// T x (U+1) lattice,
//   alpha(t,u) = lse(alpha(t-1,u) + blank(t-1,u), alpha(t,u-1) + y(t,u-1)),
//   cost = -(alpha(T-1,U) + blank(T-1,U)),
//   dcost/dlp[t,u,blank] = -exp(alpha(t,u) + blank(t,u) + beta(t+1,u) - logP)
//   dcost/dlp[t,u,y_u]   = -exp(alpha(t,u) + y(t,u)     + beta(t,u+1) - logP),  zero elsewhere.
//
// One CTA per utterance, 512 threads: 256 run alpha along anti-diagonals (cells with t+u = d are
// independent), 256 run beta from the far corner CONCURRENTLY; thread u owns column u, its
// previous cell stays in a register and its neighbour's cell comes from a shared-memory ping-pong,
// one named barrier per diagonal.  The two emissions a cell needs are gathered from the 4-D
// tensor one diagonal ahead.  Lattices are float64 (T+U serial steps), spilled to a workspace,
// then the same CTA writes the (sparse) gradient.
// Roofline: HBM-nominal (2 of V+1 entries per cell are read, the gradient tensor is written);
// bound by the (T+U)-step chain for small B.
#include "common.cuh"
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int RNNT_SIDE = 256;

struct RnntParams {
  const float* lp;        // (B, T, U1, V)
  float* grads;           // (B, T, U1, V) or null (must be zero-filled by the caller API)
  const int* labels;      // flat
  const int* label_off;   // (B)
  const int* label_lens;  // (B)  U_b
  const int* act_lens;    // (B)  T_b
  float* costs;           // (B)
  double* ws;             // (B, 2, T, U1) alpha, beta
  int B, T, U1, V, blank;
  int compact;            // lp / grads are (T, B, U1, 2), TIME-major nodes (t*B + b)*U1 + u:
                          // {blank, label of arc u -> u+1}
};

SB_DEVINL double lse2dd(double a, double b) {
  const double m = fmax(a, b);
  if (m == -INFINITY) return -INFINITY;
  return m + log1p(exp(fmin(a, b) - m));
}
SB_DEVINL void rnnt_side_barrier(int side) {
  asm volatile("bar.sync %0, %1;" ::"r"(side + 1), "r"(RNNT_SIDE) : "memory");
}

template <int NS>
__global__ void __launch_bounds__(2 * RNNT_SIDE, 1) rnnt_fwd_bwd_kernel(const RnntParams p) {
  __shared__ double nb[2][2][NS * RNNT_SIDE + 2];   // [side][parity][u + 1]
  __shared__ double s_logp;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int side = tid / RNNT_SIDE, i = tid % RNNT_SIDE;
  const int T = min(p.act_lens[b], p.T);
  const int U = min(p.label_lens[b], p.U1 - 1);      // labels of this utterance
  const int U1 = p.U1, V = p.V;
  const int* lab = p.labels + p.label_off[b];
  const float* lp = p.compact ? p.lp + (size_t)b * U1 * 2 : p.lp + (size_t)b * p.T * U1 * V;
  const size_t tstr = p.compact ? (size_t)p.B * U1 : (size_t)U1;   // nodes between two frames
  double* alpha = p.ws + (size_t)b * 2 * p.T * U1;
  double* beta = alpha + (size_t)p.T * U1;

  for (int k = tid; k < 2 * 2 * (NS * RNNT_SIDE + 2); k += 2 * RNNT_SIDE)
    (&nb[0][0][0])[k] = -INFINITY;
  __syncthreads();
  if (T <= 0) {
    if (tid == 0) p.costs[b] = (U == 0) ? 0.f : INFINITY;
    return;
  }

  int ylab[NS];
#pragma unroll
  for (int q = 0; q < NS; ++q) {
    const int u = i + RNNT_SIDE * q;
    ylab[q] = (u < U) ? lab[u] : p.blank;
  }
  // (in the compact form the only label ever asked for at node u is the one of arc u -> u+1)
  auto LP = [&](int t, int u, int k) -> double {
    const size_t node = (size_t)t * tstr + u;
    return (double)__ldg(p.compact ? lp + node * 2 + (k == p.blank ? 0 : 1) : lp + node * V + k);
  };

  double own[NS];   // this thread's previous cell in column u
#pragma unroll
  for (int q = 0; q < NS; ++q) own[q] = -INFINITY;
  const int ndiag = T + U;   // diagonals 0 .. T+U-1
  for (int d = 0; d < ndiag; ++d) {
    double* cur = nb[side][d & 1] + 1;
    const double* prv = nb[side][(d & 1) ^ 1] + 1;
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int u = i + RNNT_SIDE * q;
      if (u > U) continue;
      if (side == 0) {
        const int t = d - u;
        if (t < 0 || t >= T) continue;
        double v;
        if (t == 0 && u == 0) v = 0.0;
        else {
          const double a = (t > 0) ? own[q] + LP(t - 1, u, p.blank) : -INFINITY;
          const double c = (u > 0) ? prv[u - 1] + LP(t, u - 1, lab[u - 1]) : -INFINITY;
          v = lse2dd(a, c);
        }
        own[q] = v;
        cur[u] = v;
        alpha[(size_t)t * U1 + u] = v;
      } else {
        // beta runs the mirrored diagonal: t = T-1 - (d - (U - u))
        const int t = T - 1 - (d - (U - u));
        if (t < 0 || t >= T) continue;
        double v;
        if (t == T - 1 && u == U) v = LP(t, u, p.blank);
        else {
          const double a = (t < T - 1) ? own[q] + LP(t, u, p.blank) : -INFINITY;
          const double c = (u < U) ? prv[u + 1] + LP(t, u, ylab[q]) : -INFINITY;
          v = lse2dd(a, c);
        }
        own[q] = v;
        cur[u] = v;
        beta[(size_t)t * U1 + u] = v;
      }
    }
    rnnt_side_barrier(side);
  }
  __syncthreads();
  if (tid == 0) {
    const double logp = beta[0];
    s_logp = logp;
    p.costs[b] = (float)(-logp);
  }
  __syncthreads();
  const double logp = s_logp;
  if (p.grads == nullptr || logp == -INFINITY) return;
  const int gstride = p.compact ? 2 : V;
  float* g = p.compact ? p.grads + (size_t)b * U1 * 2 : p.grads + (size_t)b * p.T * U1 * V;
  for (int c = tid; c < T * (U + 1); c += 2 * RNNT_SIDE) {
    const int t = c / (U + 1), u = c % (U + 1);
    const double a = alpha[(size_t)t * U1 + u];
    if (a == -INFINITY) continue;
    const size_t base = ((size_t)t * tstr + u) * gstride;
    // blank transition
    double nxt = (t < T - 1) ? beta[(size_t)(t + 1) * U1 + u] : ((u == U) ? 0.0 : -INFINITY);
    if (nxt != -INFINITY)
      g[base + (p.compact ? 0 : p.blank)] = -(float)exp(a + LP(t, u, p.blank) + nxt - logp);
    if (u < U) {
      const double bn = beta[(size_t)t * U1 + u + 1];
      if (bn != -INFINITY)
        g[base + (p.compact ? 1 : lab[u])] = -(float)exp(a + LP(t, u, lab[u]) + bn - logp);
    }
  }
}

// Viterbi alignment over the compact lattice (sb_rnnt_viterbi): the alpha side's anti-diagonal
// wavefront above with max in place of log-sum-exp, 256 threads, column u on thread u % 256.  The
// two arcs a node reads for the next diagonal are loaded while the current one is formed.  Each
// warp packs its 32 columns' choice (1 = label arc) into one word per diagonal with a ballot; warp
// 0 then walks back from (T_b-1, U_b), 32 diagonals per batch of loads: over 32 diagonals u drops
// by at most 31, i.e. into the word below or its own.
struct RnntViterbi {
  const float* lat;       // (T, B, U1, 2)
  const int* label_lens;
  const int* act_lens;
  unsigned* bits;         // (B, T + U1, NS * 8) backpointers by diagonal
  int* frames;            // (B, U1 - 1)
  double* scores;         // (B)
  int B, T, U1;
};

template <int NS>
__global__ void __launch_bounds__(RNNT_SIDE) rnnt_viterbi_kernel(const RnntViterbi p) {
  constexpr int NW = NS * RNNT_SIDE / 32;   // backpointer words per diagonal
  __shared__ double nb[2][NS * RNNT_SIDE + 1];   // [parity][u + 1]
  __shared__ double s_score;
  const int b = blockIdx.x, i = threadIdx.x, warp = i >> 5, lane = i & 31;
  const int T = max(0, min(p.act_lens[b], p.T));
  const int U = max(0, min(p.label_lens[b], p.U1 - 1));
  const int U1 = p.U1;
  const size_t tstr = (size_t)p.B * U1;
  const float* lat = p.lat + (size_t)b * U1 * 2;
  unsigned* bits = p.bits + (size_t)b * (p.T + U1) * NW;
  int* frames = p.frames + (size_t)b * (U1 - 1);

  for (int k = i; k < 2 * (NS * RNNT_SIDE + 1); k += RNNT_SIDE) (&nb[0][0])[k] = -INFINITY;
  for (int u = U + i; u < U1 - 1; u += RNNT_SIDE) frames[u] = -1;
  __syncthreads();
  if (T <= 0) {
    if (i == 0) p.scores[b] = -INFINITY;
    for (int u = i; u < U; u += RNNT_SIDE) frames[u] = -1;
    return;
  }

  // arcs into (t, u) = (d - u, u): blank of (t-1, u) and label of (t, u-1), -inf where absent
  auto arcs = [&](int d, float (&bl)[NS], float (&lb)[NS]) {
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int u = i + RNNT_SIDE * q, t = d - u;
      bl[q] = lb[q] = -INFINITY;
      if (u <= U && t >= 0 && t < T) {
        if (t > 0) bl[q] = __ldg(lat + ((size_t)(t - 1) * tstr + u) * 2);
        if (u > 0) lb[q] = __ldg(lat + ((size_t)t * tstr + u - 1) * 2 + 1);
      }
    }
  };
  double own[NS];   // this thread's previous cell in column u
  float bl[NS], lb[NS];
#pragma unroll
  for (int q = 0; q < NS; ++q) own[q] = -INFINITY;
  arcs(0, bl, lb);
  const int ndiag = T + U;
  for (int d = 0; d < ndiag; ++d) {
    float bln[NS], lbn[NS];
    arcs(d + 1, bln, lbn);
    double* cur = nb[d & 1] + 1;
    const double* prv = nb[(d & 1) ^ 1] + 1;
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int u = i + RNNT_SIDE * q, t = d - u;
      bool label = false;
      if (u <= U && t >= 0 && t < T) {
        double v = 0.0;
        if (d > 0) {
          const double a = own[q] + (double)bl[q];
          const double c = prv[u - 1] + (double)lb[q];   // prv[-1] is the -inf pad
          label = c > a;   // ties take the blank arc: the label came at an earlier frame
          v = label ? c : a;
        }
        own[q] = v;
        cur[u] = v;
      }
      const unsigned w = __ballot_sync(0xffffffffu, label);
      if (lane == 0) bits[(size_t)d * NW + q * (RNNT_SIDE / 32) + warp] = w;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < NS; ++q) { bl[q] = bln[q]; lb[q] = lbn[q]; }
  }
#pragma unroll
  for (int q = 0; q < NS; ++q) {
    if (i + RNNT_SIDE * q == U) {
      const double sc = own[q] + (double)__ldg(lat + ((size_t)(T - 1) * tstr + U) * 2);
      p.scores[b] = sc;
      s_score = sc;
    }
  }
  __syncthreads();
  if (s_score == -INFINITY) {
    for (int u = i; u < U; u += RNNT_SIDE) frames[u] = -1;
    return;
  }
  if (warp != 0) return;

  int t = T - 1, u = U;
  for (int d1 = T - 1 + U; d1 > 0; d1 -= 32) {
    const int w0 = u >> 5;
    const int dl = d1 - lane;
    unsigned w_own = 0u, w_below = 0u;
    if (dl > 0) {
      w_own = __ldcg(bits + (size_t)dl * NW + w0);
      if (w0 > 0) w_below = __ldcg(bits + (size_t)dl * NW + w0 - 1);
    }
    const int n = min(32, d1);
    for (int k = 0; k < n; ++k) {
      const unsigned a = __shfl_sync(0xffffffffu, w_own, k);
      const unsigned c = __shfl_sync(0xffffffffu, w_below, k);
      const unsigned w = (u >> 5) == w0 ? a : c;
      if ((w >> (u & 31)) & 1u) {
        --u;
        if (lane == 0) frames[u] = t;
      } else {
        --t;
      }
    }
  }
}

}  // namespace sb

using namespace sb;

static int rnnt_viterbi_ns(int U1) {
  const int ns = (U1 + RNNT_SIDE - 1) / RNNT_SIDE;
  return ns <= 1 ? 1 : ns <= 2 ? 2 : ns <= 4 ? 4 : -1;
}

extern "C" int sb_rnnt_viterbi_workspace_size(int B, int T, int U1, size_t* bytes) {
  if (!bytes || B <= 0 || T <= 0 || U1 <= 0) return SB_ERR_INVALID;
  const int ns = rnnt_viterbi_ns(U1);
  if (ns < 0) return SB_ERR_UNSUPPORTED;
  *bytes = (size_t)B * (T + U1) * (ns * RNNT_SIDE / 32) * sizeof(unsigned) + 256;
  return SB_OK;
}

extern "C" int sb_rnnt_viterbi(const float* lat, const int* labels, const int* label_offsets,
                               const int* label_lens, const int* act_lens, int B, int T, int U1,
                               int* frames, double* scores, void* workspace,
                               size_t workspace_bytes, void* stream_) {
  if (!lat || !labels || !label_offsets || !label_lens || !act_lens || !frames || !scores ||
      !workspace)
    return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || U1 <= 0) return SB_ERR_INVALID;
  size_t need = 0;
  const int rc = sb_rnnt_viterbi_workspace_size(B, T, U1, &need);
  if (rc != SB_OK) return rc;
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  RnntViterbi p;
  p.lat = lat; p.label_lens = label_lens; p.act_lens = act_lens;
  p.bits = reinterpret_cast<unsigned*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  p.frames = frames; p.scores = scores;
  p.B = B; p.T = T; p.U1 = U1;
  switch (rnnt_viterbi_ns(U1)) {
    case 1: rnnt_viterbi_kernel<1><<<B, RNNT_SIDE, 0, stream>>>(p); break;
    case 2: rnnt_viterbi_kernel<2><<<B, RNNT_SIDE, 0, stream>>>(p); break;
    default: rnnt_viterbi_kernel<4><<<B, RNNT_SIDE, 0, stream>>>(p); break;
  }
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_workspace_size(int B, int T, int U1, size_t* bytes) {
  if (!bytes || B <= 0 || T <= 0 || U1 <= 0) return SB_ERR_INVALID;
  *bytes = (size_t)B * 2 * T * U1 * sizeof(double) + 256;
  return SB_OK;
}

static int rnnt_run(const float* log_probs, float* grads, const int* labels,
                    const int* label_offsets, const int* label_lens, const int* act_lens, int B,
                    int T, int U1, int V, int blank, int compact, float* costs, void* workspace,
                    size_t workspace_bytes, void* stream_) {
  if (!log_probs || !labels || !label_offsets || !label_lens || !act_lens || !costs || !workspace)
    return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || U1 <= 0 || V <= 0 || blank < 0 || blank >= V) return SB_ERR_INVALID;
  size_t need = 0;
  sb_rnnt_workspace_size(B, T, U1, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  RnntParams p;
  p.lp = log_probs; p.grads = grads; p.labels = labels; p.label_off = label_offsets;
  p.label_lens = label_lens; p.act_lens = act_lens; p.costs = costs;
  p.ws = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  p.B = B; p.T = T; p.U1 = U1; p.V = V; p.blank = blank; p.compact = compact;
  if (grads && cudaMemsetAsync(grads, 0, sizeof(float) * (size_t)B * T * U1 * (compact ? 2 : V),
                               stream) != cudaSuccess)
    return SB_ERR_CUDA;
  const int ns = (U1 + RNNT_SIDE - 1) / RNNT_SIDE;
  if (ns <= 1) rnnt_fwd_bwd_kernel<1><<<B, 2 * RNNT_SIDE, 0, stream>>>(p);
  else if (ns <= 2) rnnt_fwd_bwd_kernel<2><<<B, 2 * RNNT_SIDE, 0, stream>>>(p);
  else if (ns <= 4) rnnt_fwd_bwd_kernel<4><<<B, 2 * RNNT_SIDE, 0, stream>>>(p);
  else return SB_ERR_UNSUPPORTED;
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_fwd_bwd(const float* log_probs, float* grads, const int* labels,
                               const int* label_offsets, const int* label_lens,
                               const int* act_lens, int B, int T, int U1, int V, int blank,
                               float* costs, void* workspace, size_t workspace_bytes,
                               void* stream_) {
  return rnnt_run(log_probs, grads, labels, label_offsets, label_lens, act_lens, B, T, U1, V,
                  blank, 0, costs, workspace, workspace_bytes, stream_);
}

// Compact lattice (what sb_rnnt_joint_fwd writes): lat / garc are (T, B, U1, 2), time-major, =
// {log p(blank), log p(label of arc u -> u+1)} per node and the gradients w.r.t. them.
extern "C" int sb_rnnt_fwd_bwd_compact(const float* lat, float* garc, const int* labels,
                                       const int* label_offsets, const int* label_lens,
                                       const int* act_lens, int B, int T, int U1, int blank,
                                       float* costs, void* workspace, size_t workspace_bytes,
                                       void* stream_) {
  return rnnt_run(lat, garc, labels, label_offsets, label_lens, act_lens, B, T, U1, blank + 1,
                  blank, 1, costs, workspace, workspace_bytes, stream_);
}
