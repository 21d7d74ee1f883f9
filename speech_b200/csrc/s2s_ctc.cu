// Joint CTC/attention decoding of the attention model (Watanabe et al. 2017, "Hybrid CTC/Attention
// Architecture for End-to-End Speech Recognition", Algorithm 2): the batched attention beam search
// of s2s.cu, with every candidate's value adding lambda times the CTC prefix log-probability of the
// extended hypothesis, from the CTC head's per-frame log-probabilities y_t (B, T, C), blank C - 1.
//
// Per live row r the search keeps A_r (attention + LM part of the score), psi_r = psi(h_r) and the
// CTC forward variables gn_t(h_r), gb_t(h_r) (h_r ends in a label / in blank at frame t) for
// t < T_b.  The hypothesis score is S_r = A_r + lambda psi_r (BeamState::score).  Per step:
//   s2s_ctc_cand    CTA per live row: P(r, c) = (1 - lambda) logp[r][c] (+ alpha lm(c | h_r) +
//                   beta_c), the row's top M classes by P (ties to the lower class) in class order,
//                   then one thread per candidate runs the T_b-frame prefix recursion over the
//                   row's vectors and the frames' y, staged in shared memory a chunk at a time, and
//                   writes (class, A_r + P, psi, value = (A_r + P) + lambda psi) to the row's list;
//   s2s_ctc_select  CTA per utterance over the K*M list: the selection and bookkeeping of s2s.cu
//                   (beam_bookkeep over the list) and A' of the new rows (psi' is in their score);
//   s2s_ctc_extend  CTA per utterance, warp per new row: its vectors, recomputed from the parent
//                   row's and the chosen class, into the other of two buffers.
// Everything after the float32 y and logp is float64, with no contracted multiply-adds, so that a
// float64 restatement on the host gives the same values to rounding; lse(a, b) = max +
// log1p(exp(min - max)), -inf when both are.
#include "s2s_beam.cuh"
#include <math.h>
#include <stddef.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int CTC_MAXM = 128;        // candidates per row: the threads of s2s_ctc_cand
static constexpr int CTC_TCH = 32;          // frames staged per chunk
static constexpr int CTC_SEL_THREADS = 256;
static constexpr int CTC_MAX_PBYTES = 160 * 1024;   // the prior P of a row's C classes (smem)

SB_DEVINL double ctc_lse(double a, double b) {
  const double mx = fmax(a, b), mn = fmin(a, b);
  return mx == -INFINITY ? -INFINITY : __dadd_rn(mx, log1p(exp(__dadd_rn(mn, -mx))));
}

// The search's CTC buffers, carved from one allocation (sb_s2s_ctc_state_size); R = B*K rows.
struct CtcBufs {
  double* a;       // [R] A_r
  double* gam;     // [2][R][2][T] gn, gb of each row; buffer (step & 1) holds the step's rows
  double* val;     // [R][M] candidate values
  double* anew;    // [R][M] A_r + P(r, c)
  double* psic;    // [R][M] psi(h_r + c)
  int* cls;        // [R][M] candidate classes, ascending
};

static size_t ctc_bytes(int K, int M, int T, int B) {
  const size_t R = (size_t)B * K;
  return sizeof(double) * (R + 4 * R * T + 3 * R * M) + sizeof(int) * R * M + 64;
}
static CtcBufs ctc_carve(void* buf, int K, int M, int T, int B) {
  const size_t R = (size_t)B * K;
  CtcBufs c;
  double* d = reinterpret_cast<double*>(buf);
  c.a = d; d += R;
  c.gam = d; d += 4 * R * T;
  c.val = d; d += R * M;
  c.anew = d; d += R * M;
  c.psic = d; d += R * M;
  c.cls = reinterpret_cast<int*>(d);
  return c;
}

struct CtcParams {
  const float* y;       // (B, T, C) CTC log-probabilities, blank C - 1
  const int* lens;      // (B) frames of each utterance, or null (all T)
  CtcBufs s;
  double lam;
  int T, M, C, K, B, start_tok;

  SB_DEVINL int frames(int b) const { return lens ? min(max(__ldg(lens + b), 1), T) : T; }
  // gn of row `row` (global row b*K + r) in buffer `parity`; gb follows at + T
  SB_DEVINL double* gam(int parity, int row) const {
    return s.gam + ((size_t)parity * B * K + row) * 2 * T;
  }
  SB_DEVINL float yv(int b, int t, int c) const { return __ldg(y + ((size_t)b * T + t) * C + c); }
};

// grid B: the root row of utterance b: A = 0, gn = -inf, gb_t = sum_{tau <= t} y_tau(blank)
__global__ void s2s_ctc_init_kernel(const CtcParams q) {
  const int b = blockIdx.x, row = b * q.K;
  double* g = q.gam(0, row);
  for (int t = threadIdx.x; t < q.T; t += blockDim.x) g[t] = -INFINITY;
  if (threadIdx.x != 0) return;
  q.s.a[row] = 0.0;
  const int Tb = q.frames(b);
  double acc = 0.0;
  for (int t = 0; t < q.T; ++t) {
    if (t < Tb) acc = __dadd_rn(acc, (double)q.yv(b, t, q.C - 1));
    g[q.T + t] = t < Tb ? acc : -INFINITY;
  }
}

struct S2sNoLm {
  static constexpr bool kLm = false;
};

template <class Fuse>
struct CtcCandArgs {
  BeamParams p;       // logp, st, nodes, node_cap, K, C, end_tok of utterance 0
  CtcParams q;
  const int* done;    // batch no-op flag
  Fuse fu;
};

// grid (K, B), CTC_MAXM threads: row r of utterance b
template <class Fuse>
__global__ void __launch_bounds__(CTC_MAXM) s2s_ctc_cand_kernel(const CtcCandArgs<Fuse> args) {
  extern __shared__ double ctc_smem[];
  __shared__ int s_cls[CTC_MAXM];
  __shared__ double s_p[CTC_MAXM];
  __shared__ int s_tk[CTC_MAXM];
  __shared__ double s_tp[CTC_MAXM];
  const CtcParams& q = args.q;
  if (args.done && *args.done) return;
  const int r = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  BeamParams p = args.p;
  p.st += b;
  p.nodes += (size_t)b * 2 * p.node_cap;
  const BeamState* st = p.st;
  const int nl = st->nlive;
  if (st->done || r >= nl) return;
  const int C = q.C, M = q.M, row = b * q.K + r;
  if constexpr (Fuse::kLm) {
    // every live row's context, as the selection resolves them: a few probes per row, next to the
    // C lookups below (resolving row r alone makes ptxas spill)
    args.fu.resolve(p, st, nl);
    __syncthreads();
  }
  // ---- the prior P(r, c) of every class, and the row's top M in class order ----
  double* pc = ctc_smem;                                   // [C]
  const float* lp = p.logp + (size_t)row * C;
  const double w_att = 1.0 - q.lam;
  for (int c = tid; c < C; c += CTC_MAXM) {
    double v = __dmul_rn(w_att, (double)__ldg(lp + c));
    if constexpr (Fuse::kLm) v = __dadd_rn(v, args.fu.lm_part(p, r, c));
    pc[c] = v;
  }
  __syncthreads();
  if (M == C) {
    for (int j = tid; j < M; j += CTC_MAXM) { s_cls[j] = j; s_p[j] = pc[j]; }
  } else {
    for (int k = 0; k < M; ++k) {
      double s;
      const int c = beam_take_first<CTC_MAXM>(pc, C, s);
      if (tid == 0) { s_tk[k] = c; s_tp[k] = s; }
    }
    __syncthreads();
    if (tid < M) {                                       // distinct classes: rank = position
      const int c = s_tk[tid];
      int rank = 0;
      for (int k = 0; k < M; ++k) rank += s_tk[k] < c ? 1 : 0;
      s_cls[rank] = c;
      s_p[rank] = s_tp[tid];
    }
  }
  __syncthreads();
  // ---- the prefix recursion, thread j for candidate j, over chunks of staged frames ----
  const int Tb = q.frames(b), blank = C - 1;
  const int last = st->token[r];
  const bool root = last == q.start_tok;
  const double* gp = q.gam(p.step & 1, row);
  double* s_pb = ctc_smem + ((C + 1) & ~1);               // [TCH] gb(h) at t - 1
  double* s_phi = s_pb + CTC_TCH;                          // [TCH] lse(gb, gn)(h) at t - 1
  float* s_yb = reinterpret_cast<float*>(s_phi + CTC_TCH); // [TCH] y_t(blank)
  float* s_yc = s_yb + CTC_TCH;                            // [TCH][M] y_t(c_j)
  const int j = tid;
  const int c = j < M ? s_cls[j] : 0;
  const bool rec = j < M && c != p.end_tok;
  double gn = -INFINITY, gb = -INFINITY, psi = -INFINITY;
  if (rec) {
    gn = root ? (double)q.yv(b, 0, c) : -INFINITY;
    psi = gn;
  }
  for (int t0 = 1; t0 < Tb; t0 += CTC_TCH) {
    const int n = min(CTC_TCH, Tb - t0);
    __syncthreads();                                     // the previous chunk has been consumed
    for (int i = tid; i < n; i += CTC_MAXM) {
      const double pb = gp[q.T + t0 + i - 1], pn = gp[t0 + i - 1];
      s_pb[i] = pb;
      s_phi[i] = ctc_lse(pb, pn);
      s_yb[i] = q.yv(b, t0 + i, blank);
    }
    for (int e = tid; e < n * M; e += CTC_MAXM) {
      const int i = e / M, k = e - i * M;
      s_yc[i * M + k] = q.yv(b, t0 + i, s_cls[k]);
    }
    __syncthreads();
    if (rec) {
      for (int i = 0; i < n; ++i) {
        const double phi = c == last ? s_pb[i] : s_phi[i];
        const double yc = (double)s_yc[i * M + j];
        const double ngn = __dadd_rn(ctc_lse(gn, phi), yc);
        gb = __dadd_rn(ctc_lse(gb, gn), (double)s_yb[i]);
        psi = ctc_lse(psi, __dadd_rn(phi, yc));
        gn = ngn;
      }
    }
  }
  if (j < M) {
    if (c == p.end_tok) psi = ctc_lse(gp[Tb - 1], gp[q.T + Tb - 1]);
    const size_t o = (size_t)row * M + j;
    const double an = __dadd_rn(q.s.a[row], s_p[j]);
    q.s.cls[o] = c;
    q.s.anew[o] = an;
    q.s.psic[o] = psi;
    q.s.val[o] = __dadd_rn(an, __dmul_rn(q.lam, psi));
  }
}

// grid B, CTC_SEL_THREADS threads: utterance b's selection over its K*M list, the bookkeeping and
// A' of the new rows (psi' is in their score)
__global__ void __launch_bounds__(CTC_SEL_THREADS) s2s_ctc_select_kernel(const BeamParams pb,
                                                                         const CtcParams q) {
  extern __shared__ double sel_smem[];                     // [K * M]
  __shared__ int sel_idx[2 * BM_MAXK];
  __shared__ double sel_sc[2 * BM_MAXK];
  __shared__ int live_src[BM_MAXK];
  const int b = blockIdx.x, tid = threadIdx.x;
  const BeamParams p = pb.of(b);
  BeamState* st = p.st;
  if (st->done) return;
  const int K = p.K, M = q.M, nl = st->nlive, u0 = b * K;
  const size_t l0 = (size_t)u0 * M;
  for (int i = tid; i < K * M; i += CTC_SEL_THREADS)
    sel_smem[i] = i / M < nl ? q.s.val[l0 + i] : nan("");
  __syncthreads();
  const int want = min(2 * K, nl * M);
  for (int k = 0; k < want; ++k) {
    double bs;
    const int bi = beam_take_first<CTC_SEL_THREADS>(sel_smem, K * M, bs);
    if (tid == 0) { sel_idx[k] = bi; sel_sc[k] = bs; }
  }
  if (tid == 0) beam_bookkeep(p, sel_idx, sel_sc, want, M, q.s.cls + l0, live_src);
  __syncthreads();
  if (tid < st->nlive) q.s.a[u0 + tid] = q.s.anew[l0 + live_src[tid]];
}

// grid B, 32 K threads: warp k < nlive computes the vectors of utterance b's new row k, which
// continues row parent_row[k] (node pn) with class c = token[k], into the other buffer.  Per chunk
// of 32 frames the lanes stage Phi_{t-1} (from the parent's vectors), y_t(c) and y_t(blank) in
// shared memory; lane 0 runs the recursion over them, and the lanes store the chunk.
__global__ void __launch_bounds__(32 * BM_MAXK) s2s_ctc_extend_kernel(const BeamParams pb,
                                                                      const CtcParams q) {
  __shared__ double s_phi[BM_MAXK][32], s_gn[BM_MAXK][32], s_gb[BM_MAXK][32];
  __shared__ float s_yc[BM_MAXK][32], s_yb[BM_MAXK][32];
  const int b = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31, u0 = b * pb.K;
  const BeamParams p = pb.of(b);
  const BeamState* st = p.st;
  if (st->done || k >= st->nlive) return;                 // whole warps
  const int node = st->node[k], pn = p.nodes[2 * node];
  const int c = st->token[k], last = p.nodes[2 * pn + 1], blank = q.C - 1;
  const bool root = p.nodes[2 * pn] < 0;
  const int par = p.step & 1, Tb = q.frames(b);
  const double* gp = q.gam(par, u0 + p.parent_row[k]);
  double* g = q.gam(par ^ 1, u0 + k);
  double gn = root ? (double)q.yv(b, 0, c) : -INFINITY, gb = -INFINITY;
  if (lane == 0) { g[0] = gn; g[q.T] = gb; }
  for (int t0 = 1; t0 < Tb; t0 += 32) {
    const int n = min(32, Tb - t0), t = t0 + lane;
    if (lane < n) {
      const double pbv = gp[q.T + t - 1];
      s_phi[k][lane] = c == last ? pbv : ctc_lse(pbv, gp[t - 1]);
      s_yc[k][lane] = q.yv(b, t, c);
      s_yb[k][lane] = q.yv(b, t, blank);
    }
    __syncwarp();
    if (lane == 0) {
      for (int i = 0; i < n; ++i) {
        const double ngn = __dadd_rn(ctc_lse(gn, s_phi[k][i]), (double)s_yc[k][i]);
        gb = __dadd_rn(ctc_lse(gb, gn), (double)s_yb[k][i]);
        gn = ngn;
        s_gn[k][i] = gn;
        s_gb[k][i] = gb;
      }
    }
    __syncwarp();
    if (lane < n) { g[t] = s_gn[k][lane]; g[q.T + t] = s_gb[k][lane]; }
    __syncwarp();
  }
}

}  // namespace sb

using namespace sb;

extern "C" int sb_s2s_ctc_state_size(int K, int M, int T, int B, size_t* bytes) {
  if (!bytes || K <= 0 || M <= 0 || T <= 0 || B <= 0) return SB_ERR_INVALID;
  *bytes = ctc_bytes(K, M, T, B);
  return SB_OK;
}

// the checks every CTC entry point shares, and the parameters they describe
static int ctc_params(CtcParams* q, const float* ctc_logp, const int* lens, void* ctc_state,
                      size_t ctc_state_bytes, int K, int C, int M, int T, int start_tok,
                      int end_tok, double ctc_weight, int B) {
  if (!ctc_logp || !ctc_state) return SB_ERR_INVALID;
  if (B <= 0 || K <= 0 || T < 1 || C < 2 || M < 1 || M > C) return SB_ERR_INVALID;
  if (!(ctc_weight > 0.0 && ctc_weight < 1.0)) return SB_ERR_INVALID;
  if (end_tok != C - 1 || start_tok != C) return SB_ERR_INVALID;   // blank = end = C - 1
  if (K > BM_MAXK || M > CTC_MAXM || B > 65535) return SB_ERR_UNSUPPORTED;
  if (ctc_state_bytes < ctc_bytes(K, M, T, B)) return SB_ERR_WORKSPACE;
  q->y = ctc_logp; q->lens = lens; q->s = ctc_carve(ctc_state, K, M, T, B);
  q->lam = ctc_weight; q->T = T; q->M = M; q->C = C; q->K = K; q->B = B; q->start_tok = start_tok;
  return SB_OK;
}

extern "C" int sb_s2s_ctc_init(const float* ctc_logp, const int* lens, void* ctc_state,
                               size_t ctc_state_bytes, int K, int C, int M, int T, int start_tok,
                               int end_tok, double ctc_weight, int B, void* stream_) {
  CtcParams q;
  const int rc = ctc_params(&q, ctc_logp, lens, ctc_state, ctc_state_bytes, K, C, M, T, start_tok,
                            end_tok, ctc_weight, B);
  if (rc != SB_OK) return rc;
  s2s_ctc_init_kernel<<<B, 128, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(q);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

static size_t ctc_cand_smem(int C, int M) {
  return sizeof(double) * ((size_t)((C + 1) & ~1) + 2 * CTC_TCH) +
         sizeof(float) * (size_t)CTC_TCH * (1 + M);
}

template <class Fuse>
static int ctc_cand_launch(const CtcCandArgs<Fuse>& a, int K, int B, cudaStream_t stream) {
  const size_t smem = ctc_cand_smem(a.q.C, a.q.M);
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(s2s_ctc_cand_kernel<Fuse>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)smem) != cudaSuccess)
    return SB_ERR_CUDA;
  s2s_ctc_cand_kernel<Fuse><<<dim3(K, B), CTC_MAXM, smem, stream>>>(a);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

// the checks and parameters of the candidate entry points, for the launch of a
// CtcCandArgs<Fuse> a whose fusion policy the caller fills
template <class Fuse>
static int ctc_cand_args(CtcCandArgs<Fuse>* a, const float* logp, const float* ctc_logp,
                         const int* lens, const void* state, const int* nodes, int node_cap,
                         void* ctc_state, size_t ctc_state_bytes, int K, int C, int M, int T,
                         int start_tok, int end_tok, double ctc_weight, int step, const int* stop,
                         int B) {
  if (!logp || !state || !nodes || !stop || node_cap <= 0 || step < 0) return SB_ERR_INVALID;
  const int rc = ctc_params(&a->q, ctc_logp, lens, ctc_state, ctc_state_bytes, K, C, M, T,
                            start_tok, end_tok, ctc_weight, B);
  if (rc != SB_OK) return rc;
  if ((size_t)C * sizeof(double) > CTC_MAX_PBYTES) return SB_ERR_UNSUPPORTED;
  BeamParams p = {};
  p.logp = logp;
  p.st = reinterpret_cast<BeamState*>(const_cast<void*>(state));
  p.nodes = const_cast<int*>(nodes);
  p.node_cap = node_cap; p.K = K; p.C = C; p.end_tok = end_tok; p.step = step; p.B = B;
  a->p = p;
  a->done = stop + 1;
  return SB_OK;
}

extern "C" int sb_s2s_ctc_candidates(const float* logp, const float* ctc_logp, const int* lens,
                                     const void* state, const int* nodes, int node_cap,
                                     void* ctc_state, size_t ctc_state_bytes, int K, int C, int M,
                                     int T, int start_tok, int end_tok, double ctc_weight,
                                     int step, const int* stop, int B, const SbNgramLm* lm,
                                     double lm_weight, double insertion_bonus, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (lm) {
    CtcCandArgs<S2sLmFuse> a;
    int rc = ctc_cand_args(&a, logp, ctc_logp, lens, state, nodes, node_cap, ctc_state,
                           ctc_state_bytes, K, C, M, T, start_tok, end_tok, ctc_weight, step,
                           stop, B);
    if (rc != SB_OK) return rc;
    rc = beam_lm_fuse(lm, lm_weight, insertion_bonus, C, &a.fu);
    if (rc != SB_OK) return rc;
    return ctc_cand_launch(a, K, B, stream);
  }
  CtcCandArgs<S2sNoLm> a;
  const int rc = ctc_cand_args(&a, logp, ctc_logp, lens, state, nodes, node_cap, ctc_state,
                               ctc_state_bytes, K, C, M, T, start_tok, end_tok, ctc_weight, step,
                               stop, B);
  if (rc != SB_OK) return rc;
  if (lm_weight != 0.0 || insertion_bonus != 0.0) return SB_ERR_INVALID;
  return ctc_cand_launch(a, K, B, stream);
}

extern "C" int sb_s2s_ctc_candidates_wordlm(const float* logp, const float* ctc_logp,
                                            const int* lens, const void* state, const int* nodes,
                                            int node_cap, void* ctc_state, size_t ctc_state_bytes,
                                            int K, int C, int M, int T, int start_tok,
                                            int end_tok, double ctc_weight, int step,
                                            const int* stop, int B, const SbWordLm* lm,
                                            double lm_weight, double insertion_bonus,
                                            double oov_penalty, int* word_nodes, void* stream_) {
  CtcCandArgs<S2sWordLmFuse> a;
  int rc = beam_wordlm_fuse(lm, lm_weight, insertion_bonus, oov_penalty, C, end_tok, word_nodes,
                            nodes, &a.fu);
  if (rc != SB_OK) return rc;
  rc = ctc_cand_args(&a, logp, ctc_logp, lens, state, nodes, node_cap, ctc_state,
                     ctc_state_bytes, K, C, M, T, start_tok, end_tok, ctc_weight, step, stop, B);
  if (rc != SB_OK) return rc;
  return ctc_cand_launch(a, K, B, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int sb_s2s_ctc_select_batch(const float* ctc_logp, const int* lens, void* ctc_state,
                                       size_t ctc_state_bytes, void* state, double* c_scores,
                                       int* nodes, int* parent_row, int* tok_next,
                                       int* out_tokens, int K, int C, int M, int T, int start_tok,
                                       int end_tok, double ctc_weight, int step, int max_len,
                                       int node_cap, int c_cap, int* stop, int B, void* stream_) {
  if (!state || !c_scores || !nodes || !parent_row || !tok_next || !out_tokens || !stop ||
      step < 0)
    return SB_ERR_INVALID;
  CtcParams q;
  const int rc = ctc_params(&q, ctc_logp, lens, ctc_state, ctc_state_bytes, K, C, M, T,
                            start_tok, end_tok, ctc_weight, B);
  if (rc != SB_OK) return rc;
  BeamParams p;
  p.logp = ctc_logp; p.st = reinterpret_cast<BeamState*>(state); p.c_scores = c_scores;
  p.nodes = nodes; p.parent_row = parent_row; p.tok_next = tok_next; p.out_tokens = out_tokens;
  p.stop = stop;
  p.K = K; p.C = C; p.end_tok = end_tok; p.step = step; p.max_len = max_len;
  p.node_cap = node_cap; p.c_cap = c_cap; p.B = B;
  const size_t smem = (size_t)K * M * sizeof(double);    // <= 32 KB
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  s2s_ctc_select_kernel<<<B, CTC_SEL_THREADS, smem, stream>>>(p, q);
  s2s_ctc_extend_kernel<<<B, 32 * K, 0, stream>>>(p, q);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
