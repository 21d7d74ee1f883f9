// sb_rnnt_decode_static: transducer beam search over a PRECOMPUTED (teacher-forced) lattice, on the
// GPU, one CTA per utterance.
//
// Replaces `transducer.decoders.decode_static(lp, beam_size, blank)` of the un-vendored
// awni/transducer (imported at speech/models/transducer_model.py:10, called per utterance on a
// host numpy array at :92-101).  The dependency's source is not available, so the algorithm is
// the standard transducer beam search (Graves 2012, section 3) restricted to a static lattice:
// because lp[t, u, :] was computed with teacher forcing, the prediction-network state of a
// hypothesis is the number u of labels it has emitted.  It is restated in oracle/
// decode_static_ref.py (the CPU oracle, pinned by exhaustive enumeration on tiny lattices); this
// kernel reproduces that restatement step for step, including its tie order:
//   per frame t:  frontier = beam; done = {}
//     repeat: every frontier hypothesis (in order) adds score + lp[t,u,blank] to done[hyp]
//             (log-sum-exp when the hypothesis is already there: prefix merging);
//             every (hypothesis i, label k != blank) with u+1 < U is a candidate
//             score + lp[t,u,k]; the next frontier = the beam_size best candidates by
//             (score desc, i*V + k asc) = a stable descending sort of the candidate list
//     beam = the beam_size best of done by (score desc, insertion order asc)
//   result = beam[0] after the last frame.
// Both selections and the trie of hypotheses (prefix merging compares node ids) are those of
// beam.cuh; the rounds themselves are tsearch.cuh's, shared with the label-free search
// (rnnt_search.cu).  Scores are float64, as Python floats.
// Roofline: HBM-nominal (the lattice is read once); latency-bound by the T x U serial expansion.
//
// sb_rnnt_decode_static_shortlist: the same search from per-node shortlists instead of the full
// lattice (sb_rnnt_shortlist_rows, csrc/joint_vocab.cu): for node (t, u) the blank's lp, the kp
// best non-blank classes as (lp, k) sorted by (lp desc, k asc), and beta = the (kp+1)-th lp in
// that order (-inf when there is none).  Everything but the label expansion is the kernel above.
// The expansion is a K-way merge: K rounds of an arg-max over the heads of the frontier's lists,
// with the full search's order (score desc, i asc, k asc).
//   Scores are s_q = fr_s + (double)lp_q.  Double addition is monotone, so s_q is non-increasing
//   along a list; but distinct float32 lp can round to the same s, and the full search takes such
//   equal-score entries in class order.  So the head of list i is the smallest unconsumed class in
//   the run of equal s that holds its first unconsumed position (a 64-bit mask per hypothesis
//   records what was taken); the rank between lists only needs (s, i).
//   A hypothesis with fr_s = -inf scores -inf on every class: its candidates are the non-blank
//   classes in index order, and it reads no list.
// Exactness.  A selection (s, k) from list i is what the full search takes unless a class left
// out of the list ties with it on s and has a smaller k.  Left-out classes have lp <= beta <= every
// listed lp, so by monotonicity one ties only if fr_s + beta == s.  Given that:
//   - left-out classes with lp == beta have larger k than every listed entry with lp == beta (the
//     list is the head of the (lp desc, k asc) order), so they are safe when the selected lp ==
//     beta, and may precede it when the selected lp > beta;
//   - left-out classes with lp < beta have lp <= nextafterf(beta, -inf) and any k; they tie only
//     if fr_s + nextafterf(beta, -inf) == s as well (never when beta = -inf: nothing lies below).
// The kernel counts every selection that fails either test in out_flags[b]; the caller re-runs
// flagged utterances from longer lists.  Both tests need two distinct float32 values to round to
// one float64 sum, i.e. |fr_s| of roughly 2^29 times their gap, so real lattices never raise it.
// A hypothesis takes at most K of its entries, so kp >= K lists are never exhausted while a
// left-out class could still follow.
#include "tsearch.cuh"
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int TD_THREADS = 128;
static constexpr int TD_MAX_BEAM = 32;
static constexpr int TD_MAX_KP = 64;
static constexpr size_t TD_SMEM_MAX = 200 * 1024;

struct TdParams {
  const float* lp;      // (B, T, U1, V) log-probabilities (full lattice)
  const float* sl_val;  // (B, T, U1, kp) shortlisted log-probabilities (shortlist search)
  const int* sl_idx;    // (B, T, U1, kp) their classes, -1 past V-1 entries
  const float* sl_meta; // (B, T, U1, 2) {blank lp, beta}
  const int* tlens;     // (B) frames to search (<= T)
  const int* ulens;     // (B) lattice rows U = labels + 1 (<= U1)
  BeamTrie trie;        // utterance 0 of B
  double* done_score;   // (B, done_cap)
  int* done_node;       // (B, done_cap)
  int* done_len;        // (B, done_cap)
  int* out_labels;      // (B, U1)
  int* out_lens;        // (B)
  double* out_scores;   // (B) log-probability of the best hypothesis
  int* out_flags;       // (B) unproven shortlist selections (shortlist search)
  int B, T, U1, V, K, kp, blank, done_cap;
};

// the search of one utterance (blockIdx.x); SHORT: candidates from the shortlists
template <bool SHORT>
SB_DEVINL void td_search(const TdParams& p) {
  extern __shared__ unsigned char td_smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p.K, V = p.V;
  const int T = min(p.tlens[b], p.T), U = min(p.ulens[b], p.U1);
  double* cand = reinterpret_cast<double*>(td_smem);       // [K * V] (full lattice only)
  __shared__ double beam_s[TD_MAX_BEAM], fr_s[TD_MAX_BEAM], new_s[TD_MAX_BEAM];
  __shared__ int beam_n[TD_MAX_BEAM], beam_l[TD_MAX_BEAM];
  __shared__ int fr_n[TD_MAX_BEAM], fr_l[TD_MAX_BEAM];
  __shared__ int new_n[TD_MAX_BEAM], new_l[TD_MAX_BEAM], new_p[TD_MAX_BEAM], new_k[TD_MAX_BEAM];
  __shared__ int nbeam, nfr, ndone, round_id, nflag;

  const BeamTrie trie = p.trie.of(b);
  double* dscore = p.done_score + (size_t)b * p.done_cap;
  int* dnode = p.done_node + (size_t)b * p.done_cap;
  int* dlen = p.done_len + (size_t)b * p.done_cap;
  const float* lp = SHORT ? nullptr : p.lp + (size_t)b * p.T * p.U1 * V;
  const size_t node0 = (size_t)b * p.T * p.U1;             // batch-first node of (b, 0, 0)
  const TsNew nw{new_s, new_n, new_l, new_p, new_k};

  if (tid == 0) {
    nbeam = 1; beam_s[0] = 0.0; beam_n[0] = 0; beam_l[0] = 0;
    round_id = 0;
    nflag = 0;
  }
  trie.clear<TD_THREADS>();

  for (int t = 0; t < T; ++t) {
    if (tid < nbeam) { fr_s[tid] = beam_s[tid]; fr_n[tid] = beam_n[tid]; fr_l[tid] = beam_l[tid]; }
    if (tid == 0) { nfr = nbeam; ndone = 0; }
    __syncthreads();
    for (int level = 0; level < U; ++level) {
      // ---- 1. blank emissions into `done`, hypothesis by hypothesis (merging order matters) ----
      const int nf = nfr;
      ts_merge_blanks<TD_THREADS>(
          nf, fr_s, fr_n, fr_l, U,
          [&](int, int u) {
            const size_t node = (size_t)t * p.U1 + u;
            return SHORT ? p.sl_meta[2 * (node0 + node)] : lp[node * V + p.blank];
          },
          dscore, dnode, dlen, nullptr, 0, &ndone, p.done_cap);
      // ---- 2. label expansions: candidates (i, k), the K best form the next frontier ----
      const auto can_extend = [&](int i) { return fr_l[i] + 1 < U; };
      int nsel;
      if (!SHORT) {
        nsel = ts_expand_full<TD_THREADS>(
            cand, K, V, p.blank, nf, fr_s, fr_n, fr_l, can_extend,
            [&](int i, int k) { return lp[((size_t)t * p.U1 + fr_l[i]) * V + k]; }, trie,
            round_id, nw);
      } else {
        nsel = ts_expand_shortlist<float>(
            K, V, p.kp, p.blank, nf, fr_s, fr_n, fr_l, can_extend,
            [&](int i, const float** lv, const int** li, float* beta) {
              const size_t node = node0 + (size_t)t * p.U1 + fr_l[i];
              *lv = p.sl_val + node * p.kp;
              *li = p.sl_idx + node * p.kp;
              *beta = p.sl_meta[2 * node + 1];
            },
            trie, round_id, nw, &nflag);
      }
      if (nsel < 0) break;
      if (tid < nsel) { fr_s[tid] = new_s[tid]; fr_n[tid] = new_n[tid]; fr_l[tid] = new_l[tid]; }
      if (tid == 0) { nfr = nsel; ++round_id; }
      __syncthreads();
    }
    // ---- 3. beam = the K best of `done` ----
    const int nb = ts_select_done<TD_THREADS>(dscore, dnode, dlen, nullptr, ndone, K, beam_s,
                                              beam_n, beam_l, nullptr);
    if (tid == 0) nbeam = nb;
    __syncthreads();
  }

  if (tid == 0) {
    p.out_lens[b] = trie.backtrack(nbeam > 0 ? beam_n[0] : 0, p.out_labels + (size_t)b * p.U1);
    p.out_scores[b] = nbeam > 0 ? beam_s[0] : -INFINITY;
    if (SHORT) p.out_flags[b] = nflag;
  }
}

__global__ void __launch_bounds__(TD_THREADS) rnnt_decode_static_kernel(const TdParams p) {
  td_search<false>(p);
}

// (one CTA per SM is all a batch of utterances asks for; the bound lets ptxas keep every value of
// the merge in registers)
__global__ void __launch_bounds__(TD_THREADS, 1) rnnt_decode_static_shortlist_kernel(
    const TdParams p) {
  td_search<true>(p);
}

struct TdSizes { size_t node_cap, hcap, done_cap, total; };
static TdSizes td_sizes(int B, int T, int U1, int K) {
  TdSizes s;
  s.node_cap = (size_t)T * U1 * K + 2;
  s.hcap = (size_t)beam_pow2_cap(2 * s.node_cap);
  s.done_cap = (size_t)K * (U1 + 1) + 1;
  s.total = 1024 + (size_t)B * (2 * s.node_cap * sizeof(int) +
                                s.hcap * (sizeof(unsigned long long) + sizeof(int)) +
                                s.done_cap * (sizeof(double) + 2 * sizeof(int))) + 4096;
  return s;
}

static size_t td_full_smem(int beam_size, int V) { return (size_t)beam_size * V * sizeof(double) + 16; }

// checks shared by both searches; fills the workspace carve-up, shapes and outputs of p
static int td_setup(TdParams* p, const int* tlens, const int* ulens, int B, int T, int U1, int V,
                    int beam_size, int blank, int* out_labels, int* out_lens, double* out_scores,
                    void* workspace, size_t workspace_bytes) {
  if (!tlens || !ulens || !out_labels || !out_lens || !out_scores || !workspace)
    return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || U1 <= 0 || V <= 0 || blank < 0 || blank >= V || beam_size <= 0)
    return SB_ERR_INVALID;
  if (beam_size > TD_MAX_BEAM) return SB_ERR_UNSUPPORTED;
  const TdSizes sz = td_sizes(B, T, U1, beam_size);
  if (workspace_bytes < sz.total) return SB_ERR_WORKSPACE;
  uintptr_t w = (reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255;
  p->trie.keys = reinterpret_cast<unsigned long long*>(w);
  w += (size_t)B * sz.hcap * sizeof(unsigned long long);
  p->done_score = reinterpret_cast<double*>(w);
  w += (size_t)B * sz.done_cap * sizeof(double);
  p->trie.vals = reinterpret_cast<int*>(w);
  w += (size_t)B * sz.hcap * sizeof(int);
  p->trie.nodes = reinterpret_cast<int*>(w);
  w += (size_t)B * 2 * sz.node_cap * sizeof(int);
  p->done_node = reinterpret_cast<int*>(w);
  w += (size_t)B * sz.done_cap * sizeof(int);
  p->done_len = reinterpret_cast<int*>(w);
  p->lp = nullptr; p->sl_val = nullptr; p->sl_idx = nullptr; p->sl_meta = nullptr;
  p->out_flags = nullptr;
  p->tlens = tlens; p->ulens = ulens;
  p->out_labels = out_labels; p->out_lens = out_lens; p->out_scores = out_scores;
  p->B = B; p->T = T; p->U1 = U1; p->V = V; p->K = beam_size; p->kp = 0; p->blank = blank;
  p->trie.cap = (int)sz.hcap; p->trie.node_cap = (int)sz.node_cap; p->done_cap = (int)sz.done_cap;
  return SB_OK;
}

}  // namespace sb

using namespace sb;

extern "C" int sb_rnnt_decode_static_workspace_size(int B, int T, int U1, int beam_size,
                                                    size_t* bytes) {
  if (!bytes || B <= 0 || T <= 0 || U1 <= 0 || beam_size <= 0) return SB_ERR_INVALID;
  *bytes = td_sizes(B, T, U1, beam_size).total;
  return SB_OK;
}

extern "C" int sb_rnnt_decode_static_fits(int beam_size, int V) {
  return beam_size > 0 && beam_size <= TD_MAX_BEAM && V > 0 &&
         td_full_smem(beam_size, V) <= TD_SMEM_MAX;
}

extern "C" int sb_rnnt_decode_static(const float* lp, const int* tlens, const int* ulens, int B,
                                     int T, int U1, int V, int beam_size, int blank,
                                     int* out_labels, int* out_lens, double* out_scores,
                                     void* workspace, size_t workspace_bytes, void* stream_) {
  if (!lp) return SB_ERR_INVALID;
  TdParams p;
  const int rc = td_setup(&p, tlens, ulens, B, T, U1, V, beam_size, blank, out_labels, out_lens,
                          out_scores, workspace, workspace_bytes);
  if (rc != SB_OK) return rc;
  const size_t smem = td_full_smem(beam_size, V);
  if (smem > TD_SMEM_MAX) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (smem > 40 * 1024 &&
      cudaFuncSetAttribute(rnnt_decode_static_kernel,
                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return SB_ERR_CUDA;
  p.lp = lp;
  rnnt_decode_static_kernel<<<B, TD_THREADS, smem, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_decode_static_shortlist(const float* sl_val, const int* sl_idx,
                                               const float* sl_meta, int kp, const int* tlens,
                                               const int* ulens, int B, int T, int U1, int V,
                                               int beam_size, int blank, int* out_labels,
                                               int* out_lens, double* out_scores, int* out_flags,
                                               void* workspace, size_t workspace_bytes,
                                               void* stream_) {
  if (!sl_val || !sl_idx || !sl_meta || !out_flags) return SB_ERR_INVALID;
  TdParams p;
  const int rc = td_setup(&p, tlens, ulens, B, T, U1, V, beam_size, blank, out_labels, out_lens,
                          out_scores, workspace, workspace_bytes);
  if (rc != SB_OK) return rc;
  if (kp < beam_size) return SB_ERR_INVALID;
  if (kp > TD_MAX_KP) return SB_ERR_UNSUPPORTED;
  p.sl_val = sl_val; p.sl_idx = sl_idx; p.sl_meta = sl_meta; p.kp = kp; p.out_flags = out_flags;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  rnnt_decode_static_shortlist_kernel<<<B, TD_THREADS, 0, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
