// sb_ctc_prefix_beam: CTC prefix beam search on the GPU, one CTA per utterance.
//
// Replaces speech/models/ctc_decoder.py:38-113 `decode(probs, beam_size, blank)` (pure-Python dict
// beam, called serially per utterance from CTC.infer, ctc_model.py:55-60).  The search is restated
// so that hypotheses come out IDENTICAL to the reference, including its tie-breaks:
//   * beam entries carry (p_blank, p_non_blank) in float64 log space, as the reference's Python
//     floats; log-sum-exp is evaluated in the reference's argument order;
//   * prefixes are nodes (parent, symbol) of a per-utterance trie, so "prefix + s is already in
//     the beam" (the merge case, ctc_decoder.py:84-103) is an integer comparison;
//   * pruning = repeated arg-max over (score desc, first-touch rank asc): the reference sorts
//     a dict's items with a stable sort, so ties keep dict insertion order, which is the order
//     of first touch in its `for s in vocab: for prefix in beam:` loops (ctc_decoder.py:65-103).
// Input is log-probabilities (the host wrapper applies the same float32 log as the reference).
//
// Roofline: HBM-nominal (reads T*S floats per utterance), in practice latency-bound by the
// T-serial beam update; decode is not on the training path.
#include "common.cuh"
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int DEC_THREADS = 128;
static constexpr int DEC_MAX_BEAM = 32;

struct DecParams {
  const float* logp;   // (B, T, S)
  const int* lens;     // (B) frames per utterance (<= T)
  int* nodes;          // (B, 2*(T*K+1)) trie arena: parent, symbol
  unsigned long long* hkeys;  // (B, hcap) (parent, symbol) -> node id map: keys (0 = empty)
  int* hvals;                 // (B, hcap)
  int hcap;                   // power of two >= 2*(T*K+1)
  int* out_labels;     // (B, T)
  int* out_lens;       // (B)
  double* out_scores;  // (B)  negative log-likelihood of the best prefix
  int B, T, S, K, blank;
};

__device__ __forceinline__ double d_neg_inf() { return -INFINITY; }

// logsumexp(a, b[, c]) with the reference's evaluation order (ctc_decoder.py:27-36)
__device__ __forceinline__ double lse2d(double a, double b) {
  const double m = fmax(a, b);
  if (m == d_neg_inf()) return d_neg_inf();
  return m + log(exp(a - m) + exp(b - m));
}
__device__ __forceinline__ double lse3d(double a, double b, double c) {
  const double m = fmax(fmax(a, b), c);
  if (m == d_neg_inf()) return d_neg_inf();
  return m + log((exp(a - m) + exp(b - m)) + exp(c - m));
}

struct Beam {
  double pb[DEC_MAX_BEAM];
  double pnb[DEC_MAX_BEAM];
  int node[DEC_MAX_BEAM];    // trie node of the prefix (0 = empty prefix)
  int last[DEC_MAX_BEAM];    // last symbol (-1 for the empty prefix)
  int parent[DEC_MAX_BEAM];  // trie node of prefix[:-1]
  int size;
};

// value of the candidate "beam entry j keeps its prefix" at this frame
__device__ void stay_value(const Beam& bm, int j, const float* lp, int blank, int K, double& npb,
                           double& npnb, int& rank) {
  const double pblank = (double)lp[blank];
  npb = lse3d(d_neg_inf(), bm.pb[j] + pblank, bm.pnb[j] + pblank);
  npnb = d_neg_inf();
  rank = blank * 2 * K + 2 * j;
  const int s = bm.last[j];
  if (s >= 0) {
    const double p = (double)lp[s];
    // is the parent prefix in the beam?  then extending it by s lands on this entry
    int pi = -1;
    for (int i = 0; i < bm.size; ++i)
      if (bm.node[i] == bm.parent[j]) { pi = i; break; }
    const int self_rank = s * 2 * K + 2 * j + 1;
    if (pi >= 0) {
      const int par_rank = s * 2 * K + 2 * pi;
      const bool rep = (bm.last[pi] == s);
      if (pi < j) {
        npnb = rep ? lse2d(npnb, bm.pb[pi] + p) : lse3d(npnb, bm.pb[pi] + p, bm.pnb[pi] + p);
        npnb = lse2d(npnb, bm.pnb[j] + p);
      } else {
        npnb = lse2d(npnb, bm.pnb[j] + p);
        npnb = rep ? lse2d(npnb, bm.pb[pi] + p) : lse3d(npnb, bm.pb[pi] + p, bm.pnb[pi] + p);
      }
      rank = min(rank, min(self_rank, par_rank));
    } else {
      npnb = lse2d(npnb, bm.pnb[j] + p);
      rank = min(rank, self_rank);
    }
  }
}

// value of the candidate "beam entry i extended by symbol s" (s != blank); returns false when the
// extended prefix is already a beam entry (then it is accounted for by that entry's stay_value)
__device__ bool ext_value(const Beam& bm, int i, int s, const float* lp, int K, double& npnb,
                          int& rank) {
  for (int j = 0; j < bm.size; ++j)
    if (bm.last[j] == s && bm.parent[j] == bm.node[i] && bm.node[j] != 0) return false;
  const double p = (double)lp[s];
  if (s != bm.last[i]) npnb = lse3d(d_neg_inf(), bm.pb[i] + p, bm.pnb[i] + p);
  else npnb = lse2d(d_neg_inf(), bm.pb[i] + p);
  rank = s * 2 * K + 2 * i;
  return true;
}

// Candidate c of a frame, numbered as the full scan numbers them: c < K*S is "entry c / S extended
// by symbol c % S", c = K*S + j is "entry j keeps its prefix".  Returns false for a candidate that
// does not exist (no such entry, the blank as an extension, or an extension that is a beam entry).
__device__ __forceinline__ bool cand_value(const Beam& cur, int c, const float* lp, int K, int S,
                                           int blank, double& sc, int& rk) {
  sc = d_neg_inf();
  rk = 0x7fffffff;
  const int nb = cur.size;
  if (c < K * S) {
    const int i = c / S, s = c - i * S;
    if (i < nb && s != blank) {
      double x;
      const bool ok = ext_value(cur, i, s, lp, K, x, rk);
      if (ok) sc = x;  // logsumexp(-inf, x) == x exactly
      return ok;
    }
    return false;
  }
  const int j = c - K * S;
  if (j >= nb) return false;
  double npb, npnb;
  stay_value(cur, j, lp, blank, K, npb, npnb, rk);
  sc = lse2d(npb, npnb);
  return true;
}

// (score desc, rank asc): the order of the reference's stable sort
__device__ __forceinline__ bool dec_better(double s, int r, double bs, int br) {
  return s > bs || (s == bs && r < br);
}

// Block arg-max of the threads' (bs, br, bc) (bc < 0: none); the winner ends up in thread 0.
__device__ __forceinline__ void dec_block_argmax(double& bs, int& br, int& bc, double* red_s,
                                                 int* red_r, int* red_c) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double os = __shfl_xor_sync(0xffffffffu, bs, o);
    const int orr = __shfl_xor_sync(0xffffffffu, br, o);
    const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
    if (oc >= 0 && (bc < 0 || os > bs || (os == bs && orr < br))) { bs = os; br = orr; bc = oc; }
  }
  if ((tid & 31) == 0) { red_s[tid >> 5] = bs; red_r[tid >> 5] = br; red_c[tid >> 5] = bc; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < DEC_THREADS / 32; ++w) {
      if (red_c[w] >= 0 && (bc < 0 || red_s[w] > bs || (red_s[w] == bs && red_r[w] < br))) {
        bs = red_s[w]; br = red_r[w]; bc = red_c[w];
      }
    }
  }
}

// Per-utterance search state in global memory: trie arena and (parent, symbol) -> node map.
struct DecUtt {
  int* nodes;
  unsigned long long* hkeys;
  int* hvals;
};

__device__ __forceinline__ DecUtt dec_begin(const DecParams& p, Beam* beams) {
  const int b = blockIdx.x, tid = threadIdx.x;
  DecUtt u;
  u.nodes = p.nodes + (size_t)b * 2 * ((size_t)p.T * p.K + 1);
  u.hkeys = p.hkeys + (size_t)b * p.hcap;
  u.hvals = p.hvals + (size_t)b * p.hcap;
  // Node ids must be CANONICAL over the whole utterance: a prefix that is pruned and later
  // re-created has to get its old id back, because surviving descendants still name it as parent.
  for (int k = tid; k < p.hcap; k += DEC_THREADS) u.hkeys[k] = 0ull;

  if (tid == 0) {
    beams[0].size = 1;
    beams[0].pb[0] = 0.0;
    beams[0].pnb[0] = d_neg_inf();
    beams[0].node[0] = 0;
    beams[0].last[0] = -1;
    beams[0].parent[0] = -1;
    u.nodes[0] = -1;
    u.nodes[1] = -1;
  }
  __syncthreads();
  return u;
}

// Materialise the pruned beam of frame t from the ns selected candidates (full-scan numbering).
__device__ __forceinline__ void dec_commit(const DecParams& p, const DecUtt& u, const Beam& cur, Beam& nxt,
                           const int* sel, int ns, const float* lp, int t) {
  const int tid = threadIdx.x, K = p.K, S = p.S;
  if (tid < ns) {
    const int c = sel[tid];
    if (c < K * S) {
      const int i = c / S, s = c - i * S;
      double x; int rk;
      ext_value(cur, i, s, lp, K, x, rk);
      // find-or-insert (parent node, symbol) in the utterance's hash map
      const unsigned long long key =
          ((unsigned long long)(unsigned int)cur.node[i] << 32) | (unsigned int)(s + 1);
      unsigned int h = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 32) & (p.hcap - 1);
      int id = -1;
      for (int probe = 0; probe < p.hcap; ++probe) {
        const unsigned long long k = u.hkeys[h];
        if (k == key) { id = u.hvals[h]; break; }
        if (k == 0ull) {
          const unsigned long long old = atomicCAS(&u.hkeys[h], 0ull, key);
          if (old == 0ull) {
            id = 1 + t * K + tid;
            u.hvals[h] = id;
            u.nodes[2 * id] = cur.node[i];
            u.nodes[2 * id + 1] = s;
            break;
          }
          if (old == key) { id = u.hvals[h]; break; }
        }
        h = (h + 1) & (p.hcap - 1);
      }
      nxt.pb[tid] = d_neg_inf();
      nxt.pnb[tid] = x;
      nxt.node[tid] = id;
      nxt.last[tid] = s;
      nxt.parent[tid] = cur.node[i];
    } else {
      const int j = c - K * S;
      double npb, npnb; int rk;
      stay_value(cur, j, lp, p.blank, K, npb, npnb, rk);
      nxt.pb[tid] = npb;
      nxt.pnb[tid] = npnb;
      nxt.node[tid] = cur.node[j];
      nxt.last[tid] = cur.last[j];
      nxt.parent[tid] = cur.parent[j];
    }
  }
  if (tid == 0) nxt.size = ns;
  __syncthreads();
}

// Best hypothesis of the final beam: back-track the trie.
__device__ __forceinline__ void dec_finish(const DecParams& p, const DecUtt& u, const Beam& fin) {
  if (threadIdx.x == 0) {
    const int b = blockIdx.x;
    int n = fin.node[0];
    int len = 0;
    for (int q = n; q > 0; q = u.nodes[2 * q]) ++len;
    int* out = p.out_labels + (size_t)b * p.T;
    int k = len;
    for (int q = n; q > 0; q = u.nodes[2 * q]) out[--k] = u.nodes[2 * q + 1];
    p.out_lens[b] = len;
    p.out_scores[b] = -lse2d(fin.pb[0], fin.pnb[0]);
  }
}

__global__ void __launch_bounds__(DEC_THREADS) ctc_prefix_beam_kernel(const DecParams p) {
  extern __shared__ unsigned char dec_smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p.K, S = p.S, T = min(p.lens[b], p.T);
  const int ncand = K * S + K;
  double* score = reinterpret_cast<double*>(dec_smem);             // [ncand]
  int* rank = reinterpret_cast<int*>(score + ncand);               // [ncand]
  unsigned char* live = reinterpret_cast<unsigned char*>(rank + ncand);  // [ncand]
  __shared__ Beam beams[2];
  __shared__ double red_s[DEC_THREADS / 32];
  __shared__ int red_r[DEC_THREADS / 32];
  __shared__ int red_c[DEC_THREADS / 32];
  __shared__ int sel[DEC_MAX_BEAM];
  __shared__ int nsel;

  int* nodes = p.nodes + (size_t)b * 2 * ((size_t)p.T * K + 1);
  unsigned long long* hkeys = p.hkeys + (size_t)b * p.hcap;
  int* hvals = p.hvals + (size_t)b * p.hcap;
  const float* logp = p.logp + (size_t)b * p.T * S;
  // Node ids must be CANONICAL over the whole utterance: a prefix that is pruned and later
  // re-created has to get its old id back, because surviving descendants still name it as parent.
  for (int k = tid; k < p.hcap; k += DEC_THREADS) hkeys[k] = 0ull;

  if (tid == 0) {
    beams[0].size = 1;
    beams[0].pb[0] = 0.0;
    beams[0].pnb[0] = d_neg_inf();
    beams[0].node[0] = 0;
    beams[0].last[0] = -1;
    beams[0].parent[0] = -1;
    nodes[0] = -1;
    nodes[1] = -1;
  }
  __syncthreads();

  for (int t = 0; t < T; ++t) {
    const Beam& cur = beams[t & 1];
    Beam& nxt = beams[(t & 1) ^ 1];
    const float* lp = logp + (size_t)t * S;
    const int nb = cur.size;
    // ---- 1. score every candidate ----
    for (int c = tid; c < ncand; c += DEC_THREADS) {
      double sc = d_neg_inf();
      int rk = 0x7fffffff;
      bool ok = false;
      if (c < K * S) {
        const int i = c / S, s = c - i * S;
        if (i < nb && s != p.blank) {
          double x;
          ok = ext_value(cur, i, s, lp, K, x, rk);
          if (ok) sc = x;  // logsumexp(-inf, x) == x exactly
        }
      } else {
        const int j = c - K * S;
        if (j < nb) {
          double npb, npnb;
          stay_value(cur, j, lp, p.blank, K, npb, npnb, rk);
          sc = lse2d(npb, npnb);
          ok = true;
        }
      }
      score[c] = sc;
      rank[c] = rk;
      live[c] = ok ? 1 : 0;
    }
    __syncthreads();
    // ---- 2. K rounds of arg-max by (score desc, rank asc) ----
    if (tid == 0) nsel = 0;
    for (int r = 0; r < K; ++r) {
      double bs = d_neg_inf();
      int br = 0x7fffffff, bc = -1;
      for (int c = tid; c < ncand; c += DEC_THREADS) {
        if (!live[c]) continue;
        const double sc = score[c];
        const int rk = rank[c];
        if (bc < 0 || sc > bs || (sc == bs && rk < br)) { bs = sc; br = rk; bc = c; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, bs, o);
        const int orr = __shfl_xor_sync(0xffffffffu, br, o);
        const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
        if (oc >= 0 && (bc < 0 || os > bs || (os == bs && orr < br))) { bs = os; br = orr; bc = oc; }
      }
      if ((tid & 31) == 0) { red_s[tid >> 5] = bs; red_r[tid >> 5] = br; red_c[tid >> 5] = bc; }
      __syncthreads();
      if (tid == 0) {
        for (int w = 1; w < DEC_THREADS / 32; ++w) {
          if (red_c[w] >= 0 && (bc < 0 || red_s[w] > bs || (red_s[w] == bs && red_r[w] < br))) {
            bs = red_s[w]; br = red_r[w]; bc = red_c[w];
          }
        }
        if (bc >= 0) { sel[nsel++] = bc; live[bc] = 0; }
      }
      __syncthreads();
    }
    // ---- 3. materialise the pruned beam ----
    const int ns = nsel;
    if (tid < ns) {
      const int c = sel[tid];
      if (c < K * S) {
        const int i = c / S, s = c - i * S;
        double x; int rk;
        ext_value(cur, i, s, lp, K, x, rk);
        // find-or-insert (parent node, symbol) in the utterance's hash map
        const unsigned long long key =
            ((unsigned long long)(unsigned int)cur.node[i] << 32) | (unsigned int)(s + 1);
        unsigned int h = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 32) & (p.hcap - 1);
        int id = -1;
        for (int probe = 0; probe < p.hcap; ++probe) {
          const unsigned long long k = hkeys[h];
          if (k == key) { id = hvals[h]; break; }
          if (k == 0ull) {
            const unsigned long long old = atomicCAS(&hkeys[h], 0ull, key);
            if (old == 0ull) {
              id = 1 + t * K + tid;
              hvals[h] = id;
              nodes[2 * id] = cur.node[i];
              nodes[2 * id + 1] = s;
              break;
            }
            if (old == key) { id = hvals[h]; break; }
          }
          h = (h + 1) & (p.hcap - 1);
        }
        nxt.pb[tid] = d_neg_inf();
        nxt.pnb[tid] = x;
        nxt.node[tid] = id;
        nxt.last[tid] = s;
        nxt.parent[tid] = cur.node[i];
      } else {
        const int j = c - K * S;
        double npb, npnb; int rk;
        stay_value(cur, j, lp, p.blank, K, npb, npnb, rk);
        nxt.pb[tid] = npb;
        nxt.pnb[tid] = npnb;
        nxt.node[tid] = cur.node[j];
        nxt.last[tid] = cur.last[j];
        nxt.parent[tid] = cur.parent[j];
      }
    }
    if (tid == 0) nxt.size = ns;
    __syncthreads();
  }

  // ---- best hypothesis: back-track the trie ----
  if (tid == 0) {
    const Beam& fin = beams[T & 1];
    int n = fin.node[0];
    int len = 0;
    for (int q = n; q > 0; q = nodes[2 * q]) ++len;
    int* out = p.out_labels + (size_t)b * p.T;
    int k = len;
    for (int q = n; q > 0; q = nodes[2 * q]) out[--k] = nodes[2 * q + 1];
    p.out_lens[b] = len;
    p.out_scores[b] = -lse2d(fin.pb[0], fin.pnb[0]);
  }
}

// ------------------------------------------------------------------------------------------------
// Shortlist form of the same search, for vocabularies whose K*S + K candidates do not fit in shared
// memory.  Results (hypotheses, lengths, float64 scores) are bit-identical to the full scan.
//
// Why a short list of symbols per frame suffices.  Fix beam entry i.  Its extension by a symbol
// s != last_i scores f_i(p_s) = lse(pb_i + p_s, pnb_i + p_s), non-decreasing in p_s, and its rank
// s*2K + 2i grows with s.  So, in the (score desc, rank asc) order of the selection, the extensions
// of i come in the order (p_s desc, s asc) of their symbols.  At most K - 1 of them do not exist
// (the extended prefix is already a beam entry) and at most K are selected.  Every selected
// extension of i therefore lies among the first 2K + 1 non-blank symbols of the frame in
// (p desc, s asc) order, or is last_i (a different formula, always scored).
//
// Rounding.  The computed float64 f_i is monotone only up to a few ulps, and when every entry's
// extensions tie at -inf the selection falls back on rank alone (s ascending, not p descending).
// So the kernel does not rely on the argument; it checks it each frame.  Every symbol left out has
// p_s <= p_min, the last shortlisted probability, so in exact arithmetic its score is at most
// f_i(p_min), and the computed score exceeds the exact one by a few ulps at most.  The frame's
// selection stands if the K-th selected candidate's score is finite and exceeds
//     U + 1e-12 * (1 + |U|),   U = max_i f_i(p_min) as computed
// (or U = -inf, when every left-out candidate scores -inf exactly).  The margin is about 10^4 times
// the rounding error of f.  Otherwise (fewer than K selected, a -inf K-th score, or a near tie at
// the bound) the frame is scored again by a full streamed scan: K rounds over all K*S + K
// candidates, each round taking the best candidate after the previous one.  Both ways select the
// full scan's K candidates in its order, with the same ext_value / stay_value arithmetic.
//
// The shortlist of every frame (2K + 1 ints, or S - 1 if fewer) comes from a pre-pass over the
// B*T rows (ctc_shortlist_kernel, one CTA per frame).
// ------------------------------------------------------------------------------------------------
static constexpr int DEC_SL_THREADS = 256;

// (p desc, s asc) order of the shortlist: true if (x, s) comes strictly after (px, ps)
__device__ __forceinline__ bool sl_after(float x, int s, float px, int ps) {
  return x < px || (x == px && s > ps);
}

// grid (T, B): shortlist[(b*T + t)*LS + j], j < L, for the frames t < lens[b]
__global__ void __launch_bounds__(DEC_SL_THREADS) ctc_shortlist_kernel(
    const float* __restrict__ logp, const int* __restrict__ lens, int* __restrict__ shortlist,
    int T, int S, int blank, int L, int LS) {
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  if (t >= min(lens[b], T)) return;
  __shared__ float red_x[DEC_SL_THREADS / 32];
  __shared__ int red_s[DEC_SL_THREADS / 32];
  __shared__ float prev_x;
  __shared__ int prev_s;
  const float* lp = logp + ((size_t)b * T + t) * S;
  int* out = shortlist + ((size_t)b * T + t) * LS;
  for (int j = 0; j < L; ++j) {
    const float px = j ? prev_x : 0.f;
    const int ps = j ? prev_s : -1;
    float bx = 0.f;
    int bsym = -1;
    for (int s = tid; s < S; s += DEC_SL_THREADS) {
      if (s == blank) continue;
      const float x = __ldg(lp + s);
      if (j && !sl_after(x, s, px, ps)) continue;
      if (bsym < 0 || !sl_after(x, s, bx, bsym)) { bx = x; bsym = s; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ox = __shfl_xor_sync(0xffffffffu, bx, o);
      const int os = __shfl_xor_sync(0xffffffffu, bsym, o);
      if (os >= 0 && (bsym < 0 || !sl_after(ox, os, bx, bsym))) { bx = ox; bsym = os; }
    }
    if ((tid & 31) == 0) { red_x[tid >> 5] = bx; red_s[tid >> 5] = bsym; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < DEC_SL_THREADS / 32; ++w)
        if (red_s[w] >= 0 && (bsym < 0 || !sl_after(red_x[w], red_s[w], bx, bsym))) {
          bx = red_x[w]; bsym = red_s[w];
        }
      out[j] = bsym;
      prev_x = bx;
      prev_s = bsym;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(DEC_THREADS, 1) ctc_prefix_beam_shortlist_kernel(
    const DecParams p, const int* __restrict__ shortlist, int L, int LS) {
  extern __shared__ unsigned char dec_smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p.K, S = p.S, T = min(p.lens[b], p.T);
  const int per = L + 1;                   // shortlist + last_i per entry
  const int ncand = K * per + K;
  double* score = reinterpret_cast<double*>(dec_smem);             // [ncand]
  int* rank = reinterpret_cast<int*>(score + ncand);               // [ncand]
  int* full = rank + ncand;                                        // [ncand] full-scan number
  unsigned char* live = reinterpret_cast<unsigned char*>(full + ncand);  // [ncand]
  __shared__ Beam beams[2];
  __shared__ double red_s[DEC_THREADS / 32];
  __shared__ int red_r[DEC_THREADS / 32];
  __shared__ int red_c[DEC_THREADS / 32];
  __shared__ int sel[DEC_MAX_BEAM];
  __shared__ int nsel;
  __shared__ double last_s;
  __shared__ int last_r;
  __shared__ int rescan;
  const bool complete = L >= S - 1;        // every non-blank symbol is on the list

  const DecUtt u = dec_begin(p, beams);
  const float* logp = p.logp + (size_t)b * p.T * S;

  for (int t = 0; t < T; ++t) {
    const Beam& cur = beams[t & 1];
    Beam& nxt = beams[(t & 1) ^ 1];
    const float* lp = logp + (size_t)t * S;
    const int* sl = shortlist + ((size_t)b * p.T + t) * LS;
    const int nb = cur.size;
    // ---- 1. score the shortlisted candidates ----
    for (int c = tid; c < ncand; c += DEC_THREADS) {
      double sc = d_neg_inf();
      int rk = 0x7fffffff, fc = -1;
      bool ok = false;
      if (c < K * per) {
        const int i = c / per, j = c - i * per;
        if (i < nb) {
          int s = j < L ? sl[j] : cur.last[i];
          if (j == L) {
            for (int q = 0; q < L && s >= 0; ++q)
              if (sl[q] == s) s = -1;        // already scored as a shortlisted symbol
          }
          if (s >= 0 && s != p.blank) {
            fc = i * S + s;
            ok = cand_value(cur, fc, lp, K, S, p.blank, sc, rk);
          }
        }
      } else {
        fc = K * S + (c - K * per);
        ok = cand_value(cur, fc, lp, K, S, p.blank, sc, rk);
      }
      score[c] = sc;
      rank[c] = rk;
      full[c] = fc;
      live[c] = ok ? 1 : 0;
    }
    __syncthreads();
    // ---- 2. K rounds of arg-max by (score desc, rank asc), as the full scan ----
    if (tid == 0) nsel = 0;
    for (int r = 0; r < K; ++r) {
      double bs = d_neg_inf();
      int br = 0x7fffffff, bc = -1;
      for (int c = tid; c < ncand; c += DEC_THREADS) {
        if (!live[c]) continue;
        const double sc = score[c];
        const int rk = rank[c];
        if (bc < 0 || sc > bs || (sc == bs && rk < br)) { bs = sc; br = rk; bc = c; }
      }
      dec_block_argmax(bs, br, bc, red_s, red_r, red_c);
      if (tid == 0 && bc >= 0) {
        sel[nsel++] = full[bc];
        live[bc] = 0;
        last_s = bs;
        last_r = br;
      }
      __syncthreads();
    }
    // ---- 3. check that no left-out candidate can reach the selection ----
    if (!complete && tid < 32) {
      const double pmin = (double)lp[sl[L - 1]];
      double U = d_neg_inf();
      if (tid < nb) U = lse3d(d_neg_inf(), cur.pb[tid] + pmin, cur.pnb[tid] + pmin);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) U = fmax(U, __shfl_xor_sync(0xffffffffu, U, o));
      if (tid == 0) {
        bool ok = nsel == K && last_s != d_neg_inf();
        if (ok && U != d_neg_inf()) ok = last_s > U + 1e-12 * (1.0 + fabs(U));
        rescan = ok ? 0 : 1;
      }
    }
    __syncthreads();
    // ---- 3b. otherwise: full streamed scan of this frame ----
    if (!complete && rescan) {
      if (tid == 0) nsel = 0;
      for (int r = 0; r < K; ++r) {
        const double ps = last_s;
        const int pr = last_r;
        double bs = d_neg_inf();
        int br = 0x7fffffff, bc = -1;
        for (int c = tid; c < K * S + K; c += DEC_THREADS) {
          double sc;
          int rk;
          if (!cand_value(cur, c, lp, K, S, p.blank, sc, rk)) continue;
          if (r > 0 && !dec_better(ps, pr, sc, rk)) continue;   // selected in an earlier round
          if (bc < 0 || dec_better(sc, rk, bs, br)) { bs = sc; br = rk; bc = c; }
        }
        dec_block_argmax(bs, br, bc, red_s, red_r, red_c);
        if (tid == 0 && bc >= 0) { sel[nsel++] = bc; last_s = bs; last_r = br; }
        __syncthreads();
        if (nsel <= r) break;
      }
    }
    // ---- 4. materialise the pruned beam ----
    dec_commit(p, u, cur, nxt, sel, nsel, lp, t);
  }
  dec_finish(p, u, beams[T & 1]);
}

}  // namespace sb

using namespace sb;

static int dec_hash_cap(int T, int K) {
  size_t need = 2 * ((size_t)T * K + 1);
  size_t cap = 64;
  while (cap < need) cap <<= 1;
  return (int)cap;
}

static size_t dec_shortlist_offset(int B, int T, int K) {
  const size_t cap = (size_t)dec_hash_cap(T, K);
  return (size_t)B * 2 * ((size_t)T * K + 1) * sizeof(int) + 256 +
         (size_t)B * cap * (sizeof(unsigned long long) + sizeof(int)) + 512;
}

extern "C" int sb_ctc_prefix_beam_workspace_size(int B, int T, int K, size_t* bytes) {
  if (!bytes || B <= 0 || T < 0 || K <= 0) return SB_ERR_INVALID;
  *bytes = dec_shortlist_offset(B, T, K) + (size_t)B * T * (2 * K + 1) * sizeof(int);
  return SB_OK;
}

static size_t dec_full_smem(int S, int K) {
  return (size_t)(K * S + K) * (sizeof(double) + sizeof(int) + 1) + 16;
}

static int dec_entry(const float* logp, const int* lens, int B, int T, int S, int beam_size,
                     int blank, int* out_labels, int* out_lens, double* out_scores,
                     void* workspace, size_t workspace_bytes, void* stream_, bool force_shortlist) {
  if (!logp || !lens || !out_labels || !out_lens || !out_scores || !workspace) return SB_ERR_INVALID;
  if (B <= 0 || T <= 0 || S <= 0 || blank < 0 || blank >= S || beam_size <= 0) return SB_ERR_INVALID;
  if (beam_size > DEC_MAX_BEAM) return SB_ERR_UNSUPPORTED;
  size_t need = 0;
  sb_ctc_prefix_beam_workspace_size(B, T, beam_size, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DecParams p;
  p.logp = logp; p.lens = lens;
  p.nodes = reinterpret_cast<int*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  p.hcap = dec_hash_cap(T, beam_size);
  p.hkeys = reinterpret_cast<unsigned long long*>(
      (reinterpret_cast<uintptr_t>(p.nodes + (size_t)B * 2 * ((size_t)T * beam_size + 1)) + 255) &
      ~(uintptr_t)255);
  p.hvals = reinterpret_cast<int*>(p.hkeys + (size_t)B * p.hcap);
  p.out_labels = out_labels; p.out_lens = out_lens; p.out_scores = out_scores;
  p.B = B; p.T = T; p.S = S; p.K = beam_size; p.blank = blank;

  const size_t full_smem = dec_full_smem(S, beam_size);
  if (!force_shortlist && full_smem <= 200 * 1024) {
    if (full_smem > 40 * 1024) {
      if (cudaFuncSetAttribute(ctc_prefix_beam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)full_smem) != cudaSuccess)
        return SB_ERR_CUDA;
    }
    ctc_prefix_beam_kernel<<<B, DEC_THREADS, full_smem, stream>>>(p);
    return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
  }

  const int LS = 2 * beam_size + 1;
  const int L = S - 1 < LS ? S - 1 : LS;
  int* shortlist = reinterpret_cast<int*>(static_cast<unsigned char*>(workspace) +
                                          dec_shortlist_offset(B, T, beam_size));
  const int ncand = beam_size * (L + 1) + beam_size;
  const size_t smem = (size_t)ncand * (sizeof(double) + 2 * sizeof(int) + 1) + 16;
  if (smem > 40 * 1024) {
    if (cudaFuncSetAttribute(ctc_prefix_beam_shortlist_kernel,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return SB_ERR_CUDA;
  }
  if (L > 0)
    ctc_shortlist_kernel<<<dim3(T, B), DEC_SL_THREADS, 0, stream>>>(logp, lens, shortlist, T, S,
                                                                     blank, L, LS);
  ctc_prefix_beam_shortlist_kernel<<<B, DEC_THREADS, smem, stream>>>(p, shortlist, L, LS);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_ctc_prefix_beam(const float* logp, const int* lens, int B, int T, int S,
                                  int beam_size, int blank, int* out_labels, int* out_lens,
                                  double* out_scores, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  return dec_entry(logp, lens, B, T, S, beam_size, blank, out_labels, out_lens, out_scores,
                   workspace, workspace_bytes, stream, false);
}

extern "C" int sb_ctc_prefix_beam_shortlist(const float* logp, const int* lens, int B, int T,
                                            int S, int beam_size, int blank, int* out_labels,
                                            int* out_lens, double* out_scores, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  return dec_entry(logp, lens, B, T, S, beam_size, blank, out_labels, out_lens, out_scores,
                   workspace, workspace_bytes, stream, true);
}

// ------------------------------------------------------------------------------------------------
// sb_beam_topk: the expand/prune step of Seq2Seq.beam_search (speech/models/seq2seq.py:200-212):
// the reference sorts ALL beam x vocab candidates with a stable descending sort and keeps a
// prefix, so ties keep (beam index, vocab index) order = ascending flat index.  One CTA selects
// the top k of n float64 scores by k rounds of block arg-max on (score desc, index asc).
// ------------------------------------------------------------------------------------------------
namespace sb {
__global__ void __launch_bounds__(256) beam_topk_kernel(const double* __restrict__ scores, int n,
                                                        int k, int* out_idx, double* out_val) {
  extern __shared__ unsigned char topk_smem[];
  double* sc = reinterpret_cast<double*>(topk_smem);
  __shared__ double rs[8];
  __shared__ int ri[8];
  const int tid = threadIdx.x;
  for (int i = tid; i < n; i += 256) sc[i] = scores[i];
  __syncthreads();
  for (int r = 0; r < k; ++r) {
    double bs = 0.0;
    int bi = -1;
    for (int i = tid; i < n; i += 256) {
      const double v = sc[i];
      if (isnan(v)) continue;                      // NaN marks "already taken"
      if (bi < 0 || v > bs) { bs = v; bi = i; }    // ascending i: first index wins ties
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double os = __shfl_xor_sync(0xffffffffu, bs, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || os > bs || (os == bs && oi < bi))) { bs = os; bi = oi; }
    }
    if ((tid & 31) == 0) { rs[tid >> 5] = bs; ri[tid >> 5] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 8; ++w)
        if (ri[w] >= 0 && (bi < 0 || rs[w] > bs || (rs[w] == bs && ri[w] < bi))) {
          bs = rs[w]; bi = ri[w];
        }
      out_idx[r] = bi;
      out_val[r] = bs;
      if (bi >= 0) sc[bi] = nan("");
    }
    __syncthreads();
  }
}
}  // namespace sb

extern "C" int sb_beam_topk(const double* scores, int n, int k, int* out_idx, double* out_val,
                            void* stream_) {
  if (!scores || !out_idx || !out_val || n <= 0 || k <= 0 || k > n) return SB_ERR_INVALID;
  const size_t smem = (size_t)n * sizeof(double);
  if (smem > 200 * 1024) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (smem > 40 * 1024 &&
      cudaFuncSetAttribute(sb::beam_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)smem) != cudaSuccess)
    return SB_ERR_CUDA;
  sb::beam_topk_kernel<<<1, 256, smem, stream>>>(scores, n, k, out_idx, out_val);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
