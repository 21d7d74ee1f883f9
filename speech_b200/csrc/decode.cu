// sb_ctc_prefix_beam: CTC prefix beam search on the GPU, one CTA per utterance.
//
// Replaces speech/models/ctc_decoder.py:38-113 `decode(probs, beam_size, blank)` (pure-Python dict
// beam, called serially per utterance from CTC.infer, ctc_model.py:55-60).  The search is restated
// so that hypotheses come out IDENTICAL to the reference, including its tie-breaks:
//   * beam entries carry (p_blank, p_non_blank) in float64 log space, as the reference's Python
//     floats; log-sum-exp is evaluated in the reference's argument order;
//   * prefixes are nodes of a per-utterance trie (beam.cuh), so "prefix + s is already in the
//     beam" (the merge case, ctc_decoder.py:84-103) is an integer comparison;
//   * pruning = K rounds of the selection of beam.cuh with the first-touch rank as the key: the
//     reference sorts a dict's items with a stable sort, so ties keep dict insertion order, which
//     is the order of first touch in its `for s in vocab: for prefix in beam:` loops
//     (ctc_decoder.py:65-103).
// Input is log-probabilities (the host wrapper applies the same float32 log as the reference).
//
// Roofline: HBM-nominal (reads T*S floats per utterance), in practice latency-bound by the
// T-serial beam update; decode is not on the training path.
#include "beam.cuh"
#include "ngram.cuh"
#include <math.h>
#include <string.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int DEC_THREADS = 128;
static constexpr int DEC_MAX_BEAM = 32;

struct DecParams {
  const float* logp;   // (B, T, S)
  const int* lens;     // (B) frames per utterance (<= T)
  BeamTrie trie;       // utterance 0 of B; T*K + 1 nodes each
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

// ------------------------------------------------------------------------------------------------
// Shallow fusion.  The search is written once over a policy that gives the value q an extension
// of beam entry i by symbol s scores with, from the acoustic log-probability p = p_s:
//   NoFuse  q = p (the LM-less search, its arithmetic untouched);
//   LmFuse  q = p + (alpha * lm(s | ctx_i) + beta), lm the backoff lookup of SbNgramLm.
//   WordLmFuse  the word LM of SbWordLm (include/speech_b200.h): the LM term only on the
//           delimiter that ends a non-empty word, an OOV penalty where a word leaves the lexicon.
// Entry i's context is its last order-1 symbols (LmFuse) or completed words (WordLmFuse), kept
// most recent first in LmShared::hist (-1 stands for <s>, before which there is nothing).  Once per
// frame each entry walks the context trie along them (lm_resolve); a candidate's lookup is then at
// most `order` probes.
// ------------------------------------------------------------------------------------------------
struct NoFuse {
  static constexpr bool kLm = false;
  static constexpr bool kWord = false;
  static constexpr int kMinBlocks = 0;
  __device__ __forceinline__ double q(int, int, double p) const { return p; }
};

struct LmShared {
  int hist[2][DEC_MAX_BEAM][SB_LM_MAX_ORDER - 1];  // per beam buffer (t & 1) and entry
  int ctx[DEC_MAX_BEAM][SB_LM_MAX_ORDER];          // context nodes, [0] = root .. [depth]
  int depth[DEC_MAX_BEAM];
};
__device__ __forceinline__ LmShared& lm_shared() {
  __shared__ LmShared sh;
  return sh;
}

struct LmFuse {
  static constexpr bool kLm = true;
  static constexpr bool kWord = false;
  static constexpr int kMinBlocks = 1;
  SbNgramLm lm;
  double alpha, beta;

  // lm(s | ctx_i)
  __device__ __forceinline__ double lm_logp(int i, int s) const {
    const LmShared& sh = lm_shared();
    const int t = __ldg(lm.tok + s);
    return lm_backoff(lm, sh.ctx[i], sh.depth[i], t);
  }
  __device__ __forceinline__ double q(int i, int s, double p) const {
    return p + (alpha * lm_logp(i, s) + beta);
  }
};

// entry i of the beam in buffer par: its context nodes, thread i for i < nb; the caller syncs
__device__ __forceinline__ void lm_resolve(const LmFuse& fu, int par, int nb) {
  LmShared& sh = lm_shared();
  const int i = threadIdx.x;
  if (i >= nb) return;
  sh.depth[i] = lm_context(fu.lm, [&](int k) { return sh.hist[par][i][k]; }, sh.ctx[i]);
}

// The word LM.  Per entry, besides its history of word tokens in LmShared::hist: its lexicon node
// per beam buffer (WordShared::lex, 0 = the empty partial word, -1 = off the lexicon), and, for the
// current frame, that node and the delimiter term d_i = (alpha * lm(w | ctx_i) + beta) + g_i
// (word_resolve, thread i once per frame).  An extension by the delimiter then costs nothing more
// and any other extension one lexicon probe.  kLm is false: the shortlist route keeps the LM-less
// bound (see the comment above the shortlist body).
struct WordShared {
  int lex[2][DEC_MAX_BEAM];      // per beam buffer (t & 1) and entry
  int node[DEC_MAX_BEAM];        // the current beam's nodes
  double dterm[DEC_MAX_BEAM];    // the current beam's delimiter terms (entries with node != 0)
  double fin[DEC_MAX_BEAM];      // end of utterance: final_i
};
__device__ __forceinline__ WordShared& word_shared() {
  __shared__ WordShared sh;
  return sh;
}

struct WordLmFuse : WordTerms {
  static constexpr bool kLm = false;
  static constexpr bool kWord = true;
  static constexpr int kMinBlocks = 1;

  __device__ __forceinline__ double q(int i, int s, double p) const {
    const WordShared& ws = word_shared();
    const int node = ws.node[i];
    if (s == lm.delimiter) return node == 0 ? p : p + ws.dterm[i];
    if (node >= 0 && child(node, s) < 0) return p + gamma;
    return p;
  }
};

// entry i of the beam in buffer par: its node and delimiter term, thread i for i < nb; the caller
// syncs
__device__ __forceinline__ void word_resolve(const WordLmFuse& fu, int par, int nb) {
  LmShared& sh = lm_shared();
  WordShared& ws = word_shared();
  const int i = threadIdx.x;
  if (i >= nb) return;
  const int node = ws.lex[par][i];
  ws.node[i] = node;
  if (node != 0) ws.dterm[i] = fu.dterm(node, [&](int k) { return sh.hist[par][i][k]; }, sh.ctx[i]);
}

// value of the candidate "beam entry j keeps its prefix" at this frame
template <class Fuse>
__device__ void stay_value(const Beam& bm, int j, const float* lp, int blank, int K, double& npb,
                           double& npnb, int& rank, const Fuse& fu) {
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
      const double q = fu.q(pi, s, p);     // the parent's extension by s
      if (pi < j) {
        npnb = rep ? lse2d(npnb, bm.pb[pi] + q) : lse3d(npnb, bm.pb[pi] + q, bm.pnb[pi] + q);
        npnb = lse2d(npnb, bm.pnb[j] + p);
      } else {
        npnb = lse2d(npnb, bm.pnb[j] + p);
        npnb = rep ? lse2d(npnb, bm.pb[pi] + q) : lse3d(npnb, bm.pb[pi] + q, bm.pnb[pi] + q);
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
template <class Fuse>
__device__ bool ext_value(const Beam& bm, int i, int s, const float* lp, int K, double& npnb,
                          int& rank, const Fuse& fu) {
  for (int j = 0; j < bm.size; ++j)
    if (bm.last[j] == s && bm.parent[j] == bm.node[i] && bm.node[j] != 0) return false;
  const double q = fu.q(i, s, (double)lp[s]);
  if (s != bm.last[i]) npnb = lse3d(d_neg_inf(), bm.pb[i] + q, bm.pnb[i] + q);
  else npnb = lse2d(d_neg_inf(), bm.pb[i] + q);
  rank = s * 2 * K + 2 * i;
  return true;
}

// Candidate c of a frame, numbered as the full scan numbers them: c < K*S is "entry c / S extended
// by symbol c % S", c = K*S + j is "entry j keeps its prefix".  Returns false for a candidate that
// does not exist (no such entry, the blank as an extension, or an extension that is a beam entry).
template <class Fuse>
__device__ __forceinline__ bool cand_value(const Beam& cur, int c, const float* lp, int K, int S,
                                           int blank, double& sc, int& rk, const Fuse& fu) {
  sc = d_neg_inf();
  rk = 0x7fffffff;
  const int nb = cur.size;
  if (c < K * S) {
    const int i = c / S, s = c - i * S;
    if (i < nb && s != blank) {
      double x;
      const bool ok = ext_value(cur, i, s, lp, K, x, rk, fu);
      if (ok) sc = x;  // logsumexp(-inf, x) == x exactly
      return ok;
    }
    return false;
  }
  const int j = c - K * S;
  if (j >= nb) return false;
  double npb, npnb;
  stay_value(cur, j, lp, blank, K, npb, npnb, rk, fu);
  sc = lse2d(npb, npnb);
  return true;
}

// One selection round over the scored candidates of a frame: the first live one by (score desc,
// rank asc) is struck off and returned to every thread, with its score and rank (-1: none left).
// live[c] is read and written by thread c % DEC_THREADS only, so striking needs no barrier.
__device__ __forceinline__ int dec_take_first(const double* score, const int* rank,
                                              unsigned char* live, int ncand, double& bs, int& br) {
  const int tid = threadIdx.x;
  bs = d_neg_inf();
  br = -1;
  int bc = -1;
  for (int c = tid; c < ncand; c += DEC_THREADS) {
    if (!live[c]) continue;
    if (beam_before(score[c], rank[c], bs, br)) { bs = score[c]; br = rank[c]; bc = c; }
  }
  beam_block_first<DEC_THREADS>(bs, br, bc);
  if (bc >= 0 && (bc & (DEC_THREADS - 1)) == tid) live[bc] = 0;
  return bc;
}

// the beam of the empty prefix (one thread)
__device__ __forceinline__ void dec_empty(Beam& bm) {
  bm.size = 1;
  bm.pb[0] = 0.0;
  bm.pnb[0] = d_neg_inf();
  bm.node[0] = 0;
  bm.last[0] = -1;
  bm.parent[0] = -1;
}

template <class Fuse>
__device__ __forceinline__ void dec_begin(const DecParams& p, Beam* beams) {
  if (threadIdx.x == 0) {
    dec_empty(beams[0]);
    if constexpr (Fuse::kLm || Fuse::kWord) lm_shared().hist[0][0][0] = -1;   // <s>
    if constexpr (Fuse::kWord) word_shared().lex[0][0] = 0;
  }
  p.trie.of(blockIdx.x).clear<DEC_THREADS>();
}

// Start of frame t over the beam cur: with an LM, every entry's context nodes.
template <class Fuse>
__device__ __forceinline__ void dec_frame(const Fuse& fu, const Beam& cur, int t) {
  if constexpr (Fuse::kLm) {
    lm_resolve(fu, t & 1, cur.size);
    __syncthreads();
  }
  if constexpr (Fuse::kWord) {
    word_resolve(fu, t & 1, cur.size);
    __syncthreads();
  }
}

// Materialise the pruned beam of frame t: thread r < ns holds the r-th selected candidate in `mine`
// (full-scan numbering).  With an LM, an extension's context is its parent's shifted by one symbol
// and an entry that stays copies its own.  With a word LM, an extension by the delimiter shifts
// the word it ends into the history (none for an empty word) and goes to the root; any other
// extension moves the node to its child by s (-1 where there is none) and keeps the history.
template <class Fuse>
__device__ __forceinline__ void dec_commit(const DecParams& p, const Beam& cur, Beam& nxt, int mine,
                                           int ns, const float* lp, int t, const Fuse& fu) {
  const int tid = threadIdx.x, K = p.K, S = p.S;
  if (tid < ns) {
    const int c = mine;
    if (c < K * S) {
      const int i = c / S, s = c - i * S;
      double x; int rk;
      ext_value(cur, i, s, lp, K, x, rk, fu);
      nxt.pb[tid] = d_neg_inf();
      nxt.pnb[tid] = x;
      nxt.node[tid] = p.trie.of(blockIdx.x).find_or_insert<true>(cur.node[i], s, 1 + t * K + tid);
      nxt.last[tid] = s;
      nxt.parent[tid] = cur.node[i];
      if constexpr (Fuse::kLm) {
        LmShared& sh = lm_shared();
        const int par = t & 1;
        for (int k = fu.lm.order - 2; k > 0; --k) sh.hist[par ^ 1][tid][k] = sh.hist[par][i][k - 1];
        if (fu.lm.order > 1) sh.hist[par ^ 1][tid][0] = s;
      }
      if constexpr (Fuse::kWord) {
        LmShared& sh = lm_shared();
        WordShared& ws = word_shared();
        const int par = t & 1, node = ws.node[i], n = fu.lm.ngram.order - 1;
        if (s == fu.lm.delimiter && node != 0) {
          for (int k = n - 1; k > 0; --k) sh.hist[par ^ 1][tid][k] = sh.hist[par][i][k - 1];
          if (n > 0) sh.hist[par ^ 1][tid][0] = fu.word_tok(node);
        } else {
          for (int k = 0; k < n; ++k) sh.hist[par ^ 1][tid][k] = sh.hist[par][i][k];
        }
        ws.lex[par ^ 1][tid] = s == fu.lm.delimiter ? 0 : node < 0 ? -1 : fu.child(node, s);
      }
    } else {
      const int j = c - K * S;
      double npb, npnb; int rk;
      stay_value(cur, j, lp, p.blank, K, npb, npnb, rk, fu);
      nxt.pb[tid] = npb;
      nxt.pnb[tid] = npnb;
      nxt.node[tid] = cur.node[j];
      nxt.last[tid] = cur.last[j];
      nxt.parent[tid] = cur.parent[j];
      if constexpr (Fuse::kLm) {
        LmShared& sh = lm_shared();
        const int par = t & 1;
        for (int k = 0; k < fu.lm.order - 1; ++k) sh.hist[par ^ 1][tid][k] = sh.hist[par][j][k];
      }
      if constexpr (Fuse::kWord) {
        LmShared& sh = lm_shared();
        WordShared& ws = word_shared();
        const int par = t & 1;
        for (int k = 0; k < fu.lm.ngram.order - 1; ++k)
          sh.hist[par ^ 1][tid][k] = sh.hist[par][j][k];
        ws.lex[par ^ 1][tid] = ws.lex[par][j];
      }
    }
  }
  if (tid == 0) nxt.size = ns;
  __syncthreads();
}

// Best hypothesis of the final beam: back-track the trie.
__device__ __forceinline__ void dec_finish(const DecParams& p, const Beam& fin) {
  if (threadIdx.x == 0) {
    const int b = blockIdx.x;
    p.out_lens[b] = p.trie.of(b).backtrack(fin.node[0], p.out_labels + (size_t)b * p.T);
    p.out_scores[b] = -lse2d(fin.pb[0], fin.pnb[0]);
  }
}

// With a word LM: the end-of-utterance rule over the final beam, whose entries' histories and
// nodes are hist[i] and lex[i] (shared or global memory).  Thread i scores entry i; the largest
// final_i wins, ties going to the lowest index.  Every thread of the block calls it.
__device__ __forceinline__ void dec_finish_word(const DecParams& p, const WordLmFuse& fu,
                                                const Beam& fin,
                                                const int (*hist)[SB_LM_MAX_ORDER - 1],
                                                const int* lex) {
  WordShared& ws = word_shared();
  const int i = threadIdx.x;
  if (i < fin.size)
    ws.fin[i] = lse2d(fin.pb[i], fin.pnb[i]) +
                fu.end_term(lex[i], [&](int k) { return hist[i][k]; }, lm_shared().ctx[i]);
  __syncthreads();
  if (i == 0) {
    int best = 0;
    for (int j = 1; j < fin.size; ++j)
      if (ws.fin[j] > ws.fin[best]) best = j;
    const int b = blockIdx.x;
    p.out_lens[b] = p.trie.of(b).backtrack(fin.node[best], p.out_labels + (size_t)b * p.T);
    p.out_scores[b] = -ws.fin[best];
  }
}

// ------------------------------------------------------------------------------------------------
// Where a search's beam comes from and goes to.  The kernels below run frames [t0, t0 + n) of
// utterance b over a beam that begin() puts in beams[t0 & 1] (and, with an LM, the contexts in
// hist[t0 & 1]); end() takes the beam of frame t0 + n.  Frame t of the utterance is row t - t0 of
// the kernel's logp, and its trie nodes are numbered 1 + t*K + r, so that a resumed search names
// every prefix as one pass over the whole utterance does.
//   DecOffline  t0 = 0, n = lens[b]: a fresh beam and trie; the best prefix goes to the outputs.
//   DecResume   t0 = the frames the slot has consumed: the beam, the contexts and the trie of a
//               DecSlot (sb_ctc_stream_*), stored back at the end.
// ------------------------------------------------------------------------------------------------
struct DecOffline {
  template <class Fuse>
  __device__ __forceinline__ int begin(const DecParams& p, Beam* beams, int& n) const {
    dec_begin<Fuse>(p, beams);
    return 0;
  }
  template <class Fuse>
  __device__ __forceinline__ void end(const DecParams& p, const Fuse& fu, const Beam* beams,
                                      int t) const {
    if constexpr (Fuse::kWord)
      dec_finish_word(p, fu, beams[t & 1], lm_shared().hist[t & 1], word_shared().lex[t & 1]);
    else
      dec_finish(p, beams[t & 1]);
  }
};

// One stream of the resumable search: the beam after frame `frames` - 1 and its entries' contexts
// (and, with a word LM, lexicon nodes).
struct DecSlot {
  Beam beam;
  int hist[DEC_MAX_BEAM][SB_LM_MAX_ORDER - 1];
  int frames;     // frames consumed since the last reset
  int overflow;   // a step was asked for frames past max_frames (and clamped)
  int lex[DEC_MAX_BEAM];
};
static constexpr size_t DEC_SLOT_BYTES = (sizeof(DecSlot) + 255) / 256 * 256;
static_assert(DEC_SLOT_BYTES == 2304, "the lexicon nodes fit the slot's padding");

__device__ __forceinline__ DecSlot* dec_slot(void* base, int b) {
  return reinterpret_cast<DecSlot*>(static_cast<unsigned char*>(base) + (size_t)b * DEC_SLOT_BYTES);
}

// copy `bytes` (a multiple of 4) with the whole block
__device__ __forceinline__ void dec_copy(void* dst, const void* src, size_t bytes) {
  for (size_t k = threadIdx.x; k < bytes / 4; k += DEC_THREADS)
    static_cast<int*>(dst)[k] = static_cast<const int*>(src)[k];
}

struct DecResume {
  void* slots;      // [B] DecSlot, DEC_SLOT_BYTES apart
  int max_frames;

  template <class Fuse>
  __device__ __forceinline__ int begin(const DecParams& p, Beam* beams, int& n) const {
    const DecSlot* sl = dec_slot(slots, blockIdx.x);
    const int t0 = sl->frames;
    if (n > max_frames - t0) {            // refused by the host; never past the trie's arena
      n = max_frames - t0;
      if (threadIdx.x == 0) dec_slot(slots, blockIdx.x)->overflow = 1;
    }
    dec_copy(&beams[t0 & 1], &sl->beam, sizeof(Beam));
    if constexpr (Fuse::kLm || Fuse::kWord)
      dec_copy(lm_shared().hist[t0 & 1], sl->hist, sizeof(sl->hist));
    if constexpr (Fuse::kWord) dec_copy(word_shared().lex[t0 & 1], sl->lex, sizeof(sl->lex));
    __syncthreads();
    return t0;
  }
  template <class Fuse>
  __device__ __forceinline__ void end(const DecParams& p, const Fuse& fu, const Beam* beams,
                                      int t) const {
    DecSlot* sl = dec_slot(slots, blockIdx.x);
    dec_copy(&sl->beam, &beams[t & 1], sizeof(Beam));
    if constexpr (Fuse::kLm || Fuse::kWord)
      dec_copy(sl->hist, lm_shared().hist[t & 1], sizeof(sl->hist));
    if constexpr (Fuse::kWord) dec_copy(sl->lex, word_shared().lex[t & 1], sizeof(sl->lex));
    if (threadIdx.x == 0) sl->frames = t;
  }
};

// kMinBlocks: 0 leaves the LM-less kernel's register allocation as it was; 1 lets the LM kernel
// use 70 registers instead of 56 and an 8-byte spill (one CTA per utterance either way).
template <class Fuse, class Io>
__device__ __forceinline__ void ctc_prefix_beam_body(const DecParams p, const Fuse fu,
                                                     const Io io) {
  extern __shared__ unsigned char dec_smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p.K, S = p.S;
  int T = min(p.lens[b], p.T);
  const int ncand = K * S + K;
  double* score = reinterpret_cast<double*>(dec_smem);             // [ncand]
  int* rank = reinterpret_cast<int*>(score + ncand);               // [ncand]
  unsigned char* live = reinterpret_cast<unsigned char*>(rank + ncand);  // [ncand]
  __shared__ Beam beams[2];

  const int t0 = io.template begin<Fuse>(p, beams, T);
  const float* logp = p.logp + (size_t)b * p.T * S;

  for (int f = 0; f < T; ++f) {
    const int t = t0 + f;
    const Beam& cur = beams[t & 1];
    Beam& nxt = beams[(t & 1) ^ 1];
    const float* lp = logp + (size_t)f * S;
    dec_frame(fu, cur, t);
    // ---- 1. score every candidate ----
    for (int c = tid; c < ncand; c += DEC_THREADS) {
      double sc;
      int rk;
      live[c] = cand_value(cur, c, lp, K, S, p.blank, sc, rk, fu) ? 1 : 0;
      score[c] = sc;
      rank[c] = rk;
    }
    __syncthreads();
    // ---- 2. the K first by (score desc, rank asc); thread r keeps the r-th ----
    int ns = 0, mine = -1;
    for (int r = 0; r < K; ++r) {
      double bs;
      int br;
      const int bc = dec_take_first(score, rank, live, ncand, bs, br);
      if (bc < 0) break;
      if (tid == ns) mine = bc;
      ++ns;
    }
    // ---- 3. materialise the pruned beam ----
    dec_commit(p, cur, nxt, mine, ns, lp, t, fu);
  }
  io.end(p, fu, beams, t0 + T);
}

template <class Fuse>
__global__ void __launch_bounds__(DEC_THREADS, Fuse::kMinBlocks) ctc_prefix_beam_kernel(
    const DecParams p, const Fuse fu) {
  ctc_prefix_beam_body(p, fu, DecOffline{});
}
// The resumed kernel takes the LM kernel's bound in both forms: with 0 the LM-less one spills.
template <class Fuse>
__global__ void __launch_bounds__(DEC_THREADS, 1) ctc_stream_kernel(
    const DecParams p, const Fuse fu, const DecResume io) {
  ctc_prefix_beam_body(p, fu, io);
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
// With an LM the extension of i by s scores f_i(q_s), q_s = p_s + (alpha * lm(s | ctx_i) + beta),
// and the order of the p_s no longer orders the q_s, so the short list is only a guess; the check
// is what keeps the search exact.  For a left-out symbol, alpha >= 0 and lm(s | ctx_i) <= lm_upper
// give q_s <= q_max = p_min + (alpha * lm_upper + beta) in exact arithmetic, and U = max_i f_i(q_max)
// as computed.  Rounding now enters through every term of q as well (a lookup sums at most
// order + 1 values, each of magnitude <= lm_abs; then one product and two sums), so the margin is
//     1e-12 * (1 + |U| + |p_min| + alpha * lm_abs + |beta|),
// which bounds the magnitude of every operand on the way to f and U; the rounding error of the
// twenty-odd operations in between is below 1e-14 times it.  When p_min = -inf every left-out q_s
// is -inf exactly (the LM terms are finite), so U = -inf keeps its meaning.  A frame the check
// cannot prove is rescanned as above, with the same fused arithmetic.
//
// With a word LM (WordLmFuse) each entry also scores the delimiter on every frame, next to its
// last symbol (and deduplicated as that is), since the delimiter carries the word's LM term.
// Every other class s has q_s = p_s or q_s = p_s + gamma, and gamma <= 0, so q_s <= p_s in exact
// arithmetic and also as computed: floating-point addition rounds monotonically, so
// fl(p_s + gamma) <= fl(p_s + 0) = p_s (and p_s + -inf = -inf).  A left-out class therefore has
// q_s <= p_s <= p_min, and the LM-less bound U = max_i f_i(p_min) and margin apply unchanged: the
// word LM causes no rescans of its own.
//
// The shortlist of every frame (2K + 1 ints, or S - 1 if fewer) comes from a pre-pass over the
// B*T rows (ctc_shortlist_kernel, one CTA per frame).
// ------------------------------------------------------------------------------------------------
static constexpr int DEC_SL_THREADS = 256;

// frames the LM-fused shortlist search rescanned (sb_debug_ctc_lm_rescans)
__device__ unsigned long long dec_lm_rescans;

// grid (T, B): shortlist[(b*T + t)*LS + j], j < L, for the frames t < lens[b]
__global__ void __launch_bounds__(DEC_SL_THREADS) ctc_shortlist_kernel(
    const float* __restrict__ logp, const int* __restrict__ lens, int* __restrict__ shortlist,
    int T, int S, int blank, int L, int LS) {
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  if (t >= min(lens[b], T)) return;
  const float* lp = logp + ((size_t)b * T + t) * S;
  int* out = shortlist + ((size_t)b * T + t) * LS;
  float px = 0.f;                          // the previous round's symbol: (p desc, s asc) order
  int ps = -1;
  for (int j = 0; j < L; ++j) {
    float bx = 0.f;
    int bsym = -1;
    for (int s = tid; s < S; s += DEC_SL_THREADS) {
      if (s == blank) continue;
      const float x = __ldg(lp + s);
      if (j && !beam_order(px, ps, x, s)) continue;     // listed in an earlier round
      if (beam_before(x, s, bx, bsym)) { bx = x; bsym = s; }
    }
    beam_block_first<DEC_SL_THREADS>(bx, bsym);
    if (tid == 0) out[j] = bsym;
    px = bx;
    ps = bsym;
  }
}

template <class Fuse, class Io>
__device__ __forceinline__ void ctc_prefix_beam_shortlist_body(
    const DecParams p, const int* __restrict__ shortlist, int L, int LS, const Fuse fu,
    const Io io) {
  extern __shared__ unsigned char dec_smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p.K, S = p.S;
  int T = min(p.lens[b], p.T);
  const int per = L + 1 + (Fuse::kWord ? 1 : 0);   // shortlist + last_i (+ delimiter) per entry
  const int ncand = K * per + K;
  double* score = reinterpret_cast<double*>(dec_smem);             // [ncand]
  int* rank = reinterpret_cast<int*>(score + ncand);               // [ncand]
  int* full = rank + ncand;                                        // [ncand] full-scan number
  unsigned char* live = reinterpret_cast<unsigned char*>(full + ncand);  // [ncand]
  __shared__ Beam beams[2];
  __shared__ int rescan;
  const bool complete = L >= S - 1;        // every non-blank symbol is on the list

  const int t0 = io.template begin<Fuse>(p, beams, T);
  const float* logp = p.logp + (size_t)b * p.T * S;

  for (int f = 0; f < T; ++f) {
    const int t = t0 + f;
    const Beam& cur = beams[t & 1];
    Beam& nxt = beams[(t & 1) ^ 1];
    const float* lp = logp + (size_t)f * S;
    const int* sl = shortlist + ((size_t)b * p.T + f) * LS;
    const int nb = cur.size;
    dec_frame(fu, cur, t);
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
          if constexpr (Fuse::kWord) {
            if (j == L + 1) {                // the delimiter, unless scored above
              s = fu.lm.delimiter;
              for (int q = 0; q < L && s >= 0; ++q)
                if (sl[q] == s) s = -1;
              if (s == cur.last[i]) s = -1;
            }
          }
          if (s >= 0 && s != p.blank) {
            fc = i * S + s;
            ok = cand_value(cur, fc, lp, K, S, p.blank, sc, rk, fu);
          }
        }
      } else {
        fc = K * S + (c - K * per);
        ok = cand_value(cur, fc, lp, K, S, p.blank, sc, rk, fu);
      }
      score[c] = sc;
      rank[c] = rk;
      full[c] = fc;
      live[c] = ok ? 1 : 0;
    }
    __syncthreads();
    // ---- 2. the K first by (score desc, rank asc), as the full scan; thread r keeps the r-th,
    //         every thread the score and rank of the last ----
    int ns = 0, mine = -1, last_r = -1;
    double last_s = d_neg_inf();
    for (int r = 0; r < K; ++r) {
      double bs;
      int br;
      const int bc = dec_take_first(score, rank, live, ncand, bs, br);
      if (bc < 0) break;
      if (tid == ns) mine = full[bc];
      ++ns;
      last_s = bs;
      last_r = br;
    }
    // ---- 3. check that no left-out candidate can reach the selection ----
    if (!complete && tid < 32) {
      const double pmin = (double)lp[sl[L - 1]];
      double qmax = pmin;
      if constexpr (Fuse::kLm) qmax = pmin + (fu.alpha * fu.lm.lm_upper + fu.beta);
      double U = d_neg_inf();
      if (tid < nb) U = lse3d(d_neg_inf(), cur.pb[tid] + qmax, cur.pnb[tid] + qmax);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) U = fmax(U, __shfl_xor_sync(0xffffffffu, U, o));
      if (tid == 0) {
        bool ok = ns == K && last_s != d_neg_inf();
        if (ok && U != d_neg_inf()) {
          if constexpr (Fuse::kLm)
            ok = last_s > U + 1e-12 * (1.0 + fabs(U) + fabs(pmin) + fu.alpha * fu.lm.lm_abs +
                                       fabs(fu.beta));
          else
            ok = last_s > U + 1e-12 * (1.0 + fabs(U));
        }
        rescan = ok ? 0 : 1;
      }
    }
    __syncthreads();
    // ---- 3b. otherwise: full streamed scan of this frame ----
    if constexpr (Fuse::kLm || Fuse::kWord)
      if (!complete && rescan && tid == 0) atomicAdd(&dec_lm_rescans, 1ull);
    if (!complete && rescan) {
      ns = 0;
      for (int r = 0; r < K; ++r) {
        double bs = d_neg_inf();
        int br = -1, bc = -1;
        for (int c = tid; c < K * S + K; c += DEC_THREADS) {
          double sc;
          int rk;
          if (!cand_value(cur, c, lp, K, S, p.blank, sc, rk, fu)) continue;
          if (r > 0 && !beam_order(last_s, last_r, sc, rk)) continue;   // selected earlier
          if (beam_before(sc, rk, bs, br)) { bs = sc; br = rk; bc = c; }
        }
        beam_block_first<DEC_THREADS>(bs, br, bc);
        if (bc < 0) break;
        if (tid == ns) mine = bc;
        ++ns;
        last_s = bs;
        last_r = br;
      }
    }
    // ---- 4. materialise the pruned beam ----
    dec_commit(p, cur, nxt, mine, ns, lp, t, fu);
  }
  io.end(p, fu, beams, t0 + T);
}

template <class Fuse>
__global__ void __launch_bounds__(DEC_THREADS, 1) ctc_prefix_beam_shortlist_kernel(
    const DecParams p, const int* __restrict__ shortlist, int L, int LS, const Fuse fu) {
  ctc_prefix_beam_shortlist_body(p, shortlist, L, LS, fu, DecOffline{});
}
template <class Fuse>
__global__ void __launch_bounds__(DEC_THREADS, 1) ctc_stream_shortlist_kernel(
    const DecParams p, const int* __restrict__ shortlist, int L, int LS, const Fuse fu,
    const DecResume io) {
  ctc_prefix_beam_shortlist_body(p, shortlist, L, LS, fu, io);
}

// Slots first + blockIdx.x back to the empty prefix at frame 0, with an empty trie.
__global__ void __launch_bounds__(DEC_THREADS) ctc_stream_reset_kernel(const BeamTrie trie,
                                                                      void* slots, int first) {
  const int b = first + blockIdx.x;
  DecSlot* sl = dec_slot(slots, b);
  if (threadIdx.x == 0) {
    dec_empty(sl->beam);
    sl->hist[0][0] = -1;
    sl->lex[0] = 0;
    sl->frames = 0;
    sl->overflow = 0;
  }
  trie.of(b).clear<DEC_THREADS>();
}

// Each slot's best prefix so far (dec_finish on the stored beam) and its overflow flag.
__global__ void __launch_bounds__(32) ctc_stream_best_kernel(const DecParams p, const void* slots,
                                                             int* out_overflow) {
  const DecSlot* sl = dec_slot(const_cast<void*>(slots), blockIdx.x);
  dec_finish(p, sl->beam);
  if (threadIdx.x == 0 && out_overflow) out_overflow[blockIdx.x] = sl->overflow;
}

// The same with a word LM: the end-of-utterance rule over each stored beam (dec_finish_word).
__global__ void __launch_bounds__(32) ctc_stream_best_wordlm_kernel(const DecParams p,
                                                                    const void* slots,
                                                                    int* out_overflow,
                                                                    const WordLmFuse fu) {
  const DecSlot* sl = dec_slot(const_cast<void*>(slots), blockIdx.x);
  dec_finish_word(p, fu, sl->beam, sl->hist, sl->lex);
  if (threadIdx.x == 0 && out_overflow) out_overflow[blockIdx.x] = sl->overflow;
}

// Every stored entry of each slot: thread i < K back-tracks entry i into out_labels[b][i] and
// writes c_i = lse(p_b, p_nb); slots past the beam's size get length -1 and score -inf.
__global__ void __launch_bounds__(DEC_MAX_BEAM) ctc_stream_nbest_kernel(const BeamTrie trie,
                                                                        const void* slots, int K,
                                                                        int max_frames,
                                                                        int* out_labels,
                                                                        int* out_lens,
                                                                        double* out_scores,
                                                                        int* out_count) {
  const int b = blockIdx.x, i = threadIdx.x;
  const DecSlot* sl = dec_slot(const_cast<void*>(slots), b);
  const Beam& bm = sl->beam;
  const int nb = bm.size;
  if (i == 0) out_count[b] = nb;
  if (i >= K) return;
  const size_t e = (size_t)b * K + i;
  if (i < nb) {
    out_lens[e] = trie.of(b).backtrack(bm.node[i], out_labels + e * max_frames);
    out_scores[e] = lse2d(bm.pb[i], bm.pnb[i]);
  } else {
    out_lens[e] = -1;
    out_scores[e] = d_neg_inf();
  }
}

}  // namespace sb

using namespace sb;

static size_t dec_node_cap(int T, int K) { return (size_t)T * K + 1; }

static size_t dec_shortlist_offset(int B, int T, int K) {
  const size_t cap = (size_t)beam_pow2_cap(2 * dec_node_cap(T, K));
  return (size_t)B * 2 * dec_node_cap(T, K) * sizeof(int) + 256 +
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

// The trie arena of B utterances of node_cap nodes each at `base` (dec_shortlist_offset bytes).
static BeamTrie dec_trie(void* base, int B, size_t node_cap) {
  BeamTrie tr;
  tr.node_cap = (int)node_cap;
  tr.cap = beam_pow2_cap(2 * node_cap);
  tr.nodes = reinterpret_cast<int*>((reinterpret_cast<uintptr_t>(base) + 255) & ~(uintptr_t)255);
  tr.keys = reinterpret_cast<unsigned long long*>(
      (reinterpret_cast<uintptr_t>(tr.nodes + (size_t)B * 2 * tr.node_cap) + 255) &
      ~(uintptr_t)255);
  tr.vals = reinterpret_cast<int*>(tr.keys + (size_t)B * tr.cap);
  return tr;
}

// Both routes with the fusion policy fu, over a fresh beam (rs null) or resumed from the slots of
// *rs.  Every shape whose K*S + K full-scan candidates fit in 200 KB of shared memory takes the
// full scan; the static shared memory of any instantiation (6.7 KB at most, with a word LM's
// contexts and nodes) leaves both sizes below the per-block limit.  shortlist: B*T*(2K+1) ints.
template <class Fuse>
static int dec_launch(const DecParams& p, const Fuse& fu, const DecResume* rs, int* shortlist,
                      bool force_shortlist, cudaStream_t stream) {
  const int B = p.B, T = p.T, S = p.S, beam_size = p.K;
  const size_t full_smem = dec_full_smem(S, beam_size);
  if (!force_shortlist && full_smem <= 200 * 1024) {
    const void* kern = rs ? (const void*)ctc_stream_kernel<Fuse>
                          : (const void*)ctc_prefix_beam_kernel<Fuse>;
    if (full_smem > 40 * 1024) {
      if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)full_smem) != cudaSuccess)
        return SB_ERR_CUDA;
    }
    if (rs) ctc_stream_kernel<Fuse><<<B, DEC_THREADS, full_smem, stream>>>(p, fu, *rs);
    else ctc_prefix_beam_kernel<Fuse><<<B, DEC_THREADS, full_smem, stream>>>(p, fu);
    return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
  }

  const int LS = 2 * beam_size + 1;
  const int L = S - 1 < LS ? S - 1 : LS;
  const int ncand = beam_size * (L + 1 + (Fuse::kWord ? 1 : 0)) + beam_size;
  const size_t smem = (size_t)ncand * (sizeof(double) + 2 * sizeof(int) + 1) + 16;
  const void* kern = rs ? (const void*)ctc_stream_shortlist_kernel<Fuse>
                        : (const void*)ctc_prefix_beam_shortlist_kernel<Fuse>;
  if (smem > 40 * 1024) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
        cudaSuccess)
      return SB_ERR_CUDA;
  }
  if (L > 0)
    ctc_shortlist_kernel<<<dim3(T, B), DEC_SL_THREADS, 0, stream>>>(p.logp, p.lens, shortlist, T,
                                                                     S, p.blank, L, LS);
  if (rs)
    ctc_stream_shortlist_kernel<Fuse><<<B, DEC_THREADS, smem, stream>>>(p, shortlist, L, LS, fu,
                                                                       *rs);
  else
    ctc_prefix_beam_shortlist_kernel<Fuse><<<B, DEC_THREADS, smem, stream>>>(p, shortlist, L, LS,
                                                                            fu);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

static int dec_check(int B, int T, int S, int beam_size, int blank) {
  if (B <= 0 || T <= 0 || S <= 0 || blank < 0 || blank >= S || beam_size <= 0) return SB_ERR_INVALID;
  if (beam_size > DEC_MAX_BEAM) return SB_ERR_UNSUPPORTED;
  return SB_OK;
}

template <class Fuse>
static int dec_entry(const float* logp, const int* lens, int B, int T, int S, int beam_size,
                     int blank, int* out_labels, int* out_lens, double* out_scores,
                     void* workspace, size_t workspace_bytes, void* stream_, bool force_shortlist,
                     const Fuse& fu) {
  if (!logp || !lens || !out_labels || !out_lens || !out_scores || !workspace) return SB_ERR_INVALID;
  const int rc = dec_check(B, T, S, beam_size, blank);
  if (rc != SB_OK) return rc;
  size_t need = 0;
  sb_ctc_prefix_beam_workspace_size(B, T, beam_size, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  DecParams p;
  p.logp = logp; p.lens = lens;
  p.trie = dec_trie(workspace, B, dec_node_cap(T, beam_size));
  p.out_labels = out_labels; p.out_lens = out_lens; p.out_scores = out_scores;
  p.B = B; p.T = T; p.S = S; p.K = beam_size; p.blank = blank;
  int* shortlist = reinterpret_cast<int*>(static_cast<unsigned char*>(workspace) +
                                          dec_shortlist_offset(B, T, beam_size));
  return dec_launch(p, fu, nullptr, shortlist, force_shortlist,
                    reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int sb_ctc_prefix_beam(const float* logp, const int* lens, int B, int T, int S,
                                  int beam_size, int blank, int* out_labels, int* out_lens,
                                  double* out_scores, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  return dec_entry(logp, lens, B, T, S, beam_size, blank, out_labels, out_lens, out_scores,
                   workspace, workspace_bytes, stream, false, NoFuse{});
}

extern "C" int sb_ctc_prefix_beam_shortlist(const float* logp, const int* lens, int B, int T,
                                            int S, int beam_size, int blank, int* out_labels,
                                            int* out_lens, double* out_scores, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  return dec_entry(logp, lens, B, T, S, beam_size, blank, out_labels, out_lens, out_scores,
                   workspace, workspace_bytes, stream, true, NoFuse{});
}

// The LM needs no workspace of its own: each entry's context lives in shared memory.
extern "C" int sb_ctc_prefix_beam_lm_workspace_size(int B, int T, int K, int order,
                                                    size_t* bytes) {
  if (order < 1) return SB_ERR_INVALID;
  if (order > SB_LM_MAX_ORDER) return SB_ERR_UNSUPPORTED;
  return sb_ctc_prefix_beam_workspace_size(B, T, K, bytes);
}

// The fusion policy of an LM and its weights, or the status that refuses them.
static int dec_lm_fuse(int S, int blank, const SbNgramLm* lm, double lm_weight,
                       double insertion_bonus, LmFuse* fu) {
  if (!lm || !lm->keys || !lm->vals || !lm->logp || !lm->bow || !lm->tok) return SB_ERR_INVALID;
  if (!(lm_weight >= 0.0) || !isfinite(lm_weight) || !isfinite(insertion_bonus))
    return SB_ERR_INVALID;
  if (!isfinite(lm->lm_upper) || !isfinite(lm->lm_abs) || lm->num_classes < S) return SB_ERR_INVALID;
  if (lm->blank != blank) return SB_ERR_INVALID;
  if (lm->cap <= 0 || (lm->cap & (lm->cap - 1)) || lm->order < 1) return SB_ERR_INVALID;
  if (lm->order > SB_LM_MAX_ORDER) return SB_ERR_UNSUPPORTED;
  fu->lm = *lm;
  fu->alpha = lm_weight;
  fu->beta = insertion_bonus;
  return SB_OK;
}

static int dec_lm_entry(const float* logp, const int* lens, int B, int T, int S, int beam_size,
                        int blank, const SbNgramLm* lm, double lm_weight, double insertion_bonus,
                        int* out_labels, int* out_lens, double* out_scores, void* workspace,
                        size_t workspace_bytes, void* stream, bool force_shortlist) {
  LmFuse fu;
  const int rc = dec_lm_fuse(S, blank, lm, lm_weight, insertion_bonus, &fu);
  if (rc != SB_OK) return rc;
  return dec_entry(logp, lens, B, T, S, beam_size, blank, out_labels, out_lens, out_scores,
                   workspace, workspace_bytes, stream, force_shortlist, fu);
}

extern "C" int sb_ctc_prefix_beam_lm(const float* logp, const int* lens, int B, int T, int S,
                                     int beam_size, int blank, const SbNgramLm* lm,
                                     double lm_weight, double insertion_bonus, int* out_labels,
                                     int* out_lens, double* out_scores, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  return dec_lm_entry(logp, lens, B, T, S, beam_size, blank, lm, lm_weight, insertion_bonus,
                      out_labels, out_lens, out_scores, workspace, workspace_bytes, stream, false);
}

extern "C" int sb_ctc_prefix_beam_lm_shortlist(const float* logp, const int* lens, int B, int T,
                                               int S, int beam_size, int blank,
                                               const SbNgramLm* lm, double lm_weight,
                                               double insertion_bonus, int* out_labels,
                                               int* out_lens, double* out_scores, void* workspace,
                                               size_t workspace_bytes, void* stream) {
  return dec_lm_entry(logp, lens, B, T, S, beam_size, blank, lm, lm_weight, insertion_bonus,
                      out_labels, out_lens, out_scores, workspace, workspace_bytes, stream, true);
}

// ------------------------------------------------------------------------------------------------
// Resumable search (sb_ctc_stream_*).  State: B DecSlots, then the trie arena of B streams of
// max_frames * K + 1 nodes, laid out as the offline search's workspace lays out B utterances.
// ------------------------------------------------------------------------------------------------
static int dec_stream_check(int B, int max_frames, int beam_size) {
  if (B <= 0 || max_frames <= 0 || beam_size <= 0) return SB_ERR_INVALID;
  if (beam_size > DEC_MAX_BEAM) return SB_ERR_UNSUPPORTED;
  return SB_OK;
}

static BeamTrie dec_stream_trie(void* state, int B, int max_frames, int beam_size) {
  return dec_trie(static_cast<unsigned char*>(state) + (size_t)B * DEC_SLOT_BYTES, B,
                  dec_node_cap(max_frames, beam_size));
}

extern "C" int sb_ctc_stream_state_size(int B, int max_frames, int beam_size, int order,
                                        size_t* bytes) {
  if (!bytes || order < 0) return SB_ERR_INVALID;
  if (order > SB_LM_MAX_ORDER) return SB_ERR_UNSUPPORTED;
  const int rc = dec_stream_check(B, max_frames, beam_size);
  if (rc != SB_OK) return rc;
  *bytes = (size_t)B * DEC_SLOT_BYTES + dec_shortlist_offset(B, max_frames, beam_size);
  return SB_OK;
}

extern "C" int sb_ctc_stream_workspace_size(int B, int T, int beam_size, size_t* bytes) {
  if (!bytes || B <= 0 || T <= 0 || beam_size <= 0) return SB_ERR_INVALID;
  *bytes = (size_t)B * T * (2 * beam_size + 1) * sizeof(int);
  return SB_OK;
}

extern "C" int sb_ctc_stream_reset(void* state, int B, int max_frames, int beam_size, int first,
                                   int count, void* stream) {
  if (!state) return SB_ERR_INVALID;
  const int rc = dec_stream_check(B, max_frames, beam_size);
  if (rc != SB_OK) return rc;
  if (first < 0 || count <= 0 || count > B - first) return SB_ERR_INVALID;
  ctc_stream_reset_kernel<<<count, DEC_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      dec_stream_trie(state, B, max_frames, beam_size), state, first);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

template <class Fuse>
static int dec_stream_entry(const float* logp, const int* n, int B, int T, int S, int beam_size,
                            int blank, int max_frames, void* state, void* workspace,
                            size_t workspace_bytes, void* stream, bool force_shortlist,
                            const Fuse& fu) {
  if (!logp || !n || !state || !workspace) return SB_ERR_INVALID;
  int rc = dec_check(B, T, S, beam_size, blank);
  if (rc != SB_OK) return rc;
  rc = dec_stream_check(B, max_frames, beam_size);
  if (rc != SB_OK) return rc;
  size_t need = 0;
  sb_ctc_stream_workspace_size(B, T, beam_size, &need);
  if (workspace_bytes < need) return SB_ERR_WORKSPACE;
  DecParams p;
  memset(&p, 0, sizeof(p));
  p.logp = logp; p.lens = n;
  p.trie = dec_stream_trie(state, B, max_frames, beam_size);
  p.B = B; p.T = T; p.S = S; p.K = beam_size; p.blank = blank;
  DecResume rs;
  rs.slots = state;
  rs.max_frames = max_frames;
  return dec_launch(p, fu, &rs, static_cast<int*>(workspace), force_shortlist,
                    reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int sb_ctc_stream_step(const float* logp, const int* n, int B, int T, int S,
                                  int beam_size, int blank, int max_frames, void* state,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  return dec_stream_entry(logp, n, B, T, S, beam_size, blank, max_frames, state, workspace,
                          workspace_bytes, stream, false, NoFuse{});
}

extern "C" int sb_ctc_stream_step_shortlist(const float* logp, const int* n, int B, int T, int S,
                                            int beam_size, int blank, int max_frames, void* state,
                                            void* workspace, size_t workspace_bytes,
                                            void* stream) {
  return dec_stream_entry(logp, n, B, T, S, beam_size, blank, max_frames, state, workspace,
                          workspace_bytes, stream, true, NoFuse{});
}

static int dec_stream_lm_entry(const float* logp, const int* n, int B, int T, int S,
                               int beam_size, int blank, const SbNgramLm* lm, double lm_weight,
                               double insertion_bonus, int max_frames, void* state,
                               void* workspace, size_t workspace_bytes, void* stream,
                               bool force_shortlist) {
  LmFuse fu;
  const int rc = dec_lm_fuse(S, blank, lm, lm_weight, insertion_bonus, &fu);
  if (rc != SB_OK) return rc;
  return dec_stream_entry(logp, n, B, T, S, beam_size, blank, max_frames, state, workspace,
                          workspace_bytes, stream, force_shortlist, fu);
}

extern "C" int sb_ctc_stream_step_lm(const float* logp, const int* n, int B, int T, int S,
                                     int beam_size, int blank, const SbNgramLm* lm,
                                     double lm_weight, double insertion_bonus, int max_frames,
                                     void* state, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  return dec_stream_lm_entry(logp, n, B, T, S, beam_size, blank, lm, lm_weight, insertion_bonus,
                             max_frames, state, workspace, workspace_bytes, stream, false);
}

extern "C" int sb_ctc_stream_step_lm_shortlist(const float* logp, const int* n, int B, int T,
                                               int S, int beam_size, int blank,
                                               const SbNgramLm* lm, double lm_weight,
                                               double insertion_bonus, int max_frames,
                                               void* state, void* workspace,
                                               size_t workspace_bytes, void* stream) {
  return dec_stream_lm_entry(logp, n, B, T, S, beam_size, blank, lm, lm_weight, insertion_bonus,
                             max_frames, state, workspace, workspace_bytes, stream, true);
}

extern "C" int sb_ctc_stream_best(const void* state, int B, int max_frames, int beam_size,
                                  int* out_labels, int* out_lens, double* out_scores,
                                  int* out_overflow, void* stream) {
  if (!state || !out_labels || !out_lens || !out_scores || !out_overflow) return SB_ERR_INVALID;
  const int rc = dec_stream_check(B, max_frames, beam_size);
  if (rc != SB_OK) return rc;
  DecParams p;
  memset(&p, 0, sizeof(p));
  p.trie = dec_stream_trie(const_cast<void*>(state), B, max_frames, beam_size);
  p.out_labels = out_labels; p.out_lens = out_lens; p.out_scores = out_scores;
  p.B = B; p.T = max_frames; p.K = beam_size;
  ctc_stream_best_kernel<<<B, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, state,
                                                                              out_overflow);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_ctc_stream_nbest(const void* state, int B, int max_frames, int beam_size,
                                   int* out_labels, int* out_lens, double* out_scores,
                                   int* out_count, void* stream) {
  if (!state || !out_labels || !out_lens || !out_scores || !out_count) return SB_ERR_INVALID;
  const int rc = dec_stream_check(B, max_frames, beam_size);
  if (rc != SB_OK) return rc;
  ctc_stream_nbest_kernel<<<B, DEC_MAX_BEAM, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      dec_stream_trie(const_cast<void*>(state), B, max_frames, beam_size), state, beam_size,
      max_frames, out_labels, out_lens, out_scores, out_count);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_debug_ctc_lm_rescans(unsigned long long* frames) {
  if (!frames) return SB_ERR_INVALID;
  const unsigned long long zero = 0;
  if (cudaMemcpyFromSymbol(frames, dec_lm_rescans, sizeof(zero)) != cudaSuccess ||
      cudaMemcpyToSymbol(dec_lm_rescans, &zero, sizeof(zero)) != cudaSuccess)
    return SB_ERR_CUDA;
  return SB_OK;
}

// ------------------------------------------------------------------------------------------------
// Word LM (SbWordLm): the same routes and state over WordLmFuse.
// ------------------------------------------------------------------------------------------------
static int dec_wordlm_fuse(int S, int blank, const SbWordLm* lm, double lm_weight,
                           double insertion_bonus, double oov_penalty, WordLmFuse* fu) {
  return word_lm_terms(lm, lm_weight, insertion_bonus, oov_penalty, S,
                       [&](const SbWordLm& l) { return l.blank == blank && l.delimiter != blank; },
                       fu);
}

static int dec_wordlm_entry(const float* logp, const int* lens, int B, int T, int S, int beam_size,
                            int blank, const SbWordLm* lm, double lm_weight,
                            double insertion_bonus, double oov_penalty, int* out_labels,
                            int* out_lens, double* out_scores, void* workspace,
                            size_t workspace_bytes, void* stream, bool force_shortlist) {
  WordLmFuse fu;
  const int rc = dec_wordlm_fuse(S, blank, lm, lm_weight, insertion_bonus, oov_penalty, &fu);
  if (rc != SB_OK) return rc;
  return dec_entry(logp, lens, B, T, S, beam_size, blank, out_labels, out_lens, out_scores,
                   workspace, workspace_bytes, stream, force_shortlist, fu);
}

extern "C" int sb_ctc_prefix_beam_wordlm(const float* logp, const int* lens, int B, int T, int S,
                                         int beam_size, int blank, const SbWordLm* lm,
                                         double lm_weight, double insertion_bonus,
                                         double oov_penalty, int* out_labels, int* out_lens,
                                         double* out_scores, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  return dec_wordlm_entry(logp, lens, B, T, S, beam_size, blank, lm, lm_weight, insertion_bonus,
                          oov_penalty, out_labels, out_lens, out_scores, workspace,
                          workspace_bytes, stream, false);
}

extern "C" int sb_ctc_prefix_beam_wordlm_shortlist(const float* logp, const int* lens, int B,
                                                   int T, int S, int beam_size, int blank,
                                                   const SbWordLm* lm, double lm_weight,
                                                   double insertion_bonus, double oov_penalty,
                                                   int* out_labels, int* out_lens,
                                                   double* out_scores, void* workspace,
                                                   size_t workspace_bytes, void* stream) {
  return dec_wordlm_entry(logp, lens, B, T, S, beam_size, blank, lm, lm_weight, insertion_bonus,
                          oov_penalty, out_labels, out_lens, out_scores, workspace,
                          workspace_bytes, stream, true);
}

static int dec_stream_wordlm_entry(const float* logp, const int* n, int B, int T, int S,
                                   int beam_size, int blank, const SbWordLm* lm, double lm_weight,
                                   double insertion_bonus, double oov_penalty, int max_frames,
                                   void* state, void* workspace, size_t workspace_bytes,
                                   void* stream, bool force_shortlist) {
  WordLmFuse fu;
  const int rc = dec_wordlm_fuse(S, blank, lm, lm_weight, insertion_bonus, oov_penalty, &fu);
  if (rc != SB_OK) return rc;
  return dec_stream_entry(logp, n, B, T, S, beam_size, blank, max_frames, state, workspace,
                          workspace_bytes, stream, force_shortlist, fu);
}

extern "C" int sb_ctc_stream_step_wordlm(const float* logp, const int* n, int B, int T, int S,
                                         int beam_size, int blank, const SbWordLm* lm,
                                         double lm_weight, double insertion_bonus,
                                         double oov_penalty, int max_frames, void* state,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  return dec_stream_wordlm_entry(logp, n, B, T, S, beam_size, blank, lm, lm_weight,
                                 insertion_bonus, oov_penalty, max_frames, state, workspace,
                                 workspace_bytes, stream, false);
}

extern "C" int sb_ctc_stream_step_wordlm_shortlist(const float* logp, const int* n, int B, int T,
                                                   int S, int beam_size, int blank,
                                                   const SbWordLm* lm, double lm_weight,
                                                   double insertion_bonus, double oov_penalty,
                                                   int max_frames, void* state, void* workspace,
                                                   size_t workspace_bytes, void* stream) {
  return dec_stream_wordlm_entry(logp, n, B, T, S, beam_size, blank, lm, lm_weight,
                                 insertion_bonus, oov_penalty, max_frames, state, workspace,
                                 workspace_bytes, stream, true);
}

extern "C" int sb_ctc_stream_best_wordlm(const void* state, int B, int max_frames, int beam_size,
                                         const SbWordLm* lm, double lm_weight,
                                         double insertion_bonus, double oov_penalty,
                                         int* out_labels, int* out_lens, double* out_scores,
                                         int* out_overflow, void* stream) {
  if (!state || !out_labels || !out_lens || !out_scores || !out_overflow || !lm)
    return SB_ERR_INVALID;
  WordLmFuse fu;
  int rc = dec_wordlm_fuse(lm->num_classes, lm->blank, lm, lm_weight, insertion_bonus,
                           oov_penalty, &fu);
  if (rc != SB_OK) return rc;
  rc = dec_stream_check(B, max_frames, beam_size);
  if (rc != SB_OK) return rc;
  DecParams p;
  memset(&p, 0, sizeof(p));
  p.trie = dec_stream_trie(const_cast<void*>(state), B, max_frames, beam_size);
  p.out_labels = out_labels; p.out_lens = out_lens; p.out_scores = out_scores;
  p.B = B; p.T = max_frames; p.K = beam_size;
  ctc_stream_best_wordlm_kernel<<<B, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      p, state, out_overflow, fu);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
