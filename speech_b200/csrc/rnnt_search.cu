// Label-free transducer beam search: the search of tdecode.cu with each lattice row computed from
// the hypothesis itself instead of read from a teacher-forced lattice.  The host loop
// (transducer_decoders.search_batch) enqueues, per frame t and level l = 0 .. S
// (S = max_symbols_per_frame):
//   rows of the level's frontier at frame t (joint network, csrc/joint*.cu)
//   sb_rnnt_search_round     blank emissions into `done`; for l < S the K best extensions of
//                            hypotheses shorter than max_len, inserted into the trie; per new
//                            frontier slot its parent slot, symbol and length
//   sb_rnnt_pred_step        (l < S, once per prediction-network layer) the GRU states of the new
//                            frontier from the parents' states
// and at the end of the frame sb_rnnt_search_frame_end (the K best of `done` become the beam; their
// prediction states are gathered into the beam's slots), after the last one sb_rnnt_search_final.
// The rounds are tsearch.cuh's, so with rows lat[t, len(h)] and S = max_len = U - 1 this is
// sb_rnnt_decode_static bit for bit.  One CTA per utterance; the search state lives in the
// workspace between launches; an utterance past its frames, or whose frame has no live frontier
// left, returns at once.
//
// With an n-gram LM (shallow fusion) the loop enqueues sb_rnnt_search_lm_rows between the rows and
// the round: per live frontier slot it resolves the hypothesis's LM context once (the trie walked
// up at most order - 1 labels; the root reads as <s>) and turns the acoustic f32 row into fused
// float64 values f_k = (double)lp_k + (alpha * lm(k | h) + beta), f_blank = (double)lp_blank:
// whole rows for the full route, or the kp best by (f desc, k asc) with the (kp+1)-th value for
// the shortlist route, so that the lists are ranked by the value the search selects on.  One CTA
// of RL_THREADS per slot spreads the row's lookups over the GPU; each warp streams its classes
// through the top-P selection of shortlist.cuh and warp 0 merges the warps' lists.
// sb_rnnt_search_round_lm is then the round over float64 rows / lists: the round kernel knows
// nothing of the LM, and with alpha = beta = 0 (f = (double)lp exactly) it searches what the f32
// round searches.
//
// Prediction states live in an arena of S + 2 blocks of B x K slots: block l (1 .. S) holds the
// frontier of level l, blocks 0 and S + 1 take turns as the beam (`cur`) and the next beam.
// A frontier slot is named by the code level * K + i.
//
// sb_rnnt_pred_step is one GRU layer over R = B*K rows in fp32 on CUDA cores, the arithmetic of
// s2s_cell_fwd (csrc/s2s.cu) with its structure (one warp per hidden unit, lanes over K, a group of
// rows per CTA staged in shared memory), generalised to an input of any width (embedding_dim or H)
// gathered by symbol, and a hidden state gathered from the parent's slot.
#include "ngram.cuh"
#include "shortlist.cuh"
#include "tsearch.cuh"
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int RS_THREADS = 128;
static constexpr int RS_MAX_BEAM = 32;
static constexpr int RS_MAX_KP = 64;
static constexpr size_t RS_SMEM_MAX = 200 * 1024;

// search state of one utterance between launches
struct RsState {
  double beam_s[RS_MAX_BEAM], fr_s[RS_MAX_BEAM];
  int beam_n[RS_MAX_BEAM], beam_l[RS_MAX_BEAM], beam_src[RS_MAX_BEAM];
  int fr_n[RS_MAX_BEAM], fr_l[RS_MAX_BEAM];
  int nbeam, nfr, ndone, round_id, nflag, pad_[3];
};

struct RsSizes { size_t node_cap, hcap, done_cap, total; };
static RsSizes rs_sizes(int B, int T, int S, int K) {
  RsSizes s;
  s.node_cap = (size_t)T * S * K + 2;
  s.hcap = (size_t)beam_pow2_cap(2 * s.node_cap);
  s.done_cap = (size_t)K * (S + 1) + 1;
  s.total = 1024 + (size_t)B * (sizeof(RsState) + 2 * s.node_cap * sizeof(int) +
                                s.hcap * (sizeof(unsigned long long) + sizeof(int)) +
                                s.done_cap * (sizeof(double) + 3 * sizeof(int))) + 4096;
  return s;
}

struct RsWs {
  RsState* st;
  BeamTrie trie;         // utterance 0 of B
  double* done_score;    // (B, done_cap)
  int *done_node, *done_len, *done_src;
  int done_cap;
};

static RsWs rs_carve(void* workspace, int B, const RsSizes& sz) {
  RsWs w;
  uintptr_t a = (reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255;
  w.st = reinterpret_cast<RsState*>(a);
  a += (size_t)B * sizeof(RsState);
  w.trie.keys = reinterpret_cast<unsigned long long*>(a);
  a += (size_t)B * sz.hcap * sizeof(unsigned long long);
  w.done_score = reinterpret_cast<double*>(a);
  a += (size_t)B * sz.done_cap * sizeof(double);
  w.trie.vals = reinterpret_cast<int*>(a);
  a += (size_t)B * sz.hcap * sizeof(int);
  w.trie.nodes = reinterpret_cast<int*>(a);
  a += (size_t)B * 2 * sz.node_cap * sizeof(int);
  w.done_node = reinterpret_cast<int*>(a);
  a += (size_t)B * sz.done_cap * sizeof(int);
  w.done_len = reinterpret_cast<int*>(a);
  a += (size_t)B * sz.done_cap * sizeof(int);
  w.done_src = reinterpret_cast<int*>(a);
  w.trie.cap = (int)sz.hcap;
  w.trie.node_cap = (int)sz.node_cap;
  w.done_cap = (int)sz.done_cap;
  return w;
}

// ---- search kernels --------------------------------------------------------------------------

// utterances first + blockIdx.x: the empty hypothesis at frame 0
__global__ void __launch_bounds__(RS_THREADS) rnnt_search_init_kernel(RsWs w, int K, int* slot_lens,
                                                                      int first) {
  const int b = first + blockIdx.x, tid = threadIdx.x;
  w.trie.of(b).clear<RS_THREADS>();
  if (tid == 0) {
    RsState& s = w.st[b];
    s.nbeam = 1; s.beam_s[0] = 0.0; s.beam_n[0] = 0; s.beam_l[0] = 0; s.beam_src[0] = 0;
    s.nfr = 0; s.ndone = 0; s.round_id = 0; s.nflag = 0;
  }
  if (tid < K) slot_lens[b * K + tid] = 0;
}

// R: the value type of rows and lists, float (acoustic log-probabilities) or double (LM-fused)
template <class R>
struct RsRoundParams {
  RsWs w;
  const R* lp;            // (B, K, V) rows of the level's frontier slots (full route)
  const R* sl_val;        // (B, K, kp) shortlists of the same rows (shortlist route)
  const int* sl_idx;
  const R* sl_meta;       // (B, K, 2)
  const int* tlens;
  int* par;               // (B, K) out: parent slot of each new frontier slot, -2 = none
  int* sym;               // (B, K) out: its symbol
  int* slot_lens;         // (B, K) out: its length
  int t, level, S, max_len, K, V, kp, blank;
};

template <bool SHORT, class R>
__global__ void __launch_bounds__(RS_THREADS, 1) rnnt_search_round_kernel(const RsRoundParams<R> p) {
  extern __shared__ unsigned char rs_smem[];
  const int b = blockIdx.x, tid = threadIdx.x, K = p.K, V = p.V;
  __shared__ double fr_s[RS_MAX_BEAM], new_s[RS_MAX_BEAM];
  __shared__ int fr_n[RS_MAX_BEAM], fr_l[RS_MAX_BEAM];
  __shared__ int new_n[RS_MAX_BEAM], new_l[RS_MAX_BEAM], new_p[RS_MAX_BEAM], new_k[RS_MAX_BEAM];
  __shared__ int nfr, ndone, round_id, nflag;
  RsState& st = p.w.st[b];
  const int lvl = p.level;
  if (tid == 0) {
    nfr = p.t < p.tlens[b] ? (lvl == 0 ? st.nbeam : st.nfr) : 0;
    ndone = lvl == 0 ? 0 : st.ndone;
    round_id = st.round_id;
    nflag = st.nflag;
  }
  __syncthreads();
  const int nf = nfr;
  if (nf == 0) {                                  // past its frames, or no live frontier
    if (tid < K) p.par[b * K + tid] = -2;
    return;
  }
  if (tid < nf) {
    fr_s[tid] = lvl == 0 ? st.beam_s[tid] : st.fr_s[tid];
    fr_n[tid] = lvl == 0 ? st.beam_n[tid] : st.fr_n[tid];
    fr_l[tid] = lvl == 0 ? st.beam_l[tid] : st.fr_l[tid];
  }
  __syncthreads();
  const BeamTrie trie = p.w.trie.of(b);
  const size_t d0 = (size_t)b * p.w.done_cap;
  const size_t row0 = (size_t)b * K;              // row of frontier slot i: row0 + i
  ts_merge_blanks<RS_THREADS>(
      nf, fr_s, fr_n, fr_l, 0x7fffffff,
      [&](int i, int) {
        return SHORT ? p.sl_meta[2 * (row0 + i)] : p.lp[(row0 + i) * V + p.blank];
      },
      p.w.done_score + d0, p.w.done_node + d0, p.w.done_len + d0, p.w.done_src + d0, lvl * K,
      &ndone, p.w.done_cap);
  int nsel = -1;
  if (lvl < p.S) {
    const TsNew nw{new_s, new_n, new_l, new_p, new_k};
    const auto can_extend = [&](int i) { return fr_l[i] < p.max_len; };
    if (!SHORT) {
      nsel = ts_expand_full<RS_THREADS>(
          reinterpret_cast<double*>(rs_smem), K, V, p.blank, nf, fr_s, fr_n, fr_l, can_extend,
          [&](int i, int k) { return p.lp[(row0 + i) * V + k]; }, trie, round_id, nw);
    } else {
      nsel = ts_expand_shortlist<R>(
          K, V, p.kp, p.blank, nf, fr_s, fr_n, fr_l, can_extend,
          [&](int i, const R** lv, const int** li, R* beta) {
            *lv = p.sl_val + (row0 + i) * p.kp;
            *li = p.sl_idx + (row0 + i) * p.kp;
            *beta = p.sl_meta[2 * (row0 + i) + 1];
          },
          trie, round_id, nw, &nflag);
    }
  }
  const int ns = max(nsel, 0);
  if (tid < ns) {
    st.fr_s[tid] = new_s[tid]; st.fr_n[tid] = new_n[tid]; st.fr_l[tid] = new_l[tid];
  }
  if (tid < K) {
    p.par[row0 + tid] = tid < ns ? new_p[tid] : -2;
    p.sym[row0 + tid] = tid < ns ? new_k[tid] : -1;
    p.slot_lens[row0 + tid] = tid < ns ? new_l[tid] : 0;
  }
  if (tid == 0) {
    st.nfr = ns;
    st.ndone = ndone;
    st.round_id = round_id + (nsel >= 0 ? 1 : 0);
    st.nflag = nflag;
  }
}

// ---- LM-fused rows --------------------------------------------------------------------------
static constexpr int RL_THREADS = 256;
static constexpr int RL_WARPS = RL_THREADS / 32;

struct RsLmRowsParams {
  RsWs w;
  const float* lp;        // (B, K, V) acoustic rows of the level's frontier slots
  double* fused;          // (B, K, V) out: fused rows (full route), or null
  double* sl_val;         // (B, K, kp) out: fused shortlists (shortlist route)
  int* sl_idx;
  double* sl_meta;        // (B, K, 2) out: {blank lp, (kp+1)-th fused value or -inf}
  const int* tlens;
  SbNgramLm lm;
  double alpha, beta;
  int t, level, K, V, kp, blank;
};

// One CTA per frontier slot (b, i): grid B * K.
__global__ void __launch_bounds__(RL_THREADS) rnnt_search_lm_rows_kernel(const RsLmRowsParams p) {
  __shared__ double buf_v[RL_WARPS][SL_CAP];
  __shared__ int buf_i[RL_WARPS][SL_CAP];
  __shared__ int ctx[SB_LM_MAX_ORDER], cnt_w[RL_WARPS];
  __shared__ int depth_s;
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  const int b = blockIdx.x / p.K, i = blockIdx.x - b * p.K, V = p.V, blank = p.blank;
  const RsState& st = p.w.st[b];
  const int nf = p.t < p.tlens[b] ? (p.level == 0 ? st.nbeam : st.nfr) : 0;
  if (i >= nf) return;                            // the round reads no row of this slot
  if (tid == 0) {
    const int* nodes = p.w.trie.of(b).nodes;
    int q = p.level == 0 ? st.beam_n[i] : st.fr_n[i];
    depth_s = lm_context(p.lm, [&](int) {         // labels most recent first, then <s>
      if (q <= 0) return -1;
      const int sym = nodes[2 * q + 1];
      q = nodes[2 * q];
      return sym;
    }, ctx);
  }
  __syncthreads();
  const int depth = depth_s;
  const size_t row = (size_t)blockIdx.x;
  const float* lp = p.lp + row * V;
  const auto fuse = [&](int k, float x) {         // alpha * lm is not contracted into the + beta
    const double l = lm_backoff(p.lm, ctx, depth, __ldg(p.lm.tok + k));
    return (double)x + (__dmul_rn(p.alpha, l) + p.beta);
  };
  if (p.fused) {
    for (int k = tid; k < V; k += RL_THREADS) {
      const float x = lp[k];
      p.fused[row * V + k] = k == blank ? (double)x : fuse(k, x);
    }
    return;
  }
  // shortlist route: each warp streams classes wp*128 + [0, 128), then every RL_WARPS*128
  double* bv = buf_v[wp];
  int* bi = buf_i[wp];
  const int P = p.kp + 1;
  // f_k <= (double)lp_k + bound (alpha >= 0, rounding is monotone): a class whose bound falls below
  // the threshold cannot enter, and needs no lookup
  const double bound = __dmul_rn(p.alpha, p.lm.lm_upper) + p.beta;
  int cnt = 0, tk = 0;
  bool thr = false;
  double tv = 0.0;
  for (int base = wp * 128; base < V; base += RL_WARPS * 128) {
    double x[4];
    bool q[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = base + e * 32 + lane;
      q[e] = j < V && j != blank;
      x[e] = 0.0;
      if (q[e]) {
        const float a = lp[j];
        if (thr && (double)a + bound < tv) {
          q[e] = false;
        } else {
          x[e] = fuse(j, a);
          q[e] = !thr || sl_better(x[e], j, tv, tk);
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e)
      sl_push(bv, bi, cnt, thr, tv, tk, P, lane, q[e], x[e], base + e * 32 + lane);
  }
  sl_sort(bv, bi, cnt, lane);                     // each warp's P best first
  if (lane == 0) cnt_w[wp] = min(cnt, P);
  __syncthreads();
  if (wp != 0) return;
  // warp 0 merges the other warps' lists into its own
  cnt = cnt_w[0];
  thr = false;
  for (int w = 1; w < RL_WARPS; ++w)
    for (int c = 0; c < cnt_w[w]; c += 32) {
      const int e = c + lane;
      bool q = e < cnt_w[w];
      const double xv = q ? buf_v[w][e] : 0.0;
      const int k = q ? buf_i[w][e] : 0;
      q = q && (!thr || sl_better(xv, k, tv, tk));
      sl_push(bv, bi, cnt, thr, tv, tk, P, lane, q, xv, k);
    }
  sl_sort(bv, bi, cnt, lane);
  const int kp = p.kp;
  for (int e = lane; e < kp; e += 32) {
    p.sl_val[row * kp + e] = e < cnt ? bv[e] : -INFINITY;
    p.sl_idx[row * kp + e] = e < cnt ? bi[e] : -1;
  }
  if (lane == 0) {
    p.sl_meta[2 * row] = (double)lp[blank];
    p.sl_meta[2 * row + 1] = cnt > kp ? bv[kp] : -INFINITY;
  }
}

// block of the slot code c = level * K + i (level 0: the beam's block `cur`) and its slot i
SB_DEVINL int rs_block(int c, int K, int cur) { return c / K == 0 ? cur : c / K; }

__global__ void __launch_bounds__(RS_THREADS) rnnt_search_frame_end_kernel(
    RsWs w, const int* tlens, int t, int B, int K, int* slot_lens, float* hid, int layers, int H,
    float* fy, int Hj, int cur, int next) {
  const int b = blockIdx.x, tid = threadIdx.x;
  if (t >= tlens[b]) return;
  __shared__ double beam_s[RS_MAX_BEAM];
  __shared__ int beam_n[RS_MAX_BEAM], beam_l[RS_MAX_BEAM], beam_src[RS_MAX_BEAM];
  RsState& st = w.st[b];
  const size_t d0 = (size_t)b * w.done_cap;
  const int nb = ts_select_done<RS_THREADS>(w.done_score + d0, w.done_node + d0, w.done_len + d0,
                                            w.done_src + d0, st.ndone, K, beam_s, beam_n, beam_l,
                                            beam_src);
  __syncthreads();
  if (tid < nb) {
    st.beam_s[tid] = beam_s[tid]; st.beam_n[tid] = beam_n[tid]; st.beam_l[tid] = beam_l[tid];
    st.beam_src[tid] = beam_src[tid];
    slot_lens[b * K + tid] = beam_l[tid];
  }
  if (tid == 0) st.nbeam = nb;
  // the prediction states of the new beam into block `next`: hid [S+2][layers][B*K][H],
  // fy [S+2][B*K][Hj]
  const size_t BK = (size_t)B * K;
  for (int j = 0; j < nb; ++j) {
    const int c = beam_src[j];
    const size_t sb_ = (size_t)rs_block(c, K, cur), srow = (size_t)b * K + c % K;
    const size_t drow = (size_t)b * K + j;
    if (hid)
      for (int e = tid; e < layers * H; e += RS_THREADS) {
        const int l = e / H, h = e - l * H;
        hid[(((size_t)next * layers + l) * BK + drow) * H + h] =
            hid[((sb_ * layers + l) * BK + srow) * H + h];
      }
    if (fy)
      for (int e = tid; e < Hj; e += RS_THREADS)
        fy[((size_t)next * BK + drow) * Hj + e] = fy[(sb_ * BK + srow) * Hj + e];
  }
}

__global__ void rnnt_search_final_kernel(RsWs w, int* out_labels, int L, int* out_lens,
                                         double* out_scores, int* out_flags) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  const RsState& st = w.st[b];
  const int node = st.nbeam > 0 ? st.beam_n[0] : 0;
  out_lens[b] = w.trie.of(b).backtrack(node, out_labels + (size_t)b * L);
  out_scores[b] = st.nbeam > 0 ? st.beam_s[0] : -INFINITY;
  if (out_flags) out_flags[b] = st.nflag;
}

// ---- prediction-network step -------------------------------------------------------------------
static constexpr int PS_WARPS = 4;       // hidden units per CTA (one warp each)
static constexpr int PS_NB = 16;         // rows per CTA
static constexpr int PS_KC = 256;        // K chunk staged in shared memory

struct PredStepParams {
  const float* emb;      // [V][E] embedding (layer 0) or null
  const int* sym;        // [R] symbol of row r (-1: the zero start vector) or null (all zero)
  const float* x;        // [R][Kin] input rows (layers above 0) or null
  const float* h_prev;   // [R][H] block of the parents' states
  const int* par;        // [R] parent slot of row r in its utterance (-1: zero state, -2: skip)
  const float *w_ih, *w_hh, *b_ih, *b_hh;   // [3H][Kin], [3H][H], [3H], [3H]
  float* h;              // [R][H] out
  __nv_bfloat16* y;      // [R][ldy] out (bf16 copy of h, the fc1 GEMM operand) or null
  int R, K, Kin, H, ldy;
};

__global__ void __launch_bounds__(32 * PS_WARPS) rnnt_pred_step_kernel(const PredStepParams p) {
  __shared__ float xs[PS_NB][PS_KC];
  __shared__ int prow[PS_NB], psym[PS_NB];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = p.H, Kin = p.Kin;
  const int j = min(blockIdx.x * PS_WARPS + warp, H - 1);   // (clamped: all warps reach barriers)
  const bool owner = blockIdx.x * PS_WARPS + warp < H;
  const int r0 = blockIdx.y * PS_NB;
  const int nb = min(PS_NB, p.R - r0);
  if (tid < PS_NB) {
    const int r = r0 + tid;
    int pr = -2, sy = -1;
    if (tid < nb) {
      pr = p.par ? p.par[r] : -1;
      sy = p.sym ? p.sym[r] : -1;
      if (pr >= 0) pr += (r / p.K) * p.K;                 // the parent's row
    }
    prow[tid] = pr; psym[tid] = sy;
  }
  __syncthreads();
  float acc[PS_NB][6];
#pragma unroll
  for (int b = 0; b < PS_NB; ++b)
#pragma unroll
    for (int d = 0; d < 6; ++d) acc[b][d] = 0.f;
  // two passes over K: the input (W_ih, width Kin) and the hidden state (W_hh, width H)
  for (int pass = 0; pass < 2; ++pass) {
    const int W = pass == 0 ? Kin : H;
    const float* wm = pass == 0 ? p.w_ih : p.w_hh;
    for (int kc0 = 0; kc0 < W; kc0 += PS_KC) {
      const int nk = min(PS_KC, W - kc0);
      __syncthreads();                                   // the previous chunk has been consumed
      for (int e = tid; e < PS_NB * PS_KC; e += 32 * PS_WARPS) {
        const int r = e / PS_KC, c = e - r * PS_KC;
        float v = 0.f;
        if (r < nb && c < nk && prow[r] != -2) {
          const long long row = r0 + r;
          if (pass == 1) {
            if (prow[r] >= 0) v = p.h_prev[(long long)prow[r] * H + kc0 + c];
          } else if (p.x) {
            v = p.x[row * Kin + kc0 + c];
          } else if (psym[r] >= 0) {
            v = p.emb[(long long)psym[r] * Kin + kc0 + c];
          }
        }
        xs[r][c] = v;
      }
      __syncthreads();
      for (int c = lane; c < nk; c += 32) {
        float wv[3];
#pragma unroll
        for (int g = 0; g < 3; ++g) wv[g] = __ldg(wm + ((long long)g * H + j) * W + kc0 + c);
#pragma unroll
        for (int b = 0; b < PS_NB; ++b) {
          const float xv = xs[b][c];
#pragma unroll
          for (int g = 0; g < 3; ++g) acc[b][3 * pass + g] = fmaf(wv[g], xv, acc[b][3 * pass + g]);
        }
      }
    }
  }
  float mine[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int b = 0; b < PS_NB; ++b)
#pragma unroll
    for (int d = 0; d < 6; ++d) {
      const float v = warp_sum(acc[b][d]);
      if (lane == b) mine[d] = v;
    }
  if (owner && lane < nb && prow[lane] != -2) {
    const long long r = r0 + lane;
    const float gir = mine[0] + p.b_ih[j], giz = mine[1] + p.b_ih[H + j], gin = mine[2] + p.b_ih[2 * H + j];
    const float ghr = mine[3] + p.b_hh[j], ghz = mine[4] + p.b_hh[H + j], ghn = mine[5] + p.b_hh[2 * H + j];
    const float rg = 1.f / (1.f + expf(-(gir + ghr)));
    const float z = 1.f / (1.f + expf(-(giz + ghz)));
    const float n = tanhf(gin + rg * ghn);
    const float hp = prow[lane] >= 0 ? p.h_prev[(long long)prow[lane] * H + j] : 0.f;
    const float hn = (1.f - z) * n + z * hp;
    p.h[r * H + j] = hn;
    if (p.y) p.y[r * p.ldy + j] = __float2bfloat16(hn);
  }
}

}  // namespace sb

using namespace sb;

extern "C" int sb_rnnt_search_workspace_size(int B, int T, int S, int beam_size, size_t* bytes) {
  if (!bytes || B <= 0 || T <= 0 || S <= 0 || beam_size <= 0) return SB_ERR_INVALID;
  *bytes = rs_sizes(B, T, S, beam_size).total;
  return SB_OK;
}

static int rs_ws(void* workspace, size_t workspace_bytes, int B, int T, int S, int K, RsWs* w) {
  if (!workspace || B <= 0 || T <= 0 || S <= 0 || K <= 0) return SB_ERR_INVALID;
  if (K > RS_MAX_BEAM) return SB_ERR_UNSUPPORTED;
  const RsSizes sz = rs_sizes(B, T, S, K);
  if (workspace_bytes < sz.total) return SB_ERR_WORKSPACE;
  *w = rs_carve(workspace, B, sz);
  return SB_OK;
}

extern "C" int sb_rnnt_search_init(int* slot_lens, int B, int T, int S, int beam_size,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  RsWs w;
  const int rc = rs_ws(workspace, workspace_bytes, B, T, S, beam_size, &w);
  if (rc != SB_OK) return rc;
  if (!slot_lens) return SB_ERR_INVALID;
  rnnt_search_init_kernel<<<B, RS_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, beam_size, slot_lens, 0);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_search_reset(int* slot_lens, int B, int T, int S, int beam_size, int first,
                                    int count, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  if (!slot_lens || first < 0 || count <= 0 || count > B - first) return SB_ERR_INVALID;
  RsWs w;
  const int rc = rs_ws(workspace, workspace_bytes, B, T, S, beam_size, &w);
  if (rc != SB_OK) return rc;
  rnnt_search_init_kernel<<<count, RS_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, beam_size, slot_lens, first);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

template <class R>
static int rs_round(const R* lp, const R* sl_val, const int* sl_idx, const R* sl_meta, int kp,
                    const int* tlens, int t, int level, int max_len, int* par, int* sym,
                    int* slot_lens, int B, int T, int S, int V, int beam_size, int blank,
                    void* workspace, size_t workspace_bytes, void* stream_) {
  RsRoundParams<R> p;
  const int rc = rs_ws(workspace, workspace_bytes, B, T, S, beam_size, &p.w);
  if (rc != SB_OK) return rc;
  const bool shortlist = lp == nullptr;
  if (!tlens || !par || !sym || !slot_lens || V <= 0 || blank < 0 || blank >= V || t < 0 ||
      t >= T || level < 0 || level > S || max_len < 0)
    return SB_ERR_INVALID;
  if (shortlist && (!sl_val || !sl_idx || !sl_meta || kp < beam_size)) return SB_ERR_INVALID;
  if (shortlist && kp > RS_MAX_KP) return SB_ERR_UNSUPPORTED;
  const size_t smem = shortlist ? 0 : (size_t)beam_size * V * sizeof(double) + 16;
  if (smem > RS_SMEM_MAX) return SB_ERR_UNSUPPORTED;
  p.lp = lp; p.sl_val = sl_val; p.sl_idx = sl_idx; p.sl_meta = sl_meta; p.tlens = tlens;
  p.par = par; p.sym = sym; p.slot_lens = slot_lens;
  p.t = t; p.level = level; p.S = S; p.max_len = max_len; p.K = beam_size; p.V = V;
  p.kp = shortlist ? kp : 0; p.blank = blank;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (shortlist) {
    rnnt_search_round_kernel<true, R><<<B, RS_THREADS, 0, stream>>>(p);
  } else {
    if (smem > 40 * 1024 &&
        cudaFuncSetAttribute(rnnt_search_round_kernel<false, R>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return SB_ERR_CUDA;
    rnnt_search_round_kernel<false, R><<<B, RS_THREADS, smem, stream>>>(p);
  }
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_search_round(const float* lp, const float* sl_val, const int* sl_idx,
                                    const float* sl_meta, int kp, const int* tlens, int t,
                                    int level, int max_len, int* par, int* sym, int* slot_lens,
                                    int B, int T, int S, int V, int beam_size, int blank,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  return rs_round(lp, sl_val, sl_idx, sl_meta, kp, tlens, t, level, max_len, par, sym, slot_lens,
                  B, T, S, V, beam_size, blank, workspace, workspace_bytes, stream);
}

extern "C" int sb_rnnt_search_round_lm(const double* lp, const double* sl_val, const int* sl_idx,
                                       const double* sl_meta, int kp, const int* tlens, int t,
                                       int level, int max_len, int* par, int* sym, int* slot_lens,
                                       int B, int T, int S, int V, int beam_size, int blank,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  return rs_round(lp, sl_val, sl_idx, sl_meta, kp, tlens, t, level, max_len, par, sym, slot_lens,
                  B, T, S, V, beam_size, blank, workspace, workspace_bytes, stream);
}

extern "C" int sb_rnnt_search_lm_rows(const float* lp, double* fused, double* sl_val, int* sl_idx,
                                      double* sl_meta, int kp, const int* tlens, int t, int level,
                                      int B, int T, int S, int V, int beam_size, int blank,
                                      const SbNgramLm* lm, double lm_weight,
                                      double insertion_bonus, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  RsLmRowsParams p;
  const int rc = rs_ws(workspace, workspace_bytes, B, T, S, beam_size, &p.w);
  if (rc != SB_OK) return rc;
  const bool shortlist = fused == nullptr;
  if (!lp || !tlens || V <= 0 || blank < 0 || blank >= V || t < 0 || t >= T || level < 0 ||
      level > S)
    return SB_ERR_INVALID;
  if (shortlist && (!sl_val || !sl_idx || !sl_meta || kp < beam_size)) return SB_ERR_INVALID;
  if (!lm || !lm->keys || !lm->vals || !lm->logp || !lm->bow || !lm->tok) return SB_ERR_INVALID;
  if (!(lm_weight >= 0.0) || !isfinite(lm_weight) || !isfinite(insertion_bonus))
    return SB_ERR_INVALID;
  if (!isfinite(lm->lm_upper) || !isfinite(lm->lm_abs) || lm->num_classes < V) return SB_ERR_INVALID;
  if (lm->blank != blank) return SB_ERR_INVALID;
  if (lm->cap <= 0 || (lm->cap & (lm->cap - 1)) || lm->order < 1) return SB_ERR_INVALID;
  if (lm->order > SB_LM_MAX_ORDER) return SB_ERR_UNSUPPORTED;
  if (shortlist && kp > SL_MAX_KP) return SB_ERR_UNSUPPORTED;
  if ((long long)B * beam_size > 0x7fffffffLL) return SB_ERR_UNSUPPORTED;
  p.lp = lp; p.fused = fused; p.sl_val = sl_val; p.sl_idx = sl_idx; p.sl_meta = sl_meta;
  p.tlens = tlens; p.lm = *lm; p.alpha = lm_weight; p.beta = insertion_bonus;
  p.t = t; p.level = level; p.K = beam_size; p.V = V; p.kp = shortlist ? kp : 0; p.blank = blank;
  rnnt_search_lm_rows_kernel<<<B * beam_size, RL_THREADS, 0,
                               reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_search_frame_end(const int* tlens, int t, int* slot_lens, float* hid,
                                        int layers, int H, float* fy, int Hj, int cur, int next,
                                        int B, int T, int S, int beam_size, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  RsWs w;
  const int rc = rs_ws(workspace, workspace_bytes, B, T, S, beam_size, &w);
  if (rc != SB_OK) return rc;
  if (!tlens || !slot_lens || t < 0 || t >= T || (hid && (layers <= 0 || H <= 0)) ||
      (fy && Hj <= 0))
    return SB_ERR_INVALID;
  if ((cur != 0 && cur != S + 1) || next != S + 1 - cur) return SB_ERR_INVALID;
  rnnt_search_frame_end_kernel<<<B, RS_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, tlens, t, B, beam_size, slot_lens, hid, layers, H, fy, Hj, cur, next);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_search_final(int* out_labels, int max_len, int* out_lens,
                                    double* out_scores, int* out_flags, int B, int T, int S,
                                    int beam_size, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  RsWs w;
  const int rc = rs_ws(workspace, workspace_bytes, B, T, S, beam_size, &w);
  if (rc != SB_OK) return rc;
  if (!out_labels || !out_lens || !out_scores || max_len <= 0) return SB_ERR_INVALID;
  rnnt_search_final_kernel<<<B, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, out_labels, max_len, out_lens, out_scores, out_flags);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_rnnt_pred_step(const float* emb, const int* sym, const float* x,
                                 const float* h_prev, const int* par, const float* w_ih,
                                 const float* w_hh, const float* b_ih, const float* b_hh, float* h,
                                 void* y_bf16, int ldy, int R, int K, int Kin, int H,
                                 void* stream) {
  if (!w_ih || !w_hh || !b_ih || !b_hh || !h || R <= 0 || K <= 0 || R % K != 0 || Kin <= 0 ||
      H <= 0 || (sym && !emb) || (x && sym) || (par && !h_prev) || (y_bf16 && ldy < H))
    return SB_ERR_INVALID;
  if ((R + PS_NB - 1) / PS_NB > 65535) return SB_ERR_UNSUPPORTED;
  PredStepParams p;
  p.emb = emb; p.sym = sym; p.x = x; p.h_prev = h_prev; p.par = par;
  p.w_ih = w_ih; p.w_hh = w_hh; p.b_ih = b_ih; p.b_hh = b_hh; p.h = h;
  p.y = reinterpret_cast<__nv_bfloat16*>(y_bf16);
  p.R = R; p.K = K; p.Kin = Kin; p.H = H; p.ldy = ldy;
  const dim3 grid((H + PS_WARPS - 1) / PS_WARPS, (R + PS_NB - 1) / PS_NB);
  rnnt_pred_step_kernel<<<grid, 32 * PS_WARPS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
