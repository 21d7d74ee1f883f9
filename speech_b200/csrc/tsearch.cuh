// The rounds of the transducer beam search, shared by the static-lattice search (tdecode.cu, one
// launch per batch) and the label-free search (rnnt_search.cu, one launch per round): the blank
// emissions into `done`, the two ways of selecting the K best label extensions, and the selection
// of the next beam.  Where a row of log-probabilities comes from is the caller's: each function
// takes it as a functor of the frontier entry.  The definition, the tie order and the exactness
// argument of the shortlist route are in tdecode.cu's header comment, for float32 rows.
//
// Rows and lists may also hold float64 values: the LM-fused rows of the label-free search
// (rnnt_search.cu), f_k = (double)lp_k + (alpha * lm(k | h) + beta), blank f = (double)lp_blank.
// The full route computes fs + f_k, the fused candidate score, with no change.  The shortlist
// route's argument carries over with float64 in place of float32: a list holds the kp best classes
// by (f desc, k asc) and beta is the (kp+1)-th f, so a left-out class has f <= beta and, by the
// monotonicity of fs + f, ties with a selection s only if fs + beta == s.  Given that, a left-out
// class with f == beta follows every listed entry of value beta (safe when the selected value is
// beta), and one with f < beta has f <= nextafter(beta, -inf) (the float64 neighbour), so it ties
// only if fs + nextafter(beta, -inf) == s too.  A selection that fails either test is flagged and
// its utterance is searched again from longer lists; an unflagged selection is the full route's.
// Distinct fused values are closer than distinct float32 values can be, so flags are less rare
// than on float32 lists, but they still need |fs| of about 2^52 times the gap of two classes'
// fused values.
//
// A search that cannot be rerun (the streaming search of rnnt_search.cu keeps no past rows) reads
// lists of 64 entries from its first frame instead of kp = K lists plus a rerun, and gives the
// offline search's answer wherever it is not flagged.  An unflagged selection is the full route's
// at any kp, so until its first flag the stream is in the full route's state, as is the offline
// kp = K pass until its first flag.  A flag at kp = 64 implies a flag at kp = K on the same state
// (the kp = K list is the head of the kp = 64 one).  The selected value x sits at a list position
// below K, so x >= beta_K >= beta_64, and fs + (.) is monotone, so fs + beta_64 == s forces
// fs + beta_K == s.  Then either x > beta_K (the kp = K test holds outright), or x == beta_K and
// beta_64 <= nextafter(beta_K, -inf) < beta_K (or beta_64 == beta_K), so fs + nextafter(beta_K,
// -inf) == s as well.  Where the 64-entry list's tie scan picks an entry of equal sum at position
// >= K, the kp = K list lacks it, selects an entry of larger value and so flags by the same
// reasoning.  So a stream flags only where the offline search reruns and then raises, and it
// reports the flag instead of an unproven hypothesis.
//
// Every function is called by all N threads of the block.  Frontier, beam and the "new" arrays are
// the caller's shared memory; `done` and the trie may live anywhere.
#pragma once
#include "beam.cuh"
#include <math.h>

namespace sb {

SB_DEVINL double td_lse(double a, double b) {
  const double m = fmax(a, b);
  return m + log(exp(a - m) + exp(b - m));
}

// nextafterf(x, -inf) for finite x
SB_DEVINL float td_next_down(float x) {
  const int i = __float_as_int(x);
  if (x == 0.f) return -__int_as_float(1);                 // -(smallest subnormal)
  return __int_as_float(x > 0.f ? i - 1 : i + 1);
}

// nextafter(x, -inf) for finite x
SB_DEVINL double td_next_down(double x) {
  const long long i = __double_as_longlong(x);
  if (x == 0.0) return -__longlong_as_double(1ll);         // -(smallest subnormal)
  return __longlong_as_double(x > 0.0 ? i - 1 : i + 1);
}

// The new frontier of one round: scores, trie nodes, lengths, the frontier entry each extends and
// the symbol it adds.
struct TsNew {
  double* s;
  int *n, *l, *p, *k;
};

// Blank emissions of frontier entries 0 .. nf-1 into `done`, in order (merging order matters):
// an entry already there (same trie node) is log-sum-exp'ed.  blank_lp(i, u) is entry i's blank
// log-probability; entries with u >= U are skipped.  dsrc (may be null) records src0 + i for a new
// entry.  *ndone is shared.
template <int N, class BlankLp>
SB_DEVINL void ts_merge_blanks(int nf, const double* fr_s, const int* fr_n, const int* fr_l, int U,
                               BlankLp blank_lp, double* dscore, int* dnode, int* dlen, int* dsrc,
                               int src0, int* ndone, int done_cap) {
  __shared__ int found;
  const int tid = threadIdx.x;
  for (int i = 0; i < nf; ++i) {
    const int u = fr_l[i];
    if (u >= U) continue;                         // (uniform: shared data)
    if (tid == 0) found = -1;
    __syncthreads();
    const int nd = *ndone, me = fr_n[i];
    for (int j = tid; j < nd; j += N)
      if (dnode[j] == me) found = j;              // at most one entry holds this hypothesis
    __syncthreads();
    if (tid == 0) {
      const double bsc = fr_s[i] + (double)blank_lp(i, u);
      if (found >= 0) {
        dscore[found] = td_lse(dscore[found], bsc);
      } else if (nd < done_cap) {
        dscore[nd] = bsc; dnode[nd] = me; dlen[nd] = u;
        if (dsrc) dsrc[nd] = src0 + i;
        *ndone = nd + 1;
      }
    }
    __syncthreads();
  }
}

// The K best extensions (i, k) by (score desc, i*V + k asc) from the full candidate list cand[K*V]
// (shared or global scratch).  can_extend(i): entry i may take a label; label_lp(i, k): its row.
// Returns -1 when no entry has a candidate (the frame's rounds end), else how many were taken;
// ends in a block barrier.
template <int N, class CanExtend, class LabelLp>
SB_DEVINL int ts_expand_full(double* cand, int K, int V, int blank, int nf, const double* fr_s,
                             const int* fr_n, const int* fr_l, CanExtend can_extend,
                             LabelLp label_lp, const BeamTrie& trie, int round_id, TsNew nw) {
  const int tid = threadIdx.x;
  bool any = false;
  for (int c = tid; c < K * V; c += N) {
    const int i = c / V, k = c - i * V;
    double sc = nan("");
    if (i < nf && k != blank && can_extend(i)) {
      sc = fr_s[i] + (double)label_lp(i, k);
      any = true;
    }
    cand[c] = sc;
  }
  const int have = __syncthreads_or(any ? 1 : 0);
  if (!have) return -1;
  int nsel = 0;
  for (int r = 0; r < K; ++r) {
    double sc;
    const int c = beam_take_first<N>(cand, K * V, sc);
    if (c < 0) break;
    if (tid == 0) {
      const int i = c / V, k = c - i * V;
      nw.s[nsel] = sc;
      nw.n[nsel] = trie.find_or_insert<false>(fr_n[i], k, 1 + round_id * K + nsel);
      nw.l[nsel] = fr_l[i] + 1;
      nw.p[nsel] = i;
      nw.k[nsel] = k;
    }
    ++nsel;
  }
  __syncthreads();                                // thread 0 has read fr_* and written nw
  return nsel;
}

// The same selection as a K-way merge of the frontier's shortlists (kp entries of value type R,
// float or double, by (value desc, k asc)), one lane per entry in warp 0.  list(i, &lv, &li,
// &beta) points at entry i's list and its beta.  Unproven selections are added to *nflag
// (shared).  Returns as ts_expand_full.
template <class R, class CanExtend, class List>
SB_DEVINL int ts_expand_shortlist(int K, int V, int kp, int blank, int nf, const double* fr_s,
                                  const int* fr_n, const int* fr_l, CanExtend can_extend, List list,
                                  const BeamTrie& trie, int round_id, TsNew nw, int* nflag) {
  __shared__ int nsel_s;
  const int tid = threadIdx.x;
  bool live = false;
  if (tid < 32) {
    const int i = tid;
    live = i < nf && can_extend(i) && V > 1;
    const double fs = live ? fr_s[i] : 0.0;
    const bool all_tie = live && fs == -INFINITY;
    const int n = min(kp, V - 1);
    const R* lv = nullptr;
    const int* li = nullptr;
    R beta = -INFINITY;
    if (live && !all_tie) list(i, &lv, &li, &beta);
    const unsigned long long inlist = n >= 64 ? ~0ull : (1ull << n) - 1ull;
    unsigned long long used = 0ull;
    int taken = 0, nfl = 0, ns = 0;
    const bool have = __any_sync(0xffffffffu, live);
    for (int r = 0; r < K && have; ++r) {
      bool hv = false;
      double hs = 0.0;
      int hk = -1, hq = -1;
      if (all_tie) {
        if (taken < V - 1) { hv = true; hs = -INFINITY; hk = taken < blank ? taken : taken + 1; }
      } else if (live) {
        const unsigned long long fr = ~used & inlist;
        if (fr) {
          hq = __ffsll((long long)fr) - 1;
          hk = li[hq];
          hs = fs + (double)lv[hq];
          hv = true;
          for (int q = hq + 1; q < n && fs + (double)lv[q] == hs; ++q)
            if (!((used >> q) & 1ull) && li[q] < hk) { hk = li[q]; hq = q; }
        }
      }
      double bs = hs;
      int bi = hv ? i : -1;
      beam_warp_first(bs, bi);
      if (bi < 0) break;
      const int k = __shfl_sync(0xffffffffu, hk, bi);
      if (i == bi) {
        if (all_tie) {
          ++taken;
        } else {
          used |= 1ull << hq;
          const R x = lv[hq];
          if (fs + (double)beta == hs &&
              (x != beta || (beta != -INFINITY && fs + (double)td_next_down(beta) == hs)))
            ++nfl;
        }
      }
      if (i == 0) {
        nw.s[ns] = bs;
        nw.n[ns] = trie.find_or_insert<false>(fr_n[bi], k, 1 + round_id * K + ns);
        nw.l[ns] = fr_l[bi] + 1;
        nw.p[ns] = bi;
        nw.k[ns] = k;
      }
      ++ns;
      __syncwarp();
    }
    nfl = __reduce_add_sync(0xffffffffu, nfl);
    if (i == 0) { nsel_s = ns; *nflag += nfl; }
  }
  if (!__syncthreads_or(live ? 1 : 0)) return -1;
  return nsel_s;
}

// The next beam: the K best of done[0, nd) by (score desc, insertion order asc), written to
// beam_*[0, n) by thread 0 (bsrc may be null); returns n.  Consumes dscore (taken entries become
// NaN).  No barrier at the end: callers sync before reading beam_*.
template <int N>
SB_DEVINL int ts_select_done(double* dscore, const int* dnode, const int* dlen, const int* dsrc,
                             int nd, int K, double* beam_s, int* beam_n, int* beam_l, int* bsrc) {
  int nb = 0;
  for (int r = 0; r < K; ++r) {
    double sc;
    const int j = beam_take_first<N>(dscore, nd, sc);
    if (j < 0) break;
    if (threadIdx.x == 0) {
      beam_s[nb] = sc; beam_n[nb] = dnode[j]; beam_l[nb] = dlen[j];
      if (bsrc) bsrc[nb] = dsrc[j];
    }
    ++nb;
  }
  return nb;
}

}  // namespace sb
