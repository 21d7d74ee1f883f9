// Beam state, bookkeeping and n-gram fusion policy of the batched attention beam search, shared by
// the plain and LM-fused selection (s2s.cu) and the joint CTC/attention search (s2s_ctc.cu).
#pragma once
#include "beam.cuh"
#include "ngram.cuh"
#include <math.h>
#include <stddef.h>

#include "../../include/speech_b200.h"

namespace sb {

// ------------------------------------------------------------------------------------------------
// beam search bookkeeping on the device (Seq2Seq.beam_search, seq2seq.py:180-227, run for each of
// B utterances on its own; the K beam entries of utterance b are rows b*K .. b*K+K-1 of the step
// kernels).  Per step, ONE CTA per utterance:
//   candidates (i, c): score_i + logp[i][c] for every live row i (float64, like the reference's
//   Python floats), "sorted" by (score desc, i*C + c asc) = the reference's stable descending sort
//   over its (beam-outer, vocabulary-inner) candidate list (:200-204); the first K of them that
//   end in end_tok join `complete` (:207-209); the first K non-ended ones are the next beam
//   (:211-212, with the py3 list() fix); stop when the beam is empty (:214) or K completed
//   hypotheses beat the best live one (:217-221).
// The "sort" is the selection of beam.cuh, a round per candidate wanted.  Hypotheses are nodes
// (parent node, token) in a plain list: nothing merges prefixes here, so ids need not be canonical,
// and the root is a real token (the start token).  The best complete (else best live) hypothesis
// is back-tracked on the device when the search stops.
// A batch keeps B states and B arenas (nodes, complete scores, final hypothesis) back to back.
// Each utterance's CTA counts itself into stop[0] once, when its search stops; the CTA that makes
// the count B sets stop[1], the no-op flag of the batch's step kernels (B = 1: the same step at
// which the utterance's own `done` is set).  Utterances that stopped keep their rows in the step
// kernels until then; their select and gather CTAs do nothing.
// ------------------------------------------------------------------------------------------------
static constexpr int BM_MAXK = 32;
// done and out_len lead, at the byte offsets the header promises (the host reads them in place);
// final_score is the last 8 bytes
struct BeamState {
  int done;
  int out_len;
  double score[BM_MAXK];     // live beam scores
  int node[BM_MAXK];         // node id of each live entry
  int token[BM_MAXK];        // last token of each live entry (input of the next step)
  int nlive;
  int ncomplete;
  double best_c_score;       // best complete hypothesis (first inserted among equals)
  int best_c_node;
  int have_complete;
  int nodes_used;
  double final_score;        // float64 score of the final hypothesis (written when it stops)
};
static_assert(offsetof(BeamState, done) == 0 && offsetof(BeamState, out_len) == 4 &&
                  offsetof(BeamState, final_score) == sizeof(BeamState) - 8,
              "sb_s2s_beam_state_size: done / out_len / final_score offsets");

// Pointers are those of utterance 0; of(b) gives utterance b's.
struct BeamParams {
  const float* logp;         // [B][K][C] log-softmax of this step's logits
  BeamState* st;             // [B]
  double* c_scores;          // [B][c_cap] scores of complete hypotheses (for the stop rule)
  int* nodes;                // [B][node_cap][2] parent, token
  int* parent_row;           // [B][K] out: row of the previous beam each new entry continues
  int* tok_next;             // [B][K] out: token fed to the next step
  int* out_tokens;           // [B][max_len + 2] final hypothesis (written when the search stops)
  int* stop;                 // [2] stopped utterances, batch done flag (or null)
  int K, C, end_tok, step, max_len, node_cap, c_cap, B;

  SB_DEVINL BeamParams of(int b) const {
    BeamParams q = *this;
    q.logp += (size_t)b * K * C;
    q.st += b;
    q.c_scores += (size_t)b * c_cap;
    q.nodes += (size_t)b * 2 * node_cap;
    q.parent_row += (size_t)b * K;
    q.tok_next += (size_t)b * K;
    q.out_tokens += (size_t)b * (max_len + 2);
    return q;
  }
};

struct S2sLmShared {
  int ctx[BM_MAXK][SB_LM_MAX_ORDER];   // context nodes of each live row, [0] = root .. [depth]
  int depth[BM_MAXK];
};
SB_DEVINL S2sLmShared& s2s_lm_shared() {
  __shared__ S2sLmShared sh;
  return sh;
}

struct S2sLmFuse {
  static constexpr bool kLm = true;
  SbNgramLm lm;
  double alpha, beta;

  // thread r < nl: row r's context nodes; the caller syncs
  SB_DEVINL void resolve(const BeamParams& p, const BeamState* st, int nl) const {
    const int r = threadIdx.x;
    if (r >= nl) return;
    S2sLmShared& sh = s2s_lm_shared();
    int q = st->node[r];
    // the k-th most recent token of row r's hypothesis, -1 (<s>) at the root
    auto older = [&](int) {
      const int up = p.nodes[2 * q];
      if (up < 0) return -1;
      const int t = p.nodes[2 * q + 1];
      q = up;
      return t;
    };
    sh.depth[r] = lm_context(lm, older, sh.ctx[r]);
  }
  SB_DEVINL double value(const BeamParams& p, const BeamState* st, int r, int c) const {
    const S2sLmShared& sh = s2s_lm_shared();
    const double l = lm_backoff(lm, sh.ctx[r], sh.depth[r], __ldg(lm.tok + c));
    return st->score[r] +
           ((double)p.logp[(size_t)r * p.C + c] + (alpha * l + (c == p.end_tok ? 0.0 : beta)));
  }
  // the LM part alone, alpha * lm(c | h_r) + beta_c (the joint CTC/attention search's pre-beam)
  SB_DEVINL double lm_part(const BeamParams& p, int r, int c) const {
    const S2sLmShared& sh = s2s_lm_shared();
    const double l = lm_backoff(lm, sh.ctx[r], sh.depth[r], __ldg(lm.tok + c));
    return alpha * l + (c == p.end_tok ? 0.0 : beta);
  }
};

// The word LM (SbWordLm).  Each hypothesis node q carries its word state in the arena
// word_nodes [B][node_cap][3]: the lexicon node of its partial word, the token of its last
// completed word (-1: none, <s>), and a node whose state holds the words before that one.  The
// state of a live row's node follows from its parent's, which was a live row resolved in the
// previous step's launch, and its token: one lexicon probe or one word token at most; the root
// (the start token) is the empty state.  Its history is then read up those links, at most order - 1
// of them, so a row's resolve costs O(order) probes whatever the length of its words.  Several CTAs
// resolving the same rows write the same values, and no row reads another's node of this step.
struct S2sWordShared {
  int hist[BM_MAXK][SB_LM_MAX_ORDER - 1];   // each live row's last order-1 words, most recent first
  int ctx[BM_MAXK][SB_LM_MAX_ORDER];        // lm_context scratch
  int node[BM_MAXK];                        // each live row's lexicon node n_r
  double dterm[BM_MAXK];                    // d_r (rows with n_r != 0)
  double eterm[BM_MAXK];                    // t_r
};
SB_DEVINL S2sWordShared& s2s_word_shared() {
  __shared__ S2sWordShared sh;
  return sh;
}

struct S2sWordLmFuse {
  static constexpr bool kLm = true;
  WordTerms wt;
  int* word_nodes;          // [B][node_cap][3], parallel to BeamParams::nodes
  const int* nodes0;        // utterance 0's nodes: p.nodes - nodes0 locates utterance b's arena

  // thread r < nl: row r's word state (written to its node), history, d_r and t_r; the caller
  // syncs
  SB_DEVINL void resolve(const BeamParams& p, const BeamState* st, int nl) const {
    const int r = threadIdx.x;
    if (r >= nl) return;
    S2sWordShared& sh = s2s_word_shared();
    int* wn = word_nodes + (size_t)(p.nodes - nodes0) / 2 * 3;
    const int q = st->node[r], u = p.nodes[2 * q], t = p.nodes[2 * q + 1];
    int lex = 0, last = -1, before = -1;
    if (u >= 0) {
      const int nu = wn[3 * u];
      last = wn[3 * u + 1];
      before = wn[3 * u + 2];
      if (t == wt.lm.delimiter) {
        if (nu != 0) { last = wt.word_tok(nu); before = u; }
      } else {
        lex = nu < 0 ? -1 : wt.child(nu, t);
      }
    }
    wn[3 * q] = lex;
    wn[3 * q + 1] = last;
    wn[3 * q + 2] = before;
    const int n = wt.lm.ngram.order - 1;
    for (int k = 0; k < n; ++k) {
      sh.hist[r][k] = last;
      if (last < 0) break;
      last = wn[3 * before + 1];
      before = wn[3 * before + 2];
    }
    auto older = [&](int k) { return sh.hist[r][k]; };
    sh.node[r] = lex;
    if (lex != 0) sh.dterm[r] = wt.dterm(lex, older, sh.ctx[r]);
    sh.eterm[r] = wt.end_term(lex, older, sh.ctx[r]);
  }
  SB_DEVINL double value(const BeamParams& p, const BeamState* st, int r, int c) const {
    const S2sWordShared& sh = s2s_word_shared();
    const double lp = (double)p.logp[(size_t)r * p.C + c];
    const int n = sh.node[r];
    if (c == wt.lm.delimiter) return n == 0 ? st->score[r] + lp : st->score[r] + (lp + sh.dterm[r]);
    if (c == p.end_tok) return st->score[r] + (lp + sh.eterm[r]);
    if (n >= 0 && wt.child(n, c) < 0) return st->score[r] + (lp + wt.gamma);
    return st->score[r] + lp;
  }
  // the LM part alone: d_r, t_r, gamma or 0 (the joint CTC/attention search's pre-beam)
  SB_DEVINL double lm_part(const BeamParams& p, int r, int c) const {
    const S2sWordShared& sh = s2s_word_shared();
    const int n = sh.node[r];
    if (c == wt.lm.delimiter) return n == 0 ? 0.0 : sh.dterm[r];
    if (c == p.end_tok) return sh.eterm[r];
    return (n >= 0 && wt.child(n, c) < 0) ? wt.gamma : 0.0;
  }
};

// ---- the reference's bookkeeping of one utterance (p = BeamParams::of(b)), sequential (a handful
// of entries): the first `want` candidates in (score desc, index asc) order -> complete / next
// beam / stop rule / back-track; parent_row holds rows within the utterance.  A selected flat
// index i is candidate (r, c): r = i / per_row, c = cls[i] from a per-row candidate list, or
// c = i - r * per_row over the whole vocabulary (cls null, per_row = C).  live_src (or null) gets
// the flat index each new live entry came from ----
SB_DEVINL void beam_bookkeep(const BeamParams& p, const int* sel_idx, const double* sel_sc,
                             int want, int per_row, const int* cls = nullptr,
                             int* live_src = nullptr) {
  BeamState* st = p.st;
  const int K = p.K, C = per_row, nl = st->nlive;
  int old_node[BM_MAXK];
  for (int r = 0; r < nl; ++r) old_node[r] = st->node[r];
  int nb = 0;
  for (int q = 0; q < want; ++q) {
    const int i = sel_idx[q];
    if (i < 0) break;
    const int r = i / C, c = cls ? cls[i] : i - r * C;
    const bool ended = (c == p.end_tok);
    if (ended && q >= K) continue;                 // only the first K candidates may complete
    if (!ended && nb >= K) continue;
    int id = st->nodes_used;
    if (id >= p.node_cap) { st->done = p.step + 1; break; }
    st->nodes_used = id + 1;
    p.nodes[2 * id] = old_node[r];
    p.nodes[2 * id + 1] = c;
    if (ended) {
      if (st->ncomplete < p.c_cap) p.c_scores[st->ncomplete] = sel_sc[q];
      st->ncomplete += 1;
      if (!st->have_complete || sel_sc[q] > st->best_c_score) {
        st->have_complete = 1;
        st->best_c_score = sel_sc[q];
        st->best_c_node = id;
      }
    } else {
      st->score[nb] = sel_sc[q];
      st->node[nb] = id;
      st->token[nb] = c;
      p.parent_row[nb] = r;
      p.tok_next[nb] = c;
      if (live_src) live_src[nb] = i;
      ++nb;
    }
  }
  st->nlive = nb;
  bool stop = (nb == 0) || (p.step + 1 >= p.max_len);
  if (!stop) {
    int better = 0;
    const int nc = min(st->ncomplete, p.c_cap);
    for (int j = 0; j < nc; ++j) better += (p.c_scores[j] > st->score[0]) ? 1 : 0;
    stop = better >= K;
  }
  if (stop) {
    st->done = p.step + 1;                         // nonzero: the steps the search ran
    // best complete hypothesis, else the best live one (seq2seq.py:223-227)
    int n = st->have_complete ? st->best_c_node : (nb > 0 ? st->node[0] : -1);
    int len = 0;
    for (int q = n; q >= 0; q = p.nodes[2 * q]) ++len;
    int k = len;
    for (int q = n; q >= 0; q = p.nodes[2 * q]) p.out_tokens[--k] = p.nodes[2 * q + 1];
    st->out_len = len;
    st->final_score = st->have_complete ? st->best_c_score : (nb > 0 ? st->score[0] : -INFINITY);
  }
  // stopped in this call (here or at the node cap): count it; the last of the batch sets the flag
  if (st->done && p.stop && atomicAdd(p.stop, 1) == p.B - 1) p.stop[1] = 1;
}

}  // namespace sb

// The fusion policy of an LM entry point, after the checks the header lists (host)
static inline int beam_lm_fuse(const SbNgramLm* lm, double lm_weight, double insertion_bonus,
                               int C, sb::S2sLmFuse* fu) {
  if (!lm || !lm->keys || !lm->vals || !lm->logp || !lm->bow || !lm->tok) return SB_ERR_INVALID;
  if (!(lm_weight >= 0.0) || !isfinite(lm_weight) || !isfinite(insertion_bonus))
    return SB_ERR_INVALID;
  if (!isfinite(lm->lm_upper) || !isfinite(lm->lm_abs) || lm->num_classes < C) return SB_ERR_INVALID;
  if (lm->blank >= 0 && lm->blank < C) return SB_ERR_INVALID;   // a scored class with no LM token
  if (lm->cap <= 0 || (lm->cap & (lm->cap - 1)) || lm->order < 1) return SB_ERR_INVALID;
  if (lm->order > SB_LM_MAX_ORDER) return SB_ERR_UNSUPPORTED;
  fu->lm = *lm;
  fu->alpha = lm_weight;
  fu->beta = insertion_bonus;
  return SB_OK;
}

// The fusion policy of a word-LM entry point, after the checks the header lists (host): the blank
// (the start token) is no scored class and the delimiter is not the end token
static inline int beam_wordlm_fuse(const SbWordLm* lm, double lm_weight, double insertion_bonus,
                                   double oov_penalty, int C, int end_tok, int* word_nodes,
                                   const int* nodes, sb::S2sWordLmFuse* fu) {
  if (!word_nodes) return SB_ERR_INVALID;
  fu->word_nodes = word_nodes;
  fu->nodes0 = nodes;
  return word_lm_terms(lm, lm_weight, insertion_bonus, oov_penalty, C,
                       [&](const SbWordLm& l) {
                         return !(l.blank >= 0 && l.blank < C) && l.delimiter != end_tok;
                       },
                       &fu->wt);
}
