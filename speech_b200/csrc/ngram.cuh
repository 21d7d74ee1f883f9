// Device lookup of the backoff n-gram LM (SbNgramLm, include/speech_b200.h), shared by the searches
// that fuse it: the CTC prefix beam search (decode.cu, with a token or a word LM) and the attention
// beam search (s2s.cu).
// A search resolves each hypothesis' context once (lm_context: at most order - 1 probes), then
// scores any number of next tokens against it (lm_backoff: at most order probes each).
#pragma once
#include "common.cuh"
#include <math.h>

#include "../../include/speech_b200.h"

namespace sb {

// value of key (node, tok, kind) in an open-addressed map of include/speech_b200.h's layout, -1
// where it is not stored; Map has its keys, vals and cap: SbNgramLm, or a word LM's lexicon (LexMap)
template <class Map>
__device__ __forceinline__ int map_find(const Map& lm, int node, int tok, int kind) {
  const unsigned long long key = ((unsigned long long)(unsigned int)node << 32) |
                                 ((unsigned long long)(unsigned int)(tok + 1) << 1) |
                                 (unsigned long long)kind;
  unsigned int h = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 32) & (lm.cap - 1);
  for (int probe = 0; probe < lm.cap; ++probe) {
    const unsigned long long k = __ldg(lm.keys + h);
    if (k == key) return __ldg(lm.vals + h);
    if (k == 0ull) return -1;
    h = (h + 1) & (lm.cap - 1);
  }
  return -1;
}

__device__ __forceinline__ int lm_find(const SbNgramLm& lm, int node, int tok, int kind) {
  return map_find(lm, node, tok, kind);
}

// the lexicon map of an SbWordLm: (node, class) -> child node
struct LexMap {
  const unsigned long long* keys;
  const int* vals;
  int cap;
};

// lm(t | context), t an LM token, ctx[0] = root .. ctx[depth] the context's nodes (lm_context):
// the longest stored context first, adding the backoff of each that misses
__device__ __forceinline__ double lm_backoff(const SbNgramLm& lm, const int* ctx, int depth, int t) {
  double acc = 0.0;
  for (int d = depth; d >= 0; --d) {
    const int c = ctx[d];
    const int g = lm_find(lm, c, t, 1);
    if (g >= 0) return acc + __ldg(lm.logp + g);
    acc += __ldg(lm.bow + c);
  }
  return acc;   // not reached: every class scored maps to a token with a unigram
}

// The context nodes of a history read most recent first: older(k) gives the k-th most recent
// class of it (k = 0, 1, .. in turn, at most order - 1 of them), or -1 for <s>, before which there
// is nothing.  Writes ctx[0] = root .. ctx[depth], the walk stopping where the trie has no longer
// context; returns depth.
template <class Older>
__device__ __forceinline__ int lm_context(const SbNgramLm& lm, Older&& older, int* ctx) {
  int c = 0, d = 0;
  ctx[0] = 0;
  for (int k = 0; k < lm.order - 1; ++k) {
    const int h = older(k);
    const int nc = lm_find(lm, c, h < 0 ? lm.bos : __ldg(lm.tok + h), 0);
    if (nc < 0) break;
    c = nc;
    ctx[++d] = c;
    if (h < 0) break;
  }
  return d;
}

// The word-LM terms of SbWordLm (include/speech_b200.h), shared by the CTC prefix beam search
// (decode.cu) and the attention beam search (s2s_beam.cuh).  A history is read by older(k) as
// lm_context reads it, over word tokens; a node is a lexicon node (0 the empty partial word).
struct WordTerms {
  SbWordLm lm;
  double alpha, beta, gamma;

  // the lexicon child of node (>= 0) by class s, -1 where there is none
  __device__ __forceinline__ int child(int node, int s) const {
    return map_find(LexMap{lm.lex_keys, lm.lex_vals, lm.lex_cap}, node, s, 0);
  }
  // the token of the word a delimiter ends at node (!= 0): the node's word or <unk>
  __device__ __forceinline__ int word_tok(int node) const {
    const int w = node > 0 ? __ldg(lm.lex_word + node) : -1;
    return w >= 0 ? w : lm.ngram.bos + 2;
  }
  // the delimiter term of node (!= 0) against a history read by older (lm_context); ctx scratch
  template <class Older>
  __device__ __forceinline__ double dterm(int node, Older&& older, int* ctx) const {
    const int w = node > 0 ? __ldg(lm.lex_word + node) : -1;
    const double g = (node > 0 && w < 0) ? gamma : 0.0;   // an OOV word not charged yet
    const int d = lm_context(lm.ngram, older, ctx);
    return (alpha * lm_backoff(lm.ngram, ctx, d, w >= 0 ? w : lm.ngram.bos + 2) + beta) + g;
  }
  // e + alpha * lm(</s> | ctx') of a hypothesis at node with the history older: e its delimiter
  // term (0 at an empty partial word), ctx' the history with the trailing word
  template <class Older>
  __device__ __forceinline__ double end_term(int node, Older&& older, int* ctx) const {
    const int eos = lm.ngram.bos + 1;
    if (node == 0) {
      const int d = lm_context(lm.ngram, older, ctx);
      return 0.0 + alpha * lm_backoff(lm.ngram, ctx, d, eos);
    }
    const double e = dterm(node, older, ctx);
    const int w = word_tok(node);
    const int d = lm_context(lm.ngram, [&](int k) { return k == 0 ? w : older(k - 1); }, ctx);
    return e + alpha * lm_backoff(lm.ngram, ctx, d, eos);
  }
};

}  // namespace sb

// The checks every word-LM entry point makes (host, before any CUDA call): the tables, the
// weights and the lexicon against C scored classes; layout(*lm) is the search's own check of the
// blank and the delimiter.  Fills t on success.
template <class Layout>
static inline int word_lm_terms(const SbWordLm* lm, double lm_weight, double insertion_bonus,
                                double oov_penalty, int C, Layout&& layout, sb::WordTerms* t) {
  if (!lm) return SB_ERR_INVALID;
  const SbNgramLm& ng = lm->ngram;
  if (!ng.keys || !ng.vals || !ng.logp || !ng.bow || !ng.tok || !lm->lex_keys || !lm->lex_vals ||
      !lm->lex_word)
    return SB_ERR_INVALID;
  if (!(lm_weight >= 0.0) || !isfinite(lm_weight) || !isfinite(insertion_bonus))
    return SB_ERR_INVALID;
  if (isnan(oov_penalty) || oov_penalty > 0.0) return SB_ERR_INVALID;
  if (!lm->has_unk && oov_penalty != -INFINITY) return SB_ERR_INVALID;
  if (lm->num_classes < C || lm->delimiter < 0 || lm->delimiter >= C || !layout(*lm))
    return SB_ERR_INVALID;
  if (ng.cap <= 0 || (ng.cap & (ng.cap - 1)) || lm->lex_cap <= 0 ||
      (lm->lex_cap & (lm->lex_cap - 1)) || lm->num_words < 1 || ng.bos != lm->num_words ||
      ng.order < 1)
    return SB_ERR_INVALID;
  if (ng.order > SB_LM_MAX_ORDER) return SB_ERR_UNSUPPORTED;
  t->lm = *lm;
  t->alpha = lm_weight;
  t->beta = insertion_bonus;
  t->gamma = oov_penalty;
  return SB_OK;
}
