// Device lookup of the backoff n-gram LM (SbNgramLm, include/speech_b200.h), shared by the searches
// that fuse it: the CTC prefix beam search (decode.cu, with a token or a word LM) and the attention
// beam search (s2s.cu).
// A search resolves each hypothesis' context once (lm_context: at most order - 1 probes), then
// scores any number of next tokens against it (lm_backoff: at most order probes each).
#pragma once
#include "common.cuh"

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

}  // namespace sb
