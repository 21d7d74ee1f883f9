// Building blocks shared by the beam-search decoders (decode.cu, tdecode.cu, s2s.cu): the order in
// which candidates are taken, the block-wide selection of the first candidate, and the trie that
// holds the hypotheses.
//
// Order.  Every search here prunes by "the k best of a candidate list, ties in list order": the
// reference implementations sort with a stable descending sort.  A candidate is (score, key) with
// an integer key >= 0 that numbers the list (a flat index, or a first-touch rank); key < 0 means
// "no candidate".  (s1, k1) comes before (s2, k2) iff s1 > s2, or s1 == s2 and k1 < k2; any
// candidate comes before none.  A top-k is k rounds of "first of the block".
//
// Shape of the selection, kept fixed so that equal (score, key) pairs (keys that are ranks need
// not be unique) resolve the same way everywhere: thread tid scans tid, tid + N, ... in ascending
// order and keeps the first of equals; lanes combine by an xor butterfly 16..1; warps combine in
// ascending warp order.
#pragma once
#include "common.cuh"

namespace sb {

// among two candidates
template <typename S>
SB_DEVINL bool beam_order(S s1, int k1, S s2, int k2) {
  return s1 > s2 || (s1 == s2 && k1 < k2);
}
// when either may be none
template <typename S>
SB_DEVINL bool beam_before(S s1, int k1, S s2, int k2) {
  return k1 >= 0 && (k2 < 0 || beam_order(s1, k1, s2, k2));
}

template <bool PAYLOAD, typename S>
SB_DEVINL void beam_warp_first_impl(S& s, int& k, int& p) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const S os = __shfl_xor_sync(0xffffffffu, s, o);
    const int ok = __shfl_xor_sync(0xffffffffu, k, o);
    const int op = PAYLOAD ? __shfl_xor_sync(0xffffffffu, p, o) : 0;
    if (beam_before(os, ok, s, k)) { s = os; k = ok; p = op; }
  }
}

// first of the warp's candidates (s, k); every lane gets it
template <typename S>
SB_DEVINL void beam_warp_first(S& s, int& k) {
  int p = 0;
  beam_warp_first_impl<false>(s, k, p);
}

template <int N, bool PAYLOAD, typename S>
SB_DEVINL void beam_block_first_impl(S& s, int& k, int& p) {
  static_assert(N % 32 == 0, "whole warps");
  __shared__ S slot_s[N / 32];
  __shared__ int slot_k[N / 32];
  __shared__ int slot_p[N / 32];
  const int tid = threadIdx.x;
  beam_warp_first_impl<PAYLOAD>(s, k, p);
  __syncthreads();                                   // the previous call's slots have been read
  if ((tid & 31) == 0) {
    slot_s[tid >> 5] = s;
    slot_k[tid >> 5] = k;
    if (PAYLOAD) slot_p[tid >> 5] = p;
  }
  __syncthreads();
  s = slot_s[0];
  k = slot_k[0];
  if (PAYLOAD) p = slot_p[0];
  for (int w = 1; w < N / 32; ++w)
    if (beam_before(slot_s[w], slot_k[w], s, k)) {
      s = slot_s[w];
      k = slot_k[w];
      if (PAYLOAD) p = slot_p[w];
    }
}

// First of the candidates (s, k) of the N threads of the block, with an optional payload p (what
// the key stands for, when the key is a rank); every thread gets it.  Called by all N threads.
// The barriers its scratch needs are inside: callers may call it back to back, and what a thread
// wrote to shared memory before the call is visible to the block after it.
template <int N, typename S>
SB_DEVINL void beam_block_first(S& s, int& k) {
  int p = 0;
  beam_block_first_impl<N, false>(s, k, p);
}
template <int N, typename S>
SB_DEVINL void beam_block_first(S& s, int& k, int& p) {
  beam_block_first_impl<N, true>(s, k, p);
}

// One step of a thread's ascending scan over scores in which NaN marks "already taken": keys
// ascend, so the strict > keeps the first of equals.
SB_DEVINL void beam_scan_step(double v, int i, double& bs, int& bi) {
  if (!isnan(v) && (bi < 0 || v > bs)) { bs = v; bi = i; }
}

// One round of a top-k over sc[0, n), NaN = taken: takes the first live entry by (score desc,
// index asc), marks it taken and returns its index (-1: none left) and score to every thread.
// Between the caller's barrier after filling sc and the last round, entry i is read and written
// by thread i % N only, so the mark needs no barrier of its own.
template <int N>
SB_DEVINL int beam_take_first(double* sc, int n, double& score) {
  static_assert((N & (N - 1)) == 0, "power of two");
  const int tid = threadIdx.x;
  double bs = 0.0;
  int bi = -1;
  for (int i = tid; i < n; i += N) beam_scan_step(sc[i], i, bs, bi);
  beam_block_first<N>(bs, bi);
  if (bi >= 0 && (bi & (N - 1)) == tid) sc[bi] = nan("");
  score = bs;
  return bi;
}

// ------------------------------------------------------------------------------------------------
// The hypotheses of one utterance: nodes (parent, symbol) of a trie in an arena, node 0 = the
// empty sequence, so that "the same label sequence" is an integer comparison.
// Node ids must be CANONICAL over the whole utterance: a prefix that is pruned and later
// re-created has to get its old id back, because surviving descendants still name it as parent.
// So every node ever made stays in an open-addressed (parent, symbol) -> id map.
// ------------------------------------------------------------------------------------------------
struct BeamTrie {
  int* nodes;                  // [node_cap][2] parent, symbol
  unsigned long long* keys;    // [cap] (parent << 32 | symbol + 1), 0 = empty
  int* vals;                   // [cap] node id
  int cap;                     // power of two (beam_pow2_cap), >= 2 * node_cap
  int node_cap;

  // the trie of utterance b, when this one describes utterance 0 of a batch stored back to back
  SB_DEVINL BeamTrie of(int b) const {
    BeamTrie t = *this;
    t.nodes += (size_t)b * 2 * node_cap;
    t.keys += (size_t)b * cap;
    t.vals += (size_t)b * cap;
    return t;
  }

  // empty trie: the root alone.  All N threads of the block; ends in a block barrier.
  template <int N>
  SB_DEVINL void clear() const {
    for (int k = threadIdx.x; k < cap; k += N) keys[k] = 0ull;
    if (threadIdx.x == 0) { nodes[0] = -1; nodes[1] = -1; }
    __syncthreads();
  }

  // The node of `parent` extended by `symbol`; when there is none yet it becomes node new_id
  // (-1 when new_id is past the arena).  SHARED: other threads insert at the same time (their
  // (parent, symbol) and new_id differ), so a slot is claimed by compare-and-swap; a lone inserter
  // stores, and does not wait for the atomic's round trip.
  template <bool SHARED>
  SB_DEVINL int find_or_insert(int parent, int symbol, int new_id) const {
    const unsigned long long key =
        ((unsigned long long)(unsigned int)parent << 32) | (unsigned int)(symbol + 1);
    unsigned int h = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 32) & (cap - 1);
    for (int probe = 0; probe < cap; ++probe) {
      const unsigned long long k = keys[h];
      if (k == key) return vals[h];
      if (k == 0ull) {
        if (new_id >= node_cap) return -1;
        const unsigned long long old = SHARED ? atomicCAS(&keys[h], 0ull, key) : 0ull;
        if (old == 0ull) {
          if (!SHARED) keys[h] = key;
          vals[h] = new_id;
          nodes[2 * new_id] = parent;
          nodes[2 * new_id + 1] = symbol;
          return new_id;
        }
        if (old == key) return vals[h];
      }
      h = (h + 1) & (cap - 1);
    }
    return -1;
  }

  // writes the symbols on the path root -> node to out[0 .. length), returns the length
  SB_DEVINL int backtrack(int node, int* out) const {
    int len = 0;
    for (int q = node; q > 0; q = nodes[2 * q]) ++len;
    int k = len;
    for (int q = node; q > 0; q = nodes[2 * q]) out[--k] = nodes[2 * q + 1];
    return len;
  }
};

// capacity of the map for `need` slots (host)
static inline int beam_pow2_cap(size_t need) {
  size_t cap = 64;
  while (cap < need) cap <<= 1;
  return (int)cap;
}

}  // namespace sb
