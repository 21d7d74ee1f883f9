// Streaming top-P selection of one warp, shared by the kernels that cut a row of class scores to a
// shortlist: sb_rnnt_shortlist_rows (joint_vocab.cu, float log-probabilities) and the LM-fused
// rows of the label-free transducer search (rnnt_search.cu, float64 fused values).
//
// Order: (value desc, class asc); -inf entries are ranked like any other value.  A warp streams
// its candidates through a buffer of SL_CAP entries: a candidate enters when it ranks above the
// current threshold, and a buffer too full for the next warp's worth is sorted (bitonic) and cut
// to its P best, whose last entry becomes the threshold.  On a random row only O(P log(n / P))
// candidates ever enter.
#pragma once
#include "common.cuh"

namespace sb {

static constexpr int SL_CAP = 256;     // >= SL_MAX_KP + 1 + 32: one cut leaves room for a warp's row
static constexpr int SL_MAX_KP = 64;

template <class T>
SB_DEVINL bool sl_better(T a, int ka, T b, int kb) { return a > b || (a == b && ka < kb); }

// sorts bv / bi [0, SL_CAP) best first (entries past `cnt` are padded with the worst key first)
template <class T>
SB_DEVINL void sl_sort(T* bv, int* bi, int cnt, int lane) {
  for (int i = cnt + lane; i < SL_CAP; i += 32) { bv[i] = -INFINITY; bi[i] = 0x7fffffff; }
  __syncwarp();
  for (int k = 2; k <= SL_CAP; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < SL_CAP; i += 32) {
        const int l = i ^ j;
        if (l > i) {
          const T a = bv[i], c = bv[l];
          const int ka = bi[i], kc = bi[l];
          if ((i & k) == 0 ? sl_better(c, kc, a, ka) : sl_better(a, ka, c, kc)) {
            bv[i] = c; bi[i] = kc; bv[l] = a; bi[l] = ka;
          }
        }
      }
      __syncwarp();
    }
}

// One warp-wide step of the stream: lane's candidate (x, j) enters the buffer where q (the caller
// has already tested it against the threshold, when there is one).  A buffer that cannot take the
// warp's candidates is cut to its P best first, which raises the threshold (thr, tv, tk).
// rnnt_shortlist_rows_kernel spells this step out in its loop: written through this function its
// machine code changes, and that kernel's is kept as it was.
template <class T>
SB_DEVINL void sl_push(T* bv, int* bi, int& cnt, bool& thr, T& tv, int& tk, int P, int lane,
                       bool q, T x, int j) {
  unsigned m = __ballot_sync(0xffffffffu, q);
  if (!m) return;
  if (cnt + __popc(m) > SL_CAP) {        // cut the buffer to its P best, raise the threshold
    sl_sort(bv, bi, cnt, lane);
    cnt = P;
    thr = true;
    tv = bv[P - 1];
    tk = bi[P - 1];
    __syncwarp();
    q = q && sl_better(x, j, tv, tk);
    m = __ballot_sync(0xffffffffu, q);
  }
  if (q) {
    const int pos = cnt + __popc(m & ((1u << lane) - 1u));
    bv[pos] = x;
    bi[pos] = j;
  }
  cnt += __popc(m);
  __syncwarp();
}

}  // namespace sb
