// Teacher-forced scoring of hypotheses by the attention decoder, one decoder step at a time: the
// second pass of two-pass (CTC prefix beam search, then attention rescoring) decoding.
//
// Row r of a step is one hypothesis START, y_1 .. y_L (L = lens[r]) being forced through the
// decoder.  After step u's log-softmax, sb_s2s_score_tokens adds the log-probability of the token
// the hypothesis has next: y_{u+1} while u < L, END at u == L, nothing after.  Gathering once per
// step keeps the working set at one (R, C) row block; storing every step's rows and gathering at
// the end would need R * U * C floats.
//
// Roofline: R reads of one float and R read-modify-writes of one double per step; negligible next
// to the step kernels.
#include "common.cuh"

#include "../../include/speech_b200.h"

namespace sb {

static constexpr int SCORE_THREADS = 128;

__global__ void __launch_bounds__(SCORE_THREADS) s2s_score_tokens_kernel(
    const float* __restrict__ logp, int C, const int* __restrict__ tokens, int ld,
    const int* __restrict__ lens, int u, int end_tok, double* __restrict__ acc, long long R) {
  const long long r = (long long)blockIdx.x * SCORE_THREADS + threadIdx.x;
  if (r >= R) return;
  const int L = lens[r];
  if (u > L) return;               // past END (and every row of an empty beam slot, L = -1)
  const int tok = u < L ? tokens[r * ld + u + 1] : end_tok;
  acc[r] += (double)logp[r * C + tok];
}

}  // namespace sb

using namespace sb;

extern "C" int sb_s2s_score_tokens(const float* logp, long long R, int C, const int* tokens,
                                   int ld, const int* lens, int u, int end_tok, double* acc,
                                   void* stream) {
  if (!logp || !tokens || !lens || !acc) return SB_ERR_INVALID;
  if (R <= 0 || C <= 0 || ld <= 0 || u < 0 || end_tok < 0 || end_tok >= C) return SB_ERR_INVALID;
  const long long blocks = (R + SCORE_THREADS - 1) / SCORE_THREADS;
  if (blocks > 0x7fffffffLL) return SB_ERR_UNSUPPORTED;
  s2s_score_tokens_kernel<<<(unsigned)blocks, SCORE_THREADS, 0,
                            reinterpret_cast<cudaStream_t>(stream)>>>(logp, C, tokens, ld, lens, u,
                                                                      end_tok, acc, R);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
