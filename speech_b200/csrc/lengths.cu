// Per-utterance time alignment of time-major activations (row m = t*Bp + b), the one piece of
// data movement the exact-lengths mode needs: with every utterance's frames right-aligned to the
// end of the padded time axis, the reverse direction of the GRU recurrence (which walks t = T-1
// down to 0) meets an utterance's own last frame first and its padding last, so the unchanged
// recurrence kernels leave the real frames exactly as a batch of one would.
//   right-align: row (t, b) -> (t + T - len_b, b);  left-align: the inverse.  Vacated rows are 0.
// One CTA per destination row gathers its source row (or writes zeros); 16-byte accesses when
// rows and pointers allow, else element-wise.  Pure bandwidth: read + write of the column block.
#include "common.cuh"

#include "../../include/speech_b200.h"

namespace sb {

template <typename V>
__global__ void __launch_bounds__(256) time_align_kernel(const V* __restrict__ src, long long ld_src,
                                                         V* __restrict__ dst, long long ld_dst,
                                                         const int* __restrict__ lens, int T,
                                                         int Bp, int units, int sign) {
  const long long m = blockIdx.x;
  const int t = (int)(m / Bp), b = (int)(m % Bp);
  const int len = min(max(__ldg(lens + b), 0), T);
  const int ts = t + sign * (T - len);           // source frame of this destination row
  V* d = dst + m * ld_dst;
  if (ts < 0 || ts >= T) {                      // vacated row
    for (int c = blockIdx.y * blockDim.x + threadIdx.x; c < units; c += gridDim.y * blockDim.x)
      d[c] = V{};
    return;
  }
  const V* s = src + ((long long)ts * Bp + b) * ld_src;
  for (int c = blockIdx.y * blockDim.x + threadIdx.x; c < units; c += gridDim.y * blockDim.x)
    d[c] = s[c];
}

template <typename V>
static int launch_align(const void* src, long long ld_src, void* dst, long long ld_dst,
                        const int* lens, int T, int Bp, int units, int sign, cudaStream_t stream) {
  const int threads = units >= 256 ? 256 : (units + 31) / 32 * 32;
  int gy = (units + threads - 1) / threads;
  if (gy > 64) gy = 64;
  time_align_kernel<V><<<dim3((unsigned)((long long)T * Bp), gy), threads, 0, stream>>>(
      reinterpret_cast<const V*>(src), ld_src, reinterpret_cast<V*>(dst), ld_dst, lens, T, Bp,
      units, sign);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

}  // namespace sb

using namespace sb;

extern "C" int sb_time_align(const void* src, long long ld_src, void* dst, long long ld_dst,
                             const int* lens, int T, int Bp, int cols, int elem_bytes, int right,
                             void* stream_) {
  if (!src || !dst || !lens || src == dst) return SB_ERR_INVALID;
  if (T <= 0 || Bp <= 0 || cols <= 0 || ld_src < cols || ld_dst < cols) return SB_ERR_INVALID;
  if (elem_bytes != 2 && elem_bytes != 4) return SB_ERR_INVALID;
  if ((long long)T * Bp > 0x7fffffffLL) return SB_ERR_UNSUPPORTED;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int sign = right ? -1 : 1;
  const long long rb = (long long)cols * elem_bytes;
  const bool vec = rb % 16 == 0 && (ld_src * elem_bytes) % 16 == 0 &&
                   (ld_dst * elem_bytes) % 16 == 0 &&
                   ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  if (vec)
    return launch_align<uint4>(src, ld_src * elem_bytes / 16, dst, ld_dst * elem_bytes / 16, lens,
                               T, Bp, (int)(rb / 16), sign, stream);
  if (elem_bytes == 4)
    return launch_align<unsigned int>(src, ld_src, dst, ld_dst, lens, T, Bp, cols, sign, stream);
  return launch_align<unsigned short>(src, ld_src, dst, ld_dst, lens, T, Bp, cols, sign, stream);
}
