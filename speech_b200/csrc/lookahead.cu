// Lookahead (row) convolution of Deep Speech 2 (Amodei et al. 2016, section 3.5) over the top
// unidirectional GRU layer:  r[t, d] = sum_{j=0..tau} W[j][d] * h[t + j, d].
// Operands are the recurrence's time-major layout (row t*Bp + b, Hp columns, fp32 y of
// sb_gru_fwd).  Every unit d is independent (a depthwise convolution along t), so each thread
// owns one column: a CTA stages its time tile plus the tau-frame halo of 64 consecutive units in
// shared memory with coalesced row loads, and every output frame then reads its tau + 1 inputs
// from there.  HBM traffic is one read of h per tile plus the halo, and one write of r.
// Arithmetic contract (include/speech_b200.h): an ascending fp32 FMA chain over j, terms with
// t + j >= len_b skipped (not multiplied by zero), r = 0 at t >= len_b, rb = RNE bf16 of r.
#include "common.cuh"

#include "../../include/speech_b200.h"

namespace sb {

constexpr int LA_COLS = 64;        // units per CTA, one thread each
constexpr int LA_FWD_TT = 32;      // output frames per forward CTA
constexpr int LA_BWD_TT = 32;      // frames per backward CTA (its shared memory bounds occupancy)
constexpr int LA_MAX_TAU = 32;

SB_DEVINL int la_len(const int* lens, int b, int T) {
  return lens ? min(max(__ldg(lens + b), 0), T) : T;
}

__global__ void __launch_bounds__(LA_COLS) lookahead_fwd_kernel(
    const float* __restrict__ h, const float* __restrict__ w, const int* __restrict__ lens,
    float* __restrict__ r, __nv_bfloat16* __restrict__ rb, int T, int Bp, int Hp, int tau) {
  extern __shared__ float la_smem[];
  float* ws = la_smem;                                  // [tau + 1][LA_COLS] taps
  float* hs = la_smem + (tau + 1) * LA_COLS;            // [LA_FWD_TT + tau][LA_COLS] inputs
  const int c = threadIdx.x;
  const int d = blockIdx.x * LA_COLS + c;
  const int b = blockIdx.y;
  const int t0 = blockIdx.z * LA_FWD_TT;
  if (d >= Hp) return;                                  // every thread touches only its column
  const int len = la_len(lens, b, T);
  for (int j = 0; j <= tau; ++j) ws[j * LA_COLS + c] = __ldg(w + (long long)j * Hp + d);
  const int rows = min(LA_FWD_TT + tau, len - t0);      // inputs any output of the tile reads
#pragma unroll 8
  for (int i = 0; i < rows; ++i)
    hs[i * LA_COLS + c] = __ldg(h + ((long long)(t0 + i) * Bp + b) * Hp + d);
  const int tn = min(LA_FWD_TT, T - t0);
  for (int i = 0; i < tn; ++i) {
    const int t = t0 + i;
    float acc = 0.f;
    if (t < len) {
      const int jn = min(tau, len - 1 - t);
      for (int j = 0; j <= jn; ++j) acc = fmaf(ws[j * LA_COLS + c], hs[(i + j) * LA_COLS + c], acc);
    }
    const long long o = ((long long)t * Bp + b) * Hp + d;
    if (r) r[o] = acc;
    if (rb) rb[o] = __float2bfloat16_rn(acc);
  }
}

// dh[t] = sum_j W[j] dr[t - j] (t - j >= 0, t < len_b; else 0), and this tile's share of
// dW[j] = sum_t dr[t] h[t + j] (t + j < len_b) into its own workspace partial.
__global__ void __launch_bounds__(LA_COLS) lookahead_bwd_kernel(
    const float* __restrict__ dr, const float* __restrict__ h, const float* __restrict__ w,
    const int* __restrict__ lens, float* __restrict__ dh, float* __restrict__ part, int T, int Bp,
    int Hp, int tau) {
  extern __shared__ float la_smem[];
  float* ws = la_smem;                                  // [tau + 1][LA_COLS]
  float* ds = ws + (tau + 1) * LA_COLS;                 // [tau + LA_BWD_TT]: dr of t0 - tau ..
  float* hs = ds + (tau + LA_BWD_TT) * LA_COLS;         // [LA_BWD_TT + tau]: h of t0 ..
  const int c = threadIdx.x;
  const int d = blockIdx.x * LA_COLS + c;
  const int b = blockIdx.y;
  const int t0 = blockIdx.z * LA_BWD_TT;
  if (d >= Hp) return;
  const int len = la_len(lens, b, T);
  for (int j = 0; j <= tau; ++j) ws[j * LA_COLS + c] = __ldg(w + (long long)j * Hp + d);
  // dr of frames [max(0, t0 - tau), min(t0 + TT, len)) at ds row t - t0 + tau
#pragma unroll 8
  for (int t = max(0, t0 - tau); t < min(t0 + LA_BWD_TT, len); ++t)
    ds[(t - t0 + tau) * LA_COLS + c] = __ldg(dr + ((long long)t * Bp + b) * Hp + d);
#pragma unroll 8
  for (int t = t0; t < min(t0 + LA_BWD_TT + tau, len); ++t)
    hs[(t - t0) * LA_COLS + c] = __ldg(h + ((long long)t * Bp + b) * Hp + d);
  const int tn = min(LA_BWD_TT, T - t0);
  for (int i = 0; i < tn; ++i) {
    const int t = t0 + i;
    float acc = 0.f;
    if (t < len) {
      const int jn = min(tau, t);
      for (int j = 0; j <= jn; ++j)
        acc = fmaf(ws[j * LA_COLS + c], ds[(i - j + tau) * LA_COLS + c], acc);
    }
    dh[((long long)t * Bp + b) * Hp + d] = acc;
  }
  float* p = part + ((long long)blockIdx.z * Bp + b) * (tau + 1) * Hp + d;
  for (int j = 0; j <= tau; ++j) {
    float acc = 0.f;
    const int n = min(tn, len - j - t0);                // frames t of the tile with t + j < len
    for (int i = 0; i < n; ++i) acc = fmaf(ds[(i + tau) * LA_COLS + c], hs[(i + j) * LA_COLS + c], acc);
    p[(long long)j * Hp] = acc;
  }
}

// dW[j][d] = the sum of the partials (tile-major, then batch row) in a reduction of fixed shape:
// group g of LA_RED_GROUPS adds partials g, g + LA_RED_GROUPS, ... in ascending order, then the
// group sums are added in ascending g.  The order never depends on scheduling, and the groups
// keep many independent loads in flight per column.
constexpr int LA_RED_COLS = 32;
constexpr int LA_RED_GROUPS = 16;

__global__ void __launch_bounds__(LA_RED_COLS * LA_RED_GROUPS) lookahead_dw_reduce_kernel(
    const float* __restrict__ part, float* __restrict__ dw, long long n, int parts) {
  __shared__ float acc[LA_RED_GROUPS][LA_RED_COLS];
  const int c = threadIdx.x % LA_RED_COLS, g = threadIdx.x / LA_RED_COLS;
  const long long i = (long long)blockIdx.x * LA_RED_COLS + c;
  float s = 0.f;
  if (i < n) {
#pragma unroll 4
    for (int p = g; p < parts; p += LA_RED_GROUPS) s += __ldg(part + (long long)p * n + i);
  }
  acc[g][c] = s;
  __syncthreads();
  if (g == 0 && i < n) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < LA_RED_GROUPS; ++k) t += acc[k][c];
    dw[i] = t;
  }
}

static int la_check_shape(int T, int Bp, int Hp, int tau) {
  if (T < 1) return SB_ERR_INVALID;
  if (tau < 1 || tau > LA_MAX_TAU) return SB_ERR_UNSUPPORTED;
  if (Bp < 8 || Bp % 8 != 0 || Bp > 128 || Hp < 8 || Hp % 8 != 0) return SB_ERR_UNSUPPORTED;
  if ((long long)T * Bp * Hp > (1LL << 40)) return SB_ERR_UNSUPPORTED;
  return SB_OK;
}

static long long la_bwd_ws_bytes(int T, int Bp, int Hp, int tau) {
  const long long tiles = (T + LA_BWD_TT - 1) / LA_BWD_TT;
  return tiles * Bp * (tau + 1) * (long long)Hp * (long long)sizeof(float);
}

}  // namespace sb

using namespace sb;

extern "C" int sb_lookahead_fwd(const float* h, const float* w, const int* lens, float* r,
                                void* rb_bf16, int T, int Bp, int Hp, int tau, void* stream_) {
  if (!h || !w || (!r && !rb_bf16)) return SB_ERR_INVALID;
  const int st = la_check_shape(T, Bp, Hp, tau);
  if (st != SB_OK) return st;
  const size_t smem = (size_t)((tau + 1) + (LA_FWD_TT + tau)) * LA_COLS * sizeof(float);
  dim3 grid((Hp + LA_COLS - 1) / LA_COLS, Bp, (T + LA_FWD_TT - 1) / LA_FWD_TT);
  lookahead_fwd_kernel<<<grid, LA_COLS, smem, reinterpret_cast<cudaStream_t>(stream_)>>>(
      h, w, lens, r, reinterpret_cast<__nv_bfloat16*>(rb_bf16), T, Bp, Hp, tau);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}

extern "C" int sb_lookahead_bwd_workspace_size(int T, int Bp, int Hp, int tau, size_t* bytes) {
  if (!bytes) return SB_ERR_INVALID;
  const int st = la_check_shape(T, Bp, Hp, tau);
  if (st != SB_OK) return st;
  *bytes = (size_t)la_bwd_ws_bytes(T, Bp, Hp, tau);
  return SB_OK;
}

extern "C" int sb_lookahead_bwd(const float* dr, const float* h, const float* w, const int* lens,
                                float* dh, float* dw, void* workspace, size_t workspace_bytes,
                                int T, int Bp, int Hp, int tau, void* stream_) {
  if (!dr || !h || !w || !dh || !dw || !workspace) return SB_ERR_INVALID;
  const int st = la_check_shape(T, Bp, Hp, tau);
  if (st != SB_OK) return st;
  if (workspace_bytes < (size_t)la_bwd_ws_bytes(T, Bp, Hp, tau)) return SB_ERR_WORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int tiles = (T + LA_BWD_TT - 1) / LA_BWD_TT;
  const size_t smem =
      (size_t)((tau + 1) + 2 * (LA_BWD_TT + tau)) * LA_COLS * sizeof(float);   // <= 41.2 KB: no opt-in
  float* part = reinterpret_cast<float*>(workspace);
  lookahead_bwd_kernel<<<dim3((Hp + LA_COLS - 1) / LA_COLS, Bp, tiles), LA_COLS, smem, stream>>>(
      dr, h, w, lens, dh, part, T, Bp, Hp, tau);
  if (cudaGetLastError() != cudaSuccess) return SB_ERR_CUDA;
  const long long n = (long long)(tau + 1) * Hp;
  lookahead_dw_reduce_kernel<<<(unsigned)((n + LA_RED_COLS - 1) / LA_RED_COLS),
                               LA_RED_COLS * LA_RED_GROUPS, 0, stream>>>(part, dw, n, tiles * Bp);
  return cudaGetLastError() == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
