// Shared helpers for libfsn_b200 (error reporting, launch counting, small device utilities).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/fsn_b200.h"

namespace fsn {

void set_error(const char* fmt, ...);
int& last_error_code();
int64_t& launch_counter();
int64_t& total_launch_counter();

inline int check_cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    last_error_code() = FSN_ERR_CUDA;
    return FSN_ERR_CUDA;
  }
  return FSN_OK;
}

#define FSN_CHECK_LAUNCH(what)                                   \
  do {                                                           \
    ::fsn::launch_counter()++;                                   \
    ::fsn::total_launch_counter()++;                             \
    int _rc = ::fsn::check_cuda(cudaGetLastError(), what);       \
    if (_rc) return _rc;                                         \
  } while (0)

#define FSN_REQUIRE(cond, code, ...)  \
  do {                                \
    if (!(cond)) {                    \
      ::fsn::set_error(__VA_ARGS__);  \
      ::fsn::last_error_code() = code; \
      return code;                    \
    }                                 \
  } while (0)

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// 'reflect' padding index map (no edge repeat): -k -> k, n-1+k -> n-1-k
__device__ __forceinline__ int reflect_idx(int i, int n) {
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}

// c[r] = #{(f,k): reflect(f+k) = r, |k| <= N}: multiplicity of row r in the unfolded tensor
__host__ __device__ __forceinline__ int reflect_count(int r, int F, int N) {
  int c = 0;
  for (int k = -N; k <= N; ++k) {
    int f = r - k;                       // f + k = r
    c += (f >= 0 && f < F);
    if (r > 0) {                         // f + k = -r (left reflection)
      f = -r - k;
      c += (f >= 0 && f < F);
    }
    if (r < F - 1) {                     // f + k = 2(F-1) - r (right reflection)
      f = 2 * (F - 1) - r - k;
      c += (f >= 0 && f < F);
    }
  }
  return c;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// audio_zen/acoustics/mask.py:58-63
__device__ __forceinline__ float decompress_cirm_f(float m, float K, float limit) {
  // limit*(m>=limit) - limit*(m<=-limit) + m*(|m|<limit): NaN falls through to 0 like the reference
  m = (fabsf(m) < limit) ? m : ((m >= limit) ? limit : ((m <= -limit) ? -limit : 0.0f));
  return -K * logf((K - m) / (K + m));
}

// mask.py:38-40
__device__ __forceinline__ float compress_cirm_f(float m, float K, float C) {
  m = (m <= -100.f) ? -100.f : m;
  const float e = expf(-C * m);
  return K * (1.f - e) / (1.f + e);
}

// mask.py:22-29: the compressed cIRM (real, imag) of one bin from the noisy (a + ib) and clean (c + id) spectra
__device__ __forceinline__ float2 cirm_f(float a, float b, float c, float d) {
  const float eps = 1.1920928955078125e-07f;  // audio_zen/constant.py:9
  const float den = a * a + b * b + eps;
  return make_float2(compress_cirm_f((a * c + b * d) / den, 10.f, 0.1f), compress_cirm_f((a * d - b * c) / den, 10.f, 0.1f));
}

// fixed-order tree sum over the 256 threads of a CTA; the total reaches thread 0
template <class V>
__device__ __forceinline__ V cta_tree_sum256(V a, V* sh) {
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}

}  // namespace fsn
