// Training-data mixing on the device (SURVEY 8f rank 4): the arithmetic of Dataset.snr_mix
// (recipes/dns_interspeech_2020/dataset_train.py:136-199) for a whole batch of (clean, noise) pairs -
// optional reverberation (scipy.signal.fftconvolve(clean, rir)[:L], :161), norm_amplitude + tailor_dB_FS of both
// (audio_zen/acoustics/feature.py:99-111), SNR scaling, the common dBFS of the mixture and the anti-clipping rescale.
// The random draws of the reference (SNR, noisy target dBFS, RIR choice) stay on the host and come in as arrays,
// so that the result is a pure function of its inputs.  One CTA per clip, fixed-order reductions.
#include "fsn_internal.cuh"

namespace fsn {
namespace mix {

constexpr int THREADS = 1024;

__device__ __forceinline__ double block_sum(double v, double* sh) {
  __syncthreads();
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}
__device__ __forceinline__ float block_max(float v, double* sh) {
  __syncthreads();
  sh[threadIdx.x] = (double)v;
  __syncthreads();
  for (int s = THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  return (float)sh[0];
}

// out[b, n] = sum_k x[b, n-k] rir[b, k], n < L (the first L samples of the full convolution); clips with
// rir_len[b] == 0 are copied.  Direct form, register-blocked: each thread computes CR consecutive outputs from one
// broadcast tap load and one sample load per tap; the taps and a segment of the clip are staged through shared memory
// as doubles in chunks of CK taps.  Each output is summed k ascending in one double accumulator.  A product of two
// floats is exact in double, so every term and every partial sum is the one of the plain loop
// "for k: acc += (double)rir[k] * (double)x[n-k]"; the zero terms it adds or skips (k >= rir_len, n - k < 0) cannot
// change a sum that starts at +0.  CR is odd so the threads' sample loads (stride CR doubles) hit distinct banks.
constexpr int CT = 128, CR = 9, CO = CT * CR, CK = 128 * CR;
static_assert(CK % CR == 0, "a chunk is a whole number of register rotations");
__global__ void __launch_bounds__(CT) rir_conv_kernel(const float* __restrict__ x, const float* __restrict__ rir,
                                                      const int* __restrict__ rir_len, int L, int Lr_max,
                                                      float* __restrict__ out) {
  __shared__ double taps[CK];
  __shared__ double seg[CK + CO];  // seg[i] = x[n0 - k0 - CK + i]
  const int b = blockIdx.y, n0 = blockIdx.x * CO, t0 = threadIdx.x * CR;
  const float* xb = x + (size_t)b * L;
  float* ob = out + (size_t)b * L;
  const int lr = rir_len ? min(rir_len[b], Lr_max) : Lr_max;
  if (lr <= 0) {
    for (int i = threadIdx.x; i < CO && n0 + i < L; i += CT) ob[n0 + i] = xb[n0 + i];
    return;
  }
  const float* rb = rir + (size_t)b * Lr_max;
  double acc[CR];
#pragma unroll
  for (int r = 0; r < CR; ++r) acc[r] = 0.0;  // double accumulation: the reference's FFT convolution carries ~1e-7
                                              // relative error per output
  for (int k0 = 0; k0 < lr && k0 <= n0 + CO - 1; k0 += CK) {
    const int kn = min(CK, lr - k0);
    __syncthreads();
    for (int i = threadIdx.x; i < CK; i += CT) taps[i] = i < kn ? (double)rb[k0 + i] : 0.0;
    const int base = n0 - k0 - CK;
    for (int i = threadIdx.x; i < CK + CO; i += CT) {
      const int j = base + i;
      seg[i] = (j >= 0 && j < L) ? (double)xb[j] : 0.0;
    }
    __syncthreads();
    // x[n0 + t0 + d - k0] = sp[d]; the window w holds offsets d = r - kk (r < CR) of step kk, offset d in slot d mod CR
    const double* sp = seg + t0 + CK;
    double w[CR];
#pragma unroll
    for (int r = 0; r < CR; ++r) w[r] = sp[r];
    for (int kk = 0; kk < kn; kk += CR) {
#pragma unroll
      for (int j = 0; j < CR; ++j) {
        const double h = taps[kk + j];
#pragma unroll
        for (int r = 0; r < CR; ++r) acc[r] = fma(h, w[(r - j + CR) % CR], acc[r]);
        w[CR - 1 - j] = sp[-(kk + j + 1)];  // offset -(kk+j+1) replaces CR-1-(kk+j), which step kk+j+1 no longer needs
      }
    }
  }
#pragma unroll
  for (int r = 0; r < CR; ++r)
    if (n0 + t0 + r < L) ob[n0 + t0 + r] = (float)acc[r];
}

__global__ void __launch_bounds__(THREADS) snr_mix_kernel(const float* __restrict__ clean, const float* __restrict__ noise,
                                                          const float* __restrict__ snr, const float* __restrict__ noisy_target,
                                                          float target_dB_FS, float eps, int L, float* __restrict__ noisy_out,
                                                          float* __restrict__ clean_out) {
  __shared__ double sh[THREADS];
  const int b = blockIdx.x;
  const float* c = clean + (size_t)b * L;
  const float* n = noise + (size_t)b * L;
  float mc = 0.f, mn = 0.f;
  for (int i = threadIdx.x; i < L; i += THREADS) { mc = fmaxf(mc, fabsf(c[i])); mn = fmaxf(mn, fabsf(n[i])); }
  const float sc1 = block_max(mc, sh) + eps, sn1 = block_max(mn, sh) + eps;  // norm_amplitude: y / (max|y| + eps)
  double a = 0.0, d = 0.0;
  for (int i = threadIdx.x; i < L; i += THREADS) {
    const float u = c[i] / sc1, v = n[i] / sn1;
    a += (double)u * u; d += (double)v * v;
  }
  const float tgt = powf(10.0f, target_dB_FS / 20.0f);
  const float kc = tgt / ((float)sqrt(block_sum(a, sh) / L) + eps);   // tailor_dB_FS scalar of the clean speech
  const float kn = tgt / ((float)sqrt(block_sum(d, sh) / L) + eps);   // ... of the noise
  a = 0.0; d = 0.0;
  for (int i = threadIdx.x; i < L; i += THREADS) {
    const float u = (c[i] / sc1) * kc, v = (n[i] / sn1) * kn;
    a += (double)u * u; d += (double)v * v;
  }
  const float clean_rms = (float)sqrt(block_sum(a, sh) / L), noise_rms = (float)sqrt(block_sum(d, sh) / L);
  const float snr_scalar = clean_rms / powf(10.0f, snr[b] / 20.0f) / (noise_rms + eps);
  a = 0.0;
  for (int i = threadIdx.x; i < L; i += THREADS) {
    const float y = (c[i] / sc1) * kc + ((n[i] / sn1) * kn) * snr_scalar;
    a += (double)y * y;
  }
  const float ky = powf(10.0f, noisy_target[b] / 20.0f) / ((float)sqrt(block_sum(a, sh) / L) + eps);
  float my = 0.f;
  for (int i = threadIdx.x; i < L; i += THREADS) {
    const float y = ((c[i] / sc1) * kc + ((n[i] / sn1) * kn) * snr_scalar) * ky;
    my = fmaxf(my, fabsf(y));
  }
  my = block_max(my, sh);
  const bool clipped = my > 0.999f;                       // is_clipped (feature.py:113-114)
  const float kclip = clipped ? my / (0.99f - eps) : 1.0f;
  for (int i = threadIdx.x; i < L; i += THREADS) {
    const float u = (c[i] / sc1) * kc;
    float y = (u + ((n[i] / sn1) * kn) * snr_scalar) * ky;
    float cl = u * ky;
    if (clipped) { y = y / kclip; cl = cl / kclip; }
    noisy_out[(size_t)b * L + i] = y;
    clean_out[(size_t)b * L + i] = cl;
  }
}

}  // namespace mix
}  // namespace fsn

using namespace fsn;

extern "C" int fsn_rir_convolve(const float* x, const float* rir, const int* rir_len, int B, int L, int Lr_max, float* out,
                                fsn_stream_t stream) {
  FSN_REQUIRE(B > 0 && L > 0 && Lr_max > 0, FSN_ERR_SHAPE, "rir_convolve: empty input");
  mix::rir_conv_kernel<<<dim3(cdiv(L, mix::CO), B), mix::CT, 0, (cudaStream_t)stream>>>(x, rir, rir_len, L, Lr_max, out);
  FSN_CHECK_LAUNCH("rir_conv_kernel");
  return FSN_OK;
}

extern "C" int fsn_snr_mix(const float* clean, const float* noise, const float* snr, const float* noisy_target_dB_FS,
                           float target_dB_FS, float eps, int B, int L, float* noisy_out, float* clean_out,
                           fsn_stream_t stream) {
  FSN_REQUIRE(B > 0 && L > 0, FSN_ERR_SHAPE, "snr_mix: empty input");
  mix::snr_mix_kernel<<<B, mix::THREADS, 0, (cudaStream_t)stream>>>(clean, noise, snr, noisy_target_dB_FS, target_dB_FS, eps, L,
                                                                    noisy_out, clean_out);
  FSN_CHECK_LAUNCH("snr_mix_kernel");
  return FSN_OK;
}
