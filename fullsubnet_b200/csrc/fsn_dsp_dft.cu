// STFT / iSTFT for transform sizes that are not a power of two (the reference's 48 kHz improved_fullsubnet example
// uses n_fft = 960, hop = 480: recipes/dns_interspeech_2020/improved_fullsubnet/model.py:603-620).
//
// Same data flow as fsn_dsp.cu (two real frames packed into one complex transform, FR frames per CTA, fused mask and
// overlap-add), but the transform itself is a direct O(n^2) DFT in shared memory against a full-circle twiddle
// table: at n = 960 that is 3.7 MFLOP per frame, i.e. < 1 % of the model's 217 MFLOP per frame, so a mixed-radix
// FFT would not move the step time.  The power-of-two kernels are untouched.  Per-clip lengths (lens, nullable) follow
// the rules of the radix-2 kernels in fsn_dsp.cu.
#include "fsn_common.cuh"

namespace fsn {

constexpr int kDftFR = 16;  // frames per CTA (same tiling as the radix-2 kernels)
constexpr int kDftThreads = 256;

__device__ __forceinline__ void dft_tables(float2* tw, float* win, int n, int win_length) {
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    float s, c;
    sincospif(-2.0f * (float)k / (float)n, &s, &c);
    tw[k] = make_float2(c, s);  // exp(-2 pi i k / n)
  }
  const int left = (n - win_length) / 2;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int m = i - left;
    const float h = win_length == 1 ? 1.0f : 0.5f - 0.5f * cospif(2.0f * (float)m / (float)win_length);  // hann_window(1) = [1]
    win[i] = (m >= 0 && m < win_length) ? h : 0.0f;
  }
}

// out[p][k] = sum_i in[p][i] * tw[(i*k) mod n]   (INVERSE: conj(tw)); np transforms of length n, natural order
template <bool INVERSE>
__device__ __forceinline__ void dft_smem(const float2* in, float2* out, int np, int n, const float2* tw) {
  for (int idx = threadIdx.x; idx < np * n; idx += blockDim.x) {
    const int p = idx / n;
    const int k = idx - p * n;
    const float2* a = in + (size_t)p * n;
    float re = 0.f, im = 0.f;
    int m = 0;
    for (int i = 0; i < n; ++i) {
      float2 w = tw[m];
      if (INVERSE) w.y = -w.y;
      const float2 v = a[i];
      re = fmaf(v.x, w.x, fmaf(-v.y, w.y, re));
      im = fmaf(v.x, w.y, fmaf(v.y, w.x, im));
      m += k;
      if (m >= n) m -= n;
    }
    out[(size_t)p * n + k] = make_float2(re, im);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kDftThreads)
stft_dft_kernel(const float* __restrict__ wav, int L, int n, int hop, int win_length, int T, float* __restrict__ mag,
                float* __restrict__ phase, float* __restrict__ real, float* __restrict__ imag,
                float* __restrict__ magT, int T_pad, const int* __restrict__ lens) {
  extern __shared__ float2 smem2[];
  constexpr int NP = kDftFR / 2;
  float2* zin = smem2;
  float2* z = zin + NP * n;
  float2* tw = z + NP * n;
  float* win = reinterpret_cast<float*>(tw + n);
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * kDftFR;
  const int F = n / 2 + 1;
  const int Lb = lens ? lens[b] : L;
  const int Tb = lens ? 1 + Lb / hop : T;
  dft_tables(tw, win, n, win_length);
  __syncthreads();
  const float* x = wav + (size_t)b * L;
  for (int idx = threadIdx.x; idx < NP * n; idx += blockDim.x) {
    const int p = idx / n;
    const int i = idx - p * n;
    const int ta = t0 + 2 * p, tb = ta + 1;
    const float w = win[i];
    float va = 0.f, vb = 0.f;
    if (ta < Tb) va = x[reflect_idx(ta * hop + i - n / 2, Lb)] * w;
    if (tb < Tb) vb = x[reflect_idx(tb * hop + i - n / 2, Lb)] * w;
    zin[p * n + i] = make_float2(va, vb);  // frame A -> real lane, frame B -> imaginary lane
  }
  __syncthreads();
  dft_smem<false>(zin, z, NP, n, tw);

  const size_t plane = (size_t)F * T;
  for (int idx = threadIdx.x; idx < F * kDftFR; idx += blockDim.x) {
    const int k = idx / kDftFR;
    const int j = idx - k * kDftFR;
    const int t = t0 + j;
    if (t >= T) continue;
    const float2 zk = z[(j >> 1) * n + k];
    const float2 zn = z[(j >> 1) * n + (k == 0 ? 0 : n - k)];
    float re, im;
    if ((j & 1) == 0) { re = 0.5f * (zk.x + zn.x); im = 0.5f * (zk.y - zn.y); }
    else              { re = 0.5f * (zk.y + zn.y); im = 0.5f * (zn.x - zk.x); }
    if (t >= Tb) re = im = 0.f;
    const size_t o = (size_t)b * plane + (size_t)k * T + t;
    if (real) real[o] = re;
    if (imag) imag[o] = im;
    if (mag) mag[o] = hypotf(re, im);
    if (phase) phase[o] = atan2f(im, re);
  }
  if (magT) {
    for (int idx = threadIdx.x; idx < F * kDftFR; idx += blockDim.x) {
      const int j = idx / F;
      const int k = idx - j * F;
      const int t = t0 + j;
      if (t >= T_pad) continue;
      float m = 0.f;
      if (t < Tb) {
        const float2 zk = z[(j >> 1) * n + k];
        const float2 zn = z[(j >> 1) * n + (k == 0 ? 0 : n - k)];
        float re, im;
        if ((j & 1) == 0) { re = 0.5f * (zk.x + zn.x); im = 0.5f * (zk.y - zn.y); }
        else              { re = 0.5f * (zk.y + zn.y); im = 0.5f * (zn.x - zk.x); }
        m = hypotf(re, im);
      }
      magT[((size_t)b * T_pad + t) * F + k] = m;
    }
  }
}

__global__ void __launch_bounds__(kDftThreads)
istft_dft_kernel(const float* __restrict__ real, const float* __restrict__ imag, int cstride,
                 const float* __restrict__ crm, int mask_mode, int T, int n, int hop, int win_length, int out_len,
                 int seg, int np_max, float* __restrict__ wav, unsigned int* __restrict__ peak_bits,
                 const int* __restrict__ lens) {
  extern __shared__ float2 smem2[];
  float2* zin = smem2;
  float2* z = zin + np_max * n;
  float2* tw = z + np_max * n;
  float* win = reinterpret_cast<float*>(tw + n);
  const int b = blockIdx.y;
  const int F = n / 2 + 1;
  const int Lb = lens ? lens[b] : out_len;
  const int Tb = lens ? 1 + Lb / hop : T;
  const int s_begin = n / 2 + blockIdx.x * seg;
  const int s_end = min(s_begin + seg, n / 2 + Lb);
  const int t_min = (s_begin >= n) ? (s_begin - n) / hop + 1 : 0;
  const int t_max = min(Tb - 1, (s_end - 1) / hop);
  const int nframes = t_max - t_min + 1;
  const int np = nframes > 0 ? (nframes + 1) / 2 : 0;
  dft_tables(tw, win, n, win_length);
  const size_t plane = (size_t)F * T;
  const float* xr = real + (size_t)b * plane * cstride;
  const float* xi = imag + (size_t)b * plane * cstride;
  const float* cr = crm ? crm + (size_t)b * 2 * plane : nullptr;
  const float* ci = crm ? cr + plane : nullptr;
  for (int idx = threadIdx.x; idx < F * np; idx += blockDim.x) {
    const int k = idx / np;
    const int p = idx - k * np;
    float e[2][2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int t = t_min + 2 * p + q;
      float r = 0.f, i = 0.f;
      if (t <= t_max) {
        const size_t o = (size_t)k * T + t;
        r = xr[o * cstride];
        i = xi[o * cstride];
        if (crm && mask_mode == 2) {
          r *= cr[o];
          i *= ci[o];
        } else if (crm) {
          const float mr = decompress_cirm_f(cr[o], 10.0f, 9.9f);
          const float mi = decompress_cirm_f(ci[o], 10.0f, 9.9f);
          const float er = mr * r - mi * i;
          const float ei = mi * r + mr * i;
          r = er; i = ei;
        }
      }
      e[q][0] = r;
      e[q][1] = (k == 0 || k == n / 2) ? 0.f : i;  // irfft ignores Im of DC / Nyquist
    }
    // Z = Ea + i*Eb on the full circle (Hermitian extension of both)
    zin[p * n + k] = make_float2(e[0][0] - e[1][1], e[0][1] + e[1][0]);
    if (k > 0 && k < n / 2) zin[p * n + (n - k)] = make_float2(e[0][0] + e[1][1], -e[0][1] + e[1][0]);
  }
  __syncthreads();
  dft_smem<true>(zin, z, np, n, tw);

  const int full = n + hop * (Tb - 1);
  const float inv_n = 1.0f / (float)n;
  float* out = wav + (size_t)b * out_len;
  float peak = 0.f;
  for (int s = s_begin + threadIdx.x; s < s_end; s += blockDim.x) {
    float acc = 0.f, env = 0.f;
    if (s < full) {
      const int tl = max(t_min, (s >= n) ? (s - n) / hop + 1 : 0);
      const int th = min(t_max, s / hop);
      for (int t = tl; t <= th; ++t) {
        const int i = s - t * hop;
        const int q = t - t_min;
        const float2 v = z[(q >> 1) * n + i];
        const float w = win[i];
        acc += ((q & 1) ? v.y : v.x) * inv_n * w;
        env += w * w;
      }
    }
    const float y = (env > 1e-11f) ? acc / env : 0.f;
    out[s - n / 2] = y;
    peak = fmaxf(peak, fabsf(y));
  }
  if (lens)
    for (int s = max(s_begin, n / 2 + Lb) + threadIdx.x; s < min(s_begin + seg, n / 2 + out_len); s += blockDim.x)
      out[s - n / 2] = 0.f;
  if (peak_bits) {  // per-clip max|y| as in istft_kernel (order-independent, so the atomic is deterministic)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) peak = fmaxf(peak, __shfl_xor_sync(0xffffffffu, peak, o));
    if ((threadIdx.x & 31) == 0 && peak > 0.f) atomicMax(peak_bits + b, __float_as_uint(peak));
  }
}

// adjoint of the element-wise mask + iSTFT with respect to the mask (istft_mask_adjoint_kernel of fsn_dsp.cu on the
// direct DFT): frame t's samples g(t*hop + i) * win[i] -> forward DFT -> c_k/n scaling -> times the kept spectrum
__global__ void __launch_bounds__(kDftThreads)
istft_mask_adjoint_dft_kernel(const float* __restrict__ dwav, const float* __restrict__ real, const float* __restrict__ imag,
                              int L, int n, int hop, int win_length, int T, float* __restrict__ dcrm) {
  extern __shared__ float2 smem2[];
  constexpr int NP = kDftFR / 2;
  float2* zin = smem2;
  float2* z = zin + NP * n;
  float2* tw = z + NP * n;
  float* win = reinterpret_cast<float*>(tw + n);
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * kDftFR;
  const int F = n / 2 + 1;
  dft_tables(tw, win, n, win_length);
  __syncthreads();
  const float* g = dwav + (size_t)b * L;
  for (int idx = threadIdx.x; idx < NP * n; idx += blockDim.x) {
    const int p = idx / n;
    const int i = idx - p * n;
    const int ta = t0 + 2 * p, tb = ta + 1;
    const float w = win[i];
    float va = 0.f, vb = 0.f;
    if (ta < T) va = istft_adjoint_sample(g, win, ta * hop + i, n, hop, T, L) * w;
    if (tb < T) vb = istft_adjoint_sample(g, win, tb * hop + i, n, hop, T, L) * w;
    zin[p * n + i] = make_float2(va, vb);
  }
  __syncthreads();
  dft_smem<false>(zin, z, NP, n, tw);
  const size_t plane = (size_t)F * T;
  for (int idx = threadIdx.x; idx < (F - 1) * kDftFR; idx += blockDim.x) {
    const int k = idx / kDftFR;
    const int j = idx - k * kDftFR;
    const int t = t0 + j;
    if (t >= T) continue;
    const float2 zk = z[(j >> 1) * n + k];
    const float2 zn = z[(j >> 1) * n + (k == 0 ? 0 : n - k)];
    float re, im;
    if ((j & 1) == 0) { re = 0.5f * (zk.x + zn.x); im = 0.5f * (zk.y - zn.y); }
    else              { re = 0.5f * (zk.y + zn.y); im = -0.5f * (zk.x - zn.x); }
    const float sc = (k == 0 ? 1.f : 2.f) / (float)n;
    const size_t o = (size_t)b * plane + (size_t)k * T + t;
    dcrm[(size_t)b * plane + o] = sc * re * real[o];
    dcrm[(size_t)b * plane + plane + o] = k == 0 ? 0.f : sc * im * imag[o];
  }
}

int istft_mask_adjoint_dft_launch(const float* dwav, const float* real, const float* imag, int B, int L, int T, int n_fft,
                                  int hop, int win_length, float* dcrm, cudaStream_t st) {
  const size_t smem = (size_t)kDftFR * n_fft * 8 + (size_t)n_fft * 8 + (size_t)n_fft * 4;
  int rc = check_cuda(cudaFuncSetAttribute(istft_mask_adjoint_dft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                      "istft adjoint smem attr");
  if (rc) return rc;
  istft_mask_adjoint_dft_kernel<<<dim3(cdiv(T, kDftFR), B), kDftThreads, smem, st>>>(dwav, real, imag, L, n_fft, hop,
                                                                                      win_length, T, dcrm);
  FSN_CHECK_LAUNCH("istft_mask_adjoint_dft_kernel");
  return FSN_OK;
}

int stft_dft_launch(const float* wav, int B, int L, int n_fft, int hop, int win_length, int T, int Tg, float* mag,
                    float* phase, float* real, float* imag, float* magT, int T_pad, cudaStream_t st, const int* lens) {
  const size_t smem = (size_t)kDftFR * n_fft * 8 + (size_t)n_fft * 8 + (size_t)n_fft * 4;
  int rc = check_cuda(cudaFuncSetAttribute(stft_dft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                      "stft smem attr");
  if (rc) return rc;
  dim3 grid(cdiv(Tg, kDftFR), B);
  stft_dft_kernel<<<grid, kDftThreads, smem, st>>>(wav, L, n_fft, hop, win_length, T, mag, phase, real, imag, magT,
                                                   T_pad, lens);
  FSN_CHECK_LAUNCH("stft_dft_kernel");
  return FSN_OK;
}

static int istft_dft_np_max(int n_fft, int hop) { return (kDftFR + cdiv(n_fft, hop) + 2) / 2; }

size_t istft_dft_smem_bytes(int n_fft, int hop) {
  return (size_t)2 * istft_dft_np_max(n_fft, hop) * n_fft * 8 + (size_t)n_fft * 8 + (size_t)n_fft * 4;
}

int istft_dft_launch(const float* real, const float* imag, int cstride, const float* crm, int mask_mode, int B, int T,
                     int n_fft, int hop, int win_length, int out_len, float* wav, cudaStream_t st, unsigned int* peak_bits,
                     const int* lens) {
  const int seg = kDftFR * hop;
  const int np_max = istft_dft_np_max(n_fft, hop);
  const size_t smem = istft_dft_smem_bytes(n_fft, hop);  // istft_launch refused it above the opt-in limit
  int rc = check_cuda(cudaFuncSetAttribute(istft_dft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                      "istft smem attr");
  if (rc) return rc;
  dim3 grid(cdiv(out_len, seg), B);
  istft_dft_kernel<<<grid, kDftThreads, smem, st>>>(real, imag, cstride, crm, mask_mode, T, n_fft, hop, win_length,
                                                    out_len, seg, np_max, wav, peak_bits, lens);
  FSN_CHECK_LAUNCH("istft_dft_kernel");
  return FSN_OK;
}

}  // namespace fsn
