// STFT / iSTFT (+ fused cIRM decompress & complex mask), the iSTFT's mask adjoint, and the elementwise mask ops.
//
// Reference semantics: audio_zen/acoustics/feature.py:9-91 (-> torch.stft / torch.istft),
// audio_zen/acoustics/mask.py:7-64, recipes/dns_interspeech_2020/inferencer.py:136-143.
//
// Two real frames packed into one complex transform (frame A -> real lane, frame B -> imaginary lane), kFR frames per
// CTA so that the [B,F,T] (T-contiguous) stores / loads of the reference layout are kFR*4-byte segments.  The three
// transform kernels are templates over the transform policy:
//   Radix2     n a power of two: shared-memory radix-2 DIT, in place;
//   DirectDft  n even and not a power of two (the reference's 48 kHz improved_fullsubnet example uses n_fft = 960,
//              hop = 480: recipes/dns_interspeech_2020/improved_fullsubnet/model.py:603-620): a direct O(n^2) DFT in
//              shared memory against a full-circle twiddle table.  At n = 960 that is 3.7 MFLOP per frame, i.e. < 1 %
//              of the model's 217 MFLOP per frame, so a mixed-radix FFT would not move the step time.
#include <limits.h>
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

constexpr int kFR = 16;        // frames per CTA
constexpr int kDspThreads = 256;

__device__ __forceinline__ int ilog2(int n) { return 31 - __clz(n); }

// in-place radix-2 DIT over `npairs` independent transforms whose inputs are already in
// bit-reversed order; tw[k] = exp(-2*pi*i*k/n).  Returns z.
template <bool INVERSE>
__device__ __forceinline__ float2* fft_radix2_smem(float2* z, int zstride, int npairs, int n, int log2n,
                                                   const float2* tw) {
  const int nb_log = log2n - 1;
  const int total = npairs << nb_log;
  for (int s = 1; s <= log2n; ++s) {
    const int half = 1 << (s - 1);
    const int tw_shift = log2n - s;
    for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
      const int p = idx >> nb_log;
      const int j = idx & ((1 << nb_log) - 1);
      const int pos = j & (half - 1);
      const int i0 = ((j >> (s - 1)) << s) + pos;
      const int i1 = i0 + half;
      float2 w = tw[pos << tw_shift];
      if (INVERSE) w.y = -w.y;
      float2* zp = z + p * zstride;
      const float2 a = zp[i0], b = zp[i1];
      const float tx = b.x * w.x - b.y * w.y;
      const float ty = b.x * w.y + b.y * w.x;
      zp[i0] = make_float2(a.x + tx, a.y + ty);
      zp[i1] = make_float2(a.x - tx, a.y - ty);
    }
    __syncthreads();
  }
  return z;
}

// out[p][k] = sum_i in[p][i] * tw[(i*k) mod n]   (INVERSE: conj(tw)); np transforms of length n, natural order.
// Returns out.
template <bool INVERSE>
__device__ __forceinline__ float2* dft_smem(const float2* in, float2* out, int np, int n, const float2* tw) {
  for (int idx = threadIdx.x; idx < np * n; idx += blockDim.x) {
    const int p = idx / n;
    const int k = idx - p * n;
    const float2* a = in + (size_t)p * n;
    float re = 0.f, im = 0.f;
    int m = 0;
    // at n = 960 (one CTA per SM) this loop is latency-bound, and the compiler's default 4-way schedule of it shifts
    // with the code of the calling kernel, by up to 13 % on an H100; unrolled by 8 it is faster in all three kernels
#pragma unroll 8
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
  return out;
}

// A transform policy holds what differs between the two transforms, and nothing else: the dynamic shared memory of np
// frame pairs (the transform's input rows `stride` apart, its result, tw_len twiddles, the window of n floats), the
// input slot of sample i, the (pair, sample) of a flat fill index, and the transform, which returns the buffer that
// holds the result (row j >> 1 has frame j).
struct Radix2 {  // in place, bit-reversed input, twiddles for k < n/2
  static size_t smem_bytes(int n, int np) { return (size_t)np * (n + 1) * 8 + (size_t)n / 2 * 8 + (size_t)n * 4; }
  int n, log2n, stride, tw_len;
  float2 *in, *tw;
  float* win;
  __device__ Radix2(float2* smem, int n_, int np)
      : n(n_), log2n(ilog2(n_)), stride(n_ + 1), tw_len(n_ / 2), in(smem), tw(smem + np * stride),
        win(reinterpret_cast<float*>(tw + n_ / 2)) {}
  __device__ void split(int idx, int& p, int& i) const { p = idx >> log2n; i = idx & (n - 1); }
  __device__ int slot(int i) const { return (int)(__brev((unsigned)i) >> (32 - log2n)); }
  template <bool INVERSE>
  __device__ const float2* transform(int np) const { return fft_radix2_smem<INVERSE>(in, stride, np, n, log2n, tw); }
};

struct DirectDft {  // out of place, natural-order input, twiddles for the full circle
  static size_t smem_bytes(int n, int np) { return (size_t)2 * np * n * 8 + (size_t)n * 8 + (size_t)n * 4; }
  int n, stride, tw_len;
  float2 *in, *out, *tw;
  float* win;
  __device__ DirectDft(float2* smem, int n_, int np)
      : n(n_), stride(n_), tw_len(n_), in(smem), out(smem + np * n_), tw(out + np * n_),
        win(reinterpret_cast<float*>(tw + n_)) {}
  __device__ void split(int idx, int& p, int& i) const { p = idx / n; i = idx - p * n; }
  __device__ int slot(int i) const { return i; }
  template <bool INVERSE>
  __device__ const float2* transform(int np) const { return dft_smem<INVERSE>(in, out, np, n, tw); }
};

// tw[k] = exp(-2*pi*i*k/n) for k < tw_len; win = periodic Hann of win_length centred in n
__device__ __forceinline__ void init_tables(float2* tw, int tw_len, float* win, int n, int win_length) {
  for (int k = threadIdx.x; k < tw_len; k += blockDim.x) {
    float s, c;
    sincospif(-2.0f * (float)k / (float)n, &s, &c);
    tw[k] = make_float2(c, s);
  }
  const int left = (n - win_length) / 2;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int m = i - left;
    // torch.hann_window(1) is [1], not the 0 of the periodic formula
    const float h = win_length == 1 ? 1.0f : 0.5f - 0.5f * cospif(2.0f * (float)m / (float)win_length);
    win[i] = (m >= 0 && m < win_length) ? h : 0.0f;
  }
}

// windowed frames t0 + 2p (real lane) and t0 + 2p + 1 (imaginary lane) of np pairs into the transform's input;
// sample(t, i) is sample i of frame t < Tv, frames from Tv on enter as zeros
template <class P, class Sample>
__device__ __forceinline__ void fill_frame_pairs(const P& tr, int np, int t0, int Tv, Sample sample) {
  for (int idx = threadIdx.x; idx < np * tr.n; idx += blockDim.x) {
    int p, i;
    tr.split(idx, p, i);
    const int ta = t0 + 2 * p, tb = ta + 1;
    const float w = tr.win[i];
    float va = 0.f, vb = 0.f;
    if (ta < Tv) va = sample(ta, i) * w;
    if (tb < Tv) vb = sample(tb, i) * w;
    tr.in[p * tr.stride + tr.slot(i)] = make_float2(va, vb);
  }
}

// (Re, Im) of bin k of frame j from the packed transform result z.  At DC and Nyquist zk == zn, so both Im are +0 and
// a negative Re has phase +pi, as torch.angle gives.
__device__ __forceinline__ float2 unpack_bin(const float2* z, int stride, int n, int j, int k) {
  const float2 zk = z[(j >> 1) * stride + k];
  const float2 zn = z[(j >> 1) * stride + (k == 0 ? 0 : n - k)];
  float re, im;
  if ((j & 1) == 0) { re = 0.5f * (zk.x + zn.x); im = 0.5f * (zk.y - zn.y); }
  else              { re = 0.5f * (zk.y + zn.y); im = 0.5f * (zn.x - zk.x); }
  return make_float2(re, im);
}

// ------------------------------------------------------------------------------------------
// lens (nullable, device [B]): clip b holds lens[b] <= L samples of its row (stride L), so it reflects at lens[b] and has
// T_b = 1 + lens[b]/hop frames; frames T_b .. T-1 are written as zeros and frame T_b enters its pair's transform as
// zeros, exactly as in a call on that clip alone.  Null: every clip has L samples.
template <class P>
__global__ void __launch_bounds__(kDspThreads)
stft_kernel(const float* __restrict__ wav, int L, int n, int hop, int win_length, int T,
            float* __restrict__ mag, float* __restrict__ phase, float* __restrict__ real,
            float* __restrict__ imag, float* __restrict__ magT, int T_pad, const int* __restrict__ lens) {
  extern __shared__ float2 smem2[];
  constexpr int NP = kFR / 2;
  const P tr(smem2, n, NP);
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * kFR;
  const int F = n / 2 + 1;
  const int Lb = lens ? lens[b] : L;
  const int Tb = lens ? 1 + Lb / hop : T;
  init_tables(tr.tw, tr.tw_len, tr.win, n, win_length);
  __syncthreads();
  const float* x = wav + (size_t)b * L;
  fill_frame_pairs(tr, NP, t0, Tb, [&](int t, int i) { return x[reflect_idx(t * hop + i - n / 2, Lb)]; });
  __syncthreads();
  const float2* z = tr.template transform<false>(NP);

  // un-pack the two real transforms and store in the reference layout [B,F,T]
  const size_t plane = (size_t)F * T;
  for (int idx = threadIdx.x; idx < F * kFR; idx += blockDim.x) {
    const int k = idx / kFR;
    const int j = idx - k * kFR;
    const int t = t0 + j;
    if (t >= T) continue;
    float2 c = unpack_bin(z, tr.stride, n, j, k);
    if (t >= Tb) c = make_float2(0.f, 0.f);
    const size_t o = (size_t)b * plane + (size_t)k * T + t;
    if (real) real[o] = c.x;
    if (imag) imag[o] = c.y;
    if (mag) mag[o] = hypotf(c.x, c.y);
    if (phase) phase[o] = atan2f(c.y, c.x);
  }
  if (magT) {  // time-major copy with the look-ahead rows zeroed
    for (int idx = threadIdx.x; idx < F * kFR; idx += blockDim.x) {
      const int j = idx / F;
      const int k = idx - j * F;
      const int t = t0 + j;
      if (t >= T_pad) continue;
      float m = 0.f;
      if (t < Tb) {
        const float2 c = unpack_bin(z, tr.stride, n, j, k);
        m = hypotf(c.x, c.y);
      }
      magT[((size_t)b * T_pad + t) * F + k] = m;
    }
  }
}

// ------------------------------------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(kDspThreads)
istft_kernel(const float* __restrict__ real, const float* __restrict__ imag, int cstride,
             const float* __restrict__ crm, int mask_mode, int T, int n, int hop, int win_length, int out_len,
             int seg, int np_max, float* __restrict__ wav, unsigned int* __restrict__ peak_bits,
             const int* __restrict__ lens) {
  extern __shared__ float2 smem2[];
  const P tr(smem2, n, np_max);
  const int b = blockIdx.y;
  const int F = n / 2 + 1;
  // lens (nullable): clip b has T_b = 1 + lens[b]/hop of the T frames (row stride T) and lens[b] of the out_len output
  // samples (row stride out_len); samples lens[b] .. out_len-1 are written as 0.  The segment tiling is absolute, so
  // each CTA pairs the same frames as a call on that clip alone.
  const int Lb = lens ? lens[b] : out_len;
  const int Tb = lens ? 1 + Lb / hop : T;
  const int s_begin = n / 2 + blockIdx.x * seg;
  const int s_end = min(s_begin + seg, n / 2 + Lb);
  const int t_min = (s_begin >= n) ? (s_begin - n) / hop + 1 : 0;
  const int t_max = min(Tb - 1, (s_end - 1) / hop);
  const int nframes = t_max - t_min + 1;
  const int np = nframes > 0 ? (nframes + 1) / 2 : 0;
  init_tables(tr.tw, tr.tw_len, tr.win, n, win_length);
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
        if (crm && mask_mode == 2) {  // improved_fullsubnet/model.py:575-576: element-wise, no decompression
          r *= cr[o];
          i *= ci[o];
        } else if (crm) {  // mask.py:58-63 then inferencer.py:139-140
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
    tr.in[p * tr.stride + tr.slot(k)] = make_float2(e[0][0] - e[1][1], e[0][1] + e[1][0]);
    if (k > 0 && k < n / 2)
      tr.in[p * tr.stride + tr.slot(n - k)] = make_float2(e[0][0] + e[1][1], -e[0][1] + e[1][0]);
  }
  __syncthreads();
  const float2* z = tr.template transform<true>(np);

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
        const float2 v = z[(q >> 1) * tr.stride + i];
        const float w = tr.win[i];
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
  if (peak_bits) {
    // max|y| of the clip for the int16 scaling of the host loop (base_inferencer.py:181-182): non-negative floats
    // order like their bit patterns, and max is order-independent, so the atomic is deterministic
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) peak = fmaxf(peak, __shfl_xor_sync(0xffffffffu, peak, o));
    if ((threadIdx.x & 31) == 0 && peak > 0.f) atomicMax(peak_bits + b, __float_as_uint(peak));
  }
}

// g(s) = d loss / d (overlap-added sample s) of the iSTFT: dwav at the sample the forward wrote (s - n/2 in [0, L), s
// inside the frames) over the window-square envelope, with the same frames in the same order as istft_kernel; else 0
__device__ __forceinline__ float istft_adjoint_sample(const float* __restrict__ dwav, const float* __restrict__ win, int s,
                                                      int n, int hop, int T, int L) {
  if (s < n / 2 || s >= n / 2 + L || s >= n + hop * (T - 1)) return 0.f;
  const int tl = (s >= n) ? (s - n) / hop + 1 : 0;
  const int th = min(T - 1, s / hop);
  float env = 0.f;
  for (int t = tl; t <= th; ++t) {
    const float w = win[s - t * hop];
    env += w * w;
  }
  return (env > 1e-11f) ? dwav[s - n / 2] / env : 0.f;
}

// Adjoint of (element-wise mask, irfft, window, overlap-add, envelope, crop) with respect to the mask, same tiling as
// stft_kernel (kFR frames per CTA, two real frames per complex transform): frame t's samples g(t*hop + i) * win[i] go
// through the forward real DFT; irfft's adjoint scales bin k by c_k/n (c = 1 at DC, 2 at bins 1 .. n/2-1, the
// Im of DC gets no gradient), and the product with the kept spectrum gives dcrm[b,0,k,t] = dRe * real,
// dcrm[b,1,k,t] = dIm * imag for k < F-1.
template <class P>
__global__ void __launch_bounds__(kDspThreads)
istft_mask_adjoint_kernel(const float* __restrict__ dwav, const float* __restrict__ real, const float* __restrict__ imag,
                          int L, int n, int hop, int win_length, int T, float* __restrict__ dcrm) {
  extern __shared__ float2 smem2[];
  constexpr int NP = kFR / 2;
  const P tr(smem2, n, NP);
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * kFR;
  const int F = n / 2 + 1;
  init_tables(tr.tw, tr.tw_len, tr.win, n, win_length);
  __syncthreads();
  const float* g = dwav + (size_t)b * L;
  fill_frame_pairs(tr, NP, t0, T, [&](int t, int i) { return istft_adjoint_sample(g, tr.win, t * hop + i, n, hop, T, L); });
  __syncthreads();
  const float2* z = tr.template transform<false>(NP);
  const size_t plane = (size_t)F * T;
  for (int idx = threadIdx.x; idx < (F - 1) * kFR; idx += blockDim.x) {
    const int k = idx / kFR;
    const int j = idx - k * kFR;
    const int t = t0 + j;
    if (t >= T) continue;
    const float2 c = unpack_bin(z, tr.stride, n, j, k);
    const float sc = (k == 0 ? 1.f : 2.f) / (float)n;
    const size_t o = (size_t)b * plane + (size_t)k * T + t;
    dcrm[(size_t)b * plane + o] = sc * c.x * real[o];
    dcrm[(size_t)b * plane + plane + o] = k == 0 ? 0.f : sc * c.y * imag[o];
  }
}

// out = int16(gain * wav / peak) per clip, peak from the iSTFT epilogue (float32 mul, div, truncation like numpy);
// lens (nullable): 0 past the clip's own lens[b] samples of its row
__global__ void scale_int16_kernel(const float* __restrict__ wav, const unsigned int* __restrict__ peak_bits, int L, float gain,
                                   int16_t* __restrict__ out, size_t n, const int* __restrict__ lens) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i / L;
    const float m = __uint_as_float(peak_bits[b]);
    const bool keep = !lens || (int)(i - b * L) < lens[b];
    out[i] = (keep && m > 0.f) ? (int16_t)__fdiv_rn(__fmul_rn(gain, wav[i]), m) : (int16_t)0;
  }
}

// per-clip length table: lengths[off + i] = v[i], the values travelling in the parameter block (no host buffer is read
// after the launch, and no copy from pageable memory can synchronise the stream)
constexpr int kLenChunk = 1000;  // 4 KB parameter block with the two counts
struct LenChunk { int off, n; int v[kLenChunk]; };
__global__ void lengths_table_kernel(const __grid_constant__ LenChunk c, int* __restrict__ lengths) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c.n) lengths[c.off + i] = c.v[i];
}

// crm [B, C, T]: frames t >= 1 + lengths[b]/hop of clip b set to 0
__global__ void zero_frames_past_kernel(float* __restrict__ crm, const int* __restrict__ lengths, int C, int T, int hop,
                                        size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / ((size_t)C * T));
    if ((int)(i % T) >= 1 + lengths[b] / hop) crm[i] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------
__global__ void decompress_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t n, float K,
                                  float limit) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = decompress_cirm_f(in[i], K, limit);
}

__global__ void compress_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t n, float K, float C) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = compress_cirm_f(in[i], K, C);
}

// mask.py:22-29
__global__ void build_cirm_kernel(const float* __restrict__ nr, const float* __restrict__ ni,
                                  const float* __restrict__ cr, const float* __restrict__ ci,
                                  float2* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = cirm_f(nr[i], ni[i], cr[i], ci[i]);
}

// feature.py:332-345: output clip b' of group g <- clip g + G*i, frequency f' <- g + G*f'
__global__ void drop_band_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int F,
                                 int T, int G) {
  const int Fo = F / G;
  const int64_t total = (int64_t)B * C * Fo * T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    int64_t r = i / T;
    const int fo = (int)(r % Fo); r /= Fo;
    const int c = (int)(r % C);
    int bo = (int)(r / C);
    int g = 0;
    for (; g < G; ++g) {  // group g holds ceil((B-g)/G) clips
      const int cnt = (B - g + G - 1) / G;
      if (bo < cnt) break;
      bo -= cnt;
    }
    const int bi = g + G * bo;
    const int fi = g + G * fo;
    out[i] = in[(((int64_t)bi * C + c) * F + fi) * T + t];
  }
}

// base_inferencer.py:181-182: int16(0.8 * 32767 * y / max|y|) per clip; one CTA per clip (max reduce, then scale)
__global__ void peak_normalize_int16_kernel(const float* __restrict__ wav, int L, float gain, int16_t* __restrict__ out) {
  __shared__ float sh[256];
  const float* x = wav + (size_t)blockIdx.x * L;
  float m = 0.f;
  for (int i = threadIdx.x; i < L; i += blockDim.x) m = fmaxf(m, fabsf(x[i]));
  sh[threadIdx.x] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] = fmaxf(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  m = sh[0];
  int16_t* o = out + (size_t)blockIdx.x * L;
  for (int i = threadIdx.x; i < L; i += blockDim.x)
    o[i] = (m > 0.f) ? (int16_t)__fdiv_rn(__fmul_rn(gain, x[i]), m) : (int16_t)0;  // float32 mul, div, truncation like numpy
}

// audio_zen/metrics.py:6-31 SI_SDR(reference, estimation) per clip: alpha = <ref,est>/<ref,ref>;
// 10 log10(|alpha ref|^2 / |est - alpha ref|^2).  One CTA per clip, two passes, fixed-order tree reductions in
// double (the reference sums in float32 pairwise; both agree to ~1e-5 dB on 4 s clips).  The CTA of 256 threads reduces
// the L samples at r / e into *out.
__device__ __forceinline__ void si_sdr_clip(const float* __restrict__ r, const float* __restrict__ e, int L,
                                            float* __restrict__ out) {
  __shared__ double sa[256], sb[256];
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) { a += (double)r[i] * r[i]; b += (double)r[i] * e[i]; }
  sa[threadIdx.x] = a; sb[threadIdx.x] = b;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) { sa[threadIdx.x] += sa[threadIdx.x + s]; sb[threadIdx.x] += sb[threadIdx.x + s]; }
    __syncthreads();
  }
  const float alpha = (float)sb[0] / (float)sa[0];  // float32 like the reference's optimal_scaling
  __syncthreads();
  a = 0.0; b = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const float p = alpha * r[i];
    const float n = e[i] - p;
    a += (double)p * p; b += (double)n * n;
  }
  sa[threadIdx.x] = a; sb[threadIdx.x] = b;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) { sa[threadIdx.x] += sa[threadIdx.x + s]; sb[threadIdx.x] += sb[threadIdx.x + s]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = (float)(10.0 * log10(sa[0] / sb[0]));
}

// clip b: row b of [B, L]
__global__ void si_sdr_kernel(const float* __restrict__ ref, const float* __restrict__ est, int L, float* __restrict__ out) {
  const size_t o = (size_t)blockIdx.x * L;
  si_sdr_clip(ref + o, est + o, L, out + blockIdx.x);
}

// clip c.off + i: the first c.v[i] samples of its row of [B, L_max]
__global__ void si_sdr_lengths_kernel(const float* __restrict__ ref, const float* __restrict__ est, int L_max,
                                      const __grid_constant__ LenChunk c, float* __restrict__ out) {
  const int b = c.off + blockIdx.x;
  const size_t o = (size_t)b * L_max;
  si_sdr_clip(ref + o, est + o, c.v[blockIdx.x], out + b);
}

static bool is_pow2(int n) { return n > 0 && (n & (n - 1)) == 0; }

// the transform policy: DirectDft for these sizes, Radix2 for the powers of two
static bool dft_size_ok(int n) { return !is_pow2(n) && (n & 1) == 0 && n >= 16 && n <= 1200; }
bool dsp_size_ok(int n) { return dft_size_ok(n) || (is_pow2(n) && n >= 16 && n <= 2048); }

constexpr int kMaxGridY = 65535;            // the three DSP grids put the clip in gridDim.y
constexpr size_t kSmemOptin = 227 * 1024;  // opt-in dynamic shared memory per block on sm_90

// dynamic shared memory of np frame pairs under the policy that runs n_fft
static size_t dsp_smem_bytes(int n_fft, int np) {
  return dft_size_ok(n_fft) ? DirectDft::smem_bytes(n_fft, np) : Radix2::smem_bytes(n_fft, np);
}

// the most frame pairs one iSTFT CTA transforms: the frames overlapping its kFR * hop output samples
static int istft_np_max(int n_fft, int hop) { return (kFR + cdiv(n_fft, hop) + 2) / 2; }
static size_t istft_smem_bytes(int n_fft, int hop) { return dsp_smem_bytes(n_fft, istft_np_max(n_fft, hop)); }

// launches a DSP kernel with smem bytes of dynamic shared memory, opting in to more than the default 48 KB
template <typename... KArgs, typename... Args>
static int dsp_launch(void (*kernel)(KArgs...), dim3 grid, size_t smem, cudaStream_t st, const char* name,
                      Args... args) {
  if (smem > 48 * 1024) {
    const int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), name);
    if (rc) return rc;
  }
  kernel<<<grid, kDspThreads, smem, st>>>(args...);
  FSN_CHECK_LAUNCH(name);
  return FSN_OK;
}

// host checks of stft_launch, before any CUDA call
int stft_check(int B, int L, int n_fft, int hop, int win_length, const float* magT, int T_pad) {
  FSN_REQUIRE(B > 0 && L > 0, FSN_ERR_SHAPE, "stft: empty input (B=%d, L=%d)", B, L);
  FSN_REQUIRE(B <= kMaxGridY, FSN_ERR_UNSUPPORTED, "stft: B=%d clips, at most %d", B, kMaxGridY);
  FSN_REQUIRE(dsp_size_ok(n_fft), FSN_ERR_UNSUPPORTED,
              "stft: n_fft=%d unsupported (power of two in [16,2048], or even and <= 1200)", n_fft);
  FSN_REQUIRE(hop > 0 && win_length > 0 && win_length <= n_fft, FSN_ERR_SHAPE, "stft: bad hop/win_length");
  FSN_REQUIRE(n_fft / 2 < L, FSN_ERR_SHAPE, "stft: reflect padding %d needs L > pad (L=%d)", n_fft / 2, L);
  FSN_REQUIRE(!magT || T_pad >= 1 + L / hop, FSN_ERR_SHAPE, "stft: T_pad < T");
  return FSN_OK;
}

// host checks of istft_launch, before any CUDA call (the peak memset included)
static int istft_check(int B, int T, int n_fft, int hop, int win_length, int cstride, int length, bool lens) {
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "istft: empty input");
  FSN_REQUIRE(B <= kMaxGridY, FSN_ERR_UNSUPPORTED, "istft: B=%d clips, at most %d", B, kMaxGridY);
  FSN_REQUIRE(!lens || length > 0, FSN_ERR_UNSUPPORTED, "istft: per-clip lengths need an output length");
  FSN_REQUIRE(dsp_size_ok(n_fft), FSN_ERR_UNSUPPORTED,
              "istft: n_fft=%d unsupported (power of two in [16,2048], or even and <= 1200)", n_fft);
  FSN_REQUIRE(hop > 0 && hop <= n_fft && win_length > 0 && win_length <= n_fft, FSN_ERR_SHAPE,
              "istft: bad hop/win_length");
  FSN_REQUIRE(cstride == 1 || cstride == 2, FSN_ERR_SHAPE, "istft: cstride must be 1 or 2");
  const int out_len = length > 0 ? length : hop * (T - 1);
  FSN_REQUIRE(out_len > 0, FSN_ERR_SHAPE, "istft: output length %d", out_len);
  // a clip of lens[b] <= length samples reads frames up to lens[b]/hop
  FSN_REQUIRE(!lens || length / hop < T, FSN_ERR_SHAPE, "istft: %d frames, per-clip lengths up to %d need %d", T, length,
              1 + length / hop);
  const size_t smem = istft_smem_bytes(n_fft, hop);
  FSN_REQUIRE(smem <= kSmemOptin, FSN_ERR_UNSUPPORTED,
              "istft: n_fft=%d with hop=%d needs %zu bytes of shared memory, at most %zu", n_fft, hop, smem, kSmemOptin);
  return FSN_OK;
}

int stft_launch(const float* wav, int B, int L, int n_fft, int hop, int win_length, float* mag, float* phase,
                float* real, float* imag, float* magT, int T_pad, cudaStream_t st, const int* lens) {
  const int rc = stft_check(B, L, n_fft, hop, win_length, magT, T_pad);
  if (rc) return rc;
  const int T = 1 + L / hop;
  const int Tg = magT ? (T_pad > T ? T_pad : T) : T;
  return dsp_launch(dft_size_ok(n_fft) ? stft_kernel<DirectDft> : stft_kernel<Radix2>, dim3(cdiv(Tg, kFR), B),
                    dsp_smem_bytes(n_fft, kFR / 2), st, "stft_kernel", wav, L, n_fft, hop, win_length, T, mag, phase,
                    real, imag, magT, T_pad, lens);
}

int istft_mask_adjoint_launch(const float* dwav, const float* real, const float* imag, int B, int L, int T, int n_fft,
                              int hop, int win_length, float* dcrm, cudaStream_t st) {
  FSN_REQUIRE(B > 0 && L > 0 && T > 0 && hop > 0 && hop <= n_fft && win_length > 0 && win_length <= n_fft, FSN_ERR_SHAPE,
              "istft adjoint: bad shape");
  FSN_REQUIRE(B <= kMaxGridY, FSN_ERR_UNSUPPORTED, "istft adjoint: B=%d clips, at most %d", B, kMaxGridY);
  FSN_REQUIRE(dsp_size_ok(n_fft), FSN_ERR_UNSUPPORTED,
              "istft adjoint: n_fft=%d unsupported (power of two in [16,2048], or even and <= 1200)", n_fft);
  return dsp_launch(dft_size_ok(n_fft) ? istft_mask_adjoint_kernel<DirectDft> : istft_mask_adjoint_kernel<Radix2>,
                    dim3(cdiv(T, kFR), B), dsp_smem_bytes(n_fft, kFR / 2), st, "istft_mask_adjoint_kernel", dwav, real,
                    imag, L, n_fft, hop, win_length, T, dcrm);
}

int istft_launch(const float* real, const float* imag, int cstride, const float* crm, int B, int T, int n_fft,
                 int hop, int win_length, int length, float* wav, cudaStream_t st, int mask_mode, unsigned int* peak_bits,
                 const int* lens) {
  int rc = istft_check(B, T, n_fft, hop, win_length, cstride, length, lens != nullptr);
  if (rc) return rc;
  if (peak_bits) {
    rc = check_cuda(cudaMemsetAsync(peak_bits, 0, (size_t)B * sizeof(unsigned int), st), "istft peak memset");
    if (rc) return rc;
  }
  const int out_len = length > 0 ? length : hop * (T - 1);
  const int seg = kFR * hop;
  return dsp_launch(dft_size_ok(n_fft) ? istft_kernel<DirectDft> : istft_kernel<Radix2>, dim3(cdiv(out_len, seg), B),
                    istft_smem_bytes(n_fft, hop), st, "istft_kernel", real, imag, cstride, crm, mask_mode, T, n_fft, hop,
                    win_length, out_len, seg, istft_np_max(n_fft, hop), wav, peak_bits, lens);
}

// ---- streaming STFT / iSTFT (DESIGN 4.14).  Both compute every frame pair and every output sample with the code and
// the operation order of stft_kernel / istft_kernel: a frame's transform depends only on its absolute pair (2k, 2k+1)
// (STFT) or on the absolute segment tiling (iSTFT), never on where a call starts.

// Step j of slot b is frame m = pos0[b]/hop - c + j (negative: a step before the clip's first frame).  win [B, Wn] holds
// the slot's samples from pos0[b] - Hs on.  Writes magT [B, S, F] (0 outside [0, T_b)) and the spectrum (re | im, 2F
// per frame) of step j at frame Q + j of spec [B, Q + S, 2F].  tail[b] >= 0: the clip has pos0[b] + tail[b] samples.
template <class P>
__global__ void __launch_bounds__(kDspThreads)
stft_stream_kernel(const float* __restrict__ win, int Wn, int Hs, const int* __restrict__ pos0, const int* __restrict__ tail,
                   int n, int hop, int win_length, int c, int S, int Q, float* __restrict__ magT, float* __restrict__ spec) {
  extern __shared__ float2 smem2[];
  constexpr int NP = kFR / 2;
  const P tr(smem2, n, NP);
  const int b = blockIdx.y;
  const int F = n / 2 + 1;
  const int p0 = pos0[b], m0 = p0 / hop - c, tl = tail[b];
  const int Lb = tl >= 0 ? p0 + tl : INT_MAX;
  const int Tb = tl >= 0 ? 1 + Lb / hop : INT_MAX;
  const int t0 = (m0 >= 0 ? m0 / 2 : -((1 - m0) / 2)) * 2 + blockIdx.x * kFR;  // pairs start on even frames
  init_tables(tr.tw, tr.tw_len, tr.win, n, win_length);
  __syncthreads();
  const float* x = win + (size_t)b * Wn;
  fill_frame_pairs(tr, NP, t0, Tb, [&](int t, int i) {
    if (t < 0) return 0.f;
    const int w = reflect_idx(t * hop + i - n / 2, Lb) - (p0 - Hs);
    return x[min(max(w, 0), Wn - 1)];
  });
  __syncthreads();
  const float2* z = tr.template transform<false>(NP);
  for (int idx = threadIdx.x; idx < F * kFR; idx += blockDim.x) {
    const int j = idx / F;
    const int k = idx - j * F;
    const int t = t0 + j, js = t - m0;
    if (js < 0 || js >= S) continue;
    const bool in = t >= 0 && t < Tb;
    const float2 cb = in ? unpack_bin(z, tr.stride, n, j, k) : make_float2(0.f, 0.f);
    magT[((size_t)b * S + js) * F + k] = in ? hypotf(cb.x, cb.y) : 0.f;
    float* sp = spec + ((size_t)b * (Q + S) + Q + js) * 2 * F;
    sp[k] = cb.x;
    sp[F + k] = cb.y;
  }
}

// Output row b of wav [B, K*hop + D] holds clip samples [pos0 - D, pos0 - D + K*hop), or on the clip's last call
// [pos0 - D, pos0 + tail); 0 elsewhere.  spec / crm [B, W, 2F] hold frames T0 + i, T0 = pos0/hop - c - la - Rc, with
// W = Q + S (spectrum) and Rc + S (cRM).  CTA x covers the row's samples in absolute iSTFT segment g0 + x.
template <class P>
__global__ void __launch_bounds__(kDspThreads)
istft_stream_kernel(const float* __restrict__ spec, const float* __restrict__ crm, const int* __restrict__ pos0,
                    const int* __restrict__ act0, const int* __restrict__ tail, int K, int D, int n, int hop,
                    int win_length, int seg, int np_max, int c, int la, int Rc, int Q, int S, float* __restrict__ wav) {
  extern __shared__ float2 smem2[];
  const P tr(smem2, n, np_max);
  const int b = blockIdx.y;
  const int F = n / 2 + 1;
  const int p0 = pos0[b], tl = tail[b], rowlen = K * hop + D;
  const int x_lo = p0 - D;
  const int x_hi = !act0[b] ? x_lo : (tl >= 0 ? p0 + tl : x_lo + K * hop);
  const int Lb = tl >= 0 ? p0 + tl : INT_MAX / 2;
  const int Tb = tl >= 0 ? 1 + Lb / hop : INT_MAX / 2;
  float* out = wav + (size_t)b * rowlen;
  if (blockIdx.x == 0)
    for (int j = threadIdx.x; j < rowlen; j += blockDim.x)
      if (x_lo + j < 0 || x_lo + j >= x_hi) out[j] = 0.f;
  const int g = max(x_lo, 0) / seg + blockIdx.x;
  const int s_begin = n / 2 + g * seg;
  const int s_end = min(s_begin + seg, n / 2 + Lb);
  const int a = max(s_begin, n / 2 + max(x_lo, 0)), e = min(s_end, n / 2 + x_hi);
  if (a >= e) return;
  const int t_min = (s_begin >= n) ? (s_begin - n) / hop + 1 : 0;
  const int t_max = min(Tb - 1, (s_end - 1) / hop);
  const int tlo = max(t_min, (a >= n) ? (a - n) / hop + 1 : 0), thi = min(t_max, (e - 1) / hop);
  const int pb = t_min + 2 * ((tlo - t_min) / 2);  // first frame of the first pair the samples read
  const int np = thi >= tlo ? (thi - pb) / 2 + 1 : 0;
  const int T0 = p0 / hop - c - la - Rc;
  init_tables(tr.tw, tr.tw_len, tr.win, n, win_length);
  const float* xs = spec + (size_t)b * (Q + S) * 2 * F;
  const float* xc = crm + (size_t)b * (Rc + S) * 2 * F;
  for (int idx = threadIdx.x; idx < F * np; idx += blockDim.x) {
    const int k = idx / np;
    const int p = idx - k * np;
    float ev[2][2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int t = pb + 2 * p + q;
      float r = 0.f, i = 0.f;
      if (t <= t_max) {
        const float* sp = xs + (size_t)(t - T0) * 2 * F;
        const float* cp = xc + (size_t)(t - T0) * 2 * F;
        r = sp[k];
        i = sp[F + k];
        const float mr = decompress_cirm_f(cp[k], 10.0f, 9.9f);
        const float mi = decompress_cirm_f(cp[F + k], 10.0f, 9.9f);
        const float er = mr * r - mi * i;
        const float ei = mi * r + mr * i;
        r = er; i = ei;
      }
      ev[q][0] = r;
      ev[q][1] = (k == 0 || k == n / 2) ? 0.f : i;
    }
    tr.in[p * tr.stride + tr.slot(k)] = make_float2(ev[0][0] - ev[1][1], ev[0][1] + ev[1][0]);
    if (k > 0 && k < n / 2)
      tr.in[p * tr.stride + tr.slot(n - k)] = make_float2(ev[0][0] + ev[1][1], -ev[0][1] + ev[1][0]);
  }
  __syncthreads();
  const float2* z = tr.template transform<true>(np);
  const int full = tl >= 0 ? n + hop * (Tb - 1) : INT_MAX;
  const float inv_n = 1.0f / (float)n;
  for (int s = a + threadIdx.x; s < e; s += blockDim.x) {
    float acc = 0.f, env = 0.f;
    if (s < full) {
      const int t_lo = max(t_min, (s >= n) ? (s - n) / hop + 1 : 0);
      const int t_hi = min(t_max, s / hop);
      for (int t = t_lo; t <= t_hi; ++t) {
        const int i = s - t * hop;
        const int q = t - pb;
        const float2 v = z[(q >> 1) * tr.stride + i];
        const float w = tr.win[i];
        acc += ((q & 1) ? v.y : v.x) * inv_n * w;
        env += w * w;
      }
    }
    const float y = (env > 1e-11f) ? acc / env : 0.f;
    out[s - n / 2 - x_lo] = y;
  }
}

static int stream_np_max(int n_fft, int hop) { return istft_np_max(n_fft, hop) + 1; }

int stream_dsp_check(int n_fft, int hop, int win_length) {
  FSN_REQUIRE(is_pow2(n_fft) && n_fft >= 16 && n_fft <= 2048, FSN_ERR_UNSUPPORTED,
              "stream: n_fft=%d: streaming is built for the power-of-two (radix-2) transform in [16, 2048]", n_fft);
  FSN_REQUIRE(hop > 0 && hop <= n_fft && win_length > 0 && win_length <= n_fft, FSN_ERR_SHAPE,
              "stream: bad hop/win_length");
  FSN_REQUIRE(Radix2::smem_bytes(n_fft, stream_np_max(n_fft, hop)) <= kSmemOptin, FSN_ERR_UNSUPPORTED,
              "stream: n_fft=%d with hop=%d needs too much shared memory", n_fft, hop);
  return FSN_OK;
}

int stft_stream_launch(const float* win, int Wn, int Hs, const int* pos0, const int* tail, int B, int n_fft, int hop,
                       int win_length, int c, int S, int Q, float* magT, float* spec, cudaStream_t st) {
  return dsp_launch(stft_stream_kernel<Radix2>, dim3(cdiv(S + 1, kFR), B), Radix2::smem_bytes(n_fft, kFR / 2), st,
                    "stft_stream_kernel", win, Wn, Hs, pos0, tail, n_fft, hop, win_length, c, S, Q, magT, spec);
}

int istft_stream_launch(const float* spec, const float* crm, const int* pos0, const int* act0, const int* tail, int B,
                        int K, int D, int n_fft, int hop, int win_length, int c, int la, int Rc, int Q, int S, float* wav,
                        cudaStream_t st) {
  const int seg = kFR * hop, np_max = stream_np_max(n_fft, hop);
  return dsp_launch(istft_stream_kernel<Radix2>, dim3(cdiv(K * hop + D, seg) + 1, B), Radix2::smem_bytes(n_fft, np_max),
                    st, "istft_stream_kernel", spec, crm, pos0, act0, tail, K, D, n_fft, hop, win_length, seg, np_max, c,
                    la, Rc, Q, S, wav);
}

}  // namespace fsn

using namespace fsn;

extern "C" int fsn_stft(const float* wav, int B, int L, int n_fft, int hop, int win_length, float* mag,
                        float* phase, float* real, float* imag, float* magT, int T_pad, fsn_stream_t stream) {
  return stft_launch(wav, B, L, n_fft, hop, win_length, mag, phase, real, imag, magT, T_pad, (cudaStream_t)stream, nullptr);
}

extern "C" int fsn_istft(const float* real, const float* imag, int cstride, const float* crm, int B, int T,
                         int n_fft, int hop, int win_length, int length, float* wav, fsn_stream_t stream) {
  return istft_launch(real, imag, cstride, crm, B, T, n_fft, hop, win_length, length, wav, (cudaStream_t)stream, 1, nullptr,
                      nullptr);
}

extern "C" int fsn_peak_normalize_int16(const float* wav, int B, int L, float gain, int16_t* out, fsn_stream_t stream) {
  FSN_REQUIRE(B > 0 && L > 0, FSN_ERR_SHAPE, "peak_normalize: empty input");
  peak_normalize_int16_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(wav, L, gain, out);
  FSN_CHECK_LAUNCH("peak_normalize_int16_kernel");
  return FSN_OK;
}

extern "C" int fsn_si_sdr(const float* reference, const float* estimation, int B, int L, float* out, fsn_stream_t stream) {
  FSN_REQUIRE(B > 0 && L > 0, FSN_ERR_SHAPE, "si_sdr: empty input");
  si_sdr_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(reference, estimation, L, out);
  FSN_CHECK_LAUNCH("si_sdr_kernel");
  return FSN_OK;
}

extern "C" int fsn_si_sdr_lengths(const float* reference, const float* estimation, const int32_t* lengths, int B, int L_max,
                                  float* out, fsn_stream_t stream) {
  if (!lengths) return fsn_si_sdr(reference, estimation, B, L_max, out, stream);
  FSN_REQUIRE(B > 0 && L_max > 0, FSN_ERR_SHAPE, "si_sdr_lengths: empty input");
  for (int b = 0; b < B; ++b)
    FSN_REQUIRE(lengths[b] > 0 && lengths[b] <= L_max, FSN_ERR_SHAPE,
                "si_sdr_lengths: clip %d has length %d, outside (0, L_max] = (0, %d]", b, lengths[b], L_max);
  LenChunk c;  // the lengths travel in the parameter block, like the length table of the wav -> wav entry points
  for (int off = 0; off < B; off += kLenChunk) {
    c.off = off;
    c.n = B - off < kLenChunk ? B - off : kLenChunk;
    memcpy(c.v, lengths + off, (size_t)c.n * sizeof(int));
    si_sdr_lengths_kernel<<<c.n, 256, 0, (cudaStream_t)stream>>>(reference, estimation, L_max, c, out);
    FSN_CHECK_LAUNCH("si_sdr_lengths_kernel");
  }
  return FSN_OK;
}

// ---- the wav side of the wav -> wav entry points (fsn_internal.cuh)
namespace fsn {
void wav_carve(Carver& c, int B, int F, int T, WavWs& w) {
  const size_t BFT = (size_t)B * F * T;
  w.real = w.imag = w.crm = nullptr;
  if (BFT) { w.real = c.take<float>(BFT); w.imag = c.take<float>(BFT); w.crm = c.take<float>(2 * BFT); }
  w.peak = c.take<unsigned int>(B);
  w.lens = c.take<int>(B);
}

int wav_check(const int32_t* lengths, int B, int L_max, int n_fft, bool pow2_lengths, const float* enhanced,
              const char* who) {
  if (lengths) {
    FSN_REQUIRE(!pow2_lengths || (n_fft & (n_fft - 1)) == 0, FSN_ERR_UNSUPPORTED,
                "%s: n_fft=%d: per-clip lengths are built for the power-of-two (radix-2) transform", who, n_fft);
    int longest = 0;
    for (int b = 0; b < B; ++b) {
      FSN_REQUIRE(lengths[b] > n_fft / 2 && lengths[b] <= L_max, FSN_ERR_SHAPE,
                  "%s: clip %d has length %d, outside (n_fft/2, L_max] = (%d, %d]", who, b, lengths[b], n_fft / 2, L_max);
      longest = lengths[b] > longest ? lengths[b] : longest;
    }
    FSN_REQUIRE(longest == L_max, FSN_ERR_SHAPE, "%s: the longest clip has %d samples, L_max = %d", who, longest, L_max);
  }
  FSN_REQUIRE(enhanced, FSN_ERR_SHAPE, "%s: enhanced output buffer missing", who);
  return FSN_OK;
}

int wav_prologue(const int32_t* lengths, int B, WavWs& w, cudaStream_t st) {
  if (!lengths) {
    w.lens = nullptr;
    return FSN_OK;
  }
  LenChunk c;
  for (int off = 0; off < B; off += kLenChunk) {
    c.off = off;
    c.n = B - off < kLenChunk ? B - off : kLenChunk;
    memcpy(c.v, lengths + off, (size_t)c.n * sizeof(int));
    lengths_table_kernel<<<cdiv(c.n, 256), 256, 0, st>>>(c, w.lens);
    FSN_CHECK_LAUNCH("lengths_table_kernel");
  }
  return FSN_OK;
}

int wav_epilogue(const WavWs& w, const float* enhanced, int B, int L, int16_t* pcm, float gain, float* crm_out, int F, int T,
                 int hop, cudaStream_t st) {
  if (pcm) {
    const size_t n = (size_t)B * L;
    scale_int16_kernel<<<ew_grid((size_t)n), 256, 0, st>>>(enhanced, w.peak, L, gain, pcm, n, w.lens);
    FSN_CHECK_LAUNCH("scale_int16_kernel");
  }
  if (w.lens && crm_out) {
    const size_t n = (size_t)B * 2 * F * T;
    zero_frames_past_kernel<<<ew_grid((size_t)n), 256, 0, st>>>(crm_out, w.lens, 2 * F, T, hop, n);
    FSN_CHECK_LAUNCH("zero_frames_past_kernel");
  }
  return FSN_OK;
}
}  // namespace fsn

// ---- unit-test hooks of the signal layer (include/fsn_b200.h): the internal launchers called directly, every argument
// checked before any CUDA call; host lengths go to lens_dev through wav_prologue as in the wav -> wav entry points
extern "C" int fsn_debug_stft(const float* wav, int B, int L, int n_fft, int hop, int win_length, const int32_t* lengths,
                              int* lens_dev, float* mag, float* phase, float* real, float* imag, float* magT, int T_pad,
                              fsn_stream_t stream) {
  launch_counter() = 0;
  int rc = stft_check(B, L, n_fft, hop, win_length, magT, T_pad);
  if (rc) return rc;
  FSN_REQUIRE(!lengths || lens_dev, FSN_ERR_SHAPE, "stft hook: lengths need a device length table");
  if ((rc = wav_check(lengths, B, L, n_fft, false, wav, "stft hook"))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  WavWs w = {nullptr, nullptr, nullptr, nullptr, lens_dev};
  if ((rc = wav_prologue(lengths, B, w, st))) return rc;
  return stft_launch(wav, B, L, n_fft, hop, win_length, mag, phase, real, imag, magT, T_pad, st, w.lens);
}

extern "C" int fsn_debug_istft(const float* real, const float* imag, int cstride, const float* crm, int mask_mode, int B,
                               int T, int n_fft, int hop, int win_length, int length, const int32_t* lengths, int* lens_dev,
                               float* wav, unsigned int* peak_bits, int16_t* pcm, float gain, float* crm_out,
                               fsn_stream_t stream) {
  launch_counter() = 0;
  int rc = istft_check(B, T, n_fft, hop, win_length, cstride, length, lengths != nullptr);
  if (rc) return rc;
  FSN_REQUIRE(mask_mode >= 0 && mask_mode <= 2, FSN_ERR_SHAPE, "istft hook: unknown mask mode %d", mask_mode);
  FSN_REQUIRE((crm != nullptr) == (mask_mode != 0), FSN_ERR_SHAPE, "istft hook: mask mode %d with%s a mask", mask_mode,
              crm ? "" : "out");
  FSN_REQUIRE(real && imag, FSN_ERR_SHAPE, "istft hook: null spectrum");
  FSN_REQUIRE(!pcm || peak_bits, FSN_ERR_SHAPE, "istft hook: the int16 output needs the peak");
  FSN_REQUIRE(!crm_out || lengths, FSN_ERR_SHAPE, "istft hook: zeroing frames past each clip needs lengths");
  FSN_REQUIRE(!lengths || lens_dev, FSN_ERR_SHAPE, "istft hook: lengths need a device length table");
  const int out_len = length > 0 ? length : hop * (T - 1);
  if ((rc = wav_check(lengths, B, out_len, n_fft, false, wav, "istft hook"))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  WavWs w = {nullptr, nullptr, nullptr, peak_bits, lens_dev};
  if ((rc = wav_prologue(lengths, B, w, st))) return rc;
  if ((rc = istft_launch(real, imag, cstride, crm, B, T, n_fft, hop, win_length, length, wav, st, mask_mode, peak_bits,
                         w.lens)))
    return rc;
  if (!pcm && !crm_out) return FSN_OK;
  return wav_epilogue(w, wav, B, out_len, pcm, gain, crm_out, n_fft / 2 + 1, T, hop, st);
}

extern "C" int fsn_debug_istft_mask_adjoint(const float* dwav, const float* real, const float* imag, int B, int L, int T,
                                            int n_fft, int hop, int win_length, float* dcrm, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(dwav && real && imag && dcrm, FSN_ERR_SHAPE, "istft adjoint hook: null argument");
  return istft_mask_adjoint_launch(dwav, real, imag, B, L, T, n_fft, hop, win_length, dcrm, (cudaStream_t)stream);
}

extern "C" int fsn_debug_wav_epilogue(const float* enhanced, const unsigned int* peak_bits, int B, int L,
                                      const int32_t* lengths, int* lens_dev, float gain, int16_t* pcm, float* crm_out, int F,
                                      int T, int hop, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(B > 0 && L > 0 && F >= 2 && T > 0 && hop > 0, FSN_ERR_SHAPE, "wav epilogue hook: bad shape");
  FSN_REQUIRE(!pcm || peak_bits, FSN_ERR_SHAPE, "wav epilogue hook: the int16 output needs the peak");
  FSN_REQUIRE(!crm_out || lengths, FSN_ERR_SHAPE, "wav epilogue hook: zeroing frames past each clip needs lengths");
  FSN_REQUIRE(!lengths || lens_dev, FSN_ERR_SHAPE, "wav epilogue hook: lengths need a device length table");
  int rc = wav_check(lengths, B, L, 2 * (F - 1), false, enhanced, "wav epilogue hook");
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  WavWs w = {nullptr, nullptr, nullptr, const_cast<unsigned int*>(peak_bits), lens_dev};
  if ((rc = wav_prologue(lengths, B, w, st))) return rc;
  return wav_epilogue(w, enhanced, B, L, pcm, gain, crm_out, F, T, hop, st);
}

extern "C" int fsn_decompress_cirm(const float* in, float* out, int64_t n, float K, float limit,
                                   fsn_stream_t stream) {
  if (n <= 0) return FSN_OK;
  decompress_kernel<<<ew_grid((size_t)n), 256, 0, (cudaStream_t)stream>>>(in, out, n, K, limit);
  FSN_CHECK_LAUNCH("decompress_kernel");
  return FSN_OK;
}

extern "C" int fsn_compress_cirm(const float* in, float* out, int64_t n, float K, float C, fsn_stream_t stream) {
  if (n <= 0) return FSN_OK;
  compress_kernel<<<ew_grid((size_t)n), 256, 0, (cudaStream_t)stream>>>(in, out, n, K, C);
  FSN_CHECK_LAUNCH("compress_kernel");
  return FSN_OK;
}

extern "C" int fsn_build_cirm(const float* nr, const float* ni, const float* cr, const float* ci, float* out,
                              int64_t n, fsn_stream_t stream) {
  if (n <= 0) return FSN_OK;
  build_cirm_kernel<<<ew_grid((size_t)n), 256, 0, (cudaStream_t)stream>>>(nr, ni, cr, ci, reinterpret_cast<float2*>(out), n);
  FSN_CHECK_LAUNCH("build_cirm_kernel");
  return FSN_OK;
}

extern "C" int fsn_drop_band(const float* in, float* out, int B, int C, int F, int T, int G, fsn_stream_t stream) {
  FSN_REQUIRE(B > G, FSN_ERR_SHAPE,
              "Batch size = %d, num_groups = %d. The batch size should larger than the num_groups.", B, G);
  FSN_REQUIRE(G >= 2, FSN_ERR_SHAPE, "drop_band: G < 2 is the identity, handle on the host");
  const int64_t n = (int64_t)B * C * (F / G) * T;
  if (n <= 0) return FSN_OK;
  drop_band_kernel<<<ew_grid((size_t)n), 256, 0, (cudaStream_t)stream>>>(in, out, B, C, F, T, G);
  FSN_CHECK_LAUNCH("drop_band_kernel");
  return FSN_OK;
}
