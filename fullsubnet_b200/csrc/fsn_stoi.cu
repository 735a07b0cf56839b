// STOI (Taal et al., 2011) for a batch of clips with per-clip lengths: pystoi 0.3.3's stoi(x, y, fs_sig, extended=False)
// as audio_zen/metrics.py:STOI calls it (clean x, estimate y), in float64 from the widened float32 inputs to the final
// rounding of out[b].
//
// Five kernels, each clip's values computed in a fixed order that depends on nothing but the clip itself:
//   stoi_resample_kernel  polyphase FIR to 10 kHz (taps from the host, std::call_once per rate), one output sample per
//                         thread, taps in ascending input order; at 10 kHz the same kernel with the one tap 1.0 widens;
//   stoi_select_kernel    one CTA per clip: frame energies of the clean signal (one warp per frame, fixed shuffle tree),
//                         the keep mask against the loudest frame, and the kept-frame index list by an exclusive scan;
//   stoi_ola_kernel       overlap-add of the kept windowed frames of clean and estimate into the compacted signals;
//   stoi_bands_kernel     the one-third-octave band magnitudes of kFB frames per CTA: a direct DFT of bins 7 .. 218
//                         only (the bands use 212 of the 257 bins; every bin is one fixed-order sum of 256 terms against
//                         a float64 twiddle table in shared memory), then the band sums in ascending bin order;
//   stoi_corr_kernel      one CTA per clip: each (segment, band) correlation from its 30 + 30 values directly, then one
//                         fixed-order tree over the clip's J * 15 correlations (fewer than 30 frames: 1e-5).
// The direct DFT is chosen over a float64 variant of fsn_dsp.cu's radix-2 FFT so that the float32 transform the model
// paths depend on stays untouched; it costs ~10x the FFT's multiply-adds, which DESIGN 4.12 measures.
#include <math.h>
#include <string.h>

#include <mutex>

#include "fsn_internal.cuh"

namespace fsn {
namespace {

constexpr int kFs = 10000;                 // pystoi FS
constexpr int kFrame = 256, kHop = 128;    // N_FRAME and its hop
constexpr int kBands = 15;                 // NUMBAND
constexpr int kSeg = 30;                   // N: frames per segment
constexpr int kBin0 = 7, kBins = 219 - 7;  // bins of the bands: [7, 219)
constexpr double kEps = 2.220446049250313e-16;  // np.finfo(float).eps
constexpr double kDynRange = 40.0;
constexpr int kThreads = 256;
constexpr int kFB = 8;                     // frames per stoi_bands_kernel CTA
constexpr int kMaxHalf = 290;              // the 16 kHz filter: 2 * 290 + 1 taps
constexpr int kMaxGridY = 65535;

// band j holds bins [kEdges[j], kEdges[j+1]): the bins nearest 150 * 2^((2j -+ 1)/6) Hz on f_k = k * 10000/512
__constant__ int kEdges[kBands + 1] = {7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219};

// the resampling filter of one rate: up * h / sum(h), h[half + t] = h[half - t], so taps j <= half are stored
struct Resampler {
  int up, down, half;
  double h[kMaxHalf + 1];
};

double bessel_i0(double x) {
  double s = 1.0, t = 1.0;
  for (int k = 1; k < 500; ++k) {
    const double q = x / (2.0 * k);
    t *= q * q;
    s += t;
    if (t < s * 1e-18) break;
  }
  return s;
}

// resample_oct(x, 10000, fs): the Kaiser-windowed sinc of Octave's resample (rejection 60 dB, roll-off cutoff / 10),
// normalised to unit sum and multiplied by up as scipy.signal.resample_poly does
void make_resampler(int sr, Resampler& r) {
  int a = kFs, b = sr;
  while (b) { const int t = a % b; a = b; b = t; }
  const int p = kFs / a, q = sr / a;
  r.up = p;
  r.down = q;
  if (p == 1 && q == 1) {
    r.half = 0;
    r.h[0] = 1.0;
    return;
  }
  const double cutoff = 1.0 / (2.0 * (p > q ? p : q));
  const double roll_off = cutoff / 10.0;
  const double rejection_db = 60.0;
  const int L = (int)ceil((rejection_db - 8.0) / (28.714 * roll_off));
  const double beta = 0.1102 * (rejection_db - 8.7);
  const double pi = 3.14159265358979323846;
  double full[2 * kMaxHalf + 1], sum = 0.0;
  for (int n = 0; n <= 2 * L; ++n) {
    const double u = (n - L) / (double)L;
    const double x = 2.0 * cutoff * (n - L);
    const double sinc = n == L ? 1.0 : sin(pi * x) / (pi * x);
    full[n] = bessel_i0(beta * sqrt(1.0 - u * u)) / bessel_i0(beta) * 2.0 * p * cutoff * sinc;
    sum += full[n];
  }
  r.half = L;
  for (int j = 0; j <= L; ++j) r.h[j] = p * (full[j] / sum);
}

const Resampler& resampler(int sr) {
  static Resampler r16, r10;
  static std::once_flag f16, f10;
  if (sr == 16000) {
    std::call_once(f16, [] { make_resampler(16000, r16); });
    return r16;
  }
  std::call_once(f10, [] { make_resampler(10000, r10); });
  return r10;
}

// shapes of one call: the resampled length of an L-sample clip, and its frames (the last possible frame excluded)
struct Rate { int up, down; };
Rate rate_of(int sr) { return sr == 16000 ? Rate{5, 8} : Rate{1, 1}; }
__host__ __device__ inline int resampled_len(int L, int up, int down) {
  return (int)(((int64_t)L * up + down - 1) / down);
}
__host__ __device__ inline int n_frames(int n) { return n > kFrame ? (n - kFrame + kHop - 1) / kHop : 0; }
int min_len(int sr) { const Rate r = rate_of(sr); return kFrame * r.down / r.up + 1; }

// w = np.hanning(258)[1:-1] = 0.5 + 0.5 cos(pi (2i - 255) / 257), into shared memory
__device__ __forceinline__ void stoi_window(double* w) {
  for (int i = threadIdx.x; i < kFrame; i += blockDim.x) w[i] = 0.5 + 0.5 * cospi((2 * i - 255) / 257.0);
  __syncthreads();
}

// rs[s][b][0 .. Lr_max): signal s (0 clean, 1 estimate) of clip b at 10 kHz, zero past its own resampled length
__global__ void __launch_bounds__(kThreads) stoi_resample_kernel(const float* __restrict__ clean,
                                                                 const float* __restrict__ est,
                                                                 const int* __restrict__ lens, int L_max, int Lr_max,
                                                                 const __grid_constant__ Resampler r,
                                                                 double* __restrict__ rs) {
  __shared__ double h[kMaxHalf + 1];
  for (int j = threadIdx.x; j <= r.half; j += blockDim.x) h[j] = r.h[j];
  __syncthreads();
  const int b = blockIdx.y, s = blockIdx.z, B = gridDim.y;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Lr_max) return;
  const float* x = (s ? est : clean) + (size_t)b * L_max;
  const int Lb = lens[b];
  double* out = rs + ((size_t)s * B + b) * Lr_max;
  if (n >= resampled_len(Lb, r.up, r.down)) {
    out[n] = 0.0;
    return;
  }
  // out[n] = sum_i x[i] * taps[n * down + half - i * up] over the taps j in [0, 2 half]
  const int64_t c = (int64_t)n * r.down + r.half;
  const int64_t lo = c - 2 * r.half;
  const int i_lo = lo <= 0 ? 0 : (int)((lo + r.up - 1) / r.up);
  const int i_hi = (int)(c / r.up) < Lb - 1 ? (int)(c / r.up) : Lb - 1;
  double acc = 0.0;
  for (int i = i_lo; i <= i_hi; ++i) {
    const int j = (int)(c - (int64_t)i * r.up);
    acc += (double)x[i] * h[j <= r.half ? j : 2 * r.half - j];
  }
  out[n] = acc;
}

// one CTA per clip: energy [b][f] (dB) of the clean frames, keep [b][f], idx [b][0 .. n_kept) the kept frames in order
__global__ void __launch_bounds__(kThreads) stoi_select_kernel(const double* __restrict__ rs, const int* __restrict__ lens,
                                                               int up, int down, int Lr_max, int nf_max,
                                                               double* __restrict__ energy, int* __restrict__ keep,
                                                               int* __restrict__ idx, int* __restrict__ n_kept) {
  __shared__ double w[kFrame];
  __shared__ double red[kThreads];
  __shared__ int scan[kThreads];
  stoi_window(w);
  const int b = blockIdx.x;
  const int nf = n_frames(resampled_len(lens[b], up, down));
  const double* x = rs + (size_t)b * Lr_max;
  double* e = energy + (size_t)b * nf_max;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int f = warp; f < nf; f += kThreads / 32) {
    double a = 0.0;
#pragma unroll
    for (int k = 0; k < kFrame / 32; ++k) {
      const int i = lane + 32 * k;
      const double v = w[i] * x[(size_t)f * kHop + i];
      a += v * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) e[f] = 20.0 * log10(sqrt(a) + kEps);
  }
  __syncthreads();
  double m = -INFINITY;
  for (int f = threadIdx.x; f < nf; f += kThreads) m = fmax(m, e[f]);
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  const double floor_db = red[0] - kDynRange;
  int total = 0;
  for (int base = 0; base < nf; base += kThreads) {  // exclusive scan of the keep flags, kThreads frames at a time
    const int f = base + threadIdx.x;
    const int k = f < nf && floor_db - e[f] < 0.0;
    if (f < nf) keep[(size_t)b * nf_max + f] = k;
    scan[threadIdx.x] = k;
    __syncthreads();
    for (int o = 1; o < kThreads; o <<= 1) {
      const int v = threadIdx.x >= o ? scan[threadIdx.x - o] : 0;
      __syncthreads();
      scan[threadIdx.x] += v;
      __syncthreads();
    }
    if (k) idx[(size_t)b * nf_max + total + scan[threadIdx.x] - 1] = f;
    total += scan[kThreads - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) n_kept[b] = total;
}

// cs[s][b][j] for j < (n_kept + 1) * hop: the first half of kept frame j / hop plus the second half of the one before,
// as pystoi's overlap-add; zero from there to Lr_max
__global__ void __launch_bounds__(kThreads) stoi_ola_kernel(const double* __restrict__ rs, const int* __restrict__ idx,
                                                            const int* __restrict__ n_kept, int Lr_max, int nf_max,
                                                            double* __restrict__ cs) {
  __shared__ double w[kFrame];
  stoi_window(w);
  const int b = blockIdx.y, s = blockIdx.z, B = gridDim.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= Lr_max) return;
  const double* x = rs + ((size_t)s * B + b) * Lr_max;
  const int* id = idx + (size_t)b * nf_max;
  const int nk = n_kept[b];
  const int k1 = j / kHop, r = j - k1 * kHop;
  double v = 0.0;
  if (k1 < nk) v = w[r] * x[(size_t)id[k1] * kHop + r];
  if (k1 >= 1 && k1 <= nk) v += w[r + kHop] * x[(size_t)id[k1 - 1] * kHop + r + kHop];
  cs[((size_t)s * B + b) * Lr_max + j] = v;
}

// bands[s][b][j][t] for the n_kept - 1 frames t of the compacted signal s of clip b, kFB frames per CTA
__global__ void __launch_bounds__(kThreads) stoi_bands_kernel(const double* __restrict__ cs, const int* __restrict__ n_kept,
                                                              int Lr_max, int nf_max, double* __restrict__ bands) {
  __shared__ double w[kFrame];
  __shared__ double xw[kFB][kFrame];
  __shared__ double2 tw[2 * kFrame];
  __shared__ double pw[kFB][kBins];
  const int b = blockIdx.y, s = blockIdx.z, B = gridDim.y;
  const int T = n_kept[b] - 1;
  const int t0 = blockIdx.x * kFB;
  if (t0 >= T) return;  // uniform over the CTA
  for (int m = threadIdx.x; m < 2 * kFrame; m += blockDim.x) {
    double sn, c;
    sincospi(m / (double)kFrame, &sn, &c);  // exp(-2 pi i m / 512) = c - i sn
    tw[m] = make_double2(c, sn);
  }
  stoi_window(w);
  const double* x = cs + ((size_t)s * B + b) * Lr_max;
  for (int i = threadIdx.x; i < kFB * kFrame; i += blockDim.x) {
    const int f = i / kFrame, n = i - f * kFrame;
    xw[f][n] = t0 + f < T ? w[n] * x[(size_t)(t0 + f) * kHop + n] : 0.0;
  }
  __syncthreads();
  if (threadIdx.x < kBins) {
    const int k = kBin0 + threadIdx.x;
    double re[kFB], im[kFB];
#pragma unroll
    for (int f = 0; f < kFB; ++f) re[f] = im[f] = 0.0;
    for (int n = 0; n < kFrame; ++n) {
      const double2 c = tw[(n * k) & (2 * kFrame - 1)];
#pragma unroll
      for (int f = 0; f < kFB; ++f) {
        re[f] += xw[f][n] * c.x;
        im[f] -= xw[f][n] * c.y;
      }
    }
#pragma unroll
    for (int f = 0; f < kFB; ++f) pw[f][threadIdx.x] = re[f] * re[f] + im[f] * im[f];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kFB * kBands; i += blockDim.x) {
    const int f = i / kBands, j = i - f * kBands;
    if (t0 + f >= T) continue;
    double a = 0.0;
    for (int q = kEdges[j]; q < kEdges[j + 1]; ++q) a += pw[f][q - kBin0];
    bands[(((size_t)s * B + b) * kBands + j) * nf_max + t0 + f] = sqrt(a);
  }
}

// one CTA per clip: the mean over J = T - 29 segments and 15 bands of the clipped, normalised correlations
__global__ void __launch_bounds__(kThreads) stoi_corr_kernel(const double* __restrict__ bands, const int* __restrict__ n_kept,
                                                             int nf_max, double clip, float* __restrict__ out) {
  __shared__ double sh[kThreads];
  const int b = blockIdx.x, B = gridDim.x;
  const int T = n_kept[b] - 1;
  if (T < kSeg) {  // pystoi warns and returns 1e-5
    if (threadIdx.x == 0) out[b] = 1e-5f;
    return;
  }
  const int J = T - kSeg + 1;
  double acc = 0.0;
  for (int it = threadIdx.x; it < J * kBands; it += kThreads) {
    const int m = it / kBands, j = it - m * kBands;
    const double* X = bands + ((size_t)b * kBands + j) * nf_max + m;
    const double* Y = bands + (((size_t)B + b) * kBands + j) * nf_max + m;
    double xx = 0.0, yy = 0.0;
    for (int i = 0; i < kSeg; ++i) { xx += X[i] * X[i]; yy += Y[i] * Y[i]; }
    const double alpha = sqrt(xx) / (sqrt(yy) + kEps);
    double sx = 0.0, sy = 0.0;
    for (int i = 0; i < kSeg; ++i) { sx += X[i]; sy += fmin(Y[i] * alpha, X[i] * clip); }
    const double mx = sx / kSeg, my = sy / kSeg;
    double cx = 0.0, cy = 0.0;
    for (int i = 0; i < kSeg; ++i) {
      const double u = X[i] - mx, v = fmin(Y[i] * alpha, X[i] * clip) - my;
      cx += u * u;
      cy += v * v;
    }
    const double nx = sqrt(cx) + kEps, ny = sqrt(cy) + kEps;
    double d = 0.0;
    for (int i = 0; i < kSeg; ++i) d += ((fmin(Y[i] * alpha, X[i] * clip) - my) / ny) * ((X[i] - mx) / nx);
    acc += d;
  }
  const double total = cta_tree_sum256(acc, sh);
  if (threadIdx.x == 0) out[b] = (float)(total / ((double)J * kBands));
}

// per-clip lengths into the device table through the kernel parameters (NULL: every clip L_max)
constexpr int kLenChunk = 1000;
struct StoiLens { int off, n; int v[kLenChunk]; };
__global__ void stoi_lengths_kernel(const __grid_constant__ StoiLens c, int* __restrict__ lens) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c.n) lens[c.off + i] = c.v[i];
}

struct StoiShape { int up, down, Lr_max, nf_max; };

struct StoiBufs {
  int* lens;
  double* rs;        // [2, B, Lr_max]
  double* energy;    // [B, nf_max]
  int* keep;         // [B, nf_max]
  int* idx;          // [B, nf_max]
  int* n_kept;       // [B]
  double* cs;        // [2, B, Lr_max]
  double* bands;     // [2, B, 15, nf_max]
};

// argument checks that need no data pointer
int stoi_shape(int B, int L_max, int sr, StoiShape& sh) {
  FSN_REQUIRE(B > 0, FSN_ERR_SHAPE, "stoi: B=%d clips", B);
  FSN_REQUIRE(B <= kMaxGridY, FSN_ERR_UNSUPPORTED, "stoi: B=%d clips, at most %d", B, kMaxGridY);
  FSN_REQUIRE(sr == 16000 || sr == 10000, FSN_ERR_UNSUPPORTED, "stoi: sample rate %d Hz; 16000 and 10000 are supported",
              sr);
  FSN_REQUIRE(L_max >= min_len(sr), FSN_ERR_SHAPE,
              "stoi: L_max=%d samples; at %d Hz a clip needs at least %d (one %d-sample frame at 10 kHz)", L_max, sr,
              min_len(sr), kFrame);
  const Rate r = rate_of(sr);
  sh.up = r.up;
  sh.down = r.down;
  sh.Lr_max = resampled_len(L_max, r.up, r.down);
  sh.nf_max = n_frames(sh.Lr_max);
  return FSN_OK;
}

void stoi_carve(Carver& c, int B, const StoiShape& sh, StoiBufs& w) {
  const size_t sig = (size_t)2 * B * sh.Lr_max, fr = (size_t)B * sh.nf_max;
  w.lens = c.take<int>(B);
  w.rs = c.take<double>(sig);
  w.energy = c.take<double>(fr);
  w.keep = c.take<int>(fr);
  w.idx = c.take<int>(fr);
  w.n_kept = c.take<int>(B);
  w.cs = c.take<double>(sig);
  w.bands = c.take<double>(fr * 2 * kBands);
}

int stoi_check(const float* clean, const float* est, const int32_t* lengths, int B, int L_max, int sr, const float* out,
               const void* workspace, size_t workspace_bytes, StoiShape& sh) {
  int rc = stoi_shape(B, L_max, sr, sh);
  if (rc) return rc;
  FSN_REQUIRE(clean && est && out, FSN_ERR_SHAPE, "stoi: null clean, estimate or out");
  if (lengths) {
    for (int b = 0; b < B; ++b)
      FSN_REQUIRE(lengths[b] >= min_len(sr) && lengths[b] <= L_max, FSN_ERR_SHAPE,
                  "stoi: clip %d has length %d, outside [%d, L_max = %d] (at %d Hz a clip needs at least %d samples for "
                  "one frame)",
                  b, lengths[b], min_len(sr), L_max, sr, min_len(sr));
  }
  Carver c(nullptr);
  StoiBufs w;
  stoi_carve(c, B, sh, w);
  FSN_REQUIRE(workspace && workspace_bytes >= c.off, FSN_ERR_WORKSPACE, "stoi: workspace of %zu bytes, %zu needed",
              workspace ? workspace_bytes : (size_t)0, c.off);
  return FSN_OK;
}

int stoi_run(const float* clean, const float* est, const int32_t* lengths, int B, int L_max, int sr, const StoiShape& sh,
             const StoiBufs& w, float* out, cudaStream_t st) {
  int longest = 0;
  StoiLens c;
  for (int off = 0; off < B; off += kLenChunk) {
    c.off = off;
    c.n = B - off < kLenChunk ? B - off : kLenChunk;
    for (int i = 0; i < c.n; ++i) {
      c.v[i] = lengths ? lengths[off + i] : L_max;
      longest = c.v[i] > longest ? c.v[i] : longest;
    }
    stoi_lengths_kernel<<<cdiv(c.n, kThreads), kThreads, 0, st>>>(c, w.lens);
    FSN_CHECK_LAUNCH("stoi_lengths_kernel");
  }
  const int T_most = n_frames(resampled_len(longest, sh.up, sh.down)) - 1;  // compacted frames of any clip, at most
  stoi_resample_kernel<<<dim3(cdiv(sh.Lr_max, kThreads), B, 2), kThreads, 0, st>>>(clean, est, w.lens, L_max, sh.Lr_max,
                                                                                   resampler(sr), w.rs);
  FSN_CHECK_LAUNCH("stoi_resample_kernel");
  stoi_select_kernel<<<B, kThreads, 0, st>>>(w.rs, w.lens, sh.up, sh.down, sh.Lr_max, sh.nf_max, w.energy, w.keep, w.idx,
                                             w.n_kept);
  FSN_CHECK_LAUNCH("stoi_select_kernel");
  stoi_ola_kernel<<<dim3(cdiv(sh.Lr_max, kThreads), B, 2), kThreads, 0, st>>>(w.rs, w.idx, w.n_kept, sh.Lr_max, sh.nf_max,
                                                                              w.cs);
  FSN_CHECK_LAUNCH("stoi_ola_kernel");
  if (T_most > 0) {
    stoi_bands_kernel<<<dim3(cdiv(T_most, kFB), B, 2), kThreads, 0, st>>>(w.cs, w.n_kept, sh.Lr_max, sh.nf_max, w.bands);
    FSN_CHECK_LAUNCH("stoi_bands_kernel");
  }
  const double clip = 1.0 + pow(10.0, 15.0 / 20.0);  // 1 + 10^(-BETA/20), BETA = -15 dB
  stoi_corr_kernel<<<B, kThreads, 0, st>>>(w.bands, w.n_kept, sh.nf_max, clip, out);
  FSN_CHECK_LAUNCH("stoi_corr_kernel");
  return FSN_OK;
}

}  // namespace
}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_stoi_workspace_bytes(int B, int L_max, int sr) {
  StoiShape sh;
  if (stoi_shape(B, L_max, sr, sh)) return 0;
  Carver c(nullptr);
  StoiBufs w;
  stoi_carve(c, B, sh, w);
  return c.off;
}

extern "C" int fsn_stoi(const float* clean, const float* estimate, const int32_t* lengths, int B, int L_max, int sr,
                        float* out, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  StoiShape sh;
  const int rc = stoi_check(clean, estimate, lengths, B, L_max, sr, out, workspace, workspace_bytes, sh);
  if (rc) return rc;
  Carver c(workspace);
  StoiBufs w;
  stoi_carve(c, B, sh, w);
  return stoi_run(clean, estimate, lengths, B, L_max, sr, sh, w, out, (cudaStream_t)stream);
}

extern "C" int fsn_debug_stoi_stages(const float* clean, const float* estimate, const int32_t* lengths, int B, int L_max,
                                     int sr, double* resampled, int32_t* keep, int32_t* n_kept, double* compacted,
                                     double* bands, float* out, void* workspace, size_t workspace_bytes,
                                     fsn_stream_t stream) {
  launch_counter() = 0;
  StoiShape sh;
  const int rc = stoi_check(clean, estimate, lengths, B, L_max, sr, out, workspace, workspace_bytes, sh);
  if (rc) return rc;
  FSN_REQUIRE(resampled && keep && n_kept && compacted && bands, FSN_ERR_SHAPE, "stoi hook: null stage buffer");
  Carver c(workspace);
  StoiBufs w;
  stoi_carve(c, B, sh, w);
  w.rs = resampled;
  w.keep = keep;
  w.n_kept = n_kept;
  w.cs = compacted;
  w.bands = bands;
  return stoi_run(clean, estimate, lengths, B, L_max, sr, sh, w, out, (cudaStream_t)stream);
}
