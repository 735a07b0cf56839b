// Band-limited resampling of a batch of clips with per-clip lengths: the windowed sinc of Inferencer.resample
// (fullsubnet_b200/inferencer.py) applied to each clip, every weight and product in float64 as the host computes them.
//
// One thread per output sample n of clip b (grid: runs of kThreads outputs x clips).  The thread forms the host's
// t = n * down / up, then, for the 2 * half taps idx = floor(t) + k in ascending k, the weight
//   w = cutoff * sinc(cutoff * d) * (0.5 + 0.5 * cos(pi * clip(d / half, -1, 1))),  d = t - idx,
// with numpy's sinc, multiplies it by the (widened) input sample, 0 outside [0, N_b), and adds the product to a float64
// sum that is rounded once to float32.  Products and sums go through __dmul_rn / __dadd_rn so that no multiply-add is
// contracted into an FMA the host does not perform.  The weights are computed per output rather than read from a
// polyphase table: the host rounds t for every output, so outputs of one phase get weights that differ in the last bits,
// and only the per-output computation reproduces them.  sin / cos are CUDA's (within 2 ulp of the host's libm), which is
// why a float32 output can differ from the host's by one rounding step (DESIGN 4.10.1).
#include <math.h>

#include "fsn_internal.cuh"

namespace fsn {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxBatch = 65535;     // clips ride on grid.y
constexpr int kMaxHalf = 1 << 29;    // 2 * half taps must fit an int

struct Filter {
  int up, down, half;
  double cutoff;
};

// ceil(N * up / down) in integers: the host's float64 ceiling for N * up < 2^53
__host__ __device__ inline int64_t out_len(int N, int up, int down) {
  return ((int64_t)N * up + down - 1) / down;
}

// y[b, n] for n < N_out_max: the resampled clip for n < out_len(N_b), 0 from there on
__global__ void __launch_bounds__(kThreads) resample_kernel(const float* __restrict__ x, const int* __restrict__ lens,
                                                            int N_max, const Filter f, float* __restrict__ y,
                                                            int N_out_max) {
  const int b = blockIdx.y;
  const int n = blockIdx.x * kThreads + threadIdx.x;
  if (n >= N_out_max) return;
  const int Nb = lens ? lens[b] : N_max;
  const float* xb = x + (size_t)b * N_max;
  float* out = y + (size_t)b * N_out_max + n;
  if (n >= out_len(Nb, f.up, f.down)) {
    *out = 0.f;
    return;
  }
  if (f.up == f.down) {  // same rate: a copy
    *out = xb[n];
    return;
  }
  const double pi = 3.141592653589793;  // np.pi
  const double t = (double)n * (double)f.down / (double)f.up;
  const int64_t base = (int64_t)floor(t);
  const double half = (double)f.half;
  double acc = -0.0;  // the sum of the products alone, signed zeros included
  for (int k = -f.half + 1; k <= f.half; ++k) {
    const int64_t idx = base + k;
    const double d = t - (double)idx;
    const double xs = f.cutoff * d;
    const double ys = pi * (xs == 0.0 ? 1.0e-20 : xs);  // np.sinc: sin(pi x) / (pi x), x = 0 -> 1e-20
    const double sinc = sin(ys) / ys;
    const double win = __dadd_rn(0.5, __dmul_rn(0.5, cos(pi * fmin(fmax(d / half, -1.0), 1.0))));
    const double w = f.cutoff * sinc * win;
    const double v = (idx >= 0 && idx < Nb) ? (double)xb[idx] : 0.0;
    acc = __dadd_rn(acc, __dmul_rn(v, w));
  }
  *out = (float)acc;
}

// every check of fsn_resample_workspace_bytes: the filter of (sr_in, sr_out, zeros) and the batch limit
int resample_filter(int B, int N_max, int sr_in, int sr_out, int zeros, Filter& f) {
  FSN_REQUIRE(B > 0, FSN_ERR_SHAPE, "resample: B=%d clips", B);
  FSN_REQUIRE(B <= kMaxBatch, FSN_ERR_UNSUPPORTED, "resample: B=%d clips, at most %d", B, kMaxBatch);
  FSN_REQUIRE(N_max > 0, FSN_ERR_SHAPE, "resample: N_max=%d samples", N_max);
  FSN_REQUIRE(sr_in > 0 && sr_out > 0, FSN_ERR_SHAPE, "resample: sample rates %d -> %d Hz; both must be positive", sr_in,
              sr_out);
  FSN_REQUIRE(zeros >= 1, FSN_ERR_SHAPE, "resample: zeros=%d, at least 1", zeros);
  int a = sr_in, c = sr_out;
  while (c) { const int r = a % c; a = c; c = r; }
  f.up = sr_out / a;
  f.down = sr_in / a;
  f.cutoff = fmin(1.0, (double)f.up / (double)f.down);
  const double half = ceil((double)zeros / f.cutoff);
  FSN_REQUIRE(half <= kMaxHalf, FSN_ERR_UNSUPPORTED,
              "resample: %d -> %d Hz with zeros=%d needs a filter half-length of %.0f taps, at most %d", sr_in, sr_out,
              zeros, half, kMaxHalf);
  f.half = (int)half;
  return FSN_OK;
}

size_t resample_workspace(int B) {
  Carver c(nullptr);
  c.take<int>(B);
  return c.off;
}

}  // namespace
}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_resample_workspace_bytes(int B, int N_max, int sr_in, int sr_out, int zeros) {
  Filter f;
  if (resample_filter(B, N_max, sr_in, sr_out, zeros, f)) return 0;
  return resample_workspace(B);
}

extern "C" int fsn_resample(const float* x, const int32_t* lengths, int B, int N_max, int sr_in, int sr_out, int zeros,
                            float* y, int N_out_max, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  Filter f;
  int rc = resample_filter(B, N_max, sr_in, sr_out, zeros, f);
  if (rc) return rc;
  FSN_REQUIRE(x && y, FSN_ERR_SHAPE, "resample: null input or output");
  int longest = N_max;
  if (lengths) {
    longest = 0;
    for (int b = 0; b < B; ++b) {
      FSN_REQUIRE(lengths[b] >= 1 && lengths[b] <= N_max, FSN_ERR_SHAPE,
                  "resample: clip %d has length %d, outside [1, N_max = %d]", b, lengths[b], N_max);
      longest = lengths[b] > longest ? lengths[b] : longest;
    }
  }
  const int64_t need = out_len(longest, f.up, f.down);
  FSN_REQUIRE(N_out_max >= need, FSN_ERR_SHAPE,
              "resample: N_out_max=%d, but a %d-sample clip at %d Hz gives %lld samples at %d Hz", N_out_max, longest,
              sr_in, (long long)need, sr_out);
  const size_t ws = resample_workspace(B);
  FSN_REQUIRE(workspace && workspace_bytes >= ws, FSN_ERR_WORKSPACE, "resample: workspace of %zu bytes, %zu needed",
              workspace ? workspace_bytes : (size_t)0, ws);
  const cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace);
  WavWs w = {nullptr, nullptr, nullptr, nullptr, c.take<int>(B)};
  if ((rc = wav_prologue(lengths, B, w, st))) return rc;
  resample_kernel<<<dim3((N_out_max - 1) / kThreads + 1, B), kThreads, 0, st>>>(x, w.lens, N_max, f, y, N_out_max);
  FSN_CHECK_LAUNCH("resample_kernel");
  return FSN_OK;
}
