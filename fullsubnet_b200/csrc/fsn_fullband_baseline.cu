// fullband_baseline (recipes/dns_interspeech_2020/fullband_baseline/model.py:8-68; SURVEY 8f rank 3):
// look-ahead pad -> norm -> num_layers x LSTM(F -> H) -> Linear(H -> 2F) [+ activation] -> [B,2,F,T].
// Host orchestration of the shared fp32 kernels: layers 0-1 on the persistent wavefront kernel when it fits,
// remaining layers on the per-step kernel, one GEMM for the Linear layer, one re-layout kernel.
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

// y [B, Tp, 2F] (row = clip-major, time) -> out [B, 2, F, T] dropping the first `la` steps (model.py:58-62)
__global__ void fbb_output_kernel(const float* __restrict__ y, float* __restrict__ out, int B, int F, int T, int Tp,
                                  int la) {
  const size_t n = (size_t)B * 2 * F * T;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    size_t q = i / T;
    const int f = (int)(q % F); q /= F;
    const int c = (int)(q & 1);
    const size_t b = q >> 1;
    out[i] = y[((b * Tp) + t + la) * (size_t)(2 * F) + (size_t)c * F + f];
  }
}

struct FbbWs {
  float *magT, *inv1, *cum1, *seq[2], *c, *pp, *y;
  float2 *fs, *sums;
  unsigned int* barrier;
  size_t bytes;
};

static int fbb_check(const fsn_fullband_desc* d, int B, int T) {
  FSN_REQUIRE(d && d->num_freqs > 1 && d->hidden > 0 && d->look_ahead >= 0, FSN_ERR_SHAPE, "fullband: bad descriptor");
  FSN_REQUIRE(d->num_layers >= 1 && d->num_layers <= 8, FSN_ERR_UNSUPPORTED, "fullband: 1..8 LSTM layers");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "fullband: empty input (B=%d, T=%d)", B, T);
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE,
              FSN_ERR_UNSUPPORTED, "You must set up a type of Norm. (offline_laplace_norm / cumulative_laplace_norm are built)");
  return FSN_OK;
}

static void fbb_carve(const fsn_fullband_desc* d, int B, int T, void* base, FbbWs& w) {
  Carver c(base);
  const size_t Tp = (size_t)T + d->look_ahead, F = d->num_freqs, H = d->hidden;
  w.magT = c.take<float>(B * Tp * F);
  w.fs = c.take<float2>(B * Tp);
  w.sums = c.take<float2>(B);
  w.inv1 = c.take<float>(B);
  w.cum1 = c.take<float>(B * Tp);
  w.seq[0] = c.take<float>(B * Tp * H);
  w.seq[1] = c.take<float>(B * Tp * H);
  w.c = c.take<float>((size_t)B * H);
  w.pp = c.take<float>((size_t)2 * 256 * H);
  w.barrier = c.take<unsigned int>(64);
  w.y = c.take<float>(B * Tp * 2 * F);
  w.bytes = c.off;
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_fullband_workspace_bytes(const fsn_fullband_desc* d, int B, int T) {
  if (fbb_check(d, B, T)) return 0;
  FbbWs w;
  fbb_carve(d, B, T, nullptr, w);
  return w.bytes;
}

extern "C" int fsn_fullband_forward(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                                    const float* fc_b, const float* noisy_mag, int B, int T, float* out,
                                    void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  int rc = fbb_check(d, B, T);
  if (rc) return rc;
  FbbWs w;
  fbb_carve(d, B, T, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int F = d->num_freqs, H = d->hidden, Tp = T + d->look_ahead, NL = d->num_layers;
  const bool cum = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE;
  if ((rc = transpose_mag_launch(noisy_mag, w.magT, B, F, T, Tp, st))) return rc;
  if ((rc = clip_stats_launch(w.magT, B, Tp, F, 0, w.fs, w.sums, st))) return rc;
  if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)F * Tp, 1.f, w.inv1, nullptr, st))) return rc;
  if (cum && (rc = cum_clip_scale_launch(w.fs, B, Tp, F, 1.1920928955078125e-07f, w.cum1, st))) return rc;

  int first = 0;  // first layer still to run on the per-step kernel
  int cur = 0;    // w.seq[cur] receives the output of the layer being computed
  if (NL >= 2 && !cum && fb_persistent_supported(F, H, H)) {
    fsn_seq_weights two;
    memset(&two, 0, sizeof(two));
    for (int l = 0; l < 2; ++l) {
      two.w_ih[l] = layers[l].w_ih; two.w_hh[l] = layers[l].w_hh; two.b_ih[l] = layers[l].b_ih; two.b_hh[l] = layers[l].b_hh;
    }
    for (int b0 = 0; b0 < B; b0 += 256) {
      const int nb = (B - b0 < 256) ? B - b0 : 256;
      if ((rc = fb_persistent_launch(&two, w.magT + (size_t)b0 * Tp * F, w.inv1 + b0, w.pp,
                                     w.seq[0] + (size_t)b0 * Tp * H, w.barrier, nb, F, H, H, Tp, st)))
        return rc;
    }
    first = 2;
    cur = 1;
  }
  for (int l = first; l < NL; ++l) {
    const float* prev = w.seq[cur ^ 1];  // output sequence of layer l-1, [B, Tp, H]
    float* seq = w.seq[cur];
    for (int t = 0; t < Tp; ++t) {
      StepParams p;
      memset(&p, 0, sizeof(p));
      p.R = B; p.H = H; p.first = (t == 0);
      p.w_ih = layers[l].w_ih; p.w_hh = layers[l].w_hh; p.b_ih = layers[l].b_ih; p.b_hh = layers[l].b_hh;
      if (l == 0) {
        p.K0 = F;
        p.x0 = w.magT + (size_t)t * F; p.x0_row_stride = (size_t)Tp * F;
        p.row_scale = cum ? w.cum1 + (size_t)t * B : w.inv1;
      } else {
        p.K0 = H;
        p.x0 = prev + (size_t)t * H; p.x0_row_stride = (size_t)Tp * H;
      }
      p.h_prev = seq + (size_t)(t > 0 ? t - 1 : 0) * H; p.h_prev_stride = (size_t)Tp * H;
      p.h_out = seq + (size_t)t * H; p.h_out_stride = (size_t)Tp * H;
      p.c = w.c;
      if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
    }
    cur ^= 1;
  }
  const float* last = w.seq[cur ^ 1];
  if ((rc = fc_gemm_launch(last, fc_w, fc_b, w.y, B * Tp, H, 2 * F, d->activation, st))) return rc;
  const size_t n = (size_t)B * 2 * F * T;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  fbb_output_kernel<<<blocks, 256, 0, st>>>(w.y, out, B, F, T, Tp, d->look_ahead);
  FSN_CHECK_LAUNCH("fbb_output_kernel");
  return FSN_OK;
}
