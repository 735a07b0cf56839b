// fullband_baseline (recipes/dns_interspeech_2020/fullband_baseline/model.py:8-68; SURVEY 8f rank 3):
// look-ahead pad -> norm -> num_layers x LSTM(F -> H) -> Linear(H -> 2F) [+ activation] -> [B,2,F,T].
// Host orchestration: the norm, the fp32 SequenceModel of fsn_fullband.cu (seq_stack_forward) and one re-layout kernel.
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
  float *magT, *inv1, *cum1, *y;
  float2 *fs, *sums;
  SeqStackWs seq;
  size_t bytes;
};

static int fbb_check(const fsn_fullband_desc* d, int B, int T) {
  FSN_REQUIRE(d && d->num_freqs > 1 && d->hidden > 0 && d->look_ahead >= 0, FSN_ERR_SHAPE, "fullband: bad descriptor");
  FSN_REQUIRE(d->num_layers >= 1 && d->num_layers <= SEQ_MAX_LAYERS, FSN_ERR_UNSUPPORTED, "fullband: 1..8 LSTM layers");
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "fullband: the GRU cell is not built");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "fullband: empty input (B=%d, T=%d)", B, T);
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE,
              FSN_ERR_UNSUPPORTED, "You must set up a type of Norm. (offline_laplace_norm / cumulative_laplace_norm are built)");
  return FSN_OK;
}

// num_layers x LSTM(F -> H) + Linear(H -> 2F), rows = clips, fp32 kernels
static SeqStack fbb_stack(const fsn_fullband_desc* d, int B, int T) {
  SeqStack s;
  memset(&s, 0, sizeof(s));
  s.R = B; s.Tp = T + d->look_ahead; s.K0 = d->num_freqs; s.n = d->num_layers; s.O = 2 * d->num_freqs; s.act = d->activation;
  for (int l = 0; l < s.n; ++l) s.H[l] = d->hidden;
  s.step_scale = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE;
  return s;
}

static void fbb_carve(const fsn_fullband_desc* d, int B, int T, void* base, FbbWs& w) {
  Carver c(base);
  const size_t Tp = (size_t)T + d->look_ahead, F = d->num_freqs;
  w.magT = c.take<float>(B * Tp * F);
  w.fs = c.take<float2>(B * Tp);
  w.sums = c.take<float2>(B);
  w.inv1 = c.take<float>(B);
  w.cum1 = c.take<float>(B * Tp);
  seq_stack_carve(c, fbb_stack(d, B, T), w.seq);
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
  const int F = d->num_freqs, Tp = T + d->look_ahead;
  const bool cum = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE;
  if ((rc = transpose_mag_launch(noisy_mag, w.magT, B, F, T, Tp, st))) return rc;
  if ((rc = clip_stats_launch(w.magT, B, Tp, F, 0, w.fs, w.sums, st))) return rc;
  if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)F * Tp, 1.f, w.inv1, nullptr, st))) return rc;
  if (cum && (rc = cum_clip_scale_launch(w.fs, B, Tp, F, 1.1920928955078125e-07f, w.cum1, st))) return rc;
  SeqStack s = fbb_stack(d, B, T);
  for (int l = 0; l < s.n; ++l) s.L[l] = layers[l];
  s.x = w.magT; s.scale = cum ? w.cum1 : w.inv1; s.fc_w = fc_w; s.fc_b = fc_b; s.out = w.y;
  if ((rc = seq_stack_forward(s, w.seq, st))) return rc;
  const size_t n = (size_t)B * 2 * F * T;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  fbb_output_kernel<<<blocks, 256, 0, st>>>(w.y, out, B, F, T, Tp, d->look_ahead);
  FSN_CHECK_LAUNCH("fbb_output_kernel");
  return FSN_OK;
}
