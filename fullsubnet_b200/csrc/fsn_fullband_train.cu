// Training step of fullband_baseline (recipes/dns_interspeech_2020/fullband_baseline/trainer.py:32-71, model.py:46-68):
//   fsn_fullband_train_forward   Model.forward with gradients enabled, keeping what back-propagation through time needs
//   fsn_fullband_train_backward  output re-layout + act' -> Linear(2F) -> BPTT of the N-layer stack (stack_bwd) ->
//                                weight gradients of every LSTM layer through layer_weight_grads (fsn_train.cu)
// Everything is time-major ([Tp, B, .]) like fsn_train.cu: the input preparation, the activation-saving LSTM forward, the
// per-step backward and the weight-gradient GEMMs are the ones of the fullsubnet step.  The normalised input has no
// parameter behind it, so the norm needs no backward.  Every reduction runs in a fixed order: two runs give identical bits.
// oracle/fullband_baseline_oracle.py:fbb_forward under CPU autograd is the reference.
#include "fsn_internal.cuh"

namespace fsn {

static const int FBB_MAX_LAYERS = 8;

struct FbbTrainWs {
  float *raw, *xfb, *inv1, *cum1, *y;
  float2 *sums, *fs;
  LayerSave L[FBB_MAX_LAYERS];
  float *dY, *dH;
  float *dh_rec[FBB_MAX_LAYERS], *dc[FBB_MAX_LAYERS], *dh_mid[2];
  float *splitk, *colsum, *gT, *xT, *rec;
  size_t colsum_floats;
  float *whhT[FBB_MAX_LAYERS], *wihT[FBB_MAX_LAYERS];  // FSN_PREC_TF32_TC: transposed weights
  __half *h16[FBB_MAX_LAYERS], *w16;                   // fp16 MMA operands of the forward step kernel
  size_t bytes;
};

static int fbb_in_width(const fsn_fullband_desc* d, int l) { return l == 0 ? d->num_freqs : d->hidden; }

static void carve_fbb_train(const fsn_fullband_desc* d, int B, int T, void* base, FbbTrainWs& w) {
  Carver c(base);
  const size_t Tp = (size_t)T + d->look_ahead, F = d->num_freqs, H = d->hidden, NL = d->num_layers;
  const size_t rows = Tp * B, K0max = F > H ? F : H;
  w.raw = c.take<float>(rows * F);
  w.xfb = c.take<float>(rows * F);
  w.inv1 = c.take<float>(B);
  w.sums = c.take<float2>(B);
  w.fs = nullptr; w.cum1 = nullptr;
  if (norm_per_step(d->norm_type)) {
    w.fs = c.take<float2>(rows);
    w.cum1 = c.take<float>(rows);
  }
  for (size_t l = 0; l < NL; ++l) {
    w.L[l].G = c.take<float>(rows * 4 * H); w.L[l].C = c.take<float>(rows * H); w.L[l].H = c.take<float>(rows * H);
  }
  w.y = c.take<float>(rows * 2 * F);
  w.dY = c.take<float>(rows * 2 * F);
  w.dH = c.take<float>(rows * H);
  for (size_t l = 0; l < NL; ++l) { w.dh_rec[l] = c.take<float>((size_t)B * H); w.dc[l] = c.take<float>((size_t)B * H); }
  w.dh_mid[0] = c.take<float>((size_t)B * H);
  w.dh_mid[1] = NL > 2 ? c.take<float>((size_t)B * H) : nullptr;
  w.splitk = c.take<float>(SPLITK_SCRATCH_FLOATS);
  w.colsum_floats = (size_t)COLSUM_MAX_S * (4 * H > 2 * F ? 4 * H : 2 * F);
  w.colsum = c.take<float>(w.colsum_floats);
  w.gT = w.xT = w.rec = nullptr;
  w.w16 = nullptr;
  for (int l = 0; l < FBB_MAX_LAYERS; ++l) { w.whhT[l] = w.wihT[l] = nullptr; w.h16[l] = nullptr; }
  if (tf32_layer(d->precision, d->hidden)) {
    for (size_t l = 0; l < NL; ++l) {
      w.whhT[l] = c.take<float>(H * 4 * H);
      if (l > 0) w.wihT[l] = c.take<float>(H * 4 * H);  // layer 0 computes no dx
      w.h16[l] = c.take<__half>(rows * H);
    }
    w.gT = c.take<float>(tgemm_blocked_floats(rows, 4 * (int)H));
    w.xT = c.take<float>(tgemm_blocked_floats(rows, (int)K0max));
    w.rec = c.take<float>(4 * (size_t)B * H);
    w.w16 = c.take<__half>(4 * H * (H + K0max));
  }
  w.bytes = c.off;
}

static int fbb_train_check(const fsn_fullband_desc* d, int B, int T) {
  FSN_REQUIRE(d && d->num_freqs > 1 && d->hidden > 0 && d->look_ahead >= 0 && d->activation >= FSN_ACT_NONE &&
                  d->activation <= FSN_ACT_RELU6,
              FSN_ERR_SHAPE, "fullband training: bad descriptor");
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "fullband training: the GRU cell is not built");
  FSN_REQUIRE(d->precision == FSN_PREC_FP32 || d->precision == FSN_PREC_TF32_TC, FSN_ERR_UNSUPPORTED,
              "fullband training: precision must be fp32 or tf32_tc");
  FSN_REQUIRE(d->num_layers >= 1 && d->num_layers <= FBB_MAX_LAYERS, FSN_ERR_UNSUPPORTED, "fullband training: 1..8 LSTM layers");
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE ||
                  d->norm_type == FSN_NORM_FORGETTING,
              FSN_ERR_UNSUPPORTED,
              "fullband training: offline_laplace_norm and cumulative_laplace_norm are built");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "fullband training: empty input (B=%d, T=%d)", B, T);
  return FSN_OK;
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_fullband_train_workspace_bytes(const fsn_fullband_desc* d, int B, int T) {
  if (fbb_train_check(d, B, T)) return 0;
  FbbTrainWs w;
  carve_fbb_train(d, B, T, nullptr, w);
  return w.bytes;
}

extern "C" int fsn_fullband_train_forward(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                                          const float* fc_b, const float* noisy_mag, int B, int T, float* out,
                                          void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  int rc = fbb_train_check(d, B, T);
  if (rc) return rc;
  if ((rc = layout_clips_check(B, true, "fullband training"))) return rc;
  FSN_REQUIRE(layers && fc_w && fc_b && noisy_mag && out, FSN_ERR_SHAPE, "fullband training: null argument");
  FbbTrainWs w;
  carve_fbb_train(d, B, T, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int F = d->num_freqs, H = d->hidden, Tp = T + d->look_ahead, NL = d->num_layers;
  // look-ahead pad, norm and the time-major copies (model.py:50-56)
  if ((rc = train_input_launch(noisy_mag, B, F, T, Tp, 0, d->norm_type, w.sums, w.inv1, w.raw,
                               w.xfb, w.fs, w.cum1, st)))
    return rc;
  // num_layers x LSTM (model.py:57); on tf32_tc layer l's fp16 hidden states are layer l+1's fp16 input
  for (int l = 0; l < NL; ++l) {
    const LayerHalf half{w.h16[l], l > 0 ? w.h16[l - 1] : nullptr, w.w16};
    if ((rc = layer_forward(d->precision, layers[l], l == 0 ? w.xfb : w.L[l - 1].H, B, fbb_in_width(d, l), H, Tp, w.L[l], w.rec,
                            w.splitk, &half, st)))
      return rc;
  }
  // Linear(H -> 2F) + activation into y, kept for act' (model.py:58-62), then [B,2,F,T] without the look-ahead frames
  if ((rc = fc_gemm_launch(w.L[NL - 1].H, fc_w, fc_b, w.y, Tp * B, H, 2 * F, d->activation, st))) return rc;
  return crm_output_launch(w.y, 2 * F, (size_t)B * 2 * F, B, Tp, F, d->look_ahead, out, st);
}

extern "C" int fsn_fullband_train_backward(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                                           const float* fc_b, const float* dout, int B, int T, const fsn_fullband_grads* g,
                                           void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  int rc = fbb_train_check(d, B, T);
  if (rc) return rc;
  FSN_REQUIRE(layers && fc_w && fc_b && dout && g, FSN_ERR_SHAPE, "fullband training: null argument");
  FbbTrainWs w;
  carve_fbb_train(d, B, T, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int F = d->num_freqs, H = d->hidden, Tp = T + d->look_ahead, NL = d->num_layers;
  LayerBwd L[FBB_MAX_LAYERS];
  for (int l = 0; l < NL; ++l) {
    L[l] = LayerBwd{layers[l].w_ih, layers[l].w_hh, w.L[l], B, fbb_in_width(d, l), H, w.dh_rec[l], w.dc[l], w.whhT[l], w.wihT[l],
                    w.splitk};
    if ((rc = layer_bwd_transpose_weights(L[l], st))) return rc;
  }
  // ---- output re-layout + act', Linear(2F)
  if ((rc = train_dy_launch(dout, w.y, d->activation, B, F, T, Tp, d->look_ahead, w.dY, st))) return rc;
  if ((rc = linear_bwd(w.dY, w.L[NL - 1].H, fc_w, Tp * B, 2 * F, H, g->fc_w, g->fc_b, w.dH, w.splitk, w.colsum, w.colsum_floats, st)))
    return rc;
  // ---- BPTT of the stack from the top, one step at a time (the input is the normalised spectrogram: no dx)
  if ((rc = stack_bwd(L, NL, Tp, w.dH, nullptr, nullptr, 0, w.dh_mid[0], w.dh_mid[1], nullptr, st))) return rc;
  // ---- weight gradients: layer 0 reads the normalised input, layer l the hidden states of layer l-1
  const WgradScratch wg{w.gT, w.xT, w.splitk, w.colsum, w.colsum_floats};
  for (int l = NL - 1; l >= 0; --l) {
    const fsn_lstm_grads& q = g->layer[l];
    if ((rc = layer_weight_grads(L[l], Tp, l == 0 ? w.xfb : w.L[l - 1].H, q.w_ih, q.w_hh, q.b_ih, q.b_hh, wg, st))) return rc;
  }
  return FSN_OK;
}
