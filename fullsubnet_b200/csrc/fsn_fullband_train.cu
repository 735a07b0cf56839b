// Training step of fullband_baseline (recipes/dns_interspeech_2020/fullband_baseline/trainer.py:32-71, model.py:46-68):
//   fsn_fullband_train_forward   Model.forward with gradients enabled, keeping what back-propagation through time needs
//   fsn_fullband_train_backward  output re-layout + act' -> Linear(2F) -> BPTT of the N-layer stack (stack_bwd) ->
//                                weight gradients of every LSTM layer through layer_weight_grads (fsn_train.cu)
// Everything is time-major ([Tp, B, .]) like fsn_train.cu: the input preparation, the activation-saving LSTM forward, the
// per-step backward and the weight-gradient GEMMs are the ones of the fullsubnet step.  The normalised input has no
// parameter behind it, so the norm needs no backward.  Every reduction runs in a fixed order: two runs give identical bits.
// oracle/fullband_baseline_oracle.py:fbb_forward under CPU autograd is the reference.
#include <string.h>

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
  float *whhT[FBB_MAX_LAYERS], *wihT[FBB_MAX_LAYERS];  // FSN_PREC_TF32_TC: transposed weights
  __half *h16[FBB_MAX_LAYERS], *w16;                   // fp16 MMA operands of the forward step kernel
  size_t bytes;
};

struct FbbCarver {
  char* base; size_t off;
  explicit FbbCarver(void* p) : base((char*)p), off(0) {}
  template <class T> T* take(size_t n) {
    T* r = base ? (T*)(base + off) : nullptr;
    off = align_up(off + n * sizeof(T), 256);
    return r;
  }
};

// the same per-layer choice as fsn_train_* / fsn_fast_train_*
static bool fbb_tc(const fsn_fullband_desc* d) { return d->precision == FSN_PREC_TF32_TC && (d->hidden & 3) == 0; }

static int fbb_in_width(const fsn_fullband_desc* d, int l) { return l == 0 ? d->num_freqs : d->hidden; }

static void carve_fbb_train(const fsn_fullband_desc* d, int B, int T, void* base, FbbTrainWs& w) {
  FbbCarver c(base);
  const size_t Tp = (size_t)T + d->look_ahead, F = d->num_freqs, H = d->hidden, NL = d->num_layers;
  const size_t rows = Tp * B, K0max = F > H ? F : H;
  w.raw = c.take<float>(rows * F);
  w.xfb = c.take<float>(rows * F);
  w.inv1 = c.take<float>(B);
  w.sums = c.take<float2>(B);
  w.fs = nullptr; w.cum1 = nullptr;
  if (d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE) {
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
  w.colsum = c.take<float>((size_t)COLSUM_MAX_S * (4 * H > 2 * F ? 4 * H : 2 * F));
  w.gT = w.xT = w.rec = nullptr;
  w.w16 = nullptr;
  for (int l = 0; l < FBB_MAX_LAYERS; ++l) { w.whhT[l] = w.wihT[l] = nullptr; w.h16[l] = nullptr; }
  if (fbb_tc(d)) {
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
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE, FSN_ERR_UNSUPPORTED,
              "fullband training: offline_laplace_norm and cumulative_laplace_norm are built");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "fullband training: empty input (B=%d, T=%d)", B, T);
  return FSN_OK;
}

static LayerBwd fbb_layer_bwd(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const FbbTrainWs& w, int B, int l) {
  const bool tc = fbb_tc(d);
  return LayerBwd{layers[l].w_ih, layers[l].w_hh, w.L[l], B, fbb_in_width(d, l), d->hidden, w.dh_rec[l], w.dc[l],
                  tc ? w.whhT[l] : nullptr, tc ? w.wihT[l] : nullptr, w.splitk};
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
  FSN_REQUIRE(layers && fc_w && fc_b && noisy_mag && out, FSN_ERR_SHAPE, "fullband training: null argument");
  FbbTrainWs w;
  carve_fbb_train(d, B, T, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int F = d->num_freqs, H = d->hidden, Tp = T + d->look_ahead, NL = d->num_layers;
  // look-ahead pad, norm and the time-major copies (model.py:50-56)
  if ((rc = train_input_launch(noisy_mag, B, F, T, Tp, 0, d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE, w.sums, w.inv1, w.raw,
                               w.xfb, w.fs, w.cum1, st)))
    return rc;
  // num_layers x LSTM (model.py:57); on tf32_tc layer l's fp16 hidden states are layer l+1's fp16 input
  const bool tc = fbb_tc(d);
  for (int l = 0; l < NL; ++l) {
    fsn_seq_weights sw;
    memset(&sw, 0, sizeof(sw));
    sw.w_ih[0] = layers[l].w_ih; sw.w_hh[0] = layers[l].w_hh; sw.b_ih[0] = layers[l].b_ih; sw.b_hh[0] = layers[l].b_hh;
    const float* X = l == 0 ? w.xfb : w.L[l - 1].H;
    const int K0 = fbb_in_width(d, l);
    if (tc) {
      const LayerHalf half{w.h16[l], l > 0 ? w.h16[l - 1] : nullptr, w.w16};
      rc = layer_forward_save_tc(&sw, 0, X, B, K0, H, Tp, w.L[l], w.rec, st, w.splitk, SPLITK_SCRATCH_FLOATS, &half);
    } else {
      rc = layer_forward_save(&sw, 0, X, B, K0, H, Tp, w.L[l], st);
    }
    if (rc) return rc;
  }
  // Linear(H -> 2F) + activation into y, kept for act' (model.py:58-62), then [B,2,F,T] without the look-ahead frames
  if ((rc = fc_gemm_launch(w.L[NL - 1].H, fc_w, fc_b, w.y, Tp * B, H, 2 * F, d->activation, st))) return rc;
  return train_output_launch(w.y, B, Tp, F, d->look_ahead, out, st);
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
  if (fbb_tc(d)) {
    for (int l = 0; l < NL; ++l) {
      if ((rc = transpose_launch(layers[l].w_hh, (size_t)4 * H, H, w.whhT[l], st))) return rc;
      if (l > 0 && (rc = transpose_launch(layers[l].w_ih, (size_t)4 * H, H, w.wihT[l], st))) return rc;
    }
  }
  // ---- output re-layout + act', Linear(2F): dW = dY^T H, db = colsum dY, dH = dY W
  const float* Htop = w.L[NL - 1].H;
  if ((rc = train_dy_launch(dout, w.y, d->activation, B, F, T, Tp, d->look_ahead, w.dY, st))) return rc;
  if ((rc = sgemm_launch(true, w.dY, 2 * F, Htop, H, g->fc_w, H, 2 * F, H, Tp * B, false, w.splitk, st))) return rc;
  if ((rc = colsum_launch(w.dY, (size_t)Tp * B, 2 * F, 2 * F, g->fc_b, nullptr, w.colsum, st))) return rc;
  if ((rc = sgemm_launch(false, w.dY, 2 * F, fc_w, H, w.dH, H, Tp * B, H, 2 * F, false, nullptr, st))) return rc;
  // ---- BPTT of the stack from the top, one step at a time (the input is the normalised spectrogram: no dx)
  LayerBwd L[FBB_MAX_LAYERS];
  for (int l = 0; l < NL; ++l) L[l] = fbb_layer_bwd(d, layers, w, B, l);
  if ((rc = stack_bwd(L, NL, Tp, w.dH, nullptr, nullptr, 0, w.dh_mid[0], w.dh_mid[1], nullptr, st))) return rc;
  // ---- weight gradients: layer 0 reads the normalised input, layer l the hidden states of layer l-1
  const WgradScratch wg{w.gT, w.xT, w.splitk, w.colsum};
  for (int l = NL - 1; l >= 0; --l) {
    const fsn_lstm_grads& q = g->layer[l];
    if ((rc = layer_weight_grads(L[l], Tp, l == 0 ? w.xfb : w.L[l - 1].H, q.w_ih, q.w_hh, q.b_ih, q.b_hh, wg, st))) return rc;
  }
  return FSN_OK;
}
