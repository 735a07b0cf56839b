// Training step of fast_fullsubnet (recipes/dns_interspeech_2020/fast_fullsubnet/trainer.py:45-56, model.py:143-202):
//   fsn_fast_train_forward   Model.forward in train mode, keeping what back-propagation through time needs
//   fsn_fast_train_backward  Linear(2F) -> decoder BPTT -> up-sampling transpose -> ReLU' -> bottleneck BPTT -> second
//                            norm + down-sampling + unfold (closed form, gather; cumulative norm: per-row suffix sums
//                            over the shrunk steps) -> ReLU' -> Linear(M) -> encoder BPTT;
//                            weight gradients of every LSTM layer through layer_weight_grads (fsn_train.cu)
// Everything is time-major ([Tp, rows, .], the bottleneck [Ts, B*M, .]) like fsn_train.cu, so the LSTM layers reuse its
// activation-saving forward, its per-step backward and its weight-gradient GEMMs.  Every reduction runs in a fixed order:
// two runs give identical bits.  oracle/fast_fullsubnet_oracle.py:fast_model_forward under CPU autograd is the reference.
#include "fsn_internal.cuh"

namespace fsn {

// ------------------------------------------------------------------------------------------ backward kernels
// transpose of the up-sampling (frame t <- shrunk step min(t/S, Ts-1)) on the bottleneck half of d dec_in, times ReLU' of
// the bottleneck output: dbn[ts, r] = [bn_out > 0] * sum over the frames that read ts (ascending t)
__global__ void ftr_dbn_kernel(const float* __restrict__ ddec, const float* __restrict__ bn_out, int B, int Tp, int M, int S,
                               int Ts, float* __restrict__ dbn) {
  const size_t R = (size_t)B * M, n = (size_t)Ts * R;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int ts = (int)(i / R);
    const int r = (int)(i % R), b = r / M, m = r - b * M;
    const int t0 = ts * S, t1 = ts == Ts - 1 ? Tp : min(t0 + S, Tp);
    float acc = 0.f;
    for (int t = t0; t < t1; ++t) acc += ddec[((size_t)t * B + b) * 2 * M + M + m];
    dbn[i] = bn_out[i] > 0.f ? acc : 0.f;
  }
}

// d encT [Tp,B,M] = ReLU'(encT) * ( ddec[t,b,m] (decoder input, columns < M)
//   + inv2[b] * sum_{(m',k) : reflect(m' + k - Ne) = m} dX[ts(t), b*M+m', 2Nn+1+k] / len(ts)    (unfold^T . down-sampling^T)
//   - inv2[b] * dot[b] * c_Ne[m] / (M K Ts len(ts)) )                                           (second-norm backward)
// gather form: the (m', k) pairs of m are the direct, left-reflected and right-reflected sources of each offset k - Ne.
// CUM (cumulative norm, scaleT / suffix [Ts, B*M]): each source term is the gradient of the block mean u[ts, r', k],
//   dX[ts, r', k] s[ts, r'] + suffix[ts, r'], divided by len(ts), and there is no per-clip term
template <bool CUM>
__global__ void ftr_denc_kernel(const float* __restrict__ ddec, const float* __restrict__ dX, const float* __restrict__ encT,
                                const float* __restrict__ inv2, const float* __restrict__ dot, const float* __restrict__ scaleT,
                                const float* __restrict__ suffix, int B, int Tp, int M, int Nn, int Ne, int S, float cnt2,
                                float* __restrict__ denc) {
  const int K = (2 * Nn + 1) + (2 * Ne + 1);
  const size_t n = (size_t)Tp * B * M;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(i % M);
    const size_t tb = i / M;
    const int b = (int)(tb % B), t = (int)(tb / B);
    const int ts = t == 0 ? 0 : 1 + (t - 1) / S;
    int t0, len;
    shrink_block(ts, S, Tp, t0, len);
    const float* dx = dX + ((size_t)ts * B * M + (size_t)b * M) * K + (2 * Nn + 1);
    const size_t row0 = (size_t)ts * B * M + (size_t)b * M;  // scaleT / suffix index of (ts, row b*M)
    auto term = [&](int src, int k) {
      return CUM ? fmaf(dx[(size_t)src * K + k], scaleT[row0 + src], suffix[row0 + src]) : dx[(size_t)src * K + k];
    };
    float acc = 0.f;
    for (int k = 0; k <= 2 * Ne; ++k) {
      const int o = k - Ne;
      int src = m - o;                                        // m' + o = m
      if (src >= 0 && src < M) acc += term(src, k);
      src = -m - o;                                           // m' + o = -m < 0
      if (m > 0 && src >= 0 && src < M) acc += term(src, k);
      src = 2 * (M - 1) - m - o;                              // m' + o = 2(M-1) - m >= M
      if (m < M - 1 && src >= 0 && src < M) acc += term(src, k);
    }
    if (CUM) {
      const float v = ddec[tb * 2 * M + m] + acc / (float)len;
      denc[i] = encT[i] > 0.f ? v : 0.f;
      continue;
    }
    const float s = inv2[b], fl = (float)len;
    float v = ddec[tb * 2 * M + m] + s * acc / fl - s * dot[b] * (float)reflect_count(m, M, Ne) / (cnt2 * fl);
    denc[i] = encT[i] > 0.f ? v : 0.f;
  }
}

// backward of the second cumulative norm X[ts,r,k] = u[ts,r,k] s[ts,r] (fast_cum_bn_scale_launch):
//   d u[ts,r,k] = dX[ts,r,k] s[ts,r] + suffix[ts,r],  suffix[ts,r] = sum_{ts'' >= ts} -s[ts'',r] <dX[ts'',r,:], X[ts'',r,:]> /
//   (K (ts''+1)).  One thread per row, sequential in ts (fixed order); ftr_denc_kernel<true> maps d u back to the encoder
__global__ void ftr_cum_suffix_kernel(const float* __restrict__ dX, const float* __restrict__ X, const float* __restrict__ scaleT,
                                      int Ts, int R, int K, float* __restrict__ suffix) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float acc = 0.f;
  for (int ts = Ts - 1; ts >= 0; --ts) {
    const size_t o = ((size_t)ts * R + r) * K;
    float dot = 0.f;
    for (int k = 0; k < K; ++k) dot = fmaf(dX[o + k], X[o + k], dot);
    acc += -scaleT[(size_t)ts * R + r] * dot / ((float)K * (float)(ts + 1));
    suffix[(size_t)ts * R + r] = acc;
  }
}

int ftr_dbn_launch(const float* ddec, const float* bn_out, int B, int Tp, int M, int S, int Ts, float* dbn, cudaStream_t st) {
  ftr_dbn_kernel<<<ew_grid((size_t)Ts * B * M), 256, 0, st>>>(ddec, bn_out, B, Tp, M, S, Ts, dbn);
  FSN_CHECK_LAUNCH("ftr_dbn_kernel");
  return FSN_OK;
}

int ftr_cum_suffix_launch(const float* dX, const float* X, const float* scaleT, int Ts, int R, int K, float* suffix,
                          cudaStream_t st) {
  ftr_cum_suffix_kernel<<<cdiv(R, 128), 128, 0, st>>>(dX, X, scaleT, Ts, R, K, suffix);
  FSN_CHECK_LAUNCH("ftr_cum_suffix_kernel");
  return FSN_OK;
}

int ftr_denc_launch(bool cum, const float* ddec, const float* dX, const float* encT, const float* inv2, const float* dot,
                    const float* scaleT, const float* suffix, int B, int Tp, int M, int Nn, int Ne, int S, float cnt2,
                    float* denc, cudaStream_t st) {
  const unsigned grid = ew_grid((size_t)Tp * B * M);
  if (cum)
    ftr_denc_kernel<true><<<grid, 256, 0, st>>>(ddec, dX, encT, inv2, dot, scaleT, suffix, B, Tp, M, Nn, Ne, S, cnt2, denc);
  else
    ftr_denc_kernel<false><<<grid, 256, 0, st>>>(ddec, dX, encT, inv2, dot, scaleT, suffix, B, Tp, M, Nn, Ne, S, cnt2, denc);
  FSN_CHECK_LAUNCH("ftr_denc_kernel");
  return FSN_OK;
}

// ------------------------------------------------------------------------------------------ workspace
enum { L_ENC1, L_ENC2, L_BN0, L_BN1, L_DEC1, L_DEC2, NL };

struct FastTrainWs {
  float *magT, *melT, *xenc, *encT, *xbn, *bn_out, *dec_in, *dec_out;
  float *inv1, *inv2, *dot;
  float2 *sums1, *sums2, *fs;
  // cumulative norm: frame sums of the mel spectrogram [B*Tp], scales of (frame, clip) [Tp, B] and of (shrunk step, row)
  // [Ts, B*M] (kept for the backward), suffix sums of the second norm's backward [Ts, B*M]
  float2* fs1;
  float *cum1, *cum2, *suffix;
  LayerSave L[NL];
  float *dY, *dH, *ddec, *dbn, *dxbn, *denc;
  float *dh_rec[2], *dc[2], *dh_mid;
  float *splitk, *colsum, *gT, *xT, *rec;
  size_t colsum_floats;
  float *whhT[NL], *wihT[NL];  // FSN_PREC_TF32_TC: transposed weights of the tensor-core layers
  __half *h16[NL], *w16;       // fp16 MMA operands of the forward step kernel
  size_t bytes;
};

struct LayerShape { int R, K0, H, steps; };

static void layer_shapes(const fsn_fast_desc* d, const FastDims& m, LayerShape* s) {
  const int R = m.B * m.M;
  s[L_ENC1] = {m.B, m.M, d->enc1_hidden, m.Tp};
  s[L_ENC2] = {m.B, d->enc1_hidden, d->enc2_hidden, m.Tp};
  s[L_BN0] = {R, m.K, d->bn_hidden, m.Ts};
  s[L_BN1] = {R, d->bn_hidden, d->bn_hidden, m.Ts};
  s[L_DEC1] = {m.B, 2 * m.M, d->dec_hidden, m.Tp};
  s[L_DEC2] = {m.B, d->dec_hidden, d->dec_hidden, m.Tp};
}

// the encoder input (normalised mel spectrogram) needs no gradient: no dx GEMM, no transposed W_ih
static bool dx_tf32(int l) { return l != L_ENC1; }

static size_t smax(size_t a, size_t b) { return a > b ? a : b; }

static void carve_fast_train(const fsn_fast_desc* d, const FastDims& m, void* base, FastTrainWs& w) {
  Carver c(base);
  const size_t Tp = m.Tp, B = m.B, F = m.F, M = m.M, K = m.K, Ts = m.Ts, R = (size_t)m.B * m.M;
  LayerShape s[NL];
  layer_shapes(d, m, s);
  w.magT = c.take<float>(Tp * B * F);
  w.melT = c.take<float>(Tp * B * M);
  w.xenc = c.take<float>(Tp * B * M);
  w.encT = c.take<float>(Tp * B * M);
  w.xbn = c.take<float>(Ts * R * K);
  w.bn_out = c.take<float>(Ts * R);
  w.dec_in = c.take<float>(Tp * B * 2 * M);
  w.dec_out = c.take<float>(Tp * B * 2 * F);
  w.inv1 = c.take<float>(B); w.inv2 = c.take<float>(B); w.dot = c.take<float>(B);
  w.sums1 = c.take<float2>(B); w.sums2 = c.take<float2>(B); w.fs = c.take<float2>(B * Ts);
  size_t rh = 0, hmax = 0, wmax = 0, g_blk = 0, x_blk = 0;
  for (int l = 0; l < NL; ++l) {
    const size_t rows = (size_t)s[l].steps * s[l].R, H = s[l].H;
    w.L[l].G = c.take<float>(rows * 4 * H); w.L[l].C = c.take<float>(rows * H); w.L[l].H = c.take<float>(rows * H);
    rh = smax(rh, (size_t)s[l].R * H);
    hmax = smax(hmax, H);
    wmax = smax(wmax, 4 * H * (H + s[l].K0));
    if (tf32_layer(d->precision, s[l].H)) {
      g_blk = smax(g_blk, tgemm_blocked_floats(rows, 4 * s[l].H));
      x_blk = smax(x_blk, tgemm_blocked_floats(rows, s[l].K0 > s[l].H ? s[l].K0 : s[l].H));
    }
  }
  w.dY = c.take<float>(Tp * B * 2 * F);
  w.dH = c.take<float>(Tp * B * smax(d->dec_hidden, d->enc2_hidden));
  w.ddec = c.take<float>(Tp * B * 2 * M);
  w.dbn = c.take<float>(Ts * R);
  w.dxbn = c.take<float>(Ts * R * K);
  w.denc = c.take<float>(Tp * B * M);
  for (int i = 0; i < 2; ++i) { w.dh_rec[i] = c.take<float>(rh); w.dc[i] = c.take<float>(rh); }
  w.dh_mid = c.take<float>(rh);
  w.splitk = c.take<float>(SPLITK_SCRATCH_FLOATS);
  w.colsum_floats = (size_t)COLSUM_MAX_S * smax(4 * hmax, 2 * F);
  w.colsum = c.take<float>(w.colsum_floats);
  w.gT = w.xT = w.rec = nullptr;
  w.w16 = nullptr;
  for (int l = 0; l < NL; ++l) { w.whhT[l] = w.wihT[l] = nullptr; w.h16[l] = nullptr; }
  if (d->precision == FSN_PREC_TF32_TC) {
    for (int l = 0; l < NL; ++l) {
      if (!tf32_layer(d->precision, s[l].H)) continue;
      const size_t H = s[l].H;
      w.whhT[l] = c.take<float>(H * 4 * H);
      if (dx_tf32(l)) w.wihT[l] = c.take<float>((size_t)s[l].K0 * 4 * H);
      w.h16[l] = c.take<__half>((size_t)s[l].steps * s[l].R * H);
    }
    w.gT = c.take<float>(g_blk);
    w.xT = c.take<float>(x_blk);
    w.rec = c.take<float>(4 * rh);
    w.w16 = c.take<__half>(wmax);
  }
  w.fs1 = nullptr;
  w.cum1 = w.cum2 = w.suffix = nullptr;
  if (m.cum) {
    w.fs1 = c.take<float2>(B * Tp);
    w.cum1 = c.take<float>(Tp * B);
    w.cum2 = c.take<float>(Ts * R);
    w.suffix = c.take<float>(Ts * R);
  }
  w.bytes = c.off;
}

static int fast_train_check(const fsn_fast_desc* d, int B, int T, FastDims& m) {
  FSN_REQUIRE(d, FSN_ERR_SHAPE, "fast training: no descriptor");
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "fast training: the GRU cell is not built");
  FSN_REQUIRE(d->precision == FSN_PREC_FP32 || d->precision == FSN_PREC_TF32_TC, FSN_ERR_UNSUPPORTED,
              "fast training: precision must be fp32 or tf32_tc");
  int rc = fast_dims(d, B, T, m);
  if (rc) return rc;
  FSN_REQUIRE(d->noisy_num_neighbors >= 0 && d->enc_num_neighbors >= 0 && d->enc1_hidden > 0 && d->enc2_hidden > 0 &&
                  d->bn_hidden > 0 && d->dec_hidden > 0,
              FSN_ERR_SHAPE, "fast training: bad descriptor");
  FSN_REQUIRE(m.Ts <= 65535, FSN_ERR_SHAPE, "fast training: too many frames");
  return FSN_OK;
}

static const fsn_lstm_layer& layer_weights(const fsn_fast_weights* wt, int l) {
  switch (l) {
    case L_ENC1: return wt->enc1;
    case L_ENC2: return wt->enc2;
    case L_BN0: return wt->bn[0];
    case L_BN1: return wt->bn[1];
    case L_DEC1: return wt->dec1;
    default: return wt->dec2;
  }
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_fast_train_workspace_bytes(const fsn_fast_desc* d, int B, int T) {
  FastDims m;
  if (fast_train_check(d, B, T, m)) return 0;
  FastTrainWs w;
  carve_fast_train(d, m, nullptr, w);
  return w.bytes;
}

extern "C" int fsn_fast_train_forward(const fsn_fast_desc* d, const fsn_fast_weights* wt, const float* mix_mag, int B, int T,
                                      float* out, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  FastDims m;
  int rc = fast_train_check(d, B, T, m);
  if (rc) return rc;
  if ((rc = layout_clips_check(B, true, "fast training"))) return rc;
  FSN_REQUIRE(wt && mix_mag && out, FSN_ERR_SHAPE, "fast training: null argument");
  FastTrainWs w;
  carve_fast_train(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int Tp = m.Tp, F = m.F, M = m.M, K = m.K, Ts = m.Ts, R = B * M;
  LayerShape s[NL];
  layer_shapes(d, m, s);
  // layer l over its steps from X [steps, R, K0]; X16 = fp16 copy of X left by the layer below (or nullptr)
  auto layer = [&](int l, const float* X, const __half* X16) {
    const LayerHalf half{w.h16[l], X16, w.w16};
    return layer_forward(d->precision, layer_weights(wt, l), X, s[l].R, s[l].K0, s[l].H, s[l].steps, w.L[l], w.rec, w.splitk,
                         &half, st);
  };
  // look-ahead pad + time-major layout, Mel filtering (model.py:161-166)
  if ((rc = transpose_mag_launch(mix_mag, B, F, T, Tp, F, (size_t)B * F, w.magT, nullptr, nullptr, st))) return rc;
  if ((rc = fc_gemm_launch(w.magT, wt->mel_fb, nullptr, w.melT, Tp * B, F, M, FSN_ACT_NONE, st, /*w_kmajor=*/true))) return rc;
  // first norm (model.py:170): the mel spectrogram has no parameter behind it, only the normalised copy is kept;
  // cumulative norm: one scale per (frame, clip) from the running mean over the mel bins
  if (m.cum) {
    if ((rc = frame_stats_launch(w.melT, B, Tp, M, 0, M, (size_t)B * M, w.fs1, st))) return rc;
    if ((rc = cum_clip_scale_launch(w.fs1, B, Tp, M, TRAIN_CUM_EPS, w.cum1, st))) return rc;
    if ((rc = scale_rows_launch(w.melT, w.cum1, (size_t)Tp * B * M, M, Tp * B, 1, w.xenc, st))) return rc;
  } else {
    if ((rc = train_tm_stats_launch(w.melT, B, M, Tp, 0, w.sums1, st))) return rc;
    if ((rc = norm_scales_launch(w.sums1, w.sums1, B, (float)M * Tp, 1.f, w.inv1, nullptr, st))) return rc;
    if ((rc = scale_rows_launch(w.melT, w.inv1, (size_t)Tp * B * M, M, B, 1, w.xenc, st))) return rc;
  }
  // encoder: LSTM(M->He1), LSTM(He1->He2) + Linear(M) + ReLU (model.py:35-54,171)
  if ((rc = layer(L_ENC1, w.xenc, nullptr))) return rc;
  if ((rc = layer(L_ENC2, w.L[L_ENC1].H, nullptr))) return rc;  // He1 != He2: no shared fp16 path
  if ((rc = fc_gemm_launch(w.L[L_ENC2].H, wt->enc_fc_w, wt->enc_fc_b, w.encT, Tp * B, d->enc2_hidden, M, FSN_ACT_RELU, st)))
    return rc;
  // bottleneck input: unfold + concat + down-sampling, its norm; the normalised input is kept (model.py:174-187)
  if ((rc = fast_bn_input_launch(w.melT, w.encT, M, (size_t)B * M, B, Tp, M, d->noisy_num_neighbors, d->enc_num_neighbors,
                                 m.S, Ts, w.xbn, w.fs, st)))
    return rc;
  if (m.cum) {  // per-(shrunk step, row) scales, kept in cum2 for the backward
    if ((rc = fast_cum_bn_scale_launch(w.xbn, R, K, Ts, TRAIN_CUM_EPS, w.cum2, st))) return rc;
    if ((rc = scale_rows_launch(w.xbn, w.cum2, (size_t)Ts * R * K, K, Ts * R, 1, w.xbn, st))) return rc;
  } else {
    if ((rc = clip_reduce_only_launch(w.fs, B, Ts, w.sums2, st))) return rc;
    if ((rc = norm_scales_launch(w.sums2, w.sums2, B, (float)M * K * Ts, 1.f, w.inv2, nullptr, st))) return rc;
    if ((rc = scale_rows_launch(w.xbn, w.inv2, (size_t)Ts * R * K, K, R, M, w.xbn, st))) return rc;
  }
  // bottleneck 2xLSTM(K->Hb->Hb) + Linear(1) + ReLU over Ts steps (model.py:188-189)
  if ((rc = layer(L_BN0, w.xbn, nullptr))) return rc;
  if ((rc = layer(L_BN1, w.L[L_BN0].H, w.h16[L_BN0]))) return rc;
  if ((rc = sb_head_launch(w.L[L_BN1].H, Ts * R, d->bn_hidden, 1, wt->bn_fc_w, wt->bn_fc_b, 1, FSN_ACT_RELU, w.bn_out,
                           HeadGeom{Ts * R, 1, 0, 0, 1}, 0, st)))
    return rc;
  // up-sampling + concat, decoder LSTM(2M->Hd), LSTM(Hd->Hd) + Linear(2F) (model.py:191-196)
  if ((rc = fast_dec_input_launch(w.encT, w.bn_out, M, 1, (size_t)B * M, B, Tp, M, m.S, Ts, 1, B, w.dec_in, st))) return rc;
  if ((rc = layer(L_DEC1, w.dec_in, nullptr))) return rc;
  if ((rc = layer(L_DEC2, w.L[L_DEC1].H, w.h16[L_DEC1]))) return rc;
  if ((rc = fc_gemm_launch(w.L[L_DEC2].H, wt->dec_fc_w, wt->dec_fc_b, w.dec_out, Tp * B, d->dec_hidden, 2 * F, FSN_ACT_NONE, st)))
    return rc;
  return crm_output_launch(w.dec_out, 2 * F, (size_t)B * 2 * F, B, Tp, F, d->look_ahead, out, st);
}

extern "C" int fsn_fast_train_backward(const fsn_fast_desc* d, const fsn_fast_weights* wt, const float* dout, int B, int T,
                                       const fsn_fast_grads* g, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  FastDims m;
  int rc = fast_train_check(d, B, T, m);
  if (rc) return rc;
  FSN_REQUIRE(wt && dout && g, FSN_ERR_SHAPE, "fast training: null argument");
  FastTrainWs w;
  carve_fast_train(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int Tp = m.Tp, F = m.F, M = m.M, K = m.K, Ts = m.Ts, R = B * M;
  const int Hd = d->dec_hidden, He2 = d->enc2_hidden, Hb = d->bn_hidden;
  LayerShape s[NL];
  layer_shapes(d, m, s);
  const WgradScratch wg{w.gT, w.xT, w.splitk, w.colsum, w.colsum_floats};
  // the lower layer of each pair keeps its BPTT state in dh_rec[0] / dc[0], the upper one in dh_rec[1] / dc[1]
  LayerBwd L[NL];
  for (int l = 0; l < NL; ++l) {
    const fsn_lstm_layer& lw = layer_weights(wt, l);
    L[l] = LayerBwd{lw.w_ih, lw.w_hh, w.L[l], s[l].R, s[l].K0, s[l].H, w.dh_rec[l & 1], w.dc[l & 1], w.whhT[l], w.wihT[l],
                    w.splitk};
    if ((rc = layer_bwd_transpose_weights(L[l], st))) return rc;
  }
  // ---- decoder Linear(2F) (model.py:196-200 backwards)
  if ((rc = train_dy_launch(dout, nullptr, FSN_ACT_NONE, B, F, T, Tp, d->look_ahead, w.dY, st))) return rc;
  if ((rc = linear_bwd(w.dY, w.L[L_DEC2].H, wt->dec_fc_w, Tp * B, 2 * F, Hd, g->dec_fc_w, g->dec_fc_b, w.dH, w.splitk,
                       w.colsum, w.colsum_floats, st)))
    return rc;
  // ---- decoder BPTT, d dec_in
  if ((rc = stack_bwd(L + L_DEC1, 2, Tp, w.dH, nullptr, nullptr, 0, w.dh_mid, nullptr, w.ddec, st))) return rc;
  if ((rc = layer_weight_grads(L[L_DEC2], Tp, w.L[L_DEC1].H, g->dec2.w_ih, g->dec2.w_hh, g->dec2.b_ih, g->dec2.b_hh, wg, st)))
    return rc;
  if ((rc = layer_weight_grads(L[L_DEC1], Tp, w.dec_in, g->dec1.w_ih, g->dec1.w_hh, g->dec1.b_ih, g->dec1.b_hh, wg, st)))
    return rc;
  // ---- up-sampling transpose + ReLU' of the bottleneck output, its Linear(1)
  if ((rc = ftr_dbn_launch(w.ddec, w.bn_out, B, Tp, M, m.S, Ts, w.dbn, st))) return rc;
  if ((rc = linear_bwd(w.dbn, w.L[L_BN1].H, wt->bn_fc_w, Ts * R, 1, Hb, g->bn_fc_w, g->bn_fc_b, nullptr, w.splitk, w.colsum,
                       w.colsum_floats, st)))
    return rc;
  // ---- bottleneck BPTT (the Linear(1) backward folded into layer 1's point kernel), d X_bn
  if ((rc = stack_bwd(L + L_BN0, 2, Ts, nullptr, w.dbn, wt->bn_fc_w, 1, w.dh_mid, nullptr, w.dxbn, st))) return rc;
  if ((rc = layer_weight_grads(L[L_BN1], Ts, w.L[L_BN0].H, g->bn[1].w_ih, g->bn[1].w_hh, g->bn[1].b_ih, g->bn[1].b_hh, wg, st)))
    return rc;
  if ((rc = layer_weight_grads(L[L_BN0], Ts, w.xbn, g->bn[0].w_ih, g->bn[0].w_hh, g->bn[0].b_ih, g->bn[0].b_hh, wg, st)))
    return rc;
  // ---- second norm + down-sampling + unfold backward, ReLU' of the encoder output, its Linear(M)
  if (m.cum) {
    if ((rc = ftr_cum_suffix_launch(w.dxbn, w.xbn, w.cum2, Ts, R, K, w.suffix, st))) return rc;
    if ((rc = ftr_denc_launch(true, w.ddec, w.dxbn, w.encT, nullptr, nullptr, w.cum2, w.suffix, B, Tp, M,
                              d->noisy_num_neighbors, d->enc_num_neighbors, m.S, 0.f, w.denc, st)))
      return rc;
  } else {
    if ((rc = train_dot_launch(w.dxbn, w.xbn, Ts, R, M, K, B, w.dot, st))) return rc;
    if ((rc = ftr_denc_launch(false, w.ddec, w.dxbn, w.encT, w.inv2, w.dot, nullptr, nullptr, B, Tp, M,
                              d->noisy_num_neighbors, d->enc_num_neighbors, m.S, (float)M * K * Ts, w.denc, st)))
      return rc;
  }
  if ((rc = linear_bwd(w.denc, w.L[L_ENC2].H, wt->enc_fc_w, Tp * B, M, He2, g->enc_fc_w, g->enc_fc_b, w.dH, w.splitk, w.colsum,
                       w.colsum_floats, st)))
    return rc;
  // ---- encoder BPTT (its input is the normalised mel spectrogram: no dx)
  if ((rc = stack_bwd(L + L_ENC1, 2, Tp, w.dH, nullptr, nullptr, 0, w.dh_mid, nullptr, nullptr, st))) return rc;
  if ((rc = layer_weight_grads(L[L_ENC2], Tp, w.L[L_ENC1].H, g->enc2.w_ih, g->enc2.w_hh, g->enc2.b_ih, g->enc2.b_hh, wg, st)))
    return rc;
  return layer_weight_grads(L[L_ENC1], Tp, w.xenc, g->enc1.w_ih, g->enc1.w_hh, g->enc1.b_ih, g->enc1.b_hh, wg, st);
}

// ---- unit-test hook of the bottleneck backward (include/fsn_b200.h): the launchers fsn_fast_train_backward runs, every
// argument checked before any CUDA call
extern "C" int fsn_debug_fast_norm_unfold_bwd(const float* ddec, const float* dX, const float* X, const float* encT,
                                              const float* bn_out, const float* scale, int cum, int B, int Tp, int M, int Nn,
                                              int Ne, int S, float cnt2, float* mid, float* denc, float* dbn,
                                              fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(ddec && (!dbn || bn_out) && (!denc || (dX && X && encT && scale && mid)), FSN_ERR_SHAPE,
              "fast backward hook: null argument");
  FSN_REQUIRE(B > 0 && Tp > 0 && M > 0 && S > 0, FSN_ERR_SHAPE, "fast backward hook: bad shape B=%d Tp=%d M=%d S=%d", B, Tp,
              M, S);
  FSN_REQUIRE(Nn >= 0 && Ne >= 0 && Nn < M && Ne < M, FSN_ERR_SHAPE, "fast backward hook: reflect padding needs 0 <= Nn, Ne < M");
  FSN_REQUIRE(cum || !denc || cnt2 > 0.f, FSN_ERR_SHAPE, "fast backward hook: cnt2 must be positive");
  const int Ts = 1 + cdiv(Tp - 1, S), R = B * M, K = (2 * Nn + 1) + (2 * Ne + 1);
  FSN_REQUIRE((size_t)Tp * B * 2 * M < ((size_t)1 << 31) && (size_t)Ts * R * K < ((size_t)1 << 31), FSN_ERR_SHAPE,
              "fast backward hook: tensors must stay below 2^31 elements");
  const cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (dbn && (rc = ftr_dbn_launch(ddec, bn_out, B, Tp, M, S, Ts, dbn, st))) return rc;
  if (!denc) return FSN_OK;
  if (cum) {
    if ((rc = ftr_cum_suffix_launch(dX, X, scale, Ts, R, K, mid, st))) return rc;
    return ftr_denc_launch(true, ddec, dX, encT, nullptr, nullptr, scale, mid, B, Tp, M, Nn, Ne, S, 0.f, denc, st);
  }
  if ((rc = train_dot_launch(dX, X, Ts, R, M, K, B, mid, st))) return rc;
  return ftr_denc_launch(false, ddec, dX, encT, scale, mid, nullptr, nullptr, B, Tp, M, Nn, Ne, S, cnt2, denc, st);
}
