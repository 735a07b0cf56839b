// fast_fullsubnet (recipes/dns_interspeech_2020/fast_fullsubnet/model.py:11-202, BASELINE config 4): host
// orchestration and the second cumulative norm on top of the shared fp32 building blocks (mel filtering as a GEMM, the
// bottleneck input with its real-time down-sampling and the decoder input with its up-sampling in fsn_lstm_simt.cu).
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

// second cumulative norm (model.py:186-187 -> base_model.py:220-251 on [B*M, K, Ts]): one thread per row (b,m), sequential
// over the shrunk steps; the row sum of each step runs over the K block means fast_bn_input_launch
// wrote, so inference and training share the scales
__global__ void fast_cum_bn_scale_kernel(const float* __restrict__ bn, int R, int K, int Ts, float eps,
                                         float* __restrict__ scaleT) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float run = 0.f;
  for (int ts = 0; ts < Ts; ++ts) {
    const float* x = bn + ((size_t)ts * R + r) * K;
    float s = 0.f;
    for (int k = 0; k < K; ++k) s += x[k];
    run += s;
    scaleT[(size_t)ts * R + r] = 1.0f / (run / ((float)K * (float)(ts + 1)) + eps);
  }
}

int fast_cum_bn_scale_launch(const float* bn, int R, int K, int Ts, float eps, float* scaleT, cudaStream_t st) {
  fast_cum_bn_scale_kernel<<<cdiv(R, 128), 128, 0, st>>>(bn, R, K, Ts, eps, scaleT);
  FSN_CHECK_LAUNCH("fast_cum_bn_scale_kernel");
  return FSN_OK;
}

// GRU: the inference kernels of this model are built for LSTM only
static bool fast_tc_ok(const fsn_fast_desc* d) {
  const int K = (2 * d->noisy_num_neighbors + 1) + (2 * d->enc_num_neighbors + 1);
  return d->cell_type == FSN_CELL_LSTM && d->bn_hidden == 384 && d->bn_layers == 2 && K <= 32;
}
static bool fast_x3(const fsn_fast_desc* d) { return d->precision == FSN_PREC_F16X3_TC; }

struct FastWs {
  float *magT, *melT, *encT, *bn, *bn_out, *dec_in, *dec_out, *inv1, *inv2;
  float *cum1, *cum2;  // cumulative norm: scales of (frame, clip) [Tp, B] and of (shrunk step, row) [Ts, B*M]
  float2 *fs, *sums;
  float *bn_h0[2], *bn_h1[2], *bn_c0, *bn_c1;
  SeqStackWs seq;          // encoder and decoder LSTM pairs, one after the other
  size_t bytes;
};

static bool fast_is_tc(const fsn_fast_desc* d) { return d->precision == FSN_PREC_F16_TC || d->precision == FSN_PREC_F16X3_TC; }

// encoder / decoder pair: LSTM(K0 -> H0), LSTM(H0 -> H1) + Linear(O) over B rows of Tp steps; on the tensor cores with
// the tensor-core precisions when all three encoder / decoder hidden sizes are supported there
static SeqStack fast_pair(const fsn_fast_desc* d, const FastDims& m, int K0, int H0, int H1, int O, int act) {
  SeqStack s;
  memset(&s, 0, sizeof(s));
  s.R = m.B; s.Tp = m.Tp; s.K0 = K0; s.n = 2; s.H[0] = H0; s.H[1] = H1; s.O = O; s.act = act;
  s.x3 = fast_x3(d);
  s.tc = fast_is_tc(d) && lstm_rec_tc_supported(d->enc1_hidden, s.x3) && lstm_rec_tc_supported(d->enc2_hidden, s.x3) &&
         lstm_rec_tc_supported(d->dec_hidden, s.x3);
  return s;
}

int fast_dims(const fsn_fast_desc* d, int B, int T, FastDims& m) {
  FSN_REQUIRE(d && d->num_freqs > 1 && d->num_mels > 1 && d->shrink_size >= 1 && d->look_ahead >= 0, FSN_ERR_SHAPE,
              "fast model: bad descriptor");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "fast model: empty input (B=%d, T=%d)", B, T);
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "fast model: the GRU cell is not built");
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE, FSN_ERR_UNSUPPORTED,
              "fast model: norm_type %d is not built", d->norm_type);
  FSN_REQUIRE(d->bn_layers == 2, FSN_ERR_UNSUPPORTED, "fast model: bottleneck_num_layers must be 2 in this build");
  FSN_REQUIRE(d->noisy_num_neighbors < d->num_mels && d->enc_num_neighbors < d->num_mels, FSN_ERR_SHAPE,
              "fast model: reflect padding needs num_neighbors < num_mels");
  m.B = B; m.T = T; m.Tp = T + d->look_ahead; m.F = d->num_freqs; m.M = d->num_mels; m.S = d->shrink_size;
  m.K = (2 * d->noisy_num_neighbors + 1) + (2 * d->enc_num_neighbors + 1);
  FSN_REQUIRE(m.Tp >= 2, FSN_ERR_SHAPE, "fast model: needs at least 2 frames incl. look-ahead");
  m.Ts = 1 + cdiv(m.Tp - 1, m.S);
  m.cum = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE;
  return FSN_OK;
}

static void fast_carve(const fsn_fast_desc* d, const FastDims& m, void* base, FastWs& w) {
  Carver c(base);
  const size_t BT = (size_t)m.B * m.Tp, R = (size_t)m.B * m.M;
  w.magT = c.take<float>(BT * m.F);
  w.melT = c.take<float>(BT * m.M);
  w.encT = c.take<float>(BT * m.M);
  w.bn = c.take<float>((size_t)m.Ts * R * m.K);
  w.bn_out = c.take<float>(2 * R * m.Ts);  // [B,2,M,Ts] when written by the tensor-core kernel
  w.dec_in = c.take<float>(BT * 2 * m.M);
  w.dec_out = c.take<float>(BT * 2 * m.F);
  w.inv1 = c.take<float>(m.B);
  w.inv2 = c.take<float>(m.B);
  w.fs = c.take<float2>(BT);
  w.sums = c.take<float2>(m.B);
  w.cum1 = w.cum2 = nullptr;
  if (m.cum) {
    w.cum1 = c.take<float>(BT);
    w.cum2 = c.take<float>((size_t)m.Ts * R);
  }
  if (!fast_is_tc(d)) {
    for (int i = 0; i < 2; ++i) { w.bn_h0[i] = c.take<float>(R * d->bn_hidden); w.bn_h1[i] = c.take<float>(R * d->bn_hidden); }
    w.bn_c0 = c.take<float>(R * d->bn_hidden);
    w.bn_c1 = c.take<float>(R * d->bn_hidden);
  }
  auto mx = [](int a, int b) { return a > b ? a : b; };
  seq_stack_carve(c, fast_pair(d, m, 2 * m.M, mx(d->enc1_hidden, d->dec_hidden), mx(d->enc2_hidden, d->dec_hidden),
                               mx(m.M, 2 * m.F), 0), w.seq);
  w.bytes = c.off;
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_fast_workspace_bytes(const fsn_fast_desc* d, int B, int T) {
  FastDims m;
  if (fast_dims(d, B, T, m)) return 0;
  FastWs w;
  fast_carve(d, m, nullptr, w);
  return w.bytes;
}

extern "C" size_t fsn_fast_packed_bytes(const fsn_fast_desc* d) { return fast_tc_ok(d) ? sb_tc_packed_bytes_raw(d->bn_hidden, fast_x3(d)) : 0; }

extern "C" int fsn_fast_pack_bn_weights(const fsn_fast_desc* d, const fsn_fast_weights* wt, void* packed,
                                        fsn_stream_t stream) {
  FSN_REQUIRE(fast_tc_ok(d), FSN_ERR_UNSUPPORTED, "fast model: the tensor-core bottleneck needs bn_hidden = 384, 2 layers");
  fsn_seq_weights s;
  for (int l = 0; l < 2; ++l) { s.w_ih[l] = wt->bn[l].w_ih; s.w_hh[l] = wt->bn[l].w_hh; s.b_ih[l] = wt->bn[l].b_ih; s.b_hh[l] = wt->bn[l].b_hh; }
  s.fc_w = wt->bn_fc_w; s.fc_b = wt->bn_fc_b;
  const int K = (2 * d->noisy_num_neighbors + 1) + (2 * d->enc_num_neighbors + 1);
  return sb_tc_pack_raw(&s, d->bn_hidden, K, /*fc_out=*/1, packed, (cudaStream_t)stream, fast_x3(d));
}

extern "C" int fsn_fast_model_forward(const fsn_fast_desc* d, const fsn_fast_weights* wt, const float* mix_mag, int B,
                                      int T, float* out, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  FastDims m;
  int rc = fast_dims(d, B, T, m);
  if (rc) return rc;
  FastWs w;
  fast_carve(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int Tp = m.Tp, M = m.M, F = m.F, R = B * M;
  // look-ahead pad + time-major layout, Mel filtering (model.py:161-166)
  if ((rc = transpose_mag_launch(mix_mag, B, F, T, Tp, (size_t)Tp * F, F, w.magT, nullptr, nullptr, st))) return rc;
  if ((rc = fc_gemm_launch(w.magT, wt->mel_fb, nullptr, w.melT, B * Tp, F, M, FSN_ACT_NONE, st, /*w_kmajor=*/true)))
    return rc;
  // encoder input norm (model.py:170): per-clip mean of the mel spectrogram incl. the look-ahead frames, or (cumulative
  // norm) the running mean over the mel bins of the frames so far, time-major cum1[t*B + b] (base_model.py:220-251)
  if ((rc = clip_stats_launch(w.melT, B, Tp, M, 0, w.fs, w.sums, st))) return rc;
  if (m.cum) {
    if ((rc = cum_clip_scale_launch(w.fs, B, Tp, M, TRAIN_CUM_EPS, w.cum1, st))) return rc;
  } else if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)M * Tp, 1.f, w.inv1, nullptr, st))) {
    return rc;
  }
  // F_l2m: LSTM(M->He1), LSTM(He1->He2) + Linear(M) + ReLU (model.py:35-54,171)
  SeqStack enc = fast_pair(d, m, M, d->enc1_hidden, d->enc2_hidden, M, FSN_ACT_RELU);
  enc.L[0] = wt->enc1; enc.L[1] = wt->enc2;
  enc.x = w.melT; enc.scale = m.cum ? w.cum1 : w.inv1; enc.step_scale = m.cum;
  enc.fc_w = wt->enc_fc_w; enc.fc_b = wt->enc_fc_b; enc.out = w.encT;
  if ((rc = seq_stack_forward(enc, w.seq, st))) return rc;
  // bottleneck input: unfold + concat + real-time down-sampling, then its norm (model.py:174-187)
  if ((rc = fast_bn_input_launch(w.melT, w.encT, (size_t)Tp * M, M, B, Tp, M, d->noisy_num_neighbors, d->enc_num_neighbors,
                                 m.S, m.Ts, w.bn, w.fs, st)))
    return rc;
  if (m.cum) {
    // per-(shrunk step, row) running mean over the K block means, time-major cum2[ts*R + r]
    if ((rc = fast_cum_bn_scale_launch(w.bn, R, m.K, m.Ts, TRAIN_CUM_EPS, w.cum2, st))) return rc;
  } else {
    // per-clip sum of the per-(b,ts) partials (fixed order), then 1/(mean+1e-5)
    if ((rc = clip_reduce_only_launch(w.fs, B, m.Ts, w.sums, st))) return rc;
    if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)M * m.K * m.Ts, 1.f, w.inv2, nullptr, st))) return rc;
  }
  // S: 2xLSTM(K->Hb->Hb) + Linear(1) + ReLU on B*M rows over Ts steps (model.py:188-189)
  // bn_out element (b, m, ts): [B*M, Ts] from the fp32 path, channel 0 of the [B,2,M,Ts] the tensor-core kernel writes
  const int Hb = d->bn_hidden;
  int bn_bstride = M;
  if (fast_is_tc(d)) {
    // tensor-core kernel of the fullsubnet sub-band stack: same stack shape (K<=32 -> 384 -> 384), the gather
    // does the unfold AND the time down-sampling on the fly from melT / encT, Linear output 1 of 2 is zero-padded
    FSN_REQUIRE(wt->bn_packed && fast_tc_ok(d), FSN_ERR_UNSUPPORTED,
                "fast model: the tensor-core precisions need packed bottleneck weights, bn_hidden = 384 and input width <= 32");
    SbTcArgs a;
    memset(&a, 0, sizeof(a));
    // cumulative norm: unit_scale replaces inv2[clip] (which the kernel still loads, unwritten and unused)
    a.packed = wt->bn_packed; a.magT = w.melT; a.fbT = w.encT; a.inv2 = w.inv2; a.crm = w.bn_out;
    a.unit_scale = m.cum ? w.cum2 : nullptr;
    a.B = B; a.F = M; a.Tp = Tp; a.la = 0; a.Ns = d->noisy_num_neighbors; a.Nf = d->enc_num_neighbors;
    a.H = Hb; a.act = FSN_ACT_RELU; a.steps = m.Ts; a.shrink = m.S; a.x3 = fast_x3(d);
    a.map = RowMap{B, M, M, 1};
    if ((rc = sb_tc_forward(a, st))) return rc;
    bn_bstride = 2 * M;
  } else {
    const Step2State s2{{w.bn_h0[0], w.bn_h0[1]}, w.bn_c0, {w.bn_h1[0], w.bn_h1[1]}, w.bn_c1, Hb, 0};
    for (int t = 0; t < m.Ts; ++t) {
      StepParams p;
      memset(&p, 0, sizeof(p));
      p.R = R; p.K0 = m.K; p.H = Hb;
      p.w_ih = wt->bn[0].w_ih; p.w_hh = wt->bn[0].w_hh; p.b_ih = wt->bn[0].b_ih; p.b_hh = wt->bn[0].b_hh;
      p.x0 = w.bn + (size_t)t * R * m.K; p.x0_row_stride = m.K;
      if (m.cum) { p.row_scale = w.cum2 + (size_t)t * R; p.row_scale_div = 1; }
      else       { p.row_scale = w.inv2; p.row_scale_div = M; }
      if ((rc = lstm_step2_launch(p, SEG0_DENSE, t, wt->bn[1], s2, st))) return rc;
      if ((rc = sb_head_launch(s2.h1_at(t), R, Hb, 1, wt->bn_fc_w, wt->bn_fc_b, 1, FSN_ACT_RELU, w.bn_out,
                               HeadGeom{R, 1, 0, 0, (size_t)m.Ts}, t, st)))
        return rc;
    }
  }
  // up-sampling + concat with the encoder output (model.py:191-194)
  if ((rc = fast_dec_input_launch(w.encT, w.bn_out, (size_t)bn_bstride * m.Ts, m.Ts, 1, B, Tp, M, m.S, m.Ts, Tp, 1, w.dec_in,
                                  st)))
    return rc;
  // F_m2l: LSTM(2M->Hd), LSTM(Hd->Hd) + Linear(2F) (model.py:77-96,196)
  SeqStack dec = fast_pair(d, m, 2 * M, d->dec_hidden, d->dec_hidden, 2 * F, FSN_ACT_NONE);
  dec.L[0] = wt->dec1; dec.L[1] = wt->dec2;
  dec.x = w.dec_in; dec.fc_w = wt->dec_fc_w; dec.fc_b = wt->dec_fc_b; dec.out = w.dec_out;
  if ((rc = seq_stack_forward(dec, w.seq, st))) return rc;
  return crm_output_launch(w.dec_out, (size_t)Tp * 2 * F, 2 * F, B, Tp, F, d->look_ahead, out, st);
}
