// fast_fullsubnet (recipes/dns_interspeech_2020/fast_fullsubnet/model.py:11-202, BASELINE config 4): host
// orchestration and the few extra kernels on top of the shared fp32 building blocks (mel filtering, real-time
// down/up-sampling, bottleneck input, decoder re-layout).
#include <stdlib.h>
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

// bottleneck input (model.py:174-187 before the norm): row (b,m), feature k: 2Nn+1 reflected mel rows + 2Ne+1
// encoder-output rows, down-sampled in time (first frame alone, then means of `S` frames; the last block over its
// own length).  One CTA per (b, ts): writes bn[ts][b*M+m][k] and the deterministic per-(b,ts) sum.
__global__ void fast_bn_input_kernel(const float* __restrict__ melT, const float* __restrict__ encT, int B, int Tp,
                                     int M, int Nn, int Ne, int S, int Ts, float* __restrict__ bn,
                                     float2* __restrict__ fs) {
  __shared__ float red[256];
  const int b = blockIdx.x / Ts, ts = blockIdx.x % Ts;
  const int K = (2 * Nn + 1) + (2 * Ne + 1);
  int t0, t1;  // frames [t0, t1) averaged into this shrunk frame
  if (ts == 0) { t0 = 0; t1 = 1; }
  else { t0 = 1 + (ts - 1) * S; t1 = min(t0 + S, Tp); }
  const float inv = 1.0f / (float)(t1 - t0);
  float local = 0.f;
  for (int i = threadIdx.x; i < M * K; i += blockDim.x) {
    const int m = i / K, k = i - m * K;
    float acc = 0.f;
    for (int t = t0; t < t1; ++t) {
      const size_t base = ((size_t)b * Tp + t) * M;
      acc += (k < 2 * Nn + 1) ? melT[base + reflect_idx(m + k - Nn, M)]
                              : encT[base + reflect_idx(m + (k - (2 * Nn + 1)) - Ne, M)];
    }
    const float v = acc * inv;
    bn[((size_t)ts * B * M + (size_t)b * M + m) * K + k] = v;
    local += v;
  }
  red[threadIdx.x] = local;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) fs[(size_t)b * Ts + ts] = make_float2(red[0], red[0]);
}

// decoder input (model.py:194): [enc_out (M) | up-sampled bottleneck output (M)] per (b,t); frame t of the
// up-sampled signal is shrunk frame t / S (model.py:131-140)
// bn_out element (b, m, ts) lives at bn_out[(b*bn_bstride + m) * Ts + ts]: bn_bstride = M for the fp32 path
// ([B*M, Ts]) and 2*M for the tensor-core path, which writes a [B,2,M,Ts] tensor whose channel 0 is the output
__global__ void fast_dec_input_kernel(const float* __restrict__ encT, const float* __restrict__ bn_out, int bn_bstride,
                                      int B, int Tp, int M, int S, int Ts, float* __restrict__ dec_in) {
  const size_t total = (size_t)B * Tp * 2 * M;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % (2 * M));
    const size_t bt = i / (2 * M);
    const int t = (int)(bt % Tp), b = (int)(bt / Tp);
    float v;
    if (c < M) v = encT[bt * M + c];
    else       v = bn_out[((size_t)b * bn_bstride + (c - M)) * Ts + min(t / S, Ts - 1)];
    dec_in[i] = v;
  }
}

// dec [B,Tp,2F] (channel c*F+f) -> out [B,2,F,T], dropping the first `la` frames (model.py:197-200)
__global__ void fast_output_kernel(const float* __restrict__ dec, int B, int Tp, int F, int la, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int T = Tp - la;
  const int bc = blockIdx.z;                 // b*2 + c
  const int b = bc >> 1, c = bc & 1;
  const int f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += 8) {         // read: f contiguous
    const int t = t0 + i, f = f0 + tx;
    tile[i][tx] = (t < T && f < F) ? dec[((size_t)b * Tp + t + la) * (2 * F) + c * F + f] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {         // write: t contiguous
    const int f = f0 + i, t = t0 + tx;
    if (f < F && t < T) out[(((size_t)b * 2 + c) * F + f) * T + t] = tile[tx][i];
  }
}

static bool fast_tc_ok(const fsn_fast_desc* d) {
  const int K = (2 * d->noisy_num_neighbors + 1) + (2 * d->enc_num_neighbors + 1);
  return d->bn_hidden == 384 && d->bn_layers == 2 && K <= 32;
}
static bool fast_x3(const fsn_fast_desc* d) { return d->precision == FSN_PREC_F16X3_TC; }

struct FastWs {
  float *magT, *melT, *encT, *bn, *bn_out, *dec_in, *dec_out, *inv1, *inv2;
  float2 *fs, *sums;
  float *e1_h[2], *e1_c, *e2_hall, *e2_c;
  float *bn_h0[2], *bn_h1[2], *bn_c0, *bn_c1;
  float *d1_h[2], *d1_c, *d2_hall, *d2_c;
  float* pp;               // h0 ping-pong of the persistent LSTM kernel [2][256][max H0]
  unsigned int* barrier;
  LstmTcWs tc;             // tensor-core LSTM layers of the encoder / decoder (fsn_lstm_rec_tc.cu)
  float* tc_mid;           // first layer's output for every step [B*Tp, max(He1, Hd)]
  size_t bytes;
};

static bool fast_is_tc(const fsn_fast_desc* d) { return d->precision == FSN_PREC_F16_TC || d->precision == FSN_PREC_F16X3_TC; }
// encoder / decoder LSTM pairs on the tensor cores?
static bool fast_lstm_tc(const fsn_fast_desc* d) {
  const bool x3 = d->precision == FSN_PREC_F16X3_TC;
  return fast_is_tc(d) && lstm_rec_tc_supported(d->enc1_hidden, x3) && lstm_rec_tc_supported(d->enc2_hidden, x3) &&
         lstm_rec_tc_supported(d->dec_hidden, x3);
}

int fast_dims(const fsn_fast_desc* d, int B, int T, FastDims& m) {
  FSN_REQUIRE(d && d->num_freqs > 1 && d->num_mels > 1 && d->shrink_size >= 1 && d->look_ahead >= 0, FSN_ERR_SHAPE,
              "fast model: bad descriptor");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "fast model: empty input (B=%d, T=%d)", B, T);
  FSN_REQUIRE(d->bn_layers == 2, FSN_ERR_UNSUPPORTED, "fast model: bottleneck_num_layers must be 2 in this build");
  FSN_REQUIRE(d->noisy_num_neighbors < d->num_mels && d->enc_num_neighbors < d->num_mels, FSN_ERR_SHAPE,
              "fast model: reflect padding needs num_neighbors < num_mels");
  m.B = B; m.T = T; m.Tp = T + d->look_ahead; m.F = d->num_freqs; m.M = d->num_mels; m.S = d->shrink_size;
  m.K = (2 * d->noisy_num_neighbors + 1) + (2 * d->enc_num_neighbors + 1);
  FSN_REQUIRE(m.Tp >= 2, FSN_ERR_SHAPE, "fast model: needs at least 2 frames incl. look-ahead");
  m.Ts = 1 + cdiv(m.Tp - 1, m.S);
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
  for (int i = 0; i < 2; ++i) w.e1_h[i] = c.take<float>((size_t)m.B * d->enc1_hidden);
  w.e1_c = c.take<float>((size_t)m.B * d->enc1_hidden);
  w.e2_hall = c.take<float>(BT * d->enc2_hidden);
  w.e2_c = c.take<float>((size_t)m.B * d->enc2_hidden);
  if (!fast_is_tc(d)) {
    for (int i = 0; i < 2; ++i) { w.bn_h0[i] = c.take<float>(R * d->bn_hidden); w.bn_h1[i] = c.take<float>(R * d->bn_hidden); }
    w.bn_c0 = c.take<float>(R * d->bn_hidden);
    w.bn_c1 = c.take<float>(R * d->bn_hidden);
  }
  for (int i = 0; i < 2; ++i) w.d1_h[i] = c.take<float>((size_t)m.B * d->dec_hidden);
  w.d1_c = c.take<float>((size_t)m.B * d->dec_hidden);
  w.d2_hall = c.take<float>(BT * d->dec_hidden);
  w.d2_c = c.take<float>((size_t)m.B * d->dec_hidden);
  w.pp = c.take<float>((size_t)2 * 256 * (d->dec_hidden > d->enc1_hidden ? d->dec_hidden : d->enc1_hidden));
  w.barrier = c.take<unsigned int>(64);
  memset(&w.tc, 0, sizeof(w.tc));
  w.tc_mid = nullptr;
  if (fast_lstm_tc(d)) {
    int Hm = d->enc1_hidden > d->enc2_hidden ? d->enc1_hidden : d->enc2_hidden;
    if (d->dec_hidden > Hm) Hm = d->dec_hidden;
    int Km = Hm > 2 * m.M ? Hm : 2 * m.M;
    lstm_tc_carve(c, BT, Km, Hm, d->precision == FSN_PREC_F16X3_TC, w.tc);
    w.tc_mid = c.take<float>(BT * (d->enc1_hidden > d->dec_hidden ? d->enc1_hidden : d->dec_hidden));
  }
  w.bytes = c.off;
}

// two chained single-layer LSTMs over the same rows: layer a (x -> Ha, state ping-pong) feeds layer b
// (Ha -> Hb, output kept for every step for the Linear layer that follows)
static int run_lstm_pair(const fsn_lstm_layer& la, int Ka, int Ha, const fsn_lstm_layer& lb, int Hb, int R, int steps,
                         const float* x, size_t x_row_stride, size_t x_step_stride, const float* row_scale,
                         float* ha[2], float* ca, float* hb_all, float* cb, float* pp, unsigned int* barrier,
                         cudaStream_t st, const LstmTcWs* tc = nullptr, float* tc_mid = nullptr, bool x3 = false) {
  int rc;
  static const bool stepwise = getenv("FSN_FB_STEPWISE") != nullptr;
  if (!stepwise && tc && tc_mid && x_step_stride == (size_t)Ka && x_row_stride == (size_t)steps * Ka) {
    // tensor cores: per layer one hoisted input-projection GEMM + the persistent wgmma recurrence
    if ((rc = lstm_layer_tc(la, x, (size_t)Ka, Ka, row_scale, steps, 0, R, steps, Ha, x3, *tc, tc_mid, st))) return rc;
    return lstm_layer_tc(lb, tc_mid, (size_t)Ha, Ha, nullptr, 1, 0, R, steps, Hb, x3, *tc, hb_all, st);
  }
  if (!stepwise && x_step_stride == (size_t)Ka && x_row_stride == (size_t)steps * Ka && fb_persistent_supported(Ka, Ha, Hb)) {
    // persistent cooperative wavefront kernel (fsn_fullband.cu), chunks of <= 256 rows
    fsn_seq_weights w2;
    memset(&w2, 0, sizeof(w2));
    w2.w_ih[0] = la.w_ih; w2.w_hh[0] = la.w_hh; w2.b_ih[0] = la.b_ih; w2.b_hh[0] = la.b_hh;
    w2.w_ih[1] = lb.w_ih; w2.w_hh[1] = lb.w_hh; w2.b_ih[1] = lb.b_ih; w2.b_hh[1] = lb.b_hh;
    for (int r0 = 0; r0 < R; r0 += 256) {
      const int nb = (R - r0 < 256) ? R - r0 : 256;
      if ((rc = fb_persistent_launch(&w2, x + (size_t)r0 * x_row_stride, row_scale ? row_scale + r0 : nullptr, pp,
                                     hb_all + (size_t)r0 * steps * Hb, barrier, nb, Ka, Ha, Hb, steps, st)))
        return rc;
    }
    return FSN_OK;
  }
  for (int t = 0; t < steps; ++t) {
    StepParams p;
    memset(&p, 0, sizeof(p));
    p.R = R; p.first = (t == 0);
    p.K0 = Ka; p.H = Ha;
    p.w_ih = la.w_ih; p.w_hh = la.w_hh; p.b_ih = la.b_ih; p.b_hh = la.b_hh;
    p.h_prev = ha[(t + 1) & 1]; p.h_prev_stride = Ha;
    p.h_out = ha[t & 1]; p.h_out_stride = Ha;
    p.c = ca;
    p.x0 = x + (size_t)t * x_step_stride; p.x0_row_stride = x_row_stride; p.row_scale = row_scale;
    if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
    p.K0 = Ha; p.H = Hb;
    p.w_ih = lb.w_ih; p.w_hh = lb.w_hh; p.b_ih = lb.b_ih; p.b_hh = lb.b_hh;
    p.x0 = ha[t & 1]; p.x0_row_stride = Ha; p.row_scale = nullptr;
    p.h_prev = hb_all + (size_t)(t > 0 ? t - 1 : 0) * Hb; p.h_prev_stride = (size_t)steps * Hb;
    p.h_out = hb_all + (size_t)t * Hb; p.h_out_stride = (size_t)steps * Hb;
    p.c = cb;
    if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
  }
  return FSN_OK;
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
  const bool lstm_tc = fast_lstm_tc(d);
  static const int tc_mask = getenv("FSN_FAST_TC_MASK") ? atoi(getenv("FSN_FAST_TC_MASK")) : 15;  // debug: 1 enc LSTMs, 2 enc fc, 4 dec LSTMs, 8 dec fc
  // look-ahead pad + time-major layout, Mel filtering (model.py:161-166)
  if ((rc = transpose_mag_launch(mix_mag, w.magT, B, F, T, Tp, st))) return rc;
  if ((rc = fc_gemm_launch(w.magT, wt->mel_fb, nullptr, w.melT, B * Tp, F, M, FSN_ACT_NONE, st, /*w_kmajor=*/true)))
    return rc;
  // encoder input norm (model.py:170): per-clip mean of the mel spectrogram incl. the look-ahead frames
  if ((rc = clip_stats_launch(w.melT, B, Tp, M, 0, w.fs, w.sums, st))) return rc;
  if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)M * Tp, 1.f, w.inv1, nullptr, st))) return rc;
  // F_l2m: LSTM(M->He1), LSTM(He1->He2) + Linear(M) + ReLU (model.py:35-54,171)
  if ((rc = run_lstm_pair(wt->enc1, M, d->enc1_hidden, wt->enc2, d->enc2_hidden, B, Tp, w.melT, (size_t)Tp * M, M,
                          w.inv1, w.e1_h, w.e1_c, w.e2_hall, w.e2_c, w.pp, w.barrier, st, (lstm_tc && (tc_mask & 1)) ? &w.tc : nullptr, w.tc_mid,
                          fast_x3(d))))
    return rc;
  if (lstm_tc && (tc_mask & 2)) {
    if ((rc = linear_tc(w.e2_hall, (size_t)d->enc2_hidden, d->enc2_hidden, wt->enc_fc_w, wt->enc_fc_b, M, FSN_ACT_RELU, w.encT,
                        (size_t)M, (size_t)B * Tp, fast_x3(d), w.tc, st)))
      return rc;
  } else if ((rc = fc_gemm_launch(w.e2_hall, wt->enc_fc_w, wt->enc_fc_b, w.encT, B * Tp, d->enc2_hidden, M, FSN_ACT_RELU, st))) {
    return rc;
  }
  // bottleneck input: unfold + concat + real-time down-sampling, then its norm (model.py:174-187)
  fast_bn_input_kernel<<<B * m.Ts, 256, 0, st>>>(w.melT, w.encT, B, Tp, M, d->noisy_num_neighbors,
                                                 d->enc_num_neighbors, m.S, m.Ts, w.bn, w.fs);
  FSN_CHECK_LAUNCH("fast_bn_input_kernel");
  // per-clip sum of the per-(b,ts) partials (fixed order), then 1/(mean+1e-5)
  if ((rc = clip_reduce_only_launch(w.fs, B, m.Ts, w.sums, st))) return rc;
  if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)M * m.K * m.Ts, 1.f, w.inv2, nullptr, st))) return rc;
  // S: 2xLSTM(K->Hb->Hb) + Linear(1) + ReLU on B*M rows over Ts steps (model.py:188-189)
  const int Hb = d->bn_hidden;
  int bn_bstride = M;
  if (fast_is_tc(d)) {
    // tensor-core kernel of the fullsubnet sub-band stack: same stack shape (K<=32 -> 384 -> 384), the gather
    // does the unfold AND the time down-sampling on the fly from melT / encT, Linear output 1 of 2 is zero-padded
    FSN_REQUIRE(wt->bn_packed && fast_tc_ok(d), FSN_ERR_UNSUPPORTED,
                "fast model: the tensor-core precisions need packed bottleneck weights, bn_hidden = 384 and input width <= 32");
    SbTcArgs a;
    memset(&a, 0, sizeof(a));
    a.packed = wt->bn_packed; a.magT = w.melT; a.fbT = w.encT; a.inv2 = w.inv2; a.crm = w.bn_out;
    a.B = B; a.F = M; a.Tp = Tp; a.la = 0; a.Ns = d->noisy_num_neighbors; a.Nf = d->enc_num_neighbors;
    a.H = Hb; a.act = FSN_ACT_RELU; a.steps = m.Ts; a.shrink = m.S; a.x3 = fast_x3(d);
    a.map = RowMap{B, M, M, 1};
    if ((rc = sb_tc_forward(a, st))) return rc;
    bn_bstride = 2 * M;
  } else {
  for (int t = 0; t < m.Ts; ++t) {
    StepParams p;
    memset(&p, 0, sizeof(p));
    p.R = R; p.first = (t == 0);
    p.K0 = m.K; p.H = Hb;
    p.w_ih = wt->bn[0].w_ih; p.w_hh = wt->bn[0].w_hh; p.b_ih = wt->bn[0].b_ih; p.b_hh = wt->bn[0].b_hh;
    p.h_prev = w.bn_h0[(t + 1) & 1]; p.h_prev_stride = Hb;
    p.h_out = w.bn_h0[t & 1]; p.h_out_stride = Hb;
    p.c = w.bn_c0;
    p.x0 = w.bn + (size_t)t * R * m.K; p.x0_row_stride = m.K; p.row_scale = w.inv2; p.row_scale_div = M;
    if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
    p.K0 = Hb;
    p.w_ih = wt->bn[1].w_ih; p.w_hh = wt->bn[1].w_hh; p.b_ih = wt->bn[1].b_ih; p.b_hh = wt->bn[1].b_hh;
    p.x0 = w.bn_h0[t & 1]; p.x0_row_stride = Hb; p.row_scale = nullptr; p.row_scale_div = 0;
    p.h_prev = w.bn_h1[(t + 1) & 1]; p.h_prev_stride = Hb;
    p.h_out = w.bn_h1[t & 1]; p.h_out_stride = Hb;
    p.c = w.bn_c1;
    if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
    if ((rc = rows_fc_launch(w.bn_h1[t & 1], R, Hb, wt->bn_fc_w, wt->bn_fc_b, 1, FSN_ACT_RELU, w.bn_out + t,
                             (size_t)m.Ts, 0, st)))
      return rc;
  }
  }
  // up-sampling + concat with the encoder output (model.py:191-194)
  {
    const size_t n = (size_t)B * Tp * 2 * M;
    int g = (int)((n + 255) / 256);
    if (g > 132 * 16) g = 132 * 16;
    fast_dec_input_kernel<<<g, 256, 0, st>>>(w.encT, w.bn_out, bn_bstride, B, Tp, M, m.S, m.Ts, w.dec_in);
    FSN_CHECK_LAUNCH("fast_dec_input_kernel");
  }
  // F_m2l: LSTM(2M->Hd), LSTM(Hd->Hd) + Linear(2F) (model.py:77-96,196)
  if ((rc = run_lstm_pair(wt->dec1, 2 * M, d->dec_hidden, wt->dec2, d->dec_hidden, B, Tp, w.dec_in, (size_t)Tp * 2 * M,
                          2 * M, nullptr, w.d1_h, w.d1_c, w.d2_hall, w.d2_c, w.pp, w.barrier, st, (lstm_tc && (tc_mask & 4)) ? &w.tc : nullptr,
                          w.tc_mid, fast_x3(d))))
    return rc;
  if (lstm_tc && (tc_mask & 8)) {
    if ((rc = linear_tc(w.d2_hall, (size_t)d->dec_hidden, d->dec_hidden, wt->dec_fc_w, wt->dec_fc_b, 2 * F, FSN_ACT_NONE,
                        w.dec_out, (size_t)2 * F, (size_t)B * Tp, fast_x3(d), w.tc, st)))
      return rc;
  } else if ((rc = fc_gemm_launch(w.d2_hall, wt->dec_fc_w, wt->dec_fc_b, w.dec_out, B * Tp, d->dec_hidden, 2 * F, FSN_ACT_NONE,
                                  st))) {
    return rc;
  }
  dim3 grid(cdiv(T, 32), cdiv(F, 32), B * 2);
  fast_output_kernel<<<grid, dim3(32, 8), 0, st>>>(w.dec_out, B, Tp, F, d->look_ahead, out);
  FSN_CHECK_LAUNCH("fast_output_kernel");
  return FSN_OK;
}
