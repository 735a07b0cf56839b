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

// encoder / decoder pair over B rows of Tp steps; on the tensor cores with the tensor-core precisions when all three
// encoder / decoder hidden sizes are supported there.  dec = false: F_l2m, LSTM(M -> He1), LSTM(He1 -> He2) + Linear(M) +
// ReLU (model.py:35-54,171), per-step scale with the cumulative norm; dec: F_m2l, LSTM(2M -> Hd), LSTM(Hd -> Hd) +
// Linear(2F) (model.py:77-96,196)
static SeqStack fast_pair(const fsn_fast_desc* d, int B, int Tp, bool dec) {
  SeqStack s;
  memset(&s, 0, sizeof(s));
  const int M = d->num_mels;
  s.R = B; s.Tp = Tp; s.n = 2;
  if (dec) {
    s.K0 = 2 * M; s.H[0] = s.H[1] = d->dec_hidden; s.O = 2 * d->num_freqs; s.act = FSN_ACT_NONE;
  } else {
    s.K0 = M; s.H[0] = d->enc1_hidden; s.H[1] = d->enc2_hidden; s.O = M; s.act = FSN_ACT_RELU;
    s.step_scale = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE;
  }
  s.x3 = fast_x3(d);
  s.tc = fast_is_tc(d) && lstm_rec_tc_supported(d->enc1_hidden, s.x3) && lstm_rec_tc_supported(d->enc2_hidden, s.x3) &&
         lstm_rec_tc_supported(d->dec_hidden, s.x3);
  return s;
}

// the encoder and the decoder run one after the other on one stack workspace, carved for the larger of the two
static SeqStack fast_pair_ws(const fsn_fast_desc* d, int B, int Tp) {
  auto mx = [](int a, int b) { return a > b ? a : b; };
  SeqStack s = fast_pair(d, B, Tp, true);
  s.H[0] = mx(d->enc1_hidden, d->dec_hidden); s.H[1] = mx(d->enc2_hidden, d->dec_hidden); s.O = mx(d->num_mels, s.O);
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
  seq_stack_carve(c, fast_pair_ws(d, m.B, m.Tp), w.seq);
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
  if ((rc = layout_clips_check(B, true, "fast model"))) return rc;
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
  // F_l2m (model.py:171)
  SeqStack enc = fast_pair(d, B, Tp, false);
  enc.L[0] = wt->enc1; enc.L[1] = wt->enc2;
  enc.x = w.melT; enc.scale = m.cum ? w.cum1 : w.inv1;
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
  // F_m2l (model.py:196)
  SeqStack dec = fast_pair(d, B, Tp, true);
  dec.L[0] = wt->dec1; dec.L[1] = wt->dec2;
  dec.x = w.dec_in; dec.fc_w = wt->dec_fc_w; dec.fc_b = wt->dec_fc_b; dec.out = w.dec_out;
  if ((rc = seq_stack_forward(dec, w.seq, st))) return rc;
  return crm_output_launch(w.dec_out, (size_t)Tp * 2 * F, 2 * F, B, Tp, F, d->look_ahead, out, st);
}

// ---- chunked streaming (DESIGN 4.14).  Slot state block: the stream header (StreamSlot), then the last S-1 frames of
// the mel spectrogram and of the encoder output (M each), encoder (h | c) of both layers, the second norm's running sum
// and the latest bottleneck output of the M rows, bottleneck (h | c) of both layers (M x Hb each), decoder (h | c) of
// both layers.  The tensor-core stream (fsn_fast_stream_tc_*, DESIGN 4.14.2) keeps the same block; its bottleneck is one
// sb_phased_lstm_tc_kernel launch over all block ends of the call instead of the per-step loop.
namespace fsn {

struct FastStreamLayout : StreamSlot { size_t mel, enc, eh, ec, run, bo, bh, bc, dh, dc; };

static FastStreamLayout fast_stream_layout(const fsn_fast_desc* d, const StreamGeom& g) {
  const size_t M = d->num_mels, Hm = d->shrink_size - 1;
  const size_t He = (size_t)d->enc1_hidden + d->enc2_hidden, Hb = 2 * M * d->bn_hidden, Hd = 2 * (size_t)d->dec_hidden;
  FastStreamLayout s{StreamSlot(g, d->num_freqs)};
  s.mel = s.sec(Hm * M); s.enc = s.sec(Hm * M);
  s.eh = s.sec(He); s.ec = s.sec(He);
  s.run = s.sec(M); s.bo = s.sec(M);
  s.bh = s.sec(Hb); s.bc = s.sec(Hb);
  s.dh = s.sec(Hd); s.dc = s.sec(Hd);
  return s;
}

// tc: the tensor-core stream (fsn_fast_stream_tc_*), which takes FSN_PREC_F16X3_TC / FSN_PREC_F16_TC instead of
// FSN_PREC_FP32 and the bottleneck shapes the wgmma kernel takes
static int fast_stream_check(const fsn_fast_desc* d, int n_fft, int hop, int win_length, FastDims& m, StreamGeom& g,
                             bool tc = false) {
  int rc = fast_dims(d, 1, 2, m);
  if (rc) return rc;
  FSN_REQUIRE(d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE, FSN_ERR_UNSUPPORTED,
              "fast_stream: the offline norm needs the whole clip; streaming is built for cumulative_laplace_norm");
  if (tc) {
    FSN_REQUIRE(fast_is_tc(d), FSN_ERR_UNSUPPORTED,
                "fast_stream_tc: the tensor-core stream is built for FSN_PREC_F16X3_TC and FSN_PREC_F16_TC (precision %d); "
                "the fp32 kernels stream through fsn_fast_stream_step", d->precision);
    FSN_REQUIRE(fast_tc_ok(d), FSN_ERR_UNSUPPORTED,
                "fast_stream_tc: the tensor-core bottleneck needs bn_hidden = 384, 2 layers and input width <= 32");
  } else {
    FSN_REQUIRE(d->precision == FSN_PREC_FP32, FSN_ERR_UNSUPPORTED,
                "fast_stream: streaming is built for FSN_PREC_FP32 (precision %d)", d->precision);
  }
  FSN_REQUIRE(n_fft / 2 + 1 == d->num_freqs, FSN_ERR_SHAPE, "fast_stream: n_fft/2+1 = %d != num_freqs = %d", n_fft / 2 + 1,
              d->num_freqs);
  return stream_geom(n_fft, hop, win_length, d->look_ahead, g);
}

struct FastStreamWs : StreamWs {
  int* rst;
  float *melT, *scale1, *encT, *catM, *catE, *bn, *scale2, *bo, *dec_in, *y;
  float2* fs;
  StreamStackWs stack;                        // encoder and decoder, one after the other
  float *bh0[2], *bh1[2], *bc0, *bc1;         // bottleneck state, h ping-pong per layer (fp32 stream)
  float* x;                                   // tensor-core stream: the bottleneck's scaled input [nb, R, K]
  int *sb_rst, *store;                        // ... and per slot its restart step (0 or none) and its store step
};

// element (b, m, col) of the bottleneck outputs bo at b bs + m ms + col cs; column 0 is the output carried into the call,
// column i + 1 that of bottleneck step i.  fp32 stream: [B, M, nb + 1]; tensor-core stream: the frame-major [B, nb + 1, 2M]
// the sub-band kernel's carry output writes (its second, zero-padded output row at columns M .. 2M)
struct BoGeom { size_t bs, ms, cs; };
static BoGeom fast_bo_geom(bool tc, int M, int nb) {
  return tc ? BoGeom{(size_t)(nb + 1) * 2 * M, 1, 2 * (size_t)M} : BoGeom{(size_t)M * (nb + 1), (size_t)nb + 1, 1};
}

// St = K + E steps: a call with a clip's last chunk runs E steps past the K of the others; nb = ceil(St / S) bottleneck
// steps, the most block ends St consecutive frames can hold.  tc: the bottleneck's state stays in the slot state (no
// per-row buffers), its input is carved instead.  Returns the bytes
static size_t fast_stream_carve(const fsn_fast_desc* d, const FastDims& m, const StreamGeom& g, int B, int K, void* base,
                                FastStreamWs& w, bool tc = false) {
  Carver c(base);
  const size_t F = m.F, M = m.M, St = (size_t)K + g.E, Hm = m.S - 1, nb = cdiv((int)St, m.S), R = (size_t)B * M;
  const size_t Hb = d->bn_hidden;
  stream_carve(c, g, B, K, m.F, w);
  w.rst = c.take<int>(B);
  w.melT = c.take<float>(B * St * M);
  w.fs = c.take<float2>(B * St);
  w.scale1 = c.take<float>(St * B);
  stream_stack_carve(c, fast_pair_ws(d, B, (int)St), w.stack);
  w.encT = c.take<float>(B * St * M);
  w.catM = c.take<float>(B * (Hm + St) * M);
  w.catE = c.take<float>(B * (Hm + St) * M);
  w.bn = c.take<float>(nb * R * m.K);
  w.scale2 = c.take<float>(nb * R);
  memset(w.bh0, 0, sizeof(w.bh0)); memset(w.bh1, 0, sizeof(w.bh1));
  w.bc0 = w.bc1 = w.x = nullptr;
  w.sb_rst = w.store = nullptr;
  if (tc) {
    w.bo = c.take<float>(R * 2 * (nb + 1));
    w.x = c.take<float>(nb * R * m.K);
    w.sb_rst = c.take<int>(B);
    w.store = c.take<int>(B);
  } else {
    w.bo = c.take<float>(R * (nb + 1));
    for (int i = 0; i < 2; ++i) { w.bh0[i] = c.take<float>(R * Hb); w.bh1[i] = c.take<float>(R * Hb); }
    w.bc0 = c.take<float>(R * Hb); w.bc1 = c.take<float>(R * Hb);
  }
  w.dec_in = c.take<float>(B * St * 2 * M);
  w.y = c.take<float>(B * St * 2 * F);
  return c.off;
}

// Block ends of slot b in the call: the steps j < St whose frame m0 + j is a multiple of S and >= 0 (block m/S, shrunk
// step m/S of the whole clip, is complete at frame m).  First such step, and how many lie in [0, lim).
__device__ __forceinline__ int fs_first_end(int m0, int S) {
  const int m = m0 > 0 ? m0 : 0;
  return (m + S - 1) / S * S - m0;
}
__device__ __forceinline__ int fs_ends_before(int jf, int S, int lim) { return lim > jf ? (lim - 1 - jf) / S + 1 : 0; }

// Before the bottleneck: per slot b (grid.y), the bottleneck's h / c entering the call into h0p / h1p (the ping-pong
// halves step 0 reads) and c0 / c1, zero when the clip's frame 0 is in the call (its first block end is block 0); the
// latest bottleneck output into column 0 of bo; the decoder's restart step rst[b] (frame 0 at step rst).  Tensor-core
// stream (h0p null, sb_rst non-null): the kernel reads h / c from the state itself, so instead its restart step sb_rst[b]
// (0 when the first block end is block 0, else none) and its store step store[b] (fast_stream_commit_kernel's rule)
__global__ void fast_stream_open_kernel(const int* __restrict__ pos0, const int* __restrict__ act0, int hop, int c, int St,
                                        int K, int S, int M, int Hb, const char* __restrict__ state, size_t slot_bytes,
                                        size_t bh, size_t bc, size_t bo_off, float* __restrict__ h0p, float* __restrict__ h1p,
                                        float* __restrict__ c0, float* __restrict__ c1, float* __restrict__ bo,
                                        const BoGeom bg, int* __restrict__ rst, int* __restrict__ sb_rst,
                                        int* __restrict__ store) {
  const int b = blockIdx.y;
  const int m0 = pos0[b] / hop - c;
  const bool fresh = m0 <= 0 && -m0 < St;
  const size_t n = (size_t)M * Hb, o = (size_t)b * n;
  const char* sb = state + (size_t)b * slot_bytes;
  const float* sh = reinterpret_cast<const float*>(sb + bh);
  const float* sc = reinterpret_cast<const float*>(sb + bc);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; h0p && e < n; e += (size_t)gridDim.x * blockDim.x) {
    h0p[o + e] = fresh ? 0.f : sh[e];
    h1p[o + e] = fresh ? 0.f : sh[n + e];
    c0[o + e] = fresh ? 0.f : sc[e];
    c1[o + e] = fresh ? 0.f : sc[n + e];
  }
  if (blockIdx.x == 0) {
    const float* sbo = reinterpret_cast<const float*>(sb + bo_off);
    for (int r = threadIdx.x; r < M; r += blockDim.x) bo[(size_t)b * bg.bs + (size_t)r * bg.ms] = sbo[r];
    if (threadIdx.x == 0) {
      rst[b] = -m0;
      if (sb_rst) {
        sb_rst[b] = fresh ? 0 : -1;
        store[b] = act0[b] ? fs_ends_before(fs_first_end(m0, S), S, K) - 1 : -1;
      }
    }
  }
}

// Bottleneck input of the i-th block end of slot b (grid (nb, B)): fast_bn_input_kernel's arithmetic on the block's frames,
// read from catM / catE [B, S-1+St, M] (the carried S-1 frames, then the call's), into bn [nb, B*M, K]; 0 past the slot's
// last block end in the call.  scale non-null (the tensor-core stream): the input the sub-band kernel's gather forms
// with `shrink`, the block sum times (1/len * scale [nb, B*M] of the row), instead of the block mean
__global__ void fast_stream_bn_input_kernel(const float* __restrict__ catM, const float* __restrict__ catE,
                                            const int* __restrict__ pos0, int hop, int c, int St, int M, int Nn, int Ne,
                                            int S, float* __restrict__ bn, const float* __restrict__ scale) {
  const int i = blockIdx.x, b = blockIdx.y, B = gridDim.y;
  const int K = (2 * Nn + 1) + (2 * Ne + 1);
  const int m0 = pos0[b] / hop - c;
  const int j = fs_first_end(m0, S) + i * S;
  const bool ok = j < St;
  const int len = (m0 + j == 0) ? 1 : S;  // block 0 is frame 0 alone (model.py real_time_downsampling)
  const float inv = 1.0f / (float)len;
  const size_t W = (size_t)(S - 1 + St);
  const int q0 = S - 1 + j - (len - 1);  // first frame of the block in the cat rows
  for (int idx = threadIdx.x; idx < M * K; idx += blockDim.x) {
    const int mm = idx / K, k = idx - mm * K;
    float v = 0.f;
    if (ok) {
      float acc = 0.f;
      for (int q = q0; q < q0 + len; ++q) {
        const size_t base = ((size_t)b * W + q) * M;
        acc += (k < 2 * Nn + 1) ? catM[base + reflect_idx(mm + k - Nn, M)]
                                : catE[base + reflect_idx(mm + (k - (2 * Nn + 1)) - Ne, M)];
      }
      v = scale ? acc * (inv * scale[(size_t)i * B * M + (size_t)b * M + mm]) : acc * inv;
    }
    bn[((size_t)i * B * M + (size_t)b * M + mm) * K + k] = v;
  }
}

// Second cumulative norm over the call's block ends: fast_cum_bn_scale_kernel's recurrence per row r = b*M + mm with the
// running sum carried in the slot state (reset at block 0, stored as of the last block end before step K); scaleT [nb, R]
__global__ void fast_stream_bn_scale_kernel(const float* __restrict__ bn, const int* __restrict__ pos0,
                                            const int* __restrict__ act0, int hop, int c, int St, int K, int R, int M, int Kf,
                                            int S, int nb, float eps, char* __restrict__ state, size_t slot_bytes,
                                            size_t run_off, float* __restrict__ scaleT) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int b = r / M, mm = r - b * M;
  float* srun = reinterpret_cast<float*>(state + (size_t)b * slot_bytes + run_off) + mm;
  const int m0 = pos0[b] / hop - c, jf = fs_first_end(m0, S);
  const int commit = act0[b] ? fs_ends_before(jf, S, K) - 1 : -1;
  float run = *srun;
  for (int i = 0; i < nb; ++i) {
    const int j = jf + i * S;
    float sc = 1.f;
    if (j < St) {
      const int ts = (m0 + j) / S;
      if (ts == 0) run = 0.f;
      const float* x = bn + ((size_t)i * R + r) * Kf;
      float s = 0.f;
      for (int k = 0; k < Kf; ++k) s += x[k];
      run += s;
      sc = 1.0f / (run / ((float)Kf * (float)(ts + 1)) + eps);
    }
    scaleT[(size_t)i * R + r] = sc;
    if (i == commit) *srun = run;
  }
}

// After bottleneck step i: the slots whose last block end before step K is their i-th store the bottleneck's (h, c) and
// output (column i + 1 of bo) in their state
__global__ void fast_stream_commit_kernel(const int* __restrict__ pos0, const int* __restrict__ act0, int hop, int c, int K,
                                          int S, int M, int Hb, int nb, int i, const float* __restrict__ h0,
                                          const float* __restrict__ h1, const float* __restrict__ c0,
                                          const float* __restrict__ c1, const float* __restrict__ bo, char* __restrict__ state,
                                          size_t slot_bytes, size_t bh, size_t bc, size_t bo_off) {
  const int b = blockIdx.y;
  if (!act0[b] || fs_ends_before(fs_first_end(pos0[b] / hop - c, S), S, K) - 1 != i) return;
  const size_t n = (size_t)M * Hb, o = (size_t)b * n;
  char* sb = state + (size_t)b * slot_bytes;
  float* sh = reinterpret_cast<float*>(sb + bh);
  float* sc = reinterpret_cast<float*>(sb + bc);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    sh[e] = h0[o + e]; sh[n + e] = h1[o + e];
    sc[e] = c0[o + e]; sc[n + e] = c1[o + e];
  }
  if (blockIdx.x == 0) {
    float* sbo = reinterpret_cast<float*>(sb + bo_off);
    for (int r = threadIdx.x; r < M; r += blockDim.x) sbo[r] = bo[((size_t)b * M + r) * (nb + 1) + i + 1];
  }
}

// Tensor-core stream, after the bottleneck: slot b (block b) stores the output of its store step store[b] as its latest
// bottleneck output (the sub-band kernel stored its (h, c) after that step)
__global__ void fast_stream_bo_store_kernel(const int* __restrict__ store, int M, const float* __restrict__ bo,
                                            const BoGeom bg, char* __restrict__ state, size_t slot_bytes, size_t bo_off) {
  const int b = blockIdx.x, i = store[b];
  if (i < 0) return;
  float* sbo = reinterpret_cast<float*>(state + (size_t)b * slot_bytes + bo_off);
  for (int r = threadIdx.x; r < M; r += blockDim.x) sbo[r] = bo[(size_t)b * bg.bs + (size_t)r * bg.ms + (size_t)(i + 1) * bg.cs];
}

// Decoder input (fast_dec_input_kernel's concatenation): dec_in [B, St, 2M] row (b, j) = encoder output of step j | the
// bottleneck output of the latest block end at or before step j (column 0 of bo: the one carried into the call)
__global__ void fast_stream_dec_input_kernel(const float* __restrict__ encT, const float* __restrict__ bo, const BoGeom bg,
                                             const int* __restrict__ pos0, int hop, int c, int B, int St, int M, int S,
                                             float* __restrict__ dec_in) {
  const size_t n = (size_t)B * St * 2 * M;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int col = (int)(i % (2 * M));
    const size_t q = i / (2 * M);
    const int b = (int)(q / St), j = (int)(q % St);
    if (col < M) {
      dec_in[i] = encT[q * M + col];
    } else {
      const int e = fs_ends_before(fs_first_end(pos0[b] / hop - c, S), S, j + 1);
      dec_in[i] = bo[(size_t)b * bg.bs + (size_t)(col - M) * bg.ms + (size_t)e * bg.cs];
    }
  }
}

}  // namespace fsn

namespace fsn {

static size_t fast_stream_state_query(const fsn_fast_desc* d, int B, int n_fft, int hop, bool tc) {
  FastDims m;
  StreamGeom g;
  return stream_query_check(fast_stream_check(d, n_fft, hop, n_fft, m, g, tc), tc ? "fast_stream_tc" : "fast_stream", B, 1)
             ? 0 : fast_stream_layout(d, g).slot() * (size_t)B;
}

static size_t fast_stream_workspace_query(const fsn_fast_desc* d, int B, int K_max, int n_fft, int hop, bool tc) {
  FastDims m;
  StreamGeom g;
  FastStreamWs w;
  return stream_query_check(fast_stream_check(d, n_fft, hop, n_fft, m, g, tc), tc ? "fast_stream_tc" : "fast_stream", B,
                            K_max)
             ? 0 : fast_stream_carve(d, m, g, B, K_max, nullptr, w, tc);
}

static int fast_stream_delay_query(const fsn_fast_desc* d, int n_fft, int hop, bool tc) {
  FastDims m;
  StreamGeom g;
  return stream_delay(fast_stream_check(d, n_fft, hop, n_fft, m, g, tc), g);
}

// one call of either stream.  tc: the encoder and decoder on the path the whole-clip call takes (SEQ_PATH_TC with the
// restart table stream_open writes), and the bottleneck in one sb_phased_lstm_tc_kernel launch over all nb steps of
// every row, its input formed first by fast_stream_bn_input_kernel with the second norm's scales
static int fast_stream_run(const fsn_fast_desc* d, const fsn_fast_weights* wt, bool tc, const float* wav,
                           const int32_t* start, const int32_t* tail, int B, int K, int n_fft, int hop, int win_length,
                           float* enhanced, void* state, size_t state_bytes, void* workspace, size_t workspace_bytes,
                           cudaStream_t st) {
  launch_counter() = 0;
  FastDims m;
  StreamGeom g;
  int St, rc = fast_stream_check(d, n_fft, hop, win_length, m, g, tc);
  if (rc || (rc = stream_check(tc ? "fast_stream_tc" : "fast_stream", g, B, K, tail, wav, enhanced, St))) return rc;
  FSN_REQUIRE(wt, FSN_ERR_SHAPE, "fast_stream: null weights");
  FSN_REQUIRE(!tc || wt->bn_packed, FSN_ERR_SHAPE,
              "fast_stream_tc: the tensor-core stream needs the packed bottleneck weights (fsn_fast_pack_bn_weights)");
  const FastStreamLayout sl = fast_stream_layout(d, g);
  FastStreamWs w;
  const size_t ws = fast_stream_carve(d, m, g, B, K, workspace, w, tc);
  if ((rc = stream_check_sizes(state, state_bytes, sl.slot(), B, workspace, workspace_bytes, ws))) return rc;
  char* sb = (char*)state;
  const size_t ss = sl.slot();
  const int F = m.F, M = m.M, S = m.S, Kf = m.K, Hm = S - 1, R = B * M, nb = cdiv(St, S);
  const int Hb = d->bn_hidden;
  const size_t catw = (size_t)(Hm + St) * M * 4;
  if ((rc = stream_open(g, sl, w, F, B, K, St, win_length, start, tail, wav, sb, tc ? w.rst : nullptr, st))) return rc;
  // Mel filtering and the first norm over the mel frame sums (model.py:161-170)
  if ((rc = fc_gemm_launch(w.magT, wt->mel_fb, nullptr, w.melT, B * St, F, M, FSN_ACT_NONE, st, /*w_kmajor=*/true))) return rc;
  if ((rc = frame_stats_launch(w.melT, B, St, M, 0, (size_t)St * M, M, w.fs, st))) return rc;
  if ((rc = stream_norm_launch(w.fs, B, St, K, M, g, d->norm_type, w.pos0, w.act0, w.tail, sb, ss, w.scale1, st))) return rc;
  // encoder, (h, c) carried.  fp32: its per-step scale keeps it off the paths that read the restart table, which
  // fast_stream_open_kernel writes only later in the call; tc: on SEQ_PATH_TC it reads the table stream_open wrote
  SeqStack enc = fast_pair(d, B, St, false);
  enc.L[0] = wt->enc1; enc.L[1] = wt->enc2;
  enc.x = w.melT; enc.scale = w.scale1; enc.fc_w = wt->enc_fc_w; enc.fc_b = wt->enc_fc_b; enc.out = w.encT;
  if ((rc = stream_seq_stack(enc, w.stack, StackCarry{sb, ss, sl.eh, sl.ec, w.pos0, g, tc ? w.rst : nullptr, K}, st)))
    return rc;
  // the carried S-1 frames, then the call's, of the mel spectrogram and the encoder output: the frames the blocks average
  if (Hm > 0) {
    if ((rc = copy_rows(w.catM, catw, sb + sl.mel, ss, (size_t)Hm * M * 4, B, st))) return rc;
    if ((rc = copy_rows(w.catE, catw, sb + sl.enc, ss, (size_t)Hm * M * 4, B, st))) return rc;
  }
  if ((rc = copy_rows(w.catM + (size_t)Hm * M, catw, w.melT, (size_t)St * M * 4, (size_t)St * M * 4, B, st))) return rc;
  if ((rc = copy_rows(w.catE + (size_t)Hm * M, catw, w.encT, (size_t)St * M * 4, (size_t)St * M * 4, B, st))) return rc;
  // bottleneck: one step per block end, every row at its slot's i-th block end of the call (model.py:174-189)
  const BoGeom bg = fast_bo_geom(tc, M, nb);
  const dim3 sgrid(tc ? 1 : cdiv(M * Hb, 256), B);
  fast_stream_open_kernel<<<sgrid, 256, 0, st>>>(w.pos0, w.act0, hop, g.c, St, K, S, M, Hb, sb, ss, sl.bh, sl.bc, sl.bo,
                                                w.bh0[1], w.bh1[1], w.bc0, w.bc1, w.bo, bg, w.rst, w.sb_rst, w.store);
  FSN_CHECK_LAUNCH("fast_stream_open_kernel");
  fast_stream_bn_input_kernel<<<dim3(nb, B), 256, 0, st>>>(w.catM, w.catE, w.pos0, hop, g.c, St, M, d->noisy_num_neighbors,
                                                            d->enc_num_neighbors, S, w.bn, nullptr);
  FSN_CHECK_LAUNCH("fast_stream_bn_input_kernel");
  fast_stream_bn_scale_kernel<<<cdiv(R, 128), 128, 0, st>>>(w.bn, w.pos0, w.act0, hop, g.c, St, K, R, M, Kf, S, nb,
                                                             TRAIN_CUM_EPS, sb, ss, sl.run, w.scale2);
  FSN_CHECK_LAUNCH("fast_stream_bn_scale_kernel");
  if (tc) {
    // the input the whole-clip gather forms for each block, then all nb steps in one launch: (h, c) from and back to the
    // state, step i's output (and the zero-padded second one) into column i + 1 of bo
    fast_stream_bn_input_kernel<<<dim3(nb, B), 256, 0, st>>>(w.catM, w.catE, w.pos0, hop, g.c, St, M,
                                                              d->noisy_num_neighbors, d->enc_num_neighbors, S, w.x, w.scale2);
    FSN_CHECK_LAUNCH("fast_stream_bn_input_kernel");
    SbTcArgs a;
    memset(&a, 0, sizeof(a));
    a.packed = wt->bn_packed; a.crm = w.bo;
    a.B = B; a.F = M; a.Tp = nb; a.la = 0; a.Ns = d->noisy_num_neighbors; a.Nf = d->enc_num_neighbors; a.H = Hb;
    a.act = FSN_ACT_RELU; a.x3 = fast_x3(d); a.map = RowMap{B, M, M, 1};
    const SbCarry io{(float*)(sb + sl.bh), (float*)(sb + sl.bc), ss / 4, (size_t)M * Hb, M, w.sb_rst, -1, bg.bs, 1, w.x,
                     w.store};
    if ((rc = sb_tc_carry_forward(a, io, st))) return rc;
    fast_stream_bo_store_kernel<<<B, 64, 0, st>>>(w.store, M, w.bo, bg, sb, ss, sl.bo);
    FSN_CHECK_LAUNCH("fast_stream_bo_store_kernel");
  } else {
    for (int i = 0; i < nb; ++i) {
      StepParams p;
      memset(&p, 0, sizeof(p));
      p.R = R; p.K0 = Kf; p.H = Hb;
      p.w_ih = wt->bn[0].w_ih; p.w_hh = wt->bn[0].w_hh; p.b_ih = wt->bn[0].b_ih; p.b_hh = wt->bn[0].b_hh;
      p.x0 = w.bn + (size_t)i * R * Kf; p.x0_row_stride = Kf;
      p.row_scale = w.scale2 + (size_t)i * R; p.row_scale_div = 1;
      p.h_prev = w.bh0[(i + 1) & 1]; p.h_out = w.bh0[i & 1]; p.h_prev_stride = p.h_out_stride = Hb;
      p.c = w.bc0;
      if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
      p.K0 = Hb;
      p.w_ih = wt->bn[1].w_ih; p.w_hh = wt->bn[1].w_hh; p.b_ih = wt->bn[1].b_ih; p.b_hh = wt->bn[1].b_hh;
      p.x0 = w.bh0[i & 1]; p.x0_row_stride = Hb; p.row_scale = nullptr; p.row_scale_div = 0;
      p.h_prev = w.bh1[(i + 1) & 1]; p.h_out = w.bh1[i & 1];
      p.c = w.bc1;
      if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
      if ((rc = sb_head_launch(w.bh1[i & 1], R, Hb, 1, wt->bn_fc_w, wt->bn_fc_b, 1, FSN_ACT_RELU, w.bo,
                               HeadGeom{R, 1, 0, 0, (size_t)nb + 1}, i + 1, st)))
        return rc;
      fast_stream_commit_kernel<<<sgrid, 256, 0, st>>>(w.pos0, w.act0, hop, g.c, K, S, M, Hb, nb, i, w.bh0[i & 1],
                                                       w.bh1[i & 1], w.bc0, w.bc1, w.bo, sb, ss, sl.bh, sl.bc, sl.bo);
      FSN_CHECK_LAUNCH("fast_stream_commit_kernel");
    }
  }
  // decoder input: encoder output | up-sampled bottleneck output (model.py:191-194)
  fast_stream_dec_input_kernel<<<ew_grid((size_t)B * St * 2 * M), 256, 0, st>>>(w.encT, w.bo, bg, w.pos0, hop, g.c, B, St, M,
                                                                                 S, w.dec_in);
  FSN_CHECK_LAUNCH("fast_stream_dec_input_kernel");
  // decoder, (h, c) carried, restarting at rst
  SeqStack dec = fast_pair(d, B, St, true);
  dec.L[0] = wt->dec1; dec.L[1] = wt->dec2;
  dec.x = w.dec_in; dec.fc_w = wt->dec_fc_w; dec.fc_b = wt->dec_fc_b; dec.out = w.y;
  if ((rc = stream_seq_stack(dec, w.stack, StackCarry{sb, ss, sl.dh, sl.dc, w.pos0, g, w.rst, K}, st))) return rc;
  // carry the last S-1 frames of the mel spectrogram and the encoder output as of step K
  if (Hm > 0) {
    if ((rc = copy_rows(sb + sl.mel, ss, w.catM + (size_t)K * M, catw, (size_t)Hm * M * 4, B, st))) return rc;
    if ((rc = copy_rows(sb + sl.enc, ss, w.catE + (size_t)K * M, catw, (size_t)Hm * M * 4, B, st))) return rc;
  }
  return stream_close(g, sl, w, F, B, K, St, win_length, w.y, enhanced, sb, st);
}

}  // namespace fsn

extern "C" size_t fsn_fast_stream_state_bytes(const fsn_fast_desc* d, int B, int n_fft, int hop) {
  return fast_stream_state_query(d, B, n_fft, hop, false);
}

extern "C" size_t fsn_fast_stream_workspace_bytes(const fsn_fast_desc* d, int B, int K_max, int n_fft, int hop) {
  return fast_stream_workspace_query(d, B, K_max, n_fft, hop, false);
}

extern "C" int fsn_fast_stream_delay(const fsn_fast_desc* d, int n_fft, int hop) {
  return fast_stream_delay_query(d, n_fft, hop, false);
}

extern "C" int fsn_fast_stream_step(const fsn_fast_desc* d, const fsn_fast_weights* wt, const float* wav,
                                    const int32_t* start, const int32_t* tail, int B, int K, int n_fft, int hop,
                                    int win_length, float* enhanced, void* state, size_t state_bytes, void* workspace,
                                    size_t workspace_bytes, fsn_stream_t stream) {
  return fast_stream_run(d, wt, false, wav, start, tail, B, K, n_fft, hop, win_length, enhanced, state, state_bytes,
                         workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" size_t fsn_fast_stream_tc_state_bytes(const fsn_fast_desc* d, int B, int n_fft, int hop) {
  return fast_stream_state_query(d, B, n_fft, hop, true);
}

extern "C" size_t fsn_fast_stream_tc_workspace_bytes(const fsn_fast_desc* d, int B, int K_max, int n_fft, int hop) {
  return fast_stream_workspace_query(d, B, K_max, n_fft, hop, true);
}

extern "C" int fsn_fast_stream_tc_delay(const fsn_fast_desc* d, int n_fft, int hop) {
  return fast_stream_delay_query(d, n_fft, hop, true);
}

extern "C" int fsn_fast_stream_tc_step(const fsn_fast_desc* d, const fsn_fast_weights* wt, const float* wav,
                                       const int32_t* start, const int32_t* tail, int B, int K, int n_fft, int hop,
                                       int win_length, float* enhanced, void* state, size_t state_bytes, void* workspace,
                                       size_t workspace_bytes, fsn_stream_t stream) {
  return fast_stream_run(d, wt, true, wav, start, tail, B, K, n_fft, hop, win_length, enhanced, state, state_bytes,
                         workspace, workspace_bytes, (cudaStream_t)stream);
}

// unit-test hook (tests/test_gpu_fast_stream_tc.py): the block-phased bottleneck on caller inputs.  B slots of M rows
// (rows b M + m); slot b's call step j is frame m0[b] + j of its clip, and row q of catM / catE [B, S-1+St, M] is call
// step q - (S-1).  fast_stream_bn_input_kernel forms the input of the nb = ceil(St / S) block ends into x [nb, B M, K] with
// the scales scale [nb, B M], then sb_phased_lstm_tc_kernel runs: h / c [2, B M, H] hold the state entering step 0 and
// receive slot b's state after step store[b] (-1: none); slot b enters step restart[b] with zero state; step i's output
// of row b M + m goes to out [B, nb, 2M] at (b, i, m) (and the zero-padded second output at (b, i, M + m)).  m0, restart
// and store are device tables [B]
extern "C" int fsn_debug_sb_lstm_tc_phased(const fsn_seq_weights* bn, int H, int Ns, int Nf, int x3, const float* catM,
                                           const float* catE, int B, int M, int S, int St, const int32_t* m0,
                                           const float* scale, const int32_t* restart, const int32_t* store, float* h,
                                           float* c, void* packed, float* x, float* out, fsn_stream_t stream) {
  using namespace fsn;
  FSN_REQUIRE(bn && catM && catE && m0 && scale && restart && store && h && c && packed && x && out, FSN_ERR_SHAPE,
              "sb_phased_lstm_tc: missing buffer");
  FSN_REQUIRE(B > 0 && M > 1 && S >= 1 && St > 0 && Ns >= 0 && Nf >= 0 && Ns < M && Nf < M, FSN_ERR_SHAPE,
              "sb_phased_lstm_tc: bad shape B=%d M=%d S=%d St=%d Ns=%d Nf=%d", B, M, S, St, Ns, Nf);
  FSN_REQUIRE(H == 128 || H == 256 || H == 384, FSN_ERR_UNSUPPORTED, "sb_phased_lstm_tc: hidden size %d", H);
  const int Ksb = (2 * Ns + 1) + (2 * Nf + 1), nb = cdiv(St, S);
  FSN_REQUIRE(Ksb <= 32, FSN_ERR_UNSUPPORTED, "sb_phased_lstm_tc: input width %d > 32", Ksb);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = sb_tc_pack_raw(bn, H, Ksb, 1, packed, st, x3 != 0);
  if (rc) return rc;
  fast_stream_bn_input_kernel<<<dim3(nb, B), 256, 0, st>>>(catM, catE, m0, 1, 0, St, M, Ns, Nf, S, x, scale);
  FSN_CHECK_LAUNCH("fast_stream_bn_input_kernel");
  SbTcArgs a;
  memset(&a, 0, sizeof(a));
  a.packed = packed; a.crm = out;
  a.B = B; a.F = M; a.Tp = nb; a.Ns = Ns; a.Nf = Nf; a.H = H; a.act = FSN_ACT_RELU; a.x3 = x3 != 0;
  a.map = RowMap{B, M, M, 1};
  const size_t R = (size_t)B * M;
  const SbCarry io{h, c, (size_t)M * H, R * H, M, restart, -1, (size_t)nb * 2 * M, 0, x, store};
  return sb_tc_carry_forward(a, io, st);
}
