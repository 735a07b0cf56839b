// Host-side orchestration of Model.forward and the fused wav->wav enhancement call, plus the
// error / version entry points of the C ABI (include/fsn_b200.h).
//
// Reference: recipes/dns_interspeech_2020/fullsubnet/model.py:72-136 (Model.forward),
//            recipes/dns_interspeech_2020/inferencer.py:130-145 (full_band_crm_mask).
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

static thread_local char g_err[512] = "";
static thread_local int64_t g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static thread_local int g_err_code = 0;
int& last_error_code() { return g_err_code; }
int64_t& launch_counter() { return g_launches; }
static int64_t g_total_launches = 0;
int64_t& total_launch_counter() { return g_total_launches; }

// opt-in stage timing (bench.py): 5 events bracket the 4 stages
static thread_local bool g_prof = false;
static thread_local cudaEvent_t g_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
static thread_local bool g_ev_valid[5] = {false, false, false, false, false};
static void prof_mark(int i, cudaStream_t st) {
  if (!g_prof) return;
  if (!g_ev[i] && cudaEventCreate(&g_ev[i]) != cudaSuccess) return;
  g_ev_valid[i] = (cudaEventRecord(g_ev[i], st) == cudaSuccess);
}
static void prof_reset() { for (int i = 0; i < 5; ++i) g_ev_valid[i] = false; }

struct ModelWs {
  float *magT, *fbT, *inv1, *inv2;
  float2 *fs, *sums_mag, *sums_fb;
  float *cum1, *cum2;  // cumulative / forgetting norm: per-(step, clip) and per-(step, unit) scales
  float2* fs2;         // forgetting norm: frame sums of the full-band output (fs keeps the noisy magnitude's)
  SeqStackWs fb;
  float *sb_h0[2], *sb_h1[2], *sb_c0, *sb_c1;
  void* sb_h0ws;  // tensor-core precisions: layer 0's output for the two-pass sub-band stack
  size_t bytes;
};

// full-band stack (model.py:92-95): 2-layer LSTM / GRU (F -> Hf -> Hf) + Linear(Hf -> F), rows = B clips of Tp steps.
// On the tensor cores with the tensor-core precisions and LSTM, for every batch size, so a clip's result does not depend
// on the batch it is enhanced in.
static SeqStack fb_stack(const fsn_model_desc* d, int B, int Tp) {
  SeqStack s;
  memset(&s, 0, sizeof(s));
  const int F = d->num_freqs;
  s.R = B; s.Tp = Tp; s.K0 = F; s.n = 2; s.H[0] = s.H[1] = d->fb_hidden; s.O = F; s.act = d->fb_activation;
  s.gru = d->cell_type == FSN_CELL_GRU;
  s.step_scale = norm_per_step(d->norm_type);
  s.x3 = d->precision == FSN_PREC_F16X3_TC;
  s.tc = (s.x3 || d->precision == FSN_PREC_F16_TC) && !s.gru && lstm_rec_tc_supported(d->fb_hidden, s.x3);
  return s;
}

int make_dims(const fsn_model_desc* d, int B, int T, Dims& m) {
  FSN_REQUIRE(d && d->num_freqs > 1 && d->fb_hidden > 0 && d->sb_hidden > 0 && d->look_ahead >= 0, FSN_ERR_SHAPE,
              "model: bad descriptor");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "model: empty input (B=%d, T=%d)", B, T);
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE ||
                  d->norm_type == FSN_NORM_FORGETTING,
              FSN_ERR_UNSUPPORTED,
              "You must set up a type of Norm. (offline_laplace_norm / cumulative_laplace_norm / forgetting_norm are built)");
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM || (d->cell_type == FSN_CELL_GRU && d->precision == FSN_PREC_FP32),
              FSN_ERR_UNSUPPORTED, "model: sequence_model must be LSTM, or GRU on the fp32 kernels (precision fp32)");
  FSN_REQUIRE(d->sb_num_neighbors >= 0 && d->fb_num_neighbors >= 0 && d->sb_num_neighbors < d->num_freqs &&
                  d->fb_num_neighbors < d->num_freqs,
              FSN_ERR_SHAPE, "model: reflect padding needs num_neighbors < num_freqs");
  m.B = B; m.T = T; m.Tp = T + d->look_ahead; m.F = d->num_freqs;
  m.G = (B > 1 && d->num_groups_in_drop_band > 1) ? d->num_groups_in_drop_band : 1;
  if (B > 1)  // model.py:114-117 -> feature.py:317-319 (asserted even when G == 1)
    FSN_REQUIRE(B > d->num_groups_in_drop_band, FSN_ERR_SHAPE,
                "Batch size = %d, num_groups = %d. The batch size should larger than the num_groups.", B,
                d->num_groups_in_drop_band);
  m.Fsub = (m.G > 1) ? m.F / m.G : m.F;
  FSN_REQUIRE(m.Fsub > 0, FSN_ERR_SHAPE, "model: num_freqs < num_groups");
  m.R = B * m.Fsub;
  m.Ksb = (2 * d->sb_num_neighbors + 1) + (2 * d->fb_num_neighbors + 1);
  return FSN_OK;
}

static void carve_model(const fsn_model_desc* d, const Dims& m, void* base, ModelWs& w) {
  Carver c(base);
  const size_t BTF = (size_t)m.B * m.Tp * m.F;
  w.magT = c.take<float>(BTF);
  w.fbT = c.take<float>(BTF);
  w.fs = c.take<float2>((size_t)m.B * m.Tp);
  w.sums_mag = c.take<float2>(m.B);
  w.sums_fb = c.take<float2>(m.B);
  w.inv1 = c.take<float>(m.B);
  w.inv2 = c.take<float>(m.B);
  seq_stack_carve(c, fb_stack(d, m.B, m.Tp), w.fb);
  if (d->precision == FSN_PREC_FP32) {
    const size_t RH = (size_t)m.R * d->sb_hidden;
    for (int i = 0; i < 2; ++i) { w.sb_h0[i] = c.take<float>(RH); w.sb_h1[i] = c.take<float>(RH); }
    w.sb_c0 = c.take<float>(RH);
    w.sb_c1 = c.take<float>(RH);
  }
  w.sb_h0ws = nullptr;
  if (d->precision == FSN_PREC_F16_TC || d->precision == FSN_PREC_F16X3_TC)
    w.sb_h0ws = c.take<uint8_t>(sb_tc_split_ws_bytes(m.R, m.Tp, d->sb_hidden, d->precision == FSN_PREC_F16X3_TC));
  w.cum1 = w.cum2 = nullptr;
  w.fs2 = nullptr;
  if (norm_per_step(d->norm_type)) {
    w.cum1 = c.take<float>((size_t)m.Tp * m.B);
    w.cum2 = c.take<float>((size_t)m.Tp * m.R);
  }
  if (d->norm_type == FSN_NORM_FORGETTING) w.fs2 = c.take<float2>((size_t)m.B * m.Tp);
  w.bytes = c.off;
}

// everything after the time-major magnitude exists: norms, full-band stack, sub-band stack.  lens (nullable, device
// [B] samples, fsn_enhance): the offline norms of clip b cover only its own Tp_b = 1 + lens[b]/hop + look_ahead
// frames; every other stage is causal and runs unchanged over all Tp steps (frames past Tp_b never reach earlier ones).
static int model_core(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                      const void* sb_packed, const Dims& m, const ModelWs& w, float* crm, cudaStream_t st,
                      const int* lens = nullptr, int hop = 0) {
  int rc;
  const int F = m.F, Tp = m.Tp, B = m.B, Hs = d->sb_hidden, la = d->look_ahead;
  // with per-clip lengths the counts are per frame (norm_scales_launch multiplies by the clip's own frame count)
  const int tp_cnt = lens ? 1 : Tp;
  // per-clip statistics of the look-ahead-padded magnitude (model.py:92, :111)
  if ((rc = clip_stats_launch(w.magT, B, Tp, F, d->sb_num_neighbors, w.fs, w.sums_mag, st, lens, hop, la))) return rc;
  if ((rc = norm_scales_launch(w.sums_mag, w.sums_mag, B, (float)F * tp_cnt, 1.f, w.inv1, nullptr, st, 1e-5f, lens, hop,
                               la)))
    return rc;
  const bool cum = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE, fgt = d->norm_type == FSN_NORM_FORGETTING;
  const float cum_eps = 1.1920928955078125e-07f;  // audio_zen/constant.py:9 (np.finfo(np.float32).eps)
  if (cum && (rc = cum_clip_scale_launch(w.fs, B, Tp, F, cum_eps, w.cum1, st))) return rc;
  // forgetting norm (base_model.py:102-151): exponential running mean of the frame means, no bound needed with lens
  if (fgt && (rc = forget_scale_launch(w.fs, nullptr, B, Tp, (float)F, w.cum1, nullptr, st))) return rc;

  // ---- full-band stack -> fbT [B, Tp, F]; x = magT * 1/(mu + 1e-5) of the clip (model.py:92) or, cumulative norm, the
  // scale of (step, clip) from the time-major table cum1[t*B + b] (base_model.py:220-251), or the forgetting norm's
  SeqStack s = fb_stack(d, B, Tp);
  s.L[0] = seq_layer(*fb, 0); s.L[1] = seq_layer(*fb, 1);
  s.x = w.magT; s.scale = (cum || fgt) ? w.cum1 : w.inv1; s.fc_w = fb->fc_w; s.fc_b = fb->fc_b; s.out = w.fbT;
  if ((rc = seq_stack_forward(s, w.fb, st))) return rc;

  // ---- second norm (model.py:110-111) in closed form: never materialise [B,F,Ksb,T']
  // (the forgetting norm keeps the noisy magnitude's frame sums in fs and takes the full-band output's in fs2)
  if ((rc = clip_stats_launch(w.fbT, B, Tp, F, d->fb_num_neighbors, fgt ? w.fs2 : w.fs, w.sums_fb, st, lens, hop, la)))
    return rc;
  if ((rc = norm_scales_launch(w.sums_mag, w.sums_fb, B, 1.f, (float)F * m.Ksb * tp_cnt, nullptr, w.inv2, st, 1e-5f, lens,
                               hop, la)))
    return rc;

  prof_mark(2, st);
  RowMap map{B, F, m.Fsub, m.G};
  if (cum && (rc = cum_unit_scale_launch(w.magT, w.fbT, map, m.R, Tp, d->sb_num_neighbors, d->fb_num_neighbors, cum_eps,
                                         w.cum2, st)))
    return rc;
  // forgetting norm: one scale per (step, clip) over all F Ksb features of sb_input (model.py:111), mean from the
  // reflect-weighted frame sums of both unfolds; cum1 (the first norm's table, already consumed) holds it before the
  // broadcast to the per-(step, row) layout of the sub-band kernels
  if (fgt) {
    if ((rc = forget_scale_launch(w.fs, w.fs2, B, Tp, (float)F * m.Ksb, w.cum1, nullptr, st))) return rc;
    if ((rc = forget_unit_broadcast_launch(w.cum1, map, m.R, Tp, w.cum2, st))) return rc;
  }
  if (d->precision == FSN_PREC_F16_TC || d->precision == FSN_PREC_F16X3_TC) {
    FSN_REQUIRE(sb_packed, FSN_ERR_SHAPE, "model: the tensor-core precisions need packed sub-band weights");
    SbTcArgs a;
    memset(&a, 0, sizeof(a));
    a.packed = sb_packed; a.magT = w.magT; a.fbT = w.fbT; a.inv2 = w.inv2; a.crm = crm;
    a.B = B; a.F = F; a.Tp = Tp; a.la = d->look_ahead; a.Ns = d->sb_num_neighbors; a.Nf = d->fb_num_neighbors;
    a.H = Hs; a.act = d->sb_activation; a.map = map; a.x3 = d->precision == FSN_PREC_F16X3_TC;
    a.unit_scale = (cum || fgt) ? w.cum2 : nullptr;
    a.h0ws = w.sb_h0ws;
    rc = sb_tc_forward(a, st);
    prof_mark(3, st);
    return rc;
  }

  // ---- sub-band stack, fp32 path (model.py:121-135): rows = (clip, frequency) units
  const Step2State s2{{w.sb_h0[0], w.sb_h0[1]}, w.sb_c0, {w.sb_h1[0], w.sb_h1[1]}, w.sb_c1, Hs, 0};
  for (int t = 0; t < Tp; ++t) {
    StepParams p;
    memset(&p, 0, sizeof(p));
    p.R = m.R; p.H = Hs; p.gru = d->cell_type == FSN_CELL_GRU;
    p.K0 = m.Ksb;
    p.w_ih = sb->w_ih[0]; p.w_hh = sb->w_hh[0]; p.b_ih = sb->b_ih[0]; p.b_hh = sb->b_hh[0];
    p.magT = w.magT; p.fbT = w.fbT; p.inv2 = w.inv2;
    p.unit_scale = (cum || fgt) ? w.cum2 + (size_t)t * m.R : nullptr;
    p.F = F; p.Tp = Tp; p.t = t; p.Ns = d->sb_num_neighbors; p.Nf = d->fb_num_neighbors; p.map = map;
    if ((rc = lstm_step2_launch(p, SEG0_GATHER, t, seq_layer(*sb, 1), s2, st))) return rc;
    if (t >= d->look_ahead)
      if ((rc = sb_head_launch(s2.h1_at(t), m.R, Hs, 1, sb->fc_w, sb->fc_b, 2, d->sb_activation, crm,
                               fsn_head_geom(m.Fsub, m.T), t - d->look_ahead, st)))
        return rc;
  }
  prof_mark(3, st);
  return FSN_OK;
}

}  // namespace fsn

using namespace fsn;

extern "C" int fsn_version(void) { return 102; }
extern "C" const char* fsn_last_error(void) { return g_err; }
extern "C" int fsn_last_error_code(void) { return g_err_code; }
extern "C" int64_t fsn_last_launch_count(void) { return g_launches; }
extern "C" int64_t fsn_total_launch_count(void) { return g_total_launches; }
extern "C" int fsn_set_profiling(int enable) { g_prof = enable != 0; return FSN_OK; }
extern "C" float fsn_last_stage_ms(int stage) {
  if (stage < 0 || stage > 3 || !g_ev_valid[stage] || !g_ev_valid[stage + 1]) return -1.0f;
  float ms = -1.0f;
  if (cudaEventElapsedTime(&ms, g_ev[stage], g_ev[stage + 1]) != cudaSuccess) return -1.0f;
  return ms;
}
// host-side views of the index helpers the kernels share (tests/test_cpu_host.py checks them against the oracle)
extern "C" int fsn_debug_row_to_unit(int B, int F, int G, int r, int* b, int* f) {
  const int g = (B > 1 && G > 1) ? G : 1;
  RowMap m{B, F, g > 1 ? F / g : F, g};
  if (r < 0 || r >= B * m.Fsub) return FSN_ERR_SHAPE;
  row_to_unit(m, r, *b, *f);
  return FSN_OK;
}
extern "C" int fsn_debug_unit_to_row(int B, int F, int G, int b, int f) {
  const int g = (B > 1 && G > 1) ? G : 1;
  RowMap m{B, F, g > 1 ? F / g : F, g};
  return unit_to_row(m, b, f);
}
extern "C" int fsn_debug_reflect_count(int r, int F, int N) { return reflect_count(r, F, N); }

extern "C" int fsn_built_arch(void) {
#ifdef FSN_BUILT_ARCH
  return FSN_BUILT_ARCH;
#else
  return 0;
#endif
}

extern "C" size_t fsn_model_workspace_bytes(const fsn_model_desc* d, int B, int T) {
  Dims m;
  if (make_dims(d, B, T, m)) return 0;
  ModelWs w;
  carve_model(d, m, nullptr, w);
  return w.bytes;
}

extern "C" size_t fsn_sb_packed_bytes(const fsn_model_desc* d) { return sb_tc_packed_bytes(d); }

extern "C" int fsn_pack_sb_weights(const fsn_model_desc* d, const fsn_seq_weights* sb, void* packed,
                                   fsn_stream_t stream) {
  return sb_tc_pack(d, sb, packed, (cudaStream_t)stream);
}

extern "C" int fsn_model_forward(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                                 const void* sb_packed, const float* noisy_mag, int B, int T, float* crm,
                                 void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  g_launches = 0;
  Dims m;
  int rc = make_dims(d, B, T, m);
  if (rc) return rc;
  if ((rc = layout_clips_check(B, false, "model"))) return rc;
  FSN_REQUIRE(d->precision == FSN_PREC_FP32 || sb_tc_supported(d), FSN_ERR_UNSUPPORTED,
              "FSN_PREC_F16_TC / FSN_PREC_F16X3_TC need sb_hidden in {128,256,384} and sub-band input width <= 32");
  ModelWs w;
  carve_model(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  prof_reset();
  prof_mark(0, st);
  if ((rc = transpose_mag_launch(noisy_mag, B, m.F, T, m.Tp, (size_t)m.Tp * m.F, m.F, w.magT, nullptr, nullptr, st))) return rc;
  prof_mark(1, st);
  return model_core(d, fb, sb, sb_packed, m, w, crm, st);
}

// ---- wav -> wav (fsn_enhance).  Batched inference == loop of B=1 calls of the reference inferencer: drop_band off
// (audio_zen/inferencer/base_inferencer.py:78,173; SURVEY fact 4).  Buffers are laid out for the longest clip (L_max
// samples, T frames); with lengths, the length-dependent kernels (STFT, offline norms, iSTFT, int16 scaling) are bounded
// per clip by the device copy of the table.
static int enhance_dims(const fsn_model_desc* d, int B, int L, int n_fft, int hop, fsn_model_desc& dd, Dims& m) {
  FSN_REQUIRE(hop > 0 && n_fft > 0, FSN_ERR_SHAPE, "enhance: bad n_fft/hop");
  dd = *d;
  dd.num_groups_in_drop_band = 1;
  int rc = make_dims(&dd, B, 1 + L / hop, m);
  if (rc) return rc;
  FSN_REQUIRE(n_fft / 2 + 1 == d->num_freqs, FSN_ERR_SHAPE, "enhance: n_fft/2+1 = %d != num_freqs = %d",
              n_fft / 2 + 1, d->num_freqs);
  return FSN_OK;
}

// the wav-side buffers, then the model's; returns the bytes
static size_t carve_enhance(const fsn_model_desc* d, const Dims& m, void* base, WavWs& e, ModelWs& w) {
  Carver c(base);
  wav_carve(c, m.B, m.F, m.T, e);
  carve_model(d, m, base ? (char*)base + c.off : nullptr, w);
  return c.off + w.bytes;
}

extern "C" size_t fsn_enhance_workspace_bytes(const fsn_model_desc* d, int B, int L_max, int n_fft, int hop) {
  fsn_model_desc dd;
  Dims m;
  if (enhance_dims(d, B, L_max, n_fft, hop, dd, m)) return 0;
  WavWs e;
  ModelWs w;
  return carve_enhance(&dd, m, nullptr, e, w);
}

extern "C" int fsn_enhance(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                           const void* sb_packed, const float* wav, const int32_t* lengths, int B, int L_max, int n_fft,
                           int hop, int win_length, float* enhanced, float* crm_out, int16_t* pcm, float gain,
                           void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  g_launches = 0;
  fsn_model_desc dd;
  Dims m;
  int rc = enhance_dims(d, B, L_max, n_fft, hop, dd, m);
  if (rc) return rc;
  FSN_REQUIRE(dd.precision == FSN_PREC_FP32 || sb_tc_supported(&dd), FSN_ERR_UNSUPPORTED,
              "FSN_PREC_F16_TC / FSN_PREC_F16X3_TC need sb_hidden in {128,256,384} and sub-band input width <= 32");
  if ((rc = wav_check(lengths, B, L_max, n_fft, true, enhanced, "enhance"))) return rc;
  WavWs e;
  ModelWs w;
  const size_t bytes = carve_enhance(&dd, m, workspace, e, w);
  FSN_REQUIRE(workspace && workspace_bytes >= bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, bytes);
  cudaStream_t st = (cudaStream_t)stream;
  float* crm = crm_out ? crm_out : e.crm;
  prof_reset();
  prof_mark(0, st);
  if ((rc = wav_prologue(lengths, B, e, st))) return rc;
  if ((rc = stft_launch(wav, B, L_max, n_fft, hop, win_length, nullptr, nullptr, e.real, e.imag, w.magT, m.Tp, st,
                        e.lens)))
    return rc;
  prof_mark(1, st);
  if ((rc = model_core(&dd, fb, sb, sb_packed, m, w, crm, st, e.lens, hop))) return rc;
  rc = istft_launch(e.real, e.imag, 1, crm, B, m.T, n_fft, hop, win_length, L_max, enhanced, st, 1, pcm ? e.peak : nullptr,
                    e.lens);
  if (!rc) rc = wav_epilogue(e, enhanced, B, L_max, pcm, gain, crm_out, m.F, m.T, hop, st);
  prof_mark(4, st);
  return rc;
}

// ---- chunked streaming (DESIGN 4.14).  Slot state block: the stream header (StreamSlot), then the second norm's
// accumulator (cumulative: the running sum of each of the F sub-band units, forgetting: mu), full-band (h | c) of both
// layers (2 x fb_hidden each), sub-band (h | c) of both layers for every frequency (2 x F x sb_hidden each).
namespace fsn {

struct FsnStreamLayout : StreamSlot { size_t norm2, fbh, fbc, sbh, sbc; };

static FsnStreamLayout fsn_stream_layout(const fsn_model_desc* d, const StreamGeom& g) {
  const size_t F = d->num_freqs, Hf = 2 * (size_t)d->fb_hidden, Hs = 2 * F * d->sb_hidden;
  FsnStreamLayout s{StreamSlot(g, d->num_freqs)};
  s.norm2 = s.sec(d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE ? F : 1);
  s.fbh = s.sec(Hf); s.fbc = s.sec(Hf);
  s.sbh = s.sec(Hs); s.sbc = s.sec(Hs);
  return s;
}

// every slot is one clip of the B = 1 whole-clip call, so drop_band never applies, whatever num_groups_in_drop_band says.
// tc: the tensor-core stream (fsn_stream_tc_*), which takes FSN_PREC_F16X3_TC / FSN_PREC_F16_TC instead of FSN_PREC_FP32
static int fsn_stream_check(const fsn_model_desc* d, int n_fft, int hop, int win_length, Dims& m, StreamGeom& g,
                            bool tc) {
  FSN_REQUIRE(d, FSN_ERR_SHAPE, "stream: null descriptor");
  fsn_model_desc dd = *d;
  dd.num_groups_in_drop_band = 1;
  int rc = make_dims(&dd, 1, 1, m);
  if (rc) return rc;
  FSN_REQUIRE(norm_per_step(d->norm_type), FSN_ERR_UNSUPPORTED,
              "stream: the offline norm needs the whole clip; streaming is built for cumulative_laplace_norm and "
              "forgetting_norm");
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "stream: streaming is built for the LSTM cell");
  if (tc) {
    FSN_REQUIRE(d->precision == FSN_PREC_F16X3_TC || d->precision == FSN_PREC_F16_TC, FSN_ERR_UNSUPPORTED,
                "stream_tc: the tensor-core stream is built for FSN_PREC_F16X3_TC and FSN_PREC_F16_TC (precision %d); "
                "the fp32 kernels stream through fsn_stream_step", d->precision);
    FSN_REQUIRE(sb_tc_supported(d), FSN_ERR_UNSUPPORTED,
                "stream_tc: the tensor-core sub band needs sb_hidden in {128,256,384} and sub-band input width <= 32");
  } else {
    FSN_REQUIRE(d->precision == FSN_PREC_FP32, FSN_ERR_UNSUPPORTED,
                "stream: streaming is built for FSN_PREC_FP32 (precision %d)", d->precision);
  }
  FSN_REQUIRE(n_fft / 2 + 1 == d->num_freqs, FSN_ERR_SHAPE, "stream: n_fft/2+1 = %d != num_freqs = %d", n_fft / 2 + 1,
              d->num_freqs);
  return stream_geom(n_fft, hop, win_length, d->look_ahead, g);
}

struct FsnStreamWs : StreamWs {
  int* restart;
  float *scale1, *fbT, *scale2, *unit;
  float2 *fs, *fs2;
  StreamStackWs fb;                      // full band
  float *sh0[2], *sh1[2], *sc0, *sc1;    // sub-band state, h ping-pong per layer (fp32 stream)
};

// St = K + E steps: a call with a clip's last chunk runs E steps past the K of the others.  tc: the sub band's state
// stays in the slot state (no per-row buffers).  Returns the bytes
static size_t fsn_stream_carve(const fsn_model_desc* d, const StreamGeom& g, int B, int K, void* base, FsnStreamWs& w,
                               bool tc) {
  Carver c(base);
  const size_t F = d->num_freqs, St = (size_t)K + g.E, RH = (size_t)B * F * d->sb_hidden;
  stream_carve(c, g, B, K, d->num_freqs, w);
  w.restart = tc ? c.take<int>(B) : nullptr;
  w.fs = c.take<float2>(B * St);
  w.fs2 = d->norm_type == FSN_NORM_FORGETTING ? c.take<float2>(B * St) : nullptr;
  w.scale1 = c.take<float>(St * B);
  stream_stack_carve(c, fb_stack(d, B, (int)St), w.fb);
  w.fbT = c.take<float>(B * St * F);
  w.scale2 = d->norm_type == FSN_NORM_FORGETTING ? c.take<float>(St * B) : nullptr;
  w.unit = c.take<float>(St * B * F);
  memset(w.sh0, 0, sizeof(w.sh0)); memset(w.sh1, 0, sizeof(w.sh1));
  w.sc0 = w.sc1 = nullptr;
  if (!tc) {
    for (int i = 0; i < 2; ++i) { w.sh0[i] = c.take<float>(RH); w.sh1[i] = c.take<float>(RH); }
    w.sc0 = c.take<float>(RH); w.sc1 = c.take<float>(RH);
  }
  return c.off;
}

// one call of either stream.  The full band on the kernels of the whole-clip call (stream_seq_stack); tc: the sub band in
// one sb_carry_lstm_tc_kernel launch over all St steps
static int fsn_stream_run(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                          const void* sb_packed, bool tc, const float* wav, const int32_t* start, const int32_t* tail,
                          int B, int K, int n_fft, int hop, int win_length, float* enhanced, void* state,
                          size_t state_bytes, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  launch_counter() = 0;
  Dims m;
  StreamGeom g;
  int St, rc = fsn_stream_check(d, n_fft, hop, win_length, m, g, tc);
  if (rc || (rc = stream_check("stream", g, B, K, tail, wav, enhanced, St))) return rc;
  // the sub-band rows' (h, c) of all slots, one int-indexed element per thread in stream_reset_kernel
  FSN_REQUIRE((size_t)B * m.F * d->sb_hidden <= 0x7fffffff, FSN_ERR_SHAPE,
              "stream: B=%d slots x %d frequencies x sb_hidden %d must stay below 2^31", B, m.F, d->sb_hidden);
  FSN_REQUIRE(fb && sb, FSN_ERR_SHAPE, "stream: null weights");
  FSN_REQUIRE(!tc || sb_packed, FSN_ERR_SHAPE, "stream_tc: the tensor-core stream needs packed sub-band weights");
  const FsnStreamLayout sl = fsn_stream_layout(d, g);
  FsnStreamWs w;
  const size_t ws = fsn_stream_carve(d, g, B, K, workspace, w, tc);
  if ((rc = stream_check_sizes(state, state_bytes, sl.slot(), B, workspace, workspace_bytes, ws))) return rc;
  char* sbase = (char*)state;
  const size_t ss = sl.slot();
  const int F = m.F, Hs = d->sb_hidden, Ns = d->sb_num_neighbors, Nf = d->fb_num_neighbors;
  const int R = B * F;
  const bool fgt = d->norm_type == FSN_NORM_FORGETTING, x3 = d->precision == FSN_PREC_F16X3_TC;
  const size_t F2 = 2 * (size_t)F;
  if ((rc = stream_open(g, sl, w, F, B, K, St, win_length, start, tail, wav, sbase, w.restart, st))) return rc;
  // first norm (model_core): frame sums (.y reflect-weighted with Ns, for the second forgetting norm), running scale
  if ((rc = frame_stats_launch(w.magT, B, St, F, Ns, (size_t)St * F, F, w.fs, st))) return rc;
  if ((rc = stream_norm_launch(w.fs, B, St, K, F, g, d->norm_type, w.pos0, w.act0, w.tail, sbase, ss, w.scale1, st)))
    return rc;
  // full band, (h, c) carried; only the tensor-core stream has a restart table, and only its stack can take a path that
  // reads one (the fp32 stream's per-step scale keeps it on the per-step kernels)
  SeqStack fbs = fb_stack(d, B, St);
  fbs.L[0] = seq_layer(*fb, 0); fbs.L[1] = seq_layer(*fb, 1);
  fbs.x = w.magT; fbs.scale = w.scale1; fbs.fc_w = fb->fc_w; fbs.fc_b = fb->fc_b; fbs.out = w.fbT;
  if ((rc = stream_seq_stack(fbs, w.fb, StackCarry{sbase, ss, sl.fbh, sl.fbc, w.pos0, g, w.restart, K}, st))) return rc;
  // second norm, one scale per (step, row), rows b*F + f
  const RowMap map{B, F, F, 1};
  if (fgt) {
    if ((rc = frame_stats_launch(w.fbT, B, St, F, Nf, (size_t)St * F, F, w.fs2, st))) return rc;
    if ((rc = stream_norm_launch(w.fs, B, St, K, F * m.Ksb, g, d->norm_type, w.pos0, w.act0, w.tail, sbase, ss, w.scale2,
                                 st, w.fs2, sl.norm2)))
      return rc;
    if ((rc = forget_unit_broadcast_launch(w.scale2, map, R, St, w.unit, st))) return rc;
  } else if ((rc = stream_cum_unit_launch(w.magT, w.fbT, B, St, K, F, Ns, Nf, g, w.pos0, w.act0, sbase, ss, sl.norm2, w.unit,
                                          st))) {
    return rc;
  }
  // sub band on the B*F rows, (h, c) of every row from the state, stored after step K - 1; step j's cRM is frame Rc + j
  // of w.crm [B, Rc + St, 2F]
  if (tc) {
    SbTcArgs a;
    memset(&a, 0, sizeof(a));
    a.packed = sb_packed; a.magT = w.magT; a.fbT = w.fbT; a.unit_scale = w.unit; a.crm = w.crm;
    a.B = B; a.F = F; a.Tp = St; a.la = 0; a.Ns = Ns; a.Nf = Nf; a.H = Hs; a.act = d->sb_activation; a.map = map;
    a.x3 = x3;
    const SbCarry io{(float*)(sbase + sl.sbh), (float*)(sbase + sl.sbc), ss / 4, (size_t)F * Hs, F, w.restart, K - 1,
                     ((size_t)g.Rc + St) * F2, g.Rc};
    if ((rc = sb_tc_carry_forward(a, io, st))) return rc;
  } else {
    // (h, c) into the halves step 0 reads
    const size_t sbw = (size_t)F * Hs * 4;
    const Step2State s2{{w.sh0[0], w.sh0[1]}, w.sc0, {w.sh1[0], w.sh1[1]}, w.sc1, Hs, 0, true};
    if ((rc = copy_rows(w.sh0[1], sbw, sbase + sl.sbh, ss, sbw, B, st))) return rc;
    if ((rc = copy_rows(w.sh1[1], sbw, sbase + sl.sbh + sbw, ss, sbw, B, st))) return rc;
    if ((rc = copy_rows(w.sc0, sbw, sbase + sl.sbc, ss, sbw, B, st))) return rc;
    if ((rc = copy_rows(w.sc1, sbw, sbase + sl.sbc + sbw, ss, sbw, B, st))) return rc;
    const HeadGeom hg{F, 1, 0, F, 1, ((size_t)g.Rc + St) * F2};
    for (int j = 0; j < St; ++j) {
      if (j <= g.c) {  // a clip's frame 0 is one of the first c + 1 steps
        if ((rc = stream_reset_launch(w.pos0, B, g, j, F * Hs, w.sh0[(j + 1) & 1], (size_t)F * Hs, w.sc0, st))) return rc;
        if ((rc = stream_reset_launch(w.pos0, B, g, j, F * Hs, w.sh1[(j + 1) & 1], (size_t)F * Hs, w.sc1, st))) return rc;
      }
      StepParams p;
      memset(&p, 0, sizeof(p));
      p.R = R; p.H = Hs; p.K0 = m.Ksb;
      p.w_ih = sb->w_ih[0]; p.w_hh = sb->w_hh[0]; p.b_ih = sb->b_ih[0]; p.b_hh = sb->b_hh[0];
      p.magT = w.magT; p.fbT = w.fbT; p.unit_scale = w.unit + (size_t)j * R;
      p.F = F; p.Tp = St; p.t = j; p.Ns = Ns; p.Nf = Nf; p.map = map;
      if ((rc = lstm_step2_launch(p, SEG0_GATHER, j, seq_layer(*sb, 1), s2, st))) return rc;
      if ((rc = sb_head_launch(s2.h1_at(j), R, Hs, 1, sb->fc_w, sb->fc_b, 2, d->sb_activation, w.crm + (g.Rc + j) * F2, hg,
                               0, st)))
        return rc;
      if (j == K - 1) {
        if ((rc = copy_rows(sbase + sl.sbh, ss, w.sh0[j & 1], sbw, sbw, B, st))) return rc;
        if ((rc = copy_rows(sbase + sl.sbh + sbw, ss, w.sh1[j & 1], sbw, sbw, B, st))) return rc;
        if ((rc = copy_rows(sbase + sl.sbc, ss, w.sc0, sbw, sbw, B, st))) return rc;
        if ((rc = copy_rows(sbase + sl.sbc + sbw, ss, w.sc1, sbw, sbw, B, st))) return rc;
      }
    }
  }
  return stream_close(g, sl, w, F, B, K, St, win_length, nullptr, enhanced, sbase, st);
}

}  // namespace fsn

extern "C" size_t fsn_stream_state_bytes(const fsn_model_desc* d, int B, int n_fft, int hop) {
  Dims m;
  StreamGeom g;
  return stream_query_check(fsn_stream_check(d, n_fft, hop, n_fft, m, g, false), "stream", B, 1)
             ? 0 : fsn_stream_layout(d, g).slot() * (size_t)B;
}

extern "C" size_t fsn_stream_workspace_bytes(const fsn_model_desc* d, int B, int K_max, int n_fft, int hop) {
  Dims m;
  StreamGeom g;
  FsnStreamWs w;
  return stream_query_check(fsn_stream_check(d, n_fft, hop, n_fft, m, g, false), "stream", B, K_max)
             ? 0 : fsn_stream_carve(d, g, B, K_max, nullptr, w, false);
}

extern "C" int fsn_stream_delay(const fsn_model_desc* d, int n_fft, int hop) {
  Dims m;
  StreamGeom g;
  return stream_delay(fsn_stream_check(d, n_fft, hop, n_fft, m, g, false), g);
}

extern "C" int fsn_stream_step(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                               const float* wav, const int32_t* start, const int32_t* tail, int B, int K, int n_fft, int hop,
                               int win_length, float* enhanced, void* state, size_t state_bytes, void* workspace,
                               size_t workspace_bytes, fsn_stream_t stream) {
  return fsn_stream_run(d, fb, sb, nullptr, false, wav, start, tail, B, K, n_fft, hop, win_length, enhanced, state,
                        state_bytes, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" size_t fsn_stream_tc_state_bytes(const fsn_model_desc* d, int B, int n_fft, int hop) {
  Dims m;
  StreamGeom g;
  return stream_query_check(fsn_stream_check(d, n_fft, hop, n_fft, m, g, true), "stream", B, 1)
             ? 0 : fsn_stream_layout(d, g).slot() * (size_t)B;
}

extern "C" size_t fsn_stream_tc_workspace_bytes(const fsn_model_desc* d, int B, int K_max, int n_fft, int hop) {
  Dims m;
  StreamGeom g;
  FsnStreamWs w;
  return stream_query_check(fsn_stream_check(d, n_fft, hop, n_fft, m, g, true), "stream", B, K_max)
             ? 0 : fsn_stream_carve(d, g, B, K_max, nullptr, w, true);
}

extern "C" int fsn_stream_tc_delay(const fsn_model_desc* d, int n_fft, int hop) {
  Dims m;
  StreamGeom g;
  return stream_delay(fsn_stream_check(d, n_fft, hop, n_fft, m, g, true), g);
}

extern "C" int fsn_stream_tc_step(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                                  const void* sb_packed, const float* wav, const int32_t* start, const int32_t* tail, int B,
                                  int K, int n_fft, int hop, int win_length, float* enhanced, void* state,
                                  size_t state_bytes, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  return fsn_stream_run(d, fb, sb, sb_packed, true, wav, start, tail, B, K, n_fft, hop, win_length, enhanced, state,
                        state_bytes, workspace, workspace_bytes, (cudaStream_t)stream);
}
