// fullband_baseline (recipes/dns_interspeech_2020/fullband_baseline/model.py:8-68; SURVEY 8f rank 3):
// look-ahead pad -> norm -> num_layers x LSTM(F -> H) -> Linear(H -> 2F) [+ activation] -> [B,2,F,T].
// Host orchestration: the norm, the SequenceModel of fsn_fullband.cu (seq_stack_forward) and the output re-layout;
// fsn_fullband_enhance adds the STFT, the mask + iSTFT of Inferencer.full_band_crm_mask and the int16 output.
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

struct FbbWs {
  float *magT, *inv1, *cum1, *y;
  float2 *fs, *sums;
  SeqStackWs seq;
  WavWs wav;  // fsn_fullband_enhance
  size_t bytes;
};

static int fbb_check(const fsn_fullband_desc* d, int B, int T) {
  FSN_REQUIRE(d && d->num_freqs > 1 && d->hidden > 0 && d->look_ahead >= 0, FSN_ERR_SHAPE, "fullband: bad descriptor");
  FSN_REQUIRE(d->num_layers >= 1 && d->num_layers <= SEQ_MAX_LAYERS, FSN_ERR_UNSUPPORTED, "fullband: 1..8 LSTM layers");
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "fullband: the GRU cell is not built");
  FSN_REQUIRE(B > 0 && T > 0, FSN_ERR_SHAPE, "fullband: empty input (B=%d, T=%d)", B, T);
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE ||
                  d->norm_type == FSN_NORM_FORGETTING,
              FSN_ERR_UNSUPPORTED,
              "You must set up a type of Norm. (offline_laplace_norm / cumulative_laplace_norm / forgetting_norm are built)");
  // the tensor-core stack misses the reference gates on this model (DESIGN 4.9): f16x3_tc 1.8e-4 waveform max-abs on
  // the clipping weight set, f16_tc 1.6e-3 relative cRM
  FSN_REQUIRE(d->precision != FSN_PREC_F16X3_TC && d->precision != FSN_PREC_F16_TC, FSN_ERR_UNSUPPORTED,
              "fullband: the tensor-core precisions are not built for this model; use FSN_PREC_FP32");
  return FSN_OK;
}

// num_layers x LSTM(F -> H) + Linear(H -> 2F), rows = clips, fp32 kernels (also for the training precision
// FSN_PREC_TF32_TC).  The path does not depend on B, so a clip gets the same bits in any batch.
static SeqStack fbb_stack(const fsn_fullband_desc* d, int B, int Tp) {
  SeqStack s;
  memset(&s, 0, sizeof(s));
  s.R = B; s.Tp = Tp; s.K0 = d->num_freqs; s.n = d->num_layers; s.O = 2 * d->num_freqs; s.act = d->activation;
  for (int l = 0; l < s.n; ++l) s.H[l] = d->hidden;
  s.step_scale = norm_per_step(d->norm_type);
  return s;
}

// enhance: also the wav-side buffers of fsn_fullband_enhance (n_fft / 2 + 1 = num_freqs)
static void fbb_carve(const fsn_fullband_desc* d, int B, int T, void* base, FbbWs& w, bool enhance = false) {
  Carver c(base);
  const size_t Tp = (size_t)T + d->look_ahead, F = d->num_freqs;
  w.magT = c.take<float>(B * Tp * F);
  w.fs = c.take<float2>(B * Tp);
  w.sums = c.take<float2>(B);
  w.inv1 = c.take<float>(B);
  w.cum1 = c.take<float>(B * Tp);
  seq_stack_carve(c, fbb_stack(d, B, (int)Tp), w.seq);
  w.y = c.take<float>(B * Tp * 2 * F);
  if (enhance) wav_carve(c, B, (int)F, T, w.wav);
  w.bytes = c.off;
}

// everything after the time-major, look-ahead-padded magnitude w.magT exists: norm -> stack -> out [B,2,F,T].  lens
// (nullable, device [B] samples): the offline norm of clip b covers only its own Tp_b = 1 + lens[b]/hop + look_ahead
// frames; the cumulative and forgetting norms and the stack are causal and run over all Tp steps.
static int fbb_core(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w, const float* fc_b, int B,
                    int T, const FbbWs& w, float* out, cudaStream_t st, const int* lens = nullptr, int hop = 0) {
  int rc;
  const int F = d->num_freqs, Tp = T + d->look_ahead, la = d->look_ahead;
  const bool cum = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE, fgt = d->norm_type == FSN_NORM_FORGETTING;
  if ((rc = clip_stats_launch(w.magT, B, Tp, F, 0, w.fs, w.sums, st, lens, hop, la))) return rc;
  if ((rc = norm_scales_launch(w.sums, w.sums, B, lens ? (float)F : (float)F * Tp, 1.f, w.inv1, nullptr, st, 1e-5f, lens,
                               hop, la)))
    return rc;
  if (cum && (rc = cum_clip_scale_launch(w.fs, B, Tp, F, 1.1920928955078125e-07f, w.cum1, st))) return rc;
  if (fgt && (rc = forget_scale_launch(w.fs, nullptr, B, Tp, (float)F, w.cum1, nullptr, st))) return rc;
  SeqStack s = fbb_stack(d, B, Tp);
  for (int l = 0; l < s.n; ++l) s.L[l] = layers[l];
  s.x = w.magT; s.scale = (cum || fgt) ? w.cum1 : w.inv1; s.fc_w = fc_w; s.fc_b = fc_b; s.out = w.y;
  if ((rc = seq_stack_forward(s, w.seq, st))) return rc;
  return crm_output_launch(w.y, (size_t)Tp * 2 * F, 2 * F, B, Tp, F, la, out, st);
}

static int fbb_enhance_dims(const fsn_fullband_desc* d, int B, int L, int n_fft, int hop, int& T) {
  FSN_REQUIRE(hop > 0 && n_fft > 0 && L > 0, FSN_ERR_SHAPE, "fullband_enhance: bad n_fft/hop/L");
  T = 1 + L / hop;
  int rc = fbb_check(d, B, T);
  if (rc) return rc;
  FSN_REQUIRE(n_fft / 2 + 1 == d->num_freqs, FSN_ERR_SHAPE, "fullband_enhance: n_fft/2+1 = %d != num_freqs = %d",
              n_fft / 2 + 1, d->num_freqs);
  return FSN_OK;
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
  if ((rc = layout_clips_check(B, true, "fullband"))) return rc;
  FbbWs w;
  fbb_carve(d, B, T, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int F = d->num_freqs, Tp = T + d->look_ahead;
  if ((rc = transpose_mag_launch(noisy_mag, B, F, T, Tp, (size_t)Tp * F, F, w.magT, nullptr, nullptr, st))) return rc;
  return fbb_core(d, layers, fc_w, fc_b, B, T, w, out, st);
}

// ---- wav -> wav, clips of different lengths in one call (lengths non-null: host [B]), buffers laid out for the longest
// clip (L_max samples, T_max frames); optional int16 output with the per-clip peak of the iSTFT epilogue
extern "C" size_t fsn_fullband_enhance_workspace_bytes(const fsn_fullband_desc* d, int B, int L_max, int n_fft, int hop) {
  int T;
  if (fbb_enhance_dims(d, B, L_max, n_fft, hop, T)) return 0;
  FbbWs w;
  fbb_carve(d, B, T, nullptr, w, true);
  return w.bytes;
}

extern "C" int fsn_fullband_enhance(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                                    const float* fc_b, const float* wav, const int32_t* lengths, int B, int L_max,
                                    int n_fft, int hop, int win_length, float* enhanced, float* crm_out, int16_t* pcm,
                                    float gain, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  int T, rc = fbb_enhance_dims(d, B, L_max, n_fft, hop, T);
  if (rc) return rc;
  if ((rc = layout_clips_check(B, true, "fullband_enhance"))) return rc;
  if ((rc = wav_check(lengths, B, L_max, n_fft, true, enhanced, "fullband_enhance"))) return rc;
  FbbWs w;
  fbb_carve(d, B, T, workspace, w, true);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  WavWs& e = w.wav;
  float* crm = crm_out ? crm_out : e.crm;
  if ((rc = wav_prologue(lengths, B, e, st))) return rc;
  // STFT straight into the time-major magnitude with the look-ahead frames zeroed (model.py:46-49)
  if ((rc = stft_launch(wav, B, L_max, n_fft, hop, win_length, nullptr, nullptr, e.real, e.imag, w.magT,
                        T + d->look_ahead, st, e.lens)))
    return rc;
  if ((rc = fbb_core(d, layers, fc_w, fc_b, B, T, w, crm, st, e.lens, hop))) return rc;
  // decompress_cIRM + complex product + iSTFT (inferencer.py:130-145)
  if ((rc = istft_launch(e.real, e.imag, 1, crm, B, T, n_fft, hop, win_length, L_max, enhanced, st, 1,
                         pcm ? e.peak : nullptr, e.lens)))
    return rc;
  return wav_epilogue(e, enhanced, B, L_max, pcm, gain, crm_out, d->num_freqs, T, hop, st);
}

// ---- chunked streaming (DESIGN 4.14).  Slot state block: the stream header (StreamSlot), then h and c of every layer
// (num_layers x H floats each).
namespace fsn {

struct FbbStreamLayout : StreamSlot { size_t h, c; };

static FbbStreamLayout fbb_stream_layout(const fsn_fullband_desc* d, const StreamGeom& g) {
  const size_t nH = (size_t)d->num_layers * d->hidden;
  FbbStreamLayout s{StreamSlot(g, d->num_freqs)};
  s.h = s.sec(nH);
  s.c = s.sec(nH);
  return s;
}

static int fbb_stream_check(const fsn_fullband_desc* d, int n_fft, int hop, int win_length, StreamGeom& g) {
  int rc = fbb_check(d, 1, 1);
  if (rc) return rc;
  FSN_REQUIRE(d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE || d->norm_type == FSN_NORM_FORGETTING, FSN_ERR_UNSUPPORTED,
              "fullband_stream: the offline norm needs the whole clip; streaming is built for cumulative_laplace_norm and "
              "forgetting_norm");
  FSN_REQUIRE(n_fft / 2 + 1 == d->num_freqs, FSN_ERR_SHAPE, "fullband_stream: n_fft/2+1 = %d != num_freqs = %d",
              n_fft / 2 + 1, d->num_freqs);
  return stream_geom(n_fft, hop, win_length, d->look_ahead, g);
}

struct FbbStreamWs : StreamWs {
  float *scale, *y;
  float2* fs;
  StreamStackWs stack;
};

// St = K + E steps: a call with a clip's last chunk runs E steps past the K of the others; returns the bytes
static size_t fbb_stream_carve(const fsn_fullband_desc* d, const StreamGeom& g, int B, int K, void* base, FbbStreamWs& w) {
  Carver c(base);
  const size_t St = (size_t)K + g.E;
  stream_carve(c, g, B, K, d->num_freqs, w);
  w.fs = c.take<float2>(B * St);
  w.scale = c.take<float>(St * B);
  stream_stack_carve(c, fbb_stack(d, B, (int)St), w.stack);
  w.y = c.take<float>(B * St * 2 * d->num_freqs);
  return c.off;
}

}  // namespace fsn

extern "C" size_t fsn_fullband_stream_state_bytes(const fsn_fullband_desc* d, int B, int n_fft, int hop) {
  StreamGeom g;
  return stream_query_check(fbb_stream_check(d, n_fft, hop, n_fft, g), "fullband_stream", B, 1)
             ? 0 : fbb_stream_layout(d, g).slot() * (size_t)B;
}

extern "C" size_t fsn_fullband_stream_workspace_bytes(const fsn_fullband_desc* d, int B, int K_max, int n_fft, int hop) {
  StreamGeom g;
  FbbStreamWs w;
  return stream_query_check(fbb_stream_check(d, n_fft, hop, n_fft, g), "fullband_stream", B, K_max)
             ? 0 : fbb_stream_carve(d, g, B, K_max, nullptr, w);
}

extern "C" int fsn_fullband_stream_delay(const fsn_fullband_desc* d, int n_fft, int hop) {
  StreamGeom g;
  return stream_delay(fbb_stream_check(d, n_fft, hop, n_fft, g), g);
}

extern "C" int fsn_fullband_stream_step(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                                        const float* fc_b, const float* wav, const int32_t* start, const int32_t* tail,
                                        int B, int K, int n_fft, int hop, int win_length, float* enhanced, void* state,
                                        size_t state_bytes, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  StreamGeom g;
  int St, rc = fbb_stream_check(d, n_fft, hop, win_length, g);
  if (rc || (rc = stream_check("fullband_stream", g, B, K, tail, wav, enhanced, St))) return rc;
  FSN_REQUIRE(layers && fc_w && fc_b, FSN_ERR_SHAPE, "fullband_stream: null weights");
  const FbbStreamLayout sl = fbb_stream_layout(d, g);
  FbbStreamWs w;
  const size_t ws = fbb_stream_carve(d, g, B, K, workspace, w);
  if ((rc = stream_check_sizes(state, state_bytes, sl.slot(), B, workspace, workspace_bytes, ws))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  char* sb = (char*)state;
  const size_t ss = sl.slot();
  const int F = d->num_freqs;
  if ((rc = stream_open(g, sl, w, F, B, K, St, win_length, start, tail, wav, sb, nullptr, st))) return rc;
  // first norm (fbb_core): frame sums, then the running scale of each step
  if ((rc = frame_stats_launch(w.magT, B, St, F, 0, (size_t)St * F, F, w.fs, st))) return rc;
  if ((rc = stream_norm_launch(w.fs, B, St, K, F, g, d->norm_type, w.pos0, w.act0, w.tail, sb, ss, w.scale, st))) return rc;
  // the stack, (h, c) carried in the slot state; its per-step scale keeps it off the paths that read a restart table
  SeqStack s = fbb_stack(d, B, St);
  for (int l = 0; l < s.n; ++l) s.L[l] = layers[l];
  s.x = w.magT; s.scale = w.scale; s.fc_w = fc_w; s.fc_b = fc_b; s.out = w.y;
  if ((rc = stream_seq_stack(s, w.stack, StackCarry{sb, ss, sl.h, sl.c, w.pos0, g, nullptr, K}, st))) return rc;
  return stream_close(g, sl, w, F, B, K, St, win_length, w.y, enhanced, sb, st);
}
