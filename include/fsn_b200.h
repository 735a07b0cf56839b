/*
 * fsn_b200.h - C ABI of libfsn_b200.so: the H100 (sm_90a) implementation of FullSubNet's
 * enhancement hot path (SURVEY.md section 8).
 *
 * The reference (Audio-WestlakeU/FullSubNet) is pure Python and has no FFI; its "operator"
 * boundary is the set of Python callables listed below.  Each entry point here replaces the
 * device work of one of them and is what `fullsubnet_b200/` (the Python host mirroring the
 * reference API) binds through ctypes.  Paths are relative to the upstream repository.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to contiguous fp32 unless noted; the caller allocates
 *     all buffers including the workspace; the library never allocates, frees or retains
 *     DATA pointers across calls, so compute calls are re-entrant across streams and threads.  The
 *     only mutable state it keeps is diagnostic and host-side: the thread-local last-error string /
 *     code, the thread-local profiling switch with its per-stage CUDA events (fsn_set_profiling,
 *     fsn_last_stage_ms), a thread-local launch counter (fsn_last_launch_count) and one process-wide
 *     launch total (fsn_total_launch_count, a relaxed counter); none of it influences results;
 *   - `stream` is a cudaStream_t; nothing synchronises the host;
 *   - return value 0 = ok, non-zero = error; fsn_last_error() gives a thread-local message.
 *     Shape-contract violations that are AssertionError / NotImplementedError in the reference
 *     come back as FSN_ERR_SHAPE / FSN_ERR_UNSUPPORTED and the Python host re-raises them as
 *     the reference's exception types.
 */
#ifndef FSN_B200_H
#define FSN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* fsn_stream_t; /* cudaStream_t */

enum {
  FSN_OK = 0,
  FSN_ERR_SHAPE = 1,       /* reference: AssertionError */
  FSN_ERR_UNSUPPORTED = 2, /* reference: NotImplementedError */
  FSN_ERR_CUDA = 3,
  FSN_ERR_WORKSPACE = 4
};

enum { FSN_ACT_NONE = 0, FSN_ACT_RELU = 1, FSN_ACT_TANH = 2, FSN_ACT_RELU6 = 3 };
/* FSN_NORM_CUMULATIVE_LAPLACE (audio_zen/model/base_model.py:220-251): causal running mean per clip (first norm) and
 * per sub-band unit (second norm); built for the fp32 inference path of fsn_model_forward / fsn_enhance, and for
 * fast_fullsubnet (fsn_fast_desc.norm_type) on every precision of inference and training.
 * FSN_NORM_FORGETTING (base_model.py:102-151, forgetting_norm): causal exponential running mean per clip, mu_t =
 * a_t mu_{t-1} + b_t m_t with alpha = 191/193 from frame 192 on (a_0 = -1, so mu_0 = 2 m_0; a_1 = 0), x / (mu_t + 1e-10),
 * computed in the reference's float32 operation order.  One scale per (clip, frame) at both sites: over the F bins for
 * the first norm, over all F * (2Ns+1 + 2Nf+1) unfolded features for fullsubnet's second norm.  Built for fullsubnet
 * (fsn_model_desc) and fullband_baseline (fsn_fullband_desc) wherever FSN_NORM_CUMULATIVE_LAPLACE runs: every inference
 * precision and cell, the training steps on fp32 and tf32.  fsn_fast_desc and the improved_fullsubnet paths refuse it
 * (FSN_ERR_UNSUPPORTED before any CUDA call).  An addition at version 102 (see fsn_version). */
/* The values follow the order of the reference's norm_wrapper (base_model.py:356-372); 2 (offline_gaussian_norm) and 3
 * (cumulative_layer_norm) are not built and are refused everywhere. */
enum { FSN_NORM_OFFLINE_LAPLACE = 0, FSN_NORM_CUMULATIVE_LAPLACE = 1, FSN_NORM_FORGETTING = 4 };
enum { FSN_CELL_LSTM = 0, FSN_CELL_GRU = 1 };
/* arithmetic of the sub-band LSTM stack (99 % of the FLOPs):
 *   FSN_PREC_FP32     - fp32 FMA everywhere (bit-for-bit class of the reference CPU path, ~1e-6)
 *   FSN_PREC_TF32_TC  - training step only (fsn_train_*): every GEMM of the forward, of back-propagation through
 *                       time and of the weight gradients on wgmma tf32 (fp32 data read as tf32, fp32
 *                       accumulate); gate / cell arithmetic and all reductions stay fp32
 *   FSN_PREC_F16_TC   - fp16 operands (11-bit significand, like TF32) x fp32 accumulate on the
 *                       wgmma tensor cores, fp32 cell state; cRM within 1e-3 rel (tests)
 *   FSN_PREC_F16X3_TC - error-compensated tensor-core path: weights and state split into fp16 hi + lo terms, every
 *                       product issued as W_hi.S_hi + W_hi.S_lo + W_lo.S_hi into one fp32 accumulator (22
 *                       significand bits per operand), libm-class gate functions; the fp32 error class (cRM ~1e-6
 *                       rel), needed where decompress_cIRM amplifies mask errors x100 (|cRM| near the 9.9 clip) */
enum { FSN_PREC_FP32 = 0, FSN_PREC_F16_TC = 1, FSN_PREC_TF32_TC = 2, FSN_PREC_F16X3_TC = 3 };

/* ABI version: 101 changed fsn_enhance's argument list; 102 appended norm_type to fsn_fast_desc, so that struct grew.
 * The version counts changes that break an existing caller.  Entry points added since 102 leave every earlier argument
 * list and struct as it was, so the version stays 102; a caller finds them by symbol: fsn_cirm_mse_per_clip (+ its
 * workspace query), fsn_si_sdr_lengths (the grouped validation loss and SI-SDR), fsn_clip_adam_steps (one Adam step
 * count per tensor), fsn_stoi (+ its workspace query and the fsn_debug_stoi_stages hook) and fsn_resample (+ its
 * workspace query).  FSN_NORM_FORGETTING is a new
 * value of an existing field, refused by every older entry point it does not apply to, with the fsn_debug_forgetting_*
 * hooks.  fsn_improved_weights grew sb_packed, read only by the FSN_PREC_F16X3_TC / FSN_PREC_F16_TC precisions that
 * fsn_improved_forward / _enhance accept since, with fsn_improved_packed_bytes / fsn_improved_pack_sb_weights and the
 * fsn_debug_imp_section_lstm_tc hook: a caller of the shorter struct never selects them, so the version stays 102.  The
 * dense GEMM layer's unit-test hooks fsn_debug_fc_gemm, fsn_debug_sgemm, fsn_debug_colsum, fsn_debug_small_out_wgrad,
 * fsn_debug_transpose, fsn_debug_transpose_blocked and fsn_debug_gemm_tc are new symbols only, and so are the hooks of the
 * causal-norm scales, the layout kernels and the sub-band heads (fsn_debug_cum_clip_scale .. fsn_debug_train_dy), and of
 * the full-band recurrence alone (fsn_debug_lstm_rec_tc + its scratch query). */
int fsn_version(void);
const char* fsn_last_error(void);
/* status code (FSN_ERR_*) of the last failed call on this thread: lets the *_workspace_bytes() functions, which
 * return 0 on failure, report WHY (shape error vs unsupported configuration) */
int fsn_last_error_code(void);
/* compile-time facts for the host (sm arch the kernels were built for, e.g. 100) */
int fsn_built_arch(void);

/* ------------------------------------------------------------------------------------------
 * audio_zen/acoustics/feature.py:9-50  stft(y, n_fft, hop_length, win_length)
 *   wav [B,L] -> mag, phase, real, imag, each [B,F,T]; F = n_fft/2+1, T = 1 + L/hop.
 *   torch.stft semantics: center=True reflect pad n_fft/2, periodic hann (zero-padded to n_fft
 *   when win_length < n_fft), one-sided, un-normalised.  `phase` may be NULL (not computed).
 *   `magT` (optional, may be NULL): a second, time-major copy [B, T_pad, F] with rows
 *   T..T_pad-1 zeroed - the layout the model kernels consume (look-ahead pad fused,
 *   recipes/dns_interspeech_2020/fullsubnet/model.py:85).
 * ---------------------------------------------------------------------------------------- */
int fsn_stft(const float* wav, int B, int L, int n_fft, int hop, int win_length,
             float* mag, float* phase, float* real, float* imag,
             float* magT, int T_pad, fsn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * audio_zen/acoustics/feature.py:53-91  istft(features, n_fft, hop, win, length, input_type)
 *   real/imag [B,F,T] with element stride `cstride` (1 = planar "real_imag", 2 = interleaved
 *   complex64) -> wav [B,out_len].  torch.istft semantics: irfft (1/N), window, overlap-add,
 *   divide by the window-square envelope, trim n_fft/2, cut/zero-pad to `length`
 *   (length <= 0: hop*(T-1)).
 *   If `crm` != NULL ([B,2,F,T], recipes/dns_interspeech_2020/inferencer.py:130-145) the
 *   spectrum is first multiplied by decompress_cIRM(crm) (audio_zen/acoustics/mask.py:47-64,
 *   K=10, limit=9.9) as a complex mask - rows A9 of SURVEY 8a in one kernel.
 * ---------------------------------------------------------------------------------------- */
int fsn_istft(const float* real, const float* imag, int cstride, const float* crm,
              int B, int T, int n_fft, int hop, int win_length, int length,
              float* wav, fsn_stream_t stream);

/* audio_zen/acoustics/mask.py:47-64 / :32-44 / :7-29 (elementwise, n = number of elements) */
int fsn_decompress_cirm(const float* in, float* out, int64_t n, float K, float limit, fsn_stream_t stream);
int fsn_compress_cirm(const float* in, float* out, int64_t n, float K, float C, fsn_stream_t stream);
/* noisy/clean real/imag [n] -> cIRM [n,2] (compressed, K=10, C=0.1) */
int fsn_build_cirm(const float* nr, const float* ni, const float* cr, const float* ci,
                   float* out, int64_t n, fsn_stream_t stream);
/* audio_zen/acoustics/feature.py:309-345  drop_band: in [B,C,F,T] -> out [B,C,F/G,T] */
int fsn_drop_band(const float* in, float* out, int B, int C, int F, int T, int G, fsn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * recipes/dns_interspeech_2020/fullsubnet/model.py:9-136  Model
 * ---------------------------------------------------------------------------------------- */
typedef struct fsn_model_desc {
  int32_t num_freqs;        /* F */
  int32_t look_ahead;
  int32_t fb_num_neighbors; /* Nf */
  int32_t sb_num_neighbors; /* Ns */
  int32_t fb_hidden;        /* 512 */
  int32_t sb_hidden;        /* 384 */
  int32_t fb_activation;    /* FSN_ACT_* (fb_output_activate_function) */
  int32_t sb_activation;    /* FSN_ACT_* (sb_output_activate_function) */
  int32_t norm_type;        /* FSN_NORM_*: offline, cumulative or forgetting (inference on every precision and cell,
                             * training on fp32 and tf32) */
  int32_t num_groups_in_drop_band; /* applied when B > 1 (model.py:114), 1 = off */
  int32_t precision;        /* FSN_PREC_* for the sub-band stack */
  int32_t cell_type;        /* FSN_CELL_*: `sequence_model` = "LSTM" | "GRU" (sequence_model.py:52-66); GRU: weights
                             * [3H,K] with gate order r,z,n, inference on the fp32 kernels (FSN_PREC_FP32) only */
} fsn_model_desc;

/* One SequenceModel (audio_zen/model/module/sequence_model.py:26-125): 2-layer nn.LSTM +
 * Linear, PyTorch parameter layout (gate order i,f,g,o; weight [4H,K] row-major).  Pointers
 * go straight into the nn.Parameter storage so Adam / checkpoints / DDP keep working. */
typedef struct fsn_seq_weights {
  const float* w_ih[2];
  const float* w_hh[2];
  const float* b_ih[2];
  const float* b_hh[2];
  const float* fc_w; /* [out, H] */
  const float* fc_b; /* [out] */
} fsn_seq_weights;

/* bytes of caller-provided scratch for fsn_model_forward / fsn_enhance at batch B, T frames */
size_t fsn_model_workspace_bytes(const fsn_model_desc* d, int B, int T);

/* FSN_PREC_F16_TC / FSN_PREC_F16X3_TC only: bytes of, and packer for, the tile-ordered fp16 image of the sub-band
 * weights that the tensor-core kernel streams (cache it keyed on the parameters' version AND the precision: the
 * compensated image carries a hi and a lo stage per k range). */
size_t fsn_sb_packed_bytes(const fsn_model_desc* d);
int fsn_pack_sb_weights(const fsn_model_desc* d, const fsn_seq_weights* sb, void* packed, fsn_stream_t stream);

/* Model.forward (model.py:72-136): noisy_mag [B,1,F,T] -> crm [B,2,F',T]
 *   F' = F, or F/G with the drop_band batch permutation when B > 1 and G > 1.
 *   sb_packed: NULL for FSN_PREC_FP32. */
int fsn_model_forward(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                      const void* sb_packed, const float* noisy_mag, int B, int T, float* crm,
                      void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* recipes/dns_interspeech_2020/inferencer.py:130-145  Inferencer.full_band_crm_mask, batched over independent clips
 * (drop_band off), with the int16 output of the reference host loop: one call = stft -> model -> decompress/mask ->
 * istft [-> int16].  ABI version 101 changed this entry point: it now takes the argument list of fsn_fullband_enhance
 * (lengths, pcm and gain), and version 100's separate int16 and per-clip-length entry points are gone.  Row b of wav
 * [B, L_max] holds clip b's lengths[b] samples; samples at index >= lengths[b] are never read.  lengths: HOST int32 [B],
 * nullable (= every clip L_max samples), n_fft/2 < lengths[b] <= L_max and max(lengths) == L_max (else FSN_ERR_SHAPE
 * naming the clip); copied into the workspace through kernel parameters during the call and not retained, so it may be
 * pageable and may be reused as soon as the call returns.  Outputs, T_max = 1 + L_max/hop:
 *   enhanced [B, L_max]           required (NULL: FSN_ERR_SHAPE); 0 past lengths[b]
 *   crm_out  [B, 2, F, T_max]     nullable; the model's output, 0 for frames t >= T_b = 1 + lengths[b]/hop
 *   pcm      [B, L_max] int16     nullable; int16(gain * y / max|y|) over the clip's own samples, 0 past lengths[b]
 *                                 (audio_zen/inferencer/base_inferencer.py:181-182, gain = 0.8 * 32767; max|y| per
 *                                 clip is reduced in the iSTFT epilogue, so only 2 bytes per sample go back to the host)
 * With lengths, every clip's outputs are bit-identical to a null-lengths call on that clip alone with L = lengths[b]: the
 * recurrent stages are causal, so they run over T_max + look_ahead steps for every clip, and only the STFT, the offline
 * norms, the iSTFT and the int16 scaling are bounded per clip; n_fft must then be a power of two (else
 * FSN_ERR_UNSUPPORTED).  Never allocates, never synchronises the host. */
size_t fsn_enhance_workspace_bytes(const fsn_model_desc* d, int B, int L_max, int n_fft, int hop);
int fsn_enhance(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                const void* sb_packed, const float* wav, const int32_t* lengths, int B, int L_max, int n_fft, int hop,
                int win_length, float* enhanced, float* crm_out, int16_t* pcm, float gain, void* workspace,
                size_t workspace_bytes, fsn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * recipes/dns_interspeech_2020/fast_fullsubnet/model.py:11-202  Model (BASELINE config 4, SURVEY 8a row A13)
 *   MelScale(F->M) -> norm -> encoder LSTM(M->He1), LSTM(He1->He2)+Linear(M)+ReLU -> unfold(noisy mel, Nn) ||
 *   unfold(encoder out, Ne) -> real-time down-sampling x`shrink` -> norm -> bottleneck 2xLSTM(Hb)+Linear(1)+ReLU on
 *   B*M rows -> up-sampling -> decoder LSTM(2M->Hd), LSTM(Hd->Hd)+Linear(2F) -> [B,2,F,T].  fp32 kernels.
 * ---------------------------------------------------------------------------------------- */
typedef struct fsn_lstm_layer {
  const float* w_ih; /* [4H, K] */
  const float* w_hh; /* [4H, H] */
  const float* b_ih;
  const float* b_hh;
} fsn_lstm_layer;

typedef struct fsn_fast_desc {
  int32_t num_freqs;   /* encoder_input_size (257) */
  int32_t look_ahead;
  int32_t shrink_size;
  int32_t num_mels;    /* 64 */
  int32_t enc1_hidden; /* 384 */
  int32_t enc2_hidden; /* 257 */
  int32_t bn_hidden;   /* bottleneck_hidden_size */
  int32_t bn_layers;   /* bottleneck_num_layers (2) */
  int32_t dec_hidden;  /* 512 */
  int32_t noisy_num_neighbors; /* noisy_input_num_neighbors */
  int32_t enc_num_neighbors;   /* encoder_output_num_neighbors */
  int32_t precision;           /* FSN_PREC_* for the bottleneck stack (the tensor-core path needs bn_hidden = 384) */
  int32_t cell_type;           /* FSN_CELL_* (`sequence_model`); inference and training are built for LSTM only */
  int32_t norm_type;           /* FSN_NORM_* of both norms (model.py:170,187); every precision, inference and training.
                                * FSN_NORM_CUMULATIVE_LAPLACE: one scale per (clip, frame) over the mel bins for the
                                * encoder, one per (clip, mel row, shrunk step) over the K features for the bottleneck.
                                * Other values -> FSN_ERR_UNSUPPORTED before any CUDA call.  Appended in ABI version 102. */
} fsn_fast_desc;

typedef struct fsn_fast_weights {
  const float* mel_fb;  /* mel_scale.fb [F, M] */
  fsn_lstm_layer enc1, enc2;
  const float* enc_fc_w; const float* enc_fc_b;   /* [M, He2], [M] */
  fsn_lstm_layer bn[2];
  const float* bn_fc_w; const float* bn_fc_b;     /* [1, Hb], [1] */
  fsn_lstm_layer dec1, dec2;
  const float* dec_fc_w; const float* dec_fc_b;   /* [2F, Hd], [2F] */
  const void* bn_packed;  /* FSN_PREC_F16_TC: fsn_fast_pack_bn_weights() image of the bottleneck stack, else NULL */
} fsn_fast_weights;

size_t fsn_fast_workspace_bytes(const fsn_fast_desc* d, int B, int T);
/* FSN_PREC_F16_TC: 0 when the tensor-core path cannot run this descriptor */
size_t fsn_fast_packed_bytes(const fsn_fast_desc* d);
int fsn_fast_pack_bn_weights(const fsn_fast_desc* d, const fsn_fast_weights* w, void* packed, fsn_stream_t stream);
/* Model.forward (fast_fullsubnet/model.py:143-202): mix_mag [B,1,F,T] -> [B,2,F,T] */
int fsn_fast_model_forward(const fsn_fast_desc* d, const fsn_fast_weights* w, const float* mix_mag, int B, int T,
                           float* out, void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * recipes/dns_interspeech_2020/improved_fullsubnet/model.py:452-591  Model (BASELINE config 5, SURVEY 8a row A14)
 *   wav -> STFT -> |X|^fdrc, Nyquist bin dropped -> norm -> full-band 2xLSTM + Linear -> per sub-band section:
 *   strided unfold (centre/neighbour widths) of noisy and full-band output, concat, per-section norm, 2xLSTM +
 *   Linear(2*centre) -> cRM (Nyquist row 0) -> element-wise mask on (re, im) -> iSTFT -> wav.  n_fft: a power of two
 *   in [16, 2048] (radix-2 FFT), or even in [16, 1200] (direct DFT; the reference's 48 kHz example uses n_fft = 960).
 * ---------------------------------------------------------------------------------------- */
#define FSN_IMP_MAX_SECTIONS 8
typedef struct fsn_improved_desc {
  int32_t n_fft, hop_length, win_length, num_freqs;
  float fdrc;
  int32_t num_sections;                       /* len(sb_num_center_freqs) = len(freq_cutoffs) + 1 */
  int32_t freq_cutoffs[FSN_IMP_MAX_SECTIONS];
  int32_t sb_num_center[FSN_IMP_MAX_SECTIONS], sb_num_neighbor[FSN_IMP_MAX_SECTIONS];
  int32_t fb_num_center[FSN_IMP_MAX_SECTIONS], fb_num_neighbor[FSN_IMP_MAX_SECTIONS];
  int32_t fb_hidden, sb_hidden, fb_activation, sb_activation;
  int32_t precision; /* inference (fsn_improved_forward / _enhance):
                      *   FSN_PREC_FP32     - fp32 FMA kernels
                      *   FSN_PREC_TF32_TC  - the sections' layers on wgmma tf32, one launch per layer and step
                      *                       (sb_hidden % 4 == 0)
                      *   FSN_PREC_F16X3_TC - each section's input projection on the compensated tf32 GEMM, both LSTM
                      *                       layers of all steps in one persistent fp16 hi+lo wgmma launch, the head once
                      *                       over all steps; the full band on the compensated tensor-core layers.
                      *                       sb_hidden in {128, 256, 384}; needs w->sb_packed (the fp32 error class)
                      *   FSN_PREC_F16_TC   - the same with single fp16 / tf32 passes (cRM within 1e-3 rel)
                      * training (fsn_improved_train_*): FSN_PREC_FP32 or FSN_PREC_TF32_TC only */
  int32_t cell_type; /* FSN_CELL_* (`sequence_model`); read by the training step only, which is built for LSTM */
} fsn_improved_desc;

typedef struct fsn_improved_weights {
  fsn_seq_weights fb;                          /* fb_model */
  fsn_seq_weights sb[FSN_IMP_MAX_SECTIONS];    /* sb_model.sb_models[s] */
  /* FSN_PREC_F16X3_TC / FSN_PREC_F16_TC: fsn_improved_pack_sb_weights() image of section s, else unread (NULL).
   * Appended after 102: only those precisions read it, so a caller built against the shorter struct is unaffected. */
  const void* sb_packed[FSN_IMP_MAX_SECTIONS];
} fsn_improved_weights;

/* Packed section weights of the fp16 tensor-core precisions, mirroring fsn_fast_pack_bn_weights: the tile-ordered fp16
 * (x3: hi + lo) image of section s's W_hh0, W_ih1, W_hh1 and layer-1 biases that its persistent kernel streams (W_ih0 and
 * the Linear run outside it).  fsn_improved_packed_bytes: 0 (fsn_last_error_code set, no CUDA call) for other precisions,
 * unsupported shapes or section outside [0, num_sections).  fsn_improved_pack_sb_weights fills `packed` on `stream`
 * from w->sb[section]; rebuild it whenever those weights change (cache it keyed on their version and the precision).
 * No allocation, no host synchronisation. */
size_t fsn_improved_packed_bytes(const fsn_improved_desc* d, int section);
int fsn_improved_pack_sb_weights(const fsn_improved_desc* d, const fsn_improved_weights* w, int section, void* packed,
                                 fsn_stream_t stream);

size_t fsn_improved_workspace_bytes(const fsn_improved_desc* d, int B, int L);
/* Model.forward (improved_fullsubnet/model.py:541-591): wav [B,L] -> enhanced [B,L] (the reference returns
 * [B,1,L]); crm_out optional [B,2,F,T] */
int fsn_improved_forward(const fsn_improved_desc* d, const fsn_improved_weights* w, const float* wav, int B, int L,
                         float* enhanced, float* crm_out, void* workspace, size_t workspace_bytes,
                         fsn_stream_t stream);
/* Clips of different lengths in one call, with the int16 output of the reference host loop.  Row b of wav [B, L_max]
 * holds clip b's lengths[b] samples; samples at index >= lengths[b] are never read.  lengths: HOST int32 [B], nullable
 * (= every clip L_max samples), n_fft/2 < lengths[b] <= L_max and max(lengths) == L_max (else FSN_ERR_SHAPE naming the
 * clip); copied into the workspace through kernel parameters during the call and not retained.  Outputs, T_max = 1 +
 * L_max/hop_length:
 *   enhanced [B, L_max]           required (NULL: FSN_ERR_SHAPE); 0 past lengths[b]
 *   crm_out  [B, 2, F, T_max]     nullable; Nyquist row 0, and 0 for frames t >= T_b = 1 + lengths[b]/hop_length
 *   pcm      [B, L_max] int16     nullable; int16(gain * y / max|y|) over the clip's own samples, 0 past lengths[b]
 * Every clip's outputs are bit-identical to fsn_improved_forward on that clip alone with L = lengths[b] (and pcm to
 * fsn_peak_normalize_int16 of that waveform): the full-band stack, the section LSTMs and their Linear are causal and run
 * over T_max steps for every clip; only the STFT, the full-band and section norms, the iSTFT and the int16 scaling are
 * bounded per clip.  Same precisions and n_fft sizes as fsn_improved_forward.  Never allocates, never synchronises the
 * host. */
size_t fsn_improved_enhance_workspace_bytes(const fsn_improved_desc* d, int B, int L_max);
int fsn_improved_enhance(const fsn_improved_desc* d, const fsn_improved_weights* w, const float* wav,
                         const int32_t* lengths, int B, int L_max, float* enhanced, float* crm_out, int16_t* pcm,
                         float gain, void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* Opt-in stage timing for bench.py: when enabled, fsn_model_forward / fsn_enhance bracket their
 * stages with CUDA events on `stream` (thread-local, created lazily).  After the caller has
 * synchronised the stream, fsn_last_stage_ms(stage) returns the device time of the last call:
 * stage 0 = stft (or mag transpose), 1 = norms + full-band stack, 2 = sub-band stack, 3 = mask+istft. */
int fsn_set_profiling(int enable);
float fsn_last_stage_ms(int stage);

/* number of kernel launches issued by the last fsn_model_forward / fsn_enhance on this thread
 * (bench.py reports it as gpu_launches) */
int64_t fsn_last_launch_count(void);
/* kernels launched by this library since it was loaded (never reset): difference two readings */
int64_t fsn_total_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Training step: recipes/dns_interspeech_2020/fullsubnet/trainer.py:56-68 (SURVEY 8a row A11), fp32.
 *   fsn_train_forward   = Model.forward in train mode (model.py:72-136, drop_band on) that keeps the activations
 *                         back-propagation through time needs in `workspace` (same buffer must be passed to
 *                         fsn_train_backward, untouched in between)
 *   fsn_mse_loss        = audio_zen/loss.py:4 (torch.nn.MSELoss) between cIRM [B',F',T,2] (trainer.py:49-54) and
 *                         cRM [B',2,F',T]; also writes d loss / d cRM when dcrm != NULL.  loss: device scalar.
 *   fsn_train_backward  = loss.backward() (trainer.py:63): gradients of the 20 parameters, OVERWRITTEN into the
 *                         buffers of gfb / gsb (same shapes as the parameters)
 *   fsn_clip_adam       = clip_grad_norm_(max_norm) + Adam step (trainer.py:65-68, train.py:55-59) over a list of
 *                         tensors, no host synchronisation.  grad_scale multiplies every gradient first (1/world
 *                         after a sum all-reduce).  norm_out (optional, 2 floats on the device) receives the total
 *                         norm and the applied coefficient; gradients are left clipped like the reference.
 *                         Every tensor is at the same step (>= 1).
 *   fsn_clip_adam_steps = fsn_clip_adam with one step per tensor, as torch.optim.Adam keeps one per parameter (a
 *                         parameter skipped while its grad was None, a resumed checkpoint): steps is a HOST array of
 *                         L->n entries, each >= 1, read during the call and not retained.  Tensor i gets the bias
 *                         corrections of steps[i]; with every entry equal the outputs are those of fsn_clip_adam bit
 *                         for bit.  Arguments are checked before any CUDA call. */
typedef struct fsn_seq_grads {
  float* w_ih[2];
  float* w_hh[2];
  float* b_ih[2];
  float* b_hh[2];
  float* fc_w;
  float* fc_b;
} fsn_seq_grads;

size_t fsn_train_workspace_bytes(const fsn_model_desc* d, int B, int T);
int fsn_train_forward(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                      const float* noisy_mag, int B, int T, float* crm, void* workspace, size_t workspace_bytes,
                      fsn_stream_t stream);
int fsn_train_backward(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                       const float* dcrm, int B, int T, const fsn_seq_grads* gfb, const fsn_seq_grads* gsb,
                       void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* Training step of recipes/dns_interspeech_2020/fast_fullsubnet/trainer.py:45-56 (the fast recipe), same conventions as
 * fsn_train_*: the caller allocates the workspace and passes the same untouched buffer from forward to backward; the
 * gradients of the 30 parameters are OVERWRITTEN; no host synchronisation; arguments are checked before any CUDA call.
 *   fsn_fast_train_forward  = Model.forward in train mode (fast_fullsubnet/model.py:143-202): out [B,2,F,T], keeping the
 *                             activations back-propagation through time needs (time-major [Tp, rows, .])
 *   fsn_fast_train_backward = loss.backward() from dout = d loss / d out [B,2,F,T]
 * d->precision: FSN_PREC_FP32, or FSN_PREC_TF32_TC (every LSTM layer with H % 4 == 0 on the wgmma tf32 GEMMs, as in
 * fsn_train_*); any other precision, bn_layers != 2 or the GRU cell -> FSN_ERR_UNSUPPORTED. */
typedef struct fsn_lstm_grads { float *w_ih, *w_hh, *b_ih, *b_hh; } fsn_lstm_grads;
typedef struct fsn_fast_grads {
  fsn_lstm_grads enc1, enc2;  float *enc_fc_w, *enc_fc_b;
  fsn_lstm_grads bn[2];       float *bn_fc_w,  *bn_fc_b;
  fsn_lstm_grads dec1, dec2;  float *dec_fc_w, *dec_fc_b;
} fsn_fast_grads;
size_t fsn_fast_train_workspace_bytes(const fsn_fast_desc* d, int B, int T);
int fsn_fast_train_forward(const fsn_fast_desc* d, const fsn_fast_weights* w, const float* mix_mag, int B, int T,
                           float* out, void* workspace, size_t workspace_bytes, fsn_stream_t stream);
int fsn_fast_train_backward(const fsn_fast_desc* d, const fsn_fast_weights* w, const float* dout, int B, int T,
                            const fsn_fast_grads* g, void* workspace, size_t workspace_bytes, fsn_stream_t stream);

size_t fsn_mse_loss_scratch_bytes(void);
int fsn_mse_loss(const float* cirm, const float* crm, int B, int Fsub, int T, float* loss, float* dcrm,
                 void* scratch, size_t scratch_bytes, fsn_stream_t stream);

/* Validation loss of recipes/dns_interspeech_2020/fullsubnet/trainer.py:78-181 for B clips at once (an addition at
 * version 102, see fsn_version).  Clip b is the first lengths[b] samples of row b of noisy_wav / clean_wav [B,L_max] (lengths: host int32 [B], nullable = all
 * L_max; n_fft/2 < lengths[b] <= L_max and max == L_max), and crm [B,2,F,T_max] (F = n_fft/2+1, T_max = 1 + L_max/hop)
 * is the model output on it.  loss[b] (device [B]) = MSE between the compressed cIRM of the clip's two STFTs
 * (fsn_build_cirm) and crm over its own T_b = 1 + lengths[b]/hop frames, reduced with the partition and tree of
 * fsn_mse_loss at B = 1, T = T_b: bit-identical to fsn_stft + fsn_build_cirm + fsn_mse_loss on that clip alone.  No
 * drop_band (the reference validates at B = 1).  Every argument is checked before any CUDA call; the workspace query
 * needs no device and returns 0 for a refused shape. */
size_t fsn_cirm_mse_per_clip_workspace_bytes(int B, int L_max, int n_fft, int hop);
int fsn_cirm_mse_per_clip(const float* noisy_wav, const float* clean_wav, const int32_t* lengths, int B, int L_max,
                          int n_fft, int hop, int win_length, const float* crm, float* loss, void* workspace,
                          size_t workspace_bytes, fsn_stream_t stream);

#define FSN_MAX_PARAM_TENSORS 64
typedef struct fsn_param_list {
  int n;
  float* param[FSN_MAX_PARAM_TENSORS];
  float* grad[FSN_MAX_PARAM_TENSORS];
  float* exp_avg[FSN_MAX_PARAM_TENSORS];
  float* exp_avg_sq[FSN_MAX_PARAM_TENSORS];
  int64_t numel[FSN_MAX_PARAM_TENSORS];
} fsn_param_list;

size_t fsn_clip_adam_scratch_bytes(void);
int fsn_clip_adam(const fsn_param_list* L, float max_norm, float grad_scale, float lr, float beta1, float beta2,
                  float eps, int step, float* norm_out, void* scratch, size_t scratch_bytes, fsn_stream_t stream);
int fsn_clip_adam_steps(const fsn_param_list* L, float max_norm, float grad_scale, float lr, float beta1, float beta2,
                        float eps, const int* steps, float* norm_out, void* scratch, size_t scratch_bytes,
                        fsn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * recipes/dns_interspeech_2020/fullband_baseline/model.py:8-68  Model (SURVEY 8f rank 3)
 *   look-ahead pad -> norm -> num_layers x LSTM(F -> H) -> Linear(H -> 2F) [+ activation] -> [B,2,F,T].
 *   layers: num_layers entries (PyTorch parameter layout); fc_w [2F,H], fc_b [2F].
 * Inference (fsn_fullband_forward, fsn_fullband_enhance) runs the fp32 kernels for FSN_PREC_FP32 and FSN_PREC_TF32_TC;
 * FSN_PREC_F16X3_TC / FSN_PREC_F16_TC -> FSN_ERR_UNSUPPORTED (the tensor-core stack misses the reference gates on
 * this model). */
typedef struct fsn_fullband_desc {
  int32_t num_freqs;
  int32_t hidden;
  int32_t num_layers; /* the reference builds 3 */
  int32_t look_ahead;
  int32_t activation; /* FSN_ACT_* */
  int32_t norm_type;  /* FSN_NORM_*: offline, cumulative or forgetting, inference and training */
  int32_t precision;  /* FSN_PREC_FP32 (0) or FSN_PREC_TF32_TC (training: the tf32 GEMMs; inference: fp32 kernels) */
  int32_t cell_type;  /* FSN_CELL_* (0 = LSTM; inference and training are built for LSTM only) */
} fsn_fullband_desc;

size_t fsn_fullband_workspace_bytes(const fsn_fullband_desc* d, int B, int T);
int fsn_fullband_forward(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w, const float* fc_b,
                         const float* noisy_mag, int B, int T, float* out, void* workspace, size_t workspace_bytes,
                         fsn_stream_t stream);
/* wav -> wav: the fullband_baseline Model inside Inferencer.full_band_crm_mask (recipes/dns_interspeech_2020/
 * inferencer.py:130-145: stft -> model -> decompress_cIRM -> complex product -> istft) for B clips in one call, with the
 * int16 output of the reference host loop.  Row b of wav [B, L_max] holds clip b's lengths[b] samples; samples at index
 * >= lengths[b] are never read.  lengths: HOST int32 [B], nullable (= every clip L_max samples), n_fft/2 < lengths[b] <=
 * L_max and max(lengths) == L_max (else FSN_ERR_SHAPE naming the clip); copied into the workspace through kernel
 * parameters during the call and not retained.  n_fft / 2 + 1 must equal num_freqs.  Outputs, T_max = 1 + L_max/hop:
 *   enhanced [B, L_max]           required (NULL: FSN_ERR_SHAPE); 0 past lengths[b]
 *   crm_out  [B, 2, F, T_max]     nullable; the model's output, 0 for frames t >= T_b = 1 + lengths[b]/hop
 *   pcm      [B, L_max] int16     nullable; int16(gain * y / max|y|) over the clip's own samples, 0 past lengths[b]
 * With null lengths, enhanced equals fsn_stft -> fsn_fullband_forward -> fsn_istft bit for bit and crm_out equals
 * fsn_fullband_forward; any n_fft fsn_stft / fsn_istft accept.  With lengths, every clip's outputs are bit-identical to
 * a null-lengths call on that clip alone with L = lengths[b] (and pcm to fsn_peak_normalize_int16 of that waveform): the
 * stack is causal and runs over T_max + look_ahead steps for every clip; only the STFT, the offline norm, the iSTFT and
 * the int16 scaling are bounded per clip.  n_fft must then be a power of two (else FSN_ERR_UNSUPPORTED).  Same precisions,
 * norms and cells as fsn_fullband_forward.  Never allocates, never synchronises the host. */
size_t fsn_fullband_enhance_workspace_bytes(const fsn_fullband_desc* d, int B, int L_max, int n_fft, int hop);
int fsn_fullband_enhance(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w, const float* fc_b,
                         const float* wav, const int32_t* lengths, int B, int L_max, int n_fft, int hop, int win_length,
                         float* enhanced, float* crm_out, int16_t* pcm, float gain, void* workspace,
                         size_t workspace_bytes, fsn_stream_t stream);

/* Chunked streaming enhancement of fullband_baseline (DESIGN 4.14): many streams, each advanced by K hops per call, with
 * the output of every clip bit-identical to fsn_fullband_enhance on the whole clip (lengths NULL, B = 1).  Appended in
 * ABI version 102.
 *
 * A stream state is a caller-allocated device buffer of B slots, fsn_fullband_stream_state_bytes(d, B, n_fft, hop)
 * bytes, ZERO-FILLED before its first use (every slot then holds no clip).  Slot b's state is the contiguous block of
 * state_bytes / B bytes at b * state_bytes / B, so checkpointing or moving a stream is a device copy of its block.  A
 * block holds: the slot's position and whether a clip runs (16 bytes); the last (c+1) hop + n_fft/2 input samples; the
 * spectrum of the last Rc + look_ahead frames and the cRM of the last Rc frames (Rc = ceil(n_fft/hop) + 2); the norm's
 * accumulator (cumulative: running frame sum, forgetting: mu); h and c of every LSTM layer (2 x num_layers x hidden
 * floats).  Here c = ceil((n_fft/2) / hop).
 *
 * fsn_fullband_stream_step: wav [B, K*hop], the next K hops of every slot.  start / tail: HOST int32 [B], nullable,
 * copied through kernel parameters (not retained):
 *   start[b] != 0  slot b begins a new clip with this chunk (its state is re-initialised inside the call);
 *   tail[b] >= 0   slot b's clip ends after tail[b] <= K*hop samples of this chunk; the slot is free afterwards.
 *                  -1: the clip goes on.  Anything else -> FSN_ERR_SHAPE.  Ignored on a slot without a clip.
 * enhanced [B, K*hop + D]: for a slot whose clip is at sample pos before the call, the first K*hop samples of its row
 * are clip samples [pos - D, pos - D + K*hop) (negative indices as 0) and the rest 0; on the call that ends the clip,
 * the row holds clip samples [pos - D, pos + tail[b]) and 0 after them.  A slot without a clip gets a row of 0.
 * D = fsn_fullband_stream_delay(d, n_fft, hop) = n_fft/2 + (look_ahead + 1 + c) hop samples, the same for every K and
 * schedule (a negative return is minus the FSN_ERR_* code).  A clip must have more than n_fft/2 samples and at most
 * 2^30 (18.6 h at 16 kHz): the position is an int32 sample count.  The call cannot check either (the position lives on
 * the device); a shorter clip reflects at a clamped index and a longer one wraps, so the output of such a clip is
 * undefined, and the other slots are unaffected.  B > 65535 slots -> FSN_ERR_UNSUPPORTED.
 * The workspace is fsn_fullband_stream_workspace_bytes(d, B, K_max, n_fft, hop) bytes; it serves every K <= K_max.
 * Built for the cumulative_laplace_norm and forgetting_norm models, LSTM cell, FSN_PREC_FP32, power-of-two n_fft in
 * [16, 2048]; the offline norm (it needs the whole clip), the GRU cell, other precisions and other n_fft ->
 * FSN_ERR_UNSUPPORTED before any CUDA call, from the queries (which return 0) as from the call.  Never allocates,
 * never synchronises the host; one call may be captured in a CUDA graph. */
size_t fsn_fullband_stream_state_bytes(const fsn_fullband_desc* d, int B, int n_fft, int hop);
size_t fsn_fullband_stream_workspace_bytes(const fsn_fullband_desc* d, int B, int K_max, int n_fft, int hop);
int fsn_fullband_stream_delay(const fsn_fullband_desc* d, int n_fft, int hop);
int fsn_fullband_stream_step(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                             const float* fc_b, const float* wav, const int32_t* start, const int32_t* tail, int B, int K,
                             int n_fft, int hop, int win_length, float* enhanced, void* state, size_t state_bytes,
                             void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* Chunked streaming enhancement of fast_fullsubnet (DESIGN 4.14), with the semantics of the fullband_baseline calls
 * above: many streams, each advanced by K hops per call, the output of every clip bit-identical to fsn_stft ->
 * fsn_fast_model_forward -> fsn_istft on the whole clip (B = 1), delayed by D = fsn_fast_stream_delay(d, n_fft, hop) =
 * n_fft/2 + (look_ahead + 1 + c) hop samples, c = ceil((n_fft/2) / hop): the down-sampled bottleneck adds no delay (frame
 * t reads shrunk step floor(t / shrink_size), whose block ends at frame floor(t / shrink_size) * shrink_size <= t).
 * Appended in ABI version 102.
 *
 * State: fsn_fast_stream_state_bytes(d, B, n_fft, hop) bytes, ZERO-FILLED before its first use, slot b's block at
 * b * state_bytes / B.  A block holds the slot's position (16 bytes), the last (c+1) hop + n_fft/2 input samples, the
 * spectrum of the last Rc + look_ahead frames and the cRM of the last Rc frames (Rc = ceil(n_fft/hop) + 2), the last
 * shrink_size - 1 frames of the mel spectrogram and of the encoder output, the first norm's running sum, h and c of the
 * encoder and decoder layers, and per mel row the second norm's running sum, the latest bottleneck output and h and c of
 * both bottleneck layers (2 x 2 x num_mels x bn_hidden floats: 393 216 of the recipe's 431 360 bytes per slot).
 * fsn_fast_stream_step: wav, start, tail, enhanced, workspace (fsn_fast_stream_workspace_bytes(d, B, K_max, n_fft, hop),
 * every K <= K_max) and the clip-length limits as fsn_fullband_stream_step.  Built for the cumulative_laplace_norm model,
 * LSTM cell, FSN_PREC_FP32, power-of-two n_fft in [16, 2048] with n_fft/2 + 1 = num_freqs; the offline norm, the
 * tensor-core precisions, the GRU cell, other n_fft and B > 65535 -> FSN_ERR_UNSUPPORTED (n_fft/2 + 1 != num_freqs:
 * FSN_ERR_SHAPE) before any CUDA call, from the queries (which return 0) as from the call.  Never allocates, never
 * synchronises the host; one call may be captured in a CUDA graph. */
size_t fsn_fast_stream_state_bytes(const fsn_fast_desc* d, int B, int n_fft, int hop);
size_t fsn_fast_stream_workspace_bytes(const fsn_fast_desc* d, int B, int K_max, int n_fft, int hop);
int fsn_fast_stream_delay(const fsn_fast_desc* d, int n_fft, int hop);
int fsn_fast_stream_step(const fsn_fast_desc* d, const fsn_fast_weights* w, const float* wav, const int32_t* start,
                         const int32_t* tail, int B, int K, int n_fft, int hop, int win_length, float* enhanced,
                         void* state, size_t state_bytes, void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* The same stream on the fp16 tensor cores (DESIGN 4.14.2): d->precision FSN_PREC_F16X3_TC or FSN_PREC_F16_TC, the output
 * of every clip bit-identical to fsn_stft -> fsn_fast_model_forward -> fsn_istft of that precision on the whole clip
 * (B = 1), delayed by D = fsn_fast_stream_tc_delay(d, n_fft, hop), the fsn_fast_stream_delay of the same shape.  The state
 * is the fp32 stream's slot layout, byte for byte (fsn_fast_stream_tc_state_bytes = fsn_fast_stream_state_bytes of the
 * FSN_PREC_FP32 descriptor): h and c stay fp32, and the bottleneck kernel splits h into fp16 hi / lo on load as it does
 * after every step.  w->bn_packed: the fsn_fast_pack_bn_weights image fsn_fast_model_forward takes.  Semantics, limits
 * and buffers as fsn_fast_stream_step; FSN_PREC_FP32, the offline norm, the GRU cell, bottleneck shapes the tensor-core
 * kernel cannot take (bn_hidden != 384, bn_layers != 2, input width > 32), other n_fft and B > 65535 ->
 * FSN_ERR_UNSUPPORTED (n_fft/2 + 1 != num_freqs: FSN_ERR_SHAPE), a null bn_packed -> FSN_ERR_SHAPE, before any CUDA
 * call.  The number of kernel launches of a call does not depend on K.  Appended in ABI version 102. */
size_t fsn_fast_stream_tc_state_bytes(const fsn_fast_desc* d, int B, int n_fft, int hop);
size_t fsn_fast_stream_tc_workspace_bytes(const fsn_fast_desc* d, int B, int K_max, int n_fft, int hop);
int fsn_fast_stream_tc_delay(const fsn_fast_desc* d, int n_fft, int hop);
int fsn_fast_stream_tc_step(const fsn_fast_desc* d, const fsn_fast_weights* w, const float* wav, const int32_t* start,
                            const int32_t* tail, int B, int K, int n_fft, int hop, int win_length, float* enhanced,
                            void* state, size_t state_bytes, void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* Chunked streaming enhancement of fullsubnet (DESIGN 4.14), with the semantics of the fullband_baseline calls above:
 * many streams, each advanced by K hops per call, the output of every clip bit-identical to fsn_enhance on the whole
 * clip (lengths NULL, B = 1), delayed by D = fsn_stream_delay(d, n_fft, hop) = n_fft/2 + (look_ahead + 1 + c) hop
 * samples, c = ceil((n_fft/2) / hop).  Every slot is a B = 1 clip, so drop_band never applies, whatever
 * num_groups_in_drop_band says.  Appended in ABI version 102.
 *
 * State: fsn_stream_state_bytes(d, B, n_fft, hop) bytes, ZERO-FILLED before its first use, slot b's block at
 * b * state_bytes / B.  A block holds the slot's position and the first norm's accumulator (16 bytes), the last (c+1) hop
 * + n_fft/2 input samples, the spectrum of the last Rc + look_ahead frames and the cRM of the last Rc frames (Rc =
 * ceil(n_fft/hop) + 2), the second norm's accumulator (cumulative: one running sum per frequency, forgetting: mu), h and
 * c of both full-band layers, and h and c of both sub-band layers for every frequency (2 x 2 x num_freqs x sb_hidden
 * floats: 1 579 008 of the recipe's 1 612 032 bytes per slot with the cumulative norm).  fsn_stream_step: wav, start, tail, enhanced, workspace
 * (fsn_stream_workspace_bytes(d, B, K_max, n_fft, hop), every K <= K_max) and the clip-length limits as
 * fsn_fullband_stream_step; fb / sb as fsn_enhance.  Built for the cumulative_laplace_norm and forgetting_norm models,
 * LSTM cell, FSN_PREC_FP32, power-of-two n_fft in [16, 2048] with n_fft/2 + 1 = num_freqs; the offline norm, the GRU
 * cell, the tensor-core precisions, other n_fft and B > 65535 -> FSN_ERR_UNSUPPORTED (n_fft/2 + 1 != num_freqs:
 * FSN_ERR_SHAPE) before any CUDA call, from the queries (which return 0) as from the call; B x num_freqs x sb_hidden >=
 * 2^31 -> FSN_ERR_SHAPE from the call.  Never allocates, never synchronises the host; one call may be captured in a
 * CUDA graph. */
size_t fsn_stream_state_bytes(const fsn_model_desc* d, int B, int n_fft, int hop);
size_t fsn_stream_workspace_bytes(const fsn_model_desc* d, int B, int K_max, int n_fft, int hop);
int fsn_stream_delay(const fsn_model_desc* d, int n_fft, int hop);
int fsn_stream_step(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb, const float* wav,
                    const int32_t* start, const int32_t* tail, int B, int K, int n_fft, int hop, int win_length,
                    float* enhanced, void* state, size_t state_bytes, void* workspace, size_t workspace_bytes,
                    fsn_stream_t stream);

/* The same stream on the fp16 tensor cores (DESIGN 4.14.1): d->precision FSN_PREC_F16X3_TC or FSN_PREC_F16_TC, the
 * output of every clip bit-identical to fsn_enhance of that precision on the whole clip (lengths NULL, B = 1), delayed
 * by D = fsn_stream_tc_delay(d, n_fft, hop), the fsn_stream_delay of the same shape.  The state is the fp32 stream's
 * slot layout, byte for byte (fsn_stream_tc_state_bytes = fsn_stream_state_bytes of the FSN_PREC_FP32 descriptor): h and
 * c stay fp32, and the kernels split h into fp16 hi / lo on load as they do after every step.  sb_packed: the
 * fsn_pack_sb_weights image fsn_enhance takes.  Semantics, limits and buffers as fsn_stream_step; FSN_PREC_FP32, the
 * offline norm, the GRU cell, sub-band shapes the tensor-core kernel cannot take, other n_fft and B > 65535 ->
 * FSN_ERR_UNSUPPORTED, a null sb_packed -> FSN_ERR_SHAPE, before any CUDA call.  Appended in ABI version 102. */
size_t fsn_stream_tc_state_bytes(const fsn_model_desc* d, int B, int n_fft, int hop);
size_t fsn_stream_tc_workspace_bytes(const fsn_model_desc* d, int B, int K_max, int n_fft, int hop);
int fsn_stream_tc_delay(const fsn_model_desc* d, int n_fft, int hop);
int fsn_stream_tc_step(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                       const void* sb_packed, const float* wav, const int32_t* start, const int32_t* tail, int B, int K,
                       int n_fft, int hop, int win_length, float* enhanced, void* state, size_t state_bytes,
                       void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* Training step of recipes/dns_interspeech_2020/fullband_baseline/trainer.py:32-71, same conventions as fsn_train_*: the
 * caller allocates the workspace and passes the same untouched buffer from forward to backward; the gradients of all
 * 4 * num_layers + 2 parameters are OVERWRITTEN; no host synchronisation; arguments are checked before any CUDA call;
 * every sum runs in a fixed order (two runs give identical bits).
 *   fsn_fullband_train_forward  = Model.forward with gradients enabled: out [B,2,F,T], keeping the activations
 *                                 back-propagation through time needs (time-major [Tp, B, .])
 *   fsn_fullband_train_backward = loss.backward() from dout = d loss / d out [B,2,F,T]; g->layer[l] for l < num_layers
 * d->precision: FSN_PREC_FP32, or FSN_PREC_TF32_TC (the LSTM layers on the wgmma tf32 GEMMs when hidden % 4 == 0, as in
 * fsn_train_*); any other precision, the GRU cell, num_layers outside 1..8 or another norm -> FSN_ERR_UNSUPPORTED. */
typedef struct fsn_fullband_grads {
  fsn_lstm_grads layer[8];
  float *fc_w, *fc_b;
} fsn_fullband_grads;
size_t fsn_fullband_train_workspace_bytes(const fsn_fullband_desc* d, int B, int T);
int fsn_fullband_train_forward(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                               const float* fc_b, const float* noisy_mag, int B, int T, float* out, void* workspace,
                               size_t workspace_bytes, fsn_stream_t stream);
int fsn_fullband_train_backward(const fsn_fullband_desc* d, const fsn_lstm_layer* layers, const float* fc_w,
                                const float* fc_b, const float* dout, int B, int T, const fsn_fullband_grads* g,
                                void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* Training step of improved_fullsubnet (improved_fullsubnet/model.py:452-591 is a differentiable module, wav in and wav
 * out; upstream ships no trainer, so any loss on the enhanced waveform drives it), same conventions as fsn_train_*: the
 * caller allocates the workspace and passes the same untouched buffer from forward to backward; every gradient is
 * OVERWRITTEN; no host synchronisation; arguments are checked before any CUDA call; every sum runs in a fixed order (two
 * runs give identical bits).
 *   fsn_improved_train_forward  = Model.forward with gradients enabled: wav [B,L] -> enhanced [B,L], keeping the noisy
 *                                 spectrum, the normalised section inputs and their scales, the gates / cells / hidden
 *                                 states of every LSTM layer and the post-activation outputs (time-major [T, rows, .])
 *   fsn_improved_train_backward = loss.backward() from d_enhanced = d loss / d enhanced [B,L]; no input gradient
 * d->precision: FSN_PREC_FP32, or FSN_PREC_TF32_TC (every LSTM layer with H % 4 == 0 on the wgmma tf32 GEMMs, as in
 * fsn_train_*).  The GRU cell, another precision, fb_activation / sb_activation other than none or ReLU -> FSN_ERR_UNSUPPORTED;
 * shapes as fsn_improved_forward. */
typedef struct fsn_improved_grads {
  fsn_seq_grads fb;                          /* fb_model */
  fsn_seq_grads sb[FSN_IMP_MAX_SECTIONS];    /* sb_model.sb_models[s] */
} fsn_improved_grads;
size_t fsn_improved_train_workspace_bytes(const fsn_improved_desc* d, int B, int L);
int fsn_improved_train_forward(const fsn_improved_desc* d, const fsn_improved_weights* w, const float* wav, int B, int L,
                               float* enhanced, void* workspace, size_t workspace_bytes, fsn_stream_t stream);
int fsn_improved_train_backward(const fsn_improved_desc* d, const fsn_improved_weights* w, const float* d_enhanced, int B,
                                int L, const fsn_improved_grads* g, void* workspace, size_t workspace_bytes,
                                fsn_stream_t stream);

/* audio_zen/inferencer/base_inferencer.py:181-182 (SURVEY 8f rank 2): out = int16(gain * wav / max|wav|) per clip,
 * gain = 0.8 * 32767 in the reference; float32 multiply, divide, truncation toward zero like numpy; all-zero clip -> 0 */
int fsn_peak_normalize_int16(const float* wav, int B, int L, float gain, int16_t* out, fsn_stream_t stream);

/* audio_zen/metrics.py:6-31  SI_SDR(reference, estimation) (SURVEY 8f rank 4: the validation metric of
 * fullsubnet/trainer.py:78-181; STOI is fsn_stoi below, PESQ (ITU-T P.862) stays out).
 * reference, estimation [B,L] -> out[B] in dB; fixed-order reductions. */
int fsn_si_sdr(const float* reference, const float* estimation, int B, int L, float* out, fsn_stream_t stream);
/* fsn_si_sdr over the first lengths[b] samples of each row of [B,L_max] (lengths: host int32 [B], 0 < lengths[b] <=
 * L_max, checked before any CUDA call; NULL = fsn_si_sdr).  out[b] is bit-identical to fsn_si_sdr on that clip alone.
 * An addition at version 102 (see fsn_version). */
int fsn_si_sdr_lengths(const float* reference, const float* estimation, const int32_t* lengths, int B, int L_max,
                       float* out, fsn_stream_t stream);

/* audio_zen/metrics.py:STOI  pystoi 0.3.3 stoi(clean, estimate, sr, extended=False) (Taal et al., 2011) per clip:
 * resampling to 10 kHz (Octave-style Kaiser-windowed sinc, scipy resample_poly), silent-frame removal at 40 dB below the
 * clean clip's loudest 256-sample frame, 512-point spectra of the rebuilt signals, 15 one-third-octave bands from 150 Hz,
 * clipped (-15 dB) and normalised correlations over 30-frame segments.  Fewer than 30 frames after the removal give
 * 1e-5, as pystoi returns.  Computed in float64 from the widened inputs; out[b] float32.
 *   clean, estimate [B,L_max]; out [B]; sr 16000 or 10000 (other rates FSN_ERR_UNSUPPORTED).
 *   lengths (nullable, host int32 [B], read during the call through kernel parameters, not kept): clip b is the first
 *     lengths[b] samples of its rows, samples from there on are never read; NULL = every clip L_max.  Each clip needs one
 *     frame: at least 410 samples at 16 kHz, 257 at 10 kHz (shorter: FSN_ERR_SHAPE naming the clip).
 *   out[b] is bit-identical to the call on clip b alone with L_max = lengths[b], whatever B and the clip's position
 *   (one CTA per clip for every reduction, fixed orders, the kept frames compacted by a per-clip scan), and two calls
 *   give the same bits.  Never allocates or synchronises; every argument (B > 0, pointers, lengths, workspace size:
 *   FSN_ERR_WORKSPACE) is checked before any CUDA call.
 * fsn_stoi_workspace_bytes: the workspace of any call with these B, L_max and sr (~32 * B * L_max * 10000/sr bytes); 0
 * with fsn_last_error set on bad arguments; needs no GPU.  An addition at version 102 (see fsn_version). */
size_t fsn_stoi_workspace_bytes(int B, int L_max, int sr);
int fsn_stoi(const float* clean, const float* estimate, const int32_t* lengths, int B, int L_max, int sr, float* out,
             void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* fullsubnet_b200/inferencer.py  Inferencer.resample(y, sr_in, sr_out, zeros) per clip: the hann-windowed sinc that brings
 * a wav file at another rate to the model's (the stand-in for librosa.load(path, sr=sr)'s soxr, not bit-identical to
 * soxr).  g = gcd(sr_in, sr_out), up = sr_out/g, down = sr_in/g, cutoff = min(1, up/down), half = ceil(zeros/cutoff).
 *   x [B, N_max]; clip b is its first N_b = lengths[b] samples (lengths: nullable, host int32 [B], read during the call
 *     through kernel parameters, not kept; NULL = every clip N_max; 1 <= lengths[b] <= N_max).
 *   y [B, N_out_max]: row b holds n_out_b = ceil(N_b * up / down) samples (integer arithmetic: the host's float64
 *     ceiling for N_b * up < 2^53), 0 from there on; N_out_max must be at least the largest n_out_b.
 *   Output n, in float64 as the host: t = n * down / up, taps idx = floor(t) + k for k in [-half + 1, half], d = t - idx,
 *     w = cutoff * sinc(cutoff * d) * (0.5 + 0.5 * cos(pi * clip(d / half, -1, 1))) (numpy's sinc), taps outside
 *     [0, N_b) contribute 0; the products are summed in float64 in ascending k and the sum is rounded once to float32.
 *     CUDA's sin / cos differ from the host's libm by up to 2 ulp, so an output can differ from the host's by one float32
 *     rounding step; almost all are bit-identical (DESIGN 4.10.1).  sr_in == sr_out copies the input bits.
 *   Checks, all before any CUDA call: B > 0, N_max > 0, positive rates, zeros >= 1, x, y non-null, the lengths and
 *   N_out_max (FSN_ERR_SHAPE); B > 65535 or half > 2^29 (FSN_ERR_UNSUPPORTED); the workspace (FSN_ERR_WORKSPACE).
 *   Never allocates, never synchronises the host; one call may be captured in a CUDA graph.
 * fsn_resample_workspace_bytes: the workspace of any call with these arguments (the device length table, 256-byte
 * aligned); 0 with fsn_last_error set on bad arguments; needs no GPU.  An addition at version 102 (see fsn_version). */
size_t fsn_resample_workspace_bytes(int B, int N_max, int sr_in, int sr_out, int zeros);
int fsn_resample(const float* x, const int32_t* lengths, int B, int N_max, int sr_in, int sr_out, int zeros, float* y,
                 int N_out_max, void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* recipes/dns_interspeech_2020/dataset_train.py:136-199  Dataset.snr_mix for a batch (SURVEY 8f rank 4): the random
 * draws (snr, noisy target dBFS, which RIR) are made by the caller and passed in.
 *   fsn_rir_convolve: out[b,:L] = fftconvolve(x[b], rir[b,:rir_len[b]])[:L]  (dataset_train.py:161; direct form,
 *                     rir [B,Lr_max], rir_len[b] == 0 copies the clip; rir_len may be NULL = Lr_max everywhere)
 *   fsn_snr_mix:      norm_amplitude + tailor_dB_FS(target_dB_FS) of clean and noise, noise scaled to snr[b] dB,
 *                     mixture tailored to noisy_target_dB_FS[b] (clean by the same factor), both divided by
 *                     max|noisy| / (0.99 - eps) when the mixture exceeds 0.999 (audio_zen/acoustics/feature.py:99-114). */
int fsn_rir_convolve(const float* x, const float* rir, const int* rir_len, int B, int L, int Lr_max, float* out,
                     fsn_stream_t stream);
int fsn_snr_mix(const float* clean, const float* noise, const float* snr, const float* noisy_target_dB_FS,
                float target_dB_FS, float eps, int B, int L, float* noisy_out, float* clean_out, fsn_stream_t stream);

/* unit-test hooks (host code only): the drop_band row map of Model.forward and its inverse (-1 = unit dropped), and
 * the reflect-padding multiplicity c[r] of the closed-form second norm (SURVEY 8a rows A6 / A7) */
int fsn_debug_row_to_unit(int B, int F, int G, int r, int* b, int* f);
int fsn_debug_unit_to_row(int B, int F, int G, int b, int f);
int fsn_debug_reflect_count(int r, int F, int N);

/* unit-test hook for the tf32 wgmma GEMM of the training path: C[M,N] (+)= A[M,K] B[N,K]^T, fp32 row-major
 * operands with 16-byte aligned rows; scratch (optional) enables split-K */
int fsn_debug_tgemm(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M, int N,
                    int K, int accumulate, float* scratch, int64_t scratch_floats, fsn_stream_t stream);

/* unit-test hook for the weight-gradient GEMMs of the training step (dW = dG^T X, torch autograd of nn.LSTM):
 * C[M,N] = A[a_k0:a_k0+K, :M]^T B[b_k0:b_k0+K, :N] for row-major A [a_k0+K, M], B [b_k0+K, N]; both operands are first
 * copied into the block-tiled K-major layout the TMA loads stream (a_k0, b_k0 multiples of 32); scratch holds the two
 * copies (rounded up to 128 x 32 tiles) followed by split-K space */
int fsn_debug_tgemm_blocked(const float* A, const float* B, float* C, int M, int N, int K, int a_k0, int b_k0,
                            float* scratch, int64_t scratch_floats, fsn_stream_t stream);

/* unit-test hook for the fused forward step of the training path (one LSTM step of torch.nn.LSTM as used by
 * audio_zen/model/module/sequence_model.py:52-58): z = x W_ih^T (or the projection already in G) + b_ih + b_hh +
 * h_prev W_hh^T; G [R,4H] <- post-activation gates (i,f,g,o), c_out = f c_prev + i g, h_out = o tanh(c_out).
 * h_prev, c_prev nullable (first step); x nullable (G then holds x W_ih^T on entry).  half != 0: fp16 MMA operands
 * for h and W_hh, and for x and W_ih when K0 % 8 == 0 (else those stay tf32 in the same k loop, as in the training
 * forward); converted into scratch, >= 2 * (2 R H + 4 H (H + K0) + R K0) + 1024 bytes; H % 32 == 0 */
int fsn_debug_lstm_fwd_step(const float* h_prev, const float* w_hh, const float* x, const float* w_ih, int K0, float* G,
                            const float* b_ih, const float* b_hh, const float* c_prev, float* c_out, float* h_out, int R,
                            int H, int half, void* scratch, int64_t scratch_bytes, fsn_stream_t stream);

/* unit-test hooks of the dense GEMM layer, each running the launch function its callers use; every argument (null
 * pointers, non-positive sizes, leading dimensions, short scratch: FSN_ERR_WORKSPACE) is checked before any CUDA call.
 *   fsn_debug_fc_gemm:   out[M,O] = act(A[M,K] W^T + bias) in fp32 (bias nullable); W [O,K], or [K,O] with w_kmajor
 *   fsn_debug_sgemm:     C[M,N] (+)= op(A) B in fp32, op(A) = A [M,K] (lda) or, ta != 0, A stored [K,M]; B [K,N] (ldb);
 *                        long K with few tiles splits K over scratch (fewer slices when scratch_floats is short)
 *   fsn_debug_colsum:    out[c] (and out2[c] when given) = sum_r X[r*ldx + c]; scratch >= min(ceil(rows/2048), 512) *
 *                        cols floats
 *   fsn_debug_small_out_wgrad: dW [2,H] = dout[rows,2]^T Hm[rows,H] (the sub-band Linear's weight gradient); scratch
 *                        >= 2 H floats (more lets it split the rows)
 *   fsn_debug_transpose: out [cols,rows] = in [rows,cols]^T
 *   fsn_debug_transpose_blocked: the block-tiled K-major copy of in [K,M] (row stride ld) that the weight-gradient
 *                        GEMMs stream: element (k, m) at ((m/128 * ceil(K/32) + k/32) * 128 + m%128) * 32 + k%32, zero
 *                        padded to whole 128 x 32 tiles; colsum_part (nullable, >= max_slabs * M floats): also the
 *                        column sums of in into bias_out [M] over at most max_slabs slabs (*slabs, nullable, = count)
 *   fsn_debug_gemm_tc:   out[rows, :N] (row stride ldo) = act(x' W^T + bias) on the tf32 tensor cores (x3: hi/lo
 *                        compensated), x' = x[rows, :K] (row stride ldx) times row_scale[r / rows_per_scale] or, with
 *                        scale_B > 0, row_scale[(r % rows_per_scale) * scale_B + r / rows_per_scale] (row_scale
 *                        nullable); workspace: the prepared operands, align256(rows Kp p 4) + align256(4 max(8, ceil(N/4)) Kp p 4)
 *                        bytes with Kp = K rounded up to 4, p = 3 for x3 else 1 (fsn_debug_lstm_tc_workspace_bytes(rows,
 *                        1, K, max(8, ceil(N/4)), x3) is more than that) */
int fsn_debug_fc_gemm(const float* A, const float* W, const float* bias, float* out, int M, int K, int O, int act,
                      int w_kmajor, fsn_stream_t stream);
int fsn_debug_sgemm(int ta, const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M, int N,
                    int K, int accumulate, float* scratch, int64_t scratch_floats, fsn_stream_t stream);
int fsn_debug_colsum(const float* X, int64_t rows, int cols, int64_t ldx, float* out, float* out2, float* scratch,
                     int64_t scratch_floats, fsn_stream_t stream);
int fsn_debug_small_out_wgrad(const float* dout, const float* Hm, int64_t rows, int H, float* dW, float* scratch,
                              int64_t scratch_floats, fsn_stream_t stream);
int fsn_debug_transpose(const float* in, int64_t rows, int cols, float* out, fsn_stream_t stream);
int fsn_debug_transpose_blocked(const float* in, int64_t K, int M, int64_t ld, float* out, float* colsum_part,
                                int max_slabs, int* slabs, float* bias_out, fsn_stream_t stream);
int fsn_debug_gemm_tc(const float* x, int64_t ldx, int K, const float* row_scale, int rows_per_scale, int scale_B,
                      const float* W, int N, const float* bias, int act, int x3, float* out, int64_t ldo, int64_t rows,
                      void* workspace, size_t workspace_bytes, fsn_stream_t stream);

/* unit-test hooks for the tensor-core LSTM layer of the full-band stacks (fsn_lstm_rec_tc.cu;
 * audio_zen/model/module/sequence_model.py:52-58,117): hall[r,t,:] of nn.LSTM(K -> H, 1 layer) over x [R,T,K]
 * (hoisted input-projection GEMM + persistent wgmma recurrence), and out = act(x W^T + b) for x [rows,K], W [N,K];
 * x3 != 0 selects the compensated (fp32-class) arithmetic.  Workspace of the Linear hook: the LSTM one with
 * R*T = rows, H = max(8, ceil(N/4)). */
size_t fsn_debug_lstm_tc_workspace_bytes(int R, int T, int K, int H, int x3);
int fsn_debug_lstm_layer_tc(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* x,
                            int R, int T, int K, int H, int x3, float* hall, void* workspace, size_t workspace_bytes,
                            fsn_stream_t stream);
int fsn_debug_linear_tc(const float* x, int rows, int K, const float* W, const float* bias, int N, int act, int x3,
                        float* out, void* workspace, size_t workspace_bytes, fsn_stream_t stream);
/* the same layer continued from a carried state (the tensor-core stream's full band): row r enters step 0 with h_init /
 * c [r*H + u] and step restart[r] with zero state (restart[r] = 0: they are ignored); c after step fin_step (-1: none) is
 * written back to c, h of every step is in hall.  Workspace: fsn_debug_lstm_tc_workspace_bytes. */
int fsn_debug_lstm_tc_carry(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* x,
                            int R, int T, int K, int H, int x3, const float* h_init, float* c, const int32_t* restart,
                            int fin_step, float* hall, void* workspace, size_t workspace_bytes, fsn_stream_t stream);
/* the recurrence of that layer alone (lstm_rec_tc_kernel / lstm_rec_tc_carry_kernel), on a given input projection
 * P[r*p_row + t*p_t + gate*H + u] (gate order i, f, g, o), h_t into hall[r*h_row + t*h_t + u]; P and hall 8-byte aligned,
 * p_t >= 4H, p_row >= (T-1) p_t + 4H, h_t >= H, h_row >= (T-1) h_t + H.  restart NULL: zero initial state (h_init,
 * c_init, c_fin must be NULL); otherwise row r enters step 0 with h_init / c_init [r*c_row + u] (c_row >= H) and step
 * restart[r] with zero state, and c after step fin_step (-1: none) goes to c_fin [r*c_row + u] (c_fin may be c_init).
 * info (nullable, 4 ints): rows per cooperative launch, TMA ring stages, launches, dynamic shared memory bytes.  Scratch:
 * fsn_debug_lstm_rec_tc_scratch_bytes, the same for every H.  Every argument is checked before any CUDA call; an
 * unsupported H (FSN_ERR_UNSUPPORTED) is reported after those checks.  fsn_debug_lstm_layer_tc, fsn_debug_lstm_tc_carry
 * and fsn_debug_linear_tc check theirs the same way, except that the layer hooks report H below the kernel's minimum
 * (64) as unsupported before they look at the workspace. */
size_t fsn_debug_lstm_rec_tc_scratch_bytes(int H, int x3);
int fsn_debug_lstm_rec_tc(const float* w_hh, const float* b_ih, const float* b_hh, const float* P, int64_t p_row, int64_t p_t,
                          float* hall, int64_t h_row, int64_t h_t, int R, int T, int H, int x3, const float* h_init,
                          const float* c_init, float* c_fin, int64_t c_row, const int32_t* restart, int fin_step, int* info,
                          void* scratch, size_t scratch_bytes, fsn_stream_t stream);

/* unit-test hook for the sub-band tensor-core stack (fsn_subband_tc.cu; model.py:98-135): packs sb (2 LSTM layers of
 * hidden size H over Ksb = (2Ns+1)+(2Nf+1) inputs, Linear(H -> fc_out <= 2)) into `packed`
 * (fsn_debug_sb_lstm_tc_packed_bytes, 0 = unsupported H) and runs the stack on magT, fbT [B, src_T, F] (time-major):
 * unit (b', f') of the drop_band map (G groups, as Model.forward applies them) gathers the reflected rows of its source
 * clip, scaled by inv2[clip] or, when unit_scale [steps, B*Fsub] is given, by unit_scale[t*R + r]; shrink > 1
 * down-samples time like fast_fullsubnet.  crm [B, 2, Fsub, steps - la] receives act(Linear) of steps la..steps-1
 * (outputs beyond fc_out are act(0)).  stages (2..4) and cluster (1, 2, 4 CTA pairs that share each half's weight
 * stream; a hardware cluster is 2 x cluster CTAs) choose the launch configuration, 0 = the FSN_TC_STAGES /
 * FSN_TC_CLUSTER default.  Arguments are checked before any CUDA call. */
size_t fsn_debug_sb_lstm_tc_packed_bytes(int H, int x3);
/* *clusters = how many clusters of the sub-band kernel (2 x cluster CTAs each) can be resident at once on the current
 * device for that launch configuration (cudaOccupancyMaxActiveClusters) */
int fsn_debug_sb_lstm_tc_max_clusters(int H, int x3, int stages, int cluster, int* clusters);
int fsn_debug_sb_lstm_tc(const fsn_seq_weights* sb, int H, int Ns, int Nf, int fc_out, int act, int x3,
                         const float* magT, const float* fbT, int B, int F, int src_T, int G,
                         const float* inv2, const float* unit_scale, int la, int steps, int shrink,
                         int stages, int cluster, void* packed, float* crm, fsn_stream_t stream);
/* the two-pass stack of the whole-clip fullsubnet enhance (one kernel per layer, 48 rows per CTA pair, h0 through h0ws)
 * on the inputs of fsn_debug_sb_lstm_tc with fc_out 2 and no down-sampling; rows run chunk_pairs x 48 at a time
 * (0 = the production chunk), h0ws holds fsn_debug_sb_lstm_tc2_ws_bytes(B*Fsub, steps, H, x3, chunk_pairs) bytes (0 =
 * unsupported H).  Same bits as fsn_debug_sb_lstm_tc.  Arguments are checked before any CUDA call. */
size_t fsn_debug_sb_lstm_tc2_ws_bytes(int R, int steps, int H, int x3, int chunk_pairs);
int fsn_debug_sb_lstm_tc2(const fsn_seq_weights* sb, int H, int Ns, int Nf, int act, int x3, const float* magT,
                          const float* fbT, int B, int F, int src_T, int G, const float* inv2, const float* unit_scale,
                          int la, int steps, int stages, int chunk_pairs, void* packed, void* h0ws, float* crm,
                          fsn_stream_t stream);
/* one pass (layer 0 or 1) of that stack over one chunk: the CTA pairs [pair0, pair0 + pairs) of 48 rows, launched as
 * the production loop launches a chunk.  Layer 0 writes only h0ws: the fp16 image of the chunk's pair p at step t at
 * byte (p*steps + t)*img, img = (x3 ? 2 : 1) * H * 96, the 128B-swizzled k-blocks of 64 units x 48 rows, hi blocks
 * before lo blocks.  Layer 1 reads h0ws as given and writes only those pairs' rows of crm.  h0ws_bytes >= pairs *
 * steps * img.  Errors: FSN_ERR_SHAPE (layer, shape, pairs beyond the rows, missing buffer), FSN_ERR_WORKSPACE (h0ws),
 * FSN_ERR_UNSUPPORTED (stages, H, input width), each before any CUDA call. */
int fsn_debug_sb_tc2_pass(const fsn_seq_weights* sb, int H, int Ns, int Nf, int act, int x3, const float* magT,
                          const float* fbT, int B, int F, int src_T, int G, const float* inv2, const float* unit_scale,
                          int la, int steps, int stages, int layer, int pair0, int pairs, void* packed, void* h0ws,
                          size_t h0ws_bytes, float* crm, fsn_stream_t stream);
/* the carry instantiation of the kernel (the tensor-core stream's sub band): B clips of F rows r = b*F + f, no
 * drop_band, look-ahead 0, fc_out 2, unit_scale [steps, B*F] required.  h / c [2 layers, B*F, H] hold the state entering
 * step 0 and receive the state after store_step (-1: none); row r enters step restart[r] with zero state (0: its h / c
 * are ignored); crm [B, steps, 2F] receives act(Linear) of every step, channel-major per frame.  Arguments are checked before
 * any CUDA call. */
int fsn_debug_sb_lstm_tc_carry(const fsn_seq_weights* sb, int H, int Ns, int Nf, int act, int x3, const float* magT,
                               const float* fbT, int B, int F, int src_T, const float* unit_scale, int steps,
                               const int32_t* restart, int store_step, float* h, float* c, void* packed, float* crm,
                               fsn_stream_t stream);
/* the block-phased carry instantiation (fast_fullsubnet's tensor-core stream bottleneck): B slots of M rows r = b*M + m,
 * fc_out 1, ReLU.  Slot b's call step j is frame m0[b] + j of its clip; row q of catM / catE [B, S-1+St, M] is call
 * step q - (S-1).  The input of the nb = ceil(St / S) block ends (frame 0 alone, then blocks of S frames ending on
 * multiples of S) is formed into x [nb, B*M, K] as the whole-clip gather forms it with shrink = S, scaled by scale
 * [nb, B*M] (0 past a slot's last block end in the call); then all nb steps run in one launch.  h / c [2 layers, B*M, H]
 * hold the state entering step 0 and receive slot b's state after step store[b] (-1: none); slot b enters step restart[b]
 * with zero state; out [B, nb, 2M] receives step i's output of row b*M + m at (b, i, m) and the zero-padded second
 * output at (b, i, M + m).  m0, restart and store are device tables [B].  Arguments are checked before any CUDA call. */
int fsn_debug_sb_lstm_tc_phased(const fsn_seq_weights* bn, int H, int Ns, int Nf, int x3, const float* catM,
                                const float* catE, int B, int M, int S, int St, const int32_t* m0, const float* scale,
                                const int32_t* restart, const int32_t* store, float* h, float* c, void* packed, float* x,
                                float* out, fsn_stream_t stream);
/* the same run through the cycle-stamp instantiation of the kernel (same output bits): CTAs [0, stamp_ctas) (at most
 * the 2 * ceil(B * Fsub / 32) CTAs that own rows) record, for the loop iterations [0, stamp_steps) (stamp_steps <=
 * steps + 1: layer 1 runs one iteration behind layer 0), FSN_SB_PROBE_FIELDS int64 per (CTA, iteration, layer, slot)
 * into stamps [stamp_ctas, stamp_steps, 2, FSN_SB_PROBE_SLOTS, FSN_SB_PROBE_FIELDS]: slots 0..2 are the consumer
 * warpgroups (SM clock stamps of the block's start, MMA start, MMA end and end, then the cycles spent in each wait and
 * in the cell; field order in fsn_subband_tc.cu, ProbeField), slot 3 the weight producer (layer-0 record of each
 * iteration).  Records of blocks that do not exist (layer 1 of iteration 0, layer 0 of the last, slots beyond H / 128)
 * are left as they were.  Arguments are checked before any CUDA call. */
#define FSN_SB_PROBE_FIELDS 16
#define FSN_SB_PROBE_SLOTS 4
int fsn_debug_sb_lstm_tc_probe(const fsn_seq_weights* sb, int H, int Ns, int Nf, int fc_out, int act, int x3,
                               const float* magT, const float* fbT, int B, int F, int src_T, int G,
                               const float* inv2, const float* unit_scale, int la, int steps, int shrink,
                               int stages, int cluster, void* packed, float* crm, long long* stamps, int stamp_ctas,
                               int stamp_steps, fsn_stream_t stream);

/* unit-test hook for the LSTM layer shared by the training steps (fsn_train.cu): torch.nn.LSTM(K0, H, num_layers =
 * n_layers) over x [T,R,K0] (time-major) through the same activation-saving forward, BPTT and weight-gradient pieces
 * as fsn_train_* / fsn_fast_train_* / fsn_fullband_train_*, wired like fsn_fullband_train_*.  Layer 0 maps K0 -> H, the
 * others H -> H.  Gradient on top: dh_top [T,R,H] and / or a Linear(H -> O) folded into the top layer, dout [T,R,O] with
 * fc_w [O,H] (dout, fc_w and O >= 1 together, else NULL, NULL, 0).  Outputs: h_top [T,R,H]; dx [T,R,K0] when not NULL;
 * g[l] = the gradients of layer l (overwritten, not accumulated); trace (nullable, n_layers * 5*T*R*H floats): per layer
 * its hidden states [T,R,H] then dG [T,R,4H], the pre-activation gate gradients the weight gradients are built from.
 * precision FSN_PREC_FP32 or FSN_PREC_TF32_TC (per layer as in the training steps), else FSN_ERR_UNSUPPORTED, as are
 * n_layers outside 1..8.  Arguments are checked before any CUDA call; the workspace query needs no GPU. */
size_t fsn_debug_lstm_train_workspace_bytes(int n_layers, int R, int T, int K0, int H, int precision);
int fsn_debug_lstm_train(const fsn_lstm_layer* layers, int n_layers, int R, int T, int K0, int H, int precision,
                         const float* x, const float* dh_top, const float* dout, const float* fc_w, int O, float* h_top,
                         float* dx, const fsn_lstm_grads* g, float* trace, void* workspace, size_t workspace_bytes,
                         fsn_stream_t stream);

/* unit-test hook for the SequenceModel every inference forward runs its clip-major LSTM stacks through (seq_stack_forward,
 * fsn_fullband.cu; audio_zen/model/module/sequence_model.py:106-125): n layers (1..8; LSTM, or GRU with gru != 0) of hidden
 * sizes H[0..n-1] over x [R, Tp, K0] (layer l maps H[l-1] -> H[l]), the layer-0 input times scale[r] (scale [R]) or, with
 * step_scale, scale[t*R + r] (scale [Tp, R]); scale nullable.  Then Linear(H[n-1] -> O) + act (FSN_ACT_*) into
 * out [R, Tp, O].  tc != 0 asks for the tensor-core stack (x3 != 0: compensated) as the model files do: LSTM only, and every
 * H must be supported there (else FSN_ERR_UNSUPPORTED).  force_stepwise != 0 runs the per-step kernels as
 * FSN_FB_STEPWISE does.  *path (nullable) receives the FSN_SEQ_PATH_* the stack ran on.  Arguments are checked before any
 * CUDA call; the workspace query needs no GPU. */
enum { FSN_SEQ_PATH_TC = 0, FSN_SEQ_PATH_PERSISTENT = 1, FSN_SEQ_PATH_STEP2 = 2, FSN_SEQ_PATH_ONE_LAYER = 3 };
size_t fsn_debug_seq_stack_workspace_bytes(int n, const int* H, int R, int Tp, int K0, int gru, int step_scale, int tc, int x3,
                                           int O);
int fsn_debug_seq_stack(const fsn_lstm_layer* layers, int n, const int* H, int R, int Tp, int K0, int gru, int step_scale,
                        int tc, int x3, int force_stepwise, const float* x, const float* scale, const float* fc_w,
                        const float* fc_b, int O, int act, float* out, void* workspace, size_t workspace_bytes, int* path,
                        fsn_stream_t stream);

/* unit-test hooks for the signal layer (fsn_dsp.cu; torch.stft / torch.istft with center=True, reflect padding and a
 * periodic Hann window of win_length centred in n_fft): the internal launchers behind fsn_stft, fsn_istft and the
 * wav -> wav entry points, called directly.  n_fft a power of two in [16, 2048] (radix-2 FFT) or even in [16, 1200]
 * (direct DFT); B <= 65535; the iSTFT refuses a hop whose frames would not fit in shared memory (FSN_ERR_UNSUPPORTED).
 * lengths (nullable, host [B]): per-clip lengths n_fft/2 < lengths[b] <= L (iSTFT: <= its output length), max == L, copied
 * to lens_dev (device [B]) through the kernel parameters.
 *   fsn_debug_stft: wav [B,L] -> any of mag, phase, real, imag [B,F,T] (F = n_fft/2+1, T = 1+L/hop) and magT [B,T_pad,F]
 *     (nullable each); clip b has 1 + lengths[b]/hop frames, the rest are 0.
 *   fsn_debug_istft: [B,F,T] spectrum (real / imag cstride floats apart: 2 for interleaved complex) times crm [B,2,F,T]
 *     (mask_mode 0: none, crm NULL; 1: decompressed cIRM, complex product; 2: element-wise) -> wav [B,length]
 *     (length <= 0: hop*(T-1)); peak_bits (nullable, [B]) <- max|wav| per clip as float bits; pcm (nullable, [B,length],
 *     needs peak_bits) <- int16(gain * wav / peak); crm_out (nullable, [B,2,F,T], needs lengths) zeroed for frames
 *     t >= 1 + lengths[b]/hop.
 *   fsn_debug_istft_mask_adjoint: d loss / d crm [B,2,F,T] of mask_mode 2 with wav length L, for dwav [B,L]; rows f < F-1
 *     (the Nyquist row is not written).
 *   fsn_debug_wav_epilogue: the int16 output and crm_out zeroing of fsn_debug_istft on a caller's enhanced [B,L] and peak.
 * Arguments are checked before any CUDA call. */
int fsn_debug_stft(const float* wav, int B, int L, int n_fft, int hop, int win_length, const int32_t* lengths, int* lens_dev,
                   float* mag, float* phase, float* real, float* imag, float* magT, int T_pad, fsn_stream_t stream);
int fsn_debug_istft(const float* real, const float* imag, int cstride, const float* crm, int mask_mode, int B, int T,
                    int n_fft, int hop, int win_length, int length, const int32_t* lengths, int* lens_dev, float* wav,
                    unsigned int* peak_bits, int16_t* pcm, float gain, float* crm_out, fsn_stream_t stream);
int fsn_debug_istft_mask_adjoint(const float* dwav, const float* real, const float* imag, int B, int L, int T, int n_fft,
                                 int hop, int win_length, float* dcrm, fsn_stream_t stream);
int fsn_debug_wav_epilogue(const float* enhanced, const unsigned int* peak_bits, int B, int L, const int32_t* lengths,
                           int* lens_dev, float gain, int16_t* pcm, float* crm_out, int F, int T, int hop,
                           fsn_stream_t stream);

/* unit-test hooks for the backward of the second norm and the frequency unfold of the training steps (fsn_train.cu,
 * fsn_fast_train.cu, fsn_improved_train.cu): the launchers of the fsn_*_train_backward entry points on caller buffers.
 * Tensors are time-major as in the training steps; act (FSN_ACT_*) is the activation of the kept output whose derivative
 * is taken from that output.
 *   fsn_debug_norm_unfold_bwd (fullsubnet, model.py:98-119): sub-band input X and its gradient dX [Tp, R, K], K = 2Ns+2
 *     (the full-band unit in column K-1), R = B*Fsub rows of the drop_band map with G groups (G <= 1: none, Fsub = F;
 *     else B > G, Fsub = F/G); full-band output fbz [Tp,B,F].  cum = 0: offline norm, scale = inv2 [B], mid = dot [B],
 *     cnt2 = F K Tp in the step; cum != 0: cumulative norm, scale = scaleT [Tp,R], mid = dunit [Tp,R].  dz [Tp,B,F] is
 *     the gradient at the full-band Linear's output (drop_band's removed units keep the offline norm-mean term).
 *   fsn_debug_fast_norm_unfold_bwd (fast_fullsubnet, model.py:174-194): Ts = 1 + ceil((Tp-1)/S) shrunk steps,
 *     K = (2Nn+1)+(2Ne+1), R = B*M.  dbn (nullable) [Ts,R] <- the up-sampling transpose of the columns M..2M-1 of ddec
 *     [Tp,B,2M] times ReLU' of bn_out [Ts,R].  denc (nullable) [Tp,B,M] <- the gradient at the encoder output encT [Tp,B,M]
 *     (post-ReLU) through the second norm, down-sampling and unfold of dX, X [Ts,R,K], plus ddec's columns < M; cum = 0:
 *     scale = inv2 [B], mid = dot [B], cnt2 = M K Ts in the step; cum != 0: scale = scaleT [Ts,R], mid = suffix [Ts,R].
 *   fsn_debug_imp_unfold_bwd (improved_fullsubnet, model.py:321-443): section rows [lo, hi) of Fu with centre widths cs
 *     = cf and neighbours ns, nf (checked as the model descriptor's sections are), N = (hi-lo)/cs units of width
 *     W = (cs+2ns)+(cf+2nf); dX, Xn [T, B*N, W], invs [B].  dot [B] <- <dX, Xn> per clip; dfb [T,B,Fu] <- (first ? 0 : dfb)
 *     + the gradient at the full-band output through the section's norm and unfold, then ReLU' of y [T,B,Fu] when act is
 *     FSN_ACT_RELU (the last section in the step).
 *   fsn_debug_imp_section_input (improved_fullsubnet's forward, the same section): X [T, B*N, W] <- unit n of clip b at
 *     frame t, the noisy rows lo+n*cs-ns .. of magc then the full-band rows lo+n*cf-nf .. of fbT, reflected at rows 0 and
 *     Fu-1 (magc, fbT [B,T,Fu], or [T,B,Fu] when tm); fs [B*T] (float2) <- the sum of each (b, t) block in .x and .y.
 * Arguments are checked before any CUDA call. */
int fsn_debug_norm_unfold_bwd(const float* dX, const float* X, const float* fbz, const float* scale, int cum, int B, int F,
                              int G, int Tp, int Ns, float cnt2, int act, float* mid, float* dz, fsn_stream_t stream);
int fsn_debug_fast_norm_unfold_bwd(const float* ddec, const float* dX, const float* X, const float* encT,
                                   const float* bn_out, const float* scale, int cum, int B, int Tp, int M, int Nn, int Ne,
                                   int S, float cnt2, float* mid, float* denc, float* dbn, fsn_stream_t stream);
int fsn_debug_imp_unfold_bwd(const float* dX, const float* Xn, const float* invs, const float* y, int B, int T, int Fu,
                             int lo, int hi, int cs, int ns, int cf, int nf, int first, int act, float* dot, float* dfb,
                             fsn_stream_t stream);
int fsn_debug_imp_section_input(const float* magc, const float* fbT, int B, int T, int Fu, int lo, int hi, int cs, int ns,
                                int cf, int nf, int tm, float* X, float* fs, fsn_stream_t stream);
/* unit-test hooks of the causal-norm forward scales, the layout kernels and the sub-band heads (fsn_lstm_simt.cu,
 * fsn_fast_model.cu, fsn_improved.cu, fsn_train.cu): the launchers the forwards and training steps run, on caller
 * buffers.  Every argument is checked before any CUDA call; fsn_last_launch_count() gives the kernels a call launched.
 *   fsn_debug_cum_clip_scale: fs [B*Tp] (float2) <- the frame sums of x (element (b,t,f) at b*bs + t*ts + f), then
 *     scale1T [Tp,B] <- 1 / (running mean over the F bins of the frames so far + eps) (cumulative_laplace_norm).
 *   fsn_debug_cum_unit_scale: scaleT [Tp,R] of every sub-band unit of the drop_band map (G <= 1: none; else B > G,
 *     Fsub = F/G, R = B*Fsub): the running mean over its 2Ns+1 reflected magT rows and 2Nf+1 reflected fbT rows; magT /
 *     fbT [B,Tp,F], or [Tp,B,F] with time_major.
 *   fsn_debug_forget_unit_broadcast: unit_scale [Tp,R] <- scaleT [Tp,B] of each row's clip (same map).
 *   fsn_debug_fast_bn: fast_fullsubnet's bottleneck input bn [Ts, B*M, K] (Ts = 1 + ceil((Tp-1)/S), K = 2Nn+2Ne+2) and
 *     its (b, ts) block sums fs [B*Ts] (float2) from melT / encT (element (b,t,m) at b*bs + t*ts + m); cum: scale [Ts,B*M]
 *     <- the second cumulative norm's scales; else sums [B] (float2) and scale [B] <- 1 / (mean over M K Ts + eps).
 *   fsn_debug_fast_dec_input: dec_in rows (b,t) of 2M at b*rbs + t*rts (clip-major rbs = Tp, rts = 1; time-major rbs = 1,
 *     rts = B) <- encT row || the bottleneck output (b, m, min(t/S, Ts-1)) at b*nbs + m*nms + ts*nts.
 *   fsn_debug_transpose_mag: mag [B,F,T] -> out (b,t,f) at b*bs + t*ts + f for t < Tp (frames >= T zero); scaled
 *     (nullable) the same times scale[b].  B <= 65535.
 *   fsn_debug_crm_output: y rows (b,t) of 2F at b*bs + t*ts -> out [B,2,F,Tp-la], dropping the first la frames.
 *     B <= 32767.
 *   fsn_debug_scale_rows: out[i] = in[i] * scale[((i / cols) % rows) / div] for i < n; in may be out.
 *   fsn_debug_imp_compress: mag [B,F,T] -> |mag|^fdrc without the Nyquist bin, [B,T,F-1], or [T,B,F-1] with tm.
 *   fsn_debug_train_gather: X [Tp, R, K] (K = 2Ns+2Nf+2) of the training step's sub-band input from raw / fbz [Tp,B,F]
 *     (same map), times inv2[b], or unit_scale [Tp,R] when given.
 *   fsn_debug_sb_head: act(h W^T + bias) of h [steps, R, H], W [O,H], into frames t0 .. t0+steps-1 of the cRM: output
 *     o = ch*c + j of row r = b*N + n at out[b*bs' + (ch*rows + lo + n*c + j)*rs + t], bs' = bs or (bs = 0) 2*rows*rs;
 *     O <= 2c, R a multiple of N, lo + N c <= rows (rows = 0: one channel, O <= c).
 *   fsn_debug_sb_head_bwd: dY [steps, R, O] <- act'(y) dcrm at frame t - la of the same geometry, 0 for t < la (y, laid
 *     out like dcrm, unread for FSN_ACT_NONE).
 *   fsn_debug_train_dy: dY [Tp,B,2F] <- dout [B,2,F,T] at frame t - la (0 for t < la, Tp = T + la) times act'(y [Tp,B,2F]).
 */
int fsn_debug_cum_clip_scale(const float* x, int B, int Tp, int F, int64_t bs, int64_t ts, float eps, float* fs,
                             float* scale1T, fsn_stream_t stream);
int fsn_debug_cum_unit_scale(const float* magT, const float* fbT, int B, int F, int G, int Tp, int Ns, int Nf, float eps,
                             int time_major, float* scaleT, fsn_stream_t stream);
int fsn_debug_forget_unit_broadcast(const float* scaleT, int B, int F, int G, int Tp, float* unit_scale, fsn_stream_t stream);
int fsn_debug_fast_bn(const float* melT, const float* encT, int64_t bs, int64_t ts, int B, int Tp, int M, int Nn, int Ne,
                      int S, int cum, float eps, float* bn, float* fs, float* sums, float* scale, fsn_stream_t stream);
int fsn_debug_fast_dec_input(const float* encT, const float* bn_out, int64_t nbs, int64_t nms, int64_t nts, int B, int Tp,
                             int M, int S, int Ts, int64_t rbs, int64_t rts, float* dec_in, fsn_stream_t stream);
int fsn_debug_transpose_mag(const float* in, int B, int F, int T, int Tp, int64_t bs, int64_t ts, float* out,
                            const float* scale, float* scaled, fsn_stream_t stream);
int fsn_debug_crm_output(const float* y, int64_t bs, int64_t ts, int B, int Tp, int F, int la, float* out,
                         fsn_stream_t stream);
int fsn_debug_scale_rows(const float* in, const float* scale, int64_t n, int cols, int rows, int div, float* out,
                         fsn_stream_t stream);
int fsn_debug_imp_compress(const float* mag, int B, int F, int T, float fdrc, int tm, float* out, fsn_stream_t stream);
int fsn_debug_train_gather(const float* raw, const float* fbz, const float* inv2, const float* unit_scale, int B, int F, int G,
                           int Tp, int Ns, int Nf, float* X, fsn_stream_t stream);
int fsn_debug_sb_head(const float* h, int R, int H, int steps, const float* W, const float* bias, int O, int act, int N,
                      int c, int lo, int rows, int64_t rs, int64_t bs, int t0, float* out, fsn_stream_t stream);
int fsn_debug_sb_head_bwd(const float* dcrm, const float* y, int act, int R, int O, int steps, int la, int N, int c, int lo,
                          int rows, int64_t rs, int64_t bs, float* dY, fsn_stream_t stream);
int fsn_debug_train_dy(const float* dout, const float* y, int act, int B, int F, int T, int Tp, int la, float* dY,
                       fsn_stream_t stream);

/* unit-test hook of improved_fullsubnet's section recurrence on FSN_PREC_F16X3_TC (x3 = 1) / FSN_PREC_F16_TC (x3 = 0):
 * R independent rows of X [T, R, W] through the 2-layer LSTM of `sw` (w_ih[0] [4H, W]; fc_w / fc_b unread) -> h1 [T, R, H],
 * layer 1's hidden state of every step, by the path fsn_improved_forward runs (input projection on the tf32 GEMM, then
 * the persistent kernel).  packed receives the section image (fsn_debug_sb_lstm_tc_packed_bytes is not its size: use
 * fsn_improved_packed_bytes).  stages / cluster: weight ring depth (0, 2, 3, 4) and pairs per cluster (0, 1, 2, 4), 0 =
 * the production default.  H in {128, 256, 384}; every check precedes the first CUDA call. */
size_t fsn_debug_imp_section_lstm_tc_workspace_bytes(int R, int T, int W, int H, int x3);
int fsn_debug_imp_section_lstm_tc(const fsn_seq_weights* sw, int W, int H, int x3, const float* X, int R, int T, int stages,
                                  int cluster, void* packed, float* h1, void* workspace, size_t workspace_bytes,
                                  fsn_stream_t stream);

/* unit-test hooks for the statistics of the offline norms (fsn_lstm_simt.cu, fsn_train.cu; base_model.py:203-218 with
 * the closed-form second-norm mean of model.py:98-111).  float2 outputs are pairs of floats.
 *   fsn_debug_norm_stats: fs [B*T_pad] (float2) <- per frame (sum_f x, sum_f c_N[f] x) of x, element (b,t,f) at
 *     b*bs + t*ts + f, c_N the reflect multiplicity of row f in the N-neighbour unfold; sums [B] (float2) <- the clip's
 *     sums over its frames: all T_pad, or with lengths (nullable, host [B], copied to lens_dev) the first 1 +
 *     lengths[b]/hop + la (<= T_pad), in the order and tree of a call on that clip alone with T_pad = its frames.
 *     inv1 / inv2 (nullable, [B]) <- 1 / (sums.x / cnt1 + eps) and 1 / ((sums.y + fb_sums.y) / cnt2 + eps), fb_sums
 *     (nullable, float2 [B] of another call; NULL: sums), the counts per frame times the clip's frames with lengths.
 *   fsn_debug_train_stats: sums [B] (float2) <- (sum, sum c_N[f] x) of each clip of x [B,F,T] (tm = 0) or [T,B,F]
 *     (tm != 0), one CTA per clip.
 * Arguments are checked before any CUDA call. */
int fsn_debug_norm_stats(const float* x, int B, int T_pad, int F, int N, int64_t bs, int64_t ts, const int32_t* lengths,
                         int* lens_dev, int hop, int la, const float* fb_sums, float cnt1, float cnt2, float eps, float* fs,
                         float* sums, float* inv1, float* inv2, fsn_stream_t stream);
int fsn_debug_train_stats(const float* x, int tm, int B, int F, int T, int N, float* sums, fsn_stream_t stream);

/* unit-test hooks of forgetting_norm (FSN_NORM_FORGETTING; fsn_lstm_simt.cu, fsn_train.cu): the launchers the forwards and
 * fsn_train_backward run, on caller buffers.  Additions at version 102 (see fsn_version).
 *   fsn_debug_forgetting_scale: the forward scan.  x [B,T_pad,F] with element (b,t,f) at b*bs + t*ts + f (x2 the same
 *     layout, nullable).  fs (float2 [B*T_pad]) <- frame_stats of x with N neighbours, fs2 (needed with x2) <- those of x2
 *     with N2.  m_t = (sum_f x) / cnt without x2 (the first norm, cnt = F), else (sum_f c_N[f] x + sum_f c_N2[f] x2) / cnt
 *     (fullsubnet's second norm over the unfolded noisy and full-band rows, cnt = F K).  scale [T_pad,B] <- 1 / (mu_t +
 *     1e-10), mu (nullable, [T_pad,B]) <- mu_t.  lengths (nullable, host [B], copied to lens_dev): clip b is scanned over
 *     its own 1 + lengths[b]/hop + la (<= T_pad) frames only and its later entries are left unwritten; its frames get the
 *     bits of the unbounded scan, which is why fsn_enhance / fsn_fullband_enhance scan every clip over all T_max +
 *     look_ahead steps.
 *   fsn_debug_forgetting_bwd: the adjoint of the second norm and drop_band with respect to the full-band output (Nf = 0),
 *     tensors time-major as in the training step: sub-band input X and its gradient dX [Tp,R,K], K = 2Ns+2, R = B*Fsub rows
 *     of the drop_band map with G groups (G <= 1: none), full-band output fbz [Tp,B,F], scale [Tp,B] the forward's.  mid
 *     [Tp,B] <- d loss / d m_t / (F K) (the reverse recurrence g_t = -scale_t <dX,X>_t + a_{t+1} g_{t+1}, times b_t);
 *     dz [Tp,B,F] <- act'(fbz) (dX[t, row(b,f), K-1] scale[t,b] + mid[t,b]), the gradient at the full-band Linear's output.
 * Arguments are checked before any CUDA call. */
int fsn_debug_forgetting_scale(const float* x, int N, const float* x2, int N2, int B, int T_pad, int F, int64_t bs,
                               int64_t ts, float cnt, const int32_t* lengths, int* lens_dev, int hop, int la, float* fs,
                               float* fs2, float* scale, float* mu, fsn_stream_t stream);
int fsn_debug_forgetting_bwd(const float* dX, const float* X, const float* fbz, const float* scale, int B, int F, int G,
                             int Tp, int Ns, int act, float* mid, float* dz, fsn_stream_t stream);

/* unit-test hook of fsn_stoi (fsn_stoi.cu): the same kernels, with the intermediate buffers the caller's.  With Lr_max =
 * ceil(L_max * 10000 / sr) samples at 10 kHz and nf_max = its frames (len(range(0, Lr_max - 256, 128))):
 *   resampled [2,B,Lr_max] (float64; clean then estimate, zero past each clip's own resampled length);
 *   keep [B,nf_max] (1 = the frame survives silent-frame removal, for the clip's own frames), n_kept [B];
 *   compacted [2,B,Lr_max] (float64; the overlap-added kept frames, (n_kept + 1) * 128 samples, zero after);
 *   bands [2,B,15,nf_max] (float64; the band magnitudes of the clip's n_kept - 1 frames of the compacted signals);
 *   out [B] as fsn_stoi.  Workspace: fsn_stoi_workspace_bytes.  Arguments are checked as fsn_stoi checks them. */
int fsn_debug_stoi_stages(const float* clean, const float* estimate, const int32_t* lengths, int B, int L_max, int sr,
                          double* resampled, int32_t* keep, int32_t* n_kept, double* compacted, double* bands, float* out,
                          void* workspace, size_t workspace_bytes, fsn_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FSN_B200_H */
