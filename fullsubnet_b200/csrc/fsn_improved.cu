// improved_fullsubnet (recipes/dns_interspeech_2020/improved_fullsubnet/model.py:452-591, BASELINE config 5):
// host orchestration + the section unfold / output kernels, on top of the shared fp32 building blocks
// (STFT/iSTFT, persistent full-band LSTM, LSTM step kernel).
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

// |X|^fdrc with the Nyquist bin dropped: mag [B,F,T] -> out [B,T,F-1], or [T,B,F-1] when tm  (model.py:564-565)
__global__ void imp_compress_kernel(const float* __restrict__ mag, float* __restrict__ out, int F, int T, float fdrc, bool tm) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, Fu = F - 1;
  const int f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += 8) {
    const int f = f0 + i, t = t0 + tx;
    float v = 0.f;
    if (f < Fu && t < T) {
      const float m = mag[((size_t)b * F + f) * T + t];
      v = (fdrc == 0.5f) ? sqrtf(m) : powf(m, fdrc);
    }
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, f = f0 + tx;
    if (t < T && f < Fu) out[(tm ? (size_t)t * gridDim.z + b : (size_t)b * T + t) * Fu + f] = tile[tx][i];
  }
}

int imp_compress_launch(const float* mag, int B, int F, int T, float fdrc, bool tm, float* out, cudaStream_t st) {
  imp_compress_kernel<<<dim3(cdiv(T, 32), cdiv(F - 1, 32), B), dim3(32, 8), 0, st>>>(mag, out, F, T, fdrc, tm);
  FSN_CHECK_LAUNCH("imp_compress_kernel");
  return FSN_OK;
}

// section input (model.py:321-405, 425-442): unit n of clip b at frame t = noisy rows lo+n*cs-ns .. (+cs+2ns) and
// full-band rows lo+n*cf-nf .. (+cf+2nf), reflected (no edge repeat) at row 0 / row Fu-1.  One CTA per (b,t):
// writes X[t][b*N+n][w] and the per-(b,t) sum (for the section norm).  magc / fbT are [B,T,Fu], or [T,B,Fu] when tm.
__global__ void imp_section_input_kernel(const float* __restrict__ magc, const float* __restrict__ fbT, int B, int T,
                                         int Fu, SecGeom g, float* __restrict__ X, float2* __restrict__ fs, bool tm) {
  __shared__ float red[256];
  const int b = blockIdx.x / T, t = blockIdx.x % T;
  const int Wn = g.cs + 2 * g.ns;
  const size_t base = (tm ? (size_t)t * B + b : (size_t)b * T + t) * Fu;
  float local = 0.f;
  for (int i = threadIdx.x; i < g.N * g.W; i += blockDim.x) {
    const int n = i / g.W, w = i - n * g.W;
    int row;
    const float* src;
    if (w < Wn) { row = g.lo + n * g.cs - g.ns + w; src = magc; }
    else        { row = g.lo + n * g.cf - g.nf + (w - Wn); src = fbT; }
    row = reflect_idx(row, Fu);
    const float v = src[base + row];
    X[((size_t)t * B * g.N + (size_t)b * g.N + n) * g.W + w] = v;
    local += v;
  }
  red[threadIdx.x] = local;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) fs[(size_t)b * T + t] = make_float2(red[0], red[0]);
}

int imp_section_input_launch(const float* magc, const float* fbT, int B, int T, int Fu, const SecGeom& g, float* X, float2* fs,
                             bool tm, cudaStream_t st) {
  imp_section_input_kernel<<<B * T, 256, 0, st>>>(magc, fbT, B, T, Fu, g, X, fs, tm);
  FSN_CHECK_LAUNCH("imp_section_input_kernel");
  return FSN_OK;
}

struct ImpWs {
  float *mag, *real, *imag, *crm, *magc, *fbT, *X, *inv1, *invs;
  float2 *fs, *sums;
  SeqStackWs fb;
  float *h0[2], *h1[2], *c0, *c1;
  LayerSave tc;                        // FSN_PREC_TF32_TC: gates / cell / hidden of every step of one layer
  float *tc_h1, *tc_rec;
  ImpSecTcWs f16;                      // FSN_PREC_F16X3_TC / FSN_PREC_F16_TC: GEMM operands, P and h1 of one section
  WavWs wav;                           // fsn_improved_enhance: peak and length table (spectrum and cRM above)
  size_t bytes;
};

static bool imp_f16(const fsn_improved_desc* d) {
  return d->precision == FSN_PREC_F16X3_TC || d->precision == FSN_PREC_F16_TC;
}

// full band (model.py:567): 2 x LSTM(Fu -> Hf -> Hf) + Linear(Hf -> Fu), rows = clips; FSN_PREC_TF32_TC and
// FSN_PREC_F16_TC run it on the single-pass tensor-core layers, FSN_PREC_F16X3_TC on the compensated ones (as
// fullsubnet's full band)
static SeqStack imp_fb_stack(const fsn_improved_desc* d, const ImpDims& m) {
  SeqStack s;
  memset(&s, 0, sizeof(s));
  s.R = m.B; s.Tp = m.T; s.K0 = m.Fu; s.n = 2; s.H[0] = s.H[1] = d->fb_hidden; s.O = m.Fu; s.act = d->fb_activation;
  s.x3 = d->precision == FSN_PREC_F16X3_TC;
  s.tc = (d->precision == FSN_PREC_TF32_TC || imp_f16(d)) && lstm_rec_tc_supported(d->fb_hidden, s.x3);
  return s;
}

// the sub-band stack shape the f16 section kernel runs: sb_hidden in {128, 256, 384}
static bool imp_sb_f16_ok(int H) { return H % 128 == 0 && H >= 128 && H <= 384; }

void imp_section_tc_carve(Carver& c, size_t rows_T, int Wmax, int H, bool x3, ImpSecTcWs& w) {
  const size_t wa = (size_t)((Wmax + 3) & ~3) * (x3 ? 3 : 1);
  w.gemm.a = c.take<float>(rows_T * wa);
  w.gemm.w = c.take<float>((size_t)4 * H * wa);
  w.gemm.P = nullptr; w.gemm.rec = nullptr;
  w.P = c.take<float>(rows_T * 4 * H);
  w.h1 = c.take<float>(rows_T * H);
}

int imp_section_lstm_tc(const fsn_seq_weights& sw, const void* packed, const float* X, int R, int T, int W, int H, bool x3,
                        const ImpSecTcWs& w, cudaStream_t st, int stages, int cluster) {
  const size_t rows = (size_t)T * R;
  int rc;
  // P = (X W_ih0^T + b_ih0) + b_hh0, [T*R, 4H]: the compensated (x3) or single-pass tf32 GEMM
  if ((rc = linear_tc(X, (size_t)W, W, sw.w_ih[0], sw.b_ih[0], 4 * H, FSN_ACT_NONE, w.P, (size_t)4 * H, rows, x3, w.gemm,
                      st)))
    return rc;
  if ((rc = bias_act_launch(w.P, rows, 4 * H, (size_t)4 * H, sw.b_hh[0], FSN_ACT_NONE, st))) return rc;
  SbProjArgs a;
  memset(&a, 0, sizeof(a));
  a.packed = packed; a.P = w.P; a.h1 = w.h1; a.R = R; a.T = T; a.H = H; a.x3 = x3; a.stages = stages; a.cluster = cluster;
  return sb_proj_forward(a, st);
}

int sec_geom(int lo, int hi, int cs, int ns, int cf, int nf, int Fu, SecGeom& g) {
  g.lo = lo; g.cs = cs; g.ns = ns; g.cf = cf; g.nf = nf;
  FSN_REQUIRE(cs > 0 && cf > 0 && lo >= 0 && hi > lo && (hi - lo) % cs == 0 && (hi - lo) % cf == 0, FSN_ERR_SHAPE,
              "The number of center frequencies should be divisible by the subband freqency interval.");
  FSN_REQUIRE(cs == cf, FSN_ERR_UNSUPPORTED, "improved model: sb/fb centre widths of a section must match");
  FSN_REQUIRE(ns >= 0 && nf >= 0 && ns < Fu && nf < Fu, FSN_ERR_SHAPE, "improved model: neighbours >= num_freqs");
  g.N = (hi - lo) / cs;
  g.W = (cs + 2 * ns) + (cf + 2 * nf);
  return FSN_OK;
}

int imp_dims(const fsn_improved_desc* d, int B, int L, ImpDims& m) {
  FSN_REQUIRE(d && B > 0 && L > 0, FSN_ERR_SHAPE, "improved model: empty input");
  FSN_REQUIRE(dsp_size_ok(d->n_fft), FSN_ERR_UNSUPPORTED,
              "improved model: n_fft=%d unsupported (power of two <= 2048, or even and <= 1200)", d->n_fft);
  FSN_REQUIRE(d->num_freqs == d->n_fft / 2 + 1, FSN_ERR_SHAPE, "improved model: num_freqs != n_fft/2+1");
  FSN_REQUIRE(d->num_sections >= 1 && d->num_sections <= FSN_IMP_MAX_SECTIONS, FSN_ERR_SHAPE, "improved model: sections");
  FSN_REQUIRE(d->precision == FSN_PREC_FP32 || (d->precision == FSN_PREC_TF32_TC && (d->sb_hidden & 3) == 0) ||
                  (imp_f16(d) && imp_sb_f16_ok(d->sb_hidden)),
              FSN_ERR_UNSUPPORTED,
              "improved model: precision must be FSN_PREC_FP32, FSN_PREC_TF32_TC (sb_hidden %% 4 == 0), or FSN_PREC_F16X3_TC "
              "/ FSN_PREC_F16_TC (sb_hidden in {128, 256, 384})");
  m.B = B; m.L = L; m.T = 1 + L / d->hop_length; m.F = d->num_freqs; m.Fu = m.F - 1; m.S = d->num_sections;
  m.maxRW = 0; m.maxR = 0;
  for (int s = 0; s < m.S; ++s) {
    SecGeom& g = m.sec[s];
    const int rc = sec_geom(s == 0 ? 0 : d->freq_cutoffs[s - 1], s == m.S - 1 ? m.Fu : d->freq_cutoffs[s], d->sb_num_center[s],
                            d->sb_num_neighbor[s], d->fb_num_center[s], d->fb_num_neighbor[s], m.Fu, g);
    if (rc) return rc;
    if (g.N * g.W > m.maxRW) m.maxRW = g.N * g.W;
    if (g.N > m.maxR) m.maxR = g.N;
  }
  return FSN_OK;
}

// enhance: also the per-clip peak and length table of fsn_improved_enhance, after everything fsn_improved_forward uses
static void imp_carve(const fsn_improved_desc* d, const ImpDims& m, void* base, ImpWs& w, bool enhance = false) {
  Carver c(base);
  const size_t BFT = (size_t)m.B * m.F * m.T, BT = (size_t)m.B * m.T;
  w.mag = c.take<float>(BFT); w.real = c.take<float>(BFT); w.imag = c.take<float>(BFT);
  w.crm = c.take<float>(2 * BFT);
  w.magc = c.take<float>(BT * m.Fu);
  w.fbT = c.take<float>(BT * m.Fu);
  w.X = c.take<float>(BT * m.maxRW);
  w.inv1 = c.take<float>(m.B); w.invs = c.take<float>(m.B);
  w.fs = c.take<float2>(BT); w.sums = c.take<float2>(m.B);
  seq_stack_carve(c, imp_fb_stack(d, m), w.fb);
  const size_t RH = (size_t)m.B * m.maxR * d->sb_hidden;
  for (int i = 0; i < 2; ++i) { w.h0[i] = c.take<float>(RH); w.h1[i] = c.take<float>(RH); }
  w.c0 = c.take<float>(RH); w.c1 = c.take<float>(RH);
  w.tc.G = w.tc.C = w.tc.H = w.tc_h1 = w.tc_rec = nullptr;
  memset(&w.f16, 0, sizeof(w.f16));
  if (imp_f16(d)) {
    int maxW = 0;
    for (int s = 0; s < m.S; ++s) maxW = m.sec[s].W > maxW ? m.sec[s].W : maxW;
    imp_section_tc_carve(c, (size_t)m.T * m.B * m.maxR, maxW, d->sb_hidden, d->precision == FSN_PREC_F16X3_TC, w.f16);
  }
  if (d->precision == FSN_PREC_TF32_TC) {
    const size_t TR = (size_t)m.T * m.B * m.maxR;
    w.tc.G = c.take<float>(TR * 4 * d->sb_hidden);
    w.tc.C = c.take<float>(TR * d->sb_hidden);
    w.tc.H = c.take<float>(TR * d->sb_hidden);
    w.tc_h1 = c.take<float>(TR * d->sb_hidden);
    w.tc_rec = c.take<float>(4 * RH);
  }
  if (enhance) wav_carve(c, m.B, 0, m.T, w.wav);
  w.bytes = c.off;
}

// The forward on a carved workspace, wav [B,L] -> enhanced [B,L] (+ crm [B,2,F,T]).  lens (nullable, device [B]): clip b
// is the first lens[b] samples of its row.  Only the length-dependent kernels read it - the STFT, the full-band and
// section norms and the iSTFT (with peak, when given) - so every clip gives the bits of a call on that clip alone; the
// recurrent stacks and the section Linear are causal and run over all T steps.
static int imp_forward(const fsn_improved_desc* d, const fsn_improved_weights* wt, const ImpDims& m, const ImpWs& w,
                       const float* wav, float* enhanced, float* crm_out, unsigned int* peak, const int* lens,
                       cudaStream_t st) {
  const int B = m.B, L = m.L, T = m.T, F = m.F, Fu = m.Fu, Hs = d->sb_hidden, hop = d->hop_length;
  int rc;
  const float eps = 1.1920928955078125e-07f;  // np.finfo(np.float32).eps (model.py:23,148)
  float* crm = crm_out ? crm_out : w.crm;
  // STFT (model.py:550-557), |X|^fdrc without the Nyquist bin (564-565)
  if ((rc = stft_launch(wav, B, L, d->n_fft, hop, d->win_length, w.mag, nullptr, w.real, w.imag, nullptr, 0, st, lens)))
    return rc;
  if ((rc = imp_compress_launch(w.mag, B, F, T, d->fdrc, false, w.magc, st))) return rc;
  // full band: norm (566) -> 2xLSTM + Linear (567); with lens the counts are per frame, times the clip's own frames
  if ((rc = clip_stats_launch(w.magc, B, T, Fu, 0, w.fs, w.sums, st, lens, hop, 0))) return rc;
  if ((rc = norm_scales_launch(w.sums, w.sums, B, lens ? (float)Fu : (float)Fu * T, 1.f, w.inv1, nullptr, st, eps, lens,
                               hop, 0)))
    return rc;
  SeqStack s = imp_fb_stack(d, m);
  s.L[0] = seq_layer(wt->fb, 0); s.L[1] = seq_layer(wt->fb, 1);
  s.x = w.magc; s.scale = w.inv1; s.fc_w = wt->fb.fc_w; s.fc_b = wt->fb.fc_b; s.out = w.fbT;
  if ((rc = seq_stack_forward(s, w.fb, st))) return rc;
  // cRM, Nyquist row = 0 (572)
  if ((rc = check_cuda(cudaMemsetAsync(crm, 0, (size_t)2 * B * F * T * sizeof(float), st), "crm memset"))) return rc;
  // sub-band sections (408-447)
  for (int s = 0; s < m.S; ++s) {
    const SecGeom& g = m.sec[s];
    const int R = B * g.N;
    if ((rc = imp_section_input_launch(w.magc, w.fbT, B, T, Fu, g, w.X, w.fs, false, st))) return rc;
    if ((rc = clip_reduce_only_launch(w.fs, B, T, w.sums, st, lens, hop, 0))) return rc;
    if ((rc = norm_scales_launch(w.sums, w.sums, B, lens ? (float)g.N * g.W : (float)g.N * g.W * T, 1.f, w.invs, nullptr,
                                 st, eps, lens, hop, 0)))
      return rc;
    const fsn_seq_weights& sw = wt->sb[s];
    if (imp_f16(d)) {
      // the section on the fp16 tensor cores: P of all steps on the tf32 GEMM, both layers of all steps in one
      // persistent launch, then the head over all steps (DESIGN 4.3)
      FSN_REQUIRE(wt->sb_packed[s], FSN_ERR_SHAPE, "improved model: section %d has no packed weights (fsn_improved_pack_sb_weights)", s);
      if ((rc = scale_rows_launch(w.X, w.invs, (size_t)T * R * g.W, g.W, R, g.N, w.X, st))) return rc;
      if ((rc = imp_section_lstm_tc(sw, wt->sb_packed[s], w.X, R, T, g.W, Hs, d->precision == FSN_PREC_F16X3_TC, w.f16, st)))
        return rc;
      if ((rc = sb_head_launch(w.f16.h1, R, Hs, T, sw.fc_w, sw.fc_b, 2 * g.cs, d->sb_activation, crm, imp_head_geom(g, F, T), 0,
                               st)))
        return rc;
      continue;
    }
    if (d->precision == FSN_PREC_TF32_TC) {
      // layer by layer over all steps: hoisted input projection + per-step recurrent GEMM on wgmma (tf32), fused cell
      LayerSave l1{w.tc.G, w.tc.C, w.tc_h1};
      // scale X by the section norm in place (the tensor-core GEMM reads plain fp32 rows)
      if ((rc = scale_rows_launch(w.X, w.invs, (size_t)T * R * g.W, g.W, R, g.N, w.X, st))) return rc;
      if ((rc = layer_forward_save_tc(seq_layer(sw, 0), w.X, R, g.W, Hs, T, w.tc, w.tc_rec, st))) return rc;
      if ((rc = layer_forward_save_tc(seq_layer(sw, 1), w.tc.H, R, Hs, Hs, T, l1, w.tc_rec, st))) return rc;
      for (int t = 0; t < T; ++t)
        if ((rc = sb_head_launch(w.tc_h1 + (size_t)t * R * Hs, R, Hs, 1, sw.fc_w, sw.fc_b, 2 * g.cs, d->sb_activation, crm,
                                 imp_head_geom(g, F, T), t, st)))
          return rc;
      continue;
    }
    const Step2State s2{{w.h0[0], w.h0[1]}, w.c0, {w.h1[0], w.h1[1]}, w.c1, Hs, 0};
    for (int t = 0; t < T; ++t) {
      StepParams p;
      memset(&p, 0, sizeof(p));
      p.R = R; p.K0 = g.W; p.H = Hs;
      p.w_ih = sw.w_ih[0]; p.w_hh = sw.w_hh[0]; p.b_ih = sw.b_ih[0]; p.b_hh = sw.b_hh[0];
      p.x0 = w.X + (size_t)t * R * g.W; p.x0_row_stride = g.W; p.row_scale = w.invs; p.row_scale_div = g.N;
      if ((rc = lstm_step2_launch(p, SEG0_DENSE, t, seq_layer(sw, 1), s2, st))) return rc;
      if ((rc = sb_head_launch(s2.h1_at(t), R, Hs, 1, sw.fc_w, sw.fc_b, 2 * g.cs, d->sb_activation, crm, imp_head_geom(g, F, T),
                               t, st)))
        return rc;
    }
  }
  // element-wise mask on (re, im) + iSTFT (575-589)
  return istft_launch(w.real, w.imag, 1, crm, B, T, d->n_fft, hop, d->win_length, L, enhanced, st, 2, peak, lens);
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_improved_workspace_bytes(const fsn_improved_desc* d, int B, int L) {
  ImpDims m;
  if (imp_dims(d, B, L, m)) return 0;
  ImpWs w;
  imp_carve(d, m, nullptr, w);
  return w.bytes;
}

extern "C" int fsn_improved_forward(const fsn_improved_desc* d, const fsn_improved_weights* wt, const float* wav, int B,
                                    int L, float* enhanced, float* crm_out, void* workspace, size_t workspace_bytes,
                                    fsn_stream_t stream) {
  launch_counter() = 0;
  ImpDims m;
  int rc = imp_dims(d, B, L, m);
  if (rc) return rc;
  ImpWs w;
  imp_carve(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  return imp_forward(d, wt, m, w, wav, enhanced, crm_out, nullptr, nullptr, (cudaStream_t)stream);
}

// ---- clips of different lengths in one call (lengths non-null: host [B]), buffers laid out for the longest clip
// (L_max samples, T_max frames); optional int16 output with the per-clip peak of the iSTFT epilogue
extern "C" size_t fsn_improved_enhance_workspace_bytes(const fsn_improved_desc* d, int B, int L_max) {
  ImpDims m;
  if (imp_dims(d, B, L_max, m)) return 0;
  ImpWs w;
  imp_carve(d, m, nullptr, w, true);
  return w.bytes;
}

extern "C" int fsn_improved_enhance(const fsn_improved_desc* d, const fsn_improved_weights* wt, const float* wav,
                                    const int32_t* lengths, int B, int L_max, float* enhanced, float* crm_out,
                                    int16_t* pcm, float gain, void* workspace, size_t workspace_bytes,
                                    fsn_stream_t stream) {
  launch_counter() = 0;
  ImpDims m;
  int rc = imp_dims(d, B, L_max, m);
  if (rc) return rc;
  if ((rc = wav_check(lengths, B, L_max, d->n_fft, false, enhanced, "improved_enhance"))) return rc;
  ImpWs w;
  imp_carve(d, m, workspace, w, true);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = wav_prologue(lengths, B, w.wav, st))) return rc;
  if ((rc = imp_forward(d, wt, m, w, wav, enhanced, crm_out, pcm ? w.wav.peak : nullptr, w.wav.lens, st))) return rc;
  return wav_epilogue(w.wav, enhanced, B, L_max, pcm, gain, crm_out, m.F, m.T, d->hop_length, st);
}

// ---- unit-test hook of the section input (include/fsn_b200.h): the launcher both improved forwards run, every argument
// checked before any CUDA call
extern "C" int fsn_debug_imp_section_input(const float* magc, const float* fbT, int B, int T, int Fu, int lo, int hi, int cs,
                                           int ns, int cf, int nf, int tm, float* X, float* fs, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(magc && fbT && X && fs, FSN_ERR_SHAPE, "section input hook: null argument");
  FSN_REQUIRE(B > 0 && T > 0 && Fu >= 2 && hi <= Fu, FSN_ERR_SHAPE, "section input hook: bad shape B=%d T=%d Fu=%d", B, T,
              Fu);
  SecGeom g;
  const int rc = sec_geom(lo, hi, cs, ns, cf, nf, Fu, g);
  if (rc) return rc;
  FSN_REQUIRE((size_t)T * B * g.N * g.W < ((size_t)1 << 31) && (size_t)B * T < ((size_t)1 << 31), FSN_ERR_SHAPE,
              "section input hook: tensors must stay below 2^31 elements");
  return imp_section_input_launch(magc, fbT, B, T, Fu, g, X, reinterpret_cast<float2*>(fs), tm != 0, (cudaStream_t)stream);
}

// ---- packed section weights of the fp16 tensor-core precisions (include/fsn_b200.h)
static int imp_pack_check(const fsn_improved_desc* d, int section) {
  ImpDims m;
  int rc = imp_dims(d, 1, 1, m);
  if (rc) return rc;
  FSN_REQUIRE(imp_f16(d), FSN_ERR_UNSUPPORTED,
              "improved model: packed section weights exist for FSN_PREC_F16X3_TC / FSN_PREC_F16_TC only");
  FSN_REQUIRE(section >= 0 && section < m.S, FSN_ERR_SHAPE, "improved model: section %d of %d", section, m.S);
  return FSN_OK;
}

extern "C" size_t fsn_improved_packed_bytes(const fsn_improved_desc* d, int section) {
  if (imp_pack_check(d, section)) return 0;
  return sb_tc_packed_bytes_raw(d->sb_hidden, d->precision == FSN_PREC_F16X3_TC, true);
}

extern "C" int fsn_improved_pack_sb_weights(const fsn_improved_desc* d, const fsn_improved_weights* w, int section,
                                            void* packed, fsn_stream_t stream) {
  launch_counter() = 0;
  int rc = imp_pack_check(d, section);
  if (rc) return rc;
  FSN_REQUIRE(w && packed, FSN_ERR_SHAPE, "improved model: missing weights or packed buffer");
  const fsn_seq_weights& sw = w->sb[section];
  FSN_REQUIRE(sw.w_hh[0] && sw.w_ih[1] && sw.w_hh[1] && sw.b_ih[1] && sw.b_hh[1], FSN_ERR_SHAPE,
              "improved model: section %d has missing weights", section);
  return sb_tc_pack_raw(&sw, d->sb_hidden, 0, 0, packed, (cudaStream_t)stream, d->precision == FSN_PREC_F16X3_TC, true);
}

// ---- unit-test hook of the section recurrence alone: X [T, R, W] -> h1 [T, R, H] (layer 1's hidden state of every
// step) through the GEMM and the persistent kernel the f16 precisions run; packed receives the section image
static int imp_sec_hook_check(int R, int T, int W, int H) {
  FSN_REQUIRE(R > 0 && T > 0 && W > 0 && W <= 4096 && (size_t)T * R * 4 * H < ((size_t)1 << 31), FSN_ERR_SHAPE,
              "section recurrence hook: bad shape R=%d T=%d W=%d H=%d", R, T, W, H);
  FSN_REQUIRE(imp_sb_f16_ok(H), FSN_ERR_UNSUPPORTED, "section recurrence hook: hidden size %d (128, 256 or 384)", H);
  return FSN_OK;
}

extern "C" size_t fsn_debug_imp_section_lstm_tc_workspace_bytes(int R, int T, int W, int H, int x3) {
  if (imp_sec_hook_check(R, T, W, H)) return 0;
  Carver c(nullptr);
  ImpSecTcWs w;
  imp_section_tc_carve(c, (size_t)T * R, W, H, x3 != 0, w);
  return c.off;
}

extern "C" int fsn_debug_imp_section_lstm_tc(const fsn_seq_weights* sw, int W, int H, int x3, const float* X, int R, int T,
                                             int stages, int cluster, void* packed, float* h1, void* workspace,
                                             size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(sw && X && packed && h1, FSN_ERR_SHAPE, "section recurrence hook: null argument");
  int rc = imp_sec_hook_check(R, T, W, H);
  if (rc) return rc;
  FSN_REQUIRE(cluster == 0 || cluster == 1 || cluster == 2 || cluster == 4, FSN_ERR_UNSUPPORTED,
              "section recurrence hook: cluster size %d (0, 1, 2 or 4)", cluster);
  FSN_REQUIRE(stages == 0 || (stages >= 2 && stages <= 4), FSN_ERR_UNSUPPORTED,
              "section recurrence hook: ring depth %d (0, 2, 3 or 4)", stages);
  Carver c(workspace);
  ImpSecTcWs w;
  imp_section_tc_carve(c, (size_t)T * R, W, H, x3 != 0, w);
  FSN_REQUIRE(workspace && workspace_bytes >= c.off, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              c.off);
  w.h1 = h1;
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = sb_tc_pack_raw(sw, H, 0, 0, packed, st, x3 != 0, true))) return rc;
  return imp_section_lstm_tc(*sw, packed, X, R, T, W, H, x3 != 0, w, st, stages, cluster);
}
