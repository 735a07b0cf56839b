// Training step of improved_fullsubnet (recipes/dns_interspeech_2020/improved_fullsubnet/model.py:452-591, wav in, wav out):
//   fsn_improved_train_forward   Model.forward with gradients enabled, keeping what the backward needs
//   fsn_improved_train_backward  adjoint of the element-wise mask + iSTFT -> per section (in index order): Linear(H -> 2c),
//                                BPTT of its 2-layer stack down to its normalised input, weight gradients, then the
//                                section norm + unfold backward into the full-band output -> act', Linear(Hf -> Fu), BPTT
//                                and weight gradients of the full band
// Everything is time-major ([T, rows, .]) like fsn_train.cu and runs on the pieces the other training steps share
// (layer_forward, stack_bwd, layer_weight_grads, linear_bwd).  The noisy columns of the section inputs and the first norm
// have no parameter behind them, so they get no backward.  Every reduction runs in a fixed order: two runs give identical
// bits.  oracle/improved_fullsubnet_oracle.py:improved_forward under CPU autograd is the reference.
#include "fsn_internal.cuh"

namespace fsn {

static const float IMP_EPS = 1.1920928955078125e-07f;  // np.finfo(np.float32).eps (model.py:23,148)

struct ImpSecSave {
  float *Xn, *invs;  // normalised section input [T, B*N, W] and the section norm's scale per clip
  LayerSave L[2];
};

struct ImpTrainWs {
  float *mag, *real, *imag, *raw, *xfb, *inv1, *yfb, *crm;
  float2 *sums, *fs;
  LayerSave fb[2];
  ImpSecSave sec[FSN_IMP_MAX_SECTIONS];
  float *dcrm, *dY, *dH, *dX, *dfb, *dot;
  float *dh_rec[2], *dc[2], *dh_mid;
  float *splitk, *colsum;
  size_t colsum_floats;
  // tf32 layers: transposed weights of the stack being differentiated (a section's, then the full band's), K-major
  // copies for the weight gradients, the recurrent product of the unfused step, fp16 operands of the forward step kernel
  float *whhT[2], *wihT[2], *gT, *xT, *rec;
  __half *h16[2], *w16;
  size_t bytes;
};

static size_t zmax(size_t a, size_t b) { return a > b ? a : b; }

static void carve_imp_train(const fsn_improved_desc* d, const ImpDims& m, void* base, ImpTrainWs& w) {
  Carver c(base);
  const size_t B = m.B, T = m.T, Fu = m.Fu, Hf = d->fb_hidden, Hs = d->sb_hidden;
  const size_t BFT = B * m.F * T, TB = T * B, Rmax = B * m.maxR;
  size_t maxW = 0, maxO = Fu;  // widest section input, widest output row of a section's Linear or the full band's
  for (int s = 0; s < m.S; ++s) {
    maxW = zmax(maxW, (size_t)m.sec[s].W);
    maxO = zmax(maxO, (size_t)m.sec[s].N * 2 * m.sec[s].cs);
  }
  w.mag = c.take<float>(BFT); w.real = c.take<float>(BFT); w.imag = c.take<float>(BFT);
  w.raw = c.take<float>(TB * Fu); w.xfb = c.take<float>(TB * Fu); w.yfb = c.take<float>(TB * Fu);
  w.inv1 = c.take<float>(B);
  w.sums = c.take<float2>(B); w.fs = c.take<float2>(TB);
  w.crm = c.take<float>(2 * BFT);
  for (int l = 0; l < 2; ++l) {
    w.fb[l].G = c.take<float>(TB * 4 * Hf); w.fb[l].C = c.take<float>(TB * Hf); w.fb[l].H = c.take<float>(TB * Hf);
  }
  for (int s = 0; s < m.S; ++s) {
    const SecGeom& g = m.sec[s];
    const size_t rows = TB * g.N;
    ImpSecSave& q = w.sec[s];
    q.Xn = c.take<float>(rows * g.W);
    q.invs = c.take<float>(B);
    for (int l = 0; l < 2; ++l) {
      q.L[l].G = c.take<float>(rows * 4 * Hs); q.L[l].C = c.take<float>(rows * Hs); q.L[l].H = c.take<float>(rows * Hs);
    }
  }
  // backward
  w.dcrm = c.take<float>(2 * BFT);
  w.dY = c.take<float>(TB * maxO);
  w.dH = c.take<float>(T * zmax(B * Hf, Rmax * Hs));
  w.dX = c.take<float>(TB * m.maxRW);
  w.dfb = c.take<float>(TB * Fu);
  w.dot = c.take<float>(B);
  const size_t RH = zmax(B * Hf, Rmax * Hs);
  for (int l = 0; l < 2; ++l) { w.dh_rec[l] = c.take<float>(RH); w.dc[l] = c.take<float>(RH); }
  w.dh_mid = c.take<float>(RH);
  w.splitk = c.take<float>(SPLITK_SCRATCH_FLOATS);
  w.colsum_floats = (size_t)COLSUM_MAX_S * zmax(4 * zmax(Hf, Hs), maxO);
  w.colsum = c.take<float>(w.colsum_floats);
  for (int l = 0; l < 2; ++l) { w.whhT[l] = w.wihT[l] = nullptr; w.h16[l] = nullptr; }
  w.gT = w.xT = w.rec = nullptr;
  w.w16 = nullptr;
  const bool tf = tf32_layer(d->precision, (int)Hf), ts = tf32_layer(d->precision, (int)Hs);
  if (tf || ts) {
    const size_t Hm = zmax(tf ? Hf : 0, ts ? Hs : 0);
    const size_t rows = T * zmax(tf ? B : 0, ts ? Rmax : 0);
    const size_t K0max = zmax(zmax(Fu, maxW), Hm);
    for (int l = 0; l < 2; ++l) w.whhT[l] = c.take<float>(Hm * 4 * Hm);
    w.wihT[0] = ts ? c.take<float>(maxW * 4 * Hs) : nullptr;  // only the sections' layer 0 computes a dx
    w.wihT[1] = c.take<float>(Hm * 4 * Hm);
    w.gT = c.take<float>(tgemm_blocked_floats(rows, 4 * (int)Hm));
    w.xT = c.take<float>(tgemm_blocked_floats(rows, (int)K0max));
    w.rec = c.take<float>(4 * RH);
    for (int l = 0; l < 2; ++l) w.h16[l] = c.take<__half>(rows * Hm);
    w.w16 = c.take<__half>(4 * Hm * (Hm + K0max));
  }
  w.bytes = c.off;
}

static int imp_train_check(const fsn_improved_desc* d, int B, int L, ImpDims& m) {
  FSN_REQUIRE(d && d->hop_length > 0 && d->win_length > 0 && d->win_length <= d->n_fft && d->fb_hidden > 0 &&
                  d->sb_hidden > 0,
              FSN_ERR_SHAPE, "improved training: bad descriptor");
  // the fp16 precisions are built for inference only (imp_dims accepts them for fsn_improved_forward / _enhance)
  FSN_REQUIRE(d->precision == FSN_PREC_FP32 || d->precision == FSN_PREC_TF32_TC, FSN_ERR_UNSUPPORTED,
              "improved training: precision must be FSN_PREC_FP32 or FSN_PREC_TF32_TC");
  int rc = imp_dims(d, B, L, m);
  if (rc) return rc;
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "improved training: the GRU cell is not built");
  FSN_REQUIRE((d->fb_activation == FSN_ACT_NONE || d->fb_activation == FSN_ACT_RELU) &&
                  (d->sb_activation == FSN_ACT_NONE || d->sb_activation == FSN_ACT_RELU),
              FSN_ERR_UNSUPPORTED, "improved training: output activations none or ReLU are built");
  return FSN_OK;
}

__device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// Backward of one section's norm and full-band unfold, gather form: for every full-band output element (t, b, r),
//   v = sum over units u and offsets k of the full-band columns with reflect_idx(lo + u*cf - nf + k) == r of
//       inv_s[b] * dXn[t, b*N+u, Wn+k] - inv_s[b] * dot[b] / cnt,   dot[b] = sum dXn * Xn over the clip's section input
// (the mean of the norm covers the noisy columns as well).  dfb [T,B,Fu] = v (first section) or dfb + v (the others, in
// index order); the last section also applies act' of the kept full-band output y.
__global__ void imp_unfold_bwd_kernel(const float* __restrict__ dX, const float* __restrict__ invs, const float* __restrict__ dot,
                                      float cnt, SecGeom g, int B, int T, int Fu, bool first, int act,
                                      const float* __restrict__ y, float* __restrict__ dfb) {
  const int Wn = g.cs + 2 * g.ns, Wf = g.cf + 2 * g.nf;
  const size_t n = (size_t)T * B * Fu;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i % Fu);
    const size_t tb = i / Fu;
    const int b = (int)(tb % B), t = (int)(tb / B);
    const float s = invs[b], q = s * dot[b] / cnt;
    const float* row0 = dX + ((size_t)t * B + b) * g.N * g.W + Wn;
    float v = 0.f;
    // unfolded rows p that reflect onto r (nf < Fu: at most one reflection): r, -r, 2(Fu-1) - r
    for (int cand = 0; cand < 3; ++cand) {
      int p = r;
      if (cand == 1) { if (r == 0) continue; p = -r; }
      if (cand == 2) { if (r == Fu - 1) continue; p = 2 * (Fu - 1) - r; }
      const int e = p - g.lo + g.nf;  // = u*cf + k
      const int u0 = max(0, -floor_div(Wf - 1 - e, g.cf)), u1 = min(g.N - 1, floor_div(e, g.cf));
      for (int u = u0; u <= u1; ++u) v += s * row0[(size_t)u * g.W + (e - u * g.cf)] - q;
    }
    if (!first) v = dfb[i] + v;
    if (act == FSN_ACT_RELU && !(y[i] > 0.f)) v = 0.f;
    dfb[i] = v;
  }
}

int imp_unfold_bwd_launch(const float* dX, const float* invs, const float* dot, float cnt, const SecGeom& g, int B, int T,
                          int Fu, bool first, int act, const float* y, float* dfb, cudaStream_t st) {
  imp_unfold_bwd_kernel<<<ew_grid((size_t)T * B * Fu), 256, 0, st>>>(dX, invs, dot, cnt, g, B, T, Fu, first, act, y, dfb);
  FSN_CHECK_LAUNCH("imp_unfold_bwd_kernel");
  return FSN_OK;
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_improved_train_workspace_bytes(const fsn_improved_desc* d, int B, int L) {
  ImpDims m;
  if (imp_train_check(d, B, L, m)) return 0;
  ImpTrainWs w;
  carve_imp_train(d, m, nullptr, w);
  return w.bytes;
}

extern "C" int fsn_improved_train_forward(const fsn_improved_desc* d, const fsn_improved_weights* wt, const float* wav, int B,
                                          int L, float* enhanced, void* workspace, size_t workspace_bytes,
                                          fsn_stream_t stream) {
  launch_counter() = 0;
  ImpDims m;
  int rc = imp_train_check(d, B, L, m);
  if (rc) return rc;
  FSN_REQUIRE(wt && wav && enhanced, FSN_ERR_SHAPE, "improved training: null argument");
  ImpTrainWs w;
  carve_imp_train(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int T = m.T, F = m.F, Fu = m.Fu, Hf = d->fb_hidden, Hs = d->sb_hidden, prec = d->precision;
  // STFT (model.py:550-557), |X|^fdrc without the Nyquist bin (564-565), time-major
  if ((rc = stft_launch(wav, B, L, d->n_fft, d->hop_length, d->win_length, w.mag, nullptr, w.real, w.imag, nullptr, 0, st)))
    return rc;
  if ((rc = imp_compress_launch(w.mag, B, F, T, d->fdrc, true, w.raw, st))) return rc;
  // full band: norm (566) -> 2xLSTM + Linear + act (567), y kept for act'
  if ((rc = train_tm_stats_launch(w.raw, B, Fu, T, 0, w.sums, st))) return rc;
  if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)Fu * T, 1.f, w.inv1, nullptr, st, IMP_EPS))) return rc;
  const size_t nfb = (size_t)T * B * Fu;
  if ((rc = scale_rows_launch(w.raw, w.inv1, nfb, Fu, B, 1, w.xfb, st))) return rc;
  // fp16 operand copies of the tf32 step kernel: layer 0's hidden states double as layer 1's input
  const LayerHalf h0{w.h16[0], nullptr, w.w16}, h1{w.h16[1], w.h16[0], w.w16};
  if ((rc = layer_forward(prec, seq_layer(wt->fb, 0), w.xfb, B, Fu, Hf, T, w.fb[0], w.rec, w.splitk, &h0, st))) return rc;
  if ((rc = layer_forward(prec, seq_layer(wt->fb, 1), w.fb[0].H, B, Hf, Hf, T, w.fb[1], w.rec, w.splitk, &h1, st))) return rc;
  if ((rc = fc_gemm_launch(w.fb[1].H, wt->fb.fc_w, wt->fb.fc_b, w.yfb, T * B, Hf, Fu, d->fb_activation, st))) return rc;
  // cRM, Nyquist row = 0 (572)
  if ((rc = check_cuda(cudaMemsetAsync(w.crm, 0, (size_t)2 * B * F * T * sizeof(float), st), "crm memset"))) return rc;
  // sub-band sections (408-447): unfold + concat, per-section norm, 2xLSTM, Linear(H -> 2c) of every frame into the cRM
  for (int s = 0; s < m.S; ++s) {
    const SecGeom& g = m.sec[s];
    const ImpSecSave& q = w.sec[s];
    const int R = B * g.N;
    const fsn_seq_weights& sw = wt->sb[s];
    if ((rc = imp_section_input_launch(w.raw, w.yfb, B, T, Fu, g, q.Xn, w.fs, true, st))) return rc;
    if ((rc = clip_reduce_only_launch(w.fs, B, T, w.sums, st))) return rc;
    if ((rc = norm_scales_launch(w.sums, w.sums, B, (float)g.N * g.W * T, 1.f, q.invs, nullptr, st, IMP_EPS))) return rc;
    const size_t nx = (size_t)T * R * g.W;
    if ((rc = scale_rows_launch(q.Xn, q.invs, nx, g.W, R, g.N, q.Xn, st))) return rc;
    if ((rc = layer_forward(prec, seq_layer(sw, 0), q.Xn, R, g.W, Hs, T, q.L[0], w.rec, w.splitk, &h0, st))) return rc;
    if ((rc = layer_forward(prec, seq_layer(sw, 1), q.L[0].H, R, Hs, Hs, T, q.L[1], w.rec, w.splitk, &h1, st))) return rc;
    if ((rc = sb_head_launch(q.L[1].H, R, Hs, T, sw.fc_w, sw.fc_b, 2 * g.cs, d->sb_activation, w.crm, imp_head_geom(g, F, T), 0,
                             st)))
      return rc;
  }
  // element-wise mask on (re, im) + iSTFT (575-589)
  return istft_launch(w.real, w.imag, 1, w.crm, B, T, d->n_fft, d->hop_length, d->win_length, L, enhanced, st, 2);
}

extern "C" int fsn_improved_train_backward(const fsn_improved_desc* d, const fsn_improved_weights* wt, const float* d_enhanced,
                                           int B, int L, const fsn_improved_grads* g, void* workspace,
                                           size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  ImpDims m;
  int rc = imp_train_check(d, B, L, m);
  if (rc) return rc;
  FSN_REQUIRE(wt && d_enhanced && g, FSN_ERR_SHAPE, "improved training: null argument");
  ImpTrainWs w;
  carve_imp_train(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int T = m.T, F = m.F, Fu = m.Fu, Hf = d->fb_hidden, Hs = d->sb_hidden;
  const bool tf = tf32_layer(d->precision, Hf), ts = tf32_layer(d->precision, Hs);
  const WgradScratch wg{w.gT, w.xT, w.splitk, w.colsum, w.colsum_floats};
  // ---- mask + iSTFT adjoint: d loss / d cRM
  if ((rc = istft_mask_adjoint_launch(d_enhanced, w.real, w.imag, B, L, T, d->n_fft, d->hop_length, d->win_length, w.dcrm, st)))
    return rc;
  // ---- sections, in index order (their contributions to the full-band output's gradient are summed in that order)
  for (int s = 0; s < m.S; ++s) {
    const SecGeom& sg = m.sec[s];
    const ImpSecSave& q = w.sec[s];
    const fsn_seq_weights& sw = wt->sb[s];
    const fsn_seq_grads& sgr = g->sb[s];
    const int R = B * sg.N, O = 2 * sg.cs;
    LayerBwd Ls[2] = {
        LayerBwd{sw.w_ih[0], sw.w_hh[0], q.L[0], R, sg.W, Hs, w.dh_rec[0], w.dc[0], ts ? w.whhT[0] : nullptr,
                 ts ? w.wihT[0] : nullptr, w.splitk},
        LayerBwd{sw.w_ih[1], sw.w_hh[1], q.L[1], R, Hs, Hs, w.dh_rec[1], w.dc[1], ts ? w.whhT[1] : nullptr,
                 ts ? w.wihT[1] : nullptr, w.splitk}};
    for (int l = 0; l < 2; ++l)
      if ((rc = layer_bwd_transpose_weights(Ls[l], st))) return rc;
    if ((rc = sb_head_bwd_launch(w.dcrm, w.crm, d->sb_activation, R, O, T, 0, imp_head_geom(sg, F, T), w.dY, st))) return rc;
    if ((rc = linear_bwd(w.dY, q.L[1].H, sw.fc_w, T * R, O, Hs, sgr.fc_w, sgr.fc_b, w.dH, w.splitk, w.colsum, w.colsum_floats, st)))
      return rc;
    // BPTT down to the normalised section input
    if ((rc = stack_bwd(Ls, 2, T, w.dH, nullptr, nullptr, 0, w.dh_mid, nullptr, w.dX, st))) return rc;
    if ((rc = train_dot_launch(w.dX, q.Xn, T, R, sg.N, sg.W, B, w.dot, st))) return rc;
    if ((rc = imp_unfold_bwd_launch(w.dX, q.invs, w.dot, (float)sg.N * sg.W * T, sg, B, T, Fu, s == 0,
                                    s == m.S - 1 ? d->fb_activation : FSN_ACT_NONE, w.yfb, w.dfb, st)))
      return rc;
    if ((rc = layer_weight_grads(Ls[1], T, q.L[0].H, sgr.w_ih[1], sgr.w_hh[1], sgr.b_ih[1], sgr.b_hh[1], wg, st))) return rc;
    if ((rc = layer_weight_grads(Ls[0], T, q.Xn, sgr.w_ih[0], sgr.w_hh[0], sgr.b_ih[0], sgr.b_hh[0], wg, st))) return rc;
  }
  // ---- full band: Linear(Hf -> Fu), BPTT (its input is the normalised spectrogram: no dx), weight gradients
  const fsn_seq_weights& fw = wt->fb;
  const fsn_seq_grads& fg = g->fb;
  LayerBwd Lf[2] = {
      LayerBwd{fw.w_ih[0], fw.w_hh[0], w.fb[0], B, Fu, Hf, w.dh_rec[0], w.dc[0], tf ? w.whhT[0] : nullptr, nullptr, w.splitk},
      LayerBwd{fw.w_ih[1], fw.w_hh[1], w.fb[1], B, Hf, Hf, w.dh_rec[1], w.dc[1], tf ? w.whhT[1] : nullptr,
               tf ? w.wihT[1] : nullptr, w.splitk}};
  for (int l = 0; l < 2; ++l)
    if ((rc = layer_bwd_transpose_weights(Lf[l], st))) return rc;
  if ((rc = linear_bwd(w.dfb, w.fb[1].H, fw.fc_w, T * B, Fu, Hf, fg.fc_w, fg.fc_b, w.dH, w.splitk, w.colsum, w.colsum_floats, st)))
    return rc;
  if ((rc = stack_bwd(Lf, 2, T, w.dH, nullptr, nullptr, 0, w.dh_mid, nullptr, nullptr, st))) return rc;
  if ((rc = layer_weight_grads(Lf[1], T, w.fb[0].H, fg.w_ih[1], fg.w_hh[1], fg.b_ih[1], fg.b_hh[1], wg, st))) return rc;
  return layer_weight_grads(Lf[0], T, w.xfb, fg.w_ih[0], fg.w_hh[0], fg.b_ih[0], fg.b_hh[0], wg, st);
}

// ---- unit-test hook of one section's norm + unfold backward (include/fsn_b200.h): the launchers
// fsn_improved_train_backward runs per section, every argument checked before any CUDA call
extern "C" int fsn_debug_imp_unfold_bwd(const float* dX, const float* Xn, const float* invs, const float* y, int B, int T,
                                        int Fu, int lo, int hi, int cs, int ns, int cf, int nf, int first, int act,
                                        float* dot, float* dfb, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(dX && Xn && invs && dot && dfb && (act == FSN_ACT_NONE || y), FSN_ERR_SHAPE,
              "improved unfold backward hook: null argument");
  FSN_REQUIRE(B > 0 && T > 0 && Fu >= 2 && hi <= Fu, FSN_ERR_SHAPE, "improved unfold backward hook: bad shape B=%d T=%d Fu=%d",
              B, T, Fu);
  FSN_REQUIRE(act == FSN_ACT_NONE || act == FSN_ACT_RELU, FSN_ERR_UNSUPPORTED,
              "improved unfold backward hook: act none or ReLU are built");
  SecGeom g;
  int rc = sec_geom(lo, hi, cs, ns, cf, nf, Fu, g);
  if (rc) return rc;
  FSN_REQUIRE((size_t)T * B * g.N * g.W < ((size_t)1 << 31) && (size_t)T * B * Fu < ((size_t)1 << 31), FSN_ERR_SHAPE,
              "improved unfold backward hook: tensors must stay below 2^31 elements");
  const cudaStream_t st = (cudaStream_t)stream;
  if ((rc = train_dot_launch(dX, Xn, T, B * g.N, g.N, g.W, B, dot, st))) return rc;
  return imp_unfold_bwd_launch(dX, invs, dot, (float)g.N * g.W * T, g, B, T, Fu, first != 0, act, y, dfb, st);
}
