// Internal (non-ABI) declarations shared by the translation units of libfsn_b200.
#pragma once
#include <cudaTypedefs.h>
#include <cuda_fp16.h>

#include "fsn_common.cuh"

namespace fsn {

// Bump allocator over a caller's workspace: every block starts on a 256-byte boundary.  With a null base it hands out
// nullptr and only counts the bytes, which is how the *_workspace_bytes queries size the same layout.
struct Carver {
  char* base; size_t off;
  explicit Carver(void* p) : base((char*)p), off(0) {}
  template <class T> T* take(size_t n) {
    T* r = base ? (T*)(base + off) : nullptr;
    off = align_up(off + n * sizeof(T), 256);
    return r;
  }
};

// layer l of a two-layer stack
inline fsn_lstm_layer seq_layer(const fsn_seq_weights& w, int l) { return {w.w_ih[l], w.w_hh[l], w.b_ih[l], w.b_hh[l]}; }

// grid of a grid-stride elementwise kernel of 256 threads over n elements: one element per thread up to 132 * 16 blocks
// (16 per SM of an H100 SXM)
inline unsigned ew_grid(size_t n) {
  const size_t g = (n + 255) / 256;
  return (unsigned)(g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g));
}

// v (the gradient at the output of an activation, FSN_ACT_*) times its derivative, from the post-activation output y
// (unread for FSN_ACT_NONE)
__device__ __forceinline__ float act_grad(float v, const float* y, size_t i, int act) {
  if (act == FSN_ACT_RELU) return y[i] > 0.f ? v : 0.f;
  if (act == FSN_ACT_RELU6) { const float a = y[i]; return (a > 0.f && a < 6.f) ? v : 0.f; }
  if (act == FSN_ACT_TANH) { const float a = y[i]; return v * (1.f - a * a); }
  return v;
}

// Sub-band row -> (clip, frequency) map.  Row r = b' * Fsub + f' of the sub-band batch.
// G <= 1: identity (Fsub = F).  G > 1: drop_band (audio_zen/acoustics/feature.py:332-345):
// output clip b' of group g is input clip g + G*i, frequency f' is input bin g + G*f'.
struct RowMap {
  int B, F, Fsub, G;
};

__host__ __device__ inline void row_to_unit(const RowMap& m, int r, int& b, int& f) {
  int bq = r / m.Fsub;
  const int fq = r - bq * m.Fsub;
  if (m.G <= 1) { b = bq; f = fq; return; }
  int g = 0;
  for (; g < m.G; ++g) {
    const int cnt = (m.B - g + m.G - 1) / m.G;
    if (bq < cnt) break;
    bq -= cnt;
  }
  b = g + m.G * bq;
  f = g + m.G * fq;
}

enum { SEG0_DENSE = 0, SEG0_GATHER = 1 };

struct StepParams {
  int R, K0, H, first;
  int gru;  // 0: LSTM (4 gates i,f,g,o); 1: GRU (weights [3H,.] r,z,n; h_prev is read in the update; no cell state)
  const float* w_ih; const float* w_hh; const float* b_ih; const float* b_hh;
  const float* h_prev; size_t h_prev_stride;
  float* h_out; size_t h_out_stride;
  float* c;
  // training only (both nullable): previous cell state read from c_in instead of c; post-activation gates
  // (i,f,g,o) of this step stored at save_gates[row*4H + g*H + u]
  const float* c_in; float* save_gates;
  // SEG0_DENSE: x = x0[row * x0_row_stride + k] * (row_scale ? row_scale[row] : 1)
  const float* x0; size_t x0_row_stride; const float* row_scale;
  int row_scale_div;  // scale index = row / row_scale_div (0 or 1: per row)
  // SEG0_GATHER: sub-band unit of row r at frame t (base_model.py:13-46 + model.py:98-111)
  const float* magT; const float* fbT; const float* inv2;
  const float* unit_scale;  // nullable: per-row scale of this step (cumulative norm) instead of inv2[clip]
  int F, Tp, t, Ns, Nf;
  RowMap map;
};

int lstm_step_launch(const StepParams& p, int mode, cudaStream_t st);
// per-step state of a two-layer stack: layer 0's h ping-pong h0[2] [R,H0] and cell c0; layer 1's cell c1 and its h, either
// a ping-pong h1[2] [R,H1] (keep_steps = 0) or one [R, keep_steps, H1] tensor h1[0] that keeps every step.  carry (chunked
// streaming): step 0 continues from the state in h0[1], c0, h1_at(-1) and c1 instead of starting from zero.
struct Step2State {
  float *h0[2], *c0, *h1[2], *c1;
  int H1, keep_steps;
  bool carry;
  float* h1_at(int t) const { return keep_steps ? h1[0] + (size_t)(t > 0 ? t : 0) * H1 : h1[t & 1]; }
  size_t h1_stride() const { return (size_t)(keep_steps ? keep_steps : 1) * H1; }
};
// step t of a two-layer stack on the per-step kernels.  p: layer 0 of step t with R, H, gru, its weights and its input
// (K0 and the SEG0_DENSE / SEG0_GATHER fields of `mode`) filled in; the helper sets the step and state fields, then runs
// layer 1 (weights w1) on layer 0's h_t.  Layer 1's h_t is then at s.h1_at(t).
int lstm_step2_launch(StepParams p, int mode, int t, const fsn_lstm_layer& w1, const Step2State& s, cudaStream_t st);
// cumulative_laplace_norm (base_model.py:220-251): scale1T[t*B+b] from the frame sums fs[b*Tp+t].x, and
// scaleT[t*R+r] of every sub-band unit (running mean over its K rows and the frames so far)
int cum_clip_scale_launch(const float2* fs, int B, int Tp, int F, float eps, float* scale1T, cudaStream_t st);
int cum_unit_scale_launch(const float* magT, const float* fbT, RowMap map, int R, int Tp, int Ns, int Nf, float eps,
                          float* scaleT, cudaStream_t st, bool time_major = false);
// one frame's sum over the features of sub-band unit f, in the order of cum_unit_scale_kernel and its streaming variant:
// the 2Ns+1 reflected rows of mag, then the 2Nf+1 reflected rows of fb (both [F] of that frame)
__device__ __forceinline__ float unit_frame_sum(const float* mag, const float* fb, int f, int F, int Ns, int Nf) {
  float s = 0.f;
  for (int k = -Ns; k <= Ns; ++k) s += mag[reflect_idx(f + k, F)];
  for (int k = -Nf; k <= Nf; ++k) s += fb[reflect_idx(f + k, F)];
  return s;
}
// forgetting_norm (base_model.py:102-151): mu_t = a_t mu_{t-1} + b_t m_t per clip, m_t the mean of frame t over the
// features, scale 1 / (mu_t + 1e-10).  The coefficients are rounded as the reference rounds them: for t < 192,
// a_t = float32(min((t-1)/(t+1), alpha)) and b_t = 1 - a_t in float32 (a_0 = -1, b_0 = 2; a_1 = 0); from t = 192 on,
// a = float32(alpha) and b = float32(1 - alpha) rounded from the double.  Entry min(t, 192) holds frame t's pair.
static const int FORGET_LEN = 192;
static const float FORGET_EPS = 1e-10f;
struct ForgetCoef { float a[FORGET_LEN + 1], b[FORGET_LEN + 1]; };
ForgetCoef forget_coef();
// the norms whose first-norm scale is per (step, clip) rather than per clip
inline bool norm_per_step(int norm_type) { return norm_type != FSN_NORM_OFFLINE_LAPLACE; }
// scaleT[t*B + b] = 1 / (mu_t + 1e-10) and muT[t*B + b] = mu_t (nullable) of clip b, one thread per clip in the exact
// float32 operation order of the reference (no contraction).  fs2 == nullptr: m_t = fs[b*Tp + t].x / cnt (first norm:
// the plain frame sum); else m_t = (fs[.].y + fs2[.].y) / cnt (second norm: the reflect-weighted sums of the noisy and
// full-band unfolds, cnt = F K).  lens (nullable, device [B] samples): clip b scans only its own Tp_b = 1 + lens[b]/hop
// + la frames and leaves the rest of its entries unwritten; those frames equal the unbounded scan's (it is causal).
int forget_scale_launch(const float2* fs, const float2* fs2, int B, int Tp, float cnt, float* scaleT, float* muT,
                        cudaStream_t st, const int* lens = nullptr, int hop = 0, int la = 0);
// unit_scale[t*R + r] = scaleT[t*B + clip(r)]: the per-(step, clip) table in the per-(step, row) layout the sub-band
// consumers read (the tensor-core kernel's unit_scale, the fp32 loop's unit_scale, the training gather)
int forget_unit_broadcast_launch(const float* scaleT, RowMap map, int R, int Tp, float* unit_scale, cudaStream_t st);

// TMA tensor maps (fsn_tgemm.cu).  tmap_encoder: cuTensorMapEncodeTiled through the runtime's driver entry point (no link
// against libcuda), nullptr when the driver lacks it.  encode_tmap_2d: a row-major 2-D array of `inner` elements per row,
// `rows` rows pitch_bytes apart, read in boxes of box_inner x box_rows with 128B swizzle, zero fill outside; false when
// the encoder is missing or refuses the layout
PFN_cuTensorMapEncodeTiled_v12000 tmap_encoder();
bool encode_tmap_2d(CUtensorMap* m, CUtensorMapDataType dtype, const void* base, cuuint64_t inner, cuuint64_t rows,
                    cuuint64_t pitch_bytes, cuuint32_t box_inner, cuuint32_t box_rows);

// tf32 wgmma GEMM (fsn_tgemm.cu): C[M,N] (+)= A[M,K] B[N,K]^T, fp32 row-major operands with 16-byte aligned rows.
// tgemm_available: the device can run it (sm_90, opt-in shared memory) and the driver has the tensor-map encoder; asks
// the CUDA runtime
bool tgemm_available();
bool tgemm_supported(const float* A, size_t lda, const float* Bm, size_t ldb, int K);
int tgemm_launch(const float* A, size_t lda, const float* Bm, size_t ldb, float* C, size_t ldc, int M, int N, int K,
                 bool accumulate, float* scratch, size_t scratch_floats, cudaStream_t st);

// weight-gradient GEMMs C[M,N] (+)= A^T B over a long K with block-tiled K-major operand copies (fsn_tgemm.cu)
size_t tgemm_blocked_floats(size_t K, int M);
int transpose_blocked_launch(const float* in, size_t K, int M, size_t ld, float* out, cudaStream_t st, float* colsum_part,
                             int max_slabs, int* slabs);
// out[c] (and out2[c] when given) = sum_{z < S} part[z * cols + c] in a fixed order (fsn_train.cu): the second pass of
// a column sum, e.g. over the colsum_part slabs of transpose_blocked_launch
int colsum_final_launch(const float* part, int S, int cols, float* out, float* out2, cudaStream_t st);
int tgemm_blocked_launch(const float* Ablk, int nkb_a, int a_kb0, const float* Bblk, int nkb_b, int b_kb0, float* C, size_t ldc,
                         int M, int N, int K, bool accumulate, float* scratch, size_t scratch_floats, cudaStream_t st);

bool lstm_fwd_step_supported(const float* Hbuf, const float* w_hh, int H);
bool lstm_fwd_step_folds_input(const float* X, const float* w_ih, int K0);
// optional fp16 MMA operands of the step kernel: previous hidden state, weights, folded layer input; H16_out receives h_t
struct LstmStepHalf {
  const __half *Hprev16, *w_hh16, *Xt16, *w_ih16;
  __half* H16_out;
};
int to_half_launch(const float* in, size_t n, __half* out, cudaStream_t st);
int lstm_fwd_step_launch(const float* Hprev, const float* w_hh, const float* Xt, const float* w_ih, int K0, float* Gt,
                         const float* b_ih, const float* b_hh, const float* C_prev, float* C_out, float* H_out, int R, int H,
                         cudaStream_t st, const LstmStepHalf* h = nullptr);

// one LSTM layer over all steps on the tf32 tensor-core path (fsn_train.cu): one lstm_fwd_step_kernel per step when
// H % 32 == 0 (the layer input folded in up to 512 wide, else one hoisted projection GEMM of all steps), otherwise per
// step the recurrent GEMM into `rec` [R,4H] and the cell kernel.  G [Tp,R,4H] (post-activation gates), C, H [Tp,R,H]
// receive every step.  X [Tp,R,K0] contiguous.
struct LayerSave { float *G, *C, *H; };
// fp16 side buffers of one layer (all nullable): H16 [Tp,R,H] copy of the hidden states (written by the step kernel, the
// next layer's X16), X16 [Tp,R,K0] copy of the layer input, w16: 4H*(H+K0) halfs for the weight copies
struct LayerHalf { __half* H16; const __half* X16; __half* w16; };
int layer_forward_save_tc(const fsn_lstm_layer& w, const float* X, int R, int K0, int H, int Tp, const LayerSave& s,
                          float* rec, cudaStream_t st, float* splitk = nullptr, size_t splitk_floats = 0,
                          const LayerHalf* half = nullptr);
// fp32 variant: one SIMT step kernel per step (lstm_step_launch with save_gates)
int layer_forward_save(const fsn_lstm_layer& w, const float* X, int R, int K0, int H, int Tp, const LayerSave& s,
                       cudaStream_t st);

static const size_t SPLITK_SCRATCH_FLOATS = (size_t)16 << 20;  // 64 MB of split-K partial sums
static const int COLSUM_MAX_S = 512;                            // row slabs of a column sum

// Per-layer precision of the training steps: a layer runs on the tf32 tensor cores when the step asks for FSN_PREC_TF32_TC
// and its hidden size keeps the rows of its operands 16-byte aligned; otherwise on the fp32 kernels.  tf32_layer sizes the
// workspaces (no GPU needed); the layers themselves also need tgemm_available(), else the whole layer - forward, BPTT and
// weight gradients alike - runs the fp32 kernels in the tensor-core layout of the workspace.
inline bool tf32_layer(int precision, int H) { return precision == FSN_PREC_TF32_TC && (H & 3) == 0; }
// forward of one layer of a training step, on the variant tf32_layer and tgemm_available pick (the fp32 one ignores rec /
// splitk / half)
int layer_forward(int precision, const fsn_lstm_layer& w, const float* X, int R, int K0, int H, int Tp, const LayerSave& s,
                  float* rec, float* splitk, const LayerHalf* half, cudaStream_t st);

// ---- back-propagation through time of one LSTM layer (fsn_train.cu), shared by the training steps
struct LayerBwd {
  const float *w_ih, *w_hh;
  LayerSave s;
  int R, K0, H;
  float *dh_rec, *dc;
  float *w_hhT, *w_ihT;        // tensor-core path: [H,4H] / [K0,4H] transposed copies (else nullptr; unused when
                               // !tgemm_available())
  float* splitk;               // split-K space of the per-step GEMMs (used when the layer has only a few tiles)
};
// scratch of layer_weight_grads: K-major copies of dG / layer input (tensor-core path, tgemm_blocked_floats of the largest
// layer), split-K space (SPLITK_SCRATCH_FLOATS) and column-sum partials (colsum_floats, COLSUM_MAX_S x 4H for full slabs)
struct WgradScratch { float *gT, *xT, *splitk, *colsum; size_t colsum_floats; };
// tensor-core path: writes L.w_hhT, and L.w_ihT when the layer has one (it computes a dx); nothing when L.w_hhT is null
int layer_bwd_transpose_weights(const LayerBwd& L, cudaStream_t st);
// step t of one layer: pointwise gate gradients (d h from above = dh_above + dout W_fc for an O-output Linear on top),
// then dh_rec = dG W_hh and, when dx != nullptr, dx = dG W_ih
int layer_bwd_step(const LayerBwd& L, int t, int Tp, const float* dh_above, const float* dout, const float* fc_w, int O,
                   float* dx, cudaStream_t st);
// weight / bias gradients of one layer from dG [Tp*R,4H] (in L.s.G), its input X [Tp*R,K0] and hidden states
int layer_weight_grads(const LayerBwd& L, int Tp, const float* X, float* g_w_ih, float* g_w_hh, float* g_b_ih, float* g_b_hh,
                       const WgradScratch& w, cudaStream_t st);
// BPTT of a stack of n layers (L[0] at the bottom), one step at a time from the top: every layer at step t before any at
// t-1.  The top layer's d h comes from dh_above [steps, R, H] or from an O-output Linear on top (dout [steps, R, O],
// fc_w [O, H]); layer l < n-1 takes layer l+1's dx of the same step through dh_mid0 / dh_mid1 (alternating; dh_mid1 is
// used only when n > 2); layer 0's dx goes to dx [steps, R, K0] when given.  Each L[l] carries its own dh_rec / dc slot.
int stack_bwd(const LayerBwd* L, int n, int steps, const float* dh_above, const float* dout, const float* fc_w, int O,
              float* dh_mid0, float* dh_mid1, float* dx, cudaStream_t st);
// input of a training step (fullsubnet/model.py:85-92, fullband_baseline/model.py:46-56): look-ahead pad, first norm and
// the time-major copies raw [Tp,B,F] (unscaled) and scaled [Tp,B,F] (normalised); sums[b] = per-clip (sum, sum_f c_Ns[f]
// * row sum), inv1[b] = 1 / (mean + eps).  cum: causal running mean instead, fs [B*Tp] frame sums, cum1 [Tp*B] scales
// (fs / cum1 unused otherwise).  norm_type (FSN_NORM_*) picks the running mean: cumulative or forgetting.
static const float TRAIN_CUM_EPS = 1.1920928955078125e-07f;  // audio_zen/constant.py:9
int train_input_launch(const float* noisy_mag, int B, int F, int T, int Tp, int Ns, int norm_type, float2* sums, float* inv1,
                       float* raw, float* scaled, float2* fs, float* cum1, cudaStream_t st);
// sub-band input of a training step X [Tp, R, K] (base_model.py:13-46 + model.py:98-119) from the time-major raw / fbz
// [Tp,B,F]: unit (b,f) of row r (map), 2Ns+1 reflected raw rows || 2Nf+1 reflected fbz rows, times inv2[b], or
// unit_scale[t*R + r] when given (the causal norms); a grid-stride kernel of 132 * 8 CTAs
int train_gather_launch(const float* raw, const float* fbz, const float* inv2, const float* unit_scale, float* X, RowMap map,
                        int Tp, int R, int Ns, int Nf, cudaStream_t st);
// its backward: dY [Tp,B,2F] = dout [B,2,F,T] re-laid out, zero on the first `la` frames, times act'(y) (FSN_ACT_*) from
// the kept post-activation output y (unread for FSN_ACT_NONE)
int train_dy_launch(const float* dout, const float* y, int act, int B, int F, int T, int Tp, int la, float* dY,
                    cudaStream_t st);
// fp32 SIMT GEMM C[M,N] (+)= op(A) B (op(A) = A^T when ta), split-K over `scratch` (scratch_floats; S M N partial sums
// must fit, S drops until they do) for long K (deterministic)
int sgemm_launch(bool ta, const float* A, size_t lda, const float* Bm, size_t ldb, float* C, size_t ldc, int M, int N, int K,
                 bool accumulate, float* scratch, size_t scratch_floats, cudaStream_t st);
// out[c] (and out2[c] when given) = sum_r X[r*ldx + c], fixed order; S = min(ceil(rows / 2048), COLSUM_MAX_S) row slabs
// of partials in scratch: FSN_ERR_WORKSPACE when S * cols > scratch_floats
int colsum_launch(const float* X, size_t rows, int cols, size_t ldx, float* out, float* out2, float* scratch,
                  size_t scratch_floats, cudaStream_t st);
// dW [2,H] = dout^T Hm of the 2-output sub-band Linear (dout [rows,2], Hm [rows,H]), partials in scratch (S 2 H floats,
// S dropping until they fit; FSN_ERR_WORKSPACE when even 2 H do not)
int small_out_wgrad_launch(const float* dout, const float* Hm, size_t rows, int H, float* dW, float* scratch,
                           size_t scratch_floats, cudaStream_t st);
// backward of a Linear Y = X W^T + b over `rows` rows, dY [rows,N], X [rows,K], W [N,K]: dW = dY^T X (split-K over
// `splitk`), db = colsum dY (partials in `colsum`) and, when dX != nullptr, dX = dY W
int linear_bwd(const float* dY, const float* X, const float* W, int rows, int N, int K, float* dW, float* db, float* dX,
               float* splitk, float* colsum, size_t colsum_floats, cudaStream_t st);
// out [cols, rows] = in [rows, cols]^T
int transpose_launch(const float* in, size_t rows, int cols, float* out, cudaStream_t st);
// per-clip (sum, sum_f c_N[f] * row sum) of a time-major x [Tp,B,F] (train_tm_stats) or of mag [B,F,T]
// (train_mag_stats), one CTA per clip, fixed-order tree
int train_tm_stats_launch(const float* x, int B, int F, int Tp, int N, float2* sums, cudaStream_t st);
int train_mag_stats_launch(const float* mag, int B, int F, int T, int Ns, float2* sums, cudaStream_t st);
// dot[b'] = sum over the rows [b'*Fsub, (b'+1)*Fsub) of every step of dX * X [Tp,R,K]  (laplace-norm backward), one CTA
// per clip b' < clips
int train_dot_launch(const float* dX, const float* X, int Tp, int R, int Fsub, int K, int clips, float* dot, cudaStream_t st);
// backward of fullsubnet's second offline norm + drop_band with respect to the full-band output (Nf = 0, its column K-1
// of the sub-band input X [Tp,R,K]): dz [Tp,B,F] = act'(fbz) * (dX[t, row(b,f), K-1] inv2[b] - inv2[b] dot[b'] / cnt2),
// one grid-stride kernel; units drop_band removed keep the norm-mean term
int train_dfbz_launch(const float* dX, const float* fbz, const float* inv2, const float* dot, RowMap map, int Tp, int R, int K,
                      float cnt2, int act, float* dz, cudaStream_t st);
// the same for the second cumulative norm (scaleT [Tp,R]): dunit [Tp,R] = gradient of the full-band column of every unit
// (one thread per row, suffix sum over t), then dz = act'(fbz) * dunit of the unit's row (0 where drop_band removed it)
int train_cum_unit_bwd_launch(const float* dX, const float* X, const float* scaleT, int Tp, int R, int K, float* dunit,
                              cudaStream_t st);
int train_dfbz_cum_launch(const float* dunit, const float* fbz, RowMap map, int Tp, int R, int act, float* dz,
                          cudaStream_t st);
// the same for the second forgetting norm (scale2T [Tp,B], one scale per (step, clip) over all F K features; Nf = 0):
//   dot[t,b] = <dX, X> over the kept rows of clip b at step t (one CTA per (t, b), fixed tree);
//   reverse recurrence per clip: g_t = -s_t dot[t,b] + a_{t+1} g_{t+1}, mid[t,b] = b_t g_t / cnt  (d loss / d m_t over
//   the cnt = F K features the mean averages; dot and mid share the buffer mid [Tp,B]);
//   dz[t,b,f] = act'(fbz) * (dX[t, row(b,f), K-1] s_t + mid[t,b])  (a unit drop_band removed still feeds the mean).
int train_forget_bwd_launch(const float* dX, const float* X, const float* fbz, const float* scale2T, RowMap map, int Tp,
                            int R, int K, float cnt, int act, float* mid, float* dz, cudaStream_t st);

// shapes of one fast_fullsubnet Model.forward call (fsn_fast_model.cu): Ts = shrunk steps of the bottleneck; cum: the
// descriptor asks for the cumulative norm
struct FastDims { int B, T, Tp, F, M, K, Ts, S; bool cum; };
int fast_dims(const fsn_fast_desc* d, int B, int T, FastDims& m);
// fast_fullsubnet's second cumulative norm (model.py:186-187, base_model.py:220-251) on the down-sampled bottleneck
// input bn [Ts, R, K] (time-major, before the norm): scaleT[ts*R + r] = 1 / (mean of row r over its K features and the
// shrunk steps <= ts + eps)
int fast_cum_bn_scale_launch(const float* bn, int R, int K, int Ts, float eps, float* scaleT, cudaStream_t st);
// first frame of shrunk step ts and the number of frames averaged into it (fast_fullsubnet/model.py:108-129)
__device__ __forceinline__ void shrink_block(int ts, int S, int Tp, int& t0, int& len) {
  if (ts == 0) { t0 = 0; len = 1; return; }
  t0 = 1 + (ts - 1) * S;
  len = min(t0 + S, Tp) - t0;
}
// fast_fullsubnet bottleneck input before its norm (model.py:174-187) from melT / encT, element (b, t, m) of both at
// b*bs + t*ts + m: row (b,m) of shrunk step ts, feature k = 2Nn+1 reflected noisy-mel rows || 2Ne+1 reflected encoder
// rows, averaged over the block of ts, into bn [Ts, B*M, K]; fs[b*Ts + ts] = fixed-order sum of the (b, ts) block (.x and
// .y alike, the layout clip_reduce_only_launch reads)
int fast_bn_input_launch(const float* melT, const float* encT, size_t bs, size_t ts, int B, int Tp, int M, int Nn, int Ne,
                         int S, int Ts, float* bn, float2* fs, cudaStream_t st);
// fast_fullsubnet backward (fsn_fast_train.cu).  ftr_dbn: d bn_out [Ts, B*M] = ReLU'(bn_out) * sum of the up-sampled
// half (columns M..2M-1) of d dec_in [Tp,B,2M] over the frames that read each shrunk step.  ftr_cum_suffix (cumulative
// norm): suffix [Ts, B*M] of the second norm's backward from dX, X [Ts, B*M, K] and scaleT [Ts, B*M].  ftr_denc: d encT
// [Tp,B,M] through the second norm, down-sampling and unfold (offline: inv2 [B], dot [B], cnt2 = M K Ts; cum: scaleT,
// suffix) plus the decoder-input half ddec[., :M], times ReLU'(encT)
int ftr_dbn_launch(const float* ddec, const float* bn_out, int B, int Tp, int M, int S, int Ts, float* dbn, cudaStream_t st);
int ftr_cum_suffix_launch(const float* dX, const float* X, const float* scaleT, int Ts, int R, int K, float* suffix,
                          cudaStream_t st);
int ftr_denc_launch(bool cum, const float* ddec, const float* dX, const float* encT, const float* inv2, const float* dot,
                    const float* scaleT, const float* suffix, int B, int Tp, int M, int Nn, int Ne, int S, float cnt2,
                    float* denc, cudaStream_t st);
// fast_fullsubnet decoder input (model.py:191-194): dec_in row (b,t) = [encoder output (M) | up-sampled bottleneck output
// (M)].  Row (b,t) of encT [., M] and dec_in [., 2M] is b*rbs + t*rts (clip-major: Tp, 1; time-major: 1, B); frame t reads
// shrunk step min(t/S, Ts-1) of bn_out, element (b, m, ts) at b*nbs + m*nms + ts*nts
int fast_dec_input_launch(const float* encT, const float* bn_out, size_t nbs, size_t nms, size_t nts, int B, int Tp, int M,
                          int S, int Ts, size_t rbs, size_t rts, float* dec_in, cudaStream_t st);
// out[i] = in[i] * scale[((i / cols) % rows) / div] over n elements (in may be out): rows of `cols` elements, the scale
// of a row shared by `div` consecutive rows and repeating every `rows` rows
int scale_rows_launch(const float* in, const float* scale, size_t n, int cols, int rows, int div, float* out,
                      cudaStream_t st);

// shapes of one Model.forward call (fsn_model.cu)
struct Dims {
  int B, T, Tp, F, Fsub, G, R, Ksb;
};
int make_dims(const fsn_model_desc* d, int B, int T, Dims& m);

// (clip, frequency) -> sub-band row, or -1 when drop_band removed the unit (inverse of row_to_unit)
__host__ __device__ inline int unit_to_row(const RowMap& m, int b, int f) {
  if (m.G <= 1) return b * m.Fsub + f;
  const int g = b % m.G;
  if (f % m.G != g || f / m.G >= m.Fsub) return -1;
  int off = 0;
  for (int gg = 0; gg < g; ++gg) off += (m.B - gg + m.G - 1) / m.G;
  return (off + b / m.G) * m.Fsub + f / m.G;
}
int fc_gemm_launch(const float* A, const float* W, const float* bias, float* out, int M, int K, int O, int act,
                   cudaStream_t st, bool w_kmajor = false);
// Where a sub-band head Linear(H -> O <= 2c) writes: row r = b*N + n of the sub-band batch, output o = ch*c + j goes to
// out[((b*2 + ch)*rows + lo + n*c + j)*rs + t] at frame t, i.e. a [B, 2, rows, frames] cRM with rows rs apart and
// contiguous frames (fullsubnet/model.py:129-135: c = 1; improved_fullsubnet/model.py:239-247: one section, c its centre
// width; with N = R every row is clip 0 and channel 0 is a plain [rows, frames] table).  bs (0 = 2 rows rs, the layout
// above): clips bs elements apart instead, e.g. the frame-major [B, frames, 2, rows] cRM of the streaming call with rs = 1
struct HeadGeom {
  int N, c, lo, rows;
  size_t rs, bs;
};
// element of the cRM that output o of sub-band row r goes to at frame t
__device__ __forceinline__ size_t head_index(const HeadGeom& g, int r, int o, int t) {
  const int b = r / g.N, n = r - b * g.N, ch = o / g.c, j = o - ch * g.c;
  const size_t bs = g.bs ? g.bs : 2 * (size_t)g.rows * g.rs;
  return (size_t)b * bs + ((size_t)ch * g.rows + g.lo + n * g.c + j) * g.rs + t;
}
// out = act(h W^T + b) for `steps` frames of h [steps, R, H] into frames t0 .. t0+steps-1 of g; one warp per (step, row,
// output): lane-strided fmaf over H, warp_sum, + bias, act (FSN_ACT_*)
int sb_head_launch(const float* h, int R, int H, int steps, const float* W, const float* bias, int O, int act, float* out,
                   const HeadGeom& g, int t0, cudaStream_t st);
// its backward: dY [steps, R, O] from the cRM gradient dcrm laid out by g, zero on the first `la` steps (step t reads
// frame t - la), times act'(y) of the kept post-activation output y in the same layout (unread for FSN_ACT_NONE)
int sb_head_bwd_launch(const float* dcrm, const float* y, int act, int R, int O, int steps, int la, const HeadGeom& g,
                       float* dY, cudaStream_t st);
// fullsubnet's sub-band Linear(H -> 2): row r = b'*Fsub + f' into crm [B', 2, Fsub, T]
inline HeadGeom fsn_head_geom(int Fsub, int T) { return HeadGeom{Fsub, 1, 0, Fsub, (size_t)T}; }
// output of a Linear(H -> 2F) head: y rows (b,t) of 2F (channel c*F+f), row (b,t) at b*bs + t*ts elements -> out
// [B,2,F,Tp-la], dropping the first `la` frames
int crm_output_launch(const float* y, size_t bs, size_t ts, int B, int Tp, int F, int la, float* out, cudaStream_t st);
// mag [B,F,T] -> out, element (b,t,f) at b*bs + t*ts + f, for t < Tp with frames T..Tp-1 zero (look-ahead pad);
// scaled (nullable) receives the same elements times scale[b]
int transpose_mag_launch(const float* in, int B, int F, int T, int Tp, size_t bs, size_t ts, float* out,
                         const float* scale, float* scaled, cudaStream_t st);
// transpose_mag_launch and imp_compress_launch put the clip in gridDim.z, crm_output_launch the (clip, channel) pair:
// an entry point that reaches them checks B with layout_clips_check (crm: it runs crm_output_launch) before any CUDA
// call, FSN_ERR_UNSUPPORTED beyond the grid.  `who` prefixes the message.
static const int LAYOUT_MAX_GRID_Z = 65535;
int layout_clips_check(int B, bool crm, const char* who);
// fs[b*Tp + t] = (sum_f x, sum_f c_N[f] x) of the frames of x, element (b,t,f) at b*bs + t*ts + f
int frame_stats_launch(const float* x, int B, int Tp, int F, int N, size_t bs, size_t ts, float2* fs, cudaStream_t st);
// Per-clip lengths (lens non-null, device [B] samples): clip b sums only its own Tp_b = 1 + lens[b]/hop + la frames of
// the T_pad-strided partials, with the same per-thread stride and tree as a call with T_pad = Tp_b; norm_scales_launch
// then takes cnt1 / cnt2 per frame and multiplies them by Tp_b.
int clip_stats_launch(const float* x, int B, int T_pad, int F, int N, float2* fs, float2* sums, cudaStream_t st,
                      const int* lens = nullptr, int hop = 0, int la = 0);
int clip_reduce_only_launch(const float2* fs, int B, int T_pad, float2* sums, cudaStream_t st, const int* lens = nullptr,
                            int hop = 0, int la = 0);
int norm_scales_launch(const float2* mag_sums, const float2* fb_sums, int B, float cnt1, float cnt2, float* inv1,
                       float* inv2, cudaStream_t st, float eps = 1e-5f, const int* lens = nullptr, int hop = 0,
                       int la = 0);

// the n_fft the signal layer accepts: a power of two in [16, 2048] (radix-2 FFT) or even in [16, 1200] (direct DFT)
bool dsp_size_ok(int n_fft);
// the host checks stft_launch makes before any CUDA call, for entry points that must refuse before their own launches
int stft_check(int B, int L, int n_fft, int hop, int win_length, const float* magT, int T_pad);
// lens (nullable, device [B]): clip b has lens[b] of the L samples of its row (the *_enhance entry points)
int stft_launch(const float* wav, int B, int L, int n_fft, int hop, int win_length, float* mag, float* phase,
                float* real, float* imag, float* magT, int T_pad, cudaStream_t st, const int* lens = nullptr);
// mask_mode: 1 = decompress_cIRM + complex product (fullsubnet), 2 = element-wise re*crm0, im*crm1 (improved_fullsubnet)
int istft_launch(const float* real, const float* imag, int cstride, const float* crm, int B, int T, int n_fft,
                 int hop, int win_length, int length, float* wav, cudaStream_t st, int mask_mode = 1,
                 unsigned int* peak_bits = nullptr, const int* lens = nullptr);
// peak_bits (optional, [B]): max|wav| per clip as float bits, reduced in the iSTFT epilogue (radix-2 and direct DFT alike,
// bounded by lens when given); wav_epilogue turns it into the int16 scaling of the reference host loop
// (audio_zen/inferencer/base_inferencer.py:181-182)

// ---- the wav side of the wav -> wav entry points (fsn_enhance, fsn_fullband_enhance, fsn_improved_enhance).  Each reads
// dims -> wav_check -> carve -> workspace check -> wav_prologue -> its own STFT / model / iSTFT (peak when pcm is given,
// lens) -> wav_epilogue.
struct WavWs {
  float *real, *imag, *crm;  // spectrum of the input [B,F,T]; cRM [B,2,F,T] when the caller keeps none
  unsigned int* peak;        // per-clip max|y| of the int16 output
  int* lens;                 // device copy of the per-clip lengths; nullptr after wav_prologue when the call has none
};
// F = 0: the peak and length table only (improved_fullsubnet carves its spectrum and cRM where its forward needs them)
void wav_carve(Carver& c, int B, int F, int T, WavWs& w);
// host checks before any CUDA call.  lengths (nullable, host [B]): n_fft/2 < lengths[b] <= L_max and max == L_max, else
// FSN_ERR_SHAPE naming the clip; with pow2_lengths a non-power-of-two n_fft refuses them (FSN_ERR_UNSUPPORTED).
// enhanced must be non-null.  `who` prefixes the messages.
int wav_check(const int32_t* lengths, int B, int L_max, int n_fft, bool pow2_lengths, const float* enhanced,
              const char* who);
// device length table w.lens <- lengths through kernel parameters (the host array is not read after the call); no
// lengths: w.lens = nullptr, so the kernels that take lens run their whole-row path
int wav_prologue(const int32_t* lengths, int B, WavWs& w, cudaStream_t st);
// pcm (nullable) <- int16 scaling of enhanced [B,L] by the peak; with lengths, the caller's crm_out [B,2,F,T] (nullable)
// is zeroed for frames t >= 1 + lengths[b]/hop
int wav_epilogue(const WavWs& w, const float* enhanced, int B, int L, int16_t* pcm, float gain, float* crm_out, int F, int T,
                 int hop, cudaStream_t st);

// adjoint of the element-wise mask + iSTFT of improved_fullsubnet (istft_launch mask_mode 2) with respect to the mask:
// dwav [B,L] -> dcrm [B,2,F,T] for the rows f < F-1 (the Nyquist row of the cRM is a constant; it is not written)
int istft_mask_adjoint_launch(const float* dwav, const float* real, const float* imag, int B, int L, int T, int n_fft,
                              int hop, int win_length, float* dcrm, cudaStream_t st);

// improved_fullsubnet (fsn_improved.cu), shared by its inference forward and its training step
struct SecGeom { int lo, N, cs, ns, cf, nf, W; };  // section rows [lo, lo + N*cs), unit width W
struct ImpDims { int B, L, T, F, Fu, S; SecGeom sec[FSN_IMP_MAX_SECTIONS]; int maxRW, maxR; };
int imp_dims(const fsn_improved_desc* d, int B, int L, ImpDims& m);
// |X|^fdrc with the Nyquist bin dropped (model.py:564-565): mag [B,F,T] -> out [B,T,F-1], or [T,B,F-1] when tm
int imp_compress_launch(const float* mag, int B, int F, int T, float fdrc, bool tm, float* out, cudaStream_t st);
// section input (model.py:321-443): X [T, B*N, W] of the reflected noisy rows of magc and full-band rows of fbT ([B,T,Fu],
// or [T,B,Fu] when tm), and fs[b*T + t] = the sum of the (b, t) block (.x and .y alike), one CTA per (b, t)
int imp_section_input_launch(const float* magc, const float* fbT, int B, int T, int Fu, const SecGeom& g, float* X, float2* fs,
                             bool tm, cudaStream_t st);
// section rows [lo, hi) of Fu with sub-band / full-band centre widths cs / cf and neighbours ns / nf -> g, with the checks
// of imp_dims (FSN_ERR_SHAPE / FSN_ERR_UNSUPPORTED)
int sec_geom(int lo, int hi, int cs, int ns, int cf, int nf, int Fu, SecGeom& g);
// backward of section g's norm and full-band unfold (fsn_improved_train.cu): dfb [T,B,Fu] = (first ? 0 : dfb) + the
// gradient through the section input dX [T, B*N, W] with inv_s = invs [B], dot [B] (train_dot_launch), cnt = N W T;
// then act' of the kept full-band output y (FSN_ACT_NONE / FSN_ACT_RELU)
int imp_unfold_bwd_launch(const float* dX, const float* invs, const float* dot, float cnt, const SecGeom& g, int B, int T,
                          int Fu, bool first, int act, const float* y, float* dfb, cudaStream_t st);
// where section g's Linear(H -> 2c) writes in the cRM [B,2,F,T]
inline HeadGeom imp_head_geom(const SecGeom& g, int F, int T) { return HeadGeom{g.N, g.cs, g.lo, F, (size_t)T}; }

// persistent cooperative full-band LSTM (fsn_fullband.cu): layers L[0] (F -> H0, input x [R,Tp,F] times inv1[r] when
// given) and L[1] (H0 -> H1) of R rows into h1all [R,Tp,H1]; h0buf [2][256][H0] scratch.
// io (nullable, chunked streaming): per layer l, h_init / c_init [R, H_l] the state entering step 0 (null: zero; the c_init
// pair and the h_init pair are given or null together); h_fin / c_fin [R, H_l] receive the state after step fin_step
// (-1: none); restart [R] (nullable): row r's state after step restart[r] - 1 is zero, as at a sequence's first step
struct FbState {
  const float* h_init[2]; const float* c_init[2];
  float* h_fin[2]; float* c_fin[2];
  const int* restart;
  int fin_step;
};
bool fb_persistent_supported(int F, int H0, int H1);
int fb_persistent_launch(const fsn_lstm_layer* L, const float* x, const float* inv1, float* h0buf, float* h1all,
                         unsigned int* barrier, int R, int F, int H0, int H1, int Tp, cudaStream_t st,
                         const FbState* io = nullptr);

// tensor-core LSTM layer for a small batch of sequences (fsn_lstm_rec_tc.cu): hoisted input projection on the tf32
// GEMM (x3: three passes on tf32 hi/lo splits) + persistent cooperative wgmma recurrence (x3: fp16 hi/lo splits)
bool lstm_rec_tc_supported(int H, bool x3);
int lstm_rec_tc_rows_per_launch(int H);
size_t lstm_rec_tc_scratch_bytes(int H, bool x3);
// chunked streaming (lstm_rec_tc_carry_kernel): row r enters step 0 with h_init / c_init [r * row + u] and step
// restart[r] with zero state; c after step fin_step (-1: none) goes to c_fin (may be c_init)
struct RecCarry {
  const float *h_init, *c_init;
  float* c_fin;
  size_t row;
  const int* restart;
  int fin_step;
};
// what lstm_rec_tc_launch chose for a call (unit tests): rows per cooperative launch, TMA ring stages, launches, dynamic
// shared memory bytes per CTA
struct RecTcInfo {
  int rows_per_launch, stages, launches, smem_bytes;
};
int lstm_rec_tc_launch(const float* w_hh, const float* b_ih, const float* b_hh, const float* P, size_t p_row, size_t p_t,
                       float* hall, size_t h_row, size_t h_t, int R, int T, int H, bool x3, void* scratch,
                       cudaStream_t st, const RecCarry* io = nullptr, RecTcInfo* info = nullptr);
int split_tf32_launch(const float* in, size_t rows, int K, size_t ldi, const float* row_scale, int rows_per_scale,
                      float* out, int Kp, int cat, cudaStream_t st, int scale_B = 0);
int bias_act_launch(float* x, size_t rows, int N, size_t ld, const float* bias, int act, cudaStream_t st);
// workspace of lstm_layer_tc / linear_tc: prepared A operand [rows_T, Kmax (x3: 3 Kmax)], prepared weights
// [4 Hmax, same], hoisted projection P [rows_T, 4 Hmax], recurrence scratch
struct LstmTcWs { float *a, *w, *P; void* rec; };
void lstm_tc_carve(Carver& c, size_t rows_T, int Kmax, int Hmax, bool x3, LstmTcWs& ws);
int lstm_layer_tc(const fsn_lstm_layer& L, const float* x, size_t ldx, int K, const float* row_scale, int rows_per_scale,
                  int scale_B, int R, int T, int H, bool x3, const LstmTcWs& ws, float* hall, cudaStream_t st,
                  const RecCarry* io = nullptr);
int linear_tc(const float* x, size_t ldx, int K, const float* W, const float* bias, int N, int act, float* out, size_t ldo,
              size_t rows, bool x3, const LstmTcWs& ws, cudaStream_t st);
int gemm_tc_split_launch(const float* a, size_t lda, const float* W, int N, int K, float* w, float* C, size_t ldc, size_t M,
                         bool x3, cudaStream_t st);

// One SequenceModel of the inference forwards over clip-major rows (sequence_model.py:106-125, fsn_fullband.cu): n LSTM
// (or GRU) layers over x [R, Tp, K0] (contiguous; times scale[r], or scale[t*R + r] with step_scale), then Linear(H[n-1]
// -> O) + act into out [R*Tp, O].  tc / x3 are the caller's rule for running the stack on the tensor cores
// (lstm_layer_tc + linear_tc, x3: hi+lo compensated).  Otherwise, or under FSN_FB_STEPWISE / force_stepwise, layers 0-1
// run on the persistent kernel when it fits (LSTM, no per-step scale, not forced per-step), everything else on the
// per-step kernels, then fc_gemm.
static const int SEQ_MAX_LAYERS = 8;
struct SeqStack {
  int R, Tp, K0, n, O, act;
  int H[SEQ_MAX_LAYERS];
  fsn_lstm_layer L[SEQ_MAX_LAYERS];
  bool gru, step_scale, tc, x3;
  bool force_stepwise;  // the per-step kernels for every layer, as FSN_FB_STEPWISE (the unit-test hook sets it)
  const float *x, *scale, *fc_w, *fc_b;
  float* out;
};
// the path seq_stack_forward takes for a stack (values of fsn_debug_seq_stack's *path): tensor cores; layers 0-1 on the
// persistent kernel; layers 0-1 two per-step launches per step (lstm_step2_launch); one layer on the per-step kernel.
// Layers past the first two run the per-step kernel on every path but the tensor-core one.
enum SeqPath {
  SEQ_PATH_TC = FSN_SEQ_PATH_TC,
  SEQ_PATH_PERSISTENT = FSN_SEQ_PATH_PERSISTENT,
  SEQ_PATH_STEP2 = FSN_SEQ_PATH_STEP2,
  SEQ_PATH_ONE_LAYER = FSN_SEQ_PATH_ONE_LAYER
};
SeqPath seq_stack_path(const SeqStack& s);
// layer outputs for every step (hall[0]: top layer), per-step state, persistent-kernel scratch, tensor-core workspace
struct SeqStackWs {
  float *hall[2], *h0[2], *c0, *c1, *pp;
  unsigned int* barrier;
  LstmTcWs tc;
};
// sizes the state of every path the stack's shape, cell, scale and tc flag allow (only those fields are read); a stack
// no larger in any of K0, H[l], O (same R, Tp, n, flags) runs on the same workspace
void seq_stack_carve(Carver& c, const SeqStack& s, SeqStackWs& w);
int seq_stack_forward(const SeqStack& s, const SeqStackWs& w, cudaStream_t st);

// ---- chunked streaming (DESIGN 4.14).  Per (n_fft, hop, look_ahead): c = ceil((n/2) / hop) steps of framing lag (a
// step's frame and its pair partner are complete c hops before the chunk ends), the delay D = n/2 + (la + 1 + c) hop,
// Hs samples of history, Rc cRM frames and Q = Rc + la spectrum frames carried per slot, E extra steps on a clip's
// last call (its last frames, the look-ahead pad and the lag).
struct StreamGeom { int n, hop, la, c, D, Hs, Rc, Q, E; };
int stream_geom(int n_fft, int hop, int win_length, int la, StreamGeom& g);
// per-slot bookkeeping at the start of each slot's state block
struct StreamMeta { int pos, active; float acc; int pad; };
// host (start, tail) tables -> the call's device tables pos0 / act0 / tail (slot b: samples before the call, whether a
// clip is running, tail or -1), re-initialising the meta of slots that start; the tables travel in kernel parameters
int stream_prologue(const int32_t* start, const int32_t* tail, int B, char* state, size_t slot_bytes, int* pos0, int* act0,
                    int* tail_dev, cudaStream_t st);
// first norm of the causal norms over the call's S steps: scaleT [S, B] from the frame sums fs [B, S] and the carried
// accumulator (cumulative: running sum, forgetting: mu), frames counted from the clip start; the meta of active slots
// then advances by K steps (pos += K hop, accumulator after step K-1, inactive after a tail).  With fs2 (forgetting norm
// only): fullsubnet's second norm instead, mean (fs.y + fs2.y) / F (the caller passes F := F Ksb), mu carried at acc_off
// bytes into each block and reset at the clip's frame 0, the meta untouched
int stream_norm_launch(const float2* fs, int B, int S, int K, int F, const StreamGeom& g, int norm_type, const int* pos0,
                       const int* act0, const int* tail, char* state, size_t slot_bytes, float* scaleT, cudaStream_t st,
                       const float2* fs2 = nullptr, size_t acc_off = 0);
// fullsubnet's second cumulative norm over the call's S steps: scaleT [S, B*F] of row b*F + f from magT / fbT [B, S, F],
// the running sum of each row carried at run_off bytes into each block (F floats), reset at the clip's frame 0 and
// stored as of step K - 1 for the active slots
int stream_cum_unit_launch(const float* magT, const float* fbT, int B, int S, int K, int F, int Ns, int Nf,
                           const StreamGeom& g, const int* pos0, const int* act0, char* state, size_t slot_bytes,
                           size_t run_off, float* scaleT, cudaStream_t st);
// before step j: zero h [B rows h_row apart, H] and c [B, H] of the slots whose step j is their clip's frame 0
int stream_reset_launch(const int* pos0, int B, const StreamGeom& g, int j, int H, float* h, size_t h_row, float* c,
                        cudaStream_t st);
// restart[b] = the step of the call that is slot b's clip frame 0 (c - pos0[b] / hop; outside [0, c] when none is):
// the tensor-core stream's kernels enter it with zero state, where the per-step kernels run stream_reset_launch
int stream_restart_launch(const int* pos0, int B, const StreamGeom& g, int* restart, cudaStream_t st);
// signal layer of the streaming calls (fsn_dsp.cu), power-of-two n_fft only
int stream_dsp_check(int n_fft, int hop, int win_length);
int stft_stream_launch(const float* win, int Wn, int Hs, const int* pos0, const int* tail, int B, int n_fft, int hop,
                       int win_length, int c, int S, int Q, float* magT, float* spec, cudaStream_t st);
int istft_stream_launch(const float* spec, const float* crm, const int* pos0, const int* act0, const int* tail, int B,
                        int K, int D, int n_fft, int hop, int win_length, int c, int la, int Rc, int Q, int S, float* wav,
                        cudaStream_t st);
// An LSTM SequenceModel over a streaming call (R = B slots, Tp = the call's St steps, from the whole-clip call's builder)
// with each layer's (h, c) carried in the slot state, on the path seq_stack_path picks for the whole-clip stack, so a clip
// streams to the whole-clip bits.  TC: lstm_layer_tc with RecCarry, then linear_tc.  PERSISTENT: layers 0-1 on
// fb_persistent_launch with FbState.  Otherwise, and for layers past the second, one layer after the other on the
// per-step kernels, (h, c) zeroed before the step that is a clip's frame 0.  (h, c) after step K - 1 go back to the
// state.  Layer l's h / c are at the h / c byte offsets of each slot's block plus the floats of the layers below.
// restart (slot b's frame-0 step, stream_restart_launch) is read on the TC and persistent paths only: a stream whose
// stacks always have a per-step scale (fullband_baseline, fast_fullsubnet's encoder) never takes them and passes none.
struct StackCarry { char* state; size_t slot, h, c; const int* pos0; StreamGeom g; const int* restart; int K; };
// seq_stack_carve plus what only the carry needs: the per-step layers' output ping-pong and entering h (their c in
// seq.c0), the persistent kernel's (h, c) after step K - 1 (its entering state goes to seq.h0 / c0 / c1)
struct StreamStackWs { SeqStackWs seq; float* h; float *h_fin[2], *c_fin[2]; };
void stream_stack_carve(Carver& c, const SeqStack& s, StreamStackWs& w);
int stream_seq_stack(const SeqStack& s, const StreamStackWs& w, const StackCarry& io, cudaStream_t st);
// rows of `width` bytes: dst row b (pitch dp) <- src row b (pitch sp), B rows, on the stream
int copy_rows(void* dst, size_t dp, const void* src, size_t sp, size_t width, int B, cudaStream_t st);

// ---- the host skeleton of every model's streaming step.  Each step reads its descriptor / geometry check ->
// stream_check -> its own argument checks -> layout -> carve -> stream_check_sizes -> stream_open -> its own norms and
// stacks -> stream_close; its size queries are stream_query_check, then the layout or the carve.
// Slot state block: the meta, the sample history Hs, the spectrum Q x 2F and the cRM Rc x 2F, then the model's sections
// appended with sec; every section starts on 16 bytes and slot() closes the block on 256
struct StreamSlot {
  size_t hist, spec, crm, end;
  StreamSlot(const StreamGeom& g, int F);
  size_t sec(size_t floats) { const size_t at = end; end = align_up(end + floats * 4, 16); return at; }
  size_t slot() const { return align_up(end, 256); }
};
// the workspace every step starts with, laid out for K + E steps: stream_prologue's device tables, the samples
// [B, Hs + K hop], the magnitude [B, St, F], the spectrum [B, Q + St, 2F] and the cRM [B, Rc + St, 2F]
struct StreamWs {
  int *pos0, *act0, *tail;
  float *wav, *magT, *spec, *crm;
};
void stream_carve(Carver& c, const StreamGeom& g, int B, int K, int F, StreamWs& w);
// the state / workspace queries after the model's check rc: refuse B <= 0 or K_max <= 0 (FSN_ERR_SHAPE)
int stream_query_check(int rc, const char* who, int B, int K_max);
inline int stream_delay(int rc, const StreamGeom& g) { return rc ? -rc : g.D; }
// host checks of a call before any CUDA call and before its layout and carve: B, K > 0 (FSN_ERR_SHAPE), B <= 65535
// (FSN_ERR_UNSUPPORTED; the DSP kernels put the slot in gridDim.y), K hop + D < 2^30, non-null chunk and output, tail
// (host [B], nullable) -1 or in [0, K hop] (FSN_ERR_SHAPE).  St: the call's steps, K + E when a slot's clip ends in it,
// else K.  `who` prefixes the messages
int stream_check(const char* who, const StreamGeom& g, int B, int K, const int32_t* tail, const float* wav,
                 const float* enhanced, int& St);
// after the layout and carve: B blocks of `slot` bytes of state, then ws_need bytes of workspace (FSN_ERR_WORKSPACE)
int stream_check_sizes(const void* state, size_t state_bytes, size_t slot, int B, const void* workspace,
                       size_t workspace_bytes, size_t ws_need);
// signal front end: stream_prologue (with restart non-null, stream_restart_launch into it), the carried history and the
// chunk wav [B, K hop] into w.wav, the carried spectrum into w.spec, the STFT of the St steps into w.magT and w.spec
int stream_open(const StreamGeom& g, const StreamSlot& sl, const StreamWs& w, int F, int B, int K, int St, int win_length,
                const int32_t* start, const int32_t* tail, const float* wav, char* state, int* restart, cudaStream_t st);
// signal back end: the carried cRM into w.crm, then the model's output y [B, St, 2F] behind it (nullable: the model
// wrote w.crm itself), the iSTFT into enhanced and the carry of history, spectrum and cRM as of step K
int stream_close(const StreamGeom& g, const StreamSlot& sl, const StreamWs& w, int F, int B, int K, int St, int win_length,
                 const float* y, float* enhanced, char* state, cudaStream_t st);

// tensor-core sub-band stack (fsn_subband_tc.cu)
struct SbTcArgs {
  const void* packed;       // tile-ordered fp16 weights (fsn_pack_sb_weights / sb_tc_pack_raw)
  const float* magT; const float* fbT; const float* inv2;
  const float* unit_scale;  // nullable: per-row scale of this step (cumulative norm) instead of inv2[clip]
  float* crm;
  int B, F, Tp, la, Ns, Nf, H, act;
  int steps, shrink;      // LSTM steps (0 = Tp) and time down-sampling of the gathered input (0/1 = none)
  bool x3;                // error-compensated variant (FSN_PREC_F16X3_TC image)
  RowMap map;
  int stages, cluster;    // weight ring depth (2..4) and CTAs per cluster (1, 2, 4); 0 = FSN_TC_STAGES / FSN_TC_CLUSTER
  // non-null: run the cycle-stamp instantiation (fsn_debug_sb_lstm_tc_probe) for CTAs [0, stamp_ctas) and loop
  // iterations [0, stamp_its); the production launches leave it null
  long long* stamps;
  int stamp_ctas, stamp_its;
  // non-null (and no stamps): the two-pass path (sb_l0_tc_kernel, sb_l1_tc_kernel), h0 of split_chunk pairs at a time
  // (0: the default chunk) through this buffer of sb_tc_split_ws_bytes
  void* h0ws;
  int split_chunk;
};
size_t sb_tc_split_ws_bytes(int R, int Tp, int H, bool x3, int chunk_pairs = 0);
size_t sb_tc_packed_bytes(const fsn_model_desc* d);
// proj: the image sb_proj_forward streams (W_hh0, W_ih1, W_hh1 and layer 1's biases; no W_ih0 and no Linear)
size_t sb_tc_packed_bytes_raw(int H, bool x3, bool proj = false);
int sb_tc_pack(const fsn_model_desc* d, const fsn_seq_weights* sb, void* packed, cudaStream_t st);
// weights of a 2-layer stack of hidden size H over Ksb inputs with a Linear(H -> fc_out <= 2) on top; proj: the
// sb_proj_forward image (w_ih[0], fc_w and fc_b are not read, Ksb and fc_out are ignored)
int sb_tc_pack_raw(const fsn_seq_weights* sb, int H, int Ksb, int fc_out, void* packed, cudaStream_t st, bool x3,
                   bool proj = false);
int sb_tc_forward(const SbTcArgs& a, cudaStream_t st);
// chunked streaming (sb_carry_lstm_tc_kernel): the stack continued from a carried state.  (h, c) of row r, layer l, unit u
// at h / c [(r / rps) slot + l layer + (r % rps) H + u] (floats) are read before step 0 and written after store_step;
// row r enters step restart[r / rps] with zero state; step t's output o of row r = b F + f goes to crm[b crm_bs +
// (crm_t0 + t) 2F + o F + f].  a: unit_scale given, la = 0, no drop_band, no down-sampling.
// store_at non-null: the block-phased instantiation (sb_phased_lstm_tc_kernel, fast_fullsubnet's stream): step t's input
// of row r is x [(t R + r) Ksb + k], already down-sampled and scaled (a.unit_scale unused), and row r's state is stored
// after step store_at[r / rps] (store_step unused)
struct SbCarry {
  float *h, *c;
  size_t slot, layer;
  int rps;
  const int* restart;
  int store_step;
  size_t crm_bs;
  int crm_t0;
  const float* x;
  const int* store_at;
};
int sb_tc_carry_forward(const SbTcArgs& a, const SbCarry& io, cudaStream_t st);
bool sb_tc_supported(const fsn_model_desc* d);
// FSN_TC_STAGES / FSN_TC_CLUSTER (defaults 4 / 1), read once
void sb_tc_ring_defaults(int& stages, int& cluster);
// the same kernel with a precomputed layer-0 input (sb_proj_lstm_tc_kernel): R independent rows over T steps,
// P [T, R, 4H] = x W_ih0^T + b_ih0 + b_hh0 (fp32) -> h1 [T, R, H] (fp32), layer 1's hidden state of every step
struct SbProjArgs {
  const void* packed;       // sb_tc_pack_raw(..., proj = true) image
  const float* P;
  float* h1;
  int R, T, H;
  bool x3;
  int stages, cluster;      // 0 = FSN_TC_STAGES / FSN_TC_CLUSTER
};
int sb_proj_forward(const SbProjArgs& a, cudaStream_t st);
// improved_fullsubnet's section recurrence on the f16 precisions (fsn_improved.cu): P = (X W_ih0^T + b_ih0) + b_hh0 on the
// tf32 GEMM (x3: compensated) over X [T, R, W], then sb_proj_forward into h1 [T, R, H].  ws: imp_section_tc_carve.
struct ImpSecTcWs { LstmTcWs gemm; float *P, *h1; };
void imp_section_tc_carve(Carver& c, size_t rows_T, int Wmax, int H, bool x3, ImpSecTcWs& w);
int imp_section_lstm_tc(const fsn_seq_weights& sw, const void* packed, const float* X, int R, int T, int W, int H, bool x3,
                        const ImpSecTcWs& w, cudaStream_t st, int stages = 0, int cluster = 0);

}  // namespace fsn
