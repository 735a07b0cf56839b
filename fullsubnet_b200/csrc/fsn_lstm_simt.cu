// fp32 (FMA) kernels of the model path: layout/statistics prep, one LSTM time step as a tiled
// GEMM with the cell update fused in the epilogue, and the output Linear layers.
//
// Reference semantics:
//   audio_zen/model/module/sequence_model.py:106-125 (nn.LSTM + Linear + activation)
//   audio_zen/model/base_model.py:13-46 (freq_unfold), :203-218 (offline_laplace_norm)
//   recipes/dns_interspeech_2020/fullsubnet/model.py:85-135
//   audio_zen/acoustics/feature.py:309-345 (drop_band as a row map)
#include "fsn_internal.cuh"

namespace fsn {

// ------------------------------------------------------------------------------------------
// [B,F,T] -> [B,T_pad,F], rows T..T_pad-1 zero (model.py:85 look-ahead pad fused)
__global__ void transpose_mag_kernel(const float* __restrict__ in, float* __restrict__ out, int F, int T, int T_pad) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int f = f0 + i, t = t0 + tx;
    tile[i][tx] = (f < F && t < T) ? in[((size_t)b * F + f) * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, f = f0 + tx;
    if (t < T_pad && f < F) out[((size_t)b * T_pad + t) * F + f] = tile[tx][i];
  }
}


// one warp per (b,t) row of a time-major [B,T_pad,F] tensor: fs[row] = (sum_f x, sum_f c_N[f] x)
__global__ void frame_stats_kernel(const float* __restrict__ x, int rows, int F, int N, float2* __restrict__ fs) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* p = x + (size_t)row * F;
  float s0 = 0.f, s1 = 0.f;
  for (int f = lane; f < F; f += 32) {
    const float v = p[f];
    s0 += v;
    s1 += v * (float)reflect_count(f, F, N);
  }
  s0 = warp_sum(s0);
  s1 = warp_sum(s1);
  if (lane == 0) fs[row] = make_float2(s0, s1);
}

// one CTA per clip: fixed-order tree sum over its T_pad frame partials (deterministic); lens (nullable): only the
// clip's own 1 + lens[b]/hop + la frames
__global__ void clip_reduce_kernel(const float2* __restrict__ fs, int T_pad, float2* __restrict__ sums,
                                   const int* __restrict__ lens, int hop, int la) {
  __shared__ float2 sh[256];
  const int b = blockIdx.x;
  const int Tn = lens ? 1 + lens[b] / hop + la : T_pad;
  float2 a = make_float2(0.f, 0.f);
  for (int t = threadIdx.x; t < Tn; t += 256) {
    const float2 v = fs[(size_t)b * T_pad + t];
    a.x += v.x; a.y += v.y;
  }
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) { sh[threadIdx.x].x += sh[threadIdx.x + s].x; sh[threadIdx.x].y += sh[threadIdx.x + s].y; }
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[b] = sh[0];
}

// inv1[b] = 1/(mean(mag_pad)+1e-5)              (model.py:92)
// inv2[b] = 1/(mean(cat(unfold(mag), unfold(fb)))+1e-5) via the closed form   (model.py:110-111)
// lens (nullable): cnt1 / cnt2 are per frame, times the clip's 1 + lens[b]/hop + la frames (the float product the host
// forms for a call on that clip alone)
__global__ void norm_scales_kernel(const float2* __restrict__ mag_sums, const float2* __restrict__ fb_sums, int B,
                                   float cnt1, float cnt2, float* __restrict__ inv1, float* __restrict__ inv2, float eps,
                                   const int* __restrict__ lens, int hop, int la) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (lens) {
    const float tp = (float)(1 + lens[b] / hop + la);
    cnt1 = __fmul_rn(cnt1, tp);
    cnt2 = __fmul_rn(cnt2, tp);
  }
  if (inv1) inv1[b] = 1.0f / (mag_sums[b].x / cnt1 + eps);
  if (inv2) inv2[b] = 1.0f / ((mag_sums[b].y + fb_sums[b].y) / cnt2 + eps);
}

// ------------------------------------------------------------------------------------------
// One LSTM time step for R rows:  gates = [x_t | h_{t-1}] [W_ih | W_hh]^T + b_ih + b_hh, cell
// update fused.  CTA tile: 64 rows x 32 hidden units (x4 gates), K chunks of 16.
// GRU variant (p.gru; nn.GRU of audio_zen/model/module/sequence_model.py:59-66): the four accumulator slots hold
// r = W_ir x + W_hr h, z = W_iz x + W_hz h, n_x = W_in x and n_h = W_hn h (kept apart because n = tanh(n_x + b_in +
// r * (n_h + b_hn))); h' = (1 - z) n + z h.
constexpr int BM = 64, BU = 32, BK = 16;

template <int MODE>
__device__ __forceinline__ float load_seg0(const StepParams& p, int row, int k, int src_b, int src_f) {
  if (MODE == SEG0_DENSE) {
    const float v = p.x0[(size_t)row * p.x0_row_stride + k];
    return p.row_scale ? v * p.row_scale[p.row_scale_div > 1 ? row / p.row_scale_div : row] : v;
  } else {
    const int nmag = 2 * p.Ns + 1;
    const size_t base = ((size_t)src_b * p.Tp + p.t) * p.F;
    float v;
    if (k < nmag) v = p.magT[base + reflect_idx(src_f + k - p.Ns, p.F)];
    else          v = p.fbT[base + reflect_idx(src_f + (k - nmag) - p.Nf, p.F)];
    return v * (p.unit_scale ? p.unit_scale[row] : p.inv2[src_b]);
  }
}

template <int MODE>
__global__ void __launch_bounds__(256) lstm_step_kernel(const StepParams p) {
  __shared__ __align__(16) float As[BK][BM];
  __shared__ float Ws[BK][4 * BU + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int row0 = blockIdx.x * BM;
  const int u0 = blockIdx.y * BU;
  const int Ktot = p.K0 + (p.first ? 0 : p.H);

  // A-tile loader: thread -> (row = tid/4, 4 consecutive k)
  const int a_row = tid >> 2, a_k = (tid & 3) * 4;
  const int arow_g = row0 + a_row;
  int src_b = 0, src_f = 0;
  if (MODE == SEG0_GATHER && arow_g < p.R) row_to_unit(p.map, arow_g, src_b, src_f);
  // W-tile loader: thread -> (gate column = tid/2, 8 consecutive k)
  const int w_col = tid >> 1, w_k = (tid & 1) * 8;
  const int w_unit = u0 + (w_col & (BU - 1));
  const int w_slot = w_col / BU;                                    // accumulator slot 0..3
  const int w_gate = p.gru ? (w_slot < 2 ? w_slot : 2) : w_slot;    // gate block of the PyTorch weight
  const int w_row = w_gate * p.H + w_unit;  // row of the [4H,K] (GRU: [3H,K]) PyTorch weight
  const bool w_ok = w_unit < p.H;
  const bool w_x_ok = !(p.gru && w_slot == 3), w_h_ok = !(p.gru && w_slot == 2);  // GRU: n_x has no h part, n_h no x part

  float acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int g = 0; g < 4; ++g) acc[i][g][0] = acc[i][g][1] = 0.f;

  for (int k0 = 0; k0 < Ktot; k0 += BK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + a_k + j;
      float v = 0.f;
      if (arow_g < p.R && k < Ktot) {
        if (k < p.K0) v = load_seg0<MODE>(p, arow_g, k, src_b, src_f);
        else          v = p.h_prev[(size_t)arow_g * p.h_prev_stride + (k - p.K0)];
      }
      As[a_k + j][a_row] = v;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + w_k + j;
      float v = 0.f;
      if (w_ok && k < Ktot)
        v = (k < p.K0) ? (w_x_ok ? p.w_ih[(size_t)w_row * p.K0 + k] : 0.f)
                       : (w_h_ok ? p.w_hh[(size_t)w_row * p.H + (k - p.K0)] : 0.f);
      Ws[w_k + j][w_col] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const float w0 = Ws[kk][g * BU + tx];
        const float w1 = Ws[kk][g * BU + tx + 16];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[i][g][0] = fmaf(a[i], w0, acc[i][g][0]);
          acc[i][g][1] = fmaf(a[i], w1, acc[i][g][1]);
        }
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int u = u0 + tx + 16 * q;
    if (u >= p.H) continue;
    if (p.gru) {
      const float b_r = p.b_ih[u] + p.b_hh[u], b_z = p.b_ih[p.H + u] + p.b_hh[p.H + u];
      const float b_in = p.b_ih[2 * p.H + u], b_hn = p.b_hh[2 * p.H + u];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = row0 + ty * 4 + i;
        if (row >= p.R) continue;
        const float r = sigmoidf_(acc[i][0][q] + b_r), z = sigmoidf_(acc[i][1][q] + b_z);
        const float n = tanhf(acc[i][2][q] + b_in + r * (acc[i][3][q] + b_hn));
        const float hp = p.first ? 0.f : p.h_prev[(size_t)row * p.h_prev_stride + u];
        p.h_out[(size_t)row * p.h_out_stride + u] = (1.0f - z) * n + z * hp;
      }
      continue;
    }
    float bias[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) bias[g] = p.b_ih[g * p.H + u] + p.b_hh[g * p.H + u];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = row0 + ty * 4 + i;
      if (row >= p.R) continue;
      const float gi = acc[i][0][q] + bias[0];
      const float gf = acc[i][1][q] + bias[1];
      const float gg = acc[i][2][q] + bias[2];
      const float go = acc[i][3][q] + bias[3];
      const size_t ci = (size_t)row * p.H + u;
      const float c_prev = p.first ? 0.f : (p.c_in ? p.c_in[ci] : p.c[ci]);
      const float si = sigmoidf_(gi), sf = sigmoidf_(gf), tg = tanhf(gg), so = sigmoidf_(go);
      const float c = sf * c_prev + si * tg;
      p.c[ci] = c;
      p.h_out[(size_t)row * p.h_out_stride + u] = so * tanhf(c);
      if (p.save_gates) {
        float* gp = p.save_gates + (size_t)row * 4 * p.H + u;
        gp[0] = si; gp[p.H] = sf; gp[2 * p.H] = tg; gp[3 * p.H] = so;
      }
    }
  }
}

// ---- cumulative_laplace_norm (base_model.py:220-251): one thread per clip / per sub-band unit, sequential in time
__global__ void cum_clip_scale_kernel(const float2* __restrict__ fs, int B, int Tp, int F, float eps,
                                      float* __restrict__ scale1T) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float run = 0.f;
  for (int t = 0; t < Tp; ++t) {
    run += fs[(size_t)b * Tp + t].x;
    scale1T[(size_t)t * B + b] = 1.0f / (run / ((float)F * (float)(t + 1)) + eps);
  }
}

// mag / fb element (b, t, f) at b*bs + t*ts + f: clip-major [B,Tp,F] (inference) or time-major [Tp,B,F] (training)
__global__ void cum_unit_scale_kernel(const float* __restrict__ magT, const float* __restrict__ fbT, RowMap map, int R,
                                      int Tp, int Ns, int Nf, float eps, float* __restrict__ scaleT, size_t bs, size_t ts) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  int b, f;
  row_to_unit(map, r, b, f);
  const int K = 2 * Ns + 1 + 2 * Nf + 1;
  float run = 0.f;
  for (int t = 0; t < Tp; ++t) {
    const size_t base = (size_t)b * bs + (size_t)t * ts;
    float s = 0.f;
    for (int k = -Ns; k <= Ns; ++k) s += magT[base + reflect_idx(f + k, map.F)];
    for (int k = -Nf; k <= Nf; ++k) s += fbT[base + reflect_idx(f + k, map.F)];
    run += s;
    scaleT[(size_t)t * R + r] = 1.0f / (run / ((float)K * (float)(t + 1)) + eps);
  }
}

int cum_clip_scale_launch(const float2* fs, int B, int Tp, int F, float eps, float* scale1T, cudaStream_t st) {
  cum_clip_scale_kernel<<<cdiv(B, 64), 64, 0, st>>>(fs, B, Tp, F, eps, scale1T);
  FSN_CHECK_LAUNCH("cum_clip_scale_kernel");
  return FSN_OK;
}

int cum_unit_scale_launch(const float* magT, const float* fbT, RowMap map, int R, int Tp, int Ns, int Nf, float eps,
                          float* scaleT, cudaStream_t st, bool time_major) {
  const size_t bs = time_major ? (size_t)map.F : (size_t)Tp * map.F, ts = time_major ? (size_t)map.B * map.F : (size_t)map.F;
  cum_unit_scale_kernel<<<cdiv(R, 128), 128, 0, st>>>(magT, fbT, map, R, Tp, Ns, Nf, eps, scaleT, bs, ts);
  FSN_CHECK_LAUNCH("cum_unit_scale_kernel");
  return FSN_OK;
}

int lstm_step_launch(const StepParams& p, int mode, cudaStream_t st) {
  dim3 grid(cdiv(p.R, BM), cdiv(p.H, BU));
  if (mode == SEG0_DENSE) lstm_step_kernel<SEG0_DENSE><<<grid, 256, 0, st>>>(p);
  else                    lstm_step_kernel<SEG0_GATHER><<<grid, 256, 0, st>>>(p);
  FSN_CHECK_LAUNCH("lstm_step_kernel");
  return FSN_OK;
}

int lstm_step2_launch(StepParams p, int mode, int t, const fsn_lstm_layer& w1, const Step2State& s, cudaStream_t st) {
  const int H0 = p.H;
  p.first = (t == 0);
  p.h_prev = s.h0[(t + 1) & 1]; p.h_prev_stride = H0;
  p.h_out = s.h0[t & 1]; p.h_out_stride = H0;
  p.c = s.c0;
  int rc = lstm_step_launch(p, mode, st);
  if (rc) return rc;
  p.K0 = H0; p.H = s.H1;
  p.w_ih = w1.w_ih; p.w_hh = w1.w_hh; p.b_ih = w1.b_ih; p.b_hh = w1.b_hh;
  p.x0 = s.h0[t & 1]; p.x0_row_stride = H0; p.row_scale = nullptr; p.row_scale_div = 0;
  p.h_prev = s.h1_at(t - 1); p.h_out = s.h1_at(t); p.h_prev_stride = p.h_out_stride = s.h1_stride();
  p.c = s.c1;
  return lstm_step_launch(p, SEG0_DENSE, st);
}

// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case FSN_ACT_RELU: return fmaxf(v, 0.f);
    case FSN_ACT_TANH: return tanhf(v);
    case FSN_ACT_RELU6: return fminf(fmaxf(v, 0.f), 6.f);
    default: return v;
  }
}

// out[M,O] = act(A[M,K] W[O,K]^T + b)   (full-band Linear + ReLU over all (b,t) rows at once)
__global__ void __launch_bounds__(256)
fc_gemm_kernel(const float* __restrict__ A, const float* __restrict__ W, const float* __restrict__ bias,
               float* __restrict__ out, int M, int K, int O, int act, int w_kmajor) {
  __shared__ __align__(16) float As[16][64];
  __shared__ float Ws[16][64 + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int row0 = blockIdx.x * 64, o0 = blockIdx.y * 64;
  const int l_row = tid >> 2, l_k = (tid & 3) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + l_k + j;
      As[l_k + j][l_row] = (row0 + l_row < M && k < K) ? A[(size_t)(row0 + l_row) * K + k] : 0.f;
      Ws[l_k + j][l_row] = (o0 + l_row < O && k < K) ? (w_kmajor ? W[(size_t)k * O + o0 + l_row] : W[(size_t)(o0 + l_row) * K + k]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float w = Ws[kk][tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i][j] = fmaf(a[i], w, acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = row0 + ty * 4 + i;
    if (row >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = o0 + tx + 16 * j;
      if (o < O) out[(size_t)row * O + o] = apply_act(acc[i][j] + (bias ? bias[o] : 0.f), act);
    }
  }
}

int fc_gemm_launch(const float* A, const float* W, const float* bias, float* out, int M, int K, int O, int act,
                   cudaStream_t st, bool w_kmajor) {
  dim3 grid(cdiv(M, 64), cdiv(O, 64));
  fc_gemm_kernel<<<grid, 256, 0, st>>>(A, W, bias, out, M, K, O, act, w_kmajor ? 1 : 0);
  FSN_CHECK_LAUNCH("fc_gemm_kernel");
  return FSN_OK;
}

// sub-band Linear(H -> O, O small) for one time step, one warp per row, written straight into
// crm[b', o, f', t_out] (model.py:129-135: reshape/permute + look-ahead slice fused)
__global__ void sb_fc_step_kernel(const float* __restrict__ h, int R, int H, const float* __restrict__ W,
                                  const float* __restrict__ bias, int O, int act, float* __restrict__ crm, int Fsub,
                                  int T_out, int t_out, size_t step_stride) {
  // blockIdx.y: step (h of step y starts step_stride floats further and lands in frame t_out + y)
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= R) return;
  t_out += blockIdx.y;
  const float* hp = h + (size_t)blockIdx.y * step_stride + (size_t)row * H;
  const int bq = row / Fsub, fq = row - bq * Fsub;
  for (int o = 0; o < O; ++o) {
    float s = 0.f;
    for (int k = lane; k < H; k += 32) s = fmaf(hp[k], W[(size_t)o * H + k], s);
    s = warp_sum(s);
    if (lane == 0) crm[(((size_t)bq * O + o) * Fsub + fq) * T_out + t_out] = apply_act(s + bias[o], act);
  }
}

__global__ void rows_fc_kernel(const float* __restrict__ h, int R, int H, const float* __restrict__ W,
                               const float* __restrict__ bias, int O, int act, float* __restrict__ out, size_t row_stride,
                               size_t o_stride) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= R) return;
  const float* hp = h + (size_t)row * H;
  for (int o = 0; o < O; ++o) {
    float s = 0.f;
    for (int k = lane; k < H; k += 32) s = fmaf(hp[k], W[(size_t)o * H + k], s);
    s = warp_sum(s);
    if (lane == 0) out[(size_t)row * row_stride + (size_t)o * o_stride] = apply_act(s + bias[o], act);
  }
}

int rows_fc_launch(const float* h, int R, int H, const float* W, const float* bias, int O, int act, float* out,
                   size_t row_stride, size_t o_stride, cudaStream_t st) {
  rows_fc_kernel<<<cdiv(R, 8), 256, 0, st>>>(h, R, H, W, bias, O, act, out, row_stride, o_stride);
  FSN_CHECK_LAUNCH("rows_fc_kernel");
  return FSN_OK;
}

int sb_fc_step_launch(const float* h, int R, int H, const float* W, const float* bias, int O, int act, float* crm,
                      int Fsub, int T_out, int t_out, cudaStream_t st) {
  sb_fc_step_kernel<<<cdiv(R, 8), 256, 0, st>>>(h, R, H, W, bias, O, act, crm, Fsub, T_out, t_out, 0);
  FSN_CHECK_LAUNCH("sb_fc_step_kernel");
  return FSN_OK;
}

// the same Linear for `steps` consecutive steps of a time-major [steps, R, H] block in one launch (training forward)
int sb_fc_steps_launch(const float* h, int R, int H, int steps, const float* W, const float* bias, int O, int act, float* crm,
                       int Fsub, int T_out, int t_out0, cudaStream_t st) {
  if (steps <= 0) return FSN_OK;
  FSN_REQUIRE(steps <= 65535, FSN_ERR_SHAPE, "sb_fc_steps: too many steps");
  sb_fc_step_kernel<<<dim3(cdiv(R, 8), steps), 256, 0, st>>>(h, R, H, W, bias, O, act, crm, Fsub, T_out, t_out0, (size_t)R * H);
  FSN_CHECK_LAUNCH("sb_fc_step_kernel");
  return FSN_OK;
}

int transpose_mag_launch(const float* in, float* out, int B, int F, int T, int T_pad, cudaStream_t st) {
  dim3 grid(cdiv(T_pad, 32), cdiv(F, 32), B);
  transpose_mag_kernel<<<grid, dim3(32, 8), 0, st>>>(in, out, F, T, T_pad);
  FSN_CHECK_LAUNCH("transpose_mag_kernel");
  return FSN_OK;
}

int clip_stats_launch(const float* x, int B, int T_pad, int F, int N, float2* fs, float2* sums, cudaStream_t st,
                      const int* lens, int hop, int la) {
  const int rows = B * T_pad;
  frame_stats_kernel<<<cdiv(rows, 8), 256, 0, st>>>(x, rows, F, N, fs);
  FSN_CHECK_LAUNCH("frame_stats_kernel");
  clip_reduce_kernel<<<B, 256, 0, st>>>(fs, T_pad, sums, lens, hop, la);
  FSN_CHECK_LAUNCH("clip_reduce_kernel");
  return FSN_OK;
}

int clip_reduce_only_launch(const float2* fs, int B, int T_pad, float2* sums, cudaStream_t st, const int* lens, int hop,
                            int la) {
  clip_reduce_kernel<<<B, 256, 0, st>>>(fs, T_pad, sums, lens, hop, la);
  FSN_CHECK_LAUNCH("clip_reduce_kernel");
  return FSN_OK;
}

int norm_scales_launch(const float2* mag_sums, const float2* fb_sums, int B, float cnt1, float cnt2, float* inv1,
                       float* inv2, cudaStream_t st, float eps, const int* lens, int hop, int la) {
  norm_scales_kernel<<<cdiv(B, 128), 128, 0, st>>>(mag_sums, fb_sums, B, cnt1, cnt2, inv1, inv2, eps, lens, hop, la);
  FSN_CHECK_LAUNCH("norm_scales_kernel");
  return FSN_OK;
}

}  // namespace fsn
