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

// ------------------------------------------------------------------------------------------ layout
// Clip-major inference tensors ([B, Tp, .]) and time-major training ones ([Tp, B, .]) share these kernels: each takes
// the element strides of its (clip, frame) axes.

// [B,F,T] -> out (b,t,f) at b*bs + t*ts + f, frames T..Tp-1 zero (model.py:85 look-ahead pad fused); scaled (nullable)
// = the same times scale[b] (model.py:92)
__global__ void transpose_mag_kernel(const float* __restrict__ in, int F, int T, int Tp, size_t bs, size_t ts,
                                     float* __restrict__ out, const float* __restrict__ scale, float* __restrict__ scaled) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int f = f0 + i, t = t0 + tx;
    tile[i][tx] = (f < F && t < T) ? in[((size_t)b * F + f) * T + t] : 0.f;
  }
  __syncthreads();
  const float s = scaled ? scale[b] : 0.f;
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, f = f0 + tx;
    if (t < Tp && f < F) {
      const float v = tile[tx][i];
      const size_t o = (size_t)b * bs + (size_t)t * ts + f;
      out[o] = v;
      if (scaled) scaled[o] = v * s;
    }
  }
}

// y rows (b,t) of 2F at b*bs + t*ts (channel c*F+f) -> out [B,2,F,T], T = Tp - la, dropping the first `la` frames
// (fullsubnet/model.py:129-135, fast_fullsubnet/model.py:197-200, fullband_baseline/model.py:58-62)
__global__ void crm_output_kernel(const float* __restrict__ y, size_t bs, size_t ts, int Tp, int F, int la,
                                  float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int T = Tp - la;
  const int b = blockIdx.z >> 1, c = blockIdx.z & 1;
  const int f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += 8) {  // read: f contiguous
    const int t = t0 + i, f = f0 + tx;
    tile[i][tx] = (t < T && f < F) ? y[(size_t)b * bs + (size_t)(t + la) * ts + c * F + f] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {  // write: t contiguous
    const int f = f0 + i, t = t0 + tx;
    if (f < F && t < T) out[(((size_t)b * 2 + c) * F + f) * T + t] = tile[tx][i];
  }
}

// One CTA per (b, ts); see fast_bn_input_launch
__global__ void fast_bn_input_kernel(const float* __restrict__ melT, const float* __restrict__ encT, size_t bs, size_t ts_,
                                     int B, int Tp, int M, int Nn, int Ne, int S, int Ts, float* __restrict__ bn,
                                     float2* __restrict__ fs) {
  __shared__ float red[256];
  const int b = blockIdx.x / Ts, ts = blockIdx.x % Ts;
  const int K = (2 * Nn + 1) + (2 * Ne + 1);
  int t0, len;
  shrink_block(ts, S, Tp, t0, len);
  const float inv = 1.0f / (float)len;
  float local = 0.f;
  for (int i = threadIdx.x; i < M * K; i += blockDim.x) {
    const int m = i / K, k = i - m * K;
    float acc = 0.f;
    for (int t = t0; t < t0 + len; ++t) {
      const size_t base = (size_t)b * bs + (size_t)t * ts_;
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

// see fast_dec_input_launch; element i of dec_in is column i % 2M of row i / 2M
__global__ void fast_dec_input_kernel(const float* __restrict__ encT, const float* __restrict__ bn_out, size_t nbs,
                                      size_t nms, size_t nts, int B, int Tp, int M, int S, int Ts, size_t rbs, size_t rts,
                                      float* __restrict__ dec_in) {
  const size_t n = (size_t)B * Tp * 2 * M;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % (2 * M));
    const size_t q = i / (2 * M);
    const int b = (int)((q / rbs) % B), t = (int)((q / rts) % Tp);
    dec_in[i] = c < M ? encT[q * M + c] : bn_out[(size_t)b * nbs + (size_t)(c - M) * nms + (size_t)min(t / S, Ts - 1) * nts];
  }
}

__global__ void scale_rows_kernel(const float* in, const float* __restrict__ scale, size_t n, int cols, int rows, int div,
                                  float* out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = in[i] * scale[(int)((i / cols) % rows) / div];
}

// one warp per frame (b,t) of x, element (b,t,f) at b*bs + t*ts + f: fs[b*Tp + t] = (sum_f x, sum_f c_N[f] x)
__global__ void frame_stats_kernel(const float* __restrict__ x, int B, int Tp, int F, int N, size_t bs, size_t ts,
                                   float2* __restrict__ fs) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B * Tp) return;
  const int b = row / Tp, t = row - b * Tp;
  const float* p = x + (size_t)b * bs + (size_t)t * ts;
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
    run += unit_frame_sum(magT + base, fbT + base, f, map.F, Ns, Nf);
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

// ---- forgetting_norm (base_model.py:102-151): the reference's per-frame loop in float32, one thread per clip
ForgetCoef forget_coef() {
  ForgetCoef c;
  const double alpha = (double)(FORGET_LEN - 1) / (double)(FORGET_LEN + 1);
  const float alpha32 = (float)alpha;
  for (int t = 0; t < FORGET_LEN; ++t) {
    // alp = torch.min(torch.tensor([(t-1)/(t+1), alpha])): both rounded to float32 first; 1 - alp in float32
    const float r = (float)((double)(t - 1) / (double)(t + 1));
    const float a = r < alpha32 ? r : alpha32;
    c.a[t] = a;
    c.b[t] = 1.0f - a;
  }
  c.a[FORGET_LEN] = alpha32;            // alpha * mu: the double applied to a float32 tensor
  c.b[FORGET_LEN] = (float)(1.0 - alpha);  // (1 - alpha) evaluated in double, then applied
  return c;
}

__global__ void forget_scale_kernel(const float2* __restrict__ fs, const float2* __restrict__ fs2, int B, int Tp, float cnt,
                                    const ForgetCoef c, float* __restrict__ scaleT, float* __restrict__ muT,
                                    const int* __restrict__ lens, int hop, int la) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int Tb = lens ? min(Tp, 1 + lens[b] / hop + la) : Tp;
  float mu = 0.f;
  for (int t = 0; t < Tb; ++t) {
    const float2 v = fs[(size_t)b * Tp + t];
    const float s = fs2 ? __fadd_rn(v.y, fs2[(size_t)b * Tp + t].y) : v.x;
    const float m = __fdiv_rn(s, cnt);  // torch.mean: sum / count
    const int i = t < FORGET_LEN ? t : FORGET_LEN;
    mu = __fadd_rn(__fmul_rn(c.a[i], mu), __fmul_rn(c.b[i], m));
    if (muT) muT[(size_t)t * B + b] = mu;
    scaleT[(size_t)t * B + b] = __fdiv_rn(1.0f, __fadd_rn(mu, FORGET_EPS));
  }
}

__global__ void forget_unit_broadcast_kernel(const float* __restrict__ scaleT, RowMap map, int R, int Tp,
                                             float* __restrict__ unit_scale) {
  const size_t n = (size_t)Tp * R;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i % R), t = (int)(i / R);
    int b, f;
    row_to_unit(map, r, b, f);
    unit_scale[i] = scaleT[(size_t)t * map.B + b];
  }
}

int forget_scale_launch(const float2* fs, const float2* fs2, int B, int Tp, float cnt, float* scaleT, float* muT,
                        cudaStream_t st, const int* lens, int hop, int la) {
  forget_scale_kernel<<<cdiv(B, 64), 64, 0, st>>>(fs, fs2, B, Tp, cnt, forget_coef(), scaleT, muT, lens, hop, la);
  FSN_CHECK_LAUNCH("forget_scale_kernel");
  return FSN_OK;
}

int forget_unit_broadcast_launch(const float* scaleT, RowMap map, int R, int Tp, float* unit_scale, cudaStream_t st) {
  forget_unit_broadcast_kernel<<<ew_grid((size_t)Tp * R), 256, 0, st>>>(scaleT, map, R, Tp, unit_scale);
  FSN_CHECK_LAUNCH("forget_unit_broadcast_kernel");
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
  p.first = t == 0 && !s.carry;
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

// sub-band head Linear(H -> O <= 2c) of `steps` frames, one warp per (step, row, output), written straight into the
// cRM through g (model.py:129-135: reshape/permute + look-ahead slice fused).  The activation is a template argument: with
// a runtime switch these short warps took 4.6 % longer on the improved_fullsubnet heads (H100 SXM, 700 W)
template <int ACT>
__global__ void sb_head_kernel(const float* __restrict__ h, int R, int H, int steps, const float* __restrict__ W,
                               const float* __restrict__ bias, int O, float* __restrict__ out, HeadGeom g, int t0) {
  const size_t wid = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= (size_t)steps * R * O) return;
  const size_t step_row = wid / O;
  const int o = (int)(wid % O), t = t0 + (int)(step_row / R), row = (int)(step_row % R);
  const float* hp = h + step_row * H;
  float s = 0.f;
  for (int k = lane; k < H; k += 32) s = fmaf(hp[k], W[(size_t)o * H + k], s);
  s = warp_sum(s);
  if (lane == 0) out[head_index(g, row, o, t)] = apply_act(s + bias[o], ACT);
}

// the inverse gather of sb_head_kernel's scatter: dY[t, r, o] = act'(y) dcrm at frame t - la, 0 for t < la
__global__ void sb_head_bwd_kernel(const float* __restrict__ dcrm, const float* __restrict__ y, int act, int R, int O,
                                   int steps, int la, HeadGeom g, float* __restrict__ dY) {
  const size_t n = (size_t)steps * R * O;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int o = (int)(i % O);
    const size_t tr = i / O;
    const int r = (int)(tr % R), t = (int)(tr / R);
    float v = 0.f;
    if (t >= la) {
      const size_t idx = head_index(g, r, o, t - la);
      v = act_grad(dcrm[idx], y, idx, act);
    }
    dY[i] = v;
  }
}

int sb_head_launch(const float* h, int R, int H, int steps, const float* W, const float* bias, int O, int act, float* out,
                   const HeadGeom& g, int t0, cudaStream_t st) {
  const size_t blocks = ((size_t)steps * R * O + 7) / 8;
  if (blocks == 0) return FSN_OK;
  FSN_REQUIRE(blocks <= 0x7fffffff, FSN_ERR_SHAPE, "sub-band head: too many rows");
  const unsigned grid = (unsigned)blocks;
  switch (act) {
    case FSN_ACT_RELU: sb_head_kernel<FSN_ACT_RELU><<<grid, 256, 0, st>>>(h, R, H, steps, W, bias, O, out, g, t0); break;
    case FSN_ACT_TANH: sb_head_kernel<FSN_ACT_TANH><<<grid, 256, 0, st>>>(h, R, H, steps, W, bias, O, out, g, t0); break;
    case FSN_ACT_RELU6: sb_head_kernel<FSN_ACT_RELU6><<<grid, 256, 0, st>>>(h, R, H, steps, W, bias, O, out, g, t0); break;
    default: sb_head_kernel<FSN_ACT_NONE><<<grid, 256, 0, st>>>(h, R, H, steps, W, bias, O, out, g, t0); break;
  }
  FSN_CHECK_LAUNCH("sb_head_kernel");
  return FSN_OK;
}

int sb_head_bwd_launch(const float* dcrm, const float* y, int act, int R, int O, int steps, int la, const HeadGeom& g,
                       float* dY, cudaStream_t st) {
  sb_head_bwd_kernel<<<ew_grid((size_t)steps * R * O), 256, 0, st>>>(dcrm, y, act, R, O, steps, la, g, dY);
  FSN_CHECK_LAUNCH("sb_head_bwd_kernel");
  return FSN_OK;
}

int crm_output_launch(const float* y, size_t bs, size_t ts, int B, int Tp, int F, int la, float* out, cudaStream_t st) {
  crm_output_kernel<<<dim3(cdiv(Tp - la, 32), cdiv(F, 32), B * 2), dim3(32, 8), 0, st>>>(y, bs, ts, Tp, F, la, out);
  FSN_CHECK_LAUNCH("crm_output_kernel");
  return FSN_OK;
}

int transpose_mag_launch(const float* in, int B, int F, int T, int Tp, size_t bs, size_t ts, float* out,
                         const float* scale, float* scaled, cudaStream_t st) {
  transpose_mag_kernel<<<dim3(cdiv(Tp, 32), cdiv(F, 32), B), dim3(32, 8), 0, st>>>(in, F, T, Tp, bs, ts, out, scale, scaled);
  FSN_CHECK_LAUNCH("transpose_mag_kernel");
  return FSN_OK;
}

int fast_bn_input_launch(const float* melT, const float* encT, size_t bs, size_t ts, int B, int Tp, int M, int Nn, int Ne,
                         int S, int Ts, float* bn, float2* fs, cudaStream_t st) {
  fast_bn_input_kernel<<<B * Ts, 256, 0, st>>>(melT, encT, bs, ts, B, Tp, M, Nn, Ne, S, Ts, bn, fs);
  FSN_CHECK_LAUNCH("fast_bn_input_kernel");
  return FSN_OK;
}

int fast_dec_input_launch(const float* encT, const float* bn_out, size_t nbs, size_t nms, size_t nts, int B, int Tp, int M,
                          int S, int Ts, size_t rbs, size_t rts, float* dec_in, cudaStream_t st) {
  fast_dec_input_kernel<<<ew_grid((size_t)B * Tp * 2 * M), 256, 0, st>>>(encT, bn_out, nbs, nms, nts, B, Tp, M, S, Ts, rbs,
                                                                          rts, dec_in);
  FSN_CHECK_LAUNCH("fast_dec_input_kernel");
  return FSN_OK;
}

int scale_rows_launch(const float* in, const float* scale, size_t n, int cols, int rows, int div, float* out,
                      cudaStream_t st) {
  scale_rows_kernel<<<ew_grid(n), 256, 0, st>>>(in, scale, n, cols, rows, div, out);
  FSN_CHECK_LAUNCH("scale_rows_kernel");
  return FSN_OK;
}

int layout_clips_check(int B, bool crm, const char* who) {
  const int most = crm ? LAYOUT_MAX_GRID_Z / 2 : LAYOUT_MAX_GRID_Z;
  FSN_REQUIRE(B <= most, FSN_ERR_UNSUPPORTED, "%s: B=%d clips, at most %d", who, B, most);
  return FSN_OK;
}

int frame_stats_launch(const float* x, int B, int Tp, int F, int N, size_t bs, size_t ts, float2* fs, cudaStream_t st) {
  frame_stats_kernel<<<cdiv(B * Tp, 8), 256, 0, st>>>(x, B, Tp, F, N, bs, ts, fs);
  FSN_CHECK_LAUNCH("frame_stats_kernel");
  return FSN_OK;
}

int clip_stats_launch(const float* x, int B, int T_pad, int F, int N, float2* fs, float2* sums, cudaStream_t st,
                      const int* lens, int hop, int la) {
  int rc;
  if ((rc = frame_stats_launch(x, B, T_pad, F, N, (size_t)T_pad * F, F, fs, st))) return rc;
  return clip_reduce_only_launch(fs, B, T_pad, sums, st, lens, hop, la);
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

using namespace fsn;

// ---- unit-test hook of the frame / clip statistics and the offline-norm scales (include/fsn_b200.h): the launchers the
// inference forwards run, every argument checked before any CUDA call; host lengths go to lens_dev through wav_prologue
extern "C" int fsn_debug_norm_stats(const float* x, int B, int T_pad, int F, int N, int64_t bs, int64_t ts,
                                    const int32_t* lengths, int* lens_dev, int hop, int la, const float* fb_sums, float cnt1,
                                    float cnt2, float eps, float* fs, float* sums, float* inv1, float* inv2,
                                    fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(x && fs && sums, FSN_ERR_SHAPE, "norm stats hook: null argument");
  FSN_REQUIRE(B > 0 && T_pad > 0 && F > 0 && bs >= 0 && ts >= 0, FSN_ERR_SHAPE,
              "norm stats hook: bad shape B=%d T_pad=%d F=%d", B, T_pad, F);
  FSN_REQUIRE(N >= 0 && N < F, FSN_ERR_SHAPE, "norm stats hook: reflect padding needs 0 <= N < F");
  FSN_REQUIRE((size_t)B * T_pad < ((size_t)1 << 31), FSN_ERR_SHAPE, "norm stats hook: B*T_pad must stay below 2^31");
  FSN_REQUIRE(!inv1 || cnt1 > 0.f, FSN_ERR_SHAPE, "norm stats hook: cnt1 must be positive");
  FSN_REQUIRE(!inv2 || cnt2 > 0.f, FSN_ERR_SHAPE, "norm stats hook: cnt2 must be positive");
  if (lengths) {
    FSN_REQUIRE(lens_dev && hop > 0 && la >= 0, FSN_ERR_SHAPE, "norm stats hook: lengths need lens_dev, hop > 0, la >= 0");
    for (int b = 0; b < B; ++b)
      FSN_REQUIRE(lengths[b] >= 0 && 1 + lengths[b] / hop + la <= T_pad, FSN_ERR_SHAPE,
                  "norm stats hook: clip %d has more than T_pad frames", b);
  }
  const cudaStream_t st = (cudaStream_t)stream;
  WavWs w = {nullptr, nullptr, nullptr, nullptr, lens_dev};
  int rc = wav_prologue(lengths, B, w, st);
  if (rc) return rc;
  float2* fs2 = reinterpret_cast<float2*>(fs);
  float2* sums2 = reinterpret_cast<float2*>(sums);
  if ((rc = frame_stats_launch(x, B, T_pad, F, N, (size_t)bs, (size_t)ts, fs2, st))) return rc;
  if ((rc = clip_reduce_only_launch(fs2, B, T_pad, sums2, st, w.lens, hop, la))) return rc;
  if (!inv1 && !inv2) return FSN_OK;
  return norm_scales_launch(sums2, fb_sums ? reinterpret_cast<const float2*>(fb_sums) : sums2, B, cnt1, cnt2, inv1, inv2,
                            st, eps, w.lens, hop, la);
}

// ---- unit-test hook of the forgetting norm's forward scan (include/fsn_b200.h): frame_stats + forget_scale_launch as the
// forwards run them, every argument checked before any CUDA call
extern "C" int fsn_debug_forgetting_scale(const float* x, int N, const float* x2, int N2, int B, int T_pad, int F,
                                          int64_t bs, int64_t ts, float cnt, const int32_t* lengths, int* lens_dev, int hop,
                                          int la, float* fs, float* fs2, float* scale, float* mu, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(x && fs && scale && (!x2 || fs2), FSN_ERR_SHAPE, "forgetting scale hook: null argument");
  FSN_REQUIRE(B > 0 && T_pad > 0 && F > 0 && bs >= 0 && ts >= 0, FSN_ERR_SHAPE,
              "forgetting scale hook: bad shape B=%d T_pad=%d F=%d", B, T_pad, F);
  FSN_REQUIRE(N >= 0 && N < F && (!x2 || (N2 >= 0 && N2 < F)), FSN_ERR_SHAPE,
              "forgetting scale hook: reflect padding needs 0 <= N < F");
  FSN_REQUIRE((size_t)B * T_pad < ((size_t)1 << 31), FSN_ERR_SHAPE, "forgetting scale hook: B*T_pad must stay below 2^31");
  FSN_REQUIRE(cnt > 0.f, FSN_ERR_SHAPE, "forgetting scale hook: cnt must be positive");
  if (lengths) {
    FSN_REQUIRE(lens_dev && hop > 0 && la >= 0, FSN_ERR_SHAPE,
                "forgetting scale hook: lengths need lens_dev, hop > 0, la >= 0");
    for (int b = 0; b < B; ++b)
      FSN_REQUIRE(lengths[b] >= 0 && 1 + lengths[b] / hop + la <= T_pad, FSN_ERR_SHAPE,
                  "forgetting scale hook: clip %d has more than T_pad frames", b);
  }
  const cudaStream_t st = (cudaStream_t)stream;
  WavWs w = {nullptr, nullptr, nullptr, nullptr, lens_dev};
  int rc = wav_prologue(lengths, B, w, st);
  if (rc) return rc;
  float2* f1 = reinterpret_cast<float2*>(fs);
  float2* f2 = x2 ? reinterpret_cast<float2*>(fs2) : nullptr;
  if ((rc = frame_stats_launch(x, B, T_pad, F, N, (size_t)bs, (size_t)ts, f1, st))) return rc;
  if (x2 && (rc = frame_stats_launch(x2, B, T_pad, F, N2, (size_t)bs, (size_t)ts, f2, st))) return rc;
  return forget_scale_launch(f1, f2, B, T_pad, cnt, scale, mu, st, w.lens, hop, la);
}

// ---- unit-test hook of the fp32 Linear (include/fsn_b200.h): fc_gemm_launch, every argument checked before any CUDA call
extern "C" int fsn_debug_fc_gemm(const float* A, const float* W, const float* bias, float* out, int M, int K, int O, int act,
                                 int w_kmajor, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(A && W && out, FSN_ERR_SHAPE, "fc_gemm hook: null argument");
  FSN_REQUIRE(M > 0 && K > 0 && O > 0, FSN_ERR_SHAPE, "fc_gemm hook: bad shape M=%d K=%d O=%d", M, K, O);
  FSN_REQUIRE(O <= 65535 * 64, FSN_ERR_SHAPE, "fc_gemm hook: O=%d exceeds the grid", O);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "fc_gemm hook: unknown act %d", act);
  return fc_gemm_launch(A, W, bias, out, M, K, O, act, (cudaStream_t)stream, w_kmajor != 0);
}

// ---- unit-test hooks of the causal-norm scales, the layout kernels and the sub-band heads (include/fsn_b200.h): each
// reaches its kernels through the launchers the forwards and training steps run, every argument checked before any CUDA
// call
static const size_t HOOK_MAX_ELEMS = (size_t)1 << 31;

// the sub-band row map of B clips of F bins with drop_band groups G (<= 1: none); R = B * Fsub
static int hook_row_map(const char* who, int B, int F, int G, RowMap& map, int& R) {
  FSN_REQUIRE(B > 0 && F > 0 && G >= 0, FSN_ERR_SHAPE, "%s: bad shape B=%d F=%d G=%d", who, B, F, G);
  FSN_REQUIRE(G <= 1 || (B > G && F >= G), FSN_ERR_SHAPE, "%s: drop_band needs B > G and F >= G", who);
  const int Fsub = G > 1 ? F / G : F;
  map = RowMap{B, F, Fsub, G > 1 ? G : 1};
  R = B * Fsub;
  return FSN_OK;
}

extern "C" int fsn_debug_cum_clip_scale(const float* x, int B, int Tp, int F, int64_t bs, int64_t ts, float eps, float* fs,
                                        float* scale1T, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(x && fs && scale1T, FSN_ERR_SHAPE, "cum clip scale hook: null argument");
  FSN_REQUIRE(B > 0 && Tp > 0 && F > 0 && bs >= 0 && ts >= 0, FSN_ERR_SHAPE, "cum clip scale hook: bad shape B=%d Tp=%d F=%d",
              B, Tp, F);
  FSN_REQUIRE((size_t)B * Tp < HOOK_MAX_ELEMS, FSN_ERR_SHAPE, "cum clip scale hook: B*Tp must stay below 2^31");
  const cudaStream_t st = (cudaStream_t)stream;
  float2* f2 = reinterpret_cast<float2*>(fs);
  int rc;
  if ((rc = frame_stats_launch(x, B, Tp, F, 0, (size_t)bs, (size_t)ts, f2, st))) return rc;
  return cum_clip_scale_launch(f2, B, Tp, F, eps, scale1T, st);
}

extern "C" int fsn_debug_cum_unit_scale(const float* magT, const float* fbT, int B, int F, int G, int Tp, int Ns, int Nf,
                                        float eps, int time_major, float* scaleT, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(magT && fbT && scaleT, FSN_ERR_SHAPE, "cum unit scale hook: null argument");
  RowMap map;
  int R, rc;
  if ((rc = hook_row_map("cum unit scale hook", B, F, G, map, R))) return rc;
  FSN_REQUIRE(Tp > 0, FSN_ERR_SHAPE, "cum unit scale hook: bad shape Tp=%d", Tp);
  FSN_REQUIRE(Ns >= 0 && Ns < F && Nf >= 0 && Nf < F, FSN_ERR_SHAPE, "cum unit scale hook: reflect padding needs 0 <= Ns, Nf < F");
  FSN_REQUIRE((size_t)Tp * R < HOOK_MAX_ELEMS && (size_t)Tp * B * F < HOOK_MAX_ELEMS, FSN_ERR_SHAPE,
              "cum unit scale hook: tensors must stay below 2^31 elements");
  return cum_unit_scale_launch(magT, fbT, map, R, Tp, Ns, Nf, eps, scaleT, (cudaStream_t)stream, time_major != 0);
}

extern "C" int fsn_debug_forget_unit_broadcast(const float* scaleT, int B, int F, int G, int Tp, float* unit_scale,
                                               fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(scaleT && unit_scale, FSN_ERR_SHAPE, "unit broadcast hook: null argument");
  RowMap map;
  int R, rc;
  if ((rc = hook_row_map("unit broadcast hook", B, F, G, map, R))) return rc;
  FSN_REQUIRE(Tp > 0 && (size_t)Tp * R < HOOK_MAX_ELEMS, FSN_ERR_SHAPE, "unit broadcast hook: bad shape Tp=%d", Tp);
  return forget_unit_broadcast_launch(scaleT, map, R, Tp, unit_scale, (cudaStream_t)stream);
}

extern "C" int fsn_debug_fast_bn(const float* melT, const float* encT, int64_t bs, int64_t ts, int B, int Tp, int M, int Nn,
                                 int Ne, int S, int cum, float eps, float* bn, float* fs, float* sums, float* scale,
                                 fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(melT && encT && bn && fs && scale && (cum || sums), FSN_ERR_SHAPE, "fast bottleneck hook: null argument");
  FSN_REQUIRE(B > 0 && Tp > 0 && M > 0 && S >= 1 && bs >= 0 && ts >= 0, FSN_ERR_SHAPE,
              "fast bottleneck hook: bad shape B=%d Tp=%d M=%d S=%d", B, Tp, M, S);
  FSN_REQUIRE(Nn >= 0 && Nn < M && Ne >= 0 && Ne < M, FSN_ERR_SHAPE, "fast bottleneck hook: reflect padding needs 0 <= Nn, Ne < M");
  const int K = (2 * Nn + 1) + (2 * Ne + 1), Ts = 1 + cdiv(Tp - 1, S), R = B * M;
  FSN_REQUIRE((size_t)Ts * R * K < HOOK_MAX_ELEMS && (size_t)B * Ts < HOOK_MAX_ELEMS, FSN_ERR_SHAPE,
              "fast bottleneck hook: tensors must stay below 2^31 elements");
  const cudaStream_t st = (cudaStream_t)stream;
  float2* f2 = reinterpret_cast<float2*>(fs);
  float2* s2 = reinterpret_cast<float2*>(sums);
  int rc;
  // as fsn_fast_model_forward and fsn_fast_train_forward run them
  if ((rc = fast_bn_input_launch(melT, encT, (size_t)bs, (size_t)ts, B, Tp, M, Nn, Ne, S, Ts, bn, f2, st))) return rc;
  if (cum) return fast_cum_bn_scale_launch(bn, R, K, Ts, eps, scale, st);
  if ((rc = clip_reduce_only_launch(f2, B, Ts, s2, st))) return rc;
  return norm_scales_launch(s2, s2, B, (float)M * K * Ts, 1.f, scale, nullptr, st, eps);
}

extern "C" int fsn_debug_fast_dec_input(const float* encT, const float* bn_out, int64_t nbs, int64_t nms, int64_t nts, int B,
                                        int Tp, int M, int S, int Ts, int64_t rbs, int64_t rts, float* dec_in,
                                        fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(encT && bn_out && dec_in, FSN_ERR_SHAPE, "decoder input hook: null argument");
  FSN_REQUIRE(B > 0 && Tp > 0 && M > 0 && S >= 1 && Ts > 0 && nbs >= 0 && nms >= 0 && nts >= 0, FSN_ERR_SHAPE,
              "decoder input hook: bad shape B=%d Tp=%d M=%d S=%d Ts=%d", B, Tp, M, S, Ts);
  FSN_REQUIRE((rbs == Tp && rts == 1) || (rbs == 1 && rts == B), FSN_ERR_SHAPE,
              "decoder input hook: rows clip-major (rbs = Tp, rts = 1) or time-major (rbs = 1, rts = B)");
  FSN_REQUIRE((size_t)B * Tp * 2 * M < HOOK_MAX_ELEMS, FSN_ERR_SHAPE, "decoder input hook: tensors must stay below 2^31");
  return fast_dec_input_launch(encT, bn_out, (size_t)nbs, (size_t)nms, (size_t)nts, B, Tp, M, S, Ts, (size_t)rbs, (size_t)rts,
                               dec_in, (cudaStream_t)stream);
}

extern "C" int fsn_debug_transpose_mag(const float* in, int B, int F, int T, int Tp, int64_t bs, int64_t ts, float* out,
                                       const float* scale, float* scaled, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(in && out && (!scaled || scale), FSN_ERR_SHAPE, "transpose_mag hook: null argument");
  FSN_REQUIRE(B > 0 && F > 0 && T > 0 && Tp >= T && bs >= 0 && ts >= 0, FSN_ERR_SHAPE,
              "transpose_mag hook: bad shape B=%d F=%d T=%d Tp=%d", B, F, T, Tp);
  FSN_REQUIRE(cdiv(F, 32) <= LAYOUT_MAX_GRID_Z, FSN_ERR_UNSUPPORTED, "transpose_mag hook: F=%d exceeds the grid", F);
  int rc;
  if ((rc = layout_clips_check(B, false, "transpose_mag hook"))) return rc;
  return transpose_mag_launch(in, B, F, T, Tp, (size_t)bs, (size_t)ts, out, scale, scaled, (cudaStream_t)stream);
}

extern "C" int fsn_debug_crm_output(const float* y, int64_t bs, int64_t ts, int B, int Tp, int F, int la, float* out,
                                    fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(y && out, FSN_ERR_SHAPE, "crm_output hook: null argument");
  FSN_REQUIRE(B > 0 && F > 0 && la >= 0 && Tp > la && bs >= 0 && ts >= 0, FSN_ERR_SHAPE,
              "crm_output hook: bad shape B=%d Tp=%d F=%d la=%d", B, Tp, F, la);
  FSN_REQUIRE(cdiv(F, 32) <= LAYOUT_MAX_GRID_Z, FSN_ERR_UNSUPPORTED, "crm_output hook: F=%d exceeds the grid", F);
  int rc;
  if ((rc = layout_clips_check(B, true, "crm_output hook"))) return rc;
  return crm_output_launch(y, (size_t)bs, (size_t)ts, B, Tp, F, la, out, (cudaStream_t)stream);
}

extern "C" int fsn_debug_scale_rows(const float* in, const float* scale, int64_t n, int cols, int rows, int div, float* out,
                                    fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(in && scale && out, FSN_ERR_SHAPE, "scale_rows hook: null argument");
  FSN_REQUIRE(n > 0 && cols > 0 && rows > 0 && div > 0, FSN_ERR_SHAPE,
              "scale_rows hook: bad shape n=%lld cols=%d rows=%d div=%d", (long long)n, cols, rows, div);
  return scale_rows_launch(in, scale, (size_t)n, cols, rows, div, out, (cudaStream_t)stream);
}

extern "C" int fsn_debug_imp_compress(const float* mag, int B, int F, int T, float fdrc, int tm, float* out,
                                      fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(mag && out, FSN_ERR_SHAPE, "imp_compress hook: null argument");
  FSN_REQUIRE(B > 0 && F >= 2 && T > 0, FSN_ERR_SHAPE, "imp_compress hook: bad shape B=%d F=%d T=%d", B, F, T);
  FSN_REQUIRE(cdiv(F - 1, 32) <= LAYOUT_MAX_GRID_Z, FSN_ERR_UNSUPPORTED, "imp_compress hook: F=%d exceeds the grid", F);
  FSN_REQUIRE((size_t)B * T * F < HOOK_MAX_ELEMS, FSN_ERR_SHAPE, "imp_compress hook: tensors must stay below 2^31");
  int rc;
  if ((rc = layout_clips_check(B, false, "imp_compress hook"))) return rc;
  return imp_compress_launch(mag, B, F, T, fdrc, tm != 0, out, (cudaStream_t)stream);
}

extern "C" int fsn_debug_train_gather(const float* raw, const float* fbz, const float* inv2, const float* unit_scale, int B,
                                      int F, int G, int Tp, int Ns, int Nf, float* X, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(raw && fbz && X && (inv2 || unit_scale), FSN_ERR_SHAPE, "train_gather hook: null argument");
  RowMap map;
  int R, rc;
  if ((rc = hook_row_map("train_gather hook", B, F, G, map, R))) return rc;
  FSN_REQUIRE(Tp > 0, FSN_ERR_SHAPE, "train_gather hook: bad shape Tp=%d", Tp);
  FSN_REQUIRE(Ns >= 0 && Ns < F && Nf >= 0 && Nf < F, FSN_ERR_SHAPE, "train_gather hook: reflect padding needs 0 <= Ns, Nf < F");
  FSN_REQUIRE((size_t)Tp * R * (2 * Ns + 2 * Nf + 2) < HOOK_MAX_ELEMS && (size_t)Tp * B * F < HOOK_MAX_ELEMS, FSN_ERR_SHAPE,
              "train_gather hook: tensors must stay below 2^31 elements");
  return train_gather_launch(raw, fbz, inv2, unit_scale, X, map, Tp, R, Ns, Nf, (cudaStream_t)stream);
}

// the cRM geometry of a head: R rows of N units per clip, O <= 2c outputs, section rows [lo, lo + N c) of `rows`
// (rows = 0: one channel, a plain [R, frames] table)
static int hook_head_geom(const char* who, int R, int O, int N, int c, int lo, int rows, int64_t rs, int64_t bs,
                          HeadGeom& g) {
  FSN_REQUIRE(R > 0 && O > 0 && N > 0 && c > 0 && lo >= 0 && rows >= 0 && rs > 0 && bs >= 0, FSN_ERR_SHAPE,
              "%s: bad geometry R=%d O=%d N=%d c=%d lo=%d rows=%d", who, R, O, N, c, lo, rows);
  FSN_REQUIRE(R % N == 0, FSN_ERR_SHAPE, "%s: R=%d rows are not whole clips of N=%d units", who, R, N);
  FSN_REQUIRE(O <= 2 * c, FSN_ERR_SHAPE, "%s: O=%d outputs exceed 2c = %d", who, O, 2 * c);
  FSN_REQUIRE(rows == 0 ? O <= c : (size_t)lo + (size_t)N * c <= (size_t)rows, FSN_ERR_SHAPE,
              "%s: section rows [%d, %d + N c) exceed rows=%d", who, lo, lo, rows);
  g = HeadGeom{N, c, lo, rows, (size_t)rs, (size_t)bs};
  return FSN_OK;
}

extern "C" int fsn_debug_sb_head(const float* h, int R, int H, int steps, const float* W, const float* bias, int O, int act,
                                 int N, int c, int lo, int rows, int64_t rs, int64_t bs, int t0, float* out,
                                 fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(h && W && bias && out, FSN_ERR_SHAPE, "sub-band head hook: null argument");
  FSN_REQUIRE(H > 0 && steps > 0 && t0 >= 0, FSN_ERR_SHAPE, "sub-band head hook: bad shape H=%d steps=%d t0=%d", H, steps, t0);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "sub-band head hook: unknown act %d", act);
  HeadGeom g;
  int rc;
  if ((rc = hook_head_geom("sub-band head hook", R, O, N, c, lo, rows, rs, bs, g))) return rc;
  FSN_REQUIRE(((size_t)steps * R * O + 7) / 8 <= 0x7fffffff && (size_t)steps * R * H < HOOK_MAX_ELEMS, FSN_ERR_SHAPE,
              "sub-band head hook: steps * R * O exceeds the grid");
  return sb_head_launch(h, R, H, steps, W, bias, O, act, out, g, t0, (cudaStream_t)stream);
}

extern "C" int fsn_debug_sb_head_bwd(const float* dcrm, const float* y, int act, int R, int O, int steps, int la, int N, int c,
                                     int lo, int rows, int64_t rs, int64_t bs, float* dY, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(dcrm && dY && (act == FSN_ACT_NONE || y), FSN_ERR_SHAPE, "sub-band head backward hook: null argument");
  FSN_REQUIRE(steps > 0 && la >= 0, FSN_ERR_SHAPE, "sub-band head backward hook: bad shape steps=%d la=%d", steps, la);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "sub-band head backward hook: unknown act %d", act);
  HeadGeom g;
  int rc;
  if ((rc = hook_head_geom("sub-band head backward hook", R, O, N, c, lo, rows, rs, bs, g))) return rc;
  FSN_REQUIRE((size_t)steps * R * O < HOOK_MAX_ELEMS, FSN_ERR_SHAPE, "sub-band head backward hook: tensors must stay below 2^31");
  return sb_head_bwd_launch(dcrm, y, act, R, O, steps, la, g, dY, (cudaStream_t)stream);
}

extern "C" int fsn_debug_train_dy(const float* dout, const float* y, int act, int B, int F, int T, int Tp, int la, float* dY,
                                  fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(dout && dY && (act == FSN_ACT_NONE || y), FSN_ERR_SHAPE, "train_dy hook: null argument");
  FSN_REQUIRE(B > 0 && F > 0 && T > 0 && la >= 0 && Tp == T + la, FSN_ERR_SHAPE,
              "train_dy hook: bad shape B=%d F=%d T=%d Tp=%d la=%d (Tp = T + la)", B, F, T, Tp, la);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "train_dy hook: unknown act %d", act);
  FSN_REQUIRE((size_t)Tp * B * 2 * F < HOOK_MAX_ELEMS, FSN_ERR_SHAPE, "train_dy hook: tensors must stay below 2^31");
  return train_dy_launch(dout, y, act, B, F, T, Tp, la, dY, (cudaStream_t)stream);
}
