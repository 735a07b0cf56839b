// Training step of recipes/dns_interspeech_2020/fullsubnet/trainer.py:56-68 (SURVEY 8a row A11), fp32:
//   fsn_train_forward   Model.forward in train mode, keeping what back-propagation through time needs
//   fsn_mse_loss        audio_zen/loss.py:4 (MSELoss) + d loss / d cRM
//   fsn_train_backward  BPTT through sub-band stack -> second norm (closed form) -> drop_band row map ->
//                       full-band Linear/ReLU -> full-band stack; weight gradients as split-K GEMMs over all steps
//   fsn_clip_adam       clip_grad_norm_ + Adam in three launches, no host synchronisation
// All saved activations are time-major ([Tp, rows, ...]) so every per-step operand is one contiguous block and
// every weight gradient is one GEMM over K = Tp*rows.  oracle/train_oracle.py:manual_backward is the same
// algorithm on the CPU.
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

// ------------------------------------------------------------------------------------------ GEMM
// C[M,N] (+)= op(A) B,  B [K,N] row-major (ldb); op(A) = A [M,K] (lda) or, TA, A stored [K,M] (lda).
// 64x64 tile, 4x4 per thread.  blockIdx.z = split-K slice writing its own [M,N] slab (ldc = N) at C + z*M*N.
template <bool TA>
__global__ void __launch_bounds__(256)
sgemm_kernel(const float* __restrict__ A, size_t lda, const float* __restrict__ Bm, size_t ldb, float* __restrict__ C,
             size_t ldc, int M, int N, int K, int k_per_split, int accumulate, size_t split_stride) {
  __shared__ __align__(16) float As[16][64];
  __shared__ __align__(16) float Bs[16][64];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int kb = blockIdx.z * k_per_split;
  const int ke = (kb + k_per_split < K) ? kb + k_per_split : K;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = kb; k0 < ke; k0 += 16) {
    if (!TA) {
      const int row = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = k0 + kq + j;
        As[kq + j][row] = (m0 + row < M && k < ke) ? A[(size_t)(m0 + row) * lda + k] : 0.f;
      }
    } else {
      const int kk = tid >> 4, mq = (tid & 15) * 4, k = k0 + kk;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int m = m0 + mq + j;
        As[kk][mq + j] = (k < ke && m < M) ? A[(size_t)k * lda + m] : 0.f;
      }
    }
    {
      const int kk = tid >> 4, nq = (tid & 15) * 4, k = k0 + kk;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + nq + j;
        Bs[kk][nq + j] = (k < ke && n < N) ? Bm[(size_t)k * ldb + n] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float b = Bs[kk][tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i][j] = fmaf(a[i], b, acc[i][j]);
      }
    }
    __syncthreads();
  }
  float* Cz = C + (size_t)blockIdx.z * split_stride;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = m0 + ty * 4 + i;
    if (row >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = n0 + tx + 16 * j;
      if (col >= N) continue;
      float* dst = Cz + (size_t)row * ldc + col;
      *dst = accumulate ? *dst + acc[i][j] : acc[i][j];
    }
  }
}

// C[m,n] (+)= sum_s part[s][m][n]  (fixed order: deterministic)
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int S, int M, int N, float* __restrict__ C,
                                     size_t ldc, int accumulate) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * N) return;
  float s = 0.f;
  for (int z = 0; z < S; ++z) s += part[(size_t)z * M * N + i];
  float* dst = C + (i / N) * ldc + (i % N);
  *dst = accumulate ? *dst + s : s;
}

int splitk_reduce_launch(const float* part, int S, int M, int N, float* C, size_t ldc, bool accumulate, cudaStream_t st) {
  const size_t n = (size_t)M * N;
  splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part, S, M, N, C, ldc, accumulate ? 1 : 0);
  FSN_CHECK_LAUNCH("splitk_reduce_kernel");
  return FSN_OK;
}

int sgemm_launch(bool ta, const float* A, size_t lda, const float* Bm, size_t ldb, float* C, size_t ldc, int M,
                        int N, int K, bool accumulate, float* scratch, size_t scratch_floats, cudaStream_t st) {
  if (M <= 0 || N <= 0 || K <= 0) return FSN_OK;
  const int tiles = cdiv(M, 64) * cdiv(N, 64);
  int S = 1;
  if (scratch && K >= 4096 && tiles < 528) {  // fill 132 SMs x 4 CTAs; slices of >= 1024 k
    S = cdiv(592, tiles);
    if (S > cdiv(K, 1024)) S = cdiv(K, 1024);
    while (S > 1 && (size_t)S * M * N > scratch_floats) --S;
  }
  const int kps = cdiv(cdiv(K, S), 16) * 16;
  S = cdiv(K, kps);
  dim3 grid(cdiv(M, 64), cdiv(N, 64), S);
  float* dst = S > 1 ? scratch : C;
  const size_t ldd = S > 1 ? (size_t)N : ldc;
  const int acc = (S > 1) ? 0 : (accumulate ? 1 : 0);
  if (ta) sgemm_kernel<true><<<grid, 256, 0, st>>>(A, lda, Bm, ldb, dst, ldd, M, N, K, kps, acc, (size_t)M * N);
  else    sgemm_kernel<false><<<grid, 256, 0, st>>>(A, lda, Bm, ldb, dst, ldd, M, N, K, kps, acc, (size_t)M * N);
  FSN_CHECK_LAUNCH("sgemm_kernel");
  if (S > 1) {
    const size_t n = (size_t)M * N;
    splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(scratch, S, M, N, C, ldc, accumulate ? 1 : 0);
    FSN_CHECK_LAUNCH("splitk_reduce_kernel");
  }
  return FSN_OK;
}

// out[c] = sum_r X[r*ldx + c]: slabs of rows -> part[S][cols] -> fixed-order sum
__global__ void colsum_part_kernel(const float* __restrict__ X, size_t rows, int cols, size_t ldx, size_t rows_per,
                                   float* __restrict__ part) {
  __shared__ float sh[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const size_t r0 = (size_t)blockIdx.y * rows_per;
  const size_t r1 = (r0 + rows_per < rows) ? r0 + rows_per : rows;
  float s = 0.f;
  if (c < cols)
    for (size_t r = r0 + threadIdx.y; r < r1; r += 8) s += X[r * ldx + c];
  sh[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sh[i][threadIdx.x];
    part[(size_t)blockIdx.y * cols + c] = t;
  }
}
__global__ void colsum_final_kernel(const float* __restrict__ part, int S, int cols, float* __restrict__ out,
                                    float* __restrict__ out2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int z = 0; z < S; ++z) s += part[(size_t)z * cols + c];
  out[c] = s;
  if (out2) out2[c] = s;
}
int colsum_final_launch(const float* part, int S, int cols, float* out, float* out2, cudaStream_t st) {
  colsum_final_kernel<<<cdiv(cols, 128), 128, 0, st>>>(part, S, cols, out, out2);
  FSN_CHECK_LAUNCH("colsum_final_kernel");
  return FSN_OK;
}

// dW [O,H] = dout^T Hm for a Linear with a few outputs (the sub-band Linear, O = 2; model.py:129-135 backwards):
// dout [rows,O], Hm [rows,H].  One pass over Hm: a CTA owns a slab of rows, a thread one column; part [S][O][H], then
// the fixed-order sum of colsum_final_kernel over S slabs of O*H "columns".
template <int O>
__global__ void __launch_bounds__(128) small_out_wgrad_kernel(const float* __restrict__ dout, const float* __restrict__ Hm,
                                                              size_t rows, int H, size_t rows_per, float* __restrict__ part) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  const size_t r0 = (size_t)blockIdx.y * rows_per;
  const size_t r1 = (r0 + rows_per < rows) ? r0 + rows_per : rows;
  float acc[O];
#pragma unroll
  for (int o = 0; o < O; ++o) acc[o] = 0.f;
  if (c < H) {
    size_t r = r0;
    for (; r + 4 <= r1; r += 4) {
      float h[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) h[j] = __ldcs(Hm + (r + j) * H + c);
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int o = 0; o < O; ++o) acc[o] = fmaf(dout[(r + j) * O + o], h[j], acc[o]);
    }
    for (; r < r1; ++r) {
      const float h = Hm[r * H + c];
#pragma unroll
      for (int o = 0; o < O; ++o) acc[o] = fmaf(dout[r * O + o], h, acc[o]);
    }
#pragma unroll
    for (int o = 0; o < O; ++o) part[((size_t)blockIdx.y * O + o) * H + c] = acc[o];
  }
}
// row slabs of a column sum over `rows` rows: one per 2048 rows, at most COLSUM_MAX_S
static int colsum_slabs(size_t rows) {
  int S = (int)((rows + 2047) / 2048);
  if (S > COLSUM_MAX_S) S = COLSUM_MAX_S;
  return S < 1 ? 1 : S;
}
int colsum_launch(const float* X, size_t rows, int cols, size_t ldx, float* out, float* out2, float* scratch,
                  size_t scratch_floats, cudaStream_t st) {
  const int S = colsum_slabs(rows);
  FSN_REQUIRE((size_t)S * cols <= scratch_floats, FSN_ERR_WORKSPACE, "colsum: %d slabs x %d columns exceed the %zu-float scratch",
              S, cols, scratch_floats);
  const size_t rows_per = (rows + S - 1) / S;
  colsum_part_kernel<<<dim3(cdiv(cols, 32), S), dim3(32, 8), 0, st>>>(X, rows, cols, ldx, rows_per, scratch);
  FSN_CHECK_LAUNCH("colsum_part_kernel");
  colsum_final_kernel<<<cdiv(cols, 128), 128, 0, st>>>(scratch, S, cols, out, out2);
  FSN_CHECK_LAUNCH("colsum_final_kernel");
  return FSN_OK;
}

// dW [2,H] of the 2-output sub-band Linear from dout [rows,2] and Hm [rows,H]: one streaming pass over Hm (2.4 GB at
// config 3), partials [S][2][H] in scratch, then their fixed-order sum.  S drops until the partials fit scratch_floats.
int small_out_wgrad_launch(const float* dout, const float* Hm, size_t rows, int H, float* dW, float* scratch,
                           size_t scratch_floats, cudaStream_t st) {
  int S = (int)((rows + 2047) / 2048);
  if (S > COLSUM_MAX_S) S = COLSUM_MAX_S;
  while (S > 1 && (size_t)S * 2 * H > scratch_floats) --S;
  FSN_REQUIRE((size_t)S * 2 * H <= scratch_floats, FSN_ERR_WORKSPACE, "small_out_wgrad: %d floats of partials exceed the %zu-float scratch",
              2 * H, scratch_floats);
  const size_t rows_per = (rows + S - 1) / S;
  small_out_wgrad_kernel<2><<<dim3(cdiv(H, 128), S), 128, 0, st>>>(dout, Hm, rows, H, rows_per, scratch);
  FSN_CHECK_LAUNCH("small_out_wgrad_kernel");
  colsum_final_kernel<<<cdiv(2 * H, 128), 128, 0, st>>>(scratch, S, 2 * H, dW, nullptr);
  FSN_CHECK_LAUNCH("colsum_final_kernel");
  return FSN_OK;
}

// ------------------------------------------------------------------------------------------ forward helpers
// per-clip sums of noisy_mag [B,F,T]: (sum, sum_f c_Ns[f] * row sum), one CTA per clip, fixed-order tree
__global__ void train_mag_stats_kernel(const float* __restrict__ mag, int F, int T, int Ns, float2* __restrict__ sums) {
  __shared__ float2 sh[256];
  const int b = blockIdx.x;
  const float* p = mag + (size_t)b * F * T;
  float2 a = make_float2(0.f, 0.f);
  for (int i = threadIdx.x; i < F * T; i += 256) {
    const float v = p[i];
    a.x += v;
    a.y += v * (float)reflect_count(i / T, F, Ns);
  }
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) { sh[threadIdx.x].x += sh[threadIdx.x + s].x; sh[threadIdx.x].y += sh[threadIdx.x + s].y; }
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[b] = sh[0];
}

// same for a time-major tensor x [Tp,B,F]
__global__ void train_tm_stats_kernel(const float* __restrict__ x, int B, int F, int Tp, int N, float2* __restrict__ sums) {
  __shared__ float2 sh[256];
  const int b = blockIdx.x;
  float2 a = make_float2(0.f, 0.f);
  for (int i = threadIdx.x; i < F * Tp; i += 256) {
    const int t = i / F, f = i - t * F;
    const float v = x[((size_t)t * B + b) * F + f];
    a.x += v;
    a.y += v * (float)reflect_count(f, F, N);
  }
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) { sh[threadIdx.x].x += sh[threadIdx.x + s].x; sh[threadIdx.x].y += sh[threadIdx.x + s].y; }
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[b] = sh[0];
}

int train_mag_stats_launch(const float* mag, int B, int F, int T, int Ns, float2* sums, cudaStream_t st) {
  train_mag_stats_kernel<<<B, 256, 0, st>>>(mag, F, T, Ns, sums);
  FSN_CHECK_LAUNCH("train_mag_stats_kernel");
  return FSN_OK;
}

int train_tm_stats_launch(const float* x, int B, int F, int Tp, int N, float2* sums, cudaStream_t st) {
  train_tm_stats_kernel<<<B, 256, 0, st>>>(x, B, F, Tp, N, sums);
  FSN_CHECK_LAUNCH("train_tm_stats_kernel");
  return FSN_OK;
}

// sub-band input X[t,r,k] (base_model.py:13-46 + model.py:98-119): unit (b,f) of row r, scaled by inv2[b]
__global__ void train_gather_kernel(const float* __restrict__ raw, const float* __restrict__ fbz,
                                    const float* __restrict__ inv2, const float* __restrict__ unit_scale,
                                    float* __restrict__ X, RowMap map, int Tp, int R, int Ns, int Nf) {
  const int K = 2 * Ns + 1 + 2 * Nf + 1;
  const size_t n = (size_t)Tp * R * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    const size_t tr = i / K;
    const int r = (int)(tr % R), t = (int)(tr / R);
    int b, f;
    row_to_unit(map, r, b, f);
    const size_t base = ((size_t)t * map.B + b) * map.F;
    float v;
    if (k < 2 * Ns + 1) v = raw[base + reflect_idx(f + k - Ns, map.F)];
    else                v = fbz[base + reflect_idx(f + (k - 2 * Ns - 1) - Nf, map.F)];
    X[i] = v * (unit_scale ? unit_scale[tr] : inv2[b]);  // cumulative norm: scale of (step t, unit r) at [t*R + r]
  }
}

int train_gather_launch(const float* raw, const float* fbz, const float* inv2, const float* unit_scale, float* X, RowMap map,
                        int Tp, int R, int Ns, int Nf, cudaStream_t st) {
  train_gather_kernel<<<132 * 8, 256, 0, st>>>(raw, fbz, inv2, unit_scale, X, map, Tp, R, Ns, Nf);
  FSN_CHECK_LAUNCH("train_gather_kernel");
  return FSN_OK;
}

// ---- cumulative_laplace_norm in the training step (audio_zen/model/base_model.py:220-251)
// Backward of X[t,r,k] = u[t,r,k] * s[t,r], s = 1/(m + eps), m[t,r] = sum_{t'<=t} sum_k u[t',r,k] / (K (t+1)):
//   d u[t,r,k] = dX[t,r,k] s[t,r] + sum_{t''>=t} q[t'',r],   q[t,r] = -s[t,r] <dX[t,r,:], X[t,r,:]> / (K (t+1)).
// Only the full-band row k = K-1 has a parameter behind it (Nf = 0): dunit[t,r] = its gradient.  One thread per
// unit, sequential in t (suffix sum in a fixed order).
__global__ void train_cum_unit_bwd_kernel(const float* __restrict__ dX, const float* __restrict__ X,
                                          const float* __restrict__ scaleT, int Tp, int R, int K, float* __restrict__ dunit) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float suffix = 0.f;
  for (int t = Tp - 1; t >= 0; --t) {
    const size_t o = ((size_t)t * R + r) * K;
    float dot = 0.f;
    for (int k = 0; k < K; ++k) dot = fmaf(dX[o + k], X[o + k], dot);
    const float s = scaleT[(size_t)t * R + r];
    suffix += -s * dot / ((float)K * (float)(t + 1));
    dunit[(size_t)t * R + r] = fmaf(dX[o + K - 1], s, suffix);
  }
}
// dz[t,b,f] = act'(fbz) * dunit[t, row(b,f)]  (units removed by drop_band carry no gradient: their norm is their own)
__global__ void train_dfbz_cum_kernel(const float* __restrict__ dunit, const float* __restrict__ fbz, RowMap map, int Tp,
                                      int R, int act, float* __restrict__ dz) {
  const size_t n = (size_t)Tp * map.B * map.F;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int f = (int)(i % map.F);
    const size_t tb = i / map.F;
    const int b = (int)(tb % map.B), t = (int)(tb / map.B);
    const int r = unit_to_row(map, b, f);
    dz[i] = act_grad(r >= 0 ? dunit[(size_t)t * R + r] : 0.f, fbz, i, act);
  }
}

int train_cum_unit_bwd_launch(const float* dX, const float* X, const float* scaleT, int Tp, int R, int K, float* dunit,
                              cudaStream_t st) {
  train_cum_unit_bwd_kernel<<<cdiv(R, 128), 128, 0, st>>>(dX, X, scaleT, Tp, R, K, dunit);
  FSN_CHECK_LAUNCH("train_cum_unit_bwd_kernel");
  return FSN_OK;
}

int train_dfbz_cum_launch(const float* dunit, const float* fbz, RowMap map, int Tp, int R, int act, float* dz,
                          cudaStream_t st) {
  train_dfbz_cum_kernel<<<132 * 8, 256, 0, st>>>(dunit, fbz, map, Tp, R, act, dz);
  FSN_CHECK_LAUNCH("train_dfbz_cum_kernel");
  return FSN_OK;
}

// ---- forgetting_norm at the second norm (base_model.py:102-151 on sb_input [B,F,K,T'], one scale per (clip, step))
// Backward of X[t,r,k] = u[t,r,k] s_t, s_t = 1/(mu_t + eps), mu_t = a_t mu_{t-1} + b_t m_t, m_t = sum_{f,k} u / cnt over
// all F units of the clip (drop_band comes after the norm):
//   d mu_t (direct) = -s_t^2 <dX, u>_t = -s_t <dX, X>_t,  g_t = d mu_t + a_{t+1} g_{t+1},  d m_t = b_t g_t,
//   d u[t,r,k] = dX[t,r,k] s_t + d m_t / cnt.
// dot[t*B + b] <- <dX, X> over the Fsub rows of output clip bq at step t; one CTA per (t, bq), fixed-order tree.
__global__ void train_forget_dot_kernel(const float* __restrict__ dX, const float* __restrict__ X, RowMap map, int Tp,
                                        int R, int K, float* __restrict__ dot) {
  __shared__ float sh[256];
  const int bq = blockIdx.x % map.B, t = blockIdx.x / map.B;
  const size_t base = ((size_t)t * R + (size_t)bq * map.Fsub) * K, n = (size_t)map.Fsub * K;
  float a = 0.f;
  for (size_t i = threadIdx.x; i < n; i += 256) a = fmaf(dX[base + i], X[base + i], a);
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int b, f;
    row_to_unit(map, bq * map.Fsub, b, f);  // source clip of output clip bq
    dot[(size_t)t * map.B + b] = sh[0];
  }
}
// the reverse recurrence, one thread per clip, in place: mid[t*B + b] holds <dX, X>_t on entry, d m_t / cnt on exit
__global__ void train_forget_scan_bwd_kernel(const float* __restrict__ scale2T, int B, int Tp, float cnt, const ForgetCoef c,
                                             float* __restrict__ mid) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float g = 0.f;
  for (int t = Tp - 1; t >= 0; --t) {
    const size_t i = (size_t)t * B + b;
    const float a_next = t + 1 < FORGET_LEN ? c.a[t + 1] : c.a[FORGET_LEN];
    g = fmaf(a_next, g, -scale2T[i] * mid[i]);  // a_{t+1} g_{t+1} + d mu_t; g_{Tp} = 0
    mid[i] = c.b[t < FORGET_LEN ? t : FORGET_LEN] * g / cnt;
  }
}
// dz[t,b,f] = act'(fbz) (dX[t, row(b,f), K-1] s_t + mid[t,b])  (Nf = 0: the full-band row f enters the mean once)
__global__ void train_dfbz_forget_kernel(const float* __restrict__ dX, const float* __restrict__ fbz,
                                         const float* __restrict__ scale2T, const float* __restrict__ mid, RowMap map,
                                         int Tp, int R, int K, int act, float* __restrict__ dz) {
  const size_t n = (size_t)Tp * map.B * map.F;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int f = (int)(i % map.F);
    const size_t tb = i / map.F;
    const int b = (int)(tb % map.B), t = (int)(tb / map.B);
    float v = mid[tb];
    const int r = unit_to_row(map, b, f);
    if (r >= 0) v = fmaf(dX[((size_t)t * R + r) * K + (K - 1)], scale2T[tb], v);
    dz[i] = act_grad(v, fbz, i, act);
  }
}

int train_forget_bwd_launch(const float* dX, const float* X, const float* fbz, const float* scale2T, RowMap map, int Tp,
                            int R, int K, float cnt, int act, float* mid, float* dz, cudaStream_t st) {
  train_forget_dot_kernel<<<(unsigned)((size_t)Tp * map.B), 256, 0, st>>>(dX, X, map, Tp, R, K, mid);
  FSN_CHECK_LAUNCH("train_forget_dot_kernel");
  train_forget_scan_bwd_kernel<<<cdiv(map.B, 64), 64, 0, st>>>(scale2T, map.B, Tp, cnt, forget_coef(), mid);
  FSN_CHECK_LAUNCH("train_forget_scan_bwd_kernel");
  train_dfbz_forget_kernel<<<132 * 8, 256, 0, st>>>(dX, fbz, scale2T, mid, map, Tp, R, K, act, dz);
  FSN_CHECK_LAUNCH("train_dfbz_forget_kernel");
  return FSN_OK;
}

// LSTM cell of one step (tensor-core path): G_t [R,4H] holds x_t W_ih^T (all steps from one hoisted GEMM), rec the
// recurrent product of this step; G_t is overwritten with the post-activation gates (i,f,g,o); writes c_t and h_t
__global__ void lstm_cell_fwd_kernel(float* __restrict__ G, const float* __restrict__ rec, const float* __restrict__ b_ih,
                                     const float* __restrict__ b_hh, const float* __restrict__ C_prev,
                                     float* __restrict__ C_out, float* __restrict__ H_out, int R, int H) {
  const size_t n = (size_t)R * H;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
    const int u = (int)(idx % H);
    const size_t r = idx / H;
    float* g = G + r * 4 * H + u;
    float z[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      z[q] = g[q * H] + b_ih[q * H + u] + b_hh[q * H + u];
      if (rec) z[q] += rec[r * 4 * H + q * H + u];  // h_{t-1} W_hh^T of this step
    }
    const float si = sigmoidf_(z[0]), sf = sigmoidf_(z[1]), tg = tanhf(z[2]), so = sigmoidf_(z[3]);
    const float c = sf * (C_prev ? C_prev[idx] : 0.f) + si * tg;
    g[0] = si; g[H] = sf; g[2 * H] = tg; g[3 * H] = so;
    C_out[idx] = c;
    H_out[idx] = so * tanhf(c);
  }
}

// out[c, r] = in[r, c]   (in [rows, cols] row-major -> out [cols, rows]); operands of the K-major tensor-core GEMM
__global__ void transpose_kernel(const float* __restrict__ in, size_t rows, int cols, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const size_t r0 = (size_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const size_t r = r0 + i;
    const int c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < cols) ? in[r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i;
    const size_t r = r0 + threadIdx.x;
    if (c < cols && r < rows) out[(size_t)c * rows + r] = tile[threadIdx.x][i];
  }
}
int transpose_launch(const float* in, size_t rows, int cols, float* out, cudaStream_t st) {
  dim3 grid((unsigned)((rows + 31) / 32), cdiv(cols, 32));
  transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(in, rows, cols, out);
  FSN_CHECK_LAUNCH("transpose_kernel");
  return FSN_OK;
}

// ------------------------------------------------------------------------------------------ backward kernels
struct BwdPoint {
  int R, H;
  float* G;             // [R,4H] in: gates (post-activation), out: d(pre-activation)
  const float* C;       // [R,H] cell state of this step
  const float* C_prev;  // nullable (t == 0)
  const float* dh_above;  // nullable [R,H]
  const float* dh_rec;    // nullable [R,H]
  float* dc;              // [R,H] in (ignored when first_dc): d c_t from step t+1, out: d c_{t-1}
  int first_dc;
  const float* dout;  // nullable [R,O]: dh_above += dout W_fc   (Linear backward, small O)
  const float* fc_w;  // [O,H]
  int O;
};

__global__ void lstm_bwd_point_kernel(const BwdPoint p) {
  const size_t n = (size_t)p.R * p.H;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
    const int u = (int)(idx % p.H);
    const size_t r = idx / p.H;
    float dh = 0.f;
    if (p.dh_above) dh += p.dh_above[idx];
    if (p.dh_rec) dh += p.dh_rec[idx];
    if (p.dout)
      for (int o = 0; o < p.O; ++o) dh = fmaf(p.dout[r * p.O + o], p.fc_w[(size_t)o * p.H + u], dh);
    float* g = p.G + r * 4 * p.H + u;
    const float gi = g[0], gf = g[p.H], gg = g[2 * p.H], go = g[3 * p.H];
    const float tc = tanhf(p.C[idx]);
    const float dc_tot = (p.first_dc ? 0.f : p.dc[idx]) + dh * go * (1.f - tc * tc);
    const float c_prev = p.C_prev ? p.C_prev[idx] : 0.f;
    g[0] = dc_tot * gg * gi * (1.f - gi);
    g[p.H] = dc_tot * c_prev * gf * (1.f - gf);
    g[2 * p.H] = dc_tot * gi * (1.f - gg * gg);
    g[3 * p.H] = dh * tc * go * (1.f - go);
    p.dc[idx] = dc_tot * gf;
  }
}

// dot[b'] = sum over the rows of output clip b' and all t,k of dX * X   (second-norm backward)
__global__ void train_dot_kernel(const float* __restrict__ dX, const float* __restrict__ X, int Tp, int R, int Fsub,
                                 int K, float* __restrict__ dot) {
  __shared__ float sh[256];
  const int bq = blockIdx.x;
  const size_t per_t = (size_t)Fsub * K;
  float a = 0.f;
  for (int t = 0; t < Tp; ++t) {
    const size_t base = ((size_t)t * R + (size_t)bq * Fsub) * K;
    for (size_t i = threadIdx.x; i < per_t; i += 256) a = fmaf(dX[base + i], X[base + i], a);
  }
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) dot[bq] = sh[0];
}

// dz[t,b,f] = act'(fbz) * ( dX[t, row(b,f), K-1] * inv2[b]  -  inv2[b] * dot[b'(b)] * c_Nf[f] / cnt2 )   (Nf = 0)
__global__ void train_dfbz_kernel(const float* __restrict__ dX, const float* __restrict__ fbz,
                                  const float* __restrict__ inv2, const float* __restrict__ dot, RowMap map, int Tp,
                                  int R, int K, float cnt2, int act, float* __restrict__ dz) {
  const size_t n = (size_t)Tp * map.B * map.F;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int f = (int)(i % map.F);
    const size_t tb = i / map.F;
    const int b = (int)(tb % map.B), t = (int)(tb / map.B);
    // output clip of b: row of any kept frequency of that clip / Fsub
    int bq;
    if (map.G <= 1) bq = b;
    else bq = unit_to_row(map, b, b % map.G) / map.Fsub;
    const float s = inv2[b];
    float v = -s * dot[bq] / cnt2;
    const int r = unit_to_row(map, b, f);
    if (r >= 0) v = fmaf(dX[((size_t)t * R + r) * K + (K - 1)], s, v);
    const float y = fbz[i];
    if (act == FSN_ACT_RELU) v = y > 0.f ? v : 0.f;
    else if (act == FSN_ACT_TANH) v *= 1.f - y * y;
    else if (act == FSN_ACT_RELU6) v = (y > 0.f && y < 6.f) ? v : 0.f;
    dz[i] = v;
  }
}

int train_dot_launch(const float* dX, const float* X, int Tp, int R, int Fsub, int K, int clips, float* dot, cudaStream_t st) {
  train_dot_kernel<<<clips, 256, 0, st>>>(dX, X, Tp, R, Fsub, K, dot);
  FSN_CHECK_LAUNCH("train_dot_kernel");
  return FSN_OK;
}

int train_dfbz_launch(const float* dX, const float* fbz, const float* inv2, const float* dot, RowMap map, int Tp, int R, int K,
                      float cnt2, int act, float* dz, cudaStream_t st) {
  train_dfbz_kernel<<<132 * 8, 256, 0, st>>>(dX, fbz, inv2, dot, map, Tp, R, K, cnt2, act, dz);
  FSN_CHECK_LAUNCH("train_dfbz_kernel");
  return FSN_OK;
}

// ------------------------------------------------------------------------------------------ workspace

struct TrainWs {
  float *raw, *xfb, *fbz, *inv1, *inv2;
  float2 *sums_mag, *sums_fb;
  LayerSave fb[2], sb[2];
  float *xsb, *dxsb, *dout, *dz, *dfh1;
  float *dh_rec[2], *dc[2], *dh_mid, *dot;
  float *splitk, *colsum;
  float *splitk2, *colsum2;  // scratch of the side stream (full-band backward overlapped with the sub-band weight gradients)
  size_t colsum_floats;       // floats of colsum and of colsum2
  // FSN_PREC_TF32_TC: transposed weights ([H,4H], [K0,4H]) and transposed dG / layer inputs for the weight gradients
  float *sb_whhT[2], *sb_wihT[2], *fb_whhT[2], *fb_wihT1;
  float *gT, *xT, *rec;
  __half *fb_h16[2], *sb_h16[2], *w16;  // fp16 MMA operands of the forward step kernel (hidden states, weights)
  float *cum1, *cum2, *dunit;  // cumulative norm: scale of (step, clip), of (step, unit); gradient of the fb row per unit
  float2* fs;
  // forgetting norm: cum1 / cum2 as above (cum2 the broadcast of fg2), fs the frame sums of the noisy magnitude; fs2 those
  // of the full-band output, fg2 [Tp,B] the second norm's scale of (step, clip), fmid [Tp,B] its backward's d m_t / cnt
  float *fg2, *fmid;
  float2* fs2;
  size_t bytes;
};

static void carve_train(const fsn_model_desc* d, const Dims& m, void* base, TrainWs& w) {
  Carver c(base);
  const size_t Tp = m.Tp, B = m.B, F = m.F, R = m.R, Hf = d->fb_hidden, Hs = d->sb_hidden;
  w.raw = c.take<float>(Tp * B * F); w.xfb = c.take<float>(Tp * B * F); w.fbz = c.take<float>(Tp * B * F);
  w.inv1 = c.take<float>(B); w.inv2 = c.take<float>(B);
  w.sums_mag = c.take<float2>(B); w.sums_fb = c.take<float2>(B);
  for (int l = 0; l < 2; ++l) {
    w.fb[l].G = c.take<float>(Tp * B * 4 * Hf); w.fb[l].C = c.take<float>(Tp * B * Hf); w.fb[l].H = c.take<float>(Tp * B * Hf);
    w.sb[l].G = c.take<float>(Tp * R * 4 * Hs); w.sb[l].C = c.take<float>(Tp * R * Hs); w.sb[l].H = c.take<float>(Tp * R * Hs);
  }
  w.xsb = c.take<float>(Tp * R * m.Ksb); w.dxsb = c.take<float>(Tp * R * m.Ksb);
  w.dout = c.take<float>(Tp * R * 2);
  w.dz = c.take<float>(Tp * B * F); w.dfh1 = c.take<float>(Tp * B * Hf);
  const size_t RH = (R * Hs > B * Hf) ? R * Hs : B * Hf;
  for (int i = 0; i < 2; ++i) { w.dh_rec[i] = c.take<float>(RH); w.dc[i] = c.take<float>(RH); }
  w.dh_mid = c.take<float>(RH);
  w.dot = c.take<float>(B);
  w.cum1 = w.cum2 = w.dunit = w.fg2 = w.fmid = nullptr; w.fs = w.fs2 = nullptr;
  if (d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE) {
    w.cum1 = c.take<float>(Tp * B); w.cum2 = c.take<float>(Tp * R); w.dunit = c.take<float>(Tp * R);
    w.fs = c.take<float2>(Tp * B);
  } else if (d->norm_type == FSN_NORM_FORGETTING) {
    w.cum1 = c.take<float>(Tp * B); w.cum2 = c.take<float>(Tp * R); w.fg2 = c.take<float>(Tp * B);
    w.fmid = c.take<float>(Tp * B);
    w.fs = c.take<float2>(Tp * B); w.fs2 = c.take<float2>(Tp * B);
  }
  w.splitk = c.take<float>(SPLITK_SCRATCH_FLOATS);
  const size_t maxcols = 4 * (Hf > Hs ? Hf : Hs) > F ? 4 * (Hf > Hs ? Hf : Hs) : F;
  w.colsum_floats = (size_t)COLSUM_MAX_S * maxcols;  // each of colsum, colsum2
  w.colsum = c.take<float>(w.colsum_floats);
  w.splitk2 = c.take<float>(SPLITK_SCRATCH_FLOATS);
  w.colsum2 = c.take<float>(w.colsum_floats);
  if (d->precision == FSN_PREC_TF32_TC) {
    for (int l = 0; l < 2; ++l) {
      w.sb_whhT[l] = c.take<float>(Hs * 4 * Hs);
      w.sb_wihT[l] = c.take<float>((l == 0 ? (size_t)m.Ksb : Hs) * 4 * Hs);
      w.fb_whhT[l] = c.take<float>(Hf * 4 * Hf);
    }
    w.fb_wihT1 = c.take<float>(Hf * 4 * Hf);
    // K-major (block-tiled, zero padded: tgemm_blocked_floats) copies of dG and of the layer input / hidden states
    const size_t g_sb = tgemm_blocked_floats(Tp * R, 4 * (int)Hs), g_fb = tgemm_blocked_floats(Tp * B, 4 * (int)Hf);
    w.gT = c.take<float>(g_sb > g_fb ? g_sb : g_fb);
    const size_t x_sb = tgemm_blocked_floats(Tp * R, Hs > (size_t)m.Ksb ? (int)Hs : m.Ksb),
                 x_fb = tgemm_blocked_floats(Tp * B, Hf > F ? (int)Hf : (int)F);
    w.xT = c.take<float>(x_sb > x_fb ? x_sb : x_fb);
    w.rec = c.take<float>(4 * RH);
    for (int l = 0; l < 2; ++l) {
      w.fb_h16[l] = c.take<__half>(Tp * B * Hf);
      w.sb_h16[l] = c.take<__half>(Tp * R * Hs);
    }
    const size_t wmax = Hf > Hs ? Hf : Hs;
    w.w16 = c.take<__half>(4 * wmax * 2 * wmax);
  } else {
    w.fb_h16[0] = w.fb_h16[1] = w.sb_h16[0] = w.sb_h16[1] = w.w16 = nullptr;
  }
  w.bytes = c.off;
}

static int train_check(const fsn_model_desc* d) {
  FSN_REQUIRE(d->norm_type == FSN_NORM_OFFLINE_LAPLACE || d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE ||
                  d->norm_type == FSN_NORM_FORGETTING,
              FSN_ERR_UNSUPPORTED, "training: offline_laplace_norm, cumulative_laplace_norm and forgetting_norm are built");
  FSN_REQUIRE(d->fb_num_neighbors == 0, FSN_ERR_UNSUPPORTED,
              "training: fb_num_neighbors > 0 is not built (every shipped recipe uses 0)");
  FSN_REQUIRE(d->cell_type == FSN_CELL_LSTM, FSN_ERR_UNSUPPORTED, "training: the GRU cell is built for inference only");
  return FSN_OK;
}

// one layer forward over all steps, saving gates / cell / hidden:  X [Tp,R,K0] (row_scale == nullptr)
int layer_forward_save(const fsn_lstm_layer& w, const float* X, int R, int K0, int H, int Tp, const LayerSave& s,
                       cudaStream_t st) {
  for (int t = 0; t < Tp; ++t) {
    StepParams p;
    memset(&p, 0, sizeof(p));
    p.R = R; p.K0 = K0; p.H = H; p.first = (t == 0);
    p.w_ih = w.w_ih; p.w_hh = w.w_hh; p.b_ih = w.b_ih; p.b_hh = w.b_hh;
    p.x0 = X + (size_t)t * R * K0; p.x0_row_stride = K0;
    p.h_prev = s.H + (size_t)(t > 0 ? t - 1 : 0) * R * H; p.h_prev_stride = H;
    p.h_out = s.H + (size_t)t * R * H; p.h_out_stride = H;
    p.c = s.C + (size_t)t * R * H;
    p.c_in = s.C + (size_t)(t > 0 ? t - 1 : 0) * R * H;
    p.save_gates = s.G + (size_t)t * R * 4 * H;
    int rc = lstm_step_launch(p, SEG0_DENSE, st);
    if (rc) return rc;
  }
  return FSN_OK;
}

// tensor-core variant.  H % 32 == 0: ONE kernel per step (lstm_fwd_step_kernel, fsn_tgemm.cu): [x_t | h_{t-1}] [W_ih | W_hh]^T
// on wgmma and the cell on its accumulators, gates / cell / hidden saved.  A layer input wider than 512 or whose rows are
// not 16-byte aligned keeps a hoisted projection of all steps (one GEMM into the gate buffer) that the step kernel adds.
// H % 32 != 0: every step is a recurrent GEMM into `rec` + lstm_cell_fwd_kernel
int layer_forward_save_tc(const fsn_lstm_layer& w, const float* X, int R, int K0, int H, int Tp, const LayerSave& s,
                          float* rec, cudaStream_t st, float* splitk, size_t splitk_floats, const LayerHalf* half) {
  int rc;
  const int rows = Tp * R;
  const bool fused = lstm_fwd_step_supported(s.H, w.w_hh, H);
  // x_t W_ih^T as leading k blocks of the step kernel - no hoisted projection, G is written once and never read in the
  // forward pass
  const bool fold = fused && lstm_fwd_step_folds_input(X, w.w_ih, K0);
  // fp16 MMA operands when the caller passes the buffers: h_t (written by the step kernel next to the fp32 copy) and the
  // weights, rounded to nearest (the same 11-bit significand as a tf32 read, half the bytes through L2 and twice the
  // tensor rate); the folded layer input too when the layer below left an fp16 copy (K0 % 8: 16-byte rows).  The fp32
  // state, the saved activations and the backward pass are unchanged
  const bool h16 = fused && half && half->H16 && half->w16;
  const bool x16 = h16 && fold && half->X16 && (K0 % 8) == 0;
  __half* w_hh16 = h16 ? half->w16 : nullptr;
  __half* w_ih16 = x16 ? half->w16 + (size_t)4 * H * H : nullptr;
  if (h16 && (rc = to_half_launch(w.w_hh, (size_t)4 * H * H, w_hh16, st))) return rc;
  if (x16 && (rc = to_half_launch(w.w_ih, (size_t)4 * H * K0, w_ih16, st))) return rc;
  if (fold) {
  } else if (tgemm_supported(X, K0, w.w_ih, K0, K0)) {
    if ((rc = tgemm_launch(X, K0, w.w_ih, K0, s.G, 4 * H, rows, 4 * H, K0, false, nullptr, 0, st))) return rc;
  } else if ((rc = fc_gemm_launch(X, w.w_ih, nullptr, s.G, rows, K0, 4 * H, FSN_ACT_NONE, st))) {
    return rc;  // rows of X not 16-byte aligned (K0 % 4 != 0): fp32 SIMT GEMM
  }
  const unsigned blocks = ew_grid((size_t)R * H);
  for (int t = 0; t < Tp; ++t) {
    float* Gt = s.G + (size_t)t * R * 4 * H;
    if (fused && (t > 0 || fold)) {  // GEMM + cell in one kernel, the recurrent product stays in registers
      LstmStepHalf hs{nullptr, nullptr, nullptr, nullptr, nullptr};
      if (h16) {
        hs.Hprev16 = t > 0 ? half->H16 + (size_t)(t - 1) * R * H : nullptr;
        hs.w_hh16 = w_hh16;
        hs.H16_out = half->H16 + (size_t)t * R * H;
        if (x16) { hs.Xt16 = half->X16 + (size_t)t * R * K0; hs.w_ih16 = w_ih16; }
      }
      if ((rc = lstm_fwd_step_launch(t > 0 ? s.H + (size_t)(t - 1) * R * H : nullptr, w.w_hh,
                                     fold ? X + (size_t)t * R * K0 : nullptr, w.w_ih, K0, Gt, w.b_ih, w.b_hh,
                                     t > 0 ? s.C + (size_t)(t - 1) * R * H : nullptr, s.C + (size_t)t * R * H,
                                     s.H + (size_t)t * R * H, R, H, st, h16 ? &hs : nullptr)))
        return rc;
      continue;
    }
    // (first step of a layer with a hoisted projection: no product at all, the plain cell kernel; its h_0 also goes out
    // in fp16 below)
    if (t > 0)
      if ((rc = tgemm_launch(s.H + (size_t)(t - 1) * R * H, H, w.w_hh, H, rec, 4 * H, R, 4 * H, H, false, splitk, splitk_floats, st)))
        return rc;
    lstm_cell_fwd_kernel<<<blocks, 256, 0, st>>>(Gt, t > 0 ? rec : nullptr, w.b_ih, w.b_hh,
                                                 t > 0 ? s.C + (size_t)(t - 1) * R * H : nullptr,
                                                 s.C + (size_t)t * R * H, s.H + (size_t)t * R * H, R, H);
    FSN_CHECK_LAUNCH("lstm_cell_fwd_kernel");
    if (h16 && (rc = to_half_launch(s.H + (size_t)t * R * H, (size_t)R * H, half->H16 + (size_t)t * R * H, st))) return rc;
  }
  return FSN_OK;
}

int layer_forward(int precision, const fsn_lstm_layer& w, const float* X, int R, int K0, int H, int Tp, const LayerSave& s,
                  float* rec, float* splitk, const LayerHalf* half, cudaStream_t st) {
  if (!tf32_layer(precision, H) || !tgemm_available()) return layer_forward_save(w, X, R, K0, H, Tp, s, st);
  return layer_forward_save_tc(w, X, R, K0, H, Tp, s, rec, st, splitk, SPLITK_SCRATCH_FLOATS, half);
}

// the backward half of the rule of layer_forward: the transposed weights mark a tf32 layer
static bool tc_bwd(const LayerBwd& L) { return L.w_hhT && tgemm_available(); }

int layer_bwd_transpose_weights(const LayerBwd& L, cudaStream_t st) {
  if (!tc_bwd(L)) return FSN_OK;
  int rc;
  if ((rc = transpose_launch(L.w_hh, (size_t)4 * L.H, L.H, L.w_hhT, st))) return rc;
  if (L.w_ihT && (rc = transpose_launch(L.w_ih, (size_t)4 * L.H, L.K0, L.w_ihT, st))) return rc;
  return FSN_OK;
}

int linear_bwd(const float* dY, const float* X, const float* W, int rows, int N, int K, float* dW, float* db, float* dX,
               float* splitk, float* colsum, size_t colsum_floats, cudaStream_t st) {
  int rc;
  if ((rc = sgemm_launch(true, dY, N, X, K, dW, K, N, K, rows, false, splitk, SPLITK_SCRATCH_FLOATS, st))) return rc;
  if ((rc = colsum_launch(dY, (size_t)rows, N, N, db, nullptr, colsum, colsum_floats, st))) return rc;
  if (dX && (rc = sgemm_launch(false, dY, N, W, K, dX, K, rows, K, N, false, nullptr, 0, st))) return rc;
  return FSN_OK;
}

// step t of one layer: pointwise gate gradients, then dh_rec = dG W_hh and (optionally) dx = dG W_ih
int layer_bwd_step(const LayerBwd& L, int t, int Tp, const float* dh_above, const float* dout, const float* fc_w,
                          int O, float* dx, cudaStream_t st) {
  BwdPoint p;
  memset(&p, 0, sizeof(p));
  p.R = L.R; p.H = L.H;
  p.G = L.s.G + (size_t)t * L.R * 4 * L.H;
  p.C = L.s.C + (size_t)t * L.R * L.H;
  p.C_prev = t > 0 ? L.s.C + (size_t)(t - 1) * L.R * L.H : nullptr;
  p.dh_above = dh_above;
  p.dh_rec = (t == Tp - 1) ? nullptr : L.dh_rec;
  p.dc = L.dc; p.first_dc = (t == Tp - 1);
  p.dout = dout; p.fc_w = fc_w; p.O = O;
  lstm_bwd_point_kernel<<<ew_grid((size_t)L.R * L.H), 256, 0, st>>>(p);
  FSN_CHECK_LAUNCH("lstm_bwd_point_kernel");
  int rc;
  const bool tc = tc_bwd(L);
  if (t > 0) {
    if (tc) rc = tgemm_launch(p.G, 4 * L.H, L.w_hhT, 4 * L.H, L.dh_rec, L.H, L.R, L.H, 4 * L.H, false, L.splitk, SPLITK_SCRATCH_FLOATS, st);
    else         rc = sgemm_launch(false, p.G, 4 * L.H, L.w_hh, L.H, L.dh_rec, L.H, L.R, L.H, 4 * L.H, false, nullptr, 0, st);
    if (rc) return rc;
  }
  if (dx) {
    if (tc && L.w_ihT) rc = tgemm_launch(p.G, 4 * L.H, L.w_ihT, 4 * L.H, dx, L.K0, L.R, L.K0, 4 * L.H, false, L.splitk, SPLITK_SCRATCH_FLOATS, st);
    else         rc = sgemm_launch(false, p.G, 4 * L.H, L.w_ih, L.K0, dx, L.K0, L.R, L.K0, 4 * L.H, false, nullptr, 0, st);
    if (rc) return rc;
  }
  return FSN_OK;
}

// weight / bias gradients of one layer from dG [Tp*R,4H] (in L.s.G), its input X [Tp*R,K0] and hidden states
int layer_weight_grads(const LayerBwd& L, int Tp, const float* X, float* g_w_ih, float* g_w_hh, float* g_b_ih,
                       float* g_b_hh, const WgradScratch& w, cudaStream_t st) {
  const int H4 = 4 * L.H;
  const int rows = Tp * L.R;
  int rc;
  if (tc_bwd(L)) {
    // tensor-core path, block-tiled K-major copies (one contiguous 16 KB burst per TMA box instead of 128 rows with a
    // pitch of `rows` floats): dW_ih = dG^T X, dW_hh = dG[1:]^T H[:-1]
    const int nkb = (rows + 31) / 32;
    int slabs = 0;  // bias gradients = column sums of dG, taken while its tiles pass through shared memory
    // at most COLSUM_MAX_S slabs of H4 partial sums, fewer when the scratch holds fewer
    const size_t fit = w.colsum_floats / H4;
    FSN_REQUIRE(fit >= 1, FSN_ERR_WORKSPACE, "weight gradients: %zu floats of column-sum scratch for %d columns", w.colsum_floats, H4);
    if ((rc = transpose_blocked_launch(L.s.G, (size_t)rows, H4, (size_t)H4, w.gT, st, w.colsum,
                                       fit < (size_t)COLSUM_MAX_S ? (int)fit : COLSUM_MAX_S, &slabs)))
      return rc;
    colsum_final_kernel<<<cdiv(H4, 128), 128, 0, st>>>(w.colsum, slabs, H4, g_b_ih, g_b_hh);
    FSN_CHECK_LAUNCH("colsum_final_kernel");
    if ((rc = transpose_blocked_launch(X, (size_t)rows, L.K0, (size_t)L.K0, w.xT, st, nullptr, 0, nullptr))) return rc;
    if ((rc = tgemm_blocked_launch(w.gT, nkb, 0, w.xT, nkb, 0, g_w_ih, L.K0, H4, L.K0, rows, false, w.splitk, SPLITK_SCRATCH_FLOATS, st)))
      return rc;
    if (Tp > 1) {
      if ((rc = transpose_blocked_launch(L.s.H, (size_t)rows, L.H, (size_t)L.H, w.xT, st, nullptr, 0, nullptr))) return rc;
      int a_kb0 = L.R / 32, a_nkb = nkb;
      if (L.R & 31) {  // step offset not on a k block: a second copy that starts at step 1
        a_kb0 = 0; a_nkb = (rows - L.R + 31) / 32;
        if ((rc = transpose_blocked_launch(L.s.G + (size_t)L.R * H4, (size_t)(rows - L.R), H4, (size_t)H4, w.gT, st, nullptr, 0, nullptr)))
          return rc;
      }
      if ((rc = tgemm_blocked_launch(w.gT, a_nkb, a_kb0, w.xT, nkb, 0, g_w_hh, L.H, H4, L.H, rows - L.R, false, w.splitk,
                                     SPLITK_SCRATCH_FLOATS, st)))
        return rc;
    } else if ((rc = check_cuda(cudaMemsetAsync(g_w_hh, 0, (size_t)H4 * L.H * sizeof(float), st), "memset"))) {
      return rc;
    }
    return FSN_OK;
  }
  if ((rc = sgemm_launch(true, L.s.G, H4, X, L.K0, g_w_ih, L.K0, H4, L.K0, rows, false, w.splitk, SPLITK_SCRATCH_FLOATS,
                         st)))
    return rc;
  if (Tp > 1) {
    if ((rc = sgemm_launch(true, L.s.G + (size_t)L.R * H4, H4, L.s.H, L.H, g_w_hh, L.H, H4, L.H, rows - L.R, false,
                           w.splitk, SPLITK_SCRATCH_FLOATS, st)))
      return rc;
  } else if ((rc = check_cuda(cudaMemsetAsync(g_w_hh, 0, (size_t)H4 * L.H * sizeof(float), st), "memset"))) {
    return rc;
  }
  return colsum_launch(L.s.G, (size_t)rows, H4, H4, g_b_ih, g_b_hh, w.colsum, w.colsum_floats, st);
}

int stack_bwd(const LayerBwd* L, int n, int steps, const float* dh_above, const float* dout, const float* fc_w, int O,
              float* dh_mid0, float* dh_mid1, float* dx, cudaStream_t st) {
  float* mid[2] = {dh_mid0, dh_mid1};
  int rc;
  for (int t = steps - 1; t >= 0; --t) {
    for (int l = n - 1; l >= 0; --l) {
      const LayerBwd& q = L[l];
      const bool top = l == n - 1;
      const float* dh = top ? (dh_above ? dh_above + (size_t)t * q.R * q.H : nullptr) : mid[(n - 2 - l) & 1];
      const float* dl = top && dout ? dout + (size_t)t * q.R * O : nullptr;
      float* dxl = l > 0 ? mid[(n - 1 - l) & 1] : (dx ? dx + (size_t)t * q.R * q.K0 : nullptr);
      if ((rc = layer_bwd_step(q, t, steps, dh, dl, top ? fc_w : nullptr, top ? O : 0, dxl, st))) return rc;
    }
  }
  return FSN_OK;
}

// ------------------------------------------------------------------------------------------ shared by the training steps
int train_input_launch(const float* noisy_mag, int B, int F, int T, int Tp, int Ns, int norm_type, float2* sums, float* inv1,
                       float* raw, float* scaled, float2* fs, float* cum1, cudaStream_t st) {
  int rc;
  if ((rc = train_mag_stats_launch(noisy_mag, B, F, T, Ns, sums, st))) return rc;
  if ((rc = norm_scales_launch(sums, sums, B, (float)F * Tp, 1.f, inv1, nullptr, st))) return rc;
  // raw [Tp,B,F] and scaled = raw * inv1[b]
  if ((rc = transpose_mag_launch(noisy_mag, B, F, T, Tp, F, (size_t)B * F, raw, inv1, scaled, st))) return rc;
  if (norm_per_step(norm_type)) {  // causal running mean per clip instead of the clip mean
    if ((rc = frame_stats_launch(raw, B, Tp, F, 0, F, (size_t)B * F, fs, st))) return rc;
    if (norm_type == FSN_NORM_FORGETTING) rc = forget_scale_launch(fs, nullptr, B, Tp, (float)F, cum1, nullptr, st);
    else rc = cum_clip_scale_launch(fs, B, Tp, F, TRAIN_CUM_EPS, cum1, st);  // base_model.py:220-251
    if (rc) return rc;
    if ((rc = scale_rows_launch(raw, cum1, (size_t)Tp * B * F, F, Tp * B, 1, scaled, st))) return rc;  // scale of (t, b)
  }
  return FSN_OK;
}

// dY [Tp,B,2F] from dout [B,2,F,T], zero on the look-ahead frames, times act'(y) of the kept post-activation output
__global__ void train_dy_kernel(const float* __restrict__ dout, const float* __restrict__ y, int act, int B, int F, int T,
                                int Tp, int la, float* __restrict__ dY) {
  const size_t n = (size_t)Tp * B * 2 * F;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int cf = (int)(i % (2 * F));
    const size_t tb = i / (2 * F);
    const int b = (int)(tb % B), t = (int)(tb / B);
    dY[i] = act_grad(t >= la ? dout[((size_t)b * 2 * F + cf) * T + (t - la)] : 0.f, y, i, act);
  }
}

int train_dy_launch(const float* dout, const float* y, int act, int B, int F, int T, int Tp, int la, float* dY,
                    cudaStream_t st) {
  train_dy_kernel<<<ew_grid((size_t)Tp * B * 2 * F), 256, 0, st>>>(dout, y, act, B, F, T, Tp, la, dY);
  FSN_CHECK_LAUNCH("train_dy_kernel");
  return FSN_OK;
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_train_workspace_bytes(const fsn_model_desc* d, int B, int T) {
  Dims m;
  if (make_dims(d, B, T, m)) return 0;
  TrainWs w;
  carve_train(d, m, nullptr, w);
  return w.bytes;
}

extern "C" int fsn_train_forward(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                                 const float* noisy_mag, int B, int T, float* crm, void* workspace,
                                 size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  Dims m;
  int rc = make_dims(d, B, T, m);
  if (rc) return rc;
  if ((rc = train_check(d))) return rc;
  if ((rc = layout_clips_check(B, false, "training"))) return rc;
  TrainWs w;
  carve_train(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int Tp = m.Tp, F = m.F, Hf = d->fb_hidden, Hs = d->sb_hidden;
  // first norm (model.py:92) and the time-major copies
  const bool cum = d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE, fgt = d->norm_type == FSN_NORM_FORGETTING;
  if ((rc = train_input_launch(noisy_mag, B, F, T, Tp, d->sb_num_neighbors, d->norm_type, w.sums_mag, w.inv1, w.raw, w.xfb,
                               w.fs, w.cum1, st)))
    return rc;
  // full-band stack + Linear/activation (model.py:92-95)
  // fp16 operand copies: layer 0's hidden states double as layer 1's input
  const LayerHalf hf0{w.fb_h16[0], nullptr, w.w16}, hf1{w.fb_h16[1], w.fb_h16[0], w.w16};
  const LayerHalf hs0{w.sb_h16[0], nullptr, w.w16}, hs1{w.sb_h16[1], w.sb_h16[0], w.w16};
  const int prec = d->precision;
  if ((rc = layer_forward(prec, seq_layer(*fb, 0), w.xfb, B, F, Hf, Tp, w.fb[0], w.rec, w.splitk, &hf0, st))) return rc;
  if ((rc = layer_forward(prec, seq_layer(*fb, 1), w.fb[0].H, B, Hf, Hf, Tp, w.fb[1], w.rec, w.splitk, &hf1, st))) return rc;
  if ((rc = fc_gemm_launch(w.fb[1].H, fb->fc_w, fb->fc_b, w.fbz, Tp * B, Hf, F, d->fb_activation, st))) return rc;
  // second norm in closed form (model.py:110-111)
  if ((rc = train_tm_stats_launch(w.fbz, B, F, Tp, d->fb_num_neighbors, w.sums_fb, st))) return rc;
  if ((rc = norm_scales_launch(w.sums_mag, w.sums_fb, B, 1.f, (float)F * m.Ksb * Tp, nullptr, w.inv2, st))) return rc;
  // sub-band units (unfold + concat + norm + drop_band as one gather), then the sub-band stack (model.py:98-128)
  RowMap map{B, F, m.Fsub, m.G};
  if (cum && (rc = cum_unit_scale_launch(w.raw, w.fbz, map, m.R, Tp, d->sb_num_neighbors, d->fb_num_neighbors, TRAIN_CUM_EPS, w.cum2,
                                         st, /*time_major=*/true)))
    return rc;
  if (fgt) {  // one scale per (step, clip) over all F K features: the reflect-weighted frame sums of both unfolds
    if ((rc = frame_stats_launch(w.raw, B, Tp, F, d->sb_num_neighbors, F, (size_t)B * F, w.fs, st))) return rc;
    if ((rc = frame_stats_launch(w.fbz, B, Tp, F, d->fb_num_neighbors, F, (size_t)B * F, w.fs2, st))) return rc;
    if ((rc = forget_scale_launch(w.fs, w.fs2, B, Tp, (float)F * m.Ksb, w.fg2, nullptr, st))) return rc;
    if ((rc = forget_unit_broadcast_launch(w.fg2, map, m.R, Tp, w.cum2, st))) return rc;
  }
  if ((rc = train_gather_launch(w.raw, w.fbz, w.inv2, (cum || fgt) ? w.cum2 : nullptr, w.xsb, map, Tp, m.R,
                                d->sb_num_neighbors, d->fb_num_neighbors, st)))
    return rc;
  if ((rc = layer_forward(prec, seq_layer(*sb, 0), w.xsb, m.R, m.Ksb, Hs, Tp, w.sb[0], w.rec, w.splitk, &hs0, st))) return rc;
  if ((rc = layer_forward(prec, seq_layer(*sb, 1), w.sb[0].H, m.R, Hs, Hs, Tp, w.sb[1], w.rec, w.splitk, &hs1, st))) return rc;
  // sub-band Linear of every output frame in one launch (model.py:129-135; the first look_ahead steps have no frame)
  return sb_head_launch(w.sb[1].H + (size_t)d->look_ahead * m.R * Hs, m.R, Hs, Tp - d->look_ahead, sb->fc_w, sb->fc_b, 2,
                        d->sb_activation, crm, fsn_head_geom(m.Fsub, m.T), 0, st);
}

namespace fsn {
// Side stream of the backward pass: the full-band BPTT is a chain of ~1 900 tiny launches (64 rows), the sub-band weight
// gradients are a dozen HBM-bound kernels with no dependency on it - they run side by side.  One high-priority
// non-blocking stream and two events per device, created on first use; fork / join through events only, so the pattern
// is also legal inside a stream capture.
struct SideStream { cudaStream_t s; cudaEvent_t fork, join; };
static int side_stream(SideStream** out) {
  static SideStream per_dev[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  SideStream& x = per_dev[dev & 63];
  int rc;
  if (!x.s) {  // a failed creation is retried by the next call, keeping what it did create
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if ((rc = check_cuda(cudaStreamCreateWithPriority(&x.s, cudaStreamNonBlocking, hi), "side stream"))) return rc;
  }
  if (!x.fork && (rc = check_cuda(cudaEventCreateWithFlags(&x.fork, cudaEventDisableTiming), "side stream event"))) return rc;
  if (!x.join && (rc = check_cuda(cudaEventCreateWithFlags(&x.join, cudaEventDisableTiming), "side stream event"))) return rc;
  *out = &x;
  return FSN_OK;
}
}  // namespace fsn

extern "C" int fsn_train_backward(const fsn_model_desc* d, const fsn_seq_weights* fb, const fsn_seq_weights* sb,
                                  const float* dcrm, int B, int T, const fsn_seq_grads* gfb, const fsn_seq_grads* gsb,
                                  void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  Dims m;
  int rc = make_dims(d, B, T, m);
  if (rc) return rc;
  if ((rc = train_check(d))) return rc;
  FSN_REQUIRE(d->sb_activation == FSN_ACT_NONE, FSN_ERR_UNSUPPORTED,
              "training: sb_output_activate_function must be off (as in every shipped recipe)");
  TrainWs w;
  carve_train(d, m, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const int Tp = m.Tp, F = m.F, R = m.R, Hf = d->fb_hidden, Hs = d->sb_hidden, K = m.Ksb;
  RowMap map{B, F, m.Fsub, m.G};
  // ---- sub-band Linear (model.py:129-135 backwards)
  if ((rc = sb_head_bwd_launch(dcrm, nullptr, FSN_ACT_NONE, R, 2, Tp, d->look_ahead, fsn_head_geom(m.Fsub, T), w.dout, st)))
    return rc;
  // dW of the 2-output Linear: one streaming pass over h1
  if ((rc = small_out_wgrad_launch(w.dout, w.sb[1].H, (size_t)Tp * R, Hs, gsb->fc_w, w.splitk, SPLITK_SCRATCH_FLOATS, st)))
    return rc;
  if ((rc = colsum_launch(w.dout, (size_t)Tp * R, 2, 2, gsb->fc_b, nullptr, w.colsum, w.colsum_floats, st))) return rc;
  const bool tc_fb = tf32_layer(d->precision, Hf), tc_sb = tf32_layer(d->precision, Hs);
  // the full-band chain (second norm, full-band Linear, full-band BPTT) runs on the side stream st2, with its own split-K /
  // column-sum scratch
  SideStream* side = nullptr;
  if ((rc = side_stream(&side))) return rc;
  cudaStream_t st2 = side->s;
  // sub-band layers 0, 1, full-band layers 0, 1 (full-band layer 0 computes no dx)
  const LayerBwd L[4] = {
      {sb->w_ih[0], sb->w_hh[0], w.sb[0], R, K, Hs, w.dh_rec[0], w.dc[0], tc_sb ? w.sb_whhT[0] : nullptr,
       tc_sb ? w.sb_wihT[0] : nullptr, w.splitk},
      {sb->w_ih[1], sb->w_hh[1], w.sb[1], R, Hs, Hs, w.dh_rec[1], w.dc[1], tc_sb ? w.sb_whhT[1] : nullptr,
       tc_sb ? w.sb_wihT[1] : nullptr, w.splitk},
      {fb->w_ih[0], fb->w_hh[0], w.fb[0], B, F, Hf, w.dh_rec[0], w.dc[0], tc_fb ? w.fb_whhT[0] : nullptr, nullptr, w.splitk2},
      {fb->w_ih[1], fb->w_hh[1], w.fb[1], B, Hf, Hf, w.dh_rec[1], w.dc[1], tc_fb ? w.fb_whhT[1] : nullptr,
       tc_fb ? w.fb_wihT1 : nullptr, w.splitk2}};
  const LayerBwd *sbL = L, *fbL = L + 2;
  for (int l = 0; l < 4; ++l)
    if ((rc = layer_bwd_transpose_weights(L[l], st))) return rc;
  // ---- sub-band stack, both layers one step apart
  if ((rc = stack_bwd(sbL, 2, Tp, nullptr, w.dout, sb->fc_w, 2, w.dh_mid, nullptr, w.dxsb, st))) return rc;
  // ---- fork: sub-band weight gradients on the caller's stream, the rest of the chain on st2
  if ((rc = check_cuda(cudaEventRecord(side->fork, st), "event record"))) return rc;
  if ((rc = check_cuda(cudaStreamWaitEvent(st2, side->fork, 0), "stream wait"))) return rc;
  const WgradScratch wg{w.gT, w.xT, w.splitk, w.colsum, w.colsum_floats};
  if ((rc = layer_weight_grads(sbL[1], Tp, w.sb[0].H, gsb->w_ih[1], gsb->w_hh[1], gsb->b_ih[1], gsb->b_hh[1], wg, st)))
    return rc;
  if ((rc = layer_weight_grads(sbL[0], Tp, w.xsb, gsb->w_ih[0], gsb->w_hh[0], gsb->b_ih[0], gsb->b_hh[0], wg, st))) return rc;
  // ---- second norm + drop_band + full-band Linear/activation
  if (d->norm_type == FSN_NORM_CUMULATIVE_LAPLACE) {
    if ((rc = train_cum_unit_bwd_launch(w.dxsb, w.xsb, w.cum2, Tp, R, K, w.dunit, st2))) return rc;
    if ((rc = train_dfbz_cum_launch(w.dunit, w.fbz, map, Tp, R, d->fb_activation, w.dz, st2))) return rc;
  } else if (d->norm_type == FSN_NORM_FORGETTING) {
    if ((rc = train_forget_bwd_launch(w.dxsb, w.xsb, w.fbz, w.fg2, map, Tp, R, K, (float)F * K, d->fb_activation, w.fmid,
                                      w.dz, st2)))
      return rc;
  } else {
    if ((rc = train_dot_launch(w.dxsb, w.xsb, Tp, R, m.Fsub, K, B, w.dot, st2))) return rc;
    if ((rc = train_dfbz_launch(w.dxsb, w.fbz, w.inv2, w.dot, map, Tp, R, K, (float)F * K * Tp, d->fb_activation, w.dz,
                                st2)))
      return rc;
  }
  if ((rc = linear_bwd(w.dz, w.fb[1].H, fb->fc_w, Tp * B, F, Hf, gfb->fc_w, gfb->fc_b, w.dfh1, w.splitk2, w.colsum2,
                       w.colsum_floats, st2)))
    return rc;
  // ---- full-band stack
  if ((rc = stack_bwd(fbL, 2, Tp, w.dfh1, nullptr, nullptr, 0, w.dh_mid, nullptr, nullptr, st2))) return rc;
  // join: the full-band weight gradients share gT / xT / splitk / colsum with the sub-band ones
  if ((rc = check_cuda(cudaEventRecord(side->join, st2), "event record"))) return rc;
  if ((rc = check_cuda(cudaStreamWaitEvent(st, side->join, 0), "stream wait"))) return rc;
  if ((rc = layer_weight_grads(fbL[1], Tp, w.fb[0].H, gfb->w_ih[1], gfb->w_hh[1], gfb->b_ih[1], gfb->b_hh[1], wg, st)))
    return rc;
  return layer_weight_grads(fbL[0], Tp, w.xfb, gfb->w_ih[0], gfb->w_hh[0], gfb->b_ih[0], gfb->b_hh[0], wg, st);
}

// ------------------------------------------------------------------------------------------ unit-test hook
// An n-layer LSTM stack through the shared training pieces alone (layer_forward, layer_bwd_transpose_weights, stack_bwd,
// layer_weight_grads), wired like fsn_fullband_train_*: per-layer saves and BPTT slots, layer l's fp16 hidden states are
// layer l+1's fp16 input, one split-K / column-sum / K-major scratch for all layers.
namespace fsn {
static const int DBG_MAX_LAYERS = 8;

struct DbgLstmWs {
  LayerSave L[DBG_MAX_LAYERS];
  float *dh_rec[DBG_MAX_LAYERS], *dc[DBG_MAX_LAYERS], *dh_mid[2];
  float *splitk, *colsum, *gT, *xT, *rec;
  size_t colsum_floats;
  float *whhT[DBG_MAX_LAYERS], *wihT[DBG_MAX_LAYERS];
  __half *h16[DBG_MAX_LAYERS], *w16;
  size_t bytes;
};

static void carve_dbg_lstm(int n, int R, int T, int K0, int H, int precision, void* base, DbgLstmWs& w) {
  Carver c(base);
  const size_t rows = (size_t)T * R, Hs = H, RH = (size_t)R * H, K0max = K0 > H ? K0 : H;
  for (int l = 0; l < n; ++l) {
    w.L[l].G = c.take<float>(rows * 4 * Hs); w.L[l].C = c.take<float>(rows * Hs); w.L[l].H = c.take<float>(rows * Hs);
  }
  for (int l = 0; l < n; ++l) { w.dh_rec[l] = c.take<float>(RH); w.dc[l] = c.take<float>(RH); }
  w.dh_mid[0] = c.take<float>(RH);
  w.dh_mid[1] = c.take<float>(RH);
  w.splitk = c.take<float>(SPLITK_SCRATCH_FLOATS);
  w.colsum_floats = (size_t)COLSUM_MAX_S * 4 * Hs;
  w.colsum = c.take<float>(w.colsum_floats);
  w.gT = w.xT = w.rec = nullptr;
  w.w16 = nullptr;
  for (int l = 0; l < DBG_MAX_LAYERS; ++l) { w.whhT[l] = w.wihT[l] = nullptr; w.h16[l] = nullptr; }
  if (tf32_layer(precision, H)) {
    for (int l = 0; l < n; ++l) {
      w.whhT[l] = c.take<float>(Hs * 4 * Hs);
      w.wihT[l] = c.take<float>((l == 0 ? (size_t)K0 : Hs) * 4 * Hs);  // layer 0's is used only when dx is asked for
      w.h16[l] = c.take<__half>(rows * Hs);
    }
    w.gT = c.take<float>(tgemm_blocked_floats(rows, 4 * H));
    w.xT = c.take<float>(tgemm_blocked_floats(rows, (int)K0max));
    w.rec = c.take<float>(4 * RH);
    w.w16 = c.take<__half>(4 * Hs * (Hs + K0max));
  }
  w.bytes = c.off;
}

static int dbg_lstm_check(int n, int R, int T, int K0, int H, int precision) {
  FSN_REQUIRE(precision == FSN_PREC_FP32 || precision == FSN_PREC_TF32_TC, FSN_ERR_UNSUPPORTED,
              "lstm_train hook: precision must be fp32 or tf32_tc");
  FSN_REQUIRE(n >= 1 && n <= DBG_MAX_LAYERS, FSN_ERR_UNSUPPORTED, "lstm_train hook: 1..%d layers (got %d)", DBG_MAX_LAYERS, n);
  FSN_REQUIRE(R > 0 && T > 0 && K0 > 0 && H > 0, FSN_ERR_SHAPE, "lstm_train hook: bad dims R=%d T=%d K0=%d H=%d", R, T, K0, H);
  const size_t K0max = K0 > H ? K0 : H;
  FSN_REQUIRE((size_t)T * R * 4 * ((size_t)H > K0max ? (size_t)H : K0max) < ((size_t)1 << 31), FSN_ERR_SHAPE,
              "lstm_train hook: T*R*4*max(H,K0) must stay below 2^31");
  return FSN_OK;
}
}  // namespace fsn

extern "C" size_t fsn_debug_lstm_train_workspace_bytes(int n_layers, int R, int T, int K0, int H, int precision) {
  if (dbg_lstm_check(n_layers, R, T, K0, H, precision)) return 0;
  DbgLstmWs w;
  carve_dbg_lstm(n_layers, R, T, K0, H, precision, nullptr, w);
  return w.bytes;
}

extern "C" int fsn_debug_lstm_train(const fsn_lstm_layer* layers, int n_layers, int R, int T, int K0, int H, int precision,
                                    const float* x, const float* dh_top, const float* dout, const float* fc_w, int O,
                                    float* h_top, float* dx, const fsn_lstm_grads* g, float* trace, void* workspace,
                                    size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  const int n = n_layers;
  int rc = dbg_lstm_check(n, R, T, K0, H, precision);
  if (rc) return rc;
  FSN_REQUIRE(layers && x && h_top && g, FSN_ERR_SHAPE, "lstm_train hook: null argument");
  FSN_REQUIRE(dh_top || dout, FSN_ERR_SHAPE, "lstm_train hook: no gradient on top (dh_top and dout both null)");
  FSN_REQUIRE(dout ? (fc_w && O >= 1) : (!fc_w && O == 0), FSN_ERR_SHAPE,
              "lstm_train hook: dout, fc_w and O >= 1 come together (O=%d)", O);
  for (int l = 0; l < n; ++l)
    FSN_REQUIRE(layers[l].w_ih && layers[l].w_hh && layers[l].b_ih && layers[l].b_hh && g[l].w_ih && g[l].w_hh && g[l].b_ih &&
                    g[l].b_hh,
                FSN_ERR_SHAPE, "lstm_train hook: null weight or gradient of layer %d", l);
  DbgLstmWs w;
  carve_dbg_lstm(n, R, T, K0, H, precision, workspace, w);
  FSN_REQUIRE(workspace && workspace_bytes >= w.bytes, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              w.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t TRH = (size_t)T * R * H;
  auto in_width = [&](int l) { return l == 0 ? K0 : H; };
  for (int l = 0; l < n; ++l) {
    const LayerHalf half{w.h16[l], l > 0 ? w.h16[l - 1] : nullptr, w.w16};
    if ((rc = layer_forward(precision, layers[l], l == 0 ? x : w.L[l - 1].H, R, in_width(l), H, T, w.L[l], w.rec, w.splitk,
                            &half, st)))
      return rc;
  }
  if ((rc = check_cuda(cudaMemcpyAsync(h_top, w.L[n - 1].H, TRH * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy")))
    return rc;
  LayerBwd L[DBG_MAX_LAYERS];
  for (int l = 0; l < n; ++l) {
    L[l] = LayerBwd{layers[l].w_ih, layers[l].w_hh, w.L[l], R, in_width(l), H, w.dh_rec[l], w.dc[l], w.whhT[l],
                    (l > 0 || dx) ? w.wihT[l] : nullptr, w.splitk};
    if ((rc = layer_bwd_transpose_weights(L[l], st))) return rc;
  }
  if ((rc = stack_bwd(L, n, T, dh_top, dout, fc_w, O, w.dh_mid[0], w.dh_mid[1], dx, st))) return rc;
  const WgradScratch wg{w.gT, w.xT, w.splitk, w.colsum, w.colsum_floats};
  for (int l = n - 1; l >= 0; --l)
    if ((rc = layer_weight_grads(L[l], T, l == 0 ? x : w.L[l - 1].H, g[l].w_ih, g[l].w_hh, g[l].b_ih, g[l].b_hh, wg, st)))
      return rc;
  if (trace)  // per layer: the saved hidden states [T,R,H], then dG [T,R,4H] (the gate buffer after BPTT)
    for (int l = 0; l < n; ++l) {
      float* dst = trace + (size_t)l * 5 * TRH;
      if ((rc = check_cuda(cudaMemcpyAsync(dst, w.L[l].H, TRH * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy")) ||
          (rc = check_cuda(cudaMemcpyAsync(dst + TRH, w.L[l].G, 4 * TRH * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy")))
        return rc;
    }
  return FSN_OK;
}

// ------------------------------------------------------------------------------------------ loss
namespace fsn {
constexpr int MSE_BLOCKS = 1024;

// the partition of an MSE over n elements: min(MSE_BLOCKS, ceil(n/256)) CTAs of 256 threads, grid-stride
__host__ __device__ inline int mse_blocks(size_t n) {
  const size_t nb = (n + 255) / 256;
  return nb > MSE_BLOCKS ? MSE_BLOCKS : (int)nb;
}

// loss = mean((cirm - crm)^2) with cirm [B,Fs,T,2] (trainer.py:49-54) and crm [B,2,Fs,T] (Model.forward);
// dcrm = 2 (crm - cirm) / n.  Stage 1: per-CTA partial sums; stage 2: fixed-order sum.
__global__ void mse_part_kernel(const float* __restrict__ cirm, const float* __restrict__ crm, int Fs, int T, size_t n,
                                float* __restrict__ dcrm, float* __restrict__ part) {
  __shared__ float sh[256];
  float a = 0.f;
  const float k = 2.0f / (float)n;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) {
    // i indexes crm [b,o,f,t]
    const int t = (int)(i % T);
    size_t q = i / T;
    const int f = (int)(q % Fs); q /= Fs;
    const int o = (int)(q & 1);
    const size_t b = q >> 1;
    const float dlt = crm[i] - cirm[((b * Fs + f) * T + t) * 2 + o];
    a = fmaf(dlt, dlt, a);
    if (dcrm) dcrm[i] = k * dlt;
  }
  a = cta_tree_sum256(a, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = a;
}

// stage 2 of one MSE: the nb partials summed in double in a fixed order, over n
__device__ __forceinline__ float mse_final(const float* __restrict__ part, int nb, size_t n) {
  __shared__ double sh[256];
  double a = 0.0;
  for (int i = threadIdx.x; i < nb; i += 256) a += (double)part[i];
  return (float)(cta_tree_sum256(a, sh) / (double)n);
}

__global__ void mse_final_kernel(const float* __restrict__ part, int nb, size_t n, float* __restrict__ loss) {
  const float v = mse_final(part, nb, n);
  if (threadIdx.x == 0) *loss = v;
}

// Per-clip cIRM loss (grid (MSE_BLOCKS, B)): clip b = blockIdx.y has T_b = 1 + lens[b]/hop of the T frames (all T
// without lens), n_b = 2 F T_b elements in crm's [o,f,t] order, and the partition of fsn_mse_loss at B = 1, T = T_b.
// Each element builds its cIRM value from the four spectra [B,F,T] (fsn_build_cirm's arithmetic) and subtracts it
// from crm [B,2,F,T] as mse_part_kernel does.  Partials at part[b * MSE_BLOCKS + CTA].
__global__ void cirm_mse_part_kernel(const float* __restrict__ nr, const float* __restrict__ ni,
                                     const float* __restrict__ cr, const float* __restrict__ ci,
                                     const float* __restrict__ crm, int F, int T, int hop, const int* __restrict__ lens,
                                     float* __restrict__ part) {
  __shared__ float sh[256];
  const int b = blockIdx.y;
  const int Tb = lens ? 1 + lens[b] / hop : T;
  const size_t n = (size_t)2 * F * Tb;
  const int nb = mse_blocks(n);
  if ((int)blockIdx.x >= nb) return;  // the whole CTA: no barrier is skipped
  const size_t plane = (size_t)F * T;
  const float* c = crm + (size_t)b * 2 * plane;
  float a = 0.f;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)nb * 256) {
    const int t = (int)(i % Tb);
    const size_t q = i / Tb;
    const int f = (int)(q % F);
    const int o = (int)(q / F);
    const size_t s = (size_t)b * plane + (size_t)f * T + t;
    const float2 m = cirm_f(nr[s], ni[s], cr[s], ci[s]);
    const float dlt = c[o * plane + (size_t)f * T + t] - (o ? m.y : m.x);
    a = fmaf(dlt, dlt, a);
  }
  a = cta_tree_sum256(a, sh);
  if (threadIdx.x == 0) part[(size_t)b * MSE_BLOCKS + blockIdx.x] = a;
}

__global__ void cirm_mse_final_kernel(const float* __restrict__ part, int F, int T, int hop, const int* __restrict__ lens,
                                      float* __restrict__ loss) {
  const int b = blockIdx.x;
  const size_t n = (size_t)2 * F * (lens ? 1 + lens[b] / hop : T);
  const float v = mse_final(part + (size_t)b * MSE_BLOCKS, mse_blocks(n), n);
  if (threadIdx.x == 0) loss[b] = v;
}

// workspace of fsn_cirm_mse_per_clip: the noisy and clean spectra [B,F,T], the partials, the length table
struct CirmMseWs { float *nr, *ni, *cr, *ci, *part; int* lens; };
static size_t carve_cirm_mse(void* base, int B, int F, int T, CirmMseWs& w) {
  Carver c(base);
  const size_t BFT = (size_t)B * F * T;
  w.nr = c.take<float>(BFT); w.ni = c.take<float>(BFT); w.cr = c.take<float>(BFT); w.ci = c.take<float>(BFT);
  w.part = c.take<float>((size_t)B * MSE_BLOCKS);
  w.lens = c.take<int>(B);
  return c.off;
}
}  // namespace fsn

extern "C" size_t fsn_mse_loss_scratch_bytes(void) { return MSE_BLOCKS * sizeof(float); }

extern "C" int fsn_mse_loss(const float* cirm, const float* crm, int B, int Fsub, int T, float* loss, float* dcrm,
                            void* scratch, size_t scratch_bytes, fsn_stream_t stream) {
  FSN_REQUIRE(B > 0 && Fsub > 0 && T > 0, FSN_ERR_SHAPE, "mse_loss: empty input");
  FSN_REQUIRE(scratch && scratch_bytes >= MSE_BLOCKS * sizeof(float), FSN_ERR_WORKSPACE, "mse_loss: scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)B * 2 * Fsub * T;
  const int nb = mse_blocks(n);
  mse_part_kernel<<<nb, 256, 0, st>>>(cirm, crm, Fsub, T, n, dcrm, (float*)scratch);
  FSN_CHECK_LAUNCH("mse_part_kernel");
  mse_final_kernel<<<1, 256, 0, st>>>((const float*)scratch, nb, n, loss);
  FSN_CHECK_LAUNCH("mse_final_kernel");
  return FSN_OK;
}

extern "C" size_t fsn_cirm_mse_per_clip_workspace_bytes(int B, int L_max, int n_fft, int hop) {
  if (stft_check(B, L_max, n_fft, hop, n_fft, nullptr, 0)) return 0;  // the call's own checks, win_length aside
  CirmMseWs w;
  return carve_cirm_mse(nullptr, B, n_fft / 2 + 1, 1 + L_max / hop, w);
}

extern "C" int fsn_cirm_mse_per_clip(const float* noisy_wav, const float* clean_wav, const int32_t* lengths, int B,
                                     int L_max, int n_fft, int hop, int win_length, const float* crm, float* loss,
                                     void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  launch_counter() = 0;
  int rc = stft_check(B, L_max, n_fft, hop, win_length, nullptr, 0);
  if (rc) return rc;
  FSN_REQUIRE(noisy_wav && clean_wav && crm, FSN_ERR_SHAPE, "cirm_mse_per_clip: null input");
  if ((rc = wav_check(lengths, B, L_max, n_fft, false, loss, "cirm_mse_per_clip"))) return rc;
  const int F = n_fft / 2 + 1, T = 1 + L_max / hop;
  CirmMseWs w;
  const size_t bytes = carve_cirm_mse(workspace, B, F, T, w);
  FSN_REQUIRE(workspace && workspace_bytes >= bytes, FSN_ERR_WORKSPACE, "cirm_mse_per_clip: workspace too small: %zu < %zu",
              workspace_bytes, bytes);
  const cudaStream_t st = (cudaStream_t)stream;
  WavWs lw = {nullptr, nullptr, nullptr, nullptr, w.lens};
  if ((rc = wav_prologue(lengths, B, lw, st))) return rc;
  if ((rc = stft_launch(noisy_wav, B, L_max, n_fft, hop, win_length, nullptr, nullptr, w.nr, w.ni, nullptr, 0, st,
                        lw.lens)) ||
      (rc = stft_launch(clean_wav, B, L_max, n_fft, hop, win_length, nullptr, nullptr, w.cr, w.ci, nullptr, 0, st,
                        lw.lens)))
    return rc;
  cirm_mse_part_kernel<<<dim3(MSE_BLOCKS, B), 256, 0, st>>>(w.nr, w.ni, w.cr, w.ci, crm, F, T, hop, lw.lens, w.part);
  FSN_CHECK_LAUNCH("cirm_mse_part_kernel");
  cirm_mse_final_kernel<<<B, 256, 0, st>>>(w.part, F, T, hop, lw.lens, loss);
  FSN_CHECK_LAUNCH("cirm_mse_final_kernel");
  return FSN_OK;
}

// ------------------------------------------------------------------------------------------ clip + Adam
namespace fsn {
constexpr int ADAM_CHUNKS = 32;

__global__ void gradsq_part_kernel(const fsn_param_list L, float* __restrict__ part) {
  __shared__ float sh[256];
  const int ti = blockIdx.y;
  const float* g = L.grad[ti];
  const int64_t n = L.numel[ti];
  float a = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) a = fmaf(g[i], g[i], a);
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[ti * ADAM_CHUNKS + blockIdx.x] = sh[0];
}

// out[0] = total L2 norm of (grad * grad_scale); out[1] = grad_scale * min(1, max_norm / (norm + 1e-6))
__global__ void gradnorm_final_kernel(const float* __restrict__ part, int n, float grad_scale, float max_norm,
                                      float* __restrict__ out) {
  __shared__ double sh[256];
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) a += (double)part[i];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float norm = (float)sqrt(sh[0]) * grad_scale;
    float coef = max_norm > 0.f ? max_norm / (norm + 1e-6f) : 1.f;
    if (coef > 1.f) coef = 1.f;
    out[0] = norm;
    out[1] = coef * grad_scale;
  }
}

// bias corrections of each tensor's own step: 1 - beta1^step and sqrt(1 - beta2^step), computed on the host in float
struct AdamBias {
  float bc1[FSN_MAX_PARAM_TENSORS];
  float bc2_sqrt[FSN_MAX_PARAM_TENSORS];
};

// torch.optim.Adam single-tensor update (no weight decay / amsgrad); the clipped, scaled gradient is written back
__global__ void adam_kernel(const fsn_param_list L, const AdamBias bias, const float* __restrict__ coef_ptr, float lr,
                            float b1, float b2, float eps) {
  const int ti = blockIdx.y;
  float* p = L.param[ti];
  float* g = L.grad[ti];
  float* m = L.exp_avg[ti];
  float* v = L.exp_avg_sq[ti];
  const int64_t n = L.numel[ti];
  const float coef = coef_ptr[1];
  const float step_size = lr / bias.bc1[ti];
  const float bc2_sqrt = bias.bc2_sqrt[ti];
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const float gi = g[i] * coef;
    g[i] = gi;
    const float mi = m[i] * b1 + (1.f - b1) * gi;   // lerp(m, g, 1 - b1)
    const float vi = v[i] * b2 + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] -= step_size * (mi / denom);
  }
}
}  // namespace fsn

extern "C" size_t fsn_clip_adam_scratch_bytes(void) { return (FSN_MAX_PARAM_TENSORS * ADAM_CHUNKS + 2) * sizeof(float); }

extern "C" int fsn_clip_adam_steps(const fsn_param_list* L, float max_norm, float grad_scale, float lr, float beta1,
                                   float beta2, float eps, const int* steps, float* norm_out, void* scratch,
                                   size_t scratch_bytes, fsn_stream_t stream) {
  FSN_REQUIRE(L && L->n > 0 && L->n <= FSN_MAX_PARAM_TENSORS, FSN_ERR_SHAPE, "clip_adam: 1..%d tensors",
              FSN_MAX_PARAM_TENSORS);
  FSN_REQUIRE(steps, FSN_ERR_SHAPE, "clip_adam: no step table");
  for (int i = 0; i < L->n; ++i)
    FSN_REQUIRE(steps[i] >= 1, FSN_ERR_SHAPE, "clip_adam: step starts at 1 (tensor %d has step %d)", i, steps[i]);
  FSN_REQUIRE(scratch && scratch_bytes >= fsn_clip_adam_scratch_bytes(), FSN_ERR_WORKSPACE, "clip_adam: scratch too small");
  AdamBias bias;
  for (int i = 0; i < L->n; ++i) {
    bias.bc1[i] = 1.f - powf(beta1, (float)steps[i]);
    bias.bc2_sqrt[i] = sqrtf(1.f - powf(beta2, (float)steps[i]));
  }
  for (int i = L->n; i < FSN_MAX_PARAM_TENSORS; ++i) bias.bc1[i] = bias.bc2_sqrt[i] = 1.f;  // unread
  cudaStream_t st = (cudaStream_t)stream;
  float* part = (float*)scratch;
  float* res = norm_out ? norm_out : part + FSN_MAX_PARAM_TENSORS * ADAM_CHUNKS;
  gradsq_part_kernel<<<dim3(ADAM_CHUNKS, L->n), 256, 0, st>>>(*L, part);
  FSN_CHECK_LAUNCH("gradsq_part_kernel");
  gradnorm_final_kernel<<<1, 256, 0, st>>>(part, L->n * ADAM_CHUNKS, grad_scale, max_norm, res);
  FSN_CHECK_LAUNCH("gradnorm_final_kernel");
  adam_kernel<<<dim3(ADAM_CHUNKS * 4, L->n), 256, 0, st>>>(*L, bias, res, lr, beta1, beta2, eps);
  FSN_CHECK_LAUNCH("adam_kernel");
  return FSN_OK;
}

// every tensor at the same step: the bias corrections, and so every output bit, of the single-step launcher
extern "C" int fsn_clip_adam(const fsn_param_list* L, float max_norm, float grad_scale, float lr, float beta1,
                             float beta2, float eps, int step, float* norm_out, void* scratch, size_t scratch_bytes,
                             fsn_stream_t stream) {
  FSN_REQUIRE(L && L->n > 0 && L->n <= FSN_MAX_PARAM_TENSORS, FSN_ERR_SHAPE, "clip_adam: 1..%d tensors",
              FSN_MAX_PARAM_TENSORS);
  FSN_REQUIRE(step >= 1, FSN_ERR_SHAPE, "clip_adam: step starts at 1");
  int steps[FSN_MAX_PARAM_TENSORS];
  for (int i = 0; i < L->n; ++i) steps[i] = step;
  return fsn_clip_adam_steps(L, max_norm, grad_scale, lr, beta1, beta2, eps, steps, norm_out, scratch, scratch_bytes,
                             stream);
}

// ---- unit-test hook of the second norm + drop_band backward (include/fsn_b200.h): the launchers fsn_train_backward
// runs, every argument checked before any CUDA call
extern "C" int fsn_debug_norm_unfold_bwd(const float* dX, const float* X, const float* fbz, const float* scale, int cum,
                                         int B, int F, int G, int Tp, int Ns, float cnt2, int act, float* mid, float* dz,
                                         fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(dX && X && fbz && scale && mid && dz, FSN_ERR_SHAPE, "norm/unfold backward hook: null argument");
  FSN_REQUIRE(B > 0 && F > 0 && Tp > 0 && G >= 0, FSN_ERR_SHAPE, "norm/unfold backward hook: bad shape B=%d F=%d Tp=%d G=%d",
              B, F, Tp, G);
  FSN_REQUIRE(G <= 1 || (B > G && F >= G), FSN_ERR_SHAPE, "norm/unfold backward hook: drop_band needs B > G and F >= G");
  FSN_REQUIRE(Ns >= 0 && Ns < F, FSN_ERR_SHAPE, "norm/unfold backward hook: reflect padding needs 0 <= Ns < F");
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "norm/unfold backward hook: unknown act %d", act);
  FSN_REQUIRE(cum || cnt2 > 0.f, FSN_ERR_SHAPE, "norm/unfold backward hook: cnt2 must be positive");
  const int Fsub = G > 1 ? F / G : F, R = B * Fsub, K = 2 * Ns + 2;
  FSN_REQUIRE((size_t)Tp * R * K < ((size_t)1 << 31) && (size_t)Tp * B * F < ((size_t)1 << 31), FSN_ERR_SHAPE,
              "norm/unfold backward hook: tensors must stay below 2^31 elements");
  const RowMap map{B, F, Fsub, G > 1 ? G : 1};
  const cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (cum) {
    if ((rc = train_cum_unit_bwd_launch(dX, X, scale, Tp, R, K, mid, st))) return rc;
    return train_dfbz_cum_launch(mid, fbz, map, Tp, R, act, dz, st);
  }
  if ((rc = train_dot_launch(dX, X, Tp, R, Fsub, K, B, mid, st))) return rc;
  return train_dfbz_launch(dX, fbz, scale, mid, map, Tp, R, K, cnt2, act, dz, st);
}

// ---- unit-test hook of the second forgetting norm + drop_band backward (include/fsn_b200.h): train_forget_bwd_launch as
// fsn_train_backward runs it, every argument checked before any CUDA call
extern "C" int fsn_debug_forgetting_bwd(const float* dX, const float* X, const float* fbz, const float* scale, int B, int F,
                                        int G, int Tp, int Ns, int act, float* mid, float* dz, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(dX && X && fbz && scale && mid && dz, FSN_ERR_SHAPE, "forgetting backward hook: null argument");
  FSN_REQUIRE(B > 0 && F > 0 && Tp > 0 && G >= 0, FSN_ERR_SHAPE, "forgetting backward hook: bad shape B=%d F=%d Tp=%d G=%d",
              B, F, Tp, G);
  FSN_REQUIRE(G <= 1 || (B > G && F >= G), FSN_ERR_SHAPE, "forgetting backward hook: drop_band needs B > G and F >= G");
  FSN_REQUIRE(Ns >= 0 && Ns < F, FSN_ERR_SHAPE, "forgetting backward hook: reflect padding needs 0 <= Ns < F");
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "forgetting backward hook: unknown act %d", act);
  const int Fsub = G > 1 ? F / G : F, R = B * Fsub, K = 2 * Ns + 2;
  FSN_REQUIRE((size_t)Tp * R * K < ((size_t)1 << 31) && (size_t)Tp * B * F < ((size_t)1 << 31), FSN_ERR_SHAPE,
              "forgetting backward hook: tensors must stay below 2^31 elements");
  const RowMap map{B, F, Fsub, G > 1 ? G : 1};
  return train_forget_bwd_launch(dX, X, fbz, scale, map, Tp, R, K, (float)F * K, act, mid, dz, (cudaStream_t)stream);
}

// ---- unit-test hook of the per-clip statistics of the training steps (include/fsn_b200.h)
extern "C" int fsn_debug_train_stats(const float* x, int tm, int B, int F, int T, int N, float* sums, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(x && sums, FSN_ERR_SHAPE, "train stats hook: null argument");
  FSN_REQUIRE(B > 0 && F > 0 && T > 0 && (size_t)B * F * T < ((size_t)1 << 31) && (size_t)F * T < ((size_t)1 << 31),
              FSN_ERR_SHAPE, "train stats hook: bad shape B=%d F=%d T=%d", B, F, T);
  FSN_REQUIRE(N >= 0 && N < F, FSN_ERR_SHAPE, "train stats hook: reflect padding needs 0 <= N < F");
  float2* s = reinterpret_cast<float2*>(sums);
  const cudaStream_t st = (cudaStream_t)stream;
  return tm ? train_tm_stats_launch(x, B, F, T, N, s, st) : train_mag_stats_launch(x, B, F, T, N, s, st);
}

// ---- unit-test hooks of the fp32 GEMM layer of the training steps (include/fsn_b200.h): each runs the launch function
// its callers use, every argument checked before any CUDA call
extern "C" int fsn_debug_sgemm(int ta, const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M,
                               int N, int K, int accumulate, float* scratch, int64_t scratch_floats, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(A && B && C, FSN_ERR_SHAPE, "sgemm hook: null argument");
  FSN_REQUIRE(M > 0 && N > 0 && K > 0, FSN_ERR_SHAPE, "sgemm hook: bad shape M=%d N=%d K=%d", M, N, K);
  FSN_REQUIRE(lda >= (ta ? M : K) && ldb >= N && ldc >= N, FSN_ERR_SHAPE, "sgemm hook: a leading dimension is below its row");
  FSN_REQUIRE((N + 63) / 64 <= 65535, FSN_ERR_SHAPE, "sgemm hook: N=%d exceeds the grid", N);
  FSN_REQUIRE(scratch_floats >= 0 && (scratch || scratch_floats == 0), FSN_ERR_WORKSPACE,
              "sgemm hook: scratch_floats without scratch");
  return sgemm_launch(ta != 0, A, (size_t)lda, B, (size_t)ldb, C, (size_t)ldc, M, N, K, accumulate != 0, scratch,
                      (size_t)scratch_floats, (cudaStream_t)stream);
}

extern "C" int fsn_debug_colsum(const float* X, int64_t rows, int cols, int64_t ldx, float* out, float* out2, float* scratch,
                                int64_t scratch_floats, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(X && out, FSN_ERR_SHAPE, "colsum hook: null argument");
  FSN_REQUIRE(rows > 0 && cols > 0 && ldx >= cols, FSN_ERR_SHAPE, "colsum hook: bad shape rows=%lld cols=%d ldx=%lld",
              (long long)rows, cols, (long long)ldx);
  FSN_REQUIRE(scratch && scratch_floats > 0, FSN_ERR_WORKSPACE, "colsum hook: no scratch");
  return colsum_launch(X, (size_t)rows, cols, (size_t)ldx, out, out2, scratch, (size_t)scratch_floats, (cudaStream_t)stream);
}

extern "C" int fsn_debug_small_out_wgrad(const float* dout, const float* Hm, int64_t rows, int H, float* dW, float* scratch,
                                         int64_t scratch_floats, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(dout && Hm && dW, FSN_ERR_SHAPE, "small_out_wgrad hook: null argument");
  FSN_REQUIRE(rows > 0 && H > 0, FSN_ERR_SHAPE, "small_out_wgrad hook: bad shape rows=%lld H=%d", (long long)rows, H);
  FSN_REQUIRE(scratch && scratch_floats > 0, FSN_ERR_WORKSPACE, "small_out_wgrad hook: no scratch");
  return small_out_wgrad_launch(dout, Hm, (size_t)rows, H, dW, scratch, (size_t)scratch_floats, (cudaStream_t)stream);
}

extern "C" int fsn_debug_transpose(const float* in, int64_t rows, int cols, float* out, fsn_stream_t stream) {
  launch_counter() = 0;
  FSN_REQUIRE(in && out, FSN_ERR_SHAPE, "transpose hook: null argument");
  FSN_REQUIRE(rows > 0 && cols > 0 && (rows + 31) / 32 < ((int64_t)1 << 31) && (cols + 31) / 32 <= 65535, FSN_ERR_SHAPE,
              "transpose hook: bad shape rows=%lld cols=%d", (long long)rows, cols);
  return transpose_launch(in, (size_t)rows, cols, out, (cudaStream_t)stream);
}
