// One LSTM layer for a SMALL batch of sequences (rows = clips) on the tensor cores (wgmma, sm_90a):
//   1. the input projection of ALL steps hoisted into one GEMM  P[r,t,:] = x[r,t,:] W_ih^T   (tgemm_tma_kernel, tf32;
//      three passes on tf32 hi/lo splits for the fp32 error class), and
//   2. the recurrence  gates_t = P_t + b + h_{t-1} W_hh^T  as ONE persistent cooperative kernel (this file).
//
// Reference semantics: audio_zen/model/module/sequence_model.py:52-58,117 (nn.LSTM, gate order i,f,g,o, zero initial
// state) as used for the full-band stacks (recipes/dns_interspeech_2020/fullsubnet/model.py:43-51,92-95; rows = clips).
//
// Mapping of the recurrence.  The batch is small (<= 128 rows per group) and the steps are serial, so the HIDDEN
// dimension is spread over the chip: CTA j of a group owns 8 hidden units = 32 gate columns and keeps that slice of
// W_hh resident in shared memory for the whole sequence (fp16, K-major 128B-swizzled; compensated mode: hi and lo
// parts).  Per step every CTA needs ALL of h_{t-1}: the consumers publish h_t as fp16 (hi [+ lo]) in a ping-pong array
// in global memory (it lives in L2), a per-group counter is the step barrier, and each CTA's producer warp streams the
// [128 rows x K] state through a TMA ring.  Rows sit on the M side of the MMA (two m64 halves per warpgroup):
//     D[64 rows, 32 | 64 gate columns] += h_hi[64, 16] . [W_hi ; W_lo]^T   (N = 64: the lo product lands in
//     D[64 rows, 32]                    += h_lo[64, 16] . W_hi^T             columns 32..63 and is added in the cell)
// Column block j (8 columns) of D is gate j % 4, so the thread that holds a row's fragment holds all four gates of
// the same two units: c stays in 8 registers (4 rows x 2 units), no exchange.  Groups of 64 CTAs cover 128 clips
// each with H = 512.
//
// CARRY (lstm_rec_tc_carry_kernel, chunked streaming, DESIGN 4.14): the recurrence continued from a carried state.  The
// host writes h_{-1} as hi [/ lo] into the parity buffer step 0 reads (rec_carry_init_kernel, instead of the memset
// zeros), so step 0 runs its MMAs like every later step; c_{-1} is loaded into the consumer registers.  A row restarting
// at step j drops its c there and publishes a zero h_{j-1}; c after step fin_step is stored (h is in hall anyway).
#include <string.h>
#include <stdlib.h>

#include "fsn_internal.cuh"
#include "fsn_tc_ptx.cuh"
#include "fsn_wgmma.cuh"

namespace fsn {
namespace rec {
using namespace ptx;

constexpr int MR = 128;               // rows per group (two m64 MMA halves)
constexpr int U = 8;                  // hidden units per CTA
constexpr int NG = 4 * U;             // gate columns per CTA
constexpr int KB = 64;                // k-block: one 128-byte swizzled row of fp16
constexpr int A_TILE = MR * KB * 2;   // 16 KB
constexpr int NTHREADS = 160;         // warps 0-3: MMA + cell (one warpgroup), warp 4: TMA producer
constexpr int MAX_STAGES = 6;
constexpr int MIN_H = 64;             // smallest hidden size: see lstm_rec_tc_scratch_bytes

struct Bars {
  uint64_t full[MAX_STAGES], empty[MAX_STAGES];
};

struct Args {
  const float* w_hh; const float* b_ih; const float* b_hh;   // [4H,H], [4H], [4H] (PyTorch layout)
  const float* P; size_t p_row, p_t;                          // P[r*p_row + t*p_t + gate*H + u]
  float* hall; size_t h_row, h_t;                             // hall[r*h_row + t*h_t + u]
  __half* state;                                              // [2 parity][PARTS][Rpad][Kp]
  unsigned int* barrier;                                      // one counter per group, 32 words apart
  int R, T, H, Kp, Rpad, C, stages, fence_all;
};
// CARRY only: c of row r at c_init / c_fin [r * c_row + u], restart step of row r at restart[r], c stored after fin_step
struct CarryArgs {
  const float* c_init; float* c_fin; size_t c_row;
  const int* restart;
  int fin_step;
};

template <bool X3> __device__ __forceinline__ float act_sigmoid(float x) {
  return X3 ? 1.0f / (1.0f + expf(-x)) : fast_sigmoid(x);
}
template <bool X3> __device__ __forceinline__ float act_tanh(float x) {
  return X3 ? 1.0f - 2.0f / (1.0f + expf(2.0f * x)) : fast_tanh(x);
}

// every CARRY branch below is `if constexpr` or folds away: lstm_rec_tc_kernel is the code it was before the policy
template <bool X3, bool CARRY>
__device__ __forceinline__ void lstm_rec_tc_body(const CUtensorMap& tmap, const Args& a, const CarryArgs& io) {
  constexpr int PARTS = X3 ? 2 : 1;
  constexpr int STAGE_BYTES = PARTS * A_TILE;
  constexpr int WB_ROWS = PARTS * NG;          // rows of the resident weight operand per k-block: [W_hi ; W_lo]
  constexpr int WB_BYTES = WB_ROWS * 128;
  constexpr int NACC = WB_ROWS / 2;            // accumulator registers per m64 half
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int nkb = a.Kp / KB;
  uint8_t* ring = smem;
  uint8_t* wsm = smem + (size_t)a.stages * STAGE_BYTES;
  Bars& bars = *reinterpret_cast<Bars*>(wsm + (size_t)nkb * WB_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x / a.C, j = blockIdx.x - g * a.C;   // group, unit slice
  const int u0 = j * U;
  const int H = a.H, T = a.T;
  unsigned int* counter = a.barrier + g * 32;

  // ---------------- one-time setup: barriers, resident weight slice
  if (threadIdx.x == 0) {
    for (int s = 0; s < a.stages; ++s) { mbar_init(&bars.full[s], 1); mbar_init(&bars.empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // weight operand: k-block kb = rows [W_hi (gate col n = gate*8 + ul) ; W_lo] x 64 k, 128B swizzle
  for (int idx = threadIdx.x; idx < nkb * NG * (KB / 8); idx += NTHREADS) {
    const int kb = idx / (NG * (KB / 8));
    const int rem = idx - kb * (NG * (KB / 8));
    const int n = rem / (KB / 8), ch = rem - n * (KB / 8);
    const int gate = n / U, u = u0 + (n % U);
    __half hi[8], lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = kb * KB + ch * 8 + e;
      const float w = (u < H && k < H) ? a.w_hh[((size_t)gate * H + u) * H + k] : 0.f;
      hi[e] = __float2half_rn(w);
      lo[e] = __float2half_rn(w - __half2float(hi[e]));
    }
    uint8_t* blk = wsm + (size_t)kb * WB_BYTES;
    *reinterpret_cast<uint4*>(blk + swz128_off(n, ch * 8)) = *reinterpret_cast<const uint4*>(hi);
    if (X3) *reinterpret_cast<uint4*>(blk + swz128_off(NG + n, ch * 8)) = *reinterpret_cast<const uint4*>(lo);
  }
  fence_proxy_async();
  __syncthreads();

  if (warp == 4) {
    // ================= producer: after the group has published h_{p-1}, stream it through the ring
    uint32_t it = 0;
    for (int p = CARRY ? 0 : 1; p < T; ++p) {
      if (lane == 0) {
        const unsigned int target = (unsigned int)a.C * (unsigned int)p;
        unsigned int v, spins = 0;
        do {
          asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
          if (++spins > (1u << 27)) asm volatile("trap;");  // a lost publication traps instead of hanging
        } while (v < target);
      }
      __syncwarp();
      fence_proxy_async();  // the TMA (async proxy) reads below come after the acquire above
      const int par = CARRY ? ((p + 1) & 1) : ((p - 1) & 1);
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const uint32_t s = it % (uint32_t)a.stages, use = it / (uint32_t)a.stages;
        mbar_wait<false>(&bars.empty[s], (use & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&bars.full[s], STAGE_BYTES);
#pragma unroll
          for (int part = 0; part < PARTS; ++part)
            tma_load_2d(ring + (size_t)s * STAGE_BYTES + part * A_TILE, &tmap, kb * KB,
                        (par * PARTS + part) * a.Rpad + g * MR, &bars.full[s]);
        }
        __syncwarp();
      }
    }
  } else {
    // ================= consumers: MMA, then the cell on the fragment.  Thread rows: 16 warp + lane/4 + 8 hh + 64 half;
    // units u0 + 2 (lane % 4) + e; gate = column block % 4 (block + 4: the lo product of X3)
    const int q = warp;
    const int ul0 = 2 * (lane & 3);
    const bool vec_ok = (H & 1) == 0 && (a.p_row & 1) == 0 && (a.p_t & 1) == 0 && (a.h_row & 1) == 0 && (a.h_t & 1) == 0;
    float bias[4][2];
#pragma unroll
    for (int gate = 0; gate < 4; ++gate)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int u = u0 + ul0 + e;
        bias[gate][e] = (u < H) ? a.b_ih[gate * H + u] + a.b_hh[gate * H + u] : 0.f;
      }
    float c[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) c[i][0] = c[i][1] = 0.f;
    const int nu = (H - u0 < U) ? (H - u0) : U;  // real units of this CTA
    const bool u_ok0 = ul0 < nu, u_ok1 = ul0 + 1 < nu;
    int rst[4] = {-1, -1, -1, -1};
    if constexpr (CARRY) {
#pragma unroll
      for (int rs = 0; rs < 4; ++rs) {
        const int r = g * MR + 64 * (rs >> 1) + 16 * q + (lane >> 2) + 8 * (rs & 1);
        if (r < a.R) {
          rst[rs] = io.restart[r];
          const float* cp = io.c_init + (size_t)r * io.c_row + u0 + ul0;
          if (u_ok0) c[rs][0] = cp[0];
          if (u_ok1) c[rs][1] = cp[1];
        }
      }
    }
    uint32_t it = 0;
    const uint32_t wbase = smem_u32(wsm), rbase = smem_u32(ring);
    for (int p = 0; p < T; ++p) {
      float pre[4][4][2];  // [row slot][gate][unit]
#pragma unroll
      for (int rs = 0; rs < 4; ++rs) {  // input projection of this step (loads in flight under the MMAs)
        const int r = g * MR + 64 * (rs >> 1) + 16 * q + (lane >> 2) + 8 * (rs & 1);
        const bool valid = r < a.R;
        const float* pp = a.P + (size_t)r * a.p_row + (size_t)p * a.p_t + u0 + ul0;
#pragma unroll
        for (int gate = 0; gate < 4; ++gate) {
          if (valid && vec_ok && u_ok1) {
            const float2 v = __ldg(reinterpret_cast<const float2*>(pp + (size_t)gate * H));
            pre[rs][gate][0] = v.x; pre[rs][gate][1] = v.y;
          } else {
            pre[rs][gate][0] = (valid && u_ok0) ? __ldg(pp + (size_t)gate * H) : 0.f;
            pre[rs][gate][1] = (valid && u_ok1) ? __ldg(pp + (size_t)gate * H + 1) : 0.f;
          }
        }
      }
      if (CARRY || p > 0) {
        float acc[2][NACC];
        float accl[2][NG / 2];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
          for (int i = 0; i < NACC; ++i) acc[hf][i] = 0.f;
#pragma unroll
          for (int i = 0; i < NG / 2; ++i) accl[hf][i] = 0.f;
          wg::fence_operand(acc[hf]);
          wg::fence_operand(accl[hf]);
        }
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const uint32_t s = it % (uint32_t)a.stages, use = it / (uint32_t)a.stages;
          mbar_wait_mma(&bars.full[s], use & 1);
          wg::fence();
          const uint32_t sa = rbase + s * STAGE_BYTES;
          const uint64_t wd = wg::desc_sw128(wbase + (uint32_t)kb * WB_BYTES);
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const uint64_t ad = wg::desc_sw128(sa + hf * (64 * 128));
#pragma unroll
            for (int k = 0; k < KB / 16; ++k) {
              if constexpr (X3) {
                wg::mma_f16_n64(acc[hf], ad + (uint64_t)(2 * k), wd + (uint64_t)(2 * k), 1u);
                wg::mma_f16_n32(accl[hf], ad + (uint64_t)((A_TILE >> 4) + 2 * k), wd + (uint64_t)(2 * k), 1u);
              } else {
                wg::mma_f16_n32(acc[hf], ad + (uint64_t)(2 * k), wd + (uint64_t)(2 * k), 1u);
              }
            }
          }
          wg::commit();
          wg::wait<0>();
          if (lane == 0) mbar_arrive(&bars.empty[s]);
        }
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          wg::fence_operand(acc[hf]);
          wg::fence_operand(accl[hf]);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int gate = 0; gate < 4; ++gate)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                float v = acc[hf][4 * gate + 2 * hh + e];
                if (X3) v += acc[hf][4 * (gate + 4) + 2 * hh + e] + accl[hf][4 * gate + 2 * hh + e];
                pre[2 * hf + hh][gate][e] += v;
              }
        }
      }
#pragma unroll
      for (int rs = 0; rs < 4; ++rs) {
        const int r = g * MR + 64 * (rs >> 1) + 16 * q + (lane >> 2) + 8 * (rs & 1);
        float h[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float gi = pre[rs][0][e] + bias[0][e], gf = pre[rs][1][e] + bias[1][e];
          const float gg = pre[rs][2][e] + bias[2][e], go = pre[rs][3][e] + bias[3][e];
          const float cp = (CARRY && p == rst[rs]) ? 0.f : c[rs][e];
          const float cn = act_sigmoid<X3>(gf) * cp + act_sigmoid<X3>(gi) * act_tanh<X3>(gg);
          c[rs][e] = cn;
          h[e] = act_sigmoid<X3>(go) * act_tanh<X3>(cn);
        }
        if (r < a.R) {
          float* hp = a.hall + (size_t)r * a.h_row + (size_t)p * a.h_t + u0 + ul0;
          if (vec_ok && u_ok1) {
            *reinterpret_cast<float2*>(hp) = make_float2(h[0], h[1]);
          } else {
            if (u_ok0) hp[0] = h[0];
            if (u_ok1) hp[1] = h[1];
          }
          if constexpr (CARRY) {
            if (p == io.fin_step) {
              float* cf = io.c_fin + (size_t)r * io.c_row + u0 + ul0;
              if (u_ok0) cf[0] = c[rs][0];
              if (u_ok1) cf[1] = c[rs][1];
            }
          }
          if (p + 1 < T) {  // publish h_p for the next step: fp16 hi (and lo)
            const bool zero = CARRY && rst[rs] == p + 1;  // the row enters step p + 1 with zero state
            const float v0 = (u_ok0 && !zero) ? h[0] : 0.f, v1 = (u_ok1 && !zero) ? h[1] : 0.f;
            const __half2 hi = __floats2half2_rn(v0, v1);
            const __half2 lo = __floats2half2_rn(v0 - __low2float(hi), v1 - __high2float(hi));
            __half* sp = a.state + ((size_t)((p & 1) * PARTS) * a.Rpad + r) * a.Kp + u0 + ul0;
            *reinterpret_cast<__half2*>(sp) = hi;
            if (X3) *reinterpret_cast<__half2*>(sp + (size_t)a.Rpad * a.Kp) = lo;
          }
        }
      }
      if (p + 1 < T) {
        // publish h_p: CTA-scope barrier over the 128 writers, then ONE gpu-scope fence (cumulative over the writes
        // observed through the barrier - the grid.sync pattern) + async-proxy fence + release by the arriving thread.
        // FSN_REC_FENCE_ALL=1 (debug) makes every writer fence for itself.
        if (a.fence_all) { __threadfence(); fence_proxy_async(); }
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (threadIdx.x == 64) {
          __threadfence();
          fence_proxy_async();
          asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
        }
      }
    }
  }
}

template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) lstm_rec_tc_kernel(const __grid_constant__ CUtensorMap tmap, const Args a) {
  lstm_rec_tc_body<X3, false>(tmap, a, CarryArgs{});
}

template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) lstm_rec_tc_carry_kernel(const __grid_constant__ CUtensorMap tmap,
                                                                       const Args a, const CarryArgs io) {
  lstm_rec_tc_body<X3, true>(tmap, a, io);
}

// h_{-1} of rows [0, R) (row r at h[r * h_row], zero where the row restarts at step 0) into parity 1 of the fp16 state
// [2 parity][parts][Rpad][Kp]: hi = rn(h), lo = rn(h - hi), the split the consumers publish h with
__global__ void rec_carry_init_kernel(const float* __restrict__ h, size_t h_row, const int* __restrict__ restart, int R, int H,
                                      int Kp, int Rpad, int parts, __half* __restrict__ state) {
  const size_t n = (size_t)R * H;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / H), k = (int)(i - (size_t)r * H);
    const float v = restart[r] == 0 ? 0.f : h[(size_t)r * h_row + k];
    const __half hi = __float2half_rn(v);
    __half* sp = state + ((size_t)parts * Rpad + r) * Kp + k;
    sp[0] = hi;
    if (parts > 1) sp[(size_t)Rpad * Kp] = __float2half_rn(v - __half2float(hi));
  }
}

// Operand preparation for the tf32 GEMM.  v = in[r, k] * scale.
//   cat == 0: out[r, :Kp] = v (zero padded to Kp): plain scaled, 16-byte aligned copy, single-pass GEMM.
//   cat != 0: compensated GEMM as ONE pass over a 3x longer K: hi = tf32-truncated v (what the tensor core reads),
//             lo = v - hi (exact); the A operand (cat == 1) is laid out [hi | lo | hi], the B operand (cat == 2)
//             [hi | hi | lo], so that  A' B'^T = hi.hi + lo.hi + hi.lo  - the product to ~2^-21, one output write.
// row_scale index of row r: r / rows_per_scale (per clip), or with scale_B > 0 the time-major entry
// (r % rows_per_scale) * scale_B + r / rows_per_scale of a [T', B] table (cumulative norm).
__global__ void split_tf32_kernel(const float* __restrict__ in, size_t rows, int K, size_t ldi, const float* __restrict__ row_scale,
                                  int rows_per_scale, int scale_B, float* __restrict__ out, int Kp, int cat) {
  const size_t n = rows * (size_t)Kp;
  const size_t ldo = cat ? (size_t)3 * Kp : (size_t)Kp;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / Kp;
    const int k = (int)(i - r * Kp);
    float v = 0.f;
    if (k < K) {
      v = in[r * ldi + k];
      if (row_scale)
        v *= scale_B > 0 ? row_scale[(r % rows_per_scale) * scale_B + r / rows_per_scale] : row_scale[r / rows_per_scale];
    }
    float* o = out + r * ldo + k;
    if (cat) {
      const float hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
      const float lo = v - hi;
      o[0] = hi;
      o[Kp] = (cat == 1) ? lo : hi;
      o[2 * Kp] = (cat == 1) ? hi : lo;
    } else {
      o[0] = v;
    }
  }
}

// x[r, :N] = act(x[r, :N] + bias[:N]) in place, row stride ld
__global__ void bias_act_kernel(float* __restrict__ x, size_t rows, int N, size_t ld, const float* __restrict__ bias, int act) {
  const size_t n = rows * (size_t)N;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / N;
    const int c = (int)(i - r * N);
    float v = x[r * ld + c] + (bias ? bias[c] : 0.f);
    switch (act) {
      case FSN_ACT_RELU: v = fmaxf(v, 0.f); break;
      case FSN_ACT_TANH: v = tanhf(v); break;
      case FSN_ACT_RELU6: v = fminf(fmaxf(v, 0.f), 6.f); break;
      default: break;
    }
    x[r * ld + c] = v;
  }
}

static size_t smem_bytes(int Kp, bool x3, int stages) {
  const int parts = x3 ? 2 : 1;
  return (size_t)stages * parts * A_TILE + (size_t)(Kp / KB) * parts * NG * 128 + sizeof(Bars) + 1024;
}

}  // namespace rec

static int rec_sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// tensor-core recurrence available for hidden size H on this device?
bool lstm_rec_tc_supported(int H, bool x3) {
  static const bool off = getenv("FSN_NO_REC_TC") != nullptr;
  if (off || H < rec::MIN_H || !tmap_encoder()) return false;
  int dev = 0, coop = 0, max_smem = 0, major = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  const int Kp = (H + rec::KB - 1) / rec::KB * rec::KB;
  return coop == 1 && major == 9 && cdiv(H, rec::U) <= rec_sm_count() && rec::smem_bytes(Kp, x3, 2) <= (size_t)max_smem;
}

// rows one launch covers (groups of 128 that fit on the chip next to each other)
int lstm_rec_tc_rows_per_launch(int H) {
  const int C = cdiv(H, rec::U);
  int G = rec_sm_count() / C;
  if (G < 1) G = 1;
  return G * rec::MR;
}

// scratch of one launch: fp16 state ping-pong [2][parts][rows][Kp] + the group counters.  The same scratch serves
// layers of DIFFERENT hidden sizes (fast_fullsubnet: 384 / 257 / 512), so its size must not depend on H:
// rows_per_launch * Kp <= (SMs * 8 / H) * 128 * (H + 63) < 2 * SMs * 8 * 128 elements for H >= 64.
static size_t rec_state_capacity_bytes() { return align_up((size_t)2 * 2 * 2 * rec_sm_count() * 8 * 128 * sizeof(__half), 256); }
size_t lstm_rec_tc_scratch_bytes(int H, bool x3) {
  (void)H; (void)x3;
  return rec_state_capacity_bytes() + 64 * 32 * sizeof(unsigned int);
}

// h_t for every step of one layer, given the hoisted input projection P (see Args for the strides); R rows (any
// count: chunks of lstm_rec_tc_rows_per_launch are launched back to back).  P and hall must be 8-byte aligned: with H
// and the strides even the kernel reads P and writes hall as float2 (vec_ok), so a base at 4 mod 8 is refused
// (FSN_ERR_SHAPE) before any CUDA call rather than faulting in the kernel.  info (nullable) receives the launch choices.
int lstm_rec_tc_launch(const float* w_hh, const float* b_ih, const float* b_hh, const float* P, size_t p_row, size_t p_t,
                       float* hall, size_t h_row, size_t h_t, int R, int T, int H, bool x3, void* scratch,
                       cudaStream_t st, const RecCarry* io, RecTcInfo* info) {
  FSN_REQUIRE((reinterpret_cast<uintptr_t>(P) & 7) == 0 && (reinterpret_cast<uintptr_t>(hall) & 7) == 0, FSN_ERR_SHAPE,
              "lstm_rec_tc: P (%p) and hall (%p) must be 8-byte aligned", (const void*)P, (void*)hall);
  FSN_REQUIRE(lstm_rec_tc_supported(H, x3), FSN_ERR_UNSUPPORTED, "lstm_rec_tc: hidden size %d not supported", H);
  const int Kp = (H + rec::KB - 1) / rec::KB * rec::KB;
  const int C = cdiv(H, rec::U);
  const int rows_max = lstm_rec_tc_rows_per_launch(H);
  const int parts = x3 ? 2 : 1;
  int dev = 0, max_smem = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  int stages = x3 ? 4 : rec::MAX_STAGES;
  while (stages > 2 && rec::smem_bytes(Kp, x3, stages) > (size_t)max_smem) --stages;
  const size_t smem = rec::smem_bytes(Kp, x3, stages);
  __half* state = (__half*)scratch;
  const size_t state_bytes = align_up((size_t)2 * parts * rows_max * Kp * sizeof(__half), 256);
  FSN_REQUIRE(state_bytes <= rec_state_capacity_bytes(), FSN_ERR_UNSUPPORTED, "lstm_rec_tc: state of H=%d exceeds the scratch", H);
  unsigned int* barrier = (unsigned int*)((uint8_t*)scratch + rec_state_capacity_bytes());  // fixed place, whatever H
  int rc;
  const void* kern = io ? (x3 ? (const void*)rec::lstm_rec_tc_carry_kernel<true> : (const void*)rec::lstm_rec_tc_carry_kernel<false>)
                        : (x3 ? (const void*)rec::lstm_rec_tc_kernel<true> : (const void*)rec::lstm_rec_tc_kernel<false>);
  if ((rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "lstm_rec_tc smem attr")))
    return rc;
  if (info) *info = RecTcInfo{rows_max, stages, cdiv(R, rows_max), (int)smem};
  for (int r0 = 0; r0 < R; r0 += rows_max) {
    const int nr = (R - r0 < rows_max) ? R - r0 : rows_max;
    const int G = cdiv(nr, rec::MR);
    const int Rpad = G * rec::MR;
    // state of padded rows / padded k stays zero for the whole launch; counters start at zero
    if ((rc = check_cuda(cudaMemsetAsync(scratch, 0, state_bytes, st), "lstm_rec_tc memset"))) return rc;
    if ((rc = check_cuda(cudaMemsetAsync(barrier, 0, 64 * 32 * sizeof(unsigned int), st), "lstm_rec_tc memset"))) return rc;
    if (io) {
      rec::rec_carry_init_kernel<<<ew_grid((size_t)nr * H), 256, 0, st>>>(io->h_init + (size_t)r0 * io->row, io->row,
                                                                          io->restart + r0, nr, H, Kp, Rpad, parts, state);
      FSN_CHECK_LAUNCH("rec_carry_init_kernel");
    }
    CUtensorMap tm;
    FSN_REQUIRE(encode_tmap_2d(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, state, Kp, 2 * parts * Rpad, Kp * sizeof(__half), rec::KB,
                               rec::MR),
                FSN_ERR_CUDA, "lstm_rec_tc: cuTensorMapEncodeTiled failed");
    rec::Args a;
    a.w_hh = w_hh; a.b_ih = b_ih; a.b_hh = b_hh;
    a.P = P + (size_t)r0 * p_row; a.p_row = p_row; a.p_t = p_t;
    a.hall = hall + (size_t)r0 * h_row; a.h_row = h_row; a.h_t = h_t;
    a.state = state; a.barrier = barrier;
    a.R = nr; a.T = T; a.H = H; a.Kp = Kp; a.Rpad = Rpad; a.C = C; a.stages = stages;
    a.fence_all = getenv("FSN_REC_FENCE_ALL") != nullptr;
    rec::CarryArgs ca{};
    if (io) {
      ca.c_init = io->c_init + (size_t)r0 * io->row; ca.c_fin = io->c_fin + (size_t)r0 * io->row; ca.c_row = io->row;
      ca.restart = io->restart + r0; ca.fin_step = io->fin_step;
    }
    void* params[] = {(void*)&tm, (void*)&a, (void*)&ca};
    if ((rc = check_cuda(cudaLaunchCooperativeKernel(kern, dim3(G * C), dim3(rec::NTHREADS), params, smem, st),
                         "lstm_rec_tc cooperative launch")))
      return rc;
    FSN_CHECK_LAUNCH("lstm_rec_tc_kernel");
  }
  return FSN_OK;
}

int split_tf32_launch(const float* in, size_t rows, int K, size_t ldi, const float* row_scale, int rows_per_scale,
                      float* out, int Kp, int cat, cudaStream_t st, int scale_B) {
  if (rows == 0) return FSN_OK;
  const size_t n = rows * (size_t)Kp;
  size_t blocks = (n + 255) / 256;
  if (blocks > rec_sm_count() * 16) blocks = (size_t)rec_sm_count() * 16;
  rec::split_tf32_kernel<<<(int)blocks, 256, 0, st>>>(in, rows, K, ldi, row_scale, rows_per_scale < 1 ? 1 : rows_per_scale,
                                                      scale_B, out, Kp, cat);
  FSN_CHECK_LAUNCH("split_tf32_kernel");
  return FSN_OK;
}

int bias_act_launch(float* x, size_t rows, int N, size_t ld, const float* bias, int act, cudaStream_t st) {
  if (rows == 0) return FSN_OK;
  const size_t n = rows * (size_t)N;
  size_t blocks = (n + 255) / 256;
  if (blocks > rec_sm_count() * 16) blocks = (size_t)rec_sm_count() * 16;
  rec::bias_act_kernel<<<(int)blocks, 256, 0, st>>>(x, rows, N, ld, bias, act);
  FSN_CHECK_LAUNCH("bias_act_kernel");
  return FSN_OK;
}

// C[M,N] = A[M,K] W[N,K]^T on the tf32 tensor cores.  `a` is the prepared A operand (prep_operand: [M, Keff], lda);
// W row-major [N, K] is prepared here into `w` ([N, Keff]); x3: Keff = 3 * Kp (see split_tf32_kernel).
int gemm_tc_split_launch(const float* a, size_t lda, const float* W, int N, int K, float* w, float* C, size_t ldc, size_t M,
                         bool x3, cudaStream_t st) {
  const int Kp = (K + 3) & ~3;
  const int Keff = x3 ? 3 * Kp : K;
  int rc;
  if ((rc = split_tf32_launch(W, (size_t)N, K, (size_t)K, nullptr, 1, w, Kp, x3 ? 2 : 0, st, 0))) return rc;
  FSN_REQUIRE(M < ((size_t)1 << 31), FSN_ERR_SHAPE, "gemm_tc: too many rows");
  return tgemm_launch(a, lda, w, x3 ? (size_t)3 * Kp : (size_t)Kp, C, ldc, (int)M, N, Keff, false, nullptr, 0, st);
}

// ---------------------------------------------------------------------------------------------------------------
// One full LSTM layer and one Linear layer on top of the pieces above (what the model files call).
void lstm_tc_carve(Carver& c, size_t rows_T, int Kmax, int Hmax, bool x3, LstmTcWs& ws) {
  const size_t wa = (size_t)((Kmax + 3) & ~3) * (x3 ? 3 : 1);
  ws.a = c.take<float>(rows_T * wa);
  ws.w = c.take<float>((size_t)4 * Hmax * wa);
  ws.P = c.take<float>(rows_T * 4 * Hmax);
  ws.rec = c.take<char>(lstm_rec_tc_scratch_bytes(Hmax, x3));
}

// operand A of a GEMM: x [rows, K] (row stride ldx) -> 16-byte aligned rows, scaled; x3: the [hi | lo | hi] layout
static int prep_operand(const float* x, size_t ldx, int K, size_t rows, const float* row_scale, int rows_per_scale, int scale_B,
                        bool x3, const LstmTcWs& ws, const float*& a, size_t& lda, cudaStream_t st) {
  if (!x3 && !row_scale && (ldx & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    a = x; lda = ldx;
    return FSN_OK;
  }
  const int Kp = (K + 3) & ~3;
  a = ws.a; lda = (size_t)Kp * (x3 ? 3 : 1);
  return split_tf32_launch(x, rows, K, ldx, row_scale, rows_per_scale, ws.a, Kp, x3 ? 1 : 0, st, scale_B);
}

// hall[r, t, :] (row stride T*H) of one LSTM layer over x[(r*T + t), :K] * scale
int lstm_layer_tc(const fsn_lstm_layer& L, const float* x, size_t ldx, int K, const float* row_scale, int rows_per_scale,
                  int scale_B, int R, int T, int H, bool x3, const LstmTcWs& ws, float* hall, cudaStream_t st,
                  const RecCarry* io) {
  const size_t rows = (size_t)R * T;
  const float* a;
  size_t lda;
  int rc;
  if ((rc = prep_operand(x, ldx, K, rows, row_scale, rows_per_scale, scale_B, x3, ws, a, lda, st))) return rc;
  if ((rc = gemm_tc_split_launch(a, lda, L.w_ih, 4 * H, K, ws.w, ws.P, (size_t)4 * H, rows, x3, st))) return rc;
  return lstm_rec_tc_launch(L.w_hh, L.b_ih, L.b_hh, ws.P, (size_t)T * 4 * H, (size_t)4 * H, hall, (size_t)T * H, (size_t)H, R, T,
                            H, x3, ws.rec, st, io);
}

// out[rows, :N] (row stride ldo) = act(x[rows, :K] W[N,K]^T + bias)
int linear_tc(const float* x, size_t ldx, int K, const float* W, const float* bias, int N, int act, float* out, size_t ldo,
              size_t rows, bool x3, const LstmTcWs& ws, cudaStream_t st) {
  const float* a;
  size_t lda;
  int rc;
  if ((rc = prep_operand(x, ldx, K, rows, nullptr, 1, 0, x3, ws, a, lda, st))) return rc;
  if ((rc = gemm_tc_split_launch(a, lda, W, N, K, ws.w, out, ldo, rows, x3, st))) return rc;
  if (!bias && act == FSN_ACT_NONE) return FSN_OK;
  return bias_act_launch(out, rows, N, ldo, bias, act, st);
}

}  // namespace fsn

// unit-test hooks (tests/test_gpu_rec_tc.py): one LSTM layer / one Linear layer on the tensor-core path, and the
// recurrence alone.  Every argument is checked before any CUDA call (the scratch sizes read the device's SM count only);
// what the device supports (FSN_ERR_UNSUPPORTED) is reported after those checks.  The layer hooks report a hidden size
// below the kernel's minimum as unsupported right after the pointer and shape checks, before the workspace, whose size
// means nothing for such an H: a caller probing H gets FSN_ERR_UNSUPPORTED whatever workspace it passes.
extern "C" size_t fsn_debug_lstm_tc_workspace_bytes(int R, int T, int K, int H, int x3) {
  fsn::Carver c(nullptr);
  fsn::LstmTcWs ws;
  fsn::lstm_tc_carve(c, (size_t)R * T, K > H ? K : H, H, x3 != 0, ws);
  return c.off;
}
// the argument checks shared by the two LSTM layer hooks, before any CUDA call: pointers, sizes, the minimum H, workspace
static int lstm_layer_hook_check(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* x,
                                 int R, int T, int K, int H, int x3, float* hall, void* workspace, size_t workspace_bytes,
                                 fsn::LstmTcWs& ws) {
  FSN_REQUIRE(w_ih && w_hh && b_ih && b_hh && x && hall, FSN_ERR_SHAPE, "lstm_layer_tc hook: null argument");
  FSN_REQUIRE(R > 0 && T > 0 && K > 0 && H > 0 && (int64_t)R * T < ((int64_t)1 << 31), FSN_ERR_SHAPE,
              "lstm_layer_tc hook: bad shape R=%d T=%d K=%d H=%d", R, T, K, H);
  FSN_REQUIRE(H >= fsn::rec::MIN_H, FSN_ERR_UNSUPPORTED, "lstm_layer_tc: hidden size %d not supported (< %d)", H,
              fsn::rec::MIN_H);
  fsn::Carver c(workspace);
  fsn::lstm_tc_carve(c, (size_t)R * T, K > H ? K : H, H, x3 != 0, ws);
  FSN_REQUIRE(workspace && workspace_bytes >= c.off, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes, c.off);
  return FSN_OK;
}
extern "C" int fsn_debug_lstm_layer_tc(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                       const float* x, int R, int T, int K, int H, int x3, float* hall, void* workspace,
                                       size_t workspace_bytes, fsn_stream_t stream) {
  fsn::LstmTcWs ws;
  int rc;
  if ((rc = lstm_layer_hook_check(w_ih, w_hh, b_ih, b_hh, x, R, T, K, H, x3, hall, workspace, workspace_bytes, ws))) return rc;
  FSN_REQUIRE(fsn::lstm_rec_tc_supported(H, x3 != 0), FSN_ERR_UNSUPPORTED, "lstm_layer_tc: hidden size %d not supported", H);
  fsn_lstm_layer L{w_ih, w_hh, b_ih, b_hh};
  return fsn::lstm_layer_tc(L, x, (size_t)K, K, nullptr, 1, 0, R, T, H, x3 != 0, ws, hall, (cudaStream_t)stream);
}
extern "C" int fsn_debug_linear_tc(const float* x, int rows, int K, const float* W, const float* bias, int N, int act, int x3,
                                   float* out, void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  FSN_REQUIRE(x && W && out, FSN_ERR_SHAPE, "linear_tc hook: null argument");
  FSN_REQUIRE(rows > 0 && K > 0 && N > 0 && (N + 127) / 128 <= 65535, FSN_ERR_SHAPE, "linear_tc hook: bad shape rows=%d K=%d N=%d",
              rows, K, N);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "linear_tc hook: unknown act %d", act);
  fsn::Carver c(workspace);
  fsn::LstmTcWs ws;
  const int Hm = (N + 3) / 4 > 8 ? (N + 3) / 4 : 8;
  fsn::lstm_tc_carve(c, (size_t)rows, K, Hm, x3 != 0, ws);
  FSN_REQUIRE(workspace && workspace_bytes >= c.off, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes, c.off);
  return fsn::linear_tc(x, (size_t)K, K, W, bias, N, act, out, (size_t)N, (size_t)rows, x3 != 0, ws, (cudaStream_t)stream);
}
extern "C" int fsn_debug_lstm_tc_carry(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                       const float* x, int R, int T, int K, int H, int x3, const float* h_init, float* c,
                                       const int32_t* restart, int fin_step, float* hall, void* workspace,
                                       size_t workspace_bytes, fsn_stream_t stream) {
  FSN_REQUIRE(h_init && c && restart, FSN_ERR_SHAPE, "lstm_tc_carry hook: null carry argument");
  FSN_REQUIRE(fin_step >= -1 && fin_step < T, FSN_ERR_SHAPE, "lstm_tc_carry hook: fin_step %d outside [-1, T=%d)", fin_step, T);
  fsn::LstmTcWs ws;
  int rc;
  if ((rc = lstm_layer_hook_check(w_ih, w_hh, b_ih, b_hh, x, R, T, K, H, x3, hall, workspace, workspace_bytes, ws))) return rc;
  FSN_REQUIRE(fsn::lstm_rec_tc_supported(H, x3 != 0), FSN_ERR_UNSUPPORTED, "lstm_layer_tc: hidden size %d not supported", H);
  fsn_lstm_layer L{w_ih, w_hh, b_ih, b_hh};
  const fsn::RecCarry io{h_init, c, c, (size_t)H, restart, fin_step};
  return fsn::lstm_layer_tc(L, x, (size_t)K, K, nullptr, 1, 0, R, T, H, x3 != 0, ws, hall, (cudaStream_t)stream, &io);
}
extern "C" size_t fsn_debug_lstm_rec_tc_scratch_bytes(int H, int x3) { return fsn::lstm_rec_tc_scratch_bytes(H, x3 != 0); }
// the recurrence alone, on a given input projection P[r * p_row + t * p_t + gate * H + u], into hall[r * h_row + t * h_t
// + u], as the layers call lstm_rec_tc_launch.  restart == nullptr: the plain kernel (zero initial state; h_init, c_init
// and c_fin must be null); otherwise the carried-state kernel with RecCarry{h_init, c_init, c_fin, c_row, restart,
// fin_step} (c_fin may be c_init).  info (nullable, 4 ints): rows per launch, ring stages, launches, dynamic shared memory.
extern "C" int fsn_debug_lstm_rec_tc(const float* w_hh, const float* b_ih, const float* b_hh, const float* P, int64_t p_row,
                                     int64_t p_t, float* hall, int64_t h_row, int64_t h_t, int R, int T, int H, int x3,
                                     const float* h_init, const float* c_init, float* c_fin, int64_t c_row,
                                     const int32_t* restart, int fin_step, int* info, void* scratch, size_t scratch_bytes,
                                     fsn_stream_t stream) {
  FSN_REQUIRE(w_hh && b_ih && b_hh && P && hall, FSN_ERR_SHAPE, "lstm_rec_tc hook: null argument");
  FSN_REQUIRE(R > 0 && T > 0 && H > 0, FSN_ERR_SHAPE, "lstm_rec_tc hook: bad shape R=%d T=%d H=%d", R, T, H);
  // a row of n floats per step, steps t_stride apart, rows row_stride apart: no two (row, step) blocks overlap
  auto covers = [T](int64_t row_stride, int64_t t_stride, int64_t n) {
    return t_stride >= n && t_stride <= (INT64_MAX - n) / T && row_stride >= (T - 1) * t_stride + n;
  };
  FSN_REQUIRE(covers(p_row, p_t, (int64_t)4 * H) && covers(h_row, h_t, H), FSN_ERR_SHAPE,
              "lstm_rec_tc hook: strides P (%lld, %lld) / hall (%lld, %lld) do not cover T=%d steps of 4H / H (H=%d)",
              (long long)p_row, (long long)p_t, (long long)h_row, (long long)h_t, T, H);
  if (restart) {
    FSN_REQUIRE(h_init && c_init && c_fin, FSN_ERR_SHAPE, "lstm_rec_tc hook: a carried state needs h_init, c_init and c_fin");
    FSN_REQUIRE(c_row >= H, FSN_ERR_SHAPE, "lstm_rec_tc hook: c_row %lld < H=%d", (long long)c_row, H);
    FSN_REQUIRE(fin_step >= -1 && fin_step < T, FSN_ERR_SHAPE, "lstm_rec_tc hook: fin_step %d outside [-1, T=%d)", fin_step, T);
  } else {
    FSN_REQUIRE(!h_init && !c_init && !c_fin, FSN_ERR_SHAPE, "lstm_rec_tc hook: carry pointers without a restart table");
  }
  const size_t need = fsn::lstm_rec_tc_scratch_bytes(H, x3 != 0);
  FSN_REQUIRE(scratch && scratch_bytes >= need, FSN_ERR_WORKSPACE, "scratch too small: %zu < %zu", scratch_bytes, need);
  const fsn::RecCarry io{h_init, c_init, c_fin, (size_t)c_row, restart, fin_step};
  fsn::RecTcInfo got{};
  const int rc = fsn::lstm_rec_tc_launch(w_hh, b_ih, b_hh, P, (size_t)p_row, (size_t)p_t, hall, (size_t)h_row, (size_t)h_t, R, T,
                                         H, x3 != 0, scratch, (cudaStream_t)stream, restart ? &io : nullptr, &got);
  if (info) memcpy(info, &got, sizeof(got));
  return rc;
}
// unit-test hook of the tf32 GEMM path of the full-band stacks: out[rows, :N] (row stride ldo) = act(x' W^T + bias) with
// x' = x[rows, :K] (row stride ldx) times its row scale, i.e. the input projection of lstm_layer_tc (prep_operand,
// gemm_tc_split_launch) and the epilogue of linear_tc (bias_act_launch).  Workspace: the prepared A and W operands only,
// carved as lstm_tc_carve lays them out (so fsn_debug_lstm_tc_workspace_bytes(rows, 1, K, max(8, ceil(N / 4)), x3) is
// always enough) and sized in host arithmetic.  Every argument is checked before any CUDA call.
extern "C" int fsn_debug_gemm_tc(const float* x, int64_t ldx, int K, const float* row_scale, int rows_per_scale, int scale_B,
                                 const float* W, int N, const float* bias, int act, int x3, float* out, int64_t ldo, int64_t rows,
                                 void* workspace, size_t workspace_bytes, fsn_stream_t stream) {
  fsn::launch_counter() = 0;
  FSN_REQUIRE(x && W && out, FSN_ERR_SHAPE, "gemm_tc hook: null argument");
  FSN_REQUIRE(K > 0 && N > 0 && rows > 0 && rows < ((int64_t)1 << 31) && ldx >= K && ldo >= N, FSN_ERR_SHAPE,
              "gemm_tc hook: bad shape rows=%lld K=%d N=%d ldx=%lld ldo=%lld", (long long)rows, K, N, (long long)ldx,
              (long long)ldo);
  FSN_REQUIRE(!row_scale || (rows_per_scale >= 1 && scale_B >= 0), FSN_ERR_SHAPE,
              "gemm_tc hook: a row scale needs rows_per_scale >= 1 and scale_B >= 0");
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "gemm_tc hook: unknown act %d", act);
  FSN_REQUIRE((N + 127) / 128 <= 65535, FSN_ERR_SHAPE, "gemm_tc hook: N=%d exceeds the grid", N);
  fsn::Carver c(workspace);
  const size_t wa = (size_t)((K + 3) & ~3) * (x3 ? 3 : 1);
  const int Hm = (N + 3) / 4 > 8 ? (N + 3) / 4 : 8;
  fsn::LstmTcWs ws{};
  ws.a = c.take<float>((size_t)rows * wa);
  ws.w = c.take<float>((size_t)4 * Hm * wa);
  FSN_REQUIRE(workspace && workspace_bytes >= c.off, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes, c.off);
  cudaStream_t st = (cudaStream_t)stream;
  const float* a;
  size_t lda;
  int rc;
  if ((rc = fsn::prep_operand(x, (size_t)ldx, K, (size_t)rows, row_scale, rows_per_scale, scale_B, x3 != 0, ws, a, lda, st)))
    return rc;
  if ((rc = fsn::gemm_tc_split_launch(a, lda, W, N, K, ws.w, out, (size_t)ldo, (size_t)rows, x3 != 0, st))) return rc;
  return fsn::bias_act_launch(out, (size_t)rows, N, (size_t)ldo, bias, act, st);
}
