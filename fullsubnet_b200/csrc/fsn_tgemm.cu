// tf32 tensor-core GEMM for the training path:  C[M,N] (+)= A[M,K] * B[N,K]^T, all fp32 in global memory, both
// operands K-contiguous ("K-major"), Hopper warpgroup MMA (wgmma.mma_async, tf32) with the accumulators in registers.
//
// One CTA = one 128 x BN output tile (BN = 128 or 256), optional split-K slice (blockIdx.z).
//   warpgroups 0-1  consumers: warpgroup h multiplies rows 64h..64h+63 of the tile (m64nBNk8, 4 per stage), releases each
//                   stage once the wgmma that read it has retired (wait_group 1), and writes its accumulator fragment
//                   straight from registers after the last stage.
//   producer        one warp, one elected lane issues the TMA tiled loads (128B swizzle, rows / k beyond the matrix
//                   zero-filled by the tensor map) of a stage.
// No operand conversion pass: the tensor core reads fp32 bits as tf32 (10-bit mantissa, truncation).
//
// Also in this file, built from the same pieces (DESIGN.md 4.2):
//   tgemm_tma_kernel        BlockedOps mode streams block-tiled operand copies (transpose_blocked_kernel) for the long-K
//                           weight-gradient GEMMs dW = dG^T X
//   lstm_fwd_step_kernel    one LSTM step of the training forward: [x_t | h_{t-1}] [W_ih | W_hh]^T (fp16 / tf32 operands)
//                           and the cell in one launch; tile = 128 rows x (4 gates x 32 hidden units)
#include "fsn_internal.cuh"
#include "fsn_tc_ptx.cuh"
#include "fsn_wgmma.cuh"

namespace fsn {
namespace tg {

using namespace ptx;

constexpr int BM = 128, BK = 32;
constexpr int A_BYTES = BM * BK * 4;  // 16 KB
constexpr int CONSUMERS = 256;        // two warpgroups of 64 tile rows each

template <int BN> struct Cfg {
  static_assert(BN == 128 || BN == 256, "wgmma tile width");
  static constexpr int B_BYTES = BN * BK * 4;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // BN = 128: 3 stages (96 KB) so two CTAs share an SM - one writes its tile while the other runs its main loop
  static constexpr int STAGES = (BN == 128) ? 3 : 4;
  static constexpr int MIN_CTAS = (BN == 128) ? 2 : 1;
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

// block-tiled operand addressing of tgemm_tma_kernel (weight-gradient GEMMs, see tgemm_blocked_launch)
struct BlockedOps { int on, a_nkb, b_nkb, a_kb0, b_kb0; };

struct Bars {
  uint64_t full[8];
  uint64_t empty[8];
};

// consumer warpgroups: the tile's MMAs over nk stages into acc (rows 64 * warpgroup + fragment row)
template <int BN>
__device__ __forceinline__ void mma_loop(uint8_t* smem, Bars& bars, int nk, float (&acc)[BN / 2]) {
  using CF = Cfg<BN>;
  constexpr int STAGES = CF::STAGES;
  const int wgi = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const uint32_t smem_base = smem_u32(smem);
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  wg::fence_operand(acc);
  for (int i = 0; i < nk; ++i) {
    const int s = i % STAGES;
    mbar_wait_mma(&bars.full[s], (uint32_t)((i / STAGES) & 1));
    const uint32_t sa = smem_base + s * CF::STAGE_BYTES + wgi * (64 * 128);
    const uint32_t sb = smem_base + s * CF::STAGE_BYTES + A_BYTES;
    wg::fence();
#pragma unroll
    for (int kk = 0; kk < BK / 8; ++kk) {
      if constexpr (BN == 256) wg::mma_tf32_n256(acc, wg::desc_sw128(sa + kk * 32), wg::desc_sw128(sb + kk * 32), 1u);
      else                     wg::mma_tf32_n128(acc, wg::desc_sw128(sa + kk * 32), wg::desc_sw128(sb + kk * 32), 1u);
    }
    wg::commit();
    wg::wait<1>();  // the MMAs of stage i-1 have read their operands
    if (i > 0 && lane == 0) mbar_arrive(&bars.empty[(i - 1) % STAGES]);
  }
  wg::wait<0>();
  wg::fence_operand(acc);
}

// accumulator fragment -> global memory (all MMAs have completed)
template <int BN>
__device__ __forceinline__ void epilogue(const float (&acc)[BN / 2], float* __restrict__ C, size_t ldc, int M, int N, int m0,
                                         int n0, int accumulate, size_t split_stride) {
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31, wgi = threadIdx.x >> 7;
  float* cbase = C + (size_t)blockIdx.z * split_stride;
  const int rbase = m0 + 64 * wgi + 16 * w + (l >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (l & 3);
    if (col >= N) continue;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = rbase + 8 * hh;
      if (row >= M) continue;
      float* p = cbase + (size_t)row * ldc + col;
      float v0 = acc[4 * j + 2 * hh], v1 = acc[4 * j + 2 * hh + 1];
      if (accumulate) v0 += p[0];
      p[0] = v0;
      if (col + 1 < N) {
        if (accumulate) v1 += p[1];
        p[1] = v1;
      }
    }
  }
}

// One elected lane of the producer warp issues the tiled loads of a stage (128B hardware swizzle, rows / k beyond the
// matrix zero-filled by the tensor map), the full barrier counts the transaction bytes.
template <int BN>
__global__ void __launch_bounds__(CONSUMERS + 32, Cfg<BN>::MIN_CTAS)
tgemm_tma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, float* __restrict__ C,
                 size_t ldc, int M, int N, int K, int k_per_split, int accumulate, size_t split_stride, BlockedOps bo) {
  using CF = Cfg<BN>;
  constexpr int STAGES = CF::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  Bars& bars = *reinterpret_cast<Bars*>(smem + STAGES * CF::STAGE_BYTES);
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int kb = blockIdx.z * k_per_split;
  const int ke = (kb + k_per_split < K) ? kb + k_per_split : K;
  const int nk = (ke - kb + BK - 1) / BK;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&bars.full[s], 1); mbar_init(&bars.empty[s], CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= CONSUMERS) {
    for (int i = 0; i < nk; ++i) {
      const int s = i % STAGES;
      if (i >= STAGES) mbar_wait<false>(&bars.empty[s], (uint32_t)(((i / STAGES) - 1) & 1));
      if (elect_one()) {
        uint8_t* sa = smem + s * CF::STAGE_BYTES;
        mbar_expect_tx(&bars.full[s], CF::STAGE_BYTES);
        if (bo.on) {
          // block-tiled operands: tile (128 rows, k block of 32) = 16 contiguous KB, see tgemm_blocked_launch
          const int kblk = (kb >> 5) + i;
          tma_load_2d(sa, &tmA, 0, (blockIdx.x * bo.a_nkb + bo.a_kb0 + kblk) * 128, &bars.full[s]);
#pragma unroll
          for (int j = 0; j < BN / 128; ++j)
            tma_load_2d(sa + A_BYTES + j * 128 * 128, &tmB, 0, ((blockIdx.y * (BN / 128) + j) * bo.b_nkb + bo.b_kb0 + kblk) * 128,
                        &bars.full[s]);
        } else {
          tma_load_2d(sa, &tmA, kb + i * BK, m0, &bars.full[s]);
          tma_load_2d(sa + A_BYTES, &tmB, kb + i * BK, n0, &bars.full[s]);
        }
      }
      __syncwarp();
    }
  } else {
    float acc[BN / 2];
    mma_loop<BN>(smem, bars, nk, acc);
    epilogue<BN>(acc, C, ldc, M, N, m0, n0, accumulate, split_stride);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// One LSTM step of the training forward, GEMM and cell in one kernel (torch.nn.LSTM forward, saved for autograd):
//   z = P_t + b_ih + b_hh + h_{t-1} W_hh^T;  (i,f,g,o) = act(z);  c_t = f c_{t-1} + i g;  h_t = o tanh(c_t)
// The CTA tile is 128 rows x 128 gate columns = the FOUR gates of 32 hidden units: the B operand is four 32-row TMA
// boxes of W_hh (rows g*H + 32 j ..), so column 32 g + u of the accumulator is gate g of unit u0 + u.  In the wgmma
// fragment a thread holds columns 8 j + 2 (lane % 4) + {0, 1}, i.e. the same 8 units in all four gate blocks: the cell
// runs straight on the accumulator registers and the recurrent product never goes to memory.  The cell reads P_t (the
// hoisted input projection, overwritten in place by the post-activation gates the backward pass needs) and c_{t-1},
// writes gates, c_t, h_t.  Two CTAs per SM: one runs its cell while the other multiplies.
// 1 / (1 + 2^(-x log2 e)) and 2 sigmoid(2x) - 1 on the MUFU unit (ex2.approx + rcp.approx: ~2 ulp; saturate correctly:
// ex2 -> inf gives rcp -> 0, ex2 -> 0 gives 1)
__device__ __forceinline__ float sigmoid_mufu(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return r;
}
__device__ __forceinline__ float tanh_mufu(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -2.8853900817779268f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return fmaf(2.0f, r, -1.0f);
}

// shared memory of the step kernel: two TMA stages of the 128 x 128 tile
struct StepCfg {
  static constexpr int STAGES = 2;
  static constexpr int MAIN = STAGES * Cfg<128>::STAGE_BYTES;
  static constexpr int SMEM = MAIN + 1024 /*align*/ + 256 /*barriers*/;
};
// HT: hidden size known at compile time (0: runtime) - the strides of the cell become immediate offsets
template <bool FOLD, int HT>
__global__ void __launch_bounds__(CONSUMERS + 32, 2)
lstm_fwd_step_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmWx, float* __restrict__ G,
                     const float* __restrict__ b_ih, const float* __restrict__ b_hh, const float* __restrict__ C_prev,
                     float* __restrict__ C_out, float* __restrict__ H_out, __half* __restrict__ H16_out, int R, int H_rt, int nkx,
                     int nkh, int x16, int h16) {
  const int H = HT ? HT : H_rt;
  using CF = Cfg<128>;
  constexpr int STAGES = StepCfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  Bars& bars = *reinterpret_cast<Bars*>(smem + StepCfg::MAIN);
  const int m0 = blockIdx.x * BM, u0 = blockIdx.y * 32;
  // k blocks: first nkx of x_t W_ih^T (a narrow layer input is folded in here instead of a hoisted projection: G then
  // carries no P and is only written), then nkh of h_{t-1} W_hh^T (0 at the first step)
  const int nk = nkx + nkh;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&bars.full[s], 1); mbar_init(&bars.empty[s], CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= CONSUMERS) {
    // TMA producer
    for (int i = 0; i < nk; ++i) {
      const int s = i % STAGES;
      if (i >= STAGES) mbar_wait<false>(&bars.empty[s], (uint32_t)(((i / STAGES) - 1) & 1));
      if (elect_one()) {
        uint8_t* sa = smem + s * CF::STAGE_BYTES;
        mbar_expect_tx(&bars.full[s], CF::STAGE_BYTES);
        const CUtensorMap* ma = i < nkx ? &tmX : &tmA;
        const CUtensorMap* mb = i < nkx ? &tmWx : &tmB;
        // a stage row is 128 bytes: 32 tf32 or 64 fp16 k values
        const int k0 = (i < nkx ? i * (x16 ? 2 * BK : BK) : (i - nkx) * (h16 ? 2 * BK : BK));
        tma_load_2d(sa, ma, k0, m0, &bars.full[s]);
#pragma unroll
        for (int g = 0; g < 4; ++g) tma_load_2d(sa + A_BYTES + g * 32 * 128, mb, k0, g * H + u0, &bars.full[s]);
      }
      __syncwarp();
    }
    return;
  }
  // ---- consumers: MMA (per stage four instructions over 32 bytes of k each: 8 tf32 or 16 fp16 values; both kinds
  // accumulate into the same fp32 registers), then the cell on the fragment
  const int wgi = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  wg::fence_operand(acc);
  {
    const uint32_t smem_base = smem_u32(smem);
    for (int i = 0; i < nk; ++i) {
      const int s = i % STAGES;
      mbar_wait_mma(&bars.full[s], (uint32_t)((i / STAGES) & 1));
      const uint32_t sa = smem_base + s * CF::STAGE_BYTES + wgi * (64 * 128);
      const uint32_t sb = smem_base + s * CF::STAGE_BYTES + A_BYTES;
      const bool half_blk = i < nkx ? (x16 != 0) : (h16 != 0);
      wg::fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if (half_blk) wg::mma_f16_n128(acc, wg::desc_sw128(sa + kk * 32), wg::desc_sw128(sb + kk * 32), 1u);
        else          wg::mma_tf32_n128(acc, wg::desc_sw128(sa + kk * 32), wg::desc_sw128(sb + kk * 32), 1u);
      }
      wg::commit();
      wg::wait<1>();
      if (i > 0 && l == 0) mbar_arrive(&bars.empty[(i - 1) % STAGES]);
    }
    wg::wait<0>();
    wg::fence_operand(acc);
  }
  const unsigned H4 = 4u * (unsigned)H;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = m0 + 64 * wgi + 16 * w + (l >> 2) + 8 * hh;
    if (row >= R) continue;
    float* gr = G + (size_t)row * H4;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int u = u0 + 8 * jj + 2 * (l & 3) + e;
        float z[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const float a = acc[4 * (g * 4 + jj) + 2 * hh + e];
          const float b = b_ih[g * H + u] + b_hh[g * H + u];
          z[g] = FOLD ? a + b : (gr[g * H + u] + b) + a;
        }
        // ex2 + rcp forms (2 ulp class; the tf32 / fp16 products around them are 1e-3 class)
        const float gi = sigmoid_mufu(z[0]), gf = sigmoid_mufu(z[1]), gg = tanh_mufu(z[2]), go = sigmoid_mufu(z[3]);
        const float cp = C_prev ? C_prev[(size_t)row * H + u] : 0.f;
        const float cn = fmaf(gf, cp, gi * gg);
        const float hn = go * tanh_mufu(cn);
        gr[u] = gi; gr[H + u] = gf; gr[2 * H + u] = gg; gr[3 * H + u] = go;
        C_out[(size_t)row * H + u] = cn;
        H_out[(size_t)row * H + u] = hn;
        if (H16_out) H16_out[(size_t)row * H + u] = __float2half_rn(hn);  // next step's / next layer's MMA operand
      }
    }
  }
}

}  // namespace tg

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link against libcuda)
PFN_cuTensorMapEncodeTiled_v12000 tmap_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
    cudaGetLastError();
  }
  return fn;
}

bool encode_tmap_2d(CUtensorMap* m, CUtensorMapDataType dtype, const void* base, cuuint64_t inner, cuuint64_t rows,
                    cuuint64_t pitch_bytes, cuuint32_t box_inner, cuuint32_t box_rows) {
  PFN_cuTensorMapEncodeTiled_v12000 fn = tmap_encoder();
  if (!fn) return false;
  cuuint64_t gdim[2] = {inner, rows};
  cuuint64_t gstr[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return fn(m, dtype, 2, (void*)base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// fp32 [rows, K] row-major (ld floats) -> boxes of box_rows x 32 floats
static bool make_tmap(CUtensorMap* m, const float* base, int K, int rows, size_t ld, int box_rows) {
  return encode_tmap_2d(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, K, rows, ld * sizeof(float), tg::BK, box_rows);
}

// fp16 [rows, K] row-major (ld halfs) -> boxes of box_rows x 64 halfs (128 bytes)
static bool make_tmap16(CUtensorMap* m, const __half* base, int K, int rows, size_t ld, int box_rows) {
  return encode_tmap_2d(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, K, rows, ld * sizeof(__half), 2 * tg::BK, box_rows);
}

constexpr int TGEMM_THREADS = tg::CONSUMERS + 32;  // two consumer warpgroups + producer warp

static int tgemm_sm_count() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return sms;
}

// fixed-order sum of split-K slabs (fsn_train.cu)
int splitk_reduce_launch(const float* part, int S, int M, int N, float* C, size_t ldc, bool accumulate, cudaStream_t st);

bool tgemm_available() {
  static int ok = -1;
  if (ok < 0) {
    int dev = 0, major = 0, smem = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    ok = (major == 9 && smem >= tg::Cfg<128>::SMEM && tmap_encoder() != nullptr) ? 1 : 0;
  }
  return ok == 1;
}

bool tgemm_supported(const float* A, size_t lda, const float* Bm, size_t ldb, int K) {
  return tgemm_available() && K >= 4 && (lda & 3) == 0 && (ldb & 3) == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0 &&
         (reinterpret_cast<uintptr_t>(Bm) & 15) == 0;
}

// split-K slices of a long-K GEMM with few tiles: minimise waves(tiles * S) / S over the SM slots (1 or 2 resident CTAs
// per SM), slices of >= 2048 k, S * M * N partial sums within the scratch
static int splitk_slices(int M, int N, int K, int BN, const float* scratch, size_t scratch_floats) {
  const int tiles = cdiv(M, tg::BM) * cdiv(N, BN);
  int S = 1;
  if (scratch && K >= 8192 && tiles < 296) {
    const int slots = tgemm_sm_count() * (BN == 128 ? 2 : 1);  // resident CTAs
    double best = 1e30;
    for (int s = 1; s <= 64 && s <= cdiv(K, 2048); ++s) {
      if ((size_t)s * M * N > scratch_floats) break;
      const double cost = (double)cdiv(tiles * s, slots) / s + 1e-4 * s;
      if (cost < best) { best = cost; S = s; }
    }
  }
  return S;
}

// dynamic shared memory opt-in of both tile widths of tgemm_tma_kernel (per device)
static int tgemm_smem_optin() {
  static bool done_by_dev[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  bool& done = done_by_dev[dev & 63];
  if (done) return FSN_OK;
  int rc;
  if ((rc = check_cuda(cudaFuncSetAttribute(tg::tgemm_tma_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            tg::Cfg<256>::SMEM), "tgemm smem attr")) ||
      (rc = check_cuda(cudaFuncSetAttribute(tg::tgemm_tma_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            tg::Cfg<128>::SMEM), "tgemm smem attr")))
    return rc;
  done = true;
  return FSN_OK;
}

// C[M,N] (+)= A[M,K] B[N,K]^T; `scratch` (>= scratch_floats) enables split-K for long-K / few-tile problems
int tgemm_launch(const float* A, size_t lda, const float* Bm, size_t ldb, float* C, size_t ldc, int M, int N, int K,
                 bool accumulate, float* scratch, size_t scratch_floats, cudaStream_t st) {
  if (M <= 0 || N <= 0 || K <= 0) return FSN_OK;
  FSN_REQUIRE(tgemm_supported(A, lda, Bm, ldb, K), FSN_ERR_UNSUPPORTED, "tgemm: operands must be 16-byte aligned rows");
  // a handful of tiles (per-step GEMMs of the full-band stack, 64 rows): narrow tiles + split-K so that the weight
  // matrix is streamed by ~64 CTAs instead of 2-8
  const bool few = scratch && K < 8192 && cdiv(M, tg::BM) * cdiv(N, 128) <= 32;
  // short K, many tiles (hoisted input projections: output-write bound): 128-wide tiles, two CTAs per SM, so one CTA's
  // epilogue overlaps the other's main loop (measured 1081 -> 945 us at K = 384, 778 -> 522 us at K = 32 per 195 k rows)
  const bool short_k_many_tiles = K <= 512 && cdiv(M, tg::BM) >= 1024;
  const int BN = (N >= 256 && N % 256 == 0 && !few && !short_k_many_tiles) ? 256 : 128;
  int S = splitk_slices(M, N, K, BN, scratch, scratch_floats);
  if (few && K >= 256) {
    S = 64 / (cdiv(M, tg::BM) * cdiv(N, BN));
    if (S > K / 128) S = K / 128;
    while (S > 1 && (size_t)S * M * N > scratch_floats) --S;
    if (S < 1) S = 1;
  }
  const int kps = cdiv(cdiv(K, S), tg::BK) * tg::BK;
  S = cdiv(K, kps);
  dim3 grid(cdiv(M, tg::BM), cdiv(N, BN), S);
  float* dst = S > 1 ? scratch : C;
  const size_t ldd = S > 1 ? (size_t)N : ldc;
  const int acc = (S > 1) ? 0 : (accumulate ? 1 : 0);
  CUtensorMap tmA, tmB;
  FSN_REQUIRE(make_tmap(&tmA, A, K, M, lda, tg::BM) && make_tmap(&tmB, Bm, K, N, ldb, BN), FSN_ERR_CUDA,
              "tgemm: tensor-map encoding failed");
  int rc;
  if ((rc = tgemm_smem_optin())) return rc;
  const tg::BlockedOps plain{0, 0, 0, 0, 0};
  if (BN == 256)
    tg::tgemm_tma_kernel<256><<<grid, TGEMM_THREADS, tg::Cfg<256>::SMEM, st>>>(tmA, tmB, dst, ldd, M, N, K, kps, acc, (size_t)M * N, plain);
  else
    tg::tgemm_tma_kernel<128><<<grid, TGEMM_THREADS, tg::Cfg<128>::SMEM, st>>>(tmA, tmB, dst, ldd, M, N, K, kps, acc, (size_t)M * N, plain);
  FSN_CHECK_LAUNCH("tgemm_tma_kernel");
  if (S > 1) return splitk_reduce_launch(scratch, S, M, N, C, ldc, accumulate, st);
  return FSN_OK;
}


// fused recurrent GEMM + LSTM cell of one training-forward step (tg::lstm_fwd_step_kernel); G_t [R,4H] holds the hoisted
// input projection and receives the post-activation gates
bool lstm_fwd_step_supported(const float* Hbuf, const float* w_hh, int H) {
  return (H % 32) == 0 && tgemm_supported(Hbuf, H, w_hh, H, H);
}
// the layer input is multiplied inside the step kernel (no hoisted projection, no P round trip through HBM: 2 x 9.6 GB per
// sub-band layer at config 3).  Measured per training step: no fold 110.5 ms, fold K0 <= 64 105.6 ms, all layers 99.1 ms
static constexpr int STEP_FOLD_MAX_K = 512;  // widest layer input folded in
bool lstm_fwd_step_folds_input(const float* X, const float* w_ih, int K0) {
  return K0 <= STEP_FOLD_MAX_K && tgemm_supported(X, K0, w_ih, K0, K0);
}
// Hprev == nullptr: first step (no recurrent term).  Xt / w_ih (nullable together): fold x_t W_ih^T in, G_t is then
// write-only; otherwise G_t holds the hoisted projection P_t.  h: optional fp16 operands (see LstmStepHalf)
int lstm_fwd_step_launch(const float* Hprev, const float* w_hh, const float* Xt, const float* w_ih, int K0, float* Gt,
                         const float* b_ih, const float* b_hh, const float* C_prev, float* C_out, float* H_out, int R, int H,
                         cudaStream_t st, const LstmStepHalf* h) {
  CUtensorMap tmA, tmB, tmX, tmWx;
  const bool h16 = h && h->w_hh16 && h->H16_out, x16 = h16 && Xt && h->Xt16 && h->w_ih16;
  bool ok;
  if (h16) {
    const __half* a = Hprev ? h->Hprev16 : h->H16_out;  // any valid [R,H] block: not read when nkh == 0
    ok = make_tmap16(&tmA, a, H, R, H, tg::BM) && make_tmap16(&tmB, h->w_hh16, H, 4 * H, H, 32);
  } else {
    const float* a = Hprev ? Hprev : H_out;
    ok = make_tmap(&tmA, a, H, R, H, tg::BM) && make_tmap(&tmB, w_hh, H, 4 * H, H, 32);
  }
  if (Xt && x16) ok = ok && make_tmap16(&tmX, h->Xt16, K0, R, K0, tg::BM) && make_tmap16(&tmWx, h->w_ih16, K0, 4 * H, K0, 32);
  else if (Xt)   ok = ok && make_tmap(&tmX, Xt, K0, R, K0, tg::BM) && make_tmap(&tmWx, w_ih, K0, 4 * H, K0, 32);
  else { tmX = tmA; tmWx = tmB; }
  FSN_REQUIRE(ok, FSN_ERR_CUDA, "lstm_fwd_step: tensor-map encoding failed");
  static bool attr_by_dev[64] = {};
  int dev = 0; cudaGetDevice(&dev); bool& attr = attr_by_dev[dev & 63];
  if (!attr) {
    int rc;
#define FSN_STEP_ATTR(FOLD, HT)                                                                                            \
  if ((rc = check_cuda(cudaFuncSetAttribute(tg::lstm_fwd_step_kernel<FOLD, HT>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                            tg::StepCfg::SMEM), "lstm_fwd_step smem attr")))                               \
    return rc
    FSN_STEP_ATTR(true, 384); FSN_STEP_ATTR(true, 512); FSN_STEP_ATTR(true, 0);
    FSN_STEP_ATTR(false, 384); FSN_STEP_ATTR(false, 512); FSN_STEP_ATTR(false, 0);
#undef FSN_STEP_ATTR
    attr = true;
  }
  const int nkx = Xt ? cdiv(K0, x16 ? 2 * tg::BK : tg::BK) : 0, nkh = Hprev ? cdiv(H, h16 ? 2 * tg::BK : tg::BK) : 0;
  FSN_REQUIRE(nkx + nkh > 0, FSN_ERR_SHAPE, "lstm_fwd_step: nothing to multiply");
  const dim3 grid(cdiv(R, tg::BM), H / 32);
#define FSN_STEP_LAUNCH(FOLD, HT)                                                                                          \
  tg::lstm_fwd_step_kernel<FOLD, HT><<<grid, TGEMM_THREADS, tg::StepCfg::SMEM, st>>>(                                      \
      tmA, tmB, tmX, tmWx, Gt, b_ih, b_hh, C_prev, C_out, H_out, h16 ? h->H16_out : nullptr, R, H, nkx, nkh, x16 ? 1 : 0, \
      h16 ? 1 : 0)
  if (Xt) {
    if (H == 384) FSN_STEP_LAUNCH(true, 384); else if (H == 512) FSN_STEP_LAUNCH(true, 512); else FSN_STEP_LAUNCH(true, 0);
  } else {
    if (H == 384) FSN_STEP_LAUNCH(false, 384); else if (H == 512) FSN_STEP_LAUNCH(false, 512); else FSN_STEP_LAUNCH(false, 0);
  }
#undef FSN_STEP_LAUNCH
  FSN_CHECK_LAUNCH("lstm_fwd_step_kernel");
  return FSN_OK;
}

namespace tg {
__global__ void to_half_kernel(const float* __restrict__ in, size_t n, __half* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = __float2half_rn(in[i]);
}
}  // namespace tg
int to_half_launch(const float* in, size_t n, __half* out, cudaStream_t st) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > tgemm_sm_count() * 8) blocks = tgemm_sm_count() * 8;
  tg::to_half_kernel<<<blocks, 256, 0, st>>>(in, n, out);
  FSN_CHECK_LAUNCH("to_half_kernel");
  return FSN_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Weight-gradient GEMMs  C[M,N] = A^T B  with A [K,M] and B [K,N] row-major (dW = dG^T X, K = T'R up to 1.5 M).
// The tensor-core kernel wants K-major operands; a plain transposed copy [M,K] has a row pitch of K floats (6 MB), so
// every 128-row TMA box touches 128 DRAM pages and the GEMM ran at 15 % of the HBM bandwidth.  Here the transposed copy
// is BLOCK-TILED: tile (128 rows of M, k block of 32) = 16 contiguous KB at ((mt * nkb + kb) * 128 + row) * 32 + kk
// (zero padded in M and K), viewed by TMA as a 2-D array [rows, 32] - one box = one contiguous burst.
namespace tg {
// one CTA: m tile of 128 columns x `kb_per` k blocks of 32 rows; 512-byte row pieces in, one contiguous 16 KB tile out per
// k block.  CTAs are numbered m tile fastest, so the CTAs resident together read whole rows.  colsum_part (nullable):
// [gridDim.y][M] column sums of this CTA's rows (bias gradients = column sums of dG, free while the tile is in SMEM)
__global__ void __launch_bounds__(256) transpose_blocked_kernel(const float* __restrict__ in, size_t K, int M, size_t ld, int nkb,
                                                                 int kb_per, float* __restrict__ out, float* __restrict__ colsum_part) {
  __shared__ float tile[32][129];
  const int tid = threadIdx.x;
  const int mt = blockIdx.x, m0 = mt * 128;
  const int kb0 = blockIdx.y * kb_per;
  const int kb1 = (kb0 + kb_per < nkb) ? kb0 + kb_per : nkb;
  const int col = tid & 127, rsub = tid >> 7;
  const bool col_ok = m0 + col < M;
  float csum = 0.f;
  for (int kb = kb0; kb < kb1; ++kb) {
    const size_t k0 = (size_t)kb * 32;
    float v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const size_t k = k0 + i * 2 + rsub;
      v[i] = (col_ok && k < K) ? __ldcs(in + k * ld + m0 + col) : 0.f;
    }
    __syncthreads();  // the previous tile has been read out
#pragma unroll
    for (int i = 0; i < 16; ++i) tile[i * 2 + rsub][col] = v[i];
    __syncthreads();
    float* o = out + ((size_t)mt * nkb + kb) * (128 * 32);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int e = i * 256 + tid;
      o[e] = tile[e & 31][e >> 5];
    }
    if (colsum_part && tid < 128) {
#pragma unroll
      for (int r = 0; r < 32; ++r) csum += tile[r][tid];  // fixed order
    }
  }
  if (colsum_part && tid < 128 && m0 + tid < M) colsum_part[(size_t)blockIdx.y * M + m0 + tid] = csum;
}
}  // namespace tg

size_t tgemm_blocked_floats(size_t K, int M) { return (size_t)cdiv(M, 128) * 128 * ((K + 31) / 32) * 32; }

// in [K, M] (row stride ld) -> block-tiled transposed copy (tgemm_blocked_floats(K, M) floats).  colsum_part (nullable,
// >= max_slabs * M floats): per-slab column sums, *slabs receives the number of slabs written
int transpose_blocked_launch(const float* in, size_t K, int M, size_t ld, float* out, cudaStream_t st, float* colsum_part,
                             int max_slabs, int* slabs) {
  const int nkb = (int)((K + 31) / 32);
  int kb_per = 8;  // 256 rows per CTA
  if (colsum_part && cdiv(nkb, kb_per) > max_slabs) kb_per = cdiv(nkb, max_slabs);
  const int S = cdiv(nkb, kb_per);
  if (slabs) *slabs = S;
  dim3 grid((unsigned)cdiv(M, 128), (unsigned)S);
  FSN_REQUIRE(S <= 65535, FSN_ERR_SHAPE, "transpose_blocked: K too long");
  tg::transpose_blocked_kernel<<<grid, 256, 0, st>>>(in, K, M, ld, nkb, kb_per, out, colsum_part);
  FSN_CHECK_LAUNCH("transpose_blocked_kernel");
  return FSN_OK;
}

// C[M,N] (+)= A^T B over K, operands block-tiled (transpose_blocked_launch) with nkb_a / nkb_b k blocks per tile row;
// a_kb0 / b_kb0: first k block of each operand (lets dW_hh pair dG[1:] with H[:-1])
int tgemm_blocked_launch(const float* Ablk, int nkb_a, int a_kb0, const float* Bblk, int nkb_b, int b_kb0, float* C, size_t ldc,
                         int M, int N, int K, bool accumulate, float* scratch, size_t scratch_floats, cudaStream_t st) {
  if (M <= 0 || N <= 0 || K <= 0) return FSN_OK;
  FSN_REQUIRE(tmap_encoder(), FSN_ERR_UNSUPPORTED, "tgemm_blocked: cuTensorMapEncodeTiled unavailable");
  const int BN = (N > 128) ? 256 : 128;
  int S = splitk_slices(M, N, K, BN, scratch, scratch_floats);
  const int kps = cdiv(cdiv(K, S), tg::BK) * tg::BK;
  S = cdiv(K, kps);
  dim3 grid(cdiv(M, tg::BM), cdiv(N, BN), S);
  float* dst = S > 1 ? scratch : C;
  const size_t ldd = S > 1 ? (size_t)N : ldc;
  const int acc = (S > 1) ? 0 : (accumulate ? 1 : 0);
  // each operand viewed as [tile rows, 32] floats, one 128-row box per tile; tiles past it: zero fill
  CUtensorMap tmA, tmB;
  FSN_REQUIRE(make_tmap(&tmA, Ablk, tg::BK, cdiv(M, 128) * 128 * nkb_a, tg::BK, 128) &&
                  make_tmap(&tmB, Bblk, tg::BK, cdiv(N, 128) * 128 * nkb_b, tg::BK, 128),
              FSN_ERR_CUDA, "tgemm_blocked: tensor-map encoding failed");
  int rc;
  if ((rc = tgemm_smem_optin())) return rc;
  const tg::BlockedOps bo{1, nkb_a, nkb_b, a_kb0, b_kb0};
  if (BN == 256)
    tg::tgemm_tma_kernel<256><<<grid, TGEMM_THREADS, tg::Cfg<256>::SMEM, st>>>(tmA, tmB, dst, ldd, M, N, K, kps, acc, (size_t)M * N, bo);
  else
    tg::tgemm_tma_kernel<128><<<grid, TGEMM_THREADS, tg::Cfg<128>::SMEM, st>>>(tmA, tmB, dst, ldd, M, N, K, kps, acc, (size_t)M * N, bo);
  FSN_CHECK_LAUNCH("tgemm_tma_kernel");
  if (S > 1) return splitk_reduce_launch(scratch, S, M, N, C, ldc, accumulate, st);
  return FSN_OK;
}
}  // namespace fsn

// debug / unit-test entry point (tests/test_gpu_train.py): C[M,N] (+)= A[M,K] B[N,K]^T on the wgmma path
extern "C" int fsn_debug_tgemm(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M,
                               int N, int K, int accumulate, float* scratch, int64_t scratch_floats,
                               fsn_stream_t stream) {
  return fsn::tgemm_launch(A, (size_t)lda, B, (size_t)ldb, C, (size_t)ldc, M, N, K, accumulate != 0, scratch,
                           (size_t)scratch_floats, (cudaStream_t)stream);
}

// unit-test hook: C[M,N] = A^T B for row-major A [K,M], B [K,N] through the block-tiled transposes + tgemm_blocked_launch
// (a_k0 / b_k0: first k row of each operand, multiples of 32); scratch: tgemm_blocked_floats(K, M) + (K, N padded to the
// tile) floats for the copies, then split-K space
extern "C" int fsn_debug_tgemm_blocked(const float* A, const float* B, float* C, int M, int N, int K, int a_k0, int b_k0,
                                       float* scratch, int64_t scratch_floats, fsn_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const size_t Ka = (size_t)K + a_k0, Kb = (size_t)K + b_k0;
  const size_t fa = fsn::tgemm_blocked_floats(Ka, M), fb = fsn::tgemm_blocked_floats(Kb, N);
  FSN_REQUIRE((a_k0 & 31) == 0 && (b_k0 & 31) == 0 && scratch && (size_t)scratch_floats >= fa + fb, FSN_ERR_SHAPE,
              "tgemm_blocked hook: bad offsets or scratch");
  float *Ab = scratch, *Bb = scratch + fa;
  int rc;
  if ((rc = fsn::transpose_blocked_launch(A, Ka, M, (size_t)M, Ab, st, nullptr, 0, nullptr))) return rc;
  if ((rc = fsn::transpose_blocked_launch(B, Kb, N, (size_t)N, Bb, st, nullptr, 0, nullptr))) return rc;
  return fsn::tgemm_blocked_launch(Ab, (int)((Ka + 31) / 32), a_k0 / 32, Bb, (int)((Kb + 31) / 32), b_k0 / 32, C, (size_t)N, M, N, K,
                                   false, scratch + fa + fb, (size_t)scratch_floats - fa - fb, st);
}

// unit-test hook: the block-tiled transposed copy of in [K, M] (row stride ld) into out (tgemm_blocked_floats(K, M)
// floats); with colsum_part (>= max_slabs * M floats) also the per-slab column sums and their fixed-order total into
// bias_out [M], as layer_weight_grads takes the bias gradients; *slabs (nullable) receives the slab count
extern "C" int fsn_debug_transpose_blocked(const float* in, int64_t K, int M, int64_t ld, float* out, float* colsum_part,
                                           int max_slabs, int* slabs, float* bias_out, fsn_stream_t stream) {
  fsn::launch_counter() = 0;
  FSN_REQUIRE(in && out, FSN_ERR_SHAPE, "transpose_blocked hook: null argument");
  FSN_REQUIRE(K > 0 && M > 0 && ld >= M, FSN_ERR_SHAPE, "transpose_blocked hook: bad shape K=%lld M=%d ld=%lld", (long long)K,
              M, (long long)ld);
  FSN_REQUIRE(!colsum_part || (bias_out && max_slabs > 0), FSN_ERR_SHAPE,
              "transpose_blocked hook: column sums need bias_out and max_slabs >= 1");
  cudaStream_t st = (cudaStream_t)stream;
  int S = 0;
  int rc = fsn::transpose_blocked_launch(in, (size_t)K, M, (size_t)ld, out, st, colsum_part, max_slabs, &S);
  if (rc) return rc;
  if (slabs) *slabs = S;
  return colsum_part ? fsn::colsum_final_launch(colsum_part, S, M, bias_out, nullptr, st) : FSN_OK;
}

// unit-test hook for the fused training-forward step (tg::lstm_fwd_step_kernel; torch.nn.LSTM cell math): one step
//   z = [X W_ih^T  or  the P already in G] + b_ih + b_hh + Hprev W_hh^T;  G <- act(z) (i,f,g,o), C_out, H_out
// Hprev nullable (first step), X nullable (then G [R,4H] holds the hoisted projection on entry).  half != 0: fp16 MMA
// operands for h and the weights, converted here into `scratch` (>= 2 * (2 R H + 4 H (H + K0) + R K0) bytes); X and W_ih
// too when K0 % 8 == 0 (16-byte fp16 rows), else they stay tf32 in the same k loop, the rule of layer_forward_save_tc
extern "C" int fsn_debug_lstm_fwd_step(const float* Hprev, const float* w_hh, const float* X, const float* w_ih, int K0, float* G,
                                       const float* b_ih, const float* b_hh, const float* C_prev, float* C_out, float* H_out,
                                       int R, int H, int half, void* scratch, int64_t scratch_bytes, fsn_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  FSN_REQUIRE(R > 0 && H > 0 && w_hh && G && b_ih && b_hh && C_out && H_out && (!X || (w_ih && K0 > 0)), FSN_ERR_SHAPE,
              "lstm_fwd_step hook: missing arguments");
  FSN_REQUIRE(fsn::lstm_fwd_step_supported(H_out, w_hh, H), FSN_ERR_UNSUPPORTED,
              "lstm_fwd_step hook: needs H %% 32 == 0, 16-byte aligned operands and the TMA driver entry point");
  FSN_REQUIRE(!X || fsn::tgemm_supported(X, K0, w_ih, K0, K0), FSN_ERR_UNSUPPORTED, "lstm_fwd_step hook: X rows must be 16-byte aligned");
  if (!half) return fsn::lstm_fwd_step_launch(Hprev, w_hh, X, w_ih, K0, G, b_ih, b_hh, C_prev, C_out, H_out, R, H, st, nullptr);
  const size_t nh = (size_t)R * H, nw = (size_t)4 * H * H, nx = X ? (size_t)R * K0 : 0, nwx = X ? (size_t)4 * H * K0 : 0;
  FSN_REQUIRE((H % 8) == 0, FSN_ERR_UNSUPPORTED, "lstm_fwd_step hook: fp16 rows must be 16-byte aligned");
  const bool x16 = X && (K0 % 8) == 0;
  FSN_REQUIRE(scratch && (size_t)scratch_bytes >= 2 * (2 * nh + nw + nx + nwx) + 1024, FSN_ERR_WORKSPACE,
              "lstm_fwd_step hook: scratch too small");
  auto up = [](size_t n) { return (n + 127) & ~(size_t)127; };  // keep every block 256-byte aligned
  __half* hp = (__half*)scratch;
  __half* ho = hp + up(nh);
  __half* wh = ho + up(nh);
  __half* xx = wh + up(nw);
  __half* wx = xx + up(nx);
  FSN_REQUIRE((size_t)((char*)(wx + up(nwx)) - (char*)scratch) <= (size_t)scratch_bytes, FSN_ERR_WORKSPACE,
              "lstm_fwd_step hook: scratch too small");
  int rc;
  if (Hprev && (rc = fsn::to_half_launch(Hprev, nh, hp, st))) return rc;
  if ((rc = fsn::to_half_launch(w_hh, nw, wh, st))) return rc;
  if (x16 && ((rc = fsn::to_half_launch(X, nx, xx, st)) || (rc = fsn::to_half_launch(w_ih, nwx, wx, st)))) return rc;
  fsn::LstmStepHalf hs{Hprev ? hp : nullptr, wh, x16 ? xx : nullptr, x16 ? wx : nullptr, ho};
  return fsn::lstm_fwd_step_launch(Hprev, w_hh, X, w_ih, K0, G, b_ih, b_hh, C_prev, C_out, H_out, R, H, st, &hs);
}
