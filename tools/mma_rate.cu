// Stand-alone rate of the sub-band kernel's MMA sequence (DESIGN 4.1): m64n32k16 wgmma with both operands in shared
// memory, issued per ring stage exactly as sb_lstm_tc_kernel issues them (x3: a hi stage of 16 MMAs - hi.hi, hi.lo per
// gate and k16 - then a lo stage of 8; single pass: 8), one commit per stage, then wait_group<WAIT>.  1, 2 or 3
// consumer warpgroups issue at once, each on its own 16 KB A block (same 64B swizzle as the weight stages) against one
// shared 128B-swizzled B block (hi + lo); optionally warp 0 streams 16 KB bulk copies from L2 into a 4-slot ring of
// its own at the same time.  No barriers between the consumers; operands are zero.  132 CTAs, one per SM.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/mma_rate tools/mma_rate.cu && /tmp/mma_rate
//
// Prints per configuration the cycles per stage of one warpgroup and the per-SM cycles per MMA.
//
// The loop above has loop-invariant descriptors and no barriers, which the kernel's stage loop does not have.  The
// `ctl` variants (one warpgroup, no TMA stream) put the kernel's per-stage pieces around the same MMAs, as the kernel
// before and after its stage-loop rewrite issues them:
//   (a) every descriptor built per MMA (desc_sw64 / desc_sw128) from a ring slot and a state k range that change every
//       stage (runtime strides, 0 here, so the operands and their banks stay those of the plain loop);
//   (b) a try-wait on an already completed mbarrier per stage and the release arrive of the stage before, by lane 0 of
//       the warps q < CL (CL a kernel argument) in a divergent region, as release_stage did;
//   (c) both: the former kernel's stage loop;
//   (u) the rewritten loop: warp-uniform slot and phase, descriptor words stepped by constants (wg::mma_f16_n32_w), the
//       warp-wide wait and elected, predicated arrives.
#include <cuda_runtime.h>
#include <stdio.h>

#include "../fullsubnet_b200/csrc/fsn_tc_ptx.cuh"
#include "../fullsubnet_b200/csrc/fsn_wgmma.cuh"
using namespace fsn;
using namespace fsn::ptx;

constexpr int GRID = 132, ITERS = 2000, SMEM = 200 * 1024;

// ORDER 0: per gate hi.hi then hi.lo (the kernel's order); 1: the four hi.hi before the four hi.lo
template <bool X3, int ORDER, int WAIT>
__global__ void __launch_bounds__(512, 1) mma_rate(int nwg, int prod, long long* out, const uint8_t* gsrc) {
  extern __shared__ uint8_t raw[];
  uint8_t* sm = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + 120 * 1024);
  for (int i = threadIdx.x; i < 120 * 1024 / 16; i += blockDim.x) reinterpret_cast<uint4*>(sm)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0)
    for (int i = 0; i < 4; ++i) mbar_init(&bars[i], 1);
  fence_proxy_async_smem();
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < 4) {
    if (warp == 0 && prod) {  // one 16 KB bulk copy per stage the consumers run, 4 in flight
      const int n = nwg * ITERS * (X3 ? 2 : 1);
      const long long t0 = clock64();
      for (int i = 0; i < n + 4; ++i) {
        const int s = i & 3;
        if (i >= 4) mbar_wait_cta<false>(&bars[s], ((i >> 2) - 1) & 1);
        if (i < n && elect_one()) {
          mbar_expect_tx(&bars[s], 16384);
          bulk_g2s(sm + 56 * 1024 + s * 16384, gsrc + (size_t)(i % 64) * 16384, 16384, &bars[s]);
        }
        __syncwarp();
      }
      if (lane == 0) out[blockIdx.x * 8 + 7] = clock64() - t0;
    }
    return;
  }
  const int m = (warp - 4) >> 2;
  if (m >= nwg) return;
  const uint32_t wa = smem_u32(sm + m * 16384), sb = smem_u32(sm + 48 * 1024);
  float acc[4][16];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[g][i] = 0.f;
    wg::fence_operand(acc[g]);
  }
  named_sync(1 + m, 128);
  const long long t0 = clock64();
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int part = 0; part < (X3 ? 2 : 1); ++part) {
      wg::fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const uint64_t bd = wg::desc_sw128(sb + kk * 32), bl = wg::desc_sw128(sb + 4096 + kk * 32);
        if (ORDER == 0 || !X3 || part == 1) {
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const uint64_t ad = wg::desc_sw64(wa + g * 4096 + kk * 32);
            wg::mma_f16_n32(acc[g], ad, bd, 1u);
            if (X3 && part == 0) wg::mma_f16_n32(acc[g], ad, bl, 1u);
          }
        } else {
#pragma unroll
          for (int g = 0; g < 4; ++g) wg::mma_f16_n32(acc[g], wg::desc_sw64(wa + g * 4096 + kk * 32), bd, 1u);
#pragma unroll
          for (int g = 0; g < 4; ++g) wg::mma_f16_n32(acc[g], wg::desc_sw64(wa + g * 4096 + kk * 32), bl, 1u);
        }
      }
      wg::commit();
      wg::wait<WAIT>();
    }
  }
  wg::wait<0>();
#pragma unroll
  for (int g = 0; g < 4; ++g) wg::fence_operand(acc[g]);
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int i = 0; i < 16; ++i) s += acc[g][i];
  if ((threadIdx.x & 127) == 0) out[blockIdx.x * 8 + m] = (t1 - t0) + (s != 0.f ? 1 : 0);
}

template <bool X3, int ORDER, int WAIT>
static void run(const char* name, long long* d_out, const uint8_t* gsrc) {
  cudaFuncSetAttribute(mma_rate<X3, ORDER, WAIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
  for (int prod = 0; prod < 2; ++prod)
    for (int nwg = 1; nwg <= 3; ++nwg) {
      cudaMemset(d_out, 0, GRID * 8 * sizeof(long long));
      mma_rate<X3, ORDER, WAIT><<<GRID, 512, SMEM>>>(nwg, prod, d_out, gsrc);
      const cudaError_t e = cudaDeviceSynchronize();
      long long h[GRID * 8];
      cudaMemcpy(h, d_out, sizeof(h), cudaMemcpyDeviceToHost);
      double cyc = 0;
      for (int b = 0; b < GRID; ++b)
        for (int m = 0; m < nwg; ++m) cyc += (double)h[b * 8 + m] / (GRID * nwg);
      const int stages = ITERS * (X3 ? 2 : 1), mmas = ITERS * (X3 ? 24 : 8);
      printf("%-12s TMA stream %d, %d warpgroup(s): %s  %6.1f cycles per stage and warpgroup, %5.1f cycles per MMA per SM\n",
             name, prod, nwg, cudaGetErrorString(e), cyc / stages, cyc / ((double)mmas * nwg));
    }
}

// stage-loop controls (header): VAR 0 plain, 1 (a), 2 (b), 3 (c), 4 (u); one warpgroup (warps 4..7), nst ring slots
template <bool X3, int VAR>
__global__ void __launch_bounds__(512, 1) stage_ctl(int nst, uint32_t slot_stride, uint32_t k_stride, int CL,
                                                    long long* out) {
  constexpr int PARTS = X3 ? 2 : 1;
  extern __shared__ uint8_t raw[];
  uint8_t* sm = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + 120 * 1024);  // [0]: completed "w_full", [1]: "w_empty"
  for (int i = threadIdx.x; i < 120 * 1024 / 16; i += blockDim.x) reinterpret_cast<uint4*>(sm)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], (1u << 20) - 1);
    mbar_arrive(&bars[0]);  // phase 0 complete: every parity-0 wait below succeeds at its first poll
  }
  fence_proxy_async_smem();
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < 4 || warp >= 8) return;
  const int q = VAR == 4 ? __shfl_sync(0xffffffffu, warp & 3, 0) : warp & 3;
  const uint32_t wbase = smem_u32(sm), sbase = smem_u32(sm + 48 * 1024), LO = 4096;
  const uint32_t full = smem_u32(&bars[0]), empty = smem_u32(&bars[1]);
  const uint32_t rel_local = CL == 1 && q == 0;
  float acc[4][16];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[g][i] = 0.f;
    wg::fence_operand(acc[g]);
  }
  int stage = 0, prev = -1;
  uint32_t j = 0;
  named_sync(1, 128);
  const long long t0 = clock64();
  for (int it = 0; it < ITERS; ++it, ++j) {
#pragma unroll
    for (int part = 0; part < PARTS; ++part) {
      if (VAR & 2) mbar_wait_cta<false>(&bars[0], 0);
      if (VAR == 4) mbar_wait_cta_warp(full, 0);
      wg::fence();
      const uint32_t wa = (VAR & 1) || VAR == 4 ? wbase + stage * slot_stride : wbase;
      const uint32_t sb = (VAR & 1) || VAR == 4 ? sbase + (j >> 1) * k_stride + (j & 1) * k_stride : sbase;
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const uint64_t bd = wg::desc_sw128(sb + kk * 32), bl = wg::desc_sw128(sb + LO + kk * 32);
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          if (VAR == 4) {
            const uint32_t a_lo = wg::desc_lo(wa), b_lo = wg::desc_lo(sb);
            wg::mma_f16_n32_w(acc[g], a_lo, g * 256 + kk * 2, wg::DESC_SW64_HI, b_lo, kk * 2, wg::DESC_SW128_HI);
            if (X3 && part == 0)
              wg::mma_f16_n32_w(acc[g], a_lo, g * 256 + kk * 2, wg::DESC_SW64_HI, b_lo, LO / 16 + kk * 2, wg::DESC_SW128_HI);
          } else {
            const uint64_t ad = wg::desc_sw64(wa + g * 4096 + kk * 32);
            wg::mma_f16_n32(acc[g], ad, bd, 1u);
            if (X3 && part == 0) wg::mma_f16_n32(acc[g], ad, bl, 1u);
          }
        }
      }
      wg::commit();
      wg::wait<1>();
      if ((VAR & 2) && prev >= 0 && lane == 0 && q < CL) {
        if (CL == 1) mbar_arrive(&bars[1]);
        else mbar_arrive_remote(&bars[1], (uint32_t)(2 * q));
      }
      if (VAR == 4) mbar_arrive_elect_if(empty, (prev >= 0) & rel_local);
      prev = stage;
      if (++stage == nst) stage = 0;
    }
  }
  wg::wait<0>();
#pragma unroll
  for (int g = 0; g < 4; ++g) wg::fence_operand(acc[g]);
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int i = 0; i < 16; ++i) s += acc[g][i];
  if (threadIdx.x == 128) out[blockIdx.x] = (t1 - t0) + (s != 0.f ? 1 : 0);
}

template <bool X3, int VAR>
static void run_ctl(const char* name, long long* d_out) {
  cudaFuncSetAttribute(stage_ctl<X3, VAR>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
  cudaMemset(d_out, 0, GRID * 8 * sizeof(long long));
  stage_ctl<X3, VAR><<<GRID, 512, SMEM>>>(4, 0u, 0u, 1, d_out);
  const cudaError_t e = cudaDeviceSynchronize();
  long long h[GRID];
  cudaMemcpy(h, d_out, sizeof(h), cudaMemcpyDeviceToHost);
  double cyc = 0;
  for (int b = 0; b < GRID; ++b) cyc += (double)h[b] / GRID;
  const int stages = ITERS * (X3 ? 2 : 1), mmas = ITERS * (X3 ? 24 : 8);
  printf("%-16s 1 warpgroup: %s  %6.1f cycles per stage, %5.1f cycles per MMA\n", name, cudaGetErrorString(e),
         cyc / stages, cyc / mmas);
}

int main() {
  long long* d_out;
  uint8_t* gsrc;
  cudaMalloc(&d_out, GRID * 8 * sizeof(long long));
  cudaMalloc(&gsrc, 64 * 16384);
  cudaMemset(gsrc, 0, 64 * 16384);
  run<true, 0, 1>("x3 wait<1>", d_out, gsrc);
  run<true, 1, 1>("x3 hh-first", d_out, gsrc);
  run<true, 1, 2>("x3 wait<2>", d_out, gsrc);
  run<true, 0, 0>("x3 wait<0>", d_out, gsrc);
  run<false, 0, 1>("f16 wait<1>", d_out, gsrc);
  run<false, 0, 0>("f16 wait<0>", d_out, gsrc);
  run_ctl<true, 0>("x3 ctl plain", d_out);
  run_ctl<true, 1>("x3 ctl (a) desc", d_out);
  run_ctl<true, 2>("x3 ctl (b) bars", d_out);
  run_ctl<true, 3>("x3 ctl (c) both", d_out);
  run_ctl<true, 4>("x3 ctl (u) new", d_out);
  run_ctl<false, 0>("f16 ctl plain", d_out);
  run_ctl<false, 1>("f16 ctl (a) desc", d_out);
  run_ctl<false, 2>("f16 ctl (b) bars", d_out);
  run_ctl<false, 3>("f16 ctl (c) both", d_out);
  run_ctl<false, 4>("f16 ctl (u) new", d_out);
  cudaFree(d_out);
  cudaFree(gsrc);
  return 0;
}
