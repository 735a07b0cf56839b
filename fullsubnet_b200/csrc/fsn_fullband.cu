// Full-band 2-layer LSTM as ONE persistent cooperative kernel (fp32 FMA, exact-class arithmetic).
//
// Reference semantics: audio_zen/model/module/sequence_model.py:106-125 (nn.LSTM part) as used by
// recipes/dns_interspeech_2020/fullsubnet/model.py:92-95 (rows = clips, input = normalised magnitude).
//
// Decomposition.  The batch is small (B clips) and the recurrence is serial in t, so the hidden
// dimension is spread over the whole chip: CTA j owns `upc` hidden units of BOTH layers, i.e.
// 4*upc gate rows of W_ih/W_hh per layer, which it keeps resident in shared memory as fp32 for the
// whole sequence (F=257, H=512, upc=4: 16 x (769 + 1024) x 4 B = 115 KB) - weights are read from
// HBM exactly once.  The two layers run as a wavefront: in phase p every CTA computes its slice of
// layer 0 at step p and of layer 1 at step p-1; both only need data of phase p-1
// (x_p, h0_{p-1}, h1_{p-2}), so there is ONE grid-wide barrier per time step.  h is exchanged through
// global memory (L2); c stays in registers.
//
// Thread mapping (512 threads): row = tid/2 (clip), half = tid%2 -> gate columns [8*half, 8*half+8)
// of the CTA's 16 (= 2 complete hidden units), for both layers: 32 accumulators per thread.
//
// Below the kernel: seq_stack_forward, the SequenceModel every inference forward runs its clip-major LSTM stacks through
// (this kernel, the per-step kernels or the tensor-core layers of fsn_lstm_rec_tc.cu).
#include <cooperative_groups.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>

#include "fsn_internal.cuh"

namespace fsn {
namespace fb {

constexpr int ROWS = 256;      // clips per launch (host loops over chunks)
constexpr int THREADS = 256;
constexpr int KC = 16;         // k-chunk staged in shared memory
constexpr int RS = KC + 4;      // row stride (floats) of the A tile [row][k]: 80 B keeps 16-byte cp.async aligned and,
                               // with rows rq+8i per thread, makes the 128-bit reads bank-conflict free
constexpr int MAX_UPC = 4;     // hidden units per CTA (=> 16 gate columns)
constexpr int NSTAGE = 5;      // cp.async ring depth of the A tiles

struct Args {
  const float* w_ih[2]; const float* w_hh[2]; const float* b_ih[2]; const float* b_hh[2];
  const float* x;        // magT [B, Tp, F]
  const float* inv1;     // [B]
  float* h0buf;          // [2][B][H] ping-pong
  float* h1all;          // [B][Tp][H]
  unsigned int* barrier; // grid barrier counter (zeroed by the host before launch)
  int B, F, H0, H1, Tp, upc, G;  // layer 0: F -> H0, layer 1: H0 -> H1
  FbState io;            // streaming: carried state (all null / fin_step -1 for a whole sequence)
};

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int v;
    unsigned int spins = 0;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
      if (++spins > (1u << 28)) { printf("fsn fb: grid barrier timeout\n"); __trap(); }
    } while (v < target);
  }
  __syncthreads();
}

// 4 rows x 4 gate columns (one hidden unit) per thread and layer: acc[r][g] += a[r] * w[g]
__device__ __forceinline__ void fma_4x4(float (&acc)[16], const float (&av)[4], const float4 w) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    acc[r * 4 + 0] = fmaf(av[r], w.x, acc[r * 4 + 0]);
    acc[r * 4 + 1] = fmaf(av[r], w.y, acc[r * 4 + 1]);
    acc[r * 4 + 2] = fmaf(av[r], w.z, acc[r * 4 + 2]);
    acc[r * 4 + 3] = fmaf(av[r], w.w, acc[r * 4 + 3]);
  }
}

// shared-memory weight slice layout: W[layer][k][16] (gate column c = unit_local*4 + gate), k over
// [x | h_prev] of that layer; zero for units beyond H.
// Thread mapping (256 threads): warp w, rq = lane/4 -> rows 32w+rq+8i (i<4), cq = lane%4 -> unit u0+cq (4 gates),
// both layers: a 256x16(x2) register-tiled GEMM per phase, FMA-pipe bound.
__global__ void __launch_bounds__(THREADS, 1) fb_lstm_kernel(const Args a) {
  extern __shared__ __align__(16) float smem_f[];
  const int F = a.F, H0 = a.H0, H1 = a.H1, Tp = a.Tp, B = a.B;
  const int K0 = F + H0, K1 = H0 + H1;
  float* W0 = smem_f;                 // [K0][16]
  float* W1 = W0 + (size_t)K0 * 16;   // [K1][16]
  float* At = W1 + (size_t)K1 * 16;   // [NSTAGE][ROWS][RS]
  const int tid = threadIdx.x;
  const int cq = tid & 3;
  const int row_base = (tid >> 5) * 32 + ((tid & 31) >> 2);  // thread rows: row_base + 8*i
  const int u0 = blockIdx.x * a.upc;  // first hidden unit of this CTA
  const int u = u0 + cq;
  const bool unit_ok0 = cq < a.upc && u < H0, unit_ok1 = cq < a.upc && u < H1;

  // ---- one-time: weight slice -> shared memory
  for (int idx = tid; idx < K0 * 16; idx += THREADS) {
    const int k = idx >> 4, c = idx & 15;
    const int ul = c >> 2, g = c & 3, uu = u0 + ul;
    float w = 0.f;
    if (ul < a.upc && uu < H0) {
      const size_t wr = (size_t)g * H0 + uu;
      w = (k < F) ? a.w_ih[0][wr * F + k] : a.w_hh[0][wr * H0 + (k - F)];
    }
    W0[idx] = w;
  }
  for (int idx = tid; idx < K1 * 16; idx += THREADS) {
    const int k = idx >> 4, c = idx & 15;
    const int ul = c >> 2, g = c & 3, uu = u0 + ul;
    float w = 0.f;
    if (ul < a.upc && uu < H1) {
      const size_t wr = (size_t)g * H1 + uu;
      w = (k < H0) ? a.w_ih[1][wr * H0 + k] : a.w_hh[1][wr * H1 + (k - H0)];
    }
    W1[idx] = w;
  }
  // the A tiles' padding columns [KC, RS) are never loaded.  When H1 % KC != 0 the last chunk of the h1 segment reads
  // weight rows past W1, i.e. the start of the first tile, and multiplies them by zero-filled A: zero the padding once so
  // that stale shared memory (an Inf or NaN) cannot turn those products into NaN
  for (int idx = tid; idx < NSTAGE * ROWS; idx += THREADS)
    *reinterpret_cast<float4*>(At + (size_t)idx * RS + KC) = make_float4(0.f, 0.f, 0.f, 0.f);
  float bias0[4], bias1[4];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    bias0[g] = unit_ok0 ? a.b_ih[0][g * H0 + u] + a.b_hh[0][g * H0 + u] : 0.f;
    bias1[g] = unit_ok1 ? a.b_ih[1][g * H1 + u] + a.b_hh[1][g * H1 + u] : 0.f;
  }
  float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};  // cell state: 4 rows, both layers
  if (a.io.c_init[0])
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int row = row_base + 8 * r;
      if (row < B && unit_ok0) c0[r] = a.io.c_init[0][(size_t)row * H0 + u];
      if (row < B && unit_ok1) c1[r] = a.io.c_init[1][(size_t)row * H1 + u];
    }
  float rs[4];  // 1/(mu+1e-5) of the thread's 4 clips (model.py:92), applied to the x segment
#pragma unroll
  for (int r = 0; r < 4; ++r) rs[r] = (row_base + 8 * r < B) ? (a.inv1 ? a.inv1[row_base + 8 * r] : 1.f) : 0.f;

  // A-tile loader: 16-byte cp.async for the h segments (thread -> rows tid/4 + 64 j, k = 4*(tid%4));
  // 4-byte cp.async for the x segment whose rows (F floats) are not 16-byte aligned
  const int l_row0 = (tid >> 5) * 32 + ((tid & 31) >> 4), l_k = tid & 15;
  const int v_row0 = tid >> 2, v_k = (tid & 3) * 4;
  const bool vec_ok1 = (H0 % KC) == 0, vec_ok2 = (H1 % KC) == 0;  // 16-byte cp.async needs aligned, full chunks
  const uint32_t At_s = (uint32_t)__cvta_generic_to_shared(At);
  __syncthreads();

  for (int p = 0; p <= Tp; ++p) {
    const bool do0 = p < Tp;    // layer 0 at step p
    const bool do1 = p >= 1;    // layer 1 at step p-1
    float acc0[16], acc1[16];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int g = 0; g < 4; ++g) { acc0[r * 4 + g] = bias0[g]; acc1[r * 4 + g] = bias1[g]; }
    // h0_{p-1} (row stride H0) and h1_{p-2} (row stride h1_rs); the state entering step 0 from io.h_init when given
    const bool init0 = p == 0 && a.io.h_init[0], init1 = p == 1 && a.io.h_init[1];
    const float* h0_prev = init0 ? a.io.h_init[0] : a.h0buf + (size_t)((p + 1) & 1) * B * H0;
    const float* h1_prev = init1 ? a.io.h_init[1] : a.h1all + (size_t)(p >= 2 ? p - 2 : 0) * H1;
    const size_t h1_rs = init1 ? (size_t)H1 : (size_t)Tp * H1;
    // three k segments: x_p (F, layer 0), h0_{p-1} (H, both layers), h1_{p-2} (H, layer 1), walked as one
    // flat list of KC-wide chunks through a cp.async ring of NSTAGE tiles (NSTAGE-1 chunks in flight hide
    // the L2 latency; out-of-range elements are zero-filled with src-size 0).  Plain (non-.cg) loads are
    // correct here: every phase starts after the acquire of the grid barrier.
    const int nch_f = (F + KC - 1) / KC, nch_h = (H0 + KC - 1) / KC, nch_h1 = (H1 + KC - 1) / KC;
    const int c_begin = do0 ? 0 : nch_f;                       // skip x when layer 0 is finished
    const int c_end = nch_f + (p >= 1 || init0 ? nch_h : 0) + (p >= 2 || init1 ? nch_h1 : 0);
    auto issue = [&](int ci) {
      if (ci < c_end) {
        int seg = 0, k0 = ci * KC;
        if (ci >= nch_f) { seg = 1; k0 = (ci - nch_f) * KC; }
        if (ci >= nch_f + nch_h) { seg = 2; k0 = (ci - nch_f - nch_h) * KC; }
        const uint32_t Ab = At_s + (uint32_t)((ci - c_begin) % NSTAGE) * (ROWS * RS * 4);
        if ((seg == 1 && vec_ok1) || (seg == 2 && vec_ok2)) {
          const float* base = (seg == 1) ? h0_prev + k0 : h1_prev + k0;
          const unsigned rstride = (seg == 1) ? (unsigned)H0 : (unsigned)h1_rs;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int r = v_row0 + 64 * j;
            const bool ok = r < B;  // H % KC == 0: these chunks are always full
            const float* src = ok ? base + (size_t)r * rstride + v_k : a.x;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(Ab + (uint32_t)((r * RS + v_k) * 4)), "l"(src),
                         "r"(ok ? 16 : 0)
                         : "memory");
          }
        } else {
          const int klen = (seg == 0) ? F : ((seg == 1) ? H0 : H1);
          const int k = k0 + l_k;
          const bool kok = k < klen;
          const float* base = (seg == 0) ? a.x + (size_t)p * F + k : ((seg == 1) ? h0_prev + k : h1_prev + k);
          const size_t rstride = (seg == 0) ? (size_t)Tp * F : ((seg == 1) ? (size_t)H0 : h1_rs);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int r = l_row0 + 2 * j;
            const bool ok = kok && r < B;
            const float* src = ok ? base + (size_t)r * rstride : a.x;  // any valid address when zero-filled
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(Ab + (uint32_t)((r * RS + l_k) * 4)), "l"(src),
                         "r"(ok ? 4 : 0)
                         : "memory");
          }
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");  // (empty groups keep the wait count uniform)
    };
#pragma unroll 1
    for (int i = 0; i < NSTAGE - 1; ++i) issue(c_begin + i);
    for (int ci = c_begin; ci < c_end; ++ci) {
      asm volatile("cp.async.wait_group %0;" ::"n"(NSTAGE - 2) : "memory");
      __syncthreads();                 // chunk ci landed for everyone; buffer of chunk ci-1 is free
      issue(ci + NSTAGE - 1);
      const float* Ab = At + (size_t)((ci - c_begin) % NSTAGE) * ROWS * RS;
      if (row_base >= B) continue;
      int seg = 0, k0 = ci * KC;
      if (ci >= nch_f) { seg = 1; k0 = (ci - nch_f) * KC; }
      if (ci >= nch_f + nch_h) { seg = 2; k0 = (ci - nch_f - nch_h) * KC; }
      const float* w0 = ((seg == 0) ? W0 : W0 + (size_t)F * 16) + (size_t)k0 * 16 + cq * 4;   // layer-0 rows
      const float* w1 = ((seg == 1) ? W1 : W1 + (size_t)H0 * 16) + (size_t)k0 * 16 + cq * 4;  // layer-1 rows
      const bool use0 = (seg <= 1) && do0, use1 = (seg >= 1) && do1;
      const float* ar = Ab + row_base * RS;
      // rows beyond klen inside the chunk are zero-filled, so the full KC is always safe to consume; the three
      // segment kinds get their own straight-line code (branch once per chunk, not per FMA group)
      auto consume = [&](auto use0_c, auto use1_c, auto scale_c) {
        constexpr bool U0 = decltype(use0_c)::value, U1 = decltype(use1_c)::value, SC = decltype(scale_c)::value;
#pragma unroll
        for (int k4 = 0; k4 < KC; k4 += 4) {
          float4 a4[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) a4[r] = *reinterpret_cast<const float4*>(ar + (8 * r) * RS + k4);
          if (SC) {
#pragma unroll
            for (int r = 0; r < 4; ++r) { a4[r].x *= rs[r]; a4[r].y *= rs[r]; a4[r].z *= rs[r]; a4[r].w *= rs[r]; }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float av[4] = {q == 0 ? a4[0].x : q == 1 ? a4[0].y : q == 2 ? a4[0].z : a4[0].w,
                                 q == 0 ? a4[1].x : q == 1 ? a4[1].y : q == 2 ? a4[1].z : a4[1].w,
                                 q == 0 ? a4[2].x : q == 1 ? a4[2].y : q == 2 ? a4[2].z : a4[2].w,
                                 q == 0 ? a4[3].x : q == 1 ? a4[3].y : q == 2 ? a4[3].z : a4[3].w};
            if (U0) fma_4x4(acc0, av, *reinterpret_cast<const float4*>(w0 + (k4 + q) * 16));
            if (U1) fma_4x4(acc1, av, *reinterpret_cast<const float4*>(w1 + (k4 + q) * 16));
          }
        }
      };
      using T_ = std::true_type; using F_ = std::false_type;
      if (seg == 0) { if (use0) consume(T_{}, F_{}, T_{}); }
      else if (use0 && use1) consume(T_{}, T_{}, F_{});
      else if (use0) consume(T_{}, F_{}, F_{});
      else if (use1) consume(F_{}, T_{}, F_{});
    }
    // ---- cell updates of the thread's unit for its 4 rows (gate order i,f,g,o), write h
    if (unit_ok0 || unit_ok1) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = row_base + 8 * r;
        if (row >= B) continue;
        // io.restart: the row's state after step restart - 1 is zero (its sequence starts again at that step)
        const int rst = a.io.restart ? a.io.restart[row] : -1;
        if (do0 && unit_ok0) {
          float c = sigmoidf_(acc0[r * 4 + 1]) * c0[r] + sigmoidf_(acc0[r * 4 + 0]) * tanhf(acc0[r * 4 + 2]);
          float h = sigmoidf_(acc0[r * 4 + 3]) * tanhf(c);
          if (p + 1 == rst) c = h = 0.f;
          c0[r] = c;
          a.h0buf[(size_t)(p & 1) * B * H0 + (size_t)row * H0 + u] = h;
          if (p == a.io.fin_step) { a.io.h_fin[0][(size_t)row * H0 + u] = h; a.io.c_fin[0][(size_t)row * H0 + u] = c; }
        }
        if (do1 && unit_ok1) {
          float c = sigmoidf_(acc1[r * 4 + 1]) * c1[r] + sigmoidf_(acc1[r * 4 + 0]) * tanhf(acc1[r * 4 + 2]);
          float h = sigmoidf_(acc1[r * 4 + 3]) * tanhf(c);
          if (p == rst) c = h = 0.f;
          c1[r] = c;
          a.h1all[((size_t)row * Tp + (p - 1)) * H1 + u] = h;
          if (p - 1 == a.io.fin_step) { a.io.h_fin[1][(size_t)row * H1 + u] = h; a.io.c_fin[1][(size_t)row * H1 + u] = c; }
        }
      }
    }
    grid_barrier(a.barrier, (unsigned int)(p + 1) * gridDim.x);
  }
}

}  // namespace fb

size_t fb_persistent_smem(int F, int H0, int H1) {
  return ((size_t)(F + H0) * 16 + (size_t)(H0 + H1) * 16 + (size_t)fb::NSTAGE * fb::ROWS * fb::RS) * sizeof(float);
}

bool fb_persistent_supported(int F, int H0, int H1) {
  static int coop = -1, max_smem = 0, sms = 132;
  if (coop < 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  const int Hm = H0 > H1 ? H0 : H1;
  return coop == 1 && fb_persistent_smem(F, H0, H1) <= (size_t)max_smem && cdiv(Hm, fb::MAX_UPC) <= sms;
}

// The 2-layer LSTM wavefront, one persistent launch per chunk of <= 256 rows (fb::ROWS).
int fb_persistent_launch(const fsn_lstm_layer* L, const float* x, const float* inv1, float* h0buf, float* h1all,
                         unsigned int* barrier, int R, int F, int H0, int H1, int Tp, cudaStream_t st, const FbState* io) {
  fb::Args a;
  memset(&a.io, 0, sizeof(a.io));
  a.io.fin_step = -1;
  for (int l = 0; l < 2; ++l) { a.w_ih[l] = L[l].w_ih; a.w_hh[l] = L[l].w_hh; a.b_ih[l] = L[l].b_ih; a.b_hh[l] = L[l].b_hh; }
  a.h0buf = h0buf; a.barrier = barrier;
  a.F = F; a.H0 = H0; a.H1 = H1; a.Tp = Tp;
  int sms = 132;
  { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  const int Hm = H0 > H1 ? H0 : H1;
  int upc = 1;
  while (upc < fb::MAX_UPC && cdiv(Hm, upc) > sms) ++upc;
  FSN_REQUIRE(cdiv(Hm, upc) <= sms, FSN_ERR_UNSUPPORTED, "persistent LSTM: hidden size %d too large for %d SMs", Hm, sms);
  a.upc = upc; a.G = cdiv(Hm, upc);
  const size_t smem = fb_persistent_smem(F, H0, H1);
  int rc = check_cuda(cudaFuncSetAttribute(fb::fb_lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                      "fb_lstm smem attr");
  if (rc) return rc;
  for (int r0 = 0; r0 < R; r0 += fb::ROWS) {
    a.B = (R - r0 < fb::ROWS) ? R - r0 : fb::ROWS;
    a.x = x + (size_t)r0 * Tp * F; a.inv1 = inv1 ? inv1 + r0 : nullptr; a.h1all = h1all + (size_t)r0 * Tp * H1;
    if (io) {  // the chunk's rows of every state table
      const int Hl[2] = {H0, H1};
      for (int l = 0; l < 2; ++l) {
        a.io.h_init[l] = io->h_init[l] ? io->h_init[l] + (size_t)r0 * Hl[l] : nullptr;
        a.io.c_init[l] = io->c_init[l] ? io->c_init[l] + (size_t)r0 * Hl[l] : nullptr;
        a.io.h_fin[l] = io->h_fin[l] ? io->h_fin[l] + (size_t)r0 * Hl[l] : nullptr;
        a.io.c_fin[l] = io->c_fin[l] ? io->c_fin[l] + (size_t)r0 * Hl[l] : nullptr;
      }
      a.io.restart = io->restart ? io->restart + r0 : nullptr;
      a.io.fin_step = io->fin_step;
    }
    rc = check_cuda(cudaMemsetAsync(barrier, 0, sizeof(unsigned int), st), "fb barrier memset");
    if (rc) return rc;
    void* params[] = {(void*)&a};
    rc = check_cuda(cudaLaunchCooperativeKernel((const void*)fb::fb_lstm_kernel, dim3(a.G), dim3(fb::THREADS), params,
                                                smem, st), "fb_lstm cooperative launch");
    if (rc) return rc;
    FSN_CHECK_LAUNCH("fb_lstm_kernel");
  }
  return FSN_OK;
}

void seq_stack_carve(Carver& c, const SeqStack& s, SeqStackWs& w) {
  int Hm = 0;
  for (int l = 0; l < s.n; ++l) Hm = s.H[l] > Hm ? s.H[l] : Hm;
  const size_t rows = (size_t)s.R * s.Tp;
  w.hall[0] = c.take<float>(rows * Hm);
  w.hall[1] = (s.n > 2 || s.tc) ? c.take<float>(rows * Hm) : nullptr;
  w.h0[0] = w.h0[1] = w.c1 = w.pp = nullptr;
  w.barrier = nullptr;
  if (s.n >= 2) {
    w.h0[0] = c.take<float>((size_t)s.R * s.H[0]);
    w.h0[1] = c.take<float>((size_t)s.R * s.H[0]);
    w.c1 = c.take<float>((size_t)s.R * s.H[1]);
  }
  w.c0 = c.take<float>((size_t)s.R * Hm);  // layer 0's cell, then that of every layer past the first two
  if (s.n >= 2 && !s.gru && !s.step_scale) {
    w.pp = c.take<float>((size_t)2 * fb::ROWS * s.H[0]);
    w.barrier = c.take<unsigned int>(64);
  }
  memset(&w.tc, 0, sizeof(w.tc));
  if (s.tc) {
    const int Hw = Hm > cdiv(s.O, 4) ? Hm : cdiv(s.O, 4);  // the prepared weights of the Linear share the [4 Hmax] rows
    lstm_tc_carve(c, rows, s.K0 > Hm ? s.K0 : Hm, Hw, s.x3, w.tc);
  }
}

SeqPath seq_stack_path(const SeqStack& s) {
  static const bool env_stepwise = getenv("FSN_FB_STEPWISE") != nullptr;  // debug: force the per-step kernels
  const bool stepwise = env_stepwise || s.force_stepwise;
  if (s.tc && !stepwise) return SEQ_PATH_TC;
  if (s.n < 2) return SEQ_PATH_ONE_LAYER;
  if (!stepwise && !s.gru && !s.step_scale && fb_persistent_supported(s.K0, s.H[0], s.H[1])) return SEQ_PATH_PERSISTENT;
  return SEQ_PATH_STEP2;
}

int seq_stack_forward(const SeqStack& s, const SeqStackWs& w, cudaStream_t st) {
  const SeqPath path = seq_stack_path(s);
  const int R = s.R, Tp = s.Tp, n = s.n, Ht = s.H[n - 1];
  auto hall = [&](int l) { return w.hall[(n - 1 - l) & 1]; };  // output of layer l, [R, Tp, H[l]]; the top one in hall[0]
  int rc;
  if (path == SEQ_PATH_TC) {
    // per layer one hoisted input-projection GEMM + the persistent wgmma recurrence; the Linear on the same GEMM
    for (int l = 0; l < n; ++l) {
      const int K = l ? s.H[l - 1] : s.K0;
      const float* x = l ? hall(l - 1) : s.x;
      if ((rc = lstm_layer_tc(s.L[l], x, (size_t)K, K, l ? nullptr : s.scale, Tp, (!l && s.step_scale) ? R : 0, R, Tp,
                              s.H[l], s.x3, w.tc, hall(l), st)))
        return rc;
    }
    return linear_tc(hall(n - 1), (size_t)Ht, Ht, s.fc_w, s.fc_b, s.O, s.act, s.out, (size_t)s.O, (size_t)R * Tp, s.x3, w.tc,
                     st);
  }
  // one per-step kernel launch of layer l at step t: input x (layer 0) or layer l-1's output, h / c state set by the caller
  auto step = [&](int l, int t) {
    StepParams p;
    memset(&p, 0, sizeof(p));
    p.R = R; p.H = s.H[l]; p.first = (t == 0); p.gru = s.gru;
    p.w_ih = s.L[l].w_ih; p.w_hh = s.L[l].w_hh; p.b_ih = s.L[l].b_ih; p.b_hh = s.L[l].b_hh;
    p.K0 = l ? s.H[l - 1] : s.K0;
    p.x0 = (l ? hall(l - 1) : s.x) + (size_t)t * p.K0; p.x0_row_stride = (size_t)Tp * p.K0;
    if (!l) p.row_scale = (s.scale && s.step_scale) ? s.scale + (size_t)t * R : s.scale;
    return p;
  };
  int l = 0;  // first layer left for the single-layer loop
  if (path == SEQ_PATH_PERSISTENT) {
    // weights resident in shared memory, layer wavefront, one grid barrier per time step
    if ((rc = fb_persistent_launch(s.L, s.x, s.scale, w.pp, hall(1), w.barrier, R, s.K0, s.H[0], s.H[1], Tp, st))) return rc;
    l = 2;
  } else if (path == SEQ_PATH_STEP2) {
    const Step2State s2{{w.h0[0], w.h0[1]}, w.c0, {hall(1), nullptr}, w.c1, s.H[1], Tp};
    for (int t = 0; t < Tp; ++t)
      if ((rc = lstm_step2_launch(step(0, t), SEG0_DENSE, t, s.L[1], s2, st))) return rc;
    l = 2;
  }
  for (; l < n; ++l) {
    const size_t ld = (size_t)Tp * s.H[l];
    for (int t = 0; t < Tp; ++t) {
      StepParams p = step(l, t);
      p.h_prev = hall(l) + (size_t)(t > 0 ? t - 1 : 0) * s.H[l]; p.h_prev_stride = ld;
      p.h_out = hall(l) + (size_t)t * s.H[l]; p.h_out_stride = ld;
      p.c = w.c0;
      if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
    }
  }
  return fc_gemm_launch(hall(n - 1), s.fc_w, s.fc_b, s.out, R * Tp, Ht, s.O, s.act, st);
}

// shape checks of the unit-test hook (host only) and its SeqStack; pointers and the tensor-core rule are the hook's
static int dbg_seq_stack(int n, const int* H, int R, int Tp, int K0, int gru, int step_scale, int tc, int x3, int O,
                         SeqStack& s) {
  FSN_REQUIRE(n >= 1 && n <= SEQ_MAX_LAYERS, FSN_ERR_UNSUPPORTED, "seq_stack hook: 1..%d layers (got %d)", SEQ_MAX_LAYERS, n);
  FSN_REQUIRE(H, FSN_ERR_SHAPE, "seq_stack hook: null hidden sizes");
  FSN_REQUIRE(R > 0 && Tp > 0 && K0 > 0 && O > 0, FSN_ERR_SHAPE, "seq_stack hook: bad dims R=%d Tp=%d K0=%d O=%d", R, Tp, K0, O);
  int Hm = K0 > O ? K0 : O;
  for (int l = 0; l < n; ++l) {
    FSN_REQUIRE(H[l] > 0, FSN_ERR_SHAPE, "seq_stack hook: hidden size of layer %d is %d", l, H[l]);
    Hm = H[l] > Hm ? H[l] : Hm;
  }
  FSN_REQUIRE((size_t)R * Tp * 4 * Hm < ((size_t)1 << 31), FSN_ERR_SHAPE, "seq_stack hook: R*Tp*4*max(K0,H,O) must stay below 2^31");
  FSN_REQUIRE(!(tc && gru), FSN_ERR_UNSUPPORTED, "seq_stack hook: the tensor-core stack has no GRU cell");
  memset(&s, 0, sizeof(s));
  s.R = R; s.Tp = Tp; s.K0 = K0; s.n = n; s.O = O;
  for (int l = 0; l < n; ++l) s.H[l] = H[l];
  s.gru = gru != 0; s.step_scale = step_scale != 0; s.tc = tc != 0; s.x3 = x3 != 0;
  return FSN_OK;
}

}  // namespace fsn

using namespace fsn;

extern "C" size_t fsn_debug_seq_stack_workspace_bytes(int n, const int* H, int R, int Tp, int K0, int gru, int step_scale, int tc,
                                                      int x3, int O) {
  SeqStack s;
  if (dbg_seq_stack(n, H, R, Tp, K0, gru, step_scale, tc, x3, O, s)) return 0;
  Carver c(nullptr);
  SeqStackWs w;
  seq_stack_carve(c, s, w);
  return c.off;
}

extern "C" int fsn_debug_seq_stack(const fsn_lstm_layer* layers, int n, const int* H, int R, int Tp, int K0, int gru,
                                   int step_scale, int tc, int x3, int force_stepwise, const float* x, const float* scale,
                                   const float* fc_w, const float* fc_b, int O, int act, float* out, void* workspace,
                                   size_t workspace_bytes, int* path, fsn_stream_t stream) {
  launch_counter() = 0;
  SeqStack s;
  int rc = dbg_seq_stack(n, H, R, Tp, K0, gru, step_scale, tc, x3, O, s);
  if (rc) return rc;
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "seq_stack hook: unknown activation %d", act);
  FSN_REQUIRE(layers && x && fc_w && fc_b && out, FSN_ERR_SHAPE, "seq_stack hook: null argument");
  for (int l = 0; l < n; ++l) {
    FSN_REQUIRE(layers[l].w_ih && layers[l].w_hh && layers[l].b_ih && layers[l].b_hh, FSN_ERR_SHAPE,
                "seq_stack hook: null weight of layer %d", l);
    FSN_REQUIRE(!tc || lstm_rec_tc_supported(H[l], x3 != 0), FSN_ERR_UNSUPPORTED,
                "seq_stack hook: hidden size %d of layer %d is not supported on the tensor cores", H[l], l);
    s.L[l] = layers[l];
  }
  SeqStackWs w;
  Carver c(workspace);
  seq_stack_carve(c, s, w);
  FSN_REQUIRE(workspace && workspace_bytes >= c.off, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes,
              c.off);
  s.act = act; s.force_stepwise = force_stepwise != 0;
  s.x = x; s.scale = scale; s.fc_w = fc_w; s.fc_b = fc_b; s.out = out;
  if (path) *path = seq_stack_path(s);
  return seq_stack_forward(s, w, (cudaStream_t)stream);
}
