// Sub-band LSTM stack on the Hopper tensor cores (wgmma, sm_90a).
//
// Reference semantics: recipes/dns_interspeech_2020/fullsubnet/model.py:98-135 (unfold, concat,
// norm, drop_band, 2xLSTM(H) + Linear(H->2), re-layout, look-ahead slice) with
// audio_zen/model/module/sequence_model.py:106-125 and audio_zen/model/base_model.py:13-46.
// The same stack shape is the fast_fullsubnet bottleneck (fsn_fast_model.cu): there the gather also down-samples
// time (`shrink`) and the Linear layer has one output (the packer zero-pads the second).
//
// Formulation ("weights as the M operand", hidden units split over a CTA pair).  A PAIR of CTAs owns NB = 32 sub-band
// units (rows of the [B*F', .] batch) for all T' steps and both layers; CTA `half` of the pair owns hidden units
// [H/2 half, H/2 (half+1)).  Per step and layer the pair needs
//     gates^T [4H, NB] = W [4H, K] . S^T [K, NB],      S = [x_t | h_{t-1}]  (layer 0)
//                                                      S = [h0_t | h1_{t-1}] (layer 1)
// which runs as wgmma m64n32k16 (fp16 operands, fp32 accumulate), one m64 tile per gate of a 64-unit slice s:
//   * A operand  = 16 KB fp16 weight stages [4 gates x 64 x 32 k], pre-swizzled (64B) by the packer and streamed
//                  from L2 with cp.async.bulk (TMA engine) through a ring; each half has its own stream.  The CTAs
//                  that hold the same half in the CL pairs of a cluster consume the same stream: each loads 1/CL of
//                  a stage and multicasts it to all;
//   * B operand  = the recurrent state S of all H units, fp16, resident in shared memory (K-major, 128B-swizzled;
//                  x_t 64B-swizzled), written in place by the consumers (h: the own half directly, the peer's half
//                  by a DSMEM bulk copy from the peer) and the gather warp (x);
//   * D          = fp32 accumulators in the registers of consumer warpgroup m, which owns slice s = MT half + m, hidden
//                  units [64s, 64s+64): it issues the MMAs of its slice, keeps that slice's cell state c for all NB
//                  rows and both layers in registers, applies the gate non-linearities in fp32, writes h (fp16)
//                  straight back into the B-operand layout and copies that k-block into the peer CTA.  While one
//                  warpgroup runs its cell, the next one's MMAs consume the weight stream.
// Each streamed weight byte thus meets 32 rows, twice the rows one CTA's registers could hold for all H units.
// X3 (FSN_PREC_F16X3_TC) is the ERROR-COMPENSATED variant: weights and state are each split into two fp16 terms
// (hi = rn(v), lo = rn(v - hi)) and every product is issued as W_hi.S_hi + W_hi.S_lo + W_lo.S_hi into the same fp32
// accumulator (the dropped W_lo.S_lo term is 2^-22 relative); the stream carries a hi and a lo stage per k range and
// the gate non-linearities use expf / IEEE division.
// Nothing but the NB x 2 mask values per step (and the pair's h / Linear exchange over DSMEM) ever leaves the SM.
//
// Warp roles (128 + 128 MT threads): 0 = weight-stage producer, 1 = idle, 2 = x_t gather, 3 = Linear(H->2) + output
// staging (half 0) or the half's Linear partial sums sent to half 0 (half 1), 4.. = consumer warpgroups.
//
// PROJ (sb_proj_lstm_tc_kernel, improved_fullsubnet's sections, DESIGN 4.3): the same stack over rows whose layer-0
// input is too wide for a 32-wide x_t.  The caller computes P = X W_ih0^T + b_ih0 + b_hh0 [T, R, 4H] (fp32) for all
// steps first; the ring streams only W_hh0, W_ih1 and W_hh1 (packer mode `proj`), each layer-0 accumulator starts from
// the cell's four gate values of P[t] instead of zero, and layer 1 stores h1_t (fp32) to h1 [T, R, H] instead of
// running a Linear.  Warps 2 and 3 idle.
//
// CARRY (sb_carry_lstm_tc_kernel, chunked streaming, DESIGN 4.14): the same stack continued from a carried state.  Before
// step 0 each row's fp32 (h, c) of both layers is read from a.io_h / a.io_c: h split into hi / lo into the h0 buffer step 0
// reads and into h1 (the split the cell applies to h, so the MMAs see the bits an uninterrupted run would), c into the
// consumers' registers.  A row whose slot restarts at step j (a.restart) enters step j with zero state: its c is dropped
// there and its h of step j - 1 is written to shared memory as zero (j = 0: not loaded).  After step a.store_step the
// fp32 (h, c) go back to io_h / io_c while the kernel runs on; step t's Linear output goes to frame crm_t0 + t of a
// frame-major [clips, frames, 2F] cRM.
//
// PHASED (sb_phased_lstm_tc_kernel, fast_fullsubnet's chunked stream, DESIGN 4.14.2): CARRY over rows whose steps are
// block ends at a phase of their own slot, so step t of row r is its slot's t-th block end in the call.  The gather warp
// reads x_t dense from a.xin, which the caller wrote with the whole-clip gather's expression (so the operand bits are
// those of the whole-clip call), and row r's state goes back to io_h / io_c after step store_at[r / io_rps] instead of
// one store_step for all rows.
#include <cuda_fp16.h>

#include <algorithm>
#include <stdlib.h>
#include <string.h>

#include "fsn_internal.cuh"
#include "fsn_tc_ptx.cuh"
#include "fsn_wgmma.cuh"

namespace fsn {
namespace tc {

using namespace ptx;

constexpr int NB = 32;                 // sub-band units per CTA pair (MMA N)
constexpr int KB = 64;                 // fp16 elements per 128-byte swizzle row
constexpr int KS = 32;                 // k elements per weight stage
constexpr int US = 64;                 // hidden units per slice (MMA M): one consumer warpgroup, one k-block of h
constexpr int W_SUB = US * KS * 2;     // 4096 B: [64 gate rows x 32 k] of one gate, 64B-swizzled
constexpr int W_TILE = 4 * W_SUB;      // 16384 B: one ring stage = the 4 gates (i,f,g,o) of one (slice, k range, part)
constexpr int S_KBLK = NB * KB * 2;    // 4096 B: one k-block of the state operand (= h of one slice)
constexpr int X_BLK = NB * KS * 2;     // 2048 B: x_t, 64B-swizzled
constexpr int MAX_STAGES = 4;          // weight ring depth (FSN_TC_STAGES, default 4)
constexpr int MAX_MT = 3;              // slices per CTA (H / 128)
constexpr int OUT_T = 8;               // output frames staged before a store
constexpr int NTHREADS = 128 + 128 * MAX_MT;

// one stream per half: stage order = consumption order of that half's CTA; half 1's stream follows half 0's
struct PackedLayout {
  int H, MT, nkb0, nkb1, parts;
  size_t tiles0, tiles1;  // stages per step and half, per layer
  size_t off_bias, off_fcw, off_fcb, bytes;
};

// proj: layer 0 streams W_hh0 only (its input projection is precomputed), and the Linear block stays zero
__host__ __device__ inline PackedLayout packed_layout(int H, bool x3, bool proj = false) {
  PackedLayout L;
  L.H = H; L.MT = H / 128;
  L.nkb0 = (proj ? 0 : 1) + H / KS; L.nkb1 = 2 * H / KS;  // k ranges of 32 per slice
  L.parts = x3 ? 2 : 1;
  L.tiles0 = (size_t)L.MT * L.nkb0 * L.parts;
  L.tiles1 = (size_t)L.MT * L.nkb1 * L.parts;
  L.off_bias = 2 * (L.tiles0 + L.tiles1) * W_TILE;
  L.off_fcw = L.off_bias + (size_t)2 * 4 * H * sizeof(float);
  L.off_fcb = L.off_fcw + (size_t)2 * H * sizeof(float);
  L.bytes = L.off_fcb + 256;
  return L;
}

// ---------------------------------------------------------------- weight packer
// stage order = consumption order: half, layer, m (64-unit slice MT half + m), k range of 32, part (hi, lo);
// 4 gate sub-tiles per stage
__global__ void pack_kernel(const float* __restrict__ wih0, const float* __restrict__ whh0,
                            const float* __restrict__ wih1, const float* __restrict__ whh1,
                            const float* __restrict__ bih0, const float* __restrict__ bhh0,
                            const float* __restrict__ bih1, const float* __restrict__ bhh1,
                            const float* __restrict__ fcw, const float* __restrict__ fcb, int H, int Ksb, int x3,
                            int fc_out, int proj, uint8_t* __restrict__ out) {
  const PackedLayout L = packed_layout(H, x3 != 0, proj != 0);
  const size_t per_half = L.tiles0 + L.tiles1;
  const size_t total = 2 * per_half * 4 * US * 4;  // one thread per (stage, gate, row, 16-byte chunk)
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i & 3);
    const int r = (int)((i >> 2) & (US - 1));
    const int g = (int)((i >> 8) & 3);
    const size_t st_abs = i >> 10;
    const int half = (int)(st_abs / per_half);
    size_t st = st_abs - half * per_half;
    const int layer = st >= L.tiles0;
    if (layer) st -= L.tiles0;
    const int part = (int)(st % L.parts);
    st /= L.parts;
    const int nkb = layer ? L.nkb1 : L.nkb0;
    const int kb = (int)(st % nkb);
    const int m = (int)(st / nkb);
    const int wrow = g * H + (half * L.MT + m) * US + r;
    __half v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int kk = c * 8 + e;
      float w = 0.f;
      if (layer == 0 && proj) {
        w = whh0[(size_t)wrow * H + kb * KS + kk];
      } else if (layer == 0) {
        if (kb == 0) { if (kk < Ksb) w = wih0[(size_t)wrow * Ksb + kk]; }
        else w = whh0[(size_t)wrow * H + (kb - 1) * KS + kk];
      } else {
        const int k = kb * KS + kk;
        w = (k < H) ? wih1[(size_t)wrow * H + k] : whh1[(size_t)wrow * H + (k - H)];
      }
      const __half hi = __float2half_rn(w);
      v[e] = part ? __float2half_rn(w - __half2float(hi)) : hi;
    }
    uint8_t* dst = out + st_abs * W_TILE + g * W_SUB + swz64_off(r, c * 8);
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(v);
  }
  // biases (b_ih + b_hh, fp32) and the Linear layer (outputs beyond fc_out are zero); proj: layer 0's biases are in P
  // and there is no Linear, so both stay zero
  float* bias = reinterpret_cast<float*>(out + L.off_bias);
  float* pfcw = reinterpret_cast<float*>(out + L.off_fcw);
  float* pfcb = reinterpret_cast<float*>(out + L.off_fcb);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 4 * H; i += gridDim.x * blockDim.x) {
    bias[i] = proj ? 0.f : bih0[i] + bhh0[i];
    bias[4 * H + i] = bih1[i] + bhh1[i];
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * H; i += gridDim.x * blockDim.x)
    pfcw[i] = (!proj && i < fc_out * H) ? fcw[i] : 0.f;
  if (blockIdx.x == 0 && threadIdx.x < 2)
    pfcb[threadIdx.x] = (!proj && (int)threadIdx.x < fc_out) ? fcb[threadIdx.x] : 0.f;
}

// ---------------------------------------------------------------- shared-memory plan
struct Smem {
  uint32_t w, x, h0, h1, lo, fcw, fcp, outst, rows, bars, total;
};
__host__ __device__ inline Smem smem_plan(int H, int stages, bool x3) {
  Smem s;
  const int nkh = H / KB;
  uint32_t o = 0;
  s.w = o; o += stages * W_TILE;
  s.x = o; o += 2 * X_BLK;
  s.h0 = o; o += 2 * nkh * S_KBLK;
  s.h1 = o; o += nkh * S_KBLK;  // single buffer: h1_t overwrites h1_{t-1} once every layer-1 MMA of step t is done
  s.lo = o; o += x3 ? (o - s.x) : 0;  // X3: lo copies of x, h0, h1 at offset (lo - x) from the hi copies
  s.fcw = o; o += 4 * MAX_MT * 2 * NB * 4;  // Linear partial sums [consumer warp][o][row]
  s.fcp = o; o += 2 * 2 * NB * 4;           // half 0: half 1's Linear sums [buffer][o][row]
  s.outst = o; o += NB * 2 * OUT_T * 4;
  s.rows = o; o += NB * 16;
  s.bars = o; o += 256;
  s.total = o;
  return s;
}

struct Bars {
  uint64_t w_full[MAX_STAGES], w_empty[MAX_STAGES];
  uint64_t x_full[2], x_empty[2];
  // h0_ready[b]: h0_t (t & 1 = b) complete in buffer b, this half written here and the peer's half landed (complete_tx)
  // h0_empty[b]: the peer's consumers have read h0 buffer b (their layer-1 MMAs of step t) - this CTA may copy into it
  uint64_t h0_ready[2], h0_empty[2];
  uint64_t h1_ready, h1_empty, fc_done;
  uint64_t l1_done;   // all layer-1 MMAs of a step have completed (h1 may be overwritten)
  uint64_t fcp_full[2], fcp_empty[2];  // half 1 -> half 0 Linear sums
  // turn[m]: warpgroup m may wait on the weight ring - its predecessor in the stream has seen all of its own
  // stages land.  The ring's parity waits are only sound one phase ahead, so the warpgroups take the ring in turn
  uint64_t turn[MAX_MT];
};
static_assert(sizeof(Bars) <= 256, "barrier block too large");

struct RowInfo {
  int src_b, src_f;   // source clip / frequency (drop_band map), src_b < 0: row beyond the batch
  // 1 / (mu' + 1e-5) of the source clip.  Block-phased CARRY: the bits of the step after which the row's state is
  // stored (the carry policies read no scale here; making this a union with an int changes the code of the production
  // instantiations)
  float scale;
  union {
    int out_idx;      // crm index of (b', o=0, f', t=0) divided by T  (= (b'*2)*Fsub + f')
    int restart;      // CARRY: the step at which the row enters with zero state (none when outside [0, Tp))
  };
};

// The kernel takes KArgs as a __grid_constant__ parameter: its fields stay in parameter (constant-bank) space and are
// read where they are used.  Passed as a plain by-value struct of at most 128 bytes, the front end instead loads every
// field into a register at kernel entry and keeps it live through the whole kernel; in the x3 kernel, whose consumers
// already need nearly all of their 152 registers, that costs 248 / 434 bytes of spill stores / loads (184-byte stack
// frame) against 64 / 84 (48-byte frame), and 8 / 12 against 0 in the single pass - about 17 % of the headline step
// (DESIGN 4.1).  tests/test_cpu_subband_resources.py checks the frames of the built library.
struct KArgs {
  const uint8_t* packed;
  const float* magT; const float* fbT; const float* inv2;
  const float* unit_scale;  // nullable: cumulative norm, scale of (step t, row r) at [t*R + r] instead of inv2[clip]
  float* crm;
  int R, F, Tp, la, T, Ns, Nf, H, Ksb, act, Fsub, stages, cluster;
  int src_T, shrink;  // frames in magT/fbT; x_t = mean of `shrink` source frames (fast_fullsubnet down-sampling), 1 = none
  RowMap map;
  long long* stamps;  // PROBE instantiation only: records of CTAs [0, stamp_ctas), iterations [0, stamp_its)
  int stamp_ctas, stamp_its;
  // PROJ instantiation only: layer 0's input projection P [Tp, R, 4H] and the layer-1 output h1 [Tp, R, H] (fp32)
  const float* proj; float* h1;
  // CARRY instantiation only: (h, c) of row r, layer l, unit u at io_h / io_c [(r / io_rps) io_slot + l io_layer +
  // (r % io_rps) H + u] (floats), restart step of row r at restart[r / io_rps], state stored after step store_step;
  // output o of row r = b F + f at step t to crm[b crm_bs + (crm_t0 + t) 2F + o F + f]
  float* io_h; float* io_c;
  size_t io_slot, io_layer, crm_bs;
  const int* restart;
  int io_rps, store_step, crm_t0;
  // block-phased CARRY instantiation only: the input x_t of row r at xin [(t R + r) Ksb + k], gathered, down-sampled and
  // scaled by the caller; the state of row r stored after step store_at[r / io_rps] (none when outside [0, Tp))
  const float* xin;
  const int* store_at;
};

// ---------------------------------------------------------------- cycle stamps (PROBE instantiation)
// One record of PROBE_FIELDS int64 per (CTA, loop iteration it, layer, slot): slots 0 .. MAX_MT-1 are the consumer
// warpgroups (block = that warpgroup's MMAs and cell of one layer; layer 1 of iteration it is step it - 1), slot MAX_MT
// is the weight producer (layer-0 record of each iteration, the stages it streams in that iteration).  Durations are
// SM cycles (clock64) summed over the block, as seen by thread 0 of the warpgroup / warp.
enum ProbeField {
  PF_T_BEGIN = 0,   // clock64 at block start, before the operand waits
  PF_T_MMA0 = 1,    // first stage may be waited on (operand and turn waits done)
  PF_T_MMA1 = 2,    // every MMA of the block retired (wait_group 0)
  PF_T_END = 3,     // h written and the copy to the peer issued
  PF_OPERAND = 4,   // waits on x_full / h0_ready / h1_ready (producer: w_empty waits)
  PF_TURN = 5,      // wait on turn[m]
  PF_W_FULL = 6,    // waits on w_full (stages landing)
  PF_WAIT_GROUP = 7,// wgmma.wait_group
  PF_GROUP_LAT = 8, // sum over the stage groups of commit -> return of the wait_group that retires the group
                    // (after the NEXT stage's w_full wait and MMA issue: an upper bound on the retire latency)
  PF_STAGES = 9,    // ring stages of the block
  PF_CELL = 10,     // cell math, h stores, exchange issue (waits excluded)
  PF_L1_DONE = 11,  // wait on l1_done
  PF_H1_EMPTY = 12, // wait on h1_empty
  PF_H0_EMPTY = 13, // wait on h0_empty
  PF_FC_DONE = 14,  // wait on fc_done
  PF_GT_BEGIN = 15, // globaltimer (ns) at block start
  PROBE_FIELDS = 16
};
constexpr int PROBE_SLOTS = MAX_MT + 1;
static_assert(PROBE_FIELDS == FSN_SB_PROBE_FIELDS && PROBE_SLOTS == FSN_SB_PROBE_SLOTS,
              "probe record layout differs from fsn_b200.h (and fullsubnet_b200/_lib.py)");

__device__ __forceinline__ long long globaltimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return (long long)t;
}

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case FSN_ACT_RELU: return fmaxf(v, 0.f);
    case FSN_ACT_TANH: return tanhf(v);
    case FSN_ACT_RELU6: return fminf(fmaxf(v, 0.f), 6.f);
    default: return v;
  }
}
// MUFU-class forms for the single-pass variant, whose fp16 products are 1e-3 class anyway; expf + IEEE division
// for the compensated one, whose whole point is the fp32 error class
template <bool X3> __device__ __forceinline__ float sg(float x) { return X3 ? 1.0f / (1.0f + expf(-x)) : fast_sigmoid(x); }
template <bool X3> __device__ __forceinline__ float th(float x) { return X3 ? 1.0f - 2.0f / (1.0f + expf(2.0f * x)) : fast_tanh(x); }
// LSTM cell of one (unit, row) from its gate pre-activations (MMA sums, gate order i, f, g, o) and biases b[4]: returns
// the new c and sets h
template <bool X3>
__device__ __forceinline__ float lstm_cell(float ai, float af, float ag, float ao, const float (&b)[4], float cp,
                                           float& h) {
  const float cn = sg<X3>(af + b[1]) * cp + sg<X3>(ai + b[0]) * th<X3>(ag + b[2]);
  h = sg<X3>(ao + b[3]) * th<X3>(cn);
  return cn;
}

// Consumer warpgroup releases weight stage `bar` to the producers of the CL CTAs that share the stream (the CTAs of
// the same half, ranks 2 q + half): one arrive per warpgroup and destination CTA (w_empty counts CL), warp q
// signalling pair q so that the remote arrives go out in parallel (`local`: CL = 1 and q = 0; `remote`: CL > 1 and
// q < CL; both warp-uniform, so the arrives are predicated instructions of one elected lane and the stage loop has no
// divergent region).  `pred`: there is a stage to release.  No fence is needed: the stage is read only by
// this warpgroup's wgmma (async proxy), the wgmma.wait_group before this call has retired those reads, and the
// producers overwrite the stage with TMA (async proxy) only after the w_empty phase completes - the barrier phase
// alone orders the overwrite after the reads, so the arrive keeps its default .release.cta semantics (the hand-off of
// CUTLASS's TMA pipelines for the same hazard).  Every warp of the warpgroup has passed the w_full wait of the stage:
// the MMAs that read it are warpgroup-collective.
__device__ __forceinline__ void release_stage(uint32_t bar, uint32_t pred, uint32_t local, uint32_t remote,
                                              uint32_t rank) {
  mbar_arrive_elect_if(bar, pred & local);
  mbar_arrive_remote_elect_if(bar, rank, pred & remote);
}

// PROJ: gate g of layer 0 for accumulator register i of consumer thread (warp q, lane) of slice s at step t, P[t][row0 +
// n][g H + u] with unit u = 64 s + 16 q + lane/4 + 8 hh and row n = 8 j + 2 (lane % 4) + e for i = 4 j + 2 hh + e (rows
// past R read row R - 1; their results are never stored).  x3 starts the accumulators from it, which hides the load
// behind the ring waits; the single pass adds it after the MMAs, because there the loaded accumulators make ptxas
// serialise the MMAs (C7515), and with x3 the later add costs 120 bytes of spills instead of none (DESIGN 4.3)
__device__ __forceinline__ float proj_at(const KArgs& a, int t, int row0, int s, int q, int lane, int g, int i) {
  const int j = i >> 2, hh = (i >> 1) & 1, e = i & 1;
  const int u = s * US + 16 * q + (lane >> 2) + 8 * hh;
  const int r = min(row0 + 8 * j + 2 * (lane & 3) + e, a.R - 1);
  return __ldg(a.proj + ((size_t)t * a.R + r) * 4 * a.H + g * a.H + u);
}

// CARRY: offset of row r's unit u in the layer-0 block of io_h / io_c
__device__ __forceinline__ size_t carry_idx(const KArgs& a, int r, int u) {
  const int sl = r / a.io_rps;
  return (size_t)sl * a.io_slot + (size_t)(r - sl * a.io_rps) * a.H + u;
}

// PROBE: the same kernel with cycle stamps (ProbeField) written to a.stamps; the production launches use PROBE = false,
// where every stamp below compiles away.  PROJ: the precomputed layer-0 projection and stored h1 (see the top of the
// file); every PROJ and CARRY branch below is `if constexpr` or folds away, so the sb_lstm_tc_kernel instantiations are
// the code they were before the policies existed.  PHASED (only with CARRY): dense input and per-slot store steps
template <bool X3, bool PROBE, bool PROJ, bool CARRY, bool PHASED = false>
__device__ __forceinline__ void sb_lstm_tc_body(const KArgs& a) {
  static_assert(!PHASED || CARRY, "the block-phased policy is a carry policy");
  constexpr int PARTS = X3 ? 2 : 1;
  // probe clock: cycles since the previous mark (0 and no code without PROBE)
  long long pt = 0;
  auto mark = [&]() -> uint32_t {
    if constexpr (PROBE) {
      const long long n = clock64();
      const uint32_t d = (uint32_t)(n - pt);
      pt = n;
      return d;
    } else {
      return 0u;
    }
  };
  auto record = [&](int it, int layer, int slot) -> long long* {
    return a.stamps + ((((size_t)blockIdx.x * a.stamp_its + it) * 2 + layer) * PROBE_SLOTS + slot) * PROBE_FIELDS;
  };
  const bool probe_cta = PROBE && (int)blockIdx.x < a.stamp_ctas;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzle atoms need 1024-byte alignment in the shared window
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int H = a.H;
  const int MT = H / 128;
  const int nkh = H / KB;
  const int STAGES = a.stages;
  const int CL = a.cluster;
  // the cluster is CL pairs: rank 2 i + half, pair i; the CTAs of one half multicast that half's stream
  const uint32_t cl_rank = cluster_ctarank();
  const int half = (int)(cl_rank & 1u);
  const uint32_t peer = cl_rank ^ 1u;
  const uint16_t cl_mask = (uint16_t)((0x55u & ((1u << (2 * CL)) - 1u)) << half);
  const Smem sp = smem_plan(H, STAGES, X3);
  const uint32_t LO = sp.lo - sp.x;  // byte offset of a lo copy from its hi copy
  const PackedLayout PL = packed_layout(H, X3, PROJ);
  Bars& bars = *reinterpret_cast<Bars*>(smem + sp.bars);
  RowInfo* rows = reinterpret_cast<RowInfo*>(smem + sp.rows);
  float* fc_part = reinterpret_cast<float*>(smem + sp.fcw);
  float* fcp = reinterpret_cast<float*>(smem + sp.fcp);
  float* outst = reinterpret_cast<float*>(smem + sp.outst);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = (blockIdx.x >> 1) * NB;
  const int Tp = a.Tp;

  // ---------------- one-time setup
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&bars.w_full[s], 1); mbar_init(&bars.w_empty[s], CL); }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bars.x_full[i], 1); mbar_init(&bars.x_empty[i], 4 * MT);
      mbar_init(&bars.h0_ready[i], 5 * MT);  // 4 MT local warps + MT peer copies
      mbar_init(&bars.h0_empty[i], MT);
      mbar_init(&bars.fcp_full[i], 1); mbar_init(&bars.fcp_empty[i], 1);
    }
    mbar_init(&bars.h1_ready, 5 * MT);
    mbar_init(&bars.h1_empty, MT);
    mbar_init(&bars.fc_done, 1);
    mbar_init(&bars.l1_done, 4 * MT);
    for (int m = 0; m < MAX_MT; ++m) mbar_init(&bars.turn[m], 4);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (!PROJ && threadIdx.x < NB) {
    RowInfo ri;
    const int r = row0 + threadIdx.x;
    ri.src_b = -1; ri.src_f = 0; ri.scale = 0.f; ri.out_idx = 0;
    if (r < a.R) {
      row_to_unit(a.map, r, ri.src_b, ri.src_f);
      if constexpr (CARRY) {
        ri.restart = a.restart[r / a.io_rps];
        if constexpr (PHASED) ri.scale = __int_as_float(a.store_at[r / a.io_rps]);
      } else {
        ri.scale = a.inv2[ri.src_b];
        const int bq = r / a.Fsub, fq = r - bq * a.Fsub;
        ri.out_idx = bq * 2 * a.Fsub + fq;
      }
    }
    rows[threadIdx.x] = ri;
  }
  {  // zero the state (h_{-1} = 0, x padding)
    uint4* z = reinterpret_cast<uint4*>(smem + sp.x);
    const int n16 = (sp.fcw - sp.x) / 16;
    for (int i = threadIdx.x; i < n16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
  }
  if constexpr (CARRY) {
    // h_{-1} of both layers for all H units of the pair's rows: layer 0 into the h0 buffer step 0 reads (buffer 1),
    // layer 1 into h1, in the B-operand layout the consumers write (unit U = 64 s + u of row n)
    __syncthreads();
    const int nkh0 = H / KB;
    for (int i = threadIdx.x; i < 2 * NB * H; i += blockDim.x) {
      const int l = i / (NB * H), n = (i / H) % NB, U = i % H;
      const int r = row0 + n;
      if (r >= a.R || a.restart[r / a.io_rps] == 0) continue;
      const float v = a.io_h[carry_idx(a, r, U) + l * a.io_layer];
      uint8_t* p = smem + (l ? sp.h1 : sp.h0 + nkh0 * S_KBLK) + (U >> 6) * S_KBLK + (n >> 3) * 1024 + (n & 7) * 128 +
                   ((((U & 63) >> 3) ^ (n & 7)) << 4) + (U & 7) * 2;
      const __half hi = __float2half_rn(v);
      *reinterpret_cast<__half*>(p) = hi;
      if (X3) *reinterpret_cast<__half*>(p + (sp.lo - sp.x)) = __float2half_rn(v - __half2float(hi));
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();  // peers' barriers are initialised before any multicast, copy or remote arrive reaches them

  if (warp < 4) {
    // warpgroup 0 (producer / gather / Linear) needs few registers: hand the rest to the consumers
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
  if (warp == 0) {
    // ================= weight-stage producer: this half's (layer 0, layer 1) stream, the same every step
    const uint8_t* stream = a.packed + (size_t)half * (PL.tiles0 + PL.tiles1) * W_TILE;
    uint32_t stage = 0, phase = 0;
    for (int it = 0; it <= Tp; ++it) {
      const size_t t_begin = (it < Tp) ? 0 : PL.tiles0;
      const size_t t_end = (it >= 1) ? PL.tiles0 + PL.tiles1 : PL.tiles0;
      const uint8_t* src = stream + t_begin * W_TILE;
      long long p_t0 = 0, p_g0 = 0;
      uint32_t p_empty = 0;
      if constexpr (PROBE) { p_g0 = globaltimer(); p_t0 = clock64(); pt = p_t0; }
      for (size_t tile = t_begin; tile < t_end; ++tile, src += W_TILE) {
        // all CL CTAs' consumers have drained this stage (on the critical path: no back-off)
        mark();
        mbar_wait_cta<false>(&bars.w_empty[stage], phase ^ 1);
        p_empty += mark();
        if (elect_one()) {
          mbar_expect_tx(&bars.w_full[stage], W_TILE);
          if (CL == 1) {
            bulk_g2s(smem + sp.w + stage * W_TILE, src, W_TILE, &bars.w_full[stage]);
          } else {
            const uint32_t slice = W_TILE / CL, off = (cl_rank >> 1) * slice;
            bulk_g2s_mc(smem + sp.w + stage * W_TILE + off, src + off, slice, &bars.w_full[stage], cl_mask);
          }
        }
        __syncwarp();
        if (++stage == (uint32_t)STAGES) { stage = 0; phase ^= 1; }
      }
      if (probe_cta && it < a.stamp_its && lane == 0) {
        long long* r = record(it, 0, MAX_MT);
        r[PF_T_BEGIN] = p_t0; r[PF_T_END] = clock64(); r[PF_OPERAND] = p_empty;
        r[PF_STAGES] = (long long)(t_end - t_begin); r[PF_GT_BEGIN] = p_g0;
      }
    }
  } else if (!PROJ && warp == 2) {
    // ================= x_t gather: sub-band unit = 2Ns+1 reflected magnitude rows + 2Nf+1 full-band rows,
    // scaled by 1/(mu'+1e-5)  (base_model.py:35-44, model.py:98-111), fp16 (X3: + lo), B-operand layout.
    // Both CTAs of a pair gather all NB rows (a duplicated L2 read is cheaper than an exchange)
    const int nmag = 2 * a.Ns + 1;
    for (int t = 0; t < Tp; ++t) {
      mbar_wait_cta<true>(&bars.x_empty[t & 1], ((t >> 1) & 1) ^ 1);
      uint8_t* xb = smem + sp.x + (t & 1) * X_BLK;
      // source frames of step t: itself, or (fast_fullsubnet/model.py:108-129) frame 0 alone, then blocks of
      // `shrink` frames, the last one over its own length
      int f0 = t, f1 = t + 1;
      if (a.shrink > 1 && t > 0) { f0 = 1 + (t - 1) * a.shrink; f1 = min(f0 + a.shrink, a.src_T); }
      const float wmean = 1.0f / (float)(f1 - f0);
#pragma unroll 4
      for (int n = 0; n < NB; ++n) {
        const RowInfo ri = rows[n];
        float v = 0.f;
        if constexpr (PHASED) {
          if (ri.src_b >= 0 && lane < a.Ksb) v = a.xin[((size_t)t * a.R + row0 + n) * a.Ksb + lane];
        } else if (ri.src_b >= 0 && lane < a.Ksb) {
          const int col = (lane < nmag) ? reflect_idx(ri.src_f + lane - a.Ns, a.F)
                                        : reflect_idx(ri.src_f + (lane - nmag) - a.Nf, a.F);
          const float* src = (lane < nmag) ? a.magT : a.fbT;
          if (a.shrink <= 1) {
            v = src[((size_t)ri.src_b * a.src_T + t) * a.F + col];
            v *= a.unit_scale ? a.unit_scale[(size_t)t * a.R + row0 + n] : ri.scale;
          } else {
            for (int fr = f0; fr < f1; ++fr) v += src[((size_t)ri.src_b * a.src_T + fr) * a.F + col];
            v *= wmean * (a.unit_scale ? a.unit_scale[(size_t)t * a.R + row0 + n] : ri.scale);
          }
        }
        const __half hi = __float2half_rn(v);
        *reinterpret_cast<__half*>(xb + swz64_off(n, lane)) = hi;
        if (X3) *reinterpret_cast<__half*>(xb + LO + swz64_off(n, lane)) = __float2half_rn(v - __half2float(hi));
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars.x_full[t & 1]);
    }
  } else if (!PROJ && warp == 3) {
    // ================= Linear(H -> 2), one row per lane: sums the fp32 partial dot products of the consumer warps.
    // Half 1 sends its sums to half 0; half 0 adds the bias, its own sums and half 1's (one fixed association
    // order), stages OUT_T frames and stores crm[b', o, f', t - la]  (model.py:129-135 fused)
    const float fcb0 = half ? 0.f : reinterpret_cast<const float*>(a.packed + PL.off_fcb)[0];
    const float fcb1 = half ? 0.f : reinterpret_cast<const float*>(a.packed + PL.off_fcb)[1];
    const RowInfo ri = rows[lane];
    int staged = 0, t_stage0 = 0;
    for (int t = 0; t < Tp; ++t) {
      mbar_wait_cta<true>(&bars.h1_ready, t & 1);
      float s0 = fcb0, s1 = fcb1;
      if (t >= a.la) {
        for (int w = 0; w < 4 * MT; ++w) {
          s0 += fc_part[(w * 2 + 0) * NB + lane];
          s1 += fc_part[(w * 2 + 1) * NB + lane];
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars.fc_done);
      if (t < a.la) continue;
      const int u = t - a.la, b = u & 1;
      float* pb = fcp + b * 2 * NB;
      if (half) {
        // half 0 has read this buffer's previous sums (generic stores to another CTA: cluster-scope release/acquire)
        mbar_wait<true>(&bars.fcp_empty[b], ((u >> 1) & 1) ^ 1);
        st_remote_f32(pb + lane, peer, s0);
        st_remote_f32(pb + NB + lane, peer, s1);
        __syncwarp();
        if (lane == 0) mbar_arrive_cluster(&bars.fcp_full[b], peer);
        continue;
      }
      mbar_wait<true>(&bars.fcp_full[b], (u >> 1) & 1);
      s0 += pb[lane];
      s1 += pb[NB + lane];
      __syncwarp();
      if (lane == 0) mbar_arrive_cluster(&bars.fcp_empty[b], peer);
      if (staged == 0) t_stage0 = u;
      outst[(lane * 2 + 0) * OUT_T + staged] = act_apply(s0, a.act);
      outst[(lane * 2 + 1) * OUT_T + staged] = act_apply(s1, a.act);
      ++staged;
      if (staged == OUT_T || t == Tp - 1) {
        if (ri.src_b >= 0) {
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            if constexpr (CARRY) {
              const size_t F2 = 2 * (size_t)a.F;
              float* dst = a.crm + (size_t)ri.src_b * a.crm_bs + ((size_t)a.crm_t0 + t_stage0) * F2 + (size_t)o * a.F + ri.src_f;
              for (int i = 0; i < staged; ++i) dst[i * F2] = outst[(lane * 2 + o) * OUT_T + i];
            } else {
              float* dst = a.crm + ((size_t)ri.out_idx + (size_t)o * a.Fsub) * a.T + t_stage0;
              for (int i = 0; i < staged; ++i) dst[i] = outst[(lane * 2 + o) * OUT_T + i];
            }
          }
        }
        staged = 0;
      }
    }
  }
  } else {
    // ================= consumer warpgroup m: MMAs and cells of slice s = MT half + m, hidden units [64s, 64s+64), of
    // both layers.  Fragment of thread (warp q, lane l): unit 64 s + 16 q + l/4 + 8 hh, row n = 8 j + 2 (l%4) + e,
    // register acc[g][4 j + 2 hh + e]
    asm volatile("setmaxnreg.inc.sync.aligned.u32 152;");
    // warpgroup and warp index broadcast from lane 0, so that the compiler knows them warp-uniform: the barrier
    // addresses and MMA descriptor words of the stage loop can then live in uniform registers
    const int m = __shfl_sync(0xffffffffu, (warp - 4) >> 2, 0);
    const int q = __shfl_sync(0xffffffffu, warp & 3, 0);
    const int s = half * MT + m;
    if (m < MT) {
      const float* bias_g = reinterpret_cast<const float*>(a.packed + PL.off_bias);
      const float* fcw = reinterpret_cast<const float*>(a.packed + PL.off_fcw);
      float* my_part = fc_part + (size_t)(warp - 4) * 2 * NB;
      float c0[16], c1[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) c0[i] = c1[i] = 0.f;
      if constexpr (CARRY) {
        // c_{-1} of this thread's fragment (a row restarting at step 0 drops it in its first cell)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int hh = i >> 3, j = (i >> 1) & 3, e = i & 1;
          const int r = row0 + 8 * j + 2 * (lane & 3) + e;
          if (r < a.R) {
            const float* p = a.io_c + carry_idx(a, r, s * US + 16 * q + (lane >> 2) + 8 * hh);
            c0[i] = p[0];
            c1[i] = p[a.io_layer];
          }
        }
      }
      // per-kernel constants of the stage loop: the A descriptor of ring slot 0 (a slot is W_TILE >> 4 further), the
      // barriers, and which warps release a stage where (see release_stage)
      const uint32_t a_lo0 = wg::desc_lo(smem_u32(smem + sp.w));
      const uint32_t w_full0 = smem_u32(&bars.w_full[0]), w_empty0 = smem_u32(&bars.w_empty[0]);
      const uint32_t turn_next = smem_u32(&bars.turn[m + 1 < MT ? m + 1 : 0]);
      const uint32_t rel_local = CL == 1 && q == 0, rel_remote = CL > 1 && q < CL;
      const uint32_t rel_rank = 2 * q + half;
      int h0_seen = 0, h1_seen = 0, turns = 0;
      bool first_block = true;
      size_t tile_base = 0;  // index (in this half's stream) of this iteration's first stage
      for (int it = 0; it <= Tp; ++it) {
        for (int layer = 0; layer < 2; ++layer) {
          const int t = it - layer;
          if (t < 0 || t >= Tp) continue;
          // probe: block start, then the waits and phases of the block (ProbeField)
          long long p_t0 = 0, p_g0 = 0, p_mma0 = 0, p_mma1 = 0, p_commit = 0, p_commit_prev = 0;
          uint32_t p_opnd = 0, p_turn = 0, p_wfull = 0, p_wgw = 0, p_lat = 0, p_cell = 0, p_l1 = 0, p_h1e = 0, p_h0e = 0,
                   p_fc = 0;
          if constexpr (PROBE) { p_g0 = globaltimer(); p_t0 = clock64(); pt = p_t0; }
          // operands of this step complete in shared memory (every phase waited on once, in order).  All of this
          // kernel's waits on the weight ring and the state are CTA-scope: each of those barriers guards data written
          // by this CTA or by an async-proxy copy with complete_tx (TMA from L2, the peer's DSMEM bulk copy)
          if (layer == 0) {
            if constexpr (!PROJ) mbar_wait_cta<false>(&bars.x_full[t & 1], (t >> 1) & 1);
            for (; h0_seen < t; ++h0_seen) mbar_wait_cta<false>(&bars.h0_ready[h0_seen & 1], (h0_seen >> 1) & 1);      // h0_{t-1}
          } else {
            for (; h0_seen < t + 1; ++h0_seen) mbar_wait_cta<false>(&bars.h0_ready[h0_seen & 1], (h0_seen >> 1) & 1);  // h0_t
            for (; h1_seen < t; ++h1_seen) mbar_wait_cta<false>(&bars.h1_ready, h1_seen & 1);                          // h1_{t-1}
          }
          p_opnd += mark();
          const uint32_t x_addr = smem_u32(smem + sp.x + (t & 1) * X_BLK);
          const uint32_t h0_cur = smem_u32(smem + sp.h0 + (t & 1) * nkh * S_KBLK);        // h0_t
          const uint32_t h0_prev = smem_u32(smem + sp.h0 + ((t + 1) & 1) * nkh * S_KBLK);  // h0_{t-1}
          const uint32_t h1_prev = smem_u32(smem + sp.h1);                                    // h1_{t-1}
          const int nkb = layer ? PL.nkb1 : PL.nkb0;
          const size_t first = tile_base + (layer ? ((it < Tp) ? PL.tiles0 : 0) : 0) + (size_t)m * nkb * PARTS;
          float acc[4][16];
#pragma unroll
          for (int g = 0; g < 4; ++g) {
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[g][i] = 0.f;
            if constexpr (PROJ && X3) {
              if (layer == 0) {
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[g][i] = proj_at(a, t, row0, s, q, lane, g, i);
              }
            }
            wg::fence_operand(acc[g]);
          }
          if constexpr (PROJ && !X3) {
            // single pass: layer 0 adds P[t] after its MMAs (see proj_at); pull this warp's P lines into L2 now, 32
            // rows x 4 gates of 16 units (64 B) each
            if (layer == 0) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int idx = lane + 32 * i;
                const int r = min(row0 + (idx & 31), a.R - 1);
                const float* p = a.proj + ((size_t)t * a.R + r) * 4 * H + (idx >> 5) * H + s * US + 16 * q;
                asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
              }
            }
          }
          int prev_stage = -1;
          if (m > 0 || !first_block) { mbar_wait_cta<false>(&bars.turn[m], turns & 1); ++turns; }
          first_block = false;
          p_turn += mark();
          p_mma0 = pt;
          // ring slot and fill parity of stream stage `first`, then advanced stage by stage
          // (broadcast from lane 0 like m and q: warp-uniform by construction)
          int stage = __shfl_sync(0xffffffffu, (int)(first % (size_t)STAGES), 0);
          uint32_t wphase = __shfl_sync(0xffffffffu, (uint32_t)((first / (size_t)STAGES) & 1), 0);
          // one ring stage against the state k range of descriptor `bd` (lo copy LO bytes further): wait for it to
          // land, issue its MMAs (x3 hi part: hi.hi and hi.lo per gate and k16; lo part and single pass: one per gate
          // and k16), commit, retire the previous stage's group and release that stage.  `ends_block`: the block's
          // last stage, after whose landing the next warpgroup in the stream may take the ring
          auto issue_stage = [&](int part, uint32_t bd, uint32_t b_hi, uint32_t ends_block) {
            mark();
            mbar_wait_cta_warp(w_full0 + 8 * stage, wphase);
            p_wfull += mark();
            mbar_arrive_elect_if(turn_next, ends_block);
            wg::fence();
            const uint32_t ad = a_lo0 + stage * (W_TILE >> 4);
#pragma unroll
            for (int kk = 0; kk < 2; ++kk)
#pragma unroll
              for (int g = 0; g < 4; ++g) {
                const uint32_t a_off = g * (W_SUB >> 4) + kk * 2;
                wg::mma_f16_n32_w(acc[g], ad, a_off, wg::DESC_SW64_HI, bd, kk * 2, b_hi);
                if (X3 && part == 0) wg::mma_f16_n32_w(acc[g], ad, a_off, wg::DESC_SW64_HI, bd, (LO >> 4) + kk * 2, b_hi);
              }
            wg::commit();
            if constexpr (PROBE) p_commit = clock64();
            mark();
            wg::wait<1>();  // the MMAs of the previous stage have read it
            p_wgw += mark();
            if constexpr (PROBE) {
              if (prev_stage >= 0) p_lat += (uint32_t)(pt - p_commit_prev);
              p_commit_prev = p_commit;
            }
            release_stage(w_empty0 + 8 * prev_stage, prev_stage >= 0, rel_local, rel_remote, rel_rank);
            prev_stage = stage;
            if (++stage == STAGES) { stage = 0; wphase ^= 1; }
          };
          // B operand k ranges: layer 0: [x_t (32 k, one 64B-swizzled block)] [h0_{t-1} (H)]; layer 1: [h0_t (H)]
          // [h1_{t-1} (H)].  A k-block of h (64 k, 128B-swizzled) is two k ranges, 64 B apart in the swizzle row
          if (!PROJ && layer == 0) {
#pragma unroll
            for (int part = 0; part < PARTS; ++part) issue_stage(part, wg::desc_lo(x_addr), wg::DESC_SW64_HI, 0u);
          }
          // (do-while: H >= 128, so every segment has k-blocks and the loops need no entry test)
          const int nseg = layer ? 2 : 1;
          int seg = 0;
          do {
            uint32_t bd = wg::desc_lo(layer == 0 ? h0_prev : seg == 0 ? h0_cur : h1_prev);
            int kb = 0;
            do {
              const uint32_t ends_block = seg == nseg - 1 && kb == nkh - 1;
#pragma unroll
              for (int part = 0; part < PARTS; ++part) issue_stage(part, bd, wg::DESC_SW128_HI, 0u);
#pragma unroll
              for (int part = 0; part < PARTS; ++part)
                issue_stage(part, bd + (64 >> 4), wg::DESC_SW128_HI, part == PARTS - 1 ? ends_block : 0u);
              bd += S_KBLK >> 4;
            } while (++kb < nkh);
          } while (++seg < nseg);
          mark();
          wg::wait<0>();
#pragma unroll
          for (int g = 0; g < 4; ++g) wg::fence_operand(acc[g]);
          if constexpr (PROJ && !X3) {
            if (layer == 0) {
#pragma unroll
              for (int g = 0; g < 4; ++g)
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[g][i] += proj_at(a, t, row0, s, q, lane, g, i);
            }
          }
          p_wgw += mark();
          if constexpr (PROBE) { p_lat += (uint32_t)(pt - p_commit_prev); p_mma1 = pt; }
          release_stage(w_empty0 + 8 * prev_stage, 1u, rel_local, rel_remote, rel_rank);
          // this warpgroup's MMAs of the step have consumed x_t / h1_{t-1}
          if (lane == 0 && (!PROJ || layer)) mbar_arrive(layer ? &bars.l1_done : &bars.x_empty[t & 1]);
          if (layer == 1 && lane == 0) {
            // ... and h0_t / h1_{t-1}, including the peer's half that the peer copied in: the peer may copy again
            if (q == 2) mbar_arrive_remote(&bars.h0_empty[t & 1], peer);
            if (q == 3) mbar_arrive_remote(&bars.h1_empty, peer);
          }
          p_cell += mark();
          if (!PROJ && layer == 1 && t >= 1) mbar_wait_cta<false>(&bars.fc_done, (t - 1) & 1);  // FC(t-1) has read the partials
          p_fc += mark();
          float fsum[2][8];  // Linear partials [o][row slot j*2+e]
#pragma unroll
          for (int i = 0; i < 16; ++i) fsum[i >> 3][i & 7] = 0.f;
          __half hv[2][8];  // h (fp16 hi) [hh][row slot], held back for layer 1
          __half lv[2][8];
          uint8_t* hb = smem + (layer ? sp.h1 : sp.h0 + (t & 1) * nkh * S_KBLK) + s * S_KBLK;  // this slice's k-block
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int u = s * US + 16 * q + (lane >> 2) + 8 * hh;
            const float* bl = bias_g + (layer ? 4 * H : 0);
            const float b4[4] = {bl[u], bl[H + u], bl[2 * H + u], bl[3 * H + u]};
            const float w0 = fcw[u], w1 = fcw[H + u];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int ri = 4 * j + 2 * hh + e;
                const int ci = hh * 8 + j * 2 + e;
                float cp = layer ? c1[ci] : c0[ci];
                if constexpr (CARRY) {
                  if (rows[8 * j + 2 * (lane & 3) + e].restart == t) cp = 0.f;
                }
                float h;
                const float cn = lstm_cell<X3>(acc[0][ri], acc[1][ri], acc[2][ri], acc[3][ri], b4, cp, h);
                if (layer) c1[ci] = cn; else c0[ci] = cn;
                __half hi = __float2half_rn(h);
                __half lo = __float2half_rn(h - __half2float(hi));
                if constexpr (CARRY) {
                  const int n = 8 * j + 2 * (lane & 3) + e, r = row0 + n;
                  int store_t;
                  if constexpr (PHASED) store_t = __float_as_int(rows[n].scale); else store_t = a.store_step;
                  if (t == store_t && r < a.R) {
                    const size_t o = carry_idx(a, r, u) + layer * a.io_layer;
                    a.io_h[o] = h;
                    a.io_c[o] = cn;
                  }
                  // the row enters step t + 1 with zero state: its h_t operand is zero.  Layer 1 of step t then reads a
                  // zero h0_t, so this row's output at step t is wrong.  Exactness needs that output never read: step t
                  // is frame -1 of the slot's new clip, its cRM is frame -1 - look_ahead, and istft_stream_kernel reads
                  // frames >= 0 only (the fp32 stream's stream_reset_kernel zeroes the same operand)
                  if (rows[n].restart == t + 1) hi = lo = __float2half_rn(0.f);
                }
                hv[hh][j * 2 + e] = hi;
                lv[hh][j * 2 + e] = lo;
                if (!PROJ && layer) { fsum[0][j * 2 + e] += h * w0; fsum[1][j * 2 + e] += h * w1; }
                if constexpr (PROJ) {
                  const int r = row0 + 8 * j + 2 * (lane & 3) + e;
                  if (layer && r < a.R) a.h1[((size_t)t * a.R + r) * H + u] = h;
                }
              }
          }
          if (layer == 1) {
            if constexpr (!PROJ) {
              // Linear(H->2) in fp32: sum over the warp's units (lanes with equal lane % 4 hold the same rows)
#pragma unroll
              for (int o = 0; o < 2; ++o)
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                  float v = fsum[o][r];
                  v += __shfl_xor_sync(0xffffffffu, v, 4);
                  v += __shfl_xor_sync(0xffffffffu, v, 8);
                  v += __shfl_xor_sync(0xffffffffu, v, 16);
                  fsum[o][r] = v;
                }
              if (lane < 4) {
#pragma unroll
                for (int o = 0; o < 2; ++o)
#pragma unroll
                  for (int r = 0; r < 8; ++r) my_part[o * NB + 8 * (r >> 1) + 2 * lane + (r & 1)] = fsum[o][r];
              }
            }
            p_cell += mark();
            // every layer-1 MMA of this step in this CTA has consumed h1_{t-1}: overwrite it with h1_t
            mbar_wait_cta<false>(&bars.l1_done, t & 1);
            p_l1 += mark();
            // ... and in the peer, which also means the peer holds this slice's h1_{t-1} copy: its source may go
            mbar_wait_cta<false>(&bars.h1_empty, t & 1);
            p_h1e += mark();
          } else if (t >= 2) {
            p_cell += mark();
            // the peer's layer-1 MMAs of step t-2 have read h0_{t-2} in buffer t & 1 (and so this slice's copy of it
            // has landed there); this CTA's own readers of the buffer are ordered by the ring turn (DESIGN 4.1)
            mbar_wait_cta<false>(&bars.h0_empty[t & 1], ((t - 2) >> 1) & 1);
            p_h0e += mark();
          }
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int u = 16 * q + (lane >> 2) + 8 * hh;  // unit within the slice
            uint8_t* ub = hb + (u & 7) * 2;
            const int chunk = u >> 3;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int n = 8 * j + 2 * (lane & 3) + e;
                uint8_t* p = ub + (n >> 3) * 1024 + (n & 7) * 128 + ((chunk ^ (n & 7)) << 4);
                *reinterpret_cast<__half*>(p) = hv[hh][j * 2 + e];
                if (X3) *reinterpret_cast<__half*>(p + LO) = lv[hh][j * 2 + e];
              }
          }
          fence_proxy_async_smem();
          __syncwarp();
          uint64_t* ready = layer ? &bars.h1_ready : &bars.h0_ready[t & 1];
          if (lane == 0) mbar_arrive(ready);
          // the slice's k-block (hi, lo) into the same place of the peer, completing on the peer's ready barrier
          named_sync(1 + m, 128);
          if (q == 0 && lane == 0) {
            mbar_arrive_expect_tx_remote(ready, peer, PARTS * S_KBLK);
            bulk_s2s_remote(hb, S_KBLK, ready, peer);
            if (X3) bulk_s2s_remote(hb + LO, S_KBLK, ready, peer);
          }
          if constexpr (PROBE) {
            p_cell += mark();
            if (probe_cta && it < a.stamp_its && q == 0 && lane == 0) {
              long long* r = record(it, layer, m);
              r[PF_T_BEGIN] = p_t0; r[PF_T_MMA0] = p_mma0; r[PF_T_MMA1] = p_mma1; r[PF_T_END] = pt;
              r[PF_OPERAND] = p_opnd; r[PF_TURN] = p_turn; r[PF_W_FULL] = p_wfull; r[PF_WAIT_GROUP] = p_wgw;
              r[PF_GROUP_LAT] = p_lat; r[PF_STAGES] = nkb * PARTS; r[PF_CELL] = p_cell; r[PF_L1_DONE] = p_l1;
              r[PF_H1_EMPTY] = p_h1e; r[PF_H0_EMPTY] = p_h0e; r[PF_FC_DONE] = p_fc; r[PF_GT_BEGIN] = p_g0;
            }
          }
        }
        tile_base += ((it < Tp) ? PL.tiles0 : 0) + ((it >= 1) ? PL.tiles1 : 0);
      }
    }
  }

  // ---------------- teardown
  __syncthreads();
  cluster_sync_all();  // no CTA leaves while a peer may still signal its barriers or copy into it
}

// fullsubnet's sub-band stack and fast_fullsubnet's bottleneck: gathered x_t, fused Linear
template <bool X3, bool PROBE>
__global__ void __launch_bounds__(NTHREADS, 1) sb_lstm_tc_kernel(const __grid_constant__ KArgs a) {
  sb_lstm_tc_body<X3, PROBE, false, false>(a);
}

// improved_fullsubnet's sections: precomputed layer-0 projection, h1 stored for the caller's head
template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) sb_proj_lstm_tc_kernel(const __grid_constant__ KArgs a) {
  sb_lstm_tc_body<X3, false, true, false>(a);
}

// chunked streaming: fullsubnet's sub-band stack continued from a carried (h, c), frame-major cRM
template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) sb_carry_lstm_tc_kernel(const __grid_constant__ KArgs a) {
  sb_lstm_tc_body<X3, false, false, true>(a);
}

// chunked streaming: fast_fullsubnet's bottleneck continued from a carried (h, c), every row at its own block phase
template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) sb_phased_lstm_tc_kernel(const __grid_constant__ KArgs a) {
  sb_lstm_tc_body<X3, false, false, true, true>(a);
}

// ---------------------------------------------------------------- two-pass stack (DESIGN 4.1.1)
// The whole-clip stack as two persistent kernels over the same packed image, one per layer, with h0_t handed over
// through global memory: a CTA then holds one layer's state only, which makes room for NB2 = 48 rows per pair, so each
// streamed weight byte meets 48 rows instead of 32.  Per (gate, unit, row) both passes issue the fused kernel's MMAs in
// its k order and part order into the same accumulator, apply its cell math and sum the Linear in its order; m64n48k16
// computes every element as m64n32k16 does, so the result is the fused kernel's, bit for bit.
//   layer 0 (sb_l0_tc_kernel): gathered x_t and h0_{t-1} -> h0_t, written to the B-operand image (hi, lo) in shared
//           memory as in the fused kernel and from there by a bulk store to h0ws;
//   layer 1 (sb_l1_tc_kernel): h0_t bulk-loaded from h0ws into a single buffer, h1 single-buffered as in the fused kernel,
//           Linear(H -> 2) and the output store of the fused kernel.
// h0ws holds the image of pair p (of the launch), step t at [(p Tp + t) img], img = PARTS nkh S_KBLK2 bytes: the hi
// k-blocks of all H units, then the lo k-blocks.  Clusters are one pair, the ring is FSN_TC_STAGES deep.
constexpr int NB2 = 48;                 // rows per CTA pair (MMA N)
constexpr int S_KBLK2 = NB2 * KB * 2;   // 6144 B: one k-block of the state operand
constexpr int X_BLK2 = NB2 * KS * 2;    // 3072 B: x_t
// pairs per launch, fixed so that the workspace size does not depend on the device: two full waves of 66 resident
// pairs on the 132-SM H100 SXM (a part with fewer SMs ends each chunk in a partial wave)
constexpr int SPLIT_CHUNK_PAIRS = 132;

__host__ __device__ inline Smem smem_plan2(int H, int stages, bool x3, int layer) {
  Smem s;
  const int nkh = H / KB;
  uint32_t o = 0;
  s.w = o; o += stages * W_TILE;
  s.x = o; o += layer ? 0 : 2 * X_BLK2;
  s.h0 = o; o += (layer ? 1 : 2) * nkh * S_KBLK2;  // layer 1: h0_t as loaded; layer 0: double-buffered as in the fused kernel
  s.h1 = o; o += layer ? nkh * S_KBLK2 : 0;
  s.lo = o; o += x3 ? (o - s.x) : 0;
  s.fcw = o; o += layer ? 4 * MAX_MT * 2 * NB2 * 4 : 0;
  s.fcp = o; o += layer ? 2 * 2 * NB2 * 4 : 0;
  s.outst = o; o += layer ? NB2 * 2 * OUT_T * 4 : 0;
  s.rows = o; o += NB2 * 16;
  s.bars = o; o += 256;
  s.total = o;
  return s;
}

struct Bars2 {
  uint64_t w_full[MAX_STAGES], w_empty[MAX_STAGES];
  uint64_t x_full[2], x_empty[2];       // layer 0: the gathered x_t
  uint64_t h_ready[2], h_empty[2];      // the pass's own state (layer 0: h0 buffers, layer 1: h1 in [0])
  uint64_t h0_full, h0_free;            // layer 1: h0_t loaded / read by every MMA of this CTA
  uint64_t l1_done, fc_done;
  uint64_t fcp_full[2], fcp_empty[2];
  uint64_t turn[MAX_MT];
};
static_assert(sizeof(Bars2) <= 256, "barrier block too large");

struct SplitArgs {
  KArgs k;
  uint8_t* h0ws;
  int row_base;  // first row of this launch's pair 0
};

template <bool X3, int LAYER>
__device__ __forceinline__ void sb_split_body(const SplitArgs& sa) {
  constexpr int PARTS = X3 ? 2 : 1;
  constexpr int NJ = NB2 / 8;  // accumulator row groups
  const KArgs& a = sa.k;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int H = a.H;
  const int MT = H / 128;
  const int nkh = H / KB;
  const int STAGES = a.stages;
  const uint32_t cl_rank = cluster_ctarank();
  const int half = (int)(cl_rank & 1u);
  const uint32_t peer = cl_rank ^ 1u;
  const Smem sp = smem_plan2(H, STAGES, X3, LAYER);
  const uint32_t LO = sp.lo - sp.x;
  const PackedLayout PL = packed_layout(H, X3);
  Bars2& bars = *reinterpret_cast<Bars2*>(smem + sp.bars);
  RowInfo* rows = reinterpret_cast<RowInfo*>(smem + sp.rows);
  float* fc_part = reinterpret_cast<float*>(smem + sp.fcw);
  float* fcp = reinterpret_cast<float*>(smem + sp.fcp);
  float* outst = reinterpret_cast<float*>(smem + sp.outst);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pair = blockIdx.x >> 1;
  const int row0 = sa.row_base + pair * NB2;
  const int Tp = a.Tp;
  const uint32_t img = PARTS * nkh * S_KBLK2;
  uint8_t* ws_pair = sa.h0ws + (size_t)pair * Tp * img;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&bars.w_full[s], 1); mbar_init(&bars.w_empty[s], 1); }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bars.x_full[i], 1); mbar_init(&bars.x_empty[i], 4 * MT);
      mbar_init(&bars.h_ready[i], 5 * MT);  // 4 MT local warps + MT peer copies
      mbar_init(&bars.h_empty[i], MT);
      mbar_init(&bars.fcp_full[i], 1); mbar_init(&bars.fcp_empty[i], 1);
    }
    mbar_init(&bars.h0_full, 1);
    mbar_init(&bars.h0_free, 4 * MT);
    mbar_init(&bars.fc_done, 1);
    mbar_init(&bars.l1_done, 4 * MT);
    for (int m = 0; m < MAX_MT; ++m) mbar_init(&bars.turn[m], 4);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < NB2) {
    RowInfo ri;
    const int r = row0 + threadIdx.x;
    ri.src_b = -1; ri.src_f = 0; ri.scale = 0.f; ri.out_idx = 0;
    if (r < a.R) {
      row_to_unit(a.map, r, ri.src_b, ri.src_f);
      ri.scale = a.inv2[ri.src_b];
      const int bq = r / a.Fsub, fq = r - bq * a.Fsub;
      ri.out_idx = bq * 2 * a.Fsub + fq;
    }
    rows[threadIdx.x] = ri;
  }
  {  // zero the state (h_{-1} = 0, x padding)
    uint4* z = reinterpret_cast<uint4*>(smem + sp.x);
    const int n16 = (sp.fcw - sp.x) / 16;
    for (int i = threadIdx.x; i < n16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
  }
  fence_proxy_async_smem();
  __syncthreads();
  cluster_sync_all();

  // registers of warpgroup 0 / of each consumer thread (4 x 128 x REG0 + 12 x 128 x REG1 <= 65536).  x3 layer 1 spills
  // least with 160 for its consumers (Linear partial sums and cell state at 48 rows); everywhere else 56 / 152 spill
  // least (DESIGN 4.1.1)
  constexpr int REG0 = (LAYER == 1 && X3) ? 32 : 56, REG1 = (LAYER == 1 && X3) ? 160 : 152;
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REG0));
    if (warp == 0) {
      // ================= weight-stage producer: this half's stream of this layer, the same every step
      const uint8_t* stream = a.packed + ((size_t)half * (PL.tiles0 + PL.tiles1) + (LAYER ? PL.tiles0 : 0)) * W_TILE;
      const size_t tiles = LAYER ? PL.tiles1 : PL.tiles0;
      uint32_t stage = 0, phase = 0;
      for (int t = 0; t < Tp; ++t) {
        const uint8_t* src = stream;
        for (size_t tile = 0; tile < tiles; ++tile, src += W_TILE) {
          mbar_wait_cta<false>(&bars.w_empty[stage], phase ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&bars.w_full[stage], W_TILE);
            bulk_g2s(smem + sp.w + stage * W_TILE, src, W_TILE, &bars.w_full[stage]);
          }
          __syncwarp();
          if (++stage == (uint32_t)STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (LAYER == 0 && warp == 2) {
      // ================= x_t gather, as in the fused kernel
      const int nmag = 2 * a.Ns + 1;
      for (int t = 0; t < Tp; ++t) {
        mbar_wait_cta<true>(&bars.x_empty[t & 1], ((t >> 1) & 1) ^ 1);
        uint8_t* xb = smem + sp.x + (t & 1) * X_BLK2;
#pragma unroll 4
        for (int n = 0; n < NB2; ++n) {
          const RowInfo ri = rows[n];
          float v = 0.f;
          if (ri.src_b >= 0 && lane < a.Ksb) {
            const int col = (lane < nmag) ? reflect_idx(ri.src_f + lane - a.Ns, a.F)
                                          : reflect_idx(ri.src_f + (lane - nmag) - a.Nf, a.F);
            const float* src = (lane < nmag) ? a.magT : a.fbT;
            v = src[((size_t)ri.src_b * a.src_T + t) * a.F + col];
            v *= a.unit_scale ? a.unit_scale[(size_t)t * a.R + row0 + n] : ri.scale;
          }
          const __half hi = __float2half_rn(v);
          *reinterpret_cast<__half*>(xb + swz64_off(n, lane)) = hi;
          if (X3) *reinterpret_cast<__half*>(xb + LO + swz64_off(n, lane)) = __float2half_rn(v - __half2float(hi));
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars.x_full[t & 1]);
      }
    } else if (LAYER == 1 && warp == 2) {
      // ================= h0_t loader: the pair's image of step t, once every MMA of this CTA has read h0_{t-1}
      for (int t = 0; t < Tp; ++t) {
        if (t > 0) mbar_wait_cta<false>(&bars.h0_free, (t - 1) & 1);
        if (elect_one()) {
          const uint8_t* src = ws_pair + (size_t)t * img;
          mbar_expect_tx(&bars.h0_full, img);
          bulk_g2s(smem + sp.h0, src, nkh * S_KBLK2, &bars.h0_full);
          if (X3) bulk_g2s(smem + sp.h0 + LO, src + nkh * S_KBLK2, nkh * S_KBLK2, &bars.h0_full);
        }
        __syncwarp();
      }
    } else if (LAYER == 1 && warp == 3) {
      // ================= Linear(H -> 2) and output staging, as in the fused kernel (rows lane and lane + 32)
      const float fcb0 = half ? 0.f : reinterpret_cast<const float*>(a.packed + PL.off_fcb)[0];
      const float fcb1 = half ? 0.f : reinterpret_cast<const float*>(a.packed + PL.off_fcb)[1];
      int staged = 0, t_stage0 = 0;
      for (int t = 0; t < Tp; ++t) {
        mbar_wait_cta<true>(&bars.h_ready[0], t & 1);
        float s0[2], s1[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int n = lane + 32 * k;
          s0[k] = fcb0; s1[k] = fcb1;
          if (t >= a.la && n < NB2) {
            for (int w = 0; w < 4 * MT; ++w) {
              s0[k] += fc_part[(w * 2 + 0) * NB2 + n];
              s1[k] += fc_part[(w * 2 + 1) * NB2 + n];
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars.fc_done);
        if (t < a.la) continue;
        const int u = t - a.la, b = u & 1;
        float* pb = fcp + b * 2 * NB2;
        if (half) {
          mbar_wait<true>(&bars.fcp_empty[b], ((u >> 1) & 1) ^ 1);
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int n = lane + 32 * k;
            if (n < NB2) { st_remote_f32(pb + n, peer, s0[k]); st_remote_f32(pb + NB2 + n, peer, s1[k]); }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive_cluster(&bars.fcp_full[b], peer);
          continue;
        }
        mbar_wait<true>(&bars.fcp_full[b], (u >> 1) & 1);
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int n = lane + 32 * k;
          if (n < NB2) { s0[k] += pb[n]; s1[k] += pb[NB2 + n]; }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive_cluster(&bars.fcp_empty[b], peer);
        if (staged == 0) t_stage0 = u;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int n = lane + 32 * k;
          if (n < NB2) {
            outst[(n * 2 + 0) * OUT_T + staged] = act_apply(s0[k], a.act);
            outst[(n * 2 + 1) * OUT_T + staged] = act_apply(s1[k], a.act);
          }
        }
        ++staged;
        if (staged == OUT_T || t == Tp - 1) {
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int n = lane + 32 * k;
            if (n >= NB2) continue;
            const RowInfo ri = rows[n];
            if (ri.src_b < 0) continue;
#pragma unroll
            for (int o = 0; o < 2; ++o) {
              float* dst = a.crm + ((size_t)ri.out_idx + (size_t)o * a.Fsub) * a.T + t_stage0;
              for (int i = 0; i < staged; ++i) dst[i] = outst[(n * 2 + o) * OUT_T + i];
            }
          }
          staged = 0;
        }
      }
    }
  } else {
    // ================= consumer warpgroup m: slice s = MT half + m of this layer.  Fragment of thread (warp q, lane l):
    // unit 64 s + 16 q + l/4 + 8 hh, row n = 8 j + 2 (l%4) + e, register acc[g][4 j + 2 hh + e]
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REG1));
    const int m = __shfl_sync(0xffffffffu, (warp - 4) >> 2, 0);
    const int q = __shfl_sync(0xffffffffu, warp & 3, 0);
    const int s = half * MT + m;
    if (m < MT) {
      const float* bias_g = reinterpret_cast<const float*>(a.packed + PL.off_bias) + (LAYER ? 4 * H : 0);
      const float* fcw = reinterpret_cast<const float*>(a.packed + PL.off_fcw);
      float* my_part = fc_part + (size_t)(warp - 4) * 2 * NB2;
      float c[4 * NJ];
#pragma unroll
      for (int i = 0; i < 4 * NJ; ++i) c[i] = 0.f;
      const uint32_t a_lo0 = wg::desc_lo(smem_u32(smem + sp.w));
      const uint32_t w_full0 = smem_u32(&bars.w_full[0]), w_empty0 = smem_u32(&bars.w_empty[0]);
      const uint32_t turn_next = smem_u32(&bars.turn[m + 1 < MT ? m + 1 : 0]);
      const uint32_t rel_local = q == 0;
      const int nkb = LAYER ? PL.nkb1 : PL.nkb0;
      const size_t tiles = LAYER ? PL.tiles1 : PL.tiles0;
      int h_seen = 0, turns = 0;
      for (int t = 0; t < Tp; ++t) {
        if (LAYER == 0) {
          mbar_wait_cta<false>(&bars.x_full[t & 1], (t >> 1) & 1);
          for (; h_seen < t; ++h_seen) mbar_wait_cta<false>(&bars.h_ready[h_seen & 1], (h_seen >> 1) & 1);  // h0_{t-1}
        } else {
          mbar_wait_cta<false>(&bars.h0_full, t & 1);  // h0_t; h1_{t-1} is waited for after the h0_t k ranges
        }
        const uint32_t x_addr = smem_u32(smem + sp.x + (t & 1) * X_BLK2);
        const uint32_t h0_cur = smem_u32(smem + sp.h0);
        const uint32_t h0_prev = smem_u32(smem + sp.h0 + ((t + 1) & 1) * nkh * S_KBLK2);
        const uint32_t h1_prev = smem_u32(smem + sp.h1);
        const size_t first = (size_t)t * tiles + (size_t)m * nkb * PARTS;
        float acc[4][4 * NJ];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
#pragma unroll
          for (int i = 0; i < 4 * NJ; ++i) acc[g][i] = 0.f;
          wg::fence_operand(acc[g]);
        }
        int prev_stage = -1;
        if (m > 0 || t > 0) { mbar_wait_cta<false>(&bars.turn[m], turns & 1); ++turns; }
        int stage = __shfl_sync(0xffffffffu, (int)(first % (size_t)STAGES), 0);
        uint32_t wphase = __shfl_sync(0xffffffffu, (uint32_t)((first / (size_t)STAGES) & 1), 0);
        auto issue_stage = [&](int part, uint32_t bd, uint32_t b_hi, uint32_t ends_block) {
          mbar_wait_cta_warp(w_full0 + 8 * stage, wphase);
          mbar_arrive_elect_if(turn_next, ends_block);
          wg::fence();
          const uint32_t ad = a_lo0 + stage * (W_TILE >> 4);
#pragma unroll
          for (int kk = 0; kk < 2; ++kk)
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              const uint32_t a_off = g * (W_SUB >> 4) + kk * 2;
              wg::mma_f16_n48_w(acc[g], ad, a_off, wg::DESC_SW64_HI, bd, kk * 2, b_hi);
              if (X3 && part == 0) wg::mma_f16_n48_w(acc[g], ad, a_off, wg::DESC_SW64_HI, bd, (LO >> 4) + kk * 2, b_hi);
            }
          wg::commit();
          wg::wait<1>();
          release_stage(w_empty0 + 8 * prev_stage, prev_stage >= 0, rel_local, 0u, 0u);
          prev_stage = stage;
          if (++stage == STAGES) { stage = 0; wphase ^= 1; }
        };
        // B operand k ranges: layer 0: [x_t] [h0_{t-1} (H)]; layer 1: [h0_t (H)] [h1_{t-1} (H)] (the fused kernel's)
        if (LAYER == 0) {
#pragma unroll
          for (int part = 0; part < PARTS; ++part) issue_stage(part, wg::desc_lo(x_addr), wg::DESC_SW64_HI, 0u);
        }
        const int nseg = LAYER ? 2 : 1;
        int seg = 0;
        do {
          if (LAYER == 1 && seg == 1)
            for (; h_seen < t; ++h_seen) mbar_wait_cta<false>(&bars.h_ready[0], h_seen & 1);  // h1_{t-1}
          uint32_t bd = wg::desc_lo(LAYER == 0 ? h0_prev : seg == 0 ? h0_cur : h1_prev);
          int kb = 0;
          do {
            const uint32_t ends_block = seg == nseg - 1 && kb == nkh - 1;
#pragma unroll
            for (int part = 0; part < PARTS; ++part) issue_stage(part, bd, wg::DESC_SW128_HI, 0u);
            // layer 1: the first h1 stage's wait retired the last h0_t stage - this warp is done with h0_t
            if (LAYER == 1 && seg == 1 && kb == 0 && lane == 0) mbar_arrive(&bars.h0_free);
#pragma unroll
            for (int part = 0; part < PARTS; ++part)
              issue_stage(part, bd + (64 >> 4), wg::DESC_SW128_HI, part == PARTS - 1 ? ends_block : 0u);
            bd += S_KBLK2 >> 4;
          } while (++kb < nkh);
        } while (++seg < nseg);
        wg::wait<0>();
#pragma unroll
        for (int g = 0; g < 4; ++g) wg::fence_operand(acc[g]);
        release_stage(w_empty0 + 8 * prev_stage, 1u, rel_local, 0u, 0u);
        if (lane == 0) mbar_arrive(LAYER ? &bars.l1_done : &bars.x_empty[t & 1]);
        // this warpgroup's MMAs have read the state the peer copied in (layer 0: h0_{t-1}, buffer (t + 1) & 1)
        if (q == 2 && lane == 0) mbar_arrive_remote(&bars.h_empty[LAYER ? 0 : (t + 1) & 1], peer);
        if (LAYER == 1 && t >= 1) mbar_wait_cta<false>(&bars.fc_done, (t - 1) & 1);  // FC(t-1) has read the partials
        __half hv[2][2 * NJ], lv[2][2 * NJ];
        uint8_t* hb = smem + (LAYER ? sp.h1 : sp.h0 + (t & 1) * nkh * S_KBLK2) + s * S_KBLK2;
        float bias[2][4], fw[2][2];  // biases and Linear weights of the thread's units u(hh), hh = 0, 1
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int u = s * US + 16 * q + (lane >> 2) + 8 * hh;
#pragma unroll
          for (int g = 0; g < 4; ++g) bias[hh][g] = bias_g[g * H + u];
          fw[hh][0] = LAYER ? fcw[u] : 0.f;
          fw[hh][1] = LAYER ? fcw[H + u] : 0.f;
        }
        // row slot by row slot, both units of the slot, so that a slot's Linear partial sum (the fused kernel's: its
        // unit hh = 0 term, then hh = 1, then the warp's lane sums) is stored before the next slot's cells run
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float f0 = 0.f, f1 = 0.f;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int ri = 4 * j + 2 * hh + e;
              const int ci = hh * 2 * NJ + j * 2 + e;
              float h;
              c[ci] = lstm_cell<X3>(acc[0][ri], acc[1][ri], acc[2][ri], acc[3][ri], bias[hh], c[ci], h);
              const __half hi = __float2half_rn(h);
              hv[hh][j * 2 + e] = hi;
              lv[hh][j * 2 + e] = __float2half_rn(h - __half2float(hi));
              if (LAYER == 1) { f0 += h * fw[hh][0]; f1 += h * fw[hh][1]; }
            }
            if (LAYER == 1) {
              // Linear(H->2) in fp32: sum over the warp's units (lanes with equal lane % 4 hold the same rows)
              f0 += __shfl_xor_sync(0xffffffffu, f0, 4);
              f0 += __shfl_xor_sync(0xffffffffu, f0, 8);
              f0 += __shfl_xor_sync(0xffffffffu, f0, 16);
              f1 += __shfl_xor_sync(0xffffffffu, f1, 4);
              f1 += __shfl_xor_sync(0xffffffffu, f1, 8);
              f1 += __shfl_xor_sync(0xffffffffu, f1, 16);
              if (lane < 4) {
                my_part[8 * j + 2 * lane + e] = f0;
                my_part[NB2 + 8 * j + 2 * lane + e] = f1;
              }
            }
          }
        if (LAYER == 1) {
          // every layer-1 MMA of step t in this CTA, and in the peer, has read h1_{t-1}: overwrite it with h1_t
          mbar_wait_cta<false>(&bars.l1_done, t & 1);
          mbar_wait_cta<false>(&bars.h_empty[0], t & 1);
        } else if (t >= 1) {
          // the peer's MMAs of step t - 1 have read h0_{t-2} in buffer t & 1; this CTA's own readers of the buffer are
          // ordered by the ring turn, as in the fused kernel
          mbar_wait_cta<false>(&bars.h_empty[t & 1], ((t - 1) >> 1) & 1);
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int u = 16 * q + (lane >> 2) + 8 * hh;
          uint8_t* ub = hb + (u & 7) * 2;
          const int chunk = u >> 3;
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int n = 8 * j + 2 * (lane & 3) + e;
              uint8_t* p = ub + (n >> 3) * 1024 + (n & 7) * 128 + ((chunk ^ (n & 7)) << 4);
              *reinterpret_cast<__half*>(p) = hv[hh][j * 2 + e];
              if (X3) *reinterpret_cast<__half*>(p + LO) = lv[hh][j * 2 + e];
            }
        }
        fence_proxy_async_smem();
        __syncwarp();
        // h_t to the peer (and this CTA's readers), except layer 0's last h0, which no MMA of the pass reads: the peer
        // never waits for that copy, so it could still be in flight when the pair leaves the SMs (layer 1's last copy
        // is waited for by the peer's Linear warp before its teardown)
        const bool exchange = LAYER == 1 || t < Tp - 1;
        uint64_t* ready = &bars.h_ready[LAYER ? 0 : t & 1];
        if (exchange && lane == 0) mbar_arrive(ready);
        // layer 0: the store of step t - 1 has read its buffer, which the writes of step t + 1 reuse (they follow the
        // named barrier below)
        if (LAYER == 0 && q == 0 && lane == 0) bulk_wait_read_all();
        named_sync(1 + m, 128);
        if (q == 0 && lane == 0) {
          if (exchange) {
            mbar_arrive_expect_tx_remote(ready, peer, PARTS * S_KBLK2);
            bulk_s2s_remote(hb, S_KBLK2, ready, peer);
            if (X3) bulk_s2s_remote(hb + LO, S_KBLK2, ready, peer);
          }
          if (LAYER == 0) {
            uint8_t* dst = ws_pair + (size_t)t * img + s * S_KBLK2;
            bulk_s2g(dst, hb, S_KBLK2);
            if (X3) bulk_s2g(dst + nkh * S_KBLK2, hb + LO, S_KBLK2);
            bulk_commit();
          }
        }
      }
      if (LAYER == 0 && q == 0 && lane == 0) bulk_wait_all();
    }
  }

  __syncthreads();
  cluster_sync_all();
}

template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) sb_l0_tc_kernel(const __grid_constant__ SplitArgs a) {
  sb_split_body<X3, 0>(a);
}
template <bool X3>
__global__ void __launch_bounds__(NTHREADS, 1) sb_l1_tc_kernel(const __grid_constant__ SplitArgs a) {
  sb_split_body<X3, 1>(a);
}

}  // namespace tc

static int sb_ksb(const fsn_model_desc* d) { return (2 * d->sb_num_neighbors + 1) + (2 * d->fb_num_neighbors + 1); }

static bool sb_tc_shape_ok(int H, int Ksb) { return H % 128 == 0 && H / 128 <= tc::MAX_MT && H >= 128 && Ksb <= tc::KS; }

bool sb_tc_supported(const fsn_model_desc* d) {
  if (d->cell_type != FSN_CELL_LSTM) return false;  // GRU: fp32 kernels only
  return sb_tc_shape_ok(d->sb_hidden, sb_ksb(d));
}

size_t sb_tc_packed_bytes_raw(int H, bool x3, bool proj) { return tc::packed_layout(H, x3, proj).bytes; }

size_t sb_tc_packed_bytes(const fsn_model_desc* d) {
  if (!sb_tc_supported(d)) return 0;
  return sb_tc_packed_bytes_raw(d->sb_hidden, d->precision == FSN_PREC_F16X3_TC);
}

int sb_tc_pack_raw(const fsn_seq_weights* sb, int H, int Ksb, int fc_out, void* packed, cudaStream_t st, bool x3,
                   bool proj) {
  FSN_REQUIRE(sb_tc_shape_ok(H, proj ? 0 : Ksb), FSN_ERR_UNSUPPORTED,
              "the fp16 tensor-core LSTM stack needs a hidden size in {128,256,384} and an input width <= 32");
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  tc::pack_kernel<<<sms * 4, 256, 0, st>>>(sb->w_ih[0], sb->w_hh[0], sb->w_ih[1], sb->w_hh[1], sb->b_ih[0], sb->b_hh[0],
                                           sb->b_ih[1], sb->b_hh[1], sb->fc_w, sb->fc_b, H, Ksb, x3 ? 1 : 0, fc_out,
                                           proj ? 1 : 0, (uint8_t*)packed);
  FSN_CHECK_LAUNCH("sb pack_kernel");
  return FSN_OK;
}

int sb_tc_pack(const fsn_model_desc* d, const fsn_seq_weights* sb, void* packed, cudaStream_t st) {
  FSN_REQUIRE(sb_tc_supported(d), FSN_ERR_UNSUPPORTED,
              "FSN_PREC_F16_TC / FSN_PREC_F16X3_TC need sb_hidden in {128,256,384} and sub-band input width <= 32");
  return sb_tc_pack_raw(sb, d->sb_hidden, sb_ksb(d), 2, packed, st, d->precision == FSN_PREC_F16X3_TC);
}

// launch configuration of `pairs` CTA pairs in clusters of `cluster` pairs (2 x cluster CTAs; the caller keeps `attr`
// alive while cfg is used)
template <bool X3, bool PROBE = false>
static int sb_tc_config(int H, int stages, int cluster, int pairs, cudaStream_t st, cudaLaunchConfig_t& cfg,
                        cudaLaunchAttribute* attr, const void* kern = (const void*)tc::sb_lstm_tc_kernel<X3, PROBE>) {
  const tc::Smem sp = tc::smem_plan(H, stages, X3);
  const size_t smem = sp.total + 1024;  // slack for the 1024-byte alignment of the dynamic segment
  int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                      "sb_lstm_tc smem attr");
  if (rc) return rc;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(2 * pairs);
  cfg.blockDim = dim3(128 + 128 * (H / 128));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2 * cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return FSN_OK;
}

template <bool X3, bool PROBE>
static int sb_tc_launch(const tc::KArgs& a, int H, cudaStream_t st) {
  const int pairs = cdiv(cdiv(a.R, tc::NB), a.cluster) * a.cluster;  // padding pairs own no valid row
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  int rc = sb_tc_config<X3, PROBE>(H, a.stages, a.cluster, pairs, st, cfg, attr);
  if (rc) return rc;
  rc = check_cuda(cudaLaunchKernelEx(&cfg, tc::sb_lstm_tc_kernel<X3, PROBE>, a), "sb_lstm_tc_kernel launch");
  if (rc) return rc;
  FSN_CHECK_LAUNCH("sb_lstm_tc_kernel");
  return FSN_OK;
}

static int sb_tc_kargs(const SbTcArgs& s, tc::KArgs& a) {
  memset(&a, 0, sizeof(a));
  a.packed = (const uint8_t*)s.packed;
  a.magT = s.magT; a.fbT = s.fbT; a.inv2 = s.inv2; a.unit_scale = s.unit_scale; a.crm = s.crm;
  a.R = s.map.B * s.map.Fsub; a.F = s.F; a.Tp = s.steps > 0 ? s.steps : s.Tp; a.la = s.la; a.T = a.Tp - s.la;
  a.src_T = s.Tp; a.shrink = s.shrink > 1 ? s.shrink : 1;
  a.Ns = s.Ns; a.Nf = s.Nf; a.H = s.H; a.Ksb = (2 * s.Ns + 1) + (2 * s.Nf + 1); a.act = s.act;
  a.Fsub = s.map.Fsub; a.map = s.map;
  a.stamps = s.stamps; a.stamp_ctas = s.stamp_ctas; a.stamp_its = s.stamp_its;
  FSN_REQUIRE(sb_tc_shape_ok(a.H, a.Ksb), FSN_ERR_UNSUPPORTED, "sb_lstm_tc: unsupported hidden size %d / input width %d",
              a.H, a.Ksb);
  a.proj = nullptr; a.h1 = nullptr;
  int stages = 0, cluster = 0;
  sb_tc_ring_defaults(stages, cluster);
  // an explicit launch configuration (the unit-test hook) overrides the environment
  a.stages = s.stages ? s.stages : stages;
  a.cluster = s.cluster ? s.cluster : cluster;
  return FSN_OK;
}

size_t sb_tc_split_ws_bytes(int R, int Tp, int H, bool x3, int chunk_pairs) {
  if (!sb_tc_shape_ok(H, 0) || R <= 0 || Tp <= 0) return 0;
  const int pairs = std::min(cdiv(R, tc::NB2), chunk_pairs > 0 ? chunk_pairs : tc::SPLIT_CHUNK_PAIRS);
  return (size_t)pairs * Tp * (x3 ? 2 : 1) * (H / tc::KB) * tc::S_KBLK2;
}

template <bool X3>
static int sb_split_launch(const tc::SplitArgs& sa, int pairs, int layer, cudaStream_t st) {
  void (*kern)(tc::SplitArgs) = layer ? tc::sb_l1_tc_kernel<X3> : tc::sb_l0_tc_kernel<X3>;
  const size_t smem = tc::smem_plan2(sa.k.H, sa.k.stages, X3, layer).total + 1024;
  const char* name = layer ? "sb_l1_tc_kernel" : "sb_l0_tc_kernel";
  int rc = check_cuda(cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), name);
  if (rc) return rc;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(2 * pairs);
  cfg.blockDim = dim3(128 + 128 * (sa.k.H / 128));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if ((rc = check_cuda(cudaLaunchKernelEx(&cfg, kern, sa), name))) return rc;
  FSN_CHECK_LAUNCH(name);
  return FSN_OK;
}

// the two-pass stack (sb_l0_tc_kernel, sb_l1_tc_kernel) over chunks of s.split_chunk pairs (0: SPLIT_CHUNK_PAIRS), each
// chunk's h0 through s.h0ws (sb_tc_split_ws_bytes)
static int sb_tc_split_forward(const SbTcArgs& s, cudaStream_t st) {
  FSN_REQUIRE(s.shrink <= 1, FSN_ERR_UNSUPPORTED, "sb_lstm_tc two-pass: no time down-sampling");
  tc::SplitArgs sa;
  memset(&sa, 0, sizeof(sa));
  int rc = sb_tc_kargs(s, sa.k);
  if (rc) return rc;
  sa.k.cluster = 1;
  sa.h0ws = (uint8_t*)s.h0ws;
  const int total = cdiv(sa.k.R, tc::NB2);
  const int chunk = s.split_chunk > 0 ? s.split_chunk : tc::SPLIT_CHUNK_PAIRS;
  for (int p0 = 0; p0 < total; p0 += chunk) {
    const int pairs = std::min(chunk, total - p0);
    sa.row_base = p0 * tc::NB2;
    for (int layer = 0; layer < 2; ++layer)
      if ((rc = s.x3 ? sb_split_launch<true>(sa, pairs, layer, st) : sb_split_launch<false>(sa, pairs, layer, st)))
        return rc;
  }
  return FSN_OK;
}

int sb_tc_forward(const SbTcArgs& s, cudaStream_t st) {
  if (s.h0ws && !s.stamps) return sb_tc_split_forward(s, st);
  tc::KArgs a;
  int rc = sb_tc_kargs(s, a);
  if (rc) return rc;
  if (s.stamps) return s.x3 ? sb_tc_launch<true, true>(a, s.H, st) : sb_tc_launch<false, true>(a, s.H, st);
  return s.x3 ? sb_tc_launch<true, false>(a, s.H, st) : sb_tc_launch<false, false>(a, s.H, st);
}

int sb_tc_carry_forward(const SbTcArgs& s, const SbCarry& io, cudaStream_t st) {
  const bool phased = io.store_at != nullptr;
  FSN_REQUIRE((phased ? io.x != nullptr : s.unit_scale != nullptr) && io.h && io.c && io.restart && io.rps > 0 && s.la == 0 &&
                  s.shrink <= 1 && s.map.G <= 1,
              FSN_ERR_SHAPE,
              "sb_carry_lstm_tc: per-row scales (block-phased: the input), state, restart steps, la = 0 and no drop_band / "
              "shrink");
  tc::KArgs a;
  int rc = sb_tc_kargs(s, a);
  if (rc) return rc;
  a.io_h = io.h; a.io_c = io.c; a.io_slot = io.slot; a.io_layer = io.layer; a.io_rps = io.rps;
  a.restart = io.restart; a.store_step = io.store_step; a.crm_bs = io.crm_bs; a.crm_t0 = io.crm_t0;
  a.xin = io.x; a.store_at = io.store_at;
  const int pairs = cdiv(cdiv(a.R, tc::NB), a.cluster) * a.cluster;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  void (*kern)(tc::KArgs);
  if (phased) kern = s.x3 ? tc::sb_phased_lstm_tc_kernel<true> : tc::sb_phased_lstm_tc_kernel<false>;
  else        kern = s.x3 ? tc::sb_carry_lstm_tc_kernel<true> : tc::sb_carry_lstm_tc_kernel<false>;
  rc = s.x3 ? sb_tc_config<true>(s.H, a.stages, a.cluster, pairs, st, cfg, attr, (const void*)kern)
            : sb_tc_config<false>(s.H, a.stages, a.cluster, pairs, st, cfg, attr, (const void*)kern);
  if (rc) return rc;
  const char* name = phased ? "sb_phased_lstm_tc_kernel" : "sb_carry_lstm_tc_kernel";
  if ((rc = check_cuda(cudaLaunchKernelEx(&cfg, kern, a), name))) return rc;
  FSN_CHECK_LAUNCH(name);
  return FSN_OK;
}

int sb_proj_forward(const SbProjArgs& s, cudaStream_t st) {
  FSN_REQUIRE(s.R > 0 && s.T > 0 && sb_tc_shape_ok(s.H, 0), FSN_ERR_UNSUPPORTED,
              "sb_proj_lstm_tc: unsupported hidden size %d (R=%d, T=%d)", s.H, s.R, s.T);
  FSN_REQUIRE(s.packed && s.P && s.h1, FSN_ERR_SHAPE, "sb_proj_lstm_tc: missing buffer");
  tc::KArgs a;
  memset(&a, 0, sizeof(a));
  a.packed = (const uint8_t*)s.packed; a.proj = s.P; a.h1 = s.h1;
  a.R = s.R; a.Tp = s.T; a.T = s.T; a.H = s.H;
  int stages = 0, cluster = 0;
  sb_tc_ring_defaults(stages, cluster);
  a.stages = s.stages ? s.stages : stages;
  a.cluster = s.cluster ? s.cluster : cluster;
  const int pairs = cdiv(cdiv(a.R, tc::NB), a.cluster) * a.cluster;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  const void* kern = s.x3 ? (const void*)tc::sb_proj_lstm_tc_kernel<true> : (const void*)tc::sb_proj_lstm_tc_kernel<false>;
  int rc = s.x3 ? sb_tc_config<true>(s.H, a.stages, a.cluster, pairs, st, cfg, attr, kern)
                : sb_tc_config<false>(s.H, a.stages, a.cluster, pairs, st, cfg, attr, kern);
  if (rc) return rc;
  rc = s.x3 ? check_cuda(cudaLaunchKernelEx(&cfg, tc::sb_proj_lstm_tc_kernel<true>, a), "sb_proj_lstm_tc_kernel launch")
            : check_cuda(cudaLaunchKernelEx(&cfg, tc::sb_proj_lstm_tc_kernel<false>, a), "sb_proj_lstm_tc_kernel launch");
  if (rc) return rc;
  FSN_CHECK_LAUNCH("sb_proj_lstm_tc_kernel");
  return FSN_OK;
}

// weight ring depth and cluster size of the production launches: FSN_TC_STAGES / FSN_TC_CLUSTER, read once
void sb_tc_ring_defaults(int& stages, int& cluster) {
  static int stages_env = -1;
  if (stages_env < 0) {
    const char* e = getenv("FSN_TC_STAGES");
    stages_env = e ? atoi(e) : 4;
    if (stages_env < 2) stages_env = 2;
    if (stages_env > tc::MAX_STAGES) stages_env = tc::MAX_STAGES;
  }
  static int cluster_env = -1;
  if (cluster_env < 0) {
    const char* e = getenv("FSN_TC_CLUSTER");
    // default: pairs alone (clusters of 2 CTAs): all 66 clusters resident; multicast over 2 or 4 pairs costs residency
    // (30 / 15 clusters) and measured slower (DESIGN 4.1)
    cluster_env = e ? atoi(e) : 1;
    if (cluster_env != 1 && cluster_env != 2 && cluster_env != 4) cluster_env = 1;
  }
  stages = stages_env;
  cluster = cluster_env;
}

}  // namespace fsn

// unit-test hook (tests/test_gpu_subband_tc.py): the sub-band stack on caller-provided inputs and launch configuration
extern "C" size_t fsn_debug_sb_lstm_tc_packed_bytes(int H, int x3) {
  return fsn::sb_tc_shape_ok(H, 0) ? fsn::sb_tc_packed_bytes_raw(H, x3 != 0) : 0;
}

extern "C" int fsn_debug_sb_lstm_tc_max_clusters(int H, int x3, int stages, int cluster, int* clusters) {
  using namespace fsn;
  FSN_REQUIRE(cluster == 1 || cluster == 2 || cluster == 4, FSN_ERR_UNSUPPORTED,
              "sb_lstm_tc: cluster size %d (1, 2 or 4)", cluster);
  FSN_REQUIRE(stages >= 2 && stages <= tc::MAX_STAGES, FSN_ERR_UNSUPPORTED, "sb_lstm_tc: ring depth %d (2, 3 or 4)",
              stages);
  FSN_REQUIRE(sb_tc_shape_ok(H, 0), FSN_ERR_UNSUPPORTED, "sb_lstm_tc: unsupported hidden size %d", H);
  FSN_REQUIRE(clusters, FSN_ERR_SHAPE, "sb_lstm_tc: missing output");
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  int rc = x3 ? sb_tc_config<true>(H, stages, cluster, cluster, nullptr, cfg, attr)
              : sb_tc_config<false>(H, stages, cluster, cluster, nullptr, cfg, attr);
  if (rc) return rc;
  return x3 ? check_cuda(cudaOccupancyMaxActiveClusters(clusters, tc::sb_lstm_tc_kernel<true, false>, &cfg), "sb_lstm_tc occupancy")
            : check_cuda(cudaOccupancyMaxActiveClusters(clusters, tc::sb_lstm_tc_kernel<false, false>, &cfg), "sb_lstm_tc occupancy");
}

static int sb_lstm_tc_hook(const fsn_seq_weights* sb, int H, int Ns, int Nf, int fc_out, int act, int x3,
                           const float* magT, const float* fbT, int B, int F, int src_T, int G, const float* inv2,
                           const float* unit_scale, int la, int steps, int shrink, int stages, int cluster, void* packed,
                           float* crm, long long* stamps, int stamp_ctas, int stamp_steps, fsn_stream_t stream) {
  using namespace fsn;
  // every check precedes the first CUDA call
  FSN_REQUIRE(cluster == 0 || cluster == 1 || cluster == 2 || cluster == 4, FSN_ERR_UNSUPPORTED,
              "sb_lstm_tc: cluster size %d (0, 1, 2 or 4)", cluster);
  FSN_REQUIRE(stages == 0 || (stages >= 2 && stages <= tc::MAX_STAGES), FSN_ERR_UNSUPPORTED,
              "sb_lstm_tc: ring depth %d (0, 2, 3 or 4)", stages);
  FSN_REQUIRE(sb && magT && fbT && inv2 && packed && crm, FSN_ERR_SHAPE, "sb_lstm_tc: missing buffer");
  FSN_REQUIRE(B > 0 && F > 1 && src_T > 0 && Ns >= 0 && Nf >= 0 && Ns < F && Nf < F, FSN_ERR_SHAPE,
              "sb_lstm_tc: bad shape B=%d F=%d src_T=%d Ns=%d Nf=%d", B, F, src_T, Ns, Nf);
  FSN_REQUIRE(fc_out == 1 || fc_out == 2, FSN_ERR_SHAPE, "sb_lstm_tc: fc_out %d (1 or 2)", fc_out);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "sb_lstm_tc: activation %d", act);
  FSN_REQUIRE(shrink >= 1 && G >= 1, FSN_ERR_SHAPE, "sb_lstm_tc: shrink %d / groups %d", shrink, G);
  // drop_band as make_dims applies it
  const int g = (B > 1 && G > 1) ? G : 1;
  FSN_REQUIRE(B == 1 || B > G, FSN_ERR_SHAPE, "sb_lstm_tc: batch size %d <= num_groups %d", B, G);
  const int Fsub = g > 1 ? F / g : F;
  FSN_REQUIRE(Fsub > 0, FSN_ERR_SHAPE, "sb_lstm_tc: num_freqs < num_groups");
  // steps read frames [0, steps) of the source, or with shrink > 1 frame 0 then blocks of `shrink` frames
  const int max_steps = shrink > 1 ? 1 + cdiv(src_T - 1, shrink) : src_T;
  FSN_REQUIRE(steps > 0 && steps <= max_steps && la >= 0 && la < steps, FSN_ERR_SHAPE,
              "sb_lstm_tc: steps %d / look-ahead %d for %d source frames (shrink %d)", steps, la, src_T, shrink);
  FSN_REQUIRE(!(unit_scale && shrink > 1), FSN_ERR_UNSUPPORTED, "sb_lstm_tc: per-step scales with time down-sampling");
  FSN_REQUIRE(sb_tc_shape_ok(H, (2 * Ns + 1) + (2 * Nf + 1)), FSN_ERR_UNSUPPORTED,
              "sb_lstm_tc: unsupported hidden size %d / input width %d", H, (2 * Ns + 1) + (2 * Nf + 1));
  if (stamps) {
    // records exist for CTAs that own rows and for the loop iterations 0 .. steps (layer 1 runs one behind)
    const int ctas = 2 * cdiv(B * Fsub, tc::NB);
    FSN_REQUIRE(stamp_ctas >= 1 && stamp_ctas <= ctas, FSN_ERR_SHAPE, "sb_lstm_tc probe: %d sampled CTAs (1 .. %d)",
                stamp_ctas, ctas);
    FSN_REQUIRE(stamp_steps >= 1 && stamp_steps <= steps + 1, FSN_ERR_SHAPE,
                "sb_lstm_tc probe: %d sampled iterations (1 .. steps + 1 = %d)", stamp_steps, steps + 1);
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = sb_tc_pack_raw(sb, H, (2 * Ns + 1) + (2 * Nf + 1), fc_out, packed, st, x3 != 0);
  if (rc) return rc;
  SbTcArgs a;
  memset(&a, 0, sizeof(a));
  a.packed = packed; a.magT = magT; a.fbT = fbT; a.inv2 = inv2; a.unit_scale = unit_scale; a.crm = crm;
  a.B = B; a.F = F; a.Tp = src_T; a.la = la; a.Ns = Ns; a.Nf = Nf; a.H = H; a.act = act;
  a.steps = steps; a.shrink = shrink; a.x3 = x3 != 0;
  a.map = RowMap{B, F, Fsub, g};
  a.stages = stages; a.cluster = cluster;
  a.stamps = stamps; a.stamp_ctas = stamp_ctas; a.stamp_its = stamp_steps;
  return sb_tc_forward(a, st);
}

extern "C" int fsn_debug_sb_lstm_tc(const fsn_seq_weights* sb, int H, int Ns, int Nf, int fc_out, int act, int x3,
                                    const float* magT, const float* fbT, int B, int F, int src_T, int G,
                                    const float* inv2, const float* unit_scale, int la, int steps, int shrink, int stages,
                                    int cluster, void* packed, float* crm, fsn_stream_t stream) {
  return sb_lstm_tc_hook(sb, H, Ns, Nf, fc_out, act, x3, magT, fbT, B, F, src_T, G, inv2, unit_scale, la, steps, shrink,
                         stages, cluster, packed, crm, nullptr, 0, 0, stream);
}

// unit-test hook (tests/test_gpu_subband_two_pass.py): the two-pass stack on the inputs of fsn_debug_sb_lstm_tc, in
// chunks of chunk_pairs pairs (0: the production chunk), with h0ws of fsn_debug_sb_lstm_tc2_ws_bytes
extern "C" size_t fsn_debug_sb_lstm_tc2_ws_bytes(int R, int steps, int H, int x3, int chunk_pairs) {
  return fsn::sb_tc_split_ws_bytes(R, steps, H, x3 != 0, chunk_pairs);
}

extern "C" int fsn_debug_sb_lstm_tc2(const fsn_seq_weights* sb, int H, int Ns, int Nf, int act, int x3, const float* magT,
                                     const float* fbT, int B, int F, int src_T, int G, const float* inv2,
                                     const float* unit_scale, int la, int steps, int stages, int chunk_pairs, void* packed,
                                     void* h0ws, float* crm, fsn_stream_t stream) {
  using namespace fsn;
  FSN_REQUIRE(stages == 0 || (stages >= 2 && stages <= tc::MAX_STAGES), FSN_ERR_UNSUPPORTED,
              "sb_lstm_tc2: ring depth %d (0, 2, 3 or 4)", stages);
  FSN_REQUIRE(sb && magT && fbT && inv2 && packed && h0ws && crm && chunk_pairs >= 0, FSN_ERR_SHAPE,
              "sb_lstm_tc2: missing buffer");
  FSN_REQUIRE(B > 0 && F > 1 && src_T > 0 && Ns >= 0 && Nf >= 0 && Ns < F && Nf < F && G >= 1, FSN_ERR_SHAPE,
              "sb_lstm_tc2: bad shape B=%d F=%d src_T=%d Ns=%d Nf=%d", B, F, src_T, Ns, Nf);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "sb_lstm_tc2: activation %d", act);
  const int g = (B > 1 && G > 1) ? G : 1;
  FSN_REQUIRE(B == 1 || B > G, FSN_ERR_SHAPE, "sb_lstm_tc2: batch size %d <= num_groups %d", B, G);
  const int Fsub = g > 1 ? F / g : F;
  FSN_REQUIRE(Fsub > 0, FSN_ERR_SHAPE, "sb_lstm_tc2: num_freqs < num_groups");
  FSN_REQUIRE(steps > 0 && steps <= src_T && la >= 0 && la < steps, FSN_ERR_SHAPE,
              "sb_lstm_tc2: steps %d / look-ahead %d for %d source frames", steps, la, src_T);
  FSN_REQUIRE(sb_tc_shape_ok(H, (2 * Ns + 1) + (2 * Nf + 1)), FSN_ERR_UNSUPPORTED,
              "sb_lstm_tc2: unsupported hidden size %d / input width %d", H, (2 * Ns + 1) + (2 * Nf + 1));
  cudaStream_t st = (cudaStream_t)stream;
  int rc = sb_tc_pack_raw(sb, H, (2 * Ns + 1) + (2 * Nf + 1), 2, packed, st, x3 != 0);
  if (rc) return rc;
  SbTcArgs a;
  memset(&a, 0, sizeof(a));
  a.packed = packed; a.magT = magT; a.fbT = fbT; a.inv2 = inv2; a.unit_scale = unit_scale; a.crm = crm;
  a.B = B; a.F = F; a.Tp = src_T; a.la = la; a.Ns = Ns; a.Nf = Nf; a.H = H; a.act = act;
  a.steps = steps; a.shrink = 1; a.x3 = x3 != 0;
  a.map = RowMap{B, F, Fsub, g};
  a.stages = stages;
  a.h0ws = h0ws; a.split_chunk = chunk_pairs;
  return sb_tc_forward(a, st);
}

// unit-test hook (tests/test_gpu_subband_two_pass_layers.py): one pass of the two-pass stack over one chunk, the launch
// sb_tc_split_forward makes for it.  Layer 0 writes the images of pairs [pair0, pair0 + pairs) to h0ws (image of the
// chunk's pair p, step t at (p steps + t) img); layer 1 reads them from h0ws as the caller left it and writes those
// pairs' rows of crm.  h0ws_bytes must cover pairs x fsn_debug_sb_lstm_tc2_ws_bytes(48, steps, H, x3, 0)
extern "C" int fsn_debug_sb_tc2_pass(const fsn_seq_weights* sb, int H, int Ns, int Nf, int act, int x3, const float* magT,
                                     const float* fbT, int B, int F, int src_T, int G, const float* inv2,
                                     const float* unit_scale, int la, int steps, int stages, int layer, int pair0,
                                     int pairs, void* packed, void* h0ws, size_t h0ws_bytes, float* crm,
                                     fsn_stream_t stream) {
  using namespace fsn;
  // every check precedes the first CUDA call
  FSN_REQUIRE(stages == 0 || (stages >= 2 && stages <= tc::MAX_STAGES), FSN_ERR_UNSUPPORTED,
              "sb_tc2_pass: ring depth %d (0, 2, 3 or 4)", stages);
  FSN_REQUIRE(layer == 0 || layer == 1, FSN_ERR_SHAPE, "sb_tc2_pass: layer %d (0 or 1)", layer);
  FSN_REQUIRE(sb && magT && fbT && inv2 && packed && crm, FSN_ERR_SHAPE, "sb_tc2_pass: missing buffer");
  FSN_REQUIRE(B > 0 && F > 1 && src_T > 0 && Ns >= 0 && Nf >= 0 && Ns < F && Nf < F && G >= 1, FSN_ERR_SHAPE,
              "sb_tc2_pass: bad shape B=%d F=%d src_T=%d Ns=%d Nf=%d", B, F, src_T, Ns, Nf);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "sb_tc2_pass: activation %d", act);
  const int g = (B > 1 && G > 1) ? G : 1;
  FSN_REQUIRE(B == 1 || B > G, FSN_ERR_SHAPE, "sb_tc2_pass: batch size %d <= num_groups %d", B, G);
  const int Fsub = g > 1 ? F / g : F;
  FSN_REQUIRE(Fsub > 0, FSN_ERR_SHAPE, "sb_tc2_pass: num_freqs < num_groups");
  FSN_REQUIRE(steps > 0 && steps <= src_T && la >= 0 && la < steps, FSN_ERR_SHAPE,
              "sb_tc2_pass: steps %d / look-ahead %d for %d source frames", steps, la, src_T);
  const int total = cdiv(B * Fsub, tc::NB2);
  FSN_REQUIRE(pair0 >= 0 && pairs > 0 && pair0 < total && pairs <= total - pair0, FSN_ERR_SHAPE,
              "sb_tc2_pass: pairs [%d, %d + %d) outside the %d pairs of %d rows", pair0, pair0, pairs, total, B * Fsub);
  FSN_REQUIRE(sb_tc_shape_ok(H, (2 * Ns + 1) + (2 * Nf + 1)), FSN_ERR_UNSUPPORTED,
              "sb_tc2_pass: unsupported hidden size %d / input width %d", H, (2 * Ns + 1) + (2 * Nf + 1));
  const size_t need = (size_t)pairs * sb_tc_split_ws_bytes(tc::NB2, steps, H, x3 != 0, 1);
  FSN_REQUIRE(h0ws && h0ws_bytes >= need, FSN_ERR_WORKSPACE, "sb_tc2_pass: h0ws of %zu bytes, %zu needed", h0ws_bytes,
              need);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = sb_tc_pack_raw(sb, H, (2 * Ns + 1) + (2 * Nf + 1), 2, packed, st, x3 != 0);
  if (rc) return rc;
  SbTcArgs a;
  memset(&a, 0, sizeof(a));
  a.packed = packed; a.magT = magT; a.fbT = fbT; a.inv2 = inv2; a.unit_scale = unit_scale; a.crm = crm;
  a.B = B; a.F = F; a.Tp = src_T; a.la = la; a.Ns = Ns; a.Nf = Nf; a.H = H; a.act = act;
  a.steps = steps; a.shrink = 1; a.x3 = x3 != 0;
  a.map = RowMap{B, F, Fsub, g};
  a.stages = stages;
  tc::SplitArgs sa;
  memset(&sa, 0, sizeof(sa));
  if ((rc = sb_tc_kargs(a, sa.k))) return rc;
  sa.k.cluster = 1;
  sa.h0ws = (uint8_t*)h0ws;
  sa.row_base = pair0 * tc::NB2;
  return x3 ? sb_split_launch<true>(sa, pairs, layer, st) : sb_split_launch<false>(sa, pairs, layer, st);
}

extern "C" int fsn_debug_sb_lstm_tc_probe(const fsn_seq_weights* sb, int H, int Ns, int Nf, int fc_out, int act, int x3,
                                          const float* magT, const float* fbT, int B, int F, int src_T, int G,
                                          const float* inv2, const float* unit_scale, int la, int steps, int shrink,
                                          int stages, int cluster, void* packed, float* crm, long long* stamps,
                                          int stamp_ctas, int stamp_steps, fsn_stream_t stream) {
  using namespace fsn;
  FSN_REQUIRE(stamps, FSN_ERR_SHAPE, "sb_lstm_tc probe: missing stamp buffer");
  return sb_lstm_tc_hook(sb, H, Ns, Nf, fc_out, act, x3, magT, fbT, B, F, src_T, G, inv2, unit_scale, la, steps, shrink,
                         stages, cluster, packed, crm, stamps, stamp_ctas, stamp_steps, stream);
}

// unit-test hook (tests/test_gpu_fsn_stream_tc.py): the carry instantiation on caller-provided inputs.  B clips of F rows
// (rows b F + f), per-(step, row) scales unit_scale [steps, B F], magT / fbT [B, src_T, F]; h / c [2, B F, H] hold the
// state entering step 0 and receive the state after store_step (-1: none); restart [B F] per row; crm [B, steps, 2F]
extern "C" int fsn_debug_sb_lstm_tc_carry(const fsn_seq_weights* sb, int H, int Ns, int Nf, int act, int x3,
                                          const float* magT, const float* fbT, int B, int F, int src_T,
                                          const float* unit_scale, int steps, const int32_t* restart, int store_step,
                                          float* h, float* c, void* packed, float* crm, fsn_stream_t stream) {
  using namespace fsn;
  FSN_REQUIRE(sb && magT && fbT && unit_scale && restart && h && c && packed && crm, FSN_ERR_SHAPE,
              "sb_carry_lstm_tc: missing buffer");
  FSN_REQUIRE(B > 0 && F > 1 && src_T > 0 && Ns >= 0 && Nf >= 0 && Ns < F && Nf < F && steps > 0 && steps <= src_T &&
                  store_step >= -1 && store_step < steps,
              FSN_ERR_SHAPE, "sb_carry_lstm_tc: bad shape B=%d F=%d src_T=%d steps=%d store_step=%d", B, F, src_T, steps,
              store_step);
  FSN_REQUIRE(act >= FSN_ACT_NONE && act <= FSN_ACT_RELU6, FSN_ERR_SHAPE, "sb_carry_lstm_tc: activation %d", act);
  FSN_REQUIRE(sb_tc_shape_ok(H, (2 * Ns + 1) + (2 * Nf + 1)), FSN_ERR_UNSUPPORTED,
              "sb_carry_lstm_tc: unsupported hidden size %d / input width %d", H, (2 * Ns + 1) + (2 * Nf + 1));
  cudaStream_t st = (cudaStream_t)stream;
  int rc = sb_tc_pack_raw(sb, H, (2 * Ns + 1) + (2 * Nf + 1), 2, packed, st, x3 != 0);
  if (rc) return rc;
  SbTcArgs a;
  memset(&a, 0, sizeof(a));
  a.packed = packed; a.magT = magT; a.fbT = fbT; a.unit_scale = unit_scale; a.crm = crm;
  a.B = B; a.F = F; a.Tp = src_T; a.Ns = Ns; a.Nf = Nf; a.H = H; a.act = act; a.steps = steps; a.x3 = x3 != 0;
  a.map = RowMap{B, F, F, 1};
  const size_t R = (size_t)B * F;
  const SbCarry io{h, c, (size_t)H, R * H, 1, restart, store_step, (size_t)steps * 2 * F, 0};
  return sb_tc_carry_forward(a, io, st);
}
