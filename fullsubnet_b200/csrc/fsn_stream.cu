// Chunked streaming (DESIGN 4.14): the per-slot bookkeeping, the causal first norm with a carried accumulator and the
// recurrent-state reset of a clip's first frame, and the host skeleton every model's step is built from (the call
// checks, the slot-state header, the workspace head and the signal front and back end).  The signal layer's streaming
// kernels are in fsn_dsp.cu; each model's sections, the middle of its step and its entry points beside its enhance call.
#include <string.h>

#include "fsn_internal.cuh"

namespace fsn {

StreamSlot::StreamSlot(const StreamGeom& g, int F) : end(sizeof(StreamMeta)) {
  hist = sec(g.Hs);
  spec = sec((size_t)g.Q * 2 * F);
  crm = sec((size_t)g.Rc * 2 * F);
}

void stream_carve(Carver& c, const StreamGeom& g, int B, int K, int F, StreamWs& w) {
  const size_t St = (size_t)K + g.E;
  w.pos0 = c.take<int>(B); w.act0 = c.take<int>(B); w.tail = c.take<int>(B);
  w.wav = c.take<float>(B * ((size_t)g.Hs + (size_t)K * g.hop));
  w.magT = c.take<float>(B * St * F);
  w.spec = c.take<float>(B * ((size_t)g.Q + St) * 2 * F);
  w.crm = c.take<float>(B * ((size_t)g.Rc + St) * 2 * F);
}

int stream_query_check(int rc, const char* who, int B, int K_max) {
  if (rc) return rc;
  FSN_REQUIRE(B > 0 && K_max > 0, FSN_ERR_SHAPE, "%s: B=%d slots, K_max=%d hops", who, B, K_max);
  return FSN_OK;
}

int stream_check(const char* who, const StreamGeom& g, int B, int K, const int32_t* tail, const float* wav,
                 const float* enhanced, int& St) {
  FSN_REQUIRE(B > 0 && K > 0, FSN_ERR_SHAPE, "%s: B=%d slots, K=%d hops", who, B, K);
  FSN_REQUIRE(B <= 65535, FSN_ERR_UNSUPPORTED, "%s: B=%d slots, at most 65535", who, B);
  FSN_REQUIRE((long long)K * g.hop + g.D < (1 << 30), FSN_ERR_SHAPE, "%s: K=%d hops too long", who, K);
  FSN_REQUIRE(wav && enhanced, FSN_ERR_SHAPE, "%s: null chunk or output", who);
  bool any_tail = false;
  for (int b = 0; tail && b < B; ++b) {
    FSN_REQUIRE(tail[b] >= -1 && tail[b] <= K * g.hop, FSN_ERR_SHAPE,
                "%s: tail[%d] = %d, outside [0, K*hop] = [0, %d] and not -1", who, b, tail[b], K * g.hop);
    any_tail |= tail[b] >= 0;
  }
  St = K + (any_tail ? g.E : 0);
  return FSN_OK;
}

int stream_check_sizes(const void* state, size_t state_bytes, size_t slot, int B, const void* workspace,
                       size_t workspace_bytes, size_t ws_need) {
  FSN_REQUIRE(state && state_bytes >= slot * (size_t)B, FSN_ERR_WORKSPACE, "stream state too small: %zu < %zu",
              state_bytes, slot * (size_t)B);
  FSN_REQUIRE(workspace && workspace_bytes >= ws_need, FSN_ERR_WORKSPACE, "workspace too small: %zu < %zu",
              workspace_bytes, ws_need);
  return FSN_OK;
}

// buffers laid out for K + E steps from the workspace's start (a workspace queried for a larger K_max also fits); a
// call without a clip's last chunk runs St = K steps and strides its buffers by St
int stream_open(const StreamGeom& g, const StreamSlot& sl, const StreamWs& w, int F, int B, int K, int St, int win_length,
                const int32_t* start, const int32_t* tail, const float* wav, char* state, int* restart, cudaStream_t st) {
  int rc;
  const size_t ss = sl.slot(), F2 = 2 * (size_t)F;
  const int Kh = K * g.hop, Wn = g.Hs + Kh;
  if ((rc = stream_prologue(start, tail, B, state, ss, w.pos0, w.act0, w.tail, st))) return rc;
  if (restart && (rc = stream_restart_launch(w.pos0, B, g, restart, st))) return rc;
  // samples: the carried history, then the chunk; spectrum: the carried Q frames, then the St frames of this call
  if ((rc = copy_rows(w.wav, (size_t)Wn * 4, state + sl.hist, ss, (size_t)g.Hs * 4, B, st))) return rc;
  if ((rc = copy_rows(w.wav + g.Hs, (size_t)Wn * 4, wav, (size_t)Kh * 4, (size_t)Kh * 4, B, st))) return rc;
  if ((rc = copy_rows(w.spec, (g.Q + St) * F2 * 4, state + sl.spec, ss, g.Q * F2 * 4, B, st))) return rc;
  return stft_stream_launch(w.wav, Wn, g.Hs, w.pos0, w.tail, B, g.n, g.hop, win_length, g.c, St, g.Q, w.magT, w.spec, st);
}

int stream_close(const StreamGeom& g, const StreamSlot& sl, const StreamWs& w, int F, int B, int K, int St, int win_length,
                 const float* y, float* enhanced, char* state, cudaStream_t st) {
  int rc;
  const size_t ss = sl.slot(), F2 = 2 * (size_t)F;
  const int Kh = K * g.hop, Wn = g.Hs + Kh;
  // cRM: the carried Rc frames, then step j's output as frame pos0/hop - c + j - la
  if ((rc = copy_rows(w.crm, (g.Rc + St) * F2 * 4, state + sl.crm, ss, g.Rc * F2 * 4, B, st))) return rc;
  if (y && (rc = copy_rows(w.crm + g.Rc * F2, (g.Rc + St) * F2 * 4, y, St * F2 * 4, St * F2 * 4, B, st))) return rc;
  if ((rc = istft_stream_launch(w.spec, w.crm, w.pos0, w.act0, w.tail, B, K, g.D, g.n, g.hop, win_length, g.c, g.la, g.Rc,
                                g.Q, St, enhanced, st)))
    return rc;
  // carry what the next call reads: the windows as of step K
  if ((rc = copy_rows(state + sl.hist, ss, w.wav + Kh, (size_t)Wn * 4, (size_t)g.Hs * 4, B, st))) return rc;
  if ((rc = copy_rows(state + sl.spec, ss, w.spec + K * F2, (g.Q + St) * F2 * 4, g.Q * F2 * 4, B, st))) return rc;
  return copy_rows(state + sl.crm, ss, w.crm + K * F2, (g.Rc + St) * F2 * 4, g.Rc * F2 * 4, B, st);
}

int stream_geom(int n_fft, int hop, int win_length, int la, StreamGeom& g) {
  int rc = stream_dsp_check(n_fft, hop, win_length);
  if (rc) return rc;
  FSN_REQUIRE(la >= 0, FSN_ERR_SHAPE, "stream: look_ahead %d", la);
  g.n = n_fft; g.hop = hop; g.la = la;
  g.c = cdiv(n_fft / 2, hop);
  g.D = n_fft / 2 + (la + 1 + g.c) * hop;
  g.Hs = (g.c + 1) * hop + n_fft / 2;
  g.Rc = cdiv(n_fft, hop) + 2;
  g.Q = g.Rc + la;
  g.E = 1 + la + g.c;
  return FSN_OK;
}

constexpr int kStreamChunk = 500;  // 4 KB parameter block with the two counts
struct StreamChunk { int off, n; int start[kStreamChunk], tail[kStreamChunk]; };

__global__ void stream_prologue_kernel(const __grid_constant__ StreamChunk c, char* __restrict__ state, size_t slot_bytes,
                                       int* __restrict__ pos0, int* __restrict__ act0, int* __restrict__ tail) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n) return;
  const int b = c.off + i;
  StreamMeta* m = reinterpret_cast<StreamMeta*>(state + (size_t)b * slot_bytes);
  if (c.start[i]) { m->pos = 0; m->active = 1; m->acc = 0.f; }
  pos0[b] = m->pos;
  act0[b] = m->active;
  tail[b] = m->active ? c.tail[i] : -1;
}

int stream_prologue(const int32_t* start, const int32_t* tail, int B, char* state, size_t slot_bytes, int* pos0, int* act0,
                    int* tail_dev, cudaStream_t st) {
  StreamChunk c;
  for (int off = 0; off < B; off += kStreamChunk) {
    c.off = off;
    c.n = B - off < kStreamChunk ? B - off : kStreamChunk;
    for (int i = 0; i < c.n; ++i) {
      c.start[i] = start ? start[off + i] != 0 : 0;
      c.tail[i] = tail ? tail[off + i] : -1;
    }
    stream_prologue_kernel<<<cdiv(c.n, 128), 128, 0, st>>>(c, state, slot_bytes, pos0, act0, tail_dev);
    FSN_CHECK_LAUNCH("stream_prologue_kernel");
  }
  return FSN_OK;
}

// the arithmetic of cum_clip_scale_kernel / forget_scale_kernel, frame m of the clip at step j: the first norm (fs2 null,
// accumulator in the meta) or fullsubnet's second forgetting norm (mean of fs.y + fs2.y, mu at acc_off)
__global__ void stream_norm_kernel(const float2* __restrict__ fs, const float2* __restrict__ fs2, int B, int S, int K, int F,
                                   int hop, int c, int fgt, const ForgetCoef cf, float eps, const int* __restrict__ pos0,
                                   const int* __restrict__ act0, const int* __restrict__ tail, char* __restrict__ state,
                                   size_t slot_bytes, size_t acc_off, float* __restrict__ scaleT) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  StreamMeta* mt = reinterpret_cast<StreamMeta*>(state + (size_t)b * slot_bytes);
  float* accp = fs2 ? reinterpret_cast<float*>(state + (size_t)b * slot_bytes + acc_off) : &mt->acc;
  const int m0 = pos0[b] / hop - c;
  float acc = *accp, acc_k = acc;
  for (int j = 0; j < S; ++j) {
    const int m = m0 + j;
    float sc = 1.f;
    if (m >= 0) {
      if (m == 0) acc = 0.f;
      const float2 v = fs[(size_t)b * S + j];
      const float s = fs2 ? __fadd_rn(v.y, fs2[(size_t)b * S + j].y) : v.x;
      if (fgt) {
        const float mean = __fdiv_rn(s, (float)F);
        const int i = m < FORGET_LEN ? m : FORGET_LEN;
        acc = __fadd_rn(__fmul_rn(cf.a[i], acc), __fmul_rn(cf.b[i], mean));
        sc = __fdiv_rn(1.0f, __fadd_rn(acc, FORGET_EPS));
      } else {
        acc += s;
        sc = 1.0f / (acc / ((float)F * (float)(m + 1)) + eps);
      }
    }
    scaleT[(size_t)j * B + b] = sc;
    if (j == K - 1) acc_k = acc;
  }
  if (act0[b]) {
    *accp = acc_k;
    if (!fs2) {
      mt->pos = pos0[b] + K * hop;
      mt->active = tail[b] < 0;
    }
  }
}

int stream_norm_launch(const float2* fs, int B, int S, int K, int F, const StreamGeom& g, int norm_type, const int* pos0,
                       const int* act0, const int* tail, char* state, size_t slot_bytes, float* scaleT, cudaStream_t st,
                       const float2* fs2, size_t acc_off) {
  stream_norm_kernel<<<cdiv(B, 64), 64, 0, st>>>(fs, fs2, B, S, K, F, g.hop, g.c, norm_type == FSN_NORM_FORGETTING,
                                                 forget_coef(), 1.1920928955078125e-07f, pos0, act0, tail, state, slot_bytes,
                                                 acc_off, scaleT);
  FSN_CHECK_LAUNCH("stream_norm_kernel");
  return FSN_OK;
}

// cum_unit_scale_kernel on the call's S steps, one thread per row r = b*F + f
__global__ void stream_cum_unit_kernel(const float* __restrict__ magT, const float* __restrict__ fbT, int B, int S, int K,
                                       int F, int Ns, int Nf, int hop, int c, float eps, const int* __restrict__ pos0,
                                       const int* __restrict__ act0, char* __restrict__ state, size_t slot_bytes,
                                       size_t run_off, float* __restrict__ scaleT) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B * F) return;
  const int b = r / F, f = r - b * F;
  const int Kf = 2 * Ns + 1 + 2 * Nf + 1;
  float* srun = reinterpret_cast<float*>(state + (size_t)b * slot_bytes + run_off) + f;
  const int m0 = pos0[b] / hop - c;
  float run = *srun, run_k = run;
  for (int j = 0; j < S; ++j) {
    const int m = m0 + j;
    float sc = 1.f;
    if (m >= 0) {
      if (m == 0) run = 0.f;
      const size_t base = ((size_t)b * S + j) * F;
      run += unit_frame_sum(magT + base, fbT + base, f, F, Ns, Nf);
      sc = 1.0f / (run / ((float)Kf * (float)(m + 1)) + eps);
    }
    scaleT[(size_t)j * B * F + r] = sc;
    if (j == K - 1) run_k = run;
  }
  if (act0[b]) *srun = run_k;
}

int stream_cum_unit_launch(const float* magT, const float* fbT, int B, int S, int K, int F, int Ns, int Nf,
                           const StreamGeom& g, const int* pos0, const int* act0, char* state, size_t slot_bytes,
                           size_t run_off, float* scaleT, cudaStream_t st) {
  stream_cum_unit_kernel<<<cdiv(B * F, 128), 128, 0, st>>>(magT, fbT, B, S, K, F, Ns, Nf, g.hop, g.c, 1.1920928955078125e-07f,
                                                           pos0, act0, state, slot_bytes, run_off, scaleT);
  FSN_CHECK_LAUNCH("stream_cum_unit_kernel");
  return FSN_OK;
}

__global__ void stream_reset_kernel(const int* __restrict__ pos0, int B, int hop, int c, int j, int H, float* __restrict__ h,
                                    size_t h_row, float* __restrict__ cs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  const int b = i / H, u = i - b * H;
  if (pos0[b] / hop - c + j != 0) return;
  h[(size_t)b * h_row + u] = 0.f;
  cs[i] = 0.f;
}

int stream_reset_launch(const int* pos0, int B, const StreamGeom& g, int j, int H, float* h, size_t h_row, float* c,
                        cudaStream_t st) {
  stream_reset_kernel<<<cdiv(B * H, 256), 256, 0, st>>>(pos0, B, g.hop, g.c, j, H, h, h_row, c);
  FSN_CHECK_LAUNCH("stream_reset_kernel");
  return FSN_OK;
}

__global__ void stream_restart_kernel(const int* __restrict__ pos0, int B, int hop, int c, int* __restrict__ restart) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) restart[b] = c - pos0[b] / hop;
}

int stream_restart_launch(const int* pos0, int B, const StreamGeom& g, int* restart, cudaStream_t st) {
  stream_restart_kernel<<<cdiv(B, 128), 128, 0, st>>>(pos0, B, g.hop, g.c, restart);
  FSN_CHECK_LAUNCH("stream_restart_kernel");
  return FSN_OK;
}

void stream_stack_carve(Carver& c, const SeqStack& s, StreamStackWs& w) {
  seq_stack_carve(c, s, w.seq);
  int Hm = 0;
  for (int l = 0; l < s.n; ++l) Hm = s.H[l] > Hm ? s.H[l] : Hm;
  // seq_stack_carve's conditions: seq_stack_forward keeps only the top layer's output of a two-layer stack off the
  // tensor cores, and the persistent kernel runs stacks of two or more LSTM layers without a per-step scale
  if (s.n == 2 && !s.tc) w.seq.hall[1] = c.take<float>((size_t)s.R * s.Tp * Hm);
  w.h = (s.n >= 2 && s.H[0] == Hm) ? w.seq.h0[0] : c.take<float>((size_t)s.R * Hm);
  w.h_fin[0] = w.h_fin[1] = w.c_fin[0] = w.c_fin[1] = nullptr;
  for (int l = 0; s.n >= 2 && !s.gru && !s.step_scale && l < 2; ++l) {
    w.h_fin[l] = c.take<float>((size_t)s.R * s.H[l]);
    w.c_fin[l] = c.take<float>((size_t)s.R * s.H[l]);
  }
}

int stream_seq_stack(const SeqStack& s, const StreamStackWs& w, const StackCarry& io, cudaStream_t st) {
  const SeqPath path = seq_stack_path(s);
  const int R = s.R, S = s.Tp, n = s.n, Ht = s.H[n - 1];
  auto hall = [&](int l) { return w.seq.hall[(n - 1 - l) & 1]; };  // as in seq_stack_forward: the top one in hall[0]
  // layer l's h / c section in slot 0's block
  auto sec = [&](size_t off, int l) {
    size_t f = 0;
    for (int i = 0; i < l; ++i) f += s.H[i];
    return io.state + off + f * 4;
  };
  int rc;
  FSN_REQUIRE(io.restart || (path != SEQ_PATH_TC && path != SEQ_PATH_PERSISTENT), FSN_ERR_UNSUPPORTED,
              "stream: the stack's path (%d) restarts inside its kernels and the stream gives no restart table", (int)path);
  if (path == SEQ_PATH_TC) {
    for (int l = 0; l < n; ++l) {
      const int K = l ? s.H[l - 1] : s.K0, Hl = s.H[l];
      float* h = (float*)sec(io.h, l);
      float* c = (float*)sec(io.c, l);
      const RecCarry carry{h, c, c, io.slot / 4, io.restart, io.K - 1};
      if ((rc = lstm_layer_tc(s.L[l], l ? hall(l - 1) : s.x, (size_t)K, K, l ? nullptr : s.scale, S,
                              (!l && s.step_scale) ? R : 0, R, S, Hl, s.x3, w.seq.tc, hall(l), st, &carry)))
        return rc;
      if ((rc = copy_rows(h, io.slot, hall(l) + (size_t)(io.K - 1) * Hl, (size_t)S * Hl * 4, (size_t)Hl * 4, R, st)))
        return rc;
    }
    return linear_tc(hall(n - 1), (size_t)Ht, Ht, s.fc_w, s.fc_b, s.O, s.act, s.out, (size_t)s.O, (size_t)R * S, s.x3,
                     w.seq.tc, st);
  }
  int l = 0;  // first layer left for the per-step loop
  if (path == SEQ_PATH_PERSISTENT) {
    // the state entering the call (zero for a clip whose frame 0 is step 0; a later frame 0 restarts inside the kernel)
    float* h_init[2] = {w.seq.h0[0], w.seq.c0};
    float* c_init[2] = {w.seq.h0[1], w.seq.c1};
    for (int i = 0; i < 2; ++i) {
      const size_t hb = (size_t)s.H[i] * 4;
      if ((rc = copy_rows(h_init[i], hb, sec(io.h, i), io.slot, hb, R, st))) return rc;
      if ((rc = copy_rows(c_init[i], hb, sec(io.c, i), io.slot, hb, R, st))) return rc;
      if ((rc = stream_reset_launch(io.pos0, R, io.g, 0, s.H[i], h_init[i], s.H[i], c_init[i], st))) return rc;
    }
    const FbState fs{{h_init[0], h_init[1]}, {c_init[0], c_init[1]}, {w.h_fin[0], w.h_fin[1]}, {w.c_fin[0], w.c_fin[1]},
                     io.restart, io.K - 1};
    if ((rc = fb_persistent_launch(s.L, s.x, s.scale, w.seq.pp, hall(1), w.seq.barrier, R, s.K0, s.H[0], s.H[1], S, st, &fs)))
      return rc;
    for (int i = 0; i < 2; ++i) {
      const size_t hb = (size_t)s.H[i] * 4;
      if ((rc = copy_rows(sec(io.h, i), io.slot, w.h_fin[i], hb, hb, R, st))) return rc;
      if ((rc = copy_rows(sec(io.c, i), io.slot, w.c_fin[i], hb, hb, R, st))) return rc;
    }
    l = 2;
  }
  for (; l < n; ++l) {
    const int Hl = s.H[l];
    float* hl = hall(l);
    const size_t hrow = (size_t)S * Hl, hb = (size_t)Hl * 4;
    char* sh = sec(io.h, l);
    char* sc = sec(io.c, l);
    if ((rc = copy_rows(w.h, hb, sh, io.slot, hb, R, st))) return rc;
    if ((rc = copy_rows(w.seq.c0, hb, sc, io.slot, hb, R, st))) return rc;
    for (int j = 0; j < S; ++j) {
      float* hp = j ? hl + (size_t)(j - 1) * Hl : w.h;
      if (j <= io.g.c && (rc = stream_reset_launch(io.pos0, R, io.g, j, Hl, hp, j ? hrow : (size_t)Hl, w.seq.c0, st)))
        return rc;
      StepParams p;
      memset(&p, 0, sizeof(p));
      p.R = R; p.H = Hl; p.first = 0; p.gru = 0;
      p.w_ih = s.L[l].w_ih; p.w_hh = s.L[l].w_hh; p.b_ih = s.L[l].b_ih; p.b_hh = s.L[l].b_hh;
      p.K0 = l ? s.H[l - 1] : s.K0;
      p.x0 = (l ? hall(l - 1) : s.x) + (size_t)j * p.K0; p.x0_row_stride = (size_t)S * p.K0;
      if (!l) p.row_scale = (s.scale && s.step_scale) ? s.scale + (size_t)j * R : s.scale;
      p.h_prev = hp; p.h_prev_stride = j ? hrow : (size_t)Hl;
      p.h_out = hl + (size_t)j * Hl; p.h_out_stride = hrow;
      p.c = w.seq.c0;
      if ((rc = lstm_step_launch(p, SEG0_DENSE, st))) return rc;
      if (j == io.K - 1) {
        if ((rc = copy_rows(sh, io.slot, p.h_out, hrow * 4, hb, R, st))) return rc;
        if ((rc = copy_rows(sc, io.slot, w.seq.c0, hb, hb, R, st))) return rc;
      }
    }
  }
  return fc_gemm_launch(hall(n - 1), s.fc_w, s.fc_b, s.out, R * S, Ht, s.O, s.act, st);
}

int copy_rows(void* dst, size_t dp, const void* src, size_t sp, size_t width, int B, cudaStream_t st) {
  return check_cuda(cudaMemcpy2DAsync(dst, dp, src, sp, width, (size_t)B, cudaMemcpyDeviceToDevice, st), "stream copy");
}

}  // namespace fsn
