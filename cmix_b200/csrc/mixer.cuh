// cmix_b200/csrc/mixer.cuh
//
// The arithmetic of the three-layer gated logistic mixer + the integer SSE stage
// (reference src/mixer/mixer.cpp:16-72, src/mixer/mixer-input.cpp,
// src/predictor.cpp:388-418,432-437, src/mixer/sse.cpp; SURVEY §8 rows a3-a7), written once
// for the bulk kernel (mixer_bulk.cuh) and the lock-step kernels (mixer_lock.cuh).
//
// Parity contract: the reference sums each dot product sequentially in fp32
// (mixer.cpp:41-43, no FMA). A tree/warp-shuffle reduction changes the rounding
// and, through the 15-bit SSE quantisation (sse.cpp:321), moves the coded
// probability by >1e-5 on a fraction of bits. So each dot product is ONE serial
// FADD chain here; the kernels find their parallelism across mixers, not inside one.
#pragma once
#include <cooperative_groups.h>

#include "exact_math.h"
#include "lstm.cuh"
#include "small_models.cuh"
#include "state.h"

namespace cmixb200 {
namespace cg = cooperative_groups;

enum {
  MIX_THREADS = 512,
  MIX_PER_CTA = 13,
  MIX_CHUNKS = 8, MIX_CHUNK4 = 64,   // a layer-0 chain in 8 chunks of 64 float4; the last also takes float4 512..518
};

// Stage the 2078 layer-0 inputs of one bit (predictor.cpp:362-387 order) with all global loads issued before
// any use (2 round trips). `lut` is the stretch table of the 12-bit codes (Tables::lut12).
template <int NT>
__device__ __forceinline__ void stage_inputs(float* x, const float* lut, const u16* ext, const float* small_x,
                                             float lstm_x, int mtid) {
  enum { PER = (N_INPUTS + NT - 1) / NT };
  u32 code[PER]; float direct[PER];
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int k = mtid + q * NT;
    code[q] = 0x10000u; direct[q] = 0.0f;
    if (k < N_INPUTS) {
      if (k < 3) direct[q] = small_x[k];
      else if (k < 3 + N_EXT) code[q] = ext ? (u32)__ldcs(&ext[k - 3]) : 0xFFFFu;
      else if (k < 2076) direct[q] = small_x[k - N_EXT];
      else if (k == 2076) direct[q] = small_x[N_SMALL];
      else direct[q] = lstm_x;
    }
  }
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int k = mtid + q * NT;
    if (k < N_INPUTS) x[k] = code[q] == 0x10000u ? direct[q] : lut[code[q] == 0xFFFFu ? 4096 : (code[q] > 4095u ? 4095u : code[q])];
  }
}

// auxiliary_context_ (predictor.cpp:388-393)
__device__ __forceinline__ u32 aux_context(const float* x) {
  float avg = 0.0f;
  avg = XM_FADD(avg, xm_logistic(x[433]));
  avg = XM_FADD(avg, xm_logistic(x[2024]));
  avg = XM_FADD(avg, xm_logistic(x[2077]));
  avg = XM_FDIV(avg, 3.0f);
  return (u32)(unsigned long long)XM_FMUL(avg, 15.0f);
}

// Mixer::GetContextData (mixer.cpp:16-36): the table entry (row + 1) of context `ctx`, whose entry read so far is
// `s` (0 = not seen yet). Rows are assigned first come first served; after 10 000 every new context shares the
// overflow row (key 0xDEADBEEF).
__device__ __forceinline__ u32 assign_row(u32* table, u32 ctx, u32 s, u32& n_assigned, const u32& n_rows) {
  if (s == 0) {
    const u32 cap = n_rows - 1;                        // = min(table_size, 10000)
    if (n_assigned < cap && n_assigned < (u32)SLOT_LIMIT) { s = ++n_assigned; table[ctx] = s; }
    else s = n_rows;
  }
  return s;
}
__device__ __forceinline__ u32 resolve_slot(MixerState& m, u32 ctx) {
  return assign_row(m.slot_table, ctx, m.slot_table[ctx], m.n_assigned, m.n_rows) - 1;
}

// Mixer::Perceive's learning rate decay*lr (mixer.cpp:58-60) of a row that has taken `rs` of the mixer's `ms` steps
// at most. mixer_step counts that step (mixer.cpp:64-66) into the row's counter `steps` and the mixer's `max_steps`,
// and sets `shrink` on every 1024th step.
__device__ __forceinline__ float mixer_rate(float decay, float lr, u64 rs, u64 ms) {
  float d = decay;
  d = (float)((double)d * (1.5 - ((1.0 * (double)rs) / (double)ms)));
  return XM_FMUL(d, lr);
}
__device__ __forceinline__ void mixer_step(u64 rs, u64 ms, u64& steps, u64& max_steps, u32& shrink) {
  const u64 ns = rs + 1;
  steps = ns;
  if (ns > ms) max_steps = ns;
  shrink = ((ns & 1023) == 0) ? 1u : 0u;
}
// The SGD coefficient `update` (mixer.cpp:60) from the rate and the mixer's output p.
__device__ __forceinline__ float sgd_coeff(float rate, float p, int bit) { return XM_FMUL(rate, XM_FSUB(xm_logistic(p), (float)bit)); }
// The SGD step of weights w (mixer.cpp:62-70): w -= u*x, then the shrink of every 1024th step.
__device__ __forceinline__ float sgd_shrink(float w) { return XM_FMUL(w, 1.0f - 3.0e-6f); }
__device__ __forceinline__ void sgd_step(float& w, float u, float x, const u32& shrink) {
  float v = XM_FSUB(w, XM_FMUL(u, x));
  if (shrink) v = sgd_shrink(v);
  w = v;
}
__device__ __forceinline__ void sgd_step4(float4& w, float u, float4 x, bool shrink) {
  float4 v = w;
  v.x = XM_FSUB(v.x, XM_FMUL(u, x.x)); v.y = XM_FSUB(v.y, XM_FMUL(u, x.y));
  v.z = XM_FSUB(v.z, XM_FMUL(u, x.z)); v.w = XM_FSUB(v.w, XM_FMUL(u, x.w));
  if (shrink) { v.x = sgd_shrink(v.x); v.y = sgd_shrink(v.y); v.z = sgd_shrink(v.z); v.w = sgd_shrink(v.w); }
  w = v;
}

__device__ __forceinline__ float clamp_stretched(const Tables& T, float p) {    // mixer-input.cpp:17-27
  if (p > T.stretch_max) p = T.stretch_max; else if (p < T.stretch_min) p = T.stretch_min;
  return p;
}

// --------------------------------------------------------- layer-0 chains --
// One chunk (float4 k0 .. k1-1, k1 - k0 >= 64) of a layer-0 mixer's serial dot product (Mixer::Mix, mixer.cpp:41-43):
// ping-pong register buffers keep 8 LDS.128 in flight under the FADD chain. chain_tail adds inputs 2076 and 2077.
__device__ __forceinline__ float chain_chunk(const float4* __restrict__ x4, const float4* __restrict__ w4, int k0, int k1, float p) {
  float4 xa[4], wa[4], xb[4], wb[4];
#define CC_LOAD(X, W, k) { _Pragma("unroll") for (int q = 0; q < 4; ++q) { X[q] = x4[(k) + q]; W[q] = w4[(k) + q]; } }
#define CC_EAT(X, W) { _Pragma("unroll") for (int q = 0; q < 4; ++q) { \
    float p0_, p1_, p2_, p3_; \
    xm_fmul2(X[q].x, X[q].y, W[q].x, W[q].y, p0_, p1_); xm_fmul2(X[q].z, X[q].w, W[q].z, W[q].w, p2_, p3_); \
    p = XM_FADD(p, p0_); p = XM_FADD(p, p1_); p = XM_FADD(p, p2_); p = XM_FADD(p, p3_); } }
  CC_LOAD(xa, wa, k0);
#pragma unroll 1
  for (int k = k0; k < k0 + 56; k += 8) {          // blocks 0..13 consumed, block 14 left in A
    CC_LOAD(xb, wb, k + 4);
    CC_EAT(xa, wa);
    CC_LOAD(xa, wa, k + 8);
    CC_EAT(xb, wb);
  }
  CC_LOAD(xb, wb, k0 + 60);
  CC_EAT(xa, wa);
  CC_EAT(xb, wb);
#undef CC_LOAD
#undef CC_EAT
#pragma unroll 1
  for (int k = k0 + 64; k < k1; ++k) {              // only the last chunk: float4 512..518
    const float4 a = x4[k], b = w4[k];
    p = XM_FADD(p, XM_FMUL(a.x, b.x)); p = XM_FADD(p, XM_FMUL(a.y, b.y));
    p = XM_FADD(p, XM_FMUL(a.z, b.z)); p = XM_FADD(p, XM_FMUL(a.w, b.w));
  }
  return p;
}
__device__ __forceinline__ int chain_chunk_end(int c) { return c == MIX_CHUNKS - 1 ? 519 : (c + 1) * MIX_CHUNK4; }
__device__ __forceinline__ float chain_tail(const float* x, const float* row, float p) {
  p = XM_FADD(p, XM_FMUL(x[2076], row[2076]));
  p = XM_FADD(p, XM_FMUL(x[2077], row[2077]));
  return p;
}

// ------------------------------------------------------ layers 0-2, one warp --
// Forward substitution through the extra inputs of mixers 0..N-1 of one layer (mixer.cpp:45-53), lane i = mixer i:
// `main` is the lane's main dot product and `we` its extra-input weights. Lane k stores the clamped output of mixer k
// to out_a[k] and out_b[k]; every lane returns its own mixer's output before clamping.
template <int N>
__device__ __forceinline__ float substitute(float main, const float* we, const Tables& T, float* out_a, float* out_b, int lane) {
  float e = 0.0f, pfin = 0.0f;
  float wnext = lane < N ? we[0] : 0.0f;
#pragma unroll 1
  for (int k = 0; k < N; ++k) {
    if (lane == k) pfin = XM_FADD(main, e);
    const float pk = __shfl_sync(0xffffffffu, pfin, k);
    const float ck = clamp_stretched(T, pk);
    const float wk = wnext;
    if (lane < N && k + 1 < N) wnext = we[k + 1];
    if (lane == k) { out_a[k] = ck; out_b[k] = ck; }
    if (lane > k && lane < N) e = XM_FADD(e, XM_FMUL(ck, wk));
  }
  return pfin;
}
// The layer-2 row is kept as row 20 of the layer-1 rows (both kernels index it with ROW_PITCH_L1).
static_assert(ROW_PITCH_L1 == ROW_PITCH_L2, "layer-2 rows are stored with the layer-1 row pitch");
// Layer 1 on lanes 0..19 from its 29 inputs `in1` and row w = rows[lane] (inputs, then extra weights); the clamped
// outputs go to l1extra and to layer 2's inputs in2[26..45].
__device__ __forceinline__ float layer1_forward(const float* w, const float* in1, float* l1extra, float* in2, const Tables& T, int lane) {
  float main = 0.0f;
  if (lane < N_L1) {
#pragma unroll 4
    for (int k = 0; k < L1_IN; ++k) main = XM_FADD(main, XM_FMUL(in1[k], w[k]));
  }
  return substitute<N_L1>(main, w + L1_IN, T, l1extra, in2 + N_L0, lane);
}
// Layer 2 (one mixer, no extra inputs: p_ += 0).
__device__ __forceinline__ float layer2_forward(const float* w, const float* in2) {
  float s = 0.0f;
#pragma unroll 7
  for (int k = 0; k < L2_IN; ++k) s = XM_FADD(s, XM_FMUL(in2[k], w[k]));
  return XM_FADD(s, 0.0f);
}

// ------------------------------------------------------------------ SSE ----
__device__ __forceinline__ int sse_extrap(int p1, int C) {
  p1 = (((p1 - 16384) * C) >> 13) + 16384;
  if (p1 < 1) p1 = 1;
  if (p1 > 32767) p1 = 32767;
  return p1;
}
__device__ __forceinline__ int sse_rdiv(int x, int a, int d) { return x >= 0 ? (x + a) >> d : -((-x + a) >> d); }
__device__ __forceinline__ int sse_mixup(int w, int s1, int s0) {
  int x = s1 + sse_rdiv((w - 16384) * (s0 - s1), 1 << 14, 15);
  return (x > 0) ? (x < 32768) ? x : 32767 : 1;
}
__device__ __forceinline__ int sse_mask1(int j) {   // M_mx1mask0 (sse.cpp:190)
  if (j < 2) return 0;
  if (j <= 32) return j - 1;
  if (j <= 63) return 31 + (j - 32) / 2;
  if (j <= 127) return 47 + (j - 64) / 4;
  return 63 + (j - 128) / 8;
}
__device__ __forceinline__ int sse_pred(const u16* bucket, int iP, int* sw, int* q, int* P) {
  *q = (6 * iP) >> 15;
  *sw = (6 * iP) & 32767;
  int f = (((32768 - *sw) * (int)bucket[*q] + *sw * (int)bucket[*q + 1]) >> 15) - 8192;
  if (f <= 0) f = 1;
  if (f >= 32768) f = 32767;
  *P = f;
  return f;
}
__device__ __forceinline__ void sse_bucket_update(u16* bucket, int c, int wr0, int sw, int q, int P) {
  P = P * (32768 - wr0) >> 15;
  if (c == 0) P += wr0;
  const int dC = (int)bucket[q] - (int)bucket[q + 1];
  const int sw_dC = (sw * dC + 32767) >> 15;
  bucket[q] = (u16)(P + sw_dC + 8192);
  bucket[q + 1] = (u16)(P - (dC - sw_dC) + 8192);
}
__device__ __forceinline__ void sse_mix_update(int* w, int y, int p0, int p1, int wq, int pm) {
  const int py = 32768 - (y << 15);
  const int e = py - pm;
  int d = sse_rdiv(e * (p0 - p1), 1 << 14, 15);
  d = sse_rdiv(d * wq, 1 << 14, 15);
  *w += d;
}
// The SSE stage's input quantisation (sse.cpp:320-321, 250-258): returns the 15-bit probability and its two coarse
// levels q3 (0..2) and q4 (0..3).
__device__ __forceinline__ int sse_quantise(float pin, int& q3, int& q4) {
  const int discrete = (int)XM_FADD(1.0f, XM_FMUL(XM_FSUB(1.0f, pin), 32766.0f));
  const u32 prq = (u32)discrete >> 11;
  q3 = (prq > 0) + (prq > 14); q4 = (prq > 0) + (prq > 7) + (prq > 14);
  return discrete;
}
// The four contexts (sse.cpp:259-270) of coarse level q in byte context (j, pc, ffl): bucket sets s6/s7, weights x2/x1.
__device__ __forceinline__ size_t sse_i6(int q, u32 j, u32 pc, u32 ffl) { return (((((size_t)q << 7) + (ffl & 127)) << 8) + (pc & 255)) * 256 + j; }
__device__ __forceinline__ size_t sse_i7(int q, u32 j, u32 pc, u32 ffl) { return (((((size_t)q << 5) + (ffl & 31)) << 8) + (pc & 255)) * 255 + (j < 2 ? 0 : j - 1); }
__device__ __forceinline__ size_t sse_ix2(int q, u32 j, u32 pc, u32 ffl) { return (((((size_t)q << 1) + (ffl & 1)) << 8) + (pc & 255)) * 256 + j; }
__device__ __forceinline__ size_t sse_ix1(int q, u32 j, u32 pc, u32 ffl) { return (((((size_t)q << 8) + (ffl & 255)) << 3) + ((pc >> 5) & 7)) * 79 + sse_mask1((int)j); }
// SSE::Predict (M_Estimate, sse.cpp:243-289) from the selected bucket sets k6/k7 and mixer weights wx1/wx2; fills c
// with what sse_learn needs.
__device__ __forceinline__ float sse_estimate(SseCarry& c, const u16* __restrict__ st, const u16* __restrict__ sq, int discrete,
                                              const u16* k6, const u16* k7, int wx1, int wx2) {
  const int stp = __ldg(&st[discrete]);
  const int p1 = sse_pred(k6, __ldg(&sq[sse_extrap(stp, 10240)]), &c.sw6, &c.q6, &c.P6);
  c.s0 = sse_extrap(stp, 7935);
  c.s1 = sse_extrap(__ldg(&st[p1]), 9592);
  c.sm = sse_mixup(wx1, c.s0, c.s1);
  c.sm = sse_extrap(c.sm, 8092);
  c.mix1_p = __ldg(&sq[c.sm]);
  const int p2 = sse_pred(k7, __ldg(&sq[sse_extrap(stp, 8200)]), &c.sw7, &c.q7, &c.P7);
  c.s4 = sse_extrap(__ldg(&st[p2]), 7677);
  int s5 = sse_mixup(wx2, c.sm, c.s4);
  s5 = sse_extrap(s5, 8202);
  c.mix2_p = __ldg(&sq[s5]);
  return (float)(1.0 - ((double)(c.mix2_p - 1) / 32766.0));
}
// SSE::Perceive (M_Update, sse.cpp:291-299) on the bucket sets and weights the estimate used.
__device__ __forceinline__ void sse_learn(const SseCarry& c, int bit, u16* k6, u16* k7, int* wx1, int* wx2) {
  sse_bucket_update(k6, bit, 106, c.sw6, c.q6, c.P6);
  sse_mix_update(wx1, bit, c.s0, c.s1, 6202, c.mix1_p);
  sse_bucket_update(k7, bit, 127, c.sw7, c.q7, c.P7);
  sse_mix_update(wx2, bit, c.sm, c.s4, 8320, c.mix2_p);
}
// The SSE stage's byte context after coding `bit` (sse.cpp:300-305).
__device__ __forceinline__ void sse_advance(u32& j, u32& pc, u32& ffl, int bit) {
  u32 sj = j, spc = pc, sffl = ffl;
  sj += sj + bit;
  if (sj >= 256) { sffl = (u8)(sffl * 2 + (spc >= 0x40)); spc = (u8)sj; sj = 1; }
  j = sj; pc = spc; ffl = sffl;
}

}  // namespace cmixb200
