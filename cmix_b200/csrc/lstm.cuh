// cmix_b200/csrc/lstm.cuh
//
// Kernel "lstm": the byte-level LSTM mixer (reference src/mixer/lstm.cpp,
// src/mixer/lstm-layer.cpp, src/mixer/byte-mixer.cpp; SURVEY §8 rows a9-a12,
// Appendix E). 2 layers x 200 cells, 3 gates with RMS-norm, truncated BPTT over
// 100 bytes, Adam.
//
// Parity contract: every floating-point result is bit-identical to the strict-FP
// reference. That fixes the ORDER of every sum (the reference's scalar loops and
// libstdc++'s valarray reductions: valarray::sum() front-to-back, _Expr::sum()
// back-to-front), so parallelism comes only from independent chains: 600 gate
// rows per layer in the forward pass, 200 columns in the transposed mat-vecs and
// ~1M independent weight elements in the weight-gradient accumulation, which is
// restructured from "100 rank-1 updates" into one pass where each thread owns one
// weight and adds its 100 terms in the reference's time order (99 -> 0).
// Tensor cores are deliberately not used: wgmma rounds fp32 operands to
// TF32/BF16 and accumulate in an unspecified order; either breaks bit-exactness
// (DESIGN.md §6).
//
// Layout: one thread-block CLUSTER of 8 CTAs per stream. CTA c owns cells
// [25c, 25c+25) of every gate of both layers, and rows [32c, 32c+32) of the
// softmax layer. Weights are stored cell-block-major ([cta][column][25 cells]) so
// that a CTA's slice is one contiguous range that it stages into shared memory
// with cp.async (all 512 threads, L1-bypassing) before its 75 serial chains run
// out of shared memory. Vectors every CTA needs in full (gate pre-activations for
// the RMS norm, hidden state, gate errors, softmax logits) are all-gathered with
// distributed-shared-memory stores + one cluster barrier.
#pragma once
#include <cooperative_groups.h>

#include "exact_math.h"
#include "jitter.cuh"
#include "small_models.cuh"
#include "state.h"

namespace cmixb200 {
namespace cgl = cooperative_groups;

enum { LSTM_THREADS = 512, LSTM_CTAS = 8, LCPC = 25 /* cells per CTA */, LSTM_POOL_FLOATS = 52224 /* 204 KB */ };
#define LC LSTM_CELLS
#define LH LSTM_HORIZON

// Weight layout (per gate): [8 cell blocks][padded column][25 cells]. Columns: the V one-hot columns,
// padded to a multiple of 4, then the dense columns (input vector), padded to a multiple of 4 - so the
// dense slice of a cell block starts on a 16-byte boundary and is a whole number of 16-byte units.
__host__ __device__ __forceinline__ int lstm_vp(int V) { return (V + 3) & ~3; }
__host__ __device__ __forceinline__ int lstm_rowp(int V, int in_size) { return lstm_vp(V) + ((in_size + 3) & ~3); }
__host__ __device__ __forceinline__ size_t lstm_widx(int V, int in_size, int col, int cell) {
  const int pc = col < V ? col : lstm_vp(V) + (col - V);
  return ((size_t)(cell / LCPC) * lstm_rowp(V, in_size) + pc) * LCPC + (cell % LCPC);
}

// Pointers and hot scalars of LstmState, copied into shared memory once per kernel: every
// `state->array[...]` through HBM costs a dependent ~1 us load, and cluster barriers invalidate L1.
struct LstmPtrs {
  float* w[2][3]; float* m[2][3]; float* v[2][3]; float* state[2][3]; float* norm[2][3]; float* err[2][3]; float* ivar[2][3];
  float* tanh_state[2]; float* igs[2]; float* last_state[2]; float* input[2];
  float* out_w; float* output; const float* adam;
  int in_size[2]; int lepoch[2]; int epoch; int V;
  unsigned long long update_steps[2];
};

struct LstmShared {
  LstmPtrs P;
  float gam[2][3][LCPC], bet[2][3][LCPC];   // own cells: RMS-norm gain / bias
  float cst[2][LCPC];                        // own cells: cell state
  unsigned hist[LH];                         // Lstm::input_history_
  int bmap[256]; unsigned char vocab[256];
  float probs256[256];                       // byte-indexed distribution for the bit read-outs
  alignas(16) float in[2 * 256 + 2 * LC + 8];   // current layer input vector
  float gat[3][LC];                  // all-gathered per-gate vector (pre-activations / scaled errors)
  alignas(16) float gat2[3][LC];     // all-gathered final gate errors
  alignas(16) float prod[3][LC];     // element-wise products feeding the serial RMS-norm sums
  alignas(16) float hid[LSTM_HID + 3];   // full hidden vector (all-gathered)
  float act[3][LCPC];                // own cells: gate activations
  float eown[3][LCPC];               // own cells: gate errors
  float nown[3][LCPC];               // own cells: norm values of the step
  float logits[256];                 // all-gathered softmax logits / exps
  float err[256];
  float scal[16];
  int sym[LH];
  alignas(16) float pool[LSTM_POOL_FLOATS];
};

static_assert(sizeof(LstmShared) <= 232448, "LstmShared must fit the 227 KB of shared memory a CTA can opt into");

#define L_PROF(slot) do { if (prof) { unsigned d_ = *reinterpret_cast<volatile unsigned*>(&sh.sym[0]), k_; \
    asm volatile("mov.u32 %0, %1;" : "=r"(k_) : "r"(d_)); const long long n_ = clock64(); prof[32 + (slot)] += (unsigned long long)(n_ - *tprev) + (k_ & 0u); *tprev = n_; } } while (0)

__device__ __noinline__ float lt_tanhf(float x) { return xm_tanhf(x); }
__device__ __noinline__ float lt_logistic(float x) { return xm_logistic(x); }
__device__ __noinline__ float lt_expf(float x) { return xm_expf(x); }

// s = p[n-1] + p[n-2] + ... + p[0], one FADD chain (libstdc++ _Expr::sum() order); n % 4 == 0, p 16-byte aligned
__device__ __forceinline__ float sum_back_to_front(const float* p, int n) {
  const float4* p4 = reinterpret_cast<const float4*>(p);
  float4 v = p4[n / 4 - 1];
  float s = v.w;
  s = XM_FADD(s, v.z); s = XM_FADD(s, v.y); s = XM_FADD(s, v.x);
#pragma unroll 4
  for (int q = n / 4 - 2; q >= 0; --q) {
    v = p4[q];
    s = XM_FADD(s, v.w); s = XM_FADD(s, v.z); s = XM_FADD(s, v.y); s = XM_FADD(s, v.x);
  }
  return s;
}

// f += sum_j a[j] * w[j * stride], j = 0..n-1 in order: one FADD chain; the products come two at a time (xm_fmul2),
// the broadcast operand as LDS.128. a must be 16-byte aligned.
__device__ __forceinline__ float chain_strided(float f, const float* a, const float* w, int n, int stride) {
  const float4* a4 = reinterpret_cast<const float4*>(a);
  const int n4 = n >> 2;
#pragma unroll 4
  for (int q = 0; q < n4; ++q) {
    const float4 v = a4[q];
    const float* wq = w + (size_t)(4 * q) * stride;
    float p0, p1, p2, p3;
    xm_fmul2(v.x, v.y, wq[0], wq[stride], p0, p1);
    xm_fmul2(v.z, v.w, wq[2 * stride], wq[3 * stride], p2, p3);
    f = XM_FADD(f, p0); f = XM_FADD(f, p1); f = XM_FADD(f, p2); f = XM_FADD(f, p3);
  }
  for (int j = 4 * n4; j < n; ++j) f = XM_FADD(f, XM_FMUL(a[j], w[(size_t)j * stride]));
  return f;
}

__device__ __forceinline__ float clipf(float v, float c) { return v < -c ? -c : (v > c ? c : v); }

__device__ __forceinline__ void lcp_async16(void* smem_dst, const void* gmem_src) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void lcp_async4(void* smem_dst, const void* gmem_src) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void lcp_async_wait() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// all-gather: value of (gate g, own cell i) from every CTA into dst[g][25*rank + i] of every CTA
__device__ __forceinline__ void gather75(cgl::cluster_group& cluster, float (*dst)[LC], int rank, int tid, float v) {
  if (tid < 3 * LCPC) {
    const int g = tid / LCPC, i = tid % LCPC;
#pragma unroll 1
    for (int c = 0; c < LSTM_CTAS; ++c) {
      float (*rd)[LC] = cluster.map_shared_rank(dst, c);
      rd[g][LCPC * rank + i] = v;
    }
  }
}

// LstmLayer::ForwardPass (lstm-layer.cpp:62-99) for one layer; the whole cluster.
__device__ void lstm_layer_forward(cgl::cluster_group& cluster, LstmState& S, int l, int sym, LstmShared& sh, int rank, int tid,
                                   unsigned long long* prof, long long* tprev) {
  LstmPtrs& P = sh.P;
  const int V = P.V, e = P.lepoch[l], in_size = P.in_size[l];
  const float* in_g = P.input[l] + (size_t)e * in_size;
  // ---- stage: input vector + this CTA's weight slice (dense columns, then the symbol column) ----
  for (int j = tid; j < in_size; j += LSTM_THREADS) sh.in[j] = in_g[j];
  const int in_sizep = (in_size + 3) & ~3, rowp = lstm_rowp(V, in_size), gstride = (in_sizep + 4) * LCPC;
  for (int g = 0; g < 3; ++g) {
    const float* src = P.w[l][g] + ((size_t)rank * rowp + lstm_vp(V)) * LCPC;     // dense columns, 16-byte aligned
    float* dst = sh.pool + (size_t)g * gstride;
    const int n16 = in_sizep * LCPC / 4;
    for (int k = tid; k < n16; k += LSTM_THREADS) lcp_async16(dst + 4 * k, src + 4 * k);
    const float* ssrc = P.w[l][g] + ((size_t)rank * rowp + sym) * LCPC;           // one-hot column `sym`
    if (tid < LCPC) lcp_async4(dst + in_sizep * LCPC + tid, ssrc + tid);
  }
  lcp_async_wait();
  JIT_SYNCTHREADS();
  L_PROF(4);
  // ---- 75 serial chains out of shared memory ----
  float f = 0.0f;
  if (tid < 96 && (tid & 31) < LCPC) {
    const int g = tid >> 5, i = tid & 31;
    const float* w = sh.pool + (size_t)g * gstride + i;
    f = chain_strided(w[(size_t)in_sizep * LCPC], sh.in, w, in_size, LCPC);
#pragma unroll 1
    for (int c = 0; c < LSTM_CTAS; ++c) {
      float (*rd)[LC] = cluster.map_shared_rank(sh.gat, c);
      rd[g][LCPC * rank + i] = f;
    }
  }
  L_PROF(5);
  jit_cluster_sync(cluster, JIT_HERE);
  L_PROF(7);
  // ---- RMS norm: every CTA computes the three sums redundantly (back to front, _Expr::sum()):
  //      squares in parallel, then one FADD chain per gate ----
  for (int k = tid; k < 3 * LC; k += LSTM_THREADS) { const float v = sh.gat[k / LC][k % LC]; sh.prod[k / LC][k % LC] = XM_FMUL(v, v); }
  JIT_SYNCTHREADS();
  if (tid < 96 && (tid & 31) == 0) {
    const int g = tid >> 5;
    const float ss = sum_back_to_front(sh.prod[g], LC);
    const float iv = XM_FDIV(1.0f, __fsqrt_rn(XM_FADD(XM_FDIV(ss, (float)LC), 1e-5f)));
    sh.scal[g] = iv;
    if (rank == 0) P.ivar[l][g][e] = iv;
  }
  JIT_SYNCTHREADS();
  L_PROF(9);
  if (tid < 96 && (tid & 31) < LCPC) {
    const int g = tid >> 5, i = tid & 31, cell = LCPC * rank + i;
    const float n = XM_FMUL(sh.gat[g][cell], sh.scal[g]);
    P.norm[l][g][(size_t)e * LC + cell] = n;
    float s = XM_FADD(XM_FMUL(n, sh.gam[l][g][i]), sh.bet[l][g][i]);
    s = (g == 1) ? lt_tanhf(s) : lt_logistic(s);
    P.state[l][g][(size_t)e * LC + cell] = s;
    sh.act[g][i] = s;
  }
  JIT_SYNCTHREADS();
  L_PROF(10);
  if (tid < LCPC) {
    const int i = tid, cell = LCPC * rank + i;
    const float fs = sh.act[0][i], gs = sh.act[1][i], os = sh.act[2][i];
    float c = sh.cst[l][i];
    P.last_state[l][(size_t)e * LC + cell] = c;
    const float ig = XM_FSUB(1.0f, fs);
    P.igs[l][(size_t)e * LC + cell] = ig;
    c = XM_FMUL(c, fs);
    c = XM_FADD(c, XM_FMUL(gs, ig));
    sh.cst[l][i] = c;
    const float ts = lt_tanhf(c);
    P.tanh_state[l][(size_t)e * LC + cell] = ts;
    const float h = XM_FMUL(os, ts);
#pragma unroll 1
    for (int cc = 0; cc < LSTM_CTAS; ++cc) {
      float* rh = cluster.map_shared_rank(sh.hid, cc);
      rh[l * LC + cell] = h;
    }
  }
  JIT_SYNCTHREADS();
  if (tid == 0) P.lepoch[l] = (e + 1 == LH) ? 0 : e + 1;
  L_PROF(8);
  jit_cluster_sync(cluster, JIT_HERE);
  L_PROF(7);
}

// Lstm::Predict (lstm.cpp:120-150)
__device__ void lstm_predict(cgl::cluster_group& cluster, LstmState& S, unsigned input, LstmShared& sh, int rank, int tid,
                             unsigned long long* prof, long long* tprev) {
  LstmPtrs& P = sh.P;
  const int V = P.V, e = P.epoch, HW = LSTM_HID;
  for (int l = 0; l < 2; ++l) {
    float* in = P.input[l] + (size_t)P.lepoch[l] * P.in_size[l];
    // own h(t-1) into [V, V+200); layer 1 also gets layer 0's new h into [V+200, V+400)
    if (rank == 0) {
      if (tid < LC) in[V + tid] = sh.hid[l * LC + tid];
      if (l == 1 && tid >= 256 && tid < 256 + LC) in[V + LC + (tid - 256)] = sh.hid[tid - 256];
    }
    __threadfence();
    jit_cluster_sync(cluster, JIT_HERE);
    L_PROF(7);
    lstm_layer_forward(cluster, S, l, (int)input, sh, rank, tid, prof, tprev);
  }
  // ---- softmax layer: this CTA's rows of W_o[e] from HBM/L2 into shared memory, then 32 chains ----
  const int rpc = (V + LSTM_CTAS - 1) / LSTM_CTAS;                  // rows per CTA
  const int r0 = rank * rpc, r1 = min(V, r0 + rpc);
  const float* W = P.out_w + (size_t)e * V * HW;
  const int nrow = max(0, r1 - r0);
  for (int k = tid; k < nrow * HW; k += LSTM_THREADS) lcp_async4(sh.pool + k, W + (size_t)r0 * HW + k);
  lcp_async_wait();
  JIT_SYNCTHREADS();
  if (tid < nrow) {
    const float* wr = sh.pool + (size_t)tid * HW;
    const float sum = chain_strided(0.0f, sh.hid, wr, HW, 1);
#pragma unroll 1
    for (int c = 0; c < LSTM_CTAS; ++c) { float* rl = cluster.map_shared_rank(sh.logits, c); rl[r0 + tid] = sum; }
  }
  jit_cluster_sync(cluster, JIT_HERE);
  // every CTA: max(0, max_i), exp, front-to-back total, divide (identical results everywhere)
  float mx = 0.0f;
  for (int i = tid; i < V; i += LSTM_THREADS) mx = fmaxf(mx, sh.logits[i]);
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((tid & 31) == 0) sh.err[tid >> 5] = mx;
  JIT_SYNCTHREADS();
  if (tid == 0) { float m2 = 0.0f; for (int w = 0; w < LSTM_THREADS / 32; ++w) m2 = fmaxf(m2, sh.err[w]); sh.scal[4] = m2; }
  JIT_SYNCTHREADS();
  const float max_out = sh.scal[4];
  for (int i = tid; i < V; i += LSTM_THREADS) sh.logits[i] = lt_expf(XM_FSUB(sh.logits[i], max_out));
  JIT_SYNCTHREADS();
  if (tid == 0) {
    float total = sh.logits[0];
#pragma unroll 8
    for (int i = 1; i < V; ++i) total = XM_FADD(total, sh.logits[i]);
    sh.scal[5] = total;
  }
  JIT_SYNCTHREADS();
  for (int i = tid; i < V; i += LSTM_THREADS) {
    const float o = XM_FDIV(sh.logits[i], sh.scal[5]);
    sh.logits[i] = o;
    if (rank == 0) P.output[(size_t)e * V + i] = o;
  }
  JIT_SYNCTHREADS();
  if (tid == 0) P.epoch = (e + 1 == LH) ? 0 : e + 1;
  __threadfence();
  jit_cluster_sync(cluster, JIT_HERE);
  L_PROF(6);
}

// One (epoch, layer) step of the error recursion (LstmLayer::BackwardPass, lstm-layer.cpp:108-197)
// WITHOUT the weight-gradient accumulation and Adam (lstm_apply_updates does those afterwards).
// `rec` = this CTA's slice of the recurrent weight blocks, staged once per BPTT:
//   rec[((g*ntypes + type)*LC + j)*LCPC + i] = W_g(cell j, column 2V + type*200 + (25*rank + i)), ntypes = l + 1
__device__ void lstm_layer_backward(cgl::cluster_group& cluster, LstmState& S, int l, int ep, LstmShared& sh, const float* rec,
                                    int rank, int tid, float* gamma_u, float* beta_u, float* he_reg, float* stored_reg, float* se_reg) {
  LstmPtrs& P = sh.P;
  const float kClip = 10.0f;
  float he = 0.0f, stored = 0.0f, se = 0.0f;
  if (tid < LCPC) {
    const int i = tid, cell = LCPC * rank + i;
    const size_t o = (size_t)ep * LC + cell;
    const float ts = P.tanh_state[l][o], os = P.state[l][2][o], gs = P.state[l][1][o], fs = P.state[l][0][o];
    const float ig = P.igs[l][o], ls = P.last_state[l][o];
    he = *he_reg;
    if (ep == LH - 1) { stored = he; se = 0.0f; }
    else { stored = XM_FADD(*stored_reg, he); se = *se_reg; }
    sh.eown[2][i] = XM_FMUL(XM_FMUL(XM_FMUL(ts, stored), os), XM_FSUB(1.0f, os));
    se = XM_FADD(se, XM_FMUL(XM_FMUL(stored, os), XM_FSUB(1.0f, XM_FMUL(ts, ts))));
    sh.eown[1][i] = XM_FMUL(XM_FMUL(se, ig), XM_FSUB(1.0f, XM_FMUL(gs, gs)));
    sh.eown[0][i] = XM_FMUL(XM_FMUL(XM_FMUL(XM_FSUB(ls, gs), se), fs), ig);
    he = 0.0f;
    if (ep > 0) { se = XM_FMUL(se, fs); stored = 0.0f; }
  }
  if (tid == 0 && ep == 0) { if (P.update_steps[l] < 3000) ++P.update_steps[l]; }
  JIT_SYNCTHREADS();
  // per gate: beta_u/gamma_u accumulation, scale by gamma*ivar, all-gather for the RMS-norm backward sum
  float escaled = 0.0f;
  if (tid < 96 && (tid & 31) < LCPC) {
    const int g = tid >> 5, i = tid & 31, cell = LCPC * rank + i;
    const float n = P.norm[l][g][(size_t)ep * LC + cell];
    float e = sh.eown[g][i];
    if (ep == LH - 1) { *gamma_u = 0.0f; *beta_u = 0.0f; }
    *beta_u = XM_FADD(*beta_u, e);
    *gamma_u = XM_FADD(*gamma_u, XM_FMUL(e, n));
    escaled = XM_FMUL(e, XM_FMUL(sh.gam[l][g][i], P.ivar[l][g][ep]));
    sh.nown[g][i] = n;
#pragma unroll 1
    for (int c = 0; c < LSTM_CTAS; ++c) {
      float (*rd)[LC] = cluster.map_shared_rank(sh.gat, c);
      rd[g][cell] = escaled;
    }
  }
  // the full norm vector of this step straight from HBM/L2 into registers while the all-gather lands
  float nv[2] = {0.0f, 0.0f};
  for (int k = tid, q = 0; k < 3 * LC; k += LSTM_THREADS, ++q) nv[q] = P.norm[l][k / LC][(size_t)ep * LC + (k % LC)];
  jit_cluster_sync(cluster, JIT_HERE);
  for (int k = tid, q = 0; k < 3 * LC; k += LSTM_THREADS, ++q) sh.prod[k / LC][k % LC] = XM_FMUL(sh.gat[k / LC][k % LC], nv[q]);
  JIT_SYNCTHREADS();
  if (tid < 96 && (tid & 31) == 0) {
    const int g = tid >> 5;
    sh.scal[g] = XM_FDIV(sum_back_to_front(sh.prod[g], LC), (float)LC);
  }
  JIT_SYNCTHREADS();
  // no second cluster barrier: the sums read gat/prod only, and gat2 (written next, remotely) is not read again
  // before the barrier below; gat itself is next overwritten after that barrier.
  if (tid < 96 && (tid & 31) < LCPC) {
    const int g = tid >> 5, i = tid & 31, cell = LCPC * rank + i;
    const float e = XM_FSUB(escaled, XM_FMUL(sh.scal[g], sh.nown[g][i]));
    P.err[l][g][(size_t)ep * LC + cell] = e;         // final gate error of this step
#pragma unroll 1
    for (int c = 0; c < LSTM_CTAS; ++c) {
      float (*rd)[LC] = cluster.map_shared_rank(sh.gat2, c);
      rd[g][cell] = e;
    }
  }
  jit_cluster_sync(cluster, JIT_HERE);
  // transposed mat-vecs for the own 25 columns: hidden_error (layer below) and stored_error (previous step)
  float f1 = 0.0f, f2 = 0.0f;
  if (tid < 192 && (tid & 31) < LCPC) {
    const int wv = tid >> 5, g = wv >> 1, type = wv & 1, i = tid & 31;    // 6 warps: (gate, type)
    const bool need = type == 1 ? (l > 0) : (ep > 0);
    if (need) {
      const int ntypes = l + 1;
      const float* w = rec + ((size_t)(g * ntypes + type) * LC) * LCPC + i;
      const float f = chain_strided(0.0f, sh.gat2[g], w, LC, LCPC);
      sh.pool[LSTM_POOL_FLOATS - 256 + wv * 32 + i] = f;
    } else {
      sh.pool[LSTM_POOL_FLOATS - 256 + wv * 32 + i] = 0.0f;
    }
  }
  JIT_SYNCTHREADS();
  if (tid < LCPC) {
    const int i = tid;
    const float* sc = sh.pool + LSTM_POOL_FLOATS - 256;
    if (l > 0) { f1 = sc[1 * 32 + i]; he = XM_FADD(he, f1); f1 = sc[3 * 32 + i]; he = XM_FADD(he, f1); f1 = sc[5 * 32 + i]; he = XM_FADD(he, f1); }
    if (ep > 0) { f2 = sc[0 * 32 + i]; stored = XM_FADD(stored, f2); f2 = sc[2 * 32 + i]; stored = XM_FADD(stored, f2); f2 = sc[4 * 32 + i]; stored = XM_FADD(stored, f2); }
    *se_reg = clipf(se, kClip);
    *stored_reg = clipf(stored, kClip);
    *he_reg = clipf(he, kClip);
  }
  JIT_SYNCTHREADS();
}

// Weight-gradient accumulation in the reference's time order + Adam (lstm-layer.cpp:11-32,182-196).
// Each CTA owns its 25 cells: gate errors of all 100 steps in shared memory, inputs tiled by column.
__device__ void lstm_apply_updates(LstmState& S, LstmShared& sh, int rank, int tid, const float* gamma_u, const float* beta_u) {
  LstmPtrs& P = sh.P;
  const int V = P.V;
  const float beta1 = 0.025f, beta2 = 0.9999f, eps = 1e-6f;
  enum { TILE = 128 };
  float* err_s = sh.pool;                         // [3][LH][LCPC]
  float* in_t = sh.pool + 3 * LH * LCPC;          // [LH][TILE]
  for (int l = 0; l < 2; ++l) {
    const float* ad = P.adam + 4 * P.update_steps[l];
    const float alpha = ad[0], bc1 = ad[1], bc2 = ad[2];
    const int in_size = P.in_size[l], row = in_size + V;
    JIT_SYNCTHREADS();
    for (int k = tid; k < 3 * LH * LCPC; k += LSTM_THREADS) {
      const int g = k / (LH * LCPC), r = k - g * LH * LCPC, ep = r / LCPC, i = r - ep * LCPC;
      err_s[k] = P.err[l][g][(size_t)ep * LC + LCPC * rank + i];
    }
    for (int c0 = 0; c0 < row; c0 += TILE) {
      const int nc = min(TILE, row - c0);
      JIT_SYNCTHREADS();
      // dense columns of this tile: inputs of all 100 steps
      for (int k = tid; k < LH * TILE; k += LSTM_THREADS) {
        const int ep = k / TILE, c = k - ep * TILE, col = c0 + c;
        in_t[k] = (c < nc && col >= V) ? P.input[l][(size_t)ep * in_size + (col - V)] : 0.0f;
      }
      JIT_SYNCTHREADS();
      for (int k = tid; k < 3 * nc * LCPC; k += LSTM_THREADS) {
        const int g = k / (nc * LCPC), r = k - g * nc * LCPC, c = r / LCPC, i = r - c * LCPC, col = c0 + c;
        const float* es = err_s + (size_t)g * LH * LCPC + i;
        float acc = 0.0f;
        if (col >= V) {
          for (int ep = LH - 1; ep >= 0; --ep) acc = XM_FADD(acc, XM_FMUL(es[ep * LCPC], in_t[ep * TILE + c]));
        } else {
          for (int ep = LH - 1; ep >= 0; --ep) if (sh.sym[ep] == col) acc = XM_FADD(acc, es[ep * LCPC]);
        }
        const size_t idx = lstm_widx(V, in_size, col, LCPC * rank + i);
        float* const Gm = P.m[l][g]; float* const Gv = P.v[l][g]; float* const Gw = P.w[l][g];
        float m = Gm[idx], v = Gv[idx], w = Gw[idx];
        m = XM_FMUL(m, beta1); m = XM_FADD(m, XM_FMUL(1.0f - beta1, acc));
        v = XM_FMUL(v, beta2); v = XM_FADD(v, XM_FMUL(XM_FMUL(1.0f - beta2, acc), acc));
        w = XM_FSUB(w, XM_FMUL(alpha, XM_FDIV(XM_FDIV(m, bc1), __fsqrt_rn(XM_FADD(XM_FDIV(v, bc2), eps)))));
        Gm[idx] = m; Gv[idx] = v; Gw[idx] = w;
      }
    }
    if (tid < 96 && (tid & 31) < LCPC) {
      const int g = tid >> 5, cell = LCPC * rank + (tid & 31);
      GateState& G = S.layer[l].gate[g];
      {
        const float acc = gamma_u[l];
        float m = G.gamma_m[cell], v = G.gamma_v[cell], w = sh.gam[l][g][tid & 31];
        m = XM_FMUL(m, beta1); m = XM_FADD(m, XM_FMUL(1.0f - beta1, acc));
        v = XM_FMUL(v, beta2); v = XM_FADD(v, XM_FMUL(XM_FMUL(1.0f - beta2, acc), acc));
        w = XM_FSUB(w, XM_FMUL(alpha, XM_FDIV(XM_FDIV(m, bc1), __fsqrt_rn(XM_FADD(XM_FDIV(v, bc2), eps)))));
        G.gamma_m[cell] = m; G.gamma_v[cell] = v; G.gamma[cell] = w; sh.gam[l][g][tid & 31] = w;
      }
      {
        const float acc = beta_u[l];
        float m = G.beta_m[cell], v = G.beta_v[cell], w = sh.bet[l][g][tid & 31];
        m = XM_FMUL(m, beta1); m = XM_FADD(m, XM_FMUL(1.0f - beta1, acc));
        v = XM_FMUL(v, beta2); v = XM_FADD(v, XM_FMUL(XM_FMUL(1.0f - beta2, acc), acc));
        w = XM_FSUB(w, XM_FMUL(alpha, XM_FDIV(XM_FDIV(m, bc1), __fsqrt_rn(XM_FADD(XM_FDIV(v, bc2), eps)))));
        G.beta_m[cell] = m; G.beta_v[cell] = v; G.beta[cell] = w; sh.bet[l][g][tid & 31] = w;
      }
    }
  }
  JIT_SYNCTHREADS();
}

// ByteMixer::ByteUpdate -> Lstm::SetInput + Lstm::Perceive + Lstm::Predict (byte-mixer.cpp:22-38,
// lstm.cpp:80-150) by the whole cluster. `ppmd` = 256-entry PPMD distribution after this byte (or
// null), `byte` = the byte just completed. Leaves the new 256-entry distribution in S.bm.probs.
// Load the pointer/scalar cache and this CTA's resident slices (kernel prologue) ...
__device__ void lstm_load_cache(LstmState& S, LstmShared& sh, int rank, int tid) {
  if (tid == 0) {
    LstmPtrs& P = sh.P;
    for (int l = 0; l < 2; ++l) {
      LayerState& L = S.layer[l];
      for (int g = 0; g < 3; ++g) {
        GateState& G = L.gate[g];
        P.w[l][g] = G.w; P.m[l][g] = G.m; P.v[l][g] = G.v; P.state[l][g] = G.state; P.norm[l][g] = G.norm; P.err[l][g] = G.err;
        P.ivar[l][g] = G.ivar;
      }
      P.tanh_state[l] = L.tanh_state; P.igs[l] = L.input_gate_state; P.last_state[l] = L.last_state; P.input[l] = L.input;
      P.in_size[l] = L.in_size; P.lepoch[l] = L.epoch; P.update_steps[l] = L.update_steps;
    }
    P.out_w = S.out_w; P.output = S.output; P.adam = S.adam; P.epoch = S.epoch; P.V = S.V;
  }
  if (tid < 96 && (tid & 31) < LCPC) {
    const int g = tid >> 5, i = tid & 31, cell = LCPC * rank + i;
    for (int l = 0; l < 2; ++l) { sh.gam[l][g][i] = S.layer[l].gate[g].gamma[cell]; sh.bet[l][g][i] = S.layer[l].gate[g].beta[cell]; }
  }
  if (tid < LCPC) { sh.cst[0][tid] = S.layer[0].state[LCPC * rank + tid]; sh.cst[1][tid] = S.layer[1].state[LCPC * rank + tid]; }
  if (tid < LSTM_HORIZON) sh.hist[tid] = S.input_history[tid];
  for (int i = tid; i < 256; i += LSTM_THREADS) { sh.bmap[i] = S.byte_map[i]; sh.vocab[i] = S.vocab[i]; sh.probs256[i] = S.bm.probs[i]; }
  for (int j = tid; j < LSTM_HID; j += LSTM_THREADS) sh.hid[j] = S.hidden[j];
  JIT_SYNCTHREADS();
  {   // softmax output of the previous byte (needed by the output-layer SGD)
    const int V = sh.P.V, le = sh.P.epoch == 0 ? LSTM_HORIZON - 1 : sh.P.epoch - 1;
    for (int i = tid; i < V; i += LSTM_THREADS) sh.logits[i] = sh.P.output[(size_t)le * V + i];
  }
  JIT_SYNCTHREADS();
}
// ... and write the mutable part back (kernel epilogue).
__device__ void lstm_store_cache(LstmState& S, LstmShared& sh, int rank, int tid) {
  JIT_SYNCTHREADS();
  if (tid < LCPC) { S.layer[0].state[LCPC * rank + tid] = sh.cst[0][tid]; S.layer[1].state[LCPC * rank + tid] = sh.cst[1][tid]; }
  if (rank == 0) {
    if (tid == 0) {
      for (int l = 0; l < 2; ++l) { S.layer[l].epoch = sh.P.lepoch[l]; S.layer[l].update_steps = sh.P.update_steps[l]; }
      S.epoch = sh.P.epoch;
    }
    if (tid < LSTM_HORIZON) S.input_history[tid] = sh.hist[tid];
    for (int j = tid; j < LSTM_HID; j += LSTM_THREADS) S.hidden[j] = sh.hid[j];
    for (int i = tid; i < 256; i += LSTM_THREADS) S.bm.probs[i] = sh.probs256[i];
    if (tid == 0) { S.bm.top = 255; S.bm.bot = 0; }
  }
}

// ByteMixer::ByteUpdate -> Lstm::SetInput + Lstm::Perceive + Lstm::Predict (byte-mixer.cpp:22-38,
// lstm.cpp:80-150) by the whole cluster. `ppmd` = 256-entry PPMD distribution after this byte (or
// null), `byte` = the byte just completed. Leaves the new 256-entry distribution in sh.probs256.
__device__ void lstm_byte_update(cgl::cluster_group& cluster, LstmState& S, const float* ppmd, u32 byte, LstmShared& sh, int rank, int tid,
                                 unsigned long long* prof, long long* tprev) {
  LstmPtrs& P = sh.P;
  const int V = P.V, HW = LSTM_HID;
  const unsigned input = (unsigned)sh.bmap[byte];
  const int epoch = P.epoch;
  const int last_epoch = epoch == 0 ? LH - 1 : epoch - 1;
  const int old_input = (int)sh.hist[last_epoch];
  // SetInput: aux[k] = 2 * ppmd[k-th vocabulary byte] into both layers' input at epoch_
  if (rank == 0 && tid < 256 && sh.vocab[tid]) {
    const float p = ppmd ? ppmd[tid] : (float)(1. / 256);
    const float a = XM_FMUL(XM_FADD(0.0f, p), 2.0f);
    const int k = sh.bmap[tid];
    P.input[0][(size_t)epoch * P.in_size[0] + k] = a;
    P.input[1][(size_t)epoch * P.in_size[1] + k] = a;
  }
  JIT_SYNCTHREADS();
  if (tid == 0) sh.hist[last_epoch] = input;
  JIT_SYNCTHREADS();
  L_PROF(0);
  if (epoch == 0) {
    // ------------------------------ truncated BPTT ------------------------------
    __threadfence();
    jit_cluster_sync(cluster, JIT_HERE);                                     // rank 0's SetInput writes are visible to every CTA
    if (tid < LH) sh.sym[tid] = tid == 0 ? old_input : (int)sh.hist[tid - 1];
    float gamma_u[2] = {0.0f, 0.0f}, beta_u[2] = {0.0f, 0.0f};
    float he_reg = 0.0f, stored_reg[2] = {0.0f, 0.0f}, se_reg[2] = {0.0f, 0.0f};
    if (tid < LCPC) he_reg = S.hidden_error[LCPC * rank + tid];
    // recurrent weight blocks of both layers (constant during the BPTT) into shared memory
    float* rec[2];
    rec[0] = sh.pool;                                   // layer 0: [3][1][LC][LCPC]
    rec[1] = sh.pool + 3 * 1 * LC * LCPC;               // layer 1: [3][2][LC][LCPC]
    float* wo_s = sh.pool + 3 * 3 * LC * LCPC;          // [V][LCPC] slice of W_o[ep] for the current layer
    for (int l = 0; l < 2; ++l) {
      const int ntypes = l + 1;                         // layer 0 has no layer below: only the stored_error block
      for (int k = tid; k < 3 * ntypes * LC * LCPC; k += LSTM_THREADS) {
        const int i = k % LCPC, j = (k / LCPC) % LC, type = (k / (LCPC * LC)) % ntypes, g = k / (LCPC * LC * ntypes);
        const int col = 2 * V + type * LC + LCPC * rank + i;
        lcp_async4(rec[l] + k, P.w[l][g] + lstm_widx(V, P.in_size[l], col, j));
      }
    }
    lcp_async_wait();
    JIT_SYNCTHREADS();
    for (int ep = LH - 1; ep >= 0; --ep) {
      const float* out = P.output + (size_t)ep * V;
      const float* W = P.out_w + (size_t)ep * V * HW;
      for (int i = tid; i < V; i += LSTM_THREADS) sh.err[i] = ((unsigned)i == sh.hist[ep]) ? XM_FSUB(out[i], 1.0f) : out[i];
      for (int l = 1; l >= 0; --l) {
        // slice of W_o[ep]: columns l*200 + own 25 cells, all V rows
        JIT_SYNCTHREADS();
        for (int k = tid; k < V * LCPC; k += LSTM_THREADS) {
          const int i = k / LCPC, jj = k - i * LCPC;
          lcp_async4(wo_s + k, W + (size_t)i * HW + l * LC + LCPC * rank + jj);
        }
        lcp_async_wait();
        JIT_SYNCTHREADS();
        if (tid < LCPC) {
          float he = he_reg;
          const float* wc = wo_s + tid;
#pragma unroll 8
          for (int i = 0; i < V; ++i) he = XM_FADD(he, XM_FMUL(wc[(size_t)i * LCPC], sh.err[i]));
          he_reg = he;
        }
        lstm_layer_backward(cluster, S, l, ep, sh, rec[l], rank, tid, &gamma_u[l], &beta_u[l], &he_reg, &stored_reg[l], &se_reg[l]);
      }
    }
    if (tid < LCPC) {
      const int cell = LCPC * rank + tid;
      S.hidden_error[cell] = he_reg;
      for (int l = 0; l < 2; ++l) { S.layer[l].stored_error[cell] = stored_reg[l]; S.layer[l].state_error[cell] = se_reg[l]; }
    }
    L_PROF(1);
    lstm_apply_updates(S, sh, rank, tid, gamma_u, beta_u);
    __threadfence();
    jit_cluster_sync(cluster, JIT_HERE);
    L_PROF(2);
  }
  // ---- output layer SGD (lstm.cpp:112-116): W_o[epoch] = W_o[last_epoch] - (lr*err_i) * hidden, own rows ----
  {
    const int rpc = (V + LSTM_CTAS - 1) / LSTM_CTAS;
    const int r0 = rank * rpc, r1 = min(V, r0 + rpc);
    const float* Wl = P.out_w + (size_t)last_epoch * V * HW;
    float* We = P.out_w + (size_t)epoch * V * HW;
    // sh.logits still holds the softmax output of the previous byte (output_[last_epoch])
    for (int i = tid; i < V; i += LSTM_THREADS) sh.err[i] = XM_FMUL(0.03f, ((unsigned)i == input) ? XM_FSUB(sh.logits[i], 1.0f) : sh.logits[i]);
    JIT_SYNCTHREADS();
    for (int idx = r0 * HW + tid; idx < r1 * HW; idx += LSTM_THREADS) {
      const int i = idx / HW, j = idx - i * HW;
      We[idx] = XM_FSUB(Wl[idx], XM_FMUL(sh.err[i], sh.hid[j]));
    }
    JIT_SYNCTHREADS();
  }
  L_PROF(3);
  lstm_predict(cluster, S, input, sh, rank, tid, prof, tprev);
  // ByteMixer: scatter back to 256 bytes; ByteModel::ByteUpdate resets the range
  if (tid < 256) sh.probs256[tid] = sh.vocab[tid] ? sh.logits[sh.bmap[tid]] : 0.0f;
  JIT_SYNCTHREADS();
}

// Bit-level read-out of the byte distribution (ByteModel::Predict + the override test of
// predictor.cpp:378-387) followed by ByteModel::Perceive. Single thread.
__device__ void lstm_readout(LstmState& S, const Tables& T, float* x_out, float* override_out) {
  const float p = bytemodel_predict(S.bm.probs, S.bm.bot, S.bm.top, &S.bm.ex);
  *override_out = (p == 0.0f || p == 1.0f) ? p : -1.0f;
  *x_out = stretch(T, p);
}
// lstmpr = Discretize(p) = 1 + 4094 * p truncated (predictor.cpp:180-182), lstmex = first arg-max of the byte range
// (byte-model.cpp:13-20), packed as lstmpr | lstmex << 16.
__device__ __forceinline__ u32 lstm_feedback(const float* probs, int bot, int top, float p) {
  int ex = bot; float best = probs[bot];
  for (int i = bot + 1; i <= top; ++i) if (probs[i] > best) { best = probs[i]; ex = i; }
  const u32 pr = (u32)XM_FADD(1.0f, XM_FMUL(4094.0f, p));
  return (pr & 0xffffu) | ((u32)ex << 16);
}
__device__ void bm_perceive(ByteModelState& b, int bit) {
  b.mid = b.bot + ((b.top - b.bot) / 2);
  if (bit) b.bot = b.mid + 1; else b.top = b.mid;
}

__global__ void __cluster_dims__(LSTM_CTAS, 1, 1) __launch_bounds__(LSTM_THREADS, 1)
lstm_kernel(const ChunkArgs* __restrict__ args_all, Tables T) { jit_entry(JK_LSTM);
  cgl::cluster_group cluster = cgl::this_cluster();
  const int rank = (int)cluster.block_rank();
  const ChunkArgs a = args_all[blockIdx.x / LSTM_CTAS];
  LstmState& S = a.st->lstm;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  LstmShared& sh = *reinterpret_cast<LstmShared*>(smem_raw);
  const int tid = threadIdx.x;
  unsigned long long* prof = (a.prof && rank == 0 && tid == 0) ? a.prof : nullptr;
  long long tprev = clock64();
  lstm_load_cache(S, sh, rank, tid);
  for (u32 pos = 0; pos < a.n_bytes; ++pos) {
    const u32 byte = a.bytes[pos];
    if (rank == 0) {
      // ByteModel::Predict for the 8 bits of this byte (byte-model.cpp:8-24): the ranges are known, so
      // the 8 read-outs are 8 independent serial sums out of shared memory, one lane each.
      if (tid < 8) {
        int bot = 0, top = 255;
        for (int k = 0; k < tid; ++k) { const int mid = bot + ((top - bot) / 2); if ((byte >> (7 - k)) & 1) bot = mid + 1; else top = mid; }
        const int mid = bot + ((top - bot) / 2);
        float num = 0.0f;
#pragma unroll 8
        for (int i = mid + 1; i <= top; ++i) num = XM_FADD(num, sh.probs256[i]);
        float denom = num;
#pragma unroll 8
        for (int i = bot; i <= mid; ++i) denom = XM_FADD(denom, sh.probs256[i]);
        const float p = denom == 0 ? 0.5f : XM_FDIV(num, denom);
        const u64 t = (u64)pos * 8 + tid;
        a.lstm_x[2 * t] = stretch(T, p);
        a.lstm_x[2 * t + 1] = (p == 0.0f || p == 1.0f) ? p : -1.0f;
        // FXCM's feedback (predictor.cpp:462-465): the read-out of bit t is what FXCM sees while perceiving bit t-1
        if (a.lstm_fx && tid > 0) a.lstm_fx[t - 1] = lstm_feedback(sh.probs256, bot, top, p);
      }
    }
    lstm_byte_update(cluster, S, a.ppmd ? a.ppmd + (u64)pos * 256 : nullptr, byte, sh, rank, tid, prof, &tprev);
    if (a.lstm_fx && rank == 0 && tid == 0) {   // first bit of the next byte: range [0,255] whatever that byte is
      int ex; const float p = bytemodel_predict(sh.probs256, 0, 255, &ex);
      a.lstm_fx[(u64)pos * 8 + 7] = lstm_feedback(sh.probs256, 0, 255, p);
    }
  }
  lstm_store_cache(S, sh, rank, tid);
  __threadfence();
  jit_cluster_sync(cluster, JIT_HERE);
}

// Lock-step halves.
// Lock-step Predict(), producer half: CTA 0 = the 54 small models + contexts (small_models.cuh), CTA 1 = the
// LSTM's bit read-out (ByteModel::Predict, byte-model.cpp:8-15). Independent of each other, one launch.
__global__ void __launch_bounds__(64, 1) lock_predict_inputs_kernel(StreamState* st, Tables T) { jit_entry(JK_LSTM_INPUTS);
  if (blockIdx.x == 1) {            // the LSTM's bit read-out: the 256 probabilities come in side by side, the sums stay one serial chain
    __shared__ float probs[256];
    ByteModelState& b = st->lstm.bm;
    for (int i = threadIdx.x; i < 256; i += 64) probs[i] = b.probs[i];
    JIT_SYNCTHREADS();
    if (threadIdx.x == 0) {
      const float p = bytemodel_predict(probs, b.bot, b.top, &b.ex);
      st->lstm_override = (p == 0.0f || p == 1.0f) ? p : -1.0f;
      st->lstm_x = stretch(T, p);
    }
    return;
  }
  __shared__ SmallShared sh;
  SmallState& s = st->small;
  const int tid = threadIdx.x;
  for (int i = tid; i < 256; i += 64) { sh.bracket_probs[i] = s.bracket_bm.probs[i]; sh.ppmd_probs[i] = s.ppmd_bm.probs[i]; }
  if (tid == 0) small_refresh_tables(s, sh);
  JIT_SYNCTHREADS();
  small_predict(st->small, T, sh, st->small_x, st->sel, tid);
}
__global__ void __cluster_dims__(LSTM_CTAS, 1, 1) __launch_bounds__(LSTM_THREADS, 1)
lstm_byte_kernel(StreamState* st, u32 byte, const float* ppmd, const u32* dbit = nullptr) { jit_entry(JK_LSTM_BYTE);
  if (dbit) byte = dbit[1];
  cgl::cluster_group cluster = cgl::this_cluster();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  LstmShared& sh = *reinterpret_cast<LstmShared*>(smem_raw);
  long long tprev = 0;
  const int rank = (int)cluster.block_rank();
  lstm_load_cache(st->lstm, sh, rank, threadIdx.x);
  lstm_byte_update(cluster, st->lstm, ppmd, byte, sh, rank, threadIdx.x, nullptr, &tprev);
  lstm_store_cache(st->lstm, sh, rank, threadIdx.x);
  __threadfence();
  jit_cluster_sync(cluster, JIT_HERE);
}

#undef LC
#undef LH
}  // namespace cmixb200
