// cmix_b200/csrc/fxcm.cuh — the resident FXCM model on the device (SURVEY §8 row a14).
//
// One CTA of 10 warps per stream runs fxcm_model.h's phases for every bit of a sub-chunk. FXCM is a PRODUCER like the
// small models: in the compress direction it depends on the coded bytes and on the LSTM's bit read-out only
// (lstmpr / lstmex, reference predictor.cpp:462-466), never on the final mixer, so it runs ahead of the mixer on its
// own CUDA stream and hands over 431 12-bit codes per bit through the `ext` scratch the mixer stages from.
//
// Lane roles: every context of the 31 bucketed context maps is a lane (warps 0-7, lane = map * 8 + context). The contexts of
// a map are independent as long as they touch different buckets this bit; that is CHECKED per bit (map_touched, including
// the buckets a deferred history write-back will reach) and a map with a clash is evaluated by one lane in order instead.
// Warp 8 runs match model 2, warp 9 the sparse match model, the seven stationary maps and the run map. The ten 512-wide
// weight rows of the pending prediction are cached in shared memory between the dot product of one bit and the SGD step of
// the next (written back when a selector moves); the tail (squash, final mixers, six APMs in three dependent levels) runs
// on one warp. The mutable scalar state (9 KB), the text-analysis state (40 KB) and the hot tables (28 KB) live in shared
// memory for the launch; the per-map tables and the ~4.6 GB of model memory stay in HBM.
#pragma once
#include "exact_math.h"
#include "jitter.cuh"
#include "fxcm_model.h"
#include "bytemodel.cuh"
#include "state.h"

namespace cmixb200 {

enum { FX_THREADS = 320, FX_WARPS = 10, FX_MAP_LANES = 248, FX_SEEN = 2048, FX_TID_MATCH = 256, FX_TID_W9 = 288 };

#ifdef FX_PROF
__device__ unsigned long long g_fx_prof[2][24];
#define FX_T(k) do { if (tid == 0) { const long long now_ = clock64(); atomicAdd(&g_fx_prof[sh.prof_row][k], (unsigned long long)(now_ - sh.prof_t)); sh.prof_t = now_; } } while (0)
#else
#define FX_T(k) do { } while (0)
#endif

struct FxShared {
  fx::State S;
  fx::TextState X;
  alignas(16) unsigned char tab[fx::TABLES_HOT_BYTES];
  alignas(16) short w1[10][fx::N_IN1];    // the weight rows of the pending prediction (row i holds set w_set[i] of mixer i)
  int w_set[10];
  int dots[12];
  int clash[fx::N_MAPS]; u32 res[fx::N_MAPS];
  u32 ids[FX_MAP_LANES][5];
  unsigned long long seen[FX_SEEN];   // open-addressing set of (map, bucket) pairs touched this bit
#ifdef FX_PROF
  long long prof_t; int prof_row;
#endif
};

__device__ __forceinline__ void fx_copy_words(void* dst, const void* src, size_t bytes, int tid) {
  u32* d = (u32*)dst; const u32* s = (const u32*)src;
  for (size_t i = tid; i < bytes / 4; i += FX_THREADS) d[i] = s[i];
}
static_assert(sizeof(fx::State) % 4 == 0 && sizeof(fx::TextState) % 4 == 0, "state blocks are copied word by word");

// a 512-weight row between HBM and shared memory: two 16-byte words per lane, past L1
__device__ __forceinline__ void fx_row_load(short* dst, const short* src, int lane) {
  const uint4* s = reinterpret_cast<const uint4*>(src); uint4* d = reinterpret_cast<uint4*>(dst);
  const uint4 a = __ldcg(s + lane), b = __ldcg(s + lane + 32);
  d[lane] = a; d[lane + 32] = b;
}
__device__ __forceinline__ void fx_row_store(short* dst, const short* src, int lane) {
  const uint4* s = reinterpret_cast<const uint4*>(src); uint4* d = reinterpret_cast<uint4*>(dst);
  __stcg(d + lane, s[lane]); __stcg(d + lane + 32, s[lane + 32]);
}
static_assert(fx::N_IN1 == 512, "a first-layer weight row is 64 16-byte words");

struct FxGlobals { fx::TextState* gx; const fx::Tables* gT; };
__device__ __forceinline__ FxGlobals fx_load(FxShared& sh, fx::State* g, int tid) {
  FxGlobals r;
  r.gx = g->text; r.gT = g->T;
  fx_copy_words(&sh.S, g, sizeof(fx::State), tid);
  fx_copy_words(&sh.X, r.gx, sizeof(fx::TextState), tid);
  fx_copy_words(sh.tab, r.gT, fx::TABLES_HOT_BYTES, tid);
  JIT_SYNCTHREADS();
  if (tid == 0) { sh.S.text = &sh.X; sh.S.T = reinterpret_cast<const fx::Tables*>(sh.tab); }
  const int warp = tid >> 5, lane = tid & 31;
  if (warp < 10) {
    const fx::MixState& m = sh.S.mix[warp];
    fx_row_load(sh.w1[warp], m.w + (size_t)m.cxt * fx::N_IN1, lane);
    if (lane == 0) sh.w_set[warp] = m.cxt;
  }
  JIT_SYNCTHREADS();
  return r;
}
__device__ __forceinline__ void fx_store(FxShared& sh, fx::State* g, const FxGlobals& r, int tid) {
  JIT_SYNCTHREADS();
  const int warp = tid >> 5, lane = tid & 31;
  if (warp < 10) fx_row_store(sh.S.mix[warp].w + (size_t)sh.w_set[warp] * fx::N_IN1, sh.w1[warp], lane);
  if (tid == 0) { sh.S.text = r.gx; sh.S.T = r.gT; }
  JIT_SYNCTHREADS();
  fx_copy_words(g, &sh.S, sizeof(fx::State), tid);
  fx_copy_words(r.gx, &sh.X, sizeof(fx::TextState), tid);
}

// (map, bucket) pairs of one context into the per-bit set; true when a pair was already there (another context of the map
// touches the same bucket this bit). A context's own repeats are removed first.
__device__ bool fx_claim(unsigned long long* seen, int map, const u32* ids, int n) {
  bool clash = false;
  for (int a = 0; a < n; ++a) {
    bool dup = false;
    for (int b = 0; b < a; ++b) dup = dup || ids[b] == ids[a];
    if (dup) continue;
    const unsigned long long key = ((unsigned long long)(map + 1) << 32) | ids[a];
    u32 slot = (u32)((key * 0x9E3779B97F4A7C15ull) >> 53) & (FX_SEEN - 1);
    for (;;) {
      const unsigned long long old = atomicCAS(&seen[slot], 0ull, key);
      if (old == 0ull) break;
      if (old == key) { clash = true; break; }
      slot = (slot + 1) & (FX_SEEN - 1);
    }
  }
  return clash;
}

// The tail of a bit on one warp (fxcm_model.h bit_tail): squash of the ten first-layer outputs, the two final mixers, the six
// APMs (three dependent levels), the exports.
__device__ void fx_tail_warp(FxShared& sh, int lane) {
  using namespace fx;
  State& S = sh.S;
  const fx::Tables& T = *S.T;
  const TextState& X = *S.text;
  const unsigned full = 0xffffffffu;
  const int ei = S.ex_off[N_UNITS];
  if (lane < 10) {
    int dp = (int)((u32)sh.dots[lane] * (u32)T.mix_shift[lane]) >> 11;
    dp = clp(dp);
    const int pr = squash(T, dp);
    S.mix[lane].pr = pr;
    S.in2[lane] = (short)dp;
    S.codes[ei + lane] = (u16)pr;
  } else if (lane == 10) S.in2[10] = (short)(stretch(T, S.lstmpr) / 2);
  __syncwarp();
  int acc = 0;
  {
    const int i = 10 + (lane >> 3), k = 2 * (lane & 7);
    if (lane < 16) { const short* w = S.mix[i].w + (size_t)S.mix[i].cxt * N_IN2; acc = dot_pair(S.in2 + k, w + k); }
    acc += __shfl_xor_sync(full, acc, 1); acc += __shfl_xor_sync(full, acc, 2); acc += __shfl_xor_sync(full, acc, 4);
    if (lane < 16) {
      int dp = (int)((u32)acc * (u32)T.mix_shift[i]) >> 11;
      dp = clp(dp);
      if ((lane & 7) == 0) S.mix[i].pr = squash(T, dp);
      acc = dp;
    }
  }
  const int fin0 = __shfl_sync(full, acc, 0), fin1 = __shfl_sync(full, acc, 8);
  const int pr = squash(T, (fin0 * 7 + fin1 + 4) >> 3);
  const int y = S.y, c0 = S.c0, rate = S.rate;
  const u32 fails = S.fails;
  // level 1: three APMs refine pr
  int a = 0;
  if (lane == 0) a = apm_p(T, S.apm[0], pr, (u32)c0, 3, y);
  else if (lane == 1) a = apm_p(T, S.apm[1], pr, ((u32)(c0 * 8) ^ hash3(29, S.failz & 2047)) & 0xffff, rate + 1, y);
  else if (lane == 2) a = apm_p(T, S.apm[2], pr, ((u32)(c0 * 32) ^ X.ah2) & 0xffff, rate, y);
  const int pu0 = (__shfl_sync(full, a, 0) + 7 * pr + 4) >> 3;
  const int pv0 = __shfl_sync(full, a, 1), pt = __shfl_sync(full, a, 2);
  // level 2
  int b = 0;
  if (lane == 0) b = apm_p(T, S.apm[3], pu0, ((u32)(c0 * 2) ^ X.ah1) & 0x3ffff, rate, y);
  else if (lane == 1) {
    if (fails & 255) b = apm_p(T, S.apm[4], pv0, hash3((u32)c0, X.s2b & 0xfffc, X.s3bR & 0x1ff) & 0x3ffff, rate, y);
    else b = apm_p(T, S.apm[4], pv0, hash3((u32)c0, (X.s2bR & 0xfffc) + 0x10000, X.s3bR & 0x1ff) & 0x3ffff, rate, y);
  }
  const int pu = __shfl_sync(full, b, 0), pv = __shfl_sync(full, b, 1);
  // level 3
  if (lane == 0) {
    int pz = (int)S.failcount + 1;
    const int tri[4] = {0, 4, 3, 7}, trj[4] = {0, 6, 6, 12};
    pz += tri[(fails >> 5) & 3];
    pz += trj[(fails >> 3) & 3];
    pz += trj[(fails >> 1) & 3];
    if (fails & 1) pz += 8;
    pz = pz / 2;
    pz = apm_p(T, S.apm[5], pu, ((u32)(c0 * 4) ^ hash3((u32)imin(9, pz), X.x5 & 0x80ff)) & 0x3ffff, rate, y);
    int fin;
    if (fails & 255) fin = (pt * 6 + pu + pv * 11 + pz * 14 + 31) >> 5;
    else fin = (pt * 4 + pu * 5 + pv * 12 + pz * 11 + 31) >> 5;
    u16* c = S.codes + ei + 10;
    c[0] = (u16)pr; c[1] = (u16)pu; c[2] = (u16)pv0; c[3] = (u16)pv; c[4] = (u16)pt; c[5] = (u16)pz; c[6] = (u16)fin;
    S.pr = fin;
  }
}

// One bit: FXCM::Perceive(bit) (fxcmv1.cpp:4909-4912 -> update1 :4758). All FX_THREADS lanes call it.
__device__ void fx_bit(FxShared& sh, int y, int lstmpr, int lstmex, int tid) {
  using namespace fx;
  State& S = sh.S;
  const int warp = tid >> 5, lane = tid & 31;
#ifdef FX_PROF
  if (tid == 0) { sh.prof_t = clock64(); sh.prof_row = (S.bpos == 7) ? 0 : 1; }
#endif
  // ---- A: bookkeeping, SGD errors, failure history and (byte boundary) the text analysis
  if (tid == 0) { bit_head(S, y, lstmpr, lstmex); bit_prepare_head(S); }
  if (tid >= 32 && tid < 32 + N_MAPS) { sh.clash[tid - 32] = 0; sh.res[tid - 32] = 0; }
  for (int k = tid; k < FX_SEEN; k += FX_THREADS) sh.seen[k] = 0ull;
  JIT_SYNCTHREADS();
  FX_T(0);
  // ---- B: SGD on the cached rows (Mixer1::update), the two 16-wide final rows, the units' slices of the vectors
  for (int idx = tid; idx < 10 * (N_IN1 / 8); idx += FX_THREADS) {
    const int i = idx >> 6, q = idx & 63;
    const int err = S.mix[i].err;
    if (!err) continue;
    uint4* wp = reinterpret_cast<uint4*>(&sh.w1[i][q * 8]);
    uint4 wv = *wp;
    const uint4 xv = *reinterpret_cast<const uint4*>(&S.in1[q * 8]);
    short* w = reinterpret_cast<short*>(&wv);
    const short* x = reinterpret_cast<const short*>(&xv);
#pragma unroll
    for (int e = 0; e < 8; ++e) w[e] = train_one(x[e], w[e], err);
    *wp = wv;
  }
  if (warp == FX_WARPS - 1) {
    {
      const MixState& m = S.mix[10 + (lane >> 4)];
      if (m.err) { short* w = m.w + (size_t)m.cxt * N_IN2; const int k = lane & 15; w[k] = train_one(S.in2[k], w[k], m.err); }
    }
    const unsigned full = 0xffffffffu;
    int a0 = 0, e0 = 0, a1 = 0, e1 = 0;
    unit_counts(S, lane, a0, e0);
    if (lane + 32 < N_UNITS) unit_counts(S, lane + 32, a1, e1);
    int ia0 = a0, ie0 = e0, ia1 = a1, ie1 = e1;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int v0 = __shfl_up_sync(full, ia0, d), v1 = __shfl_up_sync(full, ie0, d), v2 = __shfl_up_sync(full, ia1, d), v3 = __shfl_up_sync(full, ie1, d);
      if (lane >= d) { ia0 += v0; ie0 += v1; ia1 += v2; ie1 += v3; }
    }
    const int ta = __shfl_sync(full, ia0, 31), te = __shfl_sync(full, ie0, 31);
    S.in_off[lane] = ia0 - a0; S.ex_off[lane] = ie0 - e0;
    if (lane + 32 <= N_UNITS) { S.in_off[lane + 32] = ta + ia1 - a1; S.ex_off[lane + 32] = te + ie1 - e1; }
  }
  JIT_SYNCTHREADS();
  FX_T(1);
  // ---- C: buckets every map context touches; the units that are one lane each
  if (tid < FX_MAP_LANES) {
    const int id = tid >> 3, i = tid & 7;
    if (i < S.map[id].cn) {
      const int n = map_touched(S, id, i, sh.ids[tid]);
      if (n && fx_claim(sh.seen, id, sh.ids[tid], n)) sh.clash[id] = 1;
    }
  } else {
    int u = -1;
    if (tid == FX_TID_MATCH) u = U_MATCH;
    else if (tid == FX_TID_W9) u = U_SMATCH;
    else if (tid > FX_TID_W9 && tid <= FX_TID_W9 + 7) u = tid - (FX_TID_W9 + 1);
    else if (tid == FX_TID_W9 + 8) u = U_RCM;
    if (u >= 0) bit_unit(S, u);
  }
  JIT_SYNCTHREADS();
  FX_T(2);
  // ---- D: the map contexts
  if (tid < FX_MAP_LANES) {
    const int id = tid >> 3, i = tid & 7;
    Out o; o.n = S.in1; o.codes = S.codes; o.ni = S.in_off[U_MAP0 + id]; o.ei = S.ex_off[U_MAP0 + id];
    if (!sh.clash[id]) {
      if (i < S.map[id].cn && map_ctx_bit(S, id, i, o)) atomicAdd(&sh.res[id], 1u);
    } else if (i == 0) {      // two contexts in one bucket: this map in order, on one lane
      u32 r = 0;
      const int cn = S.map[id].cn;
      for (int k = 0; k < cn; ++k) r += map_ctx_bit(S, id, k, o);
      sh.res[id] = r;
    }
  }
  JIT_SYNCTHREADS();
  FX_T(3);
  // ---- E: map epilogues, weight-set selection
  if (warp == 0) {
    if (lane < N_MAPS) map_finish(S, lane, sh.res[lane]);
    __syncwarp();
    if (lane == 0) bit_select(S);
  }
  JIT_SYNCTHREADS();
  FX_T(4);
  // ---- F: the ten 512-wide dot products over the cached rows (a selector that moved: write back, load)
  {
    const MixState& m = S.mix[warp];
    short* row = sh.w1[warp];
    const int old = sh.w_set[warp];
    if (old != m.cxt) {
      fx_row_store(m.w + (size_t)old * N_IN1, row, lane);
      fx_row_load(row, m.w + (size_t)m.cxt * N_IN1, lane);
      __syncwarp();
      if (lane == 0) sh.w_set[warp] = m.cxt;
    }
    int acc = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint4 wv = *reinterpret_cast<const uint4*>(row + (lane + 32 * h) * 8);
      const uint4 xv = *reinterpret_cast<const uint4*>(S.in1 + (lane + 32 * h) * 8);
      const short* w = reinterpret_cast<const short*>(&wv);
      const short* x = reinterpret_cast<const short*>(&xv);
#pragma unroll
      for (int e = 0; e < 8; e += 2) acc += dot_pair(x + e, w + e);
    }
    acc = __reduce_add_sync(0xffffffffu, acc);
    if (lane == 0) sh.dots[warp] = acc;
  }
  JIT_SYNCTHREADS();
  FX_T(5);
  // ---- G: squash, final mixers, APMs, exports
  if (warp == 0) fx_tail_warp(sh, lane);
  JIT_SYNCTHREADS();
  FX_T(6);
}

// Bulk: CTA b serves stream b of the launch group. Writes ext[t][0..430] for every bit t of the sub-chunk (the codes
// the model holds BEFORE perceiving bit t) and, when a.ext_replay is given, copies the non-resident PAQ8 slots next to them.
__global__ void __launch_bounds__(FX_THREADS, 1) fxcm_kernel(const ChunkArgs* __restrict__ args_all) { jit_entry(JK_FXCM);
  extern __shared__ __align__(16) unsigned char fx_raw[];
  FxShared& sh = *reinterpret_cast<FxShared*>(fx_raw);
  const ChunkArgs a = args_all[blockIdx.x];
  if (a.fx == nullptr) return;
  const int tid = threadIdx.x;
  const FxGlobals gl = fx_load(sh, a.fx, tid);
  const u32 n_bits = a.n_bytes * 8;
  for (u32 t = 0; t < n_bits; ++t) {
    if (!a.pretrain) {
      u16* out = a.ext_gen + (size_t)t * N_EXT;
      for (int k = tid; k < fx::N_OUT; k += FX_THREADS) out[k] = sh.S.codes[k];
      if (a.ext_replay && !a.paq8) for (int k = fx::N_OUT + tid; k < N_EXT; k += FX_THREADS) out[k] = a.ext_replay[(size_t)t * N_EXT + k];
    }
    const int y = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
    int lstmpr = 0, lstmex = 0;
    if (!a.pretrain) { const u32 v = a.lstm_fx[t]; lstmpr = (int)(v & 0xffff); lstmex = (int)(v >> 16); }
    else { lstmpr = sh.S.lstmpr; lstmex = sh.S.lstmex; }
    fx_bit(sh, y, lstmpr, lstmex, tid);
  }
  fx_store(sh, a.fx, gl, tid);
}

// Lock-step: one bit per launch (the decoder's order), queued behind the mixer / LSTM update of the same bit. Lane 0 first
// takes the LSTM's read-out of the NEXT bit (ByteMixer::Predict + Discretize, predictor.cpp:462-465); the codes for the next
// Predict() land in ext_bit[0..430].
__global__ void __launch_bounds__(FX_THREADS, 1) fxcm_bit_kernel(StreamState* st, fx::State* g, int y, int pretrain, u16* ext_bit, const u32* dbit) { jit_entry(JK_FXCM_BIT);
  if (dbit) y = (int)dbit[0];
  extern __shared__ __align__(16) unsigned char fx_raw[];
  FxShared& sh = *reinterpret_cast<FxShared*>(fx_raw);
  const int tid = threadIdx.x;
  const FxGlobals gl = fx_load(sh, g, tid);
  float* probs = reinterpret_cast<float*>(sh.seen);     // free until fx_bit clears it: the 256 probabilities arrive side by side
  if (!pretrain && tid < 256) probs[tid] = st->lstm.bm.probs[tid];
  JIT_SYNCTHREADS();
  if (tid == 0) {
    if (pretrain) { sh.dots[10] = sh.S.lstmpr; sh.dots[11] = sh.S.lstmex; }
    else {
      const ByteModelState& b = st->lstm.bm;
      int ex;
      const float p = bytemodel_predict(probs, b.bot, b.top, &ex);     // the sums stay one serial chain (byte-model.cpp:8-24)
      sh.dots[10] = (int)(u32)XM_FADD(1.0f, XM_FMUL(4094.0f, p));
      sh.dots[11] = ex;
    }
  }
  JIT_SYNCTHREADS();
  const int lstmpr = sh.dots[10], lstmex = sh.dots[11];
  JIT_SYNCTHREADS();
  fx_bit(sh, y, lstmpr, lstmex, tid);
  if (ext_bit) for (int k = tid; k < fx::N_OUT; k += FX_THREADS) ext_bit[k] = sh.S.codes[k];
  fx_store(sh, g, gl, tid);
}

}  // namespace cmixb200
