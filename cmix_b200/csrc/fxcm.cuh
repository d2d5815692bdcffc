// cmix_b200/csrc/fxcm.cuh — the resident FXCM model on the device (SURVEY §8 row a14).
//
// One cluster of two CTAs of 10 warps per stream runs fxcm_model.h's phases for every bit of a sub-chunk. FXCM is a
// PRODUCER like the small models: in the compress direction it depends on the coded bytes and on the LSTM's bit read-out
// only (lstmpr / lstmex, reference predictor.cpp:462-466), never on the final mixer, so it runs ahead of the mixer on its
// own CUDA stream and hands over 431 12-bit codes per bit through the `ext` scratch the mixer stages from.
//
// The model CTA (rank 0). Every context of the 31 bucketed context maps is a lane (warps 0-7, lane = map * 8 + context).
// The contexts of a map are independent as long as they touch different buckets this bit; that is CHECKED per bit
// (map_touched, including the buckets a deferred history write-back will reach) and a map with a clash is evaluated by one
// lane in order instead. Warp 8 runs match model 2, warp 9 the sparse match model, the seven stationary maps and the run
// map. The mutable scalar state (9 KB), the text-analysis state (40 KB) and the hot tables (28 KB) live in shared memory
// for the launch; the per-map tables and the ~4.6 GB of model memory stay in HBM.
//
// The mixer CTA (rank 1): the ten first-layer mixers, the two final mixers and the six APMs. The models never read them
// back (only mixer 9's selector reads the failure history), so this stage runs up to FX_RING bits behind the models. The
// model CTA hands each bit over through a ring slot in the mixer CTA's shared memory (cluster_mbar.cuh): the bit's
// inputs, its codes, the selectors and the few scalars and text fields the APMs read. The mixer CTA computes the error
// terms and trains on bit t-1's inputs as soon as bit t is known, then takes slot t, moves the weight rows whose
// selector changed, runs the dot products and the tail, and writes the bit's code row. The ten selected 512-wide rows and
// the final mixers' whole weight tables stay in its shared memory for the launch.
#pragma once
#include <cooperative_groups.h>
#include "exact_math.h"
#include "jitter.cuh"
#include "cluster_mbar.cuh"
#include "fxcm_model.h"
#include "bytemodel.cuh"
#include "state.h"
#include "census.cuh"

namespace cmixb200 {

enum { FX_THREADS = 320, FX_WARPS = 10, FX_MAP_LANES = 248, FX_SEEN = 2048, FX_TID_MATCH = 256, FX_TID_W9 = 288, FX_RING = 4,
       FX_FIN_SETS = 224 };   // weight sets of final mixer 10 (fxcm_host.h kMixM[10]); final mixer 11 has one

#ifdef FX_PROF
// slots 0-11: the model CTA's bit (12, 13: parts of lane 0's share of slot 0); 16-23: the mixer CTA's bit
__device__ unsigned long long g_fx_prof[2][24];
#define FX_T(k) do { if (tid == 0) { const long long now_ = clock64(); atomicAdd(&g_fx_prof[sh.prof_row][k], (unsigned long long)(now_ - sh.prof_t)); sh.prof_t = now_; } } while (0)
#else
#define FX_T(k) do { } while (0)
#endif

// One bit handed from the model CTA to the mixer CTA.
struct FxSlot {
  alignas(16) short in1[fx::N_IN1];
  alignas(16) u16 codes[fx::N_OUT + 1];   // the models' codes; [0, ei) are this bit's
  int cxt[fx::N_MIX];                      // selectors (9 is the mixer CTA's own)
  int ei, lstmpr, lstmex, c0, rate;
  u32 ah1, ah2, s2b, s2bR, s3bR, x5;       // the text state the APMs read
};

struct FxShared {
  fx::State S;
  alignas(16) unsigned char tab[fx::TABLES_HOT_BYTES];
  union {
    struct {            // model CTA
      fx::TextState X;
      int clash[fx::N_MAPS]; u32 res[fx::N_MAPS];
      u32 ids[FX_MAP_LANES][5];
      unsigned long long seen[FX_SEEN];   // open-addressing set of (map, bucket) pairs touched this bit
      int lstm[2];
      unsigned long long empty[FX_RING];
    } md;
    struct {            // mixer CTA
      alignas(16) short w1[10][fx::N_IN1];             // row i holds set w_set[i] of mixer i
      alignas(16) short w2[FX_FIN_SETS + 1][fx::N_IN2];  // final mixer 10's sets, then mixer 11's one
      int w_set[10];
      int dots[10];
      FxSlot ring[FX_RING];
      unsigned long long full[FX_RING];
    } mx;
  } u;
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
static_assert((fx::N_OUT + 1) % 8 == 0 && fx::N_IN2 == 16, "slot vectors are copied in 16-byte words");

struct FxGlobals { fx::TextState* gx; const fx::Tables* gT; };
// Both CTAs: the state block and the hot tables into shared memory, the ring's barriers; the model CTA: the text state;
// the mixer CTA: the selected first-layer rows and the final mixers' tables.
__device__ __forceinline__ FxGlobals fx_load(FxShared& sh, fx::State* g, int tid, int rank) {
  FxGlobals r;
  r.gx = g->text; r.gT = g->T;
  fx_copy_words(&sh.S, g, sizeof(fx::State), tid);
  fx_copy_words(sh.tab, r.gT, fx::TABLES_HOT_BYTES, tid);
  if (rank == 0) fx_copy_words(&sh.u.md.X, r.gx, sizeof(fx::TextState), tid);
  if (tid == 0) {
    for (int i = 0; i < FX_RING; ++i) {
      if (rank == 0) mbar_init(&sh.u.md.empty[i], 1);
      else mbar_init(&sh.u.mx.full[i], FX_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  JIT_SYNCTHREADS();
  if (tid == 0) { sh.S.text = rank == 0 ? &sh.u.md.X : nullptr; sh.S.T = reinterpret_cast<const fx::Tables*>(sh.tab); }
  const int warp = tid >> 5, lane = tid & 31;
  if (rank == 1) {
    const fx::MixState& m = sh.S.mix[warp];
    fx_row_load(sh.u.mx.w1[warp], m.w + (size_t)m.cxt * fx::N_IN1, lane);
    if (lane == 0) sh.u.mx.w_set[warp] = m.cxt;
    fx_copy_words(sh.u.mx.w2, sh.S.mix[10].w, sizeof(short) * FX_FIN_SETS * fx::N_IN2, tid);
    fx_copy_words(sh.u.mx.w2[FX_FIN_SETS], sh.S.mix[11].w, sizeof(short) * fx::N_IN2, tid);
  }
  jit_cluster_sync(cooperative_groups::this_cluster(), JIT_HERE);   // the barriers exist before the other CTA arrives on them
  return r;
}
// The mixer CTA owns mix[], the APMs, the failure history, pr, in2 and codes; the model CTA everything else. The model CTA
// writes the whole block, then the mixer CTA writes its fields over it.
__device__ __forceinline__ void fx_store(FxShared& sh, fx::State* g, const FxGlobals& r, int tid, int rank) {
  using fx::State;
  JIT_SYNCTHREADS();
  const int warp = tid >> 5, lane = tid & 31;
  if (rank == 0) {
    if (tid == 0) { sh.S.text = r.gx; sh.S.T = r.gT; }
    JIT_SYNCTHREADS();
    fx_copy_words(g, &sh.S, sizeof(State), tid);
    fx_copy_words(r.gx, &sh.u.md.X, sizeof(fx::TextState), tid);
  } else {
    fx_row_store(sh.S.mix[warp].w + (size_t)sh.u.mx.w_set[warp] * fx::N_IN1, sh.u.mx.w1[warp], lane);
    fx_copy_words(sh.S.mix[10].w, sh.u.mx.w2, sizeof(short) * FX_FIN_SETS * fx::N_IN2, tid);
    fx_copy_words(sh.S.mix[11].w, sh.u.mx.w2[FX_FIN_SETS], sizeof(short) * fx::N_IN2, tid);
  }
  jit_cluster_sync(cooperative_groups::this_cluster(), JIT_HERE);   // the model CTA's block is out before the mixer CTA's fields
  if (rank == 1) {
    static_assert(offsetof(State, fails) % 4 == 0 && offsetof(State, in2) % 4 == 0 && offsetof(State, codes) % 4 == 0 &&
                  offsetof(State, mix) % 4 == 0 && offsetof(State, apm) % 4 == 0, "owned fields are copied word by word");
    if (tid == 0) { g->pr = sh.S.pr; g->fails = sh.S.fails; g->failz = sh.S.failz; g->failcount = sh.S.failcount; }
    fx_copy_words(g->in2, sh.S.in2, sizeof(sh.S.in2), tid);
    fx_copy_words(g->codes, sh.S.codes, sizeof(sh.S.codes), tid);
    fx_copy_words(g->mix, sh.S.mix, sizeof(sh.S.mix), tid);
    fx_copy_words(g->apm, sh.S.apm, sizeof(sh.S.apm), tid);
  }
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


// Model CTA, one bit: FXCM::Perceive(bit) (fxcmv1.cpp:4909-4912 -> update1 :4758) without the mixers, then the handover
// into ring slot t % FX_RING of the mixer CTA.
__device__ void fx_model_bit(FxShared& sh, FxSlot* ring, u32 t, int y, int lstmpr, int lstmex, int tid) {
  using namespace fx;
  State& S = sh.S;
  const int warp = tid >> 5, lane = tid & 31;
#ifdef FX_PROF
  if (tid == 0) { sh.prof_t = clock64(); sh.prof_row = (S.bpos == 7) ? 0 : 1; }
#endif
  // ---- A: bookkeeping and (byte boundary) the text analysis
  if (tid == 0) {
#ifdef FX_PROF
    const long long t0 = clock64();
    bit_head_model(S, y, lstmpr, lstmex);
    const long long t1 = clock64();
    bit_prepare_model(S);
    atomicAdd(&g_fx_prof[sh.prof_row][12], (unsigned long long)(t1 - t0));
    atomicAdd(&g_fx_prof[sh.prof_row][13], (unsigned long long)(clock64() - t1));
#else
    bit_head_model(S, y, lstmpr, lstmex); bit_prepare_model(S);
#endif
  }
  if (tid >= 32 && tid < 32 + N_MAPS) { sh.u.md.clash[tid - 32] = 0; sh.u.md.res[tid - 32] = 0; }
  for (int k = tid; k < FX_SEEN; k += FX_THREADS) sh.u.md.seen[k] = 0ull;
  JIT_SYNCTHREADS();
  FX_T(0);
  // ---- B: the units' slices of the vectors
  if (warp == FX_WARPS - 1) {
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
      const int n = map_touched(S, id, i, sh.u.md.ids[tid]);
      if (n && fx_claim(sh.u.md.seen, id, sh.u.md.ids[tid], n)) sh.u.md.clash[id] = 1;
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
  if (tid == 0) CENSUS_FX_BIT(S.map[0].t, sh.u.md.clash);   // the bit's verdicts are final here
  FX_T(2);
  // ---- D: the map contexts
  if (tid < FX_MAP_LANES) {
    const int id = tid >> 3, i = tid & 7;
    Out o; o.n = S.in1; o.codes = S.codes; o.ni = S.in_off[U_MAP0 + id]; o.ei = S.ex_off[U_MAP0 + id];
    if (!sh.u.md.clash[id]) {
      if (i < S.map[id].cn && map_ctx_bit(S, id, i, o)) atomicAdd(&sh.u.md.res[id], 1u);
    } else if (i == 0) {      // two contexts in one bucket: this map in order, on one lane
      u32 r = 0;
      const int cn = S.map[id].cn;
      for (int k = 0; k < cn; ++k) r += map_ctx_bit(S, id, k, o);
      sh.u.md.res[id] = r;
    }
  }
  JIT_SYNCTHREADS();
  FX_T(3);
  // ---- E: map epilogues, weight-set selection
  if (warp == 0) {
    if (lane < N_MAPS) map_finish(S, lane, sh.u.md.res[lane]);
    __syncwarp();
    if (lane == 0) bit_select_model(S);
  }
  JIT_SYNCTHREADS();
  FX_T(4);
  // ---- handover: every warp writes its share of the slot and arrives on the slot's full barrier
  const int slot = (int)(t % FX_RING);
  if (t >= FX_RING) mbar_wait(&sh.u.md.empty[slot], (t / FX_RING - 1) & 1, JIT_HERE);
  FX_T(5);
  FxSlot& d = ring[slot];
  constexpr int N1 = N_IN1 / 8, NC = (N_OUT + 1) / 8;
  for (int q = tid; q < N1 + NC; q += FX_THREADS) {
    if (q < N1) reinterpret_cast<uint4*>(d.in1)[q] = reinterpret_cast<const uint4*>(S.in1)[q];
    else reinterpret_cast<uint4*>(d.codes)[q - N1] = reinterpret_cast<const uint4*>(S.codes)[q - N1];
  }
  if (tid < N_MIX) d.cxt[tid] = S.mix[tid].cxt;
  if (tid == 0) {     // lane 0 changes these first on the next bit
    const TextState& X = sh.u.md.X;
    d.ei = S.ex_off[N_UNITS]; d.lstmpr = S.lstmpr; d.lstmex = S.lstmex; d.c0 = S.c0; d.rate = S.rate;
    d.ah1 = X.ah1; d.ah2 = X.ah2; d.s2b = X.s2b; d.s2bR = X.s2bR; d.s3bR = X.s3bR; d.x5 = X.x5;
  }
  __syncwarp();
  if (lane == 0) mbar_arrive_remote(&sh.u.mx.full[slot], 1, JIT_HERE);
  __syncwarp();
  FX_T(6);
}

// The tail of a bit on one warp of the mixer CTA (fxcm_model.h bit_tail): squash of the ten first-layer outputs, the two
// final mixers, the six APMs (three dependent levels), the exports.
__device__ void fx_tail_warp(FxShared& sh, const FxSlot& in, int lane) {
  using namespace fx;
  State& S = sh.S;
  const fx::Tables& T = *S.T;
  const unsigned full = 0xffffffffu;
  const int ei = in.ei;
  if (lane < 10) {
    int dp = (int)((u32)sh.u.mx.dots[lane] * (u32)T.mix_shift[lane]) >> 11;
    dp = clp(dp);
    const int pr = squash(T, dp);
    S.mix[lane].pr = pr;
    S.in2[lane] = (short)dp;
    S.codes[ei + lane] = (u16)pr;
  } else if (lane == 10) S.in2[10] = (short)(stretch(T, in.lstmpr) / 2);
  __syncwarp();
  int acc = 0;
  {
    const int i = 10 + (lane >> 3), k = 2 * (lane & 7);
    if (lane < 16) { const short* w = sh.u.mx.w2[(i - 10) * FX_FIN_SETS + S.mix[i].cxt]; acc = dot_pair(S.in2 + k, w + k); }
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
  const int y = S.y, c0 = in.c0, rate = in.rate;
  const u32 fails = S.fails;
  // level 1: three APMs refine pr
  int a = 0;
  if (lane == 0) a = apm_p(T, S.apm[0], pr, (u32)c0, 3, y);
  else if (lane == 1) a = apm_p(T, S.apm[1], pr, ((u32)(c0 * 8) ^ hash3(29, S.failz & 2047)) & 0xffff, rate + 1, y);
  else if (lane == 2) a = apm_p(T, S.apm[2], pr, ((u32)(c0 * 32) ^ in.ah2) & 0xffff, rate, y);
  const int pu0 = (__shfl_sync(full, a, 0) + 7 * pr + 4) >> 3;
  const int pv0 = __shfl_sync(full, a, 1), pt = __shfl_sync(full, a, 2);
  // level 2
  int b = 0;
  if (lane == 0) b = apm_p(T, S.apm[3], pu0, ((u32)(c0 * 2) ^ in.ah1) & 0x3ffff, rate, y);
  else if (lane == 1) {
    if (fails & 255) b = apm_p(T, S.apm[4], pv0, hash3((u32)c0, in.s2b & 0xfffc, in.s3bR & 0x1ff) & 0x3ffff, rate, y);
    else b = apm_p(T, S.apm[4], pv0, hash3((u32)c0, (in.s2bR & 0xfffc) + 0x10000, in.s3bR & 0x1ff) & 0x3ffff, rate, y);
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
    pz = apm_p(T, S.apm[5], pu, ((u32)(c0 * 4) ^ hash3((u32)imin(9, pz), in.x5 & 0x80ff)) & 0x3ffff, rate, y);
    int fin;
    if (fails & 255) fin = (pt * 6 + pu + pv * 11 + pz * 14 + 31) >> 5;
    else fin = (pt * 4 + pu * 5 + pv * 12 + pz * 11 + 31) >> 5;
    u16* c = S.codes + ei + 10;
    c[0] = (u16)pr; c[1] = (u16)pu; c[2] = (u16)pv0; c[3] = (u16)pv; c[4] = (u16)pt; c[5] = (u16)pz; c[6] = (u16)fin;
    S.pr = fin;
  }
}

// Mixer CTA, one bit: the error terms, the failure history and the SGD of the rows selected for bit t-1 on its inputs
// `x_prev` need only the bit; then slot t's selectors, the row moves, the ten dot products and the tail.
__device__ void fx_mixer_bit(FxShared& sh, u32 t, int y, const short* x_prev, int tid) {
  using namespace fx;
  State& S = sh.S;
  const int warp = tid >> 5, lane = tid & 31;
#ifdef FX_PROF
  if (tid == 0) { sh.prof_t = clock64(); sh.prof_row = (S.bpos == 7) ? 0 : 1; }
#endif
  if (tid == 0) {       // its own copy of the bookkeeping gives the byte end and bpos; the model CTA owns those fields
    bit_head_mixer(S, y, bit_head_model(S, y, S.lstmpr, S.lstmex));
    bit_fail_history(S);
  }
  JIT_SYNCTHREADS();
  FX_T(16);
  // SGD on the cached rows (Mixer1::update) and on the final mixers' rows
  for (int idx = tid; idx < 10 * (N_IN1 / 8); idx += FX_THREADS) {
    const int i = idx >> 6, q = idx & 63;
    const int err = S.mix[i].err;
    if (!err) continue;
    uint4* wp = reinterpret_cast<uint4*>(&sh.u.mx.w1[i][q * 8]);
    uint4 wv = *wp;
    const uint4 xv = *reinterpret_cast<const uint4*>(&x_prev[q * 8]);
    short* w = reinterpret_cast<short*>(&wv);
    const short* x = reinterpret_cast<const short*>(&xv);
#pragma unroll
    for (int e = 0; e < 8; ++e) w[e] = train_one(x[e], w[e], err);
    *wp = wv;
  }
  if (warp == FX_WARPS - 1) {
    const int i = 10 + (lane >> 4);
    const MixState& m = S.mix[i];
    if (m.err) { short* w = sh.u.mx.w2[(i - 10) * FX_FIN_SETS + m.cxt]; const int k = lane & 15; w[k] = train_one(S.in2[k], w[k], m.err); }
  }
  JIT_SYNCTHREADS();
  if (t > 0 && tid == 0) mbar_arrive_remote(&sh.u.md.empty[(t - 1) % FX_RING], 0, JIT_HERE);   // x_prev was slot t-1's
  FX_T(17);
  const int slot = (int)(t % FX_RING);
  const FxSlot& in = sh.u.mx.ring[slot];
  mbar_wait(&sh.u.mx.full[slot], (t / FX_RING) & 1, JIT_HERE);
  FX_T(18);
  for (int q = tid; q < in.ei; q += FX_THREADS) S.codes[q] = in.codes[q];
  if (tid < N_MIX && tid != 9) S.mix[tid].cxt = in.cxt[tid];
  if (tid == 0) { S.lstmex = in.lstmex; bit_select_mixer(S); }
  JIT_SYNCTHREADS();
  // the ten 512-wide dot products over the cached rows (a selector that moved: write back, load)
  {
    const MixState& m = S.mix[warp];
    short* row = sh.u.mx.w1[warp];
    const int old = sh.u.mx.w_set[warp];
    if (old != m.cxt) {
      fx_row_store(m.w + (size_t)old * N_IN1, row, lane);
      fx_row_load(row, m.w + (size_t)m.cxt * N_IN1, lane);
      __syncwarp();
      if (lane == 0) sh.u.mx.w_set[warp] = m.cxt;
    }
    int acc = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint4 wv = *reinterpret_cast<const uint4*>(row + (lane + 32 * h) * 8);
      const uint4 xv = *reinterpret_cast<const uint4*>(in.in1 + (lane + 32 * h) * 8);
      const short* w = reinterpret_cast<const short*>(&wv);
      const short* x = reinterpret_cast<const short*>(&xv);
#pragma unroll
      for (int e = 0; e < 8; e += 2) acc += dot_pair(x + e, w + e);
    }
    acc = __reduce_add_sync(0xffffffffu, acc);
    if (lane == 0) sh.u.mx.dots[warp] = acc;
  }
  JIT_SYNCTHREADS();
  FX_T(19);
  // squash, final mixers, APMs, exports
  if (warp == 0) fx_tail_warp(sh, in, lane);
  JIT_SYNCTHREADS();
  FX_T(20);
}

// Bulk: cluster b (CTAs 2b, 2b+1) serves stream b of the launch group. The mixer CTA writes ext[t][0..430] for every bit t
// of the sub-chunk (the codes the model holds BEFORE perceiving bit t).
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(FX_THREADS, 1) fxcm_kernel(const ChunkArgs* __restrict__ args_all) { jit_entry(JK_FXCM);
  extern __shared__ __align__(16) unsigned char fx_raw[];
  FxShared& sh = *reinterpret_cast<FxShared*>(fx_raw);
  const ChunkArgs a = args_all[blockIdx.x >> 1];
  if (a.fx == nullptr) return;
  const int tid = threadIdx.x;
  const int rank = (int)cooperative_groups::this_cluster().block_rank();
  const FxGlobals gl = fx_load(sh, a.fx, tid, rank);
  const u32 n_bits = a.n_bytes * 8;
  if (rank == 0) {
    FxSlot* ring = cooperative_groups::this_cluster().map_shared_rank(&sh, 1)->u.mx.ring;
    for (u32 t = 0; t < n_bits; ++t) {
      const int y = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      int lstmpr = 0, lstmex = 0;
      if (!a.pretrain) { const u32 v = a.lstm_fx[t]; lstmpr = (int)(v & 0xffff); lstmex = (int)(v >> 16); }
      else { lstmpr = sh.S.lstmpr; lstmex = sh.S.lstmex; }
      fx_model_bit(sh, ring, t, y, lstmpr, lstmex, tid);
    }
  } else {
    for (u32 t = 0; t < n_bits; ++t) {
      if (!a.pretrain) {
        u16* out = a.ext_gen + (size_t)t * N_EXT;
        for (int k = tid; k < fx::N_OUT; k += FX_THREADS) out[k] = sh.S.codes[k];
      }
      const int y = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      fx_mixer_bit(sh, t, y, t == 0 ? sh.S.in1 : sh.u.mx.ring[(t - 1) % FX_RING].in1, tid);
    }
  }
  fx_store(sh, a.fx, gl, tid, rank);
}

// Lock-step: one bit per launch (the decoder's order), queued behind the mixer / LSTM update of the same bit, a one-slot
// handover. The model CTA first takes the LSTM's read-out of the NEXT bit (ByteMixer::Predict + Discretize,
// predictor.cpp:462-465); the codes for the next Predict() land in ext_bit[0..430].
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(FX_THREADS, 1) fxcm_bit_kernel(StreamState* st, fx::State* g, int y, int pretrain, u16* ext_bit, const u32* dbit) { jit_entry(JK_FXCM_BIT);
  if (dbit) y = (int)dbit[0];
  extern __shared__ __align__(16) unsigned char fx_raw[];
  FxShared& sh = *reinterpret_cast<FxShared*>(fx_raw);
  const int tid = threadIdx.x;
  const int rank = (int)cooperative_groups::this_cluster().block_rank();
  const FxGlobals gl = fx_load(sh, g, tid, rank);
  if (rank == 0) {
    float* probs = reinterpret_cast<float*>(sh.u.md.seen);     // free until fx_model_bit clears it: the 256 probabilities arrive side by side
    if (!pretrain && tid < 256) probs[tid] = st->lstm.bm.probs[tid];
    JIT_SYNCTHREADS();
    if (tid == 0) {
      if (pretrain) { sh.u.md.lstm[0] = sh.S.lstmpr; sh.u.md.lstm[1] = sh.S.lstmex; }
      else {
        const ByteModelState& b = st->lstm.bm;
        int ex;
        const float p = bytemodel_predict(probs, b.bot, b.top, &ex);     // the sums stay one serial chain (byte-model.cpp:8-24)
        sh.u.md.lstm[0] = (int)(u32)XM_FADD(1.0f, XM_FMUL(4094.0f, p));
        sh.u.md.lstm[1] = ex;
      }
    }
    JIT_SYNCTHREADS();
    const int lstmpr = sh.u.md.lstm[0], lstmex = sh.u.md.lstm[1];
    JIT_SYNCTHREADS();
    fx_model_bit(sh, cooperative_groups::this_cluster().map_shared_rank(&sh, 1)->u.mx.ring, 0, y, lstmpr, lstmex, tid);
  } else {
    fx_mixer_bit(sh, 0, y, sh.S.in1, tid);
    if (ext_bit) for (int k = tid; k < fx::N_OUT; k += FX_THREADS) ext_bit[k] = sh.S.codes[k];
  }
  fx_store(sh, g, gl, tid, rank);
}

}  // namespace cmixb200
