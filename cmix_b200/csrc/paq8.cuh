// cmix_b200/csrc/paq8.cuh — the resident PAQ8 model on the device (SURVEY §8 row a13).
//
// One cluster of two CTAs per stream evaluates paq8_top.h's `bit()`; 12 warps of the first spread the models over lanes:
//  * every context of every context map is a lane (210 lanes for the sixteen 7-slot maps on warps 0-6, 63 for the three
//    history maps on warps 7-8): bucket probe, bit-history step, state maps and the 5 / 7 mixer inputs of a context are
//    independent of the other contexts of its map as long as they touch different 64-byte buckets this bit. That is CHECKED
//    per bit (touched_buckets, including the buckets a deferred history write-back will reach; on the staying bits of the
//    7-slot maps, bpos 1, 3, 4, 6, 7, the slots a context reads and writes, cm_slot_keys). In a 7-slot map with a clash
//    only the contexts that share a key with another are evaluated by one lane in the reference's order (p8_number); a
//    history map with a clash is evaluated by one lane whole. On a staying bit a 7-slot lane reads its slot and run record
//    from a copy in shared memory (P8CmCache).
//  * the one global coupling of the 7-slot maps, the shared pseudo-random sequence that ages high-count states
//    (paq8.cpp:1075), is resolved between the two passes: the draws themselves depend on the generator only, so one warp
//    computes as many as a bit can take during the bookkeeping, 24 at a time (the generator is a lagged XOR:
//    x[i] = x[i-24] ^ x[i-55]); pass 1 computes each context's aged state and flags the contexts that draw; a flagged
//    context's draw is the one its rank among the flagged contexts in program order selects (ballot masks + popcounts), and
//    pass 2 applies them. On a bit with a clashing map one lane first walks the contexts that share a key, setting their
//    real flags, so that every rank counts final flags.
//  * the match models, the DMC forest, the run maps and the direct maps run one unit per lane beside the context maps; on a
//    bit inside a byte all of this is three phases (probe / number / apply), and the units take warps 9-11 and the text
//    chain's idle warps 13-15, one function per warp and phase (lane map: P8_W_*). The bit that starts a byte
//    first computes the new contexts, as chains of warps that do not wait for each other: the D-chain (order-N and x86
//    contexts, their history maps, the match model, then the sparse and record models, which consume what the order-N map
//    and the match model produce in the same bit), the word model, the text model with its stemmers, the three OLS
//    predictors (one warp each: rank-1 covariance update with coalesced columns, Cholesky with a row per lane in
//    registers, substitutions in the reference's summation order) and the nest / indirect / XML / distance / record1
//    models. They meet once, before the common probe / number / apply of the sixteen 7-slot maps.
//  * the mixer and the SSE stage run one or more bits behind the models on a second CTA of a 2-CTA cluster (nothing the
//    models compute reads them back: the mixer's output feeds only the SSE stage, `st_misses` and selector set 26). The
//    model CTA (rank 0) hands each bit over through a ring of P8_RING slots in the mixer CTA's shared memory (inputs,
//    their codes, the 28 selectors, the SSE context), one full / one empty mbarrier per slot, and blocks only when the
//    ring is full. The mixer CTA (rank 1) trains the sets picked for bit t-1 on its inputs as soon as bit t is known,
//    then runs bit t's 28 dot products, the final mixer and the SSE stage, and writes the 1591-code rows.
//  * the 28 selected int16 weight sets (1552 weights each) are CACHED in the mixer CTA's shared memory from the dot product
//    of one bit to the SGD step of the next and written back to HBM only when a selector moves to another set; dot
//    products and SGD use all 512 lanes (integer sums: exact under any association).
// The 55 KB state block and the hot read-only tables (21 KB) live in the shared memory of both CTAs for the launch, the
// 87 KB weight cache and the ring in the mixer CTA's; the ~10 GB of model memory stays in HBM. Each CTA writes back the
// fields of the state block it owns (p8_leave).
// PAQ8 is a producer like FXCM: it depends on the coded bytes only and writes 1591 codes per bit into the `ext` scratch.
#pragma once
#include <cooperative_groups.h>
#include "jitter.cuh"
#include "cluster_mbar.cuh"
#ifdef P8_PROF
namespace cmixb200 { __host__ __device__ inline void p8_leg(int k); }
#define P8_LEG(k) ::cmixb200::p8_leg(k)
#endif
#include "paq8_top.h"
#include "state.h"
#include "census.cuh"

namespace cmixb200 {

enum { P8_SEEN = 4096, P8_RING = 4 };

// -DP8_PROF: lane 0 of each CTA accumulates the cycles between phase boundaries (byte-boundary bits and the others apart):
// slots 0-11 the model CTA (2: from the end of the bookkeeping to the join of a byte boundary's chains, 10: waiting for a free
// ring slot), 16-19 the mixer CTA (16: waiting for a full one). 24+: inside a byte the per-warp times of the probe (24 + warp)
// and apply (48 + warp) phases; on a byte boundary the time from the end of the bookkeeping at which a chain got to a point
// (24-30: warps 0-6 done, 31-36: the D-chain's steps, 38: the text chain done). 64+: the longest lane of each single-lane
// unit, from its own start to its end (P8_U). Labels in tools/prof_build.py.
// Rows: 0 byte-boundary bits, 1 the others; the model CTA sums a bit in shared memory and also adds the bits inside a byte
// by class into rows 2-5 (2 + 2 * "bpos 2 or 5: the 7-slot maps move to a new bucket" + "a 7-slot map clashes"). Slot
// P8_PROF_N counts the model CTA's bits of a row. 88+: the legs of a 7-slot map context's bit (P8_LEG: the longest lane of the
// bit, each leg apart; not lane 0 on a bit with a clash, which walks the maps): probe 88 the state read, 89 touched_buckets,
// 90 p8_claim; apply 91 the draw, 92 the store and the move to the next cell (bucket_find at bpos 2, 5, 0), 93 the run
// record's input, 94 the cell's state and its StateMap load, 95 the other exports. On a staying bit leg 88 includes the
// start of both StateMap loads and 94 also counts the probe's wait for them after p8_claim. By the bpos of a bit with a
// 7-slot clash: 96 + bpos the numbering's cycles (p8_number and the barrier behind it), 104 + bpos the bits, 112 + bpos
// the contexts it walked (grouped).
#ifdef P8_PROF
enum { P8_PROF_ROWS = 6, P8_PROF_SLOTS = 128, P8_PROF_UNIT = 64, P8_PROF_LEG = 88, P8_PROF_NUMBER = 96, P8_PROF_N = P8_PROF_SLOTS - 1 };
__device__ unsigned long long g_p8_prof[P8_PROF_ROWS][P8_PROF_SLOTS];
#define P8_T(k) do { if (tid == 0) { const long long now_ = clock64(); atomicAdd(&sh.prof_dst[k], (unsigned long long)(now_ - sh.prof_t)); sh.prof_t = now_; } } while (0)
#define P8_M0 const long long m0_ = clock64()
#define P8_M(slot) atomicAdd(&sh.prof_dst[slot], (unsigned long long)(clock64() - m0_))
#define P8_C(slot, n) atomicAdd(&sh.prof_dst[slot], (unsigned long long)(n))
#define P8_U0 const long long u0_ = clock64()
#define P8_U(g) atomicMax(&sh.prof_dst[P8_PROF_UNIT + (g)], (unsigned long long)(clock64() - u0_))
#else
#define P8_T(k) do { } while (0)
#define P8_M0 do { } while (0)
#define P8_M(slot) do { } while (0)
#define P8_C(slot, n) do { } while (0)
#define P8_U0 do { } while (0)
#define P8_U(g) do { } while (0)
#endif
enum { P8_THREADS = 512, P8_WARPS = 16, P8_MAP_THREADS = 384, P8_MAP_WARPS = 12, P8_N_CM = 16, P8_N_CM2 = 3, P8_CM_LANES = 210, P8_CM2_LANES = 63, P8_N_UNITS = 53,
       P8_CM2_TID0 = 224, P8_TID_PIC = 287, P8_TID_MATCH = 288, P8_TID_W10 = 320, P8_TID_W11 = 352 };
// Inside a byte warps 0-6 hold the 7-slot maps' lanes and warps 7-8 the history maps'; each of warps 9-11 and 13-15 runs one
// function of the single-lane units per phase (lanes of one warp that diverge into different functions run one after another):
//   probe   9 match_core   10 dmc_st x10   11 smatch_head   13 pic_core   14 record_pre   15 rcm_mix x3
//   apply   9 imap_mix x3  10 pic_unit x3  11 DMC combination (and the constant input)
//           13 sm32_p x5   14 scm_mix x18  15 stm_mix x13   (the maps behind the match, record, sparse match, sparse1 and
//                                                             linear models, and the order-0/1 inputs)
// warp 12 computes ModelStats and selector sets, as on every bit. Warps 13-15 skip the numbering of a clashing bit and the
// barrier behind the maps' apply phase, so their apply overlaps both.
enum { P8_W_MATCH = 9, P8_W_DMC = 10, P8_W_SMATCH = 11, P8_W_PIC = 13, P8_W_RECORD = 14, P8_W_RCM = 15,
       P8_W_IMAP = 9, P8_W_PICU = 10, P8_W_DMCMIX = 11, P8_W_SM32 = 13, P8_W_SCM = 14, P8_W_STM = 15 };
// Who computes the new contexts on the bit that starts a byte. A long single-lane job has a warp to itself while it runs
// (lanes of one warp that diverge into different jobs run one after another):
//   warps 0-2    the OLS predictors, lane 0 then the direct map behind its prediction
//   warp 3       XML (lane 0)                     warp 4   distance, record1 (lane 0)
//   warp 5       the word model: state and stemmer on lane 0, the 57 contexts on all lanes
//   warp 6       nest, indirect, the two fixed linear predictions and their maps (lane 0)
//   warps 7-11   the D-chain: order-N contexts (lane 0 of 7) and x86 contexts (lane 0 of 9); probe and apply of those two
//                history maps with the single-lane units; then sparse (lane 0 of 9), sparse1 (lane 0 of 10), record (lane 0 of 11)
//   warp 12      ModelStats and selector sets, as on every bit
//   warps 13-15  the text chain: state on lane 0 of 13, a stemmer on lane 0 of each, the 33 contexts on warp 13
// Then all of warps 0-11 as inside a byte, with the text history map's lanes (warps 7-8) beside the 7-slot maps.

// One bit handed from the model CTA to the mixer CTA: what the models produced and the context the SSE stage reads.
struct P8Slot {
  alignas(16) short tx[p8::N_IN];    // mixer inputs [0, nx), zero-padded to a multiple of 8
  alignas(16) u16 codes[p8::N_IN];   // their exported codes [0, n2)
  int cxt[p8::N_SETS];               // the selected weight sets; set 26 is the mixer CTA's (it depends on its last prediction)
  int n2, nx, ncxt, base;
  int c0, bpos, blpos, st_type; u32 c4, st_match_length;
  u8 c1, st_match_expected, st_text_first, st_text_mask;
  u8 relayout;                       // the set count differs from the previous bit's (ordinary <-> audio mode): p8_relayout
};

// Each 7-slot map lane's copy of the 7 state bytes of its slot (t[cp0 ..]) and the 2 bytes of its run record (t[runp ..]):
// a staying bit (cm_staying) reads only these, so its probe and apply take them from shared memory. Stores go through to
// HBM, which stays the authority. A copy is filled where the lane's bucket line is read anyway: after the lane's apply on a
// move bit (bpos 0, 2, 5), or at the probe of a staying bit while it is invalid. It is valid from the fill until the lane's
// context is walked serially (p8_number) or the launch ends: a context never writes the slot or run record of a context it
// shares no key with, and the walk writes only keys of the contexts it walks.
struct P8CmCache {
  unsigned short sm[P8_CM_LANES][2];    // staying bit: smt[sm_cxt] and smt[the new cell's state], loaded by the probe
  unsigned char slot[P8_CM_LANES][8], run[P8_CM_LANES][2], valid[P8_CM_LANES];
};

struct P8Shared {
  p8::State S;
  alignas(16) unsigned char tab[p8::TABLES_HOT_BYTES];
  alignas(8) unsigned long long full[P8_RING];    // in the mixer CTA: slot i holds a bit (one arrive per model warp)
  unsigned long long empty[P8_RING];              // in the model CTA: the mixer CTA is done with slot i
  // mixer CTA
  int wc_set[p8::N_SETS];
  int dot[p8::N_SETS];
  // model CTA
  int unit_off[P8_N_UNITS + 1];
  // pass-1 results of the 7-slot maps
  short ns[P8_CM_LANES];
  u32 ids[P8_CM_LANES][5];
  u32 ids2[P8_CM2_LANES][5];
  int clash[P8_N_CM], clash2[P8_N_CM2];
  int order, res2[P8_N_CM2];
  p8::WordStats snap;          // the word statistics as the byte found them (sparseModel1 reads them beside the word model's update)
  int dmc_st[10];
  u32 flag_mask[8];            // ballot of "this context draws" per warp of map lanes (p8_number sets the walked contexts' real flags)
  u32 group_mask[8];           // on a bit with a clash: the lanes of clashing maps that share a key with another (p8_number)
#ifdef CMIXB200_CENSUS
  u32 flag_mask1[8];           // flag_mask as pass 1 left it: the census logs pass 1's flags
#endif
  u32 draws[P8_CM_LANES + 6];  // the draws of the bit in order (p8_draw_seq)
  int any_clash, text_pending;
  union {
    struct {                                                    // the model CTA
      unsigned long long seen[P8_SEEN];   // open-addressing set of (map, bucket) pairs touched this bit
      struct { double ch[3][32 * 33]; double pb[3][32]; } ols;   // Cholesky factor rows (padded) and a product buffer; byte boundaries only
                                                                 // (in audio mode `ch` holds two vectors per audio OLS warp)
      P8CmCache cc;
      int ncxt_handed;                    // the selector count of the last bit handed over (P8Slot::relayout)
#ifdef P8_PROF
      long long leg_t[P8_CM_LANES];      // P8_LEG: when a lane's current leg started
#endif
    } md;
    struct {                                                    // the mixer CTA
      alignas(16) short wc[p8::N_SETS][p8::N_IN];   // the weight sets of the pending prediction (slot i holds set wc_set[i])
      P8Slot ring[P8_RING];
    } mx;
  } u;
#ifdef P8_PROF
  long long prof_t; unsigned long long* prof_dst;   // the model CTA: prof_acc; the mixer CTA: its row of g_p8_prof
  unsigned long long prof_acc[P8_PROF_SLOTS];
#endif
};

#ifdef P8_PROF
// k >= 0 ends leg k of the calling lane's context and starts the next; k < 0 starts the first
__host__ __device__ inline void p8_leg(int k) {
#ifdef __CUDA_ARCH__
  extern __shared__ __align__(16) unsigned char p8_raw[];
  P8Shared& sh = *reinterpret_cast<P8Shared*>(p8_raw);
  const int tid = threadIdx.x;
  if (tid >= P8_CM_LANES || (tid == 0 && sh.any_clash)) return;
  const long long now = clock64();
  if (k >= 0) atomicMax(&sh.prof_dst[P8_PROF_LEG + k], (unsigned long long)(now - sh.u.md.leg_t[tid]));
  sh.u.md.leg_t[tid] = now;
#else
  (void)k;
#endif
}
#endif

// program order of the sixteen 7-slot maps, their lane capacity and the number of contexts a full byte sets
__device__ __forceinline__ p8::Cm& p8_cm(p8::State& S, int k) {
  switch (k) {
    case 0: return S.sparse.cm; case 1: return S.sparse1.cm; case 2: return S.distance.cm; case 3: return S.record.cm; case 4: return S.record.cn;
    case 5: return S.record.co; case 6: return S.record.cp; case 7: return S.record1.cm; case 8: return S.record1.cn; case 9: return S.record1.co;
    case 10: return S.record1.cq; case 11: return S.record1.cp; case 12: return S.word.cm; case 13: return S.nest.cm; case 14: return S.indirect.cm;
    default: return S.xml.cm;
  }
}
__device__ __forceinline__ p8::Cm2& p8_cm2(p8::State& S, int k) { return k == 0 ? S.cm : (k == 1 ? S.text.map : S.exe.cm); }
__constant__ unsigned char c_p8_cm_cap[P8_N_CM] = {42, 31, 3, 3, 3, 3, 16, 2, 5, 4, 3, 3, 61, 12, 15, 4};
__constant__ unsigned char c_p8_cm_base[P8_N_CM + 1] = {0, 42, 73, 76, 79, 82, 85, 101, 103, 108, 112, 115, 118, 179, 191, 206, 210};
__constant__ unsigned char c_p8_cm_full[P8_N_CM] = {42, 29, 3, 3, 3, 3, 16, 2, 5, 4, 3, 3, 57, 12, 15, 4};
__constant__ unsigned char c_p8_cm_unit[P8_N_CM] = {9, 10, 18, 20, 21, 22, 23, 36, 37, 38, 39, 40, 41, 42, 43, 45};
__constant__ unsigned char c_p8_cm2_cap[P8_N_CM2] = {10, 33, 20};
__constant__ unsigned char c_p8_cm2_unit[P8_N_CM2] = {3, 46, 47};
// unit u of the mixer-input order (paq8_top.h context_model): >= 0: fixed number of inputs, -1-k: 7-slot map k, -20-k: history map k
__constant__ signed char c_p8_unit_kind[P8_N_UNITS] = {
    1, 1, 1, -20, 1, 1, 1, 17, 11, -1, -2, 2, 2, 2, 2, 2, 2, 2, -3, 3, -4, -5, -6, -7, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2,
    -8, -9, -10, -11, -12, -13, -14, -15, 6, -16, -21, -22, 2, 2, 2, 2, 2};

// In audio mode (paq8_top.h audio8_mode) the inputs are those of units 0-7, audio8bModel's 33 stationary maps in the place of
// unit 8 and the record model's units 20-35; the other units add nothing.
__device__ __forceinline__ int p8_unit_count(p8::State& S, int u, bool byte_start, bool audio) {
  if (audio && u == 8) return 2 * p8::AUDIO_N_SCM;
  if (audio && ((u > 8 && u < 20) || u > 35)) return 0;
  const int kind = c_p8_unit_kind[u];
  if (kind >= 0) return kind;
  if (kind <= -20) { const int k = -20 - kind; return 7 * (byte_start ? (int)c_p8_cm2_cap[k] : p8_cm2(S, k).index); }
  const int k = -1 - kind;
  return 5 * (byte_start ? (int)c_p8_cm_full[k] : p8_cm(S, k).cn);
}

// unit_off[]: the mixer-input offset of every unit (one warp, prefix sums)
__device__ __noinline__ void p8_unit_offsets(P8Shared& sh, int lane, bool byte_start, bool audio) {
  const unsigned full = 0xffffffffu;
  const int a = p8_unit_count(sh.S, lane, byte_start, audio);
  const int b = lane + 32 < P8_N_UNITS ? p8_unit_count(sh.S, lane + 32, byte_start, audio) : 0;
  int ia = a, ib = b;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int va = __shfl_up_sync(full, ia, d), vb = __shfl_up_sync(full, ib, d);
    if (lane >= d) { ia += va; ib += vb; }
  }
  const int ta = __shfl_sync(full, ia, 31);
  sh.unit_off[lane] = ia - a;
  if (lane + 32 <= P8_N_UNITS) sh.unit_off[lane + 32] = ta + ib - b;
}

__device__ __forceinline__ p8::Out p8_out(P8Shared& sh, int offset) { p8::Out o; o.T = sh.S.T; o.tx = sh.S.m.tx; o.codes = sh.S.codes; o.n = offset; return o; }
// audio8bModel's stationary map q, its inputs in the place of unit 8 (p8_unit_count)
__device__ __noinline__ void p8_audio_scm(P8Shared& sh, int q) { p8::Out o = p8_out(sh, sh.unit_off[8] + 2 * q); p8::audio8b_scm(sh.S, o, q); }

__device__ __forceinline__ void p8_copy_words(void* dst, const void* src, size_t bytes, int tid) {
  u32* d = (u32*)dst; const u32* s = (const u32*)src;
  for (size_t i = tid; i < bytes / 4; i += P8_THREADS) d[i] = s[i];
}
static_assert(sizeof(p8::State) % 4 == 0, "state block is copied word by word");

// One OLS predictor of the linear-prediction model at a byte boundary, on one warp: OLS::Update(val) with the byte just
// coded, then Add() of the 32 new taps and Predict() (paq8_top.h ols_update / linear_predict, reference :4476-4502).
// Element-wise steps use any lane mapping; every SUM runs in the reference's order:
//  * covariance: lane = column, 32 coalesced rows (the matrix stays exactly symmetric, so the lane also holds row `lane`);
//  * Cholesky: lane r keeps row r in registers; column c takes row c's finished entries from shared memory;
//  * forward substitution column by column (row i subtracts w[0..i-1] in ascending order), backward substitution row by
//    row with the products gathered in shared memory and summed in ascending order.
__device__ __noinline__ void p8_ols_byte_warp(P8Shared& sh, int k, int lane) {
  using namespace p8;
  State& S = sh.S;
  LinearM& M = S.linear;
  const double lambda = 0.995, nu = 0.001, one_minus = 1.0 - 0.995;
  double* blk = M.ols + (size_t)k * OLS_STRIDE;
  double* x = blk; double* w = blk + 32; double* b = blk + 64; double* cov = blk + 96;
  double* chs = sh.u.md.ols.ch[k]; double* pb = sh.u.md.ols.pb[k];
  double* row = chs + lane * 33;
  const unsigned full = 0xffffffffu;
  const double val = (double)(u8)buf(S, 1);
  const double xl = x[lane];
  int km = M.ols_km[k] + 1;
  const bool solve = km >= 4;
  {
    double c[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) c[j] = cov[j * 32 + lane];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const double xj = __shfl_sync(full, xl, j);
      const double v = P8_DADD(P8_DMUL(lambda, c[j]), P8_DMUL(one_minus, P8_DMUL(xj, xl)));
      cov[j * 32 + lane] = v;
      if (solve) row[j] = (j == lane) ? P8_DADD(v, nu) : v;     // the matrix is exactly symmetric: column `lane` is row `lane`
    }
  }
  double bl = b[lane];
  bl = P8_DADD(P8_DMUL(lambda, bl), P8_DMUL(one_minus, P8_DMUL(xl, val)));
  b[lane] = bl;
  double wl = w[lane];
  if (solve) {
    __syncwarp();
    bool fail = false;
    for (int col = 0; col < 32 && !fail; ++col) {
      const double* rc = chs + col * 33;
      double s = row[col];
#pragma unroll 4
      for (int q = 0; q < col; ++q) s = P8_DSUB(s, P8_DMUL(row[q], rc[q]));
      const double d = __shfl_sync(full, s, col);
      if (d > 1E-8) {
        const double dd = P8_DSQRT(d);
        if (lane >= col) row[col] = (lane == col) ? dd : P8_DDIV(s, dd);
      } else fail = true;
      __syncwarp();
    }
    if (!fail) {
      double sum = bl;
      for (int q = 0; q < 32; ++q) {
        const double wq = P8_DDIV(__shfl_sync(full, sum, q), chs[q * 33 + q]);
        if (lane == q) wl = wq;
        sum = P8_DSUB(sum, P8_DMUL(row[q], wq));          // rows below q; the others hold values nobody reads
      }
      const double zl = wl;
      for (int i = 31; i >= 0; --i) {
        pb[lane] = P8_DMUL(row[i], wl);                   // ch[lane][i] * w[lane], read for lane > i only
        __syncwarp();
        double s = __shfl_sync(full, zl, i);
#pragma unroll 4
        for (int j = i + 1; j < 32; ++j) s = P8_DSUB(s, pb[j]);
        const double wi = P8_DDIV(s, chs[i * 33 + i]);
        if (lane == i) wl = wi;
        __syncwarp();
      }
      w[lane] = wl;
    }
    km = 0;
  }
  // Add() the taps of this predictor and Predict()
  const int i1 = lane + 1;
  const double xn = (double)(u8)buf(S, k == 0 ? i1 : (k == 1 ? 2 * i1 - 1 : 2 * i1));
  x[lane] = xn;
  pb[lane] = P8_DMUL(wl, xn);
  __syncwarp();
  if (lane == 0) {
    double sum = 0.;
    for (int i = 0; i < 32; ++i) sum = P8_DADD(sum, pb[i]);
    M.prd[k] = (u8)clip8((int)P8_FLOOR(sum));
    M.ols_km[k] = km;
  }
  __syncwarp();
}

// One OLS predictor k of audio8bModel at a byte boundary, on one warp (paq8_top.h audio8b_ols): OLS::Update(s) on channel
// pCh, then the taps and Predict() on channel ch. Element-wise steps use any lane mapping; every SUM runs in the reference's
// order. Rows go to lanes round robin; sums and products of a step meet in two shared-memory vectors of the warp (u, v):
//  * covariance and b: lane = column (the matrix stays exactly symmetric);
//  * Factor() column by column, the rows of a column side by side, each inner sum over k < c in ascending order. The factor
//    is kept TRANSPOSED in the block's chol[][] (column c contiguous, so a step reads consecutive doubles); a failed
//    diagonal stops it as the reference's row order does (w is kept);
//  * forward substitution column by column (row i subtracts in ascending j), backward substitution row by row with the
//    products gathered and summed in ascending order; Predict() sums on lane 0.
// Kept small on purpose: it runs once per sample, and its code shares the instruction cache with the ordinary bits.
__device__ __noinline__ void p8_audio_ols_warp(P8Shared& sh, int k, int lane) {
  using namespace p8;
  State& S = sh.S;
  AudioM& A = *S.audio;
  const int n = audio_ols_n(k), pch = A.ch ^ A.stereo;
  const double lambda = audio_ols_lambda(k), nu = 0.001, one_minus = P8_DSUB(1.0, lambda);
  double* blk = audio_ols_block(A, k, pch);
  double* x = blk; double* w = blk + n; double* b = blk + 2 * n; double* cov = blk + 3 * n; double* lt = cov + n * n;
  double* u = sh.u.md.ols.ch[0] + (k == 7 ? 6 : k) * 256; double* v = u + 128;
  const double val = (double)(buf(S, 1) - 128);
  int km = A.ols_km[k][pch] + 1;
  const bool solve = km >= audio_ols_kmax(k);
  for (int j = 0; j < n; ++j) {
    const double xj = x[j];
    for (int i = lane; i < n; i += 32) {
      const double c = P8_DADD(P8_DMUL(lambda, cov[j * n + i]), P8_DMUL(one_minus, P8_DMUL(xj, x[i])));
      cov[j * n + i] = c;
      if (solve) lt[j * n + i] = i == j ? P8_DADD(c, nu) : c;     // column j of the copy is row j: the matrix is symmetric
    }
  }
  for (int i = lane; i < n; i += 32) { b[i] = P8_DADD(P8_DMUL(lambda, b[i]), P8_DMUL(one_minus, P8_DMUL(x[i], val))); v[i] = b[i]; }
  if (solve) {
    __syncwarp();
    bool fail = false;
    for (int c = 0; c < n && !fail; ++c) {
      for (int r = c + lane; r < n; r += 32) {
        double s = lt[c * n + r];
        for (int q = 0; q < c; ++q) s = P8_DSUB(s, P8_DMUL(lt[q * n + r], lt[q * n + c]));
        u[r] = s;
      }
      __syncwarp();
      const double d = u[c];
      if (d > 1E-8) {
        const double dd = P8_DSQRT(d);
        for (int r = c + lane; r < n; r += 32) lt[c * n + r] = r == c ? dd : P8_DDIV(u[r], dd);
      } else fail = true;
      __syncwarp();
    }
    if (!fail) {
      for (int q = 0; q < n; ++q) {            // v: the rows' running sums; u: w after the forward pass
        const double wq = P8_DDIV(v[q], lt[q * n + q]);
        for (int r = q + 1 + lane; r < n; r += 32) v[r] = P8_DSUB(v[r], P8_DMUL(lt[q * n + r], wq));
        if (lane == 0) u[q] = wq;
        __syncwarp();
      }
      for (int i = n - 1; i >= 0; --i) {       // v: the products of row i; u[i]: w[i] after the backward pass
        for (int j = i + 1 + lane; j < n; j += 32) v[j] = P8_DMUL(lt[i * n + j], u[j]);
        __syncwarp();
        if (lane == 0) {
          double s = u[i];
          for (int j = i + 1; j < n; ++j) s = P8_DSUB(s, v[j]);
          u[i] = P8_DDIV(s, lt[i * n + i]);
        }
        __syncwarp();
      }
      for (int i = lane; i < n; i += 32) w[i] = u[i];
    }
    km = 0;
  }
  __syncwarp();
  if (lane == 0) { A.ols_km[k][pch] = km; audio8b_taps(S, k); }
  __syncwarp();
  const double* xc = audio_ols_block(A, k, A.ch);
  for (int i = lane; i < n; i += 32) v[i] = P8_DMUL(xc[n + i], xc[i]);
  __syncwarp();
  if (lane == 0) {
    double sum = 0.;
    for (int i = 0; i < n; ++i) sum = P8_DADD(sum, v[i]);
    audio8b_predict(S, k, sum);
  }
  __syncwarp();
}

// Insert the (map, bucket) pairs of one context into the per-bit set; returns true when a pair was already there, i.e. another
// context of the same map touches the same 64-byte bucket this bit. A context's own repeats are removed first. A pair that
// was already there is marked P8_KEY_SHARED, and ids[0..4] are replaced by the set's slots that hold the context's pairs
// (n >= 1; the first one repeated past n), so that after the probe p8_shares tells whether the context met another.
enum : unsigned long long { P8_KEY_SHARED = 1ull << 63 };
__device__ bool p8_claim(unsigned long long* seen, int map, u32* ids, int n) {
  bool clash = false;
  u32 slots[5];
#pragma unroll
  for (int a = 0; a < 5; ++a) {
    if (a >= n) { slots[a] = slots[0]; continue; }
    const u32 id = ids[a];
    bool dup = false;
    u32 slot = 0;
#pragma unroll
    for (int b = 0; b < a; ++b) if (!dup && ids[b] == id) { dup = true; slot = slots[b]; }
    if (!dup) {
      const unsigned long long key = ((unsigned long long)(map + 1) << 32) | id;
      slot = (u32)((key * 0x9E3779B97F4A7C15ull) >> 52) & (P8_SEEN - 1);
      for (;;) {
        const unsigned long long old = atomicCAS(&seen[slot], 0ull, key);
        if (old == 0ull) break;
        if ((old & ~P8_KEY_SHARED) == key) {
          clash = true;
          if (!(old & P8_KEY_SHARED)) atomicOr(&seen[slot], P8_KEY_SHARED);
          break;
        }
        slot = (slot + 1) & (P8_SEEN - 1);
      }
    }
    slots[a] = slot;
  }
#pragma unroll
  for (int a = 0; a < 5; ++a) ids[a] = slots[a];
  return clash;
}
// after the probe's barrier: whether a context's pairs (the slots p8_claim left in ids) meet another context's
__device__ __forceinline__ bool p8_shares(const unsigned long long* seen, const u32* slots) {
  bool s = false;
#pragma unroll
  for (int a = 0; a < 5; ++a) s = s || (seen[slots[a]] & P8_KEY_SHARED) != 0;
  return s;
}

// map (k, i) of a 7-slot-map lane, false if the lane is beyond the maps
__device__ __forceinline__ bool p8_cm_lane(int lane, int& k, int& i) {
  if (lane >= P8_CM_LANES) return false;
  k = 0;
#pragma unroll
  for (int q = 1; q < P8_N_CM; ++q) k += lane >= (int)c_p8_cm_base[q];
  i = lane - c_p8_cm_base[k];
  return true;
}
__device__ __forceinline__ bool p8_cm2_lane(int lane, int& k, int& i) {
  if (lane < 0 || lane >= P8_CM2_LANES) return false;
  k = (lane >= 10) + (lane >= 43);
  i = lane - (k == 0 ? 0 : (k == 1 ? 10 : 43));
  return true;
}
// how many contexts of the lanes [lo, hi) draw this bit
__device__ __forceinline__ int p8_flags_in(const u32* mask, int lo, int hi) {
  int r = 0;
  for (int w = lo >> 5; w <= ((hi - 1) >> 5) && hi > lo; ++w) {
    u32 m = mask[w];
    if (w == (lo >> 5)) m &= ~0u << (lo & 31);
    if (w == (hi >> 5)) m &= (1u << (hi & 31)) - 1u;
    r += __popc(m);
  }
  return r;
}

// ---- the pieces of a bit ----------------------------------------------------------------------------------------------
// probe of the history maps (lanes P8_CM2_TID0 ..): buckets each context touches this bit
__device__ __noinline__ void p8_probe_cm2(P8Shared& sh, int tid, int bpos, int maps) {   // maps: bit k set = history map k
  int k, i;
  if (!p8_cm2_lane(tid - P8_CM2_TID0, k, i) || !(maps >> k & 1)) return;
  p8::Cm2& m = p8_cm2(sh.S, k);
  u32* ids = sh.ids2[tid - P8_CM2_TID0];
  const int n = i < m.index ? p8::cm2_touched(m, i, bpos, ids) : 0;
  if (n && p8_claim(sh.u.md.seen, P8_N_CM + k, ids, n)) sh.clash2[k] = 1;
}
// copy context i's slot and run record from HBM into lane tid's P8CmCache entry
__device__ __forceinline__ void p8_cm_fill(P8CmCache& cc, const p8::Cm& m, int i, int tid) {
  const unsigned char* s = m.t + m.cp0[i];
  unsigned char v[9];          // every load before the first store: one round trip, not one per byte
#pragma unroll
  for (int j = 0; j < 7; ++j) v[j] = s[j];
  v[7] = m.t[m.runp[i]];
  v[8] = m.t[m.runp[i] + 1];
#pragma unroll
  for (int j = 0; j < 7; ++j) cc.slot[tid][j] = v[j];
  cc.run[tid][0] = v[7];
  cc.run[tid][1] = v[8];
  cc.valid[tid] = 1;
}
// cm_step on a staying bit from lane tid's copy (P8CmCache) and the StateMap cells its probe loaded (k: the map's index,
// key: the stream's, for the census build)
__device__ __forceinline__ int p8_cm_stay(P8CmCache& cc, p8::Cm& m, int i, int tid, p8::Out& o, int ns, int y, int c0, int bp, int k, const void* key) {
  using namespace p8;
  const p8::Tables& T = *o.T;
  u8* sl = cc.slot[tid];
  const int base = m.cp0[i];
  CENSUS_P8_COPY(key, m, k, i, sl, cc.run[tid], false, false);
  if (m.cp[i] != P8_NULL) { m.t[m.cp[i]] = (u8)ns; sl[m.cp[i] - base] = (u8)ns; }
  const int nc = cm_stay_cell(cc.run[tid][0], c0, bp);
  m.cp[i] = nc >= 0 ? base + nc : P8_NULL;
  if ((bp == 1 || bp == 4) && nc >= 0) bucket_prefetch2(m.t, m.mask, m.cxt[i], (u32)c0 * 2);
  P8_LEG(4);
  cm_run_input(T, o, cc.run[tid][0], cc.run[tid][1], c0, bp);
  P8_LEG(5);
  const int s = nc >= 0 ? sl[nc] : 0, so = m.sm_cxt[i];
  m.sm_cxt[i] = s;
  CENSUS_P8_SM(key, k, i, m.sm_t + i * 256, so, cc.sm[tid][0], s, cc.sm[tid][1]);
  return cm_cell_inputs(T, o, m.sm_t + i * 256, so, cc.sm[tid][0], s, cc.sm[tid][1], y);
}
// pass 1 of the 7-slot maps (warps 0-6, whole warps): aged state, draw flag, touched buckets (slots on a staying bit)
__device__ __noinline__ void p8_probe_cm(P8Shared& sh, int tid, int y, int c0, int bpos) {
  using namespace p8;
  int k, i;
  bool flag = false;
  if (p8_cm_lane(tid, k, i)) {
    Cm& m = p8_cm(sh.S, k);
    int ns = -1;
    if (i < m.cn) {
      P8_LEG(-1);
      const bool stay = cm_staying(bpos);
      P8CmCache& cc = sh.u.md.cc;
      u16 sm_old = 0, sm_new = 0;
      if (stay) {         // the new cell is known before the bit's stores (c0 holds y), so both StateMap loads start here
#ifdef CMIXB200_CENSUS
        const bool filled = !cc.valid[tid];
#endif
        if (!cc.valid[tid]) p8_cm_fill(cc, m, i, tid);
        CENSUS_P8_COPY(sh.S.sparse.cm.t, m, k, i, cc.slot[tid], cc.run[tid], true, filled);
        const u8* sl = cc.slot[tid];
        ns = m.cp[i] != P8_NULL ? sh.S.T->state[sl[m.cp[i] - m.cp0[i]]][y] : -1;
        const int nc = cm_stay_cell(cc.run[tid][0], c0, bpos);
        const u16* smt = m.sm_t + i * 256;
        sm_old = smt[m.sm_cxt[i]];
        sm_new = smt[nc >= 0 ? sl[nc] : 0];
      } else ns = cm_next_state(*sh.S.T, m, i, y);
      P8_LEG(0);
      const int n = stay ? cm_slot_keys(m, i, sh.ids[tid]) : cm_touched(m, i, c0, bpos, sh.ids[tid]);
      P8_LEG(1);
      if (p8_claim(sh.u.md.seen, k, sh.ids[tid], n)) { sh.clash[k] = 1; sh.any_clash = 1; }
      P8_LEG(2);
      if (stay) { cc.sm[tid][0] = sm_old; cc.sm[tid][1] = sm_new; P8_LEG(6); }
    }
    sh.ns[tid] = (short)ns;
    flag = ns >= 204;
  }
  const u32 mask = __ballot_sync(0xffffffffu, flag);
  if ((tid & 31) == 0) sh.flag_mask[tid >> 5] = mask;
#ifdef CMIXB200_CENSUS
  if ((tid & 31) == 0) sh.flag_mask1[tid >> 5] = mask;
#endif
}
// the units that are one lane each, on the bit that starts a byte (warps 8-11 of the D-chain; record_pre and the linear
// predictions' maps follow their models there)
__device__ __noinline__ void p8_probe_single(P8Shared& sh, int tid, int y, int c0, int bpos, bool audio) {
  using namespace p8;
  State& S = sh.S;
  const p8::Tables& T = *S.T;
  if (audio && (tid == P8_TID_PIC || (tid >= P8_TID_W10 && tid < P8_TID_W10 + 10) || tid == P8_TID_W11)) return;   // not in audio mode
  if (tid == P8_TID_PIC) pic_core(S);
  else if (tid == P8_TID_MATCH) { Out o = p8_out(sh, sh.unit_off[7]); match_core(S, o); }
  else if (tid >= P8_TID_W10 && tid < P8_TID_W10 + 10) sh.dmc_st[tid - P8_TID_W10] = dmc_st(T, S.dmc[tid - P8_TID_W10], y);
  else if (tid >= P8_TID_MATCH + 2 && tid < P8_TID_MATCH + 5) {
    const int r = tid - (P8_TID_MATCH + 2);
    Out o = p8_out(sh, sh.unit_off[4 + r]);
    rcm_mix(r == 0 ? S.rcm7 : r == 1 ? S.rcm9 : S.rcm10, o, c0, bpos);
  }
  else if (tid == P8_TID_W11) { Out o = p8_out(sh, sh.unit_off[8]); smatch_head(S, o); }
  else if (tid == P8_TID_W11 + 1 || tid == P8_TID_W11 + 2) {
    const int r = tid - (P8_TID_W11 + 1);
    Out o = p8_out(sh, sh.unit_off[1 + r]);
    add(o, (stretch(T, sm32_p(T, r == 0 ? S.sm0 : S.sm1, y, r == 0 ? c0 : (c0 | (buf(S, 1) << 8)))) + 1) >> 1);
  } else if (tid == P8_TID_W11 + 3) { Out o = p8_out(sh, sh.unit_off[0]); add(o, 64); }
}
// draws[j] = x[i0 + 1 + j] of the lagged generator x[i] = x[i-24] ^ x[i-55] for every j a bit without a clash can consume
// (j < P8_CM_LANES), from the table as the bit finds it (r.i = i0). One warp, 24 values per step: lane l of step s computes
// x[i0 + 1 + 24 s + l] from its own value of step s-1 and lane l-7's of step s-2 (lane l+17's of step s-3 when l < 7).
__device__ __noinline__ void p8_draw_seq(P8Shared& sh, int lane) {
  const p8::Rnd& r = sh.S.rnd;
  const unsigned full = 0xffffffffu;
  const int i1 = r.i + 1;
  u32 p1 = r.table[(i1 + lane - 24) & 63], p2 = r.table[(i1 + lane - 48) & 63], p3 = r.table[(i1 + lane - 72) & 63];   // steps -1, -2, -3
  for (int s0 = 0; s0 < P8_CM_LANES; s0 += 24) {
    const u32 a = __shfl_sync(full, p3, (lane + 17) & 31), b = __shfl_sync(full, p2, (lane - 7) & 31);
    const u32 v = p1 ^ (lane < 7 ? a : b);
    if (lane < 24 && s0 + lane < P8_CM_LANES) sh.draws[s0 + lane] = v;
    p3 = p2; p2 = p1; p1 = v;
  }
}
// advance the generator by the number of flagged contexts: the table keeps the last 64 of the draws (one warp)
__device__ __forceinline__ void p8_advance_rnd(P8Shared& sh, int lane) {
  p8::Rnd& r = sh.S.rnd;
  const int total = p8_flags_in(sh.flag_mask, 0, P8_CM_LANES);
  const int i0 = r.i;
  __syncwarp();
  for (int j = max(0, total - 64) + lane; j < total; j += 32) r.table[(i0 + 1 + j) & 63] = sh.draws[j];
  if (lane == 0) r.i = i0 + total;
}
// pass 2
__device__ __noinline__ void p8_apply_cm2(P8Shared& sh, int tid, int y, int bpos, int maps) {
  int k, i;
  if (!p8_cm2_lane(tid - P8_CM2_TID0, k, i) || !(maps >> k & 1)) return;
  p8::Cm2& m = p8_cm2(sh.S, k);
  const int off = sh.unit_off[c_p8_cm2_unit[k]];
  if (!sh.clash2[k]) {
    if (i < m.index) { p8::Out o = p8_out(sh, off + 7 * i); if (p8::cm2_step(m, i, o, y, bpos)) atomicAdd(&sh.res2[k], 1); }
  } else if (i == 0) {      // in-order evaluation by one lane (the two loops of ContextMap2::mix)
    p8::Out o = p8_out(sh, off);
    sh.res2[k] = p8::cm2_mix_body(m, o, y, bpos);
  }
}
__device__ __noinline__ void p8_apply_cm(P8Shared& sh, int tid, int y, int c0, int bpos) {
  using namespace p8;
  if (tid < 32) p8_advance_rnd(sh, tid);      // flagged lanes read their draw from draws[], not from the table
  int k, i;
  if (!p8_cm_lane(tid, k, i)) return;
  Cm& m = p8_cm(sh.S, k);
  P8CmCache& cc = sh.u.md.cc;
  if (sh.clash[k] && (sh.group_mask[tid >> 5] >> (tid & 31) & 1)) { cc.valid[tid] = 0; return; }   // walked by p8_number
  if (i >= m.cn) return;
  P8_LEG(-1);
  int ns = sh.ns[tid];
  if (ns >= 204) {
    const u32 r = sh.draws[p8_flags_in(sh.flag_mask, 0, tid)];
    if (cm_draw_hits(r, ns)) ns -= 4;
  }
  P8_LEG(3);
  Out o = p8_out(sh, sh.unit_off[c_p8_cm_unit[k]] + 5 * i);
  if (cm_staying(bpos)) p8_cm_stay(cc, m, i, tid, o, ns, y, c0, bpos, k, sh.S.sparse.cm.t);
  else {
    cm_step(m, i, o, ns, y, c0, bpos, buf(sh.S, 1));
    p8_cm_fill(cc, m, i, tid);
  }
}
// DMC forest combination, and the reset at a byte boundary (dmcForest::mix), from the dmc_st values of the probe
__device__ __forceinline__ void p8_dmc_mix(P8Shared& sh, p8::Out& o, int bpos) {
  using namespace p8;
  State& S = sh.S;
  const u32 params[10] = {2, 32, 64, 4, 128, 8, 256, 16, 1024, 1536};
  add(o, sh.dmc_st[9] >> 3);
  add(o, sh.dmc_st[8] >> 3);
  for (int i = 7; i > 0; i -= 2) add(o, (sh.dmc_st[i] + sh.dmc_st[i - 1]) >> 4);
  if (bpos == 0)
    for (int i = 7; i >= 0; --i)
      if ((S.dmc[i].extra >> 7) > S.dmc[i].size) dmc_reset(S.dmc[i], params[i]);
}
// the units that are one lane each, on the bit that starts a byte (warps 9-11 after the join)
__device__ __noinline__ void p8_apply_small(P8Shared& sh, int tid, int y, int bpos, bool audio) {
  using namespace p8;
  State& S = sh.S;
  if (audio && tid >= P8_TID_W10 + 12) return;   // audio mode: the match and record models' maps only
  if (tid >= P8_TID_MATCH && tid < P8_TID_MATCH + 9) {   // the nine maps behind the match model
    Out o = p8_out(sh, sh.unit_off[7]);
    match_unit(S, o, tid - P8_TID_MATCH);
  } else if (tid >= P8_TID_W10 && tid < P8_TID_W10 + 12) {   // the record model's 12 direct maps (contexts selected by record_pre)
    Out o = p8_out(sh, sh.unit_off[24 + (tid - P8_TID_W10)]);
    record_small(S, o, tid - P8_TID_W10);
  } else if (tid == P8_TID_W10 + 12) {                     // DMC forest combination and reset (dmcForest::mix)
    Out o = p8_out(sh, sh.unit_off[44]);
    p8_dmc_mix(sh, o, bpos);
  } else if (tid >= P8_TID_W11 && tid < P8_TID_W11 + 7) {   // sparseModel1's seven stationary maps
    Out o = p8_out(sh, sh.unit_off[11 + (tid - P8_TID_W11)]);
    scm_mix(S.sparse1.scm[tid - P8_TID_W11], o, y);
  } else if (tid >= P8_TID_W11 + 7 && tid < P8_TID_W11 + 11) {
    Out o = p8_out(sh, sh.unit_off[8]);
    smatch_unit(S, o, tid - (P8_TID_W11 + 7));
  } else if (tid >= P8_TID_W11 + 11 && tid < P8_TID_W11 + 14) {
    Out o = p8_out(sh, sh.unit_off[19]);
    pic_unit(S, o, tid - (P8_TID_W11 + 11));
  }
}

// ---- inside a byte: the single-lane units, a warp per function (lane map: P8_W_* below). Every unit writes its inputs at
// its own unit_off[] as on the bit that starts a byte; units of one phase share no state, so their order does not matter.
// In audio mode the DMC, sparse match and picture units do not run; warps 10 and 11 run audio8bModel's 33 maps instead.
__device__ __noinline__ void p8_probe_units(P8Shared& sh, int warp, int lane, int y, int c0, int bpos, bool audio) {
  using namespace p8;
  State& S = sh.S;
  P8_U0;
  if (audio && (warp == P8_W_DMC || warp == P8_W_SMATCH)) {
    const int q = warp == P8_W_DMC ? lane : 32 + lane;
    if (q < AUDIO_N_SCM) p8_audio_scm(sh, q);
    return;
  }
  if (audio && warp == P8_W_PIC) return;
  if (warp == P8_W_MATCH) {
    if (lane == 0) { Out o = p8_out(sh, sh.unit_off[7]); match_core(S, o); P8_U(1); }
  } else if (warp == P8_W_DMC) {
    if (lane < 10) { sh.dmc_st[lane] = dmc_st(*S.T, S.dmc[lane], y); P8_U(4); }
  } else if (warp == P8_W_SMATCH) {
    if (lane == 0) { Out o = p8_out(sh, sh.unit_off[8]); smatch_head(S, o); P8_U(5); }
  } else if (warp == P8_W_PIC) {
    if (lane == 0) { pic_core(S); P8_U(0); }
  } else if (warp == P8_W_RECORD) {
    if (lane == 0) { record_pre(S); P8_U(2); }
  } else if (warp == P8_W_RCM) {
    if (lane < 3) { Out o = p8_out(sh, sh.unit_off[4 + lane]); rcm_mix(lane == 0 ? S.rcm7 : lane == 1 ? S.rcm9 : S.rcm10, o, c0, bpos); P8_U(3); }
  }
}
// The apply phase groups the units by the map they end in, so that the lanes of a warp run one call of one function with
// their own arguments (the arguments are those of match_unit, record_small, smatch_unit, linear_small and the rest).
__device__ __noinline__ void p8_apply_units(P8Shared& sh, int warp, int lane, int y, int c0, int bpos, bool audio) {
  using namespace p8;
  State& S = sh.S;
  const p8::Tables& T = *S.T;
  P8_U0;
  // audio mode: the maps behind the match and record models and the constant input only
  if (audio && ((warp == P8_W_SCM && lane >= 6) || (warp == P8_W_STM && lane >= 9) || warp == P8_W_PICU || (warp == P8_W_DMCMIX && lane == 0))) return;
  if (warp == P8_W_SM32) {              // the match model's three StateMaps (match_unit 0-2), the order-0 and order-1 inputs
    if (lane >= 5) return;
    Sm32* s; int off, cx; bool on = true;
    if (lane < 3) { s = &S.match.sm[lane]; off = sh.unit_off[7] + 2 + lane; cx = (int)S.match.ctx[lane]; on = cx != 0; }
    else { s = lane == 3 ? &S.sm0 : &S.sm1; off = sh.unit_off[lane - 2]; cx = lane == 3 ? c0 : (c0 | (buf(S, 1) << 8)); }
    Out o = p8_out(sh, off);
    const int p = sm32_p(T, *s, y, cx);
    add(o, on ? (stretch(T, p) + 1) >> 1 : 0);
    P8_U(10);
  } else if (warp == P8_W_SCM) {        // match_unit 3-5, record_small 9-11, sparseModel1's seven maps, linear_small 0-4
    if (lane >= 18) return;
    Scm* c; int off, rate = 7, mul = 1, div = 4;
    if (lane < 3) { c = &S.match.scm[lane]; off = sh.unit_off[7] + 5 + 2 * lane; rate = 7 - lane; }
    else if (lane < 6) { const int k = lane - 3; c = &S.record.smap[k]; off = sh.unit_off[33 + k]; rate = k < 2 ? 6 : 5; div = k < 2 ? 3 : 2; }
    else if (lane < 13) { c = &S.sparse1.scm[lane - 6]; off = sh.unit_off[11 + lane - 6]; }
    else {
      const int i = lane - 13;
      LinearM& M = S.linear;
      c = &M.smap[i]; off = sh.unit_off[48 + i]; rate = 6; div = 2;
      scm_set(*c, (u32)((M.prd[i] - (u8)(c0 << (8 - bpos))) * 8 + bpos));
    }
    Out o = p8_out(sh, off);
    scm_mix(*c, o, y, rate, mul, div);
    P8_U(11);
  } else if (warp == P8_W_STM) {        // match_unit 6-8, record_small 0-5, smatch_unit 0-3
    if (lane >= 13 || (lane >= 9 && !S.smatch.valid)) return;
    Stm* c; int off, div = 4, limit = 1023;
    if (lane < 3) { c = &S.match.maps[lane]; off = sh.unit_off[7] + 11 + 2 * lane; limit = lane == 0 ? 255 : 1023; }
    else if (lane < 9) { c = &S.record.maps[lane - 3]; off = sh.unit_off[24 + lane - 3]; div = 3; }
    else { c = &S.smatch.maps[lane - 9]; off = sh.unit_off[8] + 3 + 2 * (lane - 9); div = 2; }
    Out o = p8_out(sh, off);
    stm_mix(*c, o, y, 1, div, limit);
    P8_U(12);
  } else if (warp == P8_W_IMAP) {       // record_small 6-8
    if (lane < 3) { Out o = p8_out(sh, sh.unit_off[30 + lane]); imap_mix(S.record.imap[lane], o, y, 1, 3, 255); P8_U(13); }
  } else if (warp == P8_W_PICU) {
    if (lane < 3) { Out o = p8_out(sh, sh.unit_off[19]); pic_unit(S, o, lane); P8_U(17); }
  } else if (warp == P8_W_DMCMIX) {     // the DMC forest's combination (from dmc_st of the probe) and the constant input
    if (lane == 0) { Out o = p8_out(sh, sh.unit_off[44]); p8_dmc_mix(sh, o, bpos); P8_U(14); }
    else if (lane == 1) { Out o = p8_out(sh, sh.unit_off[0]); add(o, 64); }
  }
}

// The SSE stage (paq8_top.h sse_stage) on one warp: the APMs of a level side by side. c1 = buf(S, 1) of the bit.
__device__ void p8_sse_warp(P8Shared& sh, int pr0, int c1, int lane) {
  using namespace p8;
  State& S = sh.S;
  const p8::Tables& T = *S.T;
  const unsigned full = 0xffffffffu;
  const int y = S.y, c0 = S.c0, bpos = S.bpos;
  const u32 c4 = S.c4;
  u16* codes = S.codes + S.m.n2 + S.m.ncxt;
  const u32 mlen = umin(3, ilog2(S.st_match_length + 1));
  int p = 0, q = 0, pr, pr1, pr2, pr3, pr0b;
  if (S.st_type == FT_TEXT) {
    const int limit = 0x3FF >> ((S.blpos < 0xFFF) * 2);
    if (lane < 4) {
      int cx;
      if (lane == 0) cx = (c0 << 8) | (S.st_text_mask & 0xF) | (int)((S.st_misses & 0xF) << 4);
      else if (lane == 1) cx = (int)finalize64(hash(sx(bpos), S.st_misses & 3, (u64)(c4 & 0xffff), (u64)(S.st_text_mask >> 4)), 16);
      else if (lane == 2) cx = (int)finalize64(hash(sx(c0), S.st_match_expected, mlen), 16);
      else cx = (int)finalize64(hash(sx(c0), (u64)(c4 & 0xffff), S.st_text_first), 16);
      p = apm_p(T, S.text_apm[lane], y, pr0, cx, limit);
    }
    pr = __shfl_sync(full, p, 0); pr1 = __shfl_sync(full, p, 1); pr2 = __shfl_sync(full, p, 2); pr3 = __shfl_sync(full, p, 3);
    pr0b = (pr0 + pr1 + pr2 + pr3 + 2) >> 2;
    if (lane < 3) {
      int cx;
      if (lane == 0) cx = (int)finalize64(hash(S.st_match_expected, mlen, (u64)(c4 & 0xff)), 16);
      else if (lane == 1) cx = (int)finalize64(hash(sx(c0), (u64)(c4 & 0x00ffffff)), 16);
      else cx = (int)finalize64(hash(sx(c0), (u64)(c4 & 0xffffff00)), 16);
      q = apm1_p(T, S.text_apm1[lane], y, lane == 0 ? pr0b : pr, cx, lane == 0 ? 7 : 6);
    }
  } else {
    const u16 ctx1 = (u16)(c0 | c1 << 8);
    const u16 ctx2 = (u16)(c0 ^ finalize64(hash((u64)(c4 & 0xffff)), 16));
    const u16 ctx3 = (u16)(c0 ^ finalize64(hash((u64)(c4 & 0xffffff)), 16));
    if (lane < 4) {
      const int cx = lane == 0 ? (int)((mlen << 11) | ((u32)c0 << 3) | (u32)(S.st_misses & 0x7)) : lane == 1 ? (int)ctx1 : lane == 2 ? (int)ctx2 : (int)ctx3;
      p = apm1_p(T, S.generic_apm1[lane], y, pr0, cx);
    }
    pr = __shfl_sync(full, p, 0); pr1 = __shfl_sync(full, p, 1); pr2 = __shfl_sync(full, p, 2); pr3 = __shfl_sync(full, p, 3);
    pr0b = (pr0 + pr1 + pr2 + pr3 + 2) >> 2;
    if (lane < 3) {
      const int cx = lane == 0 ? ((S.st_match_expected << 8) | c1) : lane == 1 ? (int)ctx2 : (int)ctx3;
      q = apm1_p(T, S.generic_apm1[4 + lane], y, pr, cx);
    }
  }
  const int q1 = __shfl_sync(full, q, 0), q2 = __shfl_sync(full, q, 1), q3 = __shfl_sync(full, q, 2);
  const int prf = (pr + q1 + q2 + q3 + 2) >> 2;
  const int fin = (prf + pr0b + 1) >> 1;
  if (lane == 0) {
    int e = 0;
    codes[e++] = (u16)pr0; codes[e++] = (u16)pr; codes[e++] = (u16)pr1; codes[e++] = (u16)pr2; codes[e++] = (u16)pr3;
    if (S.st_type == FT_TEXT) codes[e++] = (u16)pr0b;
    codes[e++] = (u16)q1; codes[e++] = (u16)q2; codes[e++] = (u16)q3; codes[e++] = (u16)prf; codes[e++] = (u16)fin;
    S.pr = fin;
    S.last_prediction = fin;
  }
}

// weight-set cache: rows move between HBM and shared memory in 16-byte words, past L1
__device__ __forceinline__ void p8_row_load(short* dst, const short* src, int lane) {
  const uint4* s = reinterpret_cast<const uint4*>(src); uint4* d = reinterpret_cast<uint4*>(dst);
  uint4 v[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) { const int q = lane + 32 * j; if (q < p8::N_IN / 8) v[j] = __ldcg(s + q); }
#pragma unroll
  for (int j = 0; j < 7; ++j) { const int q = lane + 32 * j; if (q < p8::N_IN / 8) d[q] = v[j]; }
}
__device__ __forceinline__ void p8_row_store(short* dst, const short* src, int lane) {
  const uint4* s = reinterpret_cast<const uint4*>(src); uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int j = 0; j < 7; ++j) { const int q = lane + 32 * j; if (q < p8::N_IN / 8) __stcg(d + q, s[q]); }
}
static_assert(p8::N_IN % 8 == 0 && p8::N_IN / 8 <= 7 * 32, "a weight row is at most 7 16-byte words per lane");

// named barrier 2: the model warps signal "the state the 19 order-independent selector sets read is final" (arrive), the
// first SGD warp waits for it (sync) and computes those sets beside the apply phase
__device__ __forceinline__ void p8_signal_selects(int site) { jit_point(site); asm volatile("bar.arrive 2, 416;" ::: "memory"); }
__device__ __forceinline__ void p8_await_selects(int site) { asm volatile("bar.sync 2, 416;" ::: "memory"); jit_point(site); }
// named barrier 1 (warps 0-11): in a clashing bit's numbering (behind the grouped marks, behind lane 0's walk) and behind
// the apply phase, before lane 0's epilogue reads res2 and clash; on the bit that starts a byte also between the probe and
// the numbering. Inside a byte the unit warps 13-15 are not in it (nothing behind it reads their inputs before the bit's
// last __syncthreads)
__device__ __forceinline__ void p8_sync_maps(int site) { asm volatile("bar.sync 1, 384;" ::: "memory"); jit_point(site); static_assert(P8_MAP_THREADS == 384, "named barrier width"); }
// The bit that starts a byte runs its context computation as independent chains of warps (p8_model_bit) ordered by three
// more named barriers. Every arrive / sync below is executed by whole warps, unconditionally on that bit:
//  3 (join, 480): "the new contexts of every map are set". Warps 0-11 sync on it before the probe of the 7-slot maps
//                 (384), the text chain's warps 13-15 arrive (96) and go on to the end of the bit.
//  4 (160):       the D-chain's warps 7-11 between its steps.
//  5 (96):        the text chain's warps 13-15 between its steps.
// Inside a byte barrier 3 is the probe / apply boundary, with the same warps: all of them sync (the unit warps 13-15 apply
// what warps 9-11 probed and the reverse).
__device__ __forceinline__ void p8_join_sync(int site) { asm volatile("bar.sync 3, 480;" ::: "memory"); jit_point(site); }
__device__ __forceinline__ void p8_join_arrive(int site) { jit_point(site); __threadfence_block(); asm volatile("bar.arrive 3, 480;" ::: "memory"); }
__device__ __forceinline__ void p8_sync_dchain(int site) { asm volatile("bar.sync 4, 160;" ::: "memory"); jit_point(site); }
__device__ __forceinline__ void p8_sync_text(int site) { asm volatile("bar.sync 5, 96;" ::: "memory"); jit_point(site); }
enum { P8_WARP_D = P8_CM2_TID0 / 32, P8_WARP_TEXT = P8_MAP_WARPS + 1 };   // first warp of the D-chain / of the text chain
static_assert(P8_CM2_TID0 % 32 == 0 && P8_CM_LANES <= P8_CM2_TID0 && (P8_MAP_WARPS - P8_WARP_D) * 32 == 160, "barrier 4: warps 7-11");
static_assert((P8_WARPS - P8_WARP_TEXT) * 32 == 96 && P8_MAP_THREADS + 96 == 480, "barriers 3 and 5: warps 13-15 beside the 12 map warps");
static_assert(P8_TID_MATCH == (P8_WARP_D + 2) * 32 && P8_TID_W10 == (P8_WARP_D + 3) * 32 && P8_TID_W11 == (P8_WARP_D + 4) * 32, "a warp per long job of the D-chain");
static_assert(P8_W_MATCH > (P8_CM2_TID0 + P8_CM2_LANES - 1) / 32 && (int)P8_W_SMATCH < (int)P8_MAP_WARPS && (int)P8_W_PIC == (int)P8_WARP_TEXT && (int)P8_W_RCM == (int)P8_WARPS - 1 &&
              P8_W_IMAP > (P8_CM2_TID0 + P8_CM2_LANES - 1) / 32 && (int)P8_W_DMCMIX < (int)P8_MAP_WARPS && (int)P8_W_SM32 == (int)P8_WARP_TEXT && (int)P8_W_STM == (int)P8_WARPS - 1,
              "barrier 3 inside a byte: the unit warps are 9-11 (in barriers 1 and 2 with the map warps) and 13-15 (in barrier 3 only)");

// A bit on which two contexts of a 7-slot map meet (in a bucket on a move bit, in a slot on a staying bit), warps 0-11. A
// context of a clashing map that shares a key with another is GROUPED; the others are FREE: nothing a grouped context writes
// is a key of a free one, so a free context's aged state and flag from pass 1 stand and it runs in p8_apply_cm like a lane
// of a clash-free map. Lane 0 walks the grouped contexts of all clashing maps in program order: each takes its aged state
// from HBM as the earlier ones left it, sets its real flag in flag_mask and takes the draw of its rank, which counts the
// final flags of every context before it (so the walk is one, not one per group or map). After it every flag is final.
__device__ __noinline__ void p8_number(P8Shared& sh, int tid, int y, int c0, int bpos) {
  using namespace p8;
  State& S = sh.S;
  int k, i;
  const bool grouped = p8_cm_lane(tid, k, i) && sh.clash[k] && i < p8_cm(S, k).cn && p8_shares(sh.u.md.seen, sh.ids[tid]);
  const u32 g = __ballot_sync(0xffffffffu, grouped);
  if ((tid & 31) == 0 && tid < P8_CM2_TID0) sh.group_mask[tid >> 5] = g;
  p8_sync_maps(JIT_HERE);
  if (tid != 0) return;
  const int c1 = buf(S, 1);
#ifdef P8_PROF
  int walked = 0;
#endif
  for (int w = 0; w < P8_CM2_TID0 / 32; ++w)
    for (u32 gm = sh.group_mask[w]; gm; gm &= gm - 1) {
      const int l = 32 * w + __ffs(gm) - 1;
      p8_cm_lane(l, k, i);
      Cm& m = p8_cm(S, k);
      int ns = cm_next_state(*S.T, m, i, y);
      const u32 bit = 1u << (l & 31);
      if (ns >= 204) {
        sh.flag_mask[w] |= bit;
        if (cm_draw_hits(sh.draws[p8_flags_in(sh.flag_mask, 0, l)], ns)) ns -= 4;
      } else sh.flag_mask[w] &= ~bit;
      Out o = p8_out(sh, sh.unit_off[c_p8_cm_unit[k]] + 5 * i);
      cm_step(m, i, o, ns, y, c0, bpos, c1);
#ifdef P8_PROF
      ++walked;
#endif
    }
#ifdef P8_PROF
  P8_C(P8_PROF_NUMBER + 8 + bpos, 1);
  P8_C(P8_PROF_NUMBER + 16 + bpos, walked);
#endif
}

// The mixer CTA's first bit in a new layout, on one warp: every cached row back to HBM, then the bit's sets fetched and their
// dot products (no row is fetched before every row is written back, and no other warp reads them this bit)
__device__ __noinline__ void p8_relayout(P8Shared& sh, const P8Slot& in, int lane) {
  using namespace p8;
  const Mixer& m = sh.S.m;
  for (int i = 0; i < N_SETS; ++i) if (sh.wc_set[i] >= 0) p8_row_store(m.w + (size_t)sh.wc_set[i] * N_IN, sh.u.mx.wc[i], lane);
  __syncwarp();
  if (lane < N_SETS) sh.wc_set[lane] = -1;
  for (int i = 0; i < in.ncxt; ++i) {
    short* row = sh.u.mx.wc[i];
    p8_row_load(row, m.w + (size_t)m.cxt[i] * N_IN, lane);
    __syncwarp();
    if (lane == 0) sh.wc_set[i] = m.cxt[i];
    int acc = 0;
    for (int q = lane; q < (in.nx >> 3); q += 32) {
      const uint4 wv = *reinterpret_cast<const uint4*>(row + q * 8);
      const uint4 xv = *reinterpret_cast<const uint4*>(in.tx + q * 8);
      const short* w = reinterpret_cast<const short*>(&wv);
      const short* x = reinterpret_cast<const short*>(&xv);
#pragma unroll
      for (int e = 0; e < 8; e += 2) acc += dot_pair(x + e, w + e);
    }
    acc = __reduce_add_sync(0xffffffffu, acc);
    if (lane == 0) sh.dot[i] = acc;
  }
}

// Mixer::update for the 28 cached weight sets selected for the previous bit, on its inputs tx (all lanes of the mixer CTA)
__device__ __forceinline__ void p8_sgd(P8Shared& sh, const short* tx, int y, int tid) {
  using namespace p8;
  const Mixer& m = sh.S.m;
  const int n8 = m.nx >> 3, total = m.ncxt * n8;
  if (n8 == 0) return;
  int i = tid / n8, q = tid - i * n8;
  for (int idx = tid; idx < total; idx += P8_THREADS) {
    const int err = ((y << 12) - m.pr[i]) * 7;
    if (err) {
      uint4* wp = reinterpret_cast<uint4*>(&sh.u.mx.wc[i][q * 8]);
      uint4 wv = *wp;
      const uint4 xv = *reinterpret_cast<const uint4*>(&tx[q * 8]);
      short* w = reinterpret_cast<short*>(&wv);
      const short* x = reinterpret_cast<const short*>(&xv);
#pragma unroll
      for (int e = 0; e < 8; ++e) w[e] = train_one(x[e], w[e], err);
      *wp = wv;
    }
    q += P8_THREADS;
    while (q >= n8) { q -= n8; ++i; }
  }
}

__device__ __noinline__ void p8_audio_selects(p8::State& S) { p8::audio8b_select(S); p8::record_select(S); }

// The model CTA's part of bit t of a launch: PAQ8::Perceive(y) up to the mixer's inputs and selectors, handed to slot t % P8_RING
// of the mixer CTA's ring (`ring`: that array in the mixer CTA). All P8_THREADS lanes call it: warps 0-11 evaluate the models,
// warp 12 computes ModelStats and 19 selector sets beside them.
__device__ void p8_model_bit(P8Shared& sh, P8Slot* ring, u32 t, int y, int nb, int tid, bool fresh = false) {   // nb: the bit position after this bit, (S.bpos + 1) & 7; fresh: shared memory holds nothing from the previous bit
  using namespace p8;
  State& S = sh.S;
  const p8::Tables& T = *S.T;
  const int warp = tid >> 5, lane = tid & 31;
#ifdef P8_PROF
  if (tid == 0) { sh.prof_t = clock64(); sh.prof_dst = sh.prof_acc; }
  int prof_clash = 0;   // lane 0: any_clash as the bit ends (the next bit's bookkeeping resets it beside the handover)
#endif
  // ---- phase 0: bookkeeping (bit_begin's st_misses line works on a stale S.pr here: st_misses belongs to the mixer CTA)
  if (tid == 0) {
    P8_U0;
    bit_begin(S, y);
    if (S.bpos == 0) block_parse(S);
    if (S.bpos == 0 && audio8_mode(S)) audio8b_begin(S);
    P8_U(20);
    if (S.bpos == 0) sh.snap = word_stats(S);     // read by sparse1_byte only
    P8_U(21);
  }
  if (tid >= 32 && tid < 32 + P8_N_CM) sh.clash[tid - 32] = 0;
  if (tid >= 64 && tid < 64 + P8_N_CM2) { sh.clash2[tid - 64] = 0; sh.res2[tid - 64] = 0; }
  if (tid == 67) sh.any_clash = 0;
  if (warp == 11) p8_draw_seq(sh, lane);          // beside lane 0's bit_begin: the draws depend on the generator only
  // the history maps' bit prologue; the text and x86 maps do not run in audio mode, so on the bit that starts a byte theirs
  // waits until lane 0 has parsed the byte (D-chain)
  if (tid >= P8_CM2_TID0 && tid < P8_CM2_TID0 + P8_N_CM2 && (tid == P8_CM2_TID0 || (nb != 0 && !audio8_mode(S)))) cm2_begin(p8_cm2(S, tid - P8_CM2_TID0), y, nb);
  // mixer-input offsets of the units (they change on the first two bits of a byte only). Audio mode is known here inside a
  // byte; on the bit that starts one lane 0 is deciding it, and warp 11 redoes the offsets of an audio byte after the barrier
  if (warp == P8_WARPS - 1 && (nb <= 1 || fresh)) p8_unit_offsets(sh, lane, nb == 0, nb != 0 && audio8_mode(S));
  {
    P8_U0;
    for (int k = tid; k < P8_SEEN; k += P8_THREADS) sh.u.md.seen[k] = 0ull;
    if (tid == 0) P8_U(22);
  }
  JIT_SYNCTHREADS();
  P8_T(0);
  const int bpos = S.bpos, c0 = S.c0;
  const bool byte_start = bpos == 0;
  const bool audio = audio8_mode(S);      // audioModel's bits: audio8bModel and recordModel(AUDIO) behind the shared prefix
  if (tid >= P8_MAP_THREADS) {
    if (warp == P8_MAP_WARPS) {            // ModelStats and the 19 selector sets that do not wait for the order-N map
      p8_await_selects(JIT_HERE);
      if (lane == 0 && audio) p8_audio_selects(S);   // audio mode: its own 8 sets from weight set 0
      else if (lane == 0) {
        xml_stats(S);
        smatch_select(S);
        record_select(S);
        text_select(S);
        exe_select(S);
        if (S.m.ncxt != MAIN_SET_FIRST || S.m.base != MAIN_SET_BASE) S.error |= ERR_MIXER_ALIAS;
        S.m.ncxt = N_SETS;
      }
    } else if (byte_start) {
      // ---- byte boundary, the text chain (warps 13-15): state on one lane, the three stemmers of a completed word a warp
      // each, then the 33 contexts side by side. Nothing else reads the text model before the join (in audio mode it does
      // not run: the three warps go straight to the join)
      P8_M0;
      if (!audio) {
        if (tid == P8_WARP_TEXT * 32) sh.text_pending = text_update_a(S);
        p8_sync_text(JIT_HERE);
        if (sh.text_pending) {
          const int split = S.text.stem_split;
          const int i = warp == P8_WARP_TEXT ? LANG_EN : (warp == P8_WARP_TEXT + 1 ? LANG_FR : LANG_DE);
          if (lane == 0 && i >= split) text_stem(S, i);
          p8_sync_text(JIT_HERE);
          if (tid == P8_WARP_TEXT * 32) {
            text_stem_mid(S);
            for (int j = split - 1; j > LANG_UNKNOWN; --j) text_stem(S, j);
            text_update_b(S);
          }
        }
        if (warp == P8_WARP_TEXT) {
          __syncwarp();
          const int n = text_contexts(S, CtxSel{lane, 32});
          __syncwarp();
          if (lane == 0) { S.text.map.index = n; P8_M(38); }
        }
      }
      p8_join_arrive(JIT_HERE);
    } else {
      // ---- inside a byte, warps 13-15: single-lane units beside the maps; the apply runs while lane 0 numbers a clashing bit
      {
        P8_M0;
        p8_probe_units(sh, warp, lane, y, c0, bpos, audio);
        __syncwarp();
        if (lane == 0) P8_M(24 + warp);
      }
      p8_join_sync(JIT_HERE);
      {
        P8_M0;
        p8_apply_units(sh, warp, lane, y, c0, bpos, audio);
        __syncwarp();
        if (lane == 0) P8_M(48 + warp);
      }
    }
  } else {
    if (tid == 0) { S.m.nx = S.m.base = S.m.ncxt = 0; }
    if (byte_start) {
      // ---- byte boundary: the new contexts, as chains of warps that meet at the join (lane map: DESIGN 4.5)
      {
        P8_M0;
        if (warp >= P8_WARP_D) {
          // the D-chain: order-N and x86 contexts -> their history maps and the single-lane units -> the sparse and record
          // models, which consume the order-N map's result and the match length of this bit
          // (in audio mode the order-N map, the match model and the record model only)
          if (audio && warp == P8_MAP_WARPS - 1) p8_unit_offsets(sh, lane, true, true);
          if (tid == P8_CM2_TID0) ordern_byte(S);
          else if (tid == P8_TID_MATCH && !audio) exe_byte(S);
          else if ((tid == P8_CM2_TID0 + 1 || tid == P8_CM2_TID0 + 2) && !audio) cm2_begin(p8_cm2(S, tid - P8_CM2_TID0), y, 0);
          p8_sync_dchain(JIT_HERE);
          if (tid == P8_CM2_TID0) P8_M(31);
          p8_probe_cm2(sh, tid, bpos, audio ? 1 : 5);
          p8_probe_single(sh, tid, y, c0, bpos, audio);
          p8_sync_dchain(JIT_HERE);
          if (tid == P8_CM2_TID0) P8_M(32);
          p8_apply_cm2(sh, tid, y, bpos, audio ? 1 : 5);
          p8_sync_dchain(JIT_HERE);
          if (tid == P8_CM2_TID0) P8_M(33);
          const int ismatch = ilog(T, S.match.length);
          if (tid == P8_TID_MATCH && !audio) { sparse_byte(S, ismatch, sh.res2[0]); P8_M(34); }
          else if (tid == P8_TID_W10 && !audio) { sparse1_byte(S, ismatch, sh.res2[0], sh.snap); P8_M(35); }
          else if (tid == P8_TID_W11) { record_byte(S, audio ? FT_AUDIO : S.filetype); record_pre(S); P8_M(36); }
        } else if (audio) {         // audio mode: the eight OLS predictors of the channel, a warp each (OLS 6 and 7 share warp 6)
          p8_audio_ols_warp(sh, warp, lane);
          if (warp == 6) p8_audio_ols_warp(sh, 7, lane);
        } else if (warp < 3) {      // a linear predictor per warp, then the map behind it
          p8_ols_byte_warp(sh, warp, lane);
          if (lane == 0) { Out o = p8_out(sh, sh.unit_off[48 + warp]); linear_small(S, o, warp); }
        } else if (warp == 5) {     // the word model: state on one lane, its 57 contexts side by side
          if (lane == 0) word_update(S);
          __syncwarp();
          const int n = word_contexts(S, CtxSel{lane, 32});
          __syncwarp();
          if (lane == 0) { S.word.cm.cn = n; word_finish(S); }
        } else if (lane == 0) {
          switch (warp) {
            case 3: xml_byte(S); break;
            case 4: distance_byte(S); record1_byte(S); break;
            case 6: {
              nest_byte(S); indirect_byte(S);
              const u8 W = (u8)buf(S, 1), WW = (u8)buf(S, 2), WWW = (u8)buf(S, 3);
              S.linear.prd[3] = (u8)clip8(W * 2 - WW);
              S.linear.prd[4] = (u8)clip8(W * 3 - WW * 3 + WWW);
              for (int r = 3; r < 5; ++r) { Out o = p8_out(sh, sh.unit_off[48 + r]); linear_small(S, o, r); }
            } break;
          }
        }
        if (lane == 0 && warp < P8_WARP_D) P8_M(24 + warp);
      }
      p8_join_sync(JIT_HERE);
      p8_signal_selects(JIT_HERE);
      P8_T(2);
      // ---- the sixteen 7-slot maps in one probe / number / apply (their random draws are shared), the text history map beside them
      if (warp < P8_WARP_D) p8_probe_cm(sh, tid, y, c0, bpos);
      else p8_probe_cm2(sh, tid, bpos, 2);
      p8_sync_maps(JIT_HERE);
      P8_T(6);
      if (sh.any_clash) { P8_M0; p8_number(sh, tid, y, c0, bpos); p8_sync_maps(JIT_HERE); if (tid == 0) P8_M(P8_PROF_NUMBER + bpos); }
      P8_T(7);
      p8_apply_cm(sh, tid, y, c0, bpos);
      p8_apply_cm2(sh, tid, y, bpos, 2);
      p8_apply_small(sh, tid, y, bpos, audio);
      if (audio && tid >= P8_CM2_TID0 && tid < P8_CM2_TID0 + AUDIO_N_SCM) p8_audio_scm(sh, tid - P8_CM2_TID0);   // behind the predictions
      p8_sync_maps(JIT_HERE);
      P8_T(8);
    } else {
      // ---- inside a byte: probe / number / apply, all map families side by side, the single-lane units on warps 9-11 and
      // 13-15 (lane map: P8_W_*)
      {
        P8_M0;
        if (warp < 7) p8_probe_cm(sh, tid, y, c0, bpos);
        else if (warp < P8_W_MATCH) p8_probe_cm2(sh, tid, bpos, 7);
        else p8_probe_units(sh, warp, lane, y, c0, bpos, audio);
        __syncwarp();
        if (lane == 0) P8_M(24 + warp);
      }
      p8_join_sync(JIT_HERE);
      p8_signal_selects(JIT_HERE);
      P8_T(3);
      if (sh.any_clash) { P8_M0; p8_number(sh, tid, y, c0, bpos); p8_sync_maps(JIT_HERE); if (tid == 0) P8_M(P8_PROF_NUMBER + bpos); }
      P8_T(7);
      {
        P8_M0;
        if (warp < 7) p8_apply_cm(sh, tid, y, c0, bpos);
        else if (warp < P8_W_IMAP) p8_apply_cm2(sh, tid, y, bpos, 7);
        else p8_apply_units(sh, warp, lane, y, c0, bpos, audio);
        __syncwarp();
        if (lane == 0) P8_M(48 + warp);
      }
      p8_sync_maps(JIT_HERE);
      P8_T(8);
    }
    // ---- epilogues, ModelStats, the 28 selector sets in the reference's order
    if (tid == 0) {
      P8_U0;
      if (bpos == 7) {
        for (int k = 0; k < P8_N_CM; ++k) p8_cm(S, k).cn = 0;
        for (int k = 0; k < P8_N_CM2; ++k) p8_cm2(S, k).index = 0;
      }
      if (!audio) main_select_fixed(S, sh.res2[0]);      // sets 19..27; warp 12 writes 0..18 (and the count) beside this
      Mixer& m = S.m;
      m.nx = sh.unit_off[P8_N_UNITS];
      m.n2 = m.nx;
      while (m.nx & 7) m.tx[m.nx++] = 0;
      P8_U(23);
      CENSUS_P8_BIT(S.sparse.cm.t, sh.clash, sh.clash2, sh.flag_mask1, P8_CM_LANES, bpos);   // the bit's verdicts are final here
#ifdef P8_PROF
      prof_clash = sh.any_clash != 0;
#endif
    }
  }
  JIT_SYNCTHREADS();     // warp 12 joins
  P8_T(9);
  // ---- hand the bit over. Only warp 0 reads the scalars: its lane 0 is the one that changes them at the next bit's start,
  // the other warps' data (inputs, codes) changes only after the next bit's first barrier.
  const int slot = (int)(t % P8_RING);
  if (t >= P8_RING) mbar_wait(&sh.empty[slot], (t / P8_RING - 1) & 1, JIT_HERE);
  P8_T(10);
  {
    const Mixer& m = S.m;
    P8Slot& d = ring[slot];
    if (warp == 0) {
      if (lane < N_SETS) d.cxt[lane] = m.cxt[lane];
      if (lane == 0) {
        d.n2 = m.n2; d.nx = m.nx; d.ncxt = m.ncxt; d.base = m.base;
        d.c0 = S.c0; d.bpos = S.bpos; d.blpos = S.blpos; d.st_type = S.st_type; d.c4 = S.c4; d.st_match_length = S.st_match_length;
        d.c1 = (u8)buf(S, 1); d.st_match_expected = S.st_match_expected; d.st_text_first = S.st_text_first; d.st_text_mask = S.st_text_mask;
        d.relayout = sh.u.md.ncxt_handed != m.ncxt; sh.u.md.ncxt_handed = m.ncxt;
      }
    }
    for (int q = tid; q < m.nx / 8; q += P8_THREADS) reinterpret_cast<uint4*>(d.tx)[q] = reinterpret_cast<const uint4*>(m.tx)[q];
    for (int q = tid; q < (m.n2 + 1) / 2; q += P8_THREADS) reinterpret_cast<u32*>(d.codes)[q] = reinterpret_cast<const u32*>(S.codes)[q];
    __syncwarp();
    if (lane == 0) mbar_arrive_remote(&sh.full[slot], 1, JIT_HERE);
  }
  P8_T(11);
#ifdef P8_PROF
  // the other lanes record nothing before the next bit's first barrier, which lane 0 reaches after this
  if (tid == 0) {
    const int row = S.bpos == 0 ? 0 : 2 + 2 * (S.bpos == 2 || S.bpos == 5) + prof_clash;
    sh.prof_acc[P8_PROF_N] = 1;
    for (int k = 0; k < P8_PROF_SLOTS; ++k) {
      atomicAdd(&g_p8_prof[row ? 1 : 0][k], sh.prof_acc[k]);
      if (row) atomicAdd(&g_p8_prof[row][k], sh.prof_acc[k]);
      sh.prof_acc[k] = 0;
    }
  }
#endif
}
static_assert(offsetof(p8::State, codes) % 4 == 0 && p8::N_IN % 2 == 0, "codes are handed over in 4-byte words");

// The mixer CTA's part of bit t of a launch (y, and nb as in p8_model_bit): the SGD of the sets picked for bit t-1 on its
// inputs (tx_prev) and of the final mixer, which need only the bit and so run beside the model CTA's work on it; then, from
// ring slot t % P8_RING, the 28 dot products, squash, the final mixer and the SSE stage. S.codes then holds the 1591 codes
// after the bit.
__device__ void p8_mix_bit(P8Shared& sh, u32 t, int y, int nb, const short* tx_prev, int tid) {
  using namespace p8;
  State& S = sh.S;
  const p8::Tables& T = *S.T;
  Mixer& m = S.m;
  const int warp = tid >> 5, lane = tid & 31;
  const int slot = (int)(t % P8_RING);
  const P8Slot& in = sh.u.mx.ring[slot];
#ifdef P8_PROF
  if (tid == 0) { sh.prof_t = clock64(); sh.prof_dst = g_p8_prof[nb == 0 ? 0 : 1]; }
#endif
  // ---- SGD of the previous bit's sets and of the final mixer
  p8_sgd(sh, tx_prev, y, tid);
  if (warp == P8_WARPS - 1) {
    const int err = ((y << 12) - m.pr2) * 7;
    if (err && lane < m.nx2) m.w2[lane] = train_one(m.tx2[lane], m.w2[lane], err);
  }
  P8_T(17);
  // ---- the bit's inputs and selectors (set 26 from this CTA's last prediction)
  mbar_wait(&sh.full[slot], (t / P8_RING) & 1, JIT_HERE);
  P8_T(16);
  if (tid < N_SETS) m.cxt[tid] = tid == MAIN_SET_FIRST + 7 && in.ncxt == N_SETS ? MAIN_SET_PR + S.last_prediction / 16 : in.cxt[tid];
  JIT_SYNCTHREADS();
  if (tid == 0) {
    if (t > 0) mbar_arrive_remote(&sh.empty[(t - 1) % P8_RING], 0, JIT_HERE);   // tx_prev was slot t-1's
    S.st_misses += S.st_misses + (u64)((S.pr >> 11) != y);               // bit_begin's line, on this CTA's prediction
    S.y = y; S.c0 = in.c0; S.bpos = in.bpos; S.blpos = in.blpos; S.c4 = in.c4; S.st_type = in.st_type;
    S.st_match_length = in.st_match_length; S.st_match_expected = in.st_match_expected;
    S.st_text_first = in.st_text_first; S.st_text_mask = in.st_text_mask;
    m.n2 = in.n2; m.nx = in.nx; m.ncxt = in.ncxt; m.base = in.base;
  }
  // ---- the 28 dot products over the cached sets (a selector that moved: write back, load)
  {
    for (int q = tid; q < (in.n2 + 1) / 2; q += P8_THREADS) reinterpret_cast<u32*>(S.codes)[q] = reinterpret_cast<const u32*>(in.codes)[q];
    if (warp == P8_WARPS - 2 && lane < in.ncxt) {        // two selectors on one weight set would need the reference's sequential SGD
      bool dup = false;
      for (int j = 0; j < lane; ++j) dup = dup || m.cxt[j] == m.cxt[lane];
      if (dup) S.error |= ERR_MIXER_ALIAS;
    }
    // A change of layout (ordinary <-> audio mode, 28 <-> 8 sets) gives the cached rows' selectors other meanings: a set still
    // cached under one selector could be fetched fresh from HBM under another. Such a bit writes every row back first and
    // fetches its sets on warp 0 alone.
    if (in.relayout && warp == 0) p8_relayout(sh, in, lane);
    for (int i = in.relayout ? N_SETS : warp; i < in.ncxt; i += P8_WARPS) {
      short* row = sh.u.mx.wc[i];
      const int set = m.cxt[i], old = sh.wc_set[i];
      if (old != set) {
        if (old >= 0) p8_row_store(m.w + (size_t)old * N_IN, row, lane);
        p8_row_load(row, m.w + (size_t)set * N_IN, lane);
        __syncwarp();
        if (lane == 0) sh.wc_set[i] = set;
      }
      int acc = 0;
      const int n8 = in.nx >> 3;
      for (int q = lane; q < n8; q += 32) {
        const uint4 wv = *reinterpret_cast<const uint4*>(row + q * 8);
        const uint4 xv = *reinterpret_cast<const uint4*>(in.tx + q * 8);
        const short* w = reinterpret_cast<const short*>(&wv);
        const short* x = reinterpret_cast<const short*>(&xv);
#pragma unroll
        for (int e = 0; e < 8; e += 2) acc += dot_pair(x + e, w + e);
      }
      acc = __reduce_add_sync(0xffffffffu, acc);
      if (lane == 0) sh.dot[i] = acc;
    }
  }
  JIT_SYNCTHREADS();
  P8_T(18);
  // ---- squash, final mixer, SSE stage (one warp)
  if (warp == 0) {
    const int base = m.n2, n = m.ncxt, nx2 = (n + 7) & ~7;
    int x = 0;
    if (lane < n) {
      const int pr = squash(T, (int)((u32)sh.dot[lane] * 9u) >> 9);
      m.pr[lane] = pr;
      x = stretch(T, pr);
      S.codes[base + lane] = (u16)squash(T, x);
    }
    m.tx2[lane] = (short)x;
    __syncwarp();
    int z = 2 * lane < nx2 ? dot_pair(m.tx2 + 2 * lane, m.w2 + 2 * lane) : 0;
    z = __reduce_add_sync(0xffffffffu, z);
    const int pr2 = squash(T, z >> 9);
    if (lane == 0) { m.nx2 = nx2; m.pr2 = pr2; }
    __syncwarp();
    p8_sse_warp(sh, pr2, in.c1, lane);
  }
  JIT_SYNCTHREADS();
  P8_T(19);
}

// Both CTAs: state block and hot tables into shared memory, the ring's barriers; the mixer CTA: the pending weight sets.
__device__ __forceinline__ const p8::Tables* p8_enter(P8Shared& sh, p8::State* g, int tid, int rank) {
  p8_copy_words(&sh.S, g, sizeof(p8::State), tid);
  JIT_SYNCTHREADS();
  const p8::Tables* gT = sh.S.T;
  p8_copy_words(sh.tab, gT, p8::TABLES_HOT_BYTES, tid);
  if (tid < p8::N_SETS) sh.wc_set[tid] = -1;
  if (rank == 0) for (int k = tid; k < P8_CM_LANES; k += P8_THREADS) sh.u.md.cc.valid[k] = 0;   // shared memory is new
  if (rank == 0 && tid == 0) sh.u.md.ncxt_handed = sh.S.m.ncxt;
#ifdef P8_PROF
  for (int k = tid; k < P8_PROF_SLOTS; k += P8_THREADS) sh.prof_acc[k] = 0;
#endif
  if (tid == 0) {
    for (int i = 0; i < P8_RING; ++i) {
      if (rank == 0) mbar_init(&sh.empty[i], 1);
      else mbar_init(&sh.full[i], P8_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  JIT_SYNCTHREADS();
  if (tid == 0) sh.S.T = reinterpret_cast<const p8::Tables*>(sh.tab);
  const int warp = tid >> 5, lane = tid & 31;
  if (rank == 1) {
    for (int i = warp; i < sh.S.m.ncxt; i += P8_WARPS) {
      p8_row_load(sh.u.mx.wc[i], sh.S.m.w + (size_t)sh.S.m.cxt[i] * p8::N_IN, lane);
      if (lane == 0) sh.wc_set[i] = sh.S.m.cxt[i];
    }
  }
  jit_cluster_sync(cooperative_groups::this_cluster(), JIT_HERE);   // the barriers exist before the other CTA arrives on them
  return gT;
}
// Each CTA writes back the fields it owns: the mixer CTA `m`, the APMs and `codes` (with the inputs of the last bit it
// took, `last` = its ring slot, or none), the model CTA everything before `m` and `error`, after taking `pr`,
// `last_prediction` and `st_misses` from the mixer CTA and OR-ing its error bits into its own.
__device__ __forceinline__ void p8_leave(P8Shared& sh, p8::State* g, const p8::Tables* gT, int tid, int rank, int last) {
  using namespace p8;
  cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
  const int warp = tid >> 5, lane = tid & 31;
  if (rank == 1) {
    for (int i = warp; i < N_SETS; i += P8_WARPS)
      if (sh.wc_set[i] >= 0) p8_row_store(sh.S.m.w + (size_t)sh.wc_set[i] * N_IN, sh.u.mx.wc[i], lane);
    if (last >= 0) for (int q = tid; q < sh.S.m.nx / 8; q += P8_THREADS) reinterpret_cast<uint4*>(sh.S.m.tx)[q] = reinterpret_cast<const uint4*>(sh.u.mx.ring[last].tx)[q];
  }
  jit_cluster_sync(cluster, JIT_HERE);
  if (rank == 0 && tid == 0) {
    const State& X = cluster.map_shared_rank(&sh, 1)->S;
    sh.S.pr = X.pr; sh.S.last_prediction = X.last_prediction; sh.S.st_misses = X.st_misses;
    sh.S.error |= X.error;
    sh.S.T = gT;
  }
  jit_cluster_sync(cluster, JIT_HERE);   // the mixer CTA's shared memory stays until the model CTA has read it
  const size_t m0 = offsetof(State, m), e0 = offsetof(State, error);
  static_assert(offsetof(State, m) % 4 == 0 && offsetof(State, error) % 4 == 0, "state block is copied word by word");
  if (rank == 0) {
    p8_copy_words(g, &sh.S, m0, tid);
    p8_copy_words((char*)g + e0, (const char*)&sh.S + e0, sizeof(State) - e0, tid);
  } else {
    p8_copy_words((char*)g + m0, (const char*)&sh.S + m0, e0 - m0, tid);
  }
}

// Bulk: cluster b (CTAs 2b, 2b+1) serves stream b of the launch group: writes ext[t][431..2021] for every bit t of the sub-chunk.
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(P8_THREADS, 1) paq8_kernel(const ChunkArgs* __restrict__ args_all) { jit_entry(JK_PAQ8);
  extern __shared__ __align__(16) unsigned char p8_raw[];
  P8Shared& sh = *reinterpret_cast<P8Shared*>(p8_raw);
  const ChunkArgs a = args_all[blockIdx.x >> 1];
  if (a.paq8 == nullptr) return;
  const int tid = threadIdx.x;
  const int rank = (int)cooperative_groups::this_cluster().block_rank();
  p8::State* g = (p8::State*)a.paq8;
  const p8::Tables* gT = p8_enter(sh, g, tid, rank);
  const u32 n_bits = a.n_bytes * 8;
  if (rank == 0) {
    P8Slot* ring = cooperative_groups::this_cluster().map_shared_rank(&sh, 1)->u.mx.ring;
    for (u32 t = 0; t < n_bits; ++t) {
      const int y = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      p8_model_bit(sh, ring, t, y, (int)((t + 1) & 7), tid);
    }
  } else {
    for (u32 t = 0; t < n_bits; ++t) {
      if (!a.pretrain) {
        u16* out = a.ext_gen + (size_t)t * N_EXT + 431;
        for (int k = tid; k < p8::N_OUT; k += P8_THREADS) out[k] = sh.S.codes[k];
      }
      const int y = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      p8_mix_bit(sh, t, y, (int)((t + 1) & 7), t == 0 ? sh.S.m.tx : sh.u.mx.ring[(t - 1) % P8_RING].tx, tid);
    }
  }
  p8_leave(sh, g, gT, tid, rank, n_bits ? (int)((n_bits - 1) % P8_RING) : -1);
}

// Lock-step: one bit per launch, a one-slot handover; the codes for the next Predict() land in ext_bit[431..2021].
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(P8_THREADS, 1) paq8_bit_kernel(p8::State* g, int y, u16* ext_bit, const u32* dbit) { jit_entry(JK_PAQ8_BIT);
  if (dbit) y = (int)dbit[0];
  extern __shared__ __align__(16) unsigned char p8_raw[];
  P8Shared& sh = *reinterpret_cast<P8Shared*>(p8_raw);
  const int tid = threadIdx.x;
  const int rank = (int)cooperative_groups::this_cluster().block_rank();
  const int nb = (g->bpos + 1) & 7;       // read from HBM: the shared copy is being updated by lane 0 inside p8_model_bit
  const p8::Tables* gT = p8_enter(sh, g, tid, rank);
  if (rank == 0) {
    p8_model_bit(sh, cooperative_groups::this_cluster().map_shared_rank(&sh, 1)->u.mx.ring, 0, y, nb, tid, true);
  } else {
    p8_mix_bit(sh, 0, y, nb, sh.S.m.tx, tid);
    if (ext_bit) for (int k = tid; k < p8::N_OUT; k += P8_THREADS) ext_bit[431 + k] = sh.S.codes[k];
  }
  p8_leave(sh, g, gT, tid, rank, 0);
}

}  // namespace cmixb200
