// cmix_b200/csrc/paq8_model.h — the resident PAQ8 model (SURVEY §8 row a13) as host/device code.
//
// What it reproduces: reference src/models/paq8.cpp — `Predictor::update` (:8248-8362), `contextModel2` (:8101-8206)
// on its non-image / non-audio / non-JPEG path, the two bucketed context-map flavours (:1010-1359), the int16 mixer
// with 28 selected weight sets and its final 28-input mixer (:513-598), StateMap / StateMap32 / APM / APM1 (:600-710),
// match and sparse-match models (:3520-3843), sparse / distance / pic / record / word / nest / indirect / XML / text /
// x86 / linear-prediction models, the DMC forest (:7614-7823), and the 1591 exported 12-bit codes (:497-511).
// Everything is integer arithmetic except the three 32-tap OLS predictors (double, evaluated in the reference's order
// without contraction). Image, audio and JPEG blocks are NOT modelled: a stream that reaches one raises `unsupported`
// (sticky, reported by the C-ABI) instead of producing numbers that differ from the reference.
//
// Organisation mirrors fxcm_model.h: one flat state block per stream, bit-history cells addressed by byte offsets into
// their tables, per-bit work cut into units with disjoint state and disjoint input slices. One cross-unit dependency is
// inherent: the 7-slot context maps draw from ONE global pseudo-random sequence when ageing high-count states
// (paq8.cpp:1075, :152-165), in program order over all maps; the draws of a bit are therefore numbered by a prefix count
// over the units before any unit applies them (p8_rnd_* below).
#ifndef CMIXB200_PAQ8_MODEL_H
#define CMIXB200_PAQ8_MODEL_H

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define P8_HD __host__ __device__
#else
#define P8_HD
#endif
// Host census of the device-only paths (tools/census.h): called where the in-order loops start, with the state the device's
// per-bit probe sees. Empty in every product build.
#ifndef P8_CENSUS_CM
#define P8_CENSUS_CM(T, m, y, c0, bp) do { } while (0)
#endif
#ifndef P8_CENSUS_CM2
#define P8_CENSUS_CM2(m, bpos) do { } while (0)
#endif
// Host test of the clash rule (tools/census.h with -DCENSUS_PERMUTE / -DCENSUS_REVERSE): may evaluate cm_mix's /
// cm2_mix_body's contexts in another order and return. Empty in every product build.
#ifndef P8_CM_ORDER
#define P8_CM_ORDER(T, m, o, rnd, y, c0, bp, c1) do { } while (0)
#endif
#ifndef P8_CM2_ORDER
#define P8_CM2_ORDER(m, o, y, bpos) do { } while (0)
#endif
// Profiling build of the device (paq8.cuh with -DP8_PROF): the end of leg k of a 7-slot map context's bit. Empty elsewhere.
#ifndef P8_LEG
#define P8_LEG(k) do { } while (0)
#endif

namespace cmixb200 {
namespace p8 {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int64_t i64;

enum { N_IN = 1552, N_SETS = 28, N_OUT = 1591, N_WSETS = 77472, BUF_BITS = 30, P8_NULL = -1 };
#define P8_BUF_MASK ((1u << 30) - 1)
enum Filetype { FT_DEFAULT, FT_HDR, FT_JPEG, FT_EXE, FT_TEXT, FT_IMAGE1, FT_IMAGE4, FT_IMAGE8, FT_IMAGE8GRAY, FT_IMAGE24, FT_IMAGE32, FT_AUDIO };

P8_HD inline int imin(int a, int b) { return a < b ? a : b; }
P8_HD inline int imax(int a, int b) { return a < b ? b : a; }
P8_HD inline int iabs(int a) { return a < 0 ? -a : a; }
P8_HD inline u32 umin(u32 a, u32 b) { return a < b ? a : b; }

// ---------------------------------------------------------------- read-only tables (host-built, paq8_host.h)
struct Tables {
  const u8* ilog;        // -> ilog_store below (kept out of line so that everything before ilog_store can be staged in shared memory)
  u8 state[256][4];      // State_table (paq8.cpp:277-341)
  u16 squash[4096];      // index p + 2048 (:345-367)
  short stretch[4096];   // (:369-387)
  int dt[1024];          // 16384 / (i + i + 3) (:8244)
  u8 ascii_group_c0[254], ascii_group[128];   // (:3039-3068)
  // x86 decoder tables (:6580-7040) as produced by the reference's own initialisers
  u8 exe_t1[256], exe_t2[256], exe_t3_38[256], exe_t3_3a[256], exe_tx[32];
  u8 exe_c1[256], exe_c2[256], exe_c3_38[256], exe_c3_3a[256], exe_cx[32];
  u8 exe_invalid64[19], exe_prefix64[8];
  alignas(16) u8 ilog_store[65536];   // (:253-266)
};
enum { TABLES_HOT_BYTES = offsetof(Tables, ilog_store) };
static_assert(TABLES_HOT_BYTES % 16 == 0, "the hot part of the tables is copied in 16-byte words");

P8_HD inline int squash(const Tables& T, int p) { if (p > 2047) return 4095; if (p < -2047) return 0; return T.squash[p + 2048]; }
P8_HD inline int stretch(const Tables& T, int p) { return T.stretch[p]; }
P8_HD inline int ilog(const Tables& T, u32 x) { return T.ilog[x & 0xffff]; }
P8_HD inline int llog(const Tables& T, u32 x) {
  if (x >= 0x1000000) return 256 + ilog(T, x >> 16);
  if (x >= 0x10000) return 128 + ilog(T, x >> 8);
  return ilog(T, x);
}
P8_HD inline u32 bitcount(u32 v) {
  v -= ((v >> 1) & 0x55555555); v = ((v >> 2) & 0x33333333) + (v & 0x33333333); v = ((v >> 4) + v) & 0x0f0f0f0f;
  v = ((v >> 8) + v) & 0x00ff00ff; v = ((v >> 16) + v) & 0x0000ffff; return v;
}
P8_HD inline u32 ilog2(u32 x) { x |= x >> 1; x |= x >> 2; x |= x >> 4; x |= x >> 8; x |= x >> 16; return bitcount(x >> 1); }

// hashes (paq8.cpp:714-776)
// code that runs once per byte (or more rarely) stays out of line on the device: the per-bit path is instruction-fetch sensitive
#if defined(__CUDACC__)
#define P8_COLD __noinline__
#else
#define P8_COLD
#endif
#define P8_PHI64 0x9E3779B97F4A7C15ull
#define P8_M1 0x993DDEFFB1462949ull
#define P8_M2 0xE9C91DC159AB0D2Dull
#define P8_M3 0x83D6A14F1B0CED73ull
#define P8_M4 0xA14F1B0CED5A841Full
#define P8_M5 0xC0E51314A614F4EFull
#define P8_M6 0xDA9CC2600AE45A27ull
#define P8_M7 0x826797AA04A65737ull
P8_HD inline u32 finalize64(u64 h, int bits) { return (u32)(h >> (64 - bits)); }
P8_HD inline u64 checksum64(u64 h, int bits, int cbits) { return h >> (64 - bits - cbits); }
P8_HD inline u64 hash(u64 a) { return (a + 1) * P8_PHI64; }
P8_HD inline u64 hash(u64 a, u64 b) { return (a + 1) * P8_PHI64 + (b + 1) * P8_M1; }
P8_HD inline u64 hash(u64 a, u64 b, u64 c) { return (a + 1) * P8_PHI64 + (b + 1) * P8_M1 + (c + 1) * P8_M2; }
P8_HD inline u64 hash(u64 a, u64 b, u64 c, u64 d) { return (a + 1) * P8_PHI64 + (b + 1) * P8_M1 + (c + 1) * P8_M2 + (d + 1) * P8_M3; }
P8_HD inline u64 hash(u64 a, u64 b, u64 c, u64 d, u64 e) { return (a + 1) * P8_PHI64 + (b + 1) * P8_M1 + (c + 1) * P8_M2 + (d + 1) * P8_M3 + (e + 1) * P8_M4; }
P8_HD inline u64 hash(u64 a, u64 b, u64 c, u64 d, u64 e, u64 f) {
  return (a + 1) * P8_PHI64 + (b + 1) * P8_M1 + (c + 1) * P8_M2 + (d + 1) * P8_M3 + (e + 1) * P8_M4 + (f + 1) * P8_M5;
}
P8_HD inline u64 hash(u64 a, u64 b, u64 c, u64 d, u64 e, u64 f, u64 g) {
  return (a + 1) * P8_PHI64 + (b + 1) * P8_M1 + (c + 1) * P8_M2 + (d + 1) * P8_M3 + (e + 1) * P8_M4 + (f + 1) * P8_M5 + (g + 1) * P8_M6;
}
P8_HD inline u64 combine64(u64 seed, u64 x) { return hash(seed + x); }

// ---------------------------------------------------------------- elementary adaptive maps
struct Sm16 { u16* t; int cxt; };                      // StateMap (paq8.cpp:623-643)
struct Sm32 { u32* t; int cxt, n; };                   // StateMap32 / APM (:645-710)
struct Apm1 { u16* t; int index; };                    // APM1 (:600-621)
struct Scm { u16* data; int context, mask, stride, bcount, btotal, B, cp; };   // SmallStationaryContextMap (:891-919)
struct Stm { u32* data; int context, mask, maskbits, stride, bcount, btotal, B, cp; };   // StationaryMap (:935-974)
struct Imap { u8* data; Sm32 map; int context, mask, maskbits, stride, bcount, btotal, B, cp; };   // IndirectMap (:976-1008)
template <class T> struct ICtx { T* data; u32 ctx, ctx_mask, input_mask, input_bits; };   // IndirectContext (:1469-1494)

// 7-slot context map (ContextMap, :1010-1145) and its history-aware sibling (ContextMap2, :1164-1359): bucket table of
// 64-byte buckets {u16 chk[7]; u8 last; u8 bh[7][7]}, cells addressed by byte offset, -1 = null.
enum { CM_CAP = 64, CM2_CAP = 36 };
struct Cm {
  u8* t; u16* sm_t;      // buckets; [C][256] StateMap cells
  u32 mask; int hashbits, C, cn;
  int cp[CM_CAP], cp0[CM_CAP], runp[CM_CAP], sm_cxt[CM_CAP];
  u32 cxt[CM_CAP]; u16 chk[CM_CAP];
};
struct Cm2 {
  u8* t; u32* m6_t; u32* m8_t; u32* m12_t;   // buckets; [C][72], [C][256], [C][4608] StateMap32 cells
  u32 mask; int hashbits, C, index;
  int bs[CM2_CAP], bs0[CM2_CAP], bh[CM2_CAP], m6_cxt[CM2_CAP], m8_cxt[CM2_CAP], m12_cxt[CM2_CAP];
  u32 cxt[CM2_CAP]; u16 chk[CM2_CAP]; u8 has_history[CM2_CAP];
  u32 bits; u8 last_byte, last_bit, bit_pos, pad;
};
struct Rcm { u8* t; u32 mask; int hashbits; int cp; };   // RunContextMap over BH<4> (:778-813, :857-885)

// DMC (:7614-7775)
struct DmcNode { u16 c0, c1; u32 nx0, nx1; };
struct Dmc { DmcNode* t; Sm32 sm; u32 size, top, curr, threshold, threshold_fine, extra; };

struct Mixer {
  short* w;              // [N_WSETS][N_IN] dense (the reference allocates sets lazily; zero-use sets never differ from fresh ones)
  short* w2;             // final mixer: one set of 32
  alignas(16) short tx[N_IN]; alignas(16) short tx2[32];
  int cxt[N_SETS], pr[N_SETS];
  int ncxt, base, nx, nx2, pr2, n2;
};

struct Out { const Tables* T; short* tx; u16* codes; int n; };   // mixer input + export cursor (m.add, :565-568)
P8_HD inline void add(Out& o, int x) { o.codes[o.n] = (u16)squash(*o.T, x); o.tx[o.n] = (short)x; ++o.n; }

// ---------------------------------------------------------------- primitives
P8_HD inline int sm16_p(Sm16& s, int y, int cx) {
  s.t[s.cxt] = (u16)(s.t[s.cxt] + (((y << 16) - (int)s.t[s.cxt] + 128) >> 8));
  s.cxt = cx;
  return s.t[cx] >> 4;
}
P8_HD inline void sm32_update(const Tables& T, Sm32& s, int y, int limit) {
  u32 p0 = s.t[s.cxt];
  const int n = p0 & 1023, pr = (int)(p0 >> 10);
  if (n < limit) ++p0; else p0 = (p0 & 0xfffffc00u) | (u32)limit;
  const int target = y << 22;
  const u32 delta = (u32)((target - pr) >> 3) * (u32)T.dt[n];
  p0 += delta & 0xfffffc00u;
  s.t[s.cxt] = p0;
}
// StateMap32::p with the loads hoisted: `old` is t[old_cxt] read before any store of this bit, `fresh` is t[cx] read before the
// update below is stored (both from the same table; when cx == old_cxt the updated value is forwarded). Same result as sm32_p.
P8_HD inline u32 sm32_updated(const Tables& T, u32 p0, int y, int limit) {
  const int n = p0 & 1023, pr = (int)(p0 >> 10);
  if (n < limit) ++p0; else p0 = (p0 & 0xfffffc00u) | (u32)limit;
  const int target = y << 22;
  const u32 delta = (u32)((target - pr) >> 3) * (u32)T.dt[n];
  p0 += delta & 0xfffffc00u;
  return p0;
}
P8_HD inline int sm32_p(const Tables& T, Sm32& s, int y, int cx, int limit = 1023) {
  sm32_update(T, s, y, limit);
  s.cxt = cx;
  return (int)(s.t[cx] >> 20);
}
P8_HD inline int apm_p(const Tables& T, Sm32& s, int y, int pr, int cx, int limit = 0xFF) {
  sm32_update(T, s, y, limit);
  pr = (stretch(T, pr) + 2048) * 23;
  const int wt = pr & 0xfff;
  cx = cx * 24 + (pr >> 12);
  s.cxt = cx + (wt >> 11);
  return (int)(((s.t[cx] >> 13) * (u32)(4096 - wt) + (s.t[cx + 1] >> 13) * (u32)wt) >> 19);
}
P8_HD inline int apm1_p(const Tables& T, Apm1& a, int y, int pr, int cxt, int rate = 7) {
  pr = stretch(T, pr);
  const int g = (y << 16) + (y << rate) - y - y;
  a.t[a.index] = (u16)(a.t[a.index] + ((g - (int)a.t[a.index]) >> rate));
  a.t[a.index + 1] = (u16)(a.t[a.index + 1] + ((g - (int)a.t[a.index + 1]) >> rate));
  const int w = pr & 127;
  a.index = ((pr + 2048) >> 7) + cxt * 33;
  return ((int)a.t[a.index] * (128 - w) + (int)a.t[a.index + 1] * w) >> 11;
}
P8_HD inline void scm_set(Scm& c, u32 ctx) { c.context = (int)((ctx & (u32)c.mask) * (u32)c.stride); c.bcount = c.B = 0; }
P8_HD inline void scm_mix(Scm& c, Out& o, int y, int rate = 7, int mul = 1, int div = 4) {
  const Tables& T = *o.T;
  u16& cell = c.data[c.cp];
  cell = (u16)(cell + (((y << 16) - (int)cell + (1 << (rate - 1))) >> rate));
  c.B += (y && c.B > 0);
  c.cp = c.context + c.B;
  const int p = c.data[c.cp] >> 4;
  add(o, (stretch(T, p) * mul) / div);
  add(o, ((p - 2048) * mul) / (div * 2));
  c.bcount++; c.B += c.B + 1;
  if (c.bcount == c.btotal) c.bcount = c.B = 0;
}
P8_HD inline void stm_set_direct(Stm& c, u32 ctx) { c.context = (int)((ctx & (u32)c.mask) * (u32)c.stride); c.bcount = c.B = 0; }
P8_HD inline void stm_set(Stm& c, u64 ctx) { c.context = (int)((finalize64(ctx, c.maskbits) & (u32)c.mask) * (u32)c.stride); c.bcount = c.B = 0; }
P8_HD inline void stm_mix(Stm& c, Out& o, int y, int mul = 1, int div = 4, int limit = 1023) {
  const Tables& T = *o.T;
  u32& cell = c.data[c.cp];
  const u32 count = (u32)imin(imin(limit, 0x3FF), (int)((cell & 0x3FF) + 1));
  int pred = (int)(cell >> 10), err = (y << 22) - pred;
  err = ((err / 8) * T.dt[count]) / 1024;
  pred = imin(0x3FFFFF, imax(0, pred + err));
  cell = ((u32)pred << 10) | count;
  c.B += (y && c.B > 0);
  c.cp = c.context + c.B;
  pred = (int)(c.data[c.cp] >> 20);
  add(o, (stretch(T, pred) * mul) / div);
  add(o, ((pred - 2048) * mul) / (div * 2));
  c.bcount++; c.B += c.B + 1;
  if (c.bcount == c.btotal) c.bcount = c.B = 0;
}
P8_HD inline void imap_set_direct(Imap& c, u32 ctx) { c.context = (int)((ctx & (u32)c.mask) * (u32)c.stride); c.bcount = c.B = 0; }
P8_HD inline void imap_mix(Imap& c, Out& o, int y, int mul, int div, int limit) {
  const Tables& T = *o.T;
  c.data[c.cp] = T.state[c.data[c.cp]][y];
  c.B += (y && c.B > 0);
  c.cp = c.context + c.B;
  const int p1 = sm32_p(T, c.map, y, c.data[c.cp], limit);
  add(o, (stretch(T, p1) * mul) / div);
  add(o, ((p1 - 2048) * mul) / (div * 2));
  c.bcount++; c.B += c.B + 1;
  if (c.bcount == c.btotal) c.bcount = c.B = 0;
}
template <class T> P8_HD inline void ictx_push(ICtx<T>& c, u32 i) { T& v = c.data[c.ctx]; v = (T)(v << c.input_bits); v = (T)(v | (i & c.input_mask)); }
template <class T> P8_HD inline void ictx_select(ICtx<T>& c, u32 i) { c.ctx = i & c.ctx_mask; }
template <class T> P8_HD inline T ictx_get(const ICtx<T>& c) { return c.data[c.ctx]; }

// the global generator (paq8.cpp:152-165)
struct Rnd { u32 table[64]; int i; };
P8_HD inline u32 rnd_next(Rnd& r) { ++r.i; return r.table[r.i & 63] = r.table[(r.i - 24) & 63] ^ r.table[(r.i - 55) & 63]; }

// The bucket a context moves to on the next bit is one of two neighbours (its index ends in the next coded bit): start both loads now.
P8_HD inline void bucket_prefetch2(const u8* t, u32 mask, u32 ctx, u32 add2) {
#if defined(__CUDA_ARCH__)
  asm volatile("prefetch.global.L2 [%0];" ::"l"(t + ((size_t)((ctx + add2) & mask) << 6)));
  asm volatile("prefetch.global.L2 [%0];" ::"l"(t + ((size_t)((ctx + add2 + 1) & mask) << 6)));
#else
  (void)t; (void)mask; (void)ctx; (void)add2;
#endif
}
// bucket probe shared by both map flavours (ContextMap::E::get :1038-1047, Bucket::Find :1174-1190): returns the offset of bh[slot][0]
P8_HD inline int bucket_find(u8* t, u32 bucket, u16 ch) {
  u8* e = t + ((size_t)bucket << 6);
  u16* chk = reinterpret_cast<u16*>(e);
  u8& last = e[14];
  const int bh = (int)(bucket << 6) + 15;
  if (chk[last & 15] == ch) return bh + 7 * (last & 15);
  int worst = 0xffff, idx = 0;
  for (int i = 0; i < 7; ++i) {
    if (chk[i] == ch) { last = (u8)(last << 4 | i); return bh + 7 * i; }
    const int pri = e[15 + 7 * i];
    if (pri < worst && (last & 15) != i && (last >> 4) != i) { worst = pri; idx = i; }
  }
  last = (u8)(0xF0 | idx);
  chk[idx] = ch;
  for (int k = 0; k < 7; ++k) e[15 + 7 * idx + k] = 0;
  return bh + 7 * idx;
}
P8_COLD P8_HD inline void deferred_histories(u8* t, u32 mask, u32 ctx, u16 chk, int cell0) {   // bits 2-7 of a context seen the second time
  const int c = t[cell0 + 4] + 256;
  int p = bucket_find(t, (ctx + (u32)(c >> 6)) & mask, chk);
  t[p] = (u8)(1 + ((c >> 5) & 1));
  t[p + 1 + ((c >> 5) & 1)] = (u8)(1 + ((c >> 4) & 1));
  t[p + 3 + ((c >> 4) & 3)] = (u8)(1 + ((c >> 3) & 1));
  p = bucket_find(t, (ctx + (u32)(c >> 3)) & mask, chk);
  t[p] = (u8)(1 + ((c >> 2) & 1));
  t[p + 1 + ((c >> 2) & 1)] = (u8)(1 + ((c >> 1) & 1));
  t[p + 3 + ((c >> 1) & 3)] = (u8)(1 + (c & 1));
  t[cell0 + 6] = 0;
}

P8_HD inline void cm_set(Cm& m, u64 cx) {
  cx = hash(cx, (u64)m.cn);
  m.cxt[m.cn] = finalize64(cx, m.hashbits);
  m.chk[m.cn] = (u16)(checksum64(cx, m.hashbits, 16) & 0xffff);
  m.cn++;
}
// ---- ContextMap::mix1 (:1069-1145) cut per context, so that a CTA can run the contexts of a map side by side when they touch
// disjoint buckets this bit (paq8.cuh) and walk the contexts that share a bucket in order when they do not (p8_number;
// cm_mix is the in-order loop of the host builds).
// cm_next_state: the aged bit-history state context i would store this bit, BEFORE the random down-step (read-only); -1 = no cell.
P8_HD inline int cm_next_state(const Tables& T, const Cm& m, int i, int y) { return m.cp[i] != P8_NULL ? T.state[m.t[m.cp[i]]][y] : -1; }
P8_HD inline bool cm_draw_hits(u32 r, int ns) { return (u32)(r << ((452 - ns) >> 3)) != 0; }   // `rnd() << ((452-ns)>>3)` (:1075)
// Read-only probe: which slot of `bucket` holds checksum ch (-1 = none: find would replace).
P8_HD inline int bucket_peek(const u8* t, u32 bucket, u16 ch) {
  const u8* e = t + ((size_t)bucket << 6);
  const u16* chk = reinterpret_cast<const u16*>(e);
  const u8 last = e[14];
  if (chk[last & 15] == ch) return last & 15;
  for (int i = 0; i < 7; ++i) if (chk[i] == ch) return i;
  return -1;
}
// The buckets context i reads or writes this bit (at most 5): its live cell bucket, its run-info bucket, the bucket it moves to and,
// on a byte boundary, the two buckets of a deferred history write-back. Returns how many ids were stored.
P8_HD inline int touched_buckets(const u8* t, u32 mask, int cell, int run, u32 ctx, u16 chk, u32 add, int bp, u32* ids) {
  int n = 0;
  if (cell != P8_NULL) ids[n++] = (u32)cell >> 6;
  ids[n++] = (u32)run >> 6;
  if (bp > 1 && t[run] == 0) return n;
  if (bp == 0 || bp == 2 || bp == 5) {
    const u32 b = (ctx + add) & mask;
    ids[n++] = b;
    if (bp == 0) {
      const int slot = bucket_peek(t, b, chk);
      if (slot >= 0) {
        const u8* cell0 = t + ((size_t)b << 6) + 15 + 7 * slot;
        if (cell0[3] == 2) { const int c = cell0[4] + 256; ids[n++] = (ctx + (u32)(c >> 6)) & mask; ids[n++] = (ctx + (u32)(c >> 3)) & mask; }
      }
    }
  }
  return n;
}
P8_HD inline int cm_touched(const Cm& m, int i, int c0, int bp, u32* ids) { return touched_buckets(m.t, m.mask, m.cp[i], m.runp[i], m.cxt[i], m.chk[i], (u32)c0, bp, ids); }
// A staying bit (bp 1, 3, 4, 6, 7) keeps every context of a 7-slot map in its slot: cm_step neither calls bucket_find nor
// updates a run record. Context i then writes only t[cp], in its current slot, and reads only that slot and t[runp], t[runp+1]
// (its StateMap row is its own), so contexts whose slots differ commute. Its keys: the base offsets of its current slot (none
// when the cell is null) and of its run record's slot. Other bits touch whole buckets (cm_touched).
P8_HD inline bool cm_staying(int bp) { return (0xDA >> bp) & 1; }
P8_HD inline int cm_slot_keys(const Cm& m, int i, u32* ids) {
  int n = 0;
  if (m.cp[i] != P8_NULL) ids[n++] = (u32)m.cp0[i];
  ids[n++] = (u32)(m.runp[i] - 3);
  return n;
}
// The input of a context's run record (r0, r1: its count and byte).
P8_HD inline void cm_run_input(const Tables& T, Out& o, int r0, int r1, int c0, int bp) {
  if (((r1 + 256) >> (8 - bp)) == c0) {
    const int b = ((r1 >> (7 - bp)) & 1) * 2 - 1;
    const int c = ilog(T, r0 + 1) << (2 + (~r0 & 1));
    add(o, b * c);
  } else add(o, 0);
}
// The StateMap16 update of the previous bit's cell `so` (sm_old = smt[so]) and the four inputs of the new cell's state s
// (fresh = smt[s], both read before the update is stored).
P8_HD inline int cm_cell_inputs(const Tables& T, Out& o, u16* smt, int so, u16 sm_old, int s, u16 fresh, int y) {
  const u16 upd = (u16)(sm_old + (((y << 16) - (int)sm_old + 128) >> 8));
  if (s == so) fresh = upd;
  smt[so] = upd;
  const int p1 = fresh >> 4;
  const int st = (stretch(T, p1) + 2) >> 2;
  add(o, st); P8_LEG(6);
  add(o, (p1 - 2047 + 4) >> 3);
  const int n0 = -!T.state[s][2], n1 = -!T.state[s][3];
  add(o, st * iabs(n1 - n0));
  const int p0 = 4095 - p1;
  add(o, ((p1 & n0) - (p0 & n1) + 8) >> 4); P8_LEG(7);
  return s > 0;
}
// The cell a context moves to on a staying bit, as its index in the slot (-1: null), from its run record's count r0.
P8_HD inline int cm_stay_cell(int r0, int c0, int bp) {
  if (bp > 1 && r0 == 0) return -1;
  return (bp == 4 || bp == 7) ? 3 + (c0 & 3) : 1 + (c0 & 1);
}
// One context of one bit: store the aged state `ns` (already decided, -1 = no cell), move to the next cell, emit 5 inputs at o.
P8_HD inline int cm_step(Cm& m, int i, Out& o, int ns, int y, int c0, int bp, int c1) {
  const Tables& T = *o.T;
  u8* t = m.t;
  u16* smt = m.sm_t + i * 256;
  const int so = m.sm_cxt[i];
  const u16 sm_old = smt[so];              // loaded before the bucket walk: its address is known from the previous bit
  if (m.cp[i] != P8_NULL) t[m.cp[i]] = (u8)ns;
  if (bp > 1 && t[m.runp[i]] == 0) m.cp[i] = P8_NULL;
  else {
    switch (bp) {
      case 1: case 3: case 6: m.cp[i] = m.cp0[i] + 1 + (c0 & 1); break;
      case 4: case 7: m.cp[i] = m.cp0[i] + 3 + (c0 & 3); break;
      case 2: case 5: m.cp0[i] = m.cp[i] = bucket_find(t, (m.cxt[i] + (u32)c0) & m.mask, m.chk[i]); break;
      default: {
        m.cp0[i] = m.cp[i] = bucket_find(t, (m.cxt[i] + (u32)c0) & m.mask, m.chk[i]);
        if (t[m.cp0[i] + 3] == 2) deferred_histories(t, m.mask, m.cxt[i], m.chk[i], m.cp0[i]);
        u8* rp = t + m.runp[i];
        if (rp[0] == 0) { rp[0] = 2; rp[1] = (u8)c1; }
        else if (rp[1] != c1) { rp[0] = 1; rp[1] = (u8)c1; }
        else if (rp[0] < 254) rp[0] += 2;
        else if (rp[0] == 255) rp[0] = 128;
        m.runp[i] = m.cp0[i] + 3;
      } break;
    }
  }
  if ((bp == 1 || bp == 4) && m.cp[i] != P8_NULL) bucket_prefetch2(t, m.mask, m.cxt[i], (u32)c0 * 2); P8_LEG(4);
  const u8* rp = t + m.runp[i];
  cm_run_input(T, o, rp[0], rp[1], c0, bp);
  P8_LEG(5); const int s = m.cp[i] != P8_NULL ? t[m.cp[i]] : 0;
  m.sm_cxt[i] = s;
  return cm_cell_inputs(T, o, smt, so, sm_old, s, smt[s], y);
}
// The in-order loop. `rnd` is the global generator: draws happen in context order.
P8_COLD P8_HD inline int cm_mix(Cm& m, Out& o, Rnd& rnd, int y, int c0, int bp, int c1) {
  const Tables& T = *o.T;
  P8_CENSUS_CM(T, m, y, c0, bp);
  P8_CM_ORDER(T, m, o, rnd, y, c0, bp, c1);
  int result = 0;
  for (int i = 0; i < m.cn; ++i) {
    int ns = cm_next_state(T, m, i, y);
    if (ns >= 204 && cm_draw_hits(rnd_next(rnd), ns)) ns -= 4;
    result += cm_step(m, i, o, ns, y, c0, bp, c1);
  }
  if (bp == 7) m.cn = 0;
  return result;
}

P8_HD inline void cm2_set(Cm2& m, u64 ctx) {
  ctx = hash(ctx, (u64)m.index);
  m.cxt[m.index] = finalize64(ctx, m.hashbits);
  m.chk[m.index] = (u16)(checksum64(ctx, m.hashbits, 16) & 0xffff);
  m.index++;
}
// context lists shared by a warp: lane `lane` of `lanes` computes the contexts k with k % lanes == lane (lanes == 1: all of them)
struct CtxSel { int lane, lanes; };
P8_HD inline bool ctx_mine(const CtxSel& s, int k) { return s.lanes == 1 || (k % s.lanes) == s.lane; }
P8_HD inline void cm2_put(Cm2& m, int k, u64 ctx) {
  ctx = hash(ctx, (u64)k);
  m.cxt[k] = finalize64(ctx, m.hashbits);
  m.chk[k] = (u16)(checksum64(ctx, m.hashbits, 16) & 0xffff);
}
P8_HD inline void cm_put(Cm& m, int k, u64 cx) {
  cx = hash(cx, (u64)k);
  m.cxt[k] = finalize64(cx, m.hashbits);
  m.chk[k] = (u16)(checksum64(cx, m.hashbits, 16) & 0xffff);
}
#define P8_CM_SET(sel, m, k, expr) do { if (ctx_mine(sel, k)) cm_put(m, k, (expr)); ++k; } while (0)
#define P8_CM2_SET(sel, m, k, expr) do { if (ctx_mine(sel, k)) cm2_put(m, k, (expr)); ++k; } while (0)
// ---- ContextMap2::mix (:1294-1358) including Update (:1204-1260), cut into prologue / per-context step / epilogue
P8_HD inline void cm2_begin(Cm2& m, int y, int bpos) {
  m.last_bit = (u8)y;
  m.bit_pos = (u8)bpos;
  m.bits += m.bits + (u32)y;
  m.last_byte = (u8)(m.bits & 0xFF);
  if (bpos == 0) m.bits = 1;
}
P8_HD inline int cm2_touched(const Cm2& m, int i, int bp, u32* ids) { return touched_buckets(m.t, m.mask, m.bs[i], m.bh[i], m.cxt[i], m.chk[i], m.bits, bp, ids); }
P8_HD inline int cm2_step(Cm2& m, int i, Out& o, int y, int bpos) {
  const Tables& T = *o.T;
  u8* t = m.t;
  // the three StateMap cells trained this bit: their addresses are known from the previous bit, so the loads go first
  u32* c8 = m.m8_t + i * 256; u32* c12 = m.m12_t + i * 4608; u32* c6 = m.m6_t + i * 72;
  const int o8 = m.m8_cxt[i], o12 = m.m12_cxt[i], o6 = m.m6_cxt[i];
  const u32 old8 = c8[o8], old12 = c12[o12], old6 = c6[o6];
  if (m.bs[i] != P8_NULL) t[m.bs[i]] = T.state[t[m.bs[i]]][y];
  if (bpos > 1 && t[m.bh[i]] == 0) m.bs[i] = P8_NULL;
  else {
    switch (bpos) {
      case 0: {
        m.bs[i] = m.bs0[i] = bucket_find(t, (m.cxt[i] + m.bits) & m.mask, m.chk[i]);
        if (t[m.bs0[i] + 3] == 2) deferred_histories(t, m.mask, m.cxt[i], m.chk[i], m.bs0[i]);
        u8* h = t + m.bh[i];
        h[3] = h[2];
        h[2] = h[1];
        if (h[0] == 0) { h[0] = 2; h[1] = m.last_byte; }
        else if (h[1] != m.last_byte) { h[0] = 1; h[1] = m.last_byte; }
        else if (h[0] < 254) h[0] += 2;
        else if (h[0] == 255) h[0] = 128;
        m.bh[i] = m.bs0[i] + 3;
        m.has_history[i] = t[m.bs0[i]] > 15;
        break;
      }
      case 2: case 5: m.bs[i] = m.bs0[i] = bucket_find(t, (m.cxt[i] + m.bits) & m.mask, m.chk[i]); break;
      case 1: case 3: case 6: m.bs[i] = m.bs0[i] + 1 + y; break;
      case 4: case 7: m.bs[i] = m.bs0[i] + 3 + (int)(m.bits & 3); break;
    }
  }
  if ((bpos == 1 || bpos == 4) && m.bs[i] != P8_NULL) bucket_prefetch2(t, m.mask, m.cxt[i], m.bits * 2);
  int state = m.bs[i] != P8_NULL ? t[m.bs[i]] : 0;
  const int result = state > 0;
  const u8* h = t + m.bh[i];
  const u8 h0 = h[0], h1 = h[1], h2 = h[2], h3 = h[3];
  int n0 = T.state[state][2], n1 = T.state[state][3], k = -~n1;
  k = (k * 64) / (k - ~n0);
  n0 = -!n0; n1 = -!n1;
  int hist;
  if (m.has_history[i]) {
    hist = (h1 >> (7 - bpos)) & 1;
    hist |= ((h2 >> (7 - bpos)) & 1) * 2;
    hist |= ((h3 >> (7 - bpos)) & 1) * 4;
  } else hist = 8;
  // the cells predicted from: loaded before the trained cells are stored, forwarded when a map stays on its cell
  const int x8 = state, x12 = (hist << 9) | (bpos << 6) | k, x6 = (hist << 3) | bpos;
  u32 f8 = c8[x8], f12 = c12[x12], f6 = c6[x6];
  const u32 u8v = sm32_updated(T, old8, y, 1023), u12v = sm32_updated(T, old12, y, 1023), u6v = sm32_updated(T, old6, y, 1023);
  if (x8 == o8) f8 = u8v;
  if (x12 == o12) f12 = u12v;
  if (x6 == o6) f6 = u6v;
  c8[o8] = u8v; c12[o12] = u12v; c6[o6] = u6v;
  m.m8_cxt[i] = x8; m.m12_cxt[i] = x12; m.m6_cxt[i] = x6;
  int p1 = (int)(f8 >> 20);
  if ((u32)((h1 + 256) >> (8 - bpos)) == m.bits) {
    const int rs = h0;
    const int sign = ((h1 >> (7 - bpos)) & 1) * 2 - 1;
    add(o, sign * (ilog(T, rs + 1) << (3 - (rs & 1))));
  } else if (bpos > 0 && (h0 & 1) > 0) {
    if ((u32)((h2 + 256) >> (8 - bpos)) == m.bits) add(o, (((h2 >> (7 - bpos)) & 1) * 2 - 1) * 128);
    else if (m.has_history[i] && (u32)((h3 + 256) >> (8 - bpos)) == m.bits) add(o, (((h3 >> (7 - bpos)) & 1) * 2 - 1) * 128);
    else add(o, 0);
  } else add(o, 0);
  const int st = stretch(T, p1) >> 2;
  add(o, st);
  add(o, (p1 - 2047) >> 3);
  p1 >>= 4;
  const int p0 = 255 - p1;
  add(o, st * iabs(n1 - n0));
  add(o, (p1 & n0) - (p0 & n1));
  add(o, stretch(T, (int)(f12 >> 20)) >> 2);
  add(o, stretch(T, (int)(f6 >> 20)) >> 2);
  return result;
}
// In-order evaluation. The reference updates ALL contexts before predicting from any (two loops); the per-context fusion
// below is the same computation whenever the contexts touch disjoint buckets this bit, and the two-loop order otherwise.
P8_COLD P8_HD inline int cm2_mix_body(Cm2& m, Out& o, int y, int bpos) {   // after cm2_begin(), before the byte-end reset of `index`
  P8_CM2_ORDER(m, o, y, bpos);
  const Tables& T = *o.T;
  u8* t = m.t;
  // loop 1 (Update): cells and pointers only
  for (int i = 0; i < m.index; ++i) {
    if (m.bs[i] != P8_NULL) t[m.bs[i]] = T.state[t[m.bs[i]]][y];
    if (bpos > 1 && t[m.bh[i]] == 0) m.bs[i] = P8_NULL;
    else {
      switch (bpos) {
        case 0: {
          m.bs[i] = m.bs0[i] = bucket_find(t, (m.cxt[i] + m.bits) & m.mask, m.chk[i]);
          if (t[m.bs0[i] + 3] == 2) deferred_histories(t, m.mask, m.cxt[i], m.chk[i], m.bs0[i]);
          u8* h = t + m.bh[i];
          h[3] = h[2];
          h[2] = h[1];
          if (h[0] == 0) { h[0] = 2; h[1] = m.last_byte; }
          else if (h[1] != m.last_byte) { h[0] = 1; h[1] = m.last_byte; }
          else if (h[0] < 254) h[0] += 2;
          else if (h[0] == 255) h[0] = 128;
          m.bh[i] = m.bs0[i] + 3;
          m.has_history[i] = t[m.bs0[i]] > 15;
          break;
        }
        case 2: case 5: m.bs[i] = m.bs0[i] = bucket_find(t, (m.cxt[i] + m.bits) & m.mask, m.chk[i]); break;
        case 1: case 3: case 6: m.bs[i] = m.bs0[i] + 1 + y; break;
        case 4: case 7: m.bs[i] = m.bs0[i] + 3 + (int)(m.bits & 3); break;
      }
    }
  }
  // loop 2: predictions
  int result = 0;
  for (int i = 0; i < m.index; ++i) {
    int state = m.bs[i] != P8_NULL ? t[m.bs[i]] : 0;
    result += state > 0;
    Sm32 q; q.n = 0;
    q.t = m.m8_t + i * 256; q.cxt = m.m8_cxt[i];
    int p1 = sm32_p(T, q, y, state);
    m.m8_cxt[i] = q.cxt;
    int n0 = T.state[state][2], n1 = T.state[state][3], k = -~n1;
    k = (k * 64) / (k - ~n0);
    n0 = -!n0; n1 = -!n1;
    const u8* h = t + m.bh[i];
    if ((u32)((h[1] + 256) >> (8 - bpos)) == m.bits) {
      const int rs = h[0];
      const int sign = ((h[1] >> (7 - bpos)) & 1) * 2 - 1;
      add(o, sign * (ilog(T, rs + 1) << (3 - (rs & 1))));
    } else if (bpos > 0 && (h[0] & 1) > 0) {
      if ((u32)((h[2] + 256) >> (8 - bpos)) == m.bits) add(o, (((h[2] >> (7 - bpos)) & 1) * 2 - 1) * 128);
      else if (m.has_history[i] && (u32)((h[3] + 256) >> (8 - bpos)) == m.bits) add(o, (((h[3] >> (7 - bpos)) & 1) * 2 - 1) * 128);
      else add(o, 0);
    } else add(o, 0);
    if (m.has_history[i]) {
      state = (h[1] >> (7 - bpos)) & 1;
      state |= ((h[2] >> (7 - bpos)) & 1) * 2;
      state |= ((h[3] >> (7 - bpos)) & 1) * 4;
    } else state = 8;
    const int st = stretch(T, p1) >> 2;
    add(o, st);
    add(o, (p1 - 2047) >> 3);
    p1 >>= 4;
    const int p0 = 255 - p1;
    add(o, st * iabs(n1 - n0));
    add(o, (p1 & n0) - (p0 & n1));
    q.t = m.m12_t + i * 4608; q.cxt = m.m12_cxt[i];
    add(o, stretch(T, sm32_p(T, q, y, (state << 9) | (bpos << 6) | k)) >> 2);
    m.m12_cxt[i] = q.cxt;
    q.t = m.m6_t + i * 72; q.cxt = m.m6_cxt[i];
    add(o, stretch(T, sm32_p(T, q, y, (state << 3) | bpos)) >> 2);
    m.m6_cxt[i] = q.cxt;
  }
  return result;
}
P8_HD inline int cm2_mix(Cm2& m, Out& o, int y, int bpos) {
  cm2_begin(m, y, bpos);
  P8_CENSUS_CM2(m, bpos);
  const int result = cm2_mix_body(m, o, y, bpos);
  if (bpos == 7) m.index = 0;
  return result;
}

// BH<4>::operator[] (:788-813): 8-way probe, move-to-front within the probe window
P8_HD inline int bh4_find(u8* t, u32 mask, int hashbits, u64 ctx) {
  const u16 chk = (u16)(checksum64(ctx, hashbits, 16) & 0xffff);
  const u32 i = (finalize64(ctx, hashbits) * 8) & mask;
  u8 tmp[4];
  int j;
  u32 p = 0;
  for (j = 0; j < 8; ++j) {
    p = (i + j) * 4;
    u16* c16 = reinterpret_cast<u16*>(t + p);
    if (t[p + 2] == 0) { *c16 = chk; break; }
    if (*c16 == chk) break;
  }
  if (j == 0) return (int)p + 1;
  if (j == 8) {
    --j;
    tmp[0] = (u8)(chk & 255); tmp[1] = (u8)(chk >> 8); tmp[2] = tmp[3] = 0;
    if (t[(i + j) * 4 + 2] > t[(i + j - 1) * 4 + 2]) --j;
  } else for (int k = 0; k < 4; ++k) tmp[k] = t[p + k];
  for (int k = j * 4 - 1; k >= 0; --k) t[(i + 1) * 4 + k] = t[i * 4 + k];
  for (int k = 0; k < 4; ++k) t[i * 4 + k] = tmp[k];
  return (int)(i * 4) + 1;
}
P8_HD inline void rcm_set(Rcm& r, u64 cx, int c1) {
  u8* cp = r.t + r.cp;
  if (cp[0] == 0 || cp[1] != c1) { cp[0] = 1; cp[1] = (u8)c1; }
  else if (cp[0] < 255) ++cp[0];
  r.cp = bh4_find(r.t, r.mask, r.hashbits, cx) + 1;
}
P8_HD inline void rcm_mix(const Rcm& r, Out& o, int c0, int bpos) {
  const Tables& T = *o.T;
  const u8* cp = r.t + r.cp;
  if (((cp[1] + 256) >> (8 - bpos)) == c0) add(o, (((cp[1] >> (7 - bpos)) & 1) * 2 - 1) * ilog(T, cp[0] + 1) * 8);
  else add(o, 0);
}

// DMC (:7653-7775)
P8_HD inline u8 dmc_state(const DmcNode& n) { return (u8)(((n.nx0 & 0xf) << 4) | (n.nx1 & 0xf)); }
P8_HD inline void dmc_set_state(DmcNode& n, u8 s) { n.nx0 = (n.nx0 & 0xfffffff0u) | (s >> 4); n.nx1 = (n.nx1 & 0xfffffff0u) | (s & 0xf); }
P8_HD inline u32 dmc_inc(u32 x, u32 inc) { return (((x << 6) - x) >> 6) + (inc << 10); }
P8_HD inline int dmc_st(const Tables& T, Dmc& d, int y) {
  DmcNode* t = d.t;
  {
    DmcNode& cur = t[d.curr];
    u32 c0 = cur.c0, c1 = cur.c1;
    const u32 n = y == 0 ? c0 : c1;
    cur.c0 = (u16)dmc_inc(c0, 1 - y);
    cur.c1 = (u16)dmc_inc(c1, y);
    dmc_set_state(cur, T.state[dmc_state(cur)][y]);
    if (n > d.threshold) {
      const u32 next = y == 0 ? cur.nx0 >> 4 : cur.nx1 >> 4;
      c0 = t[next].c0; c1 = t[next].c1;
      const u32 nn = c0 + c1;
      if (nn > n + d.threshold) {
        if (d.top != d.size) {
          const u32 c0_top = (u32)((u64)c0 * (u64)n / (u64)nn), c1_top = (u32)((u64)c1 * (u64)n / (u64)nn);
          c0 -= c0_top; c1 -= c1_top;
          DmcNode& nw = t[d.top];
          nw.c0 = (u16)c0_top; nw.c1 = (u16)c1_top;
          t[next].c0 = (u16)c0; t[next].c1 = (u16)c1;
          nw.nx0 = (nw.nx0 & 0xf) | (t[next].nx0 & 0xfffffff0u);
          nw.nx1 = (nw.nx1 & 0xf) | (t[next].nx1 & 0xfffffff0u);
          dmc_set_state(nw, dmc_state(t[next]));
          if (y == 0) cur.nx0 = (cur.nx0 & 0xf) | (d.top << 4); else cur.nx1 = (cur.nx1 & 0xf) | (d.top << 4);
          ++d.top;
          if (d.threshold < 8 * 1024) d.threshold = (++d.threshold_fine) >> 11;
        } else d.extra += nn >> 10;
      }
    }
    d.curr = y == 0 ? cur.nx0 >> 4 : cur.nx1 >> 4;
  }
  const DmcNode& c = t[d.curr];
#if defined(__CUDA_ARCH__)
  // the node the next bit moves to is one of the two children: have both lines on their way
  asm volatile("prefetch.global.L2 [%0];" ::"l"(t + (c.nx0 >> 4)));
  asm volatile("prefetch.global.L2 [%0];" ::"l"(t + (c.nx1 >> 4)));
#endif
  const u32 n0 = c.c0 + 1u, n1 = c.c1 + 1u;
  const int pr1 = (int)((n1 << 12) / (n0 + n1));
  const int pr2 = sm32_p(T, d.sm, y, dmc_state(c), 256);
  return stretch(T, pr1) + stretch(T, pr2);
}

// int16 mixer arithmetic (:407-432, SSE2 semantics)
P8_HD inline int sat16(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }
P8_HD inline int dot_pair(const short* t, const short* w) { return ((int)t[0] * w[0] + (int)t[1] * w[1]) >> 8; }
P8_HD inline short train_one(short t, short w, int err) {
  int v = sat16(2 * (int)t);
  v = (v * (int)(short)err) >> 16;
  v = sat16(v + 1) >> 1;
  return (short)sat16(v + (int)w);
}

}  // namespace p8
}  // namespace cmixb200
#endif
