// cmix_b200/csrc/fxcm_model.h — the resident FXCM model (SURVEY §8 row a14) as integer-only host/device code.
//
// What it reproduces: reference src/models/fxcmv1.cpp — `update1` (:4758-4834), `modelPrediction` (:3798-4755), the
// three bucketed context-map flavours (:971-1612), the SSE2 int16 mixers (:472-660), StateMaps (:672-737), APMs
// (:1622-1646), the two match models (:1742-1841, :3420-3700), the run map (:756-829) and the 429 exported 12-bit
// codes (:97-105, SURVEY Appendix B #19). Bit-exact by construction: every quantity is an integer.
//
// How it is organised for the GPU (fxcm.cuh runs it; tools/fxcm_check.cpp runs the same code on the CPU):
//  * ONE flat state block per stream (FxState) of offsets into HBM arenas; no pointers into tables are kept —
//    bit-history cells are addressed by 32-bit byte offsets into their bucket table.
//  * The per-bit work is cut into UNITS that own disjoint state and disjoint slices of the input / export vectors
//    (7 stationary maps, 2 match models, 31 context maps, 1 run map = 41 units). Units are independent of each
//    other, so a CTA runs them one lane per unit; inside a context map the contexts are walked in order because
//    two contexts of one map may share a bucket and the replacement policy is order dependent.
//  * The 10+2 int16 mixers: dot products and SGD are exact under any association (int32 wrap-around sums of
//    per-pair `>>8` terms, saturating per-weight updates), so they are spread over all lanes of the CTA.
//  * The byte-level text analysis (fxcm_text.h) runs once per byte on one lane.
// Phases of one bit (fx_bit_* below), in the reference's order: head (bit bookkeeping + mixer error terms) ->
// train (all lanes) -> [byte boundary: text analysis sets ~80 contexts] -> units (one lane each) -> select
// (mixer weight-set selection) -> dot (all lanes) -> tail (final mixers, 6 APMs, export).
#ifndef CMIXB200_FXCM_MODEL_H
#define CMIXB200_FXCM_MODEL_H

#include <stddef.h>

#include "fxcm_text.h"

// Host census of the device-only clash path (tools/census.h): called where the in-order map loop starts, with the state the
// device's per-bit probe sees. Empty in every product build.
#ifndef FX_CENSUS_MAP
#define FX_CENSUS_MAP(S, id) do { } while (0)
#endif
// Host test of the clash rule (tools/census.h with -DCENSUS_PERMUTE): may evaluate map_bit's contexts in another order and
// return. Empty in every product build.
#ifndef FX_MAP_ORDER
#define FX_MAP_ORDER(S, id, o) do { } while (0)
#endif

namespace cmixb200 {
namespace fx {

enum { N_MAPS = 31, N_UNITS = 41, N_IN1 = 512, N_IN2 = 16, N_OUT = 431, N_MIX = 12,
       BUF_MASK = 0xffffff, CW_MASK = 0xfff, IND3_SIZE = 0x2000000, MATCH_HASH = 0x200000, MAX_LEN = 62 };
#define FX_NULL 0xFFFFFFFFu
enum { U_SCM0 = 0, U_MATCH = 7, U_SMATCH = 8, U_MAP0 = 9, U_RCM = 40 };

// map ids in mix order (fxcmv1.cpp:4596-4630); the reference's cmC2[k] / cmC1[k] / cmC[k] by name
enum { M2_0 = 0, M2_1, M2_2, M2_3, M2_4, M2_5, M2_6, M2_7, M2_8, M1_0, M1_1, M1_2, M1_4, M0_0, M0_1, M0_2, M1_3, M2_9, M2_10,
       M2_11, M2_12, M2_13, M0_3, M2_14, M2_15, M0_4, M0_5, M2_16, M2_17, M1_6, M1_7 };

struct MapSpec { u32 mem; u8 kind, C, par, sta, kep, skip2, st2; };   // kind: 0 = 7-slot/64 B, 1 = 3-slot/32 B, 2 = 14-slot/128 B
#define FX_M(mem, kind, C, par, sta, kep, skip2, st2) {(u32)(mem), kind, C, par, sta, kep, skip2, st2}
// fxcmv1.cpp:3346-3397 in mix order. sta: 0..5 = STA1, STA2, STA4, STA5, STA6, STA7.
static const MapSpec kMapSpec[N_MAPS] = {
    FX_M(8u << 24, 2, 3, 0, 4, 0xf0, 1, 1), FX_M(16u << 24, 2, 1, 1, 4, 0xf0, 1, 1), FX_M(8u << 24, 2, 1, 2, 4, 0xf0, 1, 1),
    FX_M(8u << 24, 2, 1, 3, 4, 0xf0, 1, 1), FX_M(8u << 24, 2, 2, 4, 4, 0xf0, 1, 1), FX_M(8u << 24, 2, 6, 5, 4, 0xf0, 1, 1),
    FX_M((1u << 24) / 64, 2, 1, 6, 0, 0, 1, 1), FX_M(2u << 24, 2, 1, 7, 3, 0xf0, 1, 1), FX_M((8u << 24) / 2, 2, 4, 8, 2, 0, 1, 1),
    FX_M(32 * 4096, 1, 2, 9, 4, 0, 0, 0), FX_M(2 * 32 * 4096, 1, 3, 10, 5, 0, 1, 1), FX_M(32 * 4096, 1, 4, 11, 1, 0, 1, 1),
    FX_M(16 * 4096, 1, 5, 12, 5, 0, 1, 1),
    FX_M(16 * 4096, 0, 7, 13, 1, 0, 1, 1), FX_M(64 * 2 * 4096, 0, 3, 14, 3, 0xf0, 0, 0), FX_M(2 * 4096, 0, 2, 15, 1, 0xf0, 0, 0),
    FX_M(128 * 4096, 1, 2, 16, 0, 0, 0, 0),
    FX_M(8u << 24, 2, 4, 17, 4, 0xf0, 1, 1), FX_M(8u << 24, 2, 6, 18, 3, 0xf0, 1, 1), FX_M(8u << 24, 2, 5, 19, 3, 0xf0, 1, 1),
    FX_M(8u << 24, 2, 2, 20, 4, 0xf0, 1, 1), FX_M(16u << 24, 2, 2, 21, 4, 0xf0, 1, 1),
    FX_M(32 * 4096, 0, 2, 22, 1, 0, 1, 2),
    FX_M((4u << 24) / 2, 2, 1, 23, 4, 0xf0, 1, 1), FX_M(8 * 64 * 4096, 2, 1, 24, 0, 0, 0, 0),
    FX_M(512 * 4096, 0, 1, 25, 0, 0xf0, 1, 1), FX_M(512 * 4096, 0, 1, 26, 0, 0xf0, 1, 1),
    FX_M((1u << 24) / 2, 2, 1, 17, 4, 0xf0, 1, 1), FX_M(2u << 24, 2, 2, 17, 4, 0xf0, 1, 1),
    FX_M(16 * 4096, 1, 1, 5, 4, 0, 0, 1), FX_M(16 * 4096, 1, 4, 12, 1, 0, 1, 1)};
#undef FX_M
// mixer set sizes, output shifts, error dead zones and error gains (fxcmv1.cpp:3314-3325)
static const int kMixM[N_MIX] = {2048, 6 * 256, 6 * 256 * 4, 8 * 256, 6 * 256, 7 * 256 * 4, 0x4000, 0x4000, 0x20000, 0x20000, 8 * 7 * 2 * 2, 1};
static const int kMixShift[N_MIX] = {237, 204, 70, 54, 55, 55, 70, 55, 55, 55, 6, 6};
static const int kMixElim[N_MIX] = {8, 8, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0};
static const int kMixUperr[N_MIX] = {69, 19, 34, 23, 24, 24, 34, 24, 24, 24, 4, 4};

// ---------------------------------------------------------------- read-only tables (host-built, fxcm_host.h)
struct MapTab { short rc1[512]; short st1[4096]; short st8[256]; short st32[256]; };
struct Tables {
  short sqt[4096];       // squash, index d + 2047 (fxcmv1.cpp:137-155)
  short strt[4096];      // stretch (:157-175)
  u8 ilog[256];
  int dt[1024];
  u8 sta[6][1024];       // six generated bit-history state tables (:241-357), [state*4 + {next0, next1, n0, n1}]
  short rcm_rc[512];
  MapSpec spec[N_MAPS];
  int mix_m[N_MIX], mix_shift[N_MIX], mix_uperr[N_MIX];
  u8 wrt2[256], wrt3[256], wrt4[256];   // byte classes (fxcmv1.cpp:51-90, :1843-1862)
  u8 fcy[128], fcq[128];                // bracket / first-char class indices (:3702-3731)
  u32 primes[14];
  int e_l[8];
  const char* dict_chars; const u32* dict_off;   // WRT dictionary words, NUL terminated (:398-410)
  int dict_n, dict_loaded;
  // the big per-map tables stay out of line: everything above map_store can be staged in shared memory (TABLES_HOT_BYTES)
  const MapTab* map;                    // -> map_store
  const short (*st2)[4096];             // -> st2_store
  alignas(16) MapTab map_store[N_MAPS];
  short st2_store[3][4096];
};
enum { TABLES_HOT_BYTES = offsetof(Tables, map_store) };
static_assert(TABLES_HOT_BYTES % 16 == 0, "the hot part of the tables is copied in 16-byte words");

// ---------------------------------------------------------------- mutable state of one stream
struct MapState {
  u8* t;                 // bucket table
  u32* sm;               // [C][256] state -> probability (22 bits) | unused low bits
  u32 tmask;
  u32 cxt[8], cp[8], cp0[8], runp[8], sm_cxt[8];
  u32 result;
  u16 mask;              // cxtMask
  u8 cn, pad;
};
struct ScmState { u16* data; int context, mask, stride, bcount, btotal, B, cp; };
struct Sm1State { u32* t; int cxt, mask; };
struct MixState { short* w; int cxt, pr, elim, err; };
struct ApmState { u16* t; int index; };
struct MatchCand { u32 length, index, length_bak, index_bak; u8 expected, delta, pad[2]; };

struct TextState {
  // byte history and hashes
  int c1, c2, c3, pos;
  u32 t[14];
  u8 words, spaces, numbers, pad0;
  u32 word0, word00, word1, word2, word3, wshift, x4, x5, first_word, linkword, senword;
  u32 number0, number1, numlen0, numlen1, mybenum;
  u32 fc_idx, brfc_idx, ah1, ah2;
  int nl, nl1, col, fc;
  u32 ind_br_byte, ind_byte, ind_word0_pos, ind_word, u8w, ctx1_ind3, cxt_ind3, last_wt;
  u32 o3b, n3b, s3bR, s3b, s3b_mask, s3b_mask1, s3bR_mask1, s3bR_mask2;
  u32 o2b, n2b, s2bR, s2b, s2b_mask;
  u32 n4b, s4b;
  int cwpos, stem_index, cword, pword, dcw, dcwl, deccode, utf8left, last_cw;
  u32 s_verb;
  int last_art, is_nowiki, is_text, is_math, is_pre, is_paragraph;
  int so, colonstr;      // dictionary word index, -1 = empty string
  u32 t1[256];
  Word stem_words[4];
  Nest<8> br, qo, fcx;
  Nest<16> ht;
  Columns cols;
  WordList sent, para, strm;
  u8 cwbuf[CW_MASK + 1];
};

struct State {
  // bit bookkeeping (BlockData, fxcmv1.cpp:190-205)
  int y, c0, bpos, blpos, bposshift, c0shift_bpos;
  u32 c4;
  int pr;                // final 12-bit prediction
  u32 fails, failz, failcount;
  int sscmrate, rate;
  int ord_x, ord_w, is_match;
  int lstmpr, lstmex;
  // vectors
  alignas(16) short in1[N_IN1 + 48];
  short in2[N_IN2];
  u16 codes[N_OUT + 1];  // exported 12-bit codes, 0xFFFF = slot still holds 0.5
  int in_off[N_UNITS + 1], ex_off[N_UNITS + 1];
  // components
  MapState map[N_MAPS];
  ScmState scm[7];
  Sm1State sma[3];
  MixState mix[N_MIX];
  ApmState apm[6];
  // run map
  u8* rcm_t; u32 rcm_n; u32 rcm_cp;
  // match model 2
  MatchCand cand[4]; u32 n_cand; u32* mhash;   // [MATCH_HASH + 32][4]
  // sparse match model
  u32* sm_table; int sm_root, sm_index_it; int sm_prev[4], sm_next[4];
  u32 sm_hashes[4], sm_hash_index, sm_length, sm_index; u8 sm_expected, sm_valid;
  // big byte-level arrays
  u8* buffer; u16* ind3; u32* t2; int* wp;
  TextState* text;
  const Tables* T;
};

// ---------------------------------------------------------------- primitives
FX_HD inline int squash(const Tables& T, int d) { if (d < -2047) return 1; if (d > 2047) return 4095; return T.sqt[d + 2047]; }
FX_HD inline int stretch(const Tables& T, int p) { return T.strt[p]; }
FX_HD inline int clp(int z) { return z < -2047 ? -2047 : (z > 2047 ? 2047 : z); }
FX_HD inline int buf(const State& S, int i) { return S.buffer[(S.text->pos - i) & BUF_MASK]; }
FX_HD inline int bufr(const State& S, u32 i) { return S.buffer[i & BUF_MASK]; }

struct Out { short* n; u16* codes; int ni, ei; };
FX_HD inline void emit(const Tables& T, Out& o, int v, bool exported = true) {
  o.n[o.ni++] = (short)v;
  if (exported) o.codes[o.ei++] = (u16)squash(T, v);
}

// ---------------------------------------------------------------- bucketed context maps (fxcmv1.cpp:971-1612)
FX_HD inline int map_slots(int kind) { return kind == 0 ? 7 : (kind == 1 ? 3 : 14); }
FX_HD inline int map_shift(int kind) { return kind == 0 ? 6 : (kind == 1 ? 5 : 7); }

// E<A,B>::get: checksum probe with a 2-entry recency queue, lowest-priority replacement (fxcmv1.cpp:930-946).
// Returns the byte offset (in the table) of bh[slot][0].
FX_HD inline u32 bucket_get(u8* t, u32 base, int A, u16 ch, int keep) {
  u8* e = t + base;
  u16* chk = reinterpret_cast<u16*>(e);
  u8& last = e[2 * A];
  const u32 bh = base + 2 * A + 1;
  if (chk[last & 15] == ch) return bh + 7 * (last & 15);
  int b = 0xffff, bi = 0;
  for (int i = 0; i < A; ++i) {
    if (chk[i] == ch) { last = (u8)(last << 4 | i); return bh + 7 * i; }
    const int pri = t[bh + 7 * i];
    if (pri < b && (last & 15) != i && (last >> 4) != i) { b = pri; bi = i; }
  }
  last = (u8)(last << 4 | bi | keep);
  chk[bi] = ch;
  for (int k = 0; k < 7; ++k) t[bh + 7 * bi + k] = 0;
  return bh + 7 * bi;
}

FX_HD inline u32 state_byte_location(int bpos, int c0) {   // fxcmv1.cpp:950-955
  const u32 smask = (0x31031010u >> (bpos << 2)) & 0x0F;
  return smask + (c0 & smask);
}

FX_HD inline void map_set(MapState& m, u32 cx) {   // ContextMap::set (fxcmv1.cpp:1045-1052)
  const u32 i = m.cn++;
  cx = cx * 987654323u + i;
  cx = cx << 16 | cx >> 16;
  m.cxt[i] = cx * 123456791u + i;
  m.mask = (u16)(m.mask * 2);
}
FX_HD inline void map_skip(MapState& m) { m.cn++; m.mask = (u16)(m.mask + 1); m.mask = (u16)(m.mask * 2); }

// Read-only probe of E<A,B>::get: which slot of the bucket at `base` holds checksum ch (-1: get would replace one).
FX_HD inline int bucket_peek(const u8* t, u32 base, int A, u16 ch) {
  const u8* e = t + base;
  const u16* chk = reinterpret_cast<const u16*>(e);
  const u8 last = e[2 * A];
  if (chk[last & 15] == ch) return last & 15;
  for (int i = 0; i < A; ++i) if (chk[i] == ch) return i;
  return -1;
}
// The buckets context i of map `id` reads or writes this bit (at most 5): its live cell's, its run-info cell's, the one it moves
// to and, on a byte boundary, the two of a deferred history write-back. A skipped context touches none.
FX_HD inline int map_touched(const State& S, int id, int i, u32* ids) {
  const Tables& T = *S.T;
  const MapState& m = S.map[id];
  const MapSpec sp = T.spec[id];
  const int A = map_slots(sp.kind), sh = map_shift(sp.kind);
  const int bp = S.bpos;
  if ((m.mask >> (m.cn - i)) & 1) return 0;
  int n = 0;
  if (m.cp[i] != FX_NULL) ids[n++] = m.cp[i] >> sh;
  ids[n++] = m.runp[i] >> sh;
  if (bp > 1 && m.t[m.runp[i]] == 0) return n;
  if (bp == 0 || bp == 2 || bp == 5) {
    const u32 b = (m.cxt[i] + (u32)S.c0) & m.tmask;
    ids[n++] = b;
    if (bp == 0) {
      const u16 chk = (u16)((m.cxt[i] >> 16) ^ i);
      const int slot = bucket_peek(m.t, b << sh, A, chk);
      if (slot >= 0) {
        const u8* cell0 = m.t + (b << sh) + 2 * A + 1 + 7 * slot;
        if (cell0[3] == 2) { const int c = cell0[4] + 256; ids[n++] = (m.cxt[i] + (u32)(c >> 6)) & m.tmask; ids[n++] = (m.cxt[i] + (u32)(c >> 3)) & m.tmask; }
      }
    }
  }
  return n;
}
// One bit of one context of one map: train the cell with y, move to the next cell, emit the inputs (mix / mix1) at the
// context's own slice of the unit's inputs / exports. Returns 1 when the context has a non-zero state.
FX_HD inline u32 map_ctx_bit(State& S, int id, int i, const Out& unit) {
  const Tables& T = *S.T;
  MapState& m = S.map[id];
  const MapSpec sp = T.spec[id];
  const MapTab& tab = T.map[id];
  const u8* nn = T.sta[sp.sta];
  const short* st2 = T.st2[sp.st2];
  const int A = map_slots(sp.kind), sh = map_shift(sp.kind);
  const int y = S.y, bp = S.bpos, cc = S.c0;
  const u8 c1 = (u8)S.c4;
  Out o = unit;
  o.ni += i * (5 + sp.skip2); o.ei += i * (4 + sp.skip2);
  if ((m.mask >> (m.cn - i)) & 1) {   // skipped context: constant inputs
    emit(T, o, 0); if (sp.skip2) emit(T, o, 0); emit(T, o, 0); emit(T, o, 0); emit(T, o, 64, false); emit(T, o, 0);
    return 0;
  }
  u32 result = 0;
  if (m.cp[i] != FX_NULL) m.t[m.cp[i]] = nn[m.t[m.cp[i]] * 4 + y];
  int s = 0;
  if (bp > 1 && m.t[m.runp[i]] == 0) m.cp[i] = FX_NULL;
  else {
    const u16 chk = (u16)((m.cxt[i] >> 16) ^ i);
    if (bp) {
      if (bp == 2 || bp == 5) m.cp0[i] = m.cp[i] = bucket_get(m.t, ((m.cxt[i] + cc) & m.tmask) << sh, A, chk, sp.kep);
      else m.cp[i] = m.cp0[i] + state_byte_location(bp, cc);
    } else {
      m.cp0[i] = m.cp[i] = bucket_get(m.t, ((m.cxt[i] + cc) & m.tmask) << sh, A, chk, sp.kep);
      if (m.t[m.cp0[i] + 3] == 2) {   // deferred bit histories of bits 2-7 for a context seen the second time
        const int c = m.t[m.cp0[i] + 4] + 256;
        u32 p = bucket_get(m.t, ((m.cxt[i] + (c >> 6)) & m.tmask) << sh, A, chk, sp.kep);
        m.t[p] = (u8)(1 + ((c >> 5) & 1));
        m.t[p + 1 + ((c >> 5) & 1)] = (u8)(1 + ((c >> 4) & 1));
        m.t[p + 3 + ((c >> 4) & 3)] = (u8)(1 + ((c >> 3) & 1));
        p = bucket_get(m.t, ((m.cxt[i] + (c >> 3)) & m.tmask) << sh, A, chk, sp.kep);
        m.t[p] = (u8)(1 + ((c >> 2) & 1));
        m.t[p + 1 + ((c >> 2) & 1)] = (u8)(1 + ((c >> 1) & 1));
        m.t[p + 3 + ((c >> 1) & 3)] = (u8)(1 + (c & 1));
        m.t[m.cp0[i] + 6] = 0;
      }
      u8* rp = m.t + m.runp[i];
      if (rp[0] == 0) { rp[0] = 2; rp[1] = c1; }
      else if (rp[1] != c1) { rp[0] = 1; rp[1] = c1; }
      else if (rp[0] < 254) rp[0] += 2;
      m.runp[i] = m.cp0[i] + 3;
    }
    s = m.t[m.cp[i]];
  }
#if defined(__CUDA_ARCH__)
  if ((bp == 1 || bp == 4) && m.cp[i] != FX_NULL) {   // the bucket of the next bit is one of two neighbours: start both loads now
    asm volatile("prefetch.global.L2 [%0];" ::"l"(m.t + ((size_t)((m.cxt[i] + (u32)cc * 2) & m.tmask) << sh)));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(m.t + ((size_t)((m.cxt[i] + (u32)cc * 2 + 1) & m.tmask) << sh)));
  }
#endif
  if (s == 0) {
    emit(T, o, 0); if (sp.skip2) emit(T, o, 0); emit(T, o, 0); emit(T, o, 0); emit(T, o, 64, false);
  } else {
    u32* sm = m.sm + i * 256;          // StateMap::set (fxcmv1.cpp:686-704)
    u32 p0 = sm[m.sm_cxt[i]];
    p0 += (u32)((y << 19) - (int)(p0 >> 13));
    sm[m.sm_cxt[i]] = p0;
    m.sm_cxt[i] = (u32)s;
    const int p1 = (int)(sm[s] >> 20);
    emit(T, o, tab.st1[p1]); if (sp.skip2) emit(T, o, st2[p1]); emit(T, o, tab.st8[s]); emit(T, o, tab.st32[s]); emit(T, o, 0, false);
    result = 1;
  }
  const u8* rp = m.t + m.runp[i];
  int b = S.c0shift_bpos ^ (rp[1] >> S.bposshift);
  if (b <= 1) emit(T, o, tab.rc1[rp[0] + b * 256]);
  else emit(T, o, 0);
  return result;
}
FX_HD inline void map_finish(State& S, int id, u32 result) {
  MapState& m = S.map[id];
  if (S.bpos == 7) { m.cn = 0; m.mask = 0; }
  m.result = result;
}
// One bit of one context map, contexts in order (mix / mix1).
FX_HD inline void map_bit(State& S, int id, Out& o) {
  FX_CENSUS_MAP(S, id);
  FX_MAP_ORDER(S, id, o);
  u32 result = 0;
  const int cn = S.map[id].cn;
  for (int i = 0; i < cn; ++i) result += map_ctx_bit(S, id, i, o);
  map_finish(S, id, result);
}

// ---------------------------------------------------------------- small units
FX_HD inline void scm_bit(State& S, int k, Out& o) {   // SmallStationaryContextMap::mix (fxcmv1.cpp:856-869)
  const Tables& T = *S.T;
  ScmState& c = S.scm[k];
  const int rate = S.sscmrate + 7;
  u16& cell = c.data[c.cp];
  cell = (u16)(cell + (((S.y << 16) - (int)cell + (1 << (rate - 1))) >> rate));
  c.B += (S.y && c.B > 0);
  c.cp = c.context + c.B;
  const int pred = c.data[c.cp] >> 4;
  emit(T, o, stretch(T, pred) / 4);
  emit(T, o, (pred - 2048) / 8, false);
  c.bcount++; c.B += c.B + 1;
  if (c.bcount == c.btotal) c.bcount = c.B = 0;
}
FX_HD inline void scm_set(ScmState& c, u32 ctx) { c.context = (int)((ctx & (u32)c.mask) * (u32)c.stride); c.bcount = c.B = 0; }

FX_HD inline int sm1_set(const Tables& T, Sm1State& s, int y, u32 c) {   // StateMap1::set (fxcmv1.cpp:722-737), limit 1023
  u32 p0 = s.t[s.cxt];
  const int n = p0 & 1023, pr1 = (int)(p0 >> 12);
  p0 += (n < 1023);
  p0 += (u32)((int)((u32)((y << 20) - pr1) * (u32)T.dt[n]) + 512) & 0xfffffc00u;
  s.t[s.cxt] = p0;
  s.cxt = (int)(c & (u32)s.mask);
  return (int)(s.t[s.cxt] >> 20);
}

// run map (fxcmv1.cpp:756-829)
FX_HD inline u32 rcm_find(State& S, u32 i) {
  u8* t = S.rcm_t;
  const u16 chk = (u16)((i >> 16 ^ i) & 0xffff);
  i = i * 4 & S.rcm_n;
  u8 tmp[4];
  int j;
  u32 p = 0;
  for (j = 0; j < 4; ++j) {
    p = (i + j) * 4;
    u16* c16 = reinterpret_cast<u16*>(t + p);
    if (t[p + 2] == 0) { *c16 = chk; break; }
    if (*c16 == chk) break;
  }
  if (j == 0) return p + 1;
  if (j == 4) {
    --j;
    tmp[0] = (u8)(chk & 255); tmp[1] = (u8)(chk >> 8); tmp[2] = tmp[3] = 0;
    if (t[(i + j) * 4 + 2] > t[(i + j - 1) * 4 + 2]) --j;
  } else for (int k = 0; k < 4; ++k) tmp[k] = t[p + k];
  for (int k = j * 4 - 1; k >= 0; --k) t[(i + 1) * 4 + k] = t[i * 4 + k];
  for (int k = 0; k < 4; ++k) t[i * 4 + k] = tmp[k];
  return i * 4 + 1;
}
FX_HD inline void rcm_set(State& S, u32 cx, u8 c1) {
  u8* cp = S.rcm_t + S.rcm_cp;
  if (cp[0] == 0) { cp[0] = 2; cp[1] = c1; }
  else if (cp[1] != c1) { cp[0] = 1; cp[1] = c1; }
  else if (cp[0] < 254) cp[0] = (u8)(cp[0] + 2);
  S.rcm_cp = rcm_find(S, cx) + 1;
}
FX_HD inline void rcm_bit(State& S, Out& o) {
  const Tables& T = *S.T;
  const u8* cp = S.rcm_t + S.rcm_cp;
  const int b = S.c0shift_bpos ^ (cp[1] >> S.bposshift);
  emit(T, o, b <= 1 ? T.rcm_rc[b * 256 + cp[0]] : 0);
}

// sparse match model (fxcmv1.cpp:1742-1841)
FX_HD inline void smatch_update(State& S) {
  const u32 min_len[4] = {3, 4, 6, 5}, stride[4] = {1, 1, 2, 1};
  const u32 mask = 1024 * 1024 - 1;
  for (u32 i = 0; i < 4; ++i) {
    u32 h = (i + 1) * 191;
    for (u32 j = 0, k = 1; j < min_len[i]; ++j, k += stride[i]) h = h * 191 + ((u32)buf(S, k) << i);
    S.sm_hashes[i] = h & mask;
  }
  if (S.sm_length) { S.sm_index++; if (S.sm_length < 64) S.sm_length++; }
  else {
    for (int i = (S.sm_index_it = S.sm_root); i >= 0; i = (S.sm_index_it >= 0 ? (S.sm_index_it = S.sm_next[S.sm_index_it]) : S.sm_index_it)) {
      S.sm_index = S.sm_table[S.sm_hashes[i]];
      if (S.sm_index > 0) {
        u32 off = 1;
        while (S.sm_length < min_len[i] && ((buf(S, off) ^ bufr(S, S.sm_index - off))) == 0) { S.sm_length++; off += stride[i]; }
        if (S.sm_length >= min_len[i]) {
          S.sm_length -= (min_len[i] - 1);
          S.sm_hash_index = i;
          // MTFList::MoveToFront (fxcmv1.cpp:1707-1719)
          if ((S.sm_index_it = i) != S.sm_root) {
            const int p = S.sm_prev[i], n = S.sm_next[i];
            if (p >= 0) S.sm_next[p] = S.sm_next[i];
            if (n >= 0) S.sm_prev[n] = S.sm_prev[i];
            S.sm_prev[S.sm_root] = i;
            S.sm_next[i] = S.sm_root;
            S.sm_root = i;
            S.sm_prev[S.sm_root] = -1;
          }
          break;
        }
      }
      S.sm_length = S.sm_index = 0;
    }
  }
  for (u32 i = 0; i < 4; ++i) S.sm_table[S.sm_hashes[i]] = (u32)S.text->pos;
  S.sm_expected = (u8)bufr(S, S.sm_index);
  S.sm_valid = S.sm_length > 1;
}
FX_HD inline void smatch_bit(State& S, Out& o) {
  const Tables& T = *S.T;
  const u8 B = (u8)(S.c0 << (8 - S.bpos));
  if (S.bpos == 0) smatch_update(S);
  if (S.sm_length > 0 && (((S.sm_expected ^ B)) >> (8 - S.bpos)) != 0) S.sm_length = 0;
  if (S.sm_valid && S.sm_length > 1) {
    const int bit = (S.sm_expected >> (7 - S.bpos)) & 1, sign = 2 * bit - 1;
    const int len = (int)S.sm_length;
    emit(T, o, sign * (imin(len - 1, 32) << 5));
    emit(T, o, sign * (1 << imin(len - 2, 3)) * imin(len - 1, 8) << 4);
  } else { emit(T, o, 0); emit(T, o, 0); }
}

// match model 2 (fxcmv1.cpp:3420-3700)
FX_HD inline bool cand_nomatch(const MatchCand& c) { return c.length == 0 && !c.delta && c.length_bak == 0; }
FX_HD inline void cand_update(State& S, MatchCand& c) {
  if (c.length != 0) {
    const int bit = (c.expected >> ((8 - S.bpos) & 7)) & 1;
    if (S.y != bit) {
      if (c.length != 0 && c.length_bak != 0) { c.length_bak = 0; c.index_bak = 0; }
      else { c.length_bak = c.length; c.index_bak = c.index; c.delta = 1; }
      c.length = 0;
    }
  }
  if (S.bpos == 0) {
    if (c.length == 0 && !c.delta && c.length_bak != 0) {
      c.index_bak++;
      if (c.length_bak < (u32)MAX_LEN) c.length_bak++;
      if (bufr(S, c.index_bak) == S.text->c1) { c.length = c.length_bak; c.index = c.index_bak; }
      else c.length_bak = c.index_bak = 0;
    }
    if (c.length != 0) {
      c.index++;
      if (c.length < (u32)MAX_LEN) c.length++;
      if (c.length_bak != 0 && c.length - c.length_bak >= 3) c.length_bak = c.index_bak = 0;
    }
    c.delta = 0;
  }
}
FX_HD inline u32 cand_prio(const MatchCand& c) {
  return (u32)(c.length != 0) << 31 | (u32)(c.delta != 0) << 30 | (c.delta ? (c.length_bak >> 1) : (c.length >> 1)) << 24 | (c.index & 0x00ffffff);
}
FX_HD inline void match_add(State& S, u32* slot, u32 LEN) {
  u32 i = 0;
  while (S.n_cand < 4 && i < 4) {
    const u32 mp = slot[i];
    if (mp == 0) break;
    bool ok = true;
    for (int l = 1; l <= (int)LEN; ++l) if (buf(S, l) != bufr(S, mp - l)) { ok = false; break; }
    if (ok) {
      bool same = false;
      for (u32 j = 0; j < S.n_cand; ++j) { same = S.cand[j].index == mp; if (same) break; }
      if (!same) {
        MatchCand& c = S.cand[S.n_cand++];
        c.length = LEN - 5 + 1; c.index = mp; c.length_bak = c.index_bak = 0; c.expected = 0; c.delta = 0;
      }
    }
    ++i;
  }
}
FX_HD inline void match_slot(State& S, u32 hash, u32 LEN) {
  u32* slot = S.mhash + (size_t)(hash & (MATCH_HASH - 1)) * 4;
  if (S.n_cand < 4) match_add(S, slot, LEN);
  slot[3] = slot[2]; slot[2] = slot[1]; slot[1] = slot[0]; slot[0] = (u32)S.text->pos;
}
FX_HD inline void match_bit(State& S, Out& o) {
  const Tables& T = *S.T;
  const u32 n = (u32)imax((int)S.n_cand, 1);
  for (u32 i = 0; i < n; ++i) {
    MatchCand& c = S.cand[i];
    cand_update(S, c);
    if (S.n_cand != 0 && cand_nomatch(c)) {
      S.n_cand--;
      if (S.n_cand == i) break;
      for (u32 k = i; k < S.n_cand; ++k) S.cand[k] = S.cand[k + 1];
      i--;
    }
  }
  if (S.bpos == 0) {
    match_slot(S, S.text->t[9], 9);
    match_slot(S, S.text->t[7], 7);
    match_slot(S, S.text->t[5], 5);
    match_slot(S, S.text->sent.word(1), 5);
    for (u32 i = 0; i < S.n_cand; ++i) S.cand[i].expected = (u8)bufr(S, S.cand[i].index);
  }
  u32 ctx[3] = {0, 0, 0};
  int best = 0;
  for (u32 i = 1; i < S.n_cand; ++i) if (cand_prio(S.cand[i]) > cand_prio(S.cand[best])) best = (int)i;
  const u32 length = S.cand[best].length;
  const u8 eb = S.cand[best].expected;
  const bool delta = S.cand[best].delta != 0;
  const int bit = length != 0 ? (eb >> (7 - S.bpos)) & 1 : 0;
  if (length != 0) {
    const u32 dense = length <= 16 ? length - 1 : 12 + (length >> 2);
    ctx[0] = (dense << 4) | ((u32)bit << 3) | (u32)S.bpos;
    ctx[1] = ((u32)eb << 11) | ((u32)S.bpos << 8) | (u32)S.text->c1;
    emit(T, o, (2 * bit - 1) * (int)(length << 5));
  } else emit(T, o, 0);
  if (delta) ctx[2] = ((u32)eb << 8) | (u32)S.c0;
  for (int i = 0; i < 3; ++i) {
    if (ctx[i] != 0) {
      const int p1 = sm1_set(T, S.sma[i], S.y, ctx[i]);
      emit(T, o, stretch(T, p1) >> 2);
      emit(T, o, (p1 - 2048) >> 3);
    } else { emit(T, o, 0); emit(T, o, 0); }
  }
  S.is_match = (int)length;
}

// ---------------------------------------------------------------- int16 mixers (fxcmv1.cpp:472-660, SSE2 semantics)
FX_HD inline int sat16(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }
FX_HD inline int dot_pair(const short* t, const short* w) { return ((int)t[0] * w[0] + (int)t[1] * w[1]) >> 8; }   // pmaddwd, psrad 8
FX_HD inline short train_one(short t, short w, int err) {
  int v = sat16(2 * (int)t);                 // paddsw t,t
  v = (v * err) >> 16;                       // pmulhw
  v = sat16(v + 1) >> 1;                     // paddsw 1, psraw 1
  return (short)sat16(v + (int)w);           // paddsw w
}
FX_HD inline int apm_p(const Tables& T, ApmState& a, int pr, u32 cxt, int rate, int y) {   // APM::p (fxcmv1.cpp:1628-1637)
  pr = stretch(T, pr);
  const int g = (y << 16) + (y << rate) - y * 2;
  a.t[a.index] = (u16)(a.t[a.index] + ((g - (int)a.t[a.index]) >> rate));
  a.t[a.index + 1] = (u16)(a.t[a.index + 1] + ((g - (int)a.t[a.index + 1]) >> rate));
  const int w = pr & 127;
  a.index = ((pr + 2048) >> 7) + (int)cxt * 33;
  return ((int)a.t[a.index] * (128 - w) + (int)a.t[a.index + 1] * w) >> 11;
}

// ---------------------------------------------------------------- the byte-level analysis (modelPrediction, bpos == 0)
FX_HD inline int cw_back(const TextState& X, int i) { return X.cwbuf[(X.cwpos - i) & CW_MASK]; }
FX_HD inline const char* word_str(const Tables& T, int idx) { return idx < 0 ? "" : T.dict_chars + T.dict_off[idx]; }
FX_HD inline bool str_is(const Tables& T, int idx, const char* w) {
  const char* s = word_str(T, idx);
  int i = 0;
  for (; s[i] && w[i]; ++i) if (s[i] != w[i]) return false;
  return s[i] == w[i];
}
FX_HD inline int decode_codeword(const Tables& T, int cw) {   // fxcmv1.cpp:412-436
  const int loaded = T.dict_loaded;
  int c = cw & 255;
  int sym = (loaded && c >= 128) ? c - 128 : 0;
  if (sym < 80) return sym;
  int i = 80 * (sym - 80);
  c = (cw >> 8) & 255;
  sym = (loaded && c >= 128) ? c - 128 : 0;
  if (sym < 80) return i + sym + 80;
  i = (i - 2560) * 32;
  i += 80 * (sym - 80);
  c = (cw >> 16) & 255;
  sym = (loaded && c >= 128) ? c - 128 : 0;
  return i + sym + 80 * 49;
}

// setbufstem (fxcmv1.cpp:3754-3800): append to the current word or close it, stem it and file it in the word lists
FX_HD inline void text_char(State& S, int c) {
  TextState& X = *S.text;
  X.cwbuf[X.cwpos & CW_MASK] = (u8)c;
  X.cwpos++;
  Word& cw = X.stem_words[X.cword];
  c = (int)(signed char)c;
  if ((c >= 'a' && c <= 'z') || (c == kApos && X.c2 != kApos) || (c == '-' && cw.len() > 0)) { cw.append(c); return; }
  if (cw.len() > 0 && c == kSqClose && X.fcx.cxt != (u32)kHtLink && X.is_paragraph) return;
  if (cw.len() == 0) return;
  Stemmer::stem(cw, (u32)S.blpos);
  X.stem_index = (X.stem_index + 1) & 3;
  X.pword = X.cword;
  X.cword = X.stem_index;
  X.stem_words[X.cword].clear();
  Word& pw = X.stem_words[X.pword];
  if (pw.type & T_Verb) X.s_verb = pw.hash;
  if (X.last_art) pw.type |= T_Noun;
  X.last_art = (pw.type == T_Article && cw_back(X, 5) == kSpace && cw_back(X, 4) == 't' && cw_back(X, 3) == 'h' && cw_back(X, 2) == 'e') ? 1 : 0;
  u32 whash = X.is_math ? X.word0 : pw.hash;
  X.last_wt = X.last_wt * 16 + (u32)word_class(pw.type);
  if (pw.type == T_Number && X.sent.typ(1) == T_Number) {
    const u16 sb = X.sent.sb(1);
    whash = whash + X.sent.word(1);
    X.sent.remove();
    X.sent.set((u8)(sb >> 8));
  }
  X.sent.add(X.word0, (u8)X.c1, pw.type, whash);
  if ((pw.type & (T_Conjunction + T_Article + T_Male + T_Female + T_Number + T_ConjAdverb)) == 0 && X.br.cxt != (u32)kLess)
    X.para.add(X.word0, (u8)X.c1, pw.type, whash);
  if ((pw.type & (T_Conjunction + T_Article + T_Male + T_Female + T_Adposition + T_Number + T_AdverbOfManner + T_ConjAdverb)) == 0 && X.br.cxt != (u32)kLess)
    if (pw.type) X.strm.add(X.word0, (u8)X.c1, pw.type, whash);
}
// procWord (fxcmv1.cpp:3810-3822)
FX_HD inline void text_codeword(State& S) {
  const Tables& T = *S.T;
  TextState& X = *S.text;
  if (X.dcwl <= 0) return;
  if (X.dcwl == 2) X.dcw = (X.dcw / 256) + (X.dcw & 255) * 256;
  if (X.dcwl == 3) X.dcw = ((X.dcw / 256) / 256) + (X.dcw & 0xff00) + (X.dcw & 255) * 256 * 256;
  if (X.dcwl > 3) return;
  if (T.dict_loaded) {
    const int j = decode_codeword(T, X.dcw);
    if (j > 0 && j < T.dict_n) { X.last_cw = j; X.so = j; }
  }
  X.dcw = X.dcwl = 0;
  const char* s = word_str(T, X.so);
  for (int i = 0; s[i]; ++i) text_char(S, s[i]);
}

// one whole byte has been coded: advance every byte-level context and set the map contexts for the next byte
FX_HD inline void text_byte(State& S) {
  const Tables& T = *S.T;
  TextState& X = *S.text;
  MapState* M = S.map;
  u32 c4 = S.c4;
  u32 h = 0;
  X.c3 = X.c2; X.c2 = X.c1; X.c1 = (int)(c4 & 0xff);
  int c1 = X.c1;
  const int c2 = X.c2, c3 = X.c3;
  const u8* wrt2 = T.wrt2; const u8* wrt3 = T.wrt3; const u8* wrt4 = T.wrt4;
  const u8* fcy = T.fcy; const u8* fcq = T.fcq;
  X.n2b = wrt2[c1]; X.n3b = wrt3[c1]; X.n4b = wrt4[c1];
  X.s2b = X.s2b * 4 + X.n2b;
  X.s4b = X.s4b * 16 + X.n4b;
  S.buffer[X.pos & BUF_MASK] = (u8)c1;
  X.pos++;
  if (c2 == kGreater && X.is_text) {
    X.is_text = 0;
    if (c1 == kApos || c1 == kFirstUpper) {
      X.cols.update(kLF, 0, (u32)S.blpos, X.is_pre != 0);
      X.sent.clear(); X.para.clear();
      X.fc = X.is_paragraph = 0; X.first_word = 0;
      X.nl1 = X.nl; X.nl = X.pos - 2;
    }
  }
  X.cols.update(c1, c4 & 0xffffff, (u32)S.blpos, X.is_pre != 0);
  if (c1 < 'a') X.br.update(c1);
  if (c1 == kSpace && c2 == kLess) X.br.update(kGreater);
  map_set(M[M0_4], (X.br.context << 8) + (u32)c1);
  X.qo.update(c1);
  if (X.ht.cxt && c2 == 'L' && (c1 == kSpace || c1 == '!' || c1 < 128)) X.ht.update('&' * 256 + 'N');
  X.ht.update((int)(c4 & 0xffff));
  if (c1 == '$' || c1 == kSqClose || c1 == kVBar || c1 == ')' || c1 == kSqOpen) {
    if (c1 != c2) for (int i = 13; i > 0; --i) X.t[i] = X.t[i - 1] * T.primes[i];
    X.x4 = (X.x4 << 8) + (u32)c2;
    X.s2b = X.s2b * 4 + X.n2b;
    X.s2bR = (X.s2bR << 2) + X.n2b;
    X.s3bR = (X.s3bR << 3) + X.n3b;
  }
  X.x4 = (X.x4 << 8) + (u32)c1;
  for (int i = 13; i > 0; --i) X.t[i] = X.t[i - 1] * T.primes[i] + (u32)c1 + (u32)i * 256;
  if (X.fc == kSpace && c1 == kSpace) { map_skip(M[M2_0]); map_skip(M[M2_0]); map_skip(M[M2_0]); }
  else for (int i = 3; i < 6; ++i) map_set(M[M2_0], X.t[i]);
  map_set(M[M2_1], X.t[6]);
  map_set(M[M2_2], X.t[8]);
  map_set(M[M2_3], X.t[13]);

  X.words = (u8)(X.words << 1); X.spaces = (u8)(X.spaces << 1); X.numbers = (u8)(X.numbers << 1);
  const u32 j = (u32)c1;
  if (((j - 'a') <= (u32)('z' - 'a')) || (c1 > 127 && c2 != kEscape)) {
    if (X.word0 == 0) {
      if (X.is_math && c2 == '/' && c3 == kLess) X.is_math = 0;
      u8 re = (u8)c2;
      if (c2 == kFirstUpper || c2 == kUpper) {
        if (c3 != kApos) re = (u8)c3;
        else if (buf(S, 4) != kApos) re = (u8)buf(S, 4);
        else if (buf(S, 5) != kApos) re = (u8)buf(S, 5);
        else if (buf(S, 6) != kApos) re = (u8)buf(S, 6);
        else re = (u8)c3;
      } else if (c2 == '/' && c3 == kLess) re = (u8)c3;
      X.sent.set(re, c2 == kFirstUpper ? 1 : 0);
      X.para.set(re);
    }
    X.words |= 1;
    X.word0 = X.word0 * 2104 + j;
    X.word00 = X.word0;
    h = X.word0 * 271; X.u8w = 0;
    if (X.br.cxt == (u32)kSqOpen && X.fcx.cxt != (u32)kHtLink && X.fc != kHtml) X.linkword = X.linkword * 2104 + j;
    if (X.is_paragraph && X.fcx.cxt != (u32)kHtLink && !X.cols.is_temp) X.senword = X.senword * 2104 + j;
    const int w3 = X.words & 7;
    if ((w3 == 5 && c2 == kApos) || (w3 == 1 && c3 == kSqClose && c2 == kApos) || (w3 == 1 && (X.numbers & 4) && c2 == kApos)) X.qo.update((int)X.qo.cxt);
    if (c1 > 127) {
      X.dcw = X.dcw * 256 + c1; X.dcwl++;
      if (S.blpos > 6) {
        int dcw2 = 0;
        if (X.dcwl == 2) dcw2 = (X.dcw / 256) + (X.dcw & 255) * 256;
        else if (X.dcwl == 3) dcw2 = ((X.dcw / 256) / 256) + (X.dcw & 0xff00) + (X.dcw & 255) * 256 * 256;
        const int i = decode_codeword(T, dcw2);
        if (i > 0 && i < T.dict_n) X.deccode = i;
      }
    } else if (X.dcw) {
      text_codeword(S);
      if (S.blpos < 448131719) X.deccode = X.last_cw;
    }
    if (c1 == 10 || c1 == 9 || (c1 > 31 && c1 < 128)) text_char(S, char_swap(c1));
  } else {
    if (X.word0) {
      text_codeword(S);
      if (S.blpos < 448131719) X.deccode = X.last_cw;
    } else X.deccode = 0x10000 + (int)(X.s2b & 0xffff);
    if (c1 == 10 || c1 == 9 || (c1 > 31 && c1 < 128)) text_char(S, char_swap(c1));
    if (c1 >= '0' && c1 <= '9') {
      X.numbers = (u8)(X.numbers + 1);
      if ((X.numbers & 4) && c2 == ',') { X.number0 = X.number1; X.number1 = 0; X.numlen0 = X.numlen1; X.numlen1 = 0; }
      if (X.mybenum && X.numlen1 <= 2) { X.number0 = X.number1; X.number1 = 0; X.numlen0 = X.numlen1; X.numlen1 = 0; }
      X.number0 = X.number0 * 10 + (u32)(c1 & 0x0f);
      X.numlen0 = (u32)imin(19, (int)X.numlen0 + 1); X.mybenum = 0;
    } else {
      if (X.numlen0 || ((X.numbers & 0xf) == 0)) { X.number1 = X.number0; X.numlen1 = X.numlen0; X.number0 = X.numlen0 = 0; }
      if (X.numlen1 <= 2 && X.numlen1 && ((X.numbers & 5) == 5) && X.numlen0 == 0 && c2 == '.') X.mybenum = 2;
      else if (X.numlen1 <= 2 && X.numlen1 && (X.numbers & 2) && X.numlen0 == 0 && c1 == '.') X.mybenum = 1;
      else if (X.mybenum == 1 && c1 != '.') X.mybenum = 0;
    }
    const int w3 = X.words & 7;
    if ((w3 == 4 && c1 == kSpace && c2 == kApos) || (c1 == kFirstUpper && (X.numbers & 4) && c2 == kApos) ||
        (w3 == 4 && c1 == kFirstUpper && c2 == kApos) || (w3 == 4 && (X.numbers & 1) && c2 == kApos)) X.qo.update((int)X.qo.cxt);
    if (X.word00 && !(X.fcx.cxt == (u32)kSqOpen)) X.word00 = 0;
    if (X.word0) {
      Word& pw = X.stem_words[X.pword];
      if (S.blpos > 463139793 || (pw.type & (T_ConjAdverb + T_Conjunction)) == 0) { X.word3 = X.word2 * 47; X.word2 = X.word1 * 53; X.word1 = X.word0 * 83; }
      if (X.sent.typ(1) == T_Number) { X.s3bR = (X.s3bR << 7) + 1; X.s3b = (X.s3b << 7) + 1; }
      if (X.first_word == 0 && X.fcx.cxt != (u32)kSqOpen) X.first_word = X.word0;
      if (X.sent.typ() & T_Conjunction) { X.s3bR = X.s3bR << 7; X.s3b = X.s3b << 7; if (X.is_paragraph) X.senword = 0; }
      if (X.sent.typ() & T_Article) { X.s3bR = (X.s3bR << 7) + 2; X.s3b = (X.s3b << 7) + 2; }
      if ((X.sent.typ() & T_Adposition) || (X.is_paragraph && (X.sent.typ() & T_PresentParticiple))) {
        X.s2bR = (X.s2bR << 2) + (X.s2bR & 3);
        X.s2b = (X.s2b << 2) + (X.s2b & 3);
      }
      if (X.sent.typ() & T_AdverbOfManner) { if (X.is_paragraph) X.sent.remove(); }
      if ((X.sent.typ() & T_Noun) && (X.sent.typ(2) & T_Article)) {
        X.s3bR = (X.s3bR << 6) + 1; X.s3b = (X.s3b << 6) + 1;
        const u16 sb = X.sent.sb(1); const u32 w = X.sent.word(1), t = X.sent.typ(1); const u8 ca = X.sent.cap(1);
        X.sent.remove(); X.sent.remove();
        X.sent.set((u8)(sb >> 8), ca);
        X.sent.add(w, (u8)c1, t, w);
      }
      X.s3bR_mask2 = X.s3bR_mask1;
      X.s3b_mask1 = X.s3b_mask;
      X.s3b_mask = X.s2b_mask = X.s3bR_mask1 = 0;
    } else if (c1 == kVBar && X.cols.is_temp) {
      const u16 sb = X.sent.sb(1); const u32 w = X.sent.word(1), t = X.sent.typ(1); const u8 ca = X.sent.cap(1);
      X.sent.remove();
      X.sent.set((u8)(sb >> 8), ca);
      X.sent.add(w, (u8)c1, t, w);
    }
    // tag boundaries: text, nowiki, math, pre, page
    if (cw_back(X, 6) == char_swap(kLess) && cw_back(X, 5) == 't' && !X.is_text && c1 == kSpace && str_is(T, X.so, "text")) { X.is_text = 1; X.so = -1; }
    if (cw_back(X, 8) == char_swap(kLess) && !X.is_nowiki && str_is(T, X.so, "nowiki")) X.is_nowiki = 1;
    else if (cw_back(X, 9) == '/' && c1 == kGreater && X.is_nowiki && str_is(T, X.so, "nowiki")) { X.is_nowiki = X.is_pre = 0; X.so = -1; }
    if (X.is_math && ((c1 == kSpace && X.cols.lastfc() != kColon) || c1 == ',') && c2 == kGreater && str_is(T, X.so, "math")) { X.is_math = 0; X.so = -1; }
    if (X.is_math && c1 == '/' && c2 == kLess && c3 == kGreater && cw_back(X, 4) == 'h') { X.is_math = 0; X.so = -1; }
    if (!X.is_nowiki && cw_back(X, 6) == char_swap(kLess) && cw_back(X, 5) == 'm' && !X.is_math && c1 != '.' && cw_back(X, 7) != '&' && cw_back(X, 8) != '&' && str_is(T, X.so, "math")) X.is_math = 1;
    else if (cw_back(X, 6) == '/' && (c1 == kGreater || c1 == '&') && X.is_math && str_is(T, X.so, "math")) { X.is_math = 0; X.so = -1; }
    if (cw_back(X, 5) == char_swap(kLess) && c1 == kGreater && cw_back(X, 4) == 'p' && !X.is_pre && str_is(T, X.so, "pre")) { X.is_pre = 1; X.so = -1; }
    else if (cw_back(X, 5) == '/' && c1 == kGreater && cw_back(X, 4) == 'p' && str_is(T, X.so, "pre")) { X.is_pre = 0; X.so = -1; }
    if (cw_back(X, 6) == '/' && c1 == kGreater && cw_back(X, 5) == 'p' && str_is(T, X.so, "page")) X.is_pre = X.is_math = X.is_nowiki = 0;

    S.wp[X.word0 & 0xffff] = X.pos;
    X.word0 = 0; h = 0;
    if (X.linkword && c1 == kColon) X.linkword = 0;
    if (c1 == '-' && c2 == kSpace) { X.para.clear(); X.s_verb = 0; }
    int c2m = c2;   // the heading rule below rewrites the global c2
    if (c1 == kSpace) X.spaces++;
    else if (c1 == kLF) {
      X.fc = X.is_paragraph = 0; X.first_word = 0; X.last_wt = 0;
      X.nl1 = X.nl; X.nl = X.pos - 1;
      X.s3bR = X.s3bR << 7;
      X.s2b = X.s2b | 0x3fc;
      X.words = 0xfc;
      X.sent.clear(); X.para.clear();
      X.s2bR = X.s2bR << 2;
      X.s4b = X.s4b | 0xfff0;
      if (c2 == kLF) X.is_nowiki = 0;
    } else if (c1 == '.' || c1 == ')' || c1 == kQuestion) {
      X.last_wt = X.last_wt * 16;
      X.s3bR = X.s3bR << 7; X.s3b = X.s3b << 7;
      X.words = X.words | 0xfe;
      X.x5 = (X.x5 << 8) + (c4 & 0xff);
      X.s2b = X.s2b | 204;
      X.s4b = ((X.s4b & 0xffff0) << 8) + (X.s4b & 0xf);
      X.s2bR = X.s2bR & 0xffffffc0;
      if (c1 == '.') {
        X.wshift = 1;
        if (!(X.fcx.cxt == (u32)kSqOpen || X.fcx.cxt == '(' || X.cols.nl_char == kWikiTable || X.cols.lastfc() == '*')) X.sent.clear();
        X.senword = 0;
      }
      if (c1 == ')') X.senword = 0;
    } else if (c1 == ',') { X.words = X.words | 0xfc; X.senword = 0; }
    else if (c1 == '(') X.senword = 0;
    else if (c1 == kSemicolon) X.sent.clear();
    else if (c1 == kColon) {
      X.s3b = (X.s3b & 0xfffffff8) + 4;
      X.s2b = X.s2b | 12;
      X.x5 = (X.x5 << 8) + (c4 & 0xff);
      X.senword = 0;
    } else if (c1 == kCurlyClose || c1 == kCurlyOpen) {
      X.words = X.words | 0xfc;
      X.s3bR = X.s3bR & 0xffffffc0;
      X.x5 = (X.x5 << 8) + (c4 & 0xff);
      X.s3b = (X.s3b & 0xfffffff8) + 3;
    } else if (c1 == kSqClose) { X.s3b = (X.s3b & 0xfffffff8) + 3; X.linkword = 0; }
    else if (c1 == kLess || c2 == '&') X.words = X.words | 0xfc;
    else if ((c1 == '-' && X.cols.lastfc() == '*') && X.br.cxt != (u32)kSqOpen && X.is_paragraph == 0) { X.is_paragraph = 1; X.fc = kFirstUpper; }
    else if (c1 == kEquals) {
      X.s3b = (X.s3b & 0xfffffff8) + 4;
      X.c2 = '.'; c2m = '.';
      X.words = (u8)(X.words * 2);
    }
    if (c1 == '!' && c2m == '&') {
      X.c1 = c1 = kSpace;
      c4 = (c4 & 0xffffff00) + kSpace;
      X.s2b = (X.s2b & 0xfffffffc) + wrt2[kSpace];
      X.s3b = (X.s3b & 0xfffffff8) + wrt3[kSpace];
    } else if (X.cols.lastfc() == '*' && (c1 == ',' || c1 == kSpace) && c2m == kSqClose && X.is_paragraph == 0) { X.is_paragraph = 1; X.fc = kFirstUpper; }
  }
  const int c2n = X.c2;   // c2 as the rest of the function sees it (may have been rewritten to '.')
  X.x5 = (X.x5 << 8) + (c4 & 0xff);
  if (X.o2b != X.n2b) { X.s2bR = (X.s2bR << 2) + X.n2b; X.o2b = X.n2b; }
  X.s2b_mask = (X.s2b_mask << 2) + 3;
  if (X.o3b != X.n3b) {
    X.s3bR = (X.s3bR << 3) + X.n3b;
    X.s3bR_mask1 = (X.s3bR_mask1 << 3) + 7;
    X.s3bR_mask2 = (X.s3bR_mask2 << 3) + 7;
    X.o3b = X.n3b;
  }
  X.s3b = (X.s3b << 3) + X.n3b;
  X.s3b_mask = (X.s3b_mask << 3) + 7;
  X.s3b_mask1 = (X.s3b_mask1 << 3) + 7;
  const u8 brc = (u8)X.br.cxt;

  X.brfc_idx = 0;
  if (X.br.context) X.brfc_idx = fcy[brc & 127];
  if (X.br.context == 0 && X.qo.context) X.brfc_idx = fcy[(X.qo.context >> 8) & 127];

  X.col = X.cols.collen();
  int above = S.buffer[(X.nl1 + X.col) & BUF_MASK];
  int above1 = S.buffer[(X.nl1 + X.col - 1) & BUF_MASK];
  if (X.cols.nl_char == kGreater) { above = X.cols.colb(1, 0); above1 = X.cols.colb(1, 1); }
  if (X.cols.nl) {
    if ((int)(X.cols.nlpos(0) + 2 - X.cols.nlpos(1)) < 4) { X.fcx.clear(); X.br.clear(); X.qo.clear(); X.ht.clear(); }
    X.fc = X.cols.lastfc();
    if (X.fc == kGreater) X.fcx.clear();
    X.is_paragraph = X.fc == kFirstUpper ? 1 : 0;
    X.fcx.update(X.fc);
  }
  if (X.col > 2 && c1 > kFirstUpper && !X.is_math) {
    if (X.fcx.cxt == (u32)kVBar && (c1 == kSqClose || c1 == kCurlyClose)) while (X.fcx.cxt == (u32)kVBar) X.fcx.update(kLF);
    if ((X.fcx.cxt == (u32)kColon || X.fcx.cxt == (u32)kHtLink) && c1 == kSqClose) while (X.fcx.cxt == (u32)kColon || X.fcx.cxt == (u32)kHtLink) X.fcx.update(kLF);
    if (c1 < 128) X.fcx.update(c1);
  }
  if (c1 == kColon && (X.words & 2) == 2) X.colonstr = X.so;
  if (c1 == kSpace && X.fcx.cxt == (u32)kColon && X.cols.lastfc() != kColon && X.cols.nl_char != kWikiTable) {
    if (!str_is(T, X.colonstr, "image")) while (X.fcx.cxt == (u32)kColon) X.fcx.update(kLF);
  }
  if (c1 == kColon && (str_is(T, X.colonstr, "category") || str_is(T, X.colonstr, "wikipedia"))) { X.fcx.update(kLF); X.sent.remove(); }
  if (c1 == kSpace && c2n == kLess) X.fcx.update(kGreater);
  if (X.fcx.cxt == (u32)kColon && c2n == '/' && c1 == '/') { X.fcx.update(kLF); X.fcx.update(kHtLink); }
  if (X.cols.lastfc(0) == kSqOpen && c1 == kSpace && X.is_paragraph == 0) {
    if (c2n == kSqClose || c3 == kSqClose) { X.fc = kFirstUpper; X.is_paragraph = 1; X.fcx.clear(); X.fcx.update(X.fc); }
  }
  if (X.fc == kSpace && c1 != kSpace) {
    X.fc = imin(c1, kTextData);
    X.is_paragraph = X.fc == kFirstUpper ? 1 : 0;
    X.fcx.update(X.fc);
  }
  const u8 fcc = (u8)X.fcx.cxt;
  if (X.brfc_idx == 0 && X.fcx.context) X.brfc_idx = fcy[fcc & 127];
  X.fc_idx = fcq[fcc & 127];
  map_set(M[M0_5], (X.fcx.context & 0xff00) + (u32)c1 + (X.s2b & 12) * 256 + ((u32)(brc + X.br.last()) << 24));
  if (X.fc == '*' && c1 != kSpace) X.fc = imin(c1, kTextData);
  if (X.fc == '&' && c1 == kLess) X.fc = kHtml;
  if (c2n == kGreater && X.fc == kLess && c1 == kApos) X.fc = kApos;
  if ((X.cols.lastfc(0) == kApos || (X.fc == kApos && X.cols.lastfc(0) != '*')) && c1 == kSpace) {
    if (c2n == kApos || c3 == kApos) { X.fc = kFirstUpper; X.is_paragraph = 1; X.fcx.clear(); X.fcx.update(X.fc); }
  }
  if (X.fc != kFirstUpper && (c4 & 0xffffff) == 0x4a2f2f) X.fc = kHtLink;
  X.sent.drop_left(8, '(', ')'); X.para.drop_left(8, '(', ')');
  X.sent.drop_left(8, kSqOpen, kVBar); X.para.drop_left(8, kSqOpen, kVBar);
  X.sent.drop_left(8, kLess, kColon);
  if (X.cols.is_temp) X.sent.drop_right(10, kEquals, kVBar);
  X.sent.drop_left(8, kLess, kGreater); X.para.drop_left(8, kLess, kGreater);

  // indirect contexts
  X.ind_word = (c4 >> 8) & 0xffff;
  S.t2[X.ind_word] = (S.t2[X.ind_word] << 8) | (u32)c1;
  X.ind_word = c4 & 0xffff;
  X.ind_word = X.ind_word | (S.t2[X.ind_word] << 16);
  X.ind_byte = (c4 >> 8) & 0xff;
  X.t1[X.ind_byte] = (X.t1[X.ind_byte] << 8) | (u32)c1;
  X.ind_byte = (u32)c1 | (X.t1[c1] << 8);
  X.t1[brc] = (X.t1[brc] << 2) | (X.s2b & 3);
  X.ind_br_byte = (X.s3b & 7) | (X.t1[brc] << 3);
  X.ind_word0_pos = (u32)(X.pos - S.wp[X.word0 & 0xffff]);
  if (X.ind_word0_pos > 255) X.ind_word0_pos = 256 + ((u32)c1 << 16);
  else X.ind_word0_pos = X.ind_word0_pos + ((u32)buf(S, (int)X.ind_word0_pos) << 8) + ((u32)c1 << 16);
  S.ind3[X.ctx1_ind3] = (u16)((X.cxt_ind3 * 32 + (u32)c1) & (IND3_SIZE - 1));
  X.ctx1_ind3 = (X.ctx1_ind3 * 32 + (u32)c1) & (IND3_SIZE - 1);
  X.cxt_ind3 = S.ind3[X.ctx1_ind3];
  if (c2n == 12) {
    if (X.utf8left == 0) {
      if ((c1 >> 5) == 6) { X.utf8left = 1; X.u8w = X.u8w * 191 + (u32)c1; }
      else if ((c1 >> 4) == 0xE) { X.utf8left = 2; X.u8w = X.u8w * 191 + (u32)c1; }
      else if ((c1 >> 3) == 0x1E) { X.utf8left = 3; X.u8w = X.u8w * 191 + (u32)c1; }
      else X.utf8left = 0;
    } else { X.utf8left--; if ((c1 >> 6) != 2) X.utf8left = 0; }
  }
  h = h + (u32)c1;

  // map contexts
  const int col = X.col, fc = X.fc;
  const u32 s2b = X.s2b, s3b = X.s3b, s3bR = X.s3bR, s2bR = X.s2bR, x4 = X.x4;
  const u32 word0 = X.word0, word00 = X.word00, brfc = X.brfc_idx;
  Word& pw = X.stem_words[X.pword];
  rcm_set(S, X.word3 * 53 + (u32)c1 + 193 * (s3b & 0x7fff), (u8)c1);
  if (col < 2 || fc == kSpace) { map_skip(M[M2_4]); map_skip(M[M2_4]); map_skip(M[M2_17]); }
  else {
    map_set(M[M2_4], word00 + (X.number0 * 191 + X.numlen0) + X.u8w);
    if (X.cols.lastfc() == '&' || X.utf8left) map_skip(M[M2_4]); else map_set(M[M2_4], h + X.word1);
    if (X.br.cxt == (u32)kLess) map_skip(M[M2_17]); else map_set(M[M2_17], X.para.word(1) * 53 + X.para.word(2) * 11 + h + (X.last_wt & 0xf));
  }
  if (c1 == kEscape || col < 2 || X.utf8left || fc == kSpace) map_skip(M[M2_5]); else map_set(M[M2_5], h + X.word2 * 71);
  if (fc == kSpace || X.br.cxt == (u32)kLess) { for (int k = 0; k < 5; ++k) map_skip(M[M2_5]); }
  else {
    map_set(M[M2_5], X.sent.word(4) * 53 + X.para.word(1) + h + (s3b & 511));
    map_set(M[M2_5], X.sent.last(4, X.sent.typ(4) ^ T_Verb) * 53 + X.s_verb + h + (s3bR & 63));
    map_set(M[M2_5], X.sent.fword * 53 + X.para.word(1) + h + (s3b & 63));
    map_set(M[M2_5], X.strm.word(1) + X.strm.word(2) * 11 + word00 + (u32)c1);
    const u32 lpv = X.strm.last_if(1, X.sent.typ(1) & T_Verb);
    if (lpv) map_set(M[M2_5], lpv * 11 + word00 + (u32)c1); else map_skip(M[M2_5]);
  }
  map_set(M[M1_6], h + (X.sent.typ(1) & 0x1FF) + X.para.word(1));
  map_set(M[M2_6], ((s2b & 15) << 16) + (X.t[2] & 0xffff));
  if (c1 == kEscape || X.utf8left || fcc == kCurlyOpen) map_set(M[M2_7], 0); else map_set(M[M2_7], X.ind_br_byte);
  map_set(M[M2_8], ((X.ind_br_byte >> 0) & 0x7ff) * 32 + ((X.s4b & 0xfff0) << 16) + brfc);
  map_set(M[M2_8], (s3bR & 0x3fffffff) * 4 + (s2b & 3));
  map_set(M[M2_8], ((u32)fcc * 4) + ((s3bR & 0x3ffff) << 9) + brfc);
  if (fcc == kHtLink) map_skip(M[M2_8]); else map_set(M[M2_8], (c4 & 0xffffff) + ((s2b << 18) & 0xff000000));
  map_set(M[M1_0], (u32)X.cols.lastfc(0) | ((u32)fcc << 15) | ((s3b & 63) << 7) | ((u32)brc << 24));
  map_set(M[M1_0], ((u32)X.cols.lastfc(0) | ((c4 & 0xffffff) << 8)));
  map_set(M[M1_1], (s2b & 3) + word00 * 11);
  map_set(M[M1_1], c4 & 0xffff);
  map_set(M[M1_1], (((u32)fc << 11) | (u32)c1) + ((s2b & 3) << 18));
  map_set(M[M1_2], (s2b & 15) + ((s3b & 7) << 6));
  map_set(M[M1_2], (u32)c1 | ((u32)(col * (c1 == kSpace)) << 8) | ((s2b & 15) << 16));
  map_set(M[M1_2], X.is_paragraph ? X.first_word : ((u32)fc << 11));
  if (c1 == kEscape || fc == kSpace || X.utf8left) map_skip(M[M1_2]); else map_set(M[M1_2], (91u * 83u * X.sent.word(1) + 89u * word0));
  if (fc == kSpace) map_skip(M[M1_4]); else map_set(M[M1_4], ((u32)c1 + ((s3b & 0xe38) << 6)));
  map_set(M[M1_4], X.sent.fword * 11 + brfc);
  map_set(M[M1_4], (u32)c1 + word0 + X.number0 * 191);
  map_set(M[M1_4], ((c4 & 0xffff) << 16) | ((u32)fcc << 8) | (u32)fc);
  map_set(M[M1_4], ((s3bR & 0xfff) << 8) + (s2b & 0xfc));
  if (c1 == kEscape) { for (int k = 0; k < 6; ++k) map_skip(M[M0_0]); }
  else {
    if (X.is_paragraph == 1) {
      map_set(M[M0_0], X.sent.fword * 3191 + (s2b & 3));
      map_set(M[M0_0], h + X.first_word * 89);
      map_set(M[M0_0], word0 * 53 + (u32)c1 + brfc);
    } else {
      map_set(M[M0_0], (u32)above | ((s3b & 0x3f) << 9) | ((u32)X.cols.collen() << 19) | ((s2b & 3) << 16));
      map_set(M[M0_0], h + X.first_word * 89);
      map_set(M[M0_0], (u32)above | ((u32)c1 << 16) | (((u32)col + X.numlen0 + brfc) << 8) | ((u32)above1 << 24));
    }
    if (X.cols.lastfc() == '*') {
      map_set(M[M0_0], (word0 + ((u32)fcc << 8)) | (brfc << 16));
      map_set(M[M0_0], (u32)c1);
      map_set(M[M0_0], word0);
    } else {
      const u32 ab = (u32)bufr(S, (u32)X.cols.above);
      map_set(M[M0_0], wrt2[ab] | ((u32)fcc << 8) | (brfc << 16));
      map_set(M[M0_0], ab | ((u32)c1 << 8));
      map_set(M[M0_0], word0 + wrt2[ab]);
    }
  }
  map_set(M[M0_1], (s3b & 0x7fff) * word0 + brfc);
  map_set(M[M0_1], (x4 & 0xff0000ff) | ((s3b & 0xe07) << 8));
  map_set(M[M0_1], (X.ind_br_byte & 0xffff) | ((s3b & 0x38) << 16));
  if (X.is_math) map_skip(M[M0_0]); else map_set(M[M0_0], (X.ind_byte & 0xff00) + 257u * X.sent.word(1) * 53u + (u32)c1);
  map_set(M[M0_2], ((u32)c1 << 8) | (X.ind_byte >> 2) | ((u32)fc << 16));
  map_set(M[M0_2], (c4 & 0xffff) + (c2n == c3 ? 1 : 0));
  map_set(M[M1_3], (s3b & X.s3b_mask) * 256 | (s2b & X.s2b_mask & 255));
  map_set(M[M1_3], x4);
  map_set(M[M2_9], 257u * pw.hash + (u32)fcc + 193u * (s3b & X.s3b_mask));
  map_set(M[M2_9], (u32)fc | ((s2bR & 0xfff) << 9) | ((u32)c1 << 24));
  map_set(M[M2_16], X.sent.fword * 83 + (s2b & 15) * 11 + (u32)brc);
  map_set(M[M2_17], X.sent.last(1, T_Verb) + X.sent.word(1) * 83 + h);
  map_set(M[M2_9], (x4 & 0xffff00) + (u32)brc + ((u32)fcc << 24));
  if (X.linkword) map_set(M[M2_9], X.linkword);
  else if (X.is_math) map_skip(M[M2_9]);
  else if (X.senword) map_set(M[M2_9], X.senword * 1471 + (u32)c1);
  else { if (fc == kHtml || brc == kLess) map_skip(M[M2_9]); else map_set(M[M2_9], 0); }
  map_set(M[M2_10], X.ind_byte);
  map_set(M[M2_10], ((X.ind_byte & 0xffff00) >> 4) | (s2b & X.s2b_mask & 0xf) | ((s3b & 0xfff) << 20));
  map_set(M[M2_10], (x4 >> 16) | ((s2b & 255) << 24));
  if (c1 > 127) map_set(M[M2_10], ((((s2b & 12) * 256) + (u32)c1) << 11) | ((X.ind_word & 0xffffff) >> 16));
  else map_set(M[M2_10], ((u32)c1 << 11) | (brfc << 8) | ((X.ind_word & 0xffffff) >> 16));
  if (X.is_math) map_skip(M[M2_10]); else map_set(M[M2_10], ((u32)fcc * 4 + brfc) | ((c4 & 0xffff) << 9) | ((s2b & 0xff) << 24));
  map_set(M[M2_10], (X.ind_word >> 16) | ((s2b & 0x3c) << 25) | ((s3b & 0x1ff) << 16));
  map_set(M[M2_11], (u32)X.words + ((u32)X.spaces << 8) + ((s2b & 15) << 16) + (((s3bR >> 3) & 511) << 21) + ((u32)X.is_paragraph << 30));
  map_set(M[M2_11], (u32)c1 + ((s3b << 5) & 0x1fffff00));
  map_set(M[M2_11], s2bR * 16 + brfc);
  map_set(M[M2_11], ((X.ind_byte & 0xffff) >> 8) + ((64 * s2bR) & 0x3ffff00) + ((u32)brc << 25));
  if (fcc == kFirstUpper && brc == kSqOpen) map_skip(M[M2_11]); else map_set(M[M2_11], X.ind_word0_pos | ((X.ind_byte & 0xff00) << 16));
  map_set(M[M2_12], (x4 & 0x80f00000) + ((x4 & 0x0000f0ff) << 12));
  if (X.is_paragraph == 1) {
    if (c1 == kEscape || fcc == kHtLink || fcc == kCurlyOpen || X.is_math || X.is_pre) map_skip(M[M2_12]);
    else map_set(M[M2_12], h + X.sent.word(1) * 53 * 79 + X.sent.word(3) * 53 * 47 * 71);
  } else {
    if (fcc == kHtLink || brc == kLess || X.ht.cxt) map_skip(M[M2_12]);
    else if (col == 31) map_set(M[M2_12], c4 << 16);
    else map_set(M[M2_12], (u32)above | ((c4 & 0xffff) << 16) | ((u32)above1 << 8));
  }
  const bool bslash = (X.sent.sb(0) >> 8) == '\\';
  if (c1 == kEscape || X.utf8left || fcc == kCurlyOpen || fcc == kHtLink || fc == kHtml || X.ht.cxt || fc == kSpace || X.is_pre || c1 == '&' ||
      brc == kLess || X.is_math || col < 2 || bslash) { map_skip(M[M2_13]); map_skip(M[M2_13]); }
  else {
    map_set(M[M2_13], X.sent.word(1) * 83 * 1471 - word0 * 53 + X.sent.word(2));
    map_set(M[M2_13], h + X.sent.word(2) * 53 * 79 + X.sent.word(3) * 53 * 47 * 71);
  }
  map_set(M[M0_3], ((s3bR & 7) << 10) + (s2b & 3) + (u32)fc * 4 + (brfc << 24));
  map_set(M[M0_3], ((X.linkword ? X.linkword : word0) * 3301 + X.number0 * 3191));
  if (c1 == kEscape || X.utf8left || fcc == kCurlyOpen || fcc == kHtLink || fc == kSpace || fc == kHtml || brc == kLess || col < 2 || X.is_math || bslash)
    map_skip(M[M2_14]);
  else map_set(M[M2_14], brfc + X.sent.word(2) * (s3bR & X.s3bR_mask2) + (X.sent.typ(1) & 0x1ff));
  if (c1 == kEscape || X.utf8left || fc == kSpace) { for (int k = 0; k < 4; ++k) map_skip(M[M1_7]); }
  else {
    map_set(M[M1_7], X.para.word() + word00);
    map_set(M[M1_7], X.sent.word(2) + word0 * 191 + (s3bR & 63));
    map_set(M[M1_7], word0 * 191 + (s3bR & 63));
    map_set(M[M1_7], (X.ind_word0_pos & 0xffff) * 191 + word0 + (s3bR & 63));
  }
  scm_set(S.scm[0], (u32)c1);
  scm_set(S.scm[1], (u32)(c2n * X.is_paragraph));
  scm_set(S.scm[2], (X.ind_word & 0xffffff) >> 16);
  scm_set(S.scm[3], s3b & 0x1ff);
  scm_set(S.scm[4], s2b & 0xff);
  scm_set(S.scm[5], (u32)brc);
  scm_set(S.scm[6], (u32)X.is_paragraph + 2 * (s3bR & 0x3f));
  if (X.wshift || c1 == kLF) {
    X.word3 = X.word3 * 47; X.word2 = X.word2 * 53; X.word1 = X.word1 * 83;
    X.wshift = 0;
    if (c1 == kLF) X.s_verb = 0;
  }
  map_set(M[M2_15], (brfc * 256) + (u32)fc + ((s3bR & 0xFFF) << 16));
  X.ah1 = hash3((X.x5 >> 0) & 255, (X.x5 >> 8) & 255, (X.x5 >> 16) & 0x80ff);
  X.ah2 = hash3(19, X.x5 & 0x80ffff);
  S.mix[8].cxt = X.deccode;
}


// ================================================================ one bit, in phases
// Phase A (one lane): bit bookkeeping of update1 (fxcmv1.cpp:4758-4781) and the mixers' error terms. The models read only
// the first half; the second touches the mixers alone (fxcm.cuh runs the halves on different CTAs).
FX_HD inline bool bit_head_model(State& S, int y, int lstmpr, int lstmex) {   // true when the bit ends a byte
  S.y = y; S.lstmpr = lstmpr; S.lstmex = lstmex;
  S.c0 += S.c0 + y;
  const bool byte_end = S.c0 >= 256;
  if (byte_end) {
    S.c4 = (S.c4 << 8) + (u32)(S.c0 & 0xff);
    S.c0 = 1;
    ++S.blpos;
    S.sscmrate = S.blpos > 14 * 256 * 1024;
    S.rate = 6 + (S.blpos > 14 * 256 * 1024) + (S.blpos > 28 * 512 * 1024);
  }
  S.bpos = (S.bpos + 1) & 7;
  S.bposshift = 7 - S.bpos;
  S.c0shift_bpos = (S.c0 << 1) ^ (256 >> S.bposshift);
  return byte_end;
}
FX_HD inline void bit_head_mixer(State& S, int y, bool byte_end) {
  const Tables& T = *S.T;
  if (byte_end) {
    if ((S.fails & 255) == 0) { for (int i = 0; i < 10; ++i) S.mix[i].elim = imax(256, S.mix[i].elim + 1); }
    else { for (int i = 0; i < 10; ++i) S.mix[i].elim = imax(0, imin(16, S.mix[i].elim - 1)); }
  }
  for (int i = 0; i < N_MIX; ++i) {   // Mixer1::update (fxcmv1.cpp:610-619)
    MixState& m = S.mix[i];
    int err = ((y << 12) - m.pr) * T.mix_uperr[i] / 4;
    if (err > 32767) err = 32767;
    if (err < -32768) err = -32768;
    if (err >= -m.elim && err <= m.elim) err = 0;
    m.err = err;
  }
}
FX_HD inline void bit_head(State& S, int y, int lstmpr, int lstmex) { bit_head_mixer(S, y, bit_head_model(S, y, lstmpr, lstmex)); }
// Phase B (all lanes): SGD step of the 12 selected weight rows. `lane`/`lanes` partition the weights.
FX_HD inline void bit_train(State& S, int lane, int lanes) {
  for (int i = 0; i < 10; ++i) {
    const MixState& m = S.mix[i];
    if (!m.err) continue;
    short* w = m.w + (size_t)m.cxt * N_IN1;
    for (int k = lane; k < N_IN1; k += lanes) w[k] = train_one(S.in1[k], w[k], m.err);
  }
  for (int i = 10; i < N_MIX; ++i) {
    const MixState& m = S.mix[i];
    if (!m.err) continue;
    short* w = m.w + (size_t)m.cxt * N_IN2;
    for (int k = lane; k < N_IN2; k += lanes) w[k] = train_one(S.in2[k], w[k], m.err);
  }
}
// Phase C (one lane): failure history, then (byte boundary) the text analysis, then the units' slices of the vectors.
FX_HD inline void bit_fail_history(State& S) {   // the mixers' half: read by the APMs and mixer 9's selector only
  const Tables& T = *S.T;
  if (S.fails & 0x00000080) --S.failcount;
  S.fails = S.fails * 2;
  S.failz = S.failz * 2;
  int pr = S.pr;
  if (S.y) pr = 4095 - pr;
  if (pr >= T.e_l[S.bpos]) { ++S.fails; ++S.failcount; }
  if (pr >= 848) ++S.failz;
  S.pr = pr;
}
FX_HD inline void bit_prepare_model(State& S) {
  if (S.bpos == 0) text_byte(S);
  S.ord_x = S.map[M2_0].mask ? 2 : 0;      // cmC2[0].cxtMask is sampled before its mix() (fxcmv1.cpp:4590-4591)
}
FX_HD inline void bit_prepare_head(State& S) { bit_fail_history(S); bit_prepare_model(S); }
FX_HD inline void unit_counts(const State& S, int u, int& ni, int& ei) {   // inputs / exports of unit u this bit
  if (u < U_MATCH) { ni = 2; ei = 1; }
  else if (u == U_MATCH) { ni = 7; ei = 7; }
  else if (u == U_SMATCH) { ni = 2; ei = 2; }
  else if (u == U_RCM) { ni = 1; ei = 1; }
  else { const int id = u - U_MAP0; const int k = S.T->spec[id].skip2; ni = S.map[id].cn * (5 + k); ei = S.map[id].cn * (4 + k); }
}
FX_HD inline void bit_prepare(State& S) {
  bit_prepare_head(S);
  int ni = 0, ei = 0;
  for (int u = 0; u < N_UNITS; ++u) {
    S.in_off[u] = ni; S.ex_off[u] = ei;
    int a, b;
    unit_counts(S, u, a, b);
    ni += a; ei += b;
  }
  S.in_off[N_UNITS] = ni; S.ex_off[N_UNITS] = ei;
}
// Phase D (one lane per unit)
FX_HD inline void bit_unit(State& S, int u) {
  Out o; o.n = S.in1; o.codes = S.codes; o.ni = S.in_off[u]; o.ei = S.ex_off[u];
  if (u < U_MATCH) scm_bit(S, u, o);
  else if (u == U_MATCH) match_bit(S, o);
  else if (u == U_SMATCH) smatch_bit(S, o);
  else if (u == U_RCM) rcm_bit(S, o);
  else map_bit(S, u - U_MAP0, o);
}
// Phase E (one lane): weight-set selection of the ten first-layer mixers and of the final one (fxcmv1.cpp:4634-4738).
// Mixer 9 selects on the failure history, which the mixers own; the others on what the models have finished with.
FX_HD inline void bit_select_mixer(State& S) { S.mix[9].cxt = (S.bpos << 8) * 4 + (int)(S.fails & 3) * 256 + S.lstmex; }
FX_HD inline void bit_select_model(State& S) {
  const Tables& T = *S.T;
  const TextState& X = *S.text;
  const int bpos = S.bpos, c0 = S.c0;
  int ni = S.in_off[N_UNITS], ei = S.ex_off[N_UNITS];
  S.codes[ei++] = (u16)squash(T, 64);
  S.in1[ni++] = (short)stretch(T, S.lstmpr);
  S.in_off[N_UNITS] = ni; S.ex_off[N_UNITS] = ei;
  const MapState* M = S.map;
  int ord_x = S.ord_x + (int)M[M2_0].result;
  if (ord_x == 3) ord_x = 2;
  ord_x += (int)(M[M2_1].result + M[M2_2].result + M[M2_3].result);
  int ord_w = (int)(M[M2_4].result + M[M2_5].result);
  if (ord_w > 3) ord_w = 3;
  ord_w += (int)(M[M2_13].result + M[M2_14].result);
  const int is_match = S.is_match;
  const u32 s2b = X.s2b, s3b = X.s3b, s3bR = X.s3bR, brfc = X.brfc_idx, fci = X.fc_idx;
  const int words = X.words, numbers = X.numbers, para = X.is_paragraph;
  const int c0b = c0 << (8 - bpos);
  int c;
  MixState* mx = S.mix;
  if (bpos == 0) mx[0].cxt = (int)((s2b & 255) * 8 + (s3b & 7));
  else if (bpos > 3) { c = T.wrt2[c0b & 255]; mx[0].cxt = (int)((((s2b << 2) & 255) + (u32)c) * 8 + brfc); }
  else mx[0].cxt = (int)((s2b & 255) * 8 + brfc);
  if (bpos) {
    c = c0b;
    if (bpos == 1) c = c + 16 * (words * 2 & 4);
    else if (bpos > 3) c = T.wrt2[c0b & 255] * 64;
    c = imin(bpos, 5) * 256 + (int)(s3bR & 7) + (int)fci * 8 + (c & 192);
  } else c = (words & 12) * 16 + (int)(s3bR & 7) + (int)brfc * 8;
  mx[1].cxt = c;
  mx[2].cxt = ((4 * words) & 0xf0) * 4 + ord_x * 256 * 4 + (int)(s2b & 63);
  mx[6].cxt = (int)((s3bR & 0xff8) * 4) + ((2 * words) & 0x1c) + (int)(s2b & 3);
  c = c0b;
  mx[3].cxt = bpos * 256 + (((((numbers | words) << bpos) & 255) >> bpos) | (c & 255));
  mx[10].cxt = (ord_x * 8 + (brfc ? 1 : 0) * 4 + (int)(s2b & 3)) * 2 + (words & 1);
  if (bpos) {
    if (bpos == 1) c = c + 16 * (int)(s3b & 7);
    else if (bpos == 2) c = c + 16 * (int)(s2b & 3);
    else if (bpos == 3) c = c + 16 * (words & 1);
    else c = bpos + (c & 0xf0);
    if (bpos < 5) c = bpos + (c & 0xf0);
  } else c = 16 * (int)(s2b & 0xf);
  ord_x = ord_x - 1;
  if (ord_x < 0) ord_x = 0;
  if (is_match) ord_x = ord_x + 1;
  mx[4].cxt = c + ord_x * 256 + 8 * para;
  mx[5].cxt = (int)((ord_w * 256 + (s2b & 0xf0) + ((s3b & 0x38) >> 2)) * 4 + fci);
  if (bpos > 2) mx[7].cxt = (int)(((s3b & 7) * 8 + T.wrt3[c0b & 255]) * 256 + brfc * 32 + (u32)(words & 7) * 4 + (u32)para + (is_match ? 2 : 0));
  else mx[7].cxt = (int)(((s3b & 63) * 256 + brfc * 16 + (u32)(words & 7) * 2 + (u32)para) | (is_match ? 128u : 0u));
  S.ord_x = ord_x; S.ord_w = ord_w;
}
FX_HD inline void bit_select(State& S) { bit_select_model(S); bit_select_mixer(S); }
// Phase F (all lanes): the ten 512-wide dot products; lane l of `lanes` returns its partial sums in part[10].
FX_HD inline void bit_dot_partial(const State& S, int lane, int lanes, int* part) {
  for (int i = 0; i < 10; ++i) {
    const short* w = S.mix[i].w + (size_t)S.mix[i].cxt * N_IN1;
    int acc = 0;
    for (int k = 2 * lane; k < N_IN1; k += 2 * lanes) acc += dot_pair(S.in1 + k, w + k);
    part[i] = acc;
  }
}
// Phase G (one lane): squash, final mixers, the six APMs, export (fxcmv1.cpp:4742-4755, :4798-4833).
FX_HD inline void bit_tail(State& S, const int* dots) {
  const Tables& T = *S.T;
  const TextState& X = *S.text;
  int ei = S.ex_off[N_UNITS];
  for (int i = 0; i < 10; ++i) {
    int dp = (int)((u32)dots[i] * (u32)T.mix_shift[i]) >> 11;
    dp = clp(dp);
    S.mix[i].pr = squash(T, dp);
    S.in2[i] = (short)dp;
    S.codes[ei++] = (u16)S.mix[i].pr;
  }
  S.in2[10] = (short)(stretch(T, S.lstmpr) / 2);
  int fin[2];
  for (int i = 10; i < N_MIX; ++i) {
    const short* w = S.mix[i].w + (size_t)S.mix[i].cxt * N_IN2;
    int acc = 0;
    for (int k = 0; k < N_IN2; k += 2) acc += dot_pair(S.in2 + k, w + k);
    int dp = (int)((u32)acc * (u32)T.mix_shift[i]) >> 11;
    dp = clp(dp);
    S.mix[i].pr = squash(T, dp);
    fin[i - 10] = dp;
  }
  int pr = squash(T, (fin[0] * 7 + fin[1] + 4) >> 3);
  S.codes[ei++] = (u16)pr;
  const int y = S.y, c0 = S.c0, rate = S.rate;
  const u32 fails = S.fails;
  int pu = (apm_p(T, S.apm[0], pr, (u32)c0, 3, y) + 7 * pr + 4) >> 3;
  int pz = (int)S.failcount + 1;
  const int tri[4] = {0, 4, 3, 7}, trj[4] = {0, 6, 6, 12};
  pz += tri[(fails >> 5) & 3];
  pz += trj[(fails >> 3) & 3];
  pz += trj[(fails >> 1) & 3];
  if (fails & 1) pz += 8;
  pz = pz / 2;
  pu = apm_p(T, S.apm[3], pu, ((u32)(c0 * 2) ^ X.ah1) & 0x3ffff, rate, y);
  S.codes[ei++] = (u16)pu;
  int pv = apm_p(T, S.apm[1], pr, ((u32)(c0 * 8) ^ hash3(29, S.failz & 2047)) & 0xffff, rate + 1, y);
  S.codes[ei++] = (u16)pv;
  if (fails & 255) pv = apm_p(T, S.apm[4], pv, hash3((u32)c0, X.s2b & 0xfffc, X.s3bR & 0x1ff) & 0x3ffff, rate, y);
  else pv = apm_p(T, S.apm[4], pv, hash3((u32)c0, (X.s2bR & 0xfffc) + 0x10000, X.s3bR & 0x1ff) & 0x3ffff, rate, y);
  S.codes[ei++] = (u16)pv;
  const int pt = apm_p(T, S.apm[2], pr, ((u32)(c0 * 32) ^ X.ah2) & 0xffff, rate, y);
  S.codes[ei++] = (u16)pt;
  pz = apm_p(T, S.apm[5], pu, ((u32)(c0 * 4) ^ hash3((u32)imin(9, pz), X.x5 & 0x80ff)) & 0x3ffff, rate, y);
  S.codes[ei++] = (u16)pz;
  if (fails & 255) pr = (pt * 6 + pu + pv * 11 + pz * 14 + 31) >> 5;
  else pr = (pt * 4 + pu * 5 + pv * 12 + pz * 11 + 31) >> 5;
  S.codes[ei++] = (u16)pr;
  S.pr = pr;
}

// The whole bit on one lane (CPU pinning, lock-step fallback of small launches).
FX_HD inline void bit_serial(State& S, int y, int lstmpr, int lstmex) {
  bit_head(S, y, lstmpr, lstmex);
  bit_train(S, 0, 1);
  bit_prepare(S);
  for (int u = 0; u < N_UNITS; ++u) bit_unit(S, u);
  bit_select(S);
  int dots[10];
  bit_dot_partial(S, 0, 1, dots);
  bit_tail(S, dots);
}

}  // namespace fx
}  // namespace cmixb200
#endif
