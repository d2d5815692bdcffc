// cmix_b200/csrc/small_models.cuh
//
// Kernel "small": the shared context state (reference src/context-manager.cpp:69-94,
// src/contexts/*.cpp) and the 54 small cmix bit models + the PPMD bit read-out
// (reference src/models/{direct,direct-hash,indirect,match,bracket,byte-model}.cpp),
// SURVEY §8 rows a8, a16, a17, a18.
//
// One 64-thread CTA per stream; lane l owns model l (models_ order of the
// reference, FXCM/PAQ8 skipped), lane 54 owns the PPMD ByteModel read-out.
// Per bit: predict -> perceive -> context advance (-> byte update). The state
// machines are scalar and branchy; what the GPU buys here is that all 55 table
// walks (2 GB shared nibble map, 0.9 GB direct tables, 0.7 GB match maps) issue
// their dependent HBM loads concurrently instead of one after the other.
#pragma once
#include "exact_math.h"
#include "jitter.cuh"
#include "state.h"
#include "bytemodel.cuh"

namespace cmixb200 {

__constant__ u8 c_nonstat[512];      // states/nonstationary.cpp:3   [state*2+bit]
__constant__ u8 c_runmap[512];       // states/run-map.cpp:3-20      [state*2+bit]
__constant__ u8 c_ivmap[5][256];     // predictor.cpp:223-304 interval maps
__constant__ u8 c_mixer_sel[N_MIXERS];

// lane -> (kind, index) in models_ order
enum { K_BRACKET, K_DIRECT, K_DHASH, K_INDIRECT, K_MATCH, K_PPMD, K_NONE };

struct LaneRole { int kind, idx, ctx; };

__device__ __forceinline__ LaneRole lane_role(int lane) {
  // ctx: index into the per-byte context value table built by ctx_value()
  LaneRole r; r.kind = K_NONE; r.idx = 0; r.ctx = 0;
  if (lane == 0) { r.kind = K_BRACKET; }
  else if (lane == 1) { r.kind = K_DIRECT; r.idx = 0; r.ctx = 0; }           // bracket ctx
  else if (lane == 2) { r.kind = K_INDIRECT; r.idx = 0; r.ctx = 0; }
  else if (lane <= 20) { r.kind = K_INDIRECT; r.idx = lane - 2; r.ctx = 1 + (lane - 3); }   // sparse[0..17]
  else if (lane == 21) { r.kind = K_MATCH; r.idx = 0; r.ctx = 1 + 0; }
  else if (lane == 22) { r.kind = K_MATCH; r.idx = 1; r.ctx = 1 + 4; }
  else if (lane == 23) { r.kind = K_INDIRECT; r.idx = 19; r.ctx = 1 + 4; }
  else if (lane == 24) { r.kind = K_DHASH; r.idx = 0; r.ctx = 1 + 4; }
  else if (lane == 25) { r.kind = K_MATCH; r.idx = 2; r.ctx = 1 + 3; }
  else if (lane == 26) { r.kind = K_MATCH; r.idx = 3; r.ctx = 1 + 7; }
  else if (lane == 27) { r.kind = K_MATCH; r.idx = 4; r.ctx = 1 + 6; }
  else if (lane == 28) { r.kind = K_MATCH; r.idx = 5; r.ctx = 1 + 2; }
  else if (lane <= 31) { r.kind = K_DIRECT; r.idx = 1 + (lane - 29); r.ctx = 19 + (lane - 29); }   // chash[0..2]
  else if (lane == 32) { r.kind = K_DHASH; r.idx = 1; r.ctx = 19 + 3; }
  else if (lane <= 42) {                                                       // order matches
    const int k = lane - 33;                                                   // chash idx {0,1,2,4,..,10}
    r.kind = K_MATCH; r.idx = 6 + k; r.ctx = 19 + (k < 3 ? k : k + 1);
  }
  else if (lane <= 53) { r.kind = K_INDIRECT; r.idx = 20 + (lane - 43); r.ctx = 32 + (lane - 43); }   // ihash ctx
  else if (lane == 54) { r.kind = K_PPMD; }
  return r;
}

// context value table: [0] bracket, [1..18] sparse, [19..31] chash, [32..42] ihash
enum { CTXV_COUNT = 43 };

__device__ __forceinline__ int closing_bracket(u32 c, bool quotes) {
  switch (c) {
    case '(': return ')'; case '{': return '}'; case '[': return ']'; case '<': return '>';
    case '\'': return quotes ? '\'' : -1; case '"': return quotes ? '"' : -1;
  }
  return -1;
}

__device__ __forceinline__ float stretch(const Tables& T, float p) {     // mixer-input.cpp:11-15
  if (p < 1.0e-4f) p = 1.0e-4f; else if (p > 1 - 1.0e-4f) p = 1 - 1.0e-4f;
  int index = (int)XM_FMUL(p, 100001.0f);
  if (index >= 100001) index = 100000; else if (index < 0) index = 0;
  return T.logit[index];
}

struct SmallShared {
  u64 ctxv[CTXV_COUNT];
  u64 sel[S_COUNT];
  u64 ind_addr[64];
  float bracket_probs[256];
  float ppmd_probs[256];
  u32 bit_context;
  int byte_flag, max_rank;
  unsigned long long longest_match;
};

__device__ void small_refresh_tables(const SmallState& s, SmallShared& sh) {
  // single thread: gather context values + mixer selectors from the state
  sh.ctxv[0] = s.bracket_ctx;
  for (int i = 0; i < 18; ++i) sh.ctxv[1 + i] = s.sparse[i];
  for (int i = 0; i < 13; ++i) sh.ctxv[19 + i] = s.chash[i];
  for (int i = 0; i < 11; ++i) sh.ctxv[32 + i] = s.ihash[i].ctx;
  sh.sel[S_ZERO] = 0; sh.sel[S_LONGBIT] = s.long_bit_context;
  sh.sel[S_RB0] = s.recent_bytes[0]; sh.sel[S_RB1] = s.recent_bytes[1];
  sh.sel[S_RB2] = s.recent_bytes[2]; sh.sel[S_RB3] = s.recent_bytes[3];
  sh.sel[S_LINEBREAK] = s.line_break; sh.sel[S_LONGEST] = s.longest_match;
  sh.sel[S_WRT] = s.wrt_context; sh.sel[S_AUX] = 0;
  sh.sel[S_IV0] = s.interval[0]; sh.sel[S_IV1] = s.interval[1]; sh.sel[S_IV2] = s.interval[2];
  sh.sel[S_IV3] = s.interval[3]; sh.sel[S_IV4] = s.interval[4]; sh.sel[S_IV6] = s.interval[6];
  sh.sel[S_IVH] = s.ivh_ctx;
  for (int i = 0; i < 8; ++i) sh.sel[S_BC0 + i] = s.bitctx[i];
  sh.sel[S_COMB0] = s.combined[0]; sh.sel[S_COMB1] = s.combined[1];
  sh.bit_context = s.bit_context;
}

// ContextManager::UpdateContexts (context-manager.cpp:69-94) — single thread.
__device__ void contexts_update(SmallState& s, int bit) {
  s.bit_context += s.bit_context + bit;
  s.long_bit_context = s.bit_context;
  if (s.bit_context >= 256) {
    s.bit_context -= 256;
    s.long_bit_context = 1;
    s.longest_match = 0;
    const u32 c = s.bit_context;
    if (c == '\n') s.line_break = 0; else if (s.line_break < 99) ++s.line_break;
    s.history[s.history_pos] = (u8)c;                                  // UpdateHistory
    if (++s.history_pos == 100000000ull) s.history_pos = 0;
    {                                                                  // UpdateWords
      u8 w = (u8)c;
      if ((w >= 'a' && w <= 'z') || (w >= 'A' && w <= 'Z') || w >= 0x80) s.words[7] = s.words[7] * 997 * 16 + w;
      else s.words[7] = 0;
      if (w >= 'A' && w <= 'Z') w += 'a' - 'A';
      if ((w >= 'a' && w <= 'z') || (w >= '0' && w <= '9') || w == 8 || w == 6 || w >= 0x80) {
        s.words[0] = s.words[0] * 997 * 16 + w;
        s.words[0] &= 0xfffffff;
        s.words[1] = s.words[1] * 263 * 32 + w;
      } else {
        for (int i = 6; i >= 2; --i) s.words[i] = s.words[i - 1];
        s.words[1] = 0;
      }
    }
    for (int i = 7; i >= 1; --i) s.recent_bytes[i] = s.recent_bytes[i - 1];   // UpdateRecentBytes
    s.recent_bytes[0] = c;
    if (c < 0x80) {                                                    // UpdateWRTContext
      s.wrt_state = 0;
    } else {
      if (s.wrt_state == 0) s.wrt_context = 0;
      s.wrt_state = 1;
      s.wrt_context <<= 8;
      s.wrt_context += c;
      if (s.wrt_context > 0xFFEFCF) s.wrt_context = 0;
    }
    // BracketContext(256, 15): the stack is never trimmed (bracket-context.cpp:24 compares
    // the bracket MAP size, a constant 4, to the limit), so it lives in a growable HBM array.
    if (s.br_depth > 0) {
      const u32 top = s.br_depth - 1;
      if (closing_bracket(s.br_char[top], false) == (int)c || s.br_dist[top] >= 256 - 1) --s.br_depth;
      else ++s.br_dist[top];
    }
    if (closing_bracket(c, false) >= 0) {
      if (s.br_depth >= s.br_cap) { s.error |= 1u; }
      else { s.br_char[s.br_depth] = (u8)c; s.br_dist[s.br_depth] = 0; ++s.br_depth; }
    }
    s.bracket_ctx = s.br_depth == 0 ? 0 : 256ull * (s.br_char[s.br_depth - 1] + 1) + s.br_dist[s.br_depth - 1];
    // Sparse (sparse.cpp:17-22); word orders of predictor.cpp:104-108
    {
      const u64 f1 = 256, f2 = 29 * 31, f3 = 29 * 31 * 37, f4 = 29 * 31 * 37 * 41, f5 = 29u * 31 * 37 * 41 * 43;
      const u64* w = s.words;
      s.sparse[0] = w[0];
      s.sparse[1] = w[0] + f1 * w[1];
      s.sparse[2] = w[7] + f1 * w[2];
      s.sparse[3] = w[7];
      s.sparse[4] = w[1];
      s.sparse[5] = w[1] + f1 * w[2];
      s.sparse[6] = w[1] + f1 * w[2] + f2 * w[3];
      s.sparse[7] = w[1] + f1 * w[3];
      s.sparse[8] = w[1] + f1 * w[4];
      s.sparse[9] = w[1] + f1 * w[5];
      s.sparse[10] = w[2] + f1 * w[3];
      s.sparse[11] = w[3] + f1 * w[4];
      s.sparse[12] = w[1] + f1 * w[2] + f2 * w[4];
      s.sparse[13] = w[1] + f1 * w[2] + f2 * w[3] + f3 * w[4];
      s.sparse[14] = w[2] + f1 * w[3] + f2 * w[4];
      s.sparse[15] = w[2];
      s.sparse[16] = w[1] + f1 * w[2] + f2 * w[3] + f3 * w[4] + f4 * w[5];
      s.sparse[17] = w[1] + f1 * w[2] + f2 * w[3] + f3 * w[4] + f4 * w[5] + f5 * w[6];
    }
    // ContextHash (context-hash.cpp:9-11): (order,bits) list of state.h/SmallState::chash
    {
      const int ord[13] = {0, 1, 2, 3, 7, 11, 13, 15, 17, 20, 25, 2, 3};
      const int bits[13] = {8, 8, 8, 8, 4, 3, 2, 2, 2, 1, 1, 4, 2};
      for (int i = 0; i < 13; ++i) {
        const u64 size = 1ull << (bits[i] * ord[i]);
        s.chash[i] = (s.chash[i] * (u64)(1 << bits[i]) + c) % size;
      }
    }
    // Interval (interval.cpp:17-19) + IntervalHash (interval-hash.cpp:18-21)
    {
      const int map[8] = {0, 1, 2, 3, 3, 3, 4, 4}, nb[8] = {8, 8, 7, 10, 15, 7, 9, 7}, sh[8] = {4, 4, 1, 2, 2, 2, 3, 3};
      for (int i = 0; i < 8; ++i) {
        const u64 mask = (1ull << nb[i]) - 1;
        s.interval[i] = mask & ((s.interval[i] << sh[i]) + c_ivmap[map[i]][c]);
      }
      s.ivh_interval = 255 & ((s.ivh_interval << 3) + c_ivmap[4][c]);
      s.ivh_ctx = (s.ivh_ctx * 4 + s.ivh_interval) % 16384;
    }
    s.combined[0] = (s.recent_bytes[0] << 8) + s.recent_bytes[1];       // combined-context.cpp:13-15
    s.combined[1] = (s.recent_bytes[1] << 8) + s.recent_bytes[2];
  }
}

// IndirectHash::Update (indirect-hash.cpp:13-17), one lane per context.
__device__ __forceinline__ void ihash_update(IHashState& h, u32 c) {
  h.hashes[h.ctx1] = (h.ctx * (u64)(1 << h.h2) + c) % h.size;
  h.ctx1 = (h.ctx1 * (u64)(1 << h.h1) + c) % h.size1;
  h.ctx = h.hashes[h.ctx1];
}

__device__ __forceinline__ void bitcontexts_update(SmallState& s) {        // bit-context.cpp:11-13
  const u64 bc[8] = {s.chash[0], s.chash[1], s.chash[11], s.chash[12], s.interval[2],
                     s.interval[5], s.interval[7], s.recent_bytes[1]};
  for (int i = 0; i < 8; ++i) s.bitctx[i] = (bc[i] << 8) + s.long_bit_context;
}

// ---- per-model primitives ----
__device__ __forceinline__ float direct_predict(const DirectTable& d, u64 byte_ctx, u32 bit_ctx) {
  const u64 row = d.hashed ? d.index : byte_ctx;
  return d.pred[row * 256 + bit_ctx];
}
__device__ __forceinline__ void direct_perceive(DirectTable& d, u64 byte_ctx, u32 bit_ctx, int bit) {
  const u64 i = (d.hashed ? d.index : byte_ctx) * 256 + bit_ctx;
  float dv = d.divisor;
  u8 cnt = d.count[i];
  if (cnt < d.limit) {
    ++cnt; d.count[i] = cnt;
    dv = (float)(1.0 / ((double)(XM_FADD((float)cnt, d.delta))));    // 1.0 / (count + delta): int+float -> float, then double division
  }
  const float p = d.pred[i];
  d.pred[i] = XM_FADD(p, XM_FMUL(XM_FSUB((float)bit, p), dv));
}
__device__ void dhash_byte_update(DirectTable& d, u64 byte_ctx) {             // direct-hash.cpp:31-48
  u64 index = byte_ctx % d.rows;
  for (int i = 0; i < 20; ++i) {
    const u64 cs = d.checksum[index];
    if (cs == 0) { d.checksum[index] = byte_ctx; break; }
    if (cs == byte_ctx) break;
    if (i == 19) {
      for (int k = 0; k < 256; ++k) { d.pred[index * 256 + k] = 0.5f; d.count[index * 256 + k] = 0; }
      d.checksum[index] = byte_ctx;
      break;
    }
    if (++index == d.rows) index = 0;
  }
  d.index = index;
}

__device__ __forceinline__ float match_predict(const MatchState& m) {
  const float p = m.pred[m.match_length];
  return (m.cur_byte & m.bit_pos) ? p : XM_FSUB(1.0f, p);
}
__device__ __forceinline__ void match_perceive(MatchState& m, u64 byte_ctx, u32 bit_context, int bit) {
  const int match = (bit == ((m.cur_byte & m.bit_pos) != 0)) ? 1 : 0;
  m.bit_pos /= 2;
  float dv = m.divisor;
  const int len = m.match_length;
  if (m.count[len] < m.limit) {
    ++m.count[len];
    dv = (float)(1.0 / (double)XM_FADD((float)m.count[len], m.delta));
  }
  const float p = m.pred[len];
  m.pred[len] = XM_FADD(p, XM_FMUL(XM_FSUB((float)match, p), dv));
  if (match) { if (m.match_length < 255) ++m.match_length; } else m.match_length = 0;
  if (bit_context >= 128) {
    m.map[byte_ctx % m.map_size] = (u32)m.history_pos;
    ++m.history_pos;
  }
}
__device__ __forceinline__ void match_byte_update(MatchState& m, u64 byte_ctx, const u8* history,
                                                  unsigned long long* longest) {
  if (m.match_length < 8) m.cur_match = m.map[byte_ctx % m.map_size];
  else ++m.cur_match;
  m.cur_match %= 100000000ull;
  m.cur_byte = history[m.cur_match];
  m.bit_pos = 128;
  atomicMax(longest, (unsigned long long)(m.match_length / 32));
}

// Bracket::ByteUpdate (bracket.cpp:13-60), run by the whole 64-thread CTA (fill is parallel).
__device__ void bracket_byte_update(SmallState& s, float* probs, u32 byte, int tid, int nthreads,
                                    float* sh_p, int* sh_hot) {
  const u32 kDist = 200, kStack = 10, kStats = 100000;
  if (tid == 0) {
    float p = -1.0f; int hot = -1;      // p < 0: uniform 1/256
    const int close = closing_bracket(byte, true);
    u32 depth = s.bk_depth;
    if (depth == 0 || (close >= 0 && !(s.bk_active[depth - 1] == byte && (u32)close == byte))) {
      if (close >= 0) {
        s.bk_active[depth] = byte; s.bk_distance[depth] = 0; ++depth;
        if (depth > kStack) {
          for (u32 i = 1; i < depth; ++i) { s.bk_active[i - 1] = s.bk_active[i]; s.bk_distance[i - 1] = s.bk_distance[i]; }
          --depth;
        }
        p = (float)((1. * s.bk_first[byte * 200]) / s.bk_second[byte * 200]);
        hot = close;
      }
    } else {
      const u32 a = s.bk_active[depth - 1]; u32 d = s.bk_distance[depth - 1];
      const u32 idx = a * 200 + d;
      ++s.bk_second[idx];
      const int ca = closing_bracket(a, true);
      if (ca == (int)byte) ++s.bk_first[idx];
      if (s.bk_second[idx] > kStats) { s.bk_first[idx] /= 2; s.bk_second[idx] /= 2; }
      if (ca == (int)byte || d >= kDist - 1) {
        --depth;
        if (depth > 0) {
          const u32 a2 = s.bk_active[depth - 1], d2 = s.bk_distance[depth - 1];
          p = (float)((1. * s.bk_first[a2 * 200 + d2]) / s.bk_second[a2 * 200 + d2]);
          hot = closing_bracket(a2, true);
        }
      } else {
        ++s.bk_distance[depth - 1]; ++d;
        p = (float)((1. * s.bk_first[a * 200 + d]) / s.bk_second[a * 200 + d]);
        hot = ca;
      }
    }
    s.bk_depth = depth;
    *sh_p = p; *sh_hot = hot;
  }
  JIT_SYNCTHREADS();
  const float p = *sh_p; const int hot = *sh_hot;
  const float rest = p < 0.0f ? (float)(1. / 256) : XM_FDIV(XM_FSUB(1.0f, p), 255.0f);
  for (int i = tid; i < 256; i += nthreads) {
    float v = (i == hot) ? p : rest;
    if (!s.vocab[i]) v = 0.0f;                       // ByteModel::ByteUpdate (byte-model.cpp:39-45)
    probs[i] = v;
  }
  JIT_SYNCTHREADS();
}

// One bit of Predict() for the small models: writes 54 stretched inputs + PPMD input + selectors.
__device__ void small_predict(SmallState& s, const Tables& T, SmallShared& sh, float* out_x, u32* out_sel, int tid) {
  const LaneRole r = lane_role(tid);
  const u32 bc = sh.bit_context;
  float p = 0.5f; bool has = true;
  switch (r.kind) {
    case K_BRACKET: { int ex; p = bytemodel_predict(sh.bracket_probs, s.bracket_bm.bot, s.bracket_bm.top, &ex); s.bracket_bm.ex = ex; break; }
    case K_PPMD: { int ex; p = bytemodel_predict(sh.ppmd_probs, s.ppmd_bm.bot, s.ppmd_bm.top, &ex); s.ppmd_bm.ex = ex; break; }
    case K_DIRECT: p = direct_predict(r.idx == 0 ? s.direct_bracket : s.direct_o[r.idx - 1], sh.ctxv[r.ctx], bc); break;
    case K_DHASH: p = direct_predict(r.idx == 0 ? s.dhash_word : s.dhash_o3, 0, bc); break;
    case K_INDIRECT: {
      IndirectState& m = s.indirect[r.idx];
      m.map_index += bc;                                                    // indirect.cpp:17 (not idempotent)
      p = m.pred[s.shared_map[m.map_index]];
      break;
    }
    case K_MATCH: p = match_predict(s.match[r.idx]); break;
    default: has = false;
  }
  if (has) out_x[tid] = stretch(T, p);
  if (tid < N_MIXERS && out_sel) out_sel[tid] = (u32)sh.sel[c_mixer_sel[tid]];
}

// One bit of Perceive() for the small models, then contexts, then byte updates.
__device__ void small_perceive(SmallState& s, SmallShared& sh, int bit, const float* ppmd_next, int pretrain, int tid, int nthreads) {
  const LaneRole r = lane_role(tid);
  const u32 bc = sh.bit_context;
  // --- Model::Perceive ---
  u64 my_addr = ~0ull;
  switch (r.kind) {
    case K_BRACKET: { ByteModelState& b = s.bracket_bm; b.mid = b.bot + ((b.top - b.bot) / 2); if (bit) b.bot = b.mid + 1; else b.top = b.mid; break; }
    case K_PPMD: if (!pretrain) { ByteModelState& b = s.ppmd_bm; b.mid = b.bot + ((b.top - b.bot) / 2); if (bit) b.bot = b.mid + 1; else b.top = b.mid; } break;
    case K_DIRECT: direct_perceive(r.idx == 0 ? s.direct_bracket : s.direct_o[r.idx - 1], sh.ctxv[r.ctx], bc, bit); break;
    case K_DHASH: direct_perceive(r.idx == 0 ? s.dhash_word : s.dhash_o3, 0, bc, bit); break;
    case K_INDIRECT: my_addr = s.indirect[r.idx].map_index; break;
    case K_MATCH: match_perceive(s.match[r.idx], sh.ctxv[r.ctx], bc, bit); break;
    default: break;
  }
  // Indirect models share one nibble map and collide by design (indirect.cpp:10,30); the
  // reference updates them one after the other, so lanes that hit the SAME byte this bit
  // are serialised in model order.
  sh.ind_addr[tid] = my_addr;
  if (tid == 0) sh.max_rank = 0;
  JIT_SYNCTHREADS();
  int rank = 0;
  if (r.kind == K_INDIRECT) {
    for (int l = 0; l < tid; ++l) if (sh.ind_addr[l] == my_addr) ++rank;
    if (rank) atomicMax(&sh.max_rank, rank);
  }
  JIT_SYNCTHREADS();
  const int max_rank = sh.max_rank;
  for (int pass = 0; pass <= max_rank; ++pass) {
    if (r.kind == K_INDIRECT && rank == pass) {
      IndirectState& m = s.indirect[r.idx];
      const int state = s.shared_map[m.map_index];
      const float p = m.pred[state];
      m.pred[state] = XM_FADD(p, XM_FMUL(XM_FSUB((float)bit, p), m.divisor));
      s.shared_map[m.map_index] = m.run ? c_runmap[state * 2 + bit] : c_nonstat[state * 2 + bit];
      m.map_index -= bc;
    }
    if (max_rank) { __threadfence_block(); JIT_SYNCTHREADS(); }
  }
  JIT_SYNCTHREADS();
  // --- ContextManager::UpdateContexts ---
  const bool byte_update = bc >= 128;
  const u32 full = (bc * 2 + bit) & 255;          // the byte just completed (valid if byte_update)
  if (tid == 0) contexts_update(s, bit);
  if (byte_update && tid >= 32 && tid < 43) ihash_update(s.ihash[tid - 32], full);
  JIT_SYNCTHREADS();
  if (tid == 0) { bitcontexts_update(s); sh.longest_match = 0; }
  JIT_SYNCTHREADS();
  if (byte_update) {
    if (tid == 0) small_refresh_tables(s, sh);   // new byte-level context values for ByteUpdate()
    JIT_SYNCTHREADS();
    // --- Model::ByteUpdate (bit_context_ still holds the full byte, quirk 14) ---
    switch (r.kind) {
      case K_DHASH: dhash_byte_update(r.idx == 0 ? s.dhash_word : s.dhash_o3, sh.ctxv[r.ctx]); break;
      case K_INDIRECT: s.indirect[r.idx].map_index = (257 * sh.ctxv[r.ctx] + s.indirect[r.idx].map_offset) % (2048000000ull - 257); break;
      case K_MATCH: match_byte_update(s.match[r.idx], sh.ctxv[r.ctx], s.history, &sh.longest_match); break;
      default: break;
    }
    __shared__ float sh_p; __shared__ int sh_hot;
    bracket_byte_update(s, sh.bracket_probs, full, tid, nthreads, &sh_p, &sh_hot);
    // PPMD::ByteUpdate: distribution replayed (floor/vocab mask/normalisation already applied)
    if (!pretrain) for (int i = tid; i < 256; i += nthreads) {
      // no replayed PPMD stream: the slot carries a flat distribution over the vocabulary
      sh.ppmd_probs[i] = ppmd_next ? ppmd_next[i] : (s.vocab[i] ? (float)(1. / 256) : 0.0f);
    }
    JIT_SYNCTHREADS();
    if (tid == 0) {
      s.bracket_bm.top = 255; s.bracket_bm.bot = 0;
      if (!pretrain) { s.ppmd_bm.top = 255; s.ppmd_bm.bot = 0; }
      s.longest_match = sh.longest_match;
      s.bit_context = 1;                           // predictor.cpp:468
    }
    JIT_SYNCTHREADS();
  }
  if (tid == 0) small_refresh_tables(s, sh);
  JIT_SYNCTHREADS();
}

// Bulk kernel: all bits of a chunk (compress direction: the bits are known).
// The whole SmallState (68 KB: every model's adaptive tables, context registers and the POINTERS to
// the big HBM tables) lives in shared memory for the duration of the kernel: a state machine that
// chases `state->table_ptr` through HBM pays ~1 us per dependent load; out of shared memory it pays 30 ns.
__global__ void __launch_bounds__(64, 1)
small_kernel(const ChunkArgs* __restrict__ args_all, Tables T) { jit_entry(JK_SMALL);
  const ChunkArgs a = args_all[blockIdx.x];
  StreamState* st = a.st;
  extern __shared__ __align__(16) unsigned char small_raw[];
  SmallState& s = *reinterpret_cast<SmallState*>(small_raw);
  __shared__ SmallShared sh;
  const int tid = threadIdx.x;
  {
    const uint4* src = reinterpret_cast<const uint4*>(&st->small);
    uint4* dst = reinterpret_cast<uint4*>(small_raw);
    for (int i = tid; i < (int)(sizeof(SmallState) / 16); i += 64) dst[i] = src[i];
  }
  JIT_SYNCTHREADS();
  for (int i = tid; i < 256; i += 64) { sh.bracket_probs[i] = s.bracket_bm.probs[i]; sh.ppmd_probs[i] = s.ppmd_bm.probs[i]; }
  if (tid == 0) small_refresh_tables(s, sh);
  JIT_SYNCTHREADS();
  for (u32 pos = 0; pos < a.n_bytes; ++pos) {
    const u32 byte = a.bytes[pos];
    for (int j = 7; j >= 0; --j) {
      const u64 t = (u64)pos * 8 + (7 - j);
      const int bit = (byte >> j) & 1;
      small_predict(s, T, sh, a.pretrain ? st->small_x : a.small_x + t * SMALL_X_PITCH,
                    a.pretrain ? st->sel : a.sel + t * SEL_PITCH, tid);
      JIT_SYNCTHREADS();
      small_perceive(s, sh, bit, (j == 0 && a.ppmd) ? a.ppmd + (u64)pos * 256 : nullptr, (int)a.pretrain, tid, 64);
    }
  }
  for (int i = tid; i < 256; i += 64) { s.bracket_bm.probs[i] = sh.bracket_probs[i]; s.ppmd_bm.probs[i] = sh.ppmd_probs[i]; }
  JIT_SYNCTHREADS();
  {
    uint4* dst = reinterpret_cast<uint4*>(&st->small);
    const uint4* src = reinterpret_cast<const uint4*>(small_raw);
    for (int i = tid; i < (int)(sizeof(SmallState) / 16); i += 64) dst[i] = src[i];
  }
}

// Lock-step halves (Predictor::Predict / Perceive called bit by bit from the host).
__global__ void __launch_bounds__(64, 1) small_predict_kernel(StreamState* st, Tables T) { jit_entry(JK_SMALL_PREDICT);
  __shared__ SmallShared sh;
  SmallState& s = st->small;
  const int tid = threadIdx.x;
  for (int i = tid; i < 256; i += 64) { sh.bracket_probs[i] = s.bracket_bm.probs[i]; sh.ppmd_probs[i] = s.ppmd_bm.probs[i]; }
  if (tid == 0) small_refresh_tables(s, sh);
  JIT_SYNCTHREADS();
  small_predict(st->small, T, sh, st->small_x, st->sel, tid);
}
__global__ void __launch_bounds__(64, 1) small_perceive_kernel(StreamState* st, int bit, const float* ppmd_next, int pretrain, const u32* dbit = nullptr) { jit_entry(JK_SMALL_PERCEIVE);
  if (dbit) bit = (int)dbit[0];
  __shared__ SmallShared sh;
  SmallState& s = st->small;
  const int tid = threadIdx.x;
  for (int i = tid; i < 256; i += 64) { sh.bracket_probs[i] = s.bracket_bm.probs[i]; sh.ppmd_probs[i] = s.ppmd_bm.probs[i]; }
  if (tid == 0) small_refresh_tables(s, sh);
  JIT_SYNCTHREADS();
  small_perceive(st->small, sh, bit, ppmd_next, pretrain, tid, 64);
  for (int i = tid; i < 256; i += 64) { s.bracket_bm.probs[i] = sh.bracket_probs[i]; s.ppmd_bm.probs[i] = sh.ppmd_probs[i]; }
}

}  // namespace cmixb200
