// cmix_b200/csrc/paq8_predict.h — state and per-bit evaluation of the resident PAQ8 model (SURVEY §8 row a13).
//
// `bit(S, y)` is PAQ8::Perceive(y) (reference src/models/paq8.cpp:8380-8383): `Predictor::update` (:8248-8362) with
// `contextModel2` (:8101-8206) and every sub-model on its non-image path, in the reference's call order, writing the
// 1591 exported 12-bit codes into S.codes. Sub-models are separate functions over their own state blocks (`*_byte` =
// the bpos==0 part that derives contexts from the byte history, `*_bit` = the per-bit part that emits mixer inputs), so
// that the device kernel (paq8.cuh) can run them as independent units.
#ifndef CMIXB200_PAQ8_PREDICT_H
#define CMIXB200_PAQ8_PREDICT_H

#include "paq8_text.h"

namespace cmixb200 {
namespace p8 {

enum { ERR_UNSUPPORTED_BLOCK = 1, ERR_MIXER_ALIAS = 2 };

// ---------------------------------------------------------------- sub-model state blocks
struct MatchM {   // MatchModel (:3520-3693)
  u32* table; u32 mask; int hashbits;
  Sm32 sm[3]; Scm scm[3]; Stm maps[3]; ICtx<u8> ictx;
  u32 hashes[3], ctx[3], length, index; u8 expected, delta;
};
struct SparseMatchM {   // SparseMatchModel (:3694-3843)
  u32* table; u32 mask; int hashbits;
  Stm maps[4]; ICtx<u8> ictx8; ICtx<u16> ictx16;
  int root, it, prev[4], next[4];
  u32 hashes[4], hash_index, length, index; u8 expected, valid;
};
struct PicM { u32 r0, r1, r2, r3; u8* t; int cxt[3]; u16* sm_t; int sm_cxt[3]; };   // picModel (:3844-3864)
struct WordM {   // wordModel (:3872-4105)
  u64 word0, word1, word2, word3, word4, word5, xword0, xword1, xword2, cword0, ccword, number0, number1;
  u32 wrdhsh, text0, data0, type0, last_letter, first_letter, last_upper, last_digit, word_gap, mask, mask2;
  int nl1, nl, w, cword, pword, stem_index;
  int above, f_pending;  // handed from word_update to word_contexts / word_finish
  int* wpos;             // [0x10000]
  Word stem[4];
  Cm cm;
};
struct NestM { int ic, bc, pc, qc, lvc, ac, ec, uc, sense1, sense2, w; u32 vc, wc; Cm cm; };   // nestModel (:4107-4181)
struct RecordM {   // recordModel (:4204-4433)
  int cpos1[256], cpos2[256], cpos3[256], cpos4[256];
  int* wpos1;            // [0x10000]
  int rlen[3], rcount[2];
  u8 padding, N, NN, NNN, NNNN, WxNW, may_be_img24, db_version;
  int prev_transition, n_transition, col, mx_ctx, x;
  u32 db_nrecords; u16 db_record_len, db_header_len; int db_start, db_end;
  Cm cm, cn, co, cp;
  Stm maps[6]; Scm smap[3]; Imap imap[3]; ICtx<u16> ictx[5];
};
struct Record1M { int cpos1[256]; int* wpos1; Cm cm, cn, co, cp, cq; };   // recordModel1 (:4435-4474)
struct SparseM { Cm cm; };                                               // sparseModel (:4504-4536)
struct Sparse1M { Cm cm; Scm scm[7]; };                                  // sparseModel1 (:4539-4596): scm1..scm6, scma
struct DistanceM { Cm cm; int pos00, pos20, posnl; };                    // distanceModel (:4598-4612)
struct IndirectM { Cm cm; u32 t1[256]; u16* t2; u16* t3; u16* t4; ICtx<u32> ictx; };   // indirectModel (:7548-7612)
struct LinearM { Scm smap[5]; double* ols; int ols_km[3], ols_index[3]; u8 prd[5]; };  // linearPredictionModel (:4476-4502)
struct XmlTag { u32 name, length; int level; u8 end_tag, empty, pad[2]; u32 c_data, c_length, c_type; u32 a_name[4], a_value[4], a_length[4]; u32 a_index; };
struct XmlM {   // XMLModel (:7914-8097)
  Cm cm; XmlTag tags[32]; u32 index; u32 state_bh[8]; int state, pstate;
  u32 c8, ws_run, p_ws_run, indent_tab, indent_step, line_ending;
};
struct Instr { u32 data; u8 prefix, code, modrm, sib, rex, flags, bytes_read, size, category, must_check_rex, decoding, o16, imm8; };
struct ExeM {   // exeModel (:7273-7546)
  Cm2 cm; u32 cache[32]; u32 cache_index; u32 state_bh[256]; int pstate, state; Instr op;
  u32 total_ops, op_mask, op_categ_mask, context, brk_point, brk_ctx; int valid;
};
struct Sentence { Word first_word; u32 word_count, num_count; int type; u32 segment_count, verb_index, noun_index, capital_index; Word last_verb, last_noun, last_capital; };
struct Segment { Word first_word; u32 word_count, num_count; };
struct Paragraph { u32 sentence_count, type_count[3], type_mask; };
struct TextM {   // TextModel (:3070-3519)
  Cm2 map;
  Word words[4][8]; u32 words_index[4];
  Segment segments[4]; u32 seg_index;
  Sentence sentences[4]; u32 sen_index;
  Paragraph paragraphs[2]; u32 par_index;
  u32* word_pos;         // [0x10000]
  u32 byte_pos[256];
  int cw_lang, cw_slot, pw_lang, pw_slot;         // cWord / pWord as (language, cache slot)
  int state, pstate;
  u32 lang_count[3]; u64 lang_mask[3]; int lang_id, lang_pid;
  u64 numbers[2], num_hashes[2]; u8 num_length[2];
  u32 num_mask, num_diff, last_upper, mask_upper, last_letter, last_digit, last_punct, last_newline, prev_newline, word_gap, spaces,
      space_count, commas, quote_length, mask_punct, nest_hash, last_nest;
  u64 ascii_mask;
  u32 masks[5], word_length[2];
  int utf8_remaining;
  u8 first_letter, first_char, expected_digit, prev_punct;
  u8 stem_ok[3], stem_split;   // verdicts of the three stemmers; the language list whose current word IS cWord (0: none)
  Word topic;
  u64 parse_ctx;
};
struct DetectM {   // the header detectors in front of the image / audio / JPEG models (:5386-5509, :5810-5870, :6031-6060)
  int bmp_header, bmp_offset, bmp_hdrless, bmp_bitmask, tga_header, tga_id, tga_map, tga_bpp, tga_type, tga_w, tga_h, eoi, w;
  u32 wav_header, wav_channels, wav_bits, wav_chunk;   // audioModel's WAVAudio (:5806-5808)
  u32 wav_length, wav_eoi, wav_info;                   // and its statics `length`, `eoi`, `info` (:5811)
};

struct State {
  const Tables* T;
  // Predictor / globals (:167-200, :3866-3872, :4538, :8099, :8249)
  int y, c0, bpos, blpos, pos, pr, last_prediction;
  u32 c4, b2, b3, w4, w5, f4, tt, col, x4, x5;
  u32 frstchar, spafdo, spaces, spacecount, words, wordcount, wordlen, wordlen1;
  u8 grp0, pad0[3];
  u8* buf;               // 1 GiB ring (MEM()*8, :8368)
  Rnd rnd;
  // ModelStats (:204-227)
  int st_type; u64 st_misses; u32 st_match_length; u8 st_match_expected, st_text_first, st_text_mask, pad1; u32 st_xml, st_x86, st_record;
  // contextModel2 (:8102-8114)
  Cm2 cm; Rcm rcm7, rcm9, rcm10; Sm32 sm0, sm1;
  u32 cxt[16]; int ft2, filetype, size, info;
  // sub-models
  MatchM match; SparseMatchM smatch; SparseM sparse; Sparse1M sparse1; DistanceM distance; PicM pic; RecordM record; Record1M record1;
  WordM word; NestM nest; IndirectM indirect; Dmc dmc[10]; XmlM xml; TextM text; ExeM exe; LinearM linear; DetectM detect;
  // mixer and SSE stage
  Mixer m;
  Sm32 text_apm[4]; Apm1 text_apm1[3]; Apm1 generic_apm1[7];
  // outputs
  u16 codes[N_OUT + 1];
  u32 error;
};

P8_HD inline int buf(const State& S, int i) { return S.buf[(u32)(S.pos - i) & P8_BUF_MASK]; }
P8_HD inline int bufa(const State& S, u32 i) { return S.buf[i & P8_BUF_MASK]; }
P8_HD inline u64 sx(int v) { return (u64)(i64)v; }   // an int passed where the reference's hash() takes U64: sign extension
P8_HD inline bool is_alpha(int c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
P8_HD inline bool is_punct(int c) { return (c >= 33 && c <= 47) || (c >= 58 && c <= 64) || (c >= 91 && c <= 96) || (c >= 123 && c <= 126); }
P8_HD inline bool is_space(int c) { return (c >= 9 && c <= 13) || c == 32; }
P8_HD inline int clip8(int v) { return imin(0xFF, imax(0, v)); }

// mixer selector (Mixer::set, :570-573)
P8_HD inline void mset(Mixer& m, int cx, int range) { m.cxt[m.ncxt++] = m.base + cx; m.base += range; }

// ---------------------------------------------------------------- match model (:3520-3693)
// match_core: bookkeeping, contexts and the two length inputs; match_unit j = 0..8: the three StateMaps, the three stationary
// maps and the three StationaryMaps behind them (independent of each other: a lane each on the device)
P8_HD inline void match_core(State& S, Out& o) {
  const Tables& T = *S.T;
  MatchM& M = S.match;
  const int y = S.y, bpos = S.bpos, c0 = S.c0;
  if (bpos == 0) {
    M.delta = 0;
    for (u32 i = 0, min_len = 5 + 2 * 2; i < 3; ++i, min_len -= 2) {
      u64 h = 0;
      for (u32 j = min_len; j > 0; --j) h = combine64(h, (u64)buf(S, (int)j));
      M.hashes[i] = finalize64(h, M.hashbits);
    }
    if (M.length) { M.index++; if (M.length < 0xFFFF) M.length++; }
    else {
      u32 min_len = 9, best_len = 0, best_index = 0;
      for (u32 i = 0; i < 3 && M.length < min_len; ++i, min_len -= 2) {
        M.index = M.table[M.hashes[i]];
        if (M.index > 0) {
          M.length = 0;
          while (M.length < min_len && buf(S, (int)M.length + 1) == bufa(S, M.index - M.length - 1)) M.length++;
          if (M.length > best_len) { best_len = M.length; best_index = M.index; }
        }
      }
      if (best_len >= 5) { M.length = best_len - 4; M.index = best_index; }
      else M.length = M.index = 0;
    }
    for (u32 i = 0; i < 3; ++i) M.table[M.hashes[i]] = (u32)S.pos;
    M.expected = (u8)bufa(S, M.index);
    ictx_push(M.ictx, (u32)y); ictx_select(M.ictx, ((u32)buf(S, 1) << 8) | M.expected);
    scm_set(M.scm[0], M.expected);
    scm_set(M.scm[1], M.expected);
    scm_set(M.scm[2], (u32)S.pos);
    stm_set_direct(M.maps[0], ((u32)M.expected << 8) | (u32)buf(S, 1));
    stm_set(M.maps[1], hash(M.expected, (u64)c0, (u64)buf(S, 1), (u64)buf(S, 2), (u64)imin(3, (int)ilog2(M.length + 1))));
    stm_set_direct(M.maps[2], ictx_get(M.ictx));
    S.st_match_expected = M.length > 0 ? M.expected : 0;
  } else {
    const u8 B = (u8)(c0 << (8 - bpos));
    scm_set(M.scm[1], ((u32)bpos << 8) | (u32)(M.expected ^ B));
    stm_set(M.maps[1], hash(M.expected, (u64)c0, (u64)buf(S, 1), (u64)buf(S, 2), (u64)imin(3, (int)ilog2(M.length + 1))));
    ictx_push(M.ictx, (u32)y); ictx_select(M.ictx, ((u32)bpos << 16) | ((u32)buf(S, 1) << 8) | (u32)(M.expected ^ B));
    stm_set_direct(M.maps[2], ictx_get(M.ictx));
  }
  const int ebit = (M.expected >> (7 - bpos)) & 1;
  if (M.length > 0) {
    const bool ok = bpos == 0 ? (buf(S, 1) == bufa(S, M.index - 1)) : (((M.expected + 256) >> (8 - bpos)) == c0);
    if (!ok) { M.delta = (M.length + 5) > 5; M.length = 0; }
  }
  M.ctx[0] = M.ctx[1] = M.ctx[2] = 0;
  if (M.length > 0) {
    if (M.length <= 16) M.ctx[0] = (M.length - 1) * 2 + (u32)ebit;
    else M.ctx[0] = 24 + (umin(M.length - 1, 63) >> 2) * 2 + (u32)ebit;
    M.ctx[0] = (M.ctx[0] << 8) | (u32)c0;
    M.ctx[1] = (((u32)M.expected << 11) | ((u32)bpos << 8) | (u32)buf(S, 1)) + 1;
    const int sign = 2 * ebit - 1;
    add(o, sign * (imin((int)M.length, 32) << 5));
    add(o, sign * (ilog(T, M.length) << 2));
  } else { add(o, 0); add(o, 0); }
  if (M.delta) M.ctx[2] = ((u32)M.expected << 8) | (u32)c0;
  S.st_match_length = M.length;
}
P8_HD inline void match_unit(State& S, Out& o, int j) {   // o: at the model's first input
  const Tables& T = *S.T;
  MatchM& M = S.match;
  const int y = S.y;
  if (j < 3) {
    o.n += 2 + j;
    const u32 c = M.ctx[j];
    const int p = sm32_p(T, M.sm[j], y, (int)c);
    if (c != 0) add(o, (stretch(T, p) + 1) >> 1); else add(o, 0);
  } else if (j < 6) {
    o.n += 5 + 2 * (j - 3);
    scm_mix(M.scm[j - 3], o, y, 10 - j);
  } else {
    o.n += 11 + 2 * (j - 6);
    stm_mix(M.maps[j - 6], o, y, 1, 4, j == 6 ? 255 : 1023);
  }
}
P8_HD inline void match_bit(State& S, Out& o) {
  const Out b = o;
  match_core(S, o);
  for (int j = 0; j < 9; ++j) { Out u = b; match_unit(S, u, j); }
  o.n = b.n + 17;
}

// ---------------------------------------------------------------- sparse match model (:3694-3843)
// smatch_head: bookkeeping and the three length inputs (or eleven zeros); smatch_unit j = 0..3: the StationaryMaps
P8_HD inline void smatch_head(State& S, Out& o) {
  SparseMatchM& M = S.smatch;
  const u32 offset_[4] = {0, 1, 0, 0}, stride_[4] = {1, 1, 2, 1}, minlen_[4] = {5, 4, 4, 5}, bitmask_[4] = {0xDF, 0xFF, 0xDF, 0x0F};
  const int y = S.y, bpos = S.bpos, c0 = S.c0;
  const u8 B = (u8)(c0 << (8 - bpos));
  if (bpos == 0) {
    for (u32 i = 0; i < 4; ++i) {
      u64 h = 0;
      for (u32 j = 0, k = offset_[i] + 1; j < minlen_[i]; ++j, k += stride_[i]) h = combine64(h, (u64)((u32)buf(S, (int)k) & bitmask_[i]));
      M.hashes[i] = finalize64(h, M.hashbits);
    }
    if (M.length) { M.index++; if (M.length < 0xFFFF) M.length++; }
    else {
      for (int i = (M.it = M.root); i >= 0; i = (M.it >= 0 ? (M.it = M.next[M.it]) : M.it)) {
        M.index = M.table[M.hashes[i]];
        if (M.index > 0) {
          u32 off = offset_[i] + 1;
          while (M.length < minlen_[i] && ((((u32)buf(S, (int)off) ^ (u32)bufa(S, M.index - off)) & bitmask_[i]) == 0)) { M.length++; off += stride_[i]; }
          if (M.length >= minlen_[i]) {
            M.length -= (minlen_[i] - 1);
            M.hash_index = (u32)i;
            if ((M.it = i) != M.root) {   // MTFList::MoveToFront (:1516-1526)
              const int p = M.prev[i], n = M.next[i];
              if (p >= 0) M.next[p] = M.next[i];
              if (n >= 0) M.prev[n] = M.prev[i];
              M.prev[M.root] = i;
              M.next[i] = M.root;
              M.root = i;
              M.prev[M.root] = -1;
            }
            break;
          }
        }
        M.length = M.index = 0;
      }
    }
    for (u32 i = 0; i < 4; ++i) M.table[M.hashes[i]] = (u32)S.pos;
    M.expected = (u8)bufa(S, M.index);
    if (M.valid) { ictx_push(M.ictx8, (u32)y); ictx_push(M.ictx16, (u32)buf(S, 1)); }
    M.valid = M.length > 1;
    if (M.valid) {
      stm_set(M.maps[0], hash(M.expected, (u64)c0, (u64)buf(S, 1), (u64)buf(S, 2), (u64)(ilog2(M.length + 1) * 4 + M.hash_index)));
      stm_set_direct(M.maps[1], ((u32)M.expected << 8) | (u32)buf(S, 1));
      ictx_select(M.ictx8, ((u32)buf(S, 1) << 8) | M.expected); ictx_select(M.ictx16, ((u32)buf(S, 1) << 8) | M.expected);
      stm_set_direct(M.maps[2], ictx_get(M.ictx8));
      stm_set_direct(M.maps[3], ictx_get(M.ictx16));
    }
  } else if (M.valid) {
    stm_set(M.maps[0], hash(M.expected, (u64)c0, (u64)buf(S, 1), (u64)buf(S, 2), (u64)(ilog2(M.length + 1) * 4 + M.hash_index)));
    if (bpos == 4) stm_set_direct(M.maps[1], 0x10000u | ((u32)(M.expected ^ (u8)(c0 << 4)) << 8) | (u32)buf(S, 1));
    ictx_push(M.ictx8, (u32)y); ictx_select(M.ictx8, ((u32)bpos << 16) | ((u32)buf(S, 1) << 8) | (u32)(M.expected ^ B));
    stm_set_direct(M.maps[2], ictx_get(M.ictx8));
    stm_set_direct(M.maps[3], ((u32)bpos << 16) | ((u32)ictx_get(M.ictx16) ^ (u32)(B | (B << 8))));
  }
  if (M.length > 0 && ((((u32)(M.expected ^ B)) & bitmask_[M.hash_index]) >> (8 - bpos)) != 0) M.length = 0;
  if (M.valid) {
    if (M.length > 1 && ((bitmask_[M.hash_index] >> (7 - bpos)) & 1) > 0) {
      const int ebit = (M.expected >> (7 - bpos)) & 1, sign = 2 * ebit - 1;
      add(o, sign * (imin((int)M.length - 1, 64) << 4));
      add(o, sign * (1 << imin((int)M.length - 2, 3)) * imin((int)M.length - 1, 8) << 4);
      add(o, sign * 512);
    } else { add(o, 0); add(o, 0); add(o, 0); }
  } else for (int i = 0; i < 11; ++i) add(o, 0);
}
P8_HD inline void smatch_unit(State& S, Out& o, int j) {   // o: at the model's first input
  if (!S.smatch.valid) return;
  o.n += 3 + 2 * j;
  stm_mix(S.smatch.maps[j], o, S.y, 1, 2);
}
P8_HD inline void smatch_core(State& S, Out& o) {
  const Out b = o;
  smatch_head(S, o);
  for (int j = 0; j < 4; ++j) { Out u = b; smatch_unit(S, u, j); }
  o.n = b.n + 11;
}
P8_HD inline void smatch_select(State& S) {   // the model's two mixer selector sets (:3839-3840)
  const SparseMatchM& M = S.smatch;
  const int bpos = S.bpos, c0 = S.c0;
  mset(S.m, (int)((M.hash_index << 6) | ((u32)bpos << 3) | umin(7, M.length)), 4 * 64);
  mset(S.m, (int)((M.hash_index << 11) | (umin(7, ilog2(M.length + 1)) << 8) | (u32)(c0 ^ (M.expected >> (8 - bpos)))), 4 * 2048);
}

// ---------------------------------------------------------------- sparse / distance / pic models
P8_COLD P8_HD inline void sparse_byte(State& S, int seenbefore, int howmany) {   // :4504-4535
  Cm& cm = S.sparse.cm;
  const u32 c4 = S.c4, f4 = S.f4;
  u64 i = 0;
  cm_set(cm, hash(++i, sx(seenbefore)));
  cm_set(cm, hash(++i, sx(howmany)));
  cm_set(cm, hash(++i, (u64)(buf(S, 1) | buf(S, 5) << 8)));
  cm_set(cm, hash(++i, (u64)(buf(S, 1) | buf(S, 6) << 8)));
  cm_set(cm, hash(++i, (u64)(buf(S, 3) | buf(S, 6) << 8)));
  cm_set(cm, hash(++i, (u64)(buf(S, 4) | buf(S, 8) << 8)));
  cm_set(cm, hash(++i, (u64)(buf(S, 1) | buf(S, 3) << 8 | buf(S, 5) << 16)));
  cm_set(cm, hash(++i, (u64)(buf(S, 2) | buf(S, 4) << 8 | buf(S, 6) << 16)));
  cm_set(cm, hash(++i, c4 & 0x00f0f0ff));
  cm_set(cm, hash(++i, c4 & 0x00ff00ff));
  cm_set(cm, hash(++i, c4 & 0xff0000ff));
  cm_set(cm, hash(++i, c4 & 0x00f8f8f8));
  cm_set(cm, hash(++i, c4 & 0xf8f8f8f8));
  cm_set(cm, hash(++i, f4 & 0x00000fff));
  cm_set(cm, hash(++i, f4));
  cm_set(cm, hash(++i, c4 & 0x00e0e0e0));
  cm_set(cm, hash(++i, c4 & 0xe0e0e0e0));
  cm_set(cm, hash(++i, c4 & 0x810000c1));
  cm_set(cm, hash(++i, c4 & 0xC3CCC38C));
  cm_set(cm, hash(++i, c4 & 0x0081CC81));
  cm_set(cm, hash(++i, c4 & 0x00c10081));
  for (int j = 1; j < 8; ++j) {
    cm_set(cm, hash(++i, sx(seenbefore | buf(S, j) << 8)));
    cm_set(cm, hash(++i, (u64)((buf(S, j + 2) << 8) | buf(S, j + 1))));
    cm_set(cm, hash(++i, (u64)((buf(S, j + 3) << 8) | buf(S, j + 1))));
  }
}
// sparseModel1 runs BEFORE wordModel in the reference: it reads the word statistics of the previous byte. The caller passes them,
// so that a device lane can run this beside the word model's state update.
struct WordStats { u32 spaces, words, frstchar, spafdo; };
P8_HD inline WordStats word_stats(const State& S) { WordStats w; w.spaces = S.spaces; w.words = S.words; w.frstchar = S.frstchar; w.spafdo = S.spafdo; return w; }
P8_COLD P8_HD inline void sparse1_byte(State& S, int seenbefore, int howmany, const WordStats& W) {   // :4539-4586
  Sparse1M& M = S.sparse1;
  Cm& cm = M.cm;
  const u32 c4 = S.c4;
  scm_set(M.scm[4], (u32)seenbefore);
  scm_set(M.scm[5], (u32)howmany);
  u32 h = S.x4 << 6;
  cm_set(cm, (u64)((u32)buf(S, 1) + (h & 0xffffff00)));
  cm_set(cm, (u64)((u32)buf(S, 1) + (h & 0x00ffff00)));
  cm_set(cm, (u64)((u32)buf(S, 1) + (h & 0x0000ff00)));
  u32 d = c4 & 0xffff;
  h <<= 6;
  cm_set(cm, (u64)(d + (h & 0xffff0000)));
  cm_set(cm, (u64)(d + (h & 0x00ff0000)));
  h <<= 6; d = c4 & 0xffffff;
  cm_set(cm, (u64)(d + (h & 0xff000000)));
  for (int i = 1; i < 5; ++i) {
    cm_set(cm, sx(seenbefore | buf(S, i) << 8));
    cm_set(cm, (u64)((buf(S, i + 3) << 8) | buf(S, i + 1)));
  }
  cm_set(cm, W.spaces & 0x7fff);
  cm_set(cm, W.spaces & 0xff);
  cm_set(cm, W.words & 0x1ffff);
  cm_set(cm, S.f4 & 0x000fffff);
  cm_set(cm, S.tt & 0x00000fff);
  h = S.w4 << 6;
  cm_set(cm, (u64)((u32)buf(S, 1) + (h & 0xffffff00)));
  cm_set(cm, (u64)((u32)buf(S, 1) + (h & 0x00ffff00)));
  cm_set(cm, (u64)((u32)buf(S, 1) + (h & 0x0000ff00)));
  d = c4 & 0xffff;
  h <<= 6;
  cm_set(cm, (u64)(d + (h & 0xffff0000)));
  cm_set(cm, (u64)(d + (h & 0x00ff0000)));
  h <<= 6; d = c4 & 0xffffff;
  cm_set(cm, (u64)(d + (h & 0xff000000)));
  cm_set(cm, S.w4 & 0xf0f0f0ff);
  cm_set(cm, (u64)((S.w4 & 63) * 128 + (5 << 17)));
  cm_set(cm, (u64)((S.f4 & 0xffff) << 11 | W.frstchar));
  cm_set(cm, (u64)(W.spafdo * 8 * ((S.w4 & 3) == 1)));
  scm_set(M.scm[0], W.words & 127);
  scm_set(M.scm[1], (W.words & 12) * 16 + (S.w4 & 12) * 4 + ((u32)buf(S, 1) >> 4));
  scm_set(M.scm[2], S.w4 & 15);
  scm_set(M.scm[3], W.spafdo * ((S.w4 & 3) == 1));
  scm_set(M.scm[6], W.frstchar);
}
P8_COLD P8_HD inline void distance_byte(State& S) {   // :4598-4611
  DistanceM& M = S.distance;
  const int c = (int)(S.c4 & 0xff);
  if (c == 0x00) M.pos00 = S.pos;
  if (c == 0x20) M.pos20 = S.pos;
  if (c == 0xff || c == '\r' || c == '\n') M.posnl = S.pos;
  u64 i = 0;
  cm_set(M.cm, hash(++i, sx(imin(S.pos - M.pos00, 255) | c << 8)));
  cm_set(M.cm, hash(++i, sx(imin(S.pos - M.pos20, 255) | c << 8)));
  cm_set(M.cm, hash(++i, sx(imin(S.pos - M.posnl, 255) | c << 8)));
}
P8_HD inline void pic_core(State& S) {   // :3844-3858: bit-history updates and the three contexts
  const Tables& T = *S.T;
  PicM& M = S.pic;
  const int y = S.y, bpos = S.bpos;
  for (int i = 0; i < 3; ++i) M.t[M.cxt[i]] = T.state[M.t[M.cxt[i]]][y];
  M.r0 += M.r0 + (u32)y;
  M.r1 += M.r1 + (u32)((buf(S, 215) >> (7 - bpos)) & 1);
  M.r2 += M.r2 + (u32)((buf(S, 431) >> (7 - bpos)) & 1);
  M.r3 += M.r3 + (u32)((buf(S, 647) >> (7 - bpos)) & 1);
  M.cxt[0] = (int)((M.r0 & 0x7) | ((M.r1 >> 4) & 0x38) | ((M.r2 >> 3) & 0xc0));
  M.cxt[1] = (int)(0x100 + ((M.r0 & 1) | ((M.r1 >> 4) & 0x3e) | ((M.r2 >> 2) & 0x40) | ((M.r3 >> 1) & 0x80)));
  M.cxt[2] = (int)(0x200 + ((M.r0 & 0x3f) ^ (M.r1 & 0x3ffe) ^ ((M.r2 << 2) & 0x7f00) ^ ((M.r3 << 5) & 0xf800)));
}
P8_HD inline void pic_unit(State& S, Out& o, int i) {   // :3859-3863, o: at the model's first input
  const Tables& T = *S.T;
  PicM& M = S.pic;
  o.n += i;
  Sm16 s; s.t = M.sm_t + i * 256; s.cxt = M.sm_cxt[i];
  add(o, stretch(T, sm16_p(s, S.y, M.t[M.cxt[i]])));
  M.sm_cxt[i] = s.cxt;
}
P8_HD inline void pic_bit(State& S, Out& o) {
  pic_core(S);
  for (int i = 0; i < 3; ++i) { Out u = o; pic_unit(S, u, i); }
  o.n += 3;
}

// ---------------------------------------------------------------- record models (:4204-4474)
P8_COLD P8_HD inline void record_byte(State& S) {
  const Tables& T = *S.T;
  RecordM& M = S.record;
  const u32 c4 = S.c4;
  const int w = (int)(c4 & 0xffff), c = w & 255, d = w >> 8, pos = S.pos, blpos = S.blpos;
  if (S.st_record && (S.st_record >> 16) != (u32)M.rlen[0]) { M.rlen[0] = (int)(S.st_record >> 16); M.rcount[0] = M.rcount[1] = 0; }
  else {
    if (blpos == 0 || (M.db_version > 0 && blpos >= M.db_end)) M.db_version = 0;
    else if (M.db_version == 0 && (S.filetype == FT_DEFAULT || S.filetype == FT_TEXT) && blpos >= 31) {
      u8 b = (u8)buf(S, 32);
      bool ok = ((b & 7) == 3 || (b & 7) == 4 || (b >> 4) == 3 || b == 0xF5);
      if (ok) { b = (u8)buf(S, 30); ok = b > 0 && b < 13; }
      if (ok) { b = (u8)buf(S, 29); ok = b > 0 && b < 32; }
      if (ok) { M.db_nrecords = (u32)(buf(S, 28) | (buf(S, 27) << 8) | (buf(S, 26) << 16) | (buf(S, 25) << 24)); ok = M.db_nrecords > 0 && M.db_nrecords < 0xFFFFF; }
      if (ok) {
        M.db_header_len = (u16)(buf(S, 24) | (buf(S, 23) << 8));
        ok = M.db_header_len > 32;
        if (ok) {
          if (((M.db_header_len - 32 - 1) % 32) == 0) ok = true;
          else if (M.db_header_len > 255 + 8) { M.db_header_len = (u16)(M.db_header_len - (255 + 8)); ok = ((M.db_header_len - 32 - 1) % 32) == 0; }
          else ok = false;
        }
      }
      if (ok) { M.db_record_len = (u16)(buf(S, 22) | (buf(S, 21) << 8)); ok = M.db_record_len > 8; }
      if (ok) ok = buf(S, 20) == 0 && buf(S, 19) == 0 && buf(S, 17) <= 1 && buf(S, 16) <= 1;
      if (ok) {
        b = (u8)buf(S, 32);
        M.db_version = (u8)(((b >> 4) == 3) ? 3 : b & 7);
        M.db_start = blpos - 32 + M.db_header_len;
        M.db_end = M.db_start + (int)(M.db_nrecords * M.db_record_len);
        if (M.db_version == 3) { M.rlen[0] = 32; M.rcount[0] = M.rcount[1] = 0; }
      }
    } else if (M.db_version > 0 && blpos == M.db_start) { M.rlen[0] = M.db_record_len; M.rcount[0] = M.rcount[1] = 0; }
    const int r = pos - M.cpos1[c];
    if (r > 1 && r == M.cpos1[c] - M.cpos2[c] && r == M.cpos2[c] - M.cpos3[c] && (r > 32 || r == M.cpos3[c] - M.cpos4[c]) &&
        (r > 10 || ((c == buf(S, r * 5 + 1)) && c == buf(S, r * 6 + 1)))) {
      if (r == M.rlen[1]) ++M.rcount[0];
      else if (r == M.rlen[2]) ++M.rcount[1];
      else if (M.rcount[0] > M.rcount[1]) { M.rlen[2] = r; M.rcount[1] = 1; }
      else { M.rlen[1] = r; M.rcount[0] = 1; }
    }
    for (int i = 0; i < 2; ++i) {
      if (M.rcount[i] > imax(0, 12 - (int)ilog2((u32)M.rlen[i + 1]))) {
        if (M.rlen[0] != M.rlen[i + 1]) {
          if (M.may_be_img24 && M.rlen[i + 1] == 3) { M.rcount[0] >>= 1; M.rcount[1] >>= 1; continue; }
          else if ((M.rlen[i + 1] > M.rlen[0]) && (M.rlen[i + 1] % M.rlen[0] == 0)) {
            if ((M.rlen[0] > 32) && (M.rlen[i + 1] == M.rlen[0] * 2)) { M.rcount[0] >>= 1; M.rcount[1] >>= 1; continue; }
          }
          M.rlen[0] = M.rlen[i + 1];
          M.rcount[i] = 0;
          M.may_be_img24 = (M.rlen[0] > 30 && (M.rlen[0] % 3) == 0);
          M.n_transition = 0;
        } else M.rcount[i] >>= 2;
        if (M.rlen[i + 1] << 4 > M.rlen[1 + (i ^ 1)]) M.rcount[i ^ 1] = 0;
      }
    }
  }
  const int rl = M.rlen[0];
  M.col = pos % rl;
  M.x = imin(0x1F, M.col / imax(1, rl / 32));
  M.N = (u8)buf(S, rl); M.NN = (u8)buf(S, rl * 2); M.NNN = (u8)buf(S, rl * 3); M.NNNN = (u8)buf(S, rl * 4);
  for (int i = 0; i < 4; ++i) ictx_push(M.ictx[i], (u32)c);
  ictx_select(M.ictx[0], ((u32)c << 8) | M.N);
  ictx_select(M.ictx[1], ((u32)buf(S, rl - 1) << 8) | M.N);
  ictx_select(M.ictx[2], ((u32)c << 8) | (u32)buf(S, rl - 1));
  ictx_select(M.ictx[3], finalize64(hash((u64)c, M.N, (u64)buf(S, rl + 1)), 20));
  if (!M.col) M.n_transition = 0;
  if ((((c4 >> 8) == 0x20u * 0x010101u) && (c != 0x20)) || (!(c4 >> 8) && c && ((M.padding != 0x20) || (pos - M.prev_transition > rl)))) {
    M.prev_transition = pos;
    M.n_transition += (M.n_transition < 31);
    M.padding = (u8)d;
  }
  const int N = M.N, NN = M.NN, NNN = M.NNN, NNNN = M.NNNN, col = M.col;
  u64 i = 0;
  cm_set(M.cm, hash(++i, sx(c << 8 | (imin(255, pos - M.cpos1[c]) >> 2))));
  cm_set(M.cm, hash(++i, sx(w << 9 | llog(T, (u32)(pos - M.wpos1[w])) >> 2)));
  cm_set(M.cm, hash(++i, sx(rl | N << 10 | NN << 18)));
  cm_set(M.cn, hash(++i, sx(w | rl << 16)));
  cm_set(M.cn, hash(++i, sx(d | rl << 8)));
  cm_set(M.cn, hash(++i, sx(c | rl << 8)));
  cm_set(M.co, hash(++i, sx(c << 8 | imin(255, pos - M.cpos1[c]))));
  cm_set(M.co, hash(++i, sx(c << 17 | d << 9 | llog(T, (u32)(pos - M.wpos1[w])) >> 2)));
  cm_set(M.co, hash(++i, sx(c << 8 | N)));
  cm_set(M.cp, hash(++i, sx(rl | N << 10 | col << 18)));
  cm_set(M.cp, hash(++i, sx(rl | c << 10 | col << 18)));
  cm_set(M.cp, hash(++i, sx(col | rl << 12)));
  if (rl > 8) {
    cm_set(M.cp, hash(++i, sx(imin(imin(0xFF, rl), pos - M.prev_transition)), sx(imin(0x3FF, col)), sx((w & 0xF0F0) | (w == ((M.padding << 8) | M.padding))), sx(M.n_transition)));
    cm_set(M.cp, hash(++i, sx(w), (u64)(buf(S, rl + 1) == M.padding && N == M.padding), sx(col / imax(1, rl / 32))));
  } else { cm_set(M.cp, 0); cm_set(M.cp, 0); }
  cm_set(M.cp, hash(++i, sx(N | ((NN & 0xF0) << 4) | ((NNN & 0xE0) << 7) | ((NNNN & 0xE0) << 10) | ((col / imax(1, rl / 16)) << 18))));
  cm_set(M.cp, hash(++i, sx((N & 0xF8) | ((NN & 0xF8) << 8) | (col << 16))));
  cm_set(M.cp, hash(++i, (u64)N, (u64)NN));
  cm_set(M.cp, hash(++i, sx(col), ictx_get(M.ictx[0])));
  cm_set(M.cp, hash(++i, sx(col), ictx_get(M.ictx[1])));
  cm_set(M.cp, hash(++i, sx(col), (u64)(ictx_get(M.ictx[0]) & 0xFF), (u64)(ictx_get(M.ictx[1]) & 0xFF)));
  cm_set(M.cp, hash(++i, ictx_get(M.ictx[2])));
  cm_set(M.cp, hash(++i, ictx_get(M.ictx[3])));
  cm_set(M.cp, hash(++i, (u64)(ictx_get(M.ictx[1]) & 0xFF), (u64)(ictx_get(M.ictx[3]) & 0xFF)));
  M.WxNW = (u8)(c ^ buf(S, rl + 1));
  cm_set(M.cp, hash(++i, (u64)N, (u64)M.WxNW));
  cm_set(M.cp, hash(++i, (u64)(S.st_match_length > 0 ? S.st_match_expected : (0x100 | (u8)ictx_get(M.ictx[1]))), (u64)N, (u64)M.WxNW));
  int k = 0x300;
  if (M.may_be_img24) { k = (col % 3) << 8; stm_set_direct(M.maps[0], (u32)(clip8((int)((u8)(c4 >> 16)) + c - (int)(c4 >> 24)) | k)); }
  else stm_set_direct(M.maps[0], (u32)(clip8(c * 2 - d) | k));
  stm_set_direct(M.maps[1], (u32)(clip8(c + N - buf(S, rl + 1)) | k));
  stm_set_direct(M.maps[2], (u32)clip8(N + NN - NNN));
  stm_set_direct(M.maps[3], (u32)clip8(N * 2 - NN));
  stm_set_direct(M.maps[4], (u32)clip8(N * 3 - NN * 3 + NNN));
  imap_set_direct(M.imap[0], (u32)(N + NN - NNN));
  imap_set_direct(M.imap[1], (u32)(N * 2 - NN));
  imap_set_direct(M.imap[2], (u32)(N * 3 - NN * 3 + NNN));
  M.cpos4[c] = M.cpos3[c]; M.cpos3[c] = M.cpos2[c]; M.cpos2[c] = M.cpos1[c]; M.cpos1[c] = pos;
  M.wpos1[w] = pos;
  M.mx_ctx = (rl > 128) ? imin(0x7F, col / imax(1, rl / 128)) : col;
}
P8_HD inline void record_pre(State& S) {   // per-bit context selection of the direct maps (:4412-4418)
  RecordM& M = S.record;
  const int bpos = S.bpos;
  const u8 B = (u8)(S.c0 << (8 - bpos));
  const u32 ctx = (u32)(M.N ^ B) | ((u32)bpos << 8);
  ictx_push(M.ictx[4], (u32)S.y); ictx_select(M.ictx[4], ctx);
  stm_set_direct(M.maps[5], ctx);
  scm_set(M.smap[0], ctx);
  scm_set(M.smap[1], ictx_get(M.ictx[4]));
  scm_set(M.smap[2], (ctx << 8) | M.WxNW);
}
P8_HD inline void record_small(State& S, Out& o, int k) {   // the 12 direct maps behind the four context maps, k = 0..11
  RecordM& M = S.record;
  const int y = S.y;
  if (k < 6) stm_mix(M.maps[k], o, y, 1, 3);
  else if (k < 9) imap_mix(M.imap[k - 6], o, y, 1, 3, 255);
  else if (k < 11) scm_mix(M.smap[k - 9], o, y, 6, 1, 3);
  else scm_mix(M.smap[2], o, y, 5, 1, 2);
}
P8_HD inline void record_select(State& S) {   // selector sets and ModelStats (:4429-4433)
  RecordM& M = S.record;
  const int bpos = S.bpos;
  const u8 B = (u8)(S.c0 << (8 - bpos));
  mset(S.m, (M.rlen[0] > 2) * ((bpos << 7) | M.mx_ctx), 1024);
  mset(S.m, ((M.N ^ B) >> 4) | (M.x << 4), 512);
  mset(S.m, (S.grp0 << 5) | M.x, 11 * 32);
  S.st_record = ((u32)imin(0xFFFF, M.rlen[0]) << 16) | (u32)imin(0xFFFF, M.col);
}
P8_HD inline void record_core(State& S, Out& o, Rnd& rnd) {
  RecordM& M = S.record;
  const int y = S.y, bpos = S.bpos, c0 = S.c0;
  const int c1 = buf(S, 1);
  if (bpos == 0) record_byte(S);
  record_pre(S);
  cm_mix(M.cm, o, rnd, y, c0, bpos, c1);
  cm_mix(M.cn, o, rnd, y, c0, bpos, c1);
  cm_mix(M.co, o, rnd, y, c0, bpos, c1);
  cm_mix(M.cp, o, rnd, y, c0, bpos, c1);
  for (int k = 0; k < 12; ++k) record_small(S, o, k);
}
P8_COLD P8_HD inline void record1_byte(State& S) {
  const Tables& T = *S.T;
  Record1M& M = S.record1;
    const u32 c4 = S.c4;
    const int w = (int)(c4 & 0xffff), c = w & 255, d = w & 0xf0ff, e = (int)(c4 & 0xffffff), pos = S.pos;
    cm_set(M.cm, sx(c << 8 | (imin(255, pos - M.cpos1[c]) / 4)));
    cm_set(M.cm, sx(w << 9 | llog(T, (u32)(pos - M.wpos1[w])) >> 2));
    cm_set(M.cn, sx(w));
    cm_set(M.cn, sx(d << 8));
    cm_set(M.cn, sx(c << 16));
    cm_set(M.cn, (u64)(S.f4 & 0xfffff));
    const int col = pos & 3;
    cm_set(M.cn, sx(col | 2 << 12));
    cm_set(M.co, sx(c));
    cm_set(M.co, sx(w << 8));
    cm_set(M.co, (u64)(S.w5 & 0x3ffff));
    cm_set(M.co, sx(e << 3));
    cm_set(M.cp, sx(d));
    cm_set(M.cp, sx(c << 8));
    cm_set(M.cp, sx(w << 16));
    cm_set(M.cq, sx(w << 3));
    cm_set(M.cq, sx(c << 19));
    cm_set(M.cq, sx(e));
    M.cpos1[c] = pos;
    M.wpos1[w] = pos;
}
P8_HD inline void record1_bit(State& S, Out& o, Rnd& rnd) {
  Record1M& M = S.record1;
  const int y = S.y, bpos = S.bpos, c0 = S.c0, c1 = buf(S, 1);
  if (bpos == 0) record1_byte(S);
  cm_mix(M.cm, o, rnd, y, c0, bpos, c1);
  cm_mix(M.cn, o, rnd, y, c0, bpos, c1);
  cm_mix(M.co, o, rnd, y, c0, bpos, c1);
  cm_mix(M.cq, o, rnd, y, c0, bpos, c1);
  cm_mix(M.cp, o, rnd, y, c0, bpos, c1);
}

// ---------------------------------------------------------------- word model (:3872-4105)
// wordModel at a byte boundary (:3873-4104) in three pieces: word_update changes the state (one lane), word_contexts is the pure
// list of the 57 contexts (a warp can share it: CtxSel), word_finish applies the sentence-end shift the reference does between
// contexts 41 and 42 (the contexts after it use the shifted words, computed locally).
P8_COLD P8_HD inline void word_update(State& S) {
  const Tables& T = *S.T;
  WordM& M = S.word;
  const u32 c4 = S.c4;
  int c = (int)(c4 & 255);
  const int pC = (u8)(c4 >> 8);
  int f = 0;
  if (S.spaces & 0x80000000u) --S.spacecount;
  if (S.words & 0x80000000u) --S.wordcount;
  S.spaces = S.spaces * 2;
  S.words = S.words * 2;
  M.last_upper = umin(M.last_upper + 1, 255);
  M.last_letter = umin(M.last_letter + 1, 255);
  M.mask2 <<= 2;
  if (c >= 'A' && c <= 'Z') { c += 'a' - 'A'; M.last_upper = 0; }
  if ((c >= 'a' && c <= 'z') || c == '\'' || c == '-') M.stem[M.cword].append(c);
  else if (M.stem[M.cword].len() > 0) {
    StemEN::stem(M.stem[M.cword]);
    M.stem[M.cword].get_hashes();
    M.stem_index = (M.stem_index + 1) & 3;
    M.pword = M.cword;
    M.cword = M.stem_index;
    M.stem[M.cword].clear();
  }
  if ((c >= 'a' && c <= 'z') || ((c >= 128 && (S.b3 != 3)) || (c > 0 && c < 4))) {
    if (!S.wordlen) {
      // the reference's test ASSIGNS lastLetter inside the condition (paq8.cpp:3914-3915): after it lastLetter is 0 or 1
      const bool hyph = ((c4 & 0xFFFF00) == 0x2B0A00 && buf(S, 4) != 0x2B) || ((c4 & 0xFFFFFF00) == 0x2B0D0A00 && buf(S, 5) != 0x2B) ||
                        ((c4 & 0xFFFF00) == 0x2D0A00 && buf(S, 4) != 0x2D) || ((c4 & 0xFFFFFF00) == 0x2D0D0A00 && buf(S, 5) != 0x2D);
      M.last_letter = hyph ? 1 : 0;
      if (hyph) {
        M.word0 = M.word1; M.word1 = M.word2; M.word2 = M.word3; M.word3 = M.word4; M.word4 = M.word5; M.word5 = 0;
        S.wordlen = S.wordlen1;
        if (c < 128) {
          M.stem_index = (M.stem_index - 1) & 3;
          M.cword = M.pword;
          M.pword = (M.stem_index - 1) & 3;
          M.stem[M.cword].clear();
          for (u32 i = 0; i <= S.wordlen; ++i) M.stem[M.cword].append(lower(buf(S, (int)(S.wordlen - i + 1 + 2 * (i != S.wordlen)))));
        }
      } else { M.word_gap = M.last_letter; M.first_letter = (u32)c; M.wrdhsh = 0; }
    }
    M.last_letter = 0;
    ++S.words; ++S.wordcount;
    if (c > 4) M.word0 = combine64(M.word0, (u64)c);
    M.text0 = M.text0 * 997 * 16 + (u32)c;
    S.wordlen++;
    S.wordlen = umin(S.wordlen, 45);
    f = 0;
    M.w = (int)((u32)M.word0 & 0xffff);
    if ((c == 'a' || c == 'e' || c == 'i' || c == 'o' || c == 'u') || (c == 'y' && (S.wordlen > 0 && pC != 'a' && pC != 'e' && pC != 'i' && pC != 'o' && pC != 'u'))) {
      M.mask2++;
      M.wrdhsh = M.wrdhsh * 997 * 8 + (u32)(c / 4 - 22);
    } else if (c >= 'b' && c <= 'z') { M.mask2 += 2; M.wrdhsh = M.wrdhsh * 271 * 32 + (u32)(c - 97); }
    else M.wrdhsh = M.wrdhsh * 11 * 32 + (u32)c;
  } else {
    if (M.word0) {
      M.type0 = (M.type0 << 2) | 1;
      M.word5 = M.word4; M.word4 = M.word3; M.word3 = M.word2; M.word2 = M.word1; M.word1 = M.word0;
      S.wordlen1 = S.wordlen;
      M.wpos[M.w] = S.blpos;
      if (c == ':' || c == '=') M.cword0 = M.word0;
      if (c == ']' && (S.frstchar != ':')) M.xword0 = M.word0;
      M.ccword = 0;
      M.word0 = 0;
      S.wordlen = 0;
      if ((c == '.' || c == '!' || c == '?' || c == '}' || c == ')') && buf(S, 2) != 10) f = 1;
    }
    if (c == 0x20 || c == 10 || c == 5) { ++S.spaces; ++S.spacecount; if (c == 10 || c == 5) { M.nl1 = M.nl; M.nl = S.pos - 1; } }
    else if (c == '.' || c == '!' || c == '?' || c == ',' || c == ';' || c == ':') { S.spafdo = 0; M.ccword = (u64)c; M.mask2 += 3; }
    else { ++S.spafdo; S.spafdo = umin(63, S.spafdo); }
  }
  if ((c4 & 0xFFFF) == 0x3D3D && S.frstchar == 0x3d) M.xword1 = M.word1;
  if ((c4 & 0xFFFF) == 0x2727) M.xword2 = M.word1;
  M.last_digit = umin(0xFF, M.last_digit + 1);
  if (c >= '0' && c <= '9') {
    if (buf(S, 3) >= '0' && buf(S, 3) <= '9' && (buf(S, 2) == '.') && M.number0 == 0) { M.number0 = M.number1; M.number1 = 0; }
    M.number0 = combine64(M.number0, (u64)c);
    M.last_digit = 0;
  } else if (M.number0) {
    M.type0 = (M.type0 << 2) | 2;
    M.number1 = M.number0;
    M.number0 = 0; M.ccword = 0;
  }
  if (!((c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || (c >= 128))) M.data0 ^= (u32)combine64(M.data0, (u64)c);
  else if (M.data0) { M.type0 = (M.type0 << 2) | 3; M.data0 = 0; }
  S.col = (u32)imin(255, S.pos - M.nl);
  const int above = bufa(S, (u32)(M.nl1 + (int)S.col));
  if (S.col <= 2) S.frstchar = (S.col == 2 ? (u32)imin(c, 96) : 0);
  if (S.frstchar == '[' && c == 32) { if (buf(S, 3) == ']' || buf(S, 4) == ']') { S.frstchar = 96; M.xword0 = 0; } }
  {
    int fl = 0;
    const int cc = (int)(c4 & 0xff);
    if (cc != 0) {
      if (is_alpha(cc)) fl = 1;
      else if (is_punct(cc)) fl = 2;
      else if (is_space(cc)) fl = 3;
      else if (cc == 0xff) fl = 4;
      else if (cc < 16) fl = 5;
      else if (cc < 64) fl = 6;
      else fl = 7;
    }
    M.mask = (M.mask << 3) | (u32)fl;
  }
  M.above = above;
  M.f_pending = f;
}
P8_HD inline int word_contexts(State& S, const CtxSel sel) {
  const Tables& T = *S.T;
  WordM& M = S.word;
  Cm& cm = M.cm;
  const u32 c4 = S.c4;
  int c = (int)(c4 & 255);
  if (c >= 'A' && c <= 'Z') c += 'a' - 'A';
  const int above = M.above, f = M.f_pending;
  // the words as the contexts after the sentence-end shift see them (word_finish applies it to the state)
  const u64 nword1 = f ? (u64)'.' : M.word1, nword2 = f ? M.word1 : M.word2;
  int n = cm.cn;
  const u32 col = S.col, frstchar = S.frstchar, spaces = S.spaces, spafdo = S.spafdo, wordlen = S.wordlen, wordlen1 = S.wordlen1;
  P8_CM_SET(sel, cm, n, hash(513, spafdo, spaces, M.ccword));
  P8_CM_SET(sel, cm, n, hash(514, frstchar, sx(c)));
  P8_CM_SET(sel, cm, n, hash(515, col, frstchar, (u64)((M.last_upper < col) * 4 + (M.mask2 & 3))));
  P8_CM_SET(sel, cm, n, hash(516, spaces, (u64)(S.words & 255)));
  P8_CM_SET(sel, cm, n, spaces & 0x7fff);
  P8_CM_SET(sel, cm, n, spaces & 0xff);
  P8_CM_SET(sel, cm, n, hash(257, M.number0, M.word1, M.word_gap));
  P8_CM_SET(sel, cm, n, hash(258, M.number1, sx(c), M.ccword));
  P8_CM_SET(sel, cm, n, hash(259, M.number0, M.number1, M.word_gap));
  P8_CM_SET(sel, cm, n, hash(260, M.word0, M.number1, (u64)(M.last_digit < M.word_gap + wordlen)));
  P8_CM_SET(sel, cm, n, hash(274, M.number0, M.cword0));
  P8_CM_SET(sel, cm, n, hash(518, wordlen1, col));
  P8_CM_SET(sel, cm, n, hash(519, sx(c), (u64)(S.spacecount / 2), M.word_gap));
  u32 h = S.wordcount * 64 + S.spacecount;
  P8_CM_SET(sel, cm, n, hash(520, sx(c), h, M.ccword));
  P8_CM_SET(sel, cm, n, hash(517, frstchar, h, M.last_letter));
  P8_CM_SET(sel, cm, n, hash(M.data0, M.word1, M.number1, (u64)(M.type0 & 0xFFF)));
  P8_CM_SET(sel, cm, n, hash(521, h, spafdo));
  const u32 d = c4 & 0xf0ff;
  P8_CM_SET(sel, cm, n, hash(522, d, frstchar, M.ccword));
  h = (u32)(M.word0 * 271);
  h = h + (u32)buf(S, 1);
  P8_CM_SET(sel, cm, n, hash(262, h, 0));
  P8_CM_SET(sel, cm, n, hash(M.number0 * 271 + (u64)buf(S, 1), 0));
  P8_CM_SET(sel, cm, n, hash(263, M.word0, 0));
  if (M.wrdhsh) P8_CM_SET(sel, cm, n, hash(M.wrdhsh, (u64)buf(S, M.wpos[M.word1 & 0xffff]))); else P8_CM_SET(sel, cm, n, 0);
  P8_CM_SET(sel, cm, n, hash(264, h, M.word1));
  P8_CM_SET(sel, cm, n, hash(265, M.word0, M.word1));
  P8_CM_SET(sel, cm, n, hash(266, h, M.word1, M.word2, (u64)(M.last_upper < wordlen)));
  P8_CM_SET(sel, cm, n, hash(267, (u64)(M.text0 & 0xffffff), 0));
  P8_CM_SET(sel, cm, n, M.text0 & 0xfffff);
  P8_CM_SET(sel, cm, n, hash(269, M.word0, M.xword0));
  P8_CM_SET(sel, cm, n, hash(270, h, M.xword1));
  P8_CM_SET(sel, cm, n, hash(271, h, M.xword2));
  P8_CM_SET(sel, cm, n, hash(272, frstchar, M.xword2));
  P8_CM_SET(sel, cm, n, hash(273, M.word0, M.cword0));
  P8_CM_SET(sel, cm, n, hash(275, h, M.word2));
  P8_CM_SET(sel, cm, n, hash(276, h, M.word3));
  P8_CM_SET(sel, cm, n, hash(277, h, M.word4));
  P8_CM_SET(sel, cm, n, hash(278, h, M.word5));
  P8_CM_SET(sel, cm, n, hash(279, h, M.word1, M.word3));
  P8_CM_SET(sel, cm, n, hash(280, h, M.word2, M.word3));
  P8_CM_SET(sel, cm, n, (u64)(buf(S, 1) | buf(S, 3) << 8 | buf(S, 5) << 16));
  P8_CM_SET(sel, cm, n, (u64)(buf(S, 2) | buf(S, 4) << 8 | buf(S, 6) << 16));
  P8_CM_SET(sel, cm, n, (u64)(buf(S, 1) | buf(S, 4) << 8 | buf(S, 7) << 16));
  if (col < 255u) {
    P8_CM_SET(sel, cm, n, hash(523, col, (u64)buf(S, 1), sx(above)));
    P8_CM_SET(sel, cm, n, hash(524, (u64)buf(S, 1), sx(above)));
    P8_CM_SET(sel, cm, n, hash(525, col, (u64)buf(S, 1)));
    P8_CM_SET(sel, cm, n, hash(526, col, (u64)(c == 32)));
  } else { P8_CM_SET(sel, cm, n, 0); P8_CM_SET(sel, cm, n, 0); P8_CM_SET(sel, cm, n, 0); P8_CM_SET(sel, cm, n, 0); }
  if (wordlen) P8_CM_SET(sel, cm, n, hash(281, M.word0, sx(llog(T, (u32)(S.blpos - M.wpos[nword1 & 0xffff])) >> 4)));
  else P8_CM_SET(sel, cm, n, 0);
  P8_CM_SET(sel, cm, n, hash(282, (u64)buf(S, 1), sx(llog(T, (u32)(S.blpos - M.wpos[nword1 & 0xffff])) >> 2)));
  P8_CM_SET(sel, cm, n, hash(283, (u64)buf(S, 1), M.word0, sx(llog(T, (u32)(S.blpos - M.wpos[nword2 & 0xffff])) >> 2)));
  P8_CM_SET(sel, cm, n, hash(528, M.mask, 0));
  P8_CM_SET(sel, cm, n, hash(529, M.mask, (u64)buf(S, 1)));
  P8_CM_SET(sel, cm, n, hash(530, (u64)(M.mask & 0xff), col));
  P8_CM_SET(sel, cm, n, hash(531, M.mask, (u64)buf(S, 2), (u64)buf(S, 3)));
  P8_CM_SET(sel, cm, n, hash(532, (u64)(M.mask & 0x1ff), (u64)(S.f4 & 0x00fff0)));
  P8_CM_SET(sel, cm, n, hash(h, sx(llog(T, M.word_gap)), (u64)(M.mask & 0x1FF),
                  (u64)(((wordlen1 > 3) << 6) | ((wordlen > 0) << 5) | ((spafdo == wordlen + 2) << 4) | ((spafdo == wordlen + wordlen1 + 3) << 3) |
                        ((spafdo >= M.last_letter + wordlen1 + M.word_gap) << 2) | ((M.last_upper < M.last_letter + wordlen1) << 1) |
                        (M.last_upper < wordlen + wordlen1 + M.word_gap)),
                  (u64)(M.type0 & 0xFFF)));
  if (wordlen1) P8_CM_SET(sel, cm, n, hash(col, wordlen1, sx(above & 0x5F), (u64)(c4 & 0x5F))); else P8_CM_SET(sel, cm, n, 0);
  if (M.wrdhsh) P8_CM_SET(sel, cm, n, hash((u64)(M.mask2 & 0x3F), (u64)(M.wrdhsh & 0xFFF), (u64)((0x100 | M.first_letter) * (wordlen < 6)), (u64)((M.word_gap > 4) * 2 + (wordlen1 > 5))));
  else P8_CM_SET(sel, cm, n, 0);
  if (M.last_letter < 16) P8_CM_SET(sel, cm, n, hash(M.stem[M.pword].hash[2], h)); else P8_CM_SET(sel, cm, n, 0);
  return n;
}
P8_HD inline void word_finish(State& S) {
  WordM& M = S.word;
  if (M.f_pending) { M.word5 = M.word4; M.word4 = M.word3; M.word3 = M.word2; M.word2 = M.word1; M.word1 = '.'; }
}
P8_HD inline void word_byte(State& S) {
  word_update(S);
  S.word.cm.cn = word_contexts(S, CtxSel{0, 1});
  word_finish(S);
}

// ---------------------------------------------------------------- nest model (:4107-4181)
P8_COLD P8_HD inline void nest_byte(State& S) {
  NestM& M = S.nest;
  const u32 c4 = S.c4;
  const int c = (int)(c4 & 255);
  int matched = 1, vv;
  M.w *= ((M.vc & 7) > 0 && (M.vc & 7) < 3);
  if (c & 0x80) M.w = (int)((u32)M.w * 11 * 32 + (u32)c);
  const int lc = (c >= 'A' && c <= 'Z' ? c + 'a' - 'A' : c);
  if (lc == 'a' || lc == 'e' || lc == 'i' || lc == 'o' || lc == 'u') { vv = 1; M.w = (int)((u32)M.w * 997 * 8 + (u32)(lc / 4 - 22)); }
  else if (lc >= 'a' && lc <= 'z') { vv = 2; M.w = (int)((u32)M.w * 271 * 32 + (u32)(lc - 97)); }
  else if (lc == ' ' || lc == '.' || lc == ',' || lc == '!' || lc == '?' || lc == '\n') vv = 3;
  else if (lc >= '0' && lc <= '9') vv = 4;
  else if (lc == 'y') vv = 5;
  else if (lc == '\'') vv = 6;
  else vv = (c & 32) ? 7 : 0;
  M.vc = (M.vc << 3) | (u32)vv;
  if (vv != M.lvc) { M.wc = (M.wc << 3) | (u32)vv; M.lvc = vv; }
  switch (c) {
    case ' ': M.qc = 0; break;
    case '(': M.ic += 31; break;
    case ')': M.ic -= 31; break;
    case '[': M.ic += 11; break;
    case ']': M.ic -= 11; break;
    case '<': M.ic += 23; M.qc += 34; break;
    case '>': M.ic -= 23; M.qc /= 5; break;
    case ':': M.pc = 20; break;
    case '{': M.ic += 17; break;
    case '}': M.ic -= 17; break;
    case '|': M.pc += 223; break;
    case '"': M.pc += 0x40; break;
    case '\'': M.pc += 0x42; if (c != (u8)(c4 >> 8)) M.sense2 ^= 1; else M.ac += (2 * M.sense2 - 1); break;
    case '\n': M.pc = M.qc = 0; break;
    case '.': M.pc = 0; break;
    case '!': M.pc = 0; break;
    case '?': M.pc = 0; break;
    case '#': M.pc += 0x08; break;
    case '%': M.pc += 0x76; break;
    case '$': M.pc += 0x45; break;
    case '*': M.pc += 0x35; break;
    case '-': M.pc += 0x3; break;
    case '@': M.pc += 0x72; break;
    case '&': M.qc += 0x12; break;
    case ';': M.qc /= 3; break;
    case '\\': M.pc += 0x29; break;
    case '/': M.pc += 0x11; if (buf(S, 1) == '<') M.qc += 74; break;
    case '=': M.pc += 87; if (c != (u8)(c4 >> 8)) M.sense1 ^= 1; else M.ec += (2 * M.sense1 - 1); break;
    default: matched = 0;
  }
  if (c4 == 0x266C743B) M.uc = imin(7, M.uc + 1);
  else if (c4 == 0x2667743B) M.uc -= (M.uc > 0);
  if (matched) M.bc = 0; else M.bc += 1;
  if (M.bc > 300) M.bc = M.ic = M.pc = M.qc = M.uc = 0;
  const u32 vc = M.vc, wc = M.wc;
  const int ic = M.ic, pc = M.pc, qc = M.qc, bc = M.bc;
  u64 i = 0;
  cm_set(M.cm, hash(++i, sx((vv > 0 && vv < 3) ? 0 : (lc | 0x100)), sx(ic & 0x3FF), sx(M.ec & 0x7), sx(M.ac & 0x7), sx(M.uc)));
  cm_set(M.cm, hash(++i, sx(ic), sx(M.w), (u64)ilog2((u32)(bc + 1))));
  cm_set(M.cm, hash(++i, (u64)((3 * vc + 77 * (u32)pc + 373 * (u32)ic + (u32)qc) & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)((31 * vc + 27 * (u32)pc + 281 * (u32)qc) & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)((13 * vc + 271 * (u32)ic + (u32)qc + (u32)bc) & 0xffff)));
  cm_set(M.cm, hash(++i, sx((17 * pc + 7 * ic) & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)((13 * vc + (u32)ic) & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)((vc / 3 + (u32)pc) & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)((7 * wc + (u32)qc) & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)(vc & 0xffff), (u64)(S.f4 & 0xf)));
  cm_set(M.cm, hash(++i, sx((3 * pc) & 0xffff), (u64)(S.f4 & 0xf)));
  cm_set(M.cm, hash(++i, sx(ic & 0xffff), (u64)(S.f4 & 0xf)));
}

// ---------------------------------------------------------------- indirect model (:7548-7612)
P8_COLD P8_HD inline void indirect_byte(State& S) {
  IndirectM& M = S.indirect;
  const u32 c4 = S.c4;
  const u32 d = c4 & 0xffff;
  u32 c = d & 255;
  const u32 d2 = (u32)((buf(S, 1) & 31) + 32 * (buf(S, 2) & 31) + 1024 * (buf(S, 3) & 31));
  const u32 d3 = (u32)((buf(S, 1) >> 3 & 31) + 32 * (buf(S, 3) >> 3 & 31) + 1024 * (buf(S, 4) >> 3 & 31));
  u32& r1 = M.t1[d >> 8]; r1 = r1 << 8 | c;
  u16& r2 = M.t2[c4 >> 8 & 0xffff]; r2 = (u16)(r2 << 8 | c);
  u16& r3 = M.t3[(buf(S, 2) & 31) + 32 * (buf(S, 3) & 31) + 1024 * (buf(S, 4) & 31)]; r3 = (u16)(r3 << 8 | c);
  u16& r4 = M.t4[(buf(S, 2) >> 3 & 31) + 32 * (buf(S, 4) >> 3 & 31) + 1024 * (buf(S, 5) >> 3 & 31)]; r4 = (u16)(r4 << 8 | c);
  const u32 t = c | M.t1[c] << 8;
  const u32 t0 = d | (u32)M.t2[d] << 16;
  const u32 ta = d2 | (u32)M.t3[d2] << 16;
  const u32 tc = d3 | (u32)M.t4[d3] << 16;
  const u8 pc = (u8)lower((u8)(c4 >> 8));
  c = (u32)lower((int)c);
  ictx_push(M.ictx, c); ictx_select(M.ictx, ((u32)pc << 8) | c);
  const u32 ctx0 = ictx_get(M.ictx);
  const u32 mask = (u32)((u8)M.t1[c] == (u8)M.t2[d]) | ((u32)((u8)M.t1[c] == (u8)M.t3[d2]) << 1) | ((u32)((u8)M.t1[c] == (u8)M.t4[d3]) << 2) |
                   ((u32)((u8)M.t1[c] == (u8)ctx0) << 3);
  u64 i = 0;
  cm_set(M.cm, hash(++i, t));
  cm_set(M.cm, hash(++i, t0));
  cm_set(M.cm, hash(++i, ta));
  cm_set(M.cm, hash(++i, tc));
  cm_set(M.cm, hash(++i, (u64)(t & 0xff00), mask));
  cm_set(M.cm, hash(++i, (u64)(t0 & 0xff0000)));
  cm_set(M.cm, hash(++i, (u64)(ta & 0xff0000)));
  cm_set(M.cm, hash(++i, (u64)(tc & 0xff0000)));
  cm_set(M.cm, hash(++i, (u64)(t & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)(t0 & 0xffffff)));
  cm_set(M.cm, hash(++i, (u64)(ta & 0xffffff)));
  cm_set(M.cm, hash(++i, (u64)(tc & 0xffffff)));
  cm_set(M.cm, hash(++i, (u64)(ctx0 & 0xff), c));
  cm_set(M.cm, hash(++i, (u64)(ctx0 & 0xffff)));
  cm_set(M.cm, hash(++i, (u64)(ctx0 & 0x7f7fff)));
}

// ---------------------------------------------------------------- DMC forest (:7777-7822)
P8_COLD P8_HD inline void dmc_reset(Dmc& d, u32 th_start) {   // resetstategraph (:7655-7677)
  d.top = d.curr = d.extra = 0;
  d.threshold = th_start;
  d.threshold_fine = th_start << 11;
  for (int j = 0; j < 256; ++j)
    for (int i = 0; i < 255; ++i) {
      DmcNode& n = d.t[d.top];
      if (i < 127) { n.nx0 = (n.nx0 & 0xf) | ((d.top + (u32)i + 1) << 4); n.nx1 = (n.nx1 & 0xf) | ((d.top + (u32)i + 2) << 4); }
      else { const u32 root = (u32)(i - 127) * 2 * 255; n.nx0 = (n.nx0 & 0xf) | (root << 4); n.nx1 = (n.nx1 & 0xf) | ((root + 255) << 4); }
      n.c0 = n.c1 = th_start < 1024 ? 2048 : 512;
      dmc_set_state(n, 0);
      d.top++;
    }
}
P8_HD inline void dmc_bit(State& S, Out& o) {
  const Tables& T = *S.T;
  const u32 params[10] = {2, 32, 64, 4, 128, 8, 256, 16, 1024, 1536};
  int st[10];
  for (int i = 9; i >= 0; --i) st[i] = dmc_st(T, S.dmc[i], S.y);
  add(o, st[9] >> 3);
  add(o, st[8] >> 3);
  for (int i = 7; i > 0; i -= 2) add(o, (st[i] + st[i - 1]) >> 4);
  if (S.bpos == 0)
    for (int i = 7; i >= 0; --i)
      if ((S.dmc[i].extra >> 7) > S.dmc[i].size) dmc_reset(S.dmc[i], params[i]);
}

// ---------------------------------------------------------------- XML model (:7824-8097)
P8_HD inline void xml_detect(State& S, u32& type, u32 length, u32 c8, u8 B) {   // DetectContent macro (:7871-7912)
  const u32 c4 = S.c4;
  if ((c4 & 0xF0F0F0F0) == 0x30303030) {
    int i = 0, j = 0;
    while ((i < 4) && ((j = (int)((c4 >> (8 * i)) & 0xFF)) >= 0x30 && j <= 0x39)) i++;
    if (i == 4 && (((c8 & 0xFDF0F0FD) == 0x2D30302D && buf(S, 9) >= 0x30 && buf(S, 9) <= 0x39) || ((c8 & 0xF0FDF0FD) == 0x302D302D))) type |= 0x004;
  } else if (((c8 & 0xF0F0FDF0) == 0x30302D30 || (c8 & 0xF0F0F0FD) == 0x3030302D) && buf(S, 9) >= 0x30 && buf(S, 9) <= 0x39) {
    int i = 2, j = 0;
    while ((i < 4) && ((j = (int)((c8 >> (8 * i)) & 0xFF)) >= 0x30 && j <= 0x39)) i++;
    if (i == 4 && (c4 & 0xF0FDF0F0) == 0x302D3030) type |= 0x004;
  }
  if ((c4 & 0xF0FFF0F0) == 0x303A3030 && buf(S, 5) >= 0x30 && buf(S, 5) <= 0x39 &&
      ((buf(S, 6) < 0x30 || buf(S, 6) > 0x39) || ((c8 & 0xF0F0FF00) == 0x30303A00 && (buf(S, 9) < 0x30 || buf(S, 9) > 0x39)))) type |= 0x008;
  if (length >= 8 && (c8 & 0x80808080) == 0 && (c4 & 0x80808080) == 0) type |= 0x001;
  if ((c8 & 0xF0F0FF) == 0x3030C2 && (c4 & 0xFFF0F0FF) == 0xB0303027) {
    int i = 2;
    while ((i < 7) && buf(S, i) >= 0x30 && buf(S, i) <= 0x39) i += (i & 1) * 2 + 1;
    if (i == 10) type |= 0x040;
  }
  if ((c4 & 0xFFFFFA) == 0xC2B042 && B != 0x47 && (((c4 >> 24) >= 0x30 && (c4 >> 24) <= 0x39) || ((c4 >> 24) == 0x20 && (buf(S, 5) >= 0x30 && buf(S, 5) <= 0x39)))) type |= 0x080;
  if (B >= 0x30 && B <= 0x39) type |= 0x002;
  if (c4 == 0x4953424E && buf(S, 5) == 0x20) type |= 0x100;
}
P8_HD inline void xml_clear(XmlTag& t) { t.name = t.length = 0; t.level = 0; t.end_tag = t.empty = 0; t.pad[0] = t.pad[1] = 0; t.c_data = t.c_length = t.c_type = 0;
  for (int i = 0; i < 4; ++i) t.a_name[i] = t.a_value[i] = t.a_length[i] = 0; t.a_index = 0; }
P8_COLD P8_HD inline void xml_byte(State& S) {
  XmlM& M = S.xml;
  enum { None, ReadTagName, ReadTag, ReadAttributeName, ReadAttributeValue, ReadContent, ReadCDATA, ReadComment };
  const u32 c4 = S.c4;
  const u8 B = (u8)c4;
  XmlTag* pTag = &M.tags[(M.index - 1) & 31];
  XmlTag* Tag = &M.tags[M.index & 31];
  const u32 ai = Tag->a_index & 3;
  M.pstate = M.state;
  M.c8 = (M.c8 << 8) | (u32)buf(S, 5);
  const u32 c8 = M.c8;
  if ((B == 0x09 || B == 0x20) && (B == (u8)(c4 >> 8) || !M.ws_run)) { M.ws_run++; M.indent_tab = (B == 0x09); }
  else {
    if ((M.state == None || (M.state == ReadContent && Tag->c_length <= M.line_ending + M.ws_run)) && M.ws_run > 1 + M.indent_tab && M.ws_run != M.p_ws_run) {
      M.indent_step = (u32)iabs((int)(M.ws_run - M.p_ws_run));
      M.p_ws_run = M.ws_run;
    }
    M.ws_run = 0;
  }
  if (B == 0x0A) M.line_ending = 1 + ((u8)(c4 >> 8) == 0x0D);
  const int pState = M.pstate;
  switch (M.state) {
    case None: {
      if (B == 0x3C) {
        M.state = ReadTagName;
        xml_clear(*Tag);
        Tag->level = (pTag->end_tag || pTag->empty) ? pTag->level : pTag->level + 1;
      }
      if (Tag->level > 1) xml_detect(S, Tag->c_type, Tag->c_length, c8, B);
      cm_set(M.cm, hash(sx(pState), sx(M.state), (u64)((u32)(pTag->level + 1) * M.indent_step - M.ws_run)));
      break;
    }
    case ReadTagName: {
      if (Tag->length > 0 && (B == 0x09 || B == 0x0A || B == 0x0D || B == 0x20)) M.state = ReadTag;
      else if ((B == 0x3A || (B >= 'A' && B <= 'Z') || B == 0x5F || (B >= 'a' && B <= 'z')) || (Tag->length > 0 && (B == 0x2D || B == 0x2E || (B >= '0' && B <= '9')))) {
        Tag->length++;
        Tag->name = Tag->name * 263 * 32 + (B & 0xDF);
      } else if (B == 0x3E) {
        if (Tag->end_tag) { M.state = None; M.index++; }
        else M.state = ReadContent;
      } else if (B != 0x21 && B != 0x2D && B != 0x2F && B != 0x5B) { M.state = None; M.index++; }
      else if (Tag->length == 0) {
        if (B == 0x2F) { Tag->end_tag = 1; Tag->level = imax(0, Tag->level - 1); }
        else if (c4 == 0x3C212D2D) { M.state = ReadComment; Tag->level = imax(0, Tag->level - 1); }
      }
      if (Tag->length == 1 && (c4 & 0xFFFF00) == 0x3C2100) { xml_clear(*Tag); M.state = None; }
      else if (Tag->length == 5 && c8 == 0x215B4344 && c4 == 0x4154415B) { M.state = ReadCDATA; Tag->level = imax(0, Tag->level - 1); }
      int i = 1;
      do {
        pTag = &M.tags[(M.index - (u32)i) & 31];
        i += 1 + (pTag->end_tag && M.tags[(M.index - (u32)i - 1) & 31].name == pTag->name);
      } while (i < 32 && (pTag->end_tag || pTag->empty));
      cm_set(M.cm, hash(sx(pState * 8 + M.state), Tag->name, sx(Tag->level), pTag->name, (u64)(pTag->level != Tag->level)));
      break;
    }
    case ReadTag: {
      if (B == 0x2F) Tag->empty = 1;
      else if (B == 0x3E) {
        if (Tag->empty) { M.state = None; M.index++; }
        else M.state = ReadContent;
      } else if (B != 0x09 && B != 0x0A && B != 0x0D && B != 0x20) { M.state = ReadAttributeName; Tag->a_name[ai] = B & 0xDF; }
      cm_set(M.cm, hash(sx(pState), sx(M.state), Tag->name, B, Tag->a_index));
      break;
    }
    case ReadAttributeName: {
      if ((c4 & 0xFFF0) == 0x3D20 && (B == 0x22 || B == 0x27)) {
        M.state = ReadAttributeValue;
        if ((c8 & 0xDFDF) == 0x4852 && (c4 & 0xDFDF0000) == 0x45460000) Tag->c_type |= 0x020;
      } else if (B != 0x22 && B != 0x27 && B != 0x3D) Tag->a_name[ai] = Tag->a_name[ai] * 263 * 32 + (B & 0xDF);
      cm_set(M.cm, hash(sx(pState * 8 + M.state), Tag->a_name[ai], Tag->a_index, Tag->name, Tag->c_type));
      break;
    }
    case ReadAttributeValue: {
      if (B == 0x22 || B == 0x27) { Tag->a_index++; M.state = ReadTag; }
      else {
        Tag->a_value[ai] = Tag->a_value[ai] * 263 * 32 + (B & 0xDF);
        Tag->a_length[ai]++;
        if ((c8 & 0xDFDFDFDF) == 0x48545450 && ((c4 >> 8) == 0x3A2F2F || c4 == 0x733A2F2F)) Tag->c_type |= 0x010;
      }
      cm_set(M.cm, hash(sx(pState), sx(M.state), Tag->a_name[ai], Tag->c_type));
      break;
    }
    case ReadContent: {
      if (B == 0x3C) {
        M.state = ReadTagName;
        M.index++;
        xml_clear(M.tags[M.index & 31]);
        M.tags[M.index & 31].level = Tag->level + 1;
      } else {
        Tag->c_length++;
        Tag->c_data = Tag->c_data * 997 * 16 + (B & 0xDF);
        xml_detect(S, Tag->c_type, Tag->c_length, c8, B);
      }
      cm_set(M.cm, hash(sx(pState), sx(M.state), Tag->name, (u64)(c4 & 0xC0FF)));
      break;
    }
    case ReadCDATA: {
      if ((c4 & 0xFFFFFF) == 0x5D5D3E) { M.state = None; M.index++; }
      cm_set(M.cm, hash(sx(pState), sx(M.state)));
      break;
    }
    case ReadComment: {
      if ((c4 & 0xFFFFFF) == 0x2D2D3E) { M.state = None; M.index++; }
      cm_set(M.cm, hash(sx(pState), sx(M.state)));
      break;
    }
  }
  M.state_bh[M.state] = (M.state_bh[M.state] << 8) | B;
  pTag = &M.tags[(M.index - 1) & 31];
  u64 i = 64;
  cm_set(M.cm, hash(++i, sx(M.state), sx(Tag->level), sx(pState * 2 + Tag->end_tag), Tag->name));
  cm_set(M.cm, hash(++i, pTag->name, sx(M.state * 2 + pTag->end_tag), pTag->c_type, Tag->c_type));
  cm_set(M.cm, hash(++i, sx(M.state * 2 + Tag->end_tag), Tag->name, Tag->c_type, (u64)(c4 & 0xE0FF)));
}
P8_HD inline void xml_stats(State& S) {
  XmlM& M = S.xml;
  const int bpos = S.bpos;
  const u32 bh = M.state_bh[M.state];
  const u8 s = (u8)(((bh >> (28 - bpos)) & 0x08) | ((bh >> (21 - bpos)) & 0x04) | ((bh >> (14 - bpos)) & 0x02) | ((bh >> (7 - bpos)) & 0x01) | (bpos << 4));
  S.st_xml = ((u32)s << 3) | (u32)M.state;
}
P8_HD inline void xml_bit(State& S, Out& o, Rnd& rnd) {
  if (S.bpos == 0) xml_byte(S);
  cm_mix(S.xml.cm, o, rnd, S.y, S.c0, S.bpos, buf(S, 1));
  xml_stats(S);
}

}  // namespace p8
}  // namespace cmixb200
#endif
