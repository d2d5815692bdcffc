// cmix_b200/csrc/paq8_top.h — text model, x86 model, linear prediction, and the top level of the resident PAQ8 model
// (contextModel2 + Predictor::update, reference src/models/paq8.cpp:8101-8362). Continues paq8_predict.h.
#ifndef CMIXB200_PAQ8_TOP_H
#define CMIXB200_PAQ8_TOP_H

#include <math.h>

#include "paq8_predict.h"

namespace cmixb200 {
namespace p8 {

// ---------------------------------------------------------------- text model (:3070-3519)
// Cache<T,N>(i) = Data[(Index - i) & (N-1)]
P8_HD inline Word& tw(TextM& M, int lang, u32 i) { return M.words[lang][(M.words_index[lang] - i) & 7]; }
// cWord / pWord are pointers into the word caches in the reference; here (language, slot) pairs, which stay valid when the
// state block is copied. slot_of = the slot Words[lang](i) denotes right now.
P8_HD inline int slot_of(const TextM& M, int lang, u32 i) { return (int)((M.words_index[lang] - i) & 7); }
#define P8_CW (M.words[M.cw_lang][M.cw_slot])
#define P8_PW (M.words[M.pw_lang][M.pw_slot])
P8_HD inline Segment& tseg(TextM& M, u32 i) { return M.segments[(M.seg_index - i) & 3]; }
P8_HD inline Sentence& tsen(TextM& M, u32 i) { return M.sentences[(M.sen_index - i) & 3]; }
P8_HD inline void word_copy(Word& d, const Word& s) { d = s; }
P8_HD inline void sentence_clear(Sentence& s) {
  s.first_word.clear(); s.word_count = s.num_count = 0; s.type = 0; s.segment_count = s.verb_index = s.noun_index = s.capital_index = 0;
  s.last_verb.clear(); s.last_noun.clear(); s.last_capital.clear();
}
enum { TP_Unknown, TP_ReadingWord, TP_PossibleHyphenation, TP_WasAbbreviation, TP_AfterComma, TP_AfterQuote, TP_AfterAbbreviation, TP_ExpectDigit };

// TextModel::Update (:3187-3375) in pieces so that the three stemmers of a completed word can run side by side on the device:
// text_update_a does everything up to them (returns 1 when they are due), text_stem(lang) is one stemmer on its copy of the
// word, text_update_b applies their verdicts and finishes the byte. text_update is the three in order.
P8_COLD P8_HD inline void text_else_rest(State& S, u8 c, u8 pC) {
  TextM& M = S.text;
    bool skip = false;
    int stage = 0;   // fall-through emulation: 1 = sentence end, 2 = segment end, 3 = new line, 4 = white space
    switch (c) {
      case '.':
        if (M.lang_id != LANG_UNKNOWN && M.last_upper == M.word_length[1] && lang_abbrev(M.lang_id, P8_PW)) {
          M.state = TP_WasAbbreviation; M.parse_ctx = hash(sx(M.state), P8_PW.hash[1]);
          break;
        }
        stage = 1; break;
      case '?': case '!': stage = 1; break;
      case ',': case ';': case ':': stage = 2; break;
      case 0x0A: stage = 3; break;
      case 0x09: case 0x0D: case 0x20: stage = 4; break;
      case '(': M.masks[2] += 1; M.masks[3] += 6; M.nest_hash += 31; M.last_nest = 0; break;
      case '[': M.masks[2] += 2; M.nest_hash += 11; M.last_nest = 0; break;
      case '{': M.masks[2] += 3; M.nest_hash += 17; M.last_nest = 0; break;
      case '<': M.masks[2] += 4; M.nest_hash += 23; M.last_nest = 0; break;
      case 0xAB: M.masks[2] += 5; break;
      case ')': M.masks[2] += 6; M.nest_hash -= 31; M.last_nest = 0; break;
      case ']': M.masks[2] += 7; M.nest_hash -= 11; M.last_nest = 0; break;
      case '}': M.masks[2] += 8; M.nest_hash -= 17; M.last_nest = 0; break;
      case '>': M.masks[2] += 9; M.nest_hash -= 23; M.last_nest = 0; break;
      case 0xBB: M.masks[2] += 10; break;
      case '"':
        M.masks[2] += 11;
        if (M.quote_length == 0) M.quote_length = 1;
        else { M.quote_length = 0; M.state = TP_AfterQuote; M.parse_ctx = hash(sx(M.state), (u64)(0x100 | pC)); }
        break;
      case '/': case '-': case '+': case '*': case '=': case '%': M.masks[2] += 13; break;
      case '\\': case '|': case '_': case '@': case '&': case '^': M.masks[2] += 14; break;
    }
    if (stage == 1) {
      Sentence& sen = tsen(M, 0);
      Paragraph& par = M.paragraphs[M.par_index & 1];
      sen.type = (c == '.') ? 0 : (c == '?') ? 1 : 2;
      sen.segment_count++;
      par.sentence_count++;
      par.type_count[sen.type]++;
      par.type_mask <<= 2; par.type_mask |= (u32)sen.type;
      M.sen_index++; sentence_clear(M.sentences[M.sen_index & 3]);
      M.masks[3] += 3;
      skip = true;
      stage = 2;
    }
    if (stage == 2) {
      if (c == ',') {
        M.commas++;
        M.state = TP_AfterComma;
        M.parse_ctx = hash(sx(M.state), (u64)ilog2(M.quote_length + 1), (u64)ilog2(M.last_newline), (u64)(M.last_upper < M.last_letter + M.word_length[1]));
      } else if (c == ':') word_copy(M.topic, P8_PW);
      if (!skip) { tsen(M, 0).segment_count++; M.masks[3] += 4; }
      M.last_punct = 0; M.prev_punct = c;
      M.masks[0] += 3; M.masks[1] += 2; M.masks[2] += 15;
      M.seg_index++;
      Segment& ns = M.segments[M.seg_index & 3];
      ns.first_word.clear(); ns.word_count = ns.num_count = 0;
    }
    if (stage == 3) {
      M.prev_newline = M.last_newline; M.last_newline = 0;
      M.commas = 0;
      if (M.prev_newline == 1 || (M.prev_newline == 2 && pC == 0x0D)) {
        M.par_index++;
        Paragraph& np = M.paragraphs[M.par_index & 1];
        np.sentence_count = 0; np.type_count[0] = np.type_count[1] = np.type_count[2] = 0; np.type_mask = 0;
      } else if ((M.last_letter == 2 && pC == '+') || (M.last_letter == 3 && pC == 0x0D && buf(S, 3) == '+')) {
        M.parse_ctx = hash(sx(TP_ReadingWord), P8_PW.hash[1]); M.state = TP_PossibleHyphenation;
      }
      stage = 4;
    }
    if (stage == 4) {
      M.space_count++; M.spaces |= 1;
      M.masks[1] += 3; M.masks[3] += 5;
      if (c == 0x20 && M.pstate == TP_WasAbbreviation) { M.state = TP_AfterAbbreviation; M.parse_ctx = hash(sx(M.state), P8_PW.hash[1]); }
    }
    if (c >= '0' && c <= '9') {
      M.numbers[0] = M.numbers[0] * 10 + (c & 0xF); M.num_length[0] = (u8)imin(19, M.num_length[0] + 1);
      M.num_hashes[0] = combine64(M.num_hashes[0], c);
      M.expected_digit = (u8)-1;
      if (M.num_length[0] < M.num_length[1] && (M.pstate == TP_ExpectDigit || ((M.num_diff & 3) == 0 && M.num_length[0] <= 1))) {
        const u64 expected = M.numbers[1] + (M.num_mask & 3) - 2;
        u64 place = 1;
        for (int i = 0; i < M.num_length[1] - M.num_length[0]; ++i, place *= 10);
        if (expected / place == M.numbers[0]) {
          place /= 10;
          M.expected_digit = (u8)((expected / place) % 10);
          M.state = TP_ExpectDigit;
        }
      } else {
        const u8 d = (u8)buf(S, M.num_length[0] + 2);
        if (M.num_length[0] < 3 && buf(S, M.num_length[0] + 1) == ',' && d >= '0' && d <= '9') M.state = TP_ExpectDigit;
      }
      M.last_digit = 0;
      M.masks[3] += 7;
    } else if (M.numbers[0] > 0) {
      M.num_mask <<= 2; M.num_mask |= 1 + (M.numbers[0] >= M.numbers[1]) + (M.numbers[0] > M.numbers[1]);
      M.num_diff <<= 2; M.num_diff |= umin(3, ilog2((u32)iabs((int)(M.numbers[0] - M.numbers[1]))));
      M.numbers[1] = M.numbers[0]; M.numbers[0] = 0;
      M.num_hashes[1] = M.num_hashes[0]; M.num_hashes[0] = 0;
      M.num_length[1] = M.num_length[0]; M.num_length[0] = 0;
      tseg(M, 0).num_count++; tsen(M, 0).num_count++;
    }
  }
P8_COLD P8_HD inline void text_tail(State& S, u8 c) {
  TextM& M = S.text;
  if (M.last_newline == 1) M.first_char = (M.lang_id != LANG_UNKNOWN) ? c : (u8)imin(c, 96);
  if (M.last_nest > 512) M.nest_hash = 0;
  int lead = 0;
  while (((c >> (7 - lead)) & 1) != 0) lead++;
  if (M.utf8_remaining > 0 && lead == 1) M.utf8_remaining--;
  else M.utf8_remaining = (lead != 1) ? (c != 0xC0 && c != 0xC1 && c < 0xF5) ? (lead - (lead > 0)) : -1 : 0;
  const u32* bp = M.byte_pos;
  M.mask_punct = (u32)(bp[','] > bp['.']) | ((u32)(bp[','] > bp['!']) << 1) | ((u32)(bp[','] > bp['?']) << 2) | ((u32)(bp[','] > bp[':']) << 3) | ((u32)(bp[','] > bp[';']) << 4);
  S.st_text_first = M.first_letter;
  S.st_text_mask = (u8)(M.masks[1] & 0xFF);
}
P8_COLD P8_HD inline int text_update_a(State& S) {
  const Tables& T = *S.T;
  TextM& M = S.text;
  M.last_upper = umin(0xFF, M.last_upper + 1); M.mask_upper <<= 1;
  M.last_letter = umin(0x1F, M.last_letter + 1);
  M.last_digit = umin(0xFF, M.last_digit + 1);
  M.last_punct = umin(0x3F, M.last_punct + 1);
  M.last_newline++; M.prev_newline++; M.last_nest++;
  M.space_count -= (M.spaces >> 31); M.spaces <<= 1;
  M.masks[0] <<= 2; M.masks[1] <<= 2; M.masks[2] <<= 4; M.masks[3] <<= 3;
  M.pstate = M.state;
  u8 c = (u8)buf(S, 1), pC = (u8)lower(c);
  const u8 g = (c < 0x80) ? T.ascii_group[c] : 31;
  if (!((g <= 4) && g == (M.ascii_mask & 0x1f))) M.ascii_mask = ((M.ascii_mask << 5) | g) & ((1ull << 60) - 1);
  M.masks[4] = (u32)(M.ascii_mask & ((1u << 30) - 1));
  M.byte_pos[c] = (u32)S.pos;
  if (c != pC) { c = pC; M.last_upper = 0; M.mask_upper |= 1; }
  pC = (u8)buf(S, 2);
  M.state = TP_Unknown;
  M.parse_ctx = hash(sx(M.state), P8_PW.hash[1], c, (u64)((ilog2(M.last_newline) + 1) * (M.last_newline * 3 > M.prev_newline)), (u64)(M.masks[1] & 0xFC));
  if ((c >= 'a' && c <= 'z') || c == '\'' || c == '-' || c > 0x7F) {
    if (M.word_length[0] == 0) {
      if (pC == 0x0A && ((M.last_letter == 3 && buf(S, 3) == '+') || (M.last_letter == 4 && buf(S, 3) == 0x0D && buf(S, 4) == '+'))) {
        M.word_length[0] = M.word_length[1];
        for (int i = LANG_UNKNOWN; i < LANG_COUNT; ++i) M.words_index[i]--;
        // cWord = pWord, pWord = &Words[Lang.pId](1): as (lang, i) pairs relative to the decremented indices
        M.cw_lang = M.pw_lang; M.cw_slot = M.pw_slot;
        M.pw_lang = M.lang_pid; M.pw_slot = slot_of(M, M.lang_pid, 1);
        P8_CW.clear();
        for (u32 i = 0; i < M.word_length[0]; ++i) P8_CW.append(buf(S, (int)(M.word_length[0] - i + M.last_letter)));
        M.word_length[1] = P8_PW.len();
        tseg(M, 0).word_count--;
        tsen(M, 0).word_count--;
      } else { M.word_gap = M.last_letter; M.first_letter = c; }
    }
    M.last_letter = 0;
    M.word_length[0]++;
    M.masks[0] += (M.lang_id != LANG_UNKNOWN) ? 1 + (u32)lang_vowel(M.lang_id, c) : 1; M.masks[1]++; M.masks[3] += M.masks[0] & 3;
    if (c == '\'') {
      M.masks[2] += 12;
      if (M.word_length[0] == 1) {
        if (M.quote_length == 0 && pC == 0x20) M.quote_length = 1;
        else if (M.quote_length > 0 && M.last_punct == 1) { M.quote_length = 0; M.state = TP_AfterQuote; M.parse_ctx = hash(sx(M.state), pC); }
      }
    }
    P8_CW.append(c);
    P8_CW.get_hashes();
    M.state = TP_ReadingWord;
    M.parse_ctx = hash(sx(M.state), P8_CW.hash[1]);
    text_tail(S, c);
    return 0;
  }
  if (P8_CW.len() > 0) {
    if (M.lang_id != LANG_UNKNOWN) word_copy(tw(M, LANG_UNKNOWN, 0), P8_CW);
    // The reference stems the German, French, English copy in this order, each copied from cWord right before (:3227-3236).
    // When cWord is itself the current word of list `split`, that list's stemmer rewrites it and the lists below copy
    // the rewritten word: they form a second round (text_stem_mid copies for them).
    const int split = (M.cw_slot == slot_of(M, M.cw_lang, 0)) ? M.cw_lang : 0;
    M.stem_split = (u8)split;
    for (int i = LANG_COUNT - 1; i > LANG_UNKNOWN; --i) {
      M.lang_count[i - 1] -= (u32)(M.lang_mask[i - 1] >> 63); M.lang_mask[i - 1] <<= 1;
      if (i >= split && i != M.lang_id) word_copy(tw(M, i, 0), P8_CW);
    }
    return 1;
  }
  text_else_rest(S, c, pC);
  text_tail(S, c);
  return 0;
}
P8_COLD P8_HD inline void text_stem(State& S, int i) {   // i = LANG_EN .. LANG_DE
  TextM& M = S.text;
  Word& w = tw(M, i, 0);
  M.stem_ok[i - 1] = (u8)(i == LANG_EN ? StemEN::stem(w) : i == LANG_FR ? StemFR::stem(w) : StemDE::stem(w));
}
P8_HD inline void text_stem_mid(State& S) {      // between the rounds: the lists below `split` copy the rewritten cWord
  TextM& M = S.text;
  for (int i = (int)M.stem_split - 1; i > LANG_UNKNOWN; --i)
    if (i != M.lang_id) word_copy(tw(M, i, 0), P8_CW);
}
P8_COLD P8_HD inline void text_update_b(State& S) {
  TextM& M = S.text;
  const u8 c = (u8)lower((u8)buf(S, 1)), pC = (u8)buf(S, 2);
  for (int i = LANG_COUNT - 1; i > LANG_UNKNOWN; --i)
    if (M.stem_ok[i - 1]) { M.lang_count[i - 1]++; M.lang_mask[i - 1] |= 1; }
  {
      M.lang_id = LANG_UNKNOWN;
      u32 best = 4;
      for (int i = LANG_COUNT - 1; i > LANG_UNKNOWN; --i) {
        if (M.lang_count[i - 1] >= best) { best = M.lang_count[i - 1] + (i == M.lang_pid); M.lang_id = i; }
        M.words_index[i]++;
      }
      M.words_index[LANG_UNKNOWN]++;
      M.lang_pid = M.lang_id;
      M.pw_lang = M.cw_lang = M.lang_id; M.pw_slot = slot_of(M, M.lang_id, 1); M.cw_slot = slot_of(M, M.lang_id, 0);
      P8_CW.clear();
      M.word_pos[P8_PW.hash[1] & 0xffff] = (u32)S.pos;
      Segment& seg = tseg(M, 0);
      Sentence& sen = tsen(M, 0);
      if (seg.word_count == 0) word_copy(seg.first_word, P8_PW);
      seg.word_count++;
      if (sen.word_count == 0) word_copy(sen.first_word, P8_PW);
      sen.word_count++;
      M.word_length[1] = M.word_length[0]; M.word_length[0] = 0;
      M.quote_length += (M.quote_length > 0);
      if (M.quote_length > 0x1F) M.quote_length = 0;
      sen.verb_index++; sen.noun_index++; sen.capital_index++;
      if ((P8_PW.type & W_Verb) != 0) { sen.verb_index = 0; word_copy(sen.last_verb, P8_PW); }
      if ((P8_PW.type & W_Noun) != 0) { sen.noun_index = 0; word_copy(sen.last_noun, P8_PW); }
      if (sen.word_count > 1 && M.last_upper < M.word_length[1]) { sen.capital_index = 0; word_copy(sen.last_capital, P8_PW); }
      }
  text_else_rest(S, c, pC);
  text_tail(S, c);
}
P8_HD inline void text_update(State& S) {
  if (text_update_a(S)) {
    const int split = S.text.stem_split;
    for (int i = LANG_COUNT - 1; i > LANG_UNKNOWN && i >= split; --i) text_stem(S, i);
    text_stem_mid(S);
    for (int i = split - 1; i > LANG_UNKNOWN; --i) text_stem(S, i);
    text_update_b(S);
  }
}

// The 33 contexts of the text model's history map (:3376-3515). Pure apart from the sets: with sel.lanes > 1 every lane of a warp walks
// the list and computes only its own contexts (k % lanes == lane); returns the new context count for the caller to store.
P8_HD inline int text_contexts(State& S, const CtxSel sel) {
  const Tables& T = *S.T;
  TextM& M = S.text;
  Cm2& map = M.map;
  const u8 c = (u8)buf(S, 1), lc = (u8)lower(c), m2 = (u8)(M.masks[2] & 0xF), column = (u8)umin(0xFF, M.last_newline);
  const Word& cw = P8_CW; const Word& pw = P8_PW;
  const u16 w = (u16)(((M.state == TP_ReadingWord) ? cw.hash[1] : pw.hash[1]) & 0xFFFF);
  const u32 h = (u32)(((M.state == TP_ReadingWord) ? cw.hash[1] : pw.hash[2]) * 271 + c);
  const u64 i0 = (u64)M.state << 6;
  int n = map.index;
  const Word& w2 = tw(M, M.lang_pid, 2); const Word& w3 = tw(M, M.lang_pid, 3);
  Sentence& sen = tsen(M, 0); Segment& seg = tseg(M, 0);
  const u32 wl0 = M.word_length[0], wl1 = M.word_length[1], gap = M.word_gap;
  P8_CM2_SET(sel, map, n, M.parse_ctx);
  P8_CM2_SET(sel, map, n, hash((i0 + 0), cw.hash[0], pw.hash[0], (u64)((M.last_upper < wl0) | ((M.last_digit < wl0 + gap) << 1))));
  P8_CM2_SET(sel, map, n, hash((i0 + 1), cw.hash[1], w2.hash[1], (u64)imin(10, (int)ilog2((u32)M.numbers[0])),
                    (u64)((M.last_upper < M.last_letter + wl1) | ((M.last_letter > 3) << 1) | ((M.last_letter > 0 && wl1 < 3) << 2))));
  P8_CM2_SET(sel, map, n, hash((i0 + 2), cw.hash[1] & 0xFFF, (u64)(M.masks[1] & 0x3FF), w3.hash[2],
                    (u64)((M.last_digit < wl0 + gap) | ((M.last_upper < M.last_letter + wl1) << 1) | ((M.spaces & 0x7F) << 2))));
  P8_CM2_SET(sel, map, n, hash((i0 + 3), cw.hash[1], pw.hash[3], w2.hash[3]));
  P8_CM2_SET(sel, map, n, hash((i0 + 4), (u64)(h & 0x7FFF), w2.hash[1] & 0xFFF, w3.hash[1] & 0xFFF));
  P8_CM2_SET(sel, map, n, hash((i0 + 5), cw.hash[1], c, (sen.verb_index < sen.word_count) ? sen.last_verb.hash[1] : 0));
  P8_CM2_SET(sel, map, n, hash((i0 + 6), pw.hash[2], (u64)(M.masks[1] & 0xFC), lc, gap));
  P8_CM2_SET(sel, map, n, hash((i0 + 7), (M.last_letter == 0) ? cw.hash[1] : pw.hash[1], c, seg.first_word.hash[2], (u64)imin(3, (int)ilog2(seg.word_count + 1))));
  P8_CM2_SET(sel, map, n, hash((i0 + 8), cw.hash[1], c, tseg(M, 1).first_word.hash[3]));
  P8_CM2_SET(sel, map, n, hash((i0 + 9), (u64)imax(31, lc), (u64)(M.masks[1] & 0xFFC), (u64)((M.spaces & 0xFE) | (M.last_punct < M.last_letter)),
                    (u64)((M.mask_upper & 0xFF) | (((0x100 | M.first_letter) * (wl0 > 1)) << 8))));
  P8_CM2_SET(sel, map, n, hash((i0 + 10), column, (u64)imin(7, (int)ilog2(M.last_upper + 1)), (u64)ilog2(M.last_punct + 1)));
  P8_CM2_SET(sel, map, n, (u64)(u32)((column & 0xF8) | (M.masks[1] & 3) | ((M.prev_newline - M.last_newline > 63) << 2) | (umin(3, M.last_letter) << 8) | ((u32)M.first_char << 10) |
                          ((M.commas > 4) << 18) | ((m2 >= 1 && m2 <= 5) << 19) | ((m2 >= 6 && m2 <= 10) << 20) | ((m2 == 11 || m2 == 12) << 21) |
                          ((M.last_upper < column) << 22) | ((M.last_digit < column) << 23) | ((column < M.prev_newline - M.last_newline) << 24)));
  P8_CM2_SET(sel, map, n, hash((u64)((2 * column) / 3), (u64)(umin(13, M.last_punct) + (M.last_punct > 16) + (M.last_punct > 32) + M.mask_punct * 16), (u64)ilog2(M.last_upper + 1),
                    (u64)ilog2(M.prev_newline - M.last_newline), (u64)(((M.masks[1] & 3) == 0) | ((m2 < 6) << 1) | ((m2 < 11) << 2))));
  P8_CM2_SET(sel, map, n, hash((i0 + 11), (u64)(column >> 1), (u64)(M.spaces & 0xF)));
  P8_CM2_SET(sel, map, n, hash((u64)(M.masks[3] & 0x3F), (u64)imin((imax((int)wl0, 3) - 2) * (wl0 < 8), 3), (u64)(M.first_letter * (wl0 < 5)), (u64)(w & 0x3FF),
                    (u64)((c == buf(S, 2)) | ((M.masks[2] > 0) << 1) | ((M.last_punct < wl0 + gap) << 2) | ((M.last_upper < wl0) << 3) | ((M.last_digit < wl0 + gap) << 4) |
                          ((M.last_punct < 2 + wl0 + gap + wl1) << 5))));
  P8_CM2_SET(sel, map, n, hash((i0 + 12), w, c, M.num_hashes[1]));
  P8_CM2_SET(sel, map, n, hash((i0 + 13), w, c, (u64)(llog(T, (u32)S.pos - M.word_pos[w]) >> 1)));
  P8_CM2_SET(sel, map, n, hash((i0 + 14), w, c, M.topic.hash[1] & 0x7FFF));
  P8_CM2_SET(sel, map, n, hash((i0 + 15), M.num_length[0], c, M.topic.hash[1] & 0x7FFF));
  P8_CM2_SET(sel, map, n, hash((i0 + 16), (u64)((M.last_letter > 0) ? c : 0x100), (u64)(M.masks[1] & 0xFFC), (u64)(M.nest_hash & 0x7FF)));
  P8_CM2_SET(sel, map, n, hash((i0 + 17), (u64)(u32)((u32)w * 17 + c), (u64)(M.masks[3] & 0x1FF),
                    (u64)(((sen.verb_index == 0 && sen.last_verb.len() > 0) << 6) | ((wl1 > 3) << 5) | ((seg.word_count == 0) << 4) |
                          ((sen.segment_count == 0 && sen.word_count < 2) << 3) | ((M.last_punct >= M.last_letter + wl1 + gap) << 2) |
                          ((M.last_upper < M.last_letter + wl1) << 1) | (M.last_upper < wl0 + gap + wl1))));
  P8_CM2_SET(sel, map, n, hash((i0 + 18), c, pw.hash[2], (u64)(M.first_letter * (wl0 < 6)), (u64)(((M.last_punct < wl0 + gap) << 1) | (M.last_punct >= M.last_letter + wl1 + gap))));
  {
    const Word& wx = tw(M, M.lang_pid, 1 + (wl0 == 0));
    P8_CM2_SET(sel, map, n, hash((i0 + 19), (u64)(u32)((u32)w * 23 + c), wx.L[wx.s], (u64)(M.first_letter * (wl0 < 7))));
  }
  P8_CM2_SET(sel, map, n, hash((i0 + 20), column, (u64)(M.spaces & 7), (u64)(M.nest_hash & 0x7FF)));
  P8_CM2_SET(sel, map, n, hash((i0 + 21), cw.hash[1], (u64)((M.last_upper < column) | ((M.last_upper < wl0) << 1)), (u64)umin(5, wl0)));
  P8_CM2_SET(sel, map, n, M.masks[4]);
  P8_CM2_SET(sel, map, n, hash((u64)(u32)M.ascii_mask, (u64)(u32)(M.ascii_mask >> 32)));
  P8_CM2_SET(sel, map, n, M.ascii_mask & ((1 << 20) - 1));
  P8_CM2_SET(sel, map, n, M.ascii_mask & ((1 << 10) - 1));
  P8_CM2_SET(sel, map, n, hash((M.ascii_mask >> 5) & ((1 << 30) - 1), (u64)buf(S, 1)));
  P8_CM2_SET(sel, map, n, hash((M.ascii_mask >> 10) & ((1 << 30) - 1), (u64)buf(S, 1), (u64)buf(S, 2)));
  P8_CM2_SET(sel, map, n, hash((M.ascii_mask >> 15) & ((1 << 30) - 1), (u64)buf(S, 1), (u64)buf(S, 2), (u64)buf(S, 3)));
  return n;
}

P8_HD inline void text_select(State& S);
P8_HD inline void text_bit(State& S, Out& o) {
  TextM& M = S.text;
  if (S.bpos == 0) {
    text_update(S);
    M.map.index = text_contexts(S, CtxSel{0, 1});
  }
  cm2_mix(M.map, o, S.y, S.bpos);
  text_select(S);
}
P8_HD inline void text_select(State& S) {   // the model's eight mixer selector sets (:3166-3185)
  TextM& M = S.text;
  const int c0 = S.c0;
  const u32 wl0 = M.word_length[0], wl1 = M.word_length[1], gap = M.word_gap;
  const Word& pw = P8_PW;
  Mixer& m = S.m;
  mset(m, (int)finalize64(hash((u64)((M.lang_id != LANG_UNKNOWN) ? 1 + (int)lang_vowel(M.lang_id, buf(S, 1)) : 0), (u64)(M.masks[1] & 0xFF), (u64)c0), 11), 2048);
  mset(m, (int)finalize64(hash((u64)ilog2(wl0 + 1), (u64)c0,
                               (u64)((M.last_digit < wl0 + gap) | ((M.last_upper < M.last_letter + wl1) << 1) | ((M.last_punct < wl0 + gap) << 2) | ((M.last_upper < wl0) << 3))), 11), 2048);
  mset(m, (int)finalize64(hash((u64)(M.masks[1] & 0x3FF), S.grp0, (u64)(M.last_upper < wl0), (u64)(M.last_upper < M.last_letter + wl1)), 12), 4096);
  mset(m, (int)finalize64(hash((u64)(M.spaces & 0x1FF), S.grp0,
                               (u64)((M.last_upper < wl0) | ((M.last_upper < M.last_letter + wl1) << 1) | ((M.last_punct < M.last_letter) << 2) | ((M.last_punct < wl0 + gap) << 3) |
                                     ((M.last_punct < M.last_letter + wl1 + gap) << 4))), 12), 4096);
  mset(m, (int)finalize64(hash((u64)(M.first_letter * (wl0 < 4)), (u64)umin(6, wl0), (u64)c0), 11), 2048);
  mset(m, (int)finalize64(hash(pw.at(0), pw.rat(0), (u64)umin(4, wl0), (u64)(M.last_punct < M.last_letter)), 11), 2048);
  mset(m, (int)finalize64(hash((u64)umin(4, wl0), S.grp0, (u64)(M.last_upper < wl0),
                               (u64)((M.nest_hash > 0) ? M.nest_hash & 0xFF : 0x100 | (M.first_letter * (wl0 > 0 && wl0 < 4)))), 12), 4096);
  mset(m, (int)finalize64(hash(S.grp0, (u64)(M.masks[4] & 0x1F), (u64)((M.masks[4] >> 5) & 0x1F)), 13), 8192);
}

// ---------------------------------------------------------------- x86 model (:7100-7546)
enum { fNM = 0, fAM = 1, fMR = 2, fMEXTRA = 3, fMODE = 3, fNI = 0, fBI = 4, fWI = 8, fDI = 0xc, fTYPE = 0xc, fAD = 0, fDA = 4, fBR = 8, fDR = 0xc, fERR = 0xf };
enum { XS_Start, XS_PrefOpSize, XS_PrefMultiByte, XS_ParseFlags, XS_ExtraFlags, XS_ReadModRM, XS_ReadOP3_38, XS_ReadOP3_3A, XS_ReadSIB, XS_Read8, XS_Read16, XS_Read32,
       XS_Read8ModRM, XS_Read16f, XS_Read32ModRM, XS_Error };
enum : u32 { X_CodeShift = 3, X_CodeMask = 0xFFu << 3, X_PrefixMask = 7, X_OperandSizeOverride = 1u << 11, X_MultiByteOpcode = 2u << 11, X_PrefixREX = 4u << 11,
             X_Prefix38 = 8u << 11, X_Prefix3A = 0x10u << 11, X_HasExtraFlags = 0x20u << 11, X_HasModRM = 0x40u << 11, X_ModRMShift = 18, X_SIBScaleShift = 20,
             X_RegDWordDisplacement = 1u << 28, X_AddressMode = 2u << 28, X_TypeShift = 30, X_CategoryShift = 5, X_CategoryMask = 31 };
#define X_ClearCodeMask (0xFFFFFFFFu ^ X_CodeMask)
P8_HD inline void instr_clear(Instr& op) { op.data = 0; op.prefix = op.code = op.modrm = op.sib = op.rex = op.flags = op.bytes_read = op.size = op.category = 0; op.must_check_rex = op.decoding = op.o16 = op.imm8 = 0; }
P8_HD inline void exe_mode(Instr& op, int& st) {   // ProcessMode (:7155-7198)
  if ((op.flags & fMODE) == fAM) {
    op.data |= X_AddressMode;
    op.bytes_read = 0;
    switch (op.flags & fTYPE) {
      case fDR: op.data |= (2u << X_TypeShift);   // falls through
      case fDA: op.data |= (1u << X_TypeShift);   // falls through
      case fAD: st = XS_Read32; break;
      case fBR: op.data |= (2u << X_TypeShift); st = XS_Read8;
    }
  } else {
    switch (op.flags & fTYPE) {
      case fBI: st = XS_Read8; break;
      case fWI: st = XS_Read16; op.data |= (1u << X_TypeShift); op.bytes_read = 0; break;
      case fDI:
        op.imm8 = ((op.rex & 0x08) > 0 && (op.code & 0xF8) == 0xB8);
        if (!op.o16 || op.imm8) { st = XS_Read32; op.data |= (2u << X_TypeShift); }
        else { st = XS_Read16; op.data |= (3u << X_TypeShift); }
        op.bytes_read = 0;
        break;
      default: st = XS_Start;
    }
  }
}
P8_HD inline void exe_flags2(Instr& op, int& st) { if ((op.flags & fMODE) == fMR && st != XS_ExtraFlags) { st = XS_ReadModRM; return; } exe_mode(op, st); }
P8_HD inline void exe_flags(Instr& op, int& st) { if (op.code == 0x9a || op.code == 0xea || op.code == 0xc8) { op.bytes_read = 0; st = XS_Read16f; return; } exe_flags2(op, st); }
P8_HD inline void exe_check(Instr& op, int& st) {
  if (op.flags == fMEXTRA) st = XS_ExtraFlags;
  else if (op.flags == fERR) { instr_clear(op); st = XS_Error; }
  else exe_flags(op, st);
}
P8_HD inline void exe_modrm(Instr& op, int& st) {
  if ((op.modrm & 0xC0) == 0x40) st = XS_Read8ModRM;
  else if ((op.modrm & 0xC0) == 0x80 || (op.modrm & (0xC0 | 0x07)) == 0x05 || (op.modrm < 0x40 && (op.sib & 0x07) == 0x05)) { st = XS_Read32ModRM; op.bytes_read = 0; }
  else exe_mode(op, st);
}
P8_HD inline int exe_pref(const State& S, int i) { return (buf(S, i) == 0x0f) + 2 * (buf(S, i) == 0x66) + 3 * (buf(S, i) == 0x67); }
P8_HD inline u32 exe_cxt(const State& S, int i, int x) {   // execxt (:7263-7271)
  int prefix = 0, opcode = 0, modrm = 0, sib = 0;
  if (i) prefix += 4 * exe_pref(S, i--);
  if (i) prefix += exe_pref(S, i--);
  if (i) opcode += buf(S, i--);
  if (i) modrm += buf(S, i--) & (0xC0 | 0x07);
  if (i && ((modrm & 0x07) == 4) && (modrm < 0xC0)) sib = buf(S, i) & 0xC0;
  return (u32)(prefix | opcode << 4 | modrm << 12 | x << 20 | sib << (28 - 6));
}
P8_HD inline u32 exe_opn(const ExeM& M, u32 n) { return M.cache[(M.cache_index - n) & 31]; }
P8_COLD P8_HD inline void exe_byte(State& S) {
  const Tables& T = *S.T;
  ExeM& M = S.exe;
  Instr& op = M.op;
  int st = M.state;
  M.pstate = st;
  const u8 B = (u8)S.c4;
  op.size++;
  switch (st) {
    case XS_Start: case XS_Error: {
      bool skip = false, done = false;
      if (op.must_check_rex) {
        op.must_check_rex = 0;
        bool invalid = false, prefix = false;
        for (int i = 0; i < 19; ++i) if (B == T.exe_invalid64[i]) invalid = true;
        for (int i = 0; i < 8; ++i) if (B == T.exe_prefix64[i]) prefix = true;
        prefix = prefix || (B >= 0x40 && B <= 0x4F) || (B >= 0x64 && B <= 0x67);
        if (!invalid && !prefix) {
          op.rex = op.code;
          op.code = B;
          op.data = X_PrefixREX | ((u32)op.code << X_CodeShift) | (op.data & X_PrefixMask);
          skip = true;
        }
      }
      op.modrm = op.sib = op.rex = op.flags = op.bytes_read = 0;
      if (!skip) {
        op.code = B;
        op.must_check_rex = ((op.code & 0xF0) == 0x40) && (!(op.decoding && ((op.data & X_PrefixMask) == 1)));
        op.prefix = (u8)((op.code == 0x26 || op.code == 0x2E || op.code == 0x36 || op.code == 0x3E) + (op.code == 0x64) * 2 + (op.code == 0x65) * 3 + (op.code == 0x67) * 4 +
                         (op.code == 0x9B) * 5 + (op.code == 0xF0) * 6 + (op.code == 0xF2 || op.code == 0xF3) * 7);
        if (!op.decoding) {
          M.total_ops += (u32)((op.data != 0) - (M.cache_index && M.cache[M.cache_index & 31] != 0));
          M.op_mask = (M.op_mask << 1) | (u32)(st != XS_Error);
          M.op_categ_mask = (M.op_categ_mask << X_CategoryShift) | op.category;
          op.size = 0;
          M.cache[M.cache_index & 31] = op.data;
          M.cache_index++;
          if (!op.prefix) op.data = (u32)op.code << X_CodeShift;
          else {
            op.data = op.prefix;
            op.category = T.exe_c1[op.code];
            op.decoding = 1;
            M.brk_point = 0; M.brk_ctx = (u32)hash(1 + 0, op.prefix, (u64)(M.op_categ_mask & X_CategoryMask));
            done = true;
          }
        } else {
          if (!op.prefix) { op.data |= ((u32)op.code << X_CodeShift); op.decoding = 0; }
          else {
            op.data = op.prefix;
            op.category = T.exe_c1[op.code];
            M.brk_point = 1; M.brk_ctx = (u32)hash(1 + 1, op.prefix, (u64)(M.op_categ_mask & X_CategoryMask));
            done = true;
          }
        }
      }
      if (done) break;
      if ((op.o16 = (op.code == 0x66))) st = XS_PrefOpSize;
      else if (op.code == 0x0f) st = XS_PrefMultiByte;
      else { op.flags = T.exe_t1[op.code]; op.category = T.exe_c1[op.code]; exe_check(op, st); }
      M.brk_point = 2;
      M.brk_ctx = (u32)hash(1 + 2, sx(st), op.code, (u64)(M.op_categ_mask & X_CategoryMask), (u64)(exe_opn(M, 1) & ((0xC0u | 0x38u | 0x07u) << X_ModRMShift)));
      break;
    }
    case XS_PrefOpSize:
      op.code = B;
      op.data &= X_ClearCodeMask; op.data |= ((u32)op.code << X_CodeShift) | X_OperandSizeOverride;
      op.flags = T.exe_t1[op.code]; op.category = T.exe_c1[op.code]; exe_check(op, st);
      M.brk_point = 3; M.brk_ctx = (u32)hash(1 + 3, sx(st));
      break;
    case XS_PrefMultiByte:
      op.code = B;
      op.data |= X_MultiByteOpcode;
      if (op.code == 0x38) st = XS_ReadOP3_38;
      else if (op.code == 0x3A) st = XS_ReadOP3_3A;
      else {
        op.data &= X_ClearCodeMask; op.data |= ((u32)op.code << X_CodeShift);
        op.flags = T.exe_t2[op.code]; op.category = T.exe_c2[op.code];
        exe_check(op, st);
      }
      M.brk_point = 4; M.brk_ctx = (u32)hash(1 + 4, sx(st));
      break;
    case XS_ParseFlags:
      exe_flags(op, st);
      M.brk_point = 5; M.brk_ctx = (u32)hash(1 + 5, sx(st));
      break;
    case XS_ExtraFlags: case XS_ReadModRM: {
      op.modrm = B;
      op.data |= ((u32)op.modrm << X_ModRMShift) | X_HasModRM;
      op.sib = 0;
      if (op.flags == fMEXTRA) {
        op.data |= X_HasExtraFlags;
        const int i = ((op.modrm >> 3) & 0x07) | ((op.code & 0x01) << 3) | ((op.code & 0x08) << 1);
        op.flags = T.exe_tx[i];
        op.category = T.exe_cx[i];
        if (op.flags == fERR) { instr_clear(op); st = XS_Error; M.brk_point = 6; M.brk_ctx = (u32)hash(1 + 6, sx(st)); break; }
        exe_flags(op, st);
        M.brk_point = 7; M.brk_ctx = (u32)hash(1 + 7, sx(st));
        break;
      }
      if ((op.modrm & 0x07) == 4 && op.modrm < 0xC0) { st = XS_ReadSIB; M.brk_point = 8; M.brk_ctx = (u32)hash(1 + 8, sx(st)); break; }
      exe_modrm(op, st);
      M.brk_point = 9; M.brk_ctx = (u32)hash(1 + 9, sx(st), op.code);
      break;
    }
    case XS_ReadOP3_38: case XS_ReadOP3_3A:
      op.code = B;
      op.data &= X_ClearCodeMask; op.data |= ((u32)op.code << X_CodeShift) | (X_Prefix38 << (st - XS_ReadOP3_38));
      if (st == XS_ReadOP3_38) { op.flags = T.exe_t3_38[op.code]; op.category = T.exe_c3_38[op.code]; }
      else { op.flags = T.exe_t3_3a[op.code]; op.category = T.exe_c3_3a[op.code]; }
      exe_check(op, st);
      M.brk_point = 10; M.brk_ctx = (u32)hash(1 + 10, sx(st));
      break;
    case XS_ReadSIB:
      op.sib = B;
      op.data |= ((u32)(op.sib & 0xC0) << X_SIBScaleShift);
      exe_modrm(op, st);
      M.brk_point = 11; M.brk_ctx = (u32)hash(1 + 11, sx(st), (u64)(op.sib & 0xC0));
      break;
    case XS_Read8: case XS_Read16: case XS_Read32:
      if (++op.bytes_read >= ((2 * (st - XS_Read8)) << op.imm8)) { op.bytes_read = 0; op.imm8 = 0; st = XS_Start; }
      M.brk_point = 12;
      M.brk_ctx = (u32)hash(1 + 12, sx(st), (u64)(op.flags & fMODE), op.bytes_read, (u64)(((op.bytes_read > 1) ? (buf(S, op.bytes_read) << 8) : 0) | ((op.bytes_read) ? B : 0)));
      break;
    case XS_Read8ModRM:
      exe_mode(op, st);
      M.brk_point = 13; M.brk_ctx = (u32)hash(1 + 13, sx(st));
      break;
    case XS_Read16f:
      if (++op.bytes_read == 2) { op.bytes_read = 0; exe_flags2(op, st); }
      M.brk_point = 14; M.brk_ctx = (u32)hash(1 + 14, sx(st));
      break;
    case XS_Read32ModRM:
      op.data |= X_RegDWordDisplacement;
      if (++op.bytes_read == 4) { op.bytes_read = 0; exe_mode(op, st); }
      M.brk_point = 15; M.brk_ctx = (u32)hash(1 + 15, sx(st));
      break;
  }
  M.state = st;
  M.valid = (M.total_ops > 2 * 8) && ((M.op_mask & 0xFF) == 0xFF);
  M.context = (u32)(st + 16 * op.bytes_read + 16 * (op.rex & 0x08));
  M.state_bh[M.context] = (M.state_bh[M.context] << 8) | B;
  // Forced: the contexts are always set (exeModel(m, true, Stats), :8184)
  Cm2& cm = M.cm;
  int mask = 0, count0 = 0, i = 0;
  for (int j = 0; i < 10; ++i) {
    if (i > 1) { mask = mask * 2 + (buf(S, i - 1) == 0); count0 += mask & 1; }
    j = (i < 4) ? i + 1 : 5 + (i - 4) * (2 + (i > 6));
    cm2_set(cm, hash(sx(i), exe_cxt(S, j, buf(S, 1) * (j > 6)), sx(((1 << 10) | mask) * (count0 * 10 / 2 >= i)), sx((0x08 | (S.blpos & 0x07)) * (i < 4))));
  }
  cm2_set(cm, M.brk_ctx);
  u32 mk = X_PrefixMask | (0xF8u << X_CodeShift) | X_MultiByteOpcode | X_Prefix38 | X_Prefix3A;
  const int stb = st + 16 * op.bytes_read;
  cm2_set(cm, hash(sx(++i), (u64)(exe_opn(M, 1) & (mk | X_RegDWordDisplacement | X_AddressMode)), sx(stb), (u64)(op.data & mk), op.rex, op.category));
  mk = 0x04 | (0xFEu << X_CodeShift) | X_MultiByteOpcode | X_Prefix38 | X_Prefix3A | ((0xC0u | 0x38u) << X_ModRMShift);
  cm2_set(cm, hash(sx(++i), (u64)(exe_opn(M, 1) & mk), (u64)(exe_opn(M, 2) & mk), (u64)(exe_opn(M, 3) & mk), (u64)(M.context + 256 * ((op.modrm & 0xC0) == 0xC0)),
                   (u64)(op.data & ((mk | X_PrefixREX) ^ (0xC0u << X_ModRMShift)))));
  mk = 0x04 | X_CodeMask;
  cm2_set(cm, hash(sx(++i), (u64)(exe_opn(M, 1) & mk), (u64)(exe_opn(M, 2) & mk), (u64)(exe_opn(M, 3) & mk), (u64)(exe_opn(M, 4) & mk),
                   (u64)((op.data & mk) | ((u32)st << 11) | ((u32)op.bytes_read << 15))));
  mk = 0x04 | (0xFCu << X_CodeShift) | X_MultiByteOpcode | X_Prefix38 | X_Prefix3A;
  cm2_set(cm, hash(sx(++i), sx(stb), (u64)(op.data & mk), (u64)(op.category * 8 + (M.op_mask & 0x07)), op.flags,
                   (u64)(((op.sib & 0x07) == 5) * 4 + ((op.modrm & 0x38) == 0x38) * 2 + ((op.modrm & 0xC0) == 0))));
  mk = X_PrefixMask | X_CodeMask | X_OperandSizeOverride | X_MultiByteOpcode | X_PrefixREX | X_Prefix38 | X_Prefix3A | X_HasExtraFlags | X_HasModRM | ((0xC0u | 0x07u) << X_ModRMShift);
  cm2_set(cm, hash(sx(++i), (u64)(op.data & mk), sx(stb), op.flags));
  mk = X_PrefixMask | X_CodeMask | X_OperandSizeOverride | X_MultiByteOpcode | X_Prefix38 | X_Prefix3A | X_HasExtraFlags | X_HasModRM;
  cm2_set(cm, hash(sx(++i), (u64)(exe_opn(M, 1) & mk), sx(st), (u64)(op.bytes_read * 2 + ((op.rex & 0x08) > 0)), (u64)(op.data & ((u16)(mk ^ X_OperandSizeOverride)))));
  mk = 0x04 | (0xFEu << X_CodeShift) | X_MultiByteOpcode | X_Prefix38 | X_Prefix3A | (0x38u << X_ModRMShift);
  cm2_set(cm, hash(sx(++i), (u64)(exe_opn(M, 1) & mk), (u64)(exe_opn(M, 2) & mk), sx(stb), (u64)(op.data & (mk | X_PrefixMask | X_CodeMask))));
  cm2_set(cm, hash(sx(++i), sx(stb)));
  cm2_set(cm, hash(sx(++i), (u64)((0x100 | B) * (op.bytes_read > 0)), sx(st + 16 * M.pstate + 256 * op.bytes_read),
                   (u64)(((op.flags & fMODE) == fAM) * 16 + (op.rex & 0x08) + (op.o16) * 4 + ((op.code & 0xFE) == 0xE8) * 2 + ((op.data & X_MultiByteOpcode) != 0 && (op.code & 0xF0) == 0x80))));
}
P8_HD inline void exe_select(State& S);
P8_HD inline void exe_bit(State& S, Out& o) {
  ExeM& M = S.exe;
  if (S.bpos == 0) exe_byte(S);
  cm2_mix(M.cm, o, S.y, S.bpos);
  exe_select(S);
}
P8_HD inline void exe_select(State& S) {   // selector sets and ModelStats (:7526-7545)
  ExeM& M = S.exe;
  const int bpos = S.bpos, c0 = S.c0, st = M.state;
  const Instr& op = M.op;
  const u32 bh = M.state_bh[M.context];
  const u8 s = (u8)(((bh >> (28 - bpos)) & 0x08) | ((bh >> (21 - bpos)) & 0x04) | ((bh >> (14 - bpos)) & 0x02) | ((bh >> (7 - bpos)) & 0x01) |
                    ((op.category == 12) << 4) | (((c0 & ((1 << bpos) - 1)) == 0) << 5));
  Mixer& m = S.m;
  mset(m, (int)(M.context * 4 + (s >> 4)), 1024);
  mset(m, st * 64 + bpos * 8 + (op.bytes_read > 0) * 4 + (s >> 4), 1024);
  mset(m, (int)((M.brk_ctx & 0x1FF) | ((u32)(s & 0x20) << 4)), 1024);
  mset(m, (int)finalize64(hash(op.code, sx(st), (u64)(exe_opn(M, 1) & X_CodeMask)), 13), 8192);
  mset(m, (int)finalize64(hash(sx(st), sx(bpos), op.code, op.bytes_read), 13), 8192);
  mset(m, (int)finalize64(hash(sx(st), sx((bpos << 2) | (c0 & 3)), (u64)(M.op_categ_mask & X_CategoryMask),
                               (u64)(((op.category == 12) << 2) | (((op.flags & fMODE) == fAM) << 1) | (op.bytes_read > 0))), 13), 8192);
  S.st_x86 = (u32)M.valid | (M.context << 1) | ((u32)s << 9);
}

// ---------------------------------------------------------------- linear prediction (:4476-4502) with OLS<double,U8>(32, 4, 0.995) (:1363-1466)
// ols block layout per predictor k (stride OLS_STRIDE doubles): x[32], w[32], b[32], cov[32][32], chol[32][32]
enum { OLS_N = 32, OLS_STRIDE = 3 * 32 + 2 * 32 * 32 };
#if defined(__CUDA_ARCH__)
#define P8_DMUL(a, b) __dmul_rn((a), (b))
#define P8_DADD(a, b) __dadd_rn((a), (b))
#define P8_DSUB(a, b) __dsub_rn((a), (b))
#define P8_DDIV(a, b) __ddiv_rn((a), (b))
#define P8_DSQRT(a) __dsqrt_rn(a)
#define P8_FLOOR(a) floor(a)
#else
// host: compiled without FMA contraction (g++ for baseline x86-64 has no FMA; tools/paq8_check.cpp adds -ffp-contract=off)
#define P8_DMUL(a, b) ((a) * (b))
#define P8_DADD(a, b) ((a) + (b))
#define P8_DSUB(a, b) ((a) - (b))
#define P8_DDIV(a, b) ((a) / (b))
#define P8_DSQRT(a) sqrt(a)
#define P8_FLOOR(a) floor(a)
#endif
// OLS<double, T>::Update(val) (:1453-1464) on a block x[n], w[n], b[n], cov[n][n], chol[n][n]: hasZeroMean, so sub = 0,
// nu = 0.001, ftol = 1e-8; a failed Factor() keeps w.
P8_HD inline void ols_update(double* blk, int n, int kmax, double lambda, int& km, double val) {
  const double nu = 0.001, one_minus = P8_DSUB(1.0, lambda);
  double* x = blk; double* w = blk + n; double* b = blk + 2 * n; double* cov = blk + 3 * n; double* ch = cov + n * n;
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < n; ++i) cov[j * n + i] = P8_DADD(P8_DMUL(lambda, cov[j * n + i]), P8_DMUL(one_minus, P8_DMUL(x[j], x[i])));
  for (int i = 0; i < n; ++i) b[i] = P8_DADD(P8_DMUL(lambda, b[i]), P8_DMUL(one_minus, P8_DMUL(x[i], val)));
  km++;
  if (km >= kmax) {
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) ch[i * n + j] = cov[i * n + j];
    for (int i = 0; i < n; ++i) ch[i * n + i] = P8_DADD(ch[i * n + i], nu);
    bool fail = false;
    for (int i = 0; i < n && !fail; ++i) {
      for (int j = 0; j < i; ++j) {
        double sum = ch[i * n + j];
        for (int k = 0; k < j; ++k) sum = P8_DSUB(sum, P8_DMUL(ch[i * n + k], ch[j * n + k]));
        ch[i * n + j] = P8_DDIV(sum, ch[j * n + j]);
      }
      double sum = ch[i * n + i];
      for (int k = 0; k < i; ++k) sum = P8_DSUB(sum, P8_DMUL(ch[i * n + k], ch[i * n + k]));
      if (sum > 1E-8) ch[i * n + i] = P8_DSQRT(sum); else fail = true;
    }
    if (!fail) {
      for (int i = 0; i < n; ++i) {
        double sum = b[i];
        for (int j = 0; j < i; ++j) sum = P8_DSUB(sum, P8_DMUL(ch[i * n + j], w[j]));
        w[i] = P8_DDIV(sum, ch[i * n + i]);
      }
      for (int i = n - 1; i >= 0; --i) {
        double sum = w[i];
        for (int j = i + 1; j < n; ++j) sum = P8_DSUB(sum, P8_DMUL(ch[j * n + i], w[j]));
        w[i] = P8_DDIV(sum, ch[i * n + i]);
      }
    }
    km = 0;
  }
}
P8_HD inline double ols_predict(const double* blk, int n) {   // OLS::Predict() (:1446-1452); the caller resets the tap index
  const double* x = blk; const double* w = blk + n;
  double sum = 0.;
  for (int i = 0; i < n; ++i) sum = P8_DADD(sum, P8_DMUL(w[i], x[i]));
  return sum;
}
P8_HD inline void linear_predict(State& S) {   // Add() the new taps and Predict() (after the three Update() calls)
  LinearM& M = S.linear;
  {
    const u8 W = (u8)buf(S, 1), WW = (u8)buf(S, 2), WWW = (u8)buf(S, 3);
    for (int i = 1; i <= 32; ++i) {
      const int idx[3] = {i, i * 2 - 1, i * 2};
      for (int k = 0; k < 3; ++k) if (M.ols_index[k] < OLS_N) M.ols[(size_t)k * OLS_STRIDE + M.ols_index[k]++] = (double)(u8)buf(S, idx[k]);
    }
    for (int k = 0; k < 3; ++k) {
      M.ols_index[k] = 0;
      const double f = P8_FLOOR(ols_predict(M.ols + (size_t)k * OLS_STRIDE, OLS_N));
      // Clip(int Px): the double is converted to int first (values far outside int range do not occur: |sum| < 2^20)
      M.prd[k] = (u8)clip8((int)f);
    }
    M.prd[3] = (u8)clip8(W * 2 - WW);
    M.prd[4] = (u8)clip8(W * 3 - WW * 3 + WWW);
  }
}
P8_HD inline void linear_small(State& S, Out& o, int i) {
  LinearM& M = S.linear;
  const u8 B = (u8)(S.c0 << (8 - S.bpos));
  scm_set(M.smap[i], (u32)((M.prd[i] - B) * 8 + S.bpos));
  scm_mix(M.smap[i], o, S.y, 6, 1, 2);
}
P8_HD inline void linear_bit(State& S, Out& o) {
  LinearM& M = S.linear;
  if (S.bpos == 0) {
    const u8 W = (u8)buf(S, 1);
    for (int k = 0; k < 3; ++k) ols_update(M.ols + (size_t)k * OLS_STRIDE, OLS_N, 4, 0.995, M.ols_km[k], (double)W);
    linear_predict(S);
  }
  for (int i = 0; i < 5; ++i) linear_small(S, o, i);
}

// ---------------------------------------------------------------- audio8bModel (:5552-5657), 8-bit PCM mono / stereo
// At a byte boundary audio8b_begin does the scalar part (restart, channel, residuals of the sample just coded, the fixed
// predictors), audio8b_ols(k) OLS predictor k: Update(s) on channel pCh = ch ^ stereo, then the taps and Predict() on
// channel ch (independent of the other seven). Each bit audio8b_scm(q) is stationary map q = 3 * predictor + j.
P8_HD inline int audio_ols_n(int k) { return k == 0 ? 128 : (k < 6 ? 90 : 28); }
P8_HD inline int audio_ols_kmax(int k) { return k == 0 ? 24 : (k < 6 ? 29 + k : 10 - k); }
P8_HD inline double audio_ols_lambda(int k) {
  switch (k) {
    case 0: return 0.9975; case 1: return 0.9965; case 2: return 0.996; case 3: case 4: return 0.995;
    case 5: return 0.9985; case 6: return 0.98; default: return 0.992;
  }
}
// blocks of 3n + 2n^2 doubles in the order (k, c): two of n = 128, ten of n = 90, four of n = 28
enum { AUDIO_BLK128 = 3 * 128 + 2 * 128 * 128, AUDIO_BLK90 = 3 * 90 + 2 * 90 * 90, AUDIO_BLK28 = 3 * 28 + 2 * 28 * 28,
       AUDIO_OLS_DOUBLES = 2 * AUDIO_BLK128 + 10 * AUDIO_BLK90 + 4 * AUDIO_BLK28 };
P8_HD inline double* audio_ols_block(const AudioM& A, int k, int c) {
  const int q = 2 * k + c;
  const size_t off = k == 0 ? (size_t)c * AUDIO_BLK128
                   : k < 6 ? 2 * (size_t)AUDIO_BLK128 + (size_t)(q - 2) * AUDIO_BLK90
                           : 2 * (size_t)AUDIO_BLK128 + 10 * (size_t)AUDIO_BLK90 + (size_t)(q - 12) * AUDIO_BLK28;
  return A.ols + off;
}
P8_HD inline bool audio8_mode(const State& S) { return S.detect.wav_info != 0 && ((S.detect.wav_info - 1) & 2) == 0; }
// X1 / X2 (:5516-5542) for the two modes 8-bit data sets: wmode 0 (mono) and 1 (stereo; X2 only there)
P8_HD inline int audio_x1(const State& S, int i) { return (S.audio->wmode ? buf(S, i << 1) : buf(S, i)) - 128; }
P8_HD inline int audio_x2(const State& S, int i) { return buf(S, (i << 1) - 1) - 128; }
P8_HD inline int sclip8(int v) { return imax(-128, imin(127, v)); }
P8_HD inline void audio_add(AudioM& A, int k, double v) {   // OLS::Add / AddFloat on channel ch
  int& idx = A.ols_index[k][A.ch];
  if (idx < audio_ols_n(k)) audio_ols_block(A, k, A.ch)[idx++] = v;
}
P8_COLD P8_HD inline void audio8b_begin(State& S) {
  AudioM& A = *S.audio;
  const int info = (int)S.detect.wav_info - 1;
  A.rpos = (S.pos == A.last_pos + 1) ? A.rpos + 1 : 0;
  A.last_pos = S.pos;
  if (A.rpos == 0) {
    A.stereo = info & 1;
    A.mask = 0;
    S.st_record = ((u32)(A.stereo + 1) << 16) | (S.st_record & 0xFFFF);
    A.wmode = info;
  }
  A.ch = A.stereo ? S.blpos & 1 : 0;
  const int s = buf(S, 1) - 128, ch = A.ch, pch = ch ^ A.stereo;
  u32 err = 0;
  int i = 0;
  for (; i < AUDIO_N_OLS; ++i) {
    A.residuals[i][pch] = s - A.prd[i][pch][0];
    const u32 r = (u32)iabs(A.residuals[i][pch]);
    A.mask += A.mask + (r > 4);
    err += r * r;
  }
  for (; i < AUDIO_N_PRD; ++i) A.residuals[i][pch] = s - A.prd[i][pch][0];
  A.err_log = umin(0xF, ilog2(err));
  A.mx_ctx = ilog2(umin(0x1F, bitcount(A.mask))) * 2 + (u32)ch;
  const int x1 = audio_x1(S, 1), x2 = audio_x1(S, 2), x3 = audio_x1(S, 3), x4 = audio_x1(S, 4);
  A.prd[8][ch][0] = sclip8(x1 * 2 - x2);
  A.prd[9][ch][0] = sclip8(x1 * 3 - x2 * 3 + x3);
  A.prd[10][ch][0] = sclip8(x1 * 4 - x2 * 6 + x3 * 4 - x4);
  for (i = AUDIO_N_OLS; i < AUDIO_N_PRD; ++i) A.prd[i][ch][1] = sclip8(A.prd[i][ch][0] + A.residuals[i][pch]);
}
P8_HD inline void audio8b_taps(State& S, int k) {   // the Add() calls of predictor k, in the reference's order (:5599-5631)
  AudioM& A = *S.audio;
  const int st = A.stereo;
  int i, j;
  if (k >= 1 && k <= 5) {
    const int k1 = 90, k2 = k1 - 12 * st;
    if (k == 1) for (j = (i = 1); j <= k1; j++, i += 1 << ((j > 8) + (j > 16) + (j > 64))) audio_add(A, k, audio_x1(S, i));
    if (k == 2) for (j = (i = 1); j <= k2; j++, i += 1 << ((j > 5) + (j > 10) + (j > 17) + (j > 26) + (j > 37))) audio_add(A, k, audio_x1(S, i));
    if (k == 3) for (j = (i = 1); j <= k2; j++, i += 1 << ((j > 3) + (j > 7) + (j > 14) + (j > 20) + (j > 33) + (j > 49))) audio_add(A, k, audio_x1(S, i));
    if (k == 4) for (j = (i = 1); j <= k2; j++, i += 1 + (j > 4) + (j > 8)) audio_add(A, k, audio_x1(S, i));
    if (k == 5) for (j = (i = 1); j <= k1; j++, i += 2 + ((j > 3) + (j > 9) + (j > 19) + (j > 36) + (j > 61))) audio_add(A, k, audio_x1(S, i));
    if (st && k >= 2 && k <= 4) for (i = 1; i <= k1 - k2; i++) audio_add(A, k, audio_x2(S, i));
    return;
  }
  const int k1 = 28, k2 = k1 - 6 * st;
  for (i = 1; i <= k2; i++) audio_add(A, k, audio_x1(S, i));
  if (k == 0) for (; i <= 96; i++) audio_add(A, k, audio_x1(S, i));
  if (st) {
    for (i = 1; i <= k1 - k2; i++) audio_add(A, k, audio_x2(S, i));
    if (k == 0) for (; i <= 32; i++) audio_add(A, k, audio_x2(S, i));
  } else if (k == 0) for (; i <= 128; i++) audio_add(A, k, audio_x1(S, i));
}
P8_HD inline void audio8b_predict(State& S, int k, double sum) {   // Predict()'s result into the two predictions of k
  AudioM& A = *S.audio;
  const int ch = A.ch, pch = ch ^ A.stereo;
  A.ols_index[k][ch] = 0;
  A.prd[k][ch][0] = sclip8((int)P8_FLOOR(sum));
  A.prd[k][ch][1] = sclip8(A.prd[k][ch][0] + A.residuals[k][pch]);
}
P8_HD inline void audio8b_ols(State& S, int k) {
  AudioM& A = *S.audio;
  const int n = audio_ols_n(k), pch = A.ch ^ A.stereo;
  ols_update(audio_ols_block(A, k, pch), n, audio_ols_kmax(k), audio_ols_lambda(k), A.ols_km[k][pch], (double)(buf(S, 1) - 128));
  audio8b_taps(S, k);
  audio8b_predict(S, k, ols_predict(audio_ols_block(A, k, A.ch), n));
}
P8_HD inline void audio8b_scm(State& S, Out& o, int q) {
  AudioM& A = *S.audio;
  const int i = q / 3, j = q - 3 * i, bpos = S.bpos;
  const int B = (int)(signed char)(u8)(S.c0 << (8 - bpos));
  Scm& c = A.scm[i][j];
  scm_set(c, (u32)((A.prd[i][A.ch][j == 2] - B) * 8 + bpos));
  if (j == 2) scm_mix(c, o, S.y, 7, 1, 3);
  else scm_mix(c, o, S.y, j == 0 ? 6 : 9, 1, 2 + (i >= AUDIO_N_OLS));
}
P8_HD inline void audio8b_select(State& S) {
  const AudioM& A = *S.audio;
  const int bpos = S.bpos, c0 = S.c0;
  Mixer& m = S.m;
  mset(m, (int)(A.err_log << 8) | c0, 4096);
  mset(m, (int)(((A.mask & 0xFF) << 3) | ((u32)A.ch << 2) | (u32)(bpos >> 1)), 2048);
  mset(m, (int)((A.mx_ctx << 7) | ((u32)buf(S, 1) >> 1)), 1280);
  mset(m, (int)((A.err_log << 4) | ((u32)A.ch << 3) | (u32)bpos), 256);
  mset(m, (int)A.mx_ctx, 10);
}

// ---------------------------------------------------------------- header detectors in front of the unmodelled image / audio / JPEG paths
// The reference parses BMP / TGA / WAV / JPEG headers in ANY block and switches to dedicated models when one validates
// (:5386-5509, :5810-5870, :5966-6060). Apart from 8-bit audio those models are not built; a validated header raises
// ERR_UNSUPPORTED_BLOCK.
P8_HD inline u32 le4(const State& S, int i) { return (u32)buf(S, i) + 256u * (u32)buf(S, i - 1) + 65536u * (u32)buf(S, i - 2) + 16777216u * (u32)buf(S, i - 3); }
P8_HD inline int le2(const State& S, int i) { return buf(S, i) + 256 * buf(S, i - 1); }
P8_HD inline u32 be4(const State& S, int i) { return (u32)buf(S, i - 3) + 256u * (u32)buf(S, i - 2) + 65536u * (u32)buf(S, i - 1) + 16777216u * (u32)buf(S, i); }
// audioModel's parser (:5811-5866), run at the start of every byte: the WAVAudio header state, `length`, `eoi` and `info`.
// info != 0 is audio mode: on those bytes the reference runs audio8bModel / wavModel and recordModel(AUDIO) instead of the
// ordinary models. audio8bModel is built (8-bit data, info 1 and 2); wavModel is not, so 16-bit audio mode raises
// ERR_UNSUPPORTED_BLOCK. Audio mode starts on the first byte of a PCM data chunk whose length is a whole number of sample blocks. Any other RIFF stream (AVI, WebP, compressed or 24-bit WAV,
// truncated headers, "RIFF" in text) codes with the ordinary models.
P8_HD inline void wav_byte(State& S) {
  DetectM& D = S.detect;
  // the reference clears WAVAudio on bit 7 of the byte before eoi (:5865-5866); nothing reads it in between
  if (S.pos > 0 && S.pos == (int)D.wav_eoi) D.wav_header = D.wav_channels = D.wav_bits = D.wav_chunk = 0;
  if (S.pos >= (int)(D.wav_eoi + 4) && !D.wav_header && be4(S, 4) == 0x52494646u) {   // "RIFF"
    D.wav_header = (u32)S.pos; D.wav_chunk = 0; D.wav_length = 0;
  } else if (D.wav_header) {
    const int p = S.pos - (int)D.wav_header;
    const u32 len = D.wav_length;
    if (p == 4) D.wav_header *= (le4(S, 4) <= 0x3FFFFFFFu);
    else if (p == 8) D.wav_header *= (be4(S, 4) == 0x57415645u);   // "WAVE"
    else if (p == (int)(16 + len) && (be4(S, 8) != 0x666d7420u || ((D.wav_chunk = le4(S, 4) - 16) & 0xFFFFFFFDu) != 0)) {   // "fmt " of 16 or 18 bytes
      D.wav_length = ((le4(S, 4) + 1) & ~1u) + 8;
      D.wav_header *= !(be4(S, 8) == 0x666d7420u && (le4(S, 4) & 0xFFFFFFFDu) != 16);
    } else if (p == (int)(20 + len)) {   // PCM, 1 or 2 channels
      D.wav_channels = (u32)buf(S, 2);
      D.wav_header *= ((D.wav_channels == 1 || D.wav_channels == 2) && (be4(S, 4) & 0xFFFFFCFFu) == 0x01000000u);
    } else if (p == (int)(32 + len)) {   // 8 or 16 bits per sample
      D.wav_bits = (u32)buf(S, 2);
      D.wav_header *= ((D.wav_bits == 8 || D.wav_bits == 16) && ((buf(S, 2) * 256 + buf(S, 1)) & 0xE7FF) == 0);
    } else if (p == (int)(40 + len + D.wav_chunk) && be4(S, 8) != 0x64617461u) {   // a chunk other than "data": skip it
      D.wav_chunk += ((le4(S, 4) + 1) & ~1u) + 8;
      D.wav_header *= (D.wav_chunk <= 0xFFFFFu);
    } else if (p == (int)(40 + len + D.wav_chunk)) {
      // block is 0 only on headers where the reference divides by zero (channels or bits never read); those stay ordinary data
      const u32 data = (le4(S, 4) + 1) & ~1u, block = D.wav_channels * (D.wav_bits / 8);
      if (data && block && data % block == 0) {
        D.wav_info = (D.wav_channels + D.wav_bits / 4 - 3) + 1;
        D.wav_eoi = (u32)S.pos + data;
      }
    }
  }
  if (S.pos > (int)D.wav_eoi) D.wav_info = 0;
  if (D.wav_info && !audio8_mode(S)) S.error |= ERR_UNSUPPORTED_BLOCK;   // 16-bit audio mode only
}
P8_COLD P8_HD inline void detect_byte(State& S) {
  // JPEG: SOI followed by a plausible marker (:6046-6049)
  if (S.filetype != FT_EXE && buf(S, 4) == 0xFF && buf(S, 3) == 0xD8 && buf(S, 2) == 0xFF &&
      ((buf(S, 1) & 0xFE) == 0xC0 || buf(S, 1) == 0xC4 || (buf(S, 1) >= 0xDB && buf(S, 1) <= 0xFE))) S.error |= ERR_UNSUPPORTED_BLOCK;
  if (S.size > 0) {
    // BMP / DIB (:5394-5407): header-less DIBs trigger on a 40-byte BITMAPINFOHEADER
    const bool bm = buf(S, 54) == 'B' && buf(S, 53) == 'M' && ((le4(S, 44) & 0xFFFFFBF7u) == 0x36) && le4(S, 40) == 0x28;
    if (S.pos >= 40 && (bm || le4(S, 40) == 0x28)) {
      const u32 width = le4(S, 36), height = (u32)iabs((int)le4(S, 32)), palette = le4(S, 4);
      const int bpp = le2(S, 26);
      if ((le4(S, 24) == 0) && (le2(S, 28) == 1) && (bpp == 1 || bpp == 4 || bpp == 8 || bpp == 24 || bpp == 32) && width < 30000 && height < 10000 &&
          (!palette || ((u32)(1 << bpp)) >= palette)) S.error |= ERR_UNSUPPORTED_BLOCK;
    }
    // TGA (:5446-5459)
    if (S.pos >= 8) {
      if (((be4(S, 8) & 0xFFFFFF) == 0x010100 && (be4(S, 4) & 0xFFFFFFC7u) == 0x00000100 && (buf(S, 1) == 16 || buf(S, 1) == 24 || buf(S, 1) == 32)) ||
          ((be4(S, 8) & 0xFFFEFF) == 0x000200 && !be4(S, 4))) S.error |= ERR_UNSUPPORTED_BLOCK;
    }
  }
  wav_byte(S);
}

// ---------------------------------------------------------------- contextModel2 (:8101-8206) and Predictor::update (:8248-8362)
P8_HD inline void mixer_train(Mixer& m, int y) {   // Mixer::update (:527-540) for the 28 selected sets; the final mixer trains in mixer_predict
  for (int i = 0; i < m.ncxt; ++i) {
    const int err = ((y << 12) - m.pr[i]) * 7;
    if (!err) continue;
    short* w = m.w + (size_t)m.cxt[i] * N_IN;
    for (int k = 0; k < m.nx; ++k) w[k] = train_one(m.tx[k], w[k], err);
  }
  m.nx = m.base = m.ncxt = 0;
}
P8_HD inline int mixer_predict(const Tables& T, Mixer& m, int y, u16* codes) {   // Mixer::p (:575-595)
  const int base = m.nx;   // exports continue right behind the inputs added this bit (prediction_index, :504-507)
  m.n2 = base;
  while (m.nx & 7) m.tx[m.nx++] = 0;
  {   // mp->update()
    const int err = ((y << 12) - m.pr2) * 7;
    if (err) for (int k = 0; k < m.nx2; ++k) m.w2[k] = train_one(m.tx2[k], m.w2[k], err);
    m.nx2 = 0;
  }
  for (int i = 0; i < m.ncxt; ++i) {
    const short* w = m.w + (size_t)m.cxt[i] * N_IN;
    int dot = 0;
    for (int k = 0; k < m.nx; k += 2) dot += dot_pair(m.tx + k, w + k);
    m.pr[i] = squash(T, (int)((u32)dot * 9u) >> 9);
    const int x = stretch(T, m.pr[i]);
    codes[base + i] = (u16)squash(T, x);
    m.tx2[m.nx2++] = (short)x;
  }
  while (m.nx2 & 7) m.tx2[m.nx2++] = 0;
  int z = 0;
  for (int k = 0; k < m.nx2; k += 2) z += dot_pair(m.tx2 + k, m.w2 + k);
  return m.pr2 = squash(T, z >> 9);
}

// block header parsing in front of contextModel2 (:8116-8134): filetype and bytes remaining of the current block
P8_COLD P8_HD inline void block_parse(State& S) {
  --S.size;
  ++S.blpos;
  if (S.size == -1) { S.info = 0; S.ft2 = buf(S, 1); }
  if (S.size == -5 && !(S.ft2 == FT_TEXT || S.ft2 == FT_IMAGE1 || S.ft2 == FT_IMAGE4 || S.ft2 == FT_IMAGE8 || S.ft2 == FT_IMAGE8GRAY || S.ft2 == FT_IMAGE24 || S.ft2 == FT_IMAGE32)) {
    S.size = buf(S, 4) << 24 | buf(S, 3) << 16 | buf(S, 2) << 8 | buf(S, 1);
    S.blpos = 0;
  }
  if (S.size == -9) {
    S.size = buf(S, 8) << 24 | buf(S, 7) << 16 | buf(S, 6) << 8 | buf(S, 5);
    S.info = buf(S, 4) << 24 | buf(S, 3) << 16 | buf(S, 2) << 8 | buf(S, 1);
    S.blpos = 0;
    if (S.ft2 == FT_TEXT && S.info) S.size = S.info - 8;
  }
  if (!S.blpos) S.filetype = S.ft2;
  if (S.size == 0) S.filetype = FT_DEFAULT;
  S.st_type = S.filetype;
  if (S.filetype == FT_JPEG || (S.filetype >= FT_IMAGE1 && S.filetype <= FT_AUDIO)) S.error |= ERR_UNSUPPORTED_BLOCK;
  detect_byte(S);
}
P8_COLD P8_HD inline void ordern_byte(State& S) {   // :8140-8152
  const u8 B = (u8)S.c4;
  S.cxt[15] = is_alpha(B) ? (u32)combine64(S.cxt[15], (u64)lower(B)) : 0;
  cm2_set(S.cm, S.cxt[15]);
  for (int i = 14; i > 0; --i) S.cxt[i] = (u32)combine64(S.cxt[i - 1], B);
  for (int i = 0; i < 7; ++i) cm2_set(S.cm, S.cxt[i]);
  rcm_set(S.rcm7, S.cxt[7], buf(S, 1));
  cm2_set(S.cm, S.cxt[8]);
  rcm_set(S.rcm9, S.cxt[10], buf(S, 1));
  rcm_set(S.rcm10, S.cxt[12], buf(S, 1));
  cm2_set(S.cm, S.cxt[14]);
}
P8_HD inline void main_select(State& S, int order) {   // the nine selector sets of contextModel2 itself (:8187-8202)
  Mixer& m = S.m;
  const int bpos = S.bpos, c0 = S.c0;
  mset(m, (imax(0, order - 3) << 3) | bpos, 64);
  order = imax(0, order - 5);
  const u32 d = (u32)c0 << (8 - bpos);
  u32 c = (d + (bpos == 1 ? S.b3 / 2 : 0)) & 192;
  if (!bpos) c = S.words * 16 & 192;
  const u32 c1 = (u32)buf(S, 1);
  mset(m, (int)((u32)order * 256 + (S.w4 & 240) + (S.b2 >> 4)), 1536);
  mset(m, (int)((u32)order * 256 + (S.w4 & 3) * 64 + (S.words >> 1 & 63)), 1536);
  mset(m, (int)((u32)bpos * 256 + c1), 2048);
  mset(m, (int)((u32)imin(bpos, 5) * 256 + (S.tt & 63) + c), 1536);
  mset(m, (int)((u32)order * 256 + ((d | c1 >> bpos) & 248) + (u32)bpos), 1536);
  mset(m, (int)((u32)bpos * 256 + (((S.words << bpos & 255) >> bpos) | (d & 255))), 2048);
  mset(m, S.last_prediction / 16, 256);
  mset(m, c0, 256);
}

// The same nine sets written at their fixed places: the 19 sets before them always cover MAIN_SET_BASE weight sets, so a lane can
// compute these while another one is still producing the first 19 (paq8.cuh).
// MAIN_SET_PR: the first weight set of selector MAIN_SET_FIRST + 7, the one indexed by the last prediction.
enum { MAIN_SET_FIRST = 19, MAIN_SET_BASE = 66656, MAIN_SET_PR = MAIN_SET_BASE + 64 + 4 * 1536 + 2 * 2048 };
static_assert(MAIN_SET_PR + 2 * 256 == N_WSETS && MAIN_SET_FIRST + 9 == N_SETS, "selector layout");
P8_HD inline void main_select_fixed(State& S, int order) {
  Mixer& m = S.m;
  const int bpos = S.bpos, c0 = S.c0;
  int* cx = m.cxt + MAIN_SET_FIRST;
  int base = MAIN_SET_BASE;
  cx[0] = base + ((imax(0, order - 3) << 3) | bpos); base += 64;
  order = imax(0, order - 5);
  const u32 d = (u32)c0 << (8 - bpos);
  u32 c = (d + (bpos == 1 ? S.b3 / 2 : 0)) & 192;
  if (!bpos) c = S.words * 16 & 192;
  const u32 c1 = (u32)buf(S, 1);
  cx[1] = base + (int)((u32)order * 256 + (S.w4 & 240) + (S.b2 >> 4)); base += 1536;
  cx[2] = base + (int)((u32)order * 256 + (S.w4 & 3) * 64 + (S.words >> 1 & 63)); base += 1536;
  cx[3] = base + (int)((u32)bpos * 256 + c1); base += 2048;
  cx[4] = base + (int)((u32)imin(bpos, 5) * 256 + (S.tt & 63) + c); base += 1536;
  cx[5] = base + (int)((u32)order * 256 + ((d | c1 >> bpos) & 248) + (u32)bpos); base += 1536;
  cx[6] = base + (int)((u32)bpos * 256 + (((S.words << bpos & 255) >> bpos) | (d & 255))); base += 2048;
  cx[7] = base + S.last_prediction / 16; base += 256;
  cx[8] = base + c0;
}

P8_HD inline int context_model(State& S) {
  const Tables& T = *S.T;
  const int y = S.y, bpos = S.bpos;
  if (bpos == 0) block_parse(S);
  Mixer& m = S.m;
  mixer_train(m, y);
  Out o; o.T = &T; o.tx = m.tx; o.codes = S.codes; o.n = 0;
  add(o, 64);
  const int c0 = S.c0;
  if (bpos == 0) ordern_byte(S);
  add(o, (stretch(T, sm32_p(T, S.sm0, y, c0)) + 1) >> 1);
  add(o, (stretch(T, sm32_p(T, S.sm1, y, c0 | (buf(S, 1) << 8))) + 1) >> 1);
  int order = cm2_mix(S.cm, o, y, bpos);
  rcm_mix(S.rcm7, o, c0, bpos);
  rcm_mix(S.rcm9, o, c0, bpos);
  rcm_mix(S.rcm10, o, c0, bpos);
  match_bit(S, o);
  if (audio8_mode(S)) {   // audioModel returns non-zero (:8167): audio8bModel, recordModel(AUDIO), and no other model
    if (bpos == 0) { audio8b_begin(S); for (int k = 0; k < AUDIO_N_OLS; ++k) audio8b_ols(S, k); }
    for (int q = 0; q < AUDIO_N_SCM; ++q) audio8b_scm(S, o, q);
    audio8b_select(S);
    record_core(S, o, S.rnd, FT_AUDIO);
    record_select(S);
    m.nx = o.n;
    return mixer_predict(T, m, y, S.codes);
  }
  const int ismatch = ilog(T, S.match.length);
  smatch_core(S, o);
  smatch_select(S);
  if (bpos == 0) { sparse_byte(S, ismatch, order); }
  cm_mix(S.sparse.cm, o, S.rnd, y, c0, bpos, buf(S, 1));
  if (bpos == 0) sparse1_byte(S, ismatch, order, word_stats(S));
  cm_mix(S.sparse1.cm, o, S.rnd, y, c0, bpos, buf(S, 1));
  for (int k = 0; k < 7; ++k) scm_mix(S.sparse1.scm[k], o, y);
  if (bpos == 0) distance_byte(S);
  cm_mix(S.distance.cm, o, S.rnd, y, c0, bpos, buf(S, 1));
  pic_bit(S, o);
  record_core(S, o, S.rnd, S.filetype);
  record_select(S);
  record1_bit(S, o, S.rnd);
  if (bpos == 0) word_byte(S);
  cm_mix(S.word.cm, o, S.rnd, y, c0, bpos, buf(S, 1));
  if (bpos == 0) nest_byte(S);
  cm_mix(S.nest.cm, o, S.rnd, y, c0, bpos, buf(S, 1));
  if (bpos == 0) indirect_byte(S);
  cm_mix(S.indirect.cm, o, S.rnd, y, c0, bpos, buf(S, 1));
  dmc_bit(S, o);
  xml_bit(S, o, S.rnd);
  text_bit(S, o);
  exe_bit(S, o);
  linear_bit(S, o);
  m.nx = o.n;
  main_select(S, order);
  return mixer_predict(T, m, y, S.codes);
}

// bit bookkeeping of Predictor::update (:8251-8276)
P8_HD inline void bit_begin(State& S, int y) {
  const Tables& T = *S.T;
  S.y = y;
  S.c0 += S.c0 + y;
  S.st_misses += S.st_misses + (u64)((S.pr >> 11) != y);
  if (S.c0 >= 256) {
    S.buf[(u32)(S.pos++) & P8_BUF_MASK] = (u8)S.c0;
    S.c0 -= 256;
    S.c4 = (S.c4 << 8) + (u32)S.c0;
    const u8 mpw[16] = {4, 4, 3, 2, 2, 2, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0};   // WRT_mpw / WRT_mtt (:3868-3869)
    const u8 mtt[16] = {0, 0, 1, 2, 3, 4, 5, 5, 6, 6, 6, 6, 7, 7, 7, 7};
    u32 i = mpw[S.c0 >> 4];
    S.w4 = S.w4 * 4 + i;
    if (S.b2 == 3) i = 2;
    S.w5 = S.w5 * 4 + i;
    S.b3 = S.b2;
    S.b2 = (u32)S.c0;
    S.x4 = S.x4 * 256 + (u32)S.c0; S.x5 = (S.x5 << 8) + (u32)S.c0;
    if (S.c0 == '.' || S.c0 == '!' || S.c0 == '?' || S.c0 == '/' || S.c0 == ')') {
      S.w5 = (S.w5 << 8) | 0x3ff; S.f4 = (S.f4 & 0xfffffff0) + 2; S.x5 = (S.x5 << 8) + (u32)S.c0; S.x4 = S.x4 * 256 + (u32)S.c0;
      if (S.c0 != '!') { S.w4 |= 12; S.tt = (S.tt & 0xfffffff8) + 1; S.b3 = '.'; }
    }
    if (S.c0 == 32) --S.c0;
    S.tt = S.tt * 8 + mtt[S.c0 >> 4];
    S.f4 = S.f4 * 16 + (u32)(S.c0 >> 4);
    S.c0 = 1;
  }
  S.bpos = (S.bpos + 1) & 7;
  S.grp0 = (S.bpos > 0) ? T.ascii_group_c0[(1 << S.bpos) - 2 + (S.c0 & ((1 << S.bpos) - 1))] : 0;
}
// the SSE stage of Predictor::update (:8278-8358): APM chain on the mixer output pr0, exports behind the mixer's
P8_HD inline void sse_stage(State& S, int pr0) {
  const Tables& T = *S.T;
  const int y = S.y;
  u16* codes = S.codes;
  int e = S.m.n2 + S.m.ncxt;
  codes[e++] = (u16)pr0;
  const int c0 = S.c0, bpos = S.bpos;
  const u32 c4 = S.c4;
  int pr, pr1, pr2, pr3;
  const u32 mlen = umin(3, ilog2(S.st_match_length + 1));
  if (S.st_type == FT_TEXT) {
    const int limit = 0x3FF >> ((S.blpos < 0xFFF) * 2);
    pr = apm_p(T, S.text_apm[0], y, pr0, (c0 << 8) | (S.st_text_mask & 0xF) | (int)((S.st_misses & 0xF) << 4), limit); codes[e++] = (u16)pr;
    pr1 = apm_p(T, S.text_apm[1], y, pr0, (int)finalize64(hash(sx(bpos), S.st_misses & 3, (u64)(c4 & 0xffff), (u64)(S.st_text_mask >> 4)), 16), limit); codes[e++] = (u16)pr1;
    pr2 = apm_p(T, S.text_apm[2], y, pr0, (int)finalize64(hash(sx(c0), S.st_match_expected, mlen), 16), limit); codes[e++] = (u16)pr2;
    pr3 = apm_p(T, S.text_apm[3], y, pr0, (int)finalize64(hash(sx(c0), (u64)(c4 & 0xffff), S.st_text_first), 16), limit); codes[e++] = (u16)pr3;
    pr0 = (pr0 + pr1 + pr2 + pr3 + 2) >> 2; codes[e++] = (u16)pr0;
    pr1 = apm1_p(T, S.text_apm1[0], y, pr0, (int)finalize64(hash(S.st_match_expected, mlen, (u64)(c4 & 0xff)), 16)); codes[e++] = (u16)pr1;
    pr2 = apm1_p(T, S.text_apm1[1], y, pr, (int)finalize64(hash(sx(c0), (u64)(c4 & 0x00ffffff)), 16), 6); codes[e++] = (u16)pr2;
    pr3 = apm1_p(T, S.text_apm1[2], y, pr, (int)finalize64(hash(sx(c0), (u64)(c4 & 0xffffff00)), 16), 6); codes[e++] = (u16)pr3;
    pr = (pr + pr1 + pr2 + pr3 + 2) >> 2; codes[e++] = (u16)pr;
    pr = (pr + pr0 + 1) >> 1; codes[e++] = (u16)pr;
  } else {
    pr = apm1_p(T, S.generic_apm1[0], y, pr0, (int)((mlen << 11) | ((u32)c0 << 3) | (u32)(S.st_misses & 0x7))); codes[e++] = (u16)pr;
    const u16 ctx1 = (u16)(c0 | buf(S, 1) << 8);
    const u16 ctx2 = (u16)(c0 ^ finalize64(hash((u64)(c4 & 0xffff)), 16));
    const u16 ctx3 = (u16)(c0 ^ finalize64(hash((u64)(c4 & 0xffffff)), 16));
    pr1 = apm1_p(T, S.generic_apm1[1], y, pr0, ctx1); codes[e++] = (u16)pr1;
    pr2 = apm1_p(T, S.generic_apm1[2], y, pr0, ctx2); codes[e++] = (u16)pr2;
    pr3 = apm1_p(T, S.generic_apm1[3], y, pr0, ctx3); codes[e++] = (u16)pr3;
    pr0 = (pr0 + pr1 + pr2 + pr3 + 2) >> 2;
    pr1 = apm1_p(T, S.generic_apm1[4], y, pr, (S.st_match_expected << 8) | buf(S, 1)); codes[e++] = (u16)pr1;
    pr2 = apm1_p(T, S.generic_apm1[5], y, pr, ctx2); codes[e++] = (u16)pr2;
    pr3 = apm1_p(T, S.generic_apm1[6], y, pr, ctx3); codes[e++] = (u16)pr3;
    pr = (pr + pr1 + pr2 + pr3 + 2) >> 2; codes[e++] = (u16)pr;
    pr = (pr + pr0 + 1) >> 1; codes[e++] = (u16)pr;
  }
  S.pr = pr;
  S.last_prediction = pr;
}

// PAQ8::Perceive(bit): paq8::y = bit; predictor_->update() (:8380-8383) — the whole bit on one lane (CPU pinning)
P8_HD inline void bit(State& S, int y) {
  bit_begin(S, y);
  const int pr0 = context_model(S);
  sse_stage(S, pr0);
}

}  // namespace p8
}  // namespace cmixb200
#endif
