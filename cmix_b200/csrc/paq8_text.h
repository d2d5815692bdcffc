// cmix_b200/csrc/paq8_text.h — word objects and the three affix stemmers of PAQ8's text model (SURVEY §8 row a13).
//
// PAQ8's TextModel (reference src/models/paq8.cpp:3070-3519) stems EVERY word with an English, a French and a German
// stemmer (:1764-3005) to track the language of the text and to derive word-class flags and stem hashes for its
// contexts; the word model (:3873) uses the English one as well. They are deterministic string rewriting over a
// 64-byte word buffer; restated here as host/device code (one lane runs them, once per completed word).
#ifndef CMIXB200_PAQ8_TEXT_H
#define CMIXB200_PAQ8_TEXT_H

#include "paq8_model.h"

namespace cmixb200 {
namespace p8 {

P8_HD inline int cstrlen(const char* s) { int n = 0; while (s[n]) ++n; return n; }
P8_HD inline bool bytes_eq(const u8* a, const char* b, int n) { for (int i = 0; i < n; ++i) if (a[i] != (u8)b[i]) return false; return true; }
P8_HD inline bool in_set(int c, const char* set) { for (; *set; ++set) if ((u8)*set == (u8)c) return true; return false; }
P8_HD inline int lower(int c) { return (c >= 'A' && c <= 'Z') ? c + 32 : c; }     // tolower / toupper in the "C" locale
P8_HD inline int upper(int c) { return (c >= 'a' && c <= 'z') ? c - 32 : c; }

enum { LANG_UNKNOWN = 0, LANG_EN = 1, LANG_FR = 2, LANG_DE = 3, LANG_COUNT = 4 };
// Language::Flags / English::Flags (paq8.cpp:1652-1700); French and German reuse bits 2-4 with their own meaning
enum : u64 { W_Verb = 1, W_Noun = 2, EN_Adjective = 4, EN_Plural = 8, EN_Male = 16, EN_Female = 32, EN_Negation = 64, EN_PastTense = 128 | W_Verb,
             EN_PresentParticiple = 256 | W_Verb, EN_AdjSuperlative = 512 | EN_Adjective, EN_AdjWithout = 1024 | EN_Adjective,
             EN_AdjFull = 2048 | EN_Adjective, EN_AdverbOfManner = 4096, EN_NESS = 1u << 13, EN_ITY = (1u << 14) | W_Noun, EN_Capable = 1u << 15,
             EN_NCE = 1u << 16, EN_NT = 1u << 17, EN_ION = 1u << 18, EN_AL = (1u << 19) | EN_Adjective, EN_IC = (1u << 20) | EN_Adjective,
             EN_IVE = 1u << 21, EN_OUS = (1u << 22) | EN_Adjective, EN_PrefixOver = 1u << 23, EN_PrefixUnder = 1u << 24,
             FR_Adjective = 4, FR_Plural = 8, DE_Adjective = 4, DE_Plural = 8, DE_Female = 16 };

struct Word {   // paq8.cpp:1547-1622
  u8 L[64];
  u8 s, e;
  u64 hash[4], type, language;
  P8_HD void clear() { for (int i = 0; i < 64; ++i) L[i] = 0; s = e = 0; hash[0] = hash[1] = hash[2] = hash[3] = 0; type = 0; language = 0; }
  P8_HD u32 len() const { return L[s] != 0 ? (u32)(e - s + 1) : 0u; }
  P8_HD u8 at(int i) const { return (e - s >= i) ? L[s + i] : 0; }
  P8_HD u8 rat(int i) const { return (e - s >= i) ? L[e - i] : 0; }
  P8_HD void append(int c) { if (e < 63) { e = (u8)(e + (L[e] > 0)); L[e] = (u8)lower(c & 255); } }
  P8_HD bool is(const char* w) const { const int n = cstrlen(w); return (int)(e - s + (L[s] != 0)) == n && bytes_eq(&L[s], w, n); }
  P8_HD bool ends(const char* w) const { const u32 n = cstrlen(w); return len() > n && bytes_eq(&L[e - n + 1], w, (int)n); }
  P8_HD bool starts(const char* w) const { const u32 n = cstrlen(w); return len() > n && bytes_eq(&L[s], w, (int)n); }
  P8_HD bool swap_suffix(const char* from, const char* to) {
    const int n = cstrlen(from);
    if (len() > (u32)n && bytes_eq(&L[e - n + 1], from, n)) {
      const int m = cstrlen(to);
      if (m > 0) {
        const int cnt = imin(63, e + m) - e;
        for (int i = 0; i < cnt; ++i) L[e - n + 1 + i] = (u8)to[i];
        e = (u8)imin(63, (int)e - n + m);
      } else e = (u8)(e - n);
      return true;
    }
    return false;
  }
  P8_HD bool any_of(const char* list) const {
    const int n = (int)len();
    for (const char* p = list; *p;) {
      int k = 0;
      while (p[k] && p[k] != '|') ++k;
      if (k == n && bytes_eq(&L[s], p, n)) return true;
      p += k;
      if (*p == '|') ++p;
    }
    return false;
  }
  P8_HD void get_hashes() {
    hash[0] = 0xc01dfull; hash[1] = ~hash[0];
    for (int i = s; i <= e; ++i) {
      const u8 l = L[i];
      hash[0] ^= p8::hash(hash[0], (u64)l, (u64)i);
      hash[1] ^= p8::hash(hash[1], (u64)(((l & 0x80) == 0) ? l & 0x5F : ((l & 0xC0) == 0x80) ? l & 0x3F : ((l & 0xE0) == 0xC0) ? l & 0x1F : ((l & 0xF0) == 0xE0) ? l & 0xF : l & 0x7));
    }
    hash[2] = (~hash[0]) ^ hash[1];
    hash[3] = (~hash[1]) ^ hash[0];
  }
};

// Tables of suffixes / words walked in a loop keep the length and the deciding character of every entry next to the string, so
// that a candidate that cannot match costs no read of the string itself (on the device the strings live in global memory).
P8_HD inline bool ends_tab(const Word& w, const char* suf, int n, char last) {      // == w.ends(suf) with n = strlen(suf), last = suf[n-1]
  return w.len() > (u32)n && w.L[w.e] == (u8)last && bytes_eq(&w.L[w.e - n + 1], suf, n - 1);
}
P8_HD inline bool is_tab(const Word& w, const char* word, int n, char first) {      // == w.is(word) with n = strlen(word), first = word[0]
  return (int)(w.e - w.s + (w.L[w.s] != 0)) == n && w.L[w.s] == (u8)first && bytes_eq(&w.L[w.s], word, n);
}

// Stemmer::GetRegion / SuffixInRn (paq8.cpp:1731-1746) with the language's vowel set
P8_HD inline u32 region(const Word& w, u32 from, const char* vowels) {
  bool seen = false;
  for (int i = w.s + (int)from; i <= w.e; ++i) {
    if (in_set(w.L[i], vowels)) { seen = true; continue; }
    if (seen) return (u32)(i - w.s + 1);
  }
  return w.s + w.len();
}
P8_HD inline bool in_rn(const Word& w, u32 rn, int suffix_len) { return w.s != w.e && (u64)rn <= (u64)w.len() - (u64)suffix_len; }

// ---------------------------------------------------------------- English (paq8.cpp:1764-2422)
struct StemEN {
  P8_HD static bool vowel(int c) { return in_set(c, "aeiouy"); }
  P8_HD static void rehash(Word& w) {
    w.hash[2] = w.hash[3] = 0xb0a710adull;
    for (int i = w.s; i <= w.e; ++i) {
      const u8 l = w.L[i];
      w.hash[2] = w.hash[2] * 263 * 32 + l;
      if (vowel(l)) w.hash[3] = w.hash[3] * 997 * 8 + (u64)(i64)(l / 4 - 22);
      else if (l >= 'b' && l <= 'z') w.hash[3] = w.hash[3] * 271 * 32 + (l - 97);
      else w.hash[3] = w.hash[3] * 11 * 32 + l;
    }
  }
  P8_HD static u32 region1(const Word& w) {
    if (w.starts("gener")) return 5;
    if (w.starts("arsen")) return 5;
    if (w.starts("commun")) return 6;
    return region(w, 0, "aeiouy");
  }
  P8_HD static bool short_syllable(const Word& w) {
    if (w.e == w.s) return false;
    if (w.e == w.s + 1) return vowel(w.rat(1)) && !vowel(w.rat(0));
    return !vowel(w.rat(2)) && vowel(w.rat(1)) && !vowel(w.rat(0)) && !in_set(w.rat(0), "wxY");
  }
  P8_HD static bool short_word(const Word& w) { return short_syllable(w) && region1(w) == w.len(); }
  P8_HD static bool has_vowel(const Word& w) { for (int i = w.s; i <= w.e; ++i) if (vowel(w.L[i])) return true; return false; }
  P8_HD static bool prefixes(Word& w) {
    if (w.starts("irr") && w.len() > 5 && (w.at(3) == 'a' || w.at(3) == 'e')) { w.s += 2; w.type |= EN_Negation; }
    else if (w.starts("over") && w.len() > 5) { w.s += 4; w.type |= EN_PrefixOver; }
    else if (w.starts("under") && w.len() > 6) { w.s += 5; w.type |= EN_PrefixUnder; }
    else if (w.starts("unn") && w.len() > 5) { w.s += 2; w.type |= EN_Negation; }
    else if (w.starts("non") && w.len() > (u32)(5 + (w.at(3) == '-'))) { w.s += 2 + (w.at(3) == '-'); w.type |= EN_Negation; }
    else return false;
    return true;
  }
  P8_HD static bool superlatives(Word& w) {
    if (w.ends("est") && w.len() > 4) {
      const u8 keep = w.e;
      w.e -= 3;
      w.type |= EN_AdjSuperlative;
      if (w.rat(0) == w.rat(1) && w.rat(0) != 'r' && !(w.len() >= 4 && bytes_eq(&w.L[w.e - 3], "sugg", 4))) {
        w.e -= (((w.rat(0) != 'f' && w.rat(0) != 'l' && w.rat(0) != 's') ||
                 (w.len() > 4 && w.rat(1) == 'l' && (w.rat(2) == 'u' || w.rat(3) == 'u' || w.rat(3) == 'v'))) &&
                (!(w.len() == 3 && w.rat(1) == 'd' && w.rat(2) == 'o')));
        if (w.len() == 2 && (w.at(0) != 'i' || w.at(1) != 'n')) { w.e = keep; w.type &= ~(u64)EN_AdjSuperlative; }
      } else {
        switch (w.rat(0)) {
          case 'd': case 'k': case 'm': case 'y': break;
          case 'g':
            if (!(w.len() > 3 && (w.rat(1) == 'n' || w.rat(1) == 'r') && !bytes_eq(&w.L[w.e - 3], "cong", 4))) { w.e = keep; w.type &= ~(u64)EN_AdjSuperlative; }
            else w.e += (w.rat(2) == 'a');
            break;
          case 'i': w.L[w.e] = 'y'; break;
          case 'l':
            if (w.e == w.s + 1 || bytes_eq(&w.L[w.e - 2], "mo", 2)) { w.e = keep; w.type &= ~(u64)EN_AdjSuperlative; }
            else w.e += !vowel(w.rat(1));
            break;
          case 'n':
            if (w.len() < 3 || !vowel(w.rat(1)) || !vowel(w.rat(2))) { w.e = keep; w.type &= ~(u64)EN_AdjSuperlative; }
            break;
          case 'r':
            if (w.len() > 3 && vowel(w.rat(1)) && vowel(w.rat(2))) w.e += (w.rat(2) == 'u') && (w.rat(1) == 'a' || w.rat(1) == 'i');
            else { w.e = keep; w.type &= ~(u64)EN_AdjSuperlative; }
            break;
          case 's': ++w.e; break;
          case 'w':
            if (!(w.len() > 2 && vowel(w.rat(1)))) { w.e = keep; w.type &= ~(u64)EN_AdjSuperlative; }
            break;
          case 'h':
            if (!(w.len() > 2 && !vowel(w.rat(1)))) { w.e = keep; w.type &= ~(u64)EN_AdjSuperlative; }
            break;
          default: w.e += 3; w.type &= ~(u64)EN_AdjSuperlative;
        }
      }
    }
    return (w.type & EN_AdjSuperlative) > 0;
  }
  P8_HD static bool step0(Word& w) {
    if (w.ends("'s'")) { w.e -= 3; w.type |= EN_Plural; return true; }
    if (w.ends("'s")) { w.e -= 2; w.type |= EN_Plural; return true; }
    if (w.ends("'")) { w.e -= 1; w.type |= EN_Plural; return true; }
    return false;
  }
  P8_HD static bool step1a(Word& w) {
    if (w.ends("sses")) { w.e -= 2; w.type |= EN_Plural; return true; }
    if (w.ends("ied") || w.ends("ies")) { w.type |= (w.rat(0) == 'd') ? EN_PastTense : EN_Plural; w.e -= 1 + (w.len() > 4); return true; }
    if (w.ends("us") || w.ends("ss")) return false;
    if (w.rat(0) == 's' && w.len() > 2)
      for (int i = w.s; i <= w.e - 2; ++i)
        if (vowel(w.L[i])) { --w.e; w.type |= EN_Plural; return true; }
    if (w.ends("n't") && w.len() > 4) {
      switch (w.rat(3)) {
        case 'a': if (w.rat(4) == 'c') w.e -= 2; else w.swap_suffix("n't", "ll"); break;
        case 'i': w.swap_suffix("in't", "m"); break;
        case 'o': if (w.rat(4) == 'w') w.swap_suffix("on't", "ill"); else w.e -= 3; break;
        default: w.e -= 3;
      }
      w.type |= EN_Negation;
      return true;
    }
    if (w.ends("hood") && w.len() > 7) { w.e -= 4; return true; }
    return false;
  }
  P8_HD static bool step1b(Word& w, u32 r1) {
    const char* suf[6] = {"eedly", "eed", "ed", "edly", "ing", "ingly"};
    const u8 len[6] = {5, 3, 2, 4, 3, 5};
    const char last[6] = {'y', 'd', 'd', 'y', 'g', 'y'};
    const u64 typ[6] = {EN_AdverbOfManner, 0, EN_PastTense, EN_AdverbOfManner | EN_PastTense, EN_PresentParticiple, EN_AdverbOfManner | EN_PresentParticiple};
    for (int i = 0; i < 6; ++i) {
      if (!ends_tab(w, suf[i], len[i], last[i])) continue;
      if (i < 2) {
        if (in_rn(w, r1, len[i])) w.e -= 1 + i * 2;
      } else {
        const u8 keep = w.e;
        w.e -= len[i];
        if (!has_vowel(w)) { w.e = keep; return false; }
        if (w.ends("at") || w.ends("bl") || w.ends("iz") || short_word(w)) w.append('e');
        else if (w.len() > 2) {
          if (w.rat(0) == w.rat(1) && in_set(w.rat(0), "bdfgmnprt")) --w.e;
          else if (i == 2 || i == 3) {
            switch (w.rat(0)) {
              case 'c': case 's': case 'v': w.e += !(w.ends("ss") || w.ends("ias")); break;
              case 'd': w.e += vowel(w.rat(1)) && !in_set(w.rat(2), "aeio"); break;
              case 'k': w.e += w.ends("uak"); break;
              case 'l': w.e += in_set(w.rat(1), "bcdfgkptyz") || (in_set(w.rat(1), "aiou") && !vowel(w.rat(2))); break;
            }
          } else if (i >= 4) {
            switch (w.rat(0)) {
              case 'd': if (vowel(w.rat(1)) && w.rat(2) != 'a' && w.rat(2) != 'e' && w.rat(2) != 'o') w.append('e'); break;
              case 'g':
                if (in_set(w.rat(1), "adeilru") ||
                    (w.rat(1) == 'n' && (w.rat(2) == 'e' || (w.rat(2) == 'u' && w.rat(3) != 'b' && w.rat(3) != 'd') ||
                                         (w.rat(2) == 'a' && (w.rat(3) == 'r' || (w.rat(3) == 'h' && w.rat(4) == 'c'))) ||
                                         (w.ends("ring") && (w.rat(4) == 'c' || w.rat(4) == 'f')))))
                  w.append('e');
                break;
              case 'l':
                if (!(w.rat(1) == 'l' || w.rat(1) == 'r' || w.rat(1) == 'w' || (vowel(w.rat(1)) && vowel(w.rat(2))))) w.append('e');
                if (w.ends("uell") && w.len() > 4 && w.rat(4) != 'q') --w.e;
                break;
              case 'r':
                if (((w.rat(1) == 'i' && w.rat(2) != 'a' && w.rat(2) != 'e' && w.rat(2) != 'o') ||
                     (w.rat(1) == 'a' && !(w.rat(2) == 'e' || w.rat(2) == 'o' || (w.rat(2) == 'l' && w.rat(3) == 'l'))) ||
                     (w.rat(1) == 'o' && !(w.rat(2) == 'o' || (w.rat(2) == 't' && w.rat(3) != 's'))) ||
                     w.rat(1) == 'c' || w.rat(1) == 't') && !w.ends("str"))
                  w.append('e');
                break;
              case 't': if (w.rat(1) == 'o' && w.rat(2) != 'g' && w.rat(2) != 'l' && w.rat(2) != 'i' && w.rat(2) != 'o') w.append('e'); break;
              case 'u': if (!(w.len() > 3 && vowel(w.rat(1)) && vowel(w.rat(2)))) w.append('e'); break;
              case 'z':
                if (w.ends("izz") && w.len() > 3 && (w.rat(3) == 'h' || w.rat(3) == 'u')) --w.e;
                else if (w.rat(1) != 't' && w.rat(1) != 'z') w.append('e');
                break;
              case 'k': if (w.ends("uak")) w.append('e'); break;
              case 'b': case 'c': case 's': case 'v':
                if (!((w.rat(0) == 'b' && (w.rat(1) == 'm' || w.rat(1) == 'r')) || w.ends("ss") || w.ends("ias") || w.is("zinc"))) w.append('e');
                break;
            }
          }
        }
      }
      w.type |= typ[i];
      return true;
    }
    return false;
  }
  P8_HD static bool step1c(Word& w) {
    if (w.len() > 2 && lower(w.rat(0)) == 'y' && !vowel(w.rat(1))) { w.L[w.e] = 'i'; return true; }
    return false;
  }
  P8_HD static bool step2(Word& w, u32 r1) {
    const char* from[22] = {"ization", "ational", "ousness", "iveness", "fulness", "tional", "lessli", "biliti", "entli", "ation", "alism",
                            "aliti", "fulli", "ousli", "iviti", "enci", "anci", "abli", "izer", "ator", "alli", "bli"};
    const char* to[22] = {"ize", "ate", "ous", "ive", "ful", "tion", "less", "ble", "ent", "ate", "al", "al", "ful", "ous", "ive", "ence",
                          "ance", "able", "ize", "ate", "al", "ble"};
    const u64 typ[22] = {EN_ION, EN_ION | EN_AL, EN_NESS, EN_NESS, EN_NESS, EN_ION | EN_AL, EN_AdverbOfManner, EN_AdverbOfManner | EN_ITY,
                         EN_AdverbOfManner, EN_ION, 0, EN_ITY, EN_AdverbOfManner, EN_AdverbOfManner, EN_ITY, 0, 0, EN_AdverbOfManner, 0, 0,
                         EN_AdverbOfManner, EN_AdverbOfManner};
    const u8 len[22] = {7, 7, 7, 7, 7, 6, 6, 6, 5, 5, 5, 5, 5, 5, 5, 4, 4, 4, 4, 4, 4, 3};
    const char last[22] = {'n', 'l', 's', 's', 's', 'l', 'i', 'i', 'i', 'n', 'm', 'i', 'i', 'i', 'i', 'i', 'i', 'i', 'r', 'r', 'i', 'i'};
    for (int i = 0; i < 22; ++i)
      if (ends_tab(w, from[i], len[i], last[i]) && in_rn(w, r1, len[i])) { w.swap_suffix(from[i], to[i]); w.type |= typ[i]; return true; }
    if (w.ends("logi") && in_rn(w, r1, 3)) { --w.e; return true; }
    if (w.ends("li")) {
      if (in_rn(w, r1, 2) && in_set(w.rat(2), "cdeghkmnrt")) { w.e -= 2; w.type |= EN_AdverbOfManner; return true; }
      if (w.len() > 3) {
        switch (w.rat(2)) {
          case 'b': w.L[w.e] = 'e'; w.type |= EN_AdverbOfManner; return true;
          case 'i': if (w.len() > 4) { w.e -= 2; w.type |= EN_AdverbOfManner; return true; } break;
          case 'l': if (w.len() > 5 && (w.rat(3) == 'a' || w.rat(3) == 'u')) { w.e -= 2; w.type |= EN_AdverbOfManner; return true; } break;
          case 's': w.e -= 2; w.type |= EN_AdverbOfManner; return true;
          case 'e': case 'g': case 'm': case 'n': case 'r': case 'w':
            if (w.len() > (u32)(4 + (w.rat(2) == 'r'))) { w.e -= 2; w.type |= EN_AdverbOfManner; return true; }
        }
      }
    }
    return false;
  }
  P8_HD static bool step3(Word& w, u32 r1, u32 r2) {
    const char* from[8] = {"ational", "tional", "alize", "icate", "iciti", "ical", "ful", "ness"};
    const char* to[8] = {"ate", "tion", "al", "ic", "ic", "ic", "", ""};
    const u64 typ[8] = {EN_ION | EN_AL, EN_ION | EN_AL, 0, 0, EN_ITY, EN_AL, EN_AdjFull, EN_NESS};
    bool r = false;
    const u8 len[8] = {7, 6, 5, 5, 5, 4, 3, 4};
    const char last[8] = {'l', 'l', 'e', 'e', 'i', 'l', 'l', 's'};
    for (int i = 0; i < 8; ++i)
      if (ends_tab(w, from[i], len[i], last[i]) && in_rn(w, r1, len[i])) { w.swap_suffix(from[i], to[i]); w.type |= typ[i]; r = true; break; }
    if (w.ends("ative") && in_rn(w, r2, 5)) { w.e -= 5; w.type |= EN_IVE; return true; }
    if (w.len() > 5 && w.ends("less")) { w.e -= 4; w.type |= EN_AdjWithout; return true; }
    return r;
  }
  P8_HD static bool step4(Word& w, u32 r2) {
    const char* suf[20] = {"al", "ance", "ence", "er", "ic", "able", "ible", "ant", "ement", "ment", "ent", "ou", "ism", "ate", "iti", "ous",
                           "ive", "ize", "sion", "tion"};
    const u64 typ[20] = {EN_AL, EN_NCE, EN_NCE, 0, EN_IC, EN_Capable, EN_Capable, EN_NT, 0, 0, EN_NT, 0, 0, 0, EN_ITY, EN_OUS, EN_IVE, 0, EN_ION, EN_ION};
    bool r = false;
    const u8 len[20] = {2, 4, 4, 2, 2, 4, 4, 3, 5, 4, 3, 2, 3, 3, 3, 3, 3, 3, 4, 4};
    const char last[20] = {'l', 'e', 'e', 'r', 'c', 'e', 'e', 't', 't', 't', 't', 'u', 'm', 'e', 'i', 's', 'e', 'e', 'n', 'n'};
    for (int i = 0; i < 20; ++i) {
      if (ends_tab(w, suf[i], len[i], last[i]) && in_rn(w, r2, len[i])) {
        w.e -= (u8)(len[i] - (i > 17));
        if (i != 10 || w.rat(0) != 'm') w.type |= typ[i];
        if (i == 0 && w.ends("nti")) { --w.e; r = true; continue; }
        return true;
      }
    }
    return r;
  }
  P8_HD static bool step5(Word& w, u32 r1, u32 r2) {
    if (w.rat(0) == 'e' && !w.is("here")) {
      if (in_rn(w, r2, 1)) --w.e;
      else if (in_rn(w, r1, 1)) { --w.e; w.e += short_syllable(w); }
      else return false;
      return true;
    }
    if (w.len() > 1 && w.rat(0) == 'l' && in_rn(w, r2, 1) && w.rat(1) == 'l') { --w.e; return true; }
    return false;
  }
  P8_HD static bool stem(Word& w) {
    if (w.len() < 2) { rehash(w); return false; }
    bool r = (w.s != w.e && w.at(0) == '\'');
    w.s += (u8)r;
    r |= prefixes(w);
    r |= superlatives(w);
    {
      const char* a[18] = {"skis", "skies", "dying", "lying", "tying", "idly", "gently", "ugly", "early", "only", "singly", "sky", "news",
                           "howe", "atlas", "cosmos", "bias", "andes"};
      const char* b[11] = {"ski", "sky", "die", "lie", "tie", "idle", "gentle", "ugli", "earli", "onli", "singl"};
      const u64 t[18] = {W_Noun | EN_Plural, EN_Plural, EN_PresentParticiple, EN_PresentParticiple, EN_PresentParticiple, EN_AdverbOfManner,
                         EN_AdverbOfManner, EN_Adjective, EN_Adjective | EN_AdverbOfManner, 0, EN_AdverbOfManner, W_Noun, W_Noun, 0, W_Noun, W_Noun, W_Noun, 0};
      const u8 len[18] = {4, 5, 5, 5, 5, 4, 6, 4, 5, 4, 6, 3, 4, 4, 5, 6, 4, 5};
      const char first[18] = {'s', 's', 'd', 'l', 't', 'i', 'g', 'u', 'e', 'o', 's', 's', 'n', 'h', 'a', 'c', 'b', 'a'};
      for (int i = 0; i < 18; ++i)
        if (is_tab(w, a[i], len[i], first[i])) {
          if (i < 11) { const int n = cstrlen(b[i]); for (int k = 0; k < n; ++k) w.L[w.s + k] = (u8)b[i][k]; w.e = (u8)(w.s + (u8)(n - 1)); }
          rehash(w);
          w.type |= t[i];
          w.language = LANG_EN;
          return i < 11;
        }
    }
    if (w.at(0) == 'y') w.L[w.s] = 'Y';
    for (int i = w.s + 1; i <= w.e; ++i) if (vowel(w.L[i - 1]) && w.L[i] == 'y') w.L[i] = 'Y';
    const u32 r1 = region1(w), r2 = region(w, r1, "aeiouy");
    r |= step0(w);
    r |= step1a(w);
    {
      const char* a[8] = {"inning", "outing", "canning", "herring", "earring", "proceed", "exceed", "succeed"};
      const u8 len[8] = {6, 6, 7, 7, 7, 7, 6, 7};
      const char first[8] = {'i', 'o', 'c', 'h', 'e', 'p', 'e', 's'};
      for (int i = 0; i < 8; ++i)
        if (is_tab(w, a[i], len[i], first[i])) { rehash(w); w.type |= i < 5 ? W_Noun : W_Verb; w.language = LANG_EN; return r; }
    }
    r |= step1b(w, r1);
    r |= step1c(w);
    r |= step2(w, r1);
    r |= step3(w, r1, r2);
    r |= step4(w, r2);
    r |= step5(w, r1, r2);
    for (u8 i = w.s; i <= w.e; ++i) if (w.L[i] == 'Y') w.L[i] = 'y';
    if (!w.type || w.type == EN_Plural) {
      if ((w.is("he") || w.is("him") || w.is("his") || w.is("himself") || w.is("man") || w.is("men") || w.is("boy") || w.is("husband") || w.is("actor"))) { r = true; w.type |= EN_Male; }
      else if ((w.is("she") || w.is("her") || w.is("herself") || w.is("woman") || w.is("women") || w.is("girl") || w.is("wife") || w.is("actress"))) { r = true; w.type |= EN_Female; }
    }
    if (!r) r = (w.is("the") || w.is("be") || w.is("to") || w.is("of") || w.is("and") || w.is("in") || w.is("that") || w.is("you") || w.is("have") || w.is("with") || w.is("from") || w.is("but"));
    rehash(w);
    if (r) w.language = LANG_EN;
    return r;
  }
};

// ---------------------------------------------------------------- French (paq8.cpp:2433-2821)
#define P8_FR_VOWELS "aeiouy\xE2\xE0\xEB\xE9\xEA\xE8\xEF\xEE\xF4\xFB\xF9"
struct StemFR {
  P8_HD static bool vowel(int c) { return in_set(c, P8_FR_VOWELS); }
  P8_HD static void rehash(Word& w) {
    w.hash[2] = w.hash[3] = (u64)(u32)~0xeff1caceu;
    for (int i = w.s; i <= w.e; ++i) {
      const u8 l = w.L[i];
      w.hash[2] = w.hash[2] * 251 * 32 + l;
      if (vowel(l)) w.hash[3] = w.hash[3] * 997 * 16 + l;
      else if (l >= 'b' && l <= 'z') w.hash[3] = w.hash[3] * 271 * 32 + (l - 97);
      else w.hash[3] = w.hash[3] * 11 * 32 + l;
    }
  }
  P8_HD static void convert_utf8(Word& w) {
    for (int i = w.s; i < w.e; ++i) {
      const u8 c = (u8)(w.L[i + 1] + ((w.L[i + 1] < 0xA0) ? 0x60 : 0x40));
      if (w.L[i] == 0xC3 && (vowel(c) || (w.L[i + 1] & 0xDF) == 0x87)) {
        w.L[i] = c;
        if (i + 1 < w.e) for (int k = 0; k < w.e - i - 1; ++k) w.L[i + 1 + k] = w.L[i + 2 + k];
        w.e--;
      }
    }
  }
  P8_HD static void mark_vowels(Word& w) {
    for (int i = w.s; i <= w.e; ++i) {
      switch (w.L[i]) {
        case 'i': case 'u':
          if (i > w.s && i < w.e && (vowel(w.L[i - 1]) || (w.L[i - 1] == 'q' && w.L[i] == 'u')) && vowel(w.L[i + 1])) w.L[i] = (u8)upper(w.L[i]);
          break;
        case 'y':
          if ((i > w.s && vowel(w.L[i - 1])) || (i < w.e && vowel(w.L[i + 1]))) w.L[i] = (u8)upper(w.L[i]);
      }
    }
  }
  P8_HD static u32 rv(const Word& w) {
    const u32 len = w.len(), res = w.s + len;
    if (len >= 3 && ((vowel(w.L[w.s]) && vowel(w.L[w.s + 1])) || w.starts("par") || w.starts("col") || w.starts("tap"))) return w.s + 3;
    for (int i = w.s + 1; i <= w.e; ++i) if (vowel(w.L[i])) return (u32)i + 1;
    return res;
  }
  P8_HD static bool step1(Word& w, u32 RV, u32 R1, u32 R2, bool* force2a) {
    const char* S[39] = {"ance", "iqUe", "isme", "able", "iste", "eux", "ances", "iqUes", "ismes", "ables", "istes",
                         "atrice", "ateur", "ation", "atrices", "ateurs", "ations", "logie", "logies", "usion", "ution", "usions", "utions",
                         "ence", "ences", "issement", "issements", "ement", "ements", "it\xE9", "it\xE9s", "if", "ive", "ifs", "ives",
                         "euse", "euses", "ment", "ments"};
    int i = 0;
    for (; i < 11; ++i)
      if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i]))) { w.e -= (u8)cstrlen(S[i]); if (i == 3) w.type |= FR_Adjective; return true; }
    for (; i < 17; ++i)
      if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i]))) { w.e -= (u8)cstrlen(S[i]); if (w.ends("ic")) w.swap_suffix("c", "qU"); return true; }
    for (; i < 25; ++i)
      if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i]))) {
        w.e -= (u8)((u8)cstrlen(S[i]) - 1 - (i < 19) * 2);
        if (i > 22) { w.e += 2; w.L[w.e] = 't'; }
        return true;
      }
    for (; i < 27; ++i)
      if (w.ends(S[i]) && in_rn(w, R1, cstrlen(S[i])) && !vowel(w.rat((u8)cstrlen(S[i])))) { w.e -= (u8)cstrlen(S[i]); return true; }
    for (; i < 29; ++i)
      if (w.ends(S[i]) && in_rn(w, RV, cstrlen(S[i]))) {
        w.e -= (u8)cstrlen(S[i]);
        if (w.ends("iv") && in_rn(w, R2, 2)) { w.e -= 2; if (w.ends("at") && in_rn(w, R2, 2)) w.e -= 2; }
        else if (w.ends("eus")) { if (in_rn(w, R2, 3)) w.e -= 3; else if (in_rn(w, R1, 3)) w.L[w.e] = 'x'; }
        else if ((w.ends("abl") && in_rn(w, R2, 3)) || (w.ends("iqU") && in_rn(w, R2, 3))) w.e -= 3;
        else if ((w.ends("i\xE8r") && in_rn(w, RV, 3)) || (w.ends("I\xE8r") && in_rn(w, RV, 3))) { w.e -= 2; w.L[w.e] = 'i'; }
        return true;
      }
    for (; i < 31; ++i)
      if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i]))) {
        w.e -= (u8)cstrlen(S[i]);
        if (w.ends("abil")) { if (in_rn(w, R2, 4)) w.e -= 4; else { w.e--; w.L[w.e] = 'l'; } }
        else if (w.ends("ic")) { if (in_rn(w, R2, 2)) w.e -= 2; else w.swap_suffix("c", "qU"); }
        else if (w.ends("iv") && in_rn(w, R2, 2)) w.e -= 2;
        return true;
      }
    for (; i < 35; ++i)
      if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i]))) {
        w.e -= (u8)cstrlen(S[i]);
        if (w.ends("at") && in_rn(w, R2, 2)) {
          w.e -= 2;
          if (w.ends("ic")) { if (in_rn(w, R2, 2)) w.e -= 2; else w.swap_suffix("c", "qU"); }
        }
        return true;
      }
    for (; i < 37; ++i)
      if (w.ends(S[i])) {
        if (in_rn(w, R2, cstrlen(S[i]))) { w.e -= (u8)cstrlen(S[i]); return true; }
        if (in_rn(w, R1, cstrlen(S[i]))) { w.swap_suffix(S[i], "eux"); return true; }
      }
    for (; i < 39; ++i)
      if (w.ends(S[i]) && in_rn(w, RV + 1, cstrlen(S[i])) && vowel(w.rat((u8)cstrlen(S[i])))) { w.e -= (u8)cstrlen(S[i]); *force2a = true; return true; }
    if (w.ends("eaux") || w.is("eaux")) { w.e--; w.type |= FR_Plural; return true; }
    if (w.ends("aux") && in_rn(w, R1, 3)) { w.e--; w.L[w.e] = 'l'; w.type |= FR_Plural; return true; }
    if (w.ends("amment") && in_rn(w, RV, 6)) { w.swap_suffix("amment", "ant"); *force2a = true; return true; }
    if (w.ends("emment") && in_rn(w, RV, 6)) { w.swap_suffix("emment", "ent"); *force2a = true; return true; }
    return false;
  }
  P8_HD static bool step2a(Word& w, u32 RV) {
    const char* S[35] = {"issaIent", "issantes", "iraIent", "issante", "issants", "issions", "irions", "issais", "issait", "issant", "issent",
                         "issiez", "issons", "irais", "irait", "irent", "iriez", "irons", "iront", "isses", "issez", "\xEEmes", "\xEEtes", "irai",
                         "iras", "irez", "isse", "ies", "ira", "\xEEt", "ie", "ir", "is", "it", "i"};
    for (int i = 0; i < 35; ++i)
      if (w.ends(S[i]) && in_rn(w, RV + 1, cstrlen(S[i])) && !vowel(w.rat((u8)cstrlen(S[i])))) {
        w.e -= (u8)cstrlen(S[i]);
        if (i == 31) w.type |= W_Verb;
        return true;
      }
    return false;
  }
  P8_HD static bool step2b(Word& w, u32 RV, u32 R2) {
    const char* S[38] = {"eraIent", "assions", "erions", "assent", "assiez", "\xE8rent", "erais", "erait", "eriez", "erons", "eront", "aIent",
                         "antes", "asses", "ions", "erai", "eras", "erez", "\xE2mes", "\xE2tes", "ante", "ants", "asse", "\xE9" "es", "era", "iez",
                         "ais", "ait", "ant", "\xE9" "e", "\xE9s", "er", "ez", "\xE2t", "ai", "as", "\xE9", "a"};
    for (int i = 0; i < 38; ++i)
      if (w.ends(S[i]) && in_rn(w, RV, cstrlen(S[i]))) {
        if (S[i][0] == 'a' || S[i][0] == '\xE2') {
          w.e -= (u8)cstrlen(S[i]);
          if (w.ends("e") && in_rn(w, RV, 1)) w.e--;
          return true;
        }
        if (i != 14 || in_rn(w, R2, cstrlen(S[i]))) { w.e -= (u8)cstrlen(S[i]); return true; }
      }
    return false;
  }
  P8_HD static bool step4(Word& w, u32 RV, u32 R2) {
    bool r = false;
    if (w.len() >= 2 && w.L[w.e] == 's' && !in_set(w.rat(1), "aiou\xE8s")) { w.e--; r = true; }
    const char* S[7] = {"i\xE8re", "I\xE8re", "ion", "ier", "Ier", "e", "\xEB"};
    for (int i = 0; i < 7; ++i)
      if (w.ends(S[i]) && in_rn(w, RV, cstrlen(S[i]))) {
        if (i == 2) {
          const int prec = w.rat(3);
          if (in_rn(w, R2, 3) && in_rn(w, RV + 1, 3) && (prec == 's' || prec == 't')) { w.e -= 3; return true; }
        } else if (i == 5) { w.e--; return true; }
        else if (i == 6) { if (w.ends("gu\xEB")) { w.e--; return true; } }
        else { w.swap_suffix(S[i], "i"); return true; }
      }
    return r;
  }
  P8_HD static bool stem(Word& w) {
    convert_utf8(w);
    if (w.len() < 2) { rehash(w); return false; }
    {
      const char* a[3] = {"monument", "yeux", "travaux"};
      const char* b[3] = {"monument", "oeil", "travail"};
      const u64 t[3] = {W_Noun, W_Noun | FR_Plural, W_Noun | FR_Plural};
      for (int i = 0; i < 3; ++i)
        if (w.is(a[i])) {
          const int n = cstrlen(b[i]);
          for (int k = 0; k < n; ++k) w.L[w.s + k] = (u8)b[i][k];
          w.e = (u8)(w.s + (u8)(n - 1));
          rehash(w);
          w.type |= t[i];
          w.language = LANG_FR;
          return true;
        }
    }
    mark_vowels(w);
    const u32 RV = rv(w), R1 = region(w, 0, P8_FR_VOWELS), R2 = region(w, R1, P8_FR_VOWELS);
    bool next = false, r = step1(w, RV, R1, R2, &next);
    next |= !r;
    if (next) {
      next = !step2a(w, RV);
      r |= !next;
      if (next) r |= step2b(w, RV, R2);
    }
    if (r) { u8& f = w.L[w.e]; if (f == 'Y') f = 'i'; else if (f == 0xE7) f = 'c'; }
    else r |= step4(w, RV, R2);
    {   // Step5
      bool s5 = false;
      if (w.ends("enn") || w.ends("onn") || w.ends("ett") || w.ends("ell") || w.ends("eill")) { w.e--; s5 = true; }
      r |= s5;
    }
    {   // Step6
      bool s6 = false;
      for (int i = w.e; i >= w.s; --i)
        if (vowel(w.L[i])) {
          if (i < w.e && (w.L[i] & 0xFE) == 0xE8) { w.L[i] = 'e'; s6 = true; }
          break;
        }
      r |= s6;
    }
    for (int i = w.s; i <= w.e; ++i) w.L[i] = (u8)lower(w.L[i]);
    if (!r) r = (w.is("de") || w.is("la") || w.is("le") || w.is("et") || w.is("en") || w.is("un") || w.is("une") || w.is("du") || w.is("que") || w.is("pas"));
    rehash(w);
    if (r) w.language = LANG_FR;
    return r;
  }
};

// ---------------------------------------------------------------- German (paq8.cpp:2831-2996)
#define P8_DE_VOWELS "aeiouy\xE4\xF6\xFC"
struct StemDE {
  P8_HD static bool vowel(int c) { return in_set(c, P8_DE_VOWELS); }
  P8_HD static void rehash(Word& w) {
    w.hash[2] = w.hash[3] = (u64)(u32)~0xbea7ab1eu;
    for (int i = w.s; i <= w.e; ++i) {
      const u8 l = w.L[i];
      w.hash[2] = w.hash[2] * 263 * 32 + l;
      if (vowel(l)) w.hash[3] = w.hash[3] * 997 * 16 + l;
      else if (l >= 'b' && l <= 'z') w.hash[3] = w.hash[3] * 251 * 32 + (l - 97);
      else w.hash[3] = w.hash[3] * 11 * 32 + l;
    }
  }
  P8_HD static bool valid_ending(int c, bool with_r = false) { return in_set(c, "bdfghklmnt") || (with_r && c == 'r'); }
  P8_HD static void move(u8* L, int d, int s, int n) { u8 t[8]; for (int k = 0; k < n; ++k) t[k] = L[s + k]; for (int k = 0; k < n; ++k) L[d + k] = t[k]; }
  // GermanStemmer::ConvertUTF8 closes the gap with memcpy(&L[d], &L[d + 1], n) (paq8.cpp:2851): source and destination
  // overlap, so the result is whatever the compiled copy does. g++ -O2, the build the reference's outputs come from, expands
  // it inline: whole 8/4/2/1-byte loads and stores, the tail chunk after the head, then 8-byte words from the first 8-aligned
  // destination (the word's letters are 8-aligned). A word of 5-8 bytes after the umlaut thereby loses a letter and repeats
  // its last one (m ü l l e r -> m ü l e r r). Restated step for step.
  P8_HD static void close_gap(u8* L, int d, int n) {
    if (n >= 8) {
      move(L, d, d + 1, 8);
      move(L, d + n - 8, d + 1 + n - 8, 8);
      const int a = 8 - (d & 7);
      for (int k = 0; k < ((n - a) >> 3); ++k) move(L, d + a + 8 * k, d + 1 + a + 8 * k, 8);
    } else if (n & 4) {
      move(L, d, d + 1, 4);
      move(L, d + n - 4, d + 1 + n - 4, 4);
    } else if (n) {
      move(L, d, d + 1, 1);
      if (n & 2) move(L, d + n - 2, d + 1 + n - 2, 2);
    }
  }
  P8_HD static bool stem(Word& w) {
    for (int i = w.s; i < w.e; ++i) {   // ConvertUTF8
      const u8 c = (u8)(w.L[i + 1] + ((w.L[i + 1] < 0x9F) ? 0x60 : 0x40));
      if (w.L[i] == 0xC3 && (vowel(c) || c == 0xDF)) {
        w.L[i] = c;
        if (i + 1 < w.e) close_gap(w.L, i + 1, w.e - i - 1);
        w.e--;
      }
    }
    if (w.len() < 2) { rehash(w); return false; }
    for (int i = w.s; i <= w.e; ++i)    // ReplaceSharpS
      if (w.L[i] == 0xDF) {
        w.L[i] = 's';
        if (i + 1 < 64) {
          for (int k = 64 - i - 2 - 1; k >= 0; --k) w.L[i + 2 + k] = w.L[i + 1 + k];
          w.L[i + 1] = 's';
          w.e += (w.e < 63);
        }
      }
    for (int i = w.s + 1; i < w.e; ++i) {   // MarkVowelsAsConsonants
      const u8 c = w.L[i];
      if ((c == 'u' || c == 'y') && vowel(w.L[i - 1]) && vowel(w.L[i + 1])) w.L[i] = (u8)upper(c);
    }
    u32 R1 = region(w, 0, P8_DE_VOWELS);
    const u32 R2 = region(w, R1, P8_DE_VOWELS);
    R1 = (u32)imin(3, (int)R1);
    bool r = false;
    {   // Step1
      const char* S[6] = {"em", "ern", "er", "e", "en", "es"};
      bool done = false;
      for (int i = 0; i < 6 && !done; ++i)
        if (w.ends(S[i]) && in_rn(w, R1, cstrlen(S[i]))) {
          w.e -= (u8)cstrlen(S[i]);
          if (i >= 3) w.e -= (u8)w.ends("niss");
          done = true;
        }
      if (!done && w.ends("s") && in_rn(w, R1, 1) && valid_ending(w.rat(1), true)) { w.e--; done = true; }
      r |= done;
    }
    {   // Step2
      const char* S[3] = {"en", "er", "est"};
      bool done = false;
      for (int i = 0; i < 3 && !done; ++i)
        if (w.ends(S[i]) && in_rn(w, R1, cstrlen(S[i]))) { w.e -= (u8)cstrlen(S[i]); done = true; }
      if (!done && w.ends("st") && in_rn(w, R1, 2) && w.len() > 5 && valid_ending(w.rat(2))) { w.e -= 2; done = true; }
      r |= done;
    }
    {   // Step3
      const char* S[7] = {"end", "ung", "ik", "ig", "isch", "lich", "heit"};
      bool done = false;
      int i = 0;
      for (; i < 2 && !done; ++i)
        if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i]))) {
          w.e -= (u8)cstrlen(S[i]);
          if (w.ends("ig") && w.rat(2) != 'e' && in_rn(w, R2, 2)) w.e -= 2;
          if (i) w.type |= W_Noun;
          done = true;
        }
      for (i = 2; i < 5 && !done; ++i)
        if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i])) && w.rat((u8)cstrlen(S[i])) != 'e') {
          w.e -= (u8)cstrlen(S[i]);
          if (i > 2) w.type |= DE_Adjective;
          done = true;
        }
      for (i = 5; i < 7 && !done; ++i)
        if (w.ends(S[i]) && in_rn(w, R2, cstrlen(S[i]))) {
          w.e -= (u8)cstrlen(S[i]);
          if ((w.ends("er") || w.ends("en")) && in_rn(w, R1, 2)) w.e -= 2;
          if (i > 5) w.type |= W_Noun | DE_Female;
          done = true;
        }
      if (!done && w.ends("keit") && in_rn(w, R2, 4)) {
        w.e -= 4;
        if (w.ends("lich") && in_rn(w, R2, 4)) w.e -= 4;
        else if (w.ends("ig") && in_rn(w, R2, 2)) w.e -= 2;
        w.type |= W_Noun | DE_Female;
        done = true;
      }
      r |= done;
    }
    for (int i = w.s; i <= w.e; ++i) {
      switch (w.L[i]) {
        case 0xE4: w.L[i] = 'a'; break;
        case 0xF6: case 0xFC: w.L[i] = (u8)(w.L[i] - 0x87); break;
        default: w.L[i] = (u8)lower(w.L[i]);
      }
    }
    if (!r) r = (w.is("der") || w.is("die") || w.is("das") || w.is("und") || w.is("sie") || w.is("ich") || w.is("mit") || w.is("sich") || w.is("auf") || w.is("nicht"));
    rehash(w);
    if (r) w.language = LANG_DE;
    return r;
  }
};

P8_HD inline bool lang_vowel(int lang, int c) { return lang == LANG_EN ? StemEN::vowel(c) : lang == LANG_FR ? StemFR::vowel(c) : StemDE::vowel(c); }
P8_HD inline bool lang_abbrev(int lang, const Word& w) {
  return lang == LANG_EN ? (w.is("mr") || w.is("mrs") || w.is("ms") || w.is("dr") || w.is("st") || w.is("jr")) : lang == LANG_FR ? (w.is("m") || w.is("mm")) : (w.is("fr") || w.is("hr") || w.is("hrn"));
}

}  // namespace p8
}  // namespace cmixb200
#endif
