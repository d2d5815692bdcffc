// cmix_b200/csrc/paq8_host.h — host-side construction of the resident PAQ8 model (paq8_model.h / paq8_predict.h).
//
// Constant tables: the bit-history state table (reference src/models/paq8.cpp:277-341), the ASCII group tables of the text
// model (:3042-3068) and the x86 decoder's format / category tables (:6633-7050) are data, carried here as hex strings (the
// values the reference's own initialisers produce; tools/make_paq8_tables.py regenerates and checks them when the reference
// is present). squash / stretch / ilog / dt are computed as the reference computes them (integer only, :345-387, :253-266).
// Memory is obtained through the same backend concept as fxcm_host.h.
#ifndef CMIXB200_PAQ8_HOST_H
#define CMIXB200_PAQ8_HOST_H

#include <string.h>

#include <vector>

#include "paq8_top.h"

namespace cmixb200 {
namespace p8 {

inline void unhex(u8* dst, int n, const char* hex) {
  for (int i = 0; i < n; ++i) {
    auto v = [](char c) { return c <= '9' ? c - '0' : c - 'a' + 10; };
    dst[i] = (u8)(v(hex[2 * i]) * 16 + v(hex[2 * i + 1]));
  }
}

inline void build_tables(Tables& T) {
  memset(&T, 0, sizeof T);
  T.ilog = T.ilog_store;
  unhex(&T.state[0][0], 1024,
      "010200000305010004060001070a0200080c0101090d01010b0e00020f130300101702011118020112190201141b0102"
      "151c0102161d01021a1e00031f2104002023030120230301202303012023030122250202222502022225020222250202"
      "22250202222502022427010324270103242701032427010326280004292b05002a2d04012a2d04012c2f03022c2f0302"
      "2e3102032e310203303301043033010432340005352b06003639050136390501383b0402383b04023a3d03033a3d0303"
      "3c3f02043c3f02043e4101053e410105324200064337070044390601443906014649050246490502484b0403484b0403"
      "4a4d03044a4d03044c4f02054c4f02053e5101063e510106405200075345080054470701544707015649060256490602"
      "2c3b05032c3b05033a3d04043a3d04043c3103053c3103054c5902064c5902064e5b01074e5b0107505c00085d450900"
      "5e5708015e570801602d0702602d0702306302073063020758650108586501085066000967450a006857090168570901"
      "6a3908026a3908023e6d02083e6d0208586f0109586f01095070000a71550b0072570a0172570a017439090274390902"
      "3e7702093e7702095879010a5879010a5a7a000b7b550c007c610b017c610b017e390a027e390a023e81020a3e81020a"
      "6283010b6283010b5a84000c85550d0086610c0186610c0188390b0288390b023e8b020b3e8b020b628d010c628d010c"
      "5a8e000d8f5f0e0090610d0190610d0144390c0244390c023e51020c3e51020c6293010d6293010d6494000e955f0f00"
      "966b0e01966b0e016c97010e6c97010e6498000f995f10009a6b0f016c9b010f649c00109d5f11009e6b10016c9f0110"
      "64a00011a1691200a26b11016ca301116ea40012a5691300a675120176a701126ea80013a9691400aa75130176ab0113"
      "6eac0014ad691500ae75140176af01146eb00015b1691600b275150176b301156eb40016b5731700b675160176b70116"
      "78b80017b9731800ba7f170180bb011778bc0018bd731900be7f180180bf011878c00019c1731a00c27f190180c30119"
      "78c4001ac5731b00c67f1a0180c7011a78c8001bc9731c00ca7f1b0180cb011b78cc001ccd731d00ce7f1c0180cf011c"
      "78d0001dd17d1e00d27f1d0180d3011d82d4001ed57d1f00d6891e018ad7011e82d8001fd97d2000da891f018adb011f"
      "82dc0020dd7d2100de8920018adf012082e00021e17d2200e28921018ae3012182e40022e57d2300e68922018ae70122"
      "82e80023e97d2400ea8923018aeb012382ec0024ed7d2500ee8924018aef012482f00025f17d2600f28925018af30125"
      "82f40026f5872700f68926018af701268cf80027f9872800fa45270150fb01278cfc0028f9872900fa45280150fb0128"
      "8cfc0029000000000000000000000000");
  unhex(T.ascii_group_c0, 254,
      "000a00010a0a000402030a0a0a0a00000504020203030a0a0a0a0a0a0a0a000000000505090402020202030303030a0a"
      "0a0a0a0a0a0a0a0a0a0a0a0a0a0a00000000000000000508080509090605020202020202020803030303030303080a0a"
      "0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a000000000000000000000000000000000708"
      "080808080505090909090907080502020202020202020202020202020808030303030303030303030303030308080a0a"
      "0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a0a"
      "0a0a0a0a0a0a0a0a0a0a0a0a0a0a");
  unhex(T.ascii_group, 128,
      "0005050505050505050504050504050505050505050505050505050505050505060708111109110a0b0c11110d0e0f10"
      "01010101010101010101121314171516170202020202020202020202020202020202020202020202020202181b191b1a"
      "1b03030303030303030303030303030303030303030303030303031c1e1d1e1e");
  unhex(T.exe_t1, 256,
      "02020202040c000002020202040c000002020202040c000002020202040c000002020202040c000002020202040c0000"
      "02020202040c000002020202040c00000000000000000000000000000000000000000000000000000000000000000000"
      "00000202000000000c0e04060000000009090909090909090909090909090909060e0606020202020202020202020202"
      "000000000000000000000500000000000101010100000000040c00000000000004040404040404040c0c0c0c0c0c0c0c"
      "060608000202060e0400080000040f000202020204040000020202020202020209090909040404040d0d010900000000"
      "000f0000000003030000000000000303");
  unhex(T.exe_t2, 256,
      "0f0f0f0f0f0f000f00000f0f0f0f0f0f0202020202020202020f0f0f0f0f0f0f020202020f0f0f0f0202020202020202"
      "0000000000000f000f0f0f0f0f0f0f0f0202020202020202020202020202020202020202020202020202020202020202"
      "0202020202020202020202020202020206060606020202000f0f0f0f0f0f02020d0d0d0d0d0d0d0d0d0d0d0d0d0d0d0d"
      "0202020202020202020202020202020200000002060202020f0f0f0206020f0202020202020202020f0f0f0202020202"
      "020202020202020200000000000000000202020202020202020202020202020202020202020202020202020202020202"
      "0202020202020202020202020202020f");
  unhex(T.exe_t3_38, 256,
      "0202020202020202020202020f0f0f0f020f0f0f02020f020f0f0f0f0202020f0202020202020f0f020202020f0f0f0f"
      "0202020202020f02020202020202020202020f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f02020f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "02020f0f0f0f0f0f0f0f0f0f0f0f0f0f");
  unhex(T.exe_t3_3a, 256,
      "0f0f0f0f0f0f0f0f06060606060606060f0f0f0f060606060f0f0f0f0f0f0f0f0606060f0f0f0f0f0f0f0f0f0f0f0f0f"
      "0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0606060f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "060606060f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f"
      "0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f");
  unhex(T.exe_tx, 32,
      "060f0202020202020e0f02020202020202020f0f0f0f0f0f0202020f020f020f");
  unhex(T.exe_c1, 256,
      "080808080808050509090909090905020808080808080505080808080808050509090909090901070808080808080107"
      "090909090909010708080808080801070808080808080808080808080808080805050505050505050505050505050505"
      "05050e060101020205080508101010100d0d0d0d0d0d0d0d0d0d0d0d0d0d0d0d08080808080804040404040404040405"
      "040404040404040406060c0305050404040404040f0f0f0f09090f0f0f0f0f0f04040404040404040404040404040404"
      "0a0a0c0c0404040405050c0c0e0e0e0e0a0a0a0a0707040416151615161516150d0d0d0d101010100c0c0c0c10101010"
      "020e020214110808111111111111080c");
  unhex(T.exe_c2, 256,
      "141414140014141414140013001300001f1f1f1f1e1e1f1f1e1313131313131314141414140014001f1f1e1e1e1e1e1e"
      "14141414141400000200020000000000040404040404040404040404040404041f1e1e1e1e1e1e1e1e1e1e1e1e1e1e1e"
      "1d1d1d1d1d1d1d1d1d1d1d1d00001d1d1e1d1d1d1d1d1d1d0000000000001d1d0d0d0d0d0d0d0d0d0d0d0d0d0d0d0d0d"
      "040404040404040404040404040404040505130b0a0a00000505140b0a0a1c080404040b0404060600130b0b0b0b0606"
      "04041e1e1e1e1e040404040404040404001d1d1d1e1d001e1d1d1e1d1d1d1e1d1e1d1e1d1e1d001e1d1d1e1d1d1d1e1d"
      "001d1d1d1e1d1e1e1d1d1d1e1d1d1d00");
  unhex(T.exe_c3_38, 256,
      "1e1e1e1e1e1e1e1e1e1e1e1e000000001e0000001e1e001e000000001e1e1e001e1e1e1e1e1e00001e1e1e1e00000000"
      "1e1e1e1e1e1e001e1e1e1e1e1e1e1e1e1e1e000000000000000000000000000000000000000000000000000000000000"
      "000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
      "000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
      "000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
      "04040000000000000000000000000000");
  unhex(T.exe_c3_3a, 256,
      "00000000000000001e1e1e1e1e1e1e1e000000001e1e1e1e00000000000000001e1e1e00000000000000000000000000"
      "000000000000000000000000000000001e1e1e0000000000000000000000000000000000000000000000000000000000"
      "1e1e1e1e0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
      "000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
      "000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
      "00000000000000000000000000000000");
  unhex(T.exe_cx, 32,
      "09090908080808080909090808080808080800000000000008080c0c0c0c0500");
  unhex(T.exe_invalid64, 19,
      "060716171e1f272f373f606162829ad4d5d6ea");
  unhex(T.exe_prefix64, 8,
      "262e363e9bf0f2f3");
  {   // Squash / Stretch (paq8.cpp:357-387)
    static const int ts[33] = {1, 2, 3, 6, 10, 16, 27, 45, 73, 120, 194, 310, 488, 747, 1101, 1546, 2047, 2549, 2994, 3348, 3607, 3785, 3901, 3975, 4022,
                               4050, 4068, 4079, 4085, 4089, 4092, 4093, 4094};
    for (int i = -2047; i <= 2047; ++i) {
      const int w = i & 127, d = (i >> 7) + 16;
      T.squash[i + 2048] = (u16)((ts[d] * (128 - w) + ts[d + 1] * w + 64) >> 7);
    }
    int pi = 0;
    for (int x = -2047; x <= 2047; ++x) {
      const int i = squash(T, x);
      for (int j = pi; j <= i; ++j) T.stretch[j] = (short)x;
      pi = i + 1;
    }
    T.stretch[4095] = 2047;
  }
  {   // Ilog (paq8.cpp:260-266)
    u32 x = 14155776;
    for (int i = 2; i < 65536; ++i) { x += 774541002 / (i * 2 - 1); T.ilog_store[i] = (u8)(x >> 24); }
  }
  for (int i = 0; i < 1024; ++i) T.dt[i] = 16384 / (i + i + 3);
}

// Backend concept as in fxcm_host.h: alloc (zeroed), fill16, fill32, upload.
template <class B> struct P8Builder {
  B& be; const Tables& T; bool ok = true;
  template <class U> U* alloc(size_t n) { U* p = (U*)be.alloc(n * sizeof(U)); if (!p) ok = false; return p; }
  void cm(Cm& m, u64 mem, int C) {
    memset(&m, 0, sizeof m);
    const u32 buckets = (u32)(mem >> 6);
    m.t = alloc<u8>((size_t)buckets * 64);
    m.mask = buckets - 1; m.hashbits = (int)ilog2(m.mask + 1); m.C = C;
    m.sm_t = alloc<u16>((size_t)C * 256);
    std::vector<u16> init(256);
    for (int i = 0; i < 256; ++i) {
      int n0 = T.state[i][2], n1 = T.state[i][3];
      if (n0 == 0) n1 *= 64;
      if (n1 == 0) n0 *= 64;
      init[i] = (u16)(65536 * (n1 + 1) / (n0 + n1 + 2));
    }
    if (m.sm_t) for (int c = 0; c < C; ++c) be.upload(m.sm_t + c * 256, init.data(), 512);
    for (int i = 0; i < CM_CAP; ++i) { m.cp[i] = m.cp0[i] = 15; m.runp[i] = 18; }
  }
  void sm32_states(u32* dst) {   // StateMap32(256) (paq8.cpp:672-681)
    std::vector<u32> init(256);
    for (int i = 0; i < 256; ++i) {
      u32 n0 = T.state[i][2], n1 = T.state[i][3];
      if (n0 == 0) n1 *= 64;
      if (n1 == 0) n0 *= 64;
      init[i] = ((n1 << 16) / (n0 + n1 + 1)) << 16;
    }
    be.upload(dst, init.data(), 1024);
  }
  void sm32(Sm32& s, int n) {
    s.t = alloc<u32>((size_t)n); s.cxt = 0; s.n = n;
    if (!s.t) return;
    if (n == 256) sm32_states(s.t); else be.fill32(s.t, (size_t)n, 1u << 31);
  }
  void cm2(Cm2& m, u64 mem, int C) {
    memset(&m, 0, sizeof m);
    const u32 buckets = (u32)(mem >> 6);
    m.t = alloc<u8>((size_t)buckets * 64);
    m.mask = buckets - 1; m.hashbits = (int)ilog2(m.mask + 1); m.C = C;
    m.m6_t = alloc<u32>((size_t)C * 72); m.m8_t = alloc<u32>((size_t)C * 256); m.m12_t = alloc<u32>((size_t)C * 4608);
    if (!ok) return;
    be.fill32(m.m6_t, (size_t)C * 72, 1u << 31);
    be.fill32(m.m12_t, (size_t)C * 4608, 1u << 31);
    for (int c = 0; c < C; ++c) sm32_states(m.m8_t + c * 256);
    for (int i = 0; i < C; ++i) { m.bs[i] = m.bs0[i] = (i << 6) + 15; m.bh[i] = m.bs[i] + 3; }
    m.bits = 1;
  }
  void scm(Scm& c, int bits_ctx, int bits_in) {
    memset(&c, 0, sizeof c);
    c.mask = (1 << bits_ctx) - 1; c.stride = (1 << bits_in) - 1; c.btotal = bits_in;
    const size_t n = ((size_t)1 << bits_ctx) * (size_t)c.stride;
    c.data = alloc<u16>(n);
    if (c.data) be.fill16(c.data, n, 0x7FFF);
  }
  void stm(Stm& c, int bits_ctx, int bits_in) {
    memset(&c, 0, sizeof c);
    c.mask = (1 << bits_ctx) - 1; c.maskbits = bits_ctx; c.stride = (1 << bits_in) - 1; c.btotal = bits_in;
    const size_t n = ((size_t)1 << bits_ctx) * (size_t)c.stride;
    c.data = alloc<u32>(n);
    if (c.data) be.fill32(c.data, n, 0x7FFu << 20);
  }
  void imap(Imap& c, int bits_ctx, int bits_in) {
    memset(&c, 0, sizeof c);
    c.mask = (1 << bits_ctx) - 1; c.maskbits = bits_ctx; c.stride = (1 << bits_in) - 1; c.btotal = bits_in;
    c.data = alloc<u8>(((size_t)1 << bits_ctx) * (size_t)c.stride);
    sm32(c.map, 256);
  }
  template <class U> void ictx(ICtx<U>& c, int bits_ctx, int bits_in) {
    c.data = alloc<U>((size_t)1 << bits_ctx); c.ctx = 0; c.ctx_mask = (1u << bits_ctx) - 1; c.input_mask = (1u << bits_in) - 1; c.input_bits = (u32)bits_in;
  }
  void rcm(Rcm& r, u64 mem) {
    const u32 n = (u32)(mem / 4);
    r.t = alloc<u8>((size_t)n * 4); r.mask = n - 1; r.hashbits = (int)ilog2(r.mask + 1);
    r.cp = 2;   // cp = t[0] + 1: probing context 0 in the empty table returns the first element's byte 1
  }
  void apm(Sm32& s, int n) {
    s.n = n * 24; s.cxt = 0; s.t = alloc<u32>((size_t)s.n);
    if (!s.t) return;
    std::vector<u32> init((size_t)s.n);
    for (int i = 0; i < s.n; ++i) { const int p = ((i % 24 * 2 + 1) * 4096) / 48 - 2048; init[i] = ((u32)squash(T, p) << 20) + 6; }
    be.upload(s.t, init.data(), init.size() * 4);
  }
  void apm1(Apm1& a, int n) {
    a.index = 0; a.t = alloc<u16>((size_t)n * 33 + 1);
    if (!a.t) return;
    std::vector<u16> init((size_t)n * 33);
    for (size_t i = 0; i < init.size(); ++i) init[i] = (u16)(squash(T, ((int)(i % 33) - 16) * 128) * 16);
    be.upload(a.t, init.data(), init.size() * 2);
  }
};

// Fills the HOST mirror S (pointers refer to backend memory); the caller uploads it and patches S.T.
template <class B> bool build_state(B& be, const Tables& T, State& S) {
  memset(&S, 0, sizeof S);
  P8Builder<B> b{be, T};
  const u64 MEM = 0x10000ull << 11;   // level 11 (predictor.cpp:85, paq8.cpp:188-191)
  S.c0 = 1; S.pr = 2048; S.last_prediction = 2048;
  S.buf = b.template alloc<u8>((size_t)1 << 30);
  S.rnd.table[0] = 123456789; S.rnd.table[1] = 987654321;
  for (int j = 0; j < 62; ++j) S.rnd.table[j + 2] = S.rnd.table[j + 1] * 11 + S.rnd.table[j] * 23 / 16;
  for (int i = 0; i <= N_OUT; ++i) S.codes[i] = 0xFFFF;
  // contextModel2 statics
  b.cm2(S.cm, MEM * 16, 10);
  b.rcm(S.rcm7, MEM); b.rcm(S.rcm9, MEM); b.rcm(S.rcm10, MEM);
  b.sm32(S.sm0, 256); b.sm32(S.sm1, 256 * 256);
  // match model
  {
    MatchM& M = S.match;
    const u32 n = (u32)(MEM * 2 / 4);
    M.table = b.template alloc<u32>(n); M.mask = n - 1; M.hashbits = (int)ilog2(M.mask + 1);
    b.sm32(M.sm[0], 56 * 256); b.sm32(M.sm[1], 8 * 256 * 256 + 1); b.sm32(M.sm[2], 256 * 256);
    b.scm(M.scm[0], 8, 8); b.scm(M.scm[1], 11, 1); b.scm(M.scm[2], 8, 8);
    b.stm(M.maps[0], 16, 8); b.stm(M.maps[1], 22, 1); b.stm(M.maps[2], 4, 1);
    b.ictx(M.ictx, 19, 1);
  }
  {
    SparseMatchM& M = S.smatch;
    const u32 n = (u32)(MEM / 2 / 4);
    M.table = b.template alloc<u32>(n); M.mask = n - 1; M.hashbits = (int)ilog2(M.mask + 1);
    b.stm(M.maps[0], 22, 1); b.stm(M.maps[1], 14, 4); b.stm(M.maps[2], 8, 1); b.stm(M.maps[3], 19, 1);
    b.ictx(M.ictx8, 19, 1); b.ictx(M.ictx16, 16, 8);
    for (int i = 0; i < 4; ++i) { M.prev[i] = i - 1; M.next[i] = i + 1; }
    M.next[3] = -1;
  }
  b.cm(S.sparse.cm, MEM * 2, 42);
  b.cm(S.sparse1.cm, MEM * 4, 31);
  { static const int bits[7] = {7, 8, 4, 6, 4, 4, 7}; for (int k = 0; k < 7; ++k) b.scm(S.sparse1.scm[k], bits[k], 8); }
  b.cm(S.distance.cm, MEM, 3);
  S.pic.t = b.template alloc<u8>(0x10200);
  {
    Cm tmp; b.cm(tmp, 64, 3);    // three StateMaps with the state-derived initial values
    S.pic.sm_t = tmp.sm_t;
  }
  {
    RecordM& M = S.record;
    M.rlen[0] = 2; M.rlen[1] = 3; M.rlen[2] = 4;
    M.wpos1 = b.template alloc<int>(0x10000);
    b.cm(M.cm, 32768, 3); b.cm(M.cn, 32768 / 2, 3); b.cm(M.co, 32768 * 2, 3); b.cm(M.cp, MEM, 16);
    static const int mb[6][2] = {{10, 8}, {10, 8}, {8, 8}, {8, 8}, {8, 8}, {11, 1}};
    for (int k = 0; k < 6; ++k) b.stm(M.maps[k], mb[k][0], mb[k][1]);
    b.scm(M.smap[0], 11, 1); b.scm(M.smap[1], 3, 1); b.scm(M.smap[2], 19, 1);
    for (int k = 0; k < 3; ++k) b.imap(M.imap[k], 8, 8);
    b.ictx(M.ictx[0], 16, 8); b.ictx(M.ictx[1], 16, 8); b.ictx(M.ictx[2], 16, 8); b.ictx(M.ictx[3], 20, 8); b.ictx(M.ictx[4], 11, 1);
  }
  {
    Record1M& M = S.record1;
    M.wpos1 = b.template alloc<int>(0x10000);
    b.cm(M.cm, 32768, 2); b.cm(M.cn, 32768 / 2, 5); b.cm(M.co, 32768 * 4, 4); b.cm(M.cp, 32768 * 2, 3); b.cm(M.cq, 32768 * 2, 3);
  }
  {
    WordM& M = S.word;
    M.nl1 = -3; M.nl = -2; M.cword = 0; M.pword = 3;
    M.wpos = b.template alloc<int>(0x10000);
    b.cm(M.cm, MEM * 16, 61);
  }
  b.cm(S.nest.cm, MEM / 2, 12);
  {
    IndirectM& M = S.indirect;
    b.cm(M.cm, MEM, 15);
    M.t2 = b.template alloc<u16>(0x10000); M.t3 = b.template alloc<u16>(0x8000); M.t4 = b.template alloc<u16>(0x8000);
    b.ictx(M.ictx, 16, 8);
  }
  {
    static const u32 params[10] = {2, 32, 64, 4, 128, 8, 256, 16, 1024, 1536};
    static const u64 mem[10] = {6, 10, 11, 7, 12, 8, 13, 9, 2, 2};
    std::vector<DmcNode> init(255 * 256);
    for (int i = 0; i < 10; ++i) {
      Dmc& d = S.dmc[i];
      u64 n = (MEM >> 2) / mem[i] + 255 * 256;
      const u64 nmax = (1ull << 31) / sizeof(DmcNode);
      if (n > nmax) n = nmax;
      d.size = (u32)n;
      d.t = b.template alloc<DmcNode>((size_t)n);
      b.sm32(d.sm, 256);
      if (!b.ok) return false;
      Dmc h = d; h.t = init.data();
      memset(init.data(), 0, init.size() * sizeof(DmcNode));
      dmc_reset(h, params[i]);                 // the initial 256 order-1 trees (resetstategraph, paq8.cpp:7655-7677), built on the host
      be.upload(d.t, init.data(), init.size() * sizeof(DmcNode));
      d.top = h.top; d.curr = h.curr; d.extra = h.extra; d.threshold = h.threshold; d.threshold_fine = h.threshold_fine;
    }
  }
  {
    XmlM& M = S.xml;
    b.cm(M.cm, MEM / 4, 4);
    M.indent_step = 2; M.line_ending = 2;
  }
  {
    TextM& M = S.text;
    b.cm2(M.map, MEM * 16, 33);
    M.word_pos = b.template alloc<u32>(0x10000);
    M.cw_lang = 0; M.cw_slot = 0; M.pw_lang = 0; M.pw_slot = 7;
  }
  b.cm2(S.exe.cm, MEM * 2, 20);
  {
    LinearM& M = S.linear;
    for (int k = 0; k < 5; ++k) b.scm(M.smap[k], 11, 1);
    M.ols = b.template alloc<double>((size_t)3 * OLS_STRIDE);
  }
  {
    AudioM A;
    memset(&A, 0, sizeof A);
    for (int i = 0; i < AUDIO_N_PRD; ++i) for (int j = 0; j < 3; ++j) b.scm(A.scm[i][j], 11, 1);
    A.ols = b.template alloc<double>((size_t)AUDIO_OLS_DOUBLES);
    S.audio = b.template alloc<AudioM>(1);
    if (!b.ok) return false;
    be.upload(S.audio, &A, sizeof A);
  }
  S.m.w = b.template alloc<short>((size_t)N_WSETS * N_IN);
  S.m.w2 = b.template alloc<short>(32);
  if (!b.ok) return false;
  be.fill16(S.m.w, (size_t)N_WSETS * N_IN, 32);
  be.fill16(S.m.w2, 32, 0x7fff);
  for (int i = 0; i < N_SETS; ++i) S.m.pr[i] = 2048;
  S.m.pr2 = 2048;
  for (int k = 0; k < 4; ++k) b.apm(S.text_apm[k], 0x10000);
  for (int k = 0; k < 3; ++k) b.apm1(S.text_apm1[k], 0x10000);
  b.apm1(S.generic_apm1[0], 0x2000);
  for (int k = 1; k < 7; ++k) b.apm1(S.generic_apm1[k], 0x10000);
  return b.ok;
}

}  // namespace p8
}  // namespace cmixb200
#endif
