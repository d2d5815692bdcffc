// tools/fxcm_check.cpp — CPU pinning of the resident FXCM model (cmix_b200/csrc/fxcm_model.h) against per-bit dumps of
// the UNMODIFIED reference (oracle/_ref/oracle_dump, level >= 1): the 431 exported 12-bit codes of every bit must be
// identical. TEST INFRASTRUCTURE: compiled and run by tests/test_fxcm_model.py and by hand; not part of the product.
//
//   g++ -O2 -std=c++17 -I cmix_b200/csrc tools/fxcm_check.cpp -o /tmp/fxcm_check
//   /tmp/fxcm_check <dump prefix> [dictionary | -] [max_bytes] [crc_out]
//
// The dump supplies the coded stream (<prefix>.stream), the reference's codes (<prefix>.ext.u16, [bit][2022]) and the
// LSTM feedback FXCM consumed (<prefix>.lstmfx.u32). With a dictionary the reference pretrains on a 5-byte header plus
// the dictionary text (preprocessor.cpp:37-69) before the first coded bit; so does this tool.
// With crc_out it writes one CRC32 per 4096 bits of its OWN codes (fixture generation once the run is green).
// Built with -DCENSUS it also prints how often the coded bits reach the device-only clash path (tools/census.h), and writes
// the per-bit census log to the file the environment variable CENSUS_LOG names.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#ifdef CENSUS
#include "census.h"
#endif
#include "fxcm_host.h"

using namespace cmixb200::fx;

struct HostBackend {
  std::vector<void*> blocks;
  void* alloc(size_t bytes) { void* p = calloc(bytes ? bytes : 1, 1); blocks.push_back(p); return p; }
  void fill16(void* p, size_t n, u16 v) { u16* q = (u16*)p; for (size_t i = 0; i < n; ++i) q[i] = v; }
  void fill32(void* p, size_t n, u32 v) { u32* q = (u32*)p; for (size_t i = 0; i < n; ++i) q[i] = v; }
  void upload(void* d, const void* s, size_t bytes) { memcpy(d, s, bytes); }
  ~HostBackend() { for (void* p : blocks) free(p); }
};

static std::vector<unsigned char> slurp(const std::string& path) {
  std::vector<unsigned char> v;
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return v;
  fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
  v.resize(n);
  if (n && fread(v.data(), 1, n, f) != (size_t)n) v.clear();
  fclose(f);
  return v;
}

static uint32_t crc32_update(uint32_t crc, const void* data, size_t n) {
  static uint32_t table[256]; static bool init = false;
  if (!init) { for (uint32_t i = 0; i < 256; ++i) { uint32_t c = i; for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1; table[i] = c; } init = true; }
  const unsigned char* p = (const unsigned char*)data;
  crc = ~crc;
  for (size_t i = 0; i < n; ++i) crc = table[(crc ^ p[i]) & 255] ^ (crc >> 8);
  return ~crc;
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: fxcm_check <dump prefix> [dictionary|-] [max_bytes] [crc_out]\n"); return 2; }
  const std::string prefix = argv[1];
  const char* dict = (argc > 2 && strcmp(argv[2], "-") != 0) ? argv[2] : nullptr;
  size_t max_bytes = argc > 3 ? strtoull(argv[3], 0, 10) : ~(size_t)0;
  const char* crc_out = argc > 4 ? argv[4] : nullptr;
  std::vector<unsigned char> stream = slurp(prefix + ".stream");
  std::vector<unsigned char> fxraw = slurp(prefix + ".lstmfx.u32");
  const size_t n_bits_dump = fxraw.size() / 4;
  size_t n_bytes = n_bits_dump / 8;
  if (n_bytes > stream.size()) n_bytes = stream.size();
  if (n_bytes > max_bytes) n_bytes = max_bytes;
  const uint32_t* lfx = (const uint32_t*)fxraw.data();
  FILE* fext = fopen((prefix + ".ext.u16").c_str(), "rb");
  if (!n_bytes || (!fext && !crc_out)) { fprintf(stderr, "fxcm_check: dump %s incomplete\n", prefix.c_str()); return 2; }

  static Tables T;
  build_tables(T);
  HostDict D;
  D.load(dict);
  if (D.loaded) { T.dict_chars = D.chars.data(); T.dict_off = D.off.data(); T.dict_n = (int)D.off.size(); T.dict_loaded = 1; }
  HostBackend be;
  State* S = new State();
  TextState* X = new TextState();
  if (!build_state(be, T, *S, *X)) { fprintf(stderr, "allocation failed\n"); return 2; }
  S->text = X; S->T = &T;

  if (dict) {   // Predictor::Pretrain over header + dictionary (preprocessor.cpp:37-69), lstmpr = lstmex = 0
    std::vector<unsigned char> d = slurp(dict);
    const unsigned len = (unsigned)d.size();
    std::vector<unsigned char> pre = {0, (unsigned char)(len >> 24), (unsigned char)(len >> 16), (unsigned char)(len >> 8), (unsigned char)len};
    for (unsigned char c : d) pre.push_back(c == '\n' ? ' ' : c);
    for (unsigned char c : pre) for (int j = 7; j >= 0; --j) bit_serial(*S, (c >> j) & 1, 0, 0);
    fprintf(stderr, "pretrained on %zu bytes\n", pre.size());
  }
#ifdef CENSUS
  census::reset();
  census::open_log(getenv("CENSUS_LOG"), true);
#endif

  std::vector<uint16_t> want(2022);
  std::vector<uint32_t> crcs;
  uint32_t crc = 0;
  size_t bad_bits = 0;
  for (size_t pos = 0; pos < n_bytes; ++pos) {
    for (int j = 7; j >= 0; --j) {
      const size_t t = pos * 8 + (7 - j);
      if (fext) {
        if (fread(want.data(), 2, 2022, fext) != 2022) { fprintf(stderr, "short ext file at bit %zu\n", t); return 2; }
        int nbad = 0, first = -1;
        for (int k = 0; k < 431; ++k) if (want[k] != S->codes[k]) { if (first < 0) first = k; ++nbad; }
        if (nbad) {
          if (bad_bits < 3) {
            fprintf(stderr, "MISMATCH bit %zu (byte %zu '%c' bpos %d): %d slots differ, first slot %d want %u got %u\n", t, pos,
                    stream[pos] >= 32 && stream[pos] < 127 ? stream[pos] : '.', 7 - j, nbad, first, want[first], S->codes[first]);
            int shown = 0;
            for (int k = 0; k < 431 && shown < 24; ++k) if (want[k] != S->codes[k]) { fprintf(stderr, "  [%d] want %u got %u\n", k, want[k], S->codes[k]); ++shown; }
          }
          ++bad_bits;
          if (bad_bits >= 3) { printf("FAIL after %zu bits\n", t); return 1; }
        }
      }
      crc = crc32_update(crc, S->codes, 431 * 2);
      if ((t & 4095) == 4095) { crcs.push_back(crc); crc = 0; }
      bit_serial(*S, (stream[pos] >> j) & 1, (int)(lfx[t] & 0xffff), (int)(lfx[t] >> 16));
#ifdef CENSUS
      census::end_bit();
#endif
    }
  }
  if (crc_out) {
    FILE* f = fopen(crc_out, "wb");
    fwrite(crcs.data(), 4, crcs.size(), f);
    fclose(f);
  }
#ifdef CENSUS
  census::print(stdout, {});
#endif
  printf("%s: %zu bytes, %zu bits compared, %zu mismatching bits\n", bad_bits ? "FAIL" : "OK", n_bytes, n_bytes * 8, bad_bits);
  return bad_bits ? 1 : 0;
}
