// tools/paq8_check.cpp — CPU pinning of the resident PAQ8 model (cmix_b200/csrc/paq8_*.h) against per-bit dumps of the
// UNMODIFIED reference (oracle/_ref/oracle_dump level >= 1): slots 431..2021 of every bit's code vector (the 1591 PAQ8
// outputs) must be identical. TEST INFRASTRUCTURE, not part of the product.
//
//   g++ -O2 -std=c++17 -ffp-contract=off -I cmix_b200/csrc tools/paq8_check.cpp -o /tmp/paq8_check
//   /tmp/paq8_check <dump prefix> [pretrain file | -] [max_bytes] [crc_out] [first_slot last_slot]
//
// A pretrain file holds the bytes the reference's Pretrain() saw before the first coded bit (5-byte header + dictionary
// with '\n' -> ' ', preprocessor.cpp:37-69). With crc_out it writes one CRC32 per 4096 bits over its OWN 1591 codes.
// first_slot/last_slot (0-based within the 1591) restrict the comparison while a sub-model range is being brought up.
// Built with -DCENSUS it also prints how often the coded bits reach the device-only paths (tools/census.h), and writes the
// per-bit census log to the file the environment variable CENSUS_LOG names.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#ifdef CENSUS
#include "census.h"
#endif
#include "paq8_host.h"

using namespace cmixb200::p8;

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
  if (argc < 2) { fprintf(stderr, "usage: paq8_check <dump prefix> [pretrain|-] [max_bytes] [crc_out|-] [first last]\n"); return 2; }
  const std::string prefix = argv[1];
  const char* pre_path = (argc > 2 && strcmp(argv[2], "-") != 0) ? argv[2] : nullptr;
  size_t max_bytes = argc > 3 ? strtoull(argv[3], 0, 10) : ~(size_t)0;
  const char* crc_out = (argc > 4 && strcmp(argv[4], "-") != 0) ? argv[4] : nullptr;
  const int first = argc > 6 ? atoi(argv[5]) : 0, last = argc > 6 ? atoi(argv[6]) : 1590;
  std::vector<unsigned char> stream = slurp(prefix + ".stream");
  size_t n_bytes = stream.size() < max_bytes ? stream.size() : max_bytes;
  FILE* fext = fopen((prefix + ".ext.u16").c_str(), "rb");
  if (!n_bytes || (!fext && !crc_out)) { fprintf(stderr, "paq8_check: dump %s incomplete\n", prefix.c_str()); return 2; }
  static Tables T;
  build_tables(T);
  HostBackend be;
  State* S = new State();
  if (!build_state(be, T, *S)) { fprintf(stderr, "allocation failed\n"); return 2; }
  S->T = &T;
  if (pre_path) {
    std::vector<unsigned char> pre = slurp(pre_path);
    for (unsigned char c : pre) for (int j = 7; j >= 0; --j) bit(*S, (c >> j) & 1);
    fprintf(stderr, "pretrained on %zu bytes\n", pre.size());
  }
#ifdef CENSUS
  const std::vector<std::pair<std::string, const void*>> maps = {
      {"sparse", &S->sparse.cm}, {"sparse1", &S->sparse1.cm}, {"distance", &S->distance.cm}, {"record.cm", &S->record.cm},
      {"record.cn", &S->record.cn}, {"record.co", &S->record.co}, {"record.cp", &S->record.cp}, {"record1.cm", &S->record1.cm},
      {"record1.cn", &S->record1.cn}, {"record1.co", &S->record1.co}, {"record1.cq", &S->record1.cq},
      {"record1.cp", &S->record1.cp}, {"word", &S->word.cm}, {"nest", &S->nest.cm}, {"indirect", &S->indirect.cm},
      {"xml", &S->xml.cm}, {"order-n (history)", &S->cm}, {"text (history)", &S->text.map}, {"exe (history)", &S->exe.cm}};
  census::reset();
  census::set_maps(maps);
  census::open_log(getenv("CENSUS_LOG"), false);
#endif
  std::vector<uint16_t> want(2022);
  std::vector<uint32_t> crcs;
  uint32_t crc = 0;
  size_t bad_bits = 0;
  bool unsupported = false;
  for (size_t pos = 0; pos < n_bytes; ++pos) {
    for (int j = 7; j >= 0; --j) {
      const size_t t = pos * 8 + (7 - j);
      if (fext) {
        if (fread(want.data(), 2, 2022, fext) != 2022) { n_bytes = pos; j = -1; break; }
        int nbad = 0, f0 = -1;
        for (int k = first; k <= last; ++k) if (want[431 + k] != S->codes[k]) { if (f0 < 0) f0 = k; ++nbad; }
        if (nbad) {
          if (bad_bits < 2) {
            fprintf(stderr, "MISMATCH bit %zu (byte %zu 0x%02x bpos %d): %d slots differ, first slot %d want %u got %u\n", t, pos, stream[pos], 7 - j, nbad, f0,
                    want[431 + f0], S->codes[f0]);
            int shown = 0;
            for (int k = first; k <= last && shown < 16; ++k) if (want[431 + k] != S->codes[k]) { fprintf(stderr, "  [%d] want %u got %u\n", k, want[431 + k], S->codes[k]); ++shown; }
          }
          ++bad_bits;
          if (bad_bits >= 2) { printf("FAIL after %zu bits\n", t); return 1; }
        }
      }
      crc = crc32_update(crc, S->codes, 1591 * 2);
      if ((t & 4095) == 4095) { crcs.push_back(crc); crc = 0; }
      bit(*S, (stream[pos] >> j) & 1);
#ifdef CENSUS
      census::end_bit();
#endif
      if (S->error) {
        fprintf(stderr, "model raised error %u at bit %zu (unsupported block type)\n", S->error, t);
        printf("UNSUPPORTED after %zu bits\n", t);
        unsupported = true;   // the CRCs of the blocks completed before the error are still written
        n_bytes = pos;
        break;
      }
    }
  }
  if (crc_out) { FILE* f = fopen(crc_out, "wb"); fwrite(crcs.data(), 4, crcs.size(), f); fclose(f); }
  if (unsupported) return 3;
#ifdef CENSUS
  census::print(stdout, maps);
#endif
  printf("%s: %zu bytes, %zu mismatching bits (slots %d..%d)\n", bad_bits ? "FAIL" : "OK", n_bytes, bad_bits, first, last);
  return bad_bits ? 1 : 0;
}
