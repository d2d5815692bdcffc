// tools/ppmd_host.cpp - host build of cmix_b200/csrc/ppmd_model.h behind a two-function C API, for
// tests/test_ppmd_model.py (pins the model against fixtures made from dumps of the unmodified reference).
//   g++ -O2 -std=c++17 -ffp-contract=off -shared -fPIC tools/ppmd_host.cpp -o build/libppmd_host.so
#include <cstdlib>
#include <cstring>

#include "../cmix_b200/csrc/ppmd_model.h"

using namespace cmixb200;

// An arena of n elements: zeroed (fill 0), or every byte `fill`, so that a read of a cell the model has not written
// shows in its distribution.
template <class T> static T* arena(size_t n, int fill) {
  if (!fill) return (T*)calloc(n, sizeof(T));
  T* p = (T*)malloc(n * sizeof(T));
  if (p) memset(p, fill, n * sizeof(T));
  return p;
}

extern "C" {

// Runs the model over `stream` and writes PPMD::ByteUpdate's distribution after every byte (ppmd.cpp:1328-1338)
// to out[n][256]. Returns 0, or 1 when the arenas (arena_mb in total, filled with the byte `fill`) are exhausted.
int ppmd_host_run(const unsigned char* stream, size_t n, const unsigned char* vocab, float* out, unsigned arena_mb, int fill) {
  PpmdModel* m = new PpmdModel();
  memset(m, 0, sizeof *m);
  const size_t bytes = (size_t)arena_mb << 20;
  m->ctx_cap = (uint32_t)(bytes / 4 / sizeof(PpmdCtx));
  m->pool_cap = (uint32_t)(bytes / 2 / sizeof(PpmdSt));
  m->text_cap = (uint32_t)(bytes / 4);
  m->ctx = arena<PpmdCtx>(m->ctx_cap, fill);
  m->pool = arena<PpmdSt>(m->pool_cap, fill);
  m->text = arena<uint8_t>(m->text_cap, fill);
  ppmd_init(*m);
  int rc = 0;
  for (size_t t = 0; t < n && !rc; ++t) {
    ppmd_update_byte(*m, stream[t]);
    ppmd_prepare_byte(*m);
    if (m->error) { rc = 1; break; }
    float* probs = out + t * 256;
    for (int i = 0; i < 256; ++i) { probs[i] = (float)m->sqp[i]; if (probs[i] < 1) probs[i] = 1; if (!vocab[i]) probs[i] = 0; }
    float sum = probs[0];
    for (int i = 1; i < 256; ++i) sum += probs[i];
    for (int i = 0; i < 256; ++i) probs[i] /= sum;
  }
  free(m->ctx); free(m->pool); free(m->text);
  delete m;
  return rc;
}

}  // extern "C"

#ifdef PPMD_HOST_MAIN
// ppmd_host <stream file> <vocabulary file (256 bytes)>: the same run as a program, for the line-coverage build of
// tools/coverage_report.py. Returns ppmd_host_run's code.
#include <cstdio>
#include <vector>

static std::vector<unsigned char> slurp(const char* path) {
  std::vector<unsigned char> v;
  FILE* f = fopen(path, "rb");
  if (!f) return v;
  fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
  v.resize(n);
  if (n && fread(v.data(), 1, n, f) != (size_t)n) v.clear();
  fclose(f);
  return v;
}

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: ppmd_host <stream> <vocabulary>\n"); return 2; }
  std::vector<unsigned char> stream = slurp(argv[1]), vocab = slurp(argv[2]);
  if (stream.empty() || vocab.size() != 256) { fprintf(stderr, "ppmd_host: bad input\n"); return 2; }
  std::vector<float> out(stream.size() * 256);
  return ppmd_host_run(stream.data(), stream.size(), vocab.data(), out.data(), 64, 0);
}
#endif
