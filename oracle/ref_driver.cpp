// oracle/ref_driver.cpp — TEST INFRASTRUCTURE, not product code.
//
// Driver that links the UNMODIFIED reference translation units (everything in
// the reference's makefile:11 except src/runner.cpp) and exposes what the
// reference itself never exposes: the per-bit output of Predictor::Predict()
// (reference src/predictor.cpp:361) plus the intermediate vectors the CUDA
// engine needs for replay / kernel-level parity.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
// reference legs may execute the binary this builds (oracle/_ref/oracle_dump).
//
// Usage:
//   oracle_dump dump <n|c|t> <input> <out_prefix> <level> [max_bytes] [dictionary]
//   oracle_dump time <n|c|t> <input> <max_bytes> [dictionary|-] [step_bytes]
//       step_bytes > 0: also report the wall time of every step_bytes-sized step (one constructor for a whole
//       warm-up + timed series) and the cross entropy (bits per byte) of the coded prefix
//
//   n = no preprocessing (runner.cpp:187 -> preprocessor::NoPreprocess)
//   c = preprocessing     (runner.cpp:184 -> preprocessor::Encode)
//   t = forced text mode
//
// dump level 0: <prefix>.p.f32 (one float per coded bit), <prefix>.stream
//               (the preprocessed bytes that were coded), <prefix>.meta
// dump level 1: + <prefix>.ext.u16  per bit: 431 FXCM + 1591 PAQ8 12-bit codes
//                                    (0xFFFF = slot still holds its initial 0.5)
//               + <prefix>.ppmd.f32 per byte: the 256-entry PPMD distribution
//                                    valid AFTER that byte (ppmd.cpp:1328-1338)
//               + <prefix>.lstmfx.u32 per bit: lstmpr | lstmex << 16 as FXCM saw them in the
//                                    Perceive() of that bit (predictor.cpp:462-466)
// dump level 2: + <prefix>.in.f32   per bit: 2078 stretched layer-0 inputs
//               + <prefix>.mix.f32  per bit: 47 raw mixer outputs (Mixer::p_)
//               + <prefix>.ctx.u32  per bit: 47 mixer selector contexts (u32)
//               + <prefix>.lstm.f32 per byte: 256-entry byte-mixer distribution
//
// time: re-implements ONLY the orchestration of Predictor::Predict/Perceive
// (predictor.cpp:361-469) in this file, calling the reference's own component
// objects, with wall-clock timers around the PAQ8 / FXCM / PPMD calls so that
// the CPU cost of the rows this repo has on the device (SURVEY §8 a1-a12,
// a16-a18) can be reported separately from rows a13-a15.

#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <memory>
#include <set>
#include <string>
#include <unordered_map>
#include <valarray>
#include <vector>
#include <array>
#include <unistd.h>

// Standard headers are all included above, so the access hack below only
// touches the reference's own class definitions (driver TU only).
#define private public
#define protected public
#include "predictor.h"
#include "models/ppmd.h"
#undef private
#undef protected

#include "preprocess/preprocessor.h"

char* dictionary_path = NULL;  // runner.cpp:17 (read by fxcmv1.cpp:412)
extern int lstmpr, lstmex;     // predictor.cpp:359

namespace {

const unsigned kFxcmModel = 3;   // models_ order: Bracket, Direct, Indirect, FXCM, PAQ8 (predictor.cpp:28-30)
const unsigned kPaq8Model = 4;
const int kMinVocabFileSize = 10000;  // runner.cpp:14

double now_s() {
  using namespace std::chrono;
  return duration<double>(steady_clock::now().time_since_epoch()).count();
}

uint16_t code12(float p) {
  if (p == 0.5f) return 0xFFFF;
  long x = lrintf(p * 4095.0f);
  float back = x * (float)(1.0 / 4095);
  if (x < 0 || x > 4095 || back != p) {
    fprintf(stderr, "oracle_dump: probability %.9g is not k/4095\n", p);
    exit(3);
  }
  return (uint16_t)x;
}

struct Files {
  FILE *p = 0, *ext = 0, *ppmd = 0, *in = 0, *mix = 0, *ctx = 0, *lstm = 0, *lstmfx = 0;
};

FILE* open_out(const std::string& prefix, const char* suffix) {
  FILE* f = fopen((prefix + suffix).c_str(), "wb");
  if (!f) { perror("fopen"); exit(2); }
  return f;
}

unsigned int Discretize12(float p) { return 1 + 4094 * p; }  // predictor.cpp:180

}  // namespace

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: see header of oracle/ref_driver.cpp\n");
    return 1;
  }
  std::string cmd = argv[1];
  char mode = argv[2][0];
  std::string input_path = argv[3];
  std::string prefix;
  int level = 0;
  unsigned long long max_bytes = ~0ULL, step_bytes = 0;
  const char* dict = NULL;
  if (cmd == "dump") {
    if (argc < 6) return 1;
    prefix = argv[4];
    level = atoi(argv[5]);
    if (argc > 6) max_bytes = strtoull(argv[6], 0, 10);
    if (argc > 7) dict = argv[7];
  } else if (cmd == "time") {
    max_bytes = strtoull(argv[4], 0, 10);
    if (argc > 5 && strcmp(argv[5], "-") != 0) dict = argv[5];
    if (argc > 6) step_bytes = strtoull(argv[6], 0, 10);
    prefix = "/tmp/oracle_time_" + std::to_string((long)getpid());
  } else {
    return 1;
  }
  FILE* dictionary = NULL;
  if (dict) {
    dictionary = fopen(dict, "rb");
    if (!dictionary) { perror("dictionary"); return 2; }
    dictionary_path = const_cast<char*>(dict);
  }

  // --- runner.cpp:162-203: preprocess into a temp stream, extract vocab ---
  double t_start = now_s();
  std::string temp_path = prefix + ".stream";
  {
    FILE* data_in = fopen(input_path.c_str(), "rb");
    if (!data_in) { perror("input"); return 2; }
    FILE* temp_out = fopen(temp_path.c_str(), "wb");
    if (!temp_out) { perror("temp"); return 2; }
    fseek(data_in, 0L, SEEK_END);
    unsigned long long n = ftell(data_in);
    fseek(data_in, 0L, SEEK_SET);
    if (mode == 'n') preprocessor::NoPreprocess(data_in, temp_out, n);
    else preprocessor::Encode(data_in, temp_out, mode == 't', n, temp_path + ".tmp", dictionary);
    fclose(data_in);
    fclose(temp_out);
  }
  std::vector<unsigned char> stream;
  {
    std::ifstream f(temp_path, std::ios::binary);
    stream.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
  }
  unsigned long long temp_bytes = stream.size();
  std::vector<bool> vocab(256, false);
  if (temp_bytes < (unsigned long long)kMinVocabFileSize) {
    std::fill(vocab.begin(), vocab.end(), true);
  } else {
    for (unsigned char c : stream) vocab[c] = true;
  }
  unsigned long long n_bytes = std::min<unsigned long long>(temp_bytes, max_bytes);

  Predictor p(vocab);
  double t_ctor = now_s();
  if (mode != 'n') preprocessor::Pretrain(&p, dictionary);
  double t_pretrain = now_s();

  if (cmd == "dump") {
    Files f;
    f.p = open_out(prefix, ".p.f32");
    if (level >= 1) { f.ext = open_out(prefix, ".ext.u16"); f.ppmd = open_out(prefix, ".ppmd.f32"); f.lstmfx = open_out(prefix, ".lstmfx.u32"); }
    if (level >= 2) {
      f.in = open_out(prefix, ".in.f32"); f.mix = open_out(prefix, ".mix.f32");
      f.ctx = open_out(prefix, ".ctx.u32"); f.lstm = open_out(prefix, ".lstm.f32");
    }
    std::vector<uint16_t> ext(431 + 1591);
    std::vector<float> mixv(47);
    std::vector<uint32_t> ctxv(47);
    for (unsigned long long pos = 0; pos < n_bytes; ++pos) {
      unsigned char c = stream[pos];
      for (int j = 7; j >= 0; --j) {
        int bit = (c >> j) & 1;
        if (f.ext) {
          // FXCM::Predict / PAQ8::Predict are pure getters (fxcmv1.cpp:4901, paq8.cpp:8372)
          const std::valarray<float>& fx = p.models_[kFxcmModel]->Predict();
          const std::valarray<float>& pq = p.models_[kPaq8Model]->Predict();
          if (fx.size() != 431 || pq.size() != 1591) { fprintf(stderr, "unexpected sizes\n"); return 3; }
          for (int i = 0; i < 431; ++i) ext[i] = code12(fx[i]);
          for (int i = 0; i < 1591; ++i) ext[431 + i] = code12(pq[i]);
          fwrite(ext.data(), 2, ext.size(), f.ext);
        }
        float pr = p.Predict();
        fwrite(&pr, 4, 1, f.p);
        if (f.in) {
          const std::valarray<float>& in = p.layers_[0]->Inputs();
          fwrite(&in[0], 4, in.size(), f.in);
          int k = 0;
          for (unsigned l = 0; l < 3; ++l)
            for (auto& m : p.mixers_[l]) { mixv[k] = m->p_; ctxv[k] = (uint32_t)m->context_; ++k; }
          fwrite(mixv.data(), 4, 47, f.mix);
          fwrite(ctxv.data(), 4, 47, f.ctx);
        }
        p.Perceive(bit);
        if (f.lstmfx) { uint32_t v = (uint32_t)lstmpr | ((uint32_t)lstmex << 16); fwrite(&v, 4, 1, f.lstmfx); }
      }
      if (f.ppmd) {
        const std::valarray<float>& pp = p.byte_models_[0]->BytePredict();
        fwrite(&pp[0], 4, 256, f.ppmd);
      }
      if (f.lstm) {
        const std::valarray<float>& lp = p.byte_mixers_[0]->BytePredict();
        fwrite(&lp[0], 4, 256, f.lstm);
      }
    }
    double t_end = now_s();
    FILE* meta = open_out(prefix, ".meta");
    fprintf(meta, "n_bytes %llu\nstream_bytes %llu\nlevel %d\nmode %c\ndictionary %d\n", n_bytes, temp_bytes, level, mode, dict ? 1 : 0);
    fprintf(meta, "vocab ");
    for (int i = 0; i < 256; ++i) fputc(vocab[i] ? '1' : '0', meta);
    fprintf(meta, "\nctor_s %.3f\npretrain_s %.3f\ncode_s %.3f\n", t_ctor - t_start, t_pretrain - t_ctor, t_end - t_pretrain);
    fclose(meta);
    for (FILE* x : {f.p, f.ext, f.ppmd, f.in, f.mix, f.ctx, f.lstm, f.lstmfx}) if (x) fclose(x);
    return 0;
  }

  // ---------------------------------------------------------------- time ---
  // Orchestration below mirrors predictor.cpp:361-469 statement for statement;
  // the arithmetic is all inside the reference's own objects.
  double t_big = 0;      // PAQ8 + FXCM + PPMD (SURVEY §8 a13-a15)
  double checksum = 0, entropy_bits = 0;
  std::vector<double> step_s;
  double t0 = now_s(), t_step = t0;
  for (unsigned long long pos = 0; pos < n_bytes; ++pos) {
    if (step_bytes && pos && pos % step_bytes == 0) { double t = now_s(); step_s.push_back(t - t_step); t_step = t; }
    unsigned char c = stream[pos];
    for (int j = 7; j >= 0; --j) {
      int bit = (c >> j) & 1;
      float pr = p.Predict();
      checksum += pr;
      { double q = bit ? pr : 1.0 - pr; if (q < 1.0 / 65536) q = 1.0 / 65536; entropy_bits -= log2(q); }
      // ---- Perceive (predictor.cpp:421-469) with timers ----
      for (unsigned int i = 0; i < p.models_.size(); ++i) {
        if (i == p.fxcm_index_) continue;
        if (i == kPaq8Model) {
          double a = now_s(); p.models_[i]->Perceive(bit); t_big += now_s() - a;
        } else {
          p.models_[i]->Perceive(bit);
        }
      }
      for (const auto& model : p.byte_models_) model->Perceive(bit);
      for (const auto& bm : p.byte_mixers_) bm->Perceive(bit);
      for (unsigned int i = 0; i < p.mixers_.size(); ++i)
        for (const auto& mixer : p.mixers_[i]) mixer->Perceive(bit);
      p.sse_.Perceive(bit);
      bool byte_update = p.manager_.bit_context_ >= 128;
      p.manager_.UpdateContexts(bit);
      if (byte_update) {
        for (const auto& model : p.models_) model->ByteUpdate();
        {
          double a = now_s();
          for (const auto& model : p.byte_models_) model->ByteUpdate();
          t_big += now_s() - a;
        }
        for (unsigned int i = 0; i < p.byte_models_.size(); ++i) {
          const std::valarray<float>& pp = p.byte_models_[i]->BytePredict();
          for (const auto& bm : p.byte_mixers_)
            for (unsigned int k = 0; k < 256; ++k) bm->SetInput(k, pp[k]);
        }
        for (const auto& bm : p.byte_mixers_) bm->ByteUpdate();
      }
      for (const auto& bm : p.byte_mixers_) {
        float out = bm->Predict()[0];
        lstmpr = Discretize12(out);
        lstmex = bm->ex;
        double a = now_s(); p.models_[p.fxcm_index_]->Perceive(bit); t_big += now_s() - a;
      }
      if (byte_update) p.manager_.bit_context_ = 1;
    }
  }
  double t1 = now_s();
  if (step_bytes && n_bytes && n_bytes % step_bytes == 0) step_s.push_back(t1 - t_step);
  remove(temp_path.c_str());
  printf("{\"bytes\": %llu, \"ctor_s\": %.4f, \"pretrain_s\": %.4f, \"code_s\": %.6f, "
         "\"big_models_s\": %.6f, \"checksum\": %.9f, \"bpc\": %.6f, \"step_bytes\": %llu, \"step_s\": [",
         n_bytes, t_ctor - t_start, t_pretrain - t_ctor, t1 - t0, t_big, checksum, n_bytes ? entropy_bits / n_bytes : 0.0, step_bytes);
  for (size_t i = 0; i < step_s.size(); ++i) printf("%s%.6f", i ? ", " : "", step_s[i]);
  printf("]}\n");
  return 0;
}
