// cmix_b200/csrc/engine.cu — host side of the H100 predictor engine + the C-ABI
// declared in include/cmixb200.h.
//
// Host responsibilities (everything numeric runs in the kernels):
//  * build the read-only tables the reference builds with libm at start-up
//    (logit LUT sigmoid.cpp:5-10, SSE stretch/squash sse.cpp:112-135, Adam bias
//    corrections lstm-layer.cpp:17-30, per-bit decay mixer.cpp:58) with the same
//    glibc the oracle uses, and upload them;
//  * draw the initial LSTM weights / Indirect offsets from glibc's rand() stream
//    seeded with 0xDEADBEEF in the reference's construction order
//    (predictor.cpp:26-36, SURVEY §3.5);
//  * allocate the ~7 GB of per-stream HBM state and launch the bulk kernels
//    (ppmd -> small | lstm -> mix [-> encode]) on separate CUDA streams, in launch
//    groups of 8 streams, or their lock-step halves for Predict()/Perceive().
// There is NO CPU fallback: every entry point fails with CMIXB200_ERR_CUDA if
// the device or a kernel is unavailable.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/cmixb200.h"
#include "exact_math.h"
#include "coder.cuh"
#include "fxcm_model.h"
#include "fxcm_host.h"
#include "paq8_top.h"
#include "paq8_host.h"
#include "producers.h"
#include "lstm.cuh"
#include "mixer_lock.cuh"
#include "mixer_bulk.cuh"
#include "ppmd.cuh"
#include "small_models.cuh"
#include "state.h"

using namespace cmixb200;

namespace {

thread_local std::string g_last_error;

#define CK(call)                                                                         \
  do {                                                                                   \
    cudaError_t e_ = (call);                                                             \
    if (e_ != cudaSuccess) {                                                             \
      char buf_[512];                                                                    \
      snprintf(buf_, sizeof buf_, "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
      g_last_error = buf_;                                                               \
      return CMIXB200_ERR_CUDA;                                                          \
    }                                                                                    \
  } while (0)

// states/nonstationary.cpp:3 — 256x2 next-state table as hex, [state][bit].
const char kNonstatHex[] =
    "020c90050705190e3605101d1a8ca9051018540410250a620ad42d25c9001cca"
    "2017b78806d9bc2608251545083d380d16251b42558c23296bc7085b66d96411"
    "68175e05602f2bb02e3016276b331833fbf8190136223594463a5617163d4617"
    "243f3d3f07053e415ad84369442296056049462f484a494b2e3f4a311459244f"
    "148a3e51aa0e5245542215e960480ad42c3b2c3b3a4c3a4c4b3d3c3116274d59"
    "13413e5b5ad996b95e225c7f6017a7cf92934d635d660b65616967f968221341"
    "6a397a7b1627306d00cb0b6f03536c70722219f57422132771e63077a6bc3e79"
    "8c60751b7c04c2e72a228d7fa4b33f81ebcc6b837d7f6ed98604848512f5c90e"
    "3eaf308b80b70b97891e23cc87049004af958ed93eb73033c901bdab91855fb2"
    "962198995fc3a7b3234240ac9a096b9b9c9d1bef9e09269fa0a143c2a221508f"
    "a3b9c9f9a609a53400e7a88c6ebc64cfadb0b121aebc150097c0b5451b9afc8a"
    "4221bd09e48f1f28be5ab8b9bc793fbbba948d34c15380bf72b6cddcc53480c3"
    "92d4c43464d782c7c685ecefcee9fccb64cb034292fe5bcfb9c2e501d1e65fd3"
    "6411d6d8641182d740e1c9ccdaef92dba6e6f901deccc8df8601a7d7e2ae83e3"
    "ddf740ede84557e71341eedc230cc811b4ad43d91c65c5d5f0f1fcfdf2dc6ca4"
    "f3f4c9a4f62978d5c9349a017e377376737619d826c3a7d7148a400f1c580e11";

// predictor.cpp:201-356: selector and learning rate of each of the 47 mixers.
const int kSel[N_MIXERS] = {
    S_BC0, S_BC0, S_BC1, S_BC1, S_BC2, S_BC3, S_RB2, S_RB3, S_ZERO, S_LINEBREAK, S_LONGEST, S_WRT, S_AUX,
    S_IV0, S_IV1, S_IV2, S_BC_ALNUM, S_IV3, S_IV4, S_BC_W2, S_IV6, S_IVH, S_BC_W3, S_BC_RB1, S_COMB0, S_COMB1,
    S_ZERO, S_ZERO, S_LONGBIT, S_LONGBIT, S_LONGBIT, S_RB0, S_RB1, S_RB2, S_LONGEST, S_WRT,
    S_IV0, S_IV1, S_IV2, S_IV3, S_IV4, S_IV6, S_IVH, S_BC_W2, S_BC_ALNUM, S_BC_W3,
    S_ZERO};
const double kLr[N_MIXERS] = {
    0.005, 0.0005, 0.005, 0.0005, 0.005, 0.002, 0.002, 0.005, 0.00005, 0.0007, 0.0005, 0.002, 0.0005,
    0.001, 0.001, 0.001, 0.005, 0.001, 0.001, 0.005, 0.001, 0.001, 0.005, 0.005, 0.005, 0.003,
    0.005, 0.0005, 0.005, 0.0005, 0.00001, 0.005, 0.005, 0.005, 0.0005, 0.002,
    0.001, 0.001, 0.001, 0.001, 0.001, 0.001, 0.001, 0.001, 0.001, 0.001,
    0.0003};
// number of distinct values each selector can take (bounds the row table)
u32 SelRange(int s) {
  switch (s) {
    case S_ZERO: return 1;
    case S_LONGBIT: case S_RB0: case S_RB1: case S_RB2: case S_RB3: return 256;
    case S_LINEBREAK: return 100;
    case S_LONGEST: return 8;
    case S_WRT: return 0xFFEFCF + 1;
    case S_AUX: return 16;
    case S_IV0: case S_IV1: return 256;
    case S_IV2: return 128;
    case S_IV3: return 1024;
    case S_IV4: return 32768;
    case S_IV6: return 512;
    case S_IVH: return 16384;
    case S_BC0: return 256;
    case S_BC1: case S_BC2: return 65536;
    case S_BC3: return 16384;
    case S_BC_ALNUM: case S_BC_W2: case S_BC_W3: return 32768;
    case S_BC_RB1: case S_COMB0: case S_COMB1: return 65536;
  }
  return 1;
}

int IntervalMap(int which, int c) {   // predictor.cpp:223-304
  static const int t1[] = {1, 32, 64, 128, 255, 142, 138, 140, 137, 97};
  static const int t2[] = {41, 92, 124, 58, 11, 46, 36, 47, 64, 4, 61, 97, 125, 45, 48};
  static const char m4[] = "2313301233001333" "3333333333303333" "3202132133332302"
                           "1111111111322322" "2200231212222200" "2222222230232023";
  static const char m6[] = "0020560602043000" "0000000000000000" "2414474737223531"
                           "1111111111053355" "0557501545006071" "3374557022544746";
  int v = 0;
  switch (which) {
    case 0: for (int t : t1) v += c < t; return v;
    case 1: for (int t : t2) v += c < t; return v;
    case 2: return ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c >= 0x80) ? 1 : 0;
    case 3: return c < 96 ? m4[c] - '0' : (c < 208 ? 1 : 0);
    default: return c < 96 ? m6[c] - '0' : (c < 128 ? 5 : (c < 208 ? 6 : 7));
  }
}

struct GlibcRand {   // the rand() stream of one Predictor (TYPE_3 additive feedback, as rand())
  char statebuf[128];
  struct random_data rd;
  explicit GlibcRand(unsigned seed) {
    memset(&rd, 0, sizeof rd); memset(statebuf, 0, sizeof statebuf);
    initstate_r(seed, statebuf, sizeof statebuf, &rd);
  }
  int next() { int32_t r; random_r(&rd, &r); return r; }
};

__global__ void fill_f32(float* p, size_t n, float v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void fill_u32(u32* p, size_t n, u32 v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void fill_sse_rows(u16* p, size_t vol, int Wi) {   // SSEi<7>::Init (sse.cpp:25-31), 8-u16 pitch
  const int SCw = (32768 - Wi) / 6, INC = Wi / 2 + 8192;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < vol * 8; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i & 7);
    p[i] = k < 7 ? (u16)(INC + k * SCw) : 0;
  }
}

struct SharedTables {   // one per device: the tables are device memory and constant memory of THAT device
  bool ready = false;
  float* d_logit = nullptr; float* d_lut12 = nullptr; u16* d_st = nullptr; u16* d_sq = nullptr; float* d_adam = nullptr;
  Tables T;
};
std::map<int, SharedTables> g_tables_by_device;
std::mutex g_tables_mutex;

int BuildSharedTablesLocked(int device, SharedTables& g_tables);
// Returns the table set of `device` (built on first use); the caller keeps a copy of .T in its predictor.
int BuildSharedTables(int device, SharedTables** out) {
  std::lock_guard<std::mutex> lock(g_tables_mutex);
  SharedTables& t = g_tables_by_device[device];
  int r = t.ready ? CMIXB200_OK : BuildSharedTablesLocked(device, t);
  if (r == CMIXB200_OK) *out = &t;
  return r;
}

int BuildSharedTablesLocked(int device, SharedTables& g_tables) {
  (void)device;
  std::vector<float> logit(100001);
  for (int i = 0; i < 100001; ++i) {
    float p = (i + 0.5f) / 100001;
    logit[i] = logf(p / (1 - p));
  }
  auto Logit = [&](float p) { int idx = p * 100001; if (idx >= 100001) idx = 100000; else if (idx < 0) idx = 0; return logit[idx]; };
  std::vector<float> lut12(4097);
  const float cf = 1.0 / 4095;
  for (int c = 0; c <= 4096; ++c) {
    float p = c == 4096 ? 0.5f : c * cf;
    if (p < 1.0e-4f) p = 1.0e-4f; else if (p > 1 - 1.0e-4f) p = 1 - 1.0e-4f;
    lut12[c] = Logit(p);
  }
  // SSE stretch/squash (sse.cpp:78-135), double libm as the reference
  std::vector<u16> st(32768, 0), sq(32768, 0);
  {
    const double log2e = 1.44269504088896340736;
    const double st_coef = (16384 - 1) / (log2e * log((double)(32768 - 1)));
    const double sq_coef = 1.0 / st_coef;
    for (unsigned i = 1; i < 32768; ++i) {
      double a = double(int(i) - 16384) * sq_coef;
      unsigned p = (1.0 / (1.0 + exp(a / log2e))) * 32768;
      sq[i] = (u16)p;
    }
    unsigned x = 0;
    for (unsigned i = 1; i < 32768; ++i) {
      double pr = double(i) / 32768;
      unsigned s = (log2e * log((1 - pr) / pr)) * st_coef + 16384;
      st[i] = (u16)s;
      if (s != st[x]) { unsigned y = i - 1; sq[st[x]] = (u16)((x + y + 1) / 2); x = i; }
    }
  }
  // Adam step scalars (lstm-layer.cpp:11-32) for update_steps_ = 0..3000
  std::vector<float> adam(3001 * 4, 0.0f);
  {
    const float beta1 = 0.025, beta2 = 0.9999;
    const float learning_rate = 0.03;
    const unsigned long long update_limit = 3000;
    for (int ti = 0; ti <= 3000; ++ti) {
      float t = ti;
      float alpha, bc1, bc2;
      if (t < update_limit) {
        alpha = learning_rate * 0.1f / sqrt(5e-5f * t + 1.0f);
        bc1 = (float)(1.0f - pow(beta1, t));
        bc2 = (float)(1.0f - pow(beta2, t));
      } else {
        alpha = learning_rate * 0.1f / sqrt(5e-5f * update_limit + 1.0f);
        bc1 = (float)(1.0f - pow(beta1, update_limit));
        bc2 = (float)(1.0f - pow(beta2, update_limit));
      }
      adam[ti * 4] = alpha; adam[ti * 4 + 1] = bc1; adam[ti * 4 + 2] = bc2;
    }
  }
  CK(cudaMalloc(&g_tables.d_logit, logit.size() * 4));
  CK(cudaMemcpy(g_tables.d_logit, logit.data(), logit.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&g_tables.d_lut12, lut12.size() * 4));
  CK(cudaMemcpy(g_tables.d_lut12, lut12.data(), lut12.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&g_tables.d_st, st.size() * 2));
  CK(cudaMemcpy(g_tables.d_st, st.data(), st.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&g_tables.d_sq, sq.size() * 2));
  CK(cudaMemcpy(g_tables.d_sq, sq.data(), sq.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&g_tables.d_adam, adam.size() * 4));
  CK(cudaMemcpy(g_tables.d_adam, adam.data(), adam.size() * 4, cudaMemcpyHostToDevice));
  g_tables.T.logit = g_tables.d_logit;
  g_tables.T.lut12 = g_tables.d_lut12;
  g_tables.T.stretch_min = Logit(0);
  g_tables.T.stretch_max = Logit(1);
  // constant-memory tables
  u8 nonstat[512], runmap[512], ivmap[5][256], msel[N_MIXERS];
  auto hv = [](char c) { return c <= '9' ? c - '0' : c - 'a' + 10; };
  for (int i = 0; i < 512; ++i) nonstat[i] = (u8)(hv(kNonstatHex[2 * i]) * 16 + hv(kNonstatHex[2 * i + 1]));
  for (int i = 0; i < 512; ++i) {   // run-map.cpp:3-20
    int state = i / 2;
    if (i % 2 == 0) { if (state < 127) ++state; else if (state >= 128) state = 0; }
    else { if (state < 128) state = 128; else if (state < 255) ++state; }
    runmap[i] = (u8)state;
  }
  for (int m = 0; m < 5; ++m) for (int c = 0; c < 256; ++c) ivmap[m][c] = (u8)IntervalMap(m, c);
  for (int i = 0; i < N_MIXERS; ++i) msel[i] = (u8)kSel[i];
  CK(cudaMemcpyToSymbol(c_nonstat, nonstat, sizeof nonstat));
  CK(cudaMemcpyToSymbol(c_runmap, runmap, sizeof runmap));
  CK(cudaMemcpyToSymbol(c_ivmap, ivmap, sizeof ivmap));
  CK(cudaMemcpyToSymbol(c_mixer_sel, msel, sizeof msel));
  CK(cudaFuncSetAttribute(small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmallState)));
  CK(cudaFuncSetAttribute(mix_kernel_v3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MixBulkShared)));
  CK(cudaFuncSetAttribute(lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(LstmShared)));
  CK(cudaFuncSetAttribute(ppmd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(PPMD_WARPS * sizeof(PpmdWarpShared))));
  CK(cudaFuncSetAttribute(lstm_byte_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(LstmShared)));
  CK(fxcm_configure());
  CK(paq8_configure());
  g_tables.ready = true;
  return CMIXB200_OK;
}

// A device buffer that one predictor owns. Grow() replaces it by one of at least `count` elements (the contents are not kept)
// and leaves it empty if the allocation fails; the buffer is freed when the predictor is deleted.
template <class T> struct DeviceBuf {
  T* p = nullptr;
  size_t n = 0;                        // capacity in elements
  DeviceBuf() = default;
  DeviceBuf(const DeviceBuf&) = delete;
  DeviceBuf& operator=(const DeviceBuf&) = delete;
  ~DeviceBuf() { if (p) cudaFree(p); }
  cudaError_t Grow(size_t count) {
    if (count <= n) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; n = 0;
    T* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, count * sizeof(T));
    if (e == cudaSuccess) { p = q; n = count; }
    return e;
  }
};

}  // namespace

struct cmixb200_predictor {
  int device = 0;
  StreamState* d_st = nullptr;
  StreamState h;                       // host mirror of the pointer/parameter fields
  std::vector<void*> allocs;           // the models' state, allocated once by BuildStream
  cudaStream_t s_small = nullptr, s_lstm = nullptr, s_mix = nullptr;
  DeviceBuf<ChunkArgs> d_args;
  // chunk scratch
  DeviceBuf<float> d_small_x; DeviceBuf<u32> d_sel; DeviceBuf<float> d_lstm_x, d_decay, d_p;
  DeviceBuf<u8> d_bytes; DeviceBuf<u16> d_ext; DeviceBuf<float> d_ppmd;   // host staging of code_bytes
  // double-buffered host staging of the batch entry point
  DeviceBuf<u8> d_bytes2[2]; DeviceBuf<u16> d_ext2[2]; DeviceBuf<float> d_ppmd2[2];
  cudaStream_t s_copy = nullptr;
  cudaStream_t s_ppmd = nullptr; DeviceBuf<float> d_ppmd_gen;   // resident PPMD: own stream, scratch [n_bytes][256]
  PpmdModel* d_ppmd_model = nullptr;
  // order the library streams per bit, in lock-step calls and in the decoder's graphs
  cudaEvent_t ev_lock_mix = nullptr, ev_lock_small = nullptr, ev_lock_p8 = nullptr;
  DeviceBuf<DecodeState> d_dec;                      // device decoder (cmixb200_decode_bytes)
  cudaGraphExec_t dec_graph[3] = {nullptr, nullptr, nullptr};  // a bit inside a byte / the bit that completes a byte / the last bit of a call
  unsigned long long dec_launches[3] = {0, 0, 0};              // kernels in each graph
  // device arithmetic coder (compress direction)
  DeviceBuf<CoderState> d_coder; DeviceBuf<u8> d_code; bool coder_on = false;
  // lock-step state
  u64 bits_done = 0;                   // coded bits so far (Mixer::steps_)
  u32 bit_context = 1;                 // partial byte incl. leading 1 (ContextManager::bit_context_)
  DeviceBuf<u16> d_ext_bit; bool ext_bit_valid = false;
  DeviceBuf<float> d_ppmd_byte; bool ppmd_byte_valid = false;
  unsigned long long launches = 0;
  DeviceBuf<unsigned long long> d_prof;
  bool time_mix = false;               // CUDA-event timing of the bulk kernels (cmixb200_time_mix_kernel)
  struct KEv { int which; cudaEvent_t a, b; };
  std::vector<KEv> pending_kev; double kernel_ms[6] = {0, 0, 0, 0, 0, 0}; unsigned long long kernel_n[6] = {0, 0, 0, 0, 0, 0};
  u8 vocab[256];
  int V = 0;
  Tables T;                            // this device's shared read-only tables (copied at create: no global is read at launch)
  SharedTables* shared = nullptr;
  // resident FXCM (fxcm.cuh): device state, its text block and tables; `replay_mask` = CMIXB200_REPLAY_* flags of create_ex
  unsigned replay_mask = 0;
  std::string dict_path;
  fx::State* d_fx = nullptr; fx::TextState* d_fx_text = nullptr; fx::Tables* d_fx_tables = nullptr;
  cudaStream_t s_fx = nullptr;
  p8::State* d_p8 = nullptr; p8::Tables* d_p8_tables = nullptr; cudaStream_t s_p8 = nullptr;   // resident PAQ8 (paq8.cuh)
  DeviceBuf<u16> d_ext_gen; DeviceBuf<u32> d_lstm_fx;
  cudaEvent_t ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // reusable ordering events (LaunchChunk)

  template <class T> int Alloc(T** p, size_t n, bool zero = true) {
    void* q = nullptr;
    CK(cudaMalloc(&q, n * sizeof(T)));
    if (zero) CK(cudaMemset(q, 0, n * sizeof(T)));
    allocs.push_back(q);
    *p = (T*)q;
    return CMIXB200_OK;
  }
};

namespace {

#define TRY(x) do { int r_ = (x); if (r_ != CMIXB200_OK) return r_; } while (0)

int InitDirect(cmixb200_predictor* P, DirectTable& d, int limit, float delta, u64 rows, bool hashed) {
  d.limit = limit; d.delta = delta; d.divisor = 1.0 / (limit + delta); d.rows = rows; d.hashed = hashed; d.index = 0;
  TRY(P->Alloc(&d.pred, rows * 256, false));
  fill_f32<<<1024, 256>>>(d.pred, rows * 256, 0.5f);
  TRY(P->Alloc(&d.count, rows * 256));
  d.checksum = nullptr;
  if (hashed) TRY(P->Alloc(&d.checksum, rows));
  return CMIXB200_OK;
}

__global__ void fill_u16(u16* p, size_t n, u16 v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
// Memory backend of fx::build_state (fxcm_host.h): zeroed cudaMalloc, fill kernels, blocking uploads.
struct DeviceBackend {
  cmixb200_predictor* P; bool ok = true;
  void* alloc(size_t bytes) { u8* q = nullptr; if (P->Alloc(&q, bytes ? bytes : 1) != CMIXB200_OK) { ok = false; return nullptr; } return q; }
  void fill16(void* p, size_t n, u16 v) { fill_u16<<<1024, 256>>>((u16*)p, n, v); }
  void fill32(void* p, size_t n, u32 v) { fill_u32<<<1024, 256>>>((u32*)p, n, v); }
  void upload(void* d, const void* s, size_t bytes) { if (cudaMemcpy(d, s, bytes, cudaMemcpyHostToDevice) != cudaSuccess) ok = false; }
};

// The resident FXCM model (SURVEY §8 a14): tables built on the host with the oracle's glibc, ~4.6 GB of bucket tables,
// mixer weights and APMs in HBM, the WRT dictionary (runner.cpp:17's dictionary_path side channel) as flat text.
int BuildFxcm(cmixb200_predictor* P) {
  fx::Tables* T = new fx::Tables();
  fx::build_tables(*T);
  fx::HostDict D;
  D.load(P->dict_path.empty() ? nullptr : P->dict_path.c_str());
  if (!P->dict_path.empty() && !D.loaded) { delete T; g_last_error = "cannot read dictionary " + P->dict_path; return CMIXB200_ERR_ARG; }
  if (D.loaded) {
    char* d_chars = nullptr; u32* d_off = nullptr;
    TRY(P->Alloc(&d_chars, D.chars.size() + 1, false));
    TRY(P->Alloc(&d_off, D.off.size() + 1, false));
    CK(cudaMemcpy(d_chars, D.chars.data(), D.chars.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_off, D.off.data(), D.off.size() * 4, cudaMemcpyHostToDevice));
    T->dict_chars = d_chars; T->dict_off = d_off; T->dict_n = (int)D.off.size(); T->dict_loaded = 1;
  }
  TRY(P->Alloc(&P->d_fx_tables, 1, false));
  {
    fx::Tables* up = new fx::Tables(*T);               // the device copy's table pointers address the device copy
    up->map = reinterpret_cast<const fx::MapTab*>(reinterpret_cast<const u8*>(P->d_fx_tables) + offsetof(fx::Tables, map_store));
    up->st2 = reinterpret_cast<const short (*)[4096]>(reinterpret_cast<const u8*>(P->d_fx_tables) + offsetof(fx::Tables, st2_store));
    const cudaError_t ce = cudaMemcpy(P->d_fx_tables, up, sizeof *up, cudaMemcpyHostToDevice);
    delete up;
    CK(ce);
  }
  fx::State* S = new fx::State();
  fx::TextState* X = new fx::TextState();
  DeviceBackend be{P};
  const bool built = fx::build_state(be, *T, *S, *X) && be.ok;
  int r = CMIXB200_OK;
  if (!built) { if (g_last_error.empty()) g_last_error = "FXCM state allocation failed"; r = CMIXB200_ERR_CUDA; }
  if (r == CMIXB200_OK) r = P->Alloc(&P->d_fx, 1, false);
  if (r == CMIXB200_OK) r = P->Alloc(&P->d_fx_text, 1, false);
  if (r == CMIXB200_OK) {
    S->text = P->d_fx_text; S->T = P->d_fx_tables;
    if (cudaMemcpy(P->d_fx, S, sizeof *S, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(P->d_fx_text, X, sizeof *X, cudaMemcpyHostToDevice) != cudaSuccess) { g_last_error = "FXCM state upload failed"; r = CMIXB200_ERR_CUDA; }
  }
  delete S; delete X; delete T;
  return r;
}

// The resident PAQ8 model (SURVEY §8 a13): ~10 GB of bucket tables, DMC nodes, mixer weight sets and the 1 GiB byte ring.
int BuildPaq8(cmixb200_predictor* P) {
  p8::Tables* T = new p8::Tables();
  p8::build_tables(*T);
  int r = P->Alloc(&P->d_p8_tables, 1, false);
  if (r == CMIXB200_OK) {
    p8::Tables* up = new p8::Tables(*T);               // the device copy's ilog pointer addresses the device copy
    up->ilog = reinterpret_cast<const u8*>(P->d_p8_tables) + offsetof(p8::Tables, ilog_store);
    if (cudaMemcpy(P->d_p8_tables, up, sizeof *up, cudaMemcpyHostToDevice) != cudaSuccess) { g_last_error = "PAQ8 table upload failed"; r = CMIXB200_ERR_CUDA; }
    delete up;
  }
  p8::State* S = new p8::State();
  if (r == CMIXB200_OK) {
    DeviceBackend be{P};
    if (!(p8::build_state(be, *T, *S) && be.ok)) { if (g_last_error.empty()) g_last_error = "PAQ8 state allocation failed"; r = CMIXB200_ERR_CUDA; }
  }
  if (r == CMIXB200_OK) r = P->Alloc(&P->d_p8, 1, false);
  if (r == CMIXB200_OK) {
    S->T = P->d_p8_tables;
    if (cudaMemcpy(P->d_p8, S, sizeof *S, cudaMemcpyHostToDevice) != cudaSuccess) { g_last_error = "PAQ8 state upload failed"; r = CMIXB200_ERR_CUDA; }
  }
  delete S; delete T;
  return r;
}

int BuildStream(cmixb200_predictor* P) {
  StreamState& h = P->h;
  memset(&h, 0, sizeof h);
  GlibcRand rng(0xDEADBEEF);
  // ---------------- mixers ----------------
  for (int i = 0; i < N_MIXERS; ++i) {
    MixerState& m = h.mixer[i];
    m.sel = kSel[i];
    m.lr = (float)kLr[i];
    if (i < N_L0) { m.n_in = N_INPUTS; m.n_extra = i; m.pitch = ROW_PITCH_L0; }
    else if (i < N_L0 + N_L1) { m.n_in = L1_IN; m.n_extra = i - N_L0; m.pitch = ROW_PITCH_L1; }
    else { m.n_in = L2_IN; m.n_extra = 0; m.pitch = ROW_PITCH_L2; }
    m.table_size = SelRange(m.sel);
    const u32 cap = m.table_size < (u32)SLOT_LIMIT ? m.table_size : (u32)SLOT_LIMIT;
    m.n_rows = cap + 1;
    m.n_assigned = 0;
    m.max_steps = 1;
    TRY(P->Alloc(&m.slot_table, m.table_size));
    TRY(P->Alloc(&m.rows, (size_t)m.n_rows * m.pitch));
    TRY(P->Alloc(&m.row_steps, m.n_rows));
  }
  // ---------------- SSE ----------------
  {
    SseState& S = h.sse;
    const size_t kMix1Vol = 4ull * 256 * 8 * 79, kMix2Vol = 3ull * 2 * 256 * 256,
                 kSm6Vol = 3ull * 128 * 256 * 256, kSm7Vol = 3ull * 32 * 256 * 255;
    TRY(P->Alloc(&S.s6, kSm6Vol * 8, false));
    TRY(P->Alloc(&S.s7, kSm7Vol * 8, false));
    fill_sse_rows<<<2048, 256>>>(S.s6, kSm6Vol, 0);
    fill_sse_rows<<<2048, 256>>>(S.s7, kSm7Vol, 8192);
    TRY(P->Alloc(&S.x1, kMix1Vol, false));
    TRY(P->Alloc(&S.x2, kMix2Vol, false));
    fill_u32<<<512, 256>>>((u32*)S.x1, kMix1Vol, 7649 + 16384);
    fill_u32<<<512, 256>>>((u32*)S.x2, kMix2Vol, 2561 + 16384);
    S.st = P->shared->d_st; S.sq = P->shared->d_sq;
    S.j = 1; S.pc = 0; S.ffl = 0;
  }
  // ---------------- small models + contexts (construction order == rand() order) ----------------
  {
    SmallState& s = h.small;
    memcpy(s.vocab, P->vocab, 256);
    s.bit_context = 1; s.long_bit_context = 1;
    TRY(P->Alloc(&s.history, 100000000ull));
    TRY(P->Alloc(&s.shared_map, 256ull * 8000000ull));
    s.br_cap = 1u << 22;
    TRY(P->Alloc(&s.br_char, s.br_cap));
    TRY(P->Alloc(&s.br_dist, s.br_cap));
    static const int ih[11][4] = {{1, 8, 1, 8}, {2, 8, 1, 8}, {1, 8, 2, 8}, {2, 8, 2, 8}, {1, 8, 3, 8}, {3, 8, 1, 8},
                                  {4, 6, 4, 8}, {5, 5, 5, 5}, {1, 8, 4, 8}, {1, 8, 5, 6}, {6, 4, 6, 4}};
    for (int i = 0; i < 11; ++i) {
      IHashState& x = s.ihash[i];
      x.h1 = ih[i][1]; x.h2 = ih[i][3];
      x.size1 = (u32)(1ull << (ih[i][1] * ih[i][0]));
      x.size = 1ull << (ih[i][3] * ih[i][2]);
      TRY(P->Alloc(&x.hashes, x.size1));
    }
    // Bracket (model 0)
    for (int i = 0; i < 256; ++i) s.bracket_bm.probs[i] = 1.0 / 256;
    s.bracket_bm.top = 255;
    TRY(P->Alloc(&s.bk_first, 256 * 200, false));
    TRY(P->Alloc(&s.bk_second, 256 * 200, false));
    fill_u32<<<64, 256>>>(s.bk_first, 256 * 200, 1);
    fill_u32<<<64, 256>>>(s.bk_second, 256 * 200, 256);
    TRY(InitDirect(P, s.direct_bracket, 30, 0, 257 * 256, false));
    auto init_ind = [&](IndirectState& m, bool run, float delta) {
      m.run = run; m.divisor = 1.0 / delta; m.map_index = 0;
      m.map_offset = (u64)rng.next() % (2048000000ull - 257);     // indirect.cpp:10
      for (int i = 0; i < 256; ++i) m.pred[i] = !run ? 0.5f : (float)(i < 128 ? (128.0 - i) / 256 : i / 256.0);
    };
    auto init_match = [&](MatchState& m, int limit, float delta, u64 map_size) -> int {
      m.limit = limit; m.delta = delta; m.divisor = 1.0 / (limit + delta);
      m.map_size = map_size; m.bit_pos = 128;
      TRY(P->Alloc(&m.map, map_size));
      for (int i = 0; i < 256; ++i) { m.pred[i] = 0.5 + (i + 0.5) / 512; m.count[i] = 0; }
      return CMIXB200_OK;
    };
    init_ind(s.indirect[0], false, 300);
    for (int i = 0; i < 18; ++i) init_ind(s.indirect[1 + i], false, 200);
    for (int i = 0; i < 6; ++i) {
      TRY(init_match(s.match[i], 200, 0.5, 10000000));
      if (i == 1) { init_ind(s.indirect[19], true, 200); TRY(InitDirect(P, s.dhash_word, 30, 0, 500000, true)); }
    }
    TRY(InitDirect(P, s.direct_o[0], 30, 0, 1, false));
    TRY(InitDirect(P, s.direct_o[1], 30, 0, 256, false));
    TRY(InitDirect(P, s.direct_o[2], 30, 0, 65536, false));
    TRY(InitDirect(P, s.dhash_o3, 30, 0, 100000, true));
    static const u64 msize[10] = {1, 256, 65536, 20000000, 20000000, 20000000, 20000000, 20000000, 1048576, 20000000};
    for (int i = 0; i < 10; ++i) TRY(init_match(s.match[6 + i], 200, 0.5, msize[i]));
    for (int i = 0; i < 11; ++i) init_ind(s.indirect[20 + i], false, 400);
    for (int i = 0; i < 256; ++i) s.ppmd_bm.probs[i] = 1.0 / 256;
    s.ppmd_bm.top = 255;
  }
  // ---------------- LSTM (lstm.cpp:6-32, lstm-layer.cpp:34-60) ----------------
  {
    LstmState& L = h.lstm;
    const int V = P->V, C = LSTM_CELLS, H = LSTM_HORIZON;
    L.V = V; L.epoch = 0;
    memcpy(L.vocab, P->vocab, 256);
    { int k = 0; for (int i = 0; i < 256; ++i) { L.byte_map[i] = k; if (P->vocab[i]) ++k; } }
    for (int i = 0; i < 256; ++i) L.bm.probs[i] = 1.0 / 256;
    L.bm.top = 255;
    L.hidden[2 * C] = 1;
    L.adam = P->shared->d_adam;
    TRY(P->Alloc(&L.out_w, (size_t)H * V * LSTM_HID));
    TRY(P->Alloc(&L.output, (size_t)H * V, false));
    fill_f32<<<64, 256>>>(L.output, (size_t)H * V, (float)(1.0 / V));
    for (int l = 0; l < 2; ++l) {
      LayerState& Y = L.layer[l];
      Y.in_size = l == 0 ? V + C + 1 : V + 2 * C + 1;
      Y.epoch = 0; Y.update_steps = 0;
      const int row = Y.in_size + V;
      TRY(P->Alloc(&Y.tanh_state, H * C)); TRY(P->Alloc(&Y.input_gate_state, H * C)); TRY(P->Alloc(&Y.last_state, H * C));
      std::vector<float> inp((size_t)H * Y.in_size, 0.0f);
      for (int e = 0; e < H; ++e) inp[(size_t)e * Y.in_size + Y.in_size - 1] = 1;
      TRY(P->Alloc(&Y.input, inp.size(), false));
      CK(cudaMemcpy(Y.input, inp.data(), inp.size() * 4, cudaMemcpyHostToDevice));
      const size_t wsize = (size_t)lstm_rowp(V, Y.in_size) * C;
      std::vector<float> w[3];
      for (int g = 0; g < 3; ++g) w[g].assign(wsize, 0.0f);
      const float val = sqrt(6.0f / float(V + V));
      const float low = -val, range = 2 * val;
      auto rnd = [&]() { return static_cast<float>(rng.next()) / static_cast<float>(RAND_MAX); };
      for (int i = 0; i < C; ++i) {
        for (int j = 0; j < row; ++j) {
          w[0][lstm_widx(V, Y.in_size, j, i)] = low + rnd() * range;
          w[1][lstm_widx(V, Y.in_size, j, i)] = low + rnd() * range;
          w[2][lstm_widx(V, Y.in_size, j, i)] = low + rnd() * range;
        }
        w[0][lstm_widx(V, Y.in_size, row - 1, i)] = 1;
      }
      for (int g = 0; g < 3; ++g) {
        GateState& G = Y.gate[g];
        G.row = row;
        TRY(P->Alloc(&G.w, wsize, false));
        CK(cudaMemcpy(G.w, w[g].data(), w[g].size() * 4, cudaMemcpyHostToDevice));
        TRY(P->Alloc(&G.m, wsize)); TRY(P->Alloc(&G.v, wsize));
        TRY(P->Alloc(&G.state, H * C)); TRY(P->Alloc(&G.norm, H * C)); TRY(P->Alloc(&G.err, H * C));
        for (int i = 0; i < C; ++i) G.gamma[i] = 1.0f;
      }
    }
  }
  h.lstm_override = -1.0f;
  h.last_p = 0.5f;
  TRY(P->Alloc(&P->d_st, 1));
  // ---------------- PPMD (ppmd_model.h): model registers + three flat arenas ----------------
  {
    // The reference gives its PPMD model a 14 000 MB heap (predictor.cpp:101). Default: the same budget when a quarter of the
    // free HBM covers it, else that quarter (>= 64 MB); CMIXB200_PPMD_MB overrides. Text positions share the successor word
    // with context references (below PPMD_CTX_BASE), so the text arena stops short of 1 GiB and the rest goes to the states.
    const char* mb_env = getenv("CMIXB200_PPMD_MB");
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    size_t mb = mb_env ? (size_t)atol(mb_env) : std::min<size_t>(14000, free_b / 4 >> 20);
    if (mb < 64) mb = 64;
    PpmdModel pm;
    memset(&pm, 0, sizeof pm);
    const size_t bytes = mb << 20;
    const size_t text_b = std::min<size_t>(bytes / 4, (size_t)PPMD_CTX_BASE - 4096);
    const size_t ctx_b = bytes / 4;
    const size_t pool_b = bytes - text_b - ctx_b;
    pm.ctx_cap = (uint32_t)std::min<size_t>(ctx_b / sizeof(PpmdCtx), 0x7fffffffu);
    pm.pool_cap = (uint32_t)std::min<size_t>(pool_b / sizeof(PpmdSt), 0xfffffff0u);
    pm.text_cap = (uint32_t)text_b;
    TRY(P->Alloc(&pm.ctx, pm.ctx_cap, false));
    TRY(P->Alloc(&pm.pool, pm.pool_cap, false));
    TRY(P->Alloc(&pm.text, pm.text_cap, false));
    TRY(P->Alloc(&P->d_ppmd_model, 1, false));
    CK(cudaMemcpy(P->d_ppmd_model, &pm, sizeof pm, cudaMemcpyHostToDevice));
    ppmd_init_kernel<<<1, 32>>>(P->d_ppmd_model);
    h.ppmd = P->d_ppmd_model;
  }
  CK(cudaMemcpy(P->d_st, &h, sizeof h, cudaMemcpyHostToDevice));
  if (!(P->replay_mask & CMIXB200_REPLAY_FXCM)) TRY(BuildFxcm(P));
  if (!(P->replay_mask & CMIXB200_REPLAY_PAQ8)) TRY(BuildPaq8(P));
  CK(cudaDeviceSynchronize());
  return CMIXB200_OK;
}

int EnsureScratch(cmixb200_predictor* P, size_t n_bytes) {
  const size_t bits = n_bytes * 8;
  CK(P->d_small_x.Grow(bits * SMALL_X_PITCH));
  CK(P->d_sel.Grow(bits * SEL_PITCH));
  CK(P->d_lstm_x.Grow(bits * 2));
  CK(P->d_decay.Grow(bits));
  CK(P->d_p.Grow(bits));
  CK(P->d_lstm_fx.Grow(bits));
  if ((P->d_fx || P->d_p8) && P->d_ext_gen.n < bits * N_EXT) {     // codes of the resident models: 4 KB per coded bit
    CK(P->d_ext_gen.Grow(bits * N_EXT));
    CK(cudaMemset(P->d_ext_gen.p, 0xFF, bits * N_EXT * 2));   // 0xFFFF = "0.5": slots of a model that is neither resident nor replayed
  }
  return CMIXB200_OK;
}

// The mixers' learning-rate factor after `steps` coded bits (mixer.cpp:58).
float MixerDecay(u64 steps) { return 0.9 / pow(0.0000001 * steps + 0.8, 0.8); }

void FillDecay(std::vector<float>& out, u64 steps0, size_t n_bits) {
  out.resize(n_bits);
  for (size_t i = 0; i < n_bits; ++i) out[i] = MixerDecay(steps0 + i);
}

void HarvestKernelTimes(cmixb200_predictor* P) {
  for (auto& ev : P->pending_kev) {
    float ms = 0.0f;
    if (cudaEventElapsedTime(&ms, ev.a, ev.b) == cudaSuccess) { P->kernel_ms[ev.which] += ms; P->kernel_n[ev.which]++; }
    cudaEventDestroy(ev.a); cudaEventDestroy(ev.b);
  }
  P->pending_kev.clear();
}

// Waits until every library stream of P is idle.
int SyncStreams(cmixb200_predictor* P) {
  for (cudaStream_t s : {P->s_small, P->s_lstm, P->s_mix, P->s_ppmd, P->s_fx, P->s_p8}) if (s) CK(cudaStreamSynchronize(s));
  return CMIXB200_OK;
}

// PAQ8's sticky error word: a block the resident model does not cover (the reference would switch to its image / audio / JPEG
// models there) or two mixer selectors on one weight set. The stream's predictions are no longer the reference's.
int CheckPaq8(cmixb200_predictor* P) {
  if (!P->d_p8) return CMIXB200_OK;
  uint32_t err = 0;
  CK(cudaMemcpy(&err, (const char*)P->d_p8 + offsetof(p8::State, error), 4, cudaMemcpyDeviceToHost));
  if (err & p8::ERR_UNSUPPORTED_BLOCK) { g_last_error = "PAQ8: the stream holds an image / audio / JPEG block; those sub-models are not resident (replay the PAQ8 inputs: CMIXB200_REPLAY_PAQ8)"; return CMIXB200_ERR_UNSUPPORTED; }
  if (err) { g_last_error = "PAQ8: two mixer selectors met on one weight set"; return CMIXB200_ERR_UNSUPPORTED; }
  return CMIXB200_OK;
}

// The resident PPMD model's sticky error word: its arenas are full.
int CheckPpmd(cmixb200_predictor* P) {
  if (!P->d_ppmd_model) return CMIXB200_OK;
  uint32_t err = 0;
  CK(cudaMemcpy(&err, (const char*)P->d_ppmd_model + offsetof(PpmdModel, error), 4, cudaMemcpyDeviceToHost));
  if (err) { g_last_error = "PPMD arena exhausted: raise CMIXB200_PPMD_MB (the reference would cut its model off here)"; return CMIXB200_ERR_CAPACITY; }
  return CMIXB200_OK;
}

// The slots [first, last) of d_ext_bit that the caller feeds per bit (cmixb200_feed_external_bit); the device produces the
// resident models' slots.
std::pair<size_t, size_t> ReplayedSlots(const cmixb200_predictor* P) {
  return {P->d_fx ? (size_t)fx::N_OUT : 0, P->d_p8 ? (size_t)fx::N_OUT : (size_t)N_EXT};
}

// Launch the bulk kernels of one sub-chunk for a batch of streams whose ChunkArgs are already on the device:
// ppmd -> (small | lstm -> fxcm) -> mix [-> encode], each on its own CUDA stream of the group's lead predictor.
int LaunchChunk(cmixb200_predictor* lead, ChunkArgs* d_args, int n_streams, bool pretrain, bool with_coder = false,
                bool with_ppmd = false, bool with_fx = false, bool with_p8 = false) {
  const Tables T = lead->T;
  // optional CUDA-event timing of every kernel on the stream it is launched on (bench.py)
  auto tick = [&](cudaStream_t st) -> cudaEvent_t { cudaEvent_t e = nullptr; if (lead->time_mix) { cudaEventCreate(&e); cudaEventRecord(e, st); } return e; };
  auto tock = [&](int which, cudaEvent_t a, cudaStream_t st) { if (a) { cudaEvent_t b = nullptr; cudaEventCreate(&b); cudaEventRecord(b, st); lead->pending_kev.push_back({which, a, b}); } };
  for (int i = 0; i < 8; ++i) if (!lead->ev[i]) CK(cudaEventCreateWithFlags(&lead->ev[i], cudaEventDisableTiming));
  if (with_ppmd && !pretrain) {
    // the PPMD producer runs ahead on its own stream; both consumers of its distributions wait for this sub-chunk's
    { cudaEvent_t t = tick(lead->s_ppmd);
    ppmd_kernel<<<(n_streams + PPMD_WARPS - 1) / PPMD_WARPS, PPMD_WARPS * 32, PPMD_WARPS * sizeof(PpmdWarpShared), lead->s_ppmd>>>(d_args, n_streams);
    tock(3, t, lead->s_ppmd); }
    lead->launches++;
    CK(cudaEventRecord(lead->ev[0], lead->s_ppmd));
    CK(cudaStreamWaitEvent(lead->s_small, lead->ev[0], 0));
    CK(cudaStreamWaitEvent(lead->s_lstm, lead->ev[0], 0));
  }
  { cudaEvent_t t = tick(lead->s_small);
  small_kernel<<<n_streams, 64, sizeof(SmallState), lead->s_small>>>(d_args, T);
  tock(1, t, lead->s_small); }
  lead->launches++;
  if (with_p8) {   // PAQ8 depends on the coded bytes only: it starts at once on its own stream
    { cudaEvent_t t = tick(lead->s_p8);
    paq8_launch_chunk(d_args, n_streams, lead->s_p8);
    tock(5, t, lead->s_p8); }
    lead->launches++;
  }
  if (pretrain) {
    if (with_fx) { fxcm_launch_chunk(d_args, n_streams, lead->s_fx); lead->launches++; }
  } else {
    { cudaEvent_t t = tick(lead->s_lstm);
    lstm_kernel<<<LSTM_CTAS * n_streams, LSTM_THREADS, sizeof(LstmShared), lead->s_lstm>>>(d_args, T);
    tock(2, t, lead->s_lstm); }
    lead->launches++;
    CK(cudaEventRecord(lead->ev[1], lead->s_small));
    CK(cudaEventRecord(lead->ev[2], lead->s_lstm));
    if (with_fx) {
      // FXCM consumes the LSTM's bit read-outs of this sub-chunk (lstmpr / lstmex) and produces 431 codes per bit
      CK(cudaStreamWaitEvent(lead->s_fx, lead->ev[2], 0));
      { cudaEvent_t t = tick(lead->s_fx);
      fxcm_launch_chunk(d_args, n_streams, lead->s_fx);
      tock(4, t, lead->s_fx); }
      lead->launches++;
      CK(cudaEventRecord(lead->ev[3], lead->s_fx));
      CK(cudaStreamWaitEvent(lead->s_mix, lead->ev[3], 0));
    }
    if (with_p8) { CK(cudaEventRecord(lead->ev[4], lead->s_p8)); CK(cudaStreamWaitEvent(lead->s_mix, lead->ev[4], 0)); }
    // the mixer consumes what the producers write: order it after all of them
    CK(cudaStreamWaitEvent(lead->s_mix, lead->ev[1], 0));
    CK(cudaStreamWaitEvent(lead->s_mix, lead->ev[2], 0));
    { cudaEvent_t t = tick(lead->s_mix);
    mix_kernel_v3<<<2 * n_streams, MIX_THREADS, sizeof(MixBulkShared), lead->s_mix>>>(d_args, T);
    tock(0, t, lead->s_mix); }
    lead->launches++;
    if (with_coder) { encode_kernel<<<n_streams, 32, 0, lead->s_mix>>>(d_args); lead->launches++; }
    // the producers of the NEXT sub-chunk overwrite nothing the mixer still reads (scratch is indexed by bit), except
    // the LSTM feedback FXCM reads: it is per-bit scratch too, so no back edge is needed.
  }
  CK(cudaGetLastError());
  return CMIXB200_OK;
}

// Advance n_streams predictors (same device) by n_bytes each. Software pipeline over sub-chunks:
// the two producer kernels (small models, LSTM) of sub-chunk k+1 run on their own CUDA streams
// while the mixer consumes sub-chunk k. All pointers are device pointers.
int RunPipelined(cmixb200_predictor** preds, int n_streams, const u8* const* d_bytes, size_t n_bytes,
                 const u16* const* d_ext, const float* const* d_ppmd, float* const* d_p_out, bool pretrain) {
  if (n_bytes == 0 || n_streams <= 0) return CMIXB200_OK;
  cmixb200_predictor* lead = preds[0];
  CK(cudaSetDevice(lead->device));
  static const size_t kSub = getenv("CMIXB200_SUBCHUNK") ? (size_t)atol(getenv("CMIXB200_SUBCHUNK")) : 128;
  // Sub-chunk plan: a geometric head (16, 16, 32, 64), full sub-chunks, a geometric tail (64, 32, 16, 16).
  // Head: the mixer of a stream cannot start before the producers of its first sub-chunk are done, so the first one
  // is short. Tail: the call returns when the mixer of the LAST sub-chunk is done, and while it runs the producers
  // have nothing left to do (two thirds of the SMs idle), so the last one is short too.
  std::vector<std::pair<size_t, size_t>> subs;
  if (pretrain) subs.push_back({0, n_bytes});
  else {
    size_t off = 0;
    for (size_t h = 16; h < kSub && n_bytes - off > 2 * kSub; h *= 2) {
      if (h == 16) { subs.push_back({off, h}); off += h; }
      subs.push_back({off, h}); off += h;
    }
    while (n_bytes - off > kSub) { subs.push_back({off, kSub}); off += kSub; }
    size_t rem = n_bytes - off;
    while (rem > 16) { const size_t h = (rem + 1) / 2; subs.push_back({off, h}); off += h; rem -= h; }
    if (rem) subs.push_back({off, rem});
  }
  const size_t n_sub = subs.size();
  std::vector<ChunkArgs> args(n_sub * n_streams);
  std::vector<float> decay;
  u64 decay_steps0 = 0;
  bool any_coder = false, any_ppmd = false, any_fx = false, any_p8 = false;
  for (int s = 0; s < n_streams; ++s) {
    cmixb200_predictor* P = preds[s];
    if (P->device != lead->device || P->bit_context != 1) { g_last_error = "bulk coding: streams must share a device and start on a byte boundary"; return CMIXB200_ERR_ARG; }
    if ((P->d_fx != nullptr) != (lead->d_fx != nullptr) || (P->d_p8 != nullptr) != (lead->d_p8 != nullptr)) { g_last_error = "bulk coding: streams of one batch must agree on which models are resident"; return CMIXB200_ERR_ARG; }
    TRY(SyncStreams(P));                                 // a lock-step Perceive() or the decoder may still be in flight
    if (!pretrain) TRY(EnsureScratch(P, n_bytes));      // Pretrain() touches models and contexts only: no per-bit scratch
    if (!pretrain && !(d_ppmd && d_ppmd[s])) CK(P->d_ppmd_gen.Grow(n_bytes * 256));
    if (!pretrain) {
      // the decay schedule depends only on the number of coded bits: streams that advance together share it
      // (393 216 double pow() calls per 2 KiB step and stream would otherwise cost more host time than a launch set)
      if (decay.empty() || decay_steps0 != P->bits_done) { FillDecay(decay, P->bits_done, n_bytes * 8); decay_steps0 = P->bits_done; }
      CK(cudaMemcpy(P->d_decay.p, decay.data(), decay.size() * 4, cudaMemcpyHostToDevice));
    }
    for (size_t k = 0; k < n_sub; ++k) {
      const size_t off = subs[k].first, n = subs[k].second;
      ChunkArgs& a = args[k * n_streams + s];
      memset(&a, 0, sizeof a);
      a.st = P->d_st; a.bytes = d_bytes[s] + off;
      a.ext = (d_ext && d_ext[s]) ? d_ext[s] + off * 8 * N_EXT : nullptr;
      if (P->d_fx || P->d_p8) {                                    // resident FXCM / PAQ8: the mixer stages from the generated codes
        a.fx = P->d_fx; a.paq8 = P->d_p8;
        a.ext_replay = a.ext;
        if (!pretrain) { a.ext_gen = P->d_ext_gen.p + off * 8 * N_EXT; a.ext = a.ext_gen; a.lstm_fx = P->d_lstm_fx.p + off * 8; }
        any_fx = any_fx || P->d_fx != nullptr; any_p8 = any_p8 || P->d_p8 != nullptr;
      }
      a.ppmd = (d_ppmd && d_ppmd[s]) ? d_ppmd[s] + off * 256 : nullptr;
      if (!a.ppmd && !pretrain) {                                   // no replay: the resident model produces the distributions
        a.ppmd_gen = P->d_ppmd_gen.p + off * 256;
        a.ppmd = a.ppmd_gen;
        any_ppmd = true;
      }
      if (!pretrain) {
        a.decay = P->d_decay.p + off * 8;
        a.small_x = P->d_small_x.p + off * 8 * SMALL_X_PITCH; a.sel = P->d_sel.p + off * 8 * SEL_PITCH;
        a.lstm_x = P->d_lstm_x.p + off * 8 * 2;
      }
      a.p_out = (d_p_out && d_p_out[s]) ? d_p_out[s] + off * 8 : nullptr;
      if (P->coder_on && !pretrain) {
        a.coder = P->d_coder.p;
        if (!a.p_out) a.p_out = P->d_p.p + off * 8;        // the coder reads the probabilities from scratch
        any_coder = true;
      }
      a.n_bytes = (u32)n; a.pretrain = pretrain ? 1 : 0; a.prof = P->d_prof.p;
    }
  }
  CK(lead->d_args.Grow(args.size()));
  CK(cudaMemcpy(lead->d_args.p, args.data(), sizeof(ChunkArgs) * args.size(), cudaMemcpyHostToDevice));
  // Launch groups: each group of streams runs on the CUDA streams of its first predictor, so one group's mixer
  // only waits for its own producers and the groups drift apart instead of moving in lock-step waves.
  static const int kGroup = getenv("CMIXB200_GROUP") ? atoi(getenv("CMIXB200_GROUP")) : 8;
  const int gsz = kGroup > 0 ? kGroup : n_streams;
  for (size_t k = 0; k < n_sub; ++k)
    for (int g0 = 0; g0 < n_streams; g0 += gsz) {
      const int cnt = n_streams - g0 < gsz ? n_streams - g0 : gsz;
      TRY(LaunchChunk(preds[g0], lead->d_args.p + k * n_streams + g0, cnt, pretrain, any_coder, any_ppmd, any_fx, any_p8));
    }
  for (int g0 = 0; g0 < n_streams; g0 += gsz) {
    TRY(SyncStreams(preds[g0]));
    HarvestKernelTimes(preds[g0]);
  }
  if (!pretrain) for (int s = 0; s < n_streams; ++s) preds[s]->bits_done += n_bytes * 8;
  // The bulk kernels keep the resident models' codes for the next bit in their State only; a lock-step Predict() or the
  // decoder's first prediction reads them from d_ext_bit, so hand them over (the models' current outputs, predictor.cpp:361-369).
  // Replayed slots keep their rule: 0.5 until fed.
  for (int s = 0; s < n_streams; ++s) {
    cmixb200_predictor* P = preds[s];
    if (P->d_fx) CK(cudaMemcpyAsync(P->d_ext_bit.p, (const u8*)P->d_fx + offsetof(fx::State, codes), fx::N_OUT * sizeof(u16), cudaMemcpyDeviceToDevice, P->s_mix));
    if (P->d_p8) CK(cudaMemcpyAsync(P->d_ext_bit.p + fx::N_OUT, (const u8*)P->d_p8 + offsetof(p8::State, codes), p8::N_OUT * sizeof(u16), cudaMemcpyDeviceToDevice, P->s_mix));
  }
  for (int s = 0; s < n_streams; ++s) if (preds[s]->d_fx || preds[s]->d_p8) CK(cudaStreamSynchronize(preds[s]->s_mix));   // PAQ8's next Perceive() writes on s_p8
  if (any_ppmd) for (int s = 0; s < n_streams; ++s) TRY(CheckPpmd(preds[s]));
  if (any_p8) for (int s = 0; s < n_streams; ++s) TRY(CheckPaq8(preds[s]));
  return CMIXB200_OK;
}

// Bulk calls are cut into pieces so that the per-bit scratch (4 KB of model codes per coded bit when a model is resident)
// stays bounded whatever n_bytes the caller passes; a piece is long enough (16 k bits) to amortise the pipeline fill.
const size_t kMaxPiece = 2048;

int RunPieces(cmixb200_predictor** preds, int n_streams, const u8* const* d_bytes, size_t n_bytes, const u16* const* d_ext,
              const float* const* d_ppmd, float* const* d_p_out, bool pretrain) {
  bool bounded = false;                       // only the codes of resident models need per-bit scratch worth bounding
  for (int s = 0; s < n_streams; ++s) bounded = bounded || preds[s]->d_fx != nullptr || preds[s]->d_p8 != nullptr;
  if (pretrain || !bounded || n_bytes <= kMaxPiece) return RunPipelined(preds, n_streams, d_bytes, n_bytes, d_ext, d_ppmd, d_p_out, pretrain);
  std::vector<const u8*> b(n_streams); std::vector<const u16*> e(n_streams); std::vector<const float*> q(n_streams); std::vector<float*> o(n_streams);
  for (size_t off = 0; off < n_bytes; off += kMaxPiece) {
    const size_t n = n_bytes - off < kMaxPiece ? n_bytes - off : kMaxPiece;
    for (int s = 0; s < n_streams; ++s) {
      b[s] = d_bytes[s] + off;
      e[s] = (d_ext && d_ext[s]) ? d_ext[s] + off * 8 * N_EXT : nullptr;
      q[s] = (d_ppmd && d_ppmd[s]) ? d_ppmd[s] + off * 256 : nullptr;
      o[s] = (d_p_out && d_p_out[s]) ? d_p_out[s] + off * 8 : nullptr;
    }
    TRY(RunPipelined(preds, n_streams, b.data(), n, d_ext ? e.data() : nullptr, d_ppmd ? q.data() : nullptr, d_p_out ? o.data() : nullptr, false));
  }
  return CMIXB200_OK;
}

int CodeDevice(cmixb200_predictor* P, const u8* d_bytes, size_t n_bytes, const u16* d_ext, const float* d_ppmd,
               float* d_p_out, bool pretrain) {
  return RunPieces(&P, 1, &d_bytes, n_bytes, &d_ext, &d_ppmd, &d_p_out, pretrain);
}

}  // namespace

extern "C" {

const char* cmixb200_last_error(void) { return g_last_error.c_str(); }

int cmixb200_create(const uint8_t vocab[256], const char* dictionary_path, int device, cmixb200_predictor** out) {
  return cmixb200_create_ex(vocab, dictionary_path, device, 0, out);
}

int cmixb200_create_ex(const uint8_t vocab[256], const char* dictionary_path, int device, unsigned replay_mask, cmixb200_predictor** out) {
  if (!vocab || !out) { g_last_error = "null argument"; return CMIXB200_ERR_ARG; }
  int n_dev = 0;
  CK(cudaGetDeviceCount(&n_dev));
  if (device < 0 || device >= n_dev) { g_last_error = "no such CUDA device"; return CMIXB200_ERR_CUDA; }
  CK(cudaSetDevice(device));
  SharedTables* shared = nullptr;
  TRY(BuildSharedTables(device, &shared));
  cmixb200_predictor* P = new cmixb200_predictor();
  P->device = device;
  P->shared = shared; P->T = shared->T;
  P->replay_mask = replay_mask;
  if (dictionary_path) P->dict_path = dictionary_path;
  for (int i = 0; i < 256; ++i) { P->vocab[i] = vocab[i] ? 1 : 0; P->V += P->vocab[i]; }
  if (P->V == 0) { delete P; g_last_error = "empty vocabulary"; return CMIXB200_ERR_ARG; }
  int r = BuildStream(P);
  if (r == CMIXB200_OK) {
    // the mixer is the longest pole of the three and depends on both producers: when many streams
    // oversubscribe the SMs its CTAs should be placed first, then the small models, then the LSTM clusters
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    const bool use_prio = getenv("CMIXB200_NO_PRIORITY") == nullptr;
    const int p_mix = use_prio ? prio_hi : 0, p_small = use_prio ? (prio_hi + 1 <= prio_lo ? prio_hi + 1 : prio_lo) : 0, p_lstm = use_prio ? prio_lo : 0;
    cudaStreamCreateWithPriority(&P->s_small, cudaStreamNonBlocking, p_small);
    cudaStreamCreateWithPriority(&P->s_lstm, cudaStreamNonBlocking, p_lstm);
    cudaStreamCreateWithPriority(&P->s_mix, cudaStreamNonBlocking, p_mix);
    cudaStreamCreateWithPriority(&P->s_ppmd, cudaStreamNonBlocking, p_mix);      // one warp per stream, must never be the one waited for
    cudaStreamCreateWithPriority(&P->s_fx, cudaStreamNonBlocking, p_small);
    cudaStreamCreateWithPriority(&P->s_p8, cudaStreamNonBlocking, p_small);
    cudaEventCreateWithFlags(&P->ev_lock_mix, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&P->ev_lock_small, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&P->ev_lock_p8, cudaEventDisableTiming);
    cudaEventRecord(P->ev_lock_mix, P->s_mix);
    if (P->d_ext_bit.Grow(N_EXT) != cudaSuccess || P->d_ppmd_byte.Grow(256) != cudaSuccess) r = CMIXB200_ERR_CUDA;
    else cudaMemset(P->d_ext_bit.p, 0xFF, N_EXT * 2);
  }
  if (r != CMIXB200_OK) { cmixb200_destroy(P); return r; }
  *out = P;
  return CMIXB200_OK;
}

void cmixb200_destroy(cmixb200_predictor* P) {
  if (!P) return;
  cudaSetDevice(P->device);
  cudaDeviceSynchronize();
  for (void* q : P->allocs) cudaFree(q);
  for (cudaEvent_t e : {P->ev_lock_mix, P->ev_lock_small, P->ev_lock_p8}) if (e) cudaEventDestroy(e);
  for (int i = 0; i < 8; ++i) if (P->ev[i]) cudaEventDestroy(P->ev[i]);
  for (auto& g : P->dec_graph) if (g) cudaGraphExecDestroy(g);
  for (cudaStream_t s : {P->s_small, P->s_lstm, P->s_mix, P->s_ppmd, P->s_fx, P->s_p8, P->s_copy}) if (s) cudaStreamDestroy(s);
  delete P;                            // frees the DeviceBuf members
}

int cmixb200_feed_external_bit(cmixb200_predictor* P, const uint16_t* codes) {
  CK(cudaSetDevice(P->device));
  CK(cudaStreamSynchronize(P->s_mix));           // the resident models of the previous Perceive() write d_ext_bit on s_mix
  const auto [first, last] = ReplayedSlots(P);   // only the replayed slots are taken from the caller
  if (last > first) CK(cudaMemcpy(P->d_ext_bit.p + first, codes + first, (last - first) * 2, cudaMemcpyHostToDevice));
  P->ext_bit_valid = true;
  return CMIXB200_OK;
}
int cmixb200_feed_external_byte(cmixb200_predictor* P, const float* ppmd256) {
  CK(cudaSetDevice(P->device));
  CK(cudaStreamSynchronize(P->s_mix));           // small_perceive / lstm_byte kernels of the previous byte read d_ppmd_byte
  CK(cudaStreamSynchronize(P->s_small));
  CK(cudaMemcpy(P->d_ppmd_byte.p, ppmd256, 256 * 4, cudaMemcpyHostToDevice));
  P->ppmd_byte_valid = true;
  return CMIXB200_OK;
}

// The three predict launches of a bit: producers (small models || LSTM read-out) on s_small behind the previous small_perceive
// and the previous bit's mixer / LSTM update (ev_lock_mix: the LSTM's read-out is final), then 26 row CTAs (one serial chain
// each) and the final stage on s_mix behind the producers, the previous bit's FXCM update (s_mix) and its PAQ8 update (s_p8).
// Lock-step Predict() and the decoder's graphs queue them through this one function.
static int LaunchPredict(cmixb200_predictor* P) {
  const Tables T = P->T;
  CK(cudaStreamWaitEvent(P->s_small, P->ev_lock_mix, 0));
  lock_predict_inputs_kernel<<<2, 64, 0, P->s_small>>>(P->d_st, T);
  CK(cudaEventRecord(P->ev_lock_small, P->s_small));
  CK(cudaStreamWaitEvent(P->s_mix, P->ev_lock_small, 0));
  if (P->d_p8) CK(cudaStreamWaitEvent(P->s_mix, P->ev_lock_p8, 0));
  mix_predict_rows_kernel<<<N_L0, 256, 0, P->s_mix>>>(P->d_st, T, (P->ext_bit_valid || P->d_fx || P->d_p8) ? P->d_ext_bit.p : nullptr);
  mix_predict_final_kernel<<<1, MIX_THREADS, 0, P->s_mix>>>(P->d_st, T);
  P->launches += 3;
  return CMIXB200_OK;
}

float cmixb200_predict(cmixb200_predictor* P) {
  if (cudaSetDevice(P->device) != cudaSuccess) { g_last_error = "cudaSetDevice failed"; return -1.0f; }
  if (LaunchPredict(P) != CMIXB200_OK) return -1.0f;
  float p = -1.0f;
  cudaError_t e = cudaMemcpyAsync(&p, &P->d_st->last_p, 4, cudaMemcpyDeviceToHost, P->s_mix);
  if (e == cudaSuccess) e = cudaStreamSynchronize(P->s_mix);      // also surfaces errors of the previous Perceive()
  if (e != cudaSuccess) { g_last_error = std::string("predict: ") + cudaGetErrorString(e); return -1.0f; }
  if (P->bit_context == 1 && P->bits_done) {   // once per byte: the sticky error words of the resident models (s_mix is idle here)
    if (CheckPaq8(P) != CMIXB200_OK || CheckPpmd(P) != CMIXB200_OK) return -1.0f;
  }
  if (P->ext_bit_valid) {   // replayed slots fall back to "0.5" until they are fed again
    const auto [first, last] = ReplayedSlots(P);
    if (last > first) cudaMemsetAsync(P->d_ext_bit.p + first, 0xFF, (last - first) * 2, P->s_mix);
  }
  P->ext_bit_valid = false;
  return p;
}

// The perceive launches of a bit. In the decoder's graphs `dbit` (device, {bit, completed byte}, written on s_mix by
// decode_step_kernel) replaces `bit` and `full`, and the mixer takes the step's decay from the DecodeState; byte_done is
// positional either way. Queued, not awaited: the next predict launches are ordered behind them by events.
static int LaunchPerceive(cmixb200_predictor* P, int bit, u32 full, bool byte_done, float decay, const u32* dbit) {
  const float* ppmd = byte_done ? P->d_ppmd_byte.p : nullptr;
  if (dbit) {                                    // the decoded bit is produced on s_mix
    CK(cudaEventRecord(P->ev_lock_mix, P->s_mix));
    CK(cudaStreamWaitEvent(P->s_small, P->ev_lock_mix, 0));
    if (P->d_p8) CK(cudaStreamWaitEvent(P->s_p8, P->ev_lock_mix, 0));
  }
  if (byte_done && !P->ppmd_byte_valid) {
    // no replayed distribution for this byte: the resident PPMD model is updated and emits it (ppmd.cpp:1328-1338)
    ppmd_byte_kernel<<<1, 32, sizeof(PpmdWarpShared), P->s_small>>>(P->d_st, full, P->d_ppmd_byte.p, dbit);
    P->launches++;
    CK(cudaEventRecord(P->ev_lock_small, P->s_small));
    CK(cudaStreamWaitEvent(P->s_mix, P->ev_lock_small, 0));          // lstm_byte_kernel reads it too
  }
  small_perceive_kernel<<<1, 64, 0, P->s_small>>>(P->d_st, bit, ppmd, 0, dbit);      // concurrent with the mixer / LSTM update
  mix_perceive_kernel<<<N_L0 + 2, MIX_THREADS, 0, P->s_mix>>>(P->d_st, bit, decay, dbit);
  P->launches += 2;
  if (byte_done) { lstm_byte_kernel<<<LSTM_CTAS, LSTM_THREADS, sizeof(LstmShared), P->s_mix>>>(P->d_st, full, ppmd, dbit); P->launches++; }
  CK(cudaEventRecord(P->ev_lock_mix, P->s_mix));     // the LSTM's read-out is final: the next bit's producers may start
  // FXCM is perceived last and sees the LSTM's read-out of the next bit (predictor.cpp:462-466); PAQ8 needs the bit only
  if (P->d_fx) { fxcm_launch_bit(P->d_st, P->d_fx, bit, 0, P->d_ext_bit.p, P->s_mix, dbit); P->launches++; }
  if (P->d_p8) {
    paq8_launch_bit(P->d_p8, bit, P->d_ext_bit.p, P->s_p8, dbit);
    P->launches++;
    CK(cudaEventRecord(P->ev_lock_p8, P->s_p8));
  }
  CK(cudaGetLastError());
  return CMIXB200_OK;
}

int cmixb200_perceive(cmixb200_predictor* P, int bit) {
  CK(cudaSetDevice(P->device));
  bit = bit ? 1 : 0;
  const bool byte_done = P->bit_context >= 128;
  const u32 full = (P->bit_context * 2 + bit) & 255;
  // the previous Predict() waited for s_mix, so the row kernel that read d_ext_bit is done before PAQ8 rewrites its slots
  TRY(LaunchPerceive(P, bit, full, byte_done, MixerDecay(P->bits_done), nullptr));
  P->bits_done++;
  P->bit_context = byte_done ? 1 : P->bit_context * 2 + bit;
  if (byte_done) P->ppmd_byte_valid = false;
  return CMIXB200_OK;
}

// One bit of the decode loop as CUDA graph `g`: the decoder step for the standing prediction, the perceive kernels of that bit,
// then the predict kernels of the NEXT bit (its producers overlap the tail of FXCM / PAQ8), or for the last bit of a call the
// join of s_small and s_p8 into s_mix. Launches of the graph on s_mix run one after the other, so no event crosses from one bit
// to the next. Expects every library stream idle.
static int BuildDecodeGraph(cmixb200_predictor* P, int g) {
  const unsigned long long launches0 = P->launches;
  CK(cudaStreamBeginCapture(P->s_mix, cudaStreamCaptureModeThreadLocal));
  auto capture = [&]() -> int {
    decode_step_kernel<<<1, 1, 0, P->s_mix>>>(P->d_st, P->d_dec.p);
    P->launches++;
    TRY(LaunchPerceive(P, 0, 0, g > 0, 0.0f, reinterpret_cast<const u32*>(P->d_dec.p)));
    if (g < 2) return LaunchPredict(P);
    // the last bit of a call: no prediction is left standing (a bulk call or Predict() may follow)
    CK(cudaEventRecord(P->ev_lock_small, P->s_small));
    CK(cudaStreamWaitEvent(P->s_mix, P->ev_lock_small, 0));
    CK(cudaStreamWaitEvent(P->s_mix, P->ev_lock_p8, 0));
    return CMIXB200_OK;
  };
  int r = capture();
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(P->s_mix, &graph);   // ends the capture also when a launch above failed
  // Inside the capture the events only ordered the graph's nodes; record them again on the idle streams so that lock-step
  // calls can wait on them.
  if ((cudaEventRecord(P->ev_lock_mix, P->s_mix) != cudaSuccess || cudaEventRecord(P->ev_lock_small, P->s_small) != cudaSuccess ||
       cudaEventRecord(P->ev_lock_p8, P->s_p8) != cudaSuccess) && r == CMIXB200_OK) {
    g_last_error = "decode graph: event record failed"; r = CMIXB200_ERR_CUDA;
  }
  P->dec_launches[g] = P->launches - launches0;
  P->launches = launches0;                                         // counted per graph launch
  if (r == CMIXB200_OK && (ce != cudaSuccess || !graph)) { g_last_error = std::string("decode graph: ") + cudaGetErrorString(ce); r = CMIXB200_ERR_CUDA; }
  if (r == CMIXB200_OK) {
    cudaGraphExec_t exec = nullptr;
    const cudaError_t ci = cudaGraphInstantiate(&exec, graph, 0);
    if (ci == cudaSuccess) P->dec_graph[g] = exec;
    else { g_last_error = std::string("decode graph: ") + cudaGetErrorString(ci); r = CMIXB200_ERR_CUDA; }
  }
  if (graph) cudaGraphDestroy(graph);
  return r;
}

// Decoder::Decode for n_bytes on the device (SURVEY §8f rank 1): per bit one graph launch = predict kernels, one arithmetic-decoder
// step, perceive kernels; the bit never visits the host, which only queues the launches and waits once per 1 024 bits.
int cmixb200_decode_bytes(cmixb200_predictor* P, const uint8_t* archive, size_t n_archive, uint8_t* out, size_t n_bytes) {
  CK(cudaSetDevice(P->device));
  if (!archive || !out) { g_last_error = "decode_bytes: null argument"; return CMIXB200_ERR_ARG; }
  if (P->bit_context != 1) { g_last_error = "decode_bytes: the stream must stand on a byte boundary"; return CMIXB200_ERR_ARG; }
  if (!P->d_fx || !P->d_p8) { g_last_error = "decode_bytes needs every model group resident"; return CMIXB200_ERR_ARG; }
  if (n_bytes == 0) return CMIXB200_OK;
  const size_t n_bits = n_bytes * 8;
  TRY(SyncStreams(P));                           // a lock-step Perceive() or a bulk call may still be in flight
  // The graphs run the resident PPMD model at every byte, as lock-step does when no distribution was fed: one fed before
  // this call is not used.
  P->ppmd_byte_valid = false;
  CK(P->d_dec.Grow(1));
  for (int g = 0; g < 3; ++g) if (!P->dec_graph[g]) TRY(BuildDecodeGraph(P, g));
  u8 *d_arch = nullptr, *d_out = nullptr;
  float* d_decay = nullptr;
  int r = CMIXB200_OK;
  auto fail = [&](const char* what) { g_last_error = std::string("decode_bytes: ") + what; r = CMIXB200_ERR_CUDA; };
  if (cudaMalloc(&d_arch, n_archive ? n_archive : 1) != cudaSuccess || cudaMalloc(&d_out, n_bytes) != cudaSuccess ||
      cudaMalloc(&d_decay, n_bits * sizeof(float)) != cudaSuccess) fail("out of device memory");
  if (r == CMIXB200_OK) {
    std::vector<float> decay;
    FillDecay(decay, P->bits_done, n_bits);
    DecodeState h;
    memset(&h, 0, sizeof h);
    h.n_arch = n_archive; h.arch = d_arch; h.out = d_out; h.decay = d_decay;
    if (cudaMemcpy(d_arch, archive, n_archive, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(d_decay, decay.data(), n_bits * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(P->d_dec.p, &h, sizeof h, cudaMemcpyHostToDevice) != cudaSuccess) fail("upload failed");
    else {
      decode_begin_kernel<<<1, 1, 0, P->s_mix>>>(P->d_dec.p);
      P->launches++;
      r = LaunchPredict(P);                  // the first prediction; every graph leaves the next one standing
      if (r == CMIXB200_OK && cudaStreamSynchronize(P->s_mix) != cudaSuccess) fail("first prediction failed");
    }
  }
  for (size_t t = 0; r == CMIXB200_OK && t < n_bits; ++t) {
    const int g = t + 1 == n_bits ? 2 : ((t & 7) == 7 ? 1 : 0);
    const cudaError_t ce = cudaGraphLaunch(P->dec_graph[g], P->s_mix);
    if (ce != cudaSuccess) { fail(cudaGetErrorString(ce)); break; }
    P->launches += P->dec_launches[g];
    if ((t & 1023) == 1023) {      // bound the launch queue and surface device errors early
      const cudaError_t cs = cudaStreamSynchronize(P->s_mix);
      if (cs != cudaSuccess) fail(cudaGetErrorString(cs));
    }
  }
  if (r == CMIXB200_OK) {
    const cudaError_t cs = cudaStreamSynchronize(P->s_mix);
    if (cs != cudaSuccess) fail(cudaGetErrorString(cs));
    else if (cudaMemcpy(out, d_out, n_bytes, cudaMemcpyDeviceToHost) != cudaSuccess) fail("download failed");
  }
  if (r == CMIXB200_OK) {
    P->bits_done += n_bits;
    // the next lock-step Predict() is ordered behind the loop
    if (cudaEventRecord(P->ev_lock_mix, P->s_mix) != cudaSuccess) fail("event record failed");
  }
  if (r == CMIXB200_OK) r = CheckPaq8(P);
  if (r == CMIXB200_OK) r = CheckPpmd(P);
  cudaFree(d_arch); cudaFree(d_out); cudaFree(d_decay);
  return r;
}

int cmixb200_pretrain(cmixb200_predictor* P, int bit) {
  CK(cudaSetDevice(P->device));
  bit = bit ? 1 : 0;
  const Tables T = P->T;
  const bool byte_done = P->bit_context >= 128;
  small_predict_kernel<<<1, 64, 0, P->s_small>>>(P->d_st, T);
  small_perceive_kernel<<<1, 64, 0, P->s_small>>>(P->d_st, bit, nullptr, 1);
  P->launches += 2;
  if (P->d_fx) { fxcm_launch_bit(P->d_st, P->d_fx, bit, 1, P->d_ext_bit.p, P->s_mix); P->launches++; }
  if (P->d_p8) { paq8_launch_bit(P->d_p8, bit, P->d_ext_bit.p, P->s_mix); P->launches++; }
  CK(cudaGetLastError());
  P->bit_context = byte_done ? 1 : P->bit_context * 2 + bit;
  return CMIXB200_OK;
}

int cmixb200_code_bytes_device(cmixb200_predictor* P, const uint8_t* d_bytes, size_t n_bytes, const uint16_t* d_ext,
                               const float* d_ppmd, float* d_p_out) {
  return CodeDevice(P, d_bytes, n_bytes, d_ext, d_ppmd, d_p_out, false);
}

int cmixb200_code_bytes(cmixb200_predictor* P, const uint8_t* bytes, size_t n_bytes, const uint16_t* ext,
                        const float* ppmd, float* p_out) {
  CK(cudaSetDevice(P->device));
  const size_t kSub = 4096;     // host staging granularity: 4096 B of input = 132 MB of replayed codes
  CK(P->d_bytes.Grow(kSub));
  CK(P->d_ext.Grow(kSub * 8 * N_EXT));
  CK(P->d_ppmd.Grow(kSub * 256));
  for (size_t off = 0; off < n_bytes; off += kSub) {
    const size_t n = n_bytes - off < kSub ? n_bytes - off : kSub;
    CK(cudaMemcpy(P->d_bytes.p, bytes + off, n, cudaMemcpyHostToDevice));
    if (ext) CK(cudaMemcpy(P->d_ext.p, ext + off * 8 * N_EXT, n * 8 * N_EXT * 2, cudaMemcpyHostToDevice));
    if (ppmd) CK(cudaMemcpy(P->d_ppmd.p, ppmd + off * 256, n * 256 * 4, cudaMemcpyHostToDevice));
    TRY(EnsureScratch(P, n));
    TRY(CodeDevice(P, P->d_bytes.p, n, ext ? P->d_ext.p : nullptr, ppmd ? P->d_ppmd.p : nullptr, P->d_p.p, false));
    CK(cudaMemcpy(p_out + off * 8, P->d_p.p, n * 8 * 4, cudaMemcpyDeviceToHost));
  }
  return CMIXB200_OK;
}

int cmixb200_pretrain_bytes(cmixb200_predictor* P, const uint8_t* bytes, size_t n_bytes) {
  CK(cudaSetDevice(P->device));
  u8* d = nullptr;
  CK(cudaMalloc(&d, n_bytes ? n_bytes : 1));
  CK(cudaMemcpy(d, bytes, n_bytes, cudaMemcpyHostToDevice));
  int r = CodeDevice(P, d, n_bytes, nullptr, nullptr, nullptr, true);
  cudaFree(d);
  return r;
}

int cmixb200_code_batch_device(cmixb200_predictor** preds, int n_streams, const uint8_t* const* d_bytes, size_t n_bytes,
                               const uint16_t* const* d_ext, const float* const* d_ppmd, float* const* d_p_out) {
  return RunPieces(preds, n_streams, d_bytes, n_bytes, d_ext, d_ppmd, d_p_out, false);
}

int cmixb200_code_batch(cmixb200_predictor** preds, int n_streams, const uint8_t* const* bytes, size_t n_bytes,
                        const uint16_t* const* ext, const float* const* ppmd, float* const* p_out) {
  if (n_streams <= 0 || !preds || !bytes || !p_out) { g_last_error = "code_batch: bad arguments"; return CMIXB200_ERR_ARG; }
  cmixb200_predictor* lead = preds[0];
  CK(cudaSetDevice(lead->device));
  const size_t kSub = 1024;     // staging granularity per stream: 1024 B of input = 33 MB of replayed codes; long enough
                                // that a sub-step is bound by SM throughput, not by one stream's serial mixer chain
  if (!lead->s_copy) CK(cudaStreamCreateWithFlags(&lead->s_copy, cudaStreamNonBlocking));
  for (int s = 0; s < n_streams; ++s) {
    cmixb200_predictor* P = preds[s];
    if (P->device != lead->device) { g_last_error = "code_batch: all predictors must live on one device"; return CMIXB200_ERR_ARG; }
    for (int k = 0; k < 2; ++k) {
      CK(P->d_bytes2[k].Grow(kSub));
      CK(P->d_ext2[k].Grow(kSub * 8 * N_EXT));
      CK(P->d_ppmd2[k].Grow(kSub * 256));
    }
    TRY(EnsureScratch(P, kSub));
  }
  auto stage = [&](size_t off, int k) -> int {
    const size_t n = n_bytes - off < kSub ? n_bytes - off : kSub;
    for (int s = 0; s < n_streams; ++s) {
      cmixb200_predictor* P = preds[s];
      CK(cudaMemcpyAsync(P->d_bytes2[k].p, bytes[s] + off, n, cudaMemcpyHostToDevice, lead->s_copy));
      if (ext) CK(cudaMemcpyAsync(P->d_ext2[k].p, ext[s] + off * 8 * N_EXT, n * 8 * N_EXT * 2, cudaMemcpyHostToDevice, lead->s_copy));
      if (ppmd) CK(cudaMemcpyAsync(P->d_ppmd2[k].p, ppmd[s] + off * 256, n * 256 * 4, cudaMemcpyHostToDevice, lead->s_copy));
    }
    return CMIXB200_OK;
  };
  std::vector<const uint8_t*> db(n_streams); std::vector<const uint16_t*> de(n_streams);
  std::vector<const float*> dp(n_streams); std::vector<float*> dout(n_streams);
  if (n_bytes) TRY(stage(0, 0));
  int k = 0;
  for (size_t off = 0; off < n_bytes; off += kSub, k ^= 1) {
    const size_t n = n_bytes - off < kSub ? n_bytes - off : kSub;
    CK(cudaStreamSynchronize(lead->s_copy));                      // stage(off) landed, previous results are on the host
    if (off + kSub < n_bytes) TRY(stage(off + kSub, k ^ 1));      // next inputs travel while this sub-step computes
    for (int s = 0; s < n_streams; ++s) {
      db[s] = preds[s]->d_bytes2[k].p; de[s] = preds[s]->d_ext2[k].p; dp[s] = preds[s]->d_ppmd2[k].p; dout[s] = preds[s]->d_p.p;
    }
    const int rr = RunPipelined(preds, n_streams, db.data(), n, ext ? de.data() : nullptr, ppmd ? dp.data() : nullptr, dout.data(), false);
    if (rr != CMIXB200_OK) { cudaStreamSynchronize(lead->s_copy); return rr; }   // no copy into the caller's buffers stays in flight
    for (int s = 0; s < n_streams; ++s)
      if (cudaMemcpyAsync(p_out[s] + off * 8, preds[s]->d_p.p, n * 8 * 4, cudaMemcpyDeviceToHost, lead->s_copy) != cudaSuccess) {
        g_last_error = "code_batch: result copy failed"; cudaStreamSynchronize(lead->s_copy); return CMIXB200_ERR_CUDA;
      }
  }
  CK(cudaStreamSynchronize(lead->s_copy));
  return CMIXB200_OK;
}

int cmixb200_coder_begin(cmixb200_predictor* P, size_t capacity_bytes) {
  CK(cudaSetDevice(P->device));
  if (capacity_bytes == 0) { g_last_error = "coder_begin: zero capacity"; return CMIXB200_ERR_ARG; }
  CK(P->d_code.Grow(capacity_bytes));
  CK(P->d_coder.Grow(1));
  CoderState c; memset(&c, 0, sizeof c);
  c.x1 = 0; c.x2 = 0xffffffffu; c.cap = capacity_bytes; c.out = P->d_code.p;
  CK(cudaMemcpy(P->d_coder.p, &c, sizeof c, cudaMemcpyHostToDevice));
  P->coder_on = true;
  return CMIXB200_OK;
}

int cmixb200_coder_finish(cmixb200_predictor* P, uint8_t* out, size_t cap, size_t* n_out) {
  CK(cudaSetDevice(P->device));
  if (!P->coder_on) { g_last_error = "coder_finish without coder_begin"; return CMIXB200_ERR_ARG; }
  encode_flush_kernel<<<1, 1, 0, P->s_mix>>>(P->d_coder.p);
  P->launches++;
  CK(cudaStreamSynchronize(P->s_mix));
  CoderState c;
  CK(cudaMemcpy(&c, P->d_coder.p, sizeof c, cudaMemcpyDeviceToHost));
  P->coder_on = false;
  if (n_out) *n_out = (size_t)c.n_out;
  if (c.overflow) { g_last_error = "device coder: archive buffer too small"; return CMIXB200_ERR_ARG; }
  if (c.n_out > cap) { g_last_error = "coder_finish: output buffer too small"; return CMIXB200_ERR_ARG; }
  if (out && c.n_out) CK(cudaMemcpy(out, P->d_code.p, (size_t)c.n_out, cudaMemcpyDeviceToHost));
  return CMIXB200_OK;
}

unsigned long long cmixb200_kernel_launches(const cmixb200_predictor* P) { return P->launches; }
void cmixb200_time_mix_kernel(cmixb200_predictor* P, int enable) { P->time_mix = enable != 0; if (enable) for (int i = 0; i < 6; ++i) { P->kernel_ms[i] = 0; P->kernel_n[i] = 0; } }
double cmixb200_kernel_ms(const cmixb200_predictor* P, int which, unsigned long long* n_launches) {
  if (which < 0 || which > 5) return 0.0;
  if (n_launches) *n_launches = P->kernel_n[which];
  return P->kernel_ms[which];
}
void* cmixb200_mix_stream(cmixb200_predictor* P) { return (void*)P->s_mix; }

int cmixb200_debug_fetch(cmixb200_predictor* P, int what, void* out, size_t bytes) {
  CK(cudaSetDevice(P->device));
  TRY(SyncStreams(P));
  const void* src = nullptr;
  switch (what) {
    case CMIXB200_DBG_SMALL_X: src = P->d_small_x.p; break;
    case CMIXB200_DBG_SEL: src = P->d_sel.p; break;
    case CMIXB200_DBG_LSTM_X: src = P->d_lstm_x.p; break;
    case CMIXB200_DBG_LSTM_PROBS: src = &P->d_st->lstm.bm.probs[0]; break;
    case CMIXB200_DBG_ERROR_FLAGS: src = &P->d_st->small.error; break;
    case CMIXB200_DBG_PPMD_PROBS: src = P->d_ppmd_byte.p; break;
    case CMIXB200_DBG_PPMD_PROFILE: src = (const char*)P->d_ppmd_model + offsetof(PpmdModel, prof); break;
    case CMIXB200_DBG_PPMD_BULK:
      if (bytes > P->d_ppmd_gen.n * sizeof(float)) { g_last_error = "debug_fetch: more PPMD rows than the last bulk call produced"; return CMIXB200_ERR_ARG; }
      src = P->d_ppmd_gen.p; break;
    case CMIXB200_DBG_EXT_GEN:
      if (!P->d_ext_gen.p || bytes > P->d_ext_gen.n * 2) { g_last_error = "debug_fetch: no generated codes of that size"; return CMIXB200_ERR_ARG; }
      src = P->d_ext_gen.p; break;
    case CMIXB200_DBG_EXT_BIT: src = P->d_ext_bit.p; break;
    case CMIXB200_DBG_PPMD_USAGE: {
      PpmdModel pm;
      if (bytes < 6 * 4) { g_last_error = "debug_fetch: PPMD usage is 6 u32"; return CMIXB200_ERR_ARG; }
      CK(cudaMemcpy(&pm, P->d_ppmd_model, sizeof pm, cudaMemcpyDeviceToHost));
      const uint32_t u[6] = {pm.ctx_top, pm.ctx_cap, pm.pool_top, pm.pool_cap, pm.text_pos, pm.text_cap};
      memcpy(out, u, sizeof u);
      return CMIXB200_OK;
    }
    case CMIXB200_DBG_PROFILE:
      if (!P->d_prof.p) { CK(P->d_prof.Grow(64)); CK(cudaMemset(P->d_prof.p, 0, 64 * 8)); }
      src = P->d_prof.p; break;
    default: g_last_error = "unknown debug id"; return CMIXB200_ERR_ARG;
  }
  CK(cudaMemcpy(out, src, bytes, cudaMemcpyDeviceToHost));
  return CMIXB200_OK;
}

}  // extern "C"
