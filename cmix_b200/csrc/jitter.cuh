// cmix_b200/csrc/jitter.cuh — schedule jitter at every synchronisation site of the device code.
//
// Every barrier, mbarrier wait, remote arrive and flag spin of the kernels goes through a helper that carries a site id
// (JIT_HERE: the source file and line), and every kernel starts with jit_entry(). Built with -DCMIXB200_JITTER the hook
// sleeps there (__nanosleep) on a deterministic schedule, so that a test can move warps, CTAs and kernels relative to each
// other and check that every probability stays the same; a missing barrier or event then shows as a wrong bit. Without
// the flag every hook expands to nothing and the helpers compile to the bare primitive.
//
// The sleep is warp-uniform: its length is computed from values every active lane of the warp holds (the visit count is
// the lowest active lane's), and it runs unconditionally (0 ns when the site is not chosen), so the hook adds no
// divergence in front of an aligned barrier. Where only some lanes reach a site (a spin or a remote arrive on lane 0) they
// are already diverged, and a __syncwarp follows before the next aligned barrier or shuffle.
//
// Modes (cmixb200_jitter_config, exported by the jitter build only):
//   JIT_RANDOM  a = density in 1/65536: each visit sleeps 0-1 us with that probability
//   JIT_STARVE  a = group: that warp group sleeps at each of its sites, everyone else runs freely
//   JIT_HURRY   a = group: everyone but that group sleeps at each site
//   JIT_ENTRY   a = kernel (JK_*), b = microseconds (at most 200), c = every n-th launch: the kernel's CTAs start late
// The delay is a hash of (seed, site, CTA, warp, visit count of the site's file by that thread). __nanosleep(t) sleeps at
// most 2t, so one sleep is at most 2 us.
#pragma once

#define JIT_FILE_LIST "engine.cu", "coder.cuh", "fxcm.cuh", "lstm.cuh", "mixer_bulk.cuh", "mixer_lock.cuh", "paq8.cuh", \
                      "ppmd.cuh", "small_models.cuh"
enum { JF_ENGINE, JF_CODER, JF_FXCM, JF_LSTM, JF_MIX_BULK, JF_MIX_LOCK, JF_PAQ8, JF_PPMD, JF_SMALL, JIT_N_FILES,
       JIT_MAX_LINE = 2048 };
// kernels, for JIT_ENTRY
enum { JK_FILL, JK_ENCODE, JK_ENCODE_FLUSH, JK_DECODE_BEGIN, JK_DECODE_STEP, JK_FXCM, JK_FXCM_BIT, JK_LSTM, JK_LSTM_INPUTS,
       JK_LSTM_BYTE, JK_MIX, JK_MIX_ROWS, JK_MIX_FINAL, JK_MIX_PERCEIVE, JK_PAQ8, JK_PAQ8_BIT, JK_PPMD_INIT, JK_PPMD,
       JK_PPMD_BYTE, JK_SMALL, JK_SMALL_PREDICT, JK_SMALL_PERCEIVE, JIT_N_KERNELS };
// warp groups, for JIT_STARVE / JIT_HURRY
enum { JG_NONE,
       JG_P8_OLS, JG_P8_W3_6, JG_P8_DCHAIN, JG_P8_W12, JG_P8_W13_15, JG_P8_MIXER,   // PAQ8: model CTA warps, mixer CTA
       JG_MIX_C, JG_MIX_T, JG_MIX_MOVERS, JG_MIX_CTA1,                            // mix_kernel_v3: CTA 0's roles, CTA 1
       JG_LSTM_R0, JG_LSTM_R1, JG_LSTM_R2, JG_LSTM_R3, JG_LSTM_R4, JG_LSTM_R5, JG_LSTM_R6, JG_LSTM_R7,   // the LSTM cluster, by rank
       JG_FX_MODEL, JG_FX_MIXER,                                                    // FXCM: model CTA, mixer CTA
       JG_PPMD, JG_SMALL, JG_MIX_LOCK, JG_CODER, JG_ENGINE, JIT_N_GROUPS };
enum { JIT_OFF, JIT_RANDOM, JIT_STARVE, JIT_HURRY, JIT_ENTRY };

#ifdef CMIXB200_JITTER
#include <cuda_runtime.h>

namespace cmixb200 {

__host__ __device__ constexpr bool jit_streq(const char* a, const char* b) { return *a == *b && (*a == 0 || jit_streq(a + 1, b + 1)); }
__host__ __device__ constexpr const char* jit_base(const char* p, const char* b) { return *p == 0 ? b : jit_base(p + 1, *p == '/' ? p + 1 : b); }
__host__ __device__ constexpr int jit_file_at(const char* f, int i) {
  constexpr const char* names[] = {JIT_FILE_LIST};
  return i == JIT_N_FILES ? -1 : (jit_streq(f, names[i]) ? i : jit_file_at(f, i + 1));
}
__host__ __device__ constexpr int jit_site_id(const char* file, int line) {
  return jit_file_at(jit_base(file, file), 0) < 0 || line >= JIT_MAX_LINE ? -1 : jit_file_at(jit_base(file, file), 0) * JIT_MAX_LINE + line;
}
template <int S> struct JitSite { static_assert(S >= 0, "a jitter site outside the files of JIT_FILE_LIST"); static constexpr int value = S; };
#define JIT_HERE (::cmixb200::JitSite<::cmixb200::jit_site_id(__FILE__, __LINE__)>::value)

struct JitConfig { int mode; unsigned seed; int a, b, c; };

static __device__ JitConfig jit_cfg;
static __device__ unsigned jit_fired[JIT_N_FILES * JIT_MAX_LINE];        // visits that slept, per site (per warp)
static __device__ unsigned jit_visits[JIT_N_FILES][16][1024];            // per thread: sites of the file it has passed
static __device__ unsigned jit_launches[JIT_N_KERNELS][16][1024];        // per thread: launches of the kernel it has started

__device__ __forceinline__ unsigned jit_mix(unsigned h) {
  h ^= h >> 16; h *= 0x7feb352du; h ^= h >> 15; h *= 0x846ca68bu; h ^= h >> 16;
  return h;
}
__device__ __forceinline__ unsigned jit_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ int jit_group(int file, int rank, int warp) {
  switch (file) {
    case JF_PAQ8: return rank == 1 ? JG_P8_MIXER : warp < 3 ? JG_P8_OLS : warp < 7 ? JG_P8_W3_6 : warp < 12 ? JG_P8_DCHAIN : warp == 12 ? JG_P8_W12 : JG_P8_W13_15;
    case JF_MIX_BULK: return rank == 1 ? JG_MIX_CTA1 : warp == 15 ? JG_MIX_C : warp == 14 ? JG_MIX_T : (warp & 3) != 3 ? JG_MIX_MOVERS : JG_NONE;
    case JF_LSTM: return JG_LSTM_R0 + (rank & 7);
    case JF_FXCM: return rank == 1 ? JG_FX_MIXER : JG_FX_MODEL;
    case JF_PPMD: return JG_PPMD;
    case JF_SMALL: return JG_SMALL;
    case JF_MIX_LOCK: return JG_MIX_LOCK;
    case JF_CODER: return JG_CODER;
    default: return JG_ENGINE;
  }
}
// The sleep of this warp at `site` (0 when it is not chosen); counts the visit.
__device__ __forceinline__ unsigned jit_delay(int site) {
  const JitConfig c = jit_cfg;
  if (c.mode == JIT_OFF || c.mode == JIT_ENTRY) return 0;
  const int file = site / JIT_MAX_LINE;
  const int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z), warp = tid >> 5;
  unsigned& vref = jit_visits[file][blockIdx.x & 15][tid & 1023];
  const unsigned mine = vref;
  vref = mine + 1;
  const unsigned mask = __activemask(), leader = __ffs(mask) - 1;
  const unsigned visit = __shfl_sync(mask, mine, leader);
  const unsigned rank = jit_rank();
  const unsigned h = jit_mix(c.seed ^ jit_mix((unsigned)site * 0x9E3779B1u ^ jit_mix(blockIdx.x * 0x85EBCA77u + (unsigned)warp) ^ visit * 0xC2B2AE3Du));
  const int g = jit_group(file, (int)rank, warp);
  bool on;
  if (c.mode == JIT_RANDOM) on = (h & 0xffffu) < (unsigned)c.a;
  else if (c.mode == JIT_STARVE) on = g == c.a;
  else on = g != c.a;                                   // JIT_HURRY
  const unsigned d = on ? 1u + (h >> 16) % 1000u : 0u;
  if (d && (tid & 31) == (int)leader) atomicAdd(&jit_fired[site], 1u);
  return d;
}
__device__ __forceinline__ void jit_point(int site) { __nanosleep(jit_delay(site)); }
// Kernel entry: a site like any other, and in JIT_ENTRY mode every thread of a chosen launch sleeps b microseconds (every
// thread counts the kernel's launches itself, so the CTA agrees without talking).
__device__ __forceinline__ void jit_entry_point(int kernel, int site) {
  const JitConfig c = jit_cfg;
  if (c.mode == JIT_ENTRY && kernel == c.a) {
    const int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
    unsigned& lref = jit_launches[kernel][blockIdx.x & 15][tid & 1023];
    const unsigned n = lref;
    lref = n + 1;
    const unsigned mask = __activemask();
    const bool on = __shfl_sync(mask, n, __ffs(mask) - 1) % (unsigned)(c.c > 0 ? c.c : 1) == 0;
    const int us = c.b < 200 ? c.b : 200;
    for (int i = 0; i < us; ++i) __nanosleep(on ? 500u : 0u);     // at most 2 x 500 ns per microsecond asked for
    if (on && tid == 0) atomicAdd(&jit_fired[site], 1u);
  } else {
    jit_point(site);
  }
}
#define jit_entry(kernel) ::cmixb200::jit_entry_point(kernel, JIT_HERE)

// Host side, once per translation unit: JIT_MODULE(name) defines jit_set_<name> / jit_fired_<name>.
#define JIT_MODULE(name)                                                                                             \
  cudaError_t jit_set_##name(int mode, unsigned seed, int a, int b, int c) {                                         \
    const JitConfig cfg{mode, seed, a, b, c};                                                                        \
    void* p = nullptr;                                                                                               \
    cudaError_t e = cudaDeviceSynchronize();                                                                         \
    if (e == cudaSuccess) e = cudaGetSymbolAddress(&p, jit_visits);                                                  \
    if (e == cudaSuccess) e = cudaMemset(p, 0, sizeof(jit_visits));                                                  \
    if (e == cudaSuccess) e = cudaGetSymbolAddress(&p, jit_launches);                                                \
    if (e == cudaSuccess) e = cudaMemset(p, 0, sizeof(jit_launches));                                                \
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(jit_cfg, &cfg, sizeof cfg);                                         \
    if (e == cudaSuccess) e = cudaDeviceSynchronize();                                                               \
    return e;                                                                                                        \
  }                                                                                                                  \
  cudaError_t jit_fired_##name(unsigned* out) {                                                                      \
    static unsigned part[JIT_N_FILES * JIT_MAX_LINE];                                                                \
    cudaError_t e = cudaDeviceSynchronize();                                                                         \
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(part, jit_fired, sizeof part);                                    \
    if (e == cudaSuccess) for (int i = 0; i < JIT_N_FILES * JIT_MAX_LINE; ++i) out[i] += part[i];                    \
    return e;                                                                                                        \
  }
cudaError_t jit_set_engine(int, unsigned, int, int, int);
cudaError_t jit_set_fxcm(int, unsigned, int, int, int);
cudaError_t jit_set_paq8(int, unsigned, int, int, int);
cudaError_t jit_fired_engine(unsigned*);
cudaError_t jit_fired_fxcm(unsigned*);
cudaError_t jit_fired_paq8(unsigned*);

}  // namespace cmixb200

#else
#define JIT_HERE 0
#define jit_entry(kernel) ((void)0)
namespace cmixb200 {
__device__ __forceinline__ void jit_point(int) {}
}  // namespace cmixb200
#endif

namespace cmixb200 {
// The synchronisation primitives with their site. Named barriers and the mbarrier / flag helpers live beside their users.
__device__ __forceinline__ void jit_syncthreads(int site) { __syncthreads(); jit_point(site); }
template <class Cluster> __device__ __forceinline__ void jit_cluster_sync(Cluster c, int site) { c.sync(); jit_point(site); }
}  // namespace cmixb200
#define JIT_SYNCTHREADS() ::cmixb200::jit_syncthreads(JIT_HERE)
