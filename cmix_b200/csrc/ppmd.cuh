// cmix_b200/csrc/ppmd.cuh - the PPMD byte model on the device (SURVEY §8 row a15).
//
// PPMD::ByteUpdate (reference src/models/ppmd.cpp:1328-1338): after every coded byte the model is
// updated with it and emits the distribution of the next byte, which feeds (a) the byte mixer in
// front of the LSTM (byte-mixer.cpp:15-38) and (b) layer-0 input 2076 through a ByteModel read-out
// (byte-model.cpp:8-45). The model itself (ppmd_model.h) is a sequential pointer machine: ONE lane
// per stream walks the suffix chain; the other 31 lanes of its warp only help with the 256-entry
// floor / vocabulary mask / normalisation. It is a producer like the small models: in the compress
// direction it depends on the bytes only, so it runs ahead of everything else on its own CUDA
// stream, one warp per stream, all warps of a launch group in one CTA.
#pragma once
#include "exact_math.h"
#include "jitter.cuh"
#include "ppmd_model.h"
#include "state.h"

namespace cmixb200 {

enum { PPMD_WARPS = 8 };

// probs_[i] = sqp[i]; floor 1; ByteModel::ByteUpdate zeroes symbols outside the vocabulary
// (byte-model.cpp:40-45); probs_ /= probs_.sum() with valarray::sum() adding front to back.
__device__ __forceinline__ void ppmd_emit(const PpmdModel& m, const u8* __restrict__ vocab, float* __restrict__ out,
                                          float* scratch /* shared, 256 */, int lane) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = lane + 32 * k;
    float v = __uint2float_rn(m.sqp[i]);
    if (v < 1.0f) v = 1.0f;
    if (!vocab[i]) v = 0.0f;
    scratch[i] = v;
  }
  __syncwarp();
  float sum = 0.0f;
  if (lane == 0) {
    sum = scratch[0];
#pragma unroll 8
    for (int i = 1; i < 256; ++i) sum = XM_FADD(sum, scratch[i]);
  }
  sum = __shfl_sync(0xffffffffu, sum, 0);
#pragma unroll
  for (int k = 0; k < 8; ++k) { const int i = lane + 32 * k; out[i] = XM_FDIV(scratch[i], sum); }
  __syncwarp();
}

// floor(cum * freq / total) for cum < 2^32, freq < 2^16, 0 < total < 2^16: two 32-bit divisions instead of
// one emulated 64-bit division (ConvertSQ, ppmd.cpp:1126).
__device__ __forceinline__ u32 ppmd_scale(u32 cum, u32 freq, u32 total) {
  const unsigned long long prod = (unsigned long long)cum * freq;          // < 2^48
  const u32 hi = (u32)(prod >> 16), lo = (u32)prod & 0xffffu;              // prod = hi * 2^16 + lo, hi < 2^32
  const u32 q1 = hi / total, r1 = hi - q1 * total;                         // r1 < total < 2^16
  const u32 q0 = ((r1 << 16) | lo) / total;
  return (q1 << 16) + q0;                                                  // the true quotient is < 2^32, so this wraps exactly like the reference's uint
}

// ppmd_PrepareByte + ConvertSQ (ppmd.cpp:1256-1281, 1116-1140) by a whole warp. The sequential version in
// ppmd_model.h queues one (symbol, freq, total) triple per unmasked state of every context on the suffix
// chain (the order-0 context alone has 256) and then converts the queue with one 64-bit division per entry:
// 130 k cycles per byte on one lane. Here the lanes take the states of a context side by side: the mask test,
// the sum of the unmasked frequencies (a warp reduction of integers, order-free) and the scaled probabilities
// are done in one pass, and only the escape chain (one scaling per context) stays serial. Integer arithmetic
// throughout: the result is the same sqp[256]; tests compare the device against the reference's dumps.
__device__ void ppmd_prepare_byte_warp(PpmdModel& m, int lane) {
  if (m.error) return;                       // frozen after an exhausted arena (uniform across the warp: lane 0 set it before the barrier)
  for (int i = lane; i < 256; i += 32) m.sqp[i] = 0;
  const int saved_fall = m.order_fall;
  int order_fall = saved_fall, num_masked = 0;
  const u32 esc = m.esc_count;
  u32 cum = 0xFFFFFF00u;
  u32 minc = m.max_context - PPMD_CTX_BASE;
  __syncwarp();
  {
    const PpmdCtx q = m.ctx[minc];
    const PpmdSt* p = m.pool + q.stats;
    if (q.ns) {                                                                // processSymbol1_T
      const u32 total = q.summ;
      u32 low = 0;
      for (int i0 = 0; i0 <= q.ns; i0 += 32) {
        const int i = i0 + lane;
        u32 f = 0;
        if (i <= q.ns) {
          const PpmdSt st = p[i];
          f = st.freq;
          m.sqp[st.sym] = ppmd_scale(cum, f, total) + 1;
          m.char_mask[st.sym] = esc;
        }
        low += __reduce_add_sync(0xffffffffu, f);
      }
      num_masked = q.ns;
      cum = ppmd_scale(cum, (u32)(uint16_t)(total - low), total);
    } else {                                                                   // processBinSymbol_T
      const PpmdSt st = p[0];
      const int i = m.ns2bs[m.ctx[q.suffix].ns] + m.prev_success + q.flags + ((m.run_length >> 26) & 0x20);
      const int bsumm = m.bin_summ[m.qtable[st.freq - 1]][i];
      __syncwarp();
      if (lane == 0) {
        m.bsumm = bsumm;
        m.sqp[st.sym] = ppmd_scale(cum, (u32)(uint16_t)(bsumm + bsumm), PPMD_SCALE) + 1;
        m.char_mask[st.sym] = esc;
      }
      cum = ppmd_scale(cum, (u32)(uint16_t)(PPMD_SCALE - bsumm - bsumm), PPMD_SCALE);
      num_masked = 0;
    }
  }
  __syncwarp();
  for (;;) {
    bool done = false;
    PpmdCtx q;
    do {
      const u32 suffix = m.ctx[minc].suffix;
      if (!suffix) { done = true; break; }
      order_fall++;
      minc = suffix;
      q = m.ctx[minc];
    } while (q.ns == num_masked);
    if (done) break;
    const PpmdSt* p = m.pool + q.stats;                                        // processSymbol2_T
    int see_freq;
    {
      const int cnum = q.ns;
      if (cnum != 0xFF) {
        const int col = (q.summ > 10 * (cnum + 1)) + 2 * (2 * cnum < (int)m.ctx[q.suffix].ns + num_masked) + q.flags;
        const PpmdSee se = (&m.see[m.qtable[cnum + 3] - 4][0])[col];
        see_freq = (int)(se.summ >> se.shift) + 1;
      } else see_freq = 1;
    }
    // pass 1: which states are unmasked, and the sum of their frequencies (states stay in registers)
    PpmdSt mine[8];
    u32 low = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int i = lane + 32 * k;
      mine[k].freq = 0; mine[k].sym = 0;
      if (i <= q.ns) {
        const PpmdSt st = p[i];
        if (m.char_mask[st.sym] != esc) { mine[k] = st; if (st.freq == 0) mine[k].pad = 1; else mine[k].pad = 2; }
        else mine[k].pad = 0;
      } else mine[k].pad = 0;
      low += __reduce_add_sync(0xffffffffu, mine[k].pad ? (u32)mine[k].freq : 0u);
    }
    const u32 total = (u32)(uint16_t)(see_freq + (int)low);
    // pass 2: scaled probabilities of the unmasked states, then mask them
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (mine[k].pad) {
        m.sqp[mine[k].sym] = ppmd_scale(cum, mine[k].freq, total) + 1;
        m.char_mask[mine[k].sym] = esc;
      }
    }
    cum = ppmd_scale(cum, (u32)(uint16_t)see_freq, total);
    num_masked = q.ns;
    __syncwarp();
  }
  (void)order_fall;
  if (lane == 0) { m.esc_count = esc + 1; m.num_masked = 0; m.order_fall = saved_fall; m.sq_n = 0; }
  __syncwarp();
}

__global__ void ppmd_init_kernel(PpmdModel* m) { jit_entry(JK_PPMD_INIT);
  if (threadIdx.x == 0 && blockIdx.x == 0) ppmd_init(*m);
}

// The model's registers and small tables (15 KB: symbol masks, binary-context and SEE adaptation tables, the
// symbol queue) are hit several times per visited state; in global memory every store makes the next load
// of that line an L2 round trip. Each warp therefore works on a shared-memory copy and writes it back at
// the end of the launch; only the three arenas (contexts, states, text) stay in HBM/L2.
__device__ __forceinline__ void ppmd_copy_words(void* dst, const void* src, int lane) {
  static_assert(sizeof(PpmdModel) % 4 == 0, "PpmdModel is copied in 32-bit words");
  const unsigned* s = reinterpret_cast<const unsigned*>(src);
  unsigned* d = reinterpret_cast<unsigned*>(dst);
  for (int i = lane; i < (int)(sizeof(PpmdModel) / 4); i += 32) d[i] = s[i];
  __syncwarp();
}

struct PpmdWarpShared { PpmdModel m; float scratch[256]; };

// Bulk: warp w of block b serves stream b * PPMD_WARPS + w of the launch group.
__global__ void __launch_bounds__(PPMD_WARPS * 32, 1) ppmd_kernel(const ChunkArgs* __restrict__ args_all, int n_streams) { jit_entry(JK_PPMD);
  extern __shared__ __align__(16) unsigned char ppmd_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  PpmdWarpShared& sh = reinterpret_cast<PpmdWarpShared*>(ppmd_raw)[warp];
  const int s = blockIdx.x * PPMD_WARPS + warp;
  if (s >= n_streams) return;
  const ChunkArgs a = args_all[s];
  if (a.ppmd_gen == nullptr) return;
  StreamState* st = a.st;
  ppmd_copy_words(&sh.m, st->ppmd, lane);
  const u8* vocab = st->small.vocab;
  if (lane == 0) sh.m.tprev = clock64();
  for (u32 pos = 0; pos < a.n_bytes; ++pos) {
    if (lane == 0) ppmd_update_byte(sh.m, a.bytes[pos]);
    __syncwarp();
    ppmd_prepare_byte_warp(sh.m, lane);
    if (lane == 0) PP_TICK(sh.m, 2);
    ppmd_emit(sh.m, vocab, a.ppmd_gen + (size_t)pos * 256, sh.scratch, lane);
    if (lane == 0) { PP_TICK(sh.m, 4); sh.m.prof[5] += 1; }
  }
  __syncwarp();
  ppmd_copy_words(st->ppmd, &sh.m, lane);
}

// Lock-step: one byte.
__global__ void __launch_bounds__(32, 1) ppmd_byte_kernel(StreamState* st, u32 byte, float* out, const u32* dbit = nullptr) { jit_entry(JK_PPMD_BYTE);
  if (dbit) byte = dbit[1];
  extern __shared__ __align__(16) unsigned char ppmd_raw[];
  PpmdWarpShared& sh = *reinterpret_cast<PpmdWarpShared*>(ppmd_raw);
  const int lane = threadIdx.x;
  ppmd_copy_words(&sh.m, st->ppmd, lane);
  if (lane == 0) ppmd_update_byte(sh.m, (int)byte);
  __syncwarp();
  ppmd_prepare_byte_warp(sh.m, lane);
  ppmd_emit(sh.m, st->small.vocab, out, sh.scratch, lane);
  ppmd_copy_words(st->ppmd, &sh.m, lane);
}

}  // namespace cmixb200
