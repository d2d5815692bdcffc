// coder.cuh - the 32-bit binary arithmetic coder on the device (compress direction).
//
// Replaces Encoder::Encode / Encoder::Flush (reference src/coder/encoder.cpp:10-39) for the bulk
// path: the mix kernel leaves Predict()'s value for every bit in p_out, and this kernel, queued on
// the same CUDA stream right behind it, turns (p, bit) pairs into archive bytes without the
// probabilities ever leaving HBM. One thread per stream: the coder is a serial carry-less range
// update, ~20 integer instructions per bit, three orders of magnitude below the mixer's cost.
#ifndef CMIXB200_CODER_CUH
#define CMIXB200_CODER_CUH
#include "exact_math.h"
#include "jitter.cuh"
#include "state.h"

namespace cmixb200 {

__device__ __forceinline__ void coder_shift_out(CoderState& c) {
  while (((c.x1 ^ c.x2) & 0xff000000u) == 0) {          // encoder.cpp:25-29
    if (c.n_out < c.cap) c.out[c.n_out] = (u8)(c.x2 >> 24); else c.overflow = 1;
    ++c.n_out;
    c.x1 <<= 8;
    c.x2 = (c.x2 << 8) + 255;
  }
}

__global__ void __launch_bounds__(32, 1) encode_kernel(const ChunkArgs* __restrict__ args) { jit_entry(JK_ENCODE);
  const ChunkArgs a = args[blockIdx.x];
  if (a.coder == nullptr || threadIdx.x != 0) return;
  CoderState c = *a.coder;
  const u64 n_bits = (u64)a.n_bytes * 8;
  for (u64 t = 0; t < n_bits; ++t) {
    const int bit = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
    const u32 p = (u32)XM_FADD(1.0f, XM_FMUL(65534.0f, a.p_out[t]));    // Encoder::Discretize, encoder.cpp:10-12
    const u32 range = c.x2 - c.x1;
    const u32 xmid = c.x1 + (range >> 16) * p + (((range & 0xffffu) * p) >> 16);   // encoder.cpp:16-17
    if (bit) c.x2 = xmid; else c.x1 = xmid + 1;
    coder_shift_out(c);
  }
  *a.coder = c;
}

__global__ void encode_flush_kernel(CoderState* cs) { jit_entry(JK_ENCODE_FLUSH);                 // Encoder::Flush, encoder.cpp:32-39
  CoderState c = *cs;
  coder_shift_out(c);
  if (c.n_out < c.cap) c.out[c.n_out] = (u8)(c.x2 >> 24); else c.overflow = 1;
  ++c.n_out;
  *cs = c;
}

// One step of Decoder::Decode (reference src/coder/decoder.cpp:16-39) between the predict and the perceive kernels of a bit, on
// the device: the probability never leaves HBM and the decoded bit is handed to the perceive kernels through DecodeState.
__device__ __forceinline__ u32 decoder_read_byte(DecodeState& d) { return d.pos < d.n_arch ? d.arch[d.pos++] : 0u; }   // decoder.cpp:10-14
__global__ void decode_begin_kernel(DecodeState* ds) { jit_entry(JK_DECODE_BEGIN);                // Decoder::Decoder, decoder.cpp:3-8
  DecodeState d = *ds;
  d.x1 = 0; d.x2 = 0xffffffffu; d.x = 0; d.ctx = 1; d.t = 0; d.bit = d.full = 0;
  for (int i = 0; i < 4; ++i) d.x = (d.x << 8) + (decoder_read_byte(d) & 0xff);
  *ds = d;
}
__global__ void decode_step_kernel(const StreamState* st, DecodeState* ds) { jit_entry(JK_DECODE_STEP);
  DecodeState d = *ds;
  const u32 p = (u32)XM_FADD(1.0f, XM_FMUL(65534.0f, st->last_p));   // Decoder::Discretize, decoder.cpp:16-18
  const u32 range = d.x2 - d.x1;
  const u32 xmid = d.x1 + (range >> 16) * p + (((range & 0xffffu) * p) >> 16);
  u32 bit = 0;
  if (d.x <= xmid) { bit = 1; d.x2 = xmid; } else d.x1 = xmid + 1;
  while (((d.x1 ^ d.x2) & 0xff000000u) == 0) {
    d.x1 <<= 8;
    d.x2 = (d.x2 << 8) + 255;
    d.x = (d.x << 8) + decoder_read_byte(d);
  }
  d.bit = bit;
  d.ctx = d.ctx * 2 + bit;
  if (d.ctx >= 256) { d.full = d.ctx & 255; d.out[d.t >> 3] = (u8)d.full; d.ctx = 1; }
  d.t += 1;
  *ds = d;
}

}  // namespace cmixb200
#endif
