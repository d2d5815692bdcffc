// cmix_b200/csrc/poison.cuh — poison in front of every read the code claims comes after a write.
//
// Nearly every kernel assumes that it writes shared memory before it reads it, and the host engine allocates most device
// buffers without zeroing them and reuses its per-call scratch. On a quiet GPU a read before the write usually still finds
// what the previous launch or call left there, which is often the value expected; on a shared GPU it finds another user's
// data. Built with -DCMIXB200_POISON:
//  * every kernel's entry (jit_entry) fills this CTA's whole shared window with the pattern, skipping the region reserved
//    for the system, and then waits at a CTA barrier. A CTA fills only its own shared memory, before the kernel's first
//    cluster barrier, so no peer's DSMEM write can come before the fill;
//  * the host engine (engine.cu, PoisonFill) fills every buffer it allocates without zeroing, and refills the per-call
//    scratch at the start of each call that writes it before it reads it.
// A read before a write then sees the pattern, and the probabilities differ from the reference's (tests/test_poison.py).
// Without the flag nothing here is compiled and jit_entry expands to nothing.
//
// The pattern (cmixb200_poison_config, exported by the poison build only; default 0x7FC0A5A5) is one 32-bit word per
// 4 bytes of memory:
//   top bit clear: that word everywhere. 0x7FC0A5A5 is a quiet NaN as fp32, so a float read shows in every later
//     probability; as u32 or as either u16 half it is far above any 12-bit code, count or index; and a spin on >= passes
//     at once instead of hanging.
//   top bit set: a hash of (pattern, word index) with the top bit set: a different large value in every word, so that a
//     read that happens to be harmless for one constant is not harmless for all of them.
#pragma once

#ifdef CMIXB200_POISON
#ifdef CMIXB200_JITTER
#error "the poison and jitter builds are separate variants"
#endif
#include <cuda_runtime.h>

namespace cmixb200 {

constexpr unsigned POISON_DEFAULT = 0x7FC0A5A5u;

__host__ __device__ __forceinline__ unsigned poison_word(unsigned pattern, unsigned i) {
  if (!(pattern >> 31)) return pattern;
  unsigned h = pattern ^ (i * 0x9E3779B1u);
  h ^= h >> 16; h *= 0x7feb352du; h ^= h >> 15; h *= 0x846ca68bu; h ^= h >> 16;
  return h | 0x80000000u;
}

static __device__ unsigned poison_pattern = POISON_DEFAULT;   // one per translation unit: poison_set_<unit>

// Kernel entry: the pattern over the offsets [0, %total_smem_size) of this CTA's window but [%reserved_smem_offset_begin,
// %reserved_smem_offset_end) (static and dynamic shared memory), then a CTA barrier with the kernel's entry site.
// On sm_90 a shared::cta address carries the CTA's place in its cluster above bit 24 (the compiler forms every shared
// variable's address so), and offset 0 without it is rank 0's window: the window's base comes from the address of the
// dynamic shared memory. The fill also stops where the dynamic shared memory ends (it follows the static variables).
__device__ __forceinline__ void poison_entry(int site) {
  extern __shared__ __align__(16) unsigned char poison_dynamic[];
  unsigned total, rb, re, dyn;
  asm volatile("mov.u32 %0, %%total_smem_size;" : "=r"(total));
  asm volatile("mov.u32 %0, %%reserved_smem_offset_begin;" : "=r"(rb));
  asm volatile("mov.u32 %0, %%reserved_smem_offset_end;" : "=r"(re));
  asm volatile("mov.u32 %0, %%dynamic_smem_size;" : "=r"(dyn));
  const unsigned dyn_addr = (unsigned)__cvta_generic_to_shared(poison_dynamic);
  const unsigned base = dyn_addr & 0xFF000000u, own_end = (dyn_addr & 0x00FFFFFFu) + dyn;
  const unsigned end = total < own_end ? total : own_end;
  const unsigned pattern = poison_pattern;
  const unsigned n = blockDim.x * blockDim.y * blockDim.z;
  const unsigned tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  for (unsigned a = tid * 4; a + 4 <= end; a += n * 4)
    if (a < rb || a >= re) asm volatile("st.shared.u32 [%0], %1;" ::"r"(base + a), "r"(poison_word(pattern, a >> 2)) : "memory");
  jit_syncthreads(site);
}

// Host side, once per translation unit: POISON_MODULE(name) defines poison_set_<name>.
#define POISON_MODULE(name) \
  cudaError_t poison_set_##name(unsigned pattern) { return cudaMemcpyToSymbol(poison_pattern, &pattern, sizeof pattern); }
cudaError_t poison_set_engine(unsigned);
cudaError_t poison_set_fxcm(unsigned);
cudaError_t poison_set_paq8(unsigned);

}  // namespace cmixb200
#endif
