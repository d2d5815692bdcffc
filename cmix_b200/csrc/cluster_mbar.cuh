// cmix_b200/csrc/cluster_mbar.cuh — the mbarriers of a handover ring between the two CTAs of a cluster (paq8.cuh, fxcm.cuh).
//
// A ring lives in the consumer CTA's shared memory. The producer writes a slot over distributed shared memory and arrives
// on the slot's *full* barrier there; the consumer arrives on the slot's *empty* barrier in the producer CTA once it is
// done with the slot. An arrive on the other CTA's barrier releases at cluster scope what the arriving thread wrote or
// read before it; a wait acquires it.
#pragma once
#include "jitter.cuh"

namespace cmixb200 {

__device__ __forceinline__ unsigned mbar_smem(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar_smem(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_remote(unsigned long long* b, int rank, int site) {
  jit_point(site);
  unsigned r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(mbar_smem(b)), "r"(rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(r) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned parity, int site) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "MBW: mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra MBW;\n\t}" ::"r"(mbar_smem(b)), "r"(parity) : "memory");
  jit_point(site);
}

}  // namespace cmixb200
