// cmix_b200/csrc/paq8_dev.cu — translation unit of the resident PAQ8 kernels (paq8.cuh) and their launchers (producers.h).
#include "paq8.cuh"
#include "producers.h"

namespace cmixb200 {

cudaError_t paq8_configure() {
  cudaError_t e = cudaFuncSetAttribute(paq8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(P8Shared));
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(paq8_bit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(P8Shared));
}
void paq8_launch_chunk(const ChunkArgs* d_args, int n_streams, cudaStream_t s) {   // a cluster of two CTAs per stream
  paq8_kernel<<<2 * n_streams, P8_THREADS, sizeof(P8Shared), s>>>(d_args);
}
void paq8_launch_bit(p8::State* g, int y, u16* ext_bit, cudaStream_t s, const u32* dbit) {
  paq8_bit_kernel<<<2, P8_THREADS, sizeof(P8Shared), s>>>(g, y, ext_bit, dbit);
}

}  // namespace cmixb200

#ifdef P8_PROF
extern "C" int cmixb200_p8_prof(unsigned long long* out, int reset) {
  cudaDeviceSynchronize();
  if (cudaMemcpyFromSymbol(out, cmixb200::g_p8_prof, sizeof(cmixb200::g_p8_prof)) != cudaSuccess) return 1;
  if (reset) { static unsigned long long z[cmixb200::P8_PROF_ROWS][cmixb200::P8_PROF_SLOTS]; cudaMemcpyToSymbol(cmixb200::g_p8_prof, z, sizeof(z)); }
  return 0;
}
#endif

