// cmix_b200/csrc/fxcm_dev.cu — translation unit of the resident FXCM kernels (fxcm.cuh) and their launchers (producers.h).
#include "fxcm.cuh"
#include "producers.h"

namespace cmixb200 {

cudaError_t fxcm_configure() {
  cudaError_t e = cudaFuncSetAttribute(fxcm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FxShared));
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(fxcm_bit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FxShared));
}
void fxcm_launch_chunk(const ChunkArgs* d_args, int n_streams, cudaStream_t s) {
  fxcm_kernel<<<2 * n_streams, FX_THREADS, sizeof(FxShared), s>>>(d_args);
}
void fxcm_launch_bit(StreamState* st, fx::State* g, int y, int pretrain, u16* ext_bit, cudaStream_t s, const u32* dbit) {
  fxcm_bit_kernel<<<2, FX_THREADS, sizeof(FxShared), s>>>(st, g, y, pretrain, ext_bit, dbit);
}

#ifdef CMIXB200_JITTER
JIT_MODULE(fxcm)
#endif
#ifdef CMIXB200_CENSUS
CENSUS_MODULE(fxcm)
#endif
#ifdef CMIXB200_POISON
POISON_MODULE(fxcm)
#endif

}  // namespace cmixb200

#ifdef FX_PROF
extern "C" int cmixb200_fx_prof(unsigned long long* out, int reset) {
  cudaDeviceSynchronize();
  if (cudaMemcpyFromSymbol(out, cmixb200::g_fx_prof, sizeof(cmixb200::g_fx_prof)) != cudaSuccess) return 1;
  if (reset) { static unsigned long long z[2][24]; cudaMemcpyToSymbol(cmixb200::g_fx_prof, z, sizeof(z)); }
  return 0;
}
#endif

