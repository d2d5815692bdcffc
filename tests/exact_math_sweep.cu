// tests/exact_math_sweep.cu — the device build of cmix_b200/csrc/exact_math.h for tests/test_exact_math_device.py,
// compiled with the product's nvcc flags (cmix_b200.capi.NVCC_COMPILE) into a small shared library.
#include <cuda_runtime.h>
#include <stddef.h>

#include "exact_math_sweep.h"

enum { XS_THREADS = 256 };

// One CTA per block of 2^16 inputs: out[b * XS_FUNCS + f] as xs_host_sums.
__global__ void __launch_bounds__(XS_THREADS) xs_sums_kernel(uint32_t first_blk, unsigned long long* out) {
  __shared__ unsigned long long part[XS_THREADS / 32][XS_FUNCS];
  const uint32_t base = (first_blk + blockIdx.x) << XS_SUB_LOG2;
  unsigned long long acc[XS_FUNCS] = {0, 0, 0, 0};
  for (uint32_t i = threadIdx.x; i < (1u << XS_SUB_LOG2); i += XS_THREADS)
#pragma unroll
    for (int f = 0; f < XS_FUNCS; ++f) acc[f] += xs_hash(base | i, xs_eval(base | i, f));
#pragma unroll
  for (int f = 0; f < XS_FUNCS; ++f) {
    for (int o = 16; o > 0; o >>= 1) acc[f] += __shfl_down_sync(0xffffffffu, acc[f], o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5][f] = acc[f];
  }
  __syncthreads();
  if (threadIdx.x < XS_FUNCS) {
    unsigned long long s = 0;
    for (int w = 0; w < XS_THREADS / 32; ++w) s += part[w][threadIdx.x];
    out[(size_t)blockIdx.x * XS_FUNCS + threadIdx.x] = s;
  }
}

__global__ void xs_eval_kernel(const uint32_t* in, size_t n, uint32_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    for (int f = 0; f < XS_FUNCS; ++f) out[f * n + i] = xs_eval(in[i], f);
}

// Host-buffer launchers; each returns the CUDA error code (0 = success).
extern "C" int xs_device_sums(uint32_t first_blk, uint32_t n_blk, unsigned long long* out) {
  unsigned long long* d = nullptr;
  cudaError_t e = cudaMalloc(&d, (size_t)n_blk * XS_FUNCS * sizeof *d);
  if (e != cudaSuccess) return (int)e;
  xs_sums_kernel<<<n_blk, XS_THREADS>>>(first_blk, d);
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(out, d, (size_t)n_blk * XS_FUNCS * sizeof *d, cudaMemcpyDeviceToHost);
  cudaFree(d);
  return (int)e;
}

extern "C" int xs_device_eval(const uint32_t* in, size_t n, uint32_t* out) {
  if (n == 0) return 0;
  uint32_t *d_in = nullptr, *d_out = nullptr;
  cudaError_t e = cudaMalloc(&d_in, n * sizeof *d_in);
  if (e == cudaSuccess) e = cudaMalloc(&d_out, n * XS_FUNCS * sizeof *d_out);
  if (e == cudaSuccess) e = cudaMemcpy(d_in, in, n * sizeof *d_in, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    xs_eval_kernel<<<(unsigned)((n + 255) / 256), 256>>>(d_in, n, d_out);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out, d_out, n * XS_FUNCS * sizeof *d_out, cudaMemcpyDeviceToHost);
  cudaFree(d_in);
  cudaFree(d_out);
  return (int)e;
}
