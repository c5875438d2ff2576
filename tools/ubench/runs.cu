// Microbenchmark: 10 M 8-byte stores to an 80 MB array where every `run` consecutive lanes write `run` consecutive
// slots at a random base — how much does the store rate improve when a warp instruction touches fewer sectors?
// (what sorting placement tiles by destination could buy).  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o runs runs.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>

__global__ void k(uint64_t* __restrict__ out, const uint64_t* __restrict__ src, uint32_t n, uint32_t run, uint32_t groups, uint32_t mult) {
  uint64_t pol; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t g = i / run, r = i - g * run;
    const uint32_t d = (uint32_t)(((uint64_t)g * mult) % groups) * run + r;  // bijection on groups (mult coprime)
    const uint64_t v = src[i];
    asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(out + d), "l"(v), "l"(pol) : "memory");
  }
}

int main() {
  const uint32_t n = 10000000;
  uint64_t *out, *src; void* flush; size_t fbytes = 256u << 20;
  cudaMalloc(&out, (size_t)(n + 64) * 8); cudaMalloc(&src, (size_t)n * 8); cudaMalloc(&flush, fbytes);
  cudaMemset(src, 1, (size_t)n * 8);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  const uint32_t runs[] = {1, 2, 3, 4, 5, 7, 8, 16, 32};
  for (uint32_t run : runs) {
    const uint32_t groups = n / run;
    uint32_t mult = 2654435761u % groups; while (true) { uint32_t x = mult, y = groups; while (y) { uint32_t t = x % y; x = y; y = t; } if (x == 1) break; ++mult; }
    float best = 1e9;
    for (int it = 0; it < 5; ++it) {
      cudaMemsetAsync(flush, it, fbytes);
      cudaEventRecord(a);
      k<<<148 * 8, 256>>>(out, src, groups * run, run, groups, mult);
      cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b);
      if (it > 0 && ms < best) best = ms;
    }
    printf("run %2u consecutive slots per random base: %7.1f us  %6.1f Gst/s\n", run, best * 1000.f, n / (best * 1000.f) / 1e3);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
