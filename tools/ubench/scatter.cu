// Microbenchmark: what limits random small stores / loads on an H100?
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scatter scatter.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>

__device__ __forceinline__ uint32_t mixh(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }

// mode 0: st 8B; 1: st 4B; 2: st 16B; 3: st 8B evict_last hint; 4: ld 8B gather (sum); 5: st 8B .cg; 6: red.add u32
// 7: st 8B, destination = bijective permutation (each slot written once), 8: 32B (2x16B) per element
template <int MODE>
__global__ void k(uint64_t* __restrict__ out, const uint64_t* __restrict__ src, uint32_t n, uint32_t slots, uint32_t mult, uint64_t* sink) {
  uint64_t pol; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  uint64_t acc = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    uint32_t d = (MODE == 7) ? (uint32_t)(((uint64_t)i * mult) % slots) : mixh(i) % slots;
    uint64_t v = src[i];
    if (MODE == 0 || MODE == 7) out[d] = v;
    if (MODE == 1) reinterpret_cast<uint32_t*>(out)[d] = (uint32_t)v;
    if (MODE == 2) reinterpret_cast<ulonglong2*>(out)[d] = make_ulonglong2(v, v);
    if (MODE == 3) asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(out + d), "l"(v), "l"(pol) : "memory");
    if (MODE == 4) acc += out[d] + v;
    if (MODE == 5) __stcg(out + d, v);
    if (MODE == 6) atomicAdd(reinterpret_cast<unsigned int*>(out) + d, (unsigned int)v);
    if (MODE == 8) { reinterpret_cast<ulonglong2*>(out)[2 * d] = make_ulonglong2(v, v); reinterpret_cast<ulonglong2*>(out)[2 * d + 1] = make_ulonglong2(v, v); }
  }
  if (MODE == 4 && acc == 0x1234567) *sink = acc;
}

template <int MODE>
float run(uint64_t* out, const uint64_t* src, uint32_t n, uint32_t slots, uint64_t* sink, void* flush, size_t fbytes) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  float best = 1e9;
  for (int it = 0; it < 5; ++it) {
    cudaMemsetAsync(flush, it, fbytes);
    cudaEventRecord(a);
    k<MODE><<<148 * 8, 256>>>(out, src, n, slots, 2654435761u, sink);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (it > 0 && ms < best) best = ms;
  }
  return best * 1000.f;
}

int main() {
  const uint32_t n = 10000000;
  uint64_t *out, *src, *sink; void* flush; size_t fbytes = 256u << 20;
  cudaMalloc(&out, (size_t)n * 64); cudaMalloc(&src, (size_t)n * 8); cudaMalloc(&sink, 8); cudaMalloc(&flush, fbytes);
  cudaMemset(src, 1, (size_t)n * 8); cudaMemset(out, 0, (size_t)n * 64);
  const char* names[] = {"st8", "st4", "st16", "st8 evict_last", "ld8 gather", "st8 .cg", "red.add.u32", "st8 permutation", "st32"};
  uint32_t slotss[] = {10000000u, 2500000u, 1000000u, 250000u};
  for (uint32_t slots : slotss) {
    printf("--- %u elements into %u slots (8B-slot footprint %.1f MB)\n", n, slots, slots * 8 / 1e6);
    float t;
    t = run<0>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[0], t, n / t / 1e3);
    t = run<1>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[1], t, n / t / 1e3);
    t = run<2>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[2], t, n / t / 1e3);
    t = run<8>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[8], t, n / t / 1e3);
    t = run<3>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[3], t, n / t / 1e3);
    t = run<5>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[5], t, n / t / 1e3);
    t = run<6>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[6], t, n / t / 1e3);
    t = run<4>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[4], t, n / t / 1e3);
    if (slots == n) { t = run<7>(out, src, n, slots, sink, flush, fbytes); printf("%-18s %8.1f us  %6.1f Gst/s\n", names[7], t, n / t / 1e3); }
  }
  // coalesced reference: copy 80 MB
  {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    cudaMemsetAsync(flush, 3, fbytes); cudaEventRecord(a); cudaMemcpyAsync(out, src, (size_t)n * 8, cudaMemcpyDeviceToDevice); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b); printf("memcpy 80MB d2d: %.1f us\n", ms * 1000);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
