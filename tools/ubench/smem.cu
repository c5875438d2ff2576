// Microbenchmark: shared-memory op throughput with random (bin-like) addresses on an H100.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
__device__ __forceinline__ uint32_t mixh(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }
// MODE 0: atomicAdd no return (RED), 1: atomicAdd with return, 2: atomicExch, 3: LDS random, 4: STS random,
// 5: match_any, 6: atomicAdd no return, conflict-free (idx = lane + 32*k), 7: LDS.U16 sequential
template <int MODE>
__global__ void k(uint32_t K, uint32_t iters, uint32_t* out, unsigned long long* cyc) {
  extern __shared__ uint32_t s[];
  for (uint32_t i = threadIdx.x; i < K; i += blockDim.x) s[i] = 0;
  __syncthreads();
  uint32_t acc = 0, x = threadIdx.x * 2654435761u + blockIdx.x;
  unsigned long long t0 = clock64();
  for (uint32_t it = 0; it < iters; ++it) {
    x = x * 1664525u + 1013904223u;
    uint32_t idx = (MODE == 6) ? ((threadIdx.x & 31) + 32 * ((x >> 8) % (K / 32))) : (mixh(x) % K);
    if (MODE == 0 || MODE == 6) atomicAdd(&s[idx], 1u);
    if (MODE == 1) acc += atomicAdd(&s[idx], 1u);
    if (MODE == 2) acc += atomicExch(&s[idx], x);
    if (MODE == 3) acc += s[idx];
    if (MODE == 4) s[idx] = x;
    if (MODE == 5) acc += __match_any_sync(0xFFFFFFFFu, idx);
    if (MODE == 7) acc += reinterpret_cast<uint16_t*>(s)[(threadIdx.x + it * 7) % (2 * K)];
  }
  unsigned long long t1 = clock64();
  __syncthreads();
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
  if (acc == 0x12345) out[0] = acc + s[0];
}
template <int MODE>
void run(const char* name, int threads, int blocks_per_sm, uint32_t K) {
  unsigned long long* cyc; uint32_t* out; cudaMalloc(&cyc, 8 * 1024); cudaMalloc(&out, 64);
  const uint32_t iters = 4096;
  cudaFuncSetAttribute(k<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
  k<MODE><<<148 * blocks_per_sm, threads, K * 4>>>(K, iters, out, cyc);
  cudaDeviceSynchronize();
  unsigned long long h[1024]; cudaMemcpy(h, cyc, 8 * 148 * blocks_per_sm, cudaMemcpyDeviceToHost);
  double avg = 0; for (int i = 0; i < 148 * blocks_per_sm; ++i) avg += (double)h[i]; avg /= 148 * blocks_per_sm;
  double warp_instr_per_sm = (double)iters * (threads / 32) * blocks_per_sm;
  printf("%-34s thr=%4d x%d K=%6u: %7.2f cycles per warp-instr per SM (%.2f lanes/cycle)\n", name, threads, blocks_per_sm, K,
         avg / warp_instr_per_sm, 32.0 * warp_instr_per_sm / avg);
  cudaFree(cyc); cudaFree(out);
}
int main() {
  for (uint32_t K : {5004u, 10007u, 64u}) {
    run<0>("atomicAdd noret (RED) random", 1024, 1, K);
    run<1>("atomicAdd ret random", 1024, 1, K);
    run<2>("atomicExch random", 1024, 1, K);
    run<3>("LDS random", 1024, 1, K);
    run<4>("STS random", 1024, 1, K);
    run<6>("atomicAdd noret conflict-free", 1024, 1, K < 64 ? 64 : K);
  }
  run<5>("match_any (random 13-bit)", 1024, 1, 5004);
  run<7>("LDS.U16 sequential", 1024, 1, 5004);
  run<0>("atomicAdd noret random", 512, 2, 5004);
  run<2>("atomicExch random", 512, 2, 5004);
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
}
