// tools/p2p_microbench.cu — what NVLink peer memory gives a sampling kernel (design input for the frontier-sharded
// sampler, DESIGN.md §6): rate of random 8-byte loads / stores / atomicCAS / red.min on LOCAL vs PEER memory,
// coalesced peer store / load bandwidth, and the one-way latency of a flag between two GPUs.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o /tmp/p2p tools/p2p_microbench.cu && /tmp/p2p
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
typedef unsigned long long u64;
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("ERR %s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ u64 mix(u64 x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }

// mode 0 load, 1 store, 2 CAS (insert-like: expected EMPTY), 3 red.min, 4 CAS + red.min (the sampler's insert)
__global__ void k_random(u64* tab, u64* tab2, u64 mask, long n, int mode, u64* sink) {
  u64 acc = 0;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const u64 s = mix((u64)i) & mask;
    if (mode == 0) acc += tab[s];
    else if (mode == 1) tab[s] = (u64)i;
    else if (mode == 2) acc += atomicCAS(&tab[s], ~0ull, (u64)i);
    else if (mode == 3) asm volatile("red.global.min.u64 [%0], %1;" ::"l"(tab + s), "l"((u64)i) : "memory");
    else { acc += atomicCAS(&tab[s], ~0ull, (u64)i); asm volatile("red.global.min.u64 [%0], %1;" ::"l"(tab2 + s), "l"((u64)i) : "memory"); }
  }
  if (acc == 0x1234567) *sink = acc;
}
__global__ void k_copy16(const uint4* __restrict__ src, uint4* __restrict__ dst, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) dst[i] = src[i];
}
// ping-pong: `me` waits for flag value v on its own memory, then writes v+1 into the peer's flag
__global__ void k_pingpong(volatile u64* mine, volatile u64* theirs, int first, int iters, u64* t_out) {
  u64 t0, t1;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (int i = 0; i < iters; ++i) {
    if (first) { *theirs = 2 * i + 1; __threadfence_system(); while (*mine != (u64)(2 * i + 2)) {} }
    else { while (*mine != (u64)(2 * i + 1)) {} *theirs = 2 * i + 2; __threadfence_system(); }
  }
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
  *t_out = t1 - t0;
}

int main() {
  int nd = 0; CK(cudaGetDeviceCount(&nd));
  printf("devices: %d\n", nd);
  const int peer = nd > 1 ? 1 : 0;
  if (nd > 1) {
    int can = 0; CK(cudaDeviceCanAccessPeer(&can, 0, 1)); printf("can access peer 0->1: %d\n", can);
    int at = 0; cudaDeviceGetP2PAttribute(&at, cudaDevP2PAttrNativeAtomicSupported, 0, 1); printf("native atomics over the link: %d\n", at);
    CK(cudaSetDevice(0)); CK(cudaDeviceEnablePeerAccess(1, 0));
    CK(cudaSetDevice(1)); CK(cudaDeviceEnablePeerAccess(0, 0));
  }
  const u64 slots = 1ull << 25;  // 256 MB table (larger than L2)
  u64 *loc, *loc2, *rem, *rem2, *sink;
  CK(cudaSetDevice(0)); CK(cudaMalloc(&loc, slots * 8)); CK(cudaMalloc(&loc2, slots * 8)); CK(cudaMalloc(&sink, 8));
  CK(cudaSetDevice(peer)); CK(cudaMalloc(&rem, slots * 8)); CK(cudaMalloc(&rem2, slots * 8));
  CK(cudaSetDevice(0));
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const long n = 1 << 24;
  const char* names[] = {"load8", "store8", "CAS", "red.min", "CAS+red.min"};
  for (int where = 0; where < 2; ++where) {
    u64* t = where ? rem : loc; u64* t2 = where ? rem2 : loc2;
    for (int mode = 0; mode < 5; ++mode) {
      CK(cudaMemset(loc, 0xff, slots * 8)); CK(cudaMemset(loc2, 0xff, slots * 8));
      CK(cudaSetDevice(peer)); CK(cudaMemset(rem, 0xff, slots * 8)); CK(cudaMemset(rem2, 0xff, slots * 8)); CK(cudaDeviceSynchronize());
      CK(cudaSetDevice(0));
      for (int grid : {sms * 2, sms * 8}) {
        k_random<<<grid, 256>>>(t, t2, slots - 1, n / 8, mode, sink);  // warm
        CK(cudaEventRecord(e0));
        k_random<<<grid, 256>>>(t, t2, slots - 1, n, mode, sink);
        CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        printf("%-6s random %-12s grid %4d: %8.1f M ops/s (%.3f ms for %ld)\n", where ? "PEER" : "LOCAL", names[mode], grid, n / ms / 1e3, ms, n);
      }
    }
  }
  // coalesced copies: local->peer (stores over the link), peer->local (loads over the link)
  const long n16 = (long)slots / 2;  // 256 MB
  for (int dir = 0; dir < 3; ++dir) {
    const uint4* s = (const uint4*)(dir == 1 ? rem : loc); uint4* d = (uint4*)(dir == 0 ? rem2 : loc2);
    for (int grid : {sms, sms * 4, sms * 16}) {
      k_copy16<<<grid, 256>>>(s, d, n16 / 8);
      CK(cudaEventRecord(e0));
      k_copy16<<<grid, 256>>>(s, d, n16);
      CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("copy %s grid %4d: %7.1f GB/s payload\n", dir == 0 ? "local->PEER (stores)" : (dir == 1 ? "PEER->local (loads) " : "local->local        "), grid, n16 * 16.0 / ms / 1e6);
    }
  }
  if (nd > 1) {
    u64 *f0, *f1, *t0, *t1;
    CK(cudaSetDevice(0)); CK(cudaMalloc(&f0, 8)); CK(cudaMalloc(&t0, 8)); CK(cudaMemset(f0, 0, 8));
    CK(cudaSetDevice(1)); CK(cudaMalloc(&f1, 8)); CK(cudaMalloc(&t1, 8)); CK(cudaMemset(f1, 0, 8)); CK(cudaDeviceSynchronize());
    const int iters = 1000;
    CK(cudaSetDevice(1)); k_pingpong<<<1, 1>>>(f1, f0, 0, iters, t1);
    CK(cudaSetDevice(0)); k_pingpong<<<1, 1>>>(f0, f1, 1, iters, t0);
    CK(cudaDeviceSynchronize()); CK(cudaSetDevice(1)); CK(cudaDeviceSynchronize());
    u64 ns = 0; CK(cudaMemcpy(&ns, t0, 8, cudaMemcpyDeviceToHost));
    printf("flag ping-pong: %.2f us round trip (%.2f us one way)\n", ns / 1e3 / iters, ns / 2e3 / iters);
  }
  return 0;
}
