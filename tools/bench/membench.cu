// Latency of one "weight tile" fetch (40 KB contiguous per CTA, 10 x 16-byte loads per thread in flight) as a function of
// the footprint the tiles are drawn from: separates TLB-reach effects from L2/HBM effects on the GPU.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ uint4 ldw(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// each iteration every CTA fetches its own 40 KB tile located at (iter * step + blockIdx * 40 KB) mod footprint
__global__ void tile_latency(const unsigned char* base, size_t footprint, size_t step, int iters, long long* cycles, unsigned* sink) {
  const size_t tile = 40 * 1024;
  unsigned acc = 0;
  long long total = 0;
  for (int it = 0; it < iters; ++it) {
    size_t off = ((size_t)it * step + (size_t)blockIdx.x * tile) % (footprint - tile);
    off &= ~size_t(2559);
    const unsigned char* p = base + off + threadIdx.x * 16;
    __syncthreads();
    long long t0 = clock64();
    uint4 v[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) v[i] = ldw(p + i * 4096);
#pragma unroll
    for (int i = 0; i < 10; ++i) acc ^= v[i].x ^ v[i].y ^ v[i].z ^ v[i].w;
    __syncthreads();
    long long t1 = clock64();
    total += t1 - t0;
    // idle a little so that iterations do not overlap in the memory system
    for (int k = 0; k < 200; ++k) acc = acc * 1664525u + 1013904223u;
  }
  if (threadIdx.x == 0) cycles[blockIdx.x] = total / iters;
  if (acc == 0x12345) sink[0] = acc;
}

int main() {
  const size_t GB = 1ull << 30;
  unsigned char* buf;
  const size_t cap = 4 * GB;
  CK(cudaMalloc(&buf, cap));
  CK(cudaMemset(buf, 1, cap));
  long long* d_cycles;
  unsigned* d_sink;
  CK(cudaMalloc(&d_cycles, 132 * sizeof(long long)));
  CK(cudaMalloc(&d_sink, 4));
  struct Case { const char* name; size_t footprint, step; };
  Case cases[] = {
      {"same 6 MB every iteration (L2 + TLB warm)", 6ull << 20, 0},
      {"cycle within 64 MB (L2 warm, TLB warm)", 64ull << 20, 6ull << 20},
      {"cycle within 200 MB (L2 cold, inside 256 MB TLB reach)", 200ull << 20, 6ull << 20},
      {"cycle within 1 GB (L2 cold, TLB cold)", 1 * GB, 6ull << 20},
      {"cycle within 3.2 GB (L2 cold, TLB cold)", 3200ull << 20, 6ull << 20},
  };
  for (auto& c : cases) {
    for (int rep = 0; rep < 2; ++rep) {
      tile_latency<<<132, 256>>>(buf, c.footprint, c.step, 2000, d_cycles, d_sink);
      CK(cudaDeviceSynchronize());
    }
    std::vector<long long> h(132);
    CK(cudaMemcpy(h.data(), d_cycles, 132 * sizeof(long long), cudaMemcpyDeviceToHost));
    long long mn = 1ll << 60, mx = 0, sum = 0;
    for (auto v : h) { mn = v < mn ? v : mn; mx = v > mx ? v : mx; sum += v; }
    printf("%-58s  cycles/tile: mean %lld  min %lld  max %lld\n", c.name, sum / 132, mn, mx);
  }
  return 0;
}
