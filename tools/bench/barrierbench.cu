// Floor of one dependent "phase" on the GPU: all CTAs publish a little data, grid barrier, all CTAs read what the others wrote.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void grid_barrier(unsigned* bar, unsigned& epoch) {
  __syncthreads();
  epoch += gridDim.x;
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    while (ld_acquire(bar) < epoch) {}
    __threadfence();
  }
  __syncthreads();
}

// mode 0: barrier only; 1: + read 12.8 KB written by others (fp32 row slices), 2: + RMW epilogue (ld.cg + st.cg), 3: atomics epilogue
__global__ void phase_floor(float* data, unsigned* bar, int iters, int mode, long long* out) {
  unsigned epoch = 0;
  __shared__ float sink[256];
  long long t_bar = 0, t_read = 0, t_epi = 0;
  for (int it = 0; it < iters; ++it) {
    long long t0 = clock64();
    grid_barrier(bar, epoch);
    long long t1 = clock64();
    float acc = 0.f;
    if (mode >= 1) {
      // 5 rows x 1280 floats = 6400 floats: 25 per thread, batched
      float4 v[7];
#pragma unroll
      for (int i = 0; i < 7; ++i) {
        const int idx = threadIdx.x + i * 256;
        v[i] = idx < 1600 ? __ldcg(reinterpret_cast<const float4*>(data) + idx) : make_float4(0, 0, 0, 0);
      }
#pragma unroll
      for (int i = 0; i < 7; ++i) acc += v[i].x + v[i].y + v[i].z + v[i].w;
      sink[threadIdx.x] = acc;
      __syncthreads();
    }
    long long t2 = clock64();
    if (threadIdx.x < 80 && blockIdx.x < 80) {  // 80 CTAs x 16 channels x 5 rows
      float* px = data + (threadIdx.x / 16) * 1280 + blockIdx.x * 16 + (threadIdx.x & 15);
      if (mode == 2) __stcg(px, __ldcg(px) + sink[threadIdx.x] * 1e-9f + 1.f);
      else if (mode == 3) atomicAdd(px, 1.f + sink[threadIdx.x] * 1e-9f);
      else if (mode == 1) __stcg(px, 1.f + sink[threadIdx.x] * 1e-9f);
    }
    __syncthreads();
    long long t3 = clock64();
    t_bar += t1 - t0; t_read += t2 - t1; t_epi += t3 - t2;
  }
  if (threadIdx.x == 0) { out[blockIdx.x * 3] = t_bar / iters; out[blockIdx.x * 3 + 1] = t_read / iters; out[blockIdx.x * 3 + 2] = t_epi / iters; }
}

int main() {
  float* data; unsigned* bar; long long* out;
  CK(cudaMalloc(&data, 1 << 20)); CK(cudaMemset(data, 0, 1 << 20));
  CK(cudaMalloc(&bar, 4)); CK(cudaMalloc(&out, 132 * 3 * 8));
  for (int grid : {132, 66, 16}) {
    for (int mode = 0; mode < 4; ++mode) {
      CK(cudaMemset(bar, 0, 4));
      int iters = 2000;
      void* args[] = {&data, &bar, &iters, &mode, &out};
      CK(cudaLaunchCooperativeKernel((void*)phase_floor, dim3(grid), dim3(256), args, 0, 0));
      CK(cudaDeviceSynchronize());
      std::vector<long long> h(132 * 3);
      CK(cudaMemcpy(h.data(), out, grid * 3 * 8, cudaMemcpyDeviceToHost));
      double b = 0, r = 0, e = 0;
      for (int i = 0; i < grid; ++i) { b += h[i * 3]; r += h[i * 3 + 1]; e += h[i * 3 + 2]; }
      printf("grid %3d mode %d: barrier %6.0f  read %6.0f  epilogue %6.0f cycles (mean over CTAs)  -> %.2f us/phase @1.9GHz\n", grid, mode, b / grid,
             r / grid, e / grid, (b + r + e) / grid / 1900.0);
    }
  }
  return 0;
}
