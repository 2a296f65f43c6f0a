// Encoder self-attention (non-causal, T = 1500, head_dim = 64) as a flash-attention forward on Hopper wgmma.
//
// One CTA per (128-query tile, head, chunk).  A producer warp streams Q once and K/V tiles of 128 keys through a
// 2-deep TMA ring; two consumer warpgroups own 64 query rows each.  S = Q K^T is one wgmma chain (m64n128k16,
// both operands in shared memory, accumulators in registers); the online softmax runs on those registers (a row is
// spread over the four threads of a quad, so row max / row sum take two shuffles), P is rounded to fp16 in registers
// and fed straight back as the A operand of P V (m64n64k16, V consumed MN-major from the fused QKV activation layout
// — no transpose pass).  The running output is rescaled in registers before each P V chain accumulates into it.
//
// Replaces CTranslate2's batched-GEMM + softmax kernel + batched-GEMM attention (SURVEY.md §2.3 row K5)
// inside Whisper.encode (reference faster_whisper/transcribe.py:1391-1400).
#include <math.h>

#include "common.cuh"
#include "engine.h"
#include "wgmma.cuh"

namespace b2w {

constexpr int kAttnThreads = 288;         // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kTileBytes = 128 * 64 * 2;  // 16 KB: 128 rows x 64 halves, 128B-swizzled
constexpr int kKvStages = 2;

__global__ void __launch_bounds__(kAttnThreads, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tm, __half* __restrict__ out, int T, int H) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + kTileBytes;  // [stage][K|V]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kTileBytes * (1 + 2 * kKvStages));
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = kv_full + kKvStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  const int d = H * 64;
  const int n_kv = (T + 127) / 128;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < kKvStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      tma_prefetch_desc(&tm);
      mbar_expect_tx(q_full, kTileBytes);
      tma_load_3d(sQ, &tm, q_full, h * 64, q0, b);
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % kKvStages;
        mbar_wait(&kv_empty[s], ((j / kKvStages) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], 2 * kTileBytes);
        uint8_t* k_dst = sKV + s * 2 * kTileBytes;
        tma_load_3d(k_dst, &tm, &kv_full[s], d + h * 64, j * 128, b);
        tma_load_3d(k_dst + kTileBytes, &tm, &kv_full[s], 2 * d + h * 64, j * 128, b);
      }
    }
    return;
  }

  const int wg = warp >> 2, wq = warp & 3, tig = threadIdx.x & 127;
  const int g = lane >> 2, t = lane & 3;
  const float sc = 0.125f * 1.4426950408889634f;  // 1/sqrt(64) * log2(e)
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // rows g and g + 8 of this warp's 16; l: this thread's columns only
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait(q_full, 0);
  const uint64_t dq = wgmma_desc_sw128(smem_u32(sQ) + wg * (64 * 128));
  for (int j = 0; j < n_kv; ++j) {
    const int s = j % kKvStages;
    mbar_wait(&kv_full[s], (j / kKvStages) & 1);
    const uint32_t k_addr = smem_u32(sKV + s * 2 * kTileBytes);
    const uint64_t dk = wgmma_desc_sw128(k_addr);
    const uint64_t dv = wgmma_desc_sw128(k_addr + kTileBytes);
    float sacc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss_n128(sacc, dq + 2 * k, dk + 2 * k, 1);
    wgmma_commit();
    wgmma_wait<0>();
    const int kbase = j * 128 + 2 * t;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (kbase + 8 * i + (e & 1) >= T) sacc[4 * i + e] = -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], sacc[4 * i + e]);
      }
    }
    float alpha[2], m_new[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      m_new[r] = fmaxf(m_run[r], mx[r] * sc);
      alpha[r] = (m_run[r] == -INFINITY) ? 0.f : ex2_approx(m_run[r] - m_new[r]);
      m_run[r] = m_new[r];
    }
    // P as fp16 A fragments: k-step kk covers keys 16 kk .. 16 kk + 15 = accumulator column blocks 2 kk and 2 kk + 1
    uint32_t pa[8][4];
    float l_new[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float p0 = ex2_approx(sacc[4 * i + 2 * r] * sc - m_new[r]);  // masked keys: ex2(-inf) = 0
        const float p1 = ex2_approx(sacc[4 * i + 2 * r + 1] * sc - m_new[r]);
        const __half2 hh = __floats2half2_rn(p0, p1);
        // the row sum uses the rounded probabilities that the P*V product will see
        l_new[r] += __low2float(hh) + __high2float(hh);
        pa[i >> 1][(i & 1) * 2 + r] = *reinterpret_cast<const uint32_t*>(&hh);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
    l_run[0] = fmaf(l_run[0], alpha[0], l_new[0]);
    l_run[1] = fmaf(l_run[1], alpha[1], l_new[1]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_rs_n64_t(o, pa[kk], dv + kk * (2048 >> 4), 1);
    wgmma_commit();
    wgmma_wait<0>();
    if (tig == 0) mbar_arrive(&kv_empty[s]);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    const int row = q0 + wg * 64 + wq * 16 + g + 8 * r;
    if (row < T) {
      const float inv = 1.0f / l_run[r];
      __half* dst = out + ((long long)b * T + row) * d + h * 64 + 2 * t;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_half2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
    }
  }
}

static int attn_smem_bytes() { return kTileBytes * (1 + 2 * kKvStages) + 1024 + 64; }

AttnPlan attn_plan(const __half* qkv, __half* out, int B, int T, int H) {
  AttnPlan p;
  p.qkv = qkv;
  p.out = out;
  p.B = B;
  p.T = T;
  p.H = H;
  const uint64_t d3 = 3ull * H * 64;
  uint64_t dims[3] = {d3, (uint64_t)T, (uint64_t)B};
  uint64_t strides[2] = {d3 * 2, d3 * 2 * (uint64_t)T};
  uint32_t box[3] = {64, 128, 1};
  p.tm = make_tmap_f16(qkv, 3, dims, strides, box);
  return p;
}

void attn_run(const AttnPlan& p, cudaStream_t stream) {
  static unsigned long long configured = 0;
  int dev = 0;
  B2W_CUDA(cudaGetDevice(&dev));
  if (!(configured >> dev & 1)) {
    B2W_CUDA(cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem_bytes()));
    configured |= 1ull << dev;
  }
  dim3 grid(ceil_div(p.T, 128), p.H, p.B);
  attn_tc_kernel<<<grid, kAttnThreads, attn_smem_bytes(), stream>>>(p.tm, p.out, p.T, p.H);
  B2W_LAUNCHED();
}

// ---- SIMT reference (debug / bisecting only) ------------------------------------------------------------------
__global__ void attn_ref_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int T, int H) {
  extern __shared__ float sc[];  // [T] scores, then 128 scratch
  float* red = sc + T;
  const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z, d = H * 64;
  const __half* base = qkv + (long long)b * T * 3 * d;
  const __half* qp = base + (long long)t * 3 * d + h * 64;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < T; j += blockDim.x) {
    const __half* kp = base + (long long)j * 3 * d + d + h * 64;
    float s = 0.f;
    for (int e = 0; e < 64; ++e) s = fmaf(__half2float(qp[e]), __half2float(kp[e]), s);
    s *= 0.125f;
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < blockDim.x / 32; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int j = threadIdx.x; j < T; j += blockDim.x) {
    const float p = expf(sc[j] - mx);
    sc[j] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < blockDim.x / 32; ++i) sum += red[i];
  if (threadIdx.x < 64) {
    float acc = 0.f;
    for (int j = 0; j < T; ++j) acc = fmaf(sc[j], __half2float(base[(long long)j * 3 * d + 2 * d + h * 64 + threadIdx.x]), acc);
    out[((long long)b * T + t) * d + h * 64 + threadIdx.x] = __float2half_rn(acc / sum);
  }
}

void attn_ref_run(const __half* qkv, __half* out, int B, int T, int H, cudaStream_t stream) {
  dim3 grid(T, H, B);
  attn_ref_kernel<<<grid, 128, (T + 128) * sizeof(float), stream>>>(qkv, out, T, H);
  B2W_LAUNCHED();
}

}  // namespace b2w
