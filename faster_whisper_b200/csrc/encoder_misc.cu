// Small HBM-bound encoder kernels: LayerNorm (fp32 residual stream -> fp16 GEMM operand, or e4m3 codes + row scales under
// compute_type float8_float16), the fp16 -> e4m3 row quantiser, the feature
// transpose that turns the reference's [B, n_mels, 3000] float32 hand-off (transcribe.py:1873-1876) into the
// token-major fp16 layout the implicit-GEMM conv stem reads, and dtype converters for weight upload.
#include "common.cuh"
#include "engine.h"
#include "fp8.cuh"

namespace b2w {

// one warp per row; d <= 1280 -> each lane holds up to 40 values.  Loads row `row` and leaves LayerNorm(x) * g + b (or the
// plain normalisation when g is NULL) in v: lane holds float4 chunks lane + 32 i < d / 4.
__device__ __forceinline__ void layernorm_row(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ bta,
                                              int row, int d, int lane, float4 (&v)[10]) {
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)row * d);
  const int n4 = d >> 2;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int idx = lane + 32 * i;
    if (idx < n4) {
      v[i] = xr[idx];
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
  }
  const float mean = warp_sum(s) / d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int idx = lane + 32 * i;
    if (idx < n4) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      q += a * a + b * b + c * c + e * e;
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / d + 1e-5f);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(bta);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int idx = lane + 32 * i;
    if (idx < n4) {
      float4 gg = make_float4(1.f, 1.f, 1.f, 1.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
      if (g) {
        gg = __ldg(g4 + idx);
        bb = __ldg(b4 + idx);
      }
      v[i] = make_float4((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y,
                         (v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w);
    }
  }
}

template <typename OutT>
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ bta,
                                 OutT* __restrict__ out, int rows, int d) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float4 v[10];
  layernorm_row(x, g, bta, row, d, lane, v);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int idx = lane + 32 * i;
    if (idx < (d >> 2)) {
      if constexpr (sizeof(OutT) == 2) {
        reinterpret_cast<uint2*>(out + (long long)row * d)[idx] = make_uint2(pack_half2(v[i].x, v[i].y), pack_half2(v[i].z, v[i].w));
      } else {
        reinterpret_cast<float4*>(out + (long long)row * d)[idx] = v[i];
      }
    }
  }
}

// LayerNorm straight to e4m3 codes + row scale (fp8.cuh), from the fp32 normalised values
__global__ void layernorm_e4m3_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ bta,
                                      uint8_t* __restrict__ q, float* __restrict__ scale, int rows, int d) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float4 v[10];
  layernorm_row(x, g, bta, row, d, lane, v);
  const int n4 = d >> 2;
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 10; ++i)
    if (lane + 32 * i < n4) amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
  const float s = e4m3_row_scale(warp_max(amax));
  if (lane == 0) scale[row] = s;
  uint32_t* qr = reinterpret_cast<uint32_t*>(q + (long long)row * d);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int idx = lane + 32 * i;
    if (idx < n4) qr[idx] = e4m3x4(v[i].x, v[i].y, v[i].z, v[i].w, s);
  }
}

// fp16 rows [rows][K] -> e4m3 codes + row scales, one warp per row (K a multiple of 8); the second pass re-reads the row from L1/L2
__global__ void quantize_rows_e4m3_kernel(const __half* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ scale, int rows,
                                          int K) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (long long)row * K);
  const int n8 = K >> 3;
  __half2 m2 = __float2half2_rn(0.f);
  for (int i = lane; i < n8; i += 32) {
    const uint4 u = xr[i];
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) m2 = __hmax2(m2, __habs2(h[j]));
  }
  const float s = e4m3_row_scale(warp_max(fmaxf(__low2float(m2), __high2float(m2))));
  if (lane == 0) scale[row] = s;
  uint2* qr = reinterpret_cast<uint2*>(q + (long long)row * K);
  for (int i = lane; i < n8; i += 32) {
    const uint4 u = xr[i];
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f[2 * j] = __low2float(h[j]);
      f[2 * j + 1] = __high2float(h[j]);
    }
    qr[i] = make_uint2(e4m3x4(f[0], f[1], f[2], f[3], s), e4m3x4(f[4], f[5], f[6], f[7], s));
  }
}

void layernorm_f32_e4m3(const float* x, const float* g, const float* b, uint8_t* q, float* scale, int rows, int d, cudaStream_t s) {
  B2W_CHECK(d % 4 == 0 && d <= 1280, "layernorm width");
  layernorm_e4m3_kernel<<<ceil_div(rows, 8), 256, 0, s>>>(x, g, b, q, scale, rows, d);
  B2W_LAUNCHED();
}
void quantize_rows_e4m3(const __half* x, uint8_t* q, float* scale, int rows, int K, cudaStream_t s) {
  B2W_CHECK(K % 8 == 0 && K > 0, "quantised rows must be a multiple of 8 wide");
  quantize_rows_e4m3_kernel<<<ceil_div(rows, 8), 256, 0, s>>>(x, q, scale, rows, K);
  B2W_LAUNCHED();
}

void layernorm_f32_f16(const float* x, const float* g, const float* b, __half* out, int rows, int d, cudaStream_t s) {
  B2W_CHECK(d % 4 == 0 && d <= 1280, "layernorm width");
  layernorm_kernel<__half><<<ceil_div(rows, 8), 256, 0, s>>>(x, g, b, out, rows, d);
  B2W_LAUNCHED();
}
void layernorm_f32_f32(const float* x, const float* g, const float* b, float* out, int rows, int d, cudaStream_t s) {
  B2W_CHECK(d % 4 == 0 && d <= 1280, "layernorm width");
  layernorm_kernel<float><<<ceil_div(rows, 8), 256, 0, s>>>(x, g, b, out, rows, d);
  B2W_LAUNCHED();
}

// [B][n_mels][3000] f32  ->  [B][3000][cpad] f16 (zero channel padding), via a 32x32 smem transpose
__global__ void pack_features_kernel(const float* __restrict__ in, __half* __restrict__ out, int n_mels, int cpad) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, t = t0 + tx;
    tile[i][tx] = (c < n_mels && t < 3000) ? in[((long long)b * n_mels + c) * 3000 + t] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, c = c0 + tx;
    if (t < 3000 && c < cpad) out[((long long)b * 3000 + t) * cpad + c] = __float2half_rn(tile[tx][i]);
  }
}

void pack_features(const float* feats, __half* out, int B, int n_mels, int cpad, cudaStream_t s) {
  dim3 grid(ceil_div(3000, 32), ceil_div(cpad, 32), B);
  pack_features_kernel<<<grid, dim3(32, 8), 0, s>>>(feats, out, n_mels, cpad);
  B2W_LAUNCHED();
}

__global__ void cvt_f32_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __float2half_rn(in[i]);
}
__global__ void cvt_f16_f32_kernel(const __half* __restrict__ in, float* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __half2float(in[i]);
}
void convert_f32_f16(const float* in, __half* out, int64_t n, cudaStream_t s) {
  if (n == 0) return;
  int grid = (int)(ceil_div64(n, 256) < 4096 ? ceil_div64(n, 256) : 4096);
  cvt_f32_f16_kernel<<<grid, 256, 0, s>>>(in, out, n);
  B2W_LAUNCHED();
}
void convert_f16_f32(const __half* in, float* out, int64_t n, cudaStream_t s) {
  if (n == 0) return;
  int grid = (int)(ceil_div64(n, 256) < 4096 ? ceil_div64(n, 256) : 4096);
  cvt_f16_f32_kernel<<<grid, 256, 0, s>>>(in, out, n);
  B2W_LAUNCHED();
}

}  // namespace b2w
