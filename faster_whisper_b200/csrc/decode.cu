// Decoder-step kernels: HBM-bound weight streaming for R = batch x beam <= 80 rows.
//
//  * skinny_gemm : y[R,N] = x[R,K] W[N,K]^T.  Every weight byte is read from HBM exactly once, as 16-byte
//    vectors straight into mma.sync.m16n8k16 A-fragments (the k index inside each 32-wide chunk is permuted
//    identically for both operands so no shared-memory staging or ldmatrix is needed); the R x K
//    activations are tiny and come from L1/L2.  One CTA per 16 output channels, its 8 warps split K.
//    Epilogues: fused-QKV scatter into the paged self-KV cache, bias, bias+GELU, residual add with the
//    *next* LayerNorm executed by the last CTA to finish (saves a launch per sub-layer), fp32 logits.
//  * dec_self_attn : masked attention over the paged self-KV cache through the beam ancestry table
//    (no gather-copy of the cache when beams reorder).
// Cross attention is the persistent step's task launched on its own (dstep.cu, dstep_cross_attn_launch).
//
// Together these replace the per-token body of CTranslate2's Whisper.generate loop
// (reference call sites faster_whisper/transcribe.py:222-236, 1446-1459; SURVEY.md §2.3 rows K10-K15).
#include <math.h>

#include "common.cuh"
#include "decode.h"

namespace b2w {

__device__ __forceinline__ void mma16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 ldg_stream(const void* p) {  // weights: read once, keep out of L1
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

constexpr int kGvWarps = 8;
constexpr int kGvPF = 5;  // weight chunks in flight per warp (x2 with the double buffer): K = 1280 is one round trip

// LayerNorm of all active rows by one CTA (called by the last CTA of a residual-producing GEMM).
// One warp per row, the whole row in registers: every L2 load is issued before the first use.
__device__ void cta_layernorm_rows(const float* x, const float* g, const float* b, __half* xn, int R, int d) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int n4 = d >> 2;
  for (int r = warp; r < R; r += nw) {
    const float4* xr = reinterpret_cast<const float4*>(x + (long long)r * d);
    float4 v[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const int idx = lane + 32 * i;
      v[i] = (idx < n4) ? __ldcg(xr + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i) s += v[i].x + v[i].y + v[i].z + v[i].w;
    const float mean = warp_sum(s) / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      if (lane + 32 * i < n4) {
        const float a0 = v[i].x - mean, a1 = v[i].y - mean, a2 = v[i].z - mean, a3 = v[i].w - mean;
        q += a0 * a0 + a1 * a1 + a2 * a2 + a3 * a3;
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / d + 1e-5f);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    uint2* o = reinterpret_cast<uint2*>(xn + (long long)r * d);
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const int idx = lane + 32 * i;
      if (idx < n4) {
        float4 gg = make_float4(1.f, 1.f, 1.f, 1.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
        if (g) {  // decoder LayerNorm affines are folded into the consuming weights at load time (engine.cu:fold_ln)
          gg = __ldg(g4 + idx);
          bb = __ldg(b4 + idx);
        }
        o[idx] = make_uint2(pack_half2((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y),
                            pack_half2((v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w));
      }
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(kGvWarps * 32) skinny_gemm_kernel(const GvArgs a) {
  extern __shared__ float red[];  // [warps][16][NT*8]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.x * 16;
  const int K = a.K;
  const int nchunks = K >> 5;
  float acc[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;

  const __half* w_lo = a.W + (long long)(n0 + g) * K + 8 * t;
  const __half* w_hi = w_lo + 8LL * K;
  const __half* xb = a.x + (long long)g * K + 8 * t;

  uint4 wa[kGvPF], wb[kGvPF];
  int c = warp;
#pragma unroll
  for (int i = 0; i < kGvPF; ++i) {
    const int cc = c + i * kGvWarps;
    if (cc < nchunks) {
      wa[i] = ldg_stream(w_lo + cc * 32);
      wb[i] = ldg_stream(w_hi + cc * 32);
    }
  }
  for (; c < nchunks; c += kGvPF * kGvWarps) {
    uint4 na[kGvPF], nb[kGvPF];
#pragma unroll
    for (int i = 0; i < kGvPF; ++i) {
      const int cc = c + (kGvPF + i) * kGvWarps;
      if (cc < nchunks) {
        na[i] = ldg_stream(w_lo + cc * 32);
        nb[i] = ldg_stream(w_hi + cc * 32);
      }
    }
#pragma unroll
    for (int i = 0; i < kGvPF; ++i) {
      const int cc = c + i * kGvWarps;
      if (cc < nchunks) {
        uint4 xv[NT];
#pragma unroll
        for (int j = 0; j < NT; ++j) xv[j] = *reinterpret_cast<const uint4*>(xb + (long long)j * 8 * K + cc * 32);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          mma16816(acc[j], wa[i].x, wb[i].x, wa[i].y, wb[i].y, xv[j].x, xv[j].y);
          mma16816(acc[j], wa[i].z, wb[i].z, wa[i].w, wb[i].w, xv[j].z, xv[j].w);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < kGvPF; ++i) {
      wa[i] = na[i];
      wb[i] = nb[i];
    }
  }
  // cross-warp (split-K) reduction: red[warp][ch][row]
  constexpr int RP = NT * 8;
  float* my = red + warp * 16 * RP;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    my[g * RP + j * 8 + 2 * t] = acc[j][0];
    my[g * RP + j * 8 + 2 * t + 1] = acc[j][1];
    my[(g + 8) * RP + j * 8 + 2 * t] = acc[j][2];
    my[(g + 8) * RP + j * 8 + 2 * t + 1] = acc[j][3];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 16 * RP; idx += blockDim.x) {
    const int ch = idx & 15, r = idx >> 4;  // channel fastest -> 32-byte / 64-byte output segments
    if (r >= a.R) continue;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kGvWarps; ++w) v += red[w * 16 * RP + ch * RP + r];
    const int n = n0 + ch;
    if (n >= a.N) continue;
    if (a.bias) v += __ldg(a.bias + n);
    switch (a.mode) {
      case GV_QKV: {
        const int d = a.d;
        if (n < d) {
          a.out_h[(long long)r * d + n] = __float2half_rn(v);
        } else {
          const RowInfo ri = a.rows[r];
          const int which = (n >= 2 * d) ? 1 : 0;
          const int e = n - d - which * d;
          __half* base = which ? a.vcache : a.kcache;
          base[(((long long)ri.chunk * a.n_ctx + ri.pos) * a.slots + ri.slot) * d + e] = __float2half_rn(v);
        }
        break;
      }
      case GV_F16: a.out_h[(long long)r * a.N + n] = __float2half_rn(v); break;
      case GV_GELU_F16: a.out_h[(long long)r * a.N + n] = __float2half_rn(gelu_erf(v)); break;
      case GV_RESID_LN: a.xres[(long long)r * a.N + n] += v; break;
      case GV_F32: a.out_f[(long long)r * a.ldo + n] = v; break;
    }
  }
  if (a.mode == GV_RESID_LN) {
    __shared__ int is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const int ticket = atomicAdd(a.counter, 1);
      is_last = (ticket == (int)gridDim.x - 1);
      if (is_last) *a.counter = 0;
    }
    __syncthreads();
    if (is_last) {
      __threadfence();
      cta_layernorm_rows(a.xres, a.ln_g, a.ln_b, a.xn_out, a.R, a.N);
    }
  }
}

template <int NT>
static void launch_gv(const GvArgs& a, cudaStream_t s) {
  const int smem = kGvWarps * 16 * NT * 8 * sizeof(float);
  skinny_gemm_kernel<NT><<<ceil_div(a.N, 16), kGvWarps * 32, smem, s>>>(a);
  B2W_LAUNCHED();
}

void skinny_gemm(const GvArgs& a, cudaStream_t s) {
  B2W_CHECK(a.K % 32 == 0, "skinny GEMM K must be a multiple of 32");
  B2W_CHECK(a.R >= 1 && a.R <= 80, "skinny GEMM handles 1..80 rows");
  const int nt = ceil_div(a.R, 8);
  switch (nt) {
    case 1: launch_gv<1>(a, s); break;
    case 2: launch_gv<2>(a, s); break;
    case 3: launch_gv<3>(a, s); break;
    case 4: launch_gv<4>(a, s); break;
    case 5: launch_gv<5>(a, s); break;
    case 6: launch_gv<6>(a, s); break;
    case 7:
    case 8: launch_gv<8>(a, s); break;
    default: launch_gv<10>(a, s); break;
  }
}

// ---- reference skinny GEMM (debug only): one thread per output ---------------------------------------------
__global__ void skinny_ref_kernel(const __half* __restrict__ x, const __half* __restrict__ W, const float* __restrict__ bias,
                                  float* __restrict__ y, int R, int N, int K) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (n >= N) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(__half2float(x[(long long)r * K + k]), __half2float(W[(long long)n * K + k]), acc);
  y[(long long)r * N + n] = acc + (bias ? bias[n] : 0.f);
}
void skinny_ref(const __half* x, const __half* W, const float* bias, float* y, int R, int N, int K, cudaStream_t s) {
  skinny_ref_kernel<<<dim3(ceil_div(N, 128), R), 128, 0, s>>>(x, W, bias, y, R, N, K);
  B2W_LAUNCHED();
}

// ---- token + position embedding, then LayerNorm of decoder layer 0 ----------------------------------------------
__global__ void embed_ln_kernel(const int* __restrict__ tokens, const RowInfo* __restrict__ rows, const __half* __restrict__ tok_emb,
                                const float* __restrict__ pos_emb, const float* __restrict__ g, const float* __restrict__ b,
                                float* __restrict__ x, __half* __restrict__ xn, int d, int n_vocab) {
  __shared__ float red[32];
  const int r = blockIdx.x;
  int tok = tokens[r];
  tok = tok < 0 ? 0 : (tok >= n_vocab ? n_vocab - 1 : tok);
  const int pos = rows[r].pos;
  float v[5];
  float s = 0.f;
  int cnt = 0;
  for (int i = threadIdx.x; i < d; i += blockDim.x, ++cnt) {
    v[cnt] = __half2float(tok_emb[(long long)tok * d + i]) + pos_emb[(long long)pos * d + i];
    s += v[cnt];
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  const float mean = tot / d;
  __syncthreads();
  float q = 0.f;
  for (int i = 0; i < cnt; ++i) q += (v[i] - mean) * (v[i] - mean);
  q = warp_sum(q);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
  __syncthreads();
  tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  const float rstd = rsqrtf(tot / d + 1e-5f);
  cnt = 0;
  for (int i = threadIdx.x; i < d; i += blockDim.x, ++cnt) {
    x[(long long)r * d + i] = v[cnt];
    xn[(long long)r * d + i] = __float2half_rn(g ? (v[cnt] - mean) * rstd * g[i] + b[i] : (v[cnt] - mean) * rstd);
  }
}

void embed_ln(const int* tokens, const RowInfo* rows, const __half* tok_emb, const float* pos_emb, const float* g,
              const float* b, float* x, __half* xn, int R, int d, int n_vocab, cudaStream_t s) {
  B2W_CHECK(d <= 5 * 256, "embedding width");
  embed_ln_kernel<<<R, 256, 0, s>>>(tokens, rows, tok_emb, pos_emb, g, b, x, xn, d, n_vocab);
  B2W_LAUNCHED();
}

// ---- masked self-attention over the paged cache --------------------------------------------------------------------
// cache layout per layer: [chunk][pos][slot][d]; key j of row (chunk, slot, pos) lives in slot anc[chunk][slot][j] (j < pos)
// or in the row's own slot (j == pos).
__global__ void __launch_bounds__(128) dec_self_attn_kernel(const SelfAttnArgs a) {
  __shared__ float sc[B2W_MAX_TEXT_CTX];
  __shared__ float red[8];
  __shared__ float oacc[2][64];
  const int h = blockIdx.x, r = blockIdx.y;
  const RowInfo ri = a.rows[r];
  const int d = a.d, nk = ri.pos + 1;
  const int tid = threadIdx.x;
  const int cur = ri.pos & 1;
  const uint8_t* anc = a.anc + cur * a.anc_buf_stride + ((long long)ri.chunk * a.slots + ri.slot) * a.n_ctx;
  // q in registers (64 halves)
  uint4 qv[8];
  const uint4* qp = reinterpret_cast<const uint4*>(a.q + (long long)r * d + h * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) qv[i] = qp[i];
  float mx = -INFINITY;
  for (int j = tid; j < nk; j += 128) {
    const int slot = (j == ri.pos) ? ri.slot : anc[j];
    const uint4* kp = reinterpret_cast<const uint4*>(a.kcache + (((long long)ri.chunk * a.n_ctx + j) * a.slots + slot) * d + h * 64);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 kv = kp[i];
      const __half2* k2 = reinterpret_cast<const __half2*>(&kv);
      const __half2* q2 = reinterpret_cast<const __half2*>(&qv[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 kf = __half22float2(k2[e]), qf = __half22float2(q2[e]);
        s = fmaf(kf.x, qf.x, s);
        s = fmaf(kf.y, qf.y, s);
      }
    }
    s *= 0.125f;
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  float sum = 0.f;
  for (int j = tid; j < nk; j += 128) {
    const float p = __expf(sc[j] - mx);
    sc[j] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  __syncthreads();
  if ((tid & 31) == 0) red[4 + (tid >> 5)] = sum;
  __syncthreads();
  sum = red[4] + red[5] + red[6] + red[7];
  const int e = tid & 63, half = tid >> 6;
  float acc = 0.f;
  for (int j = half; j < nk; j += 2) {
    const int slot = (j == ri.pos) ? ri.slot : anc[j];
    acc = fmaf(sc[j], __half2float(a.vcache[(((long long)ri.chunk * a.n_ctx + j) * a.slots + slot) * d + h * 64 + e]), acc);
  }
  oacc[half][e] = acc;
  __syncthreads();
  if (tid < 64) a.out[(long long)r * d + h * 64 + tid] = __float2half_rn((oacc[0][tid] + oacc[1][tid]) / sum);
}

void dec_self_attn(const SelfAttnArgs& a, int R, int H, cudaStream_t s) {
  dec_self_attn_kernel<<<dim3(H, R), 128, 0, s>>>(a);
  B2W_LAUNCHED();
}

}  // namespace b2w
