// Dense GEMM C[M,N] = epilogue(A[M,K] * W[N,K]^T) for the Whisper encoder, the conv stem (implicit GEMM with
// K-block -> tap mapping done by TMA coordinates) and the cross-KV projection.
//
// sm_90a: operands move HBM -> shared memory with TMA (128-byte swizzle, 64-wide K blocks) through a ring of stages fed by
// one producer warp; two consumer warpgroups each own 64 rows of the 128-row tile and run the product on the Hopper tensor
// cores with wgmma.mma_async (m64 x {32,128} x k16, fp16 in, fp32 accumulators in registers), one wgmma group in flight while
// the stage of the previous one is handed back to the producer.  The bias / GELU / residual / position-add /
// layout-scatter epilogues are fused: each warpgroup passes its accumulators through a small shared-memory tile so that
// a thread stores 32 consecutive columns of one row.  Persistent CTAs, one per SM, static tile scheduler.
//
// Replaces what CTranslate2 does with cuBLAS GEMM + cuDNN conv + separate bias/GELU/add kernels
// (SURVEY.md §2.3 rows K1-K9) behind Whisper.encode (reference faster_whisper/transcribe.py:1391-1400).
#include "common.cuh"
#include "engine.h"
#include "wgmma.cuh"

namespace b2w {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kGemmThreads = 288;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer

struct GemmDev {
  int batch, tiles_m, tiles_n, num_kb, kb_per_tap;
  int tap_row[3], tap_col[3];
  int rows, N;
  const float* bias;
  void* out;
  long long out_ld, out_batch_stride;
  const float* resid;
  const float* pos;
  int xkv_d, xkv_heads, xkv_T, xkv_B;
  const int4* rowinfo;
  __half* kcache;
  __half* vcache;
  int qkv_d, n_ctx, slots;
};

template <int EPI>
__device__ __forceinline__ void epilogue_store(const GemmDev& p, int b, int row, int n0, const float* vin) {
  float v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = vin[i];
  if (p.bias) {
    const float4* b4 = reinterpret_cast<const float4*>(p.bias + n0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 t = __ldg(b4 + i);
      v[4 * i] += t.x;
      v[4 * i + 1] += t.y;
      v[4 * i + 2] += t.z;
      v[4 * i + 3] += t.w;
    }
  }
  if constexpr (EPI == EPI_GELU_F16 || EPI == EPI_GELU_POS_F32) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
  }
  if constexpr (EPI == EPI_F16 || EPI == EPI_GELU_F16) {
    __half* o = reinterpret_cast<__half*>(p.out) + (long long)b * p.out_batch_stride + (long long)row * p.out_ld + n0;
    uint4* o4 = reinterpret_cast<uint4*>(o);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      o4[i] = make_uint4(pack_half2(v[8 * i], v[8 * i + 1]), pack_half2(v[8 * i + 2], v[8 * i + 3]),
                         pack_half2(v[8 * i + 4], v[8 * i + 5]), pack_half2(v[8 * i + 6], v[8 * i + 7]));
  } else if constexpr (EPI == EPI_QKV_CACHE) {
    const int d = p.qkv_d;
    __half* dst;
    if (n0 < d) {
      dst = reinterpret_cast<__half*>(p.out) + (long long)row * d + n0;
    } else {
      const int4 ri = __ldg(p.rowinfo + row);  // (chunk, slot, pos, -)
      const int which = n0 >= 2 * d ? 1 : 0;
      dst = (which ? p.vcache : p.kcache) + (((long long)ri.x * p.n_ctx + ri.z) * p.slots + ri.y) * d + (n0 - d - which * d);
    }
    uint4* o4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      o4[i] = make_uint4(pack_half2(v[8 * i], v[8 * i + 1]), pack_half2(v[8 * i + 2], v[8 * i + 3]),
                         pack_half2(v[8 * i + 4], v[8 * i + 5]), pack_half2(v[8 * i + 6], v[8 * i + 7]));
  } else if constexpr (EPI == EPI_F16_XKV) {
    // column n -> (layer, k|v, head, e); destination [l][kv][b][h][t][64]
    const int two_d = 2 * p.xkv_d;
    const int l = n0 / two_d, rem = n0 - l * two_d;
    const int kv = rem / p.xkv_d, c = rem - kv * p.xkv_d;
    const int h = c >> 6, e = c & 63;
    // a (t, head) row is 128 bytes = eight 16-byte chunks stored at chunk ^ (t & 7): the decode kernels copy K/V tiles
    // to shared memory verbatim and read them bank-conflict-free (dstep.cu, decode.cu)
    long long idx = ((((long long)(l * 2 + kv) * p.xkv_B + b) * p.xkv_heads + h) * p.xkv_T + row) * 64;
    uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.out) + idx);
    const int cb = e >> 3, sw = row & 7;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      o4[(cb + i) ^ sw] = make_uint4(pack_half2(v[8 * i], v[8 * i + 1]), pack_half2(v[8 * i + 2], v[8 * i + 3]),
                         pack_half2(v[8 * i + 4], v[8 * i + 5]), pack_half2(v[8 * i + 6], v[8 * i + 7]));
  } else {
    const long long idx = (long long)b * p.out_batch_stride + (long long)row * p.out_ld + n0;
    float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + idx);
    if constexpr (EPI == EPI_RESID_F32) {
      const float4* r4 = reinterpret_cast<const float4*>(p.resid + idx);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 t = r4[i];
        o4[i] = make_float4(t.x + v[4 * i], t.y + v[4 * i + 1], t.z + v[4 * i + 2], t.w + v[4 * i + 3]);
      }
    } else if constexpr (EPI == EPI_GELU_POS_F32) {
      const float4* q4 = reinterpret_cast<const float4*>(p.pos + (long long)row * p.N + n0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 t = __ldg(q4 + i);
        o4[i] = make_float4(t.x + v[4 * i], t.y + v[4 * i + 1], t.z + v[4 * i + 2], t.w + v[4 * i + 3]);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) o4[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    }
  }
}

template <int BN>
struct GemmCfg {
  static constexpr int STAGES = BN == 128 ? 6 : 8;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EC = BN < 64 ? BN : 64;  // epilogue columns per pass through shared memory
  static constexpr int EC4 = EC / 4;          // 16-byte chunks per epilogue row, stored at chunk ^ (row % EC4) (no bank conflicts)
  static constexpr int EPI_BYTES = 2 * 64 * EC * 4;
  static constexpr int SMEM = STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmDev p) {
  using C = GemmCfg<BN>;
  constexpr int STAGES = C::STAGES, A_BYTES = C::A_BYTES, STAGE_BYTES = C::STAGE_BYTES, EC = C::EC, EC4 = C::EC4;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* epi = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + C::EPI_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int total_tiles = p.batch * p.tiles_m * p.tiles_n;  // tile = (b * tiles_m + m) * tiles_n + n

  if (warp == 8) {
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_idx = tile % p.tiles_n;
        const int rest = tile / p.tiles_n;
        const int m_idx = rest % p.tiles_m, b = rest / p.tiles_m;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], STAGE_BYTES);
          const int tap = kb / p.kb_per_tap, kc = kb - tap * p.kb_per_tap;
          uint8_t* sa = smem + stage * STAGE_BYTES;
          tma_load_3d(sa, &tmA, &full[stage], p.tap_col[tap] + kc * BK, m_idx * BM + p.tap_row[tap], b);
          tma_load_2d(sa + A_BYTES, &tmB, &full[stage], kb * BK, n_idx * BN);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2, wq = warp & 3, tig = threadIdx.x & 127;
  const int g = lane >> 2, t = lane & 3;
  float* my_epi = epi + wg * 64 * EC;
  const uint32_t bar_id = 1 + wg;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int n_idx = tile % p.tiles_n;
    const int rest = tile / p.tiles_n;
    const int m_idx = rest % p.tiles_m, b = rest / p.tiles_m;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < p.num_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
      const uint64_t da = wgmma_desc_sw128(sa + wg * (64 * 128));
      const uint64_t db = wgmma_desc_sw128(sa + A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) wgmma_ss<BN>(acc, da + 2 * k, db + 2 * k, 1);
      wgmma_commit();
      wgmma_wait<1>();  // the previous stage's products are done: hand its slot back
      if (prev >= 0 && tig == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    if (prev >= 0 && tig == 0) mbar_arrive(&empty[prev]);

    const int row_l = tig & 63, half = tig >> 6;
    const int row = m_idx * BM + wg * 64 + row_l;
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += EC) {
#pragma unroll
      for (int i = c0 / 8; i < (c0 + EC) / 8; ++i) {
        const int col = 8 * i + 2 * t - c0, r = 16 * wq + g;
        const int c4 = col >> 2, cw = col & 3;
        *reinterpret_cast<float2*>(my_epi + r * EC + ((c4 ^ (r % EC4)) << 2) + cw) = make_float2(acc[4 * i], acc[4 * i + 1]);
        *reinterpret_cast<float2*>(my_epi + (r + 8) * EC + ((c4 ^ ((r + 8) % EC4)) << 2) + cw) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
      }
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
      const int n0 = n_idx * BN + c0 + half * 32;
      if (half * 32 < EC && row < p.rows && n0 < p.N) {
        float v[32];
        const float4* src = reinterpret_cast<const float4*>(my_epi + row_l * EC);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 f = src[(half * 8 + i) ^ (row_l % EC4)];
          v[4 * i] = f.x;
          v[4 * i + 1] = f.y;
          v[4 * i + 2] = f.z;
          v[4 * i + 3] = f.w;
        }
        epilogue_store<EPI>(p, b, row, n0, v);
      }
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
    }
  }
}

template <int BN>
static int gemm_smem_bytes() {
  return GemmCfg<BN>::SMEM;
}

GemmPlan gemm_plan(const GemmArgs& a, int num_sms) {
  B2W_CHECK(a.k_per_tap % BK == 0 && a.k_per_tap > 0, "GEMM K per tap must be a multiple of 64");
  B2W_CHECK(a.N % 32 == 0, "GEMM N must be a multiple of 32");
  B2W_CHECK(a.taps >= 1 && a.taps <= 3, "1..3 taps");
  GemmPlan p;
  p.a = a;
  const int K = a.taps * a.k_per_tap;
  p.tiles_m = ceil_div(a.rows, BM);
  // 128 x 128 tiles: a 256-wide tile needs 128 accumulator registers per consumer thread, more than the 168 a 288-thread CTA may
  // hold next to the epilogue
  p.block_n = 128;
  // few rows (one M tile): a 128-wide tiling leaves most SMs without work while the weights stream through N/128 CTAs
  if (a.narrow_tiles && a.a_batch * p.tiles_m == 1 && ceil_div(a.N, 128) * 2 <= num_sms) p.block_n = 32;
  p.tiles_n = ceil_div(a.N, p.block_n);
  p.num_kb = K / BK;
  long long total = (long long)a.a_batch * p.tiles_m * p.tiles_n;
  p.grid = (int)(total < num_sms ? total : num_sms);
  {
    uint64_t dims[3] = {(uint64_t)a.a_cols, (uint64_t)a.a_rows, (uint64_t)a.a_batch};
    uint64_t strides[2] = {(uint64_t)a.a_row_stride * 2, (uint64_t)(a.a_batch > 1 ? a.a_batch_stride : a.a_row_stride * a.a_rows) * 2};
    uint32_t box[3] = {BK, BM, 1};
    p.tmA = make_tmap_f16(a.A, 3, dims, strides, box);
  }
  {
    uint64_t dims[2] = {(uint64_t)K, (uint64_t)a.N};
    uint64_t strides[1] = {(uint64_t)K * 2};
    uint32_t box[2] = {BK, (uint32_t)p.block_n};
    p.tmB = make_tmap_f16(a.W, 2, dims, strides, box);
  }
  return p;
}

template <int BN, int EPI>
static void launch_tc(const GemmPlan& pl, const GemmDev& d, cudaStream_t stream) {
  gemm_tc_kernel<BN, EPI><<<pl.grid, kGemmThreads, gemm_smem_bytes<BN>(), stream>>>(pl.tmA, pl.tmB, d);
  B2W_LAUNCHED();
}

template <int BN, int EPI>
static void configure_one() {
  B2W_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, gemm_smem_bytes<BN>()));
}
template <int BN>
static void configure_bn() {
  configure_one<BN, EPI_F16>();
  configure_one<BN, EPI_GELU_F16>();
  configure_one<BN, EPI_RESID_F32>();
  configure_one<BN, EPI_GELU_POS_F32>();
  configure_one<BN, EPI_F16_XKV>();
  configure_one<BN, EPI_F32>();
  configure_one<BN, EPI_QKV_CACHE>();
}
template <int EPI>
static void configure_fp8();
void gemm_configure() {
  configure_bn<32>();
  configure_bn<128>();
  configure_fp8<EPI_F16>();
  configure_fp8<EPI_GELU_F16>();
  configure_fp8<EPI_RESID_F32>();
}

template <int BN>
static void dispatch_epi(const GemmPlan& pl, const GemmDev& d, cudaStream_t s) {
  switch (pl.a.epilogue) {
    case EPI_F16: launch_tc<BN, EPI_F16>(pl, d, s); break;
    case EPI_GELU_F16: launch_tc<BN, EPI_GELU_F16>(pl, d, s); break;
    case EPI_RESID_F32: launch_tc<BN, EPI_RESID_F32>(pl, d, s); break;
    case EPI_GELU_POS_F32: launch_tc<BN, EPI_GELU_POS_F32>(pl, d, s); break;
    case EPI_F16_XKV: launch_tc<BN, EPI_F16_XKV>(pl, d, s); break;
    case EPI_F32: launch_tc<BN, EPI_F32>(pl, d, s); break;
    case EPI_QKV_CACHE: launch_tc<BN, EPI_QKV_CACHE>(pl, d, s); break;
    default: throw Error("unknown GEMM epilogue");
  }
}

static GemmDev make_dev(const GemmArgs& a, int tiles_m, int tiles_n, int num_kb) {
  GemmDev d{};
  d.batch = a.a_batch;
  d.tiles_m = tiles_m;
  d.tiles_n = tiles_n;
  d.num_kb = num_kb;
  d.kb_per_tap = a.k_per_tap / BK;
  for (int i = 0; i < 3; ++i) {
    d.tap_row[i] = a.tap_row[i];
    d.tap_col[i] = a.tap_col[i];
  }
  d.rows = a.rows;
  d.N = a.N;
  d.bias = a.bias;
  d.out = a.out;
  d.out_ld = a.out_ld;
  d.out_batch_stride = a.out_batch_stride;
  d.resid = a.resid;
  d.pos = a.pos;
  d.xkv_d = a.xkv_d;
  d.xkv_heads = a.xkv_heads;
  d.xkv_T = a.xkv_T;
  d.xkv_B = a.xkv_B;
  d.rowinfo = a.rowinfo;
  d.kcache = a.kcache;
  d.vcache = a.vcache;
  d.qkv_d = a.qkv_d;
  d.n_ctx = a.n_ctx;
  d.slots = a.slots;
  return d;
}

void gemm_run(const GemmPlan& pl, cudaStream_t stream) {
  const GemmDev d = make_dev(pl.a, pl.tiles_m, pl.tiles_n, pl.num_kb);
  if (pl.block_n == 128)
    dispatch_epi<128>(pl, d, stream);
  else
    dispatch_epi<32>(pl, d, stream);
}

// ---- e4m3 GEMM (compute_type float8_float16) ----------------------------------------------------------------
// The structure of gemm_tc_kernel with 8-bit operands: 128 x 128 tiles, a K block is one 128-byte swizzle row = 128 codes
// (16 KB of A + 16 KB of B per stage, the fp16 kernel's stage size; five stages leave room for a 128-column epilogue tile), wgmma m64n128k32 e4m3 x e4m3 -> fp32.  Each K block's
// four products go into a fresh set of accumulators that is then added to the tile's fp32 sum: the tensor cores' fp8
// accumulation keeps fewer bits than fp32, so a block's partial sum (128 products) is the most that passes through it.  A K
// that is a multiple of 64 but not of 128 ends with a half block; TMA fills its upper half with zeros.  The row and column
// scales multiply the sum in front of the fp16 kernel's epilogues.
constexpr int kFp8BK = 128;
constexpr int kFp8Stages = 5;
constexpr int kFp8ABytes = BM * kFp8BK, kFp8StageBytes = 2 * kFp8ABytes;
constexpr int kFp8EpiBytes = 2 * 64 * 128 * 4;  // both warpgroups' whole accumulator tiles
constexpr int kFp8Smem = kFp8Stages * kFp8StageBytes + kFp8EpiBytes + 1024 + 256;

template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmDev p,
                const float* __restrict__ a_scale, const float* __restrict__ w_scale) {
  constexpr int BN = 128, STAGES = kFp8Stages, STAGE_BYTES = kFp8StageBytes;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* epi = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + kFp8EpiBytes);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int total_tiles = p.tiles_m * p.tiles_n;  // tile = m * tiles_n + n

  if (warp == 8) {
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_idx = tile % p.tiles_n, m_idx = tile / p.tiles_n;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], STAGE_BYTES);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          tma_load_2d(sa, &tmA, &full[stage], kb * kFp8BK, m_idx * BM);
          tma_load_2d(sa + kFp8ABytes, &tmB, &full[stage], kb * kFp8BK, n_idx * BN);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2, wq = warp & 3, tig = threadIdx.x & 127;
  const int g = lane >> 2, t = lane & 3;
  float* my_epi = epi + wg * 64 * BN;
  const uint32_t bar_id = 1 + wg;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int n_idx = tile % p.tiles_n, m_idx = tile / p.tiles_n;
    float acc[BN / 2], part[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = part[i] = 0.f;
    for (int kb = 0; kb < p.num_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
      const uint64_t da = wgmma_desc_sw128(sa + wg * (64 * 128));
      const uint64_t db = wgmma_desc_sw128(sa + kFp8ABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kFp8BK / 32; ++k) wgmma_ss_e4m3_n128(part, da + 2 * k, db + 2 * k, k);
      wgmma_commit();
      wgmma_wait<0>();
      if (tig == 0) mbar_arrive(&empty[stage]);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }

    // the whole 64 x 128 accumulator tile goes to shared memory at once (one pass keeps no accumulators live next to the
    // epilogue's operands); 16-byte chunk c of row r sits at c ^ (r % 32)
    const int row_l = tig & 63, half = tig >> 6;
    const int row = m_idx * BM + wg * 64 + row_l;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int col = 8 * i + 2 * t, r = 16 * wq + g;
      const int c4 = col >> 2, cw = col & 3;
      *reinterpret_cast<float2*>(my_epi + r * BN + ((c4 ^ (r % 32)) << 2) + cw) = make_float2(acc[4 * i], acc[4 * i + 1]);
      *reinterpret_cast<float2*>(my_epi + (r + 8) * BN + ((c4 ^ ((r + 8) % 32)) << 2) + cw) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
    asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
    for (int c0 = half * 32; c0 < BN; c0 += 64) {
      const int n0 = n_idx * BN + c0;
      if (row < p.rows && n0 < p.N) {
        const float sa_r = __ldg(a_scale + row);
        const float4* ws4 = reinterpret_cast<const float4*>(w_scale + n0);
        float v[32];
        const float4* src = reinterpret_cast<const float4*>(my_epi + row_l * BN);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 f = src[(c0 / 4 + i) ^ (row_l % 32)];
          const float4 ws = __ldg(ws4 + i);
          v[4 * i] = f.x * (sa_r * ws.x);
          v[4 * i + 1] = f.y * (sa_r * ws.y);
          v[4 * i + 2] = f.z * (sa_r * ws.z);
          v[4 * i + 3] = f.w * (sa_r * ws.w);
        }
        epilogue_store<EPI>(p, 0, row, n0, v);
      }
    }
    asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
  }
}

Fp8GemmPlan gemm_fp8_plan(const Fp8GemmArgs& a, int num_sms) {
  B2W_CHECK(a.K % 64 == 0 && a.K > 0, "fp8 GEMM K must be a multiple of 64");
  B2W_CHECK(a.N % 32 == 0 && a.N > 0 && a.rows > 0, "fp8 GEMM N must be a multiple of 32");
  B2W_CHECK(a.epilogue == EPI_F16 || a.epilogue == EPI_GELU_F16 || a.epilogue == EPI_RESID_F32,
            "fp8 GEMM epilogue is F16, GELU_F16 or RESID_F32");
  Fp8GemmPlan p;
  p.a = a;
  p.tiles_m = ceil_div(a.rows, BM);
  p.tiles_n = ceil_div(a.N, 128);
  p.num_kb = ceil_div(a.K, kFp8BK);
  const long long total = (long long)p.tiles_m * p.tiles_n;
  p.grid = (int)(total < num_sms ? total : num_sms);
  {
    uint64_t dims[2] = {(uint64_t)a.K, (uint64_t)a.rows};
    uint64_t strides[1] = {(uint64_t)a.K};
    uint32_t box[2] = {kFp8BK, BM};
    p.tmA = make_tmap_u8(a.A, 2, dims, strides, box);
  }
  {
    uint64_t dims[2] = {(uint64_t)a.K, (uint64_t)a.N};
    uint64_t strides[1] = {(uint64_t)a.K};
    uint32_t box[2] = {kFp8BK, 128};
    p.tmB = make_tmap_u8(a.W, 2, dims, strides, box);
  }
  return p;
}

template <int EPI>
static void configure_fp8() {
  B2W_CUDA(cudaFuncSetAttribute(gemm_fp8_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFp8Smem));
}

template <int EPI>
static void launch_fp8(const Fp8GemmPlan& pl, const GemmDev& d, cudaStream_t stream) {
  gemm_fp8_kernel<EPI><<<pl.grid, kGemmThreads, kFp8Smem, stream>>>(pl.tmA, pl.tmB, d, pl.a.a_scale, pl.a.w_scale);
  B2W_LAUNCHED();
}

void gemm_fp8_run(const Fp8GemmPlan& pl, cudaStream_t stream) {
  GemmDev d{};
  d.batch = 1;
  d.tiles_m = pl.tiles_m;
  d.tiles_n = pl.tiles_n;
  d.num_kb = pl.num_kb;
  d.rows = pl.a.rows;
  d.N = pl.a.N;
  d.bias = pl.a.bias;
  d.out = pl.a.out;
  d.out_ld = pl.a.N;
  d.resid = reinterpret_cast<const float*>(pl.a.out);
  switch (pl.a.epilogue) {
    case EPI_F16: launch_fp8<EPI_F16>(pl, d, stream); break;
    case EPI_GELU_F16: launch_fp8<EPI_GELU_F16>(pl, d, stream); break;
    case EPI_RESID_F32: launch_fp8<EPI_RESID_F32>(pl, d, stream); break;
    default: throw Error("unknown fp8 GEMM epilogue");
  }
}

// ---- plain SIMT reference with the same contract (debug / bisecting; never the timed path) -----------------
__global__ void gemm_ref_kernel(const __half* __restrict__ A, int a_rows, int a_cols, long long a_row_stride,
                                long long a_batch_stride, int taps, int tr0, int tr1, int tr2, int tc0, int tc1, int tc2,
                                int k_per_tap, const __half* __restrict__ W, GemmDev p, int epi) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y * blockDim.y + threadIdx.y;
  const int b = blockIdx.z;
  if (n >= p.N || row >= p.rows) return;
  const int K = taps * k_per_tap;
  float acc = 0.f;
  for (int t = 0; t < taps; ++t) {
    const int r = row + (t == 0 ? tr0 : t == 1 ? tr1 : tr2);
    const int c0 = (t == 0 ? tc0 : t == 1 ? tc1 : tc2);
    if (r < 0 || r >= a_rows) continue;
    const __half* arow = A + b * a_batch_stride + r * a_row_stride;
    const __half* wrow = W + (long long)n * K + t * k_per_tap;
    for (int k = 0; k < k_per_tap; ++k) {
      if (c0 + k < a_cols) acc = fmaf(__half2float(arow[c0 + k]), __half2float(wrow[k]), acc);
    }
  }
  if (p.bias) acc += p.bias[n];
  if (epi == EPI_GELU_F16 || epi == EPI_GELU_POS_F32) acc = gelu_erf(acc);
  const long long idx = (long long)b * p.out_batch_stride + (long long)row * p.out_ld + n;
  if (epi == EPI_F16 || epi == EPI_GELU_F16) {
    reinterpret_cast<__half*>(p.out)[idx] = __float2half_rn(acc);
  } else if (epi == EPI_F16_XKV) {
    const int two_d = 2 * p.xkv_d;
    const int l = n / two_d, rem = n - l * two_d, kv = rem / p.xkv_d, c = rem - kv * p.xkv_d;
    const int e = c & 63;
    long long o = ((((long long)(l * 2 + kv) * p.xkv_B + b) * p.xkv_heads + (c >> 6)) * p.xkv_T + row) * 64 + ((((e >> 3) ^ (row & 7)) << 3) | (e & 7));
    reinterpret_cast<__half*>(p.out)[o] = __float2half_rn(acc);
  } else if (epi == EPI_QKV_CACHE) {
    const int d = p.qkv_d;
    if (n < d) {
      reinterpret_cast<__half*>(p.out)[(long long)row * d + n] = __float2half_rn(acc);
    } else {
      const int4 ri = p.rowinfo[row];
      const int which = n >= 2 * d ? 1 : 0;
      (which ? p.vcache : p.kcache)[(((long long)ri.x * p.n_ctx + ri.z) * p.slots + ri.y) * d + (n - d - which * d)] = __float2half_rn(acc);
    }
  } else if (epi == EPI_RESID_F32) {
    reinterpret_cast<float*>(p.out)[idx] = p.resid[idx] + acc;
  } else if (epi == EPI_GELU_POS_F32) {
    reinterpret_cast<float*>(p.out)[idx] = acc + p.pos[(long long)row * p.N + n];
  } else {
    reinterpret_cast<float*>(p.out)[idx] = acc;
  }
}

void gemm_ref_run(const GemmArgs& a, cudaStream_t stream) {
  const GemmDev d = make_dev(a, 0, 0, 0);
  dim3 block(32, 8);
  dim3 grid(ceil_div(a.N, 32), ceil_div(a.rows, 8), a.a_batch);
  gemm_ref_kernel<<<grid, block, 0, stream>>>(a.A, a.a_rows, a.a_cols, a.a_row_stride,
                                              a.a_batch > 1 ? a.a_batch_stride : a.a_row_stride * a.a_rows, a.taps,
                                              a.tap_row[0], a.tap_row[1], a.tap_row[2], a.tap_col[0], a.tap_col[1],
                                              a.tap_col[2], a.k_per_tap, a.W, d, a.epilogue);
  B2W_LAUNCHED();
}

// ---- TMA descriptor creation -------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static CUtensorMap make_tmap(CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box) {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    B2W_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres));
    if (!sym || qres != cudaDriverEntryPointSuccess) throw Error("cuTensorMapEncodeTiled is not available in this driver");
    fn = reinterpret_cast<PFN_encodeTiled>(sym);
  }
  CUtensorMap m;
  cuuint64_t gdims[5];
  cuuint64_t gstrides[4];
  cuuint32_t bdims[5], estrides[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    bdims[i] = box[i];
    estrides[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstrides[i] = strides_bytes[i];
  CUresult r = fn(&m, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdims, gstrides, bdims,
                  estrides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu,%llu,%llu strides %llu,%llu box %u,%u",
             (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 1 ? strides_bytes[0] : 0),
             (unsigned long long)(rank > 2 ? strides_bytes[1] : 0), box[0], rank > 1 ? box[1] : 0);
    throw Error(buf);
  }
  return m;
}

CUtensorMap make_tmap_f16(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box) {
  return make_tmap(CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, rank, dims, strides_bytes, box);
}
CUtensorMap make_tmap_u8(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rank, dims, strides_bytes, box);
}

}  // namespace b2w
