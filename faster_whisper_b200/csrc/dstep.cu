// One persistent, cooperative kernel per decode step for R <= 8 rows (one chunk x beam 5, greedy, best_of <= 8).
//
// With so few rows every sub-layer streams 3-13 MB of weights: as separate launches each costs 6-15 us, and a large-v3
// step is 257 of them.  Here one CTA per SM stays resident for the whole step and walks the phases
//   embed | L x { QKV, self-attn, out-proj, cross-q, cross-attn, cross-out, FFN1, FFN2 } | logits
// separated by grid barriers.  What shapes it (orders of magnitude; tools/bench/*.cu measures them on the GPU at hand):
//   * a dependent hop through L2 costs ~0.6 us and a grid barrier ~1.4 us, so a phase has a ~2.4 us floor.  Everything a
//     phase needs that does not depend on the previous phase is therefore fetched ahead of time: the weights are stored as
//     a stream of per-work-item tiles (dstep_pack_tiles) and a three-deep shared-memory ring is kept full across phase
//     boundaries by one producer thread, one TMA bulk copy (cp.async.bulk + mbarrier) per 42 KB tile; the cross-attention
//     K/V tile of a layer is prefetched the same way as soon as the layer's self-attention has released the buffer;
//   * LDGSTS (cp.async) is not fire-and-forget: issuing one 40 KB tile as 16-byte copies stalls the issuing warps for
//     ~4400 cycles once the SM's miss queue is full, and every bulk-copy instruction costs ~65 cycles of issue — hence one
//     contiguous block per tile instead of 16 row copies;
//   * the instruction cache: the first version of this kernel was 105 KB of SASS and ran at instruction-fetch speed.
//     The per-layer loop is written for code size: rolled loops, out-of-line phase functions;
//   * acquire fences invalidate L1 (CCTL.IVALL) and with it the stack: the barrier is red.release + relaxed polling, data
//     produced by other CTAs is read with ld.global.cg / TMA, and no phase function keeps state on the stack;
//   * LayerNorms are recomputed by each consumer CTA from the fp32 residual stream (their affine part is folded into the
//     consuming weights at load), and the residual adds are fire-and-forget fp32 reductions.
//
// Math: 16-channel weight tiles feed mma.sync.m16n8k16 fragments (rows = output channels, columns = the <= 8 token rows,
// 8 warps split K); self-attention walks the beam ancestry table; beam-shared cross attention runs QK^T and PV on
// mma.sync from a K/V cache whose 16-byte chunks are XOR-swizzled by the key index (conflict-free fragment loads without
// padding), with 7 flash-decoding key splits per (chunk, head) and a last-arriver combine.
//
// Replaces the per-token body of CTranslate2's Whisper.generate loop (reference call sites
// faster_whisper/transcribe.py:222-236, 1446-1459; SURVEY.md §2.3 rows K10-K15) — the "single persistent kernel per
// decode step" of BASELINE.json's north_star.
#include <math.h>

#include <vector>

#include "common.cuh"
#include "decode.h"
#include "dstep.h"
#include "step_common.cuh"

namespace b2w {

constexpr int kDsThreads = 256;   // compute threads (8 warps)
constexpr int kDsLaunchThreads = 320;  // + one warp streaming weight tiles, one prefetching cross-attention K/V
constexpr int kDsWarps = 8;
constexpr int kDsNBuf = 3;         // weight-tile ring: the tile being consumed + two in flight
constexpr int kDsSelfKeys = 192;   // keys staged per self-attention pass
constexpr int kDsKvBytes = 2 * kDsXKeysMax * 64 * 2;  // cross-attention K + V tile
constexpr int kDsScLd = kDsXKeysMax + 4;   // fp32 score rows
constexpr int kDsPLd = kDsXKeysMax + 8;    // fp16 probability rows
constexpr int kDsQLd = 96;                 // fp16 query rows
constexpr int kDsXScratch = kDsXQ * kDsQLd * 2 + kDsXQ * kDsScLd * 4 + kDsXQ * kDsPLd * 2 + 2 * kDsXQ * 64 * 4 + 64;

// barrier of the 256 compute threads (the producer warps never join it)
__device__ __forceinline__ void ds_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// fine-grained cycle accounting for CTA 0 (B2W_DSTEP_PROF): accumulated in shared memory, dumped to prof[3000 + kind*16 + point] at the
// end.  Compiled in only with -DB2W_STEP_TICKS (libb200whisper_ticks.so): the phase code runs once per phase, every instruction counts.
#ifdef B2W_STEP_TICKS
#define DS_TICK_DECL(tp) long long tp = clock64()
#define DS_TICK_COUNT(a, kind) do { if ((a).prof && blockIdx.x == 0 && threadIdx.x == 0) sh.ticks[(kind) * 8 + 7] += 1; } while (0)
#define DS_TICK(a, kind, point, tprev)                                    \
  do {                                                                    \
    if ((a).prof && blockIdx.x == 0 && threadIdx.x == 0) {                \
      const long long _now = clock64();                                   \
      sh.ticks[(kind) * 8 + (point)] += (unsigned)(_now - (tprev));       \
      (tprev) = _now;                                                     \
    }                                                                     \
  } while (0)
#else
#define DS_TICK_DECL(tp) do { } while (0)
#define DS_TICK_COUNT(a, kind) do { } while (0)
#define DS_TICK(a, kind, point, tprev) do { } while (0)
#endif

// per-CTA state that lives in shared memory (pointers/tables are never re-fetched from L2 inside the layer loop)
struct DsShared {
  DLayer lay[32];
  RowInfo rows[8];
  unsigned epoch;
  int prof_i;
  int flag;
  unsigned ticks[8 * 8];
  uint64_t wfull[kDsNBuf];   // weight tile landed (TMA complete_tx)
  uint64_t wempty[kDsNBuf];  // weight tile consumed (one arrival by compute thread 0)
  uint64_t kvfull;           // cross-attention K/V tile landed
  uint64_t kvfree;           // K/V buffer released by this layer's self-attention
};

// Grid barrier: every CTA arrives once; sh.epoch is the running arrival target (the host zeroes *bar before the launch).
// Arrive = red.release (orders the CTA's earlier writes, cumulative through bar.sync); wait = relaxed polling.
__device__ __forceinline__ void ds_grid_barrier(const DStepArgs& a, DsShared& sh) {
  ds_sync();
  if (threadIdx.x == 0) {
    sh.epoch += gridDim.x;
    if (a.prof && blockIdx.x == 0) a.prof[sh.prof_i] = ds_globaltimer();  // arrival of CTA 0
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.bar) : "memory");
    const unsigned target = sh.epoch;
    unsigned v;
    do {
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.bar) : "memory");
    } while (v < target);
    if (a.prof && blockIdx.x == 0) a.prof[sh.prof_i + 1] = ds_globaltimer();  // release
    sh.prof_i += 2;
  }
  ds_sync();
}

enum { DS_QKV = 0, DS_F16 = 1, DS_GELU = 2, DS_RESID = 3, DS_F32 = 4 };

// The GEMVs of a step form a static sequence s = 0 .. 6L (per layer: qkv, out, cross_q, cross_out, ffn1, ffn2; then logits).
// A work item is (16 output channels, one K range of width d): every GEMV has K = d except ffn2 (K = 4d, four ranges).
__device__ __forceinline__ void ds_geom(const DStepArgs& a, int s, int& ntiles, int& ksplit) {
  ksplit = 1;
  if (s >= 6 * a.L) {
    ntiles = a.vpad >> 4;
    return;
  }
  const int sub = s % 6, dt = a.d >> 4;
  ntiles = sub == 0 ? 3 * dt : (sub == 4 ? 4 * dt : dt);
  if (sub == 5) ksplit = 4;
}
// j-th work item of this CTA in a phase, or -1.  With four K ranges the CTAs are grouped in fours so that all items of a
// CTA share one range (it stages only that quarter of the FFN activations).
__device__ __forceinline__ int ds_item(int ntiles, int ksplit, int j) {
  if (ksplit == 1) {
    const int it = blockIdx.x + j * gridDim.x;
    return it < ntiles ? it : -1;
  }
  const int g4 = gridDim.x >> 2;
  if ((int)blockIdx.x >= 4 * g4) return -1;
  const int tl = (int)(blockIdx.x >> 2) + j * g4;
  return tl < ntiles ? tl * 4 + (int)(blockIdx.x & 3) : -1;
}
// fp16 tiles: 16 rows x (d + 32) halves + 16 fp32 bias values; int8 tiles: 16 rows x (d + 32) bytes (weights stored as q + 128)
// + 16 fp32 per-channel scales + 16 fp32 bias values
__host__ __device__ __forceinline__ uint32_t ds_tile_bytes(int d, int w8) {
  return w8 ? (uint32_t)(16 * (d + 32) + 128) : (uint32_t)(16 * (d + 32) + 32) * 2u;
}
// Weight producer (one thread of a dedicated warp): walks this CTA's work items of the whole step in order and keeps the
// ring full — wait until the buffer's previous tile has been consumed, then one TMA bulk copy per tile.  It never
// synchronises with the compute warps other than through the mbarriers, so it runs ahead across phase boundaries.
__device__ __noinline__ void ds_weight_producer(const DStepArgs& a, DsShared& sh, unsigned char* ring, int tile_stride) {
  const int last = 6 * a.L;
  const uint32_t bytes = ds_tile_bytes(a.d, a.w8);
  int n = 0;
#pragma unroll 1
  for (int s = 0; s <= last; ++s) {
    int ntiles, ksplit;
    ds_geom(a, s, ntiles, ksplit);
    const __half* base = s >= last ? a.logit_tiles : sh.lay[s / 6].wt[s % 6];
#pragma unroll 1
    for (int j = 0;; ++j) {
      const int item = ds_item(ntiles, ksplit, j);
      if (item < 0) break;
      const int buf = n % kDsNBuf;
      mbar_wait(&sh.wempty[buf], (uint32_t)(((n / kDsNBuf) & 1) ^ 1));  // passes immediately on the first lap
      fence_proxy_async();
      mbar_expect_tx(&sh.wfull[buf], bytes);
      ds_bulk_g2s(ring + (size_t)buf * tile_stride, reinterpret_cast<const unsigned char*>(base) + (long long)item * bytes, bytes, &sh.wfull[buf]);
      n += 1;
    }
  }
}

// One GEMV phase: y[R,N] = in[R,K] W[N,K]^T for this CTA's items, weights consumed from the shared-memory ring.
// Returns the updated count of consumed tiles (a warp-uniform register value; the ring index and mbarrier parity follow
// from it).
template <bool W8>
__device__ __noinline__ int ds_gemv_phase(const DStepArgs& a, DsShared& sh, int s, int consumed, unsigned char* ring, int tile_stride, __half* xs,
                                          float* red, __half* kc, __half* vc) {
  int ntiles, ksplit;
  ds_geom(a, s, ntiles, ksplit);
  if (ds_item(ntiles, ksplit, 0) < 0) return consumed;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int d = a.d, ld = d + 32, kchunks = d >> 5;
  const bool is_logits = s >= 6 * a.L;
  const int sub = is_logits ? 6 : s % 6;
  const int N = ntiles << 4;
  int mode, ln = 0, src_ld = d;
  const __half* src16 = nullptr;
  switch (sub) {
    case 0: mode = DS_QKV; ln = 1; break;
    case 1: mode = DS_RESID; src16 = a.ao; break;
    case 2: mode = DS_F16; ln = 1; break;
    case 3: mode = DS_RESID; src16 = a.ao; break;
    case 4: mode = DS_GELU; ln = 1; break;
    case 5: mode = DS_RESID; src16 = a.h + (blockIdx.x & 3) * d; src_ld = 4 * d; break;
    default: mode = DS_F32; ln = 1; break;
  }
  DS_TICK_DECL(tp);
  // ---- input rows -> xs [8][d + 32] halves, straight from L2 (one round trip) ----
  if (ln) {
    if (warp < a.R) {  // one warp per row: single-pass LayerNorm from registers (affine part folded into the weights)
      const float4* xr = reinterpret_cast<const float4*>(a.x + (long long)warp * d);
      const int n4 = d >> 2;
      float4 v[10];
      float su = 0.f, sq = 0.f;
#pragma unroll
      for (int i = 0; i < 10; ++i) {
        const int idx = lane + 32 * i;
        v[i] = idx < n4 ? __ldcg(xr + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int i = 0; i < 10; ++i) {
        su += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        sq += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
      }
      su = warp_sum(su);
      sq = warp_sum(sq);
      const float mean = su / d;
      const float rstd = rsqrtf(fmaxf(sq / d - mean * mean, 0.f) + 1e-5f);
      uint2* o = reinterpret_cast<uint2*>(xs + warp * ld);
#pragma unroll
      for (int i = 0; i < 10; ++i) {
        const int idx = lane + 32 * i;
        if (idx < n4)
          o[idx] = make_uint2(pack_half2((v[i].x - mean) * rstd, (v[i].y - mean) * rstd), pack_half2((v[i].z - mean) * rstd, (v[i].w - mean) * rstd));
      }
    }
  } else {
    // all 16-byte loads of a thread are in flight together (one L2 round trip): up to 8 rows x d/8 chunks over 256 threads
    const int c8 = d >> 3, total = a.R * c8;
    uint4 v[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int i = tid + k * kDsThreads;
      if (i < total) {
        const int r = i / c8, c = i - r * c8;
        v[k] = __ldcg(reinterpret_cast<const uint4*>(src16 + (long long)r * src_ld) + c);
      }
    }
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int i = tid + k * kDsThreads;
      if (i < total) {
        const int r = i / c8, c = i - r * c8;
        *reinterpret_cast<uint4*>(xs + r * ld + c * 8) = v[k];
      }
    }
  }
  ds_sync();
  DS_TICK(a, sub, 0, tp);  // input staged
  bool first = true;
#pragma unroll 1
  for (int j = 0;; ++j) {
    const int item = ds_item(ntiles, ksplit, j);
    if (item < 0) break;
    const int tl = ksplit == 1 ? item : item >> 2;
    const int buf = consumed % kDsNBuf;
    mbar_wait(&sh.wfull[buf], (uint32_t)((consumed / kDsNBuf) & 1));
    if (first) DS_TICK(a, sub, 1, tp);  // weight tile landed
    const __half* wt = reinterpret_cast<const __half*>(ring + (size_t)buf * tile_stride);
    const __half* xb = xs + g * ld + 8 * t;
    float acc[4] = {0.f, 0.f, 0.f, 0.f}, acc2[4] = {0.f, 0.f, 0.f, 0.f};
    if constexpr (W8) {
      // int8 weight stream: 8 bytes per (row, 32-wide k chunk) and lane, widened to fp16 in registers; the per-channel
      // scale is applied to the fp32 sum in the epilogue
      const unsigned char* w8 = ring + (size_t)buf * tile_stride;
      const unsigned char* w_lo = w8 + g * ld + 8 * t;
      const unsigned char* w_hi = w_lo + 8 * ld;
#pragma unroll 5
      for (int c = warp; c < kchunks; c += kDsWarps) {
        const uint2 wa = *reinterpret_cast<const uint2*>(w_lo + c * 32);
        const uint2 wb = *reinterpret_cast<const uint2*>(w_hi + c * 32);
        const uint4 xv = *reinterpret_cast<const uint4*>(xb + c * 32);
        ds_mma(acc, ds_cvt_u8x2(wa.x, 0x5140u), ds_cvt_u8x2(wb.x, 0x5140u), ds_cvt_u8x2(wa.x, 0x5342u), ds_cvt_u8x2(wb.x, 0x5342u), xv.x, xv.y);
        ds_mma(acc2, ds_cvt_u8x2(wa.y, 0x5140u), ds_cvt_u8x2(wb.y, 0x5140u), ds_cvt_u8x2(wa.y, 0x5342u), ds_cvt_u8x2(wb.y, 0x5342u), xv.z, xv.w);
      }
    } else {
      const __half* w_lo = wt + g * ld + 8 * t;
      const __half* w_hi = w_lo + 8 * ld;
#pragma unroll 5
      for (int c = warp; c < kchunks; c += kDsWarps) {
        const uint4 wa = *reinterpret_cast<const uint4*>(w_lo + c * 32);
        const uint4 wb = *reinterpret_cast<const uint4*>(w_hi + c * 32);
        const uint4 xv = *reinterpret_cast<const uint4*>(xb + c * 32);
        ds_mma(acc, wa.x, wb.x, wa.y, wb.y, xv.x, xv.y);
        ds_mma(acc2, wa.z, wb.z, wa.w, wb.w, xv.z, xv.w);
      }
    }
    float* rj = red + (j & 1) * (kDsWarps * 128);
    float* my = rj + warp * 128;  // [16 ch][8 rows]
    *reinterpret_cast<float2*>(my + g * 8 + 2 * t) = make_float2(acc[0] + acc2[0], acc[1] + acc2[1]);
    *reinterpret_cast<float2*>(my + (g + 8) * 8 + 2 * t) = make_float2(acc[2] + acc2[2], acc[3] + acc2[3]);
    const int ch = tid & 15, r = tid >> 4;
    float v = 0.f, wscale = 1.f;  // bias (zero for ks > 0) and, for int8 tiles, the channel's de-quantisation scale
    if (tid < 128) {
      if constexpr (W8) {
        const float* tail = reinterpret_cast<const float*>(ring + (size_t)buf * tile_stride + 16 * ld);
        wscale = tail[ch];
        v = tail[16 + ch];
      } else {
        v = reinterpret_cast<const float*>(wt + 16 * ld)[ch];
      }
    }
    ds_sync();  // partials visible; the weight buffer is free
    consumed += 1;
    if (tid == 0) mbar_arrive(&sh.wempty[buf]);
    if (first) DS_TICK(a, sub, 2, tp);  // MMAs + partials
    if (tid < 128 && r < a.R) {
      float sum = 0.f;
#pragma unroll
      for (int w = 0; w < kDsWarps; ++w) sum += rj[w * 128 + ch * 8 + r];
      v = W8 ? fmaf(sum, wscale, v) : v + sum;
      const int n = tl * 16 + ch;
      if (mode == DS_QKV) {
        if (n < d) {
          a.q[(long long)r * d + n] = __float2half_rn(v);
        } else {
          const RowInfo ri = sh.rows[r];
          const int which = (n >= 2 * d) ? 1 : 0;
          (which ? vc : kc)[(((long long)ri.chunk * a.n_ctx + ri.pos) * a.slots + ri.slot) * d + (n - d - which * d)] = __float2half_rn(v);
        }
      } else if (mode == DS_F16) {
        a.q[(long long)r * N + n] = __float2half_rn(v);
      } else if (mode == DS_GELU) {
        a.h[(long long)r * N + n] = __float2half_rn(gelu_erf(v));
      } else if (mode == DS_RESID) {
        atomicAdd(a.x + (long long)r * N + n, v);  // fire-and-forget reduction into the fp32 residual stream
      } else {
        a.logits[(long long)r * a.vpad + n] = v;
      }
    }
    if (first) {
      DS_TICK(a, sub, 3, tp);  // epilogue
      DS_TICK_COUNT(a, sub);
    }
    first = false;
  }
  return consumed;
}

// masked self-attention for one (head, row) task: the row's K/V history is gathered through the ancestry table into
// shared memory with async copies (one L2/HBM round trip per pass of kDsSelfKeys keys), then scored from there with an
// online softmax across passes
__device__ __noinline__ void ds_self_attn_task(const DStepArgs& a, const DsShared& sh, int h, int r, const __half* kc, const __half* vc, float* sm) {
  float* sc = sm;                      // [kDsSelfKeys]
  float* red = sm + kDsSelfKeys;       // [16]
  float* oacc = red + 16;              // [4][64]
  float* qf = oacc + 256;              // [64]
  __half* kt = reinterpret_cast<__half*>(qf + 64);  // [kDsSelfKeys][72]  (offset 560 floats: 16-byte aligned)
  __half* vt = kt + kDsSelfKeys * 72;               // [kDsSelfKeys][64]
  const RowInfo ri = sh.rows[r];
  const int d = a.d, nk = ri.pos + 1, tid = threadIdx.x;
  const uint8_t* anc = a.anc + (ri.pos & 1) * a.anc_buf_stride + ((long long)ri.chunk * a.slots + ri.slot) * a.n_ctx;
  if (tid < 64) qf[tid] = __half2float(__ldcg(a.q + (long long)r * d + h * 64 + tid)) * 0.125f;
  const int e = tid & 63, part = tid >> 6;
  float m_run = -INFINITY, l_run = 0.f, acc = 0.f;
#pragma unroll 1
  for (int base = 0; base < nk; base += kDsSelfKeys) {
    const int n = min(kDsSelfKeys, nk - base);
    if (tid < n) {
      const int j = base + tid;
      const int slot = (j == ri.pos) ? ri.slot : anc[j];
      const long long off = (((long long)ri.chunk * a.n_ctx + j) * a.slots + slot) * d + h * 64;
#pragma unroll 2
      for (int i = 0; i < 8; ++i) {
        ds_cp_async16(kt + tid * 72 + i * 8, kc + off + i * 8);
        ds_cp_async16(vt + tid * 64 + i * 8, vc + off + i * 8);
      }
    }
    ds_cp_commit();
    ds_cp_wait_all();
    ds_sync();
    float mx = -INFINITY;
    if (tid < n) {
      const __half2* kp = reinterpret_cast<const __half2*>(kt + tid * 72);
      float s0 = 0.f, s1 = 0.f;
#pragma unroll 4
      for (int i = 0; i < 32; i += 2) {
        const float2 k0 = __half22float2(kp[i]), k1 = __half22float2(kp[i + 1]);
        s0 = fmaf(k0.x, qf[2 * i], fmaf(k0.y, qf[2 * i + 1], s0));
        s1 = fmaf(k1.x, qf[2 * i + 2], fmaf(k1.y, qf[2 * i + 3], s1));
      }
      mx = s0 + s1;
      sc[tid] = mx;
    }
    mx = warp_max(mx);
    if ((tid & 31) == 0) red[tid >> 5] = mx;
    ds_sync();
    mx = red[0];
#pragma unroll
    for (int i = 1; i < kDsWarps; ++i) mx = fmaxf(mx, red[i]);
    const float m_new = fmaxf(m_run, mx);
    float sum = 0.f;
    if (tid < n) {
      const float p = __expf(sc[tid] - m_new);
      sc[tid] = p;
      sum = p;
    }
    sum = warp_sum(sum);
    if ((tid & 31) == 0) red[8 + (tid >> 5)] = sum;
    ds_sync();
    sum = 0.f;
#pragma unroll
    for (int i = 0; i < kDsWarps; ++i) sum += red[8 + i];
    const float alpha = (m_run == -INFINITY) ? 0.f : __expf(m_run - m_new);
    float a0 = 0.f, a1 = 0.f;
    int j = part;  // this thread's keys: part, part + 4, ...; two independent chains
#pragma unroll 2
    for (; j + 4 < n; j += 8) {
      a0 = fmaf(sc[j], __half2float(vt[j * 64 + e]), a0);
      a1 = fmaf(sc[j + 4], __half2float(vt[(j + 4) * 64 + e]), a1);
    }
    if (j < n) a0 = fmaf(sc[j], __half2float(vt[j * 64 + e]), a0);
    acc = fmaf(acc, alpha, a0 + a1);
    l_run = fmaf(l_run, alpha, sum);
    m_run = m_new;
    ds_sync();  // the staging buffers are reused by the next pass
  }
  oacc[part * 64 + e] = acc;
  ds_sync();
  if (tid < 64) a.ao[(long long)r * d + h * 64 + tid] = __float2half_rn((oacc[tid] + oacc[64 + tid] + oacc[128 + tid] + oacc[192 + tid]) / l_run);
  ds_sync();
}

// Cross-attention tasks: task = ((chunk * H + head) * QG + query group) * kDsXSplits + key split, with QG = ds_xqgroups(rows
// per chunk); task / kDsXSplits indexes the task's partials and counter.
__host__ __device__ __forceinline__ int ds_xtasks(const DStepArgs& a) { return kDsXSplits * ds_xqgroups(a.rows_per_chunk) * a.H * a.n_chunks; }

// TMA the K and V tiles of one cross-attention task into kvbuf (one thread); they depend on (key split, head, chunk) only.
__device__ __noinline__ void ds_issue_cross_kv(const DStepArgs& a, DsShared& sh, int layer, int task, unsigned char* kvbuf) {
  const int split = task % kDsXSplits, bh = task / kDsXSplits / ds_xqgroups(a.rows_per_chunk);
  const int h = bh % a.H, b = bh / a.H, T = a.T;
  const int k0 = (int)((long long)T * split / kDsXSplits), k1 = (int)((long long)T * (split + 1) / kDsXSplits), nk = k1 - k0;
  const DecBindings bd = a.bind[b];
  const long long per = (long long)bd.B_total * a.H * T * 64;
  const long long off = (((long long)bd.item * a.H + h) * T + k0) * 64;
  const __half* Kb = bd.xkv + ((long long)layer * 2 + 0) * per + off;
  const __half* Vb = bd.xkv + ((long long)layer * 2 + 1) * per + off;
  fence_proxy_async();  // the buffer was last written through the generic proxy (self-attention staging)
  mbar_expect_tx(&sh.kvfull, (uint32_t)nk * 256u);
  ds_bulk_g2s(kvbuf, Kb, (uint32_t)nk * 128u, &sh.kvfull);
  ds_bulk_g2s(kvbuf + kDsXKeysMax * 128, Vb, (uint32_t)nk * 128u, &sh.kvfull);
}

// K/V producer (one thread of a second dedicated warp): per layer, as soon as the layer's self-attention has released the
// buffer, fetch the tile of this CTA's first cross-attention task — it does not depend on the step, only on the layer.
__device__ __noinline__ void ds_kv_producer(const DStepArgs& a, DsShared& sh, unsigned char* kvbuf) {
  if ((int)blockIdx.x >= ds_xtasks(a)) return;
#pragma unroll 1
  for (int l = 0; l < a.L; ++l) {
    mbar_wait(&sh.kvfree, (uint32_t)(l & 1));
    ds_issue_cross_kv(a, sh, l, blockIdx.x, kvbuf);
  }
}

// Beam-shared cross attention: one (key split, query group, head, chunk) task for up to kDsXQ rows of the chunk; the last
// split of a (chunk, head, query group) to finish combines.  K/V rows are 128 bytes whose 16-byte chunks are XOR-swizzled by
// (key & 7) in the cache itself (gemm.cu EPI_F16_XKV), so the tile arrives conflict-free with two bulk copies.
//   S[key][q]  = K Q^T      : mma A = K rows (keys), B = Q rows; 16-byte fragment loads, k-permuted like the GEMVs
//   O^T[e][q]  = V^T P^T    : mma A = V^T via ldmatrix.trans, B = P rows (fp16 probabilities)
__device__ __noinline__ int ds_cross_attn_task(const DStepArgs& a, DsShared& sh, int layer, int task, bool prefetched, int kv_uses,
                                               unsigned char* kvbuf, unsigned char* scratch) {
  const int T = a.T, S = kDsXSplits, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int split = task % S, group = task / S, QG = ds_xqgroups(a.rows_per_chunk), qg = group % QG;
  const int h = group / QG % a.H, b = group / QG / a.H, d = a.d;
  const int row0 = b * a.rows_per_chunk + kDsXQ * qg, nq = min(kDsXQ, a.rows_per_chunk - kDsXQ * qg);
  const int k0 = (int)((long long)T * split / S), k1 = (int)((long long)T * (split + 1) / S), nk = k1 - k0;
  const int nkp = (nk + 15) & ~15;
  __half* kt = reinterpret_cast<__half*>(kvbuf);  // [224][64] swizzled
  __half* vt = kt + kDsXKeysMax * 64;
  __half* qs = reinterpret_cast<__half*>(scratch);                 // [8][96], pre-scaled by 1/8
  float* sc = reinterpret_cast<float*>(qs + kDsXQ * kDsQLd);      // [8][kDsScLd]
  __half* pr = reinterpret_cast<__half*>(sc + kDsXQ * kDsScLd);   // [8][kDsPLd]
  float* wred = reinterpret_cast<float*>(pr + kDsXQ * kDsPLd);    // [2][8][64]
  float* stat = wred + 2 * kDsXQ * 64;                            // [8][2]
  if (!prefetched && tid == 0) ds_issue_cross_kv(a, sh, layer, task, kvbuf);
  if (tid < 64) {
    const int q = tid >> 3, c = tid & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (q < nq) {
      v = __ldcg(reinterpret_cast<const uint4*>(a.q + (long long)(row0 + q) * d + h * 64) + c);
      __half2* h2 = reinterpret_cast<__half2*>(&v);
      const __half2 sc8 = __floats2half2_rn(0.125f, 0.125f);
#pragma unroll
      for (int i = 0; i < 4; ++i) h2[i] = __hmul2(h2[i], sc8);
    }
    *reinterpret_cast<uint4*>(qs + q * kDsQLd + c * 8) = v;
  }
  // rows [nk, nkp) of V are multiplied by zero probabilities: make them finite
  for (int i = tid; i < (nkp - nk) * 8; i += kDsThreads) *reinterpret_cast<uint4*>(vt + (nk + (i >> 3)) * 64 + (i & 7) * 8) = make_uint4(0u, 0u, 0u, 0u);
  mbar_wait(&sh.kvfull, (uint32_t)(kv_uses & 1));
  ds_sync();
  // ---- scores ----
#pragma unroll 1
  for (int tile = warp; tile * 16 < nkp; tile += kDsWarps) {
    const int rg = tile * 16 + g, swz = (k0 + rg) & 7;  // rows rg and rg + 8 share the swizzle
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int c2 = 0; c2 < 2; ++c2) {
      const int pc = ((4 * c2 + t) ^ swz) << 3;
      const uint4 wa = *reinterpret_cast<const uint4*>(kt + rg * 64 + pc);
      const uint4 wb = *reinterpret_cast<const uint4*>(kt + (rg + 8) * 64 + pc);
      const uint4 xv = *reinterpret_cast<const uint4*>(qs + g * kDsQLd + 32 * c2 + 8 * t);
      ds_mma(acc, wa.x, wb.x, wa.y, wb.y, xv.x, xv.y);
      ds_mma(acc, wa.z, wb.z, wa.w, wb.w, xv.z, xv.w);
    }
    sc[(2 * t) * kDsScLd + rg] = acc[0];
    sc[(2 * t + 1) * kDsScLd + rg] = acc[1];
    sc[(2 * t) * kDsScLd + rg + 8] = acc[2];
    sc[(2 * t + 1) * kDsScLd + rg + 8] = acc[3];
  }
  ds_sync();
  {  // one warp per query: partial softmax statistics, probabilities as fp16
    const int q = warp;
    if (q < nq) {
      float mx = -INFINITY;
      for (int j = lane; j < nk; j += 32) mx = fmaxf(mx, sc[q * kDsScLd + j]);
      mx = warp_max(mx);
      float sum = 0.f;
      for (int j = lane; j < nkp; j += 32) {
        const float p = j < nk ? __expf(sc[q * kDsScLd + j] - mx) : 0.f;
        const __half ph = __float2half_rn(p);
        pr[q * kDsPLd + j] = ph;
        sum += __half2float(ph);
      }
      sum = warp_sum(sum);
      if (lane == 0) {
        stat[q * 2] = mx;
        stat[q * 2 + 1] = sum;
      }
    } else {
      for (int j = lane; j < nkp; j += 32) pr[q * kDsPLd + j] = __float2half_rn(0.f);
    }
  }
  ds_sync();
  {  // ---- O^T = V^T P^T: warp -> (16 output dims, half of the key tiles) ----
    const int dtile = warp & 3, khalf = warp >> 2;
    const int mi = lane >> 3, r8 = lane & 7;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int tile = khalf; tile * 16 < nkp; tile += 2) {
      const int row = tile * 16 + 8 * (mi >> 1) + r8;
      const int pc = ((2 * dtile + (mi & 1)) ^ ((k0 + row) & 7)) << 3;
      uint32_t a0, a1, a2, a3;
      ds_ldmatrix_x4_trans(a0, a1, a2, a3, vt + row * 64 + pc);
      const uint32_t b0 = *reinterpret_cast<const uint32_t*>(pr + g * kDsPLd + tile * 16 + 2 * t);
      const uint32_t b1 = *reinterpret_cast<const uint32_t*>(pr + g * kDsPLd + tile * 16 + 2 * t + 8);
      ds_mma(acc, a0, a1, a2, a3, b0, b1);
    }
    float* w = wred + khalf * (kDsXQ * 64);
    w[(2 * t) * 64 + 16 * dtile + g] = acc[0];
    w[(2 * t + 1) * 64 + 16 * dtile + g] = acc[1];
    w[(2 * t) * 64 + 16 * dtile + g + 8] = acc[2];
    w[(2 * t + 1) * 64 + 16 * dtile + g + 8] = acc[3];
  }
  ds_sync();
  float* part = a.xpart + ((long long)group * S + split) * (kDsXQ * 66);
#pragma unroll 1
  for (int i = tid; i < nq * 64; i += kDsThreads) {
    const int q = i >> 6, e = i & 63;
    __stcg(part + q * 66 + e, wred[q * 64 + e] + wred[(kDsXQ + q) * 64 + e]);
  }
  if (tid < nq) {
    __stcg(part + tid * 66 + 64, stat[tid * 2]);
    __stcg(part + tid * 66 + 65, stat[tid * 2 + 1]);
  }
  ds_sync();
  if (tid == 0) {
    int ticket;  // release: the CTA's partials are visible before the ticket; the combiner reads them with ld.cg (L2)
    asm volatile("atom.release.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(a.xcounters + group) : "memory");
    sh.flag = (ticket == S - 1);
    if (sh.flag) a.xcounters[group] = 0;
  }
  ds_sync();
  if (sh.flag) {
    const float* pg = a.xpart + (long long)group * S * (kDsXQ * 66);
#pragma unroll 1
    for (int i = tid; i < nq * 64; i += kDsThreads) {
      const int q = i >> 6, e = i & 63;
      float pm[8], pl[8], pa[8];
#pragma unroll
      for (int s2 = 0; s2 < 8; ++s2) {  // all L2 loads in flight together
        const bool on = s2 < S;
        const float* base = pg + ((on ? s2 : 0) * kDsXQ + q) * 66;
        pm[s2] = on ? __ldcg(base + 64) : -INFINITY;
        pl[s2] = on ? __ldcg(base + 65) : 0.f;
        pa[s2] = on ? __ldcg(base + e) : 0.f;
      }
      float M = pm[0];
#pragma unroll
      for (int s2 = 1; s2 < 8; ++s2) M = fmaxf(M, pm[s2]);
      float num = 0.f, den = 0.f;
#pragma unroll
      for (int s2 = 0; s2 < 8; ++s2) {
        const float w = (s2 < S) ? __expf(pm[s2] - M) : 0.f;
        num = fmaf(w, pa[s2], num);
        den = fmaf(w, pl[s2], den);
      }
      a.ao[(long long)(row0 + q) * d + h * 64 + e] = __float2half_rn(num / den);
    }
  }
  ds_sync();
  return kv_uses + 1;
}

template <bool W8>
__global__ void __launch_bounds__(kDsLaunchThreads, 1) dstep_kernel(const DStepArgs a_param) {
  extern __shared__ __align__(128) unsigned char ds_smem[];
  // the argument block is copied to shared memory: the out-of-line phase functions take it by reference, and a reference
  // to a kernel parameter would otherwise be materialised on the (L1-cached, local-memory) stack
  __shared__ DStepArgs a_sh;
  __shared__ DsShared sh;
  if (threadIdx.x == 0) a_sh = a_param;
  __syncthreads();
  const DStepArgs& a = a_sh;
  // [weight ring: kDsNBuf tiles][cross-attention K/V tile | self-attention scratch][GEMV input xs | cross-attention scratch][red x2]
  const int d = a.d, L = a.L;
  const int tile_stride = (int)((ds_tile_bytes(d, W8 ? 1 : 0) + 127u) & ~127u);
  unsigned char* ring = ds_smem;
  unsigned char* kvbuf = ring + (size_t)kDsNBuf * tile_stride;
  unsigned char* scr = kvbuf + kDsKvBytes;
  const int xs_bytes = 8 * (d + 32) * 2;
  const int scr_bytes = ((xs_bytes > kDsXScratch ? xs_bytes : kDsXScratch) + 127) & ~127;
  float* red = reinterpret_cast<float*>(scr + scr_bytes);
  __half* xs = reinterpret_cast<__half*>(scr);
  {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(a.layers);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(sh.lay);
    for (int i = threadIdx.x; i < L * (int)(sizeof(DLayer) / 8); i += kDsLaunchThreads) dst[i] = src[i];
    if (threadIdx.x < a.R) sh.rows[threadIdx.x] = a.rows[threadIdx.x];
    if (threadIdx.x == 0) {
      sh.epoch = 0;
      sh.prof_i = 1;
      for (int i = 0; i < kDsNBuf; ++i) {
        mbar_init(&sh.wfull[i], 1);
        mbar_init(&sh.wempty[i], 1);
      }
      mbar_init(&sh.kvfull, 1);
      mbar_init(&sh.kvfree, 1);
      fence_mbar_init();
      if (a.prof && blockIdx.x == 0) a.prof[0] = ds_globaltimer();
    }
    if (threadIdx.x < 64) sh.ticks[threadIdx.x] = 0;
  }
  __syncthreads();
  // ---- role split: warp 8 streams the weight tiles, warp 9 prefetches cross-attention K/V, warps 0-7 compute ----
  if (threadIdx.x >= kDsThreads) {
    if (threadIdx.x == kDsThreads) ds_weight_producer(a, sh, ring, tile_stride);
    if (threadIdx.x == kDsThreads + 32) ds_kv_producer(a, sh, kvbuf);
    return;
  }
  int consumed = 0, kv_uses = 0;

  // ---- embed: x = tok_emb[token] + pos_emb[pos] (CTA r owns row r) ----
  if ((int)blockIdx.x < a.R) {
    const int r = blockIdx.x;
    int tok = a.tokens_in[r];
    tok = tok < 0 ? 0 : (tok >= a.n_vocab ? a.n_vocab - 1 : tok);
    const int pos = sh.rows[r].pos;
#pragma unroll 2
    for (int i = threadIdx.x; i < d; i += kDsThreads)
      __stcg(a.x + (long long)r * d + i, __half2float(a.tok_emb[(long long)tok * d + i]) + a.pos_emb[(long long)pos * d + i]);
  }
  ds_grid_barrier(a, sh);

  const int xtasks = ds_xtasks(a);
#pragma unroll 1
  for (int l = 0; l < L; ++l) {
    __half* kc = a.kcache + (long long)l * a.kv_layer_stride;
    __half* vc = a.vcache + (long long)l * a.kv_layer_stride;
#pragma unroll 1
    for (int ph = 0; ph < 8; ++ph) {
      if (ph == 1) {  // masked self-attention
#pragma unroll 1
        for (int task = blockIdx.x; task < a.H * a.R; task += gridDim.x)
          ds_self_attn_task(a, sh, task % a.H, task / a.H, kc, vc, reinterpret_cast<float*>(kvbuf));
        // the buffer is free until this layer's cross attention: let the K/V producer fetch the tile now
        if (threadIdx.x == 0) mbar_arrive(&sh.kvfree);
      } else if (ph == 4) {  // beam-shared cross attention
        bool pre = true;
#pragma unroll 1
        for (int task = blockIdx.x; task < xtasks; task += gridDim.x) {
          kv_uses = ds_cross_attn_task(a, sh, l, task, pre, kv_uses, kvbuf, scr);
          pre = false;
        }
      } else {
        // GEMV sequence index inside the layer: ph 0 -> qkv(0), 2 -> out(1), 3 -> cross_q(2), 5 -> cross_out(3), 6 -> ffn1(4), 7 -> ffn2(5)
        const int j = ph == 0 ? 0 : (ph < 4 ? ph - 1 : ph - 2);
        consumed = ds_gemv_phase<W8>(a, sh, 6 * l + j, consumed, ring, tile_stride, xs, red, kc, vc);
      }
      ds_grid_barrier(a, sh);
    }
  }
  // ---- logits = LN_f(x) E^T ----
  consumed = ds_gemv_phase<W8>(a, sh, 6 * L, consumed, ring, tile_stride, xs, red, nullptr, nullptr);
  if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) {
    a.prof[sh.prof_i] = ds_globaltimer();
    for (int k = 0; k < 8; ++k)
      for (int p2 = 0; p2 < 8; ++p2) a.prof[3000 + k * 16 + (p2 == 7 ? 15 : p2)] += sh.ticks[k * 8 + p2];
  }
}

// The same cross-attention task as a stand-alone kernel for the multi-kernel step (many chunks per call): one CTA per
// task, ~74 KB of shared memory so three CTAs per SM overlap each other's tile fetches.
__global__ void __launch_bounds__(kDsThreads) ds_cross_attn_kernel(const DStepArgs a_param, int layer) {
  extern __shared__ __align__(128) unsigned char ds_smem[];
  __shared__ DStepArgs a_sh;
  __shared__ DsShared sh;
  if (threadIdx.x == 0) {
    a_sh = a_param;
    mbar_init(&sh.kvfull, 1);
    fence_mbar_init();
  }
  __syncthreads();
  ds_cross_attn_task(a_sh, sh, layer, blockIdx.x, false, 0, ds_smem, ds_smem + kDsKvBytes);
}

// a: q, ao, bind, xpart, xcounters, H, T, d, rows_per_chunk, n_chunks
void dstep_cross_attn_launch(const DStepArgs& a, int layer, cudaStream_t s) {
  const size_t smem = kDsKvBytes + ((kDsXScratch + 127) & ~127);
  ds_cross_attn_kernel<<<ds_xtasks(a), kDsThreads, smem, s>>>(a, layer);
  B2W_LAUNCHED();
}

// ---- weight re-layout: row-major [N][K] -> stream of work-item tiles -------------------------------------------------------
__global__ void ds_pack_kernel(const __half* __restrict__ W, const float* __restrict__ bias, int K, int ksplit, __half* __restrict__ out) {
  const int item = blockIdx.x, tl = item / ksplit, ks = item - tl * ksplit;
  const int kr = K / ksplit, ld = kr + 32;
  __half* o = out + (size_t)item * (16 * ld + 32);
  for (int i = threadIdx.x; i < 16 * ld; i += blockDim.x) {
    const int r = i / ld, c = i - r * ld;
    o[i] = c < kr ? W[(size_t)(tl * 16 + r) * K + ks * kr + c] : __float2half(0.f);
  }
  float* ob = reinterpret_cast<float*>(o + 16 * ld);
  if (threadIdx.x < 16) ob[threadIdx.x] = (bias && ks == 0) ? bias[tl * 16 + threadIdx.x] : 0.f;
}

// ---- int8 weight stream: per-output-channel symmetric quantisation on the device -------------------------------------------
// One CTA per row of W[N][K]: scale = max|w| / 127; q = clamp(rint(w / scale)) stored as q + 128; W is overwritten with
// q * scale so that every other path (prefill, many-row decode) computes with exactly the weights the int8 stream encodes.
__global__ void ds_quant_rows_kernel(__half* __restrict__ W, unsigned char* __restrict__ q, float* __restrict__ scale, int K) {
  __shared__ float red[32];
  const long long row = blockIdx.x;
  __half* w = W + row * K;
  float mx = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) mx = fmaxf(mx, fabsf(__half2float(w[k])));
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  const float sc = mx > 0.f ? mx / 127.f : 1.f;
  if (threadIdx.x == 0) scale[row] = sc;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int v = max(-127, min(127, __float2int_rn(__half2float(w[k]) / sc)));
    q[row * K + k] = (unsigned char)(v + 128);
    w[k] = __float2half_rn((float)v * sc);
  }
}

__global__ void ds_pack_i8_kernel(const unsigned char* __restrict__ q, const float* __restrict__ scale, const float* __restrict__ bias, int K,
                                  int ksplit, unsigned char* __restrict__ out) {
  const int item = blockIdx.x, tl = item / ksplit, ks = item - tl * ksplit;
  const int kr = K / ksplit, ld = kr + 32;
  unsigned char* o = out + (size_t)item * (16 * ld + 128);
  for (int i = threadIdx.x; i < 16 * ld; i += blockDim.x) {
    const int r = i / ld, c = i - r * ld;
    o[i] = c < kr ? q[(size_t)(tl * 16 + r) * K + ks * kr + c] : (unsigned char)128;
  }
  float* tail = reinterpret_cast<float*>(o + 16 * ld);
  if (threadIdx.x < 16) {
    tail[threadIdx.x] = scale[tl * 16 + threadIdx.x];
    tail[16 + threadIdx.x] = (bias && ks == 0) ? bias[tl * 16 + threadIdx.x] : 0.f;
  }
}

size_t dstep_tile_halves(int kr) { return (size_t)16 * (kr + 32) + 32; }
size_t dstep_packed_halves(int N, int K, int ksplit) { return (size_t)(N / 16) * ksplit * dstep_tile_halves(K / ksplit); }
size_t dstep_packed_bytes_i8(int N, int K, int ksplit) { return (size_t)(N / 16) * ksplit * ((size_t)16 * (K / ksplit + 32) + 128); }

void dstep_pack_tiles(const __half* W, const float* bias, int N, int K, int ksplit, __half* out, cudaStream_t s) {
  B2W_CHECK(N % 16 == 0 && K % (32 * ksplit) == 0, "dstep_pack_tiles: shape");
  ds_pack_kernel<<<(N / 16) * ksplit, 256, 0, s>>>(W, bias, K, ksplit, out);
  B2W_LAUNCHED();
}

void dstep_quantize_rows(__half* W, int N, int K, unsigned char* q, float* scale, cudaStream_t s) {
  ds_quant_rows_kernel<<<N, 256, 0, s>>>(W, q, scale, K);
  B2W_LAUNCHED();
}

void dstep_pack_tiles_i8(const unsigned char* q, const float* scale, const float* bias, int N, int K, int ksplit, unsigned char* out,
                         cudaStream_t s) {
  B2W_CHECK(N % 16 == 0 && K % (32 * ksplit) == 0, "dstep_pack_tiles_i8: shape");
  ds_pack_i8_kernel<<<(N / 16) * ksplit, 256, 0, s>>>(q, scale, bias, K, ksplit, out);
  B2W_LAUNCHED();
}

size_t dstep_smem_bytes(const DStepArgs& a) {
  const size_t tile_stride = ((size_t)ds_tile_bytes(a.d, a.w8) + 127) & ~size_t(127);
  const size_t xs_bytes = (size_t)8 * (a.d + 32) * 2;
  const size_t scr = ((xs_bytes > (size_t)kDsXScratch ? xs_bytes : (size_t)kDsXScratch) + 127) & ~size_t(127);
  return kDsNBuf * tile_stride + kDsKvBytes + scr + 2 * kDsWarps * 128 * sizeof(float);
}

void dstep_configure() {
  B2W_CUDA(cudaFuncSetAttribute(dstep_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  B2W_CUDA(cudaFuncSetAttribute(dstep_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  B2W_CUDA(cudaFuncSetAttribute(ds_cross_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDsKvBytes + ((kDsXScratch + 127) & ~127)));
}

// 0 when the shape is not supported by the persistent kernel (the caller falls back to the multi-kernel step)
int dstep_max_grid(int num_sms, const DStepArgs& a) {
  const size_t smem = dstep_smem_bytes(a);
  const size_t self_scratch = (size_t)(kDsSelfKeys + 16 + 256 + 64) * sizeof(float) + (size_t)kDsSelfKeys * (72 + 64) * sizeof(__half);
  if (smem > 220 * 1024 || self_scratch > (size_t)kDsKvBytes) return 0;
  if (a.d % 64 != 0 || a.d > 1280 || a.L > 32 || a.R > 8 || num_sms < 4) return 0;
  int per_sm = 0;
  if (a.w8)
    B2W_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dstep_kernel<true>, kDsLaunchThreads, smem));
  else
    B2W_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dstep_kernel<false>, kDsLaunchThreads, smem));
  return per_sm >= 1 ? num_sms : 0;
}

void dstep_launch(const DStepArgs& a, int grid, cudaStream_t s) {
  const size_t smem = dstep_smem_bytes(a);
  B2W_CUDA(cudaMemsetAsync(a.bar, 0, sizeof(unsigned), s));
  DStepArgs copy = a;
  void* args[] = {&copy};
  void* fn = a.w8 ? reinterpret_cast<void*>(dstep_kernel<true>) : reinterpret_cast<void*>(dstep_kernel<false>);
  B2W_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kDsLaunchThreads), args, smem, s));
  count_launch();
}

// Stamps of the last step ([0] = start, then (arrive, release) of every barrier, then end) and the cycle counters at prof + 3000,
// written by dstep_kernel into a.prof; the counters are cleared after printing.
void dstep_print_profile(const DStepArgs& a, cudaStream_t s) {
  B2W_CUDA(cudaStreamSynchronize(s));
  const int L = a.L, nstamps = 1 + 2 * (1 + 8 * L) + 1;
  std::vector<unsigned long long> t(nstamps);
  B2W_CUDA(cudaMemcpy(t.data(), a.prof, nstamps * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  // work(p) = arrive_p - release_{p-1}; wait(p) = release_p - arrive_p
  static const char* names[8] = {"qkv", "self_attn", "out_proj", "cross_q", "cross_attn", "cross_out", "ffn1", "ffn2"};
  double work[8] = {0}, wait[8] = {0};
  unsigned long long prev = t[2];  // release of the embed barrier
  for (int l = 0; l < L; ++l)
    for (int ph = 0; ph < 8; ++ph) {
      const int bi = 1 + 2 * (1 + l * 8 + ph);
      work[ph] += double(t[bi] - prev);
      wait[ph] += double(t[bi + 1] - t[bi]);
      prev = t[bi + 1];
    }
  fprintf(stderr, "[dstep prof] last step: total %.1f us; embed %.1f us; logits %.1f us\n", (t[nstamps - 1] - t[0]) / 1e3,
          (t[2] - t[0]) / 1e3, (t[nstamps - 1] - prev) / 1e3);
  {
    std::vector<unsigned long long> f(8 * 16);
    B2W_CUDA(cudaMemcpy(f.data(), a.prof + 3000, f.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    B2W_CUDA(cudaMemset(a.prof + 3000, 0, f.size() * sizeof(unsigned long long)));
    static const char* kinds[7] = {"qkv", "out", "cross_q", "cross_out", "ffn1", "ffn2", "logits"};
    for (int k = 0; k < 7; ++k) {
      const double n = (double)f[k * 16 + 15];
      if (n > 0)
        fprintf(stderr, "[dstep prof]   %-9s cycles (first item): stage-input %.0f  tile-wait %.0f  mma %.0f  epilogue %.0f\n", kinds[k], f[k * 16] / n,
                f[k * 16 + 1] / n, f[k * 16 + 2] / n, f[k * 16 + 3] / n);
    }
  }
  for (int ph = 0; ph < 8; ++ph)
    fprintf(stderr, "[dstep prof]   %-10s work %.2f us  barrier wait %.2f us (CTA 0, mean over %d layers)\n", names[ph], work[ph] / L / 1e3,
            wait[ph] / L / 1e3, L);
}

}  // namespace b2w
