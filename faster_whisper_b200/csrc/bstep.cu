// One persistent, cooperative kernel per decode step for many rows: R <= 80 (BatchedInferencePipeline's 16 chunks x beam 5).
//
// At 80 rows a decode step is a chain of skinny GEMMs [R x K] x [K x N] (3-13 MB of weights each), 1600 self-attention
// (row, head) tasks over the paged self-KV cache and 2240 beam-shared cross-attention tasks that stream 3.9 GB of cross-K/V.
// As separate launches that is ~260 graph nodes; here one CTA per SM stays resident and walks
//   embed | L x { QKV, self-attn, out-proj, cross-q, cross-attn, cross-out, FFN1, GELU, FFN2 } | final LN | logits
// separated by grid barriers.  What shapes it (DESIGN.md §4):
//   * L2 -> SM bandwidth is only a small multiple of HBM bandwidth, so no phase may broadcast the [R x K] activations to
//     every CTA (205 KB x 132 per phase would cost more than the weights).  Every GEMM is therefore split over output
//     channels AND over K ("stream-K"): the weights are a stream of 16 KB atoms (128 channels x 64 K values, pre-swizzled
//     so that one 1-D TMA bulk copy lands a ready-made wgmma A tile), the atoms of a matrix are dealt out evenly to the CTAs
//     in (n-block, k-atom) order, and a CTA stages only the [R x 64] activation slices of its own k-atoms;
//   * the math is wgmma (m64 x R rows x k16 per warpgroup, fp16 in, fp32 accumulators in registers): each of the two compute
//     warpgroups multiplies its 64 channels of every atom against the staged activations;
//   * split-K partial sums meet in L2 in a fixed order, so that a step computes the same bits every run: each CTA stores its
//     [R x 128] fp32 partial tile with one bulk copy into its own slot, the CTAs of an n-block meet at a counter, and each then
//     sums a slice of the rows over the group's partials in CTA order;
//   * since no CTA ever sees a whole row of a GEMM output, everything that needs one is deferred to the consumer: the
//     LayerNorm of a residual-stream input is applied algebraically, y = rstd (W x - mean rowsum(W)) + b, with sum(x) and
//     sum(x^2) taken from the staged fp16 tiles (per k-atom, by the CTAs of n-block 0, summed in k order in the reduction); biases of
//     q/k/v/cross-q/hidden are added by the consumer; GELU gets its own (cheap, rolled) phase so that it is evaluated once per element;
//   * a weight-producer thread keeps a 5-slot ring of atoms full across phase boundaries, a K/V-producer thread double
//     buffers the cross-attention tiles; eight compute warps do the rest;
//   * the phase code runs ONCE per phase on eight warps (two per scheduler) and the ~110 KB of it cycle through a 32 KB instruction
//     cache: its cost is its instruction count.  Staging is flattened into (atom, pass) units of a handful of instructions, the atom
//     ranges are computed once per launch, wide register arrays live in leaf functions (ptxas allocates across the call graph: 40
//     registers in the GEMM phase made the self-attention loop spill), cycle counters are compiled in only with -DB2W_STEP_TICKS.
//     DESIGN.md section 4 has the measurements, including the ones that did not work (wave pipelining of independent chunks, prefetch
//     gates, a 16-lane staging, out-of-lined merges).
//
// Replaces the per-token body of CTranslate2's batched Whisper.generate loop (reference call sites
// faster_whisper/transcribe.py:222-236 driven by :580-617; SURVEY.md §2.3 rows K10-K15) for BASELINE.json configs[2..4].
#include <math.h>

#include <algorithm>

#include "bstep.h"
#include "common.cuh"
#include "dstep.h"
#include "step_common.cuh"
#include "wgmma.cuh"

namespace b2w {

constexpr int kBsThreads = 256;   // compute threads (8 warps)
constexpr int kBsLaunch = 320;    // + weight producer warp, K/V producer warp
constexpr int kBsWarps = 8;
constexpr int kBsSlots = 5;       // weight-atom ring (fp16 atoms, 16 KB each)
constexpr int kBsSlots8 = 6;      // int8 atoms (8 KB each) + two 16 KB fp16 tiles the compute warps widen them into: the same 80 KB
constexpr int kBsAtomBytes8 = 8192;
constexpr int kBsMaxSlots = 6;
constexpr int kBsKvBytes = 2 * kDsXKeysMax * 64 * 2;  // one cross-attention K + V tile (57 344 B)
constexpr int kBsXQ = 8;          // rows per chunk the cross-attention task handles
constexpr int kBsQLd = 96;
constexpr int kBsXGroups = 4;     // (chunk, head) groups one CTA's run of cross-attention tiles may touch
constexpr int kBsXScratch = kBsXGroups * kBsXQ * kBsQLd * 2 + kBsWarps * kBsXQ * 66 * 4 + 64;  // queries + per-warp partials of a piece

__host__ __device__ __forceinline__ int bs_ceil16(int v) { return (v + 15) & ~15; }

// logits: when the [R x d] fp16 activations do not fit next to the ring, adjacent CTAs split the rows in two halves and
// stream the same n-blocks (the second reader hits L2)
__host__ __device__ __forceinline__ void bs_logit_plan(int R, int d, int avail, int& nhalves, int& Rh, int& NPh) {
  nhalves = 1;
  Rh = R;
  NPh = bs_ceil16(R);
  if ((d >> 6) * NPh * 128 > avail) {
    nhalves = 2;
    Rh = (R + 1) >> 1;
    NPh = bs_ceil16(Rh);
  }
}

// ---- PTX helpers ----
__device__ __forceinline__ void bs_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void bs_bulk_store(float* gdst, const float* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bs_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bs_bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bs_bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void bs_fence_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// Atoms of one of the six matrices owned by this CTA (see bs_split); the same in every layer, computed once per launch.
struct BsRange {  // scalars only: arrays indexed at run time would live in local memory (and the L1 next to 220 KB of smem is tiny)
  int a0, a1, KA;
  int nb0, ka00, n0;  // the run's n-block, its first k-atom, its atom count
  int g0, gi, gn;     // the CTAs of n-block nb0: first CTA, this CTA's index among them, their count
};

struct BsShared {
  BLayer lay[32];
  BsRange rng[6];            // the CTA's atoms of qkv / out / cross_q / cross_out / ffn1 / ffn2
  RowInfo rows[kBsMaxRows];
  unsigned epoch;
  int prof_i;
  int flag;
  unsigned ticks[8 * 8];     // B2W_DSTEP_PROF: cycles of CTA 0 per GEMM kind: [stage, -, products + epilogue, -, sync, statistics, -, count]
  int cons;                      // ring atoms consumed so far (compute side)
  uint64_t wfull[kBsMaxSlots];   // weight atom landed (TMA complete_tx)
  uint64_t wempty[kBsMaxSlots];  // weight atom consumed (one arrival per compute warpgroup; int8 atoms: widened, compute thread 0)
  uint64_t kvfull[2];        // cross-attention K/V tile landed
  uint64_t kvfree[2];        // K/V buffer may be overwritten
};

// ---- phase numbering -------------------------------------------------------------------------------------------------------
// grid phase index: 0 embed; 1 + 9 l + {0 qkv, 1 self, 2 out, 3 cross_q, 4 cross, 5 cross_out, 6 ffn1, 7 gelu, 8 ffn2}; 1 + 9 L final LN; 2 + 9 L logits
__device__ __forceinline__ bool bs_enabled(const BStepArgs& a, int phase) { return a.stop_phase <= 0 || phase < a.stop_phase; }
// GEMM sequence s = 6 l + j (j: qkv, out, cross_q, cross_out, ffn1, ffn2) -> grid phase
__device__ __forceinline__ int bs_gemm_phase_index(int s) {
  const int l = s / 6, j = s - 6 * l;
  const int ph = j == 0 ? 0 : (j == 1 ? 2 : (j == 2 ? 3 : (j == 3 ? 5 : (j == 4 ? 6 : 8))));
  return 1 + 9 * l + ph;
}
// Atoms of GEMM s owned by this CTA.  The CTAs are dealt out to the n-blocks (as evenly as the counts allow) and the CTAs of an
// n-block split its K atoms among themselves, so a CTA's run never crosses an n-block: one accumulator, one epilogue, one partial
// tile per phase.  Needs at least as many CTAs as n-blocks (bstep_supported).
__host__ __device__ __forceinline__ void bs_split(int NB, int KA, int c, int G, int& a0, int& a1, int& idx, int& cnt) {
  const int base = G / NB, extra = G - base * NB;
  int nb;
  if (c < extra * (base + 1)) {
    nb = c / (base + 1);
    idx = c - nb * (base + 1);
    cnt = base + 1;
  } else {
    const int c2 = c - extra * (base + 1);
    nb = extra + c2 / base;
    idx = c2 - (c2 / base) * base;
    cnt = base;
  }
  // at most one CTA per k-atom: every CTA counted in a group has work, so all of them reach the group's meeting point
  if (cnt > KA) cnt = KA;
  if (idx >= cnt) {
    a0 = a1 = nb * KA;
    return;
  }
  a0 = nb * KA + KA * idx / cnt;
  a1 = nb * KA + KA * (idx + 1) / cnt;
}
__device__ __forceinline__ BsRange bs_range_compute(const BStepArgs& a, int s) {
  const int j = s % 6, d = a.d;
  const int N = j == 0 ? 3 * d : (j == 4 ? 4 * d : d);
  const int K = j == 5 ? 4 * d : d;
  BsRange r;
  r.KA = K >> 6;
  bs_split((N + 127) >> 7, r.KA, (int)blockIdx.x, (int)gridDim.x, r.a0, r.a1, r.gi, r.gn);
  r.g0 = (int)blockIdx.x - r.gi;
  r.nb0 = r.a0 / r.KA;
  r.ka00 = r.a0 - r.nb0 * r.KA;
  r.n0 = r.a1 - r.a0;
  return r;
}
__device__ __forceinline__ BsRange bs_range(const BsShared& sh, int s) { return sh.rng[s % 6]; }

// Grid barrier (compute warps only): arrive = red.release (cumulative through bar.sync), wait = relaxed polling.
__device__ __noinline__ void bs_grid_barrier(const BStepArgs& a, BsShared& sh) {
  bs_sync();
  if (threadIdx.x == 0) {
    sh.epoch += gridDim.x;
    if (a.prof && blockIdx.x == 0) a.prof[sh.prof_i] = ds_globaltimer();
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.bar) : "memory");
    const unsigned target = sh.epoch;
    unsigned v;
    do {
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.bar) : "memory");
    } while (v < target);
    if (a.prof && blockIdx.x == 0) a.prof[sh.prof_i + 1] = ds_globaltimer();
    sh.prof_i += 2;
  }
  bs_sync();
}

// ---- producer threads ------------------------------------------------------------------------------------------------------
__device__ __noinline__ void bs_weight_producer(const BStepArgs& a, BsShared& sh, unsigned char* ring) {
  int n = 0;
  const int nslots = a.w8 ? kBsSlots8 : kBsSlots;
  const uint32_t abytes = a.w8 ? kBsAtomBytes8 : kBsAtomBytes;
  auto push = [&](const unsigned char* src0, size_t index) {
    const int slot = n % nslots;
    mbar_wait(&sh.wempty[slot], (uint32_t)(((n / nslots) & 1) ^ 1));
    if (a.w8) fence_proxy_async();  // the slot was last read through the generic proxy (widening)
    mbar_expect_tx(&sh.wfull[slot], abytes);
    ds_bulk_g2s(ring + (size_t)slot * abytes, src0 + index * abytes, abytes, &sh.wfull[slot]);
    n += 1;
  };
#pragma unroll 1
  for (int s = 0; s < 6 * a.L; ++s) {
    if (!bs_enabled(a, bs_gemm_phase_index(s))) return;
    const BsRange r = bs_range(sh, s);
    const unsigned char* base = reinterpret_cast<const unsigned char*>(sh.lay[s / 6].wt[s % 6]);
#pragma unroll 1
    for (int at = r.a0; at < r.a1; ++at) push(base, (size_t)at);
  }
  if (!bs_enabled(a, 2 + 9 * a.L)) return;
  int nhalves, Rh, NPh;
  bs_logit_plan(a.R, a.d, kBsKvBytes + a.u_bytes, nhalves, Rh, NPh);
  const int groups = gridDim.x / nhalves, grp = blockIdx.x / nhalves;
  if (grp >= groups) return;
  const int KA = a.d >> 6, NBv = (a.vpad + 127) >> 7;
  const unsigned char* base = reinterpret_cast<const unsigned char*>(a.logit_atoms);
#pragma unroll 1
  for (int nb = grp; nb < NBv; nb += groups)
#pragma unroll 1
    for (int ka = 0; ka < KA; ++ka) push(base, (size_t)nb * KA + ka);
}

// cross-attention tiles (group-major: tile = (chunk * H + head) * splits + split) are dealt out as contiguous runs ("stream-K")
__device__ __forceinline__ void bs_xrange(const BStepArgs& a, int& t0, int& t1) {
  const unsigned NT = (unsigned)(kDsXSplits * a.H * a.n_chunks);
  t0 = (int)(NT * blockIdx.x / gridDim.x);
  t1 = (int)(NT * (blockIdx.x + 1) / gridDim.x);
}

// TMA the K and V tiles of one cross-attention task (key split of one (chunk, head)) into kvbuf (one thread).
__device__ __forceinline__ void bs_issue_cross_kv(const BStepArgs& a, int layer, int task, unsigned char* kvbuf, uint64_t* bar) {
  const int split = task % kDsXSplits, rest = task / kDsXSplits;
  const int h = rest % a.H, b = rest / a.H, T = a.T;
  const int k0 = T * split / kDsXSplits, k1 = T * (split + 1) / kDsXSplits, nk = k1 - k0;
  const DecBindings bd = *a.bind;
  const long long per = (long long)bd.B_total * a.H * T * 64;
  const long long off = (((long long)(bd.chunk0 + b) * a.H + h) * T + k0) * 64;
  const __half* Kb = bd.xkv + ((long long)layer * 2 + 0) * per + off;
  const __half* Vb = bd.xkv + ((long long)layer * 2 + 1) * per + off;
  fence_proxy_async();
  mbar_expect_tx(bar, (uint32_t)nk * 256u);
  ds_bulk_g2s(kvbuf, Kb, (uint32_t)nk * 128u, bar);
  ds_bulk_g2s(kvbuf + kDsXKeysMax * 128, Vb, (uint32_t)nk * 128u, bar);
}

// K/V producer: the k-th tile of this CTA's run goes to buffer k & 1.  Buffer 0 is dedicated, so the first tile
// of a layer is fetched as soon as the previous layer released it; buffer 1 lives in the multi-purpose region and is opened
// by the compute warps when the cross-attention phase starts.
__device__ __noinline__ void bs_kv_producer(const BStepArgs& a, BsShared& sh, unsigned char* kv0, unsigned char* kv1) {
  int t0, t1;
  bs_xrange(a, t0, t1);
  const int nt = t1 - t0;
  if (nt == 0) return;
  const int n_even = (nt + 1) >> 1, n_odd = nt >> 1;
#pragma unroll 1
  for (int l = 0; l < a.L; ++l) {
    if (!bs_enabled(a, 1 + 9 * l + 4)) return;
#pragma unroll 1
    for (int k = 0; k < nt; ++k) {
      const int buf = k & 1;
      if (buf == 0) {
        const int u = l * n_even + (k >> 1);
        mbar_wait(&sh.kvfree[0], (uint32_t)((u & 1) ^ 1));
      } else {
        const int u = l * n_odd + (k >> 1);
        mbar_wait(&sh.kvfree[1], (uint32_t)(u & 1));
      }
      bs_issue_cross_kv(a, l, t0 + k, buf ? kv1 : kv0, &sh.kvfull[buf]);
    }
  }
}

// ---- compute-warp phase functions ------------------------------------------------------------------------------------------
// (all out of line: the phase loop of the kernel body must not spill — with 220 KB of shared memory the L1 is ~28 KB and local
// memory lives in L2 for all practical purposes)
// The fp32 GEMM outputs (x, qkv32, cq32, h32) are stored n-block-major: element (row r, channel n) lives at
// ((n >> 7) * R + r) * 128 + (n & 127), so that the [R x 128] output tile of a GEMM segment is ONE contiguous block, like the
// partial tiles the CTAs store with one bulk copy each (bulk instructions are warp-uniform: one per row would serialise 80 issues).
__device__ __forceinline__ long long bs_bidx(int R, int r, int n) { return ((long long)(n >> 7) * R + r) * 128 + (n & 127); }

// embed: x = tok_emb[token] + pos_emb[pos] (CTA r owns row r)
__device__ __noinline__ void bs_embed_phase(const BStepArgs& a, BsShared& sh) {
  if ((int)blockIdx.x < a.R) {
    const int r = blockIdx.x, d = a.d;
    int tok = a.tokens_in[r];
    tok = tok < 0 ? 0 : (tok >= a.n_vocab ? a.n_vocab - 1 : tok);
    const int pos = sh.rows[r].pos;
    for (int i = threadIdx.x; i < d; i += kBsThreads)
      __stcg(a.x + bs_bidx(a.R, r, i), __half2float(a.tok_emb[(long long)tok * d + i]) + a.pos_emb[(long long)pos * d + i]);
  }
}

__device__ __forceinline__ void bs_row_stats(const float* st, int r, int d, float& mean, float& rstd) {
  const float2 s = __ldcg(reinterpret_cast<const float2*>(st) + r);
  mean = s.x / d;
  rstd = rsqrtf(fmaxf(s.y / d - mean * mean, 0.f) + 1e-5f);
}

// ---- staging: this CTA's activation slices as wgmma B tiles --------------------------------------------------------
// tile i = [NPw rows][64 K values] fp16, 128-byte swizzle (16-byte chunk c of row r at c ^ (r & 7)), rows beyond the last zero.
// These functions run once per GEMM run on eight warps, so their cost is their INSTRUCTION COUNT (not the rows): the work is
// flattened into units (atom, 32-row pass), G units are in flight per thread, and a unit is a handful of instructions.
__device__ __forceinline__ void bs_sts64(uint32_t addr, uint32_t v0, uint32_t v1) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v0), "r"(v1) : "memory");
}
__device__ __forceinline__ void bs_sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// atom i of the run -> k-atom: the first n0 atoms belong to the run's first segment (starting at ka00), the rest to the second
__device__ __forceinline__ int bs_atom_ka(int i, int n0, int ka00) { return i < n0 ? ka00 + i : i - n0; }

// fp32 residual stream, n-block-major -> raw fp16 (the LayerNorm is applied by the consumer of the GEMM output).  Lane c of a row's
// eight lanes loads the float4s c and 8 + c of the row's 64 values: each instruction of a warp reads whole 128-byte lines.
template <int PASSES>
__device__ __noinline__ void bs_stage_x(const float* __restrict__ x, int R, int r0, int Rw, int NPw, int natoms, int n0, int ka00, unsigned char* xs) {
  const int tid = threadIdx.x, c = tid & 7, r_lo = tid >> 3;
  constexpr int G = 9;  // 18 x 16 bytes in flight per thread
  const int row_off = (r0 + r_lo) * 128 + c * 4;          // this thread's first float inside an n-block's [R x 128] block, pass 0
  const int st_off = 8 * c;                                // its 8 bytes inside the row's first 64-byte half (before the swizzle)
  const uint32_t xs_s = smem_u32(xs);
  int li = 0, lp = 0, si = 0, sp = 0;                      // load / store cursors (atom, pass)
#pragma unroll 1
  for (int u0 = 0; u0 < natoms * PASSES; u0 += G) {
    float4 f0[G], f1[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      f0[g] = make_float4(0.f, 0.f, 0.f, 0.f);
      f1[g] = f0[g];
      if (li < natoms && r_lo + 32 * lp < Rw) {
        const int ka = bs_atom_ka(li, n0, ka00);
        const float* ptr = x + ((ka >> 1) * R + 32 * lp) * 128 + (ka & 1) * 64 + row_off;
        f0[g] = __ldcg(reinterpret_cast<const float4*>(ptr));
        f1[g] = __ldcg(reinterpret_cast<const float4*>(ptr + 32));
      }
      if (++lp == PASSES) {
        lp = 0;
        ++li;
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int r = r_lo + 32 * sp;
      if (si < natoms && r < NPw) {
        const uint32_t row = xs_s + si * (NPw * 128) + r * 128;
        const int sw = (r & 7) << 4;
        bs_sts64(row + (st_off ^ sw), pack_half2(f0[g].x, f0[g].y), pack_half2(f0[g].z, f0[g].w));
        bs_sts64(row + ((64 + st_off) ^ sw), pack_half2(f1[g].x, f1[g].y), pack_half2(f1[g].z, f1[g].w));
      }
      if (++sp == PASSES) {
        sp = 0;
        ++si;
      }
    }
  }
}

// fp16 activations [R][ld] row-major: one 16-byte chunk per unit
template <int PASSES>
__device__ __noinline__ void bs_stage_h(const __half* __restrict__ src, int ld, int r0, int Rw, int NPw, int natoms, int n0, int ka00, unsigned char* xs) {
  const int tid = threadIdx.x, c = tid & 7, r_lo = tid >> 3;
  constexpr int G = 12;
  const int row_off = (r0 + r_lo) * ld + c * 8;
  const uint32_t xs_s = smem_u32(xs);
  int li = 0, lp = 0, si = 0, sp = 0;
#pragma unroll 1
  for (int u0 = 0; u0 < natoms * PASSES; u0 += G) {
    uint4 v[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      v[g] = make_uint4(0u, 0u, 0u, 0u);
      if (li < natoms && r_lo + 32 * lp < Rw)
        v[g] = __ldcg(reinterpret_cast<const uint4*>(src + row_off + 32 * lp * ld + bs_atom_ka(li, n0, ka00) * 64));
      if (++lp == PASSES) {
        lp = 0;
        ++li;
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int r = r_lo + 32 * sp;
      if (si < natoms && r < NPw) bs_sts128(xs_s + si * (NPw * 128) + r * 128 + ((c ^ (r & 7)) << 4), v[g]);
      if (++sp == PASSES) {
        sp = 0;
        ++si;
      }
    }
  }
}

// sum(x), sum(x^2) of the rows of a residual-stream input, from the staged fp16 tiles (i.e. of exactly the values the GEMM multiplies),
// one partial per k-atom: st[ka][row][2].  The CTAs of n-block 0 stage every k-atom exactly once, so they alone write them; they also
// sum them in k order (bs_gemm_mma).
__device__ __noinline__ void bs_tile_stats(float* st, int R, int r0, int Rw, int NPw, int natoms, int ka00, const unsigned char* xs) {
  const int tid = threadIdx.x, c = tid & 7, r_lo = tid >> 3;
#pragma unroll 1
  for (int i = 0; i < natoms; ++i) {
    const int ka = ka00 + i;
    const unsigned char* tile = xs + i * (NPw * 128);
#pragma unroll 1
    for (int rb = 0; rb < NPw; rb += 32) {  // uniform trip count: the shuffles below involve whole warps
      const int r = rb + r_lo;
      float s1 = 0.f, s2 = 0.f;
      if (r < Rw) {
        const uint4 v = *reinterpret_cast<const uint4*>(tile + r * 128 + ((c ^ (r & 7)) << 4));
        const float2 a0 = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), a1 = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
        const float2 a2 = __half22float2(*reinterpret_cast<const __half2*>(&v.z)), a3 = __half22float2(*reinterpret_cast<const __half2*>(&v.w));
        s1 = ((a0.x + a0.y) + (a1.x + a1.y)) + ((a2.x + a2.y) + (a3.x + a3.y));
        s2 = ((a0.x * a0.x + a0.y * a0.y) + (a1.x * a1.x + a1.y * a1.y)) + ((a2.x * a2.x + a2.y * a2.y) + (a3.x * a3.x + a3.y * a3.y));
      }
      // the eight chunks of a row sit in eight consecutive lanes
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 4);
      s2 += __shfl_xor_sync(0xffffffffu, s2, 4);
      if (c == 0 && r < Rw) __stcg(reinterpret_cast<float2*>(st) + (long long)ka * R + r0 + r, make_float2(s1, s2));
    }
  }
}

// One weight atom of the ring against one staged activation tile: acc (+)= W[this warpgroup's 64 channels of the atom] x^T
// (all compute warps; returns once the products are complete and the ring slot is handed back).
// int8 atoms ([128 channels][64] bytes holding q + 128) are first widened by all compute warps into one of two fp16 tiles (128-byte
// swizzle): per atom a thread converts two 16-byte pieces (2 instructions per 2 weights: prmt builds 1024 + u in fp16, one hsub2
// removes 1152); the per-channel scale multiplies the fp32 accumulator in the epilogue ("per-channel dequant fused into the load
// path" of BASELINE.json configs[3]).  Two tiles suffice: a warpgroup writes tile (n + 1) & 1 only after the barrier of atom n,
// which both warpgroups reach with their products of atom n - 1 complete.
template <int NP>
__device__ __forceinline__ void bs_atom_mma(const BStepArgs& a, BsShared& sh, unsigned char* ring, int cons, uint32_t b_addr, float (&acc)[NP / 2]) {
  const int tid = threadIdx.x, wg = tid >> 7;
  uint32_t a_addr;
  int slot;
  if (a.w8) {
    slot = cons % kBsSlots8;
    mbar_wait(&sh.wfull[slot], (uint32_t)((cons / kBsSlots8) & 1));
    const unsigned char* src = ring + (size_t)slot * kBsAtomBytes8;
    unsigned char* dst = ring + (size_t)kBsSlots8 * kBsAtomBytes8 + (size_t)(cons & 1) * kBsAtomBytes;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int idx = tid + u * kBsThreads, row = idx >> 2, c4 = idx & 3;
      const uint4 w = *reinterpret_cast<const uint4*>(src + row * 64 + c4 * 16);
      const uint4 lo = make_uint4(ds_cvt_u8x2(w.x, 0x5140u), ds_cvt_u8x2(w.x, 0x5342u), ds_cvt_u8x2(w.y, 0x5140u), ds_cvt_u8x2(w.y, 0x5342u));
      const uint4 hi = make_uint4(ds_cvt_u8x2(w.z, 0x5140u), ds_cvt_u8x2(w.z, 0x5342u), ds_cvt_u8x2(w.w, 0x5140u), ds_cvt_u8x2(w.w, 0x5342u));
      *reinterpret_cast<uint4*>(dst + row * 128 + (((2 * c4) ^ (row & 7)) << 4)) = lo;
      *reinterpret_cast<uint4*>(dst + row * 128 + (((2 * c4 + 1) ^ (row & 7)) << 4)) = hi;
    }
    fence_proxy_async();
    bs_sync();
    if (tid == 0) mbar_arrive(&sh.wempty[slot]);
    a_addr = smem_u32(dst);
  } else {
    slot = cons % kBsSlots;
    mbar_wait(&sh.wfull[slot], (uint32_t)((cons / kBsSlots) & 1));
    a_addr = smem_u32(ring + (size_t)slot * kBsAtomBytes);
  }
  const uint64_t da = wgmma_desc_sw128(a_addr + wg * (64 * 128)), db = wgmma_desc_sw128(b_addr);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_ss<NP>(acc, da + 2 * k, db + 2 * k, 1);
  wgmma_commit();
  wgmma_wait<0>();
  if (!a.w8 && (tid & 127) == 0) mbar_arrive(&sh.wempty[slot]);
}

// Cycle counters of CTA 0 (B2W_DSTEP_PROF) are compiled in only with -DB2W_STEP_TICKS (python -m faster_whisper_b200.build --ticks
// builds libb200whisper_ticks.so): the phase code runs once per phase on eight warps, so every instruction of it counts, and the
// counters hold registers across loops that have none to spare.  The %globaltimer stamps at the grid barriers stay in both builds.
#ifdef B2W_STEP_TICKS
#define BS_TICK_DECL(tp) long long tp = clock64()
#define BS_TICK_COUNT(kind) do { if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) sh.ticks[(kind) * 8 + 7] += 1; } while (0)
#define BS_ATICK(kind, point, tp)                                        \
  do {                                                                   \
    if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) {                 \
      const long long _now = clock64();                                  \
      sh.ticks[(kind) * 8 + (point)] += (unsigned)(_now - (tp));         \
      (tp) = _now;                                                       \
    }                                                                    \
  } while (0)
#else
#define BS_TICK_DECL(tp) do { } while (0)
#define BS_TICK_COUNT(kind) do { } while (0)
#define BS_ATICK(kind, point, tp) do { } while (0)
#endif
#define BS_TICK(point) BS_ATICK(j, point, tp)

// Write one segment's accumulators into the fp32 staging tile [NP rows][128 channels]: y = acc * wsc + bv per channel.
template <int NP>
__device__ __forceinline__ void bs_stage_acc(const float (&acc)[NP / 2], float* stg, int c, const float (&wsc)[2], const float (&bv)[2]) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int i = 0; i < NP / 8; ++i) {
    const int r = 8 * i + 2 * t;
    stg[r * 128 + c] = fmaf(acc[4 * i], wsc[0], bv[0]);
    stg[(r + 1) * 128 + c] = fmaf(acc[4 * i + 1], wsc[0], bv[0]);
    stg[r * 128 + c + 8] = fmaf(acc[4 * i + 2], wsc[1], bv[1]);
    stg[(r + 1) * 128 + c + 8] = fmaf(acc[4 * i + 3], wsc[1], bv[1]);
  }
}

// The products of one GEMM run (one n-block segment, bstep_supported) and the fixed-order reduction of the n-block's partial tiles:
// out = sum of the group's partials in CTA order (+ the residual already in out when `resid`).  `st` (LayerNorm-consuming GEMMs):
// the CTAs of n-block 0 also sum the per-atom row statistics in k order.  A leaf function per row count: the accumulator
// registers stay out of the phase code's own live ranges.
template <int NP>
__device__ __noinline__ void bs_gemm_mma(const BStepArgs& a, BsShared& sh, const BsRange& rg, int s, unsigned char* U, unsigned char* ring,
                                         float* out, int N, const float* bias, const float* scale, bool resid, float* st) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, R = a.R;
  float acc[NP / 2];
#pragma unroll
  for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
  int cons = sh.cons;
  const uint32_t xs = smem_u32(U), xs_tile = (uint32_t)NP * 128u;
#pragma unroll 1
  for (int i = 0; i < rg.n0; ++i) bs_atom_mma<NP>(a, sh, ring, cons++, xs + i * xs_tile, acc);
  // every warpgroup's products are complete before the staging tile (which aliases the activation tiles) is written
  bs_sync();
  if (tid == 0) sh.cons = cons;
  float* stg = reinterpret_cast<float*>(U);  // [NP][128] fp32
  {
    const int c = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's channels c and c + 8 of the n-block
    float bv[2], wsc[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n_glob = rg.nb0 * 128 + c + 8 * e;
      bv[e] = (bias && rg.ka00 == 0 && n_glob < N) ? __ldg(bias + n_glob) : 0.f;
      wsc[e] = (a.w8 && n_glob < N) ? __ldg(scale + n_glob) : 1.f;
    }
    bs_stage_acc<NP>(acc, stg, c, wsc, bv);
  }
  fence_proxy_async();
  bs_sync();
  if (tid == 0) {  // rows 0 .. R-1 of the staging tile -> this CTA's partial slot; then meet the n-block's other CTAs
    bs_bulk_store(a.gpart + (long long)blockIdx.x * R * 128, stg, (uint32_t)R * 512u);
    bs_bulk_commit();
    bs_bulk_wait_all();
    bs_fence_async_all();
    unsigned* cnt = a.bar + 64 + (s % 6) * 64 + rg.nb0;  // counts up through the layers: the same groups meet once per layer
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(cnt), "r"(1u) : "memory");
    const unsigned target = (unsigned)((s / 6 + 1) * rg.gn);
    unsigned v;
    do {
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(cnt) : "memory");
    } while (v < target);
    asm volatile("fence.acq_rel.gpu;" ::: "memory");  // acquire: the group's partial tiles and statistics are read after this
  }
  bs_sync();
  const int r0 = R * rg.gi / rg.gn, r1 = R * (rg.gi + 1) / rg.gn;  // this CTA's rows of the sum
  const float* p0 = a.gpart + (long long)rg.g0 * R * 128;
  float* o = out + (long long)rg.nb0 * R * 128;
#pragma unroll 1
  for (int i = r0 * 32 + tid; i < r1 * 32; i += kBsThreads) {
    float4 t = __ldcg(reinterpret_cast<const float4*>(p0) + i);
#pragma unroll 1
    for (int k = 1; k < rg.gn; ++k) {
      const float4 u = __ldcg(reinterpret_cast<const float4*>(p0 + (long long)k * R * 128) + i);
      t = make_float4(t.x + u.x, t.y + u.y, t.z + u.z, t.w + u.w);
    }
    if (resid) {
      const float4 x = __ldcg(reinterpret_cast<const float4*>(o) + i);
      t = make_float4(x.x + t.x, x.y + t.y, x.z + t.z, x.w + t.w);
    }
    __stcg(reinterpret_cast<float4*>(o) + i, t);
  }
  if (st && rg.nb0 == 0) {
    const float2* sp = reinterpret_cast<const float2*>(a.stpart);
#pragma unroll 1
    for (int r = r0 + tid; r < r1; r += kBsThreads) {
      float2 t = __ldcg(sp + r);
#pragma unroll 1
      for (int ka = 1; ka < rg.KA; ++ka) {
        const float2 u = __ldcg(sp + (long long)ka * R + r);
        t = make_float2(t.x + u.x, t.y + u.y);
      }
      __stcg(reinterpret_cast<float2*>(st) + r, t);
    }
  }
}

// One GEMM phase (compute warps): stage -> row statistics -> products -> fixed-order reduction of the split-K partials.
__device__ __noinline__ void bs_gemm_phase(const BStepArgs& a, BsShared& sh, int s, unsigned char* U, unsigned char* ring) {
  const BsRange rg = bs_range(sh, s);
  if (rg.a1 <= rg.a0) return;
  const int l = s / 6, j = s - 6 * l, d = a.d;
  BS_TICK_DECL(tp);
  const BLayer& lay = sh.lay[l];
  {
    const int natoms = rg.a1 - rg.a0;
    if (j == 0 || j == 2 || j == 4) {  // fp32 residual stream
      if (a.NP <= 64) bs_stage_x<2>(a.x, a.R, 0, a.R, a.NP, natoms, rg.n0, rg.ka00, U);
      else bs_stage_x<3>(a.x, a.R, 0, a.R, a.NP, natoms, rg.n0, rg.ka00, U);
    } else {
      const __half* src = j == 5 ? a.h16 : a.ao;
      const int ld = j == 5 ? 4 * d : d;
      if (a.NP <= 64) bs_stage_h<2>(src, ld, 0, a.R, a.NP, natoms, rg.n0, rg.ka00, U);
      else bs_stage_h<3>(src, ld, 0, a.R, a.NP, natoms, rg.n0, rg.ka00, U);
    }
  }
  float* out = j == 0 ? a.qkv32 : (j == 2 ? a.cq32 : (j == 4 ? a.h32 : a.x));
  const int N = j == 0 ? 3 * d : (j == 4 ? 4 * d : d);
  const float* bias = (j == 1 || j == 3 || j == 5) ? lay.bias[j] : nullptr;
  BS_TICK(0);
  fence_proxy_async();
  bs_sync();
  BS_TICK(4);
  const bool ln_input = j == 0 || j == 2 || j == 4;  // a residual-stream input: LayerNorm statistics of its rows (n-block 0's CTAs)
  if (ln_input && rg.nb0 == 0) bs_tile_stats(a.stpart, a.R, 0, a.R, a.NP, rg.a1 - rg.a0, rg.ka00, U);
  float* st = ln_input ? a.stats + (long long)(3 * l + (j >> 1)) * a.R * 2 : nullptr;
  const bool resid = !ln_input;  // out-proj, cross-out and FFN2 add into the residual stream
  BS_TICK(5);
  switch (a.NP) {
    case 16: bs_gemm_mma<16>(a, sh, rg, s, U, ring, out, N, bias, lay.scale[j], resid, st); break;
    case 32: bs_gemm_mma<32>(a, sh, rg, s, U, ring, out, N, bias, lay.scale[j], resid, st); break;
    case 48: bs_gemm_mma<48>(a, sh, rg, s, U, ring, out, N, bias, lay.scale[j], resid, st); break;
    case 64: bs_gemm_mma<64>(a, sh, rg, s, U, ring, out, N, bias, lay.scale[j], resid, st); break;
    default: bs_gemm_mma<80>(a, sh, rg, s, U, ring, out, N, bias, lay.scale[j], resid, st); break;
  }
  BS_TICK(2);
  BS_TICK_COUNT(j);
}

// Masked self-attention: one (row, head) task per warp.  q, k, v of the new token come from the raw QKV sums (deferred LayerNorm +
// bias applied here); k and v are rounded to fp16 and written to the paged cache.  The history is gathered through the beam
// ancestry table in blocks of 16 keys with an online softmax.  The K and V rows of a block are copied into the warp's own
// shared-memory tile with cp.async — COALESCED: eight lanes copy the eight 16-byte chunks of one 128-byte row, so an instruction
// touches 4 cache lines, not 32 — and double buffered: the copies of block b + 1 are in flight while block b is scored.  With only
// eight compute warps per SM this is what keeps enough bytes in flight (registers cannot: 64 data registers per block spill).
constexpr int kBsSelfTile = 2 * 2 * 16 * 64 * 2;  // per warp: two buffers x (K + V) x 16 keys x 64 halves = 8 KB
__device__ __noinline__ void bs_self_attn_phase(const BStepArgs& a, BsShared& sh, int l, unsigned char* U) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int d = a.d, H = a.H, n_ctx = a.n_ctx;
  __half* tiles = reinterpret_cast<__half*>(U + (size_t)warp * kBsSelfTile);  // [buf][K|V][16 keys][64]; 16-byte chunks at chunk ^ (key & 7)
  __half* qs = reinterpret_cast<__half*>(U + (size_t)kBsWarps * kBsSelfTile) + warp * 64;  // the task's query, fp16, pre-scaled by 1/8
  const int g = lane >> 2, t = lane & 3;
  const BLayer& lay = sh.lay[l];
  const float* st = a.stats + (long long)(3 * l) * a.R * 2;
  __half* kc = a.kcache + (long long)l * a.kv_layer_stride;
  __half* vc = a.vcache + (long long)l * a.kv_layer_stride;
  const int ntasks = H * a.R, e0 = 2 * lane;
  const int pos_stride = a.slots * d;  // elements between consecutive positions of a chunk
  const int crow = lane >> 3, cchunk = lane & 7;  // copy role: row (of four per instruction) and 16-byte chunk
  const int task0 = blockIdx.x * kBsWarps + warp, tstride = gridDim.x * kBsWarps;
#pragma unroll 1
  for (int task = task0; task < ntasks; task += tstride) {
    const int r = task / H, h = task - r * H;
    const RowInfo ri = sh.rows[r];
    const int pos = ri.pos;
    BS_TICK_DECL(tp);
    const uint8_t* anc = a.anc + (pos & 1) * a.anc_buf_stride + ((long long)ri.chunk * a.slots + ri.slot) * n_ctx;
    uint32_t slots[4] = {0u, 0u, 0u, 0u};  // lane holds the slot byte of key 32 i + lane for i < 14 (n_ctx <= 448)
#pragma unroll
    for (int i = 0; i < 14; ++i) {
      const int jj = 32 * i + lane;
      const uint32_t sv = (jj < pos) ? (uint32_t)__ldg(anc + jj) : 0u;
      slots[i >> 2] |= sv << (8 * (i & 3));
    }
    float mean, rstd;
    bs_row_stats(st, r, d, mean, rstd);
    const float2 rq = __ldcg(reinterpret_cast<const float2*>(a.qkv32 + bs_bidx(a.R, r, h * 64 + e0))),
                 rk = __ldcg(reinterpret_cast<const float2*>(a.qkv32 + bs_bidx(a.R, r, d + h * 64 + e0))),
                 rv = __ldcg(reinterpret_cast<const float2*>(a.qkv32 + bs_bidx(a.R, r, 2 * d + h * 64 + e0)));
    const float* ws = lay.wsum[0] + h * 64 + e0;
    const float* bs = lay.bias[0] + h * 64 + e0;
    const float2 wq = __ldg(reinterpret_cast<const float2*>(ws)), wk = __ldg(reinterpret_cast<const float2*>(ws + d)),
                 wv = __ldg(reinterpret_cast<const float2*>(ws + 2 * d));
    const float2 bq = __ldg(reinterpret_cast<const float2*>(bs)), bk = __ldg(reinterpret_cast<const float2*>(bs + d)),
                 bvv = __ldg(reinterpret_cast<const float2*>(bs + 2 * d));
    const long long chunk_off = (long long)ri.chunk * n_ctx * pos_stride + h * 64;
    const __half* kbase = kc + chunk_off;
    const __half* vbase = vc + chunk_off;
    const int nblk = (pos + 15) >> 4;
    // copies of block b into buffer b & 1 (keys 16 b + crow + 4 i, i < 4); one commit group per block
    auto issue = [&](int b) {
      __half* kd = tiles + (b & 1) * (2 * 16 * 64);
      __half* vd = kd + 16 * 64;
      const int w32 = b >> 1;  // which 32-key group holds the slot bytes
      const uint32_t word = (w32 >> 2) == 0 ? slots[0] : ((w32 >> 2) == 1 ? slots[1] : ((w32 >> 2) == 2 ? slots[2] : slots[3]));
      const uint32_t mine = (word >> (8 * (w32 & 3))) & 255u;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int key = crow + 4 * i, j = 16 * b + key;
        const int sj = (int)__shfl_sync(0xffffffffu, mine, 16 * (b & 1) + key);
        if (j < pos) {
          const int off = j * pos_stride + sj * d + cchunk * 8;  // elements; < 2^31 for every supported shape
          ds_cp_async16(kd + key * 64 + ((cchunk ^ (key & 7)) << 3), kbase + off);
          ds_cp_async16(vd + key * 64 + ((cchunk ^ (key & 7)) << 3), vbase + off);
        }
      }
      ds_cp_commit();
    };
    __syncwarp();  // the previous task's tiles and query are no longer being read
    if (nblk > 0) issue(0);
    const float mr = mean * rstd;
#define BS_FIX(raw_, w_, b_) fmaf(rstd, raw_, fmaf(-mr, w_, b_))
    // q is rounded to fp16 like the other decode paths (they store q as fp16); the 1/8 scale is exact in fp16
    const __half2 q16 = __hmul2(__floats2half2_rn(BS_FIX(rq.x, wq.x, bq.x), BS_FIX(rq.y, wq.y, bq.y)), __floats2half2_rn(0.125f, 0.125f));
    const __half2 k16 = __floats2half2_rn(BS_FIX(rk.x, wk.x, bk.x), BS_FIX(rk.y, wk.y, bk.y));
    const __half2 v16 = __floats2half2_rn(BS_FIX(rv.x, wv.x, bvv.x), BS_FIX(rv.y, wv.y, bvv.y));
#undef BS_FIX
    const float2 qf = __half22float2(q16), kf = __half22float2(k16), vf = __half22float2(v16);
    const long long self_off = chunk_off + (long long)pos * pos_stride + ri.slot * d + e0;
    *reinterpret_cast<__half2*>(kc + self_off) = k16;
    *reinterpret_cast<__half2*>(vc + self_off) = v16;
    *reinterpret_cast<__half2*>(qs + e0) = q16;
    // online-softmax state, seeded with the new token's own key (p = 1): m uniform over the warp; the running sum and the output
    // accumulators follow the m16n8 accumulator layout, whose row 0 (lanes 0-3) is the only real query
    float m_run = warp_sum(qf.x * kf.x + qf.y * kf.y);
    float l_part = lane == 0 ? 1.f : 0.f;
    float oacc[8][4];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {  // dims 8 dt + 2 t, + 1 of v sit in lane 4 dt + t of the "lane = 2 dims" layout
      const float ox = __shfl_sync(0xffffffffu, vf.x, 4 * dt + t), oy = __shfl_sync(0xffffffffu, vf.y, 4 * dt + t);
      oacc[dt][0] = g == 0 ? ox : 0.f;
      oacc[dt][1] = g == 0 ? oy : 0.f;
      oacc[dt][2] = oacc[dt][3] = 0.f;
    }
    __syncwarp();
    uint4 qa = make_uint4(0u, 0u, 0u, 0u), qb = make_uint4(0u, 0u, 0u, 0u);  // A fragments of S = q K^T (k-permuted chunks t, 4 + t)
    if (g == 0) {
      qa = *reinterpret_cast<const uint4*>(qs + 8 * t);
      qb = *reinterpret_cast<const uint4*>(qs + 32 + 8 * t);
    }
    BS_ATICK(6, 0, tp);
#pragma unroll 1
    for (int b = 0; b < nblk; ++b) {
      if (b + 1 < nblk) {
        issue(b + 1);
        asm volatile("cp.async.wait_group 1;" ::: "memory");
      } else {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      }
      __syncwarp();
      BS_ATICK(6, 2, tp);
      const __half* kt = tiles + (b & 1) * (2 * 16 * 64);
      __half* vt = tiles + (b & 1) * (2 * 16 * 64) + 16 * 64;
      const int nvalid = min(16, pos - 16 * b);
      if (nvalid < 16) {  // rows that were not copied are multiplied by zero probabilities: make them finite
        for (int i = lane; i < (16 - nvalid) * 8; i += 32) *reinterpret_cast<uint4*>(vt + (nvalid + (i >> 3)) * 64 + (i & 7) * 8) = make_uint4(0u, 0u, 0u, 0u);
        __syncwarp();
      }
      // ---- S = q K^T: two n8 tiles (keys g and 8 + g), 16-byte k-permuted fragments ----
      float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
      {
        const int sw = g;  // (key & 7) of both rows
        const uint4 ka = *reinterpret_cast<const uint4*>(kt + g * 64 + ((t ^ sw) << 3));
        const uint4 kb4 = *reinterpret_cast<const uint4*>(kt + g * 64 + (((4 + t) ^ sw) << 3));
        const uint4 kc4 = *reinterpret_cast<const uint4*>(kt + (8 + g) * 64 + ((t ^ sw) << 3));
        const uint4 kd = *reinterpret_cast<const uint4*>(kt + (8 + g) * 64 + (((4 + t) ^ sw) << 3));
        ds_mma(s0, qa.x, 0u, qa.y, 0u, ka.x, ka.y);
        ds_mma(s0, qa.z, 0u, qa.w, 0u, ka.z, ka.w);
        ds_mma(s0, qb.x, 0u, qb.y, 0u, kb4.x, kb4.y);
        ds_mma(s0, qb.z, 0u, qb.w, 0u, kb4.z, kb4.w);
        ds_mma(s1, qa.x, 0u, qa.y, 0u, kc4.x, kc4.y);
        ds_mma(s1, qa.z, 0u, qa.w, 0u, kc4.z, kc4.w);
        ds_mma(s1, qb.x, 0u, qb.y, 0u, kd.x, kd.y);
        ds_mma(s1, qb.z, 0u, qb.w, 0u, kd.z, kd.w);
      }
      // lanes 0-3 (row 0): keys 2 t, 2 t + 1 (s0[0..1]) and 8 + 2 t, 9 + 2 t (s1[0..1]) of the block
      const bool row0 = g == 0;
      const float v00 = (row0 && 2 * t < nvalid) ? s0[0] : -INFINITY, v01 = (row0 && 2 * t + 1 < nvalid) ? s0[1] : -INFINITY;
      const float v10 = (row0 && 8 + 2 * t < nvalid) ? s1[0] : -INFINITY, v11 = (row0 && 9 + 2 * t < nvalid) ? s1[1] : -INFINITY;
      float mx = fmaxf(fmaxf(v00, v01), fmaxf(v10, v11));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      mx = __shfl_sync(0xffffffffu, mx, 0);
      const float m_new = fmaxf(m_run, mx);
      const float alpha = __expf(m_run - m_new);
      const __half2 p0 = __floats2half2_rn(__expf(v00 - m_new), __expf(v01 - m_new)), p1 = __floats2half2_rn(__expf(v10 - m_new), __expf(v11 - m_new));
      const float2 pf0 = __half22float2(p0), pf1 = __half22float2(p1);
      l_part = fmaf(l_part, alpha, (pf0.x + pf0.y) + (pf1.x + pf1.y));
      m_run = m_new;
      const uint32_t pa0 = *reinterpret_cast<const uint32_t*>(&p0), pa2 = *reinterpret_cast<const uint32_t*>(&p1);
      // ---- O (+)= P V: B = V via ldmatrix.trans (16 keys x 8 dims per tile) ----
      const int mi = lane >> 3, r8 = lane & 7;
      const int vkey = 8 * (mi & 1) + r8;
#pragma unroll
      for (int dp = 0; dp < 4; ++dp) {
        uint32_t b0, b1, b2, b3;
        ds_ldmatrix_x4_trans(b0, b1, b2, b3, vt + vkey * 64 + (((2 * dp + (mi >> 1)) ^ (vkey & 7)) << 3));
        oacc[2 * dp][0] *= alpha;
        oacc[2 * dp][1] *= alpha;
        oacc[2 * dp + 1][0] *= alpha;
        oacc[2 * dp + 1][1] *= alpha;
        ds_mma(oacc[2 * dp], pa0, 0u, pa2, 0u, b0, b1);
        ds_mma(oacc[2 * dp + 1], pa0, 0u, pa2, 0u, b2, b3);
      }
      __syncwarp();  // the buffer may be refilled by the copies issued in the next iteration
      BS_ATICK(6, 3, tp);
      BS_TICK_COUNT(6);
    }
    float l_run = l_part;
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
    if (g == 0) {
      const float inv = 1.f / l_run;
      __half* o = a.ao + (long long)r * d + h * 64 + 2 * t;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) *reinterpret_cast<uint32_t*>(o + 8 * dt) = pack_half2(oacc[dt][0] * inv, oacc[dt][1] * inv);
    }
  }
}

// Beam-shared cross attention, stream-K over key tiles.  The 1500 keys of a (chunk, head) group are 7 tiles of ~214 keys; all
// tiles of the step form one sequence (group-major) that is cut into equal contiguous runs, one per CTA.  A CTA walks its run with
// an online softmax: scores S = K Q^T and O^T = V^T P^T on mma.sync from the XOR-swizzled K/V tile (as dstep.cu), running max /
// sum per query in shared memory, output accumulators in registers across the tiles of a group.  A group that lies entirely inside
// one run is written straight to `ao`; a group cut by a run boundary leaves one partial record per piece and the piece that
// completes the group (ticket = tiles done) merges them.  With 16 chunks a run is ~15 tiles: two groups whole, two cut.
__device__ __forceinline__ bool bs_piece_starts_at(int t, unsigned NT) {  // is tile t the first tile of some CTA's run?
  const unsigned G = gridDim.x;
  const unsigned c = ((unsigned)(t + 1) * G + NT - 1) / NT - 1;
  return (int)(NT * c / G) == t;
}

__device__ __noinline__ void bs_cross_attn_phase(const BStepArgs& a, BsShared& sh, int l, unsigned char* kv0, unsigned char* U) {
  int t0, t1;
  bs_xrange(a, t0, t1);
  const int nt = t1 - t0;
  if (nt == 0) return;
  const int n_even = (nt + 1) >> 1, n_odd = nt >> 1;
  const int T = a.T, S = kDsXSplits, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int nq = a.rows_per_chunk, d = a.d;
  const unsigned NT = (unsigned)(S * a.H * a.n_chunks);
  unsigned char* kv1 = U;
  unsigned char* scratch = U + kBsKvBytes;
  __half* qs_all = reinterpret_cast<__half*>(scratch);                          // [kBsXGroups][8][96], pre-scaled by 1/8
  float* mb = reinterpret_cast<float*>(qs_all + kBsXGroups * kBsXQ * kBsQLd);  // [8 warps][8 queries][64 + m + l]
  const BLayer& lay = sh.lay[l];
  BS_TICK_DECL(tp0);
  if (lane == 0 && nt > 1) mbar_arrive(&sh.kvfree[1]);  // the multi-purpose region is free for K/V tiles now (one arrival per warp)
  // ---- queries of every group this run touches, in one round trip (deferred LayerNorm + bias, fp16 rounding, then the exact 1/8) ----
  const int g_first = t0 / S, n_groups = (t1 - 1) / S - g_first + 1;
  for (int idx = tid; idx < n_groups * 64; idx += kBsThreads) {
    const int gi = idx >> 6, q = (idx & 63) >> 3, c = idx & 7;
    const int grp = g_first + gi, h = grp % a.H, b = grp / a.H;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (q < nq) {
      const int r = b * nq + q;
      float mean, rstd;
      bs_row_stats(a.stats + (long long)(3 * l + 1) * a.R * 2, r, d, mean, rstd);
      const float mr = mean * rstd;
      const float* raw = a.cq32 + bs_bidx(a.R, r, h * 64 + c * 8);
      const float* ws = lay.wsum[1] + h * 64 + c * 8;
      const float* bs = lay.bias[2] + h * 64 + c * 8;
      const float4 r0 = __ldcg(reinterpret_cast<const float4*>(raw)), r1 = __ldcg(reinterpret_cast<const float4*>(raw) + 1);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(ws)), w1 = __ldg(reinterpret_cast<const float4*>(ws) + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bs)), b1 = __ldg(reinterpret_cast<const float4*>(bs) + 1);
#define BS_FIX(raw_, w_, b_) fmaf(rstd, raw_, fmaf(-mr, w_, b_))
      __half2 hq[4] = {__floats2half2_rn(BS_FIX(r0.x, w0.x, b0.x), BS_FIX(r0.y, w0.y, b0.y)), __floats2half2_rn(BS_FIX(r0.z, w0.z, b0.z), BS_FIX(r0.w, w0.w, b0.w)),
                       __floats2half2_rn(BS_FIX(r1.x, w1.x, b1.x), BS_FIX(r1.y, w1.y, b1.y)), __floats2half2_rn(BS_FIX(r1.z, w1.z, b1.z), BS_FIX(r1.w, w1.w, b1.w))};
#undef BS_FIX
      const __half2 sc8 = __floats2half2_rn(0.125f, 0.125f);
#pragma unroll
      for (int i = 0; i < 4; ++i) hq[i] = __hmul2(hq[i], sc8);
      v = make_uint4(*reinterpret_cast<uint32_t*>(&hq[0]), *reinterpret_cast<uint32_t*>(&hq[1]), *reinterpret_cast<uint32_t*>(&hq[2]), *reinterpret_cast<uint32_t*>(&hq[3]));
    }
    *reinterpret_cast<uint4*>(qs_all + (gi * kBsXQ + q) * kBsQLd + c * 8) = v;
  }
  bs_sync();
  BS_ATICK(7, 3, tp0);  // prologue: queries staged
  // per-thread state of the current piece: query row g (the accumulator rows g + 8 are padding), this warp's share of the keys
  float m_run = -INFINITY, l_run = 0.f;
  float oacc[8][4];
  uint4 qf0 = make_uint4(0u, 0u, 0u, 0u), qf1 = make_uint4(0u, 0u, 0u, 0u);
  int piece_first = 0;
  unsigned early_cnt = 0u;  // thread 0: the piece counter of the group the run ends in, requested one tile ahead
#pragma unroll 1
  for (int k = 0; k < nt; ++k) {
    const int tile = t0 + k, grp = tile / S, split = tile - grp * S, gi = grp - g_first;
    const int buf = k & 1;
    unsigned char* kvbuf = buf ? kv1 : kv0;
    const int u = l * (buf ? n_odd : n_even) + (k >> 1);
    const int k0 = T * split / S, k1 = T * (split + 1) / S, nk = k1 - k0;
    const __half* kt = reinterpret_cast<const __half*>(kvbuf);  // [224][64], 16-byte chunks at chunk ^ (encoder position & 7)
    __half* vt = reinterpret_cast<__half*>(kvbuf) + kDsXKeysMax * 64;
    if (k == 0 || split == 0) {  // a new piece starts
      piece_first = split;
      m_run = -INFINITY;
      l_run = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f;
      const __half* qs = qs_all + (gi * kBsXQ + g) * kBsQLd;  // k-permuted A fragments: 16-byte chunk 4 c2 + t of query row g
      qf0 = *reinterpret_cast<const uint4*>(qs + 8 * t);
      qf1 = *reinterpret_cast<const uint4*>(qs + 32 + 8 * t);
    }
    BS_TICK_DECL(tp);
    if (k == nt - 1 && tid == 0 && split != S - 1)  // the run ends inside this group: if it holds the first split it will merge the group
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(early_cnt) : "l"(a.xcounters + grp) : "memory");
    mbar_wait(&sh.kvfull[buf], (uint32_t)(u & 1));
    BS_ATICK(7, 0, tp);
    const int ngroups16 = (nk + 15) >> 4;
    {
      // this warp's keys of the tile: the 16-key groups `warp` and `warp + 8` (14 groups per tile), processed together so that the two
      // score chains, the softmax update and the two P V steps overlap
      const int kbA = warp * 16, kbB = (warp + 8) * 16;
      const bool hasA = warp < ngroups16, hasB = warp + 8 < ngroups16;
      const int kb_last = (ngroups16 - 1) * 16;
      if ((hasB ? kbB : kbA) == kb_last && kb_last + 16 > nk) {  // the tail rows of V are multiplied by zero probabilities: make them finite
        for (int i = lane; i < (kb_last + 16 - nk) * 8; i += 32) *reinterpret_cast<uint4*>(vt + (nk + (i >> 3)) * 64 + (i & 7) * 8) = make_uint4(0u, 0u, 0u, 0u);
        __syncwarp();
      }
      // ---- S = Q K^T: rows = queries (g), columns = keys (two n8 tiles per group); 16-byte k-permuted fragments ----
      float sA0[4] = {0.f, 0.f, 0.f, 0.f}, sA1[4] = {0.f, 0.f, 0.f, 0.f}, sB0[4] = {0.f, 0.f, 0.f, 0.f}, sB1[4] = {0.f, 0.f, 0.f, 0.f};
      if (hasA) {
        const int key0 = kbA + g, key1 = kbA + 8 + g;
        const int sw0 = (k0 + key0) & 7, sw1 = (k0 + key1) & 7;
        const uint4 ka = *reinterpret_cast<const uint4*>(kt + key0 * 64 + ((t ^ sw0) << 3));
        const uint4 kb4 = *reinterpret_cast<const uint4*>(kt + key0 * 64 + (((4 + t) ^ sw0) << 3));
        const uint4 kc4 = *reinterpret_cast<const uint4*>(kt + key1 * 64 + ((t ^ sw1) << 3));
        const uint4 kd = *reinterpret_cast<const uint4*>(kt + key1 * 64 + (((4 + t) ^ sw1) << 3));
        ds_mma(sA0, qf0.x, 0u, qf0.y, 0u, ka.x, ka.y);
        ds_mma(sA1, qf0.x, 0u, qf0.y, 0u, kc4.x, kc4.y);
        ds_mma(sA0, qf0.z, 0u, qf0.w, 0u, ka.z, ka.w);
        ds_mma(sA1, qf0.z, 0u, qf0.w, 0u, kc4.z, kc4.w);
        ds_mma(sA0, qf1.x, 0u, qf1.y, 0u, kb4.x, kb4.y);
        ds_mma(sA1, qf1.x, 0u, qf1.y, 0u, kd.x, kd.y);
        ds_mma(sA0, qf1.z, 0u, qf1.w, 0u, kb4.z, kb4.w);
        ds_mma(sA1, qf1.z, 0u, qf1.w, 0u, kd.z, kd.w);
      }
      if (hasB) {
        const int key0 = kbB + g, key1 = kbB + 8 + g;
        const int sw0 = (k0 + key0) & 7, sw1 = (k0 + key1) & 7;
        const uint4 ka = *reinterpret_cast<const uint4*>(kt + key0 * 64 + ((t ^ sw0) << 3));
        const uint4 kb4 = *reinterpret_cast<const uint4*>(kt + key0 * 64 + (((4 + t) ^ sw0) << 3));
        const uint4 kc4 = *reinterpret_cast<const uint4*>(kt + key1 * 64 + ((t ^ sw1) << 3));
        const uint4 kd = *reinterpret_cast<const uint4*>(kt + key1 * 64 + (((4 + t) ^ sw1) << 3));
        ds_mma(sB0, qf0.x, 0u, qf0.y, 0u, ka.x, ka.y);
        ds_mma(sB1, qf0.x, 0u, qf0.y, 0u, kc4.x, kc4.y);
        ds_mma(sB0, qf0.z, 0u, qf0.w, 0u, ka.z, ka.w);
        ds_mma(sB1, qf0.z, 0u, qf0.w, 0u, kc4.z, kc4.w);
        ds_mma(sB0, qf1.x, 0u, qf1.y, 0u, kb4.x, kb4.y);
        ds_mma(sB1, qf1.x, 0u, qf1.y, 0u, kd.x, kd.y);
        ds_mma(sB0, qf1.z, 0u, qf1.w, 0u, kb4.z, kb4.w);
        ds_mma(sB1, qf1.z, 0u, qf1.w, 0u, kd.z, kd.w);
      }
      if (hasA) {  // (a warp without keys in this tile keeps its state untouched)
        // thread (g, t): query g, keys kb + 2t, kb + 2t + 1 (s*0[0..1]) and kb + 8 + 2t, + 1 (s*1[0..1]) of each group
        const float a00 = (kbA + 2 * t < nk) ? sA0[0] : -INFINITY, a01 = (kbA + 2 * t + 1 < nk) ? sA0[1] : -INFINITY;
        const float a10 = (kbA + 8 + 2 * t < nk) ? sA1[0] : -INFINITY, a11 = (kbA + 9 + 2 * t < nk) ? sA1[1] : -INFINITY;
        const float b00 = (hasB && kbB + 2 * t < nk) ? sB0[0] : -INFINITY, b01 = (hasB && kbB + 2 * t + 1 < nk) ? sB0[1] : -INFINITY;
        const float b10 = (hasB && kbB + 8 + 2 * t < nk) ? sB1[0] : -INFINITY, b11 = (hasB && kbB + 9 + 2 * t < nk) ? sB1[1] : -INFINITY;
        float mx = fmaxf(fmaxf(fmaxf(a00, a01), fmaxf(a10, a11)), fmaxf(fmaxf(b00, b01), fmaxf(b10, b11)));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run, mx);
        const float alpha = __expf(m_run - m_new);  // 0 for the first keys of a piece (m_run = -inf, m_new finite: group A always holds a real key)
        const __half2 pA0 = __floats2half2_rn(__expf(a00 - m_new), __expf(a01 - m_new)), pA1 = __floats2half2_rn(__expf(a10 - m_new), __expf(a11 - m_new));
        const __half2 pB0 = __floats2half2_rn(__expf(b00 - m_new), __expf(b01 - m_new)), pB1 = __floats2half2_rn(__expf(b10 - m_new), __expf(b11 - m_new));
        const float2 fA0 = __half22float2(pA0), fA1 = __half22float2(pA1), fB0 = __half22float2(pB0), fB1 = __half22float2(pB1);
        // l_run is this thread's share of the row sum (its own keys); the four t-lanes are added when the piece is written out
        l_run = fmaf(l_run, alpha, ((fA0.x + fA0.y) + (fA1.x + fA1.y)) + ((fB0.x + fB0.y) + (fB1.x + fB1.y)));
        m_run = m_new;
        const uint32_t paA0 = *reinterpret_cast<const uint32_t*>(&pA0), paA2 = *reinterpret_cast<const uint32_t*>(&pA1);
        const uint32_t paB0 = *reinterpret_cast<const uint32_t*>(&pB0), paB2 = *reinterpret_cast<const uint32_t*>(&pB1);
        // ---- O (+)= P V: A = P (rows = queries, 16 keys per group), B = V via ldmatrix.trans (keys x 8 dims per tile) ----
        const int mi = lane >> 3, r8 = lane & 7;
        const int vkA = kbA + 8 * (mi & 1) + r8, vswA = (k0 + vkA) & 7;
        const int vkB = kbB + 8 * (mi & 1) + r8, vswB = (k0 + vkB) & 7;
#pragma unroll
        for (int dp = 0; dp < 4; ++dp) {
          uint32_t b0, b1, b2, b3;
          ds_ldmatrix_x4_trans(b0, b1, b2, b3, vt + vkA * 64 + (((2 * dp + (mi >> 1)) ^ vswA) << 3));
          oacc[2 * dp][0] *= alpha;
          oacc[2 * dp][1] *= alpha;
          oacc[2 * dp + 1][0] *= alpha;
          oacc[2 * dp + 1][1] *= alpha;
          ds_mma(oacc[2 * dp], paA0, 0u, paA2, 0u, b0, b1);
          ds_mma(oacc[2 * dp + 1], paA0, 0u, paA2, 0u, b2, b3);
          if (hasB) {
            ds_ldmatrix_x4_trans(b0, b1, b2, b3, vt + vkB * 64 + (((2 * dp + (mi >> 1)) ^ vswB) << 3));
            ds_mma(oacc[2 * dp], paB0, 0u, paB2, 0u, b0, b1);
            ds_mma(oacc[2 * dp + 1], paB0, 0u, paB2, 0u, b2, b3);
          }
        }
      }
    }
    const bool piece_ends = (k == nt - 1 || split == S - 1);
    if (piece_ends) {  // this warp's partial of the piece: accumulators relative to its own running max
      float* w = mb + (warp * kBsXQ + g) * 66;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) *reinterpret_cast<float2*>(w + 8 * dt + 2 * t) = make_float2(oacc[dt][0], oacc[dt][1]);
      float lr = l_run;  // the four t-lanes of a query row hold disjoint shares of the row sum
      lr += __shfl_xor_sync(0xffffffffu, lr, 1);
      lr += __shfl_xor_sync(0xffffffffu, lr, 2);
      if (t == 0) {
        w[64] = m_run;
        w[65] = lr;
      }
    }
    // release the tile (one arrival per warp): buffer 0 always, buffer 1 only when another tile of this phase will use it
    __syncwarp();
    if (lane == 0 && (buf == 0 || k + 2 < nt)) mbar_arrive(&sh.kvfree[buf]);
    BS_ATICK(7, 1, tp);
    BS_TICK_COUNT(7);
    if (!piece_ends) continue;
    bs_sync();
    const int h = grp % a.H, b = grp / a.H, row0 = b * nq;
    const int n_piece = split - piece_first + 1;
    float* part = a.xpart + ((long long)grp * S + piece_first) * (kBsXQ * 66);
    // merge the eight warps' partials (flash-decoding combine); a whole group goes straight to `ao`, a cut one leaves a record
    for (int i = tid; i < nq * 66; i += kBsThreads) {
      const int q = i / 66, e = i - q * 66;
      float M = -INFINITY;
#pragma unroll
      for (int w8 = 0; w8 < kBsWarps; ++w8) M = fmaxf(M, mb[(w8 * kBsXQ + q) * 66 + 64]);
      float den = 0.f, num = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < kBsWarps; ++w8) {
        const float* wrow = mb + (w8 * kBsXQ + q) * 66;
        const float wgt = (wrow[64] == -INFINITY) ? 0.f : __expf(wrow[64] - M);
        den = fmaf(wgt, wrow[65], den);
        num = fmaf(wgt, wrow[e < 64 ? e : 0], num);
      }
      if (n_piece == S) {
        if (e < 64) a.ao[(long long)(row0 + q) * d + h * 64 + e] = __float2half_rn(num / den);
      } else {
        __stcg(part + q * 66 + e, e < 64 ? num : (e == 64 ? M : den));
      }
    }
    if (n_piece != S) {
      // A cut group is merged by the piece that holds its FIRST split.  The runs are walked in tile order and start together, so
      // that piece is the last thing its CTA does, while the group's other pieces open the runs of the following CTAs and were
      // recorded a whole run earlier: those only post their record (a release add, no round trip), and the merger's poll finds the
      // count complete.  (Previously every piece took a ticket — an atomic round trip at the START of a run, on the critical path of
      // every CTA — and whoever came last merged.)
      bs_sync();
      const bool merger = piece_first == 0;
      unsigned* cnt = reinterpret_cast<unsigned*>(a.xcounters + grp);
      if (!merger) {
        if (tid == 0) asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(cnt), "r"((unsigned)n_piece) : "memory");
      } else {  // merge the pieces (their first splits are where some CTA's run starts, or 0)
        if (tid == 0) {
          // `early_cnt` was requested before this tile was processed: normally it already shows the count complete, and no
          // round trip is spent on polling (the records are then read AFTER the count was seen complete, as the ordering requires)
          unsigned v = early_cnt;
          while (v < (unsigned)(S - n_piece)) asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(cnt) : "memory");
          asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(cnt), "r"(0u) : "memory");  // next use: the next layer, a grid barrier away
        }
        bs_sync();
        const float* pg = a.xpart + (long long)grp * S * (kBsXQ * 66);
        unsigned present = 1u;
        for (int s2 = 1; s2 < S; ++s2) present |= bs_piece_starts_at(grp * S + s2, NT) ? (1u << s2) : 0u;
#pragma unroll 1
        for (int i = tid; i < nq * 64; i += kBsThreads) {
          const int q = i >> 6, e = i & 63;
          float pm[8], pl[8], pa[8];
#pragma unroll
          for (int s2 = 0; s2 < 8; ++s2) {
            const bool on = s2 < S && ((present >> s2) & 1u);
            const float* base = pg + ((on ? s2 : 0) * kBsXQ + q) * 66;
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
            const float wgt = (pm[s2] == -INFINITY) ? 0.f : __expf(pm[s2] - M);
            num = fmaf(wgt, pa[s2], num);
            den = fmaf(wgt, pl[s2], den);
          }
          a.ao[(long long)(row0 + q) * d + h * 64 + e] = __float2half_rn(num / den);
        }
      }
    }
    bs_sync();  // the per-warp partials are reused by the next piece
    BS_ATICK(7, 2, tp);
  }
}

// h16 = GELU(rstd (h32 - mean rowsum(W1)) + b1), evaluated once per element; h32 is zeroed for the next layer's sums.
// A thread keeps ONE column group (4 channels: folded row sum and bias loaded once) and walks the rows with a stride, the next
// row's loads in flight while the current one is evaluated: one index division per run, a rolled loop, ~200 instructions instead of
// the 900 of an unrolled version (this runs once per layer: its cost is its instruction count).
__device__ __noinline__ void bs_gelu_phase(const BStepArgs& a, BsShared& sh, int l) {
  const int d = a.d, R = a.R, wr0 = 0, r_end = R;
  const BLayer& lay = sh.lay[l];
  const float2* st = reinterpret_cast<const float2*>(a.stats + (long long)(3 * l + 2) * R * 2);
  const int gtid = blockIdx.x * kBsThreads + threadIdx.x, per_row = d;  // float4 units per row of 4d
  const int rstride = (gridDim.x * kBsThreads) / per_row;               // rows one sweep of the grid covers (>= 1: grid >= 8 CTAs, d <= 1280)
  const int rr = gtid / per_row, n = (gtid - rr * per_row) * 4;
  if (rr < rstride) {
    const float4 ws = __ldg(reinterpret_cast<const float4*>(lay.wsum[2] + n)), bb = __ldg(reinterpret_cast<const float4*>(lay.bias[4] + n));
    int r = wr0 + rr;
    float4 hv = make_float4(0.f, 0.f, 0.f, 0.f);
    float2 sv = make_float2(0.f, 0.f);
    if (r < r_end) {
      hv = __ldcg(reinterpret_cast<const float4*>(a.h32 + bs_bidx(R, r, n)));
      sv = __ldcg(st + r);
    }
#pragma unroll 1
    while (r < r_end) {
      const int rn = r + rstride;
      float4 hn = hv;
      float2 sn = sv;
      if (rn < r_end) {  // the next row's loads fly while this one is evaluated
        hn = __ldcg(reinterpret_cast<const float4*>(a.h32 + bs_bidx(R, rn, n)));
        sn = __ldcg(st + rn);
      }
      const float mean = sv.x / d;
      const float rstd = rsqrtf(fmaxf(sv.y / d - mean * mean, 0.f) + 1e-5f);
      const float mr = mean * rstd;
      const float y0 = gelu_erf(fmaf(rstd, hv.x, fmaf(-mr, ws.x, bb.x))), y1 = gelu_erf(fmaf(rstd, hv.y, fmaf(-mr, ws.y, bb.y)));
      const float y2 = gelu_erf(fmaf(rstd, hv.z, fmaf(-mr, ws.z, bb.z))), y3 = gelu_erf(fmaf(rstd, hv.w, fmaf(-mr, ws.w, bb.w)));
      *reinterpret_cast<uint2*>(a.h16 + (long long)r * 4 * d + n) = make_uint2(pack_half2(y0, y1), pack_half2(y2, y3));
      hv = hn;
      sv = sn;
      r = rn;
    }
  }
}

// xn16[r] = (x[r] - mean) * rstd  (CTA r; the final LayerNorm's affine part is folded into the output embedding)
__device__ __noinline__ void bs_final_ln_phase(const BStepArgs& a, float* red) {
  const int r = blockIdx.x, d = a.d, tid = threadIdx.x;
  if (r >= a.R) return;
  const int n4 = d >> 2;
  float4 v[2];
  float su = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = tid + i * kBsThreads;
    v[i] = idx < n4 ? __ldcg(reinterpret_cast<const float4*>(a.x + bs_bidx(a.R, r, idx * 4))) : make_float4(0.f, 0.f, 0.f, 0.f);
    su += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  su = warp_sum(su);
  if ((tid & 31) == 0) red[tid >> 5] = su;
  bs_sync();
  su = 0.f;
#pragma unroll
  for (int i = 0; i < kBsWarps; ++i) su += red[i];
  const float mean = su / d;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = tid + i * kBsThreads;
    if (idx < n4) {
      const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
      sq += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
  }
  sq = warp_sum(sq);
  bs_sync();
  if ((tid & 31) == 0) red[tid >> 5] = sq;
  bs_sync();
  sq = 0.f;
#pragma unroll
  for (int i = 0; i < kBsWarps; ++i) sq += red[i];
  const float rstd = rsqrtf(sq / d + 1e-5f);
  uint2* o = reinterpret_cast<uint2*>(a.xn16 + (long long)r * d);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = tid + i * kBsThreads;
    if (idx < n4)
      o[idx] = make_uint2(pack_half2((v[i].x - mean) * rstd, (v[i].y - mean) * rstd), pack_half2((v[i].z - mean) * rstd, (v[i].w - mean) * rstd));
  }
}

// logits of the n-blocks grp, grp + groups, ... for the staged rows [r_lo, r_lo + r_n): full K per n-block, direct fp32 stores
template <int NPH>
__device__ __noinline__ void bs_logits_mma(const BStepArgs& a, BsShared& sh, unsigned char* xs_logits, unsigned char* ring, int grp, int groups, int r_lo, int r_n) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, t = lane & 3;
  const int KA = a.d >> 6, NBv = (a.vpad + 127) >> 7;
  const int c = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
  int cons = sh.cons;
#pragma unroll 1
  for (int nb = grp; nb < NBv; nb += groups) {
    float acc[NPH / 2];
#pragma unroll
    for (int i = 0; i < NPH / 2; ++i) acc[i] = 0.f;
#pragma unroll 1
    for (int ka = 0; ka < KA; ++ka) bs_atom_mma<NPH>(a, sh, ring, cons++, smem_u32(xs_logits) + ka * (uint32_t)NPH * 128u, acc);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int vidx = nb * 128 + c + 8 * e;
      if (vidx >= a.vpad) continue;
      const float bv = __ldg(a.logit_bias + vidx);
      const float wsc = a.w8 ? __ldg(a.logit_scale + vidx) : 1.f;
#pragma unroll
      for (int i = 0; i < NPH / 8; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rr = 8 * i + 2 * t + h;
          if (rr < r_n) a.logits[(long long)(r_lo + rr) * a.vpad + vidx] = fmaf(acc[4 * i + 2 * e + h], wsc, bv);
        }
      }
    }
  }
}

// logits[r][v] = xn16[r] . E'[v] + b[v]: whole n-blocks (full K) per CTA group, direct fp32 stores
__device__ __noinline__ void bs_logits_phase(const BStepArgs& a, BsShared& sh, unsigned char* xs_logits, unsigned char* ring) {
  int nhalves, Rh, NPh;
  bs_logit_plan(a.R, a.d, kBsKvBytes + a.u_bytes, nhalves, Rh, NPh);
  const int groups = gridDim.x / nhalves, grp = blockIdx.x / nhalves, half = blockIdx.x % nhalves;
  if (grp >= groups) return;
  const int tid = threadIdx.x;
  const int d = a.d, KA = d >> 6;
  const int r_lo = half * Rh, r_n = min(a.R - r_lo, Rh);
  {  // stage all K of the rows [r_lo, r_lo + r_n): tile ka = [NPh][64]
    const int per_atom = NPh * 8, total = KA * per_atom;
    for (int q = tid; q < total; q += kBsThreads) {
      const int ka = q / per_atom, rem = q - ka * per_atom, r = rem >> 3, c = rem & 7;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (r < r_n) v = __ldcg(reinterpret_cast<const uint4*>(a.xn16 + (long long)(r_lo + r) * d + ka * 64 + c * 8));
      *reinterpret_cast<uint4*>(xs_logits + ka * (NPh * 128) + r * 128 + ((c ^ (r & 7)) << 4)) = v;
    }
  }
  fence_proxy_async();
  bs_sync();
  switch (NPh) {
    case 16: bs_logits_mma<16>(a, sh, xs_logits, ring, grp, groups, r_lo, r_n); break;
    case 32: bs_logits_mma<32>(a, sh, xs_logits, ring, grp, groups, r_lo, r_n); break;
    case 48: bs_logits_mma<48>(a, sh, xs_logits, ring, grp, groups, r_lo, r_n); break;
    case 64: bs_logits_mma<64>(a, sh, xs_logits, ring, grp, groups, r_lo, r_n); break;
    default: bs_logits_mma<80>(a, sh, xs_logits, ring, grp, groups, r_lo, r_n); break;
  }
}

__global__ void __launch_bounds__(kBsLaunch, 1) bstep_kernel(const BStepArgs a_param) {
  extern __shared__ unsigned char bs_smem_raw[];
  __shared__ BStepArgs a_sh;
  __shared__ BsShared sh;
  __shared__ float red[kBsWarps];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(bs_smem_raw) + 1023) & ~uintptr_t(1023));
  if (threadIdx.x == 0) a_sh = a_param;
  __syncthreads();
  const BStepArgs& a = a_sh;
  unsigned char* ring = smem;
  unsigned char* kv0 = ring + (size_t)kBsSlots * kBsAtomBytes;
  unsigned char* U = kv0 + kBsKvBytes;
  const int L = a.L;
  {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(a.layers);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(sh.lay);
    for (int i = threadIdx.x; i < L * (int)(sizeof(BLayer) / 8); i += kBsLaunch) dst[i] = src[i];
    if (threadIdx.x < a.R) sh.rows[threadIdx.x] = a.rows[threadIdx.x];
    if (threadIdx.x == 0) {
      sh.epoch = 0;
      sh.prof_i = 1;
      for (int i = 0; i < 8 * 8; ++i) sh.ticks[i] = 0;
      for (int i = 0; i < kBsMaxSlots; ++i) {
        mbar_init(&sh.wfull[i], 1);
        mbar_init(&sh.wempty[i], a.w8 ? 1 : 2);
      }
      sh.cons = 0;
      for (int j = 0; j < 6; ++j) sh.rng[j] = bs_range_compute(a, j);
      for (int i = 0; i < 2; ++i) {
        mbar_init(&sh.kvfull[i], 1);
        mbar_init(&sh.kvfree[i], kBsWarps);  // every compute warp releases a K/V buffer on its own
      }
      fence_mbar_init();
      if (a.prof && blockIdx.x == 0) a.prof[0] = ds_globaltimer();
    }
  }
  __syncthreads();

  if (threadIdx.x >= kBsThreads) {
    if (threadIdx.x == kBsThreads) bs_weight_producer(a, sh, ring);
    if (threadIdx.x == kBsThreads + 32) bs_kv_producer(a, sh, kv0, U);
  } else {
    int phase = 0;  // grid phases executed so far
    bs_embed_phase(a, sh);
    bool run = bs_enabled(a, ++phase);  // phase 0 done after the barrier; `phase` is the index of the next one
    bs_grid_barrier(a, sh);
#pragma unroll 1
    for (int l = 0; l < L && run; ++l) {
#pragma unroll 1
      for (int ph = 0; ph < 9 && run; ++ph) {
        switch (ph) {
          case 0: bs_gemm_phase(a, sh, 6 * l + 0, U, ring); break;
          case 1: bs_self_attn_phase(a, sh, l, U); break;
          case 2: bs_gemm_phase(a, sh, 6 * l + 1, U, ring); break;
          case 3: bs_gemm_phase(a, sh, 6 * l + 2, U, ring); break;
          case 4: bs_cross_attn_phase(a, sh, l, kv0, U); break;
          case 5: bs_gemm_phase(a, sh, 6 * l + 3, U, ring); break;
          case 6: bs_gemm_phase(a, sh, 6 * l + 4, U, ring); break;
          case 7: bs_gelu_phase(a, sh, l); break;
          default: bs_gemm_phase(a, sh, 6 * l + 5, U, ring); break;
        }
        run = bs_enabled(a, ++phase);
        bs_grid_barrier(a, sh);
      }
    }
    if (run) {
      bs_final_ln_phase(a, red);
      run = bs_enabled(a, ++phase);
      bs_grid_barrier(a, sh);
    }
    if (run) bs_logits_phase(a, sh, kv0, ring);
    if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) {
      a.prof[sh.prof_i] = ds_globaltimer();
      for (int k = 0; k < 8; ++k)
        for (int p2 = 0; p2 < 8; ++p2) a.prof[3000 + k * 16 + (p2 == 7 ? 15 : p2)] += sh.ticks[k * 8 + p2];
    }
  }
}

// ---- weight re-layout ------------------------------------------------------------------------------------------------------
// One thread per 16-byte chunk of an atom: atom (nb, ka), row i (channel nb*128 + i), chunk c (k = ka*64 + 8c .. +8) is stored at
// byte i*128 + ((c ^ (i & 7)) << 4) — the 128-byte-swizzled K-major layout wgmma reads (and TMA would write).
__global__ void bs_pack_atoms_kernel(const __half* __restrict__ W, int N, int K, uint4* __restrict__ out) {
  const int KA = K >> 6;
  const long long total = (long long)((N + 127) >> 7) * KA * 1024;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long atom = idx >> 10;
    const int w = (int)(idx & 1023), i = w >> 3, c = w & 7;
    const int nb = (int)(atom / KA), ka = (int)(atom - (long long)nb * KA);
    const int n = nb * 128 + i;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (n < N) v = *reinterpret_cast<const uint4*>(W + (long long)n * K + ka * 64 + c * 8);
    out[atom * 1024 + i * 8 + (c ^ (i & 7))] = v;
  }
}
__global__ void bs_row_sums_kernel(const __half* __restrict__ W, int N, int K, float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  const __half2* w = reinterpret_cast<const __half2*>(W + (long long)row * K);
  float s = 0.f;
  for (int k = lane; k < (K >> 1); k += 32) {
    const float2 f = __half22float2(w[k]);
    s += f.x + f.y;
  }
  s = warp_sum(s);
  if (lane == 0) out[row] = s;
}

// int8 atoms: [128 channels][64 K] bytes, row-major (the widening pass applies the swizzle); rows beyond N hold 128 (= zero)
__global__ void bs_pack_atoms_i8_kernel(const unsigned char* __restrict__ q, int N, int K, uint4* __restrict__ out) {
  const int KA = K >> 6;
  const long long total = (long long)((N + 127) >> 7) * KA * 512;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long atom = idx >> 9;
    const int w = (int)(idx & 511), i = w >> 2, c = w & 3;
    const int nb = (int)(atom / KA), ka = (int)(atom - (long long)nb * KA);
    const int n = nb * 128 + i;
    uint4 v = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
    if (n < N) v = *reinterpret_cast<const uint4*>(q + (long long)n * K + ka * 64 + c * 16);
    out[idx] = v;
  }
}
__global__ void bs_row_sums_i8_kernel(const unsigned char* __restrict__ q, const float* __restrict__ scale, int N, int K, float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  const unsigned char* w = q + (long long)row * K;
  int s = 0;
  for (int k = lane; k < K; k += 32) s += (int)w[k] - 128;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[row] = (float)s * scale[row];
}

size_t bstep_atoms_bytes_i8(int N, int K) { return (size_t)((N + 127) / 128) * (K / 64) * kBsAtomBytes8; }
void bstep_pack_atoms_i8(const unsigned char* q, int N, int K, unsigned char* out, cudaStream_t s) {
  B2W_CHECK(K % 64 == 0 && N % 8 == 0, "bstep_pack_atoms_i8: shape");
  bs_pack_atoms_i8_kernel<<<1024, 256, 0, s>>>(q, N, K, reinterpret_cast<uint4*>(out));
  B2W_LAUNCHED();
}
void bstep_row_sums_i8(const unsigned char* q, const float* scale, int N, int K, float* out, cudaStream_t s) {
  bs_row_sums_i8_kernel<<<ceil_div(N, 8), 256, 0, s>>>(q, scale, N, K, out);
  B2W_LAUNCHED();
}

size_t bstep_atoms_bytes(int N, int K) { return (size_t)((N + 127) / 128) * (K / 64) * kBsAtomBytes; }

void bstep_pack_atoms(const __half* W, int N, int K, __half* out, cudaStream_t s) {
  B2W_CHECK(K % 64 == 0 && N % 8 == 0, "bstep_pack_atoms: shape");
  bs_pack_atoms_kernel<<<1024, 256, 0, s>>>(W, N, K, reinterpret_cast<uint4*>(out));
  B2W_LAUNCHED();
}
void bstep_row_sums(const __half* W, int N, int K, float* out, cudaStream_t s) {
  bs_row_sums_kernel<<<ceil_div(N, 8), 256, 0, s>>>(W, N, K, out);
  B2W_LAUNCHED();
}

static size_t bstep_smem_bytes(const BStepArgs& a) { return (size_t)kBsSlots * kBsAtomBytes + kBsKvBytes + (size_t)a.u_bytes + 1024; }

// dynamic + static shared memory of a CTA is capped at 227 KB (232 448 B) on sm_90
static int bstep_max_dynamic_smem() {
  cudaFuncAttributes fa;
  B2W_CUDA(cudaFuncGetAttributes(&fa, bstep_kernel));
  return 232448 - (int)fa.sharedSizeBytes;
}

void bstep_configure() { B2W_CUDA(cudaFuncSetAttribute(bstep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bstep_max_dynamic_smem())); }

int bstep_phase_count(int L) { return 3 + 9 * L; }

size_t bstep_xpart_floats(const BStepArgs& a) { return (size_t)a.n_chunks * a.H * kDsXSplits * kBsXQ * 66; }

bool bstep_supported(int num_sms, BStepArgs& a) {
  if (a.R < 1 || a.R > kBsMaxRows || a.d % 64 != 0 || a.d > 1280 || a.d != 64 * a.H || a.L > 32 || a.rows_per_chunk > kBsXQ || num_sms < 8) return false;
  if ((a.T + kDsXSplits - 1) / kDsXSplits + 1 > kDsXKeysMax || a.vpad % 4 != 0 || a.n_ctx > 448) return false;
  {  // a CTA's run of cross-attention tiles may touch at most kBsXGroups (chunk, head) groups
    const int NT = kDsXSplits * a.H * a.n_chunks, run = (NT + num_sms - 1) / num_sms;
    if ((run + kDsXSplits - 1) / kDsXSplits + 1 > kBsXGroups) return false;
  }
  a.NP = bs_ceil16(a.R);
  const int d = a.d, G = num_sms;
  // activation tiles of the busiest GEMM phase (an even share of the atoms, rounded up) and the condition for two segments
  int max_atoms = 1;
  const int Ns[3] = {3 * d, 4 * d, d}, Ks[3] = {d, d, 4 * d};
  for (int i = 0; i < 3; ++i) {
    const int KA = Ks[i] / 64, NB = (Ns[i] + 127) / 128;
    if (G < NB) return false;  // every n-block needs a CTA of its own: a CTA's run stays inside one n-block
    for (int c = 0; c < G; ++c) {
      int a0, a1, gi, gn;
      bs_split(NB, KA, c, G, a0, a1, gi, gn);
      max_atoms = std::max(max_atoms, a1 - a0);
    }
  }
  size_t u = (size_t)max_atoms * a.NP * 128;
  u = std::max(u, (size_t)a.NP * 512);                                                       // fp32 staging tile of the partial tile
  u = std::max(u, (size_t)kBsKvBytes + ((kBsXScratch + 127) & ~127));                        // second K/V tile + cross-attention scratch
  u = std::max(u, (size_t)kBsWarps * (kBsSelfTile + 64 * 2));                                // self-attention: K/V tiles + query per warp
  a.u_bytes = (int)((u + 1023) & ~size_t(1023));
  int nhalves, Rh, NPh;
  bs_logit_plan(a.R, d, kBsKvBytes + a.u_bytes, nhalves, Rh, NPh);
  if ((size_t)(d / 64) * NPh * 128 > (size_t)kBsKvBytes + a.u_bytes) return false;
  const size_t smem = bstep_smem_bytes(a);
  if (smem > (size_t)bstep_max_dynamic_smem()) return false;
  int per_sm = 0;
  B2W_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bstep_kernel, kBsLaunch, smem));
  return per_sm >= 1;
}

void bstep_launch(const BStepArgs& a, int grid, cudaStream_t s) {
  const size_t smem = bstep_smem_bytes(a);
  B2W_CUDA(cudaMemsetAsync(a.bar, 0, kBsBarWords * sizeof(unsigned), s));  // grid barrier + the n-block group counters
  BStepArgs copy = a;
  void* args[] = {&copy};
  B2W_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(bstep_kernel), dim3(grid), dim3(kBsLaunch), args, smem, s));
  count_launch();
}

}  // namespace b2w
