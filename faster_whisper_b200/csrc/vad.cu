// Silero VAD v6 (16 kHz) on the GPU, fp32 throughout (faster_whisper_b200/silero.py states the graph):
//   vad_window_kernel      per window, parallel: PCM -> 576-sample input -> reflect pad -> STFT magnitude (frames 1..4)
//                          -> 4 x conv+ReLU -> LSTM input projection Gx[n][512] = W_ih x + b_ih + b_hh
//   vad_recurrence_kernel  the LSTM over all windows of a block in one launch: one cluster of 4 CTAs per stream slice, each
//                          CTA owning 32 hidden units (their 4 x 32 rows of W_hh live in registers); h goes to every CTA of the
//                          cluster through DSMEM, one cluster barrier per step; clusters never wait for each other
//   vad_decoder_kernel     per window, parallel: p = sigmoid(w . relu(h) + b)
// A launch serves several independent audio streams: its windows are the concatenation of one slice per stream (VadSlice), and
// a window's arithmetic does not depend on where in the launch it lands, so every stream gets the bits it gets alone.
// No TF32 or fp16: a probability is compared with thresholds, so error becomes a moved speech boundary.
#include "vad.h"

namespace b2w {

constexpr int kWin = 512, kCtx = 64, kIn = kWin + kCtx, kPad = 128, kPadded = kIn + 2 * kPad;  // 832
constexpr int kBins = 129, kFrames = 4, kHidden = 128, kGates = 4 * kHidden;
constexpr int kTile = 16;      // windows per CTA of the window kernel
constexpr int kThreads = 256;  // threads of the window kernel
// shared memory of the window kernel: two ping-pong activation buffers
constexpr int kBufA = kTile * kPadded;           // input [16][832], later conv0 [16][128][4], conv2 [16][64]
constexpr int kBufB = kTile * kBins * kFrames;   // magnitude [16][129][4], later conv1 [16][64][2], conv3 [16][128]
constexpr size_t kWindowSmem = (size_t)(kBufA + kBufB) * sizeof(float);
static_assert(kTile * 128 * 4 <= kBufA && kTile * 64 * 2 <= kBufB && kTile * 128 <= kBufB, "activation buffers");

// out[w][co][t] = relu(b[co] + sum_{ci,k} W[co][ci][k] in[w][ci][t*S + k - 1]) with wt = W transposed to [ci*3 + k][co]:
// thread = (output channel, group of windows); each weight is read once per CTA (coalesced over co) and used for every
// window and position of the group, the inputs come from shared memory as broadcasts.
template <int CIN, int COUT, int LIN, int S>
static __device__ __forceinline__ void conv_relu(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ wt,
                                          const float* __restrict__ bias) {
  constexpr int LOUT = (LIN - 1) / S + 1;
  constexpr int GROUPS = kThreads / COUT, WPG = kTile / GROUPS;
  const int co = threadIdx.x % COUT, w0 = (threadIdx.x / COUT) * WPG;
  float acc[WPG][LOUT];
#pragma unroll
  for (int w = 0; w < WPG; ++w)
#pragma unroll
    for (int t = 0; t < LOUT; ++t) acc[w][t] = 0.f;
  for (int ci = 0; ci < CIN; ++ci) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float wv = __ldg(wt + (ci * 3 + k) * COUT + co);
#pragma unroll
      for (int t = 0; t < LOUT; ++t) {
        const int p = t * S + k - 1;
        if (p < 0 || p >= LIN) continue;  // zero padding (compile-time)
#pragma unroll
        for (int w = 0; w < WPG; ++w) acc[w][t] = fmaf(wv, in[((w0 + w) * CIN + ci) * LIN + p], acc[w][t]);
      }
    }
  }
  const float b = __ldg(bias + co);
#pragma unroll
  for (int w = 0; w < WPG; ++w)
#pragma unroll
    for (int t = 0; t < LOUT; ++t) out[((w0 + w) * COUT + co) * LOUT + t] = fmaxf(acc[w][t] + b, 0.f);
}

// The slice holding window n of the launch (slices are in window order and none is empty).
static __device__ __forceinline__ int vad_find_slice(const VadSlice* __restrict__ slices, int n_slices, int n) {
  int lo = 0, hi = n_slices - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&slices[mid].w0) <= n) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads) vad_window_kernel(VadWeights wts, const float* __restrict__ pcm,
                                                              const VadSlice* __restrict__ slices, int n_slices, int nb,
                                                              float* __restrict__ gx) {
  extern __shared__ float smem[];
  __shared__ int64_t win_pcm[kTile];  // where window w of the tile starts in pcm (its 64 context samples first), -1: none
  __shared__ int win_flags[kTile];    // 1: context is zero (the stream's first window), 2: tail is zero (its last window)
  float* A = smem;
  float* B = smem + kBufA;
  const int n0 = blockIdx.x * kTile;
  if (threadIdx.x < kTile) {
    const int n = n0 + threadIdx.x;
    int64_t at = -1;
    int flags = 0;
    if (n < nb) {
      const VadSlice sl = slices[vad_find_slice(slices, n_slices, n)];
      const int k = n - sl.w0;
      at = sl.pcm0 + (int64_t)k * kWin;
      flags = (sl.first && k == 0 ? 1 : 0) | (sl.last && k == sl.nb - 1 ? 2 : 0);
    }
    win_pcm[threadIdx.x] = at;
    win_flags[threadIdx.x] = flags;
  }
  __syncthreads();
  // 1. inputs: window k of a slice is pcm[pcm0 + k*512 .. + 576) (a slice's pcm starts with the 64 samples before it),
  //    reflect-padded by 128; the context of a stream's first window is zero, and so are the final 64 samples of its last
  //    window (SileroVADModel zeroes them in place)
  static_assert(kTile % (kThreads / 32) == 0, "whole windows per warp");
  for (int w = threadIdx.x >> 5; w < kTile; w += kThreads / 32) {  // a warp per window: its slice entry is read once
    const int64_t at = win_pcm[w];
    const int fl = win_flags[w];
    for (int j = threadIdx.x & 31; j < kPadded; j += 32) {
      int s = j - kPad;
      s = s < 0 ? -s : (s >= kIn ? 2 * (kIn - 1) - s : s);
      const bool zero = at < 0 || ((fl & 1) && s < kCtx) || ((fl & 2) && s >= kIn - kCtx);
      A[w * kPadded + j] = zero ? 0.f : pcm[at + s];
    }
  }
  __syncthreads();
  // 2. STFT magnitude: bin b of frames 1..4 (frame 0 is dropped) for half of the tile's windows per item
  for (int item = threadIdx.x; item < 2 * kBins; item += kThreads) {
    const int b = item % kBins, w0 = (item / kBins) * (kTile / 2);
    float re[kTile / 2][kFrames], im[kTile / 2][kFrames];
#pragma unroll
    for (int w = 0; w < kTile / 2; ++w)
#pragma unroll
      for (int f = 0; f < kFrames; ++f) re[w][f] = im[w][f] = 0.f;
    for (int k = 0; k < 256; ++k) {
      const float cr = __ldg(wts.basis_t + k * 258 + b), ci = __ldg(wts.basis_t + k * 258 + kBins + b);
#pragma unroll
      for (int w = 0; w < kTile / 2; ++w)
#pragma unroll
        for (int f = 0; f < kFrames; ++f) {
          const float x = A[(w0 + w) * kPadded + 128 * (f + 1) + k];
          re[w][f] = fmaf(cr, x, re[w][f]);
          im[w][f] = fmaf(ci, x, im[w][f]);
        }
    }
#pragma unroll
    for (int w = 0; w < kTile / 2; ++w)
#pragma unroll
      for (int f = 0; f < kFrames; ++f) B[((w0 + w) * kBins + b) * kFrames + f] = sqrtf(re[w][f] * re[w][f] + im[w][f] * im[w][f]);
  }
  __syncthreads();
  // 3. the four conv + ReLU layers: [129][4] -> [128][4] -> [64][2] -> [64][1] -> [128][1]
  conv_relu<129, 128, 4, 1>(B, A, wts.conv_t[0], wts.conv_b[0]);
  __syncthreads();
  conv_relu<128, 64, 4, 2>(A, B, wts.conv_t[1], wts.conv_b[1]);
  __syncthreads();
  conv_relu<64, 64, 2, 2>(B, A, wts.conv_t[2], wts.conv_b[2]);
  __syncthreads();
  conv_relu<64, 128, 1, 1>(A, B, wts.conv_t[3], wts.conv_b[3]);
  __syncthreads();
  // 4. LSTM input projection: gate rows r and r + 256 for all windows of the tile
  const int r = threadIdx.x;
  float acc0[kTile], acc1[kTile];
#pragma unroll
  for (int w = 0; w < kTile; ++w) acc0[w] = acc1[w] = 0.f;
  for (int k = 0; k < kHidden; ++k) {
    const float w0v = __ldg(wts.w_ih_t + k * kGates + r), w1v = __ldg(wts.w_ih_t + k * kGates + r + 256);
#pragma unroll
    for (int w = 0; w < kTile; ++w) {
      const float x = B[w * kHidden + k];
      acc0[w] = fmaf(w0v, x, acc0[w]);
      acc1[w] = fmaf(w1v, x, acc1[w]);
    }
  }
  const float b0 = __ldg(wts.b_gates + r), b1 = __ldg(wts.b_gates + r + 256);
#pragma unroll
  for (int w = 0; w < kTile; ++w)
    if (n0 + w < nb) {
      gx[(int64_t)(n0 + w) * kGates + r] = acc0[w] + b0;
      gx[(int64_t)(n0 + w) * kGates + r + 256] = acc1[w] + b1;
    }
}

// ---- recurrence ------------------------------------------------------------------------------------------------------------
constexpr int kCluster = 4, kUnits = kHidden / kCluster;  // 32 hidden units per CTA
constexpr int kRecThreads = 512;                          // 4 gates x 32 units x 4 threads per row (32 of the 128 columns each)

static __device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

static __device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
static __device__ __forceinline__ void st_cluster_f32(const float* local, uint32_t rank, float v) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local)), "r"(rank));
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote), "f"(v) : "memory");
}
static __device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Lane layout of a warp: lane = 16 u + 4 g + q: unit u (0..1) of the warp's pair, gate g (i, o, f, c), quarter q of the row's
// 128 columns (interleaved by float4 so the four quarters read h from different banks).  Warp v of CTA `rank` owns hidden
// units j = 32 rank + 2 v + u.  Lane 16 u gathers the four gates of its unit, updates c (kept in its register) and h, stores
// h to H and into the next h buffer of all four CTAs.
// Cluster blockIdx.x / 4 runs slice blockIdx.x / 4 from its stream's h and c (zero when the slice starts the stream) and leaves
// them there for the stream's next slice.
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kRecThreads, 1)
    vad_recurrence_kernel(const float* __restrict__ w_hh, const VadSlice* __restrict__ slices, const float* __restrict__ gx,
                          float* __restrict__ states, float* __restrict__ H) {
  __shared__ __align__(16) float hbuf[2][kHidden];
  const VadSlice sl = slices[blockIdx.x / kCluster];
  const int nb = sl.nb;
  const bool first = sl.first;
  float* __restrict__ state_h = states + (int64_t)sl.stream * 2 * kHidden;
  float* __restrict__ state_c = state_h + kHidden;
  const int rank = (int)cluster_ctarank();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int u = lane >> 4, g = (lane >> 2) & 3, q = lane & 3;
  const int j = rank * kUnits + 2 * warp + u;
  const int row = g * kHidden + j;
  const bool owner = (lane & 15) == 0;
  float4 w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) w[i] = __ldg(reinterpret_cast<const float4*>(w_hh + (size_t)row * kHidden) + 4 * i + q);
  for (int i = threadIdx.x; i < kHidden; i += kRecThreads) hbuf[0][i] = first ? 0.f : state_h[i];
  float c = owner && !first ? state_c[j] : 0.f, h = 0.f;
  // Gx[n + 2] is loaded during step n and must have arrived when the registers rotate at the end of that step: the load
  // overlaps one whole step
  const float* __restrict__ gx_row = gx + (int64_t)sl.w0 * kGates + row;  // this unit's gate row of the slice's first window
  float* __restrict__ h_out = H + (int64_t)sl.w0 * kHidden + j;
  float gx0 = nb > 0 ? __ldg(gx_row) : 0.f;
  float gx1 = nb > 1 ? __ldg(gx_row + kGates) : 0.f;
  cluster_sync();  // every CTA of the cluster runs and holds h0 before anyone writes into its shared memory
  for (int n = 0; n < nb; ++n) {
    const float gx2 = n + 2 < nb ? __ldg(gx_row + (int64_t)(n + 2) * kGates) : 0.f;
    const float4* h4 = reinterpret_cast<const float4*>(hbuf[n & 1]);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 hv = h4[4 * i + q];
      a0 = fmaf(w[i].x, hv.x, a0);
      a1 = fmaf(w[i].y, hv.y, a1);
      a2 = fmaf(w[i].z, hv.z, a2);
      a3 = fmaf(w[i].w, hv.w, a3);
    }
    float s = (a0 + a1) + (a2 + a3);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += gx0;
    const float gi = __shfl_sync(0xffffffffu, s, lane & 16), go = __shfl_sync(0xffffffffu, s, (lane & 16) + 4);
    const float gf = __shfl_sync(0xffffffffu, s, (lane & 16) + 8), gc = __shfl_sync(0xffffffffu, s, (lane & 16) + 12);
    if (owner) {
      c = sigmoidf_(gf) * c + sigmoidf_(gi) * tanhf(gc);
      h = sigmoidf_(go) * tanhf(c);
      h_out[(int64_t)n * kHidden] = h;
      float* dst = &hbuf[(n + 1) & 1][j];
#pragma unroll
      for (int r = 0; r < kCluster; ++r) st_cluster_f32(dst, r, h);
    }
    gx0 = gx1;
    gx1 = gx2;
    cluster_sync();
  }
  if (owner && nb > 0) {
    state_h[j] = h;
    state_c[j] = c;
  }
}

__global__ void __launch_bounds__(256) vad_decoder_kernel(const float* __restrict__ H, const float* __restrict__ w,
                                                          const float* __restrict__ b, int nb, float* __restrict__ probs) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= nb) return;
  const float4 hv = reinterpret_cast<const float4*>(H + (int64_t)n * kHidden)[lane];
  const float4 wv = reinterpret_cast<const float4*>(w)[lane];
  float s = fmaxf(hv.x, 0.f) * wv.x + fmaxf(hv.y, 0.f) * wv.y + fmaxf(hv.z, 0.f) * wv.z + fmaxf(hv.w, 0.f) * wv.w;
  s = warp_sum(s);
  if (lane == 0) probs[n] = sigmoidf_(s + b[0]);
}

void vad_configure() {
  B2W_CUDA(cudaFuncSetAttribute(vad_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWindowSmem));
}

void vad_windows(const VadWeights& w, const float* pcm, const VadSlice* slices, int n_slices, int nb, float* gx, cudaStream_t s) {
  vad_window_kernel<<<ceil_div(nb, kTile), kThreads, kWindowSmem, s>>>(w, pcm, slices, n_slices, nb, gx);
  B2W_LAUNCHED();
}

void vad_recurrence(const float* w_hh, const VadSlice* slices, int n_slices, const float* gx, float* states, float* H,
                    cudaStream_t s) {
  vad_recurrence_kernel<<<kCluster * n_slices, kRecThreads, 0, s>>>(w_hh, slices, gx, states, H);
  B2W_LAUNCHED();
}

void vad_decoder(const float* H, const float* w, const float* b, int nb, float* probs, cudaStream_t s) {
  vad_decoder_kernel<<<ceil_div(nb, 8), 256, 0, s>>>(H, w, b, nb, probs);
  B2W_LAUNCHED();
}

}  // namespace b2w
