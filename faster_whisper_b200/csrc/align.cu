// Whisper.align post-processing on the device: the DTW cost matrix from the alignment heads' cross-attention capture, and the
// monotone path through it.
//
//  align_stats_kernel : thread per (item, head, frame): mean and population std over the item's tokens.
//  align_cost_kernel  : CTA per (item, kept row, 128-frame tile): per head in order, the normalised row (a - mean) / std is
//                       staged in shared memory with reflect padding, median-filtered along time, and added to the head sum;
//                       the cost is -sum / n_heads.
//  align_dtw_kernel   : CTA per item: anti-diagonal wavefront over (n_rows + 1) x (nf + 1) with the three live diagonals in
//                       shared memory, the 2-bit trace packed in shared memory too, then the backtrack by one thread.
//
// Every sum runs in the order of a plain sequential loop (tokens 0..n_tok-1 per column, heads 0..n_heads-1 per cell), in fp64,
// with explicit round-to-nearest intrinsics so that no multiply-add is contracted; fp64 sqrt and division are correctly rounded
// and the median is a selection.  The cost matrix is therefore bit-identical to the same loops run on the host.
#include <math.h>

#include "common.cuh"
#include "decode.h"

namespace b2w {

__global__ void __launch_bounds__(128) align_stats_kernel(AlignBatch a) {
  const int b = blockIdx.z, h = blockIdx.y, f = blockIdx.x * 128 + threadIdx.x;
  const int4 it = a.items[b];  // n_tok, nf, row0, n_rows
  if (it.w == 0 || f >= it.y) return;
  const float* col = a.cap + (((long long)b * a.n_heads + h) * a.tok_stride) * a.nf_stride + f;
  double mu = 0.0;
  for (int t = 0; t < it.x; ++t) mu = __dadd_rn(mu, (double)col[(long long)t * a.nf_stride]);
  mu = __ddiv_rn(mu, (double)it.x);
  double var = 0.0;
  for (int t = 0; t < it.x; ++t) {
    const double d = __dsub_rn((double)col[(long long)t * a.nf_stride], mu);
    var = __dadd_rn(var, __dmul_rn(d, d));
  }
  double* st = a.stats + (((long long)b * a.n_heads + h) * 2) * a.nf_stride;
  st[f] = mu;
  st[a.nf_stride + f] = __dsqrt_rn(__ddiv_rn(var, (double)it.x));
}

// Median filter of odd `width` along time with reflect padding (the edge sample is not repeated); no filtering when
// nf <= width / 2.  Dynamic shared memory: (128 + width - 1) doubles.
__global__ void __launch_bounds__(128) align_cost_kernel(AlignBatch a) {
  extern __shared__ double win[];
  const int b = blockIdx.z, r = blockIdx.y, f0 = blockIdx.x * 128, tid = threadIdx.x, f = f0 + tid;
  const int4 it = a.items[b];
  const int nf = it.y;
  if (r >= it.w || f0 >= nf) return;
  const int pad = (a.width / 2 > 0 && nf > a.width / 2) ? a.width / 2 : 0, span = 128 + 2 * pad;
  const long long tok = it.z + r;
  double acc = 0.0;
  for (int h = 0; h < a.n_heads; ++h) {
    const float* row = a.cap + (((long long)b * a.n_heads + h) * a.tok_stride + tok) * a.nf_stride;
    const double* mu = a.stats + (((long long)b * a.n_heads + h) * 2) * a.nf_stride;
    const double* sd = mu + a.nf_stride;
    for (int k = tid; k < span; k += 128) {
      int x = f0 - pad + k;
      if (x < 0) x = -x;
      if (x >= nf) x = 2 * (nf - 1) - x;
      x = min(max(x, 0), nf - 1);  // only for window slots past the last frame's, which no output reads
      win[k] = __ddiv_rn(__dsub_rn((double)row[x], mu[x]), sd[x]);
    }
    __syncthreads();
    if (f < nf) {
      double med = win[tid + pad];
      if (pad > 0) {
        const double* w = win + tid;
        for (int k = 0; k < 2 * pad + 1; ++k) {  // the value with at most pad smaller and more than pad not larger
          const double v = w[k];
          int lt = 0, le = 0;
          for (int j = 0; j < 2 * pad + 1; ++j) {
            lt += w[j] < v;
            le += w[j] <= v;
          }
          if (lt <= pad && pad < le) {
            med = v;
            break;
          }
        }
      }
      acc = __dadd_rn(acc, med);
    }
    __syncthreads();
  }
  if (f < nf) a.cost[((long long)b * a.row_stride + r) * a.nf_stride + f] = __ddiv_rn(-acc, (double)a.n_heads);
}

// DTW of cost[n_rows][nf] (row stride nf_stride): cell (i, j), 1 <= i <= N, 1 <= j <= M, takes the cheapest of (i-1, j-1)
// [move 0], (i-1, j) [move 1] and (i, j-1) [move 2]: move 0 only when strictly smallest, else move 1 when strictly smallest,
// else move 2.  cost(0, 0) = 0 and the rest of row 0 and column 0 is infinite; the backtrack from (N, M) takes move 2 in row 0
// and move 1 in column 0.  Writes the path as (i - 1, j - 1) pairs from (0, 0) to its slot of N_max + M_max pairs.
__global__ void __launch_bounds__(512) align_dtw_kernel(AlignBatch a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int4 it = a.items[b];
  const int N = it.w, M = it.y;
  int2* out = a.pairs + (long long)b * (a.row_stride + a.nf_stride);
  if (N == 0) {
    if (tid == 0) a.n_pairs[b] = 0;
    return;
  }
  const int S = a.row_stride + 1, W = (a.nf_stride + 16) / 16;  // diagonal length, trace words per row (16 cells each)
  double* diag = reinterpret_cast<double*>(smem);                // [3][S]
  uint32_t* trace = reinterpret_cast<uint32_t*>(diag + 3 * S);   // [S][W]
  const double* c = a.cost + (long long)b * a.row_stride * a.nf_stride;
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  if (tid == 0) {
    diag[0] = 0.0;      // d = 0: (0, 0)
    diag[S + 0] = inf;  // d = 1: (0, 1)
    diag[S + 1] = inf;  //        (1, 0)
  }
  __syncthreads();
  for (int d = 2; d <= N + M; ++d) {
    double* cur = diag + (d % 3) * S;
    const double* p1 = diag + ((d - 1) % 3) * S;
    const double* p2 = diag + ((d - 2) % 3) * S;
    const int lo = max(0, d - M), hi = min(N, d);
    for (int i = lo + tid; i <= hi; i += blockDim.x) {
      const int j = d - i;
      if (i == 0 || j == 0) {
        cur[i] = inf;
        continue;
      }
      const double c0 = p2[i - 1], c1 = p1[i - 1], c2 = p1[i];
      double best;
      uint32_t t;
      if (c0 < c1 && c0 < c2) { best = c0; t = 0; }
      else if (c1 < c0 && c1 < c2) { best = c1; t = 1; }
      else { best = c2; t = 2; }
      cur[i] = __dadd_rn(c[(long long)(i - 1) * a.nf_stride + (j - 1)], best);
      uint32_t& w = trace[i * W + (j >> 4)];  // one cell of each row per diagonal: no other thread writes this word now
      const int sh = (j & 15) * 2;
      w = (w & ~(3u << sh)) | (t << sh);
    }
    __syncthreads();
  }
  if (tid == 0) {
    int i = N, j = M, n = 0;
    while (i > 0 || j > 0) {
      out[n++] = make_int2(i - 1, j - 1);
      const uint32_t t = i == 0 ? 2u : j == 0 ? 1u : (trace[i * W + (j >> 4)] >> ((j & 15) * 2)) & 3u;
      if (t == 0) { --i; --j; }
      else if (t == 1) --i;
      else --j;
    }
    a.n_pairs[b] = n;
  }
  __syncthreads();
  const int n = a.n_pairs[b];
  for (int k = tid; k < n / 2; k += blockDim.x) {
    const int2 x = out[k];
    out[k] = out[n - 1 - k];
    out[n - 1 - k] = x;
  }
}

static size_t dtw_smem(const AlignBatch& a) {
  const size_t S = a.row_stride + 1, W = (a.nf_stride + 16) / 16;
  return 3 * S * sizeof(double) + S * W * sizeof(uint32_t);
}

void align_check(const AlignBatch& a) {
  B2W_CHECK(a.n_heads >= 1 && a.width >= 1 && a.width % 2 == 1, "align: heads and an odd median filter width");
  B2W_CHECK(a.nf_stride >= 1 && a.nf_stride <= 1500 && a.row_stride >= 1 && a.row_stride <= kAlignMaxRows,
            "align: at most 449 rows x 1500 frames");
  B2W_CHECK(dtw_smem(a) <= 227 * 1024, "align: DTW trace exceeds shared memory");
}

void align_cost(const AlignBatch& a, int n_items, cudaStream_t s) {
  align_check(a);
  const int tiles = ceil_div(a.nf_stride, 128);
  align_stats_kernel<<<dim3(tiles, a.n_heads, n_items), 128, 0, s>>>(a);
  B2W_LAUNCHED();
  const int pad = a.width / 2 < a.nf_stride ? a.width / 2 : 0;  // no item filters when width / 2 >= every nf
  align_cost_kernel<<<dim3(tiles, a.row_stride, n_items), 128, (128 + 2 * pad) * sizeof(double), s>>>(a);
  B2W_LAUNCHED();
}

void align_dtw(const AlignBatch& a, int n_items, cudaStream_t s) {
  align_check(a);
  const size_t smem = dtw_smem(a);
  B2W_CUDA(cudaFuncSetAttribute(align_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  align_dtw_kernel<<<n_items, 512, smem, s>>>(a);
  B2W_LAUNCHED();
}

}  // namespace b2w
