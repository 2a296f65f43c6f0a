// On-device decoding logic: logits processors, log-softmax, per-row top-k, beam bookkeeping.
//
// Restates CTranslate2 4.x's Whisper decoding as consumed by faster-whisper (reference call sites
// faster_whisper/transcribe.py:222-236 and 1446-1459; SURVEY.md §8a rows D4-D6): suppress_tokens,
// suppress_blank, Whisper timestamp rules, repetition penalty, no-repeat-ngram, beam search with 2K
// candidates / patience / EOS-exclusive length normalisation, greedy and random sampling (Gumbel-max).
// CTranslate2 runs these as a mix of small kernels and host loops with a device->host sync per token; here
// a decode step is two kernels and the host only polls a "chunks done" counter every few steps.
//
//  search_rows   : one CTA per row; the 51 866-float logits row lives in shared memory while the masks,
//                  the timestamp-probability rule, the log-softmax and the row top-2K run over it.
//  search_update : one CTA per chunk; merges the rows' candidates, applies CTranslate2's finished /
//                  secondary-candidate rule, and re-links token history and KV-slot ancestry (the paged
//                  self-KV cache is never copied when beams reorder).
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "decode.h"

namespace b2w {

constexpr int kRowThreads = 1024;
#define B2W_LOWEST (-FLT_MAX)

struct ArgMax {
  float v;
  int i;
};
__device__ __forceinline__ bool is_better(ArgMax c, ArgMax m) { return c.v > m.v || (c.v == m.v && c.i < m.i); }
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) { return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a; }
__device__ __forceinline__ ArgMax warp_argmax(ArgMax a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax b;
    b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, a.i, o);
    a = better(a, b);
  }
  return a;
}

__device__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) r = fmaxf(r, red[i]);
  return r;
}
__device__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) r += red[i];
  return r;
}

// counter-based uniform -> Gumbel noise; mirrored bit-for-bit (integer part) by oracle/whisper_oracle.py:gumbel_noise
__device__ __forceinline__ float gumbel_u32(unsigned long long seed, int row, int step, int idx) {
  unsigned long long x = (unsigned long long)idx * 0x9E3779B97F4A7C15ull + seed * 0xBF58476D1CE4E5B9ull +
                         (unsigned long long)row * 0x94D049BB133111EBull + (unsigned long long)step * 0xD6E8FEB86659FD93ull;
  x ^= x >> 30;
  x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27;
  x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  const float u = ((float)(unsigned)(x >> 41) + 0.5f) * (1.0f / 8388608.0f);  // 23 bits: exact, strictly in (0,1)
  return -logf(-logf(u));
}

__global__ void __launch_bounds__(kRowThreads) search_rows_kernel(const float* __restrict__ logits, const SearchBuffers bf) {
  const SearchParams p = *bf.params;
  extern __shared__ float s[];  // [vpad]
  __shared__ float red[32];
  __shared__ float wl_v[32 * kMaxCand];
  __shared__ int wl_i[32 * kMaxCand];
  __shared__ int sh_flags[4];
  const int r = blockIdx.x, tid = threadIdx.x;
  const int b = r / p.K, k = r % p.K;
  const int V = p.n_vocab;
  const RowInfo ri = bf.rows[r];
  const ChunkParams cp = bf.chunk[b];
  const int step = ri.pos - (cp.prompt_len - 1);
  const int noise_row = cp.item * p.K + k;  // the item's own row index: its draws do not depend on the slot it occupies
  const int cur = ri.pos & 1;  // history double buffer is indexed by the parity of the absolute position
  const int* hist = bf.hist + ((long long)cur * p.B * p.K + r) * bf.n_ctx;
  const int len = step;  // tokens generated so far by this row
  const float* row = logits + (long long)r * p.vpad;

  // ---- no_speech probability from the raw first-step logits (sot is the last prompt token) ----
  if (cp.ns_first && step == 0 && k == 0) {
    float mx = -INFINITY;
#pragma unroll 4
    for (int v = tid; v < V; v += kRowThreads) mx = fmaxf(mx, row[v]);
    mx = block_max(mx, red);
    float sm = 0.f;
#pragma unroll 4
    for (int v = tid; v < V; v += kRowThreads) sm += __expf(row[v] - mx);
    sm = block_sum(sm, red);
    if (tid == 0) bf.no_speech[b] = __expf(row[p.no_speech] - mx) / sm;
  }

  // ---- load + static suppression: 16-byte loads, all of a thread's loads in flight before the first store ----
  {
    const float4* row4 = reinterpret_cast<const float4*>(row);
    const uchar4* sup4 = reinterpret_cast<const uchar4*>(bf.suppress);
    float4* s4 = reinterpret_cast<float4*>(s);
    const int n4 = p.vpad >> 2;
    float4 t[13];
    uchar4 m[13];
#pragma unroll
    for (int i = 0; i < 13; ++i) {
      const int idx = tid + i * kRowThreads;
      if (idx < n4) {
        t[i] = __ldcs(row4 + idx);
        m[i] = __ldg(sup4 + idx);
      }
    }
#pragma unroll
    for (int i = 0; i < 13; ++i) {
      const int idx = tid + i * kRowThreads;
      if (idx < n4) {
        float4 v = t[i];
        if (m[i].x) v.x = B2W_LOWEST;
        if (m[i].y) v.y = B2W_LOWEST;
        if (m[i].z) v.z = B2W_LOWEST;
        if (m[i].w) v.w = B2W_LOWEST;
        s4[idx] = v;
      }
    }
    for (int idx = tid + 13 * kRowThreads; idx < n4; idx += kRowThreads) {  // vocabularies above 53 248 (none today)
      float4 v = row4[idx];
      const uchar4 mm = sup4[idx];
      s4[idx] = make_float4(mm.x ? B2W_LOWEST : v.x, mm.y ? B2W_LOWEST : v.y, mm.z ? B2W_LOWEST : v.z, mm.w ? B2W_LOWEST : v.w);
    }
  }
  __syncthreads();
  // repetition penalty on the raw value of every distinct generated token
  if (p.repetition_penalty != 1.0f) {
    for (int i = tid; i < len; i += kRowThreads) {
      const int tok = hist[i];
      bool first = true;
      for (int j = 0; j < i; ++j)
        if (hist[j] == tok) {
          first = false;
          break;
        }
      if (first && !bf.suppress[tok]) {
        const float x = row[tok];
        s[tok] = x < 0.f ? x * p.repetition_penalty : x / p.repetition_penalty;
      }
    }
    __syncthreads();
  }
  const int ng = p.no_repeat_ngram;
  if (ng > 0 && len >= ng) {
    for (int s0 = tid; s0 + ng <= len; s0 += kRowThreads) {
      bool same = true;
      for (int j = 0; j < ng - 1; ++j)
        if (hist[s0 + j] != hist[len - ng + 1 + j]) {
          same = false;
          break;
        }
      if (same) s[hist[s0 + ng - 1]] = B2W_LOWEST;
    }
    __syncthreads();
  }
  if (p.suppress_blank && step == 0 && tid < p.n_suppress_begin) s[p.suppress_begin[tid]] = B2W_LOWEST;
  __syncthreads();

  // ---- Whisper timestamp rules ----
  if (cp.timestamp_rules) {
    const int ts0 = p.timestamp_begin;
    if (tid == 0) {
      s[p.no_timestamps] = B2W_LOWEST;
      int last_ts = 0, penult_ts = 0, t_last = -1;
      if (step > 0) {
        last_ts = hist[len - 1] >= ts0;
        penult_ts = (len < 2) || (hist[len - 2] >= ts0);
        for (int i = len - 1; i >= 0; --i)
          if (hist[i] >= ts0) {
            t_last = hist[i];
            break;
          }
        if (t_last >= 0 && !(last_ts && !penult_ts)) t_last += 1;
      }
      sh_flags[0] = last_ts;
      sh_flags[1] = penult_ts;
      sh_flags[2] = t_last;
    }
    __syncthreads();
    const int last_ts = sh_flags[0], penult_ts = sh_flags[1], t_last = sh_flags[2];
    if (step == 0) {
      const int hi = ts0 + p.max_initial_ts;
#pragma unroll 4
      for (int v = tid; v < V; v += kRowThreads)
        if (v < ts0 || (p.max_initial_ts >= 0 && v > hi)) s[v] = B2W_LOWEST;
    } else {
      int lo_a = 0, hi_a = 0;  // masked range A
      if (last_ts) {
        if (penult_ts) {
          lo_a = ts0;
          hi_a = V;
        } else {
          lo_a = 0;
          hi_a = p.eot;
        }
      }
#pragma unroll 4
      for (int v = tid; v < V; v += kRowThreads)
        if ((v >= lo_a && v < hi_a) || (t_last >= 0 && v >= ts0 && v < t_last)) s[v] = B2W_LOWEST;
      __syncthreads();
      // if the timestamps' total probability beats every text token, force a timestamp
      float mx = -INFINITY;
#pragma unroll 4
      for (int v = tid; v < V; v += kRowThreads) mx = fmaxf(mx, s[v]);
      mx = block_max(mx, red);
      float sum_all = 0.f, sum_ts = 0.f, max_text = -INFINITY;
#pragma unroll 4
      for (int v = tid; v < V; v += kRowThreads) {
        const float e = __expf(s[v] - mx);
        sum_all += e;
        if (v >= ts0)
          sum_ts += e;
        else
          max_text = fmaxf(max_text, s[v]);
      }
      sum_all = block_sum(sum_all, red);
      sum_ts = block_sum(sum_ts, red);
      max_text = block_max(max_text, red);
      const float lse = mx + logf(sum_all);
      const float ts_lp = (sum_ts > 0.f) ? (mx + logf(sum_ts) - lse) : -INFINITY;
      const float text_lp = max_text - lse;
      if (ts_lp > text_lp)
#pragma unroll 4
        for (int v = tid; v < ts0; v += kRowThreads) s[v] = B2W_LOWEST;
    }
    __syncthreads();
  }

  // ---- log-softmax ----
  float mx = -INFINITY;
#pragma unroll 4
  for (int v = tid; v < V; v += kRowThreads) mx = fmaxf(mx, s[v]);
  mx = block_max(mx, red);
  float sm = 0.f;
#pragma unroll 4
  for (int v = tid; v < V; v += kRowThreads) sm += __expf(s[v] - mx);
  sm = block_sum(sm, red);
  const float lse = mx + logf(sm);
  const float cum = bf.cum[(long long)cur * p.B * p.K + r];

  // ---- candidate selection ----
  const bool sampling = (p.mode == 1 && p.sampling_topk != 1);
  const float inv_t = 1.0f / p.temperature;
  // transform in place to the ranking key; masked entries become -inf so they are never selected before real ones
#pragma unroll 4
  for (int v = tid; v < V; v += kRowThreads) {
    float x = s[v];
    if (x <= B2W_LOWEST * 0.5f) {
      x = sampling ? -INFINITY : (x - lse);  // CT2 keeps "lowest" (finite) scores for masked ids in beam search
    } else {
      x = x - lse;
      if (sampling) x = x * inv_t + gumbel_u32(p.seed, noise_row, step, v);
    }
    s[v] = x;
  }
  __syncthreads();
  // ---- row top-ncand: every warp extracts the top-ncand of its own 1/32 slice with shuffles only, then warp 0
  //      merges the 32 sorted lists (ties -> lower token id, as a stable top-k would) ----
  const int ncand = p.ncand;
  const int warp = tid >> 5, lane = tid & 31;
  // every thread tracks the best two of its own strided slice, so removing a winner rarely needs a rescan
  ArgMax mine{-INFINITY, 0x7fffffff}, second{-INFINITY, 0x7fffffff};
#pragma unroll 4
  for (int v = tid; v < V; v += kRowThreads) {
    const ArgMax c{s[v], v};
    if (is_better(c, mine)) {
      second = mine;
      mine = c;
    } else if (is_better(c, second)) {
      second = c;
    }
  }
  if (mine.v == -INFINITY) mine.i = 0x7fffffff;
  if (second.v == -INFINITY) second.i = 0x7fffffff;
  bool have_second = true;
  for (int c = 0; c < ncand; ++c) {
    const ArgMax w = warp_argmax(mine);
    if (lane == 0) {
      wl_v[warp * kMaxCand + c] = w.v;
      wl_i[warp * kMaxCand + c] = w.i;
    }
    if (w.i != 0x7fffffff && (w.i % kRowThreads) == tid) {
      s[w.i] = -INFINITY;  // only this thread ever reads or writes this element again
      if (have_second) {
        mine = second;
        have_second = false;
      } else {
        mine = ArgMax{-INFINITY, 0x7fffffff};
#pragma unroll 4
        for (int v = tid; v < V; v += kRowThreads) mine = better(mine, ArgMax{s[v], v});
        if (mine.v == -INFINITY) mine.i = 0x7fffffff;
      }
    }
  }
  __syncthreads();
  if (warp == 0) {
    int head = 0;  // lane l walks warp l's sorted list
    for (int c = 0; c < ncand; ++c) {
      ArgMax cur{-INFINITY, 0x7fffffff};
      if (head < ncand) cur = ArgMax{wl_v[lane * kMaxCand + head], wl_i[lane * kMaxCand + head]};
      if (cur.v == -INFINITY) cur.i = 0x7fffffff;
      const ArgMax best = warp_argmax(cur);
      if (best.i != 0x7fffffff && cur.i == best.i) ++head;
      if (lane == 0) {
        float sc;
        if (sampling) {
          // score of a draw: tempered log-prob (what CTranslate2's RandomSampler gathers)
          sc = (best.i == 0x7fffffff) ? B2W_LOWEST : (best.v - gumbel_u32(p.seed, noise_row, step, best.i));
        } else {
          sc = best.v;
        }
        bf.cand_score[(long long)r * kMaxCand + c] = (p.mode == 0) ? cum + sc : sc;
        bf.cand_tok[(long long)r * kMaxCand + c] = (best.i == 0x7fffffff) ? 0 : best.i;
      }
    }
  }
}

void search_configure() {
  B2W_CUDA(cudaFuncSetAttribute(search_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 210 * 1024));
}

void search_rows(const float* logits, int R, int vpad, const SearchBuffers& b, cudaStream_t s) {
  const int smem = vpad * (int)sizeof(float);
  B2W_CHECK(smem <= 210 * 1024 && vpad % 4 == 0, "vocabulary too large for the in-shared-memory row search");
  search_rows_kernel<<<R, kRowThreads, smem, s>>>(logits, b);
  B2W_LAUNCHED();
}

// ---- beam / greedy bookkeeping ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) search_update_kernel(const SearchBuffers bf) {
  const SearchParams p = *bf.params;
  __shared__ float cs[kMaxBeam * kMaxCand];
  __shared__ int ct[kMaxBeam * kMaxCand];
  __shared__ float c_score[kMaxCand];
  __shared__ int c_tok[kMaxCand], c_beam[kMaxCand];
  __shared__ int parent[kMaxBeam], newtok[kMaxBeam];
  __shared__ float newcum[kMaxBeam];
  __shared__ int fin_src[kMaxBeam], fin_slot[kMaxBeam], fin_extra[kMaxBeam];  // hypotheses finishing at this step
  __shared__ float fin_sc[kMaxBeam];
  __shared__ int n_new_fin;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int K = p.K, V = p.n_vocab, n_ctx = bf.n_ctx, ncand = p.ncand;
  const int r0 = b * K;
  const ChunkParams cp = bf.chunk[b];
  const int pos = bf.rows[r0].pos;
  const int step = pos - (cp.prompt_len - 1);
  const int cur = pos & 1, nxt = cur ^ 1;
  const bool is_last = (step + 1 >= cp.max_steps);
  const long long RB = (long long)p.B * K;
  for (int i = tid; i < K * ncand; i += blockDim.x) {
    const int k = i / ncand, c = i - k * ncand;
    cs[k * kMaxCand + c] = bf.cand_score[(long long)(r0 + k) * kMaxCand + c];
    ct[k * kMaxCand + c] = bf.cand_tok[(long long)(r0 + k) * kMaxCand + c];
  }
  __syncthreads();

  if (tid == 0) {
    const bool chunk_done = bf.done[b] != 0;
    int nf = 0;
    if (p.mode == 0) {
      // ---- merge rows' sorted candidate lists (step 0: only the first row is live) ----
      const int nrows = (step == 0) ? 1 : K;
      int head[kMaxBeam];
      for (int i = 0; i < nrows; ++i) head[i] = 0;
      for (int c = 0; c < ncand; ++c) {
        int bi = -1;
        float bs = 0.f;
        long long bflat = 0;
        for (int i = 0; i < nrows; ++i) {
          if (head[i] >= ncand) continue;
          const float sc = cs[i * kMaxCand + head[i]];
          const long long flat = (long long)i * V + ct[i * kMaxCand + head[i]];
          if (bi < 0 || sc > bs || (sc == bs && flat < bflat)) {
            bi = i;
            bs = sc;
            bflat = flat;
          }
        }
        c_score[c] = bs;
        c_beam[c] = bi;
        c_tok[c] = ct[bi * kMaxCand + head[bi]];
        head[bi]++;
      }
      // ---- CTranslate2 beam step: finished hypotheses are replaced by secondary candidates ----
      int secondary = K;
      bool top_finished = false;
      int nfin = bf.fin_count[b];
      for (int k = 0; k < K; ++k) {
        int nx = k;
        const int t = c_tok[k];
        if ((t == p.eot || is_last) && !chunk_done) {
          if (k == 0) top_finished = true;
          if (nfin < kMaxFinished) {
            fin_src[nf] = c_beam[k];
            fin_slot[nf] = nfin;
            fin_extra[nf] = (t != p.eot) ? t : -1;
            fin_sc[nf] = c_score[k];
            ++nf;
            ++nfin;
          }
          for (int j = secondary; j < ncand; ++j)
            if (c_tok[j] != p.eot) {
              nx = j;
              secondary = j + 1;
              break;
            }
        }
        parent[k] = c_beam[nx];
        newtok[k] = c_tok[nx];
        newcum[k] = c_score[nx];
      }
      if (!chunk_done) {
        bf.fin_count[b] = nfin;
        bool fin;
        if (is_last)
          fin = true;
        else if (p.allow_early_exit)
          fin = top_finished && nfin >= p.num_hyp;
        else
          fin = nfin >= p.max_finished;
        if (fin) {
          bf.done[b] = 1;
          atomicAdd(&bf.state->n_done, 1);
        }
      }
    } else {
      // ---- greedy / sampling: rows are independent hypotheses; fin slot k belongs to row k ----
      int ndone_rows = 0;
      for (int k = 0; k < K; ++k) {
        const int r = r0 + k;
        const int t = ct[k * kMaxCand];
        const float sc = cs[k * kMaxCand];
        parent[k] = k;
        newtok[k] = t;
        const bool row_done = bf.fin_len[b * kMaxFinished + k] >= 0;
        float cumv = bf.cum[(long long)cur * RB + r];
        if (!row_done) {
          cumv += sc;
          if (t == p.eot || is_last) {
            fin_src[nf] = k;
            fin_slot[nf] = k;
            fin_extra[nf] = (t != p.eot) ? t : -1;
            fin_sc[nf] = cumv;
            ++nf;
            ++ndone_rows;
          }
        } else {
          ++ndone_rows;
        }
        newcum[k] = cumv;
      }
      if (!chunk_done && ndone_rows == K) {
        bf.fin_count[b] = K;
        bf.done[b] = 1;
        atomicAdd(&bf.state->n_done, 1);
      }
    }
    n_new_fin = nf;
  }
  __syncthreads();
  const int* hist_cur = bf.hist + (long long)cur * RB * n_ctx;
  // ---- store the hypotheses that finished at this step ----
  for (int f = 0; f < n_new_fin; ++f) {
    const int* src = hist_cur + (long long)(r0 + fin_src[f]) * n_ctx;
    int* dst = bf.fin_tok + ((long long)b * kMaxFinished + fin_slot[f]) * n_ctx;
    for (int i = tid; i < step; i += blockDim.x) dst[i] = src[i];
    if (tid == 0) {
      int len = step;
      if (fin_extra[f] >= 0) dst[len++] = fin_extra[f];
      bf.fin_len[b * kMaxFinished + fin_slot[f]] = len;
      bf.fin_score[b * kMaxFinished + fin_slot[f]] = fin_sc[f];
    }
  }
  // ---- re-link history and KV ancestry into the other buffer, append the new token ----
  int* hist_nxt = bf.hist + (long long)nxt * RB * n_ctx;
  const uint8_t* anc_cur = bf.anc + (long long)cur * RB * n_ctx;
  uint8_t* anc_nxt = bf.anc + (long long)nxt * RB * n_ctx;
  for (int k = 0; k < K; ++k) {
    const int pk = parent[k];
    const int* hs = hist_cur + (long long)(r0 + pk) * n_ctx;
    int* hd = hist_nxt + (long long)(r0 + k) * n_ctx;
    for (int i = tid; i < step; i += blockDim.x) hd[i] = hs[i];
    const uint8_t* as = anc_cur + (long long)(r0 + pk) * n_ctx;
    uint8_t* ad = anc_nxt + (long long)(r0 + k) * n_ctx;
    for (int i = tid; i < pos; i += blockDim.x) ad[i] = as[i];
    if (tid == 0) {
      hd[step] = newtok[k];
      ad[pos] = (uint8_t)pk;
      bf.cum[(long long)nxt * RB + r0 + k] = newcum[k];
      bf.tokens_in[r0 + k] = newtok[k];
      // a generate call ends by max_length <= n_ctx; a finished slot of a decode session idles at the last position until reset
      bf.rows[r0 + k].pos = min(pos + 1, n_ctx - 1);
    }
  }
}

void search_update(int B, const SearchBuffers& b, cudaStream_t s) {
  search_update_kernel<<<B, 128, 0, s>>>(b);
  B2W_LAUNCHED();
}

// One CTA per reset slot: clears everything search_rows / search_update keep for the slot (cumulative scores, history and
// KV ancestry of its rows in both buffers, finished hypotheses, done flag and its share of n_done, no-speech probability),
// installs the occupant's chunk parameters and starts its rows at the last prompt position.  Other slots are not touched.
__global__ void __launch_bounds__(256) search_reset_kernel(const SlotReset* __restrict__ resets, int B, int K, const SearchBuffers bf) {
  const SlotReset rs = resets[blockIdx.x];
  const int b = rs.slot, tid = threadIdx.x, n_ctx = bf.n_ctx;
  const long long RB = (long long)B * K;
  for (int buf = 0; buf < 2; ++buf)
    for (int k = 0; k < K; ++k) {
      const long long row = buf * RB + (long long)b * K + k;
      for (int i = tid; i < n_ctx; i += blockDim.x) {
        bf.hist[row * n_ctx + i] = 0;
        bf.anc[row * n_ctx + i] = 0;
      }
      if (tid == 0) bf.cum[row] = 0.f;
    }
  for (int i = tid; i < kMaxFinished; i += blockDim.x) bf.fin_len[b * kMaxFinished + i] = -1;
  if (tid < K) {
    bf.rows[b * K + tid] = RowInfo{b, tid, rs.cp.prompt_len - 1, 0};
    bf.tokens_in[b * K + tid] = rs.last_token;
  }
  if (tid == 0) {
    bf.chunk[b] = rs.cp;
    bf.fin_count[b] = 0;
    bf.no_speech[b] = 0.f;
    const int was = bf.done[b];
    bf.done[b] = rs.done;
    if (was != rs.done) atomicAdd(&bf.state->n_done, rs.done - was);
  }
}
void search_reset_slots(const SlotReset* resets, int n, int B, int K, const SearchBuffers& b, cudaStream_t s) {
  search_reset_kernel<<<n, 256, 0, s>>>(resets, B, K, b);
  B2W_LAUNCHED();
}

// ---- deterministic stand-in for the decoder (tests of the search logic only) -------------------------------------------
// logits[r][v] = u24(hash(token_in, step, v)) * 2^-20 - 8  (+3 for timestamps, +0.25*step for EOT); mirrored in
// tests/test_search.py so the device search can be compared bit-for-bit with the oracle's search.
__global__ void fake_logits_kernel(float* __restrict__ logits, const SearchBuffers bf) {
  const SearchParams p = *bf.params;
  const int r = blockIdx.y;
  const int step = bf.rows[r].pos - (bf.chunk[r / p.K].prompt_len - 1);
  const unsigned tok = (unsigned)bf.tokens_in[r];
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < p.n_vocab; v += gridDim.x * blockDim.x) {
    unsigned h = tok * 0x9E3779B1u ^ ((unsigned)step * 0x85EBCA77u) ^ ((unsigned)v * 0xC2B2AE3Du);
    h ^= h >> 16;
    h *= 0x7FEB352Du;
    h ^= h >> 15;
    h *= 0x846CA68Bu;
    h ^= h >> 16;
    float x = __fadd_rn(__fmul_rn((float)(h >> 8), 9.5367431640625e-07f), -8.0f);
    if (v >= p.timestamp_begin) x = __fadd_rn(x, 3.0f);
    if (v == p.eot) x = __fadd_rn(x, __fmul_rn(0.25f, (float)step));
    logits[(long long)r * p.vpad + v] = x;
  }
}
void fake_logits(float* logits, int R, const SearchBuffers& b, cudaStream_t s) {
  fake_logits_kernel<<<dim3(32, R), 256, 0, s>>>(logits, b);
  B2W_LAUNCHED();
}

// softmax probability of one token for selected rows (no_speech_prob at the SOT position)
__global__ void token_prob_kernel(const float* __restrict__ logits, int row_stride, int rows_per_chunk, int row_in_chunk,
                                  int n_vocab, int tok, float* __restrict__ out) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float* row = logits + (long long)(b * rows_per_chunk + row_in_chunk) * row_stride;
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < n_vocab; v += blockDim.x) mx = fmaxf(mx, row[v]);
  mx = block_max(mx, red);
  float sm = 0.f;
  for (int v = threadIdx.x; v < n_vocab; v += blockDim.x) sm += __expf(row[v] - mx);
  sm = block_sum(sm, red);
  if (threadIdx.x == 0) out[b] = __expf(row[tok] - mx) / sm;
}
void no_speech_from_logits(const float* logits, int row_stride, int R, int rows_per_chunk, int row_in_chunk, int n_vocab,
                           int no_speech_id, float* out, cudaStream_t s) {
  token_prob_kernel<<<R / rows_per_chunk, 1024, 0, s>>>(logits, row_stride, rows_per_chunk, row_in_chunk, n_vocab, no_speech_id, out);
  B2W_LAUNCHED();
}

// softmax probability of a per-row target token (text_token_probs of Whisper.align); rows with target < 0 are skipped
__global__ void row_target_prob_kernel(const float* __restrict__ logits, int row_stride, int n_vocab, const int* __restrict__ targets,
                                       float* __restrict__ out) {
  __shared__ float red[32];
  const int r = blockIdx.x, tok = targets[r];
  if (tok < 0) return;
  const float* row = logits + (long long)r * row_stride;
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < n_vocab; v += blockDim.x) mx = fmaxf(mx, row[v]);
  mx = block_max(mx, red);
  float sm = 0.f;
  for (int v = threadIdx.x; v < n_vocab; v += blockDim.x) sm += __expf(row[v] - mx);
  sm = block_sum(sm, red);
  if (threadIdx.x == 0) out[r] = __expf(row[tok] - mx) / sm;
}
void row_target_probs(const float* logits, int row_stride, int R, int n_vocab, const int* targets, float* out, cudaStream_t s) {
  row_target_prob_kernel<<<R, 1024, 0, s>>>(logits, row_stride, n_vocab, targets, out);
  B2W_LAUNCHED();
}

// Cross-attention probabilities of the alignment heads of one layer for forced-decoding rows (Whisper.align): CTA per
// (alignment head, row); softmax over all T encoder positions, the first nf written out as out[chunk][head][pos][t] for the
// row's pass chunk (r / rows_per_chunk, the index ds_cross_attn_kernel uses too) and position, against bind[chunk].  K rows are stored with their 16-byte chunks at chunk ^ (t & 7)
// (gemm.cu EPI_F16_XKV).
__global__ void __launch_bounds__(256) align_probs_kernel(const __half* __restrict__ q, const DecBindings* __restrict__ bind,
                                                          const RowInfo* __restrict__ rows, int layer, const int2* __restrict__ heads,
                                                          float* __restrict__ out, int n_tok, int nf, int rows_per_chunk, int H, int T,
                                                          int d) {
  const int2 lh = heads[blockIdx.x];
  if (lh.x != layer) return;
  __shared__ float qs[64];
  __shared__ float sc[1536];
  __shared__ float red[32];
  const int r = blockIdx.y, h = lh.y, tid = threadIdx.x;
  const RowInfo ri = rows[r];
  const int chunk = r / rows_per_chunk;
  const DecBindings bd = bind[chunk];
  const long long per = (long long)bd.B_total * H * T * 64;
  const __half* Kb = bd.xkv + ((long long)layer * 2 + 0) * per + (((long long)bd.item * H + h) * T) * 64;
  if (tid < 64) qs[tid] = __half2float(q[(long long)r * d + h * 64 + tid]) * 0.125f;
  __syncthreads();
  float mx = -INFINITY;
  for (int t = tid; t < T; t += 256) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const uint4 kv = *reinterpret_cast<const uint4*>(Kb + (long long)t * 64 + ((c ^ (t & 7)) << 3));
      const __half2* k2 = reinterpret_cast<const __half2*>(&kv);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(k2[e]);
        s = fmaf(f.x, qs[c * 8 + 2 * e], fmaf(f.y, qs[c * 8 + 2 * e + 1], s));
      }
    }
    sc[t] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_max(mx, red);
  float sm = 0.f;
  for (int t = tid; t < T; t += 256) {
    const float e = __expf(sc[t] - mx);
    sc[t] = e;
    sm += e;
  }
  sm = block_sum(sm, red);
  float* o = out + (((long long)chunk * gridDim.x + blockIdx.x) * n_tok + ri.pos) * nf;
  for (int t = tid; t < nf; t += 256) o[t] = sc[t] / sm;
}
void align_probs(const __half* q, const DecBindings* bind, const RowInfo* rows, int layer, const int2* heads, int n_heads, float* out,
                 int n_tok, int nf, int R, int rows_per_chunk, int H, int T, int d, cudaStream_t s) {
  B2W_CHECK(T <= 1536, "align_probs: encoder length");
  align_probs_kernel<<<dim3(n_heads, R), 256, 0, s>>>(q, bind, rows, layer, heads, out, n_tok, nf, rows_per_chunk, H, T, d);
  B2W_LAUNCHED();
}

__global__ void lang_probs_kernel(const float* __restrict__ logits, int row_stride, int lang_begin, int n_lang,
                                  float* __restrict__ out) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float* row = logits + (long long)b * row_stride + lang_begin;
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < n_lang; v += blockDim.x) mx = fmaxf(mx, row[v]);
  mx = block_max(mx, red);
  float sm = 0.f;
  for (int v = threadIdx.x; v < n_lang; v += blockDim.x) sm += __expf(row[v] - mx);
  sm = block_sum(sm, red);
  for (int v = threadIdx.x; v < n_lang; v += blockDim.x) out[(long long)b * n_lang + v] = __expf(row[v] - mx) / sm;
}
void lang_probs_from_logits(const float* logits, int row_stride, int B, int lang_begin, int n_lang, float* out, cudaStream_t s) {
  lang_probs_kernel<<<B, 128, 0, s>>>(logits, row_stride, lang_begin, n_lang, out);
  B2W_LAUNCHED();
}

}  // namespace b2w
