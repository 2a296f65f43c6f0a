// Persistent decode-step kernel (dstep.cu): argument block shared with engine.cu.
#pragma once
#include "decode.h"

namespace b2w {

constexpr int kDsXSplits = 7;    // key splits of the beam-shared cross attention (20 heads x 7 = 140 tasks, about one per SM)
constexpr int kDsXKeysMax = 224;  // keys per cross-attention tile (multiple of 16, >= ceil(T / kDsXSplits) + 1)
static_assert((B2W_N_AUDIO_CTX + kDsXSplits - 1) / kDsXSplits + 1 <= kDsXKeysMax, "a key split of the encoder output must fit one tile");
constexpr int kDsXQ = 8;  // query rows per cross-attention task: a chunk's rows form ceil(rows_per_chunk / 8) query groups
__host__ __device__ __forceinline__ int ds_xqgroups(int rows_per_chunk) { return (rows_per_chunk + kDsXQ - 1) / kDsXQ; }

// Per layer: the six weight matrices of the step re-laid out as a stream of work-item tiles (dstep_pack_tiles), in the order
// qkv, out, cross_q, cross_out, ffn1, ffn2.
struct DLayer {
  const __half* wt[6];
};

struct DStepArgs {
  const DLayer* layers;  // device array [L]
  int L;
  const __half* tok_emb;
  const __half* logit_tiles;  // packed tiles of the (LayerNorm-folded) output embedding
  const float* pos_emb;
  int R, d, H, n_ctx, slots, T, vpad, n_vocab, n_chunks, rows_per_chunk;
  int w8;  // 1: the tile streams hold int8 weights + per-channel scales (compute_type int8*), 0: fp16
  const RowInfo* rows;
  const int* tokens_in;
  float* x;        // [8][d] fp32 residual stream
  __half* q;       // [8][d]
  __half* ao;      // [8][d]
  __half* h;       // [8][4d]
  float* logits;   // [8][vpad]
  __half* kcache;
  __half* vcache;
  long long kv_layer_stride;
  const uint8_t* anc;
  long long anc_buf_stride;
  const DecBindings* bind;  // [n_chunks] encoder binding of each chunk
  float* xpart;
  int* xcounters;
  unsigned* bar;
  unsigned long long* prof;  // optional: %globaltimer at every barrier (CTA 0) + cycle counters
};

// Tile stream of one matrix W[N][K] (+ bias[N] or null) split `ksplit` ways along K: item = tile * ksplit + ks holds
// 16 rows x (K/ksplit) halves, rows padded by 32 halves (bank-conflict-free 16-byte fragment reads), then 16 fp32 bias
// values (zero unless ks == 0).  One item = one contiguous block = one TMA bulk copy.
size_t dstep_tile_halves(int kr);
size_t dstep_packed_halves(int N, int K, int ksplit);
void dstep_pack_tiles(const __half* W, const float* bias, int N, int K, int ksplit, __half* out, cudaStream_t s);
// int8 variant: rows of (K/ksplit + 32) bytes holding q + 128, then 16 fp32 scales and 16 fp32 bias values per item.
// dstep_quantize_rows quantises W per output channel (symmetric, scale = max|w| / 127) and overwrites W with q * scale.
size_t dstep_packed_bytes_i8(int N, int K, int ksplit);
void dstep_quantize_rows(__half* W, int N, int K, unsigned char* q, float* scale, cudaStream_t s);
void dstep_pack_tiles_i8(const unsigned char* q, const float* scale, const float* bias, int N, int K, int ksplit, unsigned char* out,
                         cudaStream_t s);

// stand-alone beam-shared cross attention on mma.sync (the persistent kernel's task as its own launch), any rows per chunk
void dstep_cross_attn_launch(const DStepArgs& a, int layer, cudaStream_t s);

size_t dstep_smem_bytes(const DStepArgs& a);
void dstep_configure();
int dstep_max_grid(int num_sms, const DStepArgs& a);
void dstep_launch(const DStepArgs& a, int grid, cudaStream_t s);
// B2W_DSTEP_PROF: prints the per-phase timers of the last step launched with a.prof set (stderr)
void dstep_print_profile(const DStepArgs& a, cudaStream_t s);

}  // namespace b2w
