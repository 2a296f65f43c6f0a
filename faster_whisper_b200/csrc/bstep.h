// Persistent decode-step kernel for many rows (bstep.cu): up to 80 rows (16 chunks x beam 5) per step in one cooperative launch.
#pragma once
#include "decode.h"

namespace b2w {

constexpr int kBsAtomBytes = 16384;  // one weight atom: 128 output channels x 64 K values, fp16, 128-byte swizzle (a ready-made wgmma A tile)
constexpr int kBsMaxRows = 80;
constexpr int kBsBarWords = 64 + 6 * 64;

// Per layer: the six weight matrices as atom streams (order: qkv, out, cross_q, cross_out, ffn1, ffn2), their fp32 biases and, for the
// three matrices that consume a LayerNorm, the row sums of the (LayerNorm-folded, fp16-rounded) weights — the mean term of the
// deferred normalisation  y = rstd * (W x - mean * rowsum(W)) + b.
struct BLayer {
  const void* wt[6];      // fp16 atoms (16 KB) or, with w8, int8 atoms (8 KB: [128 channels][64 K] bytes holding q + 128)
  const float* bias[6];
  const float* wsum[3];   // qkv, cross_q, ffn1
  const float* scale[6];  // w8: per-output-channel de-quantisation scales (applied to the fp32 accumulator in the epilogue)
};

struct BStepArgs {
  const BLayer* layers;  // device array [L]
  int L;
  const __half* tok_emb;
  const float* pos_emb;
  const void* logit_atoms;    // (LayerNorm-folded) output embedding as an atom stream, rows padded to a multiple of 128
  const float* logit_bias;    // [vpad]
  const float* logit_scale;   // [vpad] (w8)
  int w8;                     // 1: int8 atom streams, widened to fp16 wgmma tiles in shared memory by the compute warps
  int R, NP;                  // rows, rows padded to the wgmma N (multiple of 16)
  int d, H, n_ctx, slots, T, vpad, n_vocab, n_chunks, rows_per_chunk;
  int u_bytes;                // size of the multi-purpose shared-memory region
  int stop_phase;             // debug: number of grid phases to run (<= 0: all)
  const RowInfo* rows;
  const int* tokens_in;
  float* x;       // [R][d]   fp32 residual stream
  __half* ao;     // [R][d]   attention output
  __half* h16;    // [R][4d]  GELU(hidden)
  __half* xn16;   // [R][d]   final LayerNorm output
  float* stats;   // [3L][R][2]  sum(x), sum(x^2) of the residual stream at each LayerNorm (a record for b2w_debug_fetch)
  float* stpart;  // [d/64][R][2] per-k-atom partials of the statistics of the current GEMM phase
  float* gpart;   // [grid][R][128] each CTA's split-K partial tile of the current GEMM phase
  float* logits;  // [R][vpad]
  __half* kcache;
  __half* vcache;
  long long kv_layer_stride;
  const uint8_t* anc;
  long long anc_buf_stride;
  const DecBindings* bind;  // [n_chunks] encoder binding of each chunk
  float* xpart;
  int* xcounters;
  unsigned* bar;  // [kBsBarWords]: grid barrier, then from word 64 the n-block group counters [6 matrices][64 n-blocks]
  unsigned long long* prof;  // optional: %globaltimer at every barrier (CTA 0)
};

// atom stream of W[N][K] (row-major fp16): atoms ordered (n-block, k-atom); rows beyond N are zero
size_t bstep_atoms_bytes(int N, int K);
void bstep_pack_atoms(const __half* W, int N, int K, __half* out, cudaStream_t s);
void bstep_row_sums(const __half* W, int N, int K, float* out, cudaStream_t s);
// int8 variants: q holds the biased bytes (q + 128) of W[N][K] quantised per output channel with `scale`
size_t bstep_atoms_bytes_i8(int N, int K);
void bstep_pack_atoms_i8(const unsigned char* q, int N, int K, unsigned char* out, cudaStream_t s);
void bstep_row_sums_i8(const unsigned char* q, const float* scale, int N, int K, float* out, cudaStream_t s);

void bstep_configure();
bool bstep_supported(int num_sms, BStepArgs& a);  // fills a.NP / a.u_bytes; false when the shape cannot run here
size_t bstep_xpart_floats(const BStepArgs& a);
void bstep_launch(const BStepArgs& a, int grid, cudaStream_t s);
int bstep_phase_count(int L);
// B2W_DSTEP_PROF: prints the per-phase timers of the last step launched with a.prof set (stderr)
void bstep_print_profile(const BStepArgs& a, cudaStream_t s);

}  // namespace b2w
