// Internal interfaces between the translation units of libb200whisper.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200whisper.h"

namespace b2w {

// ---- log-mel (mel.cu) ---------------------------------------------------------------------------------
struct MelChunkDesc {
  const float* pcm;   // device pointer
  int64_t n_samples;
  int32_t n_frames;   // frames taking part in the global max = 1 + n_samples/160
  int32_t n_emit;     // frames written
};
struct MelPlan {
  int n_mels;
  void* d_twiddle = nullptr;
  int *d_lo = nullptr, *d_cnt = nullptr, *d_off = nullptr;
  float* d_w = nullptr;
  explicit MelPlan(int n_mels);
  ~MelPlan();
  void run(const void* chunks_dev, int n_chunks, int max_frames, int padding, float* out, int64_t out_chunk_stride,
           int out_ld, int* chunk_max_dev, bool zero_fill, cudaStream_t stream) const;
};

// ---- dense GEMM on wgmma (gemm.cu) --------------------------------------------------------------------
enum Epilogue {
  EPI_F16 = 0,           // out(f16) = acc + bias
  EPI_GELU_F16 = 1,      // out(f16) = gelu(acc + bias)
  EPI_RESID_F32 = 2,     // out(f32) = resid + acc + bias
  EPI_GELU_POS_F32 = 3,  // out(f32) = gelu(acc + bias) + pos[row, n]
  EPI_F16_XKV = 4,       // cross-KV scatter: out[l][kv][b][h][t][64] (f16) = acc + bias
  EPI_F32 = 5,           // out(f32) = acc + bias
  EPI_QKV_CACHE = 6,     // decoder fused QKV: q -> out(f16)[row][d]; k,v -> paged self-KV cache at (chunk,pos,slot) of the row
};

struct GemmArgs {
  // A operand: fp16 tensor [a_batch][a_rows][a_cols], K index k -> (tap, kk): element (row + tap_row[tap], tap_col[tap] + kk)
  const __half* A = nullptr;
  int a_batch = 1, a_rows = 0, a_cols = 0;
  int64_t a_row_stride = 0, a_batch_stride = 0;  // in elements
  int taps = 1, tap_row[3] = {0, 0, 0}, tap_col[3] = {0, 0, 0};
  int k_per_tap = 0;  // multiple of 64; K = taps * k_per_tap
  // B operand: weights [N][K] fp16 row-major
  const __half* W = nullptr;
  int N = 0;
  // output rows per batch (M); out index = b*out_batch_stride + row*out_ld + n
  int rows = 0;
  const float* bias = nullptr;
  void* out = nullptr;
  int64_t out_ld = 0, out_batch_stride = 0;
  const float* resid = nullptr;  // EPI_RESID_F32 (same indexing as out)
  const float* pos = nullptr;    // EPI_GELU_POS_F32: [rows][N]
  int xkv_d = 0, xkv_heads = 0, xkv_T = 0, xkv_B = 0;  // EPI_F16_XKV
  const int4* rowinfo = nullptr;  // EPI_QKV_CACHE: (chunk, slot, pos, -) per row
  __half* kcache = nullptr;
  __half* vcache = nullptr;
  int qkv_d = 0, n_ctx = 0, slots = 0;
  int epilogue = EPI_F16;
  // few-row GEMMs (decode rows): prefer narrow 32-column tiles so that more than N/128 CTAs stream the weights
  bool narrow_tiles = false;
};

struct GemmPlan {
  GemmArgs a;
  CUtensorMap tmA, tmB;
  int block_n = 128;
  int tiles_m = 0, tiles_n = 0, num_kb = 0, grid = 0;
  double flops() const { return 2.0 * a.a_batch * a.rows * (double)a.N * a.taps * a.k_per_tap; }
};
GemmPlan gemm_plan(const GemmArgs& a, int num_sms);
void gemm_run(const GemmPlan& p, cudaStream_t stream);
void gemm_configure();  // per-device kernel attributes; call once per device outside stream capture
void gemm_ref_run(const GemmArgs& a, cudaStream_t stream);  // plain SIMT reference of the same contract

// e4m3 GEMM of the encoder's linear layers under compute_type float8_float16 (gemm.cu):
//   out[r][n] = epilogue(a_scale[r] * w_scale[n] * sum_k A[r][k] W[n][k] + bias[n]), A codes [rows][K], W codes [N][K] (fp8.cuh)
// epilogue EPI_F16 | EPI_GELU_F16 (out fp16 [rows][N]) or EPI_RESID_F32 (out fp32 [rows][N] += ...).  K a multiple of 64.
struct Fp8GemmArgs {
  const uint8_t* A = nullptr;
  const float* a_scale = nullptr;
  const uint8_t* W = nullptr;
  const float* w_scale = nullptr;
  int rows = 0, K = 0, N = 0;
  const float* bias = nullptr;
  void* out = nullptr;
  int epilogue = EPI_F16;
};
struct Fp8GemmPlan {
  Fp8GemmArgs a;
  CUtensorMap tmA, tmB;
  int tiles_m = 0, tiles_n = 0, num_kb = 0, grid = 0;
  double flops() const { return 2.0 * a.rows * (double)a.N * a.K; }
};
Fp8GemmPlan gemm_fp8_plan(const Fp8GemmArgs& a, int num_sms);
void gemm_fp8_run(const Fp8GemmPlan& p, cudaStream_t stream);

// ---- encoder attention on wgmma (attention.cu) ---------------------------------------------------------
struct AttnPlan {
  const __half* qkv = nullptr;  // [B][T][3*H*64]
  __half* out = nullptr;        // [B][T][H*64]
  int B = 0, T = 0, H = 0;
  CUtensorMap tm;
};
AttnPlan attn_plan(const __half* qkv, __half* out, int B, int T, int H);
void attn_run(const AttnPlan& p, cudaStream_t stream);
void attn_ref_run(const __half* qkv, __half* out, int B, int T, int H, cudaStream_t stream);

// ---- small encoder kernels (encoder_misc.cu) ---------------------------------------------------------------
void layernorm_f32_f16(const float* x, const float* gamma, const float* beta, __half* out, int rows, int d, cudaStream_t s);
void layernorm_f32_f32(const float* x, const float* gamma, const float* beta, float* out, int rows, int d, cudaStream_t s);
// e4m3 codes [rows][d] + row scales [rows] of the fp32 LayerNorm output, and of fp16 rows [rows][K] (K a multiple of 8)
void layernorm_f32_e4m3(const float* x, const float* gamma, const float* beta, uint8_t* q, float* scale, int rows, int d,
                        cudaStream_t s);
void quantize_rows_e4m3(const __half* x, uint8_t* q, float* scale, int rows, int K, cudaStream_t s);
void pack_features(const float* feats /*[B][n_mels][3000]*/, __half* out /*[B][3000][cpad]*/, int B, int n_mels, int cpad,
                   cudaStream_t s);
void convert_f32_f16(const float* in, __half* out, int64_t n, cudaStream_t s);
void convert_f16_f32(const __half* in, float* out, int64_t n, cudaStream_t s);

}  // namespace b2w
