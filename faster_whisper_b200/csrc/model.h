// Model / workspace structures of libb200whisper (host side).
#pragma once
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "decode.h"
#include "bstep.h"
#include "dstep.h"
#include "engine.h"

namespace b2w {

struct EncLayerW {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  __half *wqkv, *wo, *w1, *w2;  // NULL under compute_type float8_float16
  float *bqkv, *bo, *b1, *b2;
  // compute_type float8_float16: e4m3 codes and per-output-channel scales of the four linear layers (fp8.cuh)
  uint8_t *q_wqkv, *q_wo, *q_w1, *q_w2;
  float *s_wqkv, *s_wo, *s_w1, *s_w2;
};
struct DecLayerW {  // every LayerNorm affine is folded into the projection that consumes it (fold_ln)
  __half *wqkv, *wo, *wq_x, *wo_x, *w1, *w2;
  float *bqkv, *bo, *bq_x, *bo_x, *b1, *b2;
};

struct EncPlan {  // everything bound to the encoder workspace for one sub-batch size
  int b = 0;
  GemmPlan conv1, conv2;
  std::vector<GemmPlan> qkv, proj, ffn1, ffn2;
  std::vector<Fp8GemmPlan> qkv8, proj8, ffn1_8, ffn2_8;  // compute_type float8_float16
  AttnPlan attn;
};

struct StageTimer {
  int stage;
  cudaEvent_t start, stop;
};

// The decode step runs as the layered multi-kernel sequence or as one of the two persistent kernels; B2W_STEP forces one.
enum class StepPath { Layers, Dstep, Bstep, FakeLogits };
// kcache, sb_blob, d_xpart, d_logits, chunks, rows per chunk, path, B2W_BSTEP_STOP
using StepGraphKey = std::tuple<const void*, const void*, const void*, const void*, int, int, int, int>;

struct Model;

struct Encoded {
  Model* owner = nullptr;
  int B = 0;
  size_t enc_bytes = 0, xkv_bytes = 0;
  __half* enc_out = nullptr;  // [B][1500][d] fp16
  __half* xkv = nullptr;      // lazily: [L][2][B][H][T][64] fp16
  int refs = 1;               // the b2w_encoded handle, and one per decode-session slot or queued item that reads it
  ~Encoded();
};

struct Model {
  b2w_config cfg{};
  int device = 0;
  int num_sms = 132;
  int cpad = 128;   // mel channels padded to a multiple of 64
  int vpad = 0;     // vocabulary padded to a multiple of 16
  cudaStream_t stream = nullptr;
  std::mutex mu;
  std::vector<void*> allocs;  // allocated once (weights, decoder workspace), freed with the model
  // size-keyed free list for encoder outputs / cross-KV caches: a 3.9 GB cudaMalloc+cudaFree per call costs ~100s of ms, and a
  // cudaFree synchronises the device
  std::vector<std::pair<size_t, void*>> pool;
  size_t pool_bytes = 0;
  size_t encoded_bytes = 0;  // device bytes of the live encoder outputs (b2w_memory_get)
  void* pool_get(size_t bytes);
  void pool_put(void* p, size_t bytes);

  // encoder weights
  __half *conv1_w = nullptr, *conv2_w = nullptr;
  float *conv1_b = nullptr, *conv2_b = nullptr, *enc_pos = nullptr, *enc_lnp_g = nullptr, *enc_lnp_b = nullptr;
  std::vector<EncLayerW> enc;
  // decoder weights
  __half* tok_emb = nullptr;  // [vpad][d]
  __half* logit_w = nullptr;  // [vpad][d]  tied embedding scaled by the final LayerNorm's gamma
  float* logit_b = nullptr;   // [vpad]     E . beta_f
  float* dec_pos = nullptr;
  std::vector<DecLayerW> dec;
  __half* wxkv = nullptr;  // [L*2d][d]
  float* bxkv = nullptr;   // [L*2d]
  double dec_weight_bytes = 0;  // bytes one decode step must stream (all decoder weights incl. the tied embedding)

  std::unique_ptr<MelPlan> mel;

  // encoder workspace (sized for enc_max_b chunks)
  int enc_max_b = 0;
  float* e_feats = nullptr;   // [b][n_mels][3000] f32
  __half* e_x0 = nullptr;     // [b][3000][cpad]
  __half* e_x1 = nullptr;     // [b][3000][d]
  float* e_x = nullptr;       // [b*1500][d] residual stream
  __half* e_xn = nullptr;     // [b*1500][d]
  __half* e_qkv = nullptr;    // [b*1500][3d]
  __half* e_ao = nullptr;     // [b*1500][d]
  __half* e_h = nullptr;      // [b*1500][4d]
  uint8_t* e_q = nullptr;     // float8_float16: e4m3 codes of the next linear layer's input, [b*1500][up to 4d]
  float* e_qs = nullptr;      // their row scales [b*1500]
  float* e_pcm = nullptr;     // audio staging
  size_t e_pcm_cap = 0;
  MelChunkDesc* e_chunks = nullptr;
  int* e_chunk_max = nullptr;
  std::map<int, EncPlan> enc_plans;
  // keyed by (weights, activations, rows, mode, row table, K cache, V cache, slots): the QKV epilogue's plan holds the last four,
  // which change when the search or KV workspace is reallocated or the rows per chunk change
  std::map<std::tuple<const void*, const void*, int, int, const void*, const void*, const void*, int>, GemmPlan> dec_plans;

  // decoder workspace
  size_t kv_elems = 0;        // per layer per K|V
  __half* kcache = nullptr;   // [L][kv_elems]
  __half* vcache = nullptr;
  float* d_x = nullptr;       // [80][d]
  __half *d_xn = nullptr, *d_q = nullptr, *d_ao = nullptr, *d_h = nullptr;
  float* d_logits = nullptr;  // [80][vpad]
  float* d_xpart = nullptr;
  size_t d_xpart_floats = 0;
  int* d_counters = nullptr;  // [0]: GEMM ticket, [64..]: cross-attention groups
  uint8_t* d_suppress = nullptr;
  DecBindings* d_bind = nullptr;
  // Whisper.align: (layer, head) pairs whose cross-attention b2w_align captures; d_align_heads is their device copy, made on
  // first use
  std::vector<int2> align_heads;
  int2* d_align_heads = nullptr;
  cudaEvent_t span_a = nullptr, span_b = nullptr;  // b2w_span_begin / b2w_span_end
  const __half* logit_tiles = nullptr;  // output embedding as the persistent step kernel's tile stream
  DLayer* d_layers = nullptr;   // device copy of the decoder layer pointer table (persistent step kernel)
  unsigned* d_bar = nullptr;
  unsigned long long* d_prof = nullptr;  // B2W_DSTEP_PROF=1: per-phase timestamps of the persistent step kernels
  int dstep_grid = 0;  // grid of the <= 8-row step kernel (dstep.cu); 0 when it cannot run this model
  // compute_type int8*: the decoder's linear layers (and the output embedding) are quantised per output channel; the persistent step
  // kernels stream them as int8 (w8), every other path uses the de-quantised fp16 values.
  bool w8 = false;
  // compute_type float8_float16: the encoder's QKV, out-projection, FFN1 and FFN2 run as e4m3 GEMMs (gemm_fp8_kernel)
  bool fp8_enc = false;
  // many-row persistent step kernel (bstep.cu): decoder weights as 16 KB wgmma atoms + per-row sums for the deferred LayerNorm
  bool bstep_packed = false;
  BLayer* d_blayers = nullptr;
  const void* logit_atoms = nullptr;
  const float* logit_scale = nullptr;
  float *d_stats = nullptr, *d_gpart = nullptr, *d_stpart = nullptr;
  __half *d_h16 = nullptr, *d_xn16 = nullptr;
  std::optional<StepPath> forced_step;  // B2W_STEP=dstep|bstep|layers (tests and tools)
  DecBindings h_bind{};                // chunk 0's entry of the last bound table
  std::vector<DecBindings> h_binds;    // host copy of d_bind's entries
  SearchParams h_params{};
  // search buffers
  SearchBuffers sb{};
  void* sb_blob = nullptr;
  int sb_B = 0, sb_K = 0;
  int* h_pinned = nullptr;    // pinned host scratch

  // step graph cache
  cudaGraphExec_t step_graph = nullptr;
  int64_t step_graph_kernels = 0;
  StepGraphKey step_graph_key{};

  // measurement
  bool timing = false;
  std::vector<StageTimer> timers;
  double t_ms[B2W_T_COUNT] = {0};
  int64_t t_cnt[B2W_T_COUNT] = {0};
  int64_t launches = 0, decode_steps = 0;
  double decode_alg_bytes = 0;

  bool use_ref_gemm = false, use_ref_attn = false;

  ~Model();
};

}  // namespace b2w
