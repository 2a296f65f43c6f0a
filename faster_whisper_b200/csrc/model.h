// Model / workspace structures of libb200whisper (host side).
#pragma once
#include <map>
#include <memory>
#include <mutex>
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
  __half *wqkv, *wo, *w1, *w2;
  float *bqkv, *bo, *b1, *b2;
};
struct DecLayerW {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b, *ln3_g, *ln3_b;
  __half *wqkv, *wo, *wq_x, *wo_x, *w1, *w2;
  float *bqkv, *bo, *bq_x, *bo_x, *b1, *b2;
};

struct EncPlan {  // everything bound to the encoder workspace for one sub-batch size
  int b = 0;
  GemmPlan conv1, conv2;
  std::vector<GemmPlan> qkv, proj, ffn1, ffn2;
  AttnPlan attn;
};

struct StageTimer {
  int stage;
  cudaEvent_t start, stop;
};

struct Model;

struct Encoded {
  Model* owner = nullptr;
  int B = 0;
  size_t enc_bytes = 0, xkv_bytes = 0;
  __half* enc_out = nullptr;  // [B][1500][d] fp16
  __half* xkv = nullptr;      // lazily: [L][2][B][H][T][64] fp16
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
  std::vector<void*> allocs;  // weights
  // size-keyed free list for encoder outputs / cross-KV caches: a 3.9 GB cudaMalloc+cudaFree per call costs ~100s of ms
  std::vector<std::pair<size_t, void*>> pool;
  size_t pool_bytes = 0;
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
  float *dec_pos = nullptr, *dec_ln_g = nullptr, *dec_ln_b = nullptr;
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
  float* e_pcm = nullptr;     // audio staging
  size_t e_pcm_cap = 0;
  MelChunkDesc* e_chunks = nullptr;
  int* e_chunk_max = nullptr;
  std::map<int, EncPlan> enc_plans;
  std::map<std::tuple<const void*, const void*, int, int>, GemmPlan> dec_plans;

  // decoder workspace
  int dw_rows = 0;
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
  // Whisper.align: (layer, head) pairs whose cross-attention is captured; while `align_out` is set, decoder_layers() writes
  // the probabilities of the forced-decoding rows there
  std::vector<int2> align_heads;
  int2* d_align_heads = nullptr;
  float* align_out = nullptr;
  int align_n_tok = 0, align_nf = 0, align_pos0 = 0;
  cudaEvent_t span_a = nullptr, span_b = nullptr;  // b2w_span_begin / b2w_span_end
  const __half* logit_tiles = nullptr;  // output embedding as the persistent step kernel's tile stream
  DLayer* d_layers = nullptr;   // device copy of the decoder layer pointer table (persistent step kernel)
  unsigned* d_bar = nullptr;
  unsigned long long* d_prof = nullptr;  // B2W_DSTEP_PROF=1: per-phase timestamps of the persistent step kernel
  int dstep_grid = 0;
  // compute_type int8*: the decoder's linear layers (and the output embedding) are quantised per output channel; the persistent step
  // kernel streams them as int8 (w8), every other path uses the de-quantised fp16 values.  w8_fake keeps fp16 tiles of the same
  // de-quantised values (B2W_W8_FAKE=1: the reference the int8 stream is tested against).
  bool w8 = false, w8_fake = false;
  bool use_dstep = true;
  // many-row persistent step kernel (bstep.cu): decoder weights as 16 KB wgmma atoms + per-row sums for the deferred LayerNorm
  bool use_bstep = true;     // B2W_BSTEP=0 falls back to the multi-kernel step for R > 8
  bool bstep_all = false;    // B2W_BSTEP=all: also for R <= 8 (instead of dstep_kernel)
  int bstep_stop = 0;        // B2W_BSTEP_STOP=n: run only the first n grid phases of every step (debug)
  bool bstep_packed = false;
  BLayer* d_blayers = nullptr;
  const void* logit_atoms = nullptr;
  const float* logit_scale = nullptr;
  float *d_qkv32 = nullptr, *d_cq32 = nullptr, *d_h32 = nullptr, *d_stats = nullptr, *d_gpart = nullptr, *d_stpart = nullptr;
  __half *d_h16 = nullptr, *d_xn16 = nullptr;
  bool use_mma_xattn = true;  // decode cross attention on mma.sync (dstep.cu) instead of the SIMT kernel (B2W_XATTN_IMPL=simt)
  DecBindings h_bind{};
  SearchParams h_params{};
  // search buffers
  SearchBuffers sb{};
  void* sb_blob = nullptr;
  int sb_B = 0, sb_K = 0;
  int* h_pinned = nullptr;    // pinned host scratch

  // step graph cache
  cudaGraphExec_t step_graph = nullptr;
  int64_t step_graph_kernels = 0;
  std::vector<uint8_t> step_graph_key;

  // measurement
  bool timing = false;
  std::vector<StageTimer> timers;
  double t_ms[B2W_T_COUNT] = {0};
  int64_t t_cnt[B2W_T_COUNT] = {0};
  int64_t launches = 0, decode_steps = 0;
  double decode_alg_bytes = 0;

  bool use_ref_gemm = false, use_ref_attn = false, use_ref_gemv = false, use_graph = true;

  ~Model();
};

}  // namespace b2w
