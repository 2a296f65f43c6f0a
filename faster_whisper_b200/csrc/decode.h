// Decoder-side device structures shared by decode.cu, search.cu and engine.cu.
#pragma once
#include "engine.h"

namespace b2w {

struct RowInfo {
  int chunk;  // batch item the row belongs to
  int slot;   // self-KV slot the row writes at `pos`
  int pos;    // absolute decoder position of the token being fed
  int pad;
};

enum GvMode { GV_QKV = 0, GV_F16 = 1, GV_GELU_F16 = 2, GV_RESID_LN = 3, GV_F32 = 4 };

struct GvArgs {
  const __half* x = nullptr;  // [R_pad][K] fp16 activations
  const __half* W = nullptr;  // [N_pad16][K]
  const float* bias = nullptr;
  int R = 0, N = 0, K = 0, mode = GV_F16;
  // GV_QKV
  const RowInfo* rows = nullptr;
  __half* kcache = nullptr;
  __half* vcache = nullptr;
  int d = 0, n_ctx = 0, slots = 0;
  // outputs
  __half* out_h = nullptr;
  float* out_f = nullptr;
  long long ldo = 0;
  // GV_RESID_LN: xres[R][N] += ..., then xn_out = LN(xres) by the last CTA
  float* xres = nullptr;
  const float* ln_g = nullptr;
  const float* ln_b = nullptr;
  __half* xn_out = nullptr;
  int* counter = nullptr;
};
void skinny_gemm(const GvArgs& a, cudaStream_t s);
void skinny_ref(const __half* x, const __half* W, const float* bias, float* y, int R, int N, int K, cudaStream_t s);

void embed_ln(const int* tokens, const RowInfo* rows, const __half* tok_emb, const float* pos_emb, const float* g,
              const float* b, float* x, __half* xn, int R, int d, int n_vocab, cudaStream_t s);

struct SelfAttnArgs {
  const RowInfo* rows;
  const __half* q;        // [R][d]
  const __half* kcache;   // this layer: [chunk][pos][slot][d]
  const __half* vcache;
  const uint8_t* anc;     // [2][chunk][slot][n_ctx]; buffer (pos & 1) is current
  __half* out;            // [R][d]
  int d, n_ctx, slots;
  long long anc_buf_stride;
};
void dec_self_attn(const SelfAttnArgs& a, int R, int H, cudaStream_t s);

// Encoder binding of one decode chunk (one entry per chunk of a pass or slot of a step, in device memory): the chunk attends to
// item `item` of an encoder output whose cross-attention K/V is xkv.  The step kernels read their chunk's entry, so the captured
// CUDA graph of a decode step does not depend on which encoder outputs (or which items of them) the chunks decode.
struct DecBindings {
  const __half* xkv;  // [L][2][B_total][H][T][64]
  int B_total;
  int item;
};

void search_configure();  // per-device kernel attributes (must run outside stream capture)

// ---- search (search.cu) ------------------------------------------------------------------------------------
constexpr int kMaxBeam = 16;       // rows per chunk (beam_size or best_of)
constexpr int kMaxCand = 2 * kMaxBeam;
constexpr int kMaxFinishTarget = 32;  // largest round(beam * patience): a chunk stops once it has this many finished hypotheses
// Finished hypotheses kept per chunk.  Up to K hypotheses finish in one step, so a chunk that stops at max_finished can end with
// max_finished + K - 1 of them; every one is kept, as CTranslate2 does (32 + 16 - 1, rounded up).
constexpr int kMaxFinished = 48;

struct SearchParams {
  int n_vocab, vpad;           // real vocabulary and padded logits row stride
  int B, K;                    // chunks, rows per chunk
  int mode;                    // 0 beam, 1 greedy/sampling (independent rows)
  int ncand;                   // beam: 2K ; greedy: 1
  int max_finished;            // round(K * patience), at most kMaxFinishTarget
  int allow_early_exit;
  int num_hyp;
  float length_penalty, repetition_penalty;
  int no_repeat_ngram;
  int suppress_blank;
  int n_suppress_begin;
  int suppress_begin[8];
  int max_initial_ts;
  int eot, no_timestamps, timestamp_begin, no_speech;
  int sampling_topk;
  float temperature;
  unsigned long long seed;
  int fake_logits;
};

// Per-chunk search state that a decode session changes when it gives a slot to a new item.
struct ChunkParams {
  int prompt_len;
  int max_steps;               // generated tokens allowed (max_length - prompt_len)
  int item;                    // keys the sampling noise with the row within the chunk, so draws do not depend on the slot
  int timestamp_rules;         // the prompt has no <|notimestamps|>
  int ns_first;                // no_speech prob comes from the first decode step (sot is the last prompt token)
  int pad[3];
};

// A slot's new occupant: search_reset_slots clears the slot's search state and starts its rows at the prompt's last token.
struct SlotReset {
  int slot;
  int last_token;
  int done;                    // 1: the slot stays idle (counted as done)
  int pad;
  ChunkParams cp;
};

// All mutable search state lives on the device so a decode step needs no host round trip.
struct SearchState {
  int step;                    // generated-token index of the step being computed
  int n_done;                  // chunks finished
  int cur;                     // which history buffer is current (0/1)
  int pad;
};

struct SearchBuffers {
  SearchState* state;          // [1]
  const SearchParams* params;  // [1] device copy of the options of the running generate() call
  ChunkParams* chunk;          // [B]
  RowInfo* rows;               // [B*K]
  int* tokens_in;              // [B*K] token fed at this step
  float* cum;                  // [2][B*K]
  int* hist;                   // [2][B*K][n_ctx]   generated tokens
  uint8_t* anc;                // [2][B*K][n_ctx]   self-KV slot ancestry (indexed by absolute position)
  float* cand_score;           // [B*K][kMaxCand]
  int* cand_tok;               // [B*K][kMaxCand]
  const uint8_t* suppress;     // [vpad] 1 = always suppressed
  int* done;                   // [B]
  int* fin_count;              // [B]
  float* fin_score;            // [B][kMaxFinished]   raw cumulative log-prob
  int* fin_len;                // [B][kMaxFinished]
  int* fin_tok;                // [B][kMaxFinished][n_ctx]
  float* no_speech;            // [B]
  float* row_margin;           // [B*K] diagnostic: smallest top-1/top-2 gap seen (greedy)
  int n_ctx;
};

// `p` lives in device memory (SearchBuffers::params) so a captured step graph is independent of the options
void search_rows(const float* logits, int R, int vpad, const SearchBuffers& b, cudaStream_t s);
void search_update(int B, const SearchBuffers& b, cudaStream_t s);
// resets slot resets[i].slot of a B x K search for its new occupant; the other slots are not touched
void search_reset_slots(const SlotReset* resets, int n, int B, int K, const SearchBuffers& b, cudaStream_t s);
void fake_logits(float* logits, int R, const SearchBuffers& b, cudaStream_t s);
void no_speech_from_logits(const float* logits, int row_stride, int R, int rows_per_chunk, int row_in_chunk, int n_vocab,
                           int no_speech_id, float* out, cudaStream_t s);
void lang_probs_from_logits(const float* logits, int row_stride, int B, int lang_begin, int n_lang, float* out, cudaStream_t s);
// Whisper.align helpers (search.cu)
void row_target_probs(const float* logits, int row_stride, int R, int n_vocab, const int* targets, float* out, cudaStream_t s);
// Row r of the pass (chunk b = r / rows_per_chunk) writes out[b][head][rows[r].pos][0..nf) of an [items][n_heads][n_tok][nf]
// capture, with the keys of the encoder item bind[b] names.
void align_probs(const __half* q, const DecBindings* bind, const RowInfo* rows, int layer, const int2* heads, int n_heads, float* out,
                 int n_tok, int nf, int R, int rows_per_chunk, int H, int T, int d, cudaStream_t s);

// ---- Whisper.align post-processing (align.cu) ----------------------------------------------------------------------------
constexpr int kAlignMaxRows = 449;  // DTW rows (n_text + 1) the kernels take: more than a 448-position decoder can force

// Items of one align group, all with the same strides.  Item b: items[b] = (n_tok, nf, row0, n_rows); its capture is
// cap[b][n_heads][tok_stride][nf_stride], and the DTW runs over its rows row0 .. row0 + n_rows - 1 (n_rows = 0: no path).
struct AlignBatch {
  const float* cap;
  double* stats;      // [items][n_heads][2][nf_stride]: mean, std over the tokens
  double* cost;       // [items][row_stride][nf_stride]
  const int4* items;
  int n_heads, tok_stride, nf_stride, row_stride, width;
  int2* pairs;        // [items][row_stride + nf_stride] (text index, frame index) from (0, 0)
  int* n_pairs;       // [items]
};
void align_check(const AlignBatch& a);
void align_cost(const AlignBatch& a, int n_items, cudaStream_t s);  // cap -> stats -> cost
void align_dtw(const AlignBatch& a, int n_items, cudaStream_t s);   // cost -> pairs, n_pairs

}  // namespace b2w
