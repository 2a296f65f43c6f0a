/*
 * libb200whisper — C ABI of the H100-native Whisper engine.
 *
 * This is the drop-in boundary for the hot path of SYSTRAN/faster-whisper: every entry point replaces one
 * member of the `ctranslate2` Python API exactly as `faster_whisper/transcribe.py` consumes it (file:line
 * below are relative to the reference tree).  Plain pointers and sizes only; no torch / CUDA types.
 * All functions return 0 on success, non-zero on failure; `b2w_last_error()` holds the message of the
 * last failure on the calling thread (the Python wrapper raises ValueError / RuntimeError from it, matching
 * how CTranslate2 surfaces C++ exceptions).
 *
 * Threading: a `b2w_model` serialises its own calls (one CUDA stream per model); use one model per GPU
 * and one host thread per model for replicas (transcribe.py:646-657 describes the same replica scheme).
 */
#ifndef B200WHISPER_H_
#define B200WHISPER_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2W_ABI_VERSION 1
#define B2W_MAX_TEXT_CTX 448
#define B2W_N_AUDIO_CTX 1500
#define B2W_N_FRAMES 3000

typedef struct b2w_model b2w_model;      /* replaces ctranslate2.models.Whisper (transcribe.py:689-698) */
typedef struct b2w_encoded b2w_encoded;  /* replaces the StorageView returned by Whisper.encode (transcribe.py:1400) */

/* Geometry + control-token ids.  CTranslate2 reads these from model.bin / config.json; here the caller
 * states them (faster_whisper_b200/config.py derives them from the size name / vocabulary). */
typedef struct b2w_config {
  int32_t n_mels, n_audio_ctx, n_audio_state, n_audio_head, n_audio_layer;
  int32_t n_vocab, n_text_ctx, n_text_state, n_text_head, n_text_layer;
  int32_t eot, sot, lang_begin, num_languages, translate, transcribe, sot_lm, sot_prev;
  int32_t no_speech, no_timestamps, timestamp_begin;
  int32_t n_suppress_begin;       /* config.json "suppress_ids_begin" ([" ", eot]) used by suppress_blank */
  int32_t suppress_begin[8];
} b2w_config;

enum { B2W_F32 = 0, B2W_F16 = 1 };

/* One named weight tensor in host memory (OpenAI Whisper state-dict names, row-major). */
typedef struct b2w_tensor {
  const char* name;
  const void* data;
  int32_t dtype;  /* B2W_F32 | B2W_F16 */
  int32_t ndim;
  int64_t shape[4];
} b2w_tensor;

/* Whisper.generate keyword arguments (transcribe.py:222-236, 1446-1459) with CTranslate2's defaults. */
typedef struct b2w_gen_opts {
  int32_t beam_size;                   /* 5 */
  float patience;                      /* 1 */
  int32_t num_hypotheses;              /* 1 */
  float length_penalty;                /* 1 */
  float repetition_penalty;            /* 1 */
  int32_t no_repeat_ngram_size;        /* 0 */
  int32_t max_length;                  /* 448, counts the prompt */
  int32_t return_scores;               /* informational; scores are always written */
  int32_t return_no_speech_prob;
  int32_t max_initial_timestamp_index; /* 50 */
  int32_t suppress_blank;              /* 1 */
  const int32_t* suppress_tokens;      /* explicit ids (faster-whisper expands -1 itself, transcribe.py:1884-1907) */
  int32_t n_suppress_tokens;
  int32_t sampling_topk;               /* 1 = argmax, 0 = full-vocabulary sampling */
  float sampling_temperature;          /* 1 */
  uint64_t seed;                       /* sampling only */
  int32_t debug_fake_logits;           /* tests: replace the decoder by the hash-logits generator (see oracle) */
} b2w_gen_opts;

/* ---- diagnostics ------------------------------------------------------------------------------- */
const char* b2w_last_error(void);
int b2w_abi_version(void);
int b2w_device_count(int* count);

/* ---- model ------------------------------------------------------------------------------------- */
/* ctranslate2.models.Whisper(model_path, device, device_index, compute_type, ...) (transcribe.py:689-698).
 * compute_type: "float16" | "default" | "auto" -> fp16 weights; "int8" | "int8_float16" | ... -> the decoder's linear layers and the
 * output embedding are quantised per output channel (symmetric, scale = max|w|/127) at load; the single-stream decode kernel
 * streams them as int8 and applies the scale to the fp32 sums, all other paths multiply with the de-quantised fp16 values.
 * "float8_float16" -> the encoder's four linear layers per block (QKV, out-projection, FFN1, FFN2) run as e4m3 tensor-core GEMMs:
 * weights quantised per output channel at load, their inputs per token row (b2w_debug_quantize_e4m3's rule); everything else,
 * the decoder included, is as "float16". */
int b2w_model_create(const b2w_config* cfg, const b2w_tensor* tensors, int32_t n_tensors, int32_t device,
                     const char* compute_type, b2w_model** out);
void b2w_model_destroy(b2w_model* m);
/* Whisper.is_multilingual / n_mels / device_index (transcribe.py:379,472,1394) */
int b2w_model_info(const b2w_model* m, b2w_config* cfg_out, int32_t* device_out);
int b2w_model_sync(b2w_model* m);

/* ---- log-mel front end --------------------------------------------------------------------------
 * FeatureExtractor.__call__(waveform, padding=160) (feature_extractor.py:198-230): host PCM in,
 * host float32 [n_mels, n_frames] out, n_frames = 1 + n_samples/160 (the reference's last-frame drop
 * included).  Computed on `device` by the fused STFT+mel+log kernel. */
int b2w_logmel(int32_t device, int32_t n_mels, const float* pcm, int64_t n_samples, int32_t padding,
               float* out, int64_t out_capacity, int32_t* n_frames_out);
int b2w_logmel_frames(int64_t n_samples, int32_t padding);

/* ---- encoder ------------------------------------------------------------------------------------
 * StorageView.from_array + Whisper.encode(features, to_cpu) (transcribe.py:1391-1400, 1873-1876):
 * host float32 C-contiguous [batch, n_mels, 3000] -> device-resident encoder output. */
int b2w_encode(b2w_model* m, const float* features, int32_t batch, b2w_encoded** out);
/* Fused path used by BatchedInferencePipeline: per-chunk host PCM (<= 30 s each) -> log-mel
 * (feature_extractor(chunk)[..., :-1] + pad_or_trim, transcribe.py:463-467,514-516) -> encoder, the
 * features never leave HBM.  features_out (optional, may be NULL) receives [batch, n_mels, 3000]. */
int b2w_encode_audio(b2w_model* m, const float* const* pcm, const int64_t* n_samples, int32_t batch,
                     float* features_out, b2w_encoded** out);
int b2w_encoded_shape(const b2w_encoded* e, int64_t shape_out[3]);
/* to_cpu=True / debugging: copy [batch, 1500, d] out as float32. */
int b2w_encoded_to_host(b2w_model* m, const b2w_encoded* e, float* out);
void b2w_encoded_free(b2w_encoded* e);
/* One single-item encoder output per batch item of e: outs[b] receives item b, bit for bit (encoder output [1, 1500, d] and
 * cross-attention K/V [L][K|V][1][H][1500][64]), in device memory of its own, so each can be freed on its own.  e is not
 * changed (its cross-attention K/V is computed first when no decode has yet), and the caller still frees it. */
int b2w_encoded_split(b2w_model* m, const b2w_encoded* e, b2w_encoded** outs);
/* Device bytes of the model's live encoder outputs (including those only a decode session still holds) and bytes parked in
 * its buffer pool for reuse. */
int b2w_memory_get(b2w_model* m, int64_t* encoded_bytes, int64_t* pool_bytes);

/* ---- decoder ------------------------------------------------------------------------------------
 * Whisper.generate(encoder_output, prompts, **opts) -> [WhisperGenerationResult] (transcribe.py:222-236,
 * 1446-1459).  prompts: [batch, prompt_len] (all prompts of one call have equal length, as the reference
 * always sends).  Outputs per batch item and hypothesis h < num_hypotheses, best first:
 *   out_ids    [batch, num_hypotheses, max_length]  generated ids (prompt and EOS stripped)
 *   out_lens   [batch, num_hypotheses]
 *   out_scores [batch, num_hypotheses]              cum_logprob / len**length_penalty
 *   out_no_speech [batch]                           softmax prob of <|nospeech|> at the SOT position */
int b2w_generate(b2w_model* m, b2w_encoded* e, const int32_t* prompts, int32_t prompt_len, int32_t batch,
                 const b2w_gen_opts* opts, int32_t* out_ids, int32_t* out_lens, float* out_scores,
                 float* out_no_speech);
void b2w_gen_opts_default(b2w_gen_opts* o);

/* ---- decode session (continuous batching) ------------------------------------------------------
 * A fixed set of slots (up to 80 / K chunks of K = beam_size, or num_hypotheses when beam_size is 1, rows) decoding
 * with one set of generate options; a slot whose item finishes takes the next queued item at the next poll.
 *   b2w_session_create : *slots: 0 for as many slots as a step takes, else at most that many; receives the number of
 *                        slots (the most items one b2w_session_run returns).
 *                        The session must be destroyed before its model.
 *   b2w_session_push   : queues item item_index of e with its own prompt (any length, <|startoftranscript|> anywhere) and
 *                        max_length (prompt_len < max_length <= opts->max_length); item_id_out receives its id (0, 1, ... in
 *                        push order), which also keys its sampling noise.  The session keeps e alive while it reads it.
 *   b2w_session_run    : decodes until at least one item finishes, or returns n_out = 0 when the queue and the slots are
 *                        empty.  Outputs j < n_out: out_item_ids[j]; out_ids [slots][num_hypotheses][opts->max_length],
 *                        out_lens / out_scores [slots][num_hypotheses], out_no_speech [slots], as b2w_generate.
 *   b2w_session_pending: queued plus decoding items.
 *   b2w_session_counters: decode steps run, and rows of occupied slots summed over them (a slot counts until the poll, every
 *                        4 steps, that sees it finish: at most 3 steps past its item's last).
 *   b2w_session_debug_record / b2w_session_debug_logits (tests): for a session with one row per slot, record every step's raw
 *                        logits of each occupied slot; fetch an item's [n_steps][n_vocab] once it has finished (steps from its
 *                        first; the last steps may be idle steps after it finished). */
typedef struct b2w_session b2w_session;
int b2w_session_create(b2w_model* m, const b2w_gen_opts* opts, int32_t* slots, b2w_session** out);
int b2w_session_push(b2w_session* s, b2w_encoded* e, int32_t item_index, const int32_t* prompt, int32_t prompt_len,
                     int32_t max_length, int32_t* item_id_out);
int b2w_session_run(b2w_session* s, int32_t* n_out, int32_t* out_item_ids, int32_t* out_ids, int32_t* out_lens,
                    float* out_scores, float* out_no_speech);
int b2w_session_pending(b2w_session* s, int32_t* n_out);
int b2w_session_counters(b2w_session* s, int64_t* steps, int64_t* live_rows);
int b2w_session_debug_record(b2w_session* s);
int b2w_session_debug_logits(b2w_session* s, int32_t item_id, float* out, int32_t capacity_steps, int32_t* n_steps_out);
void b2w_session_destroy(b2w_session* s);

/* Whisper.detect_language(encoder_output) (transcribe.py:215,1193,1823): probs [batch, num_languages]
 * over the language tokens (softmax restricted to them), id order. */
int b2w_detect_language(b2w_model* m, b2w_encoded* e, float* probs);

/* Whisper.align(encoder_output, start_sequence, text_tokens, num_frames, median_filter_width=7)
 * (transcribe.py:1709-1715; consumer :1698-1766) for ONE batch item: teacher-forces
 * start_sequence + <|notimestamps|> + text_tokens + <|endoftext|>, captures the cross-attention probabilities of
 * the alignment heads over the first num_frames/2 encoder positions, normalises them over the token axis,
 * median-filters along time, averages the heads and runs DTW.  alignments_out receives n_pairs_out pairs
 * (text_index, time_index) over the n_text + 1 rows that predict text + eot, capacity in pairs
 * (n_text + 1 + num_frames/2 always suffices);
 * text_token_probs_out[n_text] = softmax probability of each text token at the position predicting it. */
int b2w_align(b2w_model* m, b2w_encoded* e, int32_t batch_index, const int32_t* start_sequence,
              int32_t n_start, const int32_t* text_tokens, int32_t n_text, int32_t num_frames,
              int32_t median_filter_width, int32_t* alignments_out, int32_t capacity_pairs,
              int32_t* n_pairs_out, float* text_token_probs_out);

/* b2w_align for every batch item of e in one call, item for item with b2w_align's contract.  Item b's text is
 * text_tokens[text_offsets[b] .. text_offsets[b+1]) (text_offsets[0] = 0, never decreasing) and its frames num_frames[b];
 * an item with no text gets no pairs.  Its pairs are alignments_out[pair_offsets_out[b] .. pair_offsets_out[b+1]) and its
 * probabilities text_token_probs_out[text_offsets[b] .. text_offsets[b+1]).  capacity_pairs must be at least the sum of
 * n_text + 1 + min(1500, num_frames/2) over the items with text.  Items are decoded in groups of consecutive chunks; the
 * cost matrix and the DTW run on the device, and the host waits once at the end. */
int b2w_align_batch(b2w_model* m, b2w_encoded* e, const int32_t* start_sequence, int32_t n_start,
                    const int32_t* text_tokens, const int32_t* text_offsets, const int32_t* num_frames,
                    int32_t median_filter_width, int32_t* alignments_out, int32_t capacity_pairs,
                    int32_t* pair_offsets_out, float* text_token_probs_out);
/* b2w_align_batch over items of several encoder outputs: item j is batch index items[j] of encs[j], and
 * text_offsets / num_frames / pair_offsets_out / probabilities are indexed by j as b2w_align_batch indexes them by b.
 * b2w_align_batch is this call with encs[j] = e and items[j] = j. */
int b2w_align_items(b2w_model* m, const b2w_encoded* const* encs, const int32_t* items, int32_t n_items,
                    const int32_t* start_sequence, int32_t n_start, const int32_t* text_tokens, const int32_t* text_offsets,
                    const int32_t* num_frames, int32_t median_filter_width, int32_t* alignments_out, int32_t capacity_pairs,
                    int32_t* pair_offsets_out, float* text_token_probs_out);

/* config.json "alignment_heads" of a converted model (transcribe.py:700-710 reads the model directory): n_pairs
 * (layer, head) pairs; n_pairs = 0 restores the default (every head of the last half of the decoder layers). */
int b2w_model_set_alignment_heads(b2w_model* m, const int32_t* layer_head_pairs, int32_t n_pairs);

/* ---- voice activity -----------------------------------------------------------------------------
 * The Silero VAD v6 network (16 kHz) of vad.py's SileroVADModel on the GPU, fp32 throughout.  Weights (float32, names and shapes
 * as faster_whisper_b200/silero.py reads them from the ONNX file): basis [258][256], conv{0..3}.weight [out][in][3] and .bias
 * [out] (129->128, 128->64, 64->64, 64->128), lstm.w_ih [512][128], lstm.w_hh [512][128], lstm.bias [512] (b_ih + b_hh; gate
 * blocks i, o, f, c), decoder.weight [128], decoder.bias [1].  Every name and shape is checked before any device work.  A handle
 * owns its stream and buffers and serialises its calls. */
typedef struct b2w_vad b2w_vad;
int b2w_vad_create(int32_t device, const b2w_tensor* weights, int32_t n_weights, b2w_vad** out);
void b2w_vad_destroy(b2w_vad* vad);
/* One speech probability per 512-sample window of host PCM (n_samples a positive multiple of 512): probs_out[n_samples / 512],
 * capacity in floats.  As SileroVADModel: window n sees the last 64 samples of window n-1 first (zeros for n = 0), and the
 * last window's own final 64 samples count as zero.  The LSTM state starts at zero; the audio runs through in blocks of windows
 * (b2w_vad_set_block) with the state carried on the device, and the result does not depend on the block size. */
int b2w_vad_probs(b2w_vad* vad, const float* pcm, int64_t n_samples, float* probs_out, int64_t capacity);
/* b2w_vad_probs for n_streams independent recordings in one sequence of launches: stream i is pcm[i][n_samples[i]] (each a
 * positive multiple of 512), and its probabilities follow those of stream i - 1 in probs_out (capacity in floats, at least the
 * total number of windows).  Each launch runs one 4-CTA LSTM cluster per stream that still has windows, with that stream's state
 * carried on the device, so every stream's probabilities are bit-identical to b2w_vad_probs on that stream alone, whatever
 * the streams, their lengths and the block size.  Every argument is checked before any device work. */
int b2w_vad_probs_multi(b2w_vad* vad, const float* const* pcm, const int64_t* n_samples, int32_t n_streams, float* probs_out,
                        int64_t capacity);
/* Windows per block (default 32768, about 17.5 min of audio), summed over the streams of a launch and split evenly over the
 * streams that still have windows.  The block buffers take 4.6 KB of device memory per window (PCM, LSTM inputs, hidden
 * states, probabilities): 151 MB at the default; each stream adds 1.3 KB (its LSTM state and the context before its slice). */
int b2w_vad_set_block(b2w_vad* vad, int64_t windows);
/* Device time of the last b2w_vad_probs or b2w_vad_probs_multi call in milliseconds: window kernel, recurrence, decoder
 * (CUDA events), summed over its launches. */
int b2w_vad_timing(b2w_vad* vad, double ms_out[3]);

/* ---- measurement --------------------------------------------------------------------------------
 * CUDA-event stage timers accumulated since the last reset (the roofline report in bench.py). */
enum { B2W_T_MEL = 0, B2W_T_ENCODER = 1, B2W_T_CROSSKV = 2, B2W_T_PREFILL = 3, B2W_T_DECODE = 4,
       B2W_T_H2D = 5, B2W_T_D2H = 6, B2W_T_COUNT = 8 };
int b2w_timing_enable(b2w_model* m, int32_t on);
int b2w_timing_reset(b2w_model* m);
int b2w_timing_get(b2w_model* m, double ms_out[B2W_T_COUNT], int64_t counts_out[B2W_T_COUNT]);
/* Device-side span timer on the model's stream (bench.py: the timed region of K steps): `begin` records a CUDA event on the
 * stream, `end` records a second one, waits for it and returns the elapsed milliseconds between the two. */
int b2w_span_begin(b2w_model* m);
int b2w_span_end(b2w_model* m, double* ms_out);
/* kernels launched by this library on this model since the last reset (bench.py "gpu_launches"),
 * decode steps executed, and bytes the decode steps had to move (algorithmic: W + B*X + R*t*S). */
int b2w_counters_get(b2w_model* m, int64_t* launches, int64_t* decode_steps, double* decode_alg_bytes);

/* ---- test hooks (used by tests/ only) ----------------------------------------------------------- */
/* Epilogues of the dense GEMM (csrc/engine.h Epilogue). */
enum { B2W_EPI_F16 = 0, B2W_EPI_GELU_F16 = 1, B2W_EPI_RESID_F32 = 2, B2W_EPI_GELU_POS_F32 = 3, B2W_EPI_F16_XKV = 4,
       B2W_EPI_F32 = 5, B2W_EPI_QKV_CACHE = 6 };

/* One dense GEMM as the engine states it (csrc/engine.h GemmArgs), with host buffers.  fp16 buffers are IEEE half bit
 * patterns.  Output buffers are in/out: they are copied to the device, run, and copied back whole, so elements the kernel must
 * not write keep whatever the caller put there. */
typedef struct b2w_gemm_desc {
  /* A: fp16 [a_batch][a_rows][a_cols] at the given element strides inside a host buffer of a_elems halves; K index k of tap t
   * reads element (row + tap_row[t], tap_col[t] + k), zero outside the a_rows x a_cols box */
  const uint16_t* a;
  int64_t a_elems;
  int32_t a_batch, a_rows, a_cols;
  int64_t a_row_stride, a_batch_stride;
  int32_t taps, tap_row[3], tap_col[3], k_per_tap; /* k_per_tap: multiple of 64 */
  const uint16_t* w;                               /* fp16 [N][taps * k_per_tap] */
  const float* bias;                               /* [N] or NULL */
  int32_t N, rows, epilogue, narrow_tiles;         /* N: multiple of 32; rows per batch item */
  /* out: fp16 (F16, GELU_F16, F16_XKV, QKV_CACHE) or float32 (RESID_F32, GELU_POS_F32, F32), out_elems elements;
   * element (b, row, n) at b * out_batch_stride + row * out_ld + n.  RESID_F32 adds to out in place, as the engine does. */
  void* out;
  int64_t out_elems, out_ld, out_batch_stride;
  const float* pos;                                /* GELU_POS_F32: [rows][N] */
  int32_t xkv_d, xkv_heads, xkv_T, xkv_B;          /* F16_XKV: out is [N / (2 xkv_d)][2][xkv_B][xkv_heads][xkv_T][64] */
  /* QKV_CACHE (a_batch = 1, N = 3 qkv_d): q -> out [rows][qkv_d]; k, v -> kcache / vcache [chunk][n_ctx][slots][qkv_d] at the
   * (chunk, slot, pos) of rowinfo [rows][4] (the fourth int is unused); both caches hold cache_elems halves */
  const int32_t* rowinfo;
  uint16_t* kcache;
  uint16_t* vcache;
  int64_t cache_elems;
  int32_t qkv_d, n_ctx, slots;
  int32_t max_ctas;            /* > 0: at most this many persistent CTAs (tests: several tiles per CTA); 0: one per SM */
  int32_t block_n_out, grid_out; /* written: the tile width and grid the plan chose (impl 0) */
} b2w_gemm_desc;

/* Run one described GEMM through the wgmma kernel (impl=0) or the plain SIMT reference of the same contract (impl=1).  Every
 * argument (shapes, strides, buffer extents, row table) is checked before anything runs on the device. */
int b2w_debug_gemm(int32_t device, int32_t impl, b2w_gemm_desc* desc);
/* compute_type "float8_float16": the encoder's e4m3 GEMM on given codes (e4m3 bytes) and scales, a [rows][K] and w [N][K]
 * (K a multiple of 64, N of 32): out[r][n] = epilogue(a_scale[r] * w_scale[n] * sum_k a[r][k] w[n][k] + bias[n]) for epilogue
 * B2W_EPI_F16 or B2W_EPI_GELU_F16 (out fp16 [rows][N]) or B2W_EPI_RESID_F32 (out float32 [rows][N], added to in place).  bias
 * may be NULL; max_ctas as in b2w_gemm_desc.  Arguments are checked before any device work. */
int b2w_debug_gemm_fp8(int32_t device, const uint8_t* a, const float* a_scale, int32_t rows, int32_t K, const uint8_t* w,
                       const float* w_scale, int32_t N, const float* bias, int32_t epilogue, void* out, int32_t max_ctas);
/* The encoder's e4m3 row quantisation (per row: scale = amax / 448, 1 when amax is 0; code = e4m3(x / scale), round to nearest
 * even, saturating): of fp16 rows x [rows][K] (K a multiple of 8), and of the float32 LayerNorm output of x [rows][d] (gamma and
 * beta both NULL for no affine).  codes [rows][K|d], scales [rows]. */
int b2w_debug_quantize_e4m3(int32_t device, const uint16_t* x, int32_t rows, int32_t K, uint8_t* codes, float* scales);
int b2w_debug_layernorm_e4m3(int32_t device, const float* x, const float* gamma, const float* beta, int32_t rows, int32_t d,
                             uint8_t* codes, float* scales);
/* softmax(QK^T/8)V for [B,T,H*64] fp16-rounded inputs through the wgmma (0) or reference (1) kernel. */
int b2w_debug_attention(int32_t device, int32_t impl, const float* qkv, int32_t B, int32_t T, int32_t H,
                        float* out);
/* Modes of the decode GEMM (csrc/decode.h GvMode). */
enum { B2W_GV_QKV = 0, B2W_GV_F16 = 1, B2W_GV_GELU_F16 = 2, B2W_GV_RESID_LN = 3, B2W_GV_F32 = 4 };

/* One decoder GEMM y = x[R,K] W[N,K]^T + bias of R <= 80 rows, with the epilogue of `mode`.  Output buffers are in/out as in
 * b2w_gemm_desc. */
typedef struct b2w_gemv_desc {
  const uint16_t* x;  /* fp16 [R][K] */
  const uint16_t* w;  /* fp16 [N][K] */
  const float* bias;  /* [N] or NULL */
  int32_t R, N, K, mode;
  int32_t route;      /* 0: the skinny mma.sync kernel; 1: the path the decoder takes for this shape */
  /* QKV (N = 3 d): q -> out [R][d]; k, v -> kcache / vcache [chunk][n_ctx][slots][d] at rows[r] = (chunk, slot, pos, -) */
  const int32_t* rows;
  uint16_t* kcache;
  uint16_t* vcache;
  int64_t cache_elems;
  int32_t d, n_ctx, slots;
  /* F16, GELU_F16: fp16 [R][N]; F32: float32 [R][ldo]; QKV: fp16 [R][d]; out_elems elements */
  void* out;
  int64_t out_elems, ldo;
  /* RESID_LN (N <= 1280): xres [R][N] += y, then xn [R][N] (fp16) = LayerNorm(xres) * ln_g + ln_b (NULL: no affine) */
  float* xres;
  const float* ln_g;
  const float* ln_b;
  uint16_t* xn;
  int32_t path_out;   /* written: 0 the skinny kernel ran, 1 the wgmma GEMM ran */
} b2w_gemv_desc;

/* Run one described decoder GEMM (impl=0), or with impl=1 and mode F32 the one-thread-per-output reference.  Every argument is
 * checked before anything runs on the device. */
int b2w_debug_gemv(int32_t device, int32_t impl, b2w_gemv_desc* desc);
/* teacher-forced logits: run the decoder over tokens [batch, n] and return float32 [batch, n, n_vocab] */
int b2w_debug_logits(b2w_model* m, b2w_encoded* e, const int32_t* tokens, int32_t n, int32_t batch,
                     float* logits_out);
/* Run the model's decode-step path (the one generate() would choose for n chunks x K rows, or B2W_STEP's) for n_steps steps with
 * forced inputs.  prompts [n][P]: positions 0..P-2 are prefilled into self-KV slot 0.  Step t feeds tokens[t][b*K+k] at position
 * P-1+t as row (chunk b, slot k).  For t >= 1 the row continues the history of slot parents[t][b*K+k] of the same chunk as it
 * stood after step t-1 (the relinking of the beam search); parents == NULL means every slot continues itself.
 * logits_out [n_steps][n*K][n_vocab].  Every argument is checked before anything runs on the device. */
int b2w_debug_step_logits(b2w_model* m, b2w_encoded* e, const int32_t* prompts, int32_t P, int32_t n, int32_t K,
                          int32_t n_steps, const int32_t* tokens, const int32_t* parents, float* logits_out);

/* Finished-hypothesis slots the search keeps per chunk (b2w_search_desc.fin_*). */
#define B2W_MAX_FINISHED 48

/* One step of the on-device search, the two kernels a decode step runs after the decoder (logits processors, log-softmax and
 * row top-k, then the beam / greedy update), on state the caller supplies.  The search parameters and the suppress mask are
 * derived from cfg, opts and prompt by the code b2w_generate uses.  Rows r = b * K + k (chunk b, slot k) sit at position
 * P - 1 + t.  In / out arrays are read before the step and overwritten with the state after it. */
typedef struct b2w_search_desc {
  const b2w_config* cfg;       /* geometry and control tokens of the model */
  const b2w_gen_opts* opts;    /* generate options; K must be beam_size, or num_hypotheses when beam_size is 1 */
  const int32_t* prompt;       /* [P], the prompt of every chunk: it fixes the SOT index and whether timestamp rules apply */
  int32_t P, n, K, t;          /* prompt length, chunks, rows per chunk, step (tokens generated so far) */
  const float* logits;         /* [n*K][n_vocab] decoder output of the step */
  int32_t* hist;               /* in [n*K][t], out [n*K][t+1]: generated tokens of each row, relinked to the parent and extended */
  uint8_t* anc;                /* in [n*K][P-1+t], out [n*K][P+t]: self-KV slot of each position; the last is the row's parent */
  float* cum;                  /* in / out [n*K] cumulative log-prob */
  int32_t* done;               /* in / out [n] */
  int32_t* fin_count;          /* in / out [n] */
  int32_t* fin_len;            /* in / out [n][B2W_MAX_FINISHED]; -1 = empty.  Greedy rows: slot k >= 0 means row k finished */
  float* fin_score;            /* in / out [n][B2W_MAX_FINISHED] cumulative log-prob */
  int32_t* fin_tok;            /* out [n][B2W_MAX_FINISHED][t+1]: tokens of the slots this step wrote, -1 elsewhere */
  float* cand_score;           /* out [n*K][ncand] each row's candidates, best first (ncand = 2K in beam search, else 1) */
  int32_t* cand_tok;           /* out [n*K][ncand] */
  float* no_speech;            /* out [n] (written when the step computes it) */
  int32_t* tokens_in;          /* out [n*K] the token each row feeds at the next step */
  int32_t* pos;                /* out [n*K] the rows' next position */
  int32_t n_done;              /* in / out: chunks done (the device counter the host polls) */
} b2w_search_desc;

/* Run one search step as described.  Every argument is checked before anything runs on the device. */
int b2w_debug_search(int32_t device, b2w_search_desc* desc);

/* The cost matrix of Whisper.align from a capture[n_heads][n_tok][nf] of cross-attention probabilities: per head and frame
 * normalised over the tokens (population std), median-filtered along time (odd width, reflect padding, none when
 * nf <= width/2), averaged over the heads and negated, for rows n_start .. n_start + n_text: cost_out[n_text + 1][nf].
 * Every argument is checked before anything runs on the device. */
int b2w_debug_align_cost(int32_t device, const float* capture, int32_t n_heads, int32_t n_tok, int32_t nf, int32_t n_start,
                         int32_t n_text, int32_t median_filter_width, double* cost_out);

/* The DTW path of Whisper.align through cost[N][M] (N <= 449, M <= 1500): n_pairs_out (text index, frame index) pairs
 * from (0, 0) to (N - 1, M - 1) in pairs_out, which must hold N + M.  Arguments are checked before any device work. */
int b2w_debug_dtw(int32_t device, const double* cost, int32_t N, int32_t M, int32_t* pairs_out, int32_t capacity_pairs,
                  int32_t* n_pairs_out);

/* decoder workspace of the last decode step as float32 (fp16 buffers are widened): which = 0 residual stream [R][d], 1 the
 * many-row step kernel's split-K partial tiles of its last GEMM phase [CTA][R][128], 2 the per-k-atom partials of its last row
 * statistics [d/64][R][2], 4 attention output [R][d], 5 GELU(hidden) [R][4d], 6 final LayerNorm output [R][d], 7 LayerNorm
 * statistics [3L][R][2], 8 logits [R][vpad], 9 / 10 the self-attention K / V cache of every layer [L][chunk][n_ctx][slot][d]
 * (n / L elements from the start of each layer's cache), 11 the cross-attention K/V of the encoder output the last step read
 * [L][2][B][H][1500][64] (16-byte chunk c of key t at c ^ (t & 7)); n = number of floats to copy, at most the buffer's size.
 * With B2W_BSTEP_STOP=<p> the many-row step kernel stops after p grid phases, so this bisects it phase by phase. */
int b2w_debug_fetch(b2w_model* m, int32_t which, float* out, int64_t n);
/* The decoder's masked self-attention kernel on fp16 inputs: rows [R][4] = (chunk, slot, pos, -), q [R][64 H], kcache / vcache
 * [n_chunks][n_ctx][slots][64 H], anc [2][n_chunks][slots][n_ctx]: row r reads buffer pos & 1, key j < pos from slot
 * anc[pos & 1][chunk][slot][j] and key pos from its own slot.  out [R][64 H] fp16.  Arguments are checked before any device work. */
int b2w_debug_self_attn(int32_t device, const uint16_t* q, const uint16_t* kcache, const uint16_t* vcache, const uint8_t* anc,
                        const int32_t* rows, int32_t R, int32_t H, int32_t n_chunks, int32_t slots, int32_t n_ctx, uint16_t* out);
/* The decoder's beam-shared cross-attention kernel on fp16 inputs: q [n_chunks * rows_per_chunk][64 H] (row b * rows_per_chunk + i
 * of chunk b), kv [2][n_chunks][H][1500][64] one layer's K and V as the encoder output stores them (16-byte chunk c of key t at
 * c ^ (t & 7)).  out [n_chunks * rows_per_chunk][64 H] fp16.  Arguments are checked before any device work. */
int b2w_debug_cross_attn(int32_t device, const uint16_t* q, const uint16_t* kv, int32_t n_chunks, int32_t rows_per_chunk, int32_t H,
                         uint16_t* out);

#ifdef __cplusplus
}
#endif
#endif /* B200WHISPER_H_ */
