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
 * streams them as int8 and applies the scale to the fp32 sums, all other paths multiply with the de-quantised fp16 values. */
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

/* config.json "alignment_heads" of a converted model (transcribe.py:700-710 reads the model directory): n_pairs
 * (layer, head) pairs; n_pairs = 0 restores the default (every head of the last half of the decoder layers). */
int b2w_model_set_alignment_heads(b2w_model* m, const int32_t* layer_head_pairs, int32_t n_pairs);

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
/* C = epilogue(A[M,K] * W[N,K]^T + bias) through the wgmma (impl=0) or reference SIMT (impl=1) GEMM. */
int b2w_debug_gemm(int32_t device, int32_t impl, const float* a, const float* w, const float* bias,
                   int32_t M, int32_t N, int32_t K, int32_t gelu, float* c_out);
/* softmax(QK^T/8)V for [B,T,H*64] fp16-rounded inputs through the wgmma (0) or reference (1) kernel. */
int b2w_debug_attention(int32_t device, int32_t impl, const float* qkv, int32_t B, int32_t T, int32_t H,
                        float* out);
/* one decode-style skinny GEMM y[R,N] = x[R,K] W[N,K]^T + b through the mma.sync (0) or reference (1) path */
int b2w_debug_gemv(int32_t device, int32_t impl, const float* x, const float* w, const float* bias,
                   int32_t R, int32_t N, int32_t K, float* y_out);
/* teacher-forced logits: run the decoder over tokens [batch, n] and return float32 [batch, n, n_vocab] */
int b2w_debug_logits(b2w_model* m, b2w_encoded* e, const int32_t* tokens, int32_t n, int32_t batch,
                     float* logits_out);

/* decoder workspace of the last decode step as float32 (fp16 buffers are widened): which = 0 residual stream [R][d], 1 raw QKV
 * sums [R][3d], 2 raw cross-q sums [R][d], 3 raw FFN hidden sums [R][4d], 4 attention output [R][d], 5 GELU(hidden) [R][4d],
 * 6 final LayerNorm output [R][d], 7 LayerNorm statistics [3L][80][2], 8 logits [R][vpad]; n = number of floats to copy.
 * With B2W_BSTEP_STOP=<p> the many-row step kernel stops after p grid phases, so this bisects it phase by phase. */
int b2w_debug_fetch(b2w_model* m, int32_t which, float* out, int64_t n);

#ifdef __cplusplus
}
#endif
#endif /* B200WHISPER_H_ */
