// Host-side engine: weight upload, encoder orchestration, generate loop, and the extern "C" ABI declared in
// include/b200whisper.h.  PyTorch is not involved: the library owns its device memory and one CUDA stream per
// model.  There is no CPU fallback — every entry point fails loudly when no sm_90 device is usable.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <deque>
#include <cmath>
#include <limits>
#include <numeric>

#include "model.h"
#include "vad.h"

namespace b2w {

// ---- error / counters ---------------------------------------------------------------------------------------
constexpr int kMaxRows = 80;  // decode rows of one step or forced pass (chunks x rows per chunk)

static thread_local std::string g_last_error;
static thread_local int64_t g_launches = 0;
void count_launch(int n) { g_launches += n; }

template <typename F>
static int guarded(F&& f) {
  try {
    f();
    return 0;
  } catch (const Error& e) {
    g_last_error = e.what();
    return e.invalid_argument ? 2 : 1;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return 1;
  }
}

struct DeviceGuard {
  int prev = 0;
  explicit DeviceGuard(int dev) {
    B2W_CUDA(cudaGetDevice(&prev));
    if (prev != dev) B2W_CUDA(cudaSetDevice(dev));
  }
  ~DeviceGuard() { cudaSetDevice(prev); }
};

static void require_hopper(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    throw Error(std::string("no CUDA device available (") + cudaGetErrorString(e) + "); libb200whisper has no CPU path");
  if (device < 0 || device >= n) throw Error("device index out of range", true);
  cudaDeviceProp prop;
  B2W_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) throw Error(std::string("device ") + prop.name + " is not sm_90 (Hopper); kernels are sm_90a only");
}

template <typename T>
static T* dalloc(size_t n) {
  void* p = nullptr;
  B2W_CUDA(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
  return reinterpret_cast<T*>(p);
}

// device memory allocated once per model: freed by ~Model through `allocs`
template <typename T>
static T* model_alloc(Model* m, size_t n) {
  T* p = dalloc<T>(n);
  m->allocs.push_back(p);
  return p;
}

// Scratch device buffers of one call, freed when the call returns or throws.
struct ScratchBufs {
  std::vector<void*> ptrs;
  ~ScratchBufs() {
    for (void* p : ptrs) cudaFree(p);
  }
  template <typename T>
  T* alloc(size_t n) {
    T* p = dalloc<T>(n);
    ptrs.push_back(p);
    return p;
  }
  // n_dev elements (at least n_host), zeroed, then the first n_host copied from `host` (nothing when it is NULL)
  template <typename T>
  T* put(const void* host, size_t n_host, size_t n_dev = 0) {
    n_dev = std::max(n_dev, n_host);
    T* p = alloc<T>(n_dev);
    B2W_CUDA(cudaMemset(p, 0, std::max<size_t>(n_dev, 1) * sizeof(T)));
    if (host && n_host) B2W_CUDA(cudaMemcpy(p, host, n_host * sizeof(T), cudaMemcpyHostToDevice));
    return p;
  }
};

Model::~Model() {
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);
  for (void* p : allocs) cudaFree(p);
  for (auto& it : pool) cudaFree(it.second);
  // the buffers that are reallocated when a larger shape arrives
  void* ws[] = {e_feats, e_x0, e_x1, e_x, e_xn, e_qkv, e_ao, e_h, e_q, e_qs, e_pcm, e_chunks, e_chunk_max, kcache, vcache, d_xpart,
                sb_blob, d_align_heads};
  for (void* p : ws)
    if (p) cudaFree(p);
  if (h_pinned) cudaFreeHost(h_pinned);
  if (step_graph) cudaGraphExecDestroy(step_graph);
  for (auto& t : timers) {
    cudaEventDestroy(t.start);
    cudaEventDestroy(t.stop);
  }
  if (stream) cudaStreamDestroy(stream);
}

void* Model::pool_get(size_t bytes) {
  for (size_t i = 0; i < pool.size(); ++i)
    if (pool[i].first == bytes) {
      void* p = pool[i].second;
      pool_bytes -= bytes;
      pool.erase(pool.begin() + i);
      return p;
    }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, std::max<size_t>(bytes, 1));
  if (e != cudaSuccess) {  // release the cache and retry once
    cudaGetLastError();
    for (auto& it : pool) cudaFree(it.second);
    pool.clear();
    pool_bytes = 0;
    B2W_CUDA(cudaMalloc(&p, std::max<size_t>(bytes, 1)));
  }
  return p;
}
// At most 24 GiB and kPoolBuffers buffers stay parked; past either, the oldest are freed.  The count covers a continuous-batching
// pipeline at any slot count: two buffers per chunk encoder output, fewer than 3 x kMaxRows chunks alive, plus a batch's two and an
// alignment's scratch.  The byte limit covers it at 16 slots x beam 5 on large-v3 (fewer than 48 chunks, 12 GB), so its steady state
// never reaches cudaFree there; with more slots at that size a drop in live outputs frees the oldest buffers past 24 GiB.
constexpr size_t kPoolBuffers = 2 * 3 * kMaxRows + 16;
void Model::pool_put(void* p, size_t bytes) {
  if (!p) return;
  pool.emplace_back(bytes, p);
  pool_bytes += bytes;
  while (pool_bytes > ((size_t)24 << 30) || pool.size() > kPoolBuffers) {
    cudaFree(pool.front().second);
    pool_bytes -= pool.front().first;
    pool.erase(pool.begin());
  }
}

// An encoder-output buffer from the pool, counted in encoded_bytes until ~Encoded returns it.
static __half* encoded_alloc(Model* m, size_t bytes) {
  __half* p = reinterpret_cast<__half*>(m->pool_get(bytes));
  m->encoded_bytes += bytes;
  return p;
}

Encoded::~Encoded() {
  if (!owner) return;
  cudaSetDevice(owner->device);
  if (enc_out) owner->encoded_bytes -= enc_bytes;
  if (xkv) owner->encoded_bytes -= xkv_bytes;
  owner->pool_put(enc_out, enc_bytes);
  owner->pool_put(xkv, xkv_bytes);
}

// ---- timing -----------------------------------------------------------------------------------------------------
struct ScopedStage {
  Model* m;
  int stage;
  cudaEvent_t a = nullptr, b = nullptr;
  ScopedStage(Model* m_, int st) : m(m_), stage(st) {
    if (!m->timing) return;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    cudaEventRecord(a, m->stream);
  }
  ~ScopedStage() {
    if (!m->timing) return;
    cudaEventRecord(b, m->stream);
    m->timers.push_back({stage, a, b});
  }
};
static void drain_timers(Model* m) {
  if (m->timers.empty()) return;
  cudaStreamSynchronize(m->stream);
  for (auto& t : m->timers) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, t.start, t.stop) == cudaSuccess) {
      m->t_ms[t.stage] += ms;
      m->t_cnt[t.stage] += 1;
    }
    cudaEventDestroy(t.start);
    cudaEventDestroy(t.stop);
  }
  m->timers.clear();
}

// ---- weight upload ------------------------------------------------------------------------------------------------
struct TensorTable {
  const b2w_tensor* t;
  int n;
  const b2w_tensor& get(const std::string& name) const {
    for (int i = 0; i < n; ++i)
      if (name == t[i].name) return t[i];
    throw Error("missing weight tensor: " + name, true);
  }
  const b2w_tensor* find(const std::string& name) const {
    for (int i = 0; i < n; ++i)
      if (name == t[i].name) return &t[i];
    return nullptr;
  }
};
static int64_t numel(const b2w_tensor& t) {
  int64_t n = 1;
  for (int i = 0; i < t.ndim; ++i) n *= t.shape[i];
  return n;
}
static void expect_shape(const b2w_tensor& t, std::initializer_list<int64_t> shape) {
  bool ok = t.ndim == (int)shape.size();
  int i = 0;
  for (int64_t s : shape) ok = ok && t.shape[i++] == s;
  if (!ok) throw Error(std::string("weight ") + t.name + " has an unexpected shape", true);
}

struct Uploader {
  Model* m;
  float* stage_f = nullptr;
  __half* stage_h = nullptr;
  size_t cap = 0;
  explicit Uploader(Model* m_) : m(m_) {}
  ~Uploader() {
    cudaFree(stage_f);
    cudaFree(stage_h);
  }
  void reserve(size_t n) {
    if (n <= cap) return;
    cudaFree(stage_f);
    cudaFree(stage_h);
    cap = n;
    stage_f = dalloc<float>(cap);
    stage_h = dalloc<__half>(cap);
  }
  // host tensor (f32|f16) -> device fp16 at dst
  void to_f16(const b2w_tensor& t, __half* dst) {
    const int64_t n = numel(t);
    if (t.dtype == B2W_F16) {
      B2W_CUDA(cudaMemcpyAsync(dst, t.data, n * 2, cudaMemcpyHostToDevice, m->stream));
    } else {
      reserve(n);
      B2W_CUDA(cudaMemcpyAsync(stage_f, t.data, n * 4, cudaMemcpyHostToDevice, m->stream));
      convert_f32_f16(stage_f, dst, n, m->stream);
    }
    B2W_CUDA(cudaStreamSynchronize(m->stream));
  }
  void to_f32(const b2w_tensor& t, float* dst) {
    const int64_t n = numel(t);
    if (t.dtype == B2W_F32) {
      B2W_CUDA(cudaMemcpyAsync(dst, t.data, n * 4, cudaMemcpyHostToDevice, m->stream));
    } else {
      reserve(n);
      B2W_CUDA(cudaMemcpyAsync(stage_h, t.data, n * 2, cudaMemcpyHostToDevice, m->stream));
      convert_f16_f32(stage_h, dst, n, m->stream);
    }
    B2W_CUDA(cudaStreamSynchronize(m->stream));
  }
  void vec_to_f16(const std::vector<float>& v, __half* dst) {
    b2w_tensor t{};
    t.name = "folded";
    t.data = v.data();
    t.dtype = B2W_F32;
    t.ndim = 1;
    t.shape[0] = (int64_t)v.size();
    to_f16(t, dst);
  }
  void vec_to_f32(const std::vector<float>& v, float* dst) {
    B2W_CUDA(cudaMemcpyAsync(dst, v.data(), v.size() * 4, cudaMemcpyHostToDevice, m->stream));
    B2W_CUDA(cudaStreamSynchronize(m->stream));
  }
  template <typename T>
  T* alloc(size_t n, bool zero = false) {
    T* p = model_alloc<T>(m, n);
    if (zero) B2W_CUDA(cudaMemset(p, 0, n * sizeof(T)));
    return p;
  }
  float* f32(const TensorTable& tt, const std::string& name, std::initializer_list<int64_t> shape) {
    const b2w_tensor& t = tt.get(name);
    expect_shape(t, shape);
    float* p = alloc<float>(numel(t));
    to_f32(t, p);
    return p;
  }
  __half* f16(const TensorTable& tt, const std::string& name, std::initializer_list<int64_t> shape) {
    const b2w_tensor& t = tt.get(name);
    expect_shape(t, shape);
    __half* p = alloc<__half>(numel(t));
    to_f16(t, p);
    return p;
  }
};

static std::vector<float> host_f32(const b2w_tensor& t) {
  const int64_t n = numel(t);
  std::vector<float> v((size_t)n);
  if (t.dtype == B2W_F32) {
    memcpy(v.data(), t.data, (size_t)n * 4);
  } else {
    const __half* h = reinterpret_cast<const __half*>(t.data);
    for (int64_t i = 0; i < n; ++i) v[(size_t)i] = __half2float(h[i]);
  }
  return v;
}

// LayerNorm affine folded into the consuming linear layer (exact algebra):
//   LN(x) W^T + b = ((x - mu) rstd) (W diag(gamma))^T + (W beta + b)
// so the decode kernels only normalise, and no gamma/beta fetch sits on the per-phase critical path.
static void fold_ln(std::vector<float>& W, std::vector<float>& bias, int N, int K, const std::vector<float>& gamma, const std::vector<float>& beta) {
  for (int n = 0; n < N; ++n) {
    float* w = W.data() + (size_t)n * K;
    double acc = 0.0;
    for (int k = 0; k < K; ++k) {
      acc += (double)w[k] * beta[k];
      w[k] *= gamma[k];
    }
    bias[n] += (float)acc;
  }
}

static float host_value(const b2w_tensor& t, int64_t i) {
  if (t.dtype == B2W_F32) return reinterpret_cast<const float*>(t.data)[i];
  return __half2float(reinterpret_cast<const __half*>(t.data)[i]);
}

// conv weight [d][cin][3] -> [d][3][cin_pad] fp16 (k = tap*cin_pad + ci)
static __half* upload_conv(Uploader& up, const TensorTable& tt, const std::string& name, int d, int cin, int cin_pad) {
  const b2w_tensor& t = tt.get(name);
  expect_shape(t, {d, cin, 3});
  std::vector<__half> h((size_t)d * 3 * cin_pad, __float2half(0.f));
  for (int o = 0; o < d; ++o)
    for (int c = 0; c < cin; ++c)
      for (int k = 0; k < 3; ++k) h[((size_t)o * 3 + k) * cin_pad + c] = __float2half_rn(host_value(t, ((int64_t)o * cin + c) * 3 + k));
  __half* p = up.alloc<__half>(h.size());
  B2W_CUDA(cudaMemcpy(p, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
  return p;
}

// every head of the last half of the decoder (OpenAI Whisper's default)
static std::vector<int2> default_alignment_heads(const b2w_config& c) {
  std::vector<int2> v;
  for (int l = c.n_text_layer / 2; l < c.n_text_layer; ++l)
    for (int hd = 0; hd < c.n_text_head; ++hd) v.push_back(make_int2(l, hd));
  return v;
}

static void build_model(Model* m, const b2w_config& cfg, const TensorTable& tt) {
  m->cfg = cfg;
  const int d = cfg.n_audio_state, dt = cfg.n_text_state;
  B2W_CHECK(d % 64 == 0 && dt % 64 == 0, "model width must be a multiple of 64");
  B2W_CHECK(d / cfg.n_audio_head == 64 && dt / cfg.n_text_head == 64, "head_dim must be 64");
  B2W_CHECK(cfg.n_audio_ctx == B2W_N_AUDIO_CTX, "n_audio_ctx must be 1500");
  B2W_CHECK(cfg.n_text_ctx <= B2W_MAX_TEXT_CTX, "n_text_ctx must be <= 448");
  B2W_CHECK(d <= 1280 && dt <= 1280, "model width above 1280 is not supported");
  m->cpad = ceil_div(cfg.n_mels, 64) * 64;
  m->vpad = ceil_div(cfg.n_vocab, 16) * 16;
  Uploader up(m);
  m->conv1_w = upload_conv(up, tt, "encoder.conv1.weight", d, cfg.n_mels, m->cpad);
  m->conv1_b = up.f32(tt, "encoder.conv1.bias", {d});
  m->conv2_w = upload_conv(up, tt, "encoder.conv2.weight", d, d, d);
  m->conv2_b = up.f32(tt, "encoder.conv2.bias", {d});
  m->enc_pos = up.f32(tt, "encoder.positional_embedding", {cfg.n_audio_ctx, d});
  auto fused_qkv = [&](const std::string& p, int n, __half*& w, float*& b) {
    w = up.alloc<__half>((size_t)3 * n * n);
    b = up.alloc<float>((size_t)3 * n, true);
    const char* parts[3] = {".query", ".key", ".value"};
    for (int i = 0; i < 3; ++i) {
      const b2w_tensor& t = tt.get(p + parts[i] + ".weight");
      expect_shape(t, {n, n});
      up.to_f16(t, w + (size_t)i * n * n);
      if (const b2w_tensor* bt = tt.find(p + parts[i] + ".bias")) {
        expect_shape(*bt, {n});
        up.to_f32(*bt, b + (size_t)i * n);
      }
    }
  };
  m->enc.resize(cfg.n_audio_layer);
  for (int i = 0; i < cfg.n_audio_layer; ++i) {
    const std::string p = "encoder.blocks." + std::to_string(i);
    EncLayerW& L = m->enc[i];
    L.ln1_g = up.f32(tt, p + ".attn_ln.weight", {d});
    L.ln1_b = up.f32(tt, p + ".attn_ln.bias", {d});
    fused_qkv(p + ".attn", d, L.wqkv, L.bqkv);
    L.wo = up.f16(tt, p + ".attn.out.weight", {d, d});
    L.bo = up.f32(tt, p + ".attn.out.bias", {d});
    L.ln2_g = up.f32(tt, p + ".mlp_ln.weight", {d});
    L.ln2_b = up.f32(tt, p + ".mlp_ln.bias", {d});
    L.w1 = up.f16(tt, p + ".mlp.0.weight", {4 * d, d});
    L.b1 = up.f32(tt, p + ".mlp.0.bias", {4 * d});
    L.w2 = up.f16(tt, p + ".mlp.2.weight", {d, 4 * d});
    L.b2 = up.f32(tt, p + ".mlp.2.bias", {d});
  }
  if (m->fp8_enc) {
    // e4m3 codes + per-channel scales from the fp16 values the float16 path multiplies with; the fp16 copies are released
    auto to_e4m3 = [&](__half*& w, int N, int K, uint8_t*& q, float*& sc) {
      q = up.alloc<uint8_t>((size_t)N * K);
      sc = up.alloc<float>((size_t)N);
      quantize_rows_e4m3(w, q, sc, N, K, m->stream);
      B2W_CUDA(cudaStreamSynchronize(m->stream));
      m->allocs.erase(std::find(m->allocs.begin(), m->allocs.end(), (void*)w));
      B2W_CUDA(cudaFree(w));
      w = nullptr;
    };
    for (EncLayerW& L : m->enc) {
      to_e4m3(L.wqkv, 3 * d, d, L.q_wqkv, L.s_wqkv);
      to_e4m3(L.wo, d, d, L.q_wo, L.s_wo);
      to_e4m3(L.w1, 4 * d, d, L.q_w1, L.s_w1);
      to_e4m3(L.w2, d, 4 * d, L.q_w2, L.s_w2);
    }
  }
  m->enc_lnp_g = up.f32(tt, "encoder.ln_post.weight", {d});
  m->enc_lnp_b = up.f32(tt, "encoder.ln_post.bias", {d});

  // decoder
  {
    const b2w_tensor& t = tt.get("decoder.token_embedding.weight");
    expect_shape(t, {cfg.n_vocab, dt});
    m->tok_emb = up.alloc<__half>((size_t)m->vpad * dt, true);
    up.to_f16(t, m->tok_emb);
  }
  m->dec_pos = up.f32(tt, "decoder.positional_embedding", {cfg.n_text_ctx, dt});
  const int L = cfg.n_text_layer;
  m->dec.resize(L);
  m->wxkv = up.alloc<__half>((size_t)L * 2 * dt * d);
  m->bxkv = up.alloc<float>((size_t)L * 2 * dt, true);
  double wbytes = (double)cfg.n_vocab * dt * 2;
  for (int i = 0; i < L; ++i) {
    const std::string p = "decoder.blocks." + std::to_string(i);
    DecLayerW& D = m->dec[i];
    // LayerNorm affines are folded into the consuming projections (fold_ln); the kernels normalise only
    {
      const std::vector<float> g1 = host_f32(tt.get(p + ".attn_ln.weight")), b1 = host_f32(tt.get(p + ".attn_ln.bias"));
      expect_shape(tt.get(p + ".attn_ln.weight"), {dt});
      D.wqkv = up.alloc<__half>((size_t)3 * dt * dt);
      D.bqkv = up.alloc<float>((size_t)3 * dt, true);
      const char* parts[3] = {".query", ".key", ".value"};
      for (int j = 0; j < 3; ++j) {
        const b2w_tensor& tw = tt.get(p + ".attn" + parts[j] + ".weight");
        expect_shape(tw, {dt, dt});
        std::vector<float> W = host_f32(tw), bias((size_t)dt, 0.f);
        if (const b2w_tensor* tb = tt.find(p + ".attn" + parts[j] + ".bias")) bias = host_f32(*tb);
        fold_ln(W, bias, dt, dt, g1, b1);
        up.vec_to_f16(W, D.wqkv + (size_t)j * dt * dt);
        up.vec_to_f32(bias, D.bqkv + (size_t)j * dt);
      }
    }
    D.wo = up.f16(tt, p + ".attn.out.weight", {dt, dt});
    D.bo = up.f32(tt, p + ".attn.out.bias", {dt});
    {
      const std::vector<float> g2 = host_f32(tt.get(p + ".cross_attn_ln.weight")), b2 = host_f32(tt.get(p + ".cross_attn_ln.bias"));
      const b2w_tensor& tw = tt.get(p + ".cross_attn.query.weight");
      expect_shape(tw, {dt, dt});
      std::vector<float> W = host_f32(tw), bias = host_f32(tt.get(p + ".cross_attn.query.bias"));
      fold_ln(W, bias, dt, dt, g2, b2);
      D.wq_x = up.alloc<__half>((size_t)dt * dt);
      D.bq_x = up.alloc<float>((size_t)dt);
      up.vec_to_f16(W, D.wq_x);
      up.vec_to_f32(bias, D.bq_x);
    }
    {
      const b2w_tensor& tk = tt.get(p + ".cross_attn.key.weight");
      const b2w_tensor& tv = tt.get(p + ".cross_attn.value.weight");
      expect_shape(tk, {dt, d});
      expect_shape(tv, {dt, d});
      up.to_f16(tk, m->wxkv + ((size_t)i * 2 + 0) * dt * d);
      up.to_f16(tv, m->wxkv + ((size_t)i * 2 + 1) * dt * d);
      up.to_f32(tt.get(p + ".cross_attn.value.bias"), m->bxkv + ((size_t)i * 2 + 1) * dt);
    }
    D.wo_x = up.f16(tt, p + ".cross_attn.out.weight", {dt, dt});
    D.bo_x = up.f32(tt, p + ".cross_attn.out.bias", {dt});
    {
      const std::vector<float> g3 = host_f32(tt.get(p + ".mlp_ln.weight")), b3 = host_f32(tt.get(p + ".mlp_ln.bias"));
      const b2w_tensor& tw = tt.get(p + ".mlp.0.weight");
      expect_shape(tw, {4 * dt, dt});
      std::vector<float> W = host_f32(tw), bias = host_f32(tt.get(p + ".mlp.0.bias"));
      fold_ln(W, bias, 4 * dt, dt, g3, b3);
      D.w1 = up.alloc<__half>((size_t)4 * dt * dt);
      D.b1 = up.alloc<float>((size_t)4 * dt);
      up.vec_to_f16(W, D.w1);
      up.vec_to_f32(bias, D.b1);
    }
    D.w2 = up.f16(tt, p + ".mlp.2.weight", {dt, 4 * dt});
    D.b2 = up.f32(tt, p + ".mlp.2.bias", {dt});
    wbytes += 2.0 * ((double)3 * dt * dt + (double)dt * dt * 3 + 8.0 * dt * dt);
  }
  {
    // logits = LN_f(x) E^T with the final LayerNorm folded: a gamma-scaled copy of the tied embedding + a per-token bias
    const std::vector<float> gf = host_f32(tt.get("decoder.ln.weight")), bf = host_f32(tt.get("decoder.ln.bias"));
    std::vector<float> E = host_f32(tt.get("decoder.token_embedding.weight")), lb((size_t)m->vpad, 0.f);
    E.resize((size_t)m->vpad * dt, 0.f);
    fold_ln(E, lb, m->vpad, dt, gf, bf);
    m->logit_w = up.alloc<__half>((size_t)m->vpad * dt);
    m->logit_b = up.alloc<float>((size_t)m->vpad);
    up.vec_to_f16(E, m->logit_w);
    up.vec_to_f32(lb, m->logit_b);
  }
  m->dec_weight_bytes = wbytes;
  m->mel.reset(new MelPlan(cfg.n_mels));
  m->d_counters = model_alloc<int>(m, 64 + 16 * 20 * 64);
  B2W_CUDA(cudaMemset(m->d_counters, 0, (64 + 16 * 20 * 64) * sizeof(int)));
  B2W_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->h_pinned), 4096));
  m->d_suppress = model_alloc<uint8_t>(m, m->vpad);
  m->d_bind = model_alloc<DecBindings>(m, kMaxRows);
  search_configure();
  gemm_configure();
  dstep_configure();
  bstep_configure();
  {
    // decoder weights re-laid out as the persistent step kernel's tile stream (a second copy: ~1.6 GB for large-v3)
    std::vector<DLayer> hl(L);
    unsigned char* q_scratch = nullptr;
    float* scale_scratch = nullptr;
    if (m->w8) {
      q_scratch = dalloc<unsigned char>((size_t)m->vpad * dt > (size_t)4 * dt * dt ? (size_t)m->vpad * dt : (size_t)4 * dt * dt);
      scale_scratch = dalloc<float>((size_t)std::max(m->vpad, 4 * dt));
    }
    // every decoder matrix is laid out twice: as the <= 8-row kernel's tile stream (dstep.cu) and as the many-row kernel's atom
    // stream (bstep.cu, + row sums for the deferred LayerNorm); with compute_type int8* both streams carry the int8 values
    const bool want_b = dt % 64 == 0 && dt == 64 * cfg.n_text_head;
    struct BPack {
      const void* atoms = nullptr;
      const float* scale = nullptr;
      const float* wsum = nullptr;
    };
    auto pack = [&](const __half* W, const float* bias, int N, int K, int ksplit, BPack* bp, bool want_wsum) -> const __half* {
      const __half* tiles = nullptr;
      if (m->w8) {
        // quantise per output channel; W now holds q * scale (what the prefill / multi-kernel paths multiply with)
        dstep_quantize_rows(const_cast<__half*>(W), N, K, q_scratch, scale_scratch, m->stream);
        unsigned char* out8 = up.alloc<unsigned char>(dstep_packed_bytes_i8(N, K, ksplit));
        dstep_pack_tiles_i8(q_scratch, scale_scratch, bias, N, K, ksplit, out8, m->stream);
        tiles = reinterpret_cast<const __half*>(out8);
        if (want_b && bp) {
          unsigned char* a8 = up.alloc<unsigned char>(bstep_atoms_bytes_i8(N, K));
          bstep_pack_atoms_i8(q_scratch, N, K, a8, m->stream);
          float* sc = up.alloc<float>((size_t)N);
          B2W_CUDA(cudaMemcpyAsync(sc, scale_scratch, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, m->stream));
          bp->atoms = a8;
          bp->scale = sc;
          if (want_wsum) {
            float* wsum = up.alloc<float>((size_t)N);
            bstep_row_sums_i8(q_scratch, scale_scratch, N, K, wsum, m->stream);
            bp->wsum = wsum;
          }
        }
      } else {
        __half* out = up.alloc<__half>(dstep_packed_halves(N, K, ksplit));
        dstep_pack_tiles(W, bias, N, K, ksplit, out, m->stream);
        tiles = out;
        if (want_b && bp) {
          __half* at = reinterpret_cast<__half*>(up.alloc<unsigned char>(bstep_atoms_bytes(N, K)));
          bstep_pack_atoms(W, N, K, at, m->stream);
          bp->atoms = at;
          if (want_wsum) {
            float* wsum = up.alloc<float>((size_t)N);
            bstep_row_sums(W, N, K, wsum, m->stream);
            bp->wsum = wsum;
          }
        }
      }
      B2W_CUDA(cudaStreamSynchronize(m->stream));  // the scratch buffers are reused by the next matrix
      return tiles;
    };
    const bool packable = dt % 64 == 0 && m->vpad % 16 == 0;
    std::vector<BLayer> bl(L);
    for (int i = 0; i < L && packable; ++i) {
      const DecLayerW& D = m->dec[i];
      const __half* Ws[6] = {D.wqkv, D.wo, D.wq_x, D.wo_x, D.w1, D.w2};
      const float* Bs[6] = {D.bqkv, D.bo, D.bq_x, D.bo_x, D.b1, D.b2};
      const int Ns[6] = {3 * dt, dt, dt, dt, 4 * dt, dt}, Ks[6] = {dt, dt, dt, dt, dt, 4 * dt};
      for (int j = 0; j < 6; ++j) {
        BPack bp;
        const bool ln_in = j == 0 || j == 2 || j == 4;
        hl[i].wt[j] = pack(Ws[j], Bs[j], Ns[j], Ks[j], j == 5 ? 4 : 1, &bp, ln_in);
        bl[i].wt[j] = bp.atoms;
        bl[i].bias[j] = Bs[j];
        bl[i].scale[j] = bp.scale;
        if (ln_in) bl[i].wsum[j >> 1] = bp.wsum;
      }
    }
    BPack lp;
    if (packable) m->logit_tiles = pack(m->logit_w, m->logit_b, m->vpad, dt, 1, &lp, false);
    if (q_scratch) {
      B2W_CUDA(cudaStreamSynchronize(m->stream));
      cudaFree(q_scratch);
      cudaFree(scale_scratch);
    }
    m->d_layers = model_alloc<DLayer>(m, L);
    B2W_CUDA(cudaMemcpy(m->d_layers, hl.data(), L * sizeof(DLayer), cudaMemcpyHostToDevice));
    if (packable) {
      DStepArgs ds{};  // the grid depends on the model only: width, depth, weight format
      ds.L = L; ds.d = dt; ds.w8 = m->w8 ? 1 : 0; ds.R = 1; ds.T = 1500;
      m->dstep_grid = dstep_max_grid(m->num_sms, ds);
    }
    if (want_b && packable) {
      m->logit_atoms = lp.atoms;
      m->logit_scale = lp.scale;
      m->d_blayers = model_alloc<BLayer>(m, L);
      B2W_CUDA(cudaMemcpy(m->d_blayers, bl.data(), L * sizeof(BLayer), cudaMemcpyHostToDevice));
      m->bstep_packed = true;
    }
    m->d_bar = model_alloc<unsigned>(m, kBsBarWords);
    B2W_CUDA(cudaMemset(m->d_bar, 0, kBsBarWords * sizeof(unsigned)));
  }
  m->align_heads = default_alignment_heads(cfg);
  B2W_CUDA(cudaStreamSynchronize(m->stream));
}

// ---- encoder ----------------------------------------------------------------------------------------------------------
static void ensure_encoder_ws(Model* m, int b) {
  if (b <= m->enc_max_b) return;
  B2W_CUDA(cudaStreamSynchronize(m->stream));
  void* old[] = {m->e_feats, m->e_x0, m->e_x1, m->e_x, m->e_xn, m->e_qkv, m->e_ao, m->e_h, m->e_q, m->e_qs, m->e_chunks, m->e_chunk_max};
  for (void* p : old)
    if (p) cudaFree(p);
  m->enc_plans.clear();
  const size_t d = m->cfg.n_audio_state, M = (size_t)b * 1500;
  m->e_feats = dalloc<float>((size_t)b * m->cfg.n_mels * 3000);
  m->e_x0 = dalloc<__half>((size_t)b * 3000 * m->cpad);
  m->e_x1 = dalloc<__half>((size_t)b * 3000 * d);
  m->e_x = dalloc<float>(M * d);
  m->e_xn = dalloc<__half>(M * d);
  m->e_qkv = dalloc<__half>(M * 3 * d);
  m->e_ao = dalloc<__half>(M * d);
  m->e_h = dalloc<__half>(M * 4 * d);
  m->e_q = m->fp8_enc ? dalloc<uint8_t>(M * 4 * d) : nullptr;
  m->e_qs = m->fp8_enc ? dalloc<float>(M) : nullptr;
  m->e_chunks = dalloc<MelChunkDesc>(b);
  m->e_chunk_max = dalloc<int>(b);
  m->enc_max_b = b;
}

static const EncPlan& encoder_plan(Model* m, int b) {
  auto it = m->enc_plans.find(b);
  if (it != m->enc_plans.end()) return it->second;
  EncPlan pl;
  pl.b = b;
  const int d = m->cfg.n_audio_state, M = b * 1500, Lc = m->cfg.n_audio_layer;
  {
    GemmArgs a;
    a.A = m->e_x0;
    a.a_batch = b;
    a.a_rows = 3000;
    a.a_cols = m->cpad;
    a.a_row_stride = m->cpad;
    a.a_batch_stride = 3000LL * m->cpad;
    a.taps = 3;
    a.tap_row[0] = -1; a.tap_row[1] = 0; a.tap_row[2] = 1;
    a.k_per_tap = m->cpad;
    a.W = m->conv1_w;
    a.N = d;
    a.rows = 3000;
    a.bias = m->conv1_b;
    a.out = m->e_x1;
    a.out_ld = d;
    a.out_batch_stride = 3000LL * d;
    a.epilogue = EPI_GELU_F16;
    pl.conv1 = gemm_plan(a, m->num_sms);
  }
  {
    GemmArgs a;  // stride-2 conv: view x1 as [b][1500][2d] row pairs
    a.A = m->e_x1;
    a.a_batch = b;
    a.a_rows = 1500;
    a.a_cols = 2 * d;
    a.a_row_stride = 2LL * d;
    a.a_batch_stride = 3000LL * d;
    a.taps = 3;
    a.tap_row[0] = -1; a.tap_col[0] = d;  // x[2t-1]
    a.tap_row[1] = 0;  a.tap_col[1] = 0;  // x[2t]
    a.tap_row[2] = 0;  a.tap_col[2] = d;  // x[2t+1]
    a.k_per_tap = d;
    a.W = m->conv2_w;
    a.N = d;
    a.rows = 1500;
    a.bias = m->conv2_b;
    a.out = m->e_x;
    a.out_ld = d;
    a.out_batch_stride = 1500LL * d;
    a.pos = m->enc_pos;
    a.epilogue = EPI_GELU_POS_F32;
    pl.conv2 = gemm_plan(a, m->num_sms);
  }
  auto flat = [&](const __half* A, int K, const __half* W, int N, const float* bias, void* out, int epi) {
    GemmArgs a;
    a.A = A;
    a.a_batch = 1;
    a.a_rows = M;
    a.a_cols = K;
    a.a_row_stride = K;
    a.k_per_tap = K;
    a.W = W;
    a.N = N;
    a.rows = M;
    a.bias = bias;
    a.out = out;
    a.out_ld = N;
    a.epilogue = epi;
    if (epi == EPI_RESID_F32) a.resid = reinterpret_cast<const float*>(out);
    return gemm_plan(a, m->num_sms);
  };
  // every fp8 GEMM reads its input's codes and row scales from e_q / e_qs, written just before it
  auto flat8 = [&](int K, const uint8_t* W, const float* ws, int N, const float* bias, void* out, int epi) {
    Fp8GemmArgs a;
    a.A = m->e_q;
    a.a_scale = m->e_qs;
    a.W = W;
    a.w_scale = ws;
    a.rows = M;
    a.K = K;
    a.N = N;
    a.bias = bias;
    a.out = out;
    a.epilogue = epi;
    return gemm_fp8_plan(a, m->num_sms);
  };
  for (int l = 0; l < Lc; ++l) {
    const EncLayerW& W = m->enc[l];
    if (m->fp8_enc) {
      pl.qkv8.push_back(flat8(d, W.q_wqkv, W.s_wqkv, 3 * d, W.bqkv, m->e_qkv, EPI_F16));
      pl.proj8.push_back(flat8(d, W.q_wo, W.s_wo, d, W.bo, m->e_x, EPI_RESID_F32));
      pl.ffn1_8.push_back(flat8(d, W.q_w1, W.s_w1, 4 * d, W.b1, m->e_h, EPI_GELU_F16));
      pl.ffn2_8.push_back(flat8(4 * d, W.q_w2, W.s_w2, d, W.b2, m->e_x, EPI_RESID_F32));
      continue;
    }
    pl.qkv.push_back(flat(m->e_xn, d, W.wqkv, 3 * d, W.bqkv, m->e_qkv, EPI_F16));
    pl.proj.push_back(flat(m->e_ao, d, W.wo, d, W.bo, m->e_x, EPI_RESID_F32));
    pl.ffn1.push_back(flat(m->e_xn, d, W.w1, 4 * d, W.b1, m->e_h, EPI_GELU_F16));
    pl.ffn2.push_back(flat(m->e_h, 4 * d, W.w2, d, W.b2, m->e_x, EPI_RESID_F32));
  }
  pl.attn = attn_plan(m->e_qkv, m->e_ao, b, 1500, m->cfg.n_audio_head);
  return m->enc_plans.emplace(b, std::move(pl)).first->second;
}

static void run_gemm(Model* m, const GemmPlan& p) {
  if (m->use_ref_gemm)
    gemm_ref_run(p.a, m->stream);
  else
    gemm_run(p, m->stream);
}

// features for `b` chunks are in m->e_feats; writes fp16 encoder output to `dst` [b][1500][d]
static void encoder_forward(Model* m, int b, __half* dst) {
  const EncPlan& pl = encoder_plan(m, b);
  const int d = m->cfg.n_audio_state, M = b * 1500;
  cudaStream_t s = m->stream;
  pack_features(m->e_feats, m->e_x0, b, m->cfg.n_mels, m->cpad, s);
  run_gemm(m, pl.conv1);
  run_gemm(m, pl.conv2);
  for (int l = 0; l < m->cfg.n_audio_layer; ++l) {
    const EncLayerW& W = m->enc[l];
    if (m->fp8_enc) {
      layernorm_f32_e4m3(m->e_x, W.ln1_g, W.ln1_b, m->e_q, m->e_qs, M, d, s);
      gemm_fp8_run(pl.qkv8[l], s);
      if (m->use_ref_attn)
        attn_ref_run(m->e_qkv, m->e_ao, b, 1500, m->cfg.n_audio_head, s);
      else
        attn_run(pl.attn, s);
      quantize_rows_e4m3(m->e_ao, m->e_q, m->e_qs, M, d, s);
      gemm_fp8_run(pl.proj8[l], s);
      layernorm_f32_e4m3(m->e_x, W.ln2_g, W.ln2_b, m->e_q, m->e_qs, M, d, s);
      gemm_fp8_run(pl.ffn1_8[l], s);
      quantize_rows_e4m3(m->e_h, m->e_q, m->e_qs, M, 4 * d, s);
      gemm_fp8_run(pl.ffn2_8[l], s);
      continue;
    }
    layernorm_f32_f16(m->e_x, W.ln1_g, W.ln1_b, m->e_xn, M, d, s);
    run_gemm(m, pl.qkv[l]);
    if (m->use_ref_attn)
      attn_ref_run(m->e_qkv, m->e_ao, b, 1500, m->cfg.n_audio_head, s);
    else
      attn_run(pl.attn, s);
    run_gemm(m, pl.proj[l]);
    layernorm_f32_f16(m->e_x, W.ln2_g, W.ln2_b, m->e_xn, M, d, s);
    run_gemm(m, pl.ffn1[l]);
    run_gemm(m, pl.ffn2[l]);
  }
  layernorm_f32_f16(m->e_x, m->enc_lnp_g, m->enc_lnp_b, dst, M, d, s);
}

constexpr int kEncSub = 16;  // chunks per encoder pass (workspace ~70 MB per chunk at large-v3)

// Encoder output of B chunks, in sub-batches of kEncSub: fill(b0, b) puts the features of chunks b0 .. b0+b into m->e_feats.
template <typename F>
static std::unique_ptr<Encoded> encode(Model* m, int B, F&& fill) {
  std::unique_ptr<Encoded> e(new Encoded);
  e->owner = m;
  e->B = B;
  const size_t d = m->cfg.n_audio_state;
  e->enc_bytes = (size_t)B * 1500 * d * sizeof(__half);
  e->enc_out = encoded_alloc(m, e->enc_bytes);
  for (int b0 = 0; b0 < B; b0 += kEncSub) {
    const int b = std::min(kEncSub, B - b0);
    ensure_encoder_ws(m, std::min(kEncSub, B));
    fill(b0, b);
    ScopedStage st(m, B2W_T_ENCODER);
    encoder_forward(m, b, e->enc_out + (size_t)b0 * 1500 * d);
  }
  return e;
}

// ---- log-mel --------------------------------------------------------------------------------------------------------------
static int mel_frames(int64_t n_samples) { return (int)(1 + n_samples / 160); }

// ---- decoder ----------------------------------------------------------------------------------------------------------------
constexpr size_t kCrossGroupCounters = 16 * 20 * 64;  // (chunk, head, query group) counters of the layered cross-attention

static void ensure_decoder_ws(Model* m, int chunks, int slots) {
  const int dt = m->cfg.n_text_state, L = m->cfg.n_text_layer, n_ctx = m->cfg.n_text_ctx;
  if (!m->d_x) {
    const size_t dt128 = (size_t)ceil_div(dt, 128) * 128;  // the many-row step kernel keeps its fp32 buffers n-block-major (128-channel blocks)
    m->d_x = model_alloc<float>(m, (size_t)kMaxRows * dt128);
    m->d_xn = model_alloc<__half>(m, (size_t)kMaxRows * dt);
    m->d_q = model_alloc<__half>(m, (size_t)kMaxRows * dt);
    m->d_ao = model_alloc<__half>(m, (size_t)kMaxRows * dt);
    m->d_h = model_alloc<__half>(m, (size_t)kMaxRows * 4 * dt);
    m->d_logits = model_alloc<float>(m, (size_t)kMaxRows * m->vpad);
    m->d_h16 = model_alloc<__half>(m, (size_t)kMaxRows * 4 * dt);
    m->d_xn16 = model_alloc<__half>(m, (size_t)kMaxRows * dt);
    m->d_stats = model_alloc<float>(m, (size_t)3 * L * kMaxRows * 2 + 4);
    m->d_gpart = model_alloc<float>(m, (size_t)m->num_sms * kMaxRows * 128);  // the many-row step kernel's per-CTA split-K partial tiles
    m->d_stpart = model_alloc<float>(m, (size_t)(dt / 64) * kMaxRows * 2);
    B2W_CUDA(cudaMemset(m->d_xn, 0, (size_t)kMaxRows * dt * 2));
    B2W_CUDA(cudaMemset(m->d_ao, 0, (size_t)kMaxRows * dt * 2));
    B2W_CUDA(cudaMemset(m->d_h, 0, (size_t)kMaxRows * 4 * dt * 2));
  }
  const size_t need = (size_t)chunks * n_ctx * slots * dt;
  if (need > m->kv_elems) {
    B2W_CUDA(cudaStreamSynchronize(m->stream));
    if (m->kcache) cudaFree(m->kcache);
    if (m->vcache) cudaFree(m->vcache);
    m->kcache = dalloc<__half>(need * L);
    m->vcache = dalloc<__half>(need * L);
    m->kv_elems = need;
    if (m->step_graph) {
      cudaGraphExecDestroy(m->step_graph);
      m->step_graph = nullptr;
    }
  }
}

static void ensure_search_ws(Model* m, int B, int K) {
  if (B <= m->sb_B && K <= m->sb_K && m->sb_blob) return;
  B2W_CUDA(cudaStreamSynchronize(m->stream));
  if (m->sb_blob) cudaFree(m->sb_blob);
  if (m->step_graph) {
    cudaGraphExecDestroy(m->step_graph);
    m->step_graph = nullptr;
  }
  B = std::max(B, m->sb_B);
  K = std::max(K, m->sb_K);
  const size_t R = (size_t)B * K, n_ctx = m->cfg.n_text_ctx;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~size_t(255);
    return o;
  };
  const size_t Rr = std::max<size_t>(R, kMaxRows);
  const size_t o_params = take(sizeof(SearchParams)), o_chunk = take(B * sizeof(ChunkParams));
  const size_t o_state = take(sizeof(SearchState)), o_rows = take(Rr * sizeof(RowInfo)), o_tok = take(Rr * 4),
               o_cum = take(2 * R * 4), o_hist = take(2 * R * n_ctx * 4), o_anc = take(2 * R * n_ctx),
               o_cs = take(R * kMaxCand * 4), o_ct = take(R * kMaxCand * 4), o_done = take(B * 4), o_fc = take(B * 4),
               o_fs = take((size_t)B * kMaxFinished * 4), o_fl = take((size_t)B * kMaxFinished * 4),
               o_ft = take((size_t)B * kMaxFinished * n_ctx * 4), o_ns = take(B * 4), o_mg = take(R * 4);
  uint8_t* blob = dalloc<uint8_t>(off);
  m->sb_blob = blob;
  SearchBuffers& sb = m->sb;
  sb.state = reinterpret_cast<SearchState*>(blob + o_state);
  sb.params = reinterpret_cast<const SearchParams*>(blob + o_params);
  sb.chunk = reinterpret_cast<ChunkParams*>(blob + o_chunk);
  sb.rows = reinterpret_cast<RowInfo*>(blob + o_rows);
  sb.tokens_in = reinterpret_cast<int*>(blob + o_tok);
  sb.cum = reinterpret_cast<float*>(blob + o_cum);
  sb.hist = reinterpret_cast<int*>(blob + o_hist);
  sb.anc = blob + o_anc;
  sb.cand_score = reinterpret_cast<float*>(blob + o_cs);
  sb.cand_tok = reinterpret_cast<int*>(blob + o_ct);
  sb.done = reinterpret_cast<int*>(blob + o_done);
  sb.fin_count = reinterpret_cast<int*>(blob + o_fc);
  sb.fin_score = reinterpret_cast<float*>(blob + o_fs);
  sb.fin_len = reinterpret_cast<int*>(blob + o_fl);
  sb.fin_tok = reinterpret_cast<int*>(blob + o_ft);
  sb.no_speech = reinterpret_cast<float*>(blob + o_ns);
  sb.row_margin = reinterpret_cast<float*>(blob + o_mg);
  sb.suppress = m->d_suppress;
  sb.n_ctx = (int)n_ctx;
  m->sb_B = B;
  m->sb_K = K;
}

static void ensure_cross_kv(Model* m, Encoded* e) {
  if (e->xkv) return;
  const int d = m->cfg.n_audio_state, dt = m->cfg.n_text_state, L = m->cfg.n_text_layer, H = m->cfg.n_text_head;
  e->xkv_bytes = (size_t)L * 2 * e->B * 1500 * dt * sizeof(__half);
  e->xkv = encoded_alloc(m, e->xkv_bytes);
  ScopedStage st(m, B2W_T_CROSSKV);
  GemmArgs a;
  a.A = e->enc_out;
  a.a_batch = e->B;
  a.a_rows = 1500;
  a.a_cols = d;
  a.a_row_stride = d;
  a.a_batch_stride = 1500LL * d;
  a.k_per_tap = d;
  a.W = m->wxkv;
  a.N = L * 2 * dt;
  a.rows = 1500;
  a.bias = m->bxkv;
  a.out = e->xkv;
  a.epilogue = EPI_F16_XKV;
  a.xkv_d = dt;
  a.xkv_heads = H;
  a.xkv_T = 1500;
  a.xkv_B = e->B;
  if (m->use_ref_gemm) {
    gemm_ref_run(a, m->stream);
  } else {
    GemmPlan p = gemm_plan(a, m->num_sms);
    gemm_run(p, m->stream);
  }
}

// Decoder and search workspaces for groups of `chunks` chunks x K rows, and the cross-attention K/V of `e` (none for fake logits).
static void prepare_decode(Model* m, Encoded* e, int chunks, int K) {
  ensure_decoder_ws(m, chunks, K);
  ensure_search_ws(m, chunks, K);
  if (e) ensure_cross_kv(m, e);
}

constexpr int kTcMinRows = 17;  // rows above which the decode GEMMs go through the wgmma path (activations reused from smem)

// whether a decode GEMM goes through the tensor-core GEMM (else the skinny mma.sync kernel)
static bool gv_uses_wgmma(const GvArgs& a) { return a.R >= kTcMinRows && a.K % 64 == 0 && a.N % 32 == 0; }

// the tensor-core GEMM that computes a decode GEMM: the same outputs, 32-wide tiles where they give more CTAs
static GemmArgs gv_gemm_args(const GvArgs& a) {
  GemmArgs g;
  g.A = a.x;
  g.a_batch = 1;
  g.a_rows = a.R;
  g.a_cols = a.K;
  g.a_row_stride = a.K;
  g.k_per_tap = a.K;
  g.W = a.W;
  g.N = a.N;
  g.rows = a.R;
  g.bias = a.bias;
  g.narrow_tiles = true;
  switch (a.mode) {
    case GV_QKV:
      g.epilogue = EPI_QKV_CACHE;
      g.out = a.out_h;
      g.rowinfo = reinterpret_cast<const int4*>(a.rows);
      g.kcache = a.kcache;
      g.vcache = a.vcache;
      g.qkv_d = a.d;
      g.n_ctx = a.n_ctx;
      g.slots = a.slots;
      break;
    case GV_F16: g.epilogue = EPI_F16; g.out = a.out_h; g.out_ld = a.N; break;
    case GV_GELU_F16: g.epilogue = EPI_GELU_F16; g.out = a.out_h; g.out_ld = a.N; break;
    case GV_RESID_LN: {
      // x += y W^T in place: every element is written by the one tile that holds all of its K (no atomics: the same bits every run)
      g.epilogue = EPI_RESID_F32;
      g.out = a.xres; g.resid = a.xres; g.out_ld = a.N;
      break;
    }
    case GV_F32: g.epilogue = EPI_F32; g.out = a.out_f; g.out_ld = a.ldo; break;
  }
  return g;
}

// decode GEMM through the tensor-core GEMM: the plan (TMA maps and the epilogue's pointers) is cached per Model::dec_plans key
static const GemmPlan& dec_plan(Model* m, const GvArgs& a) {
  const auto key = std::make_tuple((const void*)a.W, (const void*)a.x, a.R, a.mode, (const void*)a.rows, (const void*)a.kcache,
                                   (const void*)a.vcache, a.slots);
  auto it = m->dec_plans.find(key);
  if (it != m->dec_plans.end()) return it->second;
  return m->dec_plans.emplace(key, gemm_plan(gv_gemm_args(a), m->num_sms)).first->second;
}

// the wgmma route of a decode GEMM with plan `p` (gv_gemm_args(a)): the GEMM, then the next LayerNorm of a residual update
static void gv_wgmma(const GemmPlan& p, const GvArgs& a, cudaStream_t s) {
  gemm_run(p, s);
  if (a.mode == GV_RESID_LN) layernorm_f32_f16(a.xres, a.ln_g, a.ln_b, a.xn_out, a.R, a.N, s);
}

static void gv(Model* m, GvArgs a) {
  if (gv_uses_wgmma(a))
    gv_wgmma(dec_plan(m, a), a, m->stream);
  else
    skinny_gemm(a, m->stream);
}

// Uploads the encoder binding of every chunk of the next pass or step (entry b for chunk b).
static void bind_chunks(Model* m, const std::vector<DecBindings>& bind) {
  B2W_CHECK(!bind.empty() && bind.size() <= (size_t)kMaxRows, "decode chunks");
  m->h_binds = bind;
  m->h_bind = bind[0];
  B2W_CUDA(cudaMemcpyAsync(m->d_bind, m->h_binds.data(), bind.size() * sizeof(DecBindings), cudaMemcpyHostToDevice, m->stream));
}

// Bindings of items chunk0 .. chunk0 + n - 1 of `e` (null for fake logits) to chunks 0 .. n - 1.
static std::vector<DecBindings> item_range(const Encoded* e, int chunk0, int n) {
  std::vector<DecBindings> bind(n);
  for (int b = 0; b < n; ++b) bind[b] = DecBindings{e ? e->xkv : nullptr, e ? e->B : 0, chunk0 + b};
  return bind;
}

// Floats of the cross-attention partial buffer for n_chunks x rows_per_chunk rows: 64 outputs + max + sum per (chunk, head,
// query group, key split) and query row.
static size_t xpart_floats(const Model* m, int n_chunks, int rows_per_chunk) {
  return (size_t)n_chunks * m->cfg.n_text_head * ds_xqgroups(rows_per_chunk) * kDsXSplits * kDsXQ * 66;
}

// The partial buffer is grown outside graph capture (which forbids cudaMalloc and synchronisation), before any argument block
// or graph takes its pointer.
static void ensure_xpart(Model* m, size_t floats) {
  if (floats <= m->d_xpart_floats) return;
  B2W_CUDA(cudaStreamSynchronize(m->stream));
  if (m->d_xpart) cudaFree(m->d_xpart);
  m->d_xpart = dalloc<float>(floats);
  m->d_xpart_floats = floats;
}

// Whisper.align: the cross-attention probabilities of the alignment heads for the rows of forced-decoding passes, the row at
// position p of chunk b (relative to the pass's first chunk) written to out[b][head][p][0..nf) of an [n][n_heads][n_tok][nf] buffer.
struct AlignCapture {
  const int2* heads;
  int n_heads;
  float* out;
  int n_tok, nf;
};

// The layered decoder step: one launch per GEMM / attention.  Needs ensure_xpart(m, xpart_floats(m, n_chunks, rows_per_chunk)).
// Every LayerNorm normalises only: the affines are folded into the projections that consume them (fold_ln).  The slot ancestry
// buffers hold anc_chunks chunks.
static void decoder_layers(Model* m, int n_chunks, int rows_per_chunk, int slots, int anc_chunks, const AlignCapture* cap) {
  const b2w_config& c = m->cfg;
  const int dt = c.n_text_state, L = c.n_text_layer, H = c.n_text_head, R = n_chunks * rows_per_chunk;
  cudaStream_t s = m->stream;
  const SearchBuffers& sb = m->sb;
  embed_ln(sb.tokens_in, sb.rows, m->tok_emb, m->dec_pos, nullptr, nullptr, m->d_x, m->d_xn, R, dt, c.n_vocab, s);
  B2W_CHECK(m->d_xpart_floats >= xpart_floats(m, n_chunks, rows_per_chunk), "cross-attention partial buffer");
  B2W_CHECK((size_t)n_chunks * H * ds_xqgroups(rows_per_chunk) <= kCrossGroupCounters, "cross-attention group counters");
  for (int l = 0; l < L; ++l) {
    const DecLayerW& W = m->dec[l];
    __half* kc = m->kcache + (size_t)l * m->kv_elems;
    __half* vc = m->vcache + (size_t)l * m->kv_elems;
    GvArgs a;
    a.x = m->d_xn; a.W = W.wqkv; a.bias = W.bqkv; a.R = R; a.N = 3 * dt; a.K = dt; a.mode = GV_QKV;
    a.rows = sb.rows; a.kcache = kc; a.vcache = vc; a.d = dt; a.n_ctx = c.n_text_ctx; a.slots = slots; a.out_h = m->d_q;
    gv(m, a);
    SelfAttnArgs sa{sb.rows, m->d_q, kc, vc, sb.anc, m->d_ao, dt, c.n_text_ctx, slots, (long long)anc_chunks * slots * c.n_text_ctx};
    dec_self_attn(sa, R, H, s);
    GvArgs o;
    o.x = m->d_ao; o.W = W.wo; o.bias = W.bo; o.R = R; o.N = dt; o.K = dt; o.mode = GV_RESID_LN;
    o.xres = m->d_x; o.xn_out = m->d_xn; o.counter = m->d_counters;
    gv(m, o);
    GvArgs q;
    q.x = m->d_xn; q.W = W.wq_x; q.bias = W.bq_x; q.R = R; q.N = dt; q.K = dt; q.mode = GV_F16; q.out_h = m->d_q;
    gv(m, q);
    if (cap) align_probs(m->d_q, m->d_bind, sb.rows, l, cap->heads, cap->n_heads, cap->out, cap->n_tok, cap->nf, R, rows_per_chunk, H, 1500, dt, s);
    DStepArgs xa{};
    xa.q = m->d_q; xa.ao = m->d_ao; xa.bind = m->d_bind; xa.xpart = m->d_xpart; xa.xcounters = m->d_counters + 64;
    xa.H = H; xa.T = 1500; xa.d = dt; xa.rows_per_chunk = rows_per_chunk; xa.n_chunks = n_chunks;
    dstep_cross_attn_launch(xa, l, s);
    GvArgs ox;
    ox.x = m->d_ao; ox.W = W.wo_x; ox.bias = W.bo_x; ox.R = R; ox.N = dt; ox.K = dt; ox.mode = GV_RESID_LN;
    ox.xres = m->d_x; ox.xn_out = m->d_xn; ox.counter = m->d_counters;
    gv(m, ox);
    GvArgs f1;
    f1.x = m->d_xn; f1.W = W.w1; f1.bias = W.b1; f1.R = R; f1.N = 4 * dt; f1.K = dt; f1.mode = GV_GELU_F16; f1.out_h = m->d_h;
    gv(m, f1);
    GvArgs f2;
    f2.x = m->d_h; f2.W = W.w2; f2.bias = W.b2; f2.R = R; f2.N = dt; f2.K = 4 * dt; f2.mode = GV_RESID_LN;
    f2.xres = m->d_x; f2.xn_out = m->d_xn; f2.counter = m->d_counters;
    gv(m, f2);
  }
}

static void logits_gemm(Model* m, int R) {
  GvArgs a;
  a.x = m->d_xn; a.W = m->logit_w; a.bias = m->logit_b; a.R = R; a.N = m->vpad; a.K = m->cfg.n_text_state; a.mode = GV_F32;
  a.out_f = m->d_logits; a.ldo = m->vpad;
  gv(m, a);
}

static int forced_positions_per_pass(int n_chunks) { return std::max(1, kMaxRows / n_chunks); }

// The chunks of a forced decoding: chunk b attends to the encoder item bind[b] and writes its keys as chunk kv_chunk[b] of a
// self-KV cache (and slot ancestry) of anc_chunks chunks.
struct ForcedChunks {
  std::vector<DecBindings> bind;
  std::vector<int> kv_chunk;
  int anc_chunks;
};

// Items chunk0 .. chunk0 + n - 1 of `e` as chunks 0 .. n - 1 of their own cache.
static ForcedChunks forced_range(const Encoded* e, int chunk0, int n) {
  ForcedChunks fc{item_range(e, chunk0, n), std::vector<int>(n), n};
  for (int b = 0; b < n; ++b) fc.kv_chunk[b] = b;
  return fc;
}

// Forced decoding of tokens[b * stride + i], i < n_tok, for the chunks of fc, in passes of forced_positions_per_pass(n)
// positions; every row writes self-KV slot 0 of `slots`.  The slot ancestry must be zero: clear_anc zeroes it, unless the caller
// already has.  When `cap` is set, every pass captures the alignment heads' cross-attention.  After each pass's decoder layers,
// on_pass(i0, i1) may run logits_gemm: row b * (i1 - i0) + (i - i0) holds position i of chunk b.
template <typename F>
static void forced_decode(Model* m, const ForcedChunks& fc, const int32_t* tokens, int stride, int n_tok, int slots, bool clear_anc,
                          const AlignCapture* cap, F&& on_pass) {
  const int n = (int)fc.bind.size();
  if (clear_anc) B2W_CUDA(cudaMemsetAsync(m->sb.anc, 0, (size_t)2 * fc.anc_chunks * slots * m->cfg.n_text_ctx, m->stream));
  const int per_pass = forced_positions_per_pass(n);
  for (int i0 = 0; i0 < n_tok; i0 += per_pass) {
    const int i1 = std::min(n_tok, i0 + per_pass), rpc = i1 - i0, R = n * rpc;
    std::vector<RowInfo> rows(R);
    std::vector<int> toks(R);
    for (int b = 0; b < n; ++b)
      for (int i = i0; i < i1; ++i) {
        rows[b * rpc + (i - i0)] = RowInfo{fc.kv_chunk[b], 0, i, 0};
        toks[b * rpc + (i - i0)] = tokens[(size_t)b * stride + i];
      }
    B2W_CUDA(cudaMemcpyAsync(m->sb.rows, rows.data(), R * sizeof(RowInfo), cudaMemcpyHostToDevice, m->stream));
    B2W_CUDA(cudaMemcpyAsync(m->sb.tokens_in, toks.data(), R * sizeof(int), cudaMemcpyHostToDevice, m->stream));
    B2W_CUDA(cudaStreamSynchronize(m->stream));  // host vectors go out of scope
    bind_chunks(m, fc.bind);
    ensure_xpart(m, xpart_floats(m, n, rpc));
    decoder_layers(m, n, rpc, slots, fc.anc_chunks, cap);
    on_pass(i0, i1);
  }
}

// ---- generate: one group of n chunks x K rows --------------------------------------------------------------------------------
// Position of <|startoftranscript|>, which must be the same in every prompt of the group.
static int validate_prompts(const b2w_config& c, const int32_t* prompts, int n, int P) {
  int sot_index = -1;
  for (int b = 0; b < n; ++b) {
    const int32_t* p = prompts + (size_t)b * P;
    int si = -1;
    for (int i = 0; i < P; ++i) {
      B2W_CHECK(p[i] >= 0 && p[i] < c.n_vocab, "prompt token id out of range");
      if (p[i] == c.sot && si < 0) si = i;
    }
    if (si < 0) throw Error("<|startoftranscript|> token was not found in the prompt", true);
    if (sot_index < 0) sot_index = si;
    else if (si != sot_index) throw Error("<|startoftranscript|> must be at the same position in all prompts", true);
  }
  return sot_index;
}

// Checks the options of a generate call against the model; returns K, the rows per chunk (beams, or independent hypotheses).
static int check_gen_opts(const b2w_config& c, const b2w_gen_opts& o) {
  B2W_CHECK(o.beam_size >= 1 && o.beam_size <= kMaxBeam, "beam_size must be in 1..16");
  B2W_CHECK(o.num_hypotheses >= 1 && o.num_hypotheses <= kMaxBeam, "num_hypotheses must be in 1..16");
  B2W_CHECK(o.beam_size == 1 || o.num_hypotheses <= o.beam_size, "num_hypotheses must be <= beam_size");
  B2W_CHECK(o.max_length >= 1 && o.max_length <= c.n_text_ctx, "max_length must be in 1..n_text_ctx");
  B2W_CHECK(o.sampling_topk == 0 || o.sampling_topk == 1, "sampling_topk must be 0 (full vocabulary) or 1 (argmax)");
  B2W_CHECK(o.patience > 0 && o.repetition_penalty > 0, "patience and repetition_penalty must be positive");
  return o.beam_size > 1 ? o.beam_size : std::max(1, o.num_hypotheses);
}

// The always-suppressed tokens of a generate call, over the padded vocabulary (the padding columns are suppressed too).
static std::vector<uint8_t> suppress_mask(const b2w_config& c, int vpad, const b2w_gen_opts& o) {
  std::vector<uint8_t> mask(vpad, 0);
  for (int i = c.n_vocab; i < vpad; ++i) mask[i] = 1;
  for (int i = 0; i < o.n_suppress_tokens; ++i) {
    const int t = o.suppress_tokens[i];
    if (t >= 0 && t < c.n_vocab) mask[t] = 1;
  }
  return mask;
}

static SearchParams search_params(const b2w_config& c, int vpad, int n, int K, const b2w_gen_opts& o) {
  const bool beam = o.beam_size > 1;
  SearchParams sp{};
  sp.n_vocab = c.n_vocab; sp.vpad = vpad; sp.B = n; sp.K = K;
  sp.mode = beam ? 0 : 1;
  sp.ncand = beam ? 2 * K : 1;
  sp.max_finished = std::max(1, (int)lroundf(K * o.patience));
  sp.allow_early_exit = (o.patience == 1.0f && o.length_penalty == 0.0f) ? 1 : 0;
  sp.num_hyp = std::max(1, o.num_hypotheses);
  sp.length_penalty = o.length_penalty; sp.repetition_penalty = o.repetition_penalty;
  sp.no_repeat_ngram = o.no_repeat_ngram_size;
  sp.suppress_blank = o.suppress_blank;
  sp.n_suppress_begin = c.n_suppress_begin;
  for (int i = 0; i < 8; ++i) sp.suppress_begin[i] = c.suppress_begin[i];
  sp.max_initial_ts = o.max_initial_timestamp_index;
  sp.eot = c.eot; sp.no_timestamps = c.no_timestamps; sp.timestamp_begin = c.timestamp_begin; sp.no_speech = c.no_speech;
  sp.sampling_topk = o.sampling_topk; sp.temperature = o.sampling_temperature > 0 ? o.sampling_temperature : 1.0f;
  sp.seed = o.seed;
  sp.fake_logits = o.debug_fake_logits;
  B2W_CHECK(sp.max_finished <= kMaxFinishTarget, "beam_size * patience is too large");
  // a chunk stops at max_finished, but the step that reaches it can finish up to K hypotheses: all must have a slot
  B2W_CHECK(!beam || sp.max_finished + K - 1 <= kMaxFinished, "beam_size * patience is too large");
  return sp;
}

// The search state of a chunk decoding `prompt` (P tokens, <|startoftranscript|> at sot_index) up to max_length tokens.
static ChunkParams chunk_params(const b2w_config& c, const int32_t* prompt, int P, int sot_index, int max_length, int item,
                                bool no_speech) {
  ChunkParams cp{};
  cp.prompt_len = P;
  cp.max_steps = max_length - P;
  cp.item = item;
  cp.timestamp_rules = std::find(prompt, prompt + P, c.no_timestamps) == prompt + P ? 1 : 0;
  cp.ns_first = (no_speech && sot_index == P - 1) ? 1 : 0;
  return cp;
}

// Prompt[:-1] of every chunk of the group; the no-speech probability comes from the pass that holds the SOT row.  The search
// reset has cleared the slot ancestry.
static void prefill(Model* m, const Encoded* e, int chunk0, int n, const int32_t* prompts, int P, int K, int sot_index, bool no_speech) {
  ScopedStage st(m, B2W_T_PREFILL);
  const b2w_config& c = m->cfg;
  forced_decode(m, forced_range(e, chunk0, n), prompts + (size_t)chunk0 * P, P, P - 1, K, false, nullptr, [&](int i0, int i1) {
    if (!no_speech || sot_index < i0 || sot_index >= i1) return;
    logits_gemm(m, n * (i1 - i0));
    no_speech_from_logits(m->d_logits, m->vpad, n * (i1 - i0), i1 - i0, sot_index - i0, c.n_vocab, c.no_speech, m->sb.no_speech, m->stream);
  });
}

struct Step {  // one decode step of a chunk group: its path and the argument block of a persistent kernel
  StepPath path;
  int n, K;
  DStepArgs ds{};
  BStepArgs bs{};
};

// The one step-path decision: fake logits when asked for, else the <= 8-row kernel, else the many-row kernel, else the layered
// step.  B2W_STEP forces a path; a shape the forced kernel cannot take is an invalid argument.  Fills the shape of bs.
static Step choose_step(const Model* m, int n, int K, bool fake_logits) {
  const b2w_config& c = m->cfg;
  Step st{StepPath::FakeLogits, n, K};
  if (fake_logits) return st;
  BStepArgs& bs = st.bs;
  bs.L = c.n_text_layer; bs.w8 = m->w8 ? 1 : 0;
  bs.R = n * K; bs.d = c.n_text_state; bs.H = c.n_text_head; bs.n_ctx = c.n_text_ctx; bs.slots = K; bs.T = 1500;
  bs.vpad = m->vpad; bs.n_vocab = c.n_vocab; bs.n_chunks = n; bs.rows_per_chunk = K;
  const bool dstep_ok = m->dstep_grid > 0 && n * K <= 8;
  const bool bstep_ok = m->bstep_packed && bstep_supported(m->num_sms, bs);
  st.path = m->forced_step.value_or(dstep_ok ? StepPath::Dstep : bstep_ok ? StepPath::Bstep : StepPath::Layers);
  if ((st.path == StepPath::Dstep && !dstep_ok) || (st.path == StepPath::Bstep && !bstep_ok))
    throw Error("B2W_STEP forces a step kernel that cannot run " + std::to_string(n) + " chunks x " + std::to_string(K) + " rows of this model",
                true);
  return st;
}

// Sizes the partial buffer and binds the workspace into the persistent kernel's argument block.
static void step_args(Model* m, Step& st) {
  const b2w_config& c = m->cfg;
  const int n = st.n, K = st.K, R = n * K;
  const SearchBuffers& sb = m->sb;
  if (st.path != StepPath::FakeLogits) ensure_xpart(m, xpart_floats(m, n, K));
  if (st.path == StepPath::Dstep) {
    DStepArgs& ds = st.ds;
    ds.layers = m->d_layers; ds.L = c.n_text_layer; ds.tok_emb = m->tok_emb; ds.pos_emb = m->dec_pos;
    ds.logit_tiles = m->logit_tiles;
    ds.w8 = m->w8 ? 1 : 0;
    ds.R = R; ds.d = c.n_text_state; ds.H = c.n_text_head; ds.n_ctx = c.n_text_ctx; ds.slots = K; ds.T = 1500;
    ds.vpad = m->vpad; ds.n_vocab = c.n_vocab; ds.n_chunks = n; ds.rows_per_chunk = K;
    ds.rows = sb.rows; ds.tokens_in = sb.tokens_in;
    ds.x = m->d_x; ds.q = m->d_q; ds.ao = m->d_ao; ds.h = m->d_h; ds.logits = m->d_logits;
    ds.kcache = m->kcache; ds.vcache = m->vcache; ds.kv_layer_stride = (long long)m->kv_elems;
    ds.anc = sb.anc; ds.anc_buf_stride = (long long)n * K * c.n_text_ctx;
    ds.bind = m->d_bind; ds.xpart = m->d_xpart; ds.xcounters = m->d_counters + 64; ds.bar = m->d_bar;
    ds.prof = m->d_prof;
  } else if (st.path == StepPath::Bstep) {
    BStepArgs& bs = st.bs;
    B2W_CHECK(bstep_xpart_floats(bs) <= m->d_xpart_floats, "cross-attention partial buffer");
    bs.layers = m->d_blayers; bs.tok_emb = m->tok_emb; bs.pos_emb = m->dec_pos;
    bs.logit_atoms = m->logit_atoms; bs.logit_bias = m->logit_b; bs.logit_scale = m->logit_scale;
    if (const char* v = getenv("B2W_BSTEP_STOP")) bs.stop_phase = atoi(v);  // read per call: tests/test_gpu_decode_phases.py steps it
    bs.rows = sb.rows; bs.tokens_in = sb.tokens_in;
    bs.x = m->d_x; bs.ao = m->d_ao; bs.h16 = m->d_h16; bs.xn16 = m->d_xn16;
    bs.stats = m->d_stats; bs.stpart = m->d_stpart; bs.gpart = m->d_gpart; bs.logits = m->d_logits;
    bs.kcache = m->kcache; bs.vcache = m->vcache; bs.kv_layer_stride = (long long)m->kv_elems;
    bs.anc = sb.anc; bs.anc_buf_stride = (long long)n * K * c.n_text_ctx;
    bs.bind = m->d_bind; bs.xpart = m->d_xpart; bs.xcounters = m->d_counters + 64; bs.bar = m->d_bar; bs.prof = m->d_prof;
  }
}

// Uploads the first decode rows, the search parameters and the encoder binding, and fills the step's argument block.
static void bind_step(Model* m, Step& st, const Encoded* e, int chunk0, const int32_t* prompts, int P, const SearchParams& sp) {
  const int n = st.n, K = st.K, R = n * K;
  cudaStream_t s = m->stream;
  const SearchBuffers& sb = m->sb;
  {
    std::vector<RowInfo> rows(R);
    std::vector<int> toks(R);
    for (int b = 0; b < n; ++b)
      for (int k = 0; k < K; ++k) {
        rows[b * K + k] = RowInfo{b, k, P - 1, 0};
        toks[b * K + k] = prompts[(size_t)(chunk0 + b) * P + P - 1];
      }
    B2W_CUDA(cudaMemcpyAsync(sb.rows, rows.data(), R * sizeof(RowInfo), cudaMemcpyHostToDevice, s));
    B2W_CUDA(cudaMemcpyAsync(sb.tokens_in, toks.data(), R * sizeof(int), cudaMemcpyHostToDevice, s));
    B2W_CUDA(cudaStreamSynchronize(s));
  }
  step_args(m, st);
  m->h_params = sp;
  B2W_CUDA(cudaMemcpyAsync(const_cast<SearchParams*>(sb.params), &m->h_params, sizeof(SearchParams), cudaMemcpyHostToDevice, s));
  bind_chunks(m, item_range(e, chunk0, n));
}

// The decoder half of a step: the logits of every row into d_logits, from sb.rows, sb.tokens_in and sb.anc.
static void launch_decoder(Model* m, const Step& st) {
  const int R = st.n * st.K;
  switch (st.path) {
    case StepPath::FakeLogits: fake_logits(m->d_logits, R, m->sb, m->stream); break;
    case StepPath::Dstep: dstep_launch(st.ds, m->dstep_grid, m->stream); break;
    case StepPath::Bstep: bstep_launch(st.bs, m->num_sms, m->stream); break;
    case StepPath::Layers:
      decoder_layers(m, st.n, st.K, st.K, st.n, nullptr);
      logits_gemm(m, R);
      break;
  }
}

static void record_step(Model* m, const Step& st) {
  const int R = st.n * st.K;
  launch_decoder(m, st);
  search_rows(m->d_logits, R, m->vpad, m->sb, m->stream);
  search_update(st.n, m->sb, m->stream);
}

// One CUDA graph per (shape, path, buffers), replayed every step with no per-step host parameters.  The graph depends only on
// shapes and workspace pointers: options and encoder-output bindings are read from device memory by the kernels, so one
// instantiated graph serves every window / chunk group of the same shape.  Returns the kernels one replay launches.
static int64_t step_graph(Model* m, const Step& st) {
  const StepGraphKey key{m->kcache, m->sb_blob, m->d_xpart, m->d_logits, st.n, st.K, (int)st.path, st.bs.stop_phase};
  if (m->step_graph && m->step_graph_key == key) return m->step_graph_kernels;
  if (m->step_graph) {
    cudaGraphExecDestroy(m->step_graph);
    m->step_graph = nullptr;
  }
  const int64_t launches_before = g_launches;
  cudaGraph_t graph = nullptr;
  B2W_CUDA(cudaStreamBeginCapture(m->stream, cudaStreamCaptureModeThreadLocal));
  try {
    record_step(m, st);
  } catch (...) {
    cudaStreamEndCapture(m->stream, &graph);
    if (graph) cudaGraphDestroy(graph);
    throw;
  }
  B2W_CUDA(cudaStreamEndCapture(m->stream, &graph));
  B2W_CUDA(cudaGraphInstantiate(&m->step_graph, graph, 0));
  cudaGraphDestroy(graph);
  m->step_graph_key = key;
  m->step_graph_kernels = g_launches - launches_before;  // recorded, not launched
  g_launches = launches_before;
  return m->step_graph_kernels;
}

// Replays the step graph until every chunk is done or max_steps is reached; the host only polls the done counter.
static void decode_loop(Model* m, const Step& st, int P, int max_steps) {
  const int64_t per_step_kernels = step_graph(m, st);
  ScopedStage stage(m, B2W_T_DECODE);
  const b2w_config& c = m->cfg;
  const int n = st.n, R = st.n * st.K;
  // the persistent kernels stream int8 weights with compute_type int8*: half the fp16 bytes; per-channel scales are negligible
  const bool w8_stream = m->w8 && (st.path == StepPath::Dstep || st.path == StepPath::Bstep);
  const int poll = 4;
  int steps_run = 0;
  for (int step = 0; step < max_steps; ++step) {
    B2W_CUDA(cudaGraphLaunch(m->step_graph, m->stream));
    g_launches += per_step_kernels;
    ++steps_run;
    // algorithmic bytes of this step: weights + beam-shared cross-KV + self-KV read so far
    m->decode_alg_bytes += (w8_stream ? 0.5 * m->dec_weight_bytes : m->dec_weight_bytes) +
                           (double)n * c.n_text_layer * 2.0 * 1500 * c.n_text_state * 2.0 +
                           (double)R * (P + step) * c.n_text_layer * 2.0 * c.n_text_state * 2.0;
    if ((step % poll) == poll - 1 && step + 1 < max_steps) {
      B2W_CUDA(cudaMemcpyAsync(m->h_pinned, &m->sb.state->n_done, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
      B2W_CUDA(cudaStreamSynchronize(m->stream));
      if (m->h_pinned[0] >= n) break;
    }
  }
  m->decode_steps += steps_run;
  if (m->d_prof && st.path == StepPath::Bstep) bstep_print_profile(st.bs, m->stream);
  if (m->d_prof && st.path == StepPath::Dstep) dstep_print_profile(st.ds, m->stream);
}

// Finished hypotheses of chunks slot0 .. slot0 + n - 1, best first by (length-penalised) score, into outputs chunk0 .. chunk0 + n - 1.
static void collect_hypotheses(Model* m, int slot0, int chunk0, int n, int K, const b2w_gen_opts& o, int32_t* out_ids, int32_t* out_lens,
                               float* out_scores, float* out_ns) {
  ScopedStage st(m, B2W_T_D2H);
  cudaStream_t s = m->stream;
  const SearchBuffers& sb = m->sb;
  const int n_ctx = m->cfg.n_text_ctx, num_hyp = std::max(1, o.num_hypotheses);
  const bool beam = o.beam_size > 1;
  std::vector<int> fin_count(n), fin_len((size_t)n * kMaxFinished);
  std::vector<float> fin_score((size_t)n * kMaxFinished), ns(n);
  std::vector<int> fin_tok((size_t)n * kMaxFinished * n_ctx);
  B2W_CUDA(cudaMemcpyAsync(fin_count.data(), sb.fin_count + slot0, n * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(fin_len.data(), sb.fin_len + (size_t)slot0 * kMaxFinished, fin_len.size() * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(fin_score.data(), sb.fin_score + (size_t)slot0 * kMaxFinished, fin_score.size() * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(fin_tok.data(), sb.fin_tok + (size_t)slot0 * kMaxFinished * n_ctx, fin_tok.size() * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(ns.data(), sb.no_speech + slot0, n * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaStreamSynchronize(s));
  for (int b = 0; b < n; ++b) {
    out_ns[chunk0 + b] = o.return_no_speech_prob ? ns[b] : 0.f;
    std::vector<int> order;
    const int cnt = beam ? std::min(fin_count[b], kMaxFinished) : K;
    std::vector<float> norm(cnt);
    for (int i = 0; i < cnt; ++i) {
      const int len = fin_len[(size_t)b * kMaxFinished + i];
      if (len < 0) continue;  // greedy row that never finished (cannot happen: the last step always finishes)
      const float cum = fin_score[(size_t)b * kMaxFinished + i];
      norm[i] = (o.length_penalty != 0.0f) ? cum / powf((float)len, o.length_penalty) : cum;
      order.push_back(i);
    }
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
      const float a = norm[x], bb = norm[y];
      if (std::isnan(a) || std::isnan(bb)) return !std::isnan(a) && std::isnan(bb);
      return a > bb;
    });
    for (int h = 0; h < num_hyp; ++h) {
      const size_t oi = (size_t)(chunk0 + b) * num_hyp + h;
      if (h < (int)order.size()) {
        const int i = order[h];
        const int len = fin_len[(size_t)b * kMaxFinished + i];
        out_lens[oi] = len;
        out_scores[oi] = norm[i];
        memcpy(out_ids + oi * o.max_length, &fin_tok[((size_t)b * kMaxFinished + i) * n_ctx], (size_t)len * 4);
      } else {
        out_lens[oi] = 0;
        out_scores[oi] = 0.f;
      }
    }
  }
}

static void generate_group(Model* m, Encoded* e, int chunk0, int n, const int32_t* prompts, int P, const b2w_gen_opts& o,
                           int32_t* out_ids, int32_t* out_lens, float* out_scores, float* out_ns) {
  const int K = o.beam_size > 1 ? o.beam_size : std::max(1, o.num_hypotheses);
  const int sot_index = validate_prompts(m->cfg, prompts + (size_t)chunk0 * P, n, P);
  for (int b = 0; b < n; ++b) out_ns[chunk0 + b] = 0.f;
  const SearchParams sp = search_params(m->cfg, m->vpad, n, K, o);
  Step st = choose_step(m, n, K, sp.fake_logits);
  const int max_steps = o.max_length - P;
  if (max_steps <= 0) {
    const int num_hyp = std::max(1, o.num_hypotheses);
    for (int b = 0; b < n; ++b)
      for (int h = 0; h < num_hyp; ++h) {
        out_lens[(size_t)(chunk0 + b) * num_hyp + h] = 0;
        out_scores[(size_t)(chunk0 + b) * num_hyp + h] = 0.f;
      }
    return;
  }

  // reset the search state
  const SearchBuffers& sb = m->sb;
  cudaStream_t s = m->stream;
  const size_t RB = (size_t)n * K;
  B2W_CUDA(cudaMemsetAsync(sb.state, 0, sizeof(SearchState), s));
  B2W_CUDA(cudaMemsetAsync(sb.cum, 0, 2 * RB * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.anc, 0, 2 * RB * m->cfg.n_text_ctx, s));
  B2W_CUDA(cudaMemsetAsync(sb.done, 0, n * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.fin_count, 0, n * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.fin_len, 0xFF, (size_t)n * kMaxFinished * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.no_speech, 0, n * 4, s));
  {
    // the group's first prompt decides the timestamp rules of all of its chunks; item ids are the chunks' indices in the group
    std::vector<ChunkParams> cps(n);
    for (int b = 0; b < n; ++b)
      cps[b] = chunk_params(m->cfg, prompts + (size_t)chunk0 * P, P, sot_index, o.max_length, b, o.return_no_speech_prob);
    B2W_CUDA(cudaMemcpyAsync(sb.chunk, cps.data(), n * sizeof(ChunkParams), cudaMemcpyHostToDevice, s));
    B2W_CUDA(cudaStreamSynchronize(s));
  }

  if (!sp.fake_logits && P > 1) prefill(m, e, chunk0, n, prompts, P, K, sot_index, o.return_no_speech_prob);
  bind_step(m, st, e, chunk0, prompts, P, sp);
  decode_loop(m, st, P, max_steps);
  collect_hypotheses(m, 0, chunk0, n, K, o, out_ids, out_lens, out_scores, out_ns);
}

// ---- decode session: a fixed set of S slots of K rows, each refilled from a queue as soon as its item finishes ----------------
// Its decode workspace (self-KV cache, search buffers, slot binding table and step graph) is its own: swapped into the model
// for the duration of each call, so generate / align / detect_language calls in between do not disturb the slots.
struct DecodeWorkspace {
  size_t kv_elems = 0;
  __half *kcache = nullptr, *vcache = nullptr;
  SearchBuffers sb{};
  void* sb_blob = nullptr;
  int sb_B = 0, sb_K = 0;
  DecBindings* d_bind = nullptr;
  DecBindings h_bind{};
  std::vector<DecBindings> h_binds;
  SearchParams h_params{};
  cudaGraphExec_t step_graph = nullptr;
  int64_t step_graph_kernels = 0;
  StepGraphKey step_graph_key{};
};

static void swap_workspace(Model* m, DecodeWorkspace& w) {
  std::swap(m->kv_elems, w.kv_elems);
  std::swap(m->kcache, w.kcache);
  std::swap(m->vcache, w.vcache);
  std::swap(m->sb, w.sb);
  std::swap(m->sb_blob, w.sb_blob);
  std::swap(m->sb_B, w.sb_B);
  std::swap(m->sb_K, w.sb_K);
  std::swap(m->d_bind, w.d_bind);
  std::swap(m->h_bind, w.h_bind);
  std::swap(m->h_binds, w.h_binds);
  std::swap(m->h_params, w.h_params);
  std::swap(m->step_graph, w.step_graph);
  std::swap(m->step_graph_kernels, w.step_graph_kernels);
  std::swap(m->step_graph_key, w.step_graph_key);
  m->sb.suppress = m->d_suppress;
}

struct ScopedWorkspace {
  Model* m;
  DecodeWorkspace& w;
  ScopedWorkspace(Model* m_, DecodeWorkspace& w_) : m(m_), w(w_) { swap_workspace(m, w); }
  ~ScopedWorkspace() { swap_workspace(m, w); }
};

// Drops one reference to an encoder output (under the owner's lock); the last one frees it once the stream has drained.
static void release_encoded(Model* m, Encoded* e) {
  if (!e || --e->refs > 0) return;
  cudaStreamSynchronize(m->stream);
  delete e;
}

struct SessionItem {
  int id;
  Encoded* e;        // holds a reference
  int index;         // item of e
  std::vector<int32_t> prompt;
  int max_length, sot_index;
};

struct Session {
  Model* m;
  b2w_gen_opts o{};
  std::vector<int32_t> suppress_ids;  // o.suppress_tokens points here
  std::vector<uint8_t> mask;
  SearchParams sp{};
  int K = 1, S = 1, next_id = 0;
  DecodeWorkspace ws;
  std::deque<SessionItem> queue;
  std::vector<SessionItem> slot;      // slot[b].id < 0: idle
  std::vector<Encoded*> slot_enc;     // the encoder output slot b is bound to (a reference, kept until the slot is rebound)
  std::vector<DecBindings> bind;      // the step's slot table
  SlotReset* d_resets = nullptr;      // [S]
  int* d_targets = nullptr;           // [kMaxRows]
  float* d_probs = nullptr;           // [kMaxRows]
  RowInfo* d_rows_save = nullptr;     // [kMaxRows] the step's rows and input tokens while a forced pass uses the row table
  int* d_tokens_save = nullptr;       // [kMaxRows]
  bool started = false;
  int64_t steps = 0, live_rows = 0;
  // b2w_session_debug_record: every step's raw logits of each occupied slot (K = 1), kept per item until fetched
  bool record = false;
  float* d_rec = nullptr;             // [S][n_ctx][n_vocab]
  std::vector<int> rec_steps;         // [S] steps recorded since the slot's last refill
  std::map<int, std::vector<float>> rec_items;

  ~Session() {
    for (SessionItem& it : queue) release_encoded(m, it.e);
    for (Encoded* e : slot_enc) release_encoded(m, e);
    cudaStreamSynchronize(m->stream);
    for (void* p : {(void*)ws.kcache, (void*)ws.vcache, ws.sb_blob, (void*)ws.d_bind, (void*)d_resets, (void*)d_targets, (void*)d_probs,
                    (void*)d_rows_save, (void*)d_tokens_save, (void*)d_rec})
      if (p) cudaFree(p);
    if (ws.step_graph) cudaGraphExecDestroy(ws.step_graph);
  }
};

static void session_bind_slot(Session& ss, int b, Encoded* e, int index) {
  ++e->refs;
  release_encoded(ss.m, ss.slot_enc[b]);
  ss.slot_enc[b] = e;
  ss.bind[b] = DecBindings{e->xkv, e->B, index};
}

// Gives every idle slot the next queued item: one reset launch for all of them, then one forced decoding of their prompts[:-1]
// (shorter prompts padded with their last token: those keys are rewritten by the steps before any row reads them), which also
// gives the no-speech probability of items whose <|startoftranscript|> is not the last prompt token.  Runs with the session's
// workspace bound.
static void session_refill(Session& ss) {
  Model* m = ss.m;
  const b2w_config& c = m->cfg;
  cudaStream_t s = m->stream;
  if (!ss.started && ss.queue.empty()) return;
  std::vector<SlotReset> resets;
  std::vector<int> filled;
  for (int b = 0; b < ss.S && !ss.queue.empty(); ++b) {
    if (ss.slot[b].id >= 0) continue;
    SessionItem it = std::move(ss.queue.front());
    ss.queue.pop_front();
    const int P = (int)it.prompt.size();
    SlotReset r{};
    r.slot = b;
    r.last_token = it.prompt[P - 1];
    r.done = 0;
    r.cp = chunk_params(c, it.prompt.data(), P, it.sot_index, it.max_length, it.id, ss.o.return_no_speech_prob);
    resets.push_back(r);
    filled.push_back(b);
    if (ss.record) ss.rec_steps[b] = 0;
    session_bind_slot(ss, b, it.e, it.index);
    release_encoded(m, it.e);  // the queue's reference; the slot holds its own
    ss.slot[b] = std::move(it);
  }
  if (!ss.started) {  // slots that never had an item idle as done chunks bound to a live encoder output
    Encoded* any = nullptr;
    for (int b = 0; b < ss.S && !any; ++b) any = ss.slot_enc[b];
    for (int b = 0; b < ss.S; ++b) {
      if (ss.slot_enc[b]) continue;
      session_bind_slot(ss, b, any, 0);
      SlotReset r{};
      r.slot = b;
      r.last_token = c.sot;
      r.done = 1;
      r.cp = ChunkParams{1, 1, 0, 0, 0, {0, 0, 0}};
      resets.push_back(r);
    }
    B2W_CUDA(cudaMemsetAsync(m->sb.state, 0, sizeof(SearchState), s));
    B2W_CUDA(cudaMemsetAsync(m->sb.done, 0, ss.S * 4, s));
    ss.started = true;
  }
  if (resets.empty()) return;
  B2W_CUDA(cudaMemcpyAsync(ss.d_resets, resets.data(), resets.size() * sizeof(SlotReset), cudaMemcpyHostToDevice, s));
  search_reset_slots(ss.d_resets, (int)resets.size(), ss.S, ss.K, m->sb, s);
  B2W_CUDA(cudaStreamSynchronize(s));
  if (filled.empty()) return;
  int n_tok = 0;
  for (int b : filled) n_tok = std::max(n_tok, (int)ss.slot[b].prompt.size() - 1);
  if (n_tok > 0) {
    ScopedStage st(m, B2W_T_PREFILL);
    const int n = (int)filled.size(), R = ss.S * ss.K;
    // the forced passes use the row table: the occupied slots' rows and tokens are put back afterwards
    B2W_CUDA(cudaMemcpyAsync(ss.d_rows_save, m->sb.rows, R * sizeof(RowInfo), cudaMemcpyDeviceToDevice, s));
    B2W_CUDA(cudaMemcpyAsync(ss.d_tokens_save, m->sb.tokens_in, R * sizeof(int), cudaMemcpyDeviceToDevice, s));
    ForcedChunks fc{std::vector<DecBindings>(n), filled, ss.S};
    std::vector<int32_t> toks((size_t)n * n_tok);
    for (int j = 0; j < n; ++j) {
      const SessionItem& it = ss.slot[filled[j]];
      fc.bind[j] = ss.bind[filled[j]];
      for (int i = 0; i < n_tok; ++i) toks[(size_t)j * n_tok + i] = it.prompt[std::min(i, std::max(0, (int)it.prompt.size() - 2))];
    }
    forced_decode(m, fc, toks.data(), n_tok, n_tok, ss.K, false, nullptr, [&](int i0, int i1) {
      if (!ss.o.return_no_speech_prob) return;
      const int rpc = i1 - i0;
      std::vector<int> targets((size_t)n * rpc, -1);
      std::vector<int> rows_of(n, -1);
      for (int j = 0; j < n; ++j) {
        const SessionItem& it = ss.slot[filled[j]];
        if (it.sot_index >= i0 && it.sot_index < i1 && it.sot_index < (int)it.prompt.size() - 1) {
          rows_of[j] = j * rpc + it.sot_index - i0;
          targets[rows_of[j]] = c.no_speech;
        }
      }
      if (std::all_of(rows_of.begin(), rows_of.end(), [](int r) { return r < 0; })) return;
      logits_gemm(m, n * rpc);
      B2W_CUDA(cudaMemcpyAsync(ss.d_targets, targets.data(), targets.size() * 4, cudaMemcpyHostToDevice, s));
      row_target_probs(m->d_logits, m->vpad, n * rpc, c.n_vocab, ss.d_targets, ss.d_probs, s);
      for (int j = 0; j < n; ++j)
        if (rows_of[j] >= 0)
          B2W_CUDA(cudaMemcpyAsync(m->sb.no_speech + filled[j], ss.d_probs + rows_of[j], 4, cudaMemcpyDeviceToDevice, s));
      B2W_CUDA(cudaStreamSynchronize(s));  // targets goes out of scope
    });
    B2W_CUDA(cudaMemcpyAsync(m->sb.rows, ss.d_rows_save, R * sizeof(RowInfo), cudaMemcpyDeviceToDevice, s));
    B2W_CUDA(cudaMemcpyAsync(m->sb.tokens_in, ss.d_tokens_save, R * sizeof(int), cudaMemcpyDeviceToDevice, s));
  }
}

// One b2w_session_run: refill idle slots, then replay the step graph until a polled done[] shows at least one of the occupied
// slots finished; their results go to the outputs, their slots become idle.  Returns the number of finished items (0 when the
// queue and the slots are empty).
static int session_run(Session& ss, int32_t* out_item, int32_t* out_ids, int32_t* out_lens, float* out_scores, float* out_ns) {
  Model* m = ss.m;
  ScopedWorkspace bound(m, ss.ws);
  cudaStream_t s = m->stream;
  B2W_CUDA(cudaMemcpyAsync(m->d_suppress, ss.mask.data(), m->vpad, cudaMemcpyHostToDevice, s));
  prepare_decode(m, nullptr, ss.S, ss.K);
  session_refill(ss);
  int live = 0;
  for (const SessionItem& it : ss.slot) live += it.id >= 0;
  if (live == 0) return 0;
  Step st = choose_step(m, ss.S, ss.K, false);
  step_args(m, st);
  m->h_params = ss.sp;
  B2W_CUDA(cudaMemcpyAsync(const_cast<SearchParams*>(m->sb.params), &m->h_params, sizeof(SearchParams), cudaMemcpyHostToDevice, s));
  bind_chunks(m, ss.bind);
  const int64_t per_step_kernels = step_graph(m, st);
  const int poll = 4;
  std::vector<int> fin;
  {
    ScopedStage stage(m, B2W_T_DECODE);
    while (fin.empty()) {
      for (int i = 0; i < poll; ++i) {
        B2W_CUDA(cudaGraphLaunch(m->step_graph, s));
        g_launches += per_step_kernels;
        const int V = m->cfg.n_vocab, n_ctx = m->cfg.n_text_ctx;
        for (int b = 0; ss.record && b < ss.S; ++b)
          if (ss.slot[b].id >= 0 && ss.rec_steps[b] < n_ctx)
            B2W_CUDA(cudaMemcpyAsync(ss.d_rec + ((size_t)b * n_ctx + ss.rec_steps[b]++) * V, m->d_logits + (size_t)b * m->vpad,
                                     (size_t)V * 4, cudaMemcpyDeviceToDevice, s));
      }
      ss.steps += poll;
      m->decode_steps += poll;
      ss.live_rows += (int64_t)poll * live * ss.K;
      B2W_CUDA(cudaMemcpyAsync(m->h_pinned, m->sb.done, ss.S * sizeof(int), cudaMemcpyDeviceToHost, s));
      B2W_CUDA(cudaStreamSynchronize(s));
      for (int b = 0; b < ss.S; ++b)
        if (ss.slot[b].id >= 0 && m->h_pinned[b]) fin.push_back(b);
    }
  }
  for (size_t j = 0; j < fin.size(); ++j) {
    const int b = fin[j];
    collect_hypotheses(m, b, (int)j, 1, ss.K, ss.o, out_ids, out_lens, out_scores, out_ns);
    out_item[j] = ss.slot[b].id;
    if (ss.record) {
      const size_t V = m->cfg.n_vocab;
      std::vector<float>& rec = ss.rec_items[ss.slot[b].id];
      rec.resize((size_t)ss.rec_steps[b] * V);
      B2W_CUDA(cudaMemcpy(rec.data(), ss.d_rec + (size_t)b * m->cfg.n_text_ctx * V, rec.size() * 4, cudaMemcpyDeviceToHost));
    }
    ss.slot[b].id = -1;
  }
  return (int)fin.size();
}

// Debug / measurement switches, read once when a model is created (B2W_BSTEP_STOP is read per generate call, in bind_step).
static void read_env_options(Model* m) {
  if (const char* v = getenv("B2W_GEMM_IMPL")) m->use_ref_gemm = !strcmp(v, "ref");
  if (const char* v = getenv("B2W_ATTN_IMPL")) m->use_ref_attn = !strcmp(v, "ref");
  if (const char* v = getenv("B2W_STEP")) {
    if (!strcmp(v, "dstep")) m->forced_step = StepPath::Dstep;
    else if (!strcmp(v, "bstep")) m->forced_step = StepPath::Bstep;
    else if (!strcmp(v, "layers")) m->forced_step = StepPath::Layers;
    else if (*v) throw Error(std::string("B2W_STEP must be dstep, bstep or layers, not ") + v, true);
  }
  if (const char* v = getenv("B2W_DSTEP_PROF")) {
    if (strcmp(v, "0") != 0) {
      m->d_prof = model_alloc<unsigned long long>(m, 4096);
      B2W_CUDA(cudaMemset(m->d_prof, 0, 4096 * sizeof(unsigned long long)));
    }
  }
}

}  // namespace b2w

// =================================================================================================================
// C ABI
// =================================================================================================================
using namespace b2w;

struct b2w_model {
  Model m;
};
struct b2w_encoded {
  Encoded* e;
};
struct b2w_session {
  Session s;
};

// Runs f(m) with calls on the model serialised, its device current and the kernels f launches added to its counter.
template <typename F>
static void with_model(Model* m, F&& f) {
  std::lock_guard<std::mutex> lk(m->mu);
  DeviceGuard g(m->device);
  const int64_t before = g_launches;
  f(m);
  m->launches += g_launches - before;
}

// An entry point that works on a model.  f validates its arguments before any device work.
template <typename F>
static int guarded(b2w_model* h, F&& f) {
  return guarded([&] {
    B2W_CHECK(h, "null model");
    with_model(&h->m, f);
  });
}

// ---- helpers of the test hooks ----------------------------------------------------------------------------------------
static_assert(B2W_EPI_F16 == EPI_F16 && B2W_EPI_GELU_F16 == EPI_GELU_F16 && B2W_EPI_RESID_F32 == EPI_RESID_F32 &&
                  B2W_EPI_GELU_POS_F32 == EPI_GELU_POS_F32 && B2W_EPI_F16_XKV == EPI_F16_XKV && B2W_EPI_F32 == EPI_F32 &&
                  B2W_EPI_QKV_CACHE == EPI_QKV_CACHE, "public epilogue ids");
static_assert(B2W_GV_QKV == GV_QKV && B2W_GV_F16 == GV_F16 && B2W_GV_GELU_F16 == GV_GELU_F16 && B2W_GV_RESID_LN == GV_RESID_LN &&
                  B2W_GV_F32 == GV_F32, "public decode GEMM modes");

static void hook_get(void* host, const void* dev, size_t bytes) {
  if (host) B2W_CUDA(cudaMemcpy(host, dev, bytes, cudaMemcpyDeviceToHost));
}

// rows x (chunk, slot, pos, -) must address entries of a [chunk][n_ctx][slots][d] cache of cache_elems halves
static void check_row_table(const int32_t* rows, int R, int n_ctx, int slots, int d, int64_t cache_elems) {
  B2W_CHECK(rows && n_ctx >= 1 && slots >= 1 && d >= 1, "row table and cache geometry");
  for (int r = 0; r < R; ++r) {
    const int32_t* ri = rows + 4 * r;
    B2W_CHECK(ri[0] >= 0 && ri[1] >= 0 && ri[1] < slots && ri[2] >= 0 && ri[2] < n_ctx &&
                  (((int64_t)ri[0] * n_ctx + ri[2]) * slots + ri[1] + 1) * d <= cache_elems,
              "row table entry outside the cache");
  }
}


// ---- Silero VAD ------------------------------------------------------------------------------------------------------
// The weights b2w_vad_create takes: name, and shape (fp32 only).
static const struct {
  const char* name;
  std::initializer_list<int64_t> shape;
} kVadTensors[] = {
    {"basis", {258, 256}},           {"conv0.weight", {128, 129, 3}}, {"conv0.bias", {128}}, {"conv1.weight", {64, 128, 3}},
    {"conv1.bias", {64}},            {"conv2.weight", {64, 64, 3}},   {"conv2.bias", {64}},  {"conv3.weight", {128, 64, 3}},
    {"conv3.bias", {128}},           {"lstm.w_ih", {512, 128}},       {"lstm.w_hh", {512, 128}}, {"lstm.bias", {512}},
    {"decoder.weight", {128}},       {"decoder.bias", {1}},
};

struct b2w_vad {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  ScratchBufs weights;        // every weight buffer and the LSTM state
  VadWeights w;
  const float *w_hh = nullptr, *dec_w = nullptr, *dec_b = nullptr;
  int64_t block = 32768;      // windows per block, summed over the streams of a launch; the buffers below take
                              // (512 + 512 + 128 + 1) floats = 4.6 KB per window, and 64 + 256 floats and a table entry per stream
  int64_t cap = 0;            // windows the block buffers hold
  int64_t cap_streams = 0;    // streams they hold
  std::unique_ptr<ScratchBufs> bufs;
  float *pcm = nullptr, *gx = nullptr, *H = nullptr, *probs = nullptr;
  float* states = nullptr;    // per stream: h [128] then c [128], carried from launch to launch
  VadSlice* slices = nullptr; // the launch's stream table
  std::vector<VadSlice> host_slices;
  std::vector<float> host_probs;
  cudaEvent_t ev[4] = {};
  double ms[3] = {0, 0, 0};   // last call: window kernel, recurrence, decoder
  ~b2w_vad() {  // the buffers are freed after this body, once the stream has drained
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
};

// host fp32 [rows][cols] -> device [cols][rows]
static float* vad_upload_t(ScratchBufs& sb, const b2w_tensor& t, int64_t rows, int64_t cols) {
  const float* src = static_cast<const float*>(t.data);
  std::vector<float> h((size_t)(rows * cols));
  for (int64_t r = 0; r < rows; ++r)
    for (int64_t c = 0; c < cols; ++c) h[(size_t)(c * rows + r)] = src[r * cols + c];
  return sb.put<float>(h.data(), h.size());
}

extern "C" {

const char* b2w_last_error(void) { return g_last_error.c_str(); }
int b2w_abi_version(void) { return B2W_ABI_VERSION; }
int b2w_device_count(int* count) {
  return guarded([&] {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    *count = (e == cudaSuccess) ? n : 0;
  });
}

void b2w_gen_opts_default(b2w_gen_opts* o) {
  memset(o, 0, sizeof *o);
  o->beam_size = 5;
  o->patience = 1.f;
  o->num_hypotheses = 1;
  o->length_penalty = 1.f;
  o->repetition_penalty = 1.f;
  o->max_length = 448;
  o->max_initial_timestamp_index = 50;
  o->suppress_blank = 1;
  o->sampling_topk = 1;
  o->sampling_temperature = 1.f;
}

int b2w_model_create(const b2w_config* cfg, const b2w_tensor* tensors, int32_t n_tensors, int32_t device,
                     const char* compute_type, b2w_model** out) {
  return guarded([&] {
    B2W_CHECK(cfg && tensors && out, "null argument");
    require_hopper(device);
    const std::string ct = compute_type ? compute_type : "default";
    const char* ok[] = {"default", "auto", "float16", "int8_float16", "int8", "float32", "bfloat16", "int8_float32", "int8_bfloat16", "int16",
                        "float8_float16"};
    bool known = false;
    for (const char* k : ok) known = known || ct == k;
    if (!known) throw Error("unknown compute_type: " + ct, true);
    DeviceGuard g(device);
    std::unique_ptr<b2w_model> h(new b2w_model);
    Model* m = &h->m;
    m->device = device;
    cudaDeviceProp prop;
    B2W_CUDA(cudaGetDeviceProperties(&prop, device));
    m->num_sms = prop.multiProcessorCount;
    B2W_CUDA(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    m->w8 = ct.rfind("int8", 0) == 0;
    m->fp8_enc = ct == "float8_float16";
    read_env_options(m);
    if (m->fp8_enc && m->use_ref_gemm)
      throw Error("compute_type float8_float16 runs the encoder on the e4m3 wgmma GEMM; B2W_GEMM_IMPL=ref has no fp8 path", true);
    TensorTable tt{tensors, n_tensors};
    build_model(m, *cfg, tt);
    *out = h.release();
  });
}

void b2w_model_destroy(b2w_model* m) { delete m; }

// reads only what b2w_model_create fixed, so it neither waits for the model nor touches the device
int b2w_model_info(const b2w_model* m, b2w_config* cfg_out, int32_t* device_out) {
  return guarded([&] {
    B2W_CHECK(m, "null model");
    if (cfg_out) *cfg_out = m->m.cfg;
    if (device_out) *device_out = m->m.device;
  });
}

int b2w_model_sync(b2w_model* h) {
  return guarded(h, [&](Model* m) { B2W_CUDA(cudaStreamSynchronize(m->stream)); });
}

int b2w_logmel_frames(int64_t n_samples, int32_t padding) {
  (void)padding;
  return mel_frames(n_samples);
}

int b2w_logmel(int32_t device, int32_t n_mels, const float* pcm, int64_t n_samples, int32_t padding, float* out,
               int64_t out_capacity, int32_t* n_frames_out) {
  return guarded([&] {
    B2W_CHECK(n_mels > 0 && n_mels <= 128 && n_samples >= 0 && padding >= 0, "bad log-mel arguments");
    require_hopper(device);
    DeviceGuard g(device);
    static thread_local std::map<std::pair<int, int>, std::unique_ptr<MelPlan>> plans;
    auto& plan = plans[{device, n_mels}];
    if (!plan) plan.reset(new MelPlan(n_mels));
    // 1 + (len + 2*200 - 400)/160 STFT frames of the zero-padded signal, minus the dropped last one
    const int n_frames = (int)((n_samples + padding) / 160);
    if (n_frames_out) *n_frames_out = n_frames;
    B2W_CHECK((int64_t)n_frames * n_mels <= out_capacity, "output buffer too small");
    if (n_frames == 0) return;
    cudaStream_t s = nullptr;
    B2W_CUDA(cudaStreamCreate(&s));
    std::unique_ptr<CUstream_st, decltype(&cudaStreamDestroy)> own_s(s, cudaStreamDestroy);  // destroyed after the buffers
    ScratchBufs sb;
    float* d_pcm = sb.alloc<float>(n_samples);
    float* d_out = sb.alloc<float>((size_t)n_frames * n_mels);
    MelChunkDesc* d_desc = sb.alloc<MelChunkDesc>(1);
    int* d_max = sb.alloc<int>(1);
    if (n_samples) B2W_CUDA(cudaMemcpyAsync(d_pcm, pcm, n_samples * 4, cudaMemcpyHostToDevice, s));
    MelChunkDesc desc{d_pcm, n_samples, n_frames, n_frames};
    B2W_CUDA(cudaMemcpyAsync(d_desc, &desc, sizeof desc, cudaMemcpyHostToDevice, s));
    plan->run(d_desc, 1, n_frames, padding, d_out, 0, n_frames, d_max, false, s);
    B2W_CUDA(cudaMemcpyAsync(out, d_out, (size_t)n_frames * n_mels * 4, cudaMemcpyDeviceToHost, s));
    B2W_CUDA(cudaStreamSynchronize(s));
  });
}

int b2w_encode(b2w_model* h, const float* features, int32_t batch, b2w_encoded** out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(features && out && batch > 0, "bad encode arguments");
    const size_t per = (size_t)m->cfg.n_mels * 3000;
    std::unique_ptr<Encoded> e = encode(m, batch, [&](int b0, int b) {
      ScopedStage st(m, B2W_T_H2D);
      B2W_CUDA(cudaMemcpyAsync(m->e_feats, features + b0 * per, b * per * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    });
    *out = new b2w_encoded{e.release()};
  });
}

int b2w_encode_audio(b2w_model* h, const float* const* pcm, const int64_t* n_samples, int32_t batch, float* features_out,
                     b2w_encoded** out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(pcm && n_samples && out && batch > 0, "bad encode_audio arguments");
    for (int i = 0; i < batch; ++i)
      B2W_CHECK(n_samples[i] >= 0 && n_samples[i] <= 480000, "a chunk holds at most 30 s of 16 kHz audio");
    const size_t per = (size_t)m->cfg.n_mels * 3000;
    std::unique_ptr<Encoded> e = encode(m, batch, [&](int b0, int b) {
      size_t total = 0;
      for (int i = 0; i < b; ++i) total += (n_samples[b0 + i] + 3) & ~size_t(3);
      if (total > m->e_pcm_cap) {
        B2W_CUDA(cudaStreamSynchronize(m->stream));
        if (m->e_pcm) cudaFree(m->e_pcm);
        m->e_pcm = dalloc<float>(total);
        m->e_pcm_cap = total;
      }
      std::vector<MelChunkDesc> desc(b);
      int max_frames = 1;
      {
        ScopedStage st(m, B2W_T_H2D);
        size_t off = 0;
        for (int i = 0; i < b; ++i) {
          const int64_t ns = n_samples[b0 + i];
          if (ns) B2W_CUDA(cudaMemcpyAsync(m->e_pcm + off, pcm[b0 + i], ns * 4, cudaMemcpyHostToDevice, m->stream));
          const int nf = mel_frames(ns);
          // feature_extractor(chunk)[..., :-1] then pad_or_trim(3000): emit min(nf-1, 3000) frames, zero-fill the rest
          desc[i] = MelChunkDesc{m->e_pcm + off, ns, nf, std::min(nf - 1, 3000)};
          max_frames = std::max(max_frames, nf);
          off += (ns + 3) & ~size_t(3);
        }
        B2W_CUDA(cudaMemcpyAsync(m->e_chunks, desc.data(), b * sizeof(MelChunkDesc), cudaMemcpyHostToDevice, m->stream));
      }
      {
        ScopedStage st(m, B2W_T_MEL);
        m->mel->run(m->e_chunks, b, max_frames, 160, m->e_feats, (int64_t)per, 3000, m->e_chunk_max, true, m->stream);
      }
      if (features_out) {
        ScopedStage st(m, B2W_T_D2H);
        B2W_CUDA(cudaMemcpyAsync(features_out + (size_t)b0 * per, m->e_feats, (size_t)b * per * 4, cudaMemcpyDeviceToHost, m->stream));
      }
      B2W_CUDA(cudaStreamSynchronize(m->stream));  // desc vector lifetime
    });
    *out = new b2w_encoded{e.release()};
  });
}

int b2w_encoded_shape(const b2w_encoded* e, int64_t shape_out[3]) {
  return guarded([&] {
    B2W_CHECK(e && e->e, "null encoder output");
    shape_out[0] = e->e->B;
    shape_out[1] = 1500;
    shape_out[2] = e->e->owner->cfg.n_audio_state;
  });
}

int b2w_encoded_to_host(b2w_model* h, const b2w_encoded* e, float* out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(e && e->e && out, "bad arguments");
    const size_t n = (size_t)e->e->B * 1500 * m->cfg.n_audio_state;
    ScratchBufs sb;
    float* tmp = sb.alloc<float>(n);
    convert_f16_f32(e->e->enc_out, tmp, n, m->stream);
    B2W_CUDA(cudaMemcpyAsync(out, tmp, n * 4, cudaMemcpyDeviceToHost, m->stream));
    B2W_CUDA(cudaStreamSynchronize(m->stream));
  });
}

void b2w_encoded_free(b2w_encoded* e) {
  if (!e) return;
  if (e->e)  // the owner's stream may still read the output; ~Encoded returns its buffers to the owner's pool
    guarded([&] { with_model(e->e->owner, [&](Model* m) { release_encoded(m, e->e); }); });
  delete e;
}

int b2w_generate(b2w_model* h, b2w_encoded* enc, const int32_t* prompts, int32_t prompt_len, int32_t batch,
                 const b2w_gen_opts* opts, int32_t* out_ids, int32_t* out_lens, float* out_scores, float* out_no_speech) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(prompts && opts && out_ids && out_lens && out_scores && out_no_speech, "null argument");
    const b2w_gen_opts& o = *opts;
    B2W_CHECK(batch > 0 && prompt_len > 0, "empty batch or prompt");
    B2W_CHECK(o.debug_fake_logits || (enc && enc->e && enc->e->B == batch), "one prompt per encoder output row is required");
    const int K = check_gen_opts(m->cfg, o);
    const int group = std::max(1, kMaxRows / K);
    {
      const std::vector<uint8_t> mask = suppress_mask(m->cfg, m->vpad, o);
      B2W_CUDA(cudaMemcpyAsync(m->d_suppress, mask.data(), m->vpad, cudaMemcpyHostToDevice, m->stream));
      B2W_CUDA(cudaStreamSynchronize(m->stream));
    }
    Encoded* e = enc ? enc->e : nullptr;
    prepare_decode(m, o.debug_fake_logits ? nullptr : e, std::min(group, (int)batch), K);
    for (int c0 = 0; c0 < batch; c0 += group) {
      const int n = std::min(group, batch - c0);
      generate_group(m, e, c0, n, prompts, prompt_len, o, out_ids, out_lens, out_scores, out_no_speech);
    }
  });
}

int b2w_session_create(b2w_model* h, const b2w_gen_opts* opts, int32_t* slots, b2w_session** out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(opts && slots && out, "null argument");
    B2W_CHECK(*slots >= 0, "slots must be 0 (as many as fit) or positive");
    B2W_CHECK(!opts->debug_fake_logits, "a decode session decodes encoder outputs: debug_fake_logits is not supported");
    B2W_CHECK(opts->n_suppress_tokens >= 0 && (opts->n_suppress_tokens == 0 || opts->suppress_tokens), "suppress_tokens");
    const int K = check_gen_opts(m->cfg, *opts);
    std::unique_ptr<b2w_session> h2(new b2w_session);
    Session& ss = h2->s;
    ss.m = m;
    ss.o = *opts;
    ss.suppress_ids.assign(opts->suppress_tokens, opts->suppress_tokens + opts->n_suppress_tokens);
    ss.o.suppress_tokens = ss.suppress_ids.data();
    ss.mask = suppress_mask(m->cfg, m->vpad, ss.o);
    ss.K = K;
    ss.S = std::max(1, kMaxRows / K);
    if (*slots > 0) ss.S = std::min(ss.S, (int)*slots);
    ss.sp = search_params(m->cfg, m->vpad, ss.S, K, ss.o);
    ss.slot.resize(ss.S);
    for (SessionItem& it : ss.slot) it.id = -1;
    ss.slot_enc.assign(ss.S, nullptr);
    ss.bind.resize(ss.S);
    ss.ws.d_bind = dalloc<DecBindings>(kMaxRows);
    ss.d_resets = dalloc<SlotReset>(ss.S);
    ss.d_targets = dalloc<int>(kMaxRows);
    ss.d_probs = dalloc<float>(kMaxRows);
    ss.d_rows_save = dalloc<RowInfo>(kMaxRows);
    ss.d_tokens_save = dalloc<int>(kMaxRows);
    *slots = ss.S;
    *out = h2.release();
  });
}

int b2w_session_push(b2w_session* sh, b2w_encoded* enc, int32_t item_index, const int32_t* prompt, int32_t prompt_len,
                     int32_t max_length, int32_t* item_id_out) {
  return guarded([&] {
    B2W_CHECK(sh && enc && enc->e && prompt && item_id_out, "null argument");
    Session& ss = sh->s;
    with_model(ss.m, [&](Model* m) {
      Encoded* e = enc->e;
      B2W_CHECK(e->owner == m, "the encoder output belongs to another model");
      B2W_CHECK(item_index >= 0 && item_index < e->B, "item_index is outside the encoder output");
      B2W_CHECK(prompt_len >= 1, "empty prompt");
      B2W_CHECK(max_length > prompt_len && max_length <= ss.o.max_length,
                "max_length must exceed the prompt length and be at most the session's max_length");
      const int sot_index = validate_prompts(m->cfg, prompt, 1, prompt_len);
      ensure_cross_kv(m, e);
      ++e->refs;
      ss.queue.push_back(SessionItem{ss.next_id, e, item_index, std::vector<int32_t>(prompt, prompt + prompt_len), max_length, sot_index});
      *item_id_out = ss.next_id++;
    });
  });
}

int b2w_session_run(b2w_session* sh, int32_t* n_out, int32_t* out_item_ids, int32_t* out_ids, int32_t* out_lens, float* out_scores,
                    float* out_no_speech) {
  return guarded([&] {
    B2W_CHECK(sh && n_out && out_item_ids && out_ids && out_lens && out_scores && out_no_speech, "null argument");
    Session& ss = sh->s;
    with_model(ss.m, [&](Model*) { *n_out = session_run(ss, out_item_ids, out_ids, out_lens, out_scores, out_no_speech); });
  });
}

int b2w_session_pending(b2w_session* sh, int32_t* n_out) {
  return guarded([&] {
    B2W_CHECK(sh && n_out, "null argument");
    Session& ss = sh->s;
    with_model(ss.m, [&](Model*) {
      int n = (int)ss.queue.size();
      for (const SessionItem& it : ss.slot) n += it.id >= 0;
      *n_out = n;
    });
  });
}

int b2w_session_counters(b2w_session* sh, int64_t* steps, int64_t* live_rows) {
  return guarded([&] {
    B2W_CHECK(sh && steps && live_rows, "null argument");
    Session& ss = sh->s;
    with_model(ss.m, [&](Model*) {
      *steps = ss.steps;
      *live_rows = ss.live_rows;
    });
  });
}

int b2w_session_debug_record(b2w_session* sh) {
  return guarded([&] {
    B2W_CHECK(sh, "null argument");
    Session& ss = sh->s;
    with_model(ss.m, [&](Model* m) {
      B2W_CHECK(ss.K == 1, "logits are recorded for one row per slot (beam_size 1, num_hypotheses 1)");
      B2W_CHECK(!ss.started, "recording starts before the first b2w_session_run");
      if (!ss.d_rec) ss.d_rec = dalloc<float>((size_t)ss.S * m->cfg.n_text_ctx * m->cfg.n_vocab);
      ss.rec_steps.assign(ss.S, 0);
      ss.record = true;
    });
  });
}

int b2w_session_debug_logits(b2w_session* sh, int32_t item_id, float* out, int32_t capacity_steps, int32_t* n_steps_out) {
  return guarded([&] {
    B2W_CHECK(sh && n_steps_out && (out || capacity_steps == 0) && capacity_steps >= 0, "null argument");
    Session& ss = sh->s;
    with_model(ss.m, [&](Model* m) {
      auto it = ss.rec_items.find(item_id);
      B2W_CHECK(it != ss.rec_items.end(), "no recorded logits for this item (recording off, item unfinished or already fetched)");
      const size_t V = m->cfg.n_vocab, n = it->second.size() / V;
      B2W_CHECK(n <= (size_t)capacity_steps, "output buffer too small");
      std::copy(it->second.begin(), it->second.end(), out);
      *n_steps_out = (int32_t)n;
      ss.rec_items.erase(it);
    });
  });
}

void b2w_session_destroy(b2w_session* sh) {
  if (!sh) return;
  Model* m = sh->s.m;
  guarded([&] { with_model(m, [&](Model*) { delete sh; }); });
}

int b2w_detect_language(b2w_model* h, b2w_encoded* enc, float* probs) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(enc && enc->e && probs, "null argument");
    Encoded* e = enc->e;
    const int nl = m->cfg.num_languages;
    const int group = kMaxRows;
    prepare_decode(m, e, std::min(group, e->B), 1);
    ScratchBufs sb;
    float* d_probs = sb.alloc<float>((size_t)e->B * nl);
    const std::vector<int32_t> sot(group, m->cfg.sot);
    for (int c0 = 0; c0 < e->B; c0 += group) {
      const int n = std::min(group, e->B - c0);
      forced_decode(m, forced_range(e, c0, n), sot.data(), 1, 1, 1, true, nullptr, [&](int, int) {
        logits_gemm(m, n);
        lang_probs_from_logits(m->d_logits, m->vpad, n, m->cfg.lang_begin, nl, d_probs + (size_t)c0 * nl, m->stream);
      });
    }
    B2W_CUDA(cudaMemcpyAsync(probs, d_probs, (size_t)e->B * nl * 4, cudaMemcpyDeviceToHost, m->stream));
    B2W_CUDA(cudaStreamSynchronize(m->stream));
  });
}

// ---- Whisper.align --------------------------------------------------------------------------------------------------------
// Capture of one align group (items x alignment heads x positions x frames, fp32): 320 heads of a 155-position, 1500-frame
// chunk take 300 MB.  A single item may exceed it.
constexpr size_t kAlignCaptureBytes = (size_t)2 << 30;

static int align_frames(int num_frames) { return std::max(1, std::min(1500, num_frames / 2)); }

// Checks an item's forced sequence, start_sequence + <|notimestamps|> + text + <|endoftext|>, against the model.
static void check_align_sequence(const b2w_config& c, const int32_t* start, int n_start, const int32_t* text, int n_text) {
  if (n_start + n_text + 2 > c.n_text_ctx) throw Error("align: start sequence + text exceed the decoder context", true);
  for (int i = 0; i < n_start + n_text; ++i) {
    const int t = i < n_start ? start[i] : text[i - n_start];
    if (t < 0 || t >= c.n_vocab) throw Error("align: token id out of range", true);
  }
}

struct AlignItem {
  Encoded* e;               // the item's encoder output, and its index there
  int index;
  const int32_t* text;
  int n_text, nf;
  float* probs;             // host [n_text]: probability of each text token at the position that predicts it
  std::vector<int2> pairs;  // the DTW path (text index, frame index); none when n_text = 0
};

// Aligns each of `items` against its own encoder item (arguments already checked).  Consecutive items form groups whose padded
// sequences fit one pass of kMaxRows rows, so that every pass reads each chunk's cross-attention K/V once: splitting a long
// sequence over the passes of a group would re-read every chunk's K/V in each pass, which costs more than the weights it shares
// (an item longer than a pass is a group of its own).  The group's cross-attention counters and capture must fit too.  A group's
// sequences are padded with <|endoftext|> to its longest, and the padded positions' capture and probabilities are never read
// (attention is causal, so they do not change the real rows).  Per group: the forced decode with the capture and the text-token
// probabilities, then the cost matrix and the DTW on the device.  Pairs, counts and probabilities come back with one copy each
// and one synchronise.
static void align_run(Model* m, const int32_t* start, int n_start, std::vector<AlignItem>& items, int width) {
  const b2w_config& c = m->cfg;
  cudaStream_t s = m->stream;
  const int n_heads = (int)m->align_heads.size(), n_items = (int)items.size();
  B2W_CHECK(n_heads > 0, "no alignment heads");
  struct Group {
    int i0, n, T, nf;            // first item, items, padded positions, frames of the capture
    size_t tp_off, pair_off;     // offsets of the group's probabilities and pair slots in the call's buffers
  };
  std::vector<Group> groups;
  size_t tp_total = 0, pair_total = 0, cap_max = 0, stats_max = 0, cost_max = 0;
  for (int i0 = 0; i0 < n_items;) {
    Group g{i0, 0, 0, 0, tp_total, pair_total};
    while (i0 + g.n < n_items) {
      const int n = g.n + 1, T = std::max(g.T, n_start + items[i0 + g.n].n_text + 2), nf = std::max(g.nf, items[i0 + g.n].nf);
      const bool fits = n * T <= kMaxRows && (size_t)n * c.n_text_head * ds_xqgroups(forced_positions_per_pass(n)) <= kCrossGroupCounters &&
                        (size_t)n * n_heads * T * nf * sizeof(float) <= kAlignCaptureBytes;
      if (g.n > 0 && !fits) break;
      g.n = n, g.T = T, g.nf = nf;
    }
    const size_t row_stride = g.T - n_start - 1;  // n_text + 1 of the group's longest text
    tp_total += (size_t)g.n * g.T;
    pair_total += (size_t)g.n * (row_stride + g.nf);
    cap_max = std::max(cap_max, (size_t)g.n * n_heads * g.T * g.nf);
    stats_max = std::max(stats_max, (size_t)g.n * n_heads * 2 * g.nf);
    cost_max = std::max(cost_max, (size_t)g.n * row_stride * g.nf);
    groups.push_back(g);
    i0 += g.n;
  }
  // row of position i of the group's item b in its forced decode: passes of p positions of every item, pass-major
  auto row_of = [](const Group& g, int b, int i) {
    const int p = forced_positions_per_pass(g.n), i0 = i / p * p, rpc = std::min(g.T, i0 + p) - i0;
    return g.tp_off + (size_t)g.n * i0 + (size_t)b * rpc + (i - i0);
  };
  std::vector<int> targets(tp_total, -1);  // position n_start + t predicts text token t
  std::vector<int4> desc(n_items);
  for (const Group& g : groups)
    for (int b = 0; b < g.n; ++b) {
      const AlignItem& it = items[g.i0 + b];
      for (int t = 0; t < it.n_text; ++t) targets[row_of(g, b, n_start + t)] = it.text[t];
      desc[g.i0 + b] = make_int4(n_start + it.n_text + 2, it.nf, n_start, it.n_text > 0 ? it.n_text + 1 : 0);
    }
  int max_n = 0;
  for (const Group& g : groups) max_n = std::max(max_n, g.n);
  prepare_decode(m, nullptr, max_n, 1);
  for (const AlignItem& it : items) ensure_cross_kv(m, it.e);
  if (!m->d_align_heads) {
    m->d_align_heads = dalloc<int2>(n_heads);
    B2W_CUDA(cudaMemcpy(m->d_align_heads, m->align_heads.data(), n_heads * sizeof(int2), cudaMemcpyHostToDevice));
  }
  struct PoolBufs {  // returned to the model's pool when the call ends
    Model* m;
    std::vector<std::pair<void*, size_t>> v;
    void* get(size_t bytes) {
      bytes = std::max<size_t>(bytes, 1);
      v.emplace_back(m->pool_get(bytes), bytes);
      return v.back().first;
    }
    ~PoolBufs() {
      for (auto& x : v) m->pool_put(x.first, x.second);
    }
  } pb{m, {}};
  float* d_cap = static_cast<float*>(pb.get(cap_max * sizeof(float)));
  double* d_stats = static_cast<double*>(pb.get(stats_max * sizeof(double)));
  double* d_cost = static_cast<double*>(pb.get(cost_max * sizeof(double)));
  int* d_targets = static_cast<int*>(pb.get(tp_total * sizeof(int)));
  float* d_tp = static_cast<float*>(pb.get(tp_total * sizeof(float)));
  int2* d_pairs = static_cast<int2*>(pb.get(pair_total * sizeof(int2)));
  int* d_counts = static_cast<int*>(pb.get(n_items * sizeof(int)));
  int4* d_items = static_cast<int4*>(pb.get(n_items * sizeof(int4)));
  B2W_CUDA(cudaMemcpyAsync(d_targets, targets.data(), tp_total * sizeof(int), cudaMemcpyHostToDevice, s));
  B2W_CUDA(cudaMemcpyAsync(d_items, desc.data(), n_items * sizeof(int4), cudaMemcpyHostToDevice, s));
  B2W_CUDA(cudaMemsetAsync(d_tp, 0, tp_total * sizeof(float), s));
  B2W_CUDA(cudaMemsetAsync(d_counts, 0, n_items * sizeof(int), s));
  for (const Group& g : groups) {
    bool any = false;
    for (int b = 0; b < g.n; ++b) any = any || items[g.i0 + b].n_text > 0;
    if (!any) continue;
    std::vector<int32_t> toks((size_t)g.n * g.T, c.eot);
    for (int b = 0; b < g.n; ++b) {
      const AlignItem& it = items[g.i0 + b];
      int32_t* p = toks.data() + (size_t)b * g.T;
      std::copy(start, start + n_start, p);
      p[n_start] = c.no_timestamps;
      std::copy(it.text, it.text + it.n_text, p + n_start + 1);
    }
    const AlignCapture cap{m->d_align_heads, n_heads, d_cap, g.T, g.nf};
    ForcedChunks fc{std::vector<DecBindings>(g.n), std::vector<int>(g.n), g.n};
    for (int b = 0; b < g.n; ++b) {
      const AlignItem& it = items[g.i0 + b];
      fc.bind[b] = DecBindings{it.e->xkv, it.e->B, it.index};
      fc.kv_chunk[b] = b;
    }
    forced_decode(m, fc, toks.data(), g.T, g.T, 1, true, &cap, [&](int i0, int i1) {
      const int R = g.n * (i1 - i0);
      const size_t off = g.tp_off + (size_t)g.n * i0;
      logits_gemm(m, R);
      row_target_probs(m->d_logits, m->vpad, R, c.n_vocab, d_targets + off, d_tp + off, s);
    });
    const int row_stride = g.T - n_start - 1;
    const AlignBatch ab{d_cap, d_stats, d_cost, d_items + g.i0, n_heads, g.T, g.nf, row_stride, width, d_pairs + g.pair_off, d_counts + g.i0};
    align_cost(ab, g.n, s);
    align_dtw(ab, g.n, s);
  }
  std::vector<int> counts(n_items);
  std::vector<float> tp(tp_total);
  std::vector<int2> pairs(pair_total);
  B2W_CUDA(cudaMemcpyAsync(counts.data(), d_counts, n_items * sizeof(int), cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(tp.data(), d_tp, tp_total * sizeof(float), cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(pairs.data(), d_pairs, pair_total * sizeof(int2), cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaStreamSynchronize(s));
  for (const Group& g : groups) {
    const size_t slot = (size_t)(g.T - n_start - 1) + g.nf;
    for (int b = 0; b < g.n; ++b) {
      AlignItem& it = items[g.i0 + b];
      for (int t = 0; t < it.n_text; ++t) it.probs[t] = tp[row_of(g, b, n_start + t)];
      const int2* p = pairs.data() + g.pair_off + b * slot;
      it.pairs.assign(p, p + counts[g.i0 + b]);
    }
  }
}

int b2w_model_set_alignment_heads(b2w_model* h, const int32_t* layer_head_pairs, int32_t n_pairs) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK((n_pairs == 0 || layer_head_pairs) && n_pairs >= 0 && n_pairs <= 32 * 32, "bad arguments");
    std::vector<int2> v;
    for (int i = 0; i < n_pairs; ++i) {
      const int l = layer_head_pairs[2 * i], hd = layer_head_pairs[2 * i + 1];
      if (l < 0 || l >= m->cfg.n_text_layer || hd < 0 || hd >= m->cfg.n_text_head) throw Error("alignment head out of range", true);
      v.push_back(make_int2(l, hd));
    }
    m->align_heads = v.empty() ? default_alignment_heads(m->cfg) : v;
    if (m->d_align_heads) {
      cudaFree(m->d_align_heads);
      m->d_align_heads = nullptr;
    }
  });
}

int b2w_align(b2w_model* h, b2w_encoded* enc, int32_t batch_index, const int32_t* start_sequence, int32_t n_start,
              const int32_t* text_tokens, int32_t n_text, int32_t num_frames, int32_t median_filter_width, int32_t* alignments_out,
              int32_t capacity_pairs, int32_t* n_pairs_out, float* text_token_probs_out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(enc && enc->e && start_sequence && n_pairs_out && n_start >= 1 && n_text >= 0, "bad arguments");
    Encoded* e = enc->e;
    if (batch_index < 0 || batch_index >= e->B) throw Error("align: batch index out of range", true);
    if (median_filter_width < 1 || median_filter_width % 2 == 0) throw Error("align: median_filter_width must be odd", true);
    *n_pairs_out = 0;
    if (n_text == 0) return;
    B2W_CHECK(text_tokens && text_token_probs_out && (alignments_out || capacity_pairs == 0), "bad arguments");
    check_align_sequence(m->cfg, start_sequence, n_start, text_tokens, n_text);
    std::vector<AlignItem> items{AlignItem{e, batch_index, text_tokens, n_text, align_frames(num_frames), text_token_probs_out, {}}};
    align_run(m, start_sequence, n_start, items, median_filter_width);
    const std::vector<int2>& p = items[0].pairs;
    *n_pairs_out = (int32_t)p.size();
    if ((int)p.size() > capacity_pairs) throw Error("align: alignment buffer too small", true);
    for (size_t i = 0; i < p.size(); ++i) {
      alignments_out[2 * i] = p[i].x;
      alignments_out[2 * i + 1] = p[i].y;
    }
  });
}

int b2w_align_items(b2w_model* h, const b2w_encoded* const* encs, const int32_t* items_in, int32_t n_items,
                    const int32_t* start_sequence, int32_t n_start, const int32_t* text_tokens, const int32_t* text_offsets,
                    const int32_t* num_frames, int32_t median_filter_width, int32_t* alignments_out, int32_t capacity_pairs,
                    int32_t* pair_offsets_out, float* text_token_probs_out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(encs && items_in && n_items >= 1 && start_sequence && n_start >= 1 && text_offsets && num_frames && pair_offsets_out,
              "bad arguments");
    const int B = n_items;
    if (median_filter_width < 1 || median_filter_width % 2 == 0) throw Error("align: median_filter_width must be odd", true);
    if (text_offsets[0] != 0) throw Error("align: text_offsets must start at 0", true);
    for (int b = 0; b < B; ++b)
      if (text_offsets[b + 1] < text_offsets[b]) throw Error("align: text_offsets must not decrease", true);
    B2W_CHECK(text_offsets[B] == 0 || (text_tokens && text_token_probs_out), "bad arguments");
    std::vector<AlignItem> items(B);
    int64_t need = 0;
    for (int b = 0; b < B; ++b) {
      AlignItem& it = items[b];
      B2W_CHECK(encs[b] && encs[b]->e, "align: null encoder output");
      it.e = encs[b]->e;
      it.index = items_in[b];
      if (it.e->owner != m) throw Error("align: the encoder output belongs to another model", true);
      if (it.index < 0 || it.index >= it.e->B) throw Error("align: batch index out of range", true);
      it.n_text = text_offsets[b + 1] - text_offsets[b];
      it.nf = align_frames(num_frames[b]);
      if (it.n_text == 0) continue;
      it.text = text_tokens + text_offsets[b];
      it.probs = text_token_probs_out + text_offsets[b];
      check_align_sequence(m->cfg, start_sequence, n_start, it.text, it.n_text);
      need += it.n_text + 1 + it.nf;  // the longest path through (n_text + 1) x nf cells
    }
    if (need > capacity_pairs) throw Error("align: alignment buffer too small: it needs sum(n_text + 1 + nf) pairs", true);
    B2W_CHECK(need == 0 || alignments_out, "bad arguments");
    if (need > 0) align_run(m, start_sequence, n_start, items, median_filter_width);
    pair_offsets_out[0] = 0;
    for (int b = 0; b < B; ++b) {
      const std::vector<int2>& p = items[b].pairs;
      for (size_t i = 0; i < p.size(); ++i) {
        alignments_out[2 * ((size_t)pair_offsets_out[b] + i)] = p[i].x;
        alignments_out[2 * ((size_t)pair_offsets_out[b] + i) + 1] = p[i].y;
      }
      pair_offsets_out[b + 1] = pair_offsets_out[b] + (int32_t)p.size();
    }
  });
}

int b2w_align_batch(b2w_model* h, b2w_encoded* enc, const int32_t* start_sequence, int32_t n_start, const int32_t* text_tokens,
                    const int32_t* text_offsets, const int32_t* num_frames, int32_t median_filter_width, int32_t* alignments_out,
                    int32_t capacity_pairs, int32_t* pair_offsets_out, float* text_token_probs_out) {
  if (!enc || !enc->e) return guarded([] { B2W_CHECK(false, "bad arguments"); });
  const std::vector<const b2w_encoded*> encs(enc->e->B, enc);
  std::vector<int32_t> items(enc->e->B);
  for (int b = 0; b < enc->e->B; ++b) items[b] = b;
  return b2w_align_items(h, encs.data(), items.data(), enc->e->B, start_sequence, n_start, text_tokens, text_offsets, num_frames,
                         median_filter_width, alignments_out, capacity_pairs, pair_offsets_out, text_token_probs_out);
}

int b2w_encoded_split(b2w_model* h, const b2w_encoded* enc, b2w_encoded** outs) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(enc && enc->e && outs, "bad arguments");
    Encoded* e = enc->e;
    B2W_CHECK(e->owner == m, "the encoder output belongs to another model");
    ensure_cross_kv(m, e);
    const int B = e->B, rows = 2 * m->cfg.n_text_layer;
    const size_t enc_item = e->enc_bytes / B, seg = e->xkv_bytes / ((size_t)rows * B);  // one (layer, K|V) slice of one item
    int max_pitch = 0;
    B2W_CUDA(cudaDeviceGetAttribute(&max_pitch, cudaDevAttrMaxPitch, m->device));
    std::vector<std::unique_ptr<Encoded>> parts(B);
    for (int b = 0; b < B; ++b) {
      Encoded* p = new Encoded;
      parts[b].reset(p);
      p->owner = m;
      p->B = 1;
      p->enc_bytes = enc_item;
      p->enc_out = encoded_alloc(m, enc_item);
      p->xkv_bytes = seg * rows;
      p->xkv = encoded_alloc(m, p->xkv_bytes);
      const char* src = reinterpret_cast<const char*>(e->xkv) + b * seg;
      B2W_CUDA(cudaMemcpyAsync(p->enc_out, reinterpret_cast<const char*>(e->enc_out) + b * enc_item, enc_item,
                               cudaMemcpyDeviceToDevice, m->stream));
      if (seg * B <= (size_t)max_pitch) {
        B2W_CUDA(cudaMemcpy2DAsync(p->xkv, seg, src, seg * B, seg, rows, cudaMemcpyDeviceToDevice, m->stream));
      } else {
        for (int r = 0; r < rows; ++r)
          B2W_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(p->xkv) + r * seg, src + r * seg * B, seg, cudaMemcpyDeviceToDevice,
                                   m->stream));
      }
    }
    for (int b = 0; b < B; ++b) outs[b] = new b2w_encoded{parts[b].release()};
  });
}

int b2w_memory_get(b2w_model* h, int64_t* encoded_bytes, int64_t* pool_bytes) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(encoded_bytes && pool_bytes, "null argument");
    *encoded_bytes = (int64_t)m->encoded_bytes;
    *pool_bytes = (int64_t)m->pool_bytes;
  });
}

int b2w_span_begin(b2w_model* h) {
  return guarded(h, [&](Model* m) {
    if (!m->span_a) {
      B2W_CUDA(cudaEventCreate(&m->span_a));
      B2W_CUDA(cudaEventCreate(&m->span_b));
    }
    B2W_CUDA(cudaEventRecord(m->span_a, m->stream));
  });
}
int b2w_span_end(b2w_model* h, double* ms_out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(ms_out && m->span_a, "b2w_span_end without b2w_span_begin");
    B2W_CUDA(cudaEventRecord(m->span_b, m->stream));
    B2W_CUDA(cudaEventSynchronize(m->span_b));
    float ms = 0.f;
    B2W_CUDA(cudaEventElapsedTime(&ms, m->span_a, m->span_b));
    *ms_out = ms;
  });
}

int b2w_timing_enable(b2w_model* h, int32_t on) {
  return guarded(h, [&](Model* m) {
    drain_timers(m);
    m->timing = on != 0;
  });
}
int b2w_timing_reset(b2w_model* h) {
  return guarded(h, [&](Model* m) {
    drain_timers(m);
    for (int i = 0; i < B2W_T_COUNT; ++i) {
      m->t_ms[i] = 0;
      m->t_cnt[i] = 0;
    }
    m->launches = 0;
    m->decode_steps = 0;
    m->decode_alg_bytes = 0;
  });
}
int b2w_timing_get(b2w_model* h, double ms_out[B2W_T_COUNT], int64_t counts_out[B2W_T_COUNT]) {
  return guarded(h, [&](Model* m) {
    drain_timers(m);
    for (int i = 0; i < B2W_T_COUNT; ++i) {
      ms_out[i] = m->t_ms[i];
      if (counts_out) counts_out[i] = m->t_cnt[i];
    }
  });
}
int b2w_counters_get(b2w_model* h, int64_t* launches, int64_t* decode_steps, double* decode_alg_bytes) {
  return guarded(h, [&](Model* m) {
    if (launches) *launches = m->launches;
    if (decode_steps) *decode_steps = m->decode_steps;
    if (decode_alg_bytes) *decode_alg_bytes = m->decode_alg_bytes;
  });
}

// ---- test hooks -------------------------------------------------------------------------------------------------------
int b2w_debug_gemm(int32_t device, int32_t impl, b2w_gemm_desc* d) {
  return guarded([&] {
    B2W_CHECK(d && d->a && d->w && d->out, "null argument");
    B2W_CHECK(impl == 0 || impl == 1, "impl is 0 (wgmma) or 1 (SIMT reference)");
    B2W_CHECK(d->taps >= 1 && d->taps <= 3, "1..3 taps");
    B2W_CHECK(d->k_per_tap > 0 && d->k_per_tap % 64 == 0, "K per tap must be a multiple of 64");
    B2W_CHECK(d->N > 0 && d->N % 32 == 0, "N must be a multiple of 32");
    B2W_CHECK(d->a_batch >= 1 && d->a_rows >= 1 && d->a_cols >= 1 && d->rows >= 1, "empty GEMM");
    B2W_CHECK(d->a_row_stride >= d->a_cols && d->a_row_stride % 8 == 0 && (d->a_batch == 1 || d->a_batch_stride % 8 == 0),
              "A strides must be 16-byte multiples");
    B2W_CHECK((d->a_batch - 1) * d->a_batch_stride + (d->a_rows - 1) * d->a_row_stride + d->a_cols <= d->a_elems,
              "A exceeds its buffer");
    for (int t = 0; t < d->taps; ++t) B2W_CHECK(d->tap_col[t] >= 0, "tap columns must be >= 0");
    const int epi = d->epilogue;
    B2W_CHECK(epi >= EPI_F16 && epi <= EPI_QKV_CACHE, "unknown epilogue");
    const bool f16_out = epi == EPI_F16 || epi == EPI_GELU_F16 || epi == EPI_F16_XKV || epi == EPI_QKV_CACHE;
    if (epi == EPI_F16_XKV) {
      B2W_CHECK(d->xkv_heads >= 1 && d->xkv_d == 64 * d->xkv_heads && d->N % (2 * d->xkv_d) == 0,
                "XKV: d = 64 x heads and N = layers x 2d");
      B2W_CHECK(d->xkv_B == d->a_batch && d->xkv_T >= d->rows, "XKV: one output chunk per batch item and T >= rows");
      B2W_CHECK((int64_t)d->N * d->xkv_B * d->xkv_T <= d->out_elems, "XKV output exceeds its buffer");
    } else if (epi == EPI_QKV_CACHE) {
      B2W_CHECK(d->a_batch == 1 && d->qkv_d > 0 && d->qkv_d % 32 == 0 && d->N == 3 * d->qkv_d, "QKV: one batch item and N = 3d");
      B2W_CHECK((int64_t)d->rows * d->qkv_d <= d->out_elems, "q output exceeds its buffer");
      B2W_CHECK(d->kcache && d->vcache, "QKV: both caches");
      check_row_table(d->rowinfo, d->rows, d->n_ctx, d->slots, d->qkv_d, d->cache_elems);
    } else {
      const int vec = f16_out ? 8 : 4;  // 16-byte vector stores
      B2W_CHECK(d->out_ld >= d->N && d->out_ld % vec == 0 && (d->a_batch == 1 || d->out_batch_stride % vec == 0),
                "output strides must be 16-byte multiples");
      B2W_CHECK((d->a_batch - 1) * d->out_batch_stride + (int64_t)(d->rows - 1) * d->out_ld + d->N <= d->out_elems,
                "output exceeds its buffer");
      B2W_CHECK(epi != EPI_GELU_POS_F32 || d->pos, "GELU_POS needs pos");
    }
    require_hopper(device);
    DeviceGuard g(device);
    ScratchBufs hb;
    const int64_t K = (int64_t)d->taps * d->k_per_tap;
    const size_t out_bytes = (size_t)d->out_elems * (f16_out ? 2 : 4);
    GemmArgs ga;
    ga.A = hb.put<__half>(d->a, d->a_elems);
    ga.a_batch = d->a_batch; ga.a_rows = d->a_rows; ga.a_cols = d->a_cols;
    ga.a_row_stride = d->a_row_stride; ga.a_batch_stride = d->a_batch_stride;
    ga.taps = d->taps;
    for (int t = 0; t < 3; ++t) {
      ga.tap_row[t] = d->tap_row[t];
      ga.tap_col[t] = d->tap_col[t];
    }
    ga.k_per_tap = d->k_per_tap;
    ga.W = hb.put<__half>(d->w, (size_t)d->N * K);
    ga.N = d->N;
    ga.rows = d->rows;
    ga.bias = d->bias ? hb.put<float>(d->bias, d->N) : nullptr;
    ga.out = hb.put<uint8_t>(d->out, out_bytes);
    ga.out_ld = d->out_ld;
    ga.out_batch_stride = d->out_batch_stride;
    if (epi == EPI_RESID_F32) ga.resid = reinterpret_cast<const float*>(ga.out);
    if (epi == EPI_GELU_POS_F32) ga.pos = hb.put<float>(d->pos, (size_t)d->rows * d->N);
    ga.xkv_d = d->xkv_d; ga.xkv_heads = d->xkv_heads; ga.xkv_T = d->xkv_T; ga.xkv_B = d->xkv_B;
    if (epi == EPI_QKV_CACHE) {
      ga.rowinfo = reinterpret_cast<const int4*>(hb.put<int32_t>(d->rowinfo, (size_t)4 * d->rows));
      ga.kcache = hb.put<__half>(d->kcache, d->cache_elems);
      ga.vcache = hb.put<__half>(d->vcache, d->cache_elems);
      ga.qkv_d = d->qkv_d; ga.n_ctx = d->n_ctx; ga.slots = d->slots;
    }
    ga.epilogue = epi;
    ga.narrow_tiles = d->narrow_tiles != 0;
    d->block_n_out = d->grid_out = 0;
    if (impl == 0) {
      gemm_configure();  // per-device kernel attributes (build_model does this for real models)
      cudaDeviceProp prop;
      B2W_CUDA(cudaGetDeviceProperties(&prop, device));
      GemmPlan p = gemm_plan(ga, prop.multiProcessorCount);
      // fewer persistent CTAs than the plan's: the same tiles, several per CTA
      if (d->max_ctas > 0) p.grid = std::min(p.grid, (int)d->max_ctas);
      d->block_n_out = p.block_n;
      d->grid_out = p.grid;
      gemm_run(p, 0);
    } else {
      gemm_ref_run(ga, 0);
    }
    B2W_CUDA(cudaDeviceSynchronize());
    hook_get(d->out, ga.out, out_bytes);
    if (epi == EPI_QKV_CACHE) {
      hook_get(d->kcache, ga.kcache, (size_t)d->cache_elems * 2);
      hook_get(d->vcache, ga.vcache, (size_t)d->cache_elems * 2);
    }
  });
}

int b2w_debug_gemm_fp8(int32_t device, const uint8_t* a, const float* a_scale, int32_t rows, int32_t K, const uint8_t* w,
                       const float* w_scale, int32_t N, const float* bias, int32_t epilogue, void* out, int32_t max_ctas) {
  return guarded([&] {
    B2W_CHECK(a && a_scale && w && w_scale && out, "null argument");
    B2W_CHECK(rows >= 1 && K > 0 && K % 64 == 0, "fp8 GEMM K must be a multiple of 64");
    B2W_CHECK(N > 0 && N % 32 == 0, "fp8 GEMM N must be a multiple of 32");
    B2W_CHECK(epilogue == EPI_F16 || epilogue == EPI_GELU_F16 || epilogue == EPI_RESID_F32,
              "fp8 GEMM epilogue is F16, GELU_F16 or RESID_F32");
    require_hopper(device);
    DeviceGuard g(device);
    ScratchBufs hb;
    const size_t out_bytes = (size_t)rows * N * (epilogue == EPI_RESID_F32 ? 4 : 2);
    Fp8GemmArgs ga;
    ga.A = hb.put<uint8_t>(a, (size_t)rows * K);
    ga.a_scale = hb.put<float>(a_scale, rows);
    ga.W = hb.put<uint8_t>(w, (size_t)N * K);
    ga.w_scale = hb.put<float>(w_scale, N);
    ga.rows = rows;
    ga.K = K;
    ga.N = N;
    ga.bias = bias ? hb.put<float>(bias, N) : nullptr;
    ga.out = hb.put<uint8_t>(out, out_bytes);
    ga.epilogue = epilogue;
    gemm_configure();
    cudaDeviceProp prop;
    B2W_CUDA(cudaGetDeviceProperties(&prop, device));
    Fp8GemmPlan p = gemm_fp8_plan(ga, prop.multiProcessorCount);
    if (max_ctas > 0) p.grid = std::min(p.grid, (int)max_ctas);
    gemm_fp8_run(p, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    hook_get(out, ga.out, out_bytes);
  });
}

int b2w_debug_quantize_e4m3(int32_t device, const uint16_t* x, int32_t rows, int32_t K, uint8_t* codes, float* scales) {
  return guarded([&] {
    B2W_CHECK(x && codes && scales, "null argument");
    B2W_CHECK(rows >= 1 && K > 0 && K % 8 == 0, "K must be a positive multiple of 8");
    require_hopper(device);
    DeviceGuard g(device);
    ScratchBufs hb;
    const __half* dx = hb.put<__half>(x, (size_t)rows * K);
    uint8_t* dq = hb.alloc<uint8_t>((size_t)rows * K);
    float* ds = hb.alloc<float>(rows);
    quantize_rows_e4m3(dx, dq, ds, rows, K, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    hook_get(codes, dq, (size_t)rows * K);
    hook_get(scales, ds, (size_t)rows * 4);
  });
}

int b2w_debug_layernorm_e4m3(int32_t device, const float* x, const float* gamma, const float* beta, int32_t rows, int32_t d,
                             uint8_t* codes, float* scales) {
  return guarded([&] {
    B2W_CHECK(x && codes && scales, "null argument");
    B2W_CHECK((gamma == nullptr) == (beta == nullptr), "LayerNorm gamma and beta come together");
    B2W_CHECK(rows >= 1 && d > 0 && d % 4 == 0 && d <= 1280, "d must be a multiple of 4 up to 1280");
    require_hopper(device);
    DeviceGuard g(device);
    ScratchBufs hb;
    const float* dx = hb.put<float>(x, (size_t)rows * d);
    const float* dg = gamma ? hb.put<float>(gamma, d) : nullptr;
    const float* db = beta ? hb.put<float>(beta, d) : nullptr;
    uint8_t* dq = hb.alloc<uint8_t>((size_t)rows * d);
    float* ds = hb.alloc<float>(rows);
    layernorm_f32_e4m3(dx, dg, db, dq, ds, rows, d, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    hook_get(codes, dq, (size_t)rows * d);
    hook_get(scales, ds, (size_t)rows * 4);
  });
}

int b2w_debug_attention(int32_t device, int32_t impl, const float* qkv, int32_t B, int32_t T, int32_t H, float* out) {
  return guarded([&] {
    require_hopper(device);
    DeviceGuard g(device);
    const size_t n_in = (size_t)B * T * 3 * H * 64, n_out = (size_t)B * T * H * 64;
    ScratchBufs sb;
    float *dq = sb.alloc<float>(n_in), *dof = sb.alloc<float>(n_out);
    __half *hq = sb.alloc<__half>(n_in), *ho = sb.alloc<__half>(n_out);
    B2W_CUDA(cudaMemcpy(dq, qkv, n_in * 4, cudaMemcpyHostToDevice));
    convert_f32_f16(dq, hq, n_in, 0);
    if (impl == 0) {
      AttnPlan p = attn_plan(hq, ho, B, T, H);
      attn_run(p, 0);
    } else {
      attn_ref_run(hq, ho, B, T, H, 0);
    }
    convert_f16_f32(ho, dof, n_out, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    B2W_CUDA(cudaMemcpy(out, dof, n_out * 4, cudaMemcpyDeviceToHost));
  });
}

int b2w_debug_gemv(int32_t device, int32_t impl, b2w_gemv_desc* d) {
  return guarded([&] {
    B2W_CHECK(d && d->x && d->w, "null argument");
    B2W_CHECK(d->mode >= GV_QKV && d->mode <= GV_F32, "unknown mode");
    B2W_CHECK(impl == 0 || (impl == 1 && d->mode == GV_F32 && d->ldo == d->N), "impl 1 (reference) computes mode F32 with ldo = N");
    B2W_CHECK(d->route == 0 || d->route == 1, "route is 0 (skinny kernel) or 1 (the decoder's choice)");
    B2W_CHECK(d->R >= 1 && d->R <= kMaxRows, "1..80 rows");
    B2W_CHECK(d->N >= 1 && d->K >= 32 && d->K % 32 == 0, "K must be a multiple of 32");
    const int R = d->R, N = d->N, K = d->K;
    switch (d->mode) {
      case GV_QKV:
        B2W_CHECK(d->d > 0 && d->d % 32 == 0 && N == 3 * d->d, "QKV: N = 3d");
        B2W_CHECK(d->out && (int64_t)R * d->d <= d->out_elems, "q output exceeds its buffer");
        B2W_CHECK(d->kcache && d->vcache, "QKV: both caches");
        check_row_table(d->rows, R, d->n_ctx, d->slots, d->d, d->cache_elems);
        break;
      case GV_F16:
      case GV_GELU_F16: B2W_CHECK(d->out && (int64_t)R * N <= d->out_elems, "output exceeds its buffer"); break;
      case GV_RESID_LN:
        B2W_CHECK(d->xres && d->xn && N % 4 == 0 && N <= 1280, "RESID_LN: xres and xn, N a multiple of 4 up to 1280");
        B2W_CHECK((d->ln_g == nullptr) == (d->ln_b == nullptr), "LayerNorm gamma and beta come together");
        break;
      case GV_F32:
        B2W_CHECK(d->out && d->ldo >= N && d->ldo % 4 == 0 && (int64_t)(R - 1) * d->ldo + N <= d->out_elems, "output exceeds its buffer");
        break;
    }
    require_hopper(device);
    DeviceGuard g(device);
    ScratchBufs hb;
    // zero-padded like the decoder's workspaces: the skinny kernel reads activations in 8-row groups up to kMaxRows rows and
    // weights in 16-row groups
    const int Np = ceil_div(N, 16) * 16;
    const size_t out_bytes = d->out ? (size_t)d->out_elems * (d->mode == GV_F32 ? 4 : 2) : 0;
    GvArgs a;
    a.x = hb.put<__half>(d->x, (size_t)R * K, (size_t)kMaxRows * K);
    a.W = hb.put<__half>(d->w, (size_t)N * K, (size_t)Np * K);
    a.bias = d->bias ? hb.put<float>(d->bias, N) : nullptr;
    a.R = R; a.N = N; a.K = K; a.mode = d->mode;
    void* out = d->out ? hb.put<uint8_t>(d->out, out_bytes) : nullptr;
    a.out_h = reinterpret_cast<__half*>(out);
    a.out_f = reinterpret_cast<float*>(out);
    a.ldo = d->ldo;
    if (d->mode == GV_QKV) {
      a.rows = reinterpret_cast<const RowInfo*>(hb.put<int32_t>(d->rows, (size_t)4 * R));
      a.kcache = hb.put<__half>(d->kcache, d->cache_elems);
      a.vcache = hb.put<__half>(d->vcache, d->cache_elems);
      a.d = d->d; a.n_ctx = d->n_ctx; a.slots = d->slots;
    }
    if (d->mode == GV_RESID_LN) {
      a.xres = hb.put<float>(d->xres, (size_t)R * N);
      a.ln_g = d->ln_g ? hb.put<float>(d->ln_g, N) : nullptr;
      a.ln_b = d->ln_b ? hb.put<float>(d->ln_b, N) : nullptr;
      a.xn_out = hb.put<__half>(d->xn, (size_t)R * N);
      a.counter = hb.put<int>(nullptr, 1);
    }
    d->path_out = 0;
    if (impl == 1) {
      skinny_ref(a.x, a.W, a.bias, a.out_f, R, N, K, 0);
    } else if (d->route == 1 && gv_uses_wgmma(a)) {
      // what gv() runs, with a plan built here rather than cached in a model
      gemm_configure();
      cudaDeviceProp prop;
      B2W_CUDA(cudaGetDeviceProperties(&prop, device));
      gv_wgmma(gemm_plan(gv_gemm_args(a), prop.multiProcessorCount), a, 0);
      d->path_out = 1;
    } else {
      skinny_gemm(a, 0);
    }
    B2W_CUDA(cudaDeviceSynchronize());
    hook_get(d->out, out, out_bytes);
    if (d->mode == GV_QKV) {
      hook_get(d->kcache, a.kcache, (size_t)d->cache_elems * 2);
      hook_get(d->vcache, a.vcache, (size_t)d->cache_elems * 2);
    }
    if (d->mode == GV_RESID_LN) {
      hook_get(d->xres, a.xres, (size_t)R * N * 4);
      hook_get(d->xn, a.xn_out, (size_t)R * N * 2);
    }
  });
}

int b2w_debug_align_cost(int32_t device, const float* capture, int32_t n_heads, int32_t n_tok, int32_t nf, int32_t n_start,
                         int32_t n_text, int32_t median_filter_width, double* cost_out) {
  return guarded([&] {
    B2W_CHECK(capture && cost_out, "null argument");
    B2W_CHECK(n_heads >= 1 && n_heads <= 32 * 32, "n_heads must be in 1..1024");
    B2W_CHECK(nf >= 1 && nf <= 1500, "nf must be in 1..1500");
    B2W_CHECK(n_tok >= 1 && n_tok <= B2W_MAX_TEXT_CTX, "n_tok must be in 1..448");
    B2W_CHECK(n_start >= 0 && n_text >= 0 && n_start + n_text + 1 <= n_tok, "the kept rows n_start .. n_start + n_text must be tokens");
    if (median_filter_width < 1 || median_filter_width % 2 == 0) throw Error("align: median_filter_width must be odd", true);
    const AlignBatch shape{nullptr, nullptr, nullptr, nullptr, n_heads, n_tok, nf, n_text + 1, median_filter_width, nullptr, nullptr};
    align_check(shape);
    require_hopper(device);
    DeviceGuard g(device);
    const size_t n_cap = (size_t)n_heads * n_tok * nf, n_cost = (size_t)(n_text + 1) * nf;
    const int4 item = make_int4(n_tok, nf, n_start, n_text + 1);
    ScratchBufs sb;
    AlignBatch a = shape;
    a.cap = sb.put<float>(capture, n_cap);
    a.stats = sb.alloc<double>((size_t)n_heads * 2 * nf);
    a.cost = sb.alloc<double>(n_cost);
    a.items = sb.put<int4>(&item, 1);
    align_cost(a, 1, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    B2W_CUDA(cudaMemcpy(cost_out, a.cost, n_cost * sizeof(double), cudaMemcpyDeviceToHost));
  });
}

int b2w_debug_dtw(int32_t device, const double* cost, int32_t N, int32_t M, int32_t* pairs_out, int32_t capacity_pairs,
                  int32_t* n_pairs_out) {
  return guarded([&] {
    B2W_CHECK(cost && pairs_out && n_pairs_out, "null argument");
    B2W_CHECK(N >= 1 && N <= kAlignMaxRows && M >= 1 && M <= 1500, "cost must be 1..449 rows x 1..1500 frames");
    if (capacity_pairs < N + M) throw Error("align: alignment buffer too small: it needs N + M pairs", true);
    const AlignBatch shape{nullptr, nullptr, nullptr, nullptr, 1, 1, M, N, 1, nullptr, nullptr};
    align_check(shape);
    require_hopper(device);
    DeviceGuard g(device);
    const int4 item = make_int4(N + 1, M, 0, N);
    ScratchBufs sb;
    AlignBatch a = shape;
    a.cost = sb.put<double>(cost, (size_t)N * M);
    a.items = sb.put<int4>(&item, 1);
    a.pairs = sb.alloc<int2>(N + M);
    a.n_pairs = sb.alloc<int>(1);
    align_dtw(a, 1, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    B2W_CUDA(cudaMemcpy(n_pairs_out, a.n_pairs, sizeof(int), cudaMemcpyDeviceToHost));
    B2W_CUDA(cudaMemcpy(pairs_out, a.pairs, (size_t)*n_pairs_out * sizeof(int2), cudaMemcpyDeviceToHost));
  });
}

int b2w_debug_fetch(b2w_model* h, int32_t which, float* out, int64_t n) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(out && n >= 0, "null argument");
    B2W_CHECK(m->d_x, "no decoder workspace yet");
    B2W_CUDA(cudaStreamSynchronize(m->stream));
    const b2w_config& c = m->cfg;
    const int64_t dt = c.n_text_state, L = c.n_text_layer;
    const float* f32 = nullptr;
    const __half* f16 = nullptr;
    int64_t size = 0, rows = 1, pitch = 0;  // the buffer's elements; the caches are copied as L rows of n / L elements, kv_elems apart
    switch (which) {
      case 0: f32 = m->d_x; size = (int64_t)kMaxRows * ceil_div((int)dt, 128) * 128; break;
      case 1: f32 = m->d_gpart; size = (int64_t)m->num_sms * kMaxRows * 128; break;
      case 2: f32 = m->d_stpart; size = dt / 64 * kMaxRows * 2; break;
      case 4: f16 = m->d_ao; size = kMaxRows * dt; break;
      case 5: f16 = m->d_h16; size = kMaxRows * 4 * dt; break;
      case 6: f16 = m->d_xn16; size = kMaxRows * dt; break;
      case 7: f32 = m->d_stats; size = 3 * L * kMaxRows * 2; break;
      case 8: f32 = m->d_logits; size = (int64_t)kMaxRows * m->vpad; break;
      case 9:
      case 10:
        B2W_CHECK(m->kcache, "no self-attention cache yet");
        f16 = which == 9 ? m->kcache : m->vcache;
        B2W_CHECK(n % L == 0, "the caches are fetched as L equal per-layer prefixes");
        size = L * (int64_t)m->kv_elems;
        rows = L;
        pitch = (int64_t)m->kv_elems;
        break;
      case 11:
        B2W_CHECK(m->h_bind.xkv, "no encoder output bound");
        f16 = m->h_bind.xkv;
        size = L * 2 * m->h_bind.B_total * 1500 * dt;
        break;
      default: throw Error("b2w_debug_fetch: unknown buffer", true);
    }
    B2W_CHECK(n / rows <= (pitch ? pitch : size), "n exceeds the buffer");
    if (n == 0) return;
    if (f32) {
      B2W_CUDA(cudaMemcpy(out, f32, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
    } else {
      std::vector<__half> tmp((size_t)n);
      const size_t w = (size_t)(n / rows) * sizeof(__half);
      B2W_CUDA(cudaMemcpy2D(tmp.data(), w, f16, (size_t)(pitch ? pitch : n) * sizeof(__half), w, (size_t)rows, cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < n; ++i) out[i] = __half2float(tmp[(size_t)i]);
    }
  });
}

int b2w_debug_self_attn(int32_t device, const uint16_t* q, const uint16_t* kcache, const uint16_t* vcache, const uint8_t* anc,
                        const int32_t* rows, int32_t R, int32_t H, int32_t n_chunks, int32_t slots, int32_t n_ctx, uint16_t* out) {
  return guarded([&] {
    B2W_CHECK(q && kcache && vcache && anc && rows && out, "null argument");
    B2W_CHECK(R >= 1 && R <= 65535, "R must be in 1..65535");
    B2W_CHECK(H >= 1 && H <= 20, "heads must be in 1..20");
    B2W_CHECK(n_chunks >= 1 && slots >= 1 && slots <= kMaxBeam, "n_chunks >= 1 and slots in 1..16");
    B2W_CHECK(n_ctx >= 1 && n_ctx <= B2W_MAX_TEXT_CTX, "n_ctx must be in 1..448");
    const int d = 64 * H;
    const size_t n_anc = (size_t)2 * n_chunks * slots * n_ctx, cache = (size_t)n_chunks * n_ctx * slots * d;
    for (int r = 0; r < R; ++r)
      B2W_CHECK(rows[4 * r] >= 0 && rows[4 * r] < n_chunks && rows[4 * r + 1] >= 0 && rows[4 * r + 1] < slots && rows[4 * r + 2] >= 0 &&
                    rows[4 * r + 2] < n_ctx,
                "row table entry outside the cache");
    for (size_t i = 0; i < n_anc; ++i) B2W_CHECK(anc[i] < slots, "ancestry slot out of range");
    require_hopper(device);
    DeviceGuard g(device);
    ScratchBufs sb;
    SelfAttnArgs a;
    a.rows = reinterpret_cast<const RowInfo*>(sb.put<int32_t>(rows, (size_t)4 * R));
    a.q = sb.put<__half>(q, (size_t)R * d);
    a.kcache = sb.put<__half>(kcache, cache);
    a.vcache = sb.put<__half>(vcache, cache);
    a.anc = sb.put<uint8_t>(anc, n_anc);
    __half* o = sb.alloc<__half>((size_t)R * d);
    a.out = o;
    a.d = d; a.n_ctx = n_ctx; a.slots = slots;
    a.anc_buf_stride = (long long)n_chunks * slots * n_ctx;
    dec_self_attn(a, R, H, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    hook_get(out, o, (size_t)R * d * 2);
  });
}

int b2w_debug_cross_attn(int32_t device, const uint16_t* q, const uint16_t* kv, int32_t n_chunks, int32_t rows_per_chunk, int32_t H,
                         uint16_t* out) {
  return guarded([&] {
    B2W_CHECK(q && kv && out, "null argument");
    B2W_CHECK(n_chunks >= 1 && n_chunks <= 16, "n_chunks must be in 1..16");
    B2W_CHECK(rows_per_chunk >= 1 && rows_per_chunk <= kMaxBeam, "rows_per_chunk must be in 1..16");
    B2W_CHECK(H >= 1 && H <= 20, "heads must be in 1..20");
    require_hopper(device);
    DeviceGuard g(device);
    dstep_configure();  // per-device kernel attributes (build_model does this for real models)
    const int d = 64 * H, R = n_chunks * rows_per_chunk, T = 1500;
    const size_t groups = (size_t)n_chunks * H * ds_xqgroups(rows_per_chunk);
    ScratchBufs sb;
    const __half* xkv = sb.put<__half>(kv, (size_t)2 * n_chunks * H * T * 64);
    std::vector<DecBindings> bind(n_chunks);
    for (int b = 0; b < n_chunks; ++b) bind[b] = DecBindings{xkv, n_chunks, b};
    DStepArgs a{};
    a.q = sb.put<__half>(q, (size_t)R * d);
    __half* o = sb.alloc<__half>((size_t)R * d);
    a.ao = o;
    a.bind = sb.put<DecBindings>(bind.data(), bind.size());
    a.xpart = sb.alloc<float>(groups * kDsXSplits * kDsXQ * 66);
    a.xcounters = sb.put<int>(nullptr, 0, groups);
    a.H = H; a.T = T; a.d = d; a.rows_per_chunk = rows_per_chunk; a.n_chunks = n_chunks;
    dstep_cross_attn_launch(a, 0, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    hook_get(out, o, (size_t)R * d * 2);
  });
}

int b2w_debug_logits(b2w_model* h, b2w_encoded* enc, const int32_t* tokens, int32_t n_tok, int32_t batch, float* logits_out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(enc && enc->e && tokens && logits_out && enc->e->B == batch, "bad arguments");
    B2W_CHECK(n_tok >= 1 && n_tok <= m->cfg.n_text_ctx, "token count");
    for (size_t i = 0; i < (size_t)batch * n_tok; ++i) B2W_CHECK(tokens[i] >= 0 && tokens[i] < m->cfg.n_vocab, "token id out of range");
    Encoded* e = enc->e;
    const int V = m->cfg.n_vocab;
    const int group = std::min((int)batch, kMaxRows);
    prepare_decode(m, e, group, 1);
    std::vector<float> tmp((size_t)kMaxRows * m->vpad);
    for (int c0 = 0; c0 < batch; c0 += group) {
      const int n = std::min(group, batch - c0);
      forced_decode(m, forced_range(e, c0, n), tokens + (size_t)c0 * n_tok, n_tok, n_tok, 1, true, nullptr, [&](int i0, int i1) {
        const int rpc = i1 - i0;
        logits_gemm(m, n * rpc);
        B2W_CUDA(cudaMemcpyAsync(tmp.data(), m->d_logits, (size_t)n * rpc * m->vpad * 4, cudaMemcpyDeviceToHost, m->stream));
        B2W_CUDA(cudaStreamSynchronize(m->stream));
        for (int b = 0; b < n; ++b)
          for (int i = i0; i < i1; ++i)
            memcpy(logits_out + ((size_t)(c0 + b) * n_tok + i) * V, tmp.data() + (size_t)(b * rpc + i - i0) * m->vpad, (size_t)V * 4);
      });
    }
  });
}

int b2w_debug_step_logits(b2w_model* h, b2w_encoded* enc, const int32_t* prompts, int32_t P, int32_t n, int32_t K, int32_t n_steps,
                          const int32_t* tokens, const int32_t* parents, float* logits_out) {
  return guarded(h, [&](Model* m) {
    B2W_CHECK(enc && enc->e && prompts && tokens && logits_out, "null argument");
    const b2w_config& c = m->cfg;
    B2W_CHECK(enc->e->B == n, "one prompt per encoder output row is required");
    B2W_CHECK(K >= 1 && K <= kMaxBeam, "rows per chunk must be in 1..16");
    B2W_CHECK(n >= 1 && (int64_t)n * K <= kMaxRows, "chunks x rows per chunk must be in 1..80");
    const int R = n * K, V = c.n_vocab, n_ctx = c.n_text_ctx;
    B2W_CHECK(P >= 1 && n_steps >= 1 && P - 1 + n_steps <= n_ctx, "prompt length + steps exceed the text context");
    for (size_t i = 0; i < (size_t)n * P; ++i) B2W_CHECK(prompts[i] >= 0 && prompts[i] < V, "prompt token id out of range");
    for (size_t i = 0; i < (size_t)n_steps * R; ++i) B2W_CHECK(tokens[i] >= 0 && tokens[i] < V, "token id out of range");
    if (parents)
      for (size_t i = 0; i < (size_t)n_steps * R; ++i) B2W_CHECK(parents[i] >= 0 && parents[i] < K, "parent slot out of range");
    Step st = choose_step(m, n, K, false);
    Encoded* e = enc->e;
    prepare_decode(m, e, n, K);
    cudaStream_t s = m->stream;
    const SearchBuffers& sb = m->sb;
    forced_decode(m, forced_range(e, 0, n), prompts, P, P - 1, K, true, nullptr, [](int, int) {});  // the prompt's keys, as prefill writes them
    b2w_gen_opts o;
    b2w_gen_opts_default(&o);
    o.beam_size = K;
    o.max_length = P + n_steps;
    bind_step(m, st, e, 0, prompts, P, search_params(c, m->vpad, n, K, o));
    // anc[r][j]: the slot that holds key j of row r.  Keys of the prompt sit in slot 0; relinked as search_update does.
    std::vector<uint8_t> anc((size_t)R * n_ctx, 0), prev;
    std::vector<RowInfo> rows(R);
    for (int t = 0; t < n_steps; ++t) {
      const int pos = P - 1 + t;
      if (t > 0 && parents) {
        prev = anc;
        for (int r = 0; r < R; ++r) {
          const int p = parents[(size_t)t * R + r], src = (r / K) * K + p;
          memcpy(&anc[(size_t)r * n_ctx], &prev[(size_t)src * n_ctx], pos - 1);
          anc[(size_t)r * n_ctx + pos - 1] = (uint8_t)p;
        }
      } else if (t > 0) {
        for (int r = 0; r < R; ++r) anc[(size_t)r * n_ctx + pos - 1] = (uint8_t)(r % K);
      }
      for (int r = 0; r < R; ++r) rows[r] = RowInfo{r / K, r % K, pos, 0};
      B2W_CUDA(cudaMemcpyAsync(sb.rows, rows.data(), R * sizeof(RowInfo), cudaMemcpyHostToDevice, s));
      B2W_CUDA(cudaMemcpyAsync(sb.tokens_in, tokens + (size_t)t * R, R * sizeof(int32_t), cudaMemcpyHostToDevice, s));
      B2W_CUDA(cudaMemcpyAsync(sb.anc + (size_t)(pos & 1) * R * n_ctx, anc.data(), anc.size(), cudaMemcpyHostToDevice, s));
      launch_decoder(m, st);
      B2W_CUDA(cudaMemcpy2DAsync(logits_out + (size_t)t * R * V, (size_t)V * 4, m->d_logits, (size_t)m->vpad * 4, (size_t)V * 4, R,
                                 cudaMemcpyDeviceToHost, s));
      B2W_CUDA(cudaStreamSynchronize(s));  // rows / anc are rewritten for the next step
    }
  });
}

static_assert(B2W_MAX_FINISHED == kMaxFinished, "public finished-slot count");

int b2w_debug_search(int32_t device, b2w_search_desc* d) {
  return guarded([&] {
    B2W_CHECK(d && d->cfg && d->opts && d->prompt && d->logits && d->hist && d->anc && d->cum && d->done && d->fin_count &&
                  d->fin_len && d->fin_score && d->fin_tok && d->cand_score && d->cand_tok && d->no_speech && d->tokens_in && d->pos,
              "null argument");
    const b2w_config& c = *d->cfg;
    const b2w_gen_opts& o = *d->opts;
    const int V = c.n_vocab, n_ctx = c.n_text_ctx, vpad = ceil_div(std::max(V, 1), 16) * 16;
    B2W_CHECK(V >= 1 && vpad * (int)sizeof(float) <= 210 * 1024, "n_vocab must fit the in-shared-memory row search");
    B2W_CHECK(n_ctx >= 1 && n_ctx <= B2W_MAX_TEXT_CTX, "n_text_ctx must be in 1..448");
    for (int tok : {c.eot, c.sot, c.no_speech, c.no_timestamps, c.timestamp_begin})
      B2W_CHECK(tok >= 0 && tok < V, "control token id out of range");
    B2W_CHECK(c.n_suppress_begin >= 0 && c.n_suppress_begin <= 8, "n_suppress_begin must be in 0..8");
    for (int i = 0; i < c.n_suppress_begin; ++i) B2W_CHECK(c.suppress_begin[i] >= 0 && c.suppress_begin[i] < V, "suppress_begin id out of range");
    const int K = check_gen_opts(c, o);
    B2W_CHECK(d->K == K, "K must be beam_size, or num_hypotheses when beam_size is 1");
    B2W_CHECK(o.n_suppress_tokens >= 0 && (o.n_suppress_tokens == 0 || o.suppress_tokens), "suppress_tokens");
    const int n = d->n, P = d->P, t = d->t, R = n * K;
    B2W_CHECK(n >= 1 && (int64_t)n * K <= kMaxRows, "chunks x rows per chunk must be in 1..80");
    B2W_CHECK(P >= 1 && P <= n_ctx, "prompt length");
    const int sot_index = validate_prompts(c, d->prompt, 1, P);
    B2W_CHECK(t >= 0 && t < o.max_length - P, "step must be one a generate call with max_length runs");
    const SearchParams sp = search_params(c, vpad, n, K, o);
    std::vector<ChunkParams> cps(n);
    for (int b = 0; b < n; ++b) cps[b] = chunk_params(c, d->prompt, P, sot_index, o.max_length, b, o.return_no_speech_prob);
    const bool beam = sp.mode == 0;
    for (size_t i = 0; i < (size_t)R * t; ++i) B2W_CHECK(d->hist[i] >= 0 && d->hist[i] < V, "history token id out of range");
    for (size_t i = 0; i < (size_t)R * (P - 1 + t); ++i) B2W_CHECK(d->anc[i] < K, "ancestry slot out of range");
    for (int b = 0; b < n; ++b) {
      B2W_CHECK(d->done[b] == 0 || d->done[b] == 1, "done is 0 or 1");
      B2W_CHECK(d->fin_count[b] >= 0 && d->fin_count[b] <= kMaxFinished, "fin_count out of range");
      // a live beam chunk has room for the K hypotheses the step can finish, as in every state a generate call reaches unless
      // early exit (patience 1, length penalty 0) lets hypotheses pile up behind a live best one
      B2W_CHECK(!beam || d->done[b] || d->fin_count[b] + K <= kMaxFinished, "a live chunk needs K free finished slots");
    }
    for (size_t i = 0; i < (size_t)n * kMaxFinished; ++i) B2W_CHECK(d->fin_len[i] >= -1 && d->fin_len[i] <= n_ctx, "fin_len out of range");
    B2W_CHECK(d->n_done >= 0 && d->n_done <= n, "n_done must be in 0..n");
    require_hopper(device);
    DeviceGuard g(device);
    search_configure();  // per-device kernel attributes (build_model does this for real models)
    ScratchBufs hb;
    const int pos = P - 1 + t, cur = pos & 1, nxt = cur ^ 1;
    const int ncand = sp.ncand;
    SearchBuffers sb;
    SearchState state{t, d->n_done, cur, 0};
    sb.state = hb.put<SearchState>(&state, 1);
    sb.params = hb.put<SearchParams>(&sp, 1);
    sb.chunk = hb.put<ChunkParams>(cps.data(), n);
    std::vector<RowInfo> rows(R);
    for (int r = 0; r < R; ++r) rows[r] = RowInfo{r / K, r % K, pos, 0};
    sb.rows = hb.put<RowInfo>(rows.data(), R);
    sb.tokens_in = hb.put<int>(nullptr, 0, R);
    std::vector<float> cum(2 * (size_t)R, 0.f);
    std::copy(d->cum, d->cum + R, cum.begin() + (size_t)cur * R);
    sb.cum = hb.put<float>(cum.data(), cum.size());
    std::vector<int> hist(2 * (size_t)R * n_ctx, -1);
    std::vector<uint8_t> anc(2 * (size_t)R * n_ctx, 0xFF);
    for (int r = 0; r < R; ++r) {
      std::copy(d->hist + (size_t)r * t, d->hist + (size_t)(r + 1) * t, hist.begin() + ((size_t)cur * R + r) * n_ctx);
      std::copy(d->anc + (size_t)r * pos, d->anc + (size_t)(r + 1) * pos, anc.begin() + ((size_t)cur * R + r) * n_ctx);
    }
    sb.hist = hb.put<int>(hist.data(), hist.size());
    sb.anc = hb.put<uint8_t>(anc.data(), anc.size());
    sb.cand_score = hb.put<float>(nullptr, 0, (size_t)R * kMaxCand);
    sb.cand_tok = hb.put<int>(nullptr, 0, (size_t)R * kMaxCand);
    const std::vector<uint8_t> mask = suppress_mask(c, vpad, o);
    sb.suppress = hb.put<uint8_t>(mask.data(), mask.size());
    sb.done = hb.put<int>(d->done, n);
    sb.fin_count = hb.put<int>(d->fin_count, n);
    sb.fin_score = hb.put<float>(d->fin_score, (size_t)n * kMaxFinished);
    sb.fin_len = hb.put<int>(d->fin_len, (size_t)n * kMaxFinished);
    const std::vector<int> fin_tok((size_t)n * kMaxFinished * n_ctx, -1);
    sb.fin_tok = hb.put<int>(fin_tok.data(), fin_tok.size());
    sb.no_speech = hb.put<float>(nullptr, 0, n);
    sb.row_margin = hb.put<float>(nullptr, 0, R);
    sb.n_ctx = n_ctx;
    // logits at the padded row stride the decoder writes, NaN in the padding so that a read of it shows
    float* logits = hb.alloc<float>((size_t)R * vpad);
    B2W_CUDA(cudaMemset(logits, 0xFF, (size_t)R * vpad * sizeof(float)));
    B2W_CUDA(cudaMemcpy2D(logits, (size_t)vpad * 4, d->logits, (size_t)V * 4, (size_t)V * 4, R, cudaMemcpyHostToDevice));
    search_rows(logits, R, vpad, sb, 0);
    search_update(n, sb, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    B2W_CUDA(cudaMemcpy2D(d->cand_score, (size_t)ncand * 4, sb.cand_score, (size_t)kMaxCand * 4, (size_t)ncand * 4, R, cudaMemcpyDeviceToHost));
    B2W_CUDA(cudaMemcpy2D(d->cand_tok, (size_t)ncand * 4, sb.cand_tok, (size_t)kMaxCand * 4, (size_t)ncand * 4, R, cudaMemcpyDeviceToHost));
    B2W_CUDA(cudaMemcpy2D(d->hist, (size_t)(t + 1) * 4, sb.hist + (size_t)nxt * R * n_ctx, (size_t)n_ctx * 4, (size_t)(t + 1) * 4, R,
                          cudaMemcpyDeviceToHost));
    B2W_CUDA(cudaMemcpy2D(d->anc, (size_t)(pos + 1), sb.anc + (size_t)nxt * R * n_ctx, (size_t)n_ctx, (size_t)(pos + 1), R, cudaMemcpyDeviceToHost));
    hook_get(d->cum, sb.cum + (size_t)nxt * R, (size_t)R * 4);
    hook_get(d->tokens_in, sb.tokens_in, (size_t)R * 4);
    hook_get(rows.data(), sb.rows, (size_t)R * sizeof(RowInfo));
    for (int r = 0; r < R; ++r) d->pos[r] = rows[r].pos;
    hook_get(d->done, sb.done, (size_t)n * 4);
    hook_get(&state, sb.state, sizeof state);
    d->n_done = state.n_done;
    hook_get(d->fin_count, sb.fin_count, (size_t)n * 4);
    hook_get(d->fin_len, sb.fin_len, (size_t)n * kMaxFinished * 4);
    hook_get(d->fin_score, sb.fin_score, (size_t)n * kMaxFinished * 4);
    B2W_CUDA(cudaMemcpy2D(d->fin_tok, (size_t)(t + 1) * 4, sb.fin_tok, (size_t)n_ctx * 4, (size_t)(t + 1) * 4, (size_t)n * kMaxFinished,
                          cudaMemcpyDeviceToHost));
    hook_get(d->no_speech, sb.no_speech, (size_t)n * 4);
  });
}

int b2w_vad_create(int32_t device, const b2w_tensor* tensors, int32_t n_tensors, b2w_vad** out) {
  return guarded([&] {
    B2W_CHECK(tensors && out && n_tensors >= 0, "null argument");
    TensorTable tt{tensors, n_tensors};
    for (const auto& spec : kVadTensors) {
      const b2w_tensor& t = tt.get(spec.name);
      B2W_CHECK(t.data && t.dtype == B2W_F32, "VAD weights must be float32");
      expect_shape(t, spec.shape);
    }
    require_hopper(device);
    DeviceGuard g(device);
    std::unique_ptr<b2w_vad> v(new b2w_vad);
    v->device = device;
    B2W_CUDA(cudaStreamCreateWithFlags(&v->stream, cudaStreamNonBlocking));
    for (cudaEvent_t& e : v->ev) B2W_CUDA(cudaEventCreate(&e));
    vad_configure();
    ScratchBufs& sb = v->weights;
    auto raw = [&](const char* name) { const b2w_tensor& t = tt.get(name); return sb.put<float>(t.data, (size_t)numel(t)); };
    v->w.basis_t = vad_upload_t(sb, tt.get("basis"), 258, 256);
    const int cout[4] = {128, 64, 64, 128}, cin[4] = {129, 128, 64, 64};
    for (int i = 0; i < 4; ++i) {
      const std::string p = "conv" + std::to_string(i);
      v->w.conv_t[i] = vad_upload_t(sb, tt.get(p + ".weight"), cout[i], (int64_t)cin[i] * 3);
      v->w.conv_b[i] = raw((p + ".bias").c_str());
    }
    v->w.w_ih_t = vad_upload_t(sb, tt.get("lstm.w_ih"), 512, 128);
    v->w.b_gates = raw("lstm.bias");
    v->w_hh = raw("lstm.w_hh");
    v->dec_w = raw("decoder.weight");
    v->dec_b = raw("decoder.bias");
    *out = v.release();
  });
}

void b2w_vad_destroy(b2w_vad* v) { delete v; }

int b2w_vad_set_block(b2w_vad* v, int64_t windows) {
  return guarded([&] {
    B2W_CHECK(windows >= 1 && windows <= (1 << 24), "windows per block must be in 1..2^24");
    B2W_CHECK(v, "null VAD handle");
    std::lock_guard<std::mutex> lk(v->mu);
    v->block = windows;
  });
}

// Windows of stream i per launch: the block's windows split evenly over the streams that still have windows left (a launch
// takes as long as its longest slice), what a short stream leaves over going to the longer ones.
static void vad_plan_launch(int64_t block, const std::vector<int64_t>& left, std::vector<int64_t>& take) {
  std::vector<int> order;
  for (int i = 0; i < (int)left.size(); ++i)
    if (left[i] > 0) order.push_back(i);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return left[a] < left[b]; });
  std::fill(take.begin(), take.end(), 0);
  int64_t budget = block;
  for (size_t k = 0; k < order.size(); ++k) {
    const int64_t t = std::min(left[order[k]], budget / (int64_t)(order.size() - k));
    take[order[k]] = t;
    budget -= t;
  }
}

int b2w_vad_probs(b2w_vad* v, const float* pcm, int64_t n_samples, float* probs_out, int64_t capacity) {
  return b2w_vad_probs_multi(v, &pcm, &n_samples, 1, probs_out, capacity);
}

int b2w_vad_probs_multi(b2w_vad* v, const float* const* pcm, const int64_t* n_samples, int32_t n_streams, float* probs_out,
                        int64_t capacity) {
  return guarded([&] {
    B2W_CHECK(pcm && n_samples && probs_out, "null argument");
    B2W_CHECK(n_streams >= 1, "at least one stream");
    int64_t total = 0;
    for (int i = 0; i < n_streams; ++i) {
      B2W_CHECK(pcm[i], "null argument");
      B2W_CHECK(n_samples[i] > 0 && n_samples[i] % 512 == 0, "the number of samples must be a positive multiple of 512");
      total += n_samples[i] / 512;
    }
    B2W_CHECK(capacity >= total, "output buffer too small: one probability per 512 samples");
    B2W_CHECK(v, "null VAD handle");
    std::lock_guard<std::mutex> lk(v->mu);
    DeviceGuard g(v->device);
    cudaStream_t s = v->stream;
    const int S = n_streams;
    std::vector<int64_t> left(S), done(S, 0), out0(S), take(S);  // per stream: windows to go, done, first output, this launch
    for (int64_t i = 0, o = 0; i < S; ++i) {
      left[i] = n_samples[i] / 512;
      out0[i] = o;
      o += left[i];
    }
    const int64_t nb_max = std::min(v->block, total);
    if (v->cap < nb_max || v->cap_streams < S) {
      const int64_t cap = std::max(v->cap, nb_max), cap_streams = std::max<int64_t>(v->cap_streams, S);
      v->bufs.reset();
      v->cap = v->cap_streams = 0;
      std::unique_ptr<ScratchBufs> b(new ScratchBufs);
      v->pcm = b->alloc<float>((size_t)(64 * std::min(cap, cap_streams) + 512 * cap));
      v->gx = b->alloc<float>((size_t)(512 * cap));
      v->H = b->alloc<float>((size_t)(128 * cap));
      v->probs = b->alloc<float>((size_t)cap);
      v->states = b->alloc<float>((size_t)(256 * cap_streams));
      v->slices = b->alloc<VadSlice>((size_t)std::min(cap, cap_streams));
      v->bufs = std::move(b);
      v->cap = cap;
      v->cap_streams = cap_streams;
    }
    v->host_probs.resize((size_t)nb_max);
    for (double& m : v->ms) m = 0;
    for (int64_t remaining = total; remaining > 0;) {
      vad_plan_launch(nb_max, left, take);
      // the launch's table and PCM: per slice the 64 samples before it (left to the kernel at the start of a stream), then its
      // windows
      auto& tab = v->host_slices;
      tab.clear();
      int64_t w = 0, p = 0;
      for (int i = 0; i < S; ++i) {
        if (take[i] == 0) continue;
        VadSlice sl{};
        sl.pcm0 = p;
        sl.w0 = (int32_t)w;
        sl.nb = (int32_t)take[i];
        sl.stream = i;
        sl.first = done[i] == 0;
        sl.last = done[i] + take[i] == n_samples[i] / 512;
        tab.push_back(sl);
        const int64_t n_pcm = 512 * take[i];
        if (sl.first)
          B2W_CUDA(cudaMemcpyAsync(v->pcm + p + 64, pcm[i], (size_t)n_pcm * 4, cudaMemcpyHostToDevice, s));
        else
          B2W_CUDA(cudaMemcpyAsync(v->pcm + p, pcm[i] + done[i] * 512 - 64, (size_t)(64 + n_pcm) * 4, cudaMemcpyHostToDevice, s));
        w += take[i];
        p += 64 + n_pcm;
      }
      const int nb = (int)w, n_slices = (int)tab.size();
      B2W_CUDA(cudaMemcpyAsync(v->slices, tab.data(), tab.size() * sizeof(VadSlice), cudaMemcpyHostToDevice, s));
      B2W_CUDA(cudaEventRecord(v->ev[0], s));
      vad_windows(v->w, v->pcm, v->slices, n_slices, nb, v->gx, s);
      B2W_CUDA(cudaEventRecord(v->ev[1], s));
      vad_recurrence(v->w_hh, v->slices, n_slices, v->gx, v->states, v->H, s);
      B2W_CUDA(cudaEventRecord(v->ev[2], s));
      vad_decoder(v->H, v->dec_w, v->dec_b, nb, v->probs, s);
      B2W_CUDA(cudaEventRecord(v->ev[3], s));
      B2W_CUDA(cudaMemcpyAsync(v->host_probs.data(), v->probs, (size_t)nb * 4, cudaMemcpyDeviceToHost, s));
      B2W_CUDA(cudaStreamSynchronize(s));
      for (int i = 0; i < 3; ++i) {
        float ms = 0.f;
        B2W_CUDA(cudaEventElapsedTime(&ms, v->ev[i], v->ev[i + 1]));
        v->ms[i] += ms;
      }
      for (const VadSlice& sl : tab) {
        memcpy(probs_out + out0[sl.stream] + done[sl.stream], v->host_probs.data() + sl.w0, (size_t)sl.nb * 4);
        done[sl.stream] += sl.nb;
        left[sl.stream] -= sl.nb;
      }
      remaining -= nb;
    }
  });
}

int b2w_vad_timing(b2w_vad* v, double ms_out[3]) {
  return guarded([&] {
    B2W_CHECK(v && ms_out, "null argument");
    std::lock_guard<std::mutex> lk(v->mu);
    for (int i = 0; i < 3; ++i) ms_out[i] = v->ms[i];
  });
}

}  // extern "C"
