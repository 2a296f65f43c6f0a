// Host-side engine: weight upload, encoder orchestration, generate loop, and the extern "C" ABI declared in
// include/b200whisper.h.  PyTorch is not involved: the library owns its device memory and one CUDA stream per
// model.  There is no CPU fallback — every entry point fails loudly when no sm_90 device is usable.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>

#include "model.h"

namespace b2w {

// ---- error / counters ---------------------------------------------------------------------------------------
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

Model::~Model() {
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);
  for (void* p : allocs) cudaFree(p);
  for (auto& it : pool) cudaFree(it.second);
  void* ws[] = {e_feats, e_x0, e_x1, e_x, e_xn, e_qkv, e_ao, e_h, e_pcm, e_chunks, e_chunk_max, kcache, vcache, d_x, d_xn,
                d_q, d_ao, d_h, d_logits, d_xpart, d_counters, d_suppress, sb_blob, d_bind, d_layers, d_bar, d_gpart, d_stpart};
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
void Model::pool_put(void* p, size_t bytes) {
  if (!p) return;
  if (pool_bytes + bytes > (size_t)24 << 30 || pool.size() >= 16) {
    cudaFree(p);
    return;
  }
  pool.emplace_back(bytes, p);
  pool_bytes += bytes;
}

Encoded::~Encoded() {
  if (!owner) return;
  cudaSetDevice(owner->device);
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
    T* p = dalloc<T>(n);
    m->allocs.push_back(p);
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
    D.ln1_g = D.ln1_b = D.ln2_g = D.ln2_b = D.ln3_g = D.ln3_b = nullptr;
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
    m->dec_ln_g = m->dec_ln_b = nullptr;
  }
  m->dec_weight_bytes = wbytes;
  m->mel.reset(new MelPlan(cfg.n_mels));
  m->d_counters = dalloc<int>(64 + 16 * 20 * 64);
  B2W_CUDA(cudaMemset(m->d_counters, 0, (64 + 16 * 20 * 64) * sizeof(int)));
  B2W_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->h_pinned), 4096));
  m->d_suppress = dalloc<uint8_t>(m->vpad);
  m->d_bind = dalloc<DecBindings>(1);
  decode_configure();
  search_configure();
  gemm_configure();
  dstep_configure();
  bstep_configure();
  {
    // decoder weights re-laid out as the persistent step kernel's tile stream (a second copy: ~1.6 GB for large-v3)
    std::vector<DLayer> hl(L);
    unsigned char* q_scratch = nullptr;
    float* scale_scratch = nullptr;
    if (m->w8 || m->w8_fake) {
      q_scratch = dalloc<unsigned char>((size_t)m->vpad * dt > (size_t)4 * dt * dt ? (size_t)m->vpad * dt : (size_t)4 * dt * dt);
      scale_scratch = dalloc<float>((size_t)std::max(m->vpad, 4 * dt));
    }
    // every decoder matrix is laid out twice: as the <= 8-row kernel's tile stream (dstep.cu) and as the many-row kernel's atom
    // stream (bstep.cu, + row sums for the deferred LayerNorm); with compute_type int8* both streams carry the int8 values
    const bool want_b = m->use_bstep && dt % 64 == 0 && dt == 64 * cfg.n_text_head;
    struct BPack {
      const void* atoms = nullptr;
      const float* scale = nullptr;
      const float* wsum = nullptr;
    };
    auto pack = [&](const __half* W, const float* bias, int N, int K, int ksplit, BPack* bp, bool want_wsum) -> const __half* {
      const __half* tiles = nullptr;
      if (m->w8 || m->w8_fake) {
        // quantise per output channel; W now holds q * scale (what the prefill / multi-kernel paths multiply with)
        dstep_quantize_rows(const_cast<__half*>(W), N, K, q_scratch, scale_scratch, m->stream);
      }
      if (m->w8) {
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
    else m->use_dstep = false;
    if (q_scratch) {
      B2W_CUDA(cudaStreamSynchronize(m->stream));
      cudaFree(q_scratch);
      cudaFree(scale_scratch);
    }
    m->d_layers = dalloc<DLayer>(L);
    B2W_CUDA(cudaMemcpy(m->d_layers, hl.data(), L * sizeof(DLayer), cudaMemcpyHostToDevice));
    if (want_b && packable) {
      m->logit_atoms = lp.atoms;
      m->logit_scale = lp.scale;
      m->d_blayers = dalloc<BLayer>(L);
      B2W_CUDA(cudaMemcpy(m->d_blayers, bl.data(), L * sizeof(BLayer), cudaMemcpyHostToDevice));
      m->bstep_packed = true;
    }
    m->d_bar = dalloc<unsigned>(kBsBarWords);
    B2W_CUDA(cudaMemset(m->d_bar, 0, kBsBarWords * sizeof(unsigned)));
  }
  for (int l = L / 2; l < L; ++l)  // default alignment heads: every head of the last half of the decoder (OpenAI Whisper's default)
    for (int hh = 0; hh < cfg.n_text_head; ++hh) m->align_heads.push_back(make_int2(l, hh));
  B2W_CUDA(cudaStreamSynchronize(m->stream));
}

// ---- encoder ----------------------------------------------------------------------------------------------------------
static void ensure_encoder_ws(Model* m, int b) {
  if (b <= m->enc_max_b) return;
  B2W_CUDA(cudaStreamSynchronize(m->stream));
  void* old[] = {m->e_feats, m->e_x0, m->e_x1, m->e_x, m->e_xn, m->e_qkv, m->e_ao, m->e_h, m->e_chunks, m->e_chunk_max};
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
  for (int l = 0; l < Lc; ++l) {
    const EncLayerW& W = m->enc[l];
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

static Encoded* encode_features(Model* m, const float* feats_host, const float* feats_dev, int B) {
  std::unique_ptr<Encoded> e(new Encoded);
  e->owner = m;
  e->B = B;
  const size_t d = m->cfg.n_audio_state;
  e->enc_bytes = (size_t)B * 1500 * d * sizeof(__half);
  e->enc_out = reinterpret_cast<__half*>(m->pool_get(e->enc_bytes));
  const size_t per = (size_t)m->cfg.n_mels * 3000;
  for (int b0 = 0; b0 < B; b0 += kEncSub) {
    const int b = std::min(kEncSub, B - b0);
    ensure_encoder_ws(m, std::min(kEncSub, B));
    if (feats_host) {
      ScopedStage st(m, B2W_T_H2D);
      B2W_CUDA(cudaMemcpyAsync(m->e_feats, feats_host + b0 * per, b * per * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    } else if (feats_dev != m->e_feats) {
      B2W_CUDA(cudaMemcpyAsync(m->e_feats, feats_dev + b0 * per, b * per * sizeof(float), cudaMemcpyDeviceToDevice, m->stream));
    }
    ScopedStage st(m, B2W_T_ENCODER);
    encoder_forward(m, b, e->enc_out + (size_t)b0 * 1500 * d);
  }
  return e.release();
}

// ---- log-mel --------------------------------------------------------------------------------------------------------------
static int mel_frames(int64_t n_samples) { return (int)(1 + n_samples / 160); }

// ---- decoder ----------------------------------------------------------------------------------------------------------------
constexpr int kMaxRows = 80;

static void ensure_decoder_ws(Model* m, int chunks, int slots) {
  const int dt = m->cfg.n_text_state, L = m->cfg.n_text_layer, n_ctx = m->cfg.n_text_ctx;
  if (!m->d_x) {
    const size_t dt128 = (size_t)ceil_div(dt, 128) * 128;  // the many-row step kernel keeps its fp32 buffers n-block-major (128-channel blocks)
    m->d_x = dalloc<float>((size_t)kMaxRows * dt128);
    m->d_xn = dalloc<__half>((size_t)kMaxRows * dt);
    m->d_q = dalloc<__half>((size_t)kMaxRows * dt);
    m->d_ao = dalloc<__half>((size_t)kMaxRows * dt);
    m->d_h = dalloc<__half>((size_t)kMaxRows * 4 * dt);
    m->d_logits = dalloc<float>((size_t)kMaxRows * m->vpad);
    m->d_qkv32 = dalloc<float>((size_t)kMaxRows * ceil_div(3 * dt, 128) * 128);
    m->d_cq32 = dalloc<float>((size_t)kMaxRows * dt128);
    m->d_h32 = dalloc<float>((size_t)kMaxRows * ceil_div(4 * dt, 128) * 128);
    m->d_h16 = dalloc<__half>((size_t)kMaxRows * 4 * dt);
    m->d_xn16 = dalloc<__half>((size_t)kMaxRows * dt);
    m->d_stats = dalloc<float>((size_t)3 * L * kMaxRows * 2 + 4);
    m->d_gpart = dalloc<float>((size_t)m->num_sms * kMaxRows * 128);  // the many-row step kernel's per-CTA split-K partial tiles
    m->d_stpart = dalloc<float>((size_t)(dt / 64) * kMaxRows * 2);
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
  const size_t o_params = take(sizeof(SearchParams));
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
  e->xkv = reinterpret_cast<__half*>(m->pool_get(e->xkv_bytes));
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

constexpr int kTcMinRows = 17;  // rows above which the decode GEMMs go through the wgmma path (activations reused from smem)

// decode GEMM through the tensor-core GEMM: the plan (TMA maps) is cached per (weights, activations, rows)
static const GemmPlan& dec_plan(Model* m, const GvArgs& a) {
  const auto key = std::make_tuple((const void*)a.W, (const void*)a.x, a.R, a.mode);
  auto it = m->dec_plans.find(key);
  if (it != m->dec_plans.end()) return it->second;
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
  return m->dec_plans.emplace(key, gemm_plan(g, m->num_sms)).first->second;
}

static void gv(Model* m, GvArgs a) {
  if (m->use_ref_gemv && (a.mode == GV_F32)) {
    skinny_ref(a.x, a.W, a.bias, a.out_f, a.R, a.N, a.K, m->stream);
    return;
  }
  if (a.R >= kTcMinRows && a.K % 64 == 0 && a.N % 32 == 0 && !m->use_ref_gemv) {
    gemm_run(dec_plan(m, a), m->stream);
    if (a.mode == GV_RESID_LN) layernorm_f32_f16(a.xres, a.ln_g, a.ln_b, a.xn_out, a.R, a.N, m->stream);
    return;
  }
  skinny_gemm(a, m->stream);
}

static void bind_encoded(Model* m, const Encoded* e, int chunk0) {
  m->h_bind = DecBindings{e ? e->xkv : nullptr, e ? e->B : 0, chunk0};
  B2W_CUDA(cudaMemcpyAsync(m->d_bind, &m->h_bind, sizeof(DecBindings), cudaMemcpyHostToDevice, m->stream));
}

static void decoder_layers(Model* m, int n_chunks, int rows_per_chunk, int slots, int splits, int step_base) {
  const b2w_config& c = m->cfg;
  const int dt = c.n_text_state, L = c.n_text_layer, H = c.n_text_head, R = n_chunks * rows_per_chunk;
  cudaStream_t s = m->stream;
  const SearchBuffers& sb = m->sb;
  embed_ln(sb.tokens_in, sb.rows, m->tok_emb, m->dec_pos, m->dec[0].ln1_g, m->dec[0].ln1_b, m->d_x, m->d_xn, R, dt, c.n_vocab, s);
  const int qgroups = cross_attn_qgroups(rows_per_chunk);
  const size_t need_part = cross_attn_partial_floats(n_chunks, H, rows_per_chunk, splits);
  if (need_part > m->d_xpart_floats) {
    B2W_CUDA(cudaStreamSynchronize(s));
    if (m->d_xpart) cudaFree(m->d_xpart);
    m->d_xpart = dalloc<float>(need_part);
    m->d_xpart_floats = need_part;
  }
  B2W_CHECK((size_t)n_chunks * H * qgroups <= 16 * 20 * 64, "cross-attention group counters");
  for (int l = 0; l < L; ++l) {
    const DecLayerW& W = m->dec[l];
    __half* kc = m->kcache + (size_t)l * m->kv_elems;
    __half* vc = m->vcache + (size_t)l * m->kv_elems;
    GvArgs a;
    a.x = m->d_xn; a.W = W.wqkv; a.bias = W.bqkv; a.R = R; a.N = 3 * dt; a.K = dt; a.mode = GV_QKV;
    a.rows = sb.rows; a.kcache = kc; a.vcache = vc; a.d = dt; a.n_ctx = c.n_text_ctx; a.slots = slots; a.out_h = m->d_q;
    gv(m, a);
    SelfAttnArgs sa{sb.rows, m->d_q, kc, vc, sb.anc, m->d_ao, dt, c.n_text_ctx, slots,
                    (long long)n_chunks * slots * c.n_text_ctx, step_base};
    dec_self_attn(sa, R, H, s);
    GvArgs o;
    o.x = m->d_ao; o.W = W.wo; o.bias = W.bo; o.R = R; o.N = dt; o.K = dt; o.mode = GV_RESID_LN;
    o.xres = m->d_x; o.ln_g = W.ln2_g; o.ln_b = W.ln2_b; o.xn_out = m->d_xn; o.counter = m->d_counters;
    gv(m, o);
    GvArgs q;
    q.x = m->d_xn; q.W = W.wq_x; q.bias = W.bq_x; q.R = R; q.N = dt; q.K = dt; q.mode = GV_F16; q.out_h = m->d_q;
    gv(m, q);
    if (m->align_out)
      align_probs(m->d_q, m->d_bind, l, m->d_align_heads, (int)m->align_heads.size(), m->align_out, m->align_n_tok, m->align_nf,
                  m->align_pos0, R, H, 1500, dt, s);
    if (m->use_mma_xattn && splits >= kDsXSplits && dstep_cross_attn_supported(1500, rows_per_chunk)) {
      DStepArgs xa{};
      xa.q = m->d_q; xa.ao = m->d_ao; xa.bind = m->d_bind; xa.xpart = m->d_xpart; xa.xcounters = m->d_counters + 64;
      xa.H = H; xa.T = 1500; xa.d = dt; xa.rows_per_chunk = rows_per_chunk; xa.n_chunks = n_chunks;
      dstep_cross_attn_launch(xa, l, s);
    } else {
      CrossAttnArgs ca;
      ca.q = m->d_q;
      ca.bind = m->d_bind;
      ca.layer = l;
      ca.out = m->d_ao; ca.partial = m->d_xpart; ca.counters = m->d_counters + 64;
      ca.T = 1500; ca.H = H; ca.d = dt; ca.rows_per_chunk = rows_per_chunk; ca.splits = splits; ca.qgroups = qgroups;
      dec_cross_attn(ca, n_chunks, s);
    }
    GvArgs ox;
    ox.x = m->d_ao; ox.W = W.wo_x; ox.bias = W.bo_x; ox.R = R; ox.N = dt; ox.K = dt; ox.mode = GV_RESID_LN;
    ox.xres = m->d_x; ox.ln_g = W.ln3_g; ox.ln_b = W.ln3_b; ox.xn_out = m->d_xn; ox.counter = m->d_counters;
    gv(m, ox);
    GvArgs f1;
    f1.x = m->d_xn; f1.W = W.w1; f1.bias = W.b1; f1.R = R; f1.N = 4 * dt; f1.K = dt; f1.mode = GV_GELU_F16; f1.out_h = m->d_h;
    gv(m, f1);
    GvArgs f2;
    f2.x = m->d_h; f2.W = W.w2; f2.bias = W.b2; f2.R = R; f2.N = dt; f2.K = 4 * dt; f2.mode = GV_RESID_LN;
    f2.xres = m->d_x;
    f2.ln_g = (l + 1 < L) ? m->dec[l + 1].ln1_g : m->dec_ln_g;
    f2.ln_b = (l + 1 < L) ? m->dec[l + 1].ln1_b : m->dec_ln_b;
    f2.xn_out = m->d_xn; f2.counter = m->d_counters;
    gv(m, f2);
  }
}

static void logits_gemm(Model* m, int R) {
  GvArgs a;
  a.x = m->d_xn; a.W = m->logit_w; a.bias = m->logit_b; a.R = R; a.N = m->vpad; a.K = m->cfg.n_text_state; a.mode = GV_F32;
  a.out_f = m->d_logits; a.ldo = m->vpad;
  gv(m, a);
}

static int pick_splits(const Model* m, int n_chunks, int rows_per_chunk) {
  // 8 key splits (~188 keys each): the V tile fits in shared memory next to the scores and even one chunk fills the SMs
  (void)m; (void)n_chunks; (void)rows_per_chunk;
  return 8;
}

// Forced decoding of tokens[chunk][i0..i1) for chunks [chunk0, chunk0+n): rows = n*(i1-i0) <= 80, slot 0.
static void prefill_pass(Model* m, const Encoded* e, int chunk0, int n, const int32_t* tokens, int stride, int i0, int i1, int slots,
                         int step_base) {
  const int rpc = i1 - i0, R = n * rpc;
  std::vector<RowInfo> rows(R);
  std::vector<int> toks(R);
  for (int b = 0; b < n; ++b)
    for (int i = i0; i < i1; ++i) {
      rows[b * rpc + (i - i0)] = RowInfo{b, 0, i, 0};
      toks[b * rpc + (i - i0)] = tokens[(size_t)(chunk0 + b) * stride + i];
    }
  B2W_CUDA(cudaMemcpyAsync(m->sb.rows, rows.data(), R * sizeof(RowInfo), cudaMemcpyHostToDevice, m->stream));
  B2W_CUDA(cudaMemcpyAsync(m->sb.tokens_in, toks.data(), R * sizeof(int), cudaMemcpyHostToDevice, m->stream));
  B2W_CUDA(cudaStreamSynchronize(m->stream));  // host vectors go out of scope
  bind_encoded(m, e, chunk0);
  decoder_layers(m, n, rpc, slots, pick_splits(m, n, rpc), step_base);
}

struct HypOut {
  std::vector<int> ids;
  float score;
};

static void generate_group(Model* m, Encoded* e, int chunk0, int n, const int32_t* prompts, int P, const b2w_gen_opts& o,
                           int32_t* out_ids, int32_t* out_lens, float* out_scores, float* out_ns) {
  const b2w_config& c = m->cfg;
  const bool beam = o.beam_size > 1;
  const int K = beam ? o.beam_size : std::max(1, o.num_hypotheses);
  const int num_hyp = std::max(1, o.num_hypotheses);
  const int R = n * K;
  const int max_steps = o.max_length - P;
  cudaStream_t s = m->stream;
  const SearchBuffers& sb = m->sb;
  const int n_ctx = c.n_text_ctx;

  // ---- validate prompts / find SOT ----
  int sot_index = -1;
  for (int b = 0; b < n; ++b) {
    const int32_t* p = prompts + (size_t)(chunk0 + b) * P;
    int si = -1;
    for (int i = 0; i < P; ++i) {
      B2W_CHECK(p[i] >= 0 && p[i] < c.n_vocab, "prompt token id out of range");
      if (p[i] == c.sot && si < 0) si = i;
    }
    if (si < 0) throw Error("<|startoftranscript|> token was not found in the prompt", true);
    if (sot_index < 0) sot_index = si;
    else if (si != sot_index) throw Error("<|startoftranscript|> must be at the same position in all prompts", true);
  }
  for (int b = 0; b < n; ++b) out_ns[chunk0 + b] = 0.f;

  // ---- search parameters ----
  SearchParams sp{};
  sp.n_vocab = c.n_vocab; sp.vpad = m->vpad; sp.B = n; sp.K = K;
  sp.mode = beam ? 0 : 1;
  sp.ncand = beam ? 2 * K : 1;
  sp.max_steps = max_steps; sp.prompt_len = P;
  sp.max_finished = std::max(1, (int)lroundf(K * o.patience));
  sp.allow_early_exit = (o.patience == 1.0f && o.length_penalty == 0.0f) ? 1 : 0;
  sp.num_hyp = num_hyp;
  sp.length_penalty = o.length_penalty; sp.repetition_penalty = o.repetition_penalty;
  sp.no_repeat_ngram = o.no_repeat_ngram_size;
  sp.suppress_blank = o.suppress_blank;
  sp.n_suppress_begin = c.n_suppress_begin;
  for (int i = 0; i < 8; ++i) sp.suppress_begin[i] = c.suppress_begin[i];
  bool has_no_ts = false;
  for (int i = 0; i < P; ++i) has_no_ts = has_no_ts || prompts[(size_t)chunk0 * P + i] == c.no_timestamps;
  sp.timestamp_rules = has_no_ts ? 0 : 1;
  sp.max_initial_ts = o.max_initial_timestamp_index;
  sp.eot = c.eot; sp.no_timestamps = c.no_timestamps; sp.timestamp_begin = c.timestamp_begin; sp.no_speech = c.no_speech;
  sp.sampling_topk = o.sampling_topk; sp.temperature = o.sampling_temperature > 0 ? o.sampling_temperature : 1.0f;
  sp.seed = o.seed;
  sp.want_no_speech_first = (o.return_no_speech_prob && sot_index == P - 1) ? 1 : 0;
  sp.fake_logits = o.debug_fake_logits;
  B2W_CHECK(sp.max_finished <= kMaxFinished, "beam_size * patience is too large");

  if (max_steps <= 0) {
    for (int b = 0; b < n; ++b)
      for (int h = 0; h < num_hyp; ++h) {
        out_lens[(size_t)(chunk0 + b) * num_hyp + h] = 0;
        out_scores[(size_t)(chunk0 + b) * num_hyp + h] = 0.f;
      }
    return;
  }

  // ---- reset search state ----
  const size_t RB = (size_t)n * K;
  B2W_CUDA(cudaMemsetAsync(sb.state, 0, sizeof(SearchState), s));
  B2W_CUDA(cudaMemsetAsync(sb.cum, 0, 2 * RB * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.anc, 0, 2 * RB * n_ctx, s));
  B2W_CUDA(cudaMemsetAsync(sb.done, 0, n * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.fin_count, 0, n * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.fin_len, 0xFF, (size_t)n * kMaxFinished * 4, s));
  B2W_CUDA(cudaMemsetAsync(sb.no_speech, 0, n * 4, s));

  // ---- prefill: prompt[:-1] in passes of <= 80 rows ----
  if (!sp.fake_logits && P > 1) {
    ScopedStage st(m, B2W_T_PREFILL);
    const int per_pass = std::max(1, kMaxRows / n);
    for (int i0 = 0; i0 < P - 1; i0 += per_pass) {
      const int i1 = std::min(P - 1, i0 + per_pass);
      prefill_pass(m, e, chunk0, n, prompts, P, i0, i1, K, P - 1);
      if (o.return_no_speech_prob && sot_index >= i0 && sot_index < i1) {
        logits_gemm(m, n * (i1 - i0));
        no_speech_from_logits(m->d_logits, m->vpad, n * (i1 - i0), i1 - i0, sot_index - i0, c.n_vocab, c.no_speech, sb.no_speech, s);
      }
    }
  }

  // ---- decode rows ----
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
  const int splits = pick_splits(m, n, K);
  if (!sp.fake_logits) {
    // lazily-grown partial buffer of the cross attention: sized before any kernel argument block captures the pointer
    size_t need_part = cross_attn_partial_floats(n, c.n_text_head, K, splits);
    need_part = std::max(need_part, (size_t)n * c.n_text_head * kDsXSplits * 8 * 66);
    if (need_part > m->d_xpart_floats) {
      B2W_CUDA(cudaStreamSynchronize(s));
      if (m->d_xpart) cudaFree(m->d_xpart);
      m->d_xpart = dalloc<float>(need_part);
      m->d_xpart_floats = need_part;
    }
  }
  // persistent single-kernel step for <= 8 rows
  DStepArgs ds{};
  bool use_dstep = m->use_dstep && !sp.fake_logits && R <= 8 && !m->use_ref_gemv && c.n_text_layer <= 32;
  if (use_dstep) {
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
    if (m->dstep_grid == 0) {
      m->dstep_grid = dstep_max_grid(m->num_sms, ds);
      if (m->dstep_grid == 0) m->dstep_grid = -1;
    }
    if (m->dstep_grid <= 0) use_dstep = false;
  }
  // persistent many-row step (bstep.cu) for everything the <= 8-row kernel does not take
  BStepArgs bs{};
  bool use_bstep = m->use_bstep && m->bstep_packed && !sp.fake_logits && !m->use_ref_gemv && (m->bstep_all || !use_dstep) && R <= kBsMaxRows;
  if (use_bstep) {
    bs.layers = m->d_blayers; bs.L = c.n_text_layer; bs.tok_emb = m->tok_emb; bs.pos_emb = m->dec_pos;
    bs.logit_atoms = m->logit_atoms; bs.logit_bias = m->logit_b; bs.logit_scale = m->logit_scale; bs.w8 = m->w8 ? 1 : 0;
    bs.R = R; bs.d = c.n_text_state; bs.H = c.n_text_head; bs.n_ctx = c.n_text_ctx; bs.slots = K; bs.T = 1500;
    bs.vpad = m->vpad; bs.n_vocab = c.n_vocab; bs.n_chunks = n; bs.rows_per_chunk = K;
    bs.stop_phase = m->bstep_stop;
    if (const char* v = getenv("B2W_BSTEP_STOP")) bs.stop_phase = atoi(v);  // re-read per call: tools/bstep_bisect.py steps it
    bs.rows = sb.rows; bs.tokens_in = sb.tokens_in;
    bs.x = m->d_x; bs.qkv32 = m->d_qkv32; bs.cq32 = m->d_cq32; bs.h32 = m->d_h32; bs.ao = m->d_ao; bs.h16 = m->d_h16; bs.xn16 = m->d_xn16;
    bs.stats = m->d_stats; bs.stpart = m->d_stpart; bs.gpart = m->d_gpart; bs.logits = m->d_logits;
    bs.kcache = m->kcache; bs.vcache = m->vcache; bs.kv_layer_stride = (long long)m->kv_elems;
    bs.anc = sb.anc; bs.anc_buf_stride = (long long)n * K * c.n_text_ctx;
    bs.bind = m->d_bind; bs.xcounters = m->d_counters + 64; bs.bar = m->d_bar; bs.prof = m->d_prof;
    use_bstep = bstep_supported(m->num_sms, bs);
    if (use_bstep) {
      use_dstep = false;
      const size_t need_part = std::max(bstep_xpart_floats(bs), cross_attn_partial_floats(n, c.n_text_head, K, splits));
      if (need_part > m->d_xpart_floats) {
        B2W_CUDA(cudaStreamSynchronize(s));
        if (m->d_xpart) cudaFree(m->d_xpart);
        m->d_xpart = dalloc<float>(need_part);
        m->d_xpart_floats = need_part;
      }
      bs.xpart = m->d_xpart;
    }
  }
  m->h_params = sp;
  B2W_CUDA(cudaMemcpyAsync(const_cast<SearchParams*>(sb.params), &m->h_params, sizeof(SearchParams), cudaMemcpyHostToDevice, s));
  bind_encoded(m, e, chunk0);
  auto record_step = [&]() {
    if (sp.fake_logits) {
      fake_logits(m->d_logits, R, sb, s);
    } else {
      if (use_bstep) {
        bstep_launch(bs, m->num_sms, s);
      } else if (use_dstep) {
        dstep_launch(ds, m->dstep_grid, s);
      } else {
        decoder_layers(m, n, K, K, splits, P - 1);
        logits_gemm(m, R);
      }
    }
    search_rows(m->d_logits, R, m->vpad, sb, s);
    search_update(n, sb, s);
  };

  // one CUDA graph per (shape, options, buffers) — replayed every step, no per-step host parameters
  // the graph depends only on shapes and workspace pointers: options and encoder-output bindings are read from
  // device memory by the kernels, so one instantiated graph serves every window / chunk group of the same shape
  std::vector<uint8_t> key(4 * sizeof(void*) + 8 * sizeof(int));
  {
    uint8_t* k = key.data();
    const void* ptrs[4] = {m->kcache, m->sb_blob, m->d_xpart, m->d_logits};
    memcpy(k, ptrs, sizeof ptrs); k += sizeof ptrs;
    int misc[8] = {splits, m->use_ref_gemv ? 1 : 0, n, K, sp.fake_logits, use_dstep ? 1 : (use_bstep ? 3 : 0), bs.stop_phase, 0};
    memcpy(k, misc, sizeof misc);
  }
  if (sp.fake_logits == 0) {
    // make sure lazily-grown buffers exist before capture (capture forbids cudaMalloc/sync)
    const size_t need_part = cross_attn_partial_floats(n, c.n_text_head, K, splits);
    if (need_part > m->d_xpart_floats) {
      if (m->d_xpart) cudaFree(m->d_xpart);
      m->d_xpart = dalloc<float>(need_part);
      m->d_xpart_floats = need_part;
      const void* px = m->d_xpart;
      memcpy(key.data() + 2 * sizeof(void*), &px, sizeof px);
    }
  }
  const int64_t launches_before = g_launches;
  bool graph_ok = m->use_graph;
  if (graph_ok && (!m->step_graph || m->step_graph_key != key)) {
    if (m->step_graph) {
      cudaGraphExecDestroy(m->step_graph);
      m->step_graph = nullptr;
    }
    cudaGraph_t graph = nullptr;
    B2W_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    try {
      record_step();
    } catch (...) {
      cudaStreamEndCapture(s, &graph);
      if (graph) cudaGraphDestroy(graph);
      throw;
    }
    B2W_CUDA(cudaStreamEndCapture(s, &graph));
    B2W_CUDA(cudaGraphInstantiate(&m->step_graph, graph, 0));
    cudaGraphDestroy(graph);
    m->step_graph_key = key;
  }
  if (g_launches != launches_before) m->step_graph_kernels = g_launches - launches_before;  // recorded during capture
  const int64_t per_step_kernels = m->step_graph_kernels;
  g_launches = launches_before;

  // ---- step loop: the host only polls the done counter ----
  int steps_run = 0;
  {
    ScopedStage st(m, B2W_T_DECODE);
    const int poll = 4;
    for (int step = 0; step < max_steps; ++step) {
      if (graph_ok) {
        B2W_CUDA(cudaGraphLaunch(m->step_graph, s));
        g_launches += per_step_kernels;
      } else {
        record_step();
      }
      ++steps_run;
      // algorithmic bytes of this step: weights + beam-shared cross-KV + self-KV read so far
      // (the persistent kernels stream int8 weights with compute_type int8*: half the fp16 bytes; per-channel scales are negligible)
      m->decode_alg_bytes += ((m->w8 && (use_dstep || use_bstep)) ? 0.5 * m->dec_weight_bytes : m->dec_weight_bytes) +
                             (double)n * c.n_text_layer * 2.0 * 1500 * c.n_text_state * 2.0 +
                             (double)R * (P + step) * c.n_text_layer * 2.0 * c.n_text_state * 2.0;
      if ((step % poll) == poll - 1 && step + 1 < max_steps) {
        B2W_CUDA(cudaMemcpyAsync(m->h_pinned, &sb.state->n_done, sizeof(int), cudaMemcpyDeviceToHost, s));
        B2W_CUDA(cudaStreamSynchronize(s));
        if (m->h_pinned[0] >= n) break;
      }
    }
    m->decode_steps += steps_run;
    if (m->d_prof && use_bstep) {
      B2W_CUDA(cudaStreamSynchronize(s));
      const int L = c.n_text_layer, nstamps = 1 + 2 * (2 + 9 * L) + 1;
      std::vector<unsigned long long> t(nstamps);
      B2W_CUDA(cudaMemcpy(t.data(), m->d_prof, nstamps * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      static const char* names[9] = {"qkv", "self_attn", "out_proj", "cross_q", "cross_attn", "cross_out", "ffn1", "gelu", "ffn2"};
      double work[9] = {0}, wait[9] = {0};
      unsigned long long prev = t[2];
      for (int l = 0; l < L; ++l)
        for (int ph = 0; ph < 9; ++ph) {
          const int bi = 1 + 2 * (1 + l * 9 + ph);
          work[ph] += double(t[bi] - prev);
          wait[ph] += double(t[bi + 1] - t[bi]);
          prev = t[bi + 1];
        }
      const int bf = 1 + 2 * (1 + 9 * L);
      fprintf(stderr, "[bstep prof] last step (R=%d): total %.1f us; embed %.1f us; final-LN %.1f us; logits %.1f us\n", R, (t[nstamps - 1] - t[0]) / 1e3,
              (t[2] - t[0]) / 1e3, (t[bf] - prev) / 1e3, (t[nstamps - 1] - t[bf + 1]) / 1e3);
      for (int ph = 0; ph < 9; ++ph)
        fprintf(stderr, "[bstep prof]   %-10s work %.2f us  barrier wait %.2f us (CTA 0, mean over %d layers)\n", names[ph], work[ph] / L / 1e3,
                wait[ph] / L / 1e3, L);
      {
        std::vector<unsigned long long> f(8 * 16);
        B2W_CUDA(cudaMemcpy(f.data(), m->d_prof + 3000, f.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        B2W_CUDA(cudaMemset(m->d_prof + 3000, 0, f.size() * sizeof(unsigned long long)));
        if (f[6 * 16 + 15] > 0)
          fprintf(stderr, "[bstep prof]   self-attn cycles per 16-key block (CTA 0 warp 0): (unused) %.0f  issue+copy-wait %.0f  compute %.0f; prologue per task total %.0f over %llu blocks\n",
                  (double)f[6 * 16 + 1] / f[6 * 16 + 15], (double)f[6 * 16 + 2] / f[6 * 16 + 15], (double)f[6 * 16 + 3] / f[6 * 16 + 15], (double)f[6 * 16],
                  f[6 * 16 + 15]);
        if (f[7 * 16 + 15] > 0)
          fprintf(stderr, "[bstep prof]   cross-attn cycles per tile (CTA 0): tile-wait %.0f  compute %.0f; piece ends total %.0f, prologues total %.0f over %llu tiles\n",
                  (double)f[7 * 16] / f[7 * 16 + 15], (double)f[7 * 16 + 1] / f[7 * 16 + 15], (double)f[7 * 16 + 2], (double)f[7 * 16 + 3], f[7 * 16 + 15]);
        static const char* kinds[6] = {"qkv", "out", "cross_q", "cross_out", "ffn1", "ffn2"};
        for (int k = 0; k < 6; ++k) {
          const double cnt = (double)f[k * 16 + 15];
          if (cnt > 0)
            fprintf(stderr, "[bstep prof]   %-9s cycles (CTA 0): stage %.0f  sync %.0f  row statistics %.0f  products + reduction %.0f\n", kinds[k],
                    f[k * 16] / cnt, f[k * 16 + 4] / cnt, f[k * 16 + 5] / cnt, f[k * 16 + 2] / cnt);
        }
      }
    }
    if (m->d_prof && use_dstep) {
      B2W_CUDA(cudaStreamSynchronize(s));
      const int L = c.n_text_layer, nstamps = 1 + 2 * (1 + 8 * L) + 1;
      std::vector<unsigned long long> t(nstamps);
      B2W_CUDA(cudaMemcpy(t.data(), m->d_prof, nstamps * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      // stamps: [0]=start, then (arrive, release) per barrier, then end.  work(p) = arrive_p - release_{p-1}; wait(p) = release_p - arrive_p
      static const char* names[8] = {"qkv", "self_attn", "out_proj", "cross_q", "cross_attn", "cross_out", "ffn1", "ffn2"};
      double work[8] = {0}, wait[8] = {0};
      unsigned long long prev = t[2];  // release of the embed barrier
      for (int l = 0; l < L; ++l)
        for (int ph = 0; ph < 8; ++ph) {
          const int bi = 1 + 2 * (1 + l * 8 + ph);
          work[ph] += double(t[bi] - prev);
          wait[ph] += double(t[bi + 1] - t[bi]);
          prev = t[bi + 1];
        }
      fprintf(stderr, "[dstep prof] last step: total %.1f us; embed %.1f us; logits %.1f us\n", (t[nstamps - 1] - t[0]) / 1e3,
              (t[2] - t[0]) / 1e3, (t[nstamps - 1] - prev) / 1e3);
      {
        std::vector<unsigned long long> f(8 * 16);
        B2W_CUDA(cudaMemcpy(f.data(), m->d_prof + 3000, f.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        B2W_CUDA(cudaMemset(m->d_prof + 3000, 0, f.size() * sizeof(unsigned long long)));
        static const char* kinds[7] = {"qkv", "out", "cross_q", "cross_out", "ffn1", "ffn2", "logits"};
        for (int k = 0; k < 7; ++k) {
          const double n = (double)f[k * 16 + 15];
          if (n > 0)
            fprintf(stderr, "[dstep prof]   %-9s cycles (first item): stage-input %.0f  tile-wait %.0f  mma %.0f  epilogue %.0f\n", kinds[k], f[k * 16] / n,
                    f[k * 16 + 1] / n, f[k * 16 + 2] / n, f[k * 16 + 3] / n);
        }
      }
      for (int ph = 0; ph < 8; ++ph)
        fprintf(stderr, "[dstep prof]   %-10s work %.2f us  barrier wait %.2f us (CTA 0, mean over %d layers)\n", names[ph], work[ph] / L / 1e3,
                wait[ph] / L / 1e3, L);
    }
  }

  // ---- collect hypotheses ----
  ScopedStage st(m, B2W_T_D2H);
  std::vector<int> fin_count(n), fin_len((size_t)n * kMaxFinished);
  std::vector<float> fin_score((size_t)n * kMaxFinished), ns(n);
  std::vector<int> fin_tok((size_t)n * kMaxFinished * n_ctx);
  B2W_CUDA(cudaMemcpyAsync(fin_count.data(), sb.fin_count, n * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(fin_len.data(), sb.fin_len, fin_len.size() * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(fin_score.data(), sb.fin_score, fin_score.size() * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(fin_tok.data(), sb.fin_tok, fin_tok.size() * 4, cudaMemcpyDeviceToHost, s));
  B2W_CUDA(cudaMemcpyAsync(ns.data(), sb.no_speech, n * 4, cudaMemcpyDeviceToHost, s));
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
    const char* ok[] = {"default", "auto", "float16", "int8_float16", "int8", "float32", "bfloat16", "int8_float32", "int8_bfloat16", "int16"};
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
    if (const char* v = getenv("B2W_GEMM_IMPL")) m->use_ref_gemm = !strcmp(v, "ref");
    if (const char* v = getenv("B2W_ATTN_IMPL")) m->use_ref_attn = !strcmp(v, "ref");
    if (const char* v = getenv("B2W_GEMV_IMPL")) m->use_ref_gemv = !strcmp(v, "ref");
    if (const char* v = getenv("B2W_GRAPH")) m->use_graph = strcmp(v, "0") != 0;
    m->w8 = ct.rfind("int8", 0) == 0;
    if (const char* v = getenv("B2W_W8_FAKE")) {
      if (strcmp(v, "0") != 0) {
        m->w8_fake = true;
        m->w8 = false;
      }
    }
    if (const char* v = getenv("B2W_DSTEP")) {
      m->use_dstep = strcmp(v, "0") != 0;
    }
    if (const char* v = getenv("B2W_BSTEP")) {
      m->use_bstep = strcmp(v, "0") != 0;
      m->bstep_all = strcmp(v, "all") == 0;
    }
    if (const char* v = getenv("B2W_BSTEP_STOP")) m->bstep_stop = atoi(v);
    if (const char* v = getenv("B2W_XATTN_IMPL")) m->use_mma_xattn = strcmp(v, "simt") != 0;
    if (const char* v = getenv("B2W_DSTEP_PROF")) {
      if (strcmp(v, "0") != 0) {
        m->d_prof = dalloc<unsigned long long>(4096);
        B2W_CUDA(cudaMemset(m->d_prof, 0, 4096 * sizeof(unsigned long long)));
      }
    }
    TensorTable tt{tensors, n_tensors};
    build_model(m, *cfg, tt);
    *out = h.release();
  });
}

void b2w_model_destroy(b2w_model* m) { delete m; }

int b2w_model_info(const b2w_model* m, b2w_config* cfg_out, int32_t* device_out) {
  return guarded([&] {
    B2W_CHECK(m, "null model");
    if (cfg_out) *cfg_out = m->m.cfg;
    if (device_out) *device_out = m->m.device;
  });
}

int b2w_model_sync(b2w_model* h) {
  return guarded([&] {
    B2W_CHECK(h, "null model");
    DeviceGuard g(h->m.device);
    B2W_CUDA(cudaStreamSynchronize(h->m.stream));
  });
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
    float* d_pcm = dalloc<float>(n_samples);
    float* d_out = dalloc<float>((size_t)n_frames * n_mels);
    MelChunkDesc* d_desc = dalloc<MelChunkDesc>(1);
    int* d_max = dalloc<int>(1);
    try {
      if (n_samples) B2W_CUDA(cudaMemcpyAsync(d_pcm, pcm, n_samples * 4, cudaMemcpyHostToDevice, s));
      MelChunkDesc desc{d_pcm, n_samples, n_frames, n_frames};
      B2W_CUDA(cudaMemcpyAsync(d_desc, &desc, sizeof desc, cudaMemcpyHostToDevice, s));
      plan->run(d_desc, 1, n_frames, padding, d_out, 0, n_frames, d_max, false, s);
      B2W_CUDA(cudaMemcpyAsync(out, d_out, (size_t)n_frames * n_mels * 4, cudaMemcpyDeviceToHost, s));
      B2W_CUDA(cudaStreamSynchronize(s));
    } catch (...) {
      cudaFree(d_pcm); cudaFree(d_out); cudaFree(d_desc); cudaFree(d_max); cudaStreamDestroy(s);
      throw;
    }
    cudaFree(d_pcm); cudaFree(d_out); cudaFree(d_desc); cudaFree(d_max); cudaStreamDestroy(s);
  });
}

int b2w_encode(b2w_model* h, const float* features, int32_t batch, b2w_encoded** out) {
  return guarded([&] {
    B2W_CHECK(h && features && out && batch > 0, "bad encode arguments");
    Model* m = &h->m;
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    const int64_t before = g_launches;
    std::unique_ptr<b2w_encoded> r(new b2w_encoded);
    r->e = encode_features(m, features, nullptr, batch);
    m->launches += g_launches - before;
    *out = r.release();
  });
}

int b2w_encode_audio(b2w_model* h, const float* const* pcm, const int64_t* n_samples, int32_t batch, float* features_out,
                     b2w_encoded** out) {
  return guarded([&] {
    B2W_CHECK(h && pcm && n_samples && out && batch > 0, "bad encode_audio arguments");
    Model* m = &h->m;
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    const int64_t before = g_launches;
    const int n_mels = m->cfg.n_mels;
    const size_t per = (size_t)n_mels * 3000, d = m->cfg.n_audio_state;
    std::unique_ptr<Encoded> e(new Encoded);
    e->owner = m;
    e->B = batch;
    e->enc_bytes = (size_t)batch * 1500 * d * sizeof(__half);
    e->enc_out = reinterpret_cast<__half*>(m->pool_get(e->enc_bytes));
    for (int b0 = 0; b0 < batch; b0 += kEncSub) {
      const int b = std::min(kEncSub, batch - b0);
      ensure_encoder_ws(m, std::min(kEncSub, (int)batch));
      size_t total = 0;
      for (int i = 0; i < b; ++i) {
        B2W_CHECK(n_samples[b0 + i] >= 0 && n_samples[b0 + i] <= 480000, "a chunk holds at most 30 s of 16 kHz audio");
        total += (n_samples[b0 + i] + 3) & ~size_t(3);
      }
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
      ScopedStage st(m, B2W_T_ENCODER);
      encoder_forward(m, b, e->enc_out + (size_t)b0 * 1500 * d);
    }
    m->launches += g_launches - before;
    std::unique_ptr<b2w_encoded> r(new b2w_encoded);
    r->e = e.release();
    *out = r.release();
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
  return guarded([&] {
    B2W_CHECK(h && e && e->e && out, "bad arguments");
    Model* m = &h->m;
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    const size_t n = (size_t)e->e->B * 1500 * m->cfg.n_audio_state;
    float* tmp = dalloc<float>(n);
    convert_f16_f32(e->e->enc_out, tmp, n, m->stream);
    B2W_CUDA(cudaMemcpyAsync(out, tmp, n * 4, cudaMemcpyDeviceToHost, m->stream));
    B2W_CUDA(cudaStreamSynchronize(m->stream));
    cudaFree(tmp);
  });
}

void b2w_encoded_free(b2w_encoded* e) {
  if (!e) return;
  if (e->e) {
    Model* m = e->e->owner;
    std::lock_guard<std::mutex> lk(m->mu);
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->stream);
    delete e->e;
  }
  delete e;
}

int b2w_generate(b2w_model* h, b2w_encoded* enc, const int32_t* prompts, int32_t prompt_len, int32_t batch,
                 const b2w_gen_opts* opts, int32_t* out_ids, int32_t* out_lens, float* out_scores, float* out_no_speech) {
  return guarded([&] {
    B2W_CHECK(h && prompts && opts && out_ids && out_lens && out_scores && out_no_speech, "null argument");
    Model* m = &h->m;
    const b2w_gen_opts& o = *opts;
    B2W_CHECK(batch > 0 && prompt_len > 0, "empty batch or prompt");
    B2W_CHECK(o.debug_fake_logits || (enc && enc->e && enc->e->B == batch), "one prompt per encoder output row is required");
    B2W_CHECK(o.beam_size >= 1 && o.beam_size <= kMaxBeam, "beam_size must be in 1..16");
    B2W_CHECK(o.num_hypotheses >= 1 && o.num_hypotheses <= kMaxBeam, "num_hypotheses must be in 1..16");
    B2W_CHECK(o.beam_size == 1 || o.num_hypotheses <= o.beam_size, "num_hypotheses must be <= beam_size");
    B2W_CHECK(o.max_length >= 1 && o.max_length <= m->cfg.n_text_ctx, "max_length must be in 1..n_text_ctx");
    B2W_CHECK(o.sampling_topk == 0 || o.sampling_topk == 1, "sampling_topk must be 0 (full vocabulary) or 1 (argmax)");
    B2W_CHECK(o.patience > 0 && o.repetition_penalty > 0, "patience and repetition_penalty must be positive");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    const int64_t before = g_launches;
    const int K = o.beam_size > 1 ? o.beam_size : std::max(1, o.num_hypotheses);
    const int group = std::max(1, kMaxRows / K);
    // suppress mask
    {
      std::vector<uint8_t> mask(m->vpad, 0);
      for (int i = m->cfg.n_vocab; i < m->vpad; ++i) mask[i] = 1;
      for (int i = 0; i < o.n_suppress_tokens; ++i) {
        const int t = o.suppress_tokens[i];
        if (t >= 0 && t < m->cfg.n_vocab) mask[t] = 1;
      }
      B2W_CUDA(cudaMemcpyAsync(m->d_suppress, mask.data(), m->vpad, cudaMemcpyHostToDevice, m->stream));
      B2W_CUDA(cudaStreamSynchronize(m->stream));
    }
    ensure_decoder_ws(m, std::min(group, (int)batch), K);
    ensure_search_ws(m, std::min(group, (int)batch), K);
    m->sb.suppress = m->d_suppress;
    std::unique_ptr<Encoded> dummy;
    Encoded* e = enc ? enc->e : nullptr;
    if (!o.debug_fake_logits) ensure_cross_kv(m, e);
    for (int c0 = 0; c0 < batch; c0 += group) {
      const int n = std::min(group, batch - c0);
      generate_group(m, e, c0, n, prompts, prompt_len, o, out_ids, out_lens, out_scores, out_no_speech);
    }
    m->launches += g_launches - before;
  });
}

int b2w_detect_language(b2w_model* h, b2w_encoded* enc, float* probs) {
  return guarded([&] {
    B2W_CHECK(h && enc && enc->e && probs, "null argument");
    Model* m = &h->m;
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    const int64_t before = g_launches;
    Encoded* e = enc->e;
    const int nl = m->cfg.num_languages;
    ensure_cross_kv(m, e);
    const int group = kMaxRows;
    ensure_decoder_ws(m, std::min(group, e->B), 1);
    ensure_search_ws(m, std::min(group, e->B), 1);
    float* d_probs = dalloc<float>((size_t)e->B * nl);
    std::vector<int32_t> toks(e->B, m->cfg.sot);
    for (int c0 = 0; c0 < e->B; c0 += group) {
      const int n = std::min(group, e->B - c0);
      B2W_CUDA(cudaMemsetAsync(m->sb.anc, 0, (size_t)2 * n * m->cfg.n_text_ctx, m->stream));
      prefill_pass(m, e, c0, n, toks.data(), 1, 0, 1, 1, 0);
      logits_gemm(m, n);
      lang_probs_from_logits(m->d_logits, m->vpad, n, m->cfg.lang_begin, nl, d_probs + (size_t)c0 * nl, m->stream);
    }
    B2W_CUDA(cudaMemcpyAsync(probs, d_probs, (size_t)e->B * nl * 4, cudaMemcpyDeviceToHost, m->stream));
    B2W_CUDA(cudaStreamSynchronize(m->stream));
    cudaFree(d_probs);
    m->launches += g_launches - before;
  });
}

// ---- Whisper.align: host-side post-processing (fp64) ------------------------------------------------------------------------
static void median_filter_rows(std::vector<double>& x, int rows, int cols, int width) {
  const int pad = width / 2;
  if (pad == 0 || cols <= pad) return;
  std::vector<double> row(cols + 2 * pad), win(width), out(cols);
  for (int r = 0; r < rows; ++r) {
    double* p = x.data() + (size_t)r * cols;
    for (int i = 0; i < pad; ++i) {  // reflect (edge sample not repeated)
      row[pad - 1 - i] = p[i + 1];
      row[pad + cols + i] = p[cols - 2 - i];
    }
    for (int i = 0; i < cols; ++i) row[pad + i] = p[i];
    for (int i = 0; i < cols; ++i) {
      for (int k = 0; k < width; ++k) win[k] = row[i + k];
      std::nth_element(win.begin(), win.begin() + pad, win.end());
      out[i] = win[pad];
    }
    for (int i = 0; i < cols; ++i) p[i] = out[i];
  }
}

// monotone minimal-cost path through cost[N][M]; moves diagonal / down / right with the reference tie rule
static void dtw_path(const std::vector<double>& c, int N, int M, std::vector<int>& ti, std::vector<int>& fi) {
  const double inf = std::numeric_limits<double>::infinity();
  std::vector<double> cost((size_t)(N + 1) * (M + 1), inf);
  std::vector<int8_t> trace((size_t)(N + 1) * (M + 1), -1);
  auto at = [&](int i, int j) { return (size_t)i * (M + 1) + j; };
  cost[0] = 0.0;
  for (int j = 1; j <= M; ++j)
    for (int i = 1; i <= N; ++i) {
      const double c0 = cost[at(i - 1, j - 1)], c1 = cost[at(i - 1, j)], c2 = cost[at(i, j - 1)];
      double best;
      int8_t t;
      if (c0 < c1 && c0 < c2) { best = c0; t = 0; }
      else if (c1 < c0 && c1 < c2) { best = c1; t = 1; }
      else { best = c2; t = 2; }
      cost[at(i, j)] = c[(size_t)(i - 1) * M + (j - 1)] + best;
      trace[at(i, j)] = t;
    }
  for (int j = 0; j <= M; ++j) trace[at(0, j)] = 2;
  for (int i = 0; i <= N; ++i) trace[at(i, 0)] = 1;
  int i = N, j = M;
  ti.clear();
  fi.clear();
  while (i > 0 || j > 0) {
    ti.push_back(i - 1);
    fi.push_back(j - 1);
    const int8_t t = trace[at(i, j)];
    if (t == 0) { --i; --j; }
    else if (t == 1) --i;
    else --j;
  }
  std::reverse(ti.begin(), ti.end());
  std::reverse(fi.begin(), fi.end());
}

int b2w_model_set_alignment_heads(b2w_model* h, const int32_t* layer_head_pairs, int32_t n_pairs) {
  return guarded([&] {
    B2W_CHECK(h && (n_pairs == 0 || layer_head_pairs) && n_pairs >= 0 && n_pairs <= 32 * 32, "bad arguments");
    Model* m = &h->m;
    std::lock_guard<std::mutex> lk(m->mu);
    std::vector<int2> v;
    for (int i = 0; i < n_pairs; ++i) {
      const int l = layer_head_pairs[2 * i], hd = layer_head_pairs[2 * i + 1];
      if (l < 0 || l >= m->cfg.n_text_layer || hd < 0 || hd >= m->cfg.n_text_head) throw Error("alignment head out of range", true);
      v.push_back(make_int2(l, hd));
    }
    if (v.empty())
      for (int l = m->cfg.n_text_layer / 2; l < m->cfg.n_text_layer; ++l)
        for (int hd = 0; hd < m->cfg.n_text_head; ++hd) v.push_back(make_int2(l, hd));
    m->align_heads = v;
    if (m->d_align_heads) {
      DeviceGuard g(m->device);
      cudaFree(m->d_align_heads);
      m->d_align_heads = nullptr;
    }
  });
}

int b2w_align(b2w_model* h, b2w_encoded* enc, int32_t batch_index, const int32_t* start_sequence, int32_t n_start,
              const int32_t* text_tokens, int32_t n_text, int32_t num_frames, int32_t median_filter_width, int32_t* alignments_out,
              int32_t capacity_pairs, int32_t* n_pairs_out, float* text_token_probs_out) {
  return guarded([&] {
    B2W_CHECK(h && enc && enc->e && start_sequence && n_pairs_out && n_start >= 1 && n_text >= 0, "bad arguments");
    Model* m = &h->m;
    const b2w_config& c = m->cfg;
    Encoded* e = enc->e;
    if (batch_index < 0 || batch_index >= e->B) throw Error("align: batch index out of range", true);
    if (median_filter_width < 1 || median_filter_width % 2 == 0) throw Error("align: median_filter_width must be odd", true);
    *n_pairs_out = 0;
    if (n_text == 0) return;
    B2W_CHECK(text_tokens && text_token_probs_out && (alignments_out || capacity_pairs == 0), "bad arguments");
    // forced sequence: start_sequence + <|notimestamps|> + text + <|endoftext|>
    std::vector<int32_t> seq(start_sequence, start_sequence + n_start);
    seq.push_back(c.no_timestamps);
    const int n_head_rows = (int)seq.size();
    seq.insert(seq.end(), text_tokens, text_tokens + n_text);
    seq.push_back(c.eot);
    const int n_tok = (int)seq.size();
    if (n_tok > c.n_text_ctx) throw Error("align: start sequence + text exceed the decoder context", true);
    for (int t : seq)
      if (t < 0 || t >= c.n_vocab) throw Error("align: token id out of range", true);
    const int nf = std::max(1, std::min(1500, (int)num_frames / 2));
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    cudaStream_t s = m->stream;
    ensure_cross_kv(m, e);
    ensure_decoder_ws(m, 1, 1);
    ensure_search_ws(m, 1, 1);
    const int n_heads = (int)m->align_heads.size();
    B2W_CHECK(n_heads > 0, "no alignment heads");
    if (!m->d_align_heads) {
      m->d_align_heads = dalloc<int2>(n_heads);
      B2W_CUDA(cudaMemcpy(m->d_align_heads, m->align_heads.data(), n_heads * sizeof(int2), cudaMemcpyHostToDevice));
    }
    const size_t n_att = (size_t)n_heads * n_tok * nf;
    float* d_att = reinterpret_cast<float*>(m->pool_get(n_att * sizeof(float)));
    int* d_targets = reinterpret_cast<int*>(m->pool_get((size_t)n_tok * sizeof(int)));
    float* d_tp = reinterpret_cast<float*>(m->pool_get((size_t)n_tok * sizeof(float)));
    std::vector<int> targets(n_tok, -1);
    for (int t = 0; t < n_text; ++t) targets[n_head_rows - 1 + t] = text_tokens[t];  // position p predicts token p + 1
    B2W_CUDA(cudaMemcpyAsync(d_targets, targets.data(), (size_t)n_tok * sizeof(int), cudaMemcpyHostToDevice, s));
    B2W_CUDA(cudaMemsetAsync(d_tp, 0, (size_t)n_tok * sizeof(float), s));
    B2W_CUDA(cudaMemsetAsync(m->sb.anc, 0, (size_t)2 * c.n_text_ctx, s));
    std::vector<int32_t> padded((size_t)(batch_index + 1) * n_tok, 0);  // prefill_pass indexes tokens by absolute chunk
    std::copy(seq.begin(), seq.end(), padded.begin() + (size_t)batch_index * n_tok);
    m->align_out = d_att;
    m->align_n_tok = n_tok;
    m->align_nf = nf;
    try {
      for (int i0 = 0; i0 < n_tok; i0 += kMaxRows) {
        const int i1 = std::min(n_tok, i0 + kMaxRows);
        m->align_pos0 = i0;
        prefill_pass(m, e, batch_index, 1, padded.data(), n_tok, i0, i1, 1, 0);
        logits_gemm(m, i1 - i0);
        row_target_probs(m->d_logits, m->vpad, i1 - i0, c.n_vocab, d_targets + i0, d_tp + i0, s);
      }
    } catch (...) {
      m->align_out = nullptr;
      throw;
    }
    m->align_out = nullptr;
    std::vector<float> att(n_att), tp(n_tok);
    B2W_CUDA(cudaMemcpyAsync(att.data(), d_att, n_att * sizeof(float), cudaMemcpyDeviceToHost, s));
    B2W_CUDA(cudaMemcpyAsync(tp.data(), d_tp, (size_t)n_tok * sizeof(float), cudaMemcpyDeviceToHost, s));
    B2W_CUDA(cudaStreamSynchronize(s));
    m->pool_put(d_att, n_att * sizeof(float));
    m->pool_put(d_targets, (size_t)n_tok * sizeof(int));
    m->pool_put(d_tp, (size_t)n_tok * sizeof(float));
    for (int t = 0; t < n_text; ++t) text_token_probs_out[t] = tp[n_head_rows - 1 + t];
    // per head: normalise over the token axis (population std), median filter along time; then the head mean
    std::vector<double> mean_w((size_t)n_tok * nf, 0.0), w((size_t)n_tok * nf);
    for (int hd = 0; hd < n_heads; ++hd) {
      const float* a = att.data() + (size_t)hd * n_tok * nf;
      for (int f = 0; f < nf; ++f) {
        double mu = 0.0, var = 0.0;
        for (int t = 0; t < n_tok; ++t) mu += a[(size_t)t * nf + f];
        mu /= n_tok;
        for (int t = 0; t < n_tok; ++t) {
          const double dlt = a[(size_t)t * nf + f] - mu;
          var += dlt * dlt;
        }
        const double sd = std::sqrt(var / n_tok);
        for (int t = 0; t < n_tok; ++t) w[(size_t)t * nf + f] = (a[(size_t)t * nf + f] - mu) / sd;
      }
      median_filter_rows(w, n_tok, nf, median_filter_width);
      for (size_t i = 0; i < w.size(); ++i) mean_w[i] += w[i];
    }
    // rows of the inputs that predict text + eot (drop the start-sequence rows and the eot input row: the consumer indexes
    // word boundaries up to n_text, transcribe.py:1744-1746), negated, DTW
    const int n_rows = n_text + 1;
    std::vector<double> cost((size_t)n_rows * nf);
    for (int t = 0; t < n_rows; ++t)
      for (int f = 0; f < nf; ++f) cost[(size_t)t * nf + f] = -mean_w[(size_t)(n_start + t) * nf + f] / n_heads;
    std::vector<int> ti, fi;
    dtw_path(cost, n_rows, nf, ti, fi);
    *n_pairs_out = (int32_t)ti.size();
    if ((int)ti.size() > capacity_pairs) throw Error("align: alignment buffer too small", true);
    for (size_t i = 0; i < ti.size(); ++i) {
      alignments_out[2 * i] = ti[i];
      alignments_out[2 * i + 1] = fi[i];
    }
  });
}

int b2w_span_begin(b2w_model* h) {
  return guarded([&] {
    B2W_CHECK(h, "bad arguments");
    Model* m = &h->m;
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    if (!m->span_a) {
      B2W_CUDA(cudaEventCreate(&m->span_a));
      B2W_CUDA(cudaEventCreate(&m->span_b));
    }
    B2W_CUDA(cudaEventRecord(m->span_a, m->stream));
  });
}
int b2w_span_end(b2w_model* h, double* ms_out) {
  return guarded([&] {
    B2W_CHECK(h && ms_out && h->m.span_a, "b2w_span_end without b2w_span_begin");
    Model* m = &h->m;
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    B2W_CUDA(cudaEventRecord(m->span_b, m->stream));
    B2W_CUDA(cudaEventSynchronize(m->span_b));
    float ms = 0.f;
    B2W_CUDA(cudaEventElapsedTime(&ms, m->span_a, m->span_b));
    *ms_out = ms;
  });
}

int b2w_timing_enable(b2w_model* h, int32_t on) {
  return guarded([&] {
    B2W_CHECK(h, "null model");
    drain_timers(&h->m);
    h->m.timing = on != 0;
  });
}
int b2w_timing_reset(b2w_model* h) {
  return guarded([&] {
    B2W_CHECK(h, "null model");
    DeviceGuard g(h->m.device);
    drain_timers(&h->m);
    for (int i = 0; i < B2W_T_COUNT; ++i) {
      h->m.t_ms[i] = 0;
      h->m.t_cnt[i] = 0;
    }
    h->m.launches = 0;
    h->m.decode_steps = 0;
    h->m.decode_alg_bytes = 0;
  });
}
int b2w_timing_get(b2w_model* h, double ms_out[B2W_T_COUNT], int64_t counts_out[B2W_T_COUNT]) {
  return guarded([&] {
    B2W_CHECK(h, "null model");
    DeviceGuard g(h->m.device);
    drain_timers(&h->m);
    for (int i = 0; i < B2W_T_COUNT; ++i) {
      ms_out[i] = h->m.t_ms[i];
      if (counts_out) counts_out[i] = h->m.t_cnt[i];
    }
  });
}
int b2w_counters_get(b2w_model* h, int64_t* launches, int64_t* decode_steps, double* decode_alg_bytes) {
  return guarded([&] {
    B2W_CHECK(h, "null model");
    if (launches) *launches = h->m.launches;
    if (decode_steps) *decode_steps = h->m.decode_steps;
    if (decode_alg_bytes) *decode_alg_bytes = h->m.decode_alg_bytes;
  });
}

// ---- test hooks -------------------------------------------------------------------------------------------------------
int b2w_debug_gemm(int32_t device, int32_t impl, const float* a, const float* w, const float* bias, int32_t M, int32_t N,
                   int32_t K, int32_t gelu, float* c_out) {
  return guarded([&] {
    require_hopper(device);
    DeviceGuard g(device);
    cudaDeviceProp prop;
    B2W_CUDA(cudaGetDeviceProperties(&prop, device));
    float *da = dalloc<float>((size_t)M * K), *dw = dalloc<float>((size_t)N * K), *db = dalloc<float>(N);
    __half *ha = dalloc<__half>((size_t)M * K), *hw = dalloc<__half>((size_t)N * K), *hc = dalloc<__half>((size_t)M * N);
    float* dc = dalloc<float>((size_t)M * N);
    B2W_CUDA(cudaMemcpy(da, a, (size_t)M * K * 4, cudaMemcpyHostToDevice));
    B2W_CUDA(cudaMemcpy(dw, w, (size_t)N * K * 4, cudaMemcpyHostToDevice));
    if (bias) B2W_CUDA(cudaMemcpy(db, bias, (size_t)N * 4, cudaMemcpyHostToDevice));
    convert_f32_f16(da, ha, (int64_t)M * K, 0);
    convert_f32_f16(dw, hw, (int64_t)N * K, 0);
    GemmArgs ga;
    ga.A = ha; ga.a_batch = 1; ga.a_rows = M; ga.a_cols = K; ga.a_row_stride = K; ga.k_per_tap = K;
    ga.W = hw; ga.N = N; ga.rows = M; ga.bias = bias ? db : nullptr;
    if (gelu) {
      ga.out = hc; ga.out_ld = N; ga.epilogue = EPI_GELU_F16;
    } else {
      ga.out = dc; ga.out_ld = N; ga.epilogue = EPI_F32;
    }
    if (impl == 0) {
      gemm_configure();  // per-device kernel attributes (build_model does this for real models)
      GemmPlan p = gemm_plan(ga, prop.multiProcessorCount);
      gemm_run(p, 0);
    } else {
      gemm_ref_run(ga, 0);
    }
    if (gelu) convert_f16_f32(hc, dc, (int64_t)M * N, 0);
    B2W_CUDA(cudaDeviceSynchronize());
    B2W_CUDA(cudaMemcpy(c_out, dc, (size_t)M * N * 4, cudaMemcpyDeviceToHost));
    cudaFree(da); cudaFree(dw); cudaFree(db); cudaFree(ha); cudaFree(hw); cudaFree(hc); cudaFree(dc);
  });
}

int b2w_debug_attention(int32_t device, int32_t impl, const float* qkv, int32_t B, int32_t T, int32_t H, float* out) {
  return guarded([&] {
    require_hopper(device);
    DeviceGuard g(device);
    const size_t n_in = (size_t)B * T * 3 * H * 64, n_out = (size_t)B * T * H * 64;
    float *dq = dalloc<float>(n_in), *dof = dalloc<float>(n_out);
    __half *hq = dalloc<__half>(n_in), *ho = dalloc<__half>(n_out);
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
    cudaFree(dq); cudaFree(dof); cudaFree(hq); cudaFree(ho);
  });
}

int b2w_debug_gemv(int32_t device, int32_t impl, const float* x, const float* w, const float* bias, int32_t R, int32_t N,
                   int32_t K, float* y_out) {
  return guarded([&] {
    require_hopper(device);
    DeviceGuard g(device);
    const int Np = ceil_div(N, 16) * 16, Rp = ceil_div(R, 8) * 8;
    float *dx = dalloc<float>((size_t)Rp * K), *dw = dalloc<float>((size_t)Np * K), *db = dalloc<float>(Np), *dy = dalloc<float>((size_t)R * Np);
    __half *hx = dalloc<__half>((size_t)Rp * K), *hw = dalloc<__half>((size_t)Np * K);
    B2W_CUDA(cudaMemset(dx, 0, (size_t)Rp * K * 4));
    B2W_CUDA(cudaMemset(dw, 0, (size_t)Np * K * 4));
    B2W_CUDA(cudaMemset(db, 0, (size_t)Np * 4));
    B2W_CUDA(cudaMemcpy(dx, x, (size_t)R * K * 4, cudaMemcpyHostToDevice));
    B2W_CUDA(cudaMemcpy(dw, w, (size_t)N * K * 4, cudaMemcpyHostToDevice));
    if (bias) B2W_CUDA(cudaMemcpy(db, bias, (size_t)N * 4, cudaMemcpyHostToDevice));
    convert_f32_f16(dx, hx, (int64_t)Rp * K, 0);
    convert_f32_f16(dw, hw, (int64_t)Np * K, 0);
    if (impl == 0) {
      GvArgs a;
      a.x = hx; a.W = hw; a.bias = bias ? db : nullptr; a.R = R; a.N = Np; a.K = K; a.mode = GV_F32; a.out_f = dy; a.ldo = Np;
      skinny_gemm(a, 0);
    } else {
      skinny_ref(hx, hw, bias ? db : nullptr, dy, R, Np, K, 0);
    }
    B2W_CUDA(cudaDeviceSynchronize());
    std::vector<float> tmp((size_t)R * Np);
    B2W_CUDA(cudaMemcpy(tmp.data(), dy, tmp.size() * 4, cudaMemcpyDeviceToHost));
    for (int r = 0; r < R; ++r) memcpy(y_out + (size_t)r * N, tmp.data() + (size_t)r * Np, (size_t)N * 4);
    cudaFree(dx); cudaFree(dw); cudaFree(db); cudaFree(dy); cudaFree(hx); cudaFree(hw);
  });
}

int b2w_debug_fetch(b2w_model* h, int32_t which, float* out, int64_t n) {
  return guarded([&] {
    B2W_CHECK(h && out && n >= 0, "null argument");
    Model* m = &h->m;
    DeviceGuard g(m->device);
    B2W_CHECK(m->d_x, "no decoder workspace yet");
    B2W_CUDA(cudaStreamSynchronize(m->stream));
    const float* f32 = nullptr;
    const __half* f16 = nullptr;
    switch (which) {
      case 0: f32 = m->d_x; break;
      case 1: f32 = m->d_qkv32; break;
      case 2: f32 = m->d_cq32; break;
      case 3: f32 = m->d_h32; break;
      case 4: f16 = m->d_ao; break;
      case 5: f16 = m->d_h16; break;
      case 6: f16 = m->d_xn16; break;
      case 7: f32 = m->d_stats; break;
      case 8: f32 = m->d_logits; break;
      default: throw Error("b2w_debug_fetch: unknown buffer", true);
    }
    if (f32) {
      B2W_CUDA(cudaMemcpy(out, f32, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
    } else {
      std::vector<__half> tmp((size_t)n);
      B2W_CUDA(cudaMemcpy(tmp.data(), f16, (size_t)n * sizeof(__half), cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < n; ++i) out[i] = __half2float(tmp[(size_t)i]);
    }
  });
}

int b2w_debug_logits(b2w_model* h, b2w_encoded* enc, const int32_t* tokens, int32_t n_tok, int32_t batch, float* logits_out) {
  return guarded([&] {
    B2W_CHECK(h && enc && enc->e && tokens && logits_out && enc->e->B == batch, "bad arguments");
    Model* m = &h->m;
    B2W_CHECK(n_tok >= 1 && n_tok <= m->cfg.n_text_ctx, "token count");
    std::lock_guard<std::mutex> lk(m->mu);
    DeviceGuard g(m->device);
    Encoded* e = enc->e;
    ensure_cross_kv(m, e);
    const int V = m->cfg.n_vocab;
    const int group = std::min((int)batch, kMaxRows);
    ensure_decoder_ws(m, group, 1);
    ensure_search_ws(m, group, 1);
    std::vector<float> tmp((size_t)kMaxRows * m->vpad);
    for (int c0 = 0; c0 < batch; c0 += group) {
      const int n = std::min(group, batch - c0);
      B2W_CUDA(cudaMemsetAsync(m->sb.anc, 0, (size_t)2 * n * m->cfg.n_text_ctx, m->stream));
      const int per_pass = std::max(1, kMaxRows / n);
      for (int i0 = 0; i0 < n_tok; i0 += per_pass) {
        const int i1 = std::min((int)n_tok, i0 + per_pass), rpc = i1 - i0;
        prefill_pass(m, e, c0, n, tokens, n_tok, i0, i1, 1, 0);
        logits_gemm(m, n * rpc);
        B2W_CUDA(cudaMemcpyAsync(tmp.data(), m->d_logits, (size_t)n * rpc * m->vpad * 4, cudaMemcpyDeviceToHost, m->stream));
        B2W_CUDA(cudaStreamSynchronize(m->stream));
        for (int b = 0; b < n; ++b)
          for (int i = i0; i < i1; ++i)
            memcpy(logits_out + ((size_t)(c0 + b) * n_tok + i) * V, tmp.data() + (size_t)(b * rpc + i - i0) * m->vpad, (size_t)V * 4);
      }
    }
  });
}

}  // extern "C"
