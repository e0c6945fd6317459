// C-ABI layer of the fine-tuned text classifier (declared in include/issue_emb_b200.h): fastai text_classifier_learner
// (MultiBatchEncoder + PoolingLinearClassifier) in eval mode, over a borrowed encoder.
#include "encoder_host.h"

using namespace ie;

struct ie_clas {
  ie_encoder* enc = nullptr;  // borrowed: its weights, workspace, stream and error words
  int device = 0;
  std::vector<int> dims;      // {3*emb_sz, hidden..., n_class}
  int softmax = 0;
  struct Stage {
    DevBuf alpha, beta, w, b;  // BatchNorm folded to x*alpha + beta; Linear weight [N, K] and bias
    bool loaded = false;
  };
  std::vector<Stage> stages;
  long long raw_budget = 1ll << 32;  // bytes of f32 states one row group may hold (IE_CLAS_RAW_BUDGET at create time)
  DevBuf se, act[2], logits, probs, err;
  int64_t launches = 0;
  StreamOrder order;
  std::mutex mu;
};

namespace {

constexpr int kClasErrWords = 4;  // err[0] token id out of range, err[1] device wait timed out, err[2] bad window

int clas_max_width(const ie_clas* c) { return *std::max_element(c->dims.begin(), c->dims.end()); }

// the classifier's error words of the last call, then the encoder's (waits for the call; clears both)
int clas_collect(ie_clas* c) {
  if (!c->order.has_done) return IE_OK;
  const int rc_enc = collect_errors(c->enc);
  int w[kClasErrWords] = {0, 0, 0, 0};
  const int rc = read_errors(c->order, c->err, w, kClasErrWords);
  if (rc != IE_OK) return rc;
  if (rc_enc != IE_OK) return rc_enc;
  if (w[1] != 0) {
    c->enc->use_persistent = 0;
    return fail(IE_ERR_CUDA, "a device-side wait exceeded its limit and the kernel was drained; results of this call "
                             "are invalid");
  }
  if (w[0] != 0) return fail(IE_ERR_TOKEN, "token id outside [0,%d) in ids", c->enc->cfg.vocab_sz);
  if (w[2] != 0) return fail(IE_ERR_INVALID, "a window outside [0,T], empty or entirely pad was refused (NaN rows)");
  return IE_OK;
}

// encoder -> pool (-> head -> activation) over row groups of at most raw_budget bytes of states.  pooled_only: out
// [B, 3*emb_sz] receives the pool; else out [B, n_class] the activated output and logits (optional) the last Linear's.
int clas_run(ie_clas* c, const int64_t* ids, const int32_t* starts, const int32_t* ends, int B, int T, float* out,
             float* logits, bool pooled_only, int flags, void* stream) {
  if (c == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (ids == nullptr || starts == nullptr || ends == nullptr || out == nullptr) return fail(IE_ERR_INVALID, "null pointer");
  ie_encoder* h = c->enc;
  if (B < 1 || B > h->max_batch) return fail(IE_ERR_INVALID, "B=%d outside [1,%d]", B, h->max_batch);
  if (T < 1) return fail(IE_ERR_INVALID, "T=%d must be >= 1", T);
  if (!pooled_only)
    for (size_t k = 0; k < c->stages.size(); ++k)
      if (!c->stages[k].loaded) return fail(IE_ERR_STATE, "head stage %zu not loaded", k);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  const int pad = h->cfg.pad_idx;
  if (!dev) {  // every window is checked before anything is launched
    for (int b = 0; b < B; ++b) {
      if (starts[b] < 0 || ends[b] > T || starts[b] >= ends[b])
        return fail(IE_ERR_INVALID, "window [%d,%d) of row %d is empty or outside [0,%d]", starts[b], ends[b], b, T);
      const int64_t* id = ids + static_cast<long long>(b) * T;
      if (std::all_of(id + starts[b], id + ends[b], [pad](int64_t v) { return v == pad; }))
        return fail(IE_ERR_INVALID, "window [%d,%d) of row %d is entirely pad (fastai would pool NaN / -inf)",
                    starts[b], ends[b], b);
    }
  }
  std::scoped_lock lk(c->mu, h->mu);
  cudaStream_t s = call_stream(flags, stream, h->own_stream);
  CK(cudaSetDevice(h->cfg.device));
  const int E = h->cfg.emb_sz, n_class = c->dims.back(), width = pooled_only ? 3 * E : n_class;
  const Layer& LL = h->layers.back();
  const long long row_bytes = static_cast<long long>(T) * LL.out_pad * sizeof(float);
  const int g = static_cast<int>(std::max(1ll, std::min<long long>(B, c->raw_budget / row_bytes)));
  CK(c->se.reserve(2ull * h->max_batch * sizeof(int)));
  CK(c->act[0].reserve(static_cast<size_t>(g) * clas_max_width(c) * sizeof(float)));
  CK(c->act[1].reserve(static_cast<size_t>(g) * clas_max_width(c) * sizeof(float)));
  CK(c->logits.reserve(static_cast<size_t>(h->max_batch) * n_class * sizeof(float)));
  CK(c->probs.reserve(static_cast<size_t>(h->max_batch) * std::max(3 * E, n_class) * sizeof(float)));
  CK(c->err.reserve(kClasErrWords * sizeof(int), true));
  CK(c->order.begin(s));
  CK(cudaMemsetAsync(c->err.p, 0, kClasErrWords * sizeof(int), s));
  const int* st = starts;
  const int* en = ends;
  if (!dev) {
    CK(cudaMemcpyAsync(c->se.p, starts, B * sizeof(int), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(c->se.as<int>() + h->max_batch, ends, B * sizeof(int), cudaMemcpyHostToDevice, s));
    st = c->se.as<int>();
    en = c->se.as<int>() + h->max_batch;
  }
  float* out_dev = dev ? out : c->probs.as<float>();
  float* logits_dev = (dev && logits != nullptr) ? logits : c->logits.as<float>();
  for (int b0 = 0; b0 < B; b0 += g) {
    const int nb = std::min(g, B - b0);
    const int64_t* ids_g = ids + static_cast<long long>(b0) * T;
    long long t_need = 0;
    int rc = run_encoder(h, ids_g, nullptr, nb, T, nullptr, nullptr, h->cfg.n_layers - 1, flags, s, &t_need);
    if (rc != IE_OK) return rc;
    const int64_t* ids_dev = dev ? ids_g : h->ids.as<int64_t>();
    float* pooled = pooled_only ? out_dev + static_cast<long long>(b0) * 3 * E : c->act[0].as<float>();
    CK(ie::launch_clas_pool(h->raw.as<float>(), LL.out_pad, nb, T, ids_dev, st + b0, en + b0, E, pad, pooled,
                            h->err.as<int>(), c->err.as<int>(), s));
    c->launches++;
    if (!pooled_only) {
      const int n_st = static_cast<int>(c->stages.size());
      float* z = logits_dev + static_cast<long long>(b0) * n_class;
      for (int k = 0; k < n_st; ++k) {
        const ie_clas::Stage& S = c->stages[k];
        const bool last = k == n_st - 1;
        float* y = last ? z : c->act[(k + 1) & 1].as<float>();
        CK(ie::launch_clas_linear(c->act[k & 1].as<float>(), nb, c->dims[k], S.alpha.as<float>(), S.beta.as<float>(),
                                  S.w.as<float>(), S.b.as<float>(), c->dims[k + 1], last ? 0 : 1, y, s));
        c->launches++;
      }
      CK(ie::launch_clas_activate(z, nb, n_class, c->softmax, out_dev + static_cast<long long>(b0) * n_class, s));
      c->launches++;
    }
    // the encoder's workspace (states, ids) is read up to here: its next call, on any stream, waits for this point
    CK(h->order.end(s));
    if ((rc = maybe_release_workspace(h, t_need, s)) != IE_OK) return rc;
  }
  if (!dev) {
    CK(cudaMemcpyAsync(out, out_dev, static_cast<size_t>(B) * width * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (logits != nullptr && !pooled_only)
      CK(cudaMemcpyAsync(logits, logits_dev, static_cast<size_t>(B) * n_class * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  CK(c->order.end(s));
  if (dev) return IE_OK;
  return clas_collect(c);
}

}  // namespace

extern "C" {

int ie_clas_window(int32_t sl, int32_t bptt, int32_t max_len, int32_t* start) {
  if (start == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (sl < 1 || bptt < 1 || max_len < 1) return fail(IE_ERR_INVALID, "sl=%d, bptt=%d, max_len=%d must be >= 1", sl, bptt, max_len);
  // chunks i = 0, bptt, 2 bptt, ... < sl are kept when i > sl - max_len: the first kept one is the least multiple of bptt
  // above sl - max_len
  const long long d = static_cast<long long>(sl) - max_len;
  const long long s = d < 0 ? 0 : (d / bptt + 1) * bptt;
  if (s >= sl)
    return fail(IE_ERR_INVALID, "no chunk of bptt=%d is kept at sl=%d with max_len=%d (max_len <= bptt)", bptt, sl, max_len);
  *start = static_cast<int32_t>(s);
  return IE_OK;
}

int ie_clas_create(ie_encoder* enc, int32_t n_stages, const int32_t* dims, int32_t activation, ie_clas** out) {
  if (enc == nullptr || dims == nullptr || out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (n_stages < 1 || n_stages > 16) return fail(IE_ERR_INVALID, "n_stages=%d outside [1,16]", n_stages);
  if (activation != IE_CLAS_SIGMOID && activation != IE_CLAS_SOFTMAX)
    return fail(IE_ERR_INVALID, "activation %d is neither IE_CLAS_SIGMOID nor IE_CLAS_SOFTMAX", activation);
  if (dims[0] != 3 * enc->cfg.emb_sz)
    return fail(IE_ERR_INVALID, "head input width %d != 3 * emb_sz = %d", dims[0], 3 * enc->cfg.emb_sz);
  for (int k = 0; k <= n_stages; ++k)
    if (dims[k] < 1 || dims[k] > (1 << 20)) return fail(IE_ERR_INVALID, "dims[%d]=%d outside [1,2^20]", k, dims[k]);
  ie_clas* c = new ie_clas();
  c->enc = enc;
  c->device = enc->cfg.device;
  c->dims.assign(dims, dims + n_stages + 1);
  c->softmax = activation == IE_CLAS_SOFTMAX;
  c->stages.resize(n_stages);
  if (const char* v = getenv("IE_CLAS_RAW_BUDGET")) c->raw_budget = std::max(1ll, atoll(v));
  *out = c;
  return IE_OK;
}

void ie_clas_destroy(ie_clas* c) {
  if (c == nullptr) return;
  cudaSetDevice(c->device);
  c->order.wait();
  delete c;
}

int ie_clas_load_stage(ie_clas* c, int32_t stage, const float* bn_weight, const float* bn_bias, const float* bn_mean,
                       const float* bn_var, double eps, const float* lin_weight, const float* lin_bias) {
  if (c == nullptr || bn_mean == nullptr || bn_var == nullptr || lin_weight == nullptr || lin_bias == nullptr)
    return fail(IE_ERR_INVALID, "null argument");
  if (stage < 0 || stage >= static_cast<int>(c->stages.size())) return fail(IE_ERR_INVALID, "stage %d out of range", stage);
  if (!(eps >= 0.0) || !std::isfinite(eps)) return fail(IE_ERR_INVALID, "eps must be finite and >= 0");
  const int K = c->dims[stage], N = c->dims[stage + 1];
  // torch's eval BatchNorm1d on the CPU (batch_norm_cpu_collect_linear_and_constant_terms): invstd = 1 / sqrt(var + eps),
  // alpha = invstd * weight, beta = bias - mean * alpha (one rounding), y = x * alpha + beta (one rounding), all in f32
  std::vector<float> alpha(K), beta(K);
  const float eps_f = static_cast<float>(eps);
  for (int k = 0; k < K; ++k) {
    const float var = bn_var[k] + eps_f;
    if (!(var > 0.0f) || !std::isfinite(var) || !std::isfinite(bn_mean[k]))
      return fail(IE_ERR_INVALID, "stage %d: running statistics of column %d are not finite or var + eps <= 0", stage, k);
    const float invstd = 1.0f / std::sqrt(var);
    alpha[k] = invstd * (bn_weight ? bn_weight[k] : 1.0f);
    beta[k] = std::fma(-bn_mean[k], alpha[k], bn_bias ? bn_bias[k] : 0.0f);
    if (!std::isfinite(alpha[k]) || !std::isfinite(beta[k]))
      return fail(IE_ERR_INVALID, "stage %d: BatchNorm column %d is not finite", stage, k);
  }
  for (long long i = 0; i < static_cast<long long>(N) * K; ++i)
    if (!std::isfinite(lin_weight[i])) return fail(IE_ERR_INVALID, "stage %d: Linear weight is not finite", stage);
  for (int j = 0; j < N; ++j)
    if (!std::isfinite(lin_bias[j])) return fail(IE_ERR_INVALID, "stage %d: Linear bias is not finite", stage);
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->enc->cfg.device));
  CK(c->order.wait());  // an earlier call may still read this stage
  ie_clas::Stage& S = c->stages[stage];
  CK(S.alpha.reserve(K * sizeof(float)));
  CK(S.beta.reserve(K * sizeof(float)));
  CK(S.w.reserve(static_cast<size_t>(N) * K * sizeof(float)));
  CK(S.b.reserve(N * sizeof(float)));
  CK(cudaMemcpy(S.alpha.p, alpha.data(), K * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(S.beta.p, beta.data(), K * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(S.w.p, lin_weight, static_cast<size_t>(N) * K * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(S.b.p, lin_bias, N * sizeof(float), cudaMemcpyHostToDevice));
  S.loaded = true;
  return IE_OK;
}

int ie_clas_forward(ie_clas* c, const int64_t* ids, const int32_t* starts, const int32_t* ends, int32_t B, int32_t T,
                    float* out, float* logits, int32_t flags, void* stream) {
  return clas_run(c, ids, starts, ends, B, T, out, logits, false, flags, stream);
}

int ie_clas_pool(ie_clas* c, const int64_t* ids, const int32_t* starts, const int32_t* ends, int32_t B, int32_t T,
                 float* pooled, int32_t flags, void* stream) {
  return clas_run(c, ids, starts, ends, B, T, pooled, nullptr, true, flags, stream);
}

int ie_clas_check_errors(ie_clas* c) {
  if (c == nullptr) return fail(IE_ERR_INVALID, "null handle");
  std::scoped_lock lk(c->mu, c->enc->mu);
  CK(cudaSetDevice(c->enc->cfg.device));
  return clas_collect(c);
}

int64_t ie_clas_launch_count(const ie_clas* c) { return c ? c->launches : -1; }

}  // extern "C"
