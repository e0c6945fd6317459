// C-ABI layer of the MLP head (declared in include/issue_emb_b200.h): the sklearn MLPClassifier forward pass on the
// persistent GEMM, and the precision-recall threshold search over its scores.
#include "encoder_host.h"

using namespace ie;

struct ie_mlp {
  int device = 0;
  int num_sms = 132;
  std::vector<int> dims;
  struct L {
    int k_pad = 0, n_pad = 0, bn = 0;
    DevBuf w, b;
    bool loaded = false;
  };
  std::vector<L> layers;
  DevBuf xf, act[2], probs;
  DevBuf xb;                // bf16 copy of one row chunk of X
  long long act_ld = 0;
  int chunk_dev = 1 << 18;  // rows per pass in device-pointer mode (IE_MLP_CHUNK at create time)
  cudaStream_t own_stream = nullptr;
  std::mutex mu;
};

extern "C" {

int ie_mlp_create(int32_t n_layers, const int32_t* dims, int32_t device, ie_mlp** out) {
  if (dims == nullptr || out == nullptr || n_layers < 1 || n_layers > 16) return fail(IE_ERR_INVALID, "bad argument");
  for (int i = 0; i <= n_layers; ++i)
    if (dims[i] < 1) return fail(IE_ERR_INVALID, "dims[%d]=%d", i, dims[i]);
  int sms = 0;
  const int rc = open_device(device, &sms);
  if (rc != IE_OK) return rc;
  ie_mlp* m = new ie_mlp();
  m->device = device;
  m->num_sms = sms;
  m->dims.assign(dims, dims + n_layers + 1);
  m->layers.resize(n_layers);
  long long ld = 64;
  for (int l = 0; l < n_layers; ++l) {
    ie_mlp::L& L = m->layers[l];
    L.k_pad = static_cast<int>(round_up(dims[l], 64));
    // N padding: the GEMM's tiles are 256 wide (a 600-wide hidden layer is padded to 768 = 3 tiles), narrow layers are
    // padded to 16 columns and the rest of their single tile reads zero weights
    const int n16 = static_cast<int>(round_up(dims[l + 1], 16));
    L.bn = n16 >= 256 ? 256 : n16;
    L.n_pad = static_cast<int>(round_up(dims[l + 1], L.bn));
    ld = std::max<long long>(ld, round_up(std::max(L.n_pad, L.k_pad), 64));
  }
  m->act_ld = ld;
  if (const char* v = getenv("IE_MLP_CHUNK")) m->chunk_dev = static_cast<int>(round_up(std::max(256, atoi(v)), 256));
  const cudaError_t e = cudaStreamCreateWithFlags(&m->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete m; return cuda_fail(e, "cudaStreamCreate"); }
  *out = m;
  return IE_OK;
}

int ie_mlp_load_layer(ie_mlp* m, int32_t layer, const float* coef, const float* intercept) {
  if (m == nullptr || coef == nullptr || intercept == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (layer < 0 || layer >= static_cast<int>(m->layers.size())) return fail(IE_ERR_INVALID, "layer out of range");
  std::lock_guard<std::mutex> lk(m->mu);
  CK(cudaSetDevice(m->device));
  ie_mlp::L& L = m->layers[layer];
  const int fan_in = m->dims[layer], fan_out = m->dims[layer + 1];
  // sklearn coefs_[l] is [fan_in, fan_out]; the GEMM wants B = [fan_out rows, fan_in] (K-major)
  std::vector<float> wt(static_cast<size_t>(fan_out) * fan_in);
  for (int i = 0; i < fan_in; ++i)
    for (int o = 0; o < fan_out; ++o) wt[static_cast<size_t>(o) * fan_in + i] = coef[static_cast<size_t>(i) * fan_out + o];
  int rc = upload_sliced(wt.data(), fan_out, fan_in, padded_identity(fan_out, L.n_pad), L.k_pad, 1, L.w, m->own_stream);
  if (rc != IE_OK) return rc;
  std::vector<float> b(L.n_pad, 0.0f);
  std::copy(intercept, intercept + fan_out, b.begin());
  CK(L.b.reserve(b.size() * sizeof(float)));
  CK(cudaMemcpy(L.b.p, b.data(), b.size() * sizeof(float), cudaMemcpyHostToDevice));
  L.loaded = true;
  return IE_OK;
}

int ie_mlp_predict_proba(ie_mlp* m, const float* X, int32_t n, float* probs, int32_t flags, void* stream) {
  if (m == nullptr || X == nullptr || probs == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (n < 1) return fail(IE_ERR_INVALID, "n=%d", n);
  for (const auto& L : m->layers)
    if (!L.loaded) return fail(IE_ERR_STATE, "MLP layer weights not loaded");
  std::lock_guard<std::mutex> lk(m->mu);
  CK(cudaSetDevice(m->device));
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  cudaStream_t s = call_stream(flags, stream, m->own_stream);
  const int nl = static_cast<int>(m->layers.size());
  const int d_in = m->dims[0], n_labels = m->dims[nl];
  // rows per pass: host buffers are staged through a 2^16-row device buffer; device pointers take chunk_dev rows
  int chunk = dev ? m->chunk_dev : (1 << 16);
  chunk = static_cast<int>(std::min<long long>(chunk, round_up(n, 256)));
  const ie_mlp::L& LL = m->layers[nl - 1];
  // the last GEMM writes straight into the caller's array when its row pitch is a legal store width
  const bool direct_out = dev && n_labels % 16 == 0 && n_labels == LL.n_pad;
  CK(m->act[0].reserve(static_cast<size_t>(chunk) * m->act_ld * sizeof(__nv_bfloat16), true));
  CK(m->act[1].reserve(static_cast<size_t>(chunk) * m->act_ld * sizeof(__nv_bfloat16), true));
  CK(m->xb.reserve(static_cast<size_t>(chunk) * m->act_ld * sizeof(__nv_bfloat16), true));
  if (!direct_out) CK(m->probs.reserve(static_cast<size_t>(chunk) * LL.n_pad * sizeof(float)));
  if (!dev) CK(m->xf.reserve(static_cast<size_t>(chunk) * d_in * sizeof(float)));
  for (long long r0 = 0; r0 < n; r0 += chunk) {
    const int rows = static_cast<int>(std::min<long long>(chunk, n - r0));
    // whole M = 128 tiles (rows past `rows` hold stale finite data and are never stored)
    const int m_pad = static_cast<int>(round_up(rows, 128));
    const float* xsrc = X + r0 * d_in;
    if (!dev) {
      CK(cudaMemcpyAsync(m->xf.p, xsrc, static_cast<size_t>(rows) * d_in * sizeof(float), cudaMemcpyHostToDevice, s));
      xsrc = m->xf.as<float>();
    }
    __nv_bfloat16* xbuf = m->xb.as<__nv_bfloat16>();
    CK(ie::launch_convert_rows(xsrc, d_in, d_in, nullptr, rows, xbuf, m->act_ld, 0, s));   // f32 -> bf16, K padded with zeros
    const __nv_bfloat16* cur_in = xbuf;
    int cur = 0;
    for (int l = 0; l < nl; ++l) {
      const ie_mlp::L& L = m->layers[l];
      const bool last = (l == nl - 1);
      ie::GemmArgs g{};
      g.a = cur_in;
      g.lda = m->act_ld;
      g.b = L.w.as<__nv_bfloat16>();
      g.ldb = L.k_pad;
      g.bias = L.b.as<float>();
      g.m_pad = m_pad;
      g.n_pad = L.n_pad;
      g.k_pad = L.k_pad;
      g.m_store = rows;
      g.n_store = L.n_pad;
      g.bn = L.bn;
      g.num_sms = m->num_sms;
      if (last) {
        g.d = direct_out ? static_cast<void*>(probs + r0 * n_labels) : m->probs.p;
        g.ldd = L.n_pad;
        g.act = 2;
        g.out_bf16 = 0;
      } else {
        g.d = m->act[cur].p;
        g.ldd = m->act_ld;
        g.act = 1;
        g.out_bf16 = 1;
      }
      CK(ie::launch_gemm_bf16(g, s));
      cur_in = m->act[cur].as<__nv_bfloat16>();
      cur ^= 1;
    }
    if (!direct_out)
      CK(cudaMemcpy2DAsync(probs + r0 * n_labels, static_cast<size_t>(n_labels) * sizeof(float), m->probs.p,
                           static_cast<size_t>(LL.n_pad) * sizeof(float), static_cast<size_t>(n_labels) * sizeof(float),
                           rows, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s));
    if (!dev) CK(cudaStreamSynchronize(s));  // xf is reused by the next chunk
  }
  return IE_OK;
}

int ie_pr_thresholds(const float* scores, const uint8_t* truth, int32_t n, int32_t n_labels, double precision_threshold,
                     double recall_threshold, float* thresholds, double* precisions, double* recalls, int32_t device,
                     int32_t flags, void* stream) {
  if (scores == nullptr || truth == nullptr || thresholds == nullptr || precisions == nullptr || recalls == nullptr)
    return fail(IE_ERR_INVALID, "null argument");
  if (n < 1 || n_labels < 1) return fail(IE_ERR_INVALID, "n=%d n_labels=%d", n, n_labels);
  if (n > ie::kPrMaxSamples)
    return fail(IE_ERR_INVALID, "n=%d exceeds the %d samples one CTA sorts in shared memory", n, ie::kPrMaxSamples);
  int sms = 0;
  const int rc = open_device(device, &sms);
  if (rc != IE_OK) return rc;
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dev) {
    CK(ie::launch_pr_thresholds(scores, truth, n, n_labels, precision_threshold, recall_threshold, thresholds, precisions,
                                recalls, s));
    return IE_OK;
  }
  const size_t cells = static_cast<size_t>(n) * n_labels;
  for (size_t i = 0; i < cells; ++i)   // sklearn's precision_recall_curve raises on NaN / inf
    if (!std::isfinite(scores[i]))
      return fail(IE_ERR_INVALID, "scores[%zu][%zu] = %g is not finite", i / n_labels, i % n_labels,
                  static_cast<double>(scores[i]));
  DevBuf ds, dt, dth, dp, dr;
  CK(ds.reserve(cells * sizeof(float)));
  CK(dt.reserve(cells));
  CK(dth.reserve(n_labels * sizeof(float)));
  CK(dp.reserve(n_labels * sizeof(double)));
  CK(dr.reserve(n_labels * sizeof(double)));
  CK(cudaMemcpyAsync(ds.p, scores, cells * sizeof(float), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(dt.p, truth, cells, cudaMemcpyHostToDevice, s));
  CK(ie::launch_pr_thresholds(ds.as<float>(), dt.as<uint8_t>(), n, n_labels, precision_threshold, recall_threshold,
                              dth.as<float>(), dp.as<double>(), dr.as<double>(), s));
  CK(cudaMemcpyAsync(thresholds, dth.p, n_labels * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(precisions, dp.p, n_labels * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(recalls, dr.p, n_labels * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return IE_OK;
}

void ie_mlp_destroy(ie_mlp* m) {
  if (m == nullptr) return;
  cudaSetDevice(m->device);
  cudaDeviceSynchronize();
  if (m->own_stream) cudaStreamDestroy(m->own_stream);
  delete m;
}

}  // extern "C"
