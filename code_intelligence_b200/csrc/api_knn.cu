// C-ABI layer of the k-nearest-neighbour index over issue embeddings (declared in include/issue_emb_b200.h; kernels in
// knn.cu): storage, input checks and the two-stage search.
#include "host.h"

using namespace ie;

struct ie_knn {
  int dim = 0, metric = IE_KNN_COSINE, device = 0, num_sms = 132;
  int k_pad = 0;            // dim rounded up to 64
  long long n = 0, cap = 0;  // rows stored / rows the storage holds (a multiple of 256)
  DevBuf xf;                // f32 [cap, dim]: the rows as given (exact re-ranking)
  DevBuf xs;                // bf16 [cap, 2*k_pad]: split-bf16 of x - c
  DevBuf col;               // float2 [cap]: per-row terms of the stage-1 epilogue
  DevBuf center;            // f32 [k_pad]: c (fixed by the first add)
  double c2 = 0.0;          // |c|^2 in f64
  bool centred = false;
  DevBuf partial, qf, qs, rowt, cand, cnt, outd, outi, err;
  cudaStream_t own_stream = nullptr;
  StreamOrder order;
  std::mutex mu;
};

namespace {

// grow a buffer to `bytes`, keeping its first `keep` bytes
int knn_grow(DevBuf& b, size_t bytes, size_t keep, cudaStream_t s) {
  if (bytes <= b.cap) return IE_OK;
  DevBuf nb;
  CK(nb.reserve(bytes));
  if (keep) {
    CK(cudaMemcpyAsync(nb.p, b.p, keep, cudaMemcpyDeviceToDevice, s));
    CK(cudaStreamSynchronize(s));
  }
  b = std::move(nb);
  return IE_OK;
}

// host input: every value finite, every row's norm 0 or in [kKnnNormMin, kKnnNormMax] (the prep kernel's check)
int knn_check_rows(const float* x, long long rows, int dim, const char* what) {
  for (long long r = 0; r < rows; ++r) {
    const float* v = x + r * dim;
    double s = 0.0;
    for (int i = 0; i < dim; ++i) {
      if (!std::isfinite(v[i]))
        return fail(IE_ERR_INVALID, "%s[%lld][%d] = %g is not finite", what, r, i, static_cast<double>(v[i]));
      s += static_cast<double>(v[i]) * v[i];
    }
    if (s > 0.0 && (s < ie::kKnnNormMin * ie::kKnnNormMin || s > ie::kKnnNormMax * ie::kKnnNormMax))
      return fail(IE_ERR_INVALID, "%s row %lld has norm %g, outside the index's range [2^-48, 2^48] (0 is allowed)",
                  what, r, std::sqrt(s));
  }
  return IE_OK;
}

// search (dbg_score == nullptr) or stage 1 only (dbg_*: host [nq, k + 32])
int knn_search(ie_knn* h, const float* Q, int32_t nq, int32_t k, float* dist, int64_t* idx, int32_t flags, void* stream,
               float* dbg_score, int64_t* dbg_idx) {
  if (h == nullptr || Q == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (dbg_score == nullptr && (dist == nullptr || idx == nullptr)) return fail(IE_ERR_INVALID, "null argument");
  if (nq < 1) return fail(IE_ERR_INVALID, "nq=%d must be >= 1", nq);
  if (k < 1 || k > 64) return fail(IE_ERR_INVALID, "k=%d not in [1, 64]", k);
  std::lock_guard<std::mutex> lk(h->mu);
  if (h->n == 0) return fail(IE_ERR_STATE, "the index is empty: add rows before searching");
  if (k > h->n) return fail(IE_ERR_INVALID, "k=%d exceeds the %lld rows of the index", k, h->n);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0 && dbg_score == nullptr;
  if (!dev) {
    const int rc = knn_check_rows(Q, nq, h->dim, "Q");
    if (rc != IE_OK) return rc;
  }
  CK(cudaSetDevice(h->device));
  const cudaStream_t s = call_stream(flags, stream, h->own_stream);
  CK(h->order.begin(s));
  const int kp = k + ie::kKnnExtra;
  const int pass = std::min(nq, 128 * h->num_sms);
  const long long m_pad_max = round_up(pass, 128);
  const int D = h->dim;
  CK(h->qs.reserve(static_cast<size_t>(m_pad_max) * 2 * h->k_pad * sizeof(__nv_bfloat16)));
  CK(h->rowt.reserve(static_cast<size_t>(m_pad_max) * sizeof(float2)));
  if (!dev) {
    CK(h->qf.reserve(static_cast<size_t>(pass) * D * sizeof(float)));
    const int w = dbg_score ? kp : k;
    CK(h->outd.reserve(static_cast<size_t>(pass) * w * sizeof(float)));
    CK(h->outi.reserve(static_cast<size_t>(pass) * w * sizeof(int64_t)));
  }
  for (long long r0 = 0; r0 < nq; r0 += pass) {
    const int rows = static_cast<int>(std::min<long long>(pass, nq - r0));
    const int m_pad = static_cast<int>(round_up(rows, 128));
    const float* qsrc = Q + r0 * D;
    if (!dev) {
      CK(cudaMemcpyAsync(h->qf.p, qsrc, static_cast<size_t>(rows) * D * sizeof(float), cudaMemcpyHostToDevice, s));
      qsrc = h->qf.as<float>();
    }
    CK(ie::launch_knn_prep(qsrc, rows, m_pad, D, h->k_pad, h->center.as<float>(), h->c2, 2,
                           h->qs.as<__nv_bfloat16>(), h->rowt.as<float2>(), h->err.as<int>(), s));
    int S = 1, nbs = 1;
    ie::knn_plan(rows, h->n, kp, h->num_sms, &S, &nbs);
    CK(h->cand.reserve(static_cast<size_t>(rows) * S * ie::kKnnCap * sizeof(uint2)));
    CK(h->cnt.reserve(static_cast<size_t>(rows) * S * sizeof(int)));
    ie::KnnStage1Args a{};
    a.qs = h->qs.as<__nv_bfloat16>();
    a.xs = h->xs.as<__nv_bfloat16>();
    a.col = h->col.as<float2>();
    a.rowt = h->rowt.as<float2>();
    a.cand = h->cand.as<uint2>();
    a.cnt = h->cnt.as<int>();
    a.n = h->n;
    a.nq = rows;
    a.m_pad = m_pad;
    a.k_pad = h->k_pad;
    a.S = S;
    a.nbs = nbs;
    a.kp = kp;
    a.cosine = h->metric == IE_KNN_COSINE;
    a.num_sms = h->num_sms;
    CK(ie::launch_knn_stage1(a, s));
    float* od = dev ? dist + r0 * k : h->outd.as<float>();
    int64_t* oi = dev ? idx + r0 * k : h->outi.as<int64_t>();
    CK(ie::launch_knn_merge_rerank(a.cand, a.cnt, rows, S, kp, qsrc, h->xf.as<float>(), D, a.cosine, k, od, oi,
                                   dbg_score ? h->outd.as<float>() : nullptr, dbg_score ? h->outi.as<int64_t>() : nullptr,
                                   s));
    if (!dev) {
      const int w = dbg_score ? kp : k;
      float* hd = dbg_score ? dbg_score + r0 * kp : dist + r0 * k;
      int64_t* hi = dbg_score ? dbg_idx + r0 * kp : idx + r0 * k;
      CK(cudaMemcpyAsync(hd, h->outd.p, static_cast<size_t>(rows) * w * sizeof(float), cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(hi, h->outi.p, static_cast<size_t>(rows) * w * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));   // qf and the staging buffers are reused by the next pass
    }
  }
  CK(h->order.end(s));
  return IE_OK;
}

}  // namespace

extern "C" {

int ie_knn_create(int32_t dim, int32_t metric, int32_t device, ie_knn** out) {
  if (out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (dim < 1 || dim > 8192) return fail(IE_ERR_INVALID, "dim=%d not in [1, 8192]", dim);
  if (metric != IE_KNN_COSINE && metric != IE_KNN_EUCLIDEAN) return fail(IE_ERR_INVALID, "metric=%d", metric);
  int sms = 0;
  const int rc = open_device(device, &sms);
  if (rc != IE_OK) return rc;
  ie_knn* h = new ie_knn();
  h->dim = dim;
  h->metric = metric;
  h->device = device;
  h->num_sms = sms;
  h->k_pad = static_cast<int>(round_up(dim, 64));
  cudaError_t e = h->err.reserve(sizeof(int), true);
  if (e == cudaSuccess) e = h->center.reserve(static_cast<size_t>(h->k_pad) * sizeof(float));
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    ie_knn_destroy(h);
    return cuda_fail(e, "ie_knn_create");
  }
  *out = h;
  return IE_OK;
}

void ie_knn_destroy(ie_knn* h) {
  if (h == nullptr) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  delete h;
}

int ie_knn_add(ie_knn* h, const float* X, int64_t n, int32_t flags, void* stream) {
  if (h == nullptr || X == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (n < 1) return fail(IE_ERR_INVALID, "n=%lld must be >= 1", static_cast<long long>(n));
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  std::lock_guard<std::mutex> lk(h->mu);
  if (h->n + n >= (1ll << 31) - 256)
    return fail(IE_ERR_INVALID, "%lld + %lld rows exceed the index limit of 2^31", h->n, static_cast<long long>(n));
  if (!dev) {
    const int rc = knn_check_rows(X, n, h->dim, "X");
    if (rc != IE_OK) return rc;
  }
  CK(cudaSetDevice(h->device));
  const cudaStream_t s = call_stream(flags, stream, h->own_stream);
  CK(h->order.begin(s));
  int rc;
  const long long need = h->n + n;
  if (need > h->cap) {
    const long long cap = round_up(std::max(need, std::min(2 * h->cap, (1ll << 31) - 256)), 256);
    const size_t row_f = static_cast<size_t>(h->dim) * sizeof(float), row_s = 2ull * h->k_pad * sizeof(__nv_bfloat16);
    if ((rc = knn_grow(h->xf, cap * row_f, h->n * row_f, s)) != IE_OK) return rc;
    if ((rc = knn_grow(h->xs, cap * row_s, h->n * row_s, s)) != IE_OK) return rc;
    if ((rc = knn_grow(h->col, cap * sizeof(float2), h->n * sizeof(float2), s)) != IE_OK) return rc;
    h->cap = cap;
  }
  float* dst = h->xf.as<float>() + h->n * h->dim;
  CK(cudaMemcpyAsync(dst, X, static_cast<size_t>(n) * h->dim * sizeof(float),
                     dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
  if (!h->centred) {   // c = f32(f64 mean of the first add's rows), fixed from now on
    CK(h->partial.reserve(ie::knn_center_workspace(h->dim)));
    CK(ie::launch_knn_center(dst, n, h->dim, h->k_pad, h->partial.as<double>(), h->center.as<float>(), s));
    std::vector<float> c(h->dim);
    CK(cudaMemcpyAsync(c.data(), h->center.p, c.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    double c2 = 0.0;
    for (float v : c) c2 += static_cast<double>(v) * v;
    h->c2 = c2;
    h->centred = true;
  }
  CK(ie::launch_knn_prep(dst, n, n, h->dim, h->k_pad, h->center.as<float>(), h->c2,
                         h->metric == IE_KNN_COSINE ? 1 : 0, h->xs.as<__nv_bfloat16>() + h->n * 2 * h->k_pad,
                         h->col.as<float2>() + h->n, h->err.as<int>(), s));
  h->n = need;
  if (!dev) CK(cudaStreamSynchronize(s));   // the caller may reuse X
  CK(h->order.end(s));
  return IE_OK;
}

int ie_knn_search(ie_knn* h, const float* Q, int32_t nq, int32_t k, float* dist, int64_t* idx, int32_t flags,
                  void* stream) {
  return knn_search(h, Q, nq, k, dist, idx, flags, stream, nullptr, nullptr);
}

int ie_debug_knn_shortlist(ie_knn* h, const float* Q, int32_t nq, int32_t k, float* score, int64_t* idx) {
  if (score == nullptr || idx == nullptr) return fail(IE_ERR_INVALID, "null argument");
  return knn_search(h, Q, nq, k, nullptr, nullptr, 0, nullptr, score, idx);
}

int ie_knn_check_errors(ie_knn* h) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  int w = 0;
  const int rc = read_errors(h->order, h->err, &w, 1);
  if (rc != IE_OK || w == 0) return rc;
  if (w & 1) return fail(IE_ERR_INVALID, "a non-finite value was seen in device input (an added row or a query)");
  return fail(IE_ERR_INVALID, "a row of device input (an added row or a query) has a norm outside the index's range "
                              "[2^-48, 2^48] (0 is allowed)");
}

}  // extern "C"
