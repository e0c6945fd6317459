// C-ABI layer of the label-MLP trainers (declared in include/issue_emb_b200.h): the single trainer's sklearn Adam step
// sequence (mlp_train.cu + the persistent GEMM in split-bf16) and the group trainer's, the same step for many models at
// once (mlp_group.cu).
#include <utility>

#include "host.h"

using namespace ie;

struct ie_mlp_train {
  int device = 0, num_sms = 132, nl = 0;
  std::vector<int> dims;
  struct L {
    int in = 0, out = 0;
    int kp_in = 0, kp_out = 0;   // K padding (64) of the products with K = in / K = out
    int n16 = 0, bn = 0, np = 0;  // output width rounded to 16, the GEMM's N granularity and padded N of `out`
    int bn_in = 0, np_in = 0;    // same for `in` (the backward-data product's N)
    int mt_in = 0;               // `in` rounded to 128: M of the weight-gradient product
    long long woff = 0, boff = 0;  // offsets of W [in, out] and b [out] in the parameter vectors
    DevBuf wt_s, w_s;            // split-bf16 W^T [np, 2 kp_in] (forward B) and W [np_in, 2 kp_out] (backward-data B)
    DevBuf z, act_rm, act_tr, dz, d_rm, d_tr;  // per-step workspace (mlp_train_ws)
  };
  std::vector<L> layers;
  long long n_param = 0, n_coef = 0;  // parameter vector (segments 64-aligned, zero padding), coefficient part
  long long n_packed = 0;             // sklearn's packing: every coef, then every intercept, no padding
  DevBuf P, M, V, G, best, sq;
  DevBuf xtr, ytr, xval, order, lr, losses, ridx;
  long long n_tr = 0, n_val = 0;
  int cap = 0, cap_m = 0, kb_cap = 0;  // workspace rows, rounded to 128 (M) and 64 (K of the weight gradient)
  DevBuf gbuf, dwbuf, row_loss, pbuf;
  std::vector<bool> set;
  int64_t launches = 0;
  float last_epoch_ms = 0.0f;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaStream_t s = nullptr;
  std::mutex mu;
};

namespace {

#define MT(expr)             \
  do {                       \
    CK(expr);                \
    ++h->launches;           \
  } while (0)

void n_tiles(int w, int* n16, int* bn, int* np) {
  *n16 = static_cast<int>(round_up(w, 16));
  *bn = *n16 >= 256 ? 256 : *n16;
  *np = static_cast<int>(round_up(w, *bn));
}

// the layer layout of both trainers: each layer's padding and GEMM tiles, and the offsets of its W and b in the
// parameter vector
template <typename H>
void mt_layout(H* h, int n_layers, const int32_t* dims) {
  h->nl = n_layers;
  h->dims.assign(dims, dims + n_layers + 1);
  h->layers.resize(n_layers);
  long long off = 0;
  for (int l = 0; l < n_layers; ++l) {
    auto& L = h->layers[l];
    L.in = dims[l];
    L.out = dims[l + 1];
    L.kp_in = static_cast<int>(round_up(L.in, 64));
    L.kp_out = static_cast<int>(round_up(L.out, 64));
    L.mt_in = static_cast<int>(round_up(L.in, 128));
    n_tiles(L.out, &L.n16, &L.bn, &L.np);
    int n16_in;
    n_tiles(L.in, &n16_in, &L.bn_in, &L.np_in);
    L.woff = off;
    off += round_up(static_cast<long long>(L.in) * L.out, 64);
    h->n_packed += static_cast<long long>(L.in) * L.out + L.out;
  }
  h->n_coef = off;
  // each intercept segment is followed by zeros to its 64-multiple: the GEMM reads the bias to the output's 16-multiple
  for (auto& L : h->layers) {
    L.boff = off;
    off += round_up(L.out, 64);
  }
  h->n_param = off;
}

int mt_ws(ie_mlp_train* h, int rows) {
  if (rows <= h->cap) return IE_OK;
  const int cap_m = static_cast<int>(round_up(rows, 128)), kb = static_cast<int>(round_up(rows, 64));
  const size_t bf = sizeof(__nv_bfloat16);
  size_t g = 0, dw = 0;
  for (auto& L : h->layers) {
    CK(L.z.reserve(static_cast<size_t>(cap_m) * L.n16 * sizeof(float)));
    CK(L.dz.reserve(static_cast<size_t>(cap_m) * L.n16 * sizeof(float)));
    CK(L.act_rm.reserve(static_cast<size_t>(cap_m) * 2 * L.kp_in * bf));
    CK(L.act_tr.reserve(static_cast<size_t>(L.mt_in) * 2 * kb * bf));
    CK(L.d_rm.reserve(static_cast<size_t>(cap_m) * 2 * L.kp_out * bf));
    CK(L.d_tr.reserve(static_cast<size_t>(L.np) * 2 * kb * bf));
    g = std::max<size_t>(g, static_cast<size_t>(cap_m) * round_up(L.in, 16));
    dw = std::max<size_t>(dw, static_cast<size_t>(L.in) * L.n16);
  }
  CK(h->gbuf.reserve(g * sizeof(float)));
  CK(h->dwbuf.reserve(dw * sizeof(float)));
  CK(h->row_loss.reserve(static_cast<size_t>(cap_m) * sizeof(double)));
  CK(h->pbuf.reserve(static_cast<size_t>(cap_m) * h->layers.back().n16 * sizeof(float)));
  CK(h->ridx.reserve(static_cast<size_t>(cap_m) * sizeof(int)));
  h->cap = rows;
  h->cap_m = cap_m;
  h->kb_cap = kb;
  return IE_OK;
}

int mt_gemm(ie_mlp_train* h, const __nv_bfloat16* a, long long lda, int m_pad, const __nv_bfloat16* b, long long ldb,
            int n_pad, int bn, int k_pad, const float* bias, int act, float* d, long long ldd, int m_store, int n_store) {
  ie::GemmArgs g{};
  g.a = a;
  g.lda = lda;
  g.b = b;
  g.ldb = ldb;
  g.bias = bias;
  g.m_pad = m_pad;
  g.n_pad = n_pad;
  g.k_pad = k_pad;
  g.bn = bn;
  g.d = d;
  g.ldd = ldd;
  g.m_store = m_store;
  g.n_store = n_store;
  g.act = act;
  g.out_bf16 = 0;
  g.segs = 3;
  g.num_sms = h->num_sms;
  MT(ie::launch_gemm_bf16(g, h->s));
  return IE_OK;
}

// split-bf16 copies of every W in both layouts the products read, and the sum |W|^2 partials of the loss
int mt_refresh(ie_mlp_train* h) {
  for (int l = 0; l < h->nl; ++l) {
    auto& L = h->layers[l];
    ie::SplitStoreArgs a{};
    a.src = h->P.as<float>() + L.woff;
    a.ld_src = L.out;
    a.rows = L.in;
    a.cols = L.out;
    if (l > 0) {  // layer 0 has no backward-data product
      a.rm = L.w_s.as<__nv_bfloat16>();
      a.ld_rm = 2 * L.kp_out;
      a.rm_rows = L.np_in;
      a.rm_kpad = L.kp_out;
    }
    a.tr = L.wt_s.as<__nv_bfloat16>();
    a.ld_tr = 2 * L.kp_in;
    a.tr_rows = L.np;
    a.tr_kpad = L.kp_in;
    MT(ie::launch_split_store(a, h->s));
  }
  return IE_OK;
}

int mt_sq(ie_mlp_train* h) {
  ie::AdamArgs a{};
  a.p = h->P.as<float>();
  a.n = h->n_param;
  a.n_coef = h->n_coef;
  a.sq_part = h->sq.as<double>();
  MT(ie::launch_adam(a, h->s));
  return IE_OK;
}

// forward pass over b rows of x (row r = x row ridx[r], or r): hidden activations in z, probabilities in pbuf; with
// y, deltas of the output, its loss terms and the transposed operands of the weight gradients
int mt_forward(ie_mlp_train* h, const float* x, const int* ridx, int b, const uint8_t* y) {
  const int m_pad = static_cast<int>(round_up(b, 128)), kb = static_cast<int>(round_up(b, 64));
  const bool train = y != nullptr;
  ie::SplitStoreArgs a{};
  auto& L0 = h->layers[0];
  a.src = x;
  a.ld_src = L0.in;
  a.rowidx = ridx;
  a.rows = b;
  a.cols = L0.in;
  a.rm = L0.act_rm.as<__nv_bfloat16>();
  a.ld_rm = 2 * L0.kp_in;
  a.rm_rows = m_pad;
  a.rm_kpad = L0.kp_in;
  if (train) {
    a.tr = L0.act_tr.as<__nv_bfloat16>();
    a.ld_tr = 2 * h->kb_cap;
    a.tr_rows = L0.mt_in;
    a.tr_kpad = kb;
  }
  MT(ie::launch_split_store(a, h->s));
  for (int l = 0; l < h->nl; ++l) {
    auto& L = h->layers[l];
    const bool last = l == h->nl - 1;
    int rc = mt_gemm(h, L.act_rm.as<__nv_bfloat16>(), 2 * L.kp_in, m_pad, L.wt_s.as<__nv_bfloat16>(), 2 * L.kp_in, L.np,
                     L.bn, L.kp_in, h->P.as<float>() + L.boff, last ? 0 : 1, L.z.as<float>(), L.n16, b, L.n16);
    if (rc != IE_OK) return rc;
    if (last) {
      MT(ie::launch_mlp_output(L.z.as<float>(), L.n16, y, ridx, b, L.out, h->pbuf.as<float>(), L.dz.as<float>(),
                               h->row_loss.as<double>(), h->s));
      break;
    }
    auto& N = h->layers[l + 1];
    ie::SplitStoreArgs c{};
    c.src = L.z.as<float>();
    c.ld_src = L.n16;
    c.rows = b;
    c.cols = L.out;
    c.rm = N.act_rm.as<__nv_bfloat16>();
    c.ld_rm = 2 * N.kp_in;
    c.rm_rows = m_pad;
    c.rm_kpad = N.kp_in;
    if (train) {
      c.tr = N.act_tr.as<__nv_bfloat16>();
      c.ld_tr = 2 * h->kb_cap;
      c.tr_rows = N.mt_in;
      c.tr_kpad = kb;
    }
    MT(ie::launch_split_store(c, h->s));
  }
  return IE_OK;
}

// loss and every gradient of the batch mt_forward left (into G); loss -> *loss_out (device)
int mt_backward(ie_mlp_train* h, int b, double alpha, double* loss_out) {
  const int m_pad = static_cast<int>(round_up(b, 128)), kb = static_cast<int>(round_up(b, 64));
  MT(ie::launch_mlp_loss(h->row_loss.as<double>(), b, h->sq.as<double>(), ie::kAdamBlocks, alpha, loss_out, h->s));
  {
    auto& L = h->layers[h->nl - 1];
    ie::SplitStoreArgs a{};
    a.src = L.dz.as<float>();
    a.ld_src = L.n16;
    a.rows = b;
    a.cols = L.out;
    a.rm = L.d_rm.as<__nv_bfloat16>();
    a.ld_rm = 2 * L.kp_out;
    a.rm_rows = m_pad;
    a.rm_kpad = L.kp_out;
    a.tr = L.d_tr.as<__nv_bfloat16>();
    a.ld_tr = 2 * h->kb_cap;
    a.tr_rows = L.np;
    a.tr_kpad = kb;
    MT(ie::launch_split_store(a, h->s));
  }
  for (int l = h->nl - 1; l >= 0; --l) {
    auto& L = h->layers[l];
    // dW = a^T delta: M = in, N = out, K = batch
    int rc = mt_gemm(h, L.act_tr.as<__nv_bfloat16>(), 2 * h->kb_cap, L.mt_in, L.d_tr.as<__nv_bfloat16>(), 2 * h->kb_cap,
                     L.np, L.bn, kb, nullptr, 0, h->dwbuf.as<float>(), L.n16, L.in, L.n16);
    if (rc != IE_OK) return rc;
    MT(ie::launch_mlp_grad(h->dwbuf.as<float>(), L.n16, h->P.as<float>() + L.woff, L.in, L.out, L.dz.as<float>(), L.n16, b,
                           static_cast<float>(alpha), h->G.as<float>() + L.woff, h->G.as<float>() + L.boff, h->s));
    if (l == 0) break;
    // delta_{l-1} = (delta_l W_l^T) * [a_l != 0]: M = batch, N = in, K = out
    auto& P = h->layers[l - 1];
    rc = mt_gemm(h, L.d_rm.as<__nv_bfloat16>(), 2 * L.kp_out, m_pad, L.w_s.as<__nv_bfloat16>(), 2 * L.kp_out, L.np_in,
                 L.bn_in, L.kp_out, nullptr, 0, h->gbuf.as<float>(), P.n16, b, P.n16);
    if (rc != IE_OK) return rc;
    ie::SplitStoreArgs a{};
    a.src = h->gbuf.as<float>();
    a.ld_src = P.n16;
    a.rows = b;
    a.cols = P.out;
    a.mask = P.z.as<float>();
    a.ld_mask = P.n16;
    a.out_f32 = P.dz.as<float>();
    a.ld_f32 = P.n16;
    a.rm = P.d_rm.as<__nv_bfloat16>();
    a.ld_rm = 2 * P.kp_out;
    a.rm_rows = m_pad;
    a.rm_kpad = P.kp_out;
    a.tr = P.d_tr.as<__nv_bfloat16>();
    a.ld_tr = 2 * h->kb_cap;
    a.tr_rows = P.np;
    a.tr_kpad = kb;
    MT(ie::launch_split_store(a, h->s));
  }
  return IE_OK;
}

int mt_adam(ie_mlp_train* h, const double* lr_dev, int step, double beta_1, double beta_2, double epsilon) {
  ie::AdamArgs a{};
  a.p = h->P.as<float>();
  a.m = h->M.as<float>();
  a.v = h->V.as<float>();
  a.g = h->G.as<float>();
  a.n = h->n_param;
  a.n_coef = h->n_coef;
  a.beta1 = static_cast<float>(beta_1);
  a.one_m_beta1 = static_cast<float>(1.0 - beta_1);
  a.beta2 = static_cast<float>(beta_2);
  a.one_m_beta2 = static_cast<float>(1.0 - beta_2);
  a.eps = static_cast<float>(epsilon);
  a.lr = lr_dev;
  a.step = step;
  a.sq_part = h->sq.as<double>();
  MT(ie::launch_adam(a, h->s));
  return mt_refresh(h);
}

// sklearn packing (coefs_ then intercepts_, no padding) <-> the padded parameter vector
void mt_pack(const ie_mlp_train* h, const float* padded, float* packed) {
  long long o = 0;
  for (const auto& L : h->layers) {
    std::copy(padded + L.woff, padded + L.woff + static_cast<long long>(L.in) * L.out, packed + o);
    o += static_cast<long long>(L.in) * L.out;
  }
  for (const auto& L : h->layers) {
    std::copy(padded + L.boff, padded + L.boff + L.out, packed + o);
    o += L.out;
  }
}

void mt_unpack(const ie_mlp_train* h, const float* packed, float* padded) {
  std::fill(padded, padded + h->n_param, 0.0f);
  long long o = 0;
  for (const auto& L : h->layers) {
    std::copy(packed + o, packed + o + static_cast<long long>(L.in) * L.out, padded + L.woff);
    o += static_cast<long long>(L.in) * L.out;
  }
  for (const auto& L : h->layers) {
    std::copy(packed + o, packed + o + L.out, padded + L.boff);
    o += L.out;
  }
}

int mt_ready(ie_mlp_train* h, bool need_data) {
  for (bool b : h->set)
    if (!b) return fail(IE_ERR_STATE, "MLP trainer parameters not set (ie_mlp_train_set_layer for every layer)");
  if (need_data && h->n_tr == 0) return fail(IE_ERR_STATE, "no training set uploaded (ie_mlp_train_set_data)");
  return IE_OK;
}

int mt_check_rows(const int32_t* rows, long long n, long long limit) {
  for (long long i = 0; i < n; ++i)
    if (rows[i] < 0 || rows[i] >= limit) return fail(IE_ERR_INVALID, "row %lld = %d outside [0, %lld)", i, rows[i], limit);
  return IE_OK;
}

}  // namespace

extern "C" {

int ie_mlp_train_create(int32_t n_layers, const int32_t* dims, int32_t device, ie_mlp_train** out) {
  if (dims == nullptr || out == nullptr || n_layers < 2 || n_layers > 16)
    return fail(IE_ERR_INVALID, "n_layers=%d: the trainer needs 1 to 15 hidden layers", n_layers);
  for (int i = 0; i <= n_layers; ++i)
    if (dims[i] < 1 || dims[i] > (1 << 16)) return fail(IE_ERR_INVALID, "dims[%d]=%d not in [1, 65536]", i, dims[i]);
  int sms = 0;
  const int rc = open_device(device, &sms);
  if (rc != IE_OK) return rc;
  ie_mlp_train* h = new ie_mlp_train();
  h->device = device;
  h->num_sms = sms;
  mt_layout(h, n_layers, dims);
  h->set.assign(n_layers, false);
  const size_t pb = static_cast<size_t>(h->n_param) * sizeof(float), bf = sizeof(__nv_bfloat16);
  cudaError_t e = cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev1);
  for (DevBuf* b : {&h->P, &h->M, &h->V, &h->G, &h->best})
    if (e == cudaSuccess) e = b->reserve(pb, true);
  if (e == cudaSuccess) e = h->sq.reserve(ie::kAdamBlocks * sizeof(double), true);
  for (int l = 0; l < n_layers && e == cudaSuccess; ++l) {
    auto& L = h->layers[l];
    e = L.wt_s.reserve(static_cast<size_t>(L.np) * 2 * L.kp_in * bf);
    if (e == cudaSuccess && l > 0) e = L.w_s.reserve(static_cast<size_t>(L.np_in) * 2 * L.kp_out * bf);
  }
  if (e != cudaSuccess) {
    ie_mlp_train_destroy(h);
    return cuda_fail(e, "ie_mlp_train_create");
  }
  *out = h;
  return IE_OK;
}

void ie_mlp_train_destroy(ie_mlp_train* h) {
  if (h == nullptr) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  if (h->s) cudaStreamDestroy(h->s);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
}

int ie_mlp_train_set_layer(ie_mlp_train* h, int32_t layer, const float* coef, const float* intercept) {
  if (h == nullptr || coef == nullptr || intercept == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (layer < 0 || layer >= h->nl) return fail(IE_ERR_INVALID, "layer %d out of range", layer);
  const auto& L = h->layers[layer];
  for (long long i = 0; i < static_cast<long long>(L.in) * L.out; ++i)
    if (!std::isfinite(coef[i])) return fail(IE_ERR_INVALID, "coef[%lld] is not finite", i);
  for (int i = 0; i < L.out; ++i)
    if (!std::isfinite(intercept[i])) return fail(IE_ERR_INVALID, "intercept[%d] is not finite", i);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpyAsync(h->P.as<float>() + L.woff, coef, static_cast<size_t>(L.in) * L.out * sizeof(float),
                     cudaMemcpyHostToDevice, h->s));
  CK(cudaMemcpyAsync(h->P.as<float>() + L.boff, intercept, static_cast<size_t>(L.out) * sizeof(float),
                     cudaMemcpyHostToDevice, h->s));
  CK(cudaMemsetAsync(h->M.p, 0, h->n_param * sizeof(float), h->s));   // Adam restarts at t = 0
  CK(cudaMemsetAsync(h->V.p, 0, h->n_param * sizeof(float), h->s));
  h->set[layer] = true;
  int rc = mt_refresh(h);
  if (rc == IE_OK) rc = mt_sq(h);
  if (rc != IE_OK) return rc;
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int ie_mlp_train_get_layer(ie_mlp_train* h, int32_t layer, int32_t best, float* coef, float* intercept) {
  if (h == nullptr || coef == nullptr || intercept == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (layer < 0 || layer >= h->nl) return fail(IE_ERR_INVALID, "layer %d out of range", layer);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  const auto& L = h->layers[layer];
  const float* src = (best ? h->best : h->P).as<float>();
  CK(cudaMemcpyAsync(coef, src + L.woff, static_cast<size_t>(L.in) * L.out * sizeof(float), cudaMemcpyDeviceToHost, h->s));
  CK(cudaMemcpyAsync(intercept, src + L.boff, static_cast<size_t>(L.out) * sizeof(float), cudaMemcpyDeviceToHost, h->s));
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int ie_mlp_train_set_data(ie_mlp_train* h, int32_t which, const float* X, const uint8_t* Y, int64_t n) {
  if (h == nullptr || X == nullptr || (which == 0 && Y == nullptr)) return fail(IE_ERR_INVALID, "null argument");
  if (which != 0 && which != 1) return fail(IE_ERR_INVALID, "which=%d (0 training, 1 validation)", which);
  if (n < 1 || n >= (1ll << 31)) return fail(IE_ERR_INVALID, "n=%lld not in [1, 2^31)", static_cast<long long>(n));
  const int D = h->dims[0], Lo = h->dims[h->nl];
  const size_t cells = static_cast<size_t>(n) * D;
  for (size_t i = 0; i < cells; ++i)
    if (!std::isfinite(X[i])) return fail(IE_ERR_INVALID, "X[%zu][%zu] is not finite", i / D, i % D);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  DevBuf& xb = which == 0 ? h->xtr : h->xval;
  CK(xb.reserve(cells * sizeof(float)));
  CK(cudaMemcpyAsync(xb.p, X, cells * sizeof(float), cudaMemcpyHostToDevice, h->s));
  if (which == 0) {
    CK(h->ytr.reserve(static_cast<size_t>(n) * Lo));
    CK(cudaMemcpyAsync(h->ytr.p, Y, static_cast<size_t>(n) * Lo, cudaMemcpyHostToDevice, h->s));
    h->n_tr = n;
  } else {
    h->n_val = n;
  }
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int ie_mlp_train_epoch(ie_mlp_train* h, const int32_t* order, int64_t n, int32_t batch_size, const double* lr,
                       double alpha, double beta_1, double beta_2, double epsilon, double* losses) {
  if (h == nullptr || order == nullptr || lr == nullptr || losses == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  int rc = mt_ready(h, true);
  if (rc != IE_OK) return rc;
  if (n != h->n_tr) return fail(IE_ERR_INVALID, "order has %lld rows, the training set %lld", static_cast<long long>(n), h->n_tr);
  if (batch_size < 1 || batch_size > n) return fail(IE_ERR_INVALID, "batch_size=%d not in [1, %lld]", batch_size, h->n_tr);
  if ((rc = mt_check_rows(order, n, h->n_tr)) != IE_OK) return rc;
  CK(cudaSetDevice(h->device));
  const long long steps = (n + batch_size - 1) / batch_size;
  if ((rc = mt_ws(h, batch_size)) != IE_OK) return rc;
  CK(h->order.reserve(static_cast<size_t>(n) * sizeof(int)));
  CK(h->lr.reserve(static_cast<size_t>(steps) * sizeof(double)));
  CK(h->losses.reserve(static_cast<size_t>(steps) * sizeof(double)));
  CK(cudaMemcpyAsync(h->order.p, order, static_cast<size_t>(n) * sizeof(int), cudaMemcpyHostToDevice, h->s));
  CK(cudaMemcpyAsync(h->lr.p, lr, static_cast<size_t>(steps) * sizeof(double), cudaMemcpyHostToDevice, h->s));
  CK(cudaEventRecord(h->ev0, h->s));
  for (long long k = 0; k < steps; ++k) {   // every step is enqueued; the host waits once, for the losses
    const long long r0 = k * batch_size;
    const int b = static_cast<int>(std::min<long long>(batch_size, n - r0));
    if ((rc = mt_forward(h, h->xtr.as<float>(), h->order.as<int>() + r0, b, h->ytr.as<uint8_t>())) != IE_OK) return rc;
    if ((rc = mt_backward(h, b, alpha, h->losses.as<double>() + k)) != IE_OK) return rc;
    if ((rc = mt_adam(h, h->lr.as<double>(), static_cast<int>(k), beta_1, beta_2, epsilon)) != IE_OK) return rc;
  }
  CK(cudaEventRecord(h->ev1, h->s));
  CK(cudaMemcpyAsync(losses, h->losses.p, static_cast<size_t>(steps) * sizeof(double), cudaMemcpyDeviceToHost, h->s));
  CK(cudaStreamSynchronize(h->s));
  CK(cudaEventElapsedTime(&h->last_epoch_ms, h->ev0, h->ev1));
  return IE_OK;
}

int ie_mlp_train_validation_proba(ie_mlp_train* h, float* probs) {
  if (h == nullptr || probs == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  int rc = mt_ready(h, false);
  if (rc != IE_OK) return rc;
  if (h->n_val == 0) return fail(IE_ERR_STATE, "no validation set uploaded (ie_mlp_train_set_data which=1)");
  CK(cudaSetDevice(h->device));
  if ((rc = mt_ws(h, std::max(h->cap, 256))) != IE_OK) return rc;
  const int Lo = h->dims[h->nl], ldp = h->layers.back().n16;
  for (long long r0 = 0; r0 < h->n_val; r0 += h->cap) {
    const int rows = static_cast<int>(std::min<long long>(h->cap, h->n_val - r0));
    rc = mt_forward(h, h->xval.as<float>() + r0 * h->dims[0], nullptr, rows, nullptr);
    if (rc != IE_OK) return rc;
    CK(cudaMemcpy2DAsync(probs + r0 * Lo, static_cast<size_t>(Lo) * sizeof(float), h->pbuf.p, ldp * sizeof(float),
                         static_cast<size_t>(Lo) * sizeof(float), rows, cudaMemcpyDeviceToHost, h->s));
  }
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int ie_mlp_train_snapshot(ie_mlp_train* h, int32_t restore) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  int rc = mt_ready(h, false);
  if (rc != IE_OK) return rc;
  CK(cudaSetDevice(h->device));
  const size_t pb = static_cast<size_t>(h->n_param) * sizeof(float);
  if (restore) {
    CK(cudaMemcpyAsync(h->P.p, h->best.p, pb, cudaMemcpyDeviceToDevice, h->s));
    if ((rc = mt_refresh(h)) != IE_OK || (rc = mt_sq(h)) != IE_OK) return rc;
  } else {
    CK(cudaMemcpyAsync(h->best.p, h->P.p, pb, cudaMemcpyDeviceToDevice, h->s));
  }
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int64_t ie_mlp_train_launch_count(const ie_mlp_train* h) { return h ? h->launches : -1; }

int ie_mlp_train_last_epoch_ms(ie_mlp_train* h, float* ms) {
  if (h == nullptr || ms == nullptr) return fail(IE_ERR_INVALID, "null argument");
  *ms = h->last_epoch_ms;
  return IE_OK;
}

int ie_debug_mlp_train_step(ie_mlp_train* h, int32_t mode, const int32_t* rows, int32_t b, const double* consts,
                            const float* grads, float* out, int64_t cap, double* loss) {
  if (h == nullptr || consts == nullptr || out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  int rc = mt_ready(h, mode == 0);
  if (rc != IE_OK) return rc;
  CK(cudaSetDevice(h->device));
  const int Lo = h->dims[h->nl];
  if (mode == 1) {   // the optimizer alone: given gradients (sklearn packing) -> parameters, m, v
    if (grads == nullptr) return fail(IE_ERR_INVALID, "null gradients");
    if (cap < 3 * h->n_packed) return fail(IE_ERR_INVALID, "out holds %lld floats, %lld needed", static_cast<long long>(cap), 3 * h->n_packed);
    std::vector<float> pad(h->n_param);
    mt_unpack(h, grads, pad.data());
    CK(h->lr.reserve(sizeof(double)));
    CK(cudaMemcpyAsync(h->G.p, pad.data(), pad.size() * sizeof(float), cudaMemcpyHostToDevice, h->s));
    CK(cudaMemcpyAsync(h->lr.p, consts, sizeof(double), cudaMemcpyHostToDevice, h->s));
    if ((rc = mt_adam(h, h->lr.as<double>(), 0, consts[1], consts[2], consts[3])) != IE_OK) return rc;
    const DevBuf* src[3] = {&h->P, &h->M, &h->V};
    for (int i = 0; i < 3; ++i) {
      CK(cudaMemcpyAsync(pad.data(), src[i]->p, pad.size() * sizeof(float), cudaMemcpyDeviceToHost, h->s));
      CK(cudaStreamSynchronize(h->s));
      mt_pack(h, pad.data(), out + i * h->n_packed);
    }
    return IE_OK;
  }
  if (mode != 0) return fail(IE_ERR_INVALID, "mode=%d (0 forward + backward, 1 optimizer)", mode);
  if (rows == nullptr || loss == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (b < 1) return fail(IE_ERR_INVALID, "b=%d", b);
  if ((rc = mt_check_rows(rows, b, h->n_tr)) != IE_OK) return rc;
  long long need = h->n_packed + static_cast<long long>(b) * Lo;
  for (int l = 0; l < h->nl; ++l) need += static_cast<long long>(b) * h->dims[l + 1] * (l < h->nl - 1 ? 2 : 1);
  if (cap < need) return fail(IE_ERR_INVALID, "out holds %lld floats, %lld needed", static_cast<long long>(cap), need);
  if ((rc = mt_ws(h, b)) != IE_OK) return rc;
  CK(cudaMemcpyAsync(h->ridx.p, rows, static_cast<size_t>(b) * sizeof(int), cudaMemcpyHostToDevice, h->s));
  CK(h->losses.reserve(sizeof(double)));
  if ((rc = mt_forward(h, h->xtr.as<float>(), h->ridx.as<int>(), b, h->ytr.as<uint8_t>())) != IE_OK) return rc;
  if ((rc = mt_backward(h, b, consts[0], h->losses.as<double>())) != IE_OK) return rc;
  // out: a_1 .. a_{nl-1}, p, delta_0 .. delta_{nl-1} (each [b, width] f32), then the gradients in sklearn's packing
  float* o = out;
  auto rows_out = [&](const float* src, int width, long long ld) -> int {
    CK(cudaMemcpy2DAsync(o, static_cast<size_t>(width) * sizeof(float), src, ld * sizeof(float),
                         static_cast<size_t>(width) * sizeof(float), b, cudaMemcpyDeviceToHost, h->s));
    o += static_cast<long long>(b) * width;
    return IE_OK;
  };
  for (int l = 0; l < h->nl - 1; ++l)
    if ((rc = rows_out(h->layers[l].z.as<float>(), h->layers[l].out, h->layers[l].n16)) != IE_OK) return rc;
  if ((rc = rows_out(h->pbuf.as<float>(), Lo, h->layers.back().n16)) != IE_OK) return rc;
  for (int l = 0; l < h->nl; ++l)
    if ((rc = rows_out(h->layers[l].dz.as<float>(), h->layers[l].out, h->layers[l].n16)) != IE_OK) return rc;
  std::vector<float> pad(h->n_param);
  CK(cudaMemcpyAsync(pad.data(), h->G.p, pad.size() * sizeof(float), cudaMemcpyDeviceToHost, h->s));
  CK(cudaMemcpyAsync(loss, h->losses.p, sizeof(double), cudaMemcpyDeviceToHost, h->s));
  CK(cudaStreamSynchronize(h->s));
  mt_pack(h, pad.data(), o);
  return IE_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// Group trainer (mlp_group.cu): the ie_mlp_train step for many models at once.  Every per-model buffer is one
// allocation of n_models equal slots; the products' operands are padded to whole tiles per slot (rows of A to 128, of
// B to 256, the padding zero), so a model's tiles read exactly the values a single handle's TMA reads.
// ---------------------------------------------------------------------------------------------
struct ie_mlp_group {
  int device = 0, num_sms = 132, nl = 0, G = 0, bs = 0;
  std::vector<int> dims;
  struct L : ie_mlp_train::L {   // the single trainer's layer; its buffers hold one slot per model
    int wt_rows = 0, w_rows = 0, dtr_rows = 0;   // np, np_in and np rounded to 256: B rows per slot
  };
  std::vector<L> layers;
  long long n_param = 0, n_coef = 0, n_packed = 0;
  int cap = 0, cap_m = 0, kb_cap = 0, in16_max = 0;
  long long dw_max = 0;
  DevBuf P, M, V, Gr, best, sq, alpha, consts, slot_ids;
  DevBuf gbuf, dwbuf, row_loss, pbuf;
  DevBuf X, Y, order, lr, losses, vrows, lists;
  long long n = 0, lr_pitch = 0;
  std::vector<long long> n_val;
  std::vector<bool> set, hyper;
  int64_t launches = 0;
  float last_epoch_ms = 0.0f;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaStream_t s = nullptr;
  std::mutex mu;
};

namespace {

// geometry of a group's layers (mt_layout, B rows padded per slot) and its workspace rows
void mg_geometry(ie_mlp_group* h, int n_layers, const int32_t* dims, int batch_size) {
  mt_layout(h, n_layers, dims);
  h->bs = batch_size;
  h->cap = std::max(batch_size, 256);   // validation runs in chunks of `cap` rows
  h->cap_m = static_cast<int>(round_up(h->cap, 128));
  h->kb_cap = static_cast<int>(round_up(batch_size, 64));
  h->in16_max = 0;
  h->dw_max = 0;
  for (auto& L : h->layers) {
    L.wt_rows = static_cast<int>(round_up(L.np, 256));
    L.w_rows = static_cast<int>(round_up(L.np_in, 256));
    L.dtr_rows = L.wt_rows;
    h->in16_max = std::max<int>(h->in16_max, static_cast<int>(round_up(L.in, 16)));
    h->dw_max = std::max<long long>(h->dw_max, round_up(static_cast<long long>(L.in) * L.n16, 64));
  }
}

// bytes of one slot of every per-model buffer (each slot size 64-element aligned)
struct MgSlots {
  long long wt[16], w[16], z[16], arm[16], atr[16], drm[16], dtr[16];
  long long g, pb;
};
MgSlots mg_slots(const ie_mlp_group* h) {
  MgSlots s{};
  for (int l = 0; l < h->nl; ++l) {
    const auto& L = h->layers[l];
    s.wt[l] = static_cast<long long>(L.wt_rows) * 2 * L.kp_in;
    s.w[l] = l > 0 ? static_cast<long long>(L.w_rows) * 2 * L.kp_out : 0;
    s.z[l] = static_cast<long long>(h->cap_m) * L.n16;
    s.arm[l] = static_cast<long long>(h->cap_m) * 2 * L.kp_in;
    s.atr[l] = static_cast<long long>(L.mt_in) * 2 * h->kb_cap;
    s.drm[l] = static_cast<long long>(h->cap_m) * 2 * L.kp_out;
    s.dtr[l] = static_cast<long long>(L.dtr_rows) * 2 * h->kb_cap;
  }
  s.g = static_cast<long long>(h->cap_m) * h->in16_max;
  s.pb = static_cast<long long>(h->cap_m) * h->layers.back().n16;
  return s;
}

long long mg_bytes_per_model(const ie_mlp_group* h) {
  const MgSlots s = mg_slots(h);
  long long b = 5 * h->n_param * 4 + ie::kAdamBlocks * 8 + 8 + 5 * 4 + 4 + h->dw_max * 4 + s.g * 4 + s.pb * 4 +
                h->cap_m * 8;
  for (int l = 0; l < h->nl; ++l) b += (s.wt[l] + s.w[l] + s.arm[l] + s.atr[l] + s.drm[l] + s.dtr[l]) * 2 + 2 * s.z[l] * 4;
  return b;
}

int mg_refresh(ie_mlp_group* h, const int* slots, int count) {
  for (int l = 0; l < h->nl; ++l) {
    auto& L = h->layers[l];
    ie::GroupSplitArgs g{};
    g.a.src = h->P.as<float>() + L.woff;
    g.s_src = h->n_param;
    g.a.ld_src = L.out;
    g.a.rows = L.in;
    g.a.cols = L.out;
    if (l > 0) {
      g.a.rm = L.w_s.as<__nv_bfloat16>();
      g.s_rm = static_cast<long long>(L.w_rows) * 2 * L.kp_out;
      g.a.ld_rm = 2 * L.kp_out;
      g.a.rm_rows = L.np_in;
      g.a.rm_kpad = L.kp_out;
    }
    g.a.tr = L.wt_s.as<__nv_bfloat16>();
    g.s_tr = static_cast<long long>(L.wt_rows) * 2 * L.kp_in;
    g.a.ld_tr = 2 * L.kp_in;
    g.a.tr_rows = L.np;
    g.a.tr_kpad = L.kp_in;
    g.slots = slots;
    g.count = count;
    MT(ie::launch_group_split_store(g, h->s));
  }
  return IE_OK;
}

ie::GroupAdamArgs mg_adam_args(ie_mlp_group* h, const int* slots, int count) {
  ie::GroupAdamArgs a{};
  a.p = h->P.as<float>();
  a.m = h->M.as<float>();
  a.v = h->V.as<float>();
  a.n = h->n_param;
  a.n_coef = h->n_coef;
  a.s_param = h->n_param;
  a.consts = h->consts.as<float>();
  a.sq_part = h->sq.as<double>();
  a.slots = slots;
  a.count = count;
  return a;
}

int mg_sq(ie_mlp_group* h, const int* slots, int count) {
  MT(ie::launch_group_adam(mg_adam_args(h, slots, count), h->s));
  return IE_OK;
}

int mg_gemm(ie_mlp_group* h, const int* slots, int count, const __nv_bfloat16* a, long long lda, long long a_rows,
            int m_pad, const __nv_bfloat16* b, long long ldb, long long b_rows, int n_pad, int k_pad, const float* bias,
            long long s_bias, int relu, float* d, long long ldd, long long s_d, int m_store, int n_store) {
  ie::GroupGemmArgs g{};
  g.a = a;
  g.lda = lda;
  g.a_rows = a_rows;
  g.b = b;
  g.ldb = ldb;
  g.b_rows = b_rows;
  g.d = d;
  g.ldd = ldd;
  g.s_d = s_d;
  g.bias = bias;
  g.s_bias = s_bias;
  g.m_pad = m_pad;
  g.n_pad = n_pad;
  g.k_pad = k_pad;
  g.m_store = m_store;
  g.n_store = n_store;
  g.relu = relu;
  g.n_models = h->G;
  g.slots = slots;
  g.count = count;
  g.num_sms = h->num_sms;
  MT(ie::launch_group_gemm(g, h->s));
  return IE_OK;
}

// mt_forward for the models `slots`: b rows each, row r of a model = X row rowidx[slot * s_idx + r]
int mg_forward(ie_mlp_group* h, const int* slots, int count, const int* rowidx, long long s_idx, int b, bool train) {
  const MgSlots S = mg_slots(h);
  const int m_pad = static_cast<int>(round_up(b, 128)), kb = static_cast<int>(round_up(b, 64));
  auto& L0 = h->layers[0];
  ie::GroupSplitArgs a{};
  a.a.src = h->X.as<float>();
  a.a.ld_src = L0.in;
  a.a.rowidx = rowidx;
  a.s_idx = s_idx;
  a.a.rows = b;
  a.a.cols = L0.in;
  a.a.rm = L0.act_rm.as<__nv_bfloat16>();
  a.s_rm = S.arm[0];
  a.a.ld_rm = 2 * L0.kp_in;
  a.a.rm_rows = m_pad;
  a.a.rm_kpad = L0.kp_in;
  if (train) {
    a.a.tr = L0.act_tr.as<__nv_bfloat16>();
    a.s_tr = S.atr[0];
    a.a.ld_tr = 2 * h->kb_cap;
    a.a.tr_rows = L0.mt_in;
    a.a.tr_kpad = kb;
  }
  a.slots = slots;
  a.count = count;
  MT(ie::launch_group_split_store(a, h->s));
  for (int l = 0; l < h->nl; ++l) {
    auto& L = h->layers[l];
    const bool last = l == h->nl - 1;
    int rc = mg_gemm(h, slots, count, L.act_rm.as<__nv_bfloat16>(), 2 * L.kp_in, h->cap_m, m_pad,
                     L.wt_s.as<__nv_bfloat16>(), 2 * L.kp_in, L.wt_rows, L.np, L.kp_in, h->P.as<float>() + L.boff,
                     h->n_param, last ? 0 : 1, L.z.as<float>(), L.n16, S.z[l], b, L.n16);
    if (rc != IE_OK) return rc;
    if (last) {
      ie::GroupOutputArgs o{};
      o.z = L.z.as<float>();
      o.p = h->pbuf.as<float>();
      o.delta = L.dz.as<float>();
      o.ldz = L.n16;
      o.s_z = S.z[l];
      o.s_p = S.pb;
      o.Y = train ? h->Y.as<uint8_t>() : nullptr;
      o.rowidx = rowidx;
      o.s_idx = s_idx;
      o.row_loss = h->row_loss.as<double>();
      o.s_rl = h->cap_m;
      o.b = b;
      o.L = L.out;
      o.slots = slots;
      o.count = count;
      MT(ie::launch_group_output(o, h->s));
      break;
    }
    auto& N = h->layers[l + 1];
    ie::GroupSplitArgs c{};
    c.a.src = L.z.as<float>();
    c.s_src = S.z[l];
    c.a.ld_src = L.n16;
    c.a.rows = b;
    c.a.cols = L.out;
    c.a.rm = N.act_rm.as<__nv_bfloat16>();
    c.s_rm = S.arm[l + 1];
    c.a.ld_rm = 2 * N.kp_in;
    c.a.rm_rows = m_pad;
    c.a.rm_kpad = N.kp_in;
    if (train) {
      c.a.tr = N.act_tr.as<__nv_bfloat16>();
      c.s_tr = S.atr[l + 1];
      c.a.ld_tr = 2 * h->kb_cap;
      c.a.tr_rows = N.mt_in;
      c.a.tr_kpad = kb;
    }
    c.slots = slots;
    c.count = count;
    MT(ie::launch_group_split_store(c, h->s));
  }
  return IE_OK;
}

// mt_backward + mt_adam for the models `slots` (b rows each), step k of their learning-rate and loss rows
int mg_backward_adam(ie_mlp_group* h, const int* slots, int count, int b, int k) {
  const MgSlots S = mg_slots(h);
  const int m_pad = static_cast<int>(round_up(b, 128)), kb = static_cast<int>(round_up(b, 64));
  {
    ie::GroupLossArgs g{};
    g.row_loss = h->row_loss.as<double>();
    g.s_rl = h->cap_m;
    g.sq_part = h->sq.as<double>();
    g.alpha = h->alpha.as<double>();
    g.out = h->losses.as<double>() + k;
    g.s_out = h->lr_pitch;
    g.b = b;
    g.slots = slots;
    g.count = count;
    MT(ie::launch_group_loss(g, h->s));
  }
  {
    const int l = h->nl - 1;
    auto& L = h->layers[l];
    ie::GroupSplitArgs a{};
    a.a.src = L.dz.as<float>();
    a.s_src = S.z[l];
    a.a.ld_src = L.n16;
    a.a.rows = b;
    a.a.cols = L.out;
    a.a.rm = L.d_rm.as<__nv_bfloat16>();
    a.s_rm = S.drm[l];
    a.a.ld_rm = 2 * L.kp_out;
    a.a.rm_rows = m_pad;
    a.a.rm_kpad = L.kp_out;
    a.a.tr = L.d_tr.as<__nv_bfloat16>();
    a.s_tr = S.dtr[l];
    a.a.ld_tr = 2 * h->kb_cap;
    a.a.tr_rows = L.np;
    a.a.tr_kpad = kb;
    a.slots = slots;
    a.count = count;
    MT(ie::launch_group_split_store(a, h->s));
  }
  for (int l = h->nl - 1; l >= 0; --l) {
    auto& L = h->layers[l];
    int rc = mg_gemm(h, slots, count, L.act_tr.as<__nv_bfloat16>(), 2 * h->kb_cap, L.mt_in, L.mt_in,
                     L.d_tr.as<__nv_bfloat16>(), 2 * h->kb_cap, L.dtr_rows, L.np, kb, nullptr, 0, 0,
                     h->dwbuf.as<float>(), L.n16, h->dw_max, L.in, L.n16);
    if (rc != IE_OK) return rc;
    ie::GroupGradArgs g{};
    g.dw = h->dwbuf.as<float>();
    g.ld_dw = L.n16;
    g.s_dw = h->dw_max;
    g.W = h->P.as<float>() + L.woff;
    g.gW = h->Gr.as<float>() + L.woff;
    g.gb = h->Gr.as<float>() + L.boff;
    g.s_param = h->n_param;
    g.delta = L.dz.as<float>();
    g.ld_delta = L.n16;
    g.s_delta = S.z[l];
    g.fan_in = L.in;
    g.fan_out = L.out;
    g.b = b;
    g.alpha = h->alpha.as<double>();
    g.slots = slots;
    g.count = count;
    MT(ie::launch_group_grad(g, h->s));
    if (l == 0) break;
    auto& P = h->layers[l - 1];
    rc = mg_gemm(h, slots, count, L.d_rm.as<__nv_bfloat16>(), 2 * L.kp_out, h->cap_m, m_pad, L.w_s.as<__nv_bfloat16>(),
                 2 * L.kp_out, L.w_rows, L.np_in, L.kp_out, nullptr, 0, 0, h->gbuf.as<float>(), P.n16, S.g, b, P.n16);
    if (rc != IE_OK) return rc;
    ie::GroupSplitArgs a{};
    a.a.src = h->gbuf.as<float>();
    a.s_src = S.g;
    a.a.ld_src = P.n16;
    a.a.rows = b;
    a.a.cols = P.out;
    a.a.mask = P.z.as<float>();
    a.s_mask = S.z[l - 1];
    a.a.ld_mask = P.n16;
    a.a.out_f32 = P.dz.as<float>();
    a.s_f32 = S.z[l - 1];
    a.a.ld_f32 = P.n16;
    a.a.rm = P.d_rm.as<__nv_bfloat16>();
    a.s_rm = S.drm[l - 1];
    a.a.ld_rm = 2 * P.kp_out;
    a.a.rm_rows = m_pad;
    a.a.rm_kpad = P.kp_out;
    a.a.tr = P.d_tr.as<__nv_bfloat16>();
    a.s_tr = S.dtr[l - 1];
    a.a.ld_tr = 2 * h->kb_cap;
    a.a.tr_rows = P.np;
    a.a.tr_kpad = kb;
    a.slots = slots;
    a.count = count;
    MT(ie::launch_group_split_store(a, h->s));
  }
  ie::GroupAdamArgs a = mg_adam_args(h, slots, count);
  a.g = h->Gr.as<float>();
  a.lr = h->lr.as<double>();
  a.s_lr = h->lr_pitch;
  a.step = k;
  MT(ie::launch_group_adam(a, h->s));
  return mg_refresh(h, slots, count);
}

int mg_model(const ie_mlp_group* h, int model) {
  if (model < 0 || model >= h->G) return fail(IE_ERR_INVALID, "model %d not in [0, %d)", model, h->G);
  return IE_OK;
}

int mg_ready(const ie_mlp_group* h, int model) {
  for (int l = 0; l < h->nl; ++l)
    if (!h->set[static_cast<size_t>(model) * h->nl + l])
      return fail(IE_ERR_STATE, "model %d: parameters not set (ie_mlp_group_set_layer for every layer)", model);
  if (!h->hyper[model]) return fail(IE_ERR_STATE, "model %d: constants not set (ie_mlp_group_set_hyper)", model);
  return IE_OK;
}

}  // namespace

extern "C" {

int ie_mlp_group_capacity(int32_t n_layers, const int32_t* dims, int32_t batch_size, int32_t device, double fraction,
                          int64_t* bytes_per_model, int32_t* max_models) {
  if (dims == nullptr || bytes_per_model == nullptr || max_models == nullptr || n_layers < 2 || n_layers > 16)
    return fail(IE_ERR_INVALID, "n_layers=%d: the trainer needs 1 to 15 hidden layers", n_layers);
  if (batch_size < 1) return fail(IE_ERR_INVALID, "batch_size=%d", batch_size);
  if (!(fraction > 0.0 && fraction <= 1.0)) return fail(IE_ERR_INVALID, "fraction=%g not in (0, 1]", fraction);
  for (int i = 0; i <= n_layers; ++i)
    if (dims[i] < 1 || dims[i] > (1 << 16)) return fail(IE_ERR_INVALID, "dims[%d]=%d not in [1, 65536]", i, dims[i]);
  int sms = 0;
  const int rc = open_device(device, &sms);
  if (rc != IE_OK) return rc;
  ie_mlp_group g;
  mg_geometry(&g, n_layers, dims, batch_size);
  const long long per = mg_bytes_per_model(&g);
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  *bytes_per_model = per;
  // the group kernels carry the model in gridDim.y / gridDim.z, at most 65535
  *max_models = static_cast<int32_t>(std::min<long long>(static_cast<long long>(free_b * fraction) / per, 65535));
  return IE_OK;
}

int ie_mlp_group_create(int32_t n_layers, const int32_t* dims, int32_t n_models, int32_t batch_size, int32_t device,
                        ie_mlp_group** out) {
  if (dims == nullptr || out == nullptr || n_layers < 2 || n_layers > 16)
    return fail(IE_ERR_INVALID, "n_layers=%d: the trainer needs 1 to 15 hidden layers", n_layers);
  for (int i = 0; i <= n_layers; ++i)
    if (dims[i] < 1 || dims[i] > (1 << 16)) return fail(IE_ERR_INVALID, "dims[%d]=%d not in [1, 65536]", i, dims[i]);
  if (n_models < 1 || n_models > 65535) return fail(IE_ERR_INVALID, "n_models=%d not in [1, 65535]", n_models);
  if (batch_size < 1) return fail(IE_ERR_INVALID, "batch_size=%d", batch_size);
  int sms = 0;
  const int rc = open_device(device, &sms);
  if (rc != IE_OK) return rc;
  ie_mlp_group* h = new ie_mlp_group();
  h->device = device;
  h->num_sms = sms;
  h->G = n_models;
  mg_geometry(h, n_layers, dims, batch_size);
  h->set.assign(static_cast<size_t>(n_models) * n_layers, false);
  h->hyper.assign(n_models, false);
  h->n_val.assign(n_models, 0);
  const size_t G = n_models, bf = sizeof(__nv_bfloat16);
  const MgSlots S = mg_slots(h);
  cudaError_t e = cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev1);
  for (DevBuf* b : {&h->P, &h->M, &h->V, &h->Gr, &h->best})
    if (e == cudaSuccess) e = b->reserve(G * h->n_param * sizeof(float), true);
  if (e == cudaSuccess) e = h->sq.reserve(G * ie::kAdamBlocks * sizeof(double), true);
  if (e == cudaSuccess) e = h->alpha.reserve(G * sizeof(double), true);
  if (e == cudaSuccess) e = h->consts.reserve(G * 5 * sizeof(float), true);
  if (e == cudaSuccess) e = h->gbuf.reserve(G * S.g * sizeof(float), true);
  if (e == cudaSuccess) e = h->dwbuf.reserve(G * h->dw_max * sizeof(float), true);
  if (e == cudaSuccess) e = h->row_loss.reserve(G * h->cap_m * sizeof(double), true);
  if (e == cudaSuccess) e = h->pbuf.reserve(G * S.pb * sizeof(float), true);
  for (int l = 0; l < n_layers && e == cudaSuccess; ++l) {
    auto& L = h->layers[l];
    e = L.wt_s.reserve(G * S.wt[l] * bf, true);
    if (e == cudaSuccess && l > 0) e = L.w_s.reserve(G * S.w[l] * bf, true);
    if (e == cudaSuccess) e = L.z.reserve(G * S.z[l] * sizeof(float), true);
    if (e == cudaSuccess) e = L.dz.reserve(G * S.z[l] * sizeof(float), true);
    if (e == cudaSuccess) e = L.act_rm.reserve(G * S.arm[l] * bf, true);
    if (e == cudaSuccess) e = L.act_tr.reserve(G * S.atr[l] * bf, true);
    if (e == cudaSuccess) e = L.d_rm.reserve(G * S.drm[l] * bf, true);
    if (e == cudaSuccess) e = L.d_tr.reserve(G * S.dtr[l] * bf, true);
  }
  if (e == cudaSuccess) {
    std::vector<int> ids(G);
    for (size_t i = 0; i < G; ++i) ids[i] = static_cast<int>(i);
    e = h->slot_ids.reserve(G * sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(h->slot_ids.p, ids.data(), G * sizeof(int), cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {
    ie_mlp_group_destroy(h);
    return cuda_fail(e, "ie_mlp_group_create");
  }
  *out = h;
  return IE_OK;
}

void ie_mlp_group_destroy(ie_mlp_group* h) {
  if (h == nullptr) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  if (h->s) cudaStreamDestroy(h->s);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
}

int ie_mlp_group_set_data(ie_mlp_group* h, const float* X, const uint8_t* Y, int64_t n) {
  if (h == nullptr || X == nullptr || Y == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (n < 1 || n >= (1ll << 31)) return fail(IE_ERR_INVALID, "n=%lld not in [1, 2^31)", static_cast<long long>(n));
  const int D = h->dims[0], Lo = h->dims[h->nl];
  const size_t cells = static_cast<size_t>(n) * D;
  for (size_t i = 0; i < cells; ++i)
    if (!std::isfinite(X[i])) return fail(IE_ERR_INVALID, "X[%zu][%zu] is not finite", i / D, i % D);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  const size_t G = h->G;
  const long long pitch = (n + h->bs - 1) / h->bs;
  CK(h->X.reserve(cells * sizeof(float)));
  CK(h->Y.reserve(static_cast<size_t>(n) * Lo));
  CK(h->order.reserve(G * n * sizeof(int)));
  CK(h->vrows.reserve(G * n * sizeof(int)));
  CK(h->lr.reserve(G * pitch * sizeof(double)));
  CK(h->losses.reserve(G * pitch * sizeof(double)));
  CK(cudaMemcpyAsync(h->X.p, X, cells * sizeof(float), cudaMemcpyHostToDevice, h->s));
  CK(cudaMemcpyAsync(h->Y.p, Y, static_cast<size_t>(n) * Lo, cudaMemcpyHostToDevice, h->s));
  CK(cudaStreamSynchronize(h->s));
  h->n = n;
  h->lr_pitch = pitch;
  std::fill(h->n_val.begin(), h->n_val.end(), 0);
  return IE_OK;
}

int ie_mlp_group_set_layer(ie_mlp_group* h, int32_t model, int32_t layer, const float* coef, const float* intercept) {
  if (h == nullptr || coef == nullptr || intercept == nullptr) return fail(IE_ERR_INVALID, "null argument");
  int rc = mg_model(h, model);
  if (rc != IE_OK) return rc;
  if (layer < 0 || layer >= h->nl) return fail(IE_ERR_INVALID, "layer %d out of range", layer);
  const auto& L = h->layers[layer];
  for (long long i = 0; i < static_cast<long long>(L.in) * L.out; ++i)
    if (!std::isfinite(coef[i])) return fail(IE_ERR_INVALID, "coef[%lld] is not finite", i);
  for (int i = 0; i < L.out; ++i)
    if (!std::isfinite(intercept[i])) return fail(IE_ERR_INVALID, "intercept[%d] is not finite", i);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  const long long o = static_cast<long long>(model) * h->n_param;
  CK(cudaMemcpyAsync(h->P.as<float>() + o + L.woff, coef, static_cast<size_t>(L.in) * L.out * sizeof(float),
                     cudaMemcpyHostToDevice, h->s));
  CK(cudaMemcpyAsync(h->P.as<float>() + o + L.boff, intercept, static_cast<size_t>(L.out) * sizeof(float),
                     cudaMemcpyHostToDevice, h->s));
  CK(cudaMemsetAsync(h->M.as<float>() + o, 0, h->n_param * sizeof(float), h->s));
  CK(cudaMemsetAsync(h->V.as<float>() + o, 0, h->n_param * sizeof(float), h->s));
  h->set[static_cast<size_t>(model) * h->nl + layer] = true;
  const int* slot = h->slot_ids.as<int>() + model;
  if ((rc = mg_refresh(h, slot, 1)) != IE_OK || (rc = mg_sq(h, slot, 1)) != IE_OK) return rc;
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int ie_mlp_group_get_layer(ie_mlp_group* h, int32_t model, int32_t layer, int32_t best, float* coef, float* intercept) {
  if (h == nullptr || coef == nullptr || intercept == nullptr) return fail(IE_ERR_INVALID, "null argument");
  int rc = mg_model(h, model);
  if (rc != IE_OK) return rc;
  if (layer < 0 || layer >= h->nl) return fail(IE_ERR_INVALID, "layer %d out of range", layer);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  const auto& L = h->layers[layer];
  const float* src = (best ? h->best : h->P).as<float>() + static_cast<long long>(model) * h->n_param;
  CK(cudaMemcpyAsync(coef, src + L.woff, static_cast<size_t>(L.in) * L.out * sizeof(float), cudaMemcpyDeviceToHost, h->s));
  CK(cudaMemcpyAsync(intercept, src + L.boff, static_cast<size_t>(L.out) * sizeof(float), cudaMemcpyDeviceToHost, h->s));
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int ie_mlp_group_set_hyper(ie_mlp_group* h, int32_t model, double alpha, double beta_1, double beta_2, double epsilon) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null argument");
  int rc = mg_model(h, model);
  if (rc != IE_OK) return rc;
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  // the f32 roundings mt_adam makes of the same Python doubles
  const float c[5] = {static_cast<float>(beta_1), static_cast<float>(1.0 - beta_1), static_cast<float>(beta_2),
                      static_cast<float>(1.0 - beta_2), static_cast<float>(epsilon)};
  CK(cudaMemcpyAsync(h->alpha.as<double>() + model, &alpha, sizeof(double), cudaMemcpyHostToDevice, h->s));
  CK(cudaMemcpyAsync(h->consts.as<float>() + 5 * model, c, sizeof(c), cudaMemcpyHostToDevice, h->s));
  CK(cudaStreamSynchronize(h->s));
  h->hyper[model] = true;
  return IE_OK;
}

int ie_mlp_group_set_validation(ie_mlp_group* h, int32_t model, const int32_t* rows, int64_t n_val) {
  if (h == nullptr || rows == nullptr) return fail(IE_ERR_INVALID, "null argument");
  int rc = mg_model(h, model);
  if (rc != IE_OK) return rc;
  if (h->n == 0) return fail(IE_ERR_STATE, "no data uploaded (ie_mlp_group_set_data)");
  if (n_val < 1 || n_val > h->n) return fail(IE_ERR_INVALID, "n_val=%lld not in [1, %lld]", static_cast<long long>(n_val), h->n);
  if ((rc = mt_check_rows(rows, n_val, h->n)) != IE_OK) return rc;
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpyAsync(h->vrows.as<int>() + static_cast<long long>(model) * h->n, rows, static_cast<size_t>(n_val) * sizeof(int),
                     cudaMemcpyHostToDevice, h->s));
  CK(cudaStreamSynchronize(h->s));
  h->n_val[model] = n_val;
  return IE_OK;
}

int ie_mlp_group_epoch(ie_mlp_group* h, int32_t n_active, const int32_t* models, const int64_t* n_rows,
                       const int32_t* rows, const double* lr, double* losses) {
  if (h == nullptr || models == nullptr || n_rows == nullptr || rows == nullptr || lr == nullptr || losses == nullptr)
    return fail(IE_ERR_INVALID, "null argument");
  if (n_active < 1 || n_active > h->G) return fail(IE_ERR_INVALID, "n_active=%d not in [1, %d]", n_active, h->G);
  if (h->n == 0) return fail(IE_ERR_STATE, "no data uploaded (ie_mlp_group_set_data)");
  std::lock_guard<std::mutex> lk(h->mu);
  std::vector<bool> seen(h->G, false);
  std::vector<long long> steps(n_active);
  long long max_steps = 0, row_off = 0;
  int rc;
  for (int i = 0; i < n_active; ++i) {
    if ((rc = mg_model(h, models[i])) != IE_OK || (rc = mg_ready(h, models[i])) != IE_OK) return rc;
    if (seen[models[i]]) return fail(IE_ERR_INVALID, "model %d listed twice", models[i]);
    seen[models[i]] = true;
    if (n_rows[i] < h->bs || n_rows[i] > h->n)
      return fail(IE_ERR_INVALID, "model %d: %lld rows, not in [batch_size %d, %lld]", models[i],
                  static_cast<long long>(n_rows[i]), h->bs, h->n);
    if ((rc = mt_check_rows(rows + row_off, n_rows[i], h->n)) != IE_OK) return rc;
    steps[i] = (n_rows[i] + h->bs - 1) / h->bs;
    max_steps = std::max(max_steps, steps[i]);
    row_off += n_rows[i];
  }
  CK(cudaSetDevice(h->device));
  // lockstep plan: at step k, the models still stepping, one launch sequence per batch size among them (a model's
  // short last batch, or a model with fewer steps, makes its own); the slot lists go up once
  struct Launch { long long k; int b, off, count; };
  std::vector<Launch> plan;
  std::vector<int> lists;
  for (long long k = 0; k < max_steps; ++k) {
    std::vector<std::pair<int, int>> bm;   // (b, slot)
    for (int i = 0; i < n_active; ++i)
      if (k < steps[i]) bm.emplace_back(static_cast<int>(std::min<long long>(h->bs, n_rows[i] - k * h->bs)), models[i]);
    std::stable_sort(bm.begin(), bm.end(), [](const std::pair<int, int>& a, const std::pair<int, int>& b) {
      return a.first > b.first;
    });
    for (size_t j = 0; j < bm.size();) {
      size_t e = j;
      while (e < bm.size() && bm[e].first == bm[j].first) ++e;
      const int count = static_cast<int>(e - j);
      bool same = !plan.empty() && plan.back().count == count && plan.back().b == bm[j].first;
      for (size_t t = 0; same && t < static_cast<size_t>(count); ++t) same = lists[plan.back().off + t] == bm[j + t].second;
      const int off = same ? plan.back().off : static_cast<int>(lists.size());
      if (!same)
        for (size_t t = j; t < e; ++t) lists.push_back(bm[t].second);
      plan.push_back({k, bm[j].first, off, count});
      j = e;
    }
  }
  CK(h->lists.reserve(lists.size() * sizeof(int)));
  CK(cudaMemcpyAsync(h->lists.p, lists.data(), lists.size() * sizeof(int), cudaMemcpyHostToDevice, h->s));
  row_off = 0;
  long long lr_off = 0;
  for (int i = 0; i < n_active; ++i) {
    const long long m = models[i];
    CK(cudaMemcpyAsync(h->order.as<int>() + m * h->n, rows + row_off, static_cast<size_t>(n_rows[i]) * sizeof(int),
                       cudaMemcpyHostToDevice, h->s));
    CK(cudaMemcpyAsync(h->lr.as<double>() + m * h->lr_pitch, lr + lr_off, static_cast<size_t>(steps[i]) * sizeof(double),
                       cudaMemcpyHostToDevice, h->s));
    row_off += n_rows[i];
    lr_off += steps[i];
  }
  CK(cudaEventRecord(h->ev0, h->s));
  for (const Launch& p : plan) {
    const int* slots = h->lists.as<int>() + p.off;
    const int step = static_cast<int>(p.k);
    if ((rc = mg_forward(h, slots, p.count, h->order.as<int>() + p.k * h->bs, h->n, p.b, true)) != IE_OK) return rc;
    if ((rc = mg_backward_adam(h, slots, p.count, p.b, step)) != IE_OK) return rc;
  }
  CK(cudaEventRecord(h->ev1, h->s));
  lr_off = 0;
  for (int i = 0; i < n_active; ++i) {
    CK(cudaMemcpyAsync(losses + lr_off, h->losses.as<double>() + static_cast<long long>(models[i]) * h->lr_pitch,
                       static_cast<size_t>(steps[i]) * sizeof(double), cudaMemcpyDeviceToHost, h->s));
    lr_off += steps[i];
  }
  CK(cudaStreamSynchronize(h->s));
  CK(cudaEventElapsedTime(&h->last_epoch_ms, h->ev0, h->ev1));
  return IE_OK;
}

int ie_mlp_group_validation_proba(ie_mlp_group* h, int32_t model, float* probs) {
  if (h == nullptr || probs == nullptr) return fail(IE_ERR_INVALID, "null argument");
  int rc = mg_model(h, model);
  if (rc != IE_OK || (rc = mg_ready(h, model)) != IE_OK) return rc;
  if (h->n_val[model] == 0) return fail(IE_ERR_STATE, "model %d: no validation rows (ie_mlp_group_set_validation)", model);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  const int Lo = h->dims[h->nl], ldp = h->layers.back().n16;
  const int* slot = h->slot_ids.as<int>() + model;
  const long long nv = h->n_val[model];
  const float* pb = h->pbuf.as<float>() + static_cast<long long>(model) * mg_slots(h).pb;
  for (long long r0 = 0; r0 < nv; r0 += h->cap) {
    const int rows = static_cast<int>(std::min<long long>(h->cap, nv - r0));
    // the model's rows vrows[model * n + r0 ...]: slot stride n, offset r0
    if ((rc = mg_forward(h, slot, 1, h->vrows.as<int>() + r0, h->n, rows, false)) != IE_OK) return rc;
    CK(cudaMemcpy2DAsync(probs + r0 * Lo, static_cast<size_t>(Lo) * sizeof(float), pb, ldp * sizeof(float),
                         static_cast<size_t>(Lo) * sizeof(float), rows, cudaMemcpyDeviceToHost, h->s));
  }
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int ie_mlp_group_snapshot(ie_mlp_group* h, int32_t model, int32_t restore) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null argument");
  int rc = mg_model(h, model);
  if (rc != IE_OK || (rc = mg_ready(h, model)) != IE_OK) return rc;
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->device));
  const size_t pb = static_cast<size_t>(h->n_param) * sizeof(float);
  const long long o = static_cast<long long>(model) * h->n_param;
  if (restore) {
    const int* slot = h->slot_ids.as<int>() + model;
    CK(cudaMemcpyAsync(h->P.as<float>() + o, h->best.as<float>() + o, pb, cudaMemcpyDeviceToDevice, h->s));
    if ((rc = mg_refresh(h, slot, 1)) != IE_OK || (rc = mg_sq(h, slot, 1)) != IE_OK) return rc;
  } else {
    CK(cudaMemcpyAsync(h->best.as<float>() + o, h->P.as<float>() + o, pb, cudaMemcpyDeviceToDevice, h->s));
  }
  CK(cudaStreamSynchronize(h->s));
  return IE_OK;
}

int64_t ie_mlp_group_launch_count(const ie_mlp_group* h) { return h ? h->launches : -1; }

int ie_mlp_group_last_epoch_ms(ie_mlp_group* h, float* ms) {
  if (h == nullptr || ms == nullptr) return fail(IE_ERR_INVALID, "null argument");
  *ms = h->last_epoch_ms;
  return IE_OK;
}

}  // extern "C"
#undef MT
