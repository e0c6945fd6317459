// C-ABI layer of libissue_emb_b200.so (declared in include/issue_emb_b200.h): handle management, weight
// re-layout, workspace, and the launch sequence of the encoder hot path and the MLP head.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include <cuda_fp16.h>

#include "../../include/issue_emb_b200.h"
#include "kernels.h"

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

int cuda_fail(cudaError_t e, const char* what) {
  const int code = (e == cudaErrorMemoryAllocation) ? IE_ERR_OOM : IE_ERR_CUDA;
  if (e == cudaErrorMemoryAllocation) cudaGetLastError();  // clear the sticky-free OOM
  return fail(code, "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
}

#define CK(expr)                                              \
  do {                                                        \
    cudaError_t _e = (expr);                                  \
    if (_e != cudaSuccess) return cuda_fail(_e, #expr);       \
  } while (0)

inline long long round_up(long long x, long long m) { return (x + m - 1) / m * m; }

// grow-only device buffer; owns its allocation (freed on destruction, so error paths do not leak)
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t bytes, bool zero = false) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) { p = nullptr; return e; }
    cap = bytes;
    if (zero) {
      // the handle's streams are non-blocking: make the (legacy-stream) memset complete before anyone uses it
      e = cudaMemset(p, 0, bytes);
      if (e != cudaSuccess) return e;
      return cudaDeviceSynchronize();
    }
    return cudaSuccess;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct Layer {
  int in = 0, out = 0;      // logical dims
  int u = 32, n_cta = 0;    // hidden units per weight slice, slices (even: a 256-column tile owns two)
  int out_pad = 0;          // n_cta * u
  int kin_pad = 0;          // padded K of the input projection
  int kh_pad = 0;           // padded K of the recurrent projection
  int bn = 0;               // GEMM N tile for the input projection
  DevBuf w_ih, w_hh, bias;  // sliced layouts
  DevBuf w_cat;             // last layer: rows [W_ih (kin_pad) | W_hh (kh_pad)] for the fused input projection
  bool loaded = false;
};

}  // namespace

struct ie_encoder {
  ie_config cfg{};
  int num_sms = 132;
  int e_pad = 0;  // emb_sz rounded up to 64
  // one weight layout: slices of u = 32 hidden units (slice_perm); two slices = one N = 256 accumulator tile of the
  // recurrent kernel (lstm_layer.cu)
  std::vector<Layer> layers;
  int segs = 1;            // 1: bf16 operands; 3: split-bf16 ("fp32-accurate", IE_CFG_FP32)
  int gate_mode = 2;       // lstm_common.cuh: 2 tanh.approx, 1 ex2+rcp, 0 IEEE
  int gx_bf16 = 1;         // input projections (Gx, per-token table) stored as 16-bit floats -- IEEE half -- instead of f32
                           // (f32 in the fp32-accurate mode)
  int use_persistent = 1;  // cooperative persistent launch; 0 (IE_SEQ=0 or not co-resident): one launch per timestep
  int persist_checked = 0;
  int cooperative = 1;     // launch attribute (IE_COOP=0: plain launch, co-residency by the occupancy check only)
  int use_mc = 0;          // IE_MC=1: sibling CTAs share h tiles by TMA multicast (clusters of two)
  int mc_ctas = 0;         // CTAs co-resident in clusters of two
  int batches = 5;         // batches of 256 rows one launch takes (IE_BATCHES, <= kMaxBatches)
  int fuse_last = 1;       // the last layer's input projection rides its recurrent K loop (lstm_layer.cu FUSE) instead of a
                           // hoisted GEMM + Gx round trip (IE_FUSE_LAST=0: hoisted like the other layers)
  int max_batch = 1280;
  // layer 0's input projection W_ih0 . Emb[id] + b depends on the token id alone: tabulated once per weight set
  // (proj: [vocab_pad, 4*out_pad], computed by the same GEMM from the same operands => the same bits as gather + GEMM)
  // and the recurrent kernel reads row tok[t, b] of it: no embedding gather, no layer-0 GEMM, no Gx write for layer 0
  int use_proj = 1;
  bool proj_built = false;
  DevBuf proj, tok;
  DevBuf emb;  // bf16 [vocab_pad, e_pad] (split mode: [hi | lo])
  bool emb_loaded = false;
  long long spin_limit = 0;  // SM cycles a device-side wait may take (0: default ~2 s); IE_SPIN_LIMIT_MS
  int fault = 0;             // IE_DEBUG_FAULT: exercise the abort protocol
  long long chunk_t = 0;     // IE_CHUNK_T: force the time-chunk length (testing)
  // workspace
  DevBuf ids, len_in, lengths, x0, y[2], hcarry, gx, c, pool_sum, pool_max, pool_last, out, raw, err, step_done, diag;
  DevBuf trace;           // debug timeline of one layer of the persistent kernel (ie_debug_seq_trace)
  int trace_layer = -1;
  int trace_T = 0, trace_ctas = 0;
  long long y_ld = 0;
  int small_calls = 0;      // consecutive calls far below the buffers that grow with T (workspace released after a few)
  cudaStream_t own_stream = nullptr;
  cudaStream_t last_stream = nullptr;
  cudaEvent_t done_ev = nullptr;  // end of the last call: a call on another stream waits for it (shared workspace)
  bool has_done = false;
  int64_t launches = 0;
  // phase boundary events of the last encode call and what ended at each (0 start, 1 gather, 2+2l gemm_l, 3+2l steps_l,
  // 2+2L finalize)
  std::vector<cudaEvent_t> ev;
  std::vector<int> ev_tag;
  int ev_used = 0;
  int last_T = 0, last_b_pad = 0;
  std::mutex mu;
};

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

namespace {

constexpr int kErrWords = 4;  // err[0] token id out of range, err[1] device-side wait timed out (abort protocol),
                              // err[2] a length had to be clamped (device-pointer mode)

int plan_layers(ie_encoder* h) {
  const ie_config& c = h->cfg;
  h->e_pad = static_cast<int>(round_up(c.emb_sz, 64));
  h->layers.resize(c.n_layers);
  int prev_pad = h->e_pad;
  for (int l = 0; l < c.n_layers; ++l) {
    Layer& L = h->layers[l];
    L.in = (l == 0) ? c.emb_sz : c.n_hid;
    L.out = (l == c.n_layers - 1) ? c.emb_sz : c.n_hid;
    L.u = 32;
    L.n_cta = (L.out + L.u - 1) / L.u;
    if (L.n_cta & 1) ++L.n_cta;  // whole tiles: the last tile's second slice is pure padding
    L.out_pad = L.n_cta * L.u;
    L.kin_pad = prev_pad;
    L.kh_pad = L.out_pad;        // multiple of 64
    prev_pad = L.kh_pad;
    L.bn = 256;                  // 4*out_pad is a multiple of 256
  }
  return IE_OK;
}

// torch gate-major rows [4*out] -> the recurrent kernel's column order; -1 marks zero padding rows.  A 256-column tile
// holds 64 units in 16 chunks of 16 columns; chunk m = 4s + e (s, e = 0..3) of the quad lane q has (i, f) at columns
// 2q, 2q+1 and (g, o) at 8+2q, 9+2q of the chunk -- exactly the columns lane q holds in a wgmma accumulator fragment
// (lstm_layer.cu), so a thread owns all four gates of a unit -- for unit 16s + 4q + e of the tile: a thread's units come
// in runs of four (one 16-byte access of c, one 8-byte store of h) and a warp's access covers whole sectors of a row.
// Only the N position of a weight row moves, so every accumulator element sums the same products in the same order.
std::vector<int> slice_perm(const Layer& L) {
  std::vector<int> perm(4 * static_cast<size_t>(L.out_pad));
  for (int unit = 0; unit < L.out_pad; ++unit)
    for (int g = 0; g < 4; ++g) {
      const int u = unit & 63, s = u >> 4, q = (u >> 2) & 3, e = u & 3;
      const size_t col = static_cast<size_t>(unit >> 6) * 256 + (4 * s + e) * 16 + (g < 2 ? 2 * q + g : 8 + 2 * q + (g - 2));
      perm[col] = unit < L.out ? g * L.out + unit : -1;
    }
  return perm;
}

// host f32 [rows_src, cols] -> device bf16 [perm.size(), ld] (split mode: [hi(k_pad) | lo(k_pad)], ld = 2*k_pad)
int upload_sliced(const float* host, int rows_src, int cols, const std::vector<int>& perm, int k_pad, int segs, DevBuf& dst,
                  cudaStream_t s) {
  DevBuf tmp, dperm;
  const int ld_dst = segs > 1 ? 2 * k_pad : k_pad;
  CK(tmp.reserve(static_cast<size_t>(rows_src) * cols * sizeof(float)));
  CK(dperm.reserve(perm.size() * sizeof(int)));
  CK(cudaMemcpyAsync(tmp.p, host, static_cast<size_t>(rows_src) * cols * sizeof(float), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(dperm.p, perm.data(), perm.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CK(dst.reserve(perm.size() * static_cast<size_t>(ld_dst) * sizeof(__nv_bfloat16)));
  CK(ie::launch_convert_rows(tmp.as<float>(), cols, cols, dperm.as<int>(), static_cast<int>(perm.size()),
                             dst.as<__nv_bfloat16>(), ld_dst, segs > 1 ? k_pad : 0, s));
  CK(cudaStreamSynchronize(s));
  tmp.release();
  dperm.release();
  return IE_OK;
}

long long max_out_pad(const ie_encoder* h) {
  long long m = 0;
  for (const Layer& L : h->layers) m = std::max<long long>(m, L.out_pad);
  return m;
}

void release_workspace(ie_encoder* h) {
  DevBuf* bufs[] = {&h->ids, &h->x0, &h->y[0], &h->y[1], &h->gx, &h->raw, &h->step_done, &h->tok};
  for (DevBuf* b : bufs) b->release();
  h->small_calls = 0;
}

// bytes held by the buffers that grow with T (the token ids, their time-major copy and the raw states)
long long t_bytes(const ie_encoder* h) {
  return static_cast<long long>(h->ids.cap + h->tok.cap + h->raw.cap);
}

// The time dimension is processed in chunks of chunk_T steps (time-major: every layer runs a chunk before the next
// chunk starts; c and h are carried per layer), so everything but the token ids, their time-major copy and the raw
// states is bounded by chunk_T * b_pad rows.  raw_ld > 0: the f32 states of one layer of out_pad raw_ld for the B valid
// rows.  *t_need receives the bytes this call needs of the buffers that grow with T.
int ensure_workspace(ie_encoder* h, int B, int b_pad, int T, int chunk_T, long long raw_ld, bool need_x0, bool need_tok,
                     long long* t_need) {
  const ie_config& c = h->cfg;
  const long long mop = max_out_pad(h);
  const long long rows = static_cast<long long>(T) * b_pad;
  const long long crow = static_cast<long long>(chunk_T) * b_pad;
  const int ring_mul = h->segs > 1 ? 2 : 1;
  const size_t ids_bytes = static_cast<size_t>(h->max_batch) * T * sizeof(int64_t);
  const size_t raw_bytes = static_cast<size_t>(B) * T * raw_ld * sizeof(float);
  const size_t tok_bytes = need_tok ? static_cast<size_t>(rows) * sizeof(int) : 0;
  *t_need = static_cast<long long>(ids_bytes + raw_bytes + tok_bytes);
  CK(h->ids.reserve(ids_bytes));
  CK(h->len_in.reserve(h->max_batch * sizeof(int)));
  CK(h->lengths.reserve(h->max_batch * sizeof(int)));
  CK(h->err.reserve(kErrWords * sizeof(int), true));
  CK(h->diag.reserve(static_cast<size_t>(c.n_layers) * 8 * sizeof(long long), true));
  if (need_x0) CK(h->x0.reserve(static_cast<size_t>(crow) * ring_mul * h->e_pad * sizeof(__nv_bfloat16)));
  // hidden-state rings of one chunk: (chunk_T + 1) slots of b_pad rows; slot 0 = the layer's h before the chunk (carry).
  // Every column a tensor map can reach is written before it is read (padded units produce exact zeros).
  h->y_ld = ring_mul * mop;
  const size_t ybytes = static_cast<size_t>(crow + b_pad) * h->y_ld * sizeof(__nv_bfloat16);
  for (int i = 0; i < 2; ++i) CK(h->y[i].reserve(ybytes));
  CK(h->hcarry.reserve(static_cast<size_t>(c.n_layers) * h->max_batch * h->y_ld * sizeof(__nv_bfloat16)));
  CK(h->gx.reserve(static_cast<size_t>(crow) * 4 * mop * (h->gx_bf16 ? 2 : 4)));
  CK(h->c.reserve(static_cast<size_t>(c.n_layers) * h->max_batch * mop * sizeof(float)));
  const size_t pb = static_cast<size_t>(h->max_batch) * mop * sizeof(float);
  CK(h->pool_sum.reserve(pb));
  CK(h->pool_max.reserve(pb));
  CK(h->pool_last.reserve(pb));
  CK(h->out.reserve(static_cast<size_t>(h->max_batch) * 3 * c.emb_sz * sizeof(float)));
  if (raw_bytes) CK(h->raw.reserve(raw_bytes));
  CK(h->step_done.reserve(static_cast<size_t>(chunk_T) * ie::kMaxBatches * sizeof(unsigned)));
  if (need_tok) CK(h->tok.reserve(tok_bytes));
  return IE_OK;
}

int mark(ie_encoder* h, int tag, cudaStream_t s) {
  if (h->ev_used >= static_cast<int>(h->ev.size())) {
    cudaEvent_t e;
    CK(cudaEventCreate(&e));
    h->ev.push_back(e);
    h->ev_tag.push_back(0);
  }
  h->ev_tag[h->ev_used] = tag;
  CK(cudaEventRecord(h->ev[h->ev_used++], s));
  return IE_OK;
}

bool proj_usable(const ie_encoder* h) {
  if (!h->use_proj) return false;
  const Layer& L = h->layers[0];
  const long long v_pad = round_up(h->cfg.vocab_sz, 256);
  const long long bytes = v_pad * 4ll * L.out_pad * (h->gx_bf16 ? 2 : 4);
  return bytes <= (6ll << 30);  // huge vocabularies fall back to gather + GEMM
}

void fill_gemm(const ie_encoder* h, const Layer& L, ie::GemmArgs& g) {
  g.b = L.w_ih.as<__nv_bfloat16>();
  g.ldb = static_cast<long long>(h->segs > 1 ? 2 : 1) * L.kin_pad;
  g.ldd = 4ll * L.out_pad;
  g.bias = L.bias.as<float>();
  g.n_pad = 4 * L.out_pad;
  g.k_pad = L.kin_pad;
  g.n_store = 4 * L.out_pad;
  g.bn = L.bn;
  g.act = 0;
  g.out_bf16 = h->gx_bf16 ? 2 : 0;  // fp16 or f32
  g.frag = 1;                        // Gx / table rows in the recurrent kernel's fragment order, bias likewise
  g.num_sms = h->num_sms;
  g.segs = h->segs;
  g.abort_flag = h->err.as<unsigned>() + 1;
  g.spin_limit = h->spin_limit;
}

// tabulate layer 0's input projection for every token id (once per weight set)
int build_proj_table(ie_encoder* h, cudaStream_t s) {
  const Layer& L = h->layers[0];
  const long long v_pad = round_up(h->cfg.vocab_sz, 256);
  CK(h->proj.reserve(static_cast<size_t>(v_pad) * 4 * L.out_pad * (h->gx_bf16 ? 2 : 4)));
  ie::GemmArgs g{};
  fill_gemm(h, L, g);
  g.a = h->emb.as<__nv_bfloat16>();
  g.lda = static_cast<long long>(h->segs > 1 ? 2 : 1) * h->e_pad;
  g.d = h->proj.p;
  g.m_pad = static_cast<int>(v_pad);
  g.m_store = static_cast<int>(v_pad);
  CK(ie::launch_gemm_bf16(g, s));
  h->launches++;
  h->proj_built = true;
  return IE_OK;
}

int check_persistent(ie_encoder* h, cudaStream_t s) {
  if (h->persist_checked) return IE_OK;
  for (const Layer& L : h->layers) {
    ie::LstmLayerArgs q{};
    q.T = 1; q.ng = 1; q.u = L.u; q.n_cta = L.n_cta; q.out_pad = L.out_pad; q.kh_pad = L.kh_pad; q.segs = 1;
    q.num_sms = h->num_sms; q.check_only = 1;
    if (ie::launch_lstm_layer(q, s) != cudaSuccess) h->use_persistent = 0;
  }
  if (h->use_mc) {
    ie::LstmLayerArgs q{};
    const Layer& L = h->layers[0];
    q.T = 1; q.ng = 1; q.u = L.u; q.n_cta = L.n_cta; q.out_pad = L.out_pad; q.kh_pad = L.kh_pad; q.segs = 1;
    q.num_sms = h->num_sms; q.check_only = 1; q.mc = 1; q.gx_bf16 = 1;
    if (ie::launch_lstm_layer(q, s) == cudaSuccess) h->mc_ctas = ie::lstm_layer_max_ctas() & ~1;
    if (h->mc_ctas < 2) h->use_mc = 0;
  }
  cudaGetLastError();
  h->persist_checked = 1;
  return IE_OK;
}

// a handle that once served a very long sequence does not keep its T-sized buffers -- nor the time-chunk buffers a
// single long issue grows to 2^20 rows -- for ever: after four consecutive calls that need under 1/8 of the bytes
// held by the buffers that grow with T (and those hold over 64 MB) the workspace is released; the next call grows it
// to its own size.  Calls of one shape never trigger it, nor do the short calls that follow bulk encodes at T <= 4096.
int maybe_release_workspace(ie_encoder* h, long long t_need, cudaStream_t s) {
  if (t_bytes(h) > (64ll << 20) && t_need * 8 < t_bytes(h)) {
    if (++h->small_calls >= 4) {
      CK(cudaStreamSynchronize(s));
      release_workspace(h);
    }
  } else {
    h->small_calls = 0;
  }
  return IE_OK;
}

// the launch sequence shared by encode (pooled), raw_features and the layer-state hook: raw_out (optional) receives the
// f32 hidden states of layer raw_layer as its recurrent kernel computed them, [B, T, out_l].  keep_raw (optional, the
// classifier): the states stay in the workspace (h->raw, [B, T, out_pad]) for kernels the caller enqueues next on `s`;
// the workspace is then not released here, *keep_raw receives the bytes for the caller's maybe_release_workspace.
int run_encoder(ie_encoder* h, const int64_t* ids, const int32_t* lengths, int B, int T, float* out, float* raw_out,
                int raw_layer, int flags, cudaStream_t s, long long* keep_raw = nullptr) {
  const ie_config& c = h->cfg;
  if (!h->emb_loaded) return fail(IE_ERR_STATE, "embedding not loaded");
  for (const Layer& L : h->layers)
    if (!L.loaded) return fail(IE_ERR_STATE, "LSTM layer weights not loaded");
  if (B < 1 || B > h->max_batch) return fail(IE_ERR_INVALID, "B=%d outside [1,%d]", B, h->max_batch);
  if (T < 1) return fail(IE_ERR_INVALID, "T=%d must be >= 1", T);
  const bool want_raw = raw_out != nullptr || keep_raw != nullptr;
  if (ids == nullptr || (out == nullptr && !want_raw)) return fail(IE_ERR_INVALID, "null pointer");
  if (want_raw && (raw_layer < 0 || raw_layer >= c.n_layers))
    return fail(IE_ERR_INVALID, "layer %d out of range", raw_layer);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  const bool pooled = out != nullptr;
  const int ng = (B + 255) / 256;
  const int b_pad = 256 * ng;
  // IE_MAX_TOKENS: artificial cap on B_pad*T (exercises the callers' OOM batch-halving loop); real limits come from
  // cudaMalloc (-> IE_ERR_OOM) -- only the token ids grow with T, everything else is bounded by the time chunk
  long long cap = 1ll << 27;
  if (const char* e = getenv("IE_MAX_TOKENS")) cap = std::max(256ll, atoll(e));
  if (static_cast<long long>(b_pad) * T > cap)
    return fail(IE_ERR_OOM, "B_pad*T = %lld tokens exceeds the workspace cap %lld; use a smaller batch",
                static_cast<long long>(b_pad) * T, cap);
  CK(cudaSetDevice(c.device));
  // <= 2^20 (timestep, row) pairs of Gx at once (20 GB as fp16 at H = 2400, plus 10 GB of hidden-state rings: well
  // inside the H100's 80 GB); half of that with f32 projections
  long long chunk_T = std::max<long long>(1, ((h->gx_bf16 ? 2ll : 1ll) << 19) / b_pad);
  if (h->chunk_t > 0) chunk_T = h->chunk_t;
  chunk_T = std::min<long long>(chunk_T, T);
  const bool proj = proj_usable(h);
  const long long raw_ld = want_raw ? h->layers[raw_layer].out_pad : 0;
  long long t_need = 0;
  int rc = ensure_workspace(h, B, b_pad, T, static_cast<int>(chunk_T), raw_ld, !proj, proj, &t_need);
  if (rc != IE_OK) return rc;
  if (h->done_ev == nullptr) CK(cudaEventCreateWithFlags(&h->done_ev, cudaEventDisableTiming));
  // one workspace per handle: a call on another stream first waits for the previous call
  if (h->has_done && h->last_stream != s) CK(cudaStreamWaitEvent(s, h->done_ev, 0));

  CK(cudaMemsetAsync(h->err.p, 0, kErrWords * sizeof(int), s));
  CK(cudaMemsetAsync(h->diag.p, 0, static_cast<size_t>(c.n_layers) * 8 * sizeof(long long), s));
  if (pooled) {
    if (lengths == nullptr) return fail(IE_ERR_INVALID, "lengths is null");
    const int* len_src = lengths;
    if (!dev) {
      for (int b = 0; b < B; ++b)
        if (lengths[b] < 1 || lengths[b] > T)
          return fail(IE_ERR_INVALID, "lengths[%d]=%d outside [1,%d]", b, lengths[b], T);
      CK(cudaMemcpyAsync(h->len_in.p, lengths, B * sizeof(int), cudaMemcpyHostToDevice, s));
      len_src = h->len_in.as<int>();
    }
    CK(ie::launch_prep_lengths(len_src, B, T, b_pad, h->lengths.as<int>(), h->err.as<int>(), s));
  }
  const int64_t* ids_dev = ids;
  if (!dev) {
    CK(cudaMemcpyAsync(h->ids.p, ids, static_cast<size_t>(B) * T * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    ids_dev = h->ids.as<int64_t>();
  }

  h->ev_used = 0;
  h->last_T = T;
  h->last_b_pad = b_pad;
  if (proj && !h->proj_built && (rc = build_proj_table(h, s)) != IE_OK) return rc;
  if ((rc = mark(h, 0, s)) != IE_OK) return rc;
  const int ring_mul = h->segs > 1 ? 2 : 1;
  const long long mop = max_out_pad(h);
  if (proj) {
    CK(ie::launch_tokens_time_major(ids_dev, B, T, b_pad, c.vocab_sz, c.pad_idx, h->tok.as<int>(), h->err.as<int>(), s));
    h->launches++;
  }
  if (h->use_persistent) check_persistent(h, s);
  const bool persistent = h->use_persistent != 0;
  // h_{-1} = 0 for every layer
  const size_t carry_layer = static_cast<size_t>(h->max_batch) * h->y_ld;  // elements
  CK(cudaMemsetAsync(h->hcarry.p, 0, static_cast<size_t>(c.n_layers) * carry_layer * sizeof(__nv_bfloat16), s));
  const size_t slot_bytes = static_cast<size_t>(b_pad) * h->y_ld * sizeof(__nv_bfloat16);

  for (long long t0 = 0; t0 < T; t0 += chunk_T) {
    const int Tc = static_cast<int>(std::min<long long>(chunk_T, T - t0));
    const long long crow = static_cast<long long>(Tc) * b_pad;
    if (!proj) {
      CK(ie::launch_embed_gather(ids_dev, B, T, b_pad, h->emb.as<__nv_bfloat16>(), c.vocab_sz, ring_mul * h->e_pad,
                                 h->x0.as<__nv_bfloat16>(), ring_mul * h->e_pad, c.pad_idx, h->err.as<int>(),
                                 static_cast<int>(t0), Tc, s));
      h->launches++;
    }
    if ((rc = mark(h, 1, s)) != IE_OK) return rc;
    int cur = 0;
    const __nv_bfloat16* layer_in = h->x0.as<__nv_bfloat16>();
    const __nv_bfloat16* prev_ring = nullptr;  // the previous layer's ring (slot 0 included)
    long long layer_in_ld = ring_mul * h->e_pad;
    for (int l = 0; l < c.n_layers; ++l) {
      const bool last = (l == c.n_layers - 1);
      Layer& L = h->layers[l];
      const bool from_table = proj && l == 0;  // Gx rows of layer 0 are rows of the per-token table: no GEMM
      // last layer: input projection fused into the recurrent K loop (no GEMM, no Gx)
      const bool fused = persistent && last && l > 0 && h->segs == 1 && h->fuse_last && L.w_cat.p != nullptr;
      __nv_bfloat16* ybuf = h->y[cur].as<__nv_bfloat16>();
      __nv_bfloat16* carry = h->hcarry.as<__nv_bfloat16>() + static_cast<size_t>(l) * carry_layer;
      float* cstate = h->c.as<float>() + static_cast<size_t>(l) * h->max_batch * mop;
      CUtensorMap tm_h, tm_w;
      CK(ie::make_tmap_bf16_2d(&tm_h, ybuf, static_cast<uint64_t>(ring_mul) * L.kh_pad, static_cast<uint64_t>(crow + b_pad),
                               h->y_ld, 64, 128));
      if (fused)
        CK(ie::make_tmap_bf16_2d(&tm_w, L.w_cat.p, static_cast<uint64_t>(L.kin_pad + L.kh_pad), 4ull * L.out_pad,
                                 static_cast<uint64_t>(L.kin_pad + L.kh_pad), 64, 256));
      else
        CK(ie::make_tmap_bf16_2d(&tm_w, L.w_hh.p, static_cast<uint64_t>(ring_mul) * L.kh_pad, 4ull * L.out_pad,
                                 static_cast<uint64_t>(ring_mul) * L.kh_pad, 64, 256));
      CUtensorMap tm_h64 = tm_h;
      CUtensorMap tm_x = tm_h;
      if (fused)
        CK(ie::make_tmap_bf16_2d(&tm_x, prev_ring, static_cast<uint64_t>(L.kin_pad), static_cast<uint64_t>(crow + b_pad),
                                 h->y_ld, 64, 128));
      if (h->use_mc)
        CK(ie::make_tmap_bf16_2d(&tm_h64, ybuf, static_cast<uint64_t>(ring_mul) * L.kh_pad,
                                 static_cast<uint64_t>(crow + b_pad), h->y_ld, 64, 64));
      // slot 0 of the ring = this layer's h at the end of the previous chunk (zeros before the first)
      CK(cudaMemcpyAsync(ybuf, carry, slot_bytes, cudaMemcpyDeviceToDevice, s));
      if (!from_table && !fused) {
        // hoisted input projection over the chunk's Tc*b_pad rows
        ie::GemmArgs g{};
        fill_gemm(h, L, g);
        g.a = layer_in;
        g.lda = layer_in_ld;
        g.d = h->gx.p;
        g.m_pad = static_cast<int>(crow);
        g.m_store = static_cast<int>(crow);
        g.diag = h->diag.as<long long>() + 8 * l + 4;
        CK(ie::launch_gemm_bf16(g, s));
        h->launches++;
      }
      if ((rc = mark(h, 2 + 2 * l, s)) != IE_OK) return rc;

      if (persistent) CK(cudaMemsetAsync(h->step_done.p, 0, static_cast<size_t>(Tc) * ng * sizeof(unsigned), s));
      ie::LstmLayerArgs q{};
      q.tm_h = tm_h; q.tm_w = tm_w; q.tm_h64 = tm_h64; q.mc = h->use_mc; q.mc_ctas = h->mc_ctas;
      q.tm_x = tm_x; q.pre_nkb = fused ? L.kin_pad / 64 : 0; q.bias = L.bias.as<float>();
      q.gx = from_table ? h->proj.p : h->gx.p;
      q.tok = from_table ? h->tok.as<int>() : nullptr;
      q.c = cstate; q.y = ybuf;
      q.raw = (l == raw_layer && want_raw) ? h->raw.as<float>() : nullptr;
      q.pool_sum = (last && pooled) ? h->pool_sum.as<float>() : nullptr;
      q.pool_max = h->pool_max.as<float>(); q.pool_last = h->pool_last.as<float>();
      q.lengths = h->lengths.as<int>();
      q.step_done = h->step_done.as<unsigned>();
      q.abort_flag = h->err.as<unsigned>() + 1; q.spin_limit = h->spin_limit;
      q.T = Tc; q.t0 = static_cast<int>(t0); q.T_total = T; q.ng = ng;
      q.u = L.u; q.n_cta = L.n_cta; q.out_pad = L.out_pad; q.kh_pad = L.kh_pad;
      q.ldy = h->y_ld; q.raw_ld = L.out_pad; q.raw_rows = B;
      q.gate_mode = h->gate_mode; q.gx_bf16 = h->gx_bf16; q.segs = h->segs;
      q.num_sms = h->num_sms; q.check_only = 0; q.cooperative = h->cooperative; q.fault = h->fault;
      q.diag = h->diag.as<long long>() + 8 * l;
      q.trace = nullptr;
      if (persistent) {
        if (l == h->trace_layer && t0 == 0) {
          const int ctas = ie::lstm_layer_ctas(q);
          const long long items = (static_cast<long long>(Tc) * ng * L.n_cta + ctas - 1) / ctas;
          CK(h->trace.reserve(static_cast<size_t>(ctas) * items * 12 * sizeof(long long), true));
          q.trace = h->trace.as<long long>();
          q.trace_items = static_cast<int>(items);
          h->trace_T = static_cast<int>(items);
          h->trace_ctas = ctas;
        }
        cudaError_t e = ie::launch_lstm_layer(q, s);
        if (e == cudaErrorCooperativeLaunchTooLarge) {
          cudaGetLastError();
          return fail(IE_ERR_STATE, "the persistent recurrent kernel cannot be co-resident on this device "
                                   "(cooperative launch refused); set IE_SEQ=0 for the per-timestep fallback");
        }
        CK(e);
        h->launches += 1;
      } else {
        q.single_step = 1;
        q.diag = nullptr;
        for (int t = 0; t < Tc; ++t) {
          q.t_step = t;
          CK(ie::launch_lstm_layer(q, s));
        }
        h->launches += Tc;
      }
      if (t0 + Tc < T)  // carry h of the chunk's last step into the next chunk
        CK(cudaMemcpyAsync(carry, ybuf + static_cast<size_t>(Tc) * b_pad * h->y_ld, slot_bytes, cudaMemcpyDeviceToDevice, s));
      if ((rc = mark(h, 3 + 2 * l, s)) != IE_OK) return rc;
      prev_ring = ybuf;
      layer_in = ybuf + static_cast<long long>(b_pad) * h->y_ld;  // slot 1 onwards
      layer_in_ld = h->y_ld;
      cur ^= 1;
    }
  }
  const Layer& LL = h->layers.back();
  if (pooled) {
    float* out_dev = dev ? out : h->out.as<float>();
    CK(ie::launch_pool_finalize(h->pool_sum.as<float>(), h->pool_max.as<float>(), h->pool_last.as<float>(),
                                h->lengths.as<int>(), B, c.emb_sz, LL.out_pad, out_dev, s));
    h->launches++;
    if ((rc = mark(h, 2 + 2 * c.n_layers, s)) != IE_OK) return rc;
    if (!dev)
      CK(cudaMemcpyAsync(out, out_dev, static_cast<size_t>(B) * 3 * c.emb_sz * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  if (raw_out != nullptr) {
    // raw workspace is [B, T, out_pad] of the requested layer; compact to [B, T, out]
    const Layer& LR = h->layers[raw_layer];
    CK(cudaMemcpy2DAsync(raw_out, static_cast<size_t>(LR.out) * sizeof(float), h->raw.p,
                         static_cast<size_t>(LR.out_pad) * sizeof(float), static_cast<size_t>(LR.out) * sizeof(float),
                         static_cast<size_t>(B) * T, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s));
  }
  CK(cudaEventRecord(h->done_ev, s));
  h->has_done = true;
  h->last_stream = s;
  if (keep_raw != nullptr) {
    *keep_raw = t_need;
    return IE_OK;
  }
  return maybe_release_workspace(h, t_need, s);
}

// read and clear the device error words of the last call (waits for it)
int collect_errors(ie_encoder* h) {
  if (!h->has_done) return IE_OK;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventSynchronize(h->done_ev));
  int w[kErrWords] = {0, 0, 0, 0};
  CK(cudaMemcpy(w, h->err.p, sizeof(w), cudaMemcpyDeviceToHost));
  if (w[0] | w[1] | w[2]) CK(cudaMemset(h->err.p, 0, sizeof(w)));
  if (w[1] != 0) {
    h->use_persistent = h->fault ? h->use_persistent : 0;  // do not walk into the same wall again
    return fail(IE_ERR_CUDA, "a device-side wait exceeded its limit and the kernel was drained (the persistent grid lost "
                             "co-residency, or a protocol error); results of this call are invalid");
  }
  if (w[0] != 0) return fail(IE_ERR_TOKEN, "token id outside [0,%d) in ids", h->cfg.vocab_sz);
  if (w[2] != 0) return fail(IE_ERR_INVALID, "a length outside [1,T] was clamped");
  return IE_OK;
}

}  // namespace

extern "C" {

int ie_version(void) { return 200; }

const char* ie_last_error(void) { return g_last_error.c_str(); }

int ie_encoder_create(const ie_config* cfg, ie_encoder** out) {
  if (cfg == nullptr || out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (cfg->n_layers < 1 || cfg->n_layers > 16 || cfg->emb_sz < 1 || cfg->n_hid < 1 || cfg->vocab_sz < 1 ||
      cfg->pad_idx < 0 || cfg->pad_idx >= cfg->vocab_sz)
    return fail(IE_ERR_INVALID, "bad encoder config");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback",
                cudaGetErrorString(e));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", cfg->device, ndev);
  CK(cudaSetDevice(cfg->device));
  int major = 0, sms = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, cfg->device));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device));
  if (major != 9) return fail(IE_ERR_CUDA, "device compute capability %d.x is not sm_90 (H100)", major);
  ie_encoder* h = new ie_encoder();
  h->cfg = *cfg;
  h->num_sms = sms;
  if (cfg->flags & IE_CFG_FP32) {  // split-bf16 products (~fp32), f32 Gx, IEEE gates
    h->segs = 3;
    h->gx_bf16 = 0;
    h->gate_mode = 0;
  } else {
    h->gate_mode = (cfg->flags & IE_CFG_ACCURATE_GATES) ? 1 : 2;
    if (cfg->flags & IE_CFG_F32_GX) h->gx_bf16 = 0;
  }
  // development knobs (DESIGN.md section 4); none is needed in production
  if (const char* v = getenv("IE_SEQ")) h->use_persistent = atoi(v);
  if (const char* v = getenv("IE_COOP")) h->cooperative = atoi(v);
  if (const char* v = getenv("IE_MC")) h->use_mc = atoi(v);
  if (const char* v = getenv("IE_EMB_PROJ")) h->use_proj = atoi(v);
  if (const char* v = getenv("IE_GX_BF16")) { if (h->segs == 1) h->gx_bf16 = atoi(v); }
  if (const char* v = getenv("IE_FAST_MATH")) { if (h->segs == 1) h->gate_mode = atoi(v) ? 2 : 1; }
  if (const char* v = getenv("IE_FUSE_LAST")) h->fuse_last = atoi(v);
  if (const char* v = getenv("IE_BATCHES")) h->batches = std::min(ie::kMaxBatches, std::max(1, atoi(v)));
  if (const char* v = getenv("IE_SPIN_LIMIT_MS")) h->spin_limit = static_cast<long long>(atof(v) * 1.9e6);
  if (const char* v = getenv("IE_DEBUG_FAULT")) h->fault = atoi(v);
  if (const char* v = getenv("IE_CHUNK_T")) h->chunk_t = atoll(v);
  h->max_batch = 256 * h->batches;
  int rc = plan_layers(h);
  if (rc != IE_OK) { delete h; return rc; }
  e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete h; return cuda_fail(e, "cudaStreamCreate"); }
  *out = h;
  return IE_OK;
}

void ie_encoder_destroy(ie_encoder* h) {
  if (h == nullptr) return;
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  for (Layer& L : h->layers) { L.w_ih.release(); L.w_hh.release(); L.bias.release(); L.w_cat.release(); }
  DevBuf* bufs[] = {&h->emb, &h->ids, &h->len_in, &h->lengths, &h->x0, &h->y[0], &h->y[1], &h->gx, &h->c, &h->pool_sum,
                    &h->pool_max, &h->pool_last, &h->out, &h->raw, &h->err, &h->step_done, &h->trace, &h->proj, &h->tok,
                    &h->diag, &h->hcarry};
  for (DevBuf* b : bufs) b->release();
  for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
  if (h->done_ev) cudaEventDestroy(h->done_ev);
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  delete h;
}

int ie_encoder_load_embedding(ie_encoder* h, const float* emb) {
  if (h == nullptr || emb == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->cfg.device));
  // the per-token table GEMM reads the embedding as its A operand: rows padded to whole M tiles (zeros)
  const int v_rows = static_cast<int>(round_up(h->cfg.vocab_sz, 256));
  std::vector<int> ident(v_rows);
  for (int i = 0; i < v_rows; ++i) ident[i] = i < h->cfg.vocab_sz ? i : -1;
  int rc = upload_sliced(emb, h->cfg.vocab_sz, h->cfg.emb_sz, ident, h->e_pad, h->segs, h->emb, h->own_stream);
  if (rc != IE_OK) return rc;
  h->emb_loaded = true;
  h->proj_built = false;
  return IE_OK;
}

int ie_encoder_load_layer(ie_encoder* h, int32_t layer, const float* w_ih, const float* w_hh, const float* b_ih,
                          const float* b_hh) {
  if (h == nullptr || w_ih == nullptr || w_hh == nullptr || b_ih == nullptr || b_hh == nullptr)
    return fail(IE_ERR_INVALID, "null argument");
  if (layer < 0 || layer >= h->cfg.n_layers) return fail(IE_ERR_INVALID, "layer %d out of range", layer);
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->cfg.device));
  Layer& L = h->layers[layer];
  const std::vector<int> perm = slice_perm(L);
  int rc = upload_sliced(w_ih, 4 * L.out, L.in, perm, L.kin_pad, h->segs, L.w_ih, h->own_stream);
  if (rc != IE_OK) return rc;
  rc = upload_sliced(w_hh, 4 * L.out, L.out, perm, L.kh_pad, h->segs, L.w_hh, h->own_stream);
  if (rc != IE_OK) return rc;
  // b_ih + b_hh in the fragment order of the Gx it is folded into (kernels.h frag_index, f32): the projection GEMM and
  // the fused last layer read it as one float4 (i, f, g, o) per unit
  std::vector<float> bias(perm.size());
  for (size_t r = 0; r < perm.size(); ++r)
    bias[r / 256 * 256 + ie::frag_index(static_cast<int>(r % 256), 4)] = perm[r] < 0 ? 0.0f : b_ih[perm[r]] + b_hh[perm[r]];
  CK(L.bias.reserve(bias.size() * sizeof(float)));
  CK(cudaMemcpy(L.bias.p, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice));
  if (layer == h->cfg.n_layers - 1 && layer > 0 && h->segs == 1) {
    // [W_ih | W_hh] row by row: the B operand of the fused last layer (one tensor map, K = kin_pad + kh_pad)
    const size_t kc = static_cast<size_t>(L.kin_pad) + L.kh_pad, rows = 4 * static_cast<size_t>(L.out_pad);
    CK(L.w_cat.reserve(rows * kc * sizeof(__nv_bfloat16)));
    CK(cudaMemcpy2D(L.w_cat.p, kc * 2, L.w_ih.p, static_cast<size_t>(L.kin_pad) * 2, static_cast<size_t>(L.kin_pad) * 2, rows,
                    cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy2D(L.w_cat.as<__nv_bfloat16>() + L.kin_pad, kc * 2, L.w_hh.p, static_cast<size_t>(L.kh_pad) * 2,
                    static_cast<size_t>(L.kh_pad) * 2, rows, cudaMemcpyDeviceToDevice));
  }
  L.loaded = true;
  if (layer == 0) h->proj_built = false;
  return IE_OK;
}

int ie_encoder_encode(ie_encoder* h, const int64_t* ids, const int32_t* lengths, int32_t B, int32_t T, float* out,
                      int32_t flags, void* stream) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (out == nullptr) return fail(IE_ERR_INVALID, "out is null");
  if (ids == nullptr || lengths == nullptr) return fail(IE_ERR_INVALID, "null pointer");
  std::lock_guard<std::mutex> lk(h->mu);
  // device-pointer mode: `stream` is used verbatim (NULL = the legacy default stream, e.g. torch's default);
  // host-pointer mode: NULL selects the handle's own stream
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  cudaStream_t s = (stream || dev) ? static_cast<cudaStream_t>(stream) : h->own_stream;
  int rc = run_encoder(h, ids, lengths, B, T, out, nullptr, -1, flags, s);
  if (rc != IE_OK || dev) return rc;
  return collect_errors(h);  // host-pointer mode: synchronous, device-side errors are reported by this call
}

int ie_encoder_raw_features(ie_encoder* h, const int64_t* ids, int32_t B, int32_t T, float* raw, int32_t flags,
                            void* stream) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (raw == nullptr) return fail(IE_ERR_INVALID, "raw is null");
  std::lock_guard<std::mutex> lk(h->mu);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  cudaStream_t s = (stream || dev) ? static_cast<cudaStream_t>(stream) : h->own_stream;
  int rc = run_encoder(h, ids, nullptr, B, T, nullptr, raw, h->cfg.n_layers - 1, flags, s);
  if (rc != IE_OK || dev) return rc;
  return collect_errors(h);
}

int ie_debug_layer_states(ie_encoder* h, int32_t layer, const int64_t* ids, int32_t B, int32_t T, float* out,
                          int32_t flags, void* stream) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (out == nullptr) return fail(IE_ERR_INVALID, "out is null");
  std::lock_guard<std::mutex> lk(h->mu);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  cudaStream_t s = (stream || dev) ? static_cast<cudaStream_t>(stream) : h->own_stream;
  int rc = run_encoder(h, ids, nullptr, B, T, nullptr, out, layer, flags, s);
  if (rc != IE_OK || dev) return rc;
  return collect_errors(h);
}

int ie_encoder_check_errors(ie_encoder* h) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  return collect_errors(h);
}

int64_t ie_encoder_launch_count(const ie_encoder* h) { return h ? h->launches : 0; }

int32_t ie_encoder_max_batch(const ie_encoder* h) { return h ? h->max_batch : IE_MAX_BATCH; }

int64_t ie_debug_workspace_bytes(const ie_encoder* h) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  std::lock_guard<std::mutex> lk(const_cast<ie_encoder*>(h)->mu);
  const DevBuf* bufs[] = {&h->ids, &h->len_in, &h->lengths, &h->x0, &h->y[0], &h->y[1], &h->hcarry, &h->gx, &h->c,
                          &h->pool_sum, &h->pool_max, &h->pool_last, &h->out, &h->raw, &h->err, &h->step_done,
                          &h->diag, &h->trace, &h->tok};
  int64_t n = 0;
  for (const DevBuf* b : bufs) n += static_cast<int64_t>(b->cap);
  return n;
}

// debug: request a per-item timeline of `layer` in the persistent kernel on the next encode (layer < 0: off);
// with out != NULL copy the last recorded timeline [ctas][items][12] and return ctas*items
int64_t ie_debug_seq_trace(ie_encoder* h, int32_t layer, long long* out, int64_t cap) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  h->trace_layer = layer;
  if (out == nullptr) return 0;
  const int64_t n = static_cast<int64_t>(h->trace_ctas) * h->trace_T;
  if (n == 0 || n * 12 > cap) return fail(IE_ERR_STATE, "no trace recorded or buffer too small");
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  if (cudaMemcpy(out, h->trace.p, n * 12 * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess)
    return fail(IE_ERR_CUDA, "trace copy failed");
  return n;
}

int ie_encoder_last_phase_ms(ie_encoder* h, float* ms, int32_t cap) {
  if (h == nullptr || ms == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  if (h->ev_used < 2) return fail(IE_ERR_STATE, "no encode call recorded");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventSynchronize(h->ev[h->ev_used - 1]));
  const int n = 2 + 2 * h->cfg.n_layers;  // gather, (gemm_l, steps_l) x L, finalize
  std::vector<float> acc(n, 0.0f);
  for (int i = 1; i < h->ev_used; ++i) {
    float t = 0.0f;
    CK(cudaEventElapsedTime(&t, h->ev[i - 1], h->ev[i]));
    const int tag = h->ev_tag[i];
    if (tag >= 1 && tag <= n) acc[tag - 1] += t;  // time chunks of a layer add up
  }
  for (int i = 0; i < n && i < cap; ++i) ms[i] = acc[i];
  return n;
}

int ie_encoder_last_phase_mhz(ie_encoder* h, float* mhz, int32_t cap) {
  if (h == nullptr || mhz == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  if (!h->has_done) return fail(IE_ERR_STATE, "no encode call recorded");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventSynchronize(h->done_ev));
  const int L = h->cfg.n_layers;
  std::vector<long long> d(static_cast<size_t>(L) * 8);
  CK(cudaMemcpy(d.data(), h->diag.p, d.size() * sizeof(long long), cudaMemcpyDeviceToHost));
  // mhz[l] = recurrent kernel of layer l, mhz[L + l] = its input-projection GEMM (0 when the layer had none)
  for (int i = 0; i < 2 * L && i < cap; ++i) {
    const long long* q = d.data() + 8 * (i % L) + 4 * (i / L);
    const long long dc = q[2] - q[0], dn = q[3] - q[1];
    mhz[i] = (dn > 0 && dc > 0) ? static_cast<float>(1e3 * static_cast<double>(dc) / static_cast<double>(dn)) : 0.0f;
  }
  return 2 * h->cfg.n_layers;
}

// ---------------------------------------------------------------------------------------------
// MLP head
// ---------------------------------------------------------------------------------------------
int ie_mlp_create(int32_t n_layers, const int32_t* dims, int32_t device, ie_mlp** out) {
  if (dims == nullptr || out == nullptr || n_layers < 1 || n_layers > 16) return fail(IE_ERR_INVALID, "bad argument");
  for (int i = 0; i <= n_layers; ++i)
    if (dims[i] < 1) return fail(IE_ERR_INVALID, "dims[%d]=%d", i, dims[i]);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback",
                cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", device, ndev);
  CK(cudaSetDevice(device));
  int major = 0, sms = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  if (major != 9) return fail(IE_ERR_CUDA, "device compute capability %d.x is not sm_90 (H100)", major);
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
  e = cudaStreamCreateWithFlags(&m->own_stream, cudaStreamNonBlocking);
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
  std::vector<int> perm(L.n_pad);
  for (int r = 0; r < L.n_pad; ++r) perm[r] = r < fan_out ? r : -1;
  int rc = upload_sliced(wt.data(), fan_out, fan_in, perm, L.k_pad, 1, L.w, m->own_stream);
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
  cudaStream_t s = (stream || dev) ? static_cast<cudaStream_t>(stream) : m->own_stream;
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
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", device, ndev);
  CK(cudaSetDevice(device));
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
  for (auto& L : m->layers) { L.w.release(); L.b.release(); }
  m->xf.release(); m->act[0].release(); m->act[1].release(); m->probs.release(); m->xb.release();
  if (m->own_stream) cudaStreamDestroy(m->own_stream);
  delete m;
}

// frag: store in the fragment order of the encoder's input projections (kernels.h frag_index), undone here on the host
static int debug_gemm(const float* a, const float* b, const float* bias, int32_t M, int32_t N, int32_t K, int32_t act,
                      int32_t out_type, int32_t segs, float* d, int32_t device, bool frag) {
  if (a == nullptr || b == nullptr || d == nullptr || M < 1 || N < 1 || K < 1) return fail(IE_ERR_INVALID, "bad argument");
  if (act < 0 || act > 2 || out_type < 0 || out_type > 2 || (out_type == 2 && act != 0) || (segs != 1 && segs != 3))
    return fail(IE_ERR_INVALID, "act=%d out_type=%d segs=%d not supported", act, out_type, segs);
  if (frag && (bias == nullptr || act != 0 || out_type == 1 || N % 256 != 0))
    return fail(IE_ERR_INVALID, "fragment order needs a bias, act 0, f32 or fp16 output and N %% 256 == 0");
  CK(cudaSetDevice(device));
  int sms = 132;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  const int m_pad = static_cast<int>(round_up(M, 128)), k_pad = static_cast<int>(round_up(K, 64));
  const int n16 = static_cast<int>(round_up(N, 16));
  int bn = 16;
  if (n16 >= 240 && n16 % 240 == 0) bn = 240;
  else if (n16 >= 128) bn = 128;
  else bn = n16;
  if (frag) bn = 256;
  const int n_pad = static_cast<int>(round_up(N, bn));
  // split-bf16 operands are [hi(k_pad) | lo(k_pad)] per row, as upload_sliced lays out the encoder's weights
  const int ld = segs == 3 ? 2 * k_pad : k_pad;
  const size_t elt = out_type == 0 ? 4 : 2;
  DevBuf fa, fb, ba, bb, dd, db;
  cudaStream_t s = nullptr;
  CK(fa.reserve(static_cast<size_t>(M) * K * 4));
  CK(fb.reserve(static_cast<size_t>(N) * K * 4));
  CK(ba.reserve(static_cast<size_t>(m_pad) * ld * 2, true));
  CK(bb.reserve(static_cast<size_t>(n_pad) * ld * 2, true));
  CK(dd.reserve(static_cast<size_t>(m_pad) * n_pad * elt));
  CK(cudaMemcpy(fa.p, a, static_cast<size_t>(M) * K * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(fb.p, b, static_cast<size_t>(N) * K * 4, cudaMemcpyHostToDevice));
  const int lo_off = segs == 3 ? k_pad : 0;
  CK(ie::launch_convert_rows(fa.as<float>(), K, K, nullptr, M, ba.as<__nv_bfloat16>(), ld, lo_off, s));
  CK(ie::launch_convert_rows(fb.as<float>(), K, K, nullptr, N, bb.as<__nv_bfloat16>(), ld, lo_off, s));
  if (bias) {
    std::vector<float> bp(n_pad, 0.0f);
    if (frag) {
      for (int n = 0; n < N; ++n) bp[n / 256 * 256 + ie::frag_index(n % 256, 4)] = bias[n];
    } else {
      std::copy(bias, bias + N, bp.begin());
    }
    CK(db.reserve(n_pad * 4));
    CK(cudaMemcpy(db.p, bp.data(), n_pad * 4, cudaMemcpyHostToDevice));
  }
  ie::GemmArgs g{};
  g.a = ba.as<__nv_bfloat16>(); g.lda = ld;
  g.b = bb.as<__nv_bfloat16>(); g.ldb = ld;
  g.d = dd.p; g.ldd = n_pad;
  g.bias = bias ? db.as<float>() : nullptr;
  g.m_pad = m_pad; g.n_pad = n_pad; g.k_pad = k_pad;
  g.m_store = M; g.n_store = n_pad; g.bn = bn; g.act = act; g.out_bf16 = out_type; g.num_sms = sms; g.segs = segs;
  g.frag = frag ? 1 : 0;
  CK(ie::launch_gemm_bf16(g, s));
  if (frag) {
    // raw rows, then column n of each row from position frag_index(n % 256) of its tile
    std::vector<uint8_t> raw(static_cast<size_t>(M) * n_pad * elt);
    CK(cudaMemcpy(raw.data(), dd.p, raw.size(), cudaMemcpyDeviceToHost));
    for (size_t r = 0; r < static_cast<size_t>(M); ++r)
      for (int n = 0; n < N; ++n) {
        const size_t src = r * n_pad + n / 256 * 256 + ie::frag_index(n % 256, static_cast<int>(elt));
        if (out_type == 0) {
          std::memcpy(d + r * N + n, raw.data() + src * 4, 4);
        } else {
          __half_raw h;
          std::memcpy(&h.x, raw.data() + src * 2, 2);
          d[r * N + n] = __half2float(__half(h));
        }
      }
  } else if (out_type == 0) {
    CK(cudaMemcpy2D(d, static_cast<size_t>(N) * 4, dd.p, static_cast<size_t>(n_pad) * 4, static_cast<size_t>(N) * 4, M,
                    cudaMemcpyDeviceToHost));
  } else {
    // 16-bit results widened exactly to f32 on the host
    std::vector<uint16_t> h16(static_cast<size_t>(M) * N);
    CK(cudaMemcpy2D(h16.data(), static_cast<size_t>(N) * 2, dd.p, static_cast<size_t>(n_pad) * 2, static_cast<size_t>(N) * 2,
                    M, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < h16.size(); ++i) {
      if (out_type == 1) {
        const uint32_t bits = static_cast<uint32_t>(h16[i]) << 16;
        std::memcpy(d + i, &bits, 4);
      } else {
        __half_raw r;
        r.x = h16[i];
        d[i] = __half2float(__half(r));
      }
    }
  }
  return IE_OK;
}

int ie_debug_gemm_ex(const float* a, const float* b, const float* bias, int32_t M, int32_t N, int32_t K, int32_t act,
                     int32_t out_type, int32_t segs, float* d, int32_t device) {
  return debug_gemm(a, b, bias, M, N, K, act, out_type, segs, d, device, false);
}

int ie_debug_gemm_frag(const float* a, const float* b, const float* bias, int32_t M, int32_t N, int32_t K, int32_t out_type,
                       int32_t segs, float* d, int32_t device) {
  return debug_gemm(a, b, bias, M, N, K, 0, out_type, segs, d, device, true);
}

int64_t ie_debug_epilogue_layout(int32_t out_units, int32_t* perm, int64_t cap, int32_t* frag2, int32_t* frag4) {
  if (out_units < 1) return fail(IE_ERR_INVALID, "out_units=%d must be >= 1", out_units);
  Layer L;
  L.out = out_units;
  L.out_pad = static_cast<int>(round_up(out_units, 64));
  const std::vector<int> p = slice_perm(L);
  if (perm != nullptr && cap >= static_cast<int64_t>(p.size())) std::copy(p.begin(), p.end(), perm);
  for (int c = 0; c < 256; ++c) {
    if (frag2 != nullptr) frag2[c] = ie::frag_index(c, 2);
    if (frag4 != nullptr) frag4[c] = ie::frag_index(c, 4);
  }
  return static_cast<int64_t>(p.size());
}

int ie_debug_gemm(const float* a, const float* b, const float* bias, int32_t M, int32_t N, int32_t K, int32_t act,
                  float* d, int32_t device) {
  return ie_debug_gemm_ex(a, b, bias, M, N, K, act, 0, 1, d, device);
}

int ie_debug_gates(int32_t fn, const float* in, float* out, int64_t n, int32_t device, void* stream) {
  if (in == nullptr || out == nullptr || n < 0 || fn < 0 || fn > 8)
    return fail(IE_ERR_INVALID, "fn=%d n=%lld: bad argument", fn, static_cast<long long>(n));
  CK(cudaSetDevice(device));
  CK(ie::launch_debug_gates(fn, in, out, n, static_cast<cudaStream_t>(stream)));
  return IE_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// k-nearest-neighbour index (knn.cu)
// ---------------------------------------------------------------------------------------------
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
  cudaStream_t last_stream = nullptr;
  cudaEvent_t done_ev = nullptr;
  bool has_done = false;
  std::mutex mu;
};

namespace {

int knn_begin(ie_knn* h, bool dev, void* stream, cudaStream_t* s) {
  CK(cudaSetDevice(h->device));
  *s = (stream || dev) ? static_cast<cudaStream_t>(stream) : h->own_stream;
  if (h->has_done && *s != h->last_stream) CK(cudaStreamWaitEvent(*s, h->done_ev, 0));
  return IE_OK;
}

int knn_end(ie_knn* h, cudaStream_t s) {
  CK(cudaEventRecord(h->done_ev, s));
  h->last_stream = s;
  h->has_done = true;
  return IE_OK;
}

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
  cudaStream_t s;
  int rc = knn_begin(h, dev, stream, &s);
  if (rc != IE_OK) return rc;
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
  return knn_end(h, s);
}

}  // namespace

extern "C" {

int ie_knn_create(int32_t dim, int32_t metric, int32_t device, ie_knn** out) {
  if (out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (dim < 1 || dim > 8192) return fail(IE_ERR_INVALID, "dim=%d not in [1, 8192]", dim);
  if (metric != IE_KNN_COSINE && metric != IE_KNN_EUCLIDEAN) return fail(IE_ERR_INVALID, "metric=%d", metric);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", device, ndev);
  CK(cudaSetDevice(device));
  int major = 0, sms = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  if (major != 9) return fail(IE_ERR_CUDA, "device compute capability %d.x is not sm_90 (H100)", major);
  ie_knn* h = new ie_knn();
  h->dim = dim;
  h->metric = metric;
  h->device = device;
  h->num_sms = sms;
  h->k_pad = static_cast<int>(round_up(dim, 64));
  e = h->err.reserve(sizeof(int), true);
  if (e == cudaSuccess) e = h->center.reserve(static_cast<size_t>(h->k_pad) * sizeof(float));
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->done_ev, cudaEventDisableTiming);
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
  if (h->done_ev) cudaEventDestroy(h->done_ev);
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
  cudaStream_t s;
  int rc = knn_begin(h, dev, stream, &s);
  if (rc != IE_OK) return rc;
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
  return knn_end(h, s);
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
  if (h->has_done) CK(cudaEventSynchronize(h->done_ev));
  int w = 0;
  CK(cudaMemcpy(&w, h->err.p, sizeof(w), cudaMemcpyDeviceToHost));
  if (w == 0) return IE_OK;
  CK(cudaMemset(h->err.p, 0, sizeof(w)));
  CK(cudaDeviceSynchronize());
  if (w & 1) return fail(IE_ERR_INVALID, "a non-finite value was seen in device input (an added row or a query)");
  return fail(IE_ERR_INVALID, "a row of device input (an added row or a query) has a norm outside the index's range "
                              "[2^-48, 2^48] (0 is allowed)");
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// Label-MLP trainer (mlp_train.cu + the persistent GEMM in split-bf16)
// ---------------------------------------------------------------------------------------------
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
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", device, ndev);
  CK(cudaSetDevice(device));
  int major = 0, sms = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  if (major != 9) return fail(IE_ERR_CUDA, "device compute capability %d.x is not sm_90 (H100)", major);
  ie_mlp_train* h = new ie_mlp_train();
  h->device = device;
  h->num_sms = sms;
  h->nl = n_layers;
  h->dims.assign(dims, dims + n_layers + 1);
  h->layers.resize(n_layers);
  h->set.assign(n_layers, false);
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
  const size_t pb = static_cast<size_t>(h->n_param) * sizeof(float), bf = sizeof(__nv_bfloat16);
  e = cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking);
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
  struct L {
    int in = 0, out = 0, kp_in = 0, kp_out = 0, n16 = 0, bn = 0, np = 0, bn_in = 0, np_in = 0, mt_in = 0;
    int wt_rows = 0, w_rows = 0, dtr_rows = 0;   // np, np_in and np rounded to 256: B rows per slot
    long long woff = 0, boff = 0;
    DevBuf wt_s, w_s, z, dz, act_rm, act_tr, d_rm, d_tr;
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

// geometry of a group's layers (the same as ie_mlp_train_create's) and its workspace rows
void mg_geometry(ie_mlp_group* h, int n_layers, const int32_t* dims, int batch_size) {
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
    L.wt_rows = static_cast<int>(round_up(L.np, 256));
    L.w_rows = static_cast<int>(round_up(L.np_in, 256));
    L.dtr_rows = L.wt_rows;
    L.woff = off;
    off += round_up(static_cast<long long>(L.in) * L.out, 64);
    h->n_packed += static_cast<long long>(L.in) * L.out + L.out;
  }
  h->n_coef = off;
  for (auto& L : h->layers) {
    L.boff = off;
    off += round_up(L.out, 64);
  }
  h->n_param = off;
  h->bs = batch_size;
  h->cap = std::max(batch_size, 256);   // validation runs in chunks of `cap` rows
  h->cap_m = static_cast<int>(round_up(h->cap, 128));
  h->kb_cap = static_cast<int>(round_up(batch_size, 64));
  h->in16_max = 0;
  h->dw_max = 0;
  for (auto& L : h->layers) {
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
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", device, ndev);
  CK(cudaSetDevice(device));
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
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", device, ndev);
  CK(cudaSetDevice(device));
  int major = 0, sms = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  if (major != 9) return fail(IE_ERR_CUDA, "device compute capability %d.x is not sm_90 (H100)", major);
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
  e = cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking);
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

// ---------------------------------------------------------------------------------------------
// Text classifier: fastai text_classifier_learner (MultiBatchEncoder + PoolingLinearClassifier) in eval mode
// ---------------------------------------------------------------------------------------------
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
  cudaEvent_t done_ev = nullptr;
  bool has_done = false;
  cudaStream_t last_stream = nullptr;
  std::mutex mu;
};

namespace {

constexpr int kClasErrWords = 4;  // err[0] token id out of range, err[1] device wait timed out, err[2] bad window

int clas_max_width(const ie_clas* c) { return *std::max_element(c->dims.begin(), c->dims.end()); }

// the classifier's error words of the last call, then the encoder's (waits for the call; clears both)
int clas_collect(ie_clas* c) {
  if (!c->has_done) return IE_OK;
  int rc = collect_errors(c->enc);
  CK(cudaEventSynchronize(c->done_ev));
  int w[kClasErrWords] = {0, 0, 0, 0};
  CK(cudaMemcpy(w, c->err.p, sizeof(w), cudaMemcpyDeviceToHost));
  if (w[0] | w[1] | w[2]) CK(cudaMemset(c->err.p, 0, sizeof(w)));
  if (rc != IE_OK) return rc;
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
  std::lock_guard<std::mutex> lk_c(c->mu);
  std::lock_guard<std::mutex> lk_h(h->mu);
  cudaStream_t s = (stream || dev) ? static_cast<cudaStream_t>(stream) : h->own_stream;
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
  if (c->done_ev == nullptr) CK(cudaEventCreateWithFlags(&c->done_ev, cudaEventDisableTiming));
  if (c->has_done && c->last_stream != s) CK(cudaStreamWaitEvent(s, c->done_ev, 0));
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
    CK(cudaEventRecord(h->done_ev, s));
    if ((rc = maybe_release_workspace(h, t_need, s)) != IE_OK) return rc;
  }
  if (!dev) {
    CK(cudaMemcpyAsync(out, out_dev, static_cast<size_t>(B) * width * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (logits != nullptr && !pooled_only)
      CK(cudaMemcpyAsync(logits, logits_dev, static_cast<size_t>(B) * n_class * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaEventRecord(c->done_ev, s));
  c->has_done = true;
  c->last_stream = s;
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
  if (c->has_done) cudaEventSynchronize(c->done_ev);
  if (c->done_ev) cudaEventDestroy(c->done_ev);
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
  if (c->has_done) CK(cudaEventSynchronize(c->done_ev));  // an earlier call may still read this stage
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
  std::lock_guard<std::mutex> lk_c(c->mu);
  std::lock_guard<std::mutex> lk_h(c->enc->mu);
  CK(cudaSetDevice(c->enc->cfg.device));
  return clas_collect(c);
}

int64_t ie_clas_launch_count(const ie_clas* c) { return c ? c->launches : -1; }

}  // extern "C"
