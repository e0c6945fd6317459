// C-ABI layer of the language model (declared in include/issue_emb_b200.h) over a borrowed encoder: fastai
// language_model_learner's per-token cross-entropy and argmax (lm.cu), and text generation from a recurrent state
// carried across calls (lm_gen.cu).
#include "encoder_host.h"

using namespace ie;

// ---------------------------------------------------------------------------------------------
// Language model: fastai language_model_learner = SequentialRNN(AWD_LSTM, LinearDecoder), its per-token cross-entropy
// and argmax (csrc/lm.cu), evaluated chunk by chunk on the encoder's ring
// ---------------------------------------------------------------------------------------------
struct ie_lm {
  ie_encoder* enc = nullptr;  // borrowed: its weights, workspace, stream and error words
  int device = 0;
  int V = 0, E = 0, k_pad = 0;
  DevBuf w, bias;             // decoder [round_up(V, 256), (segs > 1 ? 2 : 1) * k_pad] bf16, bias [round_up(V, 256)] f32
  bool loaded = false;
  DevBuf part, tlogit, tgt, nll, lse, pred, hbuf, err;
  int64_t launches = 0;
  StreamOrder order;           // the LM's calls and the generation states' (they share the error words)
  std::mutex mu;
};

namespace {

constexpr int kLmErrWords = 4;  // err[0] bit 0: a target outside [0, V) other than -100 (device-pointer mode);
                                // bit 1: a sampled row of zero total weight; bit 2: a select index out of range

// one decoder call: the states of `rows` ring rows -> nll / lse / pred of their valid (step, batch row) entries
struct LmCall {
  ie_lm* lm;
  const int64_t* targets;   // device [B, T]
  float* nll;
  float* lse;
  int* pred;
  int B, T;
};

int lm_decode(LmCall* c, const __nv_bfloat16* ring, long long ld, int t0, int Tc, int rps, cudaStream_t s) {
  ie_lm* lm = c->lm;
  const ie_encoder* h = lm->enc;
  const long long rows = static_cast<long long>(Tc) * rps;
  CK(lm->part.reserve(static_cast<size_t>(rows) * ie::lm_slices(lm->V) * sizeof(ie::LmPart)));
  CK(lm->tlogit.reserve(static_cast<size_t>(rows) * sizeof(float)));
  ie::LmDecodeArgs a{};
  a.h = ring;
  a.ld_h = ld;
  a.w = lm->w.as<__nv_bfloat16>();
  a.bias = lm->bias.as<float>();
  a.targets = c->targets;
  a.rows = rows;
  a.rps = rps;
  a.B = c->B;
  a.T = c->T;
  a.t0 = t0;
  a.V = lm->V;
  a.k_pad = lm->k_pad;
  a.segs = h->segs;
  a.num_sms = h->num_sms;
  a.part = lm->part.as<ie::LmPart>();
  a.tlogit = lm->tlogit.as<float>();
  a.nll = c->nll;
  a.lse = c->lse;
  a.pred = c->pred;
  a.err = lm->err.as<int>();
  a.abort_flag = h->err.as<unsigned>() + 1;
  a.spin_limit = h->spin_limit;
  CK(ie::launch_lm_decode(a, s));
  lm->launches += 2;
  return IE_OK;
}

int lm_hook(void* ctx, const __nv_bfloat16* ring, long long ld, int t0, int Tc, int b_pad, cudaStream_t s) {
  return lm_decode(static_cast<LmCall*>(ctx), ring, ld, t0, Tc, b_pad, s);
}

// the LM's error words of the last call, then the encoder's (waits for the call; clears both)
int lm_collect(ie_lm* lm) {
  if (!lm->order.has_done) return IE_OK;
  const int rc_enc = collect_errors(lm->enc);
  int w[kLmErrWords] = {0, 0, 0, 0};
  const int rc = read_errors(lm->order, lm->err, w, kLmErrWords);
  if (rc != IE_OK) return rc;
  if (rc_enc != IE_OK) return rc_enc;
  if (w[0] & 1) return fail(IE_ERR_INVALID, "a target outside [0,%d) other than -100 (its nll is NaN)", lm->V);
  if (w[0] & 2) return fail(IE_ERR_INVALID, "a sampled row had no token of positive weight (token 0 was drawn)");
  if (w[0] & 4) return fail(IE_ERR_INVALID, "a select index outside the state's rows (row 0 was copied)");
  return IE_OK;
}

int lm_check_targets(const ie_lm* lm, const int64_t* targets, long long n) {
  for (long long i = 0; i < n; ++i)
    if (targets[i] != -100 && (targets[i] < 0 || targets[i] >= lm->V))
      return fail(IE_ERR_INVALID, "targets[%lld]=%lld outside [0,%d) and not -100", i, static_cast<long long>(targets[i]),
                  lm->V);
  return IE_OK;
}

// before a call on `s`: the LM's error words, cleared on `s` once the previous call (on any stream) is done with them
int lm_clear_errors(ie_lm* lm, cudaStream_t s) {
  CK(lm->err.reserve(kLmErrWords * sizeof(int), true));
  CK(lm->order.begin(s));
  CK(cudaMemsetAsync(lm->err.p, 0, kLmErrWords * sizeof(int), s));
  return IE_OK;
}

}  // namespace

extern "C" {

int ie_lm_create(ie_encoder* enc, ie_lm** out) {
  if (enc == nullptr || out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  ie_lm* lm = new ie_lm();
  lm->enc = enc;
  lm->device = enc->cfg.device;
  lm->V = enc->cfg.vocab_sz;
  lm->E = enc->cfg.emb_sz;
  lm->k_pad = enc->layers.back().out_pad;   // the ring's K: the last layer's padded width (its lo plane's offset)
  *out = lm;
  return IE_OK;
}

void ie_lm_destroy(ie_lm* lm) {
  if (lm == nullptr) return;
  cudaSetDevice(lm->device);
  lm->order.wait();
  delete lm;
}

int ie_lm_load_decoder(ie_lm* lm, const float* weight, const float* bias) {
  if (lm == nullptr || weight == nullptr) return fail(IE_ERR_INVALID, "null argument");
  const long long n = static_cast<long long>(lm->V) * lm->E;
  for (long long i = 0; i < n; ++i)
    if (!std::isfinite(weight[i])) return fail(IE_ERR_INVALID, "decoder weight element %lld is not finite", i);
  if (bias != nullptr)
    for (int j = 0; j < lm->V; ++j)
      if (!std::isfinite(bias[j])) return fail(IE_ERR_INVALID, "decoder bias element %d is not finite", j);
  std::lock_guard<std::mutex> lk(lm->mu);
  ie_encoder* h = lm->enc;
  CK(cudaSetDevice(lm->device));
  CK(lm->order.wait());   // an earlier call may still read the decoder
  const int v_pad = static_cast<int>(round_up(lm->V, 256));
  int rc = upload_sliced(weight, lm->V, lm->E, padded_identity(lm->V, v_pad), lm->k_pad, h->segs, lm->w, h->own_stream);
  if (rc != IE_OK) return rc;
  std::vector<float> b(v_pad, 0.0f);
  if (bias != nullptr) std::copy(bias, bias + lm->V, b.begin());
  CK(lm->bias.reserve(v_pad * sizeof(float)));
  CK(cudaMemcpy(lm->bias.p, b.data(), v_pad * sizeof(float), cudaMemcpyHostToDevice));
  lm->loaded = true;
  return IE_OK;
}

int ie_lm_forward(ie_lm* lm, const int64_t* ids, const int64_t* targets, int32_t B, int32_t T, float* nll, float* lse,
                  int32_t* pred, int32_t flags, void* stream) {
  if (lm == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (ids == nullptr || targets == nullptr || nll == nullptr) return fail(IE_ERR_INVALID, "null pointer");
  if (!lm->loaded) return fail(IE_ERR_STATE, "decoder not loaded");
  ie_encoder* h = lm->enc;
  if (B < 1 || B > h->max_batch) return fail(IE_ERR_INVALID, "B=%d outside [1,%d]", B, h->max_batch);
  if (T < 1) return fail(IE_ERR_INVALID, "T=%d must be >= 1", T);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  const long long n = static_cast<long long>(B) * T;
  int rc;
  if (!dev && (rc = lm_check_targets(lm, targets, n)) != IE_OK) return rc;
  std::scoped_lock lk(lm->mu, h->mu);
  cudaStream_t s = call_stream(flags, stream, h->own_stream);
  CK(cudaSetDevice(lm->device));
  if ((rc = lm_clear_errors(lm, s)) != IE_OK) return rc;
  LmCall call{lm, targets, nll, lse, pred, B, T};
  if (!dev) {
    CK(lm->tgt.reserve(n * sizeof(int64_t)));
    CK(lm->nll.reserve(n * sizeof(float)));
    CK(lm->lse.reserve(n * sizeof(float)));
    CK(lm->pred.reserve(n * sizeof(int)));
    CK(cudaMemcpyAsync(lm->tgt.p, targets, n * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    call = LmCall{lm, lm->tgt.as<int64_t>(), lm->nll.as<float>(), lm->lse.as<float>(), lm->pred.as<int>(), B, T};
  }
  const ChunkHook hook{lm_hook, &call};
  rc = run_encoder(h, ids, nullptr, B, T, nullptr, nullptr, -1, flags, s, nullptr, &hook);
  if (rc != IE_OK) return rc;
  if (!dev) {
    CK(cudaMemcpyAsync(nll, call.nll, n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (lse != nullptr) CK(cudaMemcpyAsync(lse, call.lse, n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (pred != nullptr) CK(cudaMemcpyAsync(pred, call.pred, n * sizeof(int), cudaMemcpyDeviceToHost, s));
  }
  CK(lm->order.end(s));
  if (dev) return IE_OK;
  return lm_collect(lm);
}

int ie_lm_check_errors(ie_lm* lm) {
  if (lm == nullptr) return fail(IE_ERR_INVALID, "null handle");
  std::scoped_lock lk(lm->mu, lm->enc->mu);
  CK(cudaSetDevice(lm->device));
  return lm_collect(lm);
}

int64_t ie_lm_launch_count(const ie_lm* lm) { return lm ? lm->launches : -1; }

int ie_debug_lm_decode(ie_lm* lm, const float* hs, const int64_t* targets, int32_t M, float* nll, float* lse,
                       int32_t* pred) {
  if (lm == nullptr || hs == nullptr || targets == nullptr || nll == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (!lm->loaded) return fail(IE_ERR_STATE, "decoder not loaded");
  if (M < 1 || M > (1 << 20)) return fail(IE_ERR_INVALID, "M=%d outside [1,2^20]", M);
  int rc = lm_check_targets(lm, targets, M);
  if (rc != IE_OK) return rc;
  std::scoped_lock lk(lm->mu, lm->enc->mu);
  ie_encoder* h = lm->enc;
  cudaStream_t s = h->own_stream;
  CK(cudaSetDevice(lm->device));
  CK(h->err.reserve(kErrWords * sizeof(int), true));   // the mainloop's abort word, before any encode
  if ((rc = lm_clear_errors(lm, s)) != IE_OK) return rc;
  // the states as the ring holds them: bf16 (split-bf16 [hi | lo] at offset k_pad), rows padded to whole 128-row blocks
  const int m_pad = static_cast<int>(round_up(M, 128));
  if ((rc = upload_sliced(hs, M, lm->E, padded_identity(M, m_pad), lm->k_pad, h->segs, lm->hbuf, s)) != IE_OK) return rc;
  CK(lm->tgt.reserve(M * sizeof(int64_t)));
  CK(lm->nll.reserve(M * sizeof(float)));
  CK(lm->lse.reserve(M * sizeof(float)));
  CK(lm->pred.reserve(M * sizeof(int)));
  CK(cudaMemcpyAsync(lm->tgt.p, targets, M * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  LmCall call{lm, lm->tgt.as<int64_t>(), lm->nll.as<float>(), lm->lse.as<float>(), lm->pred.as<int>(), M, 1};
  const long long ld = static_cast<long long>(h->segs > 1 ? 2 : 1) * lm->k_pad;
  if ((rc = lm_decode(&call, lm->hbuf.as<__nv_bfloat16>(), ld, 0, 1, m_pad, s)) != IE_OK) return rc;
  CK(cudaMemcpyAsync(nll, call.nll, M * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (lse != nullptr) CK(cudaMemcpyAsync(lse, call.lse, M * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (pred != nullptr) CK(cudaMemcpyAsync(pred, call.pred, M * sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(lm->order.end(s));
  CK(cudaStreamSynchronize(s));
  return IE_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// Text generation (csrc/lm_gen.cu): a recurrent state carried across language-model calls, the last step's logits by
// the persistent GEMM, and the per-step decisions of fastai's predict and beam_search
// ---------------------------------------------------------------------------------------------
struct ie_gen_state {
  ie_lm* lm = nullptr;        // borrowed
  int cap = 0;                // rows
  long long y_ld = 0;         // h row width (the encoder's ring pitch)
  long long h_layer = 0, c_layer = 0;
  DevBuf h[2], c[2];          // [n_layers][cap][y_ld] bf16, [n_layers][cap][max out_pad] f32 (EncState's layout);
                              // select gathers into the other pair
  int cur = 0;
  DevBuf logits;              // [cap, round_up(V, 256)] f32: the last step's logits
  DevBuf ids, u, out_idx, out_val, flags, parent, scores, values, tokens, nodes_in, nodes_out;   // host-pointer staging
};

namespace {

struct LmGenCall {
  ie_gen_state* st;
  int rows, T;
};

// after the last chunk's last layer: logits [rows, v_pad] = h_{T-1} W^T + b by the persistent GEMM (act 0, f32)
int lm_gen_hook(void* ctx, const __nv_bfloat16* ring, long long ld, int t0, int Tc, int b_pad, cudaStream_t s) {
  LmGenCall* call = static_cast<LmGenCall*>(ctx);
  if (t0 + Tc < call->T) return IE_OK;
  ie_lm* lm = call->st->lm;
  const ie_encoder* h = lm->enc;
  const int v_pad = static_cast<int>(round_up(lm->V, 256));
  ie::GemmArgs g{};
  g.a = ring + static_cast<size_t>(Tc - 1) * b_pad * ld;
  g.lda = ld;
  g.b = lm->w.as<__nv_bfloat16>();
  g.ldb = static_cast<long long>(h->segs > 1 ? 2 : 1) * lm->k_pad;
  g.d = call->st->logits.p;
  g.bias = lm->bias.as<float>();
  g.m_pad = b_pad;
  g.n_pad = v_pad;
  g.k_pad = lm->k_pad;
  g.ldd = v_pad;
  g.m_store = call->rows;
  g.n_store = v_pad;
  g.bn = 256;
  g.num_sms = h->num_sms;
  g.segs = h->segs;
  g.abort_flag = h->err.as<unsigned>() + 1;
  g.spin_limit = h->spin_limit;
  CK(ie::launch_gemm_bf16(g, s));
  lm->launches++;
  return IE_OK;
}

int gen_check_common(const ie_gen_state* st, const void* ids, int rows, int T) {
  if (st == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (ids == nullptr) return fail(IE_ERR_INVALID, "null pointer");
  if (!st->lm->loaded) return fail(IE_ERR_STATE, "decoder not loaded");
  if (rows < 1 || rows > st->cap) return fail(IE_ERR_INVALID, "rows=%d outside [1,%d] (the state's capacity)", rows, st->cap);
  if (T < 1) return fail(IE_ERR_INVALID, "T=%d must be >= 1", T);
  return IE_OK;
}

int gen_check_exclude(const ie_lm* lm, int exclude) {
  if (exclude < -1 || exclude >= lm->V) return fail(IE_ERR_INVALID, "exclude=%d outside [-1,%d)", exclude, lm->V);
  return IE_OK;
}

// the encoder over ids [rows, T] from the state and into it, then the last step's logits; both handles locked
int gen_forward(ie_gen_state* st, const int64_t* ids, int rows, int T, int flags, cudaStream_t s) {
  ie_lm* lm = st->lm;
  ie_encoder* h = lm->enc;
  CK(st->logits.reserve(static_cast<size_t>(st->cap) * round_up(lm->V, 256) * sizeof(float)));
  EncState es{st->h[st->cur].as<__nv_bfloat16>(), st->c[st->cur].as<float>(), st->h_layer, st->c_layer,
              st->c_layer / st->cap};
  LmGenCall call{st, rows, T};
  const ChunkHook hook{lm_gen_hook, &call};
  return run_encoder(h, ids, nullptr, rows, T, nullptr, nullptr, -1, flags, s, nullptr, &hook, &es);
}

// a host-pointer call's copies back are done: wait for it and report its device-side errors
int gen_finish(ie_lm* lm, cudaStream_t s, bool dev) {
  CK(lm->order.end(s));
  return dev ? IE_OK : lm_collect(lm);
}

}  // namespace

extern "C" {

int ie_gen_state_create(ie_lm* lm, int32_t rows, ie_gen_state** out) {
  if (lm == nullptr || out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  ie_encoder* h = lm->enc;
  if (rows < 1 || rows > h->max_batch) return fail(IE_ERR_INVALID, "rows=%d outside [1,%d]", rows, h->max_batch);
  auto* st = new ie_gen_state();
  st->lm = lm;
  st->cap = rows;
  st->y_ld = (h->segs > 1 ? 2 : 1) * max_out_pad(h);
  st->h_layer = static_cast<long long>(rows) * st->y_ld;
  st->c_layer = static_cast<long long>(rows) * max_out_pad(h);
  const int n_layers = h->cfg.n_layers;
  cudaError_t e = cudaSetDevice(lm->device);
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
    e = st->h[i].reserve(static_cast<size_t>(n_layers) * st->h_layer * sizeof(__nv_bfloat16), true);
    if (e == cudaSuccess) e = st->c[i].reserve(static_cast<size_t>(n_layers) * st->c_layer * sizeof(float), true);
  }
  if (e != cudaSuccess) {
    delete st;
    return cuda_fail(e, "ie_gen_state_create");
  }
  *out = st;
  return IE_OK;
}

void ie_gen_state_destroy(ie_gen_state* st) {
  if (st == nullptr) return;
  cudaSetDevice(st->lm->device);
  st->lm->order.wait();   // a call may still use the state's buffers
  delete st;
}

int ie_gen_state_reset(ie_gen_state* st) {
  if (st == nullptr) return fail(IE_ERR_INVALID, "null handle");
  ie_lm* lm = st->lm;
  std::scoped_lock lk(lm->mu, lm->enc->mu);
  CK(cudaSetDevice(lm->device));
  cudaStream_t s = lm->enc->own_stream;
  int rc = lm_clear_errors(lm, s);
  if (rc != IE_OK) return rc;
  CK(cudaMemsetAsync(st->h[st->cur].p, 0, st->h[st->cur].cap, s));
  CK(cudaMemsetAsync(st->c[st->cur].p, 0, st->c[st->cur].cap, s));
  CK(lm->order.end(s));
  CK(cudaStreamSynchronize(s));
  return IE_OK;
}

int ie_gen_topk(ie_gen_state* st, const int64_t* ids, int32_t rows, int32_t T, int32_t k, int32_t exclude,
                     float* values, int64_t* idx, int32_t flags, void* stream) {
  int rc = gen_check_common(st, ids, rows, T);
  if (rc != IE_OK) return rc;
  ie_lm* lm = st->lm;
  if (values == nullptr || idx == nullptr) return fail(IE_ERR_INVALID, "null pointer");
  if (k < 1 || k > std::min(ie::kLmTopkMax, lm->V)) return fail(IE_ERR_INVALID, "k=%d outside [1,%d]", k, std::min(ie::kLmTopkMax, lm->V));
  if ((rc = gen_check_exclude(lm, exclude)) != IE_OK) return rc;
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  std::scoped_lock lk(lm->mu, lm->enc->mu);
  CK(cudaSetDevice(lm->device));
  cudaStream_t s = call_stream(flags, stream, lm->enc->own_stream);
  if ((rc = lm_clear_errors(lm, s)) != IE_OK) return rc;
  if ((rc = gen_forward(st, ids, rows, T, flags, s)) != IE_OK) return rc;
  float* v = values;
  int64_t* ix = idx;
  const size_t n = static_cast<size_t>(rows) * k;
  if (!dev) {
    if ((rc = stage<float>(st->out_val, nullptr, n, s)) != IE_OK || (rc = stage<int64_t>(st->out_idx, nullptr, n, s)) != IE_OK)
      return rc;
    v = st->out_val.as<float>();
    ix = st->out_idx.as<int64_t>();
  }
  CK(ie::launch_lm_topk(st->logits.as<float>(), round_up(lm->V, 256), rows, lm->V, k, exclude, v, ix, s));
  lm->launches++;
  if (!dev) {
    CK(cudaMemcpyAsync(values, v, n * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(idx, ix, n * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  }
  return gen_finish(lm, s, dev);
}

int ie_gen_sample(ie_gen_state* st, const int64_t* ids, int32_t rows, int32_t T, const float* u, int32_t exclude,
                       double temperature, double min_p, int64_t* idx, int32_t* draw_flags, int32_t flags,
                       void* stream) {
  int rc = gen_check_common(st, ids, rows, T);
  if (rc != IE_OK) return rc;
  ie_lm* lm = st->lm;
  if (u == nullptr || idx == nullptr || draw_flags == nullptr) return fail(IE_ERR_INVALID, "null pointer");
  if ((rc = gen_check_exclude(lm, exclude)) != IE_OK) return rc;
  if (!(temperature > 0.0) || !std::isfinite(temperature))
    return fail(IE_ERR_INVALID, "temperature=%g must be finite and > 0", temperature);
  if (!(min_p == 0.0 || (min_p > 0.0 && min_p <= 1.0))) return fail(IE_ERR_INVALID, "min_p=%g outside (0,1] (0: none)", min_p);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  if (!dev)
    for (int r = 0; r < rows; ++r)
      if (!(u[r] >= 0.0f && u[r] < 1.0f)) return fail(IE_ERR_INVALID, "u[%d]=%g outside [0,1)", r, u[r]);
  std::scoped_lock lk(lm->mu, lm->enc->mu);
  CK(cudaSetDevice(lm->device));
  cudaStream_t s = call_stream(flags, stream, lm->enc->own_stream);
  if ((rc = lm_clear_errors(lm, s)) != IE_OK) return rc;
  const float* ud = u;
  int64_t* ix = idx;
  int* fl = draw_flags;
  if (!dev) {
    if ((rc = stage<float>(st->u, u, rows, s)) != IE_OK || (rc = stage<int64_t>(st->out_idx, nullptr, rows, s)) != IE_OK ||
        (rc = stage<int>(st->flags, nullptr, rows, s)) != IE_OK)
      return rc;
    ud = st->u.as<float>();
    ix = st->out_idx.as<int64_t>();
    fl = st->flags.as<int>();
  }
  if ((rc = gen_forward(st, ids, rows, T, flags, s)) != IE_OK) return rc;
  CK(ie::launch_lm_sample(st->logits.as<float>(), round_up(lm->V, 256), rows, lm->V, ud, exclude,
                          static_cast<float>(min_p), static_cast<float>(1.0 / temperature), ix, fl, lm->err.as<int>(), s));
  lm->launches++;
  if (!dev) {
    CK(cudaMemcpyAsync(idx, ix, rows * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(draw_flags, fl, rows * sizeof(int), cudaMemcpyDeviceToHost, s));
  }
  return gen_finish(lm, s, dev);
}

int ie_gen_select(ie_gen_state* st, const int32_t* parent, int32_t n, int32_t flags, void* stream) {
  if (st == nullptr || parent == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (n < 1 || n > st->cap) return fail(IE_ERR_INVALID, "n=%d outside [1,%d]", n, st->cap);
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  if (!dev)
    for (int i = 0; i < n; ++i)
      if (parent[i] < 0 || parent[i] >= st->cap)
        return fail(IE_ERR_INVALID, "parent[%d]=%d outside [0,%d)", i, parent[i], st->cap);
  ie_lm* lm = st->lm;
  std::scoped_lock lk(lm->mu, lm->enc->mu);
  CK(cudaSetDevice(lm->device));
  cudaStream_t s = call_stream(flags, stream, lm->enc->own_stream);
  int rc = lm_clear_errors(lm, s);
  if (rc != IE_OK) return rc;
  const int32_t* p = parent;
  if (!dev) {
    if ((rc = stage<int32_t>(st->parent, parent, n, s)) != IE_OK) return rc;
    p = st->parent.as<int32_t>();
  }
  const int L = lm->enc->cfg.n_layers, nxt = st->cur ^ 1;
  CK(ie::launch_gather_rows(st->h[st->cur].p, st->h[nxt].p, p, n, st->cap, st->y_ld * sizeof(__nv_bfloat16),
                            st->h_layer * sizeof(__nv_bfloat16), L, lm->err.as<int>(), s));
  CK(ie::launch_gather_rows(st->c[st->cur].p, st->c[nxt].p, p, n, st->cap, (st->c_layer / st->cap) * sizeof(float),
                            st->c_layer * sizeof(float), L, lm->err.as<int>(), s));
  lm->launches += 2;
  st->cur = nxt;
  return gen_finish(lm, s, dev);
}

int ie_gen_beam_select(ie_gen_state* st, const float* scores, const float* values, const int64_t* tokens, int32_t rows,
                      int32_t top_k, int32_t beam_sz, const int64_t* nodes, int32_t L, int32_t* parent, int64_t* token,
                      float* new_scores, int64_t* new_nodes, int32_t flags, void* stream) {
  if (st == nullptr || scores == nullptr || values == nullptr || tokens == nullptr || parent == nullptr ||
      token == nullptr || new_scores == nullptr || new_nodes == nullptr || (L > 0 && nodes == nullptr))
    return fail(IE_ERR_INVALID, "null argument");
  if (rows < 1 || top_k < 1 || beam_sz < 1 || L < 0)
    return fail(IE_ERR_INVALID, "rows=%d top_k=%d beam_sz=%d L=%d: each must be >= 1 (L >= 0)", rows, top_k, beam_sz, L);
  const long long cand = static_cast<long long>(rows) * top_k;
  if (cand > ie::kLmBeamMax)
    return fail(IE_ERR_INVALID, "rows * top_k = %lld candidates exceed %d", cand, ie::kLmBeamMax);
  const int keep = static_cast<int>(std::min<long long>(beam_sz, cand));
  const bool dev = (flags & IE_FLAG_DEVICE_PTRS) != 0;
  ie_lm* lm = st->lm;
  std::scoped_lock lk(lm->mu, lm->enc->mu);
  CK(cudaSetDevice(lm->device));
  cudaStream_t s = call_stream(flags, stream, lm->enc->own_stream);
  int rc = lm_clear_errors(lm, s);
  if (rc != IE_OK) return rc;
  const float *sc = scores, *va = values;
  const int64_t *tk = tokens, *nd = nodes;
  int32_t* pa = parent;
  int64_t *to = token, *nn = new_nodes;
  float* ns = new_scores;
  if (!dev) {
    if ((rc = stage<float>(st->scores, scores, rows, s)) != IE_OK || (rc = stage<float>(st->values, values, cand, s)) != IE_OK ||
        (rc = stage<int64_t>(st->tokens, tokens, cand, s)) != IE_OK ||
        (rc = stage<int64_t>(st->nodes_in, nullptr, static_cast<size_t>(rows) * L + 1, s)) != IE_OK ||
        (rc = stage<int32_t>(st->parent, nullptr, keep, s)) != IE_OK || (rc = stage<int64_t>(st->out_idx, nullptr, keep, s)) != IE_OK ||
        (rc = stage<float>(st->out_val, nullptr, keep, s)) != IE_OK ||
        (rc = stage<int64_t>(st->nodes_out, nullptr, static_cast<size_t>(keep) * (L + 1), s)) != IE_OK)
      return rc;
    if (L > 0) CK(cudaMemcpyAsync(st->nodes_in.p, nodes, static_cast<size_t>(rows) * L * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    sc = st->scores.as<float>();
    va = st->values.as<float>();
    tk = st->tokens.as<int64_t>();
    nd = st->nodes_in.as<int64_t>();
    pa = st->parent.as<int32_t>();
    to = st->out_idx.as<int64_t>();
    ns = st->out_val.as<float>();
    nn = st->nodes_out.as<int64_t>();
  }
  CK(ie::launch_lm_beam_select(sc, va, tk, rows, top_k, beam_sz, nd, L, pa, to, ns, nn, s));
  lm->launches++;
  if (!dev) {
    CK(cudaMemcpyAsync(parent, pa, keep * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(token, to, keep * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(new_scores, ns, keep * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(new_nodes, nn, static_cast<size_t>(keep) * (L + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  }
  return gen_finish(lm, s, dev);
}

int ie_gen_state_export(ie_gen_state* st, int32_t layer, int32_t rows, uint16_t* h_out, float* c_out) {
  if (st == nullptr || h_out == nullptr || c_out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  ie_lm* lm = st->lm;
  const ie_encoder* h = lm->enc;
  if (layer < 0 || layer >= h->cfg.n_layers) return fail(IE_ERR_INVALID, "layer %d out of range", layer);
  if (rows < 1 || rows > st->cap) return fail(IE_ERR_INVALID, "rows=%d outside [1,%d]", rows, st->cap);
  std::lock_guard<std::mutex> lk(lm->mu);
  CK(cudaSetDevice(lm->device));
  CK(lm->order.wait());
  const Layer& L = h->layers[layer];
  const int planes = h->segs > 1 ? 2 : 1;
  const __nv_bfloat16* hs = st->h[st->cur].as<__nv_bfloat16>() + layer * st->h_layer;
  for (int p = 0; p < planes; ++p)
    CK(cudaMemcpy2D(h_out + static_cast<size_t>(p) * L.out, planes * L.out * sizeof(uint16_t), hs + p * L.out_pad,
                    st->y_ld * sizeof(__nv_bfloat16), L.out * sizeof(uint16_t), rows, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy2D(c_out, L.out * sizeof(float), st->c[st->cur].as<float>() + layer * st->c_layer,
                  (st->c_layer / st->cap) * sizeof(float), L.out * sizeof(float), rows, cudaMemcpyDeviceToHost));
  return IE_OK;
}

int ie_debug_gen_topk(const float* logits, int32_t rows, int32_t V, int32_t k, int32_t exclude, float* values,
                     int64_t* idx, int32_t device) {
  if (logits == nullptr || values == nullptr || idx == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (rows < 1 || V < 1 || k < 1 || k > std::min(ie::kLmTopkMax, V) || exclude < -1 || exclude >= V)
    return fail(IE_ERR_INVALID, "rows=%d V=%d k=%d exclude=%d: bad argument", rows, V, k, exclude);
  CK(cudaSetDevice(device));
  DevBuf z, v, ix;
  const size_t n = static_cast<size_t>(rows) * k;
  CK(z.reserve(static_cast<size_t>(rows) * V * sizeof(float)));
  CK(v.reserve(n * sizeof(float)));
  CK(ix.reserve(n * sizeof(int64_t)));
  CK(cudaMemcpy(z.p, logits, static_cast<size_t>(rows) * V * sizeof(float), cudaMemcpyHostToDevice));
  CK(ie::launch_lm_topk(z.as<float>(), V, rows, V, k, exclude, v.as<float>(), ix.as<int64_t>(), nullptr));
  CK(cudaMemcpy(values, v.p, n * sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(idx, ix.p, n * sizeof(int64_t), cudaMemcpyDeviceToHost));
  return IE_OK;
}

int ie_debug_gen_sample(const float* logits, int32_t rows, int32_t V, const float* u, int32_t exclude,
                       double temperature, double min_p, int64_t* idx, int32_t* draw_flags, int32_t device) {
  if (logits == nullptr || u == nullptr || idx == nullptr || draw_flags == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (rows < 1 || V < 1 || exclude < -1 || exclude >= V || !(temperature > 0.0) || !std::isfinite(temperature) ||
      !(min_p == 0.0 || (min_p > 0.0 && min_p <= 1.0)))
    return fail(IE_ERR_INVALID, "rows=%d V=%d exclude=%d temperature=%g min_p=%g: bad argument", rows, V, exclude,
                temperature, min_p);
  CK(cudaSetDevice(device));
  DevBuf z, ud, ix, fl, err;
  CK(z.reserve(static_cast<size_t>(rows) * V * sizeof(float)));
  CK(ud.reserve(rows * sizeof(float)));
  CK(ix.reserve(rows * sizeof(int64_t)));
  CK(fl.reserve(rows * sizeof(int)));
  CK(err.reserve(sizeof(int), true));
  CK(cudaMemcpy(z.p, logits, static_cast<size_t>(rows) * V * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ud.p, u, rows * sizeof(float), cudaMemcpyHostToDevice));
  CK(ie::launch_lm_sample(z.as<float>(), V, rows, V, ud.as<float>(), exclude, static_cast<float>(min_p),
                          static_cast<float>(1.0 / temperature), ix.as<int64_t>(), fl.as<int>(), err.as<int>(), nullptr));
  CK(cudaMemcpy(idx, ix.p, rows * sizeof(int64_t), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(draw_flags, fl.p, rows * sizeof(int), cudaMemcpyDeviceToHost));
  return IE_OK;
}

}  // extern "C"
