// C-ABI layer of the encoder (declared in include/issue_emb_b200.h): handle management, weight re-layout, workspace
// and the launch sequence of the encoder hot path, plus the library's version, last error and the encoder's debug hooks.
#include <cstring>

#include <cuda_fp16.h>

#include "encoder_host.h"

using namespace ie;

namespace {

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

// one run of the launch sequence under the handle's lock; a host-pointer call is synchronous and also reports the
// device-side errors
int encoder_call(ie_encoder* h, const int64_t* ids, const int32_t* lengths, int B, int T, float* out, float* raw_out,
                 int raw_layer, int flags, void* stream) {
  std::lock_guard<std::mutex> lk(h->mu);
  const int rc = run_encoder(h, ids, lengths, B, T, out, raw_out, raw_layer, flags, call_stream(flags, stream, h->own_stream));
  if (rc != IE_OK || (flags & IE_FLAG_DEVICE_PTRS)) return rc;
  return collect_errors(h);
}

}  // namespace

namespace ie {

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

int run_encoder(ie_encoder* h, const int64_t* ids, const int32_t* lengths, int B, int T, float* out, float* raw_out,
                int raw_layer, int flags, cudaStream_t s, long long* keep_raw, const ChunkHook* hook,
                const EncState* st) {
  const ie_config& c = h->cfg;
  if (!h->emb_loaded) return fail(IE_ERR_STATE, "embedding not loaded");
  for (const Layer& L : h->layers)
    if (!L.loaded) return fail(IE_ERR_STATE, "LSTM layer weights not loaded");
  if (B < 1 || B > h->max_batch) return fail(IE_ERR_INVALID, "B=%d outside [1,%d]", B, h->max_batch);
  if (T < 1) return fail(IE_ERR_INVALID, "T=%d must be >= 1", T);
  const bool want_raw = raw_out != nullptr || keep_raw != nullptr;
  if (ids == nullptr || (out == nullptr && !want_raw && hook == nullptr)) return fail(IE_ERR_INVALID, "null pointer");
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
  CK(h->order.begin(s));

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
  // a carried state: h_{-1} of rows < B into the carry, c_{-1} into the layer's cell state (padding rows zero)
  if (st != nullptr)
    for (int l = 0; l < c.n_layers; ++l) {
      const Layer& L = h->layers[l];
      float* cl = h->c.as<float>() + static_cast<size_t>(l) * h->max_batch * mop;
      CK(cudaMemcpyAsync(h->hcarry.as<__nv_bfloat16>() + static_cast<size_t>(l) * carry_layer, st->h + l * st->h_layer,
                         static_cast<size_t>(B) * h->y_ld * sizeof(__nv_bfloat16), cudaMemcpyDeviceToDevice, s));
      CK(cudaMemsetAsync(cl, 0, static_cast<size_t>(b_pad) * L.out_pad * sizeof(float), s));
      CK(cudaMemcpy2DAsync(cl, L.out_pad * sizeof(float), st->c + l * st->c_layer, st->c_ld * sizeof(float),
                           L.out_pad * sizeof(float), B, cudaMemcpyDeviceToDevice, s));
    }

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
      q.c = cstate; q.carry_c = st != nullptr; q.y = ybuf;
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
      if (last && hook != nullptr &&
          (rc = hook->fn(hook->ctx, ybuf + static_cast<size_t>(b_pad) * h->y_ld, h->y_ld, static_cast<int>(t0), Tc, b_pad,
                         s)) != IE_OK)
        return rc;
      if (t0 + Tc < T)  // carry h of the chunk's last step into the next chunk
        CK(cudaMemcpyAsync(carry, ybuf + static_cast<size_t>(Tc) * b_pad * h->y_ld, slot_bytes, cudaMemcpyDeviceToDevice, s));
      else if (st != nullptr) {  // the state after the last step, before layer l + 2 reuses this ring
        CK(cudaMemcpyAsync(st->h + l * st->h_layer, ybuf + static_cast<size_t>(Tc) * b_pad * h->y_ld,
                           static_cast<size_t>(B) * h->y_ld * sizeof(__nv_bfloat16), cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpy2DAsync(st->c + l * st->c_layer, st->c_ld * sizeof(float), cstate, L.out_pad * sizeof(float),
                             L.out_pad * sizeof(float), B, cudaMemcpyDeviceToDevice, s));
      }
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
  CK(h->order.end(s));
  if (keep_raw != nullptr) {
    *keep_raw = t_need;
    return IE_OK;
  }
  return maybe_release_workspace(h, t_need, s);
}

int collect_errors(ie_encoder* h) {
  if (!h->order.has_done) return IE_OK;
  CK(cudaSetDevice(h->cfg.device));
  int w[kErrWords] = {0, 0, 0, 0};
  const int rc = read_errors(h->order, h->err, w, kErrWords);
  if (rc != IE_OK) return rc;
  if (w[1] != 0) {
    h->use_persistent = h->fault ? h->use_persistent : 0;  // do not walk into the same wall again
    return fail(IE_ERR_CUDA, "a device-side wait exceeded its limit and the kernel was drained (the persistent grid lost "
                             "co-residency, or a protocol error); results of this call are invalid");
  }
  if (w[0] != 0) return fail(IE_ERR_TOKEN, "token id outside [0,%d) in ids", h->cfg.vocab_sz);
  if (w[2] != 0) return fail(IE_ERR_INVALID, "a length outside [1,T] was clamped");
  return IE_OK;
}

}  // namespace ie

extern "C" {

int ie_version(void) { return 200; }

const char* ie_last_error(void) { return g_last_error.c_str(); }

int ie_encoder_create(const ie_config* cfg, ie_encoder** out) {
  if (cfg == nullptr || out == nullptr) return fail(IE_ERR_INVALID, "null argument");
  if (cfg->n_layers < 1 || cfg->n_layers > 16 || cfg->emb_sz < 1 || cfg->n_hid < 1 || cfg->vocab_sz < 1 ||
      cfg->pad_idx < 0 || cfg->pad_idx >= cfg->vocab_sz)
    return fail(IE_ERR_INVALID, "bad encoder config");
  int sms = 0;
  int rc = open_device(cfg->device, &sms);
  if (rc != IE_OK) return rc;
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
  rc = plan_layers(h);
  if (rc != IE_OK) { delete h; return rc; }
  const cudaError_t e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete h; return cuda_fail(e, "cudaStreamCreate"); }
  *out = h;
  return IE_OK;
}

void ie_encoder_destroy(ie_encoder* h) {
  if (h == nullptr) return;
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  delete h;
}

int ie_encoder_load_embedding(ie_encoder* h, const float* emb) {
  if (h == nullptr || emb == nullptr) return fail(IE_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  CK(cudaSetDevice(h->cfg.device));
  // the per-token table GEMM reads the embedding as its A operand: rows padded to whole M tiles (zeros)
  const int v_rows = static_cast<int>(round_up(h->cfg.vocab_sz, 256));
  int rc = upload_sliced(emb, h->cfg.vocab_sz, h->cfg.emb_sz, padded_identity(h->cfg.vocab_sz, v_rows), h->e_pad, h->segs, h->emb, h->own_stream);
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
  return encoder_call(h, ids, lengths, B, T, out, nullptr, -1, flags, stream);
}

int ie_encoder_raw_features(ie_encoder* h, const int64_t* ids, int32_t B, int32_t T, float* raw, int32_t flags,
                            void* stream) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (raw == nullptr) return fail(IE_ERR_INVALID, "raw is null");
  return encoder_call(h, ids, nullptr, B, T, nullptr, raw, h->cfg.n_layers - 1, flags, stream);
}

int ie_debug_layer_states(ie_encoder* h, int32_t layer, const int64_t* ids, int32_t B, int32_t T, float* out,
                          int32_t flags, void* stream) {
  if (h == nullptr) return fail(IE_ERR_INVALID, "null handle");
  if (out == nullptr) return fail(IE_ERR_INVALID, "out is null");
  return encoder_call(h, ids, nullptr, B, T, nullptr, out, layer, flags, stream);
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
  if (!h->order.has_done) return fail(IE_ERR_STATE, "no encode call recorded");
  CK(cudaSetDevice(h->cfg.device));
  CK(h->order.wait());
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
  if (in == nullptr || out == nullptr || n < 0 || fn < 0 || fn > 12)
    return fail(IE_ERR_INVALID, "fn=%d n=%lld: bad argument", fn, static_cast<long long>(n));
  CK(cudaSetDevice(device));
  CK(ie::launch_debug_gates(fn, in, out, n, static_cast<cudaStream_t>(stream)));
  return IE_OK;
}

}  // extern "C"
