// The encoder handle and the part of its host code (api_encoder.cu) that the handles built on it -- the text classifier
// (api_clas.cu) and the language model (api_lm.cu) -- call: they borrow its weights, workspace, stream, error words and
// launch sequence.
#pragma once
#include "host.h"

namespace ie {

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

constexpr int kErrWords = 4;  // err[0] token id out of range, err[1] device-side wait timed out (abort protocol),
                              // err[2] a length had to be clamped (device-pointer mode)

// Work enqueued on the encoder's stream after the last layer's recurrent launch of each time chunk (the language
// model's decoder): ring = slot 1 of the last layer's ring, Tc * b_pad time-major rows of pitch ld holding h_{t0..t0+Tc-1}
// (split-bf16 [hi | lo] planes at offset out_pad in the fp32-accurate mode).  Returns IE_OK or an error code.
struct ChunkHook {
  int (*fn)(void* ctx, const __nv_bfloat16* ring, long long ld, int t0, int Tc, int b_pad, cudaStream_t s);
  void* ctx;
};

// A recurrent state carried across calls (the language model's text generation): per layer l, h as the ring holds it
// (rows of y_ld bf16: [hi | lo] planes at offset out_pad_l in the fp32-accurate mode) at h + l * h_layer, and c (rows
// c_ld f32 apart, the first out_pad_l used) at c + l * c_layer.  A call's rows 0..B-1 start from it and it receives
// their state after the call's last step.
struct EncState {
  __nv_bfloat16* h;
  float* c;
  long long h_layer, c_layer, c_ld;   // elements (c_ld >= every layer's out_pad)
};

// host f32 [rows_src, cols] -> device bf16 [perm.size(), ld] (split mode: [hi(k_pad) | lo(k_pad)], ld = 2*k_pad)
int upload_sliced(const float* host, int rows_src, int cols, const std::vector<int>& perm, int k_pad, int segs, DevBuf& dst,
                  cudaStream_t s);

long long max_out_pad(const ie_encoder* h);

// a handle that once served a very long sequence does not keep its T-sized buffers for ever (api_encoder.cu)
int maybe_release_workspace(ie_encoder* h, long long t_need, cudaStream_t s);

// the launch sequence shared by encode (pooled), raw_features and the layer-state hook: raw_out (optional) receives the
// f32 hidden states of layer raw_layer as its recurrent kernel computed them, [B, T, out_l].  keep_raw (optional, the
// classifier): the states stay in the workspace (h->raw, [B, T, out_pad]) for kernels the caller enqueues next on `s`;
// the workspace is then not released here, *keep_raw receives the bytes for the caller's maybe_release_workspace.
// hook (optional, the language model): called once per time chunk, see ChunkHook.  st (optional): the state the call
// starts from and leaves, see EncState; without it every row starts from zero.
int run_encoder(ie_encoder* h, const int64_t* ids, const int32_t* lengths, int B, int T, float* out, float* raw_out,
                int raw_layer, int flags, cudaStream_t s, long long* keep_raw = nullptr,
                const ChunkHook* hook = nullptr, const EncState* st = nullptr);

// read and clear the device error words of the last call (waits for it)
int collect_errors(ie_encoder* h);

}  // namespace ie

struct ie_encoder {
  ie_config cfg{};
  int num_sms = 132;
  int e_pad = 0;  // emb_sz rounded up to 64
  // one weight layout: slices of u = 32 hidden units (slice_perm); two slices = one N = 256 accumulator tile of the
  // recurrent kernel (lstm_layer.cu)
  std::vector<ie::Layer> layers;
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
  ie::DevBuf proj, tok;
  ie::DevBuf emb;  // bf16 [vocab_pad, e_pad] (split mode: [hi | lo])
  bool emb_loaded = false;
  long long spin_limit = 0;  // SM cycles a device-side wait may take (0: default ~2 s); IE_SPIN_LIMIT_MS
  int fault = 0;             // IE_DEBUG_FAULT: exercise the abort protocol
  long long chunk_t = 0;     // IE_CHUNK_T: force the time-chunk length (testing)
  // workspace
  ie::DevBuf ids, len_in, lengths, x0, y[2], hcarry, gx, c, pool_sum, pool_max, pool_last, out, raw, err, step_done, diag;
  ie::DevBuf trace;       // debug timeline of one layer of the persistent kernel (ie_debug_seq_trace)
  int trace_layer = -1;
  int trace_T = 0, trace_ctas = 0;
  long long y_ld = 0;
  int small_calls = 0;      // consecutive calls far below the buffers that grow with T (workspace released after a few)
  cudaStream_t own_stream = nullptr;
  ie::StreamOrder order;    // the calls of the handle and of the handles that borrow its workspace
  int64_t launches = 0;
  // phase boundary events of the last encode call and what ended at each (0 start, 1 gather, 2+2l gemm_l, 3+2l steps_l,
  // 2+2L finalize)
  std::vector<cudaEvent_t> ev;
  std::vector<int> ev_tag;
  int ev_used = 0;
  int last_T = 0, last_b_pad = 0;
  std::mutex mu;
};
