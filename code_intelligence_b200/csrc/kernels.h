// Internal launch interfaces between the C-ABI layer (api_*.cu) and the sm_90a kernels.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace ie {

// ---- TMA descriptor helper (tmap.cu) ---------------------------------------------------------
// 2-D bf16 tensor, inner (contiguous) dimension `inner` elements, `rows` rows, row pitch `ld` elements,
// box {box_inner, box_rows}, 128-byte swizzle (box_inner must be 64).
cudaError_t make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t ld,
                              uint32_t box_inner, uint32_t box_rows);

// ---- fragment order of a 256-column tile (Gx, the per-token table, the encoder's bias) -----------------------------
// In a wgmma m64n256 accumulator, lane q = lane % 4 of a warp holds, for each of its rows, the 64 columns 16m + 2q + {0,1}
// and 16m + 8 + 2q + {0,1} (m = 0..15) -- for the recurrent kernel the gates (i, f, g, o) of 16 hidden units.  In fragment
// order these 64 values are one contiguous run per q, in that order (m-major, then i, f, g, o), cut into 16-byte chunks
// that are interleaved over q: chunk k of lane q sits at chunk position 4k + q of the row's tile.  A warp's 16-byte
// access of chunk k then covers 64 contiguous bytes of each of its rows.  Returns the element position inside the tile
// of natural column c (0..255) for elements of `elem_bytes` (2: fp16, 4: f32) bytes.
__host__ __device__ inline int frag_index(int c, int elem_bytes) {
  const int q = (c & 7) >> 1;                                     // owning lane of the quad
  const int ix = 4 * (c >> 4) + 2 * ((c >> 3) & 1) + (c & 1);    // position in that lane's run of 64 values
  const int per_chunk = 16 / elem_bytes;
  return (ix / per_chunk * 4 + q) * per_chunk + ix % per_chunk;
}

// ---- GEMM (gemm.cu) ----------------------------------------------------------------------------
struct GemmArgs {
  const __nv_bfloat16* a;  // [m_pad, lda]   (split-bf16: [hi(k_pad) | lo(k_pad)] per row)
  const __nv_bfloat16* b;  // [n_pad, ldb]
  void* d;                 // [m_store.., ldd] f32 or bf16
  const float* bias;       // [n_pad] or nullptr
  int m_pad, n_pad, k_pad;
  long long lda, ldb, ldd;
  int m_store, n_store;
  int bn;        // padding granularity of N (multiple of 16, <= 256, divides n_pad); the kernel's N tile is 256
  int act;       // 0 none, 1 relu, 2 sigmoid
  int out_bf16;  // output type: 0 f32, 1 bf16, 2 fp16 (act must be 0)
  int num_sms;
  int segs;      // 1: bf16 operands; 3: split-bf16 (K loop over [A_hi|A_lo|A_hi] x [B_hi|B_hi|B_lo], ~fp32 products)
  unsigned* abort_flag;  // optional global word raised when a wait exceeds spin_limit (ptx.cuh abort protocol)
  long long spin_limit;  // SM cycles; 0 = default
  long long* diag;       // optional [4]: {clock64, globaltimer ns} at the start and end of CTA 0
  int frag;              // 1: store D (and read bias) in fragment order (frag_index; act 0, f32 or fp16, n_store % 256 == 0)
};
cudaError_t launch_gemm_bf16(const GemmArgs& g, cudaStream_t stream);

// ---- recurrent layer (lstm_layer.cu): all timesteps of a layer (or of a time chunk) in one cooperative launch, up to
//      kMaxBatches batches of 256 rows; (timestep, batch, row half, tile) items dealt round-robin over all CTAs.  With
//      single_step the same kernel runs one timestep per launch (the fallback when the grid cannot be co-resident).
constexpr int kMaxBatches = 12;
struct LstmLayerArgs {
  CUtensorMap tm_h;        // hidden-state ring of the time chunk [(Tc+1)*b_pad rows, ring cols], box {64, 128}
  CUtensorMap tm_w;        // W_hh [4*out_pad rows, cols], box {64, 256}; rows ordered as api_encoder.cu slice_perm
  CUtensorMap tm_h64;      // same tensor as tm_h with box {64, 64}: the half tile one CTA multicasts (mc != 0)
  CUtensorMap tm_x;        // pre_nkb > 0: the PREVIOUS layer's ring (slot t+1 = this layer's x_t), box {64, 128}
  int pre_nkb;             // > 0: fuse the input projection into the K loop -- pre_nkb = kin_pad / 64 k-blocks of
                           // x_t W_ih^T precede the recurrent ones; tm_w then covers [W_ih | W_hh] (inner kin_pad + kh_pad),
                           // gx is unused and `bias` (b_ih + b_hh, permuted like the weight rows, fragment order) is added instead
  const float* bias;
  int mc;                  // 1: clusters of two CTAs share every h tile by TMA multicast (needs an even number of tiles)
  int mc_ctas;             // CTAs that can be co-resident in clusters of two (lstm_layer_max_ctas() of a check_only query)
  const void* gx;          // f16 or f32 [rows, 4*out_pad] (bias folded in, fragment order): row t*b_pad + brow of the chunk, or token id
  const int* tok;          // optional time-major token ids of the whole call (per-token input-projection table)
  float* c;                // [b_pad, out_pad] cell state
  int carry_c;             // 1: c holds c_{-1} of a carried state (global step 0 reads it); 0: c_{-1} = 0
  __nv_bfloat16* y;        // ring (slot 0 = h before the chunk (zeros at t0 = 0 without a carried state); slot t+1 = h_t)
  float* raw;              // optional [raw_rows, T_total, raw_ld] f32 copy of h (get_raw_features)
  int raw_rows;            // rows of raw: the call's valid rows B (padding rows of the batch are not stored)
  float* pool_sum;         // optional [b_pad, out_pad] (last layer only; formats: lstm_common.cuh)
  float* pool_max;
  float* pool_last;
  const int* lengths;      // [b_pad]
  unsigned* step_done;   // [T*ng] zero-initialised (step, batch) counters of this launch
  unsigned* abort_flag;
  long long spin_limit;
  int T, t0, T_total;    // timesteps in this launch, global index of the first, timesteps of the whole call
  int single_step;       // 1: only chunk-local timestep t_step, one item per CTA, no counters, not cooperative
  int t_step;
  int ng;                // batches of 256 rows
  int u, n_cta, out_pad, kh_pad;
  long long ldy, raw_ld;
  int gate_mode, gx_bf16, segs;
  int num_sms, check_only, cooperative;
  int fault;             // debug: drop one counter update (exercises the abort protocol)
  long long* trace;      // optional [grid][trace_items][12] timeline (debug)
  int trace_items;
  long long* diag;       // optional [4]: {clock64, globaltimer ns} at the start and end of CTA 0 (SM clock of the launch)
};
cudaError_t launch_lstm_layer(const LstmLayerArgs& a, cudaStream_t stream);
int lstm_layer_ctas(const LstmLayerArgs& a);  // CTAs the launch will use
int lstm_layer_max_ctas();                    // result of the last check_only query on this thread

// ---- small memory-bound kernels (misc.cu) --------------------------------------------------------
// ids [B, T] int64 (batch-first, right padded) -> x0 [(T*b_pad), ldx] bf16, time-major rows t*b_pad + b
// (t0, Tc): only timesteps [t0, t0+Tc) are gathered, into rows (t - t0)*b_pad + b
cudaError_t launch_embed_gather(const int64_t* ids, int B, int T, int b_pad, const __nv_bfloat16* emb, int vocab,
                                int e_pad, __nv_bfloat16* x0, long long ldx, int pad_idx, int* err_flag, int t0, int Tc,
                                cudaStream_t stream);
// lengths_in [B] (device) -> lengths_out [b_pad]: clamped to [1, T] (err_flag[2] raised if it had to clamp), rows >= B: 1
cudaError_t launch_prep_lengths(const int* lengths_in, int B, int T, int b_pad, int* lengths_out, int* err_flag,
                                cudaStream_t stream);
// out[b] = [sum/len | max | last], b < B, first `e` units
// ids [B, T] int64 -> tok [T*b_pad] int32 time-major (rows >= B: pad_idx), range-checked like launch_embed_gather
cudaError_t launch_tokens_time_major(const int64_t* ids, int B, int T, int b_pad, int vocab, int pad_idx, int* tok,
                                     int* err_flag, cudaStream_t stream);
cudaError_t launch_pool_finalize(const float* pool_sum, const float* pool_max, const float* pool_last,
                                 const int* lengths, int B, int e, int out_pad, float* out, cudaStream_t stream);
// f32 [rows, cols] (row pitch ld_src) -> bf16 [rows_pad, ld_dst] with optional row permutation (src row of dst row r
// = perm[r], or -1 for a zero row); columns >= cols zero filled.
// lo_off > 0: split-bf16 layout -- hi = bf16(x) in columns [0, lo_off), lo = bf16(x - hi) in [lo_off, 2*lo_off)
cudaError_t launch_convert_rows(const float* src, long long ld_src, int cols, const int* perm, int rows_dst,
                                __nv_bfloat16* dst, long long ld_dst, int lo_off, cudaStream_t stream);
cudaError_t launch_fill_f32(float* p, size_t n, float v, cudaStream_t stream);
// ie_debug_gates: fn 0..5 unary gate functions, 6 / 7 / 8 the cell update with fast / exp / IEEE gates, 9 / 10 the
// language-model decoder's ex2_approx and logf, 11 / 12 text generation's expf and powf (in = planes [x | y])
cudaError_t launch_debug_gates(int fn, const float* in, float* out, long long n, cudaStream_t stream);

// ---- precision-recall threshold search (pr_curve.cu): scores [n, n_labels] f32, truth [n, n_labels] u8 (device) ----------
constexpr int kPrMaxSamples = 16384;
cudaError_t launch_pr_thresholds(const float* scores, const uint8_t* truth, int n, int n_labels, double p_thr,
                                 double r_thr, float* out_thr, double* out_prec, double* out_rec, cudaStream_t stream);

// ---- exact k-nearest-neighbour search (knn.cu) ----------------------------------------------------------------------
constexpr int kKnnCap = 512;          // candidate-buffer entries per (query, corpus slice): k' + a whole 256-row tile fit
constexpr int kKnnMergeMax = 16384;   // S * k' bound: the merge sorts one query's candidates in shared memory
constexpr int kKnnExtra = 32;         // k' = k + kKnnExtra rows are shortlisted by stage 1 and re-ranked exactly
// Every stored row and query has |x| = 0 or kKnnNormMin <= |x| <= kKnnNormMax (f64 norm of the f32 row): then every
// stage-1 product, partial sum and score is finite and the split products stay clear of f32's subnormal range
// (DESIGN.md section 2).  Host input outside it is refused; device input raises bit 2 of the error flag.
constexpr double kKnnNormMin = 0x1p-48, kKnnNormMax = 0x1p48;
// f64 column mean of x [n, D] rounded to f32 -> center [k_pad] (zeros past D); partial: knn_center_workspace(D) bytes
size_t knn_center_workspace(int D);
cudaError_t launch_knn_center(const float* x, long long n, int D, int k_pad, double* partial, float* center,
                              cudaStream_t stream);
// rows [rows_pad] of src [rows, D] f32 -> dst [rows_pad, 2*k_pad] split-bf16 of x - center (zero rows past `rows`),
// terms [rows_pad]: mode 0 (|x~|^2/2, 0), 1 (c.x~, 1/|x| or 0), 2 (q~.c + c2, 0); a non-finite value sets *err
cudaError_t launch_knn_prep(const float* src, long long rows, long long rows_pad, int D, int k_pad, const float* center,
                            double c2, int mode, __nv_bfloat16* dst, float2* terms, int* err, cudaStream_t stream);
// corpus slices S and n-blocks per slice for nq queries against n rows
void knn_plan(int nq, long long n, int kp, int num_sms, int* S, int* nbs);
struct KnnStage1Args {
  const __nv_bfloat16* qs;  // [m_pad, 2*k_pad] split-bf16 centred queries
  const __nv_bfloat16* xs;  // [n, 2*k_pad] split-bf16 centred corpus
  const float2* col;        // [round_up(n, 256)] corpus terms
  const float2* rowt;       // [m_pad] query terms
  uint2* cand;              // [nq][S][kKnnCap]
  int* cnt;                 // [nq][S]
  long long n;
  int nq, m_pad, k_pad, S, nbs, kp, cosine, num_sms;
};
cudaError_t launch_knn_stage1(const KnnStage1Args& a, cudaStream_t stream);
// per query row: best kp candidates; dbg_score != nullptr: write them ([rows, kp]) and stop; else exact distances
// from Q [rows, D] and X [n, D] f32 and the best k -> out_dist / out_idx [rows, k]
cudaError_t launch_knn_merge_rerank(const uint2* cand, const int* cnt, int rows, int S, int kp, const float* Q,
                                    const float* X, int D, int cosine, int k, float* out_dist, int64_t* out_idx,
                                    float* dbg_score, int64_t* dbg_idx, cudaStream_t stream);

// ---- label-MLP training step (mlp_train.cu) -------------------------------------------------------------------------
// src [rows, cols] f32 (row r read from src row rowidx[r] when rowidx is set; zeroed where mask [rows, ld_mask] is 0),
// optionally copied to out_f32, stored as split-bf16 operands with exact zeros outside [rows, cols]:
//   rm [rm_rows, ld_rm]: row r = [hi(rm_kpad) | lo(rm_kpad)]   (the A operand of the next product)
//   tr [tr_rows, ld_tr]: row c = [hi(tr_kpad) | lo(tr_kpad)] of column c  (transposed: K = rows, for a weight gradient)
struct SplitStoreArgs {
  const float* src;
  long long ld_src;
  const int* rowidx;
  int rows, cols;
  const float* mask;
  long long ld_mask;
  float* out_f32;
  long long ld_f32;
  __nv_bfloat16* rm;
  long long ld_rm;
  int rm_rows, rm_kpad;
  __nv_bfloat16* tr;
  long long ld_tr;
  int tr_rows, tr_kpad;
};
cudaError_t launch_split_store(const SplitStoreArgs& a, cudaStream_t stream);
// rows b of z [b, ldz] (the last layer's pre-activation): p = sigmoid_acc(z); with Y (u8 [n, L], row rowidx[r]):
// delta = p - y and row_loss[r] = sum over labels of log(clip(p)) or log(1 - clip(p)) (f64). p and delta share ldz.
cudaError_t launch_mlp_output(const float* z, long long ldz, const uint8_t* Y, const int* rowidx, int b, int L, float* p,
                              float* delta, double* row_loss, cudaStream_t stream);
// gW [fan_in, fan_out] = f32((dw + f32(alpha) W) / b) with dw = a^T delta [fan_in, ld_dw]; gb [fan_out] = f32(sum_r delta / b)
cudaError_t launch_mlp_grad(const float* dw, long long ld_dw, const float* W, int fan_in, int fan_out, const float* delta,
                            long long ld_delta, int b, float alpha, float* gW, float* gb, cudaStream_t stream);
// *out = -sum(row_loss[0..b)) / b + 0.5 alpha sum(sq_part) / b
cudaError_t launch_mlp_loss(const double* row_loss, int b, const double* sq_part, int n_part, double alpha, double* out,
                            cudaStream_t stream);
constexpr int kAdamBlocks = 264;  // fixed grid: the sum |W|^2 partials are summed in the same order every step
struct AdamArgs {
  float *p, *m, *v;
  const float* g;        // nullptr: no update, only the sum |W|^2 partials of p
  long long n, n_coef;   // parameters, of which the first n_coef are coefficients
  float beta1, one_m_beta1, beta2, one_m_beta2, eps;  // f32 roundings of the Python doubles
  const double* lr;      // lr[step] = learning_rate_init sqrt(1 - beta2^t) / (1 - beta1^t)
  int step;
  double* sq_part;       // [kAdamBlocks]
};
cudaError_t launch_adam(const AdamArgs& a, cudaStream_t stream);

// ---- grouped label-MLP training (mlp_group.cu) ----------------------------------------------------------------------
// Each launch runs the stage above for `count` models of one architecture: model j is slot slots[j] (device array),
// its operands at base + slot * stride (strides in elements; 0 = shared by every model, as X and Y are).
struct GroupSplitArgs {
  SplitStoreArgs a;                                   // slot 0's operands
  long long s_src, s_idx, s_mask, s_f32, s_rm, s_tr;
  const int* slots;
  int count;
};
cudaError_t launch_group_split_store(const GroupSplitArgs& g, cudaStream_t stream);
struct GroupOutputArgs {   // launch_mlp_output per model; p and delta share z's pitch ldz and stride s_z
  const float* z;
  float *p, *delta;
  long long ldz, s_z, s_p;
  const uint8_t* Y;
  const int* rowidx;
  long long s_idx;
  double* row_loss;
  long long s_rl;
  int b, L;
  const int* slots;
  int count;
};
cudaError_t launch_group_output(const GroupOutputArgs& g, cudaStream_t stream);
struct GroupGradArgs {     // launch_mlp_grad per model; alpha[slot] (f64, rounded to f32 as the single step does)
  const float* dw;
  long long ld_dw, s_dw;
  const float* W;          // and gW, gb: inside the parameter vectors, stride s_param
  float *gW, *gb;
  long long s_param;
  const float* delta;
  long long ld_delta, s_delta;
  int fan_in, fan_out, b;
  const double* alpha;
  int coef_blocks;         // set by the launcher
  const int* slots;
  int count;
};
cudaError_t launch_group_grad(GroupGradArgs g, cudaStream_t stream);
struct GroupLossArgs {     // launch_mlp_loss per model: out[slot * s_out] from row_loss and sq_part[slot][kAdamBlocks]
  const double* row_loss;
  long long s_rl;
  const double* sq_part;
  const double* alpha;
  double* out;
  long long s_out;
  int b;
  const int* slots;
  int count;
};
cudaError_t launch_group_loss(const GroupLossArgs& g, cudaStream_t stream);
struct GroupAdamArgs {     // launch_adam per model: consts[slot][5] = f32 beta1, 1 - beta1, beta2, 1 - beta2, eps
  float *p, *m, *v;
  const float* g;          // nullptr: only the sum |W|^2 partials
  long long n, n_coef, s_param;
  const float* consts;
  const double* lr;        // lr[slot * s_lr + step]
  long long s_lr;
  int step;
  double* sq_part;         // [slot][kAdamBlocks]
  const int* slots;
  int count;
};
cudaError_t launch_group_adam(const GroupAdamArgs& a, cudaStream_t stream);
// D = act(A B^T + bias) for each model (segs = 3): A rows slot * a_rows + [0, m_pad), B rows slot * b_rows + [0, n_pad)
// of stacked split-bf16 operands (a_rows % 128 == 0, b_rows % 256 == 0, zero rows past each model's extent), D and bias
// at slot * s_d / s_bias; stored like launch_gemm_bf16's f32 output (rows < m_store, columns < n_store)
struct GroupGemmArgs {
  const __nv_bfloat16* a;
  const __nv_bfloat16* b;
  long long lda, ldb, a_rows, b_rows;
  float* d;
  long long ldd, s_d;
  const float* bias;
  long long s_bias;
  int m_pad, n_pad, k_pad, m_store, n_store, relu;
  int n_models;            // slots in the stacked operands
  const int* slots;
  int count;
  int num_sms;
};
cudaError_t launch_group_gemm(const GroupGemmArgs& g, cudaStream_t stream);

// ---- text classifier (clas.cu) ---------------------------------------------------------------------------------------
// raw [B, T, ld] f32 states, ids [B, T] int64, window [starts[b], ends[b]) -> out [B, 3*e_sz] = [last | max | avg] with
// fastai's pad mask (ids == pad_idx).  A window outside [0, T], empty or all pad raises err[2] and gives a NaN row.
// enc_err (optional): the encoder's error words, OR-ed into err[0] (token id) and err[1] (wait timeout).
cudaError_t launch_clas_pool(const float* raw, long long ld, int B, int T, const int64_t* ids, const int* starts,
                             const int* ends, int e_sz, int pad_idx, float* out, const int* enc_err, int* err,
                             cudaStream_t stream);
// y [rows, N] = act(fma(x, alpha, beta) . W^T + bias), x [rows, K], W [N, K] (torch Linear layout), relu 0/1
cudaError_t launch_clas_linear(const float* x, int rows, int K, const float* alpha, const float* beta, const float* W,
                               const float* bias, int N, int relu, float* y, cudaStream_t stream);
// p [rows, N] = sigmoid(z) (softmax 0) or the max-subtracted softmax of each row (softmax 1)
cudaError_t launch_clas_activate(const float* z, int rows, int N, int softmax, float* p, cudaStream_t stream);

// ---- language-model decoder (lm.cu) ---------------------------------------------------------------------------------
constexpr int kLmSliceTiles = 32;   // 256-column tiles per vocabulary slice: slice boundaries depend on V alone
struct LmPart {                      // one (row, slice) partial: max logit, sum of exp(x - max), argmax
  float m, s;
  int arg, unused;
};
struct LmDecodeArgs {
  const __nv_bfloat16* h;   // [rows, ld_h] states (split-bf16: [hi(k_pad) | lo(k_pad)]); row r = step r / rps, batch row r % rps
  long long ld_h;
  const __nv_bfloat16* w;   // [round_up(V, 256), (segs > 1 ? 2 : 1) * k_pad] decoder weight, same layout
  const float* bias;        // [round_up(V, 256)] f32, zeros past V
  const int64_t* targets;   // [B, T]: target of (batch row b, step t0 + t) at b * T + t0 + t; -100 ignored
  long long rows;           // steps * rps
  int rps, B, T, t0, V, k_pad, segs, num_sms;
  LmPart* part;             // [rows, lm_slices(V)] workspace
  float* tlogit;            // [rows] workspace
  float* nll;               // [B, T] (same indexing as targets)
  float* lse;               // optional
  int* pred;                // optional
  int* err;                 // err[0] |= 1: a target outside [0, V) other than -100 (its nll is NaN)
  unsigned* abort_flag;     // the mainloop's abort word (ptx.cuh)
  long long spin_limit;
};
int lm_slices(int V);
// logits = h W^T + bias, per valid row: lse, nll against its target and argmax; the logits are never stored
cudaError_t launch_lm_decode(const LmDecodeArgs& a, cudaStream_t stream);

// ---- text generation (lm_gen.cu): decisions on f32 logits [rows, ld] (columns < V) ------------------------------------
constexpr int kLmTopkMax = 64;       // k of lm_topk
constexpr int kLmBeamMax = 16384;    // rows * top_k candidates one CTA sorts in shared memory (fastai's defaults: 10000)
// per row: values [rows, k] = the k largest f32(z - lse), descending, ties to the lower column; idx [rows, k] their
// columns; column `exclude` (>= 0) counts in lse and is -inf among the values (fastai's no_unk)
cudaError_t launch_lm_topk(const float* logits, long long ld, int rows, int V, int k, int exclude, float* values,
                           int64_t* idx, cudaStream_t stream);
// per row: one draw from fastai's predict weights (softmax, `exclude` zeroed, min_p > 0 masking, powf(p, inv_t)) at
// the uniform u[row], never a column of weight 0: out[row] the column, flags[row] 1 when no column reached min_p (nothing masked), 2 when every
// weight is 0 (err[0] |= 2, column 0)
cudaError_t launch_lm_sample(const float* logits, long long ld, int rows, int V, const float* u, int exclude,
                             float min_p, float inv_t, int64_t* out, int* flags, int* err, cudaStream_t stream);
// the min(beam_sz, rows * top_k) lowest scores f32(parent_scores[r] - values[r, c]) in stable-sort order: their parent
// rows, tokens (tokens[r, c]), scores, and nodes_out [n, L + 1] = nodes_in [rows, L] of the parent plus the token
cudaError_t launch_lm_beam_select(const float* parent_scores, const float* values, const int64_t* tokens, int rows,
                                  int top_k, int beam_sz, const int64_t* nodes_in, int L, int* parent, int64_t* token,
                                  float* score, int64_t* nodes_out, cudaStream_t stream);
// dst row i = src row parent[i] in each of `layers` layers (rows of row_bytes, layers layer_bytes apart, both multiples
// of 16); a parent outside [0, src_rows) raises err[0] |= 4 and copies row 0
cudaError_t launch_gather_rows(const void* src, void* dst, const int* parent, int n, int src_rows, long long row_bytes,
                               long long layer_bytes, int layers, int* err, cudaStream_t stream);

}  // namespace ie
