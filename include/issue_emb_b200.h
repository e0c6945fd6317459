/* issue_emb_b200 -- C ABI of the H100-native Issue_Embeddings encoder hot path and the Label_Microservice
 * MLP head (libissue_emb_b200.so).  Plain pointers and sizes only; no torch / C++ types.
 *
 * The reference (kubeflow/Code-Intelligence) has no FFI layer for this path: its "operator API" is the Python
 * class InferenceWrapper and sklearn's MLPClassifier behind MLPWrapper.  Each entry point below states the
 * reference interface it replaces (paths relative to the reference tree); INTEGRATION.md shows the ctypes
 * binding a maintainer would add on the reference side.
 *
 * Conventions
 *   - every function returns IE_OK (0) or a negative IE_ERR_* code and never aborts; ie_last_error() returns a
 *     thread-local human-readable message for the last failing call on this thread.  Device-side waits are bounded:
 *     one that exceeds its limit drains the kernel and surfaces as IE_ERR_CUDA (no trap, the CUDA context and the
 *     handle stay usable).
 *   - a handle owns its device weights and workspace; calls on one handle are serialised internally (host mutex; a
 *     call on another stream first waits for the previous call's completion event); handles may be used from any host
 *     thread.  The persistent recurrent kernel is launched cooperatively: it runs only when its whole grid can be
 *     resident, so two handles (or other work) sharing a device serialise instead of deadlocking.
 *   - `flags & IE_FLAG_DEVICE_PTRS`: ids / lengths / out (or X / probs) are device pointers on the handle's
 *     device and the call is asynchronous on `stream`; otherwise they are host pointers (pinned or pageable)
 *     and the call returns after the result has been copied back.  In device-pointer mode data-dependent errors
 *     (token id out of range, length outside [1,T] -- clamped --, wait timeout) cannot be returned by the call itself:
 *     ie_encoder_check_errors() reports them.
 *   - `stream` is a cudaStream_t passed as void*.  With host pointers NULL selects the handle's own stream; with
 *     IE_FLAG_DEVICE_PTRS it is used verbatim (NULL = the legacy default stream, which is torch's default).
 */
#ifndef ISSUE_EMB_B200_H_
#define ISSUE_EMB_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IE_OK 0
#define IE_ERR_INVALID (-1) /* bad argument / shape (Python shim raises ValueError)                        */
#define IE_ERR_CUDA (-2)    /* CUDA runtime / launch failure (RuntimeError)                                  */
#define IE_ERR_OOM (-3)     /* device memory exhausted (RuntimeError, so the reference's batch-halving loop   */
                            /* py/code_intelligence/inference.py:214-223 keeps working)                       */
#define IE_ERR_STATE (-4)   /* weights not loaded, wrong call order                                           */
#define IE_ERR_TOKEN (-5)   /* a token id outside [0, vocab_sz) was seen (ValueError)                         */

#define IE_FLAG_DEVICE_PTRS 1

/* ie_config.flags */
#define IE_CFG_ACCURATE_GATES 1 /* ex2+rcp sigmoid/tanh (abs err ~1e-7) instead of the default single-MUFU          */
                                /* tanh.approx.f32 gates (rel err 2^-11; no measurable effect on the parity metrics) */
#define IE_CFG_FP32 2           /* "fp32-accurate" mode (BASELINE configs[1] as written; the reference computes in    */
                                /* fp32, Issue_Embeddings/flask_app/inference.py:57): every product runs as split-bf16  */
                                /* (x = hi + lo, three tensor-core passes hi*hi + lo*hi + hi*lo, f32 accumulate: ~2^-17 */
                                /* relative per product), input projections kept in f32, IEEE gates.  ~3x the MMAs.    */
#define IE_CFG_F32_GX 4         /* keep the hoisted input projections in f32 instead of fp16 (bf16 mode only)         */

#define IE_MAX_BATCH 3072 /* upper bound of rows per ie_encoder_encode call; the handle's own limit is
                             ie_encoder_max_batch() = 256 x (batches per launch, default 5): that many independent
                             256-row batches ride one launch of the persistent recurrent kernel (each as two 128-row
                             halves of wgmma items); they share the kernel, not their results */

typedef struct ie_encoder ie_encoder;
typedef struct ie_mlp ie_mlp;

/* AWD-LSTM encoder shape.  Replaces what fastai's load_learner() unpickles at
 * Issue_Embeddings/flask_app/inference.py:33-36 (model structure: notebooks/04_Inference.ipynb:157-187):
 * Embedding(vocab_sz, emb_sz, padding_idx=pad_idx) -> n_layers x LSTM, in_0 = emb_sz, hidden = n_hid,
 * out_{L-1} = emb_sz.  Output width is 3*emb_sz. */
typedef struct ie_config {
  int32_t n_layers; /* deployed reference model: 4 (north-star wording: 3) */
  int32_t emb_sz;   /* 800  */
  int32_t n_hid;    /* 2400 */
  int32_t vocab_sz; /* 60000 */
  int32_t pad_idx;  /* 1 (inference.py:36 learn.data.pad_idx) */
  int32_t device;   /* CUDA device ordinal */
  int32_t flags;    /* IE_CFG_* bits, 0 = defaults */
} ie_config;

int ie_version(void);
const char* ie_last_error(void);

/* InferenceWrapper.__init__ (Issue_Embeddings/flask_app/inference.py:29-39): create the encoder ... */
int ie_encoder_create(const ie_config* cfg, ie_encoder** out);
void ie_encoder_destroy(ie_encoder* h);

/* ... and load its weights (host pointers, f32, C-contiguous):
 *   emb   [vocab_sz, emb_sz]                     state_dict key  encoder.weight
 *   w_ih  [4*out_l, in_l]   rows i|f|g|o         rnns.{l}.module.weight_ih_l0
 *   w_hh  [4*out_l, out_l]                       rnns.{l}.weight_hh_l0_raw
 *   b_ih, b_hh [4*out_l]                         rnns.{l}.module.bias_{ih,hh}_l0
 * (torch.nn.LSTM layout; key names per fastai 1.0.53 AWD_LSTM, SURVEY.md section 8c). */
int ie_encoder_load_embedding(ie_encoder* h, const float* emb);
int ie_encoder_load_layer(ie_encoder* h, int32_t layer, const float* w_ih, const float* w_hh, const float* b_ih,
                          const float* b_hh);

/* The hot path.  Replaces InferenceWrapper._forward_pass + batch_seq_pool
 * (Issue_Embeddings/flask_app/inference.py:55-57 and :215-246; bulk loop py/code_intelligence/inference.py:207-212)
 * and, with B == 1 and lengths[0] == T, get_pooled_features (inference.py:71-90):
 *   ids     [B, T] int64, batch-first, right-padded with pad_idx (what pad_sequence builds, inference.py:201)
 *   lengths [B] int32, 1 <= lengths[b] <= T
 *   out     [B, 3*emb_sz] f32 = [mean | max | last] over the first lengths[b] steps of the last layer's hidden
 *           states, zero initial state (encoder.reset(), inference.py:56)
 * 1 <= B <= ie_encoder_max_batch(h).  T is bounded only by the workspace cap B_pad*T <= 2^27 tokens (IE_ERR_OOM
 * beyond; B_pad = B rounded up to 256): the time dimension is processed in chunks of 2^20 / B_pad steps (half that
 * with f32 input projections), so the device workspace stays under about 31 GB at the deployed shape whatever T is,
 * and a single 16k-token issue is fine.  A handle keeps its workspace between calls; after four consecutive calls
 * that need under 1/8 of the bytes held by the buffers that grow with T (over 64 MB of them), it is released. */
int ie_encoder_encode(ie_encoder* h, const int64_t* ids, const int32_t* lengths, int32_t B, int32_t T, float* out,
                      int32_t flags, void* stream);

/* InferenceWrapper.get_raw_features (inference.py:59-68): the last layer's hidden states, raw [B, T, emb_sz] f32.
 * T is bounded as for ie_encoder_encode.  Device memory: the encode workspace (bounded by the time chunk) plus
 * B * T * round_up(emb_sz, 64) * 4 bytes of f32 states for the B valid rows -- 41 MB for one 12 300-token issue at
 * emb_sz = 800, 67 MB at 20 000 tokens. */
int ie_encoder_raw_features(ie_encoder* h, const int64_t* ids, int32_t B, int32_t T, float* raw, int32_t flags,
                            void* stream);

/* Number of kernels this handle has launched so far (bench.py reports it as gpu_launches). */
int64_t ie_encoder_launch_count(const ie_encoder* h);

/* Rows one ie_encoder_encode call accepts on this handle: 1280 = five 256-row batches per launch by default
 * (environment variable IE_BATCHES=n at create time, 1 <= n <= 12, changes that to 256 n). */
int32_t ie_encoder_max_batch(const ie_encoder* h);

/* Test hook: bytes of device workspace the handle holds now (the buffers its calls grow and reuse; weights, the
 * embedding and the per-token table not included). */
int64_t ie_debug_workspace_bytes(const ie_encoder* h);

/* Device-side error state of the last call on this handle (waits for it to finish): IE_OK, IE_ERR_TOKEN (a token id
 * outside [0, vocab_sz) was remapped to 0), IE_ERR_INVALID (a length outside [1,T] was clamped; device-pointer mode
 * only -- host lengths are validated before anything is launched) or IE_ERR_CUDA (a device-side wait timed out and
 * the kernel was drained).  Host-pointer calls report these themselves; device-pointer calls are asynchronous, so
 * their caller asks here.  Clears the state. */
int ie_encoder_check_errors(ie_encoder* h);

/* Device time of each phase of the last encode call on this handle, from CUDA events recorded on the launching
 * stream: ms[0] = embedding gather, then per layer l: ms[1+2l] = input-projection GEMM, ms[2+2l] = the T recurrent
 * step launches, last = pool finalize.  Waits for the call to finish.  Returns the number of phases (or < 0). */
int ie_encoder_last_phase_ms(ie_encoder* h, float* ms, int32_t cap);

/* SM clock (MHz) the recurrent kernel of each layer ran at in the last call, from clock64 / globaltimer stamps taken
 * by the kernel itself (nvidia-smi cannot resolve single phases).  mhz[l] = recurrent kernel of layer l,
 * mhz[n_layers + l] = its input-projection GEMM (0 when the layer had none).  Returns 2 * n_layers (or < 0). */
int ie_encoder_last_phase_mhz(ie_encoder* h, float* mhz, int32_t cap);

/* Debug hook: per-item timeline of one layer of the persistent recurrent kernel (tools/trace_layer.py). */
int64_t ie_debug_seq_trace(ie_encoder* h, int32_t layer, long long* out, int64_t cap);

/* MLP head.  Replaces sklearn MLPClassifier.predict_proba as called by MLPWrapper.predict_probabilities
 * (py/label_microservice/mlp.py:56-63): relu hidden layers, logistic output (multilabel).
 *   dims [n_layers + 1] = {D_in, hidden..., n_labels};  coef_l [dims[l], dims[l+1]] f32 (sklearn coefs_[l],
 *   fan_in major), intercept_l [dims[l+1]].  X [n, D_in] f32 -> probs [n, n_labels] f32. */
int ie_mlp_create(int32_t n_layers, const int32_t* dims, int32_t device, ie_mlp** out);
int ie_mlp_load_layer(ie_mlp* m, int32_t layer, const float* coef, const float* intercept);
int ie_mlp_predict_proba(ie_mlp* m, const float* X, int32_t n, float* probs, int32_t flags, void* stream);
void ie_mlp_destroy(ie_mlp* m);

/* Threshold search.  Replaces the per-label loop of MLPWrapper.find_probability_thresholds
 * (py/label_microservice/mlp.py:81-98: sklearn precision_recall_curve + "highest precision among the points with
 * precision >= precision_threshold and recall >= recall_threshold; first such point in increasing-threshold order").
 *   scores [n, n_labels] f32 (predict_proba of the hold-out set), truth [n, n_labels] uint8 (0/1), n <= 16384
 *   thresholds [n_labels] f32 (NaN: no qualifying point, the label is excluded -- None in the reference),
 *   precisions / recalls [n_labels] f64 at the chosen point (0 when excluded).
 * Scores must be finite; -0.0 and +0.0 are the same score (a zero threshold is returned as +0.0).
 * Host pointers (synchronous; a NaN or infinite score returns IE_ERR_INVALID before anything is launched) or, with
 * IE_FLAG_DEVICE_PTRS, device pointers on `device` (asynchronous on `stream`; a label with any NaN or infinite score
 * gets threshold, precision and recall all NaN, which an excluded label -- NaN / 0 / 0 -- never has). */
int ie_pr_thresholds(const float* scores, const uint8_t* truth, int32_t n, int32_t n_labels, double precision_threshold,
                     double recall_threshold, float* thresholds, double* precisions, double* recalls, int32_t device,
                     int32_t flags, void* stream);

/* Debug / test hook: D[M,N] = act(A[M,K] * B[N,K]^T (+bias)) through the same wgmma GEMM the encoder uses.
 * a [M,K], b [N,K], bias [N] or NULL: host f32 (rounded to bf16 on the device); d [M,N] host f32;
 * act 0 none, 1 relu, 2 sigmoid. */
int ie_debug_gemm(const float* a, const float* b, const float* bias, int32_t M, int32_t N, int32_t K, int32_t act,
                  float* d, int32_t device);

/* Same GEMM with every epilogue and operand form the library uses: out_type 0 = f32, 1 = bf16 (the MLP head's hidden
 * layers), 2 = fp16 (the encoder's input projections and per-token table; act must be 0), each widened exactly to f32
 * into d; segs 1 = bf16 operands, 3 = split-bf16 (x = hi + lo, hi = bf16(x), lo = bf16(x - hi), products
 * hi*hi + lo*hi + hi*lo: the fp32-accurate mode's operands). */
int ie_debug_gemm_ex(const float* a, const float* b, const float* bias, int32_t M, int32_t N, int32_t K, int32_t act,
                     int32_t out_type, int32_t segs, float* d, int32_t device);

/* Same GEMM (act 0, bias required, N a multiple of 256) with the store the encoder's input projections use: each
 * 256-column tile of a row in fragment order (DESIGN.md section 3), the bias read in the same order.  The result is
 * put back into natural column order on the host, so d [M,N] is comparable element for element with
 * ie_debug_gemm_ex; out_type 0 = f32, 2 = fp16. */
int ie_debug_gemm_frag(const float* a, const float* b, const float* bias, int32_t M, int32_t N, int32_t K,
                       int32_t out_type, int32_t segs, float* d, int32_t device);

/* Host-only test hook: the layout maps of the recurrent kernel for a layer of `out_units` hidden units.  Returns the
 * number of weight rows 4*out_pad (out_pad = out_units rounded up to 64); if cap >= that, perm receives the torch
 * gate-major row (g*out_units + unit) behind each of them, -1 for padding.  frag2 / frag4 [256] (each optional)
 * receive the fragment-order position of each column of a 256-column tile for 2- and 4-byte elements. */
int64_t ie_debug_epilogue_layout(int32_t out_units, int32_t* perm, int64_t cap, int32_t* frag2, int32_t* frag4);

/* Debug / test hook, device pointers on `device`, asynchronous on `stream`: the gate functions and the cell update as the
 * recurrent kernel and the GEMM epilogue compute them (the same inline device functions).
 *   fn 0..5: out[i] = f(in[i]), i < n, f = sigmoid_fast, tanh_fast, sigmoid_acc, tanh_acc, sigmoid_ieee, tanh_ieee
 *   fn 6, 7, 8: the cell update with fast, exp (IE_CFG_ACCURATE_GATES) or IEEE (IE_CFG_FP32) gates:
 *   in = planes [zi | zf | zg | zo | c_prev] of n values each, out = planes [c_new | h]. */
int ie_debug_gates(int32_t fn, const float* in, float* out, int64_t n, int32_t device, void* stream);

/* Debug / test hook: the hidden states of layer `layer` of an encode of ids [B, T] (zero initial state), as that
 * layer's recurrent kernel computed them: out [B, T, out_l] f32, out_l = n_hid, or emb_sz for the last layer.  The
 * hidden-state ring the next step and the next layer read holds their bf16 round-to-nearest-even (hi + lo in the
 * fp32-accurate mode); for the last layer they are ie_encoder_raw_features.  Every development knob applies as in
 * ie_encoder_encode; the arithmetic is the same, only an extra f32 store of h is made. */
int ie_debug_layer_states(ie_encoder* h, int32_t layer, const int64_t* ids, int32_t B, int32_t T, float* out,
                          int32_t flags, void* stream);

/* Exact k-nearest-neighbour index over embeddings (similar-issue search).  Replaces the brute-force neighbour searches
 * of the reference's notebooks: the FewShot notebook's oneshotlabeler (CosineSimilarity over every stored issue) and
 * KNeighborsClassifier(metric='cosine'), and notebook 08's KNeighborsClassifier(weights='distance') label model.
 *   Rows are numbered 0.. in insertion order.  ie_knn_search returns for each query the k stored rows nearest under
 *   the metric, ascending by distance, ties to the lower index: dist [nq, k] f32 (sklearn kneighbors convention:
 *   cosine 1 - cos, computed as |q/|q| - x/|x||^2 / 2; euclidean |q - x|; a zero vector has cosine distance 1 to
 *   everything), idx [nq, k] int64.  The answer is float64 brute force on the f32 inputs whenever at most 32 rows
 *   outside the exact top k score within 2 eps of the k-th (DESIGN.md section 2): a split-bf16 tensor-core pass over
 *   the centred data shortlists k + 32 rows per query, which are re-ranked exactly.
 *   With exact stage-1 scores (small-integer data, DESIGN.md section 2) ties resolve by index however many there are.
 *   Limits: 1 <= dim <= 8192, 1 <= k <= 64, k <= rows stored, nq >= 1, rows < 2^31 (IE_ERR_OOM when the device is
 *   full).  Range: every added row and query has norm 0 or between 2^-48 and 2^48, which keeps every stage-1 score
 *   finite.  Searching an empty index returns IE_ERR_STATE.
 *   Host pointers: a NaN or infinite value, or a row outside the range, returns IE_ERR_INVALID before anything is
 *   launched.  IE_FLAG_DEVICE_PTRS: asynchronous on `stream`; such input is reported by ie_knn_check_errors() (the
 *   answers of the calls that saw it are undefined).  The first ie_knn_add fixes the centre (the f32-rounded f64 mean
 *   of its rows) and waits for it. */
#define IE_KNN_COSINE 0
#define IE_KNN_EUCLIDEAN 1
typedef struct ie_knn ie_knn;
int ie_knn_create(int32_t dim, int32_t metric, int32_t device, ie_knn** out);
void ie_knn_destroy(ie_knn* h);
/* X [n, dim] f32, appended as rows size..size+n-1 */
int ie_knn_add(ie_knn* h, const float* X, int64_t n, int32_t flags, void* stream);
int ie_knn_search(ie_knn* h, const float* Q, int32_t nq, int32_t k, float* dist, int64_t* idx, int32_t flags,
                  void* stream);
/* IE_OK, or IE_ERR_INVALID if a non-finite value or a row outside the range was seen in device-pointer input since the
 * last check (waits for the last call on this handle; clears the state). */
int ie_knn_check_errors(ie_knn* h);
/* Debug / test hook, host pointers: stage 1 alone -- the k + 32 best rows of each query by the tensor-core score
 * (larger is nearer; euclidean q~.x~ - |x~|^2/2, cosine q.x / |x|, with x~ = x - c), score descending, ties to the lower
 * index: score [nq, k + 32] f32 and idx [nq, k + 32] int64 (-1 / -inf past the rows stored). */
int ie_debug_knn_shortlist(ie_knn* h, const float* Q, int32_t nq, int32_t k, float* score, int64_t* idx);

/* Label-MLP trainer.  Replaces the step loop of sklearn MLPClassifier.fit(solver='adam', activation='relu') on a
 * logistic (multilabel / binary) output, as MLPWrapper.fit calls it (py/label_microservice/mlp.py:45-54); the host
 * driver (code_intelligence_b200/mlp_train.py) keeps every decision sklearn makes -- initialisation, validation split,
 * row orders, stopping -- and calls these once per epoch.  Host pointers only; every call returns when its work is done.
 *   dims [n_layers + 1] = {D_in, hidden..., n_labels}, n_layers >= 2 (at least one hidden layer).
 *   Parameters are f32 in sklearn's layout: coef_l [dims[l], dims[l+1]] (coefs_[l]), intercept_l [dims[l+1]].
 *   Every product is a split-bf16 GEMM (segs 3); the loss is float64; the Adam step is sklearn's AdamOptimizer on float32
 *   arrays bit for bit (DESIGN.md section 9). */
typedef struct ie_mlp_train ie_mlp_train;
int ie_mlp_train_create(int32_t n_layers, const int32_t* dims, int32_t device, ie_mlp_train** out);
void ie_mlp_train_destroy(ie_mlp_train* h);
/* Set (and reset the Adam moments of every layer to zero, t = 0) / read one layer's current (best = 0) or snapshot
 * (best = 1) parameters.  Non-finite values are refused. */
int ie_mlp_train_set_layer(ie_mlp_train* h, int32_t layer, const float* coef, const float* intercept);
int ie_mlp_train_get_layer(ie_mlp_train* h, int32_t layer, int32_t best, float* coef, float* intercept);
/* Resident data: which 0 = training set X [n, D_in] f32 and Y [n, n_labels] u8 (0/1), which 1 = validation X (Y unused).
 * A non-finite X value returns IE_ERR_INVALID. */
int ie_mlp_train_set_data(ie_mlp_train* h, int32_t which, const float* X, const uint8_t* Y, int64_t n);
/* One epoch: steps k = 0 .. ceil(n / batch_size) - 1 on training rows order[k*batch_size ...] (the last batch short),
 * learning rate lr[k] = learning_rate_init sqrt(1 - beta_2^t) / (1 - beta_1^t) of the step's t; losses[k] receives each
 * step's batch loss (log loss + 0.5 alpha sum|W|^2 / b).  The steps are enqueued without host synchronisation. */
int ie_mlp_train_epoch(ie_mlp_train* h, const int32_t* order, int64_t n, int32_t batch_size, const double* lr,
                       double alpha, double beta_1, double beta_2, double epsilon, double* losses);
/* Probabilities [n_val, n_labels] f32 of the validation set under the current parameters. */
int ie_mlp_train_validation_proba(ie_mlp_train* h, float* probs);
/* restore 0: snapshot the current parameters as the best; 1: make the snapshot current again. */
int ie_mlp_train_snapshot(ie_mlp_train* h, int32_t restore);
/* Kernels launched by this handle so far / device time (CUDA events) of the last ie_mlp_train_epoch. */
int64_t ie_mlp_train_launch_count(const ie_mlp_train* h);
int ie_mlp_train_last_epoch_ms(ie_mlp_train* h, float* ms);
/* Debug / test hook.  mode 0: one forward + backward pass on training rows rows[b] with consts[0] = alpha, parameters
 * unchanged: out = a_1 .. a_{n_layers-1} (hidden activations), p (probabilities), delta_0 .. delta_{n_layers-1} (each
 * [b, width] f32, delta_l = dLoss/dz of layer l's output, sklearn's deltas[l]), then the gradients in sklearn's packing
 * (every coef, then every intercept); *loss = the batch loss.  mode 1: one optimizer step with the given gradients
 * (sklearn's packing) and consts = {lr_t, beta_1, beta_2, epsilon}: out = parameters, m, v, each in sklearn's packing. */
int ie_debug_mlp_train_step(ie_mlp_train* h, int32_t mode, const int32_t* rows, int32_t b, const double* consts,
                            const float* grads, float* out, int64_t cap, double* loss);

/* Group trainer: n_models fits of one architecture (dims) and one batch size, trained in lockstep -- the fits of a grid
 * search (code_intelligence_b200/mlp_train.py DeviceGridSearchCV).  X [n, D_in] and Y [n, n_labels] are resident once;
 * each model trains on rows of them that the caller names (its fold, its early-stopping split) and keeps its own
 * parameters, Adam moments, snapshot, constants (alpha, beta_1, beta_2, epsilon) and workspace.  Every stage of a step
 * is one launch for all models whose batch has the same size, so a step costs the launches of one ie_mlp_train step
 * whatever the group size.  Each model's results are bit-identical to an ie_mlp_train handle given the same rows,
 * parameters and learning rates: its tiles and reductions run the same instructions over the same partitions.  A model
 * whose values turn non-finite affects no other.  Host pointers only; every call returns when its work is done. */
typedef struct ie_mlp_group ie_mlp_group;
/* Device bytes one model of such a group takes, and the models that fit in `fraction` of the device's free memory
 * (at most 65535, the largest n_models ie_mlp_group_create accepts). */
int ie_mlp_group_capacity(int32_t n_layers, const int32_t* dims, int32_t batch_size, int32_t device, double fraction,
                          int64_t* bytes_per_model, int32_t* max_models);
int ie_mlp_group_create(int32_t n_layers, const int32_t* dims, int32_t n_models, int32_t batch_size, int32_t device,
                        ie_mlp_group** out);
void ie_mlp_group_destroy(ie_mlp_group* h);
/* Shared data X [n, D_in] f32 and Y [n, n_labels] u8; non-finite X is refused. */
int ie_mlp_group_set_data(ie_mlp_group* h, const float* X, const uint8_t* Y, int64_t n);
/* Model `model`'s layer parameters (resets its Adam moments, t = 0) / current (best 0) or snapshot (best 1) parameters. */
int ie_mlp_group_set_layer(ie_mlp_group* h, int32_t model, int32_t layer, const float* coef, const float* intercept);
int ie_mlp_group_get_layer(ie_mlp_group* h, int32_t model, int32_t layer, int32_t best, float* coef, float* intercept);
/* Model `model`'s alpha and Adam constants. */
int ie_mlp_group_set_hyper(ie_mlp_group* h, int32_t model, double alpha, double beta_1, double beta_2, double epsilon);
/* Model `model`'s validation rows (indices into X), n_val >= 1. */
int ie_mlp_group_set_validation(ie_mlp_group* h, int32_t model, const int32_t* rows, int64_t n_val);
/* One epoch of the models models[0 .. n_active): model i trains on rows[i] (n_rows[i] indices into X, in step order, the
 * rows of all models concatenated), steps k = 0 .. ceil(n_rows[i] / batch_size) - 1 with learning rates lr (each model's
 * steps concatenated) and batch losses out in losses (same layout).  No host synchronisation between steps. */
int ie_mlp_group_epoch(ie_mlp_group* h, int32_t n_active, const int32_t* models, const int64_t* n_rows,
                       const int32_t* rows, const double* lr, double* losses);
/* Probabilities [n_val, n_labels] f32 of model `model`'s validation rows. */
int ie_mlp_group_validation_proba(ie_mlp_group* h, int32_t model, float* probs);
/* restore 0: snapshot model `model`'s parameters as its best; 1: make its snapshot current again. */
int ie_mlp_group_snapshot(ie_mlp_group* h, int32_t model, int32_t restore);
/* Kernels launched by this handle so far / device time (CUDA events) of the last ie_mlp_group_epoch. */
int64_t ie_mlp_group_launch_count(const ie_mlp_group* h);
int ie_mlp_group_last_epoch_ms(ie_mlp_group* h, float* ms);

/* Text classifier.  Replaces the model fastai's text_classifier_learner builds on the AWD-LSTM encoder
 * (Issue_Embeddings/notebooks/06_FineTune.ipynb: get_text_classifier = SequentialRNN(MultiBatchEncoder,
 * PoolingLinearClassifier), fastai 1.0.53) in eval mode, as learn.predict / learn.model(x) run it:
 *   encoder  the borrowed ie_encoder's states o [B, T, emb_sz] of ids [B, T] (zero initial state, every step run,
 *            pads included -- fastai's batched forward over pad_collate(pad_first=True) batches)
 *   pool     per row b over the window [starts[b], ends[b]) of W steps, mask = (ids == pad_idx):
 *            [last | max | avg] = o[b, ends[b]-1], max of the unmasked steps, (sum of the unmasked steps / W) *
 *            f32(W / (W - n_masked)) -- fastai's masked_concat_pool on the window of kept bptt chunks (ie_clas_window)
 *   head     per stage k: BatchNorm1d(dims[k]) with the running statistics, Linear(dims[k], dims[k+1]), ReLU except on
 *            the last stage; then sigmoid (IE_CLAS_SIGMOID, multi-label) or softmax (IE_CLAS_SOFTMAX) of the logits.
 * dims [n_stages + 1] = {3*emb_sz, hidden..., n_class}.  The handle borrows the encoder (weights, workspace, stream,
 * serialisation): destroy it before the encoder.  Windows are validated on the host before any launch with host
 * pointers (IE_ERR_INVALID for one outside [0, T], empty, or entirely pad); with IE_FLAG_DEVICE_PTRS such a row is NaN and
 * ie_clas_check_errors() reports it, with the encoder's own token-id and wait errors.  B <= ie_encoder_max_batch(enc);
 * rows are encoded in groups whose f32 states fit 4 GB (one row at a time beyond). */
#define IE_CLAS_SIGMOID 0
#define IE_CLAS_SOFTMAX 1
typedef struct ie_clas ie_clas;
/* First kept step of a sequence of sl steps: MultiBatchEncoder(bptt, max_len) keeps chunk i (i = 0, bptt, ...) when
 * i > sl - max_len.  IE_ERR_INVALID when no chunk is kept (only possible with max_len <= bptt).  Host only. */
int ie_clas_window(int32_t sl, int32_t bptt, int32_t max_len, int32_t* start);
int ie_clas_create(ie_encoder* enc, int32_t n_stages, const int32_t* dims, int32_t activation, ie_clas** out);
void ie_clas_destroy(ie_clas* c);
/* Stage `stage`: BatchNorm1d weight, bias (each may be NULL: 1 / 0), running_mean, running_var [dims[stage]], eps;
 * Linear weight [dims[stage+1], dims[stage]] (torch layout) and bias [dims[stage+1]].  Host f32; non-finite refused. */
int ie_clas_load_stage(ie_clas* c, int32_t stage, const float* bn_weight, const float* bn_bias, const float* bn_mean,
                       const float* bn_var, double eps, const float* lin_weight, const float* lin_bias);
/* ids [B, T] int64, starts / ends [B] int32 -> out [B, n_class] f32 (activated); logits [B, n_class] (optional, NULL). */
int ie_clas_forward(ie_clas* c, const int64_t* ids, const int32_t* starts, const int32_t* ends, int32_t B, int32_t T,
                    float* out, float* logits, int32_t flags, void* stream);
/* The pool alone: pooled [B, 3*emb_sz] f32 = [last | max | avg], the head's input. */
int ie_clas_pool(ie_clas* c, const int64_t* ids, const int32_t* starts, const int32_t* ends, int32_t B, int32_t T,
                 float* pooled, int32_t flags, void* stream);
/* Device-side errors of the last call on this handle (waits for it; clears them): IE_ERR_CUDA, IE_ERR_TOKEN or
 * IE_ERR_INVALID (a bad or all-pad window in device-pointer mode). */
int ie_clas_check_errors(ie_clas* c);
/* Kernels this handle has launched (pool, head stages, activation); the encoder's count its own. */
int64_t ie_clas_launch_count(const ie_clas* c);

#ifdef __cplusplus
}
#endif
#endif /* ISSUE_EMB_B200_H_ */
