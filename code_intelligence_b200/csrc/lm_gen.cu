// Text generation from the language model (ie_gen_state_* / ie_gen_beam_select in include/issue_emb_b200.h): fastai
// LanguageLearner's predict and beam_search, one decision per launch, on f32 logits of the last step that the
// persistent GEMM (gemm.cu, act 0, the decoder's bias) wrote for each row.
//
//   lm_topk_kernel         per row: lse, then the top k of logit - lse (ties to the lower index), one column excluded
//   lm_sample_kernel       per row: fastai's softmax -> no_unk -> min_p -> temperature weights and one inverse-CDF draw
//   lm_beam_select_kernel  one CTA: the beam_sz lowest of rows * top_k scores, as a stable sort orders them
//   gather_rows_kernel     a state's rows by parent index (fastai's select_hidden)
//
// Every sum runs in one fixed order that does not depend on the grid, so a row's result is a function of its own logits:
//   * column sums (the softmax denominator): thread t of the CTA adds columns t, t + kGenThreads, ... in ascending
//     order (the compiler fuses expf's final scale multiply into the add: s = fma(2^i, ex2(r), s)), then the
//     kGenThreads partials are reduced by xor shuffles (offsets 16, 8, 4, 2, 1) within each warp and the 32 warp sums
//     are added in warp order by warp 0 the same way;
//   * the sampling CDF: columns in chunks of kGenThreads in ascending order; a chunk's inclusive prefix is a warp scan
//     (Hillis-Steele, offsets 1 .. 16) plus the exclusive sum of the earlier warps' totals, itself a warp scan; the
//     running total S_j = carry + prefix is rounded once per element.  The carry then moves by the chunk's total as
//     the scan of the warp totals has it at lane 31 (red[31]).  That is not the chunk's last S_j: thread 1023's prefix
//     adds its warp's own prefix to red[30], another association, and on random weights the two differ in the last
//     bit in about half of all chunks.  The row's total is the final carry, so it is not S_{V-1} either, even for
//     V <= kGenThreads.
//   oracle/lm_gen_ref.py restates both kernels bit for bit in this order.
#include <climits>
#include <cstdint>

#include "kernels.h"
#include "lstm_common.cuh"

namespace ie {

namespace {

constexpr int kGenThreads = 1024;
constexpr int kGenWarps = kGenThreads / 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(~0u, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(~0u, v, o));
  return v;
}

// the fixed-order CTA sum of one partial per thread (see the file comment); every thread receives it
__device__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    float x = warp_sum(red[lane]);
    if (lane == 0) red[kGenWarps] = x;
  }
  __syncthreads();
  return red[kGenWarps];
}

__device__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    float x = warp_max(red[lane]);
    if (lane == 0) red[kGenWarps] = x;
  }
  __syncthreads();
  return red[kGenWarps];
}

// inclusive prefix of one value per thread over the CTA in thread order (see the file comment); *total gets the sum
__device__ float block_scan(float v, float* red, float* total) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float y = __shfl_up_sync(~0u, v, o);
    if (lane >= o) v += y;
  }
  __syncthreads();
  if (lane == 31) red[w] = v;
  __syncthreads();
  if (w == 0) {
    float x = red[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float y = __shfl_up_sync(~0u, x, o);
      if (lane >= o) x += y;
    }
    red[lane] = x;   // inclusive over warps
  }
  __syncthreads();
  if (w > 0) v += red[w - 1];
  *total = red[kGenWarps - 1];
  return v;
}

// the row's softmax denominator after the max: sum of exp(x - m) over all V columns (expf, fixed order)
__device__ float row_max(const float* z, int V, float* red) {
  float m = -INFINITY;
  for (int c = threadIdx.x; c < V; c += kGenThreads) m = fmaxf(m, z[c]);
  return block_max(m, red);
}

__device__ float row_expsum(const float* z, int V, float m, float* red) {
  float s = 0.0f;
  for (int c = threadIdx.x; c < V; c += kGenThreads) s += expf(z[c] - m);
  return block_sum(s, red);
}

// per row r (one CTA): lse = m + logf(sum exp(z - m)) over all columns; the excluded column (exclude >= 0) counts in
// lse, as fastai takes log_softmax before it sets that column to -inf; then the top k of f32(z - lse) with ties to the
// lower index, sorted by value descending.  Keys are enc_max of the values: the k-th largest key by a four-pass
// 8-bit radix select, then the keys above it and the lowest-indexed ties at it.
__global__ void __launch_bounds__(kGenThreads) lm_topk_kernel(const float* __restrict__ logits, long long ld, int V,
                                                               int k, int exclude, float* __restrict__ values,
                                                               int64_t* __restrict__ idx) {
  __shared__ float red[kGenWarps + 1];
  __shared__ unsigned hist[256];
  __shared__ unsigned sel[2];       // the threshold key's prefix so far, ties at it still to take
  __shared__ unsigned n_gt;         // slots filled by keys above the threshold
  __shared__ unsigned wcount[kGenWarps];
  __shared__ uint32_t ckey[kLmTopkMax];
  __shared__ int cidx[kLmTopkMax];
  const float* z = logits + static_cast<long long>(blockIdx.x) * ld;
  const int tid = threadIdx.x;
  const float m = row_max(z, V, red);
  const float lse = m + logf(row_expsum(z, V, m, red));
  auto key_of = [&](int c) -> uint32_t { return enc_max(c == exclude ? -INFINITY : z[c] - lse); };

  uint32_t prefix = 0, mask = 0;
  unsigned remaining = static_cast<unsigned>(k);
  for (int byte = 3; byte >= 0; --byte) {
    for (int i = tid; i < 256; i += kGenThreads) hist[i] = 0;
    __syncthreads();
    for (int c = tid; c < V; c += kGenThreads) {
      const uint32_t key = key_of(c);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> (8 * byte)) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      unsigned above = 0;
      int b = 255;
      for (; b > 0 && above + hist[b] < remaining; --b) above += hist[b];
      sel[0] = prefix | (static_cast<uint32_t>(b) << (8 * byte));
      sel[1] = remaining - above;
    }
    __syncthreads();
    prefix = sel[0];
    remaining = sel[1];
    mask |= 255u << (8 * byte);
    __syncthreads();
  }
  // prefix is the k-th largest key; `remaining` ties at it are taken, lowest columns first, after k - remaining above
  const unsigned n_above = static_cast<unsigned>(k) - remaining;
  if (tid == 0) n_gt = 0;
  __syncthreads();
  for (int c = tid; c < V; c += kGenThreads) {
    const uint32_t key = key_of(c);
    if (key > prefix) {
      const unsigned p = atomicAdd(&n_gt, 1u);
      ckey[p] = key;
      cidx[p] = c;
    }
  }
  const int w = tid >> 5, lane = tid & 31;
  unsigned taken = 0;
  for (int base = 0; base < V && taken < remaining; base += kGenThreads) {
    const int c = base + tid;
    const bool tie = c < V && key_of(c) == prefix;
    const unsigned bal = __ballot_sync(~0u, tie);
    if (lane == 0) wcount[w] = __popc(bal);
    __syncthreads();
    unsigned before = 0, total = 0;
    for (int i = 0; i < kGenWarps; ++i) {
      if (i < w) before += wcount[i];
      total += wcount[i];
    }
    before += __popc(bal & ((1u << lane) - 1u));
    if (tie && taken + before < remaining) {
      ckey[n_above + taken + before] = prefix;
      cidx[n_above + taken + before] = c;
    }
    taken += total;
    __syncthreads();
  }
  __syncthreads();
  // rank sort of the k entries: value descending, then column ascending
  if (tid < k) {
    const uint32_t kk = ckey[tid];
    const int ci = cidx[tid];
    int rank = 0;
    for (int j = 0; j < k; ++j) rank += (ckey[j] > kk) || (ckey[j] == kk && cidx[j] < ci);
    const long long o = static_cast<long long>(blockIdx.x) * k + rank;
    values[o] = dec_max(kk);
    idx[o] = ci;
  }
}

// per row r (one CTA): fastai's predict weights over the row's logits z,
//   p_j = expf(z_j - m) / s (torch's softmax: m the row max, s the fixed-order sum of expf(z - m));
//   w_j = 0 at the excluded column; with min_p > 0, 0 where p_j < min_p unless no column has p_j >= min_p (then
//   flags[r] = 1 and nothing is masked); with inv_t != 1, w_j = powf(w_j, inv_t);
// and the draw: the first column j of positive weight whose running sum S_j (fixed order, file comment) exceeds
// f32(u_r * total), total the final carry of the scan (the file comment: not S_{V-1}).  The scan is not monotone in
// rounding (a lane's prefix sums its terms in another order than its left neighbour's, so a zero weight can round one
// ulp above the column before it): columns of weight 0 are skipped explicitly and can never be drawn.  When no positive column's S_j exceeds the target (it rounded up to the total),
// the last column of positive weight is drawn.  A total of 0 sets flags[r] = 2 and bit 1 of err and draws column 0.
__global__ void __launch_bounds__(kGenThreads) lm_sample_kernel(const float* __restrict__ logits, long long ld, int V,
                                                                 const float* __restrict__ u, int exclude, float min_p,
                                                                 float inv_t, int64_t* __restrict__ out,
                                                                 int* __restrict__ flags, int* err) {
  __shared__ float red[kGenWarps + 1];
  __shared__ int found, last_pos, survivors;
  const float* z = logits + static_cast<long long>(blockIdx.x) * ld;
  const int tid = threadIdx.x;
  const float m = row_max(z, V, red);
  const float s = row_expsum(z, V, m, red);
  bool mask_min = false;
  if (min_p > 0.0f) {
    if (tid == 0) survivors = 0;
    __syncthreads();
    int any = 0;
    for (int c = tid; c < V; c += kGenThreads) any |= (c != exclude && expf(z[c] - m) / s >= min_p);
    if (any) atomicOr(&survivors, 1);
    __syncthreads();
    mask_min = survivors != 0;
  }
  auto weight = [&](int c) -> float {
    if (c >= V || c == exclude) return 0.0f;
    const float p = expf(z[c] - m) / s;
    if (mask_min && p < min_p) return 0.0f;
    return inv_t != 1.0f ? powf(p, inv_t) : p;
  };
  // pass 1: the total (the final carry) and the last column of positive weight; pass 2: the first S_j above the target
  if (tid == 0) { found = INT_MAX; last_pos = -1; }
  __syncthreads();
  float carry = 0.0f, chunk_total;
  for (int base = 0; base < V; base += kGenThreads) {
    const float wv = weight(base + tid);
    if (wv > 0.0f) atomicMax(&last_pos, base + tid);
    block_scan(wv, red, &chunk_total);
    carry = carry + chunk_total;   // red[31], not the chunk's last S_j (file comment)
  }
  const float total = carry;
  const float target = u[blockIdx.x] * total;
  carry = 0.0f;
  for (int base = 0; base < V && total > 0.0f; base += kGenThreads) {
    const int c = base + tid;
    const float wv = weight(c);
    const float S = carry + block_scan(wv, red, &chunk_total);
    if (wv > 0.0f && S > target) atomicMin(&found, c);
    __syncthreads();
    if (found != INT_MAX) break;
    carry = carry + chunk_total;
  }
  if (tid == 0) {
    int f = (min_p > 0.0f && !mask_min) ? 1 : 0;
    int pick = found != INT_MAX ? found : last_pos;
    if (!(total > 0.0f)) {
      f = 2;
      pick = 0;
      atomicOr(err, 2);
    }
    out[blockIdx.x] = pick;
    flags[blockIdx.x] = f;
  }
}

// One CTA: scores f32(parent_scores[r] - values[r, c]) of the n = rows * top_k candidates j = r * top_k + c, sorted
// ascending by (score, j) -- a stable sort's order -- by a bitonic sort of 64-bit keys (enc_max(score) << 32 | j) in
// shared memory; the first beam_sz survive.  Survivor i: parent[i] = j / top_k, token[i] = tokens[j], score[i], and
// nodes_out[i] = nodes_in[parent[i]] followed by the token (L columns in, L + 1 out).  -0 scores count as +0.
__global__ void __launch_bounds__(kGenThreads) lm_beam_select_kernel(
    const float* __restrict__ parent_scores, const float* __restrict__ values, const int64_t* __restrict__ tokens,
    int n, int n2, int top_k, int beam_sz, const int64_t* __restrict__ nodes_in, int L, int* __restrict__ parent,
    int64_t* __restrict__ token, float* __restrict__ score, int64_t* __restrict__ nodes_out) {
  extern __shared__ unsigned long long keys[];
  for (int j = threadIdx.x; j < n2; j += kGenThreads) {
    unsigned long long k = ~0ull;
    if (j < n) {
      float sc = parent_scores[j / top_k] - values[j];
      if (sc == 0.0f) sc = 0.0f;
      k = (static_cast<unsigned long long>(enc_max(sc)) << 32) | static_cast<unsigned>(j);
    }
    keys[j] = k;
  }
  __syncthreads();
  for (int size = 2; size <= n2; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < n2 / 2; i += kGenThreads) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
      }
      __syncthreads();
    }
  const int keep = n < beam_sz ? n : beam_sz;
  for (int i = threadIdx.x; i < keep; i += kGenThreads) {
    const unsigned long long k = keys[i];
    const int j = static_cast<int>(k & 0xffffffffu);
    const int r = j / top_k;
    parent[i] = r;
    token[i] = tokens[j];
    score[i] = dec_max(static_cast<uint32_t>(k >> 32));
  }
  for (long long e = threadIdx.x; e < static_cast<long long>(keep) * (L + 1); e += kGenThreads) {
    const int i = static_cast<int>(e / (L + 1)), col = static_cast<int>(e % (L + 1));
    const int j = static_cast<int>(keys[i] & 0xffffffffu);
    nodes_out[e] = col < L ? nodes_in[static_cast<long long>(j / top_k) * L + col] : tokens[j];
  }
}

// dst row i of every layer = src row parent[i] (rows of row_u4 16-byte words, layers layer_u4 apart); a parent outside
// [0, src_rows) raises bit 2 of err and copies row 0
__global__ void gather_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, const int* __restrict__ parent,
                                   int src_rows, long long row_u4, long long layer_u4, int* err) {
  int p = parent[blockIdx.x];
  if (p < 0 || p >= src_rows) {
    if (threadIdx.x == 0) atomicOr(err, 4);
    p = 0;
  }
  const long long lo = blockIdx.y * layer_u4;
  const uint4* s = src + lo + p * row_u4;
  uint4* d = dst + lo + blockIdx.x * row_u4;
  for (long long i = threadIdx.x; i < row_u4; i += blockDim.x) d[i] = s[i];
}

}  // namespace

cudaError_t launch_lm_topk(const float* logits, long long ld, int rows, int V, int k, int exclude, float* values,
                           int64_t* idx, cudaStream_t stream) {
  if (rows < 1 || V < 1 || k < 1 || k > kLmTopkMax || k > V) return cudaErrorInvalidValue;
  lm_topk_kernel<<<rows, kGenThreads, 0, stream>>>(logits, ld, V, k, exclude, values, idx);
  return cudaGetLastError();
}

cudaError_t launch_lm_sample(const float* logits, long long ld, int rows, int V, const float* u, int exclude,
                             float min_p, float inv_t, int64_t* out, int* flags, int* err, cudaStream_t stream) {
  if (rows < 1 || V < 1) return cudaErrorInvalidValue;
  lm_sample_kernel<<<rows, kGenThreads, 0, stream>>>(logits, ld, V, u, exclude, min_p, inv_t, out, flags, err);
  return cudaGetLastError();
}

cudaError_t launch_lm_beam_select(const float* parent_scores, const float* values, const int64_t* tokens, int rows,
                                  int top_k, int beam_sz, const int64_t* nodes_in, int L, int* parent, int64_t* token,
                                  float* score, int64_t* nodes_out, cudaStream_t stream) {
  const long long n = static_cast<long long>(rows) * top_k;
  if (rows < 1 || top_k < 1 || beam_sz < 1 || n > kLmBeamMax || L < 0) return cudaErrorInvalidValue;
  int n2 = 2;
  while (n2 < n) n2 <<= 1;
  const size_t smem = static_cast<size_t>(n2) * sizeof(unsigned long long);
  cudaError_t e = cudaFuncSetAttribute(lm_beam_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  lm_beam_select_kernel<<<1, kGenThreads, smem, stream>>>(parent_scores, values, tokens, static_cast<int>(n), n2, top_k,
                                                          beam_sz, nodes_in, L, parent, token, score, nodes_out);
  return cudaGetLastError();
}

cudaError_t launch_gather_rows(const void* src, void* dst, const int* parent, int n, int src_rows, long long row_bytes,
                               long long layer_bytes, int layers, int* err, cudaStream_t stream) {
  if (n < 1 || layers < 1 || row_bytes % 16 || layer_bytes % 16) return cudaErrorInvalidValue;
  gather_rows_kernel<<<dim3(n, layers), 256, 0, stream>>>(static_cast<const uint4*>(src), static_cast<uint4*>(dst), parent,
                                                          src_rows, row_bytes / 16, layer_bytes / 16, err);
  return cudaGetLastError();
}

}  // namespace ie
