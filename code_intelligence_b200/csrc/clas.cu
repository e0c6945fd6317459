// Text classifier (fastai's text_classifier_learner on the AWD-LSTM encoder, eval mode): the masked concat pool over a
// window of the last layer's states and the BatchNorm -> Linear (-> ReLU) head with its sigmoid / softmax output.
// Every kernel is fixed-order f32 with no atomics on values, so a row's result depends on that row alone.
#include <cmath>

#include "kernels.h"

namespace ie {
namespace {

constexpr int kPoolThreads = 128;

// one thread per (row b, unit c): a sequential pass over steps [s_b, e_b) of raw[b, :, c].
// fastai masked_concat_pool: avg = masked_fill(mask, 0).mean(1) * f32(W / (W - n_masked)); max = masked_fill(mask,
// -inf).max(1); last = o[:, -1] -- rounded as: sum in step order, mean = sum / W, avg = mean * factor.
__global__ void clas_pool_kernel(const float* __restrict__ raw, long long ld, int T, const int64_t* __restrict__ ids,
                                 const int* __restrict__ starts, const int* __restrict__ ends, int e_sz, int pad_idx,
                                 float* __restrict__ out, const int* __restrict__ enc_err, int* __restrict__ err) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * kPoolThreads + threadIdx.x;
  if (enc_err != nullptr && b == 0 && blockIdx.x == 0 && threadIdx.x == 0) {
    // the encoder's error words of this row group (its next call clears them): kept on the classifier's side
    if (enc_err[0]) atomicOr(err + 0, 1);
    if (enc_err[1]) atomicOr(err + 1, 1);
  }
  if (c >= e_sz) return;
  const int s = starts[b], e = ends[b];
  float* o = out + static_cast<long long>(b) * 3 * e_sz;
  if (s < 0 || e > T || s >= e) {
    if (c == 0) atomicOr(err + 2, 1);
    o[c] = o[e_sz + c] = o[2 * e_sz + c] = __int_as_float(0x7fc00000);
    return;
  }
  const float* r = raw + static_cast<long long>(b) * T * ld + c;
  const int64_t* id = ids + static_cast<long long>(b) * T;
  float sum = 0.0f, mx = -INFINITY;
  int n_masked = 0;
#pragma unroll 4
  for (int t = s; t < e; ++t) {
    if (id[t] == pad_idx) {
      ++n_masked;
    } else {
      const float v = r[static_cast<long long>(t) * ld];
      sum = __fadd_rn(sum, v);
      mx = fmaxf(mx, v);
    }
  }
  const int w = e - s;
  if (n_masked == w) {  // fastai gives NaN / -inf here: refused
    if (c == 0) atomicOr(err + 2, 1);
    o[c] = o[e_sz + c] = o[2 * e_sz + c] = __int_as_float(0x7fc00000);
    return;
  }
  const float mean = __fdiv_rn(sum, static_cast<float>(w));
  const float factor = __fdiv_rn(static_cast<float>(w), static_cast<float>(w - n_masked));
  o[c] = r[static_cast<long long>(e - 1) * ld];
  o[e_sz + c] = mx;
  o[2 * e_sz + c] = __fmul_rn(mean, factor);
}

constexpr int kRB = 8, kJB = 32, kKC = 128;

// y[r, j] = act(sum_k fma(x[r, k], alpha[k], beta[k]) * W[j, k] + bias[j]): the eval BatchNorm1d folded into a
// per-column scale and shift (torch's own form), then the Linear as a sequential fma chain over k = 0..K-1, the bias
// added last.  One thread per output; a CTA stages 8 normalised rows and 32 weight rows of each 128-wide k chunk.
__global__ void __launch_bounds__(kRB * kJB) clas_linear_kernel(const float* __restrict__ x, int rows, int K,
                                                                 const float* __restrict__ alpha,
                                                                 const float* __restrict__ beta,
                                                                 const float* __restrict__ W,
                                                                 const float* __restrict__ bias, int N, int relu,
                                                                 float* __restrict__ y) {
  __shared__ float xs[kRB][kKC];
  __shared__ float ws[kJB][kKC + 1];
  const int r0 = blockIdx.y * kRB, j0 = blockIdx.x * kJB;
  const int tr = threadIdx.x / kJB, tj = threadIdx.x % kJB;
  float acc = 0.0f;
  for (int k0 = 0; k0 < K; k0 += kKC) {
    for (int i = threadIdx.x; i < kRB * kKC; i += kRB * kJB) {
      const int rr = i / kKC, k = k0 + i % kKC, r = r0 + rr;
      xs[rr][i % kKC] = (r < rows && k < K) ? __fmaf_rn(x[static_cast<long long>(r) * K + k], alpha[k], beta[k]) : 0.0f;
    }
    for (int i = threadIdx.x; i < kJB * kKC; i += kRB * kJB) {
      const int jj = i / kKC, k = k0 + i % kKC, j = j0 + jj;
      ws[jj][i % kKC] = (j < N && k < K) ? W[static_cast<long long>(j) * K + k] : 0.0f;
    }
    __syncthreads();
    const int kn = min(kKC, K - k0);
    for (int kk = 0; kk < kn; ++kk) acc = __fmaf_rn(xs[tr][kk], ws[tj][kk], acc);
    __syncthreads();
  }
  const int r = r0 + tr, j = j0 + tj;
  if (r < rows && j < N) {
    float v = __fadd_rn(acc, bias[j]);
    if (relu && v < 0.0f) v = 0.0f;  // torch's ReLU: NaN stays NaN (fmaxf would return 0)
    y[static_cast<long long>(r) * N + j] = v;
  }
}

// one warp per row: sigmoid p = 1 / (1 + expf(-z)), or softmax p = expf(z - max) / sum with the sum taken as per-lane
// partials over j = lane, lane + 32, ... then a xor butterfly (every lane ends with the same bits)
__global__ void clas_activate_kernel(const float* __restrict__ z, int rows, int N, int softmax, float* __restrict__ p) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (row >= rows) return;
  const float* zr = z + static_cast<long long>(row) * N;
  float* pr = p + static_cast<long long>(row) * N;
  if (!softmax) {
    for (int j = lane; j < N; j += 32) pr[j] = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-zr[j])));
    return;
  }
  float m = -INFINITY;
  for (int j = lane; j < N; j += 32) m = fmaxf(m, zr[j]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.0f;
  for (int j = lane; j < N; j += 32) s = __fadd_rn(s, expf(__fsub_rn(zr[j], m)));
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  for (int j = lane; j < N; j += 32) pr[j] = __fdiv_rn(expf(__fsub_rn(zr[j], m)), s);
}

}  // namespace

cudaError_t launch_clas_pool(const float* raw, long long ld, int B, int T, const int64_t* ids, const int* starts,
                             const int* ends, int e_sz, int pad_idx, float* out, const int* enc_err, int* err,
                             cudaStream_t stream) {
  const dim3 grid((e_sz + kPoolThreads - 1) / kPoolThreads, B);
  clas_pool_kernel<<<grid, kPoolThreads, 0, stream>>>(raw, ld, T, ids, starts, ends, e_sz, pad_idx, out, enc_err, err);
  return cudaGetLastError();
}

cudaError_t launch_clas_linear(const float* x, int rows, int K, const float* alpha, const float* beta, const float* W,
                               const float* bias, int N, int relu, float* y, cudaStream_t stream) {
  const dim3 grid((N + kJB - 1) / kJB, (rows + kRB - 1) / kRB);
  clas_linear_kernel<<<grid, kRB * kJB, 0, stream>>>(x, rows, K, alpha, beta, W, bias, N, relu, y);
  return cudaGetLastError();
}

cudaError_t launch_clas_activate(const float* z, int rows, int N, int softmax, float* p, cudaStream_t stream) {
  const int per_block = 8;  // rows (warps) per 256-thread block
  clas_activate_kernel<<<(rows + per_block - 1) / per_block, 32 * per_block, 0, stream>>>(z, rows, N, softmax, p);
  return cudaGetLastError();
}

}  // namespace ie
