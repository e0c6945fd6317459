// Training step of the label MLP (sklearn MLPClassifier, solver 'adam', relu hidden layers, logistic output): the
// elementwise stages around the persistent GEMM (gemm.cu) that api_mlp_train.cu's ie_mlp_train_* sequence launches.
//
//   split_store_kernel   f32 [rows, cols] (optional row gather, optional relu mask) -> split-bf16 operands: row-major
//                        [hi | lo] for the next product's A, transposed [hi | lo] (K = batch) for a weight gradient, and
//                        the exact zero padding both products read
//   output_kernel        sigmoid of the last layer, delta = p - y, per-row log-loss terms (f64, fixed order)
//   grad_kernel          coef gradient (D + alpha W) / b from the a^T delta product, intercept gradient sum(delta) / b
//   loss_kernel          batch loss -sum(rows) / b + 0.5 alpha sum|W|^2 / b (f64, fixed order)
//   adam_kernel          sklearn AdamOptimizer on float32 arrays, bit for bit, plus per-block f64 partials of sum|W|^2
//
// Every reduction runs in a fixed order without atomics, so a fit is deterministic.
//
// mlp_group.cu repeats each of these kernels for many models at once, and api_mlp_train.cu's mg_* sequence repeats mt_forward /
// mt_backward / mt_adam; a grouped fit is bit-identical to a single one only while each pair does the same arithmetic
// over the same partition, so change both together (tests/test_gpu_mlp_grid_search.py checks the pairs bit for bit).
#include <cuda_bf16.h>

#include <algorithm>

#include "kernels.h"
#include "ptx.cuh"

namespace ie {

namespace {

constexpr int kTile = 32;

__device__ __forceinline__ void store_split(__nv_bfloat16* p, int lo_off, float v) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  p[0] = hi;
  p[lo_off] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

__global__ void split_store_kernel(const SplitStoreArgs a) {
  __shared__ float t[kTile][kTile + 1];
  const int c0 = blockIdx.x * kTile, r0 = blockIdx.y * kTile;
  const int tx = threadIdx.x;
  for (int i = threadIdx.y; i < kTile; i += blockDim.y) {
    const int r = r0 + i, c = c0 + tx;
    float v = 0.0f;
    if (r < a.rows && c < a.cols) {
      const long long sr = a.rowidx != nullptr ? a.rowidx[r] : r;
      v = a.src[sr * a.ld_src + c];
      // sklearn inplace_relu_derivative: delta[a == 0] = 0, on the device's own stored activation
      if (a.mask != nullptr && a.mask[static_cast<long long>(r) * a.ld_mask + c] == 0.0f) v = 0.0f;
      if (a.out_f32 != nullptr) a.out_f32[static_cast<long long>(r) * a.ld_f32 + c] = v;
    }
    t[i][tx] = v;
    if (a.rm != nullptr && r < a.rm_rows && c < a.rm_kpad) store_split(a.rm + static_cast<long long>(r) * a.ld_rm + c, a.rm_kpad, v);
  }
  if (a.tr == nullptr) return;
  __syncthreads();
  for (int i = threadIdx.y; i < kTile; i += blockDim.y) {
    const int c = c0 + i, r = r0 + tx;  // transposed: row c (feature), column r (batch row)
    if (c < a.tr_rows && r < a.tr_kpad) store_split(a.tr + static_cast<long long>(c) * a.ld_tr + r, a.tr_kpad, t[tx][i]);
  }
}

// fixed-order block sum (blockDim.x == 256) of one double per thread; the result is valid in thread 0
__device__ double block_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}

constexpr int kRedThreads = 256;

__global__ void __launch_bounds__(kRedThreads) output_kernel(const float* __restrict__ z, long long ldz,
                                                             const uint8_t* __restrict__ Y, const int* __restrict__ rowidx,
                                                             int L, float* __restrict__ p, float* __restrict__ delta,
                                                             double* __restrict__ row_loss) {
  __shared__ double sh[kRedThreads];
  const int r = blockIdx.x;
  const long long yr = static_cast<long long>(rowidx != nullptr ? rowidx[r] : r) * L;
  double acc = 0.0;
  for (int c = threadIdx.x; c < L; c += blockDim.x) {
    const float pr = sigmoid_acc(z[r * ldz + c]);
    p[r * ldz + c] = pr;
    if (Y == nullptr) continue;
    const bool y = Y[yr + c] != 0;
    delta[r * ldz + c] = __fsub_rn(pr, y ? 1.0f : 0.0f);
    // sklearn binary_log_loss: clip to [eps, 1 - eps] (float32 eps), xlogy(y, p) + xlogy(1 - y, 1 - p)
    const double pc = static_cast<double>(fminf(fmaxf(pr, 0x1p-23f), 1.0f - 0x1p-23f));
    acc += y ? log(pc) : log(1.0 - pc);
  }
  if (Y == nullptr) return;
  const double s = block_sum(acc, sh);
  if (threadIdx.x == 0) row_loss[r] = s;
}

__global__ void grad_kernel(const float* __restrict__ dw, long long ld_dw, const float* __restrict__ W, int fan_in,
                            int fan_out, const float* __restrict__ delta, long long ld_delta, int b, float alpha,
                            float* __restrict__ gW, float* __restrict__ gb, int coef_blocks) {
  const float fb = static_cast<float>(b);
  if (static_cast<int>(blockIdx.x) < coef_blocks) {
    const long long n = static_cast<long long>(fan_in) * fan_out;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(coef_blocks) * blockDim.x) {
      const long long r = i / fan_out, c = i - r * fan_out;
      // sklearn _compute_loss_grad in float32: coef_grads += alpha * coefs; coef_grads /= n  (no contraction)
      gW[i] = __fdiv_rn(__fadd_rn(dw[r * ld_dw + c], __fmul_rn(alpha, W[i])), fb);
    }
    return;
  }
  const int c = (blockIdx.x - coef_blocks) * blockDim.x + threadIdx.x;
  if (c >= fan_out) return;
  double s = 0.0;
  for (int r = 0; r < b; ++r) s += static_cast<double>(delta[static_cast<long long>(r) * ld_delta + c]);
  gb[c] = static_cast<float>(s / static_cast<double>(b));
}

__global__ void __launch_bounds__(kRedThreads) loss_kernel(const double* __restrict__ row_loss, int b,
                                                           const double* __restrict__ sq_part, int n_part, double alpha,
                                                           double* __restrict__ out) {
  __shared__ double sh[kRedThreads];
  double a = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < b; i += blockDim.x) a += row_loss[i];
  for (int i = threadIdx.x; i < n_part; i += blockDim.x) q += sq_part[i];
  const double rows = block_sum(a, sh);
  __syncthreads();
  const double sq = block_sum(q, sh);
  if (threadIdx.x == 0) *out = -rows / b + 0.5 * alpha * sq / b;
}

__global__ void __launch_bounds__(kRedThreads) adam_kernel(AdamArgs a) {
  __shared__ double sh[kRedThreads];
  double q = 0.0;
  const double neg_lr = a.lr != nullptr ? -a.lr[a.step] : 0.0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float p = a.p[i];
    if (a.g != nullptr) {
      // sklearn AdamOptimizer._get_updates on float32 arrays under NumPy 2 promotion: the Python-float constants act
      // as float32, each product and sum is rounded on its own; learning_rate is a float64 scalar, so the update is
      // float64 and `param += update` rounds f64(p) + update to float32
      const float g = a.g[i];
      const float m = __fadd_rn(__fmul_rn(a.beta1, a.m[i]), __fmul_rn(a.one_m_beta1, g));
      const float v = __fadd_rn(__fmul_rn(a.beta2, a.v[i]), __fmul_rn(a.one_m_beta2, __fmul_rn(g, g)));
      const float den = __fadd_rn(__fsqrt_rn(v), a.eps);
      const double upd = __ddiv_rn(__dmul_rn(neg_lr, static_cast<double>(m)), static_cast<double>(den));
      p = __double2float_rn(__dadd_rn(static_cast<double>(p), upd));
      a.m[i] = m;
      a.v[i] = v;
      a.p[i] = p;
    }
    if (i < a.n_coef) q += static_cast<double>(p) * static_cast<double>(p);
  }
  const double s = block_sum(q, sh);
  if (threadIdx.x == 0) a.sq_part[blockIdx.x] = s;
}

}  // namespace

cudaError_t launch_split_store(const SplitStoreArgs& a, cudaStream_t stream) {
  const int rows = std::max(a.rm != nullptr ? a.rm_rows : a.rows, a.tr != nullptr ? a.tr_kpad : 0);
  const int cols = std::max(a.rm != nullptr ? a.rm_kpad : a.cols, a.tr != nullptr ? a.tr_rows : 0);
  if (rows < 1 || cols < 1) return cudaErrorInvalidValue;
  const dim3 grid((cols + kTile - 1) / kTile, (rows + kTile - 1) / kTile);
  split_store_kernel<<<grid, dim3(kTile, 8), 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_mlp_output(const float* z, long long ldz, const uint8_t* Y, const int* rowidx, int b, int L, float* p,
                              float* delta, double* row_loss, cudaStream_t stream) {
  if (b < 1 || L < 1) return cudaErrorInvalidValue;
  output_kernel<<<b, kRedThreads, 0, stream>>>(z, ldz, Y, rowidx, L, p, delta, row_loss);
  return cudaGetLastError();
}

cudaError_t launch_mlp_grad(const float* dw, long long ld_dw, const float* W, int fan_in, int fan_out, const float* delta,
                            long long ld_delta, int b, float alpha, float* gW, float* gb, cudaStream_t stream) {
  const long long n = static_cast<long long>(fan_in) * fan_out;
  const int coef_blocks = static_cast<int>(std::min<long long>((n + 255) / 256, 132 * 8));
  const int bias_blocks = (fan_out + 255) / 256;
  grad_kernel<<<coef_blocks + bias_blocks, 256, 0, stream>>>(dw, ld_dw, W, fan_in, fan_out, delta, ld_delta, b, alpha, gW,
                                                           gb, coef_blocks);
  return cudaGetLastError();
}

cudaError_t launch_mlp_loss(const double* row_loss, int b, const double* sq_part, int n_part, double alpha, double* out,
                            cudaStream_t stream) {
  loss_kernel<<<1, kRedThreads, 0, stream>>>(row_loss, b, sq_part, n_part, alpha, out);
  return cudaGetLastError();
}

cudaError_t launch_adam(const AdamArgs& a, cudaStream_t stream) {
  adam_kernel<<<kAdamBlocks, kRedThreads, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace ie
