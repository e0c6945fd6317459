// Grouped training of the label MLP: the stages of mlp_train.cu and the persistent GEMM (gemm_kernel.cuh), each run
// once for every model of a group that shares a step's shape.  api.cu's ie_mlp_group_* sequence launches them.
//
// Model j of a launch is slot slots[j] of the group; its operands sit at base + slot * stride.  Each kernel performs,
// for every model, exactly the arithmetic of its single-model counterpart in mlp_train.cu over the same partition of
// the work, so a model's results are bit-identical to a single ie_mlp_train handle's:
//
//   group_split_store_kernel   split_store_kernel, model in blockIdx.z
//   group_output_kernel        output_kernel, model in blockIdx.y
//   group_grad_kernel          grad_kernel, model in blockIdx.y (same coef-block count per model)
//   group_loss_kernel          loss_kernel, one block per model
//   group_adam_kernel          adam_kernel, kAdamBlocks blocks per model in blockIdx.y
//   gemm_bf16_kernel<GroupEpi> the GEMM's mainloop with a sliced epilogue: the tiles of every model in one schedule,
//                              each stored as DenseEpi stores it (f32, + bias, optional relu)
//
// No value crosses from one model to another: every tile, block and reduction reads and writes one model's slot only.
#include <cuda_bf16.h>

#include <algorithm>

#include "gemm_kernel.cuh"
#include "kernels.h"
#include "ptx.cuh"

namespace ie {

namespace {

constexpr int kTile = 32;
constexpr int kRedThreads = 256;

__device__ __forceinline__ void store_split(__nv_bfloat16* p, int lo_off, float v) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  p[0] = hi;
  p[lo_off] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

__global__ void group_split_store_kernel(const GroupSplitArgs g) {
  __shared__ float t[kTile][kTile + 1];
  const long long s = g.slots[blockIdx.z];
  const SplitStoreArgs& a = g.a;
  const float* src = a.src + s * g.s_src;
  const int* rowidx = a.rowidx != nullptr ? a.rowidx + s * g.s_idx : nullptr;
  const float* mask = a.mask != nullptr ? a.mask + s * g.s_mask : nullptr;
  float* out_f32 = a.out_f32 != nullptr ? a.out_f32 + s * g.s_f32 : nullptr;
  __nv_bfloat16* rm = a.rm != nullptr ? a.rm + s * g.s_rm : nullptr;
  __nv_bfloat16* tr = a.tr != nullptr ? a.tr + s * g.s_tr : nullptr;
  const int c0 = blockIdx.x * kTile, r0 = blockIdx.y * kTile;
  const int tx = threadIdx.x;
  for (int i = threadIdx.y; i < kTile; i += blockDim.y) {
    const int r = r0 + i, c = c0 + tx;
    float v = 0.0f;
    if (r < a.rows && c < a.cols) {
      const long long sr = rowidx != nullptr ? rowidx[r] : r;
      v = src[sr * a.ld_src + c];
      if (mask != nullptr && mask[static_cast<long long>(r) * a.ld_mask + c] == 0.0f) v = 0.0f;
      if (out_f32 != nullptr) out_f32[static_cast<long long>(r) * a.ld_f32 + c] = v;
    }
    t[i][tx] = v;
    if (rm != nullptr && r < a.rm_rows && c < a.rm_kpad) store_split(rm + static_cast<long long>(r) * a.ld_rm + c, a.rm_kpad, v);
  }
  if (tr == nullptr) return;
  __syncthreads();
  for (int i = threadIdx.y; i < kTile; i += blockDim.y) {
    const int c = c0 + i, r = r0 + tx;
    if (c < a.tr_rows && r < a.tr_kpad) store_split(tr + static_cast<long long>(c) * a.ld_tr + r, a.tr_kpad, t[tx][i]);
  }
}

__device__ double block_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}

__global__ void __launch_bounds__(kRedThreads) group_output_kernel(const GroupOutputArgs g) {
  __shared__ double sh[kRedThreads];
  const long long s = g.slots[blockIdx.y];
  const int r = blockIdx.x;
  const float* z = g.z + s * g.s_z;
  float* p = g.p + s * g.s_p;
  const int* rowidx = g.rowidx != nullptr ? g.rowidx + s * g.s_idx : nullptr;
  const long long yr = static_cast<long long>(rowidx != nullptr ? rowidx[r] : r) * g.L;
  double acc = 0.0;
  for (int c = threadIdx.x; c < g.L; c += blockDim.x) {
    const float pr = sigmoid_acc(z[r * g.ldz + c]);
    p[r * g.ldz + c] = pr;
    if (g.Y == nullptr) continue;
    const bool y = g.Y[yr + c] != 0;
    g.delta[s * g.s_z + r * g.ldz + c] = __fsub_rn(pr, y ? 1.0f : 0.0f);
    const double pc = static_cast<double>(fminf(fmaxf(pr, 0x1p-23f), 1.0f - 0x1p-23f));
    acc += y ? log(pc) : log(1.0 - pc);
  }
  if (g.Y == nullptr) return;
  const double sum = block_sum(acc, sh);
  if (threadIdx.x == 0) g.row_loss[s * g.s_rl + r] = sum;
}

__global__ void group_grad_kernel(const GroupGradArgs g) {
  const long long s = g.slots[blockIdx.y];
  const float fb = static_cast<float>(g.b);
  const float alpha = static_cast<float>(g.alpha[s]);
  const float* dw = g.dw + s * g.s_dw;
  if (static_cast<int>(blockIdx.x) < g.coef_blocks) {
    const float* W = g.W + s * g.s_param;
    float* gW = g.gW + s * g.s_param;
    const long long n = static_cast<long long>(g.fan_in) * g.fan_out;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(g.coef_blocks) * blockDim.x) {
      const long long r = i / g.fan_out, c = i - r * g.fan_out;
      gW[i] = __fdiv_rn(__fadd_rn(dw[r * g.ld_dw + c], __fmul_rn(alpha, W[i])), fb);
    }
    return;
  }
  const int c = (blockIdx.x - g.coef_blocks) * blockDim.x + threadIdx.x;
  if (c >= g.fan_out) return;
  const float* delta = g.delta + s * g.s_delta;
  double sum = 0.0;
  for (int r = 0; r < g.b; ++r) sum += static_cast<double>(delta[static_cast<long long>(r) * g.ld_delta + c]);
  g.gb[s * g.s_param + c] = static_cast<float>(sum / static_cast<double>(g.b));
}

__global__ void __launch_bounds__(kRedThreads) group_loss_kernel(const GroupLossArgs g) {
  __shared__ double sh[kRedThreads];
  const long long s = g.slots[blockIdx.x];
  const double* row_loss = g.row_loss + s * g.s_rl;
  const double* sq_part = g.sq_part + s * kAdamBlocks;
  double a = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < g.b; i += blockDim.x) a += row_loss[i];
  for (int i = threadIdx.x; i < kAdamBlocks; i += blockDim.x) q += sq_part[i];
  const double rows = block_sum(a, sh);
  __syncthreads();
  const double sq = block_sum(q, sh);
  const double alpha = g.alpha[s];
  if (threadIdx.x == 0) g.out[s * g.s_out] = -rows / g.b + 0.5 * alpha * sq / g.b;
}

__global__ void __launch_bounds__(kRedThreads) group_adam_kernel(const GroupAdamArgs a) {
  __shared__ double sh[kRedThreads];
  const long long s = a.slots[blockIdx.y];
  float* P = a.p + s * a.s_param;
  const float* c = a.consts + s * 5;   // beta1, 1 - beta1, beta2, 1 - beta2, eps (f32 roundings)
  double q = 0.0;
  const double neg_lr = a.g != nullptr ? -a.lr[s * a.s_lr + a.step] : 0.0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float p = P[i];
    if (a.g != nullptr) {
      float* M = a.m + s * a.s_param;
      float* V = a.v + s * a.s_param;
      const float g = a.g[s * a.s_param + i];
      const float m = __fadd_rn(__fmul_rn(c[0], M[i]), __fmul_rn(c[1], g));
      const float v = __fadd_rn(__fmul_rn(c[2], V[i]), __fmul_rn(c[3], __fmul_rn(g, g)));
      const float den = __fadd_rn(__fsqrt_rn(v), c[4]);
      const double upd = __ddiv_rn(__dmul_rn(neg_lr, static_cast<double>(m)), static_cast<double>(den));
      p = __double2float_rn(__dadd_rn(static_cast<double>(p), upd));
      M[i] = m;
      V[i] = v;
      P[i] = p;
    }
    if (i < a.n_coef) q += static_cast<double>(p) * static_cast<double>(p);
  }
  const double sum = block_sum(q, sh);
  if (threadIdx.x == 0) a.sq_part[s * kAdamBlocks + blockIdx.x] = sum;
}

// Sliced epilogue over the models of a launch: tile t is tile t % per_model of model t / per_model (m fastest), its
// A rows at slot * a_blocks m-blocks and its B rows at slot * b_blocks n-blocks of the stacked operands; the tile is
// stored exactly as DenseEpi stores a float tile (bias add, then relu when asked).
struct GroupEpi {
  static constexpr bool kSliced = true;
  static constexpr uint64_t kHintA = kEvictNormal;
  static constexpr uint64_t kHintB = kEvictLast;
  struct State {};
  const int* slots;
  int count, mb, nb, a_blocks, b_blocks;
  float* d;
  long long ldd, s_d;
  const float* bias;
  long long s_bias;
  int m_store, n_store, relu;

  __device__ int num_tiles() const { return count * mb * nb; }
  __device__ int first_tile(int b) const { return b; }
  __device__ int next_tile(int t, int grid, int) const { return t + grid; }
  __device__ void decode(int t, int, int& m_blk, int& n_blk) const {
    const int per = mb * nb, j = t / per, r = t - j * per, n = r / mb;
    const int s = slots[j];
    m_blk = s * a_blocks + (r - n * mb);
    n_blk = s * b_blocks + n;
  }
  __device__ void tile(float (&acc)[128], int m_blk, int n_blk, int row0w, int lane, State&) const {
    const int s = n_blk / b_blocks;
    const int lm = m_blk - s * a_blocks, ln = n_blk - s * b_blocks;
    float* D = d + static_cast<long long>(s) * s_d;
    const float* bs = bias != nullptr ? bias + static_cast<long long>(s) * s_bias : nullptr;
    const int q = lane & 3;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = lm * kBlockM + row0w + (lane >> 2) + 8 * hr;
      if (row >= m_store) continue;
      float* drow = D + static_cast<long long>(row) * ldd;
#pragma unroll
      for (int jg = 0; jg < kBlockN / 8; ++jg) {
        const int n = ln * kBlockN + 8 * jg + 2 * q;
        if (n < n_store) {
          float x0 = acc[4 * jg + 2 * hr], x1 = acc[4 * jg + 2 * hr + 1];
          if (bs != nullptr) {
            const float2 b2 = __ldg(reinterpret_cast<const float2*>(bs + n));
            x0 += b2.x;
            x1 += b2.y;
          }
          if (relu) { x0 = fmaxf(x0, 0.0f); x1 = fmaxf(x1, 0.0f); }
          *reinterpret_cast<float2*>(drow + n) = make_float2(x0, x1);
        }
      }
    }
  }
  __device__ void finish(int, int, State&) const {}
};

}  // namespace

cudaError_t launch_group_split_store(const GroupSplitArgs& g, cudaStream_t stream) {
  const SplitStoreArgs& a = g.a;
  const int rows = std::max(a.rm != nullptr ? a.rm_rows : a.rows, a.tr != nullptr ? a.tr_kpad : 0);
  const int cols = std::max(a.rm != nullptr ? a.rm_kpad : a.cols, a.tr != nullptr ? a.tr_rows : 0);
  if (rows < 1 || cols < 1 || g.count < 1) return cudaErrorInvalidValue;
  const dim3 grid((cols + kTile - 1) / kTile, (rows + kTile - 1) / kTile, g.count);
  group_split_store_kernel<<<grid, dim3(kTile, 8), 0, stream>>>(g);
  return cudaGetLastError();
}

cudaError_t launch_group_output(const GroupOutputArgs& g, cudaStream_t stream) {
  if (g.b < 1 || g.L < 1 || g.count < 1) return cudaErrorInvalidValue;
  group_output_kernel<<<dim3(g.b, g.count), kRedThreads, 0, stream>>>(g);
  return cudaGetLastError();
}

cudaError_t launch_group_grad(GroupGradArgs g, cudaStream_t stream) {
  if (g.count < 1) return cudaErrorInvalidValue;
  const long long n = static_cast<long long>(g.fan_in) * g.fan_out;
  g.coef_blocks = static_cast<int>(std::min<long long>((n + 255) / 256, 132 * 8));   // as launch_mlp_grad
  const int bias_blocks = (g.fan_out + 255) / 256;
  group_grad_kernel<<<dim3(g.coef_blocks + bias_blocks, g.count), 256, 0, stream>>>(g);
  return cudaGetLastError();
}

cudaError_t launch_group_loss(const GroupLossArgs& g, cudaStream_t stream) {
  if (g.count < 1) return cudaErrorInvalidValue;
  group_loss_kernel<<<g.count, kRedThreads, 0, stream>>>(g);
  return cudaGetLastError();
}

cudaError_t launch_group_adam(const GroupAdamArgs& a, cudaStream_t stream) {
  if (a.count < 1) return cudaErrorInvalidValue;
  group_adam_kernel<<<dim3(kAdamBlocks, a.count), kRedThreads, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_group_gemm(const GroupGemmArgs& g, cudaStream_t stream) {
  if (g.m_pad % kBlockM || g.k_pad % kBlockK || g.a_rows % kBlockM || g.b_rows % kBlockN || g.m_pad > g.a_rows ||
      g.n_pad > g.b_rows || g.n_store % 16 || g.ldd % 2 || g.count < 1 || g.n_models < 1)
    return cudaErrorInvalidValue;
  CUtensorMap tmA, tmB;
  const uint64_t k_inner = 2ull * g.k_pad;   // split-bf16 operands: [hi | lo]
  cudaError_t e = make_tmap_bf16_2d(&tmA, g.a, k_inner, static_cast<uint64_t>(g.n_models) * g.a_rows, g.lda, kBlockK,
                                    kBlockM);
  if (e != cudaSuccess) return e;
  e = make_tmap_bf16_2d(&tmB, g.b, k_inner, static_cast<uint64_t>(g.n_models) * g.b_rows, g.ldb, kBlockK, kBlockN);
  if (e != cudaSuccess) return e;
  GroupEpi epi{};
  epi.slots = g.slots;
  epi.count = g.count;
  epi.mb = g.m_pad / kBlockM;
  epi.nb = (g.n_pad + kBlockN - 1) / kBlockN;
  epi.a_blocks = static_cast<int>(g.a_rows / kBlockM);
  epi.b_blocks = static_cast<int>(g.b_rows / kBlockN);
  epi.d = g.d;
  epi.ldd = g.ldd;
  epi.s_d = g.s_d;
  epi.bias = g.bias;
  epi.s_bias = g.s_bias;
  epi.m_store = g.m_store;
  epi.n_store = g.n_store;
  epi.relu = g.relu;
  const long long tiles = static_cast<long long>(g.count) * epi.mb * epi.nb;
  if (tiles >= (1ll << 31)) return cudaErrorInvalidValue;
  const int sms = g.num_sms > 0 ? g.num_sms : 132;
  const int grid = static_cast<int>(std::min<long long>(tiles, sms));
  const size_t smem = 1024 + static_cast<size_t>(kGemmStages) * kGemmStageBytes + 2 * kGemmStages * 8 + 32;
  auto kfn = gemm_bf16_kernel<float, 0, false, GroupEpi>;
  e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  kfn<<<grid, kGemmThreads, smem, stream>>>(tmA, tmB, nullptr, nullptr, 0, 0, 0, epi.mb, epi.nb, g.k_pad / kBlockK, 16,
                                            3, g.k_pad, nullptr, kSpinLimitDefault, nullptr, epi);
  return cudaGetLastError();
}

}  // namespace ie
