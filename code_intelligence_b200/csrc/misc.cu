// Memory-bound helper kernels of the encoder path (HBM-bound byte movement: coalesced 128-bit accesses, no
// tensor cores) and the TMA descriptor factory.
#include <cstring>

#include "kernels.h"
#include "lstm_common.cuh"
#include "ptx.cuh"

namespace ie {

// ---------------------------------------------------------------------------------------------
// TMA descriptors.  cuTensorMapEncodeTiled is fetched through the runtime so that the library has no link-time
// dependency on libcuda (the build container has no driver).
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

cudaError_t make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t ld,
                              uint32_t box_inner, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return cudaErrorNotSupported;
  if (box_inner != 64 || box_rows == 0 || box_rows > 256 || (ld * 2) % 16 != 0 ||
      (reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return cudaErrorInvalidValue;
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

namespace {

// ---------------------------------------------------------------------------------------------
// Embedding lookup (F.embedding inside fastai's EmbeddingDropout in eval mode; reference call site
// Issue_Embeddings/flask_app/inference.py:57).  One warp per (t, b) row, 16-byte loads/stores.
// Rows b >= B of the 128-padded batch get the pad token.
// ---------------------------------------------------------------------------------------------
__global__ void embed_gather_kernel(const int64_t* __restrict__ ids, int B, int T, int b_pad,
                                    const uint4* __restrict__ emb, int vocab, int chunks /* row bytes / 16 */,
                                    uint4* __restrict__ x0, long long ldx_chunks, int pad_idx, int* err_flag, int t0, int Tc) {
  const int warps_per_block = blockDim.x >> 5;
  const long long row = static_cast<long long>(blockIdx.x) * warps_per_block + (threadIdx.x >> 5);
  const long long total = static_cast<long long>(Tc) * b_pad;
  if (row >= total) return;
  const int lane = threadIdx.x & 31;
  const int tl = static_cast<int>(row / b_pad);
  const int b = static_cast<int>(row - static_cast<long long>(tl) * b_pad);
  const int t = t0 + tl;
  long long id = pad_idx;
  if (b < B) id = ids[static_cast<long long>(b) * T + t];
  if (id < 0 || id >= vocab) {
    if (lane == 0) atomicExch(err_flag, 1);
    id = 0;
  }
  const uint4* src = emb + id * chunks;
  uint4* dst = x0 + row * ldx_chunks;
  for (int i = lane; i < chunks; i += 32) dst[i] = __ldg(src + i);
}

// ids [B, T] int64 (batch-first) -> tok [T * b_pad] int32 (time-major, rows b >= B get the pad token), with the same
// range check as embed_gather_kernel.  Used when layer 0 reads its input projection from the per-token table
// (api.cu: IE_EMB_PROJ) instead of a GEMM over gathered embedding rows.
__global__ void tokens_time_major_kernel(const int64_t* __restrict__ ids, int B, int T, int b_pad, int vocab, int pad_idx,
                                         int* __restrict__ tok, int* err_flag) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(T) * b_pad;
  if (i >= total) return;
  const int t = static_cast<int>(i / b_pad);
  const int b = static_cast<int>(i - static_cast<long long>(t) * b_pad);
  long long id = pad_idx;
  if (b < B) id = ids[static_cast<long long>(b) * T + t];
  if (id < 0 || id >= vocab) {
    atomicExch(err_flag, 1);
    id = 0;
  }
  tok[i] = static_cast<int>(id);
}

__global__ void pool_finalize_kernel(const float* __restrict__ pool_sum, const float* __restrict__ pool_max,
                                     const float* __restrict__ pool_last, const int* __restrict__ lengths, int B, int e,
                                     int out_pad, float* __restrict__ out) {
  const int b = blockIdx.x;
  if (b >= B) return;
  const float inv = 1.0f / static_cast<float>(lengths[b]);
  const long long po = static_cast<long long>(b) * out_pad;
  float* o = out + static_cast<long long>(b) * 3 * e;
  for (int i = threadIdx.x; i < e; i += blockDim.x) {
    o[i] = pool_sum[po + i] * inv;
    o[e + i] = pool_max[po + i];
    o[2 * e + i] = pool_last[po + i];
  }
}

// device-pointer mode: the caller's lengths cannot be validated on the host -- clamp them to [1, T] here (a length of
// 0 would give 1/0 and max = -inf in pool_finalize) and raise err_flag[2]; padded rows get length 1
__global__ void prep_lengths_kernel(const int* __restrict__ in, int B, int T, int b_pad, int* __restrict__ out, int* err_flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b_pad) return;
  int v = 1;
  if (i < B) {
    v = in[i];
    if (v < 1 || v > T) {
      atomicExch(err_flag + 2, 1);
      v = v < 1 ? 1 : T;
    }
  }
  out[i] = v;
}

__global__ void convert_rows_kernel(const float* __restrict__ src, long long ld_src, int cols, const int* __restrict__ perm,
                                    int rows_dst, __nv_bfloat16* __restrict__ dst, long long ld_dst, int lo_off) {
  const int r = blockIdx.x;
  if (r >= rows_dst) return;
  const int sr = perm ? perm[r] : r;
  __nv_bfloat16* d = dst + static_cast<long long>(r) * ld_dst;
  const float* s = src + static_cast<long long>(sr < 0 ? 0 : sr) * ld_src;
  const int width = lo_off > 0 ? lo_off : static_cast<int>(ld_dst);
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    float v = 0.0f;
    if (sr >= 0 && c < cols) v = s[c];
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    d[c] = hi;
    if (lo_off > 0) d[lo_off + c] = __float2bfloat16_rn(v - __bfloat162float(hi));
  }
}

// Row-contiguous fast path of convert_rows_kernel (the MLP head's X f32 -> bf16 pass, the largest stream of that path):
// no permutation, cols % 4 == 0; one warp per row, 128-bit loads, 64-bit stores, zero fill of the K padding.
__global__ void convert_rows_vec_kernel(const float* __restrict__ src, long long ld_src, int cols, int rows,
                                        __nv_bfloat16* __restrict__ dst, long long ld_dst) {
  const int warps_per_block = blockDim.x >> 5;
  const long long r = static_cast<long long>(blockIdx.x) * warps_per_block + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const float4* s4 = reinterpret_cast<const float4*>(src + r * ld_src);
  uint2* d2 = reinterpret_cast<uint2*>(dst + r * ld_dst);
  const int n4 = cols >> 2, w4 = static_cast<int>(ld_dst >> 2);
  for (int i = lane; i < w4; i += 32) {
    uint2 o = make_uint2(0u, 0u);
    if (i < n4) {
      const float4 v = __ldcs(s4 + i);   // streaming: read once
      o = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    }
    d2[i] = o;
  }
}

__global__ void fill_f32_kernel(float* p, size_t n, float v) {
  size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

// test hook ie_debug_gates: the gate functions and the cell update exactly as the recurrent kernel and the GEMM
// epilogue inline them (ptx.cuh, lstm_common.cuh)
template <int FN>
__global__ void debug_gate_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float v = x[i];
    float r;
    if constexpr (FN == 0) r = sigmoid_fast(v);
    else if constexpr (FN == 1) r = tanh_fast(v);
    else if constexpr (FN == 2) r = sigmoid_acc(v);
    else if constexpr (FN == 3) r = tanh_acc(v);
    else if constexpr (FN == 4) r = sigmoid_ieee(v);
    else r = tanh_ieee(v);
    y[i] = r;
  }
}

// in = planes [zi | zf | zg | zo | c_prev] of n values, out = planes [c_new | h]
template <int GM>
__global__ void debug_cell_kernel(const float* __restrict__ in, float* __restrict__ out, long long n) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float c, h;
    lstm_cell1<GM>(in[i], in[n + i], in[2 * n + i], in[3 * n + i], in[4 * n + i], c, h);
    out[i] = c;
    out[n + i] = h;
  }
}

}  // namespace

cudaError_t launch_embed_gather(const int64_t* ids, int B, int T, int b_pad, const __nv_bfloat16* emb, int vocab,
                                int e_pad, __nv_bfloat16* x0, long long ldx, int pad_idx, int* err_flag, int t0, int Tc,
                                cudaStream_t stream) {
  if (e_pad % 8 || ldx % 8) return cudaErrorInvalidValue;
  const long long rows = static_cast<long long>(Tc) * b_pad;
  const int wpb = 8;
  const long long blocks = (rows + wpb - 1) / wpb;
  embed_gather_kernel<<<static_cast<unsigned>(blocks), wpb * 32, 0, stream>>>(
      ids, B, T, b_pad, reinterpret_cast<const uint4*>(emb), vocab, e_pad / 8, reinterpret_cast<uint4*>(x0), ldx / 8,
      pad_idx, err_flag, t0, Tc);
  return cudaGetLastError();
}

cudaError_t launch_tokens_time_major(const int64_t* ids, int B, int T, int b_pad, int vocab, int pad_idx, int* tok,
                                     int* err_flag, cudaStream_t stream) {
  const long long total = static_cast<long long>(T) * b_pad;
  const long long blocks = (total + 255) / 256;
  tokens_time_major_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(ids, B, T, b_pad, vocab, pad_idx, tok, err_flag);
  return cudaGetLastError();
}

cudaError_t launch_pool_finalize(const float* pool_sum, const float* pool_max, const float* pool_last,
                                 const int* lengths, int B, int e, int out_pad, float* out, cudaStream_t stream) {
  pool_finalize_kernel<<<B, 256, 0, stream>>>(pool_sum, pool_max, pool_last, lengths, B, e, out_pad, out);
  return cudaGetLastError();
}

cudaError_t launch_prep_lengths(const int* lengths_in, int B, int T, int b_pad, int* lengths_out, int* err_flag,
                                cudaStream_t stream) {
  prep_lengths_kernel<<<(b_pad + 255) / 256, 256, 0, stream>>>(lengths_in, B, T, b_pad, lengths_out, err_flag);
  return cudaGetLastError();
}

cudaError_t launch_convert_rows(const float* src, long long ld_src, int cols, const int* perm, int rows_dst,
                                __nv_bfloat16* dst, long long ld_dst, int lo_off, cudaStream_t stream) {
  if (lo_off > 0 && ld_dst < 2ll * lo_off) return cudaErrorInvalidValue;
  if (perm == nullptr && lo_off == 0 && cols % 4 == 0 && ld_src % 4 == 0 && ld_dst % 4 == 0 &&
      (reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
    const int wpb = 8;
    convert_rows_vec_kernel<<<(rows_dst + wpb - 1) / wpb, wpb * 32, 0, stream>>>(src, ld_src, cols, rows_dst, dst, ld_dst);
    return cudaGetLastError();
  }
  convert_rows_kernel<<<rows_dst, 256, 0, stream>>>(src, ld_src, cols, perm, rows_dst, dst, ld_dst, lo_off);
  return cudaGetLastError();
}

cudaError_t launch_fill_f32(float* p, size_t n, float v, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  size_t blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  fill_f32_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(p, n, v);
  return cudaGetLastError();
}

cudaError_t launch_debug_gates(int fn, const float* in, float* out, long long n, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 64) blocks = 132 * 64;
  const unsigned g = static_cast<unsigned>(blocks);
  switch (fn) {
    case 0: debug_gate_kernel<0><<<g, 256, 0, stream>>>(in, out, n); break;
    case 1: debug_gate_kernel<1><<<g, 256, 0, stream>>>(in, out, n); break;
    case 2: debug_gate_kernel<2><<<g, 256, 0, stream>>>(in, out, n); break;
    case 3: debug_gate_kernel<3><<<g, 256, 0, stream>>>(in, out, n); break;
    case 4: debug_gate_kernel<4><<<g, 256, 0, stream>>>(in, out, n); break;
    case 5: debug_gate_kernel<5><<<g, 256, 0, stream>>>(in, out, n); break;
    case 6: debug_cell_kernel<kGatesFast><<<g, 256, 0, stream>>>(in, out, n); break;
    case 7: debug_cell_kernel<kGatesExp><<<g, 256, 0, stream>>>(in, out, n); break;
    case 8: debug_cell_kernel<kGatesIeee><<<g, 256, 0, stream>>>(in, out, n); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace ie
