// The language model's decoder (ie_lm_* in include/issue_emb_b200.h): fastai's LinearDecoder followed by the
// per-token cross-entropy and argmax, fused so that the [tokens, vocab] logits never leave the registers.
//
//   stage 1  gemm_bf16_kernel<..., LmEpi>: logits = h W^T + b on the tensor cores (the encoder's ring as A, bf16 or
//            split-bf16), and per (row, vocabulary slice) a running (max, sum of exp(x - max), argmax) in registers;
//            the tile holding a row's target writes that logit
//   stage 2  lm_combine_kernel: per row, the slices in slice order -> lse = max + log(sum), nll = lse - logit[target]
//            (0 for target -100), pred = argmax (ties to the lowest index)
//
// Slices are kLmSliceTiles 256-column tiles wide whatever the grid or the batch, and every reduction runs in a fixed
// order, so a token's outputs are a function of its own state row alone.
#include <algorithm>

#include "gemm_kernel.cuh"

namespace ie {

namespace {

constexpr float kLog2e = 1.4426950408889634f;

// exp(x - m) through ex2_approx (ptx.cuh) for x <= m (0 for x = -inf); m must be finite
__device__ __forceinline__ float exp_sub(float x, float m) { return ex2_approx((x - m) * kLog2e); }

// (m, s, arg) <- (m, s, arg) merged with (m2, s2, arg2): max, rescaled sum, argmax with ties to the lower index.
// Symmetric in its two operands bit for bit (the sum of two products commutes), so both lanes of a shuffle agree.
__device__ __forceinline__ void merge(float& m, float& s, int& arg, float m2, float s2, int arg2) {
  const float mn = fmaxf(m, m2);
  if (mn == -INFINITY) return;
  const float a = m == -INFINITY ? 0.0f : s * exp_sub(m, mn);
  const float b = m2 == -INFINITY ? 0.0f : s2 * exp_sub(m2, mn);
  arg = m2 > m ? arg2 : (m > m2 ? arg : min(arg, arg2));
  s = a + b;
  m = mn;
}

}  // namespace

// Stage-1 epilogue of the persistent GEMM (gemm_kernel.cuh).  Rows are the time-major rows of a chunk of the encoder's
// ring: row r is step t0 + r / rps of batch row r % rps (rps = b_pad); rows with r % rps >= B are padding.  Work items
// are (valid 128-row block, vocabulary slice) pairs, row block fastest, dealt to the CTAs in turn (the CTAs running
// together share one slice of W in L2); a CTA sweeps its item's tiles in order.  Row blocks of padding alone are not
// scheduled.
struct LmEpi {
  static constexpr bool kSliced = true;
  static constexpr uint64_t kHintA = kEvictLast;    // the row block is read again for every tile of the slice
  static constexpr uint64_t kHintB = kEvictNormal;  // W tiles are shared by the CTAs of one slice, then done
  struct State {
    float m[2], s[2];
    int arg[2], tgt[2];   // tgt: the row's target column (-1: none)
    int item1;            // item + 1 of the rows' current partials (0: none yet)
  };
  LmPart* part;              // [rows][S]
  float* tlogit;             // [rows] logit of the row's target
  const float* bias;         // [n_pad] (zeros past V)
  const int64_t* targets;    // [B, T]
  int V, S, nbs, items, vpb;  // vpb: valid row blocks per slice = steps * vb
  int vb, bps, rps, B, T, t0;  // valid blocks per step, blocks per step, rows per step

  __device__ int num_tiles() const { return items * nbs; }
  __device__ int first_tile(int b) const { return b * nbs; }
  __device__ int next_tile(int t, int grid, int num_n_blocks) const {
    const int item = t / nbs, j = t - item * nbs;
    if (j + 1 < nbs && (item / vpb) * nbs + j + 1 < num_n_blocks) return t + 1;
    return (item + grid) * nbs;
  }
  __device__ int m_block(int item) const {
    const int v = item % vpb;
    return (v / vb) * bps + v % vb;
  }
  __device__ void decode(int t, int, int& m_blk, int& n_blk) const {
    const int item = t / nbs;
    m_blk = m_block(item);
    n_blk = (item / vpb) * nbs + (t - item * nbs);
  }
  __device__ bool valid(int row) const { return row % rps < B; }

  // the quad's partials of one slice, reduced in a fixed order, one write per valid row
  __device__ void flush(int row0w, int lane, const State& st) const {
    const int item = st.item1 - 1;
    const int slice = item / vpb;
    const int row0 = m_block(item) * 128 + row0w;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float m = st.m[hr], s = st.s[hr];
      int arg = st.arg[hr];
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1)
        merge(m, s, arg, __shfl_xor_sync(~0u, m, o), __shfl_xor_sync(~0u, s, o), __shfl_xor_sync(~0u, arg, o));
      const int row = row0 + (lane >> 2) + 8 * hr;
      if ((lane & 3) == 0 && valid(row)) part[static_cast<size_t>(row) * S + slice] = LmPart{m, s, arg, 0};
    }
  }

  // d: this thread's accumulators of the 128 x 256 tile (wgmma m64n256 layout: rows row0w + lane/4 + 8 hr, columns
  // 8 jg + 2 (lane % 4) + e at d[4 jg + 2 hr + e]); row0w: the warp's first row inside the tile
  __device__ void tile(float (&d)[128], int m_blk, int n_blk, int row0w, int lane, State& st) const {
    const int q = lane & 3, g = lane >> 2;
    const int slice = n_blk / nbs;
    const int row0 = m_blk * 128 + row0w;
    const int item = slice * vpb + (m_blk / bps) * vb + m_blk % bps;
    if (st.item1 != item + 1) {
      if (st.item1 != 0) flush(row0w, lane, st);
      st.item1 = item + 1;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        st.m[hr] = -INFINITY;
        st.s[hr] = 0.0f;
        st.arg[hr] = 0x7fffffff;
        const int row = row0 + g + 8 * hr;
        int tgt = -1;
        if (valid(row)) {
          const int64_t y = targets[static_cast<long long>(row % rps) * T + t0 + row / rps];
          if (y >= 0 && y < V) tgt = static_cast<int>(y);
        }
        st.tgt[hr] = tgt;
      }
    }
    const int cbase = n_blk * 256 + 2 * q;
#pragma unroll
    for (int jg = 0; jg < 32; ++jg) {
      const int c = cbase + 8 * jg;
      const float2 b = __ldg(reinterpret_cast<const float2*>(bias + c));
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float& v0 = d[4 * jg + 2 * hr];
        float& v1 = d[4 * jg + 2 * hr + 1];
        v0 = c < V ? v0 + b.x : -INFINITY;
        v1 = c + 1 < V ? v1 + b.y : -INFINITY;
      }
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
      int am = 0x7fffffff;
#pragma unroll
      for (int jg = 0; jg < 32; ++jg)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = d[4 * jg + 2 * hr + e];
          const int c = cbase + 8 * jg + e;
          if (v > mx) { mx = v; am = c; }   // columns ascend: ties keep the lower index
          if (c == st.tgt[hr]) tlogit[row0 + g + 8 * hr] = v;
        }
      if (mx == -INFINITY) continue;         // only columns past V in this thread's part of the tile
      const float mn = fmaxf(st.m[hr], mx);
      float ts = 0.0f;
#pragma unroll
      for (int jg = 0; jg < 32; ++jg)
#pragma unroll
        for (int e = 0; e < 2; ++e) ts += exp_sub(d[4 * jg + 2 * hr + e], mn);
      const float scale = st.m[hr] == -INFINITY ? 0.0f : exp_sub(st.m[hr], mn);
      if (mx > st.m[hr]) st.arg[hr] = am;    // earlier tiles hold lower columns: ties keep theirs
      st.s[hr] = st.s[hr] * scale + ts;
      st.m[hr] = mn;
    }
  }

  __device__ void finish(int row0w, int lane, State& st) const {
    if (st.item1 != 0) flush(row0w, lane, st);
  }
};

namespace {

// one thread per valid (step, batch row) of the chunk
__global__ void lm_combine_kernel(const LmPart* __restrict__ part, const float* __restrict__ tlogit,
                                  const int64_t* __restrict__ targets, int S, int V, int B, int T, int t0, int Tc,
                                  int rps, float* __restrict__ nll, float* __restrict__ lse, int* __restrict__ pred,
                                  int* err) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(Tc) * B) return;
  const int t = static_cast<int>(i / B), b = static_cast<int>(i - static_cast<long long>(t) * B);
  const long long r = static_cast<long long>(t) * rps + b;
  const LmPart* p = part + r * S;
  float m = p[0].m, s = p[0].s;
  int arg = p[0].arg;
  for (int k = 1; k < S; ++k) merge(m, s, arg, p[k].m, p[k].s, p[k].arg);
  const float l = m + logf(s);
  const long long o = static_cast<long long>(b) * T + t0 + t;
  const int64_t y = targets[o];
  float n;
  if (y == -100) {
    n = 0.0f;
  } else if (y < 0 || y >= V) {
    n = NAN;
    atomicOr(err, 1);
  } else {
    n = l - tlogit[r];
  }
  nll[o] = n;
  if (lse != nullptr) lse[o] = l;
  if (pred != nullptr) pred[o] = arg;
}

}  // namespace

int lm_slices(int V) { return (V + 256 * kLmSliceTiles - 1) / (256 * kLmSliceTiles); }

cudaError_t launch_lm_decode(const LmDecodeArgs& a, cudaStream_t stream) {
  if (a.k_pad % 64 || a.rps % 128 || a.rows % a.rps || a.B < 1 || a.B > a.rps || a.V < 1) return cudaErrorInvalidValue;
  CUtensorMap tmA, tmB;
  const uint64_t width = static_cast<uint64_t>(a.segs > 1 ? 2 : 1) * a.k_pad;
  cudaError_t e = make_tmap_bf16_2d(&tmA, a.h, width, static_cast<uint64_t>(a.rows), a.ld_h, kBlockK, kBlockM);
  if (e != cudaSuccess) return e;
  const int n_blocks = (a.V + kBlockN - 1) / kBlockN;
  e = make_tmap_bf16_2d(&tmB, a.w, width, static_cast<uint64_t>(n_blocks) * kBlockN, width, kBlockK, kBlockN);
  if (e != cudaSuccess) return e;
  LmEpi epi{};
  epi.part = a.part;
  epi.tlogit = a.tlogit;
  epi.bias = a.bias;
  epi.targets = a.targets;
  epi.V = a.V;
  epi.S = lm_slices(a.V);
  epi.nbs = kLmSliceTiles;
  epi.rps = a.rps;
  epi.bps = a.rps / kBlockM;
  epi.vb = (a.B + kBlockM - 1) / kBlockM;
  epi.B = a.B;
  epi.T = a.T;
  epi.t0 = a.t0;
  const long long steps = a.rows / a.rps;
  const long long vpb = steps * epi.vb;
  if (vpb * epi.S * kLmSliceTiles >= (1ll << 31)) return cudaErrorInvalidValue;
  epi.vpb = static_cast<int>(vpb);
  epi.items = static_cast<int>(vpb * epi.S);
  const int grid = std::min(epi.items, a.num_sms > 0 ? a.num_sms : 132);
  const size_t smem = 1024 + static_cast<size_t>(kGemmStages) * kGemmStageBytes + 2 * kGemmStages * 8 + 32;
  auto kfn = gemm_bf16_kernel<float, 0, false, LmEpi>;
  e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  kfn<<<grid, kGemmThreads, smem, stream>>>(tmA, tmB, nullptr, nullptr, 0, 0, 0, static_cast<int>(a.rows / kBlockM),
                                            n_blocks, a.k_pad / kBlockK, 16, a.segs, a.k_pad, a.abort_flag,
                                            a.spin_limit > 0 ? a.spin_limit : kSpinLimitDefault, nullptr, epi);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const long long n = (a.rows / a.rps) * a.B;
  lm_combine_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
      a.part, a.tlogit, a.targets, epi.S, a.V, a.B, a.T, a.t0, static_cast<int>(a.rows / a.rps), a.rps, a.nll, a.lse,
      a.pred, a.err);
  return cudaGetLastError();
}

}  // namespace ie
