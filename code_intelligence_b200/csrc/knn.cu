// Exact k-nearest-neighbour search over issue embeddings (ie_knn_* in include/issue_emb_b200.h).
//
// Reference consumers: the reference README's duplicate detection / reviewer recommendation, the FewShot notebook's
// oneshotlabeler (CosineSimilarity ranking) and KNeighborsClassifier(metric='cosine'), notebook 08's
// KNeighborsClassifier(weights='distance') label model.
//
//   ingest   knn_center_*    c = f64 column mean of the first add's rows, rounded to f32 (fixed from then on)
//            knn_prep_rows   x~ = x - c as split-bf16 [hi | lo] (the launch_convert_rows layout) + per-row f64 terms
//   stage 1  gemm_bf16_kernel<..., KnnEpi>: S~ = Q~ X~^T on the tensor cores (split-bf16, segs = 3), affine epilogue
//            (larger = nearer), running top-k' per (query, corpus slice) in a global candidate buffer -- the nq x n
//            score matrix never leaves the registers
//   stage 2  knn_merge_rerank: per query, bitonic sort of the slices' candidates -> best k', exact f64 distances
//            from the stored f32 rows, best k by (distance, index)
#include <algorithm>

#include "gemm_kernel.cuh"

namespace ie {

namespace {

// monotone map float -> uint32: larger score, larger key; every non-NaN score maps above 0 (0 = empty slot).  -0 is
// keyed as +0, so an exact-zero score ties by index whichever sign the MMA or the epilogue gave it.
__device__ __forceinline__ uint32_t order_key(float s) {
  const uint32_t b = __float_as_uint(s) == 0x80000000u ? 0u : __float_as_uint(s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_score(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Warp-collective: keep the kp best of the count entries {key, index} of buf (key descending, ties to the lower
// index) in buf[0, kp) and return the kp-th best score.  Streams buf from L1 / L2: a row compacts only when its
// buffer would overflow, a handful of times per slice once the threshold has settled.
__device__ __noinline__ float knn_compact(uint2* buf, int count, int kp, int lane) {
  __syncwarp();
  uint32_t t = 0;   // the kp-th largest key, bit by bit: the largest t with #{key >= t} >= kp
  for (int bit = 31; bit >= 0; --bit) {
    const uint32_t c = t | (1u << bit);
    int m = 0;
    for (int i = lane; i < count; i += 32) m += buf[i].x >= c;
    if (static_cast<int>(__reduce_add_sync(~0u, static_cast<unsigned>(m))) >= kp) t = c;
  }
  int gt = 0, eq = 0;
  for (int i = lane; i < count; i += 32) {
    gt += buf[i].x > t;
    eq += buf[i].x == t;
  }
  gt = static_cast<int>(__reduce_add_sync(~0u, static_cast<unsigned>(gt)));
  eq = static_cast<int>(__reduce_add_sync(~0u, static_cast<unsigned>(eq)));
  const int want = kp - gt;   // entries with key == t that stay: the `want` lowest indices
  uint32_t imax = 0xffffffffu;
  if (eq > want) {
    uint32_t lo = 0, hi = 0x7fffffffu;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      int m = 0;
      for (int i = lane; i < count; i += 32) m += (buf[i].x == t && buf[i].y <= mid);
      if (static_cast<int>(__reduce_add_sync(~0u, static_cast<unsigned>(m))) >= want) hi = mid;
      else lo = mid + 1;
    }
    imax = lo;
  }
  int base = 0;
  for (int i0 = 0; i0 < count; i0 += 32) {   // in place: a kept entry never moves past its own 32-entry chunk
    const int i = i0 + lane;
    const uint2 e = i < count ? buf[i] : make_uint2(0u, 0u);
    const bool keep = i < count && (e.x > t || (e.x == t && e.y <= imax));
    const unsigned bal = __ballot_sync(~0u, keep);
    __syncwarp();
    if (keep) buf[base + __popc(bal & ((1u << lane) - 1u))] = e;
    base += __popc(bal);
    __syncwarp();
  }
  return key_score(t);
}

}  // namespace

// Stage-1 epilogue of the persistent GEMM (gemm_kernel.cuh).  Work items are (query m-block, corpus slice) pairs,
// m-block fastest, dealt to the CTAs in turn; a CTA sweeps its item's n-blocks in order.  Each query row (the quad of
// lanes that holds it) keeps a threshold tau = the k'-th best score of its slice so far and appends the scores above
// it to its buffer; a buffer that would overflow is compacted to its best k' first, which raises tau.
struct KnnEpi {
  static constexpr bool kSliced = true;
  static constexpr uint64_t kHintA = kEvictLast;    // the query block is read again for every tile of the slice
  static constexpr uint64_t kHintB = kEvictNormal;  // corpus tiles are shared by the CTAs of one slice, then done
  struct State {
    float tau[2];
    int cnt[2];
    int item1;   // item + 1 of the rows' current buffers (0: none yet)
  };
  uint2* cand;         // [nq][S][kKnnCap] {order_key(score), corpus row}
  int* cnt;            // [nq][S] entries left in each buffer (<= kp)
  const float2* col;   // [n_pad] per corpus row: euclidean (|x~|^2 / 2, -), cosine (c.x~, 1 / |x|)
  const float2* rowt;  // [m_pad] per query row: cosine (q~.c + |c|^2, -)
  int nq, n, S, nbs, kp, cosine, m_blocks, items;

  __device__ int num_tiles() const { return items * nbs; }
  __device__ int first_tile(int b) const { return b * nbs; }
  __device__ int next_tile(int t, int grid, int num_n_blocks) const {
    const int item = t / nbs, j = t - item * nbs;
    if (j + 1 < nbs && (item / m_blocks) * nbs + j + 1 < num_n_blocks) return t + 1;
    return (item + grid) * nbs;
  }
  __device__ void decode(int t, int num_m_blocks, int& m_blk, int& n_blk) const {
    const int item = t / nbs;
    m_blk = item % num_m_blocks;
    n_blk = (item / num_m_blocks) * nbs + (t - item * nbs);
  }

  __device__ uint2* buffer(int row, int slice) const {
    return cand + (static_cast<size_t>(row) * S + slice) * kKnnCap;
  }

  // compact every row of the warp (half hr) whose quad raised `need`; warp-uniform control flow
  __device__ void compact_rows(bool need, int hr, int row0, int slice, int lane, State& st) const {
    unsigned m = __ballot_sync(~0u, need && (lane & 3) == 0);
    while (m) {
      const int leader = __ffs(m) - 1;
      const int count = __shfl_sync(~0u, st.cnt[hr], leader);
      const float t = knn_compact(buffer(row0 + (leader >> 2) + 8 * hr, slice), count, kp, lane);
      if ((lane >> 2) == (leader >> 2)) {
        st.tau[hr] = t;
        st.cnt[hr] = kp;
      }
      m &= m - 1;
    }
  }

  __device__ void flush(int row0w, int lane, State& st) const {
    const int item = st.item1 - 1;
    const int m_blk = item % m_blocks, slice = item / m_blocks;
    const int row0 = m_blk * 128 + row0w;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      compact_rows(st.cnt[hr] > kp, hr, row0, slice, lane, st);
      const int row = row0 + (lane >> 2) + 8 * hr;
      if ((lane & 3) == 0 && row < nq) cnt[static_cast<size_t>(row) * S + slice] = st.cnt[hr];
    }
  }

  // d: this thread's accumulators of the 128 x 256 tile (wgmma m64n256 layout: rows row0w + lane/4 + 8 hr, columns
  // 8 jg + 2 (lane % 4) + e at d[4 jg + 2 hr + e]); row0w: the warp's first row inside the tile
  __device__ void tile(float (&d)[128], int m_blk, int n_blk, int row0w, int lane, State& st) const {
    const int q = lane & 3, g = lane >> 2;
    const int slice = n_blk / nbs;
    const int item = slice * m_blocks + m_blk;
    const int row0 = m_blk * 128 + row0w;
    if (st.item1 != item + 1) {
      if (st.item1 != 0) flush(row0w, lane, st);
      st.item1 = item + 1;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        st.tau[hr] = row0 + g + 8 * hr < nq ? -INFINITY : INFINITY;   // padding rows never append
        st.cnt[hr] = 0;
      }
    }
    // affine epilogue, in place: larger is nearer
    float ra[2] = {0.0f, 0.0f};
    if (cosine) {
      ra[0] = rowt[row0 + g].x;
      ra[1] = rowt[row0 + g + 8].x;
    }
    const int cbase = n_blk * 256 + 2 * q;
#pragma unroll
    for (int jg = 0; jg < 32; ++jg) {
      const int c = cbase + 8 * jg;
      const float4 t = __ldg(reinterpret_cast<const float4*>(col + c));   // rows c, c + 1 (col is padded to 256)
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float& v0 = d[4 * jg + 2 * hr];
        float& v1 = d[4 * jg + 2 * hr + 1];
        if (cosine) {
          v0 = ((v0 + ra[hr]) + t.x) * t.y;
          v1 = ((v1 + ra[hr]) + t.z) * t.w;
        } else {
          v0 = v0 - t.x;
          v1 = v1 - t.z;
        }
        if (c >= n) v0 = -INFINITY;
        if (c + 1 >= n) v1 = -INFINITY;
      }
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      int mine = 0, excl = 0, total = 0;
      auto count = [&]() {
        mine = 0;
#pragma unroll
        for (int jg = 0; jg < 32; ++jg)
          mine += (d[4 * jg + 2 * hr] > st.tau[hr]) + (d[4 * jg + 2 * hr + 1] > st.tau[hr]);
        int incl = mine, u = __shfl_up_sync(~0u, incl, 1, 4);
        if (q >= 1) incl += u;
        u = __shfl_up_sync(~0u, incl, 2, 4);
        if (q >= 2) incl += u;
        total = __shfl_sync(~0u, incl, 3, 4);
        excl = incl - mine;
      };
      count();
      const bool need = st.cnt[hr] + total > kKnnCap;
      if (__any_sync(~0u, need)) {
        compact_rows(need, hr, row0, slice, lane, st);
        count();
      }
      if (mine > 0) {
        uint2* b = buffer(row0 + g + 8 * hr, slice) + st.cnt[hr] + excl;
#pragma unroll
        for (int jg = 0; jg < 32; ++jg) {
          const int c = cbase + 8 * jg;
          const float v0 = d[4 * jg + 2 * hr], v1 = d[4 * jg + 2 * hr + 1];
          if (v0 > st.tau[hr]) *b++ = make_uint2(order_key(v0), static_cast<uint32_t>(c));
          if (v1 > st.tau[hr]) *b++ = make_uint2(order_key(v1), static_cast<uint32_t>(c + 1));
        }
      }
      st.cnt[hr] += total;
    }
  }

  __device__ void finish(int row0w, int lane, State& st) const {
    if (st.item1 != 0) flush(row0w, lane, st);
  }
};

namespace {

// column sums of rows [chunk * per, (chunk + 1) * per) in f64 -> partial[chunk][col]
__global__ void knn_center_partial_kernel(const float* __restrict__ x, long long n, int D, long long per,
                                          double* __restrict__ partial) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= D) return;
  const long long r0 = blockIdx.y * per, r1 = min(n, r0 + per);
  double s = 0.0;
  for (long long r = r0; r < r1; ++r) s += static_cast<double>(x[r * D + col]);
  partial[static_cast<size_t>(blockIdx.y) * D + col] = s;
}

// c[col] = f32(sum over chunks, in order, / n); columns [D, k_pad) = 0
__global__ void knn_center_finish_kernel(const double* __restrict__ partial, int chunks, long long n, int D, int k_pad,
                                         float* __restrict__ c) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= k_pad) return;
  double s = 0.0;
  if (col < D)
    for (int k = 0; k < chunks; ++k) s += partial[static_cast<size_t>(k) * D + col];
  c[col] = col < D ? static_cast<float>(s / static_cast<double>(n)) : 0.0f;
}

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(~0u, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < nw; ++i) s += red[i];   // same order in every thread
  return s;
}

// One CTA per destination row r < rows_pad: x~ = x - c (f64) -> dst row [bf16(x~) | bf16(x~ - hi)] over k_pad columns
// (zeros past D, and whole zero rows for r >= rows); terms[r] per `mode` (0 corpus euclidean, 1 corpus cosine,
// 2 query); a non-finite input raises bit 1 of *err, a row norm outside [kKnnNormMin, kKnnNormMax] (other than 0) bit 2.
__global__ void knn_prep_rows_kernel(const float* __restrict__ src, long long rows, int D, int k_pad,
                                     const float* __restrict__ center, double c2, int mode, __nv_bfloat16* __restrict__ dst,
                                     float2* __restrict__ terms, int* err) {
  __shared__ double red[3][32];
  const long long r = blockIdx.x;
  __nv_bfloat16* hi_row = dst + r * 2 * k_pad;
  __nv_bfloat16* lo_row = hi_row + k_pad;
  double sx2 = 0.0, st2 = 0.0, sc = 0.0;
  bool bad = false;
  for (int i = threadIdx.x; i < k_pad; i += blockDim.x) {
    __nv_bfloat16 h = __float2bfloat16_rn(0.0f), l = h;
    if (r < rows && i < D) {
      const float x = src[r * D + i];
      bad |= !isfinite(x);
      const double cc = static_cast<double>(center[i]);
      const double t = static_cast<double>(x) - cc;
      h = __float2bfloat16_rn(static_cast<float>(t));
      l = __float2bfloat16_rn(static_cast<float>(t - static_cast<double>(__bfloat162float(h))));
      sx2 += static_cast<double>(x) * x;
      st2 += t * t;
      sc += cc * t;
    }
    hi_row[i] = h;
    lo_row[i] = l;
  }
  if (bad) atomicOr(err, 1);
  sx2 = block_sum(sx2, red[0]);
  st2 = block_sum(st2, red[1]);
  sc = block_sum(sc, red[2]);
  if (threadIdx.x == 0) {
    float2 t = make_float2(0.0f, 0.0f);
    if (r < rows && sx2 > 0.0 && (sx2 < kKnnNormMin * kKnnNormMin || sx2 > kKnnNormMax * kKnnNormMax)) atomicOr(err, 2);
    if (r < rows) {
      if (mode == 0) t = make_float2(static_cast<float>(0.5 * st2), 0.0f);
      else if (mode == 1) t = make_float2(static_cast<float>(sc), sx2 > 0.0 ? static_cast<float>(1.0 / sqrt(sx2)) : 0.0f);
      else t = make_float2(static_cast<float>(sc + c2), 0.0f);
    }
    terms[r] = t;
  }
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(~0u, v, o);
  return v;
}
// |v|^2 of a D-vector by one warp: the same code for queries and corpus rows, so equal rows give equal norms
__device__ __forceinline__ double warp_norm2(const float* v, int D, int lane) {
  double s = 0.0;
  for (int i = lane; i < D; i += 32) s += static_cast<double>(v[i]) * v[i];
  return warp_sum(s);
}

// One CTA per query row: best kp of the S slices' candidates (bitonic sort of {key, ~index} in shared memory), then
// (unless dbg_score) exact f64 distances and the best k by (distance, index).
__global__ void knn_merge_rerank_kernel(const uint2* __restrict__ cand, const int* __restrict__ cnt, int S, int kp, int P,
                                        const float* __restrict__ Q, const float* __restrict__ X, int D, int cosine, int k,
                                        float* __restrict__ out_dist, int64_t* __restrict__ out_idx,
                                        float* __restrict__ dbg_score, int64_t* __restrict__ dbg_idx) {
  extern __shared__ __align__(16) uint8_t knn_smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(knn_smem);
  double* cd = reinterpret_cast<double*>(keys + P);
  long long* ci = reinterpret_cast<long long*>(cd + kp);
  __shared__ double qn2;
  const int row = blockIdx.x;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const int s = i / kp, j = i - s * kp;
    unsigned long long key = 0;
    if (s < S && j < cnt[static_cast<size_t>(row) * S + s]) {
      const uint2 e = cand[(static_cast<size_t>(row) * S + s) * kKnnCap + j];
      key = (static_cast<unsigned long long>(e.x) << 32) | static_cast<uint32_t>(~e.y);
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < P / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const bool desc = (lo & size) == 0;
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
      }
      __syncthreads();
    }
  }
  if (dbg_score != nullptr) {
    for (int j = threadIdx.x; j < kp; j += blockDim.x) {
      const unsigned long long key = keys[j];
      const bool ok = (key >> 32) != 0;
      dbg_score[static_cast<size_t>(row) * kp + j] = ok ? key_score(static_cast<uint32_t>(key >> 32)) : -INFINITY;
      dbg_idx[static_cast<size_t>(row) * kp + j] = ok ? static_cast<int64_t>(~static_cast<uint32_t>(key)) : -1;
    }
    return;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* q = Q + static_cast<size_t>(row) * D;
  if (warp == 0) {
    const double v = warp_norm2(q, D, lane);
    if (lane == 0) qn2 = v;
  }
  __syncthreads();
  if (cosine && qn2 == 0.0) {   // a zero query is at distance 1 from every row: the first k rows
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
      out_dist[static_cast<size_t>(row) * k + j] = 1.0f;
      out_idx[static_cast<size_t>(row) * k + j] = j;
    }
    return;
  }
  for (int j = warp; j < kp; j += nw) {
    const unsigned long long key = keys[j];
    double dist = INFINITY;
    long long idx = (1ll << 32) + j;   // empty slot: after every real row
    if ((key >> 32) != 0) {
      idx = static_cast<long long>(~static_cast<uint32_t>(key));
      const float* x = X + static_cast<size_t>(idx) * D;
      if (cosine) {
        const double xn2 = warp_norm2(x, D, lane);
        if (xn2 == 0.0) {
          dist = 1.0;
        } else {
          const double a = sqrt(qn2), b = sqrt(xn2);
          double s = 0.0;
          for (int i = lane; i < D; i += 32) {
            const double t = static_cast<double>(q[i]) / a - static_cast<double>(x[i]) / b;
            s += t * t;
          }
          dist = 0.5 * warp_sum(s);
        }
      } else {
        double s = 0.0;
        for (int i = lane; i < D; i += 32) {
          const double t = static_cast<double>(q[i]) - static_cast<double>(x[i]);
          s += t * t;
        }
        dist = sqrt(warp_sum(s));
      }
    }
    if (lane == 0) { cd[j] = dist; ci[j] = idx; }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kp; t += blockDim.x) {
    int rank = 0;
    for (int j = 0; j < kp; ++j) rank += (cd[j] < cd[t]) || (cd[j] == cd[t] && ci[j] < ci[t]);
    if (rank < k) {
      out_dist[static_cast<size_t>(row) * k + rank] = static_cast<float>(cd[t]);
      out_idx[static_cast<size_t>(row) * k + rank] = ci[t];
    }
  }
}

constexpr int kCenterChunks = 256;

}  // namespace

size_t knn_center_workspace(int D) { return static_cast<size_t>(kCenterChunks) * D * sizeof(double); }

cudaError_t launch_knn_center(const float* x, long long n, int D, int k_pad, double* partial, float* center,
                              cudaStream_t stream) {
  const long long per = (n + kCenterChunks - 1) / kCenterChunks;
  const int chunks = static_cast<int>((n + per - 1) / per);
  knn_center_partial_kernel<<<dim3((D + 127) / 128, chunks), 128, 0, stream>>>(x, n, D, per, partial);
  knn_center_finish_kernel<<<(k_pad + 127) / 128, 128, 0, stream>>>(partial, chunks, n, D, k_pad, center);
  return cudaGetLastError();
}

cudaError_t launch_knn_prep(const float* src, long long rows, long long rows_pad, int D, int k_pad, const float* center,
                            double c2, int mode, __nv_bfloat16* dst, float2* terms, int* err, cudaStream_t stream) {
  if (rows_pad < 1 || rows_pad > 0x7fffffffll) return cudaErrorInvalidValue;
  knn_prep_rows_kernel<<<static_cast<unsigned>(rows_pad), 256, 0, stream>>>(src, rows, D, k_pad, center, c2, mode, dst,
                                                                            terms, err);
  return cudaGetLastError();
}

void knn_plan(int nq, long long n, int kp, int num_sms, int* S, int* nbs) {
  const int m_blocks = (nq + 127) / 128;
  const long long n_blocks = (n + 255) / 256;
  long long s = std::max(1, num_sms / m_blocks);   // one wave of (m-block, slice) items
  s = std::min<long long>(s, n_blocks);
  s = std::min<long long>(s, kKnnMergeMax / kp);
  *nbs = static_cast<int>((n_blocks + s - 1) / s);
  *S = static_cast<int>((n_blocks + *nbs - 1) / *nbs);
}

cudaError_t launch_knn_stage1(const KnnStage1Args& a, cudaStream_t stream) {
  if (a.m_pad % 128 || a.k_pad % 64 || a.nq > a.m_pad) return cudaErrorInvalidValue;
  CUtensorMap tmA, tmB;
  cudaError_t e = make_tmap_bf16_2d(&tmA, a.qs, 2ull * a.k_pad, a.m_pad, 2ull * a.k_pad, kBlockK, kBlockM);
  if (e != cudaSuccess) return e;
  e = make_tmap_bf16_2d(&tmB, a.xs, 2ull * a.k_pad, static_cast<uint64_t>(a.n), 2ull * a.k_pad, kBlockK, kBlockN);
  if (e != cudaSuccess) return e;
  KnnEpi epi{};
  epi.cand = a.cand;
  epi.cnt = a.cnt;
  epi.col = a.col;
  epi.rowt = a.rowt;
  epi.nq = a.nq;
  epi.n = static_cast<int>(a.n);
  epi.S = a.S;
  epi.nbs = a.nbs;
  epi.kp = a.kp;
  epi.cosine = a.cosine;
  epi.m_blocks = a.m_pad / kBlockM;
  epi.items = epi.m_blocks * a.S;
  const int num_n_blocks = static_cast<int>((a.n + kBlockN - 1) / kBlockN);
  const int grid = std::min(epi.items, a.num_sms > 0 ? a.num_sms : 132);
  const size_t smem = 1024 + static_cast<size_t>(kGemmStages) * kGemmStageBytes + 2 * kGemmStages * 8 + 32;
  auto kfn = gemm_bf16_kernel<float, 0, false, KnnEpi>;
  e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  kfn<<<grid, kGemmThreads, smem, stream>>>(tmA, tmB, nullptr, nullptr, 0, 0, 0, epi.m_blocks, num_n_blocks,
                                            a.k_pad / kBlockK, 16, 3, a.k_pad, nullptr, kSpinLimitDefault, nullptr, epi);
  return cudaGetLastError();
}

cudaError_t launch_knn_merge_rerank(const uint2* cand, const int* cnt, int rows, int S, int kp, const float* Q,
                                    const float* X, int D, int cosine, int k, float* out_dist, int64_t* out_idx,
                                    float* dbg_score, int64_t* dbg_idx, cudaStream_t stream) {
  int P = 1;
  while (P < S * kp) P <<= 1;
  const size_t smem = static_cast<size_t>(P) * 8 + static_cast<size_t>(kp) * 16;
  auto kfn = knn_merge_rerank_kernel;
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  kfn<<<rows, 512, smem, stream>>>(cand, cnt, S, kp, P, Q, X, D, cosine, k, out_dist, out_idx, dbg_score, dbg_idx);
  return cudaGetLastError();
}

}  // namespace ie
