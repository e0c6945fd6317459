// Per-label probability thresholds from the precision-recall curve, on the device.
//
// Replaces the inner loop of MLPWrapper.find_probability_thresholds (py/label_microservice/mlp.py:81-98):
//     precision, recall, threshold = precision_recall_curve(y_test[:, label], y_pred[:, label])
//     keep the point with the HIGHEST precision among those with precision >= precision_threshold and
//     recall >= recall_threshold (first such point in increasing-threshold order on ties; none -> label excluded)
// sklearn's curve (what the reference calls): thresholds = the distinct scores in increasing order; for threshold s,
// tp / fp count the samples with score >= s; precision = tp / (tp + fp), recall = tp / P (recall := 1 when the label has no
// positive sample).  All ratios in f64, like sklearn.
//
// One CTA per label: (score, truth) pairs of the label's column are packed into 64-bit keys in shared memory
// (order-preserving score encoding in the high word), bitonic-sorted descending, the truth bits are prefix-summed, and
// every position that ends a group of equal scores is a curve point.  n <= 16384 samples per call (128 KB of keys);
// larger hold-out sets stay on the host path.
//
// Input domain: finite scores.  -0.0 and +0.0 are one score (sklearn groups them, np.diff of the two is 0), so zero is
// canonicalised before encoding.  sklearn raises on NaN / inf; a device-pointer call cannot return an error, so a label
// with any non-finite score gets threshold, precision and recall NaN (an excluded label gets NaN / 0 / 0).  The host
// entry point rejects such scores before anything is launched.
#include "kernels.h"
#include "lstm_common.cuh"

namespace ie {

namespace {

constexpr int kPrThreads = 1024;

__global__ void __launch_bounds__(kPrThreads, 1)
pr_threshold_kernel(const float* __restrict__ scores, const uint8_t* __restrict__ truth, int n, int n_labels, int n_pow2,
                    double p_thr, double r_thr, float* __restrict__ out_thr, double* __restrict__ out_prec,
                    double* __restrict__ out_rec) {
  extern __shared__ unsigned long long keys[];   // [n_pow2]
  __shared__ int warp_sums[32];
  __shared__ double best_prec[32];
  __shared__ int best_idx[32];
  const int label = blockIdx.x;
  const int tid = threadIdx.x;
  int nonfinite = 0;
  for (int i = tid; i < n_pow2; i += kPrThreads) {
    unsigned long long k = 0ull;   // padding sorts to the end (real keys have the high word >= 1: enc_max(x) > 0 for finite x)
    if (i < n) {
      float s = scores[static_cast<long long>(i) * n_labels + label];
      nonfinite |= !isfinite(s);
      s = (s == 0.0f) ? 0.0f : s;   // -0.0 -> +0.0: one tie group, as in sklearn
      const unsigned t = truth[static_cast<long long>(i) * n_labels + label] ? 1u : 0u;
      k = (static_cast<unsigned long long>(enc_max(s)) << 32) | t;
    }
    keys[i] = k;
  }
  if (__syncthreads_or(nonfinite)) {   // uniform across the CTA
    if (tid == 0) {
      const float qnan = __int_as_float(0x7fc00000);
      out_thr[label] = qnan;
      out_prec[label] = static_cast<double>(qnan);
      out_rec[label] = static_cast<double>(qnan);
    }
    return;
  }
  // bitonic sort, descending
  for (int size = 2; size <= n_pow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < (n_pow2 >> 1); i += kPrThreads) {
        const int lo = 2 * i - (i & (stride - 1));   // index with bit `stride` cleared
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
      }
      __syncthreads();
    }
  }
  // inclusive prefix sum of the truth bits in sorted order: each thread owns a contiguous run
  const int per = n_pow2 / kPrThreads > 0 ? n_pow2 / kPrThreads : 1;
  const int i0 = tid * per;
  int local = 0;
  if (i0 < n_pow2)
    for (int i = i0; i < i0 + per && i < n_pow2; ++i) local += static_cast<int>(keys[i] & 1ull);
  int incl = local;
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += v;
    }
    warp_sums[lane] = w;   // inclusive over warps
  }
  __syncthreads();
  const int total_pos = warp_sums[31];
  int run = (incl - local) + (warp > 0 ? warp_sums[warp - 1] : 0);   // positives before this thread's run
  // curve points: positions that end a group of equal scores
  double bp = -1.0;
  int bi = -1;
  if (i0 < n) {
    for (int i = i0; i < i0 + per && i < n; ++i) {
      const unsigned long long k = keys[i];
      run += static_cast<int>(k & 1ull);
      const bool group_end = (i == n - 1) || ((keys[i + 1] >> 32) != (k >> 32));
      if (!group_end) continue;
      const double tp = static_cast<double>(run);
      const double prec = tp / static_cast<double>(i + 1);
      const double rec = total_pos > 0 ? tp / static_cast<double>(total_pos) : 1.0;
      if (prec >= p_thr && rec >= r_thr && prec > 0.0) {
        // highest precision; on ties the LOWEST threshold = the largest sorted index
        if (prec > bp || (prec == bp && i > bi)) { bp = prec; bi = i; }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double op = __shfl_down_sync(0xffffffffu, bp, o);
    const int oi = __shfl_down_sync(0xffffffffu, bi, o);
    if (op > bp || (op == bp && oi > bi)) { bp = op; bi = oi; }
  }
  if (lane == 0) { best_prec[warp] = bp; best_idx[warp] = bi; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kPrThreads / 32; ++w)
      if (best_prec[w] > bp || (best_prec[w] == bp && best_idx[w] > bi)) { bp = best_prec[w]; bi = best_idx[w]; }
    if (bi < 0) {
      out_thr[label] = __int_as_float(0x7fc00000);   // NaN: no qualifying point -> the label is never predicted
      out_prec[label] = 0.0;
      out_rec[label] = 0.0;
    } else {
      // recompute tp at bi: positives among sorted positions [0, bi]
      int tp = 0;
      for (int i = 0; i <= bi; ++i) tp += static_cast<int>(keys[i] & 1ull);
      out_thr[label] = dec_max(static_cast<uint32_t>(keys[bi] >> 32));
      out_prec[label] = bp;
      out_rec[label] = total_pos > 0 ? static_cast<double>(tp) / static_cast<double>(total_pos) : 1.0;
    }
  }
}

}  // namespace

cudaError_t launch_pr_thresholds(const float* scores, const uint8_t* truth, int n, int n_labels, double p_thr,
                                 double r_thr, float* out_thr, double* out_prec, double* out_rec, cudaStream_t stream) {
  if (n < 1 || n > kPrMaxSamples || n_labels < 1) return cudaErrorInvalidValue;
  int n_pow2 = kPrThreads;   // at least one element per thread keeps the scan simple
  while (n_pow2 < n) n_pow2 <<= 1;
  const size_t smem = static_cast<size_t>(n_pow2) * sizeof(unsigned long long);
  cudaError_t e = cudaFuncSetAttribute(pr_threshold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  pr_threshold_kernel<<<n_labels, kPrThreads, smem, stream>>>(scores, truth, n, n_labels, n_pow2, p_thr, r_thr, out_thr,
                                                              out_prec, out_rec);
  return cudaGetLastError();
}

}  // namespace ie
