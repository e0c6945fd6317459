// Persistent wgmma GEMM:  D[M, N] = act(A[M, K] * B[N, K]^T + bias[N])
//
//   A, B : bf16, K-major (row-major with K contiguous), K padded to a multiple of 64 and physically
//          zero-filled, A rows padded to whole 128-row tiles; B rows past n_pad read as zeros (TMA out-of-bounds fill).
//   D    : f32, bf16 or fp16, row-major with leading dimension ldd.
//
// Used for (i) the hoisted LSTM input projections  Gx = X * W_ih^T + (b_ih + b_hh)  over all T*B rows at
// once (the non-recurrent 46 % of the encoder FLOPs; reference: fastai AWD_LSTM -> torch nn.LSTM called at
// Issue_Embeddings/flask_app/inference.py:57,68) and (ii) the Label_Microservice MLP layers
// (py/label_microservice/mlp.py:63 -> sklearn predict_proba).
//
// Structure (one CTA per SM, 384 threads, warp-specialised, tiles of 128 x 256):
//   warpgroup 0      TMA producer (one thread): A tile 128x64 and B tile 256x64 per stage, 128B swizzle, mbarrier complete_tx
//   warpgroups 1, 2  consumers: wgmma m64n256k16 into registers (64 rows each), then +bias -> activation -> global
//                    stores; the producer fills the next tile's stages meanwhile
#include "gemm_kernel.cuh"

namespace ie {


// Launch.  a: [m_pad rows, k_pad] bf16 (m_pad % 128 == 0, k_pad % 64 == 0); b: [n_pad rows, k_pad] bf16 with
// n_pad % bn == 0.  Writes D rows < m_store and columns < n_store (n_store % 16 == 0).
cudaError_t launch_gemm_bf16(const GemmArgs& g, cudaStream_t stream) {
  if (g.m_pad % kBlockM || g.k_pad % kBlockK || g.bn % 16 || g.bn < 16 || g.bn > 256 || g.n_pad % g.bn ||
      g.n_store % 16 || g.ldd % 2)
    return cudaErrorInvalidValue;
  CUtensorMap tmA, tmB;
  const int segs = g.segs == 3 ? 3 : 1;
  const uint64_t k_inner = static_cast<uint64_t>(segs == 3 ? 2 : 1) * g.k_pad;  // split-bf16 operands are [hi | lo]
  const long long spin_limit = g.spin_limit > 0 ? g.spin_limit : kSpinLimitDefault;
  cudaError_t e = make_tmap_bf16_2d(&tmA, g.a, k_inner, g.m_pad, g.lda, kBlockK, kBlockM);
  if (e != cudaSuccess) return e;
  e = make_tmap_bf16_2d(&tmB, g.b, k_inner, g.n_pad, g.ldb, kBlockK, kBlockN);
  if (e != cudaSuccess) return e;

  const size_t smem = 1024 + static_cast<size_t>(kGemmStages) * kGemmStageBytes + 2 * kGemmStages * 8 + 32;
  const int num_m_blocks = g.m_pad / kBlockM;
  const int num_n_blocks = (g.n_pad + kBlockN - 1) / kBlockN;
  const int num_k_blocks = g.k_pad / kBlockK;
  const int num_tiles = num_m_blocks * num_n_blocks;
  const int sms = g.num_sms > 0 ? g.num_sms : 132;
  const int grid = num_tiles < sms ? num_tiles : sms;
  // m-blocks per panel (tile order: m fastest inside a panel, then n): the CTAs running together share ~16 A blocks
  // (4 MB at K = 1024) and ~grid/16 B tiles, far inside the 50 MB L2 next to the output stream
  const int panel = 16;

#define IE_LAUNCH(OUT, ACT, FRAG)                                                                                  \
  do {                                                                                                             \
    auto kfn = gemm_bf16_kernel<OUT, ACT, FRAG>;                                                                       \
    e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));            \
    if (e != cudaSuccess) return e;                                                                                \
    kfn<<<grid, kGemmThreads, smem, stream>>>(tmA, tmB, reinterpret_cast<OUT*>(g.d), g.bias, g.m_store, g.n_store, \
                                              g.ldd, num_m_blocks, num_n_blocks, num_k_blocks, panel, segs,        \
                                              g.k_pad, g.abort_flag, spin_limit, g.diag, DenseEpi{});              \
  } while (0)

  if (g.frag) {
    // fragment order: whole 256-column tiles, a bias in the same order, 16-byte aligned rows
    if (g.act != 0 || g.out_bf16 == 1 || g.bias == nullptr || g.n_store % kBlockN || g.n_store != g.n_pad ||
        (g.ldd * (g.out_bf16 == 2 ? 2 : 4)) % 16)
      return cudaErrorInvalidValue;
    if (g.out_bf16 == 2) IE_LAUNCH(__half, 0, true);
    else IE_LAUNCH(float, 0, true);
  } else if (g.out_bf16 == 2) {
    if (g.act != 0) return cudaErrorInvalidValue;
    IE_LAUNCH(__half, 0, false);
  } else if (g.out_bf16) {
    if (g.act == 0) IE_LAUNCH(__nv_bfloat16, 0, false);
    else if (g.act == 1) IE_LAUNCH(__nv_bfloat16, 1, false);
    else IE_LAUNCH(__nv_bfloat16, 2, false);
  } else {
    if (g.act == 0) IE_LAUNCH(float, 0, false);
    else if (g.act == 1) IE_LAUNCH(float, 1, false);
    else IE_LAUNCH(float, 2, false);
  }
#undef IE_LAUNCH
  return cudaGetLastError();
}

}  // namespace ie
