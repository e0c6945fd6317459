// The persistent wgmma GEMM kernel (gemm.cu), shared by every translation unit that runs a product through it.
//
// The epilogue is a template parameter: DenseEpi (the default) stores D = act(A B^T + bias) as gemm.cu describes; an
// epilogue with kSliced = true (knn.cu) takes over the tile schedule and consumes each accumulator tile in registers
// instead of storing it.  The mainloop -- TMA producer, 4-stage ring, two consumer warpgroups, split-bf16 K loop -- is
// the same for both.
#pragma once
#include <cuda_fp16.h>
#include <type_traits>

#include "kernels.h"
#include "ptx.cuh"

namespace ie {

// default epilogue: dense store of the accumulator tile (no state, the strided tile schedule)
struct DenseEpi {
  static constexpr bool kSliced = false;
  static constexpr uint64_t kHintA = kEvictNormal;
  static constexpr uint64_t kHintB = kEvictLast;
  struct State {};
};

namespace {

__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  const __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

constexpr int kBlockM = 128;
constexpr int kBlockN = 256;
constexpr int kBlockK = 64;  // 64 bf16 = 128 B = one swizzle atom
constexpr int kGemmThreads = 384;
constexpr int kGemmStages = 4;
constexpr uint32_t kABytes = kBlockM * kBlockK * 2;
constexpr uint32_t kBBytes = kBlockN * kBlockK * 2;
constexpr uint32_t kGemmStageBytes = kABytes + kBBytes;

template <typename OutT, int ACT, bool FRAG, typename Epi = DenseEpi>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, OutT* __restrict__ D,
                 const float* __restrict__ bias, int m_store, int n_store, long long ldd, int num_m_blocks,
                 int num_n_blocks, int num_k_blocks, int panel, int segs, int k_pad, unsigned* abort_flag,
                 long long spin_limit, long long* diag, const __grid_constant__ Epi epi) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw & 1023u)) & 1023u);

  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kGemmStages * kGemmStageBytes);
  uint64_t* empty_bar = full_bar + kGemmStages;
  uint32_t* abort_s = reinterpret_cast<uint32_t*>(empty_bar + kGemmStages);
  const Abort ab{abort_s, abort_flag, spin_limit};
  const int nkt = num_k_blocks * segs;  // split-bf16: K loop over [A_hi | A_lo | A_hi] x [B_hi | B_hi | B_lo]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (diag != nullptr && blockIdx.x == 0) {  // SM clock of this launch = d(clock64) / d(globaltimer)
      unsigned long long g;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
      diag[0] = clock64();
      diag[1] = static_cast<long long>(g);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kGemmStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    *abort_s = 0;
    fence_barrier_init();
  }
  __syncthreads();

  int num_tiles = num_m_blocks * num_n_blocks;
  if constexpr (Epi::kSliced) num_tiles = epi.num_tiles();
  const int panel_tiles = panel * num_n_blocks;
  int first_tile = blockIdx.x;
  if constexpr (Epi::kSliced) first_tile = epi.first_tile(blockIdx.x);
  auto next_tile = [&](int tile) {
    if constexpr (Epi::kSliced) return epi.next_tile(tile, gridDim.x, num_n_blocks);
    else return tile + static_cast<int>(gridDim.x);
  };
  // tile -> (m_blk, n_blk): m fastest inside a panel of `panel` m-blocks, then n, then next panel, so that
  // the CTAs running together share B tiles and the A panel stays L2 resident across the n sweep.
  auto decode = [&](int tile, int& m_blk, int& n_blk) {
    if constexpr (Epi::kSliced) {
      epi.decode(tile, num_m_blocks, m_blk, n_blk);
      return;
    }
    const int p = tile / panel_tiles;
    const int r = tile - p * panel_tiles;
    const int m0 = p * panel;
    const int mcnt = min(panel, num_m_blocks - m0);
    n_blk = r / mcnt;
    m_blk = m0 + (r - n_blk * mcnt);
  };

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = first_tile; tile < num_tiles && !aborted(ab); tile = next_tile(tile)) {
        int m_blk, n_blk;
        decode(tile, m_blk, n_blk);
        for (int kb = 0; kb < nkt; ++kb) {
          const int seg = kb / num_k_blocks, r = kb - seg * num_k_blocks;
          mbar_wait(&empty_bar[stage], phase ^ 1, ab);
          uint8_t* sa = smem + static_cast<size_t>(stage) * kGemmStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], kGemmStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[stage], (seg == 1 ? k_pad : 0) + r * kBlockK, m_blk * kBlockM, Epi::kHintA);
          tma_load_2d(sa + kABytes, &tmB, &full_bar[stage], (seg == 2 ? k_pad : 0) + r * kBlockK, n_blk * kBlockN,
                      Epi::kHintB);
          if (++stage == kGemmStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    const int wg = (warp - 4) >> 2;
    const int q = lane & 3;
    const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const uint32_t smem_base = smem_u32(smem);
    const bool signal = (threadIdx.x & 127) == 0;
    int stage = 0;
    uint32_t phase = 0;
    float d[128];
    typename Epi::State st{};
    for (int tile = first_tile; tile < num_tiles; tile = next_tile(tile)) {
      int m_blk, n_blk;
      decode(tile, m_blk, n_blk);
      int prev = -1;
      for (int kb = 0; kb < nkt; ++kb) {
        mbar_wait(&full_bar[stage], phase, ab);
        const uint32_t sa = smem_base + stage * kGemmStageBytes;
        const uint64_t da = wgmma_desc_sw128(sa + wg * (kABytes / 2));
        const uint64_t db = wgmma_desc_sw128(sa + kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) wgmma_m64n256k16(d, da + 2 * k, db + 2 * k, (kb | k) != 0);
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (signal) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == kGemmStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      if (signal && prev >= 0) mbar_arrive(&empty_bar[prev]);
      if constexpr (Epi::kSliced) {
        epi.tile(d, m_blk, n_blk, wg * 64 + (warp & 3) * 16, lane, st);
        continue;
      }
      if constexpr (FRAG) {
        // fragment order (kernels.h frag_index): this thread's values of a row are one run of 64 (m-major, gates
        // i, f, g, o), stored as 16-byte chunks at position 4k + q of the row's tile; the bias is in the same order, as
        // f32 (one float4 per m), loaded once for both rows
        constexpr int kPer = 16 / static_cast<int>(sizeof(OutT));   // values per chunk: 8 fp16 or 4 f32
        const float4* bq = reinterpret_cast<const float4*>(bias) + n_blk * (kBlockN / 4) + q;
        OutT* drow[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr)
          drow[hr] = D + static_cast<long long>(m_blk * kBlockM + rbase + 8 * hr) * ldd + n_blk * kBlockN + q * kPer;
#pragma unroll
        for (int k = 0; k < 64 / kPer; ++k) {
          float4 b[kPer / 4];
#pragma unroll
          for (int i = 0; i < kPer / 4; ++i) b[i] = __ldg(bq + 4 * (k * (kPer / 4) + i));
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            if (m_blk * kBlockM + rbase + 8 * hr >= m_store) continue;
            float x[kPer];
#pragma unroll
            for (int i = 0; i < kPer / 4; ++i) {
              const int m = k * (kPer / 4) + i;
              x[4 * i + 0] = d[8 * m + 2 * hr] + b[i].x;
              x[4 * i + 1] = d[8 * m + 2 * hr + 1] + b[i].y;
              x[4 * i + 2] = d[8 * m + 4 + 2 * hr] + b[i].z;
              x[4 * i + 3] = d[8 * m + 4 + 2 * hr + 1] + b[i].w;
            }
            uint4 v;
            if constexpr (sizeof(OutT) == 4) {
              v = make_uint4(__float_as_uint(x[0]), __float_as_uint(x[1]), __float_as_uint(x[2]), __float_as_uint(x[3]));
            } else {
              v = make_uint4(pack_f16x2(x[0], x[1]), pack_f16x2(x[2], x[3]), pack_f16x2(x[4], x[5]), pack_f16x2(x[6], x[7]));
            }
            *reinterpret_cast<uint4*>(drow[hr] + 4 * k * kPer) = v;
          }
        }
        continue;
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int row = m_blk * kBlockM + rbase + 8 * hr;
        if (row >= m_store) continue;
        OutT* drow = D + static_cast<long long>(row) * ldd;
#pragma unroll
        for (int jg = 0; jg < kBlockN / 8; ++jg) {
          const int n = n_blk * kBlockN + 8 * jg + 2 * q;
          if (n < n_store) {
            float x0 = d[4 * jg + 2 * hr], x1 = d[4 * jg + 2 * hr + 1];
            if (bias != nullptr) {
              const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + n));
              x0 += b2.x;
              x1 += b2.y;
            }
            if (ACT == 1) { x0 = fmaxf(x0, 0.0f); x1 = fmaxf(x1, 0.0f); }
            if (ACT == 2) { x0 = sigmoid_acc(x0); x1 = sigmoid_acc(x1); }
            if constexpr (sizeof(OutT) == 4) {
              *reinterpret_cast<float2*>(drow + n) = make_float2(x0, x1);
            } else if constexpr (std::is_same<OutT, __half>::value) {
              *reinterpret_cast<uint32_t*>(drow + n) = pack_f16x2(x0, x1);
            } else {
              *reinterpret_cast<uint32_t*>(drow + n) = pack_bf16x2(x0, x1);
            }
          }
        }
      }
    }
    if constexpr (Epi::kSliced) epi.finish(wg * 64 + (warp & 3) * 16, lane, st);
  }

  __syncwarp();
  if (diag != nullptr && threadIdx.x == 128 && blockIdx.x == 0) {
    unsigned long long g;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
    diag[2] = clock64();
    diag[3] = static_cast<long long>(g);
  }
}

}  // namespace

}  // namespace ie
