// THE recurrent kernel: all timesteps of one LSTM layer (or of one time chunk of it) for up to kMaxBatches independent
// batches of 256 rows in one persistent launch -- or, as the per-timestep fallback, one timestep per launch with the
// same code.  Reference call sites of the arithmetic: Issue_Embeddings/flask_app/inference.py:56-57, :66-68 (reset +
// forward), pooling :239.
//
//     z_t = Gx[t] + h_{t-1} W_hh^T ; i,f,o = sigmoid ; g = tanh ; c_t = f c_{t-1} + i g ; h_t = o tanh(c_t)
//
// Work decomposition ("rotating schedule"):
//   * an ITEM is 128 batch rows x one column tile of 256 accumulator columns = 64 hidden units x (i,f,g,o).  Weight rows
//     are pre-permuted (api_encoder.cu slice_perm) so that the wgmma fragment of a thread holds all four gates of a unit: inside
//     16-column chunk m = 4s + e, columns 2q, 2q+1 are (i, f) and 8+2q, 9+2q are (g, o) of unit 16s + 4q + e -- the cell
//     update needs no cross-thread traffic, and a thread's units come in runs of four (16-byte c, 8-byte h accesses);
//     Gx is stored in the matching fragment order (kernels.h frag_index): 16-byte loads;
//   * the items  n = t * C + g * 2 tiles + half * tiles + j  (C = ng * 2 tiles; timestep t, batch g, row half, column
//     tile j) are dealt round-robin in that global order over the P resident CTAs: CTA p runs items p, p + P, ...  Item n
//     needs h_{t-1} of batch g, i.e. items of step t-1 with smaller indices; every CTA walks its items in increasing
//     order, so the item with the globally smallest index can always run: no wait cycle for any P, C, T;
//   * per item: K/64 k-blocks of h and W_hh (TMA, 128B swizzle) through ONE 4-stage ring -- two producer threads fill the
//     halves of a stage independently (weights do not depend on the step, so their producer runs ahead of the h
//     dependency) -> two consumer warpgroups (64 rows each) issue 4 x wgmma m64n256k16 per k-block into registers and
//     then run the epilogue (+ Gx, gates, c_t, h_t as bf16 into slot t+1 of the hidden-state ring = next step's A operand
//     and the next layer's GEMM input) -> gpu-scope fence + red.add on the (step, batch) counter;
//   * the cell state moves between SMs from step to step: it lives in global memory (L2), read with ld.global.cg after
//     the CTA has seen the (t-1, g) counter; on the last layer the running max of the concat-pool travels the same way
//     and the pooled sum is an L2 reduction (lstm_common.cuh);
//   * the LAST layer runs the FUSE instantiation: its input projection x_t W_ih^T (k-blocks that depend on no step counter)
//     is accumulated in front of the recurrent k-blocks of every item instead of by a hoisted GEMM (see FUSE);
//   * split-bf16 ("fp32-accurate") mode: segs = 3 runs the K loop over [h_hi | h_lo | h_hi] x [W_hi | W_hi | W_lo]
//     (hi = bf16(x), lo = bf16(x - hi); the dropped lo*lo term is 2^-18 relative) -- same kernel, three times the MMAs.
//
// All CTAs of a persistent launch must be co-resident: the launch is cooperative (cudaLaunchAttributeCooperative), so it
// either gets the whole grid resident or fails; a wait that still exceeds its limit raises the abort protocol of ptx.cuh.
#include <cmath>

#include <cuda_fp16.h>

#include "kernels.h"
#include "lstm_common.cuh"
#include "ptx.cuh"

namespace ie {

namespace {

constexpr int kLThreads = 384;          // warpgroup 0: producers + counter watcher; warpgroups 1, 2: MMA + epilogue
constexpr int kLStages = 4;             // operand ring: 4 stages x (h k-block 16 KB + W k-block 32 KB)
constexpr int kLTileN = 256;            // accumulator columns per item = 64 hidden units
constexpr int kLRows = 128;             // batch rows per item
constexpr uint32_t kHBytes = kLRows * 64 * 2;
constexpr uint32_t kWBytes = kLTileN * 64 * 2;
constexpr uint32_t kStageBytes = kHBytes + kWBytes;
// k-blocks before the end of an item's MMAs at which each consumer thread loads its epilogue inputs into registers
// (c_{t-1}, one row of fp16 Gx, the pooled layer's running max) and prefetches the rest of its Gx lines into L2
constexpr int kEarlyLoadAhead = 8;
// setmaxnreg budgets: the launch gives every thread 168 (65 536 / 384, rounded down to a multiple of 8); warpgroup 0
// keeps 40, the two consumer warpgroups take the difference: 128 x 40 + 256 x 232 = 64 512 = 384 x 168
constexpr uint32_t kProducerRegs = 40;
constexpr uint32_t kConsumerRegs = 232;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 384 * 168, "setmaxnreg budgets exceed the launch's registers");

__device__ __forceinline__ void st_release_cta(uint32_t* p, uint32_t v) {
  asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_cta(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
  return v;
}
// bounded, backed-off spin of one lane until the shared sequence number reaches `target`
__device__ __forceinline__ void wait_seq_ge(const uint32_t* p, uint32_t target, const Abort& ab) {
  if (ld_acquire_cta(p) >= target) return;
  if (aborted(ab)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (ld_acquire_cta(p) < target) {
    __nanosleep(64);
    if (((++spins) & 0x3Fu) == 0 && abort_poll(ab, t0)) return;
  }
}

struct KArgs {
  const void* gx;        // f16 or f32 [rows, 4*out_pad] in fragment order; row = t_local*b_pad + brow, or the token id (TOK)
  const int* tok;        // TOK: time-major token ids of the whole call, index (t0 + t)*b_pad + brow
  const float* bias;     // FUSE: b_ih + b_hh, permuted, in fragment order (takes the place of Gx)
  float* cstate;         // [b_pad, out_pad]
  __nv_bfloat16* y;      // ring [(T+1)*b_pad, ldy] of this time chunk: slot 0 = h before the chunk, slot t+1 = h_t
  float* raw;            // optional [raw_rows, T_total, raw_ld]: rows brow < raw_rows only
  float* pool_sum;       // optional (last layer)
  float* pool_max;
  float* pool_last;
  const int* lengths;
  unsigned* step_done;   // [T*ng] zero-initialised (step, batch) counters (nullptr: one timestep per launch)
  unsigned* abort_flag;
  long long spin_limit;
  long long ldy, raw_ld;
  long long* trace;
  long long* diag;
  int T, t_begin, t0, T_total, ng, tiles, out_pad, nkb, segs, kh_pad, trace_items, fault, raw_rows;
  int pre_nkb;           // FUSE: k-blocks of the input projection that precede the recurrent ones in every item
  int carry_c;           // 1: global step 0 reads c_{-1} from cstate (a carried state) instead of zero
};

// TOK: Gx rows are rows of the per-token input-projection table; GXBF: Gx / table stored as fp16 (f32 otherwise);
// POOL: last layer -- the masked concat-pool accumulators ride the epilogue;
// MC: clusters of TWO CTAs that always hold items n, n+1 (n even) = the same (timestep, batch, row half) and adjacent
//     column tiles (tiles, C and P even), i.e. they need the SAME h tile: each CTA loads half of it and multicasts it
//     to both, so an h tile leaves the L2 once per two items.  A stage is refilled only when the consumers of BOTH CTAs
//     have released it (empty barriers count four arrivals).
// FUSE: the layer's input projection rides the recurrent K loop instead of a hoisted GEMM + Gx round trip: every item
//     first accumulates x_t W_ih^T -- pre_nkb k-blocks whose A operand is slot t+1 of the PREVIOUS layer's ring (tm_x)
//     and whose B operand is the W_ih part of the concatenated weights [W_ih | W_hh] (tm_w) -- and then, once the
//     (t-1, g) counter has been seen, the nkb k-blocks of h_{t-1} W_hh^T into the same accumulator; the epilogue adds
//     the bias (f32) where the other instantiations add Gx.  Used for the narrow last layer, whose few items per
//     timestep leave most CTAs waiting on the step chain: the independent W_ih k-blocks run inside that wait.  The sum
//     W_ih x + W_hh h + b stays in f32 (no fp16 rounding of Gx), so the fused layer is slightly MORE accurate than the
//     hoisted form, but its bits differ from the hoisted form's (tests compare those two with IE_FUSE_LAST=0).
template <bool TOK, bool GXBF, bool POOL, bool MC, bool FUSE, int GM>
__device__ __forceinline__ void lstm_layer_body(const CUtensorMap& tm_h, const CUtensorMap& tm_w,
                                                const CUtensorMap& tm_h64, const CUtensorMap& tm_x, const KArgs& a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t rawaddr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (rawaddr & 1023u)) & 1023u);

  uint8_t* ring = smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + kLStages * kStageBytes);  // [kLStages] 2 arrivals + bytes
  uint64_t* empty = full + kLStages;                                             // [kLStages] consumer releases
  uint32_t* cready = reinterpret_cast<uint32_t*>(empty + kLStages);  // items whose (t-1, g) counter the watcher has seen
  uint32_t* abort_s = cready + 1;
  const Abort ab{abort_s, a.abort_flag, a.spin_limit};

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  long long* const trace = a.trace;
  // optional timeline of the CTA's first `trace_items` items: [cta][k][12] (%globaltimer ns)
#define IE_TRACE(slot, kk) do { if (trace && (kk) < a.trace_items) { unsigned long long _g; \
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_g)); \
    trace[(static_cast<long long>(blockIdx.x) * a.trace_items + (kk)) * 12 + (slot)] = static_cast<long long>(_g); } } while (0)
  const uint32_t crank = MC ? cluster_ctarank() : 0u;
  const int P = static_cast<int>(gridDim.x);
  const int tiles = a.tiles, ng = a.ng;
  const int per_batch = 2 * tiles;                 // items of one (step, batch)
  const int C = ng * per_batch;
  const long long total = static_cast<long long>(a.T) * C;
  const int b_pad = 256 * ng;
  const int nkt = a.nkb * a.segs;                  // recurrent k-blocks per item
  const int pre = FUSE ? a.pre_nkb : 0;            // input-projection k-blocks per item (before them)
  auto decode = [&](long long n, int& t, int& g, int& half, int& j) {
    const long long s = n / C;
    const int c = static_cast<int>(n - s * C);
    t = a.t_begin + static_cast<int>(s);
    g = c / per_batch;
    const int r = c - g * per_batch;
    half = r / tiles;
    j = r - half * tiles;
  };

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_h);
    tma_prefetch_desc(&tm_w);
    if (MC) tma_prefetch_desc(&tm_h64);
    if (FUSE) tma_prefetch_desc(&tm_x);
    if (a.diag != nullptr && blockIdx.x == 0) {  // SM clock of this launch = d(clock64) / d(globaltimer)
      unsigned long long g;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
      a.diag[0] = clock64();
      a.diag[1] = static_cast<long long>(g);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kLStages; ++s) {
      mbar_init(&full[s], 2);
      mbar_init(&empty[s], MC ? 4 : 2);
    }
    *cready = 0;
    *abort_s = 0;
    fence_barrier_init();
  }
  if (MC) cluster_sync();
  else __syncthreads();

  if (warp < 4) {
    // warpgroup 0 is three single-lane loops and an idle warp: all 128 threads hand their registers to the consumers
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      // ---------------- h producer ------------------------------------------------------------------------------
      int stage = 0;
      uint32_t phase = 0;
      int k = 0;
      for (long long n = blockIdx.x; n < total && !aborted(ab); n += P, ++k) {
        int t, g, half, j;
        decode(n, t, g, half, j);
        const int row0 = t * b_pad + g * 256 + half * kLRows;   // ring slot t = h_{t-1} (chunk-local)
        if constexpr (FUSE) {
          // x_t = slot t+1 of the previous layer's ring (complete before this launch): no dependency on the step counters
          for (int kb = 0; kb < pre; ++kb) {
            mbar_wait(&empty[stage], phase ^ 1, ab);
            mbar_arrive_expect_tx(&full[stage], kHBytes);
            tma_load_2d(ring + stage * kStageBytes, &tm_x, &full[stage], kb * 64, row0 + b_pad, kEvictNormal);
            if (++stage == kLStages) { stage = 0; phase ^= 1; }
          }
        }
        wait_seq_ge(cready, static_cast<uint32_t>(k + 1), ab);  // the watcher (warp 2) has seen counter (t-1, g)
        if (t > a.t_begin) fence_proxy_async();  // h_{t-1} was written through the generic proxy, TMA reads it
        IE_TRACE(0, k);
        for (int kb = 0; kb < nkt; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1, ab);
          mbar_arrive_expect_tx(&full[stage], kHBytes);
          const int seg = kb / a.nkb, r = kb - seg * a.nkb;            // split-bf16: [h_hi | h_lo | h_hi]
          const int kc = (seg == 1 ? a.kh_pad : 0) + r * 64;
          if constexpr (MC) {
            // this CTA's half of the rows, to the same offset in both CTAs of the cluster
            tma_load_2d_mc(ring + stage * kStageBytes + crank * (kHBytes / 2), &tm_h64, &full[stage], kc,
                           row0 + static_cast<int>(crank) * (kLRows / 2), static_cast<uint16_t>(0x3), kEvictNormal);
          } else {
            tma_load_2d(ring + stage * kStageBytes, &tm_h, &full[stage], kc, row0, kEvictNormal);
          }
          if (++stage == kLStages) { stage = 0; phase ^= 1; }
        }
        IE_TRACE(1, k);
      }
    } else if (warp == 1 && lane == 0) {
      // ---------------- W producer: free-running ahead of h ----------------------------------------------------
      int stage = 0;
      uint32_t phase = 0;
      for (long long n = blockIdx.x; n < total && !aborted(ab); n += P) {
        int t, g, half, j;
        decode(n, t, g, half, j);
        for (int kb = 0; kb < pre + nkt; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1, ab);
          mbar_arrive_expect_tx(&full[stage], kWBytes);
          const int seg = FUSE ? 0 : kb / a.nkb, r = kb - seg * a.nkb;  // split-bf16: [W_hi | W_hi | W_lo]; FUSE: [W_ih | W_hh]
          tma_load_2d(ring + stage * kStageBytes + kHBytes, &tm_w, &full[stage], (seg == 2 ? a.kh_pad : 0) + r * 64,
                      j * kLTileN, kEvictLast);
          if (++stage == kLStages) { stage = 0; phase ^= 1; }
        }
      }
    } else if (warp == 2 && lane == 0) {
      // ---------------- counter watcher: runs ahead of the h producer and the epilogue ----------------------------
      int k = 0;
      for (long long n = blockIdx.x; n < total && !aborted(ab); n += P, ++k) {
        int t, g, half, j;
        decode(n, t, g, half, j);
        if (t > a.t_begin)   // ends with a gpu-scope fence
          wait_flag_ge_relaxed(a.step_done + (t - a.t_begin - 1) * ng + g, static_cast<unsigned>(per_batch), ab);
        st_release_cta(cready, static_cast<uint32_t>(k + 1));
      }
    }
  } else {
    // ---------------- consumers: MMA + epilogue (never leave their loop early: named barriers inside; in drain mode
    //                  their waits return at once and they run through the remaining items) ------------------------
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp - 4) >> 2;              // which 64 rows of the item
    const int q = lane & 3;
    const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const long long lo_off = a.segs > 1 ? a.kh_pad : 0;
    const uint32_t ring_base = smem_u32(ring);
    const bool signal = (threadIdx.x & 127) == 0;
    int stage = 0;
    uint32_t phase = 0;
    int k = 0;
    float d[128];
    for (long long n = blockIdx.x; n < total; n += P, ++k) {
      int t, g, half, j;
      decode(n, t, g, half, j);
      const int tg = a.t0 + t;  // global timestep
      const int brow0 = g * 256 + half * kLRows + rbase;   // this thread's rows: brow0 + 8 hr, hr = 0, 1
      const int unit0 = j * 64 + 4 * q;                    // + 16 s: this thread's units of group s are unit0 + 16 s + 0..3
      // Gx row of each of the two rows; TOK: a row of the per-token projection table, the token id loaded here at the
      // item's start (its latency passes under the MMAs instead of stalling their issue at the early-load point)
      long long grow[2];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr)
        grow[hr] = TOK ? static_cast<long long>(__ldg(a.tok + static_cast<long long>(tg) * b_pad + brow0 + 8 * hr))
                       : static_cast<long long>(t) * b_pad + brow0 + 8 * hr;
      // epilogue inputs loaded during the last MMAs (see kEarlyLoadAhead); c of both rows, pooled max (FUSE + POOL),
      // fp16 Gx of row hr = 0 in gv (row hr = 1 is loaded into gv by the epilogue once row 0 is done)
      float4 cv[2][4], mv[2][4];
      uint4 gv[4][2];
      int prev = -1;
      const int kb_early = max(pre + nkt - kEarlyLoadAhead, pre);
      for (int kb = 0; kb < pre + nkt; ++kb) {
        mbar_wait(&full[stage], phase, ab);
        if (kb == pre && signal && wg == 0) IE_TRACE(2, k);          // first h_{t-1} stage landed
        const uint32_t sa = ring_base + stage * kStageBytes;
        const uint64_t da = wgmma_desc_sw128(sa + wg * (kHBytes / 2));
        const uint64_t db = wgmma_desc_sw128(sa + kHBytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_m64n256k16(d, da + 2 * kk, db + 2 * kk, (kb | kk) != 0);
        wgmma_commit();
        if (kb == kb_early) {
          // While the last k-blocks are on the tensor cores, load what the epilogue reads into registers (other than
          // the accumulators), so that the epilogue is gate math and stores instead of a chain of L2 / HBM round
          // trips.  Not earlier: Gx is streamed once from HBM, and lines held in L2 through the whole MMA phase
          // compete with the weight k-blocks.
          // c_{t-1} (and the running max) of this chain was written by another CTA: read it only after (t-1, g) has
          // been seen here.  Already true: the h producer waited for the same count before loading the h stages
          // these MMAs read.  In drain mode the loads may return stale values; the addresses stay in range.
          if (lane == 0) wait_seq_ge(cready, static_cast<uint32_t>(k + 1), ab);
          __syncwarp();
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const long long co = static_cast<long long>(brow0 + 8 * hr) * a.out_pad + unit0;
#pragma unroll
            for (int s = 0; s < 4; ++s) {
              cv[hr][s] = (tg == 0 && !a.carry_c) ? make_float4(0.0f, 0.0f, 0.0f, 0.0f)
                                    : __ldcg(reinterpret_cast<const float4*>(a.cstate + co + 16 * s));
              if constexpr (FUSE && POOL)
                mv[hr][s] = (tg == 0) ? make_float4(0.0f, 0.0f, 0.0f, 0.0f)
                                      : __ldcg(reinterpret_cast<const float4*>(a.pool_max + co + 16 * s));
            }
          }
          // Gx lines (fragment order, kernels.h frag_index): fp16 -- row 0 into registers, 16-byte chunk k of the
          // thread's run at chunk position 4k + q; row 1 prefetched into L2, lane q of a quad taking line q of the
          // row's 4 lines of 128 B.  f32 -- both rows prefetched, 8 lines per row.
          if constexpr (!FUSE) {
            const long long gtile0 = grow[0] * (4ll * a.out_pad) + j * kLTileN;
            const long long gtile1 = grow[1] * (4ll * a.out_pad) + j * kLTileN;
            if constexpr (GXBF) {
              const uint4* gp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(a.gx) + gtile0) + q;
#pragma unroll
              for (int s = 0; s < 4; ++s)
#pragma unroll
                for (int i = 0; i < 2; ++i) gv[s][i] = __ldcs(gp + 4 * (2 * s + i));
              prefetch_l2(reinterpret_cast<const __half*>(a.gx) + gtile1 + 64 * q);
            } else {
              const float* gf = reinterpret_cast<const float*>(a.gx);
              prefetch_l2(gf + gtile0 + 32 * q);
              prefetch_l2(gf + gtile0 + 32 * q + 128);
              prefetch_l2(gf + gtile1 + 32 * q);
              prefetch_l2(gf + gtile1 + 32 * q + 128);
            }
          }
        }
        if (prev >= 0) {
          wgmma_wait<1>();
          if (signal) {
            mbar_arrive(&empty[prev]);
            if (MC) mbar_arrive_remote(&empty[prev], crank ^ 1u);
          }
        }
        prev = stage;
        if (++stage == kLStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      if (signal && prev >= 0) {
        mbar_arrive(&empty[prev]);
        if (MC) mbar_arrive_remote(&empty[prev], crank ^ 1u);
      }
      if (signal && wg == 0) IE_TRACE(3, k);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int brow = brow0 + 8 * hr;
        const int len = POOL ? a.lengths[brow] : 1;
        float* cp = a.cstate + static_cast<long long>(brow) * a.out_pad + unit0;
        __nv_bfloat16* yrow = a.y + (static_cast<long long>(t + 1) * b_pad + brow) * a.ldy + unit0;
        const long long po = static_cast<long long>(brow) * a.out_pad + unit0;
        // this thread's run of 64 Gx values (or bias values) in the row's fragment-ordered tile: 16-byte chunk k at
        // chunk position 4k + q (kernels.h frag_index)
        const long long gtile = grow[hr] * (4ll * a.out_pad) + j * kLTileN;
        // fp16 Gx of row 1: all eight chunks issued before any of the row's stores (the compiler cannot move a load
        // above a store it may alias), into the registers row 0's Gx has left; L2 hits after the prefetch
        if constexpr (GXBF && !FUSE) {
          if (hr == 1) {
            const uint4* gp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(a.gx) + gtile) + q;
#pragma unroll
            for (int s = 0; s < 4; ++s)
#pragma unroll
              for (int i = 0; i < 2; ++i) gv[s][i] = __ldcs(gp + 4 * (2 * s + i));
          }
        }
        // FUSE: the bias tile in the same order; the empty asm makes its address opaque per row, so that the compiler
        // does not hoist the row-invariant bias loads out of the row loop (64 values held across it would spill)
        const float* btile = FUSE ? a.bias + j * kLTileN : nullptr;
        if constexpr (FUSE) asm volatile("" : "+l"(btile));
        // the 16 units run in groups of four (one 16-byte c access, one 8-byte h store each)
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          // accumulator chunk m = 4s + e holds unit 16s + 4q + e: (i, f) at d[8m + 2hr (+1)], (g, o) at d[8m + 4 + 2hr (+1)]
          // Gx of the group's units e = 0..3, as loaded: fp16 -- two chunks of (i, f, g, o) x 2 units, widened only
          // where they are added; f32 Gx and the bias (FUSE) -- one chunk of (i, f, g, o) per unit, loaded next to its
          // use
          const float4 cprev = cv[hr][s];
          const float cp4[4] = {cprev.x, cprev.y, cprev.z, cprev.w};
          float cn[4], hn[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int m = 4 * s + e;
            float4 gx;
            if constexpr (FUSE) {
              gx = __ldg(reinterpret_cast<const float4*>(btile) + q + 4 * m);
            } else if constexpr (GXBF) {
              const uint4* gh = gv[s];
              const uint32_t w0 = (e & 1) ? gh[e >> 1].z : gh[e >> 1].x, w1 = (e & 1) ? gh[e >> 1].w : gh[e >> 1].y;
              const float2 f01 = __half22float2(*reinterpret_cast<const __half2*>(&w0));
              const float2 f23 = __half22float2(*reinterpret_cast<const __half2*>(&w1));
              gx = make_float4(f01.x, f01.y, f23.x, f23.y);
            } else {
              gx = __ldcs(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.gx) + gtile) + q + 4 * m);
            }
            const float zi = d[8 * m + 2 * hr] + gx.x;
            const float zf = d[8 * m + 2 * hr + 1] + gx.y;
            const float zg = d[8 * m + 4 + 2 * hr] + gx.z;
            const float zo = d[8 * m + 4 + 2 * hr + 1] + gx.w;
            lstm_cell1<GM>(zi, zf, zg, zo, cp4[e], cn[e], hn[e]);
          }
          const float4 h4 = make_float4(hn[0], hn[1], hn[2], hn[3]);
          __stcg(reinterpret_cast<float4*>(cp + 16 * s), make_float4(cn[0], cn[1], cn[2], cn[3]));
          store_h4(yrow + 16 * s, h4, lo_off);
          if (a.raw != nullptr && brow < a.raw_rows)
            *reinterpret_cast<float4*>(a.raw + (static_cast<long long>(brow) * a.T_total + tg) * a.raw_ld + unit0 + 16 * s) = h4;
          if constexpr (POOL)
            pool_accumulate4(a.pool_sum, a.pool_max, a.pool_last, po + 16 * s, h4, tg, len, FUSE ? &mv[hr][s] : nullptr);
        }
      }
      // publish (step t, batch g): h_t / c_t / pooling state visible
      named_bar_sync(1, 256);
      if (threadIdx.x == 128) {
        __threadfence();
        // fault injection for the abort-protocol test (IE_DEBUG_FAULT): item (t=1, g=0, first tile) is never published
        if (a.step_done != nullptr && !(a.fault && n == C))
          red_relaxed_add(a.step_done + (t - a.t_begin) * ng + g, 1u);
        IE_TRACE(6, k);
      }
    }
  }

  __syncwarp();
  if (MC) cluster_sync();   // no CTA leaves while its sibling may still multicast into it or arrive on its barriers
  if (a.diag != nullptr && threadIdx.x == 0 && blockIdx.x == 0) {
    unsigned long long g;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
    a.diag[2] = clock64();
    a.diag[3] = static_cast<long long>(g);
  }
#undef IE_TRACE
}

thread_local int g_last_max_ctas = 0;   // result of the last check_only query on this thread

template <bool TOK, bool GXBF, bool POOL, int GM>
__global__ void __launch_bounds__(kLThreads, 1)
lstm_layer_kernel(const __grid_constant__ CUtensorMap tm_h, const __grid_constant__ CUtensorMap tm_w,
                  const __grid_constant__ CUtensorMap tm_h64, const __grid_constant__ CUtensorMap tm_x,
                  const __grid_constant__ KArgs a) {
  lstm_layer_body<TOK, GXBF, POOL, false, false, GM>(tm_h, tm_w, tm_h64, tm_x, a);
}

// input projection fused into the K loop (the last layer by default; see FUSE above)
template <bool POOL, int GM>
__global__ void __launch_bounds__(kLThreads, 1)
lstm_layer_fused_kernel(const __grid_constant__ CUtensorMap tm_h, const __grid_constant__ CUtensorMap tm_w,
                        const __grid_constant__ CUtensorMap tm_h64, const __grid_constant__ CUtensorMap tm_x,
                        const __grid_constant__ KArgs a) {
  lstm_layer_body<false, true, POOL, false, true, GM>(tm_h, tm_w, tm_h64, tm_x, a);
}

template <bool TOK, int GM>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kLThreads, 1)
lstm_layer_mc_kernel(const __grid_constant__ CUtensorMap tm_h, const __grid_constant__ CUtensorMap tm_w,
                     const __grid_constant__ CUtensorMap tm_h64, const __grid_constant__ CUtensorMap tm_x,
                     const __grid_constant__ KArgs a) {
  lstm_layer_body<TOK, true, false, true, false, GM>(tm_h, tm_w, tm_h64, tm_x, a);
}

size_t layer_smem_bytes() { return 1024 + static_cast<size_t>(kLStages) * kStageBytes + 2 * kLStages * 8 + 32; }

template <int GM, bool TOK, bool GXBF, bool POOL, bool MC, bool FUSE = false>
cudaError_t launch_layer_t(const LstmLayerArgs& a, int ctas, int tiles, cudaStream_t stream) {
  void (*kfn)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, KArgs);
  if constexpr (MC) kfn = lstm_layer_mc_kernel<TOK, GM>;
  else if constexpr (FUSE) kfn = lstm_layer_fused_kernel<POOL, GM>;
  else kfn = lstm_layer_kernel<TOK, GXBF, POOL, GM>;
  const size_t smem = layer_smem_bytes();
  // function attributes are per device: set on every launch (cheap), never cached in a process-wide flag
  cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  if (a.check_only) {
    // how many CTAs can be co-resident (the caller reads lstm_layer_max_ctas())
    int max_ctas = 0;
    if (MC) {
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3(2 * (a.num_sms / 2));
      cfg.blockDim = dim3(kLThreads);
      cfg.dynamicSmemBytes = smem;
      cfg.stream = stream;
      int clusters = 0;
      e = cudaOccupancyMaxActiveClusters(&clusters, kfn, &cfg);
      max_ctas = 2 * clusters;
    } else {
      int per_sm = 0;
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kfn, kLThreads, smem);
      max_ctas = per_sm * a.num_sms;
    }
    if (e != cudaSuccess) return e;
    g_last_max_ctas = max_ctas;
    if (MC) return max_ctas >= 2 ? cudaSuccess : cudaErrorCooperativeLaunchTooLarge;
    return max_ctas >= a.num_sms ? cudaSuccess : cudaErrorCooperativeLaunchTooLarge;
  }
  KArgs k{};
  k.gx = a.gx; k.tok = a.tok; k.bias = a.bias; k.pre_nkb = FUSE ? a.pre_nkb : 0; k.cstate = a.c; k.y = a.y; k.raw = a.raw;
  k.raw_rows = a.raw_rows;
  k.pool_sum = a.pool_sum; k.pool_max = a.pool_max; k.pool_last = a.pool_last; k.lengths = a.lengths;
  k.step_done = a.single_step ? nullptr : a.step_done; k.abort_flag = a.abort_flag;
  k.spin_limit = a.spin_limit > 0 ? a.spin_limit : kSpinLimitDefault;
  k.ldy = a.ldy; k.raw_ld = a.raw_ld; k.trace = a.trace; k.diag = a.diag;
  k.T = a.single_step ? 1 : a.T; k.t_begin = a.single_step ? a.t_step : 0;
  k.t0 = a.t0; k.T_total = a.T_total; k.ng = a.ng; k.tiles = tiles; k.out_pad = a.out_pad;
  k.nkb = a.kh_pad / 64; k.segs = a.segs; k.kh_pad = a.kh_pad;
  k.trace_items = a.trace_items; k.fault = a.fault; k.carry_c = a.carry_c;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(ctas);
  cfg.blockDim = dim3(kLThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (a.cooperative && !a.single_step) {
    attr[na].id = cudaLaunchAttributeCooperative;
    attr[na].val.cooperative = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kfn, a.tm_h, a.tm_w, a.tm_h64, FUSE ? a.tm_x : a.tm_h, k);
}

// multicast needs sibling CTAs to hold items of the same (timestep, batch, row half): tiles (hence C and the item
// total) even
bool lstm_layer_mc_ok(const LstmLayerArgs& a) {
  return a.mc != 0 && !a.single_step && a.gx_bf16 && a.pool_sum == nullptr && a.pre_nkb == 0 && a.segs == 1 &&
         (a.n_cta / 2) % 2 == 0 && a.mc_ctas >= 2;
}

}  // namespace

int lstm_layer_max_ctas() { return g_last_max_ctas; }

int lstm_layer_ctas(const LstmLayerArgs& a) {
  const long long per_step = static_cast<long long>(a.ng) * a.n_cta;   // 2 row halves x n_cta / 2 tiles
  if (a.single_step) return static_cast<int>(per_step);                // one item per CTA
  const long long total = a.T * per_step;
  long long ctas = lstm_layer_mc_ok(a) ? a.mc_ctas : a.num_sms;
  if (ctas > total) ctas = total;
  if (lstm_layer_mc_ok(a)) ctas &= ~1ll;
  return static_cast<int>(ctas);
}

namespace {

template <int GM>
cudaError_t launch_lstm_layer_gm(const LstmLayerArgs& a, cudaStream_t stream) {
  if (a.u != 32 || a.n_cta % 2 || a.kh_pad % 64 || a.ng < 1 || a.ng > kMaxBatches || a.T < 1 || (a.segs != 1 && a.segs != 3))
    return cudaErrorInvalidValue;
  const int tiles = a.n_cta / 2;
  if (a.check_only && a.mc) return launch_layer_t<GM, false, true, false, true>(a, 0, tiles, stream);
  const int ctas = lstm_layer_ctas(a);
  if (ctas < 1) return cudaErrorInvalidValue;
  const bool tok = a.tok != nullptr;  // layer 0 reading its input projection from the per-token table
  const bool pool = a.pool_sum != nullptr;
  if (a.pre_nkb > 0) {  // input projection fused into the K loop: tm_w covers [W_ih | W_hh], tm_x the previous layer's ring
    if (a.check_only || tok || a.segs != 1 || a.bias == nullptr || a.single_step) return cudaErrorInvalidValue;
    return pool ? launch_layer_t<GM, false, true, true, false, true>(a, ctas, tiles, stream)
                : launch_layer_t<GM, false, true, false, false, true>(a, ctas, tiles, stream);
  }
  if (!a.check_only && lstm_layer_mc_ok(a))
    return tok ? launch_layer_t<GM, true, true, false, true>(a, ctas, tiles, stream)
               : launch_layer_t<GM, false, true, false, true>(a, ctas, tiles, stream);
#define IE_LAYER(T_, G_)                                                                                  \
  (pool ? launch_layer_t<GM, T_, G_, true, false>(a, ctas, tiles, stream) : launch_layer_t<GM, T_, G_, false, false>(a, ctas, tiles, stream))
  if (a.gx_bf16) return tok ? IE_LAYER(true, true) : IE_LAYER(false, true);
  return tok ? IE_LAYER(true, false) : IE_LAYER(false, false);
#undef IE_LAYER
}

}  // namespace

// a.check_only: only query co-residency (lstm_layer_max_ctas()).  Requires u == 32 per slice (64 units per tile).
cudaError_t launch_lstm_layer(const LstmLayerArgs& a, cudaStream_t stream) {
  switch (a.gate_mode) {   // compiled per gate mode (lstm_common.cuh lstm_cell1)
    case kGatesFast: return launch_lstm_layer_gm<kGatesFast>(a, stream);
    case kGatesExp: return launch_lstm_layer_gm<kGatesExp>(a, stream);
    case kGatesIeee: return launch_lstm_layer_gm<kGatesIeee>(a, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace ie
