// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), clusters, wgmma.
// Everything the kernels in this directory need and nothing else.  No CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ie {

// L2 cache-policy immediates accepted by cp.async.bulk.tensor ... .L2::cache_hint
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst  = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast   = 0x14F0000000000000ull;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// make generic-proxy writes visible to the async proxy (TMA operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// plain arrive on the barrier at the same smem offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t"
      "}\n"
      ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}
// ----------------------------------------------------------------------------------------------
// Abort protocol of every spin in this directory.  A wait that exceeds `limit` SM cycles (a protocol bug, or a
// persistent grid that lost co-residency) does NOT trap -- a trap poisons the CUDA context of every handle in the
// process, and include/issue_emb_b200.h promises error codes.  Instead the waiter raises the CTA's shared-memory flag
// and the launch's global flag (the handle's error word) and returns; from then on every wait of the CTA returns at
// once ("drain mode": role loops fall through, results are garbage, the kernel terminates), other CTAs adopt the
// global flag the next time one of their spins polls it, and the host turns the flag into IE_ERR_CUDA.
// ----------------------------------------------------------------------------------------------
struct Abort {
  uint32_t* s;      // this CTA's flag in shared memory (initialised to 0 by the thread that initialises the barriers)
  unsigned* g;      // the launch's flag in global memory (nullptr: none)
  long long limit;  // SM cycles a single wait may take
};
constexpr long long kSpinLimitDefault = 4000000000ll;  // ~2 s

__device__ __forceinline__ bool aborted(const Abort& a) {
  uint32_t v;
  asm volatile("ld.volatile.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(a.s)) : "memory");
  return v != 0;
}
// Inlined, like every helper here: an out-of-line (ABI) call in a kernel makes ptxas ignore its setmaxnreg budgets.
static __device__ __forceinline__ void abort_raise(const Abort& a) {
  asm volatile("st.volatile.shared::cta.u32 [%0], %1;" ::"r"(smem_u32(a.s)), "r"(1u) : "memory");
  if (a.g != nullptr) atomicExch(a.g, 1u);
}
// slow-path poll (every few hundred spins): true once this CTA is in drain mode
static __device__ __forceinline__ bool abort_poll(const Abort& a, long long t0) {
  if (aborted(a)) return true;
  bool hit = (clock64() - t0) > a.limit;
  if (!hit && a.g != nullptr) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.g) : "memory");
    hit = v != 0;
  }
  if (hit) abort_raise(a);
  return hit;
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, const Abort& ab) {
  if (mbar_try_wait(bar, parity)) return;
  if (aborted(ab)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 0xFFu) == 0 && abort_poll(ab, t0)) return;
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
// 2-D tiled load global -> shared, completion on an mbarrier (complete_tx::bytes). c0 = inner coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}

// multicast variant: the box is written to the same CTA-relative smem offset of every CTA in `mask`, and each
// destination CTA's mbarrier (same offset) receives the complete_tx
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                               int32_t c1, uint16_t mask, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%4, %5}], [%2], %3, %6;"
      ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// thread-block clusters
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// all threads of all CTAs in the cluster (also orders shared-memory accesses like __syncthreads)
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA)
// ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor: K-major operand tile, 128-byte swizzle, rows 128 B apart, 8-row core-matrix groups
// 1024 B apart (what a TMA box {64 bf16, rows} with SWIZZLE_128B writes).  Advancing 16 bf16 = 32 B along K inside
// the swizzle atom is +2 in the (addr >> 4) field.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);  // [0,14)  start address >> 4
  d |= 1ull << 16;                                          // [16,30) leading byte offset: unused for swizzled K-major
  d |= static_cast<uint64_t>(1024u >> 4) << 32;             // [32,46) stride byte offset >> 4
  d |= 1ull << 62;                                          // [62,64) SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keep the compiler from moving accumulator reads/writes across the asynchronous MMAs
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T: both operands K-major bf16 in shared memory (descriptors above), f32
// accumulators in the registers of the issuing warpgroup.  Fragment layout: d[4 j + {0, 1, 2, 3}] holds rows
// {r, r, r + 8, r + 8} and columns 8 j + 2 (lane % 4) + {0, 1, 0, 1}, where r = 16 (warp % 4) + lane / 4.
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// grid-scope flags in global memory (persistent kernels)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// bounded spin with relaxed loads, one acquire fence at the end (abort protocol above instead of hanging the GPU)
__device__ __forceinline__ void wait_flag_ge_relaxed(const unsigned* p, unsigned target, const Abort& ab) {
  if (ld_relaxed(p) < target && !aborted(ab)) {
    const long long t0 = clock64();
    uint32_t spins = 0;
    while (ld_relaxed(p) < target) {
      if (((++spins) & 0x3Fu) == 0 && abort_poll(ab, t0)) break;
    }
  }
  __threadfence();
}
__device__ __forceinline__ void red_relaxed_add(unsigned* p, unsigned v) {
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// bring the 128-byte line holding `p` into L2 (no register result, no completion to wait for)
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// per-thread register budget of the executing warpgroup from here on (every thread of all four warps must execute the
// same instruction): producer warpgroups give registers back to the SM's pool, consumer warpgroups take them
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float sigmoid_acc(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
// tanh(x) = 1 - 2/(exp(2x)+1): abs error ~1e-7, saturates correctly for |x| large
__device__ __forceinline__ float tanh_acc(float x) { return 1.0f - __fdividef(2.0f, __expf(2.0f * x) + 1.0f); }

// single-MUFU variants (tanh.approx.f32, max relative error 2^-11): the epilogue of the recurrent kernel is bound by
// the 16/clk/SM special-function unit (10 MUFU per cell with the accurate forms, 5 with these)
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigmoid_fast(float x) { return fmaf(0.5f, tanh_fast(0.5f * x), 0.5f); }

// 2^x, ex2.approx.ftz.f32 (the language-model decoder's exp, lm.cu): 0 below 2^-126, else within 1.46e-7 = 2^-22.7
// relative (measured over every f32 input)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

}  // namespace ie
