// Arithmetic of the recurrent kernel (lstm_layer.cu; its persistent launch and the per-timestep fallback launch run the
// same code): the LSTM cell update of one hidden unit and the masked concat-pool accumulation.
//
// Reference arithmetic: torch nn.LSTM as wrapped by fastai's AWD_LSTM, called at
// Issue_Embeddings/flask_app/inference.py:57,68 (gate rows i|f|g|o, c_t = f*c_{t-1} + i*g, h_t = o*tanh(c_t));
// pooling: inference.py:239 ([mean | max | last] over the first len_i steps).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "ptx.cuh"

namespace ie {

// gate precision levels (LstmLayerArgs::gate_mode / LstmStepArgs::gate_mode)
constexpr int kGatesFast = 2;   // tanh.approx.f32 (1 MUFU per transcendental, rel err 2^-11): the bf16 default
constexpr int kGatesExp = 1;    // ex2.approx + rcp.approx (abs err ~1e-7): IE_CFG_ACCURATE_GATES
constexpr int kGatesIeee = 0;   // expf + IEEE division: the fp32-accurate mode (IE_CFG_FP32)

__device__ __forceinline__ float sigmoid_ieee(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float tanh_ieee(float x) {
  // 1 - 2/(e^{2x}+1) loses relative accuracy near 0: use expm1 there; odd in x
  const float ax = fabsf(x);
  float t;
  if (ax < 0.55f) {
    const float e = expm1f(2.0f * ax);
    t = e / (e + 2.0f);
  } else {
    t = 1.0f - 2.0f / (expf(2.0f * ax) + 1.0f);
  }
  return copysignf(t, x);
}

// One hidden unit of one batch row.  z* = the accumulator (h_{t-1} W_hh^T, plus x_t W_ih^T when the input projection
// rides the K loop) + Gx (x_t W_ih^T + b_ih + b_hh) or the bias; gate order i, f, g, o as in torch.  The gate mode is a
// template parameter so that an epilogue holds only the one gate path it runs.
//
// The contraction of c = f c_{t-1} + i g is spelled out in every gate mode: left to the compiler, the choice of which
// product to fuse depends on the surrounding code, and outputs would change bits from one kernel to the next.  Each form
// is the one the compiler had chosen for every kernel and the ie_debug_gates hook of its mode (measured on the H100 bit
// for bit against oracle/device_numerics.teacher_forced_exact, DESIGN.md section 2): fast and exp gates round i g and
// fuse f c_{t-1} onto it, the IEEE gates round f c_{t-1} and fuse i g onto it.  h = o tanh(c) is one rounded product.
template <int GM>
__device__ __forceinline__ void lstm_cell1(float zi, float zf, float zg, float zo, float cprev, float& cnew, float& hn) {
  if constexpr (GM == kGatesFast) {
    cnew = fmaf(sigmoid_fast(zf), cprev, __fmul_rn(sigmoid_fast(zi), tanh_fast(zg)));
    hn = __fmul_rn(sigmoid_fast(zo), tanh_fast(cnew));
  } else if constexpr (GM == kGatesExp) {
    cnew = fmaf(sigmoid_acc(zf), cprev, __fmul_rn(sigmoid_acc(zi), tanh_acc(zg)));
    hn = __fmul_rn(sigmoid_acc(zo), tanh_acc(cnew));
  } else {
    cnew = fmaf(sigmoid_ieee(zi), tanh_ieee(zg), __fmul_rn(sigmoid_ieee(zf), cprev));
    hn = __fmul_rn(sigmoid_ieee(zo), tanh_ieee(cnew));
  }
}

// ---- masked concat-pool accumulators in global memory ------------------------------------------------------------
// Natural unit order [row, out_pad]; the epilogue handles four adjacent units of one row at a time (one 16-byte access).
// pool_sum : f32, sequential sum over t (one add per timestep, in timestep order): an L2 reduction (red.add.v4.f32 =
//            four independent f32 adds) -- no load, no accumulator registers.  The (step, batch) counter protocol of the
//            persistent kernel orders step t's reduction after step t-1's (gpu-scope fence before the counter
//            increment), so it is the same sequential f32 sum a register accumulator would give: identical bits on
//            every path.
// pool_max : f32 running max; it travels like the cell state (read from L2 after the (t-1, batch) counter was seen)
// pool_last: f32, h at t == len-1
__device__ __forceinline__ void red_add_v4_f32(float* p, float4 v) {
  asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
// po: offset of the first of the four units in the [row, out_pad] accumulator arrays (a multiple of 4); tg: global
// timestep; len: valid length of the row; mprev: the running max before this step if the caller already loaded it
// (read from L2 after the (t-1, batch) counter was seen), nullptr to load it here
__device__ __forceinline__ void pool_accumulate4(float* pool_sum, float* pool_max, float* pool_last, long long po,
                                                 float4 hn, int tg, int len, const float4* mprev = nullptr) {
  if (tg >= len) return;
  float4* mp = reinterpret_cast<float4*>(pool_max + po);
  if (tg == 0) {
    __stcg(reinterpret_cast<float4*>(pool_sum + po), hn);
    __stcg(mp, hn);
  } else {
    red_add_v4_f32(pool_sum + po, hn);
    const float4 m = mprev != nullptr ? *mprev : __ldcg(mp);
    __stcg(mp, make_float4(fmaxf(m.x, hn.x), fmaxf(m.y, hn.y), fmaxf(m.z, hn.z), fmaxf(m.w, hn.w)));
  }
  if (tg == len - 1) __stcg(reinterpret_cast<float4*>(pool_last + po), hn);
}

// order-preserving u32 encoding of f32 (used by pr_curve.cu to sort scores as integers)
__device__ __forceinline__ uint32_t enc_max(float x) {
  const uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float dec_max(uint32_t e) {
  const uint32_t b = (e & 0x80000000u) ? (e & 0x7FFFFFFFu) : ~e;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, 4);
  return f;
#endif
}

// h_t of four adjacent units in the ring: bf16 (hi), one 8-byte store; with `lo_off` > 0 also the bf16 residual
// h - hi at column offset lo_off (the split-bf16 fp32-accurate mode: h ~ hi + lo to ~16 mantissa bits)
__device__ __forceinline__ void store_h4(__nv_bfloat16* yp, float4 hn, long long lo_off) {
  // hi as f32 (exactly representable: re-rounding it in pack_bf16x2 is the identity)
  const float x = __bfloat162float(__float2bfloat16_rn(hn.x)), y = __bfloat162float(__float2bfloat16_rn(hn.y));
  const float z = __bfloat162float(__float2bfloat16_rn(hn.z)), w = __bfloat162float(__float2bfloat16_rn(hn.w));
  *reinterpret_cast<uint2*>(yp) = make_uint2(pack_bf16x2(x, y), pack_bf16x2(z, w));
  if (lo_off > 0)
    *reinterpret_cast<uint2*>(yp + lo_off) = make_uint2(pack_bf16x2(hn.x - x, hn.y - y), pack_bf16x2(hn.z - z, hn.w - w));
}

}  // namespace ie
