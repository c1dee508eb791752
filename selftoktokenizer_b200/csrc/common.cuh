// Shared host/device helpers for the selftok_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace stk {

// ---- host-side error plumbing (status codes mirror include/selftok_b200.h) ---------------------------------
void set_error(const std::string& msg);
#define STK_CUDA(expr)                                                                            \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      ::stk::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + \
                       std::to_string(__LINE__));                                                 \
      return -5;                                                                                  \
    }                                                                                             \
  } while (0)
#define STK_CHECK(cond, code, msg)                                                                \
  do {                                                                                            \
    if (!(cond)) {                                                                                \
      ::stk::set_error(std::string(msg) + " [" #cond "] @" + __FILE__ + ":" + std::to_string(__LINE__)); \
      return (code);                                                                              \
    }                                                                                             \
  } while (0)
#define STK_TRY(expr)                                                                             \
  do {                                                                                            \
    int _s = (expr);                                                                              \
    if (_s != 0) return _s;                                                                       \
  } while (0)

extern thread_local int64_t g_launch_count;   // bumped by every launch wrapper
inline void count_launch() { ++g_launch_count; }

// ---- device helpers ------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// torch.nn.GELU(approximate="tanh"): 0.5*x*(1+tanh(u)), u = sqrt(2/pi)*(x+0.044715*x^3)
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float inner = k0 * (x + k1 * x * x * x);
  return 0.5f * x * (1.0f + tanhf(inner));
}
// Same function as x / (1 + exp(-2u)) with the fast exp/divide intrinsics (~1e-6 relative): used by the tensor-core
// epilogues, whose operands are rounded to 16 bits right afterwards.
__device__ __forceinline__ float gelu_tanh_fast(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  return __fdividef(x, 1.0f + __expf(-2.0f * u));
}
// GELU-tanh on a pair, y = x / (1 + 2^(c2 * x * (1 + k1 x^2))),  c2 = -2 log2(e) sqrt(2/pi), with ex2 / rcp on the MUFU
// pipe.  Every step is an explicitly rounded single operation (no contraction), so the result does not depend on how the
// compiler schedules it.
__device__ __forceinline__ float gelu_tanh_fast1(float x) {
  const float k1 = 0.044715f, c2 = -2.0f * 1.4426950408889634f * 0.7978845608028654f;
  float t = __fmul_rn(x, x);                 // x^2
  t = __fmaf_rn(t, k1, 1.0f);                // 1 + k1 x^2
  t = __fmul_rn(t, x);                       // x (1 + k1 x^2)
  t = __fmul_rn(t, c2);                      // exponent (base 2)
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  e = __fadd_rn(e, 1.0f);                    // 1 + e
  asm("rcp.approx.ftz.f32 %0, %0;" : "+f"(e));
  return __fmul_rn(e, x);                    // x / (1 + e)
}
__device__ __forceinline__ float2 gelu_tanh_fast2(float2 v) { return make_float2(gelu_tanh_fast1(v.x), gelu_tanh_fast1(v.y)); }
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }

enum Act { ACT_NONE = 0, ACT_GELU = 1, ACT_SILU = 2 };
__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == ACT_GELU) return gelu_tanh(x);
  if (act == ACT_SILU) return silu(x);
  return x;
}

// bf16 split: hi = rn(x), lo = rn(x - hi).  hi + lo carries ~16 mantissa bits of x.
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
// two fp32 -> one packed 16-bit pair (lo in bits 0-15): IEEE half with saturation to +-65504 (one F2FP.SATFINITE instead of
// two clamps + convert; +-inf saturates too, NaN stays NaN), or bf16 round-to-nearest
__device__ __forceinline__ uint32_t pack2_sat16(float lo, float hi, bool fp16) {
  uint32_t r;
  if (fp16) asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// 16-bit operand planes hold either bf16 (hi [+ lo] split) or, in the single-pass fp16 mode, IEEE half values; the
// storage type is __nv_bfloat16 in both cases (the bits are what the tensor core is told they are).  The half conversion is
// the one the tensor-core epilogues use (pack2_sat16), so a value converts to the same bits on every path: a clamp with
// fminf / fmaxf would turn NaN into -65504.
__device__ __forceinline__ void split16(float x, bool fp16, uint16_t& hi, uint16_t& lo) {
  if (fp16) {
    hi = (uint16_t)(pack2_sat16(x, 0.f, true) & 0xffffu);
    lo = 0;
  } else {
    __nv_bfloat16 h = __float2bfloat16_rn(x);
    hi = __bfloat16_as_ushort(h);
    lo = __bfloat16_as_ushort(__float2bfloat16_rn(x - __bfloat162float(h)));
  }
}
// bf16 residual plane of a pair: lo = rn(x - rn_bf16(x))
__device__ __forceinline__ uint32_t pack2_resid_bf16(float a, float b, uint32_t hi_pair) {
  const float ra = a - __uint_as_float(hi_pair << 16), rb = b - __uint_as_float(hi_pair & 0xffff0000u);
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(rb), "f"(ra));
  return r;
}

// ---- e4m3 quantization (the contract in kernels.h) ----
// max that keeps NaN (fmaxf drops it)
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float warp_max_nan(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// row amax -> (inv, scale): inv = 448 / amax, scale = amax / 448, both 0 for an all-zero row
__device__ __forceinline__ void e4m3_row_scale(float amax, float& inv, float& scale) {
  inv = amax == 0.f ? 0.f : __fdiv_rn(448.f, amax);
  scale = __fdiv_rn(amax, 448.f);
}
// four fp32 -> four e4m3 codes (x0 in the low byte): cvt.rn.satfinite of x_i * inv
__device__ __forceinline__ uint32_t pack4_e4m3(float x0, float x1, float x2, float x3, float inv) {
  const float a = __fmul_rn(x0, inv), b = __fmul_rn(x1, inv), c = __fmul_rn(x2, inv), d = __fmul_rn(x3, inv);
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

// element pairs: (d0, d1) = (a0, a1) * (b0, b1) + (c0, c1) and (d0, d1) = (a0, a1) + (b0, b1), each lane rounded once
__device__ __forceinline__ void ffma2(float a0, float a1, float b0, float b1, float c0, float c1, float& d0, float& d1) {
  d0 = __fmaf_rn(a0, b0, c0);
  d1 = __fmaf_rn(a1, b1, c1);
}
// the same on pairs held as packed 64-bit registers (low word = first lane): acc = a * b + acc per lane
__device__ __forceinline__ void fma2_packed(unsigned long long& acc, unsigned long long a, unsigned long long b) {
  const float d0 = __fmaf_rn(__uint_as_float((uint32_t)a), __uint_as_float((uint32_t)b), __uint_as_float((uint32_t)acc));
  const float d1 = __fmaf_rn(__uint_as_float((uint32_t)(a >> 32)), __uint_as_float((uint32_t)(b >> 32)), __uint_as_float((uint32_t)(acc >> 32)));
  acc = (unsigned long long)__float_as_uint(d0) | ((unsigned long long)__float_as_uint(d1) << 32);
}
__device__ __forceinline__ void fadd2(float a0, float a1, float b0, float b1, float& d0, float& d1) {
  d0 = __fadd_rn(a0, b0);
  d1 = __fadd_rn(a1, b1);
}

}  // namespace stk
