// Pair-wise FP32 arithmetic on complex values and on frame pairs kept in register pairs.
//
// sm_90 has no packed FP32 instructions, so every pair operation is two scalar FADD / FMUL / FFMA.  The
// interface keeps the (lo, hi) pair in one 64-bit value so that callers can build operands such as
// `{y, x}`, `{t, t}` or `{-t, t}` without caring how they are evaluated; ptxas removes the moves.
// A complex multiply-accumulate
//     (ar + wr br - wi bi,  ai + wr bi + wi br)
// is  t = fma2(splat(wr), b, a);  p = fma2({-wi, wi}, {bi, br}, t)  -- four FFMA.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200a {

__device__ __forceinline__ uint64_t pk2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ uint64_t pk2(float2 v) { return pk2(v.x, v.y); }
__device__ __forceinline__ float2 upk2(uint64_t v) {
  float2 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
  return r;
}
__device__ __forceinline__ uint64_t add2_raw(uint64_t a, uint64_t b) {
  const float2 x = upk2(a), y = upk2(b);
  return pk2(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y));
}
__device__ __forceinline__ uint64_t mul2_raw(uint64_t a, uint64_t b) {
  const float2 x = upk2(a), y = upk2(b);
  return pk2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}
__device__ __forceinline__ uint64_t fma2_raw(uint64_t a, uint64_t b, uint64_t c) {
  const float2 x = upk2(a), y = upk2(b), z = upk2(c);
  return pk2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}

// element-wise on (x, y) pairs
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return upk2(add2_raw(pk2(a), pk2(b))); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return upk2(add2_raw(pk2(a), pk2(-b.x, -b.y))); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return upk2(mul2_raw(pk2(a), pk2(b))); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return upk2(fma2_raw(pk2(a), pk2(b), pk2(c))); }
// s * a, s * a + c with one scalar
__device__ __forceinline__ float2 scale2(float s, float2 a) { return upk2(mul2_raw(pk2(s, s), pk2(a))); }
__device__ __forceinline__ float2 fmas2(float s, float2 a, float2 c) { return upk2(fma2_raw(pk2(s, s), pk2(a), pk2(c))); }
// a + i b, a - i b  (i b = (-b.y, b.x))
__device__ __forceinline__ float2 add_i(float2 a, float2 b) { return upk2(add2_raw(pk2(a), pk2(-b.y, b.x))); }
__device__ __forceinline__ float2 sub_i(float2 a, float2 b) { return upk2(add2_raw(pk2(a), pk2(b.y, -b.x))); }
// complex product v * w
__device__ __forceinline__ float2 cmul2(float2 v, float2 w) {
  const uint64_t t = mul2_raw(pk2(v), pk2(w.x, w.x));                 // (v.x w.x, v.y w.x)
  return upk2(fma2_raw(pk2(v.y, v.x), pk2(-w.y, w.y), t));           // (- v.y w.y, + v.x w.y)
}
// a + w b for a compile-time style pair (wr, wi) held in scalars
__device__ __forceinline__ float2 cfma2(float wr, float wi, float2 b, float2 a) {
  const uint64_t t = fma2_raw(pk2(wr, wr), pk2(b), pk2(a));           // (a.x + wr b.x, a.y + wr b.y)
  return upk2(fma2_raw(pk2(b.y, b.x), pk2(-wi, wi), t));             // (- wi b.y, + wi b.x)
}

}  // namespace b200a
