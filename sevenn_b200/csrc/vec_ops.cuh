// Scalar / packed-pair arithmetic used by the generated tensor-product code.
//
// `V2` is float2: one thread processes two channels.  sm_90a has no packed FP32 instructions, so each
// operation is two scalar round-to-nearest FFMA / FMUL / FADD (bit-identical to a packed form).  When
// the same headers are compiled by a host compiler (tests/cpu_harness) the pair type is emulated with
// plain floats.
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#include <cuda_runtime.h>
#ifndef S7B_HD
#define S7B_HD __device__ __forceinline__
#endif
namespace s7b {
using V2 = float2;
S7B_HD V2 fma_(V2 a, V2 b, V2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
S7B_HD V2 fma_(float s, V2 b, V2 c) { return make_float2(__fmaf_rn(s, b.x, c.x), __fmaf_rn(s, b.y, c.y)); }
S7B_HD V2 mul_(V2 a, V2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
S7B_HD V2 mul_(V2 a, float s) { return make_float2(__fmul_rn(a.x, s), __fmul_rn(a.y, s)); }
S7B_HD V2 add_(V2 a, V2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
S7B_HD V2 splat2(float s) { return make_float2(s, s); }
}  // namespace s7b
#else
#ifndef S7B_HD
#define S7B_HD inline
#endif
namespace s7b {
struct V2 { float x, y; };
S7B_HD V2 fma_(V2 a, V2 b, V2 c) { return {std::fmaf(a.x, b.x, c.x), std::fmaf(a.y, b.y, c.y)}; }
S7B_HD V2 fma_(float s, V2 b, V2 c) { return {std::fmaf(s, b.x, c.x), std::fmaf(s, b.y, c.y)}; }
S7B_HD V2 mul_(V2 a, V2 b) { return {a.x * b.x, a.y * b.y}; }
S7B_HD V2 mul_(V2 a, float s) { return {a.x * s, a.y * s}; }
S7B_HD V2 add_(V2 a, V2 b) { return {a.x + b.x, a.y + b.y}; }
S7B_HD V2 splat2(float s) { return {s, s}; }
}  // namespace s7b
#endif

namespace s7b {
S7B_HD float fma_(float a, float b, float c) { return fmaf(a, b, c); }
S7B_HD float mul_(float a, float b) { return a * b; }
S7B_HD float add_(float a, float b) { return a + b; }
}  // namespace s7b
