// ocb_f32x2.cuh -- fp32 pairs: two independent IEEE round-to-nearest operations per call.  sm_90 has no packed fp32
// instruction, so each pair is two scalar FFMA / FMUL / FADD; the __f*_rn intrinsics keep every operation rounded on its
// own (no contraction of a multiply into a following add), which is what the callers' arithmetic order relies on.
#pragma once
#include <cuda_runtime.h>

namespace ocb {

__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
	return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fsub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 bcast2(float a) { return make_float2(a, a); }

} // namespace ocb
