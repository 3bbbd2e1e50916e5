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

// Bicubic weights of the reference's BC matrix (ocb_common.cuh bicubic_weights) as two pairs {w0, w1}, {w2, w3};
// the same Horner steps, two weights per call.
__device__ __forceinline__ void bicubic_weights2(float t, float2& w01, float2& w23) {
	const float s = 1.0f / 336.0f;
	const float2 tt = bcast2(t);
	w01 = ffma2(ffma2(ffma2(make_float2(-144.0f * s, 384.0f * s), tt, make_float2(342.0f * s, -702.0f * s)), tt, make_float2(-198.0f * s, -18.0f * s)), tt,
		make_float2(0.f, 1.0f));
	w23 = fmul2(ffma2(ffma2(make_float2(-384.0f * s, 144.0f * s), tt, make_float2(450.0f * s, -90.0f * s)), tt, make_float2(270.0f * s, -54.0f * s)), tt);
}

} // namespace ocb
