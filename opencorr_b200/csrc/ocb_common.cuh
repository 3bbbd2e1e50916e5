// ocb_common.cuh -- shared definitions for the sm_90a kernels and the C-ABI host layer.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace ocb {

// POI record field offsets (reference: src/oc_poi.h:25-33,44-51,102-136 / :62-71,93-99,187-222)
enum { P2_X = 0, P2_Y = 1, P2_DEF = 2, P2_U0 = 14, P2_V0 = 15, P2_ZNCC = 16, P2_ITER = 17, P2_CONV = 18,
       P2_FEAT = 19, P2_STRAIN = 20, P2_RX = 23, P2_RY = 24, P2_N = 25 };
// 2D deformation vector order: u ux uy uxx uxy uyy v vx vy vxx vxy vyy
enum { D2_U = 0, D2_UX = 1, D2_UY = 2, D2_UXX = 3, D2_UXY = 4, D2_UYY = 5,
       D2_V = 6, D2_VX = 7, D2_VY = 8, D2_VXX = 9, D2_VXY = 10, D2_VYY = 11 };
enum { P3_X = 0, P3_Y = 1, P3_Z = 2, P3_DEF = 3, P3_U0 = 15, P3_V0 = 16, P3_W0 = 17, P3_ZNCC = 18,
       P3_ITER = 19, P3_CONV = 20, P3_FEAT = 21, P3_STRAIN = 22, P3_RX = 28, P3_RY = 29, P3_RZ = 30, P3_N = 31 };
// 3D deformation vector order: u ux uy uz v vx vy vz w wx wy wz
// POI2DS (stereo DIC, src/oc_poi.h:140-186): x y | u v w | r1r2 r1t1 r1t2 ZNCC | r2_x r2_y t1_x t1_y t2_x t2_y | ref_coor |
// tar_coor | e[6] | subset_radius
enum { P2DS_U = 2, P2DS_ZNCC = 5, P2DS_REF = 14, P2DS_STRAIN = 20, P2DS_N = 28 };

struct Image2D {
	const float* ref;
	const float* tar;
	int w, h;
};

struct Image3D {
	const float* ref;
	const float* tar;
	const float4* rg;  // per voxel {ref, gx, gy, gz}: Gradient3D4 of ref packed with ref (built by prepare)
	const float* coef; // tricubic B-spline coefficients of tar (built by prepare)
	int dx, dy, dz;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	return v;
}

__device__ __forceinline__ bool is_nan_f(float v) { return v != v; }

// 4th-order central difference with the reference's operation order and roundings
// (src/oc_gradient.cpp:49-54): ((0 - f(+2)/12) + f(+1)*2/3) - f(-1)*2/3 + f(-2)/12, no FMA.
__device__ __forceinline__ float grad4(float m2, float m1, float p1, float p2) {
	const float first_factor = 1.f / 12.f;
	const float second_factor = 2.f / 3.f;
	float result = __fsub_rn(0.0f, __fmul_rn(p2, first_factor));
	result = __fadd_rn(result, __fmul_rn(p1, second_factor));
	result = __fsub_rn(result, __fmul_rn(m1, second_factor));
	result = __fadd_rn(result, __fmul_rn(m2, first_factor));
	return result;
}

// Bicubic weights of the reference's BC = B*C matrix (src/oc_cubic_bspline.h:52-58):
// w[m] = sum_k BC[k][m] t^(3-k).  value = sum_n sum_m wy[n] q[n][m] wx[m]  (SURVEY A.3).
__device__ __forceinline__ void bicubic_weights(float t, float* w) {
	const float s = 1.0f / 336.0f;
	w[0] = ((-144.0f * s * t + 342.0f * s) * t - 198.0f * s) * t;
	w[1] = ((384.0f * s * t - 702.0f * s) * t - 18.0f * s) * t + 1.0f;
	w[2] = ((-384.0f * s * t + 450.0f * s) * t + 270.0f * s) * t;
	w[3] = ((144.0f * s * t - 90.0f * s) * t - 54.0f * s) * t;
}

// In-register Cholesky factorisation of a symmetric positive-definite N x N matrix given by its
// lower triangle (row-major packed: a[i*(i+1)/2 + j], j <= i).  On return a holds L (same packing)
// with the diagonal replaced by 1/L_ii.  Every index is a compile-time constant after unrolling.
template <int N>
__device__ __forceinline__ void cholesky_packed(float* a) {
#pragma unroll
	for (int j = 0; j < N; j++) {
		float d = a[j * (j + 1) / 2 + j];
#pragma unroll
		for (int k = 0; k < j; k++) {
			float l = a[j * (j + 1) / 2 + k];
			d -= l * l;
		}
		float inv = rsqrtf(d);
		// one Newton step so that 1/L_jj is accurate to ~1 ulp
		inv = inv * (1.5f - 0.5f * d * inv * inv);
		a[j * (j + 1) / 2 + j] = inv;
#pragma unroll
		for (int i = j + 1; i < N; i++) {
			float v = a[i * (i + 1) / 2 + j];
#pragma unroll
			for (int k = 0; k < j; k++) v -= a[i * (i + 1) / 2 + k] * a[j * (j + 1) / 2 + k];
			a[i * (i + 1) / 2 + j] = v * inv;
		}
	}
}

// Solve L L^T x = b with the packed factor from cholesky_packed (diagonal holds 1/L_ii).
template <int N>
__device__ __forceinline__ void cholesky_solve(const float* a, const float* b, float* x) {
	float y[N];
#pragma unroll
	for (int i = 0; i < N; i++) {
		float v = b[i];
#pragma unroll
		for (int k = 0; k < i; k++) v -= a[i * (i + 1) / 2 + k] * y[k];
		y[i] = v * a[i * (i + 1) / 2 + i];
	}
#pragma unroll
	for (int i = N - 1; i >= 0; i--) {
		float v = y[i];
#pragma unroll
		for (int k = i + 1; k < N; k++) v -= a[k * (k + 1) / 2 + i] * x[k];
		x[i] = v * a[i * (i + 1) / 2 + i];
	}
}

} // namespace ocb
