// ocb_tile2d.cuh -- per-warp 2D tile staging and bicubic B-spline sampling shared by icgn2d.cu and nr2d.cu.
#pragma once
#include "ocb_common.cuh"

namespace ocb {

// Stage a (rows x cols) window of a row-major image into smem (row pitch `cols`), origin (ox, oy),
// subtracting `shift`; pixels outside the image read as -shift.  Lanes run along x (coalesced).
__device__ __forceinline__ void stage_tile(float* dst, const float* __restrict__ img, int w, int h, int ox, int oy, int cols, int rows,
	float shift, int lane) {
	for (int col = lane; col < cols; col += 32) {
		const int gx = ox + col;
		const bool colok = gx >= 0 && gx < w;
#pragma unroll 8
		for (int row = 0; row < rows; row++) {
			const int gy = oy + row;
			float v = 0.f;
			if (colok && gy >= 0 && gy < h) v = __ldg(img + (size_t)gy * w + gx);
			dst[row * cols + col] = v - shift;
		}
	}
}

// The interpolant over one 4x4 block: each block row folded with the x weights, then the rows with the y weights, in this
// FMA order.  pix(n, m) reads pixel m of block row n.  Every sampling path, and icgn2d_exact_negative's fused pre-check, goes
// through this one fold, so the same block and weights give the same bits wherever they are evaluated.
template <class Pix>
__device__ __forceinline__ float bicubic_fold(const float* wx, const float* wy, Pix pix) {
	float t = 0.f;
#pragma unroll
	for (int nn = 0; nn < 4; nn++) {
		const float row = fmaf(pix(nn, 3), wx[3], fmaf(pix(nn, 2), wx[2], fmaf(pix(nn, 1), wx[1], pix(nn, 0) * wx[0])));
		t = fmaf(row, wy[nn], t);
	}
	return t;
}

// Bicubic B-spline sample of the target at (X, Y), src/oc_cubic_bspline.cpp:134-181.
// fast: the 4x4 support lies inside the staged tile.  Otherwise read the image (caller guarantees
// 1 <= X < w-2, 1 <= Y < h-2).
__device__ __forceinline__ float bicubic_sample(const float* tile, int TW, int tx0, int ty0, const float* __restrict__ tar, int w,
	float X, float Y, bool fast) {
	const float xf = floorf(X), yf = floorf(Y);
	float wx[4], wy[4];
	bicubic_weights(X - xf, wx);
	bicubic_weights(Y - yf, wy);
	const int ix = (int)xf - 1, iy = (int)yf - 1;
	if (fast) {
		const float* q = tile + (iy - ty0) * TW + (ix - tx0);
		return bicubic_fold(wx, wy, [&](int n, int m) { return q[n * TW + m]; });
	}
	const float* q = tar + (size_t)iy * w + ix;
	return bicubic_fold(wx, wy, [&](int n, int m) { return __ldg(q + (size_t)n * w + m); });
}

} // namespace ocb
