// ocb_tile2d.cuh -- the subset guard, per-warp 2D tile loads and bicubic B-spline sampling shared by icgn2d.cu and nr2d.cu.
#pragma once
#include "ocb_common.cuh"
#include "ocb_tma.cuh"

namespace ocb {

// The reference's guard in front of a 2D subset registration (src/oc_icgn.cpp:160-167 / :701-708, src/oc_nr.cpp:165-171): the
// subset must lie inside the image, the initial displacement within the image's extent and the incoming ZNCC not negative; NaN
// coordinates fail too.  Each method writes its own code for a POI that fails it.
__device__ __forceinline__ bool subset2d_guard_fails(float px, float py, int rx, int ry, int w, int h, float u, float v, float zncc) {
	return py - ry < 0 || px - rx < 0 || py + ry > h - 1 || px + rx > w - 1 || fabsf(u) >= w || fabsf(v) >= h || zncc < 0 || is_nan_f(u)
		|| is_nan_f(v) || is_nan_f(px) || is_nan_f(py);
}

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

// A (cols x rows) tile load into smem for the threads of one POI: a TMA copy completing on the mbarrier `bar` when the launch has
// a tensor map, otherwise stage_tile by one warp.  issue() starts the load and wait() returns once the tile may be read, so work
// that does not touch the tile can run in between.  sync: the barrier of the POI's threads.
struct TileLoad {
	uint64_t* bar;
	uint32_t phase;
	int tma; // the launch has a tensor map
	template <class Sync>
	__device__ __forceinline__ void init(bool leader, Sync sync) {
		if (tma) {
			if (leader) mbar_init(bar, 1);
			sync();
		}
	}
	// STACK: map is 3D over a frame-major stack (box depth 1) and the tile comes from frame z; img is that frame.
	// leader issues the TMA copy; stager (a whole warp) stages the tile without one.
	template <bool STACK>
	__device__ __forceinline__ void issue(float* dst, const CUtensorMap* map, const float* __restrict__ img, int w, int h, int x, int y, int z,
		int cols, int rows, bool leader, bool stager, int lane) {
		if (tma) {
			if (leader) {
				fence_proxy_async(); // earlier generic-proxy accesses to dst are ordered before the async-proxy write
				mbar_expect_tx(bar, (uint32_t)(cols * rows * sizeof(float)));
				if constexpr (STACK) tma_load_3d(dst, map, x, y, z, bar);
				else tma_load_2d(dst, map, x, y, bar);
			}
		} else if (stager) stage_tile(dst, img, w, h, x, y, cols, rows, 0.f, lane);
	}
	// a TMA tile is visible to every thread that waited on the barrier; a staged one after sync()
	template <class Sync>
	__device__ __forceinline__ void wait(Sync sync) {
		if (tma) { mbar_wait(bar, phase); phase ^= 1; }
		else sync();
	}
};

// Tensor map for tile loads from one row-major (w x h) image (n_frames == 0: 2D) or from a frame-major stack of n_frames of them
// (3D, box depth 1: a load reads one frame).  false: no map can be made (see tma_make_map) and the launch stages its tiles.
inline bool tma_image_map(CUtensorMap* map, const float* base, int w, int h, int n_frames, int box_w, int box_h) {
	const int dims[3] = { w, h, n_frames }, box[3] = { box_w, box_h, 1 };
	return tma_make_map(map, base, n_frames > 0 ? 3 : 2, dims, box);
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
