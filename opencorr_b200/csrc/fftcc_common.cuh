// fftcc_common.cuh -- the rules that define what FFT-CC returns (reference FFTCC2D::compute, src/oc_fftcc.cpp:177-275, and
// FFTCC3D::compute, src/oc_fftcc.cpp:327-427), shared by the six FFT-CC kernels: which POIs are left untouched, the cross
// spectrum of the packed transform, the first-maximum argmax and the record written for a POI.  The kernels differ only in how
// they transform.
#pragma once
#include "ocb_common.cuh"

namespace ocb {

// Border guard of a (2rx x 2ry) window: true when the POI is left untouched (src/oc_fftcc.cpp:190-196).
__device__ __forceinline__ bool fftcc2d_skip(float px, float py, float u0, float v0, int rx, int ry, int w, int h) {
	return (int)px < rx || (int)px >= w - rx || (int)py < ry || (int)py >= h - ry || (int)(px + u0) < rx || (int)(px + u0) >= w - rx
		|| (int)(py + v0) < ry || (int)(py + v0) >= h - ry || is_nan_f(px) || is_nan_f(py) || is_nan_f(u0) || is_nan_f(v0);
}

// Border guard of a (2rx x 2ry x 2rz) window: true when the POI is left untouched.  The reference has no border test here
// (src/oc_fftcc.cpp:327-365) and would read out of bounds; this engine (and the oracle) leaves such a POI untouched instead.  The
// corners are computed with the reference's float coordinate arithmetic and (int) truncation.
__device__ __forceinline__ bool fftcc3d_skip(float px, float py, float pz, float u0, float v0, float w0, int rx, int ry, int rz, int dx, int dy,
	int dz) {
	const int sx = 2 * rx, sy = 2 * ry, sz = 2 * rz;
	const int x0 = (int)(px - rx), y0 = (int)(py - ry), z0 = (int)(pz - rz);
	const int x1 = (int)(px + (sx - 1) - rx), y1 = (int)(py + (sy - 1) - ry), z1 = (int)(pz + (sz - 1) - rz);
	const int tx0 = (int)(px - rx + u0), ty0 = (int)(py - ry + v0), tz0 = (int)(pz - rz + w0);
	const int tx1 = (int)(px + (sx - 1) - rx + u0), ty1 = (int)(py + (sy - 1) - ry + v0), tz1 = (int)(pz + (sz - 1) - rz + w0);
	return x0 < 0 || y0 < 0 || z0 < 0 || x1 >= dx || y1 >= dy || z1 >= dz || tx0 < 0 || ty0 < 0 || tz0 < 0 || tx1 >= dx || ty1 >= dy || tz1 >= dz
		|| px - rx < 0 || py - ry < 0 || pz - rz < 0 || px - rx + u0 < 0 || py - ry + v0 < 0 || pz - rz + w0 < 0
		|| is_nan_f(px) || is_nan_f(py) || is_nan_f(pz) || is_nan_f(u0) || is_nan_f(v0) || is_nan_f(w0);
}

// Cross spectrum, in place: (re, im) = Z(k) becomes C(k) = conj(A(k)) B(k), with (nr, ni) = Z(-k) and A, B the spectra of the
// real and imaginary parts of the packed transform z = ref + i*tar: A = (z + conj n)/2, B = (z - conj n)/(2i)
// (src/oc_fftcc.cpp:239-240).
__device__ __forceinline__ void cross_spectrum(float& re, float& im, float nr, float ni) {
	const float Ar = 0.5f * (re + nr), Ai = 0.5f * (im - ni);
	const float dr = 0.5f * (re - nr), di = 0.5f * (im + ni);
	const float Br = di, Bi = -dr;
	re = Ar * Br + Ai * Bi;
	im = Ar * Bi - Ai * Br;
}
// 4 C(k), the same operations without the four halvings: every value is exactly 4 times cross_spectrum's (scaling by a power
// of two commutes with rounding), and so is every value of a transform of it.  A kernel that uses it scans the surface from
// -8 and hands a quarter of the peak to the result, and so returns cross_spectrum's records bit for bit.
__device__ __forceinline__ void cross_spectrum4(float& re, float& im, float nr, float ni) {
	const float Ar = re + nr, Ai = im - ni;
	const float dr = re - nr, di = im + ni;
	const float Br = di, Bi = -dr;
	re = Ar * Br + Ai * Bi;
	im = Ar * Bi - Ai * Br;
}

// First-maximum argmax: the reference scans the surface in linear order from -2.f with a strict '>' (src/oc_fftcc.cpp:246-255),
// so of equal values the lowest index wins.  Partial results merge in any order.
__device__ __forceinline__ void argmax_merge(float& bv, int& bi, float v, int i) {
	if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
}
// the warp's argmax, in every lane
__device__ __forceinline__ void warp_argmax(float& bv, int& bi) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
		const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
		argmax_merge(bv, bi, ov, oi);
	}
}

// A window of constant grey is zero once its mean is taken off.  The reference transforms the two windows separately
// (src/oc_fftcc.cpp:233-243, 378-388), so its surface is then zero everywhere: index 0 wins and ZNCC is 0 / 0.  The packed
// transform only cancels Z(k) + conj Z(-k) up to rounding, which would leave noise to pick the displacement.  So a POI with a
// zero norm (na, nb: the sums of squares of the zero-mean windows) reports the peak (0, 0).
__device__ __forceinline__ void fftcc_constant_window(float& bv, int& bi, float na, float nb) {
	if (na == 0.f || nb == 0.f) { bv = 0.f; bi = 0; }
}
// ZNCC of the peak value bv of the correlation surface of two windows of m points (src/oc_fftcc.cpp:274, 426)
__device__ __forceinline__ float fftcc_zncc(float bv, float na, float nb, int m) { return bv / (sqrtf(na * nb) * (float)m); }
// peak position d in [0, 2r) along one axis -> displacement in (-r, r]
__device__ __forceinline__ int fftcc_wrap(int d, int r) { return d > r ? d - 2 * r : d; }

// The result of a POI: the guess (u0, v0) plus the displacement of the peak (value bv) at linear index bi (x fastest) of the
// (2ry x 2rx) surface, and its ZNCC.  The index is split as unsigned, so that a power-of-two width divides by a shift.
struct Fftcc2dResult {
	float u, v, zncc;
};
__device__ __forceinline__ Fftcc2dResult fftcc2d_result(float bv, int bi, float na, float nb, int rx, int ry, float u0, float v0) {
	fftcc_constant_window(bv, bi, na, nb);
	const int sw = 2 * rx;
	const unsigned k = (unsigned)bi;
	return { (float)fftcc_wrap((int)(k % sw), rx) + u0, (float)fftcc_wrap((int)(k / sw), ry) + v0, fftcc_zncc(bv, na, nb, sw * 2 * ry) };
}
__device__ __forceinline__ void fftcc2d_store(float* P, float bv, int bi, float na, float nb, int rx, int ry, float u0, float v0) {
	const Fftcc2dResult r = fftcc2d_result(bv, bi, na, nb, rx, ry, u0, v0);
	P[P2_DEF + D2_U] = r.u;
	P[P2_DEF + D2_V] = r.v;
	P[P2_U0] = u0;
	P[P2_V0] = v0;
	P[P2_ZNCC] = r.zncc;
}

// the same for the (2rz x 2ry x 2rx) surface, linear index (z * 2ry + y) * 2rx + x
__device__ __forceinline__ void fftcc3d_store(float* P, float bv, int bi, float na, float nb, int rx, int ry, int rz, float u0, float v0, float w0) {
	fftcc_constant_window(bv, bi, na, nb);
	const int sx = 2 * rx, sy = 2 * ry;
	const unsigned k = (unsigned)bi;
	P[P3_DEF + 0] = (float)fftcc_wrap((int)(k % sx), rx) + u0;
	P[P3_DEF + 4] = (float)fftcc_wrap((int)(k / sx % sy), ry) + v0;
	P[P3_DEF + 8] = (float)fftcc_wrap((int)(k / (sx * sy)), rz) + w0;
	P[P3_U0] = u0;
	P[P3_V0] = v0;
	P[P3_W0] = w0;
	P[P3_ZNCC] = fftcc_zncc(bv, na, nb, sx * sy * 2 * rz);
}

} // namespace ocb
