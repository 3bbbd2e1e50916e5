// stereo.cu -- lens-distortion maps, undistortion and stereo triangulation, for sm_90a.
//
// Replaces Calibration::prepare (reference src/oc_calibration.cpp:161-219), Calibration::undistort (:221-264) and
// Stereovision::reconstruct (src/oc_stereovision.cpp:70-133).  Every float32 operation of the reference is rounded once,
// in the reference's order (__fmul_rn / __fadd_rn / __fdiv_rn keep nvcc from contracting to FMA), so that the maps and the
// undistorted coordinates are bit-identical to the faithful oracle.  The 4x3 triangulation system is formed in float32 as
// the reference forms it and solved in FP64 registers (Householder QR), then rounded to float.
//
// Intrinsics are passed as the 13 floats of CameraIntrinsics (src/oc_calibration.h:25-35):
//   fx fy fs cx cy k1 k2 k3 k4 k5 k6 p1 p2
#include "../../include/opencorr_b200.h"
#include "ocb_kernels.h"

namespace ocb {

struct Intrinsics {
	float fx, fy, fs, cx, cy, k1, k2, k3, k4, k5, k6, p1, p2;
};

static Intrinsics load_intrinsics(const float* v) {
	Intrinsics I;
	I.fx = v[0]; I.fy = v[1]; I.fs = v[2]; I.cx = v[3]; I.cy = v[4];
	I.k1 = v[5]; I.k2 = v[6]; I.k3 = v[7]; I.k4 = v[8]; I.k5 = v[9]; I.k6 = v[10];
	I.p1 = v[11]; I.p2 = v[12];
	return I;
}

// Calibration::image_to_sensor, :117-124
__device__ __forceinline__ void image_to_sensor(const Intrinsics& I, float x, float y, float* sx, float* sy) {
	*sy = __fadd_rn(__fmul_rn(y, I.fy), I.cy);
	*sx = __fadd_rn(__fadd_rn(__fmul_rn(x, I.fx), __fmul_rn(y, I.fs)), I.cx);
}

// Calibration::distort, :136-159
__device__ __forceinline__ void distort(const Intrinsics& I, float x, float y, float* dx, float* dy) {
	const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), xy = __fmul_rn(x, y);
	const float r2 = __fadd_rn(xx, yy);
	const float r4 = __fmul_rn(r2, r2);
	const float r6 = __fmul_rn(r2, r4);
	const float num = __fadd_rn(__fadd_rn(__fadd_rn(1.f, __fmul_rn(I.k1, r2)), __fmul_rn(I.k2, r4)), __fmul_rn(I.k3, r6));
	const float den = __fadd_rn(__fadd_rn(__fadd_rn(1.f, __fmul_rn(I.k4, r2)), __fmul_rn(I.k5, r4)), __fmul_rn(I.k6, r6));
	const float radial = __fdiv_rn(num, den);
	float oy = __fmul_rn(y, radial), ox = __fmul_rn(x, radial);
	oy = __fadd_rn(oy, __fadd_rn(__fmul_rn(I.p1, __fadd_rn(r2, __fmul_rn(2.f, yy))), __fmul_rn(__fmul_rn(2.f, I.p2), xy)));
	ox = __fadd_rn(ox, __fadd_rn(__fmul_rn(__fmul_rn(2.f, I.p1), xy), __fmul_rn(I.p2, __fadd_rn(r2, __fmul_rn(2.f, xx)))));
	*dx = ox;
	*dy = oy;
}

// One thread per pixel: sensor_to_image of (c, r) (:168-178), then the fixed-point undistortion loop (:180-218).
__global__ void __launch_bounds__(256) calib_map_kernel(Intrinsics I, int height, int width, float convergence, int iteration,
	float* __restrict__ map_x, float* __restrict__ map_y) {
	const long long total = (long long)height * width;
	const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= total) return;
	const int r = (int)(t / width), c = (int)(t - (long long)r * width);
	const float rf = (float)r, cf = (float)c;
	// sensor_to_image, :126-133
	const float y0 = __fdiv_rn(__fsub_rn(rf, I.cy), I.fy);
	const float x0 = __fdiv_rn(__fsub_rn(__fsub_rn(cf, I.cx), __fmul_rn(I.fs, y0)), I.fx);
	float ix = x0, iy = y0;
	bool stop = false;
	int i = 0;
	while (i < iteration && !stop) {
		i++;
		float dx, dy, sx, sy;
		distort(I, ix, iy, &dx, &dy);
		image_to_sensor(I, dx, dy, &sx, &sy);
		float dev_y = __fsub_rn(rf, sy);
		const float dev_x = __fsub_rn(cf, sx);
		if (isinf(dev_x) || isinf(dev_y)) { // back to the start value; the update below still runs once (:198-203)
			stop = true;
			iy = y0;
			ix = x0;
		}
		if (fabsf(dev_x) > convergence || fabsf(dev_y) > convergence) {
			dev_y = __fdiv_rn(dev_y, I.fy);
			iy = __fadd_rn(iy, dev_y);
			ix = __fadd_rn(ix, __fdiv_rn(__fsub_rn(dev_x, __fmul_rn(dev_y, I.fs)), I.fx));
		} else {
			stop = true;
		}
	}
	map_x[t] = ix;
	map_y[t] = iy;
}

// Calibration::undistort, :221-264, on a point already known not to be NaN: clamp to [0, W-2] x [0, H-2] (written back to
// the caller, who passes Point2D&), bilinear lookup in both maps, image_to_sensor with the intrinsics I.
__device__ __forceinline__ void undistort_point(const float* __restrict__ map_x, const float* __restrict__ map_y, int height, int width,
	const Intrinsics& I, float* px, float* py, float* ux, float* uy) {
	float x = *px, y = *py;
	if (x < 0.f) x = 0.f;
	if (y < 0.f) y = 0.f;
	if (x > (float)(width - 2)) x = (float)(width - 2);
	if (y > (float)(height - 2)) y = (float)(height - 2);
	*px = x;
	*py = y;
	const int yi = (int)floorf(y), xi = (int)floorf(x);
	const float yd = __fsub_rn(y, (float)yi), xd = __fsub_rn(x, (float)xi);
	const float wy0 = __fsub_rn(1.f, yd), wx0 = __fsub_rn(1.f, xd);
	const size_t i00 = (size_t)yi * width + xi, i10 = i00 + width;
	float v[2];
	const float* maps[2] = { map_y, map_x };
#pragma unroll
	for (int m = 0; m < 2; m++) {
		const float* M = maps[m];
		float s = __fmul_rn(__fmul_rn(__ldg(M + i00), wy0), wx0);
		s = __fadd_rn(s, __fmul_rn(__fmul_rn(__ldg(M + i10), yd), wx0));
		s = __fadd_rn(s, __fmul_rn(__fmul_rn(__ldg(M + i00 + 1), wy0), xd));
		s = __fadd_rn(s, __fmul_rn(__fmul_rn(__ldg(M + i10 + 1), yd), xd));
		v[m] = s;
	}
	image_to_sensor(I, v[1], v[0], ux, uy);
}

// Calibration::undistort as a batch.  A NaN coordinate (undefined in the reference) gives NaN and leaves the point untouched.
__global__ void __launch_bounds__(256) calib_undistort_kernel(const float* __restrict__ map_x, const float* __restrict__ map_y, int height, int width,
	Intrinsics I, float2* __restrict__ pts, float2* __restrict__ out, long long n) {
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float2 p = pts[i];
	if (isnan(p.x) || isnan(p.y)) {
		out[i] = make_float2(NAN, NAN);
		return;
	}
	float2 u;
	undistort_point(map_x, map_y, height, width, I, &p.x, &p.y, &u.x, &u.y);
	pts[i] = p;
	out[i] = u;
}

struct StereoView {
	const float* map_x;
	const float* map_y;
	int height, width;
	Intrinsics I;
	float P[12]; // projection matrix, row-major 3x4
};

// min ||A x - b|| for a 4x3 A, Householder QR in FP64 (cond(A) is ~5-6 for the reference's rigs; the float32 column-pivoting QR of
// the reference, src/oc_stereovision.cpp:115, only adds rounding noise to the same solution)
__device__ __forceinline__ void lsq43(const float (&Af)[4][3], const float (&bf)[4], float* out) {
	double a[4][3], r[4];
#pragma unroll
	for (int i = 0; i < 4; i++) {
		r[i] = bf[i];
#pragma unroll
		for (int j = 0; j < 3; j++) a[i][j] = Af[i][j];
	}
#pragma unroll
	for (int k = 0; k < 3; k++) {
		double nrm = 0.0;
#pragma unroll
		for (int i = k; i < 4; i++) nrm += a[i][k] * a[i][k];
		nrm = sqrt(nrm);
		const double alpha = a[k][k] > 0.0 ? -nrm : nrm;
		double v[4];
#pragma unroll
		for (int i = 0; i < 4; i++) v[i] = i < k ? 0.0 : (i == k ? a[k][k] - alpha : a[i][k]);
		double vv = 0.0;
#pragma unroll
		for (int i = k; i < 4; i++) vv += v[i] * v[i];
		if (vv > 0.0) {
			const double inv = 2.0 / vv;
#pragma unroll
			for (int j = k + 1; j < 3; j++) {
				double s = 0.0;
#pragma unroll
				for (int i = k; i < 4; i++) s += v[i] * a[i][j];
				s *= inv;
#pragma unroll
				for (int i = k; i < 4; i++) a[i][j] -= s * v[i];
			}
			double s = 0.0;
#pragma unroll
			for (int i = k; i < 4; i++) s += v[i] * r[i];
			s *= inv;
#pragma unroll
			for (int i = k; i < 4; i++) r[i] -= s * v[i];
		}
		a[k][k] = alpha;
	}
	const double x2 = r[2] / a[2][2];
	const double x1 = (r[1] - a[1][2] * x2) / a[1][1];
	const double x0 = (r[0] - a[0][1] * x1 - a[0][2] * x2) / a[0][0];
	out[0] = (float)x0;
	out[1] = (float)x1;
	out[2] = (float)x2;
}

// Stereovision::reconstruct(Point2D&, Point2D&) of the pair (*pt1, *pt2) into o[0..2].  NaN in either view: (0, 0, 0), points
// untouched (:72-76).  Otherwise both points are clamped in place and undistorted (:79-80), A and b are formed in float32
// (:87-112) and the least-squares solution is rounded to float.  The one triangulation of stereo_reconstruct_kernel and
// stereo_poi2ds_kernel, so that both give the same bits.
__device__ __forceinline__ void reconstruct_pair(const StereoView& v1, const StereoView& v2, float2* pt1, float2* pt2, float* o) {
	float2 p1 = *pt1, p2 = *pt2;
	if (isnan(p1.x) || isnan(p1.y) || isnan(p2.x) || isnan(p2.y)) {
		o[0] = 0.f;
		o[1] = 0.f;
		o[2] = 0.f;
		return;
	}
	float x1, y1, x2, y2;
	undistort_point(v1.map_x, v1.map_y, v1.height, v1.width, v1.I, &p1.x, &p1.y, &x1, &y1);
	undistort_point(v2.map_x, v2.map_y, v2.height, v2.width, v2.I, &p2.x, &p2.y, &x2, &y2);
	*pt1 = p1;
	*pt2 = p2;
	const float* P = v1.P;
	const float* Q = v2.P;
	float A[4][3], b[4];
#pragma unroll
	for (int j = 0; j < 3; j++) {
		A[0][j] = __fsub_rn(__fmul_rn(x1, P[8 + j]), P[j]);
		A[1][j] = __fsub_rn(__fmul_rn(y1, P[8 + j]), P[4 + j]);
		A[2][j] = __fsub_rn(__fmul_rn(x2, Q[8 + j]), Q[j]);
		A[3][j] = __fsub_rn(__fmul_rn(y2, Q[8 + j]), Q[4 + j]);
	}
	b[0] = __fsub_rn(P[3], __fmul_rn(x1, P[11]));
	b[1] = __fsub_rn(P[7], __fmul_rn(y1, P[11]));
	b[2] = __fsub_rn(Q[3], __fmul_rn(x2, Q[11]));
	b[3] = __fsub_rn(Q[7], __fmul_rn(y2, Q[11]));
	float x[3];
	lsq43(A, b, x);
	o[0] = x[0];
	o[1] = x[1];
	o[2] = x[2];
}

// Stereovision::reconstruct(queue, queue, queue), one thread per point pair.
__global__ void __launch_bounds__(256) stereo_reconstruct_kernel(StereoView v1, StereoView v2, float2* __restrict__ pts1, float2* __restrict__ pts2,
	float* __restrict__ pts3d, long long n) {
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	reconstruct_pair(v1, v2, pts1 + i, pts2 + i, pts3d + 3 * i);
}

// The POI2DS record of POI i in frame f (reference examples/test_3d_dic_epipolar_sift.cpp:193-202, :233-245, :280-290,
// :303-317), one thread per (frame, POI): x, y of the view-1 seed; r2, t1, t2 = location + (u, v) of the stereo record and of
// both registrations, stored before the reconstruction clamps its copies; the three ZNCCs as they are (failure codes too);
// ref_coor = reconstruct((x, y), r2), tar_coor = reconstruct(t1, t2); u, v, w = tar_coor - ref_coor; strain and subset
// radius 0.  Records: stereo and seeds1 n POI2D, out1 / out2 n_frames x n POI2D and out2ds n_frames x n POI2DS, frame-major.
__global__ void __launch_bounds__(256) stereo_poi2ds_kernel(StereoView v1, StereoView v2, const float* __restrict__ stereo,
	const float* __restrict__ seeds1, const float* __restrict__ out1, const float* __restrict__ out2, float* __restrict__ out2ds, long long n,
	long long total) {
	const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= total) return;
	const long long i = t % n;
	const float* s = stereo + i * OCB_POI2D_FLOATS;
	const float* a = out1 + t * OCB_POI2D_FLOATS;
	const float* b = out2 + t * OCB_POI2D_FLOATS;
	const float x = seeds1[i * OCB_POI2D_FLOATS], y = seeds1[i * OCB_POI2D_FLOATS + 1];
	// POI2D: x 0, y 1, u 2, v 8, zncc 16
	const float2 r2 = make_float2(__fadd_rn(s[0], s[2]), __fadd_rn(s[1], s[8]));
	const float2 t1 = make_float2(__fadd_rn(a[0], a[2]), __fadd_rn(a[1], a[8]));
	const float2 t2 = make_float2(__fadd_rn(b[0], b[2]), __fadd_rn(b[1], b[8]));
	float2 c[4] = { make_float2(x, y), r2, t1, t2 };
	float ref[3], tar[3];
	reconstruct_pair(v1, v2, &c[0], &c[1], ref);
	reconstruct_pair(v1, v2, &c[2], &c[3], tar);
	float* o = out2ds + t * OCB_POI2DS_FLOATS;
	o[0] = x;
	o[1] = y;
	for (int k = 0; k < 3; k++) o[2 + k] = __fsub_rn(tar[k], ref[k]);
	o[5] = s[16];
	o[6] = a[16];
	o[7] = b[16];
	o[8] = r2.x;
	o[9] = r2.y;
	o[10] = t1.x;
	o[11] = t1.y;
	o[12] = t2.x;
	o[13] = t2.y;
	for (int k = 0; k < 3; k++) {
		o[14 + k] = ref[k];
		o[17 + k] = tar[k];
	}
	for (int k = 20; k < OCB_POI2DS_FLOATS; k++) o[k] = 0.f;
}

static unsigned int blocks_for(long long n) { return (unsigned int)((n + 255) / 256); }

cudaError_t calib_map_launch(const float* intrinsics, int height, int width, float convergence, int iteration, float* d_map_x, float* d_map_y,
	cudaStream_t stream) {
	calib_map_kernel<<<blocks_for((long long)height * width), 256, 0, stream>>>(load_intrinsics(intrinsics), height, width, convergence, iteration,
		d_map_x, d_map_y);
	return cudaGetLastError();
}

cudaError_t calib_undistort_launch(const float* d_map_x, const float* d_map_y, int height, int width, const float* intrinsics, float* d_pts, float* d_out,
	size_t n, cudaStream_t stream) {
	calib_undistort_kernel<<<blocks_for((long long)n), 256, 0, stream>>>(d_map_x, d_map_y, height, width, load_intrinsics(intrinsics),
		(float2*)d_pts, (float2*)d_out, (long long)n);
	return cudaGetLastError();
}

static void stereo_views(const StereoCam& c1, const StereoCam& c2, StereoView* v) {
	const StereoCam* c[2] = { &c1, &c2 };
	for (int k = 0; k < 2; k++) {
		v[k].map_x = c[k]->map_x;
		v[k].map_y = c[k]->map_y;
		v[k].height = c[k]->height;
		v[k].width = c[k]->width;
		v[k].I = load_intrinsics(c[k]->intrinsics);
		for (int j = 0; j < 12; j++) v[k].P[j] = c[k]->projection[j];
	}
}

cudaError_t stereo_reconstruct_launch(const StereoCam& c1, const StereoCam& c2, float* d_pts1, float* d_pts2, float* d_pts3d, size_t n,
	cudaStream_t stream) {
	StereoView v[2];
	stereo_views(c1, c2, v);
	stereo_reconstruct_kernel<<<blocks_for((long long)n), 256, 0, stream>>>(v[0], v[1], (float2*)d_pts1, (float2*)d_pts2, d_pts3d, (long long)n);
	return cudaGetLastError();
}

cudaError_t stereo_poi2ds_launch(const StereoCam& c1, const StereoCam& c2, const float* d_stereo, const float* d_seeds1, const float* d_out1,
	const float* d_out2, float* d_out2ds, size_t n, int n_frames, cudaStream_t stream) {
	StereoView v[2];
	stereo_views(c1, c2, v);
	const long long total = (long long)n * n_frames;
	stereo_poi2ds_kernel<<<blocks_for(total), 256, 0, stream>>>(v[0], v[1], d_stereo, d_seeds1, d_out1, d_out2, d_out2ds, (long long)n, total);
	return cudaGetLastError();
}

} // namespace ocb
