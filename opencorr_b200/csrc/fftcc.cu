// fftcc.cu -- FFT-accelerated cross-correlation initial guess (integer-pixel displacement + ZNCC)
// for sm_90a.  Replaces FFTCC2D::compute(POI2D*) (reference src/oc_fftcc.cpp:177-275) and
// FFTCC3D::compute(POI3D*) (src/oc_fftcc.cpp:327-427); the FFTW plans/executes the reference
// delegates to (src/oc_fftcc.cpp:40-42,233-243,378-388) are replaced by an in-kernel mixed-radix
// Stockham FFT (radix 4/2/3/5 butterflies, generic odd radix fallback) over shared memory.
//
// One CTA per POI.  The two real windows are packed as z = ref + i*tar, ONE complex transform gives
// both spectra (Hermitian split), C = conj(R) * T is formed in place and ONE inverse transform gives
// the real circular cross-correlation -- half the transforms of the reference's r2c,r2c,c2r.
//   2D: the whole (2ry x 2rx) window lives in shared memory.
//   3D: slab decomposition.  x/y passes run per z-slice in shared memory; the z pass runs on pairs
//       of ky-rows (ky, -ky) so the Hermitian partner of every bin is on chip; slices/rows are
//       exchanged through a per-CTA scratch volume in global memory (at most two CTAs per SM).
#include "fftcc_common.cuh"
#include "ocb_kernels.h"

namespace ocb {

// floor(x / d) for 0 <= x < 2^21 and d >= 1 via one FMUL (inv = 1.0f / d): exact because the
// distance of (x + 0.5) / d to the nearest integer is >= 0.5 / d, far above the fp32 rounding error.
__device__ __forceinline__ int fdiv(int x, float inv) { return __float2int_rz(((float)x + 0.5f) * inv); }

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }

// Per-stage constants of one transform pass, built once per kernel in shared memory so that the
// stage loop holds no integer or float division (they used to cost ~30 % of the 3D kernel).
struct FftStage {
	int r, m, s, tstep, per_batch;
	float inv_pb, inv_s;
};
struct FftPass {
	int n, nstage, bstride;
	FftStage st[16];
};
// s0: element stride of the transformed axis (1 for the contiguous axis); bstride: distance between
// the independent arrays of a batch.  Called by ONE thread; followed by a barrier.
__device__ void fft_build_pass(FftPass* ps, const FftAxis& ax, int s0, int bstride) {
	ps->n = ax.n;
	ps->nstage = ax.nstage;
	ps->bstride = bstride;
	int ncur = ax.n, s = s0;
	for (int st = 0; st < ax.nstage; st++) {
		FftStage& g = ps->st[st];
		g.r = ax.radix[st];
		g.m = ncur / g.r;
		g.s = s;
		g.tstep = ax.n / ncur;
		g.per_batch = g.m * s;
		g.inv_pb = 1.0f / (float)g.per_batch;
		g.inv_s = 1.0f / (float)s;
		ncur = g.m;
		s *= g.r;
	}
}

// All Stockham stages of one pass for `batch` independent arrays, each holding n points with stride
// s0 for every q in [0,s0).  Result ends in `*pin`.  tw: W_n^k = exp(-2 pi i k / n), k in [0,n);
// the inverse uses the conjugate.  Contains __syncthreads(): must be called by the whole CTA.
__device__ void fft_axis(float2** pin, float2** pout, const FftPass& ps, int batch, const float2* __restrict__ tw, bool inverse) {
	float2* in = *pin;
	float2* out = *pout;
	const int n = ps.n, bstride = ps.bstride;
	const float sgn = inverse ? -1.f : 1.f;
	for (int st = 0; st < ps.nstage; st++) {
		const int r = ps.st[st].r, m = ps.st[st].m, s = ps.st[st].s, tstep = ps.st[st].tstep, per_batch = ps.st[st].per_batch;
		const float inv_pb = ps.st[st].inv_pb, inv_s = ps.st[st].inv_s;
		const int total = batch * per_batch;
		for (int t = threadIdx.x; t < total; t += blockDim.x) {
			const int bi = fdiv(t, inv_pb);
			const int rem = t - bi * per_batch;
			const int p = fdiv(rem, inv_s);
			const int q = rem - p * s;
			const float2* src = in + bi * bstride + q + s * p;
			float2* dst = out + bi * bstride + q + s * (r * p);
			const int sm = s * m;
			if (r == 4) {
				float2 a0 = src[0], a1 = src[sm], a2 = src[2 * sm], a3 = src[3 * sm];
				float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), t3 = csub(a1, a3);
				float2 t3r = make_float2(sgn * t3.y, -sgn * t3.x); // t3 * (-i) forward, (+i) inverse
				float2 b0 = cadd(t0, t2), b1 = cadd(t1, t3r), b2 = csub(t0, t2), b3 = csub(t1, t3r);
				float2 w1 = tw[p * tstep], w2 = tw[2 * p * tstep], w3 = tw[3 * p * tstep];
				w1.y *= sgn; w2.y *= sgn; w3.y *= sgn;
				dst[0] = b0;
				dst[s] = cmul(b1, w1);
				dst[2 * s] = cmul(b2, w2);
				dst[3 * s] = cmul(b3, w3);
			} else if (r == 2) {
				float2 a0 = src[0], a1 = src[sm];
				float2 w1 = tw[p * tstep];
				w1.y *= sgn;
				dst[0] = cadd(a0, a1);
				dst[s] = cmul(csub(a0, a1), w1);
			} else if (r == 3) {
				float2 a0 = src[0], a1 = src[sm], a2 = src[2 * sm];
				const float c = -0.5f, sn = -0.86602540378443864676f * sgn; // W_3 = c + i*sn
				float2 t1 = cadd(a1, a2), t2 = csub(a1, a2);
				float2 b0 = cadd(a0, t1);
				float2 mid = make_float2(a0.x + c * t1.x, a0.y + c * t1.y);
				float2 rot = make_float2(-sn * t2.y, sn * t2.x); // i*sn*t2
				float2 b1 = cadd(mid, rot), b2 = csub(mid, rot);
				float2 w1 = tw[p * tstep], w2 = tw[2 * p * tstep];
				w1.y *= sgn; w2.y *= sgn;
				dst[0] = b0;
				dst[s] = cmul(b1, w1);
				dst[2 * s] = cmul(b2, w2);
			} else if (r == 5) {
				// radix 5 (Winograd-style pairing): a1+a4, a2+a3 and their differences
				float2 a0 = src[0], a1 = src[sm], a2 = src[2 * sm], a3 = src[3 * sm], a4 = src[4 * sm];
				const float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;             // cos(2pi/5), cos(4pi/5)
				const float s1 = -0.95105651629515357212f * sgn, s2 = -0.58778525229247312917f * sgn; // -sin(2pi/5), -sin(4pi/5) (forward)
				float2 p1 = cadd(a1, a4), m1 = csub(a1, a4), p2 = cadd(a2, a3), m2 = csub(a2, a3);
				float2 b0 = make_float2(a0.x + p1.x + p2.x, a0.y + p1.y + p2.y);
				float2 e1 = make_float2(a0.x + c1 * p1.x + c2 * p2.x, a0.y + c1 * p1.y + c2 * p2.y);
				float2 e2 = make_float2(a0.x + c2 * p1.x + c1 * p2.x, a0.y + c2 * p1.y + c1 * p2.y);
				// i * (s1 m1 + s2 m2) and i * (s2 m1 - s1 m2)
				float2 o1 = make_float2(-(s1 * m1.y + s2 * m2.y), s1 * m1.x + s2 * m2.x);
				float2 o2 = make_float2(-(s2 * m1.y - s1 * m2.y), s2 * m1.x - s1 * m2.x);
				float2 b1 = cadd(e1, o1), b4 = csub(e1, o1), b2 = cadd(e2, o2), b3 = csub(e2, o2);
				float2 w1 = tw[p * tstep], w2 = tw[2 * p * tstep], w3 = tw[3 * p * tstep], w4 = tw[4 * p * tstep];
				w1.y *= sgn; w2.y *= sgn; w3.y *= sgn; w4.y *= sgn;
				dst[0] = b0;
				dst[s] = cmul(b1, w1);
				dst[2 * s] = cmul(b2, w2);
				dst[3 * s] = cmul(b3, w3);
				dst[4 * s] = cmul(b4, w4);
			} else {
				// generic odd radix (7 ... 31): O(r^2) DFT with table twiddles W_r^k = W_n^(k*n/r)
				float2 a[31];
				const int rstep = n / r;
				for (int k = 0; k < r; k++) a[k] = src[k * sm];
				for (int j = 0; j < r; j++) {
					float2 acc = a[0];
					for (int k = 1; k < r; k++) {
						float2 wr = tw[((j * k) % r) * rstep];
						wr.y *= sgn;
						float2 pr = cmul(a[k], wr);
						acc.x += pr.x;
						acc.y += pr.y;
					}
					float2 wj = tw[p * j * tstep];
					wj.y *= sgn;
					dst[j * s] = (j == 0) ? acc : cmul(acc, wj);
				}
			}
		}
		__syncthreads();
		float2* tmp = in; in = out; out = tmp;
	}
	*pin = in;
	*pout = out;
}

// block-wide sum of two floats; result valid in every thread.  red: >= 64 floats of shared memory.
__device__ __forceinline__ void block_sum2(float& a, float& b, float* red) {
	a = warp_sum(a);
	b = warp_sum(b);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
	__syncthreads();
	if (lane == 0) { red[warp] = a; red[32 + warp] = b; }
	__syncthreads();
	float x = 0.f, y = 0.f;
	for (int i = 0; i < nw; i++) { x += red[i]; y += red[32 + i]; }
	a = x;
	b = y;
}

// block-wide first-maximum argmax; result valid in every thread.  red: >= 64 floats of shared memory.
__device__ __forceinline__ void block_argmax(float& bv, int& bi, float* red) {
	warp_argmax(bv, bi);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
	__syncthreads();
	if (lane == 0) { red[warp] = bv; ((int*)red)[32 + warp] = bi; }
	__syncthreads();
	bv = red[0];
	bi = ((int*)red)[32];
	for (int i = 1; i < nw; i++) argmax_merge(bv, bi, red[i], ((int*)red)[32 + i]);
}

struct Fft2DParams {
	FftAxis ax, ay;
	const float2* tw_x; // device twiddle tables
	const float2* tw_y;
};

__global__ void __launch_bounds__(128) fftcc2d_kernel(Image2D img, float* __restrict__ pois, int n_poi, int rx, int ry, Fft2DParams fp) {
	extern __shared__ __align__(16) float smem_f[];
	const int sw = 2 * rx, sh = 2 * ry, M = sw * sh;
	float2* bufA = (float2*)smem_f;
	float2* bufB = bufA + M;
	float2* twx = bufB + M;
	float2* twy = twx + sw;
	float* red = (float*)(twy + sh);
	__shared__ FftPass pass_x, pass_y;
	for (int i = threadIdx.x; i < sw; i += blockDim.x) twx[i] = fp.tw_x[i];
	for (int i = threadIdx.x; i < sh; i += blockDim.x) twy[i] = fp.tw_y[i];
	if (threadIdx.x == 0) fft_build_pass(&pass_x, fp.ax, 1, sw);
	if (threadIdx.x == 32) fft_build_pass(&pass_y, fp.ay, sw, 0);
	__syncthreads();
	const int w = img.w, h = img.h;
	const float inv_sw = 1.0f / (float)sw;

	for (int poi = blockIdx.x; poi < n_poi; poi += gridDim.x) {
		float* P = pois + (size_t)poi * P2_N;
		const float px = P[P2_X], py = P[P2_Y];
		const float u0 = P[P2_DEF + D2_U], v0 = P[P2_DEF + D2_V];
		if (fftcc2d_skip(px, py, u0, v0, rx, ry, w, h)) continue;
		__syncthreads(); // previous POI's readers of bufA/bufB/red are done
		// fill both windows (src/oc_fftcc.cpp:204-219): float coordinate arithmetic, then (int) truncation
		float sa = 0.f, sb = 0.f;
		for (int i = threadIdx.x; i < M; i += blockDim.x) {
			const int r = fdiv(i, inv_sw), c = i - r * sw;
			const float rpx = px + c - rx, rpy = py + r - ry;
			const float a = __ldg(img.ref + (size_t)(int)rpy * w + (int)rpx);
			const float tpx = rpx + u0, tpy = rpy + v0;
			const float b = __ldg(img.tar + (size_t)(int)tpy * w + (int)tpx);
			bufA[i] = make_float2(a, b);
			sa += a;
			sb += b;
		}
		block_sum2(sa, sb, red);
		const float ref_mean = sa / (float)M, tar_mean = sb / (float)M;
		float na = 0.f, nb = 0.f;
		for (int i = threadIdx.x; i < M; i += blockDim.x) {
			float2 z = bufA[i];
			z.x -= ref_mean;
			z.y -= tar_mean;
			na = fmaf(z.x, z.x, na);
			nb = fmaf(z.y, z.y, nb);
			bufA[i] = z;
		}
		block_sum2(na, nb, red); // ends with __syncthreads-protected reads; bufA complete after its barriers
		float2* in = bufA;
		float2* out = bufB;
		fft_axis(&in, &out, pass_x, sh, twx, false);
		fft_axis(&in, &out, pass_y, 1, twy, false);
		for (int i = threadIdx.x; i < M; i += blockDim.x) {
			const int ky = fdiv(i, inv_sw), kx = i - ky * sw;
			const int j = (ky ? sh - ky : 0) * sw + (kx ? sw - kx : 0);
			float2 z = in[i];
			cross_spectrum(z.x, z.y, in[j].x, in[j].y);
			out[i] = z;
		}
		__syncthreads();
		{ float2* t = in; in = out; out = t; }
		fft_axis(&in, &out, pass_x, sh, twx, true);
		fft_axis(&in, &out, pass_y, 1, twy, true);
		float bv = -2.f;
		int bi = 0;
		for (int i = threadIdx.x; i < M; i += blockDim.x) argmax_merge(bv, bi, in[i].x, i);
		block_argmax(bv, bi, red);
		if (threadIdx.x == 0) fftcc2d_store(P, bv, bi, na, nb, rx, ry, u0, v0);
	}
}

struct Fft3DParams {
	FftAxis ax, ay, az;
	const float2* tw_x;
	const float2* tw_y;
	const float2* tw_z;
	float2* scratch; // gridDim.x volumes of (2rz*2ry*2rx) complex
};

__global__ void __launch_bounds__(256) fftcc3d_kernel(Image3D img, float* __restrict__ pois, int n_poi, int rx, int ry, int rz, Fft3DParams fp) {
	extern __shared__ __align__(16) float smem_f[];
	const int sx = 2 * rx, sy = 2 * ry, sz = 2 * rz;
	const int slice = sx * sy;
	const int rowpair = 2 * sz * sx;
	const int nbuf = slice > rowpair ? slice : rowpair;
	const size_t M = (size_t)slice * sz;
	float2* bufA = (float2*)smem_f;
	float2* bufB = bufA + nbuf;
	float2* twx = bufB + nbuf;
	float2* twy = twx + sx;
	float2* twz = twy + sy;
	float* red = (float*)(twz + sz);
	for (int i = threadIdx.x; i < sx; i += blockDim.x) twx[i] = fp.tw_x[i];
	for (int i = threadIdx.x; i < sy; i += blockDim.x) twy[i] = fp.tw_y[i];
	for (int i = threadIdx.x; i < sz; i += blockDim.x) twz[i] = fp.tw_z[i];
	__shared__ FftPass pass_x, pass_y, pass_z;
	if (threadIdx.x == 0) fft_build_pass(&pass_x, fp.ax, 1, sx);
	if (threadIdx.x == 32) fft_build_pass(&pass_y, fp.ay, sx, 0);
	if (threadIdx.x == 64) fft_build_pass(&pass_z, fp.az, sx, sz * sx);
	__syncthreads();
	float2* S = fp.scratch + (size_t)blockIdx.x * M;
	const int dx = img.dx, dy = img.dy, dz = img.dz;
	const float inv_sx = 1.0f / (float)sx, inv_rowp = 1.0f / (float)(sz * sx);

	for (int poi = blockIdx.x; poi < n_poi; poi += gridDim.x) {
		float* P = pois + (size_t)poi * P3_N;
		const float px = P[P3_X], py = P[P3_Y], pz = P[P3_Z];
		const float u0 = P[P3_DEF + 0], v0 = P[P3_DEF + 4], w0 = P[P3_DEF + 8];
		if (fftcc3d_skip(px, py, pz, u0, v0, w0, rx, ry, rz, dx, dy, dz)) continue;
		__syncthreads();
		// pass 0: means (src/oc_fftcc.cpp:346-367)
		float sa = 0.f, sb = 0.f;
		for (int ii = 0; ii < sz; ii++) {
			const float rpz = pz + ii - rz;
			const float tpz = rpz + w0;
			for (int i = threadIdx.x; i < slice; i += blockDim.x) {
				const int j = fdiv(i, inv_sx), k = i - j * sx;
				const float rpx = px + k - rx, rpy = py + j - ry;
				sa += __ldg(img.ref + ((size_t)(int)rpz * dy + (int)rpy) * dx + (int)rpx);
				const float tpx = rpx + u0, tpy = rpy + v0;
				sb += __ldg(img.tar + ((size_t)(int)tpz * dy + (int)tpy) * dx + (int)tpx);
			}
		}
		block_sum2(sa, sb, red);
		const float ref_mean = sa / (float)M, tar_mean = sb / (float)M;
		// phase A: per z-slice, zero-mean fill + x,y transforms, slice -> scratch
		float na = 0.f, nb = 0.f;
		for (int ii = 0; ii < sz; ii++) {
			const float rpz = pz + ii - rz;
			const float tpz = rpz + w0;
			for (int i = threadIdx.x; i < slice; i += blockDim.x) {
				const int j = fdiv(i, inv_sx), k = i - j * sx;
				const float rpx = px + k - rx, rpy = py + j - ry;
				float a = __ldg(img.ref + ((size_t)(int)rpz * dy + (int)rpy) * dx + (int)rpx) - ref_mean;
				const float tpx = rpx + u0, tpy = rpy + v0;
				float b = __ldg(img.tar + ((size_t)(int)tpz * dy + (int)tpy) * dx + (int)tpx) - tar_mean;
				na = fmaf(a, a, na);
				nb = fmaf(b, b, nb);
				bufA[i] = make_float2(a, b);
			}
			__syncthreads();
			float2* in = bufA;
			float2* out = bufB;
			fft_axis(&in, &out, pass_x, sy, twx, false);
			fft_axis(&in, &out, pass_y, 1, twy, false);
			float2* dst = S + (size_t)ii * slice;
			for (int i = threadIdx.x; i < slice; i += blockDim.x) dst[i] = in[i];
			__syncthreads();
		}
		block_sum2(na, nb, red);
		// phase B: z transform, cross spectrum, inverse z transform on row pairs (ky, -ky)
		for (int ky = 0; ky <= sy / 2; ky++) {
			const int kyn = (sy - ky) % sy;
			const int nrow = (kyn == ky) ? 1 : 2;
			for (int i = threadIdx.x; i < nrow * sz * sx; i += blockDim.x) {
				const int rs = fdiv(i, inv_rowp);
				const int rem = i - rs * sz * sx;
				const int kz = fdiv(rem, inv_sx), kx = rem - kz * sx;
				bufA[i] = __ldcg(S + ((size_t)kz * sy + (rs ? kyn : ky)) * sx + kx);
			}
			__syncthreads();
			float2* in = bufA;
			float2* out = bufB;
			fft_axis(&in, &out, pass_z, nrow, twz, false);
			for (int i = threadIdx.x; i < nrow * sz * sx; i += blockDim.x) {
				const int rs = fdiv(i, inv_rowp);
				const int rem = i - rs * sz * sx;
				const int kz = fdiv(rem, inv_sx), kx = rem - kz * sx;
				const int prs = (nrow == 2) ? 1 - rs : 0;
				const int j = prs * sz * sx + (kz ? sz - kz : 0) * sx + (kx ? sx - kx : 0);
				float2 z = in[i];
			cross_spectrum(z.x, z.y, in[j].x, in[j].y);
			out[i] = z;
			}
			__syncthreads();
			{ float2* t = in; in = out; out = t; }
			fft_axis(&in, &out, pass_z, nrow, twz, true);
			for (int i = threadIdx.x; i < nrow * sz * sx; i += blockDim.x) {
				const int rs = fdiv(i, inv_rowp);
				const int rem = i - rs * sz * sx;
				const int kz = fdiv(rem, inv_sx), kx = rem - kz * sx;
				S[((size_t)kz * sy + (rs ? kyn : ky)) * sx + kx] = in[i];
			}
			__syncthreads();
		}
		// phase C: inverse x,y transforms per slice + running argmax
		float bv = -2.f;
		int bi = 0;
		for (int ii = 0; ii < sz; ii++) {
			const float2* src = S + (size_t)ii * slice;
			for (int i = threadIdx.x; i < slice; i += blockDim.x) bufA[i] = __ldcg(src + i);
			__syncthreads();
			float2* in = bufA;
			float2* out = bufB;
			fft_axis(&in, &out, pass_y, 1, twy, true);
			fft_axis(&in, &out, pass_x, sy, twx, true);
			for (int i = threadIdx.x; i < slice; i += blockDim.x) argmax_merge(bv, bi, in[i].x, ii * slice + i);
			__syncthreads();
		}
		block_argmax(bv, bi, red);
		if (threadIdx.x == 0) fftcc3d_store(P, bv, bi, na, nb, rx, ry, rz, u0, v0, w0);
	}
}

// host side ------------------------------------------------------------------------------------
cudaError_t fftcc2d_launch(const Image2D& img, float* d_pois, size_t n, int rx, int ry, const Fftcc2dPlan& plan, const float2* tw_x,
	const float2* tw_y, int grid, cudaStream_t stream) {
	Fft2DParams fp;
	fp.ax = plan.ax; fp.ay = plan.ay; fp.tw_x = tw_x; fp.tw_y = tw_y;
	return launch_smem(fftcc2d_kernel, grid, 128, plan.smem, stream, img, d_pois, (int)n, rx, ry, fp);
}

cudaError_t fftcc3d_launch(const Image3D& img, float* d_pois, size_t n, int rx, int ry, int rz, const Fftcc3dPlan& plan, const float2* tw_x,
	const float2* tw_y, const float2* tw_z, float2* scratch, int grid, cudaStream_t stream) {
	Fft3DParams fp;
	fp.ax = plan.ax; fp.ay = plan.ay; fp.az = plan.az;
	fp.tw_x = tw_x; fp.tw_y = tw_y; fp.tw_z = tw_z;
	fp.scratch = scratch;
	return launch_smem(fftcc3d_kernel, grid, 256, plan.smem, stream, img, d_pois, (int)n, rx, ry, rz, fp);
}

} // namespace ocb
