// icgn2d.cu -- inverse-compositional Gauss-Newton subset registration, 2D, first-order (6
// parameters) and second-order (12 parameters) shape functions, for sm_90a.
//
// Replaces ICGN2D1::compute(POI2D*) (reference src/oc_icgn.cpp:144-341) and
// ICGN2D2::compute(POI2D*) (src/oc_icgn.cpp:685-898), including what ICGN2D*::prepare() feeds
// them (Gradient2D4, src/oc_gradient.cpp:37-79; BicubicBspline, src/oc_cubic_bspline.cpp:84-181).
//
// Structure in one paragraph: the setup pass and the sampling loop take one subset row per lane and step, and a lane's
// per-sample constants live in shared memory.  The reference's `any sample < 0` rejection is
// re-decided in the reference's own arithmetic when the smallest sample is borderline (icgn2d_exact_negative).  What follows
// describes the common skeleton.
//
// Mapping: ONE WARP PER POI, persistent warps pulling POIs from an atomic counter, no CTA barrier.
// Lanes run along x: lane c owns column c of the subset for every row (columns >= 32 are a short
// tail), so x-dependent factors are per-lane constants and y-dependent ones are warp-uniform.
//   stage   : the reference tile (subset + 2-pixel gradient halo) is staged in the warp's smem slab.
//   setup   : one pass computes R' = R - c0 (c0 = centre pixel, a pilot value that keeps every sum
//             well conditioned), the 4th-order gradients gx, gy (recomputed from the image, nothing
//             precomputed in HBM) and stores them to smem; the Hessian is accumulated as FACTORED
//             sums  sum g_a g_b y^Q  (x^P applied once per lane afterwards), so a sample costs 15
//             (6-parameter) / 30 (12-parameter) flops instead of 21 / 78 FMAs.  Mean and norm of the
//             reference subset come from the same pass.  Cholesky factorisation in registers.
//   iterate : the target tile (subset + bicubic support + slack), minus c0, replaces the reference
//             tile in the slab.  Each iteration evaluates the bicubic interpolant from the 4x4 pixel
//             block with explicit fp32 weights (the reference's 64 B/pixel LUT is never built) and
//             accumulates ONE pass of sums with d = t - R:  sum d, sum d^2, sum R'd, sum g_a d y^Q;
//             mean/norm of the warped target, ZNSSD and the Gauss-Newton right-hand side follow
//             algebraically (DESIGN.md "single-pass IC-GN sums").  The 4x4 blocks roll down each lane's column in
//             registers: a row whose block is the previous one moved down a pixel row reads only its new bottom row.
//   update  : solve with the Cholesky factors, compose W <- W * W(dp)^-1 in registers.
// Samples whose 4x4 support leaves the staged tile (large deformation gradients) are read from
// global memory instead, so results never depend on the tile size.
#include <type_traits>

#include "ocb_kernels.h"
#include "ocb_tma.cuh"
#include "ocb_tile2d.cuh"

namespace ocb {

constexpr int ICGN2D_MIN_CTAS = 16; // resident one-warp CTAs the 6-parameter kernels' register budget is sized for (16 -> 128 registers)
constexpr int ICGN2D_ROW_UNROLL = 3; // rows in flight per lane: whole-pixel loop, 12-parameter sampling loop
// tile extents and the slab layout (icgn2d_ref_w .. icgn2d_slab_floats) and the launch plan are in ocb_kernels.h

// Shape functions: sd = g_a * phi_i, phi = [1, x, y, x^2/2, xy, y^2/2] (first 3 for NP == 6);
// phi_i = c_i x^p_i y^q_i  (reference src/oc_icgn.cpp:191-196, :725-745)
__host__ __device__ constexpr int phi_p(int i) { return i == 1 ? 1 : (i == 3 ? 2 : (i == 4 ? 1 : 0)); }
__host__ __device__ constexpr int phi_q(int i) { return i == 2 ? 1 : (i == 4 ? 1 : (i == 5 ? 2 : 0)); }
__host__ __device__ constexpr float phi_c(int i) { return (i == 3 || i == 5) ? 0.5f : 1.f; }
// index of monomial x^P y^Q among all monomials ordered by total degree then Q
__host__ __device__ constexpr int mono(int P, int Q) { return (P + Q) * (P + Q + 1) / 2 + Q; }
__host__ __device__ constexpr int pair_idx(int a, int b) { return a + b; } // (x,x)=0 (x,y)=1 (y,y)=2

__device__ __forceinline__ float ipow(float x, int p) {
	float r = 1.f;
#pragma unroll
	for (int i = 0; i < 4; i++)
		if (i < p) r *= x;
	return r;
}

// ---- per-lane sums, one flat array each -------------------------------------------------------------------------------
// Samples come in two kinds: row-mapped ones, where x is the lane's own column and y is the same for the whole warp, and
// tail ones with general x and y.  A row-mapped sample adds y powers only; expand() then applies the lane's powers of x once
// (column slots, below), and tail samples add into the expanded slots directly.

// The setup pass (R' = R - c0, gradients g = (gx, gy)):
//   R1: sum R'   R2: sum R'^2
//   M + a NM + mono(P, Q): sum gg_a x^P y^Q, gg = (gx gx, gx gy, gy gy)    (column slots: M + a (D2 + 1) + Q, sum gg_a y^Q)
//   SG + a NPHI + i: sum g_a x^p_i y^q_i                                    (column slots: SG + a (DEG + 1) + q, sum g_a y^q)
//   SRG + a NPHI + i: sum g_a R' x^p_i y^q_i                                (column slots: SRG + a (DEG + 1) + q)
template <int DEG>
struct SetupSums {
	static constexpr int D2 = 2 * DEG, NM = (D2 + 1) * (D2 + 2) / 2, NPHI = 3 * DEG;
	static constexpr int R1 = 0, R2 = 1, M = 2, SG = M + 3 * NM, SRG = SG + 2 * NPHI, N = SRG + 2 * NPHI;
	static_assert(N <= ICGN2D_RED_SETUP, "setup partials do not fit");
	float v[N];
	__device__ __forceinline__ SetupSums() {
#pragma unroll
		for (int i = 0; i < N; i++) v[i] = 0.f;
	}
	__device__ __forceinline__ void add_row(float R, float gx, float gy, float yl) {
		v[R1] += R;
		v[R2] = fmaf(R, R, v[R2]);
		float g[3] = { gx * gx, gx * gy, gy * gy };
#pragma unroll
		for (int a = 0; a < 3; a++) {
			float t = g[a];
#pragma unroll
			for (int qq = 0; qq <= D2; qq++) {
				v[M + a * (D2 + 1) + qq] += t;
				if (qq < D2) t *= yl;
			}
		}
		float g1[2] = { gx, gy };
#pragma unroll
		for (int a = 0; a < 2; a++) {
			float t = g1[a], tr = g1[a] * R;
#pragma unroll
			for (int qq = 0; qq <= DEG; qq++) {
				v[SG + a * (DEG + 1) + qq] += t;
				v[SRG + a * (DEG + 1) + qq] += tr;
				if (qq < DEG) { t *= yl; tr *= yl; }
			}
		}
	}
	__device__ __forceinline__ void expand(float xl) {
		float c[N], xp[D2 + 1];
#pragma unroll
		for (int i = 0; i < N; i++) c[i] = v[i];
		xp[0] = 1.f;
#pragma unroll
		for (int p = 1; p <= D2; p++) xp[p] = xp[p - 1] * xl;
#pragma unroll
		for (int Pp = 0; Pp <= D2; Pp++)
#pragma unroll
			for (int Q = 0; Q <= D2; Q++)
				if (Pp + Q <= D2) {
#pragma unroll
					for (int a = 0; a < 3; a++) v[M + a * NM + mono(Pp, Q)] = xp[Pp] * c[M + a * (D2 + 1) + Q];
				}
#pragma unroll
		for (int i = 0; i < NPHI; i++)
#pragma unroll
			for (int a = 0; a < 2; a++) {
				v[SG + a * NPHI + i] = xp[phi_p(i)] * c[SG + a * (DEG + 1) + phi_q(i)];
				v[SRG + a * NPHI + i] = xp[phi_p(i)] * c[SRG + a * (DEG + 1) + phi_q(i)];
			}
	}
	__device__ __forceinline__ void add(float R, float gx, float gy, float xl, float yl) {
		v[R1] += R;
		v[R2] = fmaf(R, R, v[R2]);
		float g[3] = { gx * gx, gx * gy, gy * gy };
		float g1[2] = { gx, gy };
#pragma unroll
		for (int Pp = 0; Pp <= D2; Pp++)
#pragma unroll
			for (int Q = 0; Q <= D2; Q++)
				if (Pp + Q <= D2) {
					const float mm = ipow(xl, Pp) * ipow(yl, Q);
#pragma unroll
					for (int a = 0; a < 3; a++) v[M + a * NM + mono(Pp, Q)] = fmaf(g[a], mm, v[M + a * NM + mono(Pp, Q)]);
				}
#pragma unroll
		for (int ii = 0; ii < NPHI; ii++) {
			const float mm = ipow(xl, phi_p(ii)) * ipow(yl, phi_q(ii));
#pragma unroll
			for (int a = 0; a < 2; a++) {
				v[SG + a * NPHI + ii] = fmaf(g1[a], mm, v[SG + a * NPHI + ii]);
				v[SRG + a * NPHI + ii] = fmaf(g1[a] * R, mm, v[SRG + a * NPHI + ii]);
			}
		}
	}
	__device__ __forceinline__ void reduce() {
#pragma unroll
		for (int i = 0; i < N; i++) v[i] = warp_sum(v[i]);
	}
};

// One IC-GN pass (d = t - R with the raw R, sd_k = g_a phi_i for k = a NPHI + i):
//   D1: sum d   D2: sum d^2   RD: sum R d
//   INV: not a sum; carries the warp's "a sample is invalid" flag through the combine of WPP > 1
//   SD + k: sum sd_k d                            (column slots: SD + a (DEG + 1) + q, sum g_a d y^q)
template <int DEG>
struct PassSums {
	static constexpr int NPHI = 3 * DEG;
	static constexpr int D1 = 0, D2 = 1, RD = 2, INV = 3, SD = 4, N = SD + 2 * NPHI;
	static_assert(N <= ICGN2D_RED_ITER, "iteration partials do not fit");
	float v[N];
	__device__ __forceinline__ PassSums() {
#pragma unroll
		for (int i = 0; i < N; i++) v[i] = 0.f;
	}
	__device__ __forceinline__ void add_row(float d, float R, float gx, float gy, float yl) {
		v[D1] += d;
		v[D2] = fmaf(d, d, v[D2]);
		v[RD] = fmaf(R, d, v[RD]);
		float gd[2] = { gx * d, gy * d };
#pragma unroll
		for (int a = 0; a < 2; a++) {
			float tt = gd[a];
#pragma unroll
			for (int qq = 0; qq <= DEG; qq++) {
				v[SD + a * (DEG + 1) + qq] += tt;
				if (qq < DEG) tt *= yl;
			}
		}
	}
	__device__ __forceinline__ void expand(float xl) {
		float c[N], xp[DEG + 1];
#pragma unroll
		for (int i = 0; i < N; i++) c[i] = v[i];
		xp[0] = 1.f;
#pragma unroll
		for (int p = 1; p <= DEG; p++) xp[p] = xp[p - 1] * xl;
#pragma unroll
		for (int a = 0; a < 2; a++)
#pragma unroll
			for (int i = 0; i < NPHI; i++) v[SD + a * NPHI + i] = phi_c(i) * xp[phi_p(i)] * c[SD + a * (DEG + 1) + phi_q(i)];
	}
	__device__ __forceinline__ void add(float d, float R, float gx, float gy, float xl, float yl) {
		v[D1] += d;
		v[D2] = fmaf(d, d, v[D2]);
		v[RD] = fmaf(R, d, v[RD]);
		float gd[2] = { gx * d, gy * d };
#pragma unroll
		for (int ii = 0; ii < NPHI; ii++) {
			const float mm = phi_c(ii) * ipow(xl, phi_p(ii)) * ipow(yl, phi_q(ii));
#pragma unroll
			for (int a = 0; a < 2; a++) v[SD + a * NPHI + ii] = fmaf(gd[a], mm, v[SD + a * NPHI + ii]);
		}
	}
	__device__ __forceinline__ void reduce() {
#pragma unroll
		for (int i = 0; i < N; i++)
			if (i != INV) v[i] = warp_sum(v[i]);
	}
};

// WPP > 1: every warp of the POI leaves its partial sums in the slab (red: [WPP][stride]) and then adds all of them in the
// same order, so every warp holds the same totals.
template <int WPP, int N>
__device__ __forceinline__ void combine_warps(float (&v)[N], float* red, int stride, int sub, int lane) {
	if (lane == 0) {
#pragma unroll
		for (int i = 0; i < N; i++) red[sub * stride + i] = v[i];
	}
	__syncthreads();
#pragma unroll
	for (int i = 0; i < N; i++) v[i] = 0.f;
#pragma unroll
	for (int ww = 0; ww < WPP; ww++)
#pragma unroll
		for (int i = 0; i < N; i++) v[i] += red[ww * stride + i];
}

// W(p) of the second-order shape function (reference src/oc_deformation.cpp:301-350)
__device__ __forceinline__ void warp2d2_matrix(const float* p, float* W) {
	const float u = p[0], ux = p[1], uy = p[2], uxx = p[3], uxy = p[4], uyy = p[5];
	const float v = p[6], vx = p[7], vy = p[8], vxx = p[9], vxy = p[10], vyy = p[11];
	W[0] = 1.f + 2.f * ux + ux * ux + u * uxx;
	W[1] = 2.f * u * uxy + 2.f * (1.f + ux) * uy;
	W[2] = uy * uy + u * uyy;
	W[3] = 2.f * u * (1.f + ux);
	W[4] = 2.f * u * uy;
	W[5] = u * u;
	W[6] = 0.5f * (v * uxx + 2.f * (1.f + ux) * vx + u * vxx);
	W[7] = 1.f + uy * vx + ux * vy + v * uxy + u * vxy + vy + ux;
	W[8] = 0.5f * (v * uyy + 2.f * uy * (1.f + vy) + u * vyy);
	W[9] = v + v * ux + u * vx;
	W[10] = u + v * uy + u * vy;
	W[11] = u * v;
	W[12] = vx * vx + v * vxx;
	W[13] = 2.f * v * vxy + 2.f * vx * (1.f + vy);
	W[14] = 1.f + 2.f * vy + vy * vy + v * vyy;
	W[15] = 2.f * v * vx;
	W[16] = 2.f * v * (1.f + vy);
	W[17] = v * v;
	W[18] = 0.5f * uxx; W[19] = uxy; W[20] = 0.5f * uyy; W[21] = 1.f + ux; W[22] = uy; W[23] = u;
	W[24] = 0.5f * vxx; W[25] = vxy; W[26] = 0.5f * vyy; W[27] = vx; W[28] = 1.f + vy; W[29] = v;
	// row 5 = [0 0 0 0 0 1] is implicit
}

// rows <- rows * M^-1 for the 2x6 block `rows` (rows 3,4 of the running warp) and the 6x6 warp
// increment M whose last row is [0 0 0 0 0 1] (given as its first 5 rows, 30 floats).
// Gaussian elimination without pivoting: M = W(dp) is a perturbation of the identity.
// X M = R: reduce M = L U (unit lower L), Y U = R by forward substitution over columns, X = Y L^-1.
__device__ __forceinline__ void right_divide_2x6(float* rows, float* M) {
	float Lm[5][5];
#pragma unroll
	for (int k = 0; k < 5; k++) {
		float inv = 1.0f / M[k * 6 + k];
#pragma unroll
		for (int i = k + 1; i < 5; i++) {
			float l = M[i * 6 + k] * inv;
			Lm[i][k] = l;
#pragma unroll
			for (int j = k + 1; j < 6; j++) M[i * 6 + j] -= l * M[k * 6 + j];
		}
	}
#pragma unroll
	for (int r = 0; r < 2; r++) {
		float y[6];
#pragma unroll
		for (int j = 0; j < 6; j++) {
			float v = rows[r * 6 + j];
#pragma unroll
			for (int i = 0; i < j; i++) {
				if (i < 5) v -= y[i] * M[i * 6 + j];
			}
			y[j] = (j < 5) ? v / M[j * 6 + j] : v;
		}
#pragma unroll
		for (int k = 4; k >= 0; k--) {
			float v = y[k];
#pragma unroll
			for (int i = k + 1; i < 5; i++) v -= y[i] * Lm[i][k];
			y[k] = v;
		}
#pragma unroll
		for (int j = 0; j < 6; j++) rows[r * 6 + j] = y[j];
	}
}

// ---- the running warp, one type per shape-function order ----------------------------------------------------------------
// A sample at local (x, y) lands at (pcx, pcy) + warped offset.  The warped offset is formed first and the POI centre added
// last, with ONE rounding at the large magnitude, like the reference's `center + warped` (src/oc_icgn.cpp:238-239): at
// x ~ 4096 a float ulp is 4.9e-4 px, so the association order is visible in the result.

// First order (Deformation2D1, src/oc_deformation.cpp:94-128): A = W00 W01 W02 W10 W11 W12.
struct Warp2D1 {
	static constexpr int NA = 6;
	float A[NA];
	__device__ __forceinline__ void init(float u, float ux, float uy, float v, float vx, float vy) {
		A[0] = 1.f + ux; A[1] = uy; A[2] = u; A[3] = vx; A[4] = 1.f + vy; A[5] = v;
	}
	// a lane's column at local x: X = pcx + (x1 y + x0), Y = pcy + (y1 y + y0)
	struct Column {
		float x0, x1, y0, y1;
		__device__ __forceinline__ void at(float pcx, float pcy, float yl, float& X, float& Y) const {
			X = pcx + fmaf(x1, yl, x0);
			Y = pcy + fmaf(y1, yl, y0);
		}
	};
	__device__ __forceinline__ Column column(float xl) const { return { fmaf(A[0], xl, A[2]), A[1], fmaf(A[3], xl, A[5]), A[4] }; }
	__device__ __forceinline__ void at(float pcx, float pcy, float xl, float yl, float& X, float& Y) const {
		X = pcx + fmaf(A[0], xl, fmaf(A[1], yl, A[2]));
		Y = pcy + fmaf(A[3], xl, fmaf(A[4], yl, A[5]));
	}
	// warp_matrix * (x, y, 1) in the reference's arithmetic: products summed left to right
	__device__ __forceinline__ void reference_offset(float xl, float yl, float& wx, float& wy) const {
		wx = __fadd_rn(__fadd_rn(__fmul_rn(A[0], xl), __fmul_rn(A[1], yl)), A[2]);
		wy = __fadd_rn(__fadd_rn(__fmul_rn(A[3], xl), __fmul_rn(A[4], yl)), A[5]);
	}
	// centre (cx, cy) and half-extents (ex, ey) of the parallelogram that the subset [-fx, fx] x [-fy, fy] maps to
	__device__ __forceinline__ void bounds(float pcx, float pcy, float fx, float fy, float& cx, float& cy, float& ex, float& ey) const {
		cx = pcx + A[2];
		cy = pcy + A[5];
		ex = fabsf(A[0]) * fx + fabsf(A[1]) * fy;
		ey = fabsf(A[3]) * fx + fabsf(A[4]) * fy;
	}
	// is the warp a translation, and by (kx, ky)?
	__device__ __forceinline__ bool translation(float& kx, float& ky) const {
		kx = A[2];
		ky = A[5];
		return A[0] == 1.f && A[1] == 0.f && A[3] == 0.f && A[4] == 1.f;
	}
	// W <- W * W(dp)^-1, 3x3 affine (src/oc_icgn.cpp:290)
	__device__ __forceinline__ void compose_inverse(const float* dp, bool accept) {
		const float a = dp[1], bb = dp[2], cc = dp[0], d = dp[4], e = dp[5], ff = dp[3];
		const float det = (1.f + a) * (1.f + e) - bb * d;
		const float id = 1.0f / det;
		const float i00 = (1.f + e) * id, i01 = -bb * id, i02 = (bb * ff - cc * (1.f + e)) * id;
		const float i10 = -d * id, i11 = (1.f + a) * id, i12 = (cc * d - (1.f + a) * ff) * id;
		const float n00 = A[0] * i00 + A[1] * i10, n01 = A[0] * i01 + A[1] * i11, n02 = A[0] * i02 + A[1] * i12 + A[2];
		const float n10 = A[3] * i00 + A[4] * i10, n11 = A[3] * i01 + A[4] * i11, n12 = A[3] * i02 + A[4] * i12 + A[5];
		if (accept) { A[0] = n00; A[1] = n01; A[2] = n02; A[3] = n10; A[4] = n11; A[5] = n12; }
	}
	// ||dp||^2 with the subset radii (src/oc_icgn.cpp:296-306)
	__device__ __forceinline__ static float dp_norm2(const float* dp, int rx, int ry) {
		const float rx2 = (float)(rx * rx), ry2 = (float)(ry * ry);
		return dp[0] * dp[0] + dp[1] * dp[1] * rx2 + dp[2] * dp[2] * ry2
			+ dp[3] * dp[3] + dp[4] * dp[4] * rx2 + dp[5] * dp[5] * ry2;
	}
	__device__ __forceinline__ float u() const { return A[2]; }
	__device__ __forceinline__ float v() const { return A[5]; }
	template <class Put>
	__device__ __forceinline__ void put_fields(Put put) const {
		put(P2_DEF + D2_U, A[2]); put(P2_DEF + D2_UX, A[0] - 1.f); put(P2_DEF + D2_UY, A[1]);
		put(P2_DEF + D2_V, A[5]); put(P2_DEF + D2_VX, A[3]); put(P2_DEF + D2_VY, A[4] - 1.f);
	}
};

// Second order (Deformation2D2, src/oc_deformation.cpp:268-350): A = rows 3 and 4 of the 6x6 warp, the rows that map
// (x^2, xy, y^2, x, y, 1) to X and Y.
struct Warp2D2 {
	static constexpr int NA = 12;
	float A[NA];
	// second-order terms of the incoming guess are dropped (src/oc_icgn.cpp:765-770)
	__device__ __forceinline__ void init(float u, float ux, float uy, float v, float vx, float vy) {
		A[0] = 0.f; A[1] = 0.f; A[2] = 0.f; A[3] = 1.f + ux; A[4] = uy; A[5] = u;
		A[6] = 0.f; A[7] = 0.f; A[8] = 0.f; A[9] = vx; A[10] = 1.f + vy; A[11] = v;
	}
	// a lane's column at local x: X = pcx + (x2 y^2 + x1 y + x0), Y likewise
	struct Column {
		float x0, x1, x2, y0, y1, y2;
		__device__ __forceinline__ void at(float pcx, float pcy, float yl, float& X, float& Y) const {
			X = pcx + fmaf(fmaf(x2, yl, x1), yl, x0);
			Y = pcy + fmaf(fmaf(y2, yl, y1), yl, y0);
		}
	};
	__device__ __forceinline__ Column column(float xl) const {
		return { fmaf(A[0] * xl + A[3], xl, A[5]), fmaf(A[1], xl, A[4]), A[2], fmaf(A[6] * xl + A[9], xl, A[11]), fmaf(A[7], xl, A[10]), A[8] };
	}
	__device__ __forceinline__ void at(float pcx, float pcy, float xl, float yl, float& X, float& Y) const {
		const float m0 = xl * xl, m1 = xl * yl, m2 = yl * yl;
		X = pcx + fmaf(A[0], m0, fmaf(A[1], m1, fmaf(A[2], m2, fmaf(A[3], xl, fmaf(A[4], yl, A[5])))));
		Y = pcy + fmaf(A[6], m0, fmaf(A[7], m1, fmaf(A[8], m2, fmaf(A[9], xl, fmaf(A[10], yl, A[11])))));
	}
	// rows 3, 4 of warp_matrix * (x^2, xy, y^2, x, y, 1) in the reference's arithmetic, src/oc_deformation.cpp:268-282
	__device__ __forceinline__ void reference_offset(float xl, float yl, float& wx, float& wy) const {
		const float v0 = __fmul_rn(xl, xl), v1 = __fmul_rn(xl, yl), v2 = __fmul_rn(yl, yl);
		wx = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A[0], v0), __fmul_rn(A[1], v1)), __fmul_rn(A[2], v2)), __fmul_rn(A[3], xl)),
					__fmul_rn(A[4], yl)), A[5]);
		wy = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A[6], v0), __fmul_rn(A[7], v1)), __fmul_rn(A[8], v2)), __fmul_rn(A[9], xl)),
					__fmul_rn(A[10], yl)), A[11]);
	}
	// as Warp2D1::bounds; the second-order part is bounded by qx, qy and widens the parallelogram
	__device__ __forceinline__ void bounds(float pcx, float pcy, float fx, float fy, float& cx, float& cy, float& ex, float& ey) const {
		const float qx = fabsf(A[0]) * fx * fx + fabsf(A[1]) * fx * fy + fabsf(A[2]) * fy * fy;
		const float qy = fabsf(A[6]) * fx * fx + fabsf(A[7]) * fx * fy + fabsf(A[8]) * fy * fy;
		cx = pcx + A[5];
		cy = pcy + A[11];
		ex = fabsf(A[3]) * fx + fabsf(A[4]) * fy + qx;
		ey = fabsf(A[9]) * fx + fabsf(A[10]) * fy + qy;
	}
	__device__ __forceinline__ bool translation(float& kx, float& ky) const {
		kx = A[5];
		ky = A[11];
		return A[0] == 0.f && A[1] == 0.f && A[2] == 0.f && A[3] == 1.f && A[4] == 0.f
			&& A[6] == 0.f && A[7] == 0.f && A[8] == 0.f && A[9] == 0.f && A[10] == 1.f;
	}
	// rows 3,4 of W * W(dp)^-1 (src/oc_icgn.cpp:831)
	__device__ __forceinline__ void compose_inverse(const float* dp, bool accept) {
		if (accept) {
			float Mw[30];
			warp2d2_matrix(dp, Mw);
			right_divide_2x6(A, Mw);
		}
	}
	__device__ __forceinline__ static float dp_norm2(const float* dp, int rx, int ry) {
		const int rx2 = rx * rx, ry2 = ry * ry;
		const float rxy2 = (float)(rx2 * ry2);
		const float rx4 = (float)(int)((float)(rx2 * rx2) * 0.25f); // float->int truncation, src/oc_icgn.cpp:840-841
		const float ry4 = (float)(int)((float)(ry2 * ry2) * 0.25f);
		return dp[0] * dp[0] + dp[1] * dp[1] * (float)rx2 + dp[2] * dp[2] * (float)ry2
			+ dp[3] * dp[3] * rx4 + dp[5] * dp[5] * ry4 + dp[4] * dp[4] * rxy2
			+ dp[6] * dp[6] + dp[7] * dp[7] * (float)rx2 + dp[8] * dp[8] * (float)ry2
			+ dp[9] * dp[9] * rx4 + dp[11] * dp[11] * ry4 + dp[10] * dp[10] * rxy2;
	}
	__device__ __forceinline__ float u() const { return A[5]; }
	__device__ __forceinline__ float v() const { return A[11]; }
	// Deformation2D2::setDeformation(), src/oc_deformation.cpp:284-299
	template <class Put>
	__device__ __forceinline__ void put_fields(Put put) const {
		put(P2_DEF + D2_U, A[5]); put(P2_DEF + D2_UX, A[3] - 1.f); put(P2_DEF + D2_UY, A[4]);
		put(P2_DEF + D2_UXX, A[0] * 2.f); put(P2_DEF + D2_UXY, A[1]); put(P2_DEF + D2_UYY, A[2] * 2.f);
		put(P2_DEF + D2_V, A[11]); put(P2_DEF + D2_VX, A[9]); put(P2_DEF + D2_VY, A[10] - 1.f);
		put(P2_DEF + D2_VXX, A[6] * 2.f); put(P2_DEF + D2_VXY, A[7]); put(P2_DEF + D2_VYY, A[8] * 2.f);
	}
};

// ---- the reference's `any interpolated sample < 0 -> zncc = -3` rule (src/oc_icgn.cpp:251-255, :792-796) --------------
// The sampling loops below evaluate the interpolant with explicit weights and fused multiply-adds; the reference goes
// through its 16-coefficient LUT and a 16-term polynomial (src/oc_cubic_bspline.cpp:98-129,159-177), and forms the warped
// position with separately rounded products (Deformation2D1::warp, src/oc_deformation.cpp:94-105).  Next to truly black
// pixels the B-spline overshoots by tiny amounts, so the sign of the smallest sample can hinge on those roundings.
// The loops therefore only track min(t); the decision is immediate when it is decisively negative (< -TRIGGER) or
// positive (>= TRIGGER), and otherwise re-made here sample by sample in the reference's own arithmetic: same operation
// order, every operation rounded separately (no FMA), the LUT cell rebuilt from the 4x4 pixel block.
constexpr float ICGN_NEG_TRIGGER = 0.125f; // covers one-ulp differences of the position (ulp 4.9e-4 px at x < 8192) times the steepest 8-bit edge
constexpr float ICGN_NEG_BAND = 4e-3f;     // fused vs separately rounded evaluation at the SAME position differ by < 3e-4 on 8-bit data
__constant__ float c_bc_matrix[4][4] = { // BC = B*C, src/oc_cubic_bspline.h:52-58
	{ -144.0f / 336.0f, 384.0f / 336.0f, -384.0f / 336.0f, 144.0f / 336.0f },
	{ 342.0f / 336.0f, -702.0f / 336.0f, 450.0f / 336.0f, -90.0f / 336.0f },
	{ -198.0f / 336.0f, -18.0f / 336.0f, 270.0f / 336.0f, -54.0f / 336.0f },
	{ 0.0f, 1.0f, 0.0f, 0.0f } };

// BicubicBspline::prepare for ONE cell + BicubicBspline::compute, reference operation order, no contraction.
// q: the 4x4 pixel block (row pitch `pitch`) whose element [1][1] is the pixel at (floor Y, floor X).
__device__ __noinline__ float bicubic_reference_order(const float* __restrict__ q, int pitch, float xd, float yd) {
	float coef[4][4]; // coefficient[k][l] = mat_p[3-k][3-l]
#pragma unroll 1
	for (int k = 0; k < 4; k++)
#pragma unroll 1
		for (int l = 0; l < 4; l++) {
			float acc = 0.f;
#pragma unroll
			for (int m = 0; m < 4; m++)
#pragma unroll
				for (int n = 0; n < 4; n++)
					acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(c_bc_matrix[l][m], c_bc_matrix[k][n]), q[n * pitch + m]));
			coef[3 - k][3 - l] = acc;
		}
	const float x2 = __fmul_rn(xd, xd), y2 = __fmul_rn(yd, yd), x3 = __fmul_rn(x2, xd), y3 = __fmul_rn(y2, yd);
	const float yp[4] = { 1.f, yd, y2, y3 }, xp[4] = { 1.f, xd, x2, x3 };
	float value = coef[0][0];
#pragma unroll
	for (int a = 0; a < 4; a++)
#pragma unroll
		for (int b = 0; b < 4; b++) {
			if (a == 0 && b == 0) continue;
			float term = coef[a][b];
			if (a > 0) term = __fmul_rn(term, yp[a]);
			if (b > 0) term = __fmul_rn(term, xp[b]);
			value = __fadd_rn(value, term);
		}
	return value;
}

// Does any of the samples idx = idx_begin, idx_begin + 32, ... < idx_end (row-major over the subset) of the warp Aw come
// out negative in the reference's arithmetic?  Aw: the running warp's A (Warp2D1 or Warp2D2).  Reads the target image
// directly (rare path).
template <class Warp>
__device__ __noinline__ bool icgn2d_exact_negative(const float* Aw, float pcx, float pcy, float ox, float oy, int rx, int ry,
	const float* __restrict__ tar, int w, int h, int idx_begin, int idx_end) {
	const int sw = 2 * rx + 1;
	bool negative = false;
	Warp W;
#pragma unroll
	for (int k = 0; k < Warp::NA; k++) W.A[k] = Aw[k];
	for (int idx = idx_begin; idx < idx_end; idx += 32) {
		const int r = idx / sw, c = idx - r * sw;
		const float xl = (float)(c - rx) - ox, yl = (float)(r - ry) - oy;
		float wx, wy;
		W.reference_offset(xl, yl, wx, wy);
		const float X = __fadd_rn(pcx, wx), Y = __fadd_rn(pcy, wy); // center + warped, src/oc_icgn.cpp:238-239
		if (!((X >= 1.f) && (Y >= 1.f) && (X < (float)(w - 2)) && (Y < (float)(h - 2)))) { // BicubicBspline::compute returns -1 (NaN too)
			negative = true;
			continue;
		}
		const float xf = floorf(X), yf = floorf(Y);
		const float* q = tar + (size_t)((int)yf - 1) * w + ((int)xf - 1);
		float blk[16], top = 0.f;
#pragma unroll
		for (int n = 0; n < 4; n++)
#pragma unroll
			for (int m = 0; m < 4; m++) {
				blk[n * 4 + m] = __ldg(q + (size_t)n * w + m);
				top = fmaxf(top, fabsf(blk[n * 4 + m]));
			}
		if (top == 0.f) continue; // an all-zero block gives exactly 0 in any arithmetic
		const float xd = __fsub_rn(X, xf), yd = __fsub_rn(Y, yf);
		float wxx[4], wyy[4];
		bicubic_weights(xd, wxx);
		bicubic_weights(yd, wyy);
		const float t = bicubic_fold(wxx, wyy, [&](int n, int m) { return blk[n * 4 + m]; });
		if (t >= ICGN_NEG_BAND) continue;
		if (t <= -ICGN_NEG_BAND || bicubic_reference_order(blk, 4, xd, yd) < 0.f) negative = true;
	}
	return negative;
}

// RC > 0: subset radius known at compile time (rx == ry == RC), so tile pitches and trip counts fold
// into immediates; RC == 0: any radii at run time.
// LM: inverse-compositional Levenberg-Marquardt siblings ICLM2D1 / ICLM2D2 (reference src/oc_iclm.cpp:150-358,
// :502-730): the Hessian is damped with lambda*I and re-factorised every iteration, a step is accepted only
// when ZNSSD decreased, and out-of-range samples are NOT rejected (the interpolant's -1 is used as a value).
// WPP: warps per POI.  One CTA = WPP warps = one POI at a time; the subset rows are split between the warps, which
// share the POI's slab and meet at a CTA barrier once per pass (partial sums through the slab).  Everything after the
// sums (statistics, solve, warp update) is computed redundantly by every warp from the same totals, so the warps
// never diverge in control flow.  With the slab unchanged this doubles the resident warps per SM (r=16: 22 instead
// of 11), which is what the latency-bound row loops need.
// SERIES: one reference against n_frames targets (img.tar is the frame-major stack [n_frames][h][w], tm_tar a 3D map over it).
// A POI's setup pass runs once; each frame then runs the same guard, target staging, iterations and result code as a pair
// call, seeded by the previous frame's record, which stays in registers.  Every frame's record is stored whole to
// frames_out[f n_poi + poi]; `pois` holds the seeds and is only read.  LM: what carries over is the undamped Hessian in sH
// (every iteration damps and factorises a copy of it) and the damping restarts from lm_lambda, as a pair call on the frame does.
// (the second launch bound keeps the register file from limiting residency below what the slab allows: 16 one-warp CTAs for the
//  6-parameter kernels of any radius, 12 for the r = 16 specialisation, whose 20 KB slab admits 11)
__host__ __device__ constexpr int icgn2d_min_ctas(int np, int rc, int wpp) { return np == 6 ? (rc == 16 ? 12 : ICGN2D_MIN_CTAS) / wpp : 7; }

template <int NP, int RC, bool LM, int WPP, bool SERIES>
__device__ __forceinline__ void icgn2d_poi_loop(Image2D img, float* __restrict__ pois, float* __restrict__ frames_out, int n_frames, int n_poi,
	int rx_arg, int ry_arg, float conv_criterion, float stop_condition, int* __restrict__ work_counter, const CUtensorMap& tm_ref,
	const CUtensorMap& tm_tar, int use_tma, const float* __restrict__ center_offsets, float lm_lambda, float lm_alpha, float lm_beta) {
	extern __shared__ __align__(128) float smem[];
	using Warp = std::conditional_t<NP == 6, Warp2D1, Warp2D2>;
	constexpr int NH = NP * (NP + 1) / 2;
	constexpr int NPHI = NP / 2;           // 3 or 6 shape monomials per displacement component
	constexpr int DEG = (NP == 6) ? 1 : 2; // degree of the shape function
	using Setup = SetupSums<DEG>;
	using Pass = PassSums<DEG>;
	const int rx = RC ? RC : rx_arg, ry = RC ? RC : ry_arg;
	const int lane = threadIdx.x & 31;
	const int sub = WPP > 1 ? (int)(threadIdx.x >> 5) : 0; // this warp's share of the POI
	const bool poi_leader = threadIdx.x == 0; // the thread that speaks for the POI (TMA issue, single stores)
	const int sw = 2 * rx + 1, sh = 2 * ry + 1, N = sw * sh;
	const int rows_per = (sh + WPP - 1) / WPP;
	const int r_lo = sub * rows_per, r_hi = (r_lo + rows_per) < sh ? (r_lo + rows_per) : sh; // rows [r_lo, r_hi) belong to this warp
	const int ncol = sw < 32 ? sw : 32;        // columns handled by the row-mapped main loops
	const int rem = sw - ncol;                  // columns 32.. handled by the tail loops
	const int ntail = rem * sh;
	const int RW = icgn2d_ref_w(rx), RH = icgn2d_ref_h(ry);
	const int TW = icgn2d_tar_w(rx), TH = icgn2d_tar_h(ry);
	float* slab = smem;
	int* s_poi = (int*)(slab + 8);              // WPP > 1: the POI index fetched by thread 0
	float* T = slab + 32;
	float* sC = T + icgn2d_tile_floats(rx, ry); // per-sample constants, interleaved {R, gx, gy} (12-byte lane stride: conflict-free)
	float* sH = sC + round_up32(3 * N);         // LM only: the undamped Hessian, packed lower triangle
	float* sRedS = sH + (LM ? 96 : 0);          // WPP > 1: setup partials [WPP][ICGN2D_RED_SETUP]
	float* sRedI = sRedS + WPP * ICGN2D_RED_SETUP; // WPP > 1: iteration partials [2][WPP][ICGN2D_RED_ITER]
	auto gsync = [&]() { // all warps of this POI
		if constexpr (WPP > 1) __syncthreads();
		else __syncwarp();
	};
	TileLoad tiles = { (uint64_t*)slab, 0, use_tma };
	tiles.init(poi_leader, gsync);
	const float* __restrict__ ref = img.ref;
	const int w = img.w, h = img.h;
	const float inv_n = 1.0f / (float)N;
	const bool lane_on = lane < ncol;
	const int lane_c = lane_on ? lane : ncol - 1; // idle lanes (subsets narrower than 32) shadow the last column

	// WPP == 1: the work counter is drawn and the record requested one POI AHEAD (the queue may be read in place from page-locked
	// host memory; the round trip then hides behind the current POI)
	int poi_next = 0;
	float rec_next = 0.f;
	if constexpr (WPP == 1) {
		if (lane == 0) poi_next = atomicAdd(work_counter, 1);
		poi_next = __shfl_sync(0xffffffffu, poi_next, 0);
		if (poi_next < n_poi && lane < P2_N) rec_next = pois[(size_t)poi_next * P2_N + lane];
	}
	while (true) {
		int poi = 0;
		float rec;
		if constexpr (WPP > 1) {
			gsync(); // every warp is done with the previous POI (slab, s_poi)
			if (threadIdx.x == 0) *s_poi = atomicAdd(work_counter, 1);
			gsync();
			poi = *s_poi;
			if (poi >= n_poi) break;
			rec = lane < P2_N ? pois[(size_t)poi * P2_N + lane] : 0.f;
		} else {
			poi = poi_next;
			if (poi >= n_poi) break;
			rec = rec_next;
			if (lane == 0) poi_next = atomicAdd(work_counter, 1);
			poi_next = __shfl_sync(0xffffffffu, poi_next, 0);
			if (poi_next < n_poi && lane < P2_N) rec_next = pois[(size_t)poi_next * P2_N + lane];
		}
		const float px = __shfl_sync(0xffffffffu, rec, P2_X);
		const float py = __shfl_sync(0xffffffffu, rec, P2_Y);
		// what the setup pass leaves for the iterations; SERIES: kept for every frame of the POI
		bool set_up = false;
		float c0, rbar, f2, ref_norm;
		float H[NH], S[NP], SF[NP];
		for (int f = 0; f < (SERIES ? n_frames : 1); f++) {
			float* P = SERIES ? frames_out + ((size_t)f * n_poi + poi) * P2_N : pois + (size_t)poi * P2_N;
			const float* __restrict__ tar = SERIES ? img.tar + (size_t)f * w * h : img.tar;
			// a rejected POI: only the ZNCC field changes, to `code`; SERIES stores the whole record, the next frame's seed
			auto store_rejection = [&](float code) {
				if constexpr (SERIES) {
					if (lane == P2_ZNCC) rec = code;
					if (threadIdx.x < P2_N) P[lane] = rec;
				} else {
					if (poi_leader) P[P2_ZNCC] = code;
				}
			};
			const float u_in = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_U);
			const float v_in = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_V);
			const float zncc_in = __shfl_sync(0xffffffffu, rec, P2_ZNCC);
			// guard, reference src/oc_icgn.cpp:160-167 / :701-708 (NaN coordinates are rejected too)
			if (subset2d_guard_fails(px, py, rx, ry, w, h, u_in, v_in, zncc_in)) {
				store_rejection(zncc_in >= 0 ? -3.f : zncc_in);
				continue;
			}
			gsync(); // every warp has read the record before thread 0 may write results / TMA may overwrite the slab
			// compute(POI2D*, Point2D& center_offset), src/oc_icgn.cpp:353-547 / :910-1126: local coordinates are
			// (integer - offset) and the target subset is centred at poi + offset; (0, 0) for the plain overload
			float ox = 0.f, oy = 0.f;
			if (center_offsets != nullptr) {
				ox = __ldg(center_offsets + 2 * (size_t)poi);
				oy = __ldg(center_offsets + 2 * (size_t)poi + 1);
			}
			const float xl_lane = (float)(lane - rx) - ox;
			const float xl_col = (float)(lane_c - rx) - ox; // the column a lane samples (the same as xl_lane on active lanes)
			const float pcx = px + ox, pcy = py + oy;

			if (!SERIES || !set_up) {
				set_up = true;
				// ---------------- stage the reference tile ----------------
				const int x0 = (int)px - rx, y0 = (int)py - ry; // Subset2D::fill upper-left, src/oc_subset.cpp:41-42
				const int rox = floor4(x0 - 2), ex = (x0 - 2) - rox; // 16-byte aligned tile origin, column offset 0..3
				tiles.issue<false>(T, &tm_ref, ref, w, h, rox, y0 - 2, 0, RW, RH, poi_leader, sub == 0, lane);
				tiles.wait(gsync);
				c0 = T[(ry + 2) * RW + rx + 2 + ex]; // pilot value: the centre pixel

				// ---------------- setup: R', gradients, factored Hessian sums ----------------
				Setup ss;
				// INTERIOR: every gradient of the subset is off the image's 2-pixel border, so no row or lane needs a border test
				auto setup_rows = [&](auto interior_) {
					constexpr bool INTERIOR = decltype(interior_)::value;
					const int xg = x0 + lane;
					const bool gx_ok = INTERIOR || (lane_on && xg >= 2 && xg < w - 2); // gradient maps are zero on a 2-pixel border (src/oc_gradient.cpp:42,46)
					// the lane's column at rows r - 2 .. r + 2 (the pixel and its gy taps) rolls down in registers: one new pixel per row
					const float* qn = T + r_lo * RW + lane_c + 2 + ex;
					float cm2 = qn[0], cm1 = qn[RW], cc = qn[2 * RW], cp1 = qn[3 * RW];
					qn += 4 * RW;
					for (int r = r_lo; r < r_hi; r++) {
						const float cp2 = *qn;
						qn += RW;
						const int yg = y0 + r;
						const bool gy_ok = INTERIOR || (yg >= 2 && yg < h - 2);
						const float yl = (float)(r - ry) - oy;
						if (INTERIOR || lane_on) {
							const float* q = T + (r + 2) * RW + lane + 2 + ex;
							const float R = cc - c0;
							float gx = 0.f, gy = 0.f;
							if (gx_ok) gx = grad4(q[-2], q[-1], q[1], q[2]);
							if (gy_ok) gy = grad4(cm2, cm1, cp1, cp2);
							{
								float* pc = sC + 3 * (r * sw + lane);
								pc[0] = cc; // raw R
								pc[1] = gx;
								pc[2] = gy;
							}
							ss.add_row(R, gx, gy, yl);
						}
						cm2 = cm1;
						cm1 = cc;
						cc = cp1;
						cp1 = cp2;
					}
				};
				if constexpr (RC == 16) {
					// r = 16 (all 32 lanes on): the common POI, more than 2 pixels inside the image, takes the loop without tests
					if (x0 >= 2 && x0 + sw - 1 < w - 2 && y0 >= 2 && y0 + sh - 1 < h - 2) setup_rows(std::true_type());
					else setup_rows(std::false_type());
				} else {
					setup_rows(std::false_type());
				}
				ss.expand(xl_lane);
				// tail columns (>= 32): lanes run over (row, column) pairs, general x and y
				for (int idx = sub * 32 + lane; idx < ntail; idx += 32 * WPP) {
					const int r = idx / rem, c = 32 + (idx - r * rem);
					const int xg = x0 + c, yg = y0 + r;
					const float xl = (float)(c - rx) - ox, yl = (float)(r - ry) - oy;
					const float* q = T + (r + 2) * RW + c + 2 + ex;
					const float R = q[0] - c0;
					float gx = 0.f, gy = 0.f;
					if (xg >= 2 && xg < w - 2) gx = grad4(q[-2], q[-1], q[1], q[2]);
					if (yg >= 2 && yg < h - 2) gy = grad4(q[-2 * RW], q[-RW], q[RW], q[2 * RW]);
					float* pc = sC + 3 * (r * sw + c);
					pc[0] = q[0];
					pc[1] = gx;
					pc[2] = gy;
					ss.add(R, gx, gy, xl, yl);
				}
				ss.reduce();
				if constexpr (WPP > 1) combine_warps<WPP>(ss.v, sRedS, ICGN2D_RED_SETUP, sub, lane); // its barrier: every warp is done with the reference tile
				// reference subset statistics (Subset2D::zeroMeanNorm, src/oc_subset.cpp:46-53), relative to c0
				const float r1 = ss.v[Setup::R1], r2 = ss.v[Setup::R2];
				rbar = r1 * inv_n;              // mean(R) - c0
				f2 = r2 - r1 * rbar;            // sum f^2, f = R - mean(R)
				ref_norm = sqrtf(f2);
				// S_k = sum sd_k, SF_k = sum sd_k f = sum sd_k R' - rbar * S_k ; H = sum sd sd^T (src/oc_icgn.cpp:198-205)
#pragma unroll
				for (int a = 0; a < 2; a++)
#pragma unroll
					for (int i = 0; i < NPHI; i++) {
						const int k = a * NPHI + i;
						const float sg = ss.v[Setup::SG + k], srg = ss.v[Setup::SRG + k];
						S[k] = phi_c(i) * sg;
						SF[k] = phi_c(i) * (srg - rbar * sg);
#pragma unroll
						for (int b = 0; b < 2; b++)
#pragma unroll
							for (int j = 0; j < NPHI; j++) {
								const int l = b * NPHI + j;
								if (l <= k)
									H[k * (k + 1) / 2 + l] = phi_c(i) * phi_c(j) * ss.v[Setup::M + pair_idx(a, b) * Setup::NM + mono(phi_p(i) + phi_p(j), phi_q(i) + phi_q(j))];
							}
					}
				if constexpr (LM) {
					if (threadIdx.x == 0) {
#pragma unroll
						for (int k = 0; k < NH; k++) sH[k] = H[k];
					}
					gsync();
				} else {
					cholesky_packed<NP>(H);
				}
			}
			float lm_cur = 0.f, znssd0 = 4.f; // src/oc_iclm.cpp:234-235

			// ---------------- stage the target tile over the reference tile ----------------
			// (WPP > 1: the barrier of the setup reduction already ordered every warp's last read of the reference tile)
			if constexpr (WPP == 1) __syncwarp();
			const int tx0 = floor4((int)floorf(pcx + u_in) - rx - 1 - ICGN2D_TILE_MARGIN);
			const int ty0 = (int)floorf(pcy + v_in) - ry - 1 - ICGN2D_TILE_MARGIN;
			tiles.issue<SERIES>(T, &tm_tar, tar, w, h, tx0, ty0, f, TW, TH, poi_leader, sub == 0, lane);
			tiles.wait(gsync);
			// a sample is "fast" when it is valid (src/oc_cubic_bspline.cpp:137-142) AND its support is in the tile
			const float xlo = fmaxf(1.f, (float)(tx0 + 1)), xhi = fminf((float)(w - 2), (float)(tx0 + TW - 2));
			const float ylo = fmaxf(1.f, (float)(ty0 + 1)), yhi = fminf((float)(h - 2), (float)(ty0 + TH - 2));
			const float xmax = (float)(w - 2), ymax = (float)(h - 2);
			// the checked sample at (X, Y): false when it is outside the interpolant's domain (NaN too) and IC-GN rejects the POI;
			// otherwise t is the sample, from the tile when its support is there, and IC-LM takes the interpolant's -1 outside
			auto sample_checked = [&](float X, float Y, float& t) {
				const bool fast = (X >= xlo) && (X < xhi) && (Y >= ylo) && (Y < yhi);
				const bool ok = fast || ((X >= 1.f) && (Y >= 1.f) && (X < xmax) && (Y < ymax));
				if (!ok && !LM) return false;
				t = ok ? bicubic_sample(T, TW, tx0, ty0, tar, w, X, Y, fast) : -1.f; // BicubicBspline::compute returns -1 outside
				return true;
			};

			// ---------------- IC-GN iterations ----------------
			Warp W;
			W.init(u_in, __shfl_sync(0xffffffffu, rec, P2_DEF + D2_UX), __shfl_sync(0xffffffffu, rec, P2_DEF + D2_UY), v_in,
				__shfl_sync(0xffffffffu, rec, P2_DEF + D2_VX), __shfl_sync(0xffffffffu, rec, P2_DEF + D2_VY));
			int iteration = 0;
			float dp_norm = 0.f, zncc = 0.f;
			bool left_image = false;
			float dp[NP];
			do {
				iteration++;
				Pass ps;
				bool invalid = false;
				float tmin = 3.0e38f; // smallest interpolated sample of this pass (see icgn2d_exact_negative)
				const auto col = W.column(xl_col);
				// Can every row-mapped sample take the fast path (valid + support inside the tile)?  The
				// affine part of the warp maps the subset to a parallelogram, so its 4 corners decide;
				// the second-order part is bounded and widens it.
				bool iter_fast;
				{
					const float fx = (float)rx + fabsf(ox), fy = (float)ry + fabsf(oy);
					float cx, cy, ex_, ey_;
					W.bounds(pcx, pcy, fx, fy, cx, cy, ex_, ey_);
					iter_fast = (cx - ex_ >= xlo) && (cx + ex_ < xhi) && (cy - ey_ >= ylo) && (cy + ey_ < yhi); // false for NaN
				}
				// Whole-pixel pass: when the running warp is a translation by whole pixels and pcx, pcy, ox, oy are whole numbers
				// (pass 1 of every POI seeded by FFT-CC), every warped position is an exact integer (all terms are small integers),
				// the interpolant's weights at fraction 0 are {-0, 1, +0, -0} and the weighted sum returns the pixel itself (a -0
				// pixel as +0, hence the + 0.f below).  A non-finite pixel elsewhere in a sample's 4x4 support makes that sum NaN
				// (0 * Inf), so the shortcut is taken only when every pixel of the supports is finite.
				bool whole = false;
				int wofs = 0; // whole-pixel pass: tile offset of the pixel under subset point (0, 0)
				if (iter_fast) {
					float kx, ky;
					const bool shift = W.translation(kx, ky);
					auto integral = [](float v) { return truncf(v) == v; };
					if (shift && integral(kx) && integral(ky) && integral(pcx) && integral(pcy) && integral(ox) && integral(oy)) {
						const int wrow = (int)pcy + (int)ky - (int)oy - ry - ty0, wcol = (int)pcx + (int)kx - (int)ox - rx - tx0;
						wofs = wrow * TW + wcol;
						// the supports span subset rows and columns -1 .. size + 1; iter_fast keeps them inside the tile
						bool finite = true;
						if constexpr (RC == 16) {
							// 36 x 36 support pixels inside the 44-float (16-byte aligned) tile rows: scan the aligned 36 x 40 block around
							// them as float4, lane l (l < 30) taking columns 4 (l % 10) .. + 3 of rows l / 10, l / 10 + 3, ...  The extra
							// pixels cannot change a record: a non-finite one only sends the pass to the interpolating loop, which returns
							// the same samples when the supports are finite.
							const int l = lane < 30 ? lane : 29; // lanes 30, 31 repeat lane 29
							const int a0 = min(floor4(wcol - 1), TW - 40); // wcol + 34 < TW: the block ends inside the row
							const float4* p = reinterpret_cast<const float4*>(T + (wrow - 1 + l / 10) * TW + a0) + l % 10;
#pragma unroll
							for (int k = 0; k < 12; k++) {
								const float4 q4 = p[k * 3 * TW / 4];
								finite &= fabsf(q4.x) < INFINITY;
								finite &= fabsf(q4.y) < INFINITY;
								finite &= fabsf(q4.z) < INFINITY;
								finite &= fabsf(q4.w) < INFINITY;
							}
						} else {
							for (int c = lane - 1; c <= sw + 1; c += 32) {
								const float* p = T + wofs - TW + c;
#pragma unroll 12
								for (int r = -1; r <= sh + 1; r++, p += TW) finite &= fabsf(*p) < INFINITY;
							}
						}
						whole = __all_sync(0xffffffffu, finite);
					}
				}
				if (iter_fast) {
					// branch-free row loops: no per-sample validity tests (min(t) is tested after the loop)
					float yl = (float)(r_lo - ry) - oy;
					const float* pc = sC + 3 * (r_lo * sw + lane_c);
					// everything after the sample t, the same for both loops: min(t) (idle lanes shadow the last column and feed it
					// too), d = t - R and this row's sums
					auto row_sums = [&](float t) {
						tmin = fminf(tmin, t);
						const float R = pc[0];
						ps.add_row(lane_on ? t - R : 0.f, R, pc[1], pc[2], yl);
						pc += 3 * sw;
						yl += 1.f;
					};
					if (whole) {
						const float* q = T + wofs + r_lo * TW + lane_c;
#pragma unroll ICGN2D_ROW_UNROLL
						for (int r = r_lo; r < r_hi; r++) {
							row_sums(q[0] + 0.f);
							q += TW;
						}
					} else {
						const float* tbase = T - (ty0 + 1) * TW - (tx0 + 1);
						if constexpr (NP == 6) {
							// Rolling 4x4 window.  Lane c walks down column c, and row r + 1's block is nearly always row r's moved down by
							// one pixel row (floor X unchanged, floor Y + 1): three of its rows are already in registers and only the new
							// bottom row is read.  The block rows live in four register slots fixed at compile time: a sample whose top slot
							// is S has its block rows 0..3 in slots S..S+3 (mod 4), and the next sample's bottom row replaces slot S.  Rows go
							// in batches of four (top slots 1, 2, 3, 0); a batch in which any lane's step is not regular reloads full blocks.
							// The same pixels, weights and FMA order as a full load, so the samples are the same.
							float win[4][4];
							float xfp = 0.f, yfp = 0.f; // floor X, floor Y of the previous row
							const float* qp = tbase;    // the previous row's block
							auto rows = [&](auto S_, auto NB_, auto FIRST_) {
								constexpr int S = decltype(S_)::value, NB = decltype(NB_)::value;
								constexpr bool FIRST = decltype(FIRST_)::value; // no previous row: load the full block
								float X[NB], Y[NB], xf[NB], yf[NB], t[NB];
								bool regular = true;
								float ylj = yl;
#pragma unroll
								for (int j = 0; j < NB; j++) {
									col.at(pcx, pcy, ylj, X[j], Y[j]);
									xf[j] = floorf(X[j]);
									yf[j] = floorf(Y[j]);
									regular &= xf[j] == (j ? xf[j - 1] : xfp) && yf[j] == (j ? yf[j - 1] : yfp) + 1.f;
									ylj += 1.f;
								}
								auto interpolate = [&](int j) { // sample j from the window slots S + j .. S + j + 3
									float wx[4], wy[4];
									bicubic_weights(X[j] - xf[j], wx);
									bicubic_weights(Y[j] - yf[j], wy);
									return bicubic_fold(wx, wy, [&](int n, int m) { return win[(S + j + n) & 3][m]; });
								};
								if (!FIRST && __all_sync(0xffffffffu, regular)) {
#pragma unroll
									for (int j = 0; j < NB; j++) {
										const float* q = qp + (j + 4) * TW; // bottom row of sample j's block
#pragma unroll
										for (int m = 0; m < 4; m++) win[(S + j + 3) & 3][m] = q[m];
										t[j] = interpolate(j);
									}
									qp += NB * TW;
								} else {
#pragma unroll
									for (int j = 0; j < NB; j++) {
										qp = tbase + (int)yf[j] * TW + (int)xf[j];
#pragma unroll
										for (int nn = 0; nn < 4; nn++)
#pragma unroll
											for (int m = 0; m < 4; m++) win[(S + j + nn) & 3][m] = qp[nn * TW + m];
										t[j] = interpolate(j);
									}
								}
								xfp = xf[NB - 1];
								yfp = yf[NB - 1];
#pragma unroll
								for (int j = 0; j < NB; j++) row_sums(t[j]);
							};
							using std::integral_constant;
							using one = integral_constant<int, 1>;
							using full = std::true_type;
							using rolling = std::false_type;
							if (r_lo < r_hi) {
								rows(integral_constant<int, 0>(), one(), full());
								int r = r_lo + 1;
#pragma unroll 1
								for (; r + 4 <= r_hi; r += 4) rows(one(), integral_constant<int, 4>(), rolling());
								switch (r_hi - r) { // WPP 2 and the generic radius
								case 1: rows(one(), one(), rolling()); break;
								case 2: rows(one(), integral_constant<int, 2>(), rolling()); break;
								case 3: rows(one(), integral_constant<int, 3>(), rolling()); break;
								default: break;
								}
							}
						} else {
							// The 12-parameter kernels keep one row per step with a full block load: with the rolling window, config C's
							// IC-GN kernel (ICGN2D2, r = 20, 7 warps per SM) took 2.23 instead of 2.19 ms on the H100.
#pragma unroll ICGN2D_ROW_UNROLL
							for (int r = r_lo; r < r_hi; r++) {
								float X, Y;
								col.at(pcx, pcy, yl, X, Y);
								const float xf = floorf(X), yf = floorf(Y);
								float wx[4], wy[4];
								bicubic_weights(X - xf, wx);
								bicubic_weights(Y - yf, wy);
								const float* q = tbase + (int)yf * TW + (int)xf;
								row_sums(bicubic_fold(wx, wy, [&](int n, int m) { return q[n * TW + m]; }));
							}
						}
					}
				} else {
					for (int r = r_lo; r < r_hi; r++) {
						const float yl = (float)(r - ry) - oy;
						float X, Y, t;
						col.at(pcx, pcy, yl, X, Y);
						if (lane_on) {
							if (!sample_checked(X, Y, t)) {
								invalid = true;
							} else {
								tmin = fminf(tmin, t);
								const float* pc = sC + 3 * (r * sw + lane);
								ps.add_row(t - pc[0], pc[0], pc[1], pc[2], yl);
							}
						}
					}
				}
				ps.expand(xl_lane);
				// tail columns (>= 32): lanes run over (row, column) pairs
				auto tail_sums = [&](int r, int c, float xl, float yl, float t) {
					tmin = fminf(tmin, t);
					const float* pc = sC + 3 * (r * sw + c);
					ps.add(t - pc[0], pc[0], pc[1], pc[2], xl, yl);
				};
				if (RC == 16 && iter_fast) {
					// one tail column (rem == 1: the row is the index), and the corner test of iter_fast covers column 2r: every
					// sample is valid and its support is in the tile, so no per-sample tests and no global-memory fallback
					static_assert(RC != 16 || 2 * RC + 1 == 33, "the r = 16 tail is one column wide");
					constexpr int c = 32;
					const float xl = (float)(c - rx) - ox;
					for (int r = sub * 32 + lane; r < sh; r += 32 * WPP) {
						const float yl = (float)(r - ry) - oy;
						float t;
						if (whole) {
							t = T[wofs + r * TW + c] + 0.f;
						} else {
							float X, Y;
							W.at(pcx, pcy, xl, yl, X, Y);
							t = bicubic_sample(T, TW, tx0, ty0, tar, w, X, Y, true);
						}
						tail_sums(r, c, xl, yl, t);
					}
				} else {
					for (int idx = sub * 32 + lane; idx < ntail; idx += 32 * WPP) {
						const int r = idx / rem, c = 32 + (idx - r * rem);
						const float xl = (float)(c - rx) - ox, yl = (float)(r - ry) - oy;
						float X, Y, t;
						W.at(pcx, pcy, xl, yl, X, Y);
						if (whole) t = T[wofs + r * TW + c] + 0.f; // a whole-pixel pass has every sample in the tile
						else if (!sample_checked(X, Y, t)) {
							invalid = true;
							continue;
						}
						tail_sums(r, c, xl, yl, t);
					}
				}
				if constexpr (!LM) { // src/oc_icgn.cpp:251-255: any sample < 0 rejects the POI (the ICLM siblings have no such test)
					if (tmin < -ICGN_NEG_TRIGGER) invalid = true;
					const bool borderline = !(tmin >= ICGN_NEG_TRIGGER);
					if (__any_sync(0xffffffffu, borderline) && !__any_sync(0xffffffffu, invalid)) {
						float* sA = slab + 16; // the running warp, handed over through the slab header
						if (lane == 0) {
#pragma unroll
							for (int k = 0; k < Warp::NA; k++) sA[k] = W.A[k];
						}
						__syncwarp();
						if (icgn2d_exact_negative<Warp>(sA, pcx, pcy, ox, oy, rx, ry, tar, w, h, lane, N)) invalid = true;
					}
				}
				bool any_invalid = __any_sync(0xffffffffu, invalid);
				ps.reduce();
				if constexpr (WPP > 1) {
					ps.v[Pass::INV] = any_invalid ? 1.f : 0.f;
					// double-buffered by iteration parity: one barrier per iteration
					combine_warps<WPP>(ps.v, sRedI + (iteration & 1) * WPP * ICGN2D_RED_ITER, ICGN2D_RED_ITER, sub, lane);
					any_invalid = ps.v[Pass::INV] > 0.f;
				}
				const float d1 = ps.v[Pass::D1], d2 = ps.v[Pass::D2], rd = ps.v[Pass::RD];
				const float* SD = ps.v + Pass::SD;
				if (any_invalid) { // src/oc_icgn.cpp:251-255
					left_image = true;
					break;
				}
				// warped-target statistics: g = t - mean(t) = f + (d - dbar); sum f d = sum R'd - rbar * sum d
				const float dbar = d1 * inv_n;
				const float fd = (rd - c0 * d1) - rbar * d1; // rd holds sum R d with the raw R
				const float g2 = f2 + 2.f * fd + (d2 - d1 * dbar);
				const float tar_norm = sqrtf(g2);
				const float factor = ref_norm / tar_norm; // src/oc_icgn.cpp:260
				zncc = (f2 + fd) / (ref_norm * tar_norm); // == 0.5*(2 - znssd), src/oc_icgn.cpp:263,320
				float b[NP];
#pragma unroll
				for (int k = 0; k < NP; k++) b[k] = factor * (SF[k] + SD[k] - dbar * S[k]) - SF[k];
				bool accept = true;
				if constexpr (LM) {
					const float znssd = 2.f - 2.f * zncc;
					if (iteration == 1) lm_cur = powf(lm_lambda, znssd / znssd0) - 1.f; // src/oc_iclm.cpp:258-263
#pragma unroll
					for (int k = 0; k < NH; k++) H[k] = sH[k];
#pragma unroll
					for (int k = 0; k < NP; k++) H[k * (k + 1) / 2 + k] += lm_cur; // hessian + lambda * I, :266
					cholesky_packed<NP>(H);
					accept = znssd < znssd0; // :292-310
					if (accept) { lm_cur *= lm_alpha; znssd0 = znssd; }
					else lm_cur *= lm_beta;
				}
				cholesky_solve<NP>(H, b, dp);
				W.compose_inverse(dp, accept);
				dp_norm = sqrtf(Warp::dp_norm2(dp, rx, ry));
			} while ((float)iteration < stop_condition && dp_norm >= conv_criterion);

			if (left_image) {
				store_rejection(-3.f);
				__syncwarp();
				continue;
			}
			// ---------------- results, src/oc_icgn.cpp:310-340 / :859-897 ----------------
			// Every lane holds the same final state; the record goes out as ONE coalesced store, lane k writing float k (fields the
			// reference leaves alone keep the value read at the start) -- the queue may live in page-locked host memory, where
			// separate 4-byte stores would each cross PCIe on their own.  SERIES: every warp keeps the record as the next frame's seed.
			if (SERIES || threadIdx.x < 32) {
				const float u = W.u(), v = W.v();
				float out = rec;
				auto put = [&](int field, float value) { if (lane == field) out = value; };
				W.put_fields(put);
				put(P2_U0, u_in);
				put(P2_V0, v_in);
				float zout = zncc;
				put(P2_ITER, (float)iteration);
				put(P2_CONV, dp_norm);
				put(P2_RX, (float)rx);
				put(P2_RY, (float)ry);
				if (dp_norm >= conv_criterion && (float)iteration >= stop_condition) zout = -4.f;
				if (is_nan_f(zout) || is_nan_f(u) || is_nan_f(v)) {
					put(P2_DEF + D2_U, u_in);
					put(P2_DEF + D2_V, v_in);
					zout = -5.f;
				}
				put(P2_ZNCC, zout);
				if (lane < P2_N && (!SERIES || threadIdx.x < 32)) P[lane] = out;
				if constexpr (SERIES) rec = out;
			}
			__syncwarp();
		}
	}
	if constexpr (WPP == 1) {
		// The queue head resets itself: the last worker to leave zeroes it (and the departure count 8 ints further on), so a
		// launch needs no memset in front of it (2-3 us of an otherwise empty stream per launch).  The host zeroes both once.
		if (lane == 0) {
			const int workers = (int)gridDim.x;
			__threadfence();
			if (atomicAdd(work_counter + 8, 1) == workers - 1) {
				work_counter[0] = 0;
				work_counter[8] = 0;
			}
		}
	}
}

template <int NP, int RC, bool LM, int WPP>
__global__ void __launch_bounds__(32 * WPP, icgn2d_min_ctas(NP, RC, WPP)) icgn2d_kernel(Image2D img, float* __restrict__ pois, int n_poi, int rx_arg,
	int ry_arg, float conv_criterion, float stop_condition, int* __restrict__ work_counter, const __grid_constant__ CUtensorMap tm_ref,
	const __grid_constant__ CUtensorMap tm_tar, int use_tma, const float* __restrict__ center_offsets, float lm_lambda, float lm_alpha,
	float lm_beta) {
	icgn2d_poi_loop<NP, RC, LM, WPP, false>(img, pois, nullptr, 1, n_poi, rx_arg, ry_arg, conv_criterion, stop_condition, work_counter, tm_ref, tm_tar,
		use_tma, center_offsets, lm_lambda, lm_alpha, lm_beta);
}

// img.tar: the frame-major target stack; tm_tars: its 3D map (box depth 1).  The damping comes last, so the IC-GN instantiations
// see the parameters they had before IC-LM series existed.
template <int NP, int RC, bool LM, int WPP>
__global__ void __launch_bounds__(32 * WPP, icgn2d_min_ctas(NP, RC, WPP)) icgn2d_series_kernel(Image2D img, const float* __restrict__ seeds,
	float* __restrict__ out, int n_frames, int n_poi, int rx_arg, int ry_arg, float conv_criterion, float stop_condition,
	int* __restrict__ work_counter, const __grid_constant__ CUtensorMap tm_ref, const __grid_constant__ CUtensorMap tm_tars, int use_tma,
	float lm_lambda, float lm_alpha, float lm_beta) {
	icgn2d_poi_loop<NP, RC, LM, WPP, true>(img, const_cast<float*>(seeds), out, n_frames, n_poi, rx_arg, ry_arg, conv_criterion, stop_condition,
		work_counter, tm_ref, tm_tars, use_tma, nullptr, lm_lambda, lm_alpha, lm_beta);
}

// host-side launch ---------------------------------------------------------------------------
template <bool SERIES, int NP, int RC, bool LM, int WPP>
static constexpr auto icgn2d_kernel_of() {
	if constexpr (SERIES) return icgn2d_series_kernel<NP, RC, LM, WPP>;
	else return icgn2d_kernel<NP, RC, LM, WPP>;
}

// the instantiation a launch runs: IC-LM has the generic radius only; IC-GN has r = 16 (6 parameters) and r = 20 (12 parameters)
template <bool SERIES>
static auto icgn2d_pick(int np, int rc, bool lm, int wpp) {
	auto pick = [=](auto wpp_) {
		constexpr int WPP = decltype(wpp_)::value;
		if (lm) return np == 6 ? icgn2d_kernel_of<SERIES, 6, 0, true, WPP>() : icgn2d_kernel_of<SERIES, 12, 0, true, WPP>();
		if (np == 6) return rc == 16 ? icgn2d_kernel_of<SERIES, 6, 16, false, WPP>() : icgn2d_kernel_of<SERIES, 6, 0, false, WPP>();
		return rc == 20 ? icgn2d_kernel_of<SERIES, 12, 20, false, WPP>() : icgn2d_kernel_of<SERIES, 12, 0, false, WPP>();
	};
	return wpp == 2 ? pick(std::integral_constant<int, 2>()) : pick(std::integral_constant<int, 1>());
}

// The work-queue head of a launch: [0] of the context's heads, zeroed here, for two warps per POI; [32] for the one-warp-per-POI
// kernels, which reset their head themselves (a set of heads nobody else touches; [40] is their departure count).
static cudaError_t icgn2d_counter(const Icgn2dPlan& p, int** d_counter, cudaStream_t stream) {
	if (p.wpp == 1) {
		*d_counter += 32;
		return cudaSuccess;
	}
	return cudaMemsetAsync(*d_counter, 0, sizeof(int), stream);
}

// tensor maps of the reference image and of the target (n_frames == 0: one image; else the frame-major stack); 0: stage the tiles
static int icgn2d_maps(const Image2D& img, int n_frames, int rx, int ry, CUtensorMap* tm_ref, CUtensorMap* tm_tar) {
	return tma_enabled() && tma_image_map(tm_ref, img.ref, img.w, img.h, 0, icgn2d_ref_w(rx), icgn2d_ref_h(ry))
		&& tma_image_map(tm_tar, img.tar, img.w, img.h, n_frames, icgn2d_tar_w(rx), icgn2d_tar_h(ry));
}

cudaError_t icgn2d_launch(int np, const Icgn2dPlan& p, const Image2D& img, float* d_pois, size_t n, int rx, int ry, float conv, float stop,
	int* d_counter, const float* d_center_offsets, const float* lm_damping, cudaStream_t stream) {
	const bool lm = lm_damping != nullptr;
	cudaError_t e = icgn2d_counter(p, &d_counter, stream);
	if (e != cudaSuccess) return e;
	CUtensorMap tm_ref{}, tm_tar{};
	const int use_tma = icgn2d_maps(img, 0, rx, ry, &tm_ref, &tm_tar);
	return launch_smem(icgn2d_pick<false>(np, p.rc, lm, p.wpp), p.grid, p.wpp * 32, p.smem, stream, img, d_pois, (int)n, rx, ry, conv, stop,
		d_counter, tm_ref, tm_tar, use_tma, d_center_offsets, lm ? lm_damping[0] : 0.f, lm ? lm_damping[1] : 0.f, lm ? lm_damping[2] : 0.f);
}

cudaError_t icgn2d_series_launch(int np, const Icgn2dPlan& p, const Image2D& img, int n_frames, const float* d_seeds, float* d_out, size_t n,
	int rx, int ry, float conv, float stop, int* d_counter, const float* lm_damping, cudaStream_t stream) {
	const bool lm = lm_damping != nullptr;
	cudaError_t e = icgn2d_counter(p, &d_counter, stream);
	if (e != cudaSuccess) return e;
	CUtensorMap tm_ref{}, tm_tars{};
	const int use_tma = icgn2d_maps(img, n_frames, rx, ry, &tm_ref, &tm_tars);
	return launch_smem(icgn2d_pick<true>(np, p.rc, lm, p.wpp), p.grid, p.wpp * 32, p.smem, stream, img, d_seeds, d_out, n_frames, (int)n, rx,
		ry, conv, stop, d_counter, tm_ref, tm_tars, use_tma, lm ? lm_damping[0] : 0.f, lm ? lm_damping[1] : 0.f, lm ? lm_damping[2] : 0.f);
}

} // namespace ocb
