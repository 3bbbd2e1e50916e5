// sift3d.cu -- SIFT3D (reference src/oc_sift.cpp:140-1519) on sm_90a: Gaussian pyramid, DoG extrema, orientation, descriptors
// and brute-force matching.  Compiled with -fmad=false (build.py): every product and sum is rounded on its own, in the
// reference's order, so the layers, candidates, keypoints and descriptors are bit-identical to the float32 oracle
// (oracle/oc_sift3d.cpp).  No float atomics: each sum has one owner that adds in the reference's order.
//
// The pyramid is built one octave at a time: the n_octave_layers + 3 Gaussian layers of an octave are blurred, detection,
// orientation and description run on them, and the next octave's bottom layer is downsampled from them.  The DoG is never
// stored: each DoG value is formed where it is read, by the same single subtraction.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <vector>

#include "ocb_kernels.h"

namespace ocb {
namespace {

__constant__ float c_ico_v[36] = S3_ICO_VERTICES;
__constant__ int c_ico_f[60] = S3_ICO_FACES;

// One axis of gaussianBlur (:404-540): out = k0 * s[c]; out += k_r * (s[lower tap] + s[upper tap]).  Threads run along x, so
// every pass reads and writes coalesced rows; the taps of neighbouring threads hit L1.
template <int AXIS>
__global__ void __launch_bounds__(256) blur_axis_kernel(const float* __restrict__ src, float* __restrict__ dst, int nx, int ny, int nz, int R,
	BlurW w) {
	const int x = blockIdx.x * 32 + threadIdx.x;
	const int y = blockIdx.y * 8 + threadIdx.y;
	if (x >= nx || y >= ny) return;
	for (int z = blockIdx.z; z < nz; z += gridDim.z) {
		const size_t o = ((size_t)z * ny + y) * nx + x;
		const int c = AXIS == 0 ? x : (AXIS == 1 ? y : z);
		const int n = AXIS == 0 ? nx : (AXIS == 1 ? ny : nz);
		const size_t stride = AXIS == 0 ? 1 : (AXIS == 1 ? (size_t)nx : (size_t)nx * ny);
		const float* line = src + (o - (size_t)c * stride);
		float acc = w.w[0] * line[(size_t)c * stride];
		for (int r = 1; r <= R; r++)
			acc += w.w[r] * (line[(size_t)s3::mirror_lower(c - r, n) * stride] + line[(size_t)s3::mirror_upper(c + r, n) * stride]);
		dst[o] = acc;
	}
}

// downSampling (:549-562): the even voxels.
__global__ void downsample_kernel(const float* __restrict__ src, float* __restrict__ dst, int sx, int sy, int dx, int dy, int dz) {
	const size_t n = (size_t)dx * dy * dz;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		const int x = (int)(i % dx), y = (int)((i / dx) % dy), z = (int)(i / ((size_t)dx * dy));
		dst[i] = src[((size_t)(2 * z) * sy + 2 * y) * sx + 2 * x];
	}
}

// max |G[n+1] - G[n]| of one DoG layer (:779-790); a maximum is order-free, so the integer atomicMax on the bits of the
// non-negative values is exact.  *out starts at the bits of -1.f (the reference's initial max_abs), which every
// non-negative float's bits exceed as signed integers.  NaN voxels are skipped, as the reference's comparison skips them.
__global__ void max_abs_kernel(const float* __restrict__ g0, const float* __restrict__ g1, size_t n, int* out) {
	float m = -1.f;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		const float a = fabsf(g1[i] - g0[i]);
		m = m < a ? a : m;
	}
	for (int o = 16; o; o >>= 1) {
		const float b = __shfl_xor_sync(0xffffffffu, m, o);
		m = m < b ? b : m;
	}
	if ((threadIdx.x & 31) == 0 && m >= 0.f) atomicMax(out, __float_as_int(m));
}

struct OctaveView {
	const float* g[SIFT3D_MAX_L];
	int nx, ny, nz;
	float unit[3];
	float scale[SIFT3D_MAX_L];
};

// detectExtrema (:795-847) as a predicate over the flattened (layer - 1, z, y, x) index of an octave: cub's order-preserving
// selection then lists the candidates in the reference's (layer, z, y, x) order.
struct ExtremumPred {
	OctaveView v;
	float thr[SIFT3D_MAX_L];
	__device__ bool operator()(const long long idx) const {
		const size_t N = (size_t)v.nx * v.ny * v.nz;
		const int n = 1 + (int)(idx / (long long)N);
		const size_t p = (size_t)(idx % (long long)N);
		const int x = (int)(p % v.nx), y = (int)((p / v.nx) % v.ny), z = (int)(p / ((size_t)v.nx * v.ny));
		if (x < 1 || y < 1 || z < 1 || x >= v.nx - 1 || y >= v.ny - 1 || z >= v.nz - 1) return false;
		const float* gm = v.g[n - 1];
		const float* g0 = v.g[n];
		const float* g1 = v.g[n + 1];
		const float* g2 = v.g[n + 2];
		const float d = g1[p] - g0[p];
		if (!(fabsf(d) >= thr[n])) return false;
		const size_t sy = v.nx, sz = (size_t)v.nx * v.ny;
		const float nb[8] = { g1[p - sz] - g0[p - sz], g1[p + sz] - g0[p + sz], g1[p - sy] - g0[p - sy], g1[p + sy] - g0[p + sy], g1[p - 1] - g0[p - 1],
			g1[p + 1] - g0[p + 1], g0[p] - gm[p], g2[p] - g1[p] };
		bool gt = true, lt = true;
#pragma unroll
		for (int e = 0; e < 8; e++) {
			gt = gt && d > nb[e];
			lt = lt && d < nb[e];
		}
		return gt || lt;
	}
};

__device__ __forceinline__ float grad(float hi, float lo, float unit) { return (float)(0.5 * (double)(hi - lo) / (double)unit); }

__device__ __forceinline__ float at(const float* g, const OctaveView& v, int z, int y, int x) { return g[((size_t)z * v.ny + y) * v.nx + x]; }

struct OrientParams {
	float beta, gamma, gradient_threshold;
	int octave;
};

// assignOrientation (:849-1049), one thread per candidate: the window is walked in the reference's (z, y, x) order, so every
// accumulator sees the same sequence of rounded additions.  Writes the candidate record (5 ints), the keypoint record
// (s3::KP_FLOATS floats) and keep[m].
__global__ void __launch_bounds__(128) orientation_kernel(OctaveView v, OrientParams prm, const long long* __restrict__ sel, int n_cand,
	int* __restrict__ cand_out, float* __restrict__ kp_out, int* __restrict__ keep) {
	const int m = blockIdx.x * blockDim.x + threadIdx.x;
	if (m >= n_cand) return;
	const size_t N = (size_t)v.nx * v.ny * v.nz;
	const int layer = 1 + (int)(sel[m] / (long long)N);
	const size_t p = (size_t)(sel[m] % (long long)N);
	const int cx = (int)(p % v.nx), cy = (int)((p / v.nx) % v.ny), cz = (int)(p / ((size_t)v.nx * v.ny));
	int* cr = cand_out + 5 * (size_t)m;
	cr[0] = prm.octave, cr[1] = layer, cr[2] = cz, cr[3] = cy, cr[4] = cx;
	const float* g = v.g[layer];
	const float scale = v.scale[layer];
	const float clx = (float)cx, cly = (float)cy, clz = (float)cz;
	const float ux = v.unit[0], uy = v.unit[1], uz = v.unit[2];

	const float sigma_w = 1.5f * scale;
	const float window_radius = 3.f * sigma_w;
	const int B = s3::IMG_BORDER;
	int x_min = (int)floorf(clx - window_radius / ux);
	x_min = x_min > B ? x_min : B;
	int x_max = (int)ceilf(clx + window_radius / ux);
	x_max = x_max < v.nx - B ? x_max : v.nx - B;
	int y_min = (int)floorf(cly - window_radius / uy);
	y_min = y_min > B ? y_min : B;
	int y_max = (int)ceilf(cly + window_radius * uy); // sic (:870)
	y_max = y_max < v.ny - B ? y_max : v.ny - B;
	int z_min = (int)floorf(clz - window_radius / uz);
	z_min = z_min > B ? z_min : B;
	int z_max = (int)ceilf(clz + window_radius / uz);
	z_max = z_max < v.nz - B ? z_max : v.nz - B;

	float dx = 0.f, dy = 0.f, dz = 0.f;
	float s0 = 0.f, s1 = 0.f, s2 = 0.f, s4 = 0.f, s5 = 0.f, s8 = 0.f;
	for (int i = z_min; i < z_max; i++)
		for (int j = y_min; j < y_max; j++)
			for (int k = x_min; k < x_max; k++) {
				const float px = ((float)k - clx) * ux;
				const float py = ((float)j - cly) * uy;
				const float pz = ((float)i - clz) * uz;
				const float dist = sqrtf(px * px + py * py + pz * pz);
				if (dist <= window_radius) {
					const float r = dist / sigma_w;
					const float w = s3::exp_f(-0.5f * (r * r));
					const float gx = grad(at(g, v, i, j, k + 1), at(g, v, i, j, k - 1), ux);
					const float gy = grad(at(g, v, i, j + 1, k), at(g, v, i, j - 1, k), uy);
					const float gz = grad(at(g, v, i + 1, j, k), at(g, v, i - 1, j, k), uz);
					s0 += gx * gx * w;
					s1 += gx * gy * w;
					s2 += gx * gz * w;
					s4 += gy * gy * w;
					s5 += gy * gz * w;
					s8 += gz * gz * w;
					dx += gx * w;
					dy += gy * w;
					dz += gz * w;
				}
			}
	float* kp = kp_out + (size_t)s3::KP_FLOATS * m;
	keep[m] = 0;
	if ((dx * dx + dy * dy + dz * dz) < prm.gradient_threshold) return;
	const float st[9] = { s0, s1, s2, s1, s4, s5, s2, s5, s8 };
	float ev[3], evec[9];
	s3::eig3(st, ev, evec);
	if ((ev[1] / ev[0]) > prm.beta || (ev[2] / ev[1]) > prm.beta || fabsf(ev[0] - ev[1]) < FLT_EPSILON || fabsf(ev[1] - ev[2]) < FLT_EPSILON
		|| fabsf(ev[2] - ev[0]) < FLT_EPSILON)
		return;
	const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
	float cos_phi = FLT_MAX;
	for (int e = 0; e < 2; e++) {
		float* q = evec + 3 * e;
		const float qd = q[0] * dx + q[1] * dy + q[2] * dz;
		const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
		const float c = fabsf(qd / (qn * dnorm));
		cos_phi = cos_phi < c ? cos_phi : c;
		const float sgn = qd > 0 ? 1.f : -1.f;
		q[0] *= sgn;
		q[1] *= sgn;
		q[2] *= sgn;
	}
	if (cos_phi < prm.gamma) return;
	const float* r1 = evec;
	const float* r2 = evec + 3;
	const float f = (float)(1 << prm.octave); // pow(2.f, octave) (:1044), exact
	kp[0] = clx, kp[1] = cly, kp[2] = clz;
	kp[3] = clx * f, kp[4] = cly * f, kp[5] = clz * f;
	kp[6] = (float)prm.octave, kp[7] = (float)layer, kp[8] = scale;
	for (int c = 0; c < 3; c++) {
		kp[9 + c] = r1[c];
		kp[12 + c] = r2[c];
	}
	kp[15] = r1[1] * r2[2] - r1[2] * r2[1];
	kp[16] = r1[2] * r2[0] - r1[0] * r2[2];
	kp[17] = r1[0] * r2[1] - r1[1] * r2[0];
	keep[m] = 1;
}

// Move the kept candidates' keypoint records to the image's keypoint list (order kept).
__global__ void gather_kp_kernel(const float* __restrict__ kp_tmp, const int* __restrict__ kept_idx, const int* __restrict__ n_kept, float* __restrict__ kp) {
	const int n = *n_kept;
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * s3::KP_FLOATS; i += gridDim.x * blockDim.x) {
		const int m = i / s3::KP_FLOATS, f = i % s3::KP_FLOATS;
		kp[i] = kp_tmp[(size_t)kept_idx[m] * s3::KP_FLOATS + f];
	}
}

constexpr int DESC_THREADS = 256;

// constructDescriptor (:1051-1249), one CTA per keypoint.  The window's voxels are taken DESC_THREADS at a time in the
// reference's (z, y, x) order; each thread evaluates one voxel (rotation, weight, icosahedron face, trilinear cube weights) and
// the voxels that contribute are packed in order into shared memory.  Then each of 64 owner threads, one per 4x4x4 cube, walks
// the packed voxels in order and adds their contributions to its cube's 12 bins: every bin is summed in the reference's voxel
// order, without atomics.  Normalisation sums run sequentially on one thread, as in the reference.
__global__ void __launch_bounds__(DESC_THREADS) descriptor_kernel(OctaveView v, const float* __restrict__ kps, float truncate_threshold,
	float* __restrict__ desc) {
	__shared__ float s_bins[s3::DESC];
	__shared__ float s_gm[DESC_THREADS], s_b[3][DESC_THREADS], s_dec[3][DESC_THREADS];
	__shared__ int s_base[DESC_THREADS], s_face[DESC_THREADS];
	__shared__ int s_warp[DESC_THREADS / 32];
	__shared__ float s_inv;
	const float* kp = kps + (size_t)s3::KP_FLOATS * blockIdx.x;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	for (int b = tid; b < s3::DESC; b += DESC_THREADS) s_bins[b] = 0.f;
	const float clx = kp[0], cly = kp[1], clz = kp[2];
	const int layer = (int)kp[7];
	const float scale = kp[8];
	float R[9];
	for (int c = 0; c < 9; c++) R[c] = kp[9 + c];
	const float* g = v.g[layer];
	const float ux = v.unit[0], uy = v.unit[1], uz = v.unit[2];
	const float sqrt_2 = sqrtf(2.f);
	const float sigma = 5.f * sqrt_2 * scale;
	const float sphere_radius = 2.f * sigma;
	const float cube_radius = sphere_radius / sqrt_2;
	const int B = s3::IMG_BORDER;
	int x_min = (int)floorf(clx - sphere_radius / ux);
	x_min = x_min > B ? x_min : B;
	int x_max = (int)ceilf(clx + sphere_radius / ux);
	x_max = x_max < v.nx - B ? x_max : v.nx - B;
	int y_min = (int)floorf(cly - sphere_radius / uy);
	y_min = y_min > B ? y_min : B;
	int y_max = (int)ceilf(cly + sphere_radius / uy);
	y_max = y_max < v.ny - B ? y_max : v.ny - B;
	int z_min = (int)floorf(clz - sphere_radius / uz);
	z_min = z_min > B ? z_min : B;
	int z_max = (int)ceilf(clz + sphere_radius / uz);
	z_max = z_max < v.nz - B ? z_max : v.nz - B;
	const int wx = max(x_max - x_min, 0), wy = max(y_max - y_min, 0), wz = max(z_max - z_min, 0);
	const long long total = (long long)wx * wy * wz;
	const int owner_x = tid & 3, owner_y = (tid >> 2) & 3, owner_z = (tid >> 4) & 3;
	__syncthreads();

	for (long long base = 0; base < total; base += DESC_THREADS) {
		const long long id = base + tid;
		bool ok = false;
		float gm = 0.f, bary[3] = { 0.f, 0.f, 0.f }, dec[3] = { 0.f, 0.f, 0.f };
		int face = -1, packed = 0;
		if (id < total) {
			const int k = x_min + (int)(id % wx);
			const int j = y_min + (int)((id / wx) % wy);
			const int i = z_min + (int)(id / ((long long)wx * wy));
			float p[3] = { (float)k - clx, (float)j - cly, (float)i - clz };
			p[0] *= ux;
			p[1] *= uy;
			p[2] *= uz;
			const float dist = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
			if (dist <= sphere_radius) {
				float sub[3];
				for (int a = 0; a < 3; a++) {
					const float rot = R[3 * a] * p[0] + R[3 * a + 1] * p[1] + R[3 * a + 2] * p[2];
					sub[a] = 2.f * (rot + cube_radius) / cube_radius;
					sub[a] -= 0.5f;
				}
				if (!(sub[0] <= -0.5f || sub[1] <= -0.5f || sub[2] <= -0.5f || sub[0] >= 3.5f || sub[1] >= 3.5f || sub[2] >= 3.5f)) {
					const double t = (double)(dist / sigma);
					const float w = s3::exp_f(-0.5 * (t * t));
					float gr[3] = { grad(at(g, v, i, j, k + 1), at(g, v, i, j, k - 1), ux), grad(at(g, v, i, j + 1, k), at(g, v, i, j - 1, k), uy),
						grad(at(g, v, i + 1, j, k), at(g, v, i - 1, j, k), uz) };
					gr[0] = w * gr[0];
					gr[1] = w * gr[1];
					gr[2] = w * gr[2];
					float rg[3];
					for (int a = 0; a < 3; a++) rg[a] = R[3 * a] * gr[0] + R[3 * a + 1] * gr[1] + R[3 * a + 2] * gr[2];
					gm = sqrtf(rg[0] * rg[0] + rg[1] * rg[1] + rg[2] * rg[2]);
					if (!(gm * gm < FLT_EPSILON * 10.f)) {
						face = s3::ico_face(rg, c_ico_v, c_ico_f, bary);
						if (face >= 0) {
							ok = true;
							for (int a = 0; a < 3; a++) dec[a] = sub[a] - floorf(sub[a]);
							// (int)sub truncates toward zero, as the reference's cube index does (:1185-1187)
							packed = ((int)sub[0] + 1) | (((int)sub[1] + 1) << 4) | (((int)sub[2] + 1) << 8);
						}
					}
				}
			}
		}
		// pack the contributing voxels in window order
		const unsigned bal = __ballot_sync(0xffffffffu, ok);
		if (lane == 0) s_warp[wid] = __popc(bal);
		__syncthreads();
		int pos = __popc(bal & ((1u << lane) - 1u)), count = 0;
		for (int w = 0; w < DESC_THREADS / 32; w++) {
			pos += w < wid ? s_warp[w] : 0;
			count += s_warp[w];
		}
		if (ok) {
			s_gm[pos] = gm;
			s_face[pos] = face;
			s_base[pos] = packed;
			for (int a = 0; a < 3; a++) {
				s_b[a][pos] = bary[a];
				s_dec[a][pos] = dec[a];
			}
		}
		__syncthreads();
		if (tid < 64) {
			float* bins = s_bins + 12 * tid;
			for (int e = 0; e < count; e++) {
				const int pk = s_base[e];
				const int ddx = owner_x - ((pk & 15) - 1), ddy = owner_y - (((pk >> 4) & 15) - 1), ddz = owner_z - (((pk >> 8) & 15) - 1);
				if ((unsigned)ddx > 1u || (unsigned)ddy > 1u || (unsigned)ddz > 1u) continue;
				const float iw = ((ddx == 0) ? (1.f - s_dec[0][e]) : s_dec[0][e]) * ((ddy == 0) ? (1.f - s_dec[1][e]) : s_dec[1][e])
					* ((ddz == 0) ? (1.f - s_dec[2][e]) : s_dec[2][e]);
				const int f = s_face[e];
				const float m = s_gm[e];
				bins[c_ico_f[3 * f]] += m * iw * s_b[0][e];
				bins[c_ico_f[3 * f + 1]] += m * iw * s_b[1][e];
				bins[c_ico_f[3 * f + 2]] += m * iw * s_b[2][e];
			}
		}
		__syncthreads();
	}
	for (int pass = 0; pass < 2; pass++) {
		if (tid == 0) {
			float sq = 0;
			for (int b = 0; b < s3::DESC; b++) sq += s_bins[b] * s_bins[b];
			s_inv = 1.f / (sqrtf(sq) + FLT_EPSILON);
		}
		__syncthreads();
		const float inv = s_inv;
		for (int b = tid; b < s3::DESC; b += DESC_THREADS) {
			float d = s_bins[b] * inv;
			if (pass == 0) d = (d < truncate_threshold) ? d : truncate_threshold;
			s_bins[b] = d;
		}
		__syncthreads();
	}
	float* out = desc + (size_t)s3::DESC * blockIdx.x;
	for (int b = tid; b < s3::DESC; b += DESC_THREADS) out[b] = s_bins[b];
}

// ---- matching -----------------------------------------------------------------------------------------------------------
// (distance, index) pairs ordered lexicographically: the top two under this order are exactly what the reference's sequential
// scan with strict '<' keeps (the first index wins a tie); NaN distances never enter, as in the scan.
struct Top2 {
	float d0, d1;
	int j0, j1;
};
__device__ __forceinline__ bool lex_less(float d, int j, float e, int k) { return d < e || (d == e && j < k); }
__device__ __forceinline__ void top2_insert(Top2& t, float d, int j) {
	if (lex_less(d, j, t.d0, t.j0)) {
		t.d1 = t.d0, t.j1 = t.j0, t.d0 = d, t.j0 = j;
	} else if (lex_less(d, j, t.d1, t.j1)) {
		t.d1 = d, t.j1 = j;
	}
}

constexpr int MT = 64, MK = 32; // tile: 64 reference rows x 64 target rows, 32 components per stage; 256 threads, 4 x 4 pairs each

// Squared distances of a 64-row block of reference descriptors against the target rows of one segment; each pair's sum runs over
// k = 0..767 in order with separately rounded subtract, multiply and add (:1276-1280).  Writes the segment's per-row top two.
__global__ void __launch_bounds__(256) match_kernel(const float* __restrict__ d1, int n1, const float* __restrict__ d2, int n2, int tiles_per_seg,
	float4* __restrict__ part) {
	__shared__ float sa[MK][MT + 1], sb[MK][MT + 1];
	const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
	const int row0 = blockIdx.x * MT;
	Top2 best[4];
	for (int a = 0; a < 4; a++) best[a] = Top2{ FLT_MAX, FLT_MAX, -1, -1 };
	const int tile_begin = blockIdx.y * tiles_per_seg;
	const int tile_end = min(tile_begin + tiles_per_seg, (n2 + MT - 1) / MT);
	for (int tile = tile_begin; tile < tile_end; tile++) {
		const int col0 = tile * MT;
		float acc[4][4];
		for (int a = 0; a < 4; a++)
			for (int b = 0; b < 4; b++) acc[a][b] = 0.f;
		for (int k0 = 0; k0 < s3::DESC; k0 += MK) {
			__syncthreads();
			for (int e = tid; e < MT * MK; e += 256) {
				const int r = e / MK, k = e % MK;
				sa[k][r] = row0 + r < n1 ? d1[(size_t)(row0 + r) * s3::DESC + k0 + k] : 0.f;
				sb[k][r] = col0 + r < n2 ? d2[(size_t)(col0 + r) * s3::DESC + k0 + k] : 0.f;
			}
			__syncthreads();
#pragma unroll 8
			for (int k = 0; k < MK; k++) {
				float a[4], b[4];
				for (int q = 0; q < 4; q++) {
					a[q] = sa[k][ty * 4 + q];
					b[q] = sb[k][tx * 4 + q];
				}
				for (int p = 0; p < 4; p++)
					for (int q = 0; q < 4; q++) {
						const float diff = a[p] - b[q];
						acc[p][q] = acc[p][q] + diff * diff;
					}
			}
		}
		for (int q = 0; q < 4; q++) { // columns in ascending order
			const int j = col0 + tx * 4 + q;
			if (j >= n2) break;
			for (int p = 0; p < 4; p++) top2_insert(best[p], acc[p][q], j);
		}
	}
	// merge the 16 threads of each row group (lanes ty*16 .. ty*16+15 of one warp)
	for (int p = 0; p < 4; p++) {
		Top2 t = best[p];
		for (int o = 8; o; o >>= 1) {
			const float e0 = __shfl_xor_sync(0xffffffffu, t.d0, o), e1 = __shfl_xor_sync(0xffffffffu, t.d1, o);
			const int k0 = __shfl_xor_sync(0xffffffffu, t.j0, o), k1 = __shfl_xor_sync(0xffffffffu, t.j1, o);
			if (k0 >= 0) top2_insert(t, e0, k0);
			if (k1 >= 0) top2_insert(t, e1, k1);
		}
		const int row = row0 + ty * 4 + p;
		if (tx == 0 && row < n1) part[(size_t)blockIdx.y * n1 + row] = make_float4(t.d0, __int_as_float(t.j0), t.d1, __int_as_float(t.j1));
	}
}

// Merge the segments of each row: out[i] = (d0, index0, d1) of the whole target set.
__global__ void match_merge_kernel(const float4* __restrict__ part, int n1, int segs, float* __restrict__ out) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n1) return;
	Top2 t{ FLT_MAX, FLT_MAX, -1, -1 };
	for (int s = 0; s < segs; s++) {
		const float4 p = part[(size_t)s * n1 + i];
		const int k0 = __float_as_int(p.y), k1 = __float_as_int(p.w);
		if (k0 >= 0) top2_insert(t, p.x, k0);
		if (k1 >= 0) top2_insert(t, p.z, k1);
	}
	out[3 * i] = t.d0;
	out[3 * i + 1] = __int_as_float(t.j0);
	out[3 * i + 2] = t.d1;
}

// ---- host side -----------------------------------------------------------------------------------------------------------

// Times stretches of stream work into stage slots.  A stage runs at most once between two collections, so it has one pair of
// events (Sift3d::ev); elapsed times are read after the next synchronisation.
struct StageTimer {
	Sift3d* s;
	cudaStream_t st;
	unsigned pending = 0;
	cudaError_t begin(int k) { return cudaEventRecord(s->ev[2 * k], st); }
	cudaError_t end(int k) {
		pending |= 1u << k;
		return cudaEventRecord(s->ev[2 * k + 1], st);
	}
	void collect() { // after a synchronisation
		for (int k = 0; k < SIFT3D_STAGES; k++) {
			float ms = 0.f;
			if ((pending >> k & 1) && cudaEventElapsedTime(&ms, s->ev[2 * k], s->ev[2 * k + 1]) == cudaSuccess) s->stage_ms[k] += ms;
		}
		pending = 0;
	}
	// end stage k, copy `bytes` back from the device, wait for them and collect
	cudaError_t finish(int k, void* dst, const void* src, size_t bytes) {
		cudaError_t e = end(k);
		if (e == cudaSuccess && (e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st)) == cudaSuccess) e = cudaStreamSynchronize(st);
		if (e == cudaSuccess) collect();
		return e;
	}
};

// The three passes of one blur (x, y into the scratch volume, z) of an oc.nx x oc.ny x oc.nz layer
cudaError_t blur(const float* src, float* dst, float* tmp, const Sift3dOctave& oc, const Sift3dLayer& b, cudaStream_t st, long long* launches) {
	const dim3 blk(32, 8), grd((oc.nx + 31) / 32, (oc.ny + 7) / 8, std::min(oc.nz, 64));
	cudaError_t e;
	blur_axis_kernel<0><<<grd, blk, 0, st>>>(src, dst, oc.nx, oc.ny, oc.nz, b.radius[0], b.w[0]);
	if ((e = launched(launches)) != cudaSuccess) return e;
	blur_axis_kernel<1><<<grd, blk, 0, st>>>(dst, tmp, oc.nx, oc.ny, oc.nz, b.radius[1], b.w[1]);
	if ((e = launched(launches)) != cudaSuccess) return e;
	blur_axis_kernel<2><<<grd, blk, 0, st>>>(tmp, dst, oc.nx, oc.ny, oc.nz, b.radius[2], b.w[2]);
	return launched(launches);
}

// One image's candidates, max|DoG|, keypoints and descriptors into s->img[which], octave by octave.  counters: the max|DoG| bits
// of the octave's DoG layers, then the candidate and the kept count.
cudaError_t extract(Sift3d* s, const Sift3dPlan& plan, int which, const float* d_img, const float* cfg, int sm_count, cudaStream_t st,
	StageTimer& tm, long long* launches) {
	Sift3dImage& out = s->img[which];
	const int L = plan.L, nol = L - 3;
	out.n_cand = out.n_kp = 0;
	out.max_abs.clear();
	const size_t N0 = (size_t)plan.octave[0].nx * plan.octave[0].ny * plan.octave[0].nz;
	cudaError_t e;
	if ((e = grow(s->layers, N0 * L * sizeof(float), st)) != cudaSuccess || (e = grow(s->tmp, N0 * sizeof(float), st)) != cudaSuccess
		|| (e = grow(s->sel, N0 * nol * sizeof(long long), st)) != cudaSuccess
		|| (e = grow(s->counters, (SIFT3D_MAX_L + 2) * sizeof(int), st)) != cudaSuccess)
		return e;
	float* const tmp = s->tmp.as<float>();
	long long* const sel = s->sel.as<long long>();
	int* const counters = s->counters.as<int>();
	int* const n_found = counters + SIFT3D_MAX_L; // candidates, kept
	auto layer = [&](int l) { return s->layers.as<float>() + (size_t)l * N0; };
	const int grid1d = sm_count * 8;
	for (int o = 0; o < plan.n_octave; o++) {
		const Sift3dOctave& oc = plan.octave[o];
		const Sift3dLayer* lay = &plan.layer[(size_t)o * L];
		const size_t N = (size_t)oc.nx * oc.ny * oc.nz;
		// ---- Gaussian layers
		if ((e = tm.begin(4 * which + 0)) != cudaSuccess) return e;
		if (o == 0) {
			if ((e = blur(d_img, layer(0), tmp, oc, lay[0], st, launches)) != cudaSuccess) return e;
		} else {
			downsample_kernel<<<grid1d, 256, 0, st>>>(layer(nol), tmp, plan.octave[o - 1].nx, plan.octave[o - 1].ny, oc.nx, oc.ny, oc.nz);
			if ((e = launched(launches)) != cudaSuccess) return e;
			if ((e = cudaMemcpyAsync(layer(0), tmp, N * sizeof(float), cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return e;
		}
		for (int l = 1; l < L; l++)
			if ((e = blur(layer(l - 1), layer(l), tmp, oc, lay[l], st, launches)) != cudaSuccess) return e;
		std::vector<float> init(L - 1, -1.f), ma(L - 1); // the maxima travel as the int bits of the floats
		if ((e = cudaMemcpyAsync(counters, init.data(), (L - 1) * sizeof(int), cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
		for (int n = 0; n < L - 1; n++) {
			max_abs_kernel<<<grid1d, 256, 0, st>>>(layer(n), layer(n + 1), N, counters + n);
			if ((e = launched(launches)) != cudaSuccess) return e;
		}
		if ((e = tm.finish(4 * which + 0, ma.data(), counters, (L - 1) * sizeof(int))) != cudaSuccess) return e;
		ExtremumPred pred;
		OctaveView& v = pred.v;
		for (int l = 0; l < L; l++) {
			v.g[l] = layer(l);
			v.scale[l] = lay[l].scale;
		}
		v.nx = oc.nx, v.ny = oc.ny, v.nz = oc.nz;
		for (int a = 0; a < 3; a++) v.unit[a] = oc.unit[a];
		for (int n = 0; n < L - 1; n++) pred.thr[n] = cfg[s3::CFG_ALPHA] * ma[n];
		out.max_abs.insert(out.max_abs.end(), ma.begin(), ma.end());
		// ---- extrema: order-preserving selection over (layer, z, y, x)
		const long long items = (long long)nol * (long long)N;
		thrust::counting_iterator<long long> it(0);
		size_t ws = 0;
		if ((e = tm.begin(4 * which + 1)) != cudaSuccess) return e;
		if ((e = cub::DeviceSelect::If(nullptr, ws, it, sel, n_found, items, pred, st)) != cudaSuccess || (e = grow(s->cub_ws, ws, st)) != cudaSuccess
			|| (e = cub::DeviceSelect::If(s->cub_ws.p, ws, it, sel, n_found, items, pred, st)) != cudaSuccess)
			return e;
		++*launches;
		int n_cand = 0;
		if ((e = tm.finish(4 * which + 1, &n_cand, n_found, sizeof(int))) != cudaSuccess) return e;
		if (n_cand == 0) continue;
		// ---- orientation
		if ((e = grow(out.cand, 5 * (out.n_cand + n_cand) * sizeof(int), st, 5 * out.n_cand * sizeof(int))) != cudaSuccess
			|| (e = grow(s->kp_tmp, (size_t)s3::KP_FLOATS * n_cand * sizeof(float), st)) != cudaSuccess
			|| (e = grow(s->keep, n_cand * sizeof(int), st)) != cudaSuccess || (e = grow(s->kept_idx, n_cand * sizeof(int), st)) != cudaSuccess)
			return e;
		if ((e = tm.begin(4 * which + 2)) != cudaSuccess) return e;
		OrientParams prm{ cfg[s3::CFG_BETA], cfg[s3::CFG_GAMMA], cfg[s3::CFG_GRADIENT_THRESHOLD], o };
		float* const kp_tmp = s->kp_tmp.as<float>();
		int *const keep = s->keep.as<int>(), *const kept_idx = s->kept_idx.as<int>();
		orientation_kernel<<<(n_cand + 127) / 128, 128, 0, st>>>(v, prm, sel, n_cand, out.cand.as<int>() + 5 * out.n_cand, kp_tmp, keep);
		if ((e = launched(launches)) != cudaSuccess) return e;
		const thrust::counting_iterator<int> idx(0);
		if ((e = cub::DeviceSelect::Flagged(nullptr, ws, idx, keep, kept_idx, n_found + 1, n_cand, st)) != cudaSuccess
			|| (e = grow(s->cub_ws, ws, st)) != cudaSuccess
			|| (e = cub::DeviceSelect::Flagged(s->cub_ws.p, ws, idx, keep, kept_idx, n_found + 1, n_cand, st)) != cudaSuccess)
			return e;
		++*launches;
		out.n_cand += n_cand;
		int n_kept = 0;
		if ((e = tm.finish(4 * which + 2, &n_kept, n_found + 1, sizeof(int))) != cudaSuccess) return e;
		if (n_kept == 0) continue;
		// ---- descriptors
		const size_t kp_bytes = (size_t)s3::KP_FLOATS * sizeof(float), desc_bytes = (size_t)s3::DESC * sizeof(float);
		if ((e = grow(out.kp, kp_bytes * (out.n_kp + n_kept), st, kp_bytes * out.n_kp)) != cudaSuccess
			|| (e = grow(out.desc, desc_bytes * (out.n_kp + n_kept), st, desc_bytes * out.n_kp)) != cudaSuccess)
			return e;
		if ((e = tm.begin(4 * which + 3)) != cudaSuccess) return e;
		float* kp_o = out.kp.as<float>() + (size_t)s3::KP_FLOATS * out.n_kp;
		gather_kp_kernel<<<std::max(1, std::min(grid1d, (n_kept * s3::KP_FLOATS + 255) / 256)), 256, 0, st>>>(kp_tmp, kept_idx, n_found + 1, kp_o);
		if ((e = launched(launches)) != cudaSuccess) return e;
		float* desc_o = out.desc.as<float>() + (size_t)s3::DESC * out.n_kp;
		descriptor_kernel<<<n_kept, DESC_THREADS, 0, st>>>(v, kp_o, cfg[s3::CFG_TRUNCATE_THRESHOLD], desc_o);
		if ((e = launched(launches)) != cudaSuccess || (e = tm.end(4 * which + 3)) != cudaSuccess) return e;
		out.n_kp += n_kept;
	}
	if ((e = cudaStreamSynchronize(st)) == cudaSuccess) tm.collect();
	return e;
}

// monodirectionalMatch (:1251-1418) after the brute-force scan: ratio test, many-to-one resolution and output, on the host.
// top2: n1 x (d0, index0 as int bits, d1).  pairs: (ref, tar) in output order.
void match_post(const std::vector<float>& top2, size_t n1, float ratio, std::vector<std::pair<int, int>>& pairs) {
	const float r2 = ratio * ratio;
	struct M {
		int ref_idx, tar_idx;
		float dist;
	};
	std::vector<M> km(n1, M{ -1, -1, 0.f });
	for (size_t i = 0; i < n1; i++) {
		const float d0 = top2[3 * i], d1 = top2[3 * i + 2];
		int j0;
		memcpy(&j0, &top2[3 * i + 1], sizeof(int));
		if (d0 < r2 * d1) km[i] = M{ (int)i, j0, d0 };
	}
	// the reference's two std::sort calls (:1307,1325) made stable: a run of equal tar_idx keeps descending ref_idx order
	std::stable_sort(km.begin(), km.end(), [](const M& a, const M& b) { return a.ref_idx > b.ref_idx; });
	size_t matched = 0; // stays 0 if every keypoint passed the ratio test (:1309-1317)
	for (size_t i = 0; i < n1; i++)
		if (km[i].ref_idx == -1) {
			matched = i;
			break;
		}
	pairs.clear();
	if (matched > 1) {
		km.resize(matched);
		std::stable_sort(km.begin(), km.end(), [](const M& a, const M& b) { return a.tar_idx > b.tar_idx; });
		for (size_t s = 0; s < matched;) { // every maximal run of equal tar_idx, the last one included
			size_t e = s + 1;
			while (e < matched && km[e].tar_idx == km[s].tar_idx) e++;
			if (e - s > 1) {
				int ci[2] = { -1, -1 };
				float cd[2] = { FLT_MAX, FLT_MAX };
				for (size_t c = s; c < e; c++) {
					if (km[c].dist < cd[0]) {
						ci[1] = ci[0], cd[1] = cd[0], ci[0] = km[c].ref_idx, cd[0] = km[c].dist;
					} else if (km[c].dist < cd[1]) {
						ci[1] = km[c].ref_idx, cd[1] = km[c].dist;
					}
					km[c].ref_idx = -1;
				}
				if (cd[0] < r2 * cd[1]) km[s].ref_idx = ci[0];
			}
			s = e;
		}
	}
	for (size_t i = 0; i < matched; i++)
		if (km[i].ref_idx > -1) pairs.push_back({ km[i].ref_idx, km[i].tar_idx });
}

} // namespace

cudaError_t sift3d_run(Sift3d* s, const Sift3dPlan& plan, const float* d_ref, const float* d_tar, const float* cfg, float ratio, int sm_count,
	cudaStream_t st, long long* launches) {
	for (float& t : s->stage_ms) t = 0.f;
	cudaError_t e;
	for (cudaEvent_t& ev : s->ev)
		if (!ev && (e = cudaEventCreate(&ev)) != cudaSuccess) return e;
	StageTimer tm{ s, st };
	const float* imgs[2] = { d_ref, d_tar };
	for (int w = 0; w < 2; w++)
		if ((e = extract(s, plan, w, imgs[w], cfg, sm_count, st, tm, launches)) != cudaSuccess) return e;
	s->ref_xyz.clear();
	s->tar_xyz.clear();
	const size_t n1 = s->img[0].n_kp, n2 = s->img[1].n_kp;
	if (n1 == 0) return cudaSuccess;
	if (n1 > 0x7fffffff || n2 > 0x7fffffff) return SIFT3D_TOO_MANY_KEYPOINTS;
	const int row_blocks = (int)((n1 + MT - 1) / MT), col_tiles = (int)((n2 + MT - 1) / MT);
	// split the target rows into segments so that the grid covers the GPU even when the reference set is small
	int segs = std::max(1, std::min(col_tiles, (2 * sm_count + row_blocks - 1) / row_blocks));
	const int tiles_per_seg = std::max(1, (col_tiles + segs - 1) / segs);
	segs = std::max(1, (col_tiles + tiles_per_seg - 1) / tiles_per_seg);
	if ((e = tm.begin(8)) != cudaSuccess) return e;
	if ((e = grow(s->part, (size_t)segs * n1 * sizeof(float4), st)) != cudaSuccess || (e = grow(s->top2, 3 * n1 * sizeof(float), st)) != cudaSuccess)
		return e;
	if (n2 > 0) {
		match_kernel<<<dim3(row_blocks, segs), 256, 0, st>>>(s->img[0].desc.as<float>(), (int)n1, s->img[1].desc.as<float>(), (int)n2, tiles_per_seg,
			s->part.as<float4>());
		if ((e = launched(launches)) != cudaSuccess) return e;
	}
	match_merge_kernel<<<(int)((n1 + 255) / 256), 256, 0, st>>>(s->part.as<float4>(), (int)n1, n2 > 0 ? segs : 0, s->top2.as<float>());
	if ((e = launched(launches)) != cudaSuccess) return e;
	std::vector<float> top2(3 * n1), kp1((size_t)s3::KP_FLOATS * n1), kp2((size_t)s3::KP_FLOATS * n2);
	if ((e = cudaMemcpyAsync(top2.data(), s->top2.p, top2.size() * sizeof(float), cudaMemcpyDeviceToHost, st)) != cudaSuccess
		|| (e = tm.end(8)) != cudaSuccess
		|| (e = cudaMemcpyAsync(kp1.data(), s->img[0].kp.p, kp1.size() * sizeof(float), cudaMemcpyDeviceToHost, st)) != cudaSuccess
		|| (n2 && (e = cudaMemcpyAsync(kp2.data(), s->img[1].kp.p, kp2.size() * sizeof(float), cudaMemcpyDeviceToHost, st)) != cudaSuccess)
		|| (e = cudaStreamSynchronize(st)) != cudaSuccess)
		return e;
	tm.collect();
	const auto t0 = std::chrono::steady_clock::now();
	std::vector<std::pair<int, int>> pairs;
	match_post(top2, n1, ratio, pairs);
	for (const auto& pr : pairs) {
		for (int a = 0; a < 3; a++) {
			s->ref_xyz.push_back(kp1[(size_t)s3::KP_FLOATS * pr.first + 3 + a]);
			s->tar_xyz.push_back(kp2[(size_t)s3::KP_FLOATS * pr.second + 3 + a]);
		}
	}
	s->stage_ms[9] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
	return cudaSuccess;
}

} // namespace ocb
