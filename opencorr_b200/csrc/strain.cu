// strain.cu -- Strain post-processing of a POI queue (SURVEY.md section 8(f) N4) for sm_90a.
//
// Replaces Strain::prepare + Strain::compute(std::vector<POI2D>&) / (std::vector<POI3D>&) of the
// reference (src/oc_strain.cpp:100-111,150-156,158-250,373-487): for every POI with ZNCC >= threshold,
// collect the POIs within `subregion_radius` (nanoflann kd-tree radius search in the reference,
// src/oc_nearest_neighbor.cpp:124-139: squared distance STRICTLY below radius^2), fall back to the k
// nearest POIs when fewer than `neighbor_number_min` were found (:141-157), keep those with
// ZNCC >= threshold, and fit a plane to u, v (, w) over them by least squares (Eigen
// colPivHouseholderQr in the reference); the plane's slopes are the displacement gradients, from
// which the Cauchy or Green strains follow.
//
// GPU mapping: no tree.  The POIs are binned into a uniform grid (cell edge >= |radius|) by one
// stable radix sort of (cell id, POI index); a warp per POI then scans the 3 (2D) / 9 (3D) runs of
// x-adjacent cells that can hold neighbours -- contiguous in the sorted order, found by binary
// search -- with coalesced 16-byte loads, and accumulates the normal equations in FP64 (12 / 22
// sums per lane, shuffle-reduced).  Lane 0 solves the 3x3 / 4x4 system with pivoting.  The rare
// k-nearest fallback is k brute-force selection passes over the sorted array by the same warp.
#include <string.h>

#include <algorithm>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "ocb_kernels.h"

namespace ocb {

namespace {

// MODE 2: POI2D, 3: POI3D, 23: POI2DS (stereo DIC, src/oc_strain.cpp:252-371: neighbours are searched in the image plane
// of the primary view, the plane fit runs over the reconstructed 3D coordinates ref_coor and u, v, w; a POI counts when
// r1r2, r1t1 and r1t2 ZNCC all pass the threshold).  SD = search dimensions, FD = fit dimensions, FC = offset of the
// fit coordinates in the record, Z0 / NZ = the ZNCC fields that must pass.
// POI2DS record (src/oc_poi.h:140-186), 28 floats: x y | u v w | r1r2 r1t1 r1t2 r2_x r2_y t1_x t1_y t2_x t2_y | ref_coor | tar_coor | e[6] | subset_radius
template <int MODE> struct SL;
template <> struct SL<2> { enum { NF = P2_N, SD = 2, FD = 2, FC = 0, Z0 = P2_ZNCC, NZ = 1, STRAIN = P2_STRAIN, U = P2_DEF + D2_U, V = P2_DEF + D2_V, W = P2_DEF + D2_V }; };
template <> struct SL<3> { enum { NF = P3_N, SD = 3, FD = 3, FC = 0, Z0 = P3_ZNCC, NZ = 1, STRAIN = P3_STRAIN, U = P3_DEF + 0, V = P3_DEF + 4, W = P3_DEF + 8 }; };
template <> struct SL<23> { enum { NF = 28, SD = 2, FD = 3, FC = 14, Z0 = 5, NZ = 3, STRAIN = 20, U = 2, V = 3, W = 4 }; };

struct StrainGrid {
	float lo[3];
	float inv_cell;
	int nc[3];
	unsigned int n_cells; // sentinel key for POIs with non-finite coordinates
};

__device__ __forceinline__ unsigned int float_to_ordered(float f) {
	unsigned int u = __float_as_uint(f);
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
inline float ordered_to_float(unsigned int o) {
	unsigned int u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
	float f;
	memcpy(&f, &u, sizeof(f));
	return f;
}

// bbox[0..2] = min (ordered encoding), bbox[3..5] = max
template <int MODE>
__global__ void strain_bbox_kernel(const float* __restrict__ pois, int n, unsigned int* __restrict__ bbox) {
	typedef SL<MODE> L;
	constexpr int D = L::SD;
	unsigned int mn[3] = { 0xffffffffu, 0xffffffffu, 0xffffffffu }, mx[3] = { 0u, 0u, 0u };
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float* p = pois + (size_t)i * L::NF;
		bool fin = true;
#pragma unroll
		for (int d = 0; d < D; d++) fin = fin && isfinite(p[d]);
		if (!fin) continue;
#pragma unroll
		for (int d = 0; d < D; d++) {
			const unsigned int o = float_to_ordered(p[d]);
			mn[d] = min(mn[d], o);
			mx[d] = max(mx[d], o);
		}
	}
#pragma unroll
	for (int d = 0; d < D; d++) {
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			mn[d] = min(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
			mx[d] = max(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
		}
		if ((threadIdx.x & 31) == 0) {
			atomicMin(bbox + d, mn[d]);
			atomicMax(bbox + 3 + d, mx[d]);
		}
	}
}

template <int D>
__device__ __forceinline__ void strain_cell(const StrainGrid& g, const float* p, int* c) {
#pragma unroll
	for (int d = 0; d < 3; d++) {
		if (d < D) {
			int v = (int)floorf((p[d] - g.lo[d]) * g.inv_cell);
			c[d] = v < 0 ? 0 : (v >= g.nc[d] ? g.nc[d] - 1 : v);
		} else {
			c[d] = 0;
		}
	}
}

template <int MODE>
__global__ void strain_keys_kernel(const float* __restrict__ pois, int n, StrainGrid g, unsigned int* __restrict__ keys, int* __restrict__ vals) {
	typedef SL<MODE> L;
	constexpr int D = L::SD;
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float* p = pois + (size_t)i * L::NF;
		bool fin = true;
#pragma unroll
		for (int d = 0; d < D; d++) fin = fin && isfinite(p[d]);
		unsigned int key = g.n_cells;
		if (fin) {
			int c[3];
			strain_cell<D>(g, p, c);
			key = (unsigned int)((c[2] * g.nc[1] + c[1]) * g.nc[0] + c[0]);
		}
		keys[i] = key;
		vals[i] = i;
	}
}

// sorted, compact copies: pos = {x, y, z|0, fit flag (every ZNCC >= threshold)}, disp = {u, v, w|0, 0},
// fpos = the fit coordinates when they are not the search coordinates (POI2DS: ref_coor)
template <int MODE>
__global__ void strain_gather_kernel(const float* __restrict__ pois, int n, const int* __restrict__ order, float zncc_threshold,
	float4* __restrict__ pos, float4* __restrict__ disp, float4* __restrict__ fpos) {
	typedef SL<MODE> L;
	for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
		const float* p = pois + (size_t)order[s] * L::NF;
		bool good = true;
#pragma unroll
		for (int k = 0; k < L::NZ; k++) good = good && (p[L::Z0 + k] >= zncc_threshold);
		pos[s] = make_float4(p[0], p[1], L::SD == 3 ? p[2] : 0.f, good ? 1.f : 0.f);
		disp[s] = make_float4(p[L::U], p[L::V], L::FD == 3 ? p[L::W] : 0.f, 0.f);
		if (L::FC != 0) fpos[s] = make_float4(p[L::FC], p[L::FC + 1], p[L::FC + 2], 0.f);
	}
}

__device__ __forceinline__ int lower_bound_u32(const unsigned int* __restrict__ a, int n, unsigned int key) {
	int lo = 0, hi = n;
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
	}
	return lo;
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	return v;
}

// squared distance in float, one rounding per operation, x then y then z
// (nanoflann L2_Simple_Adaptor::evalMetric accumulates diff*diff in the element type)
template <int D>
__device__ __forceinline__ float dist2(const float4& a, const float4& b) {
	float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y);
	float r = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
	if (D == 3) {
		float dz = __fsub_rn(a.z, b.z);
		r = __fadd_rn(r, __fmul_rn(dz, dz));
	}
	return r;
}

// normal-equation sums for the fit  [1, dx, dy(, dz)] * g = u | v (| w)
//   A: upper triangle of sum phi phi^T, C(C+1)/2 entries row-major; B: sum phi * disp_k, D x C
template <int D>
struct FitSums {
	static constexpr int C = D + 1;
	static constexpr int NA = C * (C + 1) / 2;
	double a[NA];
	double b[D][C];
	__device__ __forceinline__ void clear() {
#pragma unroll
		for (int i = 0; i < NA; i++) a[i] = 0.0;
#pragma unroll
		for (int k = 0; k < D; k++)
#pragma unroll
			for (int i = 0; i < C; i++) b[k][i] = 0.0;
	}
	__device__ __forceinline__ void add(const float4& centre, const float4& q, const float4& dq) {
		double phi[C];
		phi[0] = 1.0;
		phi[1] = (double)__fsub_rn(q.x, centre.x); // coefficient_matrix(i,1) = pois_fit[i].x - poi->x in float (:208-209)
		phi[2] = (double)__fsub_rn(q.y, centre.y);
		if (D == 3) phi[C - 1] = (double)__fsub_rn(q.z, centre.z);
		const double disp[3] = { (double)dq.x, (double)dq.y, (double)dq.z };
		int t = 0;
#pragma unroll
		for (int i = 0; i < C; i++)
#pragma unroll
			for (int j = i; j < C; j++) a[t++] += phi[i] * phi[j];
#pragma unroll
		for (int k = 0; k < D; k++)
#pragma unroll
			for (int i = 0; i < C; i++) b[k][i] += phi[i] * disp[k];
	}
	__device__ __forceinline__ void reduce() {
#pragma unroll
		for (int i = 0; i < NA; i++) a[i] = warp_sum_d(a[i]);
#pragma unroll
		for (int k = 0; k < D; k++)
#pragma unroll
			for (int i = 0; i < C; i++) b[k][i] = warp_sum_d(b[k][i]);
	}
};

// Solve the symmetric C x C normal equations for D right-hand sides by Gaussian elimination with diagonal
// (symmetric) pivoting; unknowns whose pivot vanishes (rank-deficient fit, e.g. collinear neighbours) are set
// to 0, the basic solution a rank-revealing QR returns.
template <int D>
__device__ void solve_normal(const FitSums<D>& s, double x[D][D + 1]) {
	constexpr int C = D + 1;
	double M[C][C], R[D][C];
	int t = 0;
	for (int i = 0; i < C; i++)
		for (int j = i; j < C; j++) { M[i][j] = s.a[t]; M[j][i] = s.a[t]; t++; }
	for (int k = 0; k < D; k++)
		for (int i = 0; i < C; i++) { R[k][i] = s.b[k][i]; x[k][i] = 0.0; }
	int perm[C];
	for (int i = 0; i < C; i++) perm[i] = i;
	double scale = 0.0;
	for (int i = 0; i < C; i++) scale = fmax(scale, fabs(M[i][i]));
	int rank = 0;
	for (int k = 0; k < C; k++) {
		int best = k;
		for (int i = k + 1; i < C; i++)
			if (M[perm[i]][perm[i]] > M[perm[best]][perm[best]]) best = i;
		const int pk = perm[best];
		perm[best] = perm[k];
		perm[k] = pk;
		const double piv = M[pk][pk];
		if (!(piv > scale * 1e-12)) break;
		rank++;
		for (int ii = k + 1; ii < C; ii++) {
			const int pi = perm[ii];
			const double f = M[pi][pk] / piv;
			for (int jj = k; jj < C; jj++) M[pi][perm[jj]] -= f * M[pk][perm[jj]];
			for (int r = 0; r < D; r++) R[r][pi] -= f * R[r][pk];
		}
	}
	for (int r = 0; r < D; r++)
		for (int k = rank - 1; k >= 0; k--) {
			const int pk = perm[k];
			double v = R[r][pk];
			for (int jj = k + 1; jj < rank; jj++) v -= M[pk][perm[jj]] * x[r][perm[jj]];
			x[r][pk] = v / M[pk][pk];
		}
}

template <int MODE>
__global__ void __launch_bounds__(256) strain_kernel(float* __restrict__ pois, int n_valid, StrainGrid g, const unsigned int* __restrict__ keys,
	const int* __restrict__ order, const float4* __restrict__ pos, const float4* __restrict__ disp, const float4* __restrict__ fpos, float radius,
	int k_min, int approximation, int only) {
	typedef SL<MODE> L;
	constexpr int D = L::SD, FD = L::FD; // search / fit dimensions
	constexpr int C = FD + 1;
	constexpr int ROWS = D == 2 ? 3 : 9;
	const int lane = threadIdx.x & 31;
	const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int n_warps = (gridDim.x * blockDim.x) >> 5;
	const float r2 = __fmul_rn(radius, radius);
	for (int s = warp_global; s < n_valid; s += n_warps) {
		const float4 centre = __ldg(pos + s);
		if (only >= 0) { // Strain::compute(POI*, queue): that POI only, whatever its own ZNCC
			if (__ldg(order + s) != only) continue;
		} else if (centre.w == 0.f) continue; // Strain::compute(queue): POIs below the ZNCC threshold are skipped (:244-248)
		int c[3];
		{
			const float pc[3] = { centre.x, centre.y, centre.z };
			strain_cell<D>(g, pc, c);
		}
		// runs of x-adjacent cells: one per (y, z) row of the 3x3(x3) cell block
		int run_lo = 0, run_hi = 0;
		if (lane < ROWS) {
			const int cy = c[1] + (lane % 3) - 1, cz = D == 3 ? c[2] + (lane / 3) - 1 : 0;
			if (cy >= 0 && cy < g.nc[1] && cz >= 0 && cz < g.nc[2]) {
				const int cx0 = max(c[0] - 1, 0), cx1 = min(c[0] + 1, g.nc[0] - 1);
				const unsigned int base = (unsigned int)((cz * g.nc[1] + cy) * g.nc[0]);
				run_lo = lower_bound_u32(keys, n_valid, base + cx0);
				run_hi = lower_bound_u32(keys, n_valid, base + cx1 + 1);
			}
		}
		const float4 fcentre = L::FC != 0 ? __ldg(fpos + s) : centre; // origin of the fit coordinates
		FitSums<FD> sums;
		sums.clear();
		int found = 0;
#pragma unroll 1
		for (int row = 0; row < ROWS; row++) {
			const int lo = __shfl_sync(0xffffffffu, run_lo, row), hi = __shfl_sync(0xffffffffu, run_hi, row);
			for (int j = lo + lane; j < hi; j += 32) {
				const float4 q = __ldg(pos + j);
				if (dist2<D>(centre, q) < r2) {
					found++;
					if (q.w != 0.f) sums.add(fcentre, L::FC != 0 ? __ldg(fpos + j) : q, __ldg(disp + j));
				}
			}
		}
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) found += __shfl_xor_sync(0xffffffffu, found, o);
		if (found < k_min) {
			// k-nearest fallback (src/oc_strain.cpp:183-196): k selection passes over all POIs, ordered by
			// (distance^2, original index)
			sums.clear();
			float prev_d = -1.f;
			int prev_i = -1;
			const int k = k_min < n_valid ? k_min : n_valid;
#pragma unroll 1
			for (int pass = 0; pass < k; pass++) {
				float bd = INFINITY;
				int bi = 0x7fffffff, bs = -1;
				for (int j = lane; j < n_valid; j += 32) {
					const float d = dist2<D>(centre, __ldg(pos + j));
					const int oi = __ldg(order + j);
					const bool after = d > prev_d || (d == prev_d && oi > prev_i);
					if (after && (d < bd || (d == bd && oi < bi))) { bd = d; bi = oi; bs = j; }
				}
#pragma unroll
				for (int o = 16; o > 0; o >>= 1) {
					const float od = __shfl_xor_sync(0xffffffffu, bd, o);
					const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
					const int os = __shfl_xor_sync(0xffffffffu, bs, o);
					if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; bs = os; }
				}
				if (bs < 0) break;
				prev_d = bd;
				prev_i = bi;
				if (lane == 0) {
					const float4 q = __ldg(pos + bs);
					if (q.w != 0.f) sums.add(fcentre, L::FC != 0 ? __ldg(fpos + bs) : q, __ldg(disp + bs));
				}
			}
		}
		sums.reduce();
		if (lane == 0 && sums.a[0] >= (double)k_min) { // enough neighbours with good ZNCC (:200-201)
			double x[FD][C];
			solve_normal<FD>(sums, x);
			float* e = pois + (size_t)__ldg(order + s) * L::NF + L::STRAIN;
			if (FD == 2) {
				const float ux = (float)x[0][1], uy = (float)x[0][2], vx = (float)x[1][1], vy = (float)x[1][2];
				if (approximation == 2) { // Green strain (:229-235)
					e[0] = ux + 0.5f * (ux * ux + vx * vx);
					e[1] = vy + 0.5f * (uy * uy + vy * vy);
					e[2] = 0.5f * (uy + vx + uy * ux + vy * vx);
				} else if (approximation == 1) { // Cauchy strain (:222-227)
					e[0] = ux;
					e[1] = vy;
					e[2] = 0.5f * (uy + vx);
				}
			} else {
				const float ux = (float)x[0][1], uy = (float)x[0][2], uz = (float)x[0][C - 1];
				const float vx = (float)x[1][1], vy = (float)x[1][2], vz = (float)x[1][C - 1];
				const float wx = (float)x[FD - 1][1], wy = (float)x[FD - 1][2], wz = (float)x[FD - 1][C - 1];
				if (approximation == 2) { // :455-463
					e[0] = ux + 0.5f * (ux * ux + vx * vx + wx * wx);
					e[1] = vy + 0.5f * (uy * uy + vy * vy + wy * wy);
					e[2] = wz + 0.5f * (uz * uz + vz * vz + wz * wz);
					e[3] = 0.5f * (uy + vx + uy * ux + vy * vx + wy * wx);
					e[4] = 0.5f * (vz + wy + uz * uy + vz * vy + wz * wy);
					e[5] = 0.5f * (wx + uz + ux * uz + vx * vz + wx * wz);
				} else if (approximation == 1) { // :444-453
					e[0] = ux;
					e[1] = vy;
					e[2] = wz;
					e[3] = 0.5f * (uy + vx);
					e[4] = 0.5f * (vz + wy);
					e[5] = 0.5f * (wx + uz);
				}
			}
		}
	}
}

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

} // namespace

// Device scratch layout (one grow-only allocation owned by the context):
//   bbox[8] | keys_in[n] | keys_out[n] | vals_in[n] | vals_out[n] | pos[n] | disp[n] | fpos[n] | cub temp
size_t strain_workspace_bytes(size_t n) {
	size_t cub_bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned int*)nullptr, (unsigned int*)nullptr, (const int*)nullptr, (int*)nullptr,
		(int)n);
	return 256 + 4 * align256(n * 4) + 3 * align256(n * 16) + align256(cub_bytes) + 256;
}

// mode: 2 (POI2D records), 3 (POI3D), 23 (POI2DS)
cudaError_t strain_launch(int mode, float* d_pois, size_t n, float radius, int k_min, float zncc_threshold, int approximation, long long only,
	void* workspace, int sm_count, cudaStream_t stream, long long* launches) {
	char* ws = (char*)workspace;
	unsigned int* d_bbox = (unsigned int*)ws; ws += 256;
	unsigned int* keys_in = (unsigned int*)ws; ws += align256(n * 4);
	unsigned int* keys_out = (unsigned int*)ws; ws += align256(n * 4);
	int* vals_in = (int*)ws; ws += align256(n * 4);
	int* vals_out = (int*)ws; ws += align256(n * 4);
	float4* pos = (float4*)ws; ws += align256(n * 16);
	float4* disp = (float4*)ws; ws += align256(n * 16);
	float4* fpos = (float4*)ws; ws += align256(n * 16);
	void* cub_temp = ws;
	const int dim = mode == 3 ? 3 : 2; // search dimensions
	size_t cub_bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned int*)nullptr, (unsigned int*)nullptr, (const int*)nullptr, (int*)nullptr,
		(int)n);
	const int threads = 256;
	int blocks = (int)((n + threads - 1) / threads);
	if (blocks > sm_count * 8) blocks = sm_count * 8;
	if (blocks < 1) blocks = 1;

	cudaError_t e;
	const unsigned int init[6] = { 0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u };
	if ((e = cudaMemcpyAsync(d_bbox, init, sizeof(init), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
	if (mode == 2) strain_bbox_kernel<2><<<blocks, threads, 0, stream>>>(d_pois, (int)n, d_bbox);
	else if (mode == 3) strain_bbox_kernel<3><<<blocks, threads, 0, stream>>>(d_pois, (int)n, d_bbox);
	else strain_bbox_kernel<23><<<blocks, threads, 0, stream>>>(d_pois, (int)n, d_bbox);
	unsigned int hb[6];
	if ((e = cudaMemcpyAsync(hb, d_bbox, sizeof(hb), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
	if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
	(*launches)++;
	if (hb[0] == 0xffffffffu && hb[3] == 0u) return cudaSuccess; // no POI with finite coordinates

	StrainGrid g;
	float extent = 0.f;
	for (int d = 0; d < 3; d++) {
		g.lo[d] = d < dim ? ordered_to_float(hb[d]) : 0.f;
		const float hi = d < dim ? ordered_to_float(hb[3 + d]) : 0.f;
		if (hi - g.lo[d] > extent) extent = hi - g.lo[d];
	}
	// cell edge >= |radius| so that the 3^D block around a POI's cell holds every point within the radius (the test is
	// dist^2 < radius^2, so a negative radius acts as its magnitude); a non-finite radius takes one cell over the bbox
	// (+-inf: every POI is a neighbour, NaN: none is); grown until the grid has < 2^30 cells
	const float abs_radius = fabsf(radius);
	double cell = !isfinite(abs_radius) ? (double)extent + 1.0 : abs_radius > 0.f ? (double)abs_radius : (double)extent / 64.0 + 1.0;
	if (!(cell > 0.0) || !isfinite(cell)) cell = 1.0;
	while (true) {
		double total = 1.0;
		for (int d = 0; d < 3; d++) {
			const float hi = d < dim ? ordered_to_float(hb[3 + d]) : 0.f;
			const double cnt = d < dim ? floor(((double)hi - (double)g.lo[d]) / cell) + 2.0 : 1.0;
			g.nc[d] = (int)(cnt < 1.0 ? 1.0 : (cnt > 2e9 ? 2e9 : cnt));
			total *= cnt;
		}
		if (total < 1073741824.0) break;
		cell *= 2.0;
	}
	g.inv_cell = (float)(1.0 / cell);
	// the float product (p - lo) * inv_cell may round a point's cell index by one; the neighbourhood scan needs
	// |cell(p) - cell(q)| <= 1 for every pair within the radius, which holds with a 0.1 % safety margin on the edge
	g.inv_cell *= 0.999f;
	g.n_cells = (unsigned int)g.nc[0] * (unsigned int)g.nc[1] * (unsigned int)g.nc[2];

	if (mode == 2) strain_keys_kernel<2><<<blocks, threads, 0, stream>>>(d_pois, (int)n, g, keys_in, vals_in);
	else if (mode == 3) strain_keys_kernel<3><<<blocks, threads, 0, stream>>>(d_pois, (int)n, g, keys_in, vals_in);
	else strain_keys_kernel<23><<<blocks, threads, 0, stream>>>(d_pois, (int)n, g, keys_in, vals_in);
	int end_bit = 1;
	while (end_bit < 32 && (g.n_cells >> end_bit) != 0) end_bit++;
	if ((e = cub::DeviceRadixSort::SortPairs(cub_temp, cub_bytes, keys_in, keys_out, vals_in, vals_out, (int)n, 0, end_bit, stream)) != cudaSuccess)
		return e;
	if (mode == 2) strain_gather_kernel<2><<<blocks, threads, 0, stream>>>(d_pois, (int)n, vals_out, zncc_threshold, pos, disp, fpos);
	else if (mode == 3) strain_gather_kernel<3><<<blocks, threads, 0, stream>>>(d_pois, (int)n, vals_out, zncc_threshold, pos, disp, fpos);
	else strain_gather_kernel<23><<<blocks, threads, 0, stream>>>(d_pois, (int)n, vals_out, zncc_threshold, pos, disp, fpos);
	// POIs with non-finite coordinates carry the sentinel key and sit at the end of the sorted order: the count
	// of valid ones comes from the keys (binary search on the device side would need another round trip)
	int n_valid = (int)n;
	{
		unsigned int last = 0;
		if ((e = cudaMemcpyAsync(&last, keys_out + (n - 1), sizeof(last), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
		if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
		if (last == g.n_cells) { // rare: find the first sentinel on the host
			std::vector<unsigned int> hk(n);
			if ((e = cudaMemcpy(hk.data(), keys_out, n * sizeof(unsigned int), cudaMemcpyDeviceToHost)) != cudaSuccess) return e;
			n_valid = (int)(std::lower_bound(hk.begin(), hk.end(), g.n_cells) - hk.begin());
		}
	}
	(*launches) += 3; // keys, sort (counted once), gather
	if (n_valid > 0) {
		long long warps_needed = n_valid;
		long long grid = (warps_needed * 32 + threads - 1) / threads;
		if (grid > (long long)sm_count * 8) grid = (long long)sm_count * 8;
		if (mode == 2)
			strain_kernel<2><<<(int)grid, threads, 0, stream>>>(d_pois, n_valid, g, keys_out, vals_out, pos, disp, fpos, radius, k_min, approximation, (int)only);
		else if (mode == 3)
			strain_kernel<3><<<(int)grid, threads, 0, stream>>>(d_pois, n_valid, g, keys_out, vals_out, pos, disp, fpos, radius, k_min, approximation, (int)only);
		else
			strain_kernel<23><<<(int)grid, threads, 0, stream>>>(d_pois, n_valid, g, keys_out, vals_out, pos, disp, fpos, radius, k_min, approximation,
				(int)only);
		(*launches)++;
	}
	return cudaGetLastError();
}

} // namespace ocb
