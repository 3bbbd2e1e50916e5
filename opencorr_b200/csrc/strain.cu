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
//
// Over a series of frames that share their positions (strain_series_kernel), the bbox, grid and sort run once on frame 0 and
// each POI's neighbours are searched once; only the fits run per frame.
//
// RegionFit2D / RegionFit3D (region_fit_kernel) is the same search and fit with the neighbours taken from a second set of POIs
// (the reliable ones, binned, sorted and gathered by the same kernels) and the fit itself as the output: its intercept and
// slopes become a queue POI's first-order deformation, an initial guess for IC-GN.
#include <stdint.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>

#include "ocb_kernels.h"

namespace ocb {

namespace {

// The record layout of each kind.  SD = search dimensions, FD = fit dimensions, FC = offset of the fit coordinates in the
// record, Z0 / NZ = the ZNCC fields that must pass.  POI2DS (src/oc_strain.cpp:252-371): neighbours are searched in the image
// plane of the primary view, the plane fit runs over the reconstructed 3D coordinates ref_coor and u, v, w; a POI counts when
// r1r2, r1t1 and r1t2 ZNCC all pass the threshold.
template <PoiKind K> struct SL;
template <> struct SL<PoiKind::POI2D> { enum { SD = 2, FD = 2, FC = 0, Z0 = P2_ZNCC, NZ = 1, STRAIN = P2_STRAIN, U = P2_DEF + D2_U, V = P2_DEF + D2_V, W = V }; };
template <> struct SL<PoiKind::POI3D> { enum { SD = 3, FD = 3, FC = 0, Z0 = P3_ZNCC, NZ = 1, STRAIN = P3_STRAIN, U = P3_DEF + 0, V = P3_DEF + 4, W = P3_DEF + 8 }; };
template <> struct SL<PoiKind::POI2DS> { enum { SD = 2, FD = 3, FC = P2DS_REF, Z0 = P2DS_ZNCC, NZ = 3, STRAIN = P2DS_STRAIN, U = P2DS_U, V = U + 1, W = U + 2 }; };

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

// only these POIs are binned, searched and fitted
template <PoiKind K>
__device__ __forceinline__ bool finite_position(const float* p) {
	bool fin = true;
#pragma unroll
	for (int d = 0; d < SL<K>::SD; d++) fin = fin && isfinite(p[d]);
	return fin;
}

// bbox[0..2] = min (ordered encoding), bbox[3..5] = max, bbox[6] += the POIs with a finite position.  SERIES: the records are
// frame 0 of n_frames frames of n records each, and bbox[7] += the POIs whose search coordinates differ, as bits, in some frame
// from frame 0's.
template <PoiKind K, bool SERIES>
__global__ void strain_bbox_kernel(const float* __restrict__ pois, int n, unsigned int* __restrict__ bbox, size_t n_frames) {
	constexpr int D = SL<K>::SD;
	unsigned int mn[3] = { 0xffffffffu, 0xffffffffu, 0xffffffffu }, mx[3] = { 0u, 0u, 0u }, finite = 0, moved = 0;
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float* p = pois + (size_t)i * poi_floats(K);
		if (SERIES) {
			for (size_t f = 1; f < n_frames; f++) {
				const float* pf = p + f * (size_t)n * poi_floats(K);
				bool same = true;
#pragma unroll
				for (int d = 0; d < D; d++) same = same && __float_as_uint(pf[d]) == __float_as_uint(p[d]);
				if (!same) { moved++; break; }
			}
		}
		if (!finite_position<K>(p)) continue;
		finite++;
#pragma unroll
		for (int d = 0; d < D; d++) {
			const unsigned int o = float_to_ordered(p[d]);
			mn[d] = min(mn[d], o);
			mx[d] = max(mx[d], o);
		}
	}
	// one atomic per warp and field; the count is per lane because the grid-stride loop ends at different trips per lane
	finite = __reduce_add_sync(0xffffffffu, finite);
	if ((threadIdx.x & 31) == 0) atomicAdd(bbox + 6, finite);
	if (SERIES) {
		moved = __reduce_add_sync(0xffffffffu, moved);
		if ((threadIdx.x & 31) == 0 && moved) atomicAdd(bbox + 7, moved);
	}
#pragma unroll
	for (int d = 0; d < D; d++) {
		mn[d] = __reduce_min_sync(0xffffffffu, mn[d]);
		mx[d] = __reduce_max_sync(0xffffffffu, mx[d]);
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

template <PoiKind K>
__global__ void strain_keys_kernel(const float* __restrict__ pois, int n, StrainGrid g, unsigned int* __restrict__ keys, int* __restrict__ vals) {
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float* p = pois + (size_t)i * poi_floats(K);
		unsigned int key = g.n_cells;
		if (finite_position<K>(p)) {
			int c[3];
			strain_cell<SL<K>::SD>(g, p, c);
			key = (unsigned int)((c[2] * g.nc[1] + c[1]) * g.nc[0] + c[0]);
		}
		keys[i] = key;
		vals[i] = i;
	}
}

// sorted, compact copies: pos = {x, y, z|0, fit flag (every ZNCC >= threshold)}, disp = {u, v, w|0, 0},
// fpos = the fit coordinates when they are not the search coordinates (POI2DS: ref_coor)
template <PoiKind K>
__global__ void strain_gather_kernel(const float* __restrict__ pois, int n, const int* __restrict__ order, float zncc_threshold,
	float4* __restrict__ pos, float4* __restrict__ disp, float4* __restrict__ fpos) {
	typedef SL<K> L;
	for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
		const float* p = pois + (size_t)order[s] * poi_floats(K);
		bool good = true;
#pragma unroll
		for (int k = 0; k < L::NZ; k++) good = good && (p[L::Z0 + k] >= zncc_threshold);
		pos[s] = make_float4(p[0], p[1], L::SD == 3 ? p[2] : 0.f, good ? 1.f : 0.f);
		disp[s] = make_float4(p[L::U], p[L::V], L::FD == 3 ? p[L::W] : 0.f, 0.f);
		if (L::FC != 0) fpos[s] = make_float4(p[L::FC], p[L::FC + 1], p[L::FC + 2], 0.f);
	}
}

// The series' sorted, compact copies of the n_valid POIs with a finite position, over n_frames frames of n records:
// pos[n_valid] = frame 0's {x, y, z|0, 0} (every frame's, as the bbox pass checked), and frame-major [n_frames][n_valid]
// disp = {u, v, w|0, fit flag} and fpos (POI2DS: ref_coor) of each frame
template <PoiKind K>
__global__ void strain_series_gather_kernel(const float* __restrict__ pois, int n, size_t n_frames, int n_valid, const int* __restrict__ order,
	float zncc_threshold, float4* __restrict__ pos, float4* __restrict__ disp, float4* __restrict__ fpos) {
	typedef SL<K> L;
	const size_t total = n_frames * (size_t)n_valid;
	for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
		const size_t f = t / (size_t)n_valid;
		const int s = (int)(t - f * (size_t)n_valid);
		const float* p = pois + (f * (size_t)n + (size_t)order[s]) * poi_floats(K);
		bool good = true;
#pragma unroll
		for (int k = 0; k < L::NZ; k++) good = good && (p[L::Z0 + k] >= zncc_threshold);
		if (f == 0) pos[s] = make_float4(p[0], p[1], L::SD == 3 ? p[2] : 0.f, 0.f);
		disp[t] = make_float4(p[L::U], p[L::V], L::FD == 3 ? p[L::W] : 0.f, good ? 1.f : 0.f);
		if (L::FC != 0) fpos[t] = make_float4(p[L::FC], p[L::FC + 1], p[L::FC + 2], 0.f);
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

// the runs of x-adjacent cells that can hold the neighbours of a POI at `centre`, one per (y, z) row of the 3x3(x3) cell block
// around its cell: lane `row` gets the sorted range [run_lo, run_hi) of row `row`
template <int D>
__device__ __forceinline__ void neighbour_runs(const StrainGrid& g, const float4& centre, const unsigned int* __restrict__ keys, int n_valid, int lane,
	int& run_lo, int& run_hi) {
	int c[3];
	const float pc[3] = { centre.x, centre.y, centre.z };
	strain_cell<D>(g, pc, c);
	run_lo = run_hi = 0;
	if (lane < (D == 2 ? 3 : 9)) {
		const int cy = c[1] + (lane % 3) - 1, cz = D == 3 ? c[2] + (lane / 3) - 1 : 0;
		if (cy >= 0 && cy < g.nc[1] && cz >= 0 && cz < g.nc[2]) {
			const int cx0 = max(c[0] - 1, 0), cx1 = min(c[0] + 1, g.nc[0] - 1);
			const unsigned int base = (unsigned int)((cz * g.nc[1] + cy) * g.nc[0]);
			run_lo = lower_bound_u32(keys, n_valid, base + cx0);
			run_hi = lower_bound_u32(keys, n_valid, base + cx1 + 1);
		}
	}
}

// The POIs in the runs within the radius (squared distance strictly below r2): each lane adds those of its share whose every
// ZNCC passed (pos.w) to sums.  Returns how many are within the radius (warp total).
template <PoiKind K>
__device__ __forceinline__ int radius_scan(FitSums<SL<K>::FD>& sums, const float4& centre, const float4& fcentre, int run_lo, int run_hi, float r2,
	const float4* __restrict__ pos, const float4* __restrict__ disp, const float4* __restrict__ fpos, int lane) {
	int found = 0;
#pragma unroll 1
	for (int row = 0; row < (SL<K>::SD == 2 ? 3 : 9); row++) {
		const int lo = __shfl_sync(0xffffffffu, run_lo, row), hi = __shfl_sync(0xffffffffu, run_hi, row);
		for (int j = lo + lane; j < hi; j += 32) {
			const float4 q = __ldg(pos + j);
			if (dist2<SL<K>::SD>(centre, q) < r2) {
				found++;
				if (q.w != 0.f) sums.add(fcentre, SL<K>::FC != 0 ? __ldg(fpos + j) : q, __ldg(disp + j));
			}
		}
	}
	return __reduce_add_sync(0xffffffffu, found);
}

// k-nearest fallback (src/oc_strain.cpp:183-196): sums restart from the k_min nearest POIs, found by k selection passes over all
// POIs ordered by (distance^2, original index); lane 0 adds those whose every ZNCC passed
template <PoiKind K>
__device__ __forceinline__ void knn_fallback(FitSums<SL<K>::FD>& sums, const float4& centre, const float4& fcentre, int k_min, int n_valid,
	const int* __restrict__ order, const float4* __restrict__ pos, const float4* __restrict__ disp, const float4* __restrict__ fpos, int lane) {
	sums.clear();
	float prev_d = -1.f;
	int prev_i = -1;
	const int k = k_min < n_valid ? k_min : n_valid;
#pragma unroll 1
	for (int pass = 0; pass < k; pass++) {
		float bd = INFINITY;
		int bi = 0x7fffffff, bs = -1;
		for (int j = lane; j < n_valid; j += 32) {
			const float d = dist2<SL<K>::SD>(centre, __ldg(pos + j));
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
			if (q.w != 0.f) sums.add(fcentre, SL<K>::FC != 0 ? __ldg(fpos + bs) : q, __ldg(disp + bs));
		}
	}
}

// The series kernel's forms of radius_scan and knn_fallback: the same search, lane for lane and pass for pass, with what is done
// with each neighbour left to the caller.  (The pair kernel keeps its own two so that its code stays as it is.)
//
// radius_scan's search: each lane calls visit(j, pos[j]) for the POIs of its share within the radius, in the order it meets
// them.  Returns how many are within the radius (warp total).
template <int D, class Visit>
__device__ __forceinline__ int radius_visit(const float4& centre, int run_lo, int run_hi, float r2, const float4* __restrict__ pos, int lane,
	Visit visit) {
	int found = 0;
#pragma unroll 1
	for (int row = 0; row < (D == 2 ? 3 : 9); row++) {
		const int lo = __shfl_sync(0xffffffffu, run_lo, row), hi = __shfl_sync(0xffffffffu, run_hi, row);
		for (int j = lo + lane; j < hi; j += 32) {
			const float4 q = __ldg(pos + j);
			if (dist2<D>(centre, q) < r2) {
				found++;
				visit(j, q);
			}
		}
	}
	return __reduce_add_sync(0xffffffffu, found);
}

// knn_fallback's search: the whole warp calls visit(j) with the sorted index j of each of the k_min nearest POIs, nearest first.
template <int D, class Visit>
__device__ __forceinline__ void knn_visit(const float4& centre, int k_min, int n_valid, const int* __restrict__ order, const float4* __restrict__ pos,
	int lane, Visit visit) {
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
		visit(bs);
	}
}

// Lane 0, with the warp's sums: the plane fit, then the strains of POI `poi` from the displacement gradients
// g_ki = G[k][i] = d u_k / d x_i (u, v, w over x, y, z): e_xx e_yy e_xy (FD = 2) or e_xx e_yy e_zz e_xy e_yz e_zx (FD = 3).
// Green (approximation 2, src/oc_strain.cpp:229-235, :455-463): e_ii = g_ii + 1/2 sum_k g_ki^2, e_ij = 1/2 (g_ij + g_ji +
// sum_k g_ki g_kj); Cauchy (1, :222-227, :444-453) drops the sums; any other approximation writes nothing.  The sums run over
// k = u, v, w, in the reference's operand order.
template <PoiKind K>
__device__ __forceinline__ void fit_and_write(const FitSums<SL<K>::FD>& sums, float* __restrict__ pois, int poi, int approximation) {
	constexpr int FD = SL<K>::FD;
	if (approximation != 1 && approximation != 2) return;
	double x[FD][FD + 1];
	solve_normal<FD>(sums, x);
	float G[FD][FD];
#pragma unroll
	for (int k = 0; k < FD; k++)
#pragma unroll
		for (int i = 0; i < FD; i++) G[k][i] = (float)x[k][1 + i];
	float* e = pois + (size_t)poi * poi_floats(K) + SL<K>::STRAIN;
	const bool green = approximation == 2;
#pragma unroll
	for (int i = 0; i < FD; i++) {
		float s = G[0][i] * G[0][i];
#pragma unroll
		for (int k = 1; k < FD; k++) s += G[k][i] * G[k][i];
		e[i] = green ? G[i][i] + 0.5f * s : G[i][i];
	}
#pragma unroll
	for (int p = 0; p < (FD == 2 ? 1 : 3); p++) { // (i, j) = (x, y), (y, z), (z, x)
		const int i = p, j = (p + 1) % 3;
		float s = G[i][j] + G[j][i];
#pragma unroll
		for (int k = 0; k < FD; k++) s = green ? s + G[k][j] * G[k][i] : s;
		e[FD + p] = 0.5f * s;
	}
}

// one warp per sorted POI s < n_valid (the POIs with a finite position)
template <PoiKind K>
__global__ void __launch_bounds__(256) strain_kernel(float* __restrict__ pois, int n_valid, StrainGrid g, const unsigned int* __restrict__ keys,
	const int* __restrict__ order, const float4* __restrict__ pos, const float4* __restrict__ disp, const float4* __restrict__ fpos, float radius,
	int k_min, int approximation, int only) {
	const int lane = threadIdx.x & 31;
	const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int n_warps = (gridDim.x * blockDim.x) >> 5;
	const float r2 = __fmul_rn(radius, radius);
	for (int s = warp_global; s < n_valid; s += n_warps) {
		const float4 centre = __ldg(pos + s);
		if (only >= 0) { // Strain::compute(POI*, queue): that POI only, whatever its own ZNCC
			if (__ldg(order + s) != only) continue;
		} else if (centre.w == 0.f) continue; // Strain::compute(queue): POIs below the ZNCC threshold are skipped (:244-248)
		int run_lo, run_hi;
		neighbour_runs<SL<K>::SD>(g, centre, keys, n_valid, lane, run_lo, run_hi);
		const float4 fcentre = SL<K>::FC != 0 ? __ldg(fpos + s) : centre; // origin of the fit coordinates
		FitSums<SL<K>::FD> sums;
		sums.clear();
		if (radius_scan<K>(sums, centre, fcentre, run_lo, run_hi, r2, pos, disp, fpos, lane) < k_min)
			knn_fallback<K>(sums, centre, fcentre, k_min, n_valid, order, pos, disp, fpos, lane);
		sums.reduce();
		if (lane == 0 && sums.a[0] >= (double)k_min) fit_and_write<K>(sums, pois, __ldg(order + s), approximation); // enough good neighbours (:200-201)
	}
}

// The indices a lane keeps of its radius-search neighbours (a warp: 32 x this), and the most k-nearest neighbours a warp keeps
constexpr int STRAIN_LIST = 32;
constexpr int STRAIN_SERIES_THREADS = 256;

// Strain over n_frames frames of n records that share their positions: one warp per sorted POI s < n_valid.  The neighbour search
// runs once: each lane keeps the sorted indices its share of radius_visit met within the radius, in the order it met them (or lane
// 0, the k-nearest visit's selection order).  Then per frame in which the POI's own ZNCC passes, the lanes replay their lists
// against that frame's disp (fit flag in .w) and fpos, so that each lane adds the same neighbours in the same order as the pair
// kernel does and the warp reduction is the same: every frame's records are bit for bit those of strain_kernel on that frame.
// A POI whose lists outgrow STRAIN_LIST per lane (or STRAIN_LIST x 32 nearest) searches again in every frame instead.
template <PoiKind K>
__global__ void __launch_bounds__(STRAIN_SERIES_THREADS) strain_series_kernel(float* __restrict__ pois, size_t n, size_t n_frames, int n_valid, StrainGrid g,
	const unsigned int* __restrict__ keys, const int* __restrict__ order, const float4* __restrict__ pos, const float4* __restrict__ disp,
	const float4* __restrict__ fpos, float radius, int k_min, int approximation) {
	typedef SL<K> L;
	__shared__ int lists[STRAIN_SERIES_THREADS / 32][STRAIN_LIST * 32];
	int* const list = lists[threadIdx.x >> 5];
	const int lane = threadIdx.x & 31;
	const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int n_warps = (gridDim.x * blockDim.x) >> 5;
	const float r2 = __fmul_rn(radius, radius);
	for (int s = warp_global; s < n_valid; s += n_warps) {
		bool fitted = false; // the POI's own ZNCC passes in some frame
		for (size_t f = lane; f < n_frames; f += 32) fitted = fitted || __ldg(disp + f * n_valid + s).w != 0.f;
		if (!__any_sync(0xffffffffu, fitted)) continue;
		const float4 centre = __ldg(pos + s);
		int run_lo, run_hi;
		neighbour_runs<L::SD>(g, centre, keys, n_valid, lane, run_lo, run_hi);
		int kept = 0; // radius: this lane's list length; k-nearest: the warp's
		const bool knn = radius_visit<L::SD>(centre, run_lo, run_hi, r2, pos, lane, [&](int j, const float4&) {
			if (kept < STRAIN_LIST) list[kept * 32 + lane] = j;
			kept++;
		}) < k_min;
		bool again; // search again in every frame
		if (knn) {
			kept = 0;
			again = (k_min < n_valid ? k_min : n_valid) > STRAIN_LIST * 32;
			if (!again) knn_visit<L::SD>(centre, k_min, n_valid, order, pos, lane, [&](int j) {
				if (lane == 0) list[kept] = j;
				kept++;
			});
		} else {
			again = __any_sync(0xffffffffu, kept > STRAIN_LIST);
		}
		__syncwarp();
		const int poi = __ldg(order + s);
		for (size_t f = 0; f < n_frames; f++) {
			const float4* const fdisp = disp + f * n_valid;
			const float4* const ffpos = fpos + f * n_valid;
			if (__ldg(fdisp + s).w == 0.f) continue; // below the threshold in this frame
			const float4 fcentre = L::FC != 0 ? __ldg(ffpos + s) : centre;
			FitSums<L::FD> sums;
			sums.clear();
			const auto add = [&](int j) {
				const float4 dq = __ldg(fdisp + j);
				if (dq.w != 0.f) sums.add(fcentre, L::FC != 0 ? __ldg(ffpos + j) : __ldg(pos + j), dq);
			};
			if (again && knn) {
				knn_visit<L::SD>(centre, k_min, n_valid, order, pos, lane, [&](int j) { if (lane == 0) add(j); });
			} else if (again) {
				radius_visit<L::SD>(centre, run_lo, run_hi, r2, pos, lane, [&](int j, const float4&) { add(j); });
			} else if (knn) {
				if (lane == 0)
					for (int t = 0; t < kept; t++) add(list[t]);
			} else {
				for (int t = 0; t < kept; t++) add(list[t * 32 + lane]);
			}
			sums.reduce();
			if (lane == 0 && sums.a[0] >= (double)k_min) fit_and_write<K>(sums, pois + f * n * poi_floats(K), poi, approximation);
		}
		__syncwarp(); // the lists are rewritten by the next POI
	}
}

// Device workspace of a call over n_frames frames of n POIs (one grow-only allocation owned by the context), regions 256-byte
// aligned: bbox[8] | keys_in[n] | keys_out[n] | vals_in[n] | vals_out[n] | pos[n] | disp[n_frames n] | fpos[n_frames n] | cub temp.
// base null: sizes only.
struct StrainWs {
	unsigned int *bbox, *keys_in, *keys_out;
	int *vals_in, *vals_out;
	float4 *pos, *disp, *fpos;
	void* cub_temp;
	size_t cub_bytes = 0, bytes = 0;
	StrainWs(void* base, size_t n, size_t n_frames) {
		cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned int*)nullptr, (unsigned int*)nullptr, (const int*)nullptr, (int*)nullptr,
			(int)n);
		auto take = [&](size_t b) { const uintptr_t p = (uintptr_t)base + bytes; bytes += (b + 255) & ~(size_t)255; return (void*)p; };
		bbox = (unsigned int*)take(8 * sizeof(unsigned int));
		keys_in = (unsigned int*)take(n * 4);
		keys_out = (unsigned int*)take(n * 4);
		vals_in = (int*)take(n * 4);
		vals_out = (int*)take(n * 4);
		pos = (float4*)take(n * 16);
		disp = (float4*)take(n_frames * n * 16);
		fpos = (float4*)take(n_frames * n * 16);
		cub_temp = take(cub_bytes);
	}
};

// bbox and finite count (the call's one readback), keys, sort, gather, strain.  moved null: the pair call over n records
// (`only`: Strain::compute(POI*, queue)); else the series over n_frames frames of n records, which sets *moved instead of
// writing anything when the positions of some frame are not frame 0's.
template <PoiKind K>
cudaError_t strain_run(float* d_pois, size_t n, size_t n_frames, float radius, int k_min, float zncc_threshold, int approximation, long long only,
	const StrainWs& w, int sm_count, cudaStream_t stream, long long* launches, bool* moved) {
	const int threads = 256;
	int blocks = (int)((n + threads - 1) / threads);
	if (blocks > sm_count * 8) blocks = sm_count * 8;
	if (blocks < 1) blocks = 1;
	cudaError_t e;
	unsigned int hb[8] = { 0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u, 0u };
	if ((e = cudaMemcpyAsync(w.bbox, hb, sizeof(hb), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
	if (n_frames > 1) strain_bbox_kernel<K, true><<<blocks, threads, 0, stream>>>(d_pois, (int)n, w.bbox, n_frames);
	else strain_bbox_kernel<K, false><<<blocks, threads, 0, stream>>>(d_pois, (int)n, w.bbox, n_frames);
	if ((e = launched(launches)) != cudaSuccess || (e = cudaMemcpyAsync(hb, w.bbox, sizeof(hb), cudaMemcpyDeviceToHost, stream)) != cudaSuccess
		|| (e = cudaStreamSynchronize(stream)) != cudaSuccess)
		return e;
	if (hb[7]) {
		*moved = true;
		return cudaSuccess;
	}
	// exactly the POIs with a finite position get keys below the sentinel, so they lead the sorted order
	const int n_valid = (int)hb[6];
	if (n_valid == 0) return cudaSuccess;
	float lo[3], hi[3];
	for (int d = 0; d < SL<K>::SD; d++) { lo[d] = ordered_to_float(hb[d]); hi[d] = ordered_to_float(hb[3 + d]); }
	StrainGrid g;
	strain_grid_plan(SL<K>::SD, lo, hi, radius, &g);
	strain_keys_kernel<K><<<blocks, threads, 0, stream>>>(d_pois, (int)n, g, w.keys_in, w.vals_in);
	if ((e = launched(launches)) != cudaSuccess) return e;
	const int end_bit = 32 - __builtin_clz(g.n_cells); // the keys' bit length (1 <= n_cells < 2^30)
	size_t cub_bytes = w.cub_bytes;
	if ((e = cub::DeviceRadixSort::SortPairs(w.cub_temp, cub_bytes, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)n, 0, end_bit, stream)) != cudaSuccess)
		return e;
	++*launches;
	long long grid = ((long long)n_valid * 32 + threads - 1) / threads;
	if (grid > (long long)sm_count * 8) grid = (long long)sm_count * 8;
	if (!moved) {
		strain_gather_kernel<K><<<blocks, threads, 0, stream>>>(d_pois, (int)n, w.vals_out, zncc_threshold, w.pos, w.disp, w.fpos);
		if ((e = launched(launches)) != cudaSuccess) return e;
		strain_kernel<K><<<(int)grid, threads, 0, stream>>>(d_pois, n_valid, g, w.keys_out, w.vals_out, w.pos, w.disp, w.fpos, radius, k_min, approximation,
			(int)only);
		return launched(launches);
	}
	long long gather_blocks = (long long)((n_frames * (size_t)n_valid + threads - 1) / threads);
	if (gather_blocks > (long long)sm_count * 8) gather_blocks = (long long)sm_count * 8;
	strain_series_gather_kernel<K><<<(int)gather_blocks, threads, 0, stream>>>(d_pois, (int)n, n_frames, n_valid, w.vals_out, zncc_threshold, w.pos,
		w.disp, w.fpos);
	if ((e = launched(launches)) != cudaSuccess) return e;
	strain_series_kernel<K><<<(int)grid, STRAIN_SERIES_THREADS, 0, stream>>>(d_pois, n, n_frames, n_valid, g, w.keys_out, w.vals_out, w.pos,
		w.disp, w.fpos, radius, k_min, approximation);
	return launched(launches);
}

// RegionFit2D::compute(POI2D*) / RegionFit3D::compute(POI3D*) (src/oc_region_fit.cpp:91-170, :268-355), one warp per queue POI
// i < n with a finite position (any other is left alone).  Its neighbours are the reliable POIs -- sorted and gathered into pos /
// disp, n_valid of them -- within the radius, or the k_min nearest when fewer are found, every one of them whatever its ZNCC (the
// fit flag pos.w is not read).  With at least k_min neighbours, lane 0 writes the plane fit's intercept and slopes to the
// first-order deformation (u, ux, uy(, uz), v, ...) and sets zncc to 0; every other field stays as it was.
template <PoiKind K>
__global__ void __launch_bounds__(256) region_fit_kernel(float* __restrict__ queue, int n, int n_valid, StrainGrid g, const unsigned int* __restrict__ keys,
	const int* __restrict__ order, const float4* __restrict__ pos, const float4* __restrict__ disp, float radius, int k_min) {
	typedef SL<K> L;
	constexpr int D = L::SD;
	const int lane = threadIdx.x & 31;
	const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int n_warps = (gridDim.x * blockDim.x) >> 5;
	const float r2 = __fmul_rn(radius, radius);
	for (int i = warp_global; i < n; i += n_warps) {
		float* const p = queue + (size_t)i * poi_floats(K);
		if (!finite_position<K>(p)) continue;
		const float4 centre = make_float4(p[0], p[1], D == 3 ? p[2] : 0.f, 0.f);
		int run_lo, run_hi;
		neighbour_runs<D>(g, centre, keys, n_valid, lane, run_lo, run_hi);
		FitSums<D> sums;
		sums.clear();
		if (radius_visit<D>(centre, run_lo, run_hi, r2, pos, lane, [&](int j, const float4& q) { sums.add(centre, q, __ldg(disp + j)); }) < k_min) {
			sums.clear(); // oc_region_fit.cpp:116-126: the k nearest replace the radius set
			knn_visit<D>(centre, k_min, n_valid, order, pos, lane, [&](int j) {
				if (lane == 0) sums.add(centre, __ldg(pos + j), __ldg(disp + j));
			});
		}
		sums.reduce();
		if (lane == 0 && sums.a[0] >= (double)k_min) {
			double x[D][D + 1];
			solve_normal<D>(sums, x);
			const int field[3] = { L::U, L::V, L::W };
#pragma unroll
			for (int k = 0; k < D; k++)
#pragma unroll
				for (int c = 0; c <= D; c++) p[field[k] + c] = (float)x[k][c];
			p[L::Z0] = 0.f;
		}
	}
}

// bbox of the reliable set and its finite count (the call's one readback), keys, sort, gather, fit: always these five launches
template <PoiKind K>
cudaError_t region_fit_run(const float* d_reliable, size_t n_reliable, float* d_queue, size_t n, float radius, int k_min, const StrainWs& w,
	int sm_count, cudaStream_t stream, long long* launches) {
	const int threads = 256;
	int blocks = (int)((n_reliable + threads - 1) / threads);
	if (blocks > sm_count * 8) blocks = sm_count * 8;
	if (blocks < 1) blocks = 1;
	cudaError_t e;
	unsigned int hb[8] = { 0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u, 0u };
	if ((e = cudaMemcpyAsync(w.bbox, hb, sizeof(hb), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
	strain_bbox_kernel<K, false><<<blocks, threads, 0, stream>>>(d_reliable, (int)n_reliable, w.bbox, 1);
	if ((e = launched(launches)) != cudaSuccess || (e = cudaMemcpyAsync(hb, w.bbox, sizeof(hb), cudaMemcpyDeviceToHost, stream)) != cudaSuccess
		|| (e = cudaStreamSynchronize(stream)) != cudaSuccess)
		return e;
	// no reliable POI with a finite position: an empty grid, so that every query finds no neighbour (and, with k_min <= 0,
	// is fitted over none, as the reference's arithmetic does)
	const int n_valid = (int)hb[6];
	float lo[3] = { 0.f, 0.f, 0.f }, hi[3] = { 0.f, 0.f, 0.f };
	for (int d = 0; d < SL<K>::SD && n_valid; d++) { lo[d] = ordered_to_float(hb[d]); hi[d] = ordered_to_float(hb[3 + d]); }
	StrainGrid g;
	strain_grid_plan(SL<K>::SD, lo, hi, radius, &g);
	strain_keys_kernel<K><<<blocks, threads, 0, stream>>>(d_reliable, (int)n_reliable, g, w.keys_in, w.vals_in);
	if ((e = launched(launches)) != cudaSuccess) return e;
	const int end_bit = 32 - __builtin_clz(g.n_cells);
	size_t cub_bytes = w.cub_bytes;
	if ((e = cub::DeviceRadixSort::SortPairs(w.cub_temp, cub_bytes, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)n_reliable, 0, end_bit,
		stream)) != cudaSuccess)
		return e;
	++*launches;
	strain_gather_kernel<K><<<blocks, threads, 0, stream>>>(d_reliable, (int)n_reliable, w.vals_out, -INFINITY, w.pos, w.disp, w.fpos);
	if ((e = launched(launches)) != cudaSuccess) return e;
	long long grid = ((long long)n * 32 + threads - 1) / threads;
	if (grid > (long long)sm_count * 8) grid = (long long)sm_count * 8;
	region_fit_kernel<K><<<(int)grid, threads, 0, stream>>>(d_queue, (int)n, n_valid, g, w.keys_out, w.vals_out, w.pos, w.disp, radius, k_min);
	return launched(launches);
}

} // namespace

size_t strain_workspace_bytes(size_t n, size_t n_frames) { return StrainWs(nullptr, n, n_frames).bytes; }

cudaError_t region_fit_launch(PoiKind kind, const float* d_reliable, size_t n_reliable, float* d_queue, size_t n, float radius, int k_min,
	void* workspace, int sm_count, cudaStream_t stream, long long* launches) {
	const StrainWs w(workspace, n_reliable, 1);
	if (kind == PoiKind::POI3D) return region_fit_run<PoiKind::POI3D>(d_reliable, n_reliable, d_queue, n, radius, k_min, w, sm_count, stream, launches);
	return region_fit_run<PoiKind::POI2D>(d_reliable, n_reliable, d_queue, n, radius, k_min, w, sm_count, stream, launches);
}

cudaError_t strain_launch(PoiKind kind, float* d_pois, size_t n, float radius, int k_min, float zncc_threshold, int approximation, long long only,
	void* workspace, int sm_count, cudaStream_t stream, long long* launches) {
	const StrainWs w(workspace, n, 1);
	switch (kind) {
	case PoiKind::POI2D: return strain_run<PoiKind::POI2D>(d_pois, n, 1, radius, k_min, zncc_threshold, approximation, only, w, sm_count, stream, launches, nullptr);
	case PoiKind::POI3D: return strain_run<PoiKind::POI3D>(d_pois, n, 1, radius, k_min, zncc_threshold, approximation, only, w, sm_count, stream, launches, nullptr);
	default: return strain_run<PoiKind::POI2DS>(d_pois, n, 1, radius, k_min, zncc_threshold, approximation, only, w, sm_count, stream, launches, nullptr);
	}
}

cudaError_t strain_series_launch(PoiKind kind, float* d_pois, size_t n_frames, size_t n, float radius, int k_min, float zncc_threshold,
	int approximation, void* workspace, int sm_count, cudaStream_t stream, long long* launches, bool* moved) {
	const StrainWs w(workspace, n, n_frames);
	*moved = false;
	switch (kind) {
	case PoiKind::POI2D:
		return strain_run<PoiKind::POI2D>(d_pois, n, n_frames, radius, k_min, zncc_threshold, approximation, -1, w, sm_count, stream, launches, moved);
	case PoiKind::POI3D:
		return strain_run<PoiKind::POI3D>(d_pois, n, n_frames, radius, k_min, zncc_threshold, approximation, -1, w, sm_count, stream, launches, moved);
	default:
		return strain_run<PoiKind::POI2DS>(d_pois, n, n_frames, radius, k_min, zncc_threshold, approximation, -1, w, sm_count, stream, launches, moved);
	}
}

} // namespace ocb
