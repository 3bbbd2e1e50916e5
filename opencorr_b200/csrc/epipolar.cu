// epipolar.cu -- the candidate sweep of EpipolarSearch as ONE batch (SURVEY.md section 8(f) N4), for sm_90a.
//
// Replaces EpipolarSearch::compute(POI2D*) (reference src/oc_epipolar_search.cpp:133-195), which for every POI of
// the primary view spawns ~2*radius/step candidate POIs along its epipolar line in the secondary view, runs
// ICGN2D1::compute(POI2D*) on each (an `omp parallel for` over the candidates of ONE POI, :184-188) and keeps the
// candidate with the highest ZNCC; compute(queue) walks the POIs serially (:197-205).
// Here the candidates of a whole block of POIs are written as one POI2D queue (fixed number of slots per POI),
// registered by the ordinary ICGN2D1 kernel in one launch, and reduced per POI by a warp.
#include "ocb_kernels.h"

namespace ocb {

// slots per POI: the centre + both directions for i = step, 2*step, ... < radius  (:151-182)
int epipolar_slots(int search_radius, int search_step) {
	int m = 0;
	for (int i = search_step; i < search_radius; i += search_step) m++;
	return 1 + 2 * m;
}

struct EpiParams {
	float f[9];          // fundamental matrix, row-major
	float par_x[3], par_y[3];
	int search_radius, search_step, rx, ry, w, h, slots;
};

// One thread per (POI, slot).  Slot 0 is the centre of the search region (no border test, :151-155); slots 2k-1 / 2k
// are x_view2 +/- k*step.  A slot that fails the border test (:164-168, :175-179) is not a candidate in the
// reference: its record gets ZNCC = -inf here, which the IC-GN guard leaves alone (src/oc_icgn.cpp:160-167 keeps a
// negative incoming ZNCC) and which can never win the selection.
__global__ void epipolar_candidates_kernel(const float* __restrict__ pois, int poi0, int n_poi, EpiParams p, float* __restrict__ cand) {
	const long long total = (long long)n_poi * p.slots;
	for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
		const int i = (int)(t / p.slots), slot = (int)(t - (long long)i * p.slots);
		const float* P = pois + (size_t)(poi0 + i) * P2_N;
		const float px = P[P2_X], py = P[P2_Y], pu = P[P2_DEF + D2_U], pv = P[P2_DEF + D2_V];
		// every operation rounded once, in the reference's order (:136-148)
		const float cxh = (float)(p.w / 2), cyh = (float)(p.h / 2);
		const float dxc = __fsub_rn(px, cxh), dyc = __fsub_rn(py, cyh);
		const float par_x = __fadd_rn(__fadd_rn(__fmul_rn(p.par_x[0], dxc), __fmul_rn(p.par_x[1], dyc)), p.par_x[2]);
		const float par_y = __fadd_rn(__fadd_rn(__fmul_rn(p.par_y[0], dxc), __fmul_rn(p.par_y[1], dyc)), p.par_y[2]);
		const float v0 = __fadd_rn(px, pu), v1 = __fadd_rn(py, pv);
		float e[3];
#pragma unroll
		for (int k = 0; k < 3; k++) e[k] = __fadd_rn(__fadd_rn(__fmul_rn(p.f[3 * k], v0), __fmul_rn(p.f[3 * k + 1], v1)), p.f[3 * k + 2]);
		const float slope = __fdiv_rn(-e[0], e[1]);
		const float intercept = __fdiv_rn(-e[2], e[1]);
		float num = __fmul_rn(slope, __fsub_rn(__fadd_rn(__fadd_rn(py, pv), par_y), intercept));
		num = __fadd_rn(__fadd_rn(__fadd_rn(num, px), pu), par_x);
		const int x_view2 = (int)__fdiv_rn(num, __fadd_rn(__fmul_rn(slope, slope), 1.f));
		int x_trial = x_view2;
		bool valid = true;
		if (slot > 0) {
			const int k = (slot + 1) >> 1;
			x_trial = (slot & 1) ? x_view2 + k * p.search_step : x_view2 - k * p.search_step;
		}
		const int y_trial = (int)__fadd_rn(__fmul_rn(slope, (float)x_trial), intercept);
		if (slot > 0)
			valid = x_trial - p.rx > 0 && x_trial + p.rx < p.w - 1 && y_trial - p.ry > 0 && y_trial + p.ry < p.h - 1;
		float* C = cand + (size_t)t * P2_N;
#pragma unroll
		for (int k = 0; k < P2_N; k++) C[k] = 0.f; // POI2D current_poi(poi->x, poi->y): everything else cleared (:152)
		C[P2_X] = px;
		C[P2_Y] = py;
		C[P2_DEF + D2_U] = __fsub_rn((float)x_trial, px);
		C[P2_DEF + D2_V] = __fsub_rn((float)y_trial, py);
		if (!valid) C[P2_ZNCC] = -INFINITY;
	}
}

// One warp per POI: first maximum of ZNCC over its slots (std::sort by ZNCC descending, :191; ties -- unspecified
// there -- go to the earlier candidate), then poi->deformation / poi->result are replaced (:193-194).
__global__ void epipolar_select_kernel(float* __restrict__ pois, int poi0, int n_poi, int slots, const float* __restrict__ cand) {
	const int lane = threadIdx.x & 31;
	const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
	for (int i = warp; i < n_poi; i += n_warps) {
		const float* C = cand + (size_t)i * slots * P2_N;
		float bz = -INFINITY;
		int bs = 0x7fffffff;
		for (int s = lane; s < slots; s += 32) {
			const float z = C[(size_t)s * P2_N + P2_ZNCC];
			if (z > bz || (z == bz && s < bs)) { bz = z; bs = s; }
		}
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			const float oz = __shfl_xor_sync(0xffffffffu, bz, o);
			const int os = __shfl_xor_sync(0xffffffffu, bs, o);
			if (oz > bz || (oz == bz && os < bs)) { bz = oz; bs = os; }
		}
		if (bs >= slots) bs = 0; // cannot happen: slot 0 always carries a finite ZNCC or a sentinel code
		const float* B = C + (size_t)bs * P2_N;
		float* P = pois + (size_t)(poi0 + i) * P2_N;
		if (lane < 12) P[P2_DEF + lane] = B[P2_DEF + lane];
		else if (lane < 18) P[P2_U0 + (lane - 12)] = B[P2_U0 + (lane - 12)]; // u0 v0 zncc iteration convergence feature
	}
}

cudaError_t epipolar_candidates_launch(const float* d_pois, size_t poi0, size_t n_poi, const float* fundamental, const float* parallax_x,
	const float* parallax_y, int search_radius, int search_step, int rx, int ry, int w, int h, int slots, float* d_cand, int sm_count,
	cudaStream_t stream) {
	EpiParams p;
	for (int k = 0; k < 9; k++) p.f[k] = fundamental[k];
	for (int k = 0; k < 3; k++) { p.par_x[k] = parallax_x[k]; p.par_y[k] = parallax_y[k]; }
	p.search_radius = search_radius; p.search_step = search_step; p.rx = rx; p.ry = ry; p.w = w; p.h = h; p.slots = slots;
	long long total = (long long)n_poi * slots;
	long long blocks = (total + 255) / 256;
	if (blocks > (long long)sm_count * 16) blocks = (long long)sm_count * 16;
	if (blocks < 1) blocks = 1;
	epipolar_candidates_kernel<<<(int)blocks, 256, 0, stream>>>(d_pois, (int)poi0, (int)n_poi, p, d_cand);
	return cudaGetLastError();
}

cudaError_t epipolar_select_launch(float* d_pois, size_t poi0, size_t n_poi, int slots, const float* d_cand, int sm_count, cudaStream_t stream) {
	long long blocks = ((long long)n_poi * 32 + 255) / 256;
	if (blocks > (long long)sm_count * 16) blocks = (long long)sm_count * 16;
	if (blocks < 1) blocks = 1;
	epipolar_select_kernel<<<(int)blocks, 256, 0, stream>>>(d_pois, (int)poi0, (int)n_poi, slots, d_cand);
	return cudaGetLastError();
}

} // namespace ocb
