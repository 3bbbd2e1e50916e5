// series_reseed.cu -- the small streaming kernels of the series calls that re-seed lost POIs (ocb_icgn2d_series_reseed,
// ocb_icgn3d_series_reseed).  The registration itself runs on the pair and series kernels; these kernels only find the lost
// POIs, gather them into a sub-queue, rebuild their records from the seeds and write the re-registered records back.
//
// Records are frame-major: out[f * n + i] is POI i's record of frame f.  POI i is lost in frame f when !(zncc >= zncc_min), so a
// NaN ZNCC and every failure code below zncc_min count as lost.
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "ocb_kernels.h"

namespace ocb {
namespace {

// Field layout of a POI2D (DIM 2) / POI3D (DIM 3) record: its length, the ZNCC, the translation components and the fields a
// rebuilt record takes from its seed (position and subset radii).
template <int DIM> struct RecLayout;
template <> struct RecLayout<2> {
	static constexpr int N = P2_N, ZNCC = P2_ZNCC;
	__device__ static int disp(int d) { return d == 0 ? P2_DEF + D2_U : P2_DEF + D2_V; }
	__device__ static int axis_of(int j) { return j == P2_DEF + D2_U ? 0 : (j == P2_DEF + D2_V ? 1 : -1); }
	__device__ static bool from_seed(int j) { return j == P2_X || j == P2_Y || j == P2_RX || j == P2_RY; }
};
template <> struct RecLayout<3> {
	static constexpr int N = P3_N, ZNCC = P3_ZNCC;
	__device__ static int disp(int d) { return P3_DEF + 4 * d; }
	__device__ static int axis_of(int j) { return (j == P3_DEF || j == P3_DEF + 4 || j == P3_DEF + 8) ? (j - P3_DEF) / 4 : -1; }
	__device__ static bool from_seed(int j) { return j == P3_X || j == P3_Y || j == P3_Z || j == P3_RX || j == P3_RY || j == P3_RZ; }
};

__device__ __forceinline__ bool is_lost(float zncc, float zncc_min) { return !(zncc >= zncc_min); }

// One thread per POI of the range (idx[k], or k itself when idx is null): first[i] = its first lost frame in [f_begin, f_end), or
// -1; hist[f] counts the POIs whose first lost frame is f.
template <int DIM>
__global__ void reseed_scan_kernel(const float* __restrict__ out, size_t n, int f_begin, int f_end, const int* __restrict__ idx, int m,
	float zncc_min, int* __restrict__ first, int* __restrict__ hist) {
	using L = RecLayout<DIM>;
	for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
		const int i = idx ? idx[k] : k;
		int lost = -1;
		for (int f = f_begin; f < f_end; f++)
			if (is_lost(out[((size_t)f * n + i) * L::N + L::ZNCC], zncc_min)) { lost = f; break; }
		first[i] = lost;
		if (lost >= 0) atomicAdd(hist + lost, 1);
	}
}

template <int DIM>
__global__ void reseed_anchor_init_kernel(const float* __restrict__ seeds, int n, float* __restrict__ anchor) {
	using L = RecLayout<DIM>;
	for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n * DIM; t += gridDim.x * blockDim.x)
		anchor[t] = seeds[(size_t)(t / DIM) * L::N + L::disp(t % DIM)];
}

// One thread per float of the sub-queue.  Record k is POI i = idx[k] (k when idx is null) rebuilt from its seed: position and
// subset radii copied, translation = the anchor, every other field 0.  With prev (POI i's final record of the frame before) good,
// the anchor becomes prev's translation first; each component's thread updates its own component.  anchor null: translation 0.
template <int DIM>
__global__ void reseed_rebuild_kernel(const float* __restrict__ seeds, const float* __restrict__ prev, const int* __restrict__ idx, int m,
	float zncc_min, float* __restrict__ anchor, float* __restrict__ sub) {
	using L = RecLayout<DIM>;
	const long long total = (long long)m * L::N;
	for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
		const int k = (int)(t / L::N), j = (int)(t % L::N);
		const int i = idx ? idx[k] : k;
		float v = 0.f;
		if (L::from_seed(j)) {
			v = seeds[(size_t)i * L::N + j];
		} else if (anchor) {
			const int d = L::axis_of(j);
			if (d >= 0) {
				if (prev && !is_lost(prev[(size_t)i * L::N + L::ZNCC], zncc_min)) {
					v = prev[(size_t)i * L::N + j];
					anchor[(size_t)i * DIM + d] = v;
				} else {
					v = anchor[(size_t)i * DIM + d];
				}
			}
		}
		sub[t] = v;
	}
}

// src holds `frames` frame-major blocks of m records; record k of block g goes to out[(f0 + g) * n + idx[k]].
template <int DIM>
__global__ void reseed_scatter_kernel(const float* __restrict__ src, int m, int frames, const int* __restrict__ idx, float* __restrict__ out,
	size_t n, int f0) {
	using L = RecLayout<DIM>;
	const long long per_frame = (long long)m * L::N, total = per_frame * frames;
	for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
		const int g = (int)(t / per_frame);
		const long long r = t - g * per_frame;
		const int k = (int)(r / L::N), j = (int)(r % L::N);
		out[(((size_t)(f0 + g)) * n + idx[k]) * L::N + j] = src[t];
	}
}

// the compaction's flag of a POI: its first lost frame is f
struct FirstLostIs {
	int f;
	__host__ __device__ char operator()(int first) const { return first == f; }
};

constexpr int RESEED_THREADS = 256;
inline int reseed_grid(long long work, int sm_count) {
	const long long b = (work + RESEED_THREADS - 1) / RESEED_THREADS, cap = (long long)sm_count * 8;
	return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

} // namespace

size_t reseed_select_bytes(size_t n) {
	size_t bytes = 0;
	cub::DeviceSelect::Flagged(nullptr, bytes, thrust::counting_iterator<int>(0), thrust::make_transform_iterator((const int*)nullptr, FirstLostIs{ 0 }),
		(int*)nullptr, (int*)nullptr, (int)n);
	return bytes;
}

cudaError_t reseed_scan_launch(int dim, const float* d_out, size_t n, int f_begin, int f_end, const int* d_idx, size_t m, float zncc_min, int* d_first,
	int* d_hist, int sm_count, cudaStream_t stream) {
	const int grid = reseed_grid((long long)m, sm_count);
	if (dim == 2) reseed_scan_kernel<2><<<grid, RESEED_THREADS, 0, stream>>>(d_out, n, f_begin, f_end, d_idx, (int)m, zncc_min, d_first, d_hist);
	else reseed_scan_kernel<3><<<grid, RESEED_THREADS, 0, stream>>>(d_out, n, f_begin, f_end, d_idx, (int)m, zncc_min, d_first, d_hist);
	return cudaGetLastError();
}

cudaError_t reseed_select_launch(const int* d_first, int f, size_t n, int* d_idx, int* d_count, void* d_temp, size_t temp_bytes, cudaStream_t stream) {
	size_t bytes = temp_bytes;
	return cub::DeviceSelect::Flagged(d_temp, bytes, thrust::counting_iterator<int>(0), thrust::make_transform_iterator(d_first, FirstLostIs{ f }), d_idx,
		d_count, (int)n, stream);
}

cudaError_t reseed_anchor_init_launch(int dim, const float* d_seeds, size_t n, float* d_anchor, int sm_count, cudaStream_t stream) {
	const int grid = reseed_grid((long long)n * dim, sm_count);
	if (dim == 2) reseed_anchor_init_kernel<2><<<grid, RESEED_THREADS, 0, stream>>>(d_seeds, (int)n, d_anchor);
	else reseed_anchor_init_kernel<3><<<grid, RESEED_THREADS, 0, stream>>>(d_seeds, (int)n, d_anchor);
	return cudaGetLastError();
}

cudaError_t reseed_rebuild_launch(int dim, const float* d_seeds, const float* d_prev, const int* d_idx, size_t m, float zncc_min, float* d_anchor,
	float* d_sub, int sm_count, cudaStream_t stream) {
	const int grid = reseed_grid((long long)m * (dim == 2 ? P2_N : P3_N), sm_count);
	if (dim == 2) reseed_rebuild_kernel<2><<<grid, RESEED_THREADS, 0, stream>>>(d_seeds, d_prev, d_idx, (int)m, zncc_min, d_anchor, d_sub);
	else reseed_rebuild_kernel<3><<<grid, RESEED_THREADS, 0, stream>>>(d_seeds, d_prev, d_idx, (int)m, zncc_min, d_anchor, d_sub);
	return cudaGetLastError();
}

cudaError_t reseed_scatter_launch(int dim, const float* d_src, size_t m, int frames, const int* d_idx, float* d_out, size_t n, int f0, int sm_count,
	cudaStream_t stream) {
	const int grid = reseed_grid((long long)m * frames * (dim == 2 ? P2_N : P3_N), sm_count);
	if (dim == 2) reseed_scatter_kernel<2><<<grid, RESEED_THREADS, 0, stream>>>(d_src, (int)m, frames, d_idx, d_out, n, f0);
	else reseed_scatter_kernel<3><<<grid, RESEED_THREADS, 0, stream>>>(d_src, (int)m, frames, d_idx, d_out, n, f0);
	return cudaGetLastError();
}

} // namespace ocb
