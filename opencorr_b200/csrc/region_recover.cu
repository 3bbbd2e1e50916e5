// region_recover.cu -- the round bookkeeping of the recovery calls (ocb_icgn2d_recover, ocb_icgn3d_recover): split a registered
// queue into its reliable and unreliable POIs, and after each round of RegionFit and IC-GN move the POIs that now pass into the
// reliable set.  The fit and the registration run on the RegionFit and pair IC-GN kernels; these only select and move records.
// The series recovery calls (ocb_icgn2d_series_recover, ocb_icgn3d_series_recover) add a scan for the frames that hold an
// unreliable record and the collection of each round's accepted queue indices.
//
// Every selection is a stable cub::DeviceSelect::Flagged over the positions 0 .. count-1, its flag read straight from the records
// (RecordTest), so the index lists come out in ascending order.  The comparisons are the literal float ones: a NaN ZNCC is neither
// below zncc_low nor at or above zncc_high, and a NaN convergence is neither above nor at or below conv.
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "ocb_kernels.h"

namespace ocb {
namespace {

// The flag of record i of `rec` (POI2D or POI3D, `floats` floats each) under one of the four tests of RecoverTest.
struct RecordTest {
	const float* rec;
	int floats, zncc, conv;
	RecoverTest test;
	float zncc_high, zncc_low, conv_max;
	__host__ __device__ char operator()(int i) const {
		const float z = rec[(size_t)i * floats + zncc], c = rec[(size_t)i * floats + conv];
		const bool unreliable = z < zncc_low || c > conv_max;
		switch (test) {
		case RecoverTest::UNRELIABLE: return unreliable;
		case RecoverTest::RELIABLE: return !unreliable && z >= zncc_high;
		case RecoverTest::ACCEPTED: return z >= zncc_high && c <= conv_max;
		default: return !(z >= zncc_high && c <= conv_max);
		}
	}
};
using FlagIter = thrust::transform_iterator<RecordTest, thrust::counting_iterator<int>>;

// One thread per float of `total` records: the first *count1 of them are the records src[list1[k]], the rest src[list2[k]].
// List 1's go to dst1 and, when q is set, also back to the queue at q[src_idx[list1[k]]]; list 2's go to dst2 with their queue
// indices (src_idx[p], or p itself when src_idx is null) in idx2.
template <int N>
__global__ void recover_move_kernel(const float* __restrict__ src, const int* __restrict__ src_idx, long long total, const int* __restrict__ list1,
	const int* __restrict__ count1, float* __restrict__ dst1, float* __restrict__ q, const int* __restrict__ list2, float* __restrict__ dst2,
	int* __restrict__ idx2) {
	const long long c1 = *count1;
	for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total * N; t += (long long)gridDim.x * blockDim.x) {
		const long long k = t / N;
		const int j = (int)(t - k * N);
		if (k < c1) {
			const int p = list1[k];
			const float v = src[(size_t)p * N + j];
			dst1[k * N + j] = v;
			if (q) q[(size_t)src_idx[p] * N + j] = v;
		} else {
			const long long k2 = k - c1;
			const int p = list2[k2];
			dst2[k2 * N + j] = src[(size_t)p * N + j];
			if (j == 0) idx2[k2] = src_idx ? src_idx[p] : p;
		}
	}
}

// One thread per position k of a round's working set: the queue index of its k-th accepted record, for k < *count1.
__global__ void recover_collect_kernel(const int* __restrict__ src_idx, int total, const int* __restrict__ list1, const int* __restrict__ count1,
	int* __restrict__ out) {
	const int c1 = *count1;
	for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < total && k < c1; k += gridDim.x * blockDim.x) out[k] = src_idx[list1[k]];
}

// One thread per POI of the range (idx[k], or k itself when idx is null) of a frame-major series of records (N floats each): first[i]
// = its first frame in [f_begin, f_end) whose record is UNRELIABLE (RecordTest's literal comparisons), or -1; hist[f] counts the POIs
// whose first such frame is f.
template <int N, int ZNCC, int CONV>
__global__ void recover_scan_kernel(const float* __restrict__ out, size_t n, int f_begin, int f_end, const int* __restrict__ idx, int m,
	float zncc_low, float conv_max, int* __restrict__ first, int* __restrict__ hist) {
	for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
		const int i = idx ? idx[k] : k;
		int hit = -1;
		for (int f = f_begin; f < f_end; f++) {
			const float* const r = out + ((size_t)f * n + i) * N;
			if (r[ZNCC] < zncc_low || r[CONV] > conv_max) { hit = f; break; }
		}
		first[i] = hit;
		if (hit >= 0) atomicAdd(hist + hit, 1);
	}
}

constexpr int RECOVER_THREADS = 256;
inline int recover_grid(long long work, int sm_count) {
	const long long b = (work + RECOVER_THREADS - 1) / RECOVER_THREADS, cap = (long long)sm_count * 8;
	return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

} // namespace

size_t recover_select_bytes(size_t n) {
	size_t bytes = 0;
	cub::DeviceSelect::Flagged(nullptr, bytes, thrust::counting_iterator<int>(0), FlagIter(thrust::counting_iterator<int>(0), RecordTest{}), (int*)nullptr,
		(int*)nullptr, (int)n);
	return bytes;
}

cudaError_t recover_select_launch(int dim, const float* d_rec, size_t count, RecoverTest test, float zncc_high, float zncc_low, float conv, int* d_idx,
	int* d_count, void* d_temp, size_t temp_bytes, cudaStream_t stream) {
	const RecordTest f = dim == 2 ? RecordTest{ d_rec, P2_N, P2_ZNCC, P2_CONV, test, zncc_high, zncc_low, conv }
								  : RecordTest{ d_rec, P3_N, P3_ZNCC, P3_CONV, test, zncc_high, zncc_low, conv };
	size_t bytes = temp_bytes;
	return cub::DeviceSelect::Flagged(d_temp, bytes, thrust::counting_iterator<int>(0), FlagIter(thrust::counting_iterator<int>(0), f), d_idx, d_count,
		(int)count, stream);
}

cudaError_t recover_move_launch(int dim, const float* d_src, const int* d_src_idx, size_t total, const int* d_list1, const int* d_count1, float* d_dst1,
	float* d_q, const int* d_list2, float* d_dst2, int* d_idx2, int sm_count, cudaStream_t stream) {
	const long long work = (long long)total * (dim == 2 ? (int)P2_N : (int)P3_N), cap = (long long)sm_count * 8;
	long long grid = (work + RECOVER_THREADS - 1) / RECOVER_THREADS;
	grid = grid < 1 ? 1 : (grid > cap ? cap : grid);
	if (dim == 2)
		recover_move_kernel<P2_N><<<(int)grid, RECOVER_THREADS, 0, stream>>>(d_src, d_src_idx, (long long)total, d_list1, d_count1, d_dst1, d_q, d_list2,
			d_dst2, d_idx2);
	else
		recover_move_kernel<P3_N><<<(int)grid, RECOVER_THREADS, 0, stream>>>(d_src, d_src_idx, (long long)total, d_list1, d_count1, d_dst1, d_q, d_list2,
			d_dst2, d_idx2);
	return cudaGetLastError();
}

cudaError_t recover_collect_launch(const int* d_src_idx, size_t total, const int* d_list1, const int* d_count1, int* d_out, int sm_count,
	cudaStream_t stream) {
	recover_collect_kernel<<<recover_grid((long long)total, sm_count), RECOVER_THREADS, 0, stream>>>(d_src_idx, (int)total, d_list1, d_count1, d_out);
	return cudaGetLastError();
}

cudaError_t recover_scan_launch(int dim, const float* d_out, size_t n, int f_begin, int f_end, const int* d_idx, size_t m, float zncc_low, float conv,
	int* d_first, int* d_hist, int sm_count, cudaStream_t stream) {
	const int grid = recover_grid((long long)m, sm_count);
	if (dim == 2)
		recover_scan_kernel<P2_N, P2_ZNCC, P2_CONV><<<grid, RECOVER_THREADS, 0, stream>>>(d_out, n, f_begin, f_end, d_idx, (int)m, zncc_low, conv, d_first,
			d_hist);
	else
		recover_scan_kernel<P3_N, P3_ZNCC, P3_CONV><<<grid, RECOVER_THREADS, 0, stream>>>(d_out, n, f_begin, f_end, d_idx, (int)m, zncc_low, conv, d_first,
			d_hist);
	return cudaGetLastError();
}

} // namespace ocb
