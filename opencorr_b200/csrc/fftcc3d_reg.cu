// fftcc3d_reg.cu -- FFT-CC for cubic windows of N = 2r points per side, N = 2^a 3^b 5^c <= 64 (other than the
// 32^3 window of fftcc3d_w32.cu): one CTA (128 threads) per POI, ONE THREAD PER 1D TRANSFORM, every N-point
// transform fully unrolled in that thread's registers (fft_codelet.cuh).  This covers the geometry of the
// reference's own DVC example (61^3 subvolumes -> 60^3 windows, examples/test_dvc_fftcc_icgn1.cpp).
//
// Same algorithm as fftcc3d_kernel (reference src/oc_fftcc.cpp:327-427), slab-decomposed:
//   pass 0 : means of both windows (coalesced rows, block reduction).
//   phase A: G = 128 / N z-slices at a time.  thread (g, t): column t of slice g while the slice is gathered
//            into a tile of odd pitch N + 1 (zero-mean, norms), then row t for the x transforms, then column
//            kx = t for the y transforms; the slice spectrum goes to the CTA's scratch volume S[z][ky][kx]
//            (threads along kx: coalesced).
//   phase B: one thread per (ky, kx) column: transform along z in registers, back to S in natural order;
//            after a barrier the same threads form C = conj(A) B from S(k) and the partner bin S(-k), inverse
//            transform along kz, and write the result to a SECOND scratch volume (a column's partner is another
//            thread's column, so S must stay intact until every column has been read).
//   phase C: per z-slice inverse along kx then ky through the tile, running first-maximum argmax with the
//            linear index (z N + y) N + x.
// The two scratch volumes (16 N^3 bytes per CTA) live in global memory / L2.
#include "fft_codelet.cuh"
#include "fftcc_common.cuh"
#include "ocb_kernels.h"

namespace ocb {

template <int N>
struct Fft3RegLayout {
	static constexpr int G = F3R_THREADS / N; // slices per round
	static constexpr int PITCH = N + 1;
	static constexpr int TILE = N * PITCH;
	static constexpr size_t SMEM = (size_t)2 * G * TILE * sizeof(float);
	static_assert(SMEM == fftcc3d_reg_smem_bytes(N), "the launch plan sizes the shared memory with fftcc3d_reg_smem_bytes");
};

template <int N>
__global__ void __launch_bounds__(F3R_THREADS, fft_reg_min_ctas(N)) fftcc3d_reg_kernel(Image3D img, float* __restrict__ pois, int n_poi,
	float2* __restrict__ scratch) {
	typedef Fft3RegLayout<N> L;
	constexpr int R = N / 2, G = L::G, PITCH = L::PITCH, NN = N * N;
	constexpr int M = N * N * N;
	extern __shared__ __align__(16) float f3r_smem[];
	__shared__ float red[4 * 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int g = tid / N, t = tid - g * N;
	const bool lane_ok = g < G;
	float* sre = f3r_smem + (size_t)(lane_ok ? g : 0) * 2 * L::TILE;
	float* sim = sre + L::TILE;
	const int dx = img.dx, dy = img.dy, dz = img.dz;
	float2* S = scratch + (size_t)blockIdx.x * 2 * M; // S[z][ky][kx]
	float2* S2 = S + M;

	for (int poi = blockIdx.x; poi < n_poi; poi += gridDim.x) {
		float* P = pois + (size_t)poi * P3_N;
		const float px = P[P3_X], py = P[P3_Y], pz = P[P3_Z];
		const float u0 = P[P3_DEF + 0], v0 = P[P3_DEF + 4], w0 = P[P3_DEF + 8];
		if (fftcc3d_skip(px, py, pz, u0, v0, w0, R, R, R, dx, dy, dz)) continue;
		__syncthreads(); // the previous POI is completely finished (record read, smem and scratch free)
		// float coordinate arithmetic then (int) truncation, as the reference (src/oc_fftcc.cpp:353-360)
		const float rpx = px + t - R;
		const int ax = (int)rpx, bx = (int)(rpx + u0);

		// ---- pass 0: means
		float sa = 0.f, sb = 0.f;
		if (lane_ok) {
			for (int z = g; z < N; z += G) {
				const float rpz = pz + z - R;
				const float* pa = img.ref + (size_t)(int)rpz * dy * dx + ax;
				const float* pb = img.tar + (size_t)(int)(rpz + w0) * dy * dx + bx;
#pragma unroll 10
				for (int r = 0; r < N; r++) {
					const float rpy = py + r - R;
					sa += __ldg(pa + (size_t)(int)rpy * dx);
					sb += __ldg(pb + (size_t)(int)(rpy + v0) * dx);
				}
			}
		}
		sa = warp_sum(sa);
		sb = warp_sum(sb);
		if (lane == 0) { red[warp] = sa; red[32 + warp] = sb; }
		__syncthreads();
		float ref_mean = 0.f, tar_mean = 0.f;
#pragma unroll
		for (int i = 0; i < F3R_THREADS / 32; i++) { ref_mean += red[i]; tar_mean += red[32 + i]; }
		ref_mean /= (float)M;
		tar_mean /= (float)M;

		float re[N], im[N];
		// ---- phase A: per z-slice forward 2D transform
		float na = 0.f, nb = 0.f;
		for (int z0 = 0; z0 < N; z0 += G) {
			const int z = z0 + g;
			const bool act = lane_ok && z < N;
			if (act) { // thread = column t: gather, zero-mean, norms
				const float rpz = pz + z - R;
				const float* pa = img.ref + (size_t)(int)rpz * dy * dx + ax;
				const float* pb = img.tar + (size_t)(int)(rpz + w0) * dy * dx + bx;
#pragma unroll 10
				for (int r = 0; r < N; r++) {
					const float rpy = py + r - R;
					const float a = __ldg(pa + (size_t)(int)rpy * dx) - ref_mean;
					const float b = __ldg(pb + (size_t)(int)(rpy + v0) * dx) - tar_mean;
					na = fmaf(a, a, na);
					nb = fmaf(b, b, nb);
					sre[r * PITCH + t] = a;
					sim[r * PITCH + t] = b;
				}
			}
			__syncthreads();
			if (act) { // thread = row t: transform along x
#pragma unroll
				for (int j = 0; j < N; j++) {
					re[j] = sre[t * PITCH + j];
					im[j] = sim[t * PITCH + j];
				}
				fft_reg<N, false>(re, im);
				fft_for_each_pos<N>([&](auto pos, auto freq) {
					sre[t * PITCH + freq.value] = re[pos.value];
					sim[t * PITCH + freq.value] = im[pos.value];
				});
			}
			__syncthreads();
			if (act) { // thread = column kx = t: transform along y, slice spectrum to S[z][ky][kx]
#pragma unroll
				for (int j = 0; j < N; j++) {
					re[j] = sre[j * PITCH + t];
					im[j] = sim[j * PITCH + t];
				}
				fft_reg<N, false>(re, im);
				float2* dst = S + (size_t)z * NN + t;
				fft_for_each_pos<N>([&](auto pos, auto freq) { dst[freq.value * N] = make_float2(re[pos.value], im[pos.value]); });
			}
			__syncthreads(); // tile free for the next round
		}
		na = warp_sum(na);
		nb = warp_sum(nb);
		if (lane == 0) { red[64 + warp] = na; red[96 + warp] = nb; }
		__syncthreads(); // S complete (same-CTA global writes are visible after the barrier), norms published

		// ---- phase B1: transform along z, one thread per (ky, kx) column; natural order back into S
		for (int col = tid; col < NN; col += F3R_THREADS) {
			float2* c = S + col;
#pragma unroll
			for (int z = 0; z < N; z++) {
				const float2 v = __ldcg(c + (size_t)z * NN);
				re[z] = v.x;
				im[z] = v.y;
			}
			fft_reg<N, false>(re, im);
			fft_for_each_pos<N>([&](auto pos, auto freq) { c[(size_t)freq.value * NN] = make_float2(re[pos.value], im[pos.value]); });
		}
		__syncthreads();
		// ---- phase B2: cross spectrum with the partner bin (src/oc_fftcc.cpp:378-388), inverse along kz, into S2
		for (int col = tid; col < NN; col += F3R_THREADS) {
			const int ky = col / N, kx = col - ky * N;
			const int pcol = (ky ? N - ky : 0) * N + (kx ? N - kx : 0);
			const float2* c = S + col;
			const float2* pc = S + pcol;
#pragma unroll
			for (int kz = 0; kz < N; kz++) {
				const int nkz = kz ? N - kz : 0;
				const float2 zv = __ldcg(c + (size_t)kz * NN), nv = __ldcg(pc + (size_t)nkz * NN);
				re[kz] = zv.x;
				im[kz] = zv.y;
				cross_spectrum(re[kz], im[kz], nv.x, nv.y);
			}
			fft_reg<N, true>(re, im);
			float2* o = S2 + col;
			fft_for_each_pos<N>([&](auto pos, auto freq) { o[(size_t)freq.value * NN] = make_float2(re[pos.value], im[pos.value]); });
		}
		__syncthreads();

		// ---- phase C: per z-slice inverse 2D transform + running argmax
		float bv = -2.f;
		int bi = 0;
		for (int z0 = 0; z0 < N; z0 += G) {
			const int z = z0 + g;
			const bool act = lane_ok && z < N;
			if (act) { // thread = column kx = t: slice into the tile
				const float2* src = S2 + (size_t)z * NN + t;
#pragma unroll 10
				for (int ky = 0; ky < N; ky++) {
					const float2 v = __ldcg(src + ky * N);
					sre[ky * PITCH + t] = v.x;
					sim[ky * PITCH + t] = v.y;
				}
			}
			__syncthreads();
			if (act) { // thread = row ky = t: inverse along kx
#pragma unroll
				for (int j = 0; j < N; j++) {
					re[j] = sre[t * PITCH + j];
					im[j] = sim[t * PITCH + j];
				}
				fft_reg<N, true>(re, im);
				fft_for_each_pos<N>([&](auto pos, auto freq) {
					sre[t * PITCH + freq.value] = re[pos.value];
					sim[t * PITCH + freq.value] = im[pos.value];
				});
			}
			__syncthreads();
			if (act) { // thread = column x = t: inverse along ky; first maximum (src/oc_fftcc.cpp:391-402)
#pragma unroll
				for (int j = 0; j < N; j++) {
					re[j] = sre[j * PITCH + t];
					im[j] = sim[j * PITCH + t];
				}
				fft_reg<N, true>(re, im);
				fft_for_each_pos<N>([&](auto pos, auto freq) { argmax_merge(bv, bi, re[pos.value], (z * N + freq.value) * N + t); });
			}
			__syncthreads();
		}
		warp_argmax(bv, bi);
		if (lane == 0) { red[warp] = bv; ((int*)red)[32 + warp] = bi; }
		__syncthreads();
		if (tid == 0) {
			float fv = red[0];
			int fi = ((int*)red)[32];
			for (int i = 1; i < F3R_THREADS / 32; i++) argmax_merge(fv, fi, red[i], ((int*)red)[32 + i]);
			float tna = 0.f, tnb = 0.f;
			for (int i = 0; i < F3R_THREADS / 32; i++) { tna += red[64 + i]; tnb += red[96 + i]; }
			fftcc3d_store(P, fv, fi, tna, tnb, R, R, R, u0, v0, w0);
		}
	}
}

cudaError_t fftcc3d_reg_launch(const Image3D& img, float* d_pois, size_t n_poi, const Fftcc3dPlan& plan, float2* scratch, int grid,
	cudaStream_t stream) {
	switch (plan.n) {
#define X(N) case N: return launch_smem(fftcc3d_reg_kernel<N>, grid, F3R_THREADS, plan.smem, stream, img, d_pois, (int)n_poi, scratch);
		OCB_FFT_REG_SIZES(X)
#undef X
	default: return cudaErrorInvalidValue;
	}
}

} // namespace ocb
