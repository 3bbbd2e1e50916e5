// fftcc2d_reg.cu -- FFT-CC for square windows of N = 2r points per side, N = 2^a 3^b 5^c <= 64 (other than the
// 32x32 window, which fftcc2d_w32.cu handles with one warp per POI): ONE THREAD PER WINDOW ROW, every
// N-point transform fully unrolled in that thread's registers (fft_codelet.cuh), rows <-> columns
// exchanged through a padded shared-memory tile.
//
// Same algorithm as fftcc2d_kernel (reference src/oc_fftcc.cpp:177-275): z = ref + i*tar packed, one
// forward 2D transform, C = conj(A) B from Z(k) and Z(-k), one inverse transform, first-maximum argmax.
// A CTA of 128 threads carries PP = 128 / N POIs at a time (N = 40: three POIs on 120 threads); thread
// (slot, t) is column t while the windows are gathered (coalesced image rows), row t for the x
// transforms and column t for the y transforms.  The tile pitch N + 1 is odd, so both the row-wise and
// the column-wise accesses of a warp fall on distinct banks.  ~9 k warp instructions per 40x40 POI against
// ~35 k for the Stockham-over-shared-memory kernel in fftcc.cu, which remains the fallback for
// non-square windows and sizes with other prime factors.
#include "fft_codelet.cuh"
#include "fftcc_common.cuh"
#include "ocb_kernels.h"

namespace ocb {

template <int N>
struct FftRegLayout {
	static constexpr int PP = FFTREG_THREADS / N;         // POIs per CTA
	static constexpr int PITCH = N + 1;
	static constexpr int TILE = N * PITCH;                // floats per plane
	static constexpr int RED = 4 * FFTREG_THREADS;        // per-thread partials: 4 floats
	static constexpr size_t SMEM = ((size_t)2 * PP * TILE + RED) * sizeof(float);
	static_assert(SMEM == fftcc2d_reg_smem_bytes(N), "the launch plan sizes the shared memory with fftcc2d_reg_smem_bytes");
};

template <int N>
__global__ void __launch_bounds__(FFTREG_THREADS, fft_reg_min_ctas(N)) fftcc2d_reg_kernel(Image2D img, float* __restrict__ pois, int n_poi) {
	typedef FftRegLayout<N> L;
	constexpr int R = N / 2, M = N * N, PP = L::PP, PITCH = L::PITCH;
	extern __shared__ __align__(16) float smem_f[];
	const int tid = threadIdx.x;
	const int slot = tid / N, t = tid - slot * N;
	const bool lane_ok = slot < PP; // threads past PP * N idle through the transforms (they still join the barriers)
	float* sre = smem_f + (size_t)(lane_ok ? slot : 0) * 2 * L::TILE;
	float* sim = sre + L::TILE;
	float* red = smem_f + (size_t)2 * PP * L::TILE; // [4][FFTREG_THREADS]
	const int w = img.w, h = img.h;
	const int n_batch = (n_poi + PP - 1) / PP;

	for (int batch = blockIdx.x; batch < n_batch; batch += gridDim.x) {
		const int poi = batch * PP + slot;
		bool active = lane_ok && poi < n_poi;
		float px = 0.f, py = 0.f, u0 = 0.f, v0 = 0.f;
		float* P = pois + (size_t)(active ? poi : 0) * P2_N;
		if (active) {
			px = P[P2_X]; py = P[P2_Y]; u0 = P[P2_DEF + D2_U]; v0 = P[P2_DEF + D2_V];
			if (fftcc2d_skip(px, py, u0, v0, R, R, w, h)) active = false;
		}
		__syncthreads(); // previous batch's readers of the tiles / red are done

		// ---- gather: thread = column; float coordinate arithmetic then (int) truncation (src/oc_fftcc.cpp:204-219)
		float sa = 0.f, sb = 0.f;
		if (active) {
			const float rpx = px + t - R;
			const int ax = (int)rpx, bx = (int)(rpx + u0);
#pragma unroll 20
			for (int r = 0; r < N; r++) {
				const float rpy = py + r - R;
				const float a = __ldg(img.ref + (size_t)(int)rpy * w + ax);
				const float b = __ldg(img.tar + (size_t)(int)(rpy + v0) * w + bx);
				sre[r * PITCH + t] = a;
				sim[r * PITCH + t] = b;
				sa += a;
				sb += b;
			}
		}
		red[tid] = sa;
		red[FFTREG_THREADS + tid] = sb;
		__syncthreads();
		float re[N], im[N];
		float na = 0.f, nb = 0.f;
		if (active) {
			float ma = 0.f, mb = 0.f;
			for (int j = 0; j < N; j++) { // every thread of the slot adds the same partials in the same order
				ma += red[slot * N + j];
				mb += red[FFTREG_THREADS + slot * N + j];
			}
			ma /= (float)M;
			mb /= (float)M;
			// ---- thread = row: zero-mean windows, norms, transform along x
#pragma unroll
			for (int j = 0; j < N; j++) {
				re[j] = sre[t * PITCH + j] - ma;
				im[j] = sim[t * PITCH + j] - mb;
				na = fmaf(re[j], re[j], na);
				nb = fmaf(im[j], im[j], nb);
			}
			fft_reg<N, false>(re, im);
			fft_for_each_pos<N>([&](auto pos, auto freq) {
				sre[t * PITCH + freq.value] = re[pos.value];
				sim[t * PITCH + freq.value] = im[pos.value];
			});
		}
		red[2 * FFTREG_THREADS + tid] = na;
		red[3 * FFTREG_THREADS + tid] = nb;
		__syncthreads();
		if (active) {
			// ---- thread = column kx: transform along y, spectrum back to the tile in natural order
#pragma unroll
			for (int j = 0; j < N; j++) {
				re[j] = sre[j * PITCH + t];
				im[j] = sim[j * PITCH + t];
			}
			fft_reg<N, false>(re, im);
		}
		__syncthreads(); // all columns read before any is overwritten
		if (active) {
			fft_for_each_pos<N>([&](auto pos, auto freq) {
				sre[freq.value * PITCH + t] = re[pos.value];
				sim[freq.value * PITCH + t] = im[pos.value];
			});
		}
		__syncthreads();
		if (active) {
			// ---- cross spectrum C(ky, kx) = conj(A) B with the partner bin Z(-ky, -kx) (src/oc_fftcc.cpp:239-240)
			const int tn = t ? N - t : 0;
#pragma unroll
			for (int ky = 0; ky < N; ky++) {
				const int kn = ky ? N - ky : 0;
				re[ky] = sre[ky * PITCH + t];
				im[ky] = sim[ky * PITCH + t];
				cross_spectrum(re[ky], im[ky], sre[kn * PITCH + tn], sim[kn * PITCH + tn]);
			}
			fft_reg<N, true>(re, im); // inverse along ky
		}
		__syncthreads(); // every partner bin read before the tile is overwritten
		if (active) {
			fft_for_each_pos<N>([&](auto pos, auto freq) {
				sre[freq.value * PITCH + t] = re[pos.value];
				sim[freq.value * PITCH + t] = im[pos.value];
			});
		}
		__syncthreads();
		float bv = -2.f;
		int bi = 0;
		if (active) {
			// ---- thread = row y: inverse along kx; first maximum in linear order y*N + x (src/oc_fftcc.cpp:246-255)
#pragma unroll
			for (int j = 0; j < N; j++) {
				re[j] = sre[t * PITCH + j];
				im[j] = sim[t * PITCH + j];
			}
			fft_reg<N, true>(re, im);
			fft_for_each_pos<N>([&](auto pos, auto freq) {
				argmax_merge(bv, bi, re[pos.value], t * N + freq.value);
			});
		}
		// (the mean partials in red[0 .. 2T) were consumed many barriers ago; the norm partials in red[2T .. 4T) stay)
		red[tid] = bv;
		((int*)red)[FFTREG_THREADS + tid] = bi;
		__syncthreads();
		if (active && t == 0) {
			float sna = 0.f, snb = 0.f;
			for (int j = 0; j < N; j++) {
				sna += red[2 * FFTREG_THREADS + slot * N + j];
				snb += red[3 * FFTREG_THREADS + slot * N + j];
				const float ov = red[slot * N + j];
				const int oi = ((int*)red)[FFTREG_THREADS + slot * N + j];
				// argmax_merge's rule, spelled out: through the function ptxas spills at N = 40 and reallocates five other sizes
				if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
			}
			fftcc2d_store(P, bv, bi, sna, snb, R, R, u0, v0);
		}
	}
}

cudaError_t fftcc2d_reg_launch(const Image2D& img, float* d_pois, size_t n, int r, const Fftcc2dPlan& plan, int grid, cudaStream_t stream) {
	switch (2 * r) {
#define X(N) case N: return launch_smem(fftcc2d_reg_kernel<N>, grid, FFTREG_THREADS, plan.smem, stream, img, d_pois, (int)n);
		OCB_FFT_REG_SIZES(X)
#undef X
	default: return cudaErrorInvalidValue;
	}
}

} // namespace ocb
