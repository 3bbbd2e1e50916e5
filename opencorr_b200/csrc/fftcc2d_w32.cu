// fftcc2d_w32.cu -- FFT-CC for the 32x32 window (subset radius 16, the headline configuration):
// ONE WARP PER POI, the 32-point transforms live entirely in registers.
//
// Same algorithm as fftcc2d_kernel (reference src/oc_fftcc.cpp:177-275), specialised:
//   lane = window column: each lane gathers its column of both windows (coalesced rows), the packed
//     z = ref + i*tar column is transformed along y with a fully unrolled radix-2 DIF FFT
//     (compile-time twiddles, natural order in -> bit-reversed order out, tracked statically);
//   transpose through a padded 32x33 shared tile of (re, im) pairs; lane = ky: DIF FFT along x;
//   cross spectrum 4C = 4 conj(A) B from Z(k) and Z(-k) (cross_spectrum4: exactly 4 times C, without its halvings): the
//     partner bin sits in lane (32-ky)%32 at a statically known register, fetched with warp shuffles;
//   inverse: the surface c is real, so it is computed as ONE 32 x 16 complex transform of z(y, n) = c(y, 2n) + i c(y, 2n+1):
//     lane = ky: the even/odd split of each row (ifft32_real_split) and a 16-point DIT along kx; transpose back (16 values
//     per lane); lane = (n, parity of y): half of the first DIF stage along ky, then a 16-point DIF;
//   first-maximum argmax over registers (each lane: 16 rows x 2 columns) + warp shuffle reduction.
// No CTA barrier, no integer division, ~2.2k warp instructions per POI (the generic kernel: ~23k).
//
// Window loads: when the POI and its guess sit on whole pixels (the normal FFT-CC case: grid POIs, integer guess) and the
// image pitch allows it, the two 32x32 windows arrive by TMA -- one cp.async.bulk.tensor.2d box of 36 x 32 floats each
// (x origin rounded down to 16 bytes), straight into the shared tiles the transposes use afterwards, completion on a
// per-warp mbarrier -- and every lane then picks its column out of shared memory.  Otherwise the lanes gather their
// columns with coalesced global loads (the reference's float-coordinate truncation, src/oc_fftcc.cpp:204-219, evaluated
// per pixel).  Both paths deliver the same 2 x 1024 values.
#include <stdlib.h>
#include <string.h>

#include "fft32.cuh"
#include "fftcc_common.cuh"
#include "ocb_kernels.h"
#include "ocb_tma.cuh"

namespace ocb {

constexpr int FFTW32_PITCH = 33;
constexpr int FFTW32_BOX_W = 36;                 // TMA box: 32 columns + up to 3 of alignment slack
constexpr int FFTW32_TILE = 32 * FFTW32_BOX_W;   // floats per TMA box (36 x 32)
// A warp's buffer holds the two boxes (reference, target) or one 32 x 33 transpose tile of complex values: (re, im) pairs
// cross it as one 64-bit access, half the shared-memory instructions of separate re and im tiles.  The odd pitch keeps
// every half-warp's 16 pairs in distinct banks both ways.
static_assert(32 * FFTW32_PITCH * 2 <= 2 * FFTW32_TILE, "the transpose tile must fit in the two boxes");

__global__ void __launch_bounds__(FFTW32_WARPS * 32) fftcc2d_w32_kernel(Image2D img, float* __restrict__ pois, int n_poi,
	const __grid_constant__ CUtensorMap tm_ref, const __grid_constant__ CUtensorMap tm_tar, int use_tma) {
	__shared__ __align__(128) float s_buf[FFTW32_WARPS][2 * FFTW32_TILE];
	__shared__ __align__(8) uint64_t s_bar[FFTW32_WARPS];
	constexpr int R = 16, M = 32 * 32;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	float* sre = s_buf[warp];              // reference box
	float* sim = s_buf[warp] + FFTW32_TILE; // target box
	float2* st = reinterpret_cast<float2*>(s_buf[warp]); // transpose tile
	uint64_t* bar = &s_bar[warp];
	uint32_t bar_phase = 0;
	if (use_tma) {
		if (lane == 0) mbar_init(bar, 1);
		__syncwarp();
	}
	const int w = img.w, h = img.h;
	const int plane = (32 - lane) & 31;

	// the record of the NEXT POI of this warp is requested one POI ahead: the queue may be read in place from page-locked host
	// memory, a few microseconds away
	const int poi_stride = gridDim.x * FFTW32_WARPS;
	int poi = blockIdx.x * FFTW32_WARPS + warp;
	float rec_next = (poi < n_poi && lane < P2_N) ? pois[(size_t)poi * P2_N + lane] : 0.f;
	for (; poi < n_poi; poi += poi_stride) {
		float* P = pois + (size_t)poi * P2_N;
		const float rec = rec_next;
		if (poi + poi_stride < n_poi && lane < P2_N) rec_next = pois[(size_t)(poi + poi_stride) * P2_N + lane];
		const float px = __shfl_sync(0xffffffffu, rec, P2_X), py = __shfl_sync(0xffffffffu, rec, P2_Y);
		const float u0 = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_U), v0 = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_V);
		if (fftcc2d_skip(px, py, u0, v0, R, R, w, h)) continue;
		// gather: lane = column; float coordinate arithmetic then (int) truncation (src/oc_fftcc.cpp:204-219)
		float re[32], im[32];
		{
			float sa = 0.f, sb = 0.f;
			// whole-pixel POI and guess (warp-uniform): every truncation below is the identity, the windows are two boxes
			if (use_tma && px == floorf(px) && py == floorf(py) && u0 == floorf(u0) && v0 == floorf(v0)) {
				const int x0r = (int)px - R, y0r = (int)py - R, x0t = (int)(px + u0) - R, y0t = (int)(py + v0) - R;
				const int axr = floor4(x0r), axt = floor4(x0t);
				if (lane == 0) {
					fence_proxy_async(); // the previous POI's generic-proxy accesses to the tiles come first
					mbar_expect_tx(bar, (uint32_t)(2 * FFTW32_TILE * sizeof(float)));
					tma_load_2d(sre, &tm_ref, axr, y0r, bar);
					tma_load_2d(sim, &tm_tar, axt, y0t, bar);
				}
				mbar_wait(bar, bar_phase);
				bar_phase ^= 1;
				const float* cr = sre + (x0r - axr) + lane;
				const float* ci = sim + (x0t - axt) + lane;
#pragma unroll
				for (int r = 0; r < 32; r++) {
					re[r] = cr[r * FFTW32_BOX_W];
					im[r] = ci[r * FFTW32_BOX_W];
					sa += re[r];
					sb += im[r];
				}
			} else {
				const float rpx = px + lane - R;
				const int ax = (int)rpx, bx = (int)(rpx + u0);
#pragma unroll
				for (int r = 0; r < 32; r++) {
					const float rpy = py + r - R;
					re[r] = __ldg(img.ref + (size_t)(int)rpy * w + ax);
					im[r] = __ldg(img.tar + (size_t)(int)(rpy + v0) * w + bx);
					sa += re[r];
					sb += im[r];
				}
			}
			sa = warp_sum(sa) / (float)M;
			sb = warp_sum(sb) / (float)M;
#pragma unroll
			for (int r = 0; r < 32; r++) {
				re[r] -= sa;
				im[r] -= sb;
			}
		}
		float na = 0.f, nb = 0.f;
#pragma unroll
		for (int r = 0; r < 32; r++) {
			na = fmaf(re[r], re[r], na);
			nb = fmaf(im[r], im[r], nb);
		}
		na = warp_sum(na);
		nb = warp_sum(nb);

		fft32_dif<false>(re, im); // along y: register i holds ky = brev5(i)
		__syncwarp();
#pragma unroll
		for (int i = 0; i < 32; i++) st[brev5(i) * FFTW32_PITCH + lane] = make_float2(re[i], im[i]);
		__syncwarp();
#pragma unroll
		for (int i = 0; i < 32; i++) { // lane = ky, register i = x
			const float2 v = st[lane * FFTW32_PITCH + i];
			re[i] = v.x;
			im[i] = v.y;
		}
		fft32_dif<false>(re, im); // along x: register i holds kx = brev5(i)

		// cross spectrum, times 4 (cross_spectrum4); partner of (ky, kx) is (-ky, -kx): lane `plane`, register brev5((32 - kx) % 32)
#pragma unroll
		for (int i = 0; i < 32; i++) {
			const int ip = brev5((32 - brev5(i)) & 31);
			if (ip < i) continue;
			const float pr_i = __shfl_sync(0xffffffffu, re[i], plane), pi_i = __shfl_sync(0xffffffffu, im[i], plane);
			if (ip == i) {
				cross_spectrum4(re[i], im[i], pr_i, pi_i);
			} else {
				const float pr_p = __shfl_sync(0xffffffffu, re[ip], plane), pi_p = __shfl_sync(0xffffffffu, im[ip], plane);
				cross_spectrum4(re[i], im[i], pr_p, pi_p);
				cross_spectrum4(re[ip], im[ip], pr_i, pi_i);
			}
		}

		// inverse: the surface (4c) is real, so it comes out of one 32 x 16 transform of z(y, n) = c(y, 2n) + i c(y, 2n+1)
		ifft32_real_split(re, im); // lane = ky, register j holds kx = brev4(j) of the packed row
		fft16_dit<true>(re, im);   // along kx: register n = column pair n
		__syncwarp();
#pragma unroll
		for (int n = 0; n < 16; n++) st[lane * FFTW32_PITCH + n] = make_float2(re[n], im[n]);
		__syncwarp();
		// along ky: lane = (column pair n, parity h of y).  The first DIF stage of the 32-point inverse is done by halves: h = 0
		// keeps the sums (even y), h = 1 the differences times W^ky (odd y), with a lane-dependent twiddle so both halves run
		// the same code; then a 16-point inverse.
		// The twiddle is t W^(h ky) = t + h (W^ky - 1) t, exact for h = 0; selecting the twiddle instead would hold 30
		// lane-dependent constants in registers.
		const int n = lane & 15, h = lane >> 4;
		const float hf = (float)h, sgn = 1.f - 2.f * hf;
#pragma unroll
		for (int ky = 0; ky < 16; ky++) {
			const float2 a = st[ky * FFTW32_PITCH + n], b = st[(ky + 16) * FFTW32_PITCH + n];
			const float tr = fmaf(sgn, b.x, a.x), ti = fmaf(sgn, b.y, a.y);
			if (ky == 0) {
				re[ky] = tr;
				im[ky] = ti;
			} else {
				const float cm1 = tw32_cos(ky) - 1.f, s = tw32_sin(ky);
				re[ky] = fmaf(hf, fmaf(tr, cm1, -ti * s), tr);
				im[ky] = fmaf(hf, fmaf(ti, cm1, tr * s), ti);
			}
		}
		fft16_dif<true>(re, im); // register j holds y = 2 brev4(j) + h; real part x = 2n, imaginary part x = 2n + 1

		// first maximum in linear order y*32 + x (src/oc_fftcc.cpp:246-255), from -2 on the surface, -8 on 4c; a lane's
		// candidates, in increasing index, are i0 + 64 m (+ 1).  The scan keeps the offset from i0, an immediate per
		// candidate; a lane without a candidate ends at 0, as the reference's scan starts.
		float bv = -8.f;
		const int i0 = h * 32 + 2 * n;
		int bi = -i0;
#pragma unroll
		for (int m = 0; m < 16; m++) {
			const int j = brev5(2 * m);
			if (re[j] > bv) { bv = re[j]; bi = m * 64; }
			if (im[j] > bv) { bv = im[j]; bi = m * 64 + 1; }
		}
		bi += i0;
		warp_argmax(bv, bi);
		{ // one store instruction for the five result fields (the queue may sit in page-locked host memory)
			const Fftcc2dResult res = fftcc2d_result(0.25f * bv, bi, na, nb, R, R, u0, v0);
			float out = 0.f;
			if (lane == P2_DEF + D2_U) out = res.u;
			if (lane == P2_DEF + D2_V) out = res.v;
			if (lane == P2_U0) out = u0;
			if (lane == P2_V0) out = v0;
			if (lane == P2_ZNCC) out = res.zncc;
			if (lane == P2_DEF + D2_U || lane == P2_DEF + D2_V || lane == P2_U0 || lane == P2_V0 || lane == P2_ZNCC) P[lane] = out;
		}
		__syncwarp();
	}
}

cudaError_t fftcc2d_w32_launch(const Image2D& img, float* d_pois, size_t n, int grid, cudaStream_t stream) {
	CUtensorMap tm_ref, tm_tar;
	memset(&tm_ref, 0, sizeof(tm_ref));
	memset(&tm_tar, 0, sizeof(tm_tar));
	const int dims[2] = { img.w, img.h }, box[2] = { FFTW32_BOX_W, 32 };
	const int use_tma = tma_enabled() && tma_make_map(&tm_ref, img.ref, 2, dims, box) && tma_make_map(&tm_tar, img.tar, 2, dims, box);
	fftcc2d_w32_kernel<<<grid, FFTW32_WARPS * 32, 0, stream>>>(img, d_pois, (int)n, tm_ref, tm_tar, use_tma);
	return cudaGetLastError();
}

} // namespace ocb
