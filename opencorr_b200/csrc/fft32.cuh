// fft32.cuh -- 32- and 16-point complex FFTs held entirely in registers (fully unrolled radix-2, compile-time
// twiddles), shared by the 32x32 and 32x32x32 FFT-CC kernels, and the split that inverts a 32-point spectrum whose
// output is real as one 16-point transform.
#pragma once
#include "ocb_common.cuh"

namespace ocb {

__host__ __device__ constexpr int brev5(int i) {
	return ((i & 1) << 4) | ((i & 2) << 2) | (i & 4) | ((i & 8) >> 2) | ((i & 16) >> 4);
}

// (cos, sin) of 2*pi*k/32
__device__ __forceinline__ float tw32_cos(int k) {
	switch (k) {
	case 0: return 1.0f;
	case 1: return 0.98078528040323044913f;
	case 2: return 0.92387953251128675613f;
	case 3: return 0.83146961230254523708f;
	case 4: return 0.70710678118654752440f;
	case 5: return 0.55557023301960222474f;
	case 6: return 0.38268343236508977173f;
	case 7: return 0.19509032201612826785f;
	case 8: return 0.0f;
	case 9: return -0.19509032201612826785f;
	case 10: return -0.38268343236508977173f;
	case 11: return -0.55557023301960222474f;
	case 12: return -0.70710678118654752440f;
	case 13: return -0.83146961230254523708f;
	case 14: return -0.92387953251128675613f;
	default: return -0.98078528040323044913f;
	}
}
__device__ __forceinline__ float tw32_sin(int k) { return k < 8 ? tw32_cos(8 - k) : tw32_cos(k - 8); }

// (yr, yi) = (xr + i xi) * W, W = exp(-+ 2 pi i k / 32)  (minus: forward, plus: inverse)
template <bool INV>
__device__ __forceinline__ void mul_tw32(float xr, float xi, int k, float& yr, float& yi) {
	if (k == 0) {
		yr = xr;
		yi = xi;
	} else if (k == 8) { // -i (forward) / +i (inverse)
		yr = INV ? -xi : xi;
		yi = INV ? xr : -xr;
	} else {
		const float c = tw32_cos(k), s = INV ? -tw32_sin(k) : tw32_sin(k); // W = c - i s
		yr = fmaf(xr, c, xi * s);
		yi = fmaf(xi, c, -xr * s);
	}
}

// One radix-2 stage of an N-point transform (N = 16 or 32) with butterflies `HALF` apart: twiddle W_{2 HALF}^k =
// W_32^{16 k / HALF}.  HALF is a template argument so that every loop below has a compile-time trip count and is unrolled
// completely (re/im then stay in registers instead of local memory).
template <int N, bool INV, int HALF>
__device__ __forceinline__ void fft_dif_stage(float* re, float* im) {
#pragma unroll
	for (int base = 0; base < N; base += 2 * HALF) {
#pragma unroll
		for (int k = 0; k < HALF; k++) {
			const int i = base + k, j = i + HALF;
			const float ar = re[i], ai = im[i], br = re[j], bi = im[j];
			re[i] = ar + br;
			im[i] = ai + bi;
			mul_tw32<INV>(ar - br, ai - bi, k * (16 / HALF), re[j], im[j]);
		}
	}
}

template <int N, bool INV, int HALF>
__device__ __forceinline__ void fft_dit_stage(float* re, float* im) {
#pragma unroll
	for (int base = 0; base < N; base += 2 * HALF) {
#pragma unroll
		for (int k = 0; k < HALF; k++) {
			const int i = base + k, j = i + HALF;
			float tr, ti;
			mul_tw32<INV>(re[j], im[j], k * (16 / HALF), tr, ti);
			const float ar = re[i], ai = im[i];
			re[i] = ar + tr;
			im[i] = ai + ti;
			re[j] = ar - tr;
			im[j] = ai - ti;
		}
	}
}

// radix-2 decimation in frequency: natural order in, bit-reversed order out
template <bool INV>
__device__ __forceinline__ void fft32_dif(float* re, float* im) {
	fft_dif_stage<32, INV, 16>(re, im);
	fft_dif_stage<32, INV, 8>(re, im);
	fft_dif_stage<32, INV, 4>(re, im);
	fft_dif_stage<32, INV, 2>(re, im);
	fft_dif_stage<32, INV, 1>(re, im);
}

// radix-2 decimation in time: bit-reversed order in, natural order out
template <bool INV>
__device__ __forceinline__ void fft32_dit(float* re, float* im) {
	fft_dit_stage<32, INV, 1>(re, im);
	fft_dit_stage<32, INV, 2>(re, im);
	fft_dit_stage<32, INV, 4>(re, im);
	fft_dit_stage<32, INV, 8>(re, im);
	fft_dit_stage<32, INV, 16>(re, im);
}

// 16 points in re[0..15], im[0..15]; natural order in, bit-reversed order out (register j holds bin brev5(2 j) = brev4(j))
template <bool INV>
__device__ __forceinline__ void fft16_dif(float* re, float* im) {
	fft_dif_stage<16, INV, 8>(re, im);
	fft_dif_stage<16, INV, 4>(re, im);
	fft_dif_stage<16, INV, 2>(re, im);
	fft_dif_stage<16, INV, 1>(re, im);
}

// 16 points in re[0..15], im[0..15]; bit-reversed order in, natural order out
template <bool INV>
__device__ __forceinline__ void fft16_dit(float* re, float* im) {
	fft_dit_stage<16, INV, 1>(re, im);
	fft_dit_stage<16, INV, 2>(re, im);
	fft_dit_stage<16, INV, 4>(re, im);
	fft_dit_stage<16, INV, 8>(re, im);
}

// Inverse 32-point transform of a spectrum C whose output c(x) is known to be real (bit-reversed order in: register i holds
// C(brev5(i))), first half.  Splitting the output into even and odd x, c(2n) = IDFT16(E)(n) and c(2n+1) = IDFT16(O)(n) with
//   E(k) = C(k) + C(k + 16),  O(k) = W^k (C(k) - C(k + 16)),  W = exp(+2 pi i / 32),
// and since both are real, one 16-point inverse of Z = E + i O gives z(n) = c(2n) + i c(2n+1).  The pair (k, k + 16) sits in
// registers (2j, 2j+1) with k = brev4(j); Z(k) is left in register j, bit-reversed order out: fft16_dit<true> finishes the
// transform in natural order.  Linear in C, so the same split applies to each row of a 2D spectrum whose 2D inverse is real.
__device__ __forceinline__ void ifft32_real_split(float* re, float* im) {
#pragma unroll
	for (int j = 0; j < 16; j++) {
		const int k = brev5(2 * j);
		const float ar = re[2 * j], ai = im[2 * j], br = re[2 * j + 1], bi = im[2 * j + 1];
		if (k == 0) { // i O = i D
			re[j] = (ar + br) - (ai - bi);
			im[j] = (ai + bi) + (ar - br);
		} else if (k == 8) { // i O = i i D = -D: Z = E - D = 2 C(24)
			re[j] = br + br;
			im[j] = bi + bi;
		} else { // i W^k D = (-dr s - di c) + i (dr c - di s)
			const float er = ar + br, ei = ai + bi, dr = ar - br, di = ai - bi;
			const float c = tw32_cos(k), s = tw32_sin(k);
			re[j] = fmaf(-dr, s, fmaf(-di, c, er));
			im[j] = fmaf(dr, c, fmaf(-di, s, ei));
		}
	}
}

} // namespace ocb
