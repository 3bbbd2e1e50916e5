// fft32.cuh -- 32-point complex FFTs held entirely in registers (fully unrolled radix-2, compile-time
// twiddles), shared by the 32x32 and 32x32x32 FFT-CC kernels.
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

// One radix-2 stage with butterflies `HALF` apart.  HALF is a template argument so that every loop below has a
// compile-time trip count and is unrolled completely (re/im then stay in registers instead of local memory).
template <bool INV, int HALF>
__device__ __forceinline__ void fft32_dif_stage(float* re, float* im) {
#pragma unroll
	for (int base = 0; base < 32; base += 2 * HALF) {
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

template <bool INV, int HALF>
__device__ __forceinline__ void fft32_dit_stage(float* re, float* im) {
#pragma unroll
	for (int base = 0; base < 32; base += 2 * HALF) {
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
	fft32_dif_stage<INV, 16>(re, im);
	fft32_dif_stage<INV, 8>(re, im);
	fft32_dif_stage<INV, 4>(re, im);
	fft32_dif_stage<INV, 2>(re, im);
	fft32_dif_stage<INV, 1>(re, im);
}

// radix-2 decimation in time: bit-reversed order in, natural order out
template <bool INV>
__device__ __forceinline__ void fft32_dit(float* re, float* im) {
	fft32_dit_stage<INV, 1>(re, im);
	fft32_dit_stage<INV, 2>(re, im);
	fft32_dit_stage<INV, 4>(re, im);
	fft32_dit_stage<INV, 8>(re, im);
	fft32_dit_stage<INV, 16>(re, im);
}

} // namespace ocb
