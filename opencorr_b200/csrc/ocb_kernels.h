// ocb_kernels.h -- host-visible launch interfaces of the sm_90a kernels (internal to the library).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <string>

#include "ocb_common.cuh"
#include "ocb_tma.cuh"

namespace ocb {

// Factorisation of one FFT axis into Stockham stages (radix 4/2/3/5, generic odd radix <= 31).
struct FftAxis {
	int n;
	int nstage;
	int radix[16];
};

inline bool fft_plan_axis(int n, FftAxis* ax) {
	ax->n = n;
	ax->nstage = 0;
	int m = n;
	while (m % 4 == 0) { ax->radix[ax->nstage++] = 4; m /= 4; }
	while (m % 2 == 0) { ax->radix[ax->nstage++] = 2; m /= 2; }
	while (m % 3 == 0) { ax->radix[ax->nstage++] = 3; m /= 3; }
	while (m % 5 == 0) { ax->radix[ax->nstage++] = 5; m /= 5; }
	for (int p = 7; m > 1; p += 2) {
		while (m % p == 0) {
			if (p > 31 || ax->nstage >= 15) return false;
			ax->radix[ax->nstage++] = p;
			m /= p;
		}
	}
	return true;
}

// sift3d.cu (SIFT3D feature extraction and matching; state kept between ocb_sift3d and the calls that read its results)
struct Sift3d;
enum { SIFT3D_STAGES = 10 }; // ref: pyramid, extrema, orientation, descriptors; tar: the same four; matching; host post-pass
Sift3d* sift3d_create();
void sift3d_destroy(Sift3d* s);
int sift3d_run(Sift3d* s, const float* d_ref, const float* d_tar, int nx, int ny, int nz, const float* cfg, const float* unit, float ratio,
	int sm_count, cudaStream_t stream, long long* launches, std::string* err);
size_t sift3d_n_matched(const Sift3d* s);
int sift3d_n_octave(const Sift3d* s, int which);
const float* sift3d_stage_ms(const Sift3d* s);
void sift3d_get_matches(const Sift3d* s, float* ref_xyz, float* tar_xyz);
int sift3d_inspect(const Sift3d* s, int which, size_t* counts, int* cand, float* max_abs, float* kp, float* desc, cudaStream_t stream, std::string* err);
// icgn2d.cu
constexpr int ICGN2D_TILE_MARGIN = 1; // slack (pixels) around subset+support in the target tile
// TMA tile loads need the innermost coordinate 16-byte aligned (x multiple of 4 floats; seen: an
// unaligned x raises 'illegal instruction'), so tile origins are rounded down to a multiple of 4 and
// the boxes are 3 columns wider.
__host__ __device__ inline int icgn2d_ref_w(int rx) { return round_up4(2 * rx + 1 + 4 + 3); }
__host__ __device__ inline int icgn2d_ref_h(int ry) { return 2 * ry + 1 + 4; }
__host__ __device__ inline int icgn2d_tar_w(int rx) { return round_up4(2 * rx + 1 + 3 + 2 * ICGN2D_TILE_MARGIN + 3); }
__host__ __device__ inline int icgn2d_tar_h(int ry) { return 2 * ry + 1 + 3 + 2 * ICGN2D_TILE_MARGIN; }
// per-warp slab (floats): [0,32) mbarrier + pad | tile T (TMA destination, 128-B aligned) | R', gx, gy
__host__ __device__ inline int icgn2d_tile_floats(int rx, int ry) {
	const int a = icgn2d_ref_w(rx) * icgn2d_ref_h(ry), b = icgn2d_tar_w(rx) * icgn2d_tar_h(ry);
	return round_up32(a > b ? a : b);
}
// lm: the Levenberg-Marquardt variant keeps the undamped Hessian (<= 78 floats) behind the constants;
// wpp > 1 (warps per POI): a reduction area follows -- wpp x 96 floats of setup partials, 2 x wpp x 32 floats of
// per-iteration partials (double-buffered by iteration parity)
constexpr int ICGN2D_RED_SETUP = 96, ICGN2D_RED_ITER = 32;
__host__ __device__ inline int icgn2d_slab_floats(int rx, int ry, bool lm, int wpp) {
	const int n = (2 * rx + 1) * (2 * ry + 1);
	return 32 + icgn2d_tile_floats(rx, ry) + round_up32(3 * n) + (lm ? 96 : 0) + (wpp > 1 ? wpp * (ICGN2D_RED_SETUP + 2 * ICGN2D_RED_ITER) : 0);
}

// Resident one-POI CTAs per SM with wpp warps per POI (0: the slab exceeds the opt-in limit per block)
inline int icgn2d_slots(int rx, int ry, bool lm, int wpp, size_t smem_optin) {
	const size_t b = (size_t)icgn2d_slab_floats(rx, ry, lm, wpp) * sizeof(float);
	if (b > smem_optin) return 0;
	const int k = (int)((228 * 1024) / (b + 1024));
	return k > 32 ? 32 : k;
}

// Launch geometry of icgn2d_kernel<NP, RC, LM, WPP> for a queue of n POIs: one CTA of wpp warps per POI at a time, persistent
// CTAs (one wave) pulling POIs from a work counter.
struct Icgn2dPlan {
	int wpp;           // warps per POI (1 or 2)
	int rc;            // radius baked into the kernel (16: ICGN2D1, 20: ICGN2D2), 0 for the generic and the LM kernels
	int blocks_per_sm; // resident CTAs per SM
	int grid;
	size_t smem;       // dynamic shared memory per CTA
};

// false when the slab does not fit in shared memory (smem_optin: the device's opt-in limit per block).  wpp_override: 1 or 2
// forces the warps per POI (2 only where its slab fits), anything else leaves the choice to the queue length.
inline bool icgn2d_plan(size_t n, int np, int rx, int ry, bool lm, int sm_count, size_t smem_optin, int wpp_override, Icgn2dPlan* p) {
	// Warps per POI (tools/ab_icgn2d.sh compares the two): with the GPU full, one warp per POI wins -- the second warp
	// doubles the resident warps but also the per-POI fixed work and adds a barrier per pass; with fewer POIs than resident
	// slots, two warps per POI shorten the tail.  So: 2 only when the queue cannot fill the machine.
	const int s2 = icgn2d_slots(rx, ry, lm, 2, smem_optin);
	int wpp = ((long long)n < (long long)sm_count * icgn2d_slots(rx, ry, lm, 1, smem_optin) && (2 * ry + 1) >= 8 && s2 > 0) ? 2 : 1;
	if (wpp_override == 1 || (wpp_override == 2 && s2 > 0)) wpp = wpp_override;
	const size_t smem = (size_t)icgn2d_slab_floats(rx, ry, lm, wpp) * sizeof(float);
	if (smem > smem_optin) return false;
	int blocks_per_sm = icgn2d_slots(rx, ry, lm, wpp, smem_optin);
	if (blocks_per_sm < 1) blocks_per_sm = 1;
	const long long resident = (long long)sm_count * blocks_per_sm;
	int grid = (int)((long long)n < resident ? (long long)n : resident);
	if (grid < 1) grid = 1;
	p->wpp = wpp;
	p->rc = lm ? 0 : (np == 6 ? (rx == 16 && ry == 16 ? 16 : 0) : (rx == 20 && ry == 20 ? 20 : 0));
	p->blocks_per_sm = blocks_per_sm;
	p->grid = grid;
	p->smem = smem;
	return true;
}

// plan_n: the queue length whose warps per POI the launch takes (icgn2d_plan); n for a plain call.  A re-seeded sub-queue passes
// the length of the whole queue, so that its POIs split their sums as they do in the launch over all of them.
int icgn2d_launch(int np, const Image2D& img, float* d_pois, size_t n, int rx, int ry, float conv, float stop, int sm_count,
	size_t smem_optin, int* d_counter, const float* d_center_offsets, const float* lm_damping, cudaStream_t stream, cudaError_t* err,
	size_t plan_n);
size_t icgn2d_slab_bytes(int rx, int ry); // shared memory one POI needs (plain IC-GN, one warp per POI)
// one reference (img.ref) against the frame-major stack img.tar [n_frames][h][w]: n seeds in, n_frames x n records out (frame-major)
int icgn2d_series_launch(int np, const Image2D& img, int n_frames, const float* d_seeds, float* d_out, size_t n, int rx, int ry, float conv, float stop,
	int sm_count, size_t smem_optin, int* d_counter, cudaStream_t stream, cudaError_t* err, size_t plan_n);
// series_reseed.cu: the lost-POI scan, compaction, rebuild and scatter of the re-seeding series calls (dim: 2 or 3; records
// frame-major, out[f * n + i]).  Each returns the launch's CUDA error.
// scan: for the POIs idx[0..m) (0..m when idx is null), first[i] = the first frame in [f_begin, f_end) with !(zncc >= zncc_min), or
// -1; hist[f] += the POIs whose first lost frame is f.
cudaError_t reseed_scan_launch(int dim, const float* d_out, size_t n, int f_begin, int f_end, const int* d_idx, size_t m, float zncc_min, int* d_first,
	int* d_hist, int sm_count, cudaStream_t stream);
// select: idx = the POIs i < n with first[i] == f, in ascending order (stable compaction), *d_count = how many
size_t reseed_select_bytes(size_t n); // temporary storage reseed_select_launch needs
cudaError_t reseed_select_launch(const int* d_first, int f, size_t n, int* d_idx, int* d_count, void* d_temp, size_t temp_bytes, cudaStream_t stream);
// anchor_init: anchor[i] = seed i's translation (dim floats per POI)
cudaError_t reseed_anchor_init_launch(int dim, const float* d_seeds, size_t n, float* d_anchor, int sm_count, cudaStream_t stream);
// rebuild: sub[k] = POI idx[k]'s seed with every field but the position and the subset radii zeroed and the translation set to its
// anchor; when prev (the frame before's records) holds a good record for the POI, its translation becomes the anchor first.
// idx null: the first m POIs; anchor null: zero translation.
cudaError_t reseed_rebuild_launch(int dim, const float* d_seeds, const float* d_prev, const int* d_idx, size_t m, float zncc_min, float* d_anchor,
	float* d_sub, int sm_count, cudaStream_t stream);
// scatter: record k of frame g of src (frames x m records, frame-major) -> out[(f0 + g) * n + idx[k]]
cudaError_t reseed_scatter_launch(int dim, const float* d_src, size_t m, int frames, const int* d_idx, float* d_out, size_t n, int f0, int sm_count,
	cudaStream_t stream);
// nr2d.cu
constexpr int NR2D_TILE_MARGIN = 1;
__host__ __device__ inline int nr2d_tar_w(int rx) { return round_up4(2 * rx + 1 + 3 + 2 * NR2D_TILE_MARGIN + 4 + 3); }
__host__ __device__ inline int nr2d_tar_h(int ry) { return 2 * ry + 1 + 3 + 2 * NR2D_TILE_MARGIN + 4; }
// per-warp slab (floats): [0,32) mbarrier + pad | tile T | gradient tile G (float2) | r~
__host__ __device__ inline int nr2d_warp_floats(int rx, int ry) {
	const int tw = nr2d_tar_w(rx), th = nr2d_tar_h(ry);
	return 32 + round_up32(tw * th) + round_up32(2 * (tw - 4) * (th - 4)) + round_up32((2 * rx + 1) * (2 * ry + 1));
}

// Launch geometry of nr2d1_kernel: CTAs of 4, 2 or 1 one-POI warps, whichever keeps the most warps resident per SM.
struct Nr2dPlan {
	int warps_per_cta;
	int ctas_per_sm;
	size_t smem; // dynamic shared memory per CTA
};

// false when one warp's slab does not fit in shared memory (smem_optin: the device's opt-in limit per block)
inline bool nr2d1_plan(int rx, int ry, size_t smem_optin, Nr2dPlan* p) {
	const size_t per_warp = (size_t)nr2d_warp_floats(rx, ry) * sizeof(float);
	int best_wpb = 0, best_warps = 0;
	for (int wpb = 4; wpb >= 1; wpb >>= 1) {
		const size_t need = per_warp * wpb;
		if (need > smem_optin) continue;
		int blocks = (int)((228 * 1024) / (need + 1024));
		if (blocks > 32) blocks = 32;
		const int warps = blocks * wpb;
		if (warps > best_warps) { best_warps = warps; best_wpb = wpb; }
	}
	if (best_wpb == 0) return false;
	p->warps_per_cta = best_wpb;
	p->ctas_per_sm = best_warps / best_wpb;
	p->smem = per_warp * best_wpb;
	return true;
}
int nr2d1_launch(const Image2D& img, float* d_pois, size_t n, int rx, int ry, float conv, float stop, int sm_count, size_t smem_optin,
	int* d_counter, cudaStream_t stream, cudaError_t* err);
// epipolar.cu
int epipolar_slots(int search_radius, int search_step);
void epipolar_candidates_launch(const float* d_pois, size_t poi0, size_t n_poi, const float* fundamental, const float* parallax_x,
	const float* parallax_y, int search_radius, int search_step, int rx, int ry, int w, int h, int slots, float* d_cand, int sm_count,
	cudaStream_t stream);
void epipolar_select_launch(float* d_pois, size_t poi0, size_t n_poi, int slots, const float* d_cand, int sm_count, cudaStream_t stream);
// strain.cu
size_t strain_workspace_bytes(size_t n);
int strain_launch(int dim, float* d_pois, size_t n, float radius, int k_min, float zncc_threshold, int approximation, long long only, void* workspace,
	int sm_count, cudaStream_t stream, cudaError_t* err, long long* launches);
// FFTCC2D: which of the three kernels a window takes, and what that kernel needs
constexpr int FFTW32_WARPS = 4;     // fftcc2d_w32.cu: one-POI warps per CTA
constexpr int FFTREG_THREADS = 128; // fftcc2d_reg.cu: one thread per window row, 128 / N POIs per CTA
// fftcc2d_reg.cu, window of n x n points: two padded tiles (pitch n + 1) per POI and four partials per thread
__host__ __device__ constexpr size_t fftcc2d_reg_smem_bytes(int n) {
	return ((size_t)2 * (FFTREG_THREADS / n) * n * (n + 1) + 4 * FFTREG_THREADS) * sizeof(float);
}
// true when a register kernel exists for the square window of 2r points
inline bool fftcc2d_reg_supported(int r) {
	switch (2 * r) {
	case 8: case 10: case 12: case 16: case 18: case 20: case 24: case 30: case 36: case 40: case 48: case 50: case 54: case 60: case 64: return true;
	default: return false;
	}
}
// fftcc.cu: two ping-pong windows of complex points, the twiddle tables of both axes, 64 floats of reduction scratch
inline size_t fftcc2d_smem_bytes(int rx, int ry) {
	const size_t M = (size_t)4 * rx * ry;
	return 2 * M * sizeof(float2) + (size_t)(2 * rx + 2 * ry) * sizeof(float2) + 64 * sizeof(float);
}

// W32 is the register-FFT kernel specialised for the 32-point window (r = 16 on both axes), REG the register FFT codelets for
// square windows of N = 2^a 3^b 5^c <= 64 points, GENERIC the shared-memory Stockham kernel for any window whose prime factors
// are <= 31.
enum class Fftcc2dPath { W32, REG, GENERIC };
enum class Fftcc2dReject { NONE, PRIME_FACTOR, SHARED_MEMORY };
struct Fftcc2dPlan {
	Fftcc2dPath path;
	FftAxis ax, ay;       // GENERIC: the Stockham stages of the 2rx- and 2ry-point transforms
	size_t smem;          // dynamic shared memory per CTA (W32: none, its tiles are static)
	int pois_per_cta;     // POIs a CTA carries at a time
	Fftcc2dReject reject; // why the plan is refused (GENERIC only)
};

// false when no kernel takes the (2rx x 2ry) window: a prime factor above 31, or more shared memory than smem_optin (the
// device's opt-in limit per block).  force_generic sends every window to the GENERIC kernel.  rx, ry >= 1.
inline bool fftcc2d_plan(int rx, int ry, bool force_generic, size_t smem_optin, Fftcc2dPlan* p) {
	p->reject = Fftcc2dReject::NONE;
	p->smem = 0;
	p->ax.n = p->ay.n = p->ax.nstage = p->ay.nstage = 0;
	if (!force_generic && rx == 16 && ry == 16) {
		p->path = Fftcc2dPath::W32;
		p->pois_per_cta = FFTW32_WARPS;
		return true;
	}
	if (!force_generic && rx == ry && fftcc2d_reg_supported(rx)) {
		p->path = Fftcc2dPath::REG;
		p->pois_per_cta = FFTREG_THREADS / (2 * rx);
		p->smem = fftcc2d_reg_smem_bytes(2 * rx);
		return true;
	}
	p->path = Fftcc2dPath::GENERIC;
	p->pois_per_cta = 1;
	p->smem = fftcc2d_smem_bytes(rx, ry);
	if (!fft_plan_axis(2 * rx, &p->ax) || !fft_plan_axis(2 * ry, &p->ay)) p->reject = Fftcc2dReject::PRIME_FACTOR;
	else if (p->smem > smem_optin) p->reject = Fftcc2dReject::SHARED_MEMORY;
	return p->reject == Fftcc2dReject::NONE;
}

// fftcc.cu
int fftcc2d_launch(const Image2D& img, float* d_pois, size_t n, int rx, int ry, const Fftcc2dPlan& plan, const float2* tw_x,
	const float2* tw_y, int sm_count, cudaStream_t stream, cudaError_t* err);
// fftcc2d_w32.cu (32x32 window, one warp per POI, register FFT)
int fftcc2d_w32_launch(const Image2D& img, float* d_pois, size_t n, int sm_count, cudaStream_t stream, cudaError_t* err);
// fftcc2d_reg.cu (square windows of 2^a 3^b 5^c <= 64 points, one thread per row, register FFT codelets)
int fftcc2d_reg_launch(const Image2D& img, float* d_pois, size_t n, int r, const Fftcc2dPlan& plan, int sm_count, cudaStream_t stream,
	cudaError_t* err);
// FFTCC3D: which of the three kernels a window takes, and what that kernel needs
constexpr int F3_WARPS = 8;        // fftcc3d_w32.cu: warps of the one-POI CTA
// fftcc3d_w32.cu: resident CTAs per SM (DESIGN.md section 5).  The launch plan sizes the grid with it in ocb_api.cu, so an A/B
// build that overrides it compiles both fftcc3d_w32.cu and ocb_api.cu with the flag.
#ifndef FFTCC3D_W32_CTAS_PER_SM
#define FFTCC3D_W32_CTAS_PER_SM 2
#endif
// fftcc3d_w32.cu: two tiles per warp, each a TMA box (36 x 32 floats) or a padded transpose tile (32 x 33)
constexpr size_t FFTCC3D_W32_SMEM = (size_t)2 * F3_WARPS * 32 * 36 * sizeof(float);
constexpr int F3R_THREADS = 128;   // fftcc3d_reg.cu: one thread per 1D transform, 128 / N z-slices per round
// fftcc3d_reg.cu, window of n^3 points: two padded tiles (pitch n + 1) per slice of a round
__host__ __device__ constexpr size_t fftcc3d_reg_smem_bytes(int n) { return (size_t)2 * (F3R_THREADS / n) * n * (n + 1) * sizeof(float); }
// resident CTAs the register budget of fftcc3d_reg_kernel<N> is sized for
__host__ __device__ constexpr int fft3reg_min_ctas(int n) { return n <= 24 ? 4 : (n <= 48 ? 3 : 2); }
#define OCB_F3R_SIZES(X) X(8) X(10) X(12) X(16) X(18) X(20) X(24) X(30) X(36) X(40) X(48) X(50) X(54) X(60) X(64)
// true when a register kernel exists for the cubic window of 2r points
inline bool fftcc3d_reg_supported(int r) {
	switch (2 * r) {
#define X(n) case n:
		OCB_F3R_SIZES(X)
#undef X
		return true;
	default: return false;
	}
}
// fftcc.cu: two ping-pong buffers (a slice or a (ky, -ky) row pair of z-x planes), the twiddle tables of the three axes, 64
// floats of reduction scratch
inline size_t fftcc3d_smem_bytes(int rx, int ry, int rz) {
	const size_t slice = (size_t)4 * rx * ry, rowpair = (size_t)2 * (2 * rz) * (2 * rx);
	const size_t nbuf = slice > rowpair ? slice : rowpair;
	return 2 * nbuf * sizeof(float2) + (size_t)(2 * rx + 2 * ry + 2 * rz) * sizeof(float2) + 64 * sizeof(float);
}

// W32 is the register-FFT kernel specialised for the 32^3 window (r = 16 on every axis), REG the register FFT codelets for cubic
// windows of N = 2^a 3^b 5^c <= 64 points, GENERIC the shared-memory Stockham kernel for any window whose prime factors are <= 31.
// Every kernel runs one POI per CTA at a time in a persistent grid, with a scratch volume per CTA in global memory.
enum class Fftcc3dPath { W32, REG, GENERIC };
enum class Fftcc3dReject { NONE, PRIME_FACTOR, SHARED_MEMORY };
struct Fftcc3dPlan {
	Fftcc3dPath path;
	int n;                // REG: points per axis, N = 2r
	int slices_per_round; // REG: z-slices transformed at once, G = 128 / N
	int idle_threads;     // REG: threads without a slice, 128 - G N
	FftAxis ax, ay, az;   // GENERIC: the Stockham stages of the 2rx-, 2ry- and 2rz-point transforms
	size_t smem;          // dynamic shared memory per CTA
	int ctas;             // CTAs of a full launch (a queue of n POIs launches min(n, ctas))
	size_t cta_scratch;   // float2 scratch elements per CTA
	Fftcc3dReject reject; // why the plan is refused (GENERIC only)
};

// false when no kernel takes the (2rx x 2ry x 2rz) window: a prime factor above 31, or more shared memory than smem_optin (the
// device's opt-in limit per block).  force_generic sends every window to the GENERIC kernel.  rx, ry, rz >= 1.
inline bool fftcc3d_plan(int rx, int ry, int rz, bool force_generic, size_t smem_optin, int sm_count, Fftcc3dPlan* p) {
	p->reject = Fftcc3dReject::NONE;
	p->n = p->slices_per_round = p->idle_threads = 0;
	p->ax.n = p->ay.n = p->az.n = p->ax.nstage = p->ay.nstage = p->az.nstage = 0;
	if (!force_generic && rx == 16 && ry == 16 && rz == 16) {
		p->path = Fftcc3dPath::W32;
		p->smem = FFTCC3D_W32_SMEM;
		p->ctas = sm_count * FFTCC3D_W32_CTAS_PER_SM;
		p->cta_scratch = (size_t)32 * 32 * 32;
		return true;
	}
	if (!force_generic && rx == ry && ry == rz && fftcc3d_reg_supported(rx)) {
		const int N = 2 * rx;
		p->path = Fftcc3dPath::REG;
		p->n = N;
		p->slices_per_round = F3R_THREADS / N;
		p->idle_threads = F3R_THREADS - p->slices_per_round * N;
		p->smem = fftcc3d_reg_smem_bytes(N);
		int per_sm = (int)((228 * 1024) / (p->smem + 2048));
		if (per_sm > fft3reg_min_ctas(N)) per_sm = fft3reg_min_ctas(N);
		if (per_sm < 1) per_sm = 1;
		p->ctas = sm_count * per_sm;
		p->cta_scratch = (size_t)2 * N * N * N; // two scratch volumes of N^3 complex
		return true;
	}
	p->path = Fftcc3dPath::GENERIC;
	p->smem = fftcc3d_smem_bytes(rx, ry, rz);
	int per_sm = (int)((228 * 1024) / (p->smem + 1024));
	if (per_sm > 2) per_sm = 2;
	if (per_sm < 1) per_sm = 1;
	p->ctas = sm_count * per_sm;
	p->cta_scratch = (size_t)8 * rx * ry * rz;
	if (!fft_plan_axis(2 * rx, &p->ax) || !fft_plan_axis(2 * ry, &p->ay) || !fft_plan_axis(2 * rz, &p->az)) p->reject = Fftcc3dReject::PRIME_FACTOR;
	else if (p->smem > smem_optin) p->reject = Fftcc3dReject::SHARED_MEMORY;
	return p->reject == Fftcc3dReject::NONE;
}

// fftcc3d_reg.cu (cubic windows of 2^a 3^b 5^c <= 64 points, one thread per 1D transform, register FFT codelets)
int fftcc3d_reg_launch(const Image3D& img, float* d_pois, size_t n_poi, const Fftcc3dPlan& plan, float2* scratch, int grid, cudaStream_t stream,
	cudaError_t* err);
// fftcc.cu
int fftcc3d_launch(const Image3D& img, float* d_pois, size_t n, int rx, int ry, int rz, const Fftcc3dPlan& plan, const float2* tw_x,
	const float2* tw_y, const float2* tw_z, float2* scratch, int grid, cudaStream_t stream, cudaError_t* err);
// fftcc3d_w32.cu (32^3 window, register FFTs)
int fftcc3d_w32_launch(const Image3D& img, float* d_pois, size_t n, const Fftcc3dPlan& plan, float2* scratch, int grid, cudaStream_t stream,
	cudaError_t* err);
// icgn3d.cu
constexpr int ICGN3D_MAX_WARPS = 16; // CTAs run 8 warps (two CTAs per SM) or, when only one slab-carrying CTA fits, 16
constexpr int NP3 = 12;
constexpr int NH3 = NP3 * (NP3 + 1) / 2;  // 78
constexpr int NSETUP = NH3 + 2 * NP3 + 2; // Hessian + S + SR + r1 + r2 = 104
constexpr int ICGN3D_TILE_MARGIN = 1;

// static shared memory of icgn3d1_kernel
struct Icgn3dShared {
	float part[ICGN3D_MAX_WARPS][NSETUP]; // per-warp partial sums
	float tot[NSETUP];
	float L[NH3];   // packed Cholesky factor (diag = 1/L_ii)
	float S[NP3], SF[NP3];
	float A[12];    // running warp rows: [1+ux uy uz u | vx 1+vy vz v | wx wy 1+wz w]
	float f2, rbar, c0;
	float dp_norm, zncc;
	int keep_going;
	int poi;
};

// What icgn3d1_kernel does with a POI's setup pass (the reference-only state: Cholesky factor L, S, SF, rbar, f2, c0).
// COMPUTE: build it, then iterate (pair calls).  STORE: build it and write it to a per-POI device cache, records untouched.
// LOAD: restore it from the cache bit for bit, then iterate (volume series, every frame).
enum Icgn3dSetup { ICGN3D_SETUP_COMPUTE = 0, ICGN3D_SETUP_STORE = 1, ICGN3D_SETUP_LOAD = 2 };
constexpr int ICGN3D_SETUP_FLOATS = NH3 + 2 * NP3 + 3; // cached floats per POI: L, S, SF, rbar, f2, c0 (105, 420 B)

// extents of the staged B-spline coefficient tile: x padded to a multiple of 4 floats (16-byte TMA rows)
__host__ __device__ inline int icgn3d_tile_x(int rx) { return (2 * rx + 1 + 3 + 2 * ICGN3D_TILE_MARGIN + 3 + 3) & ~3; }
__host__ __device__ inline int icgn3d_tile_y(int ry) { return 2 * ry + 1 + 3 + 2 * ICGN3D_TILE_MARGIN; }
__host__ __device__ inline int icgn3d_tile_z(int slab_k) { return slab_k + 3 + 2 * ICGN3D_TILE_MARGIN; }

// Launch geometry of icgn3d1_kernel for a subvolume of radii (rx, ry, rz): the (2rz+1) layers are processed in nslab z-slabs of
// slab_k layers (the last one may be thinner), each staged as one tile of icgn3d_tile_z(slab_k) layers in dynamic shared memory.
struct Icgn3dPlan {
	int ctas_per_sm; // 2 (256 threads each) or 1 (512 threads)
	int threads;
	int rc;          // radius baked into the kernel (16 or 30), 0 for the generic kernel
	int slab_k;
	int nslab;       // slabs per iteration: ceil((2rz+1) / slab_k)
	size_t smem;     // dynamic shared memory per CTA
};

// false when even a one-layer slab does not fit in shared memory (smem_optin: the device's opt-in limit per block)
inline bool icgn3d1_plan(int rx, int ry, int rz, size_t smem_optin, Icgn3dPlan* p) {
	const int sz = 2 * rz + 1;
	const size_t layer = (size_t)icgn3d_tile_x(rx) * icgn3d_tile_y(ry) * sizeof(float);
	const size_t fixed = 128 + sizeof(Icgn3dShared) + 1024; // barrier pad + static smem + per-CTA reservation
	const int halo = 3 + 2 * ICGN3D_TILE_MARGIN;
	// prefer two CTAs per SM (one loads while the other computes) when that leaves slabs of >= 6 layers
	int ctas = 2;
	long long k = (long long)(((228 * 1024) / 2 - fixed) / layer) - halo;
	if (k < 6 && k < sz) {
		ctas = 1;
		const size_t budget = smem_optin < (size_t)(227 * 1024) ? smem_optin : (size_t)(227 * 1024);
		k = (long long)((budget - 128 - sizeof(Icgn3dShared)) / layer) - halo;
	}
	if (k < 1) return false;
	if (k > sz) k = sz;
	p->ctas_per_sm = ctas;
	p->threads = ctas == 1 ? 512 : 256;
	const int nslab = (int)((sz + k - 1) / k);
	p->slab_k = (sz + nslab - 1) / nslab; // even out the slabs
	p->nslab = (sz + p->slab_k - 1) / p->slab_k;
	p->smem = 128 + layer * icgn3d_tile_z(p->slab_k);
	if (ctas == 1) p->rc = (rx == 30 && ry == 30 && rz == 30) ? 30 : 0; // 61^3: the reference's own DVC example
	else p->rc = (rx == 16 && ry == 16 && rz == 16) ? 16 : 0;
	return true;
}

// stereo.cu (intrinsics: the 13 floats of CameraIntrinsics, fx fy fs cx cy k1..k6 p1 p2; maps row-major [height][width])
struct StereoCam {
	const float* map_x;
	const float* map_y;
	int height, width;
	const float* intrinsics; // host pointer, 13 floats
	const float* projection; // host pointer, 3x4 row-major
};
void calib_map_launch(const float* intrinsics, int height, int width, float convergence, int iteration, float* d_map_x, float* d_map_y,
	cudaStream_t stream);
void calib_undistort_launch(const float* d_map_x, const float* d_map_y, int height, int width, const float* intrinsics, float* d_pts, float* d_out,
	size_t n, cudaStream_t stream);
void stereo_reconstruct_launch(const StereoCam& c1, const StereoCam& c2, float* d_pts1, float* d_pts2, float* d_pts3d, size_t n,
	cudaStream_t stream);
// the POI2DS records of a stereo series (ocb_stereo_series): n_frames x n, frame-major, from the r1 -> r2 records d_stereo (n), the
// view-1 seeds (n, for x and y) and the two registrations d_out1, d_out2 (n_frames x n POI2D each)
void stereo_poi2ds_launch(const StereoCam& c1, const StereoCam& c2, const float* d_stereo, const float* d_seeds1, const float* d_out1,
	const float* d_out2, float* d_out2ds, size_t n, int n_frames, cudaStream_t stream);

void gradient3d_launch(const float* ref, float4* rg, int dx, int dy, int dz, int sm_count, cudaStream_t s);
void prefilter3d_launch(const float* in, float* out, int dx, int dy, int dz, int axis, int sm_count, cudaStream_t s);
// setup: an Icgn3dSetup; STORE and LOAD need setup_cache, n x ICGN3D_SETUP_FLOATS floats indexed by queue position
int icgn3d1_launch(const Image3D& img, float* d_pois, size_t n, int rx, int ry, int rz, float conv, float stop, int sm_count, size_t smem_optin,
	int* d_counter, cudaStream_t stream, cudaError_t* err, int setup = ICGN3D_SETUP_COMPUTE, float* setup_cache = nullptr);

} // namespace ocb
