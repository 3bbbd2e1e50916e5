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

int icgn2d_launch(int np, const Image2D& img, float* d_pois, size_t n, int rx, int ry, float conv, float stop, int sm_count,
	size_t smem_optin, int* d_counter, const float* d_center_offsets, const float* lm_damping, cudaStream_t stream, cudaError_t* err);
size_t icgn2d_slab_bytes(int rx, int ry); // shared memory one POI needs (plain IC-GN, one warp per POI)
// one reference (img.ref) against the frame-major stack img.tar [n_frames][h][w]: n seeds in, n_frames x n records out (frame-major)
int icgn2d_series_launch(int np, const Image2D& img, int n_frames, const float* d_seeds, float* d_out, size_t n, int rx, int ry, float conv, float stop,
	int sm_count, size_t smem_optin, int* d_counter, cudaStream_t stream, cudaError_t* err);
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
// fftcc3d_reg.cu (cubic windows of 2^a 3^b 5^c <= 64 points, one thread per 1D transform, register FFT codelets)
bool fftcc3d_reg_supported(int r);
int fftcc3d_reg_grid(int r, int sm_count);
int fftcc3d_reg_launch(const Image3D& img, float* d_pois, size_t n_poi, int r, float2* scratch, int grid, cudaStream_t stream, cudaError_t* err);
size_t fftcc3d_smem_bytes(int rx, int ry, int rz);
int fftcc3d_grid(int rx, int ry, int rz, int sm_count);
int fftcc3d_launch(const Image3D& img, float* d_pois, size_t n, int rx, int ry, int rz, const FftAxis& ax, const FftAxis& ay,
	const FftAxis& az, const float2* tw_x, const float2* tw_y, const float2* tw_z, float2* scratch, int grid, cudaStream_t stream,
	cudaError_t* err);
// fftcc3d_w32.cu (32^3 window, register FFTs)
int fftcc3d_w32_grid(int sm_count);
int fftcc3d_w32_launch(const Image3D& img, float* d_pois, size_t n, float2* scratch, int grid, cudaStream_t stream, cudaError_t* err);
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

void gradient3d_launch(const float* ref, float4* rg, int dx, int dy, int dz, int sm_count, cudaStream_t s);
void prefilter3d_launch(const float* in, float* out, int dx, int dy, int dz, int axis, int sm_count, cudaStream_t s);
int icgn3d1_launch(const Image3D& img, float* d_pois, size_t n, int rx, int ry, int rz, float conv, float stop, int sm_count, size_t smem_optin,
	int* d_counter, cudaStream_t stream, cudaError_t* err);

} // namespace ocb
