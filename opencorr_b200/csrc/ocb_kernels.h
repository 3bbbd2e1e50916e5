// ocb_kernels.h -- host-visible launch interfaces of the sm_90a kernels (internal to the library).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <string.h>

#include <vector>

#include "ocb_common.cuh"
#include "ocb_tma.cuh"
#include "sift3d_common.h"

namespace ocb {

// Every *_launch below enqueues its kernels on `stream` and returns the first CUDA error among its attribute set, work-counter
// reset, copies and launches, or cudaSuccess.  It runs the plan it is given: whether a call is supported is decided by the
// caller, which makes the plan (ocb_api.cu, *_plan_or_error).

// kern<<<grid, block, smem, stream>>>(args...) with smem bytes of dynamic shared memory allowed first (beyond the default 48 KB)
template <class K, class... A>
inline cudaError_t launch_smem(K kern, int grid, int block, size_t smem, cudaStream_t stream, A... args) {
	const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (e != cudaSuccess) return e;
	kern<<<grid, block, smem, stream>>>(args...);
	return cudaGetLastError();
}

// the kernel just enqueued: its launch error, or cudaSuccess and one more launch counted
inline cudaError_t launched(long long* launches) {
	const cudaError_t e = cudaGetLastError();
	if (e == cudaSuccess) ++*launches;
	return e;
}

// Grow-only device buffer (see grow).  Released when its owner is deleted, with the owner's device current.
struct DevBuf {
	void* p = nullptr;
	size_t bytes = 0;
	DevBuf() = default;
	DevBuf(const DevBuf&) = delete;
	DevBuf& operator=(const DevBuf&) = delete;
	~DevBuf() {
		if (p) cudaFree(p);
	}
	template <class T> T* as() const { return (T*)p; }
};

// Make b hold at least `bytes` on the current device; it only grows.  The stream is drained before the old allocation is freed.
// keep_bytes = 0: the old allocation is freed first and exactly `bytes` are allocated (on failure b is left empty).  keep_bytes > 0:
// its first keep_bytes are copied into an allocation of at least twice the capacity (on failure b is left as it was).  A failed
// allocation or copy is cleared from the runtime's last error, which the next launch's check would otherwise report.
inline cudaError_t grow(DevBuf& b, size_t bytes, cudaStream_t stream, size_t keep_bytes = 0) {
	if (bytes <= b.bytes) return cudaSuccess;
	cudaError_t e;
	if (keep_bytes == 0 && b.p) {
		if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
		cudaFree(b.p);
		b.p = nullptr;
		b.bytes = 0;
	}
	if (keep_bytes && bytes < 2 * b.bytes) bytes = 2 * b.bytes;
	void* q = nullptr;
	if ((e = cudaMalloc(&q, bytes)) != cudaSuccess) {
		cudaGetLastError();
		return e;
	}
	if (b.p) {
		if ((e = cudaMemcpyAsync(q, b.p, keep_bytes, cudaMemcpyDeviceToDevice, stream)) != cudaSuccess
			|| (e = cudaStreamSynchronize(stream)) != cudaSuccess) {
			cudaGetLastError();
			cudaFree(q);
			return e;
		}
		cudaFree(b.p);
	}
	b.p = q;
	b.bytes = bytes;
	return cudaSuccess;
}

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

// sift3d.cu: SIFT3D feature extraction and matching
constexpr int SIFT3D_MAX_R = 64; // largest blur radius per axis (8 at the default settings, x2 per doubling of unit anisotropy)
constexpr int SIFT3D_MAX_L = 16; // largest n_octave_layers + 3
struct BlurW {
	float w[SIFT3D_MAX_R + 1];
};
// One Gaussian layer: its scale, and the blur that makes it from the layer below (s3::blur_kernels: sigma, radii, half kernels)
struct Sift3dLayer {
	float scale, sigma;
	int radius[3];
	BlurW w[3];
};
struct Sift3dOctave {
	int nx, ny, nz;
	float unit[3];
};
enum class Sift3dReject { NONE, OCTAVE_LAYERS, VOLUME_SIZE, BLUR_RADIUS };
// The Gaussian pyramid of createGaussianPyramid (src/oc_sift.cpp:676-739): layer l of octave o is entry o * L + l.
struct Sift3dPlan {
	int n_octave;
	int L;     // Gaussian layers per octave: n_octave_layers + 3
	float kappa; // scale ratio of neighbouring layers
	std::vector<Sift3dOctave> octave;
	std::vector<Sift3dLayer> layer; // no blur for layer 0 of octave o > 0, which is downsampled from octave o - 1
	Sift3dReject reject;          // why the plan is refused
};

// false, with the failed check in p->reject, when n_octave_layers is outside [1, SIFT3D_MAX_L - 3], n_octave_layers times the
// voxel count exceeds 2^62 (the candidates' 64-bit index), or a blur radius exceeds SIFT3D_MAX_R voxels.  cfg: the
// s3::CFG_FIELDS floats of the C ABI; unit: the voxel size.
inline bool sift3d_plan(int nx, int ny, int nz, const float* cfg, const float* unit, Sift3dPlan* p) {
	const int nol = (int)cfg[s3::CFG_N_OCTAVE_LAYERS], L = nol + 3;
	p->L = L;
	p->reject = Sift3dReject::OCTAVE_LAYERS;
	if (nol < 1 || L > SIFT3D_MAX_L) return false;
	p->reject = Sift3dReject::VOLUME_SIZE;
	if ((size_t)nol * ((size_t)nx * ny * nz) > (size_t)1 << 62) return false;
	p->reject = Sift3dReject::BLUR_RADIUS; // the check left, made layer by layer below
	const int dim_min = nx < ny ? (nx < nz ? nx : nz) : (ny < nz ? ny : nz);
	const int n_octave = s3::octave_count(dim_min, (int)cfg[s3::CFG_MIN_DIMENSION]);
	const float kappa = s3::kappa_of(nol);
	p->n_octave = n_octave;
	p->kappa = kappa;
	p->octave.assign(n_octave, Sift3dOctave{ nx, ny, nz, { unit[0], unit[1], unit[2] } });
	p->layer.assign((size_t)n_octave * L, Sift3dLayer{});
	for (int i = 0; i < n_octave * L; i++) {
		const int o = i / L, l = i % L;
		Sift3dLayer& b = p->layer[i];
		if (i == 0) {
			b.scale = 1.f / kappa * cfg[s3::CFG_SIGMA_BASE];
			b.sigma = sqrtf(b.scale * b.scale - cfg[s3::CFG_SIGMA_SOURCE] * cfg[s3::CFG_SIGMA_SOURCE]);
		} else if (l == 0) {
			const Sift3dOctave& u = p->octave[o - 1];
			p->octave[o] = Sift3dOctave{ u.nx / 2, u.ny / 2, u.nz / 2, { u.unit[0] * 2, u.unit[1] * 2, u.unit[2] * 2 } };
			b.scale = p->layer[(o - 1) * L + nol].scale;
			continue;
		} else {
			b.scale = kappa * p->layer[i - 1].scale;
			b.sigma = sqrtf(kappa * kappa - 1.f) * p->layer[l - 1].scale;
		}
		float w[3 * (SIFT3D_MAX_R + 1)] = {};
		if (!s3::blur_kernels(b.sigma, p->octave[o].unit, SIFT3D_MAX_R, b.radius, w)) return false;
		for (int a = 0; a < 3; a++) memcpy(b.w[a].w, w + a * (SIFT3D_MAX_R + 1), sizeof(BlurW));
	}
	p->reject = Sift3dReject::NONE;
	return true;
}

// One image's products of the last ocb_sift3d call, on the device
struct Sift3dImage {
	size_t n_cand = 0, n_kp = 0;
	DevBuf cand; // 5 ints per candidate
	DevBuf kp;   // s3::KP_FLOATS floats per keypoint
	DevBuf desc; // s3::DESC floats per keypoint
	std::vector<float> max_abs;
};

enum { SIFT3D_STAGES = 10 }; // ref: pyramid, extrema, orientation, descriptors; tar: the same four; matching; host post-pass
// The products of the last ocb_sift3d call and the working buffers that made them
struct Sift3d {
	Sift3dImage img[2];
	std::vector<float> ref_xyz, tar_xyz; // the matched keypoints' coor_img, 3 floats each
	float stage_ms[SIFT3D_STAGES] = {};
	DevBuf layers, tmp, kp_tmp, top2, part, sel, keep, kept_idx, counters, cub_ws;
	cudaEvent_t ev[2 * SIFT3D_STAGES] = {}; // start and end of each timed stage
	~Sift3d() {
		for (cudaEvent_t e : ev)
			if (e) cudaEventDestroy(e);
	}
};

// sift3d_run's result when an image has more than 2^31 - 1 keypoints, which the matching kernels cannot index
constexpr cudaError_t SIFT3D_TOO_MANY_KEYPOINTS = static_cast<cudaError_t>(cudaErrorUnknown + 1);
// Both images' pyramids, keypoints and descriptors as `plan` (sift3d_plan of their size) schedules them, then the matches.
// *launches grows by each kernel once it has launched (a cub selection counts as one).
cudaError_t sift3d_run(Sift3d* s, const Sift3dPlan& plan, const float* d_ref, const float* d_tar, const float* cfg, float ratio, int sm_count,
	cudaStream_t stream, long long* launches);
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

// plan: icgn2d_plan for the call's order, radii and IC-LM flag (lm_damping non-null), its grid at most n.  d_counter: the context's
// work-queue heads (64 ints; see ocb_create).
cudaError_t icgn2d_launch(int np, const Icgn2dPlan& plan, const Image2D& img, float* d_pois, size_t n, int rx, int ry, float conv, float stop,
	int* d_counter, const float* d_center_offsets, const float* lm_damping, cudaStream_t stream);
// one reference (img.ref) against the frame-major stack img.tar [n_frames][h][w]: n seeds in, n_frames x n records out (frame-major);
// lm_damping as for icgn2d_launch
cudaError_t icgn2d_series_launch(int np, const Icgn2dPlan& plan, const Image2D& img, int n_frames, const float* d_seeds, float* d_out, size_t n,
	int rx, int ry, float conv, float stop, int* d_counter, const float* lm_damping, cudaStream_t stream);
// series_reseed.cu: the lost-POI scan, compaction, rebuild and scatter of the re-seeding series calls (dim: 2 or 3; records
// frame-major, out[f * n + i]).
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
// region_recover.cu: the selections and record moves of the recovery calls (dim: 2 or 3, POI2D or POI3D records).
// The tests of a record with ZNCC z and convergence c: UNRELIABLE z < zncc_low || c > conv; RELIABLE not UNRELIABLE and
// z >= zncc_high; ACCEPTED z >= zncc_high && c <= conv; KEPT not ACCEPTED.
enum class RecoverTest { UNRELIABLE, RELIABLE, ACCEPTED, KEPT };
// select: idx = the positions i < count whose record d_rec[i] passes `test`, ascending; *d_count = how many
size_t recover_select_bytes(size_t n); // temporary storage recover_select_launch needs for count <= n
cudaError_t recover_select_launch(int dim, const float* d_rec, size_t count, RecoverTest test, float zncc_high, float zncc_low, float conv, int* d_idx,
	int* d_count, void* d_temp, size_t temp_bytes, cudaStream_t stream);
// move: total = *d_count1 + the length of list 2.  Record k < *d_count1 is src[list1[k]]: it goes to dst1[k] and, with d_q set, to
// d_q[src_idx[list1[k]]].  Record k2 of list 2 is src[list2[k2]]: it goes to dst2[k2], its queue index (src_idx[list2[k2]], or
// list2[k2] when src_idx is null) to idx2[k2].
cudaError_t recover_move_launch(int dim, const float* d_src, const int* d_src_idx, size_t total, const int* d_list1, const int* d_count1, float* d_dst1,
	float* d_q, const int* d_list2, float* d_dst2, int* d_idx2, int sm_count, cudaStream_t stream);
// collect (the series recovery calls): d_out[k] = d_src_idx[d_list1[k]] for k < *d_count1 (<= total), the queue indices of a round's
// accepted POIs in the order the move appends their records to the reliable set
cudaError_t recover_collect_launch(const int* d_src_idx, size_t total, const int* d_list1, const int* d_count1, int* d_out, int sm_count,
	cudaStream_t stream);
// scan (the series recovery calls): as reseed_scan_launch, with the UNRELIABLE test (zncc_low, conv) in place of the lost test:
// first[i] = the first frame in [f_begin, f_end) whose record of POI i is UNRELIABLE, or -1; hist[f] += the POIs whose first such
// frame is f.  reseed_select_launch compacts its result.
cudaError_t recover_scan_launch(int dim, const float* d_out, size_t n, int f_begin, int f_end, const int* d_idx, size_t m, float zncc_low, float conv,
	int* d_first, int* d_hist, int sm_count, cudaStream_t stream);
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
cudaError_t nr2d1_launch(const Nr2dPlan& plan, const Image2D& img, float* d_pois, size_t n, int rx, int ry, float conv, float stop, int sm_count,
	int* d_counter, cudaStream_t stream);
// one reference (img.ref) against the frame-major stack img.tar [n_frames][h][w]: n seeds in, n_frames x n records out (frame-major)
cudaError_t nr2d1_series_launch(const Nr2dPlan& plan, const Image2D& img, int n_frames, const float* d_seeds, float* d_out, size_t n, int rx, int ry,
	float conv, float stop, int sm_count, int* d_counter, cudaStream_t stream);
// epipolar.cu
int epipolar_slots(int search_radius, int search_step);
cudaError_t epipolar_candidates_launch(const float* d_pois, size_t poi0, size_t n_poi, const float* fundamental, const float* parallax_x,
	const float* parallax_y, int search_radius, int search_step, int rx, int ry, int w, int h, int slots, float* d_cand, int sm_count,
	cudaStream_t stream);
cudaError_t epipolar_select_launch(float* d_pois, size_t poi0, size_t n_poi, int slots, const float* d_cand, int sm_count, cudaStream_t stream);
// strain.cu: Strain over a queue of POI2D, POI3D or POI2DS (stereo DIC) records
enum class PoiKind { POI2D, POI3D, POI2DS };
__host__ __device__ constexpr int poi_floats(PoiKind k) { return k == PoiKind::POI2D ? (int)P2_N : (k == PoiKind::POI3D ? (int)P3_N : (int)P2DS_N); }

// The uniform grid the POIs are binned into: a position p lies in cell c_d = floor((p_d - lo_d) * inv_cell), clamped to
// [0, nc_d), of key (c_2 nc_1 + c_1) nc_0 + c_0; a POI with a non-finite position takes the key n_cells.
struct StrainGrid {
	float lo[3];
	float inv_cell;
	int nc[3];
	unsigned int n_cells;
};

// The grid over the bounding box [lo, hi] of the finite positions (axes d < dims) for the neighbour radius `radius`; returns
// the cell edge.  The edge is >= |radius|, so that the 3^D block around a POI's cell holds every point within the radius (the
// test is dist^2 < radius^2, so a negative radius acts as its magnitude); a non-finite radius takes one cell over the bbox
// (+-inf: every POI is a neighbour, NaN: none is).  The edge doubles until the grid has < 2^30 cells.
inline double strain_grid_plan(int dims, const float* lo, const float* hi, float radius, StrainGrid* g) {
	float extent = 0.f;
	for (int d = 0; d < 3; d++) {
		g->lo[d] = d < dims ? lo[d] : 0.f;
		const float h = d < dims ? hi[d] : 0.f;
		if (h - g->lo[d] > extent) extent = h - g->lo[d];
	}
	const float abs_radius = fabsf(radius);
	double cell = !isfinite(abs_radius) ? (double)extent + 1.0 : abs_radius > 0.f ? (double)abs_radius : (double)extent / 64.0 + 1.0;
	if (!(cell > 0.0) || !isfinite(cell)) cell = 1.0;
	while (true) {
		double total = 1.0;
		for (int d = 0; d < 3; d++) {
			const double cnt = d < dims ? floor(((double)hi[d] - (double)g->lo[d]) / cell) + 2.0 : 1.0;
			g->nc[d] = (int)(cnt < 1.0 ? 1.0 : (cnt > 2e9 ? 2e9 : cnt));
			total *= cnt;
		}
		if (total < 1073741824.0) break;
		cell *= 2.0;
	}
	g->inv_cell = (float)(1.0 / cell);
	// the float product (p - lo) * inv_cell may round a point's cell index by one; the neighbourhood scan needs
	// |cell(p) - cell(q)| <= 1 for every pair within the radius, which holds with a 0.1 % safety margin on the edge
	g->inv_cell *= 0.999f;
	g->n_cells = (unsigned int)g->nc[0] * (unsigned int)g->nc[1] * (unsigned int)g->nc[2];
	return cell;
}

// the workspace of a call over n_frames frames of n POIs (the pair call: one frame)
size_t strain_workspace_bytes(size_t n, size_t n_frames = 1);
// *launches grows by each kernel once it has launched (the radix sort counts as one)
cudaError_t strain_launch(PoiKind kind, float* d_pois, size_t n, float radius, int k_min, float zncc_threshold, int approximation, long long only,
	void* workspace, int sm_count, cudaStream_t stream, long long* launches);
// Strain over n_frames frames of n records each, frame-major, whose search coordinates are the same in every frame: frame f's records
// become those strain_launch leaves on them, with one readback and the same launches for any n_frames.  When some frame's
// search coordinates differ from frame 0's as bits, *moved is set and nothing is written.
cudaError_t strain_series_launch(PoiKind kind, float* d_pois, size_t n_frames, size_t n, float radius, int k_min, float zncc_threshold,
	int approximation, void* workspace, int sm_count, cudaStream_t stream, long long* launches, bool* moved);
// RegionFit2D / RegionFit3D (kind POI2D or POI3D): every queue POI with a finite position and at least k_min neighbours among the
// n_reliable reliable records (Strain's search over them, no ZNCC filter) takes the plane fit's intercept and slopes as its
// first-order deformation, with zncc 0.  Workspace: strain_workspace_bytes(n_reliable); one readback and five launches per call.
cudaError_t region_fit_launch(PoiKind kind, const float* d_reliable, size_t n_reliable, float* d_queue, size_t n, float radius, int k_min,
	void* workspace, int sm_count, cudaStream_t stream, long long* launches);
// FFTCC2D: which of the three kernels a window takes, and what that kernel needs
constexpr int FFTW32_WARPS = 4;     // fftcc2d_w32.cu: one-POI warps per CTA
constexpr int FFTREG_THREADS = 128; // fftcc2d_reg.cu: one thread per window row, 128 / N POIs per CTA
// fftcc2d_reg.cu, window of n x n points: two padded tiles (pitch n + 1) per POI and four partials per thread
__host__ __device__ constexpr size_t fftcc2d_reg_smem_bytes(int n) {
	return ((size_t)2 * (FFTREG_THREADS / n) * n * (n + 1) + 4 * FFTREG_THREADS) * sizeof(float);
}
// Window sizes N (points per axis) that fftcc2d_reg.cu and fftcc3d_reg.cu instantiate (fft_codelet.cuh: N = 2^a 3^b 5^c <= 64;
// N = 32 goes to the W32 kernels)
#define OCB_FFT_REG_SIZES(X) X(8) X(10) X(12) X(16) X(18) X(20) X(24) X(30) X(36) X(40) X(48) X(50) X(54) X(60) X(64)
// true when a register kernel exists for windows of 2r points per axis
inline bool fft_reg_supported(int r) {
	switch (2 * r) {
#define X(n) case n:
		OCB_FFT_REG_SIZES(X)
#undef X
		return true;
	default: return false;
	}
}
// resident CTAs the register budget of fftcc2d_reg_kernel<N> and fftcc3d_reg_kernel<N> is sized for (2 N floats of transform data
// per thread + temporaries)
__host__ __device__ constexpr int fft_reg_min_ctas(int n) { return n <= 24 ? 4 : (n <= 48 ? 3 : 2); }

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
	int ctas_per_sm;      // CTAs per SM of a full launch: a queue of n POIs launches min(ceil(n / pois_per_cta), SMs x ctas_per_sm)
	Fftcc2dReject reject; // why the plan is refused (GENERIC only)
};

// resident CTAs per SM that smem bytes of shared memory per CTA allow (228 KB per SM, 1 KB of it reserved per CTA), between 1 and cap
inline int fftcc_ctas_per_sm(size_t smem, int cap) {
	const int k = (int)((228 * 1024) / (smem + 1024));
	return k > cap ? cap : (k < 1 ? 1 : k);
}

// false when no kernel takes the (2rx x 2ry) window: a prime factor above 31, or more shared memory than smem_optin (the
// device's opt-in limit per block).  force_generic sends every window to the GENERIC kernel.  rx, ry >= 1.
inline bool fftcc2d_plan(int rx, int ry, bool force_generic, size_t smem_optin, Fftcc2dPlan* p) {
	p->reject = Fftcc2dReject::NONE;
	p->smem = 0;
	p->ax.n = p->ay.n = p->ax.nstage = p->ay.nstage = 0;
	if (!force_generic && rx == 16 && ry == 16) {
		p->path = Fftcc2dPath::W32;
		p->pois_per_cta = FFTW32_WARPS;
		p->ctas_per_sm = 16;
		return true;
	}
	if (!force_generic && rx == ry && fft_reg_supported(rx)) {
		p->path = Fftcc2dPath::REG;
		p->pois_per_cta = FFTREG_THREADS / (2 * rx);
		p->smem = fftcc2d_reg_smem_bytes(2 * rx);
		p->ctas_per_sm = fftcc_ctas_per_sm(p->smem, 8);
		return true;
	}
	p->path = Fftcc2dPath::GENERIC;
	p->pois_per_cta = 1;
	p->smem = fftcc2d_smem_bytes(rx, ry);
	p->ctas_per_sm = fftcc_ctas_per_sm(p->smem, 16) * 2;
	if (!fft_plan_axis(2 * rx, &p->ax) || !fft_plan_axis(2 * ry, &p->ay)) p->reject = Fftcc2dReject::PRIME_FACTOR;
	else if (p->smem > smem_optin) p->reject = Fftcc2dReject::SHARED_MEMORY;
	return p->reject == Fftcc2dReject::NONE;
}

// fftcc.cu
cudaError_t fftcc2d_launch(const Image2D& img, float* d_pois, size_t n, int rx, int ry, const Fftcc2dPlan& plan, const float2* tw_x,
	const float2* tw_y, int grid, cudaStream_t stream);
// fftcc2d_w32.cu (32x32 window, one warp per POI, register FFT)
cudaError_t fftcc2d_w32_launch(const Image2D& img, float* d_pois, size_t n, int grid, cudaStream_t stream);
// fftcc2d_reg.cu (square windows of 2^a 3^b 5^c <= 64 points, one thread per row, register FFT codelets)
cudaError_t fftcc2d_reg_launch(const Image2D& img, float* d_pois, size_t n, int r, const Fftcc2dPlan& plan, int grid, cudaStream_t stream);
// FFTCC3D: which of the three kernels a window takes, and what that kernel needs
constexpr int F3_WARPS = 8;        // fftcc3d_w32.cu: warps of the one-POI CTA
// fftcc3d_w32.cu: two tiles per warp, each a TMA box (36 x 32 floats) or a padded transpose tile (32 x 33)
constexpr size_t FFTCC3D_W32_SMEM = (size_t)2 * F3_WARPS * 32 * 36 * sizeof(float);
constexpr int F3R_THREADS = 128;   // fftcc3d_reg.cu: one thread per 1D transform, 128 / N z-slices per round
// fftcc3d_reg.cu, window of n^3 points: two padded tiles (pitch n + 1) per slice of a round
__host__ __device__ constexpr size_t fftcc3d_reg_smem_bytes(int n) { return (size_t)2 * (F3R_THREADS / n) * n * (n + 1) * sizeof(float); }
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
	int ctas;             // CTAs of a full launch (a queue of n POIs launches min(n, ctas): one POI per CTA at a time)
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
		p->ctas = sm_count * 2; // two resident CTAs per SM (DESIGN.md section 5)
		p->cta_scratch = (size_t)32 * 32 * 32;
		return true;
	}
	if (!force_generic && rx == ry && ry == rz && fft_reg_supported(rx)) {
		const int N = 2 * rx;
		p->path = Fftcc3dPath::REG;
		p->n = N;
		p->slices_per_round = F3R_THREADS / N;
		p->idle_threads = F3R_THREADS - p->slices_per_round * N;
		p->smem = fftcc3d_reg_smem_bytes(N);
		p->ctas = sm_count * fftcc_ctas_per_sm(p->smem + 1024, fft_reg_min_ctas(N)); // + 1 KB covering its static shared memory
		p->cta_scratch = (size_t)2 * N * N * N; // two scratch volumes of N^3 complex
		return true;
	}
	p->path = Fftcc3dPath::GENERIC;
	p->smem = fftcc3d_smem_bytes(rx, ry, rz);
	p->ctas = sm_count * fftcc_ctas_per_sm(p->smem, 2);
	p->cta_scratch = (size_t)8 * rx * ry * rz;
	if (!fft_plan_axis(2 * rx, &p->ax) || !fft_plan_axis(2 * ry, &p->ay) || !fft_plan_axis(2 * rz, &p->az)) p->reject = Fftcc3dReject::PRIME_FACTOR;
	else if (p->smem > smem_optin) p->reject = Fftcc3dReject::SHARED_MEMORY;
	return p->reject == Fftcc3dReject::NONE;
}

// fftcc3d_reg.cu (cubic windows of 2^a 3^b 5^c <= 64 points, one thread per 1D transform, register FFT codelets)
cudaError_t fftcc3d_reg_launch(const Image3D& img, float* d_pois, size_t n_poi, const Fftcc3dPlan& plan, float2* scratch, int grid,
	cudaStream_t stream);
// fftcc.cu
cudaError_t fftcc3d_launch(const Image3D& img, float* d_pois, size_t n, int rx, int ry, int rz, const Fftcc3dPlan& plan, const float2* tw_x,
	const float2* tw_y, const float2* tw_z, float2* scratch, int grid, cudaStream_t stream);
// fftcc3d_w32.cu (32^3 window, register FFTs)
cudaError_t fftcc3d_w32_launch(const Image3D& img, float* d_pois, size_t n, const Fftcc3dPlan& plan, float2* scratch, int grid,
	cudaStream_t stream);
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
cudaError_t calib_map_launch(const float* intrinsics, int height, int width, float convergence, int iteration, float* d_map_x, float* d_map_y,
	cudaStream_t stream);
cudaError_t calib_undistort_launch(const float* d_map_x, const float* d_map_y, int height, int width, const float* intrinsics, float* d_pts, float* d_out,
	size_t n, cudaStream_t stream);
cudaError_t stereo_reconstruct_launch(const StereoCam& c1, const StereoCam& c2, float* d_pts1, float* d_pts2, float* d_pts3d, size_t n,
	cudaStream_t stream);
// the POI2DS records of a stereo series (ocb_stereo_series): n_frames x n, frame-major, from the r1 -> r2 records d_stereo (n), the
// view-1 seeds (n, for x and y) and the two registrations d_out1, d_out2 (n_frames x n POI2D each)
cudaError_t stereo_poi2ds_launch(const StereoCam& c1, const StereoCam& c2, const float* d_stereo, const float* d_seeds1, const float* d_out1,
	const float* d_out2, float* d_out2ds, size_t n, int n_frames, cudaStream_t stream);

cudaError_t gradient3d_launch(const float* ref, float4* rg, int dx, int dy, int dz, int sm_count, cudaStream_t s);
cudaError_t prefilter3d_launch(const float* in, float* out, int dx, int dy, int dz, int axis, int sm_count, cudaStream_t s);
// setup: an Icgn3dSetup; STORE and LOAD need setup_cache, n x ICGN3D_SETUP_FLOATS floats indexed by queue position
cudaError_t icgn3d1_launch(const Icgn3dPlan& plan, const Image3D& img, float* d_pois, size_t n, int rx, int ry, int rz, float conv, float stop,
	int sm_count, int* d_counter, cudaStream_t stream, int setup = ICGN3D_SETUP_COMPUTE, float* setup_cache = nullptr);

} // namespace ocb
