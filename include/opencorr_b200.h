/*
 * opencorr_b200.h -- C ABI of the H100-native (sm_90a) FFT-CC -> IC-GN correlation engine.
 *
 * This is the drop-in boundary for ONE hot path of vincentjzy/OpenCorr: the per-POI
 * FFT-CC integer-pixel initial guess followed by inverse-compositional Gauss-Newton
 * registration.  Every entry point names the reference interface it replaces
 * (paths relative to the reference repo root).  Plain pointers and sizes only; no
 * C++/torch types.  The C++ shim in include/opencorr/ (same class names as the
 * reference) and the Python mirror in opencorr_b200/ are thin layers over this file.
 *
 * Conventions
 *   - POI arrays are the reference's own records, passed verbatim:
 *       POI2D  (src/oc_poi.h:102-136) = 25 floats / 100 bytes
 *         { x, y | u ux uy uxx uxy uyy v vx vy vxx vxy vyy | u0 v0 zncc iteration
 *           convergence feature | exx eyy exy | subset_radius.x subset_radius.y }
 *       POI3D  (src/oc_poi.h:187-222) = 31 floats / 124 bytes
 *         { x, y, z | u ux uy uz v vx vy vz w wx wy wz | u0 v0 w0 zncc iteration
 *           convergence feature | e[6] | subset_radius.x .y .z }
 *     They are mutated in place exactly as the reference's compute(std::vector<POI>&) does,
 *     including the sentinel ZNCC codes of src/oc_dic.h:28-34 (-3 rejected / left the image,
 *     -4 not converged, -5 NaN; a POI arriving with zncc < 0 is skipped).
 *   - Images: float32.  2D row-major [height][width] (col_major=1 accepts the reference's
 *     Eigen::MatrixXf storage, src/oc_image.h:36); volumes [z][y][x] contiguous, the payload
 *     of the reference's float*** (src/oc_array.h:56-74).
 *   - Every function returns OCB_OK (0) or a negative OCB_ERR_* code; the message is
 *     available from ocb_last_error().  There is NO CPU fallback: without a usable CUDA
 *     device ocb_create() fails (returns NULL) and says why.
 *   - Functions taking host POI arrays copy host->device, run, copy back and synchronise
 *     (the reference's blocking compute()); a page-locked array (cudaHostAlloc, ocb_host_alloc,
 *     ocb_host_register) is not copied by the 2D FFT-CC (r = 16) / IC-GN / IC-LM calls: the kernels
 *     read and write the caller's records in place.  The *_dev variants take a device pointer,
 *     enqueue on the context's stream and return without synchronising.
 *   - ocb_set_images_* return once the copies are enqueued: the host images must stay valid and
 *     unchanged until the next call that synchronises (any host-queue call, or ocb_sync()).
 *   - A context (single-device or group) is not to be used from two host threads at the same time.
 */
#ifndef OPENCORR_B200_H_
#define OPENCORR_B200_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OCB_OK 0
#define OCB_ERR_CUDA (-1)        /* CUDA runtime / driver error (message has the CUDA string) */
#define OCB_ERR_ARG (-2)         /* bad argument (null pointer, radius < 1, size mismatch ...) */
#define OCB_ERR_STATE (-3)       /* call order: images not set / prepare() not called */
#define OCB_ERR_UNSUPPORTED (-4) /* subset too large for the on-chip design (see DESIGN.md) */

#define OCB_POI2D_FLOATS 25
#define OCB_POI3D_FLOATS 31
#define OCB_POI2DS_FLOATS 28 /* stereo-DIC record, src/oc_poi.h:140-186 */

typedef struct ocb_ctx ocb_ctx;

/* ---- context ------------------------------------------------------------------------------ */
/* Number of CUDA devices visible, or a negative OCB_ERR_CUDA. */
int ocb_device_count(void);
/* One context = one GPU + one stream + the device copies the reference keeps per DIC/DVC
 * object (images, gradient / B-spline tables, scratch).  Replaces the constructors
 * FFTCC2D/FFTCC3D (src/oc_fftcc.cpp:151-163,300-313) and ICGN2D1/ICGN2D2/ICGN3D1
 * (src/oc_icgn.cpp:71-88,612-629,1197-1215): no per-thread pools are needed on the GPU.
 * Returns NULL on failure (see ocb_last_error(NULL)). */
ocb_ctx* ocb_create(int device);
/* Several devices behind ONE context (SURVEY.md section 8(e): one process, G devices): ocb_create(-1) takes every visible
 * device, ocb_create_multi() the listed ones.  A GROUP context replaces what the reference does with its OpenMP loop over
 * the POI queue, FFTCC2D::compute(std::vector<POI2D>&) src/oc_fftcc.cpp:277-285, ICGN2D1::compute(std::vector<POI2D>&)
 * src/oc_icgn.cpp:343-351 (and the siblings): setImages() uploads the pair to every member, each over its own PCIe link;
 * prepare() runs on every member; every host-queue compute() call splits the caller's array into contiguous blocks
 * (member i gets records [n*i/G, n*(i+1)/G)), and each member copies ITS block in, registers it and copies it back
 * straight into the caller's array, concurrently (one host thread per member).  Results are bit-identical to a
 * single-device context (the POIs are independent).  Queues too short to fill G devices use fewer of them.  Strain needs
 * every POI's neighbours and runs on the first member.  The *_dev / stream entry points need a single-device context:
 * use ocb_member(). */
ocb_ctx* ocb_create_multi(const int* devices, int n_devices);
/* 1 for a single-device context, G for a group; ocb_member(ctx, i) = the i-th member's single-device context (owned by the
 * group), or ctx itself for i == 0 of a single-device context. */
int ocb_member_count(const ocb_ctx* ctx);
ocb_ctx* ocb_member(ocb_ctx* ctx, int index);
void ocb_destroy(ocb_ctx* ctx);
/* Page-lock / release a caller-owned host buffer (an Image2D's pixels, a std::vector<POI2D>'s storage) so that the copies of
 * the host-buffer entry points run as asynchronous DMA at full PCIe rate instead of being staged by the driver.  Optional:
 * every entry point accepts pageable memory.  The range must stay allocated until it is unregistered. */
int ocb_host_register(void* host, size_t bytes);
int ocb_host_unregister(void* host);
/* Page-locked host memory for buffers the caller allocates anew (the shim's Image2D / Image3D keep their pixels in it).
 * ocb_host_alloc returns NULL when there is no usable CUDA device (callers then use ordinary memory). */
void* ocb_host_alloc(size_t bytes);
void* ocb_host_alloc_on(ocb_ctx* ctx, size_t bytes); /* same, after making ctx's (first) device current: no stray context on device 0 */
void ocb_host_free(void* host);
/* Last error message of this context (or of the process when ctx == NULL). Never NULL. */
const char* ocb_last_error(const ocb_ctx* ctx);
/* Enqueue on an external cudaStream_t (e.g. PyTorch's current stream).  The handle is used as given:
 * NULL is CUDA's legacy default stream, NOT "no stream".  ocb_use_own_stream() goes back to the
 * context's private non-blocking stream (the state after ocb_create). */
int ocb_set_stream(ocb_ctx* ctx, void* cuda_stream);
int ocb_use_own_stream(ocb_ctx* ctx);
/* Block until everything enqueued on the context's stream has finished. */
int ocb_sync(ocb_ctx* ctx);
/* Number of kernels this context has launched since creation (bench.py "gpu_launches"). */
long long ocb_launch_count(const ocb_ctx* ctx);

/* ---- images: DIC::setImages / DVC::setImages (src/oc_dic.cpp:22-26,44-48) ----------------- */
/* Host buffers; copied to the device (H2D on the context's stream).  A call refused by its argument checks changes nothing; one
 * that fails later (OCB_ERR_CUDA) leaves no images on the device where it failed, never a view of freed memory. */
int ocb_set_images_2d(ocb_ctx* ctx, const float* ref, const float* tar, int width, int height, int col_major);
int ocb_set_images_3d(ocb_ctx* ctx, const float* ref, const float* tar, int dim_x, int dim_y, int dim_z);
/* 8-bit host images (what cv::imread(..., IMREAD_GRAYSCALE) hands the reference before cv2eigen turns
 * them into floats, src/oc_image.cpp:39,56): uploaded as bytes (4x fewer PCIe bytes) and widened to
 * f32 on the device; results are identical to passing the float copy.  Row-major / [z][y][x]. */
int ocb_set_images_2d_u8(ocb_ctx* ctx, const unsigned char* ref, const unsigned char* tar, int width, int height);
int ocb_set_images_3d_u8(ocb_ctx* ctx, const unsigned char* ref, const unsigned char* tar, int dim_x, int dim_y, int dim_z);
/* Device buffers (row-major / [z][y][x]); BORROWED like the reference borrows Image2D*. */
int ocb_set_images_2d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tar, int width, int height);
int ocb_set_images_3d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tar, int dim_x, int dim_y, int dim_z);

/* ---- FFT-CC: FFTCC2D::compute(std::vector<POI2D>&) src/oc_fftcc.cpp:277-285 (per POI
 *      :177-275) and FFTCC3D::compute(std::vector<POI3D>&) :429-437 (per POI :327-427) ------- */
int ocb_fftcc2d(ocb_ctx* ctx, void* poi2d, size_t n, int rx, int ry);
int ocb_fftcc3d(ocb_ctx* ctx, void* poi3d, size_t n, int rx, int ry, int rz);
int ocb_fftcc2d_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, int rx, int ry);
int ocb_fftcc3d_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, int rx, int ry, int rz);

/* ---- IC-GN prepare(): ICGN2D1::prepare src/oc_icgn.cpp:138-142, ICGN2D2::prepare :679-683,
 *      ICGN3D1::prepare :1264-1268.  2D: nothing is materialised (gradients and bicubic
 *      weights are recomputed on chip); 3D: gradient volumes + tricubic B-spline coefficient
 *      volume are built on the device (src/oc_gradient.cpp:143-231, oc_cubic_bspline.cpp:214-351). */
int ocb_icgn2d_prepare(ocb_ctx* ctx);
int ocb_icgn3d_prepare(ocb_ctx* ctx);

/* ---- IC-GN compute(): ICGN2D1::compute(std::vector<POI2D>&) src/oc_icgn.cpp:343-351 (per POI
 *      :144-341); ICGN2D2 :900-908 (:685-898); ICGN3D1 :1492-1500 (:1270-1490).
 *      conv = conv_criterion, stop = stop_condition (a float in the reference, oc_icgn.h:52). */
int ocb_icgn2d1(ocb_ctx* ctx, void* poi2d, size_t n, int rx, int ry, float conv, float stop);
int ocb_icgn2d2(ocb_ctx* ctx, void* poi2d, size_t n, int rx, int ry, float conv, float stop);
int ocb_icgn3d1(ocb_ctx* ctx, void* poi3d, size_t n, int rx, int ry, int rz, float conv, float stop);
int ocb_icgn2d1_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop);
int ocb_icgn2d2_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop);
int ocb_icgn3d1_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, int rx, int ry, int rz, float conv, float stop);

/* ---- IC-GN, the remaining overloads of the reference's class API (SURVEY.md section 8(f) N1) ------
 * order = 1 (ICGN2D1) or 2 (ICGN2D2).
 * center_offsets: NULL, or n (x, y) pairs -- compute(std::vector<POI2D>&, std::vector<Point2D>&
 *   center_offset_queue), src/oc_icgn.cpp:549-557 (per POI :353-547) and :1128-1136 (:910-1126): local
 *   coordinates are taken relative to poi + offset and the target subset is centred there.
 * self_adaptive != 0: DIC::setSelfAdaptive(true) -- every POI uses its own subset_radius.x/.y fields
 *   (src/oc_icgn.cpp:152-158) and rx, ry are ignored; POIs are grouped by radius on the host and each
 *   group is one launch.  The _dev variant takes device pointers and one radius for all POIs. */
int ocb_icgn2d_ex(ocb_ctx* ctx, int order, void* poi2d, size_t n, int rx, int ry, float conv, float stop, const float* center_offsets,
	int self_adaptive);
int ocb_icgn2d_ex_dev(ocb_ctx* ctx, int order, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop, const float* d_center_offsets);

/* ---- IC-GN over an image series: one reference, n_frames targets.  Replaces the loop a reference user writes over a load
 *      series, carrying one queue from frame to frame:
 *        for f: dic.setImages(ref, tar[f]) (src/oc_dic.cpp:22-26); icgn.prepare() (src/oc_icgn.cpp:138-142 / :679-683);
 *               icgn.compute(queue) (:343-351 / :900-908)
 *      Frame f's records are, bit for bit, what ocb_icgn2d1/2 gives on (ref, tars[f]) for frame f - 1's records (frame 0: the
 *      seeds) in one launch over the same n POIs; a POI that fails in frame f keeps its code in every later frame.  The
 *      reference subset of each POI (gradients, Hessian) is built once for the whole series.
 * The series is context state of its own: the pair calls (ocb_set_images_2d*, ocb_icgn2d*) neither see nor disturb it.
 * tars: n_frames row-major images, frame-major.  On a group context the first member holds the series and runs the calls.
 * A setter refused by its argument checks changes nothing; one that fails later (OCB_ERR_CUDA) leaves no series set.
 * order = 1 (ICGN2D1) or 2 (ICGN2D2).  seeds: n POI2D records; out: n_frames x n POI2D records, frame-major (out[f n + i]),
 *   not overlapping seeds.  A long series runs in chunks: the last frame's slice of out seeds the next chunk.
 * The host variants copy (ocb_icgn2d_series blocks until out is filled); the _dev variants take BORROWED device pointers and
 *   only enqueue.  Errors write nothing to out: OCB_ERR_STATE without a series, OCB_ERR_ARG for bad arguments or sizes,
 *   OCB_ERR_UNSUPPORTED for radii past the shared-memory limit (as ocb_icgn2d1/2). */
int ocb_set_series_2d(ocb_ctx* ctx, const float* ref, const float* tars, int n_frames, int width, int height);
int ocb_set_series_2d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tars, int n_frames, int width, int height);
int ocb_icgn2d_series(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop);
int ocb_icgn2d_series_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop);

/* ---- ICGN3D1 over a volume series: one reference volume, n_frames target volumes (an in-situ CT load series).  Replaces
 *        for f: dvc.setImages(ref, tar[f]); icgn.prepare() (src/oc_icgn.cpp:1264-1268); icgn.compute(queue) (:1492-1500)
 *      Frame f's records are, bit for bit, what ocb_icgn3d1 gives on (ref, tars[f]) for frame f - 1's records (frame 0: the
 *      seeds); a POI that fails in frame f keeps its code in every later frame.  The reference's gradients and each POI's
 *      setup pass (Hessian, its Cholesky factor, the subvolume statistics) are built once per call; each frame runs the target's
 *      B-spline prefilter and the IC-GN iterations.
 * The series is context state of its own: the pair calls (ocb_set_images_3d*, ocb_icgn3d_prepare, ocb_icgn3d1*) neither see
 *   nor disturb it.  tars: n_frames [z][y][x] volumes, frame-major.  On a group context the first member holds the series and
 *   runs the calls.  ocb_set_series_3d_u8 keeps the stack as bytes on the device (1 B per voxel and frame).
 * A setter refused by its argument checks changes nothing; one that fails later (OCB_ERR_CUDA) leaves no series set.
 * seeds: n POI3D records; out: n_frames x n POI3D records, frame-major (out[f n + i]), not overlapping seeds.  A long series
 *   runs in chunks: the last frame's slice of out seeds the next chunk.
 * Device footprint beyond the stack: about 28 B per voxel (reference, packed gradients, coefficients, scratch) and 420 B per
 *   POI (cached setup state); the footprint does not grow with n_frames.  The host variant also stages seeds and out.
 * The host variants copy (ocb_icgn3d_series blocks until out is filled); the _dev variants take BORROWED device pointers and
 *   only enqueue.  Errors write nothing to out: OCB_ERR_STATE without a series, OCB_ERR_ARG for bad arguments or sizes,
 *   OCB_ERR_UNSUPPORTED for subvolumes past the shared-memory limit (as ocb_icgn3d1; r >= 44 when cubic). */
int ocb_set_series_3d(ocb_ctx* ctx, const float* ref, const float* tars, int n_frames, int dim_x, int dim_y, int dim_z);
int ocb_set_series_3d_u8(ocb_ctx* ctx, const unsigned char* ref, const unsigned char* tars, int n_frames, int dim_x, int dim_y, int dim_z);
int ocb_set_series_3d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tars, int n_frames, int dim_x, int dim_y, int dim_z);
int ocb_icgn3d_series(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, int rz, float conv, float stop);
int ocb_icgn3d_series_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv, float stop);

/* ---- Series that re-seed lost POIs with FFT-CC in the frame where they are lost.  Replaces the loop a reference user writes
 *      to keep a field alive over a load series (a crack opening under a subset, glare on one frame, a jump past IC-GN's basin):
 *        for f: dic.setImages(ref, tar[f]); icgn.prepare(); icgn.compute(queue);
 *               lost = the POIs with !(zncc >= zncc_min); rebuild each from its seed;
 *               fftcc.compute(lost) (src/oc_fftcc.cpp); icgn.compute(lost); put them back into queue
 *      over the series set by ocb_set_series_2d* / ocb_set_series_3d*, frames f = 0 ... n_frames - 1 in order:
 *        1. every POI is registered from its frame f - 1 record (frame 0: its seed), as ocb_icgn2d_series / ocb_icgn3d_series do;
 *        2. POI i is lost in frame f when its record has !(zncc >= zncc_min): a NaN ZNCC and every code below zncc_min;
 *        3. its anchor is the translation (u, v[, w]) of its latest record before frame f with zncc >= zncc_min, else the seed's;
 *        4. the lost POIs, in ascending order, are rebuilt from their seeds (x, y[, z] and the subset radii copied, the
 *           translation set to the anchor, every other field 0), then FFT-CC (radii fft_r*) and IC-GN (the series' order,
 *           radii, conv, stop) run on them against (ref, tars[f]) with the pair calls' kernels.  The result replaces the frame-f
 *           record whatever its ZNCC: a POI lost again keeps its new code and is tried again in frame f + 1;
 *        5. frame f + 1 starts from every POI's final frame-f record.
 *      reseeded[f] (n_frames counts, may be NULL) is the number of POIs re-seeded in frame f.  With zncc_min below every code
 *      (e.g. -10) nothing is lost and out is byte-identical to the plain series call.
 *      3D: the records are bit-identical to the loop of ocb_set_images_3d, ocb_icgn3d_prepare, ocb_icgn3d1 on all n POIs, then
 *      ocb_fftcc3d and ocb_icgn3d1 on the rebuilt lost POIs.  2D: the same holds when OCB_ICGN2D_WPP forces the warps per POI;
 *      otherwise every IC-GN launch of the call takes the warps per POI of a launch over all n POIs.
 * Cost: a call that loses nothing adds one scan kernel and one synchronisation (2D) or one of each per frame (3D) to the plain
 *   series; each frame with losses costs one more synchronisation.
 * The _dev variants take BORROWED device seeds and out (reseeded is a host pointer); unlike every other series call they
 *   synchronise ctx's stream, because the per-frame counts size their launches.  Pair state (images, prepared tables) is not
 *   touched.  Errors are detected before any work and write nothing to out or reseeded: OCB_ERR_STATE without a series,
 *   OCB_ERR_ARG for bad arguments or sizes, a bad order, a NaN zncc_min or an FFT-CC radius < 1, OCB_ERR_UNSUPPORTED for an FFT-CC
 *   window or a subset the pair calls reject (with their messages). */
int ocb_icgn2d_series_reseed(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, int fft_rx,
	int fft_ry, float zncc_min, size_t* reseeded);
int ocb_icgn2d_series_reseed_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop,
	int fft_rx, int fft_ry, float zncc_min, size_t* reseeded);
int ocb_icgn3d_series_reseed(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, int rz, float conv, float stop, int fft_rx,
	int fft_ry, int fft_rz, float zncc_min, size_t* reseeded);
int ocb_icgn3d_series_reseed_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv, float stop,
	int fft_rx, int fft_ry, int fft_rz, float zncc_min, size_t* reseeded);

/* ---- Series that recover unreliable POIs with rounds of RegionFit and IC-GN in the frame where they fail.  Replaces the loop a
 *      reference user writes to keep a field alive over a load series with the regfit example's recovery in every frame:
 *        for f: dic.setImages(ref, tar[f]); icgn.prepare(); icgn.compute(queue); the recovery of ocb_icgn2d_recover on queue
 *      over the series set by ocb_set_series_2d* / ocb_set_series_3d*, frames f = 0 ... n_frames - 1 in order:
 *        1. every POI is registered from its frame f - 1 record (frame 0: its seed), as ocb_icgn2d_series / ocb_icgn3d_series do;
 *        2. frame f's n records then go through ocb_icgn2d_recover's rules 1-3 against (ref, tars[f]) with (radius, min_neighbors,
 *           zncc_high, zncc_low, max_rounds): U and R classified once, each round RegionFit over the reliable set on U's working
 *           records and IC-GN on them (the plan of a _dev pair call over |U|), accepted POIs written and appended, a POI never
 *           accepted keeps its bytes;
 *        3. recovered[f * max_rounds + k] (n_frames x max_rounds counts, zero past the last round run, or NULL) is the number
 *           accepted in round k of frame f; remaining[f] (n_frames counts, or NULL) is |U| at the end of frame f;
 *        4. frame f + 1 starts from every POI's final frame-f record: a recovered POI carries its recovered record forward, and a
 *           POI whose subset was occluded in frame k comes back in frame k + 1 once its neighbours can vouch for it.
 *      out, recovered and remaining equal, byte for byte, the loop of ocb_set_images_*(ref, tars[f]), the prepare, the pair IC-GN
 *      (order; 3D ICGN3D1) on all n POIs from frame f - 1's records and ocb_icgn*_recover_dev on them.  3D: always.  2D: when
 *      OCB_ICGN2D_WPP forces the warps per POI; otherwise the series launches take the warps per POI of a launch over all n POIs
 *      and the recovery rounds those of |U|, as the loop does.  max_rounds = 0, or thresholds under which no record is
 *      unreliable, give out byte-identical to the plain series call.
 * Cost: 2D runs the plain series launch, one scan and one synchronisation; each frame that holds an unreliable record adds the
 *   recovery rounds (as ocb_icgn2d_recover_dev, plus one launch per round), one series launch of the accepted POIs over the later
 *   frames, a scatter, a rescan and one more synchronisation.  3D runs the rounds' classification (one synchronisation) in every
 *   frame.  The workspaces are the context's grow-only buffers.
 * The _dev variants take BORROWED device seeds and out (recovered, remaining are host pointers), synchronise ctx's stream
 *   (the counts size the launches) and need a single-device context; on a group context the first member runs the host
 *   variants.  Pair state (images, prepared tables) is not touched.  Errors are detected before any work and write nothing to
 *   out, recovered or remaining: OCB_ERR_STATE without a series, OCB_ERR_ARG for bad arguments or sizes, an order not 1 or 2,
 *   max_rounds < 0 or a NaN conv / zncc_high / zncc_low, OCB_ERR_UNSUPPORTED for a subset the pair calls reject. */
int ocb_icgn2d_series_recover(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, float radius,
	int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);
int ocb_icgn2d_series_recover_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop,
	float radius, int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);
int ocb_icgn3d_series_recover(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, int rz, float conv, float stop, float radius,
	int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);
int ocb_icgn3d_series_recover_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv, float stop,
	float radius, int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);

/* ---- IC-LM siblings (SURVEY.md section 8(f) N2): ICLM2D1::compute(std::vector<POI2D>&) src/oc_iclm.cpp:360-368
 *      (per POI :150-358) and ICLM2D2 :732-740 (:502-730).  Same prepare() as IC-GN (ocb_icgn2d_prepare).
 *      lambda, alpha, beta = DampingParameter (src/oc_iclm.h:32-37; defaults 100, 0.1, 10; setDamping()). */
int ocb_iclm2d(ocb_ctx* ctx, int order, void* poi2d, size_t n, int rx, int ry, float conv, float stop, float lambda, float alpha, float beta);
int ocb_iclm2d_dev(ocb_ctx* ctx, int order, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop, float lambda, float alpha, float beta);

/* ---- NR2D1, forward-additive Newton-Raphson (SURVEY.md section 8(f) N2): NR2D1::prepare src/oc_nr.cpp:119-156
 *      (nothing is precomputed here: the target gradients and the three bicubic interpolants are evaluated
 *      on chip), NR2D1::compute(std::vector<POI2D>&) :327-334 (per POI :160-325). */
int ocb_nr2d_prepare(ocb_ctx* ctx);
int ocb_nr2d1(ocb_ctx* ctx, void* poi2d, size_t n, int rx, int ry, float conv, float stop);
int ocb_nr2d1_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop);

/* ---- IC-LM over an image series.  Replaces the loop a reference user writes over a load series with an IC-LM method:
 *        for f: dic.setImages(ref, tar[f]); iclm.prepare(); iclm.compute(queue)
 *               (ICLM2D1::compute(std::vector<POI2D>&) src/oc_iclm.cpp:360-368, ICLM2D2 :732-740)
 *      over the series set by ocb_set_series_2d*.  Frame f's records are, bit for bit, what ocb_iclm2d gives on (ref, tars[f])
 *      with the same damping for frame f - 1's records (frame 0: the seeds) in one launch over the same n POIs (OCB_ICGN2D_WPP,
 *      the warps per POI, as for ocb_icgn2d_series).  Each POI's reference subset and undamped Hessian are built once for the
 *      whole series; the damping restarts from lambda in every frame, as a pair call does.  lambda, alpha, beta as for
 *      ocb_iclm2d, passed through unchecked.  Everything else (order, seeds, out, chunking, _dev borrowing, group contexts,
 *      errors) as for ocb_icgn2d_series; the _reseed variants follow ocb_icgn2d_series_reseed's rules 1-5 with IC-LM (the same
 *      damping) in place of IC-GN. */
int ocb_iclm2d_series(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, float lambda,
	float alpha, float beta);
int ocb_iclm2d_series_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop, float lambda,
	float alpha, float beta);
int ocb_iclm2d_series_reseed(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, float lambda,
	float alpha, float beta, int fft_rx, int fft_ry, float zncc_min, size_t* reseeded);
int ocb_iclm2d_series_reseed_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop,
	float lambda, float alpha, float beta, int fft_rx, int fft_ry, float zncc_min, size_t* reseeded);

/* ---- NR2D1 over an image series.  Replaces the loop a reference user writes over a load series with NR2D1:
 *        for f: dic.setImages(ref, tar[f]); nr.prepare() (NR2D1::prepare src/oc_nr.cpp:119-156);
 *               nr.compute(queue) (NR2D1::compute(std::vector<POI2D>&) :327-334)
 *      over the series set by ocb_set_series_2d*.  Frame f's records are, bit for bit, what ocb_nr2d1 gives on (ref, tars[f])
 *      for frame f - 1's records (frame 0: the seeds).  A POI that fails the guard gets the pair call's code in each later
 *      frame too: -1, or -4 / -5 from the tests NR2D1 runs on every record, so its code can change from frame to frame.  Each
 *      POI's reference subset is staged once for the whole series; the target gradients are rebuilt in every frame.
 *      No order argument; everything else (seeds, out, chunking, _dev borrowing, group contexts, errors) as for
 *      ocb_icgn2d_series, with the radius refused as by ocb_nr2d1; the _reseed variants follow ocb_icgn2d_series_reseed's
 *      rules 1-5 with NR2D1 in place of IC-GN. */
int ocb_nr2d1_series(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop);
int ocb_nr2d1_series_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop);
int ocb_nr2d1_series_reseed(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, int fft_rx, int fft_ry,
	float zncc_min, size_t* reseeded);
int ocb_nr2d1_series_reseed_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop, int fft_rx,
	int fft_ry, float zncc_min, size_t* reseeded);

/* ---- EpipolarSearch (SURVEY.md section 8(f) N4): EpipolarSearch::compute(std::vector<POI2D>&) src/oc_epipolar_search.cpp:197-205
 *      (per POI :133-195) as one batch: every POI spawns its candidates along the epipolar line of the secondary view
 *      (centre + every search_step pixels in x below search_radius, both directions), ICGN2D1(rx, ry, conv, stop) registers
 *      all of them, the candidate with the highest ZNCC replaces the POI's deformation and result.
 *      fundamental: the 3x3 fundamental matrix, row-major (updateFundementalMatrix :110-126); parallax_x/_y: the three
 *      coefficients of setParallax(float[3], float[3]) (setParallax(Point2D p) = {0, 0, p.x}, {0, 0, p.y}) -- host pointers in
 *      both variants.  Images = primary / secondary view (setImages), after ocb_icgn2d_prepare (prepareICGN :63-67). */
int ocb_epipolar_search2d(ocb_ctx* ctx, void* poi2d, size_t n, const float* fundamental, const float* parallax_x, const float* parallax_y,
	int search_radius, int search_step, int rx, int ry, float conv, float stop);
int ocb_epipolar_search2d_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, const float* fundamental, const float* parallax_x, const float* parallax_y,
	int search_radius, int search_step, int rx, int ry, float conv, float stop);

/* ---- Strain post-processing of a POI queue (SURVEY.md section 8(f) N4): Strain::prepare + Strain::compute(queue),
 *      src/oc_strain.cpp:100-111,150-156,239-250 (POI2D; per POI :158-237) and :476-487 (POI3D; per POI :373-474).
 *      radius = subregion_radius, min_neighbors = neighbor_number_min (constructor :32-36), zncc_threshold = setZnccThreshold
 *      (default 0.9, :38), approximation = setApproximation: 1 Cauchy (default), 2 Green.  Writes strain.exx.. of every POI
 *      whose own ZNCC and enough neighbours' ZNCC pass the threshold; other records are left untouched.
 *      (The stereo variant, POI2DS records, is ocb_strain2ds below.) */
int ocb_strain2d(ocb_ctx* ctx, void* poi2d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
int ocb_strain3d(ocb_ctx* ctx, void* poi3d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
/* Strain::compute(POI2D* poi, queue) / (POI3D* poi, queue) for the queue member `index`: fitted whatever its own ZNCC. */
int ocb_strain2d_single(ocb_ctx* ctx, void* poi2d, size_t n, size_t index, float radius, int min_neighbors, float zncc_threshold, int approximation);
int ocb_strain3d_single(ocb_ctx* ctx, void* poi3d, size_t n, size_t index, float radius, int min_neighbors, float zncc_threshold, int approximation);
/* Stereo-DIC queues (POI2DS records, OCB_POI2DS_FLOATS floats: x y | u v w | r1r2 r1t1 r1t2 ZNCC r2_x r2_y t1_x t1_y t2_x t2_y |
 * ref_coor | tar_coor | e[6] | subset_radius, src/oc_poi.h:140-186): Strain::compute(std::vector<POI2DS>&) src/oc_strain.cpp:362-371
 * (per POI :252-360) -- neighbours searched in the image plane, plane fit over ref_coor and u, v, w, all three ZNCCs tested. */
int ocb_strain2ds(ocb_ctx* ctx, void* poi2ds, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
int ocb_strain2ds_dev(ocb_ctx* ctx, void* d_poi2ds, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
int ocb_strain2d_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
int ocb_strain3d_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
/* Strain over a series: n_frames frames of n records each, frame-major (the layout the series calls write).  Frame f's records
 * become, bit for bit, what ocb_strain*_dev(ctx, records + f * n * floats, n, ...) leaves on them, for every radius and
 * approximation; the neighbours of each POI are searched once for all frames, and only the ZNCC filter, the displacements and
 * (POI2DS) ref_coor are read per frame.  Every frame's search coordinates (x, y; POI3D: x, y, z) must be frame 0's, bit for
 * bit (NaN included): otherwise OCB_ERR_ARG and nothing is written.  OCB_ERR_ARG as well, before any kernel runs, for NULL
 * records with n_frames * n > 0 and for n_frames * n * floats floats that overflow a size_t; n per frame has the pair call's
 * limit.  n_frames = 0 or n = 0 does nothing.  The host variants copy; the _dev variants take BORROWED device records and only
 * enqueue (single-device context); a call makes the same launches and one readback whatever n_frames.  On a group context the
 * first member runs the host variants. */
int ocb_strain2d_series(ocb_ctx* ctx, void* poi2d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
int ocb_strain3d_series(ocb_ctx* ctx, void* poi3d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation);
int ocb_strain2ds_series(ocb_ctx* ctx, void* poi2ds, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation);
int ocb_strain2d_series_dev(ocb_ctx* ctx, void* d_poi2d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation);
int ocb_strain3d_series_dev(ocb_ctx* ctx, void* d_poi3d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation);
int ocb_strain2ds_series_dev(ocb_ctx* ctx, void* d_poi2ds, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation);

/* ---- RegionFit2D / RegionFit3D (src/oc_region_fit.cpp): a new initial guess for unreliable POIs from their reliable neighbours.
 *      setNeighbor(reliable) + prepare + compute(queue), the reliable set read when the call runs.  For every queue POI with a
 *      finite position: the n_reliable reliable records (POI2D / POI3D, the same kind as the queue) whose float squared distance
 *      (x, y(, z)) is strictly below radius^2 are its neighbours (a negative radius acts as its magnitude); when fewer than
 *      min_neighbors are found, the min(min_neighbors, n_reliable) nearest take their place (ties to the lower reliable index).
 *      Every neighbour counts, whatever its ZNCC.  With at least min_neighbors of them, the least-squares plane
 *      [1, x_i - x, y_i - y(, z_i - z)] over u, v (, w) -- the basic solution when rank-deficient -- writes u ux uy v vx vy
 *      (POI3D: u ux uy uz v .. wz) and zncc = 0; every other field (POI2D: the second-order terms too) is left as it was, and a
 *      POI with too few neighbours is left untouched.  Reliable POIs with a non-finite position are no one's neighbour.
 *      OCB_ERR_ARG, with nothing written, for NULL records with a count > 0 or either count >= 2^31.  n = 0 does nothing.  The
 *      host variants copy both sets and the queue back; the _dev variants take BORROWED device records and only enqueue
 *      (single-device context).  One readback and the same five launches per call whatever the counts; on a group context the
 *      first member runs the host variants. */
int ocb_region_fit2d(ocb_ctx* ctx, const void* reliable, size_t n_reliable, void* poi2d, size_t n, float radius, int min_neighbors);
int ocb_region_fit3d(ocb_ctx* ctx, const void* reliable, size_t n_reliable, void* poi3d, size_t n, float radius, int min_neighbors);
int ocb_region_fit2d_dev(ocb_ctx* ctx, const void* d_reliable, size_t n_reliable, void* d_poi2d, size_t n, float radius, int min_neighbors);
int ocb_region_fit3d_dev(ocb_ctx* ctx, const void* d_reliable, size_t n_reliable, void* d_poi3d, size_t n, float radius, int min_neighbors);

/* ---- Recovery of unreliable POIs: rounds of RegionFit and IC-GN in one call (the loop of the reference's
 *      examples/test_3d_reconstruction_sift_icgn2_regfit.cpp:215-270).  q: n registered records (POI2D: ICGN2D<order> on the pair of
 *      ocb_set_images_2d*, prepared; POI3D: ICGN3D1 on the volume pair, prepared).
 *      1. Once: U = { i : zncc < zncc_low || convergence > conv } and R = { i not in U : zncc >= zncc_high }, both in queue order
 *         (literal float comparisons: a NaN field fails both).  Every other POI is left alone.
 *      2. Round k, while k < max_rounds and U is not empty: RegionFit (ocb_region_fit*_dev, radius, min_neighbors) over the
 *         reliable set in its current order, on U's working records; the pair IC-GN on them (the plan of a _dev pair call over
 *         |U| POIs); every one with zncc >= zncc_high && convergence <= conv is accepted: written to q and appended to the
 *         reliable set in queue order, and leaves U.  recovered[k] = how many; the loop stops after a round that accepts none.
 *      3. A POI never accepted keeps its bytes in q; its failed records only seed its next round's fit, as in the example.
 *      Unlike the example, whose erase inside its index loop skips the POI after each accepted one for that round, every POI
 *      that passes is accepted.  recovered (max_rounds entries, zero past the last round run, or NULL) and *remaining (|U| at the
 *      end, or NULL) are written only on success.  Refused with nothing written, before any device work: the pair call's checks
 *      and plan, order not 1 or 2, max_rounds < 0, NaN conv / zncc_high / zncc_low, NULL records with n > 0, n >= 2^31.
 *      The host variants stage the queue once and copy it back once; the _dev variants take device records and synchronise the
 *      stream (the per-round counts size the next launches), and need a single-device context.  On a group context the first
 *      member runs the host variants.  Launches: two for the classification, then one move and nine per round, whatever n. */
int ocb_icgn2d_recover(ocb_ctx* ctx, int order, void* poi2d, size_t n, int rx, int ry, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);
int ocb_icgn2d_recover_dev(ocb_ctx* ctx, int order, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);
int ocb_icgn3d_recover(ocb_ctx* ctx, void* poi3d, size_t n, int rx, int ry, int rz, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);
int ocb_icgn3d_recover_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, int rx, int ry, int rz, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining);

/* ---- Stereo reconstruction: Calibration::prepare / undistort (src/oc_calibration.cpp:161-264) and
 *      Stereovision::reconstruct (src/oc_stereovision.cpp:70-133) ----------------------------------------------------------
 * intrinsics: the 13 floats of CameraIntrinsics (src/oc_calibration.h:25-35), fx fy fs cx cy k1 k2 k3 k4 k5 k6 p1 p2.
 * projection: the camera's 3x4 projection matrix K [R | t], row-major (Calibration::updateProjectionMatrix, :69-77).
 * ocb_calib = one camera's distortion map (map_x, map_y: float32 [height][width] in device memory), built by ocb_calib_prepare
 * with the fixed-point loop of :180-218 (at most `iteration` rounds, stop when both deviations are <= convergence; the
 * reference's defaults are 0.001 and 40).  The handle belongs to the context it was made with; on a GROUP context the maps live
 * on the first member and the calls below run there (the point sets are small; see DESIGN.md section 6).
 * Points are n (x, y) float pairs.  As the reference takes Point2D&, every point is clamped IN PLACE to [0, W-2] x [0, H-2]
 * before the bilinear lookup (:224-239).  The intrinsics of the lookup are passed with each call ("current at call time"). */
typedef struct ocb_calib ocb_calib;
int ocb_calib_prepare(ocb_ctx* ctx, const float* intrinsics, int height, int width, float convergence, int iteration, ocb_calib** out);
void ocb_calib_destroy(ocb_calib* calib);
/* Copy the maps to host buffers of height*width floats each (row-major); either pointer may be NULL. */
int ocb_calib_get_map(ocb_ctx* ctx, const ocb_calib* calib, float* map_x, float* map_y);
/* Calibration::undistort for n host points: pts (n x 2) clamped in place, out (n x 2) = sensor coordinates.  A point with a
 * NaN coordinate (undefined in the reference) is left as it is and gives NaN.  Blocking. */
int ocb_calib_undistort(ocb_ctx* ctx, const ocb_calib* calib, const float* intrinsics, float* pts, float* out, size_t n);
/* Stereovision::reconstruct(queue, queue, queue) as one batch: pts3d (n x 3) = world coordinates.  A NaN coordinate in either view
 * gives (0, 0, 0) and leaves both points untouched; every other pair is clamped in place.  The 4x3 system of :87-112 is formed
 * in float32 and solved as least squares in FP64.  Host buffers (blocking) / device buffers (enqueue only, single-device context). */
int ocb_stereo_reconstruct(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, float* pts1, float* pts2, float* pts3d, size_t n);
int ocb_stereo_reconstruct_dev(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, float* d_pts1, float* d_pts2, float* d_pts3d, size_t n);

/* ---- Stereo DIC over a load series of stereo pairs: both views of every frame registered against reference view 1 and
 *      triangulated, the loop of the reference's 3D-DIC example (examples/test_3d_dic_epipolar_sift.cpp:178-317) over frames,
 *      each frame seeded by the previous one instead of by SIFT features.
 * State (ocb_set_stereo_series_2d*): ref1, reference view 1 (width x height), and tars1 / tars2, n_frames row-major images each,
 *   frame-major: view 1 and view 2 of frames 0 ... n_frames - 1.  All images have the same size.  The reference view-2 image is
 *   not part of it: the r1 -> r2 match is an input (from the pair calls: ocb_set_images_2d(r1, r2), ocb_icgn2d_prepare,
 *   ocb_epipolar_search2d, ocb_icgn2d2).  The state is the context's own: the pair calls and ocb_set_series_2d* neither see nor
 *   change it, and it changes neither.  On a group context the first member holds it and runs the calls.
 * A setter refused by its argument checks changes nothing; one that fails later (OCB_ERR_CUDA) leaves no stereo series set.
 * Inputs: stereo, n POI2D records of the r1 -> r2 match; seeds1 / seeds2, n POI2D frame-0 guesses of view 1 / view 2; order1,
 *   order2 = 1 (ICGN2D1) or 2 (ICGN2D2); rx, ry, conv, stop shared by both views; the cameras as ocb_stereo_reconstruct takes them.
 * For every frame f:
 *   out1[f] = IC-GN (order1) of (ref1, tars1[f]) from out1[f - 1] (frame 0: seeds1): bit for bit ocb_icgn2d_series on (ref1, tars1);
 *   out2[f] = IC-GN (order2) of (ref1, tars2[f]) from out2[f - 1] (frame 0: seeds2): bit for bit ocb_icgn2d_series on (ref1, tars2);
 *   out2ds[f][i], a POI2DS record, all float32: x, y of seeds1[i]; r2 = stereo location + (u, v), t1 = out1[f] location + (u, v),
 *   t2 = out2[f] location + (u, v), stored unclamped; ZNCCs r1r2 / r1t1 / r1t2 of stereo / out1[f] / out2[f] (failure codes
 *   included); ref_coor = reconstruct((x, y), r2), tar_coor = reconstruct(t1, t2), where reconstruct is ocb_stereo_reconstruct on
 *   copies of the points (clamped per camera; a NaN coordinate gives (0, 0, 0)); u, v, w = tar_coor - ref_coor; strain and
 *   subset_radius 0.  Strain over every frame: ocb_strain2ds_series(ctx, out2ds, n_frames, n, ...).
 * out1, out2: n_frames x n POI2D records, out2ds: n_frames x n POI2DS records, frame-major, overlapping no input.  A long series
 *   runs in chunks: the last frame's slices of out1 and out2 seed the next chunk.
 * The host variants copy (ocb_stereo_series blocks until the outputs are filled); the _dev variants take BORROWED device images,
 *   records and outputs (the camera arrays stay host pointers) and only enqueue.  Errors are detected before any kernel runs and
 *   write nothing to any output: OCB_ERR_STATE without a stereo series, OCB_ERR_ARG for a bad order, NULL pointers, sizes or a calibration
 *   handle of another context, OCB_ERR_UNSUPPORTED for radii the pair calls reject. */
int ocb_set_stereo_series_2d(ocb_ctx* ctx, const float* ref1, const float* tars1, const float* tars2, int n_frames, int width, int height);
int ocb_set_stereo_series_2d_dev(ocb_ctx* ctx, const float* d_ref1, const float* d_tars1, const float* d_tars2, int n_frames, int width, int height);
int ocb_stereo_series(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, int order1, int order2, const void* stereo, const void* seeds1, const void* seeds2,
	void* out1, void* out2, void* out2ds, size_t n, int rx, int ry, float conv, float stop);
int ocb_stereo_series_dev(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, int order1, int order2, const void* d_stereo, const void* d_seeds1, const void* d_seeds2,
	void* d_out1, void* d_out2, void* d_out2ds, size_t n, int rx, int ry, float conv, float stop);

/* ---- SIFT3D: SIFT3D::compute() src/oc_sift.cpp:234-293 on the volumes of ocb_set_images_3d / _u8 / _dev --------------------
 * Extracts the keypoints of the reference and of the target volume (Gaussian pyramid :676-754 built one octave at a time, DoG
 * extrema :795-847, orientation :849-1049, descriptors :1051-1249) and matches them (monodirectionalMatch :1251-1418).
 * config: OCB_SIFT3D_CONFIG_FLOATS floats, the fields of Sift3dConfig (src/oc_sift.h:71-83) in order:
 *   n_octave_layers, n_octave (ignored: computed, :683-684), min_dimension, alpha, beta, gamma, sigma_source, sigma_base,
 *   gradient_threshold, truncate_threshold
 * (the constructor's defaults, :142-152: 3, -, 8, 0.1, 0.9, 0.4, 1.15, 1.6, 1e-10, 0.2 * 128 / 768).
 * unit_xyz: the physical voxel size (setPhysicalUnit :197-202); matching_ratio: setMatchingRatio (:204-207, default 0.85).
 * Blocking.  *n_matched = number of matched pairs; *n_octave = the computed octave count (written back to sift_config by the
 * reference).  Either pointer may be NULL.  Results stay in the context until the next ocb_sift3d call.  A call that fails
 * before any device work (its argument checks, the pyramid plan's n_octave_layers, volume size and blur radius, or selecting the
 * device) leaves the previous call's results readable, bit for bit.  A call that fails once its device work has begun (a CUDA
 * error, or OCB_ERR_ARG "too many keypoints") leaves none: ocb_sift3d_get_matches, _inspect and _stage_times then report that
 * ocb_sift3d has not run.  Where the reference is undefined (a mirrored blur index still out of range, reads past the end of its
 * match list) DESIGN.md defines the result.
 * On a GROUP context the first member runs it.  There is no CPU path. */
#define OCB_SIFT3D_CONFIG_FLOATS 10
#define OCB_SIFT3D_KP_FLOATS 18 /* coor_layer xyz, coor_img xyz, octave, layer, scale, R[9] (rows q0, q1, q0 x q1) */
#define OCB_SIFT3D_DESC_FLOATS 768
#define OCB_SIFT3D_STAGES 10
int ocb_sift3d(ocb_ctx* ctx, const float* config, const float* unit_xyz, float matching_ratio, size_t* n_matched, int* n_octave);
/* The matched pairs: ref_matched_kp / tar_matched_kp (coor_img of each keypoint, :1392-1417), n_matched x 3 floats each. */
int ocb_sift3d_get_matches(ocb_ctx* ctx, float* ref_xyz, float* tar_xyz);
/* Inspection of one image's products (image 0 = reference, 1 = target) for parity tests.  counts[3] = { candidates, max_abs
 * entries, keypoints }; any array may be NULL (call once with NULLs to size them).  candidates: 5 ints each (octave, layer, z, y,
 * x) in the reference's push order; max_abs: one per DoG layer, octave-major (n_octave x (n_octave_layers + 2)); keypoints:
 * OCB_SIFT3D_KP_FLOATS each, the kept candidates in order; descriptors: 768 floats each. */
int ocb_sift3d_inspect(ocb_ctx* ctx, int image, size_t* counts, int* candidates, float* max_abs, float* keypoints, float* descriptors);
/* Milliseconds of the last ocb_sift3d per stage (CUDA events; the host post-pass on the host clock): ref pyramid, extrema,
 * orientation, descriptors; tar the same four; matching (distance kernels and the copy of the top-2 table); host post-pass. */
int ocb_sift3d_stage_times(ocb_ctx* ctx, float* ms);

/* ---- inspection (parity tests of the prepare() products) ----------------------------------- */
/* Copy the device tables built by ocb_icgn3d_prepare() to host buffers of dim_x*dim_y*dim_z
 * floats each; any pointer may be NULL. */
int ocb_get_tables_3d(ocb_ctx* ctx, float* gx, float* gy, float* gz, float* coefficient);

#ifdef __cplusplus
}
#endif
#endif /* OPENCORR_B200_H_ */
