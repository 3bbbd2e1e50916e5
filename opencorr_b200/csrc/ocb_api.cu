// ocb_api.cu -- host side of the C ABI declared in include/opencorr_b200.h.
// Owns the per-GPU context (device images, DVC tables, FFT twiddles/scratch, POI staging buffer)
// and forwards to the sm_90a kernels.  No CPU compute path exists here by design.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <condition_variable>
#include <functional>
#include <initializer_list>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "../../include/opencorr_b200.h"
#include "ocb_kernels.h"

namespace ocb {
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int w, int h) {
	// in: column-major [w][h] (element (r,c) at c*h + r)  ->  out: row-major [h][w]
	__shared__ float t[32][33];
	const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
	for (int j = threadIdx.y; j < 32; j += blockDim.y) {
		const int c = c0 + j, r = r0 + threadIdx.x;
		if (c < w && r < h) t[j][threadIdx.x] = in[(size_t)c * h + r];
	}
	__syncthreads();
	for (int j = threadIdx.y; j < 32; j += blockDim.y) {
		const int r = r0 + j, c = c0 + threadIdx.x;
		if (c < w && r < h) out[(size_t)r * w + c] = t[threadIdx.x][j];
	}
}
__global__ void widen_u8_kernel(const unsigned char* __restrict__ in, float* __restrict__ out, size_t n) {
	// 4 pixels per thread: one 32-bit load, one 128-bit store (n4 = n / 4 handled vectorised, tail scalar)
	const size_t n4 = n / 4;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
		const uchar4 v = reinterpret_cast<const uchar4*>(in)[i];
		reinterpret_cast<float4*>(out)[i] = make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
	}
	for (size_t i = n4 * 4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) out[i] = (float)in[i];
}
} // namespace ocb

static thread_local std::string g_last_error = "";

// One persistent host thread per extra member of a GROUP context (ocb_create(-1) / ocb_create_multi): the members' copies
// and launches are issued concurrently, each device moving its share over its own PCIe link.
struct ocb_worker {
	std::thread th;
	std::mutex mu;
	std::condition_variable cv;
	std::function<int()> job;
	int result = 0;
	std::atomic<int> state{ 0 }; // 0 idle, 1 job posted, 2 job done
	bool stop = false;
	// A call on a group context is a handful of sub-millisecond phases, so both sides first spin on `state` (a condition-variable
	// round trip costs tens of microseconds per phase and member) and only then go to sleep.
	static bool spin_until(const std::atomic<int>& st, int want) {
		for (int i = 0; i < 20000; i++) {
			if (st.load(std::memory_order_acquire) == want) return true;
#if defined(__x86_64__)
			__builtin_ia32_pause();
#endif
		}
		return false;
	}
	void loop() {
		for (;;) {
			if (!spin_until(state, 1)) {
				std::unique_lock<std::mutex> lk(mu);
				cv.wait(lk, [&] { return state.load(std::memory_order_acquire) == 1 || stop; });
			}
			if (stop && state.load(std::memory_order_acquire) != 1) return;
			result = job();
			{
				std::lock_guard<std::mutex> lk(mu);
				state.store(2, std::memory_order_release);
			}
			cv.notify_all();
		}
	}
	void post(std::function<int()> f) {
		job = std::move(f);
		{
			std::lock_guard<std::mutex> lk(mu);
			state.store(1, std::memory_order_release);
		}
		cv.notify_all();
	}
	int wait() {
		if (!spin_until(state, 2)) {
			std::unique_lock<std::mutex> lk(mu);
			cv.wait(lk, [&] { return state.load(std::memory_order_acquire) == 2; });
		}
		state.store(0, std::memory_order_release);
		return result;
	}
};

using ocb::DevBuf; // a context's buffers are freed by `delete ctx` in ocb_destroy, with its device current

// One series (ocb_set_series_2d*, ocb_set_series_3d*, ocb_set_stereo_series_2d*): a float reference against the frame-major
// stacks tars[0] and (stereo) tars[1], `frames` frames of w x h x d pixels (d = 1: images) starting `pitch` bytes apart (a float
// stack: one frame of floats; the 8-bit volume stack: the frame's bytes rounded up to 16).  The host setters upload into `own`
// ({reference, stack 0, stack 1}), the _dev setters borrow.  No reference: no series.
struct SeriesStore {
	DevBuf own[3];
	const float* ref = nullptr;
	const void* tars[2] = { nullptr, nullptr };
	size_t pitch = 0;
	int frames = 0;
	int w = 0, h = 0, d = 0;
	ocb::Image2D view2(int k) const { return ocb::Image2D{ ref, (const float*)tars[k], w, h }; }
};

struct ocb_ctx {
	// GROUP context: non-empty `members` (single-device contexts owned by the group); none of the per-device fields below
	// is used.  Host-buffer entry points shard their POI queue over the members; *_dev entry points are refused.
	std::vector<ocb_ctx*> members;
	std::vector<ocb_worker*> workers; // workers[i] serves members[i + 1]; member 0 runs on the calling thread
	bool peer_ok = false;             // group: every member can address every other member's memory (NVLink / NVSwitch)
	cudaEvent_t ev_idle = nullptr, ev_pushed = nullptr; // member of a group: see group_distribute_pair
	ocb_ctx* group = nullptr;          // member: the group it belongs to
	bool need_peer_wait = false;       // member: its stream has not yet been ordered after the peers' image pushes
	int device = 0;
	int sm_count = 0;
	size_t smem_optin = 0;
	cudaStream_t own_stream = nullptr;
	cudaStream_t stream = nullptr;
	std::string last_error;
	long long launches = 0;

	// 2D images
	DevBuf own2[2]; // {ref, tar} uploaded from the host
	ocb::Image2D img2{ nullptr, nullptr, 0, 0 };
	bool prepared2 = false;
	bool prepared_nr2 = false;

	// the image, volume and stereo series: each its own state, untouched by the pair calls and by the other two.  The stereo
	// series holds reference view 1 and the stacks of view 1 and view 2.
	SeriesStore series2d, series3d, stereo;

	// 3D images + tables
	DevBuf own3[2]; // {ref, tar} uploaded from the host
	DevBuf rg3;     // float4: packed {ref, gx, gy, gz}
	DevBuf coef3;   // tricubic B-spline coefficients
	DevBuf tmp3;
	ocb::Image3D img3{ nullptr, nullptr, nullptr, nullptr, 0, 0, 0 };
	bool prepared3 = false;

	// the volume series' work buffers: packed gradients, coefficients, scratch volume, per-POI setup cache
	DevBuf series3_rg, series3_coef, series3_tmp, series3_cache;
	// series calls that re-seed lost POIs: lost-frame/index/histogram/anchor workspace, the rebuilt sub-queue and (2D) the
	// sub-queue's continuation over the later frames
	DevBuf reseed_ws, reseed_sub, reseed_cont;

	// FFT
	std::map<int, float2*> twiddles;
	DevBuf fft_scratch; // float2

	int* d_counter = nullptr; // work-queue heads of the persistent kernels

	// POI staging
	DevBuf d_poi;
	DevBuf d_u8;  // staging for 8-bit image uploads
	DevBuf d_off; // centre offsets (2 floats per POI)
	// host-queue calls on large 2D queues are split into chunks whose H2D copy, kernel and D2H copy run on separate
	// streams, so the PCIe transfers of one chunk overlap the kernel of another
	cudaStream_t pipe[4] = { nullptr, nullptr, nullptr, nullptr };
	cudaEvent_t pipe_ready = nullptr;
	// ocb_set_images_2d uploads the pair in OCB_BANDS row bands (ref band, tar band, event) so that the FFT-CC call that follows
	// can start on the POIs of the first rows while the rest of the pair is still crossing PCIe
	cudaEvent_t band_done[4] = { nullptr, nullptr, nullptr, nullptr };
	int band_end[4] = { 0, 0, 0, 0 }; // first row NOT covered once band_done[b] has fired
	bool bands_fresh = false;         // nothing has been enqueued on `stream` since the banded upload
	DevBuf d_cand;      // EpipolarSearch candidate queue
	DevBuf d_strain_ws; // Strain: sort keys / compact neighbour arrays / cub scratch
	// the recovery calls: index lists, counts and cub scratch; the reliable set and the two working sets of records
	DevBuf recover_ws, recover_rec;
	DevBuf d_stereo;    // stereo reconstruction / undistortion: staged points
	ocb::Sift3d* sift3d = nullptr; // SIFT3D working buffers and the products of the last ocb_sift3d call
};

// One camera's distortion map (Calibration::prepare).  `owner` is the context the caller made it with (a group or a single
// device); `exec` is the single-device context that holds the maps and runs every call on them.
struct ocb_calib {
	const ocb_ctx* owner = nullptr;
	ocb_ctx* exec = nullptr;
	int device = 0;
	int height = 0, width = 0;
	float* map_x = nullptr;
	float* map_y = nullptr;
};

static int set_error(ocb_ctx* ctx, int code, const char* fmt, ...) {
	char buf[512];
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(buf, sizeof(buf), fmt, ap);
	va_end(ap);
	g_last_error = buf;
	if (ctx) ctx->last_error = buf;
	return code;
}

#define OCB_CUDA(ctx, call)                                                                                   \
	do {                                                                                                      \
		cudaError_t e_ = (call);                                                                              \
		if (e_ != cudaSuccess) return set_error(ctx, OCB_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
	} while (0)

static int ensure_device(ocb_ctx* ctx) {
	OCB_CUDA(ctx, cudaSetDevice(ctx->device));
	return OCB_OK;
}

// The outcome e of a kernel launcher (ocb_kernels.h): a launch that succeeded is counted, one that failed is reported as the
// launch of `what`.
static int launched(ocb_ctx* ctx, const char* what, cudaError_t e) {
	if (e != cudaSuccess) return set_error(ctx, OCB_ERR_CUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
	ctx->launches++;
	return OCB_OK;
}

// ocb::grow on ctx's device (current) and stream, contents not kept
static int grow(ocb_ctx* ctx, DevBuf& b, size_t bytes) {
	const cudaError_t e = ocb::grow(b, bytes, ctx->stream);
	return e == cudaSuccess ? OCB_OK : set_error(ctx, OCB_ERR_CUDA, "growing a device buffer to %zu bytes failed: %s", bytes, cudaGetErrorString(e));
}

static int get_twiddles(ocb_ctx* ctx, int n, const float2** out) {
	auto it = ctx->twiddles.find(n);
	if (it != ctx->twiddles.end()) {
		*out = it->second;
		return OCB_OK;
	}
	std::vector<float2> h(n);
	for (int k = 0; k < n; k++) {
		double a = -2.0 * M_PI * (double)k / (double)n;
		h[k] = make_float2((float)cos(a), (float)sin(a));
	}
	float2* d = nullptr;
	OCB_CUDA(ctx, cudaMalloc(&d, sizeof(float2) * n));
	OCB_CUDA(ctx, cudaMemcpy(d, h.data(), sizeof(float2) * n, cudaMemcpyHostToDevice));
	ctx->twiddles[n] = d;
	*out = d;
	return OCB_OK;
}

static const size_t OCB_PIPE_MIN = 16384;
// Device-visible address of a host queue that is page-locked (cudaHostAlloc / cudaHostRegister / ocb_host_alloc), else NULL.
static float* mapped_queue(const void* host) {
	if (getenv("OCB_NO_ZEROCOPY")) return nullptr;
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, host) != cudaSuccess) {
		cudaGetLastError();
		return nullptr;
	}
	return (a.type == cudaMemoryTypeHost && a.devicePointer) ? (float*)a.devicePointer : nullptr;
}

static const int OCB_BANDS = 4;

// How a host-queue entry point moves its records:
//   entry point                                         pipeline  in_place                    band_ry
//   fftcc2d                                             yes       if the w32 kernel runs      ry
//   icgn2d1/2, icgn2d_ex (each radius group), iclm2d    yes       yes                         0
//   nr2d1                                               yes       no                          0
//   fftcc3d, icgn3d1, epipolar_search2d, strain         no        no                          0
struct QueuePolicy {
	// Queues of >= OCB_PIPE_MIN records are processed in 4 chunks on 4 internal streams (each chunk: H2D, kernel, D2H), which
	// hides most of the POI traffic behind the kernels.  Only for operators whose POIs are independent, so that results do not
	// depend on the split.
	bool pipeline;
	// A page-locked queue is not copied at all: the kernels read each record and write its results straight through PCIe, which
	// also keeps the copy engines free for the image upload.  Only for kernels that store a record with one coalesced write.
	bool in_place;
	// > 0: the call is FFT-CC with this y radius.  Right after a banded image upload, a chunk only waits for the bands its
	// windows touch.
	int band_ry;
};
static const QueuePolicy STAGED = { false, false, 0 }, PIPELINED = { true, false, 0 }, PIPELINED_IN_PLACE = { true, true, 0 };

// Host-queue driver: checks the arguments, runs dev_call(d_queue, count, first) over the n records of rec_floats floats in
// `host` as `policy` says, and returns once the results are back in `host`.  dev_call launches on ctx->stream with
// ctx->d_counter, both of which are redirected per chunk of a pipelined queue.  `what` names the entry point in errors.
template <class F>
static int run_host_queue(ocb_ctx* ctx, const char* what, void* host, size_t n, size_t rec_floats, F dev_call, QueuePolicy policy) {
	if (!ctx || (!host && n)) return set_error(ctx, OCB_ERR_ARG, "%s: bad arguments", what);
	if (n == 0) return OCB_OK;
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const size_t rec = rec_floats * sizeof(float);
	int rc;
	const bool banded = policy.band_ry > 0 && ctx->bands_fresh && ctx->stream == ctx->own_stream;
	ctx->bands_fresh = false;
	float* const mapped = policy.in_place ? mapped_queue(host) : nullptr;
	if (mapped && !(banded && n >= OCB_PIPE_MIN)) {
		if ((rc = dev_call(mapped, n, (size_t)0))) return rc;
		OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		return OCB_OK;
	}
	if (!policy.pipeline || n < OCB_PIPE_MIN || getenv("OCB_NO_PIPELINE")) {
		if ((rc = grow(ctx, ctx->d_poi, n * rec))) return rc;
		float* const d = ctx->d_poi.as<float>();
		OCB_CUDA(ctx, cudaMemcpyAsync(d, host, n * rec, cudaMemcpyHostToDevice, ctx->stream));
		if ((rc = dev_call(d, n, (size_t)0))) return rc;
		OCB_CUDA(ctx, cudaMemcpyAsync(host, d, n * rec, cudaMemcpyDeviceToHost, ctx->stream));
		OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		return OCB_OK;
	}
	if (!mapped && (rc = grow(ctx, ctx->d_poi, n * rec))) return rc;
	const int K = 4;
	if (!ctx->pipe_ready) {
		OCB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->pipe_ready, cudaEventDisableTiming));
		for (int i = 0; i < K; i++) OCB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->pipe[i], cudaStreamNonBlocking));
	}
	// everything enqueued so far on the caller-visible stream (image uploads, prepare, offsets) comes first
	OCB_CUDA(ctx, cudaEventRecord(ctx->pipe_ready, ctx->stream));
	cudaStream_t saved_stream = ctx->stream;
	int* saved_counter = ctx->d_counter;
	rc = OCB_OK;
	for (int c = 0; c < K && rc == OCB_OK; c++) {
		const size_t a = n * (size_t)c / K, b = n * (size_t)(c + 1) / K;
		if (b == a) continue;
		char* h = (char*)host + a * rec;
		float* d = (mapped ? mapped : ctx->d_poi.as<float>()) + a * rec_floats;
		cudaEvent_t gate = ctx->pipe_ready;
		if (banded) { // last image row this chunk's windows read: max over its POIs of max(y, y + v0) + r (src/oc_fftcc.cpp:204-219)
			float ymax = -1e30f;
			bool finite = true;
			const float* q = (const float*)h;
			for (size_t i = 0; i < b - a; i++) {
				const float y = q[i * OCB_POI2D_FLOATS + 1], v0 = q[i * OCB_POI2D_FLOATS + 2 + 6];
				const float top = y > y + v0 ? y : y + v0;
				if (!(top == top) || top > 1e9f) finite = false;
				ymax = top > ymax ? top : ymax;
			}
			if (finite) {
				const int need = (int)ymax + policy.band_ry + 1;
				for (int k = 0; k < OCB_BANDS; k++)
					if (ctx->band_end[k] >= need || k == OCB_BANDS - 1) { gate = ctx->band_done[k]; break; }
			}
		}
		cudaError_t e = cudaStreamWaitEvent(ctx->pipe[c], gate, 0);
		if (e == cudaSuccess && !mapped) e = cudaMemcpyAsync(d, h, (b - a) * rec, cudaMemcpyHostToDevice, ctx->pipe[c]);
		if (e != cudaSuccess) { rc = set_error(ctx, OCB_ERR_CUDA, "pipelined upload failed: %s", cudaGetErrorString(e)); break; }
		ctx->stream = ctx->pipe[c];
		ctx->d_counter = saved_counter + c;
		rc = dev_call(d, b - a, a);
		ctx->stream = saved_stream;
		ctx->d_counter = saved_counter;
		if (rc != OCB_OK) break;
		if (!mapped) {
			e = cudaMemcpyAsync(h, d, (b - a) * rec, cudaMemcpyDeviceToHost, ctx->pipe[c]);
			if (e != cudaSuccess) rc = set_error(ctx, OCB_ERR_CUDA, "pipelined download failed: %s", cudaGetErrorString(e));
		}
	}
	for (int c = 0; c < K; c++) {
		cudaError_t e = cudaStreamSynchronize(ctx->pipe[c]);
		if (e != cudaSuccess && rc == OCB_OK) rc = set_error(ctx, OCB_ERR_CUDA, "pipelined queue failed: %s", cudaGetErrorString(e));
	}
	return rc;
}


// ---- GROUP contexts: one process, several devices -------------------------------------------------------------------
static inline bool is_group(const ocb_ctx* ctx) { return ctx && !ctx->members.empty(); }

// The single-device context that holds the state of the calls a group does not shard (the series, SIFT3D, the calibration maps):
// the group's first member, or ctx itself.
static ocb_ctx* exec_member(ocb_ctx* ctx) { return is_group(ctx) ? ctx->members[0] : ctx; }

// A failure on the executing member of a group is reported on the group as well.
static int relay_error(ocb_ctx* ctx, const ocb_ctx* exec, int rc) {
	if (rc != OCB_OK && ctx != exec) {
		ctx->last_error = exec->last_error;
		g_last_error = ctx->last_error;
	}
	return rc;
}

// f(x) on the executing member x of ctx, its failure relayed to ctx
template <class F>
static int on_exec(ocb_ctx* ctx, F f) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	ocb_ctx* const x = exec_member(ctx);
	return relay_error(ctx, x, f(x));
}

// Run f(member, index) on the first `used` members concurrently (member 0 on the calling thread); first failure wins.
// (member, on its own thread) order the member's stream after every peer's image pushes, once per upload
static int member_settle(ocb_ctx* m) {
	if (!m->need_peer_wait) return OCB_OK;
	m->need_peer_wait = false;
	if (cudaSetDevice(m->device) != cudaSuccess) return set_error(m, OCB_ERR_CUDA, "cudaSetDevice failed");
	for (ocb_ctx* other : m->group->members)
		if (other != m && cudaStreamWaitEvent(m->stream, other->ev_pushed, 0) != cudaSuccess) return set_error(m, OCB_ERR_CUDA, "cudaStreamWaitEvent failed");
	return OCB_OK;
}

template <class F>
static int group_run(ocb_ctx* g, int used, F f) {
	if (used > (int)g->members.size()) used = (int)g->members.size();
	auto job = [f](ocb_ctx* m, int i) {
		const int rc = member_settle(m);
		return rc ? rc : f(m, i);
	};
	for (int i = 1; i < used; i++) {
		ocb_ctx* m = g->members[i];
		g->workers[i - 1]->post([job, m, i]() { return job(m, i); });
	}
	int rc = job(g->members[0], 0), bad = 0;
	for (int i = 1; i < used; i++) {
		const int r = g->workers[i - 1]->wait();
		if (rc == OCB_OK && r != OCB_OK) { rc = r; bad = i; }
	}
	if (rc != OCB_OK) {
		g->last_error = "device " + std::to_string(g->members[bad]->device) + ": " + g->members[bad]->last_error;
		g_last_error = g->last_error;
	}
	return rc;
}
template <class F>
static int group_each(ocb_ctx* g, F f) {
	return group_run(g, (int)g->members.size(), [f](ocb_ctx* m, int) { return f(m); });
}
// A prepare that only sets a flag runs on every member from the calling thread: no need to wake the members' threads.
static int prepare_members(ocb_ctx* g, int (*prepare)(ocb_ctx*)) {
	for (ocb_ctx* m : g->members) {
		const int rc = prepare(m);
		if (rc) { g->last_error = m->last_error; return rc; }
	}
	return OCB_OK;
}
// Contiguous block split of a host queue of n records of rec_bytes: member i gets records [n i / G, n (i+1) / G) and
// copies them in and out of the caller's array itself (its own PCIe link, straight into the caller's slice).  Queues
// too short to fill every device use fewer of them (min_per_device records each).  f(member, slice, count, first).
template <class F>
static int group_shard(ocb_ctx* g, void* queue, size_t n, size_t rec_bytes, size_t min_per_device, F f) {
	if (n == 0) return OCB_OK;
	size_t used = n / min_per_device;
	if (used < 1) used = 1;
	if (used > g->members.size()) used = g->members.size();
	const int G = (int)used;
	char* base = (char*)queue;
	return group_run(g, G, [=](ocb_ctx* m, int i) {
		const size_t a = n * (size_t)i / (size_t)G, b = n * (size_t)(i + 1) / (size_t)G;
		if (b == a) return (int)OCB_OK;
		return f(m, (void*)(base + a * rec_bytes), b - a, a);
	});
}
// Smallest shard worth a device.  2D: a launch that cannot fill the GPU lets two warps share a POI (icgn2d_launch), which splits
// its sums differently and changes the last bits of the result; shards of >= 8192 POIs take the same one-warp-per-POI path as
// the undivided queue on one device, so sharded results stay bit-identical.
// The epipolar search (OCB_GROUP_MIN_EPIPOLAR) registers every POI at each of its candidate slots.
static const size_t OCB_GROUP_MIN_2D = 8192, OCB_GROUP_MIN_3D = 64, OCB_GROUP_MIN_EPIPOLAR = 256;
#define OCB_NO_GROUP(ctx, what) \
	if (is_group(ctx)) return set_error(ctx, OCB_ERR_ARG, what ": device-pointer / stream entry points need a single-device context (ocb_member)")

static ocb_ctx* create_group(const int* devices, int n) {
	ocb_ctx* g = new ocb_ctx;
	g->device = -1;
	for (int i = 0; i < n; i++) {
		ocb_ctx* m = ocb_create(devices[i]);
		if (!m) {
			for (ocb_ctx* p : g->members) ocb_destroy(p);
			delete g;
			return nullptr; // ocb_create left the message in the process-wide slot
		}
		m->group = g;
		g->members.push_back(m);
	}
	for (int i = 1; i < n; i++) {
		ocb_worker* w = new ocb_worker;
		w->th = std::thread([w]() { w->loop(); });
		g->workers.push_back(w);
	}
	// peer access between all members (NVLink through NVSwitch on an HGX board): images are then uploaded once, in slices, and
	// exchanged between the devices instead of crossing PCIe once per device
	g->peer_ok = n > 1 && !getenv("OCB_NO_PEER");
	for (int i = 0; i < n && g->peer_ok; i++) {
		cudaSetDevice(devices[i]);
		for (int j = 0; j < n && g->peer_ok; j++) {
			if (i == j) continue;
			int can = 0;
			if (cudaDeviceCanAccessPeer(&can, devices[i], devices[j]) != cudaSuccess || !can) { g->peer_ok = false; break; }
			const cudaError_t e = cudaDeviceEnablePeerAccess(devices[j], 0);
			if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) g->peer_ok = false;
			cudaGetLastError();
		}
	}
	for (ocb_ctx* m : g->members) {
		cudaSetDevice(m->device);
		if (cudaEventCreateWithFlags(&m->ev_idle, cudaEventDisableTiming) != cudaSuccess
			|| cudaEventCreateWithFlags(&m->ev_pushed, cudaEventDisableTiming) != cudaSuccess)
			g->peer_ok = false;
	}
	cudaGetLastError();
	return g;
}

// Forget the image pair of dimension dim (2 or 3) and what was prepared on it, before its buffers are replaced: an upload that
// fails leaves no images rather than a view of freed memory.
static void clear_pair(ocb_ctx* ctx, int dim) {
	if (dim == 2) {
		ctx->img2 = ocb::Image2D{ nullptr, nullptr, 0, 0 };
		ctx->bands_fresh = ctx->prepared2 = ctx->prepared_nr2 = false;
	} else {
		ctx->img3 = ocb::Image3D{ nullptr, nullptr, nullptr, nullptr, 0, 0, 0 };
		ctx->prepared3 = false;
	}
}

// Image pair buffers of a single-device context (dim 2 or 3), each grown to `elems` floats; the pair is cleared first
static DevBuf* own_pair(ocb_ctx* ctx, int dim) { return dim == 2 ? ctx->own2 : ctx->own3; }
static int ensure_pair(ocb_ctx* ctx, int dim, size_t elems) {
	clear_pair(ctx, dim);
	DevBuf* pair = own_pair(ctx, dim);
	const int rc = grow(ctx, pair[0], elems * sizeof(float));
	return rc ? rc : grow(ctx, pair[1], elems * sizeof(float));
}

// GROUP upload of an image pair (elems floats each) into every member's buffers: member m copies ONLY slice m of both images
// from the host (its own PCIe link, all members concurrently), then pushes the slice to every other member over NVLink
// (cudaMemcpyPeerAsync); each member's stream finally waits for everybody's pushes.  Per device the PCIe traffic drops from the
// whole pair to 1/G of it; the exchange runs at NVLink rate through the switch.  dim: 2 or 3 (which buffers).
static int group_distribute_pair(ocb_ctx* g, const float* ref, const float* tar, size_t elems, int dim) {
	const int G = (int)g->members.size();
	int rc = OCB_OK;
	for (ocb_ctx* m : g->members) clear_pair(m, dim); // a failure on any member leaves the group without images
	for (ocb_ctx* m : g->members) { // buffers first: a peer may push into them as soon as the exchange starts
		if (ensure_device(m)) return OCB_ERR_CUDA;
		rc = ensure_pair(m, dim, elems);
		if (rc == OCB_OK && cudaEventRecord(m->ev_idle, m->stream) != cudaSuccess) rc = set_error(m, OCB_ERR_CUDA, "cudaEventRecord failed");
		if (rc) {
			g->last_error = m->last_error;
			return rc;
		}
	}
	const size_t gran = 64; // floats: slices start on 256-byte boundaries
	rc = group_run(g, G, [=](ocb_ctx* m, int i) {
		if (ensure_device(m)) return (int)OCB_ERR_CUDA;
		const size_t a = (elems * (size_t)i / (size_t)G) / gran * gran, b = i + 1 == G ? elems : (elems * (size_t)(i + 1) / (size_t)G) / gran * gran;
		const size_t len = (b - a) * sizeof(float);
		const DevBuf* mine = own_pair(m, dim);
		const float* src[2] = { ref, tar };
		if (len) {
			for (int k = 0; k < 2; k++) OCB_CUDA(m, cudaMemcpyAsync(mine[k].as<float>() + a, src[k] + a, len, cudaMemcpyHostToDevice, m->stream));
			for (int jj = 1; jj < G; jj++) { // start with the next neighbour so that the pushes of all members spread over the peers
				ocb_ctx* peer = g->members[(i + jj) % G];
				OCB_CUDA(m, cudaStreamWaitEvent(m->stream, peer->ev_idle, 0)); // the peer is done with its old images
				const DevBuf* theirs = own_pair(peer, dim);
				for (int k = 0; k < 2; k++)
					OCB_CUDA(m, cudaMemcpyPeerAsync(theirs[k].as<float>() + a, peer->device, mine[k].as<float>() + a, m->device, len, m->stream));
			}
		}
		OCB_CUDA(m, cudaEventRecord(m->ev_pushed, m->stream));
		return (int)OCB_OK;
	});
	if (rc) return rc;
	// nobody uses the pair before every slice has arrived: each member orders its stream after the peers' pushes at the start of
	// its next job, on its own thread (member_settle)
	for (ocb_ctx* m : g->members) m->need_peer_wait = true;
	return OCB_OK;
}

// ---- pair calls: one kernel family on the context's image or volume pair ------------------------------------------------
// The checks of a device-pointer pair call `what`, in this order: a group context is refused; bad arguments (a null context, a
// null queue with n > 0, or args_ok false: the call's radius or index checks failed); the call's own argument refusal, when
// `refusal` is set (epipolar: the search step); the image pair of dimension `dim` not set (0: the call reads none, strain); the
// prepare flag `prepared` not set (null: none needed).  Then n = 0 leaves nothing to do, and a `capped` call refuses n >= 2^31
// because its kernels index the queue with int (epipolar runs in blocks and has no cap).
// Returns the refusal, OCB_OK when there is nothing to do, or PAIR_GO with the context's device current.
static const int PAIR_GO = 1;
static int pair_checks(ocb_ctx* ctx, const char* what, const void* d_q, size_t n, bool args_ok, const char* refusal, int dim,
	bool ocb_ctx::*prepared, bool capped) {
	if (is_group(ctx))
		return set_error(ctx, OCB_ERR_ARG, "%s_dev: device-pointer / stream entry points need a single-device context (ocb_member)", what);
	if (!ctx || (!d_q && n) || !args_ok) return set_error(ctx, OCB_ERR_ARG, "%s: bad arguments", what);
	if (refusal) return set_error(ctx, OCB_ERR_ARG, "%s: %s", what, refusal);
	if ((dim == 2 && !ctx->img2.ref) || (dim == 3 && !ctx->img3.ref)) return set_error(ctx, OCB_ERR_STATE, "%s: images not set", what);
	if (prepared && !(ctx->*prepared)) return set_error(ctx, OCB_ERR_STATE, "%s: prepare() has not been called since setImages()", what);
	if (n == 0) return OCB_OK;
	if (capped && n > 0x7fffffffull) return set_error(ctx, OCB_ERR_ARG, "%s: too many POIs in one call", what);
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	return PAIR_GO;
}

// A host-queue pair call `what` over n records of rec_floats floats: on a group context (with a queue) each member takes a
// slice of at least min_per_device records; on a single-device context the call's own argument refusal (`refusal`, if set) comes
// first, then run_host_queue runs dev(x, d_queue, count) with `policy`.
template <class F>
static int pair_host(ocb_ctx* ctx, const char* what, const char* refusal, void* q, size_t n, size_t rec_floats, size_t min_per_device,
	QueuePolicy policy, F dev) {
	if (is_group(ctx) && q)
		return group_shard(ctx, q, n, rec_floats * sizeof(float), min_per_device, [&](ocb_ctx* m, void* slice, size_t count, size_t) {
			return pair_host(m, what, refusal, slice, count, rec_floats, min_per_device, policy, dev);
		});
	if (refusal) return set_error(ctx, OCB_ERR_ARG, "%s: %s", what, refusal);
	return run_host_queue(ctx, what, q, n, rec_floats, [&](float* d, size_t count, size_t) { return dev(ctx, d, count); }, policy);
}

// ---- series: the state and host staging shared by the image, volume and stereo series ---------------------------------
// Point s at a series (the _dev setters borrow the caller's device memory): see SeriesStore; tar1 is null but for the stereo series
static void series_borrow(SeriesStore& s, const float* ref, const void* tar0, const void* tar1, size_t pitch, int frames, int w, int h, int d) {
	s.ref = ref;
	s.tars[0] = tar0;
	s.tars[1] = tar1;
	s.pitch = pitch;
	s.frames = frames;
	s.w = w;
	s.h = h;
	s.d = d;
}
static void series_clear(SeriesStore& s) { series_borrow(s, nullptr, nullptr, nullptr, 0, 0, 0, 0, 0); }

// The host setters' upload, on the executing member x after their argument checks: s.own grows to a reference of w x h x d floats
// and n_stacks stacks of `frames` frames `pitch` bytes apart, the reference (unless ref is null: the caller fills own[0]) and
// every frame (frame_bytes each) are copied in, and s points at them.  s is cleared before any buffer is replaced, so a failure
// leaves no series, never a view of freed memory.
static int series_upload(ocb_ctx* x, SeriesStore& s, const float* ref, const void* const* stacks, int n_stacks, size_t frame_bytes, size_t pitch,
	int frames, int w, int h, int d) {
	if (ensure_device(x)) return OCB_ERR_CUDA;
	series_clear(s);
	const size_t ref_bytes = (size_t)w * h * d * sizeof(float);
	int rc = grow(x, s.own[0], ref_bytes);
	for (int k = 0; k < n_stacks && rc == OCB_OK; k++) rc = grow(x, s.own[1 + k], (size_t)frames * pitch);
	if (rc) return rc;
	if (ref) OCB_CUDA(x, cudaMemcpyAsync(s.own[0].p, ref, ref_bytes, cudaMemcpyHostToDevice, x->stream));
	for (int k = 0; k < n_stacks; k++) {
		char* const dst = s.own[1 + k].as<char>();
		const char* const src = (const char*)stacks[k];
		if (pitch == frame_bytes)
			OCB_CUDA(x, cudaMemcpyAsync(dst, src, (size_t)frames * pitch, cudaMemcpyHostToDevice, x->stream));
		else
			for (int f = 0; f < frames; f++)
				OCB_CUDA(x, cudaMemcpyAsync(dst + (size_t)f * pitch, src + (size_t)f * frame_bytes, frame_bytes, cudaMemcpyHostToDevice, x->stream));
	}
	series_borrow(s, s.own[0].as<float>(), s.own[1].p, n_stacks > 1 ? s.own[2].p : nullptr, pitch, frames, w, h, d);
	return OCB_OK;
}

// A call over n POIs is refused when the kernels could not index its POIs with int or a byte count of its frames x n records of
// rec bytes (per POI and frame, every output together) would not fit in a size_t; a host call (`staged`) also stages its inputs,
// at most one frame's worth.
static int series_size_check(ocb_ctx* x, const char* what, size_t n, int frames, size_t rec, bool staged) {
	if (n > 0x7fffffffull || (size_t)frames + (staged ? 1 : 0) > SIZE_MAX / (n * rec))
		return set_error(x, OCB_ERR_ARG, "%s: too many POIs in one call", what);
	return OCB_OK;
}

// A series call with host buffers, on the executing member x of ctx: the n records of in_floats floats of every input are
// staged on the device, dev(x, d_in, d_out) runs the call's _dev body on them, the frames x n records (frame-major) of every
// output {pointer, floats per record} come back, and the call returns after one synchronisation.  With n == 0, dev runs on null
// pointers for its argument checks only.  A failure writes nothing to the outputs and is reported on ctx too.
template <class F>
static int series_host(ocb_ctx* ctx, const char* what, SeriesStore ocb_ctx::*which, size_t n, std::initializer_list<const void*> in, size_t in_floats,
	std::initializer_list<std::pair<void*, size_t>> out, F dev) {
	return on_exec(ctx, [&](ocb_ctx* x) -> int {
		const float* d_in[3] = {};
		float* d_out[3] = {};
		size_t rec_floats = 0;
		bool ptrs = true;
		for (const void* h : in) ptrs = ptrs && h;
		for (const auto& o : out) {
			ptrs = ptrs && o.first;
			rec_floats += o.second;
		}
		if (!ptrs && n) return set_error(x, OCB_ERR_ARG, "%s: bad arguments", what);
		const SeriesStore& s = x->*which;
		if (!s.ref) return set_error(x, OCB_ERR_STATE, "%s: no series set", what);
		if (n == 0) return dev(x, d_in, d_out);
		int rc;
		if ((rc = series_size_check(x, what, n, s.frames, rec_floats * sizeof(float), true))) return rc;
		if (ensure_device(x)) return OCB_ERR_CUDA;
		const size_t frames = (size_t)s.frames;
		if ((rc = grow(x, x->d_poi, (in.size() * in_floats + frames * rec_floats) * n * sizeof(float)))) return rc;
		float* p = x->d_poi.as<float>(); // the inputs, then the outputs, back to back
		for (size_t k = 0; k < in.size(); p += n * in_floats, k++) {
			d_in[k] = p;
			OCB_CUDA(x, cudaMemcpyAsync(p, in.begin()[k], n * in_floats * sizeof(float), cudaMemcpyHostToDevice, x->stream));
		}
		for (size_t k = 0; k < out.size(); p += frames * n * out.begin()[k].second, k++) d_out[k] = p;
		if ((rc = dev(x, d_in, d_out))) return rc;
		for (size_t k = 0; k < out.size(); k++)
			OCB_CUDA(x, cudaMemcpyAsync(out.begin()[k].first, d_out[k], frames * n * out.begin()[k].second * sizeof(float), cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaStreamSynchronize(x->stream));
		return OCB_OK;
	});
}

// The re-seeding entry points: call(counts) counts into a zeroed vector with one entry per frame of the series `which` of ctx's
// executing member, and the counts go to `reseeded` only when it succeeds.  A device-pointer call (`dev`) is synchronised first.
template <class F>
static int series_reseed(ocb_ctx* ctx, SeriesStore ocb_ctx::*which, bool dev, size_t n, size_t* reseeded, F call) {
	const SeriesStore* s = ctx ? &(exec_member(ctx)->*which) : nullptr;
	std::vector<size_t> counts(s && s->ref ? s->frames : 0, 0);
	const int rc = call(counts.data());
	if (rc == OCB_OK && dev && n) OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (rc == OCB_OK && reseeded) memcpy(reseeded, counts.data(), counts.size() * sizeof(size_t));
	return rc;
}

extern "C" {

int ocb_device_count(void) {
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess) return set_error(nullptr, OCB_ERR_CUDA, "cudaGetDeviceCount failed: %s", cudaGetErrorString(e));
	return n;
}

ocb_ctx* ocb_create(int device) {
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess || n == 0) {
		set_error(nullptr, OCB_ERR_CUDA, "no usable CUDA device (%s); this engine has no CPU fallback",
			e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
		return nullptr;
	}
	if (device == -1) { // every visible device: a GROUP context
		std::vector<int> all(n);
		for (int i = 0; i < n; i++) all[i] = i;
		return n == 1 ? ocb_create(0) : create_group(all.data(), n);
	}
	if (device < 0 || device >= n) {
		set_error(nullptr, OCB_ERR_ARG, "device %d out of range [0,%d)", device, n);
		return nullptr;
	}
	ocb_ctx* ctx = new ocb_ctx;
	ctx->device = device;
	cudaDeviceProp prop;
	if ((e = cudaSetDevice(device)) != cudaSuccess || (e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess
		|| (e = cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking)) != cudaSuccess) {
		set_error(nullptr, OCB_ERR_CUDA, "context creation on device %d failed: %s", device, cudaGetErrorString(e));
		delete ctx;
		return nullptr;
	}
	if (prop.major != 9 || prop.minor != 0) { // sm_90a code runs on compute capability 9.0 only
		set_error(nullptr, OCB_ERR_CUDA, "device %d is sm_%d%d; this library ships sm_90a code only", device, prop.major, prop.minor);
		cudaStreamDestroy(ctx->own_stream);
		delete ctx;
		return nullptr;
	}
	ctx->stream = ctx->own_stream;
	ctx->sm_count = prop.multiProcessorCount;
	ctx->smem_optin = prop.sharedMemPerBlockOptin;
	// work-queue heads: [0, 16) are zeroed by a memset in front of every launch that uses one; [32, 48) belong to the kernels that
	// reset their head themselves (icgn2d, one warp per POI) and are zeroed once, here
	if ((e = cudaMalloc(&ctx->d_counter, 64 * sizeof(int))) != cudaSuccess || (e = cudaMemset(ctx->d_counter, 0, 64 * sizeof(int))) != cudaSuccess) {
		set_error(nullptr, OCB_ERR_CUDA, "context creation on device %d failed: %s", device, cudaGetErrorString(e));
		cudaStreamDestroy(ctx->own_stream);
		delete ctx;
		return nullptr;
	}
	return ctx;
}

ocb_ctx* ocb_create_multi(const int* devices, int n_devices) {
	if (!devices || n_devices < 1) {
		set_error(nullptr, OCB_ERR_ARG, "create_multi: need at least one device");
		return nullptr;
	}
	for (int i = 0; i < n_devices; i++)
		for (int j = 0; j < i; j++)
			if (devices[i] == devices[j]) {
				set_error(nullptr, OCB_ERR_ARG, "create_multi: device %d listed twice", devices[i]);
				return nullptr;
			}
	return create_group(devices, n_devices);
}

int ocb_member_count(const ocb_ctx* ctx) { return !ctx ? 0 : (is_group(ctx) ? (int)ctx->members.size() : 1); }

ocb_ctx* ocb_member(ocb_ctx* ctx, int index) {
	if (!ctx) return nullptr;
	if (!is_group(ctx)) return index == 0 ? ctx : nullptr;
	if (index < 0 || index >= (int)ctx->members.size()) return nullptr;
	member_settle(ctx->members[index]); // the caller may go on with device-pointer calls on this member: its images must be complete
	return ctx->members[index];
}

void* ocb_host_alloc_on(ocb_ctx* ctx, size_t bytes) {
	if (ctx) {
		const ocb_ctx* c = is_group(ctx) ? ctx->members[0] : ctx;
		if (cudaSetDevice(c->device) != cudaSuccess) {
			cudaGetLastError();
			return nullptr;
		}
	}
	return ocb_host_alloc(bytes);
}

void* ocb_host_alloc(size_t bytes) {
	if (!bytes) return nullptr;
	void* p = nullptr;
	cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocPortable);
	if (e != cudaSuccess) {
		cudaGetLastError();
		set_error(nullptr, OCB_ERR_CUDA, "cudaHostAlloc failed: %s", cudaGetErrorString(e));
		return nullptr;
	}
	return p;
}

void ocb_host_free(void* host) {
	if (host) cudaFreeHost(host);
}

int ocb_host_register(void* host, size_t bytes) {
	if (!host || !bytes) return set_error(nullptr, OCB_ERR_ARG, "host_register: bad arguments");
	cudaError_t e = cudaHostRegister(host, bytes, cudaHostRegisterPortable);
	if (e != cudaSuccess) {
		cudaGetLastError();
		return set_error(nullptr, OCB_ERR_CUDA, "cudaHostRegister failed: %s", cudaGetErrorString(e));
	}
	return OCB_OK;
}

int ocb_host_unregister(void* host) {
	if (!host) return set_error(nullptr, OCB_ERR_ARG, "host_unregister: bad arguments");
	cudaError_t e = cudaHostUnregister(host);
	if (e != cudaSuccess) {
		cudaGetLastError();
		return set_error(nullptr, OCB_ERR_CUDA, "cudaHostUnregister failed: %s", cudaGetErrorString(e));
	}
	return OCB_OK;
}

void ocb_destroy(ocb_ctx* ctx) {
	if (!ctx) return;
	if (is_group(ctx)) {
		for (ocb_worker* w : ctx->workers) {
			{
				std::lock_guard<std::mutex> lk(w->mu);
				w->stop = true;
			}
			w->cv.notify_all();
			w->th.join();
			delete w;
		}
		for (ocb_ctx* m : ctx->members) {
			cudaSetDevice(m->device);
			if (m->ev_idle) cudaEventDestroy(m->ev_idle);
			if (m->ev_pushed) cudaEventDestroy(m->ev_pushed);
			ocb_destroy(m);
		}
		delete ctx;
		return;
	}
	cudaSetDevice(ctx->device);
	cudaDeviceSynchronize();
	for (auto& kv : ctx->twiddles) cudaFree(kv.second);
	for (int i = 0; i < 4; i++)
		if (ctx->pipe[i]) cudaStreamDestroy(ctx->pipe[i]);
	if (ctx->pipe_ready) cudaEventDestroy(ctx->pipe_ready);
	for (int i = 0; i < 4; i++)
		if (ctx->band_done[i]) cudaEventDestroy(ctx->band_done[i]);
	cudaFree(ctx->d_counter);
	delete ctx->sift3d;
	cudaStreamDestroy(ctx->own_stream);
	delete ctx; // frees the DevBuf members on this device
}

const char* ocb_last_error(const ocb_ctx* ctx) { return ctx ? ctx->last_error.c_str() : g_last_error.c_str(); }

int ocb_set_stream(ocb_ctx* ctx, void* cuda_stream) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	OCB_NO_GROUP(ctx, "set_stream");
	ctx->stream = (cudaStream_t)cuda_stream;
	return OCB_OK;
}

int ocb_use_own_stream(ocb_ctx* ctx) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	if (is_group(ctx)) return OCB_OK;
	ctx->stream = ctx->own_stream;
	return OCB_OK;
}

int ocb_sync(ocb_ctx* ctx) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	if (is_group(ctx)) return group_each(ctx, [](ocb_ctx* m) { return ocb_sync(m); });
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return OCB_OK;
}

long long ocb_launch_count(const ocb_ctx* ctx) {
	if (!ctx) return 0;
	long long total = ctx->launches;
	for (const ocb_ctx* m : ctx->members) total += m->launches;
	return total;
}

// ---- images ----------------------------------------------------------------------------------
int ocb_set_images_2d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tar, int width, int height) {
	OCB_NO_GROUP(ctx, "set_images_2d_dev");
	if (!ctx || !d_ref || !d_tar || width < 5 || height < 5) return set_error(ctx, OCB_ERR_ARG, "set_images_2d: bad arguments");
	ctx->img2 = ocb::Image2D{ d_ref, d_tar, width, height };
	ctx->bands_fresh = false;
	ctx->prepared2 = false;
	ctx->prepared_nr2 = false;
	return OCB_OK;
}

int ocb_set_images_2d(ocb_ctx* ctx, const float* ref, const float* tar, int width, int height, int col_major) {
	if (is_group(ctx)) {
		if (ctx->peer_ok && !col_major && ref && tar && width >= 5 && height >= 5) {
			int rc = group_distribute_pair(ctx, ref, tar, (size_t)width * height, 2);
			if (rc) return rc;
			for (ocb_ctx* m : ctx->members)
				if ((rc = ocb_set_images_2d_dev(m, m->own2[0].as<float>(), m->own2[1].as<float>(), width, height))) return rc;
			return OCB_OK;
		}
		return group_each(ctx, [=](ocb_ctx* m) { return ocb_set_images_2d(m, ref, tar, width, height, col_major); });
	}
	if (!ctx || !ref || !tar || width < 5 || height < 5) return set_error(ctx, OCB_ERR_ARG, "set_images_2d: bad arguments");
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const size_t elems = (size_t)width * height;
	{
		const int rcb = ensure_pair(ctx, 2, elems);
		if (rcb) return rcb;
	}
	float* const own_ref = ctx->own2[0].as<float>();
	float* const own_tar = ctx->own2[1].as<float>();
	bool banded = false;
	if (!col_major) {
		if (ctx->stream == ctx->own_stream && elems >= ((size_t)1 << 20) && !getenv("OCB_NO_PIPELINE")) {
			for (int b = 0; b < OCB_BANDS; b++) {
				if (!ctx->band_done[b]) OCB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->band_done[b], cudaEventDisableTiming));
				const size_t r0 = (size_t)height * b / OCB_BANDS, r1 = (size_t)height * (b + 1) / OCB_BANDS;
				const size_t off = r0 * (size_t)width, len = (r1 - r0) * (size_t)width * sizeof(float);
				OCB_CUDA(ctx, cudaMemcpyAsync(own_ref + off, ref + off, len, cudaMemcpyHostToDevice, ctx->stream));
				OCB_CUDA(ctx, cudaMemcpyAsync(own_tar + off, tar + off, len, cudaMemcpyHostToDevice, ctx->stream));
				OCB_CUDA(ctx, cudaEventRecord(ctx->band_done[b], ctx->stream));
				ctx->band_end[b] = (int)r1;
			}
			banded = true;
		} else {
			OCB_CUDA(ctx, cudaMemcpyAsync(own_ref, ref, elems * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
			OCB_CUDA(ctx, cudaMemcpyAsync(own_tar, tar, elems * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
		}
	} else {
		DevBuf tmp; // freed on every way out of this block
		const int rct = grow(ctx, tmp, elems * sizeof(float));
		if (rct) return rct;
		dim3 grid((width + 31) / 32, (height + 31) / 32), block(32, 8);
		const float* src[2] = { ref, tar };
		float* dst[2] = { own_ref, own_tar };
		for (int i = 0; i < 2; i++) {
			OCB_CUDA(ctx, cudaMemcpyAsync(tmp.p, src[i], elems * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
			ocb::transpose_kernel<<<grid, block, 0, ctx->stream>>>(tmp.as<float>(), dst[i], width, height);
			ctx->launches++;
		}
		OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	const int rc_dev = ocb_set_images_2d_dev(ctx, own_ref, own_tar, width, height);
	ctx->bands_fresh = banded && rc_dev == OCB_OK;
	return rc_dev;
}

// upload `elems` bytes twice (ref, tar) and widen into the context-owned float pair of dimension `dim`
static int upload_u8_pair(ocb_ctx* ctx, const unsigned char* ref, const unsigned char* tar, size_t elems, int dim) {
	int rc = ensure_pair(ctx, dim, elems);
	if (rc) return rc;
	// the widening kernel reads uchar4: the second image starts at a 16-byte aligned offset whatever the pixel count
	const size_t tar_off = (elems + 15) & ~(size_t)15;
	if ((rc = grow(ctx, ctx->d_u8, tar_off + elems))) return rc;
	unsigned char* const d_u8 = ctx->d_u8.as<unsigned char>();
	const DevBuf* dst = own_pair(ctx, dim);
	OCB_CUDA(ctx, cudaMemcpyAsync(d_u8, ref, elems, cudaMemcpyHostToDevice, ctx->stream));
	OCB_CUDA(ctx, cudaMemcpyAsync(d_u8 + tar_off, tar, elems, cudaMemcpyHostToDevice, ctx->stream));
	const int grid = ctx->sm_count * 8;
	ocb::widen_u8_kernel<<<grid, 256, 0, ctx->stream>>>(d_u8, dst[0].as<float>(), elems);
	ocb::widen_u8_kernel<<<grid, 256, 0, ctx->stream>>>(d_u8 + tar_off, dst[1].as<float>(), elems);
	ctx->launches += 2;
	OCB_CUDA(ctx, cudaGetLastError());
	return OCB_OK;
}

int ocb_set_images_2d_u8(ocb_ctx* ctx, const unsigned char* ref, const unsigned char* tar, int width, int height) {
	if (is_group(ctx)) return group_each(ctx, [=](ocb_ctx* m) { return ocb_set_images_2d_u8(m, ref, tar, width, height); });
	if (!ctx || !ref || !tar || width < 5 || height < 5) return set_error(ctx, OCB_ERR_ARG, "set_images_2d_u8: bad arguments");
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	int rc = upload_u8_pair(ctx, ref, tar, (size_t)width * height, 2);
	if (rc) return rc;
	return ocb_set_images_2d_dev(ctx, ctx->own2[0].as<float>(), ctx->own2[1].as<float>(), width, height);
}

int ocb_set_images_3d_u8(ocb_ctx* ctx, const unsigned char* ref, const unsigned char* tar, int dim_x, int dim_y, int dim_z) {
	if (is_group(ctx)) return group_each(ctx, [=](ocb_ctx* m) { return ocb_set_images_3d_u8(m, ref, tar, dim_x, dim_y, dim_z); });
	if (!ctx || !ref || !tar || dim_x < 15 || dim_y < 15 || dim_z < 15)
		return set_error(ctx, OCB_ERR_ARG, "set_images_3d_u8: bad arguments (each dimension must be >= 15)");
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	int rc = upload_u8_pair(ctx, ref, tar, (size_t)dim_x * dim_y * dim_z, 3);
	if (rc) return rc;
	return ocb_set_images_3d_dev(ctx, ctx->own3[0].as<float>(), ctx->own3[1].as<float>(), dim_x, dim_y, dim_z);
}

int ocb_set_images_3d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tar, int dim_x, int dim_y, int dim_z) {
	OCB_NO_GROUP(ctx, "set_images_3d_dev");
	if (!ctx || !d_ref || !d_tar || dim_x < 15 || dim_y < 15 || dim_z < 15) // TricubicBspline needs >= 15 (src/oc_cubic_bspline.cpp:201)
		return set_error(ctx, OCB_ERR_ARG, "set_images_3d: bad arguments (each dimension must be >= 15)");
	ctx->img3 = ocb::Image3D{ d_ref, d_tar, nullptr, nullptr, dim_x, dim_y, dim_z };
	ctx->prepared3 = false;
	return OCB_OK;
}

int ocb_set_images_3d(ocb_ctx* ctx, const float* ref, const float* tar, int dim_x, int dim_y, int dim_z) {
	if (is_group(ctx)) {
		if (ctx->peer_ok && ref && tar && dim_x >= 15 && dim_y >= 15 && dim_z >= 15) {
			int rc = group_distribute_pair(ctx, ref, tar, (size_t)dim_x * dim_y * dim_z, 3);
			if (rc) return rc;
			for (ocb_ctx* m : ctx->members)
				if ((rc = ocb_set_images_3d_dev(m, m->own3[0].as<float>(), m->own3[1].as<float>(), dim_x, dim_y, dim_z))) return rc;
			return OCB_OK;
		}
		return group_each(ctx, [=](ocb_ctx* m) { return ocb_set_images_3d(m, ref, tar, dim_x, dim_y, dim_z); });
	}
	if (!ctx || !ref || !tar || dim_x < 15 || dim_y < 15 || dim_z < 15)
		return set_error(ctx, OCB_ERR_ARG, "set_images_3d: bad arguments (each dimension must be >= 15)");
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const size_t elems = (size_t)dim_x * dim_y * dim_z;
	const int rc = ensure_pair(ctx, 3, elems);
	if (rc) return rc;
	float* const own_ref = ctx->own3[0].as<float>();
	float* const own_tar = ctx->own3[1].as<float>();
	OCB_CUDA(ctx, cudaMemcpyAsync(own_ref, ref, elems * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	OCB_CUDA(ctx, cudaMemcpyAsync(own_tar, tar, elems * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	return ocb_set_images_3d_dev(ctx, own_ref, own_tar, dim_x, dim_y, dim_z);
}

// ---- FFT-CC ----------------------------------------------------------------------------------
// Which FFT-CC kernel runs: W32 is the register-FFT kernel specialised for the 32-point window (r = 16 on every axis), REG the
// register FFT codelets for square / cubic windows of N = 2^a 3^b 5^c <= 64 points, GENERIC the shared-memory kernel for any
// window whose prime factors are <= 31.  OCB_FFTCC2D_GENERIC / OCB_FFTCC3D_GENERIC select GENERIC for every window; the choice
// is ocb::fftcc2d_plan / ocb::fftcc3d_plan (ocb_kernels.h).

// CTAs of a launch over n POIs (n >= 1): enough for the queue at pois_per_cta POIs per CTA, at most the plan's full launch
static int fftcc_grid(size_t n, int pois_per_cta, int ctas) {
	const size_t need = (n + pois_per_cta - 1) / pois_per_cta;
	const int grid = need < (size_t)ctas ? (int)need : ctas;
	return grid < 1 ? 1 : grid;
}

// The kernel that takes a (2rx x 2ry) window, or OCB_ERR_UNSUPPORTED with the reason none does.
static int fftcc2d_plan_or_error(ocb_ctx* ctx, int rx, int ry, ocb::Fftcc2dPlan* plan) {
	if (ocb::fftcc2d_plan(rx, ry, getenv("OCB_FFTCC2D_GENERIC") != nullptr, ctx->smem_optin, plan)) return OCB_OK;
	if (plan->reject == ocb::Fftcc2dReject::PRIME_FACTOR)
		return set_error(ctx, OCB_ERR_UNSUPPORTED, "fftcc2d: window size %dx%d has a prime factor > 31", 2 * rx, 2 * ry);
	return set_error(ctx, OCB_ERR_UNSUPPORTED, "fftcc2d: %dx%d window needs %zu B of shared memory (> %zu)", 2 * rx, 2 * ry, plan->smem,
		ctx->smem_optin);
}

// FFT-CC of the n device records q (1 <= n < 2^31) against img, on ctx's device (current) and stream.  The pair calls pass their
// image pair, the re-seeding series calls one frame of the series.
static int fftcc2d_run(ocb_ctx* ctx, const ocb::Image2D& img, float* q, size_t n, int rx, int ry) {
	ocb::Fftcc2dPlan plan;
	if (const int rc = fftcc2d_plan_or_error(ctx, rx, ry, &plan)) return rc;
	const int grid = fftcc_grid(n, plan.pois_per_cta, ctx->sm_count * plan.ctas_per_sm);
	if (plan.path == ocb::Fftcc2dPath::W32) return launched(ctx, "fftcc2d", ocb::fftcc2d_w32_launch(img, q, n, grid, ctx->stream));
	if (plan.path == ocb::Fftcc2dPath::REG) return launched(ctx, "fftcc2d", ocb::fftcc2d_reg_launch(img, q, n, rx, plan, grid, ctx->stream));
	const float2 *twx, *twy;
	int rc;
	if ((rc = get_twiddles(ctx, 2 * rx, &twx)) || (rc = get_twiddles(ctx, 2 * ry, &twy))) return rc;
	return launched(ctx, "fftcc2d", ocb::fftcc2d_launch(img, q, n, rx, ry, plan, twx, twy, grid, ctx->stream));
}

int ocb_fftcc2d_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, int rx, int ry) {
	const int rc = pair_checks(ctx, "fftcc2d", d_poi2d, n, rx >= 1 && ry >= 1, nullptr, 2, nullptr, true);
	return rc == PAIR_GO ? fftcc2d_run(ctx, ctx->img2, (float*)d_poi2d, n, rx, ry) : rc;
}

int ocb_fftcc2d(ocb_ctx* ctx, void* poi2d, size_t n, int rx, int ry) {
	ocb::Fftcc2dPlan plan; // only the w32 kernel stores a record with one coalesced write
	const bool w32 = rx >= 1 && ry >= 1 && ocb::fftcc2d_plan(rx, ry, getenv("OCB_FFTCC2D_GENERIC") != nullptr, (size_t)-1, &plan) && plan.path == ocb::Fftcc2dPath::W32;
	const QueuePolicy policy = { true, w32, ry > 0 ? ry : 0 };
	return pair_host(ctx, "fftcc2d", nullptr, poi2d, n, OCB_POI2D_FLOATS, OCB_GROUP_MIN_2D, policy,
		[=](ocb_ctx* x, float* d, size_t m) { return ocb_fftcc2d_dev(x, d, m, rx, ry); });
}

// The kernel that takes a (2rx x 2ry x 2rz) window, with its grid and scratch per CTA, or OCB_ERR_UNSUPPORTED with the reason none
// does.  The kernels index the window with int: it has fewer than 2^31 points.
static int fftcc3d_plan_or_error(ocb_ctx* ctx, int rx, int ry, int rz, ocb::Fftcc3dPlan* plan) {
	if ((size_t)8 * rx * ry * rz > 0x7fffffffull) return set_error(ctx, OCB_ERR_UNSUPPORTED, "fftcc3d: window too large");
	if (ocb::fftcc3d_plan(rx, ry, rz, getenv("OCB_FFTCC3D_GENERIC") != nullptr, ctx->smem_optin, ctx->sm_count, plan)) return OCB_OK;
	if (plan->reject == ocb::Fftcc3dReject::PRIME_FACTOR) return set_error(ctx, OCB_ERR_UNSUPPORTED, "fftcc3d: window size has a prime factor > 31");
	return set_error(ctx, OCB_ERR_UNSUPPORTED, "fftcc3d: window needs %zu B of shared memory (> %zu)", plan->smem, ctx->smem_optin);
}

// FFT-CC of the n device records q (1 <= n < 2^31) against img.ref / img.tar, on ctx's device (current) and stream, with
// ctx->fft_scratch.  The pair calls pass their volume pair, the re-seeding series call one frame of the series.
static int fftcc3d_run(ocb_ctx* ctx, const ocb::Image3D& img, float* q, size_t n, int rx, int ry, int rz) {
	ocb::Fftcc3dPlan plan;
	int rc;
	if ((rc = fftcc3d_plan_or_error(ctx, rx, ry, rz, &plan))) return rc;
	const float2 *twx = nullptr, *twy = nullptr, *twz = nullptr;
	if (plan.path == ocb::Fftcc3dPath::GENERIC
		&& ((rc = get_twiddles(ctx, 2 * rx, &twx)) || (rc = get_twiddles(ctx, 2 * ry, &twy)) || (rc = get_twiddles(ctx, 2 * rz, &twz))))
		return rc;
	const int grid = fftcc_grid(n, 1, plan.ctas);
	if ((rc = grow(ctx, ctx->fft_scratch, (size_t)grid * plan.cta_scratch * sizeof(float2)))) return rc;
	float2* const scratch = ctx->fft_scratch.as<float2>();
	if (plan.path == ocb::Fftcc3dPath::W32) return launched(ctx, "fftcc3d", ocb::fftcc3d_w32_launch(img, q, n, plan, scratch, grid, ctx->stream));
	if (plan.path == ocb::Fftcc3dPath::REG) return launched(ctx, "fftcc3d", ocb::fftcc3d_reg_launch(img, q, n, plan, scratch, grid, ctx->stream));
	return launched(ctx, "fftcc3d", ocb::fftcc3d_launch(img, q, n, rx, ry, rz, plan, twx, twy, twz, scratch, grid, ctx->stream));
}

int ocb_fftcc3d_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, int rx, int ry, int rz) {
	const int rc = pair_checks(ctx, "fftcc3d", d_poi3d, n, rx >= 1 && ry >= 1 && rz >= 1, nullptr, 3, nullptr, true);
	return rc == PAIR_GO ? fftcc3d_run(ctx, ctx->img3, (float*)d_poi3d, n, rx, ry, rz) : rc;
}

int ocb_fftcc3d(ocb_ctx* ctx, void* poi3d, size_t n, int rx, int ry, int rz) {
	return pair_host(ctx, "fftcc3d", nullptr, poi3d, n, OCB_POI3D_FLOATS, OCB_GROUP_MIN_3D, STAGED,
		[=](ocb_ctx* x, float* d, size_t m) { return ocb_fftcc3d_dev(x, d, m, rx, ry, rz); });
}

// ---- IC-GN -----------------------------------------------------------------------------------
int ocb_icgn2d_prepare(ocb_ctx* ctx) {
	if (is_group(ctx)) return prepare_members(ctx, ocb_icgn2d_prepare);
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	if (!ctx->img2.ref) return set_error(ctx, OCB_ERR_STATE, "icgn2d_prepare: images not set");
	ctx->prepared2 = true; // gradients and bicubic weights are recomputed on chip per POI
	return OCB_OK;
}

// The launch geometry of IC-GN (lm: IC-LM) with np shape parameters over n >= 1 POIs, or OCB_ERR_UNSUPPORTED when the radius does not
// fit in shared memory.  The warps per POI are those of a launch over plan_n POIs: n for a plain call; a re-seeded sub-queue
// passes the length of the whole queue, so that its POIs split their sums as they do in the launch over all of them.  The image
// series launches take the same plan, so a frame splits its sums as a pair call over the same POIs does.  The grid never
// exceeds n.  OCB_ICGN2D_WPP = 1 or 2 forces the warps per POI (a tuning knob, read at every call).
static int icgn2d_plan_or_error(ocb_ctx* ctx, size_t n, size_t plan_n, int np, int rx, int ry, bool lm, ocb::Icgn2dPlan* plan) {
	const char* wpp = getenv("OCB_ICGN2D_WPP");
	if (!ocb::icgn2d_plan(plan_n, np, rx, ry, lm, ctx->sm_count, ctx->smem_optin, wpp ? atoi(wpp) : 0, plan))
		return set_error(ctx, OCB_ERR_UNSUPPORTED, "icgn2d: subset radius (%d,%d) exceeds the shared-memory design limit", rx, ry);
	if ((size_t)plan->grid > n) plan->grid = (int)n;
	return OCB_OK;
}

// IC-GN (lm_damping: IC-LM) of the n device records q (1 <= n < 2^31) against img, on ctx's device (current) and stream, with the
// warps per POI of a launch over plan_n POIs (icgn2d_plan_or_error).
static int icgn2d_run(ocb_ctx* ctx, int np, const ocb::Image2D& img, float* q, size_t n, size_t plan_n, int rx, int ry, float conv, float stop,
	const float* d_offsets, const float* lm_damping) {
	ocb::Icgn2dPlan plan;
	if (const int rc = icgn2d_plan_or_error(ctx, n, plan_n, np, rx, ry, lm_damping != nullptr, &plan)) return rc;
	return launched(ctx, "icgn2d", ocb::icgn2d_launch(np, plan, img, q, n, rx, ry, conv, stop, ctx->d_counter, d_offsets, lm_damping, ctx->stream));
}

static int icgn2d_dev(ocb_ctx* ctx, int np, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop, const float* d_offsets = nullptr,
	const float* lm_damping = nullptr) {
	const int rc = pair_checks(ctx, "icgn2d", d_poi2d, n, rx >= 1 && ry >= 1, nullptr, 2, &ocb_ctx::prepared2, true);
	return rc == PAIR_GO ? icgn2d_run(ctx, np, ctx->img2, (float*)d_poi2d, n, n, rx, ry, conv, stop, d_offsets, lm_damping) : rc;
}

int ocb_icgn2d1_dev(ocb_ctx* ctx, void* d, size_t n, int rx, int ry, float conv, float stop) { return icgn2d_dev(ctx, 6, d, n, rx, ry, conv, stop); }
int ocb_icgn2d2_dev(ocb_ctx* ctx, void* d, size_t n, int rx, int ry, float conv, float stop) { return icgn2d_dev(ctx, 12, d, n, rx, ry, conv, stop); }

static int icgn2d_host(ocb_ctx* ctx, int np, void* poi2d, size_t n, int rx, int ry, float conv, float stop) {
	return pair_host(ctx, "icgn2d", nullptr, poi2d, n, OCB_POI2D_FLOATS, OCB_GROUP_MIN_2D, PIPELINED_IN_PLACE,
		[=](ocb_ctx* x, float* d, size_t m) { return icgn2d_dev(x, np, d, m, rx, ry, conv, stop); });
}
int ocb_icgn2d1(ocb_ctx* ctx, void* p, size_t n, int rx, int ry, float conv, float stop) { return icgn2d_host(ctx, 6, p, n, rx, ry, conv, stop); }
int ocb_icgn2d2(ocb_ctx* ctx, void* p, size_t n, int rx, int ry, float conv, float stop) { return icgn2d_host(ctx, 12, p, n, rx, ry, conv, stop); }

int ocb_icgn2d_ex_dev(ocb_ctx* ctx, int order, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop, const float* d_center_offsets) {
	if (order != 1 && order != 2) return set_error(ctx, OCB_ERR_ARG, "icgn2d_ex: order must be 1 or 2");
	return icgn2d_dev(ctx, order == 1 ? 6 : 12, d_poi2d, n, rx, ry, conv, stop, d_center_offsets);
}

// ---- image series: one reference, n_frames targets, each frame seeded by the previous one ------------------------------
// On a group context the first member holds the series and runs it.

int ocb_set_series_2d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tars, int n_frames, int width, int height) {
	OCB_NO_GROUP(ctx, "set_series_2d_dev");
	if (!ctx || !d_ref || !d_tars || n_frames < 1 || width < 5 || height < 5) return set_error(ctx, OCB_ERR_ARG, "set_series_2d: bad arguments");
	series_borrow(ctx->series2d, d_ref, d_tars, nullptr, (size_t)width * height * sizeof(float), n_frames, width, height, 1);
	return OCB_OK;
}

int ocb_set_series_2d(ocb_ctx* ctx, const float* ref, const float* tars, int n_frames, int width, int height) {
	return on_exec(ctx, [&](ocb_ctx* x) {
		if (!ref || !tars || n_frames < 1 || width < 5 || height < 5) return set_error(x, OCB_ERR_ARG, "set_series_2d: bad arguments");
		const size_t frame = (size_t)width * height * sizeof(float);
		if ((size_t)n_frames > SIZE_MAX / frame) return set_error(x, OCB_ERR_ARG, "set_series_2d: series too large");
		const void* stack[1] = { tars };
		return series_upload(x, x->series2d, ref, stack, 1, frame, frame, n_frames, width, height, 1);
	});
}

// What a series call that re-seeds lost POIs adds to the plain series (a null SeriesReseed: the plain series).  POI i is lost in
// frame f when its frame-f record has !(zncc >= zncc_min); its record is then rebuilt from the seed with the translation of its
// latest good record (the seed's without one), and FFT-CC (radii fft_r) and IC-GN run on it against that frame.  The result
// replaces the frame-f record and seeds frame f + 1.  counts[f]: the POIs re-seeded in frame f.
struct SeriesReseed {
	int fft_r[3];
	float zncc_min;
	size_t* counts; // n_frames host counts, zero on entry
};

// Argument checks shared by the re-seeding entry points (the FFT-CC window is checked against the plan of the pair call)
static int reseed_check(ocb_ctx* ctx, const char* what, int dim, const SeriesReseed& rs) {
	if (rs.zncc_min != rs.zncc_min) return set_error(ctx, OCB_ERR_ARG, "%s: zncc_min is NaN", what);
	for (int a = 0; a < dim; a++)
		if (rs.fft_r[a] < 1) return set_error(ctx, OCB_ERR_ARG, "%s: FFT-CC radii must be >= 1", what);
	if (dim == 2) {
		ocb::Fftcc2dPlan plan;
		return fftcc2d_plan_or_error(ctx, rs.fft_r[0], rs.fft_r[1], &plan);
	}
	ocb::Fftcc3dPlan plan;
	return fftcc3d_plan_or_error(ctx, rs.fft_r[0], rs.fft_r[1], rs.fft_r[2], &plan);
}

// Device workspace of a re-seeding call over n POIs and `frames` frames (ctx->reseed_ws): each POI's first lost frame, the
// compacted sub-queue indices, the per-frame histogram of first lost frames, the sub-queue length, dim anchor floats per POI
// and the compaction's temporary storage.
struct ReseedWs {
	int *first, *idx, *hist, *count;
	float* anchor;
	void* temp;
	size_t temp_bytes;
	std::vector<int> h_hist;
};
static int reseed_workspace(ocb_ctx* ctx, size_t n, int frames, int dim, ReseedWs* w) {
	auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
	w->temp_bytes = ocb::reseed_select_bytes(n);
	const size_t o_idx = up(n * sizeof(int)), o_hist = o_idx + up(n * sizeof(int)), o_count = o_hist + up((size_t)frames * sizeof(int));
	const size_t o_anchor = o_count + 256, o_temp = o_anchor + up(n * dim * sizeof(float));
	if (const int rc = grow(ctx, ctx->reseed_ws, o_temp + up(w->temp_bytes))) return rc;
	char* const b = ctx->reseed_ws.as<char>();
	w->first = (int*)b;
	w->idx = (int*)(b + o_idx);
	w->hist = (int*)(b + o_hist);
	w->count = (int*)(b + o_count);
	w->anchor = (float*)(b + o_anchor);
	w->temp = b + o_temp;
	w->h_hist.assign(frames, 0);
	OCB_CUDA(ctx, cudaMemsetAsync(w->hist, 0, (size_t)frames * sizeof(int), ctx->stream));
	return OCB_OK;
}
// the histogram of first lost frames, back on the host (the one synchronisation per scan)
static int reseed_read_hist(ocb_ctx* ctx, ReseedWs* w) {
	OCB_CUDA(ctx, cudaMemcpyAsync(w->h_hist.data(), w->hist, w->h_hist.size() * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
	OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return OCB_OK;
}
// gather the POIs whose first lost frame is f (m of them) into the sub-queue, rebuilt from the seeds; prev: frame f - 1's records
static int reseed_gather(ocb_ctx* ctx, int dim, ReseedWs* w, const float* d_seeds, const float* prev, size_t n, int f, size_t m, float zncc_min,
	float* sub) {
	const int rc = launched(ctx, "reseed_select", ocb::reseed_select_launch(w->first, f, n, w->idx, w->count, w->temp, w->temp_bytes, ctx->stream));
	return rc ? rc : launched(ctx, "reseed_rebuild", ocb::reseed_rebuild_launch(dim, d_seeds, prev, w->idx, m, zncc_min, w->anchor, sub, ctx->sm_count, ctx->stream));
}

// A 2D subset method of the image series calls: IC-GN (order 1 or 2), IC-LM (the same order with its damping (lambda, alpha, beta),
// passed through unchecked as by ocb_iclm2d) or NR2D1.  It supplies the series launch over frames of a stack and the pair launch
// on re-seeded records against one frame.
struct SubsetMethod2D {
	bool nr;                 // NR2D1; otherwise IC-GN / IC-LM
	int order;               // IC-GN / IC-LM: the shape-function order
	const float* lm_damping; // IC-LM: (lambda, alpha, beta); null: IC-GN
	int np() const { return order == 1 ? 6 : 12; }
};

// The launch geometry of NR2D1, or OCB_ERR_UNSUPPORTED when one warp's slab does not fit in shared memory
static int nr2d1_plan_or_error(ocb_ctx* ctx, int rx, int ry, ocb::Nr2dPlan* plan) {
	if (ocb::nr2d1_plan(rx, ry, ctx->smem_optin, plan)) return OCB_OK;
	return set_error(ctx, OCB_ERR_UNSUPPORTED, "nr2d1: subset radius (%d,%d) exceeds the shared-memory design limit", rx, ry);
}

// NR2D1 of the n device records q (1 <= n < 2^31) against img, on ctx's device (current) and stream.  The pair calls pass their
// image pair, the re-seeding series calls one frame of the series.
static int nr2d1_run(ocb_ctx* ctx, const ocb::Image2D& img, float* q, size_t n, int rx, int ry, float conv, float stop) {
	ocb::Nr2dPlan plan;
	if (const int rc = nr2d1_plan_or_error(ctx, rx, ry, &plan)) return rc;
	return launched(ctx, "nr2d1", ocb::nr2d1_launch(plan, img, q, n, rx, ry, conv, stop, ctx->sm_count, ctx->d_counter, ctx->stream));
}

// The method's series launch: the m seeds through the frames of img.tar into out (frames x m records, frame-major).  IC-GN and
// IC-LM take the warps per POI of a launch over plan_n POIs; NR2D1's plan does not depend on the queue.
static int subset2d_series_launch(ocb_ctx* ctx, const SubsetMethod2D& sm, const ocb::Image2D& img, int frames, const float* seeds, float* out,
	size_t m, size_t plan_n, int rx, int ry, float conv, float stop) {
	if (sm.nr) {
		ocb::Nr2dPlan plan;
		if (const int r = nr2d1_plan_or_error(ctx, rx, ry, &plan)) return r;
		return launched(ctx, "nr2d1_series",
			ocb::nr2d1_series_launch(plan, img, frames, seeds, out, m, rx, ry, conv, stop, ctx->sm_count, ctx->d_counter, ctx->stream));
	}
	ocb::Icgn2dPlan plan;
	if (const int r = icgn2d_plan_or_error(ctx, m, plan_n, sm.np(), rx, ry, sm.lm_damping != nullptr, &plan)) return r;
	return launched(ctx, sm.lm_damping ? "iclm2d_series" : "icgn2d_series",
		ocb::icgn2d_series_launch(sm.np(), plan, img, frames, seeds, out, m, rx, ry, conv, stop, ctx->d_counter, sm.lm_damping, ctx->stream));
}

// The method's pair launch on the m device records q against the image pair img, with the warps per POI of plan_n POIs
static int subset2d_pair_run(ocb_ctx* ctx, const SubsetMethod2D& sm, const ocb::Image2D& img, float* q, size_t m, size_t plan_n, int rx, int ry,
	float conv, float stop) {
	if (sm.nr) return nr2d1_run(ctx, img, q, m, rx, ry, conv, stop);
	return icgn2d_run(ctx, sm.np(), img, q, m, plan_n, rx, ry, conv, stop, nullptr, sm.lm_damping);
}

// The 2D series of reference s.ref against the F frames of the stack s.tar with the subset method sm, over the n device seeds
// into d_out (F x n records, frame-major), re-seeding lost POIs when rs is set.
// Without rs this is one series launch.  With it:
//   1. the same series launch over all n POIs and frames;
//   2. one scan of every record for each POI's first lost frame, whose per-frame counts come back in one copy (none: done);
//   3. for the smallest frame f with losses: its m lost POIs are gathered and rebuilt, FFT-CC and the method's pair launch run on
//      them against frame f and the results go to out[f]; then one series launch carries those m records through frames
//      f + 1 ... F - 1 (into ctx->reseed_cont) and they are scattered into out; those m POIs alone are scanned again for a later
//      loss;
//   4. step 3 repeats for the next frame with losses: one synchronisation per such frame.
// Every IC-GN / IC-LM launch takes the warps per POI of a launch over all n POIs, so each POI splits its sums as in step 1.
static int subset2d_series_run(ocb_ctx* ctx, const SubsetMethod2D& sm, const ocb::Image2D& s, int F, const float* d_seeds, float* d_out, size_t n,
	int rx, int ry, float conv, float stop, const SeriesReseed* rs) {
	const size_t frame_px = (size_t)s.w * s.h;
	int rc;
	if ((rc = subset2d_series_launch(ctx, sm, s, F, d_seeds, d_out, n, n, rx, ry, conv, stop))) return rc;
	if (!rs) return OCB_OK;
	const size_t rec = OCB_POI2D_FLOATS;
	const float zmin = rs->zncc_min;
	ReseedWs w;
	if ((rc = reseed_workspace(ctx, n, F, 2, &w))) return rc;
	if ((rc = launched(ctx, "reseed_scan", ocb::reseed_scan_launch(2, d_out, n, 0, F, nullptr, n, zmin, w.first, w.hist, ctx->sm_count, ctx->stream)))
		|| (rc = reseed_read_hist(ctx, &w)))
		return rc;
	bool any = false;
	for (int f = 0; f < F; f++) any = any || w.h_hist[f] > 0;
	if (!any) return OCB_OK;
	if ((rc = grow(ctx, ctx->reseed_sub, n * rec * sizeof(float)))) return rc;
	float* const sub = ctx->reseed_sub.as<float>();
	if ((rc = launched(ctx, "reseed_anchor_init", ocb::reseed_anchor_init_launch(2, d_seeds, n, w.anchor, ctx->sm_count, ctx->stream)))) return rc;
	for (int f = 0; f < F; f++) {
		const size_t m = (size_t)w.h_hist[f];
		if (!m) continue;
		if ((rc = reseed_gather(ctx, 2, &w, d_seeds, f ? d_out + (size_t)(f - 1) * n * rec : nullptr, n, f, m, zmin, sub))) return rc;
		const ocb::Image2D frame{ s.ref, s.tar + (size_t)f * frame_px, s.w, s.h };
		if ((rc = fftcc2d_run(ctx, frame, sub, m, rs->fft_r[0], rs->fft_r[1]))) return rc;
		if ((rc = subset2d_pair_run(ctx, sm, frame, sub, m, n, rx, ry, conv, stop))) return rc;
		if ((rc = launched(ctx, "reseed_scatter", ocb::reseed_scatter_launch(2, sub, m, 1, w.idx, d_out, n, f, ctx->sm_count, ctx->stream)))) return rc;
		rs->counts[f] = m;
		if (f + 1 == F) break;
		const int rest = F - f - 1;
		if ((rc = grow(ctx, ctx->reseed_cont, (size_t)rest * m * rec * sizeof(float)))) return rc;
		float* const cont = ctx->reseed_cont.as<float>();
		const ocb::Image2D later{ s.ref, s.tar + (size_t)(f + 1) * frame_px, s.w, s.h };
		if ((rc = subset2d_series_launch(ctx, sm, later, rest, sub, cont, m, n, rx, ry, conv, stop))) return rc;
		if ((rc = launched(ctx, "reseed_scatter", ocb::reseed_scatter_launch(2, cont, m, rest, w.idx, d_out, n, f + 1, ctx->sm_count, ctx->stream)))
			|| (rc = launched(ctx, "reseed_scan", ocb::reseed_scan_launch(2, d_out, n, f + 1, F, w.idx, m, zmin, w.first, w.hist, ctx->sm_count, ctx->stream)))
			|| (rc = reseed_read_hist(ctx, &w)))
			return rc;
	}
	return OCB_OK;
}

// Checks and runs a 2D series call on a single-device context: device seeds and output; rs null for the plain series.
static int subset2d_series_dev(ocb_ctx* ctx, const char* what, const SubsetMethod2D& sm, const void* d_seeds, void* d_out, size_t n, int rx, int ry,
	float conv, float stop, const SeriesReseed* rs) {
	if (!ctx || ((!d_seeds || !d_out) && n) || rx < 1 || ry < 1) return set_error(ctx, OCB_ERR_ARG, "%s: bad arguments", what);
	if (!sm.nr && sm.order != 1 && sm.order != 2) return set_error(ctx, OCB_ERR_ARG, "%s: order must be 1 or 2", what);
	const SeriesStore& s = ctx->series2d;
	if (!s.ref) return set_error(ctx, OCB_ERR_STATE, "%s: no series set", what);
	int rc;
	if (rs && (rc = reseed_check(ctx, what, 2, *rs))) return rc;
	if (n == 0) return OCB_OK;
	if ((rc = series_size_check(ctx, what, n, s.frames, OCB_POI2D_FLOATS * sizeof(float), false))) return rc;
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	return subset2d_series_run(ctx, sm, s.view2(0), s.frames, (const float*)d_seeds, (float*)d_out, n, rx, ry, conv, stop, rs);
}

static int subset2d_series_host(ocb_ctx* ctx, const char* what, const SubsetMethod2D& sm, const void* seeds, void* out, size_t n, int rx, int ry,
	float conv, float stop, const SeriesReseed* rs) {
	return series_host(ctx, what, &ocb_ctx::series2d, n, { seeds }, OCB_POI2D_FLOATS, { { out, OCB_POI2D_FLOATS } },
		[&](ocb_ctx* x, const float* const* d_in, float* const* d_out) { return subset2d_series_dev(x, what, sm, d_in[0], d_out[0], n, rx, ry, conv, stop, rs); });
}

// The plain and the re-seeding series calls of one method (dev: device seeds and out)
static int subset2d_series_call(ocb_ctx* ctx, const char* what, const SubsetMethod2D& sm, bool dev, const void* seeds, void* out, size_t n, int rx,
	int ry, float conv, float stop) {
	return dev ? subset2d_series_dev(ctx, what, sm, seeds, out, n, rx, ry, conv, stop, nullptr)
		: subset2d_series_host(ctx, what, sm, seeds, out, n, rx, ry, conv, stop, nullptr);
}
static int subset2d_series_reseed_call(ocb_ctx* ctx, const char* what, const SubsetMethod2D& sm, bool dev, const void* seeds, void* out, size_t n,
	int rx, int ry, float conv, float stop, int fft_rx, int fft_ry, float zncc_min, size_t* reseeded) {
	return series_reseed(ctx, &ocb_ctx::series2d, dev, n, reseeded, [&](size_t* counts) {
		const SeriesReseed rs{ { fft_rx, fft_ry, 1 }, zncc_min, counts };
		return dev ? subset2d_series_dev(ctx, what, sm, seeds, out, n, rx, ry, conv, stop, &rs)
			: subset2d_series_host(ctx, what, sm, seeds, out, n, rx, ry, conv, stop, &rs);
	});
}

int ocb_icgn2d_series_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop) {
	OCB_NO_GROUP(ctx, "icgn2d_series_dev");
	return subset2d_series_call(ctx, "icgn2d_series", { false, order, nullptr }, true, d_seeds, d_out, n, rx, ry, conv, stop);
}

int ocb_icgn2d_series(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop) {
	return subset2d_series_call(ctx, "icgn2d_series", { false, order, nullptr }, false, seeds, out, n, rx, ry, conv, stop);
}

int ocb_icgn2d_series_reseed_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop,
	int fft_rx, int fft_ry, float zncc_min, size_t* reseeded) {
	OCB_NO_GROUP(ctx, "icgn2d_series_reseed_dev");
	return subset2d_series_reseed_call(ctx, "icgn2d_series_reseed", { false, order, nullptr }, true, d_seeds, d_out, n, rx, ry, conv, stop, fft_rx,
		fft_ry, zncc_min, reseeded);
}

int ocb_icgn2d_series_reseed(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, int fft_rx,
	int fft_ry, float zncc_min, size_t* reseeded) {
	return subset2d_series_reseed_call(ctx, "icgn2d_series_reseed", { false, order, nullptr }, false, seeds, out, n, rx, ry, conv, stop, fft_rx,
		fft_ry, zncc_min, reseeded);
}

int ocb_iclm2d_series_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop, float lambda,
	float alpha, float beta) {
	OCB_NO_GROUP(ctx, "iclm2d_series_dev");
	const float damping[3] = { lambda, alpha, beta };
	return subset2d_series_call(ctx, "iclm2d_series", { false, order, damping }, true, d_seeds, d_out, n, rx, ry, conv, stop);
}

int ocb_iclm2d_series(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, float lambda, float alpha,
	float beta) {
	const float damping[3] = { lambda, alpha, beta };
	return subset2d_series_call(ctx, "iclm2d_series", { false, order, damping }, false, seeds, out, n, rx, ry, conv, stop);
}

int ocb_iclm2d_series_reseed_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop,
	float lambda, float alpha, float beta, int fft_rx, int fft_ry, float zncc_min, size_t* reseeded) {
	OCB_NO_GROUP(ctx, "iclm2d_series_reseed_dev");
	const float damping[3] = { lambda, alpha, beta };
	return subset2d_series_reseed_call(ctx, "iclm2d_series_reseed", { false, order, damping }, true, d_seeds, d_out, n, rx, ry, conv, stop, fft_rx,
		fft_ry, zncc_min, reseeded);
}

int ocb_iclm2d_series_reseed(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, float lambda,
	float alpha, float beta, int fft_rx, int fft_ry, float zncc_min, size_t* reseeded) {
	const float damping[3] = { lambda, alpha, beta };
	return subset2d_series_reseed_call(ctx, "iclm2d_series_reseed", { false, order, damping }, false, seeds, out, n, rx, ry, conv, stop, fft_rx,
		fft_ry, zncc_min, reseeded);
}

int ocb_nr2d1_series_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop) {
	OCB_NO_GROUP(ctx, "nr2d1_series_dev");
	return subset2d_series_call(ctx, "nr2d1_series", { true, 1, nullptr }, true, d_seeds, d_out, n, rx, ry, conv, stop);
}

int ocb_nr2d1_series(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop) {
	return subset2d_series_call(ctx, "nr2d1_series", { true, 1, nullptr }, false, seeds, out, n, rx, ry, conv, stop);
}

int ocb_nr2d1_series_reseed_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop, int fft_rx,
	int fft_ry, float zncc_min, size_t* reseeded) {
	OCB_NO_GROUP(ctx, "nr2d1_series_reseed_dev");
	return subset2d_series_reseed_call(ctx, "nr2d1_series_reseed", { true, 1, nullptr }, true, d_seeds, d_out, n, rx, ry, conv, stop, fft_rx, fft_ry,
		zncc_min, reseeded);
}

int ocb_nr2d1_series_reseed(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, int fft_rx, int fft_ry,
	float zncc_min, size_t* reseeded) {
	return subset2d_series_reseed_call(ctx, "nr2d1_series_reseed", { true, 1, nullptr }, false, seeds, out, n, rx, ry, conv, stop, fft_rx, fft_ry,
		zncc_min, reseeded);
}

// one launch over a host queue (all POIs share the radius), optional host offsets
static int icgn2d_host_group(ocb_ctx* ctx, int np, float* poi2d, size_t n, int rx, int ry, float conv, float stop, const float* offsets) {
	const float* d_off = nullptr;
	if (offsets) {
		const size_t ob = n * 2 * sizeof(float);
		const int rc = grow(ctx, ctx->d_off, ob);
		if (rc) return rc;
		OCB_CUDA(ctx, cudaMemcpyAsync(ctx->d_off.p, offsets, ob, cudaMemcpyHostToDevice, ctx->stream));
		d_off = ctx->d_off.as<float>();
	}
	return run_host_queue(ctx, "icgn2d_ex", poi2d, n, OCB_POI2D_FLOATS,
		[&](float* d, size_t m, size_t first) { return icgn2d_dev(ctx, np, d, m, rx, ry, conv, stop, d_off ? d_off + 2 * first : nullptr); },
		PIPELINED_IN_PLACE);
}

int ocb_icgn2d_ex(ocb_ctx* ctx, int order, void* poi2d, size_t n, int rx, int ry, float conv, float stop, const float* center_offsets,
	int self_adaptive) {
	if (is_group(ctx) && poi2d)
		return group_shard(ctx, poi2d, n, OCB_POI2D_FLOATS * sizeof(float), OCB_GROUP_MIN_2D, [=](ocb_ctx* m, void* q, size_t c, size_t first) {
			return ocb_icgn2d_ex(m, order, q, c, rx, ry, conv, stop, center_offsets ? center_offsets + 2 * first : nullptr, self_adaptive);
		});
	if (!ctx || (!poi2d && n)) return set_error(ctx, OCB_ERR_ARG, "icgn2d_ex: bad arguments");
	if (order != 1 && order != 2) return set_error(ctx, OCB_ERR_ARG, "icgn2d_ex: order must be 1 or 2");
	if (n == 0) return OCB_OK;
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const int np = order == 1 ? 6 : 12;
	float* q = (float*)poi2d;
	if (!self_adaptive) return icgn2d_host_group(ctx, np, q, n, rx, ry, conv, stop, center_offsets);
	// self-adaptive: group the POIs by their own (subset_radius.x, subset_radius.y); one launch per group
	std::map<std::pair<int, int>, std::vector<size_t>> groups;
	for (size_t i = 0; i < n; i++) {
		const float* p = q + i * OCB_POI2D_FLOATS;
		groups[std::make_pair((int)p[23], (int)p[24])].push_back(i);
	}
	for (auto& kv : groups) { // refuse before anything is launched: no partial results
		ocb::Icgn2dPlan plan;
		const size_t m = kv.second.size();
		if (kv.first.first >= 1 && kv.first.second >= 1 && icgn2d_plan_or_error(ctx, m, m, np, kv.first.first, kv.first.second, false, &plan))
			return set_error(ctx, OCB_ERR_UNSUPPORTED, "icgn2d_ex: subset radius (%d,%d) of a self-adaptive POI exceeds the shared-memory design limit",
				kv.first.first, kv.first.second);
	}
	std::vector<float> gq, goff;
	for (auto& kv : groups) {
		const int grx = kv.first.first, gry = kv.first.second;
		const std::vector<size_t>& idx = kv.second;
		if (grx < 1 || gry < 1) { // the reference would size its scratch from a radius < 1 (undefined); reject like a failed guard
			for (size_t i : idx)
				if (q[i * OCB_POI2D_FLOATS + 16] >= 0) q[i * OCB_POI2D_FLOATS + 16] = -3.f;
			continue;
		}
		gq.resize(idx.size() * OCB_POI2D_FLOATS);
		for (size_t k = 0; k < idx.size(); k++) memcpy(&gq[k * OCB_POI2D_FLOATS], q + idx[k] * OCB_POI2D_FLOATS, OCB_POI2D_FLOATS * sizeof(float));
		const float* off = nullptr;
		if (center_offsets) {
			goff.resize(idx.size() * 2);
			for (size_t k = 0; k < idx.size(); k++) { goff[2 * k] = center_offsets[2 * idx[k]]; goff[2 * k + 1] = center_offsets[2 * idx[k] + 1]; }
			off = goff.data();
		}
		int rc = icgn2d_host_group(ctx, np, gq.data(), idx.size(), grx, gry, conv, stop, off);
		if (rc) return rc;
		for (size_t k = 0; k < idx.size(); k++) memcpy(q + idx[k] * OCB_POI2D_FLOATS, &gq[k * OCB_POI2D_FLOATS], OCB_POI2D_FLOATS * sizeof(float));
	}
	return OCB_OK;
}

// ---- ICLM (SURVEY.md section 8(f) N2) ----------------------------------------------------------------
int ocb_iclm2d_dev(ocb_ctx* ctx, int order, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop, float lambda, float alpha, float beta) {
	if (order != 1 && order != 2) return set_error(ctx, OCB_ERR_ARG, "iclm2d: order must be 1 or 2");
	const float damping[3] = { lambda, alpha, beta };
	return icgn2d_dev(ctx, order == 1 ? 6 : 12, d_poi2d, n, rx, ry, conv, stop, nullptr, damping);
}

int ocb_iclm2d(ocb_ctx* ctx, int order, void* poi2d, size_t n, int rx, int ry, float conv, float stop, float lambda, float alpha, float beta) {
	return pair_host(ctx, "iclm2d", order != 1 && order != 2 ? "order must be 1 or 2" : nullptr, poi2d, n, OCB_POI2D_FLOATS, OCB_GROUP_MIN_2D,
		PIPELINED_IN_PLACE, [=](ocb_ctx* x, float* d, size_t m) { return ocb_iclm2d_dev(x, order, d, m, rx, ry, conv, stop, lambda, alpha, beta); });
}

// ---- NR2D1 (SURVEY.md section 8(f) N2) ---------------------------------------------------------------
int ocb_nr2d_prepare(ocb_ctx* ctx) {
	if (is_group(ctx)) return prepare_members(ctx, ocb_nr2d_prepare);
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	if (!ctx->img2.ref) return set_error(ctx, OCB_ERR_STATE, "nr2d_prepare: images not set");
	ctx->prepared_nr2 = true; // target gradients and the three interpolants are evaluated on chip per POI
	return OCB_OK;
}

int ocb_nr2d1_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop) {
	const int rc = pair_checks(ctx, "nr2d1", d_poi2d, n, rx >= 1 && ry >= 1, nullptr, 2, &ocb_ctx::prepared_nr2, true);
	return rc == PAIR_GO ? nr2d1_run(ctx, ctx->img2, (float*)d_poi2d, n, rx, ry, conv, stop) : rc;
}

int ocb_nr2d1(ocb_ctx* ctx, void* poi2d, size_t n, int rx, int ry, float conv, float stop) {
	return pair_host(ctx, "nr2d1", nullptr, poi2d, n, OCB_POI2D_FLOATS, OCB_GROUP_MIN_2D, PIPELINED,
		[=](ocb_ctx* x, float* d, size_t m) { return ocb_nr2d1_dev(x, d, m, rx, ry, conv, stop); });
}

// ---- EpipolarSearch candidate sweep (SURVEY.md section 8(f) N4) ----------------------------------------
int ocb_epipolar_search2d_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, const float* fundamental, const float* parallax_x, const float* parallax_y,
	int search_radius, int search_step, int rx, int ry, float conv, float stop) {
	// the search step refusal: EpipolarSearch::setSearch, src/oc_epipolar_search.cpp:44-53
	int rc = pair_checks(ctx, "epipolar_search2d", d_poi2d, n, fundamental && parallax_x && parallax_y && rx >= 1 && ry >= 1,
		search_step < 1 || search_radius < search_step ? "search radius is less than search step" : nullptr, 2, &ocb_ctx::prepared2, false);
	if (rc != PAIR_GO) return rc;
	const int slots = ocb::epipolar_slots(search_radius, search_step);
	// candidates of a block of POIs at a time: at most ~2^22 records (420 MB) in flight
	size_t block = ((size_t)1 << 22) / (size_t)slots;
	if (block < 1) block = 1;
	if (block > n) block = n;
	if ((rc = grow(ctx, ctx->d_cand, block * (size_t)slots * OCB_POI2D_FLOATS * sizeof(float)))) return rc;
	float* const cand = ctx->d_cand.as<float>();
	for (size_t p0 = 0; p0 < n; p0 += block) {
		const size_t nb = n - p0 < block ? n - p0 : block;
		if ((rc = launched(ctx, "epipolar_candidates", ocb::epipolar_candidates_launch((const float*)d_poi2d, p0, nb, fundamental, parallax_x, parallax_y,
				 search_radius, search_step, rx, ry, ctx->img2.w, ctx->img2.h, slots, cand, ctx->sm_count, ctx->stream)))
			|| (rc = icgn2d_dev(ctx, 6, cand, nb * (size_t)slots, rx, ry, conv, stop))
			|| (rc = launched(ctx, "epipolar_select", ocb::epipolar_select_launch((float*)d_poi2d, p0, nb, slots, cand, ctx->sm_count, ctx->stream))))
			return rc;
	}
	return OCB_OK;
}

int ocb_epipolar_search2d(ocb_ctx* ctx, void* poi2d, size_t n, const float* fundamental, const float* parallax_x, const float* parallax_y,
	int search_radius, int search_step, int rx, int ry, float conv, float stop) {
	return pair_host(ctx, "epipolar_search2d", nullptr, poi2d, n, OCB_POI2D_FLOATS, OCB_GROUP_MIN_EPIPOLAR, STAGED, [=](ocb_ctx* x, float* d, size_t m) {
		return ocb_epipolar_search2d_dev(x, d, m, fundamental, parallax_x, parallax_y, search_radius, search_step, rx, ry, conv, stop);
	});
}

// ---- Strain (SURVEY.md section 8(f) N4) ---------------------------------------------------------------
static_assert(ocb::poi_floats(ocb::PoiKind::POI2D) == OCB_POI2D_FLOATS && ocb::poi_floats(ocb::PoiKind::POI3D) == OCB_POI3D_FLOATS
	&& ocb::poi_floats(ocb::PoiKind::POI2DS) == OCB_POI2DS_FLOATS, "the kernels' record lengths are the C ABI's");
static int strain_dev(ocb_ctx* ctx, ocb::PoiKind kind, void* d_poi, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation, long long only = -1) {
	int rc = pair_checks(ctx, "strain", d_poi, n, only < (long long)n, nullptr, 0, nullptr, true);
	if (rc != PAIR_GO) return rc;
	if ((rc = grow(ctx, ctx->d_strain_ws, ocb::strain_workspace_bytes(n)))) return rc;
	const cudaError_t e = ocb::strain_launch(kind, (float*)d_poi, n, radius, min_neighbors, zncc_threshold, approximation, only, ctx->d_strain_ws.p,
		ctx->sm_count, ctx->stream, &ctx->launches);
	if (e != cudaSuccess) return set_error(ctx, OCB_ERR_CUDA, "strain launch failed: %s", cudaGetErrorString(e));
	return OCB_OK;
}

static int strain_host(ocb_ctx* ctx, ocb::PoiKind kind, void* poi, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation,
	long long only = -1) {
	if (is_group(ctx)) // every POI needs its neighbours wherever they are in the queue: not sharded, the first member runs it
		return on_exec(ctx, [&](ocb_ctx* x) { return strain_host(x, kind, poi, n, radius, min_neighbors, zncc_threshold, approximation, only); });
	return run_host_queue(ctx, "strain", poi, n, ocb::poi_floats(kind), [&](float* d, size_t m, size_t) {
		return strain_dev(ctx, kind, d, m, radius, min_neighbors, zncc_threshold, approximation, only);
	}, STAGED);
}

int ocb_strain2d(ocb_ctx* ctx, void* poi2d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_host(ctx, ocb::PoiKind::POI2D, poi2d, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain3d(ocb_ctx* ctx, void* poi3d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_host(ctx, ocb::PoiKind::POI3D, poi3d, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain2ds(ocb_ctx* ctx, void* poi2ds, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_host(ctx, ocb::PoiKind::POI2DS, poi2ds, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain2ds_dev(ocb_ctx* ctx, void* d_poi2ds, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_dev(ctx, ocb::PoiKind::POI2DS, d_poi2ds, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain2d_single(ocb_ctx* ctx, void* poi2d, size_t n, size_t index, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_host(ctx, ocb::PoiKind::POI2D, poi2d, n, radius, min_neighbors, zncc_threshold, approximation, (long long)index);
}
int ocb_strain3d_single(ocb_ctx* ctx, void* poi3d, size_t n, size_t index, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_host(ctx, ocb::PoiKind::POI3D, poi3d, n, radius, min_neighbors, zncc_threshold, approximation, (long long)index);
}
int ocb_strain2d_dev(ocb_ctx* ctx, void* d_poi2d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_dev(ctx, ocb::PoiKind::POI2D, d_poi2d, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain3d_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_dev(ctx, ocb::PoiKind::POI3D, d_poi3d, n, radius, min_neighbors, zncc_threshold, approximation);
}

// ---- RegionFit2D / RegionFit3D: Strain's neighbour search and plane fit over a second, reliable set ------------------
// The reliable set is checked like the queue: NULL only with n_reliable 0, and at most 2^31 - 1 records (the kernels index it
// with int).
static int region_fit_dev(ocb_ctx* ctx, ocb::PoiKind kind, const void* d_reliable, size_t n_reliable, void* d_q, size_t n, float radius,
	int min_neighbors) {
	int rc = pair_checks(ctx, "region_fit", d_q, n, (d_reliable || !n_reliable) && n_reliable <= 0x7fffffffull, nullptr, 0, nullptr, true);
	if (rc != PAIR_GO) return rc;
	if ((rc = grow(ctx, ctx->d_strain_ws, ocb::strain_workspace_bytes(n_reliable)))) return rc;
	const cudaError_t e = ocb::region_fit_launch(kind, (const float*)d_reliable, n_reliable, (float*)d_q, n, radius, min_neighbors, ctx->d_strain_ws.p,
		ctx->sm_count, ctx->stream, &ctx->launches);
	if (e != cudaSuccess) return set_error(ctx, OCB_ERR_CUDA, "region_fit launch failed: %s", cudaGetErrorString(e));
	return OCB_OK;
}

// Both sets are staged in the context's queue buffer, queue first; only the queue is copied back.
static int region_fit_host(ocb_ctx* ctx, ocb::PoiKind kind, const void* reliable, size_t n_reliable, void* q, size_t n, float radius,
	int min_neighbors) {
	if (is_group(ctx)) // every POI may need any reliable POI: not sharded, the first member runs it (as Strain)
		return on_exec(ctx, [&](ocb_ctx* x) { return region_fit_host(x, kind, reliable, n_reliable, q, n, radius, min_neighbors); });
	if (!ctx || (!q && n) || (!reliable && n_reliable) || n > 0x7fffffffull || n_reliable > 0x7fffffffull)
		return set_error(ctx, OCB_ERR_ARG, "region_fit: bad arguments");
	if (n == 0) return OCB_OK;
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const size_t rec = (size_t)ocb::poi_floats(kind) * sizeof(float);
	int rc;
	if ((rc = grow(ctx, ctx->d_poi, (n + n_reliable) * rec))) return rc;
	float* const d_q = ctx->d_poi.as<float>();
	float* const d_rel = d_q + n * (size_t)ocb::poi_floats(kind);
	OCB_CUDA(ctx, cudaMemcpyAsync(d_q, q, n * rec, cudaMemcpyHostToDevice, ctx->stream));
	if (n_reliable) OCB_CUDA(ctx, cudaMemcpyAsync(d_rel, reliable, n_reliable * rec, cudaMemcpyHostToDevice, ctx->stream));
	if ((rc = region_fit_dev(ctx, kind, d_rel, n_reliable, d_q, n, radius, min_neighbors))) return rc;
	OCB_CUDA(ctx, cudaMemcpyAsync(q, d_q, n * rec, cudaMemcpyDeviceToHost, ctx->stream));
	OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return OCB_OK;
}

int ocb_region_fit2d(ocb_ctx* ctx, const void* reliable, size_t n_reliable, void* poi2d, size_t n, float radius, int min_neighbors) {
	return region_fit_host(ctx, ocb::PoiKind::POI2D, reliable, n_reliable, poi2d, n, radius, min_neighbors);
}
int ocb_region_fit3d(ocb_ctx* ctx, const void* reliable, size_t n_reliable, void* poi3d, size_t n, float radius, int min_neighbors) {
	return region_fit_host(ctx, ocb::PoiKind::POI3D, reliable, n_reliable, poi3d, n, radius, min_neighbors);
}
int ocb_region_fit2d_dev(ocb_ctx* ctx, const void* d_reliable, size_t n_reliable, void* d_poi2d, size_t n, float radius, int min_neighbors) {
	return region_fit_dev(ctx, ocb::PoiKind::POI2D, d_reliable, n_reliable, d_poi2d, n, radius, min_neighbors);
}
int ocb_region_fit3d_dev(ocb_ctx* ctx, const void* d_reliable, size_t n_reliable, void* d_poi3d, size_t n, float radius, int min_neighbors) {
	return region_fit_dev(ctx, ocb::PoiKind::POI3D, d_reliable, n_reliable, d_poi3d, n, radius, min_neighbors);
}

// Strain over a series: n_frames frames of n records, frame-major.  Their bytes, n_frames n rec_floats floats, must fit a size_t.
static bool strain_series_fits(ocb::PoiKind kind, size_t n_frames, size_t n) {
	const size_t rec = (size_t)ocb::poi_floats(kind) * sizeof(float);
	return n == 0 || (n <= SIZE_MAX / rec && n_frames <= SIZE_MAX / (n * rec));
}

static int strain_series_dev(ocb_ctx* ctx, ocb::PoiKind kind, void* d_poi, size_t n_frames, size_t n, float radius, int min_neighbors,
	float zncc_threshold, int approximation) {
	int rc = pair_checks(ctx, "strain_series", d_poi, n_frames ? n : 0, strain_series_fits(kind, n_frames, n), nullptr, 0, nullptr, true);
	if (rc != PAIR_GO) return rc;
	if ((rc = grow(ctx, ctx->d_strain_ws, ocb::strain_workspace_bytes(n, n_frames)))) return rc;
	bool moved = false;
	const cudaError_t e = ocb::strain_series_launch(kind, (float*)d_poi, n_frames, n, radius, min_neighbors, zncc_threshold, approximation,
		ctx->d_strain_ws.p, ctx->sm_count, ctx->stream, &ctx->launches, &moved);
	if (e != cudaSuccess) return set_error(ctx, OCB_ERR_CUDA, "strain_series launch failed: %s", cudaGetErrorString(e));
	if (moved) return set_error(ctx, OCB_ERR_ARG, "strain_series: the POI positions of some frame are not those of frame 0");
	return OCB_OK;
}

static int strain_series_host(ocb_ctx* ctx, ocb::PoiKind kind, void* poi, size_t n_frames, size_t n, float radius, int min_neighbors,
	float zncc_threshold, int approximation) {
	if (is_group(ctx)) // as strain_host: the first member runs it
		return on_exec(ctx, [&](ocb_ctx* x) { return strain_series_host(x, kind, poi, n_frames, n, radius, min_neighbors, zncc_threshold, approximation); });
	if (!ctx || !strain_series_fits(kind, n_frames, n)) return set_error(ctx, OCB_ERR_ARG, "strain_series: bad arguments");
	return run_host_queue(ctx, "strain_series", poi, n_frames * n, ocb::poi_floats(kind), [&](float* d, size_t, size_t) {
		return strain_series_dev(ctx, kind, d, n_frames, n, radius, min_neighbors, zncc_threshold, approximation);
	}, STAGED);
}

int ocb_strain2d_series(ocb_ctx* ctx, void* poi2d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_series_host(ctx, ocb::PoiKind::POI2D, poi2d, n_frames, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain3d_series(ocb_ctx* ctx, void* poi3d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold, int approximation) {
	return strain_series_host(ctx, ocb::PoiKind::POI3D, poi3d, n_frames, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain2ds_series(ocb_ctx* ctx, void* poi2ds, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation) {
	return strain_series_host(ctx, ocb::PoiKind::POI2DS, poi2ds, n_frames, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain2d_series_dev(ocb_ctx* ctx, void* d_poi2d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation) {
	return strain_series_dev(ctx, ocb::PoiKind::POI2D, d_poi2d, n_frames, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain3d_series_dev(ocb_ctx* ctx, void* d_poi3d, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation) {
	return strain_series_dev(ctx, ocb::PoiKind::POI3D, d_poi3d, n_frames, n, radius, min_neighbors, zncc_threshold, approximation);
}
int ocb_strain2ds_series_dev(ocb_ctx* ctx, void* d_poi2ds, size_t n_frames, size_t n, float radius, int min_neighbors, float zncc_threshold,
	int approximation) {
	return strain_series_dev(ctx, ocb::PoiKind::POI2DS, d_poi2ds, n_frames, n, radius, min_neighbors, zncc_threshold, approximation);
}

// TricubicBspline::prepare: the B-spline coefficients of volume tar into coef, in three passes x -> coef, y -> tmp, z -> coef
static int bspline_prefilter(ocb_ctx* ctx, const float* tar, float* coef, float* tmp, int dx, int dy, int dz) {
	const float* const in[3] = { tar, coef, tmp };
	float* const out[3] = { coef, tmp, coef };
	for (int axis = 0; axis < 3; axis++)
		if (const int rc = launched(ctx, "prefilter3d", ocb::prefilter3d_launch(in[axis], out[axis], dx, dy, dz, axis, ctx->sm_count, ctx->stream)))
			return rc;
	return OCB_OK;
}

int ocb_icgn3d_prepare(ocb_ctx* ctx) {
	if (is_group(ctx)) return group_each(ctx, [](ocb_ctx* m) { return ocb_icgn3d_prepare(m); });
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	if (!ctx->img3.ref) return set_error(ctx, OCB_ERR_STATE, "icgn3d_prepare: images not set");
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const int dx = ctx->img3.dx, dy = ctx->img3.dy, dz = ctx->img3.dz;
	const size_t elems = (size_t)dx * dy * dz;
	int rc;
	if ((rc = grow(ctx, ctx->rg3, elems * sizeof(float4))) || (rc = grow(ctx, ctx->coef3, elems * sizeof(float)))
		|| (rc = grow(ctx, ctx->tmp3, elems * sizeof(float))))
		return rc;
	float4* const rg = ctx->rg3.as<float4>();
	float* const coef = ctx->coef3.as<float>();
	float* const tmp = ctx->tmp3.as<float>();
	if ((rc = launched(ctx, "gradient3d", ocb::gradient3d_launch(ctx->img3.ref, rg, dx, dy, dz, ctx->sm_count, ctx->stream)))
		|| (rc = bspline_prefilter(ctx, ctx->img3.tar, coef, tmp, dx, dy, dz)))
		return rc;
	ctx->img3.rg = rg;
	ctx->img3.coef = coef;
	ctx->prepared3 = true;
	return OCB_OK;
}

// The launch geometry of ICGN3D1, or OCB_ERR_UNSUPPORTED when the subvolume has 2^30 voxels or more (the kernel indexes it with
// int) or even a one-layer slab does not fit in shared memory
static int icgn3d1_plan_or_error(ocb_ctx* ctx, int rx, int ry, int rz, ocb::Icgn3dPlan* plan) {
	if ((size_t)(2 * rx + 1) * (2 * ry + 1) * (2 * rz + 1) > 0x3fffffffull) return set_error(ctx, OCB_ERR_UNSUPPORTED, "icgn3d1: subset too large");
	if (ocb::icgn3d1_plan(rx, ry, rz, ctx->smem_optin, plan)) return OCB_OK;
	return set_error(ctx, OCB_ERR_UNSUPPORTED, "icgn3d1: subset radius (%d,%d,%d) exceeds the shared-memory design limit", rx, ry, rz);
}

int ocb_icgn3d1_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, int rx, int ry, int rz, float conv, float stop) {
	int rc = pair_checks(ctx, "icgn3d1", d_poi3d, n, rx >= 1 && ry >= 1 && rz >= 1, nullptr, 3, &ocb_ctx::prepared3, true);
	if (rc != PAIR_GO) return rc;
	ocb::Icgn3dPlan plan;
	if ((rc = icgn3d1_plan_or_error(ctx, rx, ry, rz, &plan))) return rc;
	return launched(ctx, "icgn3d1",
		ocb::icgn3d1_launch(plan, ctx->img3, (float*)d_poi3d, n, rx, ry, rz, conv, stop, ctx->sm_count, ctx->d_counter + 1, ctx->stream));
}

int ocb_icgn3d1(ocb_ctx* ctx, void* poi3d, size_t n, int rx, int ry, int rz, float conv, float stop) {
	return pair_host(ctx, "icgn3d1", nullptr, poi3d, n, OCB_POI3D_FLOATS, OCB_GROUP_MIN_3D, STAGED,
		[=](ocb_ctx* x, float* d, size_t m) { return ocb_icgn3d1_dev(x, d, m, rx, ry, rz, conv, stop); });
}

// ---- Recovery: rounds of RegionFit and IC-GN over the unreliable POIs of a registered queue --------------------------
// The registration a recovery call runs on its working records: ICGN2D1 / ICGN2D2 (np 6 / 12) on the image pair, or ICGN3D1
// (dim 3) on the volume pair.
struct RecoverMethod {
	int dim, np, r[3];
	float conv, stop;
};

// The argument refusal of a recovery call (null: none): the order, max_rounds, NaN thresholds
static const char* recover_refusal(const RecoverMethod& m, float zncc_high, float zncc_low, int max_rounds) {
	if (m.dim == 2 && m.np != 6 && m.np != 12) return "order must be 1 or 2";
	if (max_rounds < 0) return "max_rounds must be >= 0";
	if (m.conv != m.conv || zncc_high != zncc_high || zncc_low != zncc_low) return "conv, zncc_high and zncc_low must not be NaN";
	return nullptr;
}

// The checks of a recovery call, before any device work: those of the method's pair call, then the order, max_rounds, NaN
// thresholds and the method's plan.  Returns the refusal, OCB_OK when n = 0, or PAIR_GO.
static int recover_checks(ocb_ctx* ctx, const char* what, const RecoverMethod& m, const void* q, size_t n, float zncc_high, float zncc_low,
	int max_rounds) {
	const bool radii = m.r[0] >= 1 && m.r[1] >= 1 && (m.dim == 2 || m.r[2] >= 1);
	int rc = pair_checks(ctx, what, q, n, radii, recover_refusal(m, zncc_high, zncc_low, max_rounds), m.dim,
		m.dim == 2 ? &ocb_ctx::prepared2 : &ocb_ctx::prepared3, true);
	if (rc != PAIR_GO) return rc;
	if (m.dim == 2) {
		ocb::Icgn2dPlan plan;
		rc = icgn2d_plan_or_error(ctx, n, n, m.np, m.r[0], m.r[1], false, &plan);
	} else {
		ocb::Icgn3dPlan plan;
		rc = icgn3d1_plan_or_error(ctx, m.r[0], m.r[1], m.r[2], &plan);
	}
	return rc ? rc : PAIR_GO;
}

// The pair launch of the method on the k device records q against img2 (2D) or img3 (3D: its packed gradients and coefficients),
// with the plan a _dev pair call over k POIs chooses.  The pair calls pass the context's pair, the series calls one frame.
static int recover_register(ocb_ctx* ctx, const RecoverMethod& m, const ocb::Image2D& img2, const ocb::Image3D& img3, float* q, size_t k) {
	if (m.dim == 2) return icgn2d_run(ctx, m.np, img2, q, k, k, m.r[0], m.r[1], m.conv, m.stop, nullptr, nullptr);
	ocb::Icgn3dPlan plan;
	if (const int rc = icgn3d1_plan_or_error(ctx, m.r[0], m.r[1], m.r[2], &plan)) return rc;
	return launched(ctx, "icgn3d1",
		ocb::icgn3d1_launch(plan, img3, q, k, m.r[0], m.r[1], m.r[2], m.conv, m.stop, ctx->sm_count, ctx->d_counter + 1, ctx->stream));
}

// What a series recovery call needs of recover_run besides the records: the queue indices of the POIs accepted over all rounds
// (idx, device), in the order the moves appended their records to the reliable set, where those `count` records start at `rec`.
struct RecoverAccepted {
	const int* idx = nullptr;
	const float* rec = nullptr;
	size_t count = 0;
};

// The recovery loop on the n device records d_q (1 <= n < 2^31), after recover_checks:
//   classification: two selections over the queue (reliable R, unreliable U, each in queue order) and one readback of their sizes;
//   with max_rounds = 0 or U empty, nothing more.  Otherwise one move gathers R into the reliable set and U into working set 0;
//   round k: RegionFit over the reliable set on the working records (five launches, one readback), the pair registration on them,
//   two selections (accepted, kept) and one move that appends the accepted records to the reliable set, writes them to d_q and
//   compacts the kept ones with their queue indices into the other working set; one readback of the accepted count.
// counts gets one entry per round run, *left the size of U at the end.  The registration runs against img2 / img3
// (recover_register).  With acc set, each round adds one launch that collects its accepted queue indices (RecoverAccepted).
static int recover_run(ocb_ctx* ctx, const RecoverMethod& m, const ocb::Image2D& img2, const ocb::Image3D& img3, float* d_q, size_t n, float radius,
	int min_neighbors, float zncc_high, float zncc_low, int max_rounds, std::vector<size_t>* counts, size_t* left, RecoverAccepted* acc = nullptr) {
	const ocb::PoiKind kind = m.dim == 2 ? ocb::PoiKind::POI2D : ocb::PoiKind::POI3D;
	const size_t N = (size_t)ocb::poi_floats(kind);
	auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
	const size_t list = up(n * sizeof(int)), temp_bytes = ocb::recover_select_bytes(n);
	int rc;
	if ((rc = grow(ctx, ctx->recover_ws, 4 * list + 256 + up(temp_bytes) + (acc ? list : 0)))
		|| (rc = grow(ctx, ctx->recover_rec, 3 * n * N * sizeof(float))) || (rc = grow(ctx, ctx->d_strain_ws, ocb::strain_workspace_bytes(n))))
		return rc;
	char* const b = ctx->recover_ws.as<char>();
	int* const list1 = (int*)b;                                      // reliable / accepted positions
	int* const list2 = (int*)(b + list);                             // unreliable / kept positions
	int* const widx[2] = { (int*)(b + 2 * list), (int*)(b + 3 * list) }; // the working sets' queue indices
	int* const d_counts = (int*)(b + 4 * list);                      // the sizes of list 1 and list 2
	void* const temp = b + 4 * list + 256;
	int* const acc_idx = (int*)(b + 4 * list + 256 + up(temp_bytes)); // with acc: the accepted queue indices
	float* const rel = ctx->recover_rec.as<float>();
	float* const work[2] = { rel + n * N, rel + 2 * n * N };
	auto select = [&](const float* rec, size_t k, ocb::RecoverTest test, int* out, int* count) {
		return launched(ctx, "recover_select",
			ocb::recover_select_launch(m.dim, rec, k, test, zncc_high, zncc_low, m.conv, out, count, temp, temp_bytes, ctx->stream));
	};
	int h[2] = { 0, 0 };
	auto read_counts = [&](int k) {
		OCB_CUDA(ctx, cudaMemcpyAsync(h, d_counts, k * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
		OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		return (int)OCB_OK;
	};
	if ((rc = select(d_q, n, ocb::RecoverTest::RELIABLE, list1, d_counts)) || (rc = select(d_q, n, ocb::RecoverTest::UNRELIABLE, list2, d_counts + 1))
		|| (rc = read_counts(2)))
		return rc;
	size_t n_rel = (size_t)h[0], left_now = (size_t)h[1];
	*left = left_now;
	if (acc) *acc = RecoverAccepted{ acc_idx, rel + n_rel * N, 0 };
	if (max_rounds == 0 || left_now == 0) return OCB_OK;
	if ((rc = launched(ctx, "recover_move", ocb::recover_move_launch(m.dim, d_q, nullptr, n_rel + left_now, list1, d_counts, rel, nullptr, list2, work[0],
			 widx[0], ctx->sm_count, ctx->stream))))
		return rc;
	for (int round = 0, c = 0; round < max_rounds && left_now; round++, c ^= 1) {
		const cudaError_t e = ocb::region_fit_launch(kind, rel, n_rel, work[c], left_now, radius, min_neighbors, ctx->d_strain_ws.p, ctx->sm_count,
			ctx->stream, &ctx->launches);
		if (e != cudaSuccess) return set_error(ctx, OCB_ERR_CUDA, "region_fit launch failed: %s", cudaGetErrorString(e));
		if ((rc = recover_register(ctx, m, img2, img3, work[c], left_now))
			|| (rc = select(work[c], left_now, ocb::RecoverTest::ACCEPTED, list1, d_counts))
			|| (rc = select(work[c], left_now, ocb::RecoverTest::KEPT, list2, d_counts + 1))
			|| (rc = launched(ctx, "recover_move", ocb::recover_move_launch(m.dim, work[c], widx[c], left_now, list1, d_counts, rel + n_rel * N, d_q, list2,
					work[c ^ 1], widx[c ^ 1], ctx->sm_count, ctx->stream)))
			|| (acc
				&& (rc = launched(ctx, "recover_collect",
						ocb::recover_collect_launch(widx[c], left_now, list1, d_counts, acc_idx + acc->count, ctx->sm_count, ctx->stream))))
			|| (rc = read_counts(1)))
			return rc;
		counts->push_back((size_t)h[0]);
		if (acc) acc->count += (size_t)h[0];
		n_rel += (size_t)h[0];
		left_now -= (size_t)h[0];
		*left = left_now;
		if (h[0] == 0) break;
	}
	return OCB_OK;
}

// A recovery call: checks, then (host) the queue staged once in the context's queue buffer, the loop, and the queue back once.
// recovered (max_rounds entries, zero past the last round run) and remaining are written only when the call succeeds.  A
// device-pointer call (dev) returns after synchronising the stream.  On a group context the host variants run on the first member.
static int recover_call(ocb_ctx* ctx, const char* what, bool dev, const RecoverMethod& m, void* q, size_t n, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	if (!dev && is_group(ctx)) // every POI may need any reliable POI: not sharded (as RegionFit)
		return on_exec(ctx, [&](ocb_ctx* x) {
			return recover_call(x, what, false, m, q, n, radius, min_neighbors, zncc_high, zncc_low, max_rounds, recovered, remaining);
		});
	int rc = recover_checks(ctx, what, m, q, n, zncc_high, zncc_low, max_rounds);
	std::vector<size_t> counts;
	size_t left = 0;
	if (rc == PAIR_GO) {
		const size_t bytes = n * (size_t)(m.dim == 2 ? OCB_POI2D_FLOATS : OCB_POI3D_FLOATS) * sizeof(float);
		float* d = (float*)q;
		if (!dev) {
			if ((rc = grow(ctx, ctx->d_poi, bytes))) return rc;
			d = ctx->d_poi.as<float>();
			OCB_CUDA(ctx, cudaMemcpyAsync(d, q, bytes, cudaMemcpyHostToDevice, ctx->stream));
		}
		if ((rc = recover_run(ctx, m, ctx->img2, ctx->img3, d, n, radius, min_neighbors, zncc_high, zncc_low, max_rounds, &counts, &left))) return rc;
		if (!dev) OCB_CUDA(ctx, cudaMemcpyAsync(q, d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
		OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	} else if (rc != OCB_OK) {
		return rc;
	}
	if (recovered) {
		memset(recovered, 0, (size_t)max_rounds * sizeof(size_t));
		if (!counts.empty()) memcpy(recovered, counts.data(), counts.size() * sizeof(size_t));
	}
	if (remaining) *remaining = left;
	return OCB_OK;
}

int ocb_icgn2d_recover(ocb_ctx* ctx, int order, void* poi2d, size_t n, int rx, int ry, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	return recover_call(ctx, "icgn2d_recover", false, { 2, order == 1 ? 6 : (order == 2 ? 12 : 0), { rx, ry, 0 }, conv, stop }, poi2d, n, radius,
		min_neighbors, zncc_high, zncc_low, max_rounds, recovered, remaining);
}
int ocb_icgn2d_recover_dev(ocb_ctx* ctx, int order, void* d_poi2d, size_t n, int rx, int ry, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	OCB_NO_GROUP(ctx, "icgn2d_recover_dev");
	return recover_call(ctx, "icgn2d_recover", true, { 2, order == 1 ? 6 : (order == 2 ? 12 : 0), { rx, ry, 0 }, conv, stop }, d_poi2d, n, radius,
		min_neighbors, zncc_high, zncc_low, max_rounds, recovered, remaining);
}
int ocb_icgn3d_recover(ocb_ctx* ctx, void* poi3d, size_t n, int rx, int ry, int rz, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	return recover_call(ctx, "icgn3d_recover", false, { 3, 0, { rx, ry, rz }, conv, stop }, poi3d, n, radius, min_neighbors, zncc_high, zncc_low,
		max_rounds, recovered, remaining);
}
int ocb_icgn3d_recover_dev(ocb_ctx* ctx, void* d_poi3d, size_t n, int rx, int ry, int rz, float conv, float stop, float radius, int min_neighbors,
	float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	OCB_NO_GROUP(ctx, "icgn3d_recover_dev");
	return recover_call(ctx, "icgn3d_recover", true, { 3, 0, { rx, ry, rz }, conv, stop }, d_poi3d, n, radius, min_neighbors, zncc_high, zncc_low,
		max_rounds, recovered, remaining);
}

// ---- Series that recover unreliable POIs: the recovery rounds in every frame that holds an unreliable record ---------------
// What a series recovery call adds to the plain series: the recovery arguments and the host counts, zeroed on entry.
// recovered[f * max_rounds + k]: the POIs accepted in round k of frame f; remaining[f]: |U| at the end of frame f.
struct SeriesRecover {
	float radius;
	int min_neighbors;
	float zncc_high, zncc_low;
	int max_rounds;
	size_t* recovered;
	size_t* remaining;
};

// recover_run on the n records q of frame f against img2 / img3, its counts stored in sr's slots of frame f
static int series_recover_frame(ocb_ctx* ctx, const RecoverMethod& m, const ocb::Image2D& img2, const ocb::Image3D& img3, float* q, size_t n, int f,
	const SeriesRecover& sr, RecoverAccepted* acc) {
	std::vector<size_t> counts;
	size_t left = 0;
	if (const int rc = recover_run(ctx, m, img2, img3, q, n, sr.radius, sr.min_neighbors, sr.zncc_high, sr.zncc_low, sr.max_rounds, &counts, &left, acc))
		return rc;
	for (size_t k = 0; k < counts.size(); k++) sr.recovered[(size_t)f * sr.max_rounds + k] = counts[k];
	sr.remaining[f] = left;
	return OCB_OK;
}

// The 2D series recovery of reference s.ref against the F frames of s.tar with IC-GN (m) over the n device seeds into d_out:
//   1. one series launch over all n POIs and frames, as the plain series;
//   2. one scan of every record for each POI's first UNRELIABLE frame, whose per-frame counts come back in one copy (none: done);
//   3. for the smallest frame f that holds an unreliable record: the recovery rounds on out[f] against frame f (recover_run, the
//      rounds' IC-GN with the plan of |U|), collecting the accepted POIs' queue indices; one series launch carries the accepted
//      records through frames f + 1 ... F - 1 (into ctx->reseed_cont, the plan of n) and they are scattered into out; the POIs
//      whose first unreliable frame was f, accepted or not, are scanned again from f + 1;
//   4. step 3 repeats for the next frame that holds an unreliable record.
// A POI never accepted keeps its frame-f bytes, so its records of the later frames, already in out, stand.
static int icgn2d_series_recover_run(ocb_ctx* ctx, const RecoverMethod& m, const ocb::Image2D& s, int F, const float* d_seeds, float* d_out, size_t n,
	const SeriesRecover& sr) {
	const SubsetMethod2D sm{ false, m.np == 6 ? 1 : 2, nullptr };
	const size_t frame_px = (size_t)s.w * s.h, rec = OCB_POI2D_FLOATS;
	const int rx = m.r[0], ry = m.r[1];
	int rc;
	if ((rc = subset2d_series_launch(ctx, sm, s, F, d_seeds, d_out, n, n, rx, ry, m.conv, m.stop))) return rc;
	ReseedWs w;
	auto scan = [&](int f_begin, const int* idx, size_t count) {
		const int r = launched(ctx, "recover_scan",
			ocb::recover_scan_launch(2, d_out, n, f_begin, F, idx, count, sr.zncc_low, m.conv, w.first, w.hist, ctx->sm_count, ctx->stream));
		return r ? r : reseed_read_hist(ctx, &w);
	};
	if ((rc = reseed_workspace(ctx, n, F, 2, &w)) || (rc = scan(0, nullptr, n))) return rc;
	for (int f = 0; f < F; f++) {
		const size_t held = (size_t)w.h_hist[f];
		if (!held) continue;
		const ocb::Image2D frame{ s.ref, s.tar + (size_t)f * frame_px, s.w, s.h };
		RecoverAccepted acc;
		if ((rc = series_recover_frame(ctx, m, frame, ocb::Image3D{}, d_out + (size_t)f * n * rec, n, f, sr, f + 1 < F ? &acc : nullptr))) return rc;
		if (f + 1 == F) break;
		if ((rc = launched(ctx, "reseed_select", ocb::reseed_select_launch(w.first, f, n, w.idx, w.count, w.temp, w.temp_bytes, ctx->stream)))) return rc;
		if (acc.count) {
			const int rest = F - f - 1;
			if ((rc = grow(ctx, ctx->reseed_cont, (size_t)rest * acc.count * rec * sizeof(float)))) return rc;
			float* const cont = ctx->reseed_cont.as<float>();
			const ocb::Image2D later{ s.ref, s.tar + (size_t)(f + 1) * frame_px, s.w, s.h };
			if ((rc = subset2d_series_launch(ctx, sm, later, rest, acc.rec, cont, acc.count, n, rx, ry, m.conv, m.stop))
				|| (rc = launched(ctx, "reseed_scatter",
						ocb::reseed_scatter_launch(2, cont, acc.count, rest, acc.idx, d_out, n, f + 1, ctx->sm_count, ctx->stream))))
				return rc;
		}
		if ((rc = scan(f + 1, w.idx, held))) return rc;
	}
	return OCB_OK;
}

// Checks and runs the 2D series recovery on a single-device context (device seeds and out): the series call's checks, then
// recover_refusal and the IC-GN plan, all before any device work.
static int icgn2d_series_recover_dev(ocb_ctx* ctx, const char* what, const RecoverMethod& m, const void* d_seeds, void* d_out, size_t n,
	const SeriesRecover& sr) {
	if (!ctx || ((!d_seeds || !d_out) && n) || m.r[0] < 1 || m.r[1] < 1) return set_error(ctx, OCB_ERR_ARG, "%s: bad arguments", what);
	if (m.np != 6 && m.np != 12) return set_error(ctx, OCB_ERR_ARG, "%s: order must be 1 or 2", what);
	const SeriesStore& s = ctx->series2d;
	if (!s.ref) return set_error(ctx, OCB_ERR_STATE, "%s: no series set", what);
	if (const char* refusal = recover_refusal(m, sr.zncc_high, sr.zncc_low, sr.max_rounds)) return set_error(ctx, OCB_ERR_ARG, "%s: %s", what, refusal);
	if (n == 0) return OCB_OK;
	int rc;
	if ((rc = series_size_check(ctx, what, n, s.frames, OCB_POI2D_FLOATS * sizeof(float), false))) return rc;
	ocb::Icgn2dPlan plan;
	if ((rc = icgn2d_plan_or_error(ctx, n, n, m.np, m.r[0], m.r[1], false, &plan))) return rc;
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	return icgn2d_series_recover_run(ctx, m, s.view2(0), s.frames, (const float*)d_seeds, (float*)d_out, n, sr);
}

static int icgn3d_series_dev(ocb_ctx* ctx, const char* what, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv,
	float stop, const SeriesReseed* rs, const SeriesRecover* sr);

// A series recovery call (dev: device seeds and out): the counts go to recovered / remaining only when it succeeds, and a
// device-pointer call returns after synchronising the stream.  On a group context the first member runs the host variants.
static int series_recover_call(ocb_ctx* ctx, const char* what, bool dev, const RecoverMethod& m, const void* seeds, void* out, size_t n, float radius,
	int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	SeriesStore ocb_ctx::*const which = m.dim == 2 ? &ocb_ctx::series2d : &ocb_ctx::series3d;
	const SeriesStore* s = ctx ? &(exec_member(ctx)->*which) : nullptr;
	const size_t frames = s && s->ref ? (size_t)s->frames : 0, rounds = max_rounds > 0 ? (size_t)max_rounds : 0;
	std::vector<size_t> rec_counts(frames * rounds, 0), left(frames, 0);
	const SeriesRecover sr{ radius, min_neighbors, zncc_high, zncc_low, max_rounds, rec_counts.data(), left.data() };
	auto body = [&](ocb_ctx* x, const void* d_in, void* d_o) {
		return m.dim == 2 ? icgn2d_series_recover_dev(x, what, m, d_in, d_o, n, sr)
						  : icgn3d_series_dev(x, what, d_in, d_o, n, m.r[0], m.r[1], m.r[2], m.conv, m.stop, nullptr, &sr);
	};
	int rc;
	if (dev) {
		rc = body(ctx, seeds, out);
		if (rc == OCB_OK && n) OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	} else {
		const size_t floats = m.dim == 2 ? OCB_POI2D_FLOATS : OCB_POI3D_FLOATS;
		rc = series_host(ctx, what, which, n, { seeds }, floats, { { out, floats } },
			[&](ocb_ctx* x, const float* const* d_in, float* const* d_o) { return body(x, d_in[0], d_o[0]); });
	}
	if (rc != OCB_OK) return rc;
	if (recovered && !rec_counts.empty()) memcpy(recovered, rec_counts.data(), rec_counts.size() * sizeof(size_t));
	if (remaining && !left.empty()) memcpy(remaining, left.data(), left.size() * sizeof(size_t));
	return OCB_OK;
}

int ocb_icgn2d_series_recover(ocb_ctx* ctx, int order, const void* seeds, void* out, size_t n, int rx, int ry, float conv, float stop, float radius,
	int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	return series_recover_call(ctx, "icgn2d_series_recover", false, { 2, order == 1 ? 6 : (order == 2 ? 12 : 0), { rx, ry, 0 }, conv, stop }, seeds, out,
		n, radius, min_neighbors, zncc_high, zncc_low, max_rounds, recovered, remaining);
}
int ocb_icgn2d_series_recover_dev(ocb_ctx* ctx, int order, const void* d_seeds, void* d_out, size_t n, int rx, int ry, float conv, float stop,
	float radius, int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	OCB_NO_GROUP(ctx, "icgn2d_series_recover_dev");
	return series_recover_call(ctx, "icgn2d_series_recover", true, { 2, order == 1 ? 6 : (order == 2 ? 12 : 0), { rx, ry, 0 }, conv, stop }, d_seeds,
		d_out, n, radius, min_neighbors, zncc_high, zncc_low, max_rounds, recovered, remaining);
}
int ocb_icgn3d_series_recover(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, int rz, float conv, float stop, float radius,
	int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	return series_recover_call(ctx, "icgn3d_series_recover", false, { 3, 0, { rx, ry, rz }, conv, stop }, seeds, out, n, radius, min_neighbors,
		zncc_high, zncc_low, max_rounds, recovered, remaining);
}
int ocb_icgn3d_series_recover_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv, float stop,
	float radius, int min_neighbors, float zncc_high, float zncc_low, int max_rounds, size_t* recovered, size_t* remaining) {
	OCB_NO_GROUP(ctx, "icgn3d_series_recover_dev");
	return series_recover_call(ctx, "icgn3d_series_recover", true, { 3, 0, { rx, ry, rz }, conv, stop }, d_seeds, d_out, n, radius, min_neighbors,
		zncc_high, zncc_low, max_rounds, recovered, remaining);
}

// ---- volume series: one reference volume, n_frames target volumes, each frame seeded by the previous one ------------------
// Voxels per volume, or 0 when a dimension is < 15 (TricubicBspline, src/oc_cubic_bspline.cpp:201) or n_frames volumes of
// `voxel` bytes each would not fit in a size_t.
static size_t series3_elems(int n_frames, int dim_x, int dim_y, int dim_z, size_t voxel) {
	if (n_frames < 1 || dim_x < 15 || dim_y < 15 || dim_z < 15) return 0;
	const size_t xy = (size_t)dim_x * dim_y;
	if (xy > SIZE_MAX / (size_t)dim_z) return 0;
	const size_t elems = xy * (size_t)dim_z;
	return elems > SIZE_MAX / voxel / (size_t)n_frames ? 0 : elems;
}

int ocb_set_series_3d_dev(ocb_ctx* ctx, const float* d_ref, const float* d_tars, int n_frames, int dim_x, int dim_y, int dim_z) {
	OCB_NO_GROUP(ctx, "set_series_3d_dev");
	const size_t elems = series3_elems(n_frames, dim_x, dim_y, dim_z, sizeof(float));
	if (!ctx || !d_ref || !d_tars || !elems)
		return set_error(ctx, OCB_ERR_ARG, "set_series_3d: bad arguments (each dimension must be >= 15, n_frames >= 1)");
	series_borrow(ctx->series3d, d_ref, d_tars, nullptr, elems * sizeof(float), n_frames, dim_x, dim_y, dim_z);
	return OCB_OK;
}

int ocb_set_series_3d(ocb_ctx* ctx, const float* ref, const float* tars, int n_frames, int dim_x, int dim_y, int dim_z) {
	return on_exec(ctx, [&](ocb_ctx* x) {
		const size_t elems = series3_elems(n_frames, dim_x, dim_y, dim_z, sizeof(float));
		if (!ref || !tars || !elems) return set_error(x, OCB_ERR_ARG, "set_series_3d: bad arguments (each dimension must be >= 15, n_frames >= 1)");
		const void* stack[1] = { tars };
		return series_upload(x, x->series3d, ref, stack, 1, elems * sizeof(float), elems * sizeof(float), n_frames, dim_x, dim_y, dim_z);
	});
}

// the reference of an 8-bit volume series crosses PCIe as bytes too, staged in the series' scratch volume and widened into the
// reference buffer
static int widen_series3_ref(ocb_ctx* x, const unsigned char* ref, size_t elems) {
	if (const int rc = grow(x, x->series3_tmp, elems * sizeof(float))) return rc;
	OCB_CUDA(x, cudaMemcpyAsync(x->series3_tmp.p, ref, elems, cudaMemcpyHostToDevice, x->stream));
	ocb::widen_u8_kernel<<<x->sm_count * 8, 256, 0, x->stream>>>(x->series3_tmp.as<unsigned char>(), x->series3d.own[0].as<float>(), elems);
	x->launches++;
	OCB_CUDA(x, cudaGetLastError());
	return OCB_OK;
}

int ocb_set_series_3d_u8(ocb_ctx* ctx, const unsigned char* ref, const unsigned char* tars, int n_frames, int dim_x, int dim_y, int dim_z) {
	return on_exec(ctx, [&](ocb_ctx* x) {
		// frames start on 16-byte boundaries: the widening kernel reads uchar4
		const size_t elems = series3_elems(n_frames, dim_x, dim_y, dim_z, 16);
		if (!ref || !tars || !elems)
			return set_error(x, OCB_ERR_ARG, "set_series_3d_u8: bad arguments (each dimension must be >= 15, n_frames >= 1)");
		const void* stack[1] = { tars };
		int rc = series_upload(x, x->series3d, nullptr, stack, 1, elems, (elems + 15) & ~(size_t)15, n_frames, dim_x, dim_y, dim_z);
		if (rc == OCB_OK && (rc = widen_series3_ref(x, ref, elems))) series_clear(x->series3d);
		return rc;
	});
}

// Checks and runs a volume series on a single-device context: device seeds and output; rs and sr null for the plain series.  Per
// frame: the target's prefilter, a copy of the previous frame's records and one LOAD launch; with rs, then a scan of that frame's
// records (one synchronisation), and for its m lost POIs a rebuild, FFT-CC against the raw frame, IC-GN (COMPUTE) and a scatter;
// with sr (series recovery), then the recovery rounds on that frame's records (recover_run), registered by IC-GN (COMPUTE) with the
// series' gradient and coefficient volumes.
static int icgn3d_series_dev(ocb_ctx* ctx, const char* what, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv,
	float stop, const SeriesReseed* rs, const SeriesRecover* sr) {
	if (!ctx || ((!d_seeds || !d_out) && n) || rx < 1 || ry < 1 || rz < 1) return set_error(ctx, OCB_ERR_ARG, "%s: bad arguments", what);
	const SeriesStore& s = ctx->series3d;
	if (!s.ref) return set_error(ctx, OCB_ERR_STATE, "%s: no series set", what);
	int rc;
	if (rs && (rc = reseed_check(ctx, what, 3, *rs))) return rc;
	const RecoverMethod method{ 3, 0, { rx, ry, rz }, conv, stop };
	if (sr)
		if (const char* refusal = recover_refusal(method, sr->zncc_high, sr->zncc_low, sr->max_rounds))
			return set_error(ctx, OCB_ERR_ARG, "%s: %s", what, refusal);
	if (n == 0) return OCB_OK;
	const size_t rec = OCB_POI3D_FLOATS * sizeof(float);
	if ((rc = series_size_check(ctx, what, n, s.frames, rec, false))) return rc;
	ocb::Icgn3dPlan plan;
	if ((rc = icgn3d1_plan_or_error(ctx, rx, ry, rz, &plan))) return rc;
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const int F = s.frames;
	const int dx = s.w, dy = s.h, dz = s.d;
	const size_t elems = (size_t)dx * dy * dz;
	const bool u8 = s.pitch < elems * sizeof(float); // an 8-bit stack, widened into the scratch volume frame by frame
	if ((rc = grow(ctx, ctx->series3_rg, elems * sizeof(float4))) || (rc = grow(ctx, ctx->series3_coef, elems * sizeof(float)))
		|| (rc = grow(ctx, ctx->series3_tmp, elems * sizeof(float))) || (rc = grow(ctx, ctx->series3_cache, n * ocb::ICGN3D_SETUP_FLOATS * sizeof(float))))
		return rc;
	ReseedWs w;
	if (rs && (rc = reseed_workspace(ctx, n, F, 3, &w))) return rc;
	const bool neutral = rs || sr; // the setup pass runs on neutral copies of the seeds (below)
	if (neutral && (rc = grow(ctx, ctx->reseed_sub, n * rec))) return rc;
	float* const sub = neutral ? ctx->reseed_sub.as<float>() : nullptr;
	float4* const rg = ctx->series3_rg.as<float4>();
	float* const coef = ctx->series3_coef.as<float>();
	float* const tmp = ctx->series3_tmp.as<float>();
	float* const cache = ctx->series3_cache.as<float>();
	const ocb::Image3D img{ s.ref, nullptr, rg, coef, dx, dy, dz };
	auto icgn = [&](float* q, size_t m, int setup) {
		return launched(ctx, "icgn3d_series",
			ocb::icgn3d1_launch(plan, img, q, m, rx, ry, rz, conv, stop, ctx->sm_count, ctx->d_counter + 1, ctx->stream, setup, cache));
	};
	auto frame = [&](int f) { return (const char*)s.tars[0] + (size_t)f * s.pitch; };
	auto widen = [&](int f) {
		ocb::widen_u8_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>((const unsigned char*)frame(f), tmp, elems);
		ctx->launches++;
	};
	// the reference's products, once per call: packed gradients, then each POI's setup pass (records are not written).
	// A re-seeding call stores the setup state of neutral copies of the seeds (zero translation, ZNCC 0), so every POI whose
	// subvolume lies inside the volume gets an entry, a seed the guard rejects included: re-seeded in frame f, such a POI
	// reaches frame f + 1's LOAD with a good record.  The setup state depends only on the reference, the coordinates and the
	// radii, so the entries of the POIs the plain series stores are the same; a POI without one (coordinates outside the
	// volume or NaN) is still rejected by every guard.  A recovering call stores them the same way: a POI accepted in frame f
	// reaches frame f + 1's LOAD with a good record, whatever its seed.
	if ((rc = launched(ctx, "gradient3d", ocb::gradient3d_launch(s.ref, rg, dx, dy, dz, ctx->sm_count, ctx->stream)))) return rc;
	if (neutral
		&& (rc = launched(ctx, "reseed_rebuild",
				ocb::reseed_rebuild_launch(3, (const float*)d_seeds, nullptr, nullptr, n, 0.f, nullptr, sub, ctx->sm_count, ctx->stream))))
		return rc;
	if (rs && (rc = launched(ctx, "reseed_anchor_init", ocb::reseed_anchor_init_launch(3, (const float*)d_seeds, n, w.anchor, ctx->sm_count, ctx->stream))))
		return rc;
	if ((rc = icgn(neutral ? sub : const_cast<float*>((const float*)d_seeds), n, ocb::ICGN3D_SETUP_STORE))) return rc;
	for (int f = 0; f < F; f++) {
		if (u8) widen(f);
		const float* const tar = u8 ? tmp : (const float*)frame(f);
		if ((rc = bspline_prefilter(ctx, tar, coef, tmp, dx, dy, dz))) return rc;
		float* const q = (float*)d_out + (size_t)f * n * OCB_POI3D_FLOATS;
		const float* prev = f == 0 ? (const float*)d_seeds : q - n * OCB_POI3D_FLOATS;
		OCB_CUDA(ctx, cudaMemcpyAsync(q, prev, n * rec, cudaMemcpyDeviceToDevice, ctx->stream));
		if ((rc = icgn(q, n, ocb::ICGN3D_SETUP_LOAD))) return rc;
		if (sr && (rc = series_recover_frame(ctx, method, ocb::Image2D{}, img, q, n, f, *sr, nullptr))) return rc;
		if (!rs) continue;
		if ((rc = launched(ctx, "reseed_scan",
				 ocb::reseed_scan_launch(3, (const float*)d_out, n, f, f + 1, nullptr, n, rs->zncc_min, w.first, w.hist, ctx->sm_count, ctx->stream)))
			|| (rc = reseed_read_hist(ctx, &w)))
			return rc;
		const size_t m = (size_t)w.h_hist[f];
		if (!m) continue;
		if ((rc = reseed_gather(ctx, 3, &w, (const float*)d_seeds, f ? prev : nullptr, n, f, m, rs->zncc_min, sub))) return rc;
		if (u8) widen(f); // the prefilter's y pass overwrote the widened frame
		const ocb::Image3D raw{ s.ref, tar, rg, coef, dx, dy, dz };
		if ((rc = fftcc3d_run(ctx, raw, sub, m, rs->fft_r[0], rs->fft_r[1], rs->fft_r[2]))) return rc;
		if ((rc = icgn(sub, m, ocb::ICGN3D_SETUP_COMPUTE))) return rc;
		if ((rc = launched(ctx, "reseed_scatter", ocb::reseed_scatter_launch(3, sub, m, 1, w.idx, (float*)d_out, n, f, ctx->sm_count, ctx->stream))))
			return rc;
		rs->counts[f] = m;
	}
	return OCB_OK;
}

static int icgn3d_series_host(ocb_ctx* ctx, const char* what, const void* seeds, void* out, size_t n, int rx, int ry, int rz, float conv, float stop,
	const SeriesReseed* rs) {
	return series_host(ctx, what, &ocb_ctx::series3d, n, { seeds }, OCB_POI3D_FLOATS, { { out, OCB_POI3D_FLOATS } },
		[&](ocb_ctx* x, const float* const* d_in, float* const* d_out) { return icgn3d_series_dev(x, what, d_in[0], d_out[0], n, rx, ry, rz, conv, stop, rs, nullptr); });
}

int ocb_icgn3d_series_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv, float stop) {
	OCB_NO_GROUP(ctx, "icgn3d_series_dev");
	return icgn3d_series_dev(ctx, "icgn3d_series", d_seeds, d_out, n, rx, ry, rz, conv, stop, nullptr, nullptr);
}

int ocb_icgn3d_series(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, int rz, float conv, float stop) {
	return icgn3d_series_host(ctx, "icgn3d_series", seeds, out, n, rx, ry, rz, conv, stop, nullptr);
}

int ocb_icgn3d_series_reseed_dev(ocb_ctx* ctx, const void* d_seeds, void* d_out, size_t n, int rx, int ry, int rz, float conv, float stop, int fft_rx,
	int fft_ry, int fft_rz, float zncc_min, size_t* reseeded) {
	OCB_NO_GROUP(ctx, "icgn3d_series_reseed_dev");
	return series_reseed(ctx, &ocb_ctx::series3d, true, n, reseeded, [&](size_t* counts) {
		const SeriesReseed rs{ { fft_rx, fft_ry, fft_rz }, zncc_min, counts };
		return icgn3d_series_dev(ctx, "icgn3d_series_reseed", d_seeds, d_out, n, rx, ry, rz, conv, stop, &rs, nullptr);
	});
}

int ocb_icgn3d_series_reseed(ocb_ctx* ctx, const void* seeds, void* out, size_t n, int rx, int ry, int rz, float conv, float stop, int fft_rx,
	int fft_ry, int fft_rz, float zncc_min, size_t* reseeded) {
	return series_reseed(ctx, &ocb_ctx::series3d, false, n, reseeded, [&](size_t* counts) {
		const SeriesReseed rs{ { fft_rx, fft_ry, fft_rz }, zncc_min, counts };
		return icgn3d_series_host(ctx, "icgn3d_series_reseed", seeds, out, n, rx, ry, rz, conv, stop, &rs);
	});
}

int ocb_get_tables_3d(ocb_ctx* ctx, float* gx, float* gy, float* gz, float* coefficient) {
	if (is_group(ctx)) return ocb_get_tables_3d(ctx->members[0], gx, gy, gz, coefficient);
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	if (!ctx->prepared3) return set_error(ctx, OCB_ERR_STATE, "get_tables_3d: prepare() has not been called");
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	const size_t elems = (size_t)ctx->img3.dx * ctx->img3.dy * ctx->img3.dz;
	float* dst[3] = { gx, gy, gz };
	for (int i = 0; i < 3; i++) // de-interleave component i+1 of the packed {ref, gx, gy, gz} volume (inspection path, not hot)
		if (dst[i])
			OCB_CUDA(ctx, cudaMemcpy2DAsync(dst[i], sizeof(float), ctx->rg3.as<const float>() + (i + 1), sizeof(float4), sizeof(float), elems,
				cudaMemcpyDeviceToHost, ctx->stream));
	if (coefficient) OCB_CUDA(ctx, cudaMemcpyAsync(coefficient, ctx->coef3.p, elems * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
	OCB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return OCB_OK;
}

// ---- Stereo reconstruction: Calibration::prepare / undistort, Stereovision::reconstruct --------------------------------------
static int calib_check(ocb_ctx* ctx, const ocb_calib* c, const char* what) {
	if (!c) return set_error(ctx, OCB_ERR_ARG, "%s: null calibration handle", what);
	if (c->owner != ctx) return set_error(ctx, OCB_ERR_ARG, "%s: calibration handle belongs to another context", what);
	return OCB_OK;
}

static void free_calib(ocb_calib* c) {
	if (!c) return;
	if (c->map_x || c->map_y) {
		cudaSetDevice(c->device);
		cudaFree(c->map_x);
		cudaFree(c->map_y);
	}
	delete c;
}

static int calib_build(ocb_ctx* x, ocb_calib* c, const float* intrinsics, float convergence, int iteration) {
	if (ensure_device(x)) return OCB_ERR_CUDA;
	const size_t bytes = (size_t)c->height * c->width * sizeof(float);
	OCB_CUDA(x, cudaMalloc(&c->map_x, bytes));
	OCB_CUDA(x, cudaMalloc(&c->map_y, bytes));
	return launched(x, "calib_map", ocb::calib_map_launch(intrinsics, c->height, c->width, convergence, iteration, c->map_x, c->map_y, x->stream));
}

int ocb_calib_prepare(ocb_ctx* ctx, const float* intrinsics, int height, int width, float convergence, int iteration, ocb_calib** out) {
	if (out) *out = nullptr;
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	if (!intrinsics || !out) return set_error(ctx, OCB_ERR_ARG, "calib_prepare: bad arguments");
	if (height < 2 || width < 2) return set_error(ctx, OCB_ERR_ARG, "calib_prepare: image size %d x %d is below 2 x 2", width, height);
	ocb_ctx* x = exec_member(ctx);
	ocb_calib* c = new ocb_calib;
	c->owner = ctx;
	c->exec = x;
	c->device = x->device;
	c->height = height;
	c->width = width;
	const int rc = calib_build(x, c, intrinsics, convergence, iteration);
	if (rc != OCB_OK) {
		free_calib(c);
		return relay_error(ctx, x, rc);
	}
	*out = c;
	return OCB_OK;
}

void ocb_calib_destroy(ocb_calib* calib) { free_calib(calib); }

int ocb_calib_get_map(ocb_ctx* ctx, const ocb_calib* calib, float* map_x, float* map_y) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	int rc = calib_check(ctx, calib, "calib_get_map");
	if (rc) return rc;
	ocb_ctx* x = calib->exec;
	const size_t bytes = (size_t)calib->height * calib->width * sizeof(float);
	rc = [&]() -> int {
		if (ensure_device(x)) return OCB_ERR_CUDA;
		if (map_x) OCB_CUDA(x, cudaMemcpyAsync(map_x, calib->map_x, bytes, cudaMemcpyDeviceToHost, x->stream));
		if (map_y) OCB_CUDA(x, cudaMemcpyAsync(map_y, calib->map_y, bytes, cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaStreamSynchronize(x->stream));
		return OCB_OK;
	}();
	return relay_error(ctx, x, rc);
}

int ocb_calib_undistort(ocb_ctx* ctx, const ocb_calib* calib, const float* intrinsics, float* pts, float* out, size_t n) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	int rc = calib_check(ctx, calib, "calib_undistort");
	if (rc) return rc;
	if (!intrinsics || ((!pts || !out) && n)) return set_error(ctx, OCB_ERR_ARG, "calib_undistort: bad arguments");
	if (n == 0) return OCB_OK;
	ocb_ctx* x = calib->exec;
	rc = [&]() -> int {
		if (ensure_device(x)) return OCB_ERR_CUDA;
		const size_t bytes = n * 2 * sizeof(float);
		int r = grow(x, x->d_stereo, 2 * bytes);
		if (r) return r;
		float* d_pts = x->d_stereo.as<float>();
		float* d_out = d_pts + 2 * n;
		OCB_CUDA(x, cudaMemcpyAsync(d_pts, pts, bytes, cudaMemcpyHostToDevice, x->stream));
		if ((r = launched(x, "calib_undistort", ocb::calib_undistort_launch(calib->map_x, calib->map_y, calib->height, calib->width, intrinsics, d_pts, d_out,
				 n, x->stream))))
			return r;
		OCB_CUDA(x, cudaMemcpyAsync(pts, d_pts, bytes, cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaStreamSynchronize(x->stream));
		return OCB_OK;
	}();
	return relay_error(ctx, x, rc);
}

static int stereo_check(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, const float* pts1, const float* pts2, const float* pts3d, size_t n) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	int rc = calib_check(ctx, calib1, "stereo_reconstruct");
	if (!rc) rc = calib_check(ctx, calib2, "stereo_reconstruct");
	if (rc) return rc;
	if (!intrinsics1 || !projection1 || !intrinsics2 || !projection2 || ((!pts1 || !pts2 || !pts3d) && n))
		return set_error(ctx, OCB_ERR_ARG, "stereo_reconstruct: bad arguments");
	return OCB_OK;
}

static void stereo_cams(const ocb_calib* c1, const float* i1, const float* p1, const ocb_calib* c2, const float* i2, const float* p2,
	ocb::StereoCam* s1, ocb::StereoCam* s2) {
	*s1 = ocb::StereoCam{ c1->map_x, c1->map_y, c1->height, c1->width, i1, p1 };
	*s2 = ocb::StereoCam{ c2->map_x, c2->map_y, c2->height, c2->width, i2, p2 };
}

int ocb_stereo_reconstruct_dev(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, float* d_pts1, float* d_pts2, float* d_pts3d, size_t n) {
	OCB_NO_GROUP(ctx, "stereo_reconstruct_dev");
	int rc = stereo_check(ctx, calib1, intrinsics1, projection1, calib2, intrinsics2, projection2, d_pts1, d_pts2, d_pts3d, n);
	if (rc) return rc;
	if (n == 0) return OCB_OK;
	if (ensure_device(ctx)) return OCB_ERR_CUDA;
	ocb::StereoCam s1, s2;
	stereo_cams(calib1, intrinsics1, projection1, calib2, intrinsics2, projection2, &s1, &s2);
	return launched(ctx, "stereo_reconstruct", ocb::stereo_reconstruct_launch(s1, s2, d_pts1, d_pts2, d_pts3d, n, ctx->stream));
}

int ocb_stereo_reconstruct(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, float* pts1, float* pts2, float* pts3d, size_t n) {
	int rc = stereo_check(ctx, calib1, intrinsics1, projection1, calib2, intrinsics2, projection2, pts1, pts2, pts3d, n);
	if (rc) return rc;
	if (n == 0) return OCB_OK;
	ocb_ctx* x = calib1->exec;
	rc = [&]() -> int {
		if (ensure_device(x)) return OCB_ERR_CUDA;
		const size_t b2 = n * 2 * sizeof(float), b3 = n * 3 * sizeof(float);
		int r = grow(x, x->d_stereo, 2 * b2 + b3);
		if (r) return r;
		float* d1 = x->d_stereo.as<float>();
		float* d2 = d1 + 2 * n;
		float* d3 = d2 + 2 * n;
		OCB_CUDA(x, cudaMemcpyAsync(d1, pts1, b2, cudaMemcpyHostToDevice, x->stream));
		OCB_CUDA(x, cudaMemcpyAsync(d2, pts2, b2, cudaMemcpyHostToDevice, x->stream));
		ocb::StereoCam s1, s2;
		stereo_cams(calib1, intrinsics1, projection1, calib2, intrinsics2, projection2, &s1, &s2);
		if ((r = launched(x, "stereo_reconstruct", ocb::stereo_reconstruct_launch(s1, s2, d1, d2, d3, n, x->stream)))) return r;
		OCB_CUDA(x, cudaMemcpyAsync(pts1, d1, b2, cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaMemcpyAsync(pts2, d2, b2, cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaMemcpyAsync(pts3d, d3, b3, cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaStreamSynchronize(x->stream));
		return OCB_OK;
	}();
	return relay_error(ctx, x, rc);
}

// ---- Stereo series: both views of every frame registered against reference view 1, triangulated into POI2DS records ---------
// On a group context the first member holds the series and runs the calls; the calibration maps of a group live there too.
int ocb_set_stereo_series_2d_dev(ocb_ctx* ctx, const float* d_ref1, const float* d_tars1, const float* d_tars2, int n_frames, int width, int height) {
	OCB_NO_GROUP(ctx, "set_stereo_series_2d_dev");
	if (!ctx || !d_ref1 || !d_tars1 || !d_tars2 || n_frames < 1 || width < 5 || height < 5)
		return set_error(ctx, OCB_ERR_ARG, "set_stereo_series_2d: bad arguments");
	series_borrow(ctx->stereo, d_ref1, d_tars1, d_tars2, (size_t)width * height * sizeof(float), n_frames, width, height, 1);
	return OCB_OK;
}

int ocb_set_stereo_series_2d(ocb_ctx* ctx, const float* ref1, const float* tars1, const float* tars2, int n_frames, int width, int height) {
	return on_exec(ctx, [&](ocb_ctx* x) {
		if (!ref1 || !tars1 || !tars2 || n_frames < 1 || width < 5 || height < 5) return set_error(x, OCB_ERR_ARG, "set_stereo_series_2d: bad arguments");
		const size_t frame = (size_t)width * height * sizeof(float);
		if ((size_t)n_frames > SIZE_MAX / frame) return set_error(x, OCB_ERR_ARG, "set_stereo_series_2d: series too large");
		const void* stacks[2] = { tars1, tars2 };
		return series_upload(x, x->stereo, ref1, stacks, 2, frame, frame, n_frames, width, height, 1);
	});
}

// The cameras, checked on the caller's context as ocb_stereo_reconstruct checks them
static int stereo_series_cams(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, ocb::StereoCam* s1, ocb::StereoCam* s2) {
	int rc = calib_check(ctx, calib1, "stereo_series");
	if (!rc) rc = calib_check(ctx, calib2, "stereo_series");
	if (rc) return rc;
	if (!intrinsics1 || !projection1 || !intrinsics2 || !projection2) return set_error(ctx, OCB_ERR_ARG, "stereo_series: bad arguments");
	stereo_cams(calib1, intrinsics1, projection1, calib2, intrinsics2, projection2, s1, s2);
	return OCB_OK;
}

// Checks and runs a stereo series call on the context x that holds the series (device pointers), after the cameras' checks.  Every
// check comes before any work: pointers, orders, the series, sizes and the radii (both IC-GN plans, so that a radius one order
// rejects stops the call before the other view runs).  Then the two registrations (each one 2D series launch) and the records.
static int stereo_series_dev(ocb_ctx* x, const ocb::StereoCam& c1, const ocb::StereoCam& c2, int order1, int order2, const float* d_stereo,
	const float* d_seeds1, const float* d_seeds2, float* d_out1, float* d_out2, float* d_out2ds, size_t n, int rx, int ry, float conv, float stop) {
	if (((!d_stereo || !d_seeds1 || !d_seeds2 || !d_out1 || !d_out2 || !d_out2ds) && n) || rx < 1 || ry < 1)
		return set_error(x, OCB_ERR_ARG, "stereo_series: bad arguments");
	if ((order1 != 1 && order1 != 2) || (order2 != 1 && order2 != 2)) return set_error(x, OCB_ERR_ARG, "stereo_series: order must be 1 or 2");
	const SeriesStore& s = x->stereo;
	if (!s.ref) return set_error(x, OCB_ERR_STATE, "stereo_series: no series set");
	if (n == 0) return OCB_OK;
	int rc;
	if ((rc = series_size_check(x, "stereo_series", n, s.frames, (2 * OCB_POI2D_FLOATS + OCB_POI2DS_FLOATS) * sizeof(float), false))) return rc;
	const int np1 = order1 == 1 ? 6 : 12, np2 = order2 == 1 ? 6 : 12;
	ocb::Icgn2dPlan plan;
	if ((rc = icgn2d_plan_or_error(x, n, n, np1, rx, ry, false, &plan)) || (rc = icgn2d_plan_or_error(x, n, n, np2, rx, ry, false, &plan))) return rc;
	if (ensure_device(x)) return OCB_ERR_CUDA;
	if ((rc = subset2d_series_run(x, { false, order1, nullptr }, s.view2(0), s.frames, d_seeds1, d_out1, n, rx, ry, conv, stop, nullptr))) return rc;
	if ((rc = subset2d_series_run(x, { false, order2, nullptr }, s.view2(1), s.frames, d_seeds2, d_out2, n, rx, ry, conv, stop, nullptr))) return rc;
	return launched(x, "stereo_poi2ds", ocb::stereo_poi2ds_launch(c1, c2, d_stereo, d_seeds1, d_out1, d_out2, d_out2ds, n, s.frames, x->stream));
}

int ocb_stereo_series_dev(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, int order1, int order2, const void* d_stereo, const void* d_seeds1, const void* d_seeds2,
	void* d_out1, void* d_out2, void* d_out2ds, size_t n, int rx, int ry, float conv, float stop) {
	OCB_NO_GROUP(ctx, "stereo_series_dev");
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	ocb::StereoCam s1, s2;
	if (const int rc = stereo_series_cams(ctx, calib1, intrinsics1, projection1, calib2, intrinsics2, projection2, &s1, &s2)) return rc;
	return stereo_series_dev(ctx, s1, s2, order1, order2, (const float*)d_stereo, (const float*)d_seeds1, (const float*)d_seeds2, (float*)d_out1,
		(float*)d_out2, (float*)d_out2ds, n, rx, ry, conv, stop);
}

int ocb_stereo_series(ocb_ctx* ctx, const ocb_calib* calib1, const float* intrinsics1, const float* projection1, const ocb_calib* calib2,
	const float* intrinsics2, const float* projection2, int order1, int order2, const void* stereo, const void* seeds1, const void* seeds2,
	void* out1, void* out2, void* out2ds, size_t n, int rx, int ry, float conv, float stop) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	ocb::StereoCam s1, s2;
	if (const int rc = stereo_series_cams(ctx, calib1, intrinsics1, projection1, calib2, intrinsics2, projection2, &s1, &s2)) return rc;
	return series_host(ctx, "stereo_series", &ocb_ctx::stereo, n, { stereo, seeds1, seeds2 }, OCB_POI2D_FLOATS,
		{ { out1, OCB_POI2D_FLOATS }, { out2, OCB_POI2D_FLOATS }, { out2ds, OCB_POI2DS_FLOATS } },
		[&](ocb_ctx* x, const float* const* d_in, float* const* d_out) {
			return stereo_series_dev(x, s1, s2, order1, order2, d_in[0], d_in[1], d_in[2], d_out[0], d_out[1], d_out[2], n, rx, ry, conv, stop);
		});
}

// ---- SIFT3D: SIFT3D::compute (src/oc_sift.cpp:234-293) --------------------------------------------------------------------
// On a group context the first member runs it and keeps the results (one pair of volumes; see DESIGN.md section 6).

// The pyramid of ocb_sift3d on ctx's volumes, or OCB_ERR_ARG with the check it fails
static int sift3d_plan_or_error(ocb_ctx* ctx, const float* config, const float* unit_xyz, ocb::Sift3dPlan* plan) {
	if (ocb::sift3d_plan(ctx->img3.dx, ctx->img3.dy, ctx->img3.dz, config, unit_xyz, plan)) return OCB_OK;
	if (plan->reject == ocb::Sift3dReject::OCTAVE_LAYERS)
		return set_error(ctx, OCB_ERR_ARG, "sift3d: n_octave_layers must be in [1, %d]", ocb::SIFT3D_MAX_L - 3);
	if (plan->reject == ocb::Sift3dReject::VOLUME_SIZE) return set_error(ctx, OCB_ERR_ARG, "sift3d: volume too large");
	return set_error(ctx, OCB_ERR_ARG, "sift3d: blur radius exceeds %d voxels (physical units too anisotropic)", ocb::SIFT3D_MAX_R);
}

int ocb_sift3d(ocb_ctx* ctx, const float* config, const float* unit_xyz, float matching_ratio, size_t* n_matched, int* n_octave) {
	if (!ctx || !config || !unit_xyz) return set_error(ctx, OCB_ERR_ARG, "sift3d: null argument");
	return on_exec(ctx, [&](ocb_ctx* x) -> int {
		if (!x->img3.ref) return set_error(x, OCB_ERR_STATE, "sift3d: images not set");
		for (int a = 0; a < 3; a++)
			if (!(unit_xyz[a] > 0.f) || !std::isfinite(unit_xyz[a])) return set_error(x, OCB_ERR_ARG, "sift3d: physical units must be positive");
		if (!(config[0] >= 1.f) || !(config[2] >= 1.f)) return set_error(x, OCB_ERR_ARG, "sift3d: n_octave_layers and min_dimension must be >= 1");
		ocb::Sift3dPlan plan;
		if (const int rc = sift3d_plan_or_error(x, config, unit_xyz, &plan)) return rc;
		if (ensure_device(x)) return OCB_ERR_CUDA;
		if (!x->sift3d) x->sift3d = new ocb::Sift3d;
		const cudaError_t e =
			ocb::sift3d_run(x->sift3d, plan, x->img3.ref, x->img3.tar, config, matching_ratio, x->sm_count, x->stream, &x->launches);
		if (e != cudaSuccess) { // no results (include/opencorr_b200.h)
			cudaGetLastError(); // a failed copy or event call must not surface as the next launch's error
			delete x->sift3d;
			x->sift3d = nullptr;
			if (e == ocb::SIFT3D_TOO_MANY_KEYPOINTS) return set_error(x, OCB_ERR_ARG, "sift3d: too many keypoints");
			return set_error(x, OCB_ERR_CUDA, "sift3d failed: %s", cudaGetErrorString(e));
		}
		if (n_matched) *n_matched = x->sift3d->ref_xyz.size() / 3;
		if (n_octave) *n_octave = plan.n_octave;
		return OCB_OK;
	});
}

int ocb_sift3d_get_matches(ocb_ctx* ctx, float* ref_xyz, float* tar_xyz) {
	if (!ctx) return set_error(nullptr, OCB_ERR_ARG, "null context");
	ocb_ctx* x = exec_member(ctx);
	if (!x->sift3d) return relay_error(ctx, x, set_error(x, OCB_ERR_STATE, "sift3d_get_matches: ocb_sift3d has not run"));
	if (ref_xyz) std::copy(x->sift3d->ref_xyz.begin(), x->sift3d->ref_xyz.end(), ref_xyz);
	if (tar_xyz) std::copy(x->sift3d->tar_xyz.begin(), x->sift3d->tar_xyz.end(), tar_xyz);
	return OCB_OK;
}

int ocb_sift3d_inspect(ocb_ctx* ctx, int image, size_t* counts, int* candidates, float* max_abs, float* keypoints, float* descriptors) {
	if (!ctx || !counts || (image != 0 && image != 1)) return set_error(ctx, OCB_ERR_ARG, "sift3d_inspect: bad arguments");
	return on_exec(ctx, [&](ocb_ctx* x) -> int {
		if (!x->sift3d) return set_error(x, OCB_ERR_STATE, "sift3d_inspect: ocb_sift3d has not run");
		if (ensure_device(x)) return OCB_ERR_CUDA;
		const ocb::Sift3dImage& im = x->sift3d->img[image];
		const size_t n[3] = { im.n_cand, im.max_abs.size(), im.n_kp };
		std::copy(n, n + 3, counts);
		if (max_abs) std::copy(im.max_abs.begin(), im.max_abs.end(), max_abs);
		const size_t cand_bytes = 5 * im.n_cand * sizeof(int), kp_bytes = im.n_kp * s3::KP_FLOATS * sizeof(float);
		if (candidates && im.n_cand) OCB_CUDA(x, cudaMemcpyAsync(candidates, im.cand.p, cand_bytes, cudaMemcpyDeviceToHost, x->stream));
		if (keypoints && im.n_kp) OCB_CUDA(x, cudaMemcpyAsync(keypoints, im.kp.p, kp_bytes, cudaMemcpyDeviceToHost, x->stream));
		if (descriptors && im.n_kp)
			OCB_CUDA(x, cudaMemcpyAsync(descriptors, im.desc.p, im.n_kp * s3::DESC * sizeof(float), cudaMemcpyDeviceToHost, x->stream));
		OCB_CUDA(x, cudaStreamSynchronize(x->stream));
		return OCB_OK;
	});
}

int ocb_sift3d_stage_times(ocb_ctx* ctx, float* ms) {
	if (!ctx || !ms) return set_error(ctx, OCB_ERR_ARG, "sift3d_stage_times: bad arguments");
	ocb_ctx* x = exec_member(ctx);
	if (!x->sift3d) return relay_error(ctx, x, set_error(x, OCB_ERR_STATE, "sift3d_stage_times: ocb_sift3d has not run"));
	std::copy(x->sift3d->stage_ms, x->sift3d->stage_ms + ocb::SIFT3D_STAGES, ms);
	return OCB_OK;
}

} // extern "C"
