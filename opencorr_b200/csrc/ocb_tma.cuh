// ocb_tma.cuh -- TMA (cp.async.bulk.tensor) + mbarrier primitives and the host-side tensor-map helper.
// Callers keep the innermost tile coordinate 16-byte aligned (x multiple of 4 floats; an unaligned
// x was seen to raise "illegal instruction"); negative / past-the-end coordinates are fine and read
// as zero.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

namespace ocb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
	asm volatile(
		"{\n\t"
		".reg .pred p;\n\t"
		"WAIT_LOOP:\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
		"@p bra.uni WAIT_DONE;\n\t"
		"bra.uni WAIT_LOOP;\n\t"
		"WAIT_DONE:\n\t"
		"}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// tile loads: box size is part of the tensor map; (x, y[, z]) is the box's first element
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)),
		"l"(map), "r"(x), "r"(y), "r"(smem_u32(bar))
		: "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
	asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_u32(dst)),
		"l"(map), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
		: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__host__ __device__ inline int round_up4(int v) { return (v + 3) & ~3; }
__host__ __device__ inline int round_up32(int v) { return (v + 31) & ~31; }
__host__ __device__ inline int floor4(int v) { return v & ~3; } // rounds toward -inf (two's complement)

// ---- host side ------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
	const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn tma_encode_fn() {
	static EncodeTiledFn fn = nullptr;
	static bool tried = false;
	if (!tried) {
		tried = true;
		void* p = nullptr;
		cudaDriverEntryPointQueryResult qres;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
			fn = (EncodeTiledFn)p;
	}
	return fn;
}

// false when OCB_NO_TMA is set: every launch then stages its tiles with ordinary loads.  Read at each launch, so that a
// process can switch between the two load paths.
inline bool tma_enabled() { return !getenv("OCB_NO_TMA"); }

// Tensor map over a dense row-major f32 array of rank 2 or 3 (dims[0] = innermost) for box-shaped tile
// loads.  Returns false when TMA cannot be used: pitch or base not 16-byte aligned, a box extent > 256,
// or the driver entry point is missing -- callers then stage tiles with ordinary loads.
inline bool tma_make_map(CUtensorMap* map, const float* base, int rank, const int* dims, const int* box) {
	EncodeTiledFn fn = tma_encode_fn();
	if (!fn || rank < 2 || rank > 3 || (dims[0] % 4) != 0 || ((uintptr_t)base % 16) != 0) return false;
	cuuint64_t gdims[3], gstrides[2];
	cuuint32_t gbox[3], estr[3] = { 1, 1, 1 };
	cuuint64_t pitch = sizeof(float);
	for (int i = 0; i < rank; i++) {
		if (box[i] < 1 || box[i] > 256) return false;
		gdims[i] = (cuuint64_t)dims[i];
		gbox[i] = (cuuint32_t)box[i];
		pitch *= (cuuint64_t)dims[i];
		if (i < rank - 1) gstrides[i] = pitch;
	}
	if ((box[0] % 4) != 0) return false;
	return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, (void*)base, gdims, gstrides, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
			   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

} // namespace ocb
