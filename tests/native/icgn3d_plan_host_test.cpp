// Host-side check of the ICGN3D1 launch plan (ocb::icgn3d1_plan in opencorr_b200/csrc/ocb_kernels.h): every subvolume radius
// set of tests/test_gpu_3d_geometry.py must select the kernel variant and slab layout that its GPU case is meant to cover, so
// that a retune of the plan cannot silently turn a case into a copy of another.  Built and run by tests/test_icgn3d_plan_host.py
// (needs nvcc, no GPU).  Prints one line per radius set; exit code 0 = every expectation holds.
#include <cstdio>
#include <cstring>

#include "ocb_kernels.h"
using namespace ocb;

namespace {

constexpr size_t H100_SMEM_OPTIN = 227 * 1024; // cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100

// What a case is meant to exercise.  kernel: "<RC,THREADS>" or "reject"; slabs: 1 = single slab, 2 = several slabs of equal
// thickness, 3 = several slabs with a thinner last one; tail: subset columns beyond 32 (2rx+1 > 32).
struct Case {
	const char* label;
	int rx, ry, rz;
	const char* kernel;
	int slabs;
	bool tail;
};

const Case cases[] = {
	{ "sweep", 8, 8, 8, "<0,256>", 1, false },
	{ "sweep", 12, 12, 12, "<0,256>", 3, false },
	{ "sweep", 16, 16, 16, "<16,256>", 2, true },
	{ "sweep", 16, 16, 15, "<0,256>", 3, true },
	{ "sweep", 20, 20, 20, "<0,256>", 3, true },
	{ "sweep", 22, 22, 22, "<0,512>", 2, true },
	{ "sweep", 24, 24, 24, "<0,512>", 3, true },
	{ "sweep", 30, 30, 30, "<30,512>", 3, true },
	{ "sweep", 40, 40, 40, "<0,512>", 3, true },
	{ "sweep", 24, 8, 30, "<0,256>", 3, true },
	{ "sweep", 30, 30, 12, "<0,512>", 2, true },
	{ "shear", 14, 14, 14, "<0,256>", 3, false },
	{ "long queue", 22, 22, 22, "<0,512>", 2, true },
	{ "sentinels", 24, 24, 24, "<0,512>", 3, true },
	{ "sentinels", 12, 12, 12, "<0,256>", 3, false },
	{ "large z", 8, 8, 8, "<0,256>", 1, false },
	{ "large z", 16, 16, 16, "<16,256>", 2, true },
	{ "largest", 43, 43, 43, "<0,512>", 2, true },
	{ "too large", 44, 44, 44, "reject", 0, false },
};

} // namespace

int main() {
	int failures = 0;
	for (const Case& c : cases) {
		Icgn3dPlan p;
		char kernel[32];
		const int sz = 2 * c.rz + 1, sx = 2 * c.rx + 1;
		int tail = sx > 32 ? sx - 32 : 0, slabs = 0, last = 0;
		if (!icgn3d1_plan(c.rx, c.ry, c.rz, H100_SMEM_OPTIN, &p)) {
			snprintf(kernel, sizeof(kernel), "reject");
			tail = 0;
			printf("%-10s r=(%d,%d,%d): rejected\n", c.label, c.rx, c.ry, c.rz);
		} else {
			snprintf(kernel, sizeof(kernel), "<%d,%d>", p.rc, p.threads);
			last = sz - (p.nslab - 1) * p.slab_k;
			slabs = p.nslab == 1 ? 1 : (last == p.slab_k ? 2 : 3);
			printf("%-10s r=(%d,%d,%d): %d CTA/SM x %d threads, kernel %s, %d slab(s) x %d layers (last %d), %d tail column(s), %zu B dynamic smem\n",
				c.label, c.rx, c.ry, c.rz, p.ctas_per_sm, p.threads, kernel, p.nslab, p.slab_k, last, tail, p.smem);
			// internal consistency: the slabs cover the subvolume exactly, the tile fits the CTA's share of the SM
			if ((p.nslab - 1) * p.slab_k >= sz || p.nslab * p.slab_k < sz || last < 1 || p.ctas_per_sm * p.threads != 512
				|| p.smem + sizeof(Icgn3dShared) > H100_SMEM_OPTIN || p.ctas_per_sm * (p.smem + sizeof(Icgn3dShared) + 1024) > 228 * 1024) {
				printf("  FAIL: inconsistent plan\n");
				failures++;
			}
		}
		if (strcmp(kernel, c.kernel) != 0 || slabs != c.slabs || (tail > 0) != c.tail) {
			printf("  FAIL: expected kernel %s, slab kind %d, tail %d; got %s, %d, %d\n", c.kernel, c.slabs, (int)c.tail, kernel, slabs, tail);
			failures++;
		}
	}
	printf("%d failure(s)\n", failures);
	return failures ? 1 : 0;
}
