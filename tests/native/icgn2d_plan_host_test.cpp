// Host-side check of the 2D subset-registration launch plans (ocb::icgn2d_plan and ocb::nr2d1_plan in
// opencorr_b200/csrc/ocb_kernels.h): every case of tests/test_gpu_2d_geometry.py must select the kernel instantiation, lane
// layout and row split that it is meant to cover, so that a retune of a plan cannot silently turn a case into a copy of another.
// Built and run by tests/test_icgn2d_plan_host.py (needs nvcc, no GPU).  Prints one line per case; exit code 0 = every
// expectation holds.
//
//   icgn2d_plan_host_test                          the table of cases, for an H100 (132 SMs, 227 KB opt-in)
//   icgn2d_plan_host_test query OPTIN RX RY LM     for a device with OPTIN bytes of opt-in shared memory: the largest square
//                                                  radius each kernel family accepts, and the resident one-warp CTAs per SM
//                                                  (slots) of radius (RX, RY)
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "ocb_kernels.h"
using namespace ocb;

namespace {

constexpr size_t H100_SMEM_OPTIN = 227 * 1024; // cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
constexpr int H100_SMS = 132;                  // H100 SXM

// n: queue length; AUTO_BELOW / AUTO_FULL stand for sm_count x slots(1) - 1 and sm_count x slots(1) POIs.
// wpp: 1 or 2 forces the warps per POI (OCB_ICGN2D_WPP), 0 leaves the choice to the queue length.
// kernel: "<NP,RC,LM,WPP>" or "reject"; idle: lanes without a column (2rx+1 < 32); tail: columns beyond 32 (2rx+1 > 32);
// rem: each warp's rolling-window remainder, (rows - 1) mod 4 ("a/b" for two warps per POI).
constexpr long AUTO_BELOW = -1, AUTO_FULL = -2;
struct Icgn2dCase {
	const char* label;
	long n;
	int np, rx, ry;
	bool lm;
	int wpp;
	const char* kernel;
	int idle, tail;
	const char* rem;
};

const Icgn2dCase icgn2d_cases[] = {
	{ "sweep", 32, 6, 4, 4, false, 1, "<6,0,0,1>", 23, 0, "0" },
	{ "sweep", 32, 6, 4, 4, false, 2, "<6,0,0,2>", 23, 0, "0/3" },
	{ "sweep", 32, 6, 5, 6, false, 1, "<6,0,0,1>", 21, 0, "0" },
	{ "sweep", 32, 6, 5, 6, false, 2, "<6,0,0,2>", 21, 0, "2/1" },
	{ "sweep", 32, 6, 6, 7, false, 1, "<6,0,0,1>", 19, 0, "2" },
	{ "sweep", 32, 6, 6, 7, false, 2, "<6,0,0,2>", 19, 0, "3/2" },
	{ "sweep", 32, 6, 7, 5, false, 1, "<6,0,0,1>", 17, 0, "2" },
	{ "sweep", 32, 6, 7, 5, false, 2, "<6,0,0,2>", 17, 0, "1/0" },
	{ "sweep", 32, 6, 15, 15, false, 1, "<6,0,0,1>", 1, 0, "2" },
	{ "sweep", 32, 6, 15, 15, false, 2, "<6,0,0,2>", 1, 0, "3/2" },
	{ "sweep", 32, 6, 16, 16, false, 1, "<6,16,0,1>", 0, 1, "0" },
	{ "sweep", 32, 6, 16, 16, false, 2, "<6,16,0,2>", 0, 1, "0/3" },
	{ "sweep", 32, 6, 16, 15, false, 1, "<6,0,0,1>", 0, 1, "2" },
	{ "sweep", 32, 6, 16, 15, false, 2, "<6,0,0,2>", 0, 1, "3/2" },
	{ "sweep", 32, 6, 24, 9, false, 1, "<6,0,0,1>", 0, 17, "2" },
	{ "sweep", 32, 6, 24, 9, false, 2, "<6,0,0,2>", 0, 17, "1/0" },
	{ "sweep", 8, 6, 40, 40, false, 1, "<6,0,0,1>", 0, 49, "0" },
	{ "sweep", 8, 6, 40, 40, false, 2, "<6,0,0,2>", 0, 49, "0/3" },
	{ "sweep", 32, 6, 20, 2, false, 0, "<6,0,0,1>", 0, 9, "0" }, // 5 rows: the queue length does not matter
	{ "sweep", 32, 6, 20, 2, false, 2, "<6,0,0,2>", 0, 9, "2/1" },
	{ "sweep", 32, 12, 20, 20, false, 1, "<12,20,0,1>", 0, 9, "0" },
	{ "sweep", 32, 12, 20, 20, false, 2, "<12,20,0,2>", 0, 9, "0/3" },
	{ "sweep", 32, 12, 20, 19, false, 1, "<12,0,0,1>", 0, 9, "2" },
	{ "sweep", 32, 12, 20, 19, false, 2, "<12,0,0,2>", 0, 9, "3/2" },
	{ "sweep", 32, 12, 11, 11, false, 1, "<12,0,0,1>", 9, 0, "2" },
	{ "sweep", 32, 12, 11, 11, false, 2, "<12,0,0,2>", 9, 0, "3/2" },
	{ "sweep", 16, 12, 33, 8, false, 1, "<12,0,0,1>", 0, 35, "0" },
	{ "sweep", 16, 12, 33, 8, false, 2, "<12,0,0,2>", 0, 35, "0/3" },
	{ "sweep", 32, 6, 12, 12, true, 1, "<6,0,1,1>", 7, 0, "0" },
	{ "sweep", 32, 6, 12, 12, true, 2, "<6,0,1,2>", 7, 0, "0/3" },
	{ "sweep", 32, 6, 17, 17, true, 1, "<6,0,1,1>", 0, 3, "2" },
	{ "sweep", 32, 6, 17, 17, true, 2, "<6,0,1,2>", 0, 3, "1/0" },
	{ "sweep", 32, 12, 12, 12, true, 1, "<12,0,1,1>", 7, 0, "0" },
	{ "sweep", 32, 12, 12, 12, true, 2, "<12,0,1,2>", 7, 0, "0/3" },
	{ "sweep", 32, 12, 17, 17, true, 1, "<12,0,1,1>", 0, 3, "2" },
	{ "sweep", 32, 12, 17, 17, true, 2, "<12,0,1,2>", 0, 3, "1/0" },
	// the largest square subsets, and the first rejected one
	{ "largest", 3, 6, 58, 58, false, 1, "<6,0,0,1>", 0, 85, "0" },
	{ "largest", 3, 6, 58, 58, false, 2, "<6,0,0,2>", 0, 85, "2/1" },
	{ "largest", 3, 12, 58, 58, false, 1, "<12,0,0,1>", 0, 85, "0" },
	{ "largest", 3, 12, 58, 58, false, 2, "<12,0,0,2>", 0, 85, "2/1" },
	{ "largest", 3, 6, 58, 58, true, 1, "<6,0,1,1>", 0, 85, "0" },
	{ "largest", 3, 6, 58, 58, true, 2, "<6,0,1,2>", 0, 85, "2/1" },
	{ "too large", 2, 6, 59, 59, false, 0, "reject", 0, 0, "-" },
	{ "too large", 2, 6, 59, 59, false, 2, "reject", 0, 0, "-" },
	{ "too large", 2, 12, 59, 59, false, 0, "reject", 0, 0, "-" },
	{ "too large", 2, 6, 59, 59, true, 0, "reject", 0, 0, "-" },
	// the automatic warps-per-POI rule: two warps only while the queue cannot fill every one-warp slot
	{ "auto", AUTO_BELOW, 6, 40, 40, false, 0, "<6,0,0,2>", 0, 49, "0/3" },
	{ "auto", AUTO_FULL, 6, 40, 40, false, 0, "<6,0,0,1>", 0, 49, "0" },
	// sheared targets: the corner test fails and samples leave the tile
	{ "shear", 16, 6, 16, 16, false, 1, "<6,16,0,1>", 0, 1, "0" },
	{ "shear", 16, 6, 16, 16, false, 2, "<6,16,0,2>", 0, 1, "0/3" },
	{ "shear", 16, 6, 11, 11, false, 1, "<6,0,0,1>", 9, 0, "2" },
	{ "shear", 16, 6, 11, 11, false, 2, "<6,0,0,2>", 9, 0, "3/2" },
	{ "shear", 16, 12, 20, 20, false, 1, "<12,20,0,1>", 0, 9, "0" },
	{ "shear", 16, 12, 20, 20, false, 2, "<12,20,0,2>", 0, 9, "0/3" },
	{ "shear", 16, 6, 12, 12, true, 1, "<6,0,1,1>", 7, 0, "0" },
	{ "shear", 16, 6, 12, 12, true, 2, "<6,0,1,2>", 7, 0, "0/3" },
	// non-integral centre offsets
	{ "offsets", 32, 6, 15, 15, false, 1, "<6,0,0,1>", 1, 0, "2" },
	{ "offsets", 32, 6, 15, 15, false, 2, "<6,0,0,2>", 1, 0, "3/2" },
	{ "offsets", 32, 12, 20, 20, false, 1, "<12,20,0,1>", 0, 9, "0" },
	{ "offsets", 32, 12, 20, 20, false, 2, "<12,20,0,2>", 0, 9, "0/3" },
	// samples outside the image
	{ "edges", 32, 6, 14, 14, false, 2, "<6,0,0,2>", 3, 0, "2/1" },
	{ "edges", 32, 12, 14, 14, false, 2, "<12,0,0,2>", 3, 0, "2/1" },
	{ "edges", 32, 6, 14, 14, true, 2, "<6,0,1,2>", 3, 0, "2/1" },
	{ "edges", 32, 12, 14, 14, true, 2, "<12,0,1,2>", 3, 0, "2/1" },
	// the exact-negative rescan away from r = 16
	{ "negative", 400, 6, 11, 11, false, 2, "<6,0,0,2>", 9, 0, "3/2" },
	{ "negative", 400, 12, 20, 20, false, 2, "<12,20,0,2>", 0, 9, "0/3" },
	// large image coordinates
	{ "large xy", 24, 12, 18, 18, false, 2, "<12,0,0,2>", 0, 5, "2/1" },
	{ "large xy", 24, 6, 16, 16, true, 2, "<6,0,1,2>", 0, 1, "0/3" },
};

// warps: NR2D1 warps per CTA (0: rejected); tail: columns beyond 32
struct Nr2dCase {
	const char* label;
	int rx, ry;
	int warps, tail;
};

const Nr2dCase nr2d_cases[] = {
	{ "nr sweep", 4, 4, 4, 0 },
	{ "nr sweep", 8, 8, 2, 0 },
	{ "nr sweep", 12, 12, 1, 0 },
	{ "nr sweep", 16, 16, 4, 1 },
	{ "nr sweep", 18, 18, 1, 5 },
	{ "nr sweep", 20, 20, 2, 9 },
	{ "nr sweep", 24, 9, 2, 17 },
	{ "nr sweep", 40, 40, 1, 49 },
	{ "nr shear", 14, 14, 2, 0 },
	{ "nr edges", 14, 14, 2, 0 },
	{ "nr largest", 56, 56, 1, 81 },
	{ "nr too large", 57, 57, 0, 0 },
};

void remainders(int ry, int wpp, char* out, size_t len) {
	const int sh = 2 * ry + 1, rows_per = (sh + wpp - 1) / wpp;
	out[0] = 0;
	for (int sub = 0; sub < wpp; sub++) {
		const int lo = sub * rows_per, hi = lo + rows_per < sh ? lo + rows_per : sh;
		const size_t k = strlen(out);
		snprintf(out + k, len - k, sub ? "/%d" : "%d", (hi - lo - 1) % 4);
	}
}

int largest_icgn2d(bool lm, int wpp, size_t optin) {
	int r = 0;
	Icgn2dPlan p;
	while (icgn2d_plan(1, 6, r + 1, r + 1, lm, 1, optin, wpp, &p) && p.wpp == wpp) r++;
	return r;
}

int largest_nr2d(size_t optin) {
	int r = 0;
	Nr2dPlan p;
	while (nr2d1_plan(r + 1, r + 1, optin, &p)) r++;
	return r;
}

int query(size_t optin, int rx, int ry, bool lm) {
	for (int l = 0; l < 2; l++)
		for (int w = 1; w <= 2; w++) printf("largest icgn2d lm=%d wpp=%d: %d\n", l, w, largest_icgn2d(l != 0, w, optin));
	printf("largest nr2d1: %d\n", largest_nr2d(optin));
	printf("slots r=(%d,%d) lm=%d wpp=1: %d\n", rx, ry, (int)lm, icgn2d_slots(rx, ry, lm, 1, optin));
	return 0;
}

} // namespace

int main(int argc, char** argv) {
	if (argc == 6 && strcmp(argv[1], "query") == 0) return query((size_t)atol(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]) != 0);
	int failures = 0;
	for (const Icgn2dCase& c : icgn2d_cases) {
		long n = c.n;
		if (n < 0) n = (long)H100_SMS * icgn2d_slots(c.rx, c.ry, c.lm, 1, H100_SMEM_OPTIN) - (n == AUTO_BELOW ? 1 : 0);
		const int sw = 2 * c.rx + 1;
		Icgn2dPlan p;
		char kernel[32], rem[16];
		int idle = 0, tail = 0;
		snprintf(rem, sizeof(rem), "-");
		if (!icgn2d_plan((size_t)n, c.np, c.rx, c.ry, c.lm, H100_SMS, H100_SMEM_OPTIN, c.wpp, &p)) {
			snprintf(kernel, sizeof(kernel), "reject");
			printf("%-10s np=%d r=(%d,%d) lm=%d wpp=%d n=%ld: rejected\n", c.label, c.np, c.rx, c.ry, (int)c.lm, c.wpp, n);
		} else {
			snprintf(kernel, sizeof(kernel), "<%d,%d,%d,%d>", c.np, p.rc, (int)c.lm, p.wpp);
			idle = sw < 32 ? 32 - sw : 0;
			tail = sw > 32 ? sw - 32 : 0;
			remainders(c.ry, p.wpp, rem, sizeof(rem));
			printf("%-10s np=%d r=(%d,%d) lm=%d wpp=%d n=%ld: kernel %s, %d idle lane(s), %d tail column(s), remainder %s, %d CTA/SM, grid %d, %zu B smem\n",
				c.label, c.np, c.rx, c.ry, (int)c.lm, c.wpp, n, kernel, idle, tail, rem, p.blocks_per_sm, p.grid, p.smem);
			// internal consistency: the slab fits the opt-in limit and the resident CTAs the SM
			if (p.smem > H100_SMEM_OPTIN || p.blocks_per_sm < 1 || p.blocks_per_sm * (p.smem + 1024) > 228 * 1024 || p.grid < 1
				|| (long)p.grid > (n > 0 ? n : 1) || p.grid > H100_SMS * p.blocks_per_sm) {
				printf("  FAIL: inconsistent plan\n");
				failures++;
			}
		}
		if (strcmp(kernel, c.kernel) != 0 || idle != c.idle || tail != c.tail || strcmp(rem, c.rem) != 0) {
			printf("  FAIL: expected kernel %s, %d idle, %d tail, remainder %s\n", c.kernel, c.idle, c.tail, c.rem);
			failures++;
		}
	}
	for (const Nr2dCase& c : nr2d_cases) {
		Nr2dPlan p;
		int warps = 0, tail = 0;
		if (!nr2d1_plan(c.rx, c.ry, H100_SMEM_OPTIN, &p)) {
			printf("%-12s r=(%d,%d): rejected\n", c.label, c.rx, c.ry);
		} else {
			warps = p.warps_per_cta;
			tail = 2 * c.rx + 1 > 32 ? 2 * c.rx + 1 - 32 : 0;
			printf("%-12s r=(%d,%d): %d warp(s) per CTA, %d CTA/SM, %d tail column(s), %zu B smem\n", c.label, c.rx, c.ry, warps, p.ctas_per_sm, tail,
				p.smem);
			if (p.smem > H100_SMEM_OPTIN || p.ctas_per_sm < 1 || p.ctas_per_sm * (p.smem + 1024) > 228 * 1024) {
				printf("  FAIL: inconsistent plan\n");
				failures++;
			}
		}
		if (warps != c.warps || tail != c.tail) {
			printf("  FAIL: expected %d warp(s) per CTA, %d tail; got %d, %d\n", c.warps, c.tail, warps, tail);
			failures++;
		}
	}
	// the "largest" and "too large" rows above are the limits: nothing in between
	for (int l = 0; l < 2; l++)
		for (int w = 1; w <= 2; w++)
			if (largest_icgn2d(l != 0, w, H100_SMEM_OPTIN) != 58) {
				printf("FAIL: largest ICGN2D radius (lm=%d, wpp=%d) is %d, not 58\n", l, w, largest_icgn2d(l != 0, w, H100_SMEM_OPTIN));
				failures++;
			}
	if (largest_nr2d(H100_SMEM_OPTIN) != 56) {
		printf("FAIL: largest NR2D1 radius is %d, not 56\n", largest_nr2d(H100_SMEM_OPTIN));
		failures++;
	}
	printf("%d failure(s)\n", failures);
	return failures ? 1 : 0;
}
