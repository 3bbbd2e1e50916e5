// Host-side view of the FFTCC2D routing (ocb::fftcc2d_plan in opencorr_b200/csrc/ocb_kernels.h): which of the three kernels a
// window takes, the Stockham factorisation of both axes, the shared memory and the POIs per CTA.  Built and run by
// tests/test_fftcc2d_plan_host.py (needs nvcc, no GPU), which feeds it every case of tests/test_gpu_fftcc2d_geometry.py and
// checks that each lands where that file says, so that a change of the routing cannot silently turn a case into a copy of another.
//
//   fftcc2d_plan_host_test OPTIN < cases     one line per case "rx ry force_generic n" read from stdin, for a device with OPTIN
//                                            bytes of opt-in shared memory per block
//   fftcc2d_plan_host_test limits OPTIN      the largest square radius the GENERIC kernel accepts with OPTIN bytes, and the first
//                                            radius above it that is refused for its shared memory
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "ocb_kernels.h"
using namespace ocb;

namespace {

void print_axis(const char* name, const FftAxis& a) {
	printf(" %s=[", name);
	for (int i = 0; i < a.nstage; i++) printf(i ? ",%d" : "%d", a.radix[i]);
	printf("]");
}

const char* reason(Fftcc2dReject r) { return r == Fftcc2dReject::PRIME_FACTOR ? "prime factor" : "shared memory"; }

int limits(size_t optin) {
	int largest = 0, first_smem = 0;
	Fftcc2dPlan p;
	for (int r = 1; r <= 256 && !first_smem; r++) {
		if (fftcc2d_plan(r, r, true, optin, &p)) largest = r;
		else if (p.reject == Fftcc2dReject::SHARED_MEMORY) first_smem = r;
	}
	printf("largest generic: %d\nfirst refused for shared memory: %d\n", largest, first_smem);
	return 0;
}

} // namespace

int main(int argc, char** argv) {
	if (argc == 3 && strcmp(argv[1], "limits") == 0) return limits((size_t)atol(argv[2]));
	if (argc != 2) return 2;
	const size_t optin = (size_t)atol(argv[1]);
	int rx, ry, force;
	long n;
	int failures = 0;
	while (scanf("%d %d %d %ld", &rx, &ry, &force, &n) == 4) {
		Fftcc2dPlan p;
		printf("r=(%d,%d) force=%d n=%ld: ", rx, ry, force, n);
		if (!fftcc2d_plan(rx, ry, force != 0, optin, &p)) {
			printf("rejected (%s), %zu B smem\n", reason(p.reject), p.smem);
			continue;
		}
		const int pp = p.pois_per_cta;
		if (p.path == Fftcc2dPath::W32) {
			printf("kernel W32, PP=%d, %ld CTA(s), %ld POI(s) in the last\n", pp, (n + pp - 1) / pp, (n - 1) % pp + 1);
		} else if (p.path == Fftcc2dPath::REG) {
			const int N = 2 * rx;
			printf("kernel REG, N=%d PP=%d, %d idle thread(s), %ld batch(es), %ld POI(s) in the last, %zu B smem\n", N, pp, FFTREG_THREADS - pp * N,
				(n + pp - 1) / pp, (n - 1) % pp + 1, p.smem);
		} else {
			printf("kernel GENERIC, M=%d, %zu B smem,", 4 * rx * ry, p.smem);
			print_axis("x", p.ax);
			print_axis("y", p.ay);
			printf("\n");
			// internal consistency: the stages multiply back to the axis length
			int mx = 1, my = 1;
			for (int i = 0; i < p.ax.nstage; i++) mx *= p.ax.radix[i];
			for (int i = 0; i < p.ay.nstage; i++) my *= p.ay.radix[i];
			if (mx != 2 * rx || my != 2 * ry || p.smem > optin) {
				printf("  FAIL: inconsistent plan\n");
				failures++;
			}
		}
	}
	printf("%d failure(s)\n", failures);
	return failures ? 1 : 0;
}
