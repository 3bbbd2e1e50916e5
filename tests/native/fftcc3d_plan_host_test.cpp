// Host-side view of the FFTCC3D routing (ocb::fftcc3d_plan in opencorr_b200/csrc/ocb_kernels.h): which of the three kernels a
// window takes, the slices per round of the register kernel, the Stockham factorisation of each axis, the shared memory, the CTAs
// and the scratch per CTA.  Built and run by tests/test_fftcc3d_plan_host.py (needs nvcc, no GPU), which feeds it every case of
// tests/test_gpu_fftcc3d_geometry.py and checks that each lands where that file says, so that a change of the routing cannot
// silently turn a case into a copy of another.
//
//   fftcc3d_plan_host_test OPTIN SMS < cases     one line per case "rx ry rz force_generic n" read from stdin, for a device with
//                                                OPTIN bytes of opt-in shared memory per block and SMS multiprocessors
//   fftcc3d_plan_host_test limits OPTIN          the largest cubic radius the GENERIC kernel accepts with OPTIN bytes, and the
//                                                first radius above it that is refused for its shared memory
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

int axis_product(const FftAxis& a) {
	int m = 1;
	for (int i = 0; i < a.nstage; i++) m *= a.radix[i];
	return m;
}

const char* reason(Fftcc3dReject r) { return r == Fftcc3dReject::PRIME_FACTOR ? "prime factor" : "shared memory"; }

int limits(size_t optin) {
	int largest = 0, first_smem = 0;
	Fftcc3dPlan p;
	for (int r = 1; r <= 256 && !first_smem; r++) {
		if (fftcc3d_plan(r, r, r, true, optin, 1, &p)) largest = r;
		else if (p.reject == Fftcc3dReject::SHARED_MEMORY) first_smem = r;
	}
	printf("largest generic: %d\nfirst refused for shared memory: %d\n", largest, first_smem);
	return 0;
}

} // namespace

int main(int argc, char** argv) {
	if (argc == 3 && strcmp(argv[1], "limits") == 0) return limits((size_t)atol(argv[2]));
	if (argc != 3) return 2;
	const size_t optin = (size_t)atol(argv[1]);
	const int sms = atoi(argv[2]);
	int rx, ry, rz, force;
	long n;
	int failures = 0;
	while (scanf("%d %d %d %d %ld", &rx, &ry, &rz, &force, &n) == 5) {
		Fftcc3dPlan p;
		printf("r=(%d,%d,%d) force=%d n=%ld: ", rx, ry, rz, force, n);
		if (!fftcc3d_plan(rx, ry, rz, force != 0, optin, sms, &p)) {
			printf("rejected (%s), %zu B smem\n", reason(p.reject), p.smem);
			continue;
		}
		const long grid = n < p.ctas ? n : p.ctas;
		const long rounds = (n + p.ctas - 1) / p.ctas; // POIs the busiest CTA takes
		bool ok = p.smem <= optin && p.ctas >= sms;
		if (p.path == Fftcc3dPath::W32) {
			printf("kernel W32,");
			ok = ok && p.cta_scratch == (size_t)32 * 32 * 32;
		} else if (p.path == Fftcc3dPath::REG) {
			printf("kernel REG, N=%d G=%d, %d idle thread(s),", p.n, p.slices_per_round, p.idle_threads);
			ok = ok && p.n == 2 * rx && p.slices_per_round * p.n + p.idle_threads == F3R_THREADS && p.idle_threads < p.n
				&& p.cta_scratch == (size_t)2 * p.n * p.n * p.n;
		} else {
			printf("kernel GENERIC, M=%ld,", 8L * rx * ry * rz);
			print_axis("x", p.ax);
			print_axis("y", p.ay);
			print_axis("z", p.az);
			printf(",");
			// the stages multiply back to the axis lengths
			ok = ok && axis_product(p.ax) == 2 * rx && axis_product(p.ay) == 2 * ry && axis_product(p.az) == 2 * rz
				&& p.cta_scratch == (size_t)8 * rx * ry * rz;
		}
		printf(" %zu B smem, %d CTA(s) of which %ld launched, %ld POI(s) per CTA at most, %zu B scratch per CTA\n", p.smem, p.ctas, grid,
			rounds, p.cta_scratch * 8);
		if (!ok) {
			printf("  FAIL: inconsistent plan\n");
			failures++;
		}
	}
	printf("%d failure(s)\n", failures);
	return failures ? 1 : 0;
}
