// Host-side view of the SIFT3D pyramid plan (ocb::sift3d_plan in opencorr_b200/csrc/ocb_kernels.h).  Built and run by
// tests/test_sift3d_plan_host.py (needs nvcc, no GPU), which checks the schedule against a restatement of the reference and the
// blur weights against the oracle's.
//
//   sift3d_plan_host_test < cases     one line per case "name nx ny nz ux uy uz c0 .. c9" (unit and the 10 config floats) read
//                                     from stdin.  A refused plan prints "name: reject R" (R: the Sift3dReject value); an
//                                     accepted one prints "name: plan N L KAPPA", then "name: octave o nx ny nz UX UY UZ" per
//                                     octave and "name: layer o l SCALE SIGMA r0 r1 r2 W..." per layer, W the weights
//                                     w[a][0..r_a] of the three axes in turn.  Capitals: float bits in hex.
#include <cstdio>
#include <cstring>

#include "ocb_kernels.h"
using namespace ocb;

static unsigned bits(float f) {
	unsigned u;
	memcpy(&u, &f, sizeof(u));
	return u;
}

int main() {
	char name[128];
	int n[3];
	float unit[3], cfg[s3::CFG_FIELDS];
	while (scanf("%127s %d %d %d %f %f %f", name, &n[0], &n[1], &n[2], &unit[0], &unit[1], &unit[2]) == 7) {
		for (int i = 0; i < s3::CFG_FIELDS; i++)
			if (scanf("%f", &cfg[i]) != 1) return 1;
		Sift3dPlan p;
		if (!sift3d_plan(n[0], n[1], n[2], cfg, unit, &p)) {
			printf("%s: reject %d\n", name, (int)p.reject);
			continue;
		}
		printf("%s: plan %d %d %08x\n", name, p.n_octave, p.L, bits(p.kappa));
		for (int o = 0; o < p.n_octave; o++) {
			const Sift3dOctave& v = p.octave[o];
			printf("%s: octave %d %d %d %d %08x %08x %08x\n", name, o, v.nx, v.ny, v.nz, bits(v.unit[0]), bits(v.unit[1]), bits(v.unit[2]));
			for (int l = 0; l < p.L; l++) {
				const Sift3dLayer& b = p.layer[(size_t)o * p.L + l];
				printf("%s: layer %d %d %08x %08x %d %d %d", name, o, l, bits(b.scale), bits(b.sigma), b.radius[0], b.radius[1],
					b.radius[2]);
				for (int a = 0; a < 3; a++)
					for (int r = 0; r <= b.radius[a]; r++) printf(" %08x", bits(b.w[a].w[r]));
				printf("\n");
			}
		}
	}
	return 0;
}
