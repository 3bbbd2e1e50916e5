// Host-side view of the Strain cell grid (ocb::strain_grid_plan in opencorr_b200/csrc/ocb_kernels.h): the cell edge, the cells
// per axis and the sentinel key the plan picks for a bounding box and a neighbour radius.  Built and run by
// tests/test_strain_grid_host.py (needs nvcc, no GPU), which feeds it the bbox and radius of every grid case of
// tests/strain_cases.py and checks the plan's rules on each.
//
//   strain_grid_host_test < cases     one line per case "name dims lo0 lo1 lo2 hi0 hi1 hi2 radius" (float32 values) read from
//                                     stdin; prints "name: cell=E nc=A,B,C cells=N top=X,Y,Z" per case, where top is the cell
//                                     index of the bbox maximum on each axis, computed as the kernels compute it
#include <cmath>
#include <cstdio>

#include "ocb_kernels.h"
using namespace ocb;

int main() {
	char name[128];
	int dims;
	float lo[3], hi[3], radius;
	while (scanf("%127s %d %f %f %f %f %f %f %f", name, &dims, &lo[0], &lo[1], &lo[2], &hi[0], &hi[1], &hi[2], &radius) == 9) {
		StrainGrid g;
		const double cell = strain_grid_plan(dims, lo, hi, radius, &g);
		int top[3] = { 0, 0, 0 };
		for (int d = 0; d < dims; d++) {
			const int v = (int)floorf((hi[d] - g.lo[d]) * g.inv_cell);
			top[d] = v < 0 ? 0 : (v >= g.nc[d] ? g.nc[d] - 1 : v);
		}
		printf("%s: cell=%.17g nc=%d,%d,%d cells=%u top=%d,%d,%d\n", name, cell, g.nc[0], g.nc[1], g.nc[2], g.n_cells, top[0], top[1], top[2]);
	}
	return 0;
}
