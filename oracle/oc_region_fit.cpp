// oc_region_fit.cpp -- CPU oracle of RegionFit2D / RegionFit3D (reference src/oc_region_fit.cpp).  TEST INFRASTRUCTURE ONLY.
// Built on the main oracle: oc_oracle.cpp is compiled into this library, so the fit is its lsq_qr (the column-pivoted
// Householder QR of Eigen's colPivHouseholderQr) and the records are its StrainLayout, restated nowhere else.
// ref-faithful arithmetic as oracle/Makefile: no fast-math, no FMA contraction.
#include "oc_oracle.cpp"

// ----------------------------------------------------------------------------------------------
// RegionFit2D / RegionFit3D (reference src/oc_region_fit.cpp): setNeighbor(reliable) + prepare + compute(queue).  For each queue
// POI: the reliable POIs with float squared distance strictly below radius^2 (:104-115 / :281-292), else the k nearest
// (k = min(k_min, reliable POIs), ties to the lower reliable index; :116-126 / :293-303); every one counts, whatever its ZNCC.
// With at least k_min of them the plane fit [1, dx, dy(, dz)] (colPivHouseholderQr, here lsq_qr) writes u ux uy (uz) v .. and
// zncc = 0 (:131-167 / :308-352).  Reliable and queue POIs with a non-finite position are neither neighbours nor fitted.
template <class T, int MODE>
void run_region_fit(const float* reliable, long n_rel, float* queue, long n, float radius, int k_min, int threads) {
	typedef StrainLayout<MODE> L;
	constexpr int NF = L::NF, D = L::SD, C = D + 1;
	auto finite = [&](const float* p) { for (int d = 0; d < D; d++) if (!std::isfinite(p[d])) return false; return true; };
	// uniform grid over the finite reliable positions, as run_strain's
	double lo[3] = { 0, 0, 0 }, hi[3] = { 0, 0, 0 };
	long n_fin = 0;
	for (long i = 0; i < n_rel; i++)
		if (finite(reliable + i * NF)) {
			for (int d = 0; d < D; d++) {
				const double v = reliable[i * NF + d];
				lo[d] = n_fin ? std::min(lo[d], v) : v;
				hi[d] = n_fin ? std::max(hi[d], v) : v;
			}
			n_fin++;
		}
	double extent = 0;
	for (int d = 0; d < D; d++) extent = std::max(extent, hi[d] - lo[d]);
	const double abs_radius = std::fabs((double)radius);
	double cell = !std::isfinite(abs_radius) ? extent + 1.0 : abs_radius > 0 ? abs_radius * 1.001 : 1.0;
	while (true) {
		double total = 1;
		for (int d = 0; d < D; d++) total *= std::floor((hi[d] - lo[d]) / cell) + 1;
		if (total <= 4.0 * (double)n_rel + 1024.0) break;
		cell *= 2;
	}
	long nc[3] = { 1, 1, 1 };
	for (int d = 0; d < D; d++) nc[d] = (long)std::floor((hi[d] - lo[d]) / cell) + 1;
	// a query's cell may lie outside the grid (by one at most is enough: farther cells hold no neighbour)
	auto cell_of = [&](const float* p, long* c) {
		for (int d = 0; d < 3; d++) c[d] = d < D ? (long)std::max(-1.0, std::min((double)nc[d], std::floor(((double)p[d] - lo[d]) / cell))) : 0;
	};
	std::vector<long> start((size_t)(nc[0] * nc[1] * nc[2]) + 1, 0), order(n_fin);
	for (int pass = 0; pass < 2; pass++) {
		std::vector<long> fill(start.begin(), start.end() - 1);
		for (long i = 0; i < n_rel; i++) {
			if (!finite(reliable + i * NF)) continue;
			long c[3];
			cell_of(reliable + i * NF, c);
			const long ci = (c[2] * nc[1] + c[1]) * nc[0] + c[0];
			if (pass == 0) start[ci + 1]++;
			else order[fill[ci]++] = i;
		}
		if (pass == 0)
			for (size_t k = 1; k < start.size(); k++) start[k] += start[k - 1];
	}
	const float r2 = radius * radius;
#pragma omp parallel num_threads(threads)
	{
		std::vector<long> fit;
		std::vector<std::pair<float, long>> cand;
		std::vector<T> A, B;
#pragma omp for schedule(dynamic, 64)
		for (long i = 0; i < n; i++) {
			float* p = queue + i * NF;
			if (!finite(p)) continue;
			auto d2_of = [&](const float* q) { float d2 = 0.f; for (int d = 0; d < D; d++) { float df = p[d] - q[d]; d2 += df * df; } return d2; };
			long c[3];
			cell_of(p, c);
			fit.clear();
			for (long cz = std::max(0l, c[2] - 1); cz <= std::min(nc[2] - 1, c[2] + 1); cz++)
				for (long cy = std::max(0l, c[1] - 1); cy <= std::min(nc[1] - 1, c[1] + 1); cy++)
					for (long cx = std::max(0l, c[0] - 1); cx <= std::min(nc[0] - 1, c[0] + 1); cx++) {
						const long ci = (cz * nc[1] + cy) * nc[0] + cx;
						for (long s = start[ci]; s < start[ci + 1]; s++)
							if (d2_of(reliable + order[s] * NF) < r2) fit.push_back(order[s]);
					}
			if ((long)fit.size() < k_min) {
				fit.clear();
				cand.clear();
				for (long t = 0; t < n_fin; t++) cand.push_back(std::make_pair(d2_of(reliable + order[t] * NF), order[t]));
				const long k = std::min((long)k_min, (long)cand.size());
				std::partial_sort(cand.begin(), cand.begin() + k, cand.end());
				for (long t = 0; t < k; t++) fit.push_back(cand[t].second);
			}
			std::sort(fit.begin(), fit.end());
			const int m = (int)fit.size();
			if (m < k_min) continue;
			A.resize((size_t)m * C);
			B.resize((size_t)m * D);
			for (int t = 0; t < m; t++) {
				const float* q = reliable + fit[t] * NF;
				A[(size_t)t * C] = 1;
				for (int d = 0; d < D; d++) A[(size_t)t * C + 1 + d] = (T)(q[d] - p[d]);
				B[(size_t)t * D] = q[L::U];
				B[(size_t)t * D + 1] = q[L::V];
				if (D == 3) B[(size_t)t * D + 2] = q[L::W];
			}
			T x[D][C];
			lsq_qr<T, C, D>(A, B, m, x);
			const int field[3] = { L::U, L::V, L::W };
			for (int k = 0; k < D; k++)
				for (int j = 0; j < C; j++) p[field[k] + j] = (float)x[k][j];
			p[L::Z0] = 0.f;
		}
	}
}

extern "C" {

// RegionFit2D (dim 2, POI2D records) / RegionFit3D (dim 3, POI3D): setNeighbor(reliable) + compute(queue).  exact: the fit in
// float64, else in float as the reference's Eigen::MatrixXf.
int oco_region_fit(const float* reliable, long n_reliable, float* queue, long n, int dim, float radius, int min_neighbors, int threads, int exact) {
	if (dim != 2 && dim != 3) return -1;
	if (threads < 1) threads = 1;
	if (dim == 2) {
		if (exact) run_region_fit<double, 2>(reliable, n_reliable, queue, n, radius, min_neighbors, threads);
		else run_region_fit<float, 2>(reliable, n_reliable, queue, n, radius, min_neighbors, threads);
	} else {
		if (exact) run_region_fit<double, 3>(reliable, n_reliable, queue, n, radius, min_neighbors, threads);
		else run_region_fit<float, 3>(reliable, n_reliable, queue, n, radius, min_neighbors, threads);
	}
	return 0;
}

} // extern "C"
