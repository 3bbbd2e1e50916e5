// oc_stereo.cpp -- CPU oracle of the stereo-reconstruction module (TEST INFRASTRUCTURE ONLY, like oc_oracle.cpp).
//
// Restates, from the reference's published behaviour, Calibration::prepare / undistort (src/oc_calibration.cpp:117-264) and
// Stereovision::reconstruct (src/oc_stereovision.cpp:70-133), in two flavours selected per camera / per call:
//   faithful (exact = 0): float32 in the reference's operation order, compiled with -ffp-contract=off, and the 4x3 system solved
//                         by Householder QR with column pivoting in float32 (the algorithm of Eigen's colPivHouseholderQr, which
//                         the reference calls at :115; restated from Businger & Golub 1965 / LAPACK xGEQPF, not copied);
//   exact    (exact = 1): the same algorithm in float64 throughout (maps, lookup, system and solve), rounded to float on output.
// Built by stereo.py into liboc_stereo.so; plain C entry points, prefix ocs_.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <utility>
#include <vector>

#include <omp.h>

namespace {

template <class T>
struct Intr {
	T fx, fy, fs, cx, cy, k1, k2, k3, k4, k5, k6, p1, p2;
	explicit Intr(const float* v)
		: fx(v[0]), fy(v[1]), fs(v[2]), cx(v[3]), cy(v[4]), k1(v[5]), k2(v[6]), k3(v[7]), k4(v[8]), k5(v[9]), k6(v[10]), p1(v[11]), p2(v[12]) {}
};

// Calibration::image_to_sensor (:117-124)
template <class T>
inline void image_to_sensor(const Intr<T>& I, T x, T y, T& sx, T& sy) {
	sy = y * I.fy + I.cy;
	sx = x * I.fx + y * I.fs + I.cx;
}

// Calibration::sensor_to_image (:126-133)
template <class T>
inline void sensor_to_image(const Intr<T>& I, T x, T y, T& ix, T& iy) {
	iy = (y - I.cy) / I.fy;
	ix = (x - I.cx - I.fs * iy) / I.fx;
}

// Calibration::distort (:136-159)
template <class T>
inline void distort(const Intr<T>& I, T x, T y, T& dx, T& dy) {
	const T xx = x * x, yy = y * y, xy = x * y;
	const T r2 = xx + yy;
	const T r4 = r2 * r2;
	const T r6 = r2 * r4;
	const T radial = (1 + I.k1 * r2 + I.k2 * r4 + I.k3 * r6) / (1 + I.k4 * r2 + I.k5 * r4 + I.k6 * r6);
	dy = y * radial;
	dx = x * radial;
	dy += I.p1 * (r2 + 2 * yy) + 2 * I.p2 * xy;
	dx += 2 * I.p1 * xy + I.p2 * (r2 + 2 * xx);
}

// Calibration::prepare (:161-219), row-major maps
template <class T>
void build_map(const Intr<T>& I, int height, int width, T convergence, int iteration, T* map_x, T* map_y, int threads) {
#pragma omp parallel for num_threads(threads) schedule(static)
	for (int r = 0; r < height; r++) {
		for (int c = 0; c < width; c++) {
			T x0, y0;
			sensor_to_image(I, (T)c, (T)r, x0, y0);
			T ix = x0, iy = y0;
			bool stop = false;
			int i = 0;
			while (i < iteration && !stop) {
				i++;
				T dx, dy, sx, sy;
				distort(I, ix, iy, dx, dy);
				image_to_sensor(I, dx, dy, sx, sy);
				T dev_y = (T)r - sy;
				T dev_x = (T)c - sx;
				if (std::isinf(dev_x) || std::isinf(dev_y)) {
					stop = true;
					iy = y0;
					ix = x0;
				}
				if (std::fabs(dev_x) > convergence || std::fabs(dev_y) > convergence) {
					dev_y /= I.fy;
					iy += dev_y;
					ix += (dev_x - dev_y * I.fs) / I.fx;
				} else {
					stop = true;
				}
			}
			map_x[(size_t)r * width + c] = ix;
			map_y[(size_t)r * width + c] = iy;
		}
	}
}

struct Calib {
	int height, width, exact;
	std::vector<float> mx, my;   // faithful maps
	std::vector<double> dx, dy;  // exact maps
};

// Calibration::undistort (:221-264): clamps (x, y) in place, returns sensor coordinates
template <class T>
void undistort(const T* map_x, const T* map_y, int height, int width, const Intr<T>& I, T& x, T& y, T& ux, T& uy) {
	if (x < 0) x = 0;
	if (y < 0) y = 0;
	if (x > (T)(width - 2)) x = (T)(width - 2);
	if (y > (T)(height - 2)) y = (T)(height - 2);
	const int yi = (int)std::floor(y), xi = (int)std::floor(x);
	const T yd = y - (T)yi, xd = x - (T)xi;
	const size_t i00 = (size_t)yi * width + xi, i10 = i00 + width;
	const T cy = map_y[i00] * (1 - yd) * (1 - xd) + map_y[i10] * yd * (1 - xd) + map_y[i00 + 1] * (1 - yd) * xd + map_y[i10 + 1] * yd * xd;
	const T cx = map_x[i00] * (1 - yd) * (1 - xd) + map_x[i10] * yd * (1 - xd) + map_x[i00 + 1] * (1 - yd) * xd + map_x[i10 + 1] * yd * xd;
	image_to_sensor(I, cx, cy, ux, uy);
}

// Householder QR with column pivoting, then the least-squares solve (rank-revealing: components beyond the numerical rank are 0).
// A is m x n column-major (m = 4, n = 3 here), b has m entries.
template <class T>
void colpiv_qr_solve(T A[3][4], T b[4], T x[3]) {
	const int m = 4, n = 3;
	const T eps = std::numeric_limits<T>::epsilon();
	T norm_upd[3], norm_dir[3], hcoef[3];
	int perm[3] = { 0, 1, 2 };
	auto col_norm = [&](int j, int from) {
		T s = 0;
		for (int i = from; i < m; i++) s += A[j][i] * A[j][i];
		return std::sqrt(s);
	};
	for (int j = 0; j < n; j++) norm_dir[j] = norm_upd[j] = col_norm(j, 0);
	T maxnorm = 0;
	for (int j = 0; j < n; j++) maxnorm = std::max(maxnorm, norm_upd[j]);
	const T threshold_helper = (maxnorm * eps) * (maxnorm * eps) / (T)m;
	const T downdate_threshold = std::sqrt(eps);
	int rank = n;
	for (int k = 0; k < n; k++) {
		int big = k;
		for (int j = k + 1; j < n; j++)
			if (norm_upd[j] > norm_upd[big]) big = j;
		const T big_sq = norm_upd[big] * norm_upd[big];
		if (rank == n && big_sq < threshold_helper * (T)(m - k)) rank = k;
		if (big != k) {
			for (int i = 0; i < m; i++) std::swap(A[k][i], A[big][i]);
			std::swap(norm_upd[k], norm_upd[big]);
			std::swap(norm_dir[k], norm_dir[big]);
			std::swap(perm[k], perm[big]);
		}
		// Householder reflector H = I - tau v v^T, v = (1, essential), annihilating A[k][k+1..m)
		T tail = 0;
		for (int i = k + 1; i < m; i++) tail += A[k][i] * A[k][i];
		const T c0 = A[k][k];
		T beta, tau;
		if (tail <= std::numeric_limits<T>::min()) {
			tau = 0;
			beta = c0;
			for (int i = k + 1; i < m; i++) A[k][i] = 0;
		} else {
			beta = std::sqrt(c0 * c0 + tail);
			if (c0 >= 0) beta = -beta;
			for (int i = k + 1; i < m; i++) A[k][i] = A[k][i] / (c0 - beta);
			tau = (beta - c0) / beta;
		}
		hcoef[k] = tau;
		A[k][k] = beta;
		// apply H to the remaining columns
		if (tau != 0)
			for (int j = k + 1; j < n; j++) {
				T t = 0;
				for (int i = k + 1; i < m; i++) t += A[k][i] * A[j][i];
				t += A[j][k];
				A[j][k] -= tau * t;
				for (int i = k + 1; i < m; i++) A[j][i] -= tau * A[k][i] * t;
			}
		// downdate the remaining column norms (LAPACK Working Note 176)
		for (int j = k + 1; j < n; j++) {
			if (norm_upd[j] == 0) continue;
			T t = std::fabs(A[j][k]) / norm_upd[j];
			t = (1 + t) * (1 - t);
			if (t < 0) t = 0;
			const T ratio = norm_upd[j] / norm_dir[j];
			const T t2 = t * ratio * ratio;
			if (t2 <= downdate_threshold) {
				norm_dir[j] = col_norm(j, k + 1);
				norm_upd[j] = norm_dir[j];
			} else {
				norm_upd[j] *= std::sqrt(t);
			}
		}
	}
	// c = Q^T b over the first `rank` reflectors, then R c = x by back substitution (column-oriented)
	T c[4] = { b[0], b[1], b[2], b[3] };
	for (int k = 0; k < rank; k++) {
		if (hcoef[k] == 0) continue;
		T t = c[k];
		for (int i = k + 1; i < m; i++) t += A[k][i] * c[i];
		c[k] -= hcoef[k] * t;
		for (int i = k + 1; i < m; i++) c[i] -= hcoef[k] * A[k][i] * t;
	}
	for (int k = rank - 1; k >= 0; k--) {
		c[k] /= A[k][k];
		for (int i = 0; i < k; i++) c[i] -= c[k] * A[k][i];
	}
	for (int j = 0; j < n; j++) x[perm[j]] = j < rank ? c[j] : 0;
}

// Stereovision::reconstruct(Point2D&, Point2D&) for one pair; A_out / b_out (if given) receive the system (row-major 4x3, 4)
template <class T>
void reconstruct_one(const Calib* c1, const T* m1x, const T* m1y, const Intr<T>& I1, const float* P1f, const Calib* c2, const T* m2x, const T* m2y,
	const Intr<T>& I2, const float* P2f, float* p1, float* p2, float* out, float* A_out, float* b_out) {
	if (std::isnan(p1[0]) || std::isnan(p1[1]) || std::isnan(p2[0]) || std::isnan(p2[1])) {
		out[0] = out[1] = out[2] = 0.f;
		if (A_out) std::memset(A_out, 0, 12 * sizeof(float));
		if (b_out) std::memset(b_out, 0, 4 * sizeof(float));
		return;
	}
	T x1 = p1[0], y1 = p1[1], x2 = p2[0], y2 = p2[1];
	T u1, v1, u2, v2;
	undistort(m1x, m1y, c1->height, c1->width, I1, x1, y1, u1, v1);
	undistort(m2x, m2y, c2->height, c2->width, I2, x2, y2, u2, v2);
	p1[0] = (float)x1; p1[1] = (float)y1;
	p2[0] = (float)x2; p2[1] = (float)y2;
	T P[12], Q[12];
	for (int i = 0; i < 12; i++) { P[i] = P1f[i]; Q[i] = P2f[i]; }
	T A[3][4], b[4]; // column-major
	for (int j = 0; j < 3; j++) {
		A[j][0] = u1 * P[8 + j] - P[j];
		A[j][1] = v1 * P[8 + j] - P[4 + j];
		A[j][2] = u2 * Q[8 + j] - Q[j];
		A[j][3] = v2 * Q[8 + j] - Q[4 + j];
	}
	b[0] = P[3] - u1 * P[11];
	b[1] = P[7] - v1 * P[11];
	b[2] = Q[3] - u2 * Q[11];
	b[3] = Q[7] - v2 * Q[11];
	if (A_out)
		for (int i = 0; i < 4; i++)
			for (int j = 0; j < 3; j++) A_out[3 * i + j] = (float)A[j][i];
	if (b_out)
		for (int i = 0; i < 4; i++) b_out[i] = (float)b[i];
	T x[3];
	colpiv_qr_solve(A, b, x);
	out[0] = (float)x[0];
	out[1] = (float)x[1];
	out[2] = (float)x[2];
}

} // namespace

extern "C" {

void* ocs_calib_create(const float* intrinsics, int height, int width, float convergence, int iteration, int threads, int exact) {
	if (height < 2 || width < 2) return nullptr;
	Calib* c = new Calib;
	c->height = height;
	c->width = width;
	c->exact = exact;
	const size_t n = (size_t)height * width;
	if (exact) {
		c->dx.resize(n);
		c->dy.resize(n);
		build_map(Intr<double>(intrinsics), height, width, (double)convergence, iteration, c->dx.data(), c->dy.data(), threads);
	} else {
		c->mx.resize(n);
		c->my.resize(n);
		build_map(Intr<float>(intrinsics), height, width, convergence, iteration, c->mx.data(), c->my.data(), threads);
	}
	return c;
}

void ocs_calib_destroy(void* h) { delete (Calib*)h; }

// float32 copies of the maps (the exact flavour's are rounded)
void ocs_calib_get_map(void* h, float* map_x, float* map_y) {
	const Calib* c = (const Calib*)h;
	const size_t n = (size_t)c->height * c->width;
	for (size_t i = 0; i < n; i++) {
		map_x[i] = c->exact ? (float)c->dx[i] : c->mx[i];
		map_y[i] = c->exact ? (float)c->dy[i] : c->my[i];
	}
}

// Calibration::undistort for n points (n x 2): pts clamped in place, out = sensor coordinates; NaN points are left alone and give NaN
void ocs_undistort(void* h, const float* intrinsics, float* pts, float* out, long n, int threads) {
	const Calib* c = (const Calib*)h;
#pragma omp parallel for num_threads(threads) schedule(static)
	for (long i = 0; i < n; i++) {
		float* p = pts + 2 * i;
		if (std::isnan(p[0]) || std::isnan(p[1])) {
			out[2 * i] = out[2 * i + 1] = NAN;
			continue;
		}
		if (c->exact) {
			double x = p[0], y = p[1], ux, uy;
			undistort(c->dx.data(), c->dy.data(), c->height, c->width, Intr<double>(intrinsics), x, y, ux, uy);
			p[0] = (float)x; p[1] = (float)y;
			out[2 * i] = (float)ux; out[2 * i + 1] = (float)uy;
		} else {
			float x = p[0], y = p[1], ux, uy;
			undistort(c->mx.data(), c->my.data(), c->height, c->width, Intr<float>(intrinsics), x, y, ux, uy);
			p[0] = x; p[1] = y;
			out[2 * i] = ux; out[2 * i + 1] = uy;
		}
	}
}

// Stereovision::reconstruct(queue, queue, queue).  Both cameras must be of the same flavour.  A / b: NULL or n x 12 / n x 4 floats
// receiving each pair's system (all zero for a NaN pair).  Returns 0, or -1 when the flavours differ.
int ocs_reconstruct(void* h1, const float* intrinsics1, const float* projection1, void* h2, const float* intrinsics2, const float* projection2,
	float* pts1, float* pts2, float* pts3d, float* A, float* b, long n, int threads) {
	const Calib* c1 = (const Calib*)h1;
	const Calib* c2 = (const Calib*)h2;
	if (c1->exact != c2->exact) return -1;
#pragma omp parallel for num_threads(threads) schedule(static)
	for (long i = 0; i < n; i++) {
		float* Ai = A ? A + 12 * i : nullptr;
		float* bi = b ? b + 4 * i : nullptr;
		if (c1->exact)
			reconstruct_one(c1, c1->dx.data(), c1->dy.data(), Intr<double>(intrinsics1), projection1, c2, c2->dx.data(), c2->dy.data(),
				Intr<double>(intrinsics2), projection2, pts1 + 2 * i, pts2 + 2 * i, pts3d + 3 * i, Ai, bi);
		else
			reconstruct_one(c1, c1->mx.data(), c1->my.data(), Intr<float>(intrinsics1), projection1, c2, c2->mx.data(), c2->my.data(),
				Intr<float>(intrinsics2), projection2, pts1 + 2 * i, pts2 + 2 * i, pts3d + 3 * i, Ai, bi);
	}
	return 0;
}

int ocs_max_threads() { return omp_get_max_threads(); }

} // extern "C"
