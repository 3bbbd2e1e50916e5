// oc_oracle.cpp -- CPU ORACLE for the FFT-CC -> IC-GN hot path of vincentjzy/OpenCorr.
//
// THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load it.  The product path
// (opencorr_b200/csrc + include/opencorr_b200.h) never links or calls anything in oracle/.
//
// It is a dependency-free restatement (no Eigen / FFTW / OpenCV) of the reference algorithms,
// written from the reference's behaviour, each function citing the reference file:line it follows
// (paths relative to /root/reference).  Third-party arithmetic that the reference delegates is
// restated from the published algorithm:
//   * FFTW 3.3.5 (1_Get_started.md:11) r2c/c2r transforms, call sites src/oc_fftcc.cpp:40-42,
//     233-243, 378-388  ->  own mixed-radix Stockham FFT (unnormalised, like FFTW).
//   * Eigen 3.4.0 (1_Get_started.md:9) Matrix::inverse() (src/oc_icgn.cpp:210,290,759,831,1339,1439)
//     -> partial-pivot LU inverse for 6x6/12x12, cofactor inverse for 3x3/4x4 (what Eigen does).
// Parity pin: tests/test_oracle_golden.py checks this oracle against the reference's committed
// result tables examples/2d_dic/oht_cfrp_4_fftcc_icgn1_r16*.csv and
// examples/dvc/al_foam4_1_fftcc_icgn1*_r30.csv (fixtures under tests/golden/).
//
// Two flavours, selected per call by `exact`:
//   exact=0  "ref-faithful": float32 everywhere, the reference's loop/summation order
//            (compile with -ffp-contract=off, no -ffast-math).
//   exact=1  "exact": identical algorithm with every intermediate in float64 (inputs stay f32).
//
// Memory layouts at this C boundary: images row-major float [H][W]; volumes [z][y][x];
// POI records are the reference's own structs viewed as float arrays (src/oc_poi.h:102-136,
// 187-222): POI2D = 25 floats {x,y | p[12] | u0,v0,zncc,iteration,convergence,feature |
// exx,eyy,exy | subset_rx,subset_ry}; POI3D = 31 floats {x,y,z | p[12] | u0,v0,w0,zncc,
// iteration,convergence,feature | e[6] | subset_rx,ry,rz}.

#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <utility>
#include <vector>
#include <omp.h>

namespace {

// ----------------------------------------------------------------------------------------------
// POI record field offsets (src/oc_poi.h:25-33,44-51,102-136 and :62-71,93-99,187-222)
// ----------------------------------------------------------------------------------------------
enum { P2_X = 0, P2_Y = 1, P2_DEF = 2, P2_U0 = 14, P2_V0 = 15, P2_ZNCC = 16, P2_ITER = 17, P2_CONV = 18,
       P2_FEAT = 19, P2_STRAIN = 20, P2_RX = 23, P2_RY = 24, P2_N = 25 };
// 2D deformation order: u ux uy uxx uxy uyy v vx vy vxx vxy vyy
enum { D2_U = 0, D2_UX = 1, D2_UY = 2, D2_UXX = 3, D2_UXY = 4, D2_UYY = 5, D2_V = 6, D2_VX = 7, D2_VY = 8,
       D2_VXX = 9, D2_VXY = 10, D2_VYY = 11 };
enum { P3_X = 0, P3_Y = 1, P3_Z = 2, P3_DEF = 3, P3_U0 = 15, P3_V0 = 16, P3_W0 = 17, P3_ZNCC = 18,
       P3_ITER = 19, P3_CONV = 20, P3_FEAT = 21, P3_STRAIN = 22, P3_RX = 28, P3_RY = 29, P3_RZ = 30, P3_N = 31 };
// 3D deformation order: u ux uy uz v vx vy vz w wx wy wz

// ----------------------------------------------------------------------------------------------
// Mixed-radix Stockham FFT (unnormalised both ways, like FFTW).  Transforms `n` points with
// stride `s0` for all q in [0,s0) at once, so one call does a whole axis of a row-major array.
// ----------------------------------------------------------------------------------------------
template <class T>
struct FFT {
	typedef std::complex<T> cpx;
	int n = 0;
	std::vector<int> radices;
	std::vector<cpx> tw_fwd, tw_inv; // W_n^k, k in [0,n)

	void plan(int n_) {
		n = n_;
		radices.clear();
		int m = n;
		while (m % 4 == 0) { radices.push_back(4); m /= 4; }
		while (m % 2 == 0) { radices.push_back(2); m /= 2; }
		while (m % 3 == 0) { radices.push_back(3); m /= 3; }
		while (m % 5 == 0) { radices.push_back(5); m /= 5; }
		for (int p = 7; m > 1; p += 2) {
			while (m % p == 0) { radices.push_back(p); m /= p; }
		}
		tw_fwd.resize(n);
		tw_inv.resize(n);
		for (int k = 0; k < n; k++) {
			double a = -2.0 * M_PI * (double)k / (double)n;
			tw_fwd[k] = cpx((T)std::cos(a), (T)std::sin(a));
			tw_inv[k] = cpx((T)std::cos(a), (T)-std::sin(a));
		}
	}

	// x: input/output (result ends in x), y: scratch, both of n*s0 elements.
	void run(cpx* x, cpx* y, long s0, bool inverse) const {
		const cpx* tw = inverse ? tw_inv.data() : tw_fwd.data();
		int ncur = n;
		long s = s0;
		cpx* in = x;
		cpx* out = y;
		cpx a[128], b[128]; // radix (largest prime factor) must be <= 128
		for (size_t st = 0; st < radices.size(); st++) {
			int r = radices[st];
			int m = ncur / r;
			int tstep = n / ncur; // W_ncur^k = W_n^(k*tstep)
			int rstep = n / r;    // W_r^k    = W_n^(k*rstep)
			for (int p = 0; p < m; p++) {
				for (long q = 0; q < s; q++) {
					for (int k = 0; k < r; k++) a[k] = in[q + s * (p + (long)k * m)];
					if (r == 2) {
						b[0] = a[0] + a[1];
						b[1] = a[0] - a[1];
					} else if (r == 4) {
						cpx t0 = a[0] + a[2], t1 = a[0] - a[2], t2 = a[1] + a[3], t3 = a[1] - a[3];
						// multiply t3 by -i (forward) or +i (inverse)
						cpx t3r = inverse ? cpx(-t3.imag(), t3.real()) : cpx(t3.imag(), -t3.real());
						b[0] = t0 + t2;
						b[1] = t1 + t3r;
						b[2] = t0 - t2;
						b[3] = t1 - t3r;
					} else {
						for (int j = 0; j < r; j++) {
							cpx acc = a[0];
							for (int k = 1; k < r; k++) acc += a[k] * tw[((long)j * k % r) * rstep];
							b[j] = acc;
						}
					}
					out[q + s * ((long)r * p)] = b[0];
					for (int j = 1; j < r; j++) out[q + s * ((long)r * p + j)] = b[j] * tw[(long)p * j * tstep]; // p*j*tstep < n
				}
			}
			ncur = m;
			s *= r;
			std::swap(in, out);
		}
		if (in != x) std::memcpy(x, in, sizeof(cpx) * (size_t)n * (size_t)s0);
	}
};

// FFT of every row of a row-major [rows][n] block (the contiguous axis): transpose, run the strided
// transform (long contiguous inner loops), transpose back.  tmp: rows*n elements.
template <class T>
void fft_rows(const FFT<T>& f, std::complex<T>* x, std::complex<T>* tmp, std::complex<T>* scratch, int rows, bool inverse) {
	const int n = f.n;
	for (int r = 0; r < rows; r++)
		for (int c = 0; c < n; c++) tmp[(size_t)c * rows + r] = x[(size_t)r * n + c];
	f.run(tmp, scratch, rows, inverse);
	for (int r = 0; r < rows; r++)
		for (int c = 0; c < n; c++) x[(size_t)r * n + c] = tmp[(size_t)c * rows + r];
}

// ----------------------------------------------------------------------------------------------
// Small dense linear algebra standing in for Eigen (see header).
// ----------------------------------------------------------------------------------------------
// General inverse via LU with partial pivoting (Eigen PartialPivLU::inverse for N>4).
template <class T, int N>
void inverse_lu(const T* A, T* inv) {
	T lu[N * N];
	int perm[N];
	for (int i = 0; i < N * N; i++) lu[i] = A[i];
	for (int i = 0; i < N; i++) perm[i] = i;
	for (int k = 0; k < N; k++) {
		int piv = k;
		T best = std::fabs(lu[k * N + k]);
		for (int i = k + 1; i < N; i++) {
			T v = std::fabs(lu[i * N + k]);
			if (v > best) { best = v; piv = i; }
		}
		if (piv != k) {
			for (int j = 0; j < N; j++) std::swap(lu[k * N + j], lu[piv * N + j]);
			std::swap(perm[k], perm[piv]);
		}
		T d = lu[k * N + k];
		for (int i = k + 1; i < N; i++) {
			lu[i * N + k] /= d;
			T l = lu[i * N + k];
			for (int j = k + 1; j < N; j++) lu[i * N + j] -= l * lu[k * N + j];
		}
	}
	for (int c = 0; c < N; c++) {
		T y[N];
		for (int i = 0; i < N; i++) {
			T v = (perm[i] == c) ? (T)1 : (T)0;
			for (int j = 0; j < i; j++) v -= lu[i * N + j] * y[j];
			y[i] = v;
		}
		for (int i = N - 1; i >= 0; i--) {
			T v = y[i];
			for (int j = i + 1; j < N; j++) v -= lu[i * N + j] * inv[j * N + c];
			inv[i * N + c] = v / lu[i * N + i];
		}
	}
}

// 3x3 inverse by cofactors (Eigen's fixed-size 3x3 path).
template <class T>
void inverse3(const T* m, T* o) {
	T c00 = m[4] * m[8] - m[5] * m[7];
	T c01 = m[5] * m[6] - m[3] * m[8];
	T c02 = m[3] * m[7] - m[4] * m[6];
	T det = m[0] * c00 + m[1] * c01 + m[2] * c02;
	T id = (T)1 / det;
	o[0] = c00 * id;
	o[1] = (m[2] * m[7] - m[1] * m[8]) * id;
	o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
	o[3] = c01 * id;
	o[4] = (m[0] * m[8] - m[2] * m[6]) * id;
	o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
	o[6] = c02 * id;
	o[7] = (m[1] * m[6] - m[0] * m[7]) * id;
	o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

// 4x4 inverse by cofactors (Eigen's fixed-size 4x4 path is cofactor based).
template <class T>
void inverse4(const T* m, T* inv) {
	T t[16];
	t[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
	t[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
	t[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
	t[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
	t[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
	t[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
	t[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
	t[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
	t[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
	t[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
	t[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
	t[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
	t[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
	t[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
	t[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
	t[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
	T det = m[0] * t[0] + m[1] * t[4] + m[2] * t[8] + m[3] * t[12];
	T id = (T)1 / det;
	for (int i = 0; i < 16; i++) inv[i] = t[i] * id;
}

template <class T, int N>
void matmul(const T* A, const T* B, T* C) {
	for (int i = 0; i < N; i++)
		for (int j = 0; j < N; j++) {
			T acc = 0;
			for (int k = 0; k < N; k++) acc += A[i * N + k] * B[k * N + j];
			C[i * N + j] = acc;
		}
}

template <class T>
inline bool is_nan(T v) { return v != v; }

// ----------------------------------------------------------------------------------------------
// 2D context: images + what ICGN2D1::prepare() builds (src/oc_icgn.cpp:115-142).
// ----------------------------------------------------------------------------------------------
struct Ctx2D {
	int h = 0, w = 0, threads = 1;
	std::vector<float> ref, tar;  // [h][w]
	std::vector<float> gx, gy;    // Gradient2D4 of ref
	std::vector<float> lut;       // BicubicBspline coefficient[h][w][4][4] of tar
	bool prepared = false;
	// what NR2D1::prepare() builds (src/oc_nr.cpp:119-156): gradients of TAR and the LUTs of both gradient maps
	std::vector<float> tgx, tgy, lut_tgx, lut_tgy;
	bool prepared_nr = false;
};

// Gradient2D4::getGradientX/Y, src/oc_gradient.cpp:37-79.  Borders (2 px) stay zero.
void gradient2d(const Ctx2D& c, const std::vector<float>& src, std::vector<float>& gx, std::vector<float>& gy) {
	const float first_factor = 1.f / 12.f, second_factor = 2.f / 3.f; // oc_gradient.cpp:21-22
	int h = c.h, w = c.w;
	gx.assign((size_t)h * w, 0.f);
	gy.assign((size_t)h * w, 0.f);
	const float* f = src.data();
#pragma omp parallel for num_threads(c.threads)
	for (int r = 0; r < h; r++) {
		for (int col = 2; col < w - 2; col++) {
			float result = 0.0f;
			result -= f[(size_t)r * w + col + 2] * first_factor;
			result += f[(size_t)r * w + col + 1] * second_factor;
			result -= f[(size_t)r * w + col - 1] * second_factor;
			result += f[(size_t)r * w + col - 2] * first_factor;
			gx[(size_t)r * w + col] = result;
		}
	}
#pragma omp parallel for num_threads(c.threads)
	for (int r = 2; r < h - 2; r++) {
		for (int col = 0; col < w; col++) {
			float result = 0.0f;
			result -= f[(size_t)(r + 2) * w + col] * first_factor;
			result += f[(size_t)(r + 1) * w + col] * second_factor;
			result -= f[(size_t)(r - 1) * w + col] * second_factor;
			result += f[(size_t)(r - 2) * w + col] * first_factor;
			gy[(size_t)r * w + col] = result;
		}
	}
}

// BC = B*C, src/oc_cubic_bspline.h:52-58
const float BC_MATRIX[4][4] = {
	{ -144.0f / 336.0f, 384.0f / 336.0f, -384.0f / 336.0f, 144.0f / 336.0f },
	{ 342.0f / 336.0f, -702.0f / 336.0f, 450.0f / 336.0f, -90.0f / 336.0f },
	{ -198.0f / 336.0f, -18.0f / 336.0f, 270.0f / 336.0f, -54.0f / 336.0f },
	{ 0.0f, 1.0f, 0.0f, 0.0f } };

// BicubicBspline::prepare, src/oc_cubic_bspline.cpp:84-132: 16 floats per pixel LUT.
void bicubic_prepare(const Ctx2D& c, const std::vector<float>& src, std::vector<float>& lut) {
	int h = c.h, w = c.w;
	lut.assign((size_t)h * w * 16, 0.f);
	const float* img = src.data();
#pragma omp parallel for num_threads(c.threads)
	for (int r = 1; r < h - 2; r++) {
		for (int col = 1; col < w - 2; col++) {
			float q[4][4];
			for (int i = 0; i < 4; i++)
				for (int j = 0; j < 4; j++) q[i][j] = img[(size_t)(r - 1 + i) * w + (col - 1 + j)];
			float p[4][4];
			for (int k = 0; k < 4; k++)
				for (int l = 0; l < 4; l++) {
					float acc = 0.f;
					for (int m = 0; m < 4; m++)
						for (int n = 0; n < 4; n++) acc += BC_MATRIX[l][m] * BC_MATRIX[k][n] * q[n][m];
					p[k][l] = acc;
				}
			float* dst = &lut[((size_t)r * w + col) * 16];
			for (int k = 0; k < 4; k++)
				for (int l = 0; l < 4; l++) dst[k * 4 + l] = p[3 - k][3 - l];
		}
	}
}

// BicubicBspline::compute, src/oc_cubic_bspline.cpp:134-181.
template <class T>
inline T bicubic_eval(const Ctx2D& c, const std::vector<float>& lut, T x, T y) {
	if (x < 1 || y < 1 || x >= c.w - 2 || y >= c.h - 2 || is_nan(x) || is_nan(y)) return (T)-1;
	int xi = (int)std::floor(x), yi = (int)std::floor(y);
	T xd = x - xi, yd = y - yi;
	T x2 = xd * xd, y2 = yd * yd, x3 = x2 * xd, y3 = y2 * yd;
	const float* k = &lut[((size_t)yi * c.w + xi) * 16];
	T value = (T)k[0] + (T)k[1] * xd + (T)k[2] * x2 + (T)k[3] * x3
		+ (T)k[4] * yd + (T)k[5] * yd * xd + (T)k[6] * yd * x2 + (T)k[7] * yd * x3
		+ (T)k[8] * y2 + (T)k[9] * y2 * xd + (T)k[10] * y2 * x2 + (T)k[11] * y2 * x3
		+ (T)k[12] * y3 + (T)k[13] * y3 * xd + (T)k[14] * y3 * x2 + (T)k[15] * y3 * x3;
	return value;
}
template <class T>
inline T bicubic_eval(const Ctx2D& c, T x, T y) { return bicubic_eval<T>(c, c.lut, x, y); }

// FFTCC2D::compute(POI2D*), src/oc_fftcc.cpp:177-275.
// per-thread scratch of the FFT-CC stage (the reference's FFTW instance pool, src/oc_fftcc.cpp:141-163)
template <class T>
struct FftScratch {
	std::vector<T> a, b;
	std::vector<std::complex<T>> buf, cc, scratch, tmp;
	void resize(size_t n) { a.resize(n); b.resize(n); buf.resize(n); cc.resize(n); scratch.resize(n); }
};

template <class T>
void fftcc2d_poi(const Ctx2D& c, float* poi, int rx, int ry, const FFT<T>& fx, const FFT<T>& fy, FftScratch<T>& fs) {
	typedef std::complex<T> cpx;
	int sw = 2 * rx, sh = 2 * ry, size = sw * sh;
	float px = poi[P2_X], py = poi[P2_Y];
	float u0 = poi[P2_DEF + D2_U], v0 = poi[P2_DEF + D2_V];
	// border guard, :190-196 -- returns leaving the POI untouched
	if ((int)px < rx || (int)px >= c.w - rx || (int)py < ry || (int)py >= c.h - ry
		|| int(px + u0) < rx || int(px + u0) >= c.w - rx || int(py + v0) < ry || int(py + v0) >= c.h - ry)
		return;
	fs.resize(size);
	std::vector<T>& a = fs.a;
	std::vector<T>& b = fs.b;
	cpx* buf = fs.buf.data();
	cpx* scratch = fs.scratch.data();
	std::vector<cpx>& cc = fs.cc;
	T ref_mean = 0, tar_mean = 0, ref_norm = 0, tar_norm = 0;
	for (int r = 0; r < sh; r++) {
		for (int col = 0; col < sw; col++) {
			float rpx = px + col - rx, rpy = py + r - ry; // Point2D arithmetic is float, :209
			float value = c.ref[(size_t)(int)rpy * c.w + (int)rpx];
			a[r * sw + col] = value;
			ref_mean += value;
			float tpx = rpx + u0, tpy = rpy + v0; // :215
			value = c.tar[(size_t)(int)tpy * c.w + (int)tpx];
			b[r * sw + col] = value;
			tar_mean += value;
		}
	}
	ref_mean /= size;
	tar_mean /= size;
	for (int i = 0; i < size; i++) {
		a[i] -= ref_mean;
		b[i] -= tar_mean;
		ref_norm += a[i] * a[i];
		tar_norm += b[i] * b[i];
	}
	// Z = FFT2(a + i b); A = (Z(k)+conj Z(-k))/2, B = (Z(k)-conj Z(-k))/(2i); C = conj(A) B  (:233-241)
	for (int i = 0; i < size; i++) buf[i] = cpx(a[i], b[i]);
	fft_rows(fx, buf, cc.data(), scratch, sh, false);
	fy.run(buf, scratch, sw, false);
	for (int ky = 0; ky < sh; ky++)
		for (int kx = 0; kx < sw; kx++) {
			cpx z = buf[ky * sw + kx];
			cpx zm = std::conj(buf[((sh - ky) % sh) * sw + ((sw - kx) % sw)]);
			cpx A = (z + zm) * (T)0.5;
			cpx d = (z - zm) * (T)0.5;
			cpx B = cpx(d.imag(), -d.real());
			// (:239-240) re = ArBr + AiBi ; im = ArBi - AiBr
			cc[ky * sw + kx] = cpx(A.real() * B.real() + A.imag() * B.imag(), A.real() * B.imag() - A.imag() * B.real());
		}
	fft_rows(fx, cc.data(), buf, scratch, sh, true);
	fy.run(cc.data(), scratch, sw, true);
	// A window of constant grey is zero after the mean is taken off, and the reference, which transforms the two windows
	// separately (:233-243), then gets a surface that is zero everywhere: index 0 wins and ZNCC is 0 / 0.  The packed transform
	// above only gives Z(k) + conj Z(-k) = 0 up to rounding.
	if (ref_norm == 0 || tar_norm == 0)
		for (int i = 0; i < size; i++) cc[i] = cpx(0, 0);
	// argmax, :246-255
	T max_zncc = (T)-2;
	int idx = 0;
	for (int i = 0; i < size; i++) {
		if (cc[i].real() > max_zncc) { max_zncc = cc[i].real(); idx = i; }
	}
	int du = idx % sw, dv = idx / sw;
	if (du > rx) du -= sw;
	if (dv > ry) dv -= sh;
	poi[P2_DEF + D2_U] = (float)du + u0;
	poi[P2_DEF + D2_V] = (float)dv + v0;
	poi[P2_U0] = u0;
	poi[P2_V0] = v0;
	poi[P2_ZNCC] = (float)(max_zncc / (std::sqrt(ref_norm * tar_norm) * size));
}

// Shape-function plumbing, src/oc_deformation.cpp.
template <class T>
inline void warp2d1_set(const T* p /*u ux uy v vx vy*/, T* W) { // :117-128
	W[0] = (T)1 + p[1]; W[1] = p[2]; W[2] = p[0];
	W[3] = p[4]; W[4] = (T)1 + p[5]; W[5] = p[3];
	W[6] = 0; W[7] = 0; W[8] = 1;
}
template <class T>
inline void warp2d1_get(const T* W, T* p) { // :107-115
	p[0] = W[2]; p[1] = W[0] - (T)1; p[2] = W[1];
	p[3] = W[5]; p[4] = W[3]; p[5] = W[4] - (T)1;
}
template <class T>
inline void warp2d2_set(const T* p /*u ux uy uxx uxy uyy v vx vy vxx vxy vyy*/, T* W) { // :301-350
	T u = p[0], ux = p[1], uy = p[2], uxx = p[3], uxy = p[4], uyy = p[5];
	T v = p[6], vx = p[7], vy = p[8], vxx = p[9], vxy = p[10], vyy = p[11];
	T two = 2, one = 1, half = (T)0.5;
	W[0] = one + two * ux + ux * ux + u * uxx;
	W[1] = two * u * uxy + two * (one + ux) * uy;
	W[2] = uy * uy + u * uyy;
	W[3] = two * u * (1 + ux);
	W[4] = two * u * uy;
	W[5] = u * u;
	W[6] = half * (v * uxx + two * (one + ux) * vx + u * vxx);
	W[7] = one + uy * vx + ux * vy + v * uxy + u * vxy + vy + ux;
	W[8] = half * (v * uyy + two * uy * (one + vy) + u * vyy);
	W[9] = v + v * ux + u * vx;
	W[10] = u + v * uy + u * vy;
	W[11] = u * v;
	W[12] = vx * vx + v * vxx;
	W[13] = two * v * vxy + two * vx * (one + vy);
	W[14] = one + two * vy + vy * vy + v * vyy;
	W[15] = two * v * vx;
	W[16] = two * v * (one + vy);
	W[17] = v * v;
	W[18] = half * uxx; W[19] = uxy; W[20] = half * uyy; W[21] = one + ux; W[22] = uy; W[23] = u;
	W[24] = half * vxx; W[25] = vxy; W[26] = half * vyy; W[27] = vx; W[28] = one + vy; W[29] = v;
	W[30] = 0; W[31] = 0; W[32] = 0; W[33] = 0; W[34] = 0; W[35] = 1;
}
template <class T>
inline void warp2d2_get(const T* W, T* p) { // :284-299
	p[0] = W[23]; p[1] = W[21] - (T)1; p[2] = W[22]; p[3] = W[18] * (T)2; p[4] = W[19]; p[5] = W[20] * (T)2;
	p[6] = W[29]; p[7] = W[27]; p[8] = W[28] - (T)1; p[9] = W[24] * (T)2; p[10] = W[25]; p[11] = W[26] * (T)2;
}
template <class T>
inline void warp3d1_set(const T* p /*u ux uy uz v vx vy vz w wx wy wz*/, T* W) { // :495-516
	W[0] = (T)1 + p[1]; W[1] = p[2]; W[2] = p[3]; W[3] = p[0];
	W[4] = p[5]; W[5] = (T)1 + p[6]; W[6] = p[7]; W[7] = p[4];
	W[8] = p[9]; W[9] = p[10]; W[10] = (T)1 + p[11]; W[11] = p[8];
	W[12] = 0; W[13] = 0; W[14] = 0; W[15] = 1;
}
template <class T>
inline void warp3d1_get(const T* W, T* p) { // :416-433
	p[0] = W[3]; p[1] = W[0] - (T)1; p[2] = W[1]; p[3] = W[2];
	p[4] = W[7]; p[5] = W[4]; p[6] = W[5] - (T)1; p[7] = W[6];
	p[8] = W[11]; p[9] = W[8]; p[10] = W[9]; p[11] = W[10] - (T)1;
}

// Pinning aid, OFF by default: the result tables shipped under examples/ were written before the "-4 = not converged"
// code existed (src/oc_icgn.cpp:329-332 is newer than the tables), so rows that hit the iteration limit keep their
// ZNCC there -- and EpipolarSearch, which ranks candidates by ZNCC after at most 5 iterations, picked candidates the
// current source would now discard.  With this flag the 2D IC-GN restatement skips that one rule so that the
// EpipolarSearch -> ICGN2D2 pipeline can be checked against examples/3d_dic/*_reconstruction_epipolar.csv.
static bool g_legacy_no_m4 = false;

// Per-thread scratch for 2D IC-GN (the reference's ICGN2D1_/ICGN2D2_, src/oc_icgn.h:30-43,85-98)
template <class T>
struct Scratch2D {
	std::vector<T> ref, tar, err, sd, gxw, gyw;
};

// ICGN2D1::compute(POI2D*) src/oc_icgn.cpp:144-341 (NP=6) and ICGN2D2::compute(POI2D*) :685-898 (NP=12).
// (template header follows the comment block below)
// With a centre offset (off_x, off_y) this is compute(POI2D*, Point2D& center_offset), :353-547 / :910-1126:
// local coordinates become (int - offset) and the target subset is centred at poi + offset.
// self_adaptive: the radius comes from the POI record (:152-158).
// damping != nullptr selects the Levenberg-Marquardt siblings ICLM2D1::compute (src/oc_iclm.cpp:150-358)
// and ICLM2D2::compute (:502-730): damping = {lambda, alpha, beta} (oc_iclm.h:32-37); the Hessian is damped
// with current_lambda * I and re-inverted every iteration, a step is accepted only if ZNSSD decreased, and
// -- unlike IC-GN -- out-of-range samples (-1) are NOT rejected.
template <class T, int NP>
void icgn2d_poi(const Ctx2D& c, float* poi, int rx, int ry, float conv_criterion, float stop_condition, Scratch2D<T>& s,
	float off_x = 0.f, float off_y = 0.f, bool self_adaptive = false, const float* damping = nullptr) {
	float px = poi[P2_X], py = poi[P2_Y];
	float* def = poi + P2_DEF;
	if (self_adaptive) {
		rx = (int)poi[P2_RX];
		ry = (int)poi[P2_RY];
	}
	// guard :160-167 / :701-708
	if (py - ry < 0 || px - rx < 0 || py + ry > c.h - 1 || px + rx > c.w - 1
		|| std::fabs(def[D2_U]) >= c.w || std::fabs(def[D2_V]) >= c.h
		|| poi[P2_ZNCC] < 0 || is_nan(def[D2_U]) || is_nan(def[D2_V])) {
		poi[P2_ZNCC] = poi[P2_ZNCC] >= 0 ? -3.f : poi[P2_ZNCC];
		return;
	}
	int sw = 2 * rx + 1, sh = 2 * ry + 1, n = sw * sh;
	s.ref.resize(n); s.tar.resize(n); s.err.resize(n); s.sd.resize((size_t)n * NP);
	// ref subset fill + zeroMeanNorm, src/oc_subset.cpp:39-53
	int uly = (int)(py - ry), ulx = (int)(px - rx);
	T mean = 0;
	for (int r = 0; r < sh; r++)
		for (int col = 0; col < sw; col++) {
			T v = c.ref[(size_t)(uly + r) * c.w + (ulx + col)];
			s.ref[r * sw + col] = v;
			mean += v;
		}
	mean /= n;
	T sq = 0;
	for (int i = 0; i < n; i++) { s.ref[i] -= mean; sq += s.ref[i] * s.ref[i]; }
	T ref_mean_norm = std::sqrt(sq);

	// SD images + Hessian :179-207 / :717-756
	T H[NP * NP];
	for (int i = 0; i < NP * NP; i++) H[i] = 0;
	for (int r = 0; r < sh; r++)
		for (int col = 0; col < sw; col++) {
			int xli = col - rx, yli = r - ry;
			int xg = (int)px + xli, yg = (int)py + yli;
			T gx = c.gx[(size_t)yg * c.w + xg], gy = c.gy[(size_t)yg * c.w + xg];
			T* sd = &s.sd[(size_t)(r * sw + col) * NP];
			T xl = (T)((float)xli - off_x), yl = (T)((float)yli - off_y); // exact integers when the offset is 0
			if (NP == 6) {
				sd[0] = gx; sd[1] = gx * xl; sd[2] = gx * yl;
				sd[3] = gy; sd[4] = gy * xl; sd[5] = gy * yl;
			} else {
				T xx = (xl * xl) * (T)0.5, xy = xl * yl, yy = (yl * yl) * (T)0.5;
				sd[0] = gx; sd[1] = gx * xl; sd[2] = gx * yl; sd[3] = gx * xx; sd[4] = gx * xy; sd[5] = gx * yy;
				sd[6] = gy; sd[7] = gy * xl; sd[8] = gy * yl; sd[9] = gy * xx; sd[10] = gy * xy; sd[11] = gy * yy;
			}
			for (int i = 0; i < NP; i++)
				for (int j = 0; j <= i; j++) {
					H[i * NP + j] += sd[i] * sd[j];
					H[j * NP + i] = H[i * NP + j];
				}
		}
	T invH[NP * NP];
	if (!damping) inverse_lu<T, NP>(H, invH);
	T current_lambda = 0, znssd0 = 4; // src/oc_iclm.cpp:234-235

	// initial guess: first-order terms only, also for ICGN2D2 (:216, :765-770)
	float p_init_u = def[D2_U], p_init_v = def[D2_V];
	constexpr int WN = (NP == 6) ? 3 : 6;
	T W[WN * WN], Winc[WN * WN], Winv[WN * WN], Wnew[WN * WN];
	T pcur[NP], dp[NP];
	if (NP == 6) {
		T p0[6] = { (T)def[D2_U], (T)def[D2_UX], (T)def[D2_UY], (T)def[D2_V], (T)def[D2_VX], (T)def[D2_VY] };
		for (int i = 0; i < 6; i++) pcur[i] = p0[i];
		warp2d1_set(pcur, W);
	} else {
		T p0[12] = { (T)def[D2_U], (T)def[D2_UX], (T)def[D2_UY], 0, 0, 0, (T)def[D2_V], (T)def[D2_VX], (T)def[D2_VY], 0, 0, 0 };
		for (int i = 0; i < 12; i++) pcur[i] = p0[i];
		warp2d2_set(pcur, W);
	}

	int iteration_counter = 0;
	T dp_norm_max = 0, znssd = 0;
	do {
		iteration_counter++;
		bool any_negative = false;
		for (int r = 0; r < sh; r++)
			for (int col = 0; col < sw; col++) {
				T xl = (T)((float)(col - rx) - off_x), yl = (T)((float)(r - ry) - off_y);
				T wx, wy;
				if (NP == 6) { // Deformation2D1::warp :94-105
					wx = W[0] * xl + W[1] * yl + W[2] * (T)1;
					wy = W[3] * xl + W[4] * yl + W[5] * (T)1;
				} else { // Deformation2D2::warp :268-282 (rows 3,4)
					T v0 = xl * xl, v1 = xl * yl, v2 = yl * yl;
					wx = W[18] * v0 + W[19] * v1 + W[20] * v2 + W[21] * xl + W[22] * yl + W[23] * (T)1;
					wy = W[24] * v0 + W[25] * v1 + W[26] * v2 + W[27] * xl + W[28] * yl + W[29] * (T)1;
				}
				T gxp = (T)(px + off_x) + wx, gyp = (T)(py + off_y) + wy; // center + warped (:239); center = poi + offset (:430-431)
				T val = bicubic_eval<T>(c, gxp, gyp);
				if (val < 0) any_negative = true;
				s.tar[r * sw + col] = val;
			}
		if (any_negative && !damping) { // :251-255 (the ICLM siblings have no such test)
			poi[P2_ZNCC] = -3.f;
			return;
		}
		T tmean = 0;
		for (int i = 0; i < n; i++) tmean += s.tar[i];
		tmean /= n;
		T tsq = 0;
		for (int i = 0; i < n; i++) { s.tar[i] -= tmean; tsq += s.tar[i] * s.tar[i]; }
		T tar_mean_norm = std::sqrt(tsq);
		T factor = ref_mean_norm / tar_mean_norm;
		T esq = 0;
		for (int i = 0; i < n; i++) { s.err[i] = s.tar[i] * factor - s.ref[i]; esq += s.err[i] * s.err[i]; }
		znssd = esq / (ref_mean_norm * ref_mean_norm);
		T num[NP];
		for (int i = 0; i < NP; i++) num[i] = 0;
		for (int i = 0; i < n; i++)
			for (int k = 0; k < NP; k++) num[k] += s.sd[(size_t)i * NP + k] * s.err[i];
		bool accept = true;
		if (damping) { // src/oc_iclm.cpp:258-266, :292-310
			if (iteration_counter == 1) current_lambda = (T)(std::pow((T)damping[0], znssd / znssd0) - (T)1);
			T Hd[NP * NP];
			for (int i = 0; i < NP * NP; i++) Hd[i] = H[i];
			for (int i = 0; i < NP; i++) Hd[i * NP + i] += current_lambda;
			inverse_lu<T, NP>(Hd, invH);
		}
		for (int i = 0; i < NP; i++) {
			dp[i] = 0;
			for (int j = 0; j < NP; j++) dp[i] += invH[i * NP + j] * num[j];
		}
		if (damping) {
			accept = znssd < znssd0;
			if (accept) { current_lambda = current_lambda * (T)damping[1]; znssd0 = znssd; }
			else current_lambda = current_lambda * (T)damping[2];
		}
		if (NP == 6) {
			warp2d1_set(dp, Winc);
			inverse3<T>(Winc, Winv);
			matmul<T, 3>(W, Winv, Wnew);
			if (accept) for (int i = 0; i < 9; i++) W[i] = Wnew[i];
			warp2d1_get(W, pcur);
			int rx2 = rx * rx, ry2 = ry * ry;
			dp_norm_max = dp[0] * dp[0] + dp[1] * dp[1] * rx2 + dp[2] * dp[2] * ry2
				+ dp[3] * dp[3] + dp[4] * dp[4] * rx2 + dp[5] * dp[5] * ry2;
		} else {
			warp2d2_set(dp, Winc);
			inverse_lu<T, WN>(Winc, Winv);
			matmul<T, WN>(W, Winv, Wnew);
			if (accept) for (int i = 0; i < WN * WN; i++) W[i] = Wnew[i];
			warp2d2_get(W, pcur);
			int rx2 = rx * rx, ry2 = ry * ry, rxy2 = rx2 * ry2;
			int rx4 = rx2 * rx2 * 0.25f, ry4 = ry2 * ry2 * 0.25f; // float->int truncation, :840-841
			dp_norm_max = dp[0] * dp[0] + dp[1] * dp[1] * rx2 + dp[2] * dp[2] * ry2
				+ dp[3] * dp[3] * rx4 + dp[5] * dp[5] * ry4 + dp[4] * dp[4] * rxy2
				+ dp[6] * dp[6] + dp[7] * dp[7] * rx2 + dp[8] * dp[8] * ry2
				+ dp[9] * dp[9] * rx4 + dp[11] * dp[11] * ry4 + dp[10] * dp[10] * rxy2;
		}
		dp_norm_max = std::sqrt(dp_norm_max);
	} while (iteration_counter < stop_condition && dp_norm_max >= conv_criterion);

	if (NP == 6) {
		def[D2_U] = (float)pcur[0]; def[D2_UX] = (float)pcur[1]; def[D2_UY] = (float)pcur[2];
		def[D2_V] = (float)pcur[3]; def[D2_VX] = (float)pcur[4]; def[D2_VY] = (float)pcur[5];
	} else {
		for (int i = 0; i < 12; i++) def[i] = (float)pcur[i];
	}
	poi[P2_U0] = p_init_u;
	poi[P2_V0] = p_init_v;
	poi[P2_ZNCC] = (float)((T)0.5 * ((T)2 - znssd));
	poi[P2_ITER] = (float)iteration_counter;
	poi[P2_CONV] = (float)dp_norm_max;
	poi[P2_RX] = (float)rx;
	poi[P2_RY] = (float)ry;
	if (!g_legacy_no_m4 && poi[P2_CONV] >= conv_criterion && poi[P2_ITER] >= stop_condition) poi[P2_ZNCC] = -4.f;
	if (is_nan(poi[P2_ZNCC]) || is_nan(def[D2_U]) || is_nan(def[D2_V])) {
		def[D2_U] = poi[P2_U0];
		def[D2_V] = poi[P2_V0];
		poi[P2_ZNCC] = -5.f;
	}
}

// NR2D1::compute(POI2D*), src/oc_nr.cpp:160-325: forward-additive Newton-Raphson, first-order shape function.
// Every iteration re-samples the target AND both target-gradient maps (three BicubicBspline tables,
// prepare :119-156), rebuilds the full 6x6 Hessian from the warped gradients, and adds dp to p.
// Differences from IC-GN worth pinning: the guard writes -1 (not -3) (:170); out-of-range samples (-1) are
// used as values, there is no negative-sample test; the error image is ref*(|t|/|r|) - tar and ZNSSD is
// normalised by |t|^2 (:244-247).
template <class T>
void nr2d1_poi(const Ctx2D& c, float* poi, int rx, int ry, float conv_criterion, float stop_condition, Scratch2D<T>& s) {
	float px = poi[P2_X], py = poi[P2_Y];
	float* def = poi + P2_DEF;
	if (py - ry < 0 || px - rx < 0 || py + ry > c.h - 1 || px + rx > c.w - 1
		|| std::fabs(def[D2_U]) >= c.w || std::fabs(def[D2_V]) >= c.h
		|| poi[P2_ZNCC] < 0 || is_nan(def[D2_U]) || is_nan(def[D2_V])) {
		poi[P2_ZNCC] = poi[P2_ZNCC] < -1 ? poi[P2_ZNCC] : -1.f; // :170
	} else {
		int sw = 2 * rx + 1, sh = 2 * ry + 1, n = sw * sh;
		s.ref.resize(n); s.tar.resize(n); s.err.resize(n); s.sd.resize((size_t)n * 6);
		std::vector<T>& tgx = s.gxw; std::vector<T>& tgy = s.gyw;
		tgx.resize(n); tgy.resize(n);
		int uly = (int)(py - ry), ulx = (int)(px - rx);
		T mean = 0;
		for (int r = 0; r < sh; r++)
			for (int col = 0; col < sw; col++) {
				T v = c.ref[(size_t)(uly + r) * c.w + (ulx + col)];
				s.ref[r * sw + col] = v;
				mean += v;
			}
		mean /= n;
		T sq = 0;
		for (int i = 0; i < n; i++) { s.ref[i] -= mean; sq += s.ref[i] * s.ref[i]; }
		T ref_mean_norm = std::sqrt(sq);

		float p_init_u = def[D2_U], p_init_v = def[D2_V];
		T p[6] = { (T)def[D2_U], (T)def[D2_UX], (T)def[D2_UY], (T)def[D2_V], (T)def[D2_VX], (T)def[D2_VY] };
		T W[9], dp[6];
		int iteration_counter = 0;
		T dp_norm_max = 0, znssd = 0;
		do {
			iteration_counter++;
			warp2d1_set(p, W);
			for (int r = 0; r < sh; r++)
				for (int col = 0; col < sw; col++) {
					T xl = (T)(col - rx), yl = (T)(r - ry);
					T wx = W[0] * xl + W[1] * yl + W[2] * (T)1;
					T wy = W[3] * xl + W[4] * yl + W[5] * (T)1;
					T gxp = (T)px + wx, gyp = (T)py + wy;
					s.tar[r * sw + col] = bicubic_eval<T>(c, c.lut, gxp, gyp);
					tgx[r * sw + col] = bicubic_eval<T>(c, c.lut_tgx, gxp, gyp);
					tgy[r * sw + col] = bicubic_eval<T>(c, c.lut_tgy, gxp, gyp);
				}
			T tmean = 0;
			for (int i = 0; i < n; i++) tmean += s.tar[i];
			tmean /= n;
			T tsq = 0;
			for (int i = 0; i < n; i++) { s.tar[i] -= tmean; tsq += s.tar[i] * s.tar[i]; }
			T tar_mean_norm = std::sqrt(tsq);
			T H[36], invH[36];
			for (int i = 0; i < 36; i++) H[i] = 0;
			for (int r = 0; r < sh; r++)
				for (int col = 0; col < sw; col++) {
					T xl = (T)(col - rx), yl = (T)(r - ry);
					T gx = tgx[r * sw + col], gy = tgy[r * sw + col];
					T* sd = &s.sd[(size_t)(r * sw + col) * 6];
					sd[0] = gx; sd[1] = gx * xl; sd[2] = gx * yl;
					sd[3] = gy; sd[4] = gy * xl; sd[5] = gy * yl;
					for (int i = 0; i < 6; i++)
						for (int j = 0; j < 6; j++) H[i * 6 + j] += sd[i] * sd[j];
				}
			inverse_lu<T, 6>(H, invH);
			T factor = tar_mean_norm / ref_mean_norm;
			T esq = 0;
			for (int i = 0; i < n; i++) { s.err[i] = s.ref[i] * factor - s.tar[i]; esq += s.err[i] * s.err[i]; }
			znssd = esq / (tar_mean_norm * tar_mean_norm);
			T num[6] = { 0, 0, 0, 0, 0, 0 };
			for (int i = 0; i < n; i++)
				for (int k = 0; k < 6; k++) num[k] += s.sd[(size_t)i * 6 + k] * s.err[i];
			for (int i = 0; i < 6; i++) {
				dp[i] = 0;
				for (int j = 0; j < 6; j++) dp[i] += invH[i * 6 + j] * num[j];
			}
			for (int i = 0; i < 6; i++) p[i] += dp[i];
			int rx2 = rx * rx, ry2 = ry * ry;
			dp_norm_max = dp[0] * dp[0] + dp[1] * dp[1] * rx2 + dp[2] * dp[2] * ry2
				+ dp[3] * dp[3] + dp[4] * dp[4] * rx2 + dp[5] * dp[5] * ry2;
			dp_norm_max = std::sqrt(dp_norm_max);
		} while (iteration_counter < stop_condition && dp_norm_max >= conv_criterion);
		def[D2_U] = (float)p[0]; def[D2_UX] = (float)p[1]; def[D2_UY] = (float)p[2];
		def[D2_V] = (float)p[3]; def[D2_VX] = (float)p[4]; def[D2_VY] = (float)p[5];
		poi[P2_U0] = p_init_u;
		poi[P2_V0] = p_init_v;
		poi[P2_ZNCC] = (float)((T)0.5 * ((T)2 - znssd));
		poi[P2_ITER] = (float)iteration_counter;
		poi[P2_CONV] = (float)dp_norm_max;
	}
	// evaluated for every POI, also the guarded ones (:314-324)
	if (poi[P2_CONV] >= conv_criterion && poi[P2_ITER] >= stop_condition) poi[P2_ZNCC] = -4.f;
	if (is_nan(poi[P2_ZNCC]) || is_nan(def[D2_U]) || is_nan(def[D2_V])) {
		def[D2_U] = poi[P2_U0];
		def[D2_V] = poi[P2_V0];
		poi[P2_ZNCC] = -5.f;
	}
}

// ----------------------------------------------------------------------------------------------
// 3D context.
// ----------------------------------------------------------------------------------------------
struct Ctx3D {
	int dx = 0, dy = 0, dz = 0, threads = 1;
	std::vector<float> ref, tar;       // [z][y][x]
	std::vector<float> gx, gy, gz;     // Gradient3D4 of ref
	std::vector<float> coef;           // TricubicBspline coefficient of tar
	bool prepared = false;
	inline size_t at(int z, int y, int x) const { return ((size_t)z * dy + y) * dx + x; }
};

// Gradient3D4::getGradientX/Y/Z, src/oc_gradient.cpp:143-231.
void gradient3d(Ctx3D& c) {
	const float first_factor = 1.f / 12.f, second_factor = 2.f / 3.f;
	size_t total = (size_t)c.dx * c.dy * c.dz;
	c.gx.assign(total, 0.f); c.gy.assign(total, 0.f); c.gz.assign(total, 0.f);
	const float* f = c.ref.data();
#pragma omp parallel for num_threads(c.threads)
	for (int i = 0; i < c.dz; i++)
		for (int j = 0; j < c.dy; j++) {
			for (int k = 2; k < c.dx - 2; k++) {
				float result = 0.0f;
				result -= f[c.at(i, j, k + 2)] * first_factor;
				result += f[c.at(i, j, k + 1)] * second_factor;
				result -= f[c.at(i, j, k - 1)] * second_factor;
				result += f[c.at(i, j, k - 2)] * first_factor;
				c.gx[c.at(i, j, k)] = result;
			}
			if (j >= 2 && j < c.dy - 2)
				for (int k = 0; k < c.dx; k++) {
					float result = 0.0f;
					result -= f[c.at(i, j + 2, k)] * first_factor;
					result += f[c.at(i, j + 1, k)] * second_factor;
					result -= f[c.at(i, j - 1, k)] * second_factor;
					result += f[c.at(i, j - 2, k)] * first_factor;
					c.gy[c.at(i, j, k)] = result;
				}
			if (i >= 2 && i < c.dz - 2)
				for (int k = 0; k < c.dx; k++) {
					float result = 0.0f;
					result -= f[c.at(i + 2, j, k)] * first_factor;
					result += f[c.at(i + 1, j, k)] * second_factor;
					result -= f[c.at(i - 1, j, k)] * second_factor;
					result += f[c.at(i - 2, j, k)] * first_factor;
					c.gz[c.at(i, j, k)] = result;
				}
		}
}

// src/oc_cubic_bspline.h:80-90
const float BSPLINE_PREFILTER[8] = { 1.732176555412860f, -0.464135309171000f, 0.124364681271139f, -0.033323415913556f,
	0.008928982383084f, -0.002392513618779f, 0.000641072092032f, -0.000171774749350f };

inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// One 15-tap symmetric FIR pass with index clamping (src/oc_cubic_bspline.cpp:224-348).  The
// reference's three code branches (interior / low edge / high edge) all reduce to this
// expression with clamped indices; the summation order b0, b1..b7 is kept.
void prefilter_axis(const std::vector<float>& in, std::vector<float>& out, int dx, int dy, int dz, int axis, int threads) {
	size_t sx = 1, sy = (size_t)dx, sz = (size_t)dx * dy;
	size_t stride = axis == 0 ? sx : (axis == 1 ? sy : sz);
	int dim = axis == 0 ? dx : (axis == 1 ? dy : dz);
#pragma omp parallel for num_threads(threads)
	for (int i = 0; i < dz; i++)
		for (int j = 0; j < dy; j++)
			for (int k = 0; k < dx; k++) {
				size_t base = (size_t)i * sz + (size_t)j * sy + k;
				int pos = axis == 0 ? k : (axis == 1 ? j : i);
				const float* line = &in[base - (size_t)pos * stride];
				float v = BSPLINE_PREFILTER[0] * line[(size_t)pos * stride];
				for (int t = 1; t <= 7; t++)
					v = v + BSPLINE_PREFILTER[t] * (line[(size_t)clampi(pos - t, 0, dim - 1) * stride] + line[(size_t)clampi(pos + t, 0, dim - 1) * stride]);
				out[base] = v;
			}
}

// TricubicBspline::prepare, src/oc_cubic_bspline.cpp:214-351: x -> y -> z passes.
void tricubic_prepare(Ctx3D& c) {
	size_t total = (size_t)c.dx * c.dy * c.dz;
	std::vector<float> tmp(total);
	c.coef.assign(total, 0.f);
	prefilter_axis(c.tar, c.coef, c.dx, c.dy, c.dz, 0, c.threads);
	prefilter_axis(c.coef, tmp, c.dx, c.dy, c.dz, 1, c.threads);
	prefilter_axis(tmp, c.coef, c.dx, c.dy, c.dz, 2, c.threads);
}

// basis functions, src/oc_cubic_bspline.cpp:35-53
template <class T> inline T basis0(T t) { return ((T)1 / (T)6) * (t * (t * (-t + (T)3) - (T)3) + (T)1); }
template <class T> inline T basis1(T t) { return ((T)1 / (T)6) * (t * t * ((T)3 * t - (T)6) + (T)4); }
template <class T> inline T basis2(T t) { return ((T)1 / (T)6) * (t * (t * ((T)-3 * t + (T)3) + (T)3) + (T)1); }
template <class T> inline T basis3(T t) { return ((T)1 / (T)6) * (t * t * t); }

// TricubicBspline::compute, src/oc_cubic_bspline.cpp:353-405
template <class T>
inline T tricubic_eval(const Ctx3D& c, T x, T y, T z) {
	if (x < 1 || y < 1 || z < 1 || x >= c.dx - 2 || y >= c.dy - 2 || z >= c.dz - 2 || is_nan(x) || is_nan(y) || is_nan(z)) return (T)-1;
	int xi = (int)std::floor(x), yi = (int)std::floor(y), zi = (int)std::floor(z);
	T xd = x - xi, yd = y - yi, zd = z - zi;
	T bx[4] = { basis0(xd), basis1(xd), basis2(xd), basis3(xd) };
	T by[4] = { basis0(yd), basis1(yd), basis2(yd), basis3(yd) };
	T bz[4] = { basis0(zd), basis1(zd), basis2(zd), basis3(zd) };
	T sum_x[4], sum_y[4];
	for (int i = 0; i < 4; i++) {
		for (int j = 0; j < 4; j++) {
			const float* row = &c.coef[c.at(zi + i - 1, yi + j - 1, xi - 1)];
			sum_x[j] = bx[0] * (T)row[0] + bx[1] * (T)row[1] + bx[2] * (T)row[2] + bx[3] * (T)row[3];
		}
		sum_y[i] = by[0] * sum_x[0] + by[1] * sum_x[1] + by[2] * sum_x[2] + by[3] * sum_x[3];
	}
	return bz[0] * sum_y[0] + bz[1] * sum_y[1] + bz[2] * sum_y[2] + bz[3] * sum_y[3];
}

// FFTCC3D::compute(POI3D*), src/oc_fftcc.cpp:327-427.  No border guard in the reference; the
// oracle refuses (leaves the POI untouched) instead of reading out of bounds.
template <class T>
void fftcc3d_poi(const Ctx3D& c, float* poi, int rx, int ry, int rz, const FFT<T>& fx, const FFT<T>& fy, const FFT<T>& fz, FftScratch<T>& fs) {
	typedef std::complex<T> cpx;
	int sx = 2 * rx, sy = 2 * ry, sz = 2 * rz;
	size_t size = (size_t)sx * sy * sz;
	float px = poi[P3_X], py = poi[P3_Y], pz = poi[P3_Z];
	float u0 = poi[P3_DEF + 0], v0 = poi[P3_DEF + 4], w0 = poi[P3_DEF + 8];
	// a NaN position or guess is refused, as the kernels do, before it reaches an (int) conversion
	if (is_nan(px) || is_nan(py) || is_nan(pz) || is_nan(u0) || is_nan(v0) || is_nan(w0)) return;
	{
		int x0 = (int)(px - rx), y0 = (int)(py - ry), z0 = (int)(pz - rz);
		int x1 = (int)(px + sx - 1 - rx), y1 = (int)(py + sy - 1 - ry), z1 = (int)(pz + sz - 1 - rz);
		int tx0 = (int)(px - rx + u0), ty0 = (int)(py - ry + v0), tz0 = (int)(pz - rz + w0);
		int tx1 = (int)(px + sx - 1 - rx + u0), ty1 = (int)(py + sy - 1 - ry + v0), tz1 = (int)(pz + sz - 1 - rz + w0);
		if (x0 < 0 || y0 < 0 || z0 < 0 || x1 >= c.dx || y1 >= c.dy || z1 >= c.dz
			|| tx0 < 0 || ty0 < 0 || tz0 < 0 || tx1 >= c.dx || ty1 >= c.dy || tz1 >= c.dz
			|| px - rx < 0 || py - ry < 0 || pz - rz < 0 || px - rx + u0 < 0 || py - ry + v0 < 0 || pz - rz + w0 < 0)
			return;
	}
	fs.resize(size);
	std::vector<T>& a = fs.a;
	std::vector<T>& b = fs.b;
	std::vector<cpx>& buf = fs.buf;
	std::vector<cpx>& cc = fs.cc;
	std::vector<cpx>& scratch = fs.scratch;
	T ref_mean = 0, tar_mean = 0, ref_norm = 0, tar_norm = 0;
	for (int i = 0; i < sz; i++)
		for (int j = 0; j < sy; j++)
			for (int k = 0; k < sx; k++) {
				float rpx = px + k - rx, rpy = py + j - ry, rpz = pz + i - rz; // :353
				float value = c.ref[c.at((int)rpz, (int)rpy, (int)rpx)];
				size_t o = ((size_t)i * sy + j) * sx + k;
				a[o] = value;
				ref_mean += value;
				float tpx = rpx + u0, tpy = rpy + v0, tpz = rpz + w0; // :359
				value = c.tar[c.at((int)tpz, (int)tpy, (int)tpx)];
				b[o] = value;
				tar_mean += value;
			}
	ref_mean /= size;
	tar_mean /= size;
	for (size_t i = 0; i < size; i++) {
		a[i] -= ref_mean;
		b[i] -= tar_mean;
		ref_norm += a[i] * a[i];
		tar_norm += b[i] * b[i];
	}
	for (size_t i = 0; i < size; i++) buf[i] = cpx(a[i], b[i]);
	std::vector<cpx>& tmp = fs.tmp;
	tmp.resize((size_t)sx * sy);
	auto fft3 = [&](std::vector<cpx>& d, bool inv) {
		for (int i = 0; i < sz; i++) fft_rows(fx, d.data() + (size_t)i * sy * sx, tmp.data(), scratch.data(), sy, inv);
		for (int i = 0; i < sz; i++) fy.run(d.data() + (size_t)i * sy * sx, scratch.data(), sx, inv);
		fz.run(d.data(), scratch.data(), (long)sx * sy, inv);
	};
	fft3(buf, false);
	for (int kz = 0; kz < sz; kz++)
		for (int ky = 0; ky < sy; ky++)
			for (int kx = 0; kx < sx; kx++) {
				cpx z = buf[((size_t)kz * sy + ky) * sx + kx];
				cpx zm = std::conj(buf[((size_t)((sz - kz) % sz) * sy + ((sy - ky) % sy)) * sx + ((sx - kx) % sx)]);
				cpx A = (z + zm) * (T)0.5;
				cpx d = (z - zm) * (T)0.5;
				cpx B = cpx(d.imag(), -d.real());
				cc[((size_t)kz * sy + ky) * sx + kx] = cpx(A.real() * B.real() + A.imag() * B.imag(), A.real() * B.imag() - A.imag() * B.real());
			}
	fft3(cc, true);
	// A window of constant grey is zero after the mean is taken off, and the reference, which transforms the two windows
	// separately (:378-379), then gets a surface that is zero everywhere: index 0 wins and ZNCC is 0 / 0.  The packed transform
	// above only gives Z(k) + conj Z(-k) = 0 up to rounding.
	if (ref_norm == 0 || tar_norm == 0)
		for (size_t i = 0; i < size; i++) cc[i] = cpx(0, 0);
	T max_zncc = (T)-2;
	size_t idx = 0;
	for (size_t i = 0; i < size; i++) {
		if (cc[i].real() > max_zncc) { max_zncc = cc[i].real(); idx = i; }
	}
	int du = (int)(idx % sx), dv = (int)((idx / sx) % sy), dw = (int)(idx / ((size_t)sx * sy));
	if (du > rx) du -= sx;
	if (dv > ry) dv -= sy;
	if (dw > rz) dw -= sz;
	poi[P3_DEF + 0] = (float)du + u0;
	poi[P3_DEF + 4] = (float)dv + v0;
	poi[P3_DEF + 8] = (float)dw + w0;
	poi[P3_U0] = u0; poi[P3_V0] = v0; poi[P3_W0] = w0;
	poi[P3_ZNCC] = (float)(max_zncc / (std::sqrt(ref_norm * tar_norm) * size));
}

template <class T>
struct Scratch3D {
	std::vector<T> ref, tar, err, sd;
};

// ICGN3D1::compute(POI3D*), src/oc_icgn.cpp:1270-1490.
template <class T>
void icgn3d1_poi(const Ctx3D& c, float* poi, int rx, int ry, int rz, float conv_criterion, float stop_condition, Scratch3D<T>& s) {
	float px = poi[P3_X], py = poi[P3_Y], pz = poi[P3_Z];
	float* def = poi + P3_DEF;
	if ((px - rx) < 0 || (py - ry) < 0 || (pz - rz) < 0
		|| (px + rx) > (c.dx - 1) || (py + ry) > (c.dy - 1) || (pz + rz) > (c.dz - 1)
		|| std::fabs(def[0]) >= c.dx || std::fabs(def[4]) >= c.dy || std::fabs(def[8]) >= c.dz
		|| poi[P3_ZNCC] < 0 || is_nan(def[0]) || is_nan(def[4]) || is_nan(def[8])) {
		poi[P3_ZNCC] = poi[P3_ZNCC] >= 0 ? -3.f : poi[P3_ZNCC];
		return;
	}
	int sx = 2 * rx + 1, sy = 2 * ry + 1, sz = 2 * rz + 1;
	size_t n = (size_t)sx * sy * sz;
	s.ref.resize(n); s.tar.resize(n); s.err.resize(n); s.sd.resize(n * 12);
	// Subset3D::fill + zeroMeanNorm, src/oc_subset.cpp:89-135
	float stx = px - rx, sty = py - ry, stz = pz - rz;
	T mean = 0;
	for (int i = 0; i < sz; i++)
		for (int j = 0; j < sy; j++)
			for (int k = 0; k < sx; k++) {
				T v = c.ref[c.at(int(stz + i), int(sty + j), int(stx + k))];
				s.ref[((size_t)i * sy + j) * sx + k] = v;
				mean += v;
			}
	mean /= n;
	T sq = 0;
	for (size_t i = 0; i < n; i++) { s.ref[i] -= mean; sq += s.ref[i] * s.ref[i]; }
	T ref_mean_norm = std::sqrt(sq);

	T H[144];
	for (int i = 0; i < 144; i++) H[i] = 0;
	for (int i = 0; i < sz; i++)
		for (int j = 0; j < sy; j++)
			for (int k = 0; k < sx; k++) {
				int xl = k - rx, yl = j - ry, zl = i - rz;
				size_t g = c.at((int)pz + zl, (int)py + yl, (int)px + xl);
				T gx = c.gx[g], gy = c.gy[g], gz = c.gz[g];
				T* sd = &s.sd[(((size_t)i * sy + j) * sx + k) * 12];
				sd[0] = gx; sd[1] = gx * xl; sd[2] = gx * yl; sd[3] = gx * zl;
				sd[4] = gy; sd[5] = gy * xl; sd[6] = gy * yl; sd[7] = gy * zl;
				sd[8] = gz; sd[9] = gz * xl; sd[10] = gz * yl; sd[11] = gz * zl;
				for (int r = 0; r < 12; r++)
					for (int cc = 0; cc <= r; cc++) {
						H[r * 12 + cc] += sd[r] * sd[cc];
						H[cc * 12 + r] = H[r * 12 + cc];
					}
			}
	T invH[144];
	inverse_lu<T, 12>(H, invH);

	float u_init = def[0], v_init = def[4], w_init = def[8];
	T pcur[12], dp[12], W[16], Winc[16], Winv[16], Wnew[16];
	for (int i = 0; i < 12; i++) pcur[i] = def[i];
	warp3d1_set(pcur, W);
	int iteration_counter = 0;
	T dp_norm_max = 0, znssd = 0;
	do {
		iteration_counter++;
		bool out_of_range = false;
		for (int i = 0; i < sz; i++)
			for (int j = 0; j < sy; j++)
				for (int k = 0; k < sx; k++) {
					T xl = (T)(k - rx), yl = (T)(j - ry), zl = (T)(i - rz);
					T wx = W[0] * xl + W[1] * yl + W[2] * zl + W[3] * (T)1;
					T wy = W[4] * xl + W[5] * yl + W[6] * zl + W[7] * (T)1;
					T wz = W[8] * xl + W[9] * yl + W[10] * zl + W[11] * (T)1;
					T val = tricubic_eval<T>(c, (T)px + wx, (T)py + wy, (T)pz + wz);
					if (val < 0) out_of_range = true;
					s.tar[((size_t)i * sy + j) * sx + k] = val;
				}
		if (out_of_range) {
			poi[P3_ZNCC] = -3.f;
			return;
		}
		T tmean = 0;
		for (size_t i = 0; i < n; i++) tmean += s.tar[i];
		tmean /= n;
		T tsq = 0;
		for (size_t i = 0; i < n; i++) { s.tar[i] -= tmean; tsq += s.tar[i] * s.tar[i]; }
		T tar_mean_norm = std::sqrt(tsq);
		T factor = ref_mean_norm / tar_mean_norm;
		T esq = 0;
		for (size_t i = 0; i < n; i++) { s.err[i] = factor * s.tar[i] - s.ref[i]; esq += s.err[i] * s.err[i]; }
		znssd = esq / (ref_mean_norm * ref_mean_norm);
		T num[12];
		for (int i = 0; i < 12; i++) num[i] = 0;
		for (size_t i = 0; i < n; i++)
			for (int l = 0; l < 12; l++) num[l] += s.sd[i * 12 + l] * s.err[i];
		for (int i = 0; i < 12; i++) {
			dp[i] = 0;
			for (int j = 0; j < 12; j++) dp[i] += invH[i * 12 + j] * num[j];
		}
		warp3d1_set(dp, Winc);
		inverse4<T>(Winc, Winv);
		matmul<T, 4>(W, Winv, Wnew);
		for (int i = 0; i < 16; i++) W[i] = Wnew[i];
		warp3d1_get(W, pcur);
		dp_norm_max = std::sqrt(dp[0] * dp[0] + dp[4] * dp[4] + dp[8] * dp[8]); // :1445, translation only
	} while (iteration_counter < stop_condition && dp_norm_max >= conv_criterion);

	for (int i = 0; i < 12; i++) def[i] = (float)pcur[i];
	poi[P3_U0] = u_init; poi[P3_V0] = v_init; poi[P3_W0] = w_init;
	poi[P3_ZNCC] = (float)((T)0.5 * ((T)2 - znssd));
	poi[P3_ITER] = (float)iteration_counter;
	poi[P3_CONV] = (float)dp_norm_max;
	poi[P3_RX] = (float)rx; poi[P3_RY] = (float)ry; poi[P3_RZ] = (float)rz;
	if (poi[P3_CONV] >= conv_criterion && poi[P3_ITER] >= stop_condition) poi[P3_ZNCC] = -4.f;
	if (is_nan(poi[P3_ZNCC]) || is_nan(def[0]) || is_nan(def[4]) || is_nan(def[8])) {
		def[0] = poi[P3_U0]; def[4] = poi[P3_V0]; def[8] = poi[P3_W0];
		poi[P3_ZNCC] = -5.f;
	}
}

template <class T>
void run_fftcc2d(const Ctx2D& c, float* pois, long n, int rx, int ry) {
	FFT<T> fx, fy;
	fx.plan(2 * rx);
	fy.plan(2 * ry);
#pragma omp parallel num_threads(c.threads)
	{
		FftScratch<T> fs;
#pragma omp for schedule(dynamic, 64)
		for (long i = 0; i < n; i++) fftcc2d_poi<T>(c, pois + i * P2_N, rx, ry, fx, fy, fs);
	}
}
template <class T, int NP>
void run_icgn2d(const Ctx2D& c, float* pois, long n, int rx, int ry, float conv, float stop, const float* offsets = nullptr, bool self_adaptive = false,
	const float* damping = nullptr) {
#pragma omp parallel num_threads(c.threads)
	{
		Scratch2D<T> s;
#pragma omp for schedule(dynamic, 64)
		for (long i = 0; i < n; i++)
			icgn2d_poi<T, NP>(c, pois + i * P2_N, rx, ry, conv, stop, s, offsets ? offsets[2 * i] : 0.f, offsets ? offsets[2 * i + 1] : 0.f, self_adaptive, damping);
	}
}
template <class T>
void run_nr2d1(const Ctx2D& c, float* pois, long n, int rx, int ry, float conv, float stop) {
#pragma omp parallel num_threads(c.threads)
	{
		Scratch2D<T> s;
#pragma omp for schedule(dynamic, 64)
		for (long i = 0; i < n; i++) nr2d1_poi<T>(c, pois + i * P2_N, rx, ry, conv, stop, s);
	}
}
template <class T>
void run_fftcc3d(const Ctx3D& c, float* pois, long n, int rx, int ry, int rz) {
	FFT<T> fx, fy, fz;
	fx.plan(2 * rx); fy.plan(2 * ry); fz.plan(2 * rz);
#pragma omp parallel num_threads(c.threads)
	{
		FftScratch<T> fs;
#pragma omp for schedule(dynamic, 1)
		for (long i = 0; i < n; i++) fftcc3d_poi<T>(c, pois + i * P3_N, rx, ry, rz, fx, fy, fz, fs);
	}
}
template <class T>
void run_icgn3d1(const Ctx3D& c, float* pois, long n, int rx, int ry, int rz, float conv, float stop) {
#pragma omp parallel num_threads(c.threads)
	{
		Scratch3D<T> s;
#pragma omp for schedule(dynamic, 1)
		for (long i = 0; i < n; i++) icgn3d1_poi<T>(c, pois + i * P3_N, rx, ry, rz, conv, stop, s);
	}
}

// ----------------------------------------------------------------------------------------------
// Strain (reference src/oc_strain.cpp): per-POI least-squares plane fit of the displacement field over the
// neighbours found by NearestNeighbor (src/oc_nearest_neighbor.cpp: a nanoflann kd-tree, third-party header
// not vendored in the reference tree; nanoflann >= 1.5.0 semantics restated: radiusSearch returns the points
// with squared L2 distance STRICTLY below radius^2 -- RadiusResultSet::addPoint `if (dist < radius)` -- and
// knnSearch the k nearest, ties in unspecified order; here ties go to the lower index).
// Strain::compute(POI2D*, queue) :158-237, Strain::compute(POI3D*, queue) :373-474, batch :239-250 / :476-487.
// D = 2: POI2D records (25 floats), strain = {exx, eyy, exy}; D = 3: POI3D (31 floats), {exx, eyy, ezz, exy, eyz, ezx}.
// ----------------------------------------------------------------------------------------------
// MODE 2: POI2D, MODE 3: POI3D, MODE 23: POI2DS (stereo DIC: neighbours are searched in the image plane of the primary
// view, the plane fit runs over the reconstructed 3D coordinates ref_coor and u, v, w; a POI counts when all of
// r1r2 / r1t1 / r1t2 ZNCC pass the threshold, src/oc_strain.cpp:252-371).  SD = search dimensions, FD = fit dimensions,
// FC = offset of the fit coordinates in the record, Z0.. = the ZNCC fields that must pass.
template <int MODE> struct StrainLayout;
template <> struct StrainLayout<2> { enum { NF = P2_N, SD = 2, FD = 2, FC = 0, NZ = 1, Z0 = P2_ZNCC, STRAIN = P2_STRAIN, U = P2_DEF + D2_U, V = P2_DEF + D2_V, W = -1 }; };
template <> struct StrainLayout<3> { enum { NF = P3_N, SD = 3, FD = 3, FC = 0, NZ = 1, Z0 = P3_ZNCC, STRAIN = P3_STRAIN, U = P3_DEF + 0, V = P3_DEF + 4, W = P3_DEF + 8 }; };
// POI2DS record (src/oc_poi.h:140-186): x y | u v w | r1r2 r1t1 r1t2 r2_x r2_y t1_x t1_y t2_x t2_y | ref_coor | tar_coor | e[6] | subset_radius
enum { PS_N = 28, PS_U = 2, PS_Z = 5, PS_REF = 14, PS_STRAIN = 20 };
template <> struct StrainLayout<23> { enum { NF = PS_N, SD = 2, FD = 3, FC = PS_REF, NZ = 3, Z0 = PS_Z, STRAIN = PS_STRAIN, U = PS_U, V = PS_U + 1, W = PS_U + 2 }; };
template <int MODE>
inline bool strain_good(const float* p, float thr) {
	typedef StrainLayout<MODE> L;
	for (int k = 0; k < L::NZ; k++)
		if (!(p[L::Z0 + k] >= thr)) return false;
	return true;
}

// least squares A x = b_k for NB right-hand sides by column-pivoted Householder QR (what Eigen's
// colPivHouseholderQr().solve does), A is m x C row-major in `a`, b is m x NB row-major; destroys both.
template <class T, int C, int NB>
void lsq_qr(std::vector<T>& a, std::vector<T>& b, int m, T x[NB][C]) {
	int perm[C];
	for (int j = 0; j < C; j++) perm[j] = j;
	int rank = 0;
	T first_norm = 0;
	for (int k = 0; k < C && k < m; k++) {
		// pivot: remaining column with the largest norm
		int best = k;
		T bestn = -1;
		for (int j = k; j < C; j++) {
			T s = 0;
			for (int i = k; i < m; i++) s += a[(size_t)i * C + j] * a[(size_t)i * C + j];
			if (s > bestn) { bestn = s; best = j; }
		}
		if (k == 0) first_norm = bestn;
		if (bestn <= first_norm * (T)1e-12) break; // rank deficient: remaining unknowns stay 0
		if (best != k) {
			for (int i = 0; i < m; i++) std::swap(a[(size_t)i * C + k], a[(size_t)i * C + best]);
			std::swap(perm[k], perm[best]);
		}
		T alpha = std::sqrt(bestn);
		if (a[(size_t)k * C + k] > 0) alpha = -alpha;
		std::vector<T> v(m - k);
		for (int i = k; i < m; i++) v[i - k] = a[(size_t)i * C + k];
		v[0] -= alpha;
		T vn = 0;
		for (T e : v) vn += e * e;
		if (vn > 0) {
			for (int j = k; j < C; j++) {
				T d = 0;
				for (int i = k; i < m; i++) d += v[i - k] * a[(size_t)i * C + j];
				d = (T)2 * d / vn;
				for (int i = k; i < m; i++) a[(size_t)i * C + j] -= d * v[i - k];
			}
			for (int j = 0; j < NB; j++) {
				T d = 0;
				for (int i = k; i < m; i++) d += v[i - k] * b[(size_t)i * NB + j];
				d = (T)2 * d / vn;
				for (int i = k; i < m; i++) b[(size_t)i * NB + j] -= d * v[i - k];
			}
		}
		rank++;
	}
	for (int j = 0; j < NB; j++) {
		T y[C];
		for (int k = 0; k < C; k++) y[k] = 0;
		for (int k = rank - 1; k >= 0; k--) {
			T s = b[(size_t)k * NB + j];
			for (int l = k + 1; l < rank; l++) s -= a[(size_t)k * C + l] * y[l];
			y[k] = s / a[(size_t)k * C + k];
		}
		for (int k = 0; k < C; k++) x[j][perm[k]] = y[k];
	}
}

// only < 0: Strain::compute(queue), every POI whose ZNCC passes the threshold.  only >= 0: Strain::compute(POI*, queue)
// (:158-237, :373-474) on POI `only` alone, whatever its own ZNCC.  POIs with a non-finite position are neither fitted
// nor anyone's neighbour (a kd-tree cannot place them).
template <class T, int MODE>
void run_strain(float* pois, long n, float radius, int k_min, float zncc_threshold, int approximation, int threads, long only = -1) {
	typedef StrainLayout<MODE> L;
	constexpr int NF = L::NF, D = L::SD, FD = L::FD, NE = FD == 2 ? 3 : 6; // D: search dimensions
	auto finite = [&](const float* p) { for (int d = 0; d < D; d++) if (!std::isfinite(p[d])) return false; return true; };
	if (approximation != 1 && approximation != 2) return; // the reference writes no strain for any other value (:220-233)
	// uniform grid over the POI positions
	double lo[3] = { 0, 0, 0 }, hi[3] = { 0, 0, 0 };
	for (int d = 0; d < D; d++) { lo[d] = HUGE_VAL; hi[d] = -HUGE_VAL; }
	for (long i = 0; i < n; i++)
		if (finite(pois + i * NF))
			for (int d = 0; d < D; d++) { lo[d] = std::min(lo[d], (double)pois[i * NF + d]); hi[d] = std::max(hi[d], (double)pois[i * NF + d]); }
	if (lo[0] > hi[0]) return; // no POI with a finite position
	// cell edge > |radius| (the test is dist^2 < radius^2, so a negative radius acts as its magnitude; the 0.1 % covers a
	// float dist^2 that rounds below radius^2), one cell over the bbox for a non-finite radius (+-inf: every POI is a
	// neighbour, NaN: none is), doubled until the grid has no more cells than a few per POI
	double extent = 0;
	for (int d = 0; d < D; d++) extent = std::max(extent, hi[d] - lo[d]);
	const double abs_radius = std::fabs((double)radius);
	double cell = !std::isfinite(abs_radius) ? extent + 1.0 : abs_radius > 0 ? abs_radius * 1.001 : 1.0;
	long nc[3] = { 1, 1, 1 };
	while (true) {
		double total = 1;
		for (int d = 0; d < D; d++) total *= std::floor((hi[d] - lo[d]) / cell) + 1;
		if (total <= 4.0 * (double)n + 1024.0) break;
		cell *= 2;
	}
	for (int d = 0; d < D; d++) nc[d] = (long)std::floor((hi[d] - lo[d]) / cell) + 1;
	auto cell_of = [&](const float* p, long* c) {
		for (int d = 0; d < 3; d++) c[d] = d < D ? std::min(nc[d] - 1, (long)std::floor(((double)p[d] - lo[d]) / cell)) : 0;
	};
	std::vector<long> start((size_t)(nc[0] * nc[1] * nc[2]) + 1, 0), order(n);
	for (long i = 0; i < n; i++) {
		if (!finite(pois + i * NF)) continue;
		long c[3];
		cell_of(pois + i * NF, c);
		start[(c[2] * nc[1] + c[1]) * nc[0] + c[0] + 1]++;
	}
	for (size_t k = 1; k < start.size(); k++) start[k] += start[k - 1];
	{
		std::vector<long> fill(start.begin(), start.end() - 1);
		for (long i = 0; i < n; i++) {
			if (!finite(pois + i * NF)) continue;
			long c[3];
			cell_of(pois + i * NF, c);
			order[fill[(c[2] * nc[1] + c[1]) * nc[0] + c[0]]++] = i;
		}
	}
	std::vector<float> out((size_t)n * NE);
	std::vector<char> done(n, 0);
	const float r2 = radius * radius;
#pragma omp parallel num_threads(threads)
	{
		std::vector<long> fit;
		std::vector<std::pair<float, long>> cand;
		std::vector<T> A, B;
#pragma omp for schedule(dynamic, 64)
		for (long i = 0; i < n; i++) {
			const float* p = pois + i * NF;
			if (!finite(p)) continue;
			if (only >= 0) {
				if (i != only) continue;
			} else if (!strain_good<MODE>(p, zncc_threshold)) continue; // :244-248 / :362-368
			long c[3];
			cell_of(p, c);
			fit.clear();
			long found = 0;
			for (long cz = std::max(0l, c[2] - 1); cz <= std::min(nc[2] - 1, c[2] + 1); cz++)
				for (long cy = std::max(0l, c[1] - 1); cy <= std::min(nc[1] - 1, c[1] + 1); cy++)
					for (long cx = std::max(0l, c[0] - 1); cx <= std::min(nc[0] - 1, c[0] + 1); cx++) {
						long ci = (cz * nc[1] + cy) * nc[0] + cx;
						for (long s = start[ci]; s < start[ci + 1]; s++) {
							long j = order[s];
							const float* q = pois + j * NF;
							float d2 = 0.f; // L2_Simple_Adaptor: float accumulation over the 3 coordinates
							for (int d = 0; d < D; d++) { float df = p[d] - q[d]; d2 += df * df; }
							if (d2 < r2) {
								found++;
								if (strain_good<MODE>(q, zncc_threshold)) fit.push_back(j);
							}
						}
					}
			if (found < k_min) { // KNN fallback :183-196
				fit.clear();
				cand.clear();
				for (long j = 0; j < n; j++) {
					const float* q = pois + j * NF;
					if (!finite(q)) continue;
					float d2 = 0.f;
					for (int d = 0; d < D; d++) { float df = p[d] - q[d]; d2 += df * df; }
					cand.push_back(std::make_pair(d2, j));
				}
				long k = std::min((long)k_min, (long)cand.size());
				std::partial_sort(cand.begin(), cand.begin() + k, cand.end());
				for (long t = 0; t < k; t++)
					if (strain_good<MODE>(pois + cand[t].second * NF, zncc_threshold)) fit.push_back(cand[t].second);
			}
			std::sort(fit.begin(), fit.end());
			const int m = (int)fit.size();
			if (m < k_min) continue; // :200-201
			constexpr int C = FD + 1;
			A.resize((size_t)m * C);
			B.resize((size_t)m * FD);
			for (int t = 0; t < m; t++) {
				const float* q = pois + fit[t] * NF;
				A[(size_t)t * C] = 1;
				for (int d = 0; d < FD; d++) A[(size_t)t * C + 1 + d] = (T)(q[L::FC + d] - p[L::FC + d]);
				B[(size_t)t * FD] = q[L::U];
				B[(size_t)t * FD + 1] = q[L::V];
				if (FD == 3) B[(size_t)t * FD + 2] = q[L::W];
			}
			T x[FD][C];
			lsq_qr<T, C, FD>(A, B, m, x);
			float* e = &out[(size_t)i * NE];
			if (FD == 2) {
				float ux = (float)x[0][1], uy = (float)x[0][2], vx = (float)x[1][1], vy = (float)x[1][2];
				if (approximation == 2) { // Green strain :229-235
					e[0] = ux + 0.5f * (ux * ux + vx * vx);
					e[1] = vy + 0.5f * (uy * uy + vy * vy);
					e[2] = 0.5f * (uy + vx + uy * ux + vy * vx);
				} else { // Cauchy strain :222-227
					e[0] = ux; e[1] = vy; e[2] = 0.5f * (uy + vx);
				}
			} else {
				float ux = (float)x[0][1], uy = (float)x[0][2], uz = (float)x[0][3];
				float vx = (float)x[1][1], vy = (float)x[1][2], vz = (float)x[1][3];
				float wx = (float)x[2 % FD][1], wy = (float)x[2 % FD][2], wz = (float)x[2 % FD][3 % C];
				if (approximation == 2) { // :455-463
					e[0] = ux + 0.5f * (ux * ux + vx * vx + wx * wx);
					e[1] = vy + 0.5f * (uy * uy + vy * vy + wy * wy);
					e[2] = wz + 0.5f * (uz * uz + vz * vz + wz * wz);
					e[3] = 0.5f * (uy + vx + uy * ux + vy * vx + wy * wx);
					e[4] = 0.5f * (vz + wy + uz * uy + vz * vy + wz * wy);
					e[5] = 0.5f * (wx + uz + ux * uz + vx * vz + wx * wz);
				} else { // :444-453
					e[0] = ux; e[1] = vy; e[2] = wz;
					e[3] = 0.5f * (uy + vx); e[4] = 0.5f * (vz + wy); e[5] = 0.5f * (wx + uz);
				}
			}
			done[i] = 1;
		}
	}
	for (long i = 0; i < n; i++)
		if (done[i])
			for (int k = 0; k < NE; k++) pois[i * NF + L::STRAIN + k] = out[(size_t)i * NE + k];
}

// ----------------------------------------------------------------------------------------------
// EpipolarSearch::compute(POI2D*), src/oc_epipolar_search.cpp:133-195: candidate POIs are spawned along the
// epipolar line of the secondary view (centre + every `search_step` pixels in x up to `search_radius`, both
// directions, kept when the subset stays inside the image), ICGN2D1 runs on each, the candidate with the highest
// ZNCC wins (std::sort by ZNCC descending; ties -- unspecified there -- go to the earlier candidate here).
// fundamental: 3x3 row-major (updateFundementalMatrix :110-126); parallax_x/y: the linear parallax model (:74-95).
// ----------------------------------------------------------------------------------------------
struct EpiCandidate { float u, v; };

inline void epipolar_candidates(const Ctx2D& c, const float* poi, const float* F, const float* parallax_x, const float* parallax_y,
	int search_radius, int search_step, int rx, int ry, std::vector<EpiCandidate>& out) {
	out.clear();
	const float px = poi[P2_X], py = poi[P2_Y], pu = poi[P2_DEF + D2_U], pv = poi[P2_DEF + D2_V];
	// :136-137 (int(width / 2) is an integer division)
	const float par_x = parallax_x[0] * (px - (float)(int)(c.w / 2)) + parallax_x[1] * (py - (float)(int)(c.h / 2)) + parallax_x[2];
	const float par_y = parallax_y[0] * (px - (float)(int)(c.w / 2)) + parallax_y[1] * (py - (float)(int)(c.h / 2)) + parallax_y[2];
	const float v1[3] = { px + pu, py + pv, 1.f }; // :140-141
	float e[3];
	for (int i = 0; i < 3; i++) e[i] = (F[i * 3] * v1[0] + F[i * 3 + 1] * v1[1]) + F[i * 3 + 2] * v1[2]; // :144
	const float line_slope = -e[0] / e[1];
	const float line_intercept = -e[2] / e[1];
	const int x_view2 = (int)((line_slope * (py + pv + par_y - line_intercept) + px + pu + par_x) / (line_slope * line_slope + 1)); // :147
	const int y_view2 = (int)(line_slope * x_view2 + line_intercept);
	out.push_back({ (float)x_view2 - px, (float)y_view2 - py }); // :151-155 (centre: no border test)
	for (int i = search_step; i < search_radius; i += search_step) { // :159-182
		for (int sgn = 1; sgn >= -1; sgn -= 2) {
			const int x_trial = x_view2 + sgn * i;
			const int y_trial = (int)(line_slope * x_trial + line_intercept);
			if (x_trial - rx > 0 && x_trial + rx < c.w - 1 && y_trial - ry > 0 && y_trial + ry < c.h - 1)
				out.push_back({ (float)x_trial - px, (float)y_trial - py });
		}
	}
}

template <class T>
void run_epipolar(const Ctx2D& c, float* pois, long n, const float* F, const float* parallax_x, const float* parallax_y, int search_radius,
	int search_step, int rx, int ry, float conv, float stop) {
#pragma omp parallel num_threads(c.threads)
	{
		Scratch2D<T> s;
		std::vector<EpiCandidate> cand;
		float q[P2_N], best[P2_N];
#pragma omp for schedule(dynamic, 4)
		for (long i = 0; i < n; i++) {
			float* poi = pois + i * P2_N;
			epipolar_candidates(c, poi, F, parallax_x, parallax_y, search_radius, search_step, rx, ry, cand);
			bool have = false;
			for (const EpiCandidate& k : cand) {
				for (int j = 0; j < P2_N; j++) q[j] = 0.f; // POI2D current_poi(poi->x, poi->y): everything else cleared (:152)
				q[P2_X] = poi[P2_X];
				q[P2_Y] = poi[P2_Y];
				q[P2_DEF + D2_U] = k.u;
				q[P2_DEF + D2_V] = k.v;
				icgn2d_poi<T, 6>(c, q, rx, ry, conv, stop, s);
				if (!have || q[P2_ZNCC] > best[P2_ZNCC]) {
					for (int j = 0; j < P2_N; j++) best[j] = q[j];
					have = true;
				}
			}
			for (int j = 0; j < 12; j++) poi[P2_DEF + j] = best[P2_DEF + j]; // poi->deformation = ... (:193)
			for (int j = P2_U0; j <= P2_FEAT; j++) poi[j] = best[j];          // poi->result = ... (:194)
		}
	}
}

} // namespace

// ----------------------------------------------------------------------------------------------
// C boundary (ctypes).  All functions are oracle-only (prefix oco_).
// ----------------------------------------------------------------------------------------------
extern "C" {

void* oco_create2d(const float* ref, const float* tar, int height, int width, int threads) {
	Ctx2D* c = new Ctx2D;
	c->h = height; c->w = width; c->threads = threads > 0 ? threads : 1;
	c->ref.assign(ref, ref + (size_t)height * width);
	c->tar.assign(tar, tar + (size_t)height * width);
	return c;
}
void oco_destroy2d(void* h) { delete (Ctx2D*)h; }
// ICGN2D1::prepare / ICGN2D2::prepare (src/oc_icgn.cpp:138-142, :679-683)
void oco_prepare2d(void* h) {
	Ctx2D* c = (Ctx2D*)h;
	gradient2d(*c, c->ref, c->gx, c->gy);
	bicubic_prepare(*c, c->tar, c->lut);
	c->prepared = true;
}
void oco_get_gradient2d(void* h, float* gx, float* gy) {
	Ctx2D* c = (Ctx2D*)h;
	std::memcpy(gx, c->gx.data(), c->gx.size() * sizeof(float));
	std::memcpy(gy, c->gy.data(), c->gy.size() * sizeof(float));
}
void oco_bicubic_eval(void* h, const float* xy, long n, float* out, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	for (long i = 0; i < n; i++)
		out[i] = exact ? (float)bicubic_eval<double>(*c, (double)xy[2 * i], (double)xy[2 * i + 1]) : bicubic_eval<float>(*c, xy[2 * i], xy[2 * i + 1]);
}
void oco_fftcc2d(void* h, float* pois, long n, int rx, int ry, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	if (exact) run_fftcc2d<double>(*c, pois, n, rx, ry); else run_fftcc2d<float>(*c, pois, n, rx, ry);
}
int oco_icgn2d1(void* h, float* pois, long n, int rx, int ry, float conv, float stop, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	if (!c->prepared) return -1;
	if (exact) run_icgn2d<double, 6>(*c, pois, n, rx, ry, conv, stop); else run_icgn2d<float, 6>(*c, pois, n, rx, ry, conv, stop);
	return 0;
}
int oco_icgn2d2(void* h, float* pois, long n, int rx, int ry, float conv, float stop, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	if (!c->prepared) return -1;
	if (exact) run_icgn2d<double, 12>(*c, pois, n, rx, ry, conv, stop); else run_icgn2d<float, 12>(*c, pois, n, rx, ry, conv, stop);
	return 0;
}

// compute(std::vector<POI2D>&, std::vector<Point2D>& center_offset_queue) (src/oc_icgn.cpp:549-557, :1128-1136)
// and the self-adaptive mode; order = 1 (ICGN2D1) or 2 (ICGN2D2); offsets may be NULL.
int oco_icgn2d_ex(void* h, int order, float* pois, long n, int rx, int ry, float conv, float stop, const float* offsets, int self_adaptive, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	if (!c->prepared) return -1;
	if (order == 1) {
		if (exact) run_icgn2d<double, 6>(*c, pois, n, rx, ry, conv, stop, offsets, self_adaptive != 0);
		else run_icgn2d<float, 6>(*c, pois, n, rx, ry, conv, stop, offsets, self_adaptive != 0);
	} else {
		if (exact) run_icgn2d<double, 12>(*c, pois, n, rx, ry, conv, stop, offsets, self_adaptive != 0);
		else run_icgn2d<float, 12>(*c, pois, n, rx, ry, conv, stop, offsets, self_adaptive != 0);
	}
	return 0;
}

// ICLM2D1::compute(queue) src/oc_iclm.cpp:360-368, ICLM2D2::compute(queue) :732-740; damping = {lambda, alpha, beta}
int oco_iclm2d(void* h, int order, float* pois, long n, int rx, int ry, float conv, float stop, const float* damping, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	if (!c->prepared || !damping) return -1;
	if (order == 1) {
		if (exact) run_icgn2d<double, 6>(*c, pois, n, rx, ry, conv, stop, nullptr, false, damping);
		else run_icgn2d<float, 6>(*c, pois, n, rx, ry, conv, stop, nullptr, false, damping);
	} else {
		if (exact) run_icgn2d<double, 12>(*c, pois, n, rx, ry, conv, stop, nullptr, false, damping);
		else run_icgn2d<float, 12>(*c, pois, n, rx, ry, conv, stop, nullptr, false, damping);
	}
	return 0;
}

// NR2D1::prepare (src/oc_nr.cpp:119-156) and NR2D1::compute(queue) (:327-334)
void oco_prepare_nr2d(void* h) {
	Ctx2D* c = (Ctx2D*)h;
	gradient2d(*c, c->tar, c->tgx, c->tgy);
	if (c->lut.empty()) bicubic_prepare(*c, c->tar, c->lut);
	bicubic_prepare(*c, c->tgx, c->lut_tgx);
	bicubic_prepare(*c, c->tgy, c->lut_tgy);
	c->prepared_nr = true;
}
int oco_nr2d1(void* h, float* pois, long n, int rx, int ry, float conv, float stop, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	if (!c->prepared_nr) return -1;
	if (exact) run_nr2d1<double>(*c, pois, n, rx, ry, conv, stop); else run_nr2d1<float>(*c, pois, n, rx, ry, conv, stop);
	return 0;
}

void* oco_create3d(const float* ref, const float* tar, int dim_x, int dim_y, int dim_z, int threads) {
	Ctx3D* c = new Ctx3D;
	c->dx = dim_x; c->dy = dim_y; c->dz = dim_z; c->threads = threads > 0 ? threads : 1;
	size_t total = (size_t)dim_x * dim_y * dim_z;
	c->ref.assign(ref, ref + total);
	c->tar.assign(tar, tar + total);
	return c;
}
void oco_destroy3d(void* h) { delete (Ctx3D*)h; }
// ICGN3D1::prepare (src/oc_icgn.cpp:1264-1268)
void oco_prepare3d(void* h) {
	Ctx3D* c = (Ctx3D*)h;
	gradient3d(*c);
	tricubic_prepare(*c);
	c->prepared = true;
}
void oco_get_gradient3d(void* h, float* gx, float* gy, float* gz) {
	Ctx3D* c = (Ctx3D*)h;
	std::memcpy(gx, c->gx.data(), c->gx.size() * sizeof(float));
	std::memcpy(gy, c->gy.data(), c->gy.size() * sizeof(float));
	std::memcpy(gz, c->gz.data(), c->gz.size() * sizeof(float));
}
void oco_get_coefficient3d(void* h, float* coef) {
	Ctx3D* c = (Ctx3D*)h;
	std::memcpy(coef, c->coef.data(), c->coef.size() * sizeof(float));
}
void oco_tricubic_eval(void* h, const float* xyz, long n, float* out, int exact) {
	Ctx3D* c = (Ctx3D*)h;
	for (long i = 0; i < n; i++)
		out[i] = exact ? (float)tricubic_eval<double>(*c, (double)xyz[3 * i], (double)xyz[3 * i + 1], (double)xyz[3 * i + 2])
			: tricubic_eval<float>(*c, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
}
void oco_fftcc3d(void* h, float* pois, long n, int rx, int ry, int rz, int exact) {
	Ctx3D* c = (Ctx3D*)h;
	if (exact) run_fftcc3d<double>(*c, pois, n, rx, ry, rz); else run_fftcc3d<float>(*c, pois, n, rx, ry, rz);
}
int oco_icgn3d1(void* h, float* pois, long n, int rx, int ry, int rz, float conv, float stop, int exact) {
	Ctx3D* c = (Ctx3D*)h;
	if (!c->prepared) return -1;
	if (exact) run_icgn3d1<double>(*c, pois, n, rx, ry, rz, conv, stop); else run_icgn3d1<float>(*c, pois, n, rx, ry, rz, conv, stop);
	return 0;
}
// EpipolarSearch::compute(queue), src/oc_epipolar_search.cpp:197-205 (needs oco_prepare2d, like prepareICGN :63-67)
int oco_epipolar_search(void* h, float* pois, long n, const float* fundamental, const float* parallax_x, const float* parallax_y, int search_radius,
	int search_step, int rx, int ry, float conv, float stop, int exact) {
	Ctx2D* c = (Ctx2D*)h;
	if (!c->prepared || search_step < 1) return -1;
	if (exact) run_epipolar<double>(*c, pois, n, fundamental, parallax_x, parallax_y, search_radius, search_step, rx, ry, conv, stop);
	else run_epipolar<float>(*c, pois, n, fundamental, parallax_x, parallax_y, search_radius, search_step, rx, ry, conv, stop);
	return 0;
}
// Strain::prepare + Strain::compute(queue) on POI2D (dim 2) / POI3D (dim 3) records, src/oc_strain.cpp:100-111,239-250,476-487.
// approximation: 1 Cauchy, 2 Green (setApproximation); zncc_threshold default 0.9 (:38).  only >= 0: Strain::compute(POI*, queue)
// on that POI alone (-1 when only >= n).
int oco_strain_single(float* pois, long n, int dim, long only, float radius, int min_neighbors, float zncc_threshold, int approximation, int threads,
	int exact) {
	if (dim != 2 && dim != 3 && dim != 23) return -1; // 23: POI2DS records (28 floats), the stereo-DIC variant
	if (only >= n) return -1;
	if (threads < 1) threads = 1;
	if (dim == 2) {
		if (exact) run_strain<double, 2>(pois, n, radius, min_neighbors, zncc_threshold, approximation, threads, only);
		else run_strain<float, 2>(pois, n, radius, min_neighbors, zncc_threshold, approximation, threads, only);
	} else if (dim == 3) {
		if (exact) run_strain<double, 3>(pois, n, radius, min_neighbors, zncc_threshold, approximation, threads, only);
		else run_strain<float, 3>(pois, n, radius, min_neighbors, zncc_threshold, approximation, threads, only);
	} else {
		if (exact) run_strain<double, 23>(pois, n, radius, min_neighbors, zncc_threshold, approximation, threads, only);
		else run_strain<float, 23>(pois, n, radius, min_neighbors, zncc_threshold, approximation, threads, only);
	}
	return 0;
}
int oco_strain(float* pois, long n, int dim, float radius, int min_neighbors, float zncc_threshold, int approximation, int threads, int exact) {
	return oco_strain_single(pois, n, dim, -1, radius, min_neighbors, zncc_threshold, approximation, threads, exact);
}
void oco_set_legacy_no_minus4(int on) { g_legacy_no_m4 = on != 0; }
int oco_max_threads(void) { return omp_get_num_procs(); }

} // extern "C"
