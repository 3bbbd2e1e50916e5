// SIFT3D arithmetic shared by the CUDA kernels (sift3d.cu, compiled with -fmad=false) and the CPU oracle (oracle/oc_sift3d.cpp,
// compiled with -ffp-contract=off): the exponential, the 3x3 symmetric eigen-decomposition, the icosahedron and the blur
// weights.  Every routine here is plain IEEE arithmetic without library calls whose rounding differs between the host's libm
// and CUDA's, so both sides produce the same bits.
#pragma once
#include <float.h>
#include <math.h>

#ifdef __CUDACC__
#define S3_HD __host__ __device__
#else
#define S3_HD
#endif

namespace s3 {

// Sift3dConfig (src/oc_sift.h:71-83) as the float array of the C ABI, in the struct's field order.
enum {
	CFG_N_OCTAVE_LAYERS = 0,
	CFG_N_OCTAVE,
	CFG_MIN_DIMENSION,
	CFG_ALPHA,
	CFG_BETA,
	CFG_GAMMA,
	CFG_SIGMA_SOURCE,
	CFG_SIGMA_BASE,
	CFG_GRADIENT_THRESHOLD,
	CFG_TRUNCATE_THRESHOLD,
	CFG_FIELDS
};
// Keypoint record: coor_layer xyz, coor_img xyz, octave, layer, scale, R[9] (rows q0, q1, q0 x q1).
enum { KP_FLOATS = 18, DESC = 768, IMG_BORDER = 1 };

// exp(x) evaluated in double (Cody-Waite reduction, degree-12 Taylor polynomial) and rounded to float.  Within 1 ulp of libm's
// expf / (float)exp; used for every Gaussian weight of SIFT3D so that host and device agree bit for bit.
S3_HD inline float exp_f(double x) {
	if (x < -104.0) return 0.f;
	if (x > 89.0) return INFINITY;
	const double k = floor(x * 1.4426950408889634 + 0.5);
	const double r = (x - k * 6.93147180369123816490e-01) - k * 1.90821492927058770002e-10;
	double p = 1.0 / 479001600.0;
	p = p * r + 1.0 / 39916800.0;
	p = p * r + 1.0 / 3628800.0;
	p = p * r + 1.0 / 362880.0;
	p = p * r + 1.0 / 40320.0;
	p = p * r + 1.0 / 5040.0;
	p = p * r + 1.0 / 720.0;
	p = p * r + 1.0 / 120.0;
	p = p * r + 1.0 / 24.0;
	p = p * r + 1.0 / 6.0;
	p = p * r + 0.5;
	p = p * r + 1.0;
	p = p * r + 1.0;
	return (float)ldexp(p, (int)k);
}

// Eigen-decomposition of the symmetric 3x3 float matrix m (row-major) by cyclic Jacobi rotations in double.  val: the three
// eigenvalues rounded to float, in descending order (ties keep the column order); vec[3 * i + c]: component c of the unit
// eigenvector of val[i].  This replaces Eigen::EigenSolver<Matrix3f>::pseudoEigenvectors (src/oc_sift.cpp:948-970), whose
// normalisation is not reproduced: the reference treats the vectors as a rotation (it transposes R to invert it).
S3_HD inline void eig3(const float* m, float* val, float* vec) {
	double a[3][3], v[3][3];
	for (int i = 0; i < 3; i++)
		for (int j = 0; j < 3; j++) {
			a[i][j] = (double)m[3 * i + j];
			v[i][j] = i == j ? 1.0 : 0.0;
		}
	for (int sweep = 0; sweep < 64; sweep++) {
		const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
		const double diag = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
		if (off == 0.0 || off <= 1e-36 * diag) break;
		for (int pq = 0; pq < 3; pq++) {
			const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
			if (a[p][q] == 0.0) continue;
			const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
			const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
			const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
			for (int k = 0; k < 3; k++) { // A <- A J
				const double akp = a[k][p], akq = a[k][q];
				a[k][p] = c * akp - s * akq;
				a[k][q] = s * akp + c * akq;
			}
			for (int k = 0; k < 3; k++) { // A <- J^T A
				const double apk = a[p][k], aqk = a[q][k];
				a[p][k] = c * apk - s * aqk;
				a[q][k] = s * apk + c * aqk;
			}
			for (int k = 0; k < 3; k++) { // V <- V J
				const double vkp = v[k][p], vkq = v[k][q];
				v[k][p] = c * vkp - s * vkq;
				v[k][q] = s * vkp + c * vkq;
			}
		}
	}
	float ev[3];
	int order[3] = { 0, 1, 2 };
	for (int i = 0; i < 3; i++) ev[i] = (float)a[i][i];
	for (int i = 1; i < 3; i++) // insertion sort, descending, stable
		for (int j = i; j > 0 && ev[order[j]] > ev[order[j - 1]]; j--) {
			const int t = order[j];
			order[j] = order[j - 1];
			order[j - 1] = t;
		}
	for (int i = 0; i < 3; i++) {
		const int c = order[i];
		const double n = sqrt(v[0][c] * v[0][c] + v[1][c] * v[1][c] + v[2][c] * v[2][c]);
		val[i] = ev[c];
		for (int k = 0; k < 3; k++) vec[3 * i + k] = (float)(v[k][c] / n);
	}
}

// The icosahedron of SIFT3D::prepare (src/oc_sift.cpp:209-232): 12 vertices (as written there, 6 decimals) and 20 faces as
// vertex-id triplets in the reference's face order.  The descriptor bins of a cube are indexed by vertex id.
#define S3_ICO_VERTICES                                                                                                              \
	{ 0.000000f, 0.525731f, 0.850651f, 0.000000f, -0.525731f, 0.850651f, 0.000000f, 0.525731f, -0.850651f, 0.000000f, -0.525731f,      \
		-0.850651f, 0.525731f, 0.850651f, 0.000000f, -0.525731f, 0.850651f, 0.000000f, 0.525731f, -0.850651f, 0.000000f, -0.525731f, \
		-0.850651f, 0.000000f, 0.850651f, 0.000000f, 0.525731f, -0.850651f, 0.000000f, 0.525731f, 0.850651f, 0.000000f, -0.525731f,  \
		-0.850651f, 0.000000f, -0.525731f }
#define S3_ICO_FACES                                                                                                                 \
	{ 1, 0, 8, 8, 0, 4, 4, 0, 5, 5, 0, 9, 9, 0, 1, 6, 1, 8, 6, 8, 10, 10, 8, 4, 10, 4, 2, 2, 4, 5, 2, 5, 11, 11, 5, 9, 11, 9, 7, 7, 9, 1, \
		7, 1, 6, 6, 3, 7, 7, 3, 11, 11, 3, 2, 2, 3, 10, 10, 3, 6 }

// cartisan2Barycentric (src/oc_sift.cpp:579-623): 1 if the ray along g hits the triangle (v0, v1, v2), with its barycentric
// coordinates in b; -1 otherwise.  Same float operations in the same order (Point3D dot / cross products, oc_point.h:186-208).
S3_HD inline int ray_triangle(const float* g, const float* v0, const float* v1, const float* v2, float* b) {
	const float e1[3] = { v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2] };
	const float e2[3] = { v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2] };
	const float t[3] = { -1.f * v0[0], -1.f * v0[1], -1.f * v0[2] };
	const float p[3] = { g[1] * e2[2] - g[2] * e2[1], g[2] * e2[0] - g[0] * e2[2], g[0] * e2[1] - g[1] * e2[0] };
	const float q[3] = { t[1] * e1[2] - t[2] * e1[1], t[2] * e1[0] - t[0] * e1[2], t[0] * e1[1] - t[1] * e1[0] };
	const float det = e1[0] * p[0] + e1[1] * p[1] + e1[2] * p[2];
	if (fabsf(det) < FLT_EPSILON * 10.f) return -1;
	const float inv = 1.f / det;
	const float bz = inv * (g[0] * q[0] + g[1] * q[1] + g[2] * q[2]);
	const float by = inv * (p[0] * t[0] + p[1] * t[1] + p[2] * t[2]);
	const float bx = 1.f - by - bz;
	const float k = inv * (q[0] * e2[0] + q[1] * e2[1] + q[2] * e2[2]);
	if (k < 0) return -1;
	if (bx < -FLT_EPSILON * 10.f || by < -FLT_EPSILON * 10.f || bz < -FLT_EPSILON * 10.f) return -1;
	float r[3];
	for (int c = 0; c < 3; c++) r[c] = k * g[c] - bx * v0[c] - by * v1[c] - bz * v2[c];
	if (sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]) > FLT_EPSILON * 10.f) return -1;
	b[0] = bx;
	b[1] = by;
	b[2] = bz;
	return 1;
}

// First face (in face order) hit by the ray along g, or -1; verts / faces are the two tables above.
S3_HD inline int ico_face(const float* g, const float* verts, const int* faces, float* b) {
	for (int f = 0; f < 20; f++)
		if (ray_triangle(g, verts + 3 * faces[3 * f], verts + 3 * faces[3 * f + 1], verts + 3 * faces[3 * f + 2], b) > 0) return f;
	return -1;
}

// Mirror extension of gaussianBlur (mirrorLow / mirrorHigh, src/oc_sift.cpp:1505-1517) for the taps c - r (lower) and c + r
// (upper) of a line of n voxels.  Where the reference's mirrored index is still outside [0, n) (n not larger than the blur
// radius), it reads out of bounds; here the index is then clamped into the line.
S3_HD inline int mirror_lower(int i, int n) {
	i = i < 0 ? -i : i;
	return i > n - 1 ? n - 1 : i;
}
S3_HD inline int mirror_upper(int i, int n) {
	i = i > n - 1 ? 2 * (n - 1) - i : i;
	return i < 0 ? 0 : i;
}

// Blur radii and weights of gaussianBlur (src/oc_sift.cpp:367-399,438-454,490-506) for one layer: radius[a] per axis, and
// w[a][0..radius[a]] the normalised half kernel.  Host only.  Returns false if a radius exceeds max_radius.
inline bool blur_kernels(float sigma, const float* unit, int max_radius, int* radius, float* w /* 3 * (max_radius + 1) */) {
	float unit_max = unit[0] > unit[1] ? unit[0] : unit[1];
	unit_max = unit_max > unit[2] ? unit_max : unit[2];
	int kernel_radius;
	if (sigma > 0) {
		kernel_radius = (int)(ceilf(3.f * sigma) > 1 ? ceilf(3.f * sigma) : 1);
	} else {
		sigma = 0.f;
		kernel_radius = 1;
	}
	radius[0] = (int)(kernel_radius * floorf(unit_max / unit[0] + 0.5f));
	radius[1] = (int)(kernel_radius * floor(unit_max / unit[1] + 0.5)); // the y axis rounds in double (:439)
	radius[2] = (int)(kernel_radius * floorf(unit_max / unit[2] + 0.5f));
	for (int a = 0; a < 3; a++) {
		if (radius[a] > max_radius || radius[a] < 0) return false;
		float* k = w + a * (max_radius + 1);
		k[0] = 1.f;
		for (int i = 1; i <= radius[a]; i++) {
			const float x = i / (sigma + FLT_EPSILON);
			k[i] = exp_f(-0.5f * x * x);
			k[0] += (k[i] * 2.f);
		}
		k[0] = 1.f / k[0];
		for (int i = 1; i <= radius[a]; i++) k[i] *= k[0];
	}
	return true;
}

// Pyramid geometry of createGaussianPyramid (src/oc_sift.cpp:676-739): the octave count, kappa, and per layer of an octave the
// scale and the sigma of its blur.  scale[o * L + i] for every octave o and layer i (L = n_octave_layers + 3).
inline int octave_count(int dim_min, int min_dimension) {
	int n = (int)floor(log2((float)dim_min) - log2((float)min_dimension)) + 1;
	return n > 0 ? n : 1;
}
inline float kappa_of(int n_octave_layers) { return powf(2.f, 1.f / n_octave_layers); }

} // namespace s3
