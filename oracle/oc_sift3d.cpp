// CPU oracle of SIFT3D (reference src/oc_sift.cpp:140-1519): TEST INFRASTRUCTURE ONLY, like oc_oracle.cpp.
//
// A float32 restatement of the reference's feature extraction and monodirectional matching, compiled with -ffp-contract=off
// so that every product and sum is rounded on its own, as written.  The pyramid is built one octave at a time (the layers of
// one octave are all that detection, orientation and description need); the arithmetic is the reference's.
//
// Where the reference is undefined or cannot be reproduced here, this file defines it, and the CUDA kernels follow:
//   - exp: every Gaussian weight uses s3::exp_f (double evaluation rounded to float, within 1 ulp of libm's expf);
//     pow(x, 2.f) of the orientation weight (:902) is x * x.
//   - Eigen::EigenSolver (:948-950) is replaced by s3::eig3 (Jacobi in double, unit eigenvectors).
//   - A mirrored blur index that is still out of range (:424-536, when a line is not longer than the blur radius) is clamped
//     into the line, and only the voxels of the line are written (the reference's border loops can run past its end).
//   - y_max of the orientation window multiplies by the unit where the other bounds divide (:870): reproduced.
//   - Matching post-pass (:1306-1390): kp_matches[j + 1] is read one past the resized end (:1335), where the stale element is a
//     row that failed the ratio test (tar_idx -1), so a many-to-one run that ends the list is closed like the others: here
//     every maximal run, the last one included.  std::sort (not stable) orders runs of equal tar_idx; here both sorts are stable, so a run keeps the descending ref_idx order of the first sort.  If every
//     reference keypoint passes the ratio test, matched_amount stays 0 and nothing is returned (:1309-1317): reproduced.
//
// Besides the reference's products, the oracle reports float64 margins of the decisions a rounding difference could flip:
// per candidate the orientation tests (gradient threshold, the two beta ratios, the gamma cosine) and per reference keypoint
// the ratio test, each as the relative distance of the float64 value from its threshold.
#include <omp.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../opencorr_b200/csrc/sift3d_common.h"

namespace {

struct Vol {
	std::vector<float> v;
	int d[3] = { 0, 0, 0 }; // x, y, z
	float at(int z, int y, int x) const { return v[((size_t)z * d[1] + y) * d[0] + x]; }
	size_t n() const { return (size_t)d[0] * d[1] * d[2]; }
};

const float kIcoV[36] = S3_ICO_VERTICES;
const int kIcoF[60] = S3_ICO_FACES;

struct Cfg {
	int n_octave_layers, n_octave, min_dimension;
	float alpha, beta, gamma, sigma_source, sigma_base, gradient_threshold, truncate_threshold;
};

Cfg read_cfg(const float* c) {
	Cfg g;
	g.n_octave_layers = (int)c[s3::CFG_N_OCTAVE_LAYERS];
	g.n_octave = (int)c[s3::CFG_N_OCTAVE];
	g.min_dimension = (int)c[s3::CFG_MIN_DIMENSION];
	g.alpha = c[s3::CFG_ALPHA];
	g.beta = c[s3::CFG_BETA];
	g.gamma = c[s3::CFG_GAMMA];
	g.sigma_source = c[s3::CFG_SIGMA_SOURCE];
	g.sigma_base = c[s3::CFG_SIGMA_BASE];
	g.gradient_threshold = c[s3::CFG_GRADIENT_THRESHOLD];
	g.truncate_threshold = c[s3::CFG_TRUNCATE_THRESHOLD];
	return g;
}

// gaussianBlur (:365-547): x into dst, y into a buffer, z into dst; each output acc = k0 * s[c]; acc += k_r * (s[lo] + s[hi]).
void blur(const Vol& src, Vol& dst, const float* unit, float sigma) {
	const int R = 64;
	int rad[3];
	std::vector<float> w(3 * (R + 1));
	s3::blur_kernels(sigma, unit, R, rad, w.data());
	const int nx = src.d[0], ny = src.d[1], nz = src.d[2];
	dst.d[0] = nx, dst.d[1] = ny, dst.d[2] = nz;
	dst.v.assign(src.n(), 0.f);
	std::vector<float> buf(src.n());
	const float* kx = &w[0];
	const float* ky = &w[R + 1];
	const float* kz = &w[2 * (R + 1)];
#pragma omp parallel for
	for (int i = 0; i < nz; i++)
		for (int j = 0; j < ny; j++) {
			const float* s = &src.v[((size_t)i * ny + j) * nx];
			float* o = &dst.v[((size_t)i * ny + j) * nx];
			for (int k = 0; k < nx; k++) {
				float acc = kx[0] * s[k];
				for (int r = 1; r <= rad[0]; r++) acc += kx[r] * (s[s3::mirror_lower(k - r, nx)] + s[s3::mirror_upper(k + r, nx)]);
				o[k] = acc;
			}
		}
#pragma omp parallel for
	for (int i = 0; i < nz; i++)
		for (int k = 0; k < nx; k++)
			for (int j = 0; j < ny; j++) {
				const float* s = &dst.v[(size_t)i * ny * nx + k];
				float acc = ky[0] * s[(size_t)j * nx];
				for (int r = 1; r <= rad[1]; r++)
					acc += ky[r] * (s[(size_t)s3::mirror_lower(j - r, ny) * nx] + s[(size_t)s3::mirror_upper(j + r, ny) * nx]);
				buf[((size_t)i * ny + j) * nx + k] = acc;
			}
	const size_t plane = (size_t)nx * ny;
#pragma omp parallel for
	for (int j = 0; j < ny; j++)
		for (int k = 0; k < nx; k++)
			for (int i = 0; i < nz; i++) {
				const float* s = &buf[(size_t)j * nx + k];
				float acc = kz[0] * s[i * plane];
				for (int r = 1; r <= rad[2]; r++) acc += kz[r] * (s[s3::mirror_lower(i - r, nz) * plane] + s[s3::mirror_upper(i + r, nz) * plane]);
				dst.v[i * plane + (size_t)j * nx + k] = acc;
			}
}

struct Kp {
	float cl[3], ci[3];
	int octave, layer;
	float scale;
	float R[9];
};

// float32 gradient of the reference (:905-907, :1131-1133): 0.5 * (difference) in double, divided by the unit in double.
inline float grad(float hi, float lo, float unit) { return (float)(0.5 * (double)(hi - lo) / (double)unit); }

// assignOrientation (:849-1049) for one candidate on Gaussian layer g.  Returns true if kept (R filled); margin = the float64
// relative distance of the decisive quantities from their thresholds (smallest of the tests evaluated).
bool orient(const Vol& g, const float* unit, const Cfg& cfg, Kp& kp, double* margin) {
	const float sigma_w = 1.5f * kp.scale;
	const float window_radius = 3.f * sigma_w;
	const int B = s3::IMG_BORDER;
	int x_min = (int)floorf(kp.cl[0] - window_radius / unit[0]);
	x_min = x_min > B ? x_min : B;
	int x_max = (int)ceilf(kp.cl[0] + window_radius / unit[0]);
	x_max = x_max < g.d[0] - B ? x_max : g.d[0] - B;
	int y_min = (int)floorf(kp.cl[1] - window_radius / unit[1]);
	y_min = y_min > B ? y_min : B;
	int y_max = (int)ceilf(kp.cl[1] + window_radius * unit[1]); // sic (:870)
	y_max = y_max < g.d[1] - B ? y_max : g.d[1] - B;
	int z_min = (int)floorf(kp.cl[2] - window_radius / unit[2]);
	z_min = z_min > B ? z_min : B;
	int z_max = (int)ceilf(kp.cl[2] + window_radius / unit[2]);
	z_max = z_max < g.d[2] - B ? z_max : g.d[2] - B;

	float dx = 0.f, dy = 0.f, dz = 0.f;
	float st[9] = { 0.f };
	double dd[3] = { 0.0, 0.0, 0.0 };
	for (int i = z_min; i < z_max; i++)
		for (int j = y_min; j < y_max; j++)
			for (int k = x_min; k < x_max; k++) {
				const float px = ((float)k - kp.cl[0]) * unit[0];
				const float py = ((float)j - kp.cl[1]) * unit[1];
				const float pz = ((float)i - kp.cl[2]) * unit[2];
				const float dist = sqrtf(px * px + py * py + pz * pz);
				if (dist <= window_radius) {
					const float r = dist / sigma_w;
					const float w = s3::exp_f(-0.5f * (r * r));
					const float gx = grad(g.at(i, j, k + 1), g.at(i, j, k - 1), unit[0]);
					const float gy = grad(g.at(i, j + 1, k), g.at(i, j - 1, k), unit[1]);
					const float gz = grad(g.at(i + 1, j, k), g.at(i - 1, j, k), unit[2]);
					st[0] += gx * gx * w;
					st[1] += gx * gy * w;
					st[2] += gx * gz * w;
					st[4] += gy * gy * w;
					st[5] += gy * gz * w;
					st[8] += gz * gz * w;
					dx += gx * w;
					dy += gy * w;
					dz += gz * w;
					dd[0] += (double)gx * w;
					dd[1] += (double)gy * w;
					dd[2] += (double)gz * w;
				}
			}
	st[3] = st[1];
	st[6] = st[2];
	st[7] = st[5];

	const double dn2 = dd[0] * dd[0] + dd[1] * dd[1] + dd[2] * dd[2];
	double m = fabs(dn2 - cfg.gradient_threshold) / std::max(fabs((double)cfg.gradient_threshold), 1e-300);
	*margin = m;
	if ((dx * dx + dy * dy + dz * dz) < cfg.gradient_threshold) return false;

	float ev[3], evec[9];
	s3::eig3(st, ev, evec);
	{ // beta tests: the eigenvalue ratios in double (the eigenvalues come from the float tensor, as the decision does)
		const double r1 = (double)ev[1] / (double)ev[0], r2 = (double)ev[2] / (double)ev[1];
		m = std::min(m, std::min(fabs(r1 - cfg.beta), fabs(r2 - cfg.beta)) / cfg.beta);
		*margin = m;
	}
	if ((ev[1] / ev[0]) > cfg.beta || (ev[2] / ev[1]) > cfg.beta || fabsf(ev[0] - ev[1]) < FLT_EPSILON || fabsf(ev[1] - ev[2]) < FLT_EPSILON
		|| fabsf(ev[2] - ev[0]) < FLT_EPSILON)
		return false;

	const float d[3] = { dx, dy, dz };
	const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
	float cos_phi = FLT_MAX;
	double cos64 = 1e300;
	for (int e = 0; e < 2; e++) {
		float* q = evec + 3 * e;
		const float qd = q[0] * d[0] + q[1] * d[1] + q[2] * d[2];
		const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
		const float c = fabsf(qd / (qn * dnorm));
		cos_phi = cos_phi < c ? cos_phi : c;
		const double qd64 = (double)q[0] * dd[0] + (double)q[1] * dd[1] + (double)q[2] * dd[2];
		cos64 = std::min(cos64, fabs(qd64 / sqrt(dn2)));
		const float sgn = qd > 0 ? 1.f : -1.f;
		q[0] *= sgn;
		q[1] *= sgn;
		q[2] *= sgn;
	}
	*margin = std::min(m, fabs(cos64 - cfg.gamma) / cfg.gamma);
	if (cos_phi < cfg.gamma) return false;

	const float* r1 = evec;
	const float* r2 = evec + 3;
	const float rc[3] = { r1[1] * r2[2] - r1[2] * r2[1], r1[2] * r2[0] - r1[0] * r2[2], r1[0] * r2[1] - r1[1] * r2[0] };
	for (int c = 0; c < 3; c++) {
		kp.R[c] = r1[c];
		kp.R[3 + c] = r2[c];
		kp.R[6 + c] = rc[c];
	}
	return true;
}

// constructDescriptor (:1051-1249) for one keypoint on Gaussian layer g; out: 768 floats.
void describe(const Vol& g, const float* unit, const Cfg& cfg, const Kp& kp, float* out) {
	const float sqrt_2 = sqrtf(2.f);
	const float sigma = 5.f * sqrt_2 * kp.scale;
	const float sphere_radius = 2.f * sigma;
	const float cube_radius = sphere_radius / sqrt_2;
	const int B = s3::IMG_BORDER;
	int x_min = (int)floorf(kp.cl[0] - sphere_radius / unit[0]);
	x_min = x_min > B ? x_min : B;
	int x_max = (int)ceilf(kp.cl[0] + sphere_radius / unit[0]);
	x_max = x_max < g.d[0] - B ? x_max : g.d[0] - B;
	int y_min = (int)floorf(kp.cl[1] - sphere_radius / unit[1]);
	y_min = y_min > B ? y_min : B;
	int y_max = (int)ceilf(kp.cl[1] + sphere_radius / unit[1]);
	y_max = y_max < g.d[1] - B ? y_max : g.d[1] - B;
	int z_min = (int)floorf(kp.cl[2] - sphere_radius / unit[2]);
	z_min = z_min > B ? z_min : B;
	int z_max = (int)ceilf(kp.cl[2] + sphere_radius / unit[2]);
	z_max = z_max < g.d[2] - B ? z_max : g.d[2] - B;

	for (int b = 0; b < s3::DESC; b++) out[b] = 0.f;
	const float* R = kp.R;
	for (int i = z_min; i < z_max; i++)
		for (int j = y_min; j < y_max; j++)
			for (int k = x_min; k < x_max; k++) {
				float p[3] = { (float)k - kp.cl[0], (float)j - kp.cl[1], (float)i - kp.cl[2] };
				p[0] *= unit[0];
				p[1] *= unit[1];
				p[2] *= unit[2];
				const float dist = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
				if (dist > sphere_radius) continue;
				float sub[3];
				for (int a = 0; a < 3; a++) {
					const float rot = R[3 * a] * p[0] + R[3 * a + 1] * p[1] + R[3 * a + 2] * p[2];
					sub[a] = 2.f * (rot + cube_radius) / cube_radius;
					sub[a] -= 0.5f;
				}
				if (sub[0] <= -0.5f || sub[1] <= -0.5f || sub[2] <= -0.5f || sub[0] >= 3.5f || sub[1] >= 3.5f || sub[2] >= 3.5f) continue;
				const double t = (double)(dist / sigma);
				const float w = s3::exp_f(-0.5 * (t * t));
				float gr[3] = { grad(g.at(i, j, k + 1), g.at(i, j, k - 1), unit[0]), grad(g.at(i, j + 1, k), g.at(i, j - 1, k), unit[1]),
					grad(g.at(i + 1, j, k), g.at(i - 1, j, k), unit[2]) };
				gr[0] = w * gr[0];
				gr[1] = w * gr[1];
				gr[2] = w * gr[2];
				float rg[3];
				for (int a = 0; a < 3; a++) rg[a] = R[3 * a] * gr[0] + R[3 * a + 1] * gr[1] + R[3 * a + 2] * gr[2];
				const float gm = sqrtf(rg[0] * rg[0] + rg[1] * rg[1] + rg[2] * rg[2]);
				if (gm * gm < FLT_EPSILON * 10.f) continue;
				float bary[3];
				const int f = s3::ico_face(rg, kIcoV, kIcoF, bary);
				if (f < 0) continue;
				const float dec[3] = { sub[0] - floorf(sub[0]), sub[1] - floorf(sub[1]), sub[2] - floorf(sub[2]) };
				for (int dz = 0; dz < 2; dz++)
					for (int dy = 0; dy < 2; dy++)
						for (int dx = 0; dx < 2; dx++) {
							const int lx = (int)sub[0] + dx, ly = (int)sub[1] + dy, lz = (int)sub[2] + dz;
							if (lx < 0 || ly < 0 || lz < 0 || lx >= 4 || ly >= 4 || lz >= 4) continue;
							const int cube = lx + ly * 4 + lz * 16;
							const float iw = ((dx == 0) ? (1.f - dec[0]) : dec[0]) * ((dy == 0) ? (1.f - dec[1]) : dec[1])
								* ((dz == 0) ? (1.f - dec[2]) : dec[2]);
							for (int v = 0; v < 3; v++) out[cube * 12 + kIcoF[3 * f + v]] += gm * iw * bary[v];
						}
			}
	for (int pass = 0; pass < 2; pass++) {
		float sq = 0;
		for (int b = 0; b < s3::DESC; b++) sq += out[b] * out[b];
		const float inv = 1.f / (sqrtf(sq) + FLT_EPSILON);
		for (int b = 0; b < s3::DESC; b++) out[b] *= inv;
		if (pass == 0)
			for (int b = 0; b < s3::DESC; b++) out[b] = (out[b] < cfg.truncate_threshold) ? out[b] : cfg.truncate_threshold;
	}
}

struct Result {
	int n_octave = 0;
	std::vector<int> cand;      // 5 ints per candidate: octave, layer, z, y, x
	std::vector<float> max_abs; // per DoG layer, octave-major
	std::vector<float> kp;      // s3::KP_FLOATS per kept keypoint
	std::vector<float> desc;    // 768 per kept keypoint
	std::vector<double> margin; // per candidate
	std::vector<int> kept;      // per candidate
};

void extract(const float* img, int dx, int dy, int dz, Cfg& cfg, const float* unit0, Result& out) {
	int dim_min = dx < dy ? dx : dy;
	dim_min = dim_min < dz ? dim_min : dz;
	cfg.n_octave = s3::octave_count(dim_min, cfg.min_dimension);
	out.n_octave = cfg.n_octave;
	const int nol = cfg.n_octave_layers, L = nol + 3;
	const float kappa = s3::kappa_of(nol);
	// scales of every layer (:705-729)
	std::vector<float> scale((size_t)cfg.n_octave * L), sigma((size_t)cfg.n_octave * L, 0.f);
	scale[0] = 1.f / kappa * cfg.sigma_base;
	sigma[0] = sqrtf(scale[0] * scale[0] - cfg.sigma_source * cfg.sigma_source);
	for (int i = 1; i < cfg.n_octave * L; i++) {
		const int octave = i / L, lio = i % L;
		if (lio == 0) {
			scale[i] = scale[(octave - 1) * L + nol];
		} else {
			scale[i] = kappa * scale[i - 1];
			sigma[i] = sqrtf(kappa * kappa - 1.f) * scale[lio - 1];
		}
	}
	Vol input;
	input.d[0] = dx, input.d[1] = dy, input.d[2] = dz;
	input.v.assign(img, img + input.n());
	float unit[3] = { unit0[0], unit0[1], unit0[2] };
	std::vector<Vol> G(L);
	for (int o = 0; o < cfg.n_octave; o++) {
		if (o == 0) {
			blur(input, G[0], unit, sigma[0]);
		} else { // downSampling (:549-562) of layer i - 3 = layer nol of the previous octave
			Vol down;
			const Vol& s = G[nol];
			for (int a = 0; a < 3; a++) {
				down.d[a] = s.d[a] / 2;
				unit[a] *= 2;
			}
			down.v.resize(down.n());
			for (int i = 0; i < down.d[2]; i++)
				for (int j = 0; j < down.d[1]; j++)
					for (int k = 0; k < down.d[0]; k++) down.v[((size_t)i * down.d[1] + j) * down.d[0] + k] = s.at(2 * i, 2 * j, 2 * k);
			G[0] = std::move(down);
		}
		for (int l = 1; l < L; l++) blur(G[l - 1], G[l], unit, sigma[o * L + l]);
		// DoG (:756-793)
		std::vector<Vol> D(L - 1);
		for (int n = 0; n < L - 1; n++) {
			D[n].d[0] = G[n].d[0], D[n].d[1] = G[n].d[1], D[n].d[2] = G[n].d[2];
			D[n].v.resize(G[n].n());
			float mx = -1.f;
			for (size_t v = 0; v < D[n].n(); v++) {
				D[n].v[v] = G[n + 1].v[v] - G[n].v[v];
				const float a = fabsf(D[n].v[v]);
				mx = mx < a ? a : mx;
			}
			out.max_abs.push_back(mx);
		}
		// detectExtrema (:795-847)
		std::vector<Kp> cands;
		for (int n = 1; n < nol + 1; n++) {
			const Vol& c = D[n];
			const float thr = cfg.alpha * out.max_abs[(size_t)o * (L - 1) + n];
			for (int i = 1; i < c.d[2] - 1; i++)
				for (int j = 1; j < c.d[1] - 1; j++)
					for (int k = 1; k < c.d[0] - 1; k++) {
						const float v = c.at(i, j, k);
						if (!(fabsf(v) >= thr)) continue;
						const float nb[8] = { c.at(i - 1, j, k), c.at(i + 1, j, k), c.at(i, j - 1, k), c.at(i, j + 1, k), c.at(i, j, k - 1), c.at(i, j, k + 1),
							D[n - 1].at(i, j, k), D[n + 1].at(i, j, k) };
						bool gt = true, lt = true;
						for (int e = 0; e < 8; e++) {
							gt = gt && v > nb[e];
							lt = lt && v < nb[e];
						}
						if (gt || lt) {
							Kp kp;
							kp.cl[0] = (float)k, kp.cl[1] = (float)j, kp.cl[2] = (float)i;
							kp.layer = n;
							kp.octave = o;
							kp.scale = scale[o * L + n];
							cands.push_back(kp);
							const int rec[5] = { o, n, i, j, k };
							out.cand.insert(out.cand.end(), rec, rec + 5);
						}
					}
		}
		// assignOrientation, then constructDescriptor for the survivors (candidate order kept)
		const int nc = (int)cands.size();
		std::vector<int> keep(nc);
		std::vector<double> margin(nc);
#pragma omp parallel for schedule(dynamic, 4)
		for (int m = 0; m < nc; m++) keep[m] = orient(G[cands[m].layer], unit, cfg, cands[m], &margin[m]) ? 1 : 0;
		std::vector<Kp> kept;
		for (int m = 0; m < nc; m++) {
			out.margin.push_back(margin[m]);
			out.kept.push_back(keep[m]);
			if (!keep[m]) continue;
			Kp kp = cands[m];
			const float f = powf(2.f, (float)kp.octave);
			for (int a = 0; a < 3; a++) kp.ci[a] = kp.cl[a] * f;
			kept.push_back(kp);
		}
		const size_t base = out.desc.size();
		out.desc.resize(base + kept.size() * s3::DESC);
#pragma omp parallel for schedule(dynamic, 1)
		for (int m = 0; m < (int)kept.size(); m++) describe(G[kept[m].layer], unit, cfg, kept[m], &out.desc[base + (size_t)m * s3::DESC]);
		for (const Kp& kp : kept) {
			const float rec[s3::KP_FLOATS] = { kp.cl[0], kp.cl[1], kp.cl[2], kp.ci[0], kp.ci[1], kp.ci[2], (float)kp.octave, (float)kp.layer, kp.scale,
				kp.R[0], kp.R[1], kp.R[2], kp.R[3], kp.R[4], kp.R[5], kp.R[6], kp.R[7], kp.R[8] };
			out.kp.insert(out.kp.end(), rec, rec + s3::KP_FLOATS);
		}
	}
}

} // namespace

extern "C" {

int os3_max_threads() { return omp_get_max_threads(); }

// SIFT3D feature extraction of one volume [z][y][x].  config: CFG_FIELDS floats (Sift3dConfig order; n_octave is computed).
void* os3_extract(const float* vol, int dx, int dy, int dz, const float* config, const float* unit, int threads) {
	if (threads > 0) omp_set_num_threads(threads);
	Result* r = new Result;
	Cfg cfg = read_cfg(config);
	extract(vol, dx, dy, dz, cfg, unit, *r);
	return r;
}

// counts: n_octave, candidates, max_abs entries, kept keypoints
void os3_counts(void* h, long* counts) {
	const Result* r = (const Result*)h;
	counts[0] = r->n_octave;
	counts[1] = (long)r->cand.size() / 5;
	counts[2] = (long)r->max_abs.size();
	counts[3] = (long)r->kp.size() / s3::KP_FLOATS;
}

void os3_get(void* h, int* cand, float* max_abs, float* kp, float* desc, double* margin, int* kept) {
	const Result* r = (const Result*)h;
	if (cand) memcpy(cand, r->cand.data(), r->cand.size() * sizeof(int));
	if (max_abs) memcpy(max_abs, r->max_abs.data(), r->max_abs.size() * sizeof(float));
	if (kp) memcpy(kp, r->kp.data(), r->kp.size() * sizeof(float));
	if (desc) memcpy(desc, r->desc.data(), r->desc.size() * sizeof(float));
	if (margin) memcpy(margin, r->margin.data(), r->margin.size() * sizeof(double));
	if (kept) memcpy(kept, r->kept.data(), r->kept.size() * sizeof(int));
}

void os3_free(void* h) { delete (Result*)h; }

// monodirectionalMatch (:1251-1418).  top2: n1 x 3 (d0, index0, d1) of the brute-force scan; ratio_margin: n1 float64 relative
// margins |d0 - ratio^2 d1| / d1.  pairs: up to n1 (ref index, tar index) in output order; returns their number.
long os3_match(const float* d1, long n1, const float* d2, long n2, float ratio, int threads, float* top2, double* ratio_margin, int* pairs) {
	if (threads > 0) omp_set_num_threads(threads);
	const float r2 = ratio * ratio;
	struct M {
		int ref_idx, tar_idx;
		float dist;
	};
	std::vector<M> km(n1, M{ -1, -1, 0.f });
#pragma omp parallel for schedule(dynamic, 16)
	for (long i = 0; i < n1; i++) {
		int ci[2] = { -1, -1 };
		float cd[2] = { FLT_MAX, FLT_MAX };
		for (long j = 0; j < n2; j++) {
			float sq = 0;
			for (int k = 0; k < s3::DESC; k++) {
				const float diff = d1[i * s3::DESC + k] - d2[j * s3::DESC + k];
				sq += diff * diff;
			}
			if (sq < cd[0]) {
				ci[1] = ci[0];
				cd[1] = cd[0];
				ci[0] = (int)j;
				cd[0] = sq;
			} else if (sq < cd[1]) {
				ci[1] = (int)j;
				cd[1] = sq;
			}
		}
		if (top2) {
			top2[3 * i] = cd[0];
			top2[3 * i + 1] = (float)ci[0];
			top2[3 * i + 2] = cd[1];
		}
		if (ratio_margin) ratio_margin[i] = fabs((double)cd[0] - (double)r2 * (double)cd[1]) / (double)cd[1];
		if (cd[0] < r2 * cd[1]) km[i] = M{ (int)i, ci[0], cd[0] };
	}
	std::stable_sort(km.begin(), km.end(), [](const M& a, const M& b) { return a.ref_idx > b.ref_idx; });
	long matched = 0;
	for (long i = 0; i < n1; i++)
		if (km[i].ref_idx == -1) {
			matched = i;
			break;
		}
	if (matched > 1) {
		km.resize(matched);
		std::stable_sort(km.begin(), km.end(), [](const M& a, const M& b) { return a.tar_idx > b.tar_idx; });
		for (long s = 0; s < matched;) { // each maximal run of equal tar_idx
			long e = s + 1;
			while (e < matched && km[e].tar_idx == km[s].tar_idx) e++;
			if (e - s > 1) {
				int ci[2] = { -1, -1 };
				float cd[2] = { FLT_MAX, FLT_MAX };
				for (long c = s; c < e; c++) {
					if (km[c].dist < cd[0]) {
						ci[1] = ci[0];
						cd[1] = cd[0];
						ci[0] = km[c].ref_idx;
						cd[0] = km[c].dist;
					} else if (km[c].dist < cd[1]) {
						ci[1] = km[c].ref_idx;
						cd[1] = km[c].dist;
					}
					km[c].ref_idx = -1;
				}
				if (cd[0] < r2 * cd[1]) km[s].ref_idx = ci[0];
			}
			s = e;
		}
	}
	long n = 0;
	for (long i = 0; i < matched; i++)
		if (km[i].ref_idx > -1) {
			pairs[2 * n] = km[i].ref_idx;
			pairs[2 * n + 1] = km[i].tar_idx;
			n++;
		}
	return n;
}

// Building blocks, for the unit tests.
void os3_blur(const float* src, float* dst, int dx, int dy, int dz, const float* unit, float sigma) {
	Vol s, d;
	s.d[0] = dx, s.d[1] = dy, s.d[2] = dz;
	s.v.assign(src, src + s.n());
	blur(s, d, unit, sigma);
	memcpy(dst, d.v.data(), d.n() * sizeof(float));
}

void os3_blur_kernel(float sigma, const float* unit, int* radius, float* w /* 3 x 65 */) { s3::blur_kernels(sigma, unit, 64, radius, w); }

void os3_eig3(const float* m, float* val, float* vec) { s3::eig3(m, val, vec); }

int os3_ico_face(const float* g, float* bary) { return s3::ico_face(g, kIcoV, kIcoF, bary); }

float os3_exp(float x) { return s3::exp_f(x); }

} // extern "C"
