// nr2d.cu -- forward-additive Newton-Raphson subset registration, 2D, first-order shape function
// (6 parameters), for sm_90a.  Replaces NR2D1::compute(POI2D*) (reference src/oc_nr.cpp:160-325)
// including what NR2D1::prepare() feeds it (:119-156): Gradient2D4 of the TARGET image and three
// BicubicBspline tables (target, d/dx target, d/dy target) -- none of which is built here: the
// gradients are recomputed per POI from the staged target tile and all three interpolants are
// evaluated from 4x4 pixel blocks with explicit fp32 weights.
//
// Mapping (same skeleton as icgn2d.cu): ONE WARP PER POI, persistent warps pulling POIs from an atomic
// counter; lanes run along x, so x-dependent factors are per-lane constants.
//   stage   : reference subset -> smem as r~ = r - mean(r); target tile (subset + bicubic support +
//             2-pixel gradient halo + slack) -> smem by TMA; gradient tile {gx, gy} of the target
//             computed once from the tile (zero on the image's 2-pixel border, src/oc_gradient.cpp:42,46).
//   iterate : every iteration samples t, tx, ty at the warped positions (one set of weights, three
//             4x4 blocks), and accumulates ONE pass of factored sums:
//               sum g_a g_b y^Q (Hessian, x^P applied per lane afterwards), sum g_a y^Q, sum g_a r~ y^Q,
//               sum g_a t' y^Q, sum t', sum t'^2, sum r~ t'            (t' = t - c0, c0 a pilot value)
//             from which mean/norm of the warped target, ZNSSD, the 6x6 Hessian and the right-hand side
//             sum sd (r~ |t|/|r| - t~) follow algebraically.  Cholesky solve, p <- p + dp.
// Out-of-range samples take the interpolant's -1 for all three maps, as in the reference (no rejection).
// Samples whose support leaves the staged tile are evaluated from global memory.

#include "ocb_kernels.h"
#include "ocb_tile2d.cuh"
#include "ocb_tma.cuh"

namespace ocb {

// tile extents, the per-warp slab (nr2d_tar_w .. nr2d_warp_floats) and the launch plan are in ocb_kernels.h

// gradient pixel of the target at global (x, y), from global memory (slow path only)
__device__ __forceinline__ float2 nr_grad_global(const float* __restrict__ tar, int w, int h, int x, int y) {
	float2 g = make_float2(0.f, 0.f);
	const float* q = tar + (size_t)y * w + x;
	if (x >= 2 && x < w - 2) g.x = grad4(__ldg(q - 2), __ldg(q - 1), __ldg(q + 1), __ldg(q + 2));
	if (y >= 2 && y < h - 2) g.y = grad4(__ldg(q - 2 * (size_t)w), __ldg(q - w), __ldg(q + w), __ldg(q + 2 * (size_t)w));
	return g;
}

// SERIES: one reference against n_frames targets (img.tar is the frame-major stack [n_frames][h][w], tm_tar a 3D map over it).
// A POI's reference subset r~ is staged, with its mean and norm, once, at the first frame that passes the guard, and stays in the
// warp's slab; each frame then runs the same guard, target staging, gradient tile, iterations and result code as a pair call,
// seeded by the previous frame's record, which stays in registers.  Every frame's record is stored whole to
// frames_out[f n_poi + poi]; `pois` holds the seeds and is only read.
template <bool SERIES>
__device__ __forceinline__ void nr2d1_poi_loop(Image2D img, float* __restrict__ pois, float* __restrict__ frames_out, int n_frames, int n_poi,
	int rx, int ry, float conv_criterion, float stop_condition, int* __restrict__ work_counter, const CUtensorMap& tm_tar, int use_tma) {
	extern __shared__ __align__(128) float smem[];
	const int lane = threadIdx.x & 31;
	const int warp = threadIdx.x >> 5;
	const int sw = 2 * rx + 1, sh = 2 * ry + 1, N = sw * sh;
	const int ncol = sw < 32 ? sw : 32;
	const int rem = sw - ncol;
	const int ntail = rem * sh;
	const int TW = nr2d_tar_w(rx), TH = nr2d_tar_h(ry);
	const int GW = TW - 4, GH = TH - 4;
	float* slab = smem + (size_t)warp * nr2d_warp_floats(rx, ry);
	float* T = slab + 32;
	float2* G = (float2*)(T + round_up32(TW * TH));
	float* sR = (float*)G + round_up32(2 * GW * GH);
	TileLoad tile = { (uint64_t*)slab, 0, use_tma };
	tile.init(lane == 0, [] { __syncwarp(); });
	const float* __restrict__ ref = img.ref;
	const int w = img.w, h = img.h;
	const float inv_n = 1.0f / (float)N;
	const bool lane_on = lane < ncol;
	const int lane_c = lane_on ? lane : ncol - 1;
	const float xl_lane = (float)(lane - rx);

	while (true) {
		int poi = 0;
		if (lane == 0) poi = atomicAdd(work_counter, 1);
		poi = __shfl_sync(0xffffffffu, poi, 0);
		if (poi >= n_poi) break;
		float* P = pois + (size_t)poi * P2_N; // SERIES: the seed, then frame f's record
		float rec = lane < P2_N ? P[lane] : 0.f; // lane k holds field k of the record
		auto put = [&](int field, float value) { if (lane == field) rec = value; };
		// src/oc_nr.cpp:314-324, run for every POI: -4 when the iterations ran out unconverged, -5 (and u, v restored) on a NaN;
		// then the whole record goes out as one coalesced store, fields nothing changed with the bits they were read with
		auto finish = [&](float z, float conv, float iter, float u, float v, float u_back, float v_back) {
			if (conv >= conv_criterion && iter >= stop_condition) z = -4.f;
			if (is_nan_f(z) || is_nan_f(u) || is_nan_f(v)) {
				put(P2_DEF + D2_U, u_back);
				put(P2_DEF + D2_V, v_back);
				z = -5.f;
			}
			put(P2_ZNCC, z);
			if (lane < P2_N) P[lane] = rec;
		};
		const float px = __shfl_sync(0xffffffffu, rec, P2_X);
		const float py = __shfl_sync(0xffffffffu, rec, P2_Y);
		// the reference subset's statistics; SERIES: kept for every frame of the POI
		bool set_up = false;
		float rs, ref_norm;
		for (int f = 0; f < (SERIES ? n_frames : 1); f++) {
			if constexpr (SERIES) P = frames_out + ((size_t)f * n_poi + poi) * P2_N;
			const float* __restrict__ tar = SERIES ? img.tar + (size_t)f * w * h : img.tar;
			const float u_in = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_U);
			const float v_in = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_V);
			const float zncc_in = __shfl_sync(0xffffffffu, rec, P2_ZNCC);
			const float iter_in = __shfl_sync(0xffffffffu, rec, P2_ITER);
			const float conv_in = __shfl_sync(0xffffffffu, rec, P2_CONV);
			const float u0_in = __shfl_sync(0xffffffffu, rec, P2_U0);
			const float v0_in = __shfl_sync(0xffffffffu, rec, P2_V0);
			// guard: NR2D1 writes -1 (not -3), then the -4 / -5 tests
			if (subset2d_guard_fails(px, py, rx, ry, w, h, u_in, v_in, zncc_in)) {
				finish(zncc_in < -1.f ? zncc_in : -1.f, conv_in, iter_in, u_in, v_in, u0_in, v0_in);
				continue;
			}
			__syncwarp();

			// ---------------- stage the target tile (TMA) and the reference subset ----------------
			const int tx0 = floor4((int)floorf(px + u_in) - rx - 1 - NR2D_TILE_MARGIN - 2);
			const int ty0 = (int)floorf(py + v_in) - ry - 1 - NR2D_TILE_MARGIN - 2;
			tile.issue<SERIES>(T, &tm_tar, tar, w, h, tx0, ty0, f, TW, TH, lane == 0, true, lane);
			if (!SERIES || !set_up) {
				set_up = true;
				const int x0 = (int)(px - rx), y0 = (int)(py - ry); // Subset2D::fill upper-left
				float r1 = 0.f;
				for (int c = lane; c < sw; c += 32) {
#pragma unroll 4
					for (int r = 0; r < sh; r++) {
						const float v = __ldg(ref + (size_t)(y0 + r) * w + x0 + c);
						sR[r * sw + c] = v;
						r1 += v;
					}
				}
				r1 = warp_sum(r1);
				const float rmean = r1 * inv_n; // Subset2D::zeroMeanNorm, src/oc_subset.cpp:46-53
				float r2 = 0.f, r1t = 0.f;
				for (int c = lane; c < sw; c += 32) {
#pragma unroll 4
					for (int r = 0; r < sh; r++) {
						const float v = sR[r * sw + c] - rmean;
						sR[r * sw + c] = v;
						r2 = fmaf(v, v, r2);
						r1t += v;
					}
				}
				r2 = warp_sum(r2);
				rs = warp_sum(r1t); // sum r~ (zero up to rounding)
				ref_norm = sqrtf(r2);
			}
			tile.wait([] {});
			__syncwarp(); // the staged tile and sR are visible to the whole warp
			// gradient tile of the target: G(c, r) <-> T(c + 2, r + 2)
			for (int c = lane; c < GW; c += 32) {
				const int xg = tx0 + 2 + c;
				const bool gx_ok = xg >= 2 && xg < w - 2;
				for (int r = 0; r < GH; r++) {
					const int yg = ty0 + 2 + r;
					const float* q = T + (r + 2) * TW + c + 2;
					float2 g = make_float2(0.f, 0.f);
					if (gx_ok && yg >= 0 && yg < h) g.x = grad4(q[-2], q[-1], q[1], q[2]);
					if (yg >= 2 && yg < h - 2 && xg >= 0 && xg < w) g.y = grad4(q[-2 * TW], q[-TW], q[TW], q[2 * TW]);
					G[r * GW + c] = g;
				}
			}
			__syncwarp();
			const float c0 = T[(TH / 2) * TW + TW / 2]; // pilot value
			// fast samples: valid (src/oc_cubic_bspline.cpp:137-142) and 4x4 support inside the gradient tile
			const int gx0 = tx0 + 2, gy0 = ty0 + 2;
			const float xlo = fmaxf(1.f, (float)(gx0 + 1)), xhi = fminf((float)(w - 2), (float)(gx0 + GW - 2));
			const float ylo = fmaxf(1.f, (float)(gy0 + 1)), yhi = fminf((float)(h - 2), (float)(gy0 + GH - 2));
			const float xmax = (float)(w - 2), ymax = (float)(h - 2);

			float p[6];
			p[0] = u_in;
			p[1] = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_UX);
			p[2] = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_UY);
			p[3] = v_in;
			p[4] = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_VX);
			p[5] = __shfl_sync(0xffffffffu, rec, P2_DEF + D2_VY);
			int iteration = 0;
			float dp_norm = 0.f, zncc = 0.f;
			do {
				iteration++;
				// warp matrix of the current p (Deformation2D1::setWarp, src/oc_deformation.cpp:117-128)
				const float A0 = 1.f + p[1], A1 = p[2], A2 = p[0], A3 = p[4], A4 = 1.f + p[5], A5 = p[3];
				float hA[3][3], sA[2][2], rA[2][2], tA[2][2];
#pragma unroll
				for (int a = 0; a < 3; a++)
#pragma unroll
					for (int q = 0; q < 3; q++) hA[a][q] = 0.f;
#pragma unroll
				for (int a = 0; a < 2; a++)
#pragma unroll
					for (int q = 0; q < 2; q++) { sA[a][q] = 0.f; rA[a][q] = 0.f; tA[a][q] = 0.f; }
				float t1 = 0.f, t2 = 0.f, rt = 0.f;

				// one sample: t' = t - c0, gradient (gx, gy) of the target at (X, Y)
				auto sample = [&](float X, float Y, float& tv, float& gxv, float& gyv) {
					const bool fast = (X >= xlo) && (X < xhi) && (Y >= ylo) && (Y < yhi);
					const bool ok = fast || ((X >= 1.f) && (Y >= 1.f) && (X < xmax) && (Y < ymax)); // NaN fails
					if (!ok) { // BicubicBspline::compute returns -1 for all three tables
						tv = -1.f - c0; gxv = -1.f; gyv = -1.f;
						return;
					}
					const float xf = floorf(X), yf = floorf(Y);
					float wx[4], wy[4];
					bicubic_weights(X - xf, wx);
					bicubic_weights(Y - yf, wy);
					const int ix = (int)xf - 1, iy = (int)yf - 1;
					float t, gx = 0.f, gy = 0.f;
					if (fast) {
						const float* q = T + (iy - ty0) * TW + (ix - tx0);
						const float2* g = G + (iy - gy0) * GW + (ix - gx0);
						t = bicubic_fold(wx, wy, [&](int n, int m) { return q[n * TW + m]; });
						gx = bicubic_fold(wx, wy, [&](int n, int m) { return g[n * GW + m].x; });
						gy = bicubic_fold(wx, wy, [&](int n, int m) { return g[n * GW + m].y; });
					} else {
						const float* q = tar + (size_t)iy * w + ix;
						t = bicubic_fold(wx, wy, [&](int n, int m) { return __ldg(q + (size_t)n * w + m); });
#pragma unroll 1
						for (int nn = 0; nn < 4; nn++) {
							float rgx = 0.f, rgy = 0.f;
#pragma unroll
							for (int mm = 0; mm < 4; mm++) {
								const float2 gg = nr_grad_global(tar, w, h, ix + mm, iy + nn);
								rgx = fmaf(gg.x, wx[mm], rgx);
								rgy = fmaf(gg.y, wx[mm], rgy);
							}
							gx = fmaf(rgx, wy[nn], gx);
							gy = fmaf(rgy, wy[nn], gy);
						}
					}
					tv = t - c0; gxv = gx; gyv = gy;
				};

				{
					// the warped offset is formed first and the POI centre added last (`center + warped`, src/oc_nr.cpp:203)
					const float xl = (float)(lane_c - rx);
					const float xs0 = fmaf(A0, xl, A2), ys0 = fmaf(A3, xl, A5);
					float yl = (float)(-ry);
					const float* pr = sR + lane_c;
					for (int r = 0; r < sh; r++) {
						const float X = px + fmaf(A1, yl, xs0);
						const float Y = py + fmaf(A4, yl, ys0);
						float tv, gx, gy;
						sample(X, Y, tv, gx, gy);
						if (lane_on) {
							const float R = pr[0];
							t1 += tv;
							t2 = fmaf(tv, tv, t2);
							rt = fmaf(R, tv, rt);
							const float gg[3] = { gx * gx, gx * gy, gy * gy };
#pragma unroll
							for (int a = 0; a < 3; a++) {
								hA[a][0] += gg[a];
								hA[a][1] = fmaf(gg[a], yl, hA[a][1]);
								hA[a][2] = fmaf(gg[a] * yl, yl, hA[a][2]);
							}
							const float g1[2] = { gx, gy };
#pragma unroll
							for (int a = 0; a < 2; a++) {
								sA[a][0] += g1[a];
								sA[a][1] = fmaf(g1[a], yl, sA[a][1]);
								rA[a][0] = fmaf(g1[a], R, rA[a][0]);
								rA[a][1] = fmaf(g1[a] * R, yl, rA[a][1]);
								tA[a][0] = fmaf(g1[a], tv, tA[a][0]);
								tA[a][1] = fmaf(g1[a] * tv, yl, tA[a][1]);
							}
						}
						pr += sw;
						yl += 1.f;
					}
				}
				// expand with this lane's x powers.  Monomials x^P y^Q, P + Q <= 2, index m(P,Q) = (P+Q)(P+Q+1)/2 + Q
				float Hm[3][6], S[2][3], SR[2][3], ST[2][3];
				{
					const float x1 = xl_lane, x2 = xl_lane * xl_lane;
#pragma unroll
					for (int a = 0; a < 3; a++) {
						Hm[a][0] = hA[a][0];       // 1
						Hm[a][1] = x1 * hA[a][0];  // x
						Hm[a][2] = hA[a][1];       // y
						Hm[a][3] = x2 * hA[a][0];  // x^2
						Hm[a][4] = x1 * hA[a][1];  // x y
						Hm[a][5] = hA[a][2];       // y^2
					}
#pragma unroll
					for (int a = 0; a < 2; a++) {
						S[a][0] = sA[a][0]; S[a][1] = x1 * sA[a][0]; S[a][2] = sA[a][1];
						SR[a][0] = rA[a][0]; SR[a][1] = x1 * rA[a][0]; SR[a][2] = rA[a][1];
						ST[a][0] = tA[a][0]; ST[a][1] = x1 * tA[a][0]; ST[a][2] = tA[a][1];
					}
				}
				// tail columns (>= 32)
				for (int idx = lane; idx < ntail; idx += 32) {
					const int r = idx / rem, c = 32 + (idx - r * rem);
					const float xl = (float)(c - rx), yl = (float)(r - ry);
					const float X = px + fmaf(A0, xl, fmaf(A1, yl, A2));
					const float Y = py + fmaf(A3, xl, fmaf(A4, yl, A5));
					float tv, gx, gy;
					sample(X, Y, tv, gx, gy);
					const float R = sR[r * sw + c];
					t1 += tv;
					t2 = fmaf(tv, tv, t2);
					rt = fmaf(R, tv, rt);
					const float mono[6] = { 1.f, xl, yl, xl * xl, xl * yl, yl * yl };
					const float gg[3] = { gx * gx, gx * gy, gy * gy };
#pragma unroll
					for (int a = 0; a < 3; a++)
#pragma unroll
						for (int m = 0; m < 6; m++) Hm[a][m] = fmaf(gg[a], mono[m], Hm[a][m]);
					const float g1[2] = { gx, gy };
#pragma unroll
					for (int a = 0; a < 2; a++)
#pragma unroll
						for (int m = 0; m < 3; m++) {
							S[a][m] = fmaf(g1[a], mono[m], S[a][m]);
							SR[a][m] = fmaf(g1[a] * R, mono[m], SR[a][m]);
							ST[a][m] = fmaf(g1[a] * tv, mono[m], ST[a][m]);
						}
				}
				t1 = warp_sum(t1);
				t2 = warp_sum(t2);
				rt = warp_sum(rt);
#pragma unroll
				for (int a = 0; a < 3; a++)
#pragma unroll
					for (int m = 0; m < 6; m++) Hm[a][m] = warp_sum(Hm[a][m]);
#pragma unroll
				for (int a = 0; a < 2; a++)
#pragma unroll
					for (int m = 0; m < 3; m++) { S[a][m] = warp_sum(S[a][m]); SR[a][m] = warp_sum(SR[a][m]); ST[a][m] = warp_sum(ST[a][m]); }

				// warped-target statistics (Subset2D::zeroMeanNorm on the target subset, src/oc_nr.cpp:210)
				const float tbar = t1 * inv_n;
				const float tn2 = t2 - t1 * tbar;
				const float tar_norm = sqrtf(tn2);
				const float rtt = rt - tbar * rs; // sum r~ t~
				zncc = rtt / (ref_norm * tar_norm); // 0.5 * (2 - znssd), znssd = sum (r~ a - t~)^2 / |t|^2, a = |t|/|r| (:244-247)
				const float a = tar_norm / ref_norm;
				// H = sum sd sd^T (:213-238), phi = [1, x, y]: phi_i phi_j -> monomial index
				float H[21], b[6], dp[6];
#pragma unroll
				for (int k = 0; k < 6; k++) {
					const int ka = k / 3, ki = k % 3;
					b[k] = a * SR[ka][ki] - (ST[ka][ki] - tbar * S[ka][ki]); // sum sd_k (a r~ - t~), :250-261
#pragma unroll
					for (int l = 0; l <= k; l++) {
						const int la = l / 3, li = l % 3;
						const int Pp = (ki == 1) + (li == 1), Q = (ki == 2) + (li == 2);
						H[k * (k + 1) / 2 + l] = Hm[ka + la][(Pp + Q) * (Pp + Q + 1) / 2 + Q];
					}
				}
				cholesky_packed<6>(H);
				cholesky_solve<6>(H, b, dp);
#pragma unroll
				for (int k = 0; k < 6; k++) p[k] += dp[k]; // :276-278
				const float rx2 = (float)(rx * rx), ry2 = (float)(ry * ry);
				dp_norm = dp[0] * dp[0] + dp[1] * dp[1] * rx2 + dp[2] * dp[2] * ry2 + dp[3] * dp[3] + dp[4] * dp[4] * rx2 + dp[5] * dp[5] * ry2;
				dp_norm = sqrtf(dp_norm);
			} while ((float)iteration < stop_condition && dp_norm >= conv_criterion);

			// ---------------- results, src/oc_nr.cpp:294-324; SERIES: rec is the next frame's seed ----------------
			put(P2_DEF + D2_U, p[0]); put(P2_DEF + D2_UX, p[1]); put(P2_DEF + D2_UY, p[2]);
			put(P2_DEF + D2_V, p[3]); put(P2_DEF + D2_VX, p[4]); put(P2_DEF + D2_VY, p[5]);
			put(P2_U0, u_in);
			put(P2_V0, v_in);
			put(P2_ITER, (float)iteration);
			put(P2_CONV, dp_norm);
			finish(zncc, dp_norm, (float)iteration, p[0], p[3], u_in, v_in);
			__syncwarp();
		}
	}
}

__global__ void __launch_bounds__(128) nr2d1_kernel(Image2D img, float* __restrict__ pois, int n_poi, int rx, int ry, float conv_criterion,
	float stop_condition, int* __restrict__ work_counter, const __grid_constant__ CUtensorMap tm_tar, int use_tma) {
	nr2d1_poi_loop<false>(img, pois, nullptr, 1, n_poi, rx, ry, conv_criterion, stop_condition, work_counter, tm_tar, use_tma);
}

// img.tar: the frame-major target stack; tm_tars: its 3D map (box depth 1)
__global__ void __launch_bounds__(128) nr2d1_series_kernel(Image2D img, const float* __restrict__ seeds, float* __restrict__ out, int n_frames,
	int n_poi, int rx, int ry, float conv_criterion, float stop_condition, int* __restrict__ work_counter,
	const __grid_constant__ CUtensorMap tm_tars, int use_tma) {
	nr2d1_poi_loop<true>(img, const_cast<float*>(seeds), out, n_frames, n_poi, rx, ry, conv_criterion, stop_condition, work_counter, tm_tars,
		use_tma);
}

// persistent CTAs: as many as are resident, never more than the POIs need
static int nr2d1_grid(const Nr2dPlan& p, size_t n, int sm_count) {
	long long blocks_needed = ((long long)n + p.warps_per_cta - 1) / p.warps_per_cta;
	long long resident = (long long)sm_count * p.ctas_per_sm;
	int grid = (int)(blocks_needed < resident ? blocks_needed : resident);
	if (grid < 1) grid = 1;
	return grid;
}

cudaError_t nr2d1_launch(const Nr2dPlan& p, const Image2D& img, float* d_pois, size_t n, int rx, int ry, float conv, float stop, int sm_count,
	int* d_counter, cudaStream_t stream) {
	CUtensorMap tm_tar{};
	const int use_tma = tma_enabled() && tma_image_map(&tm_tar, img.tar, img.w, img.h, 0, nr2d_tar_w(rx), nr2d_tar_h(ry));
	const cudaError_t e = cudaMemsetAsync(d_counter, 0, sizeof(int), stream);
	if (e != cudaSuccess) return e;
	return launch_smem(nr2d1_kernel, nr2d1_grid(p, n, sm_count), p.warps_per_cta * 32, p.smem, stream, img, d_pois, (int)n, rx, ry, conv, stop,
		d_counter, tm_tar, use_tma);
}

cudaError_t nr2d1_series_launch(const Nr2dPlan& p, const Image2D& img, int n_frames, const float* d_seeds, float* d_out, size_t n, int rx, int ry,
	float conv, float stop, int sm_count, int* d_counter, cudaStream_t stream) {
	CUtensorMap tm_tars{};
	const int use_tma = tma_enabled() && tma_image_map(&tm_tars, img.tar, img.w, img.h, n_frames, nr2d_tar_w(rx), nr2d_tar_h(ry));
	const cudaError_t e = cudaMemsetAsync(d_counter, 0, sizeof(int), stream);
	if (e != cudaSuccess) return e;
	return launch_smem(nr2d1_series_kernel, nr2d1_grid(p, n, sm_count), p.warps_per_cta * 32, p.smem, stream, img, d_seeds, d_out, n_frames,
		(int)n, rx, ry, conv, stop, d_counter, tm_tars, use_tma);
}

} // namespace ocb
