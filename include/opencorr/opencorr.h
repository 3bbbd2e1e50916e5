/*
 * opencorr.h -- API-compatible C++ shim for the FFT-CC -> IC-GN path of OpenCorr, running on the
 * H100 engine behind include/opencorr_b200.h.  Header-only; link with -lopencorr_b200.
 *
 * It re-declares (same names, same signatures, same public members, same POI record layout) the
 * part of the reference's `namespace opencorr` that examples/test_2d_dic_fftcc_icgn1.cpp and
 * examples/test_dvc_fftcc_icgn1.cpp use, so that those two programs compile and run UNCHANGED:
 *     Point2D / Point3D (+ operators)            reference src/oc_point.h:25-210
 *     POI2D / POI3D and their unions             src/oc_poi.h:25-222
 *     Image2D / Image3D                          src/oc_image.h:28-65 (file loading: 8-bit BMP, .bin)
 *     DIC / DVC bases                            src/oc_dic.h:43-84
 *     FFTCC2D / FFTCC3D                          src/oc_fftcc.h:56-90
 *     ICGN2D1 / ICGN2D2 / ICGN3D1                src/oc_icgn.h:45-181
 *     IO2D / IO3D (setters + the 4 writers used) src/oc_io.h:25-149, src/oc_io.cpp:318-504,1004-1089
 *     Calibration / Stereovision                 src/oc_calibration.h:47-98, src/oc_stereovision.cpp:21-133
 * Nothing else of OpenCorr is provided (see DESIGN.md "out of scope").  No Eigen / OpenCV / FFTW.
 *
 * Error behaviour follows the reference: per-POI failures are sentinel ZNCC codes (src/oc_dic.h:28-34),
 * per-call failures throw std::string (src/oc_icgn.cpp:65, src/oc_image.cpp:43).
 */
#pragma once
#ifndef _OPENCORR_B200_SHIM_H_
#define _OPENCORR_B200_SHIM_H_

#include <algorithm>
#include <atomic>
#if __cplusplus >= 201703L
#include <charconv>
#endif
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <iterator>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../opencorr_b200.h"

namespace opencorr
{
	// ------------------------------------------------------------------ src/oc_point.h
	class Point2D
	{
	public:
		float x, y;
		inline Point2D() { x = 0.f; y = 0.f; }
		inline Point2D(float x, float y) { this->x = x; this->y = y; }
		inline Point2D(int x, int y) { this->x = (float)x; this->y = (float)y; }
		inline ~Point2D() {}
		inline float vectorNorm() const { return std::sqrt(x * x + y * y); }
		inline friend std::ostream& operator<<(std::ostream& output, const Point2D& point)
		{
			output << point.x << "," << point.y;
			return output;
		}
	};
	inline Point2D operator+(Point2D point, Point2D offset) { return Point2D(point.x + offset.x, point.y + offset.y); }
	inline Point2D operator-(Point2D point, Point2D offset) { return point + Point2D(-offset.x, -offset.y); }
	inline Point2D operator*(float factor, Point2D point) { return Point2D(factor * point.x, factor * point.y); }
	inline Point2D operator*(int factor, Point2D point) { return float(factor) * point; }
	inline Point2D operator*(Point2D point, float factor) { return factor * point; }
	inline Point2D operator*(Point2D point, int factor) { return float(factor) * point; }
	inline float operator*(Point2D point1, Point2D point2) { return (point1.x * point2.x + point1.y * point2.y); }
	inline Point2D operator/(Point2D point, float factor) { return Point2D(point.x / factor, point.y / factor); }
	inline Point2D operator/(Point2D point, int factor) { return point / float(factor); }
	inline float operator/(Point2D point1, Point2D point2) { return (point1.x * point2.y - point1.y * point2.x); }

	class Point3D
	{
	public:
		float x, y, z;
		inline Point3D() { x = 0.f; y = 0.f; z = 0.f; }
		inline Point3D(float x, float y, float z) { this->x = x; this->y = y; this->z = z; }
		inline Point3D(int x, int y, int z) { this->x = (float)x; this->y = (float)y; this->z = (float)z; }
		inline ~Point3D() {}
		inline float vectorNorm() const { return std::sqrt(x * x + y * y + z * z); }
		inline friend std::ostream& operator<<(std::ostream& output, const Point3D& point)
		{
			output << point.x << "," << point.y << "," << point.z;
			return output;
		}
	};
	inline Point3D operator+(Point3D point, Point3D offset) { return Point3D(point.x + offset.x, point.y + offset.y, point.z + offset.z); }
	inline Point3D operator-(Point3D point, Point3D offset) { return point + Point3D(-offset.x, -offset.y, -offset.z); }
	inline Point3D operator*(float factor, Point3D point) { return Point3D(factor * point.x, factor * point.y, factor * point.z); }
	inline Point3D operator*(int factor, Point3D point) { return float(factor) * point; }
	inline Point3D operator*(Point3D point, float factor) { return factor * point; }
	inline Point3D operator*(Point3D point, int factor) { return float(factor) * point; }
	inline float operator*(Point3D point1, Point3D point2) { return (point1.x * point2.x + point1.y * point2.y + point1.z * point2.z); }
	inline Point3D operator/(Point3D point, float factor) { return Point3D(point.x / factor, point.y / factor, point.z / factor); }
	inline Point3D operator/(Point3D point, int factor) { return point / float(factor); }
	inline Point3D operator/(Point3D point1, Point3D point2)
	{
		return Point3D((point1.y * point2.z - point1.z * point2.y), (point1.z * point2.x - point1.x * point2.z), (point1.x * point2.y - point1.y * point2.x));
	}

	// ------------------------------------------------------------------ src/oc_poi.h (wire format of the boundary)
	union DeformationVector2D
	{
		struct { float u, ux, uy, uxx, uxy, uyy; float v, vx, vy, vxx, vxy, vyy; };
		float p[12];
	};
	union StrainVector2D
	{
		struct { float exx, eyy, exy; };
		float e[3];
	};
	union Result2D
	{
		struct { float u0, v0, zncc, iteration, convergence, feature; };
		float r[6];
	};
	union DeformationVector3D
	{
		struct { float u, ux, uy, uz; float v, vx, vy, vz; float w, wx, wy, wz; };
		float p[12];
	};
	union StrainVector3D
	{
		struct { float exx, eyy, ezz; float exy, eyz, ezx; };
		float e[6];
	};
	union Result3D
	{
		struct { float u0, v0, w0, zncc, iteration, convergence, feature; };
		float r[7];
	};

	union DisplacementVector3D
	{
		struct { float u, v, w; };
		float p[3];
	};
	union Result2DS
	{
		struct { float r1r2_zncc, r1t1_zncc, r1t2_zncc, r2_x, r2_y, t1_x, t1_y, t2_x, t2_y; };
		float r[9];
	};

	class POI2D : public Point2D
	{
	public:
		DeformationVector2D deformation;
		Result2D result;
		StrainVector2D strain;
		Point2D subset_radius;
		inline POI2D(int x, int y) : Point2D(x, y) { clear(); }
		inline POI2D(float x, float y) : Point2D(x, y) { clear(); }
		inline POI2D(Point2D location) : Point2D(location) { clear(); }
		inline ~POI2D() {}
		inline void clear()
		{
			std::fill(std::begin(deformation.p), std::end(deformation.p), 0.f);
			std::fill(std::begin(result.r), std::end(result.r), 0.f);
			std::fill(std::begin(strain.e), std::end(strain.e), 0.f);
			subset_radius.x = 0.f;
			subset_radius.y = 0.f;
		}
	};

	class POI3D : public Point3D
	{
	public:
		DeformationVector3D deformation;
		Result3D result;
		StrainVector3D strain;
		Point3D subset_radius;
		inline POI3D(int x, int y, int z) : Point3D(x, y, z) { clear(); }
		inline POI3D(float x, float y, float z) : Point3D(x, y, z) { clear(); }
		inline POI3D(Point3D location) : Point3D(location) { clear(); }
		inline ~POI3D() {}
		inline void clear()
		{
			std::fill(std::begin(deformation.p), std::end(deformation.p), 0.f);
			std::fill(std::begin(result.r), std::end(result.r), 0.f);
			std::fill(std::begin(strain.e), std::end(strain.e), 0.f);
			subset_radius.x = 0.f;
			subset_radius.y = 0.f;
			subset_radius.z = 0.f;
		}
	};
	// stereo / 3D DIC record (src/oc_poi.h:140-186)
	class POI2DS : public Point2D
	{
	public:
		DisplacementVector3D deformation;
		Result2DS result;
		Point3D ref_coor, tar_coor;
		StrainVector3D strain;
		Point2D subset_radius;
		inline POI2DS(int x, int y) : Point2D(x, y) { clear(); }
		inline POI2DS(float x, float y) : Point2D(x, y) { clear(); }
		inline POI2DS(Point2D location) : Point2D(location) { clear(); }
		inline ~POI2DS() {}
		inline void clear()
		{
			std::fill(std::begin(deformation.p), std::end(deformation.p), 0.f);
			std::fill(std::begin(result.r), std::end(result.r), 0.f);
			ref_coor = Point3D();
			tar_coor = Point3D();
			std::fill(std::begin(strain.e), std::end(strain.e), 0.f);
			subset_radius.x = 0.f;
			subset_radius.y = 0.f;
		}
	};
	static_assert(sizeof(POI2DS) == OCB_POI2DS_FLOATS * sizeof(float), "POI2DS must be the 112-byte record of the C ABI");
	static_assert(sizeof(POI2D) == OCB_POI2D_FLOATS * sizeof(float), "POI2D must be the 100-byte record of the C ABI");
	static_assert(sizeof(POI3D) == OCB_POI3D_FLOATS * sizeof(float), "POI3D must be the 124-byte record of the C ABI");
	static_assert(sizeof(Point2D) == 2 * sizeof(float), "Point2D must be two packed floats (centre-offset queues cross the C ABI verbatim)");

	// ------------------------------------------------------------------ src/oc_image.h
	// Row-major float matrix standing in for the reference's Eigen::MatrixXf member `eg_mat`.
	namespace b200
	{
		// Page-locked memory from the engine's device context, or nullptr without a usable GPU (defined with Engine below).
		// The first call waits for the context that warmEngineAsync() started.
		inline void* pinnedAlloc(size_t bytes);

		// Pixel storage of Image2D / Image3D: page-locked host memory (ocb_host_alloc) when a CUDA device is present, so that
		// every upload of the image runs as asynchronous DMA at the PCIe rate instead of being staged through the driver's
		// bounce buffers (about 5x slower for a 2048 x 2048 pair); ordinary memory on a machine without a GPU (loading and
		// saving images must work there).  Zero-initialised like the reference's containers.
		class PixelBuffer
		{
			float* p = nullptr;
			size_t n = 0;
			bool pinned = false;

		public:
			PixelBuffer() = default;
			PixelBuffer(const PixelBuffer& o) { *this = o; }
			PixelBuffer& operator=(const PixelBuffer& o)
			{
				if (this != &o) {
					assign(o.n, 0.f);
					if (o.n) std::memcpy(p, o.p, o.n * sizeof(float));
				}
				return *this;
			}
			~PixelBuffer() { release(); }
			static float* allocate(size_t count, bool& pinned_out)
			{
				float* q = count ? (float*)pinnedAlloc(count * sizeof(float)) : nullptr;
				pinned_out = q != nullptr;
				if (!q && count) q = (float*)std::malloc(count * sizeof(float));
				if (!q && count) throw std::string("opencorr_b200: out of host memory");
				return q;
			}
			static void deallocate(float* q, bool was_pinned)
			{
				if (!q) return;
				if (was_pinned) ocb_host_free(q);
				else std::free(q);
			}
			void release()
			{
				deallocate(p, pinned);
				p = nullptr;
				n = 0;
			}
			void assign(size_t count, float value)
			{
				if (count != n) {
					release();
					p = allocate(count, pinned);
					n = count;
				}
				if (value == 0.f) { if (n) std::memset(p, 0, n * sizeof(float)); }
				else std::fill(p, p + n, value);
			}
			float* data() { return p; }
			const float* data() const { return p; }
			size_t size() const { return n; }
			float& operator[](size_t i) { return p[i]; }
			float operator[](size_t i) const { return p[i]; }
		};
	} // namespace b200

	class MatrixXf
	{
	public:
		int n_rows = 0, n_cols = 0;
		b200::PixelBuffer data; // row-major [rows][cols]
		inline void resize(int rows, int cols) { n_rows = rows; n_cols = cols; data.assign((size_t)rows * cols, 0.f); }
		inline float& operator()(int r, int c) { return data[(size_t)r * n_cols + c]; }
		inline float operator()(int r, int c) const { return data[(size_t)r * n_cols + c]; }
		inline int rows() const { return n_rows; }
		inline int cols() const { return n_cols; }
	};

	namespace b200
	{
		// Every load / allocation of an image gets a process-wide unique id, so that a new Image2D that happens to sit at
		// the address of a destroyed one is never mistaken for it by the engine's "already on the device?" test.
		inline unsigned long long nextGeneration()
		{
			static std::atomic<unsigned long long> counter{ 0 };
			return ++counter;
		}
		// Starts creating the GPU context on a background thread (defined with Engine below): called from the image
		// constructors, i.e. as early as an OpenCorr program can tell that it is going to correlate something, so that driver
		// and context start-up overlap the image decoding and the POI set-up instead of landing in the first compute().
		inline void warmEngineAsync();

		// Baseline TIFF reader (no OpenCV here): classic TIFF (not BigTIFF), grayscale, 8 or 16 bits per sample (16-bit is scaled
		// to 8 bits like cv::IMREAD_GRAYSCALE), strips, uncompressed or PackBits, any number of pages.  Returns one 8-bit
		// plane per page, all of the first page's size.
		inline std::vector<std::vector<unsigned char>> readTiffPages(const std::string& file_path, int& width, int& height)
		{
			std::ifstream in(file_path, std::ios::in | std::ios::binary);
			if (!in.is_open()) throw std::string("Fail to load tiff: " + file_path);
			std::vector<unsigned char> buf((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
			if (buf.size() < 8) throw std::string("Not a TIFF file: " + file_path);
			const bool le = buf[0] == 'I' && buf[1] == 'I';
			if (!le && !(buf[0] == 'M' && buf[1] == 'M')) throw std::string("Not a TIFF file: " + file_path);
			auto rd16 = [&](size_t o) -> uint32_t {
				if (o + 2 > buf.size()) throw std::string("Truncated TIFF: " + file_path);
				return le ? (uint32_t)buf[o] | ((uint32_t)buf[o + 1] << 8) : (uint32_t)buf[o + 1] | ((uint32_t)buf[o] << 8);
			};
			auto rd32 = [&](size_t o) -> uint32_t {
				if (o + 4 > buf.size()) throw std::string("Truncated TIFF: " + file_path);
				return le ? (uint32_t)buf[o] | ((uint32_t)buf[o + 1] << 8) | ((uint32_t)buf[o + 2] << 16) | ((uint32_t)buf[o + 3] << 24)
						  : (uint32_t)buf[o + 3] | ((uint32_t)buf[o + 2] << 8) | ((uint32_t)buf[o + 1] << 16) | ((uint32_t)buf[o] << 24);
			};
			if (rd16(2) != 42) throw std::string("Unsupported TIFF flavour (BigTIFF?): " + file_path);
			struct Page { uint32_t w = 0, h = 0, bits = 8, comp = 1, photo = 1, spp = 1, rps = 0xffffffffu; std::vector<uint32_t> off, cnt; };
			std::vector<Page> pages;
			uint32_t ifd = rd32(4);
			while (ifd != 0) {
				Page pg;
				const uint32_t n = rd16(ifd);
				for (uint32_t e = 0; e < n; e++) {
					const size_t o = (size_t)ifd + 2 + 12 * (size_t)e;
					const uint32_t tag = rd16(o), type = rd16(o + 2), count = rd32(o + 4);
					const uint32_t tsize = type == 3 ? 2 : (type == 4 ? 4 : 1);
					const size_t vo = (size_t)count * tsize <= 4 ? o + 8 : rd32(o + 8);
					auto val = [&](uint32_t i) -> uint32_t { return type == 3 ? rd16(vo + 2 * (size_t)i) : (type == 4 ? rd32(vo + 4 * (size_t)i) : buf.at(vo + i)); };
					switch (tag) {
					case 256: pg.w = val(0); break;
					case 257: pg.h = val(0); break;
					case 258: pg.bits = val(0); break;
					case 259: pg.comp = val(0); break;
					case 262: pg.photo = val(0); break;
					case 277: pg.spp = val(0); break;
					case 278: pg.rps = val(0); break;
					case 273: for (uint32_t i = 0; i < count; i++) pg.off.push_back(val(i)); break;
					case 279: for (uint32_t i = 0; i < count; i++) pg.cnt.push_back(val(i)); break;
					default: break;
					}
				}
				if (pg.spp != 1 || (pg.bits != 8 && pg.bits != 16) || (pg.comp != 1 && pg.comp != 32773) || pg.off.empty() || pg.off.size() != pg.cnt.size())
					throw std::string("Unsupported TIFF page (need grayscale, 8/16 bit, uncompressed or PackBits strips): " + file_path);
				pages.push_back(pg);
				ifd = rd32((size_t)ifd + 2 + 12 * (size_t)n);
			}
			if (pages.empty()) throw std::string("Fail to load tiff: " + file_path);
			width = (int)pages[0].w;
			height = (int)pages[0].h;
			std::vector<std::vector<unsigned char>> out(pages.size());
			std::vector<unsigned char> raw;
			for (size_t z = 0; z < pages.size(); z++) {
				const Page& pg = pages[z];
				if ((int)pg.w != width || (int)pg.h != height) throw std::string("TIFF pages differ in size: " + file_path);
				const size_t bps = pg.bits / 8, want = (size_t)pg.w * pg.h * bps;
				raw.clear();
				for (size_t k = 0; k < pg.off.size(); k++) {
					if ((size_t)pg.off[k] + pg.cnt[k] > buf.size()) throw std::string("Truncated TIFF: " + file_path);
					const unsigned char* p = &buf[pg.off[k]];
					if (pg.comp == 1) raw.insert(raw.end(), p, p + pg.cnt[k]);
					else { // PackBits
						size_t i = 0;
						while (i < pg.cnt[k]) {
							const int c = (signed char)p[i++];
							if (c >= 0) { for (int t = 0; t <= c && i < pg.cnt[k]; t++) raw.push_back(p[i++]); }
							else if (c != -128 && i < pg.cnt[k]) { raw.insert(raw.end(), (size_t)(1 - c), p[i]); i++; }
						}
					}
				}
				if (raw.size() < want) throw std::string("Truncated TIFF page: " + file_path);
				out[z].resize((size_t)pg.w * pg.h);
				for (size_t i = 0; i < (size_t)pg.w * pg.h; i++) {
					uint32_t v = bps == 1 ? raw[i] : (le ? (uint32_t)raw[2 * i + 1] : (uint32_t)raw[2 * i]); // 16 -> 8 bit: the high byte
					if (pg.photo == 0) v = 255 - v; // WhiteIsZero
					out[z][i] = (unsigned char)v;
				}
			}
			return out;
		}
	} // namespace b200

	class Image2D
	{
	public:
		int height, width;
		unsigned int size;
		std::string file_path;
		MatrixXf eg_mat;
		unsigned long long generation = 0; // unique per load()/construction; lets the engine know when to re-upload

		inline Image2D(int width, int height)
		{
			b200::warmEngineAsync();
			generation = b200::nextGeneration();
			eg_mat.resize(height, width);
			this->width = width;
			this->height = height;
			size = height * width;
		}
		inline Image2D(std::string file_path) : height(0), width(0), size(0)
		{
			b200::warmEngineAsync();
			load(file_path);
		}
		~Image2D() = default;
		// a copy is a new image as far as the engine is concerned (it may be edited independently of the original)
		inline Image2D(const Image2D& o) : height(o.height), width(o.width), size(o.size), file_path(o.file_path), eg_mat(o.eg_mat), generation(b200::nextGeneration()) {}
		inline Image2D& operator=(const Image2D& o)
		{
			if (this != &o) {
				height = o.height; width = o.width; size = o.size; file_path = o.file_path; eg_mat = o.eg_mat;
				generation = b200::nextGeneration();
			}
			return *this;
		}

		// cv::imread(path, IMREAD_GRAYSCALE) for what the reference's examples feed it: uncompressed
		// 8-bit palettised / 24-bit / 32-bit BMP (src/oc_image.cpp:37-57).  Binary PGM (P5) is accepted too.
		inline void load(std::string file_path)
		{
			std::ifstream in(file_path, std::ios::binary);
			if (!in.is_open()) throw std::string("Fail to load file: " + file_path);
			std::vector<unsigned char> buf((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
			if (buf.size() > 54 && buf[0] == 'B' && buf[1] == 'M') {
				auto rd32 = [&](size_t o) { return (int32_t)(buf[o] | (buf[o + 1] << 8) | (buf[o + 2] << 16) | ((uint32_t)buf[o + 3] << 24)); };
				auto rd16 = [&](size_t o) { return (int)(buf[o] | (buf[o + 1] << 8)); };
				const int off = rd32(10), dib = rd32(14), w = rd32(18), hraw = rd32(22), bpp = rd16(28), comp = rd32(30);
				const int h = hraw < 0 ? -hraw : hraw;
				if (comp != 0 || (bpp != 8 && bpp != 24 && bpp != 32)) throw std::string("Fail to load file (unsupported BMP flavour): " + file_path);
				const size_t stride = ((size_t)w * bpp / 8 + 3) / 4 * 4;
				if (buf.size() < (size_t)off + stride * h) throw std::string("Fail to load file (truncated BMP): " + file_path);
				float pal[256];
				for (int i = 0; i < 256; i++) pal[i] = (float)i;
				if (bpp == 8) {
					int ncol = rd32(46);
					if (ncol <= 0 || ncol > 256) ncol = 256;
					const size_t po = 14 + (size_t)dib;
					for (int i = 0; i < ncol && po + 4 * (size_t)i + 3 < buf.size(); i++) {
						const float b = buf[po + 4 * i], g = buf[po + 4 * i + 1], r = buf[po + 4 * i + 2];
						pal[i] = (b == g && g == r) ? b : std::floor(0.299f * r + 0.587f * g + 0.114f * b + 0.5f);
					}
				}
				width = w; height = h; size = (unsigned int)(w * h);
				eg_mat.resize(h, w);
				for (int r = 0; r < h; r++) {
					const unsigned char* row = &buf[(size_t)off + stride * (size_t)(hraw > 0 ? h - 1 - r : r)];
					for (int c = 0; c < w; c++) {
						if (bpp == 8) eg_mat(r, c) = pal[row[c]];
						else {
							const unsigned char* px = row + (size_t)c * (bpp / 8);
							eg_mat(r, c) = std::floor(0.299f * px[2] + 0.587f * px[1] + 0.114f * px[0] + 0.5f);
						}
					}
				}
			} else if (buf.size() > 10 && buf[0] == 'P' && buf[1] == '5') {
				size_t pos = 2;
				int vals[3], nv = 0;
				while (nv < 3 && pos < buf.size()) {
					while (pos < buf.size() && (buf[pos] == ' ' || buf[pos] == '\n' || buf[pos] == '\r' || buf[pos] == '\t')) pos++;
					if (pos < buf.size() && buf[pos] == '#') { while (pos < buf.size() && buf[pos] != '\n') pos++; continue; }
					int v = 0;
					while (pos < buf.size() && buf[pos] >= '0' && buf[pos] <= '9') v = v * 10 + (buf[pos++] - '0');
					vals[nv++] = v;
				}
				pos++;
				if (nv < 3 || vals[2] > 255 || buf.size() < pos + (size_t)vals[0] * vals[1]) throw std::string("Fail to load file (bad PGM): " + file_path);
				width = vals[0]; height = vals[1]; size = (unsigned int)(width * height);
				eg_mat.resize(height, width);
				for (size_t i = 0; i < (size_t)width * height; i++) eg_mat.data[i] = (float)buf[pos + i];
			} else if (buf.size() > 8 && ((buf[0] == 'I' && buf[1] == 'I') || (buf[0] == 'M' && buf[1] == 'M'))) {
				int w = 0, h = 0;
				const std::vector<std::vector<unsigned char>> pages = b200::readTiffPages(file_path, w, h); // first page
				width = w; height = h; size = (unsigned int)(w * h);
				eg_mat.resize(h, w);
				for (size_t i = 0; i < (size_t)w * h; i++) eg_mat.data[i] = (float)pages[0][i];
			} else {
				throw std::string("Fail to load file: " + file_path);
			}
			this->file_path = file_path;
			generation = b200::nextGeneration();
		}
	};

	class Image3D
	{
	public:
		int dim_x, dim_y, dim_z;
		unsigned long size;
		std::string file_path;
		float*** vol_mat = nullptr; // [z][y][x]; payload is one contiguous block at vol_mat[0][0] (src/oc_array.h:56-74)
		unsigned long long generation = 0;
		bool payload_pinned = false;

		inline Image3D(int dim_x, int dim_y, int dim_z)
		{
			b200::warmEngineAsync();
			allocate(dim_x, dim_y, dim_z);
		}
		inline Image3D(std::string file_path) : dim_x(0), dim_y(0), dim_z(0), size(0)
		{
			b200::warmEngineAsync();
			load(file_path);
		}
		~Image3D() = default; // like the reference, the volume is released explicitly with release()

		inline void allocate(int dx, int dy, int dz)
		{
			release();
			dim_x = dx; dim_y = dy; dim_z = dz;
			size = (unsigned long)dz * dy * dx;
			float* p1 = b200::PixelBuffer::allocate(size, payload_pinned); // page-locked when a GPU is present (see PixelBuffer)
			std::memset(p1, 0, size * sizeof(float));
			float** p2 = (float**)malloc((size_t)dz * dy * sizeof(float*));
			vol_mat = (float***)malloc((size_t)dz * sizeof(float**));
			for (int i = 0; i < dz; i++) {
				for (int j = 0; j < dy; j++) p2[(size_t)i * dy + j] = p1 + ((size_t)i * dy + j) * dx;
				vol_mat[i] = p2 + (size_t)i * dy;
			}
			generation = b200::nextGeneration();
		}
		// binary volume: int32[3] header (dim_x, dim_y, dim_z) + float32 payload (src/oc_image.cpp:76-110)
		inline void loadBin(std::string file_path)
		{
			std::ifstream in(file_path, std::ios::in | std::ios::binary);
			if (!in.is_open()) throw std::string("Failed to open bin file: " + file_path);
			int dims[3];
			in.read((char*)dims, sizeof(int) * 3);
			allocate(dims[0], dims[1], dims[2]);
			in.read((char*)**vol_mat, sizeof(float) * size);
			if (!in) throw std::string("Failed to read bin file: " + file_path);
		}
		// multi-page TIFF, one page per z slice (src/oc_image.cpp:112-150 reads it with cv::imreadmulti(IMREAD_GRAYSCALE))
		inline void loadTiff(std::string file_path)
		{
			int w = 0, h = 0;
			const std::vector<std::vector<unsigned char>> pages = b200::readTiffPages(file_path, w, h);
			allocate(w, h, (int)pages.size());
			for (size_t z = 0; z < pages.size(); z++) {
				float* dst = vol_mat[z][0];
				for (size_t i = 0; i < (size_t)w * h; i++) dst[i] = (float)pages[z][i];
			}
		}
		inline void load(std::string file_path)
		{
			this->file_path = file_path;
			size_t dot_pos = file_path.find_last_of(".");
			std::string ext = file_path.substr(dot_pos + 1);
			if (ext == "bin" || ext == "BIN") loadBin(file_path);
			else if (ext == "tif" || ext == "TIF" || ext == "tiff" || ext == "TIFF") loadTiff(file_path);
			else throw std::string("Not binary file or multi-page tiff: " + file_path);
		}
		inline void release()
		{
			if (vol_mat != nullptr) {
				b200::PixelBuffer::deallocate(vol_mat[0][0], payload_pinned);
				free(vol_mat[0]);
				free(vol_mat);
				vol_mat = nullptr;
			}
		}
	};

	// ------------------------------------------------------------------ engine plumbing (not in the reference)
	namespace b200
	{
		// One process-wide GPU context shared by every DIC/DVC object, so that FFTCC and ICGN objects
		// set up on the same Image pair share ONE device copy (the reference's objects share the host
		// Image2D through borrowed pointers, src/oc_dic.cpp:22-26).
		//   OPENCORR_B200_DEVICES=all | 0,1,3   several GPUs behind the one context (ocb_create(-1) / ocb_create_multi):
		//                                        compute(std::vector<POI>&) shards the queue over them inside the C ABI
		//   OPENCORR_B200_DEVICE=<n>             one GPU (default 0)
		struct Engine
		{
			ocb_ctx* ctx = nullptr;
			std::mutex lock;
			std::thread warm_thread;
			bool warm_started = false;
			std::string warm_error;
			const void* ref_key = nullptr;
			const void* tar_key = nullptr;
			unsigned long long ref_gen = 0, tar_gen = 0;
			unsigned long long upload_serial = 0; // bumped by every upload: an object's prepare() is valid while this has not moved

			static Engine& get()
			{
				static Engine e;
				return e;
			}
			static ocb_ctx* create(std::string& error)
			{
				ocb_ctx* c = nullptr;
				const char* list = std::getenv("OPENCORR_B200_DEVICES");
				if (list && *list) {
					if (std::string(list) == "all") c = ocb_create(-1);
					else {
						std::vector<int> devs;
						for (const char* p = list; *p;) {
							char* end = nullptr;
							const long v = std::strtol(p, &end, 10);
							if (end == p) break;
							devs.push_back((int)v);
							p = (*end == ',') ? end + 1 : end;
						}
						c = ocb_create_multi(devs.data(), (int)devs.size());
					}
				} else {
					int dev = 0;
					if (const char* s = std::getenv("OPENCORR_B200_DEVICE")) dev = std::atoi(s);
					c = ocb_create(dev);
				}
				if (!c) error = ocb_last_error(nullptr);
				return c;
			}
			// (callers hold `lock`; the warm-up thread itself never takes it)
			void startWarm()
			{
				if (ctx || warm_started) return;
				warm_started = true;
				warm_thread = std::thread([this]() { ctx = create(warm_error); });
			}
			ocb_ctx* context()
			{
				if (warm_thread.joinable()) warm_thread.join();
				if (!ctx) {
					if (warm_error.empty()) ctx = create(warm_error);
					if (!ctx) throw std::string("opencorr_b200: " + warm_error);
				}
				return ctx;
			}
			void check(int rc)
			{
				if (rc != OCB_OK) throw std::string(std::string("opencorr_b200: ") + ocb_last_error(ctx));
			}
			void warm()
			{
				std::lock_guard<std::mutex> g(lock);
				startWarm();
			}

			~Engine()
			{
				if (warm_thread.joinable()) warm_thread.join();
				if (ctx) ocb_destroy(ctx);
			}
			// Make (ref, tar) the pair on the device.  force = false: skip the copy when this very pair (same objects, same
			// load generation) is already there -- what FFT-CC's compute() uses.  force = true: copy the pixels as they are NOW,
			// what prepare() means in the reference (its tables are built from the live image, src/oc_icgn.cpp:138-142).
			void useImages(Image2D* ref, Image2D* tar, bool force)
			{
				if (!ref || !tar) throw std::string("opencorr_b200: setImages() has not been called");
				if (!force && ref_key == ref && tar_key == tar && ref_gen == ref->generation && tar_gen == tar->generation) return;
				if (ref->width != tar->width || ref->height != tar->height) throw std::string("opencorr_b200: reference and target image sizes differ");
				check(ocb_set_images_2d(context(), ref->eg_mat.data.data(), tar->eg_mat.data.data(), ref->width, ref->height, 0));
				ref_key = ref; tar_key = tar; ref_gen = ref->generation; tar_gen = tar->generation;
				upload_serial++;
			}
			void useImages(Image3D* ref, Image3D* tar, bool force)
			{
				if (!ref || !tar || !ref->vol_mat || !tar->vol_mat) throw std::string("opencorr_b200: setImages() has not been called");
				if (!force && ref_key == ref && tar_key == tar && ref_gen == ref->generation && tar_gen == tar->generation) return;
				if (ref->dim_x != tar->dim_x || ref->dim_y != tar->dim_y || ref->dim_z != tar->dim_z) throw std::string("opencorr_b200: reference and target volume sizes differ");
				check(ocb_set_images_3d(context(), **ref->vol_mat, **tar->vol_mat, ref->dim_x, ref->dim_y, ref->dim_z));
				ref_key = ref; tar_key = tar; ref_gen = ref->generation; tar_gen = tar->generation;
				upload_serial++;
			}
		};
		inline void warmEngineAsync() { Engine::get().warm(); }
		inline void* pinnedAlloc(size_t bytes)
		{
			Engine& e = Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.startWarm();
			try {
				return ocb_host_alloc_on(e.context(), bytes);
			} catch (const std::string&) {
				return nullptr; // no GPU here: images live in ordinary memory (loading / saving still works)
			}
		}

		// What an object with a prepare() step remembers: the reference keeps per-object tables, so objects prepared on
		// different pairs can be used in any order.  Here the device holds ONE pair at a time; an object whose pair has been
		// displaced since its prepare() uploads it again and redoes the (cheap, on-device) prepare before computing.
		struct Prepared
		{
			bool called = false;
			unsigned long long serial = 0;
			template <class Img, class F>
			void prepare(Engine& e, Img* ref, Img* tar, F device_prepare)
			{
				e.useImages(ref, tar, true);
				e.check(device_prepare(e.context()));
				called = true;
				serial = e.upload_serial;
			}
			template <class Img, class F>
			void bind(Engine& e, Img* ref, Img* tar, F device_prepare)
			{
				if (!called) throw std::string("opencorr_b200: prepare() must be called before compute()");
				if (serial != e.upload_serial) prepare(e, ref, tar, device_prepare);
			}
		};
	} // namespace b200

	// ------------------------------------------------------------------ src/oc_dic.h
	class DIC
	{
	public:
		Image2D* ref_img = nullptr;
		Image2D* tar_img = nullptr;
		int subset_radius_x, subset_radius_y;
		int thread_number; // kept for signature compatibility; the GPU path has no CPU worker threads
		bool self_adaptive;

		// The GPU context is created with the first DIC/DVC object (the reference allocates its per-thread instance pools and
		// FFTW plans in the constructors), so that its ~0.2 s start-up is not charged to the first compute() call.
		DIC() : subset_radius_x(0), subset_radius_y(0), thread_number(1), self_adaptive(false) { b200::Engine::get().warm(); }
		virtual ~DIC() = default;
		// (pointers only, like the reference: the device copy is made by the first prepare()/compute() that needs it, so
		// images filled in after setImages() are seen)
		void setImages(Image2D& ref_img, Image2D& tar_img) { this->ref_img = &ref_img; this->tar_img = &tar_img; }
		void setSubset(int radius_x, int radius_y) { subset_radius_x = radius_x; subset_radius_y = radius_y; }
		void setSelfAdaptive(bool is_self_adaptive) { self_adaptive = is_self_adaptive; }
		virtual void prepare() = 0;
		virtual void compute(POI2D* poi) = 0;
		virtual void compute(std::vector<POI2D>& poi_queue) = 0;
	};

	class DVC
	{
	public:
		Image3D* ref_img = nullptr;
		Image3D* tar_img = nullptr;
		int subset_radius_x, subset_radius_y, subset_radius_z;
		int thread_number;

		DVC() : subset_radius_x(0), subset_radius_y(0), subset_radius_z(0), thread_number(1) { b200::Engine::get().warm(); }
		virtual ~DVC() = default;
		void setImages(Image3D& ref_img, Image3D& tar_img) { this->ref_img = &ref_img; this->tar_img = &tar_img; }
		void setSubset(int radius_x, int radius_y, int radius_z) { subset_radius_x = radius_x; subset_radius_y = radius_y; subset_radius_z = radius_z; }
		virtual void prepare() = 0;
		virtual void compute(POI3D* POI) = 0;
		virtual void compute(std::vector<POI3D>& poi_queue) = 0;
	};

	inline bool sortByZNCC(const POI2D& p1, const POI2D& p2) { return p1.result.zncc > p2.result.zncc; }

	// ------------------------------------------------------------------ src/oc_fftcc.h
	class FFTCC2D : public DIC
	{
	public:
		FFTCC2D(int subset_radius_x, int subset_radius_y, int thread_number)
		{
			this->subset_radius_x = subset_radius_x;
			this->subset_radius_y = subset_radius_y;
			this->thread_number = thread_number;
		}
		~FFTCC2D() {}
		void prepare() {}
		void compute(POI2D* poi) { run(poi, 1); }
		void compute(std::vector<POI2D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

	private:
		void run(POI2D* p, size_t n)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.useImages(ref_img, tar_img, false);
			e.check(ocb_fftcc2d(e.context(), p, n, subset_radius_x, subset_radius_y));
		}
	};

	class FFTCC3D : public DVC
	{
	public:
		FFTCC3D(int subset_radius_x, int subset_radius_y, int subset_radius_z, int thread_number)
		{
			this->subset_radius_x = subset_radius_x;
			this->subset_radius_y = subset_radius_y;
			this->subset_radius_z = subset_radius_z;
			this->thread_number = thread_number;
		}
		~FFTCC3D() {}
		void prepare() {}
		void compute(POI3D* poi) { run(poi, 1); }
		void compute(std::vector<POI3D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

	private:
		void run(POI3D* p, size_t n)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.useImages(ref_img, tar_img, false);
			e.check(ocb_fftcc3d(e.context(), p, n, subset_radius_x, subset_radius_y, subset_radius_z));
		}
	};

	// ------------------------------------------------------------------ src/oc_feature.h:46-63, src/oc_sift.h:71-155
	class Feature3D
	{
	protected:
		Image3D* ref_img = nullptr;
		Image3D* tar_img = nullptr;

	public:
		virtual ~Feature3D() = default;
		inline void setImages(Image3D& ref_img, Image3D& tar_img)
		{
			this->ref_img = &ref_img;
			this->tar_img = &tar_img;
		}
		virtual void prepare() = 0;
		virtual void compute() = 0;
	};

	struct Sift3dConfig
	{
		int n_octave_layers;
		int n_octave;
		int min_dimension;
		float alpha;
		float beta;
		float gamma;
		float sigma_source;
		float sigma_base;
		float gradient_threshold;
		float truncate_threshold;
	};

	// SIFT3D on the GPU (ocb_sift3d).  The reference's helpers on host float*** layers (gaussianBlur, createGaussianPyramid,
	// detectExtrema, ...) are not provided: the pyramid lives on the device, one octave at a time.
	class SIFT3D : public Feature3D
	{
	protected:
		Sift3dConfig sift_config;
		float matching_ratio;
		float physical_unit[3];

	public:
		std::vector<Point3D> ref_matched_kp;
		std::vector<Point3D> tar_matched_kp;

		SIFT3D()
		{
			sift_config.n_octave_layers = 3; // src/oc_sift.cpp:142-158
			sift_config.n_octave = 0;
			sift_config.min_dimension = 8;
			sift_config.alpha = 0.1f;
			sift_config.beta = 0.9f;
			sift_config.gamma = 0.4f;
			sift_config.sigma_source = 1.15f;
			sift_config.sigma_base = 1.6f;
			sift_config.gradient_threshold = 0.0000000001f;
			sift_config.truncate_threshold = 0.2f * 128 / 768;
			matching_ratio = 0.85f;
			physical_unit[0] = physical_unit[1] = physical_unit[2] = 1.f;
			b200::Engine::get().warm();
		}
		~SIFT3D() {}

		Sift3dConfig getSiftConfig() const { return sift_config; }
		float getPhysicalUnit(int dim) const { return (dim >= 0 && dim < 3) ? physical_unit[dim] : 0.f; }
		float getMatchingRatio() const { return matching_ratio; }
		void setSiftConfig(Sift3dConfig sift_config) { this->sift_config = sift_config; }
		void setPhysicalUnit(float unit_x, float unit_y, float unit_z)
		{
			physical_unit[0] = unit_x;
			physical_unit[1] = unit_y;
			physical_unit[2] = unit_z;
		}
		void setMatchingRatio(float matching_ratio) { this->matching_ratio = matching_ratio; }
		void prepare() {} // the icosahedron (:209-232) is built into the kernels
		void compute()
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.useImages(ref_img, tar_img, false);
			const float cfg[OCB_SIFT3D_CONFIG_FLOATS] = { (float)sift_config.n_octave_layers, (float)sift_config.n_octave, (float)sift_config.min_dimension,
				sift_config.alpha, sift_config.beta, sift_config.gamma, sift_config.sigma_source, sift_config.sigma_base, sift_config.gradient_threshold,
				sift_config.truncate_threshold };
			size_t n = 0, counts[2][3];
			int n_octave = 0;
			e.check(ocb_sift3d(e.context(), cfg, physical_unit, matching_ratio, &n, &n_octave));
			sift_config.n_octave = n_octave;
			for (int i = 0; i < 2; i++) e.check(ocb_sift3d_inspect(e.context(), i, counts[i], nullptr, nullptr, nullptr, nullptr));
			std::cout << counts[0][2] << " features are extracted from the reference image." << std::endl;
			std::cout << counts[1][2] << " features are extracted from the target image." << std::endl;
			clear();
			std::vector<float> r(3 * n), t(3 * n);
			e.check(ocb_sift3d_get_matches(e.context(), r.data(), t.data()));
			for (size_t i = 0; i < n; i++) {
				ref_matched_kp.push_back(Point3D(r[3 * i], r[3 * i + 1], r[3 * i + 2]));
				tar_matched_kp.push_back(Point3D(t[3 * i], t[3 * i + 1], t[3 * i + 2]));
			}
		}
		void clear()
		{
			std::vector<Point3D>().swap(ref_matched_kp);
			std::vector<Point3D>().swap(tar_matched_kp);
		}
	};

	// ------------------------------------------------------------------ src/oc_icgn.h
	namespace b200
	{
		template <int ORDER>
		class ICGN2D : public DIC
		{
		protected:
			float conv_criterion;
			float stop_condition;
			Prepared prepared;

		public:
			ICGN2D(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition, int thread_number)
			{
				this->subset_radius_x = subset_radius_x;
				this->subset_radius_y = subset_radius_y;
				this->conv_criterion = conv_criterion;
				this->stop_condition = stop_condition;
				this->thread_number = thread_number;
				self_adaptive = false;
			}
			void setIteration(float conv_criterion, float stop_condition)
			{
				this->conv_criterion = conv_criterion;
				this->stop_condition = stop_condition;
			}
			void setIteration(POI2D* poi) // src/oc_icgn.cpp:109-113 / :650-654
			{
				conv_criterion = poi->result.convergence;
				stop_condition = (ORDER == 1) ? (float)(int)poi->result.iteration : poi->result.iteration;
			}
			void prepareRef() { prepare(); }
			void prepareTar() { prepare(); }
			void prepare()
			{
				Engine& e = Engine::get();
				std::lock_guard<std::mutex> g(e.lock);
				prepared.prepare(e, ref_img, tar_img, ocb_icgn2d_prepare);
			}
			// (engine lock held) make this object's pair and prepare() current on the device
			void bindLocked(Engine& e) { prepared.bind(e, ref_img, tar_img, ocb_icgn2d_prepare); }
			void compute(POI2D* poi) { run(poi, 1, nullptr); }
			void compute(std::vector<POI2D>& poi_queue) { run(poi_queue.data(), poi_queue.size(), nullptr); }
			// off-centre subsets, src/oc_icgn.cpp:353-557 / :910-1136 (Point2D is two packed floats)
			void compute(POI2D* poi, Point2D& center_offset) { run(poi, 1, &center_offset.x); }
			void compute(std::vector<POI2D>& poi_queue, std::vector<Point2D>& center_offset_queue)
			{
				if (center_offset_queue.size() < poi_queue.size()) throw std::string("opencorr_b200: center_offset_queue is shorter than poi_queue");
				run(poi_queue.data(), poi_queue.size(), poi_queue.empty() ? nullptr : &center_offset_queue[0].x);
			}

		private:
			void run(POI2D* p, size_t n, const float* offsets)
			{
				Engine& e = Engine::get();
				std::lock_guard<std::mutex> g(e.lock);
				bindLocked(e);
				if (self_adaptive || offsets)
					e.check(ocb_icgn2d_ex(e.context(), ORDER, p, n, subset_radius_x, subset_radius_y, conv_criterion, stop_condition, offsets, self_adaptive ? 1 : 0));
				else if (ORDER == 1) e.check(ocb_icgn2d1(e.context(), p, n, subset_radius_x, subset_radius_y, conv_criterion, stop_condition));
				else e.check(ocb_icgn2d2(e.context(), p, n, subset_radius_x, subset_radius_y, conv_criterion, stop_condition));
			}
		};
	} // namespace b200

	class ICGN2D1 : public b200::ICGN2D<1>
	{
	public:
		ICGN2D1(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition, int thread_number)
			: b200::ICGN2D<1>(subset_radius_x, subset_radius_y, conv_criterion, stop_condition, thread_number) {}
	};

	class ICGN2D2 : public b200::ICGN2D<2>
	{
	public:
		ICGN2D2(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition, int thread_number)
			: b200::ICGN2D<2>(subset_radius_x, subset_radius_y, conv_criterion, stop_condition, thread_number) {}
	};

	// ------------------------------------------------------------------ src/oc_iclm.h (SURVEY 8(f) N2)
	struct DampingParameter
	{
		float lambda = 100.f;
		float alpha = 0.1f;
		float beta = 10.f;
	};

	namespace b200
	{
		template <int ORDER>
		class ICLM2D : public DIC
		{
		protected:
			float conv_criterion;
			float stop_condition;
			DampingParameter damping;
			Prepared prepared;

		public:
			ICLM2D(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition, int thread_number)
			{
				this->subset_radius_x = subset_radius_x;
				this->subset_radius_y = subset_radius_y;
				this->conv_criterion = conv_criterion;
				this->stop_condition = stop_condition;
				this->thread_number = thread_number;
				self_adaptive = false;
			}
			void setIteration(float conv_criterion, float stop_condition)
			{
				this->conv_criterion = conv_criterion;
				this->stop_condition = stop_condition;
			}
			void setIteration(POI2D* poi)
			{
				conv_criterion = poi->result.convergence;
				stop_condition = (float)(int)poi->result.iteration;
			}
			void setDamping(float lambda, float alpha, float beta) // src/oc_iclm.cpp:114-119
			{
				damping.lambda = lambda;
				damping.alpha = alpha;
				damping.beta = beta;
			}
			void prepareRef() { prepare(); }
			void prepareTar() { prepare(); }
			void prepare()
			{
				Engine& e = Engine::get();
				std::lock_guard<std::mutex> g(e.lock);
				prepared.prepare(e, ref_img, tar_img, ocb_icgn2d_prepare);
			}
			void compute(POI2D* poi) { run(poi, 1); }
			void compute(std::vector<POI2D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

		private:
			void run(POI2D* p, size_t n)
			{
				if (self_adaptive) throw std::string("opencorr_b200: self-adaptive subsets are implemented for ICGN2D1/ICGN2D2 only");
				Engine& e = Engine::get();
				std::lock_guard<std::mutex> g(e.lock);
				prepared.bind(e, ref_img, tar_img, ocb_icgn2d_prepare);
				e.check(ocb_iclm2d(e.context(), ORDER, p, n, subset_radius_x, subset_radius_y, conv_criterion, stop_condition, damping.lambda, damping.alpha,
					damping.beta));
			}
		};
	} // namespace b200

	class ICLM2D1 : public b200::ICLM2D<1>
	{
	public:
		ICLM2D1(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition, int thread_number)
			: b200::ICLM2D<1>(subset_radius_x, subset_radius_y, conv_criterion, stop_condition, thread_number) {}
	};

	class ICLM2D2 : public b200::ICLM2D<2>
	{
	public:
		ICLM2D2(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition, int thread_number)
			: b200::ICLM2D<2>(subset_radius_x, subset_radius_y, conv_criterion, stop_condition, thread_number) {}
	};

	// Strain (reference src/oc_strain.h:33-70, src/oc_strain.cpp): least-squares plane fit of the displacement field
	// over each POI's neighbourhood.  prepare() builds kd-trees in the reference; here the spatial binning is part of
	// the GPU call, so prepare() is empty.  
	class Strain
	{
	protected:
		float subregion_radius;
		int neighbor_number_min;
		float zncc_threshold;
		int description;
		int approximation;
		int thread_number;

	public:
		Strain(float subregion_radius, int neighbor_number_min, int thread_number)
		{
			this->subregion_radius = subregion_radius;
			this->neighbor_number_min = neighbor_number_min;
			zncc_threshold = 0.9f; // src/oc_strain.cpp:38-40
			description = 1;
			approximation = 1;
			this->thread_number = thread_number;
		}
		~Strain() {}
		float getSubregionRadius() const { return subregion_radius; }
		int getNeighborMin() const { return neighbor_number_min; }
		float getZnccThreshold() const { return zncc_threshold; }
		void setSubregionRadius(float subregion_radius) { this->subregion_radius = subregion_radius; }
		void setNeighborMin(int neighbor_number_min) { this->neighbor_number_min = neighbor_number_min; }
		void setZnccThreshold(float zncc_threshold) { this->zncc_threshold = zncc_threshold; }
		void setDescription(int description) { this->description = description; }
		void setApproximation(int approximation) { this->approximation = approximation; }

		void prepare(std::vector<POI2D>&) {}
		void prepare(std::vector<POI2DS>&) {}
		void prepare(std::vector<POI3D>&) {}

		void compute(std::vector<POI2D>& poi_queue)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_strain2d(e.context(), poi_queue.data(), poi_queue.size(), subregion_radius, neighbor_number_min, zncc_threshold, approximation));
		}
		void compute(std::vector<POI2DS>& poi_queue) // src/oc_strain.cpp:362-371 (per POI :252-360)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_strain2ds(e.context(), poi_queue.data(), poi_queue.size(), subregion_radius, neighbor_number_min, zncc_threshold, approximation));
		}
		void compute(std::vector<POI3D>& poi_queue)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_strain3d(e.context(), poi_queue.data(), poi_queue.size(), subregion_radius, neighbor_number_min, zncc_threshold, approximation));
		}
		// single-POI overloads (src/oc_strain.cpp:158-237, :373-474); `poi` must be an element of `poi_queue`
		// (the reference searches the tree built from the queue by prepare()).  One POI per call is a poor fit for a
		// GPU: prefer the queue overloads.
		void compute(POI2D* poi, std::vector<POI2D>& poi_queue)
		{
			if (poi < poi_queue.data() || poi >= poi_queue.data() + poi_queue.size()) throw std::string("opencorr_b200: Strain::compute(poi, queue) needs poi inside queue");
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_strain2d_single(e.context(), poi_queue.data(), poi_queue.size(), (size_t)(poi - poi_queue.data()), subregion_radius, neighbor_number_min,
				zncc_threshold, approximation));
		}
		void compute(POI3D* poi, std::vector<POI3D>& poi_queue)
		{
			if (poi < poi_queue.data() || poi >= poi_queue.data() + poi_queue.size()) throw std::string("opencorr_b200: Strain::compute(poi, queue) needs poi inside queue");
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_strain3d_single(e.context(), poi_queue.data(), poi_queue.size(), (size_t)(poi - poi_queue.data()), subregion_radius, neighbor_number_min,
				zncc_threshold, approximation));
		}
	};

	// RegionFit2D / RegionFit3D (reference src/oc_region_fit.h:25-85, src/oc_region_fit.cpp): a POI's new initial guess from the
	// plane fit of its reliable neighbours' displacements (include/opencorr_b200.h ocb_region_fit2d).  setNeighbor keeps a pointer
	// to the reliable queue, read when compute() runs; prepare() builds kd-trees in the reference and is empty here.
	class RegionFit2D : public DIC
	{
	protected:
		std::vector<POI2D>* neighbor_reliable = nullptr;
		float neighbor_search_radius;
		int neighbor_number_min;

	public:
		RegionFit2D(float neighbor_search_radius, int neighbor_number_min, int thread_number)
		{
			this->neighbor_search_radius = neighbor_search_radius;
			this->neighbor_number_min = neighbor_number_min;
			this->thread_number = thread_number;
		}
		~RegionFit2D() {}
		float getSearchRadius() const { return neighbor_search_radius; }
		int getNeighborMin() const { return neighbor_number_min; }
		void setSearchRadius(float neighbor_search_radius) { this->neighbor_search_radius = neighbor_search_radius; }
		void setNeighborMin(int neighbor_number_min) { this->neighbor_number_min = neighbor_number_min; }
		void setNeighbor(std::vector<POI2D>& reliable_pois) { neighbor_reliable = &reliable_pois; }

		void prepare() {}
		void compute(POI2D* poi) { run(poi, 1); }
		void compute(std::vector<POI2D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

	private:
		void run(POI2D* q, size_t n)
		{
			if (!neighbor_reliable) throw std::string("opencorr_b200: RegionFit2D::compute needs setNeighbor() first");
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_region_fit2d(e.context(), neighbor_reliable->data(), neighbor_reliable->size(), q, n, neighbor_search_radius, neighbor_number_min));
		}
	};

	class RegionFit3D : public DVC
	{
	protected:
		std::vector<POI3D>* neighbor_reliable = nullptr;
		float neighbor_search_radius;
		int neighbor_number_min;

	public:
		RegionFit3D(float neighbor_search_radius, int neighbor_number_min, int thread_number)
		{
			this->neighbor_search_radius = neighbor_search_radius;
			this->neighbor_number_min = neighbor_number_min;
			this->thread_number = thread_number;
		}
		~RegionFit3D() {}
		float getSearchRadius() const { return neighbor_search_radius; }
		int getNeighborMin() const { return neighbor_number_min; }
		void setSearchRadius(float neighbor_search_radius) { this->neighbor_search_radius = neighbor_search_radius; }
		void setNeighborMin(int neighbor_number_min) { this->neighbor_number_min = neighbor_number_min; }
		void setNeighbor(std::vector<POI3D>& reliable_pois) { neighbor_reliable = &reliable_pois; }

		void prepare() {}
		void compute(POI3D* poi) { run(poi, 1); }
		void compute(std::vector<POI3D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

	private:
		void run(POI3D* q, size_t n)
		{
			if (!neighbor_reliable) throw std::string("opencorr_b200: RegionFit3D::compute needs setNeighbor() first");
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_region_fit3d(e.context(), neighbor_reliable->data(), neighbor_reliable->size(), q, n, neighbor_search_radius, neighbor_number_min));
		}
	};

	// NR2D1 (forward-additive Newton-Raphson), reference src/oc_nr.h:46-71, src/oc_nr.cpp:66-334
	class NR2D1 : public DIC
	{
	private:
		float conv_criterion;
		float stop_condition;
		b200::Prepared prepared;

	public:
		NR2D1(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition, int thread_number)
		{
			this->subset_radius_x = subset_radius_x;
			this->subset_radius_y = subset_radius_y;
			this->conv_criterion = conv_criterion;
			this->stop_condition = stop_condition;
			this->thread_number = thread_number;
		}
		~NR2D1() {}
		void setIteration(float conv_criterion, float stop_condition)
		{
			this->conv_criterion = conv_criterion;
			this->stop_condition = stop_condition;
		}
		void setIteration(POI2D* poi) // src/oc_nr.cpp:113-117
		{
			conv_criterion = poi->result.convergence;
			stop_condition = (float)(int)poi->result.iteration;
		}
		void prepare()
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			prepared.prepare(e, ref_img, tar_img, ocb_nr2d_prepare);
		}
		void compute(POI2D* poi) { run(poi, 1); }
		void compute(std::vector<POI2D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

	private:
		void run(POI2D* p, size_t n)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			prepared.bind(e, ref_img, tar_img, ocb_nr2d_prepare);
			e.check(ocb_nr2d1(e.context(), p, n, subset_radius_x, subset_radius_y, conv_criterion, stop_condition));
		}
	};

	// ---------------------------------------------------------------- EpipolarSearch (SURVEY.md section 8(f) N4)
	// Camera parameters, reference src/oc_calibration.h:25-45
	union CameraIntrinsics
	{
		struct
		{
			float fx, fy, fs;
			float cx, cy;
			float k1, k2, k3, k4, k5, k6;
			float p1, p2;
		};
		float cam_i[13];
	};

	union CameraExtrinsics
	{
		struct
		{
			float tx, ty, tz;
			float rx, ry, rz;
		};
		float cam_e[6];
	};

	// Calibration, reference src/oc_calibration.h:47-98, src/oc_calibration.cpp:21-264: intrinsic / rotation / translation /
	// projection matrices (row-major plain arrays instead of Eigen types) and the lens-distortion correction.  prepare(height,
	// width) builds the map of undistorted image coordinates on the GPU (ocb_calib_prepare); undistort(Point2D&) looks one
	// point up in it, and Stereovision::reconstruct looks up whole queues.  The map stays in device memory: the reference's
	// public map_x / map_y Eigen members are not reproduced (no example program reads them).  Copies of a Calibration share
	// the map (EpipolarSearch keeps copies of its cameras); the last copy frees it.
	class Calibration
	{
	public:
		CameraIntrinsics intrinsics;
		CameraExtrinsics extrinsics;
		float intrinsic_matrix[3][3];
		float rotation_matrix[3][3];
		float translation_vector[3];
		float projection_matrix[3][4];
		std::shared_ptr<ocb_calib> map; // device map of prepare(), on the process-wide engine

		Calibration()
		{
			std::fill(std::begin(intrinsics.cam_i), std::end(intrinsics.cam_i), 0.f);
			std::fill(std::begin(extrinsics.cam_e), std::end(extrinsics.cam_e), 0.f);
		}
		Calibration(CameraIntrinsics& intrinsics, CameraExtrinsics& extrinsics) { updateCalibration(intrinsics, extrinsics); }
		~Calibration() {}

		float getConvergence() const { return convergence; }
		int getIteration() const { return iteration; }
		void setUndistortion(float convergence, int iteration) // :111-115
		{
			this->convergence = convergence;
			this->iteration = iteration;
		}

		// single-point formulas, :117-159 (float32, the reference's operation order)
		Point2D image_to_sensor(Point2D& point)
		{
			float sensor_y = point.y * intrinsics.fy + intrinsics.cy;
			float sensor_x = point.x * intrinsics.fx + point.y * intrinsics.fs + intrinsics.cx;
			return Point2D(sensor_x, sensor_y);
		}
		Point2D sensor_to_image(Point2D& point)
		{
			float image_y = (point.y - intrinsics.cy) / intrinsics.fy;
			float image_x = (point.x - intrinsics.cx - intrinsics.fs * image_y) / intrinsics.fx;
			return Point2D(image_x, image_y);
		}
		Point2D distort(Point2D& point)
		{
			float xx = point.x * point.x, yy = point.y * point.y, xy = point.x * point.y;
			float r2 = xx + yy;
			float r4 = r2 * r2;
			float r6 = r2 * r4;
			float radial = (1 + intrinsics.k1 * r2 + intrinsics.k2 * r4 + intrinsics.k3 * r6) / (1 + intrinsics.k4 * r2 + intrinsics.k5 * r4 + intrinsics.k6 * r6);
			float distorted_y = point.y * radial;
			float distorted_x = point.x * radial;
			distorted_y += intrinsics.p1 * (r2 + 2 * yy) + 2 * intrinsics.p2 * xy;
			distorted_x += 2 * intrinsics.p1 * xy + intrinsics.p2 * (r2 + 2 * xx);
			return Point2D(distorted_x, distorted_y);
		}

		// :161-219 on the GPU (one thread per pixel)
		void prepare(int height, int width)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			ocb_calib* c = nullptr;
			e.check(ocb_calib_prepare(e.context(), intrinsics.cam_i, height, width, convergence, iteration, &c));
			map.reset(c, ocb_calib_destroy);
		}
		// :221-264 as a batch of one: the point is clamped in place, the sensor coordinates are returned
		Point2D undistort(Point2D& point)
		{
			if (!map) throw std::string("opencorr_b200: Calibration::prepare() must be called before undistort()");
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			float p[2] = { point.x, point.y }, out[2];
			e.check(ocb_calib_undistort(e.context(), map.get(), intrinsics.cam_i, p, out, 1));
			point.x = p[0];
			point.y = p[1];
			return Point2D(out[0], out[1]);
		}

		void updateIntrinsicMatrix() // src/oc_calibration.cpp:36-48
		{
			const float k[3][3] = { { intrinsics.fx, intrinsics.fs, intrinsics.cx }, { 0.f, intrinsics.fy, intrinsics.cy }, { 0.f, 0.f, 1.f } };
			std::memcpy(intrinsic_matrix, k, sizeof(k));
			if (intrinsics.fx == 1.f && intrinsics.fy == 1.f && intrinsics.fs == 0.f && intrinsics.cx == 0.f && intrinsics.cy == 0.f)
				throw std::string("Null intrinsics matrix");
		}
		void updateRotationMatrix() // src/oc_calibration.cpp:50-60 (Eigen::AngleAxisf::toRotationMatrix)
		{
			const float rx = extrinsics.rx, ry = extrinsics.ry, rz = extrinsics.rz;
			const float theta = std::sqrt(rx * rx + ry * ry + rz * rz);
			float x = rx, y = ry, z = rz;
			if (theta > 0.f) { x /= theta; y /= theta; z /= theta; }
			const float c = std::cos(theta), s = std::sin(theta), t = 1.f - c;
			const float r[3][3] = { { t * x * x + c, t * x * y - s * z, t * x * z + s * y },
				{ t * x * y + s * z, t * y * y + c, t * y * z - s * x },
				{ t * x * z - s * y, t * y * z + s * x, t * z * z + c } };
			std::memcpy(rotation_matrix, r, sizeof(r));
		}
		void updateTranslationVector()
		{
			translation_vector[0] = extrinsics.tx;
			translation_vector[1] = extrinsics.ty;
			translation_vector[2] = extrinsics.tz;
		}
		void updateProjectionMatrix() // K [R | t], src/oc_calibration.cpp:69-77
		{
			for (int i = 0; i < 3; i++)
				for (int j = 0; j < 4; j++) {
					float v = 0.f;
					for (int k = 0; k < 3; k++) v += intrinsic_matrix[i][k] * (j < 3 ? rotation_matrix[k][j] : translation_vector[k]);
					projection_matrix[i][j] = v;
				}
		}
		void updateMatrices()
		{
			updateIntrinsicMatrix();
			updateRotationMatrix();
			updateTranslationVector();
			updateProjectionMatrix();
		}
		void updateCalibration(CameraIntrinsics& intrinsics, CameraExtrinsics& extrinsics)
		{
			this->intrinsics = intrinsics;
			this->extrinsics = extrinsics;
			updateMatrices();
		}
		void clear()
		{
			std::fill(std::begin(intrinsics.cam_i), std::end(intrinsics.cam_i), 0.f);
			std::fill(std::begin(extrinsics.cam_e), std::end(extrinsics.cam_e), 0.f);
		}

	private:
		float convergence = 0.001f; // :21-32
		int iteration = 40;
	};

	namespace b200
	{
		inline void inverse3(const float m[3][3], float inv[3][3])
		{
			const double a = m[0][0], b = m[0][1], c = m[0][2], d = m[1][0], e = m[1][1], f = m[1][2], g = m[2][0], h = m[2][1], i = m[2][2];
			const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
			const double r[3][3] = { { e * i - f * h, c * h - b * i, b * f - c * e }, { f * g - d * i, a * i - c * g, c * d - a * f }, { d * h - e * g, b * g - a * h, a * e - b * d } };
			for (int p = 0; p < 3; p++)
				for (int q = 0; q < 3; q++) inv[p][q] = (float)(r[p][q] / det);
		}
		inline void matmul3(const float a[3][3], const float b[3][3], float c[3][3])
		{
			for (int i = 0; i < 3; i++)
				for (int j = 0; j < 3; j++) c[i][j] = a[i][0] * b[0][j] + a[i][1] * b[1][j] + a[i][2] * b[2][j];
		}
		// K2^-T [t2]x R2 K1^-1, row-major: EpipolarSearch::updateFundementalMatrix (src/oc_epipolar_search.cpp:110-126) and
		// Stereovision::updateFundementalMatrix (src/oc_stereovision.cpp:36-54)
		inline void fundamentalMatrix(const Calibration& view1_cam, const Calibration& view2_cam, float fundamental_matrix[9])
		{
			float k2_inv[3][3], k2_inv_t[3][3], k1_inv[3][3], e[3][3], tmp[3][3], f[3][3];
			inverse3(view2_cam.intrinsic_matrix, k2_inv);
			for (int i = 0; i < 3; i++)
				for (int j = 0; j < 3; j++) k2_inv_t[i][j] = k2_inv[j][i];
			const float* t = view2_cam.translation_vector;
			const float t_anti[3][3] = { { 0.f, -t[2], t[1] }, { t[2], 0.f, -t[0] }, { -t[1], t[0], 0.f } };
			matmul3(t_anti, view2_cam.rotation_matrix, e);
			inverse3(view1_cam.intrinsic_matrix, k1_inv);
			matmul3(k2_inv_t, e, tmp);
			matmul3(tmp, k1_inv, f);
			for (int i = 0; i < 3; i++)
				for (int j = 0; j < 3; j++) fundamental_matrix[3 * i + j] = f[i][j];
		}
	} // namespace b200

	// Stereovision, reference src/oc_stereovision.h / .cpp:21-133.  Both cameras must have been prepare()d.  The queue overload of
	// reconstruct() is one GPU batch (ocb_stereo_reconstruct): every pair is undistorted and triangulated by its own thread, the
	// 4x3 least-squares system solved in FP64; as in the reference the input points are clamped in place and a pair with a NaN
	// coordinate gives (0, 0, 0).
	class Stereovision
	{
	public:
		Calibration* view1_cam;
		Calibration* view2_cam;
		int thread_number; // kept for signature compatibility
		float fundamental_matrix[9]; // row-major

		Stereovision(Calibration* view1_cam, Calibration* view2_cam, int thread_number)
		{
			this->view1_cam = view1_cam;
			this->view2_cam = view2_cam;
			this->thread_number = thread_number;
			std::fill(std::begin(fundamental_matrix), std::end(fundamental_matrix), 0.f);
		}
		~Stereovision() {}

		void updateCameras(Calibration* view1_cam, Calibration* view2_cam)
		{
			this->view1_cam = view1_cam;
			this->view2_cam = view2_cam;
		}
		void updateFundementalMatrix() { b200::fundamentalMatrix(*view1_cam, *view2_cam, fundamental_matrix); }
		void prepare() // :56-68
		{
			view1_cam->updateMatrices();
			view2_cam->updateMatrices();
			updateFundementalMatrix();
		}
		Point3D reconstruct(Point2D& view1_2d_point, Point2D& view2_2d_point)
		{
			Point3D out;
			run(&view1_2d_point, &view2_2d_point, &out, 1);
			return out;
		}
		void reconstruct(std::vector<Point2D>& view1_2d_point_queue, std::vector<Point2D>& view2_2d_point_queue, std::vector<Point3D>& space_3d_point_queue)
		{
			const size_t n = view1_2d_point_queue.size();
			if (view2_2d_point_queue.size() < n || space_3d_point_queue.size() < n)
				throw std::string("opencorr_b200: Stereovision::reconstruct needs queues of equal length");
			run(view1_2d_point_queue.data(), view2_2d_point_queue.data(), space_3d_point_queue.data(), n);
		}

	private:
		static_assert(sizeof(Point2D) == 2 * sizeof(float) && sizeof(Point3D) == 3 * sizeof(float), "points are passed as float arrays");
		void run(Point2D* p1, Point2D* p2, Point3D* p3, size_t n)
		{
			if (!view1_cam->map || !view2_cam->map) throw std::string("opencorr_b200: Calibration::prepare() must be called before reconstruct()");
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			e.check(ocb_stereo_reconstruct(e.context(), view1_cam->map.get(), view1_cam->intrinsics.cam_i, &view1_cam->projection_matrix[0][0],
				view2_cam->map.get(), view2_cam->intrinsics.cam_i, &view2_cam->projection_matrix[0][0], &p1->x, &p2->x, &p3->x, n));
		}
	};

	// EpipolarSearch, reference src/oc_epipolar_search.h:30-63 / .cpp:21-205.  compute(queue) runs the candidate sweep of ALL
	// POIs as one GPU batch (ocb_epipolar_search2d) instead of one POI at a time.
	class EpipolarSearch : public DIC
	{
	protected:
		int search_radius = 0;
		int search_step = 1;
		Calibration view1_cam;
		Calibration view2_cam;
		float fundamental_matrix[9]; // row-major
		Point2D parallax;
		float parallax_x[3] = { 0.f, 0.f, 0.f }, parallax_y[3] = { 0.f, 0.f, 0.f };

	public:
		std::unique_ptr<ICGN2D1> icgn1;

		EpipolarSearch(Calibration& view1_cam, Calibration& view2_cam, int thread_number)
		{
			this->view1_cam = view1_cam;
			this->view2_cam = view2_cam;
			this->thread_number = thread_number;
			std::fill(std::begin(fundamental_matrix), std::end(fundamental_matrix), 0.f);
		}
		~EpipolarSearch() { destoryICGN(); }

		int getSearchRadius() const { return search_radius; }
		int getSearchStep() const { return search_step; }
		void setSearch(int search_radius, int search_step)
		{
			if (search_radius < search_step) throw std::string("Search radius is less than search step");
			this->search_radius = search_radius;
			this->search_step = search_step;
		}
		void createICGN(int subset_radius_x, int subset_radius_y, float conv_criterion, float stop_condition)
		{
			icgn1 = std::make_unique<ICGN2D1>(subset_radius_x, subset_radius_y, conv_criterion, stop_condition, thread_number);
			icgn_conv = conv_criterion;
			icgn_stop = stop_condition;
		}
		void prepareICGN()
		{
			icgn1->setImages(*ref_img, *tar_img);
			icgn1->prepare();
		}
		void destoryICGN()
		{
			if (icgn1 != nullptr) icgn1.reset();
		}
		void setParallax(Point2D parallax)
		{
			this->parallax = parallax;
			parallax_x[0] = 0; parallax_x[1] = 0; parallax_x[2] = parallax.x;
			parallax_y[0] = 0; parallax_y[1] = 0; parallax_y[2] = parallax.y;
		}
		void setParallax(float coefficient_x[3], float coefficient_y[3])
		{
			for (int i = 0; i < 3; i++) { parallax_x[i] = coefficient_x[i]; parallax_y[i] = coefficient_y[i]; }
		}
		void updateCameras(Calibration& view1_cam, Calibration& view2_cam)
		{
			this->view1_cam = view1_cam;
			this->view2_cam = view2_cam;
		}
		void updateFundementalMatrix() { b200::fundamentalMatrix(view1_cam, view2_cam, fundamental_matrix); } // src/oc_epipolar_search.cpp:110-126
		void prepare()
		{
			view1_cam.updateMatrices();
			view2_cam.updateMatrices();
			updateFundementalMatrix();
			prepareICGN();
		}
		void compute(POI2D* poi) { run(poi, 1); }
		void compute(std::vector<POI2D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

	private:
		float icgn_conv = 0.001f, icgn_stop = 10.f;
		void run(POI2D* p, size_t n)
		{
			if (icgn1 == nullptr) throw std::string("opencorr_b200: createICGN() and prepare() must be called before compute()");
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			icgn1->bindLocked(e);
			e.check(ocb_epipolar_search2d(e.context(), p, n, fundamental_matrix, parallax_x, parallax_y, search_radius, search_step, icgn1->subset_radius_x,
				icgn1->subset_radius_y, icgn_conv, icgn_stop));
		}
	};

	class ICGN3D1 : public DVC
	{
	private:
		float conv_criterion;
		float stop_condition;
		b200::Prepared prepared;

	public:
		ICGN3D1(int subset_radius_x, int subset_radius_y, int subset_radius_z, float conv_criterion, float stop_condition, int thread_number)
		{
			this->subset_radius_x = subset_radius_x;
			this->subset_radius_y = subset_radius_y;
			this->subset_radius_z = subset_radius_z;
			this->conv_criterion = conv_criterion;
			this->stop_condition = stop_condition;
			this->thread_number = thread_number;
		}
		~ICGN3D1() {}
		void setIteration(float conv_criterion, float stop_condition)
		{
			this->conv_criterion = conv_criterion;
			this->stop_condition = stop_condition;
		}
		void setIteration(POI3D* poi) // src/oc_icgn.cpp:1234-1238
		{
			conv_criterion = poi->result.convergence;
			stop_condition = (float)(int)poi->result.iteration;
		}
		void prepareRef() { prepare(); }
		void prepareTar() { prepare(); }
		void prepare()
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			prepared.prepare(e, ref_img, tar_img, ocb_icgn3d_prepare);
		}
		void compute(POI3D* poi) { run(poi, 1); }
		void compute(std::vector<POI3D>& poi_queue) { run(poi_queue.data(), poi_queue.size()); }

	private:
		void run(POI3D* p, size_t n)
		{
			b200::Engine& e = b200::Engine::get();
			std::lock_guard<std::mutex> g(e.lock);
			prepared.bind(e, ref_img, tar_img, ocb_icgn3d_prepare);
			e.check(ocb_icgn3d1(e.context(), p, n, subset_radius_x, subset_radius_y, subset_radius_z, conv_criterion, stop_condition));
		}
	};

	// ------------------------------------------------------------------ fast "%.8f" table writer (not in the reference)
	// The reference writes tables with `ofstream << setprecision(8) << fixed`, one number at a time
	// (src/oc_io.cpp:320-322); at GPU speed that becomes the slowest stage of a run (500 k rows x 15
	// numbers).  This buffer produces byte-identical text with std::to_chars (C++17) or snprintf.
	namespace b200
	{
		class TableWriter
		{
			std::string buf;
			std::string delim;

		public:
			explicit TableWriter(const std::string& delimiter) : delim(delimiter) { buf.reserve(1 << 20); }
			inline void text(const char* t) { buf.append(t); buf.append(delim); }
			inline void num(float v)
			{
				char tmp[64];
#if __cplusplus >= 201703L && defined(__cpp_lib_to_chars)
				auto r = std::to_chars(tmp, tmp + sizeof(tmp), (double)v, std::chars_format::fixed, 8);
				buf.append(tmp, r.ptr - tmp);
#else
				int n = std::snprintf(tmp, sizeof(tmp), "%.8f", (double)v);
				buf.append(tmp, (size_t)n);
#endif
				buf.append(delim);
			}
			inline void endRow() { buf.push_back('\n'); }
			inline bool save(const std::string& path)
			{
				std::ofstream out(path, std::ios::binary);
				if (!out.is_open()) return false;
				out.write(buf.data(), (std::streamsize)buf.size());
				return true;
			}
		};
	} // namespace b200

	// ------------------------------------------------------------------ src/oc_io.h (subset used by the two examples)
	enum OutputVariable
	{
		u = 1, v = 2, w = 3, e_xx = 4, e_yy = 5, e_zz = 6, e_xy = 7, e_yz = 8, e_zx = 9, zncc = 10, zncc_r1r2 = 11, zncc_r1t2 = 12,
		deformation_increment = 13, iteration_step = 14, feature_nearby = 15, u_x = 16, u_y = 17, u_z = 18, v_x = 19, v_y = 20, v_z = 21,
		w_x = 22, w_y = 23, w_z = 24,
	};

	namespace b200
	{
		// Reads the numeric rows of a delimiter-separated table written by saveTable2D/saveTable3D (header line skipped;
		// empty fields skipped like the reference's loaders, src/oc_io.cpp:264-283).  Rows shorter than `min_cols` are
		// padded with zeros: the result tables shipped with the reference predate the subset_rx/ry(/rz) columns.
		inline std::vector<std::vector<float>> readTable(const std::string& file_path, const std::string& delimiter, size_t min_cols)
		{
			std::ifstream file_in(file_path);
			if (!file_in.is_open()) throw std::string("failed to open csv file " + file_path);
			std::vector<std::vector<float>> rows;
			std::string line;
			std::getline(file_in, line);
			while (std::getline(file_in, line)) {
				if (!line.empty() && line.back() == '\r') line.pop_back();
				std::vector<float> key_buffer;
				size_t position1 = 0, position2 = 0;
				do {
					position2 = line.find(delimiter, position1);
					if (position2 == std::string::npos) position2 = line.length();
					const std::string variable = line.substr(position1, position2 - position1);
					if (!variable.empty()) key_buffer.push_back(std::stof(variable));
					position1 = position2 + delimiter.length();
				} while (position2 < line.length() && position1 < line.length());
				if (key_buffer.empty()) continue;
				if (key_buffer.size() < min_cols) key_buffer.resize(min_cols, 0.f);
				rows.push_back(std::move(key_buffer));
			}
			return rows;
		}
	} // namespace b200

	class IO2D
	{
	private:
		std::string file_path;
		std::string delimiter = ",";
		int width = 0, height = 0;

	public:
		IO2D() {}
		~IO2D() {}
		OutputVariable out_var;
		std::string getPath() const { return file_path; }
		std::string getDelimiter() const { return delimiter; }
		int getWidth() const { return width; }
		int getHeight() const { return height; }
		void setPath(std::string file_path) { this->file_path = file_path; }
		void setDelimiter(std::string delimiter) { this->delimiter = delimiter; }
		void setWidth(int width) { this->width = width; }
		void setHeight(int height) { this->height = height; }

		// src/oc_io.cpp:249-316
		std::vector<POI2D> loadTable2D()
		{
			std::vector<POI2D> poi_queue;
			for (const std::vector<float>& k : b200::readTable(file_path, delimiter, 15)) {
				POI2D poi(k[0], k[1]);
				poi.deformation.u = k[2];
				poi.deformation.v = k[3];
				for (int i = 0; i < 6; i++) poi.result.r[i] = k[4 + i];
				for (int i = 0; i < 3; i++) poi.strain.e[i] = k[10 + i];
				poi.subset_radius.x = k[13];
				poi.subset_radius.y = k[14];
				poi_queue.push_back(poi);
			}
			return poi_queue;
		}
		// src/oc_io.cpp:506-584
		std::vector<POI2DS> loadTable2DS()
		{
			std::vector<POI2DS> poi_queue;
			for (const std::vector<float>& k : b200::readTable(file_path, delimiter, 28)) {
				POI2DS poi(k[0], k[1]);
				for (int i = 0; i < 3; i++) poi.deformation.p[i] = k[2 + i];
				for (int i = 0; i < 9; i++) poi.result.r[i] = k[5 + i];
				poi.ref_coor.x = k[14]; poi.ref_coor.y = k[15]; poi.ref_coor.z = k[16];
				poi.tar_coor.x = k[17]; poi.tar_coor.y = k[18]; poi.tar_coor.z = k[19];
				for (int i = 0; i < 6; i++) poi.strain.e[i] = k[20 + i];
				poi.subset_radius.x = k[26];
				poi.subset_radius.y = k[27];
				poi_queue.push_back(poi);
			}
			return poi_queue;
		}
		// src/oc_io.cpp:586-670
		void saveTable2DS(std::vector<POI2DS>& poi_queue)
		{
			b200::TableWriter t(delimiter);
			const char* head[] = { "x", "y", "u", "v", "w", "r1r2 ZNCC", "r1t1 ZNCC", "r1t2 ZNCC", "r2_x", "r2_y", "t1_x", "t1_y", "t2_x", "t2_y", "ref_x", "ref_y",
				"ref_z", "tar_x", "tar_y", "tar_z", "exx", "eyy", "ezz", "exy", "eyz", "ezx", "subset_rx", "subset_ry" };
			for (const char* h : head) t.text(h);
			t.endRow();
			for (auto iter = poi_queue.begin(); iter != poi_queue.end(); iter++) {
				t.num(iter->x); t.num(iter->y);
				for (int i = 0; i < 3; i++) t.num(iter->deformation.p[i]);
				for (int i = 0; i < 9; i++) t.num(iter->result.r[i]);
				t.num(iter->ref_coor.x); t.num(iter->ref_coor.y); t.num(iter->ref_coor.z);
				t.num(iter->tar_coor.x); t.num(iter->tar_coor.y); t.num(iter->tar_coor.z);
				for (int i = 0; i < 6; i++) t.num(iter->strain.e[i]);
				t.num(iter->subset_radius.x); t.num(iter->subset_radius.y);
				t.endRow();
			}
			t.save(file_path);
		}
		// src/oc_io.cpp:318-373
		void saveTable2D(std::vector<POI2D>& poi_queue)
		{
			b200::TableWriter t(delimiter);
			const char* head[] = { "x", "y", "u", "v", "u0", "v0", "ZNCC", "iteration", "convergence", "feature", "exx", "eyy", "exy", "subset_rx", "subset_ry" };
			for (const char* h : head) t.text(h);
			t.endRow();
			for (auto iter = poi_queue.begin(); iter != poi_queue.end(); iter++) {
				t.num(iter->x); t.num(iter->y);
				t.num(iter->deformation.u); t.num(iter->deformation.v);
				for (int i = 0; i < 6; i++) t.num(iter->result.r[i]);
				for (int i = 0; i < 3; i++) t.num(iter->strain.e[i]);
				t.num(iter->subset_radius.x); t.num(iter->subset_radius.y);
				t.endRow();
			}
			t.save(file_path);
		}
		// src/oc_io.cpp:375-421
		void saveDeformationTable2D(std::vector<POI2D>& poi_queue)
		{
			b200::TableWriter t(delimiter);
			const char* head[] = { "x", "y", "u", "ux", "uy", "uxx", "uxy", "uyy", "v", "vx", "vy", "vxx", "vxy", "vyy", "subset_rx", "subset_ry" };
			for (const char* h : head) t.text(h);
			t.endRow();
			for (auto iter = poi_queue.begin(); iter != poi_queue.end(); iter++) {
				t.num(iter->x); t.num(iter->y);
				for (int i = 0; i < 12; i++) t.num(iter->deformation.p[i]);
				t.num(iter->subset_radius.x); t.num(iter->subset_radius.y);
				t.endRow();
			}
			t.save(file_path);
		}
		// src/oc_io.cpp:423-504
		void saveMap2D(std::vector<POI2D>& poi_queue, OutputVariable variable)
		{
			std::vector<float> output_map((size_t)height * width, 0.f);
			for (size_t i = 0; i < poi_queue.size(); i++) {
				const POI2D& p = poi_queue[i];
				float val;
				switch (variable) {
				case u: val = p.deformation.u; break;
				case v: val = p.deformation.v; break;
				case zncc: val = p.result.zncc; break;
				case deformation_increment: val = p.result.convergence; break;
				case iteration_step: val = p.result.iteration; break;
				case feature_nearby: val = p.result.feature; break;
				case e_xx: val = p.strain.exx; break;
				case e_yy: val = p.strain.eyy; break;
				case e_xy: val = p.strain.exy; break;
				default: return;
				}
				output_map[(size_t)(int)p.y * width + (int)p.x] = val;
			}
			b200::TableWriter t(delimiter);
			for (int r = 0; r < height; r++) {
				for (int c = 0; c < width; c++) t.num(output_map[(size_t)r * width + c]);
				t.endRow();
			}
			t.save(file_path);
		}
	};

	class IO3D
	{
	private:
		std::string file_path;
		std::string delimiter;
		int dim_x = 0, dim_y = 0, dim_z = 0;

	public:
		IO3D() {}
		~IO3D() {}
		std::string getPath() const { return file_path; }
		std::string getDelimiter() const { return delimiter; }
		void setPath(std::string file_path) { this->file_path = file_path; }
		void setDelimiter(std::string delimiter) { this->delimiter = delimiter; }
		int getDimX() { return dim_x; }
		int getDimY() { return dim_y; }
		int getDimZ() { return dim_z; }
		void setDimX(int dim_x) { this->dim_x = dim_x; }
		void setDimY(int dim_y) { this->dim_y = dim_y; }
		void setDimZ(int dim_z) { this->dim_z = dim_z; }

		// src/oc_io.cpp:920-1002
		std::vector<POI3D> loadTable3D()
		{
			std::vector<POI3D> poi_queue;
			for (const std::vector<float>& k : b200::readTable(file_path, delimiter, 31)) {
				POI3D poi(k[0], k[1], k[2]);
				poi.deformation.u = k[3];
				poi.deformation.v = k[4];
				poi.deformation.w = k[5];
				for (int i = 0; i < 7; i++) poi.result.r[i] = k[6 + i];
				poi.deformation.ux = k[13]; poi.deformation.uy = k[14]; poi.deformation.uz = k[15];
				poi.deformation.vx = k[16]; poi.deformation.vy = k[17]; poi.deformation.vz = k[18];
				poi.deformation.wx = k[19]; poi.deformation.wy = k[20]; poi.deformation.wz = k[21];
				for (int i = 0; i < 6; i++) poi.strain.e[i] = k[22 + i];
				poi.subset_radius.x = k[28];
				poi.subset_radius.y = k[29];
				poi.subset_radius.z = k[30];
				poi_queue.push_back(poi);
			}
			return poi_queue;
		}
		// src/oc_io.cpp:1004-1089
		void saveTable3D(std::vector<POI3D>& poi_queue)
		{
			b200::TableWriter t(delimiter);
			const char* head[] = { "x", "y", "z", "u", "v", "w", "u0", "v0", "w0", "ZNCC", "iteration", "convergence", "feature",
				"ux", "uy", "uz", "vx", "vy", "vz", "wx", "wy", "wz", "exx", "eyy", "ezz", "exy", "eyz", "ezx", "subset_rx", "subset_ry", "subset_rz" };
			for (const char* h : head) t.text(h);
			t.endRow();
			for (auto iter = poi_queue.begin(); iter != poi_queue.end(); iter++) {
				t.num(iter->x); t.num(iter->y); t.num(iter->z);
				t.num(iter->deformation.u); t.num(iter->deformation.v); t.num(iter->deformation.w);
				for (int i = 0; i < 7; i++) t.num(iter->result.r[i]);
				t.num(iter->deformation.ux); t.num(iter->deformation.uy); t.num(iter->deformation.uz);
				t.num(iter->deformation.vx); t.num(iter->deformation.vy); t.num(iter->deformation.vz);
				t.num(iter->deformation.wx); t.num(iter->deformation.wy); t.num(iter->deformation.wz);
				for (int i = 0; i < 6; i++) t.num(iter->strain.e[i]);
				t.num(iter->subset_radius.x); t.num(iter->subset_radius.y); t.num(iter->subset_radius.z);
				t.endRow();
			}
			t.save(file_path);
		}
	};

} // namespace opencorr

#endif // _OPENCORR_B200_SHIM_H_
