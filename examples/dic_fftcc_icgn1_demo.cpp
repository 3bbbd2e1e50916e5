// dic_fftcc_icgn1_demo.cpp -- path-independent 2D DIC (FFT-CC initial guess + IC-GN, first-order
// shape function) on the H100 engine through the OpenCorr-compatible C++ shim.
// Usage: dic_fftcc_icgn1_demo <ref.bmp> <tar.bmp> <out.csv> [radius=16] [grid_step=2]
#include <chrono>
#include <iostream>
#include <string>
#include <vector>

#include "opencorr.h"

using namespace opencorr;

int main(int argc, char** argv)
{
	if (argc < 4) {
		std::cerr << "usage: " << argv[0] << " <ref.bmp> <tar.bmp> <out.csv> [radius=16] [grid_step=2]" << std::endl;
		return 2;
	}
	try {
		const int radius = argc > 4 ? std::atoi(argv[4]) : 16;
		const int step = argc > 5 ? std::atoi(argv[5]) : 2;
		Image2D ref_img(argv[1]);
		Image2D tar_img(argv[2]);

		std::vector<POI2D> poi_queue;
		const int margin = radius + 14;
		for (int y = margin; y < ref_img.height - margin; y += step)
			for (int x = margin; x < ref_img.width - margin; x += step)
				poi_queue.push_back(POI2D(Point2D(x, y)));

		auto t0 = std::chrono::steady_clock::now();
		FFTCC2D fftcc(radius, radius, 1);
		fftcc.setImages(ref_img, tar_img);
		fftcc.compute(poi_queue);
		auto t1 = std::chrono::steady_clock::now();
		ICGN2D1 icgn(radius, radius, 0.001f, 10, 1);
		icgn.setImages(ref_img, tar_img);
		icgn.prepare();
		icgn.compute(poi_queue);
		auto t2 = std::chrono::steady_clock::now();

		size_t converged = 0;
		for (const POI2D& p : poi_queue) converged += p.result.zncc >= 0.f;
		std::cout << poi_queue.size() << " POIs, " << converged << " converged; FFTCC "
			<< std::chrono::duration<double>(t1 - t0).count() << " s (includes context creation + image upload), ICGN "
			<< std::chrono::duration<double>(t2 - t1).count() << " s" << std::endl;

		IO2D in_out;
		in_out.setDelimiter(",");
		in_out.setHeight(ref_img.height);
		in_out.setWidth(ref_img.width);
		in_out.setPath(argv[3]);
		in_out.saveTable2D(poi_queue);
	} catch (const std::string& msg) {
		std::cerr << "error: " << msg << std::endl;
		return 1;
	}
	return 0;
}
