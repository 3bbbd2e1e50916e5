// Strain::compute(POI2D*, queue) -- the single-POI overload of the reference's Strain (src/oc_strain.cpp:158-237) -- on the C++
// shim: read a POI2D queue (raw 100-byte records), compute the strain of one POI and write the queue back.
//   strain_single_shim_test <in.bin> <out.bin> <index> <radius> <neighbor_min> <zncc_threshold> <approximation>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <vector>

#include "opencorr.h"

using namespace opencorr;
using namespace std;

int main(int argc, char** argv)
{
	if (argc != 8) {
		cerr << "usage: strain_single_shim_test <in.bin> <out.bin> <index> <radius> <neighbor_min> <zncc_threshold> <approximation>" << endl;
		return 2;
	}
	try {
		ifstream in(argv[1], ios::binary | ios::ate);
		const size_t n = (size_t)in.tellg() / sizeof(POI2D);
		in.seekg(0);
		vector<POI2D> poi_queue(n, POI2D(0.f, 0.f));
		in.read(reinterpret_cast<char*>(poi_queue.data()), n * sizeof(POI2D));

		Strain* strain = new Strain((float)atof(argv[4]), atoi(argv[5]), 1);
		strain->setZnccThreshold((float)atof(argv[6]));
		strain->setApproximation(atoi(argv[7]));
		strain->prepare(poi_queue);
		strain->compute(&poi_queue[(size_t)atol(argv[3])], poi_queue);
		delete strain;

		ofstream out(argv[2], ios::binary);
		out.write(reinterpret_cast<const char*>(poi_queue.data()), n * sizeof(POI2D));
	} catch (const string& e) {
		cerr << e << endl;
		return 1;
	}
	return 0;
}
