// RegionFit2D / RegionFit3D on the C++ shim (the reference's src/oc_region_fit.h interface): read a reliable set and a queue
// (raw POI2D or POI3D records), run setNeighbor + prepare + compute and write the queue back.  index < 0: compute(queue); else
// compute(&queue[index]) alone.
//   region_fit_shim_test <2|3> <reliable.bin> <queue.bin> <out.bin> <radius> <neighbor_min> <index>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <vector>

#include "opencorr.h"

using namespace opencorr;
using namespace std;

template <class POI>
static vector<POI> read_pois(const char* path, const POI& blank)
{
	ifstream in(path, ios::binary | ios::ate);
	const size_t n = (size_t)in.tellg() / sizeof(POI);
	in.seekg(0);
	vector<POI> v(n, blank);
	in.read(reinterpret_cast<char*>(v.data()), n * sizeof(POI));
	return v;
}

template <class Fit, class POI>
static void run(char** argv, const POI& blank)
{
	vector<POI> reliable = read_pois(argv[2], blank), queue = read_pois(argv[3], blank);
	Fit* fit = new Fit((float)atof(argv[5]), atoi(argv[6]), 4);
	if (fit->getSearchRadius() != (float)atof(argv[5]) || fit->getNeighborMin() != atoi(argv[6])) throw string("getters disagree");
	fit->setSearchRadius(1.f); // the setters replace what the constructor set
	fit->setNeighborMin(1);
	fit->setSearchRadius((float)atof(argv[5]));
	fit->setNeighborMin(atoi(argv[6]));
	fit->setNeighbor(reliable);
	fit->prepare();
	const long index = atol(argv[7]);
	if (index < 0) fit->compute(queue);
	else fit->compute(&queue[(size_t)index]);
	delete fit;
	ofstream out(argv[4], ios::binary);
	out.write(reinterpret_cast<const char*>(queue.data()), queue.size() * sizeof(POI));
}

int main(int argc, char** argv)
{
	if (argc != 8) {
		cerr << "usage: region_fit_shim_test <2|3> <reliable.bin> <queue.bin> <out.bin> <radius> <neighbor_min> <index>" << endl;
		return 2;
	}
	try {
		if (atoi(argv[1]) == 3) run<RegionFit3D>(argv, POI3D(0.f, 0.f, 0.f));
		else run<RegionFit2D>(argv, POI2D(0.f, 0.f));
	} catch (const string& e) {
		cerr << e << endl;
		return 1;
	}
	return 0;
}
