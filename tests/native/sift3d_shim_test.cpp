// The SIFT3D half of the reference's examples/test_dvc_sift_icgn1.cpp (:81-110) on the C++ shim: load a volume pair (.bin),
// extract and match 3D SIFT features, and write <target>_matched_kp.csv in that example's format.
//   sift3d_shim_test <ref.bin> <tar.bin>
#include <fstream>
#include <iostream>

#include "opencorr.h"

using namespace opencorr;
using namespace std;

int main(int argc, char** argv)
{
	if (argc != 3) {
		cerr << "usage: sift3d_shim_test <ref.bin> <tar.bin>" << endl;
		return 2;
	}
	try {
		string ref_image_path = argv[1], tar_image_path = argv[2];
		Image3D ref_img(ref_image_path);
		Image3D tar_img(tar_image_path);
		string delimiter = ",";

		SIFT3D* sift = new SIFT3D();
		sift->setImages(ref_img, tar_img);
		sift->prepare();
		sift->compute();

		int kp_amount = (int)sift->ref_matched_kp.size();
		cout << "Extraction and matching of " << kp_amount << " 3D SIFT features." << endl;

		string file_path = tar_image_path.substr(0, tar_image_path.find_last_of(".")) + "_matched_kp.csv";
		ofstream csv_out(file_path);
		if (csv_out.is_open()) {
			csv_out << "x_ref" << delimiter << "y_ref" << delimiter << "z_ref" << delimiter << "x_tar" << delimiter << "y_tar" << delimiter << "z_tar" << endl;
			for (int i = 0; i < kp_amount; i++) csv_out << sift->ref_matched_kp[i] << delimiter << sift->tar_matched_kp[i] << endl;
		}
		csv_out.close();
		delete sift;
		ref_img.release();
		tar_img.release();
	} catch (const string& e) {
		cerr << e << endl;
		return 1;
	}
	return 0;
}
