"""opencorr_b200 -- H100-native (sm_90a) FFT-CC -> IC-GN correlation engine behind OpenCorr's API.

Only the hot path of vincentjzy/OpenCorr is implemented: FFTCC2D/FFTCC3D and
ICGN2D1/ICGN2D2/ICGN3D1.  The compute lives in opencorr_b200/csrc (CUDA) behind the C ABI of
include/opencorr_b200.h; this package is the Python mirror of the reference's operator interface.
"""
from ._capi import OpenCorrB200Error, LIB_PATH  # noqa: F401
from .api import (Calibration, Engine, EpipolarSearch, FFTCC2D, FFTCC3D, ICGN2D1, ICGN2D2, ICGN3D1, ICLM2D1, ICLM2D2, NR2D1, Strain, P2, P3, POI2D_FLOATS,  # noqa: F401
                  POI3D_FLOATS, RegionFit2D, RegionFit3D, SIFT3D, SIFT3D_DEFAULT_CONFIG, Stereovision, default_engine, make_poi2d, make_poi3d)
