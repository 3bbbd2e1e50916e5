"""The SIFT3D cases of tests/test_gpu_sift3d.py (checked against the oracle on the GPU) and tests/test_sift3d_plan_host.py (their
pyramid plans, on the host): name -> (dims (x, y, z), physical unit, config fields that differ from the defaults)."""
import numpy as np

import opencorr_b200 as ob
from opencorr_b200 import synth

CROP = "tests/golden/al_foam4_crop.npz"

CASES = {
    "al_foam4_crop": ((100, 100, 100), (1.0, 1.0, 1.0), {}),  # CROP
    "synthetic_120": ((120, 120, 120), (1.0, 1.0, 1.0), {}),
    "odd_101x77x130": ((101, 77, 130), (1.0, 1.0, 1.0), {}),
    "anisotropic_112x104x60": ((112, 104, 60), (1.0, 1.0, 2.0), {}),
    "two_octave_layers": ((96, 90, 84), (1.0, 1.0, 1.0), {"n_octave_layers": 2}),
    "mirror_clamp_128": ((128, 128, 128), (1.0, 1.0, 1.0), {}),  # top octave 8^3: blur radius 8 >= side
}


def crop():
    z = np.load(CROP)
    return z["ref"].astype(np.float32), z["tar"].astype(np.float32)


def volumes(name):
    """(ref, tar) float32 [z, y, x] of a case: the crop, or a synthetic pair whose target is displaced by synth.displacement_3d"""
    if name == "al_foam4_crop":
        return crop()
    ref, tar = synth.speckle_pair_3d(*CASES[name][0])
    return ref.astype(np.float32), tar.astype(np.float32)


def cfg(**kw):
    c = ob.SIFT3D_DEFAULT_CONFIG.copy()
    for k, v in kw.items():
        c[ob.api.SIFT3D_CONFIG_FIELDS.index(k)] = v
    return c
