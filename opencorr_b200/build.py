"""Build the sm_90a shared library in-tree: opencorr_b200/lib/libopencorr_b200.so.

nvcc cross-compiles without a GPU.  The library is a plain C-ABI .so (static cudart, no torch).
"""
import glob
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libopencorr_b200.so")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper)
NVCC_FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC"]
# per-source additions: SIFT3D reproduces the float32 oracle bit for bit, so no multiply-add is contracted into an FMA
SOURCE_FLAGS = {"sift3d.cu": ["-fmad=false"]}


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libopencorr_b200.so")


def sources():
    csrc = os.path.join(_HERE, "csrc")
    return sorted(glob.glob(os.path.join(csrc, "*.cu"))), sorted(
        glob.glob(os.path.join(csrc, "*.cuh")) + glob.glob(os.path.join(csrc, "*.h"))
        + [os.path.join(_HERE, "..", "include", "opencorr_b200.h")])


def is_stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    cu, hdr = sources()
    return any(os.path.exists(p) and os.path.getmtime(p) > t for p in cu + hdr)


def _compile(nvcc, flags, src, obj):
    subprocess.check_call(nvcc + flags + ["-c", "-o", obj, src])
    return obj


def build(force=False, verbose=False, variant=None, variant_flags=(), variant_sources=()):
    """Compile every CUDA source for sm_90a into one shared library (objects in parallel, then one link).  Objects are kept
    under lib/obj/ so that only stale sources are recompiled.

    variant: build lib/variants/<variant>.so instead (A/B experiments, selected at run time with OCB_LIB_PATH): the
    sources named in variant_sources are compiled with variant_flags added (e.g. -DNAME=VALUE for a macro an experiment
    tests), the rest is linked from the regular objects."""
    if variant is None and not force and not is_stale():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    cu, hdr = sources()
    nvcc = [_nvcc()]
    # the image's CXX points at a gcc without OpenMP specs; nvcc only needs a host g++
    if os.path.exists("/usr/bin/g++"):
        nvcc += ["-ccbin", "/usr/bin/g++"]
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    compile_flags = [f for f in NVCC_FLAGS if f != "-shared"] + (["-Xptxas", "-v"] if verbose else [])
    newest_hdr = max([os.path.getmtime(p) for p in hdr if os.path.exists(p)] + [os.path.getmtime(__file__)])
    jobs, objs = [], []
    for src in cu:
        base = os.path.basename(src)
        if variant is not None and base in variant_sources:
            vdir = os.path.join(obj_dir, variant)
            os.makedirs(vdir, exist_ok=True)
            obj = os.path.join(vdir, base[:-3] + ".o")
            jobs.append((compile_flags + SOURCE_FLAGS.get(base, []) + list(variant_flags), src, obj))
        else:
            obj = os.path.join(obj_dir, base[:-3] + ".o")
            stale = not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), newest_hdr)
            if stale or (force and variant is None) or verbose:
                jobs.append((compile_flags + SOURCE_FLAGS.get(base, []), src, obj))
        objs.append(obj)
    from concurrent.futures import ThreadPoolExecutor
    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as pool:
            list(pool.map(lambda j: _compile(nvcc, *j), jobs))
    out = LIB_PATH
    if variant is not None:
        os.makedirs(os.path.join(LIB_DIR, "variants"), exist_ok=True)
        out = os.path.join(LIB_DIR, "variants", variant + ".so")
    subprocess.check_call(nvcc + GENCODE + ["-shared", "-Xcompiler", "-fPIC", "-o", out] + objs)
    return out


if __name__ == "__main__":
    import sys
    if "--variant" in sys.argv:  # python -m opencorr_b200.build --variant NAME --sources a.cu,b.cu -- -DFLAG=1 ...
        i = sys.argv.index("--variant")
        srcs = sys.argv[sys.argv.index("--sources") + 1].split(",")
        flags = sys.argv[sys.argv.index("--") + 1:] if "--" in sys.argv else []
        print(build(variant=sys.argv[i + 1], variant_flags=flags, variant_sources=srcs))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
