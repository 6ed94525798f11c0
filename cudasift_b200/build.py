"""Build recipes for cudasift_b200 (no build system: plain nvcc / gcc command lines).

build_library()  -> cudasift_b200/lib/libcudasift_b200.so   (the product, sm_90a only)
build_library(managed=True) -> cudasift_b200/lib/libcudasift_b200_managed.so  (the MANAGEDMEM flavour of the API,
                    cudaSift.h:35-40: SiftData::m_data in unified memory)
build_oracle()   -> oracle/liboracle.so                      (CPU checker, test infrastructure)
build_reference()-> oracle/_ref/libcudasift_ref.so           (the unmodified reference, compiled where its
                    sources lie: CUDASIFT_REFERENCE_SRC, else a `reference` checkout beside this
                    repository; see oracle/build_reference.py)

All outputs are git-ignored.
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cudasift_b200", "csrc")
LIBDIR = os.path.join(ROOT, "cudasift_b200", "lib")
LIB = os.path.join(LIBDIR, "libcudasift_b200.so")
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liboracle.so")
REF_DIR = os.path.join(ORACLE_DIR, "_ref")
REF_LIB = os.path.join(REF_DIR, "libcudasift_ref.so")

SOURCES = ["api.cu", "pipeline2.cu", "pyramid.cu", "pyramid2.cu", "detect.cu", "detect2.cu", "cap32.cu", "describe.cu",
           "match.cu", "match_tc.cu", "homography.cu", "geom.cu", "rank.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-O2,-Wall", "-shared"]


def _newer(target, deps):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps if os.path.exists(d))


def _run(cmd, **kw):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("command failed: " + " ".join(cmd))
    return r.stdout


def nvcc_path():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


LIB_MANAGED = os.path.join(LIBDIR, "libcudasift_b200_managed.so")
MANAGED_UNITS = ("api.cu", "homography.cu", "geom.cu")     # the translation units that look at MANAGEDMEM
OBJDIR = os.path.join(LIBDIR, "obj")


def build_library(force=False, verbose=False, managed=False):
    """Every translation unit to its own object (in parallel, rebuilt when a source or header is newer), one link."""
    from concurrent.futures import ThreadPoolExecutor
    lib = LIB_MANAGED if managed else LIB
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    hdrs = [os.path.join(CSRC, h) for h in ("common.cuh", "tma.cuh", "pipeline2.h")] + [
        os.path.join(ROOT, "include", h) for h in ("cudaSift.h", "cudaImage.h", "cudasift_b200.h")]
    if not force and _newer(lib, srcs + hdrs):
        return lib
    nvcc = nvcc_path()
    if nvcc is None:
        if os.path.exists(lib):
            return lib   # GPU box without a toolkit: use the prebuilt library that travelled
        raise RuntimeError("nvcc not found and no prebuilt " + os.path.basename(lib))
    os.makedirs(OBJDIR, exist_ok=True)
    flags = [f for f in NVCC_FLAGS if f != "-shared"] + (["-Xptxas", "-v"] if verbose else [])

    def compile_unit(name):
        tag = "_managed" if managed and name in MANAGED_UNITS else ""
        obj = os.path.join(OBJDIR, name.replace(".cu", tag + ".o"))
        src = os.path.join(CSRC, name)
        if force or not _newer(obj, [src] + hdrs):
            out = _run([nvcc] + flags + (["-DMANAGEDMEM"] if tag else []) + ["-c", src, "-o", obj])
            if verbose:
                print(out)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(compile_unit, SOURCES))
    _run([nvcc] + ARCH + ["-shared"] + objs + ["-o", lib])
    return lib


def build_oracle(force=False):
    src = os.path.join(ORACLE_DIR, "sift_oracle.c")
    if not force and _newer(ORACLE_LIB, [src, os.path.join(ORACLE_DIR, "sift_oracle.h")]):
        return ORACLE_LIB
    if shutil.which("gcc") is None:
        if os.path.exists(ORACLE_LIB):
            return ORACLE_LIB
        raise RuntimeError("gcc not found and no prebuilt liboracle.so")
    _run(["gcc", "-O2", "-mfma", "-ffp-contract=off", "-fPIC", "-shared", "-o", ORACLE_LIB, src, "-lm", "-lpthread"])
    return ORACLE_LIB


def build_reference(force=False):
    """The unmodified reference in oracle/_ref/ (recipe: oracle/build_reference.py)."""
    sys.path.insert(0, ROOT)
    from oracle.build_reference import build_reference as b
    return b(nvcc_path(), force)


DEMO = os.path.join(LIBDIR, "sift_demo")
DEMO_MANAGED = os.path.join(LIBDIR, "sift_demo_managed")


def build_demo(force=False, managed=False):
    """examples/sift_demo.cpp: a plain g++ caller of the drop-in headers, linked against the library
    (managed=True: compiled with -DMANAGEDMEM against the unified-memory flavour)."""
    src = os.path.join(ROOT, "examples", "sift_demo.cpp")
    lib = build_library(managed=managed)
    demo = DEMO_MANAGED if managed else DEMO
    if not force and _newer(demo, [src, lib]):
        return demo
    if shutil.which("g++") is None:
        return demo if os.path.exists(demo) else None
    _run(["g++", "-O2", "-std=c++17", "-Wall"] + (["-DMANAGEDMEM"] if managed else []) +
         ["-I" + os.path.join(ROOT, "include"), src, "-L" + LIBDIR,
          "-lcudasift_b200_managed" if managed else "-lcudasift_b200", "-lz", "-Wl,-rpath,$ORIGIN", "-o", demo])
    return demo


def build_all(force=False, verbose=False):
    out = build_library(force, verbose), build_oracle(force), build_reference(force), build_demo(force)
    build_library(force, verbose, managed=True)
    build_demo(force, managed=True)
    return out


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
