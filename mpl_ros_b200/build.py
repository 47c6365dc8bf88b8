"""In-tree build of libmplb.so for sm_90a (H100; nvcc cross-compiles without a GPU).

One object per translation unit (kept next to the sources, git-ignored), linked into mpl_ros_b200/libmplb.so; a unit is
recompiled only when it or one of its headers is newer than its object."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INC = os.path.join(HERE, "..", "include", "mplb.h")
SRC = os.path.join(CSRC, "mplb.cu")  # the search runtime
_COMMON = [INC, os.path.join(CSRC, "mplb_internal.h")]
UNITS = {
    "mplb.cu": [os.path.join(CSRC, h) for h in ("mplb_search.cuh", "mplb_device.cuh", "mplb_trig.cuh", "mplb_ref.h")] + _COMMON,
    "mplb_trajsolve.cu": [os.path.join(CSRC, "mplb_ref.h")] + _COMMON,
    "mplb_lpa.cu": [os.path.join(CSRC, h) for h in ("mplb_lpa_core.h", "mplb_ref.h")] + _COMMON,
    "mplb_voxel.cu": [os.path.join(CSRC, "mplb_ref.h")] + _COMMON,
    "mplb_fleet.cu": _COMMON,
}
DEPS = [SRC] + UNITS["mplb.cu"]
OUT = os.path.join(HERE, "libmplb.so")

# -fmad=false: the reference is built without FMA contraction (MPL/CMakeLists.txt:5-8); the kernels also use
# explicit __d*_rn intrinsics, the flag covers whatever remains.  -ffp-contract=off does the same for the host half of
# mplb_ref.h's functions (prior-trajectory table, search-region builder), as in the host build of the LPA* core.
ARCH_FLAGS = ["-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-fmad=false",
              "-Xcompiler", "-ffp-contract=off"]
NVCC_FLAGS = ["-shared", "-Xcompiler", "-fPIC"] + ARCH_FLAGS


def _newer(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(target) < os.path.getmtime(d) for d in deps)


def build_lib(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs, relink = [], force or not os.path.exists(OUT)
    for unit, deps in UNITS.items():
        src = os.path.join(CSRC, unit)
        if not os.path.exists(src):
            continue
        obj = src[:-3] + ".o"
        objs.append(obj)
        deps = [src] + [d for d in deps if os.path.exists(d)]
        if os.path.exists(OUT) and not force and not _newer(OUT, deps):
            if not os.path.exists(obj):
                objs[-1] = None  # the library is current; this unit's object was not shipped — relink would need it
            continue
        if force or _newer(obj, deps):
            subprocess.check_call([nvcc, "-c", "-Xcompiler", "-fPIC"] + ARCH_FLAGS +
                                  (["-Xptxas", "-v"] if verbose else []) + ["-o", obj, src])
        relink = True
    if not relink:
        return OUT
    for i, obj in enumerate(objs):  # a relink needs every object: compile the ones that are missing
        if obj is None:
            unit = list(u for u in UNITS if os.path.exists(os.path.join(CSRC, u)))[i]
            src = os.path.join(CSRC, unit)
            obj = objs[i] = src[:-3] + ".o"
            subprocess.check_call([nvcc, "-c", "-Xcompiler", "-fPIC"] + ARCH_FLAGS + ["-o", obj, src])
    tmp = OUT + ".tmp"
    subprocess.check_call([nvcc, "-shared", "-Xcompiler", "-fPIC"] + ARCH_FLAGS + ["-o", tmp] + objs)
    os.replace(tmp, OUT)  # rename: a process that has the old file mapped keeps it
    return OUT
