"""In-tree build of the CUDA extension (sm_90a, Hopper H100, only).

    python -m yolact_b200.build            # incremental
    python -m yolact_b200.build --force

Produces yolact_b200/libyolact_b200.so (C ABI of include/yolact_b200.h).  nvcc cross-compiles
without a GPU; the .so and the objects are build products (git-ignored).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "build")
LIB = os.path.join(HERE, "libyolact_b200.so")

SOURCES = ["capi.cu", "engine.cu", "tc_conv.cu", "stem_tc.cu", "simt_conv.cu", "pointwise.cu", "detect.cu", "mask.cu", "dcn.cu", "dcn_tc.cu", "dcn_pool.cu", "evalops.cu", "evalmap.cu", "render.cu", "cocorle.cu", "evaliou.cu", "plans.cu"]
HEADERS = ["common.cuh", "kernels.cuh", "engine.cuh", "tc_common.cuh", "mask_math.cuh", "staged_mask.cuh", os.path.join(ROOT, "include", "yolact_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-std=c++17", "-O3", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
]


# the one source that embeds the build id (yb_build_id, the plan file's `build` field)
BUILD_ID_SOURCE = "plans.cu"


def build_id(flags=NVCC_FLAGS):
    """Hash of every compiled source, header and compiler flag: plan files written by one library are refused by a
    library built from anything else."""
    h = hashlib.sha256()
    for f in list(flags) + ["--"]:
        h.update(f.encode() + b"\0")
    for name in SOURCES + HEADERS:
        path = name if os.path.isabs(name) else os.path.join(CSRC, name)
        h.update(os.path.basename(path).encode() + b"\0")
        with open(path, "rb") as fp:
            h.update(hashlib.sha256(fp.read()).digest())
    return h.hexdigest()[:16]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _newer(path, deps):
    if not os.path.exists(path):
        return True
    t = os.path.getmtime(path)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, watchdog=False):
    """watchdog=True builds libyolact_b200_wd.so with -DYB_WATCHDOG (mbarrier waits trap after ~2 s instead of
    hanging the GPU): the library to point YB_LIB at while a new kernel protocol is being brought up."""
    global OBJ, LIB
    flags = list(NVCC_FLAGS)
    obj_dir, lib = OBJ, LIB
    if watchdog:
        flags.append("-DYB_WATCHDOG")
        obj_dir = OBJ + "_wd"
        lib = os.path.join(HERE, "libyolact_b200_wd.so")
    return _build(force, verbose, flags, obj_dir, lib)


def _build(force, verbose, NVCC_FLAGS, OBJ, LIB):
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    hdrs = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    objs = []
    srcs = [os.path.join(CSRC, src) for src in SOURCES]
    for src, s in zip(SOURCES, srcs):
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(o)
        flags, deps = NVCC_FLAGS, [s] + hdrs
        if src == BUILD_ID_SOURCE:   # rebuilt whenever anything the id hashes changes
            flags, deps = NVCC_FLAGS + ['-DYB_BUILD_ID="%s"' % build_id(NVCC_FLAGS)], srcs + hdrs
        if force or _newer(o, deps):
            jobs.append([nvcc] + flags + ["-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout)
        return r.stdout

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    if force or jobs or _newer(LIB, objs):
        # C ABI symbols are the only exported ones (visibility=hidden + extern "C" default)
        run([nvcc, "-shared", "-o", LIB] + objs + ["-cudart", "static", "-Xcompiler", "-fPIC",
                                                  "-Xlinker", "--no-undefined", "-lpthread", "-ldl", "-lrt"])
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True, watchdog="--watchdog" in sys.argv)
    print("built", p)
