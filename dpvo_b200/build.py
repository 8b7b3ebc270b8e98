"""In-tree build of the sm_90a library and its torch-extension shims.

    python -m dpvo_b200.build            # build what is out of date
    python -m dpvo_b200.build --force    # rebuild everything

Products (git-ignored):
    dpvo_b200/lib/libdpvo_b200.so                  C-ABI library (nvcc, no torch dependency)
    dpvo_b200/_ext/{cuda_corr,cuda_ba,lietorch_backends,dpvo_b200_ext}<EXT_SUFFIX>
                                                   pybind shims, one object copied four times
nvcc cross-compiles for sm_90a without a GPU, so this also is the CPU-side "does it build" check.
"""
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
LIBDIR = os.path.join(ROOT, "lib")
EXTDIR = os.path.join(ROOT, "_ext")
OBJDIR = os.path.join(os.path.dirname(ROOT), "build", "obj")
INCLUDE = os.path.join(os.path.dirname(ROOT), "include")

CU_SOURCES = ["common.cu", "chain.cu", "corr.cu", "corr_tc.cu", "patchify.cu", "lie.cu", "graph.cu", "pgraph.cu", "ba.cu", "ba_wide.cu", "update_ops.cu", "gemm.cu"]
SHIM_MODULES = ["cuda_corr", "cuda_ba", "lietorch_backends", "dpvo_b200_ext"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
]
# the bundle adjustment's phase timestamps (DPVO_B200_BA_TIMING, ba.cu) exist only in builds made with
# DPVO_B200_PERF_EXPERIMENTS=1; the release library has none
if os.environ.get("DPVO_B200_PERF_EXPERIMENTS"):
    NVCC_FLAGS.append("-DDPVO_B200_PERF_EXPERIMENTS")


def _nvcc():
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else "nvcc"


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build step failed:\n  %s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(INCLUDE, "dpvo_b200.h"))
    return hs


def build_library(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = [s for s in CU_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    hdrs = _headers()
    objs, jobs = [], []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJDIR, s[:-3] + ".o")
        objs.append(obj)
        if force or _newer(obj, [src] + hdrs):
            jobs.append([_nvcc()] + NVCC_FLAGS + ["-I", INCLUDE, "-c", src, "-o", obj])
    if jobs:
        # the CPUs this process may run on (a container or batch slot can have far fewer than the host reports)
        workers = min(len(jobs), len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 4))
        if verbose:
            print("[dpvo_b200.build] nvcc: %d translation units, %d at a time" % (len(jobs), workers), flush=True)

        def compile_one(cmd):
            _run(cmd)
            if verbose:
                print("[dpvo_b200.build]   %s" % os.path.basename(cmd[cmd.index("-c") + 1]), flush=True)

        with ThreadPoolExecutor(max_workers=workers) as ex:
            list(ex.map(compile_one, jobs))
    lib = os.path.join(LIBDIR, "libdpvo_b200.so")
    if force or jobs or _newer(lib, objs):
        _run([_nvcc(), "-shared", "-o", lib] + objs + ["-lcudart", "-Xlinker", "--no-undefined"])
    return lib


def build_shims(force=False, verbose=False):
    import torch
    from torch.utils import cpp_extension as ce

    os.makedirs(EXTDIR, exist_ok=True)
    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    src = os.path.join(CSRC, "shim.cpp")
    base = os.path.join(EXTDIR, "_shim.so")
    lib = os.path.join(LIBDIR, "libdpvo_b200.so")
    if force or _newer(base, [src, os.path.join(INCLUDE, "dpvo_b200.h")]):
        if verbose:
            print("[dpvo_b200.build] g++: shim.cpp", flush=True)
        cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
        cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-fvisibility=hidden", src, "-o", base,
               "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI),
               "-I", INCLUDE, "-I", sysconfig.get_paths()["include"], "-I", os.path.join(cuda_home, "include")]
        for p in ce.include_paths():
            cmd += ["-isystem", p]
        tl = ce.library_paths()[0]
        cmd += ["-L", tl, "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda",
                "-L", LIBDIR, "-ldpvo_b200",
                "-Wl,-rpath," + tl, "-Wl,-rpath,$ORIGIN/../lib", "-Wl,-rpath," + os.path.join(cuda_home, "lib64")]
        _run(cmd)
        force = True
    for m in SHIM_MODULES:
        dst = os.path.join(EXTDIR, m + suffix)
        if force or _newer(dst, [base]):
            shutil.copyfile(base, dst)
    assert os.path.exists(lib)
    return EXTDIR


def build_all(force=False, verbose=False):
    build_library(force, verbose)
    build_shims(force, verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose=True)
    print("[dpvo_b200.build] ok")
