"""ORACLE (test infrastructure): compile the REFERENCE's own CUDA extensions for sm_90a into
oracle/_ref/ so the GPU box can compare our kernels against the reference's kernels directly.

Sources are read where they lie under /root/reference; nothing is copied into the repository.  The
minimal edits the toolchain forces (SURVEY 8(c)) are applied with sed to throw-away copies in a temp
directory:
  cuda_corr   correlation_kernel.cu: the four `x.type()` dispatch arguments (lines 211, 273, 299,
              325) -> `x.scalar_type()` (torch 2.11 no longer accepts DeprecatedTypeProperties).
              correlation.cpp is used unmodified.
  cuda_ba     ba_cuda.cu unmodified.  ba.cpp without its Eigen includes (lines 6-7), without
              solve / solve_system (lines 99-180) and its m.def (line 187): Eigen is not in the image.
              block_e.cu with `#include <Eigen/Core>` dropped and the single
              `typedef Eigen::Array<long,-1,-1> IndexLookup` (line 36) replaced by a 10-line
              std::vector-backed struct with the same Constant(r,c,v) / operator()(i,j) surface.
lietorch_backends cannot be built (every kernel is Eigen template code): no _ref for it.

Outputs: oracle/_ref/ref_cuda_corr<EXT>, oracle/_ref/ref_cuda_ba<EXT> (module names prefixed so they
can be imported next to ours).  git-ignored.  Run: python oracle/build_ref.py

stage_python(): the reference's *Python* package (dpvo/*.py, altcorr/, fastba/, lietorch/ wrappers,
config/*.yaml -- interpreted code, no build step) packed UNMODIFIED into oracle/_ref/dpvo_ref_py.zip so that the GPU
box, where /root/reference does not exist, can run the reference's own host code (DPVO.update,
net.Update, altcorr.corr, fastba.BA, lietorch/run_tests.py) on top of either set of native modules:
ours (the drop-in being exercised) or oracle/_ref (the reference-CUDA arm of bench.py).  Same status
as oracle/_ref: a build output of the checker, git-ignored, never part of the repository history.
"""
import os
import re
import subprocess
import sys
import sysconfig
import tempfile
from concurrent.futures import ThreadPoolExecutor

REF = "/root/reference/dpvo"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")

INDEX_LOOKUP = r'''
struct IndexLookup {
  std::vector<long> d; long r = 0, c = 0;
  static IndexLookup Constant(long rows, long cols, long v) { IndexLookup t; t.r = rows; t.c = cols; t.d.assign(rows * cols, v); return t; }
  long& operator()(long i, long j) { return d[i * c + j]; }
  const long& operator()(long i, long j) const { return d[i * c + j]; }
  long rows() const { return r; } long cols() const { return c; }
};
'''


def _flags():
    import torch
    from torch.utils import cpp_extension as ce
    inc = []
    for p in ce.include_paths():
        inc += ["-isystem", p]
    inc += ["-I", sysconfig.get_paths()["include"]]
    abi = "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)
    tl = ce.library_paths()[0]
    link = ["-L", tl, "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart",
            "-Xlinker", "-rpath," + tl]
    return inc, abi, link


def _sh(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        raise RuntimeError("reference build failed:\n%s\n%s" % (" ".join(cmd), r.stdout[-4000:]))


def build(force=False):
    if not os.path.isdir(REF):
        return False
    os.makedirs(OUT, exist_ok=True)
    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    t_corr = os.path.join(OUT, "ref_cuda_corr" + suffix)
    t_ba = os.path.join(OUT, "ref_cuda_ba" + suffix)
    if not force and os.path.exists(t_corr) and os.path.exists(t_ba):
        return True
    inc, abi, link = _flags()
    nv = ["nvcc", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
          "-Xcompiler", "-fPIC", abi] + inc
    with tempfile.TemporaryDirectory(prefix="dpvo_ref_") as tmp:
        # ---- cuda_corr
        src = open(os.path.join(REF, "altcorr", "correlation_kernel.cu")).read()
        src, n = re.subn(r"\.type\(\), \"", ".scalar_type(), \"", src)
        assert n == 4, "expected 4 dispatch sites, found %d" % n
        open(os.path.join(tmp, "correlation_kernel.cu"), "w").write(src)
        # ---- cuda_ba
        lines = open(os.path.join(REF, "fastba", "ba.cpp")).read().split("\n")
        keep = [l for i, l in enumerate(lines, 1) if not (i in (6, 7) or 99 <= i <= 180 or i == 187)]
        open(os.path.join(tmp, "ba.cpp"), "w").write("\n".join(keep))
        be = open(os.path.join(REF, "fastba", "block_e.cu")).read()
        be = be.replace("#include <Eigen/Core>", "#include <vector>")
        be, n = re.subn(r"typedef Eigen::Array<long,\s*-1,\s*-1>\s*IndexLookup;", INDEX_LOOKUP, be)
        assert n == 1, "IndexLookup typedef not found"
        open(os.path.join(tmp, "block_e.cu"), "w").write(be)
        fb = ["-I", os.path.join(REF, "fastba")]
        corr = nv + ["-DTORCH_EXTENSION_NAME=ref_cuda_corr"]
        ba = nv + fb + ["-DTORCH_EXTENSION_NAME=ref_cuda_ba"]
        # the five translation units are independent (and each takes minutes): compile them concurrently
        compiles = [corr + ["-c", os.path.join(tmp, "correlation_kernel.cu"), "-o", os.path.join(tmp, "ck.o")],
                    corr + ["-x", "cu", "-c", os.path.join(REF, "altcorr", "correlation.cpp"), "-o", os.path.join(tmp, "cc.o")],
                    ba + ["-c", os.path.join(REF, "fastba", "ba_cuda.cu"), "-o", os.path.join(tmp, "bk.o")],
                    ba + ["-c", os.path.join(tmp, "block_e.cu"), "-o", os.path.join(tmp, "be.o")],
                    ba + ["-x", "cu", "-c", os.path.join(tmp, "ba.cpp"), "-o", os.path.join(tmp, "bc.o")]]
        with ThreadPoolExecutor(max_workers=len(compiles)) as ex:
            list(ex.map(_sh, compiles))
        _sh(["nvcc", "-shared", "-o", t_corr, os.path.join(tmp, "ck.o"), os.path.join(tmp, "cc.o")] + link)
        _sh(["nvcc", "-shared", "-o", t_ba, os.path.join(tmp, "bk.o"), os.path.join(tmp, "be.o"), os.path.join(tmp, "bc.o")] + link)
    return True


PY_ZIP = os.path.join(OUT, "dpvo_ref_py.zip")
_PY_SKIP = ("data_readers", "retrieval", "include", "src", "__pycache__")


def stage_python(force=False):
    """pack the reference's .py files (and the two yaml configs), byte for byte, into oracle/_ref/dpvo_ref_py.zip;
    Python imports packages straight from a zip on sys.path, so nothing is ever unpacked into the tree"""
    import zipfile
    if not os.path.isdir(REF):
        return os.path.exists(PY_ZIP)
    if os.path.exists(PY_ZIP) and not force:
        return True
    os.makedirs(OUT, exist_ok=True)
    with zipfile.ZipFile(PY_ZIP, "w", zipfile.ZIP_DEFLATED) as z:
        for dirpath, dirnames, filenames in os.walk(REF):
            dirnames[:] = sorted(d for d in dirnames if d not in _PY_SKIP)
            rel = os.path.relpath(dirpath, os.path.dirname(REF))
            z.writestr(rel + "/", b"")        # directory entry: dpvo/loop_closure has no __init__.py (namespace package)
            for f in sorted(filenames):
                if f.endswith(".py"):
                    z.write(os.path.join(dirpath, f), os.path.join(rel, f))
        for f in ("default.yaml", "fast.yaml"):
            z.write(os.path.join(os.path.dirname(REF), "config", f), os.path.join("config", f))
    return True


if __name__ == "__main__":
    stage_python(force="--force" in sys.argv)
    ok = build(force="--force" in sys.argv)
    print("oracle/_ref:", "built" if ok else "reference tree not mounted; skipped")
