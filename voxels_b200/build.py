"""Builds every native artefact of the repo, in-tree (nothing is JIT-cached under ~/.cache):

  oracle/_ref/...                 everything compiled from the reference checkout (oracle/Makefile): the Transvoxel
                                  tables re-packed for the device (_ref/gen), the reference itself (test oracle) and
                                  the drop-in's objects that need the reference's headers (_ref/dropin), and the
                                  SDF-program harness over the reference (oracle/programs.mk)
  voxels_b200/lib/libvxb200.so    CUDA kernels + C ABI (include/vxb200.h), sm_90a (H100) only
  voxels_b200/lib/libvoxels_b200.so, build/libvxh_b200.so   C++ drop-in Polygonizer + test harness over it
  build/oracle/libvxr_restate.so  CPU restatement (test infrastructure)

With the reference checkout present (VOXELS_REFERENCE, default /root/reference) oracle/_ref is (re)built from it;
without it, a prebuilt oracle/_ref is used as it is and everything else is compiled from this repo's sources.
"""
import os
import shutil
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("VOXELS_REFERENCE", "/root/reference")
ORACLE = os.path.join(REPO, "oracle")
GEN = os.path.join(ORACLE, "_ref", "gen")
LIB = os.path.join(REPO, "voxels_b200", "lib")
CSRC = os.path.join(REPO, "voxels_b200", "csrc")
TABLES = os.path.join(GEN, "vxb_tables_data.h")
LIBVXB = os.path.join(LIB, "libvxb200.so")

CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-fmad=false",
              "-Xcompiler", "-fPIC,-fopenmp", "-ccbin", CXX]


def _run(cmd, **kw):
    print("+", " ".join(cmd), flush=True)
    subprocess.run(cmd, check=True, **kw)


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.exists(s) and os.path.getmtime(s) <= t for s in sources)


def have_reference():
    return os.path.exists(os.path.join(REF, "src", "Transvoxel.inl"))


def build_oracle():
    """oracle/_ref from the reference checkout when it is there; the CPU restatement always."""
    if have_reference():
        targets = ["ref", "tables", "dropin", "restate"]
    else:
        if not os.path.exists(TABLES):
            raise RuntimeError("%s is missing and the reference checkout (%s) is not available to generate it from"
                               % (os.path.relpath(TABLES, REPO), REF))
        targets = ["restate"]
    _run(["make", "-C", ORACLE] + targets + ["REF=" + REF], stdout=subprocess.DEVNULL)
    if have_reference():
        # the SDF-program harness over the reference (tests/program_harness.py)
        _run(["make", "-C", ORACLE, "-f", "programs.mk", "programs", "REF=" + REF], stdout=subprocess.DEVNULL)


def build_cuda(force=False, verbose=False):
    srcs = [os.path.join(CSRC, n) for n in os.listdir(CSRC) if n.endswith((".cu", ".cuh", ".h"))] + \
           [TABLES, os.path.join(REPO, "include", "vxb200.h")]
    if not force and _newer(LIBVXB, srcs):
        return
    os.makedirs(LIB, exist_ok=True)
    cmd = [NVCC] + NVCC_FLAGS + ["-shared", "-I", GEN, "-o", LIBVXB, os.path.join(CSRC, "vxb200.cu")]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    _run(cmd)


def build_dropin():
    """C++ drop-in (Voxels::Polygonizer & co.) + the test harness over it, linked from oracle/_ref/dropin."""
    _run(["make", "-C", CSRC, "-f", "Makefile.dropin"])


def build_all(force=False, verbose=False):
    build_oracle()
    build_cuda(force, verbose)
    build_dropin()


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
