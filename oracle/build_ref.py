"""Build oracle/_ref/ — the REFERENCE's own sources compiled as a checker.

TEST INFRASTRUCTURE ONLY.  The reference (mihaidusmanu/local-feature-refinement,
multi-view-refinement/) needs Eigen, Ceres, COLMAP, Boost.program_options and
protoc-generated code, none of which exist in this image, so its own build
system cannot run here.  What CAN be done is to compile its source files
UNMODIFIED, from where they lie under /root/reference (never copied into this
repository), against the small shim headers in oracle/ref_shims/ that declare
exactly the third-party API those files use:

  libref_cost.so  <- cost.cc (via oracle/ref_cost_shim.cc)        Eigen/Core, ceres/ceres.h (Jet, AutoDiffCostFunction)
  solve           <- solve.cc (which #includes cost.cc) + graph.cc + the shims' implementations:
                     mini_ceres.cc (restated Ceres 1.14 minimizer), types_pb_shim.cc (protobuf wire
                     format of types.proto), colmap shims (ThreadPool; the 2-way cut is the same
                     deterministic stand-in the product uses: Graclus is not available on either side)
  libref_solve.so <- the same, with main() renamed (via oracle/ref_solve_shim.cc): create_and_solve_problem
                     callable on any constant mask and start point

Outputs go to oracle/_ref/ only (git-ignored, NOT gpurun-ignored: the binaries
travel to the GPU box, where /root/reference does not exist).  Flags follow the
reference's CMakeLists.txt:4 (`-std=c++11 -g`, no optimisation level) plus
-ffp-contract=off (x86-64 g++ does not contract at -O0 anyway).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("LFR_REFERENCE_DIR", "/root/reference")
REF_SRC = os.path.join(REF, "multi-view-refinement")
OUT = os.path.join(HERE, "_ref")
SHIMS = os.path.join(HERE, "ref_shims")
CXX = os.environ.get("CXX", "g++")


def reference_available() -> bool:
    return os.path.exists(os.path.join(REF_SRC, "cost.cc"))


def _newer(out, deps):
    if not os.path.exists(out):
        return False
    t = os.path.getmtime(out)
    return all(os.path.getmtime(d) <= t for d in deps if os.path.exists(d))


def _shim_files():
    files = []
    for root, _, names in os.walk(SHIMS):
        files += [os.path.join(root, n) for n in names]
    return files


def build_cost(force: bool = False) -> str:
    """cost.cc -> oracle/_ref/libref_cost.so.  Returns the path (existing file when the reference
    is absent, e.g. on the GPU box), or raises if neither exists."""
    out = os.path.join(OUT, "libref_cost.so")
    if not reference_available():
        if os.path.exists(out):
            return out
        raise RuntimeError("oracle/_ref/libref_cost.so is missing and %s is not present" % REF_SRC)
    deps = [os.path.join(HERE, "ref_cost_shim.cc"), os.path.join(REF_SRC, "cost.cc")] + _shim_files()
    if not force and _newer(out, deps):
        return out
    os.makedirs(OUT, exist_ok=True)
    cmd = [CXX, "-std=c++11", "-g", "-O0", "-ffp-contract=off", "-fPIC", "-shared",
           "-I", SHIMS, "-I", REF_SRC, "-o", out, os.path.join(HERE, "ref_cost_shim.cc")]
    subprocess.check_call(cmd)
    return out


def build_solve(force: bool = False, optimized: bool = False) -> str:
    """solve.cc (+ cost.cc, which it #includes) + graph.cc -> oracle/_ref/solve: the reference's own
    executable, with the shims' implementations linked in.  optimized=False follows the reference's
    CMakeLists.txt:4 (no -O flag); optimized=True builds oracle/_ref/solve_O2 (-O2), the fairer CPU
    baseline for bench.py's reference arm."""
    out = os.path.join(OUT, "solve_O2" if optimized else "solve")
    if not reference_available():
        if os.path.exists(out):
            return out
        raise RuntimeError("%s is missing and %s is not present" % (out, REF_SRC))
    srcs = [os.path.join(REF_SRC, "solve.cc"), os.path.join(REF_SRC, "graph.cc"),
            os.path.join(SHIMS, "mini_ceres.cc"), os.path.join(SHIMS, "types_pb_shim.cc")]
    deps = srcs + [os.path.join(REF_SRC, "cost.cc"), os.path.join(REF_SRC, "graph.h"),
                   os.path.join(HERE, "..", "local-feature-refinement_b200", "csrc", "lfr_cut.h")] + _shim_files()
    if not force and _newer(out, deps):
        return out
    os.makedirs(OUT, exist_ok=True)
    cmd = [CXX, "-std=c++11", "-g", "-O2" if optimized else "-O0", "-ffp-contract=off", "-pthread",
           "-I", SHIMS, "-I", REF_SRC, "-o", out] + srcs
    subprocess.check_call(cmd)
    return out


def build_solve_lib(force: bool = False) -> str:
    """solve.cc's create_and_solve_problem as a C function (oracle/ref_solve_shim.cc) ->
    oracle/_ref/libref_solve.so: the sources of build_solve() plus the shim, -O2 (no contraction, so
    the same bits as the -O0 build; -O2 only makes the tests that call it fast enough)."""
    out = os.path.join(OUT, "libref_solve.so")
    if not reference_available():
        if os.path.exists(out):
            return out
        raise RuntimeError("%s is missing and %s is not present" % (out, REF_SRC))
    srcs = [os.path.join(HERE, "ref_solve_shim.cc"), os.path.join(REF_SRC, "graph.cc"),
            os.path.join(SHIMS, "mini_ceres.cc"), os.path.join(SHIMS, "types_pb_shim.cc")]
    include = os.path.join(HERE, "..", "include")
    deps = srcs + [os.path.join(REF_SRC, "solve.cc"), os.path.join(REF_SRC, "cost.cc"), os.path.join(REF_SRC, "graph.h"),
                   os.path.join(include, "lfr.h"),
                   os.path.join(HERE, "..", "local-feature-refinement_b200", "csrc", "lfr_cut.h")] + _shim_files()
    if not force and _newer(out, deps):
        return out
    os.makedirs(OUT, exist_ok=True)
    cmd = [CXX, "-std=c++11", "-g", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread",
           "-I", SHIMS, "-I", REF_SRC, "-I", include, "-o", out] + srcs
    subprocess.check_call(cmd)
    return out


def build(force: bool = False):
    return [build_cost(force), build_solve(force), build_solve(force, optimized=True), build_solve_lib(force)]


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
