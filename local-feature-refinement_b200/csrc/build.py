"""Build the in-tree libraries (git-ignored, but they travel to the GPU box):

  liblfr_b200.so  the product: CUDA kernels + the C ABI of include/lfr.h      (nvcc, sm_90a; cross-compiles without a GPU;
                  links liblfr_host.so for the wire codec)
  liblfr_host.so  CPU-only host utilities behind include/lfr_wire.h and include/lfr_host.h
                  (protobuf wire codec, host graph stage) — no CUDA dependency, so the
                  reference arm of bench.py and the tests can use them without mapping the product library
  liblfr_b200_lmstep.so
                  the product built with -DLFR_DBG_LM_STEP: every component stops after its first LM step
                  and reports it (csrc/lfr_lm.cuh), for tests/test_gpu_lm_step.py
  liblfr_b200_lsprobe.so
                  the product built with -DLFR_DBG_LS_PROBE: every component takes its first LM step, then one
                  line-search trial, its slope and the accepted step's bookkeeping, optionally a second LM step,
                  or the step after a rejected one, and reports them (csrc/lfr_lm.cuh), for
                  tests/test_gpu_ls_probe.py
  multi-view-refinement/build/solve_native
                  the native drop-in executable (lfr_solve_main.cc), linked against the two libraries
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "liblfr_b200.so")
OUT_HOST = os.path.join(HERE, "liblfr_host.so")
OUT_LM_STEP = os.path.join(HERE, "liblfr_b200_lmstep.so")
OUT_LS_PROBE = os.path.join(HERE, "liblfr_b200_lsprobe.so")
SOURCES = ["lfr_capi.cu"]
HOST_SOURCES = ["lfr_wire.cc", "lfr_host.cc"]
EXE_SOURCE = "lfr_solve_main.cc"
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT_EXE = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")
INC = os.path.join("..", "..", "include")
# build.py itself: a change of NVCC_FLAGS (e.g. the target architecture) must rebuild the library
DEPS = SOURCES + ["build.py", "lfr_setup.cuh", "lfr_solve_warp.cuh", "lfr_solve_warp2.cuh", "lfr_solve_cta.cuh", "lfr_lm.cuh", "lfr_math.cuh", "lfr_graph.cuh", "lfr_wire.cuh", "lfr_solution.cuh", "lfr_diff.cuh", "lfr_record.h", "lfr_record.cuh", "lfr_cut.h", "lfr_cut.cuh", "lfr_join.h", "lfr_start.cuh",
                  os.path.join(INC, "lfr.h"), os.path.join(INC, "lfr_graph.h"), os.path.join(INC, "lfr_host.h"),
                  os.path.join(INC, "lfr_wire.h")]
HOST_DEPS = HOST_SOURCES + ["lfr_cut.h", "lfr_join.h", "lfr_record.h", os.path.join(INC, "lfr.h"), os.path.join(INC, "lfr_wire.h"),
                            os.path.join(INC, "lfr_host.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared", "-cudart", "shared"]
# the product calls the wire codec of liblfr_host.so (the SolutionFile decode of lfr_plan_start_from_solution),
# found next to it wherever the checkout is mounted
HOST_LINK = ["-L" + HERE, "-llfr_host", "-Xlinker", "-rpath,$ORIGIN"]


def build_variant(out: str, defines) -> str:
    """Diagnostic variant of the library (e.g. -DLFR_POLY_PROF) next to the product .so."""
    build_host()
    cmd = [NVCC] + NVCC_FLAGS + ["-D" + d for d in defines] + ["-o", os.path.join(HERE, out)] + \
          [os.path.join(HERE, s) for s in SOURCES] + HOST_LINK
    subprocess.check_call(cmd)
    return os.path.join(HERE, out)


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(os.path.join(HERE, d)) > t for d in deps)


def build_host(force: bool = False) -> str:
    if force or _stale(OUT_HOST, HOST_DEPS):
        subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-shared", "-pthread", "-Wall", "-o", OUT_HOST] +
                              [os.path.join(HERE, s) for s in HOST_SOURCES])
    return OUT_HOST


def build_exe(force: bool = False, out: str = OUT_EXE, solve_lib_dir: str = HERE, solve_lib: str = "lfr_b200") -> str:
    """The native `solve`.  The product links csrc/liblfr_b200.so; tests/ link the same source against the
    CPU checker (oracle/liblfr_ref.so exports the same C ABI) to compare it with the reference binary."""
    deps = [EXE_SOURCE, os.path.join(INC, "lfr.h"), os.path.join(INC, "lfr_wire.h"), os.path.join(INC, "lfr_host.h"),
            os.path.join(INC, "lfr_graph.h"), "lfr_record.h"]
    if force or _stale(out, deps) or not os.path.exists(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", out, os.path.join(HERE, EXE_SOURCE),
                               "-L" + solve_lib_dir, "-l" + solve_lib, "-L" + HERE, "-llfr_host",
                               # found next to the checkout wherever it is mounted, then by absolute path
                               "-Wl,-rpath,$ORIGIN/../../local-feature-refinement_b200/csrc",
                               "-Wl,-rpath," + solve_lib_dir, "-Wl,-rpath," + HERE])
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    build_host(force)
    _build_cuda(force, verbose)
    build_exe(force)
    build_lm_step(force)
    build_ls_probe(force)
    return OUT


def build_lm_step(force: bool = False) -> str:
    """The first-LM-step variant, rebuilt when the product's sources change."""
    if force or _stale(OUT_LM_STEP, DEPS):
        build_variant(os.path.basename(OUT_LM_STEP), ["LFR_DBG_LM_STEP"])
    return OUT_LM_STEP


def build_ls_probe(force: bool = False) -> str:
    """The line-search probe variant, rebuilt when the product's sources change."""
    if force or _stale(OUT_LS_PROBE, DEPS):
        build_variant(os.path.basename(OUT_LS_PROBE), ["LFR_DBG_LS_PROBE"])
    return OUT_LS_PROBE


def _build_cuda(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale(OUT, DEPS):
        return OUT
    cmd = [NVCC] + NVCC_FLAGS + ["-o", OUT] + [os.path.join(HERE, s) for s in SOURCES] + HOST_LINK
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    if "--poly-prof" in sys.argv:
        print(build_variant("liblfr_b200_polyprof.so", ["LFR_POLY_PROF"]))
        sys.exit(0)
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
