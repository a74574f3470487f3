"""The warp-register queue kernel keeps one copy of the solve: its register classes (NREG = 8..32) share
everything but the elimination (RegTier<32, 0>, csrc/lfr_solve_warp2.cuh).  Four inlined whole solves
made it 55 k instructions (862 KB), more than the SMs' instruction caches hold for the LM loop of four
classes at once; the bound below keeps that duplication from coming back unnoticed.  Reads the SASS of
the built library: no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "local-feature-refinement_b200", "csrc", "liblfr_b200.so")


def cuobjdump():
    for c in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if c and os.path.exists(c):
            return c
    pytest.fail("cuobjdump not found (CUDA toolkit): the library's SASS cannot be read")


def sass_sizes():
    """Instructions per kernel of the built library (mangled names)."""
    assert os.path.exists(LIB), "build the library first (__graft_entry__.build)"
    out = subprocess.run([cuobjdump(), "-sass", LIB], capture_output=True, text=True, check=True).stdout
    sizes, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            sizes[name] = 0
        elif name and re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", line):
            sizes[name] += 1
    return sizes


def test_queue_kernel_holds_one_copy_of_the_solve():
    sizes = sass_sizes()
    queue = [n for n in sizes if "solve_warp2_queue_kernel" in n]
    # solve_warp2_kernel<1, 32>: one whole solve of the widest class, compiled alone
    single = [n for n in sizes if "solve_warp2_kernelILi1ELi32EE" in n]
    assert len(queue) == 1 and len(single) == 1, sorted(sizes)
    q, s = sizes[queue[0]], sizes[single[0]]
    # one solve plus the three narrower eliminations; four whole solves would be about 3.3 x
    assert q <= 1.5 * s, "queue kernel %d instructions, one-class warp kernel %d" % (q, s)
    assert q <= 30000, "queue kernel %d instructions" % q
