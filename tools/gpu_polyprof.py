"""Cycle split of the line-search polynomial (diagnostic build, -DLFR_POLY_PROF).
Build first: python local-feature-refinement_b200/csrc/build.py --poly-prof"""
import ctypes as C
import os
import sys

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
import numpy as np  # noqa: E402

from lfr_b200 import build_problem, synth  # noqa: E402
from lfr_b200 import capi  # noqa: E402

lib = capi.Library(os.path.join(R, "local-feature-refinement_b200", "csrc", "liblfr_b200_polyprof.so"))
cfg = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
p = build_problem(synth.generate(cfg))
plan = capi.Plan(lib, p)
out = np.zeros(16, dtype=np.uint64)
lib.lib.lfr_debug_poly_prof.argtypes = [C.c_void_p, C.c_int]
plan.solve()
import torch  # noqa: E402

torch.cuda.synchronize()
lib.lib.lfr_debug_poly_prof(out.ctypes.data, 1)
plan.solve()
torch.cuda.synchronize()
lib.lib.lfr_debug_poly_prof(out.ctypes.data, 1)
names = ["coefficients", "first evals", "grid classify", "extremum cells", "root solves", "final evals"]
nq, nc = int(out[6]), int(out[7])
print("quintic calls", nq, "cubic calls", nc, "Horner evaluations", int(out[8]), "polished roots", int(out[9]))
for i, nm in enumerate(names):
    print("  %-14s %8.0f cycles / quintic call" % (nm, out[i] / max(nq, 1)))
print("  quintic total  %8.0f" % (out[:6].sum() / max(nq, 1)))
print("  cubic call     %8.0f cycles / call" % (out[10] / max(nc, 1)))
if out[9]:
    print("  Horner evaluations per polished root %.2f" % (out[8] / out[9]))
