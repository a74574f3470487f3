"""Timeline of a zero-copy lfr_solve() (pinned caller buffers): when does each component start /
finish relative to the first one, per launch bucket size class."""
import ctypes as C
import os
import sys

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
import torch  # noqa: E402
from lfr_b200 import build_problem, synth  # noqa: E402
from lfr_b200.capi import load_b200, profile_record  # noqa: E402

sys.path.insert(0, R)
import bench  # noqa: E402

lib = load_b200()
cfg = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
flags = int(sys.argv[2]) if len(sys.argv) > 2 else 0
p = build_problem(synth.generate(cfg))
s2, keep, pos_pinned, h2d = bench.pinned_problem(lib, p)
opts = lib.default_options(debug_flags=0x10 | 0x20 | flags)   # LFR_DBG_PROFILE | LFR_DBG_ZERO_COPY
stt, bufs = lib.make_stats(p.n_components)
for _ in range(4):
    pos_pinned.zero_()
    rc = lib.lib.lfr_solve(C.byref(s2), C.byref(opts), pos_pinned.data_ptr(), C.byref(stt))
    lib.check(rc, "lfr_solve")
print("stages ms", stt.h2d_ms, stt.kernel_ms, stt.d2h_ms)
cyc = np.zeros((p.n_components, 8), dtype=np.uint64)
tm = np.zeros((p.n_components, 2), dtype=np.uint64)
f = lib.lib.lfr_debug_last_solve_profile
f.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
assert f(0, cyc.ctypes.data, tm.ctypes.data) == 0
rec = profile_record(cyc)
sel = tm[:, 0] > 0
t0 = tm[sel, 0].min()
start = (tm[:, 0].astype(np.float64) - t0) / 1e3
end = (tm[:, 1].astype(np.float64) - t0) / 1e3
sizes = np.diff(p.comp_ptr.astype(np.int64))
print("components", int(sel.sum()), "span us: first start 0, last end %.1f" % end[sel].max())
setup_us = rec["setup"].astype(np.float64) / 1965.0
for lo, hi in ((2, 4), (5, 8), (9, 12), (13, 16), (17, 64)):
    m = sel & (sizes >= lo) & (sizes <= hi)
    if m.any():
        print("nodes %2d-%2d: n %5d  start p50 %.1f p99 %.1f  setup p50 %.1f p99 %.1f max %.1f  end p50 %.1f max %.1f" % (
            lo, hi, m.sum(), np.median(start[m]), np.percentile(start[m], 99), np.median(setup_us[m]),
            np.percentile(setup_us[m], 99), setup_us[m].max(), np.median(end[m]), end[m].max()))
w = np.argsort(-end)[:6]
for i in w:
    print("  slot", int(i), "nodes", int(sizes[i]), "start %.1f setup %.1f end %.1f  total cycles %d" % (start[i], setup_us[i], end[i], int(rec["total"][i])))
