"""Per-component timeline of a plan solve (LFR_DBG_PROFILE) by tier: when components start / end, how
long they run, how many run at once — what bounds a scene's solve time."""
import os
import sys

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
import numpy as np  # noqa: E402

from lfr_b200 import build_problem, synth  # noqa: E402
from lfr_b200.capi import PROFILE_TIERS, Plan, load_b200  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "cfg4"
flags = int(sys.argv[2], 0) if len(sys.argv) > 2 else 0
p = build_problem(synth.generate(name))
lib = load_b200()
import torch  # noqa: E402

plan = Plan(lib, p, lib.default_options(debug_flags=0x10 | flags))
s = torch.cuda.current_stream().cuda_stream
sizes = np.diff(p.comp_ptr.astype(np.int64))
Cn = p.n_components
for i in range(2):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); plan.solve(s); e1.record(); torch.cuda.synchronize()
_, stt = plan.download(s)
iters = stt["iterations"].astype(np.float64)
rec, tm = plan.profile()
ran = tm[:, 0] > 0
t0 = tm[ran, 0].min()
st = (tm[:, 0].astype(np.float64) - t0) / 1e3
en = (tm[:, 1].astype(np.float64) - t0) / 1e3
dur = en - st
print("%s: solve %.3f ms by events; %d components timed; last end %.1f us; launches %d" % (name, e0.elapsed_time(e1), int(ran.sum()), en[ran].max(), plan.num_launches()))
tier = rec["tier"]
for t, nm in PROFILE_TIERS.items():
    m = ran & (tier == t)
    if not m.any():
        continue
    print("  %-4s n %5d  nodes p50 %3d max %3d | start p50 %7.1f max %7.1f | duration p50 %7.1f p99 %7.1f max %7.1f us | end max %7.1f | sum of durations %.1f ms | LM its p50 %d max %d" % (
        nm, int(m.sum()), int(np.median(sizes[m])), int(sizes[m].max()), np.median(st[m]), st[m].max(), np.median(dur[m]), np.percentile(dur[m], 99), dur[m].max(),
        en[m].max(), dur[m].sum() / 1e3, int(np.median(iters[m])), int(iters[m].max())))
    tot = rec["total"][m].astype(np.float64); lm = rec["solve"][m].astype(np.float64)
    print("       cycles: linear solves %.1f%% of total; per LM iteration p50 %.0f cycles (linear solve %.0f)" % (
        100 * lm.sum() / tot.sum(), np.median(tot / np.maximum(iters[m], 1)), np.median(lm / np.maximum(iters[m], 1))))
T = en[ran].max()
for frac in (0.05, 0.25, 0.5, 0.75, 0.9, 0.97):
    t = frac * T
    print("  t=%7.1f us running: %s" % (t, "  ".join("%s %d" % (nm, int((ran & (tier == k) & (st <= t) & (en > t)).sum())) for k, nm in PROFILE_TIERS.items())))
w = np.argsort(-en)[:6]
for i in w:
    print("  last: slot %d tier %s nodes %d start %.1f dur %.1f end %.1f LM its %d" % (int(i), PROFILE_TIERS.get(int(tier[i])), int(sizes[i]), st[i], dur[i], en[i], int(iters[i])))
