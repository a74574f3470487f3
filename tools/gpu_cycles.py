"""Per-component cycle breakdown of the solve kernels (LFR_DBG_PROFILE); for the ten longest components
also when their solve started and finished (%globaltimer, µs after the first component's start)."""
import os
import sys

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
import numpy as np  # noqa: E402

from lfr_b200 import build_problem, synth  # noqa: E402
from lfr_b200.capi import PROFILE_TIERS, Plan, load_b200  # noqa: E402

lib = load_b200()
cfg = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
p = build_problem(synth.generate(cfg))
plan = Plan(lib, p, lib.default_options(debug_flags=0x10))  # LFR_DBG_PROFILE
import torch  # noqa: E402

for _ in range(3):
    plan.solve()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s = torch.cuda.current_stream().cuda_stream
e0.record()
plan.solve(s)
e1.record()
torch.cuda.synchronize()
print("solve ms", e0.elapsed_time(e1), "launches", plan.num_launches())
pos, st = plan.download()
rec, tm = plan.profile()
it = st["iterations"]
sel = it > 0
t0 = tm[sel, 0].min()
tot = rec["total"][sel].astype(np.float64)
print("components", sel.sum(), "iters sum", it.sum())
print("cycles per component: mean %.0f  p50 %.0f  p99 %.0f  max %.0f" % (
    tot.mean(), np.median(tot), np.percentile(tot, 99), tot.max()))
names = ["total", "setup", "eval", "assemble", "solve", "rest"]
for k in names:
    print("  %-9s sum %.3e  share %.1f%%  per-iter %.0f" % (
        k, rec[k][sel].sum(), 100.0 * rec[k][sel].sum() / tot.sum(), rec[k][sel].sum() / max(1, it[sel].sum())))
w = np.argsort(-tot)[:10]
idx = np.nonzero(sel)[0][w]
for i in idx:
    print("  slot", i, "tier", PROFILE_TIERS.get(int(rec["tier"][i])), "nodes", int(p.comp_ptr[i + 1] - p.comp_ptr[i]),
          "iters", it[i], "ls_steps", int(rec["ls_steps"][i]), "cycles", [int(rec[k][i]) for k in names],
          "counter", int(rec["counter"][i]), "sm", int(rec["smid"][i]),
          "start/end us %.1f %.1f" % ((int(tm[i, 0]) - int(t0)) / 1e3, (int(tm[i, 1]) - int(t0)) / 1e3))
