"""cfg5, one GPU, plan path with LFR_DBG_PROFILE: per-component start / end (%globaltimer) and SM of
the CTA tier for consecutive solves — why is the same solve 382 ms one time and 541 ms the next?"""
import os
import sys

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
import numpy as np  # noqa: E402

from lfr_b200 import build_problem, synth  # noqa: E402
from lfr_b200.capi import Plan, load_b200  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "cfg5"
n_solves = int(sys.argv[2]) if len(sys.argv) > 2 else 6
p = build_problem(synth.generate(name))
lib = load_b200()
import torch  # noqa: E402

plan = Plan(lib, p, lib.default_options(debug_flags=0x10))
s = torch.cuda.current_stream().cuda_stream
sizes = np.diff(p.comp_ptr.astype(np.int64))
Cn = p.n_components
for i in range(n_solves):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    plan.solve(s)
    e1.record()
    torch.cuda.synchronize()
    _, stt = plan.download(s)
    p_iters = stt["iterations"].astype(np.float64)
    rec, tm = plan.profile()
    ran = tm[:, 0] > 0
    t0 = tm[ran, 0].min()
    st = (tm[:, 0].astype(np.float64) - t0) / 1e6
    en = (tm[:, 1].astype(np.float64) - t0) / 1e6
    dur = en - st
    cta = ran & (rec["tier"] == 4)
    print("solve %d: %.1f ms by events; components timed %d (CTA tier %d); last end %.1f ms" % (
        i, e0.elapsed_time(e1), int(ran.sum()), int(cta.sum()), en[ran].max()))
    if cta.any():
        sm = rec["smid"][cta]
        print("   CTA tier: sum of durations %.0f ms over %d SMs -> /296 = %.1f ms;  start p50 %.1f p90 %.1f max %.1f;  duration p50 %.2f p99 %.1f max %.1f" % (
            dur[cta].sum(), len(np.unique(sm)), dur[cta].sum() / 296.0, np.median(st[cta]), np.percentile(st[cta], 90), st[cta].max(),
            np.median(dur[cta]), np.percentile(dur[cta], 99), dur[cta].max()))
        tot = rec["total"][cta].astype(np.float64); lm = rec["solve"][cta].astype(np.float64); ev = rec["eval"][cta].astype(np.float64)
        cg = rec["counter"][cta].astype(np.float64); its = np.maximum(1, p_iters[cta])
        print("   CTA tier cycles: total %.3g  PCG %.1f%%  eval %.1f%%;  cycles per CG iteration p50 %.0f p90 %.0f;  CG iterations per LM step p50 %.0f p90 %.0f" % (
            tot.sum(), 100 * lm.sum() / tot.sum(), 100 * ev.sum() / tot.sum(), np.median(lm / np.maximum(cg, 1)), np.percentile(lm / np.maximum(cg, 1), 90),
            np.median(cg / its), np.percentile(cg / its, 90)))
        for lo, hi in ((49, 100), (101, 250), (251, 504), (505, 1000)):
            m = (sizes[cta] >= lo) & (sizes[cta] <= hi)
            if m.any():
                print("      nodes %4d-%4d: n %5d  cycles/CG-iteration p50 %.0f  CG its/LM step p50 %.0f  LM its p50 %.0f  duration p50 %.2f ms" % (
                    lo, hi, int(m.sum()), np.median((lm / np.maximum(cg, 1))[m]), np.median((cg / its)[m]), np.median(its[m]), np.median(dur[cta][m])))
        idx = np.where(cta)[0]
        order = idx[np.argsort(-en[idx])[:5]]
        for k in order:
            print("     slot %5d nodes %4d start %7.1f dur %7.1f end %7.1f  sm %3d  cg_iters %d" % (
                k, sizes[k], st[k], dur[k], en[k], int(rec["smid"][k]), int(rec["counter"][k])))
        # concurrency: CTA-tier components running at a few instants
        for t in (5, 50, 100, 200, 300, 350, 400, 500):
            print("     t=%3d ms running %d" % (t, int(((st[cta] <= t) & (en[cta] > t)).sum())), end="")
        print()
        # per-SM busy time
        busy = np.bincount(sm, weights=dur[cta], minlength=torch.cuda.get_device_properties(0).multi_processor_count)
        print("   per-SM sum of durations: min %.0f p50 %.0f max %.0f" % (busy.min(), np.median(busy), busy.max()))
    oth = ran & ~cta
    if oth.any():
        print("   other tiers: %d components, start p50 %.1f max %.1f, end max %.1f" % (int(oth.sum()), np.median(st[oth]), st[oth].max(), en[oth].max()))
