"""Host graph stage vs the graph stage on the GPU, per synthetic workload cfg1-cfg5.

Per workload, best of --reps wall-clock times of:
  host stage    lfr_host_stage_create + export with the edge records written in place (edges_out), as
                the native drop-in (csrc/lfr_solve_main.cc) runs it (lfr_b200.graph.host_stage_export)
  device route  lfr_plan_create_from_matches: uploads, the stage on the device, the per-node downloads
                and plan creation
  drop-in       the "Total time" line (solve.cc:487-641 scope) of multi-view-refinement/build/solve_native
                on the workload written as a MatchingFile.  The drop-in runs the host stage on every
                input, so there is no device-route figure for it ("not routed").
and the card's name and power limit, read in the same run.

    python tools/gpu_graph_stage_time.py [--reps 3] [--cfgs cfg1,cfg2,cfg3,cfg4,cfg5]
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from lfr_b200 import synth, wire  # noqa: E402
from lfr_b200.capi import Plan, load_b200  # noqa: E402
from lfr_b200.graph import host_input_arrays, host_stage_export  # noqa: E402

DROP_IN = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def best_of(reps, fn):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return min(t)


def drop_in_total_ms(ms, reps, tmp):
    path, out = os.path.join(tmp, "m.pb"), os.path.join(tmp, "s.pb")
    wire.write_matching_file(ms, path)
    best = None
    for _ in range(reps):
        r = subprocess.run([DROP_IN, "--matches_file", path, "--output_file", out], capture_output=True, text=True)
        m = re.search(r"^Total time: (\d+)ms$", r.stdout, re.M)
        if r.returncode != 0 or not m:
            return "failed (%d)" % r.returncode
        best = int(m.group(1)) if best is None else min(best, int(m.group(1)))
    return "%d" % best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cfgs", default="cfg1,cfg2,cfg3,cfg4,cfg5")
    a = ap.parse_args()
    lib = load_b200()
    print("card, power limit: %s" % card())
    print("%-6s %10s %10s %10s %8s %18s %18s" % ("cfg", "matches", "host ms", "device ms", "h / d",
                                                 "drop-in total ms", "drop-in (device)"))
    with tempfile.TemporaryDirectory() as tmp:
        for cfg in a.cfgs.split(","):
            ms = synth.generate(cfg)
            arrs = host_input_arrays(ms)[1]
            n_img = len(ms.image_names)
            Plan.from_matches(lib, arrs, n_images=n_img).close()  # context, kernels loaded
            th = best_of(a.reps, lambda: host_stage_export(arrs, n_img))
            td = best_of(a.reps, lambda: Plan.from_matches(lib, arrs, n_images=n_img).close())
            total = drop_in_total_ms(ms, a.reps, tmp)
            print("%-6s %10d %10.1f %10.1f %8.2f %18s %18s" % (cfg, ms.n_matches, th, td, th / td, total, "not routed"),
                  flush=True)


if __name__ == "__main__":
    main()
