"""Host graph stage vs the graph stage on the GPU, per synthetic workload: where the drop-in's route
rule (lfr_graph_stage_on_device, include/lfr_graph.h) should switch.

Per workload (cfg1-cfg5 and cfg2 scaled down between cfg1 and cfg2), over --reps repetitions:
  host / device ms    the stage alone through the library: lfr_host_stage_create + export with the edge
                      records written in place (edges_out), as the native drop-in runs it
                      (lfr_b200.graph.host_stage_export), against lfr_plan_create_from_matches (uploads, the
                      stage on the device, the per-node downloads and plan creation); best of --reps
  drop-in             multi-view-refinement/build/solve_native on the workload written as a MatchingFile,
                      run with LFR_GRAPH_STAGE=host and =device alternately: the "Total time" line
                      (solve.cc:487-641 scope) and the process wall time, best / median of --reps each.
                      The two routes' SolutionFiles and untimed stdout lines are checked to be equal.
  auto                the route the rule picks for the workload (no hook set)
and the card's name and power limit, read in the same run.

    python tools/gpu_graph_stage_time.py [--reps 5] [--workloads cfg1,cfg2@0.05,...] [--json out.json]
"""
import argparse
import json
import os
import re
import statistics
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
WORKLOADS = "cfg1,cfg2@0.02,cfg2@0.05,cfg2@0.1,cfg2@0.25,cfg2@0.5,cfg2,cfg3,cfg4,cfg5"


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


def drop_in(path, out, route):
    """One run of the drop-in with the route forced: (Total time ms, wall ms, untimed stdout, SolutionFile)."""
    env = dict(os.environ, LFR_GRAPH_STAGE=route)
    t0 = time.perf_counter()
    r = subprocess.run([DROP_IN, "--matches_file", path, "--output_file", out], capture_output=True, text=True, env=env)
    wall = (time.perf_counter() - t0) * 1e3
    m = re.search(r"^Total time: (\d+)ms$", r.stdout, re.M)
    if r.returncode != 0 or not m:
        raise RuntimeError("solve_native (%s route) failed (%d): %s" % (route, r.returncode, r.stderr))
    untimed = [l for l in r.stdout.splitlines() if " time:" not in l]
    with open(out, "rb") as fh:
        return int(m.group(1)), wall, untimed, fh.read()


def spread(xs):
    return "%d / %d" % (round(min(xs)), round(statistics.median(xs)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", default=WORKLOADS, help="cfg or cfg@scale, comma-separated")
    ap.add_argument("--json", default=None, help="also write the rows here")
    a = ap.parse_args()
    lib = load_b200()
    name = card()
    print("card, power limit: %s" % name)
    print("drop-in columns: best / median of %d runs per route, routes alternated" % a.reps)
    hdr = ("workload", "dir. edges", "auto", "host ms", "device ms", "total host", "total device", "wall host",
           "wall device")
    print("%-10s %11s %6s %8s %9s %12s %12s %12s %12s" % hdr, flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        path, out = os.path.join(tmp, "m.pb"), os.path.join(tmp, "s.pb")
        for w in a.workloads.split(","):
            cfg, _, scale = w.partition("@")
            ms = synth.generate(cfg, scale=float(scale) if scale else 1.0)
            arrs = host_input_arrays(ms)[1]
            n_img = len(ms.image_names)
            auto = "device" if lib.graph_stage_on_device(arrs, n_img) else "host"
            Plan.from_matches(lib, arrs, n_images=n_img).close()  # context, kernels loaded
            th = best_of(a.reps, lambda: host_stage_export(arrs, n_img))
            td = best_of(a.reps, lambda: Plan.from_matches(lib, arrs, n_images=n_img).close())
            wire.write_matching_file(ms, path)
            runs = {"host": [], "device": []}
            ref = None
            for _ in range(a.reps):
                for route in ("host", "device"):
                    total, wall, lines, sol = drop_in(path, out, route)
                    if ref is None:
                        ref = (lines, sol)
                    elif (lines, sol) != ref:
                        raise RuntimeError("%s: the %s route's output differs from the host route's" % (w, route))
                    runs[route].append((total, wall))
            tot = {r: [t for t, _ in v] for r, v in runs.items()}
            wall = {r: [x for _, x in v] for r, v in runs.items()}
            print("%-10s %11d %6s %8.1f %9.1f %12s %12s %12s %12s" % (
                w, 2 * ms.n_matches, auto, th, td, spread(tot["host"]), spread(tot["device"]), spread(wall["host"]),
                spread(wall["device"])), flush=True)
            rows.append(dict(workload=w, directed_edges=2 * ms.n_matches, auto=auto, host_stage_ms=th, device_stage_ms=td,
                             total_ms=tot, wall_ms=wall))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(dict(card=name, reps=a.reps, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
