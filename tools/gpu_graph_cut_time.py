"""The recursive cut of oversized meta-components: the parent build's host cut (lfr_cut.h on host threads)
against this build's device cut (lfr_cut.cuh), alternated in one process, per synthetic workload.  The
device cut is forced: LFR_DBG_DEVICE_CUT for the plans, LFR_DEVICE_CUT=1 for the drop-in.  Both libraries
get the same options and environment; the parent build does not know the flag and cuts on the host.

Per workload (cfg2 ... cfg5), --reps repetitions of each library, alternated:
  cut ms        lfr_host_sizes.graph_cut_ms of lfr_plan_create_from_matches (H4: meta-graph, components,
                the recursive cut, final components)
  stage ms      lfr_plan_create_from_matches + plan destroy, host clock (ends in a device synchronise)
  total ms      the native drop-in's "Total time" line with LFR_GRAPH_STAGE=device and LFR_DEVICE_CUT=1,
                the baseline library selected through LD_LIBRARY_PATH
best / median of each, and the card's name, power limit and SM clock read in the same run.  Both
libraries' exported graphs and SolutionFiles are checked to be equal.

    python tools/gpu_graph_cut_time.py --baseline DIR [--reps 5] [--workloads cfg2,cfg3,cfg4,cfg5] [--json out.json]

DIR holds liblfr_b200.so built from the parent commit (local-feature-refinement_b200/csrc/build.py).
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

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from lfr_b200 import synth, wire  # noqa: E402
from lfr_b200.capi import DBG_DEVICE_CUT, Library, Plan, load_b200  # noqa: E402
from lfr_b200.graph import host_input_arrays  # noqa: E402

DROP_IN = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stage(lib, arrs, n_img):
    t0 = time.perf_counter()
    plan = Plan.from_matches(lib, arrs, options=lib.default_options(debug_flags=DBG_DEVICE_CUT), n_images=n_img)
    ms = (time.perf_counter() - t0) * 1e3
    cut = float(plan.sizes["graph_cut_ms"])
    g = plan.export_graph()
    plan.close()
    return cut, ms, g


def drop_in(path, out, lib_dir):
    env = dict(os.environ, LFR_GRAPH_STAGE="device", LFR_DEVICE_CUT="1")
    if lib_dir:
        env["LD_LIBRARY_PATH"] = lib_dir + ((":" + env["LD_LIBRARY_PATH"]) if env.get("LD_LIBRARY_PATH") else "")
    r = subprocess.run([DROP_IN, "--matches_file", path, "--output_file", out], capture_output=True, text=True, env=env)
    m = re.search(r"^Total time: (\d+)ms$", r.stdout, re.M)
    if r.returncode != 0 or not m:
        raise RuntimeError("solve_native failed (%d): %s" % (r.returncode, r.stderr))
    with open(out, "rb") as fh:
        return int(m.group(1)), fh.read()


def spread(xs):
    return "%.1f / %.1f" % (min(xs), statistics.median(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", required=True, help="directory of the parent commit's liblfr_b200.so")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", default="cfg2,cfg3,cfg4,cfg5")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    base_dir = os.path.abspath(a.baseline)
    libs = {"host cut (parent)": (Library(os.path.join(base_dir, "liblfr_b200.so")), base_dir), "device cut": (load_b200(), None)}
    name = card()
    print("card, power limit, SM clock, max SM clock: %s" % name)
    print("best / median of %d runs per library, libraries alternated" % a.reps)
    print("%-8s %-18s %10s %14s %14s %14s" % ("workload", "library", "cut groups", "cut ms", "stage ms", "total ms"), flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        path, out = os.path.join(tmp, "m.pb"), os.path.join(tmp, "s.pb")
        for w in a.workloads.split(","):
            cfg, _, scale = w.partition("@")
            ms = synth.generate(cfg, scale=float(scale) if scale else 1.0)
            arrs = host_input_arrays(ms)[1]
            n_img = len(ms.image_names)
            wire.write_matching_file(ms, path)
            res = {k: dict(cut=[], stage=[], total=[]) for k in libs}
            graphs, sols = {}, {}
            for k, (lib, _) in libs.items():  # warm-up: context, modules
                stage(lib, arrs, n_img)
            for _ in range(a.reps):
                for k, (lib, lib_dir) in libs.items():
                    cut, st, g = stage(lib, arrs, n_img)
                    total, sol = drop_in(path, out, lib_dir)
                    res[k]["cut"].append(cut)
                    res[k]["stage"].append(st)
                    res[k]["total"].append(float(total))
                    graphs.setdefault(k, g)
                    sols.setdefault(k, sol)
            (k0, g0), (k1, g1) = list(graphs.items())
            if any(not np.array_equal(g0[f], g1[f]) for f in g0) or sols[k0] != sols[k1]:
                raise RuntimeError("%s: the two libraries' outputs differ" % w)
            plan = Plan.from_matches(libs["device cut"][0], arrs, n_images=n_img)
            groups = int(plan.sizes["n_cut_groups"])
            plan.close()
            for k in libs:
                print("%-8s %-18s %10d %14s %14s %14s" % (w, k, groups, spread(res[k]["cut"]), spread(res[k]["stage"]),
                                                           spread(res[k]["total"])), flush=True)
            rows.append(dict(workload=w, cut_groups=groups, runs=res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(dict(card=name, reps=a.reps, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
