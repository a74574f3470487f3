"""MatchingFile bytes -> device-resident plan, two ways, per device-route workload:

  (a) host   lfr_wire_decode_matches (wire.decode_matching_file) + lfr_plan_create_from_matches
  (b) wire   lfr_wire_walk_matches + lfr_plan_create_from_wire (Plan.from_wire): the matches decoded on the GPU

alternated in one process, --reps runs each, best / median ms.  (a) is split into the host decode and the
call that uploads the decoded arrays and runs the stage; (b) into the pair walk (timed on its own in the same
iteration), the staged upload of the bytes and offsets and the decode kernels (lfr_debug_last_wire_times:
decode = CUDA events around the kernels, upload = the rest of that phase's host time), and the whole call.
Both plans' lfr_plan_export_graph arrays are checked to be equal.

Then the native drop-in on the same workload written as one MatchingFile, automatic route: "Total time"
and process wall time, best / median of --reps; with --baseline-exe (a build of the drop-in from before
the device decoder) both are alternated.  The card's name and power limit are read in the same run.

    python tools/gpu_wire_decode_time.py [--reps 5] [--workloads cfg2@0.25,cfg2,cfg3,cfg4,cfg5]
                                         [--baseline-exe PATH] [--json out.json]
"""
import argparse
import ctypes as C
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

DROP_IN = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")
WORKLOADS = "cfg2@0.25,cfg2,cfg3,cfg4,cfg5"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def ms_since(t0):
    return (time.perf_counter() - t0) * 1e3


def spread(xs):
    return "%.1f / %.1f" % (min(xs), statistics.median(xs))


def drop_in(exe, path, out):
    t0 = time.perf_counter()
    r = subprocess.run([exe, "--matches_file", path, "--output_file", out], capture_output=True, text=True)
    wall = ms_since(t0)
    m = re.search(r"^Total time: (\d+)ms$", r.stdout, re.M)
    if r.returncode != 0 or not m:
        raise RuntimeError("%s failed (%d): %s" % (exe, r.returncode, r.stderr))
    with open(out, "rb") as fh:
        return float(m.group(1)), wall, [l for l in r.stdout.splitlines() if " time:" not in l], fh.read()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", default=WORKLOADS, help="cfg or cfg@scale, comma-separated")
    ap.add_argument("--baseline-exe", default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    lib = load_b200()
    wire_times = lib.lib.lfr_debug_last_wire_times
    wire_times.argtypes = [C.c_void_p]
    name = card()
    print("card, power limit, max SM clock: %s" % name)
    print("ms, best / median of %d runs, (a) and (b) alternated" % a.reps, flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        path, out = os.path.join(tmp, "m.pb"), os.path.join(tmp, "s.pb")
        for w in a.workloads.split(","):
            cfg, _, scale = w.partition("@")
            ms = synth.generate(cfg, scale=float(scale) if scale else 1.0)
            data = wire.encode_matching_file(ms)
            del ms
            t = {k: [] for k in ("a_decode", "a_create", "a_total", "b_walk", "b_upload", "b_decode", "b_total")}
            Plan.from_wire(lib, [data]).close()  # context, kernels loaded
            for _ in range(a.reps):
                t0 = time.perf_counter()
                dec = wire.decode_matching_file(data)
                t["a_decode"].append(ms_since(t0))
                t1 = time.perf_counter()
                pa = Plan.from_matches(lib, dec)
                t["a_create"].append(ms_since(t1))
                t["a_total"].append(ms_since(t0))
                t0 = time.perf_counter()
                wire.walk_matching_file(data)
                t["b_walk"].append(ms_since(t0))
                t0 = time.perf_counter()
                pb = Plan.from_wire(lib, [data])
                t["b_total"].append(ms_since(t0))
                wt = (C.c_double * 2)()
                wire_times(wt)
                t["b_upload"].append(wt[0])
                t["b_decode"].append(wt[1])
                ga, gb = pa.export_graph(), pb.export_graph()
                if any(ga[k].tobytes() != gb[k].tobytes() for k in ga):
                    raise RuntimeError("%s: the two plans differ" % w)
                pa.close()
                pb.close()
                del dec
            with open(path, "wb") as fh:
                fh.write(data)
            exes = [("new", DROP_IN)] + ([("baseline", a.baseline_exe)] if a.baseline_exe else [])
            runs = {k: [] for k, _ in exes}
            ref = None
            for _ in range(a.reps):
                for k, exe in exes:
                    total, wall, lines, sol = drop_in(exe, path, out)
                    if ref is None:
                        ref = (lines, sol)
                    elif (lines, sol) != ref:
                        raise RuntimeError("%s: the %s drop-in's output differs" % (w, k))
                    runs[k].append((total, wall))
            row = dict(workload=w, bytes=len(data), n_matches=int(wire.walk_matching_file(data)["match_off"].shape[0]),
                       **t, drop_in={k: dict(total_ms=[x for x, _ in v], wall_ms=[y for _, y in v]) for k, v in runs.items()})
            rows.append(row)
            print("%s: %d MB, %d matches" % (w, len(data) >> 20, row["n_matches"]))
            print("  (a) host decode %s + from_matches %s = %s" % (spread(t["a_decode"]), spread(t["a_create"]), spread(t["a_total"])))
            print("  (b) walk %s; from_wire %s, of which upload %s, decode %s" % (
                spread(t["b_walk"]), spread(t["b_total"]), spread(t["b_upload"]), spread(t["b_decode"])))
            for k, v in row["drop_in"].items():
                print("  drop-in %-8s Total time %s, wall %s" % (k, spread(v["total_ms"]), spread(v["wall_ms"])), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(dict(card=name, reps=a.reps, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
