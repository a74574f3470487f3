"""The SolutionFile of a solved device-resident plan, two ways, per device-route workload:

  (a) host    lfr_plan_download + the output assembly (solver.assemble_solution, numpy) + lfr_wire_encode_solution
  (b) device  lfr_plan_encode_solution, one call into page-locked memory sized by the largest encoding (as the
              native drop-in calls it), split into the kernels (with the upload of names and facts) and the
              device-to-host copy of the bytes (lfr_debug_last_encode_times)

alternated in one process on one plan (Plan.from_matches, solved once), --reps runs each, best / median ms.
The two outputs are checked to be equal byte for byte.

Then, on --drop-in workloads, the native drop-in's process wall time and "Total time" on the same input
written as one MatchingFile, automatic route; with --baseline-exe (a build of the drop-in from before the
encoder on the device) the two are alternated and their outputs compared.  The card's name, power limit and
maximum SM clock are read in the same run.

    python tools/gpu_solution_encode_time.py [--reps 5] [--workloads cfg2@0.1,cfg2,cfg3,cfg4,cfg5]
                                             [--drop-in cfg4,cfg5] [--baseline-exe PATH] [--json out.json]
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
from types import SimpleNamespace

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from lfr_b200 import synth, wire  # noqa: E402
from lfr_b200.capi import Plan, load_b200  # noqa: E402
from lfr_b200.solver import assemble_solution  # noqa: E402

DROP_IN = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def ms_since(t0):
    return (time.perf_counter() - t0) * 1e3


def spread(xs):
    return "%.2f / %.2f" % (min(xs), statistics.median(xs))


def image_facts(ms):
    fact = np.zeros(len(ms.image_names), np.float32)
    seen = np.zeros(len(ms.image_names), bool)
    for a, b, fa, fb in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist(), ms.pair_fact1, ms.pair_fact2):
        for i, f in ((a, fa), (b, fb)):
            if not seen[i]:
                seen[i], fact[i] = True, f
    return fact


def drop_in(exe, path, out):
    t0 = time.perf_counter()
    r = subprocess.run([exe, "--matches_file", path, "--output_file", out], capture_output=True, text=True)
    wall = ms_since(t0)
    m = re.search(r"^Total time: (\d+)ms$", r.stdout, re.M)
    if r.returncode != 0 or not m:
        raise RuntimeError("%s failed (%d): %s" % (exe, r.returncode, r.stderr))
    with open(out, "rb") as fh:
        return float(m.group(1)), wall, [l for l in r.stdout.splitlines() if " time:" not in l], fh.read()


def library_level(lib, ms, reps):
    names, fact = ms.image_names, image_facts(ms)
    plan = Plan.from_matches(lib, ms)
    plan.solve()
    g = plan.export_graph()
    graph = SimpleNamespace(n_nodes=plan.n_nodes, node_image=g["node_image"].astype(np.int64), node_feat=g["node_feat"],
                            image_names=names, image_fact=fact)
    blob, off = wire._names_blob(names)
    cap = 18 * plan.n_nodes + sum(27 + len(n.encode("utf-8", "surrogateescape")) for n in names)
    L = lib.lib
    L.lfr_host_alloc.restype = C.c_void_p
    L.lfr_host_alloc.argtypes = [C.c_uint64]
    L.lfr_host_free.argtypes = [C.c_void_p]
    times = L.lfr_debug_last_encode_times
    times.argtypes = [C.c_void_p]
    buf = L.lfr_host_alloc(cap)
    t = {k: [] for k in ("a_download", "a_assemble", "a_encode", "a_total", "b_kernels", "b_d2h", "b_total")}
    try:
        for i in range(reps + 1):                    # the first round warms up both
            t0 = time.perf_counter()
            pos, _ = plan.download()
            t1 = time.perf_counter()
            s = assemble_solution(SimpleNamespace(graph=graph), pos)
            t2 = time.perf_counter()
            want = wire.encode_solution(s.image_names, s.fact, s.img_ptr, s.feature_idx, s.di, s.dj)
            t3 = time.perf_counter()
            a = [(t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3, (t3 - t0) * 1e3]
            n_out = C.c_uint64()
            t0 = time.perf_counter()
            need = L.lfr_plan_encode_solution(plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data,
                                              fact.ctypes.data, buf, cap, C.byref(n_out))
            b_total = ms_since(t0)
            if need != len(want) or C.string_at(buf, need) != want or n_out.value != s.n_outside:
                raise RuntimeError("the device encoding differs from the host's")
            kd = (C.c_double * 2)()
            times(kd)
            if i:
                for k, v in zip(("a_download", "a_assemble", "a_encode", "a_total"), a):
                    t[k].append(v)
                t["b_kernels"].append(kd[0])
                t["b_d2h"].append(kd[1])
                t["b_total"].append(b_total)
    finally:
        L.lfr_host_free(buf)
        plan.close()
    return t, plan.n_nodes, len(want)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", default="cfg2@0.1,cfg2,cfg3,cfg4,cfg5", help="cfg or cfg@scale, comma-separated")
    ap.add_argument("--drop-in", default="cfg4,cfg5")
    ap.add_argument("--baseline-exe", default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    lib = load_b200()
    name = card()
    print("card, power limit, max SM clock: %s" % name)
    print("ms, best / median of %d runs, (a) and (b) alternated" % a.reps, flush=True)
    rows = []
    for w in a.workloads.split(","):
        cfg, _, scale = w.partition("@")
        ms = synth.generate(cfg, scale=float(scale) if scale else 1.0)
        t, n, nbytes = library_level(lib, ms, a.reps)
        row = dict(workload=w, n_nodes=n, bytes=nbytes, **t)
        print("%s: %d nodes, %d bytes" % (w, n, nbytes))
        print("  (a) download %s + assemble %s + encode %s = %s" % (
            spread(t["a_download"]), spread(t["a_assemble"]), spread(t["a_encode"]), spread(t["a_total"])))
        print("  (b) kernels %s + D2H %s; call %s" % (spread(t["b_kernels"]), spread(t["b_d2h"]), spread(t["b_total"])),
              flush=True)
        if cfg in a.drop_in.split(",") and not scale:
            exes = [("new", DROP_IN)] + ([("baseline", a.baseline_exe)] if a.baseline_exe else [])
            runs = {k: [] for k, _ in exes}
            with tempfile.TemporaryDirectory() as tmp:
                path, out = os.path.join(tmp, "m.pb"), os.path.join(tmp, "s.pb")
                wire.write_matching_file(ms, path)
                ref = None
                for _ in range(a.reps):
                    for k, exe in exes:
                        total, wall, lines, sol = drop_in(exe, path, out)
                        if ref is None:
                            ref = (lines, sol)
                        elif (lines, sol) != ref:
                            raise RuntimeError("%s: the %s drop-in's output differs" % (w, k))
                        runs[k].append((total, wall))
            row["drop_in"] = {k: dict(total_ms=[x for x, _ in v], wall_ms=[y for _, y in v]) for k, v in runs.items()}
            for k, v in row["drop_in"].items():
                print("  drop-in %-8s Total time %s, wall %s" % (k, spread(v["total_ms"]), spread(v["wall_ms"])), flush=True)
        rows.append(row)
        del ms
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(dict(card=name, reps=a.reps, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
