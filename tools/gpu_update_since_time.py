"""Time --previous_matches_file: the update of an earlier SolutionFile that re-solves every component whose
problem changed since the earlier MatchingFile, against the full run and the plain update.

    python tools/gpu_update_since_time.py [--configs cfg4,cfg5] [--cases k1,k20,banned1,flow1] [--reps 5] [--out FILE]

Per config and case, OLD.pb and NEW.pb are MatchingFiles and A.pb is the native drop-in's solution of OLD.pb:
  kN       OLD.pb = the scene without the pairs of its last N images, NEW.pb = OLD.pb's pairs then those;
  banned1  OLD.pb = NEW.pb = the scene; the runs on NEW.pb ban one image (the middle one);
  flow1    NEW.pb = OLD.pb = the scene, with one pair's flow floats moved by one ulp.
Three runs of the native drop-in on NEW.pb, alternated, `reps` times each:
  full     no option;
  update   --initial_solution A.pb --update_initial_solution;
  since    the same with --previous_matches_file OLD.pb.
Each reports the best and median of its "Solver time" and "Total time" lines and of the process's wall time.
In process, best of `reps`: the earlier graph stage (Plan.from_wire on OLD.pb, which the since run adds) and
Plan.update_solution with and without `previous` (their difference is the compare on the device).  Prints one
JSON object with the GPU's name and power limit (read, never set)."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lfr_b200 import synth, wire  # noqa: E402
from lfr_b200.capi import Plan, load_b200  # noqa: E402

NATIVE = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")


def run(args):
    """(Solver time ms, Total time ms, wall ms) of one native run."""
    t0 = time.perf_counter()
    r = subprocess.run([NATIVE] + args, capture_output=True, text=True, check=True)
    wall = (time.perf_counter() - t0) * 1e3
    return (int(re.search(r"Solver time: (\d+)ms", r.stdout).group(1)),
            int(re.search(r"Total time: (\d+)ms", r.stdout).group(1)), wall)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def reencode(ms):
    return wire.decode_matching_file(wire.encode_matching_file(ms))


def files(ms, case):
    """(OLD MatchSet, NEW MatchSet, banned names) of one case."""
    if case.startswith("k"):
        k = int(case[1:])
        new_img = np.arange(len(ms.image_names) - k, len(ms.image_names))
        touch = np.isin(ms.pair_img1, new_img) | np.isin(ms.pair_img2, new_img)
        old_idx, new_idx = np.nonzero(~touch)[0], np.nonzero(touch)[0]
        return reencode(ms.select_pairs(old_idx)), reencode(ms.select_pairs(np.concatenate([old_idx, new_idx]))), ()
    if case == "banned1":
        return ms, ms, (ms.image_names[len(ms.image_names) // 2],)
    if case == "flow1":
        new = reencode(ms)
        p = new.n_pairs // 2
        lo, hi = int(new.pair_ptr[p]), int(new.pair_ptr[p + 1])
        new.disp1 = new.disp1.copy()
        new.disp1[lo:hi] = np.nextafter(new.disp1[lo:hi], np.float32(np.inf))
        return ms, new, ()
    raise ValueError(case)


def best_ms(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(min(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg4,cfg5")
    ap.add_argument("--cases", default="k1,k20,banned1,flow1")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = load_b200()
    res = {"gpu": gpu_info(), "reps": a.reps}
    with tempfile.TemporaryDirectory() as tmp:
        for cfg in a.configs.split(","):
            base = synth.generate(cfg)
            for case in a.cases.split(","):
                old, new, banned = files(base, case)
                o, n, a_pb, out = (os.path.join(tmp, "%s_%s_%s" % (cfg, case, x)) for x in ("old.pb", "new.pb", "a.pb", "o.pb"))
                with open(o, "wb") as fh:
                    fh.write(wire.encode_matching_file(old))
                with open(n, "wb") as fh:
                    fh.write(wire.encode_matching_file(new))
                run(["--matches_file", o, "--output_file", a_pb])
                with open(a_pb, "rb") as fh:
                    data = fh.read()
                with open(o, "rb") as fh:
                    old_bytes = fh.read()
                ban = [x for nm in banned for x in ("--banned_images", nm)]
                # in process: the earlier stage, and the update with and without the compare
                plan = Plan.from_matches(lib, new, banned_images=banned)
                prev = Plan.from_wire(lib, [old_bytes])
                stage_ms = best_ms(lambda: Plan.from_wire(lib, [old_bytes]).close(), a.reps)
                plain_ms = best_ms(lambda: plan.update_solution(data, new.image_names), a.reps)
                since_ms = best_ms(lambda: plan.update_solution(data, new.image_names, previous=prev), a.reps)
                n_held, n_touched, n_changed = plan.update_solution(data, new.image_names, previous=prev)
                _, n_touched_plain = plan.update_solution(data, new.image_names)
                row = dict(n_nodes=plan.n_nodes, n_components=plan.n_components, n_edges=int(plan.sizes["n_edges"]),
                           n_changed=n_changed, n_touched_since=n_touched, n_touched_update=n_touched_plain,
                           n_held_nodes_since=n_held, earlier_stage_ms=stage_ms, update_call_ms=plain_ms,
                           update_since_call_ms=since_ms, compare_ms=since_ms - plain_ms)
                prev.close()
                plan.close()
                start = ["--initial_solution", a_pb]
                runs = {"full": ["--matches_file", n, "--output_file", out] + ban,
                        "update": ["--matches_file", n, "--output_file", out] + ban + start + ["--update_initial_solution"],
                        "since": ["--matches_file", n, "--output_file", out] + ban + start
                        + ["--update_initial_solution", "--previous_matches_file", o]}
                got = {x: [] for x in runs}
                for _ in range(a.reps):
                    for x, args in runs.items():
                        got[x].append(run(args))
                for x, v in got.items():
                    v = np.array(v, np.float64)
                    for j, what in enumerate(("solver_ms", "total_ms", "wall_ms")):
                        row["%s_%s_best" % (x, what)] = float(v[:, j].min())
                        row["%s_%s_median" % (x, what)] = float(np.median(v[:, j]))
                res["%s_%s" % (cfg, case)] = row
                print(json.dumps({"%s_%s" % (cfg, case): row}), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
