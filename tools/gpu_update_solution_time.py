"""Time the drop-in's incremental runs when k images are added to a refined scene, with
--update_initial_solution among them.

    python tools/gpu_update_solution_time.py [--configs cfg4,cfg5] [--ks 1,20] [--reps 5] [--out FILE]

Per config and k: A.pb is the native drop-in's solution of the scene without its last k images (those
banned).  Then four runs of the native drop-in, alternated, `reps` times each:
  plain        every pair, no option;
  keep         every pair, --initial_solution A.pb --keep_initial_solution;
  update       every pair, --initial_solution A.pb --update_initial_solution;
  carry_keep   only the pairs that touch a new image, --initial_solution A.pb --keep_initial_solution
               --carry_initial_solution.
Each reports the best and median of its "Solver time" and "Total time" lines and of the process's wall time.
The touched components and their nodes come from Plan.update_solution on the every-pair plan.  Prints one
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg4,cfg5")
    ap.add_argument("--ks", default="1,20")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = load_b200()
    res = {"gpu": gpu_info(), "reps": a.reps}
    with tempfile.TemporaryDirectory() as tmp:
        for cfg in a.configs.split(","):
            ms = synth.generate(cfg)
            m = os.path.join(tmp, cfg + "_m.pb")
            with open(m, "wb") as fh:
                fh.write(wire.encode_matching_file(ms))
            for k in (int(x) for x in a.ks.split(",")):
                new = set(ms.image_names[-k:])
                a_pb, o, m_new = (os.path.join(tmp, "%s_%d_%s" % (cfg, k, x)) for x in ("a.pb", "o.pb", "new.pb"))
                args = ["--matches_file", m, "--output_file", a_pb]
                for nm in sorted(new):
                    args += ["--banned_images", nm]
                run(args)
                touch = np.array([ms.image_names[i] in new or ms.image_names[j] in new
                                  for i, j in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist())], bool)
                with open(m_new, "wb") as fh:
                    fh.write(wire.encode_matching_file(ms.select_pairs(np.nonzero(touch)[0])))
                with open(a_pb, "rb") as fh:
                    data = fh.read()
                plan = Plan.from_matches(lib, ms)
                n_held, n_touched = plan.update_solution(data, ms.image_names)
                n_nodes, n_comp = plan.n_nodes, int(plan.export_graph()["comp_ptr"].shape[0] - 1)
                plan.close()
                start = ["--initial_solution", a_pb]
                runs = {"plain": ["--matches_file", m, "--output_file", o],
                        "keep": ["--matches_file", m, "--output_file", o] + start + ["--keep_initial_solution"],
                        "update": ["--matches_file", m, "--output_file", o] + start + ["--update_initial_solution"],
                        "carry_keep": ["--matches_file", m_new, "--output_file", o] + start
                        + ["--keep_initial_solution", "--carry_initial_solution"]}
                got = {x: [] for x in runs}
                for _ in range(a.reps):
                    for x, args in runs.items():
                        got[x].append(run(args))
                row = dict(n_nodes=n_nodes, n_components=n_comp, n_touched_components=n_touched,
                           n_touched_nodes=n_nodes - n_held, n_new_pairs=int(touch.sum()), n_pairs=int(ms.n_pairs))
                for x, v in got.items():
                    v = np.array(v, np.float64)
                    for j, what in enumerate(("solver_ms", "total_ms", "wall_ms")):
                        row["%s_%s_best" % (x, what)] = float(v[:, j].min())
                        row["%s_%s_median" % (x, what)] = float(np.median(v[:, j]))
                res["%s_k%d" % (cfg, k)] = row
                print(json.dumps({"%s_k%d" % (cfg, k): row}), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
