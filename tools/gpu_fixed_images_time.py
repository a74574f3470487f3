"""Time the fixed-image mask and the start-point join of a device-resident plan (lfr_plan_fix_images,
lfr_plan_start_from_solution), and the drop-in's "Total time" with --fixed_images / --initial_solution.

    python tools/gpu_fixed_images_time.py [--configs cfg4,cfg5] [--reps 5] [--out tools_out/fixed_images.json]

Per config: the plan is built from the matches once; a SolutionFile with every node of the scene is
encoded from it; then best-of-`reps` host-clock times of fix_images (a third of the images) and of
start_from_solution, each call synchronised.  Then the native drop-in on the same matches, without and
with both options (the "Total time" lines, best of `reps`).  Prints one JSON object."""
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


def best(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return min(ts)


def total_ms(args, reps):
    out = []
    for _ in range(reps):
        r = subprocess.run([NATIVE] + args, capture_output=True, text=True, check=True)
        out.append(int(re.search(r"Total time: (\d+)ms", r.stdout).group(1)))
    return min(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg4,cfg5")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = load_b200()
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for cfg in a.configs.split(","):
            ms = synth.generate(cfg)
            plan = Plan.from_matches(lib, ms)
            fact = np.zeros(len(ms.image_names), np.float32)
            sol, _ = plan.encode_solution(ms.image_names, fact)
            fixed = np.arange(len(ms.image_names)) % 3 == 0
            t_fix = best(lambda: plan.fix_images(fixed), a.reps)
            t_join = best(lambda: plan.start_from_solution(sol, ms.image_names), a.reps)
            n_nodes = plan.n_nodes
            plan.close()
            m, s, o = (os.path.join(tmp, x) for x in ("m.pb", "s.pb", "o.pb"))
            with open(m, "wb") as fh:
                fh.write(wire.encode_matching_file(ms))
            with open(s, "wb") as fh:
                fh.write(sol)
            base = ["--matches_file", m, "--output_file", o]
            extra = ["--initial_solution", s] + sum((["--fixed_images", n] for n, f in zip(ms.image_names, fixed) if f), [])
            res[cfg] = dict(n_nodes=n_nodes, n_images=len(ms.image_names), solution_bytes=len(sol),
                            fix_images_ms=t_fix, start_from_solution_ms=t_join,
                            total_ms_default=total_ms(base, a.reps), total_ms_with_options=total_ms(base + extra, a.reps))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
