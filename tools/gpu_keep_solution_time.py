"""Time keeping an earlier solution on a device-resident plan (lfr_plan_keep_solution) against starting
from it (lfr_plan_start_from_solution), and the drop-in's "Total time" with --keep_initial_solution.

    python tools/gpu_keep_solution_time.py [--configs cfg4,cfg5] [--reps 5] [--out tools_out/keep_solution.json]

Per config: the plan is built from the matches once and its solution encoded; the SolutionFile used is
that solution restricted to the first two thirds of the images (the scene before the last third was
added).  Then best-of-`reps` host-clock times of start_from_solution and keep_solution, alternated, each
call synchronised (keep_solution also builds the mask and the schedule again).  Then the native drop-in on
the same matches: without options, with --initial_solution, and with --initial_solution
--keep_initial_solution (the "Total time" lines, best of `reps`, alternated).  Prints one JSON object with
the GPU's name and power limit."""
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


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def total_ms(args):
    r = subprocess.run([NATIVE] + args, capture_output=True, text=True, check=True)
    return int(re.search(r"Total time: (\d+)ms", r.stdout).group(1))


def first_images(sol: bytes, names) -> bytes:
    """The SolutionFile `sol` restricted to the images in `names`."""
    keep = set(names)
    msgs = [m for m in wire.decode_solution(sol) if m[0] in keep]
    img_ptr = np.concatenate([[0], np.cumsum([m[2].shape[0] for m in msgs])]).astype(np.int64)
    cat = lambda k, dt: np.concatenate([m[k] for m in msgs]).astype(dt) if msgs else np.zeros(0, dt)  # noqa: E731
    return wire.encode_solution([m[0] for m in msgs], np.array([m[1] for m in msgs], np.float32), img_ptr,
                                cat(2, np.uint32), cat(3, np.float32), cat(4, np.float32))


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg4,cfg5")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = load_b200()
    res = {"gpu": gpu_info()}
    with tempfile.TemporaryDirectory() as tmp:
        for cfg in a.configs.split(","):
            ms = synth.generate(cfg)
            plan = Plan.from_matches(lib, ms)
            plan.solve()
            sol, _ = plan.encode_solution(ms.image_names, np.zeros(len(ms.image_names), np.float32))
            data = first_images(sol, ms.image_names[: 2 * len(ms.image_names) // 3])
            t_start, t_keep, n_kept = [], [], 0
            for _ in range(a.reps):
                t_start.append(timed(lambda: plan.start_from_solution(data, ms.image_names)))
                t0 = time.perf_counter()
                n_kept = plan.keep_solution(data, ms.image_names)
                t_keep.append((time.perf_counter() - t0) * 1e3)
            n_nodes = plan.n_nodes
            plan.close()
            m, s, o = (os.path.join(tmp, x) for x in ("m.pb", "s.pb", "o.pb"))
            with open(m, "wb") as fh:
                fh.write(wire.encode_matching_file(ms))
            with open(s, "wb") as fh:
                fh.write(data)
            base = ["--matches_file", m, "--output_file", o]
            runs = {"default": base, "initial_solution": base + ["--initial_solution", s],
                    "keep_initial_solution": base + ["--initial_solution", s, "--keep_initial_solution"]}
            tot = {k: [] for k in runs}
            for _ in range(a.reps):
                for k, args in runs.items():
                    tot[k].append(total_ms(args))
            res[cfg] = dict(n_nodes=n_nodes, n_kept=n_kept, n_images=len(ms.image_names), solution_bytes=len(data),
                            start_from_solution_ms=min(t_start), keep_solution_ms=min(t_keep),
                            start_from_solution_ms_median=float(np.median(t_start)),
                            keep_solution_ms_median=float(np.median(t_keep)),
                            **{"total_ms_" + k: min(v) for k, v in tot.items()})
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
