"""Time --earlier_record_file: the update of an earlier SolutionFile against the earlier run's problem record,
against the full run and the update since the earlier MatchingFile.

    python tools/gpu_update_record_time.py [--configs cfg4,cfg5] [--cases k1,k20,banned1,flow1] [--reps 5] [--out FILE]

Per config and case, OLD.pb and NEW.pb are MatchingFiles (the cases of tools/gpu_update_since_time.py), and A.pb
and A.rec are the native drop-in's solution and problem record of OLD.pb (--record_file).  Three runs of the
native drop-in on NEW.pb, alternated, `reps` times each:
  full     no option;
  since    --initial_solution A.pb --update_initial_solution --previous_matches_file OLD.pb;
  record   --initial_solution A.pb --update_initial_solution --earlier_record_file A.rec.
Each reports the best and median of its "Solver time" and "Total time" lines and of the process's wall time.
In process, best of `reps`: lfr_plan_problem_record on a plan of NEW.pb, lfr_host_problem_record on its host
stage (default helper threads, and one), and the record's size.  Prints one JSON object with the GPU's name and
power limit (read, never set)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_update_since_time import best_ms, files, gpu_info, run  # noqa: E402
from lfr_b200 import synth, wire  # noqa: E402
from lfr_b200.capi import Plan, load_b200  # noqa: E402
from lfr_b200.graph import host_input_arrays, host_stage_export, problem_from_stage  # noqa: E402


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
                o, n, a_pb, a_rec, out = (os.path.join(tmp, "%s_%s_%s" % (cfg, case, x))
                                          for x in ("old.pb", "new.pb", "a.pb", "a.rec", "o.pb"))
                with open(o, "wb") as fh:
                    fh.write(wire.encode_matching_file(old))
                with open(n, "wb") as fh:
                    fh.write(wire.encode_matching_file(new))
                run(["--matches_file", o, "--output_file", a_pb, "--record_file", a_rec])
                ban = [x for nm in banned for x in ("--banned_images", nm)]
                # in process: the record on the device and on the host
                plan = Plan.from_matches(lib, new, banned_images=banned)
                dev_ms = best_ms(lambda: plan.problem_record(new.image_names), a.reps)
                record = plan.problem_record(new.image_names)
                plan.close()
                skip, arrs = host_input_arrays(new, banned)
                rc, g, sz = host_stage_export(arrs, len(new.image_names))
                p = problem_from_stage(new, skip, g, sz, "native")
                host_ms = best_ms(lambda: wire.problem_record(p, new.image_names), a.reps)
                os.environ["LFR_HOST_THREADS"] = "1"
                host1_ms = best_ms(lambda: wire.problem_record(p, new.image_names), a.reps)
                del os.environ["LFR_HOST_THREADS"]
                assert wire.problem_record(p, new.image_names) == record
                row = dict(n_nodes=int(sz["n_nodes"]), n_components=int(sz["n_components"]), n_edges=int(sz["n_edges"]),
                           record_bytes=len(record), device_record_ms=dev_ms, host_record_ms=host_ms,
                           host_record_1thread_ms=host1_ms)
                start = ["--initial_solution", a_pb, "--update_initial_solution"]
                runs = {"full": ["--matches_file", n, "--output_file", out] + ban,
                        "since": ["--matches_file", n, "--output_file", out] + ban + start + ["--previous_matches_file", o],
                        "record": ["--matches_file", n, "--output_file", out] + ban + start + ["--earlier_record_file", a_rec]}
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
