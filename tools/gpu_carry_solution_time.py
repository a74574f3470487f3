"""Time carrying an earlier SolutionFile into the output (--carry_initial_solution): the device merge
(lfr_plan_encode_solution_carried) against the host one (download + lfr_wire_encode_solution_carried), and
the drop-in's incremental run over the new pairs alone against a run over every pair.

    python tools/gpu_carry_solution_time.py [--configs cfg4,cfg5] [--ks 1,20] [--reps 5] [--out tools_out/carry.json]

Per config and k: A.pb is the native drop-in's solution of the scene without its last k images (the pairs
that touch none of them); the new-pairs file holds the pairs that touch one of them.  A plan is built from
the new pairs, given A with lfr_plan_keep_solution and solved; then, alternated, `reps` times each:
  (a) plan.encode_solution_carried (the device merge, host clock, synchronised),
  (b) plan.download + the output assembly + wire.encode_solution_carried (the host merge),
  the host decode of A alone (the two lfr_wire_decode_solution passes the merge repeats after the join).
Then the native drop-in, alternated: every pair with --initial_solution A --keep_initial_solution, and the
new pairs with --initial_solution A --keep_initial_solution --carry_initial_solution: its "Total time" line
and the process's wall time.  Best and median of `reps`.  Prints one JSON object with the GPU's name and
power limit."""
import argparse
import ctypes as C
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
from lfr_b200.solver import assemble_solution  # noqa: E402
from lfr_b200.graph import host_input_arrays, problem_from_stage  # noqa: E402

NATIVE = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def drop_in(args):
    """(Total time ms, wall ms) of one native run"""
    t0 = time.perf_counter()
    r = subprocess.run([NATIVE] + args, capture_output=True, text=True, check=True)
    wall = (time.perf_counter() - t0) * 1e3
    return int(re.search(r"Total time: (\d+)ms", r.stdout).group(1)), wall


def host_decode(data):
    L = wire._lib()
    buf = np.frombuffer(data, np.uint8)
    ni, nd = C.c_uint64(), C.c_uint64()
    L.lfr_wire_decode_solution(buf.ctypes.data, buf.size, C.byref(ni), C.byref(nd), *([None] * 7))
    I, D = int(ni.value), int(nd.value)
    arrs = [np.empty(I + 1, np.uint64), np.empty(I, np.uint64), np.empty(I, np.uint32), np.empty(I, np.float32),
            np.empty(D, np.uint32), np.empty(D, np.float32), np.empty(D, np.float32)]
    L.lfr_wire_decode_solution(buf.ctypes.data, buf.size, C.byref(ni), C.byref(nd), *[a.ctypes.data for a in arrs])


def stats(v):
    return {"best": float(min(v)), "median": float(np.median(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg4,cfg5")
    ap.add_argument("--ks", default="1,20")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = load_b200()
    res = {"gpu": gpu_info()}
    with tempfile.TemporaryDirectory() as tmp:
        for cfg in a.configs.split(","):
            ms = synth.generate(cfg)
            m_all = os.path.join(tmp, "all.pb")
            with open(m_all, "wb") as fh:
                fh.write(wire.encode_matching_file(ms))
            for k in (int(x) for x in a.ks.split(",")):
                new_names = set(ms.image_names[-k:])
                touch = np.array([ms.image_names[i] in new_names or ms.image_names[j] in new_names
                                  for i, j in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist())], bool)
                old, new = ms.select_pairs(np.nonzero(~touch)[0]), ms.select_pairs(np.nonzero(touch)[0])
                m_old, m_new, s, o = (os.path.join(tmp, x) for x in ("old.pb", "new.pb", "a.pb", "o.pb"))
                with open(m_old, "wb") as fh:
                    fh.write(wire.encode_matching_file(old))
                with open(m_new, "wb") as fh:
                    fh.write(wire.encode_matching_file(new))
                subprocess.run([NATIVE, "--matches_file", m_old, "--output_file", s], capture_output=True, check=True)
                with open(s, "rb") as fh:
                    A = fh.read()
                del old
                names = new.image_names
                plan = Plan.from_matches(lib, new)
                plan.keep_solution(A, names)
                plan.solve()
                skip, _ = host_input_arrays(new)
                p = problem_from_stage(new, skip, plan.export_graph(), plan.sizes, "device")
                fact = np.array([p.graph.image_fact.get(i, 0.0) for i in range(len(names))], np.float32)
                t_dev, t_host, t_dec = [], [], []
                n_carried = 0
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    dev, _, n_carried = plan.encode_solution_carried(names, fact, A)
                    t_dev.append((time.perf_counter() - t0) * 1e3)
                    t0 = time.perf_counter()
                    pos, _ = plan.download()
                    sol = assemble_solution(p, pos)
                    host, _ = wire.encode_solution_carried(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di,
                                                           sol.dj, A)
                    t_host.append((time.perf_counter() - t0) * 1e3)
                    t0 = time.perf_counter()
                    host_decode(A)
                    t_dec.append((time.perf_counter() - t0) * 1e3)
                assert dev == host
                n_nodes, n_new_matches = plan.n_nodes, new.n_matches
                plan.close()
                del new
                runs = {"all_pairs_keep": ["--matches_file", m_all, "--output_file", o, "--initial_solution", s,
                                           "--keep_initial_solution"],
                        "new_pairs_keep_carry": ["--matches_file", m_new, "--output_file", o, "--initial_solution", s,
                                                 "--keep_initial_solution", "--carry_initial_solution"]}
                tot = {r: [] for r in runs}
                wall = {r: [] for r in runs}
                for _ in range(a.reps):
                    for r, args in runs.items():
                        t, w = drop_in(args)
                        tot[r].append(t)
                        wall[r].append(w)
                res["%s_k%d" % (cfg, k)] = dict(
                    n_images=len(ms.image_names), n_matches=ms.n_matches, n_new_matches=n_new_matches,
                    n_nodes_new_pairs=n_nodes, solution_bytes=len(A), output_bytes=len(dev), n_carried=n_carried,
                    device_merge_ms=stats(t_dev), host_merge_ms=stats(t_host), host_decode_ms=stats(t_dec),
                    **{"total_ms_" + r: stats(v) for r, v in tot.items()},
                    **{"wall_ms_" + r: stats(v) for r, v in wall.items()})
            del ms
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
