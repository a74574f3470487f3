"""Measure a change to the solve's schedule against another checkout (the parent commit, say).

  ab      DIR_A DIR_B [--workload cfg2] [--runs 5] [--steps 30] [--debug-flags F]
          alternates `bench.py --gpus 1` of the two checkouts, prints every run's ms_per_step_median,
          the card and its power limit
  sweep   DIR [--workload cfg2] [--steps 30] [--warps 4,6,8]
          bench.py of one checkout at each warp2 queue width (LFR_DBG_WARP2_WARPS_SHIFT, 1..8)
  reset   [--workload cfg2]   (run from a checkout) the device-to-device reset of the positions that
          precedes every plan solve, timed alone (CUDA events, L2 flushed), against the plan solve
  dump    OUT_DIR    (run from a checkout) every output of plan / lfr_solve / pinned lfr_solve_multi
          solves of cfg4 and ring60 on the default, TILE_FROM_1, copy and zero-copy routes, as .npy
  compare DIR_A DIR_B   bitwise comparison of two dump (or bench.py --dump-outputs) directories
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def bench(tree, workload, steps, flags=0, warmup=5):
    tree = os.path.abspath(tree)
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
           str(warmup), "--workload", workload]
    if flags:
        cmd += ["--debug-flags", str(flags)]
    out = subprocess.run(cmd, capture_output=True, text=True, cwd=tree)
    for line in out.stdout.splitlines()[::-1]:
        if line.startswith("{"):
            return json.loads(line)
    raise SystemExit("bench.py in %s failed:\n%s" % (tree, out.stderr[-2000:]))


def cmd_ab(a):
    print("card:", card())
    res = {"A": [], "B": []}
    for _ in range(a.runs):
        for k, tree in (("A", a.dir_a), ("B", a.dir_b)):
            res[k].append(bench(tree, a.workload, a.steps, a.debug_flags)["ms_per_step_median"])
            print("%s %s ms_per_step_median %.4f" % (a.workload, k, res[k][-1]), flush=True)
    for k in ("A", "B"):
        v = np.array(res[k])
        print("%s: median %.4f  min %.4f  max %.4f" % (k, np.median(v), v.min(), v.max()))
    print("every B below every A:", bool(max(res["B"]) < min(res["A"])))


def cmd_sweep(a):
    ws = [int(x) for x in a.warps.split(",")]
    if any(not 1 <= w <= 8 for w in ws):
        raise SystemExit("sweep: the queue kernel runs 1..8 warps per SM")
    print("card:", card())
    for w in ws:
        ms = [bench(a.dir, a.workload, a.steps, w << 16)["ms_per_step_median"] for _ in range(a.runs)]
        print("W %2d: ms_per_step_median %s" % (w, " ".join("%.4f" % m for m in ms)), flush=True)


def cmd_dump(a):
    sys.path.insert(0, os.getcwd())
    from lfr_b200 import build_problem, synth
    from lfr_b200.capi import DBG_PROFILE, DBG_TILE_FROM_SHIFT, DBG_ZERO_COPY, Plan, load_b200

    lib = load_b200()
    os.makedirs(a.out, exist_ok=True)
    keys = ("iterations", "termination", "initial_cost", "final_cost")
    for name in ("cfg4", "ring60"):
        p = build_problem(synth.generate(name))
        runs = {}
        for route, flags in (("plan", 0), ("plan_tile_from_1", 1 << DBG_TILE_FROM_SHIFT), ("plan_profile", DBG_PROFILE)):
            plan = Plan(lib, p, lib.default_options(debug_flags=flags))
            plan.solve()
            plan.solve()  # the second solve resets the positions and runs the queue again
            pos, st = plan.download()
            runs[route] = (pos, st)
            if flags == DBG_PROFILE:
                rec, _ = plan.profile()
                ran = st["iterations"] > 0
                parts = sum(rec[k][ran].astype(np.int64) for k in ("setup", "eval", "assemble", "solve", "rest"))
                print("%s profile: words 1-5 add up to word 0 on %d/%d components" % (
                    name, int((parts == rec["total"][ran].astype(np.int64)).sum()), int(ran.sum())))
        runs["copy"] = lib.solve(p, lib.default_options())
        runs["zero_copy"] = lib.solve(p, lib.default_options(debug_flags=DBG_ZERO_COPY))
        runs["pinned_multi"] = lib.solve_multi(p, [0], pinned=True)
        for route, (pos, st) in runs.items():
            np.save(os.path.join(a.out, "%s_%s_positions.npy" % (name, route)), pos)
            for k in keys:
                if k in st:
                    np.save(os.path.join(a.out, "%s_%s_%s.npy" % (name, route, k)), np.asarray(st[k]))
            np.save(os.path.join(a.out, "%s_%s_totals.npy" % (name, route)),
                    np.array([st["total_iterations"], st["total_line_search_steps"]], dtype=np.uint64))
        print(name, "launches", Plan(lib, p, lib.default_options()).num_launches())


def cmd_reset(a):
    sys.path.insert(0, os.getcwd())
    import torch
    from lfr_b200 import build_problem, synth
    from lfr_b200.capi import Plan, load_b200

    lib = load_b200()
    p = build_problem(synth.generate(a.workload))
    n = 2 * p.graph.n_nodes
    src = torch.zeros(n, dtype=torch.float64, device="cuda")
    dst = torch.empty_like(src)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    plan = Plan(lib, p, lib.default_options())
    s = torch.cuda.current_stream().cuda_stream

    def timed(fn, reps=30):
        t = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            t.append(1e3 * e0.elapsed_time(e1))
        return float(np.median(t))
    for _ in range(3):
        plan.solve(s)
    copy_us = timed(lambda: dst.copy_(src))
    solve_us = timed(lambda: plan.solve(s))
    print("card:", card())
    print("%s: reset copy of %d bytes %.1f us alone (median of 30); plan solve incl. the reset %.1f us" % (
        a.workload, 8 * n, copy_us, solve_us))


def cmd_compare(a):
    names = sorted(f for f in os.listdir(a.dir_a) if f.endswith(".npy"))
    bad = 0
    for f in names:
        x = np.load(os.path.join(a.dir_a, f))
        y = np.load(os.path.join(a.dir_b, f)) if os.path.exists(os.path.join(a.dir_b, f)) else None
        same = y is not None and x.dtype == y.dtype and x.shape == y.shape and \
            np.array_equal(x.view(np.uint8), y.view(np.uint8))
        bad += not same
        if not same:
            print("DIFFERS", f)
    print("%d arrays compared, %d differ" % (len(names), bad))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    s = sub.add_parser("ab")
    s.add_argument("dir_a"); s.add_argument("dir_b")
    s.add_argument("--workload", default="cfg2"); s.add_argument("--runs", type=int, default=5)
    s.add_argument("--steps", type=int, default=30); s.add_argument("--debug-flags", type=int, default=0)
    s = sub.add_parser("sweep")
    s.add_argument("dir"); s.add_argument("--workload", default="cfg2"); s.add_argument("--steps", type=int, default=30)
    s.add_argument("--runs", type=int, default=2); s.add_argument("--warps", default="4,6,8")
    s = sub.add_parser("reset")
    s.add_argument("--workload", default="cfg2")
    s = sub.add_parser("dump")
    s.add_argument("out")
    s = sub.add_parser("compare")
    s.add_argument("dir_a"); s.add_argument("dir_b")
    a = ap.parse_args()
    {"ab": cmd_ab, "sweep": cmd_sweep, "reset": cmd_reset, "dump": cmd_dump, "compare": cmd_compare}[a.cmd](a)


if __name__ == "__main__":
    main()
