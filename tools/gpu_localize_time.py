"""Time --query_images: one batch run that localizes Q queries against a Fountain-like database, against a loop
of one process per query.

    python tools/gpu_localize_time.py [--queries 100,1000] [--loop 100] [--reps 3] [--out FILE]

The database is synth's cfg2 layout (11 images, like Fountain) at 0.2 of its keypoints.  Eight query templates
are synthesized against it, each matched to 4 database images; query i is template i mod 8 under its own name.
The batch file holds every query's pairs; the own file of a query holds its pairs alone.  Per Q:
  batch  the native drop-in with --query_images for every query, best and median of `reps` runs;
  loop   the native drop-in once per own file, for the first min(Q, --loop) queries, summed; `loop_wall_ms_per_q`
         scales that sum to all Q queries (exact when Q <= --loop).
Each run reports the process's wall time and its "Total time" and "Solver time" lines.  Every timed own run's
query Image message is checked against the batch's bytes.  Prints one JSON object with the GPU's name and
power limit (read, never set)."""
import argparse
import dataclasses
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_update_since_time import NATIVE, gpu_info  # noqa: E402
from lfr_b200 import synth, wire  # noqa: E402
from lfr_b200.matchset import MatchSet  # noqa: E402

DB, K, TEMPLATES = 11, 4, 8


def templates(scale):
    """Query templates: (MatchSet of the query's pairs, the query's image id in it)."""
    out = []
    for t in range(TEMPLATES):
        cfg = dataclasses.replace(synth.CONFIGS["cfg2"], n_images=DB + 1)
        ms = synth.generate(cfg, scale=scale, seed=500 + t)
        rng = np.random.default_rng(t)
        ds = rng.choice(DB, K, replace=False)
        keep = np.nonzero(((ms.pair_img1 == DB) & np.isin(ms.pair_img2, ds)) | ((ms.pair_img2 == DB) & np.isin(ms.pair_img1, ds)))[0]
        out.append(ms.select_pairs(keep))
    return out


def query_part(tpl, name):
    ms = dataclasses.replace(tpl, image_names=list(tpl.image_names))
    ms.image_names[DB] = name
    return ms


def run(args):
    t0 = time.perf_counter()
    r = subprocess.run([NATIVE] + args, capture_output=True, text=True, check=True)
    wall = (time.perf_counter() - t0) * 1e3
    return (wall, int(re.search(r"Total time: (\d+)ms", r.stdout).group(1)),
            int(re.search(r"Solver time: (\d+)ms", r.stdout).group(1)))


def image_messages(data):
    out, i = {}, 0
    while i < len(data):
        j, n, s = i + 1, 0, 0
        while True:
            b = data[j]
            n |= (b & 0x7F) << s
            s += 7
            j += 1
            if b < 0x80:
                break
        out[wire.decode_solution(data[i:j + n])[0][0]] = data[i:j + n]
        i = j + n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", default="100,1000")
    ap.add_argument("--loop", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scale", type=float, default=0.2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tpls = templates(a.scale)
    res = dict(gpu=gpu_info(), scale=a.scale, database_images=DB, pairs_per_query=K, cases=[])
    with tempfile.TemporaryDirectory() as d:
        for Q in [int(x) for x in a.queries.split(",")]:
            names = ["q%05d.png" % i for i in range(Q)]
            parts = [query_part(tpls[i % TEMPLATES], names[i]) for i in range(Q)]
            batch = MatchSet.concatenate(parts)
            bf, bo = os.path.join(d, "batch.pb"), os.path.join(d, "batch_out.pb")
            wire.write_matching_file(batch, bf)
            args = ["--matches_file", bf, "--output_file", bo]
            for nm in names:
                args += ["--query_images", nm]
            runs = [run(args) for _ in range(a.reps)]
            got = image_messages(open(bo, "rb").read())
            n_loop = min(Q, a.loop)
            loop = np.zeros(3)
            for i in range(n_loop):
                qf, qo = os.path.join(d, "q.pb"), os.path.join(d, "q_out.pb")
                wire.write_matching_file(parts[i], qf)
                loop += run(["--matches_file", qf, "--output_file", qo])
                assert image_messages(open(qo, "rb").read())[names[i]] == got[names[i]], names[i]
            w = np.array(runs)
            res["cases"].append(dict(
                queries=Q, matches=int(batch.n_matches),
                batch_wall_ms=dict(best=float(w[:, 0].min()), median=float(np.median(w[:, 0]))),
                batch_total_ms=dict(best=int(w[:, 1].min()), median=float(np.median(w[:, 1]))),
                batch_solver_ms=dict(best=int(w[:, 2].min()), median=float(np.median(w[:, 2]))),
                loop_processes_timed=n_loop, loop_wall_ms=float(loop[0]), loop_total_ms=int(loop[1]),
                loop_solver_ms=int(loop[2]), loop_wall_ms_per_q=float(loop[0]) * Q / n_loop))
            print(json.dumps(res["cases"][-1]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
