"""Time --additional_scenes: one process that refines S six-image scenes against S processes, one per scene.

    python tools/gpu_scene_batch_time.py [--scenes 116] [--reps 3] [--out FILE]

Every scene is HPatches-shaped: six images named 1.ppm .. 6.ppm, all 15 pairs matched (synth, 0.1 of cfg2's
keypoints per image, its own seed).  116 scenes are the HPatches Sequences.  Per repetition:
  batch  the native drop-in once, scene 0 on the command line and the other S - 1 in the --additional_scenes list;
  loop   the native drop-in once per scene.
Each reports the wall time of the processes and the sums of their "Total time" lines.  Every loop output is
checked against the batch's file for that scene, byte for byte.  Prints one JSON object with the GPU's name and
power limit (read, never set)."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_update_since_time import NATIVE, gpu_info  # noqa: E402
from lfr_b200 import synth, wire  # noqa: E402


def scene(seed):
    cfg = synth.SynthConfig("hp", 6, synth.CONFIGS["cfg2"].kpts, "exhaustive", 0.8, seed=seed)
    ms = synth.generate(cfg, scale=0.1, seed=seed)
    ms.image_names = ["%d.ppm" % (i + 1) for i in range(6)]
    return ms


def run(args):
    t0 = time.perf_counter()
    r = subprocess.run([NATIVE] + args, capture_output=True, text=True, check=True)
    return (time.perf_counter() - t0) * 1e3, int(re.search(r"Total time: (\d+)ms", r.stdout).group(1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=116)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="lfr_scene_batch_")
    paths, n_matches = [], 0
    for k in range(a.scenes):
        ms = scene(1000 + k)
        n_matches += ms.n_matches
        paths.append(os.path.join(tmp, "seq_%03d.pb" % k))
        wire.write_matching_file(ms, paths[-1])
    with open(os.path.join(tmp, "list.txt"), "w") as fh:
        fh.writelines("%s\t%s.batch\n" % (m, m) for m in paths[1:])
    batch_args = ["--matches_file", paths[0], "--output_file", paths[0] + ".batch", "--additional_scenes",
                  os.path.join(tmp, "list.txt")]
    run(batch_args)                                   # warm-up: page cache, driver
    res = dict(gpu=gpu_info(), scenes=a.scenes, images=6 * a.scenes, matches=n_matches, batch=[], loop=[])
    for _ in range(a.reps):
        res["batch"].append(dict(zip(("wall_ms", "total_time_ms"), run(batch_args))))
        walls, totals = 0.0, 0
        for m in paths:
            w, t = run(["--matches_file", m, "--output_file", m + ".own"])
            walls += w
            totals += t
        res["loop"].append(dict(wall_ms=walls, total_time_ms=totals))
    res["identical"] = all(open(m + ".own", "rb").read() == open(m + ".batch", "rb").read() for m in paths)
    best = lambda xs: min(x["wall_ms"] for x in xs)
    res["wall_speedup_best"] = best(res["loop"]) / best(res["batch"])
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
