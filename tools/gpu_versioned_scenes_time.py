"""Time --versioned_scenes: one process that updates S six-image scenes after one new image per scene, against S
processes, one per scene.

    python tools/gpu_versioned_scenes_time.py [--scenes 116] [--reps 3] [--out FILE]

Every scene is HPatches-shaped (tools/gpu_scene_batch_time.py's scenes).  Round 0 runs every scene on five of its
six images, one process per scene, each writing its SolutionFile and problem record.  Round 1 adds the sixth image
to every scene and, per repetition:
  batch  the native drop-in once, scene 0 on the command line (--initial_solution --update_initial_solution
         --earlier_record_file --record_file) and the other S - 1 in the --versioned_scenes list;
  loop   the native drop-in once per scene with the same flags.
Each reports the wall time of the processes and the sums of their "Total time" lines.  Every loop output and record
is checked against the batch's files for that scene, byte for byte.  Prints one JSON object with the GPU's name and
power limit (read, never set)."""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_scene_batch_time import run, scene  # noqa: E402
from gpu_update_since_time import gpu_info  # noqa: E402
from lfr_b200 import wire  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=116)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="lfr_versioned_scenes_")
    paths, n_matches = [], 0
    for k in range(a.scenes):
        ms = scene(1000 + k)
        n_matches += ms.n_matches
        p = os.path.join(tmp, "seq_%03d" % k)
        wire.write_matching_file(ms.without_images(["6.ppm"]), p + ".0.pb")
        wire.write_matching_file(ms, p + ".1.pb")
        run(["--matches_file", p + ".0.pb", "--output_file", p + ".0.sol", "--record_file", p + ".0.rec"])
        paths.append(p)

    def flags(p, tag):
        return ["--matches_file", p + ".1.pb", "--output_file", p + ".%s.sol" % tag, "--initial_solution", p + ".0.sol",
                "--update_initial_solution", "--earlier_record_file", p + ".0.rec", "--record_file", p + ".%s.rec" % tag]
    with open(os.path.join(tmp, "list.txt"), "w") as fh:
        fh.writelines("%s.1.pb\t%s.batch.sol\t%s.0.sol\t%s.0.rec\t%s.batch.rec\n" % (p, p, p, p, p) for p in paths[1:])
    batch_args = flags(paths[0], "batch") + ["--versioned_scenes", os.path.join(tmp, "list.txt")]
    run(batch_args)                                   # warm-up: page cache, driver
    res = dict(gpu=gpu_info(), scenes=a.scenes, images=6 * a.scenes, matches=n_matches, batch=[], loop=[])
    for _ in range(a.reps):
        res["batch"].append(dict(zip(("wall_ms", "total_time_ms"), run(batch_args))))
        walls, totals = 0.0, 0
        for p in paths:
            w, t = run(flags(p, "own"))
            walls += w
            totals += t
        res["loop"].append(dict(wall_ms=walls, total_time_ms=totals))
    same = lambda x, y: open(x, "rb").read() == open(y, "rb").read()  # noqa: E731
    res["identical"] = all(same(p + ".own.sol", p + ".batch.sol") and same(p + ".own.rec", p + ".batch.rec")
                           for p in paths)
    best = lambda xs: min(x["wall_ms"] for x in xs)  # noqa: E731
    res["wall_speedup_best"] = best(res["loop"]) / best(res["batch"])
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
