"""Time --listed_pairs: K match lists refined out of one superset MatchingFile.

    python tools/gpu_listed_pairs_time.py [--configs cfg4,cfg5] [--ks 1,4,8] [--reps 3] [--out FILE]

The superset is synth's scene of the config.  Its lists are sequential windows (pairs whose two images are at
most w apart in the file's image order, w = 1, 2, ...) and retrieval-style subsets (a random half of the pairs in
a random order), alternating, K in all.  Per (config, K) and repetition:
  batch     the native drop-in once: --matches_file the superset (list 0, every pair) and the K lists in the
            --listed_pairs file;
  loop      the native drop-in once per list on that list's own MatchingFile (filtered out of the superset
            beforehand, not timed), plus once on the superset for list 0;
  per_list  in one process, the plan of the same batch made by lfr_plan_create_from_wire() with one part per
            list: the superset's bytes once per list, each with the match offsets of that list's pairs, so the
            file goes up and is decoded K + 1 times instead of expanded — against
            Plan.from_wire_listed() on the same batch (`expand`; its time also holds that call's pair walk in
            Python, so it is an upper bound of the expand route).
Wall times in ms.  Every loop output is checked against the batch's file for that list, byte for byte, and the
two plans' exported arrays against each other.  Prints one JSON object with the GPU's name and power limit (read,
never set)."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_update_since_time import NATIVE, gpu_info  # noqa: E402
from lfr_b200 import synth, wire  # noqa: E402
from lfr_b200.capi import LfrWirePart, Plan, load_b200  # noqa: E402
from lfr_b200.graph import HostInput, HostSizes  # noqa: E402
from lfr_b200.matchset import sub_scene_ids  # noqa: E402


def run(args):
    t0 = time.perf_counter()
    r = subprocess.run([NATIVE] + args, capture_output=True, text=True, check=True)
    return (time.perf_counter() - t0) * 1e3, int(re.search(r"Total time: (\d+)ms", r.stdout).group(1))


def make_lists(ms, k, seed):
    lines = [(ms.image_names[a], ms.image_names[b]) for a, b in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist())]
    order = {n: i for i, n in enumerate(ms.image_names)}
    rng = np.random.default_rng(seed)
    out = []
    for i in range(k):
        if i % 2 == 0:
            w = i // 2 + 1
            out.append([l for l in lines if abs(order[l[1]] - order[l[0]]) <= w])
        else:
            out.append([lines[j] for j in rng.permutation(len(lines))[: len(lines) // 2]])
    return out


def per_list_parts(ms, data, lists):
    """The parts of lfr_plan_create_from_wire() for the batch of Plan.from_wire_listed(data, [None] + lists): one
    per list, the superset's bytes with that list's match offsets in list order.  Returns (parts, the offset
    arrays they point into, the file's pair of every entry per list)."""
    a = wire.walk_matching_file(data)
    sp = np.ascontiguousarray(a["pair_ptr"], np.uint64)
    buf = np.frombuffer(data, np.uint8)
    groups = [np.arange(ms.n_pairs)] + [ms.listed_pair_index(l) for l in lists]
    offs = [np.ascontiguousarray(np.concatenate([a["match_off"][sp[p]:sp[p + 1]] for p in g.tolist()] or
                                                [np.zeros(0, np.uint64)]), np.uint64) for g in groups]
    parts = (LfrWirePart * len(groups))(*[LfrWirePart(buf=buf.ctypes.data, len=buf.size,
                                                      match_off=o.ctypes.data if o.size else None, n_matches=o.size)
                                          for o in offs])
    return parts, offs, groups


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg4,cfg5")
    ap.add_argument("--ks", default="1,4,8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = load_b200()
    res = dict(gpu=gpu_info(), runs=[])
    for cfg in a.configs.split(","):
        tmp = tempfile.mkdtemp(prefix="lfr_listed_pairs_")
        ms = synth.generate(cfg)
        sup = os.path.join(tmp, "superset.pb")
        wire.write_matching_file(ms, sup)
        data = open(sup, "rb").read()
        for k in [int(x) for x in a.ks.split(",")]:
            lists = make_lists(ms, k, seed=k)
            paths = []
            for i, ls in enumerate(lists):
                p = os.path.join(tmp, "k%d_l%d" % (k, i))
                with open(p + ".txt", "w") as fh:
                    fh.writelines("%s %s\n" % l for l in ls)
                with open(p + ".pb", "wb") as fh:
                    fh.write(wire.encode_matching_file(ms.select_listed_pairs(ls)))
                paths.append(p)
            with open(os.path.join(tmp, "pairs.txt"), "w") as fh:
                fh.writelines("%s.txt\t%s.batch\n" % (p, p) for p in paths)
            batch_args = ["--matches_file", sup, "--output_file", sup + ".batch", "--listed_pairs",
                          os.path.join(tmp, "pairs.txt")]
            run(batch_args)                                   # warm-up: page cache, driver
            r = dict(config=cfg, k=k, pairs=ms.n_pairs, matches=ms.n_matches,
                     listed_matches=[int(ms.select_listed_pairs(l).n_matches) for l in lists], batch=[], loop=[],
                     expand_ms=[], per_list_ms=[])
            for _ in range(a.reps):
                r["batch"].append(dict(zip(("wall_ms", "total_time_ms"), run(batch_args))))
                walls, totals = 0.0, 0
                for m in [sup] + [p + ".pb" for p in paths]:
                    w, t = run(["--matches_file", m, "--output_file", m + ".own"])
                    walls += w
                    totals += t
                r["loop"].append(dict(wall_ms=walls, total_time_ms=totals))
            r["identical"] = all(open(p + ".pb.own", "rb").read() == open(p + ".batch", "rb").read() for p in paths) and \
                open(sup + ".own", "rb").read() == open(sup + ".batch", "rb").read()
            # the plan alone, in this process: the expand against one decode per list
            opts = lib.default_options()
            ref = None
            for _ in range(a.reps):
                t0 = time.perf_counter()
                pl = Plan.from_wire_listed(lib, [data], [None] + lists, (), opts)
                r["expand_ms"].append((time.perf_counter() - t0) * 1e3)
                ref = pl.export_graph()
                pl.close()
            parts, offs, groups = per_list_parts(ms, data, lists)
            src = np.concatenate(groups).astype(np.int64)
            label = np.repeat(np.arange(len(groups)), [g.shape[0] for g in groups])
            e1, e2, orig_of, group = sub_scene_ids(ms.pair_img1[src], ms.pair_img2[src], label)
            cnt = (ms.pair_ptr[1:] - ms.pair_ptr[:-1])[src]
            ptr = np.zeros(src.shape[0] + 1, np.uint64)
            np.cumsum(cnt, out=ptr[1:])
            arrs = dict(pair_img1=e1.astype(np.uint32), pair_img2=e2.astype(np.uint32),
                        pair_skip=np.zeros(src.shape[0], np.uint8), pair_ptr=ptr, image_group=group)
            inp = HostInput(n_pairs=src.shape[0], n_matches=int(ptr[-1]), n_images=len(orig_of),
                            **{kk: (v.ctypes.data if v.size else None) for kk, v in arrs.items()})
            same = True
            for _ in range(a.reps):
                h, sz = C.c_void_p(), HostSizes()
                t0 = time.perf_counter()
                lib.check(lib.lib.lfr_plan_create_from_wire(C.byref(inp), parts, len(groups), C.byref(opts), None,
                                                            C.byref(h), C.byref(sz)), "lfr_plan_create_from_wire")
                r["per_list_ms"].append((time.perf_counter() - t0) * 1e3)
                pl = Plan.__new__(Plan)
                pl.lib, pl.problem, pl.handle = lib, None, h
                pl.sizes = {kk: getattr(sz, kk) for kk in ("n_edges",)}
                pl.n_nodes, pl.n_components = int(sz.n_nodes), int(sz.n_components)
                got = pl.export_graph()
                same = same and all(got[kk].tobytes() == ref[kk].tobytes() for kk in ref)
                pl.close()
            r["per_list_plan_identical"] = same
            best = lambda xs: min(x["wall_ms"] for x in xs)  # noqa: E731
            r["wall_speedup_best"] = best(r["loop"]) / best(r["batch"])
            res["runs"].append(r)
            print(json.dumps(r), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
