"""`multi-view-refinement/build/solve` — command-line surface of solve.cc:375-682.

    solve --matches_file X.pb --output_file Y.pb [--n_threads 8]
          [--banned_images NAME]...                      (solve.cc:379-385)

Same flags, same `.part.N` handling (solve.cc:416-424), same stdout lines
(solve.cc:484-485,534,549,589,591,606,638,641,670) and exit codes (0; 1 on a
command-line error, solve.cc:397-401; -1 = 255 when the input does not parse or
the output cannot be written, solve.cc:433-436,674-677), so
local-feature-evaluation/benchmark.py:100-104, eth/benchmark.py:108-112 and
custom_demo.py:101-105 run unchanged.  `--n_threads` is accepted and ignored
(the solve runs on the GPU).  Opt-in extras: --device, --gpus N (one process drives N GPUs), --stats_json.

The graph stage (solve.cc:438-606) runs where the library's size rule says
(lfr_graph_stage_on_device, include/lfr_graph.h): on the device for large inputs
(Plan.from_matches; the problem is solved where it was built), on the host
otherwise and for torchrun ranks and --gpus N.  LFR_GRAPH_STAGE=host|device
forces a route (a test and measurement hook); `--stats_json` reports it as
info.host_stage ("device", or "native" / "numpy" on the host route).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

USAGE = """Options:
  --help                    print the help
  --matches_file arg        path to the matches file
  --output_file arg         path to the output file
  --n_threads arg (=8)      # threads
  --banned_images arg (={}) banned images
"""


class _CliError(Exception):
    pass


# (name, takes an argument, repeatable) — solve.cc:379-385 plus the opt-in extras
_OPTIONS = [("help", False, False), ("matches_file", True, False), ("output_file", True, False),
            ("n_threads", True, False), ("banned_images", True, True),
            ("device", True, False), ("gpus", True, False), ("stats_json", True, False)]


def _find_option(name):
    """Exact name, else unambiguous prefix (Boost.Program_options' default allow_guessing)."""
    hits = [o for o in _OPTIONS if o[0].startswith(name)]
    for o in _OPTIONS:
        if o[0] == name:
            return o
    if len(hits) == 1:
        return hits[0]
    if len(hits) > 1:
        raise _CliError("option '--%s' is ambiguous" % name)
    raise _CliError("unrecognised option '--%s'" % name)


def _parse(argv):
    """Boost.Program_options semantics of solve.cc:387-401 (long options, `--name value` or
    `--name=value`, no positional arguments), with Boost's error messages."""
    vals = {}
    i = 0
    while i < len(argv):
        tok = argv[i]
        i += 1
        if tok.startswith("--") and len(tok) > 2:
            name, eq, adjacent = tok[2:].partition("=")
            oname, takes, repeat = _find_option(name)
            if takes:
                if eq:
                    v = adjacent
                elif i < len(argv) and not (argv[i].startswith("-") and len(argv[i]) > 1):
                    v = argv[i]
                    i += 1
                else:
                    raise _CliError("the required argument for option '--%s' is missing" % oname)
                if repeat:
                    vals.setdefault(oname, []).append(v)
                elif oname in vals:
                    raise _CliError("option '--%s' cannot be specified more than once" % oname)
                else:
                    vals[oname] = v
            else:
                if eq:
                    raise _CliError("option '--%s' does not take any arguments" % oname)
                vals[oname] = True
        elif tok.startswith("-") and len(tok) > 1:
            raise _CliError("unrecognised option '%s'" % tok)
        else:
            raise _CliError("too many positional options have been specified on the command line")
    return vals


def _as_uint(vals, name, default):
    if name not in vals:
        return default
    v = vals[name]
    if not v.isdigit():      # lexical_cast<size_t>
        raise _CliError("the argument ('%s') for option '--%s' is invalid" % (v, name))
    return int(v)


def parse_args(argv):
    try:
        vals = _parse(list(argv))
        if vals.get("help"):
            sys.stdout.write("Patch Match graph problem solver\n\n" + USAGE)
            raise SystemExit(0)
        for req in ("matches_file", "output_file"):        # po::notify: required options, in declaration order
            if req not in vals:
                raise _CliError("the option '--%s' is required but missing" % req)
        return argparse.Namespace(
            matches_file=vals["matches_file"], output_file=vals["output_file"],
            n_threads=_as_uint(vals, "n_threads", 8), banned_images=vals.get("banned_images", []),
            device=_as_uint(vals, "device", 0), gpus=_as_uint(vals, "gpus", 1), stats_json=vals.get("stats_json"))
    except _CliError as e:                                  # solve.cc:397-401
        sys.stderr.write("ERROR: %s\n\n" % e)
        sys.stderr.write(USAGE)
        raise SystemExit(1)


def main(argv=None) -> int:
    args = parse_args(sys.argv[1:] if argv is None else argv)

    from . import wire
    from .solver import GraphStageRouteError, refine
    from .capi import load_b200
    from .graph import refined_track_count

    rank = int(os.environ.get("RANK", "0"))
    say = (lambda s: print(s, flush=True)) if rank == 0 else (lambda s: None)
    if not wire.matches_files(args.matches_file):
        # the reference parses zero files and writes an empty solution
        pass
    try:
        if args.matches_file.endswith(".npz") and os.path.exists(args.matches_file):
            from .matchset import MatchSet
            ms = MatchSet.load_npz(args.matches_file)   # packed arrays written by MatchSet.save_npz (opt-in extra)
        else:
            ms = wire.read_matching_file(args.matches_file) if wire.matches_files(args.matches_file) else None
    except wire.ParseError:
        sys.stderr.write("Failed to parse proto object.\n")
        return 255
    if ms is None:
        from .matchset import MatchSet
        import numpy as np
        ms = MatchSet([], np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32),
                      np.zeros(0, np.float32), np.zeros(1, np.int64), np.zeros(0, np.uint32),
                      np.zeros(0, np.uint32), np.zeros(0, np.float32), np.zeros((0, 18), np.float32),
                      np.zeros((0, 18), np.float32))

    lib = load_b200()   # fails loudly when the CUDA library is missing
    opts = lib.default_options(device=args.device, n_threads=args.n_threads)
    t_start = time.perf_counter()
    timing = {}

    def solve_fn(p):
        t1 = time.perf_counter()
        if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1:
            from .dist import solve_distributed       # launched under torchrun: one rank per GPU
            pos, st = solve_distributed(p)
        elif args.gpus > 1:
            # one call drives the GPUs (lfr_solve_multi, include/lfr.h): components LPT-packed over the
            # devices, each pulling only its own edge records from the page-locked arrays
            pos, st = lib.solve_multi(p, range(args.gpus), opts, pinned=True)
        else:
            from .solver import solve_problem
            pos, st = solve_problem(p, opts)
        timing["solver_ms"] = (time.perf_counter() - t1) * 1e3
        return pos, st

    # torchrun ranks and --gpus N solve a host lfr_problem: the size rule keeps them on the host route
    torchrun = "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1
    n_devices = int(os.environ["WORLD_SIZE"]) if torchrun else max(args.gpus, 1)
    try:
        p, pos, st, sol = refine(ms, args.banned_images, opts, log=say, solve_fn=solve_fn, n_devices=n_devices,
                                 timing=timing)
    except GraphStageRouteError as e:
        sys.stderr.write("ERROR: %s\n" % e)
        return 2
    say("Solver time: %dms" % int(timing.get("solver_ms", 0.0)))                       # solve.cc:638
    say("Total time: %dms" % int((time.perf_counter() - t_start) * 1e3))               # solve.cc:641
    say("# points with at least one coordinate > 0.5: %d" % sol.n_outside)             # solve.cc:670
    if rank != 0:
        return 0
    try:
        data = wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj)
        with open(args.output_file, "wb") as fh:
            fh.write(data)
    except OSError:
        sys.stderr.write("Failed to write proto object.\n")
        return 255
    if args.stats_json:
        n_tracks = refined_track_count(p)
        solver_s = max(timing.get("solver_ms", 0.0), 1e-9) / 1e3
        out = dict(n_nodes=p.graph.n_nodes, n_edges=p.graph.n_edges, info=p.info,
                   tracks_refined=n_tracks, lm_iterations=int(st.get("total_iterations", 0)),
                   solver_ms=timing.get("solver_ms"), kernel_ms=st.get("kernel_ms"), h2d_ms=st.get("h2d_ms"),
                   d2h_ms=st.get("d2h_ms"), tracks_per_s=n_tracks / solver_s,
                   lm_iters_per_s=int(st.get("total_iterations", 0)) / solver_s)
        with open(args.stats_json, "w") as fh:
            json.dump(out, fh, indent=1, default=float)
    return 0


if __name__ == "__main__":
    if __package__ in (None, ""):
        sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        import lfr_b200.cli as _cli
        raise SystemExit(_cli.main())
    raise SystemExit(main())
