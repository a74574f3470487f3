"""`multi-view-refinement/build/solve` — command-line surface of solve.cc:375-682.

    solve --matches_file X.pb --output_file Y.pb [--n_threads 8]
          [--banned_images NAME]...                      (solve.cc:379-385)

Same flags, same `.part.N` handling (solve.cc:416-424), same stdout lines
(solve.cc:484-485,534,549,589,591,606,638,641,670) and exit codes (0; 1 on a
command-line error, solve.cc:397-401; -1 = 255 when the input does not parse or
the output cannot be written, solve.cc:433-436,674-677), so
local-feature-evaluation/benchmark.py:100-104, eth/benchmark.py:108-112 and
custom_demo.py:101-105 run unchanged.  `--n_threads` is accepted and ignored
(the solve runs on the GPU).  Opt-in extras: --device, --gpus N (one process drives N GPUs), --stats_json,
--fixed_images NAME (repeatable: the image's keypoints are held constant, as roots are) and
--initial_solution FILE (start values from a SolutionFile instead of zeros): together they refine new
images against an already-refined scene.  --keep_initial_solution (with --initial_solution) also holds
every keypoint that has an entry in that file constant, and refines only the others.
--carry_initial_solution (with --initial_solution) writes the whole scene: the output also holds every entry
of that file the solve does not refine (wire.encode_solution_carried), so new pairs alone can be solved.
--update_initial_solution (with --initial_solution, not with --keep_initial_solution) solves every component
that a keypoint without an entry in that file joins from zeros, as a run without the file does, and holds
every other component at the file's values (wire.update_solution, Plan.update_solution).
--previous_matches_file OLD.pb (with --update_initial_solution; `.part.N` pieces as for --matches_file) names
the MatchingFile that produced the initial solution: a component is then also solved again when its problem
is not the one OLD.pb's run solved, so banned images, new pairs between old images and changed network output
no longer leave stale values (the rule is in include/lfr_graph.h).
--record_file FILE writes this run's problem record (one 128-bit digest per component, include/lfr_graph.h)
after the SolutionFile, and --earlier_record_file FILE (with --update_initial_solution, not with
--previous_matches_file) reads the record the run that produced the initial solution wrote, in place of its
MatchingFile: a component is unchanged when its digest is in that record (wire.problem_record,
Plan.problem_record, Plan.update_solution(previous_record=...)).
--query_images NAME (repeatable) localizes many queries in one run: a pair that names one query image belongs
to that query's sub-scene, a pair that names none is not solved, and each query is refined as a run on its
sub-scene's pairs alone refines it (solver.refine(query_images=...)).  Only query images are written.
--joint_queries (with --query_images) refines queries that a kept pair names together, such as the frames of a
sequence or the cameras of a rig, in one sub-scene: each query is refined as a run on its group's pairs alone
refines it (solver.refine(joint_queries=True)).
--additional_scenes FILE (lines `MATCHES_FILE<TAB>OUTPUT_FILE`) refines many scenes in one run: the scene of
--matches_file / --output_file and every listed one, each output file byte for byte what that scene's own run
writes (solver.refine_scenes).
--listed_pairs FILE (lines `MATCH_LIST<TAB>OUTPUT_FILE`) refines the pairs of many match lists (`NAME1 NAME2` per
line, as compute_match_graph.py reads them) out of --matches_file in one run: each output file byte for byte
what the run on a MatchingFile of that list's pairs in line order writes (solver.refine_lists).

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
            ("device", True, False), ("gpus", True, False), ("stats_json", True, False),
            ("fixed_images", True, True), ("initial_solution", True, False),
            ("keep_initial_solution", False, False), ("carry_initial_solution", False, False),
            ("update_initial_solution", False, False), ("previous_matches_file", True, False),
            ("record_file", True, False), ("earlier_record_file", True, False), ("query_images", True, True),
            ("joint_queries", False, False), ("additional_scenes", True, False),
            ("listed_pairs", True, False)]


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
            device=_as_uint(vals, "device", 0), gpus=_as_uint(vals, "gpus", 1), stats_json=vals.get("stats_json"),
            fixed_images=vals.get("fixed_images", []), initial_solution=vals.get("initial_solution"),
            keep_initial_solution=bool(vals.get("keep_initial_solution")),
            carry_initial_solution=bool(vals.get("carry_initial_solution")),
            update_initial_solution=bool(vals.get("update_initial_solution")),
            previous_matches_file=vals.get("previous_matches_file"),
            record_file=vals.get("record_file"), earlier_record_file=vals.get("earlier_record_file"),
            query_images=vals.get("query_images"), joint_queries=bool(vals.get("joint_queries")),
            additional_scenes=vals.get("additional_scenes"), listed_pairs=vals.get("listed_pairs"))
    except _CliError as e:                                  # solve.cc:397-401
        sys.stderr.write("ERROR: %s\n\n" % e)
        sys.stderr.write(USAGE)
        raise SystemExit(1)


def read_scene_list(path, matches_file, output_file):
    """--additional_scenes FILE: [(matches file, output file)] of scene 0 (--matches_file / --output_file) and
    of every line `MATCHES_FILE<TAB>OUTPUT_FILE` (raw bytes; the last newline optional), or the bytes of the one
    ERROR line for an unreadable file, a malformed line or two scenes with the same output path (lfr_solve_main.cc
    writes the same lines)."""
    try:
        with open(path, "rb") as fh:
            text = fh.read()
    except OSError:
        return b"ERROR: cannot read the scene list file '%s'\n" % os.fsencode(path)
    scenes = [(os.fsencode(matches_file), os.fsencode(output_file))]
    lines = text.split(b"\n")
    if lines[-1] == b"":
        lines.pop()
    for k, line in enumerate(lines, 1):
        why = ("it is empty" if not line else "it has no TAB" if b"\t" not in line
               else "it has more than one TAB" if line.count(b"\t") > 1
               else "its matches file is empty" if line.startswith(b"\t")
               else "its output file is empty" if line.endswith(b"\t")
               else "it holds a NUL byte" if b"\0" in line else None)
        if why:
            return b"ERROR: --additional_scenes: line %d is not MATCHES_FILE<TAB>OUTPUT_FILE: %s\n" % (k, why.encode())
        scenes.append(tuple(line.split(b"\t")))
    seen = set()
    for _, o in scenes:
        if o in seen:
            return b"ERROR: --additional_scenes: two scenes write '%s'\n" % o
        seen.add(o)
    return [(os.fsdecode(m), os.fsdecode(o)) for m, o in scenes]


def read_pair_lists(path, output_file):
    """--listed_pairs FILE: [(match list path or None, output file, [(name1, name2)] or None)], list 0 being every
    pair of --matches_file written to `output_file`, or the bytes of the one ERROR line for an unreadable file,
    a malformed line, two lists with the same output path, an unreadable match list or a malformed line of one
    (lfr_solve_main.cc writes the same lines, in the same order).  A match list's line is split as
    compute_match_graph.py:97 splits it: the newline stripped, split on single spaces, exactly two fields."""
    try:
        with open(path, "rb") as fh:
            text = fh.read()
    except OSError:
        return b"ERROR: cannot read the pair list file '%s'\n" % os.fsencode(path)
    lists = [(None, os.fsencode(output_file))]
    lines = text.split(b"\n")
    if lines[-1] == b"":
        lines.pop()
    for k, line in enumerate(lines, 1):
        why = ("it is empty" if not line else "it has no TAB" if b"\t" not in line
               else "it has more than one TAB" if line.count(b"\t") > 1
               else "its match list is empty" if line.startswith(b"\t")
               else "its output file is empty" if line.endswith(b"\t")
               else "it holds a NUL byte" if b"\0" in line else None)
        if why:
            return b"ERROR: --listed_pairs: line %d is not MATCH_LIST<TAB>OUTPUT_FILE: %s\n" % (k, why.encode())
        lists.append(tuple(line.split(b"\t")))
    seen = set()
    for _, o in lists:
        if o in seen:
            return b"ERROR: --listed_pairs: two lists write '%s'\n" % o
        seen.add(o)
    out = [(None, output_file, None)]
    for k, (m, o) in enumerate(lists[1:], 1):
        try:
            with open(m, "rb") as fh:
                t = fh.read()
        except OSError:
            return b"ERROR: --listed_pairs: line %d: cannot read the match list '%s'\n" % (k, m)
        rows = t.split(b"\n")
        if rows[-1] == b"":
            rows.pop()
        pairs = []
        for j, row in enumerate(rows, 1):
            f = row.split(b" ")
            if len(f) != 2:
                return (b"ERROR: --listed_pairs: line %d of the match list '%s' is not NAME1 NAME2: it has %d fields\n"
                        % (j, m, len(f)))
            pairs.append(tuple(x.decode("utf-8", errors="surrogateescape") for x in f))
        out.append((os.fsdecode(m), os.fsdecode(o), pairs))
    return out


def _run_lists(args, lists, ms, opts, say, solve_fn, n_devices, timing, t_start) -> int:
    """--listed_pairs after the lists were read: one refine_lists() run, the stdout lines once, then the output
    files in list order."""
    from .matchset import UnheldPairError
    from .solver import GraphStageRouteError, refine_lists
    sols = []
    try:
        data = refine_lists(ms, [pairs for _, _, pairs in lists], args.banned_images, opts, log=say, solve_fn=solve_fn,
                            n_devices=n_devices, timing=timing, solutions=sols)
    except UnheldPairError as e:
        enc = lambda x: x.encode("utf-8", errors="surrogateescape")  # noqa: E731
        msg = b"ERROR: --listed_pairs: line %d of the match list '%s': the matches file holds no pair '%s' '%s'" % (
            e.line, os.fsencode(lists[e.list][0]), enc(e.name1), enc(e.name2))
        if e.reverse:
            msg += b"; it holds only '%s' '%s'" % (enc(e.name2), enc(e.name1))
        sys.stderr.flush()
        sys.stderr.buffer.write(msg + b"\n")
        sys.stderr.buffer.flush()
        return 2
    except GraphStageRouteError as e:
        sys.stderr.write("ERROR: %s\n" % e)
        return 2
    except ValueError as e:   # more than 65535 image ids
        sys.stderr.write("ERROR: --%s\n" % e)
        return 2
    say("Solver time: %dms" % int(timing.get("solver_ms", 0.0)))                       # solve.cc:638
    say("Total time: %dms" % int((time.perf_counter() - t_start) * 1e3))               # solve.cc:641
    say("# points with at least one coordinate > 0.5: %d" % sum(s.n_outside for s in sols))   # solve.cc:670
    try:
        for (_, out, _), d in zip(lists, data):
            with open(out, "wb") as fh:
                fh.write(d)
    except OSError:
        sys.stderr.write("Failed to write proto object.\n")
        return 255
    return 0


def _run_scenes(args, scenes, ms, opts, say, solve_fn, n_devices, timing, t_start) -> int:
    """--additional_scenes after the scenes were read: one refine_scenes() run, the stdout lines once, then the
    output files in scene order."""
    from .solver import GraphStageRouteError, refine_scenes
    sols = []
    try:
        data = refine_scenes([m for m, _ in scenes], args.banned_images, opts, log=say, solve_fn=solve_fn,
                             n_devices=n_devices, timing=timing, solutions=sols)
    except GraphStageRouteError as e:
        sys.stderr.write("ERROR: %s\n" % e)
        return 2
    except ValueError as e:   # more than 65535 image ids
        sys.stderr.write("ERROR: --%s\n" % e)
        return 2
    say("Solver time: %dms" % int(timing.get("solver_ms", 0.0)))                       # solve.cc:638
    say("Total time: %dms" % int((time.perf_counter() - t_start) * 1e3))               # solve.cc:641
    say("# points with at least one coordinate > 0.5: %d" % sum(s.n_outside for s in sols))   # solve.cc:670
    try:
        for (_, out), d in zip(scenes, data):
            with open(out, "wb") as fh:
                fh.write(d)
    except OSError:
        sys.stderr.write("Failed to write proto object.\n")
        return 255
    return 0


def main(argv=None) -> int:
    args = parse_args(sys.argv[1:] if argv is None else argv)

    from . import wire
    from .solver import GraphStageRouteError, refine
    from .capi import load_b200
    from .graph import refined_track_count

    # the start solution is read and checked before any other work: its errors come before any output
    if args.keep_initial_solution and not args.initial_solution:
        sys.stderr.write("ERROR: --keep_initial_solution needs --initial_solution FILE\n")
        return 2
    if args.carry_initial_solution and not args.initial_solution:
        sys.stderr.write("ERROR: --carry_initial_solution needs --initial_solution FILE\n")
        return 2
    if args.update_initial_solution and not args.initial_solution:
        sys.stderr.write("ERROR: --update_initial_solution needs --initial_solution FILE\n")
        return 2
    if args.update_initial_solution and args.keep_initial_solution:
        sys.stderr.write("ERROR: --update_initial_solution and --keep_initial_solution exclude each other\n")
        return 2
    if args.previous_matches_file is not None and not args.update_initial_solution:
        sys.stderr.write("ERROR: --previous_matches_file needs --update_initial_solution\n")
        return 2
    if args.earlier_record_file is not None and not args.update_initial_solution:
        sys.stderr.write("ERROR: --earlier_record_file needs --update_initial_solution\n")
        return 2
    if args.earlier_record_file is not None and args.previous_matches_file is not None:
        sys.stderr.write("ERROR: --earlier_record_file and --previous_matches_file exclude each other\n")
        return 2
    if args.query_images is not None:
        for on, opt in ((args.update_initial_solution, "--update_initial_solution"),
                        (args.previous_matches_file is not None, "--previous_matches_file"),
                        (args.record_file is not None, "--record_file"),
                        (args.earlier_record_file is not None, "--earlier_record_file"),
                        (args.carry_initial_solution, "--carry_initial_solution")):
            if on:
                sys.stderr.write("ERROR: --query_images and %s exclude each other\n" % opt)
                return 2
    if args.joint_queries and args.query_images is None:
        sys.stderr.write("ERROR: --joint_queries needs --query_images\n")
        return 2
    lists = None
    if args.listed_pairs is not None:   # as --additional_scenes, whose batches it excludes too
        for on, opt in ((bool(args.fixed_images), "--fixed_images"), (args.initial_solution is not None, "--initial_solution"),
                        (args.keep_initial_solution, "--keep_initial_solution"),
                        (args.carry_initial_solution, "--carry_initial_solution"),
                        (args.update_initial_solution, "--update_initial_solution"),
                        (args.previous_matches_file is not None, "--previous_matches_file"),
                        (args.record_file is not None, "--record_file"),
                        (args.earlier_record_file is not None, "--earlier_record_file"),
                        (args.query_images is not None, "--query_images"), (args.joint_queries, "--joint_queries"),
                        (args.additional_scenes is not None, "--additional_scenes")):
            if on:
                sys.stderr.write("ERROR: --listed_pairs and %s exclude each other\n" % opt)
                return 2
        lists = read_pair_lists(args.listed_pairs, args.output_file)
        if isinstance(lists, bytes):
            sys.stderr.flush()
            sys.stderr.buffer.write(lists)
            sys.stderr.buffer.flush()
            return 2
    scenes = None
    if args.additional_scenes is not None:
        for on, opt in ((bool(args.fixed_images), "--fixed_images"), (args.initial_solution is not None, "--initial_solution"),
                        (args.keep_initial_solution, "--keep_initial_solution"),
                        (args.carry_initial_solution, "--carry_initial_solution"),
                        (args.update_initial_solution, "--update_initial_solution"),
                        (args.previous_matches_file is not None, "--previous_matches_file"),
                        (args.record_file is not None, "--record_file"),
                        (args.earlier_record_file is not None, "--earlier_record_file"),
                        (args.query_images is not None, "--query_images"), (args.joint_queries, "--joint_queries")):
            if on:
                sys.stderr.write("ERROR: --additional_scenes and %s exclude each other\n" % opt)
                return 2
        scenes = read_scene_list(args.additional_scenes, args.matches_file, args.output_file)
        if isinstance(scenes, bytes):
            sys.stderr.flush()
            sys.stderr.buffer.write(scenes)
            sys.stderr.buffer.flush()
            return 2
    start = None
    if args.initial_solution is not None:
        try:
            with open(args.initial_solution, "rb") as fh:
                start = fh.read()
        except OSError:
            sys.stderr.write("ERROR: cannot read the initial solution file '%s'\n" % args.initial_solution)
            return 2
        try:
            wire.decode_solution(start)
        except wire.ParseError:
            sys.stderr.write("Failed to parse proto object.\n")
            return 255
    previous = None
    if args.previous_matches_file is not None:
        try:
            if not wire.matches_files(args.previous_matches_file):
                raise OSError(args.previous_matches_file)
            previous = wire.read_matching_file(args.previous_matches_file)
        except OSError:
            sys.stderr.write("ERROR: cannot read the previous matches file '%s'\n" % args.previous_matches_file)
            return 2
        except wire.ParseError:
            sys.stderr.write("Failed to parse proto object.\n")
            return 255
    earlier_record = None
    if args.earlier_record_file is not None:
        try:
            with open(args.earlier_record_file, "rb") as fh:
                earlier_record = fh.read()
        except OSError:
            sys.stderr.write("ERROR: cannot read the earlier record file '%s'\n" % args.earlier_record_file)
            return 2
        if not wire.record_is_valid(earlier_record):
            sys.stderr.write("ERROR: '%s' is not a problem record\n" % args.earlier_record_file)
            return 2

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
    from .matchset import MatchSet
    if ms is None:
        ms = MatchSet.empty()
    if scenes is not None:
        # every scene's input is read before any output is written
        try:
            scenes = [(ms, scenes[0][1])] + [(wire.read_matching_file(m) if wire.matches_files(m) else MatchSet.empty(), o)
                                             for m, o in scenes[1:]]
        except wire.ParseError:
            sys.stderr.write("Failed to parse proto object.\n")
            return 255

    lib = load_b200()   # fails loudly when the CUDA library is missing
    opts = lib.default_options(device=args.device, n_threads=args.n_threads)
    t_start = time.perf_counter()
    timing = {}

    def solve_fn(p, positions=None):
        t1 = time.perf_counter()
        if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1:
            from .dist import solve_distributed       # launched under torchrun: one rank per GPU
            if positions is not None:
                raise GraphStageRouteError("--initial_solution: torchrun ranks start from zeros; use --gpus N")
            pos, st = solve_distributed(p)
        elif args.gpus > 1:
            # one call drives the GPUs (lfr_solve_multi, include/lfr.h): components LPT-packed over the
            # devices, each pulling only its own edge records from the page-locked arrays
            pos, st = lib.solve_multi(p, range(args.gpus), opts, positions=positions, pinned=True)
        else:
            from .solver import solve_problem
            pos, st = solve_problem(p, opts, positions)
        timing["solver_ms"] = (time.perf_counter() - t1) * 1e3
        return pos, st

    # torchrun ranks and --gpus N solve a host lfr_problem: the size rule keeps them on the host route
    torchrun = "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1
    n_devices = int(os.environ["WORLD_SIZE"]) if torchrun else max(args.gpus, 1)
    if torchrun and (args.record_file is not None or args.earlier_record_file is not None):
        sys.stderr.write("ERROR: --record_file / --earlier_record_file: torchrun ranks do not write or read "
                         "problem records; use --gpus N\n")
        return 2
    if torchrun and args.query_images is not None:
        sys.stderr.write("ERROR: --query_images: torchrun ranks do not localize queries; use --gpus N\n")
        return 2
    if torchrun and scenes is not None:
        sys.stderr.write("ERROR: --additional_scenes: torchrun ranks do not refine scene batches; use --gpus N\n")
        return 2
    if torchrun and lists is not None:
        sys.stderr.write("ERROR: --listed_pairs: torchrun ranks do not refine list batches; use --gpus N\n")
        return 2
    if lists is not None:
        return _run_lists(args, lists, ms, opts, say, solve_fn, n_devices, timing, t_start)
    if scenes is not None:
        return _run_scenes(args, scenes, ms, opts, say, solve_fn, n_devices, timing, t_start)
    try:
        p, pos, st, sol = refine(ms, args.banned_images, opts, log=say, solve_fn=solve_fn, n_devices=n_devices,
                                 timing=timing, fixed_images=args.fixed_images, initial_solution=start,
                                 keep_initial_solution=args.keep_initial_solution,
                                 update_initial_solution=args.update_initial_solution, previous_matches=previous,
                                 previous_record=earlier_record, record_problem=args.record_file is not None,
                                 query_images=args.query_images, joint_queries=args.joint_queries)
    except GraphStageRouteError as e:
        sys.stderr.write("ERROR: %s\n" % e)
        return 2
    except ValueError as e:   # --query_images: a pair that names two query images, or too many images
        if args.query_images is None:
            raise
        msg = str(e)   # refine() names its argument, the command line its option (lfr_solve_main.cc's line)
        sys.stderr.write("ERROR: %s\n" % ("--" + msg if msg.startswith("query_images:") else msg))
        return 2
    say("Solver time: %dms" % int(timing.get("solver_ms", 0.0)))                       # solve.cc:638
    say("Total time: %dms" % int((time.perf_counter() - t_start) * 1e3))               # solve.cc:641
    say("# points with at least one coordinate > 0.5: %d" % sol.n_outside)             # solve.cc:670
    if rank != 0:
        return 0
    try:
        if args.carry_initial_solution:
            data, _ = wire.encode_solution_carried(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di,
                                                   sol.dj, start)
        else:
            data = wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj)
        with open(args.output_file, "wb") as fh:
            fh.write(data)
    except OSError:
        sys.stderr.write("Failed to write proto object.\n")
        return 255
    if args.record_file is not None:
        try:
            with open(args.record_file, "wb") as fh:
                fh.write(sol.record)
        except OSError:
            sys.stderr.write("ERROR: cannot write the record file '%s'\n" % args.record_file)
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
