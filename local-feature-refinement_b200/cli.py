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
--versioned_scenes FILE (lines `MATCHES_FILE<TAB>OUTPUT_FILE<TAB>INITIAL_SOLUTION<TAB>EARLIER_RECORD<TAB>RECORD_FILE`,
the last three fields may be empty) updates many scenes in one run: a scene with an initial solution is updated
from it (and against its earlier record) as --update_initial_solution updates it alone, one without solves from
zeros, and each output and record file is byte for byte what that scene's own run writes (solver.refine_scenes with
initial_solutions, previous_records and record_problem).  Scene 0's start comes from the ordinary flags.
--task_stream FILE (with --device, --gpus and --n_threads alone) runs every line of FILE, read as it arrives, as a task
in one process: each line's TAB-separated fields are the argument vector of one main() run, and `# task K: exit C`
follows each on stdout, so torch and the library are loaded once (run_task_stream).

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
import traceback

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
            ("listed_pairs", True, False), ("versioned_scenes", True, False), ("task_stream", True, False)]


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
            if req not in vals and "task_stream" not in vals:   # a task stream's tasks name their own files
                raise _CliError("the option '--%s' is required but missing" % req)
        return argparse.Namespace(
            matches_file=vals.get("matches_file"), output_file=vals.get("output_file"),
            n_threads=_as_uint(vals, "n_threads", 8), banned_images=vals.get("banned_images", []),
            device=_as_uint(vals, "device", 0), gpus=_as_uint(vals, "gpus", 1), stats_json=vals.get("stats_json"),
            fixed_images=vals.get("fixed_images", []), initial_solution=vals.get("initial_solution"),
            keep_initial_solution=bool(vals.get("keep_initial_solution")),
            carry_initial_solution=bool(vals.get("carry_initial_solution")),
            update_initial_solution=bool(vals.get("update_initial_solution")),
            previous_matches_file=vals.get("previous_matches_file"),
            record_file=vals.get("record_file"), earlier_record_file=vals.get("earlier_record_file"),
            query_images=vals.get("query_images"), joint_queries=bool(vals.get("joint_queries")),
            additional_scenes=vals.get("additional_scenes"), listed_pairs=vals.get("listed_pairs"),
            versioned_scenes=vals.get("versioned_scenes"), task_stream=vals.get("task_stream"), named=set(vals))
    except _CliError as e:                                  # solve.cc:397-401
        sys.stderr.write("ERROR: %s\n\n" % e)
        sys.stderr.write(USAGE)
        raise SystemExit(1)


# The rules between the opt-in options, in order: with two conflicts, the first rule that fires writes the message
# (lfr_solve_main.cc has the same table).  (option, "needs" or "excludes", the others)
_ONE_SCENE = ["--fixed_images", "--initial_solution", "--keep_initial_solution", "--carry_initial_solution",
              "--update_initial_solution", "--previous_matches_file", "--record_file", "--earlier_record_file",
              "--query_images", "--joint_queries"]   # a batch's scenes or lists exclude what belongs to one scene
_RULES = [("--keep_initial_solution", "needs", ["--initial_solution"]),
          ("--carry_initial_solution", "needs", ["--initial_solution"]),
          ("--update_initial_solution", "needs", ["--initial_solution"]),
          ("--update_initial_solution", "excludes", ["--keep_initial_solution"]),
          ("--previous_matches_file", "needs", ["--update_initial_solution"]),
          ("--earlier_record_file", "needs", ["--update_initial_solution"]),
          ("--earlier_record_file", "excludes", ["--previous_matches_file"]),
          # each query is refined against the scene as it stands; the incremental modes update one scene
          ("--query_images", "excludes", ["--update_initial_solution", "--previous_matches_file", "--record_file",
                                          "--earlier_record_file", "--carry_initial_solution"]),
          ("--joint_queries", "needs", ["--query_images"]),
          ("--listed_pairs", "excludes", _ONE_SCENE + ["--additional_scenes"]),
          ("--additional_scenes", "excludes", _ONE_SCENE),
          # every scene of --versioned_scenes starts from its own solution and record, scene 0 from the ordinary flags
          ("--versioned_scenes", "excludes", ["--fixed_images", "--keep_initial_solution", "--carry_initial_solution",
                                              "--previous_matches_file", "--query_images", "--joint_queries",
                                              "--additional_scenes", "--listed_pairs"]),
          # a task stream's command line sets the process alone (--device, --gpus, --n_threads): every task names
          # its own files and options
          ("--task_stream", "excludes", ["--matches_file", "--output_file", "--banned_images", "--stats_json"]
           + _ONE_SCENE + ["--additional_scenes", "--listed_pairs", "--versioned_scenes"])]


def _broken_rule(args):
    """The ERROR line of the first rule in _RULES the command line breaks, or None.  An option is given when the
    command line names it; a needed option must also have a value (an empty --initial_solution names no file)."""
    value = lambda opt: getattr(args, opt[2:])  # noqa: E731
    given = lambda opt: value(opt) not in (None, False, [])  # noqa: E731
    for opt, kind, others in _RULES:
        for other in (others if given(opt) else ()):
            if kind == "needs" and not value(other):
                return "ERROR: %s needs %s%s\n" % (opt, other, " FILE" if other == "--initial_solution" else "")
            if kind == "excludes" and given(other):
                return "ERROR: %s and %s exclude each other\n" % (opt, other)
    # a batch's scenes are updated or solved from zeros: a start point alone belongs to one scene
    if given("--versioned_scenes") and args.initial_solution and not args.update_initial_solution:
        return "ERROR: --versioned_scenes: --initial_solution needs --update_initial_solution\n"
    return None


def _lines(data):
    """The lines of `data`; the last newline is optional."""
    lines = data.split(b"\n")
    if lines[-1] == b"":
        lines.pop()
    return lines


# the nouns of the two list files: (option, file, first column, what an empty first column is, rows)
_SCENE_LIST = (b"--additional_scenes", b"scene list", b"MATCHES_FILE", b"its matches file is empty", b"scenes")
_PAIR_LIST = (b"--listed_pairs", b"pair list", b"MATCH_LIST", b"its match list is empty", b"lists")


def _read_tab_list(path, kind, row0):
    """The list file of --additional_scenes or --listed_pairs (`kind`): [row0] and a (first, output) row of bytes for
    every line `FIRST<TAB>OUTPUT_FILE` (raw bytes; the last newline optional), or the bytes of the one ERROR line
    for an unreadable file, a malformed line or two rows with the same output path (lfr_solve_main.cc writes the
    same lines)."""
    option, noun, first, first_empty, rows_noun = kind
    try:
        with open(path, "rb") as fh:
            text = fh.read()
    except OSError:
        return b"ERROR: cannot read the %s file '%s'\n" % (noun, os.fsencode(path))
    rows = [row0]
    for k, line in enumerate(_lines(text), 1):
        why = (b"it is empty" if not line else b"it has no TAB" if b"\t" not in line
               else b"it has more than one TAB" if line.count(b"\t") > 1
               else first_empty if line.startswith(b"\t")
               else b"its output file is empty" if line.endswith(b"\t")
               else b"it holds a NUL byte" if b"\0" in line else None)
        if why:
            return b"ERROR: %s: line %d is not %s<TAB>OUTPUT_FILE: %s\n" % (option, k, first, why)
        rows.append(tuple(line.split(b"\t")))
    seen = set()
    for _, o in rows:
        if o in seen:
            return b"ERROR: %s: two %s write '%s'\n" % (option, rows_noun, o)
        seen.add(o)
    return rows


def read_scene_list(path, matches_file, output_file):
    """--additional_scenes FILE: [(matches file, output file)] of scene 0 (--matches_file / --output_file) and
    of every line `MATCHES_FILE<TAB>OUTPUT_FILE`, or the bytes of the one ERROR line (_read_tab_list)."""
    scenes = _read_tab_list(path, _SCENE_LIST, (os.fsencode(matches_file), os.fsencode(output_file)))
    return scenes if isinstance(scenes, bytes) else [(os.fsdecode(m), os.fsdecode(o)) for m, o in scenes]


_VERSIONED_LINE = b"MATCHES_FILE<TAB>OUTPUT_FILE<TAB>INITIAL_SOLUTION<TAB>EARLIER_RECORD<TAB>RECORD_FILE"


def read_versioned_list(path, row0):
    """--versioned_scenes FILE: [row0] and a (matches, output, initial solution, earlier record, record file) row of
    bytes (empty: none; a record file is None when the scene writes none, so scene 0's is None without
    --record_file and its path, empty or not, with it) for every line, or the bytes of the one ERROR line for an unreadable file, a malformed line or
    a file that two outputs or records would write (lfr_solve_main.cc writes the same lines)."""
    try:
        with open(path, "rb") as fh:
            text = fh.read()
    except OSError:
        return b"ERROR: cannot read the scene list file '%s'\n" % os.fsencode(path)
    rows = [row0]
    for k, line in enumerate(_lines(text), 1):
        f = line.split(b"\t")
        why = (b"it is empty" if not line else b"it has fewer than four TABs" if len(f) < 5
               else b"it has more than four TABs" if len(f) > 5
               else b"its matches file is empty" if not f[0]
               else b"its output file is empty" if not f[1]
               else b"it holds a NUL byte" if b"\0" in line
               else b"it has an earlier record but no initial solution" if f[3] and not f[2] else None)
        if why:
            return b"ERROR: --versioned_scenes: line %d is not %s: %s\n" % (k, _VERSIONED_LINE, why)
        rows.append(tuple(f[:4]) + (f[4] or None,))
    seen = set()
    for row in rows:
        for w in (row[1], row[4]):
            if w and w in seen:
                return b"ERROR: --versioned_scenes: two files written are '%s'\n" % w
            seen.add(w)
    return rows


def read_versioned_starts(rows, start, earlier_record):
    """Every scene's (initial solution bytes or None, earlier record bytes or None) of the read_versioned_list() rows,
    scene 0's being `start` and `earlier_record`, or the bytes of the one ERROR line naming the list's line."""
    from . import wire
    out = [(start, earlier_record)]
    for k, (_, _, init, earlier, _) in enumerate(rows[1:], 1):
        sol = rec = None
        if init:
            try:
                with open(init, "rb") as fh:
                    sol = fh.read()
            except OSError:
                return b"ERROR: --versioned_scenes: line %d: cannot read the initial solution file '%s'\n" % (k, init)
            try:
                wire.decode_solution(sol)
            except wire.ParseError:
                return b"ERROR: --versioned_scenes: line %d: the initial solution file '%s' does not parse\n" % (k, init)
        if earlier:
            try:
                with open(earlier, "rb") as fh:
                    rec = fh.read()
            except OSError:
                return b"ERROR: --versioned_scenes: line %d: cannot read the earlier record file '%s'\n" % (k, earlier)
            if not wire.record_is_valid(rec):
                return b"ERROR: --versioned_scenes: line %d: '%s' is not a problem record\n" % (k, earlier)
        out.append((sol, rec))
    return out


def read_pair_lists(path, output_file):
    """--listed_pairs FILE: [(match list path or None, output file, [(name1, name2)] or None)], list 0 being every
    pair of --matches_file written to `output_file`, or the bytes of the one ERROR line for what _read_tab_list
    refuses, an unreadable match list or a malformed line of one (lfr_solve_main.cc writes the same lines, in the
    same order).  A match list's line is split as compute_match_graph.py:97 splits it: the newline stripped, split
    on single spaces, exactly two fields."""
    lists = _read_tab_list(path, _PAIR_LIST, (None, os.fsencode(output_file)))
    if isinstance(lists, bytes):
        return lists
    out = [(None, output_file, None)]
    for k, (m, o) in enumerate(lists[1:], 1):
        try:
            with open(m, "rb") as fh:
                t = fh.read()
        except OSError:
            return b"ERROR: --listed_pairs: line %d: cannot read the match list '%s'\n" % (k, m)
        pairs = []
        for j, row in enumerate(_lines(t), 1):
            f = row.split(b" ")
            if len(f) != 2:
                return (b"ERROR: --listed_pairs: line %d of the match list '%s' is not NAME1 NAME2: it has %d fields\n"
                        % (j, m, len(f)))
            pairs.append(tuple(x.decode("utf-8", errors="surrogateescape") for x in f))
        out.append((os.fsdecode(m), os.fsdecode(o), pairs))
    return out


def _run_batch(refine_batch, inputs, rows, args, opts, say, solve_fn, n_devices, timing, t_start, starts=None) -> int:
    """--additional_scenes, --listed_pairs or --versioned_scenes after the rows (scenes or lists, each with its output
    file second; with --versioned_scenes its record file fifth) were read: one refine_batch(*inputs, ...) run
    (refine_scenes or refine_lists; `starts`: every scene's (initial solution, earlier record)), the stdout lines
    once, then the output files in row order and the record files in row order."""
    from .matchset import UnheldPairError
    from .solver import GraphStageRouteError
    sols = []
    extra = {}
    records = [None if r[4] is None else os.fsdecode(r[4]) for r in rows] if starts is not None else []
    if starts is not None:
        extra = dict(initial_solutions=[s for s, _ in starts], previous_records=[r for _, r in starts],
                     record_problem=any(r is not None for r in records))
    try:
        data = refine_batch(*inputs, args.banned_images, opts, log=say, solve_fn=solve_fn, n_devices=n_devices,
                            timing=timing, solutions=sols, **extra)
    except UnheldPairError as e:   # --listed_pairs: a list line whose pair the file does not hold
        enc = lambda x: x.encode("utf-8", errors="surrogateescape")  # noqa: E731
        msg = b"ERROR: --listed_pairs: line %d of the match list '%s': the matches file holds no pair '%s' '%s'" % (
            e.line, os.fsencode(rows[e.list][0]), enc(e.name1), enc(e.name2))
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
        for row, d in zip(rows, data):
            with open(row[1], "wb") as fh:
                fh.write(d)
    except OSError:
        sys.stderr.write("Failed to write proto object.\n")
        return 255
    for path, sol in zip(records, sols):
        if path is None:
            continue
        try:
            with open(path, "wb") as fh:
                fh.write(sol.record)
        except OSError:
            sys.stderr.write("ERROR: cannot write the record file '%s'\n" % path)
            return 255
    return 0


def main(argv=None) -> int:
    args = parse_args(sys.argv[1:] if argv is None else argv)
    if args.task_stream is not None:
        return run_task_stream(args)
    return _run(args)


# library return codes after which the CUDA context may be unusable (include/lfr.h)
_LOST = (-2, -3)   # LFR_ENODEV, LFR_ECUDA


def _run_task(argv, stream):
    """One task of a stream: (exit code, whether the context may be lost) of the run of `argv` as a one-shot process
    runs it, under the stream's --device and --gpus; a task may not set those or --task_stream (exit code 2)."""
    try:
        args = parse_args(argv)
        for name in ("task_stream", "device", "gpus"):
            if name in args.named:
                sys.stderr.write("ERROR: --%s is set once, on the task stream's command line\n" % name)
                return 2, False
        args.device, args.gpus = stream.device, stream.gpus
        return _run(args), False
    except SystemExit as e:   # as the interpreter turns it into an exit code
        if e.code is None or isinstance(e.code, int):
            return (e.code or 0) & 0xFF, False
        sys.stderr.write("%s\n" % e.code)
        return 1, False
    except Exception as e:     # an uncaught exception: the traceback and exit code 1, as the interpreter ends a run
        traceback.print_exc()
        return 1, getattr(e, "lfr_rc", None) in _LOST


def run_task_stream(args) -> int:
    """--task_stream FILE: every line of FILE, read as it arrives (a FIFO or /dev/stdin serves), is one task whose
    argument vector is the line's TAB-separated fields (none for an empty line), run as main() runs it.  After each,
    its files are closed and `# task K: exit C` is on stdout, flushed, before the next line is read.  A failed task
    ends itself alone, unless a library call returned LFR_ECUDA or LFR_ENODEV: the stream then ends with exit code 2.
    The end of FILE ends it with 0.  lfr_solve_main.cc runs the same loop."""
    broken = _broken_rule(args)
    if broken:
        sys.stderr.write(broken)
        return 2
    if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        sys.stderr.write("ERROR: --task_stream: torchrun ranks do not run task streams; use --gpus N\n")
        return 2
    try:
        fh = open(args.task_stream, "rb", buffering=0)
    except OSError:
        sys.stderr.write("ERROR: cannot read the task stream file '%s'\n" % args.task_stream)
        return 2
    with fh:
        k = 0
        while True:
            line = _read_line(fh)
            if line is None:
                return 0
            code, lost = _run_task([os.fsdecode(a) for a in line.split(b"\t")] if line else [], args)
            sys.stderr.flush()
            sys.stdout.write("# task %d: exit %d\n" % (k, code))
            sys.stdout.flush()
            if lost:
                return 2
            k += 1


def _read_line(fh):
    """The next line of the unbuffered file `fh` without its newline (the last one is optional), or None at its end.
    Bytes are read one at a time, so no byte past the newline is taken before the task is done."""
    buf = bytearray()
    while True:
        c = fh.read(1)
        if not c:
            return bytes(buf) if buf else None
        if c == b"\n":
            return bytes(buf)
        buf += c


def _run(args) -> int:
    """One run of the parsed command line `args`."""
    from . import wire
    from .solver import GraphStageRouteError, refine, refine_lists, refine_scenes

    from .capi import load_b200
    from .graph import refined_track_count

    # the rules, then the start solution read and checked before any other work: their errors come before any output
    broken = _broken_rule(args)
    if broken:
        sys.stderr.write(broken)
        return 2
    lists = None
    if args.listed_pairs is not None:
        lists = read_pair_lists(args.listed_pairs, args.output_file)
        if isinstance(lists, bytes):
            sys.stderr.flush()
            sys.stderr.buffer.write(lists)
            sys.stderr.buffer.flush()
            return 2
    scenes = None
    if args.additional_scenes is not None:
        scenes = read_scene_list(args.additional_scenes, args.matches_file, args.output_file)
        if isinstance(scenes, bytes):
            sys.stderr.flush()
            sys.stderr.buffer.write(scenes)
            sys.stderr.buffer.flush()
            return 2
    versioned = None
    if args.versioned_scenes is not None:
        enc = lambda x: b"" if x is None else os.fsencode(x)  # noqa: E731
        versioned = read_versioned_list(args.versioned_scenes, (enc(args.matches_file), enc(args.output_file),
                                                                enc(args.initial_solution), enc(args.earlier_record_file),
                                                                None if args.record_file is None
                                                                else os.fsencode(args.record_file)))
        if isinstance(versioned, bytes):
            sys.stderr.flush()
            sys.stderr.buffer.write(versioned)
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
    starts = None
    if versioned is not None:
        starts = read_versioned_starts(versioned, start, earlier_record)
        if isinstance(starts, bytes):
            sys.stderr.flush()
            sys.stderr.buffer.write(starts)
            sys.stderr.buffer.flush()
            return 2
        scenes = [(os.fsdecode(r[0]), os.fsdecode(r[1])) for r in versioned]

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
    for on, msg in ((args.record_file is not None or args.earlier_record_file is not None,
                     "--record_file / --earlier_record_file: torchrun ranks do not write or read problem records"),
                    (args.query_images is not None, "--query_images: torchrun ranks do not localize queries"),
                    (args.additional_scenes is not None, "--additional_scenes: torchrun ranks do not refine scene batches"),
                    (lists is not None, "--listed_pairs: torchrun ranks do not refine list batches"),
                    (versioned is not None, "--versioned_scenes: torchrun ranks do not refine scene batches")):
        if torchrun and on:
            sys.stderr.write("ERROR: %s; use --gpus N\n" % msg)
            return 2
    batch = (args, opts, say, solve_fn, n_devices, timing, t_start)
    if lists is not None:
        return _run_batch(refine_lists, (ms, [pairs for _, _, pairs in lists]), lists, *batch)
    if versioned is not None:
        return _run_batch(refine_scenes, ([m for m, _ in scenes],), versioned, *batch, starts=starts)
    if scenes is not None:
        return _run_batch(refine_scenes, ([m for m, _ in scenes],), scenes, *batch)
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
