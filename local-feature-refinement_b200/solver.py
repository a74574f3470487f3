"""High-level host API: MatchSet -> refined displacements -> SolutionFile.

Mirrors the tail of solve.cc's main(): problem initialisation (positions = 0,
solve.cc:609-612), the solve (solve.cc:614-635, here one lfr_solve call into
csrc/liblfr_b200.so) and the output assembly (solve.cc:643-679).
"""
from __future__ import annotations

import dataclasses
import os
import time
from dataclasses import dataclass
from typing import Callable, List, Optional

import numpy as np

from .graph import Problem, build_problem
from .matchset import MatchSet


@dataclass
class Solution:
    """SolutionFile content (types.proto:30-46) in the reference's order:
    images by first node appearance, displacements by node index (solve.cc:647-664)."""
    image_names: List[str]
    fact: np.ndarray          # [I] float32
    img_ptr: np.ndarray       # [I+1]
    feature_idx: np.ndarray   # [N] uint32
    di: np.ndarray            # [N] float32 (row displacement, positions[node][0])
    dj: np.ndarray            # [N] float32 (col displacement, positions[node][1])
    n_outside: int            # "# points with at least one coordinate > 0.5" (solve.cc:666-670)
    record: Optional[bytes] = None  # the run's problem record (include/lfr_graph.h), with refine(record_problem=True)


def assemble_solution(p: Problem, positions: np.ndarray, written: Optional[np.ndarray] = None) -> Solution:
    """`written` [n_images] bool (--query_images): only these images get an Image message; every node still
    counts towards n_outside."""
    g = p.graph
    N = g.n_nodes
    if N == 0:
        return Solution([], np.zeros(0, np.float32), np.zeros(1, np.uint64), np.zeros(0, np.uint32),
                        np.zeros(0, np.float32), np.zeros(0, np.float32), 0)
    img_ids, first = np.unique(g.node_image, return_index=True)
    order = np.argsort(first, kind="stable")
    img_ids = img_ids[order]                      # images by first node appearance
    pos = np.asarray(positions, dtype=np.float64).reshape(N, 2)
    n_out = int(np.count_nonzero((np.abs(pos[:, 1]) > 0.5) | (np.abs(pos[:, 0]) > 0.5)))
    nodes = np.arange(N)
    if written is not None:
        img_ids = img_ids[np.asarray(written, dtype=bool)[img_ids]]
        nodes = np.nonzero(np.asarray(written, dtype=bool)[g.node_image])[0]
    rank = np.full(int(g.node_image.max()) + 1, -1, dtype=np.int64)
    rank[img_ids] = np.arange(img_ids.shape[0])
    node_rank = rank[g.node_image[nodes]]
    perm = nodes[np.argsort(node_rank, kind="stable")]   # nodes grouped by image, ascending node index
    counts = np.bincount(node_rank, minlength=img_ids.shape[0])
    img_ptr = np.zeros(img_ids.shape[0] + 1, dtype=np.uint64)
    np.cumsum(counts, out=img_ptr[1:])
    return Solution(
        image_names=[g.image_names[i] for i in img_ids.tolist()],
        fact=np.array([g.image_fact[i] for i in img_ids.tolist()], dtype=np.float32),
        img_ptr=img_ptr,
        feature_idx=g.node_feat[perm].astype(np.uint32),
        di=pos[perm, 0].astype(np.float32),
        dj=pos[perm, 1].astype(np.float32),
        n_outside=n_out,
    )


def assemble_scene_solutions(p: Problem, positions: np.ndarray, image_group: np.ndarray, n_groups: int) -> List[Solution]:
    """--additional_scenes: the Solution of every group g < n_groups (image_group[id] = the group of image id),
    each equal to assemble_solution(p, positions, written=image_group == g) with n_outside counted on the
    group's own nodes; one sort of the images by (group, first node) for all groups."""
    g = p.graph
    N = g.n_nodes
    empty = Solution([], np.zeros(0, np.float32), np.zeros(1, np.uint64), np.zeros(0, np.uint32),
                     np.zeros(0, np.float32), np.zeros(0, np.float32), 0)
    if N == 0:
        return [dataclasses.replace(empty) for _ in range(n_groups)]
    image_group = np.asarray(image_group, dtype=np.int64)
    img_ids, first = np.unique(g.node_image, return_index=True)
    order = np.lexsort((first, image_group[img_ids]))
    img_ids = img_ids[order]                      # by group, then by first node appearance
    pos = np.asarray(positions, dtype=np.float64).reshape(N, 2)
    node_group = image_group[g.node_image]
    outside = (np.abs(pos[:, 1]) > 0.5) | (np.abs(pos[:, 0]) > 0.5)
    n_out = np.bincount(node_group[outside], minlength=n_groups)
    rank = np.full(int(g.node_image.max()) + 1, -1, dtype=np.int64)
    rank[img_ids] = np.arange(img_ids.shape[0])
    node_rank = rank[g.node_image]
    perm = np.argsort(node_rank, kind="stable")   # nodes by image in output order, ascending node index
    node_ptr = np.zeros(img_ids.shape[0] + 1, dtype=np.int64)
    np.cumsum(np.bincount(node_rank, minlength=img_ids.shape[0]), out=node_ptr[1:])
    img_bound = np.searchsorted(image_group[img_ids], np.arange(n_groups + 1))
    feat, di, dj = g.node_feat[perm].astype(np.uint32), pos[perm, 0].astype(np.float32), pos[perm, 1].astype(np.float32)
    out = []
    for k in range(n_groups):
        a, b = int(img_bound[k]), int(img_bound[k + 1])
        lo, hi = int(node_ptr[a]), int(node_ptr[b])
        ids = img_ids[a:b].tolist()
        out.append(Solution(image_names=[g.image_names[i] for i in ids],
                            fact=np.array([g.image_fact[i] for i in ids], dtype=np.float32),
                            img_ptr=(node_ptr[a:b + 1] - lo).astype(np.uint64), feature_idx=feat[lo:hi], di=di[lo:hi],
                            dj=dj[lo:hi], n_outside=int(n_out[k])))
    return out


def solve_problem(p: Problem, options=None, positions: Optional[np.ndarray] = None):
    """One lfr_solve call on the CUDA library.  Returns (positions [N,2], stats)."""
    from .capi import load_b200
    lib = load_b200()
    if p.graph.n_nodes == 0:
        return np.zeros((0, 2)), dict(total_iterations=0, n_solved=0, total_ms=0.0, kernel_ms=0.0,
                                      h2d_ms=0.0, d2h_ms=0.0, n_kernel_launches=0,
                                      total_line_search_steps=0)
    return lib.solve(p, options, positions)


class GraphStageRouteError(RuntimeError):
    """LFR_GRAPH_STAGE asks for a route this run cannot take."""


def graph_stage_on_device(lib, arrs: dict, n_images: int, n_devices: int = 1) -> bool:
    """Where the graph stage of the flat lfr_host_input arrays `arrs` (graph.host_input_arrays) runs:
    the library's size rule (lfr_graph_stage_on_device, include/lfr_graph.h), unless LFR_GRAPH_STAGE=host|device
    forces a route (a test and measurement hook).  Forcing the device route where `lib` has no graph stage
    on the GPU, or for more than one device, raises GraphStageRouteError: it never runs the host stage instead."""
    force = os.environ.get("LFR_GRAPH_STAGE") or ""
    if force == "host":
        return False
    if force == "device":
        if not lib.has_graph_stage:
            raise GraphStageRouteError("LFR_GRAPH_STAGE=device: the solve library has no graph stage on the GPU")
        if n_devices != 1:
            raise GraphStageRouteError("LFR_GRAPH_STAGE=device: the graph stage on the GPU drives one device (--gpus 1)")
        return True
    if force:
        raise GraphStageRouteError("LFR_GRAPH_STAGE must be 'host' or 'device'")
    return lib.graph_stage_on_device(arrs, n_images, n_devices)


def fixed_image_mask(image_names: List[str], fixed_images) -> np.ndarray:
    """[n_images] bool by image id: the images named in `fixed_images` (names not in the scene are ignored,
    as banned names are)."""
    fixed = set(fixed_images)
    return np.array([n in fixed for n in image_names], dtype=bool).reshape(-1)


def constant_problem(p: Problem, fixed_images=(), initial_solution: Optional[bytes] = None,
                     keep_initial_solution: bool = False, update_initial_solution: bool = False,
                     previous_matches: Optional[MatchSet] = None, previous_record: Optional[bytes] = None,
                     image_group: Optional[np.ndarray] = None, scene_solutions=None, scene_records=None):
    """The host route's problem initialisation with fixed images and a start solution: (the Problem to solve,
    whose is_root is the constant mask = reference root OR node of a fixed image OR, with
    `keep_initial_solution`, node with an entry in the start solution OR, with `update_initial_solution`,
    node of a component the start solution covers whole (wire.update_solution) and, with `previous_matches`,
    that is unchanged since that MatchingFile's run (wire.update_solution_since) or, with `previous_record`,
    whose digest is in that run's problem record (wire.update_solution_since_record); start positions [N, 2]
    from wire.join_solution or wire.update_solution(_since(_record)), or None for zeros).

    With `scene_solutions` (one per scene of `image_group`: SolutionFile bytes or None) every scene is updated as its
    own run from its own file and, where scene_records[g] is not None, against that earlier record
    (wire.update_solution_groups); a scene without a file solves from zeros."""
    from . import wire
    g = p.graph
    const = np.asarray(p.is_root) != 0
    if len(fixed_images) and g.n_nodes:
        const = const | fixed_image_mask(g.image_names, fixed_images)[np.asarray(g.node_image, np.int64)]
    start = None
    if scene_solutions is not None:
        if any(x is not None for x in scene_solutions):
            start, held, _, _, _ = wire.update_solution_groups(scene_solutions, p, image_group, scene_records)
            const = const | held
    elif initial_solution is not None and update_initial_solution and previous_record is not None:
        start, held, _, _, _ = wire.update_solution_since_record(initial_solution, p, previous_record)
        const = const | held
    elif initial_solution is not None and update_initial_solution and previous_matches is not None:
        start, held, _, _, _ = wire.update_solution_since(initial_solution, p, previous_matches)
        const = const | held
    elif initial_solution is not None and update_initial_solution:
        start, held, _, _ = wire.update_solution(initial_solution, g.image_names, g.node_image, g.node_feat, p.comp,
                                                 p.n_components)
        const = const | held
    elif initial_solution is not None:
        start, _, has_entry = wire.join_solution(initial_solution, g.image_names, g.node_image, g.node_feat, entries=True)
        if keep_initial_solution:
            const = const | has_entry
    if (len(fixed_images) or keep_initial_solution or update_initial_solution or scene_solutions is not None) and g.n_nodes:
        return dataclasses.replace(p, is_root=const.astype(np.uint8)), start
    return p, start


def refine(ms: MatchSet, banned_images=(), options=None, log: Optional[Callable[[str], None]] = None,
           solve_fn=None, n_devices: int = 1, timing: Optional[dict] = None, fixed_images=(),
           initial_solution: Optional[bytes] = None, keep_initial_solution: bool = False,
           update_initial_solution: bool = False, previous_matches=None, previous_record: Optional[bytes] = None,
           record_problem: bool = False, query_images=None, joint_queries: bool = False,
           image_group: Optional[np.ndarray] = None, scene_solutions=None, scene_records=None,
           n_groups: Optional[int] = None):
    """MatchSet -> (Problem, positions, stats, Solution).  `solve_fn(problem)`
    may be supplied to drive a different executor (the multi-GPU path; give `n_devices`); with a start
    solution it is called as `solve_fn(problem, positions)`.

    `fixed_images` (names) hold every node of those images constant, as a root is: it keeps its start value.
    `initial_solution` (SolutionFile bytes) gives the start values (wire.join_solution) instead of zeros.
    Together they refine new images against an already-refined scene.  `keep_initial_solution` (needs
    `initial_solution`) also holds every node with an entry in that file constant (the rule of
    wire.join_solution), so only the keypoints it does not list are refined.  `update_initial_solution`
    (needs `initial_solution`, excludes `keep_initial_solution`) solves every component with a keypoint the
    file does not list from zeros, as without the file, and holds every other component at the file's
    values (wire.update_solution, Plan.update_solution).  `previous_matches` (needs `update_initial_solution`;
    a MatchSet or MatchingFile bytes) is the MatchingFile that produced `initial_solution`: a component is then
    also touched when its problem is not the one that file's run solved (include/lfr_graph.h states the
    rule; wire.update_solution_since, Plan.update_solution(previous=...)).  `previous_record` (needs
    `update_initial_solution`, excludes `previous_matches`) is that run's problem record instead: a component is
    unchanged when its digest is in the record (wire.update_solution_since_record,
    Plan.update_solution(previous_record=...)).  With `record_problem` the returned Solution's `record` is this
    run's problem record (wire.problem_record on the host route, Plan.problem_record on the device route; the
    same bytes), for the next update.  The returned Problem keeps the reference's is_root.

    The graph stage runs where graph_stage_on_device() says.  On the device (Plan.from_matches) the problem
    stays in HBM and is solved there, `solve_fn` is not called, and the Problem's arrays come from
    Plan.export_graph(); `timing["solver_ms"]` (when `timing` is given) then covers solve + download.

    `query_images` (names; names not in `ms` are ignored) localizes many queries in one run: every query is
    refined against the rest of the scene on its own (MatchSet.query_subscenes), and each query's Image
    message is the one a run on its sub-scene's pairs alone writes.  Only query images are written.  It
    excludes update_initial_solution, previous_matches, previous_record and record_problem (ValueError); a
    pair that names two query images, or sub-scenes of more than 65535 images in all, raise ValueError too.
    `joint_queries` (needs `query_images`) refines queries that a kept pair names together (sequences, rigs) in
    one sub-scene: a group is a connected component of the queries under such pairs, and each query's Image
    message is the one a run on its group's pairs alone writes.

    `image_group` ([n_images], MatchSet.join_scenes) stages every group of ids as a scene of its own, as
    refine_scenes() does; it excludes query_images (ValueError).  With it, `n_groups` scenes, `scene_solutions`
    (one SolutionFile or None per scene) and `scene_records` (one earlier problem record or None per scene) update
    every scene as its own run (Plan.update_solution_groups, wire.update_solution_groups), and `record_problem`
    makes the Solution's `record` the list of every scene's problem record (Plan.problem_record_groups,
    wire.problem_record_groups)."""
    from .capi import Plan, load_b200
    from .graph import host_input_arrays, problem_from_stage
    if keep_initial_solution and initial_solution is None:
        raise ValueError("keep_initial_solution needs initial_solution")
    if update_initial_solution and initial_solution is None:
        raise ValueError("update_initial_solution needs initial_solution")
    if update_initial_solution and keep_initial_solution:
        raise ValueError("update_initial_solution and keep_initial_solution exclude each other")
    if previous_matches is not None and not update_initial_solution:
        raise ValueError("previous_matches needs update_initial_solution")
    if previous_record is not None and not update_initial_solution:
        raise ValueError("previous_record needs update_initial_solution")
    if previous_record is not None and previous_matches is not None:
        raise ValueError("previous_record and previous_matches exclude each other")
    if previous_record is not None:
        from .wire import record_is_valid
        previous_record = bytes(previous_record)
        if not record_is_valid(previous_record):
            raise ValueError("malformed problem record")
    if joint_queries and query_images is None:
        raise ValueError("joint_queries needs query_images")
    if image_group is not None and query_images is not None:
        raise ValueError("image_group and query_images exclude each other")
    if query_images is not None:
        for on, what in ((update_initial_solution, "update_initial_solution"), (previous_matches is not None, "previous_matches"),
                         (previous_record is not None, "previous_record"), (record_problem, "record_problem")):
            if on:
                raise ValueError("query_images and %s exclude each other" % what)
        # one scene of disjoint sub-scenes: database images get one id per sub-scene (their names repeat, and
        # the joins and the fixed mask, which go by name, give every copy the same values)
        ms, image_group = ms.query_subscenes(query_images, banned_images, joint=joint_queries)
        banned_images = ()
        if len(ms.image_names) > 65535:
            raise ValueError("query_images: the sub-scenes hold %d images, more than 65535; split the query list over "
                             "several runs" % len(ms.image_names))
        queries = set(query_images)
        written = np.array([n in queries for n in ms.image_names], dtype=bool)
    else:
        written = None
    if isinstance(previous_matches, (bytes, bytearray, memoryview)):
        from .wire import decode_matching_file
        previous_matches = decode_matching_file(bytes(previous_matches))
    lib = load_b200()
    skip, arrs = host_input_arrays(ms, banned_images, image_group)
    if not graph_stage_on_device(lib, arrs, len(ms.image_names), n_devices):
        p = build_problem(ms, banned_images, log=log, image_group=image_group)
        q, start = constant_problem(p, fixed_images, initial_solution, keep_initial_solution, update_initial_solution,
                                    previous_matches, previous_record, image_group, scene_solutions, scene_records)
        fn = solve_fn if solve_fn is not None else (lambda q_, x=None: solve_problem(q_, options, x))
        pos, st = fn(q) if start is None else fn(q, start)
        sol = assemble_solution(p, pos, written)
        if record_problem and image_group is not None:
            from .wire import problem_record_groups
            sol.record = problem_record_groups(p, image_group, n_groups)
        elif record_problem:
            from .wire import problem_record
            sol.record = problem_record(p, ms.image_names)
        return p, pos, st, sol
    plan = Plan.from_matches(lib, arrs, options=options, n_images=len(ms.image_names))
    try:
        if len(fixed_images) and fixed_image_mask(ms.image_names, fixed_images).any():
            plan.fix_images(fixed_image_mask(ms.image_names, fixed_images))
        if scene_solutions is not None:
            if any(x is not None for x in scene_solutions):
                plan.update_solution_groups(scene_solutions, ms.image_names, image_group, scene_records)
        elif update_initial_solution and previous_record is not None:
            plan.update_solution(initial_solution, ms.image_names, previous_record=previous_record)
        elif update_initial_solution and previous_matches is not None:
            prev = Plan.from_matches(lib, previous_matches, options=options)
            try:
                plan.update_solution(initial_solution, ms.image_names, previous=prev)
            finally:
                prev.close()
        elif update_initial_solution:
            plan.update_solution(initial_solution, ms.image_names)
        elif keep_initial_solution:
            plan.keep_solution(initial_solution, ms.image_names)
        elif initial_solution is not None:
            plan.start_from_solution(initial_solution, ms.image_names)
        p = problem_from_stage(ms, skip, plan.export_graph(), plan.sizes, "device", log)
        t1 = time.perf_counter()
        if p.graph.n_nodes:
            plan.solve()
            pos, st = plan.download()
        else:
            pos, st = solve_problem(p, options)
        if timing is not None:
            timing["solver_ms"] = (time.perf_counter() - t1) * 1e3
        if record_problem and image_group is not None:
            record = plan.problem_record_groups(ms.image_names, image_group, n_groups)
        else:
            record = plan.problem_record(ms.image_names) if record_problem else None
    finally:
        plan.close()
    sol = assemble_solution(p, pos, written)
    sol.record = record
    return p, pos, st, sol


def refine_scenes(match_sets: List[MatchSet], banned_images=(), options=None, log: Optional[Callable[[str], None]] = None,
                  solve_fn=None, n_devices: int = 1, timing: Optional[dict] = None,
                  solutions: Optional[list] = None, initial_solutions=None, previous_records=None,
                  record_problem: bool = False) -> List[bytes]:
    """--additional_scenes: refine many scenes in one run and return one SolutionFile per scene, each byte for
    byte what refine() + wire.encode_solution write for that scene alone with the same `banned_images` (names,
    applied to every scene).  The scenes are one ordinary run (MatchSet.join_scenes: every scene a sub-scene
    with its own image ids), so its route, `log` lines and statistics are those of the whole batch: the counts
    are the sums over the scenes' own runs and the maxima their maxima.  `solutions`, when given, receives
    every scene's Solution (its n_outside is the scene's own count).  More than 65535 image ids over all
    scenes raise ValueError.

    `initial_solutions` and `previous_records` (--versioned_scenes) are per-scene lists, None meaning none for that
    scene: a scene with a SolutionFile is updated from it as refine(update_initial_solution=True) updates a scene
    alone, against its own earlier problem record when it has one (a record without a SolutionFile raises
    ValueError); a scene without one solves from zeros.  With `record_problem` every scene's Solution in
    `solutions` gets the problem record of its own run in `record`.  Each scene's bytes and record are those of its
    own run."""
    G = len(match_sets)
    for name, lst in (("initial_solutions", initial_solutions), ("previous_records", previous_records)):
        if lst is not None and len(lst) != G:
            raise ValueError("%s has %d entries for %d scenes" % (name, len(lst), G))
    if previous_records is not None:
        from .wire import record_is_valid
        for k, r in enumerate(previous_records):
            if r is not None and (initial_solutions is None or initial_solutions[k] is None):
                raise ValueError("previous_records[%d] needs initial_solutions[%d]" % (k, k))
            if r is not None and not record_is_valid(bytes(r)):
                raise ValueError("previous_records[%d] is not a problem record" % k)
    if initial_solutions is not None and previous_records is None:
        previous_records = [None] * G
    return _refine_batch(match_sets, banned_images, options, log, solve_fn, n_devices, timing, solutions,
                         "additional_scenes: the scenes hold %d images, more than 65535; split the scene list over "
                         "several runs", initial_solutions, previous_records, record_problem)


def _refine_batch(match_sets, banned_images, options, log, solve_fn, n_devices, timing, solutions, too_many: str,
                  initial_solutions=None, previous_records=None, record_problem=False):
    """refine_scenes() and refine_lists(): `too_many` % n_ids is the ValueError past 65535 image ids."""
    from .wire import encode_solution
    ms, image_group = MatchSet.join_scenes(match_sets, banned_images)
    if len(ms.image_names) > 65535:
        raise ValueError(too_many % len(ms.image_names))
    p, pos, _, whole = refine(ms, (), options, log=log, solve_fn=solve_fn, n_devices=n_devices, timing=timing,
                              image_group=image_group, scene_solutions=initial_solutions, scene_records=previous_records,
                              n_groups=len(match_sets), record_problem=record_problem)
    sols = assemble_scene_solutions(p, pos, image_group, len(match_sets))
    if record_problem:
        for sol, rec in zip(sols, whole.record):
            sol.record = rec
    if solutions is not None:
        solutions.extend(sols)
    return [encode_solution(s.image_names, s.fact, s.img_ptr, s.feature_idx, s.di, s.dj) for s in sols]


def refine_lists(ms: MatchSet, match_lists, banned_images=(), options=None, log: Optional[Callable[[str], None]] = None,
                 solve_fn=None, n_devices: int = 1, timing: Optional[dict] = None,
                 solutions: Optional[list] = None) -> List[bytes]:
    """--listed_pairs: refine the pairs of many match lists out of one superset MatchingFile `ms` and return one
    SolutionFile per list.  A list is a sequence of (name1, name2) lines, or None for every pair of `ms` in file
    order.  List L's bytes are those of refine() + wire.encode_solution on the MatchingFile that holds one pair
    per line of L in line order (MatchSet.select_listed_pairs: the first pair of `ms` with exactly those two
    names), with the same `banned_images`.  The lists run as one scene batch (refine_scenes' code), so the
    stdout lines and `solutions` are those of a scene batch.  A line whose pair `ms` does not hold raises
    matchset.UnheldPairError (its `list` attribute is the list's index); more than 65535 image ids over all
    lists raise ValueError."""
    from .matchset import UnheldPairError
    sets = []
    for k, lines in enumerate(match_lists):
        try:
            sets.append(ms if lines is None else ms.select_listed_pairs(lines))
        except UnheldPairError as e:
            e.list = k
            raise
    return _refine_batch(sets, banned_images, options, log, solve_fn, n_devices, timing, solutions,
                         "listed_pairs: the lists hold %d images, more than 65535; split the pair list over several runs")
