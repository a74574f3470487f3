"""High-level host API: MatchSet -> refined displacements -> SolutionFile.

Mirrors the tail of solve.cc's main(): problem initialisation (positions = 0,
solve.cc:609-612), the solve (solve.cc:614-635, here one lfr_solve call into
csrc/liblfr_b200.so) and the output assembly (solve.cc:643-679).
"""
from __future__ import annotations

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


def assemble_solution(p: Problem, positions: np.ndarray) -> Solution:
    g = p.graph
    N = g.n_nodes
    if N == 0:
        return Solution([], np.zeros(0, np.float32), np.zeros(1, np.uint64), np.zeros(0, np.uint32),
                        np.zeros(0, np.float32), np.zeros(0, np.float32), 0)
    img_ids, first = np.unique(g.node_image, return_index=True)
    order = np.argsort(first, kind="stable")
    img_ids = img_ids[order]                      # images by first node appearance
    rank = np.full(int(g.node_image.max()) + 1, -1, dtype=np.int64)
    rank[img_ids] = np.arange(img_ids.shape[0])
    node_rank = rank[g.node_image]
    perm = np.argsort(node_rank, kind="stable")   # nodes grouped by image, ascending node index
    counts = np.bincount(node_rank, minlength=img_ids.shape[0])
    img_ptr = np.zeros(img_ids.shape[0] + 1, dtype=np.uint64)
    np.cumsum(counts, out=img_ptr[1:])
    pos = np.asarray(positions, dtype=np.float64).reshape(N, 2)
    n_out = int(np.count_nonzero((np.abs(pos[:, 1]) > 0.5) | (np.abs(pos[:, 0]) > 0.5)))
    return Solution(
        image_names=[g.image_names[i] for i in img_ids.tolist()],
        fact=np.array([g.image_fact[i] for i in img_ids.tolist()], dtype=np.float32),
        img_ptr=img_ptr,
        feature_idx=g.node_feat[perm].astype(np.uint32),
        di=pos[perm, 0].astype(np.float32),
        dj=pos[perm, 1].astype(np.float32),
        n_outside=n_out,
    )


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


def refine(ms: MatchSet, banned_images=(), options=None, log: Optional[Callable[[str], None]] = None,
           solve_fn=None, n_devices: int = 1, timing: Optional[dict] = None):
    """MatchSet -> (Problem, positions, stats, Solution).  `solve_fn(problem)`
    may be supplied to drive a different executor (the multi-GPU path; give `n_devices`).

    The graph stage runs where graph_stage_on_device() says.  On the device (Plan.from_matches) the problem
    stays in HBM and is solved there, `solve_fn` is not called, and the Problem's arrays come from
    Plan.export_graph(); `timing["solver_ms"]` (when `timing` is given) then covers solve + download."""
    from .capi import Plan, load_b200
    from .graph import host_input_arrays, problem_from_stage
    lib = load_b200()
    skip, arrs = host_input_arrays(ms, banned_images)
    if not graph_stage_on_device(lib, arrs, len(ms.image_names), n_devices):
        p = build_problem(ms, banned_images, log=log)
        fn = solve_fn if solve_fn is not None else (lambda q: solve_problem(q, options))
        pos, st = fn(p)
        return p, pos, st, assemble_solution(p, pos)
    plan = Plan.from_matches(lib, arrs, options=options, n_images=len(ms.image_names))
    try:
        p = problem_from_stage(ms, skip, plan.export_graph(), plan.sizes, "device", log)
        t1 = time.perf_counter()
        if p.graph.n_nodes:
            plan.solve()
            pos, st = plan.download()
        else:
            pos, st = solve_problem(p, options)
        if timing is not None:
            timing["solver_ms"] = (time.perf_counter() - t1) * 1e3
    finally:
        plan.close()
    return p, pos, st, assemble_solution(p, pos)
