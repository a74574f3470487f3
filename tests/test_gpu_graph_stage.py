"""The graph stage on the GPU (include/lfr_graph.h, csrc/lfr_graph.cuh) against the host stage
(include/lfr_host.h, csrc/lfr_host.cc): every exported array, the 80-byte edge records included, and
every count of lfr_host_sizes must be bitwise equal; a plan made from matches must solve to exactly
what lfr_solve() gives on the host-stage problem.

The CPU tests check the algorithm the device Kruskal uses — deterministic reservations over a window
of the pending edges — against the sequential constrained Kruskal, in numpy, without a device.
"""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from lfr_b200 import synth
from lfr_b200.capi import GRAPH_SYMBOLS, Plan
from lfr_b200.graph import HOST_SIZES_FIELDS, host_input_arrays, host_stage_export

LFR_EINVAL, LFR_EUNSUPPORTED = -1, -5
ARRAYS = ("row_ptr", "edges", "track", "comp", "is_root", "comp_ptr", "comp_nodes", "comp_order", "node_image", "node_feat")
COUNTS = tuple(k for k in HOST_SIZES_FIELDS if not k.endswith("_ms"))


# ---------------------------------------------------------------------------------------------------
# CPU: deterministic reservations reproduce the sequential constrained Kruskal
# ---------------------------------------------------------------------------------------------------
def _sequential(node_image, n1, n2):
    """solve.cc:499-523 as lfr_host.cc runs it: edges in the given order; smaller image set under the
    larger, tie: root2 under root1; an image clash rejects."""
    parent = np.full(len(node_image), -1, np.int64)
    sets = [{int(i)} for i in node_image]

    def find(x):
        while parent[x] != -1:
            x = parent[x]
        return x
    for a, b in zip(n1, n2):
        r1, r2 = find(a), find(b)
        if r1 == r2 or sets[r1] & sets[r2]:
            continue
        if len(sets[r1]) < len(sets[r2]):
            parent[r1] = r2
            sets[r2] |= sets[r1]
        else:
            parent[r2] = r1
            sets[r1] |= sets[r2]
    return parent


def _reservations(node_image, n1, n2, window):
    """The device's rounds (kr_reserve / kr_decide / kr_release in lfr_graph.cuh), in numpy."""
    parent = np.full(len(node_image), -1, np.int64)
    sets = [{int(i)} for i in node_image]
    M = len(n1)

    def find(x):
        while parent[x] != -1:
            x = parent[x]
        return x
    win, nxt, rounds = list(range(min(window, M))), min(window, M), 0
    while win:
        rounds += 1
        roots = [(find(n1[r]), find(n2[r])) for r in win]            # reserve: all finds first
        res = {}
        for r, (r1, r2) in zip(win, roots):
            if r1 != r2:
                res[r1] = min(res.get(r1, M), r)
                res[r2] = min(res.get(r2, M), r)
        keep = []
        decisions = []
        for r, (r1, r2) in zip(win, roots):                           # decide on the reserved state
            if r1 == r2:
                continue
            if res[r1] == r and res[r2] == r:
                decisions.append((r1, r2))
            else:
                keep.append(r)
        for r1, r2 in decisions:                                       # disjoint roots: order is irrelevant
            if sets[r1] & sets[r2]:
                continue
            if len(sets[r1]) < len(sets[r2]):
                parent[r1] = r2
                sets[r2] |= sets[r1]
            else:
                parent[r2] = r1
                sets[r1] |= sets[r2]
        add = min(window - len(keep), M - nxt)
        win = keep + list(range(nxt, nxt + add))
        nxt += add
    return parent, rounds


def _random_case(rng, n_nodes, n_images, n_edges, kind):
    node_image = rng.integers(0, n_images, n_nodes)
    if kind == "random":
        n1 = rng.integers(0, n_nodes, n_edges)
        n2 = rng.integers(0, n_nodes, n_edges)
    elif kind == "star":          # every edge touches node 0: one reservation winner per round
        n1 = np.zeros(n_edges, np.int64)
        n2 = rng.integers(0, n_nodes, n_edges)
    elif kind == "chain":         # a path, then its edges again reversed and duplicated
        a = np.arange(n_nodes - 1)
        n1 = np.concatenate([a, a[::-1], a])
        n2 = np.concatenate([a + 1, a[::-1] + 1, a + 1])
    else:                         # "clash": few images, so most unions are refused
        node_image = rng.integers(0, 3, n_nodes)
        n1 = rng.integers(0, n_nodes, n_edges)
        n2 = rng.integers(0, n_nodes, n_edges)
    return node_image, n1.astype(np.int64), n2.astype(np.int64)


@pytest.mark.parametrize("kind", ["random", "star", "chain", "clash"])
@pytest.mark.parametrize("window", [1, 2, 7, 64, 100000])
def test_reservation_rounds_equal_sequential_kruskal(kind, window):
    rng = np.random.default_rng(zlib.crc32(("%s/%d" % (kind, window)).encode()))
    for trial in range(3):
        node_image, n1, n2 = _random_case(rng, 300, 40 + 30 * trial, 900, kind)
        want = _sequential(node_image, n1, n2)
        got, rounds = _reservations(node_image, n1, n2, window)
        assert np.array_equal(want, got)
        assert rounds >= -(-len(n1) // window)


def test_reservation_rounds_on_a_scene_order():
    """cfg1's matches in the stage's own (sim, n1, n2) order, with heavy similarity ties."""
    from lfr_b200 import build_graph
    ms = synth.generate("cfg1")
    ms.sim[:] = np.round(ms.sim * 10) / 10
    g = build_graph(ms)
    order = np.lexsort((np.arange(g.und_n1.shape[0]), g.und_n2, g.und_n1, g.und_sim.astype(np.float32)))[::-1]
    n1, n2 = g.und_n1[order], g.und_n2[order]
    want = _sequential(g.node_image, n1, n2)
    for window in (1, 5, 333, 1 << 18):
        got, _ = _reservations(g.node_image, n1, n2, window)
        assert np.array_equal(want, got)


# ---------------------------------------------------------------------------------------------------
# GPU: the device stage against the host stage
# ---------------------------------------------------------------------------------------------------
def host_stage(arrs, n_images):
    """lfr_host_stage_create + export, edge records in place: (rc, arrays, sizes)."""
    return host_stage_export(arrs, n_images)


def device_stage(b200, arrs, n_images):
    """lfr_plan_create_from_matches + lfr_plan_export_graph: (rc, arrays, sizes, plan)."""
    try:
        plan = Plan.from_matches(b200, arrs, n_images=n_images)
    except RuntimeError as e:
        return int(str(e).split("(")[1].split(")")[0]), None, None, None
    return 0, plan.export_graph(), plan.sizes, plan


def assert_same_stage(b200, arrs, n_images):
    rc_h, a, sa = host_stage(arrs, n_images)
    rc_d, b, sb, plan = device_stage(b200, arrs, n_images)
    assert rc_h == rc_d
    if rc_h:
        return rc_h, None
    for k in ARRAYS:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert a[k].tobytes() == b[k].tobytes(), k
    for k in COUNTS:
        assert sa[k] == sb[k], (k, sa[k], sb[k])
    return 0, (a, sa, plan)


def _arrs(ms, banned=()):
    """Private copies: the tests edit them, and host_input_arrays() may return views of `ms`."""
    return {k: v.copy() for k, v in host_input_arrays(ms, banned)[1].items()}


def _ring1400():
    cfg = synth.SynthConfig("ring1400", 1400, 2000, "ring", 0.7, match_prob=0.3, window=20, n_random=5,
                            vis_halfwidth=12, seed=1400, outlier_match_ratio=0.125)
    return synth.generate(cfg, scale=0.03)


SCENES = [("cfg1", 1.0, None), ("cfg2", 1.0, None), ("cfg3", 1.0, None), ("cfg4", 1.0, None), ("ring60", 1.0, None),
          ("cfg5", 0.1, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,scale,seed", SCENES)
def test_device_stage_equals_host_stage(b200, cfg, scale, seed):
    ms = synth.generate(cfg, scale=scale, seed=seed)
    rc, (a, sizes, _) = assert_same_stage(b200, _arrs(ms), len(ms.image_names))
    assert rc == 0 and sizes["n_nodes"] > 0 and sizes["n_components"] > 1


@pytest.mark.gpu
def test_device_stage_bitset_image_sets(b200):
    """More than 64 images: image sets as lists, then pool bitsets; tracks of more than 12 images."""
    ms = _ring1400()
    rc, (a, sizes, _) = assert_same_stage(b200, _arrs(ms), len(ms.image_names))
    assert sizes["max_track_size"] > 12 and len(ms.image_names) > 64
    assert sizes["n_oversized_meta_components"] > 0 and sizes["n_cut_groups"] > 0


@pytest.mark.gpu
def test_device_stage_banned_images_and_parts(b200, tmp_path):
    from lfr_b200 import wire
    ms = synth.generate("cfg2")
    for banned in ([ms.image_names[1]], [ms.image_names[i] for i in (0, 3, 7)]):
        arrs = _arrs(ms, banned)
        assert arrs["pair_skip"].any()
        assert_same_stage(b200, arrs, len(ms.image_names))
    path = str(tmp_path / "m.pb")
    files = wire.write_matching_file(ms, path, pairs_per_part=max(1, ms.n_pairs // 3))
    assert len(files) > 1 and files[0].endswith(".part.0")
    parts = wire.read_matching_file(path)
    assert_same_stage(b200, _arrs(parts), len(parts.image_names))


@pytest.mark.gpu
def test_device_stage_similarity_ties(b200):
    """Many equal similarities: the (sim, n1, n2) order of the Kruskal decides; all equal as the extreme."""
    ms = synth.generate("cfg2", scale=0.5, seed=3)
    ms.sim[:] = np.round(ms.sim * 20) / 20
    assert_same_stage(b200, _arrs(ms), len(ms.image_names))
    ms.sim[:] = 0.5
    assert_same_stage(b200, _arrs(ms), len(ms.image_names))


@pytest.mark.gpu
@pytest.mark.parametrize("window", ["1", "7", "1000"])
def test_device_stage_kruskal_window(b200, window, monkeypatch):
    """The reservation window changes the rounds, never the result."""
    monkeypatch.setenv("LFR_KRUSKAL_WINDOW", window)
    ms = synth.generate("cfg1")
    ms.sim[:] = np.round(ms.sim * 10) / 10
    assert_same_stage(b200, _arrs(ms), len(ms.image_names))


@pytest.mark.gpu
def test_device_stage_same_image_twice(b200):
    """A pair listing one image on both sides, with distinct and with equal feature indices (a self edge)."""
    ms = synth.generate("cfg1")
    arrs = _arrs(ms)
    arrs["pair_img2"][0] = arrs["pair_img1"][0]
    lo = int(arrs["pair_ptr"][0])
    arrs["feat2"][lo] = arrs["feat1"][lo]
    assert_same_stage(b200, arrs, len(ms.image_names))


@pytest.mark.gpu
def test_device_stage_empty_and_all_banned(b200):
    ms = synth.generate("cfg1")
    z = dict(pair_img1=np.zeros(0, np.uint32), pair_img2=np.zeros(0, np.uint32), pair_skip=np.zeros(0, np.uint8),
             pair_ptr=np.zeros(1, np.uint64), feat1=np.zeros(0, np.uint32), feat2=np.zeros(0, np.uint32),
             sim=np.zeros(0, np.float32), disp1=np.zeros((0, 18), np.float32), disp2=np.zeros((0, 18), np.float32))
    for arrs in (z, _arrs(ms, ms.image_names)):
        rc, (a, sizes, plan) = assert_same_stage(b200, arrs, len(ms.image_names))
        assert sizes["n_nodes"] == 0 and a["row_ptr"].tolist() == [0] and a["comp_ptr"].tolist() == [0]
        plan.solve()
        pos, st = plan.download()
        assert pos.shape == (0, 2)


@pytest.mark.gpu
def test_device_stage_errors(b200):
    ms = synth.generate("cfg1")
    arrs = _arrs(ms)
    arrs["sim"][5] = np.nan
    assert assert_same_stage(b200, arrs, len(ms.image_names))[0] == LFR_EINVAL
    arrs = _arrs(ms)
    arrs["pair_img1"][2] = len(ms.image_names)
    assert assert_same_stage(b200, arrs, len(ms.image_names))[0] == LFR_EINVAL
    arrs = _arrs(ms)
    arrs["pair_img1"][:] = 69990
    arrs["pair_img2"][:] = 69999
    assert assert_same_stage(b200, arrs, 70000)[0] == LFR_EUNSUPPORTED
    # a refusal leaves the library usable
    assert_same_stage(b200, _arrs(ms), len(ms.image_names))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["cfg2", "cfg4"])
def test_plan_from_matches_solves_like_lfr_solve(b200, cfg):
    """Positions and per-slot stats of the device-built plan equal lfr_solve() on the host-stage problem."""
    from lfr_b200 import build_problem
    ms = synth.generate(cfg)
    p = build_problem(ms, native=True)
    want_pos, want = b200.solve(p)
    plan = Plan.from_matches(b200, ms)
    plan.solve()
    got_pos, got = plan.download()
    assert got_pos.tobytes() == want_pos.tobytes()
    for k in ("iterations", "termination", "initial_cost", "final_cost"):
        assert got[k].tobytes() == want[k].tobytes(), k
    for k in ("total_iterations", "total_line_search_steps", "n_solved"):
        assert got[k] == want[k], k
    plan.close()


def test_cpu_oracle_refuses_the_graph_stage(oracle):
    """The CPU oracle has no device and no plans: a plan from matches is refused with LFR_EUNSUPPORTED."""
    ms = synth.generate("cfg1")
    rc, _, _, _ = device_stage(oracle, _arrs(ms), len(ms.image_names))
    assert rc == LFR_EUNSUPPORTED


def test_host_stage_helper_writes_records_in_place():
    """host_stage_export() runs the host stage as the drop-in does (edges_out) and equals build_problem()."""
    from lfr_b200 import build_problem
    ms = synth.generate("cfg1")
    rc, a, sizes = host_stage_export(_arrs(ms), len(ms.image_names))
    p = build_problem(ms, native=True)
    assert rc == 0 and sizes["n_nodes"] == p.graph.n_nodes
    assert a["edges"].tobytes() == p.graph.edges.tobytes() and np.array_equal(a["comp_nodes"], p.comp_nodes)


def test_graph_symbols_exported():
    """The product library exports include/lfr_graph.h (checked on the built .so, no device needed)."""
    from lfr_b200.capi import B200_LIB_PATH
    if not os.path.exists(B200_LIB_PATH):
        pytest.skip("product library not built")
    lib = C.CDLL(B200_LIB_PATH)
    for s in GRAPH_SYMBOLS:
        assert hasattr(lib, s), s
