"""--versioned_scenes on the GPU: both drop-in hosts on every graph-stage route against every scene's own run on the
CPU checker, and the C ABI: lfr_plan_update_solution_groups() and lfr_plan_problem_record_groups() against each
scene's own plan, against their host forms and, with one group, against the single-scene calls; and their device
operation counts, which must not grow with the number of scenes."""
import ctypes as C

import numpy as np
import pytest

import test_versioned_scenes as tvs
from lfr_b200 import synth, wire
from lfr_b200.capi import Plan
from lfr_b200.graph import host_input_arrays
from lfr_b200.matchset import MatchSet
from lfr_b200.solver import refine
from test_fixed_images import checker_exe  # noqa: F401
from test_gpu_query_images import ROUTES, _run
from test_versioned_scenes import rounds  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", [0, 1])
@pytest.mark.parametrize("python", [False, True], ids=["native", "python"])
@pytest.mark.parametrize("route", sorted(ROUTES))
def test_drop_in_on_every_route_writes_every_scenes_own_run(rounds, route, python, k):  # noqa: F811
    d, rows, own = rounds[k]
    args, tagged = tvs.batch_args(d, rows, "gpu_%s_%d_%d" % (route, python, k))
    r = _run(args, ROUTES[route], python=python)
    assert r.returncode == 0, r.stderr
    tvs.check(tagged, r.stdout.decode(), own)


def test_combinations_agree_on_both_hosts(tmp_path):
    """Every opt-in option with --versioned_scenes: the same exit code, stdout (timers aside) and stderr."""
    import os
    tiny = os.path.join(tvs.GOLD, "tiny_matches.pb")
    sub = {"S": os.path.join(tvs.GOLD, "tiny_solution.pb"), "M": tiny, "R": str(tmp_path / "r.rec"),
           "L": str(tmp_path / "l.txt")}
    tvs.write_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb", "", "", tmp_path / "1.rec")])
    strip = lambda s: [l for l in s.splitlines() if b" time:" not in l]  # noqa: E731
    for opt in sorted(tvs.OPT_IN):
        for with_start in (False, True):
            args = ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), "--versioned_scenes",
                    str(tmp_path / "l.txt"), opt] + [sub.get(a, a) for a in tvs.OPT_IN[opt]]
            if with_start and opt not in ("--initial_solution", "--update_initial_solution"):
                args += ["--initial_solution", sub["S"], "--update_initial_solution"]
            a, b = _run(args, {}), _run(args, {}, python=True)
            assert (a.returncode, strip(a.stdout), a.stderr) == (b.returncode, strip(b.stdout), b.stderr), args


@pytest.mark.parametrize("versioned", [False, True], ids=["plain", "versioned"])
def test_an_empty_record_path_fails_alike_on_both_hosts(tmp_path, versioned):
    import os
    tiny = os.path.join(tvs.GOLD, "tiny_matches.pb")
    args = ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), "--record_file", ""]
    if versioned:
        tvs.write_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb", "", "", tmp_path / "1.rec")])
        args += ["--versioned_scenes", str(tmp_path / "l.txt")]
    strip = lambda s: [l for l in s.splitlines() if b" time:" not in l]  # noqa: E731
    a, b = _run(args, {}), _run(args, {}, python=True)
    assert (a.returncode, a.stderr) == (255, b"ERROR: cannot write the record file ''\n")
    assert (a.returncode, strip(a.stdout), a.stderr) == (b.returncode, strip(b.stdout), b.stderr)


def _scene_batch(sets):
    """(joined MatchSet, image_group) of `sets` as --versioned_scenes stages them (no banned image)."""
    return MatchSet.join_scenes(sets, ())


def _own_plan(b200, ms):
    _, arrs = host_input_arrays(ms)
    return Plan.from_matches(b200, arrs, n_images=len(ms.image_names))


def _ops(b200):
    out = (C.c_ulonglong * 3)()
    b200.lib.lfr_debug_device_ops(out, 1)
    return tuple(out)


def _versions(n_scenes, seed, big=False):
    """Round-0 scenes, their SolutionFiles and records from each scene's own plan on the device, and round-1 scenes:
    every third scene gained an image, every fifth had its flows changed."""
    sets0, sets1 = [], []
    for k in range(n_scenes):
        sets0.append(tvs.hpatches_scene(seed + k, 5))
        sets1.append(tvs.hpatches_scene(seed + k, 6) if k % 3 == 0 else
                     tvs.changed_flows(sets0[-1], k) if k % 5 == 0 else sets0[-1])
    if big:
        ms = synth.generate("cfg2", scale=1.0, seed=seed)
        sets0.append(ms)
        sets1.append(tvs.changed_flows(ms, 1))
    return sets0, sets1


def _own_outputs(b200, sets):
    sols, recs = [], []
    for ms in sets:
        _, _, _, sol = refine(ms, (), record_problem=True)
        sols.append(wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj))
        recs.append(sol.record)
    return sols, recs


@pytest.mark.parametrize("with_records", [False, True], ids=["plain", "records"])
def test_grouped_update_is_every_scenes_own_update(b200, monkeypatch, with_records):
    monkeypatch.setenv("LFR_GRAPH_STAGE", "device")
    sets0, sets1 = _versions(12, 300)
    sols0, recs0 = _own_outputs(b200, sets0)
    files = [None if k == 4 else s for k, s in enumerate(sols0)]          # scene 4 starts from zeros
    records = [r if with_records and files[k] is not None and k != 7 else None for k, r in enumerate(recs0)]
    if with_records:
        records[8] = recs0[9]                                             # another scene's record
        # scene 11 listed again, from moved values and scene 0's record: its digests are in the batch's records
        # (the first copy's) but not in the one it is given, so every component of the copy is touched
        sets1.append(sets1[11])
        files.append(tvs.nudged(sols0[11]))
        records.append(recs0[0])
    # every scene's own update
    want_counts = np.zeros(3, np.int64)
    want_out, want_rec = [], []
    for ms, f, r in zip(sets1, files, records):
        plan = _own_plan(b200, ms)
        try:
            if f is not None and r is not None:
                want_counts += plan.update_solution(f, ms.image_names, previous_record=r)
            elif f is not None:
                want_counts[:2] += plan.update_solution(f, ms.image_names)
            else:   # no file: every component of the scene is touched, and solves as from zeros
                want_counts[1] += plan.n_components
            plan.solve()
            plan.download()
            want_out.append(plan.encode_solution(ms.image_names, _facts(ms))[0])
            want_rec.append(plan.problem_record(ms.image_names))
        finally:
            plan.close()
    # one grouped update
    ms, group = _scene_batch(sets1)
    _, arrs = host_input_arrays(ms, (), group)
    plan = Plan.from_matches(b200, arrs, n_images=len(ms.image_names))
    try:
        got = plan.update_solution_groups(files, ms.image_names, group, records)
        assert list(got) == list(want_counts)
        plan.solve()
        plan.download()
        outs, _ = plan.encode_solution_groups(ms.image_names, _facts(ms), group, len(sets1))
        assert outs == want_out
        assert plan.problem_record_groups(ms.image_names, group, len(sets1)) == want_rec
    finally:
        plan.close()
    # the host forms give the same bits: the update's start and held flags, and the records
    from lfr_b200.graph import build_problem
    p = build_problem(ms, (), image_group=group)
    pos_h, held_h, *counts_h = wire.update_solution_groups(files, p, group, records)
    assert counts_h == list(want_counts)
    assert wire.problem_record_groups(p, group, len(sets1)) == want_rec
    plan = Plan.from_matches(b200, arrs, n_images=len(ms.image_names))
    try:
        plan.update_solution_groups(files, ms.image_names, group, records)
        pos_d, _ = plan.download()
        assert np.array_equal(pos_d.view(np.uint64), pos_h.view(np.uint64))
    finally:
        plan.close()


def _facts(ms):
    fact = np.zeros(len(ms.image_names), np.float32)
    for p in range(ms.n_pairs - 1, -1, -1):
        fact[ms.pair_img2[p]] = ms.pair_fact2[p]
        fact[ms.pair_img1[p]] = ms.pair_fact1[p]
    return fact


def test_one_group_is_the_single_scene_call(b200):
    sets0, sets1 = _versions(1, 500)
    sols0, recs0 = _own_outputs(b200, sets0)
    ms = sets1[0]
    group = np.zeros(len(ms.image_names), np.uint32)
    for records, call in (([None], lambda pl: pl.update_solution(sols0[0], ms.image_names)),
                          (recs0, lambda pl: pl.update_solution(sols0[0], ms.image_names, previous_record=recs0[0]))):
        a, b = _own_plan(b200, ms), _own_plan(b200, ms)
        try:
            ra = call(a)
            rb = b.update_solution_groups(sols0, ms.image_names, group, records)
            assert tuple(rb[:len(ra)]) == tuple(ra)
            for pl in (a, b):
                pl.solve()
            pa, _ = a.download()
            pb, _ = b.download()
            assert np.array_equal(pa.view(np.uint64), pb.view(np.uint64))
            assert a.problem_record(ms.image_names) == b.problem_record_groups(ms.image_names, group, 1)[0]
        finally:
            a.close()
            b.close()


def test_a_thousand_scenes_and_a_large_one_cost_one_call_each(b200):
    """About 1000 small scenes plus one cfg2-scale scene: the grouped calls' device operations are those of a
    ten-scene batch, and their bits those of the host forms."""
    from lfr_b200.graph import build_problem
    counts = []
    for n in (10, 1000):
        sets0, sets1 = _versions(n, 1000, big=True)
        ms0, g0 = _scene_batch(sets0)
        _, arrs0 = host_input_arrays(ms0, (), g0)
        plan = Plan.from_matches(b200, arrs0, n_images=len(ms0.image_names))
        try:
            plan.solve()
            plan.download()
            sols, _ = plan.encode_solution_groups(ms0.image_names, _facts(ms0), g0, len(sets0))
            recs = plan.problem_record_groups(ms0.image_names, g0, len(sets0))
        finally:
            plan.close()
        ms, group = _scene_batch(sets1)
        _, arrs = host_input_arrays(ms, (), group)
        plan = Plan.from_matches(b200, arrs, n_images=len(ms.image_names))
        try:
            _ops(b200)
            got = plan.update_solution_groups(sols, ms.image_names, group, recs)
            ops_update = _ops(b200)
            rec = plan.problem_record_groups(ms.image_names, group, len(sets1))
            ops_record = _ops(b200)
            pos_d, _ = plan.download()
        finally:
            plan.close()
        counts.append((ops_update, ops_record))
        p = build_problem(ms, (), image_group=group)
        pos_h, _, *counts_h = wire.update_solution_groups(sols, p, group, recs)
        assert counts_h == list(got) and got[1] > 0 and got[2] > 0
        assert np.array_equal(pos_d.view(np.uint64), pos_h.view(np.uint64))
        assert rec == wire.problem_record_groups(p, group, len(sets1))
    assert counts[0] == counts[1], counts
    assert all(c[0] > 0 for pair in counts for c in pair)
