"""--query_images on batches whose sub-scenes outgrow the 64-bit image mask (CPU).

The cases (tests/subscene_cases.py) put sub-scenes of 64, 65, 81, 90 - 129 images next to sub-scenes of 2 - 3,
so the union-find image sets take the 12-entry lists and bitsets of 2 and 3 words, indexed by an image's id
inside its sub-scene; they cut meta-components at sub-scene caps of 2, 3, 65 and 129, and reach the 65 535-id
limit.  The grouped host stage equals the numpy stage and, sub-scene by sub-scene, the stage on each
sub-scene's pairs alone; the native drop-in (CPU checker) writes every query's own run byte for byte, and on
three cases the own runs are the reference's own main()'s."""
import os
import random
import subprocess

import numpy as np
import pytest

import subscene_cases as S
from lfr_b200 import wire
from lfr_b200.graph import host_input_arrays, host_stage_export
from lfr_b200.solver import refine
from test_fixed_images import checker_exe, run  # noqa: F401
from test_query_images import (REF_SOLVE, _both_hosts, assert_stages_agree_by_sub_scene, check_batch, messages,
                               own_runs, stdout_values)

#: own runs also compared with the reference's own main()
REF_CASES = ("bitset65", "bitset129", "caps")


def query_args(d, name, out, queries, banned, extra=()):
    args = ["--matches_file", str(d / name), "--output_file", str(out), "--banned_images", banned] + list(extra)
    for q in queries:
        args += ["--query_images", q]
    return args


def test_cases_have_the_structure_they_are_named_for():
    for name in S.STAGED:
        S.check_structure(name)


@pytest.mark.parametrize("threads", ["1", "8"])
@pytest.mark.parametrize("case", [c for c in S.STAGED if not c.startswith("ids_")])
def test_stages_agree_sub_scene_by_sub_scene(case, threads, monkeypatch):
    """Native host stage with groups = numpy stage, and each sub-scene = the stage on its pairs alone."""
    monkeypatch.setenv("LFR_HOST_THREADS", threads)
    batch, queries, banned = S.make(case)
    assert_stages_agree_by_sub_scene(batch, queries, banned, S.grouped(case) if case in S.SWAPS else None)


@pytest.mark.parametrize("case", S.SOLVED)
def test_native_batch_equals_every_querys_own_run(tmp_path, checker_exe, case):  # noqa: F811
    batch, queries, banned = S.make(case)
    wire.write_matching_file(batch, str(tmp_path / "batch.pb"))
    o = tmp_path / "batch_out.pb"
    r = run(checker_exe, query_args(tmp_path, "batch.pb", o, queries, banned))
    assert r.returncode == 0, r.stderr
    own = own_runs(checker_exe, tmp_path, batch, queries, [], banned)
    got = check_batch(o.read_bytes(), r.stdout.decode(), own, queries)
    assert sorted(nm for nm, _ in got) == sorted(q for q in queries if own[q][0] is not None) and got
    if case in REF_CASES and os.path.exists(REF_SOLVE):   # built where the reference's sources are
        for q in queries:
            o2 = tmp_path / ("ref_%s.pb" % q)
            r2 = subprocess.run([REF_SOLVE, "--matches_file", str(tmp_path / ("own_%s.pb" % q)), "--output_file", str(o2),
                                 "--banned_images", banned], capture_output=True)
            assert r2.returncode == 0, r2.stderr
            mine = [m for nm, m in messages(o2.read_bytes()) if nm == q]
            assert (mine[0] if mine else None) == own[q][0], q


# ---------------------------------------------------------------------------------------------------
# the 65 535-id limit
# ---------------------------------------------------------------------------------------------------
def test_65535_ids_are_taken_by_the_stage_and_both_hosts(tmp_path, checker_exe, oracle, monkeypatch):  # noqa: F811
    """The native drop-in (CPU checker) and the Python host's refine() on the host route write the same bytes."""
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    batch, queries, banned = S.make("ids_65535")
    S.check_structure("ids_65535")
    wire.write_matching_file(batch, str(tmp_path / "batch.pb"))
    r = run(checker_exe, query_args(tmp_path, "batch.pb", tmp_path / "native.pb", queries, banned))
    assert r.returncode == 0, r.stderr
    a = (tmp_path / "native.pb").read_bytes()
    opts = oracle.default_options(n_threads=4)
    _, _, _, sol = refine(wire.read_matching_file(str(tmp_path / "batch.pb")), [banned], opts,
                          solve_fn=lambda p, x=None: oracle.solve(p, opts, positions=x), query_images=queries)
    assert wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj) == a
    assert sol.n_outside == stdout_values(r.stdout.decode())["# points with at least one coordinate > 0.5"]
    got = dict(messages(a))
    assert len(got) == len(queries)
    sample = random.Random(65535).sample(queries, 18) + [queries[0], queries[-1]]
    own = own_runs(checker_exe, tmp_path, batch, sample, [], banned)
    for q in sample:
        assert got[q] == own[q][0], q


def test_65536_ids_are_refused_by_the_stage_both_hosts_and_refine(tmp_path, checker_exe, oracle):  # noqa: F811
    batch, queries, banned = S.make("ids_65536")
    sub, group = batch.query_subscenes(queries, [banned])
    assert len(sub.image_names) == 65536
    _, arrs = host_input_arrays(sub, (), group)
    assert host_stage_export(arrs, len(sub.image_names))[0] == S.LFR_EUNSUPPORTED
    wire.write_matching_file(batch, str(tmp_path / "batch.pb"))
    o = tmp_path / "o.pb"
    ra, rb = _both_hosts(checker_exe, query_args(tmp_path, "batch.pb", o, queries, banned))
    assert (ra.returncode, ra.stdout) == (2, b"")
    assert ra.stderr.startswith(b"ERROR: --query_images: the sub-scenes hold 65536 images, more than 65535")
    assert ra.stderr.count(b"\n") == 1
    assert (rb.returncode, rb.stdout, rb.stderr) == (ra.returncode, ra.stdout, ra.stderr)
    assert not o.exists()
    opts = oracle.default_options(n_threads=1)
    with pytest.raises(ValueError, match="more than 65535"):
        refine(batch, [banned], opts, solve_fn=lambda p, x=None: oracle.solve(p, opts, positions=x), query_images=queries)
