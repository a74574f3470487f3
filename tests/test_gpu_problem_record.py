"""The problem record on the GPU: lfr_plan_problem_record (csrc/lfr_record.cuh) byte for byte against the host
form (lfr_host_problem_record) on synthetic scenes up to cfg4, ring60, ring1400 (CTA-tier components past 1024
nodes) and the adversarial goldens, with plans from matches and from wire bytes; a solve after the call is the
plan's solve without it; lfr_plan_update_solution_since_record against lfr_plan_update_solution_since on every
case of tests/test_update_since.py; the drop-in's device route against its host route through both hosts; and
the new kernels' resource use."""
import re
import subprocess

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import Plan
from lfr_b200.graph import problem_from_stage
from test_fixed_images import stage
from test_fixed_images_ref import bits
from test_gpu_fixed_images import _run
from test_gpu_update_since import gpu_case
from test_graph_stage_adversarial import E2E_CASES, make_case
from test_sass_footprint import LIB, cuobjdump
from test_update_since import CASES, banned_args

pytestmark = pytest.mark.gpu


def _ring1400():
    cfg = synth.SynthConfig("ring1400", 1400, 2000, "ring", 0.7, match_prob=0.3, window=20, n_random=5,
                            vis_halfwidth=12, seed=1400, outlier_match_ratio=0.125)
    return synth.generate(cfg, scale=0.03)


SCENES = {"cfg1": lambda: synth.generate("cfg1"), "cfg2": lambda: synth.generate("cfg2"),
          "cfg3": lambda: synth.generate("cfg3"), "cfg4": lambda: synth.generate("cfg4"),
          "ring60": lambda: synth.generate("ring60"), "ring1400": _ring1400}
for _c in E2E_CASES:
    SCENES["adv-" + _c] = (lambda c=_c: make_case(c))


def host_record(ms, banned=()):
    skip, h, sz = stage(ms, banned)
    return wire.problem_record(problem_from_stage(ms, skip, h, sz, "native"), ms.image_names), h


@pytest.mark.parametrize("name", list(SCENES))
def test_device_record_equals_the_host_form(b200, name):
    ms = wire.decode_matching_file(wire.encode_matching_file(SCENES[name]()))
    want, h = host_record(ms)
    if name == "ring1400":
        assert np.bincount(h["comp"].astype(np.int64)).max() > 1024
    for make in (lambda: Plan.from_matches(b200, ms), lambda: Plan.from_wire(b200, [wire.encode_matching_file(ms)])):
        plan = make()
        try:
            assert plan.problem_record(ms.image_names) == want
        finally:
            plan.close()


@pytest.mark.parametrize("name", ["cfg2", "ring1400"])
def test_solve_after_the_record_is_the_solve_without_it(b200, name):
    ms = SCENES[name]()
    outs = []
    for with_record in (False, True):
        plan = Plan.from_matches(b200, ms)
        try:
            if with_record:
                plan.problem_record(ms.image_names)
            plan.solve()
            pos, st = plan.download()
            again = plan.problem_record(ms.image_names)
        finally:
            plan.close()
        outs.append((bits(pos).tobytes(), {k: np.asarray(v).tobytes() for k, v in st.items()
                                            if k in ("iterations", "termination", "initial_cost", "final_cost")}, again))
    assert outs[0] == outs[1]


@pytest.mark.parametrize("name", list(CASES))
def test_update_since_record_equals_update_since(b200, tmp_path, name):
    old, new, banned, o, n, a, A = gpu_case(tmp_path, name)
    prev = Plan.from_matches(b200, wire.decode_matching_file(o.read_bytes()))
    try:
        record = prev.problem_record(prev.image_names)
        res = []
        for kw in (dict(previous=prev), dict(previous_record=record)):
            plan = Plan.from_matches(b200, new, banned_images=banned)
            try:
                counts = plan.update_solution(A, new.image_names, **kw)
                start, _ = plan.download()
                plan.solve()
                pos, st = plan.download()
            finally:
                plan.close()
            res.append((counts, bits(start).tobytes(), bits(pos).tobytes(), np.asarray(st["termination"]).tobytes()))
    finally:
        prev.close()
    assert res[0] == res[1]
    skip, h, sz = stage(new, banned)
    want = wire.update_solution_since_record(A, problem_from_stage(new, skip, h, sz, "native"), record)
    assert res[1][0] == want[2:]


@pytest.mark.parametrize("name", ["same", "new-k3", "banned", "sim"])
def test_drop_in_device_route_equals_host_route(tmp_path, name):
    old, new, banned, o, n, a, A = gpu_case(tmp_path, name)
    outs, recs = [], []
    for python in (False, True):
        for route in ("host", "device"):
            tag = "%d_%s" % (python, route)
            a_out, a_rec = tmp_path / ("a_%s.pb" % tag), tmp_path / ("a_%s.rec" % tag)
            r = _run(["--matches_file", str(o), "--output_file", str(a_out), "--record_file", str(a_rec)],
                     python=python, route=route)
            assert r.returncode == 0, (python, route, r.stderr)
            out, rec = tmp_path / ("o_%s.pb" % tag), tmp_path / ("o_%s.rec" % tag)
            r = _run(["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a),
                      "--update_initial_solution", "--earlier_record_file", str(a_rec), "--record_file", str(rec)]
                     + banned_args(banned), python=python, route=route)
            assert r.returncode == 0, (python, route, r.stderr)
            outs.append(out.read_bytes())
            recs.append((a_rec.read_bytes(), rec.read_bytes()))
    assert all(x == outs[0] for x in outs[1:]) and all(x == recs[0] for x in recs[1:])
    since = tmp_path / "since.pb"
    r = _run(["--matches_file", str(n), "--output_file", str(since), "--initial_solution", str(a),
              "--update_initial_solution", "--previous_matches_file", str(o)] + banned_args(banned), route="device")
    assert r.returncode == 0, r.stderr
    assert since.read_bytes() == outs[0]
    assert recs[0][1] == host_record(new, banned)[0]


def test_python_host_refuses_an_unwritable_record_file(tmp_path, capfd):
    from lfr_b200.cli import main as cli_main
    m, out = tmp_path / "m.pb", tmp_path / "out.pb"
    m.write_bytes(wire.encode_matching_file(synth.generate("cfg1")))
    bad = str(tmp_path / "no-such-dir" / "r.rec")
    assert cli_main(["--matches_file", str(m), "--output_file", str(out), "--record_file", bad]) == 255
    assert out.exists()
    assert capfd.readouterr().err == "ERROR: cannot write the record file '%s'\n" % bad


def test_record_kernels_compile_for_sm90a_without_spills():
    out = subprocess.run([cuobjdump(), "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S*record\S*(digest|lookup)_kernel\S*)", line)
        if m:
            found[m.group(2)] = lines[i + 1]
    assert set(found) == {"digest", "lookup"}, out[:2000]
    for usage in found.values():
        assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), usage
    assert "sm_90a" in subprocess.run([cuobjdump(), "-lelf", LIB], capture_output=True, text=True, check=True).stdout
