"""Carrying an earlier SolutionFile into the output on the GPU: lfr_plan_encode_solution_carried against
lfr_wire_encode_solution_carried on the plan's host assembly (bytes, "> 0.5" count, carried count), on the
golden scenes, synthetic and adversarial scenes, a CTA-tier scene and adversarial files; the plan left as it
was; the size protocol; and the drop-in's incremental scenario (the new pairs alone, on the device route by
the size rule) through both hosts and both routes."""
import ctypes as C
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import Plan
from lfr_b200.graph import host_input_arrays
from lfr_b200.solver import assemble_solution
from test_carry_solution import (NEW, SPECIAL, carried, every_entry_comes_back, image_bits, messages, split_pairs,
                                 untimed_lines)
from test_fixed_images import random_solution
from test_gpu_fixed_images import PRODUCT, SCENES, scene
from test_gpu_solution_encode import image_facts
from test_ref_solve import GOLD, GOLDEN_NAMES, LAUNCHER

pytestmark = pytest.mark.gpu


def adversarial_file(ms, g, seed):
    """random_solution's repeats and unknown names, plus every image of `ms` (those without nodes included)
    listed again with special float bits, feature 0, empty messages and non-UTF-8 names."""
    rng = np.random.default_rng(seed)
    data = random_solution(ms, g, rng)
    msgs = []
    for k, nm in enumerate(ms.image_names):
        feats = np.unique(g["node_feat"][g["node_image"] == k])
        pick = feats[rng.random(feats.shape[0]) < 0.3].tolist() + [0, int(feats.max()) + 3 if feats.size else 7]
        rng.shuffle(pick)
        msgs.append(image_bits(nm, [(f, int(rng.choice(SPECIAL)), int(rng.choice(SPECIAL))) for f in pick],
                               int(rng.choice(SPECIAL))))
    msgs.insert(int(rng.integers(0, len(msgs) + 1)), image_bits(b"\xff\xfe-not-utf8.png", [(0, 0x7FC12345, 1)]))
    msgs.insert(int(rng.integers(0, len(msgs) + 1)), image_bits(b"empty.png", []))
    msgs.append(image_bits(b"", [(5, 0x80000000, 0)]))
    return data + b"".join(msgs)


def host_carried(plan, names, fact, data):
    """lfr_wire_encode_solution_carried on the plan's host assembly: (bytes, n_outside, n_carried)."""
    pos, _ = plan.download()
    g = plan.export_graph()
    graph = SimpleNamespace(n_nodes=plan.n_nodes, node_image=g["node_image"].astype(np.int64), node_feat=g["node_feat"],
                            image_names=names, image_fact=fact)
    s = assemble_solution(SimpleNamespace(graph=graph), pos)
    out, n = wire.encode_solution_carried(s.image_names, s.fact, s.img_ptr, s.feature_idx, s.di, s.dj, data)
    return out, s.n_outside, n


def assert_same(plan, names, fact, data):
    got = plan.encode_solution_carried(names, fact, data)
    want = host_carried(plan, names, fact, data)
    assert got[1:] == want[1:]
    assert got[0] == want[0]
    return got


def golden(name):
    data = open(os.path.join(GOLD, "%s_matches.pb" % name), "rb").read()
    return wire.decode_matching_file(data), ()


@pytest.mark.parametrize("name", ["golden:" + n for n in GOLDEN_NAMES] + SCENES)
def test_device_bytes_equal_the_host_function(b200, name):
    ms, banned = golden(name[7:]) if name.startswith("golden:") else scene(name)
    plan = Plan.from_matches(b200, ms, banned_images=banned)
    g = plan.export_graph()
    names, fact = ms.image_names, image_facts(ms, banned)
    files = [random_solution(ms, g, np.random.default_rng(1)), adversarial_file(ms, g, 2), b""]
    for data in files:                               # the start point, unsolved
        assert_same(plan, names, fact, data)
    if plan.n_nodes:
        plan.solve()
    for data in files:
        _, _, n = assert_same(plan, names, fact, data)
        if data:
            assert n > 0
    # an empty file is the plain encoder's output; an absent name list entry for a banned image goes after
    assert plan.encode_solution_carried(names, fact, b"")[:2] == plan.encode_solution(names, fact)
    for nm in banned:
        got, _, _ = plan.encode_solution_carried(names, fact, files[1])
        out = [m[0] for m in messages(got)]
        assert out.count(nm.encode()) == 1
    plan.close()


def test_cta_tier_scene(b200):
    ms = synth.generate("ring60", scale=0.3)
    plan = Plan.from_matches(b200, ms)
    g = plan.export_graph()
    plan.solve()
    fact = image_facts(ms)
    for seed in (3, 4):
        assert_same(plan, ms.image_names, fact, adversarial_file(ms, g, seed))
    plan.close()


def test_plan_is_unchanged_and_size_protocol(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    plan = Plan.from_matches(b200, ms)
    g = plan.export_graph()
    plan.solve()
    names, fact = ms.image_names, image_facts(ms)
    before = plan.encode_solution(names, fact), plan.download()[0].tobytes()
    data = adversarial_file(ms, g, 9)
    want, n_out, n_car = plan.encode_solution_carried(names, fact, data)
    assert (plan.encode_solution(names, fact), plan.download()[0].tobytes()) == before
    # cap = need - 1 writes nothing; cap = need writes the bytes
    blob, off = wire._names_blob(list(names))
    buf = np.frombuffer(data, np.uint8)
    f = b200.lib.lfr_plan_encode_solution_carried
    args = (plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact.ctypes.data, buf.ctypes.data, buf.size)
    need = f(*args, None, 0, None, None)
    assert need == len(want)
    out = np.full(need + 4, 0xAB, np.uint8)
    a, b = C.c_uint64(), C.c_uint64()
    assert f(*args, out.ctypes.data, need - 1, C.byref(a), C.byref(b)) == need and (out == 0xAB).all()
    assert (a.value, b.value) == (n_out, n_car)
    assert f(*args, out.ctypes.data, need, None, None) == need and out[:need].tobytes() == want and (out[need:] == 0xAB).all()
    # refusals: malformed bytes and repeated names
    with pytest.raises(RuntimeError):
        plan.encode_solution_carried(names, fact, b"\x0a\xff\xff\xff\xff\x0f not a protobuf")
    with pytest.raises(RuntimeError):
        plan.encode_solution_carried(list(names[:-1]) + [names[0]], fact, data)
    assert (plan.encode_solution(names, fact), plan.download()[0].tobytes()) == before
    plan.close()


def test_incremental_carry_through_both_hosts_and_routes(b200, tmp_path):
    """cfg2 solved from the pairs without images 8-10 (A), then the pairs that touch them alone, with keep and
    carry: the size rule sends them to the device; both hosts and both routes write the same bytes, every
    entry of A comes back bit for bit, and the scene's part is the run without --carry_initial_solution."""
    ms = synth.generate("cfg2")
    old, new = split_pairs(ms, ms.image_names[NEW])
    m_old, m_new, a = tmp_path / "old.pb", tmp_path / "new.pb", tmp_path / "a.pb"
    m_old.write_bytes(wire.encode_matching_file(old))
    m_new.write_bytes(wire.encode_matching_file(new))
    _, arrs = host_input_arrays(new)
    assert b200.graph_stage_on_device(arrs, len(new.image_names), 1)
    r = subprocess.run([PRODUCT, "--matches_file", str(m_old), "--output_file", str(a)], capture_output=True)
    assert r.returncode == 0, r.stderr
    A = a.read_bytes()
    base = ["--matches_file", str(m_new), "--initial_solution", str(a), "--keep_initial_solution"]
    outs, lines = [], []
    for python in (False, True):
        for route in (None, "host", "device"):
            o = tmp_path / ("o_%d_%s.pb" % (python, route))
            env = dict(os.environ)
            env.pop("LFR_GRAPH_STAGE", None)
            if route:
                env["LFR_GRAPH_STAGE"] = route
            cmd = [PRODUCT]
            if python:
                env["LFR_SOLVE_PYTHON"] = "1"
                cmd = [sys.executable, LAUNCHER]
            r = subprocess.run(cmd + base + ["--output_file", str(o), "--carry_initial_solution"], capture_output=True, env=env)
            assert r.returncode == 0, r.stderr
            outs.append(o.read_bytes())
            lines.append(untimed_lines(r))
    assert all(x == outs[0] for x in outs[1:])
    assert all(x == lines[0] for x in lines[1:])
    o0 = tmp_path / "o0.pb"
    r0 = subprocess.run([PRODUCT] + base + ["--output_file", str(o0)], capture_output=True)
    assert r0.returncode == 0, r0.stderr
    assert untimed_lines(r0) == lines[0]
    scene_part = messages(o0.read_bytes())
    assert outs[0] == carried(scene_part, A)[0]
    assert every_entry_comes_back(A, outs[0]) > 0
    assert {m[0] for m in messages(outs[0])} == {m[0] for m in messages(A)} | {m[0] for m in scene_part}
