"""Keeping an earlier SolutionFile on the CPU: the entries join (lfr_wire_join_solution_entries,
include/lfr_wire.h) against a plain statement of its rule, the drop-in's --keep_initial_solution through the
native executable linked against the CPU checker (oracle/liblfr_ref.so) and the Python launcher, and the
kept mask run through the reference's own create_and_solve_problem (oracle/_ref/libref_solve.so)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import USAGE
from lfr_b200.graph import problem_from_stage
from lfr_b200.solver import assemble_solution, constant_problem
from refsrc_util import ref_solve
from test_fixed_images import checker_exe, displacement, image, join_model, random_solution, run, stage  # noqa: F401
from test_fixed_images_ref import (CPU_SCALES, assert_matches_reference, bits, constant_of, host_scene,
                                   planted_solution, sizes_of, with_mask)
from test_ref_solve import GOLD, LAUNCHER

LFR_EINVAL = -1
KEEP_ERROR = b"ERROR: --keep_initial_solution needs --initial_solution FILE\n"


def entries_model(data, image_names, node_image, node_feat):
    """join_model's rule, and which nodes have an entry: a feature of a scene image's last Image message."""
    pos, n = join_model(data, image_names, node_image, node_feat)
    msgs = wire.decode_solution(data)
    last = {m[0]: i for i, m in enumerate(msgs)}
    id_of = {nm: k for k, nm in enumerate(image_names)}
    keys = {(id_of[nm], int(f)) for nm, i in last.items() if nm in id_of for f in msgs[i][2].tolist()}
    has = np.array([(int(a), int(b)) in keys for a, b in zip(np.asarray(node_image).tolist(), np.asarray(node_feat).tolist())],
                   bool).reshape(-1)
    assert int(has.sum()) == n
    return pos, n, has


def check_entries(data, names, node_image, node_feat):
    pos, n, has = wire.join_solution(data, names, node_image, node_feat, entries=True)
    want_pos, want_n, want_has = entries_model(data, names, node_image, node_feat)
    assert n == want_n and pos.tobytes() == want_pos.tobytes() and np.array_equal(has, want_has)
    plain, n_plain = wire.join_solution(data, names, node_image, node_feat)     # the positions of the plain join
    assert n_plain == n and plain.tobytes() == pos.tobytes()
    return has


# ---------------------------------------------------------------------------------------------------
# the entries join
# ---------------------------------------------------------------------------------------------------
def test_entries_join_equals_the_rule_on_a_synthetic_scene():
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    _, out, _ = stage(ms)
    has = check_entries(random_solution(ms, out, np.random.default_rng(4)), ms.image_names, out["node_image"], out["node_feat"])
    assert 0 < has.sum() < has.shape[0]


def test_entries_join_duplicate_rule():
    names = ["a.png", "b.png", "c.png"]
    node_image = np.array([0, 0, 0, 1, 1, 2, 2], np.uint32)
    node_feat = np.array([1, 2, 3, 1, 7, 4, 5], np.uint32)
    data = (image("a.png", [displacement(1, 0.1, 0.2), displacement(2, 0.3, 0.4)])     # overridden as a whole
            + image("b.png", [displacement(7, -0.5, 0.5), displacement(7, 0.0, -0.0), displacement(9, 1, 1)])
            + image("zzz.png", [displacement(4, 0.9, 0.9)])                            # not in the scene
            + image("c.png", [displacement(5, 0.0, 0.0)])                              # an entry of value 0
            + image("a.png", [displacement(3, 0.75, -0.75)]))
    has = check_entries(data, names, node_image, node_feat)
    # a.png features 1 and 2 appear only in the overridden message: no entry; b.png 7 once, c.png 4 absent
    assert has.tolist() == [False, False, True, False, True, False, True]
    pos, _, _ = wire.join_solution(data, names, node_image, node_feat, entries=True)
    assert bits(pos[4]).tolist() == bits(np.array([0.0, -0.0])).tolist()            # the last displacement of 7


def test_entries_join_empty_file_and_unknown_entries():
    names = ["a.png", "b.png"]
    node_image = np.array([0, 1, 1], np.uint32)
    node_feat = np.array([0, 0, 5], np.uint32)
    assert not check_entries(b"", names, node_image, node_feat).any()
    other = image("c.png", [displacement(0, 0.5, 0.5)]) + image("a.png", [displacement(9, 0.5, 0.5)])
    assert not check_entries(other, names, node_image, node_feat).any()
    pos, n, has = wire.join_solution(b"", [], np.zeros(0, np.uint32), np.zeros(0, np.uint32), entries=True)
    assert n == 0 and pos.shape == (0, 2) and has.shape == (0,)


@pytest.mark.parametrize("bad", [b"\x0a\xff", b"\x0a\x05\x0a\x09abc", b"\x0a\xff\xff\xff\xff\x0f not a protobuf",
                                 image("a.png", [displacement(1, 0.5, 0.5)])[:-3]])
def test_entries_join_refuses_malformed_bytes(bad):
    L = wire._lib()
    buf = np.frombuffer(bad, np.uint8)
    pos = np.full(2, 7.0)
    has = np.full(1, 9, np.uint8)
    n = C.c_uint64(5)
    blob, off = wire._names_blob(["a.png"])
    rc = L.lfr_wire_join_solution_entries(buf.ctypes.data, buf.size, 1, blob.ctypes.data, off.ctypes.data, 1,
                                          np.zeros(1, np.uint32).ctypes.data, np.ones(1, np.uint32).ctypes.data,
                                          pos.ctypes.data, C.byref(n), has.ctypes.data)
    assert rc == LFR_EINVAL and (pos == 7.0).all() and (has == 9).all() and n.value == 5
    with pytest.raises(wire.ParseError):
        wire.join_solution(bad, ["a.png"], np.zeros(1, np.uint32), np.ones(1, np.uint32), entries=True)


def test_entries_join_refuses_a_null_flag_array():
    L = wire._lib()
    blob, off = wire._names_blob(["a.png"])
    pos = np.zeros(2)
    rc = L.lfr_wire_join_solution_entries(None, 0, 1, blob.ctypes.data, off.ctypes.data, 1, np.zeros(1, np.uint32).ctypes.data,
                                          np.ones(1, np.uint32).ctypes.data, pos.ctypes.data, None, None)
    assert rc == LFR_EINVAL


# ---------------------------------------------------------------------------------------------------
# the incremental scenario through the native executable on the CPU checker
# ---------------------------------------------------------------------------------------------------
SCENE = dict(cfg="cfg2", scale=0.1, seed=3)
NEW = slice(8, 11)            # images added after solution A


def expected(oracle, ms, a_bytes, fixed_names=()):
    """The checker's lfr_solve on the composed mask (root OR fixed image OR entry in A) and the joined start,
    both stated here from the host stage: (SolutionFile bytes, positions, start, is_const, graph arrays)."""
    skip, g, sz = stage(ms)
    p = problem_from_stage(ms, skip, g, sz, "native")
    start, _, has = entries_model(a_bytes, ms.image_names, g["node_image"], g["node_feat"])
    fixed = np.array([n in set(fixed_names) for n in ms.image_names], bool)
    const = (constant_of(g, fixed) != 0) | has
    pos, _ = oracle.solve(with_mask(p, const), oracle.default_options(n_threads=4), positions=start)
    sol = assemble_solution(p, pos)
    return wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj), pos, start, const, g


@pytest.fixture(scope="module")
def incremental(checker_exe, tmp_path_factory):  # noqa: F811
    """(MatchSet, matches path, solution A's path and bytes): A refines the scene without images 8-10."""
    d = tmp_path_factory.mktemp("incremental")
    ms = synth.generate(SCENE["cfg"], scale=SCENE["scale"], seed=SCENE["seed"])
    m, a = d / "m.pb", d / "a.pb"
    m.write_bytes(wire.encode_matching_file(ms))
    args = ["--matches_file", str(m), "--output_file", str(a)]
    for nm in ms.image_names[NEW]:
        args += ["--banned_images", nm]
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    return ms, m, a, a.read_bytes()


def kept_nodes_come_back(a_bytes, out_bytes):
    got = {nm: dict(zip(fi.tolist(), zip(bits(di).tolist(), bits(dj).tolist())))
           for nm, _, fi, di, dj in wire.decode_solution(out_bytes)}
    n = 0
    for nm, _, fi, di, dj in wire.decode_solution(a_bytes):
        for f, x, y in zip(fi.tolist(), bits(di).tolist(), bits(dj).tolist()):
            assert got[nm][f] == (x, y), (nm, f)
            n += 1
    return n


@pytest.mark.parametrize("fixed", [(), ("new", 1)], ids=["keep", "keep+fixed"])
def test_native_keep_initial_solution_equals_the_checker(checker_exe, oracle, incremental, tmp_path, fixed):  # noqa: F811
    ms, m, a, A = incremental
    fixed_names = [ms.image_names[NEW][0] if k == "new" else ms.image_names[k] for k in fixed]
    o = tmp_path / "o.pb"
    args = ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a), "--keep_initial_solution"]
    for nm in fixed_names:
        args += ["--fixed_images", nm]
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    want, pos, start, const, g = expected(oracle, ms, A, fixed_names)
    assert o.read_bytes() == want
    assert kept_nodes_come_back(A, o.read_bytes()) > 0                  # every node listed in A, bit for bit
    assert np.array_equal(bits(pos[const]), bits(start[const]))
    # old images' keypoints that A never listed exist, are free, and at least one of them moves
    old = np.isin(g["node_image"].astype(np.int64), np.arange(NEW.start)) & ~const
    assert old.any()
    assert (pos[old] != 0).any()
    # the same stdout lines as the run without the flag (the outside count depends on the positions)
    r0 = run(checker_exe, ["--matches_file", str(m), "--output_file", str(tmp_path / "o0.pb"), "--initial_solution", str(a)])
    assert r0.returncode == 0
    lines = [[l.split(":")[0] if l.startswith("# points with") else l for l in x.stdout.decode().splitlines()
              if " time:" not in l] for x in (r, r0)]
    assert lines[0] == lines[1]


def test_python_host_route_equals_the_native_host(checker_exe, incremental, tmp_path):  # noqa: F811
    """The library's Python API on the host route (constant_problem) builds the mask the native host builds."""
    ms, m, a, A = incremental
    skip, g, sz = stage(ms)
    p = problem_from_stage(ms, skip, g, sz, "native")
    q, start = constant_problem(p, [ms.image_names[2]], A, keep_initial_solution=True)
    _, _, has = entries_model(A, ms.image_names, g["node_image"], g["node_feat"])
    fixed = np.array([k == 2 for k in range(len(ms.image_names))])
    assert np.array_equal(q.is_root, ((constant_of(g, fixed) != 0) | has).astype(np.uint8))
    assert np.array_equal(p.is_root, g["is_root"])                      # the returned problem keeps the roots
    assert start.tobytes() == join_model(A, ms.image_names, g["node_image"], g["node_feat"])[0].tobytes()
    q2, _ = constant_problem(p, [ms.image_names[2]], A)
    assert np.array_equal(q2.is_root, constant_of(g, fixed))           # without the flag: as before


# ---------------------------------------------------------------------------------------------------
# the command line
# ---------------------------------------------------------------------------------------------------
def _both_hosts(checker_exe, args, env=None):  # noqa: F811
    a = subprocess.run([checker_exe] + args, capture_output=True, env=env)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=dict(env or os.environ, LFR_SOLVE_PYTHON="1"))
    return a, b


def test_keep_without_initial_solution_is_refused_first(checker_exe, tmp_path):  # noqa: F811
    m = os.path.join(GOLD, "tiny_matches.pb")
    o = tmp_path / "o.pb"
    for argv in (["--matches_file", m, "--output_file", str(o), "--keep_initial_solution"],
                 ["--keep", "--matches_file", m, "--output_file", str(o), "--initial_solution="]):
        a, b = _both_hosts(checker_exe, argv)
        for r in (a, b):
            assert (r.returncode, r.stdout, r.stderr) == (2, b"", KEEP_ERROR)
    assert not o.exists()


def test_keep_takes_no_value(checker_exe, tmp_path):  # noqa: F811
    m = os.path.join(GOLD, "tiny_matches.pb")
    for flag in ("--keep_initial_solution=x", "--keep=", "--k=1"):
        a, b = _both_hosts(checker_exe, ["--matches_file", m, "--output_file", str(tmp_path / "o.pb"), "--initial_solution",
                                         m, flag])
        for r in (a, b):
            assert r.returncode == 1 and r.stdout == b""
            assert r.stderr == (b"ERROR: option '--keep_initial_solution' does not take any arguments\n\n" + USAGE.encode())


def test_prefixes(checker_exe, incremental, tmp_path):  # noqa: F811
    """--k and --keep are --keep_initial_solution; --fix, --init and --h keep their meaning; --help does not
    list the new option."""
    ms, m, a, A = incremental
    outs = []
    for i, flag in enumerate(["--keep_initial_solution", "--keep", "--k"]):
        o = tmp_path / ("o%d.pb" % i)
        r = run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--init", str(a), flag,
                              "--fix", ms.image_names[9]])
        assert r.returncode == 0, r.stderr
        outs.append(o.read_bytes())
    assert outs[0] == outs[1] == outs[2]
    o = tmp_path / "full.pb"
    r = run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a),
                          "--keep_initial_solution", "--fixed_images", ms.image_names[9]])
    assert r.returncode == 0 and o.read_bytes() == outs[0]
    a_, b_ = _both_hosts(checker_exe, ["--h"])
    for r in (a_, b_):
        assert r.returncode == 0 and r.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
        assert b"keep" not in r.stdout


def test_torchrun_ranks_refuse_a_kept_solution(incremental, tmp_path):
    """A start solution is not supported for torchrun ranks: the flag is refused as --initial_solution is."""
    ms, m, a, A = incremental
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", str(m), "--output_file", str(tmp_path / "o.pb"),
                        "--initial_solution", str(a), "--keep_initial_solution"], capture_output=True, env=env)
    assert r.returncode == 2
    assert r.stderr == b"ERROR: --initial_solution: torchrun ranks start from zeros; use --gpus N\n"
    assert not (tmp_path / "o.pb").exists()


# ---------------------------------------------------------------------------------------------------
# the reference's own create_and_solve_problem on the kept mask
# ---------------------------------------------------------------------------------------------------
def partial_solution(ms, g, seed):
    """planted_solution over the first two thirds of the images only, so that the kept set is partial."""
    full = wire.decode_solution(planted_solution(ms, g, seed))
    keep = set(ms.image_names[: 2 * len(ms.image_names) // 3])
    return b"".join(image(nm, [displacement(f, a, b) for f, a, b in zip(fi.tolist(), di, dj)])
                    for nm, _, fi, di, dj in full if nm in keep)


@pytest.mark.parametrize("name", ["cfg2", "cfg4", "ring60"])
@pytest.mark.parametrize("with_fixed", [False, True], ids=["keep", "keep+fixed"])
def test_reference_function_on_the_kept_mask(oracle, name, with_fixed):
    ms, g, p = host_scene(name)
    data = partial_solution(ms, g, 23)
    x0, _, has = wire.join_solution(data, ms.image_names, g["node_image"], g["node_feat"], entries=True)
    fixed = np.zeros(len(ms.image_names), bool)
    if with_fixed:
        fixed[-1] = True                                                  # an image the file does not list
    const = ((constant_of(g, fixed) != 0) | has).astype(np.uint8)
    c = const.astype(bool)
    assert has.any() and not c.all()
    assert ((sizes_of(g) > 1) & (np.add.reduceat(~c[g["comp_nodes"].astype(np.int64)],
                                                g["comp_ptr"][:-1].astype(np.int64)) > 0)).any()
    ref = ref_solve(p, const, x0)
    pos, st = oracle.solve(with_mask(p, const), oracle.default_options(n_threads=8), positions=x0)
    err = assert_matches_reference(with_mask(p, const), (pos, st), ref, (name, with_fixed))
    assert err <= 1e-12, (name, err)
    assert np.array_equal(bits(pos[c]), bits(x0[c])) and np.array_equal(bits(ref[0][c]), bits(x0[c]))
    assert ref[1]["n_solved"] == int((sizes_of(g) > 1).sum()) == st["n_solved"]
    assert name in CPU_SCALES
