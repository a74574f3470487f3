"""Updating an earlier SolutionFile on the CPU: the host update (lfr_wire_update_solution, include/lfr_wire.h)
against a plain statement of its rule, and the drop-in's --update_initial_solution through the native
executable linked against the CPU checker (oracle/liblfr_ref.so) and the Python host's path.  A component a
new keypoint joins is solved as the every-pair run without a file solves it; every other component comes
back with the file's float bits.  The reference's own solve binary (oracle/_ref/solve) anchors the touched
nodes."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import USAGE
from lfr_b200.graph import problem_from_stage
from lfr_b200.solver import constant_problem
from refsrc_util import _build_mod
from test_fixed_images import checker_exe, displacement, image, random_solution, run, stage  # noqa: F401
from test_fixed_images_ref import bits, constant_of
from test_keep_solution import KEEP_ERROR, entries_model
from test_ref_solve import GOLD, LAUNCHER

LFR_EINVAL = -1
EMPTY, SKIPPED = 7, 0
UPDATE_ERROR = b"ERROR: --update_initial_solution needs --initial_solution FILE\n"
BOTH_ERROR = b"ERROR: --update_initial_solution and --keep_initial_solution exclude each other\n"
# float bits A.pb carries through held components: -0.0, the smallest denormal, a quiet NaN with a payload
SPECIAL_BITS = [0x80000000, 0x00000001, 0x7FC12345, 0x807FFFFF]


def update_model(data, names, node_image, node_feat, node_comp, n_components):
    """The rule in plain Python: a component is touched when one of its nodes has no entry (the join rule of
    entries_model); held = entry AND not touched; positions = the entry when held, else 0."""
    pos, _, has = entries_model(data, names, node_image, node_feat)
    comp = np.asarray(node_comp, np.int64)
    touched = np.zeros(n_components, bool)
    touched[comp[~has]] = True
    held = has & ~touched[comp]
    pos = np.where(held[:, None], pos, 0.0)
    return pos, held, int(held.sum()), int(touched.sum())


def check_update(data, names, g):
    C_ = int(g["comp_ptr"].shape[0] - 1)
    got = wire.update_solution(data, names, g["node_image"], g["node_feat"], g["comp"], C_)
    want = update_model(data, names, g["node_image"], g["node_feat"], g["comp"], C_)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]) and got[2:] == want[2:]
    return got


# ---------------------------------------------------------------------------------------------------
# the host update
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [4, 5, 6])
def test_update_equals_the_rule_on_a_synthetic_scene(seed):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    _, g, _ = stage(ms)
    pos, held, n_held, n_touched = check_update(random_solution(ms, g, np.random.default_rng(seed), frac=0.97),
                                                ms.image_names, g)
    assert 0 < n_held < held.shape[0] and 0 < n_touched < g["comp_ptr"].shape[0] - 1


def test_update_duplicate_rule_and_single_node_components():
    """a.png's first message would cover component 0, but the later one wins as a whole; component 2 is a
    single node with an entry, component 3 one without."""
    names = ["a.png", "b.png", "c.png"]
    g = dict(node_image=np.array([0, 0, 1, 1, 2, 2, 0], np.uint32), node_feat=np.array([1, 2, 7, 8, 4, 5, 3], np.uint32),
             comp=np.array([0, 0, 1, 1, 2, 3, 0], np.uint32), comp_ptr=np.array([0, 3, 5, 6, 7], np.uint32))
    data = (image("a.png", [displacement(1, 0.1, 0.2), displacement(2, 0.3, 0.4), displacement(3, 0.1, 0.1)])
            + image("b.png", [displacement(7, -0.5, 0.5), displacement(8, 0.25, 0.0), displacement(8, 0.0, -0.0)])
            + image("c.png", [displacement(4, 0.125, -0.125)])
            + image("a.png", [displacement(1, 0.75, -0.75), displacement(3, 0.5, 0.5)]))
    pos, held, n_held, n_touched = check_update(data, names, g)
    assert held.tolist() == [False, False, True, True, True, False, False]
    assert (n_held, n_touched) == (3, 2)
    assert bits(pos[3]).tolist() == bits(np.array([0.0, -0.0])).tolist()        # the last displacement of 8
    assert pos[0].tolist() == [0.0, 0.0] and bits(pos[0]).tolist() == [0, 0]      # touched: +0, not its entry


def test_update_empty_file_touches_every_component_and_full_file_none():
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    _, g, _ = stage(ms)
    C_ = int(g["comp_ptr"].shape[0] - 1)
    pos, held, n_held, n_touched = check_update(b"", ms.image_names, g)
    assert n_held == 0 and n_touched == C_ and not held.any() and not pos.any()
    full = random_solution(ms, g, np.random.default_rng(1), frac=1.01, extra_names=())
    pos, held, n_held, n_touched = check_update(full, ms.image_names, g)
    assert n_touched == 0 and held.all() and n_held == held.shape[0]
    assert pos.tobytes() == wire.join_solution(full, ms.image_names, g["node_image"], g["node_feat"])[0].tobytes()


def _raw(data, names, n_nodes=1, comp=(0,), n_comp=1, held_null=False, comp_null=False):
    L = wire._lib()
    buf = np.frombuffer(data, np.uint8)
    pos = np.full(2 * n_nodes, 7.0)
    held = np.full(n_nodes, 9, np.uint8)
    n, t = C.c_uint64(5), C.c_uint32(6)
    blob, off = wire._names_blob(names)
    comp = np.asarray(comp, np.uint32)
    rc = L.lfr_wire_update_solution(buf.ctypes.data if buf.size else None, buf.size, len(names), blob.ctypes.data,
                                    off.ctypes.data, n_nodes, np.zeros(n_nodes, np.uint32).ctypes.data,
                                    np.ones(n_nodes, np.uint32).ctypes.data, None if comp_null else comp.ctypes.data,
                                    n_comp, pos.ctypes.data, None if held_null else held.ctypes.data, C.byref(n), C.byref(t))
    return rc, pos, held, n.value, t.value


@pytest.mark.parametrize("bad", [b"\x0a\xff", b"\x0a\x05\x0a\x09abc", b"\x0a\xff\xff\xff\xff\x0f not a protobuf",
                                 image("a.png", [displacement(1, 0.5, 0.5)])[:-3]])
def test_update_refuses_malformed_bytes(bad):
    rc, pos, held, n, t = _raw(bad, ["a.png"])
    assert rc == LFR_EINVAL and (pos == 7.0).all() and (held == 9).all() and (n, t) == (5, 6)
    with pytest.raises(wire.ParseError):
        wire.update_solution(bad, ["a.png"], np.zeros(1, np.uint32), np.ones(1, np.uint32), np.zeros(1, np.uint32), 1)


def test_update_refuses_null_arrays_and_component_ids_out_of_range():
    ok = image("a.png", [displacement(1, 0.5, 0.5)])
    assert _raw(ok, ["a.png"])[0] == 0
    for kw in (dict(held_null=True), dict(comp_null=True), dict(comp=(1,)), dict(comp=(0,), n_comp=0)):
        rc, pos, held, n, t = _raw(ok, ["a.png"], **kw)
        assert rc == LFR_EINVAL and (pos == 7.0).all() and (n, t) == (5, 6), kw
    with pytest.raises(ValueError):
        wire.update_solution(ok, ["a.png"], np.zeros(1, np.uint32), np.ones(1, np.uint32), np.ones(1, np.uint32), 1)


# ---------------------------------------------------------------------------------------------------
# the incremental scenario through the native executable on the CPU checker
# ---------------------------------------------------------------------------------------------------
# (generator, scale, seed, k): A.pb is the plain solve without the last k images.  ring60 at 0.3 has
# oversized meta-components, so its components come from cuts.
SCENARIOS = {"cfg2-k1": ("cfg2", 0.1, 3, 1), "cfg2-k3": ("cfg2", 0.1, 3, 3), "ring60-k2": ("ring60", 0.3, None, 2)}
_scenarios = {}


def with_special_values(a_bytes, held_keys):
    """A.pb with SPECIAL_BITS written over the di / dj of the first held (name, feature) keys: they must come
    back bit for bit."""
    msgs = wire.decode_solution(a_bytes)
    todo = {k: SPECIAL_BITS[i % len(SPECIAL_BITS)] for i, k in enumerate(held_keys[:2 * len(SPECIAL_BITS)])}
    out = []
    for nm, fact, fi, di, dj in msgs:
        di, dj = di.copy(), dj.copy()
        for j, f in enumerate(fi.tolist()):
            if (nm, f) in todo:
                di.view(np.uint32)[j] = todo[(nm, f)]
                dj.view(np.uint32)[j] = todo[(nm, f)] ^ 0x80000000
        out.append((nm, fact, fi, di, dj))
    return encode_msgs(out), len(todo)


def encode_msgs(msgs):
    ptr = np.cumsum([0] + [m[2].shape[0] for m in msgs]).astype(np.uint64)
    cat = (lambda k, dt: np.concatenate([m[k] for m in msgs]).astype(dt) if msgs else np.zeros(0, dt))
    return wire.encode_solution([m[0] for m in msgs], np.array([m[1] for m in msgs], np.float32), ptr,
                                cat(2, np.uint32), cat(3, np.float32), cat(4, np.float32))


def table(data):
    """(name, feature) -> (di bits, dj bits) under the join rule."""
    t = {}
    last = {}
    for nm, _, fi, di, dj in wire.decode_solution(data):
        last[nm] = {f: (int(a), int(b)) for f, a, b in zip(fi.tolist(), di.view(np.uint32), dj.view(np.uint32))}
    for nm, d in last.items():
        for f, v in d.items():
            t[(nm, f)] = v
    return t


def assembled(plain_bytes, a_bytes, held_keys):
    """The plain run's SolutionFile with every held (name, feature) given A's float bits."""
    a = table(a_bytes)
    held = set(held_keys)
    out = []
    for nm, fact, fi, di, dj in wire.decode_solution(plain_bytes):
        di, dj = di.copy(), dj.copy()
        for j, f in enumerate(fi.tolist()):
            if (nm, f) in held:
                di.view(np.uint32)[j], dj.view(np.uint32)[j] = a[(nm, f)]
        out.append((nm, fact, fi, di, dj))
    return encode_msgs(out)


def scenario(checker_exe, tmp_path_factory, key):  # noqa: F811
    """(MatchSet, every-pair path, A's path, A's bytes, graph, Problem, held, touched-by-component)."""
    if key not in _scenarios:
        gen, scale, seed, k = SCENARIOS[key]
        d = tmp_path_factory.mktemp("update_" + key)
        ms = synth.generate(gen, scale=scale) if seed is None else synth.generate(gen, scale=scale, seed=seed)
        m, a0, a = d / "m.pb", d / "a0.pb", d / "a.pb"
        m.write_bytes(wire.encode_matching_file(ms))
        args = ["--matches_file", str(m), "--output_file", str(a0)]
        for nm in ms.image_names[-k:]:
            args += ["--banned_images", nm]
        r = run(checker_exe, args)
        assert r.returncode == 0, r.stderr
        skip, g, sz = stage(ms)
        p = problem_from_stage(ms, skip, g, sz, "native")
        C_ = p.n_components
        _, held, _, _ = update_model(a0.read_bytes(), ms.image_names, g["node_image"], g["node_feat"], g["comp"], C_)
        keys = [(ms.image_names[i], int(f)) for i, f in zip(g["node_image"][held].tolist(), g["node_feat"][held].tolist())]
        data, n_special = with_special_values(a0.read_bytes(), keys)
        assert n_special == 2 * len(SPECIAL_BITS)
        a.write_bytes(data)
        _, held, n_held, n_touched = update_model(data, ms.image_names, g["node_image"], g["node_feat"], g["comp"], C_)
        assert 0 < n_held < held.shape[0] and 0 < n_touched < C_
        _scenarios[key] = (ms, m, a, data, g, p, held)
    return _scenarios[key]


def held_keys(ms, g, held):
    return [(ms.image_names[i], int(f)) for i, f in zip(g["node_image"][held].tolist(), g["node_feat"][held].tolist())]


@pytest.mark.parametrize("key", list(SCENARIOS))
def test_scenarios_extend_old_tracks_and_cut_the_ring(checker_exe, tmp_path_factory, key):  # noqa: F811
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, key)
    if key.startswith("ring60"):
        assert p.info.get("n_oversized_meta_components", 0) > 0, p.info
    # the new images extend tracks of old images: a touched component holds nodes of both
    new = np.isin(g["node_image"].astype(np.int64), np.arange(len(ms.image_names) - SCENARIOS[key][3], len(ms.image_names)))
    comp = g["comp"].astype(np.int64)
    has_new = np.bincount(comp[new], minlength=p.n_components) > 0
    has_old = np.bincount(comp[~new], minlength=p.n_components) > 0
    assert (has_new & has_old).any()


VARIANTS = {"plain": [], "carry": ["--carry_initial_solution"], "fixed": ["--fixed_images", 1],
            "fixed-new": ["--fixed_images", -1]}


def _variant(ms, variant):
    return [ms.image_names[x] if isinstance(x, int) else x for x in VARIANTS[variant]]


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("key", list(SCENARIOS))
def test_native_update_is_the_plain_run_on_touched_components_and_a_elsewhere(checker_exe, tmp_path_factory, tmp_path,
                                                                             key, variant):  # noqa: F811
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, key)
    extra = _variant(ms, variant)
    o, o0 = tmp_path / "o.pb", tmp_path / "o0.pb"
    plain_extra = [x for x in extra if x != "--carry_initial_solution"]
    r = run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a),
                          "--update_initial_solution"] + extra)
    assert r.returncode == 0, r.stderr
    r0 = run(checker_exe, ["--matches_file", str(m), "--output_file", str(o0)] + plain_extra)
    assert r0.returncode == 0, r0.stderr
    want = assembled(o0.read_bytes(), A, held_keys(ms, g, held))
    if "--carry_initial_solution" in extra:
        sol = wire.decode_solution(want)
        ptr = np.cumsum([0] + [x[2].shape[0] for x in sol]).astype(np.uint64)
        want, _ = wire.encode_solution_carried([x[0] for x in sol], np.array([x[1] for x in sol], np.float32), ptr,
                                               np.concatenate([x[2] for x in sol]), np.concatenate([x[3] for x in sol]),
                                               np.concatenate([x[4] for x in sol]), A)
    assert o.read_bytes() == want
    # the special values of A come back bit for bit
    got, a_t = table(o.read_bytes()), table(A)
    n = sum(1 for k in held_keys(ms, g, held) if a_t[k][0] in SPECIAL_BITS and got[k] == a_t[k])
    assert n == 2 * len(SPECIAL_BITS)
    # the same stdout lines as the plain run, except the outside count (held values differ)
    lines = [[l.split(":")[0] if l.startswith("# points with") else l for l in x.stdout.decode().splitlines()
              if " time:" not in l] for x in (r, r0)]
    assert lines[0] == lines[1]


@pytest.mark.parametrize("key", ["cfg2-k1", "ring60-k2"])
def test_touched_component_stats_are_the_plain_runs(checker_exe, tmp_path_factory, oracle, key):  # noqa: F811
    """In-process on the checker: the update's mask and start solve every touched component with the plain
    run's positions, iterations and termination, bit for bit; held components end EMPTY or SKIPPED."""
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, key)
    opts = oracle.default_options(n_threads=4)
    q, start = constant_problem(p, (), A, update_initial_solution=True)
    assert np.array_equal(q.is_root, ((g["is_root"] != 0) | held).astype(np.uint8))
    pos, st = oracle.solve(q, opts, positions=start)
    pos0, st0 = oracle.solve(p, opts)
    comp = g["comp"].astype(np.int64)
    touched = np.zeros(p.n_components, bool)
    touched[comp[~held]] = True
    touched = touched[p.comp_order.astype(np.int64)]           # by dispatch slot, as the stats are
    free = ~held
    assert pos[free].tobytes() == pos0[free].tobytes()
    assert bits(pos[held]).tobytes() == bits(start[held]).tobytes()
    for k in ("iterations", "termination"):
        assert np.array_equal(st[k][touched], st0[k][touched]), k
    for k in ("initial_cost", "final_cost"):
        if k in st:
            assert bits(st[k][touched]).tobytes() == bits(st0[k][touched]).tobytes(), k
    size = np.diff(p.comp_ptr.astype(np.int64))
    assert np.all(st["termination"][~touched & (size > 1)] == EMPTY)
    assert np.all(st["termination"][~touched & (size == 1)] == SKIPPED)


def test_python_host_path_equals_the_native_host(checker_exe, tmp_path_factory, tmp_path, oracle, monkeypatch):  # noqa: F811
    """refine(..., update_initial_solution=True) on the host route with the checker as the solve, with and
    without carry: the native executable's bytes."""
    from lfr_b200.solver import refine
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, "cfg2-k3")
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    opts = oracle.default_options(n_threads=4)
    for extra in ([], ["--carry_initial_solution", "--fixed_images", ms.image_names[2]]):
        o = tmp_path / "o.pb"
        r = run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a), "--u"] + extra)
        assert r.returncode == 0, r.stderr
        fixed = [x for f, x in zip(extra, extra[1:]) if f == "--fixed_images"]
        _, _, _, sol = refine(wire.read_matching_file(str(m)), (), solve_fn=lambda q, x=None: oracle.solve(q, opts, positions=x),
                              fixed_images=fixed, initial_solution=A, update_initial_solution=True)
        args = (sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj)
        data = wire.encode_solution_carried(*args, A)[0] if extra else wire.encode_solution(*args)
        assert data == o.read_bytes(), extra


def test_empty_and_covering_files(checker_exe, tmp_path_factory, tmp_path):  # noqa: F811
    """An empty A.pb gives the plain run's bytes; an A.pb covering every node touches nothing and gives A's
    values back."""
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, "cfg2-k1")
    empty, o, o0 = tmp_path / "empty.pb", tmp_path / "o.pb", tmp_path / "o0.pb"
    empty.write_bytes(b"")
    assert run(checker_exe, ["--matches_file", str(m), "--output_file", str(o0)]).returncode == 0
    assert run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(empty),
                             "--update_initial_solution"]).returncode == 0
    assert o.read_bytes() == o0.read_bytes()
    full = tmp_path / "full.pb"
    rng = np.random.default_rng(8)
    full.write_bytes(random_solution(ms, g, rng, frac=1.01, extra_names=()))
    _, held_f, n_held, n_touched = update_model(full.read_bytes(), ms.image_names, g["node_image"], g["node_feat"], g["comp"],
                                                p.n_components)
    assert n_touched == 0 and held_f.all()
    assert run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(full),
                             "--update_initial_solution"]).returncode == 0
    got, f_t = table(o.read_bytes()), table(full.read_bytes())
    keys = held_keys(ms, g, held_f)
    assert all(got.get(k, (0, 0)) == f_t[k] for k in keys)
    assert o.read_bytes() == assembled(o0.read_bytes(), full.read_bytes(), keys)


def test_repeated_image_name_follows_the_join_rule(checker_exe, tmp_path_factory, tmp_path):  # noqa: F811
    """A later, partial message of an old image wins as a whole: the components its missing features join are
    touched and solved as in the plain run."""
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, "cfg2-k1")
    nm = ms.image_names[0]
    msgs = wire.decode_solution(A)
    first = [x for x in msgs if x[0] == nm][0]
    data = A + encode_msgs([(nm, first[1], first[2][:1], first[3][:1], first[4][:1])])
    f = tmp_path / "dup.pb"
    f.write_bytes(data)
    _, held2, _, n_t2 = update_model(data, ms.image_names, g["node_image"], g["node_feat"], g["comp"], p.n_components)
    assert held2.sum() < held.sum() and not (held2 & ~held).any()
    o, o0 = tmp_path / "o.pb", tmp_path / "o0.pb"
    assert run(checker_exe, ["--matches_file", str(m), "--output_file", str(o0)]).returncode == 0
    assert run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(f),
                             "--update_initial_solution"]).returncode == 0
    assert o.read_bytes() == assembled(o0.read_bytes(), data, held_keys(ms, g, held2))


def test_reference_binary_anchors_the_touched_nodes(checker_exe, tmp_path_factory, tmp_path):  # noqa: F811
    """The reference's own solve (oracle/_ref/solve) on the every-pair MatchingFile: every touched node of the
    update run has its float bits."""
    ref_exe = _build_mod().build_solve()
    for key in ("cfg2-k3", "ring60-k2"):
        ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, key)
        o, o_ref = tmp_path / "o.pb", tmp_path / "ref.pb"
        r = subprocess.run([ref_exe, "--matches_file", str(m), "--output_file", str(o_ref)], capture_output=True)
        assert r.returncode == 0, r.stderr
        assert run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a),
                                 "--update_initial_solution"]).returncode == 0
        got, ref = table(o.read_bytes()), table(o_ref.read_bytes())
        n = 0
        for i, f in zip(g["node_image"][~held].tolist(), g["node_feat"][~held].tolist()):
            k = (ms.image_names[i], int(f))
            assert got.get(k, (0, 0)) == ref.get(k, (0, 0)), (key, k)
            n += 1
        assert n > 0


# ---------------------------------------------------------------------------------------------------
# the command line
# ---------------------------------------------------------------------------------------------------
def _both_hosts(checker_exe, args, env=None):  # noqa: F811
    a = subprocess.run([checker_exe] + args, capture_output=True, env=env)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=dict(env or os.environ, LFR_SOLVE_PYTHON="1"))
    return a, b


def test_bad_combinations_are_refused_first(checker_exe, tmp_path):  # noqa: F811
    m = os.path.join(GOLD, "tiny_matches.pb")
    o = tmp_path / "o.pb"
    base = ["--matches_file", m, "--output_file", str(o)]
    cases = [(base + ["--update_initial_solution"], UPDATE_ERROR),
             (["--update"] + base + ["--initial_solution="], UPDATE_ERROR),
             (base + ["--initial_solution", m, "--update_initial_solution", "--keep_initial_solution"], BOTH_ERROR),
             (base + ["--u", "--keep_initial_solution"], KEEP_ERROR),                 # the keep line comes first
             (base + ["--u", "--carry_initial_solution"],
              b"ERROR: --carry_initial_solution needs --initial_solution FILE\n")]
    for argv, err in cases:
        a, b = _both_hosts(checker_exe, argv)
        for r in (a, b):
            assert (r.returncode, r.stdout, r.stderr) == (2, b"", err), argv
    assert not o.exists()


def test_update_takes_no_value_and_foo_stays_unrecognised(checker_exe, tmp_path):  # noqa: F811
    m = os.path.join(GOLD, "tiny_matches.pb")
    base = ["--matches_file", m, "--output_file", str(tmp_path / "o.pb"), "--initial_solution", m]
    for flag in ("--update_initial_solution=x", "--update=", "--u=1"):
        a, b = _both_hosts(checker_exe, base + [flag])
        for r in (a, b):
            assert r.returncode == 1 and r.stdout == b""
            assert r.stderr == b"ERROR: option '--update_initial_solution' does not take any arguments\n\n" + USAGE.encode()
    a, b = _both_hosts(checker_exe, base + ["--foo"])
    for r in (a, b):
        assert r.returncode == 1 and r.stderr == b"ERROR: unrecognised option '--foo'\n\n" + USAGE.encode()


def test_prefixes_and_help(checker_exe, tmp_path_factory, tmp_path):  # noqa: F811
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, "cfg2-k1")
    outs = []
    for i, flag in enumerate(["--update_initial_solution", "--update", "--u"]):
        o = tmp_path / ("o%d.pb" % i)
        r = run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--init", str(a), flag])
        assert r.returncode == 0, r.stderr
        outs.append(o.read_bytes())
    assert outs[0] == outs[1] == outs[2]
    a_, b_ = _both_hosts(checker_exe, ["--help"])
    for r in (a_, b_):
        assert r.returncode == 0 and r.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
        assert b"update" not in r.stdout


def test_torchrun_ranks_refuse_an_update(checker_exe, tmp_path_factory, tmp_path):  # noqa: F811
    ms, m, a, A, g, p, held = scenario(checker_exe, tmp_path_factory, "cfg2-k1")
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", str(m), "--output_file", str(tmp_path / "o.pb"),
                        "--initial_solution", str(a), "--update_initial_solution"], capture_output=True, env=env)
    assert r.returncode == 2
    assert r.stderr == b"ERROR: --initial_solution: torchrun ranks start from zeros; use --gpus N\n"
    assert not (tmp_path / "o.pb").exists()


def test_refine_refuses_the_bad_combinations():
    from lfr_b200.solver import refine
    ms = synth.generate("cfg1", scale=0.2)
    with pytest.raises(ValueError, match="needs initial_solution"):
        refine(ms, update_initial_solution=True)
    with pytest.raises(ValueError, match="exclude each other"):
        refine(ms, initial_solution=b"", update_initial_solution=True, keep_initial_solution=True)


def test_constant_problem_without_the_flag_is_unchanged():
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    skip, g, sz = stage(ms)
    p = problem_from_stage(ms, skip, g, sz, "native")
    data = random_solution(ms, g, np.random.default_rng(2))
    q, start = constant_problem(p, [ms.image_names[1]], data)
    fixed = np.array([k == 1 for k in range(len(ms.image_names))])
    assert np.array_equal(q.is_root, constant_of(g, fixed))
    q2, start2 = constant_problem(p, [ms.image_names[1]], data, update_initial_solution=True)
    pos, held, _, _ = update_model(data, ms.image_names, g["node_image"], g["node_feat"], g["comp"], p.n_components)
    assert np.array_equal(q2.is_root, ((constant_of(g, fixed) != 0) | held).astype(np.uint8))
    assert start2.tobytes() == pos.tobytes()
    assert np.array_equal(p.is_root, g["is_root"])
