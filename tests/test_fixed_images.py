"""Fixed images and start solutions on the CPU: the host join of a SolutionFile against a scene
(lfr_wire_join_solution, include/lfr_wire.h) against a plain statement of its rule, and the drop-in's
--fixed_images / --initial_solution through the native executable linked against the CPU checker
(oracle/liblfr_ref.so), compared with the checker's lfr_solve on arrays built here from the host stage."""
import ctypes as C
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import USAGE
from lfr_b200.graph import host_input_arrays, host_stage_export, problem_from_stage
from lfr_b200.solver import assemble_solution
from test_ref_solve import GOLD, LAUNCHER, untimed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LFR_EINVAL = -1


# ---------------------------------------------------------------------------------------------------
# a SolutionFile written field by field, and the join rule stated plainly
# ---------------------------------------------------------------------------------------------------
def varint(n, pad=0):
    """`n` as a varint; pad > 0 adds that many redundant continuation bytes (a non-canonical encoding)."""
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        out.append(b | 0x80 if n else b)
        if not n:
            break
    if pad:
        out[-1] |= 0x80
        out += b"\x80" * (pad - 1) + b"\x00"
    return bytes(out)


def field(num, wt, payload):
    if wt == 2:
        return varint(num << 3 | 2) + varint(len(payload)) + payload
    return varint(num << 3 | wt) + payload


def f32(x):
    return np.float32(x).tobytes()


def displacement(feat, di, dj, order=(1, 2, 3), pad=0, unknown=False):
    parts = {1: field(1, 0, varint(int(feat), pad)), 2: field(2, 5, f32(di)), 3: field(3, 5, f32(dj))}
    body = b"".join(parts[k] for k in order)
    if unknown:
        body += field(9, 0, varint(7)) + field(10, 2, b"skip me")
    return body


def image(name, disps, fact=1.0, name_first=True, decoy=None):
    name_f = field(1, 2, name.encode("utf-8", errors="surrogateescape"))
    if decoy is not None:  # a repeated singular field: the last one counts
        name_f = field(1, 2, decoy.encode()) + name_f
    body = b"".join(field(3, 2, d) for d in disps)
    body = (name_f + field(2, 5, f32(fact)) + body) if name_first else (body + field(2, 5, f32(fact)) + name_f)
    return field(1, 2, body)


def join_model(data, image_names, node_image, node_feat):
    """The rule in plain Python: the last Image message of a name wins as a whole, within it the last
    displacement of a feature; start = ((double) di, (double) dj), 0 without an entry."""
    msgs = wire.decode_solution(data)
    last = {}
    for i, m in enumerate(msgs):
        last[m[0]] = i
    id_of = {n: k for k, n in enumerate(image_names)}
    table = {}
    for nm, i in last.items():
        if nm not in id_of:
            continue
        _, _, fi, di, dj = msgs[i]
        for f, a, b in zip(fi.tolist(), di, dj):
            table[(id_of[nm], int(f))] = (np.float64(a), np.float64(b))
    pos = np.zeros((len(node_image), 2), np.float64)
    n = 0
    for v, (im, ft) in enumerate(zip(np.asarray(node_image).tolist(), np.asarray(node_feat).tolist())):
        if (im, ft) in table:
            pos[v] = table[(im, ft)]
            n += 1
    return pos, n


def stage(ms, banned=()):
    skip, arrs = host_input_arrays(ms, banned)
    rc, out, sz = host_stage_export(arrs, len(ms.image_names))
    assert rc == 0
    return skip, out, sz


def random_solution(ms, out, rng, frac=0.7, dup_images=2, extra_names=("not-in-scene.png",)):
    """A SolutionFile over a scene's nodes: a random subset per image, shuffled, some features repeated,
    some images listed twice (an earlier, partial message), names and features not in the scene."""
    msgs = []
    for k, name in enumerate(ms.image_names):
        feats = np.unique(out["node_feat"][out["node_image"] == k])
        if rng.random() < 0.2:
            feats = np.concatenate([feats, [feats.max() + 1 if feats.size else 5]])      # a feature not in the scene
        pick = feats[rng.random(feats.shape[0]) < frac]
        rng.shuffle(pick)
        disps = [displacement(f, *rng.uniform(-0.6, 0.6, 2)) for f in pick]
        if pick.size and rng.random() < 0.5:
            disps.append(displacement(pick[0], *rng.uniform(-0.6, 0.6, 2)))           # repeated feature: last wins
        msgs.append(image(name, disps))
    for k in rng.choice(len(ms.image_names), size=min(dup_images, len(ms.image_names)), replace=False):
        msgs.insert(0, image(ms.image_names[k], [displacement(f, 0.25, -0.25) for f in range(40)]))  # loses as a whole
    for nm in extra_names:
        msgs.append(image(nm, [displacement(1, 0.1, 0.1)]))
    return b"".join(msgs)


# ---------------------------------------------------------------------------------------------------
# the host join
# ---------------------------------------------------------------------------------------------------
def test_host_join_equals_the_rule_on_a_synthetic_scene():
    rng = np.random.default_rng(3)
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    _, out, _ = stage(ms)
    data = random_solution(ms, out, rng)
    got, n = wire.join_solution(data, ms.image_names, out["node_image"], out["node_feat"])
    want, n_want = join_model(data, ms.image_names, out["node_image"], out["node_feat"])
    assert n == n_want and 0 < n < out["node_image"].shape[0]
    assert got.tobytes() == want.tobytes()


def test_host_join_duplicate_rule():
    names = ["a.png", "b.png", "c.png"]
    node_image = np.array([0, 0, 0, 1, 1, 2], np.uint32)
    node_feat = np.array([1, 2, 3, 1, 7, 4], np.uint32)
    data = (image("a.png", [displacement(1, 0.1, 0.2), displacement(2, 0.3, 0.4)])     # replaced as a whole below
            + image("b.png", [displacement(7, -0.5, 0.5), displacement(7, 0.125, -0.125), displacement(9, 1, 1)])
            + image("zzz.png", [displacement(4, 0.9, 0.9)])
            + image("a.png", [displacement(3, 0.75, -0.75)]))
    pos, n = wire.join_solution(data, names, node_image, node_feat)
    assert n == 2
    want = np.zeros((6, 2))
    want[2] = (0.75, -0.75)          # a.png's last message alone: features 1 and 2 are not started
    want[4] = (0.125, -0.125)        # b.png feature 7: the last displacement
    assert pos.tobytes() == want.tobytes()
    assert pos.tobytes() == join_model(data, names, node_image, node_feat)[0].tobytes()


def test_host_join_empty_file_and_unknown_entries():
    names = ["a.png", "b.png"]
    node_image = np.array([0, 1, 1], np.uint32)
    node_feat = np.array([0, 0, 5], np.uint32)
    pos, n = wire.join_solution(b"", names, node_image, node_feat)
    assert n == 0 and not pos.any()
    pos, n = wire.join_solution(image("c.png", [displacement(0, 0.5, 0.5)]) + image("a.png", [displacement(9, 0.5, 0.5)]),
                                names, node_image, node_feat)
    assert n == 0 and not pos.any()
    pos, n = wire.join_solution(b"", [], np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    assert n == 0 and pos.shape == (0, 2)


def test_host_join_non_canonical_encodings():
    """Fields out of order, redundant varint bytes, unknown fields, a repeated name field, an Image whose
    name comes last: decoded as protobuf does, so they join like the canonical bytes."""
    names = ["a.png", "b.png"]
    node_image = np.array([0, 0, 1], np.uint32)
    node_feat = np.array([3, 300, 2], np.uint32)
    canon = image("a.png", [displacement(3, 0.1, -0.2), displacement(300, 0.3, 0.4)]) + image("b.png", [displacement(2, -0.5, 0.25)])
    odd = (image("a.png", [displacement(3, 0.1, -0.2, order=(3, 1, 2), pad=2, unknown=True),
                           displacement(300, 0.3, 0.4, order=(2, 3, 1), pad=1)], decoy="b.png")
           + image("b.png", [displacement(2, -0.5, 0.25, unknown=True)], name_first=False))
    a, na = wire.join_solution(canon, names, node_image, node_feat)
    b, nb = wire.join_solution(odd, names, node_image, node_feat)
    assert na == nb == 3 and a.tobytes() == b.tobytes()
    assert b.tobytes() == join_model(odd, names, node_image, node_feat)[0].tobytes()


@pytest.mark.parametrize("bad", [b"\x0a\xff", b"\x0a\x05\x0a\x09abc", b"\x0a\xff\xff\xff\xff\x0f not a protobuf",
                                 image("a.png", [displacement(1, 0.5, 0.5)])[:-3]])
def test_host_join_refuses_malformed_bytes(bad):
    L = wire._lib()
    buf = np.frombuffer(bad, np.uint8)
    pos = np.full(2, 7.0)
    n = C.c_uint64(5)
    blob, off = wire._names_blob(["a.png"])
    rc = L.lfr_wire_join_solution(buf.ctypes.data, buf.size, 1, blob.ctypes.data, off.ctypes.data, 1,
                                  np.zeros(1, np.uint32).ctypes.data, np.ones(1, np.uint32).ctypes.data, pos.ctypes.data,
                                  C.byref(n))
    assert rc == LFR_EINVAL and (pos == 7.0).all()
    with pytest.raises(wire.ParseError):
        wire.join_solution(bad, ["a.png"], np.zeros(1, np.uint32), np.ones(1, np.uint32))


# ---------------------------------------------------------------------------------------------------
# the native executable on the CPU checker
# ---------------------------------------------------------------------------------------------------
def _csrc_build():
    spec = importlib.util.spec_from_file_location("lfr_csrc_build", os.path.join(ROOT, "local-feature-refinement_b200", "csrc", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def checker_exe(tmp_path_factory, oracle):
    """lfr_solve_main.cc linked against the CPU checker instead of the CUDA library (host route only)."""
    out = str(tmp_path_factory.mktemp("native") / "solve_native_checker")
    b = _csrc_build()
    b.build_host()
    return b.build_exe(force=True, out=out, solve_lib_dir=os.path.join(ROOT, "oracle"), solve_lib="lfr_ref")


def run(exe, args):
    return subprocess.run([exe] + args, capture_output=True)


def oracle_expected(oracle, ms, fixed_names, start_bytes, banned=()):
    """SolutionFile bytes of the checker's lfr_solve on is_const / start built here from the host stage."""
    skip, out, sz = stage(ms, banned)
    p = problem_from_stage(ms, skip, out, sz, "native")
    fixed = np.array([n in set(fixed_names) for n in ms.image_names], bool)
    is_const = ((out["is_root"] != 0) | fixed[out["node_image"].astype(np.int64)]).astype(np.uint8)
    start = np.zeros((sz["n_nodes"], 2))
    if start_bytes is not None:
        start, _ = join_model(start_bytes, ms.image_names, out["node_image"], out["node_feat"])
    p_const = problem_from_stage(ms, skip, out, sz, "native")
    p_const.is_root = is_const
    pos, st = oracle.solve(p_const, oracle.default_options(n_threads=4), positions=start)
    sol = assemble_solution(p, pos)
    return wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj), pos, start, is_const, out


def test_native_host_route_with_both_options_equals_the_checker(checker_exe, oracle, tmp_path):
    rng = np.random.default_rng(11)
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    _, out, _ = stage(ms)
    start = random_solution(ms, out, rng)
    m, s, o = tmp_path / "m.pb", tmp_path / "start.pb", tmp_path / "o.pb"
    m.write_bytes(wire.encode_matching_file(ms))
    s.write_bytes(start)
    fixed = [ms.image_names[1], ms.image_names[4], "not-an-image.png"]
    r = run(checker_exe, ["--matches_file", str(m), "--output_file", str(o), "--fixed_images", fixed[0],
                          "--fixed_images=" + fixed[1], "--fix", fixed[2], "--initial_solution", str(s)])
    assert r.returncode == 0, r.stderr
    want, pos, x0, is_const, _ = oracle_expected(oracle, ms, fixed, start)
    assert o.read_bytes() == want
    # fixed nodes keep their start values bit for bit
    c = is_const.astype(bool)
    assert pos[c].tobytes() == x0[c].tobytes()


@pytest.mark.parametrize("name", ["tiny", "linesearch"])
def test_fixed_names_outside_the_scene_change_nothing(checker_exe, tmp_path, name):
    o = tmp_path / "o.pb"
    r = run(checker_exe, ["--matches_file", os.path.join(GOLD, name + "_matches.pb"), "--output_file", str(o),
                          "--fixed_images", "no-such-image.png", "--fixed_images", ""])
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == open(os.path.join(GOLD, name + "_solution.pb"), "rb").read()
    assert untimed(r.stdout.decode()) == open(os.path.join(GOLD, name + "_stdout.txt")).read().splitlines()


def test_initial_solution_of_zeros_changes_nothing(checker_exe, tmp_path):
    """An all-zero start is the reference's start: the goldens come out unchanged."""
    m = os.path.join(GOLD, "tiny_matches.pb")
    ms = wire.read_matching_file(m)
    _, out, _ = stage(ms)
    zero = b"".join(image(ms.image_names[k], [displacement(f, 0.0, 0.0) for f in np.unique(out["node_feat"][out["node_image"] == k])])
                    for k in range(len(ms.image_names)))
    s, o = tmp_path / "zero.pb", tmp_path / "o.pb"
    s.write_bytes(zero)
    r = run(checker_exe, ["--matches_file", m, "--output_file", str(o), "--init", str(s)])
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read()


def _both_hosts(checker_exe, args):
    """(native on the checker, Python launcher): their exit code, stdout and stderr."""
    a = run(checker_exe, args)
    env = dict(os.environ, LFR_SOLVE_PYTHON="1")
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=env)
    return a, b


def test_start_solution_errors_come_first(checker_exe, tmp_path):
    m = os.path.join(GOLD, "tiny_matches.pb")
    missing = str(tmp_path / "absent.pb")
    a, b = _both_hosts(checker_exe, ["--matches_file", m, "--output_file", str(tmp_path / "o.pb"), "--initial_solution", missing])
    for r in (a, b):
        assert r.returncode == 2 and r.stdout == b""
        assert r.stderr == ("ERROR: cannot read the initial solution file '%s'\n" % missing).encode()
    bad = tmp_path / "bad.pb"
    bad.write_bytes(b"\x0a\xff\xff\xff\xff\x0f not a protobuf")
    a, b = _both_hosts(checker_exe, ["--matches_file", m, "--output_file", str(tmp_path / "o.pb"), "--initial_solution=" + str(bad)])
    for r in (a, b):
        assert (r.returncode, r.stdout, r.stderr) == (255, b"", b"Failed to parse proto object.\n")
    assert not (tmp_path / "o.pb").exists()


def test_command_line_of_the_new_options(checker_exe, tmp_path):
    m = os.path.join(GOLD, "tiny_matches.pb")
    # --help stays the reference's: the extras are not listed
    a, b = _both_hosts(checker_exe, ["--help"])
    assert a.returncode == b.returncode == 0 and a.stdout == b.stdout
    assert b"fixed_images" not in a.stdout and b"initial_solution" not in a.stdout
    assert a.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
    # --initial_solution is single-valued; a missing argument; an ambiguous prefix is still none of ours
    for argv, msg in [(["--matches_file", m, "--output_file", "o", "--initial_solution", "a", "--initial_solution", "b"],
                       b"option '--initial_solution' cannot be specified more than once"),
                      (["--matches_file", m, "--output_file", "o", "--fixed_images"],
                       b"the required argument for option '--fixed_images' is missing"),
                      (["--matches_file", m, "--output_file", "o", "--initial_solution"],
                       b"the required argument for option '--initial_solution' is missing")]:
        a, b = _both_hosts(checker_exe, argv)
        assert a.returncode == b.returncode == 1 and a.stderr == b.stderr and a.stderr.startswith(b"ERROR: " + msg)
