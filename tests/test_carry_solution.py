"""Carrying an earlier SolutionFile into the output on the CPU: lfr_wire_encode_solution_carried
(include/lfr_wire.h) against a plain Python statement of its rule, the reader's view through
consumer.apply_solution, the size protocol and refusals, and the drop-in's --carry_initial_solution through
the native executable linked against the CPU checker (oracle/liblfr_ref.so) and the Python host's path with
the checker as its solve: an earlier scene solved from the old pairs, then the new pairs alone.  The Python
launcher itself runs the scenario on the GPU (tests/test_gpu_carry_solution.py)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import consumer, synth, wire
from lfr_b200.cli import USAGE
from test_fixed_images import checker_exe, field, run, varint  # noqa: F401
from test_keep_solution import KEEP_ERROR
from test_ref_solve import GOLD, LAUNCHER

LFR_EINVAL = -1
CARRY_ERROR = b"ERROR: --carry_initial_solution needs --initial_solution FILE\n"


# ---------------------------------------------------------------------------------------------------
# SolutionFiles with exact float bits, and the rule stated plainly
# ---------------------------------------------------------------------------------------------------
def f32_bits(x):
    return int(np.float32(x).view(np.uint32))


def disp_bits(feat, a, b):
    """A Displacement with di / dj given as float32 bit patterns (every field written, zeros included)."""
    return field(1, 0, varint(int(feat))) + field(2, 5, int(a).to_bytes(4, "little")) + field(3, 5, int(b).to_bytes(4, "little"))


def image_bits(name, disps, fact_bits=f32_bits(1.0)):
    nm = name if isinstance(name, bytes) else name.encode("utf-8", errors="surrogateescape")
    return field(1, 2, field(1, 2, nm) + field(2, 5, int(fact_bits).to_bytes(4, "little")) +
                 b"".join(field(3, 2, disp_bits(*d)) for d in disps))


def messages(data):
    """[(name bytes, fact bits, [(feature, di bits, dj bits)] in file order)], through the codec's decoder
    with every float kept as its bits (wire.decode_solution returns fact as a Python float)"""
    L = wire._lib()
    buf = np.frombuffer(data, np.uint8)
    ptr = buf.ctypes.data if buf.size else None
    ni, nd = C.c_uint64(), C.c_uint64()
    assert L.lfr_wire_decode_solution(ptr, buf.size, C.byref(ni), C.byref(nd), *([None] * 7)) == 0
    I, D = int(ni.value), int(nd.value)
    img_ptr, noff, nlen = np.zeros(I + 1, np.uint64), np.zeros(I, np.uint64), np.zeros(I, np.uint32)
    fact, fi, di, dj = np.zeros(I, np.uint32), np.zeros(D, np.uint32), np.zeros(D, np.uint32), np.zeros(D, np.uint32)
    assert L.lfr_wire_decode_solution(ptr, buf.size, C.byref(ni), C.byref(nd), *[a.ctypes.data for a in
                                      (img_ptr, noff, nlen, fact, fi, di, dj)]) == 0
    out = []
    for i in range(I):
        a, b = int(img_ptr[i]), int(img_ptr[i + 1])
        out.append((data[int(noff[i]): int(noff[i]) + int(nlen[i])], int(fact[i]),
                    list(zip(fi[a:b].tolist(), di[a:b].tolist(), dj[a:b].tolist()))))
    return out


def effective(entries):
    """the last displacement of each feature, in ascending feature"""
    last = {}
    for f, a, b in entries:
        last[f] = (a, b)
    return [(f,) + last[f] for f in sorted(last)]


def carry_model(scene, data):
    """The rule: scene images (name, fact bits, entries) in order, each followed by the winning message's
    entries it lacks; then the other winning messages in file order.  -> [(name, fact bits, entries)]"""
    msgs = messages(data)
    last = {}
    for i, (nm, _, _) in enumerate(msgs):
        last[nm] = i
    names = {nm for nm, _, _ in scene}
    out = []
    for nm, fb, entries in scene:
        have = {f for f, _, _ in entries}
        extra = [e for e in effective(msgs[last[nm]][2]) if e[0] not in have] if nm in last else []
        out.append((nm, fb, list(entries) + extra))
    for i, (nm, fb, entries) in enumerate(msgs):
        if last[nm] == i and nm not in names:
            out.append((nm, fb, effective(entries)))
    return out


def scene_arrays(scene):
    names = [nm.decode("utf-8", errors="surrogateescape") for nm, _, _ in scene]
    fact = np.array([fb for _, fb, _ in scene], np.uint32).view(np.float32)
    img_ptr = np.zeros(len(scene) + 1, np.uint64)
    img_ptr[1:] = np.cumsum([len(e) for _, _, e in scene])
    ent = [e for _, _, es in scene for e in es]
    fi = np.array([e[0] for e in ent], np.uint32)
    di = np.array([e[1] for e in ent], np.uint32).view(np.float32)
    dj = np.array([e[2] for e in ent], np.uint32).view(np.float32)
    return names, fact, img_ptr, fi, di, dj


def encode(scene):
    return wire.encode_solution(*scene_arrays(scene))


def carried(scene, data):
    return wire.encode_solution_carried(*scene_arrays(scene), data)


SPECIAL = [0, 0x80000000, 0x7FC12345, 0xFFA00001, 0x00000001, 0x807FFFFF, f32_bits(0.25), f32_bits(-0.5)]


def random_case(rng, n_scene=6, n_other=3):
    """A scene and a FILE over its names and others: repeated Image messages, repeated features, empty
    messages, feature 0, -0.0, NaN with payloads, denormals, non-UTF-8 names."""
    pool = [b"a.png", b"b.png", b"\xff\xfe.png", b"", b"caf\xc3\xa9.jpg", b"d.png", b"e\x00.png", b"f.png", b"g.png"]
    rng.shuffle(pool)
    scene_names, other = pool[:n_scene], pool[n_scene:n_scene + n_other]

    def val():
        return int(rng.choice(SPECIAL)) if rng.random() < 0.3 else f32_bits(rng.uniform(-0.6, 0.6))

    scene = []
    for nm in scene_names:
        feats = rng.choice(40, size=int(rng.integers(0, 12)), replace=False)
        scene.append((nm, val(), [(int(f), val(), val()) for f in feats]))
    msgs = []
    for _ in range(int(rng.integers(0, 12))):
        nm = [*scene_names, *other][int(rng.integers(0, n_scene + n_other))]
        k = int(rng.integers(0, 10))
        msgs.append(image_bits(nm, [(int(rng.integers(0, 45)), val(), val()) for _ in range(k)], val()))
    return scene, b"".join(msgs)


def as_table(out_bytes):
    """the reader's view: {name: {feature: (di bits, dj bits)}}, the last Image of a name and the last
    displacement of a feature"""
    t = {}
    for nm, _, entries in messages(out_bytes):
        t[nm] = {f: (a, b) for f, a, b in entries}
    return t


# ---------------------------------------------------------------------------------------------------
# the host function against the rule
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(40))
def test_host_function_equals_the_rule(seed):
    rng = np.random.default_rng(seed)
    scene, data = random_case(rng)
    want = carry_model(scene, data)
    got, n = carried(scene, data)
    assert got == encode(want)
    assert n == sum(len(e) for _, _, e in want) - sum(len(e) for _, _, e in scene)
    # the reader's view: the scene's value where the scene has the keypoint, else the file's, else nothing
    table = as_table(got)
    file_t = {}
    for nm, _, entries in messages(data):
        file_t[nm] = {f: (a, b) for f, a, b in entries}
    scene_t = {nm: {f: (a, b) for f, a, b in e} for nm, _, e in scene}
    for nm in set(scene_t) | set(file_t):
        for f in set(scene_t.get(nm, {})) | set(file_t.get(nm, {})):
            want_v = scene_t[nm][f] if f in scene_t.get(nm, {}) else file_t[nm][f]
            assert table[nm][f] == want_v, (nm, f)
    assert all(f in scene_t.get(nm, {}) or f in file_t.get(nm, {}) for nm, t in table.items() for f in t)


def test_worked_example():
    scene = [(b"a.png", f32_bits(2.0), [(3, f32_bits(0.5), 0), (1, f32_bits(0.1), f32_bits(0.2))]),
             (b"b.png", f32_bits(1.0), [(0, f32_bits(0.3), f32_bits(0.3))])]
    data = (image_bits(b"a.png", [(9, f32_bits(0.9), f32_bits(0.9))])              # loses as a whole
            + image_bits(b"z.png", [(4, 1, 2)], f32_bits(3.0))
            + image_bits(b"a.png", [(7, 0x7FC12345, 0x80000000), (3, 5, 5), (2, 0, 0), (7, 6, 6)], f32_bits(8.0))
            + image_bits(b"empty.png", [])
            + image_bits(b"z.png", [(5, 1, 0), (0, 0x80000000, 1)], f32_bits(4.0)))
    want = [(b"a.png", f32_bits(2.0), [(3, f32_bits(0.5), 0), (1, f32_bits(0.1), f32_bits(0.2)), (2, 0, 0), (7, 6, 6)]),
            (b"b.png", f32_bits(1.0), [(0, f32_bits(0.3), f32_bits(0.3))]),
            (b"empty.png", f32_bits(1.0), []),
            (b"z.png", f32_bits(4.0), [(0, 0x80000000, 1), (5, 1, 0)])]
    got, n = carried(scene, data)
    assert got == encode(want) and n == 4
    assert [nm for nm, _, _ in messages(got)] == [b"a.png", b"b.png", b"empty.png", b"z.png"]


def test_apply_solution_reads_the_merged_scene():
    """consumer.apply_solution over the merged output: every keypoint gets the scene's displacement where the
    scene has one, else the file's, else none, at the output image's fact."""
    rng = np.random.default_rng(11)
    for _ in range(10):
        scene, data = random_case(rng)
        got, _ = carried(scene, data)
        names = {nm for nm, _, _ in scene} | {nm for nm, _, _ in messages(data)}
        kp = {nm.decode("utf-8", errors="surrogateescape"): rng.uniform(0, 100, (50, 2)).astype(np.float32) for nm in names}
        with np.errstate(all="ignore"):      # NaN displacements: the same arithmetic on both sides
            applied = consumer.apply_solution(kp, got)
        facts = {nm: fb for nm, fb, _ in carry_model(scene, data)}
        table = as_table(got)
        for nm in names:
            s = nm.decode("utf-8", errors="surrogateescape")
            t = table.get(nm, {})
            fi = np.array(sorted(t), np.int64)
            di = np.array([t[f][0] for f in sorted(t)], np.uint32).view(np.float32)
            dj = np.array([t[f][1] for f in sorted(t)], np.uint32).view(np.float32)
            fact = np.uint32(facts.get(nm, f32_bits(1.0))).view(np.float32)
            with np.errstate(all="ignore"):
                want = consumer.apply_to_keypoints(kp[s], fi, di, dj, fact)
            assert applied[s].tobytes() == want.tobytes(), nm


def test_empty_file_is_the_plain_encoding_and_empty_scene_normalises_the_file():
    rng = np.random.default_rng(5)
    for _ in range(10):
        scene, data = random_case(rng)
        got, n = carried(scene, b"")
        assert got == encode(scene) and n == 0
        got, n = carried([], data)
        want = carry_model([], data)
        assert got == encode(want) and n == sum(len(e) for _, _, e in want)
    assert carried([], b"") == (b"", 0)


def _call(scene, data, out=None, cap=0, n=None, **null):
    L = wire._lib()
    names, fact, img_ptr, fi, di, dj = scene_arrays(scene)
    blob, off = wire._names_blob(names)
    args = dict(img_ptr=img_ptr.ctypes.data, names=blob.ctypes.data, name_off=off.ctypes.data, fact=fact.ctypes.data,
                fi=fi.ctypes.data, di=di.ctypes.data, dj=dj.ctypes.data)
    args.update(null)
    buf = np.frombuffer(data, np.uint8)
    fptr = null.get("file", buf.ctypes.data if buf.size else None)
    return L.lfr_wire_encode_solution_carried(len(names), args["img_ptr"], args["names"], args["name_off"], args["fact"],
                                              args["fi"], args["di"], args["dj"], fptr, buf.size,
                                              out.ctypes.data if out is not None else None, cap, n)


def test_size_protocol():
    scene, data = random_case(np.random.default_rng(2))
    want, n_want = carried(scene, data)
    need = _call(scene, data)
    assert need == len(want) > 0
    out = np.full(need + 8, 0xAB, np.uint8)
    n = C.c_uint64(77)
    assert _call(scene, data, out, need - 1, C.byref(n)) == need and (out == 0xAB).all() and n.value == n_want
    assert _call(scene, data, out, need + 8) == need
    assert out[:need].tobytes() == want and (out[need:] == 0xAB).all()


@pytest.mark.parametrize("bad", [b"\x0a\xff", b"\x0a\x05\x0a\x09abc", b"\x0a\xff\xff\xff\xff\x0f not a protobuf",
                                 image_bits(b"a.png", [(1, 1, 1)])[:-3]])
def test_refuses_malformed_bytes(bad):
    scene = [(b"a.png", f32_bits(1.0), [(1, 0, 0)])]
    out = np.full(64, 0xAB, np.uint8)
    n = C.c_uint64(5)
    assert _call(scene, bad, out, 64, C.byref(n)) == LFR_EINVAL and (out == 0xAB).all() and n.value == 5
    with pytest.raises(wire.ParseError):
        carried(scene, bad)


def test_refuses_repeated_scene_names_and_null_arrays():
    scene = [(b"a.png", f32_bits(1.0), [(1, 0, 0)]), (b"b.png", 0, []), (b"a.png", 0, [(2, 0, 0)])]
    assert _call(scene, b"") == LFR_EINVAL
    with pytest.raises(ValueError):
        carried(scene, b"")
    scene = scene[:2]
    data = image_bits(b"a.png", [(1, 1, 1)])
    assert _call(scene, data) > 0
    for k in ("img_ptr", "names", "name_off", "fact", "fi", "di", "dj", "file"):
        assert _call(scene, data, **{k: None}) == LFR_EINVAL, k


# ---------------------------------------------------------------------------------------------------
# the incremental scenario through the native executable on the CPU checker and the Python launcher
# ---------------------------------------------------------------------------------------------------
SCENE = dict(cfg="cfg2", scale=0.1, seed=3)
NEW = slice(8, 11)            # images added after solution A


def split_pairs(ms, new_names):
    """(old pairs, new pairs): the pairs that touch none of `new_names`, and those that touch one."""
    new = set(new_names)
    touch = np.array([ms.image_names[a] in new or ms.image_names[b] in new
                      for a, b in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist())], bool)
    return ms.select_pairs(np.nonzero(~touch)[0]), ms.select_pairs(np.nonzero(touch)[0])


@pytest.fixture(scope="module")
def incremental(checker_exe, tmp_path_factory):  # noqa: F811
    """(MatchSet, old pairs path, new pairs path, A's path and bytes): A solves the old pairs."""
    d = tmp_path_factory.mktemp("carry")
    ms = synth.generate(SCENE["cfg"], scale=SCENE["scale"], seed=SCENE["seed"])
    old, new = split_pairs(ms, ms.image_names[NEW])
    m_old, m_new, a = d / "old.pb", d / "new.pb", d / "a.pb"
    m_old.write_bytes(wire.encode_matching_file(old))
    m_new.write_bytes(wire.encode_matching_file(new))
    r = run(checker_exe, ["--matches_file", str(m_old), "--output_file", str(a)])
    assert r.returncode == 0, r.stderr
    return ms, m_old, m_new, a, a.read_bytes()


def every_entry_comes_back(a_bytes, out_bytes):
    got = as_table(out_bytes)
    n = 0
    for nm, _, entries in messages(a_bytes):
        for f, x, y in effective(entries):
            assert got[nm][f] == (x, y), (nm, f)
            n += 1
    return n


def untimed_lines(r):
    return [l for l in r.stdout.decode().splitlines() if " time:" not in l]


def python_host(oracle, matches, extra, a_bytes, monkeypatch):
    """The Python drop-in's path (cli.main) on the host route with the checker as the solve: refine() with the
    options of `extra`, then wire.encode_solution_carried on its assembly."""
    from lfr_b200.solver import refine
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    ms = wire.read_matching_file(str(matches))
    opt = {k: [v for f, v in zip(extra, extra[1:]) if f == k] for k in ("--fixed_images", "--banned_images")}
    opts = oracle.default_options(n_threads=4)
    _, _, _, sol = refine(ms, opt["--banned_images"], solve_fn=lambda q, x=None: oracle.solve(q, opts, positions=x),
                          fixed_images=opt["--fixed_images"], initial_solution=a_bytes,
                          keep_initial_solution="--keep_initial_solution" in extra)
    return wire.encode_solution_carried(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj, a_bytes)[0]


VARIANTS = {"keep": ["--keep_initial_solution"], "start": [], "keep+fixed": ["--keep_initial_solution", "--fixed_images", 9],
            "keep+banned": ["--keep_initial_solution", "--banned_images", 2]}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_incremental_carry_through_both_hosts(checker_exe, oracle, incremental, tmp_path, monkeypatch, variant):  # noqa: F811
    ms, m_old, m_new, a, A = incremental
    extra = [ms.image_names[x] if isinstance(x, int) else x for x in VARIANTS[variant]]
    base = ["--matches_file", str(m_new), "--initial_solution", str(a)] + extra
    o, o0 = tmp_path / "o.pb", tmp_path / "o0.pb"
    r = run(checker_exe, base + ["--output_file", str(o), "--carry_initial_solution"])
    assert r.returncode == 0, r.stderr
    r0 = run(checker_exe, base + ["--output_file", str(o0)])
    assert r0.returncode == 0, r0.stderr
    B, B0 = o.read_bytes(), o0.read_bytes()
    assert python_host(oracle, m_new, extra, A, monkeypatch) == B        # both hosts write the same bytes
    assert untimed_lines(r) == untimed_lines(r0)                          # the stdout does not change
    # the scene's output is the run without the flag's, entry for entry, and the rest is A's
    scene = messages(B0)
    assert B == encode(carry_model(scene, A))
    out = messages(B)
    for (nm, fb, entries), (nm2, fb2, entries2) in zip(scene, out):
        assert (nm, fb) == (nm2, fb2) and entries2[:len(entries)] == entries
    if variant == "start":
        # without keep, A's entries of the scene's keypoints are refined again: the scene's values win
        t = as_table(B)
        assert all(t[nm][f] == (x, y) for nm, _, e in scene for f, x, y in e)
    else:
        assert every_entry_comes_back(A, B) > 0
    names_b = [nm for nm, _, _ in out]
    assert len(names_b) == len(set(names_b))
    assert {nm for nm, _, _ in messages(A)} | {nm for nm, _, _ in scene} == set(names_b)
    if variant == "keep+banned":
        banned = ms.image_names[2].encode()
        assert banned not in {nm for nm, _, _ in scene}
        assert [e for nm, _, e in out if nm == banned] == [effective(e) for nm, _, e in messages(A) if nm == banned]


# ---------------------------------------------------------------------------------------------------
# the command line
# ---------------------------------------------------------------------------------------------------
def _both_hosts(checker_exe, args, env=None):  # noqa: F811
    a = subprocess.run([checker_exe] + args, capture_output=True, env=env)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=dict(env or os.environ, LFR_SOLVE_PYTHON="1"))
    return a, b


def test_carry_without_initial_solution_is_refused_first(checker_exe, tmp_path):  # noqa: F811
    m = os.path.join(GOLD, "tiny_matches.pb")
    o = tmp_path / "o.pb"
    for argv, err in ((["--matches_file", m, "--output_file", str(o), "--carry_initial_solution"], CARRY_ERROR),
                      (["--c", "--matches_file", m, "--output_file", str(o), "--initial_solution="], CARRY_ERROR),
                      (["--carry", "--keep", "--matches_file", m, "--output_file", str(o)], KEEP_ERROR)):
        a, b = _both_hosts(checker_exe, argv)
        for r in (a, b):
            assert (r.returncode, r.stdout, r.stderr) == (2, b"", err)
    assert not o.exists()


def test_carry_takes_no_value(checker_exe, tmp_path):  # noqa: F811
    m = os.path.join(GOLD, "tiny_matches.pb")
    for flag in ("--carry_initial_solution=x", "--carry=", "--c=1"):
        a, b = _both_hosts(checker_exe, ["--matches_file", m, "--output_file", str(tmp_path / "o.pb"), "--initial_solution",
                                         m, flag])
        for r in (a, b):
            assert r.returncode == 1 and r.stdout == b""
            assert r.stderr == (b"ERROR: option '--carry_initial_solution' does not take any arguments\n\n" + USAGE.encode())


def test_prefixes_and_help(checker_exe, incremental, tmp_path):  # noqa: F811
    """--c and --carry are --carry_initial_solution; --k, --fix, --init and --m keep their meaning; --help does
    not list the new option."""
    ms, m_old, m_new, a, A = incremental
    outs = []
    for i, flag in enumerate(["--carry_initial_solution", "--carry", "--c"]):
        o = tmp_path / ("o%d.pb" % i)
        r = run(checker_exe, ["--m", str(m_new), "--output_file", str(o), "--init", str(a), flag, "--k",
                              "--fix", ms.image_names[9]])
        assert r.returncode == 0, r.stderr
        outs.append(o.read_bytes())
    assert outs[0] == outs[1] == outs[2]
    o = tmp_path / "full.pb"
    r = run(checker_exe, ["--matches_file", str(m_new), "--output_file", str(o), "--initial_solution", str(a),
                          "--keep_initial_solution", "--carry_initial_solution", "--fixed_images", ms.image_names[9]])
    assert r.returncode == 0 and o.read_bytes() == outs[0]
    a_, b_ = _both_hosts(checker_exe, ["--help"])
    for r in (a_, b_):
        assert r.returncode == 0 and r.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
        assert b"carry" not in r.stdout


def test_torchrun_ranks_refuse_a_carried_solution(incremental, tmp_path):
    ms, m_old, m_new, a, A = incremental
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", str(m_new), "--output_file", str(tmp_path / "o.pb"),
                        "--initial_solution", str(a), "--carry_initial_solution"], capture_output=True, env=env)
    assert r.returncode == 2
    assert r.stderr == b"ERROR: --initial_solution: torchrun ranks start from zeros; use --gpus N\n"
    assert not (tmp_path / "o.pb").exists()
