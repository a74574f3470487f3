"""--query_images on the GPU with sub-scenes past the 64-bit image mask (tests/subscene_cases.py).

The device stage with image groups against the host stage, bitwise, at every Kruskal window and with both
cuts; the native drop-in on every graph-stage route against the CPU checker's bytes and every query's own
run, and on a batch the device route decodes on the GPU; the 65 535-id limit on the device; and
lfr_plan_encode_solution_images() against the plain encoder's bytes with the unflagged images' messages
left out."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import subscene_cases as S
from lfr_b200 import wire
from lfr_b200.capi import DBG_DEVICE_CUT, Plan
from lfr_b200.graph import host_input_arrays
from lfr_b200.wire import _names_blob
from test_gpu_graph_stage import ARRAYS, COUNTS
from test_gpu_query_images import ROUTES, _run
from test_native_exe import checker_exe, product_exe  # noqa: F401
from test_query_images import check_batch, messages, own_matches, own_runs, stdout_values
from test_query_images_adversarial import query_args
from test_ref_solve import untimed

pytestmark = pytest.mark.gpu

LFR_EINVAL = -1


def _stage_input(case):
    sub, group = S.grouped(case)
    return host_input_arrays(sub, (), group)[1], len(sub.image_names), sub


# ---------------------------------------------------------------------------------------------------
# the device stage
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("device_cut", [False, True], ids=["host_cut", "device_cut"])
@pytest.mark.parametrize("case", S.STAGED)
def test_device_stage_equals_the_host_stage_at_every_window(b200, case, device_cut, monkeypatch):
    want, sz, _, _ = S.stage(case)
    arrs, n, _ = _stage_input(case)
    M = arrs["feat1"].shape[0]
    opts = b200.default_options(debug_flags=DBG_DEVICE_CUT) if device_cut else None
    for window in (None, 1, 2, 31, 32, 33, M + 1):
        if window is None:
            monkeypatch.delenv("LFR_KRUSKAL_WINDOW", raising=False)
        else:
            monkeypatch.setenv("LFR_KRUSKAL_WINDOW", str(window))
        plan = Plan.from_matches(b200, arrs, options=opts, n_images=n)
        try:
            got = plan.export_graph()
            for k in COUNTS:
                assert plan.sizes[k] == sz[k], (window, k, plan.sizes[k], sz[k])
        finally:
            plan.close()
        for k in ARRAYS:
            assert got[k].dtype == want[k].dtype and got[k].tobytes() == want[k].tobytes(), (window, k)


def test_device_stage_takes_65535_ids_and_refuses_65536(b200):
    arrs, n, _ = _stage_input("ids_65535")
    plan = Plan.from_matches(b200, arrs, n_images=n)
    assert n == 65535 and plan.sizes["n_nodes"] == S.stage("ids_65535")[1]["n_nodes"]
    plan.close()
    batch, queries, banned = S.make("ids_65536")
    sub, group = batch.query_subscenes(queries, [banned])
    _, arrs = host_input_arrays(sub, (), group)
    with pytest.raises(RuntimeError, match=r"\(%d\)" % S.LFR_EUNSUPPORTED):
        Plan.from_matches(b200, arrs, n_images=len(sub.image_names))
    assert not b200.graph_stage_on_device(arrs, len(sub.image_names))


# ---------------------------------------------------------------------------------------------------
# the drop-in
# ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def checked(tmp_path_factory, checker_exe):  # noqa: F811
    """case -> (directory with batch.pb, the checker's batch run, the own runs on the checker)."""
    cache = {}

    def get(case):
        if case not in cache:
            d = tmp_path_factory.mktemp(case)
            batch, queries, banned = S.make(case)
            wire.write_matching_file(batch, str(d / "batch.pb"))
            r = subprocess.run([checker_exe] + query_args(d, "batch.pb", d / "checker.pb", queries, banned), capture_output=True)
            assert r.returncode == 0, r.stderr
            cache[case] = (d, r, own_runs(checker_exe, d, batch, queries, [], banned))
        return cache[case]
    return get


@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("case", S.SOLVED)
def test_drop_in_on_every_route_equals_the_checker_and_the_own_runs(checked, product_exe, case, route):  # noqa: F811
    d, rc, own = checked(case)
    batch, queries, banned = S.make(case)
    o = d / ("gpu_%s.pb" % route)
    r = _run(query_args(d, "batch.pb", o, queries, banned), ROUTES[route])
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == (d / "checker.pb").read_bytes()
    assert untimed(r.stdout.decode()) == untimed(rc.stdout.decode())
    check_batch(o.read_bytes(), r.stdout.decode(), own, queries)


def test_batch_decoded_on_the_gpu(b200, tmp_path, product_exe):  # noqa: F811
    batch, queries, banned = S.make("decoded_on_device")
    assert b200.lib.lfr_wire_decode_on_device(batch.n_matches) == 1
    wire.write_matching_file(batch, str(tmp_path / "batch.pb"))
    outs = {}
    for route, env in (("auto", {}), ("host", ROUTES["host"]), ("device_cut", ROUTES["device_cut"])):
        o = tmp_path / ("%s.pb" % route)
        r = _run(query_args(tmp_path, "batch.pb", o, queries, banned), env)
        assert r.returncode == 0, r.stderr
        outs[route] = (o.read_bytes(), untimed(r.stdout.decode()), r.stdout.decode())
    assert outs["auto"][:2] == outs["host"][:2] == outs["device_cut"][:2]
    own = {}
    for q in queries:
        mq = tmp_path / ("own_%s.pb" % q)
        wire.write_matching_file(own_matches(batch, q, [banned]), str(mq))
        oq = tmp_path / ("own_%s_out.pb" % q)
        rq = _run(["--matches_file", str(mq), "--output_file", str(oq), "--banned_images", banned], {})
        assert rq.returncode == 0, rq.stderr
        mine = [m for nm, m in messages(oq.read_bytes()) if nm == q]
        own[q] = (mine[0] if mine else None, stdout_values(rq.stdout.decode()))
    check_batch(outs["auto"][0], outs["auto"][2], own, queries)


# ---------------------------------------------------------------------------------------------------
# lfr_plan_encode_solution_images
# ---------------------------------------------------------------------------------------------------
def _encode_images(b200, plan, names, fact, written, cap=None, out=None):
    f = b200.lib.lfr_plan_encode_solution_images
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_uint64, C.POINTER(C.c_uint64)]
    f.restype = C.c_int64
    blob, off = _names_blob(list(names))
    fact = np.ascontiguousarray(fact, np.float32)
    w = None if written is None else np.ascontiguousarray(written, np.uint8)
    n_out = C.c_uint64(12345)
    args = (plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact.ctypes.data,
            None if w is None else w.ctypes.data)
    if out is None:
        need = f(*args, None, 0, C.byref(n_out))
        if need < 0:
            return need, None, None
        buf = np.empty(max(int(need), 1), np.uint8)
        got = f(*args, buf.ctypes.data, int(need), C.byref(n_out))
        assert got == need
        return int(need), buf[:need].tobytes(), int(n_out.value)
    got = f(*args, out.ctypes.data, int(cap), C.byref(n_out))
    return int(got), None, int(n_out.value)


def _expected(full, node_image, written):
    """The plain encoding with the Image messages of unflagged ids left out: the messages are in order of
    each id's lowest node."""
    _, first = np.unique(node_image, return_index=True)
    ids = np.unique(node_image)[np.argsort(first, kind="stable")]
    msgs = messages(full)
    assert len(msgs) == ids.shape[0]
    return b"".join(m for i, (_, m) in zip(ids.tolist(), msgs) if written[i])


@pytest.mark.parametrize("case", ["bitset129", "caps", "wide1101"])
def test_encode_solution_images_leaves_out_the_unflagged_images(b200, case):
    arrs, n, sub = _stage_input(case)
    plan = Plan.from_matches(b200, arrs, n_images=n)
    try:
        plan.solve()
        node_image = plan.export_graph()["node_image"].astype(np.int64)
        extra = 3                                               # ids past the plan's: names, no nodes
        names = list(sub.image_names) + ["extra_%d.png" % i for i in range(extra)]
        fact = np.random.default_rng(3).uniform(0.5, 2.0, len(names)).astype(np.float32)
        full, n_full = plan.encode_solution(names, fact)
        assert full
        n_ids = len(names)
        has_node = np.zeros(n_ids, bool)
        has_node[node_image] = True
        rng = np.random.default_rng(11)
        db_name = [nm for nm in sub.image_names if sub.image_names.count(nm) > 1]
        patterns = {
            "all": np.ones(n_ids, np.uint8), "none": np.zeros(n_ids, np.uint8),
            "alternating": (np.arange(n_ids) % 2).astype(np.uint8),
            "random": (rng.random(n_ids) < 0.4).astype(np.uint8),
            "no_nodes": (~has_node).astype(np.uint8),
        }
        if db_name:    # every copy of one database image (they share a name), and one copy alone
            copies = np.array([nm == db_name[0] for nm in names])
            patterns["copies"] = copies.astype(np.uint8)
            one = np.zeros(n_ids, np.uint8)
            one[np.nonzero(copies)[0][-1]] = 1
            patterns["one_copy"] = one
        assert (~has_node).any()
        for pname, w in patterns.items():
            need, got, n_out = _encode_images(b200, plan, names, fact, w)
            assert got == _expected(full, node_image, w), pname
            assert n_out == n_full, pname
            if need:                                             # one byte short: nothing written
                canary = np.full(need + 16, 0xA5, np.uint8)
                r, _, _ = _encode_images(b200, plan, names, fact, w, cap=need - 1, out=canary)
                assert r == need and (canary == 0xA5).all(), pname
        assert _encode_images(b200, plan, names, fact, None)[0] == LFR_EINVAL
    finally:
        plan.close()
