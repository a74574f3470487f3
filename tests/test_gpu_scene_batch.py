"""--additional_scenes on the GPU: both drop-in hosts on every graph-stage route against every scene's own run
on the CPU checker, a batch the device route decodes on the GPU, and lfr_plan_encode_solution_groups()
against lfr_plan_encode_solution_images() with each group's mask."""
import numpy as np
import pytest

import test_scene_batch as tsb
from lfr_b200 import synth, wire
from lfr_b200.graph import host_input_arrays
from lfr_b200.matchset import MatchSet
from lfr_b200.capi import Plan
from test_gpu_query_images import ROUTES, _run
from test_gpu_query_images_adversarial import LFR_EINVAL, _encode_images
from test_native_exe import product_exe  # noqa: F401
from test_fixed_images import checker_exe  # noqa: F401
from test_ref_solve import untimed
from test_scene_batch import batch, own_runs  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def checker_batch(batch, checker_exe):  # noqa: F811
    d, scenes = batch
    args, outs = tsb.batch_args(d, scenes, "checker")
    r = tsb.run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    return r


@pytest.mark.parametrize("python", [False, True], ids=["native", "python"])
@pytest.mark.parametrize("route", sorted(ROUTES))
def test_drop_in_on_every_route_writes_every_scenes_own_run(batch, own_runs, checker_batch, product_exe, route,  # noqa: F811
                                                            python):
    d, scenes = batch
    args, outs = tsb.batch_args(d, scenes, "%s_%d" % (route, python))
    r = _run(args, ROUTES[route], python=python)
    assert r.returncode == 0, r.stderr
    tsb.check_batch(outs, r.stdout.decode(), own_runs)
    assert untimed(r.stdout.decode()) == untimed(checker_batch.stdout.decode())


def test_batch_decoded_on_the_gpu(b200, tmp_path, product_exe):  # noqa: F811
    sets, total = [], 0
    while total < 300000:
        ms = synth.generate("cfg2", scale=0.25, seed=50 + len(sets))
        ms.image_names = ["%04d.png" % i for i in range(len(ms.image_names))]    # every scene reuses the names
        sets.append(ms)
        total += ms.n_matches
    assert total >= 262144 and b200.lib.lfr_wire_decode_on_device(total) == 1
    assert all(b200.lib.lfr_wire_decode_on_device(ms.n_matches) == 0 for ms in sets)
    paths = []
    for k, ms in enumerate(sets):
        wire.write_matching_file(ms, str(tmp_path / ("s%d.pb" % k)))
        paths.append(str(tmp_path / ("s%d.pb" % k)))
    own = []
    for k, m in enumerate(paths):
        r = _run(["--matches_file", m, "--output_file", m + ".own"], {})
        assert r.returncode == 0, r.stderr
        own.append((open(m + ".own", "rb").read(), tsb.stdout_values(r.stdout.decode())))
    for route, env in (("auto", {}), ("host", ROUTES["host"]), ("device_cut", ROUTES["device_cut"])):
        outs = [m + "." + route for m in paths]
        lst = tsb.scene_list(tmp_path / "l.txt", list(zip(paths[1:], outs[1:])))
        r = _run(["--matches_file", paths[0], "--output_file", outs[0], "--additional_scenes", str(lst)], env)
        assert r.returncode == 0, r.stderr
        tsb.check_batch(outs, r.stdout.decode(), own)


# ---------------------------------------------------------------------------------------------------
# lfr_plan_encode_solution_groups
# ---------------------------------------------------------------------------------------------------
def _encode_groups(b200, plan, names, fact, group, n_groups, cap=None, out=None):
    f = b200.lib.lfr_plan_encode_solution_groups
    blob, off = wire._names_blob(list(names))
    fact = np.ascontiguousarray(fact, np.float32)
    group = np.ascontiguousarray(group, np.uint32)
    goff = np.full(n_groups + 1, 77, np.uint64)
    n_out = np.full(max(n_groups, 1), 77, np.uint64)
    args = (plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact.ctypes.data, group.ctypes.data, n_groups)
    if out is None:
        need = f(*args, None, 0, goff.ctypes.data, n_out.ctypes.data)
        if need < 0:
            return int(need), None, None, None
        buf = np.empty(max(int(need), 1), np.uint8)
        assert f(*args, buf.ctypes.data, int(need), goff.ctypes.data, n_out.ctypes.data) == need
        return int(need), buf[:need].tobytes(), goff, n_out[:n_groups]
    got = f(*args, out.ctypes.data, int(cap), goff.ctypes.data, n_out.ctypes.data)
    return int(got), None, goff, n_out[:n_groups]


def _scene_plan(b200, positions=None):
    """A plan of six scenes (three HPatches-shaped, the hub scene, one all banned, a cfg2 scene), with ids past
    the plan's: a group of images without nodes and an empty group."""
    sets = [tsb.hpatches_scene(200 + k) for k in range(3)] + [tsb.hub_scene(), tsb.star_scene(),
                                                                 synth.generate("cfg2", scale=0.05, seed=4)]
    ms, group = MatchSet.join_scenes(sets, tsb.BANNED)
    _, arrs = host_input_arrays(ms, (), group)
    arrs["image_group"] = group
    plan = Plan.from_matches(b200, arrs, n_images=len(ms.image_names), positions=positions)
    names = list(ms.image_names) + ["extra_%d.png" % i for i in range(3)]
    group = np.concatenate([group, np.full(3, len(sets), np.uint32)])   # group 6: images without a node
    return plan, names, group, len(sets) + 2                              # group 7: no image at all


def _check_groups(b200, plan, names, group, n_groups, pos=None):
    """Solved when `pos` (the plan's start positions) is not given."""
    try:
        if pos is None:
            plan.solve()
            pos, _ = plan.download()
        node_image = plan.export_graph()["node_image"].astype(np.int64)
        fact = np.random.default_rng(5).uniform(0.5, 2.0, len(names)).astype(np.float32)
        need, data, goff, n_out = _encode_groups(b200, plan, names, fact, group, n_groups)
        assert goff[0] == 0 and goff[-1] == need == len(data) and (np.diff(goff.astype(np.int64)) >= 0).all()
        p = np.asarray(pos, np.float64).reshape(-1, 2)
        outside = (np.abs(p[:, 0]) > 0.5) | (np.abs(p[:, 1]) > 0.5)
        for g in range(n_groups):
            _, want, _ = _encode_images(b200, plan, names, fact, (group == g).astype(np.uint8))[:3]
            assert data[int(goff[g]):int(goff[g + 1])] == want, g
            assert int(n_out[g]) == int(outside[group[node_image] == g].sum()), g
        assert goff[n_groups - 1] == goff[n_groups - 2] == goff[n_groups] and n_out[-2:].tolist() == [0, 0]
        # one byte short: the size, and nothing written
        canary = np.full(need + 16, 0xA5, np.uint8)
        r, _, _, _ = _encode_groups(b200, plan, names, fact, group, n_groups, cap=need - 1, out=canary)
        assert r == need and (canary == 0xA5).all()
        # a group id past n_groups, NULL arrays
        assert _encode_groups(b200, plan, names, fact, group, n_groups - 3)[0] == LFR_EINVAL
        f = b200.lib.lfr_plan_encode_solution_groups
        blob, off = wire._names_blob(names)
        goff = np.zeros(n_groups + 1, np.uint64)
        g32 = np.ascontiguousarray(group, np.uint32)
        assert f(plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact.ctypes.data, None, n_groups, None, 0,
                 goff.ctypes.data, goff.ctypes.data) == LFR_EINVAL
        assert f(plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact.ctypes.data, g32.ctypes.data,
                 n_groups, None, 0, None, goff.ctypes.data) == LFR_EINVAL
        assert f(plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact.ctypes.data, g32.ctypes.data,
                 n_groups, None, 0, goff.ctypes.data, None) == LFR_EINVAL
    finally:
        plan.close()


def test_encode_groups_equals_the_masked_encoder(b200):
    plan, names, group, n_groups = _scene_plan(b200)
    _check_groups(b200, plan, names, group, n_groups)


def test_encode_groups_keeps_nan_payloads(b200):
    """Start positions that reach the encoder unsolved: NaN payloads of both signs, infinities, past 0.5."""
    plan, _, _, _ = _scene_plan(b200)
    n = plan.n_nodes
    plan.close()
    rng = np.random.default_rng(9)
    bits = rng.integers(0, 2 ** 52, 2 * n, dtype=np.uint64) | np.uint64(0x7FF0000000000001)
    bits[::3] |= np.uint64(1 << 63)
    pos = bits.view(np.float64).copy()
    pos[1::4] = rng.uniform(-1, 1, pos[1::4].shape[0])
    pos[2::8] = np.inf
    plan, names, group, n_groups = _scene_plan(b200, positions=pos.reshape(n, 2))
    _check_groups(b200, plan, names, group, n_groups, pos=pos)


def test_plan_encode_solution_groups_binding(b200, own_runs, batch):  # noqa: F811
    """Plan.encode_solution_groups on the test batch: every scene's own run, from one device encode."""
    d, scenes = batch
    sets = [wire.read_matching_file(m) if wire.matches_files(m) else MatchSet.empty() for m, _, _ in scenes]
    ms, group = MatchSet.join_scenes(sets, tsb.BANNED)
    _, arrs = host_input_arrays(ms, (), group)
    arrs["image_group"] = group
    plan = Plan.from_matches(b200, arrs, n_images=len(ms.image_names))
    try:
        plan.solve()
        data, n_out = plan.encode_solution_groups(ms.image_names, _first_facts(ms), group, len(sets))
    finally:
        plan.close()
    assert data == [b for b, _ in own_runs]
    assert n_out == [v.get("# points with at least one coordinate > 0.5", 0) for _, v in own_runs]


def _first_facts(ms):
    """The first fact seen of every image id, as the hosts take it."""
    fact = np.zeros(len(ms.image_names), np.float32)
    seen = np.zeros(len(ms.image_names), bool)
    for p in range(ms.n_pairs):
        for img, f in ((int(ms.pair_img1[p]), ms.pair_fact1[p]), (int(ms.pair_img2[p]), ms.pair_fact2[p])):
            if not seen[img]:
                seen[img], fact[img] = True, f
    return fact
