"""--task_stream on the GPU: the product binary and the Python host run streams whose tasks take both graph-stage
routes, and every task must be its own one-shot run (files, untimed stdout, stderr, exit code).  The harness is
tests/test_task_stream.py's: each line is written after the previous completion line was read."""
import os
import shutil
import subprocess
import sys

import pytest

from lfr_b200 import synth, wire
from test_drop_in_device_stage import solution_close
from test_native_exe import PRODUCT, checker_exe, product_exe  # noqa: F401
from test_query_images import localization_scene
from test_ref_solve import GOLD, LAUNCHER
from test_task_stream import TIMEOUT, Stream, grown, stream_and_one_shots

pytestmark = pytest.mark.gpu

HOSTS = ["native", "python"]


def host(name):
    if name == "native":
        return [PRODUCT], {}
    return [sys.executable, LAUNCHER], {"LFR_SOLVE_PYTHON": "1"}


def env_of(extra, stage=None):
    env = {k: v for k, v in os.environ.items() if k not in ("LFR_GRAPH_STAGE", "RANK", "WORLD_SIZE", "LOCAL_RANK")}
    env.update(extra)
    if stage:
        env["LFR_GRAPH_STAGE"] = stage
    return env


@pytest.fixture(scope="module")
def routes_dir(tmp_path_factory):
    """The goldens (host route under the size rule), a cfg2-scale scene (device route, decoded on the host) and a
    cfg4 scene past the GPU decoder's 262 144 matches (device route, decoded on the GPU)."""
    d = tmp_path_factory.mktemp("gpu_stream")
    for name in ("tiny", "fountain_2pct"):
        shutil.copy(os.path.join(GOLD, name + "_matches.pb"), d / (name + ".pb"))
    dev = synth.generate("cfg2", scale=0.25, seed=11)
    big = synth.generate("cfg4", scale=0.45, seed=7)
    assert 2 * dev.n_matches >= 32768 and big.n_matches >= 262144
    wire.write_matching_file(dev, str(d / "dev.pb"))
    wire.write_matching_file(big, str(d / "big.pb"))
    return d


ROUTE_LINES = [b"--matches_file\ttiny.pb\t--output_file\ttiny.out",
               b"--matches_file\tdev.pb\t--output_file\tdev.out\t--record_file\tdev.rec",
               b"--matches_file\tmissing dir/x.pb\t--output_file\tnone/x.out",                 # exit 255: unwritable
               b"--matches_file\tbig.pb\t--output_file\tbig.out",
               b"--matches_file\tfountain_2pct.pb\t--output_file\tfountain.out",
               b"--matches_file\tdev.pb\t--output_file\tdev2.out\t--initial_solution\tdev.out\t--update_initial_solution"
               b"\t--earlier_record_file\tdev.rec"]


@pytest.mark.parametrize("stage", [None, "host", "device"])
@pytest.mark.parametrize("name", HOSTS)
def test_gpu_routes_mixed_in_one_process(product_exe, checker_exe, routes_dir, tmp_path, name, stage):  # noqa: F811
    cmd, extra = host(name)
    env = env_of(extra, stage)
    streamed, one_shot = stream_and_one_shots(cmd, env, str(routes_dir), ROUTE_LINES, tmp_path)
    for k, (a, b) in enumerate(zip(streamed, one_shot)):
        assert a == b, (k, ROUTE_LINES[k], a[:3], b[:3])
    assert [c for c, _, _, _ in streamed] == [0, 0, 255, 0, 0, 0]
    if name != "native" or stage is not None:
        return
    # the checker's one-shot runs (the host-route goldens and the cfg2 scene): the same solution within the solve's
    # tolerance
    files = streamed[-1][3]
    for k in (0, 1, 4):
        args = [a.decode() for a in ROUTE_LINES[k].split(b"\t")]
        out = args[args.index("--output_file") + 1]
        r = subprocess.run([checker_exe] + args[:args.index("--output_file") + 1] + [str(tmp_path / "c.out")],
                           cwd=routes_dir, capture_output=True, timeout=TIMEOUT)
        assert r.returncode == 0, r.stderr
        assert solution_close(files[out], (tmp_path / "c.out").read_bytes()), out


@pytest.mark.parametrize("name", HOSTS)
def test_gpu_chain_queries_and_versioned_scenes(product_exe, tmp_path, name):  # noqa: F811
    d = tmp_path / "w"
    d.mkdir()
    ms = synth.generate("cfg2", scale=0.25, seed=4)
    lines = []
    for k in range(3, 8):
        (d / ("m%d.pb" % k)).write_bytes(wire.encode_matching_file(grown(ms, k)))
        line = b"--matches_file\tm%d.pb\t--output_file\ts%d.pb\t--record_file\tr%d.rec" % (k, k, k)
        if k > 3:
            line += b"\t--initial_solution\ts%d.pb\t--update_initial_solution\t--earlier_record_file\tr%d.rec" % (k - 1, k - 1)
        lines.append(line)
    (d / "versioned.txt").write_bytes(b"m6.pb\tv1.out\ts5.pb\tr5.rec\tv1.rec\nm4.pb\tv2.out\t\t\t\n")
    lines.append(b"--matches_file\tm7.pb\t--output_file\tv0.out\t--initial_solution\ts6.pb\t--update_initial_solution"
                 b"\t--earlier_record_file\tr6.rec\t--record_file\tv0.rec\t--versioned_scenes\tversioned.txt")
    # localization: one task per query, against the --query_images batch
    _, batch, queries, _ = localization_scene()
    queries = [q for q in queries if q not in ("nomatch.png", "absent.png")]   # the queries with matches
    (d / "q.pb").write_bytes(wire.encode_matching_file(batch))
    for k, q in enumerate(queries):
        lines.append(b"--matches_file\tq.pb\t--output_file\tq%d.out\t--query_images\t%s" % (k, q.encode()))
    cmd, extra = host(name)
    streamed, one_shot = stream_and_one_shots(cmd, env_of(extra, "device"), str(d), lines, tmp_path)
    for k, (a, b) in enumerate(zip(streamed, one_shot)):
        assert a == b, (k, lines[k], a[:3], b[:3])
    codes = [c for c, _, _, _ in streamed]
    assert codes == [0] * len(lines), (codes, [e for _, _, e, _ in streamed if e])
    files = streamed[-1][3]
    assert all(files["s%d.pb" % k] for k in range(3, 8)) and files["v1.out"] and files["v1.rec"]
    args = ["--matches_file", "q.pb", "--output_file", "batch.out"]
    for q in queries:
        args += ["--query_images", q]
    r = subprocess.run(cmd + args, cwd=d, env=env_of(extra, "device"), capture_output=True, timeout=TIMEOUT)
    assert r.returncode == 0, r.stderr
    per_image = {m[0]: m for m in wire.decode_solution((d / "batch.out").read_bytes())}
    for k, q in enumerate(queries):
        own = wire.decode_solution(files["q%d.out" % k])
        for m in own:
            want = per_image[m[0]]
            assert m[0] == want[0] and m[1] == want[1] and all((x == y).all() for x, y in zip(m[2:], want[2:])), q


def _device_mib(pid):
    try:
        out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout
    except (OSError, subprocess.TimeoutExpired):
        return None
    for line in out.splitlines():
        f = [x.strip() for x in line.split(",")]
        if len(f) == 2 and f[0] == str(pid):
            return f[1]
    return None


def test_gpu_device_memory_is_flat_over_tasks(product_exe, routes_dir, tmp_path):  # noqa: F811
    if shutil.which("nvidia-smi") is None:
        pytest.skip("nvidia-smi is absent")
    work = tmp_path / "w"
    shutil.copytree(routes_dir, work)
    s = Stream([PRODUCT], str(work), env_of({}), tmp_path / "err")
    used = {}
    try:
        for k in range(30):
            code, _, err = s.task(b"--matches_file\tbig.pb\t--output_file\tbig.out\t--record_file\tbig.rec")
            assert code == 0, err
            if k + 1 in (3, 30):
                used[k + 1] = _device_mib(s.p.pid)
        assert s.close() == 0
    finally:
        s.kill()
    if used[3] is None:
        pytest.skip("nvidia-smi lists no process of this container")
    assert used[3] == used[30], used
