"""--task_stream FILE: one process runs a stream of tasks, each line of FILE one task (CPU).

Each task must do what the same host does when run once with the line's argument vector: the same files, the same
stdout but for the values of the timed lines, the same stderr and the same exit code, and `# task K: exit C` after
it.  The native host is lfr_solve_main.cc linked against the CPU checker; the Python host is lfr_b200/cli.py with the
solve swapped for the checker, stream and one-shot runs alike.  Every stream here is fed through a pipe one line at
a time: line K is written only after `# task K-1:` was read, and the working directory is read between tasks, so
every task's files, stdout and stderr are its own.  Every wait is bounded and every child is killed in a `finally`."""
import os
import select
import shutil
import subprocess
import sys
import time

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import USAGE
from test_native_exe import checker_exe  # noqa: F401
from test_ref_solve import GOLD, LAUNCHER

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT = 120

# the Python host with the checker as the solve (as tests/test_cli.py drives cli.main in-process)
PYTHON_HOST = """import os, sys
sys.path[:0] = [%r, %r]
from oracle_util import load_oracle
import lfr_b200.solver as solver
orc = load_oracle()
opts = orc.default_options(n_threads=4)
plain = solver.solve_problem
solver.solve_problem = lambda p, options=None, positions=None: (
    plain(p) if p.graph.n_nodes == 0 else orc.solve(p, opts, positions=positions))
from lfr_b200.cli import main
raise SystemExit(main())
""" % (ROOT, os.path.join(ROOT, "tests"))


class Stream:
    """A `--task_stream /dev/stdin` process fed one line at a time; stderr goes to a file, so that everything a task
    wrote there is in it once its completion line has been read."""

    def __init__(self, cmd, cwd, env, err_path):
        self.err = open(err_path, "w+b")
        self.p = subprocess.Popen(cmd + ["--task_stream", "/dev/stdin"], cwd=cwd, env=env, stdin=subprocess.PIPE,
                                  stdout=subprocess.PIPE, stderr=self.err)
        self.buf, self.err_at, self.k = b"", 0, 0

    def task(self, line):
        """(exit code, stdout, stderr) of the task `line` (bytes), from its completion line."""
        self.p.stdin.write(line + b"\n")
        self.p.stdin.flush()
        marker = b"# task %d: exit " % self.k
        deadline = time.monotonic() + TIMEOUT
        while True:
            i = self.buf.find(marker)
            if i >= 0 and (i == 0 or self.buf[i - 1:i] == b"\n") and b"\n" in self.buf[i:]:
                j = self.buf.index(b"\n", i)
                out, code, self.buf = self.buf[:i], int(self.buf[i + len(marker):j]), self.buf[j + 1:]
                break
            ready, _, _ = select.select([self.p.stdout], [], [], max(0.0, deadline - time.monotonic()))
            assert ready, "task %d: no completion line within %d s" % (self.k, TIMEOUT)
            chunk = os.read(self.p.stdout.fileno(), 1 << 16)
            assert chunk, "task %d: the stream ended (exit %s) before its completion line" % (self.k, self.p.poll())
            self.buf += chunk
        self.err.seek(self.err_at)
        err = self.err.read()
        self.err_at += len(err)
        self.k += 1
        return code, out, err

    def close(self):
        """The exit code once stdin is closed."""
        self.p.stdin.close()
        rest = self.p.stdout.read()
        assert rest == self.buf == b"", rest
        return self.p.wait(timeout=TIMEOUT)

    def kill(self):
        if self.p.poll() is None:
            self.p.kill()
            self.p.wait()
        self.err.close()


def untimed(out):
    return [l for l in out.decode(errors="surrogateescape").splitlines() if " time:" not in l]


def snapshot(d, inputs):
    """Every file of `d` but the inputs, with its bytes."""
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d)) if f not in inputs}


def reset(d, inputs):
    for f in os.listdir(d):
        if f not in inputs:
            os.remove(os.path.join(d, f))


def host_cmd(host, exe, tmp):
    if host == "native":
        return [exe], dict(os.environ)
    driver = tmp / "python_host.py"
    driver.write_text(PYTHON_HOST)
    return [sys.executable, str(driver)], dict(os.environ, LFR_GRAPH_STAGE="host")


def stream_and_one_shots(cmd, env, d, lines, tmp, set_once=()):
    """[(exit code, untimed stdout, stderr, files after the task)] of every line, by one stream and by one-shot
    processes in the same order on the same directory.  The lines `set_once` maps to an option a task may not set are
    not run one-shot: what stands for them is the refusal, which leaves the files as they are."""
    inputs = set(os.listdir(d))
    streamed = []
    s = Stream(cmd, d, env, tmp / "stream.err")
    try:
        for line in lines:
            code, out, err = s.task(line)
            streamed.append((code, untimed(out), err, snapshot(d, inputs)))
        assert s.close() == 0
    finally:
        s.kill()
    reset(d, inputs)
    one_shot = []
    for k, line in enumerate(lines):
        if k in dict(set_once):
            msg = b"ERROR: --%s is set once, on the task stream's command line\n" % dict(set_once)[k].encode()
            one_shot.append((2, [], msg, snapshot(d, inputs)))
            continue
        r = subprocess.run(cmd + ([a for a in line.split(b"\t")] if line else []), cwd=d, env=env, capture_output=True,
                           timeout=TIMEOUT)
        one_shot.append((r.returncode, untimed(r.stdout), r.stderr, snapshot(d, inputs)))
    reset(d, inputs)
    return streamed, one_shot


def grown(ms, k):
    """The pairs of `ms` between its first k images: the scene after its k-th image arrived."""
    keep = np.nonzero((ms.pair_img1 < k) & (ms.pair_img2 < k))[0]
    return ms.select_pairs(keep)


@pytest.fixture(scope="module")
def scene_dir(tmp_path_factory):
    """The inputs of the option stream: the goldens, a growing synthetic scene, a malformed file and the list files."""
    d = tmp_path_factory.mktemp("stream_inputs")
    for name in ("tiny", "linesearch", "fountain_2pct"):
        shutil.copy(os.path.join(GOLD, name + "_matches.pb"), d / (name + ".pb"))
    ms = synth.generate("cfg2", scale=0.08, seed=21)
    for k in (4, 5, 6, 7):
        (d / ("g%d.pb" % k)).write_bytes(wire.encode_matching_file(grown(ms, k)))
    half = ms.n_pairs // 2
    for k, part in enumerate([ms.select_pairs(np.arange(0, half)), ms.select_pairs(np.arange(half, ms.n_pairs))]):
        (d / ("split.pb.part.%d" % k)).write_bytes(wire.encode_matching_file(part))
    (d / "bad.pb").write_bytes(b"\x0a\xff\xff\xff\xff\x0f not a protobuf")
    fm = wire.read_matching_file(str(d / "fountain_2pct.pb"))
    pairs = [(fm.image_names[fm.pair_img1[p]], fm.image_names[fm.pair_img2[p]]) for p in range(0, fm.n_pairs, 3)]
    (d / "list one.txt").write_bytes(b"".join(b"%s %s\n" % (a.encode(), b.encode()) for a, b in pairs))
    (d / "lists.txt").write_bytes(b"list one.txt\tlist one.out\n")
    (d / "scenes.txt").write_bytes(b"linesearch.pb\tscene1.out\ng5.pb\tscene2.out\n")
    (d / "versioned.txt").write_bytes(b"g6.pb\tv1.out\tg4.out\tg4.rec\tv1.rec\ng7.pb\tv2.out\t\t\t\n")
    return d, ms.image_names


def option_lines(names):
    """Tasks over every option and combination the suites use, failing ones between them."""
    n = [x.encode() for x in names]
    return [
        b"--matches_file\ttiny.pb\t--output_file\tt.out\t--n_threads\t4",
        b"--matches_file\tfountain_2pct.pb\t--output_file\tf.out\t--banned_images\t" + wire.read_matching_file(
            os.path.join(GOLD, "fountain_2pct_matches.pb")).image_names[1].encode(),
        b"--help",
        b"",                                                                              # exit 1, as an empty command line
        b"--matches_file\tsplit.pb\t--output_file\tsplit.out",                            # .part.N pieces
        b"--matches_file\tg4.pb\t--output_file\tg4.out\t--record_file\tg4.rec",
        b"--matches_file\tg5.pb\t--output_file\tg5.out\t--initial_solution\tg4.out\t--update_initial_solution"
        b"\t--earlier_record_file\tg4.rec\t--record_file\tg5.rec",
        b"--bogus\t1",                                                                    # exit 1
        b"--matches_file\tg5.pb\t--output_file\tg5p.out\t--initial_solution\tg4.out\t--update_initial_solution"
        b"\t--previous_matches_file\tg4.pb",
        b"--matches_file\tbad.pb\t--output_file\tbad.out",                                # exit 255
        b"--matches_file\tg5.pb\t--output_file\tg5k.out\t--initial_solution\tg4.out\t--keep_initial_solution"
        b"\t--carry_initial_solution",
        b"--matches_file\tg5.pb\t--output_file\tg5j.out\t--initial_solution\tg4.out\t--fixed_images\t" + n[0],
        b"--matches_file\ttiny.pb\t--output_file\tx.out\t--initial_solution\tmissing.pb",  # exit 2
        b"--matches_file\tg6.pb\t--output_file\tg6u.out\t--initial_solution\tg5.out\t--update_initial_solution",
        b"--matches_file\ttiny.pb\t--output_file\tx.out\t--keep_initial_solution",         # exit 2: a rule
        b"--matches_file\tg7.pb\t--output_file\tq.out\t--query_images\t" + n[6] + b"\t--query_images\t" + n[5]
        + b"\t--joint_queries",
        b"--matches_file\tg7.pb\t--output_file\tq1.out\t--query_images\t" + n[6],
        b"--matches_file\ttiny.pb\t--output_file\tx.out\t--device\t0",                    # exit 2: set once
        b"--matches_file\ttiny.pb\t--output_file\tscene0.out\t--additional_scenes\tscenes.txt",
        b"--matches_file\tfountain_2pct.pb\t--output_file\tlist0.out\t--listed_pairs\tlists.txt",
        b"--matches_file\tg5.pb\t--output_file\tv0.out\t--initial_solution\tg4.out\t--update_initial_solution"
        b"\t--earlier_record_file\tg4.rec\t--record_file\tv0.rec\t--versioned_scenes\tversioned.txt",
        b"--t\tx",                                                                         # exit 2: set once
        b"--matches_file\ttiny.pb\t--output_file\tt space.out\t--gpus\t2",                 # exit 2: set once
        b"--matches_file\ttiny.pb\t--output_file\tt space.out",
        b"--matches_file\tlinesearch.pb\t--output_file\tt.out",                            # overwrites task 0's file
    ]


@pytest.mark.parametrize("host", ["native", "python"])
def test_every_option_in_one_stream_is_its_one_shot_run(checker_exe, scene_dir, tmp_path, host):  # noqa: F811
    d, names = scene_dir
    cmd, env = host_cmd(host, checker_exe, tmp_path)
    lines = option_lines(names)
    streamed, one_shot = stream_and_one_shots(cmd, env, str(d), lines, tmp_path,
                                              {17: "device", 21: "task_stream", 22: "gpus"})
    for k, (a, b) in enumerate(zip(streamed, one_shot)):
        assert a == b, (k, lines[k], a[:3], b[:3])
    codes = [c for c, _, _, _ in streamed]
    assert codes == [0, 0, 0, 1, 0, 0, 0, 1, 0, 255, 0, 0, 2, 0, 2, 0, 0, 2, 0, 0, 0, 2, 2, 0, 0], codes
    assert streamed[2][1] == ("Patch Match graph problem solver\n\n" + USAGE).splitlines()
    # every output the suites' options write is there, and the last task overwrote the first one's file
    files = streamed[-1][3]
    for f in ("g5.rec", "g5p.out", "g5k.out", "g5j.out", "g6u.out", "q.out", "q1.out", "scene1.out", "scene2.out",
              "list one.out", "v0.rec", "v1.out", "v1.rec", "v2.out", "split.out", "t space.out"):
        assert files.get(f), f
    assert files["t.out"] != streamed[0][3]["t.out"]


@pytest.mark.parametrize("host", ["native", "python"])
def test_a_live_chain_through_a_pipe_is_the_chain_of_processes(checker_exe, tmp_path, host):  # noqa: F811
    """An incremental registration: every task updates the previous task's SolutionFile against its record."""
    d = tmp_path / "chain"
    d.mkdir()
    ms = synth.generate("cfg2", scale=0.08, seed=4)
    lines = []
    for k in range(3, 9):
        (d / ("m%d.pb" % k)).write_bytes(wire.encode_matching_file(grown(ms, k)))
        line = b"--matches_file\tm%d.pb\t--output_file\ts%d.pb\t--record_file\tr%d.rec" % (k, k, k)
        if k > 3:
            line += b"\t--initial_solution\ts%d.pb\t--update_initial_solution\t--earlier_record_file\tr%d.rec" % (k - 1, k - 1)
        lines.append(line)
    cmd, env = host_cmd(host, checker_exe, tmp_path)
    streamed, one_shot = stream_and_one_shots(cmd, env, str(d), lines, tmp_path)
    assert streamed == one_shot
    assert all(c == 0 for c, _, _, _ in streamed)
    last = streamed[-1][3]
    assert len(last) == 2 * len(lines) and all(last.values())


def _both_hosts(exe, args, env=None, **kw):
    a = subprocess.run([exe] + args, capture_output=True, env=env, timeout=TIMEOUT, **kw)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, timeout=TIMEOUT,
                       env=dict(env or os.environ, LFR_SOLVE_PYTHON="1"), **kw)
    return a, b


def test_the_streams_own_command_line(checker_exe, tmp_path):  # noqa: F811
    tasks = tmp_path / "tasks.txt"
    tasks.write_bytes(b"--help\n\n--bogus")          # the last newline is optional
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    ends = {}
    for args in (["--task_stream", str(tasks)], ["--t", str(tasks)], ["--task", str(tasks), "--device", "0",
                                                                      "--n_threads", "3"]):
        a, b = _both_hosts(checker_exe, args, env)
        assert (a.returncode, a.stdout, a.stderr) == (b.returncode, b.stdout, b.stderr), args
        ends[tuple(args[:1])] = a
    usage = ("Patch Match graph problem solver\n\n" + USAGE).encode()
    r = ends[("--t",)]
    assert r.returncode == 0
    assert r.stdout == usage + b"# task 0: exit 0\n# task 1: exit 1\n# task 2: exit 1\n"
    assert r.stderr == (b"ERROR: the option '--matches_file' is required but missing\n\n" + USAGE.encode()
                        + b"ERROR: unrecognised option '--bogus'\n\n" + USAGE.encode())
    # what the stream's command line may not hold, and an unreadable FILE
    missing = str(tmp_path / "missing.txt")
    for args, msg in (
            (["--task_stream", str(tasks), "--matches_file", "m.pb"], b"ERROR: --task_stream and --matches_file exclude each other\n"),
            (["--task_stream", str(tasks), "--output_file", "o.pb", "--banned_images", "x"],
             b"ERROR: --task_stream and --output_file exclude each other\n"),
            (["--task_stream", str(tasks), "--initial_solution", ""], b"ERROR: --task_stream and --initial_solution exclude each other\n"),
            (["--task_stream", str(tasks), "--versioned_scenes", "v"], b"ERROR: --task_stream and --versioned_scenes exclude each other\n"),
            # the earlier rules keep their order: the first that fires writes the message
            (["--task_stream", str(tasks), "--keep_initial_solution"], b"ERROR: --keep_initial_solution needs --initial_solution FILE\n"),
            (["--task_stream", missing], b"ERROR: cannot read the task stream file '%s'\n" % missing.encode())):
        for r in _both_hosts(checker_exe, args, env):
            assert (r.returncode, r.stdout, r.stderr) == (2, b"", msg), (args, r)
    # --help is unchanged, with and without the option
    for args in (["--help"], ["--task_stream", str(tasks), "--help"]):
        for r in _both_hosts(checker_exe, args, env):
            assert (r.returncode, r.stdout, r.stderr) == (0, usage, b"")
    # without it the reference's errors are unchanged
    for r in _both_hosts(checker_exe, ["--output_file", "o.pb"], env):
        assert r.returncode == 1 and r.stderr.startswith(b"ERROR: the option '--matches_file' is required but missing\n")
    # an empty FILE runs no task
    (tmp_path / "empty.txt").write_bytes(b"")
    for r in _both_hosts(checker_exe, ["--task_stream", str(tmp_path / "empty.txt")], env):
        assert (r.returncode, r.stdout, r.stderr) == (0, b"", b"")


def test_torchrun_ranks_refuse_the_task_stream(tmp_path):
    (tmp_path / "t.txt").write_bytes(b"")
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, LAUNCHER, "--task_stream", str(tmp_path / "t.txt")], capture_output=True,
                       env=env, timeout=TIMEOUT)
    assert (r.returncode, r.stdout) == (2, b"")
    assert r.stderr == b"ERROR: --task_stream: torchrun ranks do not run task streams; use --gpus N\n"


def _vm_rss_kb(pid):
    with open("/proc/%d/status" % pid) as fh:
        for line in fh:
            if line.startswith("VmRSS:"):
                return int(line.split()[1])
    raise AssertionError("no VmRSS")


def test_no_growth_over_many_tasks(checker_exe, scene_dir, tmp_path):  # noqa: F811
    """300 tasks, a third of them failing at different stages: the resident set after task 300 is the one after 30."""
    d, _ = scene_dir
    work = tmp_path / "w"
    shutil.copytree(d, work)
    # (line, exit code): a third fail, one as its input is read, one after the solve when its output cannot be written
    kinds = [(b"--matches_file\tfountain_2pct.pb\t--output_file\to.out\t--record_file\to.rec", 0),
             (b"--matches_file\tbad.pb\t--output_file\tx.out", 255),
             (b"--matches_file\tg5.pb\t--output_file\tq.out\t--query_images\t0000.png", 0),
             (b"--matches_file\tlinesearch.pb\t--output_file\tl.out", 0),
             (b"--matches_file\tg6.pb\t--output_file\tno/such/dir.out", 255),
             (b"--matches_file\tfountain_2pct.pb\t--output_file\tlist0.out\t--listed_pairs\tlists.txt", 0)]
    s = Stream([checker_exe], str(work), dict(os.environ), tmp_path / "err")
    try:
        rss = {}
        for k in range(300):
            line, want = kinds[k % len(kinds)]
            assert s.task(line)[0] == want, k
            if k + 1 in (30, 300):
                rss[k + 1] = _vm_rss_kb(s.p.pid)
        assert s.close() == 0
    finally:
        s.kill()
    assert rss[300] - rss[30] <= 2048, rss
