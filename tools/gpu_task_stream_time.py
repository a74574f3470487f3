"""Time --task_stream: one process that runs a stream of tasks, against one process per task.

    python tools/gpu_task_stream_time.py [--queries 100] [--chain 10] [--device_tasks 10] [--out FILE]

Three workloads, each run as a stream (the native drop-in with `--task_stream`, fed one line at a time through a
pipe: line K is written after `# task K-1:` was read) and as the same sequence of one-shot processes:
  (a) localize  gpu_localize_time.py's workload: every query's own file, one task per query;
  (b) chain     a cfg2-scale scene grown one image per task, each task updating the previous task's SolutionFile
                against its record (--update_initial_solution --earlier_record_file --record_file);
  (c) device    a cfg4-scale scene on the device route, the same task again and again; per task the wall time (from
                writing the line to reading its completion line) against its "Total time" line: the gap is what a
                stream still pays per task outside the timed work (plan creation and teardown, the stage's
                cudaMallocs, the page-locked staging).
Each task's output and record bytes are checked against the one-shot run's.  Prints one JSON object with the
GPU's name and power limit (read, never set)."""
import argparse
import dataclasses
import json
import os
import re
import select
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_localize_time import TEMPLATES, query_part, templates  # noqa: E402
from gpu_update_since_time import NATIVE, gpu_info  # noqa: E402
from lfr_b200 import synth, wire  # noqa: E402

TIMEOUT = 600


class Stream:
    def __init__(self, cwd):
        self.p = subprocess.Popen([NATIVE, "--task_stream", "/dev/stdin"], cwd=cwd, stdin=subprocess.PIPE,
                                  stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
        self.buf, self.k = b"", 0

    def task(self, line):
        """(wall ms, stdout) of one task, which must succeed."""
        t0 = time.perf_counter()
        self.p.stdin.write(line + b"\n")
        self.p.stdin.flush()
        marker = b"# task %d: exit " % self.k
        deadline = time.monotonic() + TIMEOUT
        while marker not in self.buf or not self.buf.split(marker, 1)[1].count(b"\n"):
            ready, _, _ = select.select([self.p.stdout], [], [], max(0.0, deadline - time.monotonic()))
            chunk = os.read(self.p.stdout.fileno(), 1 << 16) if ready else b""
            if not chunk:
                raise RuntimeError("task %d: no completion line" % self.k)
            self.buf += chunk
        wall = (time.perf_counter() - t0) * 1e3
        out, rest = self.buf.split(marker, 1)
        code, self.buf = rest.split(b"\n", 1)
        if int(code) != 0:
            raise RuntimeError("task %d exited %s" % (self.k, code.decode()))
        self.k += 1
        return wall, out.decode()

    def close(self):
        self.p.stdin.close()
        self.p.stdout.read()
        if self.p.wait(timeout=TIMEOUT) != 0:
            raise RuntimeError("the stream exited %d" % self.p.returncode)


def one_shot(line, cwd):
    t0 = time.perf_counter()
    r = subprocess.run([NATIVE] + [a.decode() for a in line.split(b"\t")], cwd=cwd, capture_output=True, text=True,
                       check=True, timeout=TIMEOUT)
    return (time.perf_counter() - t0) * 1e3, r.stdout


def total_ms(stdout):
    return int(re.search(r"Total time: (\d+)ms", stdout).group(1))


def outputs(line, cwd):
    """The bytes of the files a task line writes (its output and record files)."""
    f = line.split(b"\t")
    return {p: open(os.path.join(cwd, p.decode()), "rb").read()
            for o, p in zip(f, f[1:]) if o in (b"--output_file", b"--record_file")}


def compare(lines, cwd):
    """Both ways over `lines`: per task (stream wall ms, stream Total ms, process wall ms, process Total ms); every
    task's files must be the one-shot run's."""
    s = Stream(cwd)
    streamed, files = [], []
    try:
        for line in lines:
            w, out = s.task(line)
            streamed.append((w, total_ms(out)))
            files.append(outputs(line, cwd))
        s.close()
    finally:
        if s.p.poll() is None:
            s.p.kill()
            s.p.wait()
    procs = []
    for line, want in zip(lines, files):
        w, out = one_shot(line, cwd)
        procs.append((w, total_ms(out)))
        if outputs(line, cwd) != want:
            raise AssertionError("a task's files differ from its one-shot run's: %r" % line)
    return np.array([a + b for a, b in zip(streamed, procs)], dtype=np.float64)


def summary(t):
    return dict(tasks=len(t), stream_wall_ms=float(t[:, 0].sum()), stream_total_ms=int(t[:, 1].sum()),
                processes_wall_ms=float(t[:, 2].sum()), processes_total_ms=int(t[:, 3].sum()),
                stream_wall_ms_per_task=dict(median=float(np.median(t[:, 0])), best=float(t[:, 0].min())),
                process_wall_ms_per_task=dict(median=float(np.median(t[:, 2])), best=float(t[:, 2].min())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=100)
    ap.add_argument("--chain", type=int, default=10)
    ap.add_argument("--device_tasks", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info())
    with tempfile.TemporaryDirectory() as d:
        # (a) one task per localization query
        tpls = templates(0.2)
        lines = []
        for i in range(a.queries):
            name = "q%05d.png" % i
            wire.write_matching_file(query_part(tpls[i % TEMPLATES], name), os.path.join(d, "q%05d.pb" % i))
            lines.append(b"--matches_file\tq%05d.pb\t--output_file\tq%05d.out" % (i, i))
        res["localize"] = summary(compare(lines, d))
        print(json.dumps(res["localize"]), flush=True)
        # (b) an incremental chain: a cfg2-scale scene grown one image per task
        cfg = dataclasses.replace(synth.CONFIGS["cfg2"], n_images=a.chain + 2)
        ms = synth.generate(cfg, scale=1.0, seed=3)
        lines = []
        for k in range(3, a.chain + 3):
            keep = np.nonzero((ms.pair_img1 < k) & (ms.pair_img2 < k))[0]
            wire.write_matching_file(ms.select_pairs(keep), os.path.join(d, "c%d.pb" % k))
            line = b"--matches_file\tc%d.pb\t--output_file\tc%d.out\t--record_file\tc%d.rec" % (k, k, k)
            if k > 3:
                line += b"\t--initial_solution\tc%d.out\t--update_initial_solution\t--earlier_record_file\tc%d.rec" % (
                    k - 1, k - 1)
            lines.append(line)
        res["chain"] = summary(compare(lines, d))
        print(json.dumps(res["chain"]), flush=True)
        # (c) cfg4-scale device-route tasks: the per-task gap between wall time and "Total time"
        wire.write_matching_file(synth.generate("cfg4", scale=1.0, seed=7), os.path.join(d, "cfg4.pb"))
        t = compare([b"--matches_file\tcfg4.pb\t--output_file\tcfg4.out"] * a.device_tasks, d)
        gap = t[:, 0] - t[:, 1]
        res["device"] = dict(summary(t), stream_gap_ms_per_task=dict(median=float(np.median(gap[1:])),
                                                                       first=float(gap[0])),
                             stream_total_ms_per_task=dict(median=float(np.median(t[1:, 1]))),
                             process_total_ms_per_task=dict(median=float(np.median(t[:, 3]))))
        print(json.dumps(res["device"]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
