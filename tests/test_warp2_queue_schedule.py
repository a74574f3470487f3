"""The register warp tier's queue launches as the host schedule lays them out (lfr_debug_time_schedule
with LFR_SCHED_DUMP: host-only, no device involved): which scenes get a queue, how many launches, how
many warps per SM, and the LFR_DBG_WARP2_WARPS_SHIFT override."""
import ctypes as C
import re

import pytest

from lfr_b200.capi import DBG_WARP2_WARPS_SHIFT


def schedule(b200, capfd, monkeypatch, name, warps=0):
    from lfr_b200 import build_problem, synth
    f = b200.lib.lfr_debug_time_schedule
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    p = build_problem(synth.generate(name))
    s, keep = b200.marshal(p)
    o = b200.default_options(debug_flags=warps << DBG_WARP2_WARPS_SHIFT)
    monkeypatch.setenv("LFR_SCHED_DUMP", "1")
    capfd.readouterr()
    us, nl, dg = C.c_double(), C.c_int(), C.c_uint64()
    assert f(C.byref(s), C.byref(o), 1, C.byref(us), C.byref(nl), C.byref(dg)) == 0
    err = capfd.readouterr().err
    queues = [(int(n), int(slot), int(w)) for n, slot, w in
              re.findall(r"warp2 queue\s+n\s+(\d+)\s+slot\s+(\d+)\s+warps/SM (\d+)", err)]
    buckets = [int(v) for v in re.findall(r"bucket variant\s+(\d+)", err)]
    return nl.value, queues, buckets


def test_cfg2_is_one_queue_launch(b200, capfd, monkeypatch):
    n, queues, buckets = schedule(b200, capfd, monkeypatch, "cfg2")
    assert n == 1 and buckets == []
    assert len(queues) == 1 and queues[0][0] == 4218 and queues[0][2] == 8


def test_members_past_the_slot_go_to_a_second_queue(b200, capfd, monkeypatch):
    """cfg4: the members whose own slot does not fit 8 to an SM form a second queue at fewer warps;
    at 4 warps per SM every member fits one slot and one queue takes them all."""
    n8, q8, b8 = schedule(b200, capfd, monkeypatch, "cfg4")
    n4, q4, b4 = schedule(b200, capfd, monkeypatch, "cfg4", warps=4)
    assert len(q8) == 2 and q8[0][2] == 8 and 4 <= q8[1][2] < 8
    assert q8[0][1] <= 227 * 1024 // 8 < q8[1][1] and q8[1][1] * q8[1][2] <= 227 * 1024
    assert len(q4) == 1 and q4[0][2] == 4 and q4[0][0] == q8[0][0] + q8[1][0]
    assert b4 == b8 and n8 == n4 + 1


@pytest.mark.parametrize("warps", [1, 6, 8, 12, 15])
def test_warps_override_is_clamped_to_the_kernel(b200, capfd, monkeypatch, warps):
    n, queues, _ = schedule(b200, capfd, monkeypatch, "cfg2", warps)
    assert n == 1 and queues[0][2] == min(warps, 8)


def test_scenes_without_wide_members_keep_the_bucket_launches(b200, capfd, monkeypatch):
    """cfg3 (no register-tier component above 16 unknowns): the 12-warp per-bucket kernels stay."""
    n, queues, buckets = schedule(b200, capfd, monkeypatch, "cfg3")
    assert queues == [] and buckets and set(buckets) <= {8, 16} and n == len(buckets)
