"""The C-ABI library loads on a machine without a GPU, exports every symbol the
headers declare, and refuses to compute without a device (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(lfr_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(b200):
    """include/lfr.h -> csrc/liblfr_b200.so (the product); include/lfr_wire.h and include/lfr_host.h ->
    csrc/liblfr_host.so (CPU-only host utilities)."""
    from lfr_b200.capi import ABI_SYMBOLS, load_host
    from lfr_b200.wire import WIRE_SYMBOLS
    core = declared("lfr.h")
    assert "lfr_solve" in core
    for n in core:
        assert hasattr(b200.lib, n), n
    assert b200.backend == "b200"
    assert sorted(ABI_SYMBOLS) == core
    host_lib = load_host()
    host_names = sorted(set(declared("lfr_wire.h") + declared("lfr_host.h")))
    assert "lfr_wire_decode_matches" in host_names and "lfr_host_stage_create" in host_names
    for n in host_names:
        assert hasattr(host_lib, n), n
    host = ["lfr_host_stage_create", "lfr_host_stage_export", "lfr_host_stage_destroy"]
    assert sorted(WIRE_SYMBOLS + host) == host_names


def test_host_library_has_no_cuda_dependency():
    import subprocess
    from lfr_b200.capi import HOST_LIB_PATH, load_host
    load_host()
    out = subprocess.check_output(["ldd", HOST_LIB_PATH]).decode()
    assert "cuda" not in out.lower() and "nvidia" not in out.lower(), out


def test_oracle_exports_the_same_abi(oracle):
    for n in declared("lfr.h"):
        assert hasattr(oracle.lib, n), n
    assert oracle.backend == "cpu-oracle"


def test_struct_layouts_match_the_header(b200, oracle):
    from lfr_b200.capi import LfrOptions, LfrProblem, LfrStats
    from lfr_b200 import EDGE_DTYPE
    assert C.sizeof(LfrProblem) == 72 and C.sizeof(LfrStats) == 88 and EDGE_DTYPE.itemsize == 80
    for lib in (b200, oracle):     # same defaults from both implementations
        o = lib.default_options()
        assert (o.bound, o.cauchy_a, o.tukey_a, o.max_num_iterations) == (1.0, 0.25, 0.0625, 100)
        assert (o.function_tolerance, o.gradient_tolerance, o.parameter_tolerance) == (1e-4, 1e-8, 1e-4)
        assert o.min_line_search_step_size == 1e-9 and o.n_threads == 8 and o.linear_solver == 0
    assert C.sizeof(LfrOptions) == 160


def test_ctypes_structs_agree_with_the_c_compiler(tmp_path):
    import subprocess
    from lfr_b200.capi import LfrOptions, LfrProblem, LfrStats
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lfr.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n", '
                   'sizeof(lfr_edge), sizeof(lfr_problem), sizeof(lfr_options), sizeof(lfr_stats), '
                   'offsetof(lfr_options, n_threads), offsetof(lfr_stats, total_iterations));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [80, C.sizeof(LfrProblem), C.sizeof(LfrOptions), C.sizeof(LfrStats),
                   LfrOptions.n_threads.offset, LfrStats.total_iterations.offset]


def test_no_cpu_fallback_without_a_device(b200):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lfr_b200 import build_problem, synth
    p = build_problem(synth.generate("cfg1", scale=0.2))
    with pytest.raises(RuntimeError, match=r"\(-2\)|no CUDA|CUDA"):
        b200.solve(p)


def test_invalid_problems_are_rejected(oracle):
    from lfr_b200 import build_problem, synth
    from lfr_b200.capi import LfrStats
    p = build_problem(synth.generate("cfg1", scale=0.2))
    s, keep = oracle.marshal(p)
    s.n_edges += 1
    pos = np.zeros((p.graph.n_nodes, 2))
    assert oracle.lib.lfr_solve(C.byref(s), None, pos.ctypes.data, None) == -1
    assert b"row_ptr" in oracle.lib.lfr_last_error()


def test_oracle_exports_solve_multi_with_single_device_semantics(oracle):
    """lfr_solve_multi is part of include/lfr.h; the CPU oracle ignores `devices` and returns what lfr_solve does."""
    from lfr_b200 import build_problem, synth
    p = build_problem(synth.generate("cfg1", scale=0.3))
    pos1, st1 = oracle.solve(p, oracle.default_options(n_threads=2))
    pos2, st2 = oracle.solve_multi(p, [0, 1], oracle.default_options(n_threads=2))
    assert np.array_equal(pos1, pos2) and np.array_equal(st1["iterations"], st2["iterations"])


def test_schedule_does_not_depend_on_the_thread_count(b200, monkeypatch):
    """The launch schedule (buckets, launch lists, CTA-tier components) is built on the host by range
    workers for large dispatch lists; merged in range order, it must be the same for any thread count.
    (Host-only hook of the product library: no device involved.)"""
    from lfr_b200 import build_problem, synth
    f = b200.lib.lfr_debug_time_schedule
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    for name, scale in (("cfg3", 1.0), ("ring60", 1.0), ("cfg5", 0.05)):
        p = build_problem(synth.generate(name, scale=scale))
        s, keep = b200.marshal(p)
        seen = set()
        for n_thr in ("1", "2", "5", "8"):
            monkeypatch.setenv("LFR_SCHEDULE_THREADS", n_thr)
            us, nl, dg = C.c_double(), C.c_int(), C.c_uint64()
            assert f(C.byref(s), None, 1, C.byref(us), C.byref(nl), C.byref(dg)) == 0
            seen.add((nl.value, dg.value))
        assert len(seen) == 1, (name, seen)


def test_profile_record_decodes_every_word():
    """capi.profile_record on hand-built LFR_DBG_PROFILE records: the word layout and tier codes of
    LmProfile in csrc/lfr_lm.cuh."""
    from lfr_b200.capi import PROFILE_TIERS, profile_record
    src = open(os.path.join(ROOT, "local-feature-refinement_b200", "csrc", "lfr_lm.cuh")).read()
    words = re.search(r"enum Word \{([^}]*)\}", src).group(1)
    assert [w.split("=")[0].strip() for w in words.split(",")] == [
        "kTotal", "kSetup", "kEval", "kAssemble", "kSolve", "kRest", "kSteps", "kTierWord"]
    tiers = dict(re.findall(r"k(\w+) = (\d+)", re.search(r"enum Tier : unsigned \{([^}]*)\}", src).group(1)))
    assert {int(v): k.lower() for k, v in tiers.items()} == PROFILE_TIERS
    rec = np.zeros((3, 8), dtype=np.uint64)
    rec[0] = [1000, 10, 200, 300, 400, 50, (7 << 32) | 131, (1 << 56) | 40]   # warp2, 40 polynomial cycles
    rec[1] = [5000, 0, 600, 700, 3000, 700, (0 << 32) | 3, (4 << 56) | 1234]  # CTA, 1234 CG iterations
    d = profile_record(rec)                                                   # rec[2]: no record (empty component)
    for k, col in (("total", 0), ("setup", 1), ("eval", 2), ("assemble", 3), ("solve", 4), ("rest", 5)):
        assert d[k].tolist() == rec[:, col].tolist(), k
    assert d["ls_steps"].tolist() == [7, 0, 0]
    assert d["smid"].tolist() == [131, 3, 0]
    assert d["tier"].tolist() == [1, 4, 0]
    assert d["counter"].tolist() == [40, 1234, 0]
    assert [PROFILE_TIERS.get(t) for t in d["tier"].tolist()] == ["warp2", "cta", None]
    assert profile_record(rec.ravel())["total"].shape == (3,)
