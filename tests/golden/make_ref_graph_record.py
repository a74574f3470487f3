"""Record what the reference's own main() produces on the adversarial match graphs of
tests/test_graph_stage_adversarial.py: tests/golden/ref_record_graph.json (per case the SHA-256 of the
SolutionFile and the untimed stdout lines) and, for the cases the GPU tests compare end to end,
tests/golden/adv_<case>_solution.pb (the SolutionFile itself).

Runs only where the reference sources are present (LFR_REFERENCE_DIR, see oracle/build_ref.py), with
oracle/_ref/solve as make_ref_record.py runs it.

    python tests/golden/make_ref_graph_record.py
"""
import hashlib
import importlib.util
import json
import os
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lfr_b200 import wire  # noqa: E402
import test_graph_stage_adversarial as adv  # noqa: E402
from test_ref_solve import untimed  # noqa: E402


def main():
    spec = importlib.util.spec_from_file_location("lfr_build_ref", os.path.join(ROOT, "oracle", "build_ref.py"))
    build_ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build_ref)
    assert build_ref.reference_available(), "the reference sources are not available here"
    exe = build_ref.build_solve()
    tmp = Path(tempfile.mkdtemp(prefix="lfr_graph_record_"))
    rec = {}
    for case in adv.REF_CASES:
        m, o = tmp / "m.pb", tmp / "s.pb"
        m.write_bytes(wire.encode_matching_file(adv.make_case(case)))
        r = subprocess.run([exe, "--matches_file", str(m), "--output_file", str(o), "--n_threads", "4"],
                           capture_output=True, text=True)
        assert r.returncode == 0, (case, r.stderr)
        sol = o.read_bytes()
        rec[case] = {"solution_sha256": hashlib.sha256(sol).hexdigest(), "stdout": untimed(r.stdout)}
        if case in adv.E2E_CASES:
            with open(adv.solution_path(case), "wb") as fh:
                fh.write(sol)
        print(case, rec[case]["stdout"][:2], flush=True)
    with open(adv.RECORD, "w") as fh:
        json.dump(rec, fh, indent=1, sort_keys=True)
        fh.write("\n")
    shutil.rmtree(tmp, ignore_errors=True)
    print("wrote", os.path.basename(adv.RECORD), "and %d SolutionFiles" % len(adv.E2E_CASES))


if __name__ == "__main__":
    main()
