"""The drop-in `solve`'s rules between its opt-in options, native and Python: every option alone, every pair and
every triple run through multi-view-refinement/build/solve_native and through lfr_b200/cli.py, which must end
with the same exit code, stdout and stderr.

LFR_GRAPH_STAGE=bogus stops every command line that passes the rules and reads its inputs at the route
message, before any solve, so each combination ends on a rule message, a file message or the route message.
With two conflicts the first rule in order wins, so this pins the order of the rules in both hosts.  The
option files exist ("present") or not ("absent"); triples are run with the files present."""
import itertools
import os
import subprocess

import pytest

from lfr_b200 import build_problem, wire
from lfr_b200.cli import main as cli_main
from test_native_exe import product_exe  # noqa: F401
from test_ref_solve import GOLD

# the opt-in options (--stats_json is the Python host's alone); a file option's argument is a key of _files()
OPTIONS = [("n_threads", "4"), ("banned_images", "@banned"), ("device", "0"), ("gpus", "2"),
           ("fixed_images", "@fixed"), ("initial_solution", "initial_solution"), ("keep_initial_solution", None),
           ("carry_initial_solution", None), ("update_initial_solution", None),
           ("previous_matches_file", "previous_matches_file"), ("record_file", "record_file"),
           ("earlier_record_file", "earlier_record_file"), ("query_images", "@query"), ("joint_queries", None),
           ("additional_scenes", "additional_scenes"), ("listed_pairs", "listed_pairs")]


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    """The MatchingFile, three of its image names, and every option file written under `present`."""
    d = tmp_path_factory.mktemp("option_rules")
    matches = os.path.join(GOLD, "tiny_matches.pb")
    ms = wire.read_matching_file(matches)
    names = ms.image_names
    n1, n2 = names[int(ms.pair_img1[0])], names[int(ms.pair_img2[0])]
    present = d / "present"
    present.mkdir()
    (present / "initial_solution").write_bytes(open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read())
    (present / "previous_matches_file").write_bytes(open(matches, "rb").read())
    (present / "earlier_record_file").write_bytes(wire.problem_record(build_problem(ms)))
    (present / "scene.pb").write_bytes(open(matches, "rb").read())
    (present / "additional_scenes").write_text("%s\t%s\n" % (present / "scene.pb", d / "scene_out.pb"))
    (present / "pairs.txt").write_text("%s %s\n" % (n1, n2))
    (present / "listed_pairs").write_text("%s\t%s\n" % (present / "pairs.txt", d / "list_out.pb"))
    return dict(dir=d, matches=matches, banned=names[-1], fixed=names[-2], query=names[0])


def _argv(inputs, combo, files):
    argv = ["--matches_file", inputs["matches"], "--output_file", str(inputs["dir"] / "out.pb")]
    for name, value in combo:
        argv.append("--" + name)
        if value is None:
            continue
        if value.startswith("@"):
            argv.append(inputs[value[1:]])
        elif name == "record_file":
            argv.append(str(inputs["dir"] / "record.rec"))
        else:
            argv.append(str(inputs["dir"] / files / value))
    return argv


def _python(argv, capfd):
    try:
        rc = cli_main(argv)
    except SystemExit as e:
        rc = e.code
    out, err = capfd.readouterr()
    return rc, out, err


@pytest.mark.parametrize("arity,files", [(1, "absent"), (1, "present"), (2, "absent"), (2, "present"), (3, "present")])
def test_native_and_python_hosts_apply_the_same_rules_in_the_same_order(product_exe, inputs, arity, files,  # noqa: F811
                                                                         capfd, monkeypatch):
    monkeypatch.setenv("LFR_GRAPH_STAGE", "bogus")
    for var in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(var, raising=False)
    # no command line reaches a device: hiding them all keeps CUDA's start-up out of every native run
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    differ, endings = [], set()
    for combo in itertools.combinations(OPTIONS, arity):
        argv = _argv(inputs, combo, files)
        r = subprocess.run([product_exe] + argv, capture_output=True, text=True, env=env)
        native = (r.returncode, r.stdout, r.stderr)
        python = _python(argv, capfd)
        if native != python:
            differ.append((argv, native, python))
        endings.add(r.stderr.splitlines()[0] if r.stderr else "")
        assert not (inputs["dir"] / "out.pb").exists()
    assert not differ, differ[:5]
    assert "ERROR: LFR_GRAPH_STAGE must be 'host' or 'device'" in endings
