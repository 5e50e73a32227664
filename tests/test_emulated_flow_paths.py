"""The semi-dense optical flow on every schedule its dispatch can choose, on the CPU emulator (no GPU needed).

tests/flow_paths.py runs one case table through ops.semi_dense_optical_flow and vppb_sdof_u8 once per policy (the default,
VPPB_SDOF_OCC=3 / 4, VPPB_SDOF_SCHEDULE=dataflow / levels / antidiagonals) in a child process; valid, pos and dist of every
keypoint must equal vo_semi_dense_flow's bit for bit.  The H100 counterpart is tests/test_gpu_flow_paths.py.

The emulated library is built with UBSan's alignment and bounds checks, and the AddressSanitizer leg catches reads past a pyramid
allocation (rows that end on the last byte of it, the SAD's aligned words), past the keypoints, outputs or workspace (each ends on the
last byte of its allocation).  The emulator reports 2 SMs and lets a cooperative grid have one CTA: every fused call with more than 8
warps of work runs its grid-stride loops, and no VPPB_SDOF_OCC changes that grid.  The 65800-column frame runs here under the
default, dataflow and levels policies only, with one sweep: its k_sdof_levels walks 65802 anti-diagonals with 1024 emulated threads."""
import glob
import json
import os
import subprocess
import sys

import pytest

from tests import flow_paths as fp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _libasan():
    p = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return p if os.path.isabs(p) and os.path.exists(p) else None


def _run(tmp_path, policy, asan):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    build_emu.build(asan=asan)  # here, not in the child: the ASan child runs with libasan preloaded
    env = dict(os.environ, VPPB_EMU_LOG=str(tmp_path / "emu_fail.log"), UBSAN_OPTIONS="log_path=%s" % (tmp_path / "ubsan"))
    if asan:
        env.update(VPPB_EMU_ASAN="1", VPPB_EMU_STACK_KB="96", LD_PRELOAD=_libasan(),
                   ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:log_path=%s" % (tmp_path / "asan"))
    else:
        env.pop("VPPB_EMU_ASAN", None)
    rc, res, err = fp.run_child("emu", policy, env=env)
    reports = "".join(open(f).read() for f in sorted(glob.glob(str(tmp_path / "ubsan*")) + glob.glob(str(tmp_path / "asan*"))))
    assert rc == 0 and res is not None, "child exited with %d:\n%s\n%s" % (rc, err[-3000:], reports[:4000])
    errors = [l for l in reports.splitlines() if "runtime error" in l or "ERROR: AddressSanitizer" in l or "SUMMARY: " in l]
    assert not errors, "sanitizer reports from the emulated kernels:\n" + reports[:4000]
    bad = fp.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    assert res["sms"] == 2
    unmet = fp.unmet(res, policy)
    assert not unmet, "the case table no longer reaches: " + "; ".join(unmet)
    assert all(r["stats"]["grid"] == 1 for r in res["results"] if r["stats"]), "the emulator's cooperative grid is one CTA"


@pytest.mark.parametrize("policy", list(fp.POLICIES))
def test_flow_paths_emulated(built, tmp_path, policy):
    _run(tmp_path, policy, asan=False)


@pytest.mark.parametrize("policy", list(fp.POLICIES))
def test_flow_paths_emulated_asan(built, tmp_path, policy):
    if not _libasan():
        pytest.skip("libasan.so not available")
    _run(tmp_path, policy, asan=True)


def test_flow_policies_reach_every_path():
    """the policies' shares of the reach assertions together name every schedule, both outcomes of `levels`, the relaxation
    kernel's grid-stride loops and long relaxations, and the rejection of a 256th dataflow sweep"""
    union = set().union(*(fp.expected(p) for p in fp.POLICIES)) | {"schedule rejected"}
    assert fp.every_path() <= union, sorted(fp.every_path() - union)
    assert "schedule rejected" in fp.reached(dict(results=[dict(plan=dict(schedule="rejected"), prop=256, ncols=22)]))


def test_sdof_dispatch_transcription():
    """the transcribed dispatch on calls whose path is known"""
    import numpy as np

    one = np.array([[7, 9]], np.int32)
    plan = lambda prop, env, nscales=1, kps=one, shape=(40, 60), patch=5: fp.sdof_plan(shape[0], shape[1], 9, nscales, 0, prop, patch, kps, env)
    assert plan(30, {})["schedule"] == "relaxation" and plan(31, {})["schedule"] == "dataflow"
    assert plan(2, {"VPPB_SDOF_SCHEDULE": "dataflow"})["schedule"] == "dataflow"
    assert plan(255, {})["schedule"] == "dataflow" and plan(256, {})["schedule"] == "rejected"
    assert plan(256, {"VPPB_SDOF_SCHEDULE": "dataflow"})["schedule"] == "rejected"
    assert plan(128, {}, nscales=2)["schedule"] == "dataflow" and plan(129, {}, nscales=2)["schedule"] == "rejected"
    assert plan(256, {"VPPB_SDOF_SCHEDULE": "antidiagonals"})["schedule"] == "antidiagonals"
    assert plan(2, {"VPPB_SDOF_OCC": "4"})["minb"] == 4 and plan(2, {"VPPB_SDOF_OCC": "5"})["minb"] == 2 and plan(2, {})["minb"] == 2
    # 40 x 60, patch 5: 8 x 12 cells = 96 warps of work, 12 blocks of 8 warps; 1000 keypoints ask for 125 blocks
    assert plan(2, {})["want_blocks"] == 12 and plan(2, {}, kps=np.zeros((1000, 2), np.int32))["want_blocks"] == 125
    # levels: a horizontal pair is two levels in either direction, a lone cell one, a keypoint outside the frame none
    lv = {"VPPB_SDOF_SCHEDULE": "levels"}
    pair = np.array([[7, 9], [7, 14], [39, 60]], np.int32)
    sw = plan(2, lv, kps=pair)["sweeps"]
    assert [(s["forward"], s["nlevels"], s["path"]) for s in sw] == [(0, 2, "levels"), (1, 2, "levels")]
    assert [s["nlevels"] for s in plan(1, lv, kps=np.array([[60, 7]], np.int32))["sweeps"]] == [0]
    # a keypoint in every cell of 8 x 12 cells: 12 + 2 * 7 = 26 anti-diagonals and as many levels, so the sweep falls back
    every = np.array([[r, c] for r in range(2, 40, 5) for c in range(2, 60, 5)], np.int32)
    assert all(s["nlevels"] == 26 and s["path"] == "antidiagonals" for s in plan(3, lv, kps=every)["sweeps"])
    # a partial last cell row (43 rows, patch 5): backward sweeps start on it; its keypoints claim nothing
    assert fp.marked_cells(np.array([[41, 3], [39, 3]], np.int32), 43, 60, 5, 0) == {(7, 0)}
    # coarser levels round up: (40 x 60) -> (21 x 31); a keypoint at column 60 would be inside level 1 but is outside the frame
    assert fp.level_dims(40, 60, 3) == [(40, 60), (21, 31), (11, 16)] and fp.cell_dims(40, 60, 5, 1) == (5, 7)
    assert fp.marked_cells(np.array([[3, 60], [3, 58]], np.int32), 40, 60, 5, 1) == {(0, 5)}
    assert fp.parse_stats("x\nvppb_sdof_u8: grid 264 x 256, 13 grid barriers, 22 relaxation rounds after the first of each sweep, 9 re-evaluations\n") == \
        [dict(grid=264, barriers=13, rounds=22, reevals=9)]
