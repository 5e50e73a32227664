"""The semi-dense optical flow on every schedule and grid its dispatch can choose, on the GPU (`-m gpu`).

tests/flow_paths.py runs the case table (windows 1 .. 15 with even ones, patches 1 .. 16, 1 .. 8 scales with every min_scale, 0 .. 4,
30, 31, 32, 128, 255 and 256 sweeps, frames smaller than one patch and with partial cell rows and columns, no keypoints, several per
cell in shuffled order, duplicates, keypoints outside the frame, more keypoints than resident warps, shifted / periodic / flat /
saturated scenes, a 65800-column frame with patch 1) through ops.semi_dense_optical_flow and vppb_sdof_u8 on pyramids at
alignments 128 / 16 / 4 / 1, views at odd columns and borders of exactly winsize / 2, against vo_semi_dense_flow, whole arrays
bit for bit.  Here the table adds 1080p and 4K with a keypoint in every cell and a 70000-column levels frame.  One child per
policy: the default, VPPB_SDOF_OCC=3 / 4, VPPB_SDOF_SCHEDULE=dataflow / levels / antidiagonals.

From the SM count the child reports and the grids the library prints under VPPB_SDOF_STATS=1, each policy asserts the paths it is
there for (tests/test_emulated_flow_paths.py checks that the policies together reach every path); VPPB_SDOF_OCC=3 / 4 must give
a capped case another grid than the default."""
import json
import time

import pytest

from tests import flow_paths as fp

pytestmark = pytest.mark.gpu

_RESULTS = {}


def _child(policy):
    if policy not in _RESULTS:
        t0 = time.time()
        rc, res, err = fp.run_child("gpu", policy, big=True)
        assert rc == 0 and res is not None, "child exited with %d:\n%s" % (rc, err[-4000:])
        print("policy %s: %d SMs, %d runs, %.1f s" % (policy, res["sms"], len(res["results"]), time.time() - t0))
        _RESULTS[policy] = res
    return _RESULTS[policy]


@pytest.mark.parametrize("policy", list(fp.POLICIES))
def test_flow_paths_gpu(gpu, policy):
    res = _child(policy)
    bad = fp.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    unmet = fp.unmet(res, policy)
    assert not unmet, "with %d SMs the case table no longer reaches: %s" % (res["sms"], "; ".join(unmet))
    if policy in ("occ3", "occ4"):
        mine, base = fp.capped_grids(res), fp.capped_grids(_child("default"))
        assert any(k in base and base[k] != g for k, g in mine.items()), "no capped case changed its grid: %s vs %s" % (mine, base)
