"""FAST9 and the square-window Lucas-Kanade matcher on every kernel their dispatch can choose, on the GPU (`-m gpu`).

tests/detector_paths.py runs the FAST case table (widths around the 32-pixel words and the 2016-pixel band boxes, rows around the
4-row bands and 8-row emit CTAs, alignments 128 / 16 / 8 / 4 / 1, views at odd columns, borders 3 and 5, both rings, masks with holes,
thresholds 0 / 20 / 127 / 255, a warp-path frame larger than the detection grid, a 32800-row frame) through fast9 (all, local maxima,
blockwise), fast9_blockwise_rank and fast9_scores against the C oracle, exactly; and the LK case table (every odd window 1 .. 15 with
int and float gradients, 1 .. 8 levels, min_scale 0 .. 2, keypoint counts 1 .. 65 and beyond a wave of resident CTAs, keypoints on,
off and just outside the frame, in a flat patch, pushed off by a prediction) through lucas_kanade, pyrlk_match and vppb_lk_match_u8
against the oracle, bit for bit.  One child per policy (default, VPPB_FAST_IMPL=warp, VPPB_LK_V1=1, VPPB_LK_WARPS=1 / 2), because the
library reads some of these knobs once per process.  The default policy also runs a level 0 of more than 2 GiB (64 MiB pitch),
which only the one-keypoint-per-warp kernel with 64-bit offsets may take.

From the SM count the child reports, a transcription of the dispatch rules checks that each policy still reaches the kernels it is
there for; together they reach every k_fast9_band instantiation and k_fast9_detect in each FAST mode, every v2 PPL x WARPS x gradient
and every v1 PPL x gradient (tests/test_emulated_detector_paths.py checks that union)."""
import json
import time

import pytest

from tests import detector_paths as dp

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("policy", list(dp.POLICIES))
def test_detector_paths_gpu(gpu, policy):
    t0 = time.time()
    big = policy == "default"
    rc, res, err = dp.run_child("gpu", policy, big=big)
    assert rc == 0 and res is not None, "child exited with %d:\n%s" % (rc, err[-4000:])
    print("policy %s: %d SMs, %d runs, %.1f s" % (policy, res["sms"], len(res["results"]), time.time() - t0))
    bad = dp.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    unmet = dp.unmet(res, policy, big=big)
    assert not unmet, "with %d SMs the case tables no longer reach: %s" % (res["sms"], "; ".join(unmet))
