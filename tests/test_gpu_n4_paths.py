"""lbp_transform, local_maxima_filter and the oriented LK matcher on every path their dispatch can choose, and the workspace alignment
of every entry point that takes one, on the GPU (`-m gpu`).

tests/n4_paths.py runs, in a child process:
  * lbp: widths 1 .. 1000 around the 16-pixel groups, heights 1 .. 131 (every nrows % 4), input and output alignments 1 / 4 / 16 / 128
    chosen independently, views at odd columns, mirror and value borders, 4K and 8K frames and a u8 frame of more than 2 GiB
    (40000 x 56000), against the oracle over both whole allocations;
  * local_maxima_filter, u8 and int: the oracle scenes, alternating chains of 1100 links (254 for u8) along N, NW, NE and W, int
    images with negative pixels and border values, widths around the 16-pixel runs, single rows and columns, views, a frame small
    enough for one trip and frames large enough to loop (4K, 8K, the 2 GiB frame), against the oracle over the whole allocation
    and the bytes past the workspace size;
  * the oriented LK matcher: every odd window with int and float gradients, 1 .. 5 keypoints and more CTAs than one wave, keypoints
    on, near and outside the frame, rotated windows, predictions that leave the search margin, flat patches, max_iter 0 / 1 / 21,
    tiny and huge max_step, alignments and views of A and B, against the oracle bit for bit;
  * every entry point that takes a workspace, with a misaligned one: VPPB_E_ARG, nothing written.
From the SM count the child reports, a transcription of the launch rules checks that the tables still reach both lbp
instantiations and the ragged edge, local_maxima_filter's single-trip and grid-stride regimes for both pixel types, and all twelve
k_lk_match_oriented<PPL, GF> instantiations."""
import json
import time

import pytest

from tests import n4_paths as n4

pytestmark = pytest.mark.gpu


def test_n4_paths_gpu(gpu):
    t0 = time.time()
    rc, res, err = n4.run_child("gpu", big=True)
    assert rc == 0 and res is not None, "child exited with %d:\n%s" % (rc, err[-4000:])
    print("%d SMs, %d runs, %.1f s" % (res["sms"], len(res["results"]), time.time() - t0))
    bad = n4.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    unmet = n4.unmet(res)
    assert not unmet, "with %d SMs the case tables no longer reach: %s" % (res["sms"], "; ".join(unmet))
