"""The pyramid, Scharr and pyrlk_prepare kernels on every variant their dispatch can choose, on the GPU (`-m gpu`).

tests/pyramid_paths.py runs the stand-alone table (Scharr widths at every residue mod 8, low-pass parents around the 16-byte groups,
1 x N, N x 1, 2 x 2, 3 x 3, outputs smaller than 1 + n/2, borders of exactly 1 / 2 and output borders up to the level size, input and
output alignments 128 .. 1 chosen independently, views at odd columns, at 8-but-not-16-byte offsets, column windows and row bands,
vint2 data of either sign, vfloat2 data whose sums depend on their order) and the vppb_pyrlk_prepare table (1 .. 8, 9, 12 and 16
levels, no / a vint2 / a vfloat2 gradient pyramid, borders 2 .. 22, unaligned and view inputs, a fused grid the cooperative cap
certainly cuts and one it certainly does not, 70 calls queued on one stream, and rejected calls that must write nothing) against the
oracle, whole allocations byte for byte.  One child per policy (the default, VPPB_PREPARE=fused, VPPB_PREPARE=streams), and the
default again with 1080p, 4K and 8K pyramids with and without a gradient pyramid.

From the SM count the child reports, each policy asserts the paths it is there for (tests/test_emulated_pyramid_paths.py checks that
the policies together reach every path)."""
import json
import time

import pytest

from tests import pyramid_paths as pp

pytestmark = pytest.mark.gpu

RUNS = [(p, False) for p in pp.POLICIES] + [("default", True)]


@pytest.mark.parametrize("policy,big", RUNS, ids=["%s%s" % (p, "_big" if b else "") for p, b in RUNS])
def test_pyramid_paths_gpu(gpu, policy, big):
    t0 = time.time()
    rc, res, err = pp.run_child("gpu", policy, big=big)
    assert rc == 0 and res is not None, "child exited with %d:\n%s" % (rc, err[-4000:])
    print("policy %s%s: %d SMs, %d runs, %.1f s" % (policy, " --big" if big else "", res["sms"], len(res["results"]), time.time() - t0))
    bad = pp.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    unmet = pp.unmet(res, policy)
    assert not unmet, "with %d SMs the case tables no longer reach: %s" % (res["sms"], "; ".join(unmet))
    if big:
        assert sum(r["case"].startswith("big_") for r in res["results"]) == 6
