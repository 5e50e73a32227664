"""FAST9 and the square-window Lucas-Kanade matcher on every kernel their dispatch can choose, on the CPU emulator (no GPU needed).

tests/detector_paths.py runs the FAST and LK case tables once per policy (default, VPPB_FAST_IMPL=warp, VPPB_LK_V1=1,
VPPB_LK_WARPS=1 / 2) in a child process, because the library reads some of these knobs once per process.  FAST keypoints, ranks and
scores must equal the C oracle's exactly, LK flows and errors bit for bit.  The H100 counterpart is tests/test_gpu_detector_paths.py.

The emulated library is built with UBSan's alignment and bounds checks, and the AddressSanitizer leg catches reads that leave an
allocation (a view's ring, a detection grid that overruns its bitmask).  The emulator reports 2 SMs: the reach assertions are
evaluated for that count.  The 32800-row FAST frame (rows past 32767 in the blockwise and rank modes' packed cell keypoints) runs
here under VPPB_FAST_IMPL=warp only: the band path's 8200 CTAs of 256 emulated threads take over a minute, and the band and warp
paths feed the same blockwise and rank kernels."""
import glob
import json
import os
import subprocess
import sys

import pytest

from tests import detector_paths as dp

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
    rc, res, err = dp.run_child("emu", policy, tall=policy == "fast_warp", env=env)
    reports = "".join(open(f).read() for f in sorted(glob.glob(str(tmp_path / "ubsan*")) + glob.glob(str(tmp_path / "asan*"))))
    assert rc == 0 and res is not None, "child exited with %d:\n%s\n%s" % (rc, err[-3000:], reports[:4000])
    errors = [l for l in reports.splitlines() if "runtime error" in l or "ERROR: AddressSanitizer" in l or "SUMMARY: " in l]
    assert not errors, "sanitizer reports from the emulated kernels:\n" + reports[:4000]
    bad = dp.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    assert res["sms"] == 2
    unmet = dp.unmet(res, policy)
    assert not unmet, "the case tables no longer reach: " + "; ".join(unmet)


@pytest.mark.parametrize("policy", list(dp.POLICIES))
def test_detector_paths_emulated(built, tmp_path, policy):
    _run(tmp_path, policy, asan=False)


@pytest.mark.parametrize("policy", list(dp.POLICIES))
def test_detector_paths_emulated_asan(built, tmp_path, policy):
    if not _libasan():
        pytest.skip("libasan.so not available")
    _run(tmp_path, policy, asan=True)


def test_detector_policies_reach_every_kernel():
    """the policies' shares of the reach assertions together name every kernel instantiation both dispatches can choose"""
    union = set().union(*(dp.expected(p) for p in dp.POLICIES))
    assert dp.every_kernel() <= union, sorted(dp.every_kernel() - union)


def test_fast_dispatch_transcription():
    """the transcribed FAST dispatch on descriptors whose path is known: the library layout at 16 / 128 takes the band kernel,
    alignment 8 / a view at an odd column / VPPB_FAST_IMPL=warp the warp kernel, which loops over its grid beyond sms * 64 words"""
    from types import SimpleNamespace as NS

    lib = NS(nrows=9, ncols=2017, border=3, elem_bytes=1, align=128, base=4096, pitch=2304)  # 2017 + 2 x 128 rounded up to 128
    assert dp.fast_band_eligible(lib)
    assert dp.fast_plan(lib, "all", 1, True, 132, {})["kernels"] == ["band<1,mask>", "emit_bands"]
    assert dp.fast_plan(lib, "all", 1, True, 132, {"VPPB_FAST_IMPL": "warp"})["kernels"] == ["detect", "scan", "emit"]
    assert not dp.fast_band_eligible(NS(**dict(vars(lib), base=4096 + 5)))
    assert not dp.fast_band_eligible(NS(**dict(vars(lib), align=8, pitch=2017 + 16 + 7)))
    assert dp.fast_band_eligible(NS(**dict(vars(lib), align=16, pitch=2017 + 32 + 15)))
    big = NS(**dict(vars(lib), nrows=133, align=8, pitch=2040))  # 133 x 64 words > 132 x 64
    assert dp.fast_plan(big, "blockwise", 0, False, 132, {})["loops"] and not dp.fast_plan(NS(**dict(vars(big), nrows=132)), "rank", 0, False, 132, {})["loops"]


def test_lk_dispatch_transcription():
    from types import SimpleNamespace as NS

    lvl = NS(nrows=97, ncols=129, border=3, pitch=256)
    huge = NS(nrows=36, ncols=100, border=3, pitch=64 << 20)
    assert dp.lk_plan(9, 1, [lvl], [lvl], {}) == dict(kernel="v2", ppl=11, warps=4, grad="float", small=True)
    assert dp.lk_plan(3, 0, [lvl], [lvl], {"VPPB_LK_WARPS": "2"})["warps"] == 2
    assert dp.lk_plan(3, 0, [lvl], [lvl], {"VPPB_LK_WARPS": "3"})["warps"] == 4
    assert dp.lk_plan(13, 0, [lvl], [lvl], {})["kernel"] == "v1" and dp.lk_plan(13, 0, [lvl], [lvl], {})["ppl"] == 6
    assert dp.lk_plan(11, 0, [lvl], [lvl], {"VPPB_LK_V1": "1"}) == dict(kernel="v1", ppl=4, grad="int", small=True)
    assert dp.lk_plan(7, 0, [huge], [lvl], {}) == dict(kernel="v1", ppl=2, grad="int", small=False)
    assert [dp.v1_ppl(w) for w in range(1, 16, 2)] == [1, 1, 1, 2, 3, 4, 6, 8]
