"""lbp_transform, local_maxima_filter and the oriented LK matcher on every path their dispatch can choose, and the workspace alignment
of every entry point that takes one, on the CPU emulator (no GPU needed).

tests/n4_paths.py runs the case tables in a child process: lbp and local_maxima_filter results must equal the C oracle's exactly over
their whole allocations (sentinels outside the domain, and past the local_maxima_filter workspace), oriented LK flows and errors bit
for bit.  The child runs once under the library built with UBSan's alignment and bounds checks and once under AddressSanitizer.  The
emulator reports 2 SMs, and the reach assertions are evaluated for that count: local_maxima_filter's grid-stride regime starts above
8 x 256 x 2 items here.  The H100 counterpart is tests/test_gpu_n4_paths.py.

Left to the GPU leg: the 8K frames of lbp and local_maxima_filter (the 4K ones already reach every path here), and the u8 frame of
more than 2 GiB, which needs that much memory three times over."""
import glob
import json
import os
import subprocess
import sys

import pytest

from tests import n4_paths as n4

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _libasan():
    p = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return p if os.path.isabs(p) and os.path.exists(p) else None


def _run(tmp_path, asan):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    build_emu.build(asan=asan)  # here, not in the child: the ASan child runs with libasan preloaded
    env = dict(os.environ, VPPB_EMU_LOG=str(tmp_path / "emu_fail.log"), UBSAN_OPTIONS="log_path=%s" % (tmp_path / "ubsan"))
    if asan:
        env.update(VPPB_EMU_ASAN="1", VPPB_EMU_STACK_KB="96", LD_PRELOAD=_libasan(),
                   ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:log_path=%s" % (tmp_path / "asan"))
    else:
        env.pop("VPPB_EMU_ASAN", None)
    rc, res, err = n4.run_child("emu", no_8k=True, env=env)
    reports = "".join(open(f).read() for f in sorted(glob.glob(str(tmp_path / "ubsan*")) + glob.glob(str(tmp_path / "asan*"))))
    assert rc == 0 and res is not None, "child exited with %d:\n%s\n%s" % (rc, err[-3000:], reports[:4000])
    errors = [l for l in reports.splitlines() if "runtime error" in l or "ERROR: AddressSanitizer" in l or "SUMMARY: " in l]
    assert not errors, "sanitizer reports from the emulated kernels:\n" + reports[:4000]
    bad = n4.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    assert res["sms"] == 2
    unmet = n4.unmet(res)
    assert not unmet, "the case tables no longer reach: " + "; ".join(unmet)


def test_n4_paths_emulated(built, tmp_path):
    _run(tmp_path, asan=False)


def test_n4_paths_emulated_asan(built, tmp_path):
    if not _libasan():
        pytest.skip("libasan.so not available")
    _run(tmp_path, asan=True)


def test_lbp_dispatch_transcription():
    """<true> needs both images' pixel (0,0) and pitch 16-byte aligned; inside it a width that is not a multiple of 16 leaves a
    ragged group to the scalar path"""
    from types import SimpleNamespace as NS

    a = NS(base=4096 + 128, pitch=1280, nrows=9, ncols=1000)
    assert n4.lbp_plan(a, a) == dict(kernel="true", vector_groups=True, ragged=True, rows_mod4=1)
    assert n4.lbp_plan(a, NS(**dict(vars(a), base=4096 + 4)))["kernel"] == "false"
    assert n4.lbp_plan(NS(**dict(vars(a), pitch=1004)), a)["kernel"] == "false"
    assert n4.lbp_plan(NS(**dict(vars(a), ncols=15)), a)["vector_groups"] is False
    assert n4.lbp_plan(NS(**dict(vars(a), ncols=32)), a)["ragged"] is False


def test_lmf_regime_bounds():
    """single trip up to one CTA of 256 threads per SM, grid-stride beyond 8 such CTAs per SM, whatever the occupancy between"""
    assert n4.lmf_plan(132, 256 * 16, 1, 132)["regime"] == "single-trip"  # 132 x 256 items
    assert n4.lmf_plan(133, 256 * 16, 1, 132)["regime"] == "either"
    assert n4.lmf_plan(8 * 132, 256 * 16, 4, 132)["regime"] == "either"
    assert n4.lmf_plan(8 * 132 + 1, 256 * 16, 4, 132) == dict(pix="int", items=(8 * 132 + 1) * 256, regime="grid-stride")
    assert n4.lmf_plan(2160, 3840, 1, 132)["regime"] == "grid-stride"  # 4K: 518400 items > 270336
    assert n4.lmf_plan(1, 17, 1, 2)["items"] == 2


def test_oriented_dispatch_covers_every_instantiation():
    """every odd window maps onto one of the six PPL instantiations, and the windows 1 .. 15 reach all of them"""
    assert [n4.oriented_plan(w, 1, 1, 132)["ppl"] for w in range(1, 16, 2)] == [1, 1, 1, 2, 3, 4, 6, 8]
    assert {n4.oriented_plan(w, 1, 1, 132)["ppl"] for w in range(1, 16, 2)} == set(n4.ORIENTED_PPLS)
    assert not n4.oriented_plan(5, 0, 4 * 16 * 132, 132)["beyond_wave"] and n4.oriented_plan(5, 0, 4 * 16 * 132 + 1, 132)["beyond_wave"]


def test_chain_scenes_alternate():
    """the chains of local_maxima_filter's table are what they claim: strictly decreasing, one link a successor of the one before,
    at least 1000 links for int and 254 for u8"""
    import numpy as np

    for pix, L in (("int", 1000), ("u8", 254)):
        for d in ("N", "NW", "NE", "W"):
            a = n4.chain_scene(d, pix)
            bg = a.min()
            pts = sorted(zip(*np.nonzero(a != bg)), key=lambda p: -a[p])
            assert len(pts) >= L, (pix, d)
            for (r0, c0), (r1, c1) in zip(pts, pts[1:]):
                assert a[r0, c0] > a[r1, c1] and ((r1 - r0, c1 - c0) in ((1, 0), (1, 1), (1, -1)) if d != "W" else (r1, c1) == (r0, c0 + 1)), (pix, d)
