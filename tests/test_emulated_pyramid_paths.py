"""The pyramid, Scharr and pyrlk_prepare kernels on every variant their dispatch can choose, on the CPU emulator (no GPU needed).

tests/pyramid_paths.py runs the stand-alone table (vppb_scharr_u8[_mirror], vppb_lowpass_sub2[_mirror] kinds 0 / 1 / 2,
vppb_copy2d_mirror) and the vppb_pyrlk_prepare table once per policy (the default, VPPB_PREPARE=fused, VPPB_PREPARE=streams) in a
child process; every output allocation must equal the oracle's bytes and keep its sentinel wherever the call must not write, and a
rejected call must return its exact code and write nothing.  The H100 counterpart is tests/test_gpu_pyramid_paths.py.

The emulated library is built with UBSan's alignment and bounds checks (a misaligned vector load of the v8 / px8 / u8 fast paths), and
the AddressSanitizer leg allocates every image at its exact size, so a read past the last row of a tight or view layout is reported.
The emulator reports 2 SMs and runs a cooperative launch on one CTA: every fused call of more than 256 items per phase runs its
grid-stride loops, and a grid barrier between several CTAs never runs here (the GPU module covers that)."""
import glob
import json
import os
import subprocess
import sys
from types import SimpleNamespace as D

import pytest

from tests import pyramid_paths as pp

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
    rc, res, err = pp.run_child("emu", policy, env=env)
    reports = "".join(open(f).read() for f in sorted(glob.glob(str(tmp_path / "ubsan*")) + glob.glob(str(tmp_path / "asan*"))))
    assert rc == 0 and res is not None, "child exited with %d:\n%s\n%s" % (rc, err[-3000:], reports[:4000])
    errors = [l for l in reports.splitlines() if "runtime error" in l or "ERROR: AddressSanitizer" in l or "SUMMARY: " in l]
    assert not errors, "sanitizer reports from the emulated kernels:\n" + reports[:4000]
    bad = pp.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    assert res["sms"] == 2
    unmet = pp.unmet(res, policy)
    assert not unmet, "the case tables no longer reach: " + "; ".join(unmet)


@pytest.mark.parametrize("policy", list(pp.POLICIES))
def test_pyramid_paths_emulated(built, tmp_path, policy):
    _run(tmp_path, policy, asan=False)


@pytest.mark.parametrize("policy", list(pp.POLICIES))
def test_pyramid_paths_emulated_asan(built, tmp_path, policy):
    if not _libasan():
        pytest.skip("libasan.so not available")
    _run(tmp_path, policy, asan=True)


def test_pyramid_policies_reach_every_path():
    """the policies' shares of the reach assertions together name every kernel, PREP_* kind and form of the dispatch"""
    union = set().union(*(pp.expected(p) for p in pp.POLICIES))
    assert pp.every_path() <= union, sorted(pp.every_path() - union)


def _img(nrows, ncols, elem=1, border=2, align=128, base=1 << 20, pitch=None):
    if pitch is None:
        bs = -(-border * elem // align) * align
        pitch = -(-(ncols * elem + 2 * bs) // align) * align
    return D(base=base, nrows=nrows, ncols=ncols, pitch=pitch, border=border, elem_bytes=elem, align=align)


def test_pyramid_dispatch_transcription():
    """the transcribed dispatch on descriptors whose path is known"""
    u8, v2 = _img(40, 56), _img(21, 29, elem=8)
    # Scharr: the v8 kernel on the library layout; the 1-pixel kernel on an 8-aligned output, an input view at an odd column, an
    # input with align < 16, or a row without room right of the last group
    assert pp.scharr_plan(u8, _img(40, 56, elem=8), 1, 1)["kernel"] == "k_scharr_u8_v8<1>"
    assert pp.scharr_plan(u8, _img(40, 56, elem=8, base=(1 << 20) + 8), 0, 0)["kernel"] == "k_scharr_u8<0>"
    assert pp.scharr_plan(_img(40, 56, base=(1 << 20) + 3), _img(40, 56, elem=8), 0, 1)["prep"] == "PREP_SCHARR_PX"
    assert pp.scharr_plan(_img(40, 56, border=1, align=8), _img(40, 56, elem=8), 0, 1)["kernel"] == "k_scharr_u8<0>"
    assert pp.scharr_plan(_img(7, 41, border=1, align=16, pitch=64), _img(7, 41, elem=8), 0, 1)["kernel"] == "k_scharr_u8<0>"
    assert pp.scharr_plan(_img(7, 40, border=1, align=16, pitch=64), _img(7, 40, elem=8), 0, 1)["kernel"] == "k_scharr_u8_v8<0>"
    assert pp.scharr_plan(_img(7, 40, border=0), _img(7, 40, elem=8), 0, 1)["rejected"] == pp.E_BORDER
    assert pp.scharr_plan(u8, _img(40, 56, elem=8, border=41), 0, 1)["rejected"] == pp.E_BORDER
    assert "rejected" not in pp.scharr_plan(u8, _img(40, 56, elem=8, border=41), 0, 0)  # the plain entry never writes the border
    # low-pass: the u8 fast path with tail items for an even parent (40 x 56 -> 21 x 29: the last row, 29 items, and the last column
    # without its corner, 20)
    p = pp.lowpass_plan(u8, _img(21, 29), 0, 1)
    assert (p["kernel"], p["tail_items"]) == ("k_lowpass_sub2_u8_fast", 29 + 20)
    assert pp.lowpass_plan(_img(41, 57), _img(21, 29), 0, 1)["tail_items"] == 0
    assert pp.lowpass_plan(_img(40, 56, align=16), _img(21, 29), 0, 1)["kernel"] == "k_lowpass_sub2<0>"
    assert pp.lowpass_plan(_img(3, 56), _img(2, 29), 0, 1)["kernel"] == "k_lowpass_sub2<0>"
    assert pp.lowpass_plan(u8, _img(21, 29, base=(1 << 20) + 4), 0, 1)["kernel"] == "k_lowpass_sub2<0>"
    assert pp.lowpass_plan(u8, _img(22, 29), 0, 1)["rejected"] == pp.E_ARG
    assert pp.lowpass_plan(_img(40, 56, border=1), _img(21, 29), 0, 1)["rejected"] == pp.E_BORDER
    assert pp.lowpass_plan(_img(41, 57, elem=8), v2, 2, 1)["aligned16"] == 1
    assert pp.lowpass_plan(_img(41, 57, elem=8, base=(1 << 20) + 8), v2, 1, 1)["aligned16"] == 0
    # copy + mirror: one launch on 16-byte aligned rows, copy + fill otherwise
    dst = _img(40, 56, border=3, base=1 << 24)
    assert pp.copy_plan(u8, dst)["kernel"] == "k_copy_mirror" and pp.copy_plan(u8, u8)["kernel"] == "fill"
    assert pp.copy_plan(_img(40, 56, base=(1 << 20) + 1), dst)["kernel"] == "copy+fill"
    # pyrlk_prepare: fused without a gradient pyramid, streams with one, fallback above 8 levels or off the library layout; fused
    # refuses with the reason; a rejected step rejects the call whatever the policy
    def sizes(n, b=2, elem=1):
        out, (r, c) = [], (40, 56)
        for l in range(n):
            out.append(_img(r, c, elem=elem, border=b, base=(1 << 24) * (l + 2)))
            r, c = 1 + r // 2, 1 + c // 2
        return out

    i1 = _img(40, 56, border=0)
    plan = lambda n, grad=None, env={}, b=2, i=i1: pp.prepare_plan(i, i, sizes(n, b), sizes(n, b), grad, n, 0, env, 132)
    assert plan(3)["form"] == "fused" and plan(3, grad=sizes(3, elem=8))["form"] == "streams"
    assert plan(3, grad=sizes(3, elem=8), env={"VPPB_PREPARE": "fused"})["form"] == "fused"
    assert plan(9)["fell_back"] == "more than 8 levels"
    assert plan(9, env={"VPPB_PREPARE": "fused"}) == dict(form="rejected", code=pp.E_ARG, reason="more than 8 levels")
    odd = _img(40, 56, border=0, base=(1 << 20) + 3)
    assert plan(3, i=odd)["fell_back"] == "the images do not have the library layout"
    assert plan(3, i=odd, env={"VPPB_PREPARE": "fused"})["reason"] == "the images do not have the library layout"
    assert plan(2, b=1)["code"] == pp.E_BORDER and plan(2, b=1, env={"VPPB_PREPARE": "fused"})["code"] == pp.E_BORDER
    assert plan(6, b=4)["code"] == pp.E_BORDER  # the sixth level is 3 x 3
    assert pp.prepare_plan(i1, i1, sizes(1), sizes(1), None, 0, 0, {}, 132)["code"] == pp.E_ARG
    # phases: copies, then (scharr | lowpass of the gradient) + the two u8 low-passes; without a gradient pyramid one phase fewer
    p = plan(3, grad=sizes(3, elem=8), env={"VPPB_PREPARE": "fused"})
    assert p["phases"] == [["PREP_COPY_MIRROR"] * 2, ["PREP_SCHARR_V8", "PREP_LP_U8_FAST", "PREP_LP_U8_FAST"],
                           ["PREP_LP_PX8", "PREP_LP_U8_FAST", "PREP_LP_U8_FAST"], ["PREP_LP_PX8"]]
    assert plan(3)["phases"] == [["PREP_COPY_MIRROR"] * 2, ["PREP_LP_U8_FAST"] * 2, ["PREP_LP_U8_FAST"] * 2]
    # 40 x 56 u8 copies with border 2: 40 * (3 + 8) + 2 * 2 * 60 + 2 * 40 * 2 = 840 items each; 1680 items ask for 7 CTAs
    assert plan(1)["most"] == 1680 and plan(1)["blocks"] == 7 and plan(1)["cap"] == "uncapped"
    tall = _img(18000, 31, border=0)
    assert pp.prepare_plan(tall, tall, [_img(18000, 31, base=1 << 30)], [_img(18000, 31, base=1 << 31)], None, 1, 0, {}, 132)["cap"] == "capped"
    tiny = _img(7, 9, border=0)
    assert pp.prepare_plan(tiny, tiny, [_img(7, 9, base=1 << 30)], [_img(7, 9, base=1 << 31)], None, 1, 0, {}, 2)["cap"] == "uncapped"
