"""The 5x5 box byte kernels at every geometry their launch policy can choose, on the CPU emulator (no GPU needed).

tests/box_geometry.py runs one case table (strip widths, row counts around every forced R, output and input layouts,
TMA-eligible views, row tiles, batches of up to 257 images) through the single, _batch and _tiles entry points, once per
policy (VPPB_BOX_SINGLE / _TH / _R) in a child process, because the library reads those knobs once per process.  Every output
allocation must equal a numpy 5x5 box of the input buffer inside the domain and still hold its sentinel outside it.

The emulator reports 2 SMs (6 resident streaming CTAs), so here most streaming launches give a CTA several tasks; the
H100 counterpart is tests/test_gpu_box_geometry.py.  The emulated library is built with UBSan's alignment and bounds checks:
a report fails the policy (a 16-byte store to an output without 16-byte alignment is silent on x86 otherwise).  The
AddressSanitizer leg catches a view or a row tile whose reads leave its allocation.

Two hypothesis sweeps (in this process, default policy) add rows ending around the streaming kernel's strips, and batches in
which every image has its own content."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

from tests import box_geometry as bg
from tests.test_emulated_property import SCALE, SET, _box_oracle, vpp  # noqa: F401  (the emulated library, loaded in this process)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# rows around the streaming kernel's strips: u8 rows of 2016 bytes are one strip of G = 126 groups (a 2048-byte TMA box), 2017 and 2033
# bytes two strips of 64 groups (the last with 63 groups or a 1-byte last group), 4032 bytes two strips of 126, 4033 bytes three
# (85, 85, 83); vuchar3 rows of 672 / 673 pixels are 2016 / 2019 bytes
STREAM_WIDTHS = [672, 673, 2016, 2017, 2032, 2033, 4032, 4033]


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
    rc, res, err = bg.run_child("emu", policy, env=env)
    reports = "".join(open(f).read() for f in sorted(glob.glob(str(tmp_path / "ubsan*")) + glob.glob(str(tmp_path / "asan*"))))
    assert rc == 0 and res is not None, "child exited with %d:\n%s\n%s" % (rc, err[-3000:], reports[:4000])
    errors = [l for l in reports.splitlines() if "runtime error" in l or "ERROR: AddressSanitizer" in l or "SUMMARY: " in l]
    assert not errors, "sanitizer reports from the emulated kernels:\n" + reports[:4000]
    bad = bg.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    assert res["sms"] == 2
    unmet = bg.unmet_claims(res, multi_task=True)
    assert not unmet, "the case table no longer reaches: " + "; ".join(unmet)


@pytest.mark.parametrize("policy", list(bg.POLICIES))
def test_box_geometry_emulated(built, tmp_path, policy):
    _run(tmp_path, policy, asan=False)


@pytest.mark.parametrize("policy", list(bg.POLICIES))
def test_box_geometry_emulated_asan(built, tmp_path, policy):
    if not _libasan():
        pytest.skip("libasan.so not available")
    _run(tmp_path, policy, asan=True)


@settings(max_examples=int(40 * SCALE), **SET)
@given(nr=st.integers(2, 70), nc=st.one_of(st.integers(2, 60), st.integers(325, 340), st.sampled_from(STREAM_WIDTHS)), n=st.integers(2, 35),
       pix=st.sampled_from(["vuchar3", "u8"]), seed=st.integers(0, 1000))
def test_box_batch_distinct_images(vpp, nr, nc, n, pix, seed):
    """the streaming kernel over a batch in which every image has its own content, rows around its strips included: a kernel that
    mixed up the tensor maps or outputs of two images of the batch fails"""
    ch = 3 if pix == "vuchar3" else 1
    r = np.random.default_rng(seed)
    imgs = [r.integers(0, 256, (nr, nc) + ((ch,) if ch > 1 else ()), dtype=np.uint8) for _ in range(n)]
    srcs, dsts = [], []
    for img in imgs:
        S = vpp.Image2d.from_host(img, pix, border=2)
        vpp.fill_border_mirror(S)
        srcs.append(S)
        dsts.append(vpp.Image2d(nr, nc, pix))
    vpp.box5x5_batch(srcs, dsts)
    for i in range(n):
        assert np.array_equal(dsts[i].download(), _box_oracle(imgs[i], pix)), (i, nr, nc, n)


@settings(max_examples=int(30 * SCALE), **SET)
@given(nr=st.one_of(st.integers(2, 40), st.sampled_from([47, 48, 49, 63, 64, 65])), nc=st.sampled_from(STREAM_WIDTHS), pix=st.sampled_from(["vuchar3", "u8"]),
       seed=st.integers(0, 1000))
def test_box_single_at_stream_strip_widths(vpp, nr, nc, pix, seed):
    """single frames (the tile kernel) whose rows end around the streaming kernel's strips"""
    ch = 3 if pix == "vuchar3" else 1
    data = np.random.default_rng(seed).integers(0, 256, (nr, nc) + ((ch,) if ch > 1 else ()), dtype=np.uint8)
    S = vpp.Image2d.from_host(data, pix, border=2)
    vpp.fill_border_mirror(S)
    D = vpp.Image2d(nr, nc, pix)
    vpp.box5x5(S, D)
    assert np.array_equal(D.download(), _box_oracle(data, pix)), (nr, nc, pix)
