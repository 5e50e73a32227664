"""The streaming 5x5 box kernel's row bands on the CPU emulator (no GPU needed): tests/box_bands.py's case table, without its
large cases, under the default rows per task and under VPPB_BOX_R = 21, each in a child process.  The emulator reports 2 SMs, so
most launches give a CTA several tasks.  The emulated library is built with UBSan's alignment and bounds checks; a report fails
the policy.  The H100 counterpart is tests/test_gpu_box_bands.py."""
import glob
import json
import os
import sys

import pytest

from tests import box_bands as bb
from tests import box_geometry as bg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("policy", list(bb.POLICIES))
def test_box_bands_emulated(built, tmp_path, policy):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    build_emu.build(asan=False)
    env = dict(os.environ, VPPB_EMU_LOG=str(tmp_path / "emu_fail.log"), UBSAN_OPTIONS="log_path=%s" % (tmp_path / "ubsan"))
    env.pop("VPPB_EMU_ASAN", None)
    rc, res, err = bb.run_child("emu", policy, env=env)
    reports = "".join(open(f).read() for f in sorted(glob.glob(str(tmp_path / "ubsan*"))))
    assert rc == 0 and res is not None, "child exited with %d:\n%s\n%s" % (rc, err[-3000:], reports[:4000])
    assert not [l for l in reports.splitlines() if "runtime error" in l], "sanitizer reports from the emulated kernels:\n" + reports[:4000]
    bad = bg.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    assert res["sms"] == 2
    unmet = bb.unmet_claims(res, policy)
    assert not unmet, "the case table no longer reaches: " + "; ".join(unmet)
