"""The 5x5 box byte kernels at every geometry their launch policy can choose, on the GPU (`-m gpu`).

tests/box_geometry.py runs one case table through the single, _batch and _tiles entry points, once per policy
(VPPB_BOX_SINGLE / _TH / _R) in a child process, because the library reads those knobs once per process; every output
allocation must equal a numpy 5x5 box of the input buffer inside the domain and still hold its sentinel outside it.  The
default policy also runs the frames on either side of the 96 MiB rule (vuchar3 4400 x 7680 takes the streaming kernel,
4320 x 7680 the tile kernel) and u8 (40, 7680) x 128, which the default R sends to 1024 tasks on an H100's 396 CTAs.

From the SM count the child reports, the test checks with a transcription of the launch rules (bg.plan) that the table still
reaches what it was written for: G = 126, a ragged last strip, the NB = 1 streaming kernel on a plain frame and, under the
default and the forced R = 16 / 21 policies, more tasks than resident CTAs (a CTA's producer carrying its ring of stages
from one task into the next)."""
import json

import pytest

from tests import box_geometry as bg

pytestmark = pytest.mark.gpu

# policies under which the table gives a CTA several tasks on an H100 (132 SMs, 396 CTAs): 1024, 832 and 640 tasks in one launch
MULTI_TASK = ("default", "r16", "r21")


@pytest.mark.parametrize("policy", list(bg.POLICIES))
def test_box_geometry_gpu(gpu, policy):
    rc, res, err = bg.run_child("gpu", policy, big=policy == "default")
    assert rc == 0 and res is not None, "child exited with %d:\n%s" % (rc, err[-4000:])
    print("policy %s: %d SMs, %d runs" % (policy, res["sms"], len(res["results"])))
    bad = bg.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    unmet = bg.unmet_claims(res, multi_task=policy in MULTI_TASK)
    assert not unmet, "with %d SMs the case table no longer reaches: %s" % (res["sms"], "; ".join(unmet))
