"""The streaming 5x5 box kernel's row bands on the GPU (`-m gpu`): tests/box_bands.py's case table under the default rows per
task and under VPPB_BOX_R = 21, each in a child process (the library reads the knob once per process).  Every output allocation
must equal a numpy 5x5 box of the input inside the domain and keep its sentinel outside it, and by the transcribed launch rule the
table must still reach one and several bands per image, ragged strips inside a band, more tasks than resident CTAs, the widest
band a CTA holds and rows one strip wider, a narrower last band, row-tile seams inside a band and (forced R) a short last band."""
import json

import pytest

from tests import box_bands as bb
from tests import box_geometry as bg

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("policy", list(bb.POLICIES))
def test_box_bands_gpu(gpu, policy):
    rc, res, err = bb.run_child("gpu", policy, big=True)
    assert rc == 0 and res is not None, "child exited with %d:\n%s" % (rc, err[-4000:])
    bad = bg.failures(res)
    assert not bad, "%d of %d runs differ, first ones:\n%s" % (len(bad), len(res["results"]), json.dumps(bad[:5], indent=1))
    unmet = bb.unmet_claims(res, policy)
    assert not unmet, "with %d SMs the case table no longer reaches: %s" % (res["sms"], "; ".join(unmet))
