"""The chamfer distance transform oracle (oracle/vpp_oracle_dt.c) against the reference's own header (oracle/_ref/libvppref_dt.so,
skipped where it was not built), bit for bit over whole output buffers, and against the numpy closed form of tests/dt_cases.py."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from tests import dt_cases as dc


def run_ref(case, kind):
    _, iv, op, ov, _ = dc.make_case(case)
    assert dc.reference().vppref_distance_transform(C.addressof(iv.desc), int(case[3] == "i32"), C.addressof(ov.desc), kind) == 0
    return op.buf.copy()


@pytest.fixture(scope="module")
def ref(built):
    if dc.reference() is None:
        pytest.skip("oracle/_ref/libvppref_dt.so not built (needs the reference tree)")
    return True


@pytest.mark.parametrize("case", dc.CASES, ids=dc.case_id)
def test_oracle_equals_reference(ref, case):
    exp, _ = dc.expected(case)
    for kind, buf in exp.items():
        assert np.array_equal(run_ref(case, kind), buf), (case, kind)


@pytest.mark.parametrize("case", dc.CASES, ids=dc.case_id)
def test_oracle_equals_closed_form(built, case):
    exp, a = dc.expected(case)
    b = case[4]
    for kind, buf in exp.items():
        _, _, op, ov, _ = dc.make_case(case)
        op.buf[:] = buf
        got = np.ndarray((ov.nrows + 2 * b, ov.ncols + 2 * b), np.int32, buffer=op.buf, offset=ov.origin - b * ov.pitch - 4 * b,
                         strides=(ov.pitch, 4))
        assert np.array_equal(got, dc.closed_form(a, kind, b)), (case, kind)


def test_oracle_rejects_bad_arguments(built):
    o = dc.oracle()
    a = dc.host_image(5, 6, "u8", 0, 16, fill=1)
    for kind, b, rc in ((3, 1, -3), (0, 0, -3), (4, 2, -2), (-1, 2, -2)):
        s = dc.host_image(5, 6, "i32", b, 16)
        assert o.vo_distance_transform(C.addressof(a.desc), C.addressof(s.desc), kind) == rc
        assert (s.buf == dc.SENTINEL).all()
    s = dc.host_image(5, 7, "i32", 2, 16)
    assert o.vo_distance_transform(C.addressof(a.desc), C.addressof(s.desc), 0) == -2


@settings(max_examples=300, deadline=None)
@given(nr=st.integers(1, 64), nc=st.integers(1, 64), pat=st.sampled_from(["random", "dense", "none", "all", "corner", "corner0", "sparse", "edges"]),
       pixel=st.sampled_from(["u8", "i32"]), border=st.integers(1, 4), seed=st.integers(0, 2 ** 16))
def test_oracle_sweep_against_reference_and_closed_form(built, nr, nc, pat, pixel, border, seed):
    case = (nr, nc, pat, pixel, border, 16, None)
    exp, a = dc.expected(case, seed)
    have_ref = dc.reference() is not None
    for kind, buf in exp.items():
        _, _, op, _, _ = dc.make_case(case, seed)
        frame = np.ndarray((nr + 2 * border, nc + 2 * border), np.int32, buffer=buf, offset=op.origin - border * op.pitch - 4 * border,
                           strides=(op.pitch, 4))
        assert np.array_equal(frame, dc.closed_form(a, kind, border)), (case, kind)
        if have_ref:
            _, iv, op2, ov, _ = dc.make_case(case, seed)
            assert dc.reference().vppref_distance_transform(C.addressof(iv.desc), int(pixel == "i32"), C.addressof(ov.desc), kind) == 0
            assert np.array_equal(op2.buf, buf), (case, kind)
