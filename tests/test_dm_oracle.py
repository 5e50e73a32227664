"""The SAD descriptor matcher oracle (oracle/vpp_oracle_dm.c) against the reference's own headers (oracle/_ref/libvppref_dm.so,
skipped where it was not built).  Brute force: index and distance exactly.  Grid-local at _approximation = 1: the distance on
every query, and the index wherever the reference's choice is determined - its winning cell holds a single train at the minimum
(inside a cell the reference orders ties by an unstable std::sort)."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from tests import dm_cases as dc


@pytest.fixture(scope="module")
def ref(built):
    if dc.reference() is None:
        pytest.skip("oracle/_ref/libvppref_dm.so not built (needs the reference tree)")
    return dc.reference()


def determined(t, tp, s, q, i, d, j_ref):
    """True when the reference's pick for query i is forced: the winning cell holds one train at distance d"""
    cell = tuple(np.asarray(tp[j_ref]) // s)
    cells = np.stack([tp[:, 0] // s, tp[:, 1] // s], 1)
    ok = (tp[:, 0] > -s) & (tp[:, 1] > -s) & (cells[:, 0] == cell[0]) & (cells[:, 1] == cell[1])
    dd = np.abs(t[ok].astype(np.int64) - q[i].astype(np.int64)).sum(1)
    return int((dd == d).sum()) == 1


def check_local(ref, q, t, qp, tp, R, s):
    oi, od = dc.oracle_local(q, t, qp, tp, R, s)
    ri, rd = dc.ref_local(q, t, qp, tp, R, s, lib=ref)
    assert np.array_equal(od, rd), np.argwhere(od != rd)[:8]
    assert np.array_equal(oi < 0, ri < 0)
    tpc = np.where(tp < 0, 0, tp)  # C division: (-s, 0) truncates to cell 0
    for i in np.nonzero((oi != ri) & (oi >= 0))[0]:
        assert not determined(t, tpc, s, q, i, od[i], ri[i]), (i, oi[i], ri[i], od[i])
    return oi, od


def ref_can_run(nq, tp, R, s):
    """the reference takes no train at a coordinate <= -s, and it visits every cell of every window (grid_index.hh:61): keep
    that walk small"""
    cells = (2 * R // s + 2) ** 2
    return cells * max(nq, 1) <= 4 * 10 ** 6 and (len(tp) == 0 or ((tp[:, 0] > -s) & (tp[:, 1] > -s)).all())


@pytest.mark.parametrize("case", dc.CASES, ids=dc.case_id)
def test_oracle_equals_reference(ref, case):
    q, t, qp, tp = dc.make(case)
    R, s = case[5], case[6]
    if len(t):
        assert [np.array_equal(a, b) for a, b in zip(dc.oracle_bruteforce(q, t), dc.ref_bruteforce(q, t, lib=ref))] == [True, True]
    if ref_can_run(len(q), tp, R, s):
        check_local(ref, q, t, qp, tp, R, s)


def test_reference_own_case(ref):
    """the reference's tests/descriptor_matcher.cc: 100 x 10 and 200 x 10 int descriptors in [0, 10000), positions in [0, 1000),
    R = 10000, s = 300: every query matched, at the global minimum"""
    rng = np.random.default_rng(1)
    q = rng.integers(0, 10000, (100, 10)).astype(np.int32)
    t = rng.integers(0, 10000, (200, 10)).astype(np.int32)
    qp = rng.integers(0, 1000, (100, 2)).astype(np.int32)
    tp = rng.integers(0, 1000, (200, 2)).astype(np.int32)
    bi, bd = dc.oracle_bruteforce(q, t)
    assert [np.array_equal(a, b) for a, b in zip((bi, bd), dc.ref_bruteforce(q, t, lib=ref))] == [True, True]
    full = np.abs(q[:, None, :].astype(np.int64) - t[None]).sum(2)
    assert np.array_equal(bd, full.min(1)) and np.array_equal(bi, full.argmin(1))
    li, ld = check_local(ref, q, t, qp, tp, 10000, 300)
    assert (li >= 0).all() and np.array_equal(ld, full.min(1))


def test_trains_beyond_minus_s_are_never_matched(built):
    q = np.zeros((3, 4), np.uint8)
    t = np.zeros((3, 4), np.uint8)
    qp = np.array([[0, 0], [5, 5], [-20, -20]], np.int32)
    tp = np.array([[-10, 3], [2, -10], [-9, -9]], np.int32)  # s = 10: the first two are excluded, (-9, -9) is cell (0, 0)
    idx, dist = dc.oracle_local(q, t, qp, tp, 0, 10)
    assert idx.tolist() == [2, 2, -1] and dist.tolist() == [0, 0, dc.INT_MAX]


def test_oracle_rejects_bad_arguments(built):
    import ctypes as C

    o = dc.oracle()
    q, t = np.zeros((2, 3), np.uint8), np.zeros((2, 4), np.uint8)
    idx = np.full(2, -7, np.int32)
    dq, dt = dc._vo(q), dc._vo(t)
    assert o.vo_match_bruteforce_sad(C.addressof(dq), C.addressof(dt), idx.ctypes.data, idx.ctypes.data) == -2
    p = np.zeros((2, 2), np.int32)
    dt = dc._vo(q)
    for R, s in ((0, 0), (-1, 5)):
        assert o.vo_match_local_sad(C.addressof(dq), C.addressof(dt), p.ctypes.data, p.ctypes.data, R, s, idx.ctypes.data, idx.ctypes.data) == -2
    assert (idx == -7).all()


@settings(max_examples=150, deadline=None)
@given(nq=st.integers(0, 40), nt=st.integers(0, 60), D=st.integers(1, 12), elem=st.sampled_from([1, 4]), alphabet=st.integers(0, 4),
       R=st.sampled_from([0, 1, 5, 17, 40, 100, 10000]), s=st.sampled_from([1, 2, 7, 16, 33, 300]),
       layout=st.sampled_from(["frame", "neg", "far"]), seed=st.integers(0, 2 ** 16))
def test_oracle_sweep_against_reference(ref, nq, nt, D, elem, alphabet, R, s, layout, seed):
    case = (nq, nt, D, elem, alphabet, R, s, layout)
    q, t, qp, tp = dc.make(case, seed)
    if nt:
        assert [np.array_equal(a, b) for a, b in zip(dc.oracle_bruteforce(q, t), dc.ref_bruteforce(q, t, lib=ref))] == [True, True]
    if ref_can_run(nq, tp, R, s):
        check_local(ref, q, t, qp, tp, R, s)
