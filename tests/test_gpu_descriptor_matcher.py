"""The descriptor matchers and patch extraction on the H100 (end of vpp_b200/csrc/kpc.cu) against the C oracle: the case table of
tests/dm_cases.py, descriptor views at odd columns and row alignments 1..128, realistic sizes checked against the OpenMP build of
the oracle, train counts on both sides of the brute-force kernel's tile and split boundaries, FAST keypoints and extracted patches
of two shifted 1080p scenes, and every error case with the outputs' sentinels intact."""
import ctypes as C
import os

import numpy as np
import pytest

import vpp_b200 as vpp
from tests import dm_cases as dc
from vpp_b200 import capi
from vpp_b200.ops import _DeviceBuffer

pytestmark = pytest.mark.gpu
BF_T, BF_Q = 64, 128  # kpc.cu's trains per tile and queries per CTA


def view_image(a, align, col0):
    """Image2d view at column col0 of a parent whose rows have alignment `align`, holding `a`"""
    n, D = a.shape
    pixel = "u8" if a.dtype == np.uint8 else "i32"
    parent = vpp.Image2d(n, D + col0, pixel, aligned=align)
    v = parent | vpp.Box2d((0, col0), (n - 1, col0 + D - 1))
    v.upload(a)
    return v


@pytest.mark.parametrize("case", dc.CASES, ids=dc.case_id)
def test_table_matches_oracle(gpu, case):
    q, t, qp, tp = dc.make(case)
    R, s = case[5], case[6]
    bi, bd = dc.oracle_bruteforce(q, t)
    li, ld = dc.oracle_local(q, t, qp, tp, R, s)
    gi, gd = vpp.bruteforce_sad_matcher(q, t)
    assert np.array_equal(gi, bi) and np.array_equal(gd, bd)
    gi, gd = vpp.local_sad_descriptor_matcher(q, t, qp, tp, search_radius=R, cell_width=s)
    assert np.array_equal(gi, li) and np.array_equal(gd, ld)


@pytest.mark.parametrize("align", [1, 2, 4, 8, 16, 32, 64, 128])
def test_views_at_every_alignment(gpu, align):
    rng = np.random.default_rng(align)
    for elem, D in ((1, 37), (1, 64), (4, 10)):
        if elem == 4 and align < 4:
            continue
        q = dc.descriptors(300, D, elem, 3, rng)
        t = dc.descriptors(500, D, elem, 3, rng, dup=50)
        qp, tp = rng.integers(0, 300, (300, 2)).astype(np.int32), rng.integers(0, 300, (500, 2)).astype(np.int32)
        for col0 in ((0, 1, 3) if elem == 1 else (0, 1)):
            qv, tv = view_image(q, align, col0), view_image(t, align, col0 + 2)
            assert [np.array_equal(a, b) for a, b in zip(vpp.bruteforce_sad_matcher(qv, tv), dc.oracle_bruteforce(q, t))] == [True, True]
            got = vpp.local_sad_descriptor_matcher(qv, tv, qp, tp, search_radius=40, cell_width=25)
            assert [np.array_equal(a, b) for a, b in zip(got, dc.oracle_local(q, t, qp, tp, 40, 25))] == [True, True]


@pytest.mark.parametrize("elem,D", [(1, 25), (1, 49), (1, 64), (1, 128), (4, 10), (1, 131), (4, 37)])
def test_realistic_sizes_against_the_openmp_oracle(gpu, elem, D):
    rng = np.random.default_rng(D)
    n = 10000
    q, t = dc.descriptors(n, D, elem, 0, rng), dc.descriptors(n, D, elem, 0, rng, dup=500)
    q[:100] = t[rng.integers(0, n, 100)]
    omp = dc.oracle_omp()
    bi, bd = dc.oracle_bruteforce(q, t, lib=omp)
    gi, gd = vpp.bruteforce_sad_matcher(q, t)
    assert np.array_equal(gi, bi) and np.array_equal(gd, bd), np.argwhere((gi != bi) | (gd != bd))[:8]
    qp, tp = rng.integers(0, 1080, (n, 2)).astype(np.int32), rng.integers(0, 1080, (n, 2)).astype(np.int32)
    li, ld = dc.oracle_local(q, t, qp, tp, 100, 32, lib=omp)
    gi, gd = vpp.local_sad_descriptor_matcher(q, t, qp, tp, search_radius=100, cell_width=32)
    assert np.array_equal(gi, li) and np.array_equal(gd, ld)


def test_train_counts_around_tiles_and_splits(gpu):
    """trains on both sides of a tile (64) and of the split spans the launch policy picks for 1000 and 10000 queries"""
    from vpp_b200.capi import lib
    rng = np.random.default_rng(5)
    omp = dc.oracle_omp()
    for nq in (1000, 10000):
        nqb = -(-nq // BF_Q)
        counts = {1, 63, 64, 65, 127, 129}
        for sm in (114, 132):
            want = -(-16 * sm // nqb)
            counts |= {want * BF_T - 1, want * BF_T, want * BF_T + 1, 2 * want * BF_T + 1}
        for nt in sorted(counts):
            q, t = dc.descriptors(nq, 49, 1, 4, rng), dc.descriptors(nt, 49, 1, 4, rng, dup=nt // 4)
            gi, gd = vpp.bruteforce_sad_matcher(q, t)
            bi, bd = dc.oracle_bruteforce(q, t, lib=omp)
            assert np.array_equal(gi, bi) and np.array_equal(gd, bd), (nq, nt)


def test_fast_keypoints_and_patches_on_shifted_1080p_scenes(gpu):
    from tests.scenes import rectangles_scene

    a = rectangles_scene(1080, 1920, seed=11)
    b = np.roll(a, (4, -7), axis=(0, 1))
    imgs, kps = [], []
    for x in (a, b):
        G = vpp.Image2d.from_host(x, "u8", border=3)
        vpp.fill_border_mirror(G)
        imgs.append(G)
        kps.append(vpp.fast9(G, 20))
    assert min(len(k) for k in kps) > 500
    pats = [vpp.extract_patches(G, k, 7) for G, k in zip(imgs, kps)]
    for G, k, P in zip(imgs, kps, pats):
        frame = G.download(with_border=True)
        assert np.array_equal(P.download(), dc.patches(frame, 3, k, 7))
    q, t = pats[1].download(), pats[0].download()
    omp = dc.oracle_omp()
    for R in (32, 100):
        li, ld = dc.oracle_local(q, t, kps[1], kps[0], R, 32, lib=omp)
        gi, gd = vpp.local_sad_descriptor_matcher(pats[1], pats[0], kps[1], kps[0], search_radius=R, cell_width=32)
        assert np.array_equal(gi, li) and np.array_equal(gd, ld)
        assert (gd == 0).mean() > 0.3  # the shifted scene's corners find themselves
    # patches of a keypoint whose window leaves the border are zero, inside ones are the window
    edge = np.array([[0, 0], [-1, 5], [1079, 1919], [1080 + 3 - 3, 10], [540, 960]], np.int32)
    P = vpp.extract_patches(imgs[0], edge, 7).download()
    assert np.array_equal(P, dc.patches(imgs[0].download(with_border=True), 3, edge, 7))
    assert (P[1] == 0).all() and (P[3] == 0).all()


def test_errors_write_nothing(gpu):
    from vpp_b200.capi import lib

    q = vpp.Image2d.from_host(np.ones((4, 6), np.uint8), "u8")
    t7 = vpp.Image2d.from_host(np.ones((5, 7), np.uint8), "u8")
    ti = vpp.Image2d.from_host(np.ones((5, 6), np.int32), "i32")
    t = vpp.Image2d.from_host(np.ones((5, 6), np.uint8), "u8")
    ws = _DeviceBuffer(8192)
    ws.from_host(np.full(8192, 0xAB, np.uint8))
    out = _DeviceBuffer(32)
    out.from_host(np.full(32, 0x5A, np.uint8))
    pos = _DeviceBuffer(40).from_host(np.zeros(10, np.int32))
    o_idx, o_dist = out.ptr, out.ptr + 16
    BF = lambda a, b, n=64, w=ws.ptr, o=o_idx: lib.vppb_match_bruteforce_sad(a.ptr(), b.ptr(), w, n, o, o_dist, None)
    assert BF(q, t7) == capi.VPPB_E_ARG
    assert BF(q, ti) == capi.VPPB_E_ARG
    assert BF(q, t, n=31) == capi.VPPB_E_ARG
    assert BF(q, t, w=None) == capi.VPPB_E_ARG
    assert BF(q, t, o=None) == capi.VPPB_E_ARG
    LM = lambda R, s, n=8192, b=t, qp=pos.ptr: lib.vppb_match_local_sad(q.ptr(), b.ptr(), qp, pos.ptr, R, s, ws.ptr, n, o_idx, o_dist, None)
    assert LM(10, 0) == capi.VPPB_E_ARG
    assert LM(-1, 10) == capi.VPPB_E_ARG
    assert LM(10, 10, n=64) == capi.VPPB_E_ARG
    assert LM(10, 10, qp=None) == capi.VPPB_E_ARG
    assert LM(10, 10, b=t7) == capi.VPPB_E_ARG
    img = vpp.Image2d(8, 8, "u8", border=1)
    p9 = vpp.Image2d(5, 9, "u8")
    p25 = vpp.Image2d(5, 25, "u8")
    vpp.fill_with_border(p9, 0x5A)
    vpp.fill_with_border(p25, 0x5A)
    assert lib.vppb_extract_patches(img.ptr(), pos.ptr, 5, 5, p9.ptr(), None) == capi.VPPB_E_ARG
    assert lib.vppb_extract_patches(img.ptr(), pos.ptr, 5, 5, p25.ptr(), None) == capi.VPPB_E_BORDER
    assert lib.vppb_extract_patches(img.ptr(), pos.ptr, 5, 0, p25.ptr(), None) == capi.VPPB_E_ARG
    capi.check(lib.vppb_sync(None))
    assert (out.to_host(np.uint8, 32) == 0x5A).all() and (ws.to_host(np.uint8, 8192) == 0xAB).all()
    assert (p9.download() == 0x5A).all() and (p25.download() == 0x5A).all()


def test_cpp_dm_tests(gpu):
    import subprocess

    exe = os.path.join(dc.ROOT, "tests", "cpp", "_build", "dm_tests")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
