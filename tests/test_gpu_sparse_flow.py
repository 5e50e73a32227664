"""vpp_b200.sparse_optical_flow / vppb_sparse_flow_u8 on the H100 against the composite oracle of tests/sof_cases.py: the case table in
both modes, a 1080p and a 4K pair against the OpenMP build of the oracle, a sanity figure on a textured 1080p scene shifted by a whole
number of FAST cells, the rejected calls with the outputs' sentinels intact, and the C++ overloads of vpp/algorithms/optical_flow.hh
(tests/cpp/sof_tests.cu) against the Python entry."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import vpp_b200 as vpp
from tests import dm_cases as dc
from tests import sof_cases as sc
from vpp_b200 import capi
from vpp_b200.ops import _DeviceBuffer

pytestmark = pytest.mark.gpu


def device_frame(frame, b):
    """Image2d holding `frame` (border included) with border b"""
    img = vpp.Image2d(frame.shape[0] - 2 * b, frame.shape[1] - 2 * b, "u8", border=b)
    img.upload(frame, with_border=True)
    return img


def run(f1, f2, b, case, subpixelic):
    o = sc.opts(case)
    return vpp.sparse_optical_flow(device_frame(f1, b), device_frame(f2, b), keypoints=sc.keypoints(case), detector_th=o["th"], block_size=o["bs"],
                                   winsize=o["ws"], search_radius=o["R"], cell_width=o["s"], subpixelic=subpixelic, lk_iterations=o["it"],
                                   nscales=o["nscales"])


def assert_same(got, exp):
    assert len(got[0]) == len(exp[0]), (len(got[0]), len(exp[0]))
    for g, e, nm in zip(got, exp, ("position", "flow", "distance", "valid")):
        same = np.array_equal(g.view(np.uint32), np.asarray(e, np.float32).view(np.uint32)) if nm == "flow" else np.array_equal(g, e)
        assert same, (nm, int((g != e).sum()), np.argwhere(g != e)[:8])


@pytest.mark.parametrize("subpixelic", [False, True], ids=["integer", "subpixel"])
@pytest.mark.parametrize("case", sc.CASES, ids=sc.case_id)
def test_table_matches_composite_oracle(gpu, case, subpixelic):
    f1, f2 = sc.frames(case)
    assert_same(run(f1, f2, case["b"], case, subpixelic), sc.oracle_sparse_flow(f1, f2, case["b"], case, subpixelic))


def big_pair(nr, nc, b, shift, seed):
    from tests.scenes import rectangles_scene, warp

    a = rectangles_scene(nr + 2 * b, nc + 2 * b, seed=seed).astype(np.float64)
    f2 = np.clip(np.round(warp(a, -shift[0], -shift[1])), 0, 255).astype(np.uint8)
    return a.astype(np.uint8), f2


@pytest.mark.parametrize("subpixelic", [False, True], ids=["integer", "subpixel"])
@pytest.mark.parametrize("size", [(1080, 1920), (2160, 3840)], ids=["1080p", "4K"])
def test_realistic_sizes_against_the_openmp_oracle(gpu, size, subpixelic):
    nr, nc = size
    b = 5
    f1, f2 = big_pair(nr, nc, b, (3, -2), seed=nr)
    # a detector threshold and matcher grid that keep the serial-per-query oracle match within seconds (the default R = 100,
    # s = 300 puts thousands of trains in every window: tools/sof_bench.py measures that one)
    case = dict(id="big", nr=nr, nc=nc, b=b, th=20, bs=10, R=50, s=100)
    from tests import oracle as orc

    exp = sc.oracle_sparse_flow(f1, f2, b, case, subpixelic, lib=orc.load(omp=True), omp=dc.oracle_omp())
    got = run(f1, f2, b, case, subpixelic)
    assert len(got[0]) > 1000
    assert_same(got, exp)


def textured_pair(shift, b=5, seed=17):
    from tests.scenes import smooth_noise, warp

    a = smooth_noise(1080 + 2 * b, 1920 + 2 * b, seed=seed, sigmas=(1.0, 2.5, 6.0))
    return np.clip(np.round(a * 255), 0, 255).astype(np.uint8), np.clip(np.round(warp(a, -shift[0], -shift[1]) * 255), 0, 255).astype(np.uint8)


def test_sanity_on_a_shifted_textured_scene(gpu):
    """A shift by whole FAST cells (block_size 5) maps interior cells onto cells of the same content, so their blockwise maxima
    correspond: most integer flows are the shift.  The subpixel mode's median error on a (10.4, -5.3) shift is printed."""
    b = 5
    f1, f2 = textured_pair((10, -5), b)
    pos, flow, dist, valid = vpp.sparse_optical_flow(device_frame(f1, b), device_frame(f2, b))
    frac = float((flow[valid] == np.float32([10, -5])).all(1).mean())
    print("\ninteger mode, shift (10, -5): %d keypoints, %d valid, %.3f of the valid flows equal the shift" % (len(pos), valid.sum(), frac))
    assert valid.sum() > 1000 and frac >= 0.9
    g1, g2 = textured_pair((10.4, -5.3), b)
    pos, flow, dist, valid = vpp.sparse_optical_flow(device_frame(g1, b), device_frame(g2, b), subpixelic=True)
    ok = valid & ~(flow == -1).all(1) & ~(flow == 0).all(1)
    err = np.hypot(flow[ok, 0] - 10.4, flow[ok, 1] + 5.3)
    print("subpixel mode, shift (10.4, -5.3): %d keypoints, %d converged, median error %.3f px" % (len(pos), ok.sum(), float(np.median(err))))
    assert ok.sum() > 1000


def test_errors_write_nothing(gpu):
    from vpp_b200.capi import lib

    case = sc.CASES[0]
    f1, f2 = sc.frames(case)
    b = case["b"]
    nr, nc = f1.shape[0] - 2 * b, f1.shape[1] - 2 * b
    i1, i2 = device_frame(f1, b), device_frame(f2, b)
    small = device_frame(f1[1:-1, 1:-1], b - 1)
    other = device_frame(f1[:-2], b)
    P = sc.params(case, False)
    nbytes = lib.vppb_sparse_flow_workspace_bytes(nr, nc, C.byref(P), -1)
    ws = _DeviceBuffer(nbytes).from_host(np.full(nbytes, 0xAB, np.uint8))
    out = _DeviceBuffer(64 * 21).from_host(np.full(64 * 21, 0x5A, np.uint8))
    kp = _DeviceBuffer(16).from_host(np.array([[5, 5], [10, 10]], np.int32))
    o = out.ptr

    def call(a=i1, bimg=i2, p=P, k=None, n=0, nb=nbytes, cap=64):
        cnt = C.c_int32(-1)
        rc = lib.vppb_sparse_flow_u8(a.ptr(), bimg.ptr(), C.byref(p), k, n, ws.ptr, nb, o, o + 64 * 8, o + 64 * 16, o + 64 * 20, cap, C.byref(cnt), None)
        return rc, cnt.value

    sp = lambda **kw: sc.params(dict(case, **kw), True)
    assert call(a=small)[0] == capi.VPPB_E_BORDER
    assert call(bimg=small)[0] == capi.VPPB_E_BORDER
    assert call(bimg=other)[0] == capi.VPPB_E_ARG
    for w in (10, 3, 17, 4):
        assert call(p=sp(ws=w))[0] == capi.VPPB_E_ARG, w
    assert call(p=sp(nscales=9))[0] == capi.VPPB_E_ARG
    assert call(nb=nbytes - 1)[0] == capi.VPPB_E_ARG
    assert call(k=kp.ptr, n=-1)[0] == capi.VPPB_E_ARG
    rc, cnt = call(k=kp.ptr, n=2, cap=1)
    assert rc == capi.VPPB_E_CAPACITY and cnt == 2
    capi.check(lib.vppb_sync(None))
    assert (out.to_host(np.uint8, 64 * 21) == 0x5A).all() and (ws.to_host(np.uint8, nbytes) == 0xAB).all()
    rc, cnt = call(cap=1)
    assert rc == capi.VPPB_E_CAPACITY and cnt > 1
    assert (out.to_host(np.uint8, 64 * 21) == 0x5A).all()


def test_cpp_overloads_equal_the_python_entry(gpu, tmp_path):
    case = dict(id="cpp", nr=90, nc=130, b=5, scene="noise", shift=(2.4, -1.2), kps="edge", seed=9)
    f1, f2 = sc.frames(case)
    kps = sc.keypoints(case)
    nr, nc, b = case["nr"], case["nc"], case["b"]
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(src, "wb") as fh:
        fh.write(np.array([nr, nc, b, len(kps)], np.int32).tobytes() + f1.tobytes() + f2.tobytes() + np.ascontiguousarray(kps, np.int32).tobytes())
    exe = os.path.join(dc.ROOT, "tests", "cpp", "_build", "sof_tests")
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    rec = np.dtype([("i", "<i4"), ("r", "<i4"), ("c", "<i4"), ("fr", "<f4"), ("fc", "<f4"), ("d", "<i4")])
    raw = open(dst, "rb").read()
    off = 0
    I1, I2 = device_frame(f1, b), device_frame(f2, b)
    for sub in (False, True):
        common = dict(winsize=9, search_radius=40, cell_width=30, subpixelic=sub, nscales=2)
        for k in (None, kps):
            n = int(np.frombuffer(raw, np.int32, 1, off)[0])
            got = np.frombuffer(raw, rec, n, off + 4)
            off += 4 + n * rec.itemsize
            pos, flow, dist, valid = vpp.sparse_optical_flow(I1, I2, keypoints=k, **common)
            idx = np.flatnonzero(valid)
            assert n == len(idx), (sub, k is None)
            assert np.array_equal(got["r"], pos[idx, 0]) and np.array_equal(got["c"], pos[idx, 1]) and np.array_equal(got["d"], dist[idx])
            if k is None:
                assert np.array_equal(got["fr"], flow[idx, 0]) and np.array_equal(got["fc"], flow[idx, 1])
            else:  # new_position = K1[i] + flow, in float
                assert np.array_equal(got["i"], idx)
                assert np.array_equal(got["fr"], pos[idx, 0].astype(np.float32) + flow[idx, 0])
                assert np.array_equal(got["fc"], pos[idx, 1].astype(np.float32) + flow[idx, 1])
