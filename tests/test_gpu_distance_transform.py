"""The chamfer distance transforms on the H100 against the C oracle, bit for bit over whole output buffers: the border at its full
width becomes B, pitch padding and the parent pixels around a view keep their sentinel.  The shared table of tests/dt_cases.py,
each transform at 1080p, 4K and 8K on an edge map, on about 0.1 % zero pixels, on a single zero in a corner and on no zero at all,
out borders 1-4 at alignments 1, 4, 16 and 128 on views at odd columns, every error case, and tests/cpp/dt_tests.cu."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import dt_cases as dc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev(h):
    """device copy of a HostImage's whole buffer (256-byte aligned, so the host buffer's row alignment carries over)"""
    from vpp_b200 import ops

    return ops._DeviceBuffer(h.total).from_host(h.buf)


def _desc(raw, host_parent, h, align):
    from vpp_b200 import capi

    off = h.desc.base - host_parent.buf.ctypes.data
    return capi.VppbImg(raw.ptr + off, None, h.nrows, h.ncols, h.pitch, h.desc.border, h.elem, align)


def gpu_run(ip, iv, op, ov, kind, align):
    from vpp_b200 import capi, ops
    from vpp_b200.capi import lib

    di, do = _dev(ip), _dev(op)
    din, dout = _desc(di, ip, iv, align), _desc(do, op, ov, align)
    n = lib.vppb_distance_transform_workspace_bytes(iv.nrows, iv.ncols, kind)
    ws = ops._DeviceBuffer(n)
    rc = lib.vppb_distance_transform(C.byref(din), C.byref(dout), kind, ws.ptr, ws.nbytes, None)
    capi.check(lib.vppb_sync(None))
    return rc, do.to_host(np.uint8, op.total)


@pytest.mark.parametrize("case", dc.CASES, ids=dc.case_id)
def test_table(gpu, case):
    exp, _ = dc.expected(case)
    for kind, buf in exp.items():
        ip, iv, op, ov, _ = dc.make_case(case)
        rc, got = gpu_run(ip, iv, op, ov, kind, case[5])
        assert rc == 0
        assert np.array_equal(got, buf), (case, kind, np.argwhere(got != buf)[:8])


@pytest.mark.parametrize("align", [1, 4, 16, 128])
@pytest.mark.parametrize("border", [1, 2, 3, 4])
def test_views_borders_alignments(gpu, align, border):
    for view in ((0, 1), (3, 5), (1, 7)):
        case = (45, 77, "random", "u8", border, align, view)
        exp, _ = dc.expected(case, seed=border * 10 + align)
        for kind, buf in exp.items():
            ip, iv, op, ov, _ = dc.make_case(case, seed=border * 10 + align)
            rc, got = gpu_run(ip, iv, op, ov, kind, align)
            assert rc == 0 and np.array_equal(got, buf), (case, kind)


@pytest.mark.parametrize("size", [(1080, 1920), (2160, 3840), (4320, 7680)], ids=["1080p", "4k", "8k"])
@pytest.mark.parametrize("pat", ["edges", "sparse", "corner", "none"])
def test_large(gpu, size, pat):
    case = (size[0], size[1], pat, "u8", 2, 128, None)
    exp, a = dc.expected(case)
    for kind, buf in exp.items():
        ip, iv, op, ov, _ = dc.make_case(case)
        rc, got = gpu_run(ip, iv, op, ov, kind, 128)
        assert rc == 0 and np.array_equal(got, buf), (pat, size, kind)
        if pat == "corner" and kind in (2, 3):  # the far corner is further than B
            frame = np.ndarray((size[0], size[1]), np.int32, buffer=got, offset=op.origin, strides=(op.pitch, 4))
            assert frame[0, 0] == size[0] + size[1]


def test_errors_leave_the_output_untouched(gpu):
    from vpp_b200 import capi, ops
    from vpp_b200.capi import lib

    a = dc.host_image(6, 7, "u8", 0, 16, fill=0)
    for shape, pixel, b, kind, want in [((6, 7), "i32", 1, 3, capi.VPPB_E_BORDER), ((6, 7), "i32", 0, 0, capi.VPPB_E_BORDER),
                                        ((6, 7), "i32", 2, 4, capi.VPPB_E_ARG), ((6, 7), "i32", 2, -1, capi.VPPB_E_ARG),
                                        ((6, 8), "i32", 2, 0, capi.VPPB_E_ARG), ((6, 7), "u8", 2, 0, capi.VPPB_E_ARG)]:
        s = dc.host_image(shape[0], shape[1], pixel, b, 16)
        di, do = _dev(a), _dev(s)
        ws = ops._DeviceBuffer(1 << 16)
        rc = lib.vppb_distance_transform(C.byref(_desc(di, a, a, 16)), C.byref(_desc(do, s, s, 16)), kind, ws.ptr, ws.nbytes, None)
        assert rc == want, (shape, pixel, b, kind, rc)
        assert (do.to_host(np.uint8, s.total) == dc.SENTINEL).all()
    # input and output sharing memory: the input is the output's own buffer
    s = dc.host_image(6, 7, "i32", 2, 16)
    do = _dev(s)
    dout = _desc(do, s, s, 16)
    din = capi.VppbImg(dout.base, None, 6, 7, s.pitch, 0, 1, 16)
    ws = ops._DeviceBuffer(1 << 16)
    assert lib.vppb_distance_transform(C.byref(din), C.byref(dout), 0, ws.ptr, ws.nbytes, None) == capi.VPPB_E_ARG
    assert (do.to_host(np.uint8, s.total) == dc.SENTINEL).all()
    # too small a workspace
    assert lib.vppb_distance_transform(C.byref(_desc(_dev(a), a, a, 16)), C.byref(dout), 3, ws.ptr, 8, None) == capi.VPPB_E_ARG
    assert (do.to_host(np.uint8, s.total) == dc.SENTINEL).all()


def test_python_api(gpu):
    import vpp_b200 as vpp

    a = dc.pattern("random", 50, 61, 3)
    A = vpp.Image2d.from_host(a, "u8")
    for name, kind in dc.KINDS.items():
        S = getattr(vpp, name + "_distance_transform")(A)
        assert S.border == dc.REACH[kind] and S.pixel == "i32"
        assert np.array_equal(S.download(with_border=True), dc.closed_form(a, kind, S.border)), name


def test_cpp_dt_tests(gpu):
    exe = os.path.join(ROOT, "tests", "cpp", "_build", "dt_tests")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
