"""Shared by the distance transform tests: the case table, the input patterns, the numpy closed form, ctypes bindings of the
C oracle (oracle/vpp_oracle_dt.c) and of the reference's own header (oracle/_ref/libvppref_dt.so), and the emulator builds.

Closed form (DESIGN §3.7): every border pixel is B = nrows + ncols, every domain pixel min(B, gauge(p - z)) over the zero pixels z,
with a = max(|dr|, |dc|), b = min(|dr|, |dc|): d4 a + b, d8 a, d3-4 3a + b, d5-7-11 5a + b if a >= 2b else 4a + 3b."""
import ctypes as C
import os
import sys

import numpy as np

from tests import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = {"d4": 0, "d8": 1, "d3_4": 2, "d5_7_11": 3}
REACH = {0: 1, 1: 1, 2: 1, 3: 2}
SENTINEL = 0xCD


def gauge(kind, dr, dc):
    a = np.maximum(np.abs(dr), np.abs(dc)).astype(np.int64)
    b = np.minimum(np.abs(dr), np.abs(dc)).astype(np.int64)
    if kind == 0:
        return a + b
    if kind == 1:
        return a
    if kind == 2:
        return 3 * a + b
    return np.where(a >= 2 * b, 5 * a + b, 4 * a + 3 * b)


def closed_form(a, kind, border):
    """(nrows + 2 border, ncols + 2 border) int32 frame of the transform of `a` (zeros are a == 0)"""
    nr, nc = a.shape
    B = nr + nc
    out = np.full((nr + 2 * border, nc + 2 * border), B, np.int64)
    zr, zc = np.nonzero(a == 0)
    if len(zr):
        rr, cc = np.mgrid[0:nr, 0:nc]
        best = np.full((nr, nc), B, np.int64)
        for i in range(0, len(zr), 256):
            g = gauge(kind, rr[None] - zr[i:i + 256, None, None], cc[None] - zc[i:i + 256, None, None])
            best = np.minimum(best, g.min(axis=0))
        out[border:border + nr, border:border + nc] = best
    return out.astype(np.int32)


def pattern(name, nr, nc, seed, pixel="u8"):
    """input image: zeros placed by `name`, other pixels non-zero (negative and large values too for i32)"""
    rng = np.random.default_rng(seed)
    dt = np.uint8 if pixel == "u8" else np.int32
    if pixel == "u8":
        a = rng.integers(1, 256, (nr, nc)).astype(dt)
    else:
        a = rng.integers(-2 ** 31, 2 ** 31, (nr, nc), dtype=np.int64)
        a[a == 0] = 7
        a = a.astype(dt)
    if name == "sparse":  # about 0.1 % zero pixels
        a[rng.random((nr, nc)) < 0.001] = 0
    elif name == "random":
        a[rng.random((nr, nc)) < 0.05] = 0
    elif name == "dense":
        a[rng.random((nr, nc)) < 0.6] = 0
    elif name == "all":
        a[:] = 0
    elif name == "corner":  # one zero at the bottom-right corner: the longest lines, B reached for d3-4 and d5-7-11
        a[-1, -1] = 0
    elif name == "corner0":
        a[0, 0] = 0
    elif name == "edges":  # an edge map: zeros on the outlines of a few rectangles and a circle
        for _ in range(6):
            r0, c0 = rng.integers(0, nr), rng.integers(0, nc)
            r1, c1 = min(nr - 1, r0 + rng.integers(1, max(2, nr // 3))), min(nc - 1, c0 + rng.integers(1, max(2, nc // 3)))
            a[r0, c0:c1 + 1] = 0
            a[r1, c0:c1 + 1] = 0
            a[r0:r1 + 1, c0] = 0
            a[r0:r1 + 1, c1] = 0
        rr, cc = np.mgrid[0:nr, 0:nc]
        d = np.hypot(rr - nr / 2, cc - nc / 2)
        a[np.abs(d - min(nr, nc) / 3) < 0.5] = 0
    else:
        assert name == "none", name
    return a


# (nrows, ncols, pattern, input pixel, out border, alignment, view).  view: None, or (r0, c0) of the output view inside a parent
# with margin 3 on every side, with the input a view at odd column offset 3 of a wider parent
CASES = []
for _nr, _nc in [(1, 1), (1, 2), (2, 1), (1, 37), (37, 1), (2, 5), (3, 4), (4, 3), (5, 9), (16, 40), (33, 70), (31, 33), (64, 65),
                 (65, 64), (97, 130), (130, 17), (200, 3), (3, 200)]:
    for _pat in ("random", "dense", "corner", "none"):
        CASES.append((_nr, _nc, _pat, "u8", 2, 128, None))
    CASES.append((_nr, _nc, "all", "i32", 3, 16, None))
    CASES.append((_nr, _nc, "random", "i32", 4, 4, None))
    CASES.append((_nr, _nc, "edges", "u8", 2, 1, (3, 5)))
CASES += [(70, 90, "random", "u8", 1, 128, None), (70, 90, "corner0", "i32", 1, 1, (1, 3)), (128, 256, "sparse", "u8", 2, 16, None),
          (257, 300, "edges", "u8", 3, 128, None), (96, 64, "corner", "i32", 2, 128, (2, 1)),
          # rows of several 256-column tiles of k_dt_rows, with zeros in some tiles only
          (3, 1500, "sparse", "u8", 2, 128, None), (2, 1300, "corner0", "u8", 1, 4, None), (40, 1100, "edges", "u8", 2, 16, (1, 3)),
          (5, 777, "corner", "i32", 2, 128, None)]


def case_id(c):
    return "%dx%d-%s-%s-b%d-a%d%s" % (c[0], c[1], c[2], c[3], c[4], c[5], "-view" if c[6] else "")


# ---- the C oracle and the reference ------------------------------------------------------------------------------------------
def oracle():
    o = orc.load()
    o.vo_distance_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    o.vo_distance_transform.restype = C.c_int
    return o


def reference():
    """oracle/_ref/libvppref_dt.so (the reference's own header), or None where it was not built"""
    path = os.path.join(ROOT, "oracle", "_ref", "libvppref_dt.so")
    if not os.path.exists(path):
        return None
    lib = C.CDLL(path)
    lib.vppref_distance_transform.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    lib.vppref_distance_transform.restype = C.c_int
    return lib


def host_image(nr, nc, pixel, border, aligned, fill=SENTINEL):
    """orc.HostImage whose whole buffer (border and pitch padding included) starts as `fill`"""
    h = orc.HostImage(nr, nc, pixel, border=border, aligned=aligned)
    h.buf[:] = fill
    return h


def subview(parent, r0, c0, nr, nc):
    """HostImage-like view of rows r0.. and cols c0.. of `parent`, keeping the parent's border (as vppb_subimage)"""
    v = orc.HostImage.__new__(orc.HostImage)
    v.__dict__.update(parent.__dict__)
    v.nrows, v.ncols = nr, nc
    v.origin = parent.origin + r0 * parent.pitch + c0 * parent.elem
    v.desc = orc.VoImg(parent.buf.ctypes.data + v.origin, nr, nc, parent.pitch, parent.border, parent.elem)
    return v


def make_case(case, seed=0):
    """(input parent, input view, output parent, output view): the views are the parents themselves without `view`"""
    nr, nc, pat, pixel, b, al, view = case
    a = pattern(pat, nr, nc, seed + nr * 1000 + nc, pixel)
    if view:
        ip = host_image(nr + 2, nc + 6, pixel, 1, al, fill=0)  # zero pixels around the view must not count
        iv = subview(ip, 1, 3, nr, nc)
        iv.set(a)
        r0, c0 = view
        op = host_image(nr + r0 + b + 3, nc + c0 + b + 3, "i32", b, al)
        op.view()[...] = -5  # parent pixels, some of which are the view's border
        ov = subview(op, r0, c0, nr, nc)
        return ip, iv, op, ov, a
    ip = host_image(nr, nc, pixel, 2, al, fill=0)  # the input border is never read: zeros there would change the result
    ip.set(a)
    op = host_image(nr, nc, "i32", b, al)
    return ip, ip, op, op, a


def expected(case, seed=0):
    """{kind: whole output buffer after the oracle} for every kind the case's border allows, and the input array"""
    out = {}
    for kind in range(4):
        if case[4] < REACH[kind]:
            continue
        _, iv, op, ov, a = make_case(case, seed)
        assert oracle().vo_distance_transform(C.addressof(iv.desc), C.addressof(ov.desc), kind) == 0
        out[kind] = op.buf.copy()
    return out, a


# ---- the CPU emulator ---------------------------------------------------------------------------------------------------------
def emu_lib(asan=False):
    """tests/emu/_build/libvppb_emu[_asan].so: the emulated library, distance transform kernels included"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    return build_emu.build(asan=asan)


def cpp_dt_emu():
    """tests/cpp/dt_tests.cu built against the emulated library"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    return build_emu.build_cpp_test("dt_tests")
