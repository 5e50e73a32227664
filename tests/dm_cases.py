"""Shared by the descriptor matcher tests: the case table, ctypes bindings of the C oracle (oracle/vpp_oracle_dm.c) and of the
reference's own headers (oracle/_ref/libvppref_dm.so), the numpy restatement of patch extraction, and the emulator builds.

A case is (nq, nt, D, elem, alphabet, R, s, layout): alphabet = number of distinct element values (1-4 make ties the rule
decides), or 0 for the full range; layout names how the positions are drawn (see positions())."""
import ctypes as C
import os
import sys

import numpy as np

from tests import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MAX = 2 ** 31 - 1


def descriptors(n, D, elem, alphabet, rng, dup=0):
    """(n, D) uint8 / int32 descriptors; `dup` of them copies of others"""
    if elem == 1:
        hi = 256 if alphabet == 0 else alphabet
        a = rng.integers(0, hi, (n, D)).astype(np.uint8)
        if alphabet:
            a = (a * (255 // max(1, alphabet - 1))).astype(np.uint8) if alphabet > 1 else a
    else:
        a = rng.integers(-10000, 10000, (n, D)).astype(np.int32) if alphabet == 0 else rng.integers(0, alphabet, (n, D)).astype(np.int32) * 1000
    if dup and n > 1:
        src = rng.integers(0, n, dup)
        dst = rng.integers(0, n, dup)
        a[dst] = a[src]
    return a


def positions(layout, n, rng, s, train):
    """(n, 2) int32 (row, col).  frame: inside 0..199; neg: queries reach -60 and 260 (trains in (-s, 200), which the reference
    takes); far: queries up to +-10^6; wide: 0..1999; excluded: as frame, with some trains at a coordinate <= -s (oracle and GPU only)"""
    if n == 0:
        return np.zeros((0, 2), np.int32)
    if layout == "frame" or (layout in ("neg", "far") and train):
        lo = -(s - 1) if layout == "neg" else 0
        return rng.integers(lo, 200, (n, 2)).astype(np.int32)
    if layout == "neg":
        return rng.integers(-60, 260, (n, 2)).astype(np.int32)
    if layout == "wide":  # cells past 255 in both coordinates at s = 1: two radix digits each
        return rng.integers(0, 2000, (n, 2)).astype(np.int32)
    if layout == "far":
        p = rng.integers(0, 200, (n, 2))
        k = rng.random(n) < 0.3
        p[k] = rng.integers(-10 ** 6, 10 ** 6, (int(k.sum()), 2))
        return p.astype(np.int32)
    assert layout == "excluded"
    p = rng.integers(0, 200, (n, 2))
    if train:
        k = rng.random(n) < 0.3
        p[k, rng.integers(0, 2)] = -s - rng.integers(0, 50, int(k.sum()))
    return p.astype(np.int32)


def make(case, seed=0):
    nq, nt, D, elem, alphabet, R, s, layout = case
    rng = np.random.default_rng(seed * 7919 + nq * 31 + nt * 17 + D)
    q = descriptors(nq, D, elem, alphabet, rng)
    t = descriptors(nt, D, elem, alphabet, rng, dup=nt // 5)
    if nq and nt and alphabet:  # some queries equal to trains: distance 0, in every cell
        k = min(nq, nt) // 4
        q[:k] = t[rng.integers(0, nt, k)]
    return q, t, positions(layout, nq, rng, s, False), positions(layout, nt, rng, s, True)


# (nq, nt, D, elem, alphabet, R, s, layout)
CASES = [
    (0, 10, 8, 1, 0, 30, 20, "frame"), (10, 0, 8, 1, 0, 30, 20, "frame"), (0, 0, 3, 4, 0, 5, 5, "frame"),
    (40, 50, 1, 1, 2, 30, 20, "frame"), (40, 50, 1, 4, 1, 30, 20, "frame"), (60, 70, 3, 1, 3, 0, 20, "neg"),
    (60, 70, 5, 1, 4, 10, 50, "neg"), (60, 90, 7, 4, 2, 45, 15, "neg"), (50, 80, 4, 1, 1, 25, 1, "frame"),
    (80, 100, 9, 1, 0, 1000, 7, "far"), (80, 100, 10, 4, 0, 10000, 300, "frame"), (70, 60, 16, 1, 2, 0, 1, "frame"),
    (100, 200, 10, 4, 0, 10000, 300, "frame"), (60, 80, 13, 1, 3, 20, 30, "excluded"), (60, 80, 6, 4, 2, 35, 25, "excluded"),
    (64, 130, 25, 1, 0, 40, 32, "neg"), (129, 65, 49, 1, 4, 50, 32, "frame"), (33, 200, 64, 1, 2, 60, 40, "far"),
    (40, 70, 130, 1, 3, 70, 64, "frame"), (30, 66, 129, 4, 2, 70, 64, "neg"), (20, 40, 300, 1, 0, 10 ** 6, 3, "frame"),
    (50, 60, 33, 4, 3, 90, 11, "excluded"),
    # more trains than one 1024-item tile of the cell sort, cells over several radix digits
    (24, 1500, 4, 1, 2, 40, 1, "wide"), (16, 1100, 3, 4, 0, 300, 2, "wide"),
]


def case_id(c):
    return "q%d-t%d-D%d-%s-a%d-R%d-s%d-%s" % (c[0], c[1], c[2], "u8" if c[3] == 1 else "i32", c[4], c[5], c[6], c[7])


# ---- host images ---------------------------------------------------------------------------------------------------------------
class Strided:
    """a's rows in host memory at row alignment `align` (pitch a multiple of it), as a view at column col0 of a wider parent: the
    emulator's "device" memory.  exact=True: one ctypes block that ends on the last byte of the last row (AddressSanitizer sees any
    access past it).  desc() is the vppb_img."""

    def __init__(self, a, align=16, col0=0, exact=False):
        from vpp_b200 import capi

        self.a = a
        n, D = a.shape
        e = a.itemsize
        self.pitch = max(1, -(-(col0 + D) * e // align) * align)
        need = self.pitch * max(n - 1, 0) + (col0 + D) * e
        if exact:
            self.raw = (C.c_ubyte * max(need, 1))()
            start = C.addressof(self.raw)
            self.buf = np.ctypeslib.as_array(self.raw)
        else:
            self.buf = np.full(need + 2 * align + 64, 0xCD, np.uint8)
            start = self.buf.ctypes.data + (-self.buf.ctypes.data) % align
        self.base = start + col0 * e
        off = self.base - self.buf.ctypes.data
        for r in range(n):
            self.buf[off + r * self.pitch:off + r * self.pitch + D * e] = np.frombuffer(a[r].tobytes(), np.uint8)
        self.desc = capi.VppbImg(self.base if n else None, None, n, D, self.pitch, 0, e, align)


def _vo(a):
    """vo_img over a C-contiguous 2-D array (kept alive by the caller)"""
    return orc.VoImg(a.ctypes.data, a.shape[0], a.shape[1], max(1, a.shape[1] * a.itemsize), 0, a.itemsize)


def oracle():
    o = orc.load()
    o.vo_match_bruteforce_sad.argtypes = [C.c_void_p] * 4
    o.vo_match_local_sad.argtypes = [C.c_void_p] * 4 + [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    return o


def oracle_omp():
    path = os.path.join(ROOT, "oracle", "_build", "libvpp_oracle_omp.so")
    o = C.CDLL(path)
    o.vo_match_bruteforce_sad.argtypes = [C.c_void_p] * 4
    o.vo_match_local_sad.argtypes = [C.c_void_p] * 4 + [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    return o


def oracle_bruteforce(q, t, lib=None):
    q, t = np.ascontiguousarray(q), np.ascontiguousarray(t)
    idx, dist = np.full(len(q), -7, np.int32), np.full(len(q), -7, np.int32)
    dq, dt = _vo(q), _vo(t)
    assert (lib or oracle()).vo_match_bruteforce_sad(C.addressof(dq), C.addressof(dt), idx.ctypes.data, dist.ctypes.data) == 0
    return idx, dist


def oracle_local(q, t, qp, tp, R, s, lib=None):
    q, t = np.ascontiguousarray(q), np.ascontiguousarray(t)
    qp, tp = np.ascontiguousarray(qp, np.int32), np.ascontiguousarray(tp, np.int32)
    idx, dist = np.full(len(q), -7, np.int32), np.full(len(q), -7, np.int32)
    dq, dt = _vo(q), _vo(t)
    assert (lib or oracle()).vo_match_local_sad(C.addressof(dq), C.addressof(dt), qp.ctypes.data, tp.ctypes.data, R, s,
                                                idx.ctypes.data, dist.ctypes.data) == 0
    return idx, dist


def reference(omp=False):
    """oracle/_ref/libvppref_dm[_omp].so (the reference's own headers), or None where it was not built"""
    path = os.path.join(ROOT, "oracle", "_ref", "libvppref_dm_omp.so" if omp else "libvppref_dm.so")
    if not os.path.exists(path):
        return None
    lib = C.CDLL(path)
    lib.vppref_match_bruteforce_sad.argtypes = [C.c_void_p] * 4
    lib.vppref_match_local_sad.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def ref_bruteforce(q, t, lib=None):
    q, t = np.ascontiguousarray(q), np.ascontiguousarray(t)
    idx, dist = np.full(len(q), -7, np.int32), np.full(len(q), -7, np.int32)
    dq, dt = _vo(q), _vo(t)
    assert (lib or reference()).vppref_match_bruteforce_sad(C.addressof(dq), C.addressof(dt), idx.ctypes.data, dist.ctypes.data) == 0
    return idx, dist


def ref_local(q, t, qp, tp, R, s, approximation=1, lib=None):
    q, t = np.ascontiguousarray(q), np.ascontiguousarray(t)
    qp, tp = np.ascontiguousarray(qp, np.int32), np.ascontiguousarray(tp, np.int32)
    idx, dist = np.full(len(q), -7, np.int32), np.full(len(q), -7, np.int32)
    dq, dt = _vo(q), _vo(t)
    assert (lib or reference()).vppref_match_local_sad(C.addressof(dq), C.addressof(dt), qp.ctypes.data, tp.ctypes.data, R, s,
                                                       approximation, idx.ctypes.data, dist.ctypes.data) == 0
    return idx, dist


def patches(img_with_border, border, kps, winsize):
    """numpy restatement of patch extraction: img_with_border is the (nr + 2b, nc + 2b) frame; row k = the window centred on
    kps[k], row-major from element 0, or zeros where it leaves the domain plus border"""
    nr, nc = img_with_border.shape[0] - 2 * border, img_with_border.shape[1] - 2 * border
    h = winsize // 2
    out = np.zeros((len(kps), winsize * winsize), img_with_border.dtype)
    for k, (r, c) in enumerate(np.asarray(kps, np.int64)):
        if r - h >= -border and r - h + winsize - 1 <= nr - 1 + border and c - h >= -border and c - h + winsize - 1 <= nc - 1 + border:
            out[k] = img_with_border[r - h + border:r - h + border + winsize, c - h + border:c - h + border + winsize].reshape(-1)
    return out


# ---- the CPU emulator ---------------------------------------------------------------------------------------------------------
def emu_lib(asan=False):
    """tests/emu/_build/libvppb_emu[_asan].so: the emulated library, matcher kernels included (kpc.cu)"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    return build_emu.build(asan=asan)


def cpp_dm_emu():
    """tests/cpp/dm_tests.cu built against the emulated library"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    return build_emu.build_cpp_test("dm_tests")
