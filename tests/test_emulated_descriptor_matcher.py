"""The descriptor matcher and patch extraction kernels (end of vpp_b200/csrc/kpc.cu) on the CPU emulator of tests/emu (kernels compiled
by g++ and run thread by thread, warp ballots and shuffles included) against the C oracle and the numpy restatement.  Every case
runs with the threads of each launch in forward, reversed and shuffled order under UBSan, on descriptor rows at several
alignments and column offsets; the table runs again under AddressSanitizer with exact-size allocations in a subprocess; and the
C++ test tests/cpp/dm_tests.cu runs on the emulator."""
import ctypes as C
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import dm_cases as dc
from vpp_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UBSAN_LOG = os.path.join(ROOT, "tests", "emu", "_build", "ubsan.log")
ASAN = os.environ.get("VPPB_EMU_ASAN") == "1"
SCHEDULES = ["forward"] if ASAN else ["forward", "reversed", "shuffled"]


@pytest.fixture(autouse=True)
def no_sanitizer_reports():
    yield
    logs = glob.glob(UBSAN_LOG + "*")
    text = "".join(open(f).read() for f in logs)
    for f in logs:
        os.remove(f)
    assert not text, "UBSan report from an emulated kernel:\n" + text[:4000]


@pytest.fixture(scope="module")
def emu(built):
    path = dc.emu_lib(asan=ASAN)
    if not ASAN:
        os.environ["UBSAN_OPTIONS"] = "log_path=%s" % UBSAN_LOG
    lib = C.CDLL(path)
    I, VP, I32, I64 = C.POINTER(capi.VppbImg), C.c_void_p, C.c_int32, C.c_int64
    lib.vppb_match_bruteforce_sad.argtypes = [I, I, VP, I64, VP, VP, VP]
    lib.vppb_match_bruteforce_sad_workspace_bytes.argtypes = [I32, I32, I32]
    lib.vppb_match_bruteforce_sad_workspace_bytes.restype = I64
    lib.vppb_match_local_sad.argtypes = [I, I, VP, VP, I32, I32, VP, I64, VP, VP, VP]
    lib.vppb_match_local_sad_workspace_bytes.argtypes = [I32, I32, I32, I32, I32]
    lib.vppb_match_local_sad_workspace_bytes.restype = I64
    lib.vppb_extract_patches.argtypes = [I, VP, I32, I32, I, VP]
    lib.vppb_last_error.restype = C.c_char_p
    return lib


class Run:
    """set the emulator's thread order for one call"""

    def __init__(self, emu, schedule):
        self.emu, self.schedule = emu, schedule

    def __enter__(self):
        self.emu.vppb_emu_set_reverse(int(self.schedule == "reversed"))
        self.emu.vppb_emu_set_shuffle(4242 if self.schedule == "shuffled" else 0)

    def __exit__(self, *a):
        self.emu.vppb_emu_set_reverse(0)
        self.emu.vppb_emu_set_shuffle(0)


def exact_array(n, dtype, fill):
    size = np.dtype(dtype).itemsize
    raw = (C.c_ubyte * (max(1, n) * size))()
    a = np.ctypeslib.as_array(raw).view(dtype)[:n]
    a[:] = fill
    return raw, a


def layouts(elem):
    """(align, col0) of the descriptor rows: aligned, and views at odd columns with pitches that are not multiples of 4"""
    return [(128, 0), (4, 0)] + ([(1, 3), (2, 1)] if elem == 1 else [(16, 1)])


def emu_bruteforce(emu, q, t, align, col0, schedule):
    sq, st = dc.Strided(q, align, col0, exact=ASAN), dc.Strided(t, align, col0 + 1, exact=ASAN)
    n = emu.vppb_match_bruteforce_sad_workspace_bytes(len(q), len(t), q.shape[1])
    ws_raw, _ = exact_array(max(n // 8, 1), np.uint64, 0)
    ri, idx = exact_array(len(q), np.int32, -7)
    rd, dist = exact_array(len(q), np.int32, -7)
    with Run(emu, schedule):
        rc = emu.vppb_match_bruteforce_sad(C.byref(sq.desc), C.byref(st.desc), C.addressof(ws_raw), n, C.addressof(ri), C.addressof(rd), None)
    assert rc == 0, emu.vppb_last_error()
    return idx.copy(), dist.copy()


def emu_local(emu, q, t, qp, tp, R, s, align, col0, schedule):
    sq, st = dc.Strided(q, align, col0, exact=ASAN), dc.Strided(t, align, col0, exact=ASAN)
    n = emu.vppb_match_local_sad_workspace_bytes(len(q), len(t), q.shape[1], R, s)
    ws = np.zeros(n + 256, np.uint8)
    wp = ws.ctypes.data + (-ws.ctypes.data) % 256
    rqp, aqp = exact_array(2 * len(qp), np.int32, 0)
    rtp, atp = exact_array(2 * len(tp), np.int32, 0)
    aqp[:] = qp.reshape(-1)
    atp[:] = tp.reshape(-1)
    ri, idx = exact_array(len(q), np.int32, -7)
    rd, dist = exact_array(len(q), np.int32, -7)
    with Run(emu, schedule):
        rc = emu.vppb_match_local_sad(C.byref(sq.desc), C.byref(st.desc), C.addressof(rqp), C.addressof(rtp), R, s, wp, n, C.addressof(ri),
                                      C.addressof(rd), None)
    assert rc == 0, emu.vppb_last_error()
    return idx.copy(), dist.copy()


@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("case", dc.CASES, ids=dc.case_id)
def test_matchers_match_oracle(emu, case, schedule):
    q, t, qp, tp = dc.make(case)
    R, s = case[5], case[6]
    bi, bd = dc.oracle_bruteforce(q, t)
    li, ld = dc.oracle_local(q, t, qp, tp, R, s)
    for k, (align, col0) in enumerate(layouts(case[3])):
        if k and schedule != "forward":
            continue  # the thread orders on the aligned layout; the layouts in forward order
        gi, gd = emu_bruteforce(emu, q, t, align, col0, schedule)
        assert np.array_equal(gi, bi) and np.array_equal(gd, bd), (align, col0, np.argwhere((gi != bi) | (gd != bd))[:8])
        gi, gd = emu_local(emu, q, t, qp, tp, R, s, align, col0, schedule)
        assert np.array_equal(gi, li) and np.array_equal(gd, ld), (align, col0, np.argwhere((gi != li) | (gd != ld))[:8])


# (nrows, ncols, pixel, border, winsize)
PATCH_CASES = [(20, 30, "u8", 2, 5), (20, 30, "u8", 3, 4), (17, 9, "i32", 1, 3), (12, 40, "u8", 0, 1), (40, 50, "u8", 5, 11),
               (9, 9, "i32", 4, 8)]


@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("pc", PATCH_CASES, ids=lambda c: "%dx%d-%s-b%d-w%d" % c)
def test_extract_patches_matches_numpy(emu, pc, schedule):
    nr, nc, pixel, b, w = pc
    rng = np.random.default_rng(nr * nc + w)
    dt = np.uint8 if pixel == "u8" else np.int32
    frame = rng.integers(0, 256 if pixel == "u8" else 2 ** 31 - 1, (nr + 2 * b, nc + 2 * b)).astype(dt)
    img = dc.Strided(frame, 4 if pixel == "i32" else 1, 0, exact=ASAN)
    e = frame.itemsize
    desc = capi.VppbImg(img.base + b * img.pitch + b * e, None, nr, nc, img.pitch, b, e, 0)
    kps = rng.integers(-w - 3, max(nr, nc) + w + 3, (70, 2)).astype(np.int32)
    kps[:5] = [[0, 0], [nr - 1, nc - 1], [-b + w // 2, -b + w // 2], [nr - 1 + b - (w - 1 - w // 2), 0], [2 ** 31 - 1, -2 ** 31]]
    rk, ak = exact_array(2 * len(kps), np.int32, 0)
    ak[:] = kps.reshape(-1)
    out = dc.Strided(np.full((len(kps), w * w), 0x5A, dt), 4, 1 if pixel == "u8" else 0, exact=ASAN)
    with Run(emu, schedule):
        rc = emu.vppb_extract_patches(C.byref(desc), C.addressof(rk), len(kps), w, C.byref(out.desc), None)
    assert rc == 0, emu.vppb_last_error()
    got = np.stack([np.frombuffer(bytes(out.buf[out.base - out.buf.ctypes.data + r * out.pitch:][:w * w * e]), dt) for r in range(len(kps))])
    exp = dc.patches(frame, b, kps, w)
    assert np.array_equal(got, exp), np.argwhere(got != exp)[:8]
    assert (got[2] != 0).any() or (exp[2] == 0).all()


def test_errors_write_nothing(emu):
    q = dc.Strided(np.ones((4, 6), np.uint8))
    t = dc.Strided(np.ones((5, 6), np.uint8))
    t7 = dc.Strided(np.ones((5, 7), np.uint8))
    ti = dc.Strided(np.ones((5, 6), np.int32))
    ws = np.zeros(8192, np.uint8)
    wp = ws.ctypes.data + (-ws.ctypes.data) % 256
    idx, dist = np.full(4, -7, np.int32), np.full(4, -7, np.int32)
    pos = np.zeros((5, 2), np.int32)
    bad_elem = capi.VppbImg(q.desc.base, None, 4, 6, q.pitch, 0, 2, 0)
    BF = lambda a, b, n=64, w=wp, o=idx.ctypes.data: emu.vppb_match_bruteforce_sad(C.byref(a), C.byref(b), w, n, o, dist.ctypes.data, None)
    assert BF(q.desc, t7.desc) == capi.VPPB_E_ARG  # lengths differ
    assert BF(q.desc, ti.desc) == capi.VPPB_E_ARG  # element types differ
    assert BF(bad_elem, bad_elem) == capi.VPPB_E_ARG
    assert BF(q.desc, t.desc, n=31) == capi.VPPB_E_ARG  # workspace too small
    assert BF(q.desc, t.desc, w=None) == capi.VPPB_E_ARG
    assert BF(q.desc, t.desc, o=None) == capi.VPPB_E_ARG
    LM = lambda R, s, n=8192, a=q.desc, b=t.desc, qp=pos.ctypes.data: emu.vppb_match_local_sad(
        C.byref(a), C.byref(b), qp, pos.ctypes.data, R, s, wp, n, idx.ctypes.data, dist.ctypes.data, None)
    assert LM(10, 0) == capi.VPPB_E_ARG
    assert LM(-1, 10) == capi.VPPB_E_ARG
    assert LM(10, 10, n=64) == capi.VPPB_E_ARG
    assert LM(10, 10, qp=None) == capi.VPPB_E_ARG
    assert LM(10, 10, b=t7.desc) == capi.VPPB_E_ARG
    assert (idx == -7).all() and (dist == -7).all() and (ws == 0).all()
    img = dc.Strided(np.ones((10, 10), np.uint8))
    d1 = capi.VppbImg(img.base + 1 * img.pitch + 1, None, 8, 8, img.pitch, 1, 1, 0)
    out = dc.Strided(np.full((5, 9), 0x5A, np.uint8))
    PE = lambda im, w, o=out.desc: emu.vppb_extract_patches(C.byref(im), pos.ctypes.data, 5, w, C.byref(o), None)
    assert PE(d1, 5) == capi.VPPB_E_ARG  # output is 5 x 9, not 5 x 25
    out25 = dc.Strided(np.full((5, 25), 0x5A, np.uint8))
    assert PE(d1, 5, out25.desc) == capi.VPPB_E_BORDER  # border 1 < 2
    assert PE(d1, 0) == capi.VPPB_E_ARG
    assert (out.buf[out.base - out.buf.ctypes.data:] != 0).all() and (out25.buf != 0).all()


@pytest.mark.skipif(ASAN, reason="the C++ test runs once, without AddressSanitizer")
def test_cpp_dm_tests_on_the_emulator(emu):
    exe = dc.cpp_dm_emu()
    env = dict(os.environ, VPPB_EMU_LOG=os.path.join(ROOT, "tests", "emu", "_build", "emu_fail.log"), VPPB_EMU_SHUFFLE="77")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0 and "ALL OK" in r.stdout and "runtime error" not in r.stderr, r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.skipif(ASAN, reason="this is the driver of the AddressSanitizer run")
def test_under_address_sanitizer(built, tmp_path):
    libasan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan) or not os.path.exists(libasan):
        pytest.skip("libasan.so not available")
    log = str(tmp_path / "asan")
    env = dict(os.environ, VPPB_EMU_ASAN="1", VPPB_EMU_STACK_KB="96", LD_PRELOAD=libasan,
               ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:log_path=%s" % log)
    env.pop("UBSAN_OPTIONS", None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider"],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=1500)
    reports = "".join(open(f).read() for f in glob.glob(log + "*"))
    errors = [l for l in reports.splitlines() if "ERROR: AddressSanitizer" in l or "SUMMARY: AddressSanitizer" in l]
    assert r.returncode == 0 and not errors, r.stdout[-3000:] + r.stderr[-2000:] + reports[:4000]
    assert " passed" in r.stdout
