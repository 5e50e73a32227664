"""vppb_sparse_flow_u8 (end of vpp_b200/csrc/sdof.cu, and the entries it chains) on the CPU emulator of tests/emu, against the composite
oracle of tests/sof_cases.py: every case of the table in both modes, with the threads of each launch in forward and shuffled order,
under UBSan; the table again under AddressSanitizer in a subprocess; and the rejected calls, which must leave every output and
workspace byte as it was."""
import ctypes as C
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import dm_cases as dc
from tests import sof_cases as sc
from vpp_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UBSAN_LOG = os.path.join(ROOT, "tests", "emu", "_build", "ubsan_sof.log")
ASAN = os.environ.get("VPPB_EMU_ASAN") == "1"
SCHEDULES = ["forward"] if ASAN else ["forward", "shuffled"]


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
    PP = C.POINTER(capi.VppbSofParams)
    lib.vppb_sparse_flow_workspace_bytes.argtypes = [I32, I32, PP, I32]
    lib.vppb_sparse_flow_workspace_bytes.restype = I64
    lib.vppb_sparse_flow_u8.argtypes = [I, I, PP, VP, I32, VP, I64, VP, VP, VP, VP, I32, C.POINTER(I32), VP]
    lib.vppb_alloc.argtypes = [I, I32, I32, I32, I32, I32]
    lib.vppb_free.argtypes = [I]
    lib.vppb_upload.argtypes = [I, VP, I64, C.c_int, VP]
    lib.vppb_last_error.restype = C.c_char_p
    return lib


class Run:
    def __init__(self, emu, schedule):
        self.emu, self.schedule = emu, schedule

    def __enter__(self):
        self.emu.vppb_emu_set_shuffle(4242 if self.schedule == "shuffled" else 0)

    def __exit__(self, *a):
        self.emu.vppb_emu_set_shuffle(0)


def exact_array(n, dtype, fill):
    raw = (C.c_ubyte * (max(1, n) * np.dtype(dtype).itemsize))()
    a = np.ctypeslib.as_array(raw).view(dtype)[:n]
    a[:] = fill
    return raw, a


class EmuImage:
    """frame (border included) in an emulated vppb_alloc'ed image with the library layout"""

    def __init__(self, emu, frame, b):
        self.emu = emu
        self.desc = capi.VppbImg()
        nr, nc = frame.shape[0] - 2 * b, frame.shape[1] - 2 * b
        assert emu.vppb_alloc(C.byref(self.desc), nr, nc, 1, b, 128) == 0
        f = np.ascontiguousarray(frame)
        self.f = f
        assert emu.vppb_upload(C.byref(self.desc), f.ctypes.data + b * f.shape[1] + b, f.shape[1], 1, None) == 0

    def __del__(self):
        self.emu.vppb_free(C.byref(self.desc))


def emu_sparse_flow(emu, f1, f2, b, case, subpixelic, schedule, capacity=None):
    P = sc.params(case, subpixelic)
    ck = sc.keypoints(case)
    n = -1 if ck is None else len(ck)
    nbytes = emu.vppb_sparse_flow_workspace_bytes(f1.shape[0] - 2 * b, f1.shape[1] - 2 * b, C.byref(P), n)
    assert nbytes > 0
    ws = capi.VppbImg()
    assert emu.vppb_alloc(C.byref(ws), 1, nbytes, 1, 0, 256) == 0
    try:
        i1, i2 = EmuImage(emu, f1, b), EmuImage(emu, f2, b)
        kraw = None
        if ck is not None:
            kraw, ka = exact_array(2 * len(ck), np.int32, 0)
            ka[:] = ck.reshape(-1)
        nr, nc = f1.shape[0] - 2 * b, f1.shape[1] - 2 * b
        cells = -(-nr // P.block_size) * -(-nc // P.block_size)
        cap = capacity if capacity is not None else (len(ck) if ck is not None else cells)
        rp, pos = exact_array(2 * cap, np.int32, -7)
        rf, flow = exact_array(2 * cap, np.float32, -7)
        rd, dist = exact_array(cap, np.int32, -7)
        rv, valid = exact_array(cap, np.uint8, 0xEE)
        count = C.c_int32(-1)
        with Run(emu, schedule):
            rc = emu.vppb_sparse_flow_u8(C.byref(i1.desc), C.byref(i2.desc), C.byref(P), C.addressof(kraw) if kraw is not None else None, max(n, 0),
                                         ws.base, nbytes, C.addressof(rp), C.addressof(rf), C.addressof(rd), C.addressof(rv), cap, C.byref(count), None)
        assert rc == 0, emu.vppb_last_error()
        m = count.value
        assert (dist[m:] == -7).all() and (valid[m:] == 0xEE).all()  # nothing beyond the count
        return pos[:2 * m].reshape(-1, 2).copy(), flow[:2 * m].reshape(-1, 2).copy(), dist[:m].copy(), valid[:m].astype(bool)
    finally:
        emu.vppb_free(C.byref(ws))


def assert_same(got, exp):
    names = ("position", "flow", "distance", "valid")
    assert len(got[0]) == len(exp[0]), (len(got[0]), len(exp[0]))
    for g, e, nm in zip(got, exp, names):
        if nm == "flow":
            same = np.array_equal(g.view(np.uint32), np.asarray(e, np.float32).view(np.uint32))  # bit for bit
        else:
            same = np.array_equal(g, e)
        assert same, (nm, np.argwhere(g != e)[:8])


@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("subpixelic", [False, True], ids=["integer", "subpixel"])
@pytest.mark.parametrize("case", sc.CASES, ids=sc.case_id)
def test_table_matches_composite_oracle(emu, case, subpixelic, schedule):
    if schedule != "forward" and subpixelic and case["id"] not in ("subpixel-shift", "window-leaves-border"):
        pytest.skip("the shuffled order runs the subpixel mode on two cases: LK is the slowest stage on the emulator")
    f1, f2 = sc.frames(case)
    b = case["b"]
    exp = sc.oracle_sparse_flow(f1, f2, b, case, subpixelic)
    got = emu_sparse_flow(emu, f1, f2, b, case, subpixelic, schedule)
    assert_same(got, exp)
    cid = case["id"]
    if cid == "no-keypoint":
        assert len(got[0]) == 0
    if cid == "no-train-in-window" and not subpixelic:
        assert 0 < got[3].sum() < len(got[3])
    if cid in ("int-shift", "defaults") and not subpixelic:
        assert got[3].mean() > 0.5
    if cid == "window-leaves-border":
        assert not got[3][7:13].any()  # outside the frame: never valid
    if cid == "lk-flat" and subpixelic:  # a flat window makes G singular: the iteration turns non-finite and LK returns (0, 0)
        assert (got[1] == 0).all(1).sum() > len(got[1]) // 2


def test_errors_write_nothing(emu):
    case = dict(sc.CASES[0])
    f1, f2 = sc.frames(case)
    b = case["b"]
    nr, nc = f1.shape[0] - 2 * b, f1.shape[1] - 2 * b
    i1, i2 = EmuImage(emu, f1, b), EmuImage(emu, f2, b)
    small = EmuImage(emu, f1[1:-1, 1:-1], b - 1)  # same domain, border 4
    other = EmuImage(emu, f1[:-2, :], b)  # two rows fewer
    P = sc.params(case, False)
    nbytes = emu.vppb_sparse_flow_workspace_bytes(nr, nc, C.byref(P), -1)
    ws = np.full(nbytes + 256, 0xAB, np.uint8)
    wp = ws.ctypes.data + (-ws.ctypes.data) % 256
    outs = np.full(64 * 21, 0x5A, np.uint8)
    o = outs.ctypes.data
    kp = np.array([[5, 5], [10, 10]], np.int32)

    def call(a=i1, bimg=i2, p=P, k=None, n=0, nb=nbytes, cap=64):
        cnt = C.c_int32(-1)
        rc = emu.vppb_sparse_flow_u8(C.byref(a.desc), C.byref(bimg.desc), C.byref(p), k, n, wp, nb, o, o + 64 * 8, o + 64 * 16, o + 64 * 20, cap,
                                     C.byref(cnt), None)
        return rc, cnt.value

    def sp(**kw):  # subpixel-mode parameters
        return sc.params(dict(case, **kw), True)

    assert call(a=small)[0] == capi.VPPB_E_BORDER  # border 4 < max(3, winsize / 2) = 5
    assert call(bimg=small)[0] == capi.VPPB_E_BORDER
    assert call(bimg=other)[0] == capi.VPPB_E_ARG  # domains differ
    for w in (10, 3, 17, 4):  # with subpixelic: even, or outside 5 .. 15
        assert call(p=sp(ws=w))[0] in (capi.VPPB_E_ARG,), w
    assert call(p=sp(nscales=9))[0] == capi.VPPB_E_ARG
    assert call(nb=nbytes - 1)[0] == capi.VPPB_E_ARG  # workspace too small
    assert call(k=kp.ctypes.data, n=-1)[0] == capi.VPPB_E_ARG  # n < 0
    rc, cnt = call(k=kp.ctypes.data, n=2, cap=1)  # capacity too small, known on the host
    assert rc == capi.VPPB_E_CAPACITY and cnt == 2
    assert (outs == 0x5A).all() and (ws == 0xAB).all()
    # capacity too small, known after the detection: the count comes back, the outputs stay untouched
    rc, cnt = call(cap=1)
    assert rc == capi.VPPB_E_CAPACITY and cnt > 1
    assert (outs == 0x5A).all()


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
