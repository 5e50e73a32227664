"""The distance transform kernels (vpp_b200/csrc/stencils.cu) on the CPU emulator of tests/emu (kernels compiled by g++ and run thread by thread, warp shuffles
included) against the C oracle, over whole output buffers: the border at its full width, and pitch padding and parent pixels that
must keep their sentinel.  Every case runs with the threads of each launch in forward, reversed and shuffled order, under UBSan;
the table runs again under AddressSanitizer with exact-size allocations in a subprocess; and the C++ test tests/cpp/dt_tests.cu
runs on the emulator."""
import ctypes as C
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import dt_cases as dc
from vpp_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UBSAN_LOG = os.path.join(ROOT, "tests", "emu", "_build", "ubsan.log")
ASAN = os.environ.get("VPPB_EMU_ASAN") == "1"


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
    I, VP = C.POINTER(capi.VppbImg), C.c_void_p
    lib.vppb_distance_transform.argtypes = [I, I, C.c_int32, VP, C.c_int64, VP]
    lib.vppb_distance_transform_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.vppb_distance_transform_workspace_bytes.restype = C.c_int64
    lib.vppb_last_error.restype = C.c_char_p
    return lib


def E(h, align):
    return capi.VppbImg(h.desc.base, None, h.nrows, h.ncols, h.pitch, h.desc.border, h.elem, align)


def exact(h):
    """re-home a HostImage into a heap block of exactly its size (AddressSanitizer then sees any access outside it)"""
    raw = (C.c_ubyte * h.total)()
    C.memmove(raw, h.buf.ctypes.data, h.total)
    h._raw = raw
    h.buf = np.ctypeslib.as_array(raw)
    h.desc = type(h.desc)(h.buf.ctypes.data + h.origin, h.nrows, h.ncols, h.pitch, h.border, h.elem)
    return h


def run(emu, case, kind, schedule):
    ip, iv, op, ov, _ = dc.make_case(case)
    if ASAN and case[6] is None:
        ip, op = exact(ip), exact(op)
        iv, ov = ip, op
    elif ASAN:
        ip, op = exact(ip), exact(op)
        iv = dc.subview(ip, 1, 3, case[0], case[1])
        ov = dc.subview(op, case[6][0], case[6][1], case[0], case[1])
    n = emu.vppb_distance_transform_workspace_bytes(case[0], case[1], kind)
    ws = (C.c_ubyte * max(n, 1))()
    emu.vppb_emu_set_reverse(int(schedule == "reversed"))
    emu.vppb_emu_set_shuffle(4242 if schedule == "shuffled" else 0)
    try:
        rc = emu.vppb_distance_transform(C.byref(E(iv, case[5])), C.byref(E(ov, case[5])), kind, C.addressof(ws), n, None)
    finally:
        emu.vppb_emu_set_reverse(0)
        emu.vppb_emu_set_shuffle(0)
    assert rc == 0, emu.vppb_last_error()
    return op.buf.copy()


@pytest.mark.parametrize("schedule", ["forward", "reversed", "shuffled"])
@pytest.mark.parametrize("case", dc.CASES, ids=dc.case_id)
def test_distance_transform_matches_oracle(emu, case, schedule):
    exp, _ = dc.expected(case)
    for kind, buf in exp.items():
        got = run(emu, case, kind, schedule)
        assert np.array_equal(got, buf), (case, kind, schedule, np.argwhere(got != buf)[:8])


def test_errors_leave_the_output_untouched(emu):
    a = dc.host_image(6, 7, "u8", 0, 16, fill=0)
    cases = [(dc.host_image(6, 7, "i32", 1, 16), 3, capi.VPPB_E_BORDER), (dc.host_image(6, 7, "i32", 2, 16), 4, capi.VPPB_E_ARG),
             (dc.host_image(6, 8, "i32", 2, 16), 0, capi.VPPB_E_ARG), (dc.host_image(6, 7, "u8", 2, 16), 0, capi.VPPB_E_ARG)]
    ws = (C.c_ubyte * 4096)()
    for s, kind, rc in cases:
        assert emu.vppb_distance_transform(C.byref(E(a, 16)), C.byref(E(s, 16)), kind, C.addressof(ws), 4096, None) == rc
        assert (s.buf == dc.SENTINEL).all()
    # input and output in one allocation
    s = dc.host_image(6, 7, "i32", 2, 16)
    v = dc.subview(s, 0, 0, 6, 7)
    v.elem = 1
    iv = capi.VppbImg(s.desc.base, None, 6, 7, s.pitch, 0, 1, 16)
    assert emu.vppb_distance_transform(C.byref(iv), C.byref(E(s, 16)), 0, C.addressof(ws), 4096, None) == capi.VPPB_E_ARG
    assert (s.buf == dc.SENTINEL).all()


@pytest.mark.skipif(ASAN, reason="the C++ test runs once, without AddressSanitizer")
def test_cpp_dt_tests_on_the_emulator(emu):
    exe = dc.cpp_dt_emu()
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
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-k", "forward", "-p", "no:cacheprovider"],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=1500)
    reports = "".join(open(f).read() for f in glob.glob(log + "*"))
    errors = [l for l in reports.splitlines() if "ERROR: AddressSanitizer" in l or "SUMMARY: AddressSanitizer" in l]
    assert r.returncode == 0 and not errors, r.stdout[-3000:] + r.stderr[-2000:] + reports[:4000]
    assert " passed" in r.stdout
