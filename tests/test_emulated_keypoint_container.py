"""The device keypoint container (the vppb_kpc_* entries of vpp_b200/csrc/kpc.cu) on the CPU emulator of tests/emu, step by step
against the model of tests/kpc_cases.py: the case table with the threads and blocks of each launch in forward, reversed and
shuffled order (the merge builds its cell lists with unordered atomicExch), and once more under AddressSanitizer in a subprocess,
with every detection buffer exactly as long as max_detections says."""
import ctypes as C
import gc
import glob
import os
import subprocess
import sys

import pytest

from tests import kpc_cases as kc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UBSAN_LOG = os.path.join(ROOT, "tests", "emu", "_build", "ubsan_kpc.log")
ASAN = os.environ.get("VPPB_EMU_ASAN") == "1"
SCHEDULES = ["forward"] if ASAN else ["forward", "reversed", "shuffled"]
SMS = 2  # the emulator's cudaDevAttrMultiProcessorCount (tests/emu/cuda_runtime.h)


@pytest.fixture(scope="module")
def emu(built):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu

    from vpp_b200 import capi, ops

    path = build_emu.build(asan=ASAN)
    mp = pytest.MonkeyPatch()
    if not ASAN:
        mp.setenv("UBSAN_OPTIONS", "log_path=%s" % UBSAN_LOG)
    lib = C.CDLL(path)
    for name, (res, args) in capi.PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    mp.setattr(capi, "lib", lib)
    mp.setattr(ops, "lib", lib)
    yield lib
    gc.collect()  # buffers allocated by the emulated library must be freed by it
    mp.undo()


@pytest.fixture(autouse=True)
def no_sanitizer_reports():
    yield
    logs = glob.glob(UBSAN_LOG + "*")
    text = "".join(open(f).read() for f in logs)
    for f in logs:
        os.remove(f)
    assert not text, "UBSan report from an emulated kernel:\n" + text[:4000]


@pytest.fixture(params=SCHEDULES)
def schedule(emu, request):
    emu.vppb_emu_set_reverse(1 if request.param == "reversed" else 0)
    emu.vppb_emu_set_shuffle(777 if request.param == "shuffled" else 0)
    yield request.param
    emu.vppb_emu_set_reverse(0)
    emu.vppb_emu_set_shuffle(0)


def test_model_equals_host_orchestration(built):
    kc.check_model_against_orchestration()


@pytest.mark.parametrize("case", kc.cases(SMS), ids=lambda c: c["id"])
def test_case_table(schedule, case):
    ev = kc.run_case(case, host_memory=True, exact=ASAN)
    cid = case["id"]
    if case["n"] > 1024:
        assert ev["max_n"] > 1024
    if cid in ("crowded", "spacing1", "regrow-10-then-1", "n2049", "past-grid-cap"):
        assert ev["removed_by_merge"] > 0
    if cid.startswith("traj"):
        assert ev["wrapped"] > 0
    if case["n"] >= 32:
        assert ev["dead"] > 0 and ev["compacted"] > 0


@pytest.mark.parametrize("cid,steps", kc.edge_cases(), ids=[c[0] for c in kc.edge_cases()])
def test_capacity_and_caller_detections(schedule, cid, steps):
    m = kc.run_edge_case(steps, host_memory=True, exact=ASAN)
    assert not (m.pos == kc.SENTINEL).all(1).any()
    if cid == "count-over-max-detections":
        assert m.n == 4
    if cid in ("exactly-full", "one-over"):
        assert m.n == 64


def test_rejected_calls_leave_the_state(emu):
    kc.check_rejected_calls(host_memory=True)


@pytest.mark.skipif(ASAN, reason="this is the driver of the AddressSanitizer run")
def test_under_address_sanitizer(built, tmp_path):
    libasan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan) or not os.path.exists(libasan):
        pytest.skip("libasan.so not available")
    log = str(tmp_path / "asan")
    env = dict(os.environ, VPPB_EMU_ASAN="1", VPPB_EMU_STACK_KB="96", LD_PRELOAD=libasan,
               ASAN_OPTIONS="detect_leaks=0:halt_on_error=1:log_path=%s" % log)
    env.pop("UBSAN_OPTIONS", None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-p", "no:cacheprovider"],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=1500)
    reports = "".join(open(f).read() for f in glob.glob(log + "*"))
    errors = [l for l in reports.splitlines() if "ERROR: AddressSanitizer" in l or "SUMMARY: AddressSanitizer" in l]
    assert r.returncode == 0 and not errors, r.stdout[-3000:] + r.stderr[-2000:] + reports[:4000]
    assert " passed" in r.stdout
