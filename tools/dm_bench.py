#!/usr/bin/env python
"""Timing of the SAD descriptor matchers (GPU only): brute force at 10k x 10k (u8 D = 49 and 128, int D = 10), and the grid-local
matcher on FAST keypoints and 7x7 extract_patches descriptors of two shifted 1080p scenes (R = 32 and 100, s = 32).
Per entry: warm-up, then CUDA events on the launch stream around as many calls as fill at least 0.5 s; descriptor pairs compared
per second (grid-local: the candidate pairs its windows hold); for brute force, the SASS instructions per pair of the kernel's
inner loop (cuobjdump of vpp_b200/lib/libvppb.so) and the fraction of the SM integer-issue bound (4 warp instructions per clock
per SM at the card's maximum SM clock) that the measured rate reaches; a parity flag against the C oracle (OpenMP build); and
the reference header's time for one call (oracle/_ref/libvppref_dm_omp.so, host clock) where that library exists, "not
measured" otherwise.  The card name, power limit, SM count and clock are read in the same run.  Prints one JSON document.
Usage: python tools/dm_bench.py [--min-seconds S] > dm_bench.json"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, "vpp_b200", "lib", "libvppb.so")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power + " W", "max_sm_clock_mhz": float(clock)}
    except Exception as e:  # the timing still stands; say why the card is unknown
        return {"name": "unknown (%s)" % e, "power_limit": "unknown", "max_sm_clock_mhz": None}


def sass_instructions_per_pair(word, qw):
    """instructions of k_bf_sad<word, qw>'s innermost loop over the tile divided by the trains it compares per iteration (each train's qw words
    are read from shared memory once, 4 per LDS.128), or None where cuobjdump is missing"""
    sym = "_ZN4vppb8k_bf_sadI%sLi%dEEEvNS_3ImgES1_iiiiiiPy" % ("j" if word == "u8" else "i", qw)
    try:
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", sym, LIB], capture_output=True, text=True, timeout=120).stdout
    except Exception:
        return None
    ins = [(int(m.group(1), 16), m.group(2)) for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", sass)]
    best = None
    for addr, text in ins:
        m = re.search(r"BRA\s+(?:\w+,\s*)?0x([0-9a-f]+)", text)
        if not m or int(m.group(1), 16) >= addr:
            continue
        body = [t for a, t in ins if int(m.group(1), 16) <= a <= addr]
        lds = sum(1 for t in body if "LDS.128" in t)
        if lds and (best is None or len(body) < best[0]):  # the innermost loop that reads train words
            best = (len(body), lds)
    if best is None:
        return None
    trains = best[1] * 4 / qw
    return round(best[0] / trains, 2)


def timed(call, stream, min_s):
    import torch

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    reps = 2
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            call()
        e1.record(stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= min_s * 1e3:
            return ms * 1e-3 / reps, reps
        reps = int(reps * max(2.0, 1.2 * min_s * 1e3 / max(ms, 1e-3)))


def host_time(fn):
    t0 = time.perf_counter()
    fn()
    return round((time.perf_counter() - t0) * 1e3, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import torch

    import vpp_b200 as vpp
    from vpp_b200 import capi, ops
    from vpp_b200.capi import lib
    from tests import dm_cases as dc
    from tests.scenes import rectangles_scene

    assert torch.cuda.is_available(), "tools/dm_bench.py measures on a GPU; there is none"
    capi.check(lib.vppb_init(0))
    info = card()
    info["sms"] = torch.cuda.get_device_properties(0).multi_processor_count
    omp = dc.oracle_omp()
    ref = dc.reference(omp=True)
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    results = []

    for word, D, qw in (("u8", 49, 16), ("u8", 128, 32), ("i32", 10, 12)):
        rng = np.random.default_rng(D)
        n = 10000
        elem = 1 if word == "u8" else 4
        q, t = dc.descriptors(n, D, elem, 0, rng), dc.descriptors(n, D, elem, 0, rng)
        Q, T = vpp.Image2d.from_host(q, word), vpp.Image2d.from_host(t, word)
        nb = lib.vppb_match_bruteforce_sad_workspace_bytes(n, n, D)
        ws, di, dd = ops._DeviceBuffer(nb), ops._DeviceBuffer(n * 4), ops._DeviceBuffer(n * 4)

        def call():
            capi.check(lib.vppb_match_bruteforce_sad(Q.ptr(), T.ptr(), ws.ptr, nb, di.ptr, dd.ptr, sp))

        sec, reps = timed(call, stream, args.min_seconds)
        gi, gd = di.to_host(np.int32, n, stream), dd.to_host(np.int32, n, stream)
        bi, bd = dc.oracle_bruteforce(q, t, lib=omp)
        pairs = n * n / sec
        ipp = sass_instructions_per_pair(word, qw)
        frac = None
        if ipp and info["max_sm_clock_mhz"]:
            bound = info["sms"] * 4 * 32 * info["max_sm_clock_mhz"] * 1e6 / ipp
            frac = round(pairs / bound, 3)
        ref_ms = host_time(lambda: dc.ref_bruteforce(q, t, lib=ref)) if ref is not None else "not measured"
        results.append({"entry": "bruteforce %s D=%d 10k x 10k" % (word, D), "calls": reps, "ms": round(sec * 1e3, 4),
                        "pairs_per_s": float("%.4g" % pairs), "sass_instructions_per_pair": ipp, "fraction_of_int_issue_bound": frac,
                        "parity": bool(np.array_equal(gi, bi) and np.array_equal(gd, bd)), "reference_ms": ref_ms})
        print(json.dumps(results[-1]), file=sys.stderr)

    a = rectangles_scene(1080, 1920, seed=11)
    b = np.roll(a, (4, -7), axis=(0, 1))
    imgs, kps = [], []
    for x in (a, b):
        G = vpp.Image2d.from_host(x, "u8", border=3)
        vpp.fill_border_mirror(G)
        imgs.append(G)
        kps.append(np.ascontiguousarray(vpp.fast9(G, 20)))
    pats = [vpp.extract_patches(G, k, 7) for G, k in zip(imgs, kps)]
    q, t = pats[1].download(), pats[0].download()
    nq, nt = len(q), len(t)
    d_qp, d_tp = ops._DeviceBuffer(nq * 8).from_host(kps[1]), ops._DeviceBuffer(nt * 8).from_host(kps[0])
    di, dd = ops._DeviceBuffer(nq * 4), ops._DeviceBuffer(nq * 4)
    for R in (32, 100):
        s = 32
        nb = lib.vppb_match_local_sad_workspace_bytes(nq, nt, 49, R, s)
        ws = ops._DeviceBuffer(nb + 256)

        def call():
            capi.check(lib.vppb_match_local_sad(pats[1].ptr(), pats[0].ptr(), d_qp.ptr, d_tp.ptr, R, s, ws.ptr, nb, di.ptr, dd.ptr, sp))

        sec, reps = timed(call, stream, args.min_seconds)
        gi, gd = di.to_host(np.int32, nq, stream), dd.to_host(np.int32, nq, stream)
        li, ld = dc.oracle_local(q, t, kps[1], kps[0], R, s, lib=omp)
        # candidate pairs: trains whose cell lies in each query's window
        tc = kps[0] // s
        cand = 0
        for p in kps[1]:
            lo, hi = (p.astype(np.int64) - R) // 1, (p.astype(np.int64) + R)
            r0, r1 = np.trunc(lo / s), np.trunc(hi / s)
            cand += int(((tc[:, 0] >= r0[0]) & (tc[:, 0] <= r1[0]) & (tc[:, 1] >= r0[1]) & (tc[:, 1] <= r1[1])).sum())
        ref_ms = host_time(lambda: dc.ref_local(q, t, kps[1], kps[0], R, s, lib=ref)) if ref is not None else "not measured"
        results.append({"entry": "local 1080p FAST %d x %d, 7x7 u8 patches, R=%d s=%d" % (nq, nt, R, s), "calls": reps,
                        "ms": round(sec * 1e3, 4), "candidate_pairs": cand, "pairs_per_s": float("%.4g" % (cand / sec)),
                        "parity": bool(np.array_equal(gi, li) and np.array_equal(gd, ld)), "reference_ms": ref_ms})
        print(json.dumps(results[-1]), file=sys.stderr)
    print(json.dumps({"card": info, "results": results}, indent=1))
    return 0 if all(r["parity"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
