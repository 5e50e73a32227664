#!/usr/bin/env python
"""Timing of the chamfer distance transforms (vppb_distance_transform, GPU only): each transform at 1080p, 4K and 8K, u8 input,
on about 0.1 % random zero pixels ("sparse") and on a single zero in the bottom-right corner ("corner", the longest lines).
Per entry: warm-up, then CUDA events on the launch stream around as many calls as fill at least 0.5 s; the bytes moved under this
script's model of the kernels; the fraction of 3.35 TB/s (H100 SXM HBM3, data sheet) that the 5 B/px minimum (1 B in, 4 B out)
would need; a parity flag of the whole output frame against the C oracle; and the reference header's time for one call
(oracle/_ref/libvppref_dt_omp.so, serial passes, host clock) where that library exists, "not measured" otherwise.  The card name
and power limit are read in the same run.  Prints one JSON document.
Usage: python tools/dt_bench.py [--min-seconds S] > dt_bench.json"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(1080, 1920, "1080p"), (2160, 3840, "4k"), (4320, 7680, "8k")]
KINDS = [("d4", 0, 1), ("d8", 1, 3), ("d3_4", 2, 3), ("d5_7_11", 3, 7)]  # name, VPPB_DT_*, line-scan generators besides the rows
HBM_BPS = 3.35e12


def model_bytes(nr, nc, ngen, in_bytes=1):
    """k_dt_rows: the input read twice, the output row written, read back and written again (2 in + 12 B/px); per further
    generator: k_dt_summary reads the image, k_dt_apply reads and writes it (12 B/px); the carries are < 1 % and not counted"""
    return nr * nc * (2 * in_bytes + 12 + 12 * ngen)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the timing still stands; say why the card is unknown
        return {"name": "unknown (%s)" % e, "power_limit": "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import torch

    import vpp_b200 as vpp
    from vpp_b200 import capi, ops
    from vpp_b200.capi import lib
    from tests import dt_cases as dc
    from tests import oracle as orc

    assert torch.cuda.is_available(), "tools/dt_bench.py measures on a GPU; there is none"
    capi.check(lib.vppb_init(0))
    info = card()
    o = dc.oracle()
    ref_path = os.path.join(ROOT, "oracle", "_ref", "libvppref_dt_omp.so")
    ref = None
    if os.path.exists(ref_path):
        ref = C.CDLL(ref_path)
        ref.vppref_distance_transform.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    results = []
    for nr, nc, size in SIZES:
        for pat in ("sparse", "corner"):
            a = dc.pattern(pat, nr, nc, 11)
            A = vpp.Image2d.from_host(a, "u8")
            ha = orc.HostImage(nr, nc, "u8", data=a)
            for name, kind, ngen in KINDS:
                reach = dc.REACH[kind]
                S = vpp.Image2d(nr, nc, "i32", border=reach)
                n = lib.vppb_distance_transform_workspace_bytes(nr, nc, kind)
                ws = ops._DeviceBuffer(n)

                def call():
                    capi.check(lib.vppb_distance_transform(A.ptr(), S.ptr(), kind, ws.ptr, n, sp))

                for _ in range(3):
                    call()
                torch.cuda.synchronize()
                reps, ms = 4, 0.0
                while True:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    for _ in range(reps):
                        call()
                    e1.record(stream)
                    e1.synchronize()
                    ms = e0.elapsed_time(e1)
                    if ms >= args.min_seconds * 1e3:
                        break
                    reps = int(reps * max(2.0, 1.2 * args.min_seconds * 1e3 / max(ms, 1e-3)))
                t = ms * 1e-3 / reps
                got = S.download(with_border=True)
                hs = orc.HostImage(nr, nc, "i32", border=reach)
                assert o.vo_distance_transform(C.addressof(ha.desc), C.addressof(hs.desc), kind) == 0
                parity = bool(np.array_equal(got, hs.get(with_border=True)))
                ref_ms = "not measured"
                if ref is not None:
                    hr = orc.HostImage(nr, nc, "i32", border=reach)
                    best = None
                    for _ in range(2):
                        t0 = time.perf_counter()
                        ref.vppref_distance_transform(C.addressof(ha.desc), 0, C.addressof(hr.desc), kind)
                        dt = time.perf_counter() - t0
                        best = dt if best is None else min(best, dt)
                    ref_ms = round(best * 1e3, 3)
                mb = model_bytes(nr, nc, ngen)
                results.append({"kind": name, "size": size, "input": pat, "calls": reps, "ms": round(t * 1e3, 4),
                                "model_bytes": mb, "model_GBps": round(mb / t / 1e9, 1),
                                "min_bytes_fraction_of_hbm": round(5 * nr * nc / HBM_BPS / t, 4),
                                "parity_vs_oracle": parity, "reference_ms": ref_ms})
                print(json.dumps(results[-1]), file=sys.stderr)
    print(json.dumps({"card": info, "hbm_bytes_per_s": HBM_BPS, "results": results}, indent=1))
    return 0 if all(r["parity_vs_oracle"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
