#!/usr/bin/env python
"""Timing of vppb_sparse_flow_u8 (GPU only) at 1080p and 4K with the default options (detector_th 5, block_size 5, winsize 11,
search_radius 100, cell_width 300, lk_iterations 5, nscales 3), integer and subpixel mode, on a rectangles scene shifted by (3, -2).
Per entry: warm-up, then CUDA events on the launch stream around as many calls as fill at least --min-seconds (a call includes its one
host synchronisation); the same stages queued one entry at a time on the same buffers for a per-stage split (2x FAST, 2x patches, the
grid-local match, pyramids + LK with a zero prediction); "rest" is the total minus those stages (the seed / refine kernels, the 8-byte count read and the
host work of the call); the host clock until one call returns (the work queued after its count read is
still running then); keypoint counts and the candidate pairs the match windows hold; a parity flag against the composite oracle
of tests/sof_cases.py (OpenMP build of the C oracle); and the host time of one call of that composite.  The card name and power
limit are read in the same run.  Prints one JSON document.
Usage: python tools/sof_bench.py [--min-seconds S] > sof_bench.json"""
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                             timeout=30).stdout
        name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power + " W"}
    except Exception as e:
        return {"name": "unknown (%s)" % e, "power_limit": "unknown"}


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
            return ms / reps
        reps = int(reps * max(2.0, 1.2 * min_s * 1e3 / max(ms, 1e-3)))


def candidates(k1, k2, R, s):
    """query-train pairs inside the grid-local windows: sum over queries of the trains in their window's cells"""
    if len(k1) == 0 or len(k2) == 0:
        return 0
    cr, cc = k2[:, 0] // s, k2[:, 1] // s
    H = np.zeros((cr.max() + 2, cc.max() + 2), np.int64)
    np.add.at(H, (cr + 1, cc + 1), 1)
    S = H.cumsum(0).cumsum(1)  # S[r + 1, c + 1] = trains in cells [0, r] x [0, c]
    r0 = np.clip((k1[:, 0] - R) // s, 0, None)  # the coordinates are >= 0: floor division equals the C truncation here
    r1 = np.clip((k1[:, 0] + R) // s, None, cr.max())
    c0 = np.clip((k1[:, 1] - R) // s, 0, None)
    c1 = np.clip((k1[:, 1] + R) // s, None, cc.max())
    ok = (r0 <= r1) & (c0 <= c1)
    r0, r1, c0, c1 = r0[ok], r1[ok], c0[ok], c1[ok]
    return int((S[r1 + 1, c1 + 1] - S[r0, c1 + 1] - S[r1 + 1, c0] + S[r0, c0]).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import torch

    import vpp_b200 as vpp
    from vpp_b200 import capi, ops
    from vpp_b200.capi import lib
    from tests import dm_cases as dc
    from tests import oracle as orc
    from tests import sof_cases as sc
    from tests.scenes import rectangles_scene, warp

    assert torch.cuda.is_available(), "tools/sof_bench.py measures on a GPU; there is none"
    capi.check(lib.vppb_init(0))
    info = card()
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    o = sc.DEFAULTS
    results = []
    for nr, nc in ((1080, 1920), (2160, 3840)):
        b = 5
        a = rectangles_scene(nr + 2 * b, nc + 2 * b, seed=nr).astype(np.float64)
        f1 = a.astype(np.uint8)
        f2 = np.clip(np.round(warp(a, -3, 2)), 0, 255).astype(np.uint8)
        I1, I2 = vpp.Image2d(nr, nc, "u8", border=b), vpp.Image2d(nr, nc, "u8", border=b)
        I1.upload(f1, with_border=True)
        I2.upload(f2, with_border=True)
        cells = -(-nr // o["bs"]) * -(-nc // o["bs"])
        for sub in (False, True):
            P = capi.VppbSofParams(o["th"], o["bs"], o["ws"], o["R"], o["s"], int(sub), o["it"], o["nscales"])
            nb = lib.vppb_sparse_flow_workspace_bytes(nr, nc, C.byref(P), -1)
            ws = ops._DeviceBuffer(nb)
            outs = [ops._DeviceBuffer(cells * k) for k in (8, 8, 4, 1)]
            cnt = C.c_int32(0)

            def call():
                capi.check(lib.vppb_sparse_flow_u8(I1.ptr(), I2.ptr(), C.byref(P), None, 0, ws.ptr, nb, outs[0].ptr, outs[1].ptr, outs[2].ptr, outs[3].ptr,
                                                   cells, C.byref(cnt), sp))

            total = timed(call, stream, args.min_seconds)
            t0 = time.perf_counter()
            call()
            host_ms = (time.perf_counter() - t0) * 1e3
            n1 = cnt.value
            got = (outs[0].to_host(np.int32, 2 * n1, sp).reshape(-1, 2), outs[1].to_host(np.float32, 2 * n1, sp).reshape(-1, 2),
                   outs[2].to_host(np.int32, n1, sp), outs[3].to_host(np.uint8, n1, sp).astype(bool))

            # the stages one entry at a time on the same inputs
            fb = lib.vppb_fast9_workspace_bytes(nr, nc, o["bs"])
            fws, k1, k2, dcnt = ops._DeviceBuffer(fb), ops._DeviceBuffer(cells * 8), ops._DeviceBuffer(cells * 8), ops._DeviceBuffer(8)
            fast = lambda img, k, c: capi.check(lib.vppb_fast9_u8_async(img.ptr(), o["th"], None, capi.FAST_BLOCKWISE, o["bs"], 0, fws.ptr, fb, k.ptr, None, cells,
                                                                        c, sp))
            fast(I1, k1, dcnt.ptr)
            fast(I2, k2, dcnt.ptr + 4)
            n1_, n2 = [int(x) for x in dcnt.to_host(np.int32, 2, sp)]
            D = o["ws"] ** 2
            P1, P2 = vpp.Image2d(n1_, D, "u8"), vpp.Image2d(n2, D, "u8")
            mb = lib.vppb_match_local_sad_workspace_bytes(n1_, n2, D, o["R"], o["s"])
            mws, di, dd = ops._DeviceBuffer(mb), ops._DeviceBuffer(n1_ * 4), ops._DeviceBuffer(n1_ * 4)
            stages = {
                "fast_x2_ms": timed(lambda: (fast(I1, k1, dcnt.ptr), fast(I2, k2, dcnt.ptr + 4)), stream, args.min_seconds),
                "patches_x2_ms": timed(lambda: (capi.check(lib.vppb_extract_patches(I1.ptr(), k1.ptr, n1_, o["ws"], P1.ptr(), sp)),
                                                capi.check(lib.vppb_extract_patches(I2.ptr(), k2.ptr, n2, o["ws"], P2.ptr(), sp))), stream, args.min_seconds),
                "match_ms": timed(lambda: capi.check(lib.vppb_match_local_sad(P1.ptr(), P2.ptr(), k1.ptr, k2.ptr, o["R"], o["s"], mws.ptr, mb, di.ptr, dd.ptr, sp)),
                                  stream, args.min_seconds),
            }
            if sub:
                bd = o["ws"] // 2
                prev, nxt = ops.Pyramid2d((nr, nc), o["nscales"], 2, pixel="u8", border=bd), ops.Pyramid2d((nr, nc), o["nscales"], 2, pixel="u8", border=bd)
                grad = ops.Pyramid2d((nr, nc), o["nscales"], 2, pixel="vint2", border=bd)
                L = capi.VppbLkParams(nlevels=o["nscales"], min_scale=0, winsize=o["ws"], max_iter=o["it"], grad_is_float=0, err_mode=capi.LK_ERR_SAD,
                                      gate_on_max_err=0, min_ev=0.0, delta=0.0, max_err=0.0, factor=2.0, pred_div=float(2 ** o["nscales"]))
                kf = ops._DeviceBuffer(n1_ * 8).from_host(k1.to_host(np.int32, 2 * n1_, sp).astype(np.float32), sp)
                pr = ops._DeviceBuffer(n1_ * 8).from_host(np.zeros(2 * n1_, np.float32), sp)
                fo, eo = ops._DeviceBuffer(n1_ * 8), ops._DeviceBuffer(n1_ * 4)

                def lk():
                    capi.check(lib.vppb_pyrlk_prepare(I1.ptr(), I2.ptr(), prev.desc_array(), nxt.desc_array(), grad.desc_array(), o["nscales"], 0, sp))
                    capi.check(lib.vppb_lk_match_u8(prev.desc_array(), nxt.desc_array(), grad.desc_array(), C.byref(L), kf.ptr, pr.ptr, n1_, fo.ptr, eo.ptr, sp))

                stages["pyramids_lk_ms"] = timed(lk, stream, args.min_seconds)
            stages["rest_ms"] = total - sum(stages.values())

            case = dict(id="bench", nr=nr, nc=nc, b=b)
            t0 = time.perf_counter()
            exp = sc.oracle_sparse_flow(f1, f2, b, case, sub, lib=orc.load(omp=True), omp=dc.oracle_omp())
            oracle_ms = (time.perf_counter() - t0) * 1e3
            parity = len(got[0]) == len(exp[0]) and all(
                np.array_equal(g.view(np.uint32), np.asarray(e, np.float32).view(np.uint32)) if k == 1 else np.array_equal(g, e)
                for k, (g, e) in enumerate(zip(got, exp)))
            results.append({"size": "%dx%d" % (nc, nr), "mode": "subpixel" if sub else "integer", "total_ms": round(total, 3),
                            "host_return_ms": round(host_ms, 3),
                            "stages": {k: round(v, 3) for k, v in stages.items()}, "keypoints_frame1": n1, "keypoints_frame2": n2,
                            "valid": int(got[3].sum()), "candidate_pairs": candidates(exp[0], sc.oracle_fast_blockwise(f2, b, o["th"], o["bs"]), o["R"], o["s"]),
                            "parity": bool(parity), "oracle_composite_host_ms": round(oracle_ms, 1)})
            print(json.dumps(results[-1]), file=sys.stderr)
    print(json.dumps({"card": info, "options": o, "results": results}, indent=1))


if __name__ == "__main__":
    main()
