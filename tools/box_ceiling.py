#!/usr/bin/env python
"""The copy ceiling of bench.py's headline batch: 128 separately allocated 1080x1920 vuchar3 inputs (border 2, alignment 128)
and 128 outputs (alignment 128), allocated with vppb_alloc as bench.py does.  Each variant is timed as us per launch of the
128 frame pairs (CUDA events, 20 launches after 3 warm-up launches) and as a fraction of the H100 SXM data sheet's 3.35 TB/s
at 6 B/px (3 read + 3 written):

  kernel, copy, compute   vppb_box5x5_u8c3_batch and its two ablations (VPPB_BOX_ABLATE, one child process each, as
                          tools/box_bench.py does: the library reads the knob once per process);
  strips_copy             a plain LSU copy, one CTA per 1920-byte column strip of an image walking down all its rows;
  bands_copy[_2|_68|_8]   the same copy with one CTA per band of whole rows: one band per image (_2: two; _68, _8: bands of 68
                          or 8 rows, so that the CTAs resident at a time work on a few neighbouring images, or one);
  memcpy2d                cudaMemcpy2DAsync of each pair;
  torch_copy              one contiguous device-to-device copy of the same total bytes (copy_ between two 1.6 GB tensors);
  bands_read, bands_write the bands copy's loads alone (folded into a register) and its stores alone, over the same images.

The plain kernels come from tools/box_ceiling.cu, compiled with nvcc for sm_90a into a temporary directory.  The variants run
in turn, --rounds times, in one process (the ablations in children), so that clock drift or other work on the GPU shows up as
spread.  Prints one JSON object with the card name, power limit and SM clock read in the same run (nvidia-smi queries only).
Usage: python tools/box_ceiling.py [--rounds 3] > ceiling.json"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, N, CS = 1080, 1920, 128, 3
PEAK_GBS = 3350.0  # H100 SXM data sheet (700 W card)
REPS = 20
ABLATIONS = {"kernel": {}, "copy": {"VPPB_BOX_ABLATE": "copy"}, "compute": {"VPPB_BOX_ABLATE": "compute"}}


def frames(vpp):
    """the bench's geometry: 128 inputs with border 2 and 128 outputs, alignment 128, each its own vppb_alloc"""
    S = [vpp.Image2d(H, W, "vuchar3", border=2, aligned=128) for _ in range(N)]
    D = [vpp.Image2d(H, W, "vuchar3", aligned=128) for _ in range(N)]
    return S, D


def timer(torch, stream):
    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(REPS):
            fn()
        b.record(stream)
        torch.cuda.synchronize()
        return a.elapsed_time(b) * 1e3 / REPS  # us per launch
    return timed


def child():
    """one libvppb variant (the environment selects it): us per vppb_box5x5_u8c3_batch launch of the 128 pairs"""
    import numpy as np
    import torch

    import vpp_b200 as vpp
    from vpp_b200 import capi

    capi.check(capi.lib.vppb_init(0))
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)
    S, D = frames(vpp)
    f = np.random.default_rng(0).integers(0, 256, (H, W, CS), dtype=np.uint8)
    for s in S:
        s.upload(f)
        vpp.fill_border_mirror(s)
    bi, bo = (capi.VppbImg * N)(*[x.desc for x in S]), (capi.VppbImg * N)(*[x.desc for x in D])
    us = timer(torch, stream)(lambda: capi.check(capi.lib.vppb_box5x5_u8c3_batch(bi, bo, N, sp)))
    print(json.dumps({"us": us}))


def build_plain(tmp):
    so = os.path.join(tmp, "box_ceiling.so")
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-Xcompiler", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tools", "box_ceiling.cu")])
    lib = C.CDLL(so)
    lib.ceiling_launch.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p]
    lib.ceiling_memcpy2d.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return lib


def plain_variants(lib, torch, vpp, stream):
    """name -> fn() doing one launch's worth of the plain variants over the bench geometry"""
    rowbytes = W * CS
    S, D = frames(vpp)
    sp = C.c_void_p(stream.cuda_stream)
    in_h = (C.c_ulonglong * N)(*[s.desc.base for s in S])
    out_h = (C.c_ulonglong * N)(*[d.desc.base for d in D])
    in_d = torch.tensor([s.desc.base for s in S], dtype=torch.int64, device="cuda")
    out_d = torch.tensor([d.desc.base for d in D], dtype=torch.int64, device="cuda")
    sink = torch.zeros(1, dtype=torch.int32, device="cuda")
    ip, op = S[0].desc.pitch, D[0].desc.pitch
    total = N * H * rowbytes
    big_a = torch.empty(total, dtype=torch.uint8, device="cuda")
    big_b = torch.empty(total, dtype=torch.uint8, device="cuda")
    keep = (S, D, in_h, out_h, in_d, out_d, sink, big_a, big_b)

    def k(mode, seg, band, block):
        def fn():
            rc = lib.ceiling_launch(mode, in_d.data_ptr(), out_d.data_ptr(), N, ip, op, H, rowbytes, seg, band, block, sink.data_ptr(), sp)
            if rc:
                raise RuntimeError("ceiling_launch: CUDA error %d" % rc)
        return fn

    def m2d():
        rc = lib.ceiling_memcpy2d(in_h, out_h, N, ip, op, H, rowbytes, sp)
        if rc:
            raise RuntimeError("cudaMemcpy2DAsync: CUDA error %d" % rc)

    return keep, {
        "strips_copy": k(0, 1920, H, 128),
        "bands_copy": k(0, rowbytes, H, 384),
        "bands_copy_2": k(0, rowbytes, H // 2, 384),
        "bands_copy_68": k(0, rowbytes, 68, 384),
        "bands_copy_8": k(0, rowbytes, 8, 384),
        "memcpy2d": m2d,
        "torch_copy": lambda: big_b.copy_(big_a),
        "bands_read": k(1, rowbytes, H, 384),
        "bands_write": k(2, rowbytes, H, 384),
    }


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        return "unavailable (%r)" % ex


class ClockSampler:
    """SM clock every 100 ms while the variants run (nvidia-smi query loop, stopped before the script ends)"""

    def __enter__(self):
        self.lines = []
        self.p = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "100"],
                                  stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        self.t = threading.Thread(target=lambda: [self.lines.append(l) for l in self.p.stdout], daemon=True)
        self.t.start()
        return self

    def __exit__(self, *a):
        self.p.terminate()
        self.p.wait(timeout=10)
        self.t.join(timeout=2)

    def mhz(self):
        v = sorted(float(l) for l in self.lines if l.strip().replace(".", "").isdigit())
        return {"median": v[len(v) // 2], "min": v[0], "max": v[-1], "samples": len(v)} if v else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch

    import vpp_b200 as vpp
    from vpp_b200 import capi

    capi.check(capi.lib.vppb_init(0))
    stream = torch.cuda.current_stream()
    timed = timer(torch, stream)
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_plain(tmp)
        keep, plain = plain_variants(lib, torch, vpp, stream)
        with ClockSampler() as clk:
            for rnd in range(max(args.rounds, 3)):
                for name, env in ABLATIONS.items():
                    e = dict(os.environ)
                    e.pop("VPPB_BOX_ABLATE", None)
                    e.update(env)
                    r = subprocess.run([sys.executable, os.path.abspath(__file__), "child"], env=e, capture_output=True, text=True, timeout=600)
                    if r.returncode != 0:
                        raise RuntimeError("%s child failed:\n%s" % (name, r.stderr[-2000:]))
                    res.setdefault(name, []).append(json.loads(r.stdout.strip().splitlines()[-1])["us"])
                for name, fn in plain.items():
                    res.setdefault(name, []).append(timed(fn))
                print(rnd, json.dumps({k: round(v[-1], 1) for k, v in res.items()}), file=sys.stderr)
        del keep
    bytes_per_launch = 2 * CS * H * W * N
    table = {}
    for name, v in res.items():
        med = sorted(v)[len(v) // 2]
        # the read-only and write-only passes move half the bytes: their fraction is of 3 B/px
        b = bytes_per_launch // 2 if name in ("bands_read", "bands_write") else bytes_per_launch
        table[name] = {"us_per_launch": [round(x, 1) for x in v], "median_us": round(med, 1),
                       "spread": round((max(v) - min(v)) / med, 4), "frac_of_3350": round(b / (med * 1e-6) / 1e9 / PEAK_GBS, 3)}
    out = {"gpu": smi("name,power.limit,clocks.max.sm"), "sm_mhz_during_run": clk.mhz(), "batch": "%d x %dx%d vuchar3, border 2, align 128" % (N, H, W),
           "bytes_per_launch": bytes_per_launch, "rounds": max(args.rounds, 3), "variants": table}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "child":
        child()
        sys.exit(0)
    main()
