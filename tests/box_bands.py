"""Child process of the row-band tests of the streaming 5x5 box kernel (tests/test_gpu_box_bands.py, tests/test_emulated_box_bands.py).

A task of k_box5_stream is a band of R rows of one image across S <= 3 adjacent strips of its rows: a row of up to 3 strips is one
band wide, a wider row is cut into bands of as equal strip counts.  The CTA holds S groups of 4 consumer warps, and S sets how many
CTAs are resident per SM (3, 2, 1) and so the rows per task the launch picks.  This module runs a case table that reaches each of
those choices through tests/box_geometry.py's harness (numpy reference, sentinel-filled outputs, row tiles with garbage halo
rows), under the environment it was started with (VPPB_BOX_R is read once per process):

    python -m tests.box_bands --backend gpu|emu [--big]

and prints one JSON object: the SM count, and per case and entry point pass / fail with the band launches `band_plan` (a
transcription of box5_stream_launch_nb's rules in vpp_b200/csrc/box.cu) says the library makes."""
import argparse
import json
import os
import subprocess
import sys

from tests import box_geometry as bg

ROOT = bg.ROOT
POLICIES = {"default": {}, "r21": {"VPPB_BOX_R": "21"}}
BS_K, BS_MAX_G, BS_MAX_S = 5, 126, 3
CTAS_PER_SM = {1: 3, 2: 2, 3: 1}  # by strips per band
_kernel_plan = bg.plan  # which kernel each call takes and how batches are split: unchanged by the band schedule


def stream_rows(tasks_per_chunk, nrows, ctas, forced):
    """box_stream_rows(): (R, chunks)"""
    m_max = max(4, (nrows + 4 + BS_K - 1) // BS_K)
    best_r, best = 16, float("inf")
    for m in range(4, m_max + 1):
        r = 5 * m - 4
        if forced > 0 and r != forced:
            continue
        tasks = (nrows + r - 1) // r * tasks_per_chunk
        cost = (tasks + ctas - 1) // ctas * (5.0 * m + 2.0)
        if cost < best:
            best, best_r = cost, r
    return best_r, (nrows + best_r - 1) // best_r


def band_launch(rowbytes, nrows, n, sms, forced, tiles):
    groups = (rowbytes + 15) // 16
    strips = (groups + BS_MAX_G - 1) // BS_MAX_G
    G = (groups + strips - 1) // strips
    bands = (strips + BS_MAX_S - 1) // BS_MAX_S
    S = (strips + bands - 1) // bands
    resident = sms * CTAS_PER_SM[S]
    R, chunks = stream_rows(bands * n, nrows, resident, forced)
    return dict(n=n, strips=strips, G=G, last=groups - (strips - 1) * G, bands=bands, S=S, last_band_strips=strips - (bands - 1) * S,
                R=R, chunks=chunks, last_rows=nrows - (chunks - 1) * R, tasks=n * bands * chunks, resident=resident, tiles=tiles)


def band_plan(entry, ins, outs, sms, env, neighbours=False):
    """the streaming launches of `entry` (box_geometry.plan picks the kernel and the batches), with their band geometry"""
    forced = bg._knob(env, "VPPB_BOX_R")
    rowbytes = ins[0].ncols * ins[0].elem_bytes
    return [band_launch(rowbytes, ins[0].nrows, l["n"], sms, forced, neighbours)
            for l in _kernel_plan(entry, ins, outs, sms, env, neighbours=neighbours) if l["kernel"] == "stream"]


def unmet_claims(result, policy):
    """the band geometries the table is written to reach: names of those the launches no longer reach"""
    ls = [l for r in result["results"] for l in r["launches"]]
    claims = {
        "one band per image": any(l["bands"] == 1 and l["chunks"] == 1 and l["S"] == 3 for l in ls),
        "several bands per image": any(l["chunks"] > 1 and l["S"] == 3 for l in ls),
        "a band whose last strip ends ragged": any(l["S"] > 1 and l["last"] < l["G"] for l in ls),
        "more tasks than resident CTAs": any(l["tasks"] > l["resident"] for l in ls),
        "the widest band (3 strips of G = 126)": any(l["S"] == 3 and l["G"] == 126 for l in ls),
        "a row one strip wider (2 bands of 2 strips)": any(l["strips"] == 4 and l["bands"] == 2 for l in ls),
        "a narrower last band (5 strips: 3 + 2)": any(l["strips"] == 5 and l["last_band_strips"] == 2 for l in ls),
        "a row-tile seam inside a band of several strips": any(l["tiles"] and l["S"] > 1 for l in ls),
    }
    if policy == "r21":
        claims["a short last band under VPPB_BOX_R"] = any(l["R"] == 21 and 0 < l["last_rows"] < 21 for l in ls)
    return [k for k, ok in claims.items() if not ok]


def cases(big=False):
    c = bg._case
    B, T = ("batch",), ("tiles",)
    K = [
        # one band per image (on 2 SMs: 4 images; on 132: 128) and several (tall images)
        c("one_band_c3_24x1920x4", "vuchar3", 24, 1920, n=4, entries=B),
        c("bands_c3_300x1920x2", "vuchar3", 300, 1920, n=2, entries=B),
        c("bands_c3_61x1920x3_out_a4", "vuchar3", 61, 1920, n=3, oa=4, entries=B),
        # ragged last strips inside a band: 2 strips of 64 + 63 groups, 3 of 85 + 85 + 83
        c("ragged_c3_673", "vuchar3", 23, 673, n=3, entries=B),
        c("ragged_u8_4033", "u8", 19, 4033, n=3, entries=B),
        # the widest band (378 groups: 3 strips of 126), one byte wider (4 strips: 2 bands of 2), 5 strips (bands of 3 + 2)
        c("widest_u8_6048", "u8", 21, 6048, n=2, entries=B),
        c("widest_c3_2016", "vuchar3", 13, 2016, n=2, entries=B),
        c("wider_u8_6049", "u8", 21, 6049, n=2, entries=B),
        c("five_strips_u8_9000", "u8", 17, 9000, n=2, entries=B),
        # rows around the forced R = 21: a short last band
        c("rows_50_c3_1920", "vuchar3", 50, 1920, n=2, entries=B),
        c("rows_43_u8_6049", "u8", 43, 6049, n=2, entries=B),
        # more tasks than resident CTAs
        c("tasks_c3_100x1920x33", "vuchar3", 100, 1920, n=33, entries=B),
        # row-tile seams inside bands of 3 and of 2 strips, and a 2 + 3 tile chain in a 5-strip row
        c("tiles_c3_60x1920", "vuchar3", 60, 1920, tiles=3, entries=T),
        c("tiles_a16_u8_44x4033", "u8", 44, 4033, ia=16, tiles=2, entries=T),
        c("tiles_u8_90x9000", "u8", 90, 9000, ib=3, ia=32, tiles=3, entries=T),
    ]
    if big:
        K.append(c("one_band_c3_24x1920x128", "vuchar3", 24, 1920, n=128, entries=B))
        K.append(c("bands_c3_1080x3840x16", "vuchar3", 1080, 3840, n=16, entries=B))
        K.append(c("tasks_c3_12x7680x128", "vuchar3", 12, 7680, n=128, entries=B))  # 8K rows: 4 bands of 3 strips, 512 tasks
    return K


class Runner(bg.Runner):
    """box_geometry's runner with the band plan in place of the strip plan"""

    def run_case(self, k):
        bg.plan = band_plan  # the launches run_case reports
        try:
            return super().run_case(k)
        finally:
            bg.plan = _kernel_plan


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=("gpu", "emu"), required=True)
    ap.add_argument("--big", action="store_true", help="add 128 images of one band each, 4K x 16 and 128 images of 8K rows")
    args = ap.parse_args()
    vpp, sms = bg._load(args.backend)
    env = {k: os.environ[k] for k in bg.KNOBS if k in os.environ}
    run = Runner(vpp, sms, env)
    results = []
    for k in cases(big=args.big):
        results.extend(run.run_case(k))
    print(json.dumps(dict(backend=args.backend, sms=sms, env=env, results=results)))


def run_child(backend, policy, big=False, env=None, timeout=1200):
    """the table in a child process under POLICIES[policy]: (returncode, parsed JSON or None, stderr)"""
    e = {k: v for k, v in (env if env is not None else os.environ).items() if k not in bg.KNOBS}
    e.update(POLICIES[policy])
    cmd = [sys.executable, "-m", "tests.box_bands", "--backend", backend] + (["--big"] if big else [])
    r = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=timeout)
    try:
        res = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    except (ValueError, IndexError):
        res = None
    return r.returncode, res, r.stderr


if __name__ == "__main__":
    main()
