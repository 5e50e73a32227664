"""Child process of the semi-dense flow dispatch tests (tests/test_gpu_flow_paths.py, tests/test_emulated_flow_paths.py).

vppb_sdof_u8 (vpp_b200/csrc/sdof.cu) hides several schedules behind one entry point:
  * propagation <= 30: the relaxation kernel k_sdof_fused<MINB>, the whole call in one cooperative launch whose grid is capped at
    what is resident at once (grid-stride loops cover the rest); VPPB_SDOF_OCC=3|4 selects another MINB, hence another cap;
  * propagation > 30: the dataflow schedule, k_sdof_sweep, one persistent launch per sweep;
  * VPPB_SDOF_SCHEDULE=dataflow|levels|antidiagonals forces one of the launch-per-sweep schedules; `levels` itself runs a sweep as
    anti-diagonal launches when the dependency levels of the marked cells would not halve the launches.
So each policy runs in a process of its own:

    python -m tests.flow_paths --backend gpu|emu --policy NAME [--big]

runs the case table below through ops.semi_dense_optical_flow ("ops", which builds 128-byte aligned pyramids with a 2 * winsize
border) and vppb_sdof_u8 on pyramids built here ("direct": the oracle's levels computed on the host, each whole allocation uploaded,
at alignments 128 / 16 / 4 / 1, as views at odd columns, with borders of exactly winsize / 2, and a workspace reused across calls of
different sizes).  It prints one JSON object: the SM count the library sees and, per case and entry point, pass / fail with the
first mismatch and the plan, a transcription of sdof.cu's dispatch.  Under VPPB_SDOF_STATS=1 the library prints the grid, grid
barriers and relaxation rounds of every fused call on fd 2, which the child captures around each call.

Results are compared with vo_semi_dense_flow whole, bit for bit: valid, pos and dist of every keypoint, invalid entries (zeros on
both sides) included.  A keypoint outside the frame is undefined behaviour in the reference; the library reports it invalid with
zeros and leaves the others as they would be without it, so the oracle runs on the in-frame keypoints only."""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile
import zlib

import numpy as np

from tests.box_geometry import Alloc, _load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

POLICIES = {
    "default": {},
    "occ3": {"VPPB_SDOF_OCC": "3"},
    "occ4": {"VPPB_SDOF_OCC": "4"},
    "dataflow": {"VPPB_SDOF_SCHEDULE": "dataflow"},
    "levels": {"VPPB_SDOF_SCHEDULE": "levels"},
    "antidiagonals": {"VPPB_SDOF_SCHEDULE": "antidiagonals"},
}
KNOBS = ("VPPB_SDOF_SCHEDULE", "VPPB_SDOF_OCC", "VPPB_SDOF_STATS", "VPPB_PREPARE")
SENTINEL = 0x5A
E_ARG = -2


def _atoi(s):
    m = re.match(r"\s*[+-]?\d+", s or "")
    return int(m.group()) if m else 0


# ------------------------------------------------------------------ the dispatch of vpp_b200/csrc/sdof.cu, transcribed
def cell_dims(nrows, ncols, patch, level):
    """cell_dims(): the cell map of a pyramid level (pyramid.hh:140 on pf_domain), float arithmetic as in C"""
    cr, cc = nrows // patch, ncols // patch
    for _ in range(level):
        cr, cc = int(np.float32(1) + np.float32(cr) / np.float32(2)), int(np.float32(1) + np.float32(cc) / np.float32(2))
    return cr, cc


def level_dims(nrows, ncols, nscales):
    dims = []
    for _ in range(nscales):
        dims.append((nrows, ncols))
        nrows, ncols = int(np.float32(1) + np.float32(nrows) / np.float32(2)), int(np.float32(1) + np.float32(ncols) / np.float32(2))
    return dims


def marked_cells(kps, nrows, ncols, patch, scale):
    """the cells k_sdof_claim marks at `scale` (they stay marked through every sweep): a set of (fr, fc)"""
    cr, cc = cell_dims(nrows, ncols, patch, scale)
    lr, lc = level_dims(nrows, ncols, scale + 1)[scale]
    out = set()
    d = 1 << scale
    for r, c in kps:
        if r < 0 or c < 0 or r >= nrows or c >= ncols:  # outside the frame: claims nothing at any scale
            continue
        pr, pc = int(r) // d, int(c) // d
        if pr // patch < cr and pc // patch < cc and pr < lr and pc < lc:
            out.add((pr // patch, pc // patch))
    return out


def dependency_levels(marks, lr, lc, cr, cc, patch, forward):
    """k_sdof_levels: the number of levels of one sweep (1 + the longest chain of marked cells ordered by the sweep)"""
    sgn = 1 if forward else -1
    qr, qc = (lr - 1) // patch, (lc - 1) // patch
    order = []
    for fr, fc in marks:
        kr, kc = (fr, fc) if forward else (qr - fr, qc - fc)
        order.append((kc + 2 * kr, kr, fr, fc))
    order.sort()
    lv = {}
    for _, _, fr, fc in order:
        v = 0
        for pr, pc in ((fr, fc - sgn), (fr - sgn, fc - sgn), (fr - sgn, fc), (fr - sgn, fc + sgn)):
            if 0 <= pr < cr and 0 <= pc < cc and (pr, pc) in marks:
                v = max(v, lv[(pr, pc)] + 1)
        lv[(fr, fc)] = v
    return max(lv.values()) + 1 if lv else 0


def sdof_plan(nrows, ncols, ws, nscales, min_scale, prop, patch, kps, env):
    """the schedule vppb_sdof_u8 takes for this call: relaxation (with the MINB and the grid the work asks for before the cap),
    dataflow, rejected (VPPB_E_ARG, nothing launched), antidiagonals, or levels with the outcome of every (scale, sweep)"""
    sched = env.get("VPPB_SDOF_SCHEDULE")
    levels, waves, flags = sched == "levels", sched == "antidiagonals", sched == "dataflow"
    if not (levels or waves or flags) and prop <= 30:
        occ = _atoi(env.get("VPPB_SDOF_OCC")) if "VPPB_SDOF_OCC" in env else 2
        cr0, cc0 = cell_dims(nrows, ncols, patch, min_scale)
        want = max(len(kps), cr0 * cc0)
        return dict(schedule="relaxation", minb=4 if occ == 4 else 3 if occ == 3 else 2, want_blocks=max(1, (want + 7) // 8))
    if not (levels or waves):
        if prop > 255 or nscales * prop > 256:
            return dict(schedule="rejected")
        return dict(schedule="dataflow")
    if waves:
        return dict(schedule="antidiagonals")
    outcomes = []
    dims = level_dims(nrows, ncols, nscales)
    for s in range(nscales - 1, min_scale - 1, -1):
        lr, lc = dims[s]
        cr, cc = cell_dims(nrows, ncols, patch, s)
        nkr, nkc = (lr + patch - 1) // patch, (lc + patch - 1) // patch
        marks = marked_cells(kps, nrows, ncols, patch, s)
        for fwd in sorted({k % 2 for k in range(prop)}):
            nl = dependency_levels(marks, lr, lc, cr, cc, patch, fwd)
            outcomes.append(dict(scale=s, forward=fwd, nlevels=nl, waves=nkc + 2 * (nkr - 1), path="levels" if 2 * nl <= nkc + 2 * (nkr - 1) else "antidiagonals"))
    return dict(schedule="levels", sweeps=outcomes)


STATS = re.compile(r"vppb_sdof_u8: grid (\d+) x 256, (\d+) grid barriers, (\d+) relaxation rounds after the first of each sweep, (\d+) re-evaluations")


def parse_stats(text):
    m = STATS.findall(text)
    return [dict(grid=int(g), barriers=int(b), rounds=int(r), reevals=int(e)) for g, b, r, e in m]


# ------------------------------------------------------------------ what each policy's table must reach
def reached(res):
    out = set()
    for r in res["results"]:
        p, st = r["plan"], r.get("stats")
        out.add("schedule " + p["schedule"])
        if p["schedule"] == "relaxation" and st:
            if st["grid"] < p["want_blocks"]:
                out.add("a fused grid smaller than its work")
            if st["rounds"] >= 20:
                out.add("at least 20 relaxation rounds")
        if p["schedule"] == "dataflow" and r["prop"] == 31:
            out.add("propagation 31 on the dataflow schedule")
        if p["schedule"] == "rejected" and r["prop"] == 256:
            out.add("256 sweeps rejected")
        if p["schedule"] == "levels":
            out.update("levels: %s" % s["path"] for s in p["sweeps"])
            if r.get("moved_beyond_65535") and any(s["path"] == "levels" and s["nlevels"] > 1 for s in p["sweeps"]):
                out.add("levels: a chain of cells beyond column 65535")
    return out


def expected(policy):
    env = POLICIES[policy]
    if env.get("VPPB_SDOF_SCHEDULE") == "levels":
        return {"schedule levels", "levels: levels", "levels: antidiagonals", "levels: a chain of cells beyond column 65535"}
    if env.get("VPPB_SDOF_SCHEDULE") == "antidiagonals":
        return {"schedule antidiagonals"}
    if env.get("VPPB_SDOF_SCHEDULE") == "dataflow":
        return {"schedule dataflow", "256 sweeps rejected"}
    return {"schedule relaxation", "schedule dataflow", "a fused grid smaller than its work", "at least 20 relaxation rounds",
            "propagation 31 on the dataflow schedule", "256 sweeps rejected"}


def every_path():
    """every schedule, both outcomes of `levels`, the relaxation kernel's grid-stride loops and long relaxations, the rejection"""
    return {"schedule relaxation", "schedule dataflow", "schedule levels", "schedule antidiagonals", "schedule rejected", "levels: levels",
            "levels: antidiagonals", "a fused grid smaller than its work", "at least 20 relaxation rounds", "propagation 31 on the dataflow schedule",
            "256 sweeps rejected"}


def capped_grids(res):
    """{case/entry: grid} of the relaxation calls whose grid the cap cut below the work"""
    return {"%s/%s" % (r["case"], r["entry"]): r["stats"]["grid"] for r in res["results"]
            if r["plan"]["schedule"] == "relaxation" and r.get("stats") and r["stats"]["grid"] < r["plan"]["want_blocks"]}


# ------------------------------------------------------------------ the case table
LAYOUTS = ("a128", "a16", "a4", "a1", "view", "mixed")


def _case(name, shape, ws=7, patch=5, nscales=2, min_scale=0, prop=2, kps="grid", scene="shift", shift=(2.0, -1.0), layout="a16",
          entries=("ops", "direct"), policies=None):
    """kps: grid (one per cell, partial cells included), multi (several per cell, duplicates, shuffled), edge (corners, partial cell
    row / column, out of frame), none (n = 0, NULL arrays on the direct entry), many (more than the resident warps), pairs (horizontal
    pairs beyond column 65535), every (the centre of every cell); layout: the direct entry's pyramids (see Runner._level)"""
    return dict(name=name, shape=shape, ws=ws, patch=patch, nscales=nscales, min_scale=min_scale, prop=prop, kps=kps, scene=scene, shift=shift,
                layout=layout, entries=entries, policies=policies)


WIDE = (4, 65800)  # patch 1: cells beyond column 65535 overflowed the levels schedule's (kr << 16 | kc) cell records


def cases(sms, big=False):
    T = []
    # every window size (even ones too) with its own patch, scales, min_scale, sweeps and layout
    for i, (ws, patch, ns, shape) in enumerate([(1, 3, 1, (31, 47)), (2, 5, 2, (37, 53)), (3, 2, 3, (29, 38)), (4, 7, 2, (45, 59)),
                                                (8, 1, 2, (17, 23)), (13, 16, 1, (41, 70)), (15, 5, 3, (43, 57))]):
        T.append(_case("ws%d_p%d_s%d" % (ws, patch, ns), shape, ws=ws, patch=patch, nscales=ns, min_scale=i % ns, prop=i % 5,
                       kps=("grid", "multi", "edge")[i % 3], layout=LAYOUTS[i % len(LAYOUTS)]))
    # every patch size against window 9 / 5
    for i, patch in enumerate((1, 2, 3, 5, 7, 16)):
        T.append(_case("patch%d" % patch, (21, 26) if patch == 1 else (47, 61), ws=(9, 5)[i % 2], patch=patch, nscales=1 + i % 3, min_scale=(i // 2) % (1 + i % 3),
                       prop=(1, 2, 3, 4, 0, 2)[i], kps=("multi", "edge", "grid")[i % 3], layout=LAYOUTS[(i + 2) % len(LAYOUTS)]))
    # 1 .. 8 scales (coarse levels smaller than one patch), every min_scale of 4 and 8 scales
    for ns in range(1, 9):
        T.append(_case("scales%d" % ns, (45, 61), ws=5, patch=5, nscales=ns, min_scale=ns // 2, prop=1 + ns % 3, kps=("grid", "multi")[ns % 2],
                       layout=LAYOUTS[ns % len(LAYOUTS)]))
    for ms in range(4):
        T.append(_case("scales4_min%d" % ms, (40, 56), ws=7, patch=3, nscales=4, min_scale=ms, prop=2, kps="edge", layout=LAYOUTS[(ms + 3) % len(LAYOUTS)]))
    for ms in (1, 3, 7):
        T.append(_case("scales8_min%d" % ms, (33, 44), ws=3, patch=2, nscales=8, min_scale=ms, prop=3, kps="multi", layout=LAYOUTS[ms % len(LAYOUTS)], entries=("direct",)))
    # sweeps: 30 (the last relaxation case), 31 / 32 (the first dataflow cases, ending on a backward / forward sweep), on a shift the
    # descent cannot reach from a zero prediction: long chains of moving cells
    for prop in (30, 31, 32):
        T.append(_case("prop%d" % prop, (36, 51), ws=9, patch=3, nscales=2, prop=prop, kps="grid", shift=(6.0, -5.0), layout=("a1", "view", "a4")[prop - 30]))
    T.append(_case("chains_prop4", (64, 96), ws=9, patch=3, nscales=1, prop=4, kps="grid", shift=(6.0, -5.0), layout="a128"))
    T.append(_case("chains_p2_prop6", (60, 150), ws=7, patch=2, nscales=1, prop=6, kps="grid", shift=(6.0, -5.0), layout="a16"))
    T.append(_case("prop255_s1", (16, 22), ws=3, patch=3, nscales=1, prop=255, kps="grid", shift=(4.0, 3.0), layout="a1", entries=("direct",)))
    T.append(_case("prop128_s2", (20, 27), ws=5, patch=3, nscales=2, prop=128, kps="multi", shift=(4.0, 3.0), layout="mixed", entries=("direct",)))
    T.append(_case("prop256_s1", (16, 22), ws=3, patch=3, nscales=1, prop=256, kps="grid", shift=(4.0, 3.0), layout="a4"))
    # frames smaller than one patch: an empty cell map at level 0, one cell at the coarser levels
    T.append(_case("tiny_3x4_p5", (3, 4), ws=3, patch=5, nscales=3, prop=2, kps="edge", layout="a1"))
    T.append(_case("tiny_2x2_p3", (2, 2), ws=1, patch=3, nscales=2, min_scale=1, prop=1, kps="multi", layout="view"))
    # keypoints: none; more than the resident warps on a small frame
    T.append(_case("no_keypoints", (30, 40), ws=5, patch=5, nscales=2, prop=2, kps="none", layout="a16"))
    T.append(_case("many_keypoints", (30, 41), ws=5, patch=5, nscales=2, prop=2, kps="many", layout="a4"))
    # scenes where SADs tie (the visiting order decides) and saturated content
    T.append(_case("periodic", (35, 49), ws=5, patch=3, nscales=2, prop=3, kps="multi", scene="periodic", layout="a1"))
    T.append(_case("flat", (40, 52), ws=7, patch=4, nscales=2, prop=2, kps="grid", scene="flat", layout="mixed"))
    T.append(_case("saturated", (33, 47), ws=9, patch=5, nscales=3, min_scale=1, prop=3, kps="multi", scene="saturated", layout="view"))
    # the wide frame of the levels schedule: horizontal pairs of cells (two dependency levels) whose sweeps move them, beyond column 65535
    T.append(_case("wide_p1", WIDE, ws=3, patch=1, nscales=1, prop=1, kps="pairs", shift=(0.0, 4.0), layout="a128", entries=("direct",),
                   policies=("default", "dataflow", "levels")))
    if big:
        # video_extruder's settings with a keypoint in every cell
        for shape in ((1080, 1920), (2160, 3840)):
            T.append(_case("every_cell_%dx%d" % shape, shape, ws=9, patch=5, nscales=3, prop=2, kps="every", shift=(3.0, -2.0), layout="a128"))
        T.append(_case("wide_p1_big", (7, 70000), ws=5, patch=1, nscales=1, prop=3, kps="pairs", shift=(0.0, 4.0), layout="a1", entries=("direct",)))
    return T


# ------------------------------------------------------------------ scenes and keypoints
def scene(k):
    from tests import scenes

    nr, nc = k["shape"]
    seed = zlib.crc32(k["name"].encode()) & 0xFFFF
    if k["scene"] in ("shift", "flat"):
        f1, f2, _ = scenes.lk_pair(nr, nc, 4, seed=seed, shift=k["shift"], margin=1)
        if k["scene"] == "flat":
            f1[nr // 4:nr // 4 + nr // 2, nc // 3:nc // 3 + nc // 2] = 140
            f2[nr // 4:nr // 4 + nr // 2, nc // 3:nc // 3 + nc // 2] = 140
        return f1, f2
    rr, cc = np.meshgrid(np.arange(nr), np.arange(nc), indexing="ij")
    if k["scene"] == "periodic":  # period 4 x 3: every window has exact copies two and three pixels away
        f1 = ((cc % 4) * 50 + (rr % 3) * 30 + 20).astype(np.uint8)
        return f1, np.roll(f1, (1, 2), axis=(0, 1))
    f1 = np.where(scenes.smooth_noise(nr, nc, seed) > 0.5, 255, 0).astype(np.uint8)  # saturated
    return f1, np.roll(f1, (2, -1), axis=(0, 1))


def keypoints(k, sms):
    nr, nc = k["shape"]
    p = k["patch"]
    rng = np.random.default_rng(zlib.crc32(k["name"].encode()))
    kind = k["kps"]
    if kind == "none":
        return np.zeros((0, 2), np.int32)
    if kind == "every":
        rr, cc = np.meshgrid(np.arange(p // 2, nr, p), np.arange(p // 2, nc, p), indexing="ij")
        return np.stack([rr.ravel(), cc.ravel()], 1).astype(np.int32)
    if kind == "grid":  # one per cell, the partial last cell row and column included, in raster order
        rr, cc = np.meshgrid(np.arange(0, nr, p), np.arange(0, nc, p), indexing="ij")
        pts = np.stack([rr.ravel(), cc.ravel()], 1) + rng.integers(0, p, (rr.size, 2))
        return np.minimum(pts, [nr - 1, nc - 1]).astype(np.int32)
    if kind == "multi":  # several keypoints per cell in shuffled order (the owner is the lowest index), duplicates
        n = max(4, 3 * (nr // p + 1) * (nc // p + 1))
        pts = np.stack([rng.integers(0, nr, n), rng.integers(0, nc, n)], 1)
        pts = np.concatenate([pts, pts[rng.integers(0, n, n // 4)]])
        return pts[rng.permutation(len(pts))].astype(np.int32)
    if kind == "many":  # more keypoints than resident warps (64 per SM)
        n = 64 * sms + 37
        return np.stack([rng.integers(0, nr, n), rng.integers(0, nc, n)], 1).astype(np.int32)
    if kind == "pairs":
        pts = []
        for j in range(240):
            c = nc - 480 + 2 * j + int(rng.integers(0, 2))
            r = int(rng.integers(0, nr))
            pts += [(r, c), (r, min(c + 1, nc - 1))]
        pts += [(int(rng.integers(0, nr)), int(rng.integers(0, nc - 500))) for _ in range(40)]
        return np.array(pts, np.int32)
    # edge: corners, the partial cell row and column, a few interior points, outside the frame
    inner = [(int(rng.integers(0, nr)), int(rng.integers(0, nc))) for _ in range(max(6, (nr // p) * (nc // p) // 2))]
    edge = [(0, 0), (nr - 1, nc - 1), (nr - 1, 0), (0, nc - 1), (nr - 1, nc // 2), (nr // 2, nc - 1), ((nr // p) * p, 1), (1, (nc // p) * p)]
    out = [(-1, 5), (5, -3), (nr, 2), (2, nc), (-7, -7), (nr + 100, nc + 100)]
    pts = [q for q in inner + edge + out]
    pts = [pts[i] for i in rng.permutation(len(pts))]
    return np.array(pts, np.int32)


def oracle_flow(o, f1, f2, kps, k):
    """vo_semi_dense_flow on the in-frame keypoints; zeros for the others"""
    from tests import oracle as orc

    nr, nc = k["shape"]
    n = len(kps)
    pos, dist, valid = np.zeros((n, 2), np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint8)
    inside = np.flatnonzero((kps[:, 0] >= 0) & (kps[:, 1] >= 0) & (kps[:, 0] < nr) & (kps[:, 1] < nc)) if n else np.zeros(0, np.int64)
    kin = np.ascontiguousarray(kps[inside])
    m = len(kin)
    rp, rd, rv = np.zeros((max(m, 1), 2), np.int32), np.zeros(max(m, 1), np.int32), np.zeros(max(m, 1), np.uint8)
    h1, h2 = orc.HostImage(nr, nc, "u8", data=f1), orc.HostImage(nr, nc, "u8", data=f2)
    o.vo_semi_dense_flow(h1.ptr(), h2.ptr(), kin.ctypes.data if m else None, m, k["ws"], k["nscales"], k["min_scale"], k["prop"], k["patch"],
                         rp.ctypes.data, rd.ctypes.data, rv.ctypes.data)
    pos[inside], dist[inside], valid[inside] = rp[:m], rd[:m], rv[:m]
    return pos, dist, valid


def first_diff(got, want):
    """None, or the first keypoint where (valid, pos, dist) differ"""
    g = np.concatenate([got[2].reshape(-1, 1).astype(np.int64), got[0].reshape(-1, 2), got[1].reshape(-1, 1)], 1)
    w = np.concatenate([want[2].reshape(-1, 1).astype(np.int64), want[0].reshape(-1, 2), want[1].reshape(-1, 1)], 1)
    bad = np.flatnonzero((g != w).any(axis=1))
    if not len(bad):
        return None
    i = int(bad[0])
    return dict(index=i, got=g[i].tolist(), want=w[i].tolist(), n_differ=int(len(bad)))


class _Fd2:
    """what the library writes on fd 2 (VPPB_SDOF_STATS) while the block runs"""

    def __enter__(self):
        sys.stderr.flush()
        self.tmp = tempfile.TemporaryFile()
        self.saved = os.dup(2)
        os.dup2(self.tmp.fileno(), 2)
        return self

    def __exit__(self, *a):
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.tmp.seek(0)
        self.text = self.tmp.read().decode("utf-8", "replace")
        self.tmp.close()
        sys.stderr.write(STATS.sub("", self.text).strip("\n"))  # anything else the call printed stays visible


class Runner:
    def __init__(self, vpp, sms, env, backend):
        from tests import oracle as orc
        from vpp_b200 import capi, ops

        self.vpp, self.sms, self.env, self.backend = vpp, sms, env, backend
        self.capi, self.ops, self.orc = capi, ops, orc
        self.ws_buf, self.ws_size = None, 0

    def _workspace(self, need):
        """the end of one buffer reused by every direct call (garbage at first, then whatever the last call left): a call that
        wrote past its workspace would leave the allocation"""
        if need > self.ws_size:
            self.ws_size = (max(need, 2 * self.ws_size) + 255) // 256 * 256
            self.ws_buf = self.ops._DeviceBuffer(self.ws_size)
            self.ws_buf.from_host(np.random.default_rng(9).integers(0, 256, self.ws_size, dtype=np.uint8))
        return self.ws_buf.ptr + self.ws_size - need

    def _at_end(self, a, keep):
        """a device copy of `a` that ends on the last byte of its allocation; None for an empty array"""
        if a.nbytes == 0:
            return None
        size = (a.nbytes + 255) // 256 * 256
        buf = self.ops._DeviceBuffer(size)
        keep.append(buf)
        v = self.capi.VppbImg(buf.img.base + size - a.nbytes, None, 1, a.nbytes, size, 0, 1, 256)
        self.capi.check(self.capi.lib.vppb_upload(C.byref(v), np.ascontiguousarray(a).ctypes.data, a.nbytes, 0, None))
        return v

    def _level(self, h, ws, layout, which, rng, keep):
        """device copy of oracle level h (border 2 * ws, mirror-filled) in `layout`: a128 (border ws / 2 + 3), a16 / a4 / a1 (border
        exactly ws / 2; a1 rows end where the allocation ends), view (a view at an odd column of an a16 parent whose border is ws / 2),
        mixed (the first frame a4, the second a1).  Every byte the SAD window cannot reach holds garbage."""
        hb = ws // 2
        if layout == "mixed":
            layout = ("a4", "a1")[which]
        nr, nc = h.nrows, h.ncols
        if layout == "view":
            vr, vc = hb + 1, hb + 3 - hb % 2  # an odd column
            a = Alloc(self.vpp, nr + vr + hb + 2, nc + vc + hb + 3, "u8", hb, 16)
            img = a.img.subimage(self.vpp.Box2d((vr, vc), (vr + nr - 1, vc + nc - 1)))
        else:
            align = int(layout[1:])
            a = Alloc(self.vpp, nr, nc, "u8", hb + 3 if align == 128 else hb, align)
            img = a.img
        host = rng.integers(0, 256, a.shape, dtype=np.uint8)
        r0, c0 = a.at(img.desc)
        host[r0 - hb:r0 + nr + hb, c0 - hb:c0 + nc + hb] = h._frame_view(hb)
        a.put(host)
        keep.append(a)
        return img.desc

    def run_case(self, k):
        from tests.oracle_ops import oracle_pyramid

        capi, ops = self.capi, self.ops
        nr, nc = k["shape"]
        f1, f2 = scene(k)
        kps = keypoints(k, self.sms)
        n = len(kps)
        o = self.orc.load()
        want = oracle_flow(o, f1, f2, kps, k)
        moved = None
        if k["kps"] == "pairs":  # the sweeps move cells beyond column 65535: the oracle without propagation differs there
            still = oracle_flow(o, f1, f2, kps, dict(k, prop=0))
            moved = int(((still[0] != want[0]).any(axis=1) & (kps[:, 1] > 65535)).sum())
        plan = sdof_plan(nr, nc, k["ws"], k["nscales"], k["min_scale"], k["prop"], k["patch"], kps, self.env)
        P = capi.VppbSdofParams(k["ws"], k["nscales"], k["min_scale"], k["prop"], k["patch"])
        results = []
        for entry in k["entries"]:
            if entry == "ops" and any(min(d) < 2 * k["ws"] for d in level_dims(nr, nc, k["nscales"])):
                continue  # the library's mirror fill takes no border wider than the level: the direct entry covers these pyramids
            rc, got, fd2 = 0, None, None
            if entry == "ops":
                i1, i2 = self.vpp.Image2d.from_host(f1, "u8"), self.vpp.Image2d.from_host(f2, "u8")
                with _Fd2() as fd2:
                    try:
                        pos, dist, valid = ops.semi_dense_optical_flow(kps, i1, i2, winsize=k["ws"], nscales=k["nscales"], min_scale=k["min_scale"],
                                                                       propagation=k["prop"], patchsize=k["patch"])
                        got = (pos, dist, valid.astype(np.uint8))
                    except capi.VppbError as e:
                        rc = e.code
            else:
                rng = np.random.default_rng(zlib.crc32((k["name"] + "/levels").encode()))
                keep = []
                hp = oracle_pyramid(f1, k["nscales"], "u8", 2 * k["ws"], o)
                hn = oracle_pyramid(f2, k["nscales"], "u8", 2 * k["ws"], o)
                d1 = [self._level(h, k["ws"], k["layout"], 0, rng, keep) for h in hp]
                d2 = [self._level(h, k["ws"], k["layout"], 1, rng, keep) for h in hn]
                need = capi.lib.vppb_sdof_workspace_bytes(nr, nc, C.byref(P))
                ws = self._workspace(need)
                kp = self._at_end(kps, keep)
                outs = [self._at_end(np.full(n * s, SENTINEL, np.uint8), keep) for s in (8, 4, 1)]
                ptr = lambda v: v.base if v is not None else None
                with _Fd2() as fd2:
                    rc = capi.lib.vppb_sdof_u8((capi.VppbImg * len(d1))(*d1), (capi.VppbImg * len(d2))(*d2), C.byref(P), ptr(kp), n, ws, need,
                                               ptr(outs[0]), ptr(outs[1]), ptr(outs[2]), None)
                    capi.check(capi.lib.vppb_sync(None))
                raw = []
                for v, s in zip(outs, (8, 4, 1)):
                    a = np.empty(n * s, np.uint8)
                    if v is not None:
                        capi.check(capi.lib.vppb_download(C.byref(v), a.ctypes.data, a.nbytes, 0, None))
                    raw.append(a)
                capi.check(capi.lib.vppb_sync(None))
                if rc == 0:
                    got = (raw[0].view(np.int32).reshape(-1, 2), raw[1].view(np.int32), raw[2])
                elif not all((a == SENTINEL).all() for a in raw):
                    rc = "rejected after writing its outputs"
                del keep
            stats = parse_stats(fd2.text)
            bad, err = None, None
            if plan["schedule"] == "rejected":
                err = None if rc == E_ARG else "expected VPPB_E_ARG, got %r" % (rc,)
            elif rc != 0:
                err = "returned %r" % (rc,)
            else:
                bad = first_diff(got, want)
            if (plan["schedule"] == "relaxation") != (len(stats) == 1):
                err = err or "the plan says %s, the library printed %d relaxation statistics" % (plan["schedule"], len(stats))
            if stats and plan["schedule"] == "relaxation" and stats[0]["grid"] > plan["want_blocks"]:
                err = err or "grid %d above the %d blocks the work asks for" % (stats[0]["grid"], plan["want_blocks"])
            results.append(dict(case=k["name"], entry=entry, ok=bad is None and err is None, mismatch=bad, error=err, n=n, prop=k["prop"], ncols=nc,
                                plan=plan, stats=stats[0] if stats else None, valid=int(want[2].sum()), moved_beyond_65535=moved))
        return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=("gpu", "emu"), required=True)
    ap.add_argument("--policy", choices=list(POLICIES), required=True)
    ap.add_argument("--big", action="store_true", help="add 1080p and 4K with a keypoint in every cell, and a wider levels frame")
    ap.add_argument("--only", default=None, help="run the cases whose name contains this string")
    args = ap.parse_args()
    vpp, sms = _load(args.backend)
    env = {k: os.environ[k] for k in KNOBS if k in os.environ}
    run = Runner(vpp, sms, env, args.backend)
    results = []
    for k in cases(sms, big=args.big):
        if (k["policies"] is None or args.policy in k["policies"]) and (args.only is None or args.only in k["name"]):
            results.extend(run.run_case(k))
    print(json.dumps(dict(backend=args.backend, policy=args.policy, sms=sms, env=env, results=results)))


def run_child(backend, policy, big=False, env=None, timeout=3000, only=None):
    """run the table under POLICIES[policy] (the other knobs cleared, VPPB_SDOF_STATS=1) in a child process:
    (returncode, parsed JSON or None, stderr)"""
    e = {k: v for k, v in (env if env is not None else os.environ).items() if k not in KNOBS}
    e.update(POLICIES[policy])
    e["VPPB_SDOF_STATS"] = "1"
    cmd = [sys.executable, "-m", "tests.flow_paths", "--backend", backend, "--policy", policy] + (["--big"] if big else []) + (["--only", only] if only else [])
    r = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=timeout)
    try:
        res = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    except (ValueError, IndexError):
        res = None
    return r.returncode, res, r.stderr


def failures(res):
    return [r for r in res["results"] if not r["ok"]]


def unmet(res, policy):
    """what the policy's table is written to reach and, by the transcribed dispatch and the captured statistics, no longer reaches"""
    return sorted(expected(policy) - reached(res))


if __name__ == "__main__":
    main()
