"""Child process of the FAST9 / Lucas-Kanade dispatch tests (tests/test_gpu_detector_paths.py, tests/test_emulated_detector_paths.py).

Both hot paths hide several kernels behind one entry point:
  * fast9_core runs the TMA band kernel k_fast9_band<ring, mask> on images in the library layout and k_fast9_detect on every other
    image (views, alignment below 16, foreign pitches) or under VPPB_FAST_IMPL=warp, which the library reads once per process;
  * vppb_lk_match_u8 runs k_lk_match_v2<PPL, GF, WARPS> for windows up to 11 (WARPS from VPPB_LK_WARPS, read on every call) and the
    one-keypoint-per-warp k_lk_match<PPL, GF> for windows 13 and 15, for pyramids with a level of 2 GiB or more, or under VPPB_LK_V1=1
    (read once per process).
So each policy runs in a process of its own:

    python -m tests.detector_paths --backend gpu|emu --policy NAME [--big]

runs the FAST case table (policies that touch FAST) and the LK case table (policies that touch LK) under that policy's knobs, the
others cleared, and prints one JSON object: the SM count the library sees and, per case and entry point, pass / fail with the first
mismatch and the kernels the dispatch takes for it (`plan`, a transcription of fast.cu's and lk.cu's dispatch rules).

FAST results (keypoints, ranks, scores) must equal the C oracle's exactly; the oracle reads the same bytes the kernel reads (the
whole allocation is uploaded from the host, border and pitch padding included, and a view's ring reaches into its parent's pixels).
LK flows and errors must equal the oracle's bit for bit, failure codes included: the kernels replay the oracle's float sequence.  The
one exception is the payload of a NaN error (a flat template under SAD / MAD divides 0 by 0): the H100 writes 0x7FFFFFFF where x86
writes 0xFFC00000, so NaN compares equal to NaN and to nothing else."""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import zlib

import numpy as np

from tests.box_geometry import Alloc, _load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# one child per policy: VPPB_FAST_IMPL and VPPB_LK_V1 are read once per process; "tables" are the case tables the policy can change
POLICIES = {
    "default": dict(env={}, tables=("fast", "lk")),
    "fast_warp": dict(env={"VPPB_FAST_IMPL": "warp"}, tables=("fast",)),
    "lk_v1": dict(env={"VPPB_LK_V1": "1"}, tables=("lk",)),
    "lk_warps1": dict(env={"VPPB_LK_WARPS": "1"}, tables=("lk",)),
    "lk_warps2": dict(env={"VPPB_LK_WARPS": "2"}, tables=("lk",)),
}
KNOBS = ("VPPB_FAST_IMPL", "VPPB_LK_V1", "VPPB_LK_WARPS")
FLT_MAX = float(np.finfo(np.float32).max)


def _atoi(s):
    m = re.match(r"\s*[+-]?\d+", s or "")
    return int(m.group()) if m else 0


# ------------------------------------------------------------------ the dispatch of vpp_b200/csrc/fast.cu, transcribed
FB_MAXW = 65535
FAST_MODES = ("all", "local_maxima", "blockwise", "rank")
FAST_DETECTORS = ("band<0,nomask>", "band<0,mask>", "band<1,nomask>", "band<1,mask>", "detect")


def fast_band_eligible(d):
    """fast_band_eligible(): the library layout with >= 16 bytes left of column 0, 16-byte aligned pixel (0,0) and pitch"""
    if d.align < 16 or d.base % 16 or d.pitch % 16:
        return False
    bs = d.border * d.elem_bytes
    if bs % d.align:
        bs += d.align - bs % d.align
    pch = d.ncols * d.elem_bytes + 2 * bs
    if pch % d.align:
        pch += d.align - pch % d.align
    return pch == d.pitch and bs >= 16 and d.ncols <= FB_MAXW


def fast_plan(d, mode, ring, has_mask, sms, env):
    """fast9_core's launches for `mode`: the detection kernel, whether k_fast9_detect loops over its grid, and the kernels after it"""
    wpr = (d.ncols + 31) // 32
    words = d.nrows * wpr
    if mode == "scores":
        return dict(detect=None, loops=False, kernels=["scores"])
    if fast_band_eligible(d) and env.get("VPPB_FAST_IMPL") != "warp":
        det, loops = "band<%d,%s>" % (ring, "mask" if has_mask else "nomask"), False
    else:
        grid = min((words + 7) // 8, sms * 8)  # CTAs of 8 warps, one 32-pixel word per warp and trip
        det, loops = "detect", words > grid * 8
    rest = {"all": ["emit_bands"] if det != "detect" else ["scan", "emit"], "local_maxima": ["local_max", "scan", "emit"],
            "blockwise": ["block_max", "scan", "emit_cells"], "rank": ["block_rank", "scan", "emit_rank"]}[mode]
    return dict(detect=det, loops=loops, kernels=[det] + rest)


# ------------------------------------------------------------------ the dispatch of vpp_b200/csrc/lk.cu, transcribed
V2_PPL = {1: 4, 3: 4, 5: 4, 7: 7, 9: 11, 11: 16}  # lk_launch_v2w: 8 lanes per keypoint
V1_PPLS = (1, 2, 3, 4, 6, 8)
V2_PPLS = (4, 7, 11, 16)


def v1_ppl(ws):
    p = (ws * ws + 31) // 32
    return {5: 6, 7: 8}.get(p, p)


def lk_small(prev, nxt):
    """the v2 kernel addresses samples with 32-bit offsets: every prev / next level's frame (border rows included) below 2 GiB"""
    return all((p.nrows + 2 * p.border) * p.pitch < 1 << 31 and (n.nrows + 2 * n.border) * n.pitch < 1 << 31 for p, n in zip(prev, nxt))


def lk_plan(ws, gf, prev, nxt, env):
    g = "float" if gf else "int"
    if not _atoi(env.get("VPPB_LK_V1")) and lk_small(prev, nxt) and ws in V2_PPL:
        w = _atoi(env["VPPB_LK_WARPS"]) if "VPPB_LK_WARPS" in env else 4
        return dict(kernel="v2", ppl=V2_PPL[ws], warps=w if w in (1, 2) else 4, grad=g, small=True)
    return dict(kernel="v1", ppl=v1_ppl(ws), grad=g, small=lk_small(prev, nxt))


# ------------------------------------------------------------------ what each policy's tables must reach
def reached(res):
    """the kernel instantiations and LK outcomes the runs of one child reached (strings)"""
    out = set()
    for r in res["results"]:
        p = r["plan"]
        if r["table"] == "fast" and p["detect"]:
            out.add("fast %s %s" % (r["mode"], p["detect"]))
            if p["loops"]:
                out.add("fast detect loops over its grid")
        elif r["table"] == "lk":
            if p["kernel"] == "v2":
                out.add("lk v2 ppl=%d warps=%d %s" % (p["ppl"], p["warps"], p["grad"]))
            else:
                out.add("lk v1 ppl=%d %s" % (p["ppl"], p["grad"]))
                if not p["small"]:
                    out.add("lk v1 on a level of 2 GiB or more")
            out.update("lk outcome " + o for o in r["outcomes"])
    return out


def expected(policy, big=False):
    """what the tables are written to reach under `policy`; the union over POLICIES is every kernel of both dispatches"""
    env, tables = POLICIES[policy]["env"], POLICIES[policy]["tables"]
    want = set()
    if "fast" in tables:
        dets = ("detect",) if env.get("VPPB_FAST_IMPL") == "warp" else FAST_DETECTORS
        want |= {"fast %s %s" % (m, d) for m in FAST_MODES for d in dets}
        want.add("fast detect loops over its grid")
    if "lk" in tables:
        want |= {"lk outcome " + o for o in ("converged", "rejected", "left the domain")}
        if _atoi(env.get("VPPB_LK_V1")):
            want |= {"lk v1 ppl=%d %s" % (p, g) for p in V1_PPLS for g in ("int", "float")}
        else:
            w = _atoi(env["VPPB_LK_WARPS"]) if "VPPB_LK_WARPS" in env else 4
            want |= {"lk v2 ppl=%d warps=%d %s" % (p, w, g) for p in V2_PPLS for g in ("int", "float")}
            want |= {"lk v1 ppl=%d %s" % (p, g) for p in (6, 8) for g in ("int", "float")}
            if big:
                want.add("lk v1 on a level of 2 GiB or more")
    return want


def every_kernel():
    """all four k_fast9_band instantiations and k_fast9_detect in each mode; v2 PPL x WARPS x gradient; v1 PPL x gradient"""
    s = {"fast %s %s" % (m, d) for m in FAST_MODES for d in FAST_DETECTORS}
    s |= {"lk v2 ppl=%d warps=%d %s" % (p, w, g) for p in V2_PPLS for w in (1, 2, 4) for g in ("int", "float")}
    s |= {"lk v1 ppl=%d %s" % (p, g) for p in V1_PPLS for g in ("int", "float")}
    return s


# ------------------------------------------------------------------ the FAST case table
def _fcase(name, nrows, ncols, border=3, align=128, view=None, ring=0, mask=None, th=20, bs=7, maxp=3, content="noise", entries=None):
    """view: (row, col) of the image in a parent of the same border / alignment (the ring reads the parent's pixels);
    mask: None or the byte of the mask's set pixels (a quarter of the mask is 0); entries: (mode, block size, max points)"""
    if entries is None:
        entries = [("all", 0, 0), ("local_maxima", 0, 0), ("blockwise", bs, 0), ("rank", bs, maxp), ("scores", 0, 0)]
    return dict(name=name, nrows=nrows, ncols=ncols, border=border, align=align, view=view, ring=ring, mask=mask, th=th, content=content,
                entries=entries)


TALL = (32800, 48)  # rows at and above 32768 held a negative packed cell keypoint (row << 16 | col in an int)


def fast_cases(sms, tall=True):
    T = []
    # widths around the 32-pixel bitmask words and the 2016-pixel band boxes, rows around the 4-row bands and the 8-row emit CTAs
    rows = (3, 4, 5, 7, 8, 9)
    for i, nc in enumerate((3, 31, 32, 33, 63, 64, 65, 2015, 2016, 2017, 4033)):
        for j, nr in enumerate((rows[i % 6], rows[(i + 3) % 6])):
            T.append(_fcase("shape_%dx%d" % (nr, nc), nr, nc, ring=(i + j) % 2, mask=(None, 0xFF)[j], th=(20, 127)[i % 2], bs=(1, 3, 7, 10, 32)[i % 5],
                            maxp=(1, 2, 3, 16)[i % 4], content=("noise", "rect")[j]))
    # both rings x no mask / masks 0xFF, 0x01, 0x10 with holes, on the band path (and on the warp path under VPPB_FAST_IMPL=warp)
    for ring in (0, 1):
        for m in (None, 0xFF, 0x01, 0x10):
            T.append(_fcase("ring%d_mask%s" % (ring, "none" if m is None else "%02x" % m), 9, 2017, ring=ring, mask=m, bs=10, maxp=3))
    # thresholds 0 (every strict arc), 127 (the packed compare's high-bit branch), 255 (nothing passes; the band kernel skips its phases)
    for th in (0, 20, 127, 255):
        T.append(_fcase("th%d" % th, 8, 65, th=th, ring=th % 2, mask=0x10 if th == 127 else None, bs=3, maxp=2))
    # alignments: 128 and 16 take the band path, 8 / 4 / 1 the warp path; border 5
    for a in (128, 16, 8, 4, 1):
        T.append(_fcase("align%d_7x33" % a, 7, 33, align=a, ring=a % 2, mask=0x01 if a in (16, 4) else None, bs=7, maxp=16))
        T.append(_fcase("align%d_9x2017" % a, 9, 2017, align=a, ring=1 - a % 2, mask=0xFF if a == 8 else None, bs=10, maxp=3))
        T.append(_fcase("border5_align%d" % a, 8, 64, border=5, align=a, ring=a % 2, bs=3, maxp=1, content="rect"))
    # views at an odd column of a library-layout parent: the warp path, the ring reading the parent's pixels around the view
    T.append(_fcase("view_0_1_8x63", 8, 63, view=(0, 1), ring=0, mask=0x10, bs=7, maxp=3))
    T.append(_fcase("view_3_7_9x2017", 9, 2017, view=(3, 7), ring=1, bs=10, maxp=2, content="rect"))
    T.append(_fcase("view_2_5_5x33_b5", 5, 33, border=5, view=(2, 5), ring=0, mask=0xFF, bs=1, maxp=16))
    # a warp-path frame of more than sms * 64 words: k_fast9_detect and k_fast9_local_max loop over their grids
    nr = max(9, sms + 5)  # 2017 pixels = 64 words per row
    T.append(_fcase("warp_loop_%dx2017" % nr, nr, 2017, align=8, ring=0, bs=10, maxp=3, content="rect"))
    if tall:
        T.append(_fcase("tall_%dx%d" % TALL, TALL[0], TALL[1], ring=0, th=20, content="tall",
                        entries=[("all", 0, 0), ("local_maxima", 0, 0), ("blockwise", 7, 0), ("blockwise", 10, 0), ("rank", 10, 1), ("rank", 7, 3),
                                 ("scores", 0, 0)]))
    return T


def fast_content(k, shape, rng):
    """bytes of the whole allocation (rows x pitch)"""
    if k["content"] == "noise":  # six grey levels: corners everywhere, scores that tie and differ
        return (rng.integers(0, 6, shape) * 51).astype(np.uint8)
    if k["content"] == "rect":
        from tests import scenes

        return scenes.rectangles_scene(shape[0], shape[1], seed=int(rng.integers(1 << 30)), nrect=max(8, shape[0] * shape[1] // 60), noise=2)
    # tall: a flat field (noise +-2, below every threshold) with isolated dots - each one a corner of its own score - near the top and
    # in the last hundred rows of a 32800-row frame
    a = rng.integers(100, 104, shape).astype(np.uint8)
    return a


def tall_dots(host, r0, c0, rng):
    """isolated dots in rows 5 .. 44 and 32700 .. 32799 of the image whose pixel (0,0) is host[r0, c0]"""
    pts = []
    for band in ((5, 45), (TALL[0] - 100, TALL[0])):
        for r in range(band[0], band[1], 5):
            for c in range(3 + (r // 5) % 4, TALL[1] - 3, 9):
                if rng.random() < 0.7:
                    host[r0 + r, c0 + c] = rng.integers(150, 256) if rng.random() < 0.6 else rng.integers(0, 60)
                    pts.append((r, c))
    return pts


# ------------------------------------------------------------------ the LK case table
COUNTS = (1, 2, 3, 4, 5, 15, 16, 17, 63, 65)


def _lcase(name, entry, ws, gf=0, n=17, nlevels=3, min_scale=0, border=None, err_mode=0, gate=0, min_ev=1.0, pred=None, niter=12, shape=(97, 129)):
    """entry: "direct" (vppb_lk_match_u8 on pyramids built by the oracle), "lucas_kanade", "pyrlk_match"; pred: None, "small"
    (prediction within 2 pixels, some keypoints pushed off the frame) - direct and lucas_kanade only"""
    if border is None:
        border = max(1, ws // 2)
    return dict(name=name, entry=entry, ws=ws, gf=gf, n=n, nlevels=nlevels, min_scale=min_scale, border=border, err_mode=err_mode, gate=gate,
                min_ev=min_ev, pred=pred, niter=niter, shape=shape)


def lk_cases(sms, big=False):
    T = []
    i = 0
    for ws in range(1, 16, 2):  # every window, both gradients, through the C entry point; borders down to 1
        for gf in (0, 1):
            T.append(_lcase("direct_ws%d_%s" % (ws, ("int", "float")[gf]), "direct", ws, gf, n=COUNTS[i % len(COUNTS)], nlevels=1 + (ws // 2 + gf) % 3,
                            err_mode=i % 2, gate=(i // 2) % 2, min_ev=(1.0, 0.0)[(i // 4) % 2] if i % 3 else 1.0, pred="small" if i % 3 != 1 else None))
            i += 1
    for ws, gf, nl, ms in ((3, 0, 5, 1), (5, 1, 6, 2), (9, 0, 7, 1), (13, 1, 8, 2), (7, 1, 8, 0), (11, 0, 5, 2), (1, 1, 6, 1), (15, 0, 5, 1)):
        T.append(_lcase("levels%d_min%d_ws%d" % (nl, ms, ws), "direct", ws, gf, n=COUNTS[(i + ws) % len(COUNTS)], nlevels=nl, min_scale=ms,
                        err_mode=ms % 2, gate=ms % 2, pred="small", shape=(150, 203)))
        i += 1
    for ws in range(5, 16, 2):  # lucas_kanade: SAD, ungated, prediction / 2^nscales, int gradient, border ws / 2
        T.append(_lcase("lucas_kanade_ws%d" % ws, "lucas_kanade", ws, 0, n=COUNTS[(3 * ws) % len(COUNTS)], nlevels=1 + ws % 3, pred="small" if ws % 4 == 1 else None,
                        niter=(21, 7, 1)[ws % 3]))
    for ws in range(1, 16, 2):  # pyrlk_match: SAD / MAD, gated, min_scale 0 or 1
        for gf in (0, 1):
            T.append(_lcase("pyrlk_match_ws%d_%s" % (ws, ("int", "float")[gf]), "pyrlk_match", ws, gf, n=COUNTS[(ws + 5 * gf) % len(COUNTS)],
                            nlevels=2 + gf, min_scale=(ws // 2) % 2, border=max(2, ws // 2), err_mode=1, gate=1))
    # more keypoints than a wave of resident CTAs (64 warps per SM, 4 keypoints per warp in v2, 1 in v1)
    wave = 64 * 4 * sms
    T.append(_lcase("wave_ws7", "direct", 7, 0, n=wave + 37, nlevels=2, pred="small"))
    T.append(_lcase("wave_ws13", "direct", 13, 1, n=wave + 37, nlevels=2, err_mode=1, gate=1))
    if big:
        # level 0 of prev with a 64 MiB pitch: 42 rows (36 + border) of 64 MiB = 2.6 GiB, so the v2 kernel's 32-bit offsets cannot
        # reach it and v1 runs with 64-bit offsets; keypoints down to row 35 sample beyond 2 GiB
        T.append(_lcase("prev_2gib", "direct", 7, 0, n=17, nlevels=1, border=3, shape=(36, 100), pred="small"))
    return T


def lk_points(n, nr, nc, flat, rng, off):
    """n keypoints that cycle through: integer and fractional interior positions, the frame edge, just outside it, the flat patch"""
    edge = [(0, 0), (nr - 1, nc - 1), (0, nc // 2), (nr // 2, 0), (nr - 1, 7), (11, nc - 1)]
    out = [(-0.5, 40), (-3.25, 60.5), (nr - 0.5, 30), (nr + 2, 70.25), (20, -0.5), (30.5, nc + 2)]
    (fr0, fr1), (fc0, fc1) = flat
    fl = [((fr0 + fr1) // 2, (fc0 + fc1) // 2), ((fr0 + fr1) / 2 + 0.25, (fc0 + fc1) / 2 - 0.5)]
    pts = []
    for i in range(n):
        cat = (i + off) % 5
        if cat == 0:
            pts.append((float(rng.integers(3, nr - 3)), float(rng.integers(3, nc - 3))))
        elif cat == 1:
            pts.append((float(rng.uniform(1, nr - 2)), float(rng.uniform(1, nc - 2))))
        elif cat == 2:
            pts.append(edge[(i // 5) % len(edge)])
        elif cat == 3:
            pts.append(out[(i // 5) % len(out)])
        else:
            pts.append(fl[(i // 5) % len(fl)])
    return np.array(pts, np.float32).reshape(-1, 2)


def lk_bits(flow, err):
    """(n, 3) int32: the bits of flow and error per keypoint, every NaN as 0x7FC00000.  A flat template under SAD / MAD gives 0 / 0:
    the GPU's NaN is 0x7FFFFFFF, x86's 0xFFC00000 - a NaN on one side only is still a difference"""
    a = np.concatenate([np.asarray(flow, np.float32).reshape(-1, 2), np.asarray(err, np.float32).reshape(-1, 1)], axis=1)
    bits = a.view(np.int32).copy()
    bits[np.isnan(a)] = 0x7FC00000
    return bits


def lk_outcome(flow, err):
    if err == FLT_MAX and flow[0] == -1 and flow[1] == -1:
        return "rejected"
    if err == FLT_MAX and flow[0] == 0 and flow[1] == 0:
        return "left the domain"
    return "converged" if np.isfinite(err) and err < FLT_MAX else "other"


# ------------------------------------------------------------------ comparisons
def first_diff(got, want):
    """None, or the first record (row of a 2-d array) where got and want differ"""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape == want.shape and np.array_equal(got, want):
        return None
    m = min(len(got), len(want))
    bad = np.flatnonzero((got[:m].reshape(m, -1) != want[:m].reshape(m, -1)).any(axis=1)) if m else np.zeros(0, np.int64)
    i = int(bad[0]) if len(bad) else m
    return dict(index=i, got=got[i].tolist() if i < len(got) else None, want=want[i].tolist() if i < len(want) else None, n_got=len(got),
                n_want=len(want), n_differ=int(len(bad)) + abs(len(got) - len(want)))


class Runner:
    def __init__(self, vpp, sms, env, backend):
        from tests import oracle as orc
        from vpp_b200 import capi, ops

        self.vpp, self.sms, self.env, self.backend = vpp, sms, env, backend
        self.capi, self.ops, self.orc = capi, ops, orc
        self._scenes = {}

    # ---- FAST
    def run_fast(self, k):
        vpp, orc, ops = self.vpp, self.orc, self.ops
        o = orc.load(omp=True)
        rng = np.random.default_rng(zlib.crc32(k["name"].encode()))
        nr, nc, b = k["nrows"], k["ncols"], k["border"]
        if k["view"] is None:
            a = Alloc(vpp, nr, nc, "u8", b, k["align"])
            img = a.img
        else:
            vr, vc = k["view"]
            a = Alloc(vpp, nr + vr + 2, nc + vc + 4, "u8", b, k["align"])
            img = a.img.subimage(vpp.Box2d((vr, vc), (vr + nr - 1, vc + nc - 1)))
        host = fast_content(k, a.shape, rng)
        r0, c0 = a.at(img.desc)
        if k["content"] == "tall":
            tall_dots(host, r0, c0, rng)
        host = np.ascontiguousarray(host)
        a.put(host)
        ov = orc.VoImg(host.ctypes.data + r0 * a.pitch + c0, nr, nc, a.pitch, b, 1)
        M = om = mhost = None
        if k["mask"] is not None:
            mhost = np.where(rng.random((nr, nc)) < 0.75, k["mask"], 0).astype(np.uint8)
            M = vpp.Image2d.from_host(mhost, "u8")
            om = orc.VoImg(mhost.ctypes.data, nr, nc, nc, 0, 1)
        ring, th = k["ring"], k["th"]
        rname = "true" if ring else "reference"
        cap = nr * nc + 16
        results = []
        for mode, bs, maxp in k["entries"]:
            plan = fast_plan(img.desc, mode, ring, M is not None, self.sms, self.env)
            name = mode if mode in ("all", "local_maxima", "scores") else "%s bs=%d" % (mode, bs) + (" maxp=%d" % maxp if mode == "rank" else "")
            if mode == "rank":
                sc = []
                got = ops.fast9_blockwise_rank(img, th, block_size=bs, max_points_per_block=maxp, mask=M, scores=sc, ring=rname)
                wk, ws = np.zeros((cap * 3, 3), np.int32), np.zeros(cap * 3, np.int32)
                n = o.vo_fast9_blockwise_rank(C.byref(ov), th, C.byref(om) if om else None, bs, maxp, ring, wk.ctypes.data, ws.ctypes.data, cap * 3)
                assert n >= 0
                want, want_sc = wk[:n], ws[:n]
            elif mode == "scores":  # the detected corners of the oracle, plus points on and outside the frame (score 0 there)
                wk = np.zeros((cap, 2), np.int32)
                n = o.vo_fast9_u8(C.byref(ov), th, None, 0, 1, ring, wk.ctypes.data, None, cap)
                step = max(1, n // 3000)
                pts = np.concatenate([wk[:n:step], np.array([[0, 0], [nr - 1, nc - 1], [-1, 0], [0, -1], [nr, 0], [0, nc], [-5, -5]], np.int32)])
                got, sc = np.zeros((len(pts), 2), np.int32), ops.fast9_scores(img, th, pts)
                want = got
                inside = (pts[:, 0] >= 0) & (pts[:, 0] < nr) & (pts[:, 1] >= 0) & (pts[:, 1] < nc)
                want_sc = np.array([o.vo_fast9_score(C.byref(ov), th, int(r), int(c)) if ok else 0 for (r, c), ok in zip(pts, inside)], np.int32)
            else:
                m = {"all": 0, "local_maxima": 1, "blockwise": 2}[mode]
                sc = []
                got = ops.fast9(img, th, local_maxima=m == 1, blockwise=m == 2, block_size=bs if m == 2 else 10, mask=M, scores=sc, ring=rname)
                wk, ws = np.zeros((cap, 2), np.int32), np.zeros(cap, np.int32)
                n = o.vo_fast9_u8(C.byref(ov), th, C.byref(om) if om else None, m, bs if m == 2 else 10, ring, wk.ctypes.data, ws.ctypes.data, cap)
                assert n >= 0
                want, want_sc = wk[:n], ws[:n]
            bad = first_diff(np.asarray(got, np.int32), want)
            what = "keypoints"
            if bad is None:
                bad, what = first_diff(np.asarray(sc, np.int32), want_sc), "scores"
            if bad is not None:
                bad["what"] = what
            results.append(dict(table="fast", case=k["name"], entry=name, mode=mode, ok=bad is None, mismatch=bad, n=int(len(want)), plan=plan))
        return results

    # ---- LK
    def _scene(self, shape, seed):
        key = (shape, seed)
        if key not in self._scenes:
            from tests import scenes

            nr, nc = shape
            f1, f2, _ = scenes.lk_pair(nr, nc, 4, seed=seed, shift=(1.3, -0.8), margin=8)
            fr, fc = (nr * 5 // 8, nr * 5 // 8 + 20), (nc * 7 // 10, nc * 7 // 10 + 30)  # a flat patch: zero gradient, G = 0
            f1[fr[0]:fr[1], fc[0]:fc[1]] = 140
            f2[fr[0]:fr[1], fc[0]:fc[1]] = 140
            self._scenes[key] = (f1, f2, (fr, fc))
        return self._scenes[key]

    def run_lk(self, k):
        from tests.oracle_ops import oracle_grad_pyramid, oracle_lk, oracle_lucas_kanade, oracle_pyramid

        vpp, orc, ops, capi = self.vpp, self.orc, self.ops, self.capi
        ws, gf, nl = k["ws"], k["gf"], k["nlevels"]
        gpix = "vfloat2" if gf else "vint2"
        rng = np.random.default_rng(zlib.crc32(k["name"].encode()))
        f1, f2, flat = self._scene(k["shape"], 3)
        nr, nc = k["shape"]
        pts = lk_points(k["n"], nr, nc, flat, rng, off=int(rng.integers(5)))
        pred = None
        if k["pred"]:
            pred = rng.uniform(-2, 2, pts.shape).astype(np.float32)
            pred[3::7] = (4000.0, -2500.0)  # pushed off the frame
        o = orc.load(omp=len(pts) > 2000)
        keep = []
        if k["entry"] == "lucas_kanade":
            i1, i2 = vpp.Image2d.from_host(f1, "u8"), vpp.Image2d.from_host(f2, "u8")
            if pred is not None:
                pred = pred * float(2 ** nl)
            flow, err = ops.lucas_kanade(i1, i2, pts, niterations=k["niter"], winsize=ws, nscales=nl, prediction=pred)
            rflow, rerr = oracle_lucas_kanade(f1, f2, pts, niterations=k["niter"], winsize=ws, nscales=nl, prediction=pred, lib=o)
            descs, (r, c) = [], (nr, nc)
            for _ in range(nl):  # the levels lucas_kanade allocates: border ws / 2, 1 + n / 2 per level
                descs.append(_Desc(r, c, ws // 2, capi.lib))
                r, c = int(1 + r / 2), int(1 + c / 2)
            plan = lk_plan(ws, 0, descs, descs, self.env)
        else:
            B = max(2, k["border"])  # the 5-tap low-pass of the oracle's pyramid reads 2 pixels out
            hp, hn = oracle_pyramid(f1, nl, "u8", B, o), oracle_pyramid(f2, nl, "u8", B, o)
            hg = oracle_grad_pyramid(hp, gpix, B, o)
            P = dict(nlevels=nl, min_scale=k["min_scale"], winsize=ws, max_iter=k["niter"], grad_is_float=gf, err_mode=k["err_mode"], gate_on_max_err=k["gate"],
                     min_ev=k["min_ev"], delta=0.05, max_err=0.5, factor=2.0, pred_div=1.0)
            if k["entry"] == "pyrlk_match":
                i1, i2 = vpp.Image2d.from_host(f1, "u8"), vpp.Image2d.from_host(f2, "u8")
                dp, dn = ops.Pyramid2d((nr, nc), nl, 2, pixel="u8", border=B), ops.Pyramid2d((nr, nc), nl, 2, pixel="u8", border=B)
                dg = ops.Pyramid2d((nr, nc), nl, 2, pixel=gpix, border=B)
                ops.pyrlk_prepare(i1, i2, dp, dn, dg)
                plan = lk_plan(ws, gf, [l.desc for l in dp.levels], [l.desc for l in dn.levels], self.env)
                flow, err, _ = ops.pyrlk_match(dp, dg, dn, pts, ws, k["min_ev"], 0.5, k["niter"], 0.05, min_scale=k["min_scale"])
                P.update(err_mode=1, gate_on_max_err=1)
                rflow, rerr = oracle_lk(hp, hn, hg, orc.VoLkParams(**P), pts, None, o)
            else:
                lb = k["border"]
                hp, hn, hg = [_reframe(orc, h, lb) for h in hp], [_reframe(orc, h, lb) for h in hn], [_reframe(orc, h, lb) for h in hg]
                dp, dn, dg = _Levels([_upload(vpp, h) for h in hp]), _Levels([_upload(vpp, h) for h in hn]), _Levels([_upload(vpp, h) for h in hg])
                if k["name"] == "prev_2gib":
                    keep.append(_huge_level0(dp, hp[0], capi))
                plan = lk_plan(ws, gf, dp.descs, dn.descs, self.env)
                flow, err = _lk_direct(capi, ops, dp, dn, dg, capi.VppbLkParams(**P), pts, pred)
                rflow, rerr = oracle_lk(hp, hn, hg, orc.VoLkParams(**P), pts, pred, o)
        del keep[:]  # the 64 MiB-pitch allocation goes here, within its case
        got, want = lk_bits(flow, err), lk_bits(rflow, rerr)
        bad = first_diff(got, want)
        if bad is not None:
            i = bad["index"]
            bad.update(keypoint=pts[i].tolist() if i < len(pts) else None, got_float=[float(flow[i, 0]), float(flow[i, 1]), float(err[i])] if i < len(flow) else None,
                       want_float=[float(rflow[i, 0]), float(rflow[i, 1]), float(rerr[i])] if i < len(rflow) else None)
        outcomes = sorted({lk_outcome(rflow[i], rerr[i]) for i in range(len(pts))})
        return [dict(table="lk", case=k["name"], entry=k["entry"], ok=bad is None, mismatch=bad, n=int(len(pts)), plan=plan, outcomes=outcomes)]


class _Desc:
    """the fields of a library-layout u8 level that lk_plan reads"""

    def __init__(self, nrows, ncols, border, lib):
        p, t, _ = C.c_int32(), C.c_int64(), C.c_int64()
        lib.vppb_layout(nrows, ncols, 1, border, 128, C.byref(p), C.byref(t), C.byref(_))
        self.nrows, self.ncols, self.border, self.pitch = nrows, ncols, border, p.value


class _Levels:
    """device pyramid levels with the desc_array() of ops.Pyramid2d (what vppb_lk_match_u8 takes)"""

    def __init__(self, imgs):
        self.imgs = imgs
        self.descs = [i.desc for i in imgs]

    def desc_array(self):
        from vpp_b200 import capi

        return (capi.VppbImg * len(self.descs))(*self.descs)


def _reframe(orc, h, b):
    """a copy of host level h with border b (b <= h.border): the bytes the oracle and the device then both read"""
    if b == h.border:
        return h
    r = orc.HostImage(h.nrows, h.ncols, h.pixel, border=b)
    r.view(True)[...] = h._frame_view(b)
    return r


def _upload(vpp, h):
    d = vpp.Image2d(h.nrows, h.ncols, h.pixel, border=h.border)
    return d.upload(h.get(True), with_border=True)


def _lk_direct(capi, ops, prev, nxt, grad, params, pts, pred):
    """vppb_lk_match_u8 with the keypoint and prediction arrays ending on the last byte of their allocations, as a caller's exact-size
    arrays do: a kernel that read past keypoint n - 1 (the idle lanes of the last CTA) would leave the allocation, which the
    AddressSanitizer leg reports"""
    n, bufs = len(pts), []

    def at_end(a):
        a = np.ascontiguousarray(a, np.float32)
        size = (a.nbytes + 255) // 256 * 256
        buf = ops._DeviceBuffer(size)
        v = capi.VppbImg(buf.img.base + size - a.nbytes, None, 1, a.nbytes, size, 0, 1, 256)
        capi.check(capi.lib.vppb_upload(C.byref(v), a.ctypes.data, a.nbytes, 0, None))
        bufs.append(buf)
        return v.base

    kp = at_end(pts)
    pr = at_end(pred) if pred is not None else None
    d_flow, d_err = ops._DeviceBuffer(n * 8), ops._DeviceBuffer(n * 4)
    capi.check(capi.lib.vppb_lk_match_u8(prev.desc_array(), nxt.desc_array(), grad.desc_array(), C.byref(params), kp, pr, n, d_flow.ptr, d_err.ptr, None))
    return d_flow.to_host(np.float32, n * 2).reshape(-1, 2), d_err.to_host(np.float32, n)


def _huge_level0(levels, h, capi):
    """replace level 0 of `levels` by a hand-built descriptor over one device allocation with a 64 MiB pitch holding h's bytes
    (border included); returns the allocation"""
    import torch

    pitch, b = 64 << 20, h.border
    rows = h.nrows + 2 * b
    buf = torch.zeros(rows * pitch, dtype=torch.uint8, device="cuda")
    frame = h.get(True)
    for j in range(rows):
        buf[j * pitch:j * pitch + frame.shape[1]].copy_(torch.from_numpy(np.ascontiguousarray(frame[j])))
    torch.cuda.synchronize()
    d = capi.VppbImg(buf.data_ptr() + b * pitch + b, None, h.nrows, h.ncols, pitch, b, 1, 1)
    levels.descs[0] = d
    return buf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=("gpu", "emu"), required=True)
    ap.add_argument("--policy", choices=list(POLICIES), required=True)
    ap.add_argument("--big", action="store_true", help="add the LK case whose level 0 spans more than 2 GiB (default policy, GPU)")
    ap.add_argument("--no-tall", action="store_true", help="leave the 32800-row FAST frame out")
    args = ap.parse_args()
    vpp, sms = _load(args.backend)
    env = {k: os.environ[k] for k in KNOBS if k in os.environ}
    run = Runner(vpp, sms, env, args.backend)
    tables = POLICIES[args.policy]["tables"]
    results = []
    if "fast" in tables:
        for k in fast_cases(sms, tall=not args.no_tall):
            results.extend(run.run_fast(k))
    if "lk" in tables:
        for k in lk_cases(sms, big=args.big):
            results.extend(run.run_lk(k))
    print(json.dumps(dict(backend=args.backend, policy=args.policy, sms=sms, env=env, results=results)))


def run_child(backend, policy, big=False, tall=True, env=None, timeout=3000):
    """run the tables of POLICIES[policy] in a child process: (returncode, parsed JSON or None, stderr)"""
    e = {k: v for k, v in (env if env is not None else os.environ).items() if k not in KNOBS}
    e.update(POLICIES[policy]["env"])
    cmd = [sys.executable, "-m", "tests.detector_paths", "--backend", backend, "--policy", policy] + (["--big"] if big else []) + ([] if tall else ["--no-tall"])
    r = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=timeout)
    try:
        res = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    except (ValueError, IndexError):
        res = None
    return r.returncode, res, r.stderr


def failures(res):
    return [r for r in res["results"] if not r["ok"]]


def unmet(res, policy, big=False):
    """what the policy's tables are written to reach and, by the transcribed dispatch, no longer reach"""
    return sorted(expected(policy, big) - reached(res))


if __name__ == "__main__":
    main()
