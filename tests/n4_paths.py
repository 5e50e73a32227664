"""Child process of the N4 dispatch-path tests (tests/test_gpu_n4_paths.py, tests/test_emulated_n4_paths.py).

Three kernels of SURVEY 8(f) N4 hide several paths behind one entry point:
  * vppb_lbp_u8 runs k_lbp_u8<true> when input and output rows are 16-byte aligned (pixel (0,0) and pitch), else k_lbp_u8<false>;
    inside <true> a thread whose 16-pixel group crosses the right edge takes the scalar path, and the last group of LBP_ROWS = 4 rows
    is clipped at nrows;
  * vppb_local_maxima_filter is one cooperative launch of k_local_maxima_filter<unsigned char | int> whose grid is capped at what is
    resident at once: a frame of more items (runs of 16 pixels of a row) than threads walks them in grid-stride loops, pass after
    pass, with a grid-wide barrier and a ring of three pass counters between the passes;
  * vppb_lk_match_oriented_u8 runs k_lk_match_oriented<PPL, GF>, PPL = ceil(winsize^2 / 32) rounded up to 6 / 8, GF the gradient type.
There are no knobs, so one process runs everything:

    python -m tests.n4_paths --backend gpu|emu [--big] [--no-8k]

runs the lbp, local_maxima_filter, oriented LK and workspace tables and prints one JSON object: the SM count the library sees and, per
case, pass / fail with the first mismatch and what the dispatch takes for it (`plan`, a transcription of stencils.cu's and lk.cu's
launch rules).

lbp and local_maxima_filter results must equal the C oracle's (vo_lbp_u8, vo_local_maxima_filter) exactly, over the whole allocation:
the input allocation is uploaded from the host, border and pitch padding included, so the oracle reads the bytes the kernel reads (a
view's neighbours are its parent's pixels), and everything outside an output's domain must keep its sentinel.  local_maxima_filter
gets a workspace larger than vppb_local_maxima_filter_workspace_bytes: the bytes past that size must keep theirs.  Oriented LK flows
and errors must equal vo_lk_match_oriented_u8 bit for bit, failure codes included; as in tests/detector_paths.py every NaN error
compares equal to every other NaN (the H100 and x86 write different payloads for 0 / 0) and to nothing else.

The workspace table calls every entry point that takes a caller workspace with one that breaks its documented alignment (base + 4,
and base + 128 where 256 bytes are required; the distance transform and the brute-force matcher require 8): the call must return VPPB_E_ARG and leave the
workspace and every output untouched, and the same call on an aligned workspace must succeed.  No call of the table ever reaches a
kernel with a misaligned workspace, whatever library it runs against: a probe one byte short of the workspace size, which every
version of the entry points rejects before launching, has to be refused for its alignment first."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import zlib

import numpy as np

from tests.box_geometry import Alloc, _load
from tests.detector_paths import first_diff, lk_bits, lk_outcome, v1_ppl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xA7
WS_SENTINEL = 0x5C

# ------------------------------------------------------------------ the dispatch of stencils.cu and lk.cu, transcribed
LBP_ROWS = 4
LMF_RUN = 16
LMF_THREADS = 256  # threads per CTA of k_local_maxima_filter
MAX_THREADS_PER_SM = 2048  # an H100 SM holds at most 2048 threads: 8 CTAs of 256, 16 of 128
LK_OR_KPS_PER_CTA = 4  # k_lk_match_oriented: 128 threads, one warp per keypoint
ORIENTED_PPLS = (1, 2, 3, 4, 6, 8)


def lbp_plan(i, o):
    """vppb_lbp_u8: the instantiation and what runs inside it"""
    vec = i.base % 16 == 0 and i.pitch % 16 == 0 and o.base % 16 == 0 and o.pitch % 16 == 0
    return dict(kernel="true" if vec else "false", vector_groups=bool(vec and i.ncols >= 16), ragged=bool(vec and i.ncols % 16 != 0),
                rows_mod4=i.nrows % LBP_ROWS)


def lmf_plan(nrows, ncols, elem, sms):
    """vppb_local_maxima_filter: the work items, and the regime bounds that hold whatever the occupancy: a grid of one CTA per SM is
    always resident (so items <= 256 * SMs run in one trip), and no SM holds more than 8 CTAs of 256 threads (so items beyond
    8 * 256 * SMs always loop)"""
    items = nrows * ((ncols + LMF_RUN - 1) // LMF_RUN)
    if items <= LMF_THREADS * sms:
        regime = "single-trip"
    elif items > (MAX_THREADS_PER_SM // LMF_THREADS) * LMF_THREADS * sms:
        regime = "grid-stride"
    else:
        regime = "either"
    return dict(pix="u8" if elem == 1 else "int", items=items, regime=regime)


def oriented_plan(ws, gf, n, sms):
    ctas = (n + LK_OR_KPS_PER_CTA - 1) // LK_OR_KPS_PER_CTA
    return dict(ppl=v1_ppl(ws), grad="float" if gf else "int", ctas=ctas, beyond_wave=ctas > (MAX_THREADS_PER_SM // 128) * sms)


WS_ENTRIES = {  # entry point: the workspace alignment it documents
    "vppb_fast9_u8": 256, "vppb_fast9_u8_async": 256, "vppb_fast9_blockwise_rank_u8": 256, "vppb_local_maxima_filter": 256,
    "vppb_distance_transform": 8, "vppb_sdof_u8": 256, "vppb_match_bruteforce_sad": 8, "vppb_match_local_sad": 256,
    "vppb_sparse_flow_u8": 256,
}


def reached(res):
    out = set()
    for r in res["results"]:
        p = r["plan"]
        if r["table"] == "lbp":
            out.add("lbp <%s>" % p["kernel"])
            if p["kernel"] == "true":
                if p["vector_groups"]:
                    out.add("lbp <true> vector group")
                if p["ragged"]:
                    out.add("lbp <true> ragged scalar group")
                out.add("lbp <true> nrows %% 4 == %d" % p["rows_mod4"])
        elif r["table"] == "lmf":
            out.add("lmf %s %s" % (p["pix"], p["regime"]))
        elif r["table"] == "oriented":
            out.add("oriented ppl=%d %s" % (p["ppl"], p["grad"]))
            if p["beyond_wave"]:
                out.add("oriented more CTAs than one wave")
            out.update("oriented outcome " + o for o in r["outcomes"])
        elif r["table"] == "ws":
            out.add("ws %s offset %d" % (r["case"], p["offset"]))
    return out


def expected():
    want = {"lbp <true>", "lbp <false>", "lbp <true> vector group", "lbp <true> ragged scalar group"}
    want |= {"lbp <true> nrows %% 4 == %d" % k for k in range(4)}
    want |= {"lmf %s %s" % (p, r) for p in ("u8", "int") for r in ("single-trip", "grid-stride")}
    want |= {"oriented ppl=%d %s" % (p, g) for p in ORIENTED_PPLS for g in ("int", "float")}
    want |= {"oriented more CTAs than one wave"} | {"oriented outcome " + o for o in ("converged", "rejected", "left the domain")}
    want |= {"ws %s offset %d" % (e, off) for e, a in WS_ENTRIES.items() for off in ((4, 128) if a == 256 else (4,))}
    return want


def unmet(res):
    return sorted(expected() - reached(res))


def failures(res):
    return [r for r in res["results"] if not r["ok"]]


# ------------------------------------------------------------------ case tables
ALIGNS = (1, 4, 16, 128)
VEC_PAIRS = ((16, 128), (128, 16), (128, 128), (16, 16))
SCALAR_PAIRS = tuple((a, b) for a in ALIGNS for b in ALIGNS if not (a >= 16 and b >= 16))


def _lbp(name, nrows, ncols, ia=128, oa=128, ib=1, ob=0, border="mirror", view=None, oview=None, content="levels"):
    """view / oview: (row, col) of the input / output as a view of a larger parent; border: how the input's border is filled
    ("mirror", "value", or the parent's pixels for a view); content: "levels" (six grey levels: ties and strict orders), "noise",
    "tile" (a random block repeated: affordable at any size)"""
    return dict(table="lbp", name=name, nrows=nrows, ncols=ncols, ia=ia, oa=oa, ib=ib, ob=ob, border=border, view=view, oview=oview, content=content)


def lbp_cases(big8k=True, big=False):
    T = []
    i = 0
    for nc in (1, 15, 16, 17, 31, 32, 33, 1000):
        for nr in (1, 2, 3, 4, 5, 8, 9, 131):
            for ia, oa in (VEC_PAIRS[i % 4], SCALAR_PAIRS[i % len(SCALAR_PAIRS)]):
                T.append(_lbp("lbp_%dx%d_a%d_%d" % (nr, nc, ia, oa), nr, nc, ia, oa, ib=1 + i % 2, ob=(0, 1, 3)[i % 3], border=("mirror", "value")[(i // 2) % 2]))
            i += 1
    for view, oview in (((1, 1), (0, 3)), ((2, 5), None), (None, (1, 7)), ((3, 17), (2, 1))):
        for nr, nc in ((9, 33), (6, 16), (131, 1000)):
            T.append(_lbp("lbp_view_%s_%s_%dx%d" % (view, oview, nr, nc), nr, nc, view=view, oview=oview))
    T.append(_lbp("lbp_4k", 2160, 3840, content="tile"))
    T.append(_lbp("lbp_4k_out_a4", 2160, 3840, oa=4, border="value", content="tile"))
    if big8k:
        T.append(_lbp("lbp_8k", 4320, 7680, content="tile"))
    if big:
        T.append(_lbp("lbp_big_40000x56000", 40000, 56000, content="tile"))
    return T


def _lmf(name, pix, nrows, ncols, content, align=128, border_value=0, view=None, seed=0):
    return dict(table="lmf", name=name, pix=pix, nrows=nrows, ncols=ncols, content=content, align=align, border_value=border_value, view=view, seed=seed)


CHAIN = 1100  # links of an int chain; a u8 chain has one link per grey level at most (255 .. 1)


def lmf_cases(sms, big8k=True, big=False):
    T = []
    for pix in ("u8", "int"):
        for shape in ((9, 14), (40, 67), (64, 96)):
            for s in range(6):
                T.append(_lmf("lmf_%s_scene%d_%dx%d" % (pix, s, shape[0], shape[1]), pix, shape[0], shape[1], "scene%d" % s, seed=s))
        for d in ("N", "NW", "NE", "W"):
            T.append(_lmf("lmf_%s_chain_%s" % (pix, d), pix, 0, 0, "chain_" + d))
        # widths around the 16-pixel runs, single rows and columns
        for nr, nc in ((23, 1), (23, 15), (23, 16), (23, 17), (11, 32), (11, 33), (11, 47), (1, 1), (1, 40), (1, 513), (70, 1), (300, 2)):
            T.append(_lmf("lmf_%s_%dx%d" % (pix, nr, nc), pix, nr, nc, "noise" if nc % 2 else "scene1", align=(128, 4, 16, 1)[nc % 4]))
        # views at odd columns: the parent's pixels are the view's neighbours
        for vr, vc, nr, nc in ((1, 1, 17, 33), (2, 5, 9, 16), (0, 3, 30, 17)):
            T.append(_lmf("lmf_%s_view_%d_%d" % (pix, vr, vc), pix, nr, nc, "noise", view=(vr, vc)))
    # int: negative values, non-zero border values
    for bv in (-5, 7, -2147483648):
        T.append(_lmf("lmf_int_negative_border%d" % bv, "int", 37, 45, "negative", border_value=bv))
    # the regimes: one trip (items <= 256 * SMs) and grid-stride loops (items > 8 * 256 * SMs), both pixel types
    small = max(1, LMF_THREADS * sms // 4)  # rows of 64 pixels = 4 items
    T.append(_lmf("lmf_u8_single_trip", "u8", small, 64, "scene2"))
    T.append(_lmf("lmf_int_single_trip", "int", small, 64, "scene1"))
    loops = 8 * LMF_THREADS * sms // 16 + 7  # rows of 256 pixels = 16 items
    T.append(_lmf("lmf_u8_grid_stride_%d" % loops, "u8", loops, 256, "chains_mixed"))
    T.append(_lmf("lmf_int_grid_stride_%d" % loops, "int", loops, 256, "chains_mixed"))
    T.append(_lmf("lmf_u8_4k", "u8", 2160, 3840, "tile"))
    T.append(_lmf("lmf_int_4k", "int", 2160, 3840, "tile"))
    if big8k:
        T.append(_lmf("lmf_u8_8k", "u8", 4320, 7680, "tile"))
        T.append(_lmf("lmf_int_8k", "int", 4320, 7680, "tile"))
    if big:
        T.append(_lmf("lmf_big_40000x56000", "u8", 40000, 56000, "tile"))
    return T


def _ocase(name, ws, gf, n, max_iter=21, max_step=1.0, aa=128, ba=128, view_a=None, view_b=None, border=3, shape=(61, 83)):
    return dict(table="oriented", name=name, ws=ws, gf=gf, n=n, max_iter=max_iter, max_step=max_step, aa=aa, ba=ba, view_a=view_a, view_b=view_b,
                border=border, shape=shape)


def oriented_cases(sms):
    T = []
    i = 0
    wave = 4 * (MAX_THREADS_PER_SM // 128) * sms
    counts = (1, 3, 4, 5, 37, wave + 4 * 3 + 1)
    for ws in range(1, 16, 2):
        for gf in (0, 1):
            T.append(_ocase("oriented_ws%d_%s" % (ws, ("int", "float")[gf]), ws, gf, counts[i % len(counts)], max_iter=(21, 1, 0)[i % 3],
                            max_step=(1.0, 1e-3, 1e6)[(i // 3) % 3], border=(1, 3, 8)[i % 3]))
            i += 1
    # more CTAs than one wave, at a small and a large window
    T.append(_ocase("oriented_wave_ws5", 5, 1, wave + 4 * 7 + 1))
    T.append(_ocase("oriented_wave_ws13", 13, 0, wave + 4 * 5 + 1, max_step=0.5))
    # A and B at alignments 1 / 16 / 128 and as views at odd columns (their clamped taps read the parent's pixels)
    for aa, ba in ((1, 16), (16, 1), (128, 1), (1, 128)):
        T.append(_ocase("oriented_align_%d_%d" % (aa, ba), 7 + 2 * (aa == 1), aa % 2, 41, aa=aa, ba=ba, border=2))
    T.append(_ocase("oriented_views", 9, 1, 45, view_a=(2, 3), view_b=(1, 5), border=1))
    T.append(_ocase("oriented_view_b", 15, 0, 23, view_b=(3, 1), border=4, max_iter=1))
    return T


# ------------------------------------------------------------------ scenes
def _tile_block(nr, nc, pix, seed):
    """a frame that repeats a random 997 x 1009 block (primes: no alignment with the 16-pixel runs or rows), cheap at any size"""
    rng = np.random.default_rng(seed)
    if pix == "u8":
        blk = rng.integers(0, 256, (997, 1009)).astype(np.uint8)
    else:
        blk = rng.integers(-1000, 100000, (997, 1009)).astype(np.int32)
    return np.tile(blk, ((nr + 996) // 997, (nc + 1008) // 1009))[:nr, :nc]


def chain_scene(direction, pix):
    """a one-pixel-wide chain of strictly decreasing values on a lower background, each link a successor (S, SE / SW, E) of the one
    before: every chain pixel is a maximum iff its predecessor is not, so the decisions alternate along the whole chain.  NW / NE
    chains zig-zag (runs of 40 diagonal steps) to stay in a narrow frame; u8 chains are capped at 254 links"""
    L = CHAIN if pix == "int" else 254
    if direction == "W":
        pts = [(1, 2 + k) for k in range(L)]
        shape = (3, L + 5)
    elif direction == "N":
        pts = [(k, 6) for k in range(L)]
        shape = (L + 2, 13)
    else:
        sgn = 1 if direction == "NW" else -1  # NW: the chain steps SE first
        c0 = 2 if sgn > 0 else 43
        pts, c = [], c0
        for k in range(L):
            pts.append((k, c))
            c += sgn if (k // 40) % 2 == 0 else -sgn
        shape = (L + 2, 46)
    if pix == "u8":
        bg, vals = 0, [255 - k for k in range(L)]
    else:
        bg, vals = -3, [5 * L + 40 - 5 * k for k in range(L)]
    a = np.full(shape, bg, np.int64)
    for (r, c), v in zip(pts, vals):
        a[r, c] = v
    return a


def lmf_content(k):
    from tests.test_n4_oracle import lmf_scenes

    pix, nr, nc, c = k["pix"], k["nrows"], k["ncols"], k["content"]
    rng = np.random.default_rng(zlib.crc32(k["name"].encode()))
    dt = np.uint8 if pix == "u8" else np.int32
    if c.startswith("scene"):
        return lmf_scenes((nr, nc), "u8" if pix == "u8" else "i32", k["seed"])[int(c[5:])]
    if c.startswith("chain_"):
        return chain_scene(c[6:], pix).astype(dt)
    if c == "noise":
        return rng.integers(0, 256 if pix == "u8" else 1000, (nr, nc)).astype(dt)
    if c == "negative":
        return rng.integers(-50, 50, (nr, nc)).astype(dt)
    if c == "tile":
        return _tile_block(nr, nc, pix, 5).astype(dt)
    if c == "chains_mixed":  # noise with vertical decreasing chains (as long as the grey levels allow) every 37 columns
        a = rng.integers(0, 60, (nr, nc)).astype(np.int64)
        L = min(nr, 190 if pix == "u8" else nr)
        for col in range(5, nc, 37):
            a[:L, col] = (250 if pix == "u8" else 5 * L + 100) - np.arange(L) * (1 if pix == "u8" else 5)
        return a.astype(dt)
    raise ValueError(c)


def lbp_content(k, shape, rng):
    if k["content"] == "tile":
        return _tile_block(shape[0], shape[1], "u8", 3)
    if k["content"] == "noise":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    return (rng.integers(0, 6, shape) * 51).astype(np.uint8)


# ------------------------------------------------------------------ comparisons
def alloc_mismatch(got, want, r0, c0, nrows, rowbytes):
    """None, or the first byte where two whole allocations differ, in (row, byte) of the image and whether it is in the domain"""
    for y0 in range(0, got.shape[0], 4096):
        g, w = got[y0:y0 + 4096], want[y0:y0 + 4096]
        if np.array_equal(g, w):
            continue
        bad = np.flatnonzero(g != w)
        br, bc = divmod(int(bad[0]), got.shape[1])
        br += y0
        y, x = br - r0, bc - c0
        return dict(row=y, byte=x, inside=bool(0 <= y < nrows and 0 <= x < rowbytes), got=int(got[br, bc]), want=int(want[br, bc]),
                    count_in_block=int(len(bad)))
    return None


class Runner:
    def __init__(self, vpp, sms, backend):
        from tests import oracle as orc
        from vpp_b200 import capi, ops

        self.vpp, self.sms, self.backend = vpp, sms, backend
        self.capi, self.ops, self.orc = capi, ops, orc

    def _sync(self):
        self.capi.check(self.capi.lib.vppb_sync(None))

    # ---- lbp
    def _lbp_input(self, k, rng):
        vpp, nr, nc = self.vpp, k["nrows"], k["ncols"]
        if k["view"] is None:
            a = Alloc(vpp, nr, nc, "u8", k["ib"], k["ia"])
            img = a.img
        else:
            vr, vc = k["view"]
            a = Alloc(vpp, nr + vr + 2, nc + vc + 3, "u8", k["ib"], k["ia"])
            img = a.img.subimage(vpp.Box2d((vr, vc), (vr + nr - 1, vc + nc - 1)))
        host = lbp_content(k, a.shape, rng)
        a.put(host)
        if k["view"] is None:
            if k["border"] == "mirror" and img.desc.border <= min(nr, nc):  # (a mirror needs as many pixels as the border is wide)
                vpp.fill_border_mirror(img)
            else:
                vpp.fill_border_with_value(img, int(rng.integers(0, 256)))
            self._sync()
            host = a.get()
        return a, img, host

    def _output(self, nr, nc, pix, border, align, oview):
        vpp = self.vpp
        if oview is None:
            a = Alloc(vpp, nr, nc, pix, border, align)
            img = a.img
        else:
            vr, vc = oview
            a = Alloc(vpp, nr + vr + 2, nc + vc + 2, pix, border, align)
            img = a.img.subimage(vpp.Box2d((vr, vc), (vr + nr - 1, vc + nc - 1)))
        a.put(np.full(a.shape, SENTINEL, np.uint8))
        return a, img

    def run_lbp(self, k):
        capi, orc = self.capi, self.orc
        nr, nc = k["nrows"], k["ncols"]
        rng = np.random.default_rng(zlib.crc32(k["name"].encode()))
        ia, iimg, ihost = self._lbp_input(k, rng)
        oa, oimg = self._output(nr, nc, "u8", k["ob"], k["oa"], k["oview"])
        plan = lbp_plan(iimg.desc, oimg.desc)
        capi.check(capi.lib.vppb_lbp_u8(C.byref(iimg.desc), C.byref(oimg.desc), None))
        self._sync()
        got = oa.get()
        want = np.full(oa.shape, SENTINEL, np.uint8)
        r0, c0 = oa.at(oimg.desc)
        ir0, ic0 = ia.at(iimg.desc)
        o = orc.load(omp=nr * nc > 1 << 20)
        src = orc.VoImg(ihost.ctypes.data + ir0 * ia.pitch + ic0, nr, nc, ia.pitch, 1, 1)
        dst = orc.VoImg(want.ctypes.data + r0 * oa.pitch + c0, nr, nc, oa.pitch, 0, 1)
        o.vo_lbp_u8(C.byref(src), C.byref(dst))
        bad = alloc_mismatch(got, want, r0, c0, nr, nc)
        if bad is None:  # the input is read only
            bad = alloc_mismatch(ia.get(), ihost, ir0, ic0, nr, nc)
            if bad is not None:
                bad["what"] = "input changed"
        return [dict(table="lbp", case=k["name"], ok=bad is None, mismatch=bad, plan=plan)]

    # ---- local_maxima_filter
    def run_lmf(self, k):
        capi, orc, ops, vpp = self.capi, self.orc, self.ops, self.vpp
        frame = lmf_content(k)
        nr, nc = frame.shape
        pix = "u8" if k["pix"] == "u8" else "i32"
        elem = 1 if pix == "u8" else 4
        rng = np.random.default_rng(zlib.crc32(k["name"].encode()) + 1)
        if k["view"] is None:
            a = Alloc(vpp, nr, nc, pix, 1, k["align"])
            img = a.img
        else:
            vr, vc = k["view"]
            a = Alloc(vpp, nr + vr + 2, nc + vc + 3, pix, 1, k["align"])
            img = a.img.subimage(vpp.Box2d((vr, vc), (vr + nr - 1, vc + nc - 1)))
        r0, c0 = a.at(img.desc)
        if a.shape[0] * a.shape[1] > 1 << 28:
            host = np.full(a.shape, SENTINEL, np.uint8)
        else:
            host = rng.integers(0, 256, a.shape, dtype=np.uint8)  # pitch padding, and a view's parent
        dom = host[r0:r0 + nr, c0:c0 + nc * elem]
        dom[...] = np.ascontiguousarray(frame).view(np.uint8).reshape(nr, nc * elem)
        del frame, dom
        a.put(host)
        if k["view"] is None:
            vpp.fill_border_with_value(img, k["border_value"])
            self._sync()
            host = a.get()
        need = capi.lib.vppb_local_maxima_filter_workspace_bytes(nr, nc, elem)
        size = need + 4096
        if size < 1 << 31:
            ws = ops._DeviceBuffer(size).from_host(np.full(size, WS_SENTINEL, np.uint8))
            ws_ptr, tail = ws.ptr, lambda: ws.to_host(np.uint8, size)[need:]
        else:  # vppb_alloc takes an int32 width: a workspace of 2 GiB or more comes from torch (512-byte aligned)
            import torch

            ws = torch.full((size,), WS_SENTINEL, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            ws_ptr, tail = ws.data_ptr(), lambda: ws[need:].cpu().numpy()
        plan = lmf_plan(nr, nc, elem, self.sms)
        capi.check(capi.lib.vppb_local_maxima_filter(C.byref(img.desc), ws_ptr, size, None))
        self._sync()
        got = a.get()
        o = orc.load()
        orc_img = orc.VoImg(host.ctypes.data + r0 * a.pitch + c0, nr, nc, a.pitch, 1, elem)
        o.vo_local_maxima_filter(C.byref(orc_img))  # in place, on the bytes the kernel read
        bad = alloc_mismatch(got, host, r0, c0, nr, nc * elem)
        if bad is None:
            tail = tail()
            if (tail != WS_SENTINEL).any():
                bad = dict(what="workspace past vppb_local_maxima_filter_workspace_bytes written", offset=int(need + np.flatnonzero(tail != WS_SENTINEL)[0]))
        return [dict(table="lmf", case=k["name"], ok=bad is None, mismatch=bad, plan=plan, shape=[nr, nc])]

    # ---- oriented LK
    def _oriented_scene(self, shape):
        from tests import scenes

        nr, nc = shape
        f1, f2, _ = scenes.lk_pair(nr, nc, 4, seed=11, shift=(1.3, -0.8), margin=8)
        fr, fc = (nr * 5 // 8, nr * 5 // 8 + 18), (nc * 7 // 10, nc * 7 // 10 + 20)  # a flat patch: G = 0
        f1[fr[0]:fr[1], fc[0]:fc[1]] = 140
        f2[fr[0]:fr[1], fc[0]:fc[1]] = 140
        return f1, f2, (fr, fc)

    def _u8_frame(self, frame, border, align, view, rng):
        """a device u8 image holding `frame`: the library layout at `align` with a mirror border, or a view of a random parent"""
        vpp = self.vpp
        nr, nc = frame.shape
        if view is None:
            a = Alloc(vpp, nr, nc, "u8", border, align)
            img = a.img
        else:
            vr, vc = view
            a = Alloc(vpp, nr + vr + 2, nc + vc + 3, "u8", border, align)
            img = a.img.subimage(vpp.Box2d((vr, vc), (vr + nr - 1, vc + nc - 1)))
        host = rng.integers(0, 256, a.shape, dtype=np.uint8)
        r0, c0 = a.at(img.desc)
        host[r0:r0 + nr, c0:c0 + nc] = frame
        a.put(host)
        if view is None:
            vpp.fill_border_mirror(img)
            self._sync()
            host = a.get()
        vo = self.orc.VoImg(host.ctypes.data + r0 * a.pitch + c0, nr, nc, a.pitch, img.desc.border, 1)
        return a, img, host, vo

    def run_oriented(self, k):
        from tests.detector_paths import _upload, lk_points
        from tests.oracle_ops import oracle_grad_pyramid

        orc, ops = self.orc, self.ops
        ws, gf, n = k["ws"], k["gf"], k["n"]
        gpix = "vfloat2" if gf else "vint2"
        rng = np.random.default_rng(zlib.crc32(k["name"].encode()))
        f1, f2, flat = self._oriented_scene(k["shape"])
        nr, nc = k["shape"]
        b = k["border"]
        A = self._u8_frame(f1, b, k["aa"], k["view_a"], rng)
        B = self._u8_frame(f2, b, k["ba"], k["view_b"], rng)
        o = orc.load(omp=n > 2000)
        Ah = orc.HostImage(nr, nc, "u8", border=max(1, b), data=f1, fill_border="mirror")
        Gh = oracle_grad_pyramid([Ah], gpix, b, o)[0]
        G = _upload(self.vpp, Gh)
        pts = lk_points(n, nr, nc, flat, rng, off=int(rng.integers(5)))
        ang1, ang2 = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
        ang2[::2] = ang1[::2]  # half of the points search along the template's own direction
        d1 = np.stack([np.cos(ang1), np.sin(ang1)], axis=1).astype(np.float32)
        d2 = np.stack([np.cos(ang2), np.sin(ang2)], axis=1).astype(np.float32)
        d1[::5], d2[::5] = (0.0, 1.0), (0.0, 1.0)  # the axis-aligned window
        d1[3::10], d2[3::10] = (1.0, 0.0), (-1.0, 0.0)  # quarter and half turns
        pred = rng.uniform(-1.5, 1.5, (n, 2)).astype(np.float32)
        pred[3::7] = (4000.0, -2500.0)  # the first step leaves the 3-pixel margin (or, without steps, the error is taken out there)
        pred[6::13] = (0.0, -float(nc))
        min_ev, delta = 1e-3, 0.01
        plan = oriented_plan(ws, gf, n, self.sms)
        flow, err = ops.oriented_lk_match(A[1], B[1], G, pts, pred, d1, d2, ws, min_ev, k["max_iter"], delta, k["max_step"])
        rf, re = np.zeros((n, 2), np.float32), np.zeros(n, np.float32)
        o.vo_lk_match_oriented_u8(C.byref(A[3]), C.byref(B[3]), Gh.ptr(), gf, ws, min_ev, k["max_iter"], delta, k["max_step"], pts.ctypes.data,
                                  pred.ctypes.data, d1.ctypes.data, d2.ctypes.data, n, rf.ctypes.data, re.ctypes.data)
        bad = first_diff(lk_bits(flow, err), lk_bits(rf, re))
        if bad is not None:
            i = bad["index"]
            bad.update(keypoint=pts[i].tolist(), dir1=d1[i].tolist(), dir2=d2[i].tolist(), pred=pred[i].tolist(),
                       got_float=[float(flow[i, 0]), float(flow[i, 1]), float(err[i])], want_float=[float(rf[i, 0]), float(rf[i, 1]), float(re[i])])
        outcomes = sorted({lk_outcome(rf[i], re[i]) for i in range(n)})
        return [dict(table="oriented", case=k["name"], ok=bad is None, mismatch=bad, plan=plan, n=n, outcomes=outcomes)]

    # ---- workspace alignment
    def run_workspaces(self):
        out = []
        for entry, align in WS_ENTRIES.items():
            for off in (4, 128) if align == 256 else (4,):
                out.append(self._ws_case(entry, align, off))
        return out

    def _ws_case(self, entry, align, off):
        capi, ops, vpp = self.capi, self.ops, self.vpp
        lib = capi.lib
        rng = np.random.default_rng(zlib.crc32(entry.encode()) + off)
        keep, outs = [], []  # outs: device buffers / images that must keep their bytes; host ints likewise

        def dbuf(nbytes):
            b = ops._DeviceBuffer(nbytes).from_host(np.full(nbytes, SENTINEL, np.uint8))
            outs.append(b)
            return b.ptr

        def image(nr, nc, pix, border=3, content=True):
            im = vpp.Image2d(nr, nc, pix, border=border)
            if content:
                im.upload(rng.integers(0, 256, (nr, nc)).astype(np.uint8 if pix == "u8" else np.int32))
                vpp.fill_border_mirror(im)
            keep.append(im)
            return im

        cnt = C.c_int32(-7)
        if entry in ("vppb_fast9_u8", "vppb_fast9_u8_async", "vppb_fast9_blockwise_rank_u8"):
            img = image(24, 40, "u8")
            if entry == "vppb_fast9_blockwise_rank_u8":
                need = lib.vppb_fast9_rank_workspace_bytes(24, 40, 5, 3)
                call = lambda w, nb: lib.vppb_fast9_blockwise_rank_u8(img.ptr(), 20, None, 5, 3, 0, w, nb, kp, sc, 256, C.byref(cnt), None)
                kp, sc = dbuf(256 * 12), dbuf(256 * 4)
            else:
                need = lib.vppb_fast9_workspace_bytes(24, 40, 10)
                kp, sc = dbuf(64 * 8), dbuf(64 * 4)
                if entry == "vppb_fast9_u8":
                    call = lambda w, nb: lib.vppb_fast9_u8(img.ptr(), 20, None, 2, 10, 0, w, nb, kp, sc, 64, C.byref(cnt), None)
                else:
                    cd = dbuf(4)
                    call = lambda w, nb: lib.vppb_fast9_u8_async(img.ptr(), 20, None, 2, 10, 0, w, nb, kp, sc, 64, cd, None)
        elif entry == "vppb_local_maxima_filter":
            img = image(20, 37, "u8", border=1)
            need = lib.vppb_local_maxima_filter_workspace_bytes(20, 37, 1)
            call = lambda w, nb: lib.vppb_local_maxima_filter(img.ptr(), w, nb, None)
            outs.append(img)
        elif entry == "vppb_distance_transform":
            a = image(20, 37, "u8", border=0, content=False)
            a.upload(np.where(rng.random((20, 37)) < 0.1, 0, 1).astype(np.uint8))
            s = image(20, 37, "i32", border=2, content=False)
            outs.append(s)
            need = lib.vppb_distance_transform_workspace_bytes(20, 37, 3)
            call = lambda w, nb: lib.vppb_distance_transform(a.ptr(), s.ptr(), 3, w, nb, None)
        elif entry == "vppb_sdof_u8":
            i1, i2 = image(40, 56, "u8"), image(40, 56, "u8")
            P = capi.VppbSdofParams(5, 2, 0, 2, 5)
            p1 = ops.Pyramid2d((40, 56), 2, 2, pixel="u8", border=10)
            p2 = ops.Pyramid2d((40, 56), 2, 2, pixel="u8", border=10)
            capi.check(lib.vppb_pyrlk_prepare(i1.ptr(), i2.ptr(), p1.desc_array(), p2.desc_array(), None, 2, 0, None))
            keep += [p1, p2]
            kps = np.array([[5, 5], [10, 20], [30, 50], [39, 0], [20, 30]], np.int32)
            dk = ops._DeviceBuffer(kps.nbytes).from_host(kps)
            keep.append(dk)
            need = lib.vppb_sdof_workspace_bytes(40, 56, C.byref(P))
            pos, dist, valid = dbuf(5 * 8), dbuf(5 * 4), dbuf(5)
            call = lambda w, nb: lib.vppb_sdof_u8(p1.desc_array(), p2.desc_array(), C.byref(P), dk.ptr, 5, w, nb, pos, dist, valid, None)
        elif entry in ("vppb_match_bruteforce_sad", "vppb_match_local_sad"):
            q, t = image(6, 9, "u8", border=0), image(8, 9, "u8", border=0)
            idx, dist = dbuf(6 * 4), dbuf(6 * 4)
            if entry == "vppb_match_bruteforce_sad":
                need = lib.vppb_match_bruteforce_sad_workspace_bytes(6, 8, 9)
                call = lambda w, nb: lib.vppb_match_bruteforce_sad(q.ptr(), t.ptr(), w, nb, idx, dist, None)
            else:
                qp = ops._DeviceBuffer(6 * 8).from_host(rng.integers(0, 30, (6, 2)).astype(np.int32))
                tp = ops._DeviceBuffer(8 * 8).from_host(rng.integers(0, 30, (8, 2)).astype(np.int32))
                keep += [qp, tp]
                need = lib.vppb_match_local_sad_workspace_bytes(6, 8, 9, 5, 4)
                call = lambda w, nb: lib.vppb_match_local_sad(q.ptr(), t.ptr(), qp.ptr, tp.ptr, 5, 4, w, nb, idx, dist, None)
        else:  # vppb_sparse_flow_u8
            i1, i2 = image(32, 48, "u8", border=5), image(32, 48, "u8", border=5)
            P = capi.VppbSofParams(5, 5, 5, 100, 300, 0, 5, 3)
            need = lib.vppb_sparse_flow_workspace_bytes(32, 48, C.byref(P), -1)
            cap = 7 * 10
            pos, flow, dist, valid = dbuf(cap * 8), dbuf(cap * 8), dbuf(cap * 4), dbuf(cap)
            call = lambda w, nb: lib.vppb_sparse_flow_u8(i1.ptr(), i2.ptr(), C.byref(P), None, 0, w, nb, pos, flow, dist, valid, cap, C.byref(cnt), None)
        self._sync()
        snap = [self._bytes(o) for o in outs]
        size = need + 512
        ws = ops._DeviceBuffer(size).from_host(np.full(size, WS_SENTINEL, np.uint8))
        # A library that does not check the alignment would launch its kernels on the misaligned workspace: a misaligned-address
        # fault on a GPU.  So the alignment is first probed with a workspace one byte too small, which every library rejects before
        # it launches anything (the alignment check comes first, so its message must name the alignment); only a library that
        # passes the probe gets the full-size misaligned workspace.
        rc = call(ws.ptr + off, need - 1)
        msg = lib.vppb_last_error().decode("utf-8", "replace") if rc else ""
        bad = None
        if rc != capi.VPPB_E_ARG or "align" not in msg:
            bad = dict(what="probe: a misaligned workspace one byte too small is not rejected for its alignment", got=int(rc), message=msg)
        else:
            rc = call(ws.ptr + off, need)
            msg = lib.vppb_last_error().decode("utf-8", "replace") if rc else ""
        self._sync()
        if bad is not None:
            pass
        elif rc != capi.VPPB_E_ARG:
            bad = dict(what="return code", got=int(rc), want=capi.VPPB_E_ARG)
        elif "align" not in msg:
            bad = dict(what="message", got=msg)
        elif (ws.to_host(np.uint8, size) != WS_SENTINEL).any():
            bad = dict(what="workspace written")
        elif cnt.value != -7:
            bad = dict(what="count written", got=cnt.value)
        else:
            for i, (o, before) in enumerate(zip(outs, snap)):
                if not np.array_equal(self._bytes(o), before):
                    bad = dict(what="output %d written" % i)
                    break
        if bad is None:  # the same call on an aligned workspace is accepted
            rc = call(ws.ptr + (8 if align == 8 else 256), need)
            self._sync()
            if rc != capi.VPPB_OK:
                bad = dict(what="aligned control call", got=int(rc), error=lib.vppb_last_error().decode("utf-8", "replace"))
        return dict(table="ws", case=entry, ok=bad is None, mismatch=bad, plan=dict(offset=off, align=align), message=msg)

    def _bytes(self, o):
        if isinstance(o, self.ops._DeviceBuffer):
            return o.to_host(np.uint8, o.nbytes)
        return o.download(with_border=True).view(np.uint8).copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=("gpu", "emu"), required=True)
    ap.add_argument("--big", action="store_true", help="add a u8 frame of more than 2 GiB through lbp and local_maxima_filter (GPU)")
    ap.add_argument("--no-8k", action="store_true", help="leave the 8K frames out")
    ap.add_argument("--only", default="", help="comma-separated tables to run (lbp, lmf, oriented, ws); all by default")
    args = ap.parse_args()
    vpp, sms = _load(args.backend)
    run = Runner(vpp, sms, args.backend)
    only = set(filter(None, args.only.split(",")))
    results = []
    if not only or "ws" in only:
        results.extend(run.run_workspaces())
    if not only or "lbp" in only:
        for k in lbp_cases(big8k=not args.no_8k, big=args.big):
            results.extend(run.run_lbp(k))
    if not only or "lmf" in only:
        for k in lmf_cases(sms, big8k=not args.no_8k, big=args.big):
            results.extend(run.run_lmf(k))
    if not only or "oriented" in only:
        for k in oriented_cases(sms):
            results.extend(run.run_oriented(k))
    print(json.dumps(dict(backend=args.backend, sms=sms, results=results)))


def run_child(backend, big=False, no_8k=False, env=None, timeout=3000, only=""):
    """run the tables in a child process: (returncode, parsed JSON or None, stderr)"""
    cmd = [sys.executable, "-m", "tests.n4_paths", "--backend", backend] + (["--big"] if big else []) + (["--no-8k"] if no_8k else [])
    cmd += ["--only", only] if only else []
    r = subprocess.run(cmd, cwd=ROOT, env=env if env is not None else dict(os.environ), capture_output=True, text=True, timeout=timeout)
    try:
        res = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    except (ValueError, IndexError):
        res = None
    return r.returncode, res, r.stderr


if __name__ == "__main__":
    main()
