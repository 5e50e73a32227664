"""Child process of the pyramid dispatch tests (tests/test_gpu_pyramid_paths.py, tests/test_emulated_pyramid_paths.py).

vpp_b200/csrc/pyramid.cu and vppb_copy2d_mirror (pixelwise.cu) choose a kernel per call from the layout of its images:
  * Scharr: k_scharr_u8_v8<as_float> (8-byte aligned input rows with room right of the last 8-pixel group, 16-byte aligned output
    rows) or k_scharr_u8<as_float>; plain, or with the output's mirror border written by the same launch;
  * low-pass + subsample: k_lowpass_sub2_u8_fast (input align >= 32, 16-byte aligned input rows, 8-byte aligned output rows, a
    parent of at least 4 x 4; tail items for the mirrored last row / column of an even parent), k_lowpass_sub2<0> otherwise, and
    k_lowpass_sub2_px8<1|2> for vint2 / vfloat2 with aligned16 = 0 or 1;
  * vppb_copy2d_mirror: one k_copy_mirror launch, or a copy and a border fill when the rows are not 16-byte aligned;
  * vppb_pyrlk_prepare: ONE cooperative launch of PREP_* work items (phases separated by grid barriers, grid capped at what is
    resident at once) or three chains of the launches above on three streams.  The default takes the fused form exactly when there
    is no gradient pyramid and falls back to the streams when the layout or more than 8 levels do not fit it; VPPB_PREPARE=fused|streams
    forces one form (`fused` returns VPPB_E_ARG and says why when the call does not fit it).
The choice of form is read per call from the environment, so each policy runs in a process of its own:

    python -m tests.pyramid_paths --backend gpu|emu --policy NAME [--big]

runs the stand-alone table (vppb_scharr_u8[_mirror], vppb_lowpass_sub2[_mirror] kinds 0 / 1 / 2, vppb_copy2d_mirror) and the
vppb_pyrlk_prepare table and prints one JSON object: the SM count the library sees and, per case, pass / fail with the first mismatch
and the plan, a transcription of the dispatch.

Every output allocation is compared byte for byte, border and pitch padding included, with the oracle run on a host copy of the same
bytes (vo_scharr_u8, vo_lowpass_sub2, vo_copy + vo_fill_border_mirror; oracle_pyramid / oracle_grad_pyramid for whole pyramids) and
the sentinel it was filled with everywhere the call must not write; floats compare as their bit patterns.  A rejected call must
return the plan's code and leave every byte of its outputs (and inputs) as it was, once the device is idle."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import zlib

import numpy as np

from tests.box_geometry import Alloc, _load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

POLICIES = {"default": {}, "fused": {"VPPB_PREPARE": "fused"}, "streams": {"VPPB_PREPARE": "streams"}}
SENTINEL = 0xC3
OK, E_ARG, E_BORDER = 0, -2, -3
PREP_MAX_LEVELS = 8
CTAS_PER_SM_MAX = 8  # 2048 threads per H100 SM: at most 8 resident CTAs of 256


# ------------------------------------------------------------------ the dispatch of pyramid.cu and vppb_copy2d_mirror, transcribed
def copy_check(src, dst):
    if not (src.base and dst.base) or src.elem_bytes != dst.elem_bytes or src.elem_bytes > 64:
        return E_ARG
    if (src.nrows, src.ncols) != (dst.nrows, dst.ncols):
        return E_ARG
    if dst.border > dst.nrows or dst.border > dst.ncols:
        return E_BORDER
    return OK


def scharr_check(i, o, mirror):
    if not (i.base and o.base) or i.elem_bytes != 1 or o.elem_bytes != 8 or i.nrows < o.nrows or i.ncols < o.ncols:
        return E_ARG
    if i.border < 1:
        return E_BORDER
    if o.base % 8 or o.pitch % 8:
        return E_ARG
    if mirror and (o.border > o.nrows or o.border > o.ncols):
        return E_BORDER
    return OK


def lowpass_check(i, o, kind, mirror):
    e = 1 if kind == 0 else 8
    if not (i.base and o.base) or i.elem_bytes != e or o.elem_bytes != e:
        return E_ARG
    if i.border < 2:
        return E_BORDER
    if o.nrows > 1 + i.nrows // 2 or o.ncols > 1 + i.ncols // 2:
        return E_ARG
    if mirror and (o.border > o.nrows or o.border > o.ncols):
        return E_BORDER
    return OK


def border_items(nr, nc, mb):
    return 2 * mb * (nc + 2 * mb) + 2 * nr * mb


def scharr_plan(i, o, as_float, mirror):
    rc = scharr_check(i, o, mirror)
    if rc:
        return dict(op="scharr", rejected=rc)
    mb = o.border if mirror else 0
    groups = (o.ncols + 7) // 8
    fast = i.base % 8 == 0 and i.pitch % 8 == 0 and o.base % 16 == 0 and o.pitch % 16 == 0 and i.align >= 16 and groups * 8 + 4 <= i.pitch - i.align
    items = (o.nrows * groups if fast else o.nrows * o.ncols) + border_items(o.nrows, o.ncols, mb)
    return dict(op="scharr", kernel="%s<%d>" % ("k_scharr_u8_v8" if fast else "k_scharr_u8", 1 if as_float else 0), prep="PREP_SCHARR_V8" if fast else "PREP_SCHARR_PX",
                mirrored=mb > 0, items=items)


def lowpass_u8_fast_items(onr, onc, fast_rows, fast_cols, groups):
    n_row = onc if onr > fast_rows else 0
    n_col = onr - (1 if n_row else 0) if onc > fast_cols else 0
    return ((fast_rows + 1) // 2) * groups + n_row + n_col, n_row + n_col


def lowpass_plan(i, o, kind, mirror):
    rc = lowpass_check(i, o, kind, mirror)
    if rc:
        return dict(op="lowpass", rejected=rc)
    p = dict(op="lowpass", mirrored=mirror and o.border > 0)
    if kind == 0:
        fast = i.align >= 32 and i.base % 16 == 0 and i.pitch % 16 == 0 and o.base % 8 == 0 and o.pitch % 8 == 0 and i.nrows >= 4 and i.ncols >= 4
        if fast:
            fr, fc = min(o.nrows, (i.nrows + 1) // 2), min(o.ncols, (i.ncols + 1) // 2)
            items, tail = lowpass_u8_fast_items(o.nrows, o.ncols, fr, fc, (fc + 7) // 8)
            p.update(kernel="k_lowpass_sub2_u8_fast", prep="PREP_LP_U8_FAST", items=items, tail_items=tail)
        else:
            p.update(kernel="k_lowpass_sub2<0>", prep="PREP_LP_GENERIC", items=o.nrows * o.ncols)
    else:
        a16 = int(i.base % 16 == 0 and i.pitch % 16 == 0)
        p.update(kernel="k_lowpass_sub2_px8<%d>" % kind, prep="PREP_LP_PX8", aligned16=a16, items=o.nrows * o.ncols)
    return p


def copy_plan(src, dst):
    rc = copy_check(src, dst)
    if rc:
        return dict(op="copy", rejected=rc)
    al = src.base % 16 == 0 and dst.base % 16 == 0 and src.pitch % 16 == 0 and dst.pitch % 16 == 0
    wbytes = src.ncols * src.elem_bytes
    nvec, tail = wbytes // 16, wbytes % 16
    b = dst.border
    items = dst.nrows * (nvec + tail) + 2 * b * (dst.ncols + 2 * b) + 2 * b * dst.nrows
    if not al or src.base == dst.base:
        return dict(op="copy", kernel="fill" if src.base == dst.base else "copy+fill", prep=None, items=items, mirrored=b > 0)
    return dict(op="copy", kernel="k_copy_mirror", prep="PREP_COPY_MIRROR", items=items, mirrored=b > 0)


def prepare_check(i1, i2, prev, nxt, grad, n, gf):
    """pyrlk_prepare_check(): every step's checks, in the order of the steps"""
    if not (1 <= n <= 16):
        return E_ARG
    for rc in (copy_check(i1, prev[0]), copy_check(i2, nxt[0]), scharr_check(prev[0], grad[0], 1) if grad else OK):
        if rc:
            return rc
    for l in range(1, n):
        for rc in (lowpass_check(prev[l - 1], prev[l], 0, 1), lowpass_check(nxt[l - 1], nxt[l], 0, 1),
                   lowpass_check(grad[l - 1], grad[l], 2 if gf else 1, 1) if grad else OK):
            if rc:
                return rc
    return OK


def prepare_plan(i1, i2, prev, nxt, grad, n, gf, env, sms):
    """the form vppb_pyrlk_prepare takes: rejected (code, and under VPPB_PREPARE=fused the reason), fused (its phases, the items of the
    largest phase, the CTAs they ask for and whether the cooperative cap certainly cuts that grid) or streams (its launches)"""
    rc = prepare_check(i1, i2, prev, nxt, grad, n, gf)
    if rc:
        return dict(form="rejected", code=rc)
    e = env.get("VPPB_PREPARE")
    want_fused = (e == "fused") if e is not None else grad is None
    gk = 2 if gf else 1
    if want_fused:
        why = None
        if n > PREP_MAX_LEVELS:
            why = "more than 8 levels"
        else:
            phases = [[copy_plan(i1, prev[0]), copy_plan(i2, nxt[0])]]
            for l in range(1, n + 1):
                ph = []
                if grad:
                    ph.append(scharr_plan(prev[0], grad[0], gf, 1) if l == 1 else lowpass_plan(grad[l - 2], grad[l - 1], gk, 1))
                elif l == n:
                    break
                if l < n:
                    ph += [lowpass_plan(prev[l - 1], prev[l], 0, 1), lowpass_plan(nxt[l - 1], nxt[l], 0, 1)]
                phases.append(ph)
            # prep_copy_mirror: 16-byte aligned rows and distinct buffers (the other ops take any layout the checks accept)
            if any(op["prep"] is None for op in phases[0]):
                why = "the images do not have the library layout"
        if why is None:
            most = max(sum(op["items"] for op in ph) for ph in phases)
            blocks = max(1, (most + 255) // 256)
            cap = "capped" if blocks > CTAS_PER_SM_MAX * sms else "uncapped" if blocks <= sms else "either"
            return dict(form="fused", nphases=len(phases), phases=[[op["prep"] for op in ph] for ph in phases], most=most, blocks=blocks, cap=cap,
                        aligned16=sorted({op["aligned16"] for ph in phases for op in ph if "aligned16" in op}),
                        tails=any(op.get("tail_items") for ph in phases for op in ph), grad=grad is not None, nlevels=n)
        if e == "fused":
            return dict(form="rejected", code=E_ARG, reason=why)
        fell_back = why
    else:
        fell_back = None
    ops = [copy_plan(i2, nxt[0])] + [lowpass_plan(nxt[l - 1], nxt[l], 0, 1) for l in range(1, n)] + [copy_plan(i1, prev[0])]
    if grad:
        ops += [scharr_plan(prev[0], grad[0], gf, 1)] + [lowpass_plan(grad[l - 1], grad[l], gk, 1) for l in range(1, n)]
    ops += [lowpass_plan(prev[l - 1], prev[l], 0, 1) for l in range(1, n)]
    return dict(form="streams", fell_back=fell_back, launches=[op["kernel"] for op in ops], grad=grad is not None, nlevels=n)


# ------------------------------------------------------------------ what the tables must reach
def _kernel_names(p):
    """reach names of one stand-alone plan"""
    if "rejected" in p:
        return {"%s rejected" % p["op"]}
    out = {p["kernel"] + (" mirrored" if p["mirrored"] else " plain") if p["op"] == "scharr" else p["kernel"]}
    if p.get("tail_items"):
        out.add("k_lowpass_sub2_u8_fast with tail items")
    if "aligned16" in p:
        out.add("%s aligned16=%d" % (p["kernel"], p["aligned16"]))
    return out


def reached(res):
    out = set()
    for r in res["results"]:
        p = r["plan"]
        if r["kind"] == "prepare":
            g = "with" if p.get("grad") else "without"
            if p["form"] == "fused":
                out.add("fused %s a gradient pyramid" % g)
                out.add("fused %s %s a gradient pyramid" % (p["cap"], g))
                out.update(k for ph in p["phases"] for k in ph)
                out.update("PREP_LP_PX8 aligned16=%d" % a for a in p["aligned16"])
                if p["tails"]:
                    out.add("PREP_LP_U8_FAST with tail items")
                if p["nlevels"] >= 5:
                    out.add("fused with 5 to 8 levels")
                if r.get("calls", 1) > 64:
                    out.add("more than 64 fused calls on one stream")
            elif p["form"] == "streams":
                out.add("streams %s a gradient pyramid" % g)
                if p["fell_back"] == "more than 8 levels":
                    out.add("fallback above 8 levels")
                elif p["fell_back"]:
                    out.add("fallback for the layout")
            else:
                out.add("prepare rejected" + (": " + p["reason"] if p.get("reason") else ""))
        else:
            out |= _kernel_names(p)
    return out


STANDALONE = {"k_scharr_u8_v8<0> plain", "k_scharr_u8_v8<1> plain", "k_scharr_u8<0> plain", "k_scharr_u8<1> plain",
              "k_scharr_u8_v8<0> mirrored", "k_scharr_u8_v8<1> mirrored", "k_scharr_u8<0> mirrored", "k_scharr_u8<1> mirrored",
              "k_lowpass_sub2_u8_fast", "k_lowpass_sub2_u8_fast with tail items", "k_lowpass_sub2<0>",
              "k_lowpass_sub2_px8<1> aligned16=0", "k_lowpass_sub2_px8<1> aligned16=1", "k_lowpass_sub2_px8<2> aligned16=0",
              "k_lowpass_sub2_px8<2> aligned16=1", "k_copy_mirror", "copy+fill", "scharr rejected", "lowpass rejected", "copy rejected"}
PREP_KINDS = {"PREP_COPY_MIRROR", "PREP_SCHARR_V8", "PREP_SCHARR_PX", "PREP_LP_U8_FAST", "PREP_LP_GENERIC", "PREP_LP_PX8"}


def expected(policy):
    common = STANDALONE | {"prepare rejected"}
    if policy == "fused":
        return common | PREP_KINDS | {"PREP_LP_PX8 aligned16=0", "PREP_LP_PX8 aligned16=1", "PREP_LP_U8_FAST with tail items",
                                      "fused capped with a gradient pyramid", "fused uncapped with a gradient pyramid",
                                      "fused capped without a gradient pyramid", "fused uncapped without a gradient pyramid",
                                      "fused with 5 to 8 levels", "more than 64 fused calls on one stream",
                                      "prepare rejected: more than 8 levels", "prepare rejected: the images do not have the library layout"}
    if policy == "streams":
        return common | {"streams with a gradient pyramid", "streams without a gradient pyramid"}
    return common | {"PREP_COPY_MIRROR", "PREP_LP_U8_FAST", "PREP_LP_GENERIC", "PREP_LP_U8_FAST with tail items",
                     "fused capped without a gradient pyramid", "fused uncapped without a gradient pyramid", "fused with 5 to 8 levels",
                     "more than 64 fused calls on one stream", "streams with a gradient pyramid", "streams without a gradient pyramid",
                     "fallback above 8 levels", "fallback for the layout"}


def every_path():
    return STANDALONE | PREP_KINDS | {"fused capped with a gradient pyramid", "fused uncapped with a gradient pyramid",
                                      "fused capped without a gradient pyramid", "fused uncapped without a gradient pyramid",
                                      "streams with a gradient pyramid", "streams without a gradient pyramid", "fallback above 8 levels"}


# ------------------------------------------------------------------ the case tables
ALIGNS = (128, 64, 32, 16, 8, 4, 1)


def _sa(name, op, shape, pix="u8", oshape=None, ib=1, ia=128, ob=0, oa=128, mirror=1, as_float=0, iview=None, oview=None, expect=None):
    """one stand-alone call: op scharr / lowpass / copy on an input of `shape` (pix; border ib, alignment ia, or a view: ("col", c) at
    column c, ("band", r) rows r .. of a taller parent, ("tight",) 16 bytes left and the row padded to 16 bytes only); output of `oshape`
    (default: the level size), border ob, alignment oa or oview; expect: the code the call must return (else the plan's)"""
    return dict(kind="sa", name=name, op=op, shape=shape, pix=pix, oshape=oshape, ib=ib, ia=ia, ob=ob, oa=oa, mirror=mirror, as_float=as_float,
                iview=iview, oview=oview, expect=expect)


def standalone_cases():
    T = []
    # Scharr: every residue of the width mod 8 around the 8-pixel groups, 1 x N, N x 1, 2 x 2, 3 x 3; input border exactly 1
    for i, nc in enumerate(list(range(40, 48)) + [1, 2, 3, 7, 8, 9, 15, 17]):
        nr = (5, 3, 1, 2, 7, 9, 4, 6)[i % 8]
        T.append(_sa("scharr_%dx%d" % (nr, nc), "scharr", (nr, nc), ob=(0, 1, 2, 3)[i % 4] if min(nr, nc) >= 3 else min(nr, nc, i % 3),
                     as_float=i % 2, mirror=(i // 2) % 2 or i >= 8))
    for shape in ((1, 1), (1, 33), (33, 1), (2, 2), (3, 3)):
        for af in (0, 1):
            T.append(_sa("scharr_small_%dx%d_f%d" % (shape + (af,)), "scharr", shape, as_float=af, ob=min(shape), mirror=1))
    # alignments chosen independently for input and output (8-byte elements: an output is 8- or 16-byte aligned); output borders
    # 0 .. 6 (6 = the level size)
    for ai in ALIGNS:
        for oa in (128, 16, 8, 4):
            T.append(_sa("scharr_a%d_o%d" % (ai, oa), "scharr", (6, 29 + ai % 7), ia=ai, oa=oa, ob=(ai + oa) % 7, as_float=(ai // 4) % 2, mirror=1))
    # the right-hand room of v8's last group: a tight row with 16 bytes left of column 0 (40: room for 5 groups; 41, 47: not for 6)
    for nc in (40, 41, 47):
        for af in (0, 1):
            for mirror in (0, 1):
                T.append(_sa("scharr_tight_%d_f%d_m%d" % (nc, af, mirror), "scharr", (7, nc), iview=("tight",), ob=2, as_float=af, mirror=mirror))
    # views: an odd column (byte loads), column 8 (8- but not 16-byte aligned), 16-aligned column windows / row bands; vint2 / vfloat2
    # output views at an odd column (8 mod 16: the 1-pixel kernel) and at column 2
    for iv, ov in ((("col", 3), None), (("col", 8), None), (("col", 16), None), (("band", 5), None), (None, ("col", 1)), (None, ("col", 2)),
                   (("col", 8), ("col", 2))):
        for af in (0, 1):
            T.append(_sa("scharr_view_%s_%s_f%d" % (iv, ov, af), "scharr", (9, 37), iview=iv, oview=ov, ob=2, as_float=af))
    # rejected: input border 0, output border larger than the level, output larger than the input, wrong element size
    T.append(_sa("scharr_rej_inborder0", "scharr", (8, 20), ib=0, ob=1, expect=E_BORDER))
    T.append(_sa("scharr_rej_outborder", "scharr", (4, 20), ob=5, expect=E_BORDER))
    T.append(_sa("scharr_rej_bigger", "scharr", (8, 20), oshape=(9, 20), ob=1, expect=E_ARG))
    T.append(_sa("scharr_rej_elem", "scharr", (8, 20), pix="f32", ob=1, expect=E_ARG))
    # low-pass u8: parent widths 16k-1 .. 16k+2 around the fast path's 16-byte groups, even and odd parents, rows / cols below 4
    for i, nc in enumerate((15, 16, 17, 18, 31, 32, 33, 34, 47, 48, 49, 50)):
        nr = (9, 10, 7, 4, 12, 5, 6, 11)[i % 8]
        T.append(_sa("lp_u8_%dx%d" % (nr, nc), "lowpass", (nr, nc), ib=2 + i % 2, ob=i % 4, mirror=i % 3 != 0))
    for shape in ((2, 2), (3, 3), (2, 17), (17, 2), (3, 40), (40, 3), (4, 4), (5, 5)):
        for pix in ("u8", "vint2", "vfloat2"):
            T.append(_sa("lp_small_%s_%dx%d" % ((pix,) + shape), "lowpass", shape, pix=pix, ib=2, ob=min(1 + shape[0] // 2, 1 + shape[1] // 2)))
    # outputs smaller than 1 + n/2 (even and odd parents), output borders 0 .. 6 with one equal to the level size
    for pix in ("u8", "vint2", "vfloat2"):
        for (nr, nc), (onr, onc), ob in (((24, 40), (12, 20), 6), ((25, 41), (13, 21), 4), ((24, 41), (10, 21), 5), ((25, 40), (13, 6), 6),
                                         ((26, 38), (14, 20), 0), ((13, 13), (7, 7), 7)):
            T.append(_sa("lp_out_%s_%dx%d_%dx%d_b%d" % (pix, nr, nc, onr, onc, ob), "lowpass", (nr, nc), pix=pix, oshape=(onr, onc), ib=2, ob=ob))
    # alignments, input and output independently
    for pix in ("u8", "vint2", "vfloat2"):
        for ai in ALIGNS:
            for oa in (128, 8, 4, 1):
                T.append(_sa("lp_%s_a%d_o%d" % (pix, ai, oa), "lowpass", (11 + ai % 3, 35 + oa % 5), pix=pix, ib=2, ia=ai, oa=oa, ob=(ai + oa) % 4))
    # views: u8 at an odd column / a 16-aligned column window / a row band; vint2 / vfloat2 at an odd column (8 mod 16: the unaligned
    # px8 loads) and at column 2
    for iv in (("col", 3), ("col", 16), ("col", 32), ("band", 4)):
        T.append(_sa("lp_u8_view_%s_%d" % iv, "lowpass", (14, 45), ib=2, iview=iv, ob=3))
    for pix in ("vint2", "vfloat2"):
        for iv in (("col", 1), ("col", 2), ("band", 3)):
            T.append(_sa("lp_%s_view_%s_%d" % ((pix,) + iv), "lowpass", (13, 21), pix=pix, ib=2, iview=iv, ob=2))
        T.append(_sa("lp_%s_oview" % pix, "lowpass", (13, 21), pix=pix, ib=2, oview=("col", 1), ob=2))
    T.append(_sa("lp_u8_oview", "lowpass", (14, 45), ib=2, oview=("col", 3), ob=2))
    # rejected: input border 1, output border larger than the level, output larger than 1 + n/2, element sizes
    T.append(_sa("lp_rej_inborder1", "lowpass", (20, 30), ib=1, ob=2, expect=E_BORDER))
    T.append(_sa("lp_rej_outborder", "lowpass", (8, 30), ib=2, ob=6, expect=E_BORDER))
    T.append(_sa("lp_rej_bigger", "lowpass", (20, 30), oshape=(11, 17), ib=2, ob=1, expect=E_ARG))
    T.append(_sa("lp_rej_elem", "lowpass", (20, 30), pix="f32", ib=2, ob=1, expect=E_ARG))
    # copy + mirror: alignments, borders 0 .. 6 (= the image size), views, u8 and vint2
    for i, (ai, oa) in enumerate(((128, 128), (16, 128), (128, 16), (4, 128), (128, 4), (1, 1), (16, 16), (8, 64))):
        for pix in ("u8", "vint2"):
            T.append(_sa("copy_%s_a%d_o%d" % (pix, ai, oa), "copy", (6 + i, 23 + 3 * i), pix=pix, ib=1, ia=ai, oa=oa, ob=min(i, 6)))
    T.append(_sa("copy_border_eq_size", "copy", (6, 9), ob=6))
    T.append(_sa("copy_view_odd", "copy", (7, 30), iview=("col", 3), ob=2))
    T.append(_sa("copy_oview_odd", "copy", (7, 30), oview=("col", 5), ob=2))
    T.append(_sa("copy_rej_border", "copy", (4, 9), ob=5, expect=E_BORDER))
    return T


def _pp(name, shape, n, border=2, grad=None, gborder=None, ia=128, prev0=None, grad0=None, mutate=None, calls=1, expect=None, big=False):
    """one vppb_pyrlk_prepare call: frames of `shape`, n levels, prev / next border `border`, grad None / "vint2" / "vfloat2" with border
    gborder (default: border); ia: alignment of i1 / i2 (128 / 16 / 4 / 1) or "view" (at an odd column); prev0 = 16: prev[0] and next[0]
    at alignment 16 (the generic low-pass); grad0 = 8: grad[0] 8- but not 16-byte aligned (the 1-pixel Scharr, unaligned px8 loads);
    mutate: one invalid descriptor (see Runner._prepare_images); calls: that many calls queued on one stream before the first sync"""
    return dict(kind="prepare", name=name, shape=shape, n=n, border=border, grad=grad, gborder=border if gborder is None else gborder, ia=ia,
                prev0=prev0, grad0=grad0, mutate=mutate, calls=calls, expect=expect, big=big)


def prepare_cases(big=False):
    T = []
    # 1 .. 8 levels, with no / a vint2 / a vfloat2 gradient pyramid, odd and even frames, borders 2 .. 18
    shapes = ((5, 5), (6, 7), (13, 9), (40, 56), (37, 61), (64, 65), (120, 97), (270, 481))
    for n in range(1, 9):
        for j, g in enumerate((None, "vint2", "vfloat2")):
            shape = shapes[(n + 3 * j) % len(shapes)]
            lv = [shape]
            for _ in range(n - 1):
                lv.append((1 + lv[-1][0] // 2, 1 + lv[-1][1] // 2))
            b = min(min(lv[-1]), (2, 3, 4, 7, 14, 18)[(n + j) % 6])
            T.append(_pp("n%d_%s_%dx%d_b%d" % (n, g, shape[0], shape[1], b), shape, n, border=max(2, b), grad=g, ia=(128, 16, 4, 1)[(n + j) % 4]))
    # borders up to the flow's 2 * winsize (winsize 9 -> 18, 11 -> 22) on a frame whose levels are large enough
    for b, g in ((18, None), (22, "vint2"), (9, "vfloat2"), (5, None)):
        T.append(_pp("border%d_%s" % (b, g), (270, 481), 4, border=b, grad=g, gborder=b // 2 + 1))
    # 9, 12 and 16 levels: the streams fallback under the default, VPPB_E_ARG under VPPB_PREPARE=fused
    for n, g in ((9, None), (12, "vint2"), (16, None), (16, "vfloat2")):
        T.append(_pp("n%d_%s" % (n, g), (131, 203), n, grad=g))
    # i1 / i2 at alignments 128 / 16 / 4 / 1 and as views (the streams fallback); prev[0] at alignment 16; grad[0] 8-aligned
    for ia in (128, 16, 4, 1, "view"):
        for g in (None, "vfloat2"):
            T.append(_pp("i_%s_%s" % (ia, g), (45, 77), 3, grad=g, ia=ia))
    for g in (None, "vint2", "vfloat2"):
        T.append(_pp("prev0_a16_%s" % g, (47, 66), 4, grad=g, prev0=16))
    for g in ("vint2", "vfloat2"):
        T.append(_pp("grad0_a8_%s" % g, (39, 58), 4, grad=g, grad0=8))
        T.append(_pp("prev0_a16_grad0_a8_%s" % g, (33, 50), 5, border=3, grad=g, prev0=16, grad0=8))
    # a fused grid the cooperative cap certainly cuts (more than 8 CTAs per SM of work in the copy phase: 31-byte rows are 16 items each)
    for g in (None, "vint2", "vfloat2"):
        T.append(_pp("tall_%s" % g, (18000, 31), 3, grad=g))
    # a fused grid certainly below one CTA per SM (every phase fits in two CTAs)
    for g in (None, "vint2"):
        T.append(_pp("tiny_%s" % g, (7, 9), 2, grad=g))
    # more than 64 fused calls queued on one stream: the 64 barrier counters are handed out again
    T.append(_pp("queued_70", (23, 37), 3, calls=70))
    # rejected calls: nothing may be written
    T.append(_pp("rej_scharr_inborder0", (24, 30), 1, border=0, grad="vint2", expect=E_BORDER))
    T.append(_pp("rej_lp_inborder1", (40, 56), 2, border=1, expect=E_BORDER))
    T.append(_pp("rej_lp_inborder1_grad", (40, 56), 2, border=1, grad="vint2", expect=E_BORDER))
    T.append(_pp("rej_border_gt_level", (40, 56), 6, border=4, grad="vint2", expect=E_BORDER))
    T.append(_pp("rej_border_gt_level_nograd", (40, 56), 6, border=4, expect=E_BORDER))
    T.append(_pp("rej_gborder_gt_level", (40, 56), 6, border=2, grad="vfloat2", gborder=4, expect=E_BORDER))
    T.append(_pp("rej_level0_border", (3, 30), 2, border=4, expect=E_BORDER))
    T.append(_pp("rej_grad_elem4", (40, 56), 3, grad="vint2", mutate="grad_elem4", expect=E_ARG))
    T.append(_pp("rej_next1_elem8", (40, 56), 3, mutate="next1_elem8", expect=E_ARG))
    T.append(_pp("rej_next2_bigger", (40, 56), 4, grad="vint2", mutate="next2_bigger", expect=E_ARG))
    T.append(_pp("rej_grad2_bigger", (40, 56), 4, grad="vfloat2", mutate="grad2_bigger", expect=E_ARG))
    T.append(_pp("rej_i2_domain", (40, 56), 3, mutate="i2_domain", expect=E_ARG))
    T.append(_pp("rej_nlevels0", (40, 56), 1, mutate="nlevels0", expect=E_ARG))
    T.append(_pp("rej_nlevels17", (40, 56), 17, expect=E_ARG))
    if big:
        for shape in ((1080, 1920), (2160, 3840), (4320, 7680)):
            for g in (None, "vfloat2" if shape[0] == 2160 else "vint2"):
                T.append(_pp("big_%dx%d_%s" % (shape + (g,)), shape, 4 if shape[0] < 4000 else 5, border=9 if g else 18, grad=g, big=True))
    return T


# ------------------------------------------------------------------ device images and references
class Tight:
    """a u8 image with 16 bytes left of column 0 and rows padded to 16 bytes only (align 16, border 1): less room right of the
    last 8-pixel group than the library layout leaves"""

    def __init__(self, vpp, nrows, ncols):
        from vpp_b200 import capi

        self.capi = capi
        self.pitch = (16 + ncols + 1 + 15) // 16 * 16
        self.shape = (nrows + 3, self.pitch)  # one row above, one below, and a spare row: the 1-pixel kernel reads column ncols
        self.mem = capi.VppbImg()
        capi.check(capi.lib.vppb_alloc(C.byref(self.mem), 1, self.shape[0] * self.pitch, 1, 0, 256))
        self.start = self.mem.base
        self.raw = capi.VppbImg(self.start, None, self.shape[0], self.pitch, self.pitch, 0, 1, 1)
        self.desc = capi.VppbImg(self.start + self.pitch + 16, None, nrows, ncols, self.pitch, 1, 1, 16)

    put, get, at = Alloc.put, Alloc.get, Alloc.at

    def __del__(self):
        self.capi.lib.vppb_free(C.byref(self.mem))


def host_data(pix, shape, rng):
    """bytes of a whole allocation: u8 noise; vint2: ints of either sign, |v| < 2^26, rarely multiples of 16; vfloat2 / f32: finite
    floats over 40 binades, so that the result depends on the order of the additions"""
    if pix in ("u8", "i8"):
        return rng.integers(0, 256, shape, dtype=np.uint8)
    n = shape[0] * shape[1] // 4
    if pix in ("vint2", "i32"):
        v = rng.integers(-(1 << 26) + 1, 1 << 26, n).astype(np.int32)
    else:
        v = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    return v.view(np.uint8).reshape(shape)


def vo_at(orc, host, r, c, desc):
    """a VoImg of desc's image inside `host`, the host copy of its allocation, pixel (0,0) at byte (r, c)"""
    return orc.VoImg(host.ctypes.data + r * host.shape[1] + c, desc.nrows, desc.ncols, desc.pitch, desc.border, desc.elem_bytes)


def frame_bytes(h, b):
    """rows [-b, nrows + b) x columns [-b, ncols + b) of oracle image h as bytes"""
    v = np.ascontiguousarray(h._frame_view(b))
    return v.view(np.uint8).reshape(h.nrows + 2 * b, -1)


def first_mismatch(got, want, r, c, elem):
    bad = np.flatnonzero(got != want)
    if not len(bad):
        return None
    br, bc = divmod(int(bad[0]), got.shape[1])
    return dict(row=br - r, byte=bc - c, col=(bc - c) // elem, got=int(got[br, bc]), want=int(want[br, bc]), count=int(len(bad)))


class Runner:
    def __init__(self, vpp, sms, env, backend):
        from tests import oracle as orc
        from vpp_b200 import capi

        self.vpp, self.sms, self.env, self.backend, self.orc, self.capi = vpp, sms, env, backend, orc, capi
        self.lib = capi.lib

    def idle(self):
        """wait for the whole device, side streams included"""
        self.capi.check(self.lib.vppb_sync(None))
        if self.backend == "gpu":
            import torch

            torch.cuda.synchronize()

    def _image(self, shape, pix, border, align, view, rng, fill):
        """(alloc, desc, host bytes of the allocation as uploaded, (row, byte) of pixel (0,0)); fill: "data" or "sentinel"""
        nr, nc = shape
        if view is None:
            a = Alloc(self.vpp, nr, nc, pix, border, align)
            desc = a.img.desc
        elif view[0] == "tight":
            a = Tight(self.vpp, nr, nc)
            desc = a.desc
        elif view[0] == "col":
            a = Alloc(self.vpp, nr + 2, nc + view[1] + 3, pix, border, align)
            desc = a.img.subimage(self.vpp.Box2d((1, view[1]), (nr, view[1] + nc - 1))).desc
        else:
            a = Alloc(self.vpp, nr + 2 * view[1], nc, pix, border, align)
            desc = a.img.subimage(self.vpp.Box2d((view[1], 0), (view[1] + nr - 1, nc - 1))).desc
        host = host_data(pix, a.shape, rng) if fill == "data" else np.full(a.shape, SENTINEL, np.uint8)
        a.put(host)
        return a, desc, host, a.at(desc)

    # ---- stand-alone calls
    def run_standalone(self, k):
        lib, orc = self.lib, self.orc
        o = orc.load()
        rng = np.random.default_rng(zlib.crc32(k["name"].encode()))
        nr, nc = k["shape"]
        pix = k["pix"]
        if k["op"] == "scharr":
            opix, oshape = ("vfloat2" if k["as_float"] else "vint2"), k["oshape"] or (nr, nc)
            if pix != "u8":
                opix = "vint2"
        elif k["op"] == "lowpass":
            opix, oshape = pix, k["oshape"] or (1 + nr // 2, 1 + nc // 2)
        else:
            opix, oshape = pix, (nr, nc)
        ia, ida, ih, (ir, ic) = self._image((nr, nc), pix, k["ib"], k["ia"], k["iview"], rng, "data")
        oa, oda, oh, (orow, ocol) = self._image(oshape, opix, k["ob"], k["oa"], k["oview"], rng, "sentinel")
        kind = {"u8": 0, "vint2": 1, "vfloat2": 2}.get(pix, 1)
        if k["op"] == "scharr":
            plan = scharr_plan(ida, oda, k["as_float"], k["mirror"])
            fn = lib.vppb_scharr_u8_mirror if k["mirror"] else lib.vppb_scharr_u8
            rc = fn(C.byref(ida), C.byref(oda), k["as_float"], None)
        elif k["op"] == "lowpass":
            plan = lowpass_plan(ida, oda, kind, k["mirror"])
            fn = lib.vppb_lowpass_sub2_mirror if k["mirror"] else lib.vppb_lowpass_sub2
            rc = fn(C.byref(ida), C.byref(oda), kind, None)
        else:
            plan = copy_plan(ida, oda)
            rc = lib.vppb_copy2d_mirror(C.byref(ida), C.byref(oda), None)
        err = lib.vppb_last_error().decode("utf-8", "replace") if rc else None
        self.idle()
        want = oh.copy()
        code = plan.get("rejected", OK)
        if code == OK:
            vi, vo = vo_at(orc, ih, ir, ic, ida), vo_at(orc, want, orow, ocol, oda)
            if k["op"] == "scharr":
                o.vo_scharr_u8(C.byref(vi), C.byref(vo), k["as_float"])
            elif k["op"] == "lowpass":
                o.vo_lowpass_sub2(C.byref(vi), C.byref(vo), kind)
            else:
                o.vo_copy(C.byref(vi), C.byref(vo), 0)
            if k["op"] == "copy" or k["mirror"]:
                o.vo_fill_border_mirror(C.byref(vo))
        problems = []
        if k["expect"] is not None and code != k["expect"]:
            problems.append("the plan says %d, the case expects %d" % (code, k["expect"]))
        if rc != code:
            problems.append("returned %d (%s), the plan says %d" % (rc, err, code))
        bad = first_mismatch(oa.get(), want, orow, ocol, oda.elem_bytes)
        bad_in = first_mismatch(ia.get(), ih, ir, ic, ida.elem_bytes)
        if bad_in:
            problems.append("the input changed")
        return [dict(kind="sa", case=k["name"], ok=not problems and bad is None, error="; ".join(problems) or None, mismatch=bad, rc=rc, plan=plan)]

    # ---- vppb_pyrlk_prepare
    def _prepare_images(self, k, rng):
        """descriptors and allocations of one call; the mutations make one of them invalid"""
        nr, nc = k["shape"]
        n, b, g, gb, mut = k["n"], k["border"], k["grad"], k["gborder"], k["mutate"]
        view = ("col", 3) if k["ia"] == "view" else None
        ia = 128 if view else k["ia"]
        ims = {}
        ims["i1"] = self._image((nr, nc), "u8", 0, ia, view, rng, "data")
        ims["i2"] = self._image((nr, nc + (1 if mut == "i2_domain" else 0)), "u8", 1, ia, view, rng, "data")
        sizes = [(nr, nc)]
        for _ in range(max(n, 1) - 1):
            sizes.append((1 + sizes[-1][0] // 2, 1 + sizes[-1][1] // 2))
        for name in ("prev", "next", "grad"):
            if name == "grad" and not g:
                continue
            for l, (lr, lc) in enumerate(sizes):
                pix, border, align, lview = ("u8", b, 128, None) if name != "grad" else (g, gb, 128, None)
                if l == 0 and name != "grad" and k["prev0"]:
                    align = k["prev0"]
                if l == 0 and name == "grad" and k["grad0"]:
                    lview = ("col", 1)  # 8 bytes past a 16-byte boundary in a 128-aligned parent
                if (mut == "grad_elem4" and name == "grad" and l == 1) or (mut == "next1_elem8" and name == "next" and l == 1):
                    pix = "f32" if name == "grad" else "vint2"
                if (mut == "next2_bigger" and name == "next" and l == 2) or (mut == "grad2_bigger" and name == "grad" and l == 2):
                    lr += 1
                ims["%s%d" % (name, l)] = self._image((lr, lc), pix, border, align, lview, rng, "sentinel")
        if k["grad0"] and g:
            assert ims["grad0"][1].base % 16 == 8, "grad[0] should be 8- but not 16-byte aligned"
        return ims, len(sizes)

    def _expected(self, k, ims, nl, o, f1, f2):
        """the oracle's pyramids placed in copies of the sentinel-filled allocations"""
        from tests.oracle_ops import oracle_grad_pyramid, oracle_pyramid

        want = {}
        hp = oracle_pyramid(f1, nl, "u8", k["border"], o)
        hn = oracle_pyramid(f2, nl, "u8", k["border"], o)
        hg = oracle_grad_pyramid(hp, k["grad"], k["gborder"], o) if k["grad"] else []
        for name, hs, b in (("prev", hp, k["border"]), ("next", hn, k["border"]), ("grad", hg, k["gborder"])):
            for l, h in enumerate(hs):
                _, d, host, (r, c) = ims["%s%d" % (name, l)]
                w = host.copy()
                e = d.elem_bytes
                w[r - b:r + d.nrows + b, c - b * e:c + (d.ncols + b) * e] = frame_bytes(h, b)
                want["%s%d" % (name, l)] = w
        return want

    def run_prepare(self, k):
        capi, lib = self.capi, self.lib
        big = k["big"]
        o = self.orc.load(omp=big)
        results = []
        sets = []
        for call in range(k["calls"]):
            rng = np.random.default_rng([zlib.crc32(k["name"].encode()), call])
            ims, nl = self._prepare_images(k, rng)
            arr = lambda name: (capi.VppbImg * nl)(*[ims["%s%d" % (name, l)][1] for l in range(nl)])
            prev, nxt = arr("prev"), arr("next")
            grad = arr("grad") if k["grad"] else None
            n = 0 if k["mutate"] == "nlevels0" else k["n"]
            plan = prepare_plan(ims["i1"][1], ims["i2"][1], list(prev), list(nxt), list(grad) if grad else None, n, k["grad"] == "vfloat2", self.env, self.sms)
            rc = lib.vppb_pyrlk_prepare(C.byref(ims["i1"][1]), C.byref(ims["i2"][1]), prev, nxt, grad, n, int(k["grad"] == "vfloat2"), None)
            err = lib.vppb_last_error().decode("utf-8", "replace") if rc else None
            sets.append((ims, nl, plan, rc, err))
        self.idle()
        for call, (ims, nl, plan, rc, err) in enumerate(sets):
            code = plan.get("code", OK)
            problems = []
            if k["expect"] is not None and code != k["expect"]:
                problems.append("the plan says %d, the case expects %d" % (code, k["expect"]))
            if rc != code:
                problems.append("returned %d (%s), the plan says %d" % (rc, err, code))
            elif plan.get("reason") and plan["reason"] not in (err or ""):
                problems.append("the error %r does not say %r" % (err, plan["reason"]))
            if code == OK:
                f = lambda name: ims[name][2][ims[name][3][0]:ims[name][3][0] + ims[name][1].nrows, ims[name][3][1]:ims[name][3][1] + ims[name][1].ncols]
                want = self._expected(k, ims, nl, o, f("i1"), f("i2"))
            else:
                want = {name: v[2] for name, v in ims.items() if name not in ("i1", "i2")}
            bad = None
            for name in ims:
                a, d, host, (r, c) = ims[name]
                m = first_mismatch(a.get(), want.get(name, host), r, c, d.elem_bytes)
                if m:
                    bad = dict(m, image=name)
                    break
            results.append(dict(kind="prepare", case=k["name"] + ("#%d" % call if k["calls"] > 1 else ""), ok=not problems and bad is None,
                                error="; ".join(problems) or None, mismatch=bad, rc=rc, plan=plan, calls=k["calls"]))
        return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=("gpu", "emu"), required=True)
    ap.add_argument("--policy", choices=list(POLICIES), required=True)
    ap.add_argument("--big", action="store_true", help="add 1080p, 4K and 8K pyramids with and without a gradient pyramid")
    ap.add_argument("--only", default=None, help="run the cases whose name contains this string")
    args = ap.parse_args()
    vpp, sms = _load(args.backend)
    env = {k: v for k, v in os.environ.items() if k == "VPPB_PREPARE"}
    run = Runner(vpp, sms, env, args.backend)
    results = []
    for k in standalone_cases() + prepare_cases(big=args.big):
        if args.only is None or args.only in k["name"]:
            results.extend(run.run_standalone(k) if k["kind"] == "sa" else run.run_prepare(k))
    print(json.dumps(dict(backend=args.backend, policy=args.policy, sms=sms, env=env, results=results)))


def run_child(backend, policy, big=False, env=None, timeout=3000, only=None):
    """run the tables under POLICIES[policy] in a child process, every other library knob (VPPB_*, the emulator's VPPB_EMU_* aside)
    cleared: (returncode, parsed JSON or None, stderr)"""
    e = {k: v for k, v in (env if env is not None else os.environ).items() if not k.startswith("VPPB_") or k.startswith("VPPB_EMU_")}
    e.update(POLICIES[policy])
    cmd = [sys.executable, "-m", "tests.pyramid_paths", "--backend", backend, "--policy", policy] + (["--big"] if big else []) + (["--only", only] if only else [])
    r = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=timeout)
    try:
        res = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    except (ValueError, IndexError):
        res = None
    return r.returncode, res, r.stderr


def failures(res):
    return [r for r in res["results"] if not r["ok"]]


def unmet(res, policy):
    """what the policy's tables are written to reach and, by the transcribed dispatch, no longer reach"""
    return sorted(expected(policy) - reached(res))


if __name__ == "__main__":
    main()
