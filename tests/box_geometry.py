"""Child process of the 5x5 box geometry tests (tests/test_gpu_box_geometry.py, tests/test_emulated_box_geometry.py).

The byte box kernels choose their geometry at launch time: strips per row and 16-byte groups per strip (G), rows per task (R),
tasks per CTA, the tile or the streaming kernel for a single frame, 8 or 16 rows per tile.  That choice depends on the SM count
and on knobs (VPPB_BOX_SINGLE, VPPB_BOX_TH, VPPB_BOX_R) the library reads once per process, so each policy runs in a process
of its own:

    python -m tests.box_geometry --backend gpu|emu [--big]

runs the case table below through vppb_box5x5_{u8,u8c3}, _batch and _tiles under the environment it was started with and
prints one JSON object: the SM count the library sees and, per case and entry point, pass / fail with the first mismatching
byte and the launches the policy makes for it (`plan`, a transcription of vpp_b200/csrc/box.cu's launch rules).

Every output allocation is compared byte for byte, border and pitch padding included, with
  * a numpy reference: the 25 shifted slices of the input buffer as the kernel finds it in memory (its border, the parent's
    pixels around a view, the neighbouring tiles), summed in int64 and floor-divided by 25, channel by channel;
  * the sentinel it was filled with, everywhere outside the output's domain.
The numpy reference itself is checked against the C oracle (vo_box5x5_u8) on the same bytes."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# one child per policy: the knobs are read once per process
POLICIES = {
    "default": {},
    "single_stream": {"VPPB_BOX_SINGLE": "stream"},
    "th8": {"VPPB_BOX_TH": "8"},
    "th16": {"VPPB_BOX_TH": "16"},
    "r16": {"VPPB_BOX_R": "16"},
    "r21": {"VPPB_BOX_R": "21"},
    "r41": {"VPPB_BOX_R": "41"},
}
KNOBS = ("VPPB_BOX_SINGLE", "VPPB_BOX_TH", "VPPB_BOX_R", "VPPB_BOX_ABLATE")
SENTINEL = 0xA7

# ------------------------------------------------------------------ the launch policy of vpp_b200/csrc/box.cu, transcribed
BS_K, BS_MAX_G, BS_CTAS_PER_SM, BS_MAX_BATCH = 5, 126, 3, 128
BX_OUTW = 992
SINGLE_STREAM_BYTES = 96 * 1024 * 1024  # single frames of at least this many pixel bytes take the streaming kernel


def _knob(env, name):
    try:
        return int(env.get(name, "0"))
    except ValueError:
        return 0


def layout_pitch(ncols, elem, border, align):
    bs = border * elem
    if bs % align:
        bs += align - bs % align
    p = ncols * elem + 2 * bs
    if p % align:
        p += align - p % align
    return p


def tma_eligible(d):
    """box.cu's tma_eligible(): the library layout, a 16-byte aligned pixel (0,0) and pitch, border >= 2"""
    if d.align < 16 or d.border < 2 or d.base % 16 or d.pitch % 16:
        return False
    return layout_pitch(d.ncols, d.elem_bytes, d.border, d.align) == d.pitch


def stream_rows(strips_x_imgs, nrows, sms, forced):
    """box_stream_rows(): (R, chunks)"""
    ctas = sms * BS_CTAS_PER_SM
    m_max = max(4, (nrows + 4 + BS_K - 1) // BS_K)
    best_r, best = 16, float("inf")
    for m in range(4, m_max + 1):
        r = 5 * m - 4
        if forced > 0 and r != forced:
            continue
        tasks = (nrows + r - 1) // r * strips_x_imgs
        cost = (tasks + ctas - 1) // ctas * (5.0 * m + 2.0)
        if cost < best:
            best, best_r = cost, r
    return best_r, (nrows + best_r - 1) // best_r


def stream_launch(rowbytes, nrows, n, sms, env, plain):
    """one launch of k_box5_stream over n images (box5_stream_launch_nb); plain: not a row tile with neighbours"""
    groups = (rowbytes + 15) // 16
    strips = (groups + BS_MAX_G - 1) // BS_MAX_G
    G = (groups + strips - 1) // strips
    R, chunks = stream_rows(strips * n, nrows, sms, _knob(env, "VPPB_BOX_R"))
    tasks = n * strips * chunks
    return dict(kernel="stream", nb=1 if n == 1 else 4 if n <= 4 else 32 if n <= 32 else BS_MAX_BATCH, n=n, plain=plain, strips=strips, G=G,
                last=groups - (strips - 1) * G, R=R, chunks=chunks, tasks=tasks, ctas=min(tasks, sms * BS_CTAS_PER_SM))


def single_launch(d, sms, env):
    """box5_bytes(): streaming kernel, tile kernel or direct kernel for one frame"""
    rowbytes = d.ncols * d.elem_bytes
    if not tma_eligible(d):
        return dict(kernel="direct")
    if env.get("VPPB_BOX_SINGLE") == "stream" or rowbytes * d.nrows >= SINGLE_STREAM_BYTES:
        return stream_launch(rowbytes, d.nrows, 1, sms, env, plain=True)
    strips = (rowbytes + BX_OUTW - 1) // BX_OUTW
    th = _knob(env, "VPPB_BOX_TH")
    if th not in (8, 16):
        th = 16 if strips * ((d.nrows + 15) // 16) >= 4 * sms else 8
    return dict(kernel="tile", th=th, tiles=strips * ((d.nrows + th - 1) // th))


def plan(entry, ins, outs, sms, env, neighbours=False):
    """the launches box.cu makes for `entry` ("single": one call per image, "batch", "tiles") on these descriptors"""
    if entry == "single":
        return [single_launch(d, sms, env) for d in ins]
    if entry == "batch":
        o0 = outs[0]
        uniform = all(tma_eligible(i) and (i.nrows, i.ncols) == (ins[0].nrows, ins[0].ncols) and o.pitch == o0.pitch and (o.base % 16 == 0) == (o0.base % 16 == 0)
                      for i, o in zip(ins, outs))
        if not uniform or len(ins) == 1:
            return [single_launch(d, sms, env) for d in ins]
    rowbytes, n = ins[0].ncols * ins[0].elem_bytes, len(ins)
    return [stream_launch(rowbytes, ins[0].nrows, min(BS_MAX_BATCH, n - i0), sms, env, plain=not neighbours) for i0 in range(0, n, BS_MAX_BATCH)]


def unmet_claims(result, multi_task):
    """the geometries the table is written to reach, by the launches `plan` reports: names of those it no longer reaches"""
    st = [l for r in result["results"] for l in r["launches"] if l["kernel"] == "stream"]
    claims = {
        "G == 126 (a 2048-byte box)": any(l["G"] == 126 for l in st),
        "a last strip shorter than G": any(l["last"] < l["G"] for l in st),
        "the NB = 1 streaming kernel on a plain frame": any(l["nb"] == 1 and l["plain"] for l in st),
    }
    if multi_task:
        claims["more tasks than 3 x %d SMs" % result["sms"]] = any(l["tasks"] > BS_CTAS_PER_SM * result["sms"] for l in st)
    return [k for k, ok in claims.items() if not ok]


# ------------------------------------------------------------------ the case table
ENTRIES = ("single", "batch", "tiles")


def _case(name, pix, nrows, ncols, n=1, ib=2, ia=128, ob=0, oa=128, ocol=None, view=None, tiles=None, entries=ENTRIES):
    """n images (the batch entry takes 2 when n == 1); input border ib / alignment ia, output border ob / alignment oa;
    ocol: the output is a view at this column (row 1) of a larger sentinel-filled image; view: the input is a view of a
    parent image, ("band", position 0 / 1 / 2 of 3 row bands, mirror-filled parent) or ("cols", first column, parent columns);
    tiles: row tiles the tiles entry cuts a single frame into (default: 3 or 2 when the rows divide, else 1; a view goes whole)"""
    if view is not None:
        tiles = 1
    elif tiles is None:
        tiles = 3 if nrows % 3 == 0 and nrows >= 6 else 2 if nrows % 2 == 0 and nrows >= 4 else 1
    return dict(name=name, pix=pix, nrows=nrows, ncols=ncols, n=n, ib=ib, ia=ia, ob=ob, oa=oa, ocol=ocol, view=view, tiles=tiles, entries=entries)


def cases(big=False):
    T = []
    # strips: G = 126 (a 2048-byte box, TMA's 256 8-byte elements); 127 / 128 groups = 2 strips of 64 (+ 63, or a 1-byte last group);
    # 253 groups = 85 + 85 + 83; vuchar3 rows of 2016 / 2019 bytes
    for pix, nc in [("u8", 2016), ("u8", 2017), ("u8", 2033), ("u8", 4033), ("vuchar3", 672), ("vuchar3", 673)]:
        T.append(_case("strip_%s_%d" % (pix, nc), pix, 23 if nc < 4000 else 19, nc))
    for nc in range(1, 6):  # rows narrower than one 16-byte group
        T.append(_case("narrow_u8_%d" % nc, "u8", 7, nc))
        T.append(_case("narrow_c3_%d" % nc, "vuchar3", 8, nc))
    # rows around every forced R, and 2 .. 6 rows (fewer than one stage of 5)
    for r in (16, 21, 41):
        for nr in (r - 1, r, r + 1):
            T.append(_case("rows_%d_c3" % nr, "vuchar3", nr, 331 if nr % 2 else 673))
            T.append(_case("rows_%d_u8" % nr, "u8", nr, 2017 if nr % 2 else 1000))
    for nr in range(2, 7):
        T.append(_case("rows_%d" % nr, "u8" if nr % 2 else "vuchar3", nr, 2033 if nr % 2 else 673))
    # many tasks per CTA (on the H100: 832 and 462 tasks on 396 CTAs under R = 16)
    T.append(_case("tasks_u8_200x2017x32", "u8", 200, 2017, n=32))
    T.append(_case("tasks_c3_100x673x33", "vuchar3", 100, 673, n=33))
    # outputs: 16 / 4 / 1-byte alignment (byte stores under the TMA kernels), borders 1 and 3, a view at an odd column
    for pix, nr, nc in [("u8", 17, 2017), ("vuchar3", 21, 673)]:
        for oa in (16, 4, 1):
            T.append(_case("out_a%d_%s" % (oa, pix), pix, nr, nc, oa=oa))
        for ob in (1, 3):
            T.append(_case("out_b%d_%s" % (ob, pix), pix, nr, nc, ob=ob))
        T.append(_case("out_b3_a4_%s" % pix, pix, nr, nc, ob=3, oa=4))
        T.append(_case("out_view_odd_%s" % pix, pix, nr, nc, ob=2, ocol=1))
        T.append(_case("out_view_c5_a16_%s" % pix, pix, nr, nc, ob=1, oa=16, ocol=5))
    # inputs: borders 2 .. 5 with alignments 16 .. 128 (vuchar3, border 2, alignment 16: the box starts at the first byte of the row)
    for ib in (2, 3, 4, 5):
        for ia in (16, 32, 64, 128):
            T.append(_case("in_b%d_a%d_c3" % (ib, ia), "vuchar3", 12, 673, ib=ib, ia=ia))
            T.append(_case("in_b%d_a%d_u8" % (ib, ia), "u8", 10, 2033, ib=ib, ia=ia))
    # row tiles: alignment 16 with a ragged last strip (the seam stage copies less than a box row), seams in multi-chunk tiles
    T.append(_case("tiles_a16_u8_2017", "u8", 40, 2017, ia=16, tiles=2))
    T.append(_case("tiles_a16_c3_673", "vuchar3", 44, 673, ia=16, tiles=2))
    T.append(_case("tiles_a16_u8_4033", "u8", 120, 4033, ia=16, tiles=3))
    T.append(_case("tiles_multichunk_c3", "vuchar3", 150, 673, ib=3, ia=32, tiles=3))
    T.append(_case("tiles_multichunk_u8", "u8", 168, 2017, ia=16, tiles=4))
    # TMA-eligible views: full-width row bands of a mirror-bordered parent, an interior column window that keeps the pitch
    for pos in (0, 1, 2):
        T.append(_case("view_band%d_c3" % pos, "vuchar3", 20, 673, view=("band", pos)))
        T.append(_case("view_band%d_u8" % pos, "u8", 17, 2016, ib=3, ia=16, view=("band", pos)))
    T.append(_case("view_cols_u8", "u8", 23, 84, view=("cols", 16, 100)))
    # batches: the 4 / 32 / 128-image kernels, a second launch, its last image alone (the NB = 1 kernel)
    for n in (4, 5, 32, 33, 128, 129, 257):
        T.append(_case("batch_%d" % n, "u8" if n % 2 else "vuchar3", 9, 40 if n % 2 else 17, n=n))
    if big:
        # the 96 MiB rule: 4400 x 7680 vuchar3 (101.4 MB) takes the streaming kernel, 4320 x 7680 (99.5 MB) the tile kernel
        T.append(_case("big_8k_4400", "vuchar3", 4400, 7680, entries=("single",)))
        T.append(_case("big_8k_4320", "vuchar3", 4320, 7680, entries=("single",)))
        T.append(_case("big_u8_40x7680x128", "u8", 40, 7680, n=128))
    return T


# ------------------------------------------------------------------ device images, references, comparisons
class Alloc:
    """an Image2d and a byte view of its whole allocation: border, pitch padding and all"""

    def __init__(self, vpp, nrows, ncols, pix, border, aligned):
        from vpp_b200 import capi
        from vpp_b200.image import layout

        self.capi = capi
        self.img = vpp.Image2d(nrows, ncols, pix, border=border, aligned=aligned)
        pitch, total, origin = layout(nrows, ncols, self.img.elem_bytes, border, aligned)
        self.pitch, self.shape, self.start = pitch, (total // pitch, pitch), self.img.desc.base - origin
        self.raw = capi.VppbImg(self.start, None, total // pitch, pitch, pitch, 0, 1, 1)

    def put(self, a):
        a = np.ascontiguousarray(a, np.uint8)
        assert a.shape == self.shape
        self.capi.check(self.capi.lib.vppb_upload(C.byref(self.raw), a.ctypes.data, self.pitch, 0, None))
        self.capi.check(self.capi.lib.vppb_sync(None))

    def get(self):
        a = np.empty(self.shape, np.uint8)
        self.capi.check(self.capi.lib.vppb_download(C.byref(self.raw), a.ctypes.data, self.pitch, 0, None))
        self.capi.check(self.capi.lib.vppb_sync(None))
        return a

    def at(self, desc):
        """(row, byte) of desc's pixel (0,0) in the allocation"""
        return divmod(desc.base - self.start, self.pitch)


def box_reference(raw, r, c, nrows, rowbytes, cs):
    """the 5x5 box of the image whose pixel (0,0) is byte (r, c) of raw: 25 shifted slices summed in int64, // 25"""
    assert r >= 2 and c >= 2 * cs and r + nrows + 2 <= raw.shape[0] and c + rowbytes + 2 * cs <= raw.shape[1], "neighbourhood outside the buffer"
    out = np.empty((nrows, rowbytes), np.uint8)
    for y0 in range(0, nrows, 512):
        y1 = min(nrows, y0 + 512)
        acc = np.zeros((y1 - y0, rowbytes), np.int64)
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                acc += raw[r + y0 + dy:r + y1 + dy, c + dx * cs:c + dx * cs + rowbytes]
        out[y0:y1] = acc // 25
    return out


def oracle_box(raw, r, c, nrows, ncols, cs):
    from tests import oracle as orc

    raw = np.ascontiguousarray(raw)
    out = np.zeros((nrows, ncols * cs), np.uint8)
    src = orc.VoImg(raw.ctypes.data + r * raw.shape[1] + c, nrows, ncols, raw.shape[1], 2, cs)
    dst = orc.VoImg(out.ctypes.data, nrows, ncols, ncols * cs, 0, cs)
    orc.load(omp=nrows * ncols * cs > 32 << 20).vo_box5x5_u8(C.byref(src), C.byref(dst), cs)
    return out


def first_mismatch(alloc, desc, ref):
    """None, or where the output allocation differs from `ref` inside desc's domain + the sentinel outside it"""
    got = alloc.get()
    want = np.full_like(got, SENTINEL)
    r, c = alloc.at(desc)
    want[r:r + ref.shape[0], c:c + ref.shape[1]] = ref
    bad = np.flatnonzero(got != want)
    if not len(bad):
        return None
    br, bc = divmod(int(bad[0]), got.shape[1])
    y, x = br - r, bc - c
    return dict(row=y, byte=x, inside=bool(0 <= y < ref.shape[0] and 0 <= x < ref.shape[1]), got=int(got[br, bc]), want=int(want[br, bc]), count=int(len(bad)))


class Runner:
    def __init__(self, vpp, sms, env):
        self.vpp, self.sms, self.env = vpp, sms, env
        from vpp_b200 import capi

        self.capi = capi

    def _input(self, k, i):
        """image i of case k: (desc, keep-alive, host bytes of its allocation, (row, byte) of its pixel (0,0) there)"""
        vpp, cs = self.vpp, 3 if k["pix"] == "vuchar3" else 1
        rng = np.random.default_rng([zlib.crc32(k["name"].encode()), i])
        nr, nc = k["nrows"], k["ncols"]
        v = k["view"]
        if v is None:
            a = Alloc(vpp, nr, nc, k["pix"], k["ib"], k["ia"])
            desc = a.img.desc
        elif v[0] == "band":
            a = Alloc(vpp, 3 * nr, nc, k["pix"], k["ib"], k["ia"])
            desc = a.img.subimage(vpp.Box2d((v[1] * nr, 0), (v[1] * nr + nr - 1, nc - 1))).desc
        else:
            a = Alloc(vpp, nr, v[2], k["pix"], k["ib"], k["ia"])
            desc = a.img.subimage(vpp.Box2d((0, v[1]), (nr - 1, v[1] + nc - 1))).desc
        host = rng.integers(0, 256, a.shape, dtype=np.uint8)
        a.put(host)
        if v is not None and v[0] == "band":
            vpp.fill_border_mirror(a.img)
            host = a.get()
        r, c = a.at(desc)
        if v is not None:  # the view passes box.cu's own test, and the TMA tensor rows (16 bytes left, up to 23 right) stay in the parent's rows
            assert tma_eligible(desc), k["name"]
            assert r >= 2 and r + nr + 2 <= a.shape[0] and c >= 16 and c - 16 + (nc * cs + 32 + 7) // 8 * 8 <= a.pitch, k["name"]
        return desc, a, host, (r, c)

    def _output(self, k, nrows):
        vpp, nc = self.vpp, k["ncols"]
        if k["ocol"] is None:
            a = Alloc(vpp, nrows, nc, k["pix"], k["ob"], k["oa"])
            desc = a.img.desc
        else:
            a = Alloc(vpp, nrows + 2, nc + k["ocol"] + 2, k["pix"], k["ob"], k["oa"])
            desc = a.img.subimage(vpp.Box2d((1, k["ocol"]), (nrows, k["ocol"] + nc - 1))).desc
        a.put(np.full(a.shape, SENTINEL, np.uint8))
        return desc, a

    def run_case(self, k):
        capi, cs = self.capi, 3 if k["pix"] == "vuchar3" else 1
        nr, nc = k["nrows"], k["ncols"]
        lib = capi.lib
        single = lib.vppb_box5x5_u8c3 if cs == 3 else lib.vppb_box5x5_u8
        batch = lib.vppb_box5x5_u8c3_batch if cs == 3 else lib.vppb_box5x5_u8_batch
        tiles = lib.vppb_box5x5_u8c3_tiles if cs == 3 else lib.vppb_box5x5_u8_tiles
        nimg = max(k["n"], 2) if "batch" in k["entries"] else k["n"]
        ins = [self._input(k, i) for i in range(nimg)]
        refs = []
        for i, (_, _, host, (r, c)) in enumerate(ins):
            refs.append(box_reference(host, r, c, nr, nc * cs, cs))
            if i < 4 and not np.array_equal(refs[-1], oracle_box(host, r, c, nr, nc, cs)):
                return [dict(case=k["name"], entry="reference", ok=False, error="numpy reference and C oracle disagree on image %d" % i, launches=[])]
        results = []
        for entry in k["entries"]:
            m = k["n"] if entry != "batch" else nimg
            if entry == "tiles" and (m > 1 or k["tiles"] == 1):
                if not all(tma_eligible(d) for d, _, _, _ in ins[:m]) or nr < 2:
                    continue
                src = [d for d, _, _, _ in ins[:m]]
                want = refs[:m]
                nbs, keep = None, []
            elif entry == "tiles":
                src, want, nbs, keep = self._row_tiles(k, ins[0], refs[0], cs)
            else:
                src, want, nbs, keep = [d for d, _, _, _ in ins[:m]], refs[:m], None, []
            outs = [self._output(k, w.shape[0]) for w in want]
            od = [d for d, _ in outs]
            arr = lambda ds: (capi.VppbImg * len(ds))(*ds)
            launches = plan(entry, src, od, self.sms, self.env, neighbours=nbs is not None)
            if entry == "single":
                for s, o in zip(src, od):
                    capi.check(single(C.byref(s), C.byref(o), None))
            elif entry == "batch":
                capi.check(batch(arr(src), arr(od), len(src), None))
            else:
                ups, dns = nbs if nbs else (None, None)
                capi.check(tiles(arr(src), ups, dns, arr(od), len(src), None))
            capi.check(lib.vppb_sync(None))
            bad = None
            for i, ((d, a), w) in enumerate(zip(outs, want)):
                bad = first_mismatch(a, d, w)
                if bad:
                    bad["image"] = i
                    break
            results.append(dict(case=k["name"], entry=entry, ok=bad is None, mismatch=bad, launches=launches))
            del keep
        return results

    def _row_tiles(self, k, frame, ref, cs):
        """the frame cut into k["tiles"] row tiles, each its own allocation whose top / bottom border rows hold garbage where a
        neighbour tile exists: the kernel must take those halo rows from the neighbours"""
        capi, t, b = self.capi, k["tiles"], k["ib"]
        _, _, host, (r, _) = frame
        h = k["nrows"] // t
        allocs = []
        for j in range(t):
            a = Alloc(self.vpp, h, k["ncols"], k["pix"], b, k["ia"])
            blk = np.array(host[r - b + j * h:r - b + j * h + h + 2 * b])  # same layout as the frame: its rows are the tile's rows
            if j > 0:
                blk[:b] = 0xA5
            if j < t - 1:
                blk[-b:] = 0x5A
            a.put(blk)
            allocs.append(a)
        null = capi.VppbImg()
        d = [a.img.desc for a in allocs]
        ups = (capi.VppbImg * t)(*[d[j - 1] if j > 0 else null for j in range(t)])
        dns = (capi.VppbImg * t)(*[d[j + 1] if j < t - 1 else null for j in range(t)])
        return d, [ref[j * h:(j + 1) * h] for j in range(t)], (ups, dns), allocs


def _load(backend):
    sys.path.insert(0, ROOT)
    import vpp_b200
    from vpp_b200 import capi, ops

    if backend == "emu":
        sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
        import build_emu

        emu = C.CDLL(build_emu.build(asan=os.environ.get("VPPB_EMU_ASAN") == "1"))
        for name, (res, args) in capi.PROTOTYPES.items():
            fn = getattr(emu, name)
            fn.restype, fn.argtypes = res, args
        capi.lib = ops.lib = emu
        return vpp_b200, 2  # the emulator's cudaDevAttrMultiProcessorCount
    import torch

    capi.check(capi.lib.vppb_init(0))
    return vpp_b200, torch.cuda.get_device_properties(0).multi_processor_count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=("gpu", "emu"), required=True)
    ap.add_argument("--big", action="store_true", help="add the frames around the 96 MiB rule and u8 (40, 7680) x 128")
    args = ap.parse_args()
    vpp, sms = _load(args.backend)
    env = {k: os.environ[k] for k in KNOBS if k in os.environ}
    run = Runner(vpp, sms, env)
    results = []
    for k in cases(big=args.big):
        results.extend(run.run_case(k))
    print(json.dumps(dict(backend=args.backend, sms=sms, env=env, results=results)))


def run_child(backend, policy, big=False, env=None, timeout=1200):
    """run the table in a child process under POLICIES[policy]: (returncode, parsed JSON or None, stderr)"""
    e = {k: v for k, v in (env if env is not None else os.environ).items() if k not in KNOBS}
    e.update(POLICIES[policy])
    cmd = [sys.executable, "-m", "tests.box_geometry", "--backend", backend] + (["--big"] if big else [])
    r = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=timeout)
    try:
        res = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    except (ValueError, IndexError):
        res = None
    return r.returncode, res, r.stderr


def failures(res):
    return [r for r in res["results"] if not r["ok"]]


if __name__ == "__main__":
    main()
