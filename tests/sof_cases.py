"""Shared by the sparse optical flow tests: the composite oracle and the case table.

The oracle chains the stage oracles that are pinned to the reference elsewhere: blockwise FAST of the C oracle (vo_fast9_u8, mode 2),
patch extraction (dm_cases.patches), the grid-local SAD matcher (dm_cases.oracle_local), lucas_kanade with a prediction
(oracle_ops.oracle_lucas_kanade), and a numpy SAD for the refinement.  The semantics are those of include/vppb.h / DESIGN §3.9.

A case is a dict: frame size, border, scene, shift of frame 2, options (th, bs, ws, R, s, nscales, it), and `kps` (None: detect on
frame 1, or the name of a caller keypoint set)."""
import ctypes as C

import numpy as np

from tests import dm_cases as dc
from tests import oracle as orc
from tests import oracle_ops
from tests import scenes

INT_MAX = 2 ** 31 - 1
DEFAULTS = dict(th=5, bs=5, ws=11, R=100, s=300, nscales=3, it=5)


def opts(case):
    o = dict(DEFAULTS)
    o.update({k: case[k] for k in DEFAULTS if k in case})
    return o


def _scene(kind, H, W, seed):
    """float image in [0, 1] of the whole frame, border included"""
    if kind == "rect":
        return scenes.rectangles_scene(H, W, seed=seed, nrect=max(8, H * W // 300)).astype(np.float64) / 255.0
    if kind == "noise":
        return scenes.smooth_noise(H, W, seed=seed, sigmas=(1.0, 3.0))
    if kind == "blank":
        return np.full((H, W), 0.5)
    if kind == "flat":  # texture in the left third only: keypoints placed in the flat rest make LK fail (its (0, 0) code)
        a = np.full((H, W), 0.5)
        a[:, :W // 3] = scenes.smooth_noise(H, W // 3, seed=seed, sigmas=(1.0, 3.0))
        return a
    raise ValueError(kind)


def frames(case):
    """(f1, f2): (nr + 2b, nc + 2b) uint8 frames, border included (the caller fills the border: here with scene content).
    frame2(p) = frame1(p - shift); `split` scenes put frame 1's texture in the left half and frame 2's in the right half."""
    nr, nc, b = case["nr"], case["nc"], case["b"]
    H, W = nr + 2 * b, nc + 2 * b
    a = _scene(case["scene"], H, W, case.get("seed", 1))
    dr, dc_ = case.get("shift", (0, 0))
    w = scenes.warp(a, -dr, -dc_)
    f1 = np.clip(np.round(a * 255), 0, 255).astype(np.uint8)
    f2 = np.clip(np.round(w * 255), 0, 255).astype(np.uint8)
    if case.get("split"):
        f1[:, W // 2:] = 128
        f2[:, :W // 2] = 128
    return f1, f2


def keypoints(case):
    """the caller keypoints of a case (int32 (n, 2)), or None to detect on frame 1"""
    name, nr, nc = case.get("kps"), case["nr"], case["nc"]
    if name is None:
        return None
    rng = np.random.default_rng(nr * 131 + nc)
    if name == "edge":  # corners, edges, a few just outside the frame, and interior points
        pts = [[0, 0], [0, nc - 1], [nr - 1, 0], [nr - 1, nc - 1], [1, 2], [nr - 2, nc // 2], [nr // 2, 0], [-1, 3], [4, -2], [nr, 5],
               [7, nc], [-30, -40], [nr + 25, nc + 9]]
        pts += rng.integers(0, [nr, nc], (20, 2)).tolist()
        return np.array(pts, np.int32)
    if name == "flat":  # in the flat two thirds of a "flat" scene
        return np.stack([rng.integers(4, nr - 4, 24), rng.integers(nc // 3 + 8, nc - 4, 24)], 1).astype(np.int32)
    if name == "empty":
        return np.zeros((0, 2), np.int32)
    raise ValueError(name)


# ---- the composite oracle --------------------------------------------------------------------------------------------------------
def oracle_fast_blockwise(frame, b, th, bs, lib=None):
    nr, nc = frame.shape[0] - 2 * b, frame.shape[1] - 2 * b
    o = lib or orc.load()
    h = orc.HostImage(nr, nc, "u8", border=b)
    h.set(frame, with_border=True)
    cap = ((nr + bs - 1) // bs) * ((nc + bs - 1) // bs)
    k = np.zeros((max(cap, 1), 2), np.int32)
    n = o.vo_fast9_u8(h.ptr(), th, None, 2, bs, 0, k.ctypes.data, None, len(k))
    return k[:n].copy()


def oracle_sparse_flow(f1, f2, b, case, subpixelic, lib=None, omp=None):
    """(positions, flow float32, distance, valid) of vppb_sparse_flow_u8 for frames f1 / f2 (border b included)"""
    o = opts(case)
    nr, nc = f1.shape[0] - 2 * b, f1.shape[1] - 2 * b
    ck = keypoints(case)
    K1 = oracle_fast_blockwise(f1, b, o["th"], o["bs"], lib) if ck is None else ck
    K2 = oracle_fast_blockwise(f2, b, o["th"], o["bs"], lib)
    n = len(K1)
    flow = np.zeros((n, 2), np.float32)
    dist = np.full(n, INT_MAX, np.int32)
    valid = np.zeros(n, bool)
    if n == 0:
        return K1, flow, dist, valid
    ws = o["ws"]
    D1, D2 = dc.patches(f1, b, K1, ws), dc.patches(f2, b, K2, ws)
    t, d = dc.oracle_local(D1, D2, K1, K2, o["R"], o["s"], lib=omp)
    inside = (K1[:, 0] >= 0) & (K1[:, 0] < nr) & (K1[:, 1] >= 0) & (K1[:, 1] < nc)
    pred = np.zeros((n, 2), np.float32)
    m = t >= 0
    pred[m] = (K2[t[m]].astype(np.int64) - K1[m].astype(np.int64)).astype(np.float32)
    if not subpixelic:
        valid = m & inside
        flow[valid] = pred[valid]
        dist[valid] = d[valid]
        return K1, flow, dist, valid
    lkf, _ = oracle_ops.oracle_lucas_kanade(f1[b:b + nr, b:b + nc], f2[b:b + nr, b:b + nc], K1.astype(np.float32), niterations=o["it"], winsize=ws,
                                            nscales=o["nscales"], prediction=pred, lib=lib)
    lkf = np.asarray(lkf, np.float32)
    y = K1.astype(np.float32) + lkf  # float32 sum, as on the device
    h = ws // 2
    for i in np.flatnonzero(inside):
        valid[i] = True
        flow[i] = lkf[i]
        win = np.zeros(ws * ws, np.int64)
        if np.isfinite(y[i]).all() and (np.abs(y[i]) < 2.0 ** 30).all():
            r, c = int(y[i, 0]), int(y[i, 1])  # int(): truncation toward zero
            if r - h >= -b and r - h + ws - 1 <= nr - 1 + b and c - h >= -b and c - h + ws - 1 <= nc - 1 + b:
                win = f2[r - h + b:r - h + b + ws, c - h + b:c - h + b + ws].reshape(-1).astype(np.int64)
        dist[i] = int(np.abs(D1[i].astype(np.int64) - win).sum())
    return K1, flow, dist, valid


# ---- the case table --------------------------------------------------------------------------------------------------------------
CASES = [
    dict(id="int-shift", nr=40, nc=50, b=5, scene="rect", shift=(2, -3), th=5, bs=5, ws=11, R=10, s=8),
    dict(id="subpixel-shift", nr=36, nc=44, b=5, scene="noise", shift=(1.4, -0.6), th=5, bs=6, ws=9, R=6, s=5, nscales=2),
    dict(id="defaults", nr=45, nc=40, b=5, scene="noise", shift=(3, 1)),
    dict(id="odd-sizes", nr=37, nc=53, b=4, scene="rect", shift=(-1, 2), th=8, bs=4, ws=7, R=9, s=7, seed=3),
    dict(id="odd-sizes-2", nr=29, nc=41, b=3, scene="noise", shift=(0.5, 0.5), th=5, bs=7, ws=5, R=5, s=3, nscales=2, it=3, seed=4),
    dict(id="no-keypoint", nr=30, nc=34, b=5, scene="blank", shift=(0, 0), ws=9),
    dict(id="no-train-in-window", nr=32, nc=48, b=4, scene="noise", split=True, shift=(0, 0), th=5, bs=4, ws=7, R=3, s=4, seed=5),
    dict(id="window-leaves-border", nr=34, nc=40, b=7, scene="noise", shift=(-4, -4), kps="edge", th=5, bs=5, ws=15, R=8, s=6, nscales=2, seed=6),
    dict(id="lk-flat", nr=32, nc=60, b=5, scene="flat", shift=(0.7, 0.3), kps="flat", th=5, bs=6, ws=9, R=10, s=10, nscales=2, seed=7),
    dict(id="caller-edge", nr=31, nc=45, b=5, scene="rect", shift=(1, 1), kps="edge", th=5, bs=5, ws=11, R=20, s=9, seed=8),
    dict(id="caller-empty", nr=20, nc=24, b=5, scene="noise", shift=(0, 0), kps="empty"),
]


def case_id(c):
    return c["id"]


def params(case, subpixelic):
    from vpp_b200 import capi

    o = opts(case)
    return capi.VppbSofParams(o["th"], o["bs"], o["ws"], o["R"], o["s"], 1 if subpixelic else 0, o["it"], o["nscales"])
