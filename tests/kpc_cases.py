"""Shared by the keypoint container tests: a per-step model of the container behind video_extruder_update_device, the case table,
and a driver that runs a case on the vppb_kpc_* entries one step at a time and compares every step with the model.

The model is a plain transcription of video_extruder.hpp:45-133 (keypoint_container.hpp:22-200, keypoint_trajectory.hh:11-73),
one method per vppb_kpc_* entry, plus the two rules the C-ABI adds where the reference has undefined behaviour: an entry outside
the frame is skipped the way fast9_scores skips an out-of-frame keypoint (the merge and the score filter remove it, the mask gets
nothing painted for it), and add_and_compact appends the first min(count, max_detections, capacity - size) detections.
check_model_against_orchestration() pins the model to vpp_b200.video_extruder.video_extruder_update, which the parity tests pin to
the reference."""
import ctypes as C

import numpy as np

from tests import oracle as orc

def in_frame(p, nr, nc):
    return 0 <= p[0] < nr and 0 <= p[1] < nc


def _cdiv(a, b):
    return int(a / b) if a < 0 else a // b


class Model:
    def __init__(self, capacity, max_traj):
        self.capacity, self.T = capacity, max_traj
        self.pos = np.zeros((0, 2), np.int64)
        self.vel = np.zeros((0, 2), np.int64)
        self.age = np.zeros(0, np.int64)
        self.tstart = np.zeros(0, np.int64)
        self.talive = np.zeros(0, np.int64)
        self.hist = np.zeros((0, max_traj, 2), np.float32)  # newest first, NaN past the length
        self.tlen = np.zeros(0, np.int64)

    @property
    def n(self):
        return len(self.pos)

    def flow(self, newpos, valid, nr, nc):  # :45-56, keypoint_container.hpp:136-167 (entries are independent: vectorised)
        newpos, valid = np.asarray(newpos, np.int64), np.asarray(valid).astype(bool)
        inside = (newpos[:, 0] >= 0) & (newpos[:, 0] < nr) & (newpos[:, 1] >= 0) & (newpos[:, 1] < nc)
        move = valid & inside
        self.vel[move] = newpos[move] - self.pos[move]
        self.pos[move] = newpos[move]
        self.age[move] += 1
        self.age[valid & ~inside] = 0

    def merge(self, nr, nc, s):  # :59-84, serial
        idx, age = {}, self.age
        for i in range(self.n):
            p = self.pos[i]
            if not in_frame(p, nr, nc):
                age[i] = 0
                continue
            cell = (_cdiv(int(p[0]), s), _cdiv(int(p[1]), s))
            j = idx.get(cell, -1)
            if j >= 0:
                other = age[j]
                if other < age[i]:
                    age[j] = 0
                    idx[cell] = i
                if other > age[i]:
                    age[i] = 0
            else:
                idx[cell] = i

    def score_filter(self, scores, min_score):  # :87-91; scores from fast9_scores() (0 outside the frame)
        self.age[np.asarray(scores) < min_score] = 0

    def paint(self, nr, nc, s):  # :97-109: (nr + 2s, nc + 2s) mask, border included
        mask = np.ones((nr + 2 * s, nc + 2 * s), np.uint8)
        for r, c in self.pos:
            if in_frame((r, c), nr, nc):
                mask[r:r + 2 * s, c:c + 2 * s] = 0
        return mask

    def add_and_compact(self, det, count, max_detections, frame_id):  # :111-118, keypoint_container.hpp:22-110
        m = max(0, min(count, max_detections, self.capacity - self.n))
        d = np.asarray(det, np.int64).reshape(-1, 2)[:m]
        self.pos = np.concatenate([self.pos, d])
        self.vel = np.concatenate([self.vel, np.zeros((m, 2), np.int64)])
        self.age = np.concatenate([self.age, np.ones(m, np.int64)])
        self.tstart = np.concatenate([self.tstart, np.full(m, frame_id, np.int64)])
        self.talive = np.concatenate([self.talive, np.ones(m, np.int64)])
        self.tlen = np.concatenate([self.tlen, np.zeros(m, np.int64)])
        self.hist = np.concatenate([self.hist, np.full((m, self.T, 2), np.nan, np.float32)])
        keep = self.age > 0
        for a in ("pos", "vel", "age", "tstart", "talive", "tlen", "hist"):
            setattr(self, a, getattr(self, a)[keep])

    def trajectories(self):  # :122-133: move_to pushes the newest in front and the oldest beyond T drops out
        alive = self.age > 0
        h = self.hist[alive]
        h[:, 1:] = h[:, :-1].copy()
        h[:, 0] = self.pos[alive]
        self.hist[alive] = h
        self.tlen[alive] = np.minimum(self.tlen[alive] + 1, self.T)
        self.talive[~alive] = 0

    def table(self):
        return np.column_stack([self.pos, self.age, self.tstart, self.tlen, self.talive]).astype(np.int32).reshape(-1, 6)


def oracle_scores(frame, th, pos):
    """fast9_score of every position on a mirror-bordered copy of frame (vo_fast9_score), 0 outside the frame"""
    nr, nc = frame.shape
    h = orc.HostImage(nr, nc, "u8", border=3, data=frame, fill_border="mirror")
    o = orc.load()
    return np.array([o.vo_fast9_score(h.ptr(), th, int(r), int(c)) if in_frame((r, c), nr, nc) else 0 for r, c in pos], np.int64)


# ---- the model against the host orchestration --------------------------------------------------------------------------------
class ScriptedOps:
    """video_extruder_update's ops backend returning predetermined flows, scores and detections; records the masks it is given"""

    def __init__(self, script):
        self.script, self.masks = script, []

    def flow(self, kps, f1, f2, winsize, nscales, propagation, patchsize):
        newpos, valid = self.script["flow"].pop(0)
        assert len(newpos) == len(kps)
        return newpos, np.zeros(len(kps), np.int32), valid

    def fast_scores(self, frame, th, pts):
        sc = self.script["scores"].pop(0)
        assert len(sc) == len(pts)
        return sc

    def fast_blockwise(self, frame, th, block_size, mask):
        self.masks.append(np.array(mask))
        return self.script["det"].pop(0)


def check_model_against_orchestration(seed=5, nr=60, nc=80, nframes=9, s=6, period=3, T=3):
    """video_extruder_update driven by scripted ops, and the model driven by the same script, give equal tables, velocities,
    histories and masks on every frame"""
    from vpp_b200 import video_extruder as ve

    rng = np.random.default_rng(seed)
    ctx, m = ve.video_extruder_init(nr, nc), Model(10 ** 9, T)
    frame = np.zeros((nr, nc), np.uint8)
    events = dict(dead=0, merged=0, scored=0, dropped=0)
    for f in range(nframes):
        n = len(ctx.pos)
        pos = np.asarray(ctx.pos, np.int64).reshape(-1, 2)
        newpos = pos + rng.integers(-3, 4, (n, 2))
        newpos[rng.random(n) < 0.1] = (-1, nc)  # leaves the frame: removed
        valid = (rng.random(n) < 0.85).astype(np.uint8)
        script = dict(flow=[(newpos.astype(np.int32), valid)] if n else [], scores=[], det=[])
        ops = ScriptedOps(script)
        if n:
            m.flow(newpos, valid, nr, nc)
        before = m.age.copy()
        m.merge(nr, nc, s)
        events["merged"] += int(((before > 0) & (m.age == 0)).sum())
        scores = rng.integers(0, 6, n)
        script["scores"].append(scores)
        before = m.age.copy()
        if n:
            m.score_filter(scores, 3)
        events["scored"] += int(((before > 0) & (m.age == 0)).sum())
        if f % period == 0:
            mask = m.paint(nr, nc, s)
            det = np.stack([rng.integers(0, nr, 40), rng.integers(0, nc, 40)], 1).astype(np.int32)
            script["det"].append(det)
            events["dropped"] += int((m.age == 0).sum())
            m.add_and_compact(det, len(det), len(det), f)
        m.trajectories()
        ve.video_extruder_update(ctx, frame, frame, ops, keypoint_spacing=s, detector_period=period, max_trajectory_length=T)
        if f % period == 0:
            assert np.array_equal(ops.masks[-1], mask[s:s + nr, s:s + nc]), f
        assert np.array_equal(m.table(), ve.state_table(ctx)), f
        vel, hist = ve.trajectories(ctx, T)
        assert np.array_equal(m.vel, vel) and np.array_equal(m.hist, hist, equal_nan=True), f
        events["dead"] += int((m.age == 0).sum())
    assert all(events.values()), events
    return events


# ---- the case table ------------------------------------------------------------------------------------------------------------
def test_image(nr, nc, seed):
    """flat blocks (FAST score 0: the filter removes their entries) next to noisy ones (entries survive)"""
    r = np.random.default_rng(seed)
    blocks = r.integers(0, 256, (nr // 8 + 1, nc // 8 + 1))
    img = np.kron(blocks, np.ones((8, 8), np.int64))[:nr, :nc]
    noisy = np.kron(r.random((nr // 8 + 1, nc // 8 + 1)) < 0.5, np.ones((8, 8), bool))[:nr, :nc]
    img = np.where(noisy, r.integers(0, 256, (nr, nc)), img)
    return img.astype(np.uint8)


def positions(rng, n, nr, nc, layout="uniform"):
    if layout == "uniform":
        return np.stack([rng.integers(0, nr, n), rng.integers(0, nc, n)], 1).astype(np.int32)
    if layout == "edges":  # every entry on a frame edge, corners included
        side = rng.integers(0, 4, n)
        r, c = rng.integers(0, nr, n), rng.integers(0, nc, n)
        r = np.where(side == 0, 0, np.where(side == 1, nr - 1, r))
        c = np.where(side == 2, 0, np.where(side == 3, nc - 1, c))
        p = np.stack([r, c], 1)
        p[:4] = [(0, 0), (0, nc - 1), (nr - 1, 0), (nr - 1, nc - 1)][:min(4, n)]
        return p.astype(np.int32)
    assert layout == "crowded"  # a few cells of spacing 32 hold 100+ entries each
    cells = np.array([(1, 1), (2, 3), (0, 0)])
    k = cells[rng.integers(0, len(cells), n)]
    return (k * 32 + rng.integers(0, 32, (n, 2))).clip(0, [nr - 1, nc - 1]).astype(np.int32)


def case(cid, n, nr=96, nc=128, s=10, T=3, frames=3, layout="uniform", capacity=None, seed=None, spacings=None, period=2):
    """frame 0 adds n detections; then frames 1..frames-1 run flow, merge, score filter, every `period` frames paint + add, and the
    trajectory update"""
    return dict(id=cid, n=n, nr=nr, nc=nc, s=s, T=T, frames=frames, layout=layout, capacity=capacity or 2 * n + 64,
                seed=seed if seed is not None else n + 7 * nr + s, spacings=spacings or [s], period=period)


def cases(sms):
    """grid_for caps a k_kpc_* grid at sms * 16 CTAs of 256 threads, k_kpc_paint at sms * 16 * 8 warps"""
    grid_cap, paint_cap = sms * 16 * 256, sms * 16 * 8
    t = [case("n%d" % n, n) for n in (0, 1, 32, 33, 1023, 1024, 1025)]
    t += [case("n2049", 2049, nr=128, nc=160, s=3),
          case("past-paint-cap", paint_cap + 1, nr=200, nc=256, s=3, frames=2, period=1),
          case("past-grid-cap", grid_cap + 1, nr=max(256, int((grid_cap + 1) ** 0.5)), nc=max(256, int((grid_cap + 1) ** 0.5)), s=1, frames=2, period=1),
          case("crowded", 600, s=32, frames=5, layout="crowded"),
          case("edges", 300, nr=50, nc=70, layout="edges", frames=4),
          case("spacing1", 700, s=1), case("spacing3", 700, s=3), case("spacing32", 700, s=32),
          case("regrow-10-then-1", 900, spacings=[10, 1]),
          case("traj1", 120, T=1, frames=5, period=3), case("traj2", 120, T=2, frames=6, period=4),
          case("traj15", 150, T=15, frames=19, period=7)]
    return t


# capacity edges and caller detections: (id, steps) with steps run on a fresh container of capacity 64, frame 40 x 50, T 3.
# ("add", detections, count, max_detections): detections = buffer rows the caller owns, beyond max_detections sentinel rows
# that must never be read (an exact-size buffer holds only the first max_detections rows)
SENTINEL = (7777, 7777)


def edge_cases():
    rng = np.random.default_rng(99)

    def dets(k):
        return positions(rng, k, 40, 50)

    def padded(k, total):
        d = np.full((total, 2), SENTINEL, np.int32)
        d[:k] = dets(k)
        return d

    outside = np.array([(-1, 5), (5, -1), (40, 10), (10, 50), (-3, -3), (43, 53), (0, 0), (39, 49), (-30, 20), (20, 80)], np.int32)
    return [
        ("exactly-full", [("add", dets(64), 64, 64), ("traj",), ("add", dets(5), 5, 5)]),
        ("one-over", [("add", dets(65), 65, 65), ("traj",)]),
        ("count-over-max-detections", [("add", padded(4, 100), 100, 4), ("traj",)]),
        ("max-detections-0", [("add", dets(10), 10, 10), ("add", padded(0, 8), 5, 0), ("traj",)]),
        ("negative-count", [("add", dets(20), 20, 20), ("add", padded(0, 4), -3, 4), ("traj",)]),
        ("full-then-partial", [("add", dets(60), 60, 60), ("add", dets(10), 10, 10), ("traj",)]),
        ("outside-frame", [("add", outside, len(outside), len(outside)), ("traj",), ("flow",), ("merge",), ("score",), ("paint",),
                           ("traj",), ("add", outside[:3], 3, 3), ("merge",), ("paint",), ("traj",)]),
    ]


# ---- the driver ----------------------------------------------------------------------------------------------------------------
_LIBC = []


def _libc():
    if not _LIBC:
        libc = C.CDLL(None)
        libc.malloc.restype, libc.malloc.argtypes = C.c_void_p, [C.c_size_t]
        libc.free.argtypes = [C.c_void_p]
        _LIBC.append(libc)
    return _LIBC[0]


class Driver:
    """One vppb_kpc container on capi.lib (the GPU library, or the emulated one swapped in).  host_memory: the emulator, whose
    kernels read host memory: inputs and outputs are malloc'ed buffers of exactly their size (AddressSanitizer sees any overrun)."""

    def __init__(self, capacity, T, host_memory):
        from vpp_b200 import capi

        self.capi, self.lib, self.host = capi, capi.lib, host_memory
        self.h = C.c_void_p()
        capi.check(self.lib.vppb_kpc_create(capacity, T, C.byref(self.h)))
        self.model, self.T, self.keep, self.mallocs = Model(capacity, T), T, [], []

    def close(self):
        self.lib.vppb_kpc_destroy(self.h)
        for p in self.mallocs:
            _libc().free(p)
        self.mallocs = []

    def _malloc(self, nbytes):
        p = _libc().malloc(nbytes)
        assert p
        self.mallocs.append(p)
        return p

    def dev(self, arr):
        """device copy of arr (None: a NULL pointer)"""
        if arr is None:
            return None
        a = np.ascontiguousarray(arr)
        if self.host:
            if a.nbytes == 0:
                return None
            p = self._malloc(a.nbytes)
            C.memmove(p, a.ctypes.data, a.nbytes)
            return p
        from vpp_b200.ops import _DeviceBuffer

        b = _DeviceBuffer(a.nbytes).from_host(a)
        self.keep.append(b)
        return b.ptr

    def _out(self, nbytes, dtype):
        if self.host:
            p = self._malloc(nbytes)
            return p, lambda: np.ctypeslib.as_array((C.c_ubyte * nbytes).from_address(p)).view(dtype).copy()
        from vpp_b200.ops import _DeviceBuffer

        b = _DeviceBuffer(nbytes)
        return b.ptr, lambda: b.to_host(dtype, nbytes // np.dtype(dtype).itemsize)

    def state(self):
        n = self.lib.vppb_kpc_size(self.h)
        if n == 0:
            return n, np.zeros((0, 6), np.int32), np.zeros((0, 2), np.int32), np.zeros((0, self.T, 2), np.float32)
        tp, tget = self._out(n * 24, np.int32)
        vp, vget = self._out(n * 8, np.int32)
        hp, hget = self._out(n * self.T * 8, np.float32)
        self.capi.check(self.lib.vppb_kpc_state_table(self.h, tp, None))
        self.capi.check(self.lib.vppb_kpc_history(self.h, vp, hp, None))
        self.capi.check(self.lib.vppb_sync(None))
        return n, tget().reshape(-1, 6), vget().reshape(-1, 2), hget().reshape(n, self.T, 2)

    def compare(self, what):
        m = self.model
        n, tab, vel, hist = self.state()
        assert n == m.n, (what, n, m.n)
        bad = np.argwhere((tab != m.table()).any(1))[:, 0]
        assert len(bad) == 0, (what, "table rows", bad[:8], tab[bad[:4]], m.table()[bad[:4]])
        assert np.array_equal(vel, m.vel), (what, "velocities")
        assert np.array_equal(hist, m.hist, equal_nan=True), (what, "histories")

    # every step runs the entry and the model, then compares
    def add(self, det, count, max_detections, frame_id, exact):
        d = np.asarray(det, np.int32).reshape(-1, 2)
        buf = d[:max_detections] if exact else d
        ptr = self.dev(buf) if len(buf) else (None if exact else self.dev(np.full((1, 2), SENTINEL, np.int32)))
        self.capi.check(self.lib.vppb_kpc_add_and_compact(self.h, ptr, self.dev(np.array([count], np.int32)), max_detections, frame_id, None))
        self.model.add_and_compact(d, count, max_detections, frame_id)
        self.compare("add_and_compact")

    def flow(self, newpos, valid, nr, nc):
        self.capi.check(self.lib.vppb_kpc_flow_update(self.h, self.dev(np.asarray(newpos, np.int32)), self.dev(np.asarray(valid, np.uint8)), nr, nc, None))
        self.model.flow(newpos, valid, nr, nc)
        self.compare("flow_update")

    def merge(self, nr, nc, s):
        self.capi.check(self.lib.vppb_kpc_merge(self.h, nr, nc, s, None))
        self.model.merge(nr, nc, s)
        self.compare("merge s=%d" % s)

    def score(self, frame, th):
        from vpp_b200.image import Image2d

        nr, nc = frame.shape
        host = orc.HostImage(nr, nc, "u8", border=3, data=frame, fill_border="mirror")
        g = Image2d(nr, nc, "u8", border=3)
        g.upload(host.get(with_border=True), with_border=True)
        self.capi.check(self.lib.vppb_kpc_score_filter(self.h, g.ptr(), th, 3, None))
        self.model.score_filter(oracle_scores(frame, th, self.model.pos), 3)
        self.compare("score_filter")

    def paint(self, nr, nc, s):
        from vpp_b200.image import Image2d

        mask = Image2d(nr, nc, "u8", border=s)
        mask.upload(np.full((nr + 2 * s, nc + 2 * s), 9, np.uint8), with_border=True)
        self.capi.check(self.lib.vppb_kpc_paint_mask(self.h, mask.ptr(), s, None))
        got = mask.download(with_border=True)
        want = self.model.paint(nr, nc, s)
        bad = np.argwhere(got != want)
        assert len(bad) == 0, ("paint_mask", bad[:8])
        self.compare("paint_mask")

    def traj(self):
        self.capi.check(self.lib.vppb_kpc_trajectories_update(self.h, None))
        self.model.trajectories()
        self.compare("trajectories_update")


def flow_targets(rng, pos, nr, nc, dead_share=0.08):
    n = len(pos)
    newpos = pos.astype(np.int64) + rng.integers(-4, 5, (n, 2))
    k = np.flatnonzero(rng.random(n) < dead_share)  # some targets leave the frame: valid ones are removed
    newpos[k, 0] = rng.choice([-1, nr, -7], len(k))
    newpos[k, 1] = rng.integers(0, nc, len(k))
    valid = (rng.random(n) < 0.85).astype(np.uint8)
    return newpos.astype(np.int32), valid


def run_case(c, host_memory, exact=False):
    """the standard script of a case (see case()); returns counters of the events it went through"""
    rng = np.random.default_rng(c["seed"])
    nr, nc, T = c["nr"], c["nc"], c["T"]
    d = Driver(c["capacity"], T, host_memory)
    frame = test_image(nr, nc, c["seed"])
    ev = dict(max_n=0, dead=0, removed_by_merge=0, compacted=0, wrapped=0)
    try:
        d.add(positions(rng, c["n"], nr, nc, c["layout"]), c["n"], c["n"], 0, exact)
        d.traj()
        for f in range(1, c["frames"]):
            newpos, valid = flow_targets(rng, d.model.pos, nr, nc)
            if c["layout"] == "crowded":  # keep the crowd together: the ages (and their ties) are what varies
                newpos = np.where((newpos[:, :1] >= 0) & (newpos[:, :1] < nr), d.model.pos, newpos).astype(np.int32)
            d.flow(newpos, valid, nr, nc)
            for s in c["spacings"]:
                before = int((d.model.age > 0).sum())
                d.merge(nr, nc, s)
                ev["removed_by_merge"] += before - int((d.model.age > 0).sum())
            d.score(frame, 10)
            if f % c["period"] == 0:
                d.paint(nr, nc, c["s"])
                ev["dead"] += int((d.model.age == 0).sum())
                k = max(1, c["n"] // 8)
                before = d.model.n
                d.add(positions(rng, k, nr, nc), k, k, f, exact)
                ev["compacted"] += before + k - d.model.n
            d.traj()
            ev["max_n"] = max(ev["max_n"], d.model.n)
            ev["wrapped"] += int((d.model.tlen == T).sum())
        return ev
    finally:
        d.close()


def run_edge_case(steps, host_memory, exact=False):
    nr, nc, s = 40, 50, 10
    d = Driver(64, 3, host_memory)
    frame = test_image(nr, nc, 3)
    rng = np.random.default_rng(4)
    try:
        for f, st in enumerate(steps):
            if st[0] == "add":
                d.add(st[1], st[2], st[3], f, exact)
            elif st[0] == "traj":
                d.traj()
            elif st[0] == "flow":
                d.flow(*flow_targets(rng, d.model.pos, nr, nc, 0.0), nr, nc)
            elif st[0] == "merge":
                d.merge(nr, nc, s)
            elif st[0] == "score":
                d.score(frame, 10)
            elif st[0] == "paint":
                d.paint(nr, nc, s)
        return d.model
    finally:
        d.close()


def check_rejected_calls(host_memory):
    """calls the entries reject: an error code, and the container (and the mask) as before"""
    from vpp_b200.image import Image2d

    nr, nc = 40, 50
    d = Driver(64, 3, host_memory)
    lib, capi = d.lib, d.capi
    try:
        d.add(positions(np.random.default_rng(1), 30, nr, nc), 30, 30, 0, True)
        d.traj()
        det, cnt = d.dev(positions(np.random.default_rng(2), 8, nr, nc)), d.dev(np.array([8], np.int32))
        thin = Image2d(nr, nc, "u8", border=2)
        mask = Image2d(nr, nc, "u8", border=4)
        mask.upload(np.full((nr + 8, nc + 8), 9, np.uint8), with_border=True)
        rejected = [
            ("add max_detections < 0", lambda: lib.vppb_kpc_add_and_compact(d.h, det, cnt, -1, 1, None), capi.VPPB_E_ARG),
            ("add NULL count", lambda: lib.vppb_kpc_add_and_compact(d.h, det, None, 8, 1, None), capi.VPPB_E_ARG),
            ("add NULL detections", lambda: lib.vppb_kpc_add_and_compact(d.h, None, cnt, 8, 1, None), capi.VPPB_E_ARG),
            ("merge spacing 0", lambda: lib.vppb_kpc_merge(d.h, nr, nc, 0, None), capi.VPPB_E_ARG),
            ("score border 2", lambda: lib.vppb_kpc_score_filter(d.h, thin.ptr(), 10, 3, None), capi.VPPB_E_BORDER),
            ("paint border < spacing", lambda: lib.vppb_kpc_paint_mask(d.h, mask.ptr(), 5, None), capi.VPPB_E_BORDER),
            ("paint spacing 0", lambda: lib.vppb_kpc_paint_mask(d.h, mask.ptr(), 0, None), capi.VPPB_E_ARG),
            ("flow NULL", lambda: lib.vppb_kpc_flow_update(d.h, None, None, nr, nc, None), capi.VPPB_E_ARG),
        ]
        for what, call, code in rejected:
            assert call() == code, what
            capi.check(lib.vppb_sync(None))
            d.compare(what)
            assert (mask.download(with_border=True) == 9).all(), what
    finally:
        d.close()
