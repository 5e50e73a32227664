"""video_extruder_init / video_extruder_update (reference: vpp/algorithms/video_extruder.hh:10-45,
video_extruder/video_extruder.hpp:15-135): per-frame keypoint tracker = semi-dense flow -> merge ->
FAST score filter -> periodic masked blockwise FAST re-detection -> trajectories.

Host orchestration in Python (the reference's is host C++ over keypoint_container); every pixel operation
goes through a small `ops` backend so the same orchestration runs on the CUDA path (GpuOps below) and, in the
tests, on the oracle.  keypoint_container semantics kept: dead keypoints stay in the container (and keep
taking part in the flow / merge / mask painting) until a detection frame compacts it; move() increments the
age, so a dead keypoint that still receives a flow callback comes back to life (keypoint_container.hpp:136-167)."""
import numpy as np


class Trajectory:  # keypoint_trajectory.hh:11-73
    def __init__(self, start_frame):
        self.start_frame, self.alive, self.history = start_frame, True, []

    def move_to(self, p):
        self.history.insert(0, (float(p[0]), float(p[1])))


class VideoExtruderCtx:
    def __init__(self, nrows, ncols):
        self.nrows, self.ncols = nrows, ncols
        self.pos, self.vel, self.age, self.trajectories = [], [], [], []
        self.frame_id = -1  # video_extruder.hpp:18


def video_extruder_init(nrows, ncols):
    return VideoExtruderCtx(nrows, ncols)


def video_extruder_update(ctx, frame1, frame2, ops, detector_th=10, keypoint_spacing=10, detector_period=5,
                          max_trajectory_length=15, nscales=3, winsize=9, propagation=2):
    """frame1 / frame2: (nrows, ncols) uint8 arrays; `ops` supplies flow / fast_scores / fast_blockwise."""
    ctx.frame_id += 1
    nr, nc, s = ctx.nrows, ctx.ncols, keypoint_spacing
    n = len(ctx.pos)
    # ---- optical flow (:45-56): every container entry takes part, dead or alive
    if n:
        pos, dist, valid = ops.flow(np.asarray(ctx.pos, np.int32).reshape(-1, 2), frame1, frame2, winsize, nscales, propagation, 5)
        for i in range(n):
            if valid[i]:
                p = (int(pos[i][0]), int(pos[i][1]))
                if 0 <= p[0] < nr and 0 <= p[1] < nc:  # move (keypoint_container.hpp:136-149)
                    ctx.vel[i] = (p[0] - ctx.pos[i][0], p[1] - ctx.pos[i][1])
                    ctx.pos[i] = p
                    ctx.age[i] += 1
                else:
                    ctx.age[i] = 0  # remove
    # ---- merge keypoints that fell in the same spacing cell, keeping the older (:59-84)
    idx = {}
    for i in range(n):
        cell = (_cdiv(ctx.pos[i][0], s), _cdiv(ctx.pos[i][1], s))
        j = idx.get(cell, -1)
        if j >= 0:
            other_age = ctx.age[j]
            if other_age < ctx.age[i]:
                ctx.age[j] = 0
                idx[cell] = i
            if other_age > ctx.age[i]:
                ctx.age[i] = 0
        else:
            idx[cell] = i
    # ---- drop keypoints whose FAST score fell under 3 (:87-91)
    if n:
        sc = ops.fast_scores(frame2, detector_th, np.asarray(ctx.pos, np.int32).reshape(-1, 2))
        for i in range(n):
            if sc[i] < 3:
                ctx.age[i] = 0
    # ---- periodic re-detection away from the existing keypoints (:94-119)
    if ctx.frame_id % detector_period == 0:
        mask = np.ones((nr + 2 * s, nc + 2 * s), np.uint8)  # value 1 => only darker arcs pass (fast.hpp:310-317)
        for (r, c) in ctx.pos:
            mask[r:r + 2 * s, c:c + 2 * s] = 0  # rows r-s .. r+s-1 in border coordinates
        kps = ops.fast_blockwise(frame2, detector_th, s, mask[s:s + nr, s:s + nc])
        for kp in kps:
            ctx.pos.append((int(kp[0]), int(kp[1])))
            ctx.vel.append((0, 0))
            ctx.age.append(1)
        # compact() + sync_attributes(trajectories, keypoint_trajectory(frame_id)) (keypoint_container.hpp:22-110)
        keep = [i for i in range(len(ctx.pos)) if ctx.age[i] > 0]
        traj = []
        for i in keep:
            traj.append(ctx.trajectories[i] if i < len(ctx.trajectories) else Trajectory(ctx.frame_id))
        ctx.pos, ctx.vel, ctx.age = [ctx.pos[i] for i in keep], [ctx.vel[i] for i in keep], [ctx.age[i] for i in keep]
        ctx.trajectories = traj
    # ---- trajectories (:122-133)
    for i in range(len(ctx.pos)):
        if ctx.age[i] > 0:
            ctx.trajectories[i].move_to(ctx.pos[i])
            if len(ctx.trajectories[i].history) > max_trajectory_length:
                ctx.trajectories[i].history.pop()
        else:
            ctx.trajectories[i].alive = False
    return ctx


def _cdiv(a, b):
    """C++ integer division (truncation toward zero); positions are never negative here."""
    return int(a / b) if a < 0 else a // b


def state_table(ctx):
    """(n, 6) int array: row, col, age, trajectory start frame, trajectory length, trajectory alive."""
    return np.array([[p[0], p[1], a, t.start_frame, len(t.history), int(t.alive)] for p, a, t in zip(ctx.pos, ctx.age, ctx.trajectories)],
                    dtype=np.int32).reshape(-1, 6)


class GpuOps:
    """The CUDA path (through vpp_b200.ops / the C-ABI)."""

    def __init__(self):
        from . import ops as _ops
        from .image import Image2d
        self.o, self.Image2d = _ops, Image2d

    def _img(self, frame, border=0):
        im = self.Image2d.from_host(frame, "u8", border=border)
        if border:
            self.o.fill_border_mirror(im)
        return im

    def flow(self, kps, f1, f2, winsize, nscales, propagation, patchsize):
        return self.o.semi_dense_optical_flow(kps, self._img(f1), self._img(f2), winsize=winsize, nscales=nscales, min_scale=0,
                                              propagation=propagation, patchsize=patchsize)

    def fast_scores(self, frame, th, pts):
        return self.o.fast9_scores(self._img(frame, 3), th, pts)

    def fast_blockwise(self, frame, th, block_size, mask):
        return self.o.fast9(self._img(frame, 3), th, blockwise=True, block_size=block_size, mask=self.Image2d.from_host(mask, "u8"))


# ---- the same loop with the container in HBM (SURVEY 8f N3) -------------------------------------------------------------------
class DeviceVideoExtruderCtx:
    """video_extruder_ctx whose keypoint_container and trajectories live on the GPU (vppb_kpc_*): a frame costs no host round
    trip of keypoints, flows, scores or masks; only the 4-byte entry count is read back on detection frames."""

    def __init__(self, nrows, ncols, capacity=None, max_trajectory_length=15):
        import ctypes as C

        from . import capi

        self.nrows, self.ncols, self.frame_id = nrows, ncols, -1
        self.capacity = capacity or max(1024, (nrows * ncols) // 16)
        self.max_traj = max_trajectory_length
        self.handle = C.c_void_p()
        capi.check(capi.lib.vppb_kpc_create(self.capacity, max_trajectory_length, C.byref(self.handle)))
        self._bufs = None

    def __del__(self):
        try:
            from . import capi
            capi.lib.vppb_kpc_destroy(self.handle)
        except Exception:
            pass


def video_extruder_update_device(ctx, frame1, frame2, detector_th=10, keypoint_spacing=10, detector_period=5, nscales=3, winsize=9, propagation=2,
                                 stream=None):
    """video_extruder_update (video_extruder.hpp:24-135) on a DeviceVideoExtruderCtx.  frame1 / frame2: (nrows, ncols) uint8 arrays
    or u8 Image2d (any border); max_trajectory_length is the one the context was created with."""
    import ctypes as C

    from . import capi, ops
    from .image import Image2d

    lib, check = capi.lib, capi.check
    ctx.frame_id += 1
    nr, nc, s = ctx.nrows, ctx.ncols, keypoint_spacing
    f1 = frame1 if isinstance(frame1, Image2d) else Image2d.from_host(frame1, "u8")
    f2 = frame2 if isinstance(frame2, Image2d) else Image2d.from_host(frame2, "u8")
    if ctx._bufs is None:
        P = capi.VppbSdofParams(winsize, nscales, 0, propagation, 5)
        ctx._bufs = {"P": P, "ws": ops._DeviceBuffer(lib.vppb_sdof_workspace_bytes(nr, nc, C.byref(P))), "pos": ops._DeviceBuffer(ctx.capacity * 8),
                     "dist": ops._DeviceBuffer(ctx.capacity * 4), "valid": ops._DeviceBuffer(ctx.capacity),
                     "p1": ops.Pyramid2d((nr, nc), nscales, 2, pixel="u8", border=2 * winsize), "p2": ops.Pyramid2d((nr, nc), nscales, 2, pixel="u8", border=2 * winsize),
                     "g2": Image2d(nr, nc, "u8", border=3), "mask": Image2d(nr, nc, "u8", border=s), "det": ops._DeviceBuffer(ctx.capacity * 8),
                     "cnt": ops._DeviceBuffer(4), "fws": ops._DeviceBuffer(lib.vppb_fast9_workspace_bytes(nr, nc, s)), "table": ops._DeviceBuffer(ctx.capacity * 24)}
    b = ctx._bufs
    n = lib.vppb_kpc_size(ctx.handle)
    if n:  # optical flow of every entry, dead or alive (:45-56)
        b["p1"].update(f1, stream); b["p2"].update(f2, stream)
        check(lib.vppb_sdof_u8(b["p1"].desc_array(), b["p2"].desc_array(), C.byref(b["P"]), lib.vppb_kpc_positions(ctx.handle), n, b["ws"].ptr, b["ws"].nbytes,
                               b["pos"].ptr, b["dist"].ptr, b["valid"].ptr, stream))
        check(lib.vppb_kpc_flow_update(ctx.handle, b["pos"].ptr, b["valid"].ptr, nr, nc, stream))
    check(lib.vppb_kpc_merge(ctx.handle, nr, nc, s, stream))
    check(lib.vppb_copy2d_mirror(f2.ptr(), b["g2"].ptr(), stream))  # frame2 with a mirror border of 3 for the ring reads
    check(lib.vppb_kpc_score_filter(ctx.handle, b["g2"].ptr(), detector_th, 3, stream))
    if ctx.frame_id % detector_period == 0:
        check(lib.vppb_kpc_paint_mask(ctx.handle, b["mask"].ptr(), s, stream))
        check(lib.vppb_fast9_u8_async(b["g2"].ptr(), detector_th, b["mask"].ptr(), capi.FAST_BLOCKWISE, s, capi.FAST_REFERENCE_RING, b["fws"].ptr, b["fws"].nbytes,
                                      b["det"].ptr, None, ctx.capacity, b["cnt"].ptr, stream))
        check(lib.vppb_kpc_add_and_compact(ctx.handle, b["det"].ptr, b["cnt"].ptr, ctx.capacity, ctx.frame_id, stream))
    check(lib.vppb_kpc_trajectories_update(ctx.handle, stream))
    return ctx


def device_state_table(ctx, stream=None):
    """(n, 6) int array like state_table(): row, col, age, trajectory start frame, trajectory length, trajectory alive."""
    from . import capi

    n = capi.lib.vppb_kpc_size(ctx.handle)
    if n == 0 or ctx._bufs is None:
        return np.zeros((0, 6), dtype=np.int32)
    capi.check(capi.lib.vppb_kpc_state_table(ctx.handle, ctx._bufs["table"].ptr, stream))
    return ctx._bufs["table"].to_host(np.int32, n * 6, stream).reshape(-1, 6)


def device_trajectories(ctx, stream=None):
    """(vel, hist): (n, 2) int velocities and (n, max_trajectory_length, 2) float trajectory points (row, col), newest first,
    NaN past each trajectory's length - the histories trajectories() of the host context holds."""
    from . import capi
    from .ops import _DeviceBuffer

    n = capi.lib.vppb_kpc_size(ctx.handle)
    if n == 0:
        return np.zeros((0, 2), np.int32), np.zeros((0, ctx.max_traj, 2), np.float32)
    vel, hist = _DeviceBuffer(n * 8), _DeviceBuffer(n * ctx.max_traj * 8)
    capi.check(capi.lib.vppb_kpc_history(ctx.handle, vel.ptr, hist.ptr, stream))
    return vel.to_host(np.int32, n * 2, stream).reshape(n, 2), hist.to_host(np.float32, n * ctx.max_traj * 2, stream).reshape(n, ctx.max_traj, 2)


def trajectories(ctx, max_trajectory_length):
    """(vel, hist) of a host context in the layout of device_trajectories()."""
    n = len(ctx.pos)
    hist = np.full((n, max_trajectory_length, 2), np.nan, np.float32)
    for i, t in enumerate(ctx.trajectories):
        if t.history:
            hist[i, :len(t.history)] = t.history
    return np.asarray(ctx.vel, np.int32).reshape(n, 2), hist
