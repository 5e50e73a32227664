"""The device keypoint container (vppb_kpc_*, vpp_b200/csrc/kpc.cu) on the GPU: the case table of tests/kpc_cases.py step by step
against its model, with the counts past the launch caps computed from this GPU's SM count; and video_extruder_update_device against
the host orchestration video_extruder_update(GpuOps()) at 1080p and 2160p, frame by frame, tables, velocities and trajectories."""
import numpy as np
import pytest

from tests import kpc_cases as kc
from tests import scenes


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c["id"] for c in kc.cases(1)])
def test_case_table(gpu, cid):
    import torch

    # the library's launch caps come from the SM count of device 0, so the counts past them are computed here, not at collection
    case = {c["id"]: c for c in kc.cases(torch.cuda.get_device_properties(0).multi_processor_count)}[cid]
    ev = kc.run_case(case, host_memory=False)
    if case["n"] > 1024:
        assert ev["max_n"] > 1024
    if case["id"].startswith("traj"):
        assert ev["wrapped"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("cid,steps", kc.edge_cases(), ids=[c[0] for c in kc.edge_cases()])
def test_capacity_and_caller_detections(gpu, cid, steps):
    m = kc.run_edge_case(steps, host_memory=False)
    assert not (m.pos == kc.SENTINEL).all(1).any()


@pytest.mark.gpu
def test_rejected_calls_leave_the_state(gpu):
    kc.check_rejected_calls(host_memory=False)


def eventful_frames(nr, nc, nf, seed):
    """the sequence of tests/golden/make_video_extruder_fixture.py scaled to the frame: a scene translating by (-3, 2) pixels a
    frame, a flat occluder from frame 3 (corners under it fade) and a mirrored patch from frame 5 (the flow goes astray there)"""
    m = 3 * nf + 8
    base = scenes.rectangles_scene(nr + 2 * m, nc + 2 * m, seed=seed, noise=2)
    r = np.random.default_rng(seed)
    out = []
    for f in range(nf):
        a = base[m - 3 * f:m - 3 * f + nr, m + 2 * f:m + 2 * f + nc].astype(np.int32) + r.integers(-1, 2, (nr, nc))
        a = np.clip(a, 0, 255).astype(np.uint8)
        if f >= 3:
            a[nr * 20 // 121:nr * 70 // 121, nc * 30 // 161:nc * 110 // 161] = 128
        if f >= 5:
            a[nr * 80 // 121:, :nc * 60 // 161] = a[nr * 80 // 121:, :nc * 60 // 161][:, ::-1]
        out.append(a)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("nr,nc", [(1080, 1920), (2160, 3840)], ids=["1080p", "2160p"])
def test_video_extruder_device_equals_host_orchestration(gpu, nr, nc):
    from vpp_b200 import video_extruder as ve

    T, period = 5, 3
    frames = eventful_frames(nr, nc, 10, seed=nr + 77)
    kw = dict(detector_th=5, keypoint_spacing=10, detector_period=period, nscales=3, winsize=9, propagation=2)
    d, g = ve.DeviceVideoExtruderCtx(nr, nc, max_trajectory_length=T), ve.video_extruder_init(nr, nc)
    gops = ve.GpuOps()
    ev = dict(max_n=0, dead=0, dropped=0, kept_with_history=0)
    prev_n = 0
    for f in range(1, len(frames)):
        ve.video_extruder_update_device(d, frames[f - 1], frames[f], **kw)
        ve.video_extruder_update(g, frames[f - 1], frames[f], gops, max_trajectory_length=T, **kw)
        tab = ve.device_state_table(d)
        assert np.array_equal(tab, ve.state_table(g)), "frame %d: tables" % f
        vel, hist = ve.device_trajectories(d)
        gvel, ghist = ve.trajectories(g, T)
        assert np.array_equal(vel, gvel), "frame %d: velocities" % f
        assert np.array_equal(hist, ghist, equal_nan=True), "frame %d: trajectories" % f
        fid = d.frame_id
        ev["max_n"] = max(ev["max_n"], len(tab))
        ev["dead"] += int((tab[:, 2] == 0).sum())
        if fid % period == 0 and fid > 0:  # a compaction: what came before either left or kept its trajectory
            carried = tab[tab[:, 3] < fid]
            ev["dropped"] += prev_n - len(carried)
            ev["kept_with_history"] += int((carried[:, 4] > 1).sum())
        prev_n = len(tab)
    assert ev["max_n"] > 1024 and all(ev.values()), ev
