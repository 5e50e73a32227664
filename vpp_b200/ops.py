"""Host-side mirror of the Video++ operator surface for the dense-pixel path (Python flavour).

Same names, argument meaning and error behaviour as the reference templates they cite; all
pixel work happens in the CUDA library behind include/vppb.h.  (The C++14 flavour of the same
surface lives in vpp_b200/include/vpp.)
"""
import ctypes as C

import numpy as np

from . import capi
from .capi import check, lib
from .image import DEFAULT_ALIGNMENT, Image2d


def _val(img, value):
    return np.ascontiguousarray(np.broadcast_to(np.asarray(value, dtype=img.dtype), (img.channels,)))


# ---- pixel_wise named kernels ---------------------------------------------------------------
def pixel_wise_add(a, b, c, stream=None):
    """pixel_wise(A,B,C) | [](int& a,int& b,int& c){ a = b + c; }  (benchmarks/image_add.cc:51-57)"""
    check(lib.vppb_pw_add_i32(a.ptr(), b.ptr(), c.ptr(), stream))


def fill(img, value, stream=None):  # fill.hh:12-15
    v = _val(img, value)
    check(lib.vppb_fill(img.ptr(), v.ctypes.data, 0, stream))


def fill_with_border(img, value, stream=None):  # fill.hh:24-28
    v = _val(img, value)
    check(lib.vppb_fill(img.ptr(), v.ctypes.data, 1, stream))


def fill_border_with_value(img, value, stream=None):  # fill.hh:32-45
    v = _val(img, value)
    check(lib.vppb_fill_border_value(img.ptr(), v.ctypes.data, stream))


def fill_border_mirror(img, stream=None):  # fill.hh:48-83
    check(lib.vppb_fill_border_mirror(img.ptr(), stream))


def fill_border_closest(img, stream=None):  # fill.hh:86-121
    check(lib.vppb_fill_border_closest(img.ptr(), stream))


def copy(src, dst, stream=None):  # copy.hh:10-19
    check(lib.vppb_copy2d(src.ptr(), dst.ptr(), 0, stream))


def copy_with_border(src, dst, stream=None):  # copy.hh:22-27
    check(lib.vppb_copy2d(src.ptr(), dst.ptr(), 1, stream))


def clone(img, border=None, aligned=None):  # clone.hh:10-20
    n = Image2d(img.nrows, img.ncols, img.pixel, border=img.border if border is None else border,
                aligned=(img.alignment or DEFAULT_ALIGNMENT) if aligned is None else aligned)
    copy_with_border(img, n)
    return n


def sum(img, stream=None):  # sum.hh:12-19 (char / uchar / int images; accumulator int)
    out = C.c_int64()
    check(lib.vppb_sum_i32(img.ptr(), 1 if img.pixel in ("i8", "i32") else 0, C.byref(out), stream))
    return out.value


# ---- frame ingest -----------------------------------------------------------------------------
def rgb_to_graylevel(src, dst=None, stream=None):
    """rgb_to_graylevel<unsigned char>(image2d<vuchar3 | vuchar4>) (colorspace_conversions.hh:10-47): (r + g + b) / 3,
    truncating, over domain_with_border; without `dst` the result has the input's border and alignment, as there."""
    if dst is None:
        dst = Image2d(src.nrows, src.ncols, "u8", border=src.border, aligned=src.alignment or DEFAULT_ALIGNMENT)
    check(lib.vppb_rgb_to_graylevel_u8(src.ptr(), dst.ptr(), stream))
    return dst


def ingest_rgb_frame(src, border, dst=None, stream=None):
    """clone(frame, _border = border); fill_border_mirror; rgb_to_graylevel<unsigned char> - what every caller of the
    path does with a decoded frame (examples/video_extruder.cc:46-48) - as ONE launch: gray level of the domain plus
    the mirror border of the result.  `src` may have any border (it is not read)."""
    if dst is None:
        dst = Image2d(src.nrows, src.ncols, "u8", border=border)
    check(lib.vppb_rgb_to_graylevel_u8_mirror(src.ptr(), dst.ptr(), stream))
    return dst


# ---- stencils -------------------------------------------------------------------------------
def box5x5_batch(srcs, dsts, stream=None):
    """box5x5 over a batch of (src, dst) pairs in as few launches as possible (vppb_box5x5_*_batch): one persistent launch per
    128 equally shaped images.  Same results as calling box5x5 pair by pair."""
    assert len(srcs) == len(dsts) and len(srcs) > 0
    n = len(srcs)
    ins, outs = (capi.VppbImg * n)(), (capi.VppbImg * n)()
    for i in range(n):
        ins[i], outs[i] = srcs[i].desc, dsts[i].desc
    fn = {"vuchar3": lib.vppb_box5x5_u8c3_batch, "u8": lib.vppb_box5x5_u8_batch}[srcs[0].pixel]
    check(fn(ins, outs, n, stream))


def box5x5(src, dst, stream=None):
    """pixel_wise(dst, relative_access(src)) | sum of the 5x5 neighbourhood / 25
    (benchmarks/box_5x5_filter2.cc:71-81; vuchar3 form examples/box_filter.cc:23-32)."""
    fn = {"vuchar3": lib.vppb_box5x5_u8c3, "u8": lib.vppb_box5x5_u8, "i32": lib.vppb_box5x5_i32}[src.pixel]
    check(fn(src.ptr(), dst.ptr(), stream))


def scharr(src, dst, stream=None):  # scharr.hh:46-87
    check(lib.vppb_scharr_u8(src.ptr(), dst.ptr(), 1 if dst.pixel == "vfloat2" else 0, stream))


_LP_KIND = {"u8": 0, "vint2": 1, "vfloat2": 2}


class Pyramid2d:
    """pyramid2d<V> (pyramid.hh:126-215): levels of size 1 + n/factor, factor 2 only."""

    def __init__(self, src_or_shape, nlevels, factor=2, pixel=None, border=0, aligned=DEFAULT_ALIGNMENT):
        assert factor == 2, "only the factor-2 path (pyramid.hh:174-182) is built"
        self.factor = float(factor)
        img = src_or_shape if isinstance(src_or_shape, Image2d) else None
        nr, nc = (img.nrows, img.ncols) if img is not None else src_or_shape
        self.pixel = pixel or img.pixel
        self.levels = []
        for _ in range(nlevels):
            self.levels.append(Image2d(nr, nc, self.pixel, border=border, aligned=aligned))
            nr, nc = int(1 + nr / factor), int(1 + nc / factor)  # pyramid.hh:140,154
        if img is not None:
            self.update(img)

    def __getitem__(self, i):
        return self.levels[i]

    def __len__(self):
        return len(self.levels)

    size = __len__

    def propagate_level0(self, stream=None, level0_mirrored=False):  # pyramid.hh:169-192
        if not level0_mirrored:
            fill_border_mirror(self.levels[0], stream)
        for i in range(1, len(self.levels)):
            # low-pass + subsample + mirror border of the new level: one launch
            check(lib.vppb_lowpass_sub2_mirror(self.levels[i - 1].ptr(), self.levels[i].ptr(), _LP_KIND[self.pixel], stream))

    def update(self, img, stream=None):  # pyramid.hh:194-198: copy, mirror, levels
        check(lib.vppb_copy2d_mirror(img.ptr(), self.levels[0].ptr(), stream))
        self.propagate_level0(stream, level0_mirrored=True)

    def update_from_scharr(self, src, stream=None):
        """scharr(src, pyr[0]); pyr.propagate_level0() — the gradient pyramid of lucas_kanade.hpp:156-157 and
        video_extruder.hpp:60-61 — with level 0's mirror border written by the Scharr launch itself."""
        check(lib.vppb_scharr_u8_mirror(src.ptr(), self.levels[0].ptr(), 1 if self.pixel == "vfloat2" else 0, stream))
        self.propagate_level0(stream, level0_mirrored=True)

    def desc_array(self):
        arr = (capi.VppbImg * len(self.levels))()
        for i, l in enumerate(self.levels):
            arr[i] = l.desc
        return arr


# ---- FAST9 ----------------------------------------------------------------------------------
class _DeviceBuffer:
    def __init__(self, nbytes):
        self.img = capi.VppbImg()
        check(lib.vppb_alloc(C.byref(self.img), 1, max(int(nbytes), 1), 1, 0, 256))
        self.nbytes = int(nbytes)

    @property
    def ptr(self):
        return self.img.base

    def to_host(self, dtype, count, stream=None):
        """Copy back on `stream` - the stream the producing kernels were launched on - and wait for it."""
        out = np.empty(count, dtype=dtype)
        if count:
            view = capi.VppbImg()
            C.memmove(C.byref(view), C.byref(self.img), C.sizeof(capi.VppbImg))
            view.ncols = out.nbytes
            check(lib.vppb_download(C.byref(view), out.ctypes.data, out.nbytes, 0, stream))
            check(lib.vppb_sync(stream))
        return out

    def from_host(self, arr, stream=None):
        arr = np.ascontiguousarray(arr)
        if arr.nbytes:
            view = capi.VppbImg()
            C.memmove(C.byref(view), C.byref(self.img), C.sizeof(capi.VppbImg))
            view.ncols = arr.nbytes
            check(lib.vppb_upload(C.byref(view), arr.ctypes.data, arr.nbytes, 0, stream))
            check(lib.vppb_sync(stream))  # the host array may be a temporary
        return self

    def __del__(self):
        try:
            lib.vppb_free(C.byref(self.img))
        except Exception:
            pass


_FAST_CACHE = {}  # (nrows, ncols, block_size) -> workspace; (capacity, with_scores) -> output buffers: allocated once, reused


def _fast_buffers(img, block_size, cap, want_scores):
    key = (img.nrows, img.ncols, block_size)
    ent = _FAST_CACHE.get(key)
    if ent is None:
        if len(_FAST_CACHE) > 8:
            _FAST_CACHE.clear()
        ent = {"ws": _DeviceBuffer(lib.vppb_fast9_workspace_bytes(img.nrows, img.ncols, block_size)), "count": _DeviceBuffer(4), "cap": 0}
        _FAST_CACHE[key] = ent
    if ent["cap"] < cap:
        ent["kps"], ent["sc"], ent["cap"] = _DeviceBuffer(cap * 8), _DeviceBuffer(cap * 4), cap
    return ent


def fast9(img, th, local_maxima=False, blockwise=False, block_size=10, mask=None, scores=None, ring="reference",
          capacity=None, stream=None):
    """std::vector<vint2> fast9(A, th, [_local_maxima | _blockwise, _block_size=, _mask=, _scores=&vec])
    (fast.hpp:931-955).  Returns an (n, 2) int32 array of (row, col) in raster order (blockwise: cell raster order, the
    reference's serial order); if `scores` is a
    list it is replaced by the matching scores.  Raises RuntimeError if A.border() < 3 (fast.hpp:937-938).
    Workspace and output buffers are allocated once per image shape and reused; the device work is queued without a
    host synchronisation (vppb_fast9_u8_async), then the 4-byte count and the keypoints are read back on `stream`."""
    mode = capi.FAST_LOCAL_MAXIMA if local_maxima else (capi.FAST_BLOCKWISE if blockwise else capi.FAST_ALL)
    ring_id = capi.FAST_REFERENCE_RING if ring == "reference" else capi.FAST_TRUE_RING
    cap = capacity if capacity is not None else max(1024, (img.nrows * img.ncols) // 8)
    while True:
        ent = _fast_buffers(img, block_size, cap, scores is not None)
        kps, sc = ent["kps"], ent["sc"] if scores is not None else None
        check(lib.vppb_fast9_u8_async(img.ptr(), th, mask.ptr() if mask is not None else None, mode, block_size, ring_id, ent["ws"].ptr,
                                      ent["ws"].nbytes, kps.ptr, sc.ptr if sc else None, cap, ent["count"].ptr, stream))
        count = int(ent["count"].to_host(np.int32, 1, stream)[0])
        if count > cap:
            if capacity is not None:
                raise capi.VppbError(capi.VPPB_E_CAPACITY, "fast9: %d keypoints exceed the capacity %d" % (count, cap))
            cap = count
            continue
        break
    out = kps.to_host(np.int32, count * 2, stream).reshape(-1, 2)
    if scores is not None:
        scores[:] = list(sc.to_host(np.int32, count, stream))
    return out


def fast9_scores(img, th, keypoints, stream=None):  # fast.hpp:643-652
    kp = np.ascontiguousarray(keypoints, dtype=np.int32).reshape(-1, 2)
    d_kp = _DeviceBuffer(kp.nbytes).from_host(kp, stream)
    d_sc = _DeviceBuffer(len(kp) * 4)
    check(lib.vppb_fast9_scores(img.ptr(), th, d_kp.ptr, len(kp), d_sc.ptr, stream))
    return d_sc.to_host(np.int32, len(kp), stream)


def fast9_blockwise_rank(img, th, block_size=10, max_points_per_block=3, mask=None, scores=None, ring="reference", stream=None):
    """std::vector<vint3> fast_detector9_blockwise_rank(A, th, block_size, max_point_per_block, mask, scores) (fast.hpp:801-886):
    (n, 3) int32 array of (row, col, rank), blocks in raster order; `scores` (a list) receives the raw scores."""
    ring_id = capi.FAST_REFERENCE_RING if ring == "reference" else capi.FAST_TRUE_RING
    cells = ((img.nrows + block_size - 1) // block_size) * ((img.ncols + block_size - 1) // block_size)
    cap = max(1, cells * max_points_per_block)
    ws = _DeviceBuffer(lib.vppb_fast9_rank_workspace_bytes(img.nrows, img.ncols, block_size, max_points_per_block))
    kps, sc = _DeviceBuffer(cap * 12), _DeviceBuffer(cap * 4)
    count = C.c_int32(0)
    check(lib.vppb_fast9_blockwise_rank_u8(img.ptr(), th, mask.ptr() if mask is not None else None, block_size, max_points_per_block, ring_id, ws.ptr,
                                           ws.nbytes, kps.ptr, sc.ptr, cap, C.byref(count), stream))
    out = kps.to_host(np.int32, count.value * 3, stream).reshape(-1, 3)
    if scores is not None:
        scores[:] = list(sc.to_host(np.int32, count.value, stream))
    return out


# ---- the remaining 3x3 stencils (SURVEY 8(f) N4) ------------------------------------------------------
def lbp_transform(a, b=None, stream=None):  # lbp_transform.hh:7-38
    """lbp_transform(A, B): A u8 with a filled border >= 1, B u8 of the same domain (allocated if None)."""
    if b is None:
        b = Image2d(a.nrows, a.ncols, "u8")
    check(lib.vppb_lbp_u8(a.ptr(), b.ptr(), stream))
    return b


def local_maxima_filter(a, nbh_size=3, stream=None):  # fast.hpp:555-575 (nbh_size is ignored by the reference too)
    """In place: pixels that are not strict 3x3 maxima become 0, in the reference's serial raster order.  u8 or i32, border >= 1."""
    ws = _DeviceBuffer(lib.vppb_local_maxima_filter_workspace_bytes(a.nrows, a.ncols, a.desc.elem_bytes))
    check(lib.vppb_local_maxima_filter(a.ptr(), ws.ptr, ws.nbytes, stream))
    check(lib.vppb_sync(stream))  # the workspace is released on return
    return a


# ---- chamfer distance transforms (distance_transforms.hh:86-152) --------------------------------------------------------
def _distance_transform(kind, reach, a, b, stream):
    """b(p) = mask distance from p to the nearest zero of a, capped at B = nrows + ncols; b's whole border becomes B.  a: u8 or
    i32 (its border is not read); b: i32 of a's domain with a border >= reach, allocated with exactly that border when None."""
    if b is None:
        b = Image2d(a.nrows, a.ncols, "i32", border=reach)
    ws = _DeviceBuffer(lib.vppb_distance_transform_workspace_bytes(a.nrows, a.ncols, kind))
    check(lib.vppb_distance_transform(a.ptr(), b.ptr(), kind, ws.ptr, ws.nbytes, stream))
    check(lib.vppb_sync(stream))  # the workspace is released on return
    return b


def d4_distance_transform(a, b=None, stream=None):  # distance_transforms.hh:120-126, 4-neighbourhood, weight 1
    return _distance_transform(capi.DT_D4, 1, a, b, stream)


def d8_distance_transform(a, b=None, stream=None):  # distance_transforms.hh:128-134, 8-neighbourhood, weight 1
    return _distance_transform(capi.DT_D8, 1, a, b, stream)


def d3_4_distance_transform(a, b=None, stream=None):  # distance_transforms.hh:136-142, weights 3 (axes) and 4 (diagonals)
    return _distance_transform(capi.DT_D3_4, 1, a, b, stream)


def d5_7_11_distance_transform(a, b=None, stream=None):  # distance_transforms.hh:144-152, 5x5 with knight moves; border >= 2
    return _distance_transform(capi.DT_D5_7_11, 2, a, b, stream)


# ---- SAD descriptor matching (descriptor_matcher/*.hh) and patch extraction (patch.hh:32-47) ----------------------------
_DESC_PIXEL = {np.dtype(np.uint8): "u8", np.dtype(np.int32): "i32"}


def _descriptors(d, stream):
    """(keep-alive, VppbImg) of a descriptor set: an Image2d of u8 or i32 (one descriptor per row), or a 2-D uint8 / int32 array
    uploaded here; an empty array becomes a descriptor of zero rows"""
    if isinstance(d, Image2d):
        return d, d.desc
    a = np.asarray(d)
    if a.ndim != 2 or a.dtype not in _DESC_PIXEL:
        raise TypeError("descriptors: 2-D uint8 or int32 array or Image2d expected, got %s %s" % (a.dtype, a.shape))
    if a.shape[0] == 0:
        desc = capi.VppbImg(None, None, 0, a.shape[1], max(1, a.shape[1] * a.itemsize), 0, a.itemsize, 0)
        return desc, desc
    img = Image2d(a.shape[0], a.shape[1], _DESC_PIXEL[a.dtype])
    img.upload(a, stream=stream)
    return img, img.desc


def _positions(p, n, stream):
    kp = np.ascontiguousarray(p, dtype=np.int32).reshape(-1, 2)
    if len(kp) != n:
        raise ValueError("%d positions for %d descriptors" % (len(kp), n))
    return _DeviceBuffer(kp.nbytes).from_host(kp, stream)


def bruteforce_sad_matcher(query, train, stream=None):
    """bruteforce_matcher(query.nrows, train.nrows, _distance = sad_distance, _match) (bruteforce_matcher.hh:11-47): for every query
    the train of smallest SAD, ties to the lowest train index.  query / train: Image2d of u8 or i32, or 2-D uint8 / int32 arrays, one
    descriptor per row.  Returns (index[nq], distance[nq]) int32; (-1, INT32_MAX) for every query when there are no trains."""
    qk, qd = _descriptors(query, stream)
    tk, td = _descriptors(train, stream)
    nq = qd.nrows
    ws = _DeviceBuffer(lib.vppb_match_bruteforce_sad_workspace_bytes(nq, td.nrows, qd.ncols))
    d_idx, d_dist = _DeviceBuffer(nq * 4), _DeviceBuffer(nq * 4)
    check(lib.vppb_match_bruteforce_sad(C.byref(qd), C.byref(td), ws.ptr, ws.nbytes, d_idx.ptr, d_dist.ptr, stream))
    return d_idx.to_host(np.int32, nq, stream), d_dist.to_host(np.int32, nq, stream)


def local_sad_descriptor_matcher(query, train, query_positions, train_positions, search_radius=300, cell_width=300, stream=None):
    """local_index1d_sad_descriptor_matcher(_query, _train, _query_positions, _train_positions, _search_radius, _cell_width,
    _distance = sad_distance, _match) (local_index1d_sad_descriptor_matcher.hh:10-57; defaults grid_index.hh:16-17): for every query
    the train of smallest SAD among the trains whose cell (p / cell_width) lies in the query's window of cells
    ((q - search_radius) / cell_width .. (q + search_radius) / cell_width), ties to the smallest (cell row, cell col, train index).
    Positions: (n, 2) int (row, col).  Returns (index[nq], distance[nq]) int32; (-1, INT32_MAX) where the window holds no train."""
    qk, qd = _descriptors(query, stream)
    tk, td = _descriptors(train, stream)
    nq, nt = qd.nrows, td.nrows
    d_qp, d_tp = _positions(query_positions, nq, stream), _positions(train_positions, nt, stream)
    ws = _DeviceBuffer(lib.vppb_match_local_sad_workspace_bytes(nq, nt, qd.ncols, search_radius, cell_width))
    d_idx, d_dist = _DeviceBuffer(nq * 4), _DeviceBuffer(nq * 4)
    check(lib.vppb_match_local_sad(C.byref(qd), C.byref(td), d_qp.ptr, d_tp.ptr, search_radius, cell_width, ws.ptr, ws.nbytes, d_idx.ptr, d_dist.ptr,
                                   stream))
    return d_idx.to_host(np.int32, nq, stream), d_dist.to_host(np.int32, nq, stream)


def extract_patches(img, keypoints, winsize, stream=None):
    """extract_patches(kps, img, winsize) (patch.hh:32-47) with the layout the reference intends: row k of the returned Image2d
    (len(keypoints) x winsize^2, img's pixel type) is the winsize x winsize window centred on keypoints[k], row-major; a window
    leaving img's domain plus border gives a zero row.  img: u8 or i32 with border >= winsize / 2."""
    kp = np.ascontiguousarray(keypoints, dtype=np.int32).reshape(-1, 2)
    n = len(kp)
    d_kp = _DeviceBuffer(kp.nbytes).from_host(kp, stream)
    if n == 0:
        out = Image2d(0, 0, img.pixel, _desc=capi.VppbImg(None, None, 0, winsize * winsize, max(1, winsize * winsize * img.elem_bytes),
                                                          0, img.elem_bytes, 0))
    else:
        out = Image2d(n, winsize * winsize, img.pixel)
    check(lib.vppb_extract_patches(img.ptr(), d_kp.ptr, n, winsize, out.ptr(), stream))
    check(lib.vppb_sync(stream))  # the keypoint buffer is released on return
    return out


# ---- Lucas-Kanade -----------------------------------------------------------------------------
def oriented_lk_match(a, b, grad, keypoints, prediction, dir1, dir2, winsize, min_ev, max_iterations, convergence_delta, max_step_norm, stream=None):
    """oriented_lk_match_point_square_win<winsize>()(p, tr_prediction, A, B, Ag, min_ev, max_iterations, convergence_delta, max_step_norm,
    match_direction1, match_direction2) (lk.hh:180-317) for every keypoint: returns (flow (n, 2) float32, err (n,) float32)."""
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32).reshape(-1, 2)
    kp, pr, d1, d2 = f32(keypoints), f32(prediction), f32(dir1), f32(dir2)
    n = len(kp)
    bufs = [_DeviceBuffer(x.nbytes).from_host(x, stream) for x in (kp, pr, d1, d2)]
    d_flow, d_err = _DeviceBuffer(n * 8), _DeviceBuffer(n * 4)
    check(lib.vppb_lk_match_oriented_u8(a.ptr(), b.ptr(), grad.ptr(), 1 if grad.pixel == "vfloat2" else 0, winsize, min_ev, max_iterations, convergence_delta,
                                        max_step_norm, bufs[0].ptr, bufs[1].ptr, bufs[2].ptr, bufs[3].ptr, n, d_flow.ptr, d_err.ptr, stream))
    return d_flow.to_host(np.float32, n * 2, stream).reshape(-1, 2), d_err.to_host(np.float32, n, stream)


def _lk_run(pyr_prev, pyr_next, pyr_grad, params, keypoints, prediction, stream):
    kp = np.ascontiguousarray(keypoints, dtype=np.float32).reshape(-1, 2)
    n = len(kp)
    d_kp = _DeviceBuffer(kp.nbytes).from_host(kp, stream)
    d_pred = None
    if prediction is not None:
        d_pred = _DeviceBuffer(kp.nbytes).from_host(np.ascontiguousarray(prediction, dtype=np.float32).reshape(-1, 2), stream)
    d_flow = _DeviceBuffer(n * 8)
    d_err = _DeviceBuffer(n * 4)
    check(lib.vppb_lk_match_u8(pyr_prev.desc_array(), pyr_next.desc_array(), pyr_grad.desc_array(), C.byref(params), d_kp.ptr,
                               d_pred.ptr if d_pred else None, n, d_flow.ptr, d_err.ptr, stream))
    return d_flow.to_host(np.float32, n * 2, stream).reshape(-1, 2), d_err.to_host(np.float32, n, stream)


def lucas_kanade(i1, i2, keypoints, niterations=21, winsize=11, nscales=3, min_ev=0.0001, delta=0.1, prediction=None,
                 stream=None):
    """lucas_kanade(i1, i2, _keypoints=, _flow=, ...) (lucas_kanade.hpp:135-184).
    Returns (flow[n,2], dist[n]) — the values the reference hands to the _flow callback.
    As in the reference, min_ev and delta are stored in `int` (lucas_kanade.hpp:143-144) and so
    truncate (0.0001 -> 0, 0.1 -> 0); pyramids and the vint2 Scharr gradient pyramid are built here.
    winsize < 5 gives the pyramids a border < 2, which the reference's 5-tap low-pass reads past (undefined values
    there); here that raises VppbError(VPPB_E_BORDER) instead."""
    border = winsize // 2
    prev = Pyramid2d((i1.nrows, i1.ncols), nscales, 2, pixel="u8", border=border)
    nxt = Pyramid2d((i1.nrows, i1.ncols), nscales, 2, pixel="u8", border=border)
    grad = Pyramid2d((i1.nrows, i1.ncols), nscales, 2, pixel="vint2", border=border)
    pyrlk_prepare(i1, i2, prev, nxt, grad, stream)
    P = capi.VppbLkParams(nlevels=nscales, min_scale=0, winsize=winsize, max_iter=niterations, grad_is_float=0,
                          err_mode=capi.LK_ERR_SAD, gate_on_max_err=0, min_ev=float(int(min_ev)), delta=float(int(delta)),
                          max_err=0.0, factor=2.0, pred_div=float(2 ** nscales))
    return _lk_run(prev, nxt, grad, P, keypoints, prediction, stream)


def pyrlk_prepare(i1, i2, prev, nxt, grad, stream=None):
    """The two u8 pyramids and the Scharr gradient pyramid of frame 1 (lucas_kanade.hpp:150-157) in one call: three
    independent chains (vppb_pyrlk_prepare: one cooperative launch for images in the library layout)."""
    check(lib.vppb_pyrlk_prepare(i1.ptr(), i2.ptr(), prev.desc_array(), nxt.desc_array(), grad.desc_array(), len(prev),
                                 1 if grad.pixel == "vfloat2" else 0, stream))


def pyrlk_match(pyr_prev, pyr_prev_grad, pyr_next, keypoints, winsize, min_ev, max_err, max_iteration, convergence_delta,
                min_scale=0, stream=None):
    """pyrlk_match(..., lk_match_point_square_win<WS>(), min_ev, max_err, max_iter, delta[, min_scale])
    (pyrlk_match.hh:15-55).  Returns (flow, dist, keep): keep[i] is False where the reference calls
    keypoints.remove(i) (dist > max_err or the moved point leaves the level-0 domain)."""
    P = capi.VppbLkParams(nlevels=len(pyr_prev), min_scale=min_scale, winsize=winsize, max_iter=int(max_iteration),
                          grad_is_float=1 if pyr_prev_grad.pixel == "vfloat2" else 0, err_mode=capi.LK_ERR_SAD_OVER_MAD,
                          gate_on_max_err=1, min_ev=min_ev, delta=convergence_delta, max_err=max_err,
                          factor=pyr_prev.factor, pred_div=1.0)
    flow, dist = _lk_run(pyr_prev, pyr_next, pyr_prev_grad, P, keypoints, None, stream)
    kp = np.asarray(keypoints, dtype=np.float32).reshape(-1, 2)
    moved = (kp + flow).astype(np.int32)  # cast<vint2>: truncation
    inside = (moved[:, 0] >= 0) & (moved[:, 0] < pyr_prev[0].nrows) & (moved[:, 1] >= 0) & (moved[:, 1] < pyr_prev[0].ncols)
    keep = ~(dist > max_err) & inside
    return flow, dist, keep


# ---- semi-dense optical flow ------------------------------------------------------------------
def semi_dense_optical_flow(keypoints, i1, i2, winsize=7, nscales=4, min_scale=0, propagation=2, patchsize=5, stream=None):
    """semi_dense_optical_flow(keypoints, match_callback, i1, i2, _winsize, _nscales, _min_scale, _propagation, _patchsize)
    (semi_dense_optical_flow.hpp:46-214; defaults :57-61).  keypoints: (n, 2) int (row, col).
    Returns (pos[n,2], dist[n], valid[n]): for every i with valid[i] the reference calls match_callback(i, pos[i], dist[i])."""
    kp = np.ascontiguousarray(keypoints, dtype=np.int32).reshape(-1, 2)
    n = len(kp)
    p1 = Pyramid2d((i1.nrows, i1.ncols), nscales, 2, pixel="u8", border=2 * winsize)  # :72-73
    p2 = Pyramid2d((i2.nrows, i2.ncols), nscales, 2, pixel="u8", border=2 * winsize)
    check(lib.vppb_pyrlk_prepare(i1.ptr(), i2.ptr(), p1.desc_array(), p2.desc_array(), None, nscales, 0, stream))  # both pyramids in one launch
    P = capi.VppbSdofParams(winsize, nscales, min_scale, propagation, patchsize)
    ws = _DeviceBuffer(lib.vppb_sdof_workspace_bytes(i1.nrows, i1.ncols, C.byref(P)))
    d_kp = _DeviceBuffer(kp.nbytes).from_host(kp, stream)
    d_pos, d_dist, d_valid = _DeviceBuffer(n * 8), _DeviceBuffer(n * 4), _DeviceBuffer(n)
    check(lib.vppb_sdof_u8(p1.desc_array(), p2.desc_array(), C.byref(P), d_kp.ptr, n, ws.ptr, ws.nbytes, d_pos.ptr, d_dist.ptr,
                           d_valid.ptr, stream))
    return (d_pos.to_host(np.int32, n * 2, stream).reshape(-1, 2), d_dist.to_host(np.int32, n, stream),
            d_valid.to_host(np.uint8, n, stream).astype(bool))


# ---- sparse optical flow ----------------------------------------------------------------------
_SOF_CACHE = {}  # (nrows, ncols, params, nkeypoints) -> workspace: allocated once per shape, reused


def sparse_optical_flow(i1, i2, keypoints=None, detector_th=5, block_size=5, winsize=11, search_radius=100, cell_width=300,
                        subpixelic=False, lk_iterations=5, nscales=3, stream=None):
    """sparse_optical_flow(i1, i2, _flow = f, ...) / sparse_optical_flow(keypoints, match_callback, i1, i2, ...)
    (optical_flow.hh:52-73; defaults sparse_optical_flow.hh:45-49, grid_index.hh:16; semantics DESIGN §3.9): blockwise FAST
    keypoints K1 of i1 (or `keypoints`, (n, 2) int (row, col)) matched to those of i2 by the grid-local SAD of their winsize x
    winsize patches, refined by Lucas-Kanade when `subpixelic`.  i1, i2: u8 images of one domain with borders >= max(3, winsize / 2),
    filled by the caller.  Returns (positions (n, 2) int32 = K1, flow (n, 2) float32, distance (n,) int32, valid (n,) bool): the
    reference calls its callback for the valid entries, in this order."""
    P = capi.VppbSofParams(detector_th, block_size, winsize, search_radius, cell_width, 1 if subpixelic else 0, lk_iterations, nscales)
    d_kp, n = None, -1
    if keypoints is not None:
        kp = np.ascontiguousarray(keypoints, dtype=np.int32).reshape(-1, 2)
        n = len(kp)
        d_kp = _DeviceBuffer(kp.nbytes).from_host(kp, stream)
    key = (i1.nrows, i1.ncols, tuple(getattr(P, f) for f, _ in P._fields_), n)
    ws = _SOF_CACHE.get(key)
    if ws is None:
        if len(_SOF_CACHE) > 8:
            _SOF_CACHE.clear()
        ws = _SOF_CACHE[key] = _DeviceBuffer(lib.vppb_sparse_flow_workspace_bytes(i1.nrows, i1.ncols, C.byref(P), n))
    bs = max(1, block_size)
    cap = n if n >= 0 else ((i1.nrows + bs - 1) // bs) * ((i1.ncols + bs - 1) // bs)
    d_pos, d_flow, d_dist, d_valid = _DeviceBuffer(cap * 8), _DeviceBuffer(cap * 8), _DeviceBuffer(cap * 4), _DeviceBuffer(cap)
    count = C.c_int32(0)
    check(lib.vppb_sparse_flow_u8(i1.ptr(), i2.ptr(), C.byref(P), d_kp.ptr if d_kp else None, max(n, 0), ws.ptr, ws.nbytes, d_pos.ptr, d_flow.ptr,
                                  d_dist.ptr, d_valid.ptr, cap, C.byref(count), stream))
    m = count.value
    return (d_pos.to_host(np.int32, m * 2, stream).reshape(-1, 2), d_flow.to_host(np.float32, m * 2, stream).reshape(-1, 2),
            d_dist.to_host(np.int32, m, stream), d_valid.to_host(np.uint8, m, stream).astype(bool))
