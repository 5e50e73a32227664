"""ctypes binding of the C-ABI in include/vppb.h (vpp_b200/lib/libvppb.so).

This is the only door into the CUDA path from Python.  There is no CPU fallback: if the
shared library is missing the import of this module raises, and every compute entry returns
VPPB_E_CUDA on a machine without a GPU.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvppb.so")

VPPB_OK = 0
VPPB_E_CUDA = -1
VPPB_E_ARG = -2
VPPB_E_BORDER = -3
VPPB_E_CAPACITY = -4
VPPB_E_NCCL = -5

FAST_REFERENCE_RING, FAST_TRUE_RING = 0, 1
FAST_ALL, FAST_LOCAL_MAXIMA, FAST_BLOCKWISE = 0, 1, 2
LK_ERR_SAD, LK_ERR_SAD_OVER_MAD = 0, 1
DT_D4, DT_D8, DT_D3_4, DT_D5_7_11 = 0, 1, 2, 3


class VppbImg(C.Structure):
    _fields_ = [
        ("base", C.c_void_p),
        ("alloc", C.c_void_p),
        ("nrows", C.c_int32),
        ("ncols", C.c_int32),
        ("pitch", C.c_int32),
        ("border", C.c_int32),
        ("elem_bytes", C.c_int32),
        ("align", C.c_int32),
    ]


class VppbInt2(C.Structure):
    _fields_ = [("r", C.c_int32), ("c", C.c_int32)]


class VppbFloat2(C.Structure):
    _fields_ = [("r", C.c_float), ("c", C.c_float)]


class VppbLkParams(C.Structure):
    _fields_ = [
        ("nlevels", C.c_int32),
        ("min_scale", C.c_int32),
        ("winsize", C.c_int32),
        ("max_iter", C.c_int32),
        ("grad_is_float", C.c_int32),
        ("err_mode", C.c_int32),
        ("gate_on_max_err", C.c_int32),
        ("min_ev", C.c_float),
        ("delta", C.c_float),
        ("max_err", C.c_float),
        ("factor", C.c_float),
        ("pred_div", C.c_float),
    ]


class VppbSdofParams(C.Structure):
    _fields_ = [("winsize", C.c_int32), ("nscales", C.c_int32), ("min_scale", C.c_int32), ("propagation", C.c_int32),
                ("patchsize", C.c_int32)]


class VppbSofParams(C.Structure):
    _fields_ = [("detector_th", C.c_int32), ("block_size", C.c_int32), ("winsize", C.c_int32), ("search_radius", C.c_int32),
                ("cell_width", C.c_int32), ("subpixelic", C.c_int32), ("lk_iterations", C.c_int32), ("nscales", C.c_int32)]


_P = C.POINTER
_IMG = _P(VppbImg)
_VP = C.c_void_p
_I32 = C.c_int32
_I64 = C.c_int64

# name -> (restype, argtypes): every symbol include/vppb.h declares
PROTOTYPES = {
    "vppb_version": (C.c_int, []),
    "vppb_last_error": (C.c_char_p, []),
    "vppb_init": (C.c_int, [C.c_int]),
    "vppb_device_count": (C.c_int, [_P(C.c_int)]),
    "vppb_sync": (C.c_int, [_VP]),
    "vppb_layout": (C.c_int, [_I32, _I32, _I32, _I32, _I32, _P(_I32), _P(_I64), _P(_I64)]),
    "vppb_alloc": (C.c_int, [_IMG, _I32, _I32, _I32, _I32, _I32]),
    "vppb_wrap": (C.c_int, [_IMG, _VP, _I32, _I32, _I32, _I32, _I32]),
    "vppb_free": (C.c_int, [_IMG]),
    "vppb_subimage": (C.c_int, [_IMG, _I32, _I32, _I32, _I32, _IMG]),
    "vppb_upload": (C.c_int, [_IMG, _VP, _I64, C.c_int, _VP]),
    "vppb_download": (C.c_int, [_IMG, _VP, _I64, C.c_int, _VP]),
    "vppb_pw_add_i32": (C.c_int, [_IMG, _IMG, _IMG, _VP]),
    "vppb_fill": (C.c_int, [_IMG, _VP, C.c_int, _VP]),
    "vppb_copy2d": (C.c_int, [_IMG, _IMG, C.c_int, _VP]),
    "vppb_copy2d_mirror": (C.c_int, [_IMG, _IMG, _VP]),
    "vppb_fill_border_value": (C.c_int, [_IMG, _VP, _VP]),
    "vppb_fill_border_mirror": (C.c_int, [_IMG, _VP]),
    "vppb_fill_border_closest": (C.c_int, [_IMG, _VP]),
    "vppb_sum_i32": (C.c_int, [_IMG, C.c_int, _P(_I64), _VP]),
    "vppb_box5x5_u8c3": (C.c_int, [_IMG, _IMG, _VP]),
    "vppb_box5x5_i32": (C.c_int, [_IMG, _IMG, _VP]),
    "vppb_box5x5_u8": (C.c_int, [_IMG, _IMG, _VP]),
    "vppb_box5x5_u8c3_batch": (C.c_int, [_IMG, _IMG, _I32, _VP]),
    "vppb_box5x5_u8_batch": (C.c_int, [_IMG, _IMG, _I32, _VP]),
    "vppb_rgb_to_graylevel_u8": (C.c_int, [_IMG, _IMG, _VP]),
    "vppb_rgb_to_graylevel_u8_mirror": (C.c_int, [_IMG, _IMG, _VP]),
    "vppb_scharr_u8": (C.c_int, [_IMG, _IMG, C.c_int, _VP]),
    "vppb_scharr_u8_mirror": (C.c_int, [_IMG, _IMG, C.c_int, _VP]),
    "vppb_lowpass_sub2": (C.c_int, [_IMG, _IMG, C.c_int, _VP]),
    "vppb_lowpass_sub2_mirror": (C.c_int, [_IMG, _IMG, C.c_int, _VP]),
    "vppb_pyrlk_prepare": (C.c_int, [_IMG, _IMG, _IMG, _IMG, _IMG, _I32, _I32, _VP]),
    "vppb_fast9_workspace_bytes": (_I64, [_I32, _I32, _I32]),
    "vppb_fast9_u8": (C.c_int, [_IMG, _I32, _IMG, _I32, _I32, _I32, _VP, _I64, _VP, _VP, _I32, _P(_I32), _VP]),
    "vppb_fast9_u8_async": (C.c_int, [_IMG, _I32, _IMG, _I32, _I32, _I32, _VP, _I64, _VP, _VP, _I32, _VP, _VP]),
    "vppb_fast9_scores": (C.c_int, [_IMG, _I32, _VP, _I32, _VP, _VP]),
    "vppb_fast9_rank_workspace_bytes": (_I64, [_I32, _I32, _I32, _I32]),
    "vppb_fast9_blockwise_rank_u8": (C.c_int, [_IMG, _I32, _IMG, _I32, _I32, _I32, _VP, _I64, _VP, _VP, _I32, _P(_I32), _VP]),
    "vppb_lbp_u8": (C.c_int, [_IMG, _IMG, _VP]),
    "vppb_local_maxima_filter_workspace_bytes": (_I64, [_I32, _I32, _I32]),
    "vppb_local_maxima_filter": (C.c_int, [_IMG, _VP, _I64, _VP]),
    "vppb_distance_transform_workspace_bytes": (_I64, [_I32, _I32, _I32]),
    "vppb_distance_transform": (C.c_int, [_IMG, _IMG, _I32, _VP, _I64, _VP]),
    "vppb_match_bruteforce_sad_workspace_bytes": (_I64, [_I32, _I32, _I32]),
    "vppb_match_bruteforce_sad": (C.c_int, [_IMG, _IMG, _VP, _I64, _VP, _VP, _VP]),
    "vppb_match_local_sad_workspace_bytes": (_I64, [_I32, _I32, _I32, _I32, _I32]),
    "vppb_match_local_sad": (C.c_int, [_IMG, _IMG, _VP, _VP, _I32, _I32, _VP, _I64, _VP, _VP, _VP]),
    "vppb_extract_patches": (C.c_int, [_IMG, _VP, _I32, _I32, _IMG, _VP]),
    "vppb_lk_match_oriented_u8": (C.c_int, [_IMG, _IMG, _IMG, _I32, _I32, C.c_float, _I32, C.c_float, C.c_float, _VP, _VP, _VP, _VP, _I32, _VP, _VP, _VP]),
    "vppb_lk_match_u8": (C.c_int, [_IMG, _IMG, _IMG, _P(VppbLkParams), _VP, _VP, _I32, _VP, _VP, _VP]),
    "vppb_sdof_workspace_bytes": (_I64, [_I32, _I32, _P(VppbSdofParams)]),
    "vppb_sdof_u8": (C.c_int, [_IMG, _IMG, _P(VppbSdofParams), _VP, _I32, _VP, _I64, _VP, _VP, _VP, _VP]),
    "vppb_sparse_flow_workspace_bytes": (_I64, [_I32, _I32, _P(VppbSofParams), _I32]),
    "vppb_sparse_flow_u8": (C.c_int, [_IMG, _IMG, _P(VppbSofParams), _VP, _I32, _VP, _I64, _VP, _VP, _VP, _VP, _I32, _P(_I32), _VP]),
    "vppb_halo_bytes": (_I64, [_IMG, _I32]),
    "vppb_halo_pack": (C.c_int, [_IMG, _I32, C.c_int, _VP, _VP]),
    "vppb_halo_unpack": (C.c_int, [_IMG, _I32, C.c_int, _VP, _VP]),
    "vppb_halo_pack_batch": (C.c_int, [_IMG, _I32, _I32, C.c_int, _VP, _VP]),
    "vppb_halo_unpack_batch": (C.c_int, [_IMG, _I32, _I32, C.c_int, _VP, _VP]),
    "vppb_kpc_create": (C.c_int, [_I32, _I32, _P(_VP)]),
    "vppb_kpc_destroy": (C.c_int, [_VP]),
    "vppb_kpc_size": (_I32, [_VP]),
    "vppb_kpc_positions": (_VP, [_VP]),
    "vppb_kpc_flow_update": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _VP]),
    "vppb_kpc_merge": (C.c_int, [_VP, _I32, _I32, _I32, _VP]),
    "vppb_kpc_score_filter": (C.c_int, [_VP, _IMG, _I32, _I32, _VP]),
    "vppb_kpc_paint_mask": (C.c_int, [_VP, _IMG, _I32, _VP]),
    "vppb_kpc_add_and_compact": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _VP]),
    "vppb_kpc_trajectories_update": (C.c_int, [_VP, _VP]),
    "vppb_kpc_state_table": (C.c_int, [_VP, _VP, _VP]),
    "vppb_kpc_history": (C.c_int, [_VP, _VP, _VP, _VP]),
    "vppb_box5x5_u8c3_tiles": (C.c_int, [_IMG, _IMG, _IMG, _IMG, _I32, _VP]),
    "vppb_box5x5_u8_tiles": (C.c_int, [_IMG, _IMG, _IMG, _IMG, _I32, _VP]),
    "vppb_ipc_export": (C.c_int, [_IMG, _VP, _P(_I64)]),
    "vppb_ipc_open": (C.c_int, [_VP, _I64, _IMG, _IMG]),
    "vppb_ipc_close": (C.c_int, [_IMG]),
    "vppb_comm_unique_id": (C.c_int, [_VP]),
    "vppb_comm_init": (C.c_int, [_VP, _I32, _I32, _P(_VP)]),
    "vppb_comm_destroy": (C.c_int, [_VP]),
    "vppb_halo_exchange": (C.c_int, [_VP, _I32, _I32, _IMG, _I32, _I32, _VP]),
}


class VppbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("vppb error %d: %s" % (code, msg))
        self.code = code


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the vpp_b200 path)" % LIB_PATH
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError here == the ABI header and the library disagree
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(rc):
    if rc != 0:
        raise VppbError(rc, lib.vppb_last_error().decode("utf-8", "replace"))
    return rc
