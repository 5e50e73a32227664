"""vpp_b200 — H100-native (sm_90a) dense-pixel path behind the Video++ (matt-42/vpp) API.

The package holds the CUDA kernels + C-ABI (csrc/, include/vppb.h at the repo root), the ctypes
binding (capi) and the Python host mirror of the reference operator surface (image, ops).
Importing it loads vpp_b200/lib/libvppb.so and fails loudly if the library has not been built.
"""
from . import capi  # noqa: F401  (raises ImportError when libvppb.so is missing)
from .image import Box2d, Image2d, make_box2d, layout, DEFAULT_ALIGNMENT  # noqa: F401
from .ops import (  # noqa: F401
    Pyramid2d, box5x5, box5x5_batch, clone, copy, copy_with_border, fast9, fast9_scores, fill, fill_border_closest,
    fill_border_mirror, fill_border_with_value, fill_with_border, ingest_rgb_frame, lucas_kanade, pixel_wise_add,
    pyrlk_match, pyrlk_prepare, rgb_to_graylevel, scharr, semi_dense_optical_flow, sum, fast9_blockwise_rank, lbp_transform,
    local_maxima_filter, oriented_lk_match, d4_distance_transform, d8_distance_transform, d3_4_distance_transform,
    d5_7_11_distance_transform, bruteforce_sad_matcher, local_sad_descriptor_matcher, extract_patches,
    sparse_optical_flow,
)
from . import video_extruder  # noqa: F401,E402
