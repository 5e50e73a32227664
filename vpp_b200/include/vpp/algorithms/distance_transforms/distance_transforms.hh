// d4_distance_transform, d8_distance_transform, d3_4_distance_transform and d5_7_11_distance_transform(A, S) (reference:
// vpp/algorithms/distance_transforms/distance_transforms.hh:86-152): S = the mask distance from every pixel to the nearest zero
// pixel of A, capped at B = A.nrows() + A.ncols(); S's whole border becomes B.  A: image2d<unsigned char> or image2d<int> (its
// border is not read); S: image2d<int> of A's domain with a border >= 1 (>= 2 for d5_7_11).  The result is the reference's serial
// forward / backward passes bit for bit, computed by the CUDA kernels behind vppb_distance_transform.
// Not provided: euclide_distance_transform (its result depends on the serial visiting order) and
// generic_incremental_distance_transform with caller-supplied masks.
#pragma once
#include <type_traits>
#include <vpp/algorithms/fast_detector/fast.hh>  // internals::device_array
#include <vpp/core/image2d.hh>

namespace vpp {

namespace internals {
template <typename T>
void chamfer_distance_transform(const image2d<T>& a, const image2d<int>& s, int kind) {
  static_assert(std::is_same<T, unsigned char>::value || std::is_same<T, int>::value,
                "distance transforms: image2d<unsigned char> or image2d<int> input");
  const int64_t bytes = vppb_distance_transform_workspace_bytes(a.nrows(), a.ncols(), kind);
  device_array ws((size_t)bytes);
  vppb_check(vppb_distance_transform(a.device_read(), s.device_write(), kind, ws.ptr(), bytes, nullptr));
  vppb_check(vppb_sync(nullptr));  // the workspace is released on return
}
}  // namespace internals

const auto d4_distance_transform = [](auto& a, auto& b) { internals::chamfer_distance_transform(a, b, VPPB_DT_D4); };
const auto d8_distance_transform = [](auto& a, auto& b) { internals::chamfer_distance_transform(a, b, VPPB_DT_D8); };
const auto d3_4_distance_transform = [](auto& a, auto& b) { internals::chamfer_distance_transform(a, b, VPPB_DT_D3_4); };
const auto d5_7_11_distance_transform = [](auto& a, auto& b) { internals::chamfer_distance_transform(a, b, VPPB_DT_D5_7_11); };

}  // namespace vpp
