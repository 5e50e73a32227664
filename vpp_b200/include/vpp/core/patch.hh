// extract_patches(kps, img, winsize) (reference: vpp/core/patch.hh:32-47): row k of the result (kps.size() x winsize^2, img's
// pixel type) is the winsize x winsize window centred on kps[k], row-major from element 0: element (r + h) * winsize + (c + h) for
// r, c in [-h, winsize - h), h = winsize / 2.  Deviation: the reference writes element r * winsize + c, which lands before each
// row (out of bounds for keypoint 0); this is the layout it plainly intends.  img: image2d<unsigned char> or image2d<int> with a
// border >= h; a keypoint whose window leaves the domain plus border gets a zero row.  kps must not be empty.  Runs the CUDA
// gather behind vppb_extract_patches.  Not provided: patch<V> and extract_patch for one position.
#pragma once
#include <type_traits>
#include <vector>
#include <vpp/algorithms/fast_detector/fast.hh>  // internals::device_array
#include <vpp/core/image2d.hh>

namespace vpp {

template <typename V>
image2d<V> extract_patches(const std::vector<vint2>& kps, const image2d<V>& img, int winsize) {
  static_assert(std::is_same<V, unsigned char>::value || std::is_same<V, int>::value, "extract_patches: image2d<unsigned char> or image2d<int>");
  const int n = (int)kps.size();
  image2d<V> patches(n, winsize * winsize);
  internals::device_array dk((size_t)n * 8);
  dk.from_host(kps.data(), (size_t)n * 8);
  vppb_check(vppb_extract_patches(img.device_read(), (const vppb_int2*)dk.ptr(), n, winsize, patches.device_write(), nullptr));
  vppb_check(vppb_sync(nullptr));  // the keypoint buffer is released on return
  return patches;
}

}  // namespace vpp
