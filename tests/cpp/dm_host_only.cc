// Plain g++ -std=c++14 translation unit: the descriptor matchers and extract_patches are host-callable C++14 (syntax check by
// build.sh, like host_only.cc).
#include <vpp/vpp.hh>
#include <vpp/algorithms/descriptor_matcher.hh>
#include <vpp/core/patch.hh>

int dm_host_only_demo() {
  using namespace vpp;
  image2d<unsigned char> img(270, 480, _border = 3);
  std::vector<vint2> kps = {vint2(10, 10), vint2(100, 200)};
  image2d<unsigned char> d = extract_patches(kps, img, 7);
  int n = 0;
  bruteforce_sad_matcher(d, d, _match = [&](int, int, int) { n++; });
  local_index1d_sad_descriptor_matcher(_query = d, _train = d, _query_positions = kps, _train_positions = kps, _search_radius = 32,
                                       _cell_width = 32, _approximation = 2, _match = [&](int, int, int) { n++; });
  return n;
}
