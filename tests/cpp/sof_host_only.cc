// Plain g++ -std=c++14 translation unit: the sparse optical flow is host-callable C++14, and the flow header, the tracker and the
// descriptor matcher can be included together (their shared option symbols live in vpp/core/symbols.hh).  Syntax check by build.sh.
#include <vpp/vpp.hh>
#include <vpp/algorithms/descriptor_matcher.hh>
#include <vpp/algorithms/optical_flow.hh>
#include <vpp/algorithms/video_extruder.hh>

int sof_host_only_demo() {
  using namespace vpp;
  image2d<unsigned char> f1(270, 480, _border = 5), f2(270, 480, _border = 5);
  int n = 0;
  sparse_optical_flow(f1, f2, _flow = [&](vint2, vfloat2, int) { n++; }, _detector_th = 10, _search_radius = 50, _cell_width = 40);
  std::vector<vint2> kps = {vint2(10, 10), vint2(100, 200)};
  sparse_optical_flow(kps, [&](int, vfloat2, int) { n++; }, f1, f2, _subpixelic, _lk_iterations = 3, _winsize = 9, _nscales = 2);
  auto ctx = video_extruder_init(f1.domain());
  video_extruder_update(ctx, f1, f2, _detector_th = 10);
  local_index1d_sad_descriptor_matcher(_query = f1, _train = f2, _query_positions = kps, _train_positions = kps, _search_radius = 32,
                                       _cell_width = 32, _match = [&](int, int, int) { n++; });
  return n;
}
