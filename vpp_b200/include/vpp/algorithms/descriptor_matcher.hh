// SAD descriptor matchers (reference: vpp/algorithms/descriptor_matcher.hh, descriptor_matcher/bruteforce_matcher.hh:11-47,
// local_index1d_sad_descriptor_matcher.hh:10-57, grid_index.hh:11-88).  Descriptors are the rows of an image2d<unsigned char> or
// image2d<int> (one descriptor per row, ncols = its length); the distance is the reference's sad_distance, sum |q[k] - t[k]|.
// The GPU computes every match (vppb_match_bruteforce_sad / vppb_match_local_sad), then _match(i, j, d) is called serially from
// the host in query order, for every query that has a match.
//
//   bruteforce_sad_matcher(query, train, _match = f): the train of smallest SAD, ties to the lowest train index - index and
//     distance equal the reference's bruteforce_matcher with sad_distance.  The reference takes an arbitrary host _distance, which
//     no GPU path can run; without trains nothing is called (the reference reads train 0).
//   local_index1d_sad_descriptor_matcher(_query, _train, _query_positions, _train_positions, _search_radius = 300,
//     _cell_width = 300, _match): the smallest SAD over the trains whose cell (p / s) lies in the query's window of cells
//     ((q - R) / s .. (q + R) / s), ties to the smallest (cell row, cell col, train index).  The distance equals the reference's
//     at _approximation = 1; the index equals it wherever the reference's choice is determined (inside one cell it orders ties
//     by an unstable std::sort).  _approximation is accepted for source compatibility and ignored: the result is the exact one.
//     A train at a coordinate <= -s is never matched (the reference asserts).
#pragma once
#include <type_traits>
#include <vector>
#include <vpp/algorithms/fast_detector/fast.hh>  // internals::device_array
#include <vpp/core/image2d.hh>

namespace vpp {

namespace s {
VPP_DEFINE_SYMBOL(query)
VPP_DEFINE_SYMBOL(train)
VPP_DEFINE_SYMBOL(query_positions)
VPP_DEFINE_SYMBOL(train_positions)
VPP_DEFINE_SYMBOL(approximation)
VPP_DEFINE_SYMBOL(distance)
VPP_DEFINE_SYMBOL(match)
}  // namespace s

namespace internals {
template <typename T>
void check_descriptor_type() {
  static_assert(std::is_same<T, unsigned char>::value || std::is_same<T, int>::value,
                "descriptor matchers: image2d<unsigned char> or image2d<int> descriptors");
}

template <typename F>
void report_matches(int nq, const device_array& di, const device_array& dd, F match) {
  std::vector<int> idx(nq), dist(nq);
  di.to_host(idx.data(), (size_t)nq * 4);
  dd.to_host(dist.data(), (size_t)nq * 4);
  for (int i = 0; i < nq; i++)
    if (idx[i] >= 0) match(i, idx[i], dist[i]);
}
}  // namespace internals

template <typename T, typename F>
void bruteforce_sad_matcher(const image2d<T>& query, const image2d<T>& train, const s::opt<s::_match_t, F>& match) {
  internals::check_descriptor_type<T>();
  const int nq = query.nrows();
  if (nq == 0) return;
  const int64_t wsb = vppb_match_bruteforce_sad_workspace_bytes(nq, train.nrows(), query.ncols());
  internals::device_array ws((size_t)wsb), di((size_t)nq * 4), dd((size_t)nq * 4);
  vppb_check(vppb_match_bruteforce_sad(query.device_read(), train.device_read(), ws.ptr(), wsb, (int32_t*)di.ptr(), (int32_t*)dd.ptr(), nullptr));
  internals::report_matches(nq, di, dd, match.value);
}

template <typename... OPTS>
void local_index1d_sad_descriptor_matcher(OPTS... options) {
  auto opts = s::D(options...);
  typedef decltype(opts) O;
  static_assert(!O::has(s::_distance), "local_index1d_sad_descriptor_matcher: _distance is not supported - pass the descriptor images "
                                       "as _query / _train; the distance is SAD, computed on the GPU");
  static_assert(O::has(s::_query) && O::has(s::_train), "local_index1d_sad_descriptor_matcher: _query / _train missing");
  static_assert(O::has(s::_query_positions) && O::has(s::_train_positions), "local_index1d_sad_descriptor_matcher: positions missing");
  static_assert(O::has(s::_match), "local_index1d_sad_descriptor_matcher: _match callback is missing");
  const auto query = opts.get(s::_query, 0);
  const auto train = opts.get(s::_train, 0);
  const auto& qpos = opts.get(s::_query_positions, 0);
  const auto& tpos = opts.get(s::_train_positions, 0);
  const int R = opts.get(s::_search_radius, 300), cw = opts.get(s::_cell_width, 300);  // grid_index.hh:16-17
  (void)opts.get(s::_approximation, 1);
  auto match = opts.get(s::_match, 0);
  internals::check_descriptor_type<typename std::decay<decltype(query)>::type::value_type>();
  const int nq = query.nrows(), nt = train.nrows();
  if ((int)qpos.size() != nq || (int)tpos.size() != nt) vppb_check(VPPB_E_ARG);
  if (nq == 0) return;
  std::vector<vint2> qp(qpos.begin(), qpos.end()), tp(tpos.begin(), tpos.end());
  const int64_t wsb = vppb_match_local_sad_workspace_bytes(nq, nt, query.ncols(), R, cw);
  internals::device_array ws((size_t)wsb), dq((size_t)nq * 8), dt((size_t)nt * 8), di((size_t)nq * 4), dd((size_t)nq * 4);
  dq.from_host(qp.data(), (size_t)nq * 8);
  dt.from_host(tp.data(), (size_t)nt * 8);
  vppb_check(vppb_match_local_sad(query.device_read(), train.device_read(), (const vppb_int2*)dq.ptr(), (const vppb_int2*)dt.ptr(), R, cw,
                                  ws.ptr(), wsb, (int32_t*)di.ptr(), (int32_t*)dd.ptr(), nullptr));
  internals::report_matches(nq, di, dd, match);
}

}  // namespace vpp
