// semi_dense_optical_flow(keypoints, match_callback, i1, i2, _winsize =, _nscales =, _min_scale =,
// _propagation =, _patchsize =) (reference: vpp/algorithms/optical_flow.hh:29-35,
// optical_flow/semi_dense_optical_flow.hpp:46-214).  keypoints: anything with size() and operator[] -> vint2.
// match_callback(i, new_position, distance) is invoked serially, in keypoint order, as in the reference.
//
// sparse_optical_flow(i1, i2, _flow = f, opts...) and sparse_optical_flow(keypoints, match_callback, i1, i2, opts...)
// (reference: optical_flow.hh:52-73; its body, optical_flow/sparse_optical_flow.hh:36-112, never compiled: the semantics are
// this library's, include/vppb.h and DESIGN §3.9).  Blockwise FAST keypoints K1 of i1 (or `keypoints`) and K2 of i2, their
// winsize x winsize patches matched by the grid-local SAD matcher; with _subpixelic, refined by lucas_kanade.  Options and defaults:
// _detector_th = 5, _block_size = 5, _winsize = 11, _lk_iterations = 5, _search_radius = 100, _cell_width = 300, _nscales = 3,
// _subpixelic = false.  i1 / i2 need a border >= max(3, winsize / 2), filled by the caller.  Callbacks run serially in K1 order,
// for the valid entries only: f(vint2 p, vfloat2 flow, int distance), match_callback(int i, vfloat2 new_position = K1[i] + flow,
// int distance).
#pragma once
#include <vector>
#include <vpp/algorithms/fast_detector/fast.hh>
#include <vpp/core/pyramid.hh>

namespace vpp {

namespace s {
VPP_DEFINE_SYMBOL(min_scale)
VPP_DEFINE_SYMBOL(propagation)
VPP_DEFINE_SYMBOL(patchsize)
VPP_DEFINE_SYMBOL(lk_iterations)
VPP_DEFINE_SYMBOL(subpixelic)
}  // namespace s

template <typename K, typename MC, typename... OPTS>
void semi_dense_optical_flow(const K& keypoints, MC match_callback, const image2d<unsigned char>& i1, const image2d<unsigned char>& i2,
                             OPTS... options) {
  auto opts = s::D(options...);
  vppb_sdof_params P;
  P.winsize = opts.get(s::_winsize, 7);   // defaults: semi_dense_optical_flow.hpp:57-61
  P.nscales = opts.get(s::_nscales, 4);
  P.min_scale = opts.get(s::_min_scale, 0);
  P.propagation = opts.get(s::_propagation, 2);
  P.patchsize = opts.get(s::_patchsize, 5);
  const int n = (int)keypoints.size();
  std::vector<vint2> kps(n);
  for (int i = 0; i < n; i++) kps[i] = keypoints[i];
  // both pyramids (semi_dense_optical_flow.hpp:70-100) in one launch
  pyramid2d<unsigned char> p1(i1.domain(), P.nscales, 2, s::_border = 2 * P.winsize), p2(i2.domain(), P.nscales, 2, s::_border = 2 * P.winsize);
  std::vector<vppb_img> a(P.nscales), b(P.nscales);
  for (int l = 0; l < P.nscales; l++) { a[l] = *p1[l].device_write(); b[l] = *p2[l].device_write(); }
  vppb_check(vppb_pyrlk_prepare(i1.device_read(), i2.device_read(), a.data(), b.data(), nullptr, P.nscales, 0, nullptr));
  const int64_t wsb = vppb_sdof_workspace_bytes(i1.nrows(), i1.ncols(), &P);
  internals::device_array ws((size_t)wsb), dk((size_t)n * 8), dpos((size_t)n * 8), ddist((size_t)n * 4), dvalid((size_t)n);
  dk.from_host(kps.data(), (size_t)n * 8);
  vppb_check(vppb_sdof_u8(a.data(), b.data(), &P, (const vppb_int2*)dk.ptr(), n, ws.ptr(), wsb, (vppb_int2*)dpos.ptr(), (int32_t*)ddist.ptr(),
                          (unsigned char*)dvalid.ptr(), nullptr));
  std::vector<vint2> pos(n);
  std::vector<int> dist(n);
  std::vector<unsigned char> valid(n);
  dpos.to_host(pos.data(), (size_t)n * 8);
  ddist.to_host(dist.data(), (size_t)n * 4);
  dvalid.to_host(valid.data(), (size_t)n);
  for (int i = 0; i < n; i++)
    if (valid[i]) match_callback(i, pos[i], dist[i]);  // :205-212
}

namespace internals {
// one vppb_sparse_flow_u8 call; `kps` NULL: detect on i1.  cb(i, K1[i], flow[i], distance[i]) for the valid entries, in K1 order.
template <typename O, typename CB>
void sparse_flow_run(const O& opts, const image2d<unsigned char>& i1, const image2d<unsigned char>& i2, const std::vector<vint2>* kps, CB cb) {
  vppb_sof_params P;
  P.detector_th = opts.get(s::_detector_th, 5);  // sparse_optical_flow.hh:45-49
  P.block_size = opts.get(s::_block_size, 5);
  P.winsize = opts.get(s::_winsize, 11);
  P.search_radius = opts.get(s::_search_radius, 100);
  P.cell_width = opts.get(s::_cell_width, 300);  // grid_index.hh:16
  P.subpixelic = opts.get(s::_subpixelic, false) ? 1 : 0;
  P.lk_iterations = opts.get(s::_lk_iterations, 5);
  P.nscales = opts.get(s::_nscales, 3);
  const int n = kps ? (int)kps->size() : -1;
  const int bs = P.block_size > 0 ? P.block_size : 1;
  const int cap = kps ? n : ((i1.nrows() + bs - 1) / bs) * ((i1.ncols() + bs - 1) / bs);
  const int64_t wsb = vppb_sparse_flow_workspace_bytes(i1.nrows(), i1.ncols(), &P, n);
  device_array ws((size_t)wsb), dk((size_t)(kps ? n : 0) * 8), dpos((size_t)cap * 8), dflow((size_t)cap * 8), ddist((size_t)cap * 4), dvalid((size_t)cap);
  if (kps) dk.from_host(kps->data(), (size_t)n * 8);
  int32_t count = 0;
  vppb_check(vppb_sparse_flow_u8(i1.device_read(), i2.device_read(), &P, kps ? (const vppb_int2*)dk.ptr() : nullptr, kps ? n : 0, ws.ptr(), wsb,
                                 (vppb_int2*)dpos.ptr(), (vppb_float2*)dflow.ptr(), (int32_t*)ddist.ptr(), (unsigned char*)dvalid.ptr(), cap, &count,
                                 nullptr));
  std::vector<vint2> pos(count);
  std::vector<vfloat2> flow(count);
  std::vector<int> dist(count);
  std::vector<unsigned char> valid(count);
  dpos.to_host(pos.data(), (size_t)count * 8);
  dflow.to_host(flow.data(), (size_t)count * 8);
  ddist.to_host(dist.data(), (size_t)count * 4);
  dvalid.to_host(valid.data(), (size_t)count);
  for (int i = 0; i < count; i++)
    if (valid[i]) cb(i, pos[i], flow[i], dist[i]);
}
}  // namespace internals

template <typename... OPTS>
void sparse_optical_flow(const image2d<unsigned char>& i1, const image2d<unsigned char>& i2, OPTS... options) {
  auto opts = s::D(options...);
  static_assert(decltype(opts)::has(s::_flow), "sparse_optical_flow: the _flow callback is missing");
  auto f = opts.get(s::_flow, 0);
  internals::sparse_flow_run(opts, i1, i2, nullptr, [&](int, vint2 p, vfloat2 fl, int d) { f(p, fl, d); });
}

template <typename K, typename F, typename... OPTS>
void sparse_optical_flow(const K& keypoints, F match_callback, const image2d<unsigned char>& i1, const image2d<unsigned char>& i2, OPTS... options) {
  auto opts = s::D(options...);
  std::vector<vint2> kps(keypoints.size());
  for (size_t i = 0; i < kps.size(); i++) kps[i] = keypoints[i];
  internals::sparse_flow_run(opts, i1, i2, &kps, [&](int i, vint2 p, vfloat2 fl, int d) {
    match_callback(i, vfloat2((float)p[0] + fl[0], (float)p[1] + fl[1]), d);
  });
}

}  // namespace vpp
