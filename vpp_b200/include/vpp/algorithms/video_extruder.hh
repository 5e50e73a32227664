// video_extruder_init / video_extruder_update: the per-frame keypoint tracker
//   semi-dense optical flow -> merge keypoints that share a spacing cell -> drop weak FAST corners ->
//   every `detector_period` frames: masked blockwise FAST9 re-detection, compact, sync trajectories -> trajectories
// (reference: vpp/algorithms/video_extruder.hh:10-45, video_extruder/video_extruder.hpp:15-135).
//
// The pixel work runs on the GPU (semi_dense_optical_flow, fast9_scores, fast9 through the C-ABI); the keypoint
// container, the merge grid, the detector mask and the trajectories are host-side bookkeeping exactly as in the reference.
// As there, frame2 must carry a border >= 3 filled by the caller (fast9 / fast9_score sample a radius-3 ring).
// Options and defaults (video_extruder.hpp:34-40): _detector_th = 10, _keypoint_spacing = 10, _detector_period = 5,
// _max_trajectory_length = 15, _nscales = 3, _winsize = 9, _propagation = 2.
#pragma once
#include <vector>

#include <vpp/algorithms/fast_detector/fast.hh>
#include <vpp/algorithms/optical_flow.hh>
#include <vpp/core/keypoint_container.hh>
#include <vpp/core/keypoint_trajectory.hh>

namespace vpp {

namespace s {
VPP_DEFINE_SYMBOL(keypoint_spacing)
VPP_DEFINE_SYMBOL(detector_period)
VPP_DEFINE_SYMBOL(max_trajectory_length)
}  // namespace s

struct video_extruder_ctx {  // video_extruder.hh:10-25
  video_extruder_ctx(box2d domain) : keypoints(domain), frame_id(0) {}
  keypoint_container<keypoint<int>, int> keypoints;   // ctx.keypoints[i]: the i-th keypoint
  std::vector<keypoint_trajectory> trajectories;      // ctx.trajectories[i].position_at_frame(j)
  int frame_id;
};

inline video_extruder_ctx video_extruder_init(box2d domain) {  // video_extruder.hpp:15-20
  video_extruder_ctx res(domain);
  res.frame_id = -1;
  return res;
}

namespace internals {
struct keypoint_positions {  // the iod::array_view of video_extruder.hpp:46-47: i -> ctx.keypoints[i].position
  const keypoint_container<keypoint<int>, int>* c;
  size_t size() const { return (size_t)c->size(); }
  vint2 operator[](size_t i) const { return (*c)[(unsigned)i].position; }
};
}  // namespace internals

template <typename... OPTS>
void video_extruder_update(video_extruder_ctx& ctx, const image2d<unsigned char>& frame1, const image2d<unsigned char>& frame2, OPTS... options) {
  ctx.frame_id++;
  auto opts = s::D(options...);
  const int detector_th = opts.get(s::_detector_th, 10);
  const int keypoint_spacing = opts.get(s::_keypoint_spacing, 10);
  const int detector_period = opts.get(s::_detector_period, 5);
  const int max_trajectory_length = opts.get(s::_max_trajectory_length, 15);
  const int nscales = opts.get(s::_nscales, 3);
  const int winsize = opts.get(s::_winsize, 9);
  const int regularisation_niters = opts.get(s::_propagation, 2);
  auto& kps = ctx.keypoints;

  // 1. flow of every container entry, dead ones included (video_extruder.hpp:43-56); the callbacks run serially in
  //    keypoint order: a position inside the frame moves the keypoint (age + 1), anything else removes it
  kps.prepare_matching();
  if (kps.size() > 0)
    semi_dense_optical_flow(internals::keypoint_positions{&kps},
                            [&](int i, vint2 pos, int) {
                              if (frame1.has(pos)) kps.move(i, pos);
                              else kps.remove(i);
                            },
                            frame1, frame2, s::_winsize = winsize, s::_patchsize = 5, s::_propagation = regularisation_niters, s::_nscales = nscales);

  // 2. keypoints that converged into the same spacing cell: the older one survives, equal ages both stay (:59-84)
  {
    const int gr = frame2.nrows() / keypoint_spacing + 2, gc = frame2.ncols() / keypoint_spacing + 2;  // domain + the border of 1
    std::vector<int> idx((size_t)gr * gc, -1);
    for (int i = 0; i < kps.size(); i++) {
      const vint2 cell = kps[i].position / keypoint_spacing;
      int& slot = idx[(size_t)(cell[0] + 1) * gc + (cell[1] + 1)];
      if (slot >= 0) {
        const int other_age = kps[slot].age;  // a copy: the removals below must not change what is compared
        const int other = slot;
        if (other_age < kps[i].age) { kps.remove(other); slot = i; }
        if (other_age > kps[i].age) kps.remove(i);
      } else {
        slot = i;
      }
    }
  }

  // 3. corners that faded: FAST score < 3 (:87-91); one batched launch for all keypoints
  if (kps.size() > 0) {
    std::vector<vint2> where((size_t)kps.size());
    for (int i = 0; i < kps.size(); i++) where[i] = kps[i].position;
    std::vector<int> scores;
    fast9_scores(frame2, detector_th, where, scores);
    for (int i = 0; i < kps.size(); i++)
      if (scores[i] < 3) kps.remove(i);
  }

  // 4. new keypoints away from the existing ones (:94-119).  Mask value 1 seeds FAST's `possible` flags with bit 0
  //    only, i.e. only darker arcs are detected (fast.hpp:310-317).
  if (!(ctx.frame_id % detector_period)) {
    image2d<unsigned char> mask(frame2.nrows(), frame2.ncols(), s::_border = keypoint_spacing);
    mask.host_fill_with_border(1);
    for (int i = 0; i < kps.size(); i++) {
      const int r = kps[i].position[0], c = kps[i].position[1];
      for (int dr = -keypoint_spacing; dr < keypoint_spacing; dr++) {
        unsigned char* row = mask[r + dr];
        for (int dc = -keypoint_spacing; dc < keypoint_spacing; dc++) row[c + dc] = 0;
      }
    }
    const std::vector<vint2> found = fast9(frame2, detector_th, s::_blockwise, s::_block_size = keypoint_spacing, s::_mask = mask);
    for (const vint2& kp : found) kps.add(keypoint<int>(kp));
    kps.compact();
    kps.sync_attributes(ctx.trajectories, keypoint_trajectory(ctx.frame_id));
  }

  // 5. trajectories (:122-133)
  for (int i = 0; i < kps.size(); i++) {
    if (kps[i].alive()) {
      ctx.trajectories[i].move_to(cast<vfloat2>(kps[i].position));
      if (ctx.trajectories[i].size() > max_trajectory_length) ctx.trajectories[i].pop_oldest_position();
    } else {
      ctx.trajectories[i].die();
    }
  }
}

}  // namespace vpp
