// Device-resident keypoint_container<keypoint<int>> + keypoint trajectories for video_extruder (SURVEY 8f N3), and, at the end of
// the file, the descriptor matchers and patch extraction that match keypoints across frames or views (DESIGN §3.8).
// Reference: vpp/core/keypoint_container.hpp:22-200 (add / remove / move / compact / sync_attributes),
// vpp/core/keypoint_trajectory.hh:11-73, vpp/algorithms/video_extruder/video_extruder.hpp:45-133 (the update loop).
//
// The reference keeps the container on the host and walks it serially after every step of video_extruder_update; here
// the arrays (position, velocity, age, trajectory ring) live in HBM and every step of the loop is a kernel, so a frame
// needs no host round trip of keypoints or masks - only the 4-byte entry count crosses PCIe on detection frames (the host
// sizes its launches with it).  All steps reproduce the SERIAL semantics of the reference:
//   flow step    : entry i moves (velocity = new - old, age + 1) or is removed (age = 0)           (:45-56, container :136-167)
//   merge        : entries that share a keypoint_spacing cell: visiting them in index order, the first becomes the cell's
//                  holder; a later entry older than the holder removes it and takes over, a younger one is removed, an
//                  equally old one stays (:59-84).  Closed form per entry i with M = max age of its cell mates before it:
//                  removed  <=>  age_i < M,  or  (no mate before it or age_i > M) and a later mate is older than it.
//   score filter : fast9_score(frame2, th, position) < 3 removes the entry (:87-91)
//   mask         : 1 everywhere incl. the border, 0 in [-s, s)^2 around EVERY entry, dead ones included (:97-109)
//   add/compact  : detections are appended with age 1, dead entries leave, order kept; kept entries keep their trajectory,
//                  new ones start one at this frame (:111-118, keypoint_container.hpp:22-110)
//   trajectories : alive entries push their position and drop the oldest beyond max_trajectory_length, dead ones die (:122-133)
#include "common.cuh"

#include <limits.h>

#include <algorithm>

namespace vppb {

struct Kpc {
  int capacity, max_traj, n;  // n: entries (dead ones included), host copy
  // double-buffered entry arrays (compaction gathers from one set into the other)
  vppb_int2* pos[2];
  vppb_int2* vel[2];
  int* age[2];
  int* tstart[2];
  int* tlen[2];
  int* thead[2];               // ring position of the newest history entry
  unsigned char* talive[2];
  vppb_float2* thist[2];       // capacity x max_traj
  int cur;
  int* map;                    // compaction: new index of an entry or -1
  int* count;                  // device: entry count after the last add / compact
  int* cell_head;              // merge grid: head of the cell's list, next[] links
  int* next;
  unsigned char* removed;
  long long cells_cap;
};

__device__ __forceinline__ int c_div(int a, int b) { return a / b; }  // C++ integer division (truncation)
// An entry outside the frame (only a caller's detection can put one there) is treated like fast9_scores treats an out-of-frame
// keypoint: the merge and the score filter remove it and the mask gets nothing painted for it, so no kernel indexes past its buffers.
__device__ __forceinline__ bool in_frame(vppb_int2 p, int nrows, int ncols) { return p.r >= 0 && p.r < nrows && p.c >= 0 && p.c < ncols; }

__global__ void k_kpc_flow(vppb_int2* pos, vppb_int2* vel, int* age, int n, const vppb_int2* newpos, const unsigned char* valid, int nrows, int ncols) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!valid[i]) continue;
    const vppb_int2 p = newpos[i];
    if (p.r >= 0 && p.r < nrows && p.c >= 0 && p.c < ncols) {
      vel[i] = vppb_int2{p.r - pos[i].r, p.c - pos[i].c};
      pos[i] = p;
      age[i] += 1;
    } else {
      age[i] = 0;
    }
  }
}

__global__ void k_kpc_fill_int(int* a, long long n, int v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) a[i] = v;
}

__global__ void k_kpc_link(const vppb_int2* pos, int n, int nrows, int ncols, int spacing, int stride, int* cell_head, int* next) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!in_frame(pos[i], nrows, ncols)) continue;  // left out of the grid
    const int cell = (c_div(pos[i].r, spacing) + 1) * stride + c_div(pos[i].c, spacing) + 1;
    next[i] = atomicExch(&cell_head[cell], i);
  }
}

__global__ void k_kpc_merge(const vppb_int2* pos, const int* age, int n, int nrows, int ncols, int spacing, int stride, const int* cell_head, const int* next,
                            unsigned char* removed) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!in_frame(pos[i], nrows, ncols)) { removed[i] = 1; continue; }
    const int cell = (c_div(pos[i].r, spacing) + 1) * stride + c_div(pos[i].c, spacing) + 1;
    const int a = age[i];
    int before_max = INT_MIN;
    bool any_before = false, later_older = false;
    for (int j = cell_head[cell]; j >= 0; j = next[j]) {
      if (j < i) { any_before = true; before_max = max(before_max, age[j]); }
      else if (j > i && age[j] > a) later_older = true;
    }
    const bool holder_once = !any_before || a > before_max;
    removed[i] = (unsigned char)((any_before && a < before_max) || (holder_once && later_older));
  }
}

__global__ void k_kpc_apply_removed(int* age, const unsigned char* removed, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (removed[i]) age[i] = 0;
}

__constant__ signed char c_true_ring[16][2] = {{-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}, {0, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3}, {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}};

// fast.hpp:36-77 (true ring), entries with a score under min_score are removed
__global__ void k_kpc_score_filter(Img im, int th, int min_score, const vppb_int2* pos, int* age, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!in_frame(pos[i], im.nrows, im.ncols)) { age[i] = 0; continue; }  // its ring would leave the 3-pixel border
    const unsigned char* p = im.base + (long long)pos[i].r * im.pitch + pos[i].c;
    const int v = *p;
    int sum_inf = 0, sum_sup = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const int diff = v - (int)p[(long long)c_true_ring[k][0] * im.pitch + c_true_ring[k][1]];
      if (diff < -th) sum_inf -= diff;
      else if (diff > th) sum_sup += diff;
    }
    if (max(sum_sup, sum_inf) < min_score) age[i] = 0;
  }
}

// one warp per entry zeroes its 2s x 2s square of the mask (the mask has a border of s pixels, so an entry inside the frame needs
// no clipping; one outside paints nothing)
__global__ void k_kpc_paint(Img mask, const vppb_int2* pos, int n, int s) {
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
    const int r = pos[i].r, c = pos[i].c;
    if (!in_frame(pos[i], mask.nrows, mask.ncols)) continue;
    for (int k = lane; k < 4 * s * s; k += 32) {
      const int dr = k / (2 * s) - s, dc = k % (2 * s) - s;
      mask.base[(long long)(r + dr) * mask.pitch + (c + dc)] = 0;
    }
  }
}

// the first min(count, max_detections, capacity - n) detections enter: a detector's count may exceed what it stored (the total it
// found), and a negative count adds none
__global__ void k_kpc_add(vppb_int2* pos, vppb_int2* vel, int* age, int n, const vppb_int2* det, const int* det_count, int max_detections, int capacity,
                          int* count) {
  const int m = max(0, min(*det_count, min(max_detections, capacity - n)));
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    pos[n + i] = det[i];
    vel[n + i] = vppb_int2{0, 0};
    age[n + i] = 1;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *count = n + m;
}

// exclusive scan of the alive flags of *count entries by ONE CTA: map[i] = new index or -1; count <- survivors
__global__ void __launch_bounds__(1024) k_kpc_scan(const int* age, int* map, int* count) {
  __shared__ int warp_sums[32];
  __shared__ int carry;
  const int n = *count;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = (i < n && age[i] > 0) ? 1 : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int s = warp_sums[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, s, o);
        if (threadIdx.x >= o) s += y;
      }
      warp_sums[threadIdx.x] = s;
    }
    __syncthreads();
    const int warp_prefix = (threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0;
    const int incl = x + warp_prefix + carry;
    if (i < n) map[i] = v ? incl - 1 : -1;
    __syncthreads();
    if (threadIdx.x == 1023) carry = incl;
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x == 0) { map[n] = carry; }  // survivors, picked up by the gather kernel's thread 0
}

struct KpcArrays {
  vppb_int2 *pos, *vel;
  int *age, *tstart, *tlen, *thead;
  unsigned char* talive;
  vppb_float2* thist;
};

// gather the survivors into the other buffer set; entries that had no trajectory yet (index >= n_traj) start one at frame_id
__global__ void k_kpc_gather(KpcArrays src, KpcArrays dst, const int* map, int* count, int n_traj, int frame_id, int max_traj) {
  const int n = *count;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int j = map[i];
    if (j < 0) continue;
    dst.pos[j] = src.pos[i]; dst.vel[j] = src.vel[i]; dst.age[j] = src.age[i];
    if (i < n_traj) {
      dst.tstart[j] = src.tstart[i]; dst.tlen[j] = src.tlen[i]; dst.thead[j] = src.thead[i]; dst.talive[j] = src.talive[i];
      for (int k = 0; k < max_traj; k++) dst.thist[(long long)j * max_traj + k] = src.thist[(long long)i * max_traj + k];
    } else {
      dst.tstart[j] = frame_id; dst.tlen[j] = 0; dst.thead[j] = 0; dst.talive[j] = 1;
    }
  }
}
__global__ void k_kpc_set_count(const int* map, int* count) { *count = map[*count]; }

__global__ void k_kpc_traj(KpcArrays a, int n, int max_traj) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (a.age[i] > 0) {  // move_to: push front; pop the oldest beyond max_traj (keypoint_trajectory.hh)
      const int h = (a.thead[i] + max_traj - 1) % max_traj;  // the ring grows downwards: head = newest
      a.thist[(long long)i * max_traj + h] = vppb_float2{(float)a.pos[i].r, (float)a.pos[i].c};
      a.thead[i] = h;
      a.tlen[i] = min(a.tlen[i] + 1, max_traj);
    } else {
      a.talive[i] = 0;
    }
  }
}

// velocities, and the trajectories newest first with NaN past their length
__global__ void k_kpc_history(KpcArrays a, int n, int max_traj, vppb_int2* vel, vppb_float2* hist) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (vel) vel[i] = a.vel[i];
    if (hist) {
      const int len = a.tlen[i], h = a.thead[i];
      const float nan = __uint_as_float(0x7fc00000u);
      for (int k = 0; k < max_traj; k++)
        hist[(long long)i * max_traj + k] = k < len ? a.thist[(long long)i * max_traj + (h + k) % max_traj] : vppb_float2{nan, nan};
    }
  }
}

__global__ void k_kpc_table(KpcArrays a, int n, int* out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    out[6 * i + 0] = a.pos[i].r; out[6 * i + 1] = a.pos[i].c; out[6 * i + 2] = a.age[i];
    out[6 * i + 3] = a.tstart[i]; out[6 * i + 4] = a.tlen[i]; out[6 * i + 5] = a.talive[i];
  }
}

static KpcArrays arrays(const Kpc* k, int which) {
  return KpcArrays{k->pos[which], k->vel[which], k->age[which], k->tstart[which], k->tlen[which], k->thead[which], k->talive[which], k->thist[which]};
}
static int grid_for(long long n, int threads = 256) {
  long long b = (n + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace vppb

using namespace vppb;

extern "C" {

int vppb_kpc_create(int32_t capacity, int32_t max_trajectory_length, void** handle) {
  VPPB_REQUIRE(handle && capacity > 0 && max_trajectory_length > 0, VPPB_E_ARG, "vppb_kpc_create: bad argument");
  Kpc* k = new Kpc();
  memset(k, 0, sizeof(*k));
  k->capacity = capacity; k->max_traj = max_trajectory_length;
  for (int w = 0; w < 2; w++) {
    VPPB_CUDA(cudaMalloc(&k->pos[w], (size_t)capacity * 8)); VPPB_CUDA(cudaMalloc(&k->vel[w], (size_t)capacity * 8));
    VPPB_CUDA(cudaMalloc(&k->age[w], (size_t)capacity * 4)); VPPB_CUDA(cudaMalloc(&k->tstart[w], (size_t)capacity * 4));
    VPPB_CUDA(cudaMalloc(&k->tlen[w], (size_t)capacity * 4)); VPPB_CUDA(cudaMalloc(&k->thead[w], (size_t)capacity * 4));
    VPPB_CUDA(cudaMalloc(&k->talive[w], (size_t)capacity));
    VPPB_CUDA(cudaMalloc(&k->thist[w], (size_t)capacity * max_trajectory_length * 8));
  }
  VPPB_CUDA(cudaMalloc(&k->map, ((size_t)capacity + 1) * 4));
  VPPB_CUDA(cudaMalloc(&k->next, (size_t)capacity * 4));
  VPPB_CUDA(cudaMalloc(&k->removed, (size_t)capacity));
  VPPB_CUDA(cudaMalloc(&k->count, 4));
  VPPB_CUDA(cudaMemset(k->count, 0, 4));
  *handle = k;
  return VPPB_OK;
}

int vppb_kpc_destroy(void* handle) {
  if (!handle) return VPPB_OK;
  Kpc* k = static_cast<Kpc*>(handle);
  for (int w = 0; w < 2; w++) {
    cudaFree(k->pos[w]); cudaFree(k->vel[w]); cudaFree(k->age[w]); cudaFree(k->tstart[w]); cudaFree(k->tlen[w]); cudaFree(k->thead[w]);
    cudaFree(k->talive[w]); cudaFree(k->thist[w]);
  }
  cudaFree(k->map); cudaFree(k->next); cudaFree(k->removed); cudaFree(k->count); cudaFree(k->cell_head);
  delete k;
  return VPPB_OK;
}

int32_t vppb_kpc_size(void* handle) { return handle ? static_cast<Kpc*>(handle)->n : 0; }
const vppb_int2* vppb_kpc_positions(void* handle) { Kpc* k = static_cast<Kpc*>(handle); return k ? k->pos[k->cur] : nullptr; }

int vppb_kpc_flow_update(void* handle, const vppb_int2* new_pos, const unsigned char* valid, int32_t nrows, int32_t ncols, void* stream) {
  VPPB_REQUIRE(handle, VPPB_E_ARG, "vppb_kpc_flow_update: NULL container");
  Kpc* k = static_cast<Kpc*>(handle);
  if (k->n == 0) return VPPB_OK;
  VPPB_REQUIRE(new_pos && valid, VPPB_E_ARG, "vppb_kpc_flow_update: NULL argument");
  k_kpc_flow<<<grid_for(k->n), 256, 0, as_stream(stream)>>>(k->pos[k->cur], k->vel[k->cur], k->age[k->cur], k->n, new_pos, valid, nrows, ncols);
  VPPB_LAUNCH_CHECK("vppb_kpc_flow_update");
  return VPPB_OK;
}

int vppb_kpc_merge(void* handle, int32_t nrows, int32_t ncols, int32_t spacing, void* stream) {
  VPPB_REQUIRE(handle && spacing > 0, VPPB_E_ARG, "vppb_kpc_merge: bad argument");
  Kpc* k = static_cast<Kpc*>(handle);
  if (k->n == 0) return VPPB_OK;
  const int stride = ncols / spacing + 3;
  const long long cells = (long long)(nrows / spacing + 3) * stride;
  if (cells > k->cells_cap) {
    if (k->cell_head) VPPB_CUDA(cudaFree(k->cell_head));
    VPPB_CUDA(cudaMalloc(&k->cell_head, (size_t)cells * 4));
    k->cells_cap = cells;
  }
  cudaStream_t st = as_stream(stream);
  k_kpc_fill_int<<<grid_for(cells), 256, 0, st>>>(k->cell_head, cells, -1);
  k_kpc_link<<<grid_for(k->n), 256, 0, st>>>(k->pos[k->cur], k->n, nrows, ncols, spacing, stride, k->cell_head, k->next);
  k_kpc_merge<<<grid_for(k->n), 256, 0, st>>>(k->pos[k->cur], k->age[k->cur], k->n, nrows, ncols, spacing, stride, k->cell_head, k->next, k->removed);
  k_kpc_apply_removed<<<grid_for(k->n), 256, 0, st>>>(k->age[k->cur], k->removed, k->n);
  VPPB_LAUNCH_CHECK("vppb_kpc_merge");
  return VPPB_OK;
}

int vppb_kpc_score_filter(void* handle, const vppb_img* img, int32_t th, int32_t min_score, void* stream) {
  VPPB_REQUIRE(handle && img && img->base && img->elem_bytes == 1, VPPB_E_ARG, "vppb_kpc_score_filter: bad argument");
  VPPB_REQUIRE(img->border >= 3, VPPB_E_BORDER, "vppb_kpc_score_filter: border %d < 3", img->border);
  Kpc* k = static_cast<Kpc*>(handle);
  if (k->n == 0) return VPPB_OK;
  k_kpc_score_filter<<<grid_for(k->n), 256, 0, as_stream(stream)>>>(view(img), th, min_score, k->pos[k->cur], k->age[k->cur], k->n);
  VPPB_LAUNCH_CHECK("vppb_kpc_score_filter");
  return VPPB_OK;
}

int vppb_kpc_paint_mask(void* handle, const vppb_img* mask, int32_t spacing, void* stream) {
  VPPB_REQUIRE(handle && mask && mask->base && mask->elem_bytes == 1 && spacing > 0, VPPB_E_ARG, "vppb_kpc_paint_mask: bad argument");
  VPPB_REQUIRE(mask->border >= spacing, VPPB_E_BORDER, "vppb_kpc_paint_mask: the mask needs a border of keypoint_spacing = %d pixels", spacing);
  Kpc* k = static_cast<Kpc*>(handle);
  const unsigned char one = 1;
  int rc = vppb_fill(mask, &one, 1, stream);  // fill_with_border(mask, 1)
  if (rc) return rc;
  if (k->n == 0) return VPPB_OK;
  const long long blocks = ((long long)k->n + 7) / 8;
  k_kpc_paint<<<(int)(blocks < (long long)sm_count() * 16 ? blocks : (long long)sm_count() * 16), 256, 0, as_stream(stream)>>>(view(mask), k->pos[k->cur], k->n, spacing);
  VPPB_LAUNCH_CHECK("vppb_kpc_paint_mask");
  return VPPB_OK;
}

// append the detections (device array + device count, as vppb_fast9_u8_async leaves them), compact, start trajectories for
// the newcomers; reads the new entry count back (4 bytes, one synchronisation) because the host sizes later launches with it
int vppb_kpc_add_and_compact(void* handle, const vppb_int2* detections, const int32_t* det_count_dev, int32_t max_detections, int32_t frame_id, void* stream) {
  VPPB_REQUIRE(handle && det_count_dev && max_detections >= 0 && (detections || max_detections == 0), VPPB_E_ARG, "vppb_kpc_add_and_compact: NULL argument");
  Kpc* k = static_cast<Kpc*>(handle);
  cudaStream_t st = as_stream(stream);
  const int cur = k->cur, n_traj = k->n;
  const long long upper = std::min<long long>((long long)k->n + max_detections, k->capacity);
  k_kpc_add<<<grid_for(std::max(1, max_detections)), 256, 0, st>>>(k->pos[cur], k->vel[cur], k->age[cur], k->n, detections, det_count_dev, max_detections, k->capacity, k->count);
  k_kpc_scan<<<1, 1024, 0, st>>>(k->age[cur], k->map, k->count);
  k_kpc_gather<<<grid_for(std::max<long long>(1, upper)), 256, 0, st>>>(arrays(k, cur), arrays(k, cur ^ 1), k->map, k->count, n_traj, frame_id, k->max_traj);
  k_kpc_set_count<<<1, 1, 0, st>>>(k->map, k->count);
  VPPB_LAUNCH_CHECK("vppb_kpc_add_and_compact");
  int n = 0;
  VPPB_CUDA(cudaMemcpyAsync(&n, k->count, 4, cudaMemcpyDeviceToHost, st));
  VPPB_CUDA(cudaStreamSynchronize(st));
  k->cur = cur ^ 1;
  k->n = n;
  return VPPB_OK;
}

int vppb_kpc_trajectories_update(void* handle, void* stream) {
  VPPB_REQUIRE(handle, VPPB_E_ARG, "vppb_kpc_trajectories_update: NULL container");
  Kpc* k = static_cast<Kpc*>(handle);
  if (k->n == 0) return VPPB_OK;
  k_kpc_traj<<<grid_for(k->n), 256, 0, as_stream(stream)>>>(arrays(k, k->cur), k->n, k->max_traj);
  VPPB_LAUNCH_CHECK("vppb_kpc_trajectories_update");
  return VPPB_OK;
}

int vppb_kpc_history(void* handle, vppb_int2* velocity_dev, vppb_float2* history_dev, void* stream) {
  VPPB_REQUIRE(handle, VPPB_E_ARG, "vppb_kpc_history: NULL container");
  Kpc* k = static_cast<Kpc*>(handle);
  if (k->n == 0 || (!velocity_dev && !history_dev)) return VPPB_OK;
  k_kpc_history<<<grid_for(k->n), 256, 0, as_stream(stream)>>>(arrays(k, k->cur), k->n, k->max_traj, velocity_dev, history_dev);
  VPPB_LAUNCH_CHECK("vppb_kpc_history");
  return VPPB_OK;
}

// rows of 6 ints per entry (row, col, age, trajectory start frame, trajectory length, trajectory alive) into a DEVICE buffer
int vppb_kpc_state_table(void* handle, int32_t* table_dev, void* stream) {
  VPPB_REQUIRE(handle, VPPB_E_ARG, "vppb_kpc_state_table: NULL container");
  Kpc* k = static_cast<Kpc*>(handle);
  if (k->n == 0) return VPPB_OK;
  VPPB_REQUIRE(table_dev, VPPB_E_ARG, "vppb_kpc_state_table: NULL output");
  k_kpc_table<<<grid_for(k->n), 256, 0, as_stream(stream)>>>(arrays(k, k->cur), k->n, table_dev);
  VPPB_LAUNCH_CHECK("vppb_kpc_state_table");
  return VPPB_OK;
}

}  // extern "C"

// ==== descriptor matching and patch extraction ====================================================================================
// Reference: vpp/algorithms/descriptor_matcher/* and vpp/core/patch.hh:32-47.  The brute-force SAD matcher, the grid-local SAD
// matcher and the gather that builds descriptors from image windows: the GPU end of the keypoint pipeline whose container lives
// above (FAST -> extract_patches -> match across frames).  Descriptors are the rows of a pitched image (one descriptor per row,
// ncols = its length) of unsigned char or int.  See DESIGN §3.8.
namespace vppb {

// ---- SAD of one pair of elements ---------------------------------------------------------------------------------------------
// unsigned char: four byte pairs of two packed words; int: |a - b| as max - min in unsigned arithmetic, which is exact whenever
// the full SAD fits in int (the only case in which the reference's `int` sum is defined)
__device__ __forceinline__ unsigned sad_word(unsigned a, unsigned b, unsigned acc) { return __vsadu4(a, b) + acc; }
__device__ __forceinline__ unsigned sad_word(int a, int b, unsigned acc) { return acc + ((unsigned)max(a, b) - (unsigned)min(a, b)); }

// ---- brute force -------------------------------------------------------------------------------------------------------------
// One thread per query, BF_Q queries per CTA, the trains of one split streamed through shared memory BF_T at a time.  A "word" is
// 4 packed bytes of an unsigned char descriptor or one int; descriptors are zero-padded to whole words (|0 - 0| adds nothing).
// The query's words live in registers, QW at a time; a descriptor longer than QW words goes in chunks whose partial sums wait
// in shared memory (only the QW = 32 instantiation chunks).
constexpr int BF_Q = 128;
constexpr int BF_T = 64;
constexpr int BF_QW_MAX = 32;

// word w of descriptor row `row` (zero beyond the descriptor)
__device__ __forceinline__ unsigned bf_word_u8(const unsigned char* row, int D, int w) {
  unsigned v = 0;
  const int k0 = 4 * w;
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (k0 + k < D) v |= (unsigned)row[k0 + k] << (8 * k);
  return v;
}

template <typename W>
__device__ __forceinline__ W bf_load(const Img& im, int row, int D, int w);
template <>
__device__ __forceinline__ unsigned bf_load<unsigned>(const Img& im, int row, int D, int w) {
  return bf_word_u8(im.base + (long long)row * im.pitch, D, w);
}
template <>
__device__ __forceinline__ int bf_load<int>(const Img& im, int row, int D, int w) {
  return w < D ? reinterpret_cast<const int*>(im.base + (long long)row * im.pitch)[w] : 0;
}

// W: unsigned (packed unsigned char) or int.  CTA b handles queries (b % nqb) * BF_Q.. and trains [split * span, + span) of
// split b / nqb, and merges each query's minimum into keys[i] = (distance << 32 | train) with atomicMin.
template <typename W, int QW>
__global__ void __launch_bounds__(BF_Q) k_bf_sad(Img q, Img t, int nq, int nt, int D, int words, int nqb, int span,
                                                 unsigned long long* keys) {
  __align__(16) __shared__ W tile[BF_T][QW];
  __shared__ unsigned partial[QW == BF_QW_MAX ? BF_T * BF_Q : 1];
  const int qb = blockIdx.x % nqb, split = blockIdx.x / nqb;
  const int i = qb * BF_Q + threadIdx.x;
  const int j0 = split * span, j1 = min(nt, j0 + span);
  const int nchunks = (words + QW - 1) / QW;
  W qr[QW];
  unsigned best = 0xffffffffu;
  int best_j = -1;
  for (int jt = j0; jt < j1; jt += BF_T) {
    for (int c = 0; c < nchunks; c++) {
      __syncthreads();  // the previous tile / chunk has been read by every thread
      for (int e = threadIdx.x; e < BF_T * QW; e += BF_Q) {
        const int k = e / QW, w = e - k * QW;
        tile[k][w] = (jt + k < j1 && c * QW + w < words) ? bf_load<W>(t, jt + k, D, c * QW + w) : W(0);
      }
      if (jt == j0 || nchunks > 1) {
#pragma unroll
        for (int w = 0; w < QW; w++) qr[w] = (i < nq && c * QW + w < words) ? bf_load<W>(q, i, D, c * QW + w) : W(0);
      }
      __syncthreads();
      const int kn = min(BF_T, j1 - jt);
      for (int k = 0; k < kn; k++) {
        unsigned s = 0;
#pragma unroll
        for (int w = 0; w < QW; w++) s = sad_word(qr[w], tile[k][w], s);
        if (QW == BF_QW_MAX && nchunks > 1) {
          unsigned* p = &partial[k * BF_Q + threadIdx.x];
          if (c > 0) s += *p;
          if (c + 1 < nchunks) {
            *p = s;
            continue;
          }
        }
        if (s < best) {  // trains in increasing order, strict <: ties keep the lowest train index
          best = s;
          best_j = jt + k;
        }
      }
    }
  }
  if (i < nq && best_j >= 0) atomicMin(&keys[i], ((unsigned long long)best << 32) | (unsigned)best_j);
}

// keys -> (index, distance); a query no train reached gets (-1, INT32_MAX)
__global__ void __launch_bounds__(256) k_match_unpack(const unsigned long long* keys, int n, int32_t* index, int32_t* dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  index[i] = k == ~0ull ? -1 : (int32_t)(unsigned)(k & 0xffffffffu);
  dist[i] = k == ~0ull ? 0x7fffffff : (int32_t)(unsigned)(k >> 32);
}

__global__ void __launch_bounds__(256) k_fill_u64(unsigned long long* p, int n, unsigned long long v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

struct BfPlan {
  int words, qw, nqb, span, splits;
};

static BfPlan bf_plan(int nq, int nt, int D, int elem) {
  BfPlan p;
  p.words = elem == 1 ? (D + 3) / 4 : D;
  p.qw = p.words <= 4 ? 4 : p.words <= 8 ? 8 : p.words <= 12 ? 12 : p.words <= 16 ? 16 : p.words <= 24 ? 24 : 32;
  p.nqb = (nq + BF_Q - 1) / BF_Q;
  // split the trains until there are 16 CTAs per SM (a full SM of 128-thread CTAs: each thread is one long dependent chain of
  // VABSDIFF4s, so issue needs every warp slot), each split a whole number of train tiles
  const int tiles = (nt + BF_T - 1) / BF_T;
  const int want = std::min(std::max(tiles, 1), std::max(1, (16 * sm_count() + p.nqb - 1) / std::max(p.nqb, 1)));
  const int per = (std::max(tiles, 1) + want - 1) / want;
  p.span = per * BF_T;
  p.splits = (tiles + per - 1) / per;
  return p;
}

template <typename W>
static void bf_launch(const BfPlan& p, const Img& q, const Img& t, int nq, int nt, int D, unsigned long long* keys, cudaStream_t st) {
  const int grid = p.nqb * p.splits;
  switch (p.qw) {
    case 4: k_bf_sad<W, 4><<<grid, BF_Q, 0, st>>>(q, t, nq, nt, D, p.words, p.nqb, p.span, keys); break;
    case 8: k_bf_sad<W, 8><<<grid, BF_Q, 0, st>>>(q, t, nq, nt, D, p.words, p.nqb, p.span, keys); break;
    case 12: k_bf_sad<W, 12><<<grid, BF_Q, 0, st>>>(q, t, nq, nt, D, p.words, p.nqb, p.span, keys); break;
    case 16: k_bf_sad<W, 16><<<grid, BF_Q, 0, st>>>(q, t, nq, nt, D, p.words, p.nqb, p.span, keys); break;
    case 24: k_bf_sad<W, 24><<<grid, BF_Q, 0, st>>>(q, t, nq, nt, D, p.words, p.nqb, p.span, keys); break;
    default: k_bf_sad<W, 32><<<grid, BF_Q, 0, st>>>(q, t, nq, nt, D, p.words, p.nqb, p.span, keys); break;
  }
}

// ---- grid-local --------------------------------------------------------------------------------------------------------------
// Workspace: header {max cell row, max cell col}, then two (key, train) arrays of ntrain entries for the radix sort's ping-pong.
// key = cell row << 32 | cell col; a train at a coordinate <= -s gets the row max + 1, beyond every clamped window.
constexpr int LM_SORT_THREADS = 1024;
constexpr int LM_WARPS_PER_CTA = 8;

struct LmWs {
  int* hdr;
  unsigned long long *key_a, *key_b;
  int *idx_a, *idx_b;
};

static int64_t lm_align(int64_t n) { return (n + 255) & ~(int64_t)255; }

static int64_t lm_ws_bytes(int nt) {
  return lm_align(16) + 2 * lm_align((int64_t)nt * 8) + 2 * lm_align((int64_t)nt * 4);
}

static LmWs lm_ws(void* base, int nt) {
  unsigned char* p = static_cast<unsigned char*>(base);
  LmWs w;
  w.hdr = reinterpret_cast<int*>(p);
  p += lm_align(16);
  w.key_a = reinterpret_cast<unsigned long long*>(p);
  p += lm_align((int64_t)nt * 8);
  w.key_b = reinterpret_cast<unsigned long long*>(p);
  p += lm_align((int64_t)nt * 8);
  w.idx_a = reinterpret_cast<int*>(p);
  p += lm_align((int64_t)nt * 4);
  w.idx_b = reinterpret_cast<int*>(p);
  return w;
}

__device__ __forceinline__ int bits_of(unsigned v) { return v ? 32 - __clz((int)v) : 0; }

// One CTA: cell keys, then a stable LSD radix sort on 8-bit digits of only the bits the largest cell row and column use.  The
// rank of an item among the equal digits of its 1024-item tile comes from eight ballots per warp plus per-warp digit counts, so
// items keep their input order (train index) inside a cell.  The result ends in key_a / idx_a.
__global__ void __launch_bounds__(LM_SORT_THREADS) k_lm_sort(const vppb_int2* tpos, int nt, int s, LmWs w) {
  __shared__ int hist[256];
  __shared__ int wcount[LM_SORT_THREADS / 32][256];
  __shared__ int maxr, maxc;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    maxr = -1;
    maxc = -1;
  }
  __syncthreads();
  for (int j = tid; j < nt; j += LM_SORT_THREADS) {
    const vppb_int2 p = tpos[j];
    if (p.r > -s && p.c > -s) {  // a coordinate in (-s, 0) truncates to cell 0, as the reference's p / s
      atomicMax(&maxr, p.r / s);
      atomicMax(&maxc, p.c / s);
    }
  }
  __syncthreads();
  const int mr = maxr, mc = maxc;
  for (int j = tid; j < nt; j += LM_SORT_THREADS) {
    const vppb_int2 p = tpos[j];
    const bool ok = p.r > -s && p.c > -s;
    const unsigned cr = ok ? (unsigned)(p.r / s) : (unsigned)mr + 1u, cc = ok ? (unsigned)(p.c / s) : 0u;
    w.key_a[j] = ((unsigned long long)cr << 32) | cc;
    w.idx_a[j] = j;
  }
  if (tid == 0) {
    w.hdr[0] = mr;
    w.hdr[1] = mc;
  }
  const int low_passes = (bits_of((unsigned)max(mc, 0)) + 7) / 8, high_passes = (bits_of((unsigned)mr + 1u) + 7) / 8;
  unsigned long long *ks = w.key_a, *kd = w.key_b;
  int *is = w.idx_a, *id = w.idx_b;
  for (int pass = 0; pass < low_passes + high_passes; pass++) {
    const int shift = pass < low_passes ? 8 * pass : 32 + 8 * (pass - low_passes);
    __syncthreads();  // the previous pass's scatter is complete
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int j = tid; j < nt; j += LM_SORT_THREADS) atomicAdd(&hist[(int)((ks[j] >> shift) & 255)], 1);
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      for (int d = 0; d < 256; d++) {
        const int c = hist[d];
        hist[d] = run;
        run += c;
      }
    }
    for (int t0 = 0; t0 < nt; t0 += LM_SORT_THREADS) {
      const int j = t0 + tid;
      const bool has = j < nt;
      const unsigned long long k = has ? ks[j] : 0ull;
      const int d = (int)((k >> shift) & 255);
      unsigned peers = __ballot_sync(0xffffffffu, has);
#pragma unroll
      for (int b = 0; b < 8; b++) {
        const unsigned m = __ballot_sync(0xffffffffu, (d >> b) & 1);
        peers &= ((d >> b) & 1) ? m : ~m;
      }
      const int rank = __popc(peers & ((1u << lane) - 1u));
      __syncthreads();  // hist holds this tile's bases; wcount is free
      for (int e = tid; e < (LM_SORT_THREADS / 32) * 256; e += LM_SORT_THREADS) wcount[e >> 8][e & 255] = 0;
      __syncthreads();
      if (has && rank == 0) wcount[warp][d] = __popc(peers);
      __syncthreads();
      if (tid < 256) {
        int run = hist[tid];
        for (int x = 0; x < LM_SORT_THREADS / 32; x++) {
          const int c = wcount[x][tid];
          wcount[x][tid] = run;
          run += c;
        }
        hist[tid] = run;
      }
      __syncthreads();
      if (has) {
        const int dst = wcount[warp][d] + rank;
        kd[dst] = k;
        id[dst] = is[j];
      }
    }
    unsigned long long* tk = ks;
    ks = kd;
    kd = tk;
    int* ti = is;
    is = id;
    id = ti;
  }
  if (ks != w.key_a) {  // an odd number of passes: bring the result home
    __syncthreads();
    for (int j = tid; j < nt; j += LM_SORT_THREADS) {
      w.key_a[j] = ks[j];
      w.idx_a[j] = is[j];
    }
  }
}

// first position in keys[0, n) whose key is >= k
__device__ __forceinline__ int lower_bound_u64(const unsigned long long* keys, int n, unsigned long long k) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// truncating (C) division of a 64-bit numerator, clamped into int
__device__ __forceinline__ long long tdiv(long long a, int s) { return a / s; }

template <typename E, bool WORDS>
__device__ __forceinline__ unsigned lm_sad(const unsigned char* a, const unsigned char* b, int D) {
  unsigned s = 0;
  if (sizeof(E) == 4) {
    const int* x = reinterpret_cast<const int*>(a);
    const int* y = reinterpret_cast<const int*>(b);
    for (int k = 0; k < D; k++) s = sad_word(__ldg(x + k), __ldg(y + k), s);
  } else if (WORDS) {
    const unsigned* x = reinterpret_cast<const unsigned*>(a);
    const unsigned* y = reinterpret_cast<const unsigned*>(b);
    int k = 0;
    for (; 4 * k + 3 < D; k++) s = __vsadu4(__ldg(x + k), __ldg(y + k)) + s;
    for (int e = 4 * k; e < D; e++) s += (unsigned)abs((int)__ldg(a + e) - (int)__ldg(b + e));
  } else {
    for (int e = 0; e < D; e++) s += (unsigned)abs((int)__ldg(a + e) - (int)__ldg(b + e));
  }
  return s;
}

// One warp per query: the window's cell rows one at a time, each a contiguous run of the sorted trains found by two binary
// searches, its candidates spread over the lanes.  Each lane keeps min(distance << 32 | sorted position); the sorted order is
// (cell row, cell col, train index), so the smallest key is the tie rule itself.
template <typename E, bool WORDS>
__global__ void __launch_bounds__(32 * LM_WARPS_PER_CTA) k_lm_query(Img q, Img t, const vppb_int2* qpos, int nq, int nt, int D, int R,
                                                                   int s, LmWs w, int32_t* index, int32_t* dist) {
  const int qi = blockIdx.x * LM_WARPS_PER_CTA + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (qi >= nq) return;
  const int mr = w.hdr[0], mc = w.hdr[1];
  const vppb_int2 p = qpos[qi];
  const long long r0 = max(0LL, tdiv((long long)p.r - R, s)), r1 = min((long long)mr, tdiv((long long)p.r + R, s));
  const long long c0 = max(0LL, tdiv((long long)p.c - R, s)), c1 = min((long long)mc, tdiv((long long)p.c + R, s));
  const unsigned char* qrow = q.base + (long long)qi * q.pitch;
  unsigned long long best = ~0ull;
  for (long long cr = r0; cr <= r1 && c0 <= c1; cr++) {
    const int lo = lower_bound_u64(w.key_a, nt, ((unsigned long long)cr << 32) | (unsigned long long)c0);
    const int hi = lower_bound_u64(w.key_a, nt, ((unsigned long long)cr << 32) | (unsigned long long)(c1 + 1));
    for (int x = lo + lane; x < hi; x += 32) {
      const unsigned d = lm_sad<E, WORDS>(qrow, t.base + (long long)w.idx_a[x] * t.pitch, D);
      best = min(best, ((unsigned long long)d << 32) | (unsigned)x);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) {
    index[qi] = best == ~0ull ? -1 : w.idx_a[(int)(best & 0xffffffffu)];
    dist[qi] = best == ~0ull ? 0x7fffffff : (int32_t)(unsigned)(best >> 32);
  }
}

// ---- patch extraction --------------------------------------------------------------------------------------------------------
// One warp per keypoint: output row k = the winsize x winsize window of `img` centred on kps[k], row-major from element 0, or
// zeros where the window leaves the domain plus border.
template <typename E>
__global__ void __launch_bounds__(256) k_extract_patches(Img img, const vppb_int2* kps, int n, int winsize, Img out) {
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= n) return;
  const vppb_int2 p = kps[k];
  const int h = winsize / 2;
  const long long b = img.border;
  const bool inside = (long long)p.r - h >= -b && (long long)p.r - h + winsize - 1 <= img.nrows - 1 + b && (long long)p.c - h >= -b &&
                      (long long)p.c - h + winsize - 1 <= img.ncols - 1 + b;
  E* o = reinterpret_cast<E*>(out.base + (long long)k * out.pitch);
  const int n2 = winsize * winsize;
  for (int e = lane; e < n2; e += 32) {
    E v = E(0);
    if (inside) {
      const int r = e / winsize, c = e - r * winsize;
      v = reinterpret_cast<const E*>(img.base + (long long)(p.r - h + r) * img.pitch)[p.c - h + c];
    }
    o[e] = v;
  }
}

// ---- host checks ---------------------------------------------------------------------------------------------------------------
static bool desc_ok(const vppb_img* d) { return d && (d->nrows == 0 || d->base) && d->nrows >= 0; }

static int check_descriptors(const char* fn, const vppb_img* q, const vppb_img* t) {
  VPPB_REQUIRE(desc_ok(q) && desc_ok(t), VPPB_E_ARG, "%s: NULL descriptor image", fn);
  VPPB_REQUIRE((q->elem_bytes == 1 || q->elem_bytes == 4) && q->elem_bytes == t->elem_bytes, VPPB_E_ARG,
               "%s: unsigned char or int descriptors of one type expected (elem_bytes %d and %d)", fn, q->elem_bytes, t->elem_bytes);
  VPPB_REQUIRE(q->ncols == t->ncols && q->ncols >= 1, VPPB_E_ARG, "%s: descriptor lengths %d and %d", fn, q->ncols, t->ncols);
  VPPB_REQUIRE((int64_t)q->ncols * q->elem_bytes <= q->pitch || q->nrows <= 1, VPPB_E_ARG, "%s: query pitch %d < row bytes", fn, q->pitch);
  VPPB_REQUIRE((int64_t)t->ncols * t->elem_bytes <= t->pitch || t->nrows <= 1, VPPB_E_ARG, "%s: train pitch %d < row bytes", fn, t->pitch);
  VPPB_REQUIRE(q->elem_bytes == 1 || ((uintptr_t)q->base % 4 == 0 && q->pitch % 4 == 0 && (uintptr_t)t->base % 4 == 0 && t->pitch % 4 == 0),
               VPPB_E_ARG, "%s: int descriptors need 4-byte aligned rows", fn);
  return VPPB_OK;
}

}  // namespace vppb

using namespace vppb;

extern "C" {

int64_t vppb_match_bruteforce_sad_workspace_bytes(int32_t nquery, int32_t ntrain, int32_t ncols) {
  (void)ntrain;
  (void)ncols;
  return nquery > 0 ? (int64_t)nquery * 8 : 0;
}

int vppb_match_bruteforce_sad(const vppb_img* query, const vppb_img* train, void* workspace, int64_t workspace_bytes, int32_t* index_out,
                              int32_t* dist_out, void* stream) {
  const char* fn = "vppb_match_bruteforce_sad";
  const int rc = check_descriptors(fn, query, train);
  if (rc) return rc;
  const int nq = query->nrows, nt = train->nrows, D = query->ncols;
  VPPB_REQUIRE(nq == 0 || (index_out && dist_out), VPPB_E_ARG, "%s: NULL output", fn);
  const int64_t need = vppb_match_bruteforce_sad_workspace_bytes(nq, nt, D);
  VPPB_REQUIRE(need == 0 || (workspace && workspace_bytes >= need && (uintptr_t)workspace % 8 == 0), VPPB_E_ARG,
               "%s: workspace %lld < %lld bytes (or not 8-byte aligned)", fn, (long long)workspace_bytes, (long long)need);
  if (nq == 0) return VPPB_OK;
  cudaStream_t st = as_stream(stream);
  unsigned long long* keys = static_cast<unsigned long long*>(workspace);
  k_fill_u64<<<(nq + 255) / 256, 256, 0, st>>>(keys, nq, ~0ull);
  if (nt > 0) {
    const BfPlan p = bf_plan(nq, nt, D, query->elem_bytes);
    if (query->elem_bytes == 1) bf_launch<unsigned>(p, view(query), view(train), nq, nt, D, keys, st);
    else bf_launch<int>(p, view(query), view(train), nq, nt, D, keys, st);
  }
  k_match_unpack<<<(nq + 255) / 256, 256, 0, st>>>(keys, nq, index_out, dist_out);
  VPPB_LAUNCH_CHECK(fn);
  return VPPB_OK;
}

int64_t vppb_match_local_sad_workspace_bytes(int32_t nquery, int32_t ntrain, int32_t ncols, int32_t search_radius, int32_t cell_width) {
  (void)nquery;
  (void)ncols;
  (void)search_radius;
  (void)cell_width;
  return ntrain >= 0 ? lm_ws_bytes(ntrain) : 0;
}

int vppb_match_local_sad(const vppb_img* query, const vppb_img* train, const vppb_int2* query_positions, const vppb_int2* train_positions,
                         int32_t search_radius, int32_t cell_width, void* workspace, int64_t workspace_bytes, int32_t* index_out,
                         int32_t* dist_out, void* stream) {
  const char* fn = "vppb_match_local_sad";
  const int rc = check_descriptors(fn, query, train);
  if (rc) return rc;
  const int nq = query->nrows, nt = train->nrows, D = query->ncols;
  VPPB_REQUIRE(cell_width >= 1 && search_radius >= 0, VPPB_E_ARG, "%s: cell_width %d must be >= 1 and search_radius %d >= 0", fn,
               cell_width, search_radius);
  VPPB_REQUIRE((nq == 0 || (query_positions && index_out && dist_out)) && (nt == 0 || train_positions), VPPB_E_ARG,
               "%s: NULL positions or output", fn);
  const int64_t need = lm_ws_bytes(nt);
  VPPB_REQUIRE(workspace && workspace_bytes >= need && (uintptr_t)workspace % 256 == 0, VPPB_E_ARG,
               "%s: workspace %lld < %lld bytes (or not 256-byte aligned)", fn, (long long)workspace_bytes, (long long)need);
  if (nq == 0) return VPPB_OK;
  cudaStream_t st = as_stream(stream);
  const LmWs w = lm_ws(workspace, nt);
  k_lm_sort<<<1, LM_SORT_THREADS, 0, st>>>(train_positions, nt, cell_width, w);
  const int grid = (nq + LM_WARPS_PER_CTA - 1) / LM_WARPS_PER_CTA, block = 32 * LM_WARPS_PER_CTA;
  const Img vq = view(query), vt = view(train);
  const bool words = (uintptr_t)query->base % 4 == 0 && query->pitch % 4 == 0 && (uintptr_t)train->base % 4 == 0 && train->pitch % 4 == 0;
  if (query->elem_bytes == 4)
    k_lm_query<int, true><<<grid, block, 0, st>>>(vq, vt, query_positions, nq, nt, D, search_radius, cell_width, w, index_out, dist_out);
  else if (words)
    k_lm_query<unsigned char, true><<<grid, block, 0, st>>>(vq, vt, query_positions, nq, nt, D, search_radius, cell_width, w, index_out, dist_out);
  else
    k_lm_query<unsigned char, false><<<grid, block, 0, st>>>(vq, vt, query_positions, nq, nt, D, search_radius, cell_width, w, index_out, dist_out);
  VPPB_LAUNCH_CHECK(fn);
  return VPPB_OK;
}

int vppb_extract_patches(const vppb_img* img, const vppb_int2* keypoints, int32_t n, int32_t winsize, const vppb_img* out, void* stream) {
  const char* fn = "vppb_extract_patches";
  VPPB_REQUIRE(img && out && img->base && n >= 0 && (n == 0 || keypoints), VPPB_E_ARG, "%s: NULL argument or negative count", fn);
  VPPB_REQUIRE(winsize >= 1 && winsize <= 4096, VPPB_E_ARG, "%s: winsize %d out of [1, 4096]", fn, winsize);
  VPPB_REQUIRE((img->elem_bytes == 1 || img->elem_bytes == 4) && out->elem_bytes == img->elem_bytes, VPPB_E_ARG,
               "%s: unsigned char or int image and patches of the same type expected", fn);
  VPPB_REQUIRE(out->nrows == n && out->ncols == winsize * winsize && (n == 0 || out->base), VPPB_E_ARG,
               "%s: the output must be %d x %d", fn, n, winsize * winsize);
  VPPB_REQUIRE(img->elem_bytes == 1 || ((uintptr_t)img->base % 4 == 0 && img->pitch % 4 == 0 && (uintptr_t)out->base % 4 == 0 &&
                                        out->pitch % 4 == 0), VPPB_E_ARG, "%s: int images need 4-byte aligned rows", fn);
  VPPB_REQUIRE(img->border >= winsize / 2, VPPB_E_BORDER, "%s: input border %d < winsize / 2 = %d", fn, img->border, winsize / 2);
  if (n == 0) return VPPB_OK;
  cudaStream_t st = as_stream(stream);
  const int grid = (n + 7) / 8;
  if (img->elem_bytes == 1) k_extract_patches<unsigned char><<<grid, 256, 0, st>>>(view(img), keypoints, n, winsize, view(out));
  else k_extract_patches<int><<<grid, 256, 0, st>>>(view(img), keypoints, n, winsize, view(out));
  VPPB_LAUNCH_CHECK(fn);
  return VPPB_OK;
}

}  // extern "C"
