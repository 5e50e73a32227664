// The remaining neighbourhood operators of the path: the 3x3 stencils lbp_transform and local_maxima_filter (SURVEY 8(f) N4), and the
// chamfer distance transforms, whose 3x3 / 5x5 masks the reference runs in serial raster order like local_maxima_filter.
// Reference: vpp/algorithms/lbp/lbp_transform.hh:7-38, vpp/algorithms/fast_detector/fast.hpp:555-575,
// vpp/algorithms/distance_transforms/distance_transforms.hh:86-152.
#include <algorithm>

#include "common.cuh"

namespace vppb {

// ---- lbp_transform (unsigned char -> unsigned char) ---------------------------------------------------------------------------
// bit k of out(r, c) = neighbour k > centre, neighbours in the order (-1,-1) (-1,0) (-1,1) (0,-1) (0,1) (1,-1) (1,0) (1,1).
// HBM-bound (1 B in + 1 B out per pixel).  A thread owns 16 consecutive pixels of LBP_ROWS consecutive rows: it slides a window of
// three 16-byte row vectors down the image (each input row is loaded once per thread), forms the left / right neighbours of a row by
// funnel shifts across the four words (+ one byte on either side) and evaluates four pixels per packed byte compare.
constexpr int LBP_ROWS = 4;

struct LbpRow { uint32_t w[4]; uint32_t left, right; };  // bytes x0 .. x0+15, the byte before (in bits 24-31) and the byte after (bits 0-7)

__device__ __forceinline__ LbpRow lbp_load(const unsigned char* row, int x0) {
  LbpRow v;
  const uint4 q = *reinterpret_cast<const uint4*>(row + x0);
  v.w[0] = q.x; v.w[1] = q.y; v.w[2] = q.z; v.w[3] = q.w;
  v.left = (uint32_t)row[x0 - 1] << 24;
  v.right = (uint32_t)row[x0 + 16];
  return v;
}
// word k of the row shifted so that byte i holds pixel i - 1 (L) / pixel i + 1 (R)
__device__ __forceinline__ uint32_t lbp_l(const LbpRow& v, int k) { return __funnelshift_l(k ? v.w[k - 1] : v.left, v.w[k], 8); }
__device__ __forceinline__ uint32_t lbp_r(const LbpRow& v, int k) { return __funnelshift_r(v.w[k], k < 3 ? v.w[k + 1] : v.right, 8); }

__device__ __forceinline__ unsigned char lbp_scalar(const unsigned char* r0, const unsigned char* r1, const unsigned char* r2, int i) {
  const int c = r1[i];
  return (unsigned char)(((r0[i - 1] > c) << 0) + ((r0[i] > c) << 1) + ((r0[i + 1] > c) << 2) + ((r1[i - 1] > c) << 3) + ((r1[i + 1] > c) << 4) +
                         ((r2[i - 1] > c) << 5) + ((r2[i] > c) << 6) + ((r2[i + 1] > c) << 7));
}

template <bool VEC>
__global__ void __launch_bounds__(256) k_lbp_u8(Img in, Img out, int xthreads) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int xt = (int)(tid % xthreads);
  const int r_first = (int)(tid / xthreads) * LBP_ROWS;
  if (r_first >= in.nrows) return;
  const int x0 = xt * 16;
  const int r_end = min(r_first + LBP_ROWS, in.nrows);
  if (VEC && x0 + 16 <= in.ncols) {
    // all LBP_ROWS + 2 input rows of the thread are requested before the first is used: one memory latency per thread, not one per row
    LbpRow v[LBP_ROWS + 2];
#pragma unroll
    for (int j = 0; j < LBP_ROWS + 2; j++) {
      const int r = min(r_first - 1 + j, in.nrows);  // rows below the bottom border row are not read (nor used)
      v[j] = lbp_load(in.base + (long long)r * in.pitch, x0);
    }
#pragma unroll
    for (int j = 0; j < LBP_ROWS; j++) {
      const int r = r_first + j;
      if (r >= r_end) break;
      const LbpRow &a = v[j], &b = v[j + 1], &c = v[j + 2];
      uint32_t o[4];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const uint32_t ctr = b.w[k];
        uint32_t acc = __vcmpgtu4(lbp_l(a, k), ctr) & 0x01010101u;
        acc |= __vcmpgtu4(a.w[k], ctr) & 0x02020202u;
        acc |= __vcmpgtu4(lbp_r(a, k), ctr) & 0x04040404u;
        acc |= __vcmpgtu4(lbp_l(b, k), ctr) & 0x08080808u;
        acc |= __vcmpgtu4(lbp_r(b, k), ctr) & 0x10101010u;
        acc |= __vcmpgtu4(lbp_l(c, k), ctr) & 0x20202020u;
        acc |= __vcmpgtu4(c.w[k], ctr) & 0x40404040u;
        acc |= __vcmpgtu4(lbp_r(c, k), ctr) & 0x80808080u;
        o[k] = acc;
      }
      *reinterpret_cast<uint4*>(out.base + (long long)r * out.pitch + x0) = make_uint4(o[0], o[1], o[2], o[3]);
    }
    return;
  }
  for (int r = r_first; r < r_end; r++) {  // ragged right edge, unaligned images
    const unsigned char* r1 = in.base + (long long)r * in.pitch;
    unsigned char* o = out.base + (long long)r * out.pitch;
    for (int i = x0; i < min(x0 + 16, in.ncols); i++) o[i] = lbp_scalar(r1 - in.pitch, r1, r1 + in.pitch, i);
  }
}

// ---- local_maxima_filter (in place) ---------------------------------------------------------------------------------------------
// The reference zeroes every pixel that is not strictly greater than its 8 neighbours IN PLACE, so a pixel sees the already
// filtered values of the neighbours above and to the left (serial raster order; its pixel_wise runs rows in parallel and races).
// The result of the serial order is the unique solution X of
//     X(p) = orig(p)  if  orig(p) > max(X(NW), X(N), X(NE), X(W), orig(E), orig(SW), orig(S), orig(SE)),  else 0
// - a triangular system (X(p) only depends on X of earlier pixels), solved here by relaxation exactly like the sweeps of the
// semi-dense flow: every pass re-evaluates all pixels on the current X of their predecessors (runs of 16 pixels of a row are
// walked serially, so chains along a row shorten 16-fold), passes are separated by a
// grid-wide barrier, and a pass that changes nothing has reached the fixed point.  X only ever takes the values orig(p) and 0, the
// number of passes is the longest chain of decisions that flip (2 - 4 on score images, the length of a ramp at worst).
template <typename T> __device__ __forceinline__ T ld_cg(const T* p) { return __ldcg(p); }

constexpr int LMF_RUN = 16;
template <typename T>
__global__ void __launch_bounds__(256) k_local_maxima_filter(Img im, T* orig, int wcols, int* ctr) {
  const long long gthreads = (long long)gridDim.x * blockDim.x, gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int gen = 0;
  // orig <- the image with its border of 1 (tight rows of wcols = ncols + 2 elements)
  const long long wtotal = (long long)(im.nrows + 2) * wcols;
  for (long long i = gtid; i < wtotal; i += gthreads) {
    const int r = (int)(i / wcols) - 1, c = (int)(i % wcols) - 1;
    orig[i] = reinterpret_cast<const T*>(im.base + (long long)r * im.pitch)[c];
  }
  grid_barrier(ctr, gen);
  // a thread owns a run of LMF_RUN consecutive pixels of a row and walks it left to right with its own fresh result as the left
  // neighbour (Gauss-Seidel inside the run): a horizontal chain of dependent decisions costs one pass per run it crosses, not one per pixel
  const int runs_per_row = (im.ncols + LMF_RUN - 1) / LMF_RUN;
  const long long total = (long long)im.nrows * runs_per_row;
  for (int pass = 0;; pass++) {
    int changed = 0;
    for (long long i = gtid; i < total; i += gthreads) {
      const int r = (int)(i / runs_per_row), c0 = (int)(i % runs_per_row) * LMF_RUN;
      const int c1 = min(c0 + LMF_RUN, im.ncols);
      const T* o1 = orig + (long long)(r + 1) * wcols + (c0 + 1);   // orig(r, c0)
      const T* o2 = o1 + wcols;                                       // orig(r + 1, c0)
      T* x1 = reinterpret_cast<T*>(im.base + (long long)r * im.pitch) + c0;
      const T* x0 = reinterpret_cast<const T*>(im.base + (long long)(r - 1) * im.pitch) + c0;
      // successors: original values; predecessors: their current X (read from L2: other CTAs rewrite it between passes)
      T w = ld_cg(x1 - 1);
      T nl = ld_cg(x0 - 1), nm = ld_cg(x0);
      T sl = o2[-1], sm = o2[0];
      T a = o1[0];
      for (int c = c0; c < c1; c++, o1++, o2++, x0++, x1++) {
        const T nr = ld_cg(x0 + 1), sr = o2[1], e = o1[1];
        const bool is_max = a > e && a > sl && a > sm && a > sr && a > nl && a > nm && a > nr && a > w;
        const T res = is_max ? a : (T)0;
        if (ld_cg(x1) != res) { *x1 = res; changed = 1; }
        w = res; nl = nm; nm = nr; sl = sm; sm = sr; a = e;
      }
    }
    if (__any_sync(0xffffffffu, changed) && (threadIdx.x & 31) == 0) atomicAdd(ctr + 1 + pass % 3, 1);
    if (gtid == 0) ctr[1 + (pass + 1) % 3] = 0;  // next pass's counter: nobody reads or writes it during this pass
    grid_barrier(ctr, gen);
    if (ld_cg(ctr + 1 + pass % 3) == 0) break;  // grid-uniform: the counter is stable until every CTA has passed the next barrier
  }
}

}  // namespace vppb

using namespace vppb;

extern "C" {

int vppb_lbp_u8(const vppb_img* in, const vppb_img* out, void* stream) {
  VPPB_REQUIRE(in && out && in->base && out->base, VPPB_E_ARG, "vppb_lbp_u8: NULL argument");
  VPPB_REQUIRE(in->elem_bytes == 1 && out->elem_bytes == 1 && same_domain(in, out), VPPB_E_ARG, "vppb_lbp_u8: u8 images of one domain expected");
  VPPB_REQUIRE(in->border >= 1, VPPB_E_BORDER, "vppb_lbp_u8: the input needs a border of 1 pixel");
  if (in->nrows == 0 || in->ncols == 0) return VPPB_OK;
  const bool vec = ((uintptr_t)in->base % 16) == 0 && (in->pitch % 16) == 0 && ((uintptr_t)out->base % 16) == 0 && (out->pitch % 16) == 0;
  const int xthreads = (in->ncols + 15) / 16;
  const long long threads = (long long)xthreads * ((in->nrows + LBP_ROWS - 1) / LBP_ROWS);
  const int grid = (int)((threads + 255) / 256);
  if (vec) k_lbp_u8<true><<<grid, 256, 0, as_stream(stream)>>>(view(in), view(out), xthreads);
  else k_lbp_u8<false><<<grid, 256, 0, as_stream(stream)>>>(view(in), view(out), xthreads);
  VPPB_LAUNCH_CHECK("vppb_lbp_u8");
  return VPPB_OK;
}

int64_t vppb_local_maxima_filter_workspace_bytes(int32_t nrows, int32_t ncols, int32_t elem_bytes) {
  if (nrows < 0 || ncols < 0 || (elem_bytes != 1 && elem_bytes != 4)) return 0;
  return (((int64_t)(nrows + 2) * (ncols + 2) * elem_bytes + 255) / 256) * 256 + 256;
}

int vppb_local_maxima_filter(const vppb_img* img, void* workspace, int64_t workspace_bytes, void* stream) {
  VPPB_REQUIRE(img && img->base && workspace, VPPB_E_ARG, "vppb_local_maxima_filter: NULL argument");
  VPPB_REQUIRE(img->elem_bytes == 1 || img->elem_bytes == 4, VPPB_E_ARG, "vppb_local_maxima_filter: unsigned char or int pixels expected");
  VPPB_REQUIRE(img->border >= 1, VPPB_E_BORDER, "vppb_local_maxima_filter: the image needs a border of 1 pixel");
  const int64_t need = vppb_local_maxima_filter_workspace_bytes(img->nrows, img->ncols, img->elem_bytes);
  VPPB_REQUIRE((uintptr_t)workspace % 256 == 0, VPPB_E_ARG, "vppb_local_maxima_filter: workspace not 256-byte aligned");
  VPPB_REQUIRE(workspace_bytes >= need, VPPB_E_ARG, "vppb_local_maxima_filter: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
  if (img->nrows == 0 || img->ncols == 0) return VPPB_OK;
  cudaStream_t st = as_stream(stream);
  int* ctr = reinterpret_cast<int*>(static_cast<unsigned char*>(workspace) + need - 256);
  VPPB_CUDA(cudaMemsetAsync(ctr, 0, 256, st));
  const long long total = (long long)img->nrows * ((img->ncols + LMF_RUN - 1) / LMF_RUN);
  long long blocks = (total + 255) / 256;
  if (img->elem_bytes == 1) {
    const int cap = cooperative_grid_limit(k_local_maxima_filter<unsigned char>, 256);
    if (blocks > cap) blocks = cap;
    VPPB_CUDA(launch_cooperative(k_local_maxima_filter<unsigned char>, (int)blocks, 256, st, view(img), static_cast<unsigned char*>(workspace), img->ncols + 2, ctr));
  } else {
    const int cap = cooperative_grid_limit(k_local_maxima_filter<int>, 256);
    if (blocks > cap) blocks = cap;
    VPPB_CUDA(launch_cooperative(k_local_maxima_filter<int>, (int)blocks, 256, st, view(img), static_cast<int*>(workspace), img->ncols + 2, ctr));
  }
  VPPB_LAUNCH_CHECK("vppb_local_maxima_filter");
  return VPPB_OK;
}

}  // extern "C"

// ---- chamfer distance transforms d4, d8, d3-4 and d5-7-11 (vpp/algorithms/distance_transforms/distance_transforms.hh:86-152) ----
//
// The reference fills S with B = nrows + ncols (border included), sets S = 0 where A == 0, then runs a forward and a backward
// raster pass of its half-masks, serially.  The result has a closed form (DESIGN §3.7): a border pixel keeps B, a domain pixel p
// gets min(B, min over the zero pixels z of gauge(p - z)), where the gauge is the cheapest combination of the mask's moves.  Each
// mask is a set of generators g with weights w, and the transform is the composition, in any order, of one min-plus line scan per
// generator:  X(p) <- min over t of X(p + t g) + |t| w, along every line p + t g clipped to the domain (an optimal path uses two
// neighbouring generators, and either order of its two legs keeps the corner inside the bounding box of its ends).
//
// Kernels, in stream order:
//   k_dt_rows     one warp per buffer row: the whole border becomes B; a domain row gets the init and the horizontal generator
//                 (0, 1) fused: min(B, w * distance to the nearest zero of the row), from a warp max- and min-scan of zero columns.
//   then per remaining generator (gr, gc), gr in {1, 2}, three launches over bands of DT_H rows:
//   k_dt_summary  one thread per (band, line): the segment's min-plus exit values at both ends (workspace);
//   k_dt_carry    one thread per line: serial over the bands, turns the exit values into the carries entering each segment;
//   k_dt_apply    one thread per (band, line): forward and backward scan of the segment seeded with the carries, written back.
// Adjacent threads own adjacent lines, which cross a row at adjacent columns: every access of a warp is coalesced.  Values are
// capped at B throughout (exact: nothing at or above B can produce a value below B).  The launch count depends on the mask only.
namespace vppb {

constexpr int DT_H = 32;  // rows per band: a segment is DT_H / gr pixels, kept in registers by k_dt_apply
constexpr int DT_PX = 8;  // consecutive columns per lane in k_dt_rows

struct DtGen { int gr, gc, w; };
struct DtMask { int reach, w_row, ngen; DtGen gen[7]; };

// the generators of each mask other than (0, 1), which k_dt_rows applies with weight w_row
static const DtMask DT_MASKS[4] = {
    {1, 1, 1, {{1, 0, 1}}},                                                                       // d4
    {1, 1, 3, {{1, 0, 1}, {1, 1, 1}, {1, -1, 1}}},                                                // d8
    {1, 3, 3, {{1, 0, 3}, {1, 1, 4}, {1, -1, 4}}},                                                // d3-4
    {2, 5, 7, {{1, 0, 5}, {1, 1, 7}, {1, -1, 7}, {1, 2, 11}, {1, -2, 11}, {2, 1, 11}, {2, -1, 11}}},  // d5-7-11
};

// Lines of generator (gr, gc): pixel (r, c) lies at step t = r / gr of line (r % gr, c - t * gc).  Line ids are
// par * nq + (q - qmin) over every (par, q) some domain pixel has; band b holds steps [b * kb, (b + 1) * kb).
struct DtLines {
  int gr, gc, w, kb, qmin, nq, nlines, nbands;
};

static DtLines dt_lines(int nrows, int ncols, const DtGen& g) {
  DtLines L;
  L.gr = g.gr; L.gc = g.gc; L.w = g.w;
  L.kb = DT_H / g.gr;
  const int tmax = (nrows - 1) / g.gr;
  L.qmin = g.gc > 0 ? -tmax * g.gc : 0;
  L.nq = ncols + tmax * (g.gc < 0 ? -g.gc : g.gc);
  L.nlines = g.gr * L.nq;
  L.nbands = (nrows + DT_H - 1) / DT_H;
  return L;
}

// ---- init + horizontal generator + border ---------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_dt_rows(Img in, Img out, int bo, int B, int w) {
  const int warp = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  const int r = warp - bo;
  if (r >= in.nrows + bo) return;
  int* o = row_ptr<int>(out, r);
  if (r < 0 || r >= in.nrows) {
    for (int c = lane - bo; c < in.ncols + bo; c += 32) o[c] = B;
    return;
  }
  for (int c = lane; c < bo; c += 32) { o[-1 - c] = B; o[in.ncols + c] = B; }
  const T* a = row_ptr<const T>(in, r);
  constexpr int NONE = 1 << 30;  // ncols < 2^29 (int pitch), so c -/+ NONE never reaches the cap from below
  // left to right: distance to the last zero at or before c, stored as w * d (capped)
  int last = -NONE;
  for (int c0 = 0; c0 < in.ncols; c0 += 32 * DT_PX) {
    const int cl = c0 + lane * DT_PX;
    int z[DT_PX];
#pragma unroll
    for (int j = 0; j < DT_PX; j++) z[j] = cl + j < in.ncols && a[cl + j] == 0;
    int mine = -NONE;
#pragma unroll
    for (int j = 0; j < DT_PX; j++) mine = z[j] ? cl + j : mine;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, mine, s);
      if (lane >= s) mine = max(mine, v);
    }
    int run = max(last, __shfl_up_sync(0xffffffffu, mine, 1));
    if (lane == 0) run = last;
#pragma unroll
    for (int j = 0; j < DT_PX; j++) {
      const int c = cl + j;
      if (z[j]) run = c;
      if (c < in.ncols) o[c] = (int)min((long long)B, (long long)w * (c - run));
    }
    last = max(last, __shfl_sync(0xffffffffu, mine, 31));  // a tile without a zero keeps the carry
  }
  // right to left: distance to the first zero at or after c, combined with the stored value
  int next = NONE;
  const int ntiles = (in.ncols + 32 * DT_PX - 1) / (32 * DT_PX);
  for (int tile = ntiles - 1; tile >= 0; tile--) {
    const int cl = tile * 32 * DT_PX + lane * DT_PX;
    int z[DT_PX];
#pragma unroll
    for (int j = 0; j < DT_PX; j++) z[j] = cl + j < in.ncols && a[cl + j] == 0;
    int mine = NONE;
#pragma unroll
    for (int j = DT_PX - 1; j >= 0; j--) mine = z[j] ? cl + j : mine;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int v = __shfl_down_sync(0xffffffffu, mine, s);
      if (lane + s < 32) mine = min(mine, v);
    }
    int run = min(next, __shfl_down_sync(0xffffffffu, mine, 1));
    if (lane == 31) run = next;
#pragma unroll
    for (int j = DT_PX - 1; j >= 0; j--) {
      const int c = cl + j;
      if (z[j]) run = c;
      if (c < in.ncols) o[c] = min(o[c], (int)min((long long)B, (long long)w * (run - c)));
    }
    next = min(next, __shfl_sync(0xffffffffu, mine, 0));
  }
}

// ---- one generator: segment summaries, carries, apply ---------------------------------------------------------------------------
// The pixel at step k of the segment of line `line` in band b, or nullptr outside the domain.
template <int GR>
__device__ __forceinline__ int* dt_at(const Img& im, const DtLines& L, int b, int line, int k) {
  const int par = line / L.nq, q = line - par * L.nq + L.qmin;
  const int t = b * (DT_H / GR) + k;
  const int r = t * GR + par, c = q + t * L.gc;
  if (r >= im.nrows || c < 0 || c >= im.ncols) return nullptr;
  return row_ptr<int>(im, r) + c;
}

// ws[b * nlines + line] = (F, G): F = min_k X_k + w (kb - 1 - k), the segment's value at its last step; G = min_k X_k + w k, at its first
template <int GR>
__global__ void __launch_bounds__(256) k_dt_summary(Img out, DtLines L, int B, int2* ws) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)L.nbands * L.nlines) return;
  const int b = (int)(i / L.nlines), line = (int)(i - (long long)b * L.nlines);
  int f = B, g = B;
#pragma unroll
  for (int k = 0; k < DT_H / GR; k++) {
    const int* p = dt_at<GR>(out, L, b, line, k);
    const int x = p ? *p : B;
    f = min(f + L.w, x);
    g = min(g, x + L.w * k);
  }
  ws[i] = make_int2(f, min(g, B));
}

// in place: ws[b].x <- the value entering band b from above (at step b kb - 1), ws[b].y <- from below (at step (b + 1) kb)
__global__ void __launch_bounds__(256) k_dt_carry(DtLines L, int B, int2* ws) {
  const int line = blockIdx.x * blockDim.x + threadIdx.x;
  if (line >= L.nlines) return;
  const int span = L.w * L.kb;
  int carry = B;
  for (int b = 0; b < L.nbands; b++) {
    int2* p = ws + (long long)b * L.nlines + line;
    const int f = p->x;
    p->x = carry;
    carry = min(B, min(carry + span, f));
  }
  carry = B;
  for (int b = L.nbands - 1; b >= 0; b--) {
    int2* p = ws + (long long)b * L.nlines + line;
    const int g = p->y;
    p->y = carry;
    carry = min(B, min(carry + span, g));
  }
}

template <int GR>
__global__ void __launch_bounds__(256) k_dt_apply(Img out, DtLines L, const int2* ws) {
  constexpr int KB = DT_H / GR;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)L.nbands * L.nlines) return;
  const int b = (int)(i / L.nlines), line = (int)(i - (long long)b * L.nlines);
  const int2 cin = ws[i];
  int v[KB];
  int run = cin.x;  // <= B, and every X is <= B: no value computed here exceeds B
#pragma unroll
  for (int k = 0; k < KB; k++) {
    const int* p = dt_at<GR>(out, L, b, line, k);
    run = p ? min(run + L.w, *p) : run + L.w;
    v[k] = run;
  }
  run = cin.y;
#pragma unroll
  for (int k = KB - 1; k >= 0; k--) {
    run = min(run + L.w, v[k]);
    int* p = dt_at<GR>(out, L, b, line, k);
    if (p) *p = run;
  }
}

static int64_t dt_ws_bytes(int nrows, int ncols, const DtMask& m) {
  int64_t need = 0;
  for (int i = 0; i < m.ngen; i++) {
    const DtLines L = dt_lines(nrows, ncols, m.gen[i]);
    need = std::max(need, (int64_t)L.nbands * L.nlines * (int64_t)sizeof(int2));
  }
  return need;
}

// byte span [lo, hi) of rows -b .. nrows - 1 + b, columns -b .. ncols - 1 + b
static void dt_span(const vppb_img* im, int b, uintptr_t& lo, uintptr_t& hi) {
  const uintptr_t base = (uintptr_t)im->base;
  lo = base - (uintptr_t)((int64_t)b * im->pitch + (int64_t)b * im->elem_bytes);
  hi = base + (uintptr_t)((int64_t)(im->nrows - 1 + b) * im->pitch + (int64_t)(im->ncols + b) * im->elem_bytes);
}

}  // namespace vppb

using namespace vppb;

extern "C" {

int64_t vppb_distance_transform_workspace_bytes(int32_t nrows, int32_t ncols, int32_t kind) {
  if (nrows <= 0 || ncols <= 0 || kind < VPPB_DT_D4 || kind > VPPB_DT_D5_7_11) return 0;
  return dt_ws_bytes(nrows, ncols, DT_MASKS[kind]);
}

int vppb_distance_transform(const vppb_img* in, const vppb_img* out, int32_t kind, void* workspace, int64_t workspace_bytes, void* stream) {
  VPPB_REQUIRE(in && out && in->base && out->base, VPPB_E_ARG, "vppb_distance_transform: NULL argument");
  VPPB_REQUIRE(kind >= VPPB_DT_D4 && kind <= VPPB_DT_D5_7_11, VPPB_E_ARG, "vppb_distance_transform: unknown kind %d", kind);
  VPPB_REQUIRE((in->elem_bytes == 1 || in->elem_bytes == 4) && out->elem_bytes == 4, VPPB_E_ARG,
               "vppb_distance_transform: unsigned char or int input and int output expected");
  VPPB_REQUIRE(same_domain(in, out) && in->nrows > 0 && in->ncols > 0, VPPB_E_ARG, "vppb_distance_transform: the images need one non-empty domain");
  VPPB_REQUIRE((int64_t)in->nrows + in->ncols < (1 << 30), VPPB_E_ARG, "vppb_distance_transform: nrows + ncols must stay below 2^30");
  VPPB_REQUIRE((uintptr_t)out->base % 4 == 0 && out->pitch % 4 == 0 && (in->elem_bytes == 1 || ((uintptr_t)in->base % 4 == 0 && in->pitch % 4 == 0)),
               VPPB_E_ARG, "vppb_distance_transform: int images need 4-byte aligned rows");
  const DtMask& m = DT_MASKS[kind];
  VPPB_REQUIRE(out->border >= m.reach, VPPB_E_BORDER, "vppb_distance_transform: the output needs a border of %d pixel(s)", m.reach);
  uintptr_t ilo, ihi, olo, ohi;
  dt_span(in, 0, ilo, ihi);
  dt_span(out, out->border, olo, ohi);
  VPPB_REQUIRE(!(in->alloc && in->alloc == out->alloc) && (ihi <= olo || ohi <= ilo), VPPB_E_ARG,
               "vppb_distance_transform: the input and the output share memory");
  const int64_t need = dt_ws_bytes(in->nrows, in->ncols, m);
  // the workspace holds int2 segment summaries: 8-byte alignment is what they need (a host or malloc'ed block qualifies)
  VPPB_REQUIRE(need == 0 || (uintptr_t)workspace % 8 == 0, VPPB_E_ARG, "vppb_distance_transform: workspace not 8-byte aligned");
  VPPB_REQUIRE(need == 0 || (workspace && workspace_bytes >= need), VPPB_E_ARG, "vppb_distance_transform: workspace %lld < %lld bytes",
               (long long)workspace_bytes, (long long)need);

  cudaStream_t st = as_stream(stream);
  const Img vi = view(in), vo = view(out);
  const int B = in->nrows + in->ncols;
  const long long row_threads = 32LL * (in->nrows + 2 * out->border);
  const int row_grid = (int)((row_threads + 255) / 256);
  if (in->elem_bytes == 1) k_dt_rows<unsigned char><<<row_grid, 256, 0, st>>>(vi, vo, out->border, B, m.w_row);
  else k_dt_rows<int><<<row_grid, 256, 0, st>>>(vi, vo, out->border, B, m.w_row);
  VPPB_LAUNCH_CHECK("vppb_distance_transform");
  int2* ws = static_cast<int2*>(workspace);
  for (int gi = 0; gi < m.ngen; gi++) {
    const DtLines L = dt_lines(in->nrows, in->ncols, m.gen[gi]);
    const long long items = (long long)L.nbands * L.nlines;
    const int grid = (int)((items + 255) / 256), cgrid = (L.nlines + 255) / 256;
    if (L.gr == 1) k_dt_summary<1><<<grid, 256, 0, st>>>(vo, L, B, ws);
    else k_dt_summary<2><<<grid, 256, 0, st>>>(vo, L, B, ws);
    k_dt_carry<<<cgrid, 256, 0, st>>>(L, B, ws);
    if (L.gr == 1) k_dt_apply<1><<<grid, 256, 0, st>>>(vo, L, ws);
    else k_dt_apply<2><<<grid, 256, 0, st>>>(vo, L, ws);
    VPPB_LAUNCH_CHECK("vppb_distance_transform");
  }
  return VPPB_OK;
}

}  // extern "C"
