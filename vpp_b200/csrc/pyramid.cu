// Scharr gradient and the fused low-pass + subsample pyramid step.
// Reference: vpp/algorithms/filters/scharr.hh:46-87, vpp/core/pyramid.hh:12-59 (1-4-6-4-1
// separable low-pass, H pass then mirror then V pass) and :62-81 (subsample2).
// Both are streaming stencils bounded by HBM: scharr moves 1 + 8 bytes per pixel, a pyramid
// step reads N_{l-1} and writes N_l pixels (no temp image: the reference's H temp and its
// mirror fill are reproduced by index mirroring inside the kernel).
// The library is compiled with -fmad=false: float results must match the reference's
// un-contracted evaluation order bit for bit.
#include "common.cuh"

#include <atomic>

#include <algorithm>

namespace vppb {

// ------------------------------------------------------------------ Scharr
// 8 pixels per thread.  Each of the rows r-1, r, r+1 is fetched as one 16-byte load (columns c0 ..
// c0+15, of which c0..c0+8 are used) plus one 4-byte load for column c0-1; the eight vector<Vt,2>
// results leave as four 16-byte stores (a warp writes 2 KB contiguous).  Output-dominated: 1 B read,
// 8 B written per pixel.
__device__ __forceinline__ int byte_of(uint32_t w, int k) { return (int)((w >> (8 * k)) & 0xFFu); }
__device__ __forceinline__ int mirror_idx(int i, int n) { return i < 0 ? -i - 1 : (i >= n ? 2 * n - i - 1 : i); }

// one pixel, byte loads (scharr.hh:64-83), stored at out(orow, ocol)
template <bool AS_FLOAT>
__device__ __forceinline__ void scharr_px(const Img& in, const Img& out, int r, int c, int orow, int ocol) {
  const unsigned char* r1 = row_ptr<unsigned char>(in, r - 1) + c - 1;
  const unsigned char* r2 = row_ptr<unsigned char>(in, r) + c - 1;
  const unsigned char* r3 = row_ptr<unsigned char>(in, r + 1) + c - 1;
  const int a = 3 * (int)r3[0] + 10 * (int)r3[1] + 3 * (int)r3[2] - 3 * (int)r1[0] - 10 * (int)r1[1] - 3 * (int)r1[2];
  const int b = 3 * (int)r1[2] + 10 * (int)r2[2] + 3 * (int)r3[2] - 3 * (int)r1[0] - 10 * (int)r2[0] - 3 * (int)r3[0];
  const float fa = __fmul_rn((float)a, 0.03125f), fb = __fmul_rn((float)b, 0.03125f);  // x / 32.f exactly
  if (AS_FLOAT) reinterpret_cast<float2*>(row_ptr<unsigned char>(out, orow))[ocol] = make_float2(fa, fb);
  else reinterpret_cast<int2*>(row_ptr<unsigned char>(out, orow))[ocol] = make_int2((int)fa, (int)fb);  // trunc toward 0
}

// Border pixel number j of `out` (frame of width mb), filled as fill_border_mirror would: the gradient at the
// mirrored domain position, recomputed from `in` so the item does not depend on any other thread's store.
template <bool AS_FLOAT>
__device__ __forceinline__ void scharr_border_item(const Img& in, const Img& out, long long j, int mb) {
  const int nr = out.nrows, nc = out.ncols;
  const long long wfull = nc + 2LL * mb, n_top = (long long)mb * wfull, n_side = (long long)nr * mb;
  int r, c;
  if (j < n_top) { r = (int)(j / wfull) - mb; c = (int)(j % wfull) - mb; }
  else if (j < 2 * n_top) { j -= n_top; r = nr + (int)(j / wfull); c = (int)(j % wfull) - mb; }
  else if (j < 2 * n_top + n_side) { j -= 2 * n_top; r = (int)(j / mb); c = (int)(j % mb) - mb; }
  else { j -= 2 * n_top + n_side; r = (int)(j / mb); c = nc + (int)(j % mb); }
  scharr_px<AS_FLOAT>(in, out, mirror_idx(r, nr), mirror_idx(c, nc), r, c);
}
__host__ __device__ __forceinline__ long long border_items(int nr, int nc, int mb) { return 2LL * mb * (nc + 2LL * mb) + 2LL * nr * mb; }

// loads of image data: read-only path (NC) in the one-kernel-per-step launches; plain loads inside the cooperative kernel of
// vppb_pyrlk_prepare, where an earlier phase of the same kernel wrote the image
template <bool NC, typename T> __device__ __forceinline__ T ld_img(const T* p) { return NC ? __ldg(p) : *p; }

// work item i of scharr (8 pixels of a row per item, then one item per mirror-border pixel)
template <bool AS_FLOAT, bool NC>
__device__ __forceinline__ void scharr_v8_item(const Img& in, const Img& out, int groups_per_row, int mb, long long i) {
  const long long total = (long long)out.nrows * groups_per_row;
  {
    if (i >= total) { scharr_border_item<AS_FLOAT>(in, out, i - total, mb); return; }
    int r, c0;
    item_divmod(i, groups_per_row, r, c0);
    c0 *= 8;
    int px[3][10];  // columns c0-1 .. c0+8
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const unsigned char* row = row_ptr<unsigned char>(in, r - 1 + k) + c0;
      const uint32_t left = ld_img<NC>(reinterpret_cast<const uint32_t*>(row - 4));
      const uint2 mid = ld_img<NC>(reinterpret_cast<const uint2*>(row));
      const uint32_t right = ld_img<NC>(reinterpret_cast<const uint32_t*>(row + 8));
      px[k][0] = byte_of(left, 3);
#pragma unroll
      for (int j = 0; j < 4; j++) { px[k][1 + j] = byte_of(mid.x, j); px[k][5 + j] = byte_of(mid.y, j); }
      px[k][9] = byte_of(right, 0);
    }
    unsigned char* orow = row_ptr<unsigned char>(out, r) + (long long)c0 * 8;
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      int a[2], b[2];
#pragma unroll
      for (int t = 0; t < 2; t++) {
        const int* r1 = &px[0][j + t];
        const int* r2 = &px[1][j + t];
        const int* r3 = &px[2][j + t];
        a[t] = 3 * r3[0] + 10 * r3[1] + 3 * r3[2] - 3 * r1[0] - 10 * r1[1] - 3 * r1[2];  // scharr.hh:64-83
        b[t] = 3 * r1[2] + 10 * r2[2] + 3 * r3[2] - 3 * r1[0] - 10 * r2[0] - 3 * r3[0];
      }
      const float fa0 = __fmul_rn((float)a[0], 0.03125f), fb0 = __fmul_rn((float)b[0], 0.03125f);  // x / 32.f exactly
      const float fa1 = __fmul_rn((float)a[1], 0.03125f), fb1 = __fmul_rn((float)b[1], 0.03125f);
      if (c0 + j + 1 < out.ncols) {
        if (AS_FLOAT) *reinterpret_cast<float4*>(orow + j * 8) = make_float4(fa0, fb0, fa1, fb1);
        else *reinterpret_cast<int4*>(orow + j * 8) = make_int4((int)fa0, (int)fb0, (int)fa1, (int)fb1);
      } else if (c0 + j < out.ncols) {
        if (AS_FLOAT) *reinterpret_cast<float2*>(orow + j * 8) = make_float2(fa0, fb0);
        else *reinterpret_cast<int2*>(orow + j * 8) = make_int2((int)fa0, (int)fb0);
      }
    }
  }
}
template <bool AS_FLOAT>
__global__ void __launch_bounds__(256) k_scharr_u8_v8(Img in, Img out, int groups_per_row, int mb) {
  const long long total = (long long)out.nrows * groups_per_row + border_items(out.nrows, out.ncols, mb);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    scharr_v8_item<AS_FLOAT, true>(in, out, groups_per_row, mb, i);
}

// any layout: 1 pixel per thread, byte loads
template <bool AS_FLOAT>
__device__ __forceinline__ void scharr_px_item(const Img& in, const Img& out, int mb, long long i) {
  const long long total = (long long)out.nrows * out.ncols;
  if (i >= total) { scharr_border_item<AS_FLOAT>(in, out, i - total, mb); return; }
  int r, c;
  item_divmod(i, out.ncols, r, c);
  scharr_px<AS_FLOAT>(in, out, r, c, r, c);
}
template <bool AS_FLOAT>
__global__ void __launch_bounds__(256) k_scharr_u8(Img in, Img out, int mb) {
  const long long total = (long long)out.nrows * out.ncols + border_items(out.nrows, out.ncols, mb);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) scharr_px_item<AS_FLOAT>(in, out, mb, i);
}

// ------------------------------------------------------------------ low-pass + subsample2
template <int KIND> struct LpT;
template <> struct LpT<0> { typedef unsigned char elem; typedef int acc; static constexpr int comps = 1; };
template <> struct LpT<1> { typedef int elem; typedef int acc; static constexpr int comps = 2; };
template <> struct LpT<2> { typedef float elem; typedef float acc; static constexpr int comps = 2; };

__device__ __forceinline__ int lp5(int a, int b, int c, int d, int e) { return (1 * a + 4 * b + 6 * c + 4 * d + 1 * e) / 16; }
__device__ __forceinline__ float lp5(float a, float b, float c, float d, float e) {
  // ((((1*a + 4*b) + 6*c) + 4*d) + 1*e) / 16, no contraction (pyramid.hh:27-32)
  // 1 * x is x and s / 16 is s * 0.0625 for every float (power-of-two scale: one rounding either way): no division routine
  float s = __fadd_rn(a, __fmul_rn(4.f, b));
  s = __fadd_rn(s, __fmul_rn(6.f, c));
  s = __fadd_rn(s, __fmul_rn(4.f, d));
  s = __fadd_rn(s, e);
  return __fmul_rn(s, 0.0625f);
}


// Store out(r, c) = v and, when mb > 0, every border pixel that fill_border_mirror (border.hh mirror rule:
// border(-1-k) = image(k), border(n+k) = image(n-1-k)) would copy from (r, c): up to 3 rows x 3 columns.
// Every border pixel has exactly one source pixel, so a kernel in which each output pixel is produced by one
// thread fills the whole mirror border without races.  `comps`/`k` address one component of a COMPS-vector.
template <typename T>
__device__ __forceinline__ void store_mirrored(const Img& out, int r, int c, T v, int mb, int comps = 1, int k = 0) {
  row_ptr<T>(out, r)[c * comps + k] = v;
  if (mb <= 0) return;
  const bool rt = r < mb, rb = r >= out.nrows - mb, cl = c < mb, cr = c >= out.ncols - mb;
  if (!(rt | rb | cl | cr)) return;  // interior pixel: no border pixel mirrors it
#pragma unroll
  for (int a = 0; a < 3; a++) {      // a / b: 0 = the pixel's own row / column, 1 = mirrored above / left, 2 = below / right
    if (!(a == 0 || (a == 1 ? rt : rb))) continue;
    T* row = row_ptr<T>(out, a == 0 ? r : (a == 1 ? -1 - r : 2 * out.nrows - 1 - r));
#pragma unroll
    for (int b = 0; b < 3; b++) {
      if (!(b == 0 || (b == 1 ? cl : cr)) || (a == 0 && b == 0)) continue;
      row[(b == 0 ? c : (b == 1 ? -1 - c : 2 * out.ncols - 1 - c)) * comps + k] = v;
    }
  }
}

// One thread per output pixel component.  out(r,c) = LP(mirror(2r), mirror(2c)); LP's V pass reads
// H rows with mirrored indices (the mirror-filled temp of pyramid.hh:36), H reads in(row, x-2..x+2)
// from the image's own (caller-filled) column border.
template <int KIND>
__device__ __forceinline__ void lowpass_sub2_item(const Img& in, const Img& out, int step, int mb, long long i) {
  typedef typename LpT<KIND>::elem E;
  typedef typename LpT<KIND>::acc A;
  constexpr int COMPS = LpT<KIND>::comps;
  {
    const int k = (int)(i % COMPS);
    int r, c;
    item_divmod(i / COMPS, out.ncols, r, c);
    const int y = mirror_idx(r * step, in.nrows);
    const int x = mirror_idx(c * step, in.ncols);
    A h[5];
#pragma unroll
    for (int d = 0; d < 5; d++) {
      const int yy = mirror_idx(y - 2 + d, in.nrows);
      const E* row = row_ptr<E>(in, yy);
      h[d] = (A)(E)lp5((A)row[(x - 2) * COMPS + k], (A)row[(x - 1) * COMPS + k], (A)row[x * COMPS + k], (A)row[(x + 1) * COMPS + k],
                       (A)row[(x + 2) * COMPS + k]);
    }
    store_mirrored<E>(out, r, c, (E)lp5(h[0], h[1], h[2], h[3], h[4]), mb, COMPS, k);
  }
}
template <int KIND>
__global__ void __launch_bounds__(256) k_lowpass_sub2(Img in, Img out, int step, int mb) {
  const long long total = (long long)out.nrows * out.ncols * LpT<KIND>::comps;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) lowpass_sub2_item<KIND>(in, out, step, mb, i);
}

// u8 fast path: one thread = 8 x 2 outputs.  The 7 input rows it needs (mirrored indices at the top /
// bottom, as the mirror-filled H temp of pyramid.hh:36) are fetched as 4 + 16 + 4 bytes each, H is
// evaluated at the 8 even columns per row, V on the H columns; ~1.3 loads per output instead of 25.
// Covers the outputs whose centre (2r, 2c) lies inside the parent; the mirrored last row / column of
// an even-sized parent (centre on an odd pixel) is handled by the tail work items of the same launch.
// One 8-byte group of row `tr` (a domain row or one of its mirrored border rows) + the mirrored border columns.
__device__ __forceinline__ void put_u8x8(const Img& out, int tr, int c0, uint32_t lo, uint32_t hi, int valid_cols, int mb) {
  unsigned char* rowp = row_ptr<unsigned char>(out, tr);
  if (c0 + 8 <= valid_cols) *reinterpret_cast<uint2*>(rowp + c0) = make_uint2(lo, hi);
  else
    for (int k = 0; k < 8 && c0 + k < valid_cols; k++) rowp[c0 + k] = (unsigned char)((k < 4 ? lo >> (8 * k) : hi >> (8 * (k - 4))) & 0xFF);
  if (mb > 0 && (c0 < mb || c0 + 8 > out.ncols - mb)) {
    for (int k = 0; k < 8 && c0 + k < valid_cols; k++) {
      const int c = c0 + k;
      const unsigned char v = (unsigned char)((k < 4 ? lo >> (8 * k) : hi >> (8 * (k - 4))) & 0xFF);
      if (c < mb) rowp[-1 - c] = v;
      if (c >= out.ncols - mb) rowp[2 * out.ncols - 1 - c] = v;
    }
  }
}

// Work items [0, total) are 8 x 2 output groups; items [total, total + n_row + n_col) are the outputs of the
// mirrored last row / last column of an even-sized parent (centre on an odd pixel), one per thread, with the
// arithmetic of k_lowpass_sub2<0>.  mb > 0: the mirror border of `out` is written too (store_mirrored).
__host__ __device__ __forceinline__ long long lowpass_u8_fast_items(int out_nrows, int out_ncols, int fast_rows, int fast_cols, int groups_per_row) {
  const int n_row = out_nrows > fast_rows ? out_ncols : 0;
  const int n_col = out_ncols > fast_cols ? out_nrows - (n_row ? 1 : 0) : 0;
  return (long long)((fast_rows + 1) / 2) * groups_per_row + n_row + n_col;
}
template <bool NC>
__device__ __forceinline__ void lowpass_sub2_u8_fast_item(const Img& in, const Img& out, int fast_rows, int fast_cols, int groups_per_row, int mb, long long i) {
  const int row_pairs = (fast_rows + 1) / 2;
  const long long total = (long long)row_pairs * groups_per_row;
  const int n_row = out.nrows > fast_rows ? out.ncols : 0;
  {
    if (i >= total) {
      const int e = (int)(i - total);
      const int r = e < n_row ? out.nrows - 1 : e - n_row;
      const int c = e < n_row ? e : out.ncols - 1;
      const int y = mirror_idx(r * 2, in.nrows), x = mirror_idx(c * 2, in.ncols);
      int h[5];
#pragma unroll
      for (int d = 0; d < 5; d++) {
        const unsigned char* row = row_ptr<unsigned char>(in, mirror_idx(y - 2 + d, in.nrows));
        h[d] = lp5((int)row[x - 2], (int)row[x - 1], (int)row[x], (int)row[x + 1], (int)row[x + 2]);
      }
      store_mirrored<unsigned char>(out, r, c, (unsigned char)lp5(h[0], h[1], h[2], h[3], h[4]), mb);
      return;
    }
    int rp, g;
    item_divmod(i, groups_per_row, rp, g);
    const int r0 = 2 * rp, c0 = 8 * g;
    int H[7][8];
#pragma unroll
    for (int d = 0; d < 7; d++) {
      const int yy = mirror_idx(2 * r0 - 2 + d, in.nrows);
      const unsigned char* row = row_ptr<unsigned char>(in, yy) + 16 * g;
      const uint32_t left = ld_img<NC>(reinterpret_cast<const uint32_t*>(row - 4));
      const uint4 mid = ld_img<NC>(reinterpret_cast<const uint4*>(row));
      const uint32_t right = ld_img<NC>(reinterpret_cast<const uint32_t*>(row + 16));
      int p[19];  // bytes 16g-2 .. 16g+16
      p[0] = byte_of(left, 2); p[1] = byte_of(left, 3);
#pragma unroll
      for (int j = 0; j < 4; j++) { p[2 + j] = byte_of(mid.x, j); p[6 + j] = byte_of(mid.y, j); p[10 + j] = byte_of(mid.z, j); p[14 + j] = byte_of(mid.w, j); }
      p[18] = byte_of(right, 0);
#pragma unroll
      for (int k = 0; k < 8; k++) H[d][k] = (p[2 * k] + 4 * p[2 * k + 1] + 6 * p[2 * k + 2] + 4 * p[2 * k + 3] + p[2 * k + 4]) >> 4;  // pyramid.hh:27-32
    }
#pragma unroll
    for (int t = 0; t < 2; t++) {
      const int r = r0 + t;
      if (r >= fast_rows) break;
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int v = (H[2 * t][k] + 4 * H[2 * t + 1][k] + 6 * H[2 * t + 2][k] + 4 * H[2 * t + 3][k] + H[2 * t + 4][k]) >> 4;  // pyramid.hh:50-55
        if (k < 4) lo |= (uint32_t)v << (8 * k); else hi |= (uint32_t)v << (8 * (k - 4));
      }
      put_u8x8(out, r, c0, lo, hi, fast_cols, mb);
      if (mb > 0) {
        if (r < mb) put_u8x8(out, -1 - r, c0, lo, hi, fast_cols, mb);
        if (r >= out.nrows - mb) put_u8x8(out, 2 * out.nrows - 1 - r, c0, lo, hi, fast_cols, mb);
      }
    }
  }
}
__global__ void __launch_bounds__(128) k_lowpass_sub2_u8_fast(Img in, Img out, int fast_rows, int fast_cols, int groups_per_row, int mb) {
  const long long total = lowpass_u8_fast_items(out.nrows, out.ncols, fast_rows, fast_cols, groups_per_row);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    lowpass_sub2_u8_fast_item<true>(in, out, fast_rows, fast_cols, groups_per_row, mb, i);
}

// 8-byte pixels (vint2 / vfloat2 gradient pyramids): one thread per output pixel, both components;
// each of the 5 rows is read as 16 + 16 + 8 bytes when the centre column is even (always, except for
// the mirrored last column of an even-sized parent).
template <typename A> struct vec2_of;
template <> struct vec2_of<int> { typedef int2 type; typedef int4 type4; };
template <> struct vec2_of<float> { typedef float2 type; typedef float4 type4; };

template <int KIND>
__device__ __forceinline__ void lowpass_sub2_px8_item(const Img& in, const Img& out, int aligned16, int mb, long long i) {
  typedef typename LpT<KIND>::acc A;
  typedef typename vec2_of<A>::type V2;
  typedef typename vec2_of<A>::type4 V4;
  {
    int r, c;
    item_divmod(i, out.ncols, r, c);
    const int y = mirror_idx(r * 2, in.nrows), x = mirror_idx(c * 2, in.ncols);
    A hx[5], hy[5];
#pragma unroll
    for (int d = 0; d < 5; d++) {
      const unsigned char* row = row_ptr<unsigned char>(in, mirror_idx(y - 2 + d, in.nrows)) + (long long)(x - 2) * 8;
      V2 p0, p1, p2, p3, p4;
      if (aligned16 && !(x & 1)) {
        const V4 a = *reinterpret_cast<const V4*>(row), b = *reinterpret_cast<const V4*>(row + 16);
        p0.x = a.x; p0.y = a.y; p1.x = a.z; p1.y = a.w; p2.x = b.x; p2.y = b.y; p3.x = b.z; p3.y = b.w;
        p4 = *reinterpret_cast<const V2*>(row + 32);
      } else {
        const V2* q = reinterpret_cast<const V2*>(row);
        p0 = q[0]; p1 = q[1]; p2 = q[2]; p3 = q[3]; p4 = q[4];
      }
      hx[d] = lp5(p0.x, p1.x, p2.x, p3.x, p4.x);
      hy[d] = lp5(p0.y, p1.y, p2.y, p3.y, p4.y);
    }
    V2 o;
    o.x = lp5(hx[0], hx[1], hx[2], hx[3], hx[4]);
    o.y = lp5(hy[0], hy[1], hy[2], hy[3], hy[4]);
    store_mirrored<V2>(out, r, c, o, mb);
  }
}
template <int KIND>
__global__ void __launch_bounds__(256) k_lowpass_sub2_px8(Img in, Img out, int aligned16, int mb) {
  const long long total = (long long)out.nrows * out.ncols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) lowpass_sub2_px8_item<KIND>(in, out, aligned16, mb, i);
}

// ---- vppb_pyrlk_prepare as ONE cooperative launch -----------------------------------------------------------------------------------
// Everything lucas_kanade() / a pyrlk_match caller builds before matching is a short DAG of the work-item loops above:
//   phase 0: prev[0] <- copy + mirror(i1), next[0] <- copy + mirror(i2)
//   phase 1: grad[0] <- scharr + mirror(prev[0]), prev[1] <- lowpass(prev[0]), next[1] <- lowpass(next[0])
//   phase l: grad[l-1] <- lowpass(grad[l-2]), prev[l] <- ..., next[l] <- ...;   last phase: grad[L-1] <- lowpass(grad[L-2])
// The ops of a phase are independent: their work items are concatenated and shared out over the whole (resident) grid; phases are
// separated by a grid-wide barrier.  L barriers instead of 3 L launches on three streams with four event hops.
enum { PREP_COPY_MIRROR = 0, PREP_SCHARR_V8, PREP_SCHARR_PX, PREP_LP_U8_FAST, PREP_LP_GENERIC, PREP_LP_PX8 };
struct PrepOp {
  int kind, variant;  // variant: as_float (scharr) / KIND (lowpass)
  Img in, out;
  int p0, p1, p2, mb;
  long long items;
};
constexpr int PREP_MAX_LEVELS = 8;
struct PrepProg {
  PrepOp op[3 * PREP_MAX_LEVELS + 3];
  int phase_end[PREP_MAX_LEVELS + 2];
  int nphases;
  int* bar;
};

__device__ __forceinline__ void prep_item(const PrepOp& o, long long i) {
  switch (o.kind) {
    case PREP_COPY_MIRROR: copy_mirror_item(o.in, o.out, o.p0, o.p1, o.p2, i); break;
    case PREP_SCHARR_V8:
      if (o.variant) scharr_v8_item<true, false>(o.in, o.out, o.p0, o.mb, i); else scharr_v8_item<false, false>(o.in, o.out, o.p0, o.mb, i);
      break;
    case PREP_SCHARR_PX:
      if (o.variant) scharr_px_item<true>(o.in, o.out, o.mb, i); else scharr_px_item<false>(o.in, o.out, o.mb, i);
      break;
    case PREP_LP_U8_FAST: lowpass_sub2_u8_fast_item<false>(o.in, o.out, o.p0, o.p1, o.p2, o.mb, i); break;
    case PREP_LP_GENERIC:
      if (o.variant == 0) lowpass_sub2_item<0>(o.in, o.out, 2, o.mb, i);
      else if (o.variant == 1) lowpass_sub2_item<1>(o.in, o.out, 2, o.mb, i);
      else lowpass_sub2_item<2>(o.in, o.out, 2, o.mb, i);
      break;
    default:
      if (o.variant == 1) lowpass_sub2_px8_item<1>(o.in, o.out, o.p0, o.mb, i); else lowpass_sub2_px8_item<2>(o.in, o.out, o.p0, o.mb, i);
      break;
  }
}

__global__ void __launch_bounds__(256) k_pyrlk_prepare(const __grid_constant__ PrepProg P) {
  const long long gthreads = (long long)gridDim.x * blockDim.x, gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int gen = 0;
  for (int ph = 0; ph < P.nphases; ph++) {
    const int first = ph ? P.phase_end[ph - 1] : 0, last = P.phase_end[ph];
    long long total = 0;
    for (int o = first; o < last; o++) total += P.op[o].items;
    for (long long i = gtid; i < total; i += gthreads) {
      long long j = i;
      int o = first;
      while (j >= P.op[o].items) { j -= P.op[o].items; o++; }
      prep_item(P.op[o], j);
    }
    if (ph + 1 < P.nphases) grid_barrier(P.bar, gen);
  }
}

static int grid_for(long long items, int threads) {
  long long blocks = (items + threads - 1) / threads;
  long long cap = (long long)sm_count() * 16;
  if (blocks < 1) blocks = 1;
  return (int)(blocks < cap ? blocks : cap);
}

}  // namespace vppb

using namespace vppb;

extern "C" {

// ---- argument checks of one step: the stand-alone entry points run them, and vppb_pyrlk_prepare runs those of all its steps before it
// queues anything.  `who` names the step in the error text.
static int check_copy_mirror(const vppb_img* src, const vppb_img* dst, const char* who) {  // those of vppb_copy2d_mirror (pixelwise.cu)
  VPPB_REQUIRE(src && dst && src->base && dst->base, VPPB_E_ARG, "%s: NULL image", who);
  VPPB_REQUIRE(src->elem_bytes == dst->elem_bytes && src->elem_bytes <= 64, VPPB_E_ARG, "%s: element sizes differ", who);
  VPPB_REQUIRE(same_domain(src, dst), VPPB_E_ARG, "%s: needs equal domains", who);
  VPPB_REQUIRE(dst->border <= dst->nrows && dst->border <= dst->ncols, VPPB_E_BORDER, "%s: border %d larger than the image", who, dst->border);
  return VPPB_OK;
}
static int check_scharr(const vppb_img* in, const vppb_img* out, int mirror, const char* who) {
  VPPB_REQUIRE(in && out && in->base && out->base, VPPB_E_ARG, "%s: NULL image", who);
  VPPB_REQUIRE(in->elem_bytes == 1 && out->elem_bytes == 8, VPPB_E_ARG, "%s: needs u8 input and 8-byte output elements", who);
  VPPB_REQUIRE(in->nrows >= out->nrows && in->ncols >= out->ncols, VPPB_E_ARG, "%s: input smaller than output", who);
  VPPB_REQUIRE(in->border >= 1, VPPB_E_BORDER, "%s: input border %d < 1", who, in->border);
  VPPB_REQUIRE(((uintptr_t)out->base % 8) == 0 && (out->pitch % 8) == 0, VPPB_E_ARG, "%s: output not 8-byte aligned", who);
  const int mb = mirror ? out->border : 0;
  VPPB_REQUIRE(mb <= out->nrows && mb <= out->ncols, VPPB_E_BORDER, "%s: border %d larger than the output image", who, mb);
  return VPPB_OK;
}
static int check_lowpass(const vppb_img* in, const vppb_img* out, int kind, int mirror, const char* who) {
  VPPB_REQUIRE(in && out && in->base && out->base, VPPB_E_ARG, "%s: NULL image", who);
  VPPB_REQUIRE(kind >= 0 && kind <= 2, VPPB_E_ARG, "%s: kind %d", who, kind);
  const int e = kind == 0 ? 1 : 8;
  VPPB_REQUIRE(in->elem_bytes == e && out->elem_bytes == e, VPPB_E_ARG, "%s: element size must be %d for kind %d", who, e, kind);
  VPPB_REQUIRE(in->border >= 2, VPPB_E_BORDER, "%s: input border %d < 2", who, in->border);
  // pyramid.hh:140,154: level size 1 + n/2; any smaller output is a prefix of it
  VPPB_REQUIRE(out->nrows <= 1 + in->nrows / 2 && out->ncols <= 1 + in->ncols / 2, VPPB_E_ARG,
               "%s: output %dx%d larger than 1+n/2 of input %dx%d", who, out->nrows, out->ncols, in->nrows, in->ncols);
  const int mb = mirror ? out->border : 0;
  VPPB_REQUIRE(mb <= out->nrows && mb <= out->ncols, VPPB_E_BORDER, "%s: border %d larger than the output image", who, mb);
  return VPPB_OK;
}

static int scharr_u8(const vppb_img* in, const vppb_img* out, int as_float, int mirror, void* stream) {
  const int rc = check_scharr(in, out, mirror, mirror ? "vppb_scharr_u8_mirror" : "vppb_scharr_u8");
  if (rc != VPPB_OK) return rc;
  // fast path: 8-byte aligned input rows with >= 4 addressable bytes left of column 0 and enough row to the right
  // of the last group (the library layout pads rows to 128 B), 16-byte aligned output rows
  const int mb = mirror ? out->border : 0;
  const long long nb = border_items(out->nrows, out->ncols, mb);
  const int groups = (out->ncols + 7) / 8;
  const bool fast = ((uintptr_t)in->base % 8) == 0 && (in->pitch % 8) == 0 && ((uintptr_t)out->base % 16) == 0 && (out->pitch % 16) == 0 &&
                    in->align >= 16 && in->border >= 1 && (long long)groups * 8 + 4 <= in->pitch - (long long)in->align;
  if (fast) {
    const int grid = grid_for((long long)out->nrows * groups + nb, 256);
    if (as_float) k_scharr_u8_v8<true><<<grid, 256, 0, as_stream(stream)>>>(view(in), view(out), groups, mb);
    else k_scharr_u8_v8<false><<<grid, 256, 0, as_stream(stream)>>>(view(in), view(out), groups, mb);
  } else {
    const int grid = grid_for((long long)out->nrows * out->ncols + nb, 256);
    if (as_float) k_scharr_u8<true><<<grid, 256, 0, as_stream(stream)>>>(view(in), view(out), mb);
    else k_scharr_u8<false><<<grid, 256, 0, as_stream(stream)>>>(view(in), view(out), mb);
  }
  VPPB_LAUNCH_CHECK("vppb_scharr_u8");
  return VPPB_OK;
}

int vppb_scharr_u8(const vppb_img* in, const vppb_img* out, int as_float, void* stream) { return scharr_u8(in, out, as_float, 0, stream); }
int vppb_scharr_u8_mirror(const vppb_img* in, const vppb_img* out, int as_float, void* stream) { return scharr_u8(in, out, as_float, 1, stream); }

static int lowpass_sub2(const vppb_img* in, const vppb_img* out, int kind, int mirror, void* stream) {
  const int rc = check_lowpass(in, out, kind, mirror, mirror ? "vppb_lowpass_sub2_mirror" : "vppb_lowpass_sub2");
  if (rc != VPPB_OK) return rc;
  const int mb = mirror ? out->border : 0;
  cudaStream_t st = as_stream(stream);
  const long long items = (long long)out->nrows * out->ncols * (kind == 0 ? 1 : 2);
  const int grid = grid_for(items, 256);
  if (kind == 0) {
    // fast path needs the library layout (4 bytes left / 20 bytes right of the domain inside the row) and 8-byte aligned output rows
    const bool fast = in->align >= 32 && ((uintptr_t)in->base % 16) == 0 && (in->pitch % 16) == 0 && ((uintptr_t)out->base % 8) == 0 &&
                      (out->pitch % 8) == 0 && in->nrows >= 4 && in->ncols >= 4;
    if (fast) {
      const int fast_rows = std::min(out->nrows, (in->nrows + 1) / 2), fast_cols = std::min(out->ncols, (in->ncols + 1) / 2);
      const int groups = (fast_cols + 7) / 8;
      const long long work = (long long)((fast_rows + 1) / 2) * groups + out->nrows + out->ncols;
      k_lowpass_sub2_u8_fast<<<grid_for(work, 128), 128, 0, st>>>(view(in), view(out), fast_rows, fast_cols, groups, mb);
    } else {
      k_lowpass_sub2<0><<<grid, 256, 0, st>>>(view(in), view(out), 2, mb);
    }
  }
  else {
    const int aligned16 = (((uintptr_t)in->base % 16) == 0 && (in->pitch % 16) == 0) ? 1 : 0;
    const int g2 = grid_for((long long)out->nrows * out->ncols, 256);
    if (kind == 1) k_lowpass_sub2_px8<1><<<g2, 256, 0, st>>>(view(in), view(out), aligned16, mb);
    else k_lowpass_sub2_px8<2><<<g2, 256, 0, st>>>(view(in), view(out), aligned16, mb);
  }
  VPPB_LAUNCH_CHECK("vppb_lowpass_sub2");
  return VPPB_OK;
}

int vppb_lowpass_sub2(const vppb_img* in, const vppb_img* out, int kind, void* stream) { return lowpass_sub2(in, out, kind, 0, stream); }
int vppb_lowpass_sub2_mirror(const vppb_img* in, const vppb_img* out, int kind, void* stream) { return lowpass_sub2(in, out, kind, 1, stream); }


// ---- the ops of the fused vppb_pyrlk_prepare: the same checks and the same choice of variant as the stand-alone entry points ----
static bool prep_copy_mirror(const vppb_img* src, const vppb_img* dst, PrepOp& o) {
  if (!src || !dst || !src->base || !dst->base || src->elem_bytes != dst->elem_bytes || src->elem_bytes > 64 || !same_domain(src, dst)) return false;
  if (dst->border > dst->nrows || dst->border > dst->ncols || src->base == dst->base) return false;
  if (((uintptr_t)src->base % 16) || ((uintptr_t)dst->base % 16) || (src->pitch % 16) || (dst->pitch % 16)) return false;
  const long long wbytes = (long long)src->ncols * src->elem_bytes;
  o.kind = PREP_COPY_MIRROR; o.variant = 0; o.in = view(src); o.out = view(dst);
  o.p0 = (int)(wbytes / 16); o.p1 = (int)(wbytes - (long long)o.p0 * 16); o.p2 = src->elem_bytes; o.mb = dst->border;
  o.items = copy_mirror_items(o.out, o.p0, o.p1);
  return true;
}
static bool prep_scharr(const vppb_img* in, const vppb_img* out, int as_float, PrepOp& o) {
  if (!in || !out || !in->base || !out->base || in->elem_bytes != 1 || out->elem_bytes != 8 || in->nrows < out->nrows || in->ncols < out->ncols) return false;
  if (in->border < 1 || ((uintptr_t)out->base % 8) || (out->pitch % 8) || out->border > out->nrows || out->border > out->ncols) return false;
  const int mb = out->border, groups = (out->ncols + 7) / 8;
  const bool fast = ((uintptr_t)in->base % 8) == 0 && (in->pitch % 8) == 0 && ((uintptr_t)out->base % 16) == 0 && (out->pitch % 16) == 0 &&
                    in->align >= 16 && (long long)groups * 8 + 4 <= in->pitch - (long long)in->align;
  o.kind = fast ? PREP_SCHARR_V8 : PREP_SCHARR_PX; o.variant = as_float ? 1 : 0; o.in = view(in); o.out = view(out);
  o.p0 = groups; o.p1 = o.p2 = 0; o.mb = mb;
  o.items = (fast ? (long long)out->nrows * groups : (long long)out->nrows * out->ncols) + border_items(out->nrows, out->ncols, mb);
  return true;
}
static bool prep_lowpass(const vppb_img* in, const vppb_img* out, int kind, PrepOp& o) {
  const int e = kind == 0 ? 1 : 8;
  if (!in || !out || !in->base || !out->base || in->elem_bytes != e || out->elem_bytes != e || in->border < 2) return false;
  if (out->nrows > 1 + in->nrows / 2 || out->ncols > 1 + in->ncols / 2 || out->border > out->nrows || out->border > out->ncols) return false;
  o.variant = kind; o.in = view(in); o.out = view(out); o.mb = out->border; o.p0 = o.p1 = o.p2 = 0;
  if (kind == 0) {
    const bool fast = in->align >= 32 && ((uintptr_t)in->base % 16) == 0 && (in->pitch % 16) == 0 && ((uintptr_t)out->base % 8) == 0 &&
                      (out->pitch % 8) == 0 && in->nrows >= 4 && in->ncols >= 4;
    if (fast) {
      o.kind = PREP_LP_U8_FAST;
      o.p0 = std::min(out->nrows, (in->nrows + 1) / 2); o.p1 = std::min(out->ncols, (in->ncols + 1) / 2); o.p2 = (o.p1 + 7) / 8;
      o.items = lowpass_u8_fast_items(out->nrows, out->ncols, o.p0, o.p1, o.p2);
    } else {
      o.kind = PREP_LP_GENERIC;
      o.items = (long long)out->nrows * out->ncols;
    }
  } else {
    o.kind = PREP_LP_PX8;
    o.p0 = (((uintptr_t)in->base % 16) == 0 && (in->pitch % 16) == 0) ? 1 : 0;
    o.items = (long long)out->nrows * out->ncols;
  }
  return true;
}

// barrier counters of the cooperative launches (64 slots handed out round-robin: a slot is zeroed on the stream right before its launch)
static int* prep_barrier_slot() {
  static std::atomic<int*> pool{nullptr};
  static std::atomic<unsigned> next{0};
  int* p = pool.load(std::memory_order_acquire);
  if (!p) {
    int* q = nullptr;
    if (cudaMalloc(&q, 64 * 256) != cudaSuccess) return nullptr;
    int* expected = nullptr;
    if (!pool.compare_exchange_strong(expected, q, std::memory_order_acq_rel)) { cudaFree(q); q = expected; }
    p = q;
  }
  return p + (size_t)(next.fetch_add(1) % 64) * 64;
}

// *why_not: NULL when the call was queued, else why the images do not fit the fused form (the caller has checked the arguments)
static int pyrlk_prepare_fused(const vppb_img* i1, const vppb_img* i2, const vppb_img* prev, const vppb_img* next, const vppb_img* grad, int nlevels,
                               int grad_is_float, cudaStream_t st, const char** why_not) {
  *why_not = "more than 8 levels";
  if (nlevels > PREP_MAX_LEVELS) return VPPB_OK;
  *why_not = "the images do not have the library layout";
  PrepProg P;
  memset(&P, 0, sizeof(P));
  int n = 0, ph = 0;
  const int gk = grad_is_float ? 2 : 1;
  if (!prep_copy_mirror(i1, &prev[0], P.op[n]) || !prep_copy_mirror(i2, &next[0], P.op[n + 1])) return VPPB_OK;
  n += 2; P.phase_end[ph++] = n;
  for (int l = 1; l <= nlevels; l++) {  // phase l
    if (grad) {
      if (l == 1) { if (!prep_scharr(&prev[0], &grad[0], grad_is_float, P.op[n])) return VPPB_OK; n++; }
      else { if (!prep_lowpass(&grad[l - 2], &grad[l - 1], gk, P.op[n])) return VPPB_OK; n++; }
    } else if (l == nlevels) {
      break;  // without a gradient pyramid the last phase is the one that writes level nlevels - 1 of the two u8 pyramids
    }
    if (l < nlevels) {
      if (!prep_lowpass(&prev[l - 1], &prev[l], 0, P.op[n]) || !prep_lowpass(&next[l - 1], &next[l], 0, P.op[n + 1])) return VPPB_OK;
      n += 2;
    }
    P.phase_end[ph++] = n;
  }
  P.nphases = ph;
  // the images of one call must be distinct buffers (a phase reads what an earlier phase wrote, never what it writes itself)
  P.bar = prep_barrier_slot();
  *why_not = "its grid barrier counters could not be allocated";
  if (!P.bar) return VPPB_OK;
  long long most = 0;
  for (int p = 0, first = 0; p < P.nphases; first = P.phase_end[p], p++) {
    long long t = 0;
    for (int o = first; o < P.phase_end[p]; o++) t += P.op[o].items;
    most = std::max(most, t);
  }
  long long blocks = (most + 255) / 256;
  const int cap = cooperative_grid_limit(k_pyrlk_prepare, 256);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  VPPB_CUDA(cudaMemsetAsync(P.bar, 0, sizeof(int), st));
  VPPB_CUDA(launch_cooperative(k_pyrlk_prepare, (int)blocks, 256, st, P));
  VPPB_LAUNCH_CHECK("vppb_pyrlk_prepare");
  *why_not = nullptr;
  return VPPB_OK;
}

// Every check each step of either form makes, in the order of the steps, before anything is queued: a rejected call writes nothing
// (and leaves no fork of `stream` unjoined).
static int pyrlk_prepare_check(const vppb_img* i1, const vppb_img* i2, const vppb_img* prev, const vppb_img* next, const vppb_img* grad, int nlevels,
                               int grad_is_float) {
  VPPB_REQUIRE(i1 && i2 && prev && next, VPPB_E_ARG, "vppb_pyrlk_prepare: NULL argument");
  VPPB_REQUIRE(nlevels >= 1 && nlevels <= 16, VPPB_E_ARG, "vppb_pyrlk_prepare: nlevels %d outside 1 .. 16", nlevels);
  int rc;
  if ((rc = check_copy_mirror(i1, &prev[0], "vppb_pyrlk_prepare: prev[0] <- i1"))) return rc;
  if ((rc = check_copy_mirror(i2, &next[0], "vppb_pyrlk_prepare: next[0] <- i2"))) return rc;
  if (grad && (rc = check_scharr(&prev[0], &grad[0], 1, "vppb_pyrlk_prepare: grad[0] <- scharr(prev[0])"))) return rc;
  char who[64];
  for (int l = 1; l < nlevels; l++) {
    snprintf(who, sizeof(who), "vppb_pyrlk_prepare: prev[%d] <- prev[%d]", l, l - 1);
    if ((rc = check_lowpass(&prev[l - 1], &prev[l], 0, 1, who))) return rc;
    snprintf(who, sizeof(who), "vppb_pyrlk_prepare: next[%d] <- next[%d]", l, l - 1);
    if ((rc = check_lowpass(&next[l - 1], &next[l], 0, 1, who))) return rc;
    snprintf(who, sizeof(who), "vppb_pyrlk_prepare: grad[%d] <- grad[%d]", l, l - 1);
    if (grad && (rc = check_lowpass(&grad[l - 1], &grad[l], grad_is_float ? 2 : 1, 1, who))) return rc;
  }
  return VPPB_OK;
}

// pyramid2d<uchar> of two frames + the Scharr gradient pyramid of the first (what lucas_kanade.hpp:150-157 and every
// pyrlk_match caller build before matching: pyramid2d::update(i1), ::update(i2), scharr(prev[0], grad[0]),
// grad.propagate_level0()).  Nine small launches; the three chains (prev levels, next levels, gradient levels) are
// independent after the copy of frame 1, so they are queued on three streams (fork / join with events on `stream`, also
// valid inside a stream capture): the critical path is 4 launches instead of 9.
int vppb_pyrlk_prepare(const vppb_img* i1, const vppb_img* i2, const vppb_img* prev, const vppb_img* next, const vppb_img* grad, int32_t nlevels,
                       int32_t grad_is_float, void* stream) {
  int rc = pyrlk_prepare_check(i1, i2, prev, next, grad, nlevels, grad_is_float);
  if (rc != VPPB_OK) return rc;
  {  // Two forms.  "streams": one launch per step, the three independent chains on three streams (forked from / joined into `stream`);
     // "fused": ONE cooperative launch, the steps of a level concatenated into a phase, grid barriers between phases (needs the library
     // layout).  With the gradient pyramid the three concurrent chains are the default (a phase lasts as long as its slowest step, and
     // the chains overlap steps of different levels), without it (the two u8 pyramids of the semi-dense flow) the single launch is: see
     // DESIGN.md 3.3 for the H100 timings of both forms.  VPPB_PREPARE=fused|streams
     // overrides the choice ("fused" fails instead of falling back: tests).
    const char* e = getenv("VPPB_PREPARE");
    const bool want_fused = e ? !strcmp(e, "fused") : (grad == nullptr);
    if (want_fused) {
      const char* why_not = nullptr;
      rc = pyrlk_prepare_fused(i1, i2, prev, next, grad, nlevels, grad_is_float, as_stream(stream), &why_not);
      if (rc != VPPB_OK || !why_not) return rc;
      VPPB_REQUIRE(!e, VPPB_E_ARG, "vppb_pyrlk_prepare: VPPB_PREPARE=fused but %s", why_not);
    }
  }
  static thread_local cudaStream_t side[2] = {nullptr, nullptr};
  static thread_local cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  static thread_local int side_dev = -1;
  int dev = 0;
  VPPB_CUDA(cudaGetDevice(&dev));
  if (side_dev != dev) {
    for (int k = 0; k < 2; k++) VPPB_CUDA(cudaStreamCreateWithFlags(&side[k], cudaStreamNonBlocking));
    for (int k = 0; k < 4; k++) VPPB_CUDA(cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming));
    side_dev = dev;
  }
  cudaStream_t st = as_stream(stream);
  const int gk = grad_is_float ? 2 : 1;
  // fork: frame 2's pyramid on side[1]
  VPPB_CUDA(cudaEventRecord(ev[0], st));
  VPPB_CUDA(cudaStreamWaitEvent(side[1], ev[0], 0));
  if ((rc = vppb_copy2d_mirror(i2, &next[0], side[1]))) return rc;
  for (int l = 1; l < nlevels; l++)
    if ((rc = vppb_lowpass_sub2_mirror(&next[l - 1], &next[l], 0, side[1]))) return rc;
  VPPB_CUDA(cudaEventRecord(ev[1], side[1]));
  // frame 1: level 0, then the gradient chain forks on side[0]
  if ((rc = vppb_copy2d_mirror(i1, &prev[0], st))) return rc;
  VPPB_CUDA(cudaEventRecord(ev[2], st));
  VPPB_CUDA(cudaStreamWaitEvent(side[0], ev[2], 0));
  if (grad) {
    if ((rc = vppb_scharr_u8_mirror(&prev[0], &grad[0], grad_is_float, side[0]))) return rc;
    for (int l = 1; l < nlevels; l++)
      if ((rc = vppb_lowpass_sub2_mirror(&grad[l - 1], &grad[l], gk, side[0]))) return rc;
  }
  VPPB_CUDA(cudaEventRecord(ev[3], side[0]));
  for (int l = 1; l < nlevels; l++)
    if ((rc = vppb_lowpass_sub2_mirror(&prev[l - 1], &prev[l], 0, st))) return rc;
  // join
  VPPB_CUDA(cudaStreamWaitEvent(st, ev[1], 0));
  VPPB_CUDA(cudaStreamWaitEvent(st, ev[3], 0));
  return VPPB_OK;
}

}  // extern "C"
