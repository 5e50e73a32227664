/* Chamfer distance transforms (vpp/algorithms/distance_transforms/distance_transforms.hh:86-152): a literal serial restatement
 * of generic_incremental_distance_transform and its four masks - fill, zero, a forward raster pass of the forward half-mask,
 * the mirrored backward pass, both in place.  Deliberately NOT the closed form the CUDA kernels rely on, so that the closed form
 * (tests/dt_cases.py) stays an independent check of both.  TEST INFRASTRUCTURE ONLY, like vpp_oracle.c. */
#include "vpp_oracle_dt.h"

typedef struct { int dr, dc, w; } vo_dt_tap;

/* distance_transforms.hh:120-152, in the reference's order (the order does not change a min) */
static const vo_dt_tap FW4[] = {{-1, 0, 1}, {0, -1, 1}};
static const vo_dt_tap BW4[] = {{1, 0, 1}, {0, 1, 1}};
static const vo_dt_tap FW8[] = {{-1, -1, 1}, {-1, 0, 1}, {-1, 1, 1}, {0, -1, 1}};
static const vo_dt_tap BW8[] = {{1, 1, 1}, {1, 0, 1}, {1, -1, 1}, {0, 1, 1}};
static const vo_dt_tap FW34[] = {{-1, -1, 4}, {-1, 0, 3}, {-1, 1, 4}, {0, -1, 3}};
static const vo_dt_tap BW34[] = {{1, 1, 4}, {1, 0, 3}, {1, -1, 4}, {0, 1, 3}};
static const vo_dt_tap FW5711[] = {{-2, -1, 11}, {-2, 1, 11}, {-1, -2, 11}, {-1, -1, 7}, {-1, 0, 5}, {-1, 1, 7}, {-1, 2, 11}, {0, -1, 5}};
static const vo_dt_tap BW5711[] = {{0, 1, 5}, {1, -2, 11}, {1, -1, 7}, {1, 0, 5}, {1, 1, 7}, {1, 2, 11}, {2, -1, 11}, {2, 1, 11}};

static int32_t* at(const vo_img* s, int r, int c) { return (int32_t*)(s->base + (int64_t)r * s->pitch) + c; }

static void pass(const vo_img* s, const vo_dt_tap* taps, int n, int forward) {
  for (int k = 0; k < s->nrows; k++) {
    const int r = forward ? k : s->nrows - 1 - k;
    for (int j = 0; j < s->ncols; j++) {
      const int c = forward ? j : s->ncols - 1 - j;
      int32_t m = *at(s, r, c);
      for (int i = 0; i < n; i++) {
        const int32_t v = taps[i].w + *at(s, r + taps[i].dr, c + taps[i].dc);
        if (v < m) m = v;
      }
      *at(s, r, c) = m;
    }
  }
}

int vo_distance_transform(const vo_img* in, const vo_img* out, int kind) {
  static const vo_dt_tap* const fw[4] = {FW4, FW8, FW34, FW5711};
  static const vo_dt_tap* const bw[4] = {BW4, BW8, BW34, BW5711};
  static const int ntaps[4] = {2, 4, 4, 8};
  if (kind < 0 || kind > 3 || (in->elem != 1 && in->elem != 4) || out->elem != 4 || in->nrows != out->nrows || in->ncols != out->ncols)
    return -2;
  if (out->border < (kind == 3 ? 2 : 1)) return -3;
  const int32_t B = in->nrows + in->ncols;
  const int b = out->border;
  for (int r = -b; r < out->nrows + b; r++) /* fill_with_border(sedt, B) */
    for (int c = -b; c < out->ncols + b; c++) *at(out, r, c) = B;
  for (int r = 0; r < in->nrows; r++) /* if (i == 0) s = 0, on the domain */
    for (int c = 0; c < in->ncols; c++) {
      const unsigned char* p = in->base + (int64_t)r * in->pitch + (int64_t)c * in->elem;
      if (in->elem == 1 ? *p == 0 : *(const int32_t*)p == 0) *at(out, r, c) = 0;
    }
  pass(out, fw[kind], ntaps[kind], 1);
  pass(out, bw[kind], ntaps[kind], 0);
  return 0;
}
