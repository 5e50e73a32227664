/* vpp_oracle_dm.c — the SAD descriptor matchers, restated plainly (see vpp_oracle_dm.h).  Queries are independent: the timing
 * build runs them in parallel. */
#include "vpp_oracle_dm.h"

#include <limits.h>
#include <stdlib.h>

static int sad(const vo_img* q, const vo_img* t, int i, int j) {
  const unsigned char* a = q->base + (int64_t)i * q->pitch;
  const unsigned char* b = t->base + (int64_t)j * t->pitch;
  int s = 0;
  if (q->elem == 1) {
    for (int k = 0; k < q->ncols; k++) s += abs((int)a[k] - (int)b[k]);
  } else {
    const int32_t* x = (const int32_t*)a;
    const int32_t* y = (const int32_t*)b;
    for (int k = 0; k < q->ncols; k++) s += (int)((x[k] > y[k]) ? (uint32_t)x[k] - (uint32_t)y[k] : (uint32_t)y[k] - (uint32_t)x[k]);
  }
  return s;
}

static int descriptors_ok(const vo_img* q, const vo_img* t) {
  return q->ncols == t->ncols && q->elem == t->elem && (q->elem == 1 || q->elem == 4);
}

int vo_match_bruteforce_sad(const vo_img* q, const vo_img* t, int32_t* idx, int32_t* dist) {
  if (!descriptors_ok(q, t)) return -2;
#pragma omp parallel for schedule(dynamic, 16)
  for (int i = 0; i < q->nrows; i++) {
    int bj = -1, bd = INT_MAX;
    for (int j = 0; j < t->nrows; j++) {
      const int d = sad(q, t, i, j);
      if (bj < 0 || d < bd) {
        bj = j;
        bd = d;
      }
    }
    idx[i] = bj;
    dist[i] = bd;
  }
  return 0;
}

/* C's truncating division of a 64-bit numerator */
static int64_t cell_of(int64_t v, int32_t s) { return v / s; }

int vo_match_local_sad(const vo_img* q, const vo_img* t, const int32_t* qpos, const int32_t* tpos, int32_t R, int32_t s, int32_t* idx,
                       int32_t* dist) {
  if (!descriptors_ok(q, t) || s < 1 || R < 0) return -2;
#pragma omp parallel for schedule(dynamic, 16)
  for (int i = 0; i < q->nrows; i++) {
    const int64_t r0 = cell_of((int64_t)qpos[2 * i] - R, s), r1 = cell_of((int64_t)qpos[2 * i] + R, s);
    const int64_t c0 = cell_of((int64_t)qpos[2 * i + 1] - R, s), c1 = cell_of((int64_t)qpos[2 * i + 1] + R, s);
    int bj = -1, bd = INT_MAX;
    int64_t br = 0, bc = 0;
    for (int j = 0; j < t->nrows; j++) {
      if (tpos[2 * j] <= -s || tpos[2 * j + 1] <= -s) continue;
      const int64_t cr = tpos[2 * j] / s, cc = tpos[2 * j + 1] / s;
      if (cr < r0 || cr > r1 || cc < c0 || cc > c1) continue;
      const int d = sad(q, t, i, j);
      /* (distance, cell row, cell col, train index) lexicographically; j only grows */
      if (bj < 0 || d < bd || (d == bd && (cr < br || (cr == br && cc < bc)))) {
        bj = j;
        bd = d;
        br = cr;
        bc = cc;
      }
    }
    idx[i] = bj;
    dist[i] = bd;
  }
  return 0;
}
