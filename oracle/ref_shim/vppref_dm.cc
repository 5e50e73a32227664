// C entry points over the reference's OWN descriptor matchers (/root/reference/vpp/algorithms/descriptor_matcher/, included
// verbatim): bruteforce_matcher and local_index1d_sad_descriptor_matcher with the reference's sad_distance, so that
// oracle/vpp_oracle_dm.c can be pinned to them and timed against them.  Built only where /root/reference exists
// (oracle/ref_shim/build_ref_dm.sh -> oracle/_ref/libvppref_dm*.so).  Descriptors are described like vo_img (host pointer to
// row 0, pitch); positions are (row, col) int pairs.
#include <vpp/vpp.hh>
#include <vpp/algorithms/descriptor_matcher.hh>
#include <stdint.h>
#include <climits>
#include <vector>

using namespace vpp;

extern "C" {
typedef struct vo_img { unsigned char* base; int32_t nrows, ncols, pitch, border, elem; } vo_img;
}

template <typename T>
static const T* row(const vo_img* d, int i) { return reinterpret_cast<const T*>(d->base + (int64_t)i * d->pitch); }

template <typename T>
static void bruteforce(const vo_img* q, const vo_img* t, int32_t* idx, int32_t* dist) {
  const int D = q->ncols;
  bruteforce_matcher(q->nrows, t->nrows,
                     _distance = [&](int i, int j, int th) { return sad_distance<int>(D, row<T>(q, i), row<T>(t, j), th); },
                     _match = [&](int i, int j, int d) { idx[i] = j; dist[i] = d; });
}

template <typename T>
static void local(const vo_img* q, const vo_img* t, const int32_t* qpos, const int32_t* tpos, int R, int s, int approximation,
                  int32_t* idx, int32_t* dist) {
  const int D = q->ncols;
  std::vector<vint2> P1, P2;
  for (int i = 0; i < q->nrows; i++) P1.push_back(vint2(qpos[2 * i], qpos[2 * i + 1]));
  for (int j = 0; j < t->nrows; j++) P2.push_back(vint2(tpos[2 * j], tpos[2 * j + 1]));
  for (int i = 0; i < q->nrows; i++) {
    idx[i] = -1;
    dist[i] = INT_MAX;
  }
  local_index1d_sad_descriptor_matcher(
      _query_positions = P1, _train_positions = P2,
      _query = iod::array_view(q->nrows, [&](int i) { return iod::array_view(D, row<T>(q, i)); }),
      _train = iod::array_view(t->nrows, [&](int j) { return iod::array_view(D, row<T>(t, j)); }),
      _approximation = approximation, _search_radius = R, _cell_width = s,
      _distance = [&](int i, int j, int th) { return sad_distance<int>(D, row<T>(q, i), row<T>(t, j), th); },
      _match = [&](int i, int j, int d) { idx[i] = j; dist[i] = d; });
}

extern "C" {
// bruteforce_matcher (bruteforce_matcher.hh:11-47) with sad_distance: needs at least one train (the reference reads train 0).
// Returns -2 for an argument the reference cannot take.
int vppref_match_bruteforce_sad(const vo_img* q, const vo_img* t, int32_t* idx, int32_t* dist) {
  if (t->nrows < 1 || q->ncols != t->ncols || q->elem != t->elem || (q->elem != 1 && q->elem != 4)) return -2;
  if (q->elem == 1) bruteforce<unsigned char>(q, t, idx, dist);
  else bruteforce<int>(q, t, idx, dist);
  return 0;
}

// local_index1d_sad_descriptor_matcher (local_index1d_sad_descriptor_matcher.hh:10-57, grid_index.hh, index1d.hh): queries
// without a match keep (-1, INT_MAX).  Needs every train coordinate > -s (the reference asserts) and s >= 1, R >= 0.
int vppref_match_local_sad(const vo_img* q, const vo_img* t, const int32_t* qpos, const int32_t* tpos, int R, int s, int approximation,
                           int32_t* idx, int32_t* dist) {
  if (s < 1 || R < 0 || q->ncols != t->ncols || q->elem != t->elem || (q->elem != 1 && q->elem != 4)) return -2;
  for (int j = 0; j < t->nrows; j++)
    if (tpos[2 * j] <= -s || tpos[2 * j + 1] <= -s) return -2;
  if (q->elem == 1) local<unsigned char>(q, t, qpos, tpos, R, s, approximation, idx, dist);
  else local<int>(q, t, qpos, tpos, R, s, approximation, idx, dist);
  return 0;
}
}  // extern "C"
