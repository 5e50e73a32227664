// C++ host API test of the SAD descriptor matchers (vpp/algorithms/descriptor_matcher.hh) and extract_patches (vpp/core/patch.hh):
// the reference's tests/descriptor_matcher.cc rewritten on this API - 100 x 10 and 200 x 10 int descriptors, brute force, then the
// grid-local matcher at R = 10000, s = 300 - checked the way the reference checks them (the reported distance is the pair's SAD
// and no train is closer), plus exact tie rules on duplicated u8 descriptors and the patch layout.
#undef NDEBUG
#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <vpp/vpp.hh>
#include <vpp/algorithms/descriptor_matcher.hh>
#include <vpp/core/patch.hh>

using namespace vpp;

template <typename T>
static int sad(const image2d<T>& a, int i, const image2d<T>& b, int j) {
  int s = 0;
  for (int k = 0; k < a.ncols(); k++) s += std::abs((int)a(i, k) - (int)b(j, k));
  return s;
}

struct match { int j, d; };

int main() {
  vppb_check(vppb_init(0));
  int bad = 0;
  image2d<int> D1(100, 10), D2(200, 10);
  for (int r = 0; r < 100; r++)
    for (int c = 0; c < 10; c++) D1(r, c) = rand() % 10000;
  for (int r = 0; r < 200; r++)
    for (int c = 0; c < 10; c++) D2(r, c) = rand() % 10000;

  std::vector<match> m(D1.nrows(), match{-1, -1});
  int calls = 0, last = -1;
  bruteforce_sad_matcher(D1, D2, _match = [&](int i, int j, int d) { m[i] = match{j, d}; calls++; bad += i <= last; last = i; });
  bad += calls != D1.nrows();
  for (int i = 0; i < D1.nrows(); i++) {
    bad += m[i].j < 0 || sad(D1, i, D2, m[i].j) != m[i].d;
    for (int j = 0; j < D2.nrows(); j++) bad += sad(D1, i, D2, j) < m[i].d || (sad(D1, i, D2, j) == m[i].d && j < m[i].j);
  }

  m.assign(D1.nrows(), match{-1, -1});
  std::vector<vint2> P1, P2;
  for (int i = 0; i < D1.nrows(); i++) P1.push_back(vint2(rand() % 1000, rand() % 1000));
  for (int i = 0; i < D2.nrows(); i++) P2.push_back(vint2(rand() % 1000, rand() % 1000));
  local_index1d_sad_descriptor_matcher(_query_positions = P1, _train_positions = P2, _query = D1, _train = D2, _approximation = 1,
                                       _search_radius = 10000, _cell_width = 300, _match = [&](int i, int j, int d) { m[i] = match{j, d}; });
  for (int i = 0; i < D1.nrows(); i++) {
    bad += m[i].j < 0 || m[i].j >= D2.nrows() || sad(D1, i, D2, m[i].j) != m[i].d;
    for (int j = 0; j < D2.nrows(); j++) bad += sad(D1, i, D2, j) < m[i].d;
  }

  // ties: every train equal, two per cell: brute force takes train 0; the local matcher the lowest train of the first cell of its
  // window in raster order
  image2d<unsigned char> Q(3, 5), T(6, 5);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 5; c++) Q(r, c) = 7;
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 5; c++) T(r, c) = 9;
  std::vector<vint2> qp = {vint2(15, 15), vint2(35, 5), vint2(500, 500)};
  std::vector<vint2> tp = {vint2(25, 25), vint2(12, 28), vint2(11, 19), vint2(5, 5), vint2(28, 1), vint2(-9, -9)};  // s = 10
  std::vector<match> mq(3, match{-1, -1});
  bruteforce_sad_matcher(Q, T, _match = [&](int i, int j, int d) { mq[i] = match{j, d}; });
  for (int i = 0; i < 3; i++) bad += mq[i].j != 0 || mq[i].d != 10;
  mq.assign(3, match{-1, -1});
  local_index1d_sad_descriptor_matcher(_query = Q, _train = T, _query_positions = qp, _train_positions = tp, _search_radius = 10,
                                       _cell_width = 10, _match = [&](int i, int j, int d) { mq[i] = match{j, d}; });
  // query 0: window cells (0..2, 0..2): (0, 0) holds trains 3 and 5 -> 3.  query 1: cells (2..4, 0..1): (2, 0) holds train 4.
  bad += mq[0].j != 3 || mq[0].d != 10 || mq[1].j != 4 || mq[2].j != -1;

  // patches: the layout element (r + h) * w + (c + h), zero rows outside domain + border
  image2d<unsigned char> img(12, 14, _border = 2);
  for (int r = -2; r < 14; r++)
    for (int c = -2; c < 16; c++) img(r, c) = (unsigned char)(r * 16 + c + 40);
  std::vector<vint2> kps = {vint2(0, 0), vint2(11, 13), vint2(-1, 4), vint2(5, 6)};
  image2d<unsigned char> P = extract_patches(kps, img, 5);
  bad += P.nrows() != 4 || P.ncols() != 25;
  for (int k = 0; k < 4; k++)
    for (int r = -2; r < 3; r++)
      for (int c = -2; c < 3; c++) {
        const int e = (r + 2) * 5 + (c + 2);
        const bool inside = kps[k][0] - 2 >= -2 && kps[k][0] + 2 <= 13 && kps[k][1] - 2 >= -2 && kps[k][1] + 2 <= 15;
        bad += P(k, e) != (inside ? img(kps[k][0] + r, kps[k][1] + c) : 0);
      }
  if (bad) printf("FAIL: %d checks\n", bad);
  else printf("ALL OK\n");
  return bad ? 1 : 0;
}
