// C++ host API test of the chamfer distance transforms (vpp/algorithms/distance_transforms/distance_transforms.hh): the four names
// on small images - unsigned char and int inputs, borders 1 to 3, a view - against a serial restatement of the reference's two raster
// passes written out here, over the whole output buffer (borders included).
#undef NDEBUG
#include <cassert>
#include <cstdio>
#include <vector>
#include <vpp/vpp.hh>
#include <vpp/algorithms/distance_transforms/distance_transforms.hh>

using namespace vpp;

struct tap { int dr, dc, w; };

// fill with B, zero where the input is 0, forward pass with the forward half-mask, backward pass with its mirror
static std::vector<int> serial(const std::vector<int>& in, int nr, int nc, int b, int kind) {
  static const std::vector<tap> fw[4] = {
      {{-1, 0, 1}, {0, -1, 1}},
      {{-1, -1, 1}, {-1, 0, 1}, {-1, 1, 1}, {0, -1, 1}},
      {{-1, -1, 4}, {-1, 0, 3}, {-1, 1, 4}, {0, -1, 3}},
      {{-2, -1, 11}, {-2, 1, 11}, {-1, -2, 11}, {-1, -1, 7}, {-1, 0, 5}, {-1, 1, 7}, {-1, 2, 11}, {0, -1, 5}}};
  const int w = nc + 2 * b;
  std::vector<int> s((size_t)(nr + 2 * b) * w, nr + nc);
  auto at = [&](int r, int c) -> int& { return s[(size_t)(r + b) * w + (c + b)]; };
  for (int r = 0; r < nr; r++)
    for (int c = 0; c < nc; c++)
      if (in[(size_t)r * nc + c] == 0) at(r, c) = 0;
  for (int dir = 1; dir >= -1; dir -= 2)
    for (int k = 0; k < nr * nc; k++) {
      const int r = dir > 0 ? k / nc : nr - 1 - k / nc, c = dir > 0 ? k % nc : nc - 1 - k % nc;
      int m = at(r, c);
      for (const tap& t : fw[kind]) m = std::min(m, t.w + at(r + dir * t.dr, c + dir * t.dc));
      at(r, c) = m;
    }
  return s;
}

template <typename T, typename F>
static int check(F transform, int kind, int nr, int nc, int b, unsigned seed, int density) {
  std::vector<int> v((size_t)nr * nc);
  for (auto& x : v) {
    seed = seed * 1103515245u + 12345u;
    x = (int)((seed >> 16) % 100) < density ? 0 : (int)((seed >> 8) % 7) - 3 + 10;
  }
  image2d<T> a(nr, nc);
  for (int r = 0; r < nr; r++)
    for (int c = 0; c < nc; c++) a(r, c) = (T)v[(size_t)r * nc + c];
  image2d<int> s(nr, nc, _border = b);
  transform(a, s);
  const std::vector<int> ref = serial(v, nr, nc, b, kind);
  int bad = 0;
  for (int r = -b; r < nr + b; r++)
    for (int c = -b; c < nc + b; c++)
      if (s(r, c) != ref[(size_t)(r + b) * (nc + 2 * b) + (c + b)]) bad++;
  if (bad) printf("FAIL kind %d %dx%d border %d elem %d: %d pixels differ\n", kind, nr, nc, b, (int)sizeof(T), bad);
  return bad;
}

template <typename T>
static int all_kinds(int nr, int nc, int b, unsigned seed, int density) {
  int bad = 0;
  bad += check<T>(d4_distance_transform, 0, nr, nc, b, seed, density);
  bad += check<T>(d8_distance_transform, 1, nr, nc, b, seed, density);
  bad += check<T>(d3_4_distance_transform, 2, nr, nc, b, seed, density);
  if (b >= 2) bad += check<T>(d5_7_11_distance_transform, 3, nr, nc, b, seed, density);
  return bad;
}

int main() {
  vppb_check(vppb_init(0));
  int bad = 0;
  const int shapes[][2] = {{1, 1}, {1, 9}, {9, 1}, {2, 3}, {5, 9}, {17, 33}, {40, 3}, {3, 70}, {66, 65}};
  unsigned seed = 1;
  for (auto& sh : shapes)
    for (int b = 1; b <= 3; b++) {
      bad += all_kinds<unsigned char>(sh[0], sh[1], b, seed++, 5);
      bad += all_kinds<int>(sh[0], sh[1], b, seed++, 30);
    }
  bad += all_kinds<unsigned char>(20, 30, 2, 99, 0);    // no zero: every pixel is B
  bad += all_kinds<unsigned char>(20, 30, 2, 98, 100);  // only zeros

  {  // a view: its border is the parent's memory, and it becomes B
    image2d<unsigned char> a(12, 15);
    for (int r = 0; r < 12; r++)
      for (int c = 0; c < 15; c++) a(r, c) = (unsigned char)((r * 7 + c * 3) % 11);
    image2d<int> parent(20, 24, _border = 2);
    for (int r = -2; r < 22; r++)
      for (int c = -2; c < 26; c++) parent(r, c) = -7;
    image2d<int> view = parent | box2d(vint2(3, 5), vint2(14, 19));
    d5_7_11_distance_transform(a, view);
    std::vector<int> v(12 * 15);
    for (int r = 0; r < 12; r++)
      for (int c = 0; c < 15; c++) v[r * 15 + c] = a(r, c);
    const std::vector<int> ref = serial(v, 12, 15, 2, 3);
    for (int r = -2; r < 22; r++)
      for (int c = -2; c < 26; c++) {
        const int vr = r - 3, vc = c - 5;
        const bool inside = vr >= -2 && vr < 14 && vc >= -2 && vc < 17;
        const int want = inside ? ref[(size_t)(vr + 2) * 19 + (vc + 2)] : -7;
        if (parent(r, c) != want) { bad++; printf("FAIL view at (%d, %d): %d, expected %d\n", r, c, parent(r, c), want); }
      }
  }
  {  // a border below the mask's reach is refused
    image2d<unsigned char> a(4, 4);
    image2d<int> s(4, 4, _border = 1);
    bool threw = false;
    try { d5_7_11_distance_transform(a, s); } catch (std::runtime_error&) { threw = true; }
    assert(threw);
  }
  if (bad) return 1;
  printf("ALL OK\n");
  return 0;
}
