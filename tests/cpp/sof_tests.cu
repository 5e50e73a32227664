// C++ host API test of sparse_optical_flow (vpp/algorithms/optical_flow.hh): both overloads, both modes, on frames the Python test
// writes to argv[1] (int32 nrows, ncols, border, nkeypoints; both frames border included; the keypoints).  Every callback is written to
// argv[2] in the order it fired, and tests/test_gpu_sparse_flow.py compares them with vpp_b200.sparse_optical_flow.  Checked here:
// the keypoints overload reports strictly increasing indices.
#undef NDEBUG
#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <vpp/vpp.hh>
#include <vpp/algorithms/optical_flow.hh>

using namespace vpp;

struct rec { int32_t i, r, c; float fr, fc; int32_t d; };

int main(int argc, char** argv) {
  if (argc != 3) { printf("usage: sof_tests in.bin out.bin\n"); return 2; }
  vppb_check(vppb_init(0));
  FILE* in = fopen(argv[1], "rb");
  int32_t hdr[4];
  assert(in && fread(hdr, 4, 4, in) == 4);
  const int nr = hdr[0], nc = hdr[1], b = hdr[2], nk = hdr[3];
  const int W = nc + 2 * b, H = nr + 2 * b;
  std::vector<unsigned char> f[2] = {std::vector<unsigned char>((size_t)H * W), std::vector<unsigned char>((size_t)H * W)};
  assert(fread(f[0].data(), 1, f[0].size(), in) == f[0].size() && fread(f[1].data(), 1, f[1].size(), in) == f[1].size());
  std::vector<vint2> kps(nk);
  assert(fread(kps.data(), 8, nk, in) == (size_t)nk);
  fclose(in);
  image2d<unsigned char> i1(nr, nc, _border = b), i2(nr, nc, _border = b);
  for (int r = -b; r < nr + b; r++)
    for (int c = -b; c < nc + b; c++) {
      i1(r, c) = f[0][(size_t)(r + b) * W + (c + b)];
      i2(r, c) = f[1][(size_t)(r + b) * W + (c + b)];
    }

  int bad = 0;
  FILE* out = fopen(argv[2], "wb");
  assert(out);
  for (int sub = 0; sub < 2; sub++) {
    std::vector<rec> a, k;
    auto f1 = [&](vint2 p, vfloat2 fl, int d) { a.push_back(rec{-1, p[0], p[1], fl[0], fl[1], d}); };
    if (sub) sparse_optical_flow(i1, i2, _flow = f1, _subpixelic, _winsize = 9, _search_radius = 40, _cell_width = 30, _nscales = 2);
    else sparse_optical_flow(i1, i2, _flow = f1, _winsize = 9, _search_radius = 40, _cell_width = 30);
    auto cb = [&](int i, vfloat2 np, int d) { k.push_back(rec{i, kps[i][0], kps[i][1], np[0], np[1], d}); };
    sparse_optical_flow(kps, cb, i1, i2, _subpixelic = sub == 1, _winsize = 9, _search_radius = 40, _cell_width = 30, _nscales = 2);
    for (size_t j = 1; j < k.size(); j++) bad += k[j].i <= k[j - 1].i;
    for (const std::vector<rec>* v : {&a, &k}) {
      const int32_t n = (int32_t)v->size();
      fwrite(&n, 4, 1, out);
      fwrite(v->data(), sizeof(rec), v->size(), out);
    }
  }
  fclose(out);
  if (bad) printf("FAIL: %d checks\n", bad);
  else printf("ALL OK\n");
  return bad ? 1 : 0;
}
