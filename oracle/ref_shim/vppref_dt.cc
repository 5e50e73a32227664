// C entry point over the reference's OWN distance transforms (/root/reference/vpp/algorithms/distance_transforms/
// distance_transforms.hh, included verbatim): the four chamfer lambdas, so that oracle/vpp_oracle_dt.c can be pinned to them and
// timed against them.  Built only where /root/reference exists (oracle/ref_shim/build_ref_dt.sh -> oracle/_ref/libvppref_dt*.so).
// Images are described like vo_img (host pointer to pixel (0,0), pitch, border) and wrapped zero-copy with the reference's
// `_data = , _pitch = ` constructor (imageNd.hpp:99-141), as in vppref.cc.
#include <vpp/vpp.hh>
#include <vpp/algorithms/distance_transforms/distance_transforms.hh>
#include <stdint.h>

using namespace vpp;

extern "C" {
typedef struct vo_img { unsigned char* base; int32_t nrows, ncols, pitch, border, elem; } vo_img;
}

template <typename V>
static image2d<V> wrap(const vo_img* d) {
  return image2d<V>(make_box2d(d->nrows, d->ncols), _data = (V*)d->base, _pitch = d->pitch, _border = d->border);
}

template <typename T>
static void run(const vo_img* in, const vo_img* out, int kind) {
  image2d<T> a = wrap<T>(in);
  image2d<int> s = wrap<int>(out);
  switch (kind) {
    case 0: d4_distance_transform(a, s); break;
    case 1: d8_distance_transform(a, s); break;
    case 2: d3_4_distance_transform(a, s); break;
    default: d5_7_11_distance_transform(a, s); break;
  }
}

extern "C" {
// kind 0 = d4, 1 = d8, 2 = d3-4, 3 = d5-7-11; in: unsigned char (in_is_i32 = 0) or int; out: int with border >= the mask's reach
// (the reference reads outside smaller borders).  Returns -2 for an argument the reference cannot take.
int vppref_distance_transform(const vo_img* in, int in_is_i32, const vo_img* out, int kind) {
  if (kind < 0 || kind > 3 || out->border < (kind == 3 ? 2 : 1) || in->nrows != out->nrows || in->ncols != out->ncols) return -2;
  if (in_is_i32) run<int>(in, out, kind);
  else run<unsigned char>(in, out, kind);
  return 0;
}
}  // extern "C"
