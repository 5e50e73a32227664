// iod::array_view(size, f) for the descriptor matcher build (build_ref_dm.sh puts this directory ahead of oracle/ref_shim): the
// i-th element is f(i) for a callable, as in ../../iod/array_view.hh, or f[i] for a pointer - the reference's
// sad_distance(size, int*, int*, th) (descriptor_matcher/distances.hh:33-37) wraps raw pointers.
#pragma once
#include <iod/symbol.hh>
#include <utility>
namespace iod {
template <typename F>
struct array_view_ {
  int size_; F f;
  int size() const { return size_; }
  template <typename G = F> auto operator[](int i) const -> decltype(std::declval<const G&>()(i)) { return f(i); }
  template <typename G = F> auto operator[](int i) const -> decltype(std::declval<const G&>()[i]) { return f[i]; }
};
template <typename F>
array_view_<F> array_view(int size, F f) { return array_view_<F>{size, f}; }
}  // namespace iod
