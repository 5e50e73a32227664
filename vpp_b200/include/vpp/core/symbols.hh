// Named-argument options `_border = 3`, flags `_no_threads`: the subset of iod (github.com/matt-42/iod)
// that the Video++ dense-pixel API uses (reference: vpp/core/symbol_definitions.hh, vpp/algorithms/symbols.hh,
// iod::D / sio::has / sio::get as used in vpp/core/imageNd.hpp:106-121,153-158).
#pragma once
#include <tuple>
#include <type_traits>
#include <utility>

namespace vpp {
namespace s {

template <typename S, typename T>
struct opt {
  typedef S symbol_type;
  typedef T value_type;
  T value;
};

template <typename S>
struct symbol {
  typedef S symbol_type;
  template <typename T>
  constexpr opt<S, typename std::decay<T>::type> operator=(T&& v) const {
    return opt<S, typename std::decay<T>::type>{std::forward<T>(v)};
  }
};

#define VPP_DEFINE_SYMBOL(name)                      \
  struct _##name##_t : symbol<_##name##_t> {         \
    using symbol<_##name##_t>::operator=;            \
    constexpr _##name##_t() {}                       \
  };                                                 \
  static constexpr _##name##_t _##name{};

VPP_DEFINE_SYMBOL(border)
VPP_DEFINE_SYMBOL(aligned)
VPP_DEFINE_SYMBOL(data)
VPP_DEFINE_SYMBOL(pitch)
VPP_DEFINE_SYMBOL(no_threads)
VPP_DEFINE_SYMBOL(left_to_right)
VPP_DEFINE_SYMBOL(right_to_left)
VPP_DEFINE_SYMBOL(top_to_bottom)
VPP_DEFINE_SYMBOL(bottom_to_top)
VPP_DEFINE_SYMBOL(block_size)
VPP_DEFINE_SYMBOL(blockwise)
VPP_DEFINE_SYMBOL(local_maxima)
VPP_DEFINE_SYMBOL(mask)
VPP_DEFINE_SYMBOL(scores)
VPP_DEFINE_SYMBOL(max_points_per_block)
VPP_DEFINE_SYMBOL(keypoints)
VPP_DEFINE_SYMBOL(flow)
VPP_DEFINE_SYMBOL(winsize)
VPP_DEFINE_SYMBOL(nscales)
VPP_DEFINE_SYMBOL(niterations)
VPP_DEFINE_SYMBOL(min_ev)
VPP_DEFINE_SYMBOL(delta)
VPP_DEFINE_SYMBOL(prediction)
VPP_DEFINE_SYMBOL(ring)  // extension: _ring = 1 selects the true FAST ring (see include/vppb.h)
// shared by several algorithm headers (video_extruder, descriptor_matcher, optical_flow), which may be included together
VPP_DEFINE_SYMBOL(detector_th)
VPP_DEFINE_SYMBOL(search_radius)
VPP_DEFINE_SYMBOL(cell_width)

// symbol type of an option or of a bare flag
template <typename O>
struct symbol_of {
  typedef typename std::decay<O>::type::symbol_type type;
};

template <typename S, typename... O>
struct has_symbol;
template <typename S>
struct has_symbol<S> : std::false_type {};
template <typename S, typename O1, typename... O>
struct has_symbol<S, O1, O...>
    : std::conditional<std::is_same<S, typename symbol_of<O1>::type>::value, std::true_type, has_symbol<S, O...>>::type {};

template <typename... O>
struct options {
  std::tuple<O...> values;

  template <typename S>
  static constexpr bool has(const S&) {
    return has_symbol<S, O...>::value;
  }

  // get(_sym, default): the option's value if present, else the default
  template <typename S, typename D>
  auto get(const S&, const D& dflt) const {
    return get_impl<S, D, 0>(dflt, std::integral_constant<bool, (sizeof...(O) > 0)>());
  }

 private:
  template <typename S, typename D, std::size_t I>
  auto get_impl(const D& dflt, std::false_type) const {
    return dflt;
  }
  template <typename S, typename D, std::size_t I>
  auto get_impl(const D& dflt, std::true_type) const {
    typedef typename std::tuple_element<I, std::tuple<O...>>::type Oi;
    return pick<S, D, I>(dflt, std::integral_constant<bool, std::is_same<S, typename symbol_of<Oi>::type>::value>());
  }
  template <typename S, typename D, std::size_t I>
  auto pick(const D&, std::true_type) const {
    return value_of(std::get<I>(values));
  }
  template <typename S, typename D, std::size_t I>
  auto pick(const D& dflt, std::false_type) const {
    return get_impl<S, D, I + 1>(dflt, std::integral_constant<bool, (I + 1 < sizeof...(O))>());
  }
  template <typename S2, typename T>
  static T value_of(const opt<S2, T>& o) {
    return o.value;
  }
  template <typename F>
  static bool value_of(const symbol<F>&) {
    return true;
  }
};

template <typename... O>
options<typename std::decay<O>::type...> D(O&&... o) {
  return options<typename std::decay<O>::type...>{std::make_tuple(std::forward<O>(o)...)};
}

}  // namespace s

using namespace s;
}  // namespace vpp
