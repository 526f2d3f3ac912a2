// ORACLE — TEST INFRASTRUCTURE ONLY.
// Stand-in for the parts of Boost that the vendored odeint integrate.hpp (and with it integrate_adaptive, controlled_runge_kutta and
// runge_kutta_dopri5) and the reference's Quadrotor.cpp include. oracle/sim.mk generates one forwarding header per Boost header name
// (boost/config.hpp, boost/array.hpp, ...) that includes this file. Type traits, enable_if, ref, array and range begin / end / copy are
// defined; the fusion, units and mpl find_if / end / divides / placeholders names are only declared, since odeint uses them only in the
// specialisations for fusion sequences and unit-carrying states, which a boost::array<double, 22> state never instantiates.
#pragma once
#include <type_traits>
#include <functional>
#include <cstddef>
#include <algorithm>
#include <iterator>
#include <stdexcept>
#define BOOST_USING_STD_MAX() using std::max
#define BOOST_USING_STD_MIN() using std::min
#define BOOST_PREVENT_MACRO_SUBSTITUTION
#define BOOST_STATIC_ASSERT(x) static_assert(x, #x)
#define BOOST_MPL_HAS_XXX_TRAIT_DEF(name) \
    template <class T, class = void> struct has_##name : ::boost::mpl::bool_<false> {}; \
    template <class T> struct has_##name<T, typename ::boost::shim_void<typename T::name>::type> : ::boost::mpl::bool_<true> {};
#define BOOST_STATIC_ASSERT_MSG(x, msg) static_assert(x, msg)
namespace boost {
template <class T, T v> using integral_constant = std::integral_constant<T, v>;
typedef std::true_type true_type;
typedef std::false_type false_type;
template <class A, class B> struct is_same : std::is_same<A, B> {};
template <class T> struct remove_reference : std::remove_reference<T> {};
template <class T> struct remove_const : std::remove_const<T> {};
template <bool B, class T = void> struct enable_if_c { typedef T type; };
template <class T> struct enable_if_c<false, T> {};
template <class C, class T = void> struct enable_if : enable_if_c<C::value, T> {};
template <bool B, class T = void> struct disable_if_c { typedef T type; };
template <class T> struct disable_if_c<true, T> {};
template <class C, class T = void> struct disable_if : disable_if_c<C::value, T> {};
template <class T> class reference_wrapper {
    T *p;
public:
    typedef T type;
    explicit reference_wrapper(T &t) : p(&t) {}
    operator T &() const { return *p; }
    T &get() const { return *p; }
};
template <class T> reference_wrapper<T> ref(T &t) { return reference_wrapper<T>(t); }
template <class T> struct unwrap_reference { typedef T type; };
template <class T> struct unwrap_reference<reference_wrapper<T>> { typedef T type; };
template <class T> struct shim_void { typedef void type; };
template <class T, std::size_t N> struct array {
    T elems[N];
    typedef T value_type; typedef T *iterator; typedef const T *const_iterator; typedef std::size_t size_type;
    typedef T &reference; typedef const T &const_reference;
    T &operator[](std::size_t i) { return elems[i]; }
    const T &operator[](std::size_t i) const { return elems[i]; }
    T *begin() { return elems; } T *end() { return elems + N; }
    const T *begin() const { return elems; } const T *end() const { return elems + N; }
    static constexpr std::size_t size() { return N; }
};
template <class R> auto begin(R &r) -> decltype(r.begin()) { return r.begin(); }
template <class R> auto begin(const R &r) -> decltype(r.begin()) { return r.begin(); }
template <class R> auto end(R &r) -> decltype(r.end()) { return r.end(); }
template <class R> auto end(const R &r) -> decltype(r.end()) { return r.end(); }
template <class R> auto size(const R &r) -> decltype(r.size()) { return r.size(); }
template <class R, class O> O copy(const R &r, O out) { return std::copy(r.begin(), r.end(), out); }
namespace range { using boost::copy; }
namespace mpl {
template <bool B> struct bool_ : std::integral_constant<bool, B> { typedef bool_ type; };
typedef bool_<true> true_;
typedef bool_<false> false_;
template <std::size_t N> struct size_t : std::integral_constant<std::size_t, N> {};
template <class C, class T, class F> struct if_ { typedef typename std::conditional<C::value, T, F>::type type; };
template <class A, class B, class C = true_, class D = true_, class E = true_> struct and_ : bool_<A::value && B::value && C::value && D::value && E::value> {};
template <class A> struct not_ : bool_<!A::value> {};
template <class S, class P> struct find_if;
template <class S> struct end;
template <class A, class B> struct divides;
namespace placeholders { struct _1; }
using placeholders::_1;
}  // namespace mpl
namespace units {
template <class U, class T> class quantity;
template <class Q> struct get_dimension;
template <class Q> struct get_system;
template <class D, class S, class E = void> class unit;
struct dimensionless_type;
}  // namespace units
namespace fusion {
namespace traits { template <class T> struct is_sequence : std::false_type {}; }
template <class... T> struct vector;
template <class S> struct zip_view;
template <class... A> void for_each(A &&...);
template <class... A> bool all(A &&...);
template <class... A> int make_fused(A &&...);
}  // namespace fusion
}  // namespace boost
