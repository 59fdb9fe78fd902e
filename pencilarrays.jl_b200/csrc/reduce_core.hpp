// Maps, ops and finalisation of the distributed reductions (reduce.cu), shared by the kernel and
// the CPU check (tests/reduce_host_check.cpp).  Everything here is __host__ __device__ and gives
// the same bits on both sides: products and sums that Julia evaluates with two roundings are
// written with the round-to-nearest intrinsics on the device, so that nvcc cannot contract them
// into FMAs.
//
// Semantics are Julia's (Base): abs of a complex value is hypot(re, im), abs2 of an integer wraps
// in the element type, max / min propagate NaN and order -0.0 below 0.0, sum of Int32 widens to
// Int64, any / all give Bool.
#pragma once
#include <cstdint>
#include <cmath>
#include <climits>
#include <cfloat>
#include <cstring>

#ifdef __CUDACC__
#define RHD __host__ __device__ __forceinline__
#else
#define RHD inline
#endif

namespace pa {
namespace red {

struct alignas(16) c64 { double re, im; };
struct alignas(8) c32 { float re, im; };

// values of pa_dtype / pa_reduce_map / pa_reduce_op and the predicates (op >> 4)
enum Dt { D_F64 = 0, D_F32 = 1, D_C64 = 2, D_C32 = 3, D_I32 = 4, D_I64 = 5, D_BOOL = 6 };
enum Map { M_ID = 0, M_ABS = 1, M_ABS2 = 2, M_DOT = 3 };
enum Op { O_SUM = 0, O_MAX = 1, O_MIN = 2, O_ANY = 3, O_ALL = 4 };
enum Pred { P_NONE = 0, P_EQ, P_NE, P_LT, P_LE, P_GT, P_GE, P_ISNAN, P_ISFINITE };

// ---- IEEE arithmetic without contraction -----------------------------------------------------
RHD double mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
RHD double add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
RHD double sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
RHD float mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
RHD float add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

RHD bool is_nan(double x) { return x != x; }
RHD bool is_nan(float x) { return x != x; }
RHD bool is_finite(double x) { return !is_nan(x) && fabs(x) != (double)INFINITY; }
RHD bool is_finite(float x) { return !is_nan(x) && fabsf(x) != INFINITY; }
RHD bool sign_bit(double x) {
  uint64_t u;
  memcpy(&u, &x, 8);
  return (u >> 63) != 0;
}
RHD bool sign_bit(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  return (u >> 31) != 0;
}

// ---- hypot without overflow or underflow for finite inputs ----------------------------------
// Borges' correction step ("An improved algorithm for hypot(a, b)", 2019, the variant without
// FMA): h = sqrt(a^2 + b^2) is refined by one Newton step whose residual is evaluated exactly
// enough to give the correctly rounded result in all but rare cases; inputs are scaled by 2^-600
// / 2^600 when a^2 would overflow or b^2 underflow.
RHD double hypot_kernel(double ax, double ay) {  // ax >= ay >= 0, no scaling needed
  const double h = sqrt(add(mul(ax, ax), mul(ay, ay)));
  double t1, t2;
  if (h <= mul(2.0, ay)) {
    const double d = sub(h, ay);
    t1 = mul(ax, sub(mul(2.0, d), ax));
    t2 = mul(sub(d, mul(2.0, sub(ax, ay))), d);
  } else {
    const double d = sub(h, ax);
    t1 = mul(mul(2.0, d), sub(ax, mul(2.0, ay)));
    t2 = add(mul(sub(mul(4.0, d), ay), ay), mul(d, d));
  }
  return sub(h, add(t1, t2) / mul(2.0, h));
}
RHD double hypot_d(double x, double y) {
  if (!is_finite(x) || !is_finite(y)) {
    if (fabs(x) == (double)INFINITY || fabs(y) == (double)INFINITY) return (double)INFINITY;
    return add(x, y);  // NaN
  }
  x = fabs(x);
  y = fabs(y);
  const double ax = x < y ? y : x, ay = x < y ? x : y;
  const double scale = 0x1p-600, large = 0x1p+511, tiny = 0x1p-511, eps = 0x1p-54;
  if (ax > large) {
    if (ay <= mul(ax, eps)) return add(ax, ay);
    return hypot_kernel(mul(ax, scale), mul(ay, scale)) / scale;
  }
  if (ay < tiny) {
    if (ax >= ay / eps) return add(ax, ay);
    return mul(hypot_kernel(ax / scale, ay / scale), scale);
  }
  if (ay <= mul(ax, eps)) return add(ax, ay);
  return hypot_kernel(ax, ay);
}
// single precision: squares and their sum are exact enough in double that one rounding of the
// double square root to float gives hypotf
RHD float hypot_f(float x, float y) {
  if (fabsf(x) == INFINITY || fabsf(y) == INFINITY) return INFINITY;
  const double xd = x, yd = y;
  return (float)sqrt(add(mul(xd, xd), mul(yd, yd)));
}

// ---- the value a map produces ----------------------------------------------------------------
template <class E> struct RealOf { using T = E; };
template <> struct RealOf<c64> { using T = double; };
template <> struct RealOf<c32> { using T = float; };
template <class E, int M> struct Mapped { using T = typename RealOf<E>::T; };
template <class E> struct Mapped<E, M_ID> { using T = E; };

RHD double f_abs(double x) { return fabs(x); }
RHD float f_abs(float x) { return fabsf(x); }
RHD int32_t f_abs(int32_t x) { return x < 0 ? (int32_t)(0u - (uint32_t)x) : x; }  // typemin stays
RHD long long f_abs(long long x) { return x < 0 ? (long long)(0ull - (unsigned long long)x) : x; }
RHD double f_abs(c64 z) { return hypot_d(z.re, z.im); }
RHD float f_abs(c32 z) { return hypot_f(z.re, z.im); }

// real(x * conj(y)); with y == x this is abs2(x), expression for expression
RHD double f_dot(double x, double y) { return mul(x, y); }
RHD float f_dot(float x, float y) { return mul(x, y); }
RHD int32_t f_dot(int32_t x, int32_t y) { return (int32_t)((uint32_t)x * (uint32_t)y); }
RHD long long f_dot(long long x, long long y) {
  return (long long)((unsigned long long)x * (unsigned long long)y);
}
RHD double f_dot(c64 x, c64 y) { return add(mul(x.re, y.re), mul(x.im, y.im)); }
RHD float f_dot(c32 x, c32 y) { return add(mul(x.re, y.re), mul(x.im, y.im)); }

template <int M> struct MapF;
template <> struct MapF<M_ID> {
  template <class E> RHD static E f(E x, E) { return x; }
};
template <> struct MapF<M_ABS> {
  template <class E> RHD static typename RealOf<E>::T f(E x, E) { return f_abs(x); }
};
template <> struct MapF<M_ABS2> {
  template <class E> RHD static typename RealOf<E>::T f(E x, E) { return f_dot(x, x); }
};
template <> struct MapF<M_DOT> {
  template <class E> RHD static typename RealOf<E>::T f(E x, E y) { return f_dot(x, y); }
};

// ---- predicates of any / all --------------------------------------------------------------------
template <class T> RHD bool p_nan(T x) { return is_nan(x); }
RHD bool p_nan(int32_t) { return false; }
RHD bool p_nan(long long) { return false; }
RHD bool p_nan(c64 z) { return is_nan(z.re) || is_nan(z.im); }
RHD bool p_nan(c32 z) { return is_nan(z.re) || is_nan(z.im); }
template <class T> RHD bool p_finite(T x) { return is_finite(x); }
RHD bool p_finite(int32_t) { return true; }
RHD bool p_finite(long long) { return true; }
RHD bool p_finite(c64 z) { return is_finite(z.re) && is_finite(z.im); }
RHD bool p_finite(c32 z) { return is_finite(z.re) && is_finite(z.im); }
template <class T> RHD bool p_eq(T a, T b) { return a == b; }
RHD bool p_eq(c64 a, c64 b) { return a.re == b.re && a.im == b.im; }
RHD bool p_eq(c32 a, c32 b) { return a.re == b.re && a.im == b.im; }

template <class T> struct Ordered { static constexpr bool value = true; };
template <> struct Ordered<c64> { static constexpr bool value = false; };
template <> struct Ordered<c32> { static constexpr bool value = false; };

template <class T, bool = Ordered<T>::value> struct Cmp {
  RHD static bool f(T x, T v, int p) {
    switch (p) {
      case P_LT: return x < v;
      case P_LE: return x <= v;
      case P_GT: return x > v;
      case P_GE: return x >= v;
    }
    return false;
  }
};
template <class T> struct Cmp<T, false> {  // refused on the host: no isless for complex values
  RHD static bool f(T, T, int) { return false; }
};

template <class T> RHD bool pred(T x, T v, int p) {
  switch (p) {
    case P_EQ: return p_eq(x, v);
    case P_NE: return !p_eq(x, v);
    case P_ISNAN: return p_nan(x);
    case P_ISFINITE: return p_finite(x);
  }
  return Cmp<T>::f(x, v, p);
}

// ---- accumulators and results ----------------------------------------------------------------
// sum: Float32 / ComplexF32 accumulate in fp64 (rounded once at the end), Int32 in Int64 (Julia's
// add_sum widens); max / min: the mapped type; any / all: 0 / 1
template <class T, int O> struct AccOf { using T_ = T; };
template <> struct AccOf<float, O_SUM> { using T_ = double; };
template <> struct AccOf<c32, O_SUM> { using T_ = c64; };
template <> struct AccOf<int32_t, O_SUM> { using T_ = long long; };
template <class T> struct AccOf<T, O_ANY> { using T_ = int; };
template <class T> struct AccOf<T, O_ALL> { using T_ = int; };

template <class T, int O> struct ResOf { using T_ = T; };
template <> struct ResOf<int32_t, O_SUM> { using T_ = long long; };
template <class T> struct ResOf<T, O_ANY> { using T_ = unsigned char; };
template <class T> struct ResOf<T, O_ALL> { using T_ = unsigned char; };

// element -> accumulator (before the op combines it)
RHD double lift_sum(float x) { return (double)x; }
RHD c64 lift_sum(c32 z) { return c64{(double)z.re, (double)z.im}; }
RHD long long lift_sum(int32_t x) { return (long long)x; }
template <class T> RHD T lift_sum(T x) { return x; }

// accumulator -> result (rounded once)
RHD float round_to(double a, float*) { return (float)a; }
RHD c32 round_to(c64 a, c32*) { return c32{(float)a.re, (float)a.im}; }
template <class A, class R> RHD R round_to(A a, R*) { return (R)a; }

// Julia's max / min on floats: NaN wins, -0.0 < 0.0 (fmax / fmin would drop the NaN)
template <class T> RHD T jl_max(T x, T y) {
  if (is_nan(x)) return x;
  if (is_nan(y)) return y;
  return (y > x || (sign_bit(y) < sign_bit(x))) ? y : x;
}
template <class T> RHD T jl_min(T x, T y) {
  if (is_nan(x)) return x;
  if (is_nan(y)) return y;
  return (y < x || (sign_bit(y) > sign_bit(x))) ? y : x;
}
RHD int32_t jl_max(int32_t x, int32_t y) { return y > x ? y : x; }
RHD int32_t jl_min(int32_t x, int32_t y) { return y < x ? y : x; }
RHD long long jl_max(long long x, long long y) { return y > x ? y : x; }
RHD long long jl_min(long long x, long long y) { return y < x ? y : x; }

RHD double plus(double a, double b) { return add(a, b); }
RHD float plus(float a, float b) { return add(a, b); }
RHD long long plus(long long a, long long b) {  // wraps like Julia's Int64 +
  return (long long)((unsigned long long)a + (unsigned long long)b);
}
RHD int32_t plus(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
RHD c64 plus(c64 a, c64 b) { return c64{add(a.re, b.re), add(a.im, b.im)}; }
RHD c32 plus(c32 a, c32 b) { return c32{add(a.re, b.re), add(a.im, b.im)}; }

template <class T> struct Lim;
template <> struct Lim<double> {
  RHD static double lo() { return -(double)INFINITY; }
  RHD static double hi() { return (double)INFINITY; }
};
template <> struct Lim<float> {
  RHD static float lo() { return -INFINITY; }
  RHD static float hi() { return INFINITY; }
};
template <> struct Lim<int32_t> {
  RHD static int32_t lo() { return INT32_MIN; }
  RHD static int32_t hi() { return INT32_MAX; }
};
template <> struct Lim<long long> {
  RHD static long long lo() { return LLONG_MIN; }
  RHD static long long hi() { return LLONG_MAX; }
};
template <class T> RHD T zero_of() { return T(0); }
template <> RHD c64 zero_of<c64>() { return c64{0.0, 0.0}; }
template <> RHD c32 zero_of<c32>() { return c32{0.f, 0.f}; }

// The op on accumulators: neutral element, combine, and how a mapped value enters.
template <int O> struct OpF;
template <> struct OpF<O_SUM> {
  template <class A> RHD static A neutral() { return zero_of<A>(); }
  template <class A> RHD static A comb(A a, A b) { return plus(a, b); }
  template <class A, class T> RHD static A in(T v, T, int) { return lift_sum(v); }
};
template <> struct OpF<O_MAX> {
  template <class A> RHD static A neutral() { return Lim<A>::lo(); }
  template <class A> RHD static A comb(A a, A b) { return jl_max(a, b); }
  template <class A, class T> RHD static A in(T v, T, int) { return v; }
};
template <> struct OpF<O_MIN> {
  template <class A> RHD static A neutral() { return Lim<A>::hi(); }
  template <class A> RHD static A comb(A a, A b) { return jl_min(a, b); }
  template <class A, class T> RHD static A in(T v, T, int) { return v; }
};
template <> struct OpF<O_ANY> {
  template <class A> RHD static A neutral() { return 0; }
  template <class A> RHD static A comb(A a, A b) { return a | b; }
  template <class A, class T> RHD static A in(T v, T ref, int p) { return pred(v, ref, p) ? 1 : 0; }
};
template <> struct OpF<O_ALL> {
  template <class A> RHD static A neutral() { return 1; }
  template <class A> RHD static A comb(A a, A b) { return a & b; }
  template <class A, class T> RHD static A in(T v, T ref, int p) { return pred(v, ref, p) ? 1 : 0; }
};

// Everything about one (element type, map, op): the types, one element's contribution, the
// combine and the final rounding.
template <class E, int M, int O> struct Red {
  using T = typename Mapped<E, M>::T;   // what the map produces (and the predicate compares)
  using A = typename AccOf<T, O>::T_;   // accumulator: rank partials and window slots
  using R = typename ResOf<T, O>::T_;   // the result's element type
  RHD static A neutral() { return OpF<O>::template neutral<A>(); }
  RHD static A elem(E x, E y, T ref, int p) {
    return OpF<O>::template in<A>(MapF<M>::f(x, y), ref, p);
  }
  RHD static A comb(A a, A b) { return OpF<O>::comb(a, b); }
  RHD static R finish(A a) { return round_to(a, (R*)nullptr); }
};

// ---- the result-type table (pa_reduce_result_type) -------------------------------------------
// dtype / map / op as the C ABI passes them (op: the pa_reduce_op in the low 4 bits, the
// predicate above them).  Returns the result dtype, or -1 for a combination Julia refuses or the
// library does not provide; *why names the reason.
inline int result_dtype(int dtype, int map, int op, const char** why) {
  const int base = op & 15, p = op >> 4;
  *why = "";
  if (dtype < D_F64 || dtype > D_I64) return *why = "unknown element type", -1;
  if (map < M_ID || map > M_DOT) return *why = "unknown map", -1;
  if (base < O_SUM || base > O_ALL) return *why = "unknown op", -1;
  const bool cplx = dtype == D_C64 || dtype == D_C32;
  const bool pred_op = base == O_ANY || base == O_ALL;
  if (pred_op && (p < P_EQ || p > P_ISFINITE))
    return *why = "any / all need one predicate (PA_PRED_*)", -1;
  if (!pred_op && p != P_NONE) return *why = "a predicate goes with any / all only", -1;
  // the value the op sees: complex only under identity
  const bool cval = cplx && map == M_ID;
  const int real = dtype == D_C64 ? D_F64 : dtype == D_C32 ? D_F32 : dtype;
  const int val = cval ? dtype : real;
  if (cval && (base == O_MAX || base == O_MIN))
    return *why = "max / min of complex values: complex numbers are not ordered (no isless)", -1;
  if (cval && pred_op && p >= P_LT && p <= P_GE)
    return *why = "ordered comparison of complex values (no isless)", -1;
  if (pred_op) return D_BOOL;
  if (base == O_SUM && val == D_I32) return D_I64;
  return val;
}

// ---- shell-binned spectra (pa_shell_spectrum, DESIGN §3m) ---------------------------------------
// The one place that knows the geometry of a spectrum; the kernel, the default bin count and the
// CPU check (tests/spectrum_host_check.cpp) all call these.  Every floating operation is one
// correctly rounded IEEE operation, so a mode's bin is bit for bit what NumPy computes.
RHD double sqrt_rn(double x) {
#ifdef __CUDA_ARCH__
  return __dsqrt_rn(x);
#else
  return sqrt(x);
#endif
}
RHD double div_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// integer wavenumber of global index i along a dim of global extent n (numpy's fftfreq order);
// along the r2c dim the index is the wavenumber
RHD long long spec_wavenumber(long long i, long long n, bool r2c) {
  return r2c || i < (n + 1) / 2 ? i : i - n;
}
// Hermitian weight along the r2c dim of a real length n: 1 at i = 0 and (n even) i = n / 2, else 2
RHD int spec_weight(long long i, long long n) {
  return i == 0 || (n % 2 == 0 && i == n / 2) ? 1 : 2;
}
// k_d = s_d * wavenumber, and its square (the term of q)
RHD double spec_k(double s, long long nt) { return mul(s, (double)nt); }
// the shell of q = k_1^2 + k_2^2 + ... (summed in logical-dim order): floor(sqrt(q) / width + 0.5)
// as a double (it may exceed every integer type); width == 1 divides exactly
RHD double spec_shell(double q, double width) {
  return floor(add(div_rn(sqrt_rn(q), width), 0.5));
}
// the bin of a mode, or -1 when it is at or beyond nbins
RHD int spec_bin(double q, double width, int nbins) {
  const double b = spec_shell(q, width);
  return b < (double)nbins ? (int)b : -1;
}

// Spectra over chosen dims (pa_shell_spectrum_dims, DESIGN §3n): only the bin dims enter |k|.
// mask bit d set: logical dim d + 1 is a bin dim (every bit of the N dims: pa_shell_spectrum).
// q of a mode from its k_d in logical-dim order, the unbinned dims skipped
RHD double spec_q(int N, const double (&k)[8], unsigned mask) {
  double q = 0.0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int d = 0; d < 8; ++d)
    if (d < N && ((mask >> d) & 1)) q = add(q, mul(k[d], k[d]));
  return q;
}
// the bin of the extreme mode plus one (the default nbins): |k| grows with every |wavenumber|, so
// the corner of the largest |wavenumber| along each bin dim holds the last bin (a dim of extent 0
// or 1 adds 0); n: global extents in logical order, rfft_dim 1-based (0: none).  Saturates at
// 2^31 when the bin does not fit an int.
inline long long spec_default_bins(int N, const long long* n, int rfft_dim, const double* scales,
                                   double width, unsigned mask) {
  double k[8] = {0};
  for (int d = 0; d < N && d < 8; ++d) {
    const long long top = n[d] == 0 ? 0 : d + 1 == rfft_dim ? n[d] - 1 : n[d] / 2;
    k[d] = spec_k(scales ? scales[d] : 1.0, top);
  }
  const double b = spec_shell(spec_q(N, k, mask), width);
  return b + 1.0 > (double)INT32_MAX ? (long long)INT32_MAX + 1 : (long long)b + 1;
}

}  // namespace red
}  // namespace pa
