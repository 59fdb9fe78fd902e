// Radix passes of the in-shared-memory 1-d complex FFT that the fused
// unpack+FFT kernel (fft.cu) runs on every line it has just transposed.
// SURVEY.md §8(f2): the permutation of a pencil exists to make the FFT axis
// contiguous (reference docs/src/Pencils.md:210-214,
// docs/src/Transpositions.md:7-9) -- here the transform is applied before the
// line ever leaves the SM.
//
// Algorithm: decimation in frequency (Gentleman-Sande), mixed radix
// {2, 4, 8}, in place.  A pass of radix R over sub-length M takes, for every
// group g and offset j < M/R, the R points x[g*M + j + q*M/R], replaces them
// by their R-point DFT and multiplies output s by W_M^(j*s).  After all
// passes the element at position p = s1*L/R1 + s2*L/(R1*R2) + ... holds
// X[s1 + R1*(s2 + R2*(...))]: fft_position_of() inverts that for the final
// natural-order read-out.  Twiddles come from a table W_L^k = exp(-2*pi*i*k/L),
// k < L, computed on the host in extended precision; the backward transform
// conjugates them (unnormalised, like FFTW / PencilFFTs).
//
// Everything is __host__ __device__ so that tests/fft_host_check.cpp can run
// the very same index arithmetic and butterflies on the CPU against numpy.fft.
#pragma once

#if defined(__CUDACC__)
#define PA_HD __host__ __device__ __forceinline__
#else
#define PA_HD inline
#endif

namespace pa_fft {

// complex of real type T: double (ComplexF64) or float (ComplexF32, PA_FFT_F32).  Both the
// storage and the arithmetic are in T; `cplx` is the double-precision type.
template <class T>
struct cplx_t {
  T x, y;
};
using cplx = cplx_t<double>;
using cplxf = cplx_t<float>;

template <class T>
PA_HD cplx_t<T> cadd(cplx_t<T> a, cplx_t<T> b) { return cplx_t<T>{a.x + b.x, a.y + b.y}; }
template <class T>
PA_HD cplx_t<T> csub(cplx_t<T> a, cplx_t<T> b) { return cplx_t<T>{a.x - b.x, a.y - b.y}; }
template <class T>
PA_HD cplx_t<T> cmul(cplx_t<T> a, cplx_t<T> b) {
  return cplx_t<T>{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x};
}
// multiplication by -i (forward) / +i (backward): sign = -1 forward, +1 backward
template <class T>
PA_HD cplx_t<T> mul_i(cplx_t<T> a, int sign) {
  return sign < 0 ? cplx_t<T>{a.y, -a.x} : cplx_t<T>{-a.y, a.x};
}

// storage index of logical position i: one pad element after every 8, 64 and 512
// elements, so that accesses at every power-of-8 stride (the strides of the radix-8
// passes and of the digit-reversed read-out) fall into different 16-byte bank groups.
// The same padding serves 8-byte (ComplexF32) elements: strides of 8, 64 and 512 points
// become 9, 73 and 585 stored elements, each 18 banks mod 32, and 18 i mod 32 is a distinct
// even bank for each of the 16 threads of a 64-bit shared-memory phase (DESIGN §3d)
PA_HD int pad_index(int i) { return i + (i >> 3) + (i >> 6) + (i >> 9); }
// elements per padded line, forced to 1 mod 8 (the C lines of a CTA are written
// column-wise by 8 consecutive threads; for 8-byte elements by 16, and 2 pitch mod 32 is
// then 2 or 18: distinct banks for all 16)
PA_HD int padded_pitch(int L) {
  int n = pad_index(L - 1) + 1;
  while ((n & 7) != 1) ++n;
  return n;
}

constexpr int MAX_PASSES = 5;
struct Radices {
  int n;
  int r[MAX_PASSES];
};

// small radix first (its stride is the longest: conflict-free), then radix 8
PA_HD Radices radices_of(int logL) {
  Radices R;
  R.n = 0;
  int rem = logL % 3;
  if (rem == 1) R.r[R.n++] = 2;
  if (rem == 2) R.r[R.n++] = 4;
  for (int i = 0; i < logL / 3; ++i) R.r[R.n++] = 8;
  return R;
}

// same, with a given first radix (the fused kernel's in-register first pass)
PA_HD Radices radices_with_first(int logL, int logR1) {
  Radices R;
  R.n = 0;
  if (logR1 > 0) R.r[R.n++] = 1 << logR1;
  const Radices rest = radices_of(logL - logR1);
  for (int i = 0; i < rest.n; ++i) R.r[R.n++] = rest.r[i];
  return R;
}

// position (after all passes) of output frequency k
PA_HD int fft_position_of(int k, int L, const Radices& R) {
  int p = 0, stride = L;
  for (int i = 0; i < R.n; ++i) {
    stride /= R.r[i];
    p += (k % R.r[i]) * stride;
    k /= R.r[i];
  }
  return p;
}

// R-point DFT in registers, a[q] -> A[s] = sum_q a[q] * w^(q*s), w = exp(sign*2*pi*i/R)
template <class T>
PA_HD void dft2(cplx_t<T>* a) {
  cplx_t<T> t = a[0];
  a[0] = cadd(t, a[1]);
  a[1] = csub(t, a[1]);
}
template <class T>
PA_HD void dft4(cplx_t<T>* a, int sign) {
  cplx_t<T> t0 = cadd(a[0], a[2]), t1 = csub(a[0], a[2]);
  cplx_t<T> t2 = cadd(a[1], a[3]), t3 = mul_i(csub(a[1], a[3]), sign);
  a[0] = cadd(t0, t2);
  a[1] = cadd(t1, t3);
  a[2] = csub(t0, t2);
  a[3] = csub(t1, t3);
}
template <class T>
PA_HD void dft8(cplx_t<T>* a, int sign) {
  using cplx = cplx_t<T>;
  const T h = T(0.70710678118654752440);
  // even / odd 4-point transforms
  cplx e[4] = {a[0], a[2], a[4], a[6]};
  cplx o[4] = {a[1], a[3], a[5], a[7]};
  dft4(e, sign);
  dft4(o, sign);
  // o[s] *= w8^s, w8 = exp(sign*i*pi/4)
  cplx w1 = cplx{h, sign * h}, w3 = cplx{-h, sign * h};
  o[1] = cmul(o[1], w1);
  o[2] = mul_i(o[2], sign);
  o[3] = cmul(o[3], w3);
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int s = 0; s < 4; ++s) {
    a[s] = cadd(e[s], o[s]);
    a[s + 4] = csub(e[s], o[s]);
  }
}

// 16 = 4 x 4: a[4*q1 + q2] -> A[s1 + 4*s2]
template <class T>
PA_HD void dft16(cplx_t<T>* a, int sign) {
  using cplx = cplx_t<T>;
  const T c1 = T(0.92387953251128675613), s1 = T(0.38268343236508977173);  // cos, sin(pi/8)
  const T h = T(0.70710678118654752440);
  cplx b[4][4];
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int q2 = 0; q2 < 4; ++q2) {
    cplx t[4] = {a[q2], a[4 + q2], a[8 + q2], a[12 + q2]};
    dft4(t, sign);
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int k = 0; k < 4; ++k) b[q2][k] = t[k];
  }
  // b[q2][s1] *= w16^(q2*s1), w16 = exp(sign*i*pi/8)
  const cplx w1 = cplx{c1, sign * s1}, w2 = cplx{h, sign * h}, w3 = cplx{s1, sign * c1};
  const cplx w6 = cplx{-h, sign * h}, w9 = cplx{-c1, -sign * s1};
  b[1][1] = cmul(b[1][1], w1);
  b[1][2] = cmul(b[1][2], w2);
  b[1][3] = cmul(b[1][3], w3);
  b[2][1] = cmul(b[2][1], w2);
  b[2][2] = mul_i(b[2][2], sign);   // w4 = sign*i
  b[2][3] = cmul(b[2][3], w6);
  b[3][1] = cmul(b[3][1], w3);
  b[3][2] = cmul(b[3][2], w6);
  b[3][3] = cmul(b[3][3], w9);
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 0; k < 4; ++k) {
    cplx t[4] = {b[0][k], b[1][k], b[2][k], b[3][k]};
    dft4(t, sign);
    a[k] = t[0];
    a[k + 4] = t[1];
    a[k + 8] = t[2];
    a[k + 12] = t[3];
  }
}

// the R-1 twiddles W^(step*s), s = 1..R-1, of one butterfly from the table entries at
// step, 2 step, 4 step (and 8 step): the others are one or two complex products away
template <int R, class T, class Tw>
PA_HD void butterfly_twiddles(cplx_t<T>* w, int step, int L, int sign, const Tw& tw) {
#if defined(PA_FFT_TWIDDLE_LOOKUPS) && PA_FFT_TWIDDLE_LOOKUPS == 1
  // one table lookup per butterfly, the powers by squaring / products (<= 4 roundings
  // more than a direct lookup: still far inside 8 eps log2(L))
  w[1] = tw(step & (L - 1));
  if (sign > 0) w[1].y = -w[1].y;
  if (R > 2) w[2] = cmul(w[1], w[1]);
  if (R > 4) w[4] = cmul(w[2], w[2]);
  if (R > 8) w[8] = cmul(w[4], w[4]);
#else
  w[1] = tw(step & (L - 1));
  if (R > 2) w[2] = tw((2 * step) & (L - 1));
  if (R > 4) w[4] = tw((4 * step) & (L - 1));
  if (R > 8) w[8] = tw((8 * step) & (L - 1));
  if (sign > 0) {
    w[1].y = -w[1].y;
    if (R > 2) w[2].y = -w[2].y;
    if (R > 4) w[4].y = -w[4].y;
    if (R > 8) w[8].y = -w[8].y;
  }
#endif
  if (R > 2) w[3] = cmul(w[1], w[2]);
  if (R > 4) {
    w[5] = cmul(w[4], w[1]);
    w[6] = cmul(w[4], w[2]);
    w[7] = cmul(w[4], w[3]);
  }
  if (R > 8) {
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int s = 1; s < 8; ++s) w[8 + s] = cmul(w[8], w[s]);
  }
}

// The R-point transform + twiddles of one butterfly on values already in registers
// (the fused kernel's first pass works on the rows it has just loaded from HBM).
template <int R, class T, class Tw>
PA_HD void butterfly_regs(cplx_t<T>* a, int j, int L, int M, int sign, const Tw& tw) {
  if (R == 2) dft2(a);
  if (R == 4) dft4(a, sign);
  if (R == 8) dft8(a, sign);
  if (R == 16) dft16(a, sign);
  const int step = j * (L / M);   // W_M^(j*s) = W_L^(j*s*L/M)
  if (step > 0) {
    cplx_t<T> w[R > 1 ? R : 2];
    butterfly_twiddles<R>(w, step, L, sign, tw);
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int s = 1; s < R; ++s) a[s] = cmul(a[s], w[s]);
  }
}

// One butterfly `u` (< L/R) of a pass with radix R over sub-length M on one line.
// x.get / x.put map a logical position to the (padded) storage; tw(i) = forward table
// entry W_L^i.  Only W^step, W^(2 step) and W^(4 step) are looked up: the other four
// twiddles of a radix-8 butterfly are one complex product away (<= 2 roundings more),
// which keeps the table traffic -- it shares the load/store path with shared memory --
// at 3/8 of the data traffic instead of 7/8.
template <int R, class Line, class Tw>
PA_HD void butterfly(Line& x, int u, int L, int M, int sign, const Tw& tw) {
  const int Q = M / R;            // stride between the R inputs
  const int g = u / Q, j = u % Q;
  const int base = g * M + j;
  decltype(x.get(0)) a[R];   // the line's element type: cplx or cplxf
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int q = 0; q < R; ++q) a[q] = x.get(base + q * Q);
  butterfly_regs<R>(a, j, L, M, sign, tw);
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int s = 0; s < R; ++s) x.put(base + s * Q, a[s]);
}

// ---- real lines through the complex core (rfft_ / brfft_, fft.cu) ----
// A real line x of N = 2L points is read as the complex line z[n] = x[2n] + i x[2n+1] of L
// points (its bytes, unchanged).  With Z = FFT_L(z) and w = W_N^k = exp(-2 pi i k / N):
//   X[k]     = E + w O,   E = (Z[k] + conj Z[L-k]) / 2,   O = -i (Z[k] - conj Z[L-k]) / 2
//   X[L - k] = conj(E - w O)
// (indices of Z mod L).  One call per pair k = 0 ... L/2 yields all N/2 + 1 bins: k = 0 gives X[0]
// and X[L] (both real), k = L/2 gives X[L/2] twice.
template <class T>
PA_HD void rfft_post_pair(cplx_t<T> zk, cplx_t<T> zl, cplx_t<T> w, cplx_t<T>* xk, cplx_t<T>* xl) {
  using cplx = cplx_t<T>;
  const T half = T(0.5);
  const cplx e = cplx{half * (zk.x + zl.x), half * (zk.y - zl.y)};
  const cplx o = cplx{half * (zk.y + zl.y), -half * (zk.x - zl.x)};
  const cplx wo = cmul(w, o);
  *xk = cadd(e, wo);
  *xl = cplx{e.x - wo.x, wo.y - e.y};
}

// Inverse of the above, unnormalised (FFTW's c2r): from the bins X[k], X[L-k] the pair of the
// complex spectrum whose inverse L-point transform is z[n] = x[2n] + i x[2n+1], N x = brfft(X):
//   F = X[k] + conj X[L-k],   G = (X[k] - conj X[L-k]) conj(w)
//   Z[k] = F + i G,   Z[L-k] = conj F + i conj G
// At k = 0 the partner is X[L]; the imaginary parts of X[0] and X[L] are dropped, as numpy and
// FFTW drop them (a real signal cannot have them); Z[L] is Z[0] and is not produced.
template <class T>
PA_HD void brfft_pre_pair(int k, cplx_t<T> xk, cplx_t<T> xl, cplx_t<T> w, cplx_t<T>* zk,
                          cplx_t<T>* zl) {
  using cplx = cplx_t<T>;
  if (k == 0) {
    xk.y = T(0);
    xl.y = T(0);
  }
  const cplx f = cplx{xk.x + xl.x, xk.y - xl.y};
  const cplx g = cmul(cplx{xk.x - xl.x, xk.y + xl.y}, cplx{w.x, -w.y});
  *zk = cplx{f.x - g.y, f.y + g.x};
  *zl = cplx{f.x + g.y, g.x - f.y};
}

// ---- real-to-real lines through the real-line core (r2r_, fft.cu; Makhoul's reordering) ----
// DCT-II (FFTW REDFT10) of x, N points: the line v[n] = x[2n], v[N-1-n] = x[2n+1] (n < N/2) goes
// through the forward real-line path (z[m] = v[2m] + i v[2m+1], the N/2-point passes,
// rfft_post_pair), which yields the bins V[0..N/2] of its N-point FFT.  With
// w = w_k = exp(-i pi k / 2N) and a = w V[k]:
//   Y[k] = 2 Re a,   Y[N-k] = -2 Im a          (k = 1 ... N/2; k = 0: Y[0] = 2 Re V[0])
// Both give the same value at k = N/2.
template <class T>
PA_HD void dct2_post_pair(cplx_t<T> v, cplx_t<T> w, T* yk, T* ynk) {
  const cplx_t<T> a = cmul(w, v);
  *yk = T(2) * a.x;
  *ynk = T(-2) * a.y;
}

// DCT-III (FFTW REDFT01), the inverse path: from s = (X[k], X[N-k]) (X[N] := 0) and w = w_k the
// bin V[k] = conj(w) (X[k] - i X[N-k]) = conj(w s), k = 0 ... N/2 (V[0] and V[N/2] are real).
// brfft_pre_pair and the inverse N/2-point passes then give z[m] = v[2m] + i v[2m+1], and
// x[2n] = v[n], x[2n+1] = v[N-1-n] undoes the reordering: REDFT01(REDFT10(x)) = 2N x.
template <class T>
PA_HD cplx_t<T> dct3_pre_pair(cplx_t<T> s, cplx_t<T> w) {
  const cplx_t<T> a = cmul(w, s);
  return cplx_t<T>{a.x, -a.y};
}

}  // namespace pa_fft
