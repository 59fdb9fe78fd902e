// CPU run of the single-precision instantiation of the shared FFT core
// (pencilarrays.jl_b200/csrc/fft_core.hpp with T = float): the radix plan, butterflies, padded
// indexing, digit-reversed read-out and real-line post- / pre-passes the PA_FFT_F32 kernels run,
// in fp32 arithmetic, with fp32 twiddles rounded from the same long-double values.
// TEST INFRASTRUCTURE -- not linked into libpa_b200, never used by the product.
//   fft32_host_check c L sign [logR1]  < L complex floats   > L complex floats
//   fft32_host_check r N -1            < N floats           > N/2+1 complex floats  (r2c)
//   fft32_host_check r N  1            < N/2+1 complex      > N floats   (unnormalised c2r)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

// the twiddle scheme the kernels compile (fft.cu): one table lookup per butterfly, the other
// powers by squaring / products
#define PA_FFT_TWIDDLE_LOOKUPS 1
#include "../pencilarrays.jl_b200/csrc/fft_core.hpp"

using namespace pa_fft;

struct Line {
  cplxf* p;
  cplxf get(int i) const { return p[pad_index(i)]; }
  void put(int i, cplxf v) { p[pad_index(i)] = v; }
};

static std::vector<cplxf> twiddles(int L) {
  std::vector<cplxf> tw(L);
  for (int k = 0; k < L; ++k) {
    long double a = -2.0L * 3.141592653589793238462643383279502884L * k / L;
    tw[k] = cplxf{(float)cosl(a), (float)sinl(a)};
  }
  return tw;
}

template <class Tw>
static void passes(Line& x, int L, int sign, const Radices& R, const Tw& twf) {
  int M = L;
  for (int pss = 0; pss < R.n; ++pss) {
    const int r = R.r[pss];
    for (int u = 0; u < L / r; ++u) {
      if (r == 2) butterfly<2>(x, u, L, M, sign, twf);
      if (r == 4) butterfly<4>(x, u, L, M, sign, twf);
      if (r == 8) butterfly<8>(x, u, L, M, sign, twf);
      if (r == 16) butterfly<16>(x, u, L, M, sign, twf);
    }
    M /= r;
  }
}

static int log2_exact(int n) {
  int k = 0;
  while ((1 << k) < n) ++k;
  return (1 << k) == n ? k : -1;
}

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const bool real = !strcmp(argv[1], "r");
  const int n = atoi(argv[2]), sign = atoi(argv[3]);
  if (!real) {
    const int L = n, logL = log2_exact(L);
    if (logL < 0) return 3;
    std::vector<cplxf> in(L), buf(padded_pitch(L));
    const std::vector<cplxf> tw = twiddles(L);
    if (fread(in.data(), sizeof(cplxf), L, stdin) != (size_t)L) return 4;
    Line x{buf.data()};
    for (int i = 0; i < L; ++i) x.put(i, in[i]);
    const int logR1 = argc > 4 ? atoi(argv[4]) : 0;
    const Radices R = logR1 > 0 ? radices_with_first(logL, logR1) : radices_of(logL);
    passes(x, L, sign, R, [&](int i) { return tw[i]; });
    std::vector<cplxf> out(L);
    for (int k = 0; k < L; ++k) out[k] = x.get(fft_position_of(k, L, R));
    fwrite(out.data(), sizeof(cplxf), L, stdout);
    return 0;
  }
  const int N = n, L = N / 2, logL = log2_exact(L);
  if (N < 4 || logL < 0) return 3;
  const std::vector<cplxf> twN = twiddles(N);
  std::vector<cplxf> buf(padded_pitch(L + 1));
  Line x{buf.data()};
  if (sign < 0) {  // the real line's bytes are the complex line z
    std::vector<cplxf> in(L);
    if (fread(in.data(), sizeof(cplxf), L, stdin) != (size_t)L) return 4;
    for (int i = 0; i < L; ++i) x.put(i, in[i]);
  } else {  // N/2 + 1 bins, then the pre-pass in place
    std::vector<cplxf> in(L + 1);
    if (fread(in.data(), sizeof(cplxf), L + 1, stdin) != (size_t)(L + 1)) return 4;
    for (int i = 0; i <= L; ++i) x.put(i, in[i]);
    for (int k = 0; k <= L / 2; ++k) {
      cplxf zk, zl;
      brfft_pre_pair(k, x.get(k), x.get(L - k), twN[k], &zk, &zl);
      x.put(k, zk);
      if (k > 0) x.put(L - k, zl);
    }
  }
  const Radices R = radices_of(logL);
  passes(x, L, sign, R, [&](int i) { return twN[2 * i]; });
  auto Z = [&](int k) { return x.get(fft_position_of(k & (L - 1), L, R)); };
  if (sign < 0) {
    std::vector<cplxf> out(L + 1);
    for (int k = 0; k <= L / 2; ++k) rfft_post_pair(Z(k), Z(L - k), twN[k], &out[k], &out[L - k]);
    fwrite(out.data(), sizeof(cplxf), L + 1, stdout);
  } else {
    std::vector<cplxf> out(L);
    for (int i = 0; i < L; ++i) out[i] = Z(i);
    fwrite(out.data(), sizeof(cplxf), L, stdout);
  }
  return 0;
}
