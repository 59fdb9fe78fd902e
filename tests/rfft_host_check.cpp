// CPU run of the real-line transforms of the shared FFT core (pencilarrays.jl_b200/csrc/fft_core.hpp)
// in the order the rfft / brfft kernels run them: the same radix plan, butterflies, padded
// indexing, twiddle table of N entries (read at stride 2 by the L-point passes), post-pass /
// pre-pass on pairs (k, L - k) and digit-reversed read-out.
// TEST INFRASTRUCTURE -- not linked into libpa_b200, never used by the product.
//   rfft_host_check N -1 < N doubles > N/2+1 complex doubles      (forward, r2c)
//   rfft_host_check N  1 < N/2+1 complex doubles > N doubles      (backward, unnormalised c2r)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../pencilarrays.jl_b200/csrc/fft_core.hpp"

using namespace pa_fft;

struct Line {
  cplx* p;
  cplx get(int i) const { return p[pad_index(i)]; }
  void put(int i, cplx v) { p[pad_index(i)] = v; }
};

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const int N = atoi(argv[1]), sign = atoi(argv[2]);
  const int L = N / 2;
  int logL = 0;
  while ((1 << logL) < L) ++logL;
  if (N < 4 || (1 << logL) != L) return 3;
  std::vector<cplx> twN(N), buf(padded_pitch(L + 1));
  for (int k = 0; k < N; ++k) {
    long double a = -2.0L * 3.141592653589793238462643383279502884L * k / N;
    twN[k] = cplx{(double)cosl(a), (double)sinl(a)};
  }
  Line x{buf.data()};
  if (sign < 0) {  // the real line's bytes are the complex line z
    std::vector<cplx> in(L);
    if (fread(in.data(), sizeof(cplx), L, stdin) != (size_t)L) return 4;
    for (int i = 0; i < L; ++i) x.put(i, in[i]);
  } else {  // N/2 + 1 bins, then the pre-pass in place
    std::vector<cplx> in(L + 1);
    if (fread(in.data(), sizeof(cplx), L + 1, stdin) != (size_t)(L + 1)) return 4;
    for (int i = 0; i <= L; ++i) x.put(i, in[i]);
    for (int k = 0; k <= L / 2; ++k) {
      cplx zk, zl;
      brfft_pre_pair(k, x.get(k), x.get(L - k), twN[k], &zk, &zl);
      x.put(k, zk);
      if (k > 0) x.put(L - k, zl);
    }
  }
  const Radices R = radices_of(logL);
  auto twf = [&](int i) { return twN[2 * i]; };
  int M = L;
  for (int pss = 0; pss < R.n; ++pss) {
    const int r = R.r[pss];
    for (int u = 0; u < L / r; ++u) {
      if (r == 2) butterfly<2>(x, u, L, M, sign, twf);
      if (r == 4) butterfly<4>(x, u, L, M, sign, twf);
      if (r == 8) butterfly<8>(x, u, L, M, sign, twf);
    }
    M /= r;
  }
  auto Z = [&](int k) { return x.get(fft_position_of(k & (L - 1), L, R)); };
  if (sign < 0) {
    std::vector<cplx> out(L + 1);
    for (int k = 0; k <= L / 2; ++k) rfft_post_pair(Z(k), Z(L - k), twN[k], &out[k], &out[L - k]);
    fwrite(out.data(), sizeof(cplx), L + 1, stdout);
  } else {
    std::vector<cplx> out(L);
    for (int n = 0; n < L; ++n) out[n] = Z(n);
    fwrite(out.data(), sizeof(cplx), L, stdout);
  }
  return 0;
}
