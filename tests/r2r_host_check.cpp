// CPU run of the real-to-real line transforms of the shared FFT core
// (pencilarrays.jl_b200/csrc/fft_core.hpp) in the order the r2r kernel (fft.cu, k_r2r) runs them:
// the reordering load into the padded complex slots, the DCT-III pre step + brfft_pre_pair, the
// N/2-point passes (twiddle table of N entries read at stride 2), rfft_post_pair + the DCT-II post
// step, and the stores, with the DST sign and order changes in the load and the store.
// TEST INFRASTRUCTURE -- not linked into libpa_b200, never used by the product.
//   r2r_host_check d|f KIND N  < lines of N reals (double | float)  > as many lines of N reals
//   KIND: FFTW's value, 5 REDFT10 (DCT-II), 4 REDFT01 (DCT-III), 9 RODFT10, 8 RODFT01
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define PA_FFT_TWIDDLE_LOOKUPS 1
#include "../pencilarrays.jl_b200/csrc/fft_core.hpp"

using namespace pa_fft;

template <class T>
struct Line {
  cplx_t<T>* p;
  cplx_t<T> get(int i) const { return p[pad_index(i)]; }
  void put(int i, cplx_t<T> v) { p[pad_index(i)] = v; }
};

template <class T>
static std::vector<cplx_t<T>> twiddles(int L) {
  std::vector<cplx_t<T>> tw(L);
  for (int k = 0; k < L; ++k) {
    long double a = -2.0L * 3.141592653589793238462643383279502884L * k / L;
    tw[k] = cplx_t<T>{(T)cosl(a), (T)sinl(a)};
  }
  return tw;
}

template <class T>
static int run(int kind, int N) {
  const int L = N / 2;
  int logL = 0;
  while ((1 << logL) < L) ++logL;
  if (N < 4 || (1 << logL) != L) return 3;
  const bool fwd = kind == 5 || kind == 9, sine = kind == 8 || kind == 9;
  const std::vector<cplx_t<T>> twN = twiddles<T>(N), tw4 = twiddles<T>(4 * N);
  std::vector<T> in(N), out(N);
  while (fread(in.data(), sizeof(T), N, stdin) == (size_t)N) {
    std::vector<cplx_t<T>> buf(padded_pitch(fwd ? L : L + 1));
    Line<T> x{buf.data()};
    T* lr = reinterpret_cast<T*>(buf.data());
    for (int m = 0; m < L; ++m) {
      const T a = in[2 * m], b = in[2 * m + 1];
      if (fwd) {
        lr[2 * pad_index(m >> 1) + (m & 1)] = a;
        lr[2 * pad_index((N - 1 - m) >> 1) + ((N - 1 - m) & 1)] = sine ? -b : b;
      } else {
        const int ja = sine ? N - 1 - 2 * m : 2 * m, jb = sine ? N - 2 - 2 * m : 2 * m + 1;
        if (ja <= L) lr[2 * pad_index(ja)] = a;
        if (ja >= L) lr[2 * pad_index(N - ja) + 1] = a;
        if (jb <= L) lr[2 * pad_index(jb)] = b;
        if (jb >= L) lr[2 * pad_index(N - jb) + 1] = b;
      }
    }
    if (!fwd) {
      lr[1] = T(0);
      for (int k = 0; k <= L / 2; ++k) {
        const cplx_t<T> vk = dct3_pre_pair(x.get(k), tw4[k]);
        const cplx_t<T> vl = dct3_pre_pair(x.get(L - k), tw4[L - k]);
        cplx_t<T> zk, zl;
        brfft_pre_pair(k, vk, vl, twN[k], &zk, &zl);
        x.put(k, zk);
        if (k > 0) x.put(L - k, zl);
      }
    }
    const int sign = fwd ? -1 : 1;
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
    auto pos = [&](int k) { return fft_position_of(k & (L - 1), L, R); };
    if (fwd) {
      auto put = [&](int j, T y) { out[sine ? N - 1 - j : j] = y; };
      for (int k = 0; k <= L / 2; ++k) {
        cplx_t<T> vk, vl;
        rfft_post_pair(x.get(pos(k)), x.get(pos(L - k)), twN[k], &vk, &vl);
        T yk, ynk, yl, ynl;
        dct2_post_pair(vk, tw4[k], &yk, &ynk);
        dct2_post_pair(vl, tw4[L - k], &yl, &ynl);
        put(k, yk);
        if (k > 0 && k < L / 2) put(N - k, ynk);
        if (k < L / 2) put(L - k, yl);
        if (k > 0) put(L + k, ynl);
      }
    } else {
      for (int m = 0; m < L; ++m) {
        const int i = N - 1 - m;
        const T a = lr[2 * pad_index(pos(m >> 1)) + (m & 1)];
        const T b = lr[2 * pad_index(pos(i >> 1)) + (i & 1)];
        out[2 * m] = a;
        out[2 * m + 1] = sine ? -b : b;
      }
    }
    fwrite(out.data(), sizeof(T), N, stdout);
  }
  return 0;
}

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const int kind = atoi(argv[2]), N = atoi(argv[3]);
  if (kind != 4 && kind != 5 && kind != 8 && kind != 9) return 2;
  return !strcmp(argv[1], "f") ? run<float>(kind, N) : run<double>(kind, N);
}
