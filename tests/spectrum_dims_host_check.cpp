// CPU run of the spectrum geometry of reduce_core.hpp over chosen bin dims (spec_wavenumber,
// spec_weight, spec_k, spec_q with a bin mask, spec_bin), composed as k_spectrum_dims composes it
// (reduce.cu): for every mode of a global grid, its bin (-1: dropped) and weight.  Used by
// tests/test_spectrum_dims_capi.py to check bin assignment bit for bit against NumPy.
//
//   spectrum_dims_host_check <N> <n_1> .. <n_N> <rfft_dim> <rfft_n> <width> <nbins> <mask> <s_1> .. <s_N>
// mask bit d: logical dim d + 1 is a bin dim.  stdout: per mode in column-major order (dim 1
// fastest) the bin as int32, then the weight as int32, in two consecutive arrays.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../pencilarrays.jl_b200/csrc/reduce_core.hpp"

using namespace pa::red;

int main(int argc, char** argv) {
  int a = 1;
  const int N = atoi(argv[a++]);
  if (N < 1 || N > 8) return 2;
  std::vector<long long> n(N);
  long long total = 1;
  for (int d = 0; d < N; ++d) total *= (n[d] = atoll(argv[a++]));
  const int rfft_dim = atoi(argv[a++]);
  const long long rfft_n = atoll(argv[a++]);
  const double width = atof(argv[a++]);
  const int nbins = atoi(argv[a++]);
  const unsigned mask = (unsigned)atoi(argv[a++]);
  std::vector<double> s(N);
  for (int d = 0; d < N; ++d) s[d] = strtod(argv[a++], nullptr);
  if (a != argc) return 2;
  std::vector<int> bins(total), wts(total);
  std::vector<long long> c(N, 0);
  for (long long e = 0; e < total; ++e) {
    double k[8] = {0};
    int w = 1;
    for (int d = 0; d < N; ++d) {
      const bool r2c = d + 1 == rfft_dim;
      k[d] = spec_k(s[d], spec_wavenumber(c[d], n[d], r2c));
      if (r2c) w = spec_weight(c[d], rfft_n);
    }
    bins[e] = spec_bin(spec_q(N, k, mask), width, nbins);
    wts[e] = w;
    for (int d = 0; d < N; ++d) {
      if (++c[d] < n[d]) break;
      c[d] = 0;
    }
  }
  fwrite(bins.data(), sizeof(int), total, stdout);
  fwrite(wts.data(), sizeof(int), total, stdout);
  return 0;
}
