// CPU run of the reductions' shared functors (pencilarrays.jl_b200/csrc/reduce_core.hpp) in the
// kernel's tree order (reduce.cu): per-thread runs over 16-byte units, the warp shuffle tree, the
// tree over the warps, the same two trees over the CTA partials, then the left fold of the rank
// partials and the final rounding.  Used by tests/test_reduce_core.py.
//
//   reduce_host_check <dtype> <map> <op> <G> <P> <n>
// stdin: a (n elements), b (n elements, PA_MAP_DOT only), the predicate's value (16 bytes);
// the n elements are dealt to P ranks in contiguous runs (rank r: [n r / P, n (r + 1) / P)), each
// rank reduced with G CTAs.  stdout: the result's bytes.
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <vector>

#include "../pencilarrays.jl_b200/csrc/reduce_core.hpp"

using namespace pa::red;

constexpr int RT = 256, RU = 4;  // as reduce.cu

template <class Rd> using AccT = typename Rd::A;

template <class Rd> static AccT<Rd> tree(std::vector<AccT<Rd>> v) {  // v: 32 lanes -> lane 0
  for (int o = 16; o > 0; o >>= 1) {
    std::vector<AccT<Rd>> w = v;
    for (int l = 0; l < 32; ++l) w[l] = Rd::comb(v[l], l + o < 32 ? v[l + o] : v[l]);
    v = w;
  }
  return v[0];
}
template <class Rd> static AccT<Rd> block(const std::vector<AccT<Rd>>& th) {  // RT threads
  std::vector<AccT<Rd>> warps(32, Rd::neutral());
  for (int w = 0; w < RT / 32; ++w)
    warps[w] = tree<Rd>(std::vector<AccT<Rd>>(th.begin() + 32 * w, th.begin() + 32 * w + 32));
  // second stage: offsets RT/64 .. 1 over lanes holding the warp results, neutral elsewhere
  std::vector<AccT<Rd>> v = warps;
  for (int o = RT / 64; o > 0; o >>= 1) {
    std::vector<AccT<Rd>> w = v;
    for (int l = 0; l < 32; ++l) w[l] = Rd::comb(v[l], l + o < 32 ? v[l + o] : v[l]);
    v = w;
  }
  return v[0];
}

template <class E, int M, int O>
static AccT<Red<E, M, O>> rank_partial(const E* a, const E* b, long long n, typename Red<E, M, O>::T ref,
                                       int p, int G) {
  using Rd = Red<E, M, O>;
  using A = AccT<Rd>;
  constexpr int V = 16 / sizeof(E);
  const long long nunits = n / V, tail = n - nunits * V;  // host arrays: head = 0
  const long long chunk = (nunits + G - 1) / G;
  std::vector<A> parts(G);
  for (int c = 0; c < G; ++c) {
    std::vector<A> th(RT, Rd::neutral());
    const long long u1 = std::min<long long>((c + 1) * chunk, nunits);
    for (int t = 0; t < RT; ++t) {
      A acc = Rd::neutral();
      for (long long u = c * chunk + t; u < u1; u += (long long)RT * RU)
        for (int k = 0; k < RU; ++k)
          if (u + k * RT < u1)
            for (int j = 0; j < V; ++j) {
              const long long i = (u + k * RT) * V + j;
              acc = Rd::comb(acc, Rd::elem(a[i], b[i], ref, p));
            }
      if (c == G - 1 && t < tail) {
        const long long i = nunits * V + t;
        acc = Rd::comb(acc, Rd::elem(a[i], b[i], ref, p));
      }
      th[t] = acc;
    }
    parts[c] = block<Rd>(th);
  }
  if (G == 1) return parts[0];
  std::vector<A> th(RT, Rd::neutral());
  for (int t = 0; t < RT; ++t)
    for (int i = t; i < G; i += RT) th[t] = Rd::comb(th[t], parts[i]);
  return block<Rd>(th);
}

template <class E, int M, int O>
static void run(const std::vector<unsigned char>& in, long long n, int G, int P, int p) {
  using Rd = Red<E, M, O>;
  const E* a = (const E*)in.data();
  const E* b = M == M_DOT ? a + n : a;
  typename Rd::T ref;
  memcpy(&ref, in.data() + (M == M_DOT ? 2 : 1) * n * sizeof(E), sizeof ref);
  AccT<Rd> acc = Rd::neutral();
  for (int r = 0; r < P; ++r) {
    const long long lo = n * r / P, hi = n * (r + 1) / P;
    acc = Rd::comb(acc, rank_partial<E, M, O>(a + lo, b + lo, hi - lo, ref, p, G));
  }
  const typename Rd::R res = Rd::finish(acc);
  fwrite(&res, sizeof res, 1, stdout);
}

template <class E, int M> static void by_op(int op, const std::vector<unsigned char>& in, long long n,
                                            int G, int P) {
  const int p = op >> 4;
  switch (op & 15) {
    case O_SUM: return run<E, M, O_SUM>(in, n, G, P, p);
    case O_ANY: return run<E, M, O_ANY>(in, n, G, P, p);
    case O_ALL: return run<E, M, O_ALL>(in, n, G, P, p);
  }
  if constexpr (Ordered<typename Mapped<E, M>::T>::value) {
    if ((op & 15) == O_MAX) return run<E, M, O_MAX>(in, n, G, P, p);
    if ((op & 15) == O_MIN) return run<E, M, O_MIN>(in, n, G, P, p);
  }
  exit(3);
}
template <class E> static void by_map(int map, int op, const std::vector<unsigned char>& in, long long n,
                                      int G, int P) {
  switch (map) {
    case M_ID: return by_op<E, M_ID>(op, in, n, G, P);
    case M_ABS: return by_op<E, M_ABS>(op, in, n, G, P);
    case M_ABS2: return by_op<E, M_ABS2>(op, in, n, G, P);
    case M_DOT: return by_op<E, M_DOT>(op, in, n, G, P);
  }
  exit(3);
}

int main(int argc, char** argv) {
  if (argc != 7) return 2;
  const int dtype = atoi(argv[1]), map = atoi(argv[2]), op = atoi(argv[3]), G = atoi(argv[4]),
            P = atoi(argv[5]);
  const long long n = atoll(argv[6]);
  const char* why = "";
  if (result_dtype(dtype, map, op, &why) < 0) {
    fprintf(stderr, "refused: %s\n", why);
    return 4;
  }
  std::vector<unsigned char> in;
  unsigned char buf[1 << 16];
  size_t k;
  while ((k = fread(buf, 1, sizeof buf, stdin)) > 0) in.insert(in.end(), buf, buf + k);
  switch (dtype) {
    case D_F64: by_map<double>(map, op, in, n, G, P); break;
    case D_F32: by_map<float>(map, op, in, n, G, P); break;
    case D_C64: by_map<c64>(map, op, in, n, G, P); break;
    case D_C32: by_map<c32>(map, op, in, n, G, P); break;
    case D_I32: by_map<int32_t>(map, op, in, n, G, P); break;
    case D_I64: by_map<long long>(map, op, in, n, G, P); break;
    default: return 3;
  }
  return 0;
}
