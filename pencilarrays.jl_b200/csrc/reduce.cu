// Distributed reductions over a PencilArray's parent array (reductions.jl:10-38): the local
// mapreduce and the combine across ranks in ONE kernel per rank and call.
//
// Local pass.  The array is one dense run of n elements.  G CTAs of RT threads (G =
// ceil(n / (V * RT * RU)) with V = 16 / elsize, at most R_CTAS_PER_SM per SM: it depends only on n
// and the device's SM count) each own a contiguous chunk of
// 16-byte units; thread t of a CTA folds units t, t + RT, t + 2 RT, ... in that order, RU units in
// flight per array (evict-first streaming loads: the data is read once).  The elements before the
// first 16-byte boundary (head, CTA 0) and after the last whole unit (tail, last CTA) are folded
// one by one, a whole array whose base is not 16-byte aligned modulo its element (ComplexF64 at an
// odd 8 bytes) or a second array aligned differently from the first loads every element alone.
// Each CTA reduces its threads with a warp shuffle tree (offsets 16 .. 1) and a tree over its
// warps (4, 2, 1), and writes its partial to a workspace; the last CTA to finish (fence + atomic
// ticket) folds the G partials with the same two trees, thread t taking partials t, t + RT, ...
// in order, and resets the ticket.
//
// Tree depth of a Float64 sum (a bound on the roundings any one element goes through):
//   run + 5 + 3 + ceil(G / RT) + 5 + 3 + (P - 1),
// run = the per-thread sequential run, ceil(ceil(nunits / G) / RT) * (16 / elsize) + 2 (head,
// tail); P - 1 for the fold of the P rank partials.  So |sum - exact| <= depth * eps * sum |f(x)|.
// Float32 / ComplexF32 sums accumulate in fp64 and are rounded once at the end.  The order of a
// float sum depends on n, the device, P and the base address modulo 16 (which elements are head
// and tail): the same array at the same address gives the same bits on every call, the same
// values at another alignment (an offset view) may differ in the last bits.
//
// Cross-rank step (P > 1), by thread 0 of the last CTA, through the communicator's flag window:
// store the rank partial into slot [parity][me] of every rank's window, signal FK_REDUCE with the
// call's sequence number seq to every peer, wait for every peer's signal >= seq, fold the P slots
// [parity][0 .. P-1] of the local window in rank order, finalise, store the result.  Every rank
// folds the same P values in the same order: every rank gets the same bits.
//
// Why two slot sets (parity = seq & 1) suffice.  Rank A stores into rank B's slot [k & 1][A] in
// call k and next in call k + 2.  A's call k + 2 kernel starts after A's call k + 1 kernel has
// finished (the reductions on one communicator are serialised by `done`), and that kernel waited
// for B's signal of seq k + 1.  B sends that signal from its call k + 1 kernel, which started
// after B's call k kernel finished -- the one that read slot [k & 1][A].  So the store of call
// k + 2 cannot overtake the read of call k.  Call k + 1 uses the other set, which call k does not
// touch.
//
// Without a flag window (an NCCL communicator across nodes, or nccl_fences) the kernel writes the
// rank partial, ncclAllGather collects the P partials and a one-CTA kernel folds them in rank order.
#include <cuda_runtime.h>

#include <cstring>
#include <map>
#include <mutex>

#include "flags.cuh"
#include "pa_internal.hpp"
#include "reduce_core.hpp"

namespace pa {

using namespace red;
typedef unsigned long long ull;

constexpr int RT = 256;            // threads per CTA
constexpr int RU = 4;              // 16-byte units in flight per thread and array
constexpr int R_CTAS_PER_SM = 4;   // grid cap: 1024 threads per SM, 64 KiB of loads in flight

#define CU(call)                                                                  \
  do {                                                                            \
    cudaError_t e_ = (call);                                                      \
    if (e_ != cudaSuccess) {                                                      \
      cudaGetLastError();                                                         \
      set_error("%s failed: %s", #call, cudaGetErrorString(e_));                  \
      return e_ == cudaErrorMemoryAllocation ? PA_ENOMEM : PA_ECUDA;              \
    }                                                                             \
  } while (0)

enum Combine { C_LOCAL = 0, C_FLAGS = 1, C_GATHER = 2 };

struct RArgs {
  const void* a;
  const void* b;
  i64 head, tail, nunits, chunk;  // elements before / after the units; units; units per CTA
  int G;
  int vec_a, vec_b;               // 16-byte loads possible on a / on b
  int pred;
  alignas(16) unsigned char ref[16];
  unsigned* ticket;
  unsigned char* part;            // G partials, 16 bytes each
  int mode;                       // Combine
  int nranks, rank;
  ull seq;
  ull* local_words;
  int word_stride;
  ull* const* remote_words;       // device table [nranks]
  unsigned char* const* peer_slots;  // device table [nranks]
  unsigned char* local_slots;
  ull timeout_ns;
  int* err;
  void* result;
  unsigned char* partial_out;     // C_GATHER: the rank partial
};

// ---- loads and 16-byte slots -----------------------------------------------------------------
__device__ __forceinline__ double ld1(const double* p) { return __ldcs(p); }
__device__ __forceinline__ float ld1(const float* p) { return __ldcs(p); }
__device__ __forceinline__ int32_t ld1(const int32_t* p) { return __ldcs((const int*)p); }
__device__ __forceinline__ long long ld1(const long long* p) { return __ldcs(p); }
__device__ __forceinline__ c64 ld1(const c64* p) { return c64{__ldcs(&p->re), __ldcs(&p->im)}; }
__device__ __forceinline__ c32 ld1(const c32* p) { return c32{__ldcs(&p->re), __ldcs(&p->im)}; }

template <class E>
__device__ __forceinline__ void ld_unit(const E* p, bool vec, E (&out)[16 / sizeof(E)]) {
  constexpr int V = 16 / sizeof(E);
  if (vec) {
    const int4 w = __ldcs((const int4*)p);
    memcpy(out, &w, 16);
  } else {
#pragma unroll
    for (int j = 0; j < V; ++j) out[j] = ld1(p + j);
  }
}

template <class A> __device__ __forceinline__ void st16(unsigned char* p, A v) {
  int4 w = make_int4(0, 0, 0, 0);
  memcpy(&w, &v, sizeof(A));
  *(int4*)p = w;
}
template <class A> __device__ __forceinline__ A ld16_cg(const unsigned char* p) {  // other SMs' stores
  const int4 w = __ldcg((const int4*)p);
  A v;
  memcpy(&v, &w, sizeof(A));
  return v;
}
template <class A> __device__ __forceinline__ A ld16_cv(const unsigned char* p) {  // other GPUs' stores
  const int4 w = __ldcv((const int4*)p);
  A v;
  memcpy(&v, &w, sizeof(A));
  return v;
}

template <class A> __device__ __forceinline__ A shfl_down(A v, int o) { return __shfl_down_sync(~0u, v, o); }
template <> __device__ __forceinline__ c64 shfl_down<c64>(c64 v, int o) {
  return c64{__shfl_down_sync(~0u, v.re, o), __shfl_down_sync(~0u, v.im, o)};
}

// shuffle tree over each warp (16, 8, 4, 2, 1), then over the RT/32 warp results (4, 2, 1);
// the CTA's value ends in thread 0
template <class Rd>
__device__ __forceinline__ typename Rd::A block_reduce(typename Rd::A v, typename Rd::A* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = Rd::comb(v, shfl_down(v, o));
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();  // (sh may still be read from an earlier call)
  if (l == 0) sh[w] = v;
  __syncthreads();
  if (w == 0) {
    v = l < RT / 32 ? sh[l] : Rd::neutral();
#pragma unroll
    for (int o = RT / 64; o > 0; o >>= 1) v = Rd::comb(v, shfl_down(v, o));
  }
  return v;
}

template <class E, int M, int O>
__global__ void __launch_bounds__(RT, R_CTAS_PER_SM) k_reduce(const RArgs g) {
  using Rd = Red<E, M, O>;
  using T = typename Rd::T;
  using A = typename Rd::A;
  constexpr int V = 16 / sizeof(E);
  __shared__ A sh[RT / 32];
  __shared__ int last;
  const E* a = (const E*)g.a;
  const E* b = M == M_DOT ? (const E*)g.b : a;
  T ref;
  memcpy(&ref, g.ref, sizeof(T));
  const int t = threadIdx.x, c = blockIdx.x;

  A acc = Rd::neutral();
  if (c == 0 && t < g.head) acc = Rd::comb(acc, Rd::elem(ld1(a + t), ld1(b + t), ref, g.pred));
  const E* ua = a + g.head;
  const E* ub = b + g.head;
  const i64 u1 = min(((i64)c + 1) * g.chunk, g.nunits);
  for (i64 u = (i64)c * g.chunk + t; u < u1; u += (i64)RT * RU) {
    E xa[RU][V], xb[RU][V];
#pragma unroll
    for (int k = 0; k < RU; ++k)
      if (u + k * RT < u1) {
        ld_unit(ua + (u + k * RT) * V, g.vec_a, xa[k]);
        if (M == M_DOT) ld_unit(ub + (u + k * RT) * V, g.vec_b, xb[k]);
      }
#pragma unroll
    for (int k = 0; k < RU; ++k)
      if (u + k * RT < u1) {
#pragma unroll
        for (int j = 0; j < V; ++j)
          acc = Rd::comb(acc, Rd::elem(xa[k][j], M == M_DOT ? xb[k][j] : xa[k][j], ref, g.pred));
      }
  }
  if (c == g.G - 1 && t < g.tail) {
    const i64 i = g.head + g.nunits * V + t;
    acc = Rd::comb(acc, Rd::elem(ld1(a + i), ld1(b + i), ref, g.pred));
  }

  acc = block_reduce<Rd>(acc, sh);
  if (g.G > 1) {
    if (t == 0) {
      st16(g.part + (size_t)c * 16, acc);
      __threadfence();
      last = atomicAdd(g.ticket, 1u) == (unsigned)g.G - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    acc = Rd::neutral();
    for (int i = t; i < g.G; i += RT) acc = Rd::comb(acc, ld16_cg<A>(g.part + (size_t)i * 16));
    acc = block_reduce<Rd>(acc, sh);
    if (t == 0) *g.ticket = 0;  // the next call (ordered after this one) starts from zero
  }
  if (t != 0) return;

  if (g.mode == C_GATHER) {
    st16(g.partial_out, acc);
    return;
  }
  if (g.mode == C_FLAGS) {
    const int P = g.nranks, me = g.rank;
    const size_t set = (size_t)(g.seq & 1) * P;
    st16(g.local_slots + (set + me) * 16, acc);
    for (int k = 1; k < P; ++k) {
      const int q = (me + k) % P;
      st16(g.peer_slots[q] + (set + me) * 16, acc);
    }
    for (int k = 1; k < P; ++k) flag_signal(g.remote_words[(me + k) % P], g.seq);
    for (int k = 1; k < P; ++k) {
      const int q = (me + P - k) % P;
      flag_wait(g.local_words + (size_t)q * g.word_stride, g.seq, g.timeout_ns, g.err);
    }
    acc = Rd::neutral();
    for (int q = 0; q < P; ++q) acc = Rd::comb(acc, ld16_cv<A>(g.local_slots + (set + q) * 16));
  }
  *(typename Rd::R*)g.result = Rd::finish(acc);
}

// ---- reductions along dims (pa_reduce_dims, DESIGN §3l) -----------------------------------------
// The local parent's dims (memory order, extra dims last), extent-1 dims dropped and neighbours of
// the same class merged, are kept (K) and reduced (R) runs.  Output o (column-major over the K
// runs, which is the result's layout) folds the elements koff(o) + roff(r) + i: r over the "rows"
// (the outer R runs, an odometer), i over the inner run -- the fastest run when it is reduced and
// long enough (the row regime: contiguous, 16-byte units when aligned), else length 1 (the column
// regime: consecutive threads own consecutive outputs).  A team of Wi x Wr threads folds one
// output: Wi lanes interleaved along each row's units, Wr contiguous blocks of rows; the CTA holds
// Oc teams (Wi * Wr * Oc = RT).  With few outputs the rows x units of each output tile are split
// over S = Sr x Si CTAs; their partials go to the workspace and the tile's last CTA (ticket) folds
// them.  With P > 1 each tile's rank partials go to this rank's own area of the flag window, and the
// last tile to finish (a second ticket) runs the combine.
constexpr int D_RUNS = PA_MAX_DIMS / 2;  // K runs and R runs alternate: at most 4 of each
// resident CTAs per SM the kernel is compiled for: 3 (at most 85 registers); 4 (64 registers)
// spills 24-224 bytes per thread in every instantiation
constexpr int D_CTAS_PER_SM = 3;

// The combine of a replicated or sliced result across ranks (P > 1): every rank has stored its
// nout partials (16-byte accumulators) into its own partial area of the flag window; the caller's
// last CTA signals every peer, waits for every peer and folds the group's areas in rank order.
struct GroupCombine {
  int nranks, rank;
  ull seq;
  ull* local_words;
  int word_stride;
  ull* const* remote_words;        // device table [nranks]
  unsigned char* const* areas;     // device table [nranks]: every rank's partial area as mapped here
  size_t area_off;                 // the parity set's offset in an area
  int topo_M;                      // the combine group: the ranks whose coordinates agree with
  int topo_dims[PA_MAX_TOPO];      //   mine on every grid dim of keep_grid (0: every rank)
  int coords[PA_MAX_TOPO];
  unsigned keep_grid;
  ull timeout_ns;
  int* err;
};

__device__ __forceinline__ bool in_group(const GroupCombine& g, int q) {
  for (int i = g.topo_M - 1; i >= 0; --i) {  // row-major rank numbering: the last coordinate fastest
    const int c = q % g.topo_dims[i];
    q /= g.topo_dims[i];
    if (((g.keep_grid >> i) & 1) && c != g.coords[i]) return false;
  }
  return true;
}

struct DArgs {
  const void* a;
  const void* b;
  i64 nout;                        // local outputs
  int nk, nr;                      // K runs; outer R runs (the rows' odometer)
  i64 ke[D_RUNS], ks[D_RUNS];      // extents and element strides, fastest first
  i64 re[D_RUNS], rs[D_RUNS];
  i64 nrows;                       // product of re (0: the reduced range is empty)
  i64 lu;                          // units per row (16-byte units when vec, else elements)
  int vec;
  int Wi, Wr, Oc;
  int S, Sr;                       // splits per tile (S = Sr * Si): Sr along rows, Si along units
  i64 rchunk, uchunk;              // rows / units per split
  i64 tiles;                       // output tiles (at least 1)
  int pred;
  alignas(16) unsigned char ref[16];
  unsigned* tickets;               // [tiles] when S > 1, then the all-tiles ticket
  unsigned char* part;             // [tiles][S][Oc] 16-byte partials
  GroupCombine cb;
  void* result;
};

// The last CTA's half of the combine (NT threads, every one calls it): signal every peer, wait for
// every peer, then res[o] = the group's partials of output o folded in rank order, read in place
// from each member's area.  Every member folds the same values in the same order.
template <class Rd, int NT>
__device__ __forceinline__ void group_combine(const GroupCombine& g, i64 nout, typename Rd::R* res) {
  using A = typename Rd::A;
  const int t = threadIdx.x, P = g.nranks, me = g.rank;
  if (t == 0) {
    for (int k = 1; k < P; ++k) flag_signal(g.remote_words[(me + k) % P], g.seq);
    for (int k = 1; k < P; ++k) {  // every peer, not only the group: see DESIGN §3l
      const int q = (me + P - k) % P;
      flag_wait(g.local_words + (size_t)q * g.word_stride, g.seq, g.timeout_ns, g.err);
    }
  }
  // the group's areas, in rank order, listed once per call (up to NT members in shared memory)
  __shared__ const unsigned char* grp[NT];
  __shared__ int ng;
  if (t == 0) {
    int n = 0;
    for (int q = 0; q < P; ++q)
      if (in_group(g, q)) {
        if (n < NT) grp[n] = g.areas[q] + g.area_off;
        ++n;
      }
    ng = n;
  }
  __syncthreads();
  if (ng > NT) {  // (a group of more than NT ranks: test membership per rank)
    for (i64 oo = t; oo < nout; oo += NT) {
      A v = Rd::neutral();
      for (int q = 0; q < P; ++q)
        if (in_group(g, q)) v = Rd::comb(v, ld16_cv<A>(g.areas[q] + g.area_off + (size_t)oo * 16));
      res[oo] = Rd::finish(v);
    }
    return;
  }
  // RU outputs per thread at once: their loads from one member are independent
  for (i64 o0 = t; o0 < nout; o0 += (i64)NT * RU) {
    A v[RU];
#pragma unroll
    for (int k = 0; k < RU; ++k) v[k] = Rd::neutral();
    for (int i = 0; i < ng; ++i) {
      A x[RU];
#pragma unroll
      for (int k = 0; k < RU; ++k)
        if (o0 + (i64)k * NT < nout) x[k] = ld16_cv<A>(grp[i] + (size_t)(o0 + (i64)k * NT) * 16);
#pragma unroll
      for (int k = 0; k < RU; ++k)
        if (o0 + (i64)k * NT < nout) v[k] = Rd::comb(v[k], x[k]);
    }
#pragma unroll
    for (int k = 0; k < RU; ++k)
      if (o0 + (i64)k * NT < nout) res[o0 + (i64)k * NT] = Rd::finish(v[k]);
  }
}

// tree over the W members of each team (sh[t] holds member t's value): member m takes m + h for
// h = W/2 .. 1; the team's value ends in member 0.  Every thread of the CTA calls it.
template <class Rd>
__device__ __forceinline__ typename Rd::A team_reduce(typename Rd::A v, typename Rd::A* sh,
                                                      const DArgs& g, int m, int oc) {
  const int W = g.Wi * g.Wr;
  auto tid = [&](int mm) { return ((mm / g.Wi) * g.Oc + oc) * g.Wi + mm % g.Wi; };
  __syncthreads();  // (sh may still be read from an earlier tree)
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int h = W / 2; h > 0; h >>= 1) {
    if (m < h) sh[threadIdx.x] = Rd::comb(sh[threadIdx.x], sh[tid(m + h)]);
    __syncthreads();
  }
  return sh[tid(0)];
}

template <class E, int M, int O>
__global__ void __launch_bounds__(RT, D_CTAS_PER_SM) k_reduce_dims(const DArgs g) {
  using Rd = Red<E, M, O>;
  using T = typename Rd::T;
  using A = typename Rd::A;
  constexpr int V = 16 / sizeof(E);
  __shared__ A sh[RT];
  __shared__ int last;
  const E* a = (const E*)g.a;
  const E* b = M == M_DOT ? (const E*)g.b : a;
  T ref;
  memcpy(&ref, g.ref, sizeof(T));
  const int t = threadIdx.x;
  const int wi = t % g.Wi, oc = (t / g.Wi) % g.Oc, wr = t / (g.Wi * g.Oc);
  const int m = wr * g.Wi + wi, W = g.Wi * g.Wr;
  const i64 tile = blockIdx.x / g.S;
  const int s = blockIdx.x % g.S;
  const i64 o = tile * g.Oc + oc;
  const int vx = g.vec ? V : 1;

  A acc = Rd::neutral();
  if (o < g.nout) {
    i64 koff = 0, q = o;
#pragma unroll
    for (int k = 0; k < D_RUNS; ++k)
      if (k < g.nk) {
        koff += (q % g.ke[k]) * g.ks[k];
        q /= g.ke[k];
      }
    const int sr = s % g.Sr, si = s / g.Sr;
    const i64 R0 = (i64)sr * g.rchunk, R1 = min(g.nrows, R0 + g.rchunk);
    const i64 nb = R1 > R0 ? (R1 - R0 + g.Wr - 1) / g.Wr : 0;
    i64 r = R0 + wr * nb;
    const i64 rend = min(R1, r + nb);
    const i64 U0 = (i64)si * g.uchunk, U1 = min(g.lu, U0 + g.uchunk);
    i64 u = U0 + wi;
    if (r < rend && u < U1) {
      i64 c[D_RUNS], roff = 0, rq = r;
#pragma unroll
      for (int k = 0; k < D_RUNS; ++k)
        if (k < g.nr) {
          c[k] = rq % g.re[k];
          roff += c[k] * g.rs[k];
          rq /= g.re[k];
        }
      const E* pa0 = a + koff;
      const E* pb0 = b + koff;
      bool more = true;
      while (more) {
        E xa[RU][V], xb[RU][V];
        i64 off[RU];
        int nin = 0;
#pragma unroll
        for (int k = 0; k < RU; ++k) {
          if (!more) break;
          off[k] = roff + u * vx;
          nin = k + 1;
          u += g.Wi;  // next item: the next unit of the row, else the next row (odometer)
          if (u >= U1) {
            u = U0 + wi;
            if (++r >= rend) {
              more = false;
            } else {
#pragma unroll
              for (int j = 0; j < D_RUNS; ++j)
                if (j < g.nr) {
                  roff += g.rs[j];
                  if (++c[j] < g.re[j]) break;
                  roff -= g.re[j] * g.rs[j];
                  c[j] = 0;
                }
            }
          }
        }
#pragma unroll
        for (int k = 0; k < RU; ++k)
          if (k < nin) {
            if (g.vec) {
              ld_unit(pa0 + off[k], true, xa[k]);
              if (M == M_DOT) ld_unit(pb0 + off[k], true, xb[k]);
            } else {
              xa[k][0] = ld1(pa0 + off[k]);
              if (M == M_DOT) xb[k][0] = ld1(pb0 + off[k]);
            }
          }
#pragma unroll
        for (int k = 0; k < RU; ++k)
          if (k < nin) {
#pragma unroll
            for (int j = 0; j < V; ++j)
              if (j < vx) acc = Rd::comb(acc, Rd::elem(xa[k][j], M == M_DOT ? xb[k][j] : xa[k][j], ref, g.pred));
          }
      }
    }
  }
  acc = team_reduce<Rd>(acc, sh, g, m, oc);

  if (g.S > 1) {  // the tile's last CTA folds its S partials (members take s = m, m + W, ...)
    unsigned char* part = g.part + (size_t)tile * g.S * g.Oc * 16;
    if (m == 0 && o < g.nout) {
      st16(part + ((size_t)s * g.Oc + oc) * 16, acc);
      __threadfence();
    }
    __syncthreads();
    if (t == 0) last = atomicAdd(g.tickets + tile, 1u) == (unsigned)g.S - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    acc = Rd::neutral();
    if (o < g.nout)
      for (int i = m; i < g.S; i += W) acc = Rd::comb(acc, ld16_cg<A>(part + ((size_t)i * g.Oc + oc) * 16));
    acc = team_reduce<Rd>(acc, sh, g, m, oc);
    if (t == 0) g.tickets[tile] = 0;  // the next call (ordered after this one) starts from zero
  }

  typename Rd::R* res = (typename Rd::R*)g.result;
  if (g.cb.nranks == 1) {
    if (m == 0 && o < g.nout) res[o] = Rd::finish(acc);
    return;
  }
  // P > 1: the tile's rank partials into my own area; the last tile runs the combine
  if (m == 0 && o < g.nout) {
    st16(g.cb.areas[g.cb.rank] + g.cb.area_off + (size_t)o * 16, acc);
    __threadfence_system();
  }
  __syncthreads();
  unsigned* all = g.tickets + (g.S > 1 ? g.tiles : 0);
  if (t == 0) last = atomicAdd(all, 1u) == (unsigned)(g.tiles - 1);
  __syncthreads();
  if (!last) return;
  __threadfence_system();
  if (t == 0) *all = 0;
  group_combine<Rd, RT>(g.cb, g.nout, res);
}

// the NCCL fallback's second kernel: fold the P gathered partials in rank order
template <class E, int M, int O>
__global__ void k_reduce_fold(const unsigned char* slots, int P, void* result) {
  using Rd = Red<E, M, O>;
  typename Rd::A acc = Rd::neutral();
  for (int q = 0; q < P; ++q) acc = Rd::comb(acc, ld16_cg<typename Rd::A>(slots + (size_t)q * 16));
  *(typename Rd::R*)result = Rd::finish(acc);
}

// ---- shell-binned spectra (pa_shell_spectrum, DESIGN §3m) ---------------------------------------
// E(b) = sum over the modes of bin b of w * f(x).  G CTAs of ST threads own contiguous chunks of
// 16-byte units (k_reduce's split: head, units, tail).  Each thread walks its elements with an
// odometer over the spatial memory dims (no index tensor): its first element's coordinates by
// division, then steps of ST * V elements added digit by digit.  Per step every lane of a warp has
// one (bin, contribution) pair: the lanes of equal bins (__match_any_sync) are summed in lane order
// by the lowest one, which adds the sum into the warp's histogram in shared memory (distinct bins
// per step: no atomics).  The SW warp histograms are folded in warp order into the CTA's partial;
// the last CTA (fence + ticket) folds the G partials in CTA order; with P > 1 the rank partial goes
// to this rank's partial area and group_combine folds every rank's in rank order.
constexpr int ST = 128;               // threads per CTA
constexpr int SW = ST / 32;           // warps per CTA: one histogram each
constexpr int S_CTAS_PER_SM = 4;      // grid cap per SM (512 threads); shared memory may allow fewer

struct SArgs {
  const void* a;
  const void* b;
  i64 head, tail, nunits, chunk;      // as RArgs
  int G;
  int vec_a, vec_b;
  int N;                              // spatial dims
  int ext[PA_MAX_DIMS];               // memory dim m: local extent,
  int lo[PA_MAX_DIMS];                //   global index of the first local element,
  int ng[PA_MAX_DIMS];                //   global extent,
  double s[PA_MAX_DIMS];              //   scale,
  int step[PA_MAX_DIMS];              //   digit of ST * V elements
  int lpos[PA_MAX_DIMS];              // logical dim l is memory dim lpos[l]
  int r2c;                            // memory dim of the r2c dim, -1: none
  i64 rfft_n;
  double width;
  int nbins;
  unsigned* ticket;
  double* part;                       // [G][nbins]
  GroupCombine cb;
  void* result;
};

// coordinates (memory order) of local element i
__device__ __forceinline__ void spec_coords(const SArgs& g, i64 i, int (&c)[PA_MAX_DIMS]) {
#pragma unroll
  for (int m = 0; m < PA_MAX_DIMS; ++m)
    if (m < g.N) {
      c[m] = (int)(i % g.ext[m]);
      i /= g.ext[m];
    }
}
// c += d (digits), the carry out of the last spatial dim dropped (extra dims do not bin)
__device__ __forceinline__ void spec_advance(const SArgs& g, int (&c)[PA_MAX_DIMS], const int* d) {
  int carry = 0;
#pragma unroll
  for (int m = 0; m < PA_MAX_DIMS; ++m)
    if (m < g.N) {
      c[m] += d[m] + carry;
      carry = c[m] >= g.ext[m];
      if (carry) c[m] -= g.ext[m];
    }
}
__device__ __forceinline__ void spec_inc(const SArgs& g, int (&c)[PA_MAX_DIMS]) {
#pragma unroll
  for (int m = 0; m < PA_MAX_DIMS; ++m)
    if (m < g.N) {
      if (++c[m] < g.ext[m]) return;
      c[m] = 0;
    }
}
// the bin of the mode at c (-1: dropped) and its weight
__device__ __forceinline__ int spec_mode(const SArgs& g, const int (&c)[PA_MAX_DIMS], int* w) {
  double k2[PA_MAX_DIMS];
  *w = 1;
#pragma unroll
  for (int m = 0; m < PA_MAX_DIMS; ++m)
    if (m < g.N) {
      const int i = g.lo[m] + c[m];
      const double k = spec_k(g.s[m], spec_wavenumber(i, g.ng[m], m == g.r2c));
      k2[m] = mul(k, k);
      if (m == g.r2c) *w = spec_weight(i, g.rfft_n);
    }
  double q = 0.0;  // in logical-dim order
#pragma unroll
  for (int l = 0; l < PA_MAX_DIMS; ++l)
    if (l < g.N) {
      double v = k2[0];
#pragma unroll
      for (int m = 1; m < PA_MAX_DIMS; ++m)
        if (m < g.N && g.lpos[l] == m) v = k2[m];
      q = add(q, v);
    }
  return spec_bin(q, g.width, g.nbins);
}

template <class E, int M>
__global__ void __launch_bounds__(ST, S_CTAS_PER_SM) k_spectrum(const SArgs g) {
  using Rd = Red<E, M, O_SUM>;
  using A = typename Rd::A;  // double
  constexpr int V = 16 / sizeof(E);
  extern __shared__ double hist[];  // [SW][nbins]
  __shared__ double sv[SW][32];
  __shared__ int last;
  const E* a = (const E*)g.a;
  const E* b = M == M_DOT ? (const E*)g.b : a;
  const int t = threadIdx.x, c = blockIdx.x, lane = t & 31, wp = t >> 5;
  const int nb = g.nbins;
  for (int i = t; i < SW * nb; i += ST) hist[i] = 0.0;
  __syncthreads();
  double* h = hist + (size_t)wp * nb;
  // one warp step: lane's (bin, contribution) into the warp's histogram
  auto put = [&](int bin, A v) {
    const unsigned grp = __match_any_sync(~0u, bin);
    sv[wp][lane] = v;
    __syncwarp();
    if (bin >= 0 && (grp & ((1u << lane) - 1)) == 0) {
      A sum = v;
      for (unsigned r = grp & (grp - 1); r; r &= r - 1) sum = add(sum, sv[wp][__ffs(r) - 1]);
      h[bin] = add(h[bin], sum);
    }
    __syncwarp();
  };
  auto contrib = [&](const E& x, const E& y, const int (&cc)[PA_MAX_DIMS], int* bin) {
    int w;
    *bin = spec_mode(g, cc, &w);
    const A v = Rd::elem(x, y, typename Rd::T(), 0);
    return w == 2 ? mul(2.0, v) : v;  // an exact doubling
  };

  int cc[PA_MAX_DIMS] = {0};
  if (c == 0 && t < 32) {  // head: warp 0, one element per lane
    int bin = -1;
    A v = 0.0;
    if (t < g.head) {
      spec_coords(g, t, cc);
      v = contrib(ld1(a + t), ld1(b + t), cc, &bin);
    }
    put(bin, v);
  }
  const E* ua = a + g.head;
  const E* ub = b + g.head;
  const i64 u0 = (i64)c * g.chunk, u1 = min(u0 + g.chunk, g.nunits);
  if (u0 + t < u1) spec_coords(g, g.head + (u0 + t) * V, cc);
  for (i64 ubase = u0; ubase < u1; ubase += (i64)ST * RU) {  // the same trip count in every warp
    E xa[RU][V], xb[RU][V];
#pragma unroll
    for (int k = 0; k < RU; ++k) {
      const i64 u = ubase + t + (i64)k * ST;
      if (u < u1) {
        ld_unit(ua + u * V, g.vec_a, xa[k]);
        if (M == M_DOT) ld_unit(ub + u * V, g.vec_b, xb[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < RU; ++k) {
      const bool in = ubase + t + (i64)k * ST < u1;
      int ce[PA_MAX_DIMS];
#pragma unroll
      for (int m = 0; m < PA_MAX_DIMS; ++m) ce[m] = cc[m];
#pragma unroll
      for (int j = 0; j < V; ++j) {
        int bin = -1;
        A v = 0.0;
        if (in) v = contrib(xa[k][j], M == M_DOT ? xb[k][j] : xa[k][j], ce, &bin);
        put(bin, v);
        if (j + 1 < V) spec_inc(g, ce);
      }
      if (in) spec_advance(g, cc, g.step);
    }
  }
  if (c == g.G - 1 && t < 32) {  // tail: warp 0 of the last CTA
    int bin = -1;
    A v = 0.0;
    if (t < g.tail) {
      const i64 i = g.head + g.nunits * V + t;
      spec_coords(g, i, cc);
      v = contrib(ld1(a + i), ld1(b + i), cc, &bin);
    }
    put(bin, v);
  }
  __syncthreads();

  // the CTA's partial (warps in order), then the last CTA folds the G partials in CTA order
  for (int i = t; i < nb; i += ST) {
    A v = hist[i];
#pragma unroll
    for (int w = 1; w < SW; ++w) v = add(v, hist[(size_t)w * nb + i]);
    g.part[(size_t)c * nb + i] = v;
  }
  __threadfence();
  __syncthreads();
  if (t == 0) last = atomicAdd(g.ticket, 1u) == (unsigned)g.G - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (t == 0) *g.ticket = 0;  // the next call (ordered after this one) starts from zero
  typename Rd::R* res = (typename Rd::R*)g.result;
  for (int i0 = t; i0 < nb; i0 += ST * RU) {  // RU bins per thread: independent loads
    A v[RU];
#pragma unroll
    for (int k = 0; k < RU; ++k)
      if (i0 + k * ST < nb) v[k] = __ldcg(g.part + i0 + k * ST);
    for (int q = 1; q < g.G; ++q) {
      A x[RU];
#pragma unroll
      for (int k = 0; k < RU; ++k)
        if (i0 + k * ST < nb) x[k] = __ldcg(g.part + (size_t)q * nb + i0 + k * ST);
#pragma unroll
      for (int k = 0; k < RU; ++k)
        if (i0 + k * ST < nb) v[k] = add(v[k], x[k]);
    }
#pragma unroll
    for (int k = 0; k < RU; ++k)
      if (i0 + k * ST < nb) {
        if (g.cb.nranks == 1) res[i0 + k * ST] = Rd::finish(v[k]);
        else st16(g.cb.areas[g.cb.rank] + g.cb.area_off + (size_t)(i0 + k * ST) * 16, v[k]);
      }
  }
  if (g.cb.nranks == 1) return;
  __threadfence_system();
  __syncthreads();
  group_combine<Rd, ST>(g.cb, nb, res);
}

// ---- spectra over chosen dims (pa_shell_spectrum_dims, DESIGN §3n) ------------------------------
// Every dim of the parent (memory order, extra dims last) is kept, binned or summed.  Output o
// (column-major over the kept dims' local extents) owns the slab of the other dims: nslab items j
// (column-major over the slab dims).  A CTA owns a tile of Kc consecutive outputs and a split of
// its slab (S splits of jchunk items); lane = kc + Kc * r takes output kc of the tile and items
// j = J0 + r + Rw * (warp + SW * step), Rw = 32 / Kc.  Kc = 1 unless the fastest memory dim is kept:
// then Kc consecutive kept indices are consecutive elements and the lanes' loads coalesce.  Each
// warp bins into its own histogram of Kc x nbins doubles with k_spectrum's match / lane-order step
// (key kc * nbins + bin; a key held by all 32 lanes is summed by a shuffle tree instead of the
// lane-order chain: a bin dim slow in memory keeps one bin over long runs of items), the warps are folded in warp order, the S splits of a tile in split order by
// the tile's last CTA (fence + ticket); with P > 1 every tile's rank partial goes to the partial
// area and the last tile (a second ticket) runs group_combine.
constexpr int SD_KC = 8;                         // most outputs per tile (8 x 16 bytes: a line)
constexpr size_t SD_SMEM = 48u << 10;            // warp histograms at Kc > 1: 4 CTAs per SM

struct SDArgs {
  const void* a;
  const void* b;
  int vec;                            // whole-element loads (the bases aligned to the element)
  int nd, N;                          // memory dims (extra dims included); spatial dims
  int kept[PA_MAX_DIMS];              // memory dim m: kept (1) or in the slab (0),
  int ext[PA_MAX_DIMS];               //   local extent,
  i64 str[PA_MAX_DIMS];               //   element stride,
  int sstep[PA_MAX_DIMS];             //   digit of Rw * SW slab items (0 for kept dims)
  int lo[PA_MAX_DIMS];                // spatial memory dim m: global index of the first local element,
  int ng[PA_MAX_DIMS];                //   global extent,
  double s[PA_MAX_DIMS];              //   scale
  int lpos[PA_MAX_DIMS];              // logical dim l is memory dim lpos[l]
  unsigned mask;                      // bin dims (logical)
  int r2c;                            // memory dim of the r2c dim, -1: none
  i64 rfft_n;
  double width;
  int nbins, Kc, Rw, S;
  i64 nout, nslab, jchunk, tiles;
  unsigned* tickets;                  // [tiles] when S > 1, then the all-tiles ticket
  double* part;                       // [tiles][S][Kc * nbins] when S > 1
  GroupCombine cb;
  void* result;
};

__device__ __forceinline__ c64 ld_elem(const c64* p, bool vec) {
  if (vec) {
    const double2 w = __ldcs((const double2*)p);
    return c64{w.x, w.y};
  }
  return ld1(p);
}
__device__ __forceinline__ c32 ld_elem(const c32* p, bool vec) {
  if (vec) {
    const float2 w = __ldcs((const float2*)p);
    return c32{w.x, w.y};
  }
  return ld1(p);
}

// c += the slab digits d (kept dims skipped), *off updated; the carry out of the last dim dropped
__device__ __forceinline__ void sd_advance(const SDArgs& g, int (&c)[PA_MAX_DIMS], i64* off) {
  int carry = 0;
#pragma unroll
  for (int m = 0; m < PA_MAX_DIMS; ++m)
    if (m < g.nd && !g.kept[m]) {
      const int d = g.sstep[m] + carry;
      c[m] += d;
      *off += (i64)d * g.str[m];
      carry = c[m] >= g.ext[m];
      if (carry) {
        c[m] -= g.ext[m];
        *off -= (i64)g.ext[m] * g.str[m];
      }
    }
}
// the bin of the mode at c (-1: dropped) and its weight; only the bin dims enter q
__device__ __forceinline__ int sd_mode(const SDArgs& g, const int (&c)[PA_MAX_DIMS], int* w) {
  double km[PA_MAX_DIMS], k[PA_MAX_DIMS];
  *w = 1;
#pragma unroll
  for (int m = 0; m < PA_MAX_DIMS; ++m)
    if (m < g.N) {
      const int i = g.lo[m] + c[m];
      km[m] = spec_k(g.s[m], spec_wavenumber(i, g.ng[m], m == g.r2c));
      if (m == g.r2c) *w = spec_weight(i, g.rfft_n);
    }
#pragma unroll
  for (int l = 0; l < PA_MAX_DIMS; ++l)
    if (l < g.N) {
      double v = km[0];
#pragma unroll
      for (int m = 1; m < PA_MAX_DIMS; ++m)
        if (m < g.N && g.lpos[l] == m) v = km[m];
      k[l] = v;
    } else {
      k[l] = 0.0;
    }
  return spec_bin(spec_q(g.N, k, g.mask), g.width, g.nbins);
}

template <class E, int M>
__global__ void __launch_bounds__(ST, S_CTAS_PER_SM) k_spectrum_dims(const SDArgs g) {
  using Rd = Red<E, M, O_SUM>;
  using A = typename Rd::A;  // double
  extern __shared__ double hist[];  // [SW][Kc * nbins]
  __shared__ double sv[SW][32];
  __shared__ int last;
  const E* a = (const E*)g.a;
  const E* b = M == M_DOT ? (const E*)g.b : a;
  const int t = threadIdx.x, lane = t & 31, wp = t >> 5;
  const int nb = g.nbins, KN = g.Kc * nb;
  const i64 tile = blockIdx.x / g.S;
  const int s = blockIdx.x % g.S;
  for (int i = t; i < SW * KN; i += ST) hist[i] = 0.0;
  __syncthreads();
  double* h = hist + (size_t)wp * KN;
  const int kc = lane % g.Kc, r = lane / g.Kc;
  const i64 o = tile * g.Kc + kc;
  const bool own = o < g.nout;

  // the lane's first item: kept coordinates from o, slab coordinates from j
  const i64 J0 = (i64)s * g.jchunk, J1 = min(g.nslab, J0 + g.jchunk);
  const i64 jstep = (i64)g.Rw * SW;
  int cc[PA_MAX_DIMS] = {0};
  i64 off = 0;
  if (own && g.nslab > 0) {  // (no extent is 0)
    i64 q = o, j = J0 + (i64)wp * g.Rw + r;
#pragma unroll
    for (int m = 0; m < PA_MAX_DIMS; ++m)
      if (m < g.nd) {
        const i64 e = g.ext[m];
        if (g.kept[m]) {
          cc[m] = (int)(q % e);
          q /= e;
        } else {
          cc[m] = (int)(j % e);
          j /= e;
        }
        off += (i64)cc[m] * g.str[m];
      }
  }
  auto put = [&](int key, A v) {
    const unsigned grp = __match_any_sync(~0u, key);
    if (grp == ~0u) {  // one key in the whole warp (a bin constant along the items): a shuffle tree
      if (key < 0) return;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) v = add(v, __shfl_down_sync(~0u, v, d));
      if (lane == 0) h[key] = add(h[key], v);
      __syncwarp();
      return;
    }
    sv[wp][lane] = v;
    __syncwarp();
    if (key >= 0 && (grp & ((1u << lane) - 1)) == 0) {
      A sum = v;
      for (unsigned rr = grp & (grp - 1); rr; rr &= rr - 1) sum = add(sum, sv[wp][__ffs(rr) - 1]);
      h[key] = add(h[key], sum);
    }
    __syncwarp();
  };

  int co[PA_MAX_DIMS];  // the load odometer runs RU steps ahead of the binning one
  i64 offl = off;
#pragma unroll
  for (int m = 0; m < PA_MAX_DIMS; ++m) co[m] = cc[m];
  for (i64 jb = J0 + (i64)wp * g.Rw; jb < J1; jb += jstep * RU) {  // uniform over the warp
    E xa[RU], xb[RU];
#pragma unroll
    for (int k = 0; k < RU; ++k)
      if (own && jb + r + k * jstep < J1) {
        xa[k] = ld_elem(a + offl, g.vec);
        if (M == M_DOT) xb[k] = ld_elem(b + offl, g.vec);
        sd_advance(g, co, &offl);
      }
#pragma unroll
    for (int k = 0; k < RU; ++k) {
      const bool in = own && jb + r + k * jstep < J1;
      int key = -1;
      A v = 0.0;
      if (in) {
        int w;
        const int bin = sd_mode(g, cc, &w);
        v = Rd::elem(xa[k], M == M_DOT ? xb[k] : xa[k], typename Rd::T(), 0);
        if (w == 2) v = mul(2.0, v);  // an exact doubling
        key = bin < 0 ? -1 : kc * nb + bin;
        sd_advance(g, cc, &off);
      }
      put(key, v);
    }
  }
  __syncthreads();

  // the CTA's partial (warps in order); with S > 1 the tile's last CTA folds the S partials in order
  typename Rd::R* res = (typename Rd::R*)g.result;
  const i64 nv = min((i64)KN, (g.nout - tile * g.Kc) * nb);  // the tile's values
  if (g.S > 1) {
    double* part = g.part + (size_t)tile * g.S * KN;
    for (int i = t; i < nv; i += ST) {
      A v = hist[i];
#pragma unroll
      for (int w = 1; w < SW; ++w) v = add(v, hist[(size_t)w * KN + i]);
      part[(size_t)s * KN + i] = v;
    }
    __threadfence();
    __syncthreads();
    if (t == 0) last = atomicAdd(g.tickets + tile, 1u) == (unsigned)g.S - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (t == 0) g.tickets[tile] = 0;  // the next call (ordered after this one) starts from zero
  }
  for (int i0 = t; i0 < nv; i0 += ST * RU) {  // RU values per thread: independent loads
    A v[RU];
#pragma unroll
    for (int k = 0; k < RU; ++k) {
      const int i = i0 + k * ST;
      if (i < nv) {
        if (g.S > 1) {
          const double* part = g.part + (size_t)tile * g.S * KN + i;
          v[k] = __ldcg(part);
          for (int q = 1; q < g.S; ++q) v[k] = add(v[k], __ldcg(part + (size_t)q * KN));
        } else {
          v[k] = hist[i];
#pragma unroll
          for (int w = 1; w < SW; ++w) v[k] = add(v[k], hist[(size_t)w * KN + i]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < RU; ++k) {
      const i64 i = tile * KN + i0 + k * ST;  // = b + nbins * o
      if (i0 + k * ST < nv) {
        if (g.cb.nranks == 1) res[i] = Rd::finish(v[k]);
        else st16(g.cb.areas[g.cb.rank] + g.cb.area_off + (size_t)i * 16, v[k]);
      }
    }
  }
  if (g.cb.nranks == 1) return;
  __threadfence_system();
  __syncthreads();
  unsigned* all = g.tickets + (g.S > 1 ? g.tiles : 0);
  if (t == 0) last = atomicAdd(all, 1u) == (unsigned)(g.tiles - 1);
  __syncthreads();
  if (!last) return;
  __threadfence_system();
  if (t == 0) *all = 0;
  group_combine<Rd, ST>(g.cb, g.nout * nb, res);
}

// ---- state: workspace, window tables and the event serialising the calls ----------------------
struct ReduceState {
  int device = 0, G_max = 1;
  unsigned* ticket = nullptr;
  unsigned char* part = nullptr;    // G_max partials
  unsigned char* gather = nullptr;  // [0]: the rank partial; [1 + r]: gathered partials (fallback)
  void** tables = nullptr;          // remote_words[nranks], peer_slots[nranks], areas[nranks]
  bool tables_ready = false;
  unsigned* dtickets = nullptr;     // pa_reduce_dims: G_max + 1 tickets and G_max * RT partials,
  unsigned char* dpart = nullptr;   //   made by the first such call (stream-ordered)
  unsigned* sticket = nullptr;      // pa_shell_spectrum: one ticket and G x nbins partials, made
  double* spart = nullptr;          //   and grown by the calls (stream-ordered); the partials are
  size_t spart_n = 0;               //   shared with pa_shell_spectrum_dims
  unsigned* sdtickets = nullptr;    // pa_shell_spectrum_dims: G_max + 1 tickets
  cudaEvent_t done = nullptr;       // the previous reduction's last kernel
  ull seq = 0;
  // held from the wait on `done` to its record: host threads calling at once cannot both order
  // their kernels after the same previous call and run them together on one workspace
  std::mutex mu;
};

void reduce_state_destroy(ReduceState* s) {
  if (!s) return;
  if (s->done) {
    cudaEventSynchronize(s->done);
    cudaEventDestroy(s->done);
  }
  cudaFree(s->ticket);
  cudaFree(s->part);
  cudaFree(s->gather);
  cudaFree(s->tables);
  cudaFree(s->dtickets);
  cudaFree(s->dpart);
  cudaFree(s->sticket);
  cudaFree(s->spart);
  cudaFree(s->sdtickets);
  cudaGetLastError();
  delete s;
}

// A communicator's state is made while the communicator is set up (comm_init*, synchronous
// like the rest of that setup) and its window tables are uploaded when the flag window is complete
// (reduce_state_set_tables), so no reduction on it touches the host's timeline.  The one-rank
// state of a device is made by its first reduction with stream-ordered allocations on the
// caller's stream, so that call does not synchronise the host either.
static pa_status make_state(int nranks, cudaStream_t stream, bool ordered, ReduceState** out) {
  std::unique_ptr<ReduceState> s(new ReduceState);
  CU(cudaGetDevice(&s->device));
  int sms = 0;
  CU(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device));
  s->G_max = R_CTAS_PER_SM * sms;
  auto alloc = [&](void** p, size_t bytes) {
    return ordered ? cudaMallocAsync(p, bytes, stream) : cudaMalloc(p, bytes);
  };
  CU(alloc((void**)&s->ticket, sizeof(unsigned)));
  CU(cudaMemsetAsync(s->ticket, 0, sizeof(unsigned), stream));
  CU(alloc((void**)&s->part, (size_t)s->G_max * 16));
  CU(alloc((void**)&s->gather, (size_t)(nranks + 1) * 16));
  if (nranks > 1) CU(alloc((void**)&s->tables, 3 * sizeof(void*) * (size_t)nranks));
  CU(cudaEventCreateWithFlags(&s->done, cudaEventDisableTiming));
  if (!ordered) CU(cudaStreamSynchronize(stream));
  *out = s.release();
  return PA_OK;
}

pa_status reduce_state_create(int nranks, ReduceState** out) {
  return make_state(nranks, nullptr, false, out);
}

pa_status reduce_state_set_tables(ReduceState* s, int nranks, unsigned long long* const* remote_words,
                                  unsigned char* const* peer_slots, unsigned char* const* areas) {
  std::vector<void*> tab(3 * (size_t)nranks);
  for (int r = 0; r < nranks; ++r) {
    tab[r] = remote_words[r];
    tab[nranks + r] = peer_slots[r];
    tab[2 * nranks + r] = areas[r];
  }
  CU(cudaMemcpy(s->tables, tab.data(), tab.size() * sizeof(void*), cudaMemcpyHostToDevice));
  s->tables_ready = true;
  return PA_OK;
}

// the state of one-rank reductions without a communicator: one per device
static std::mutex g_local_mu;
static std::map<int, ReduceState*> g_local_states;

// ---- dispatch over (element type, map, op) -----------------------------------------------------
struct Launch {
  RArgs g;
  cudaStream_t stream;
  const unsigned char* gathered;  // C_GATHER: the fold kernel's input (NULL: no fold)
  int nranks;
  const DArgs* d;                 // pa_reduce_dims (k_reduce_dims instead of k_reduce)
};

template <class E, int M, int O> static pa_status run(const Launch& L) {
  if (L.d)
    k_reduce_dims<E, M, O><<<(unsigned)(L.d->tiles * L.d->S), RT, 0, L.stream>>>(*L.d);
  else
    k_reduce<E, M, O><<<L.g.G, RT, 0, L.stream>>>(L.g);
  count_launch();
  CU(cudaGetLastError());
  return PA_OK;
}
template <class E, int M, int O> static pa_status run_fold(const Launch& L) {
  k_reduce_fold<E, M, O><<<1, 1, 0, L.stream>>>(L.gathered, L.nranks, L.g.result);
  count_launch();
  CU(cudaGetLastError());
  return PA_OK;
}

template <class E, int M> static pa_status by_op(int op, bool fold, const Launch& L) {
  switch (op & 15) {
    case O_SUM: return fold ? run_fold<E, M, O_SUM>(L) : run<E, M, O_SUM>(L);
    case O_ANY: return fold ? run_fold<E, M, O_ANY>(L) : run<E, M, O_ANY>(L);
    case O_ALL: return fold ? run_fold<E, M, O_ALL>(L) : run<E, M, O_ALL>(L);
  }
  if constexpr (Ordered<typename Mapped<E, M>::T>::value) {
    if ((op & 15) == O_MAX) return fold ? run_fold<E, M, O_MAX>(L) : run<E, M, O_MAX>(L);
    if ((op & 15) == O_MIN) return fold ? run_fold<E, M, O_MIN>(L) : run<E, M, O_MIN>(L);
  }
  set_error("reduction: op %d not instantiated", op);
  return PA_EINVAL;
}
template <class E> static pa_status by_map(int map, int op, bool fold, const Launch& L) {
  switch (map) {
    case M_ID: return by_op<E, M_ID>(op, fold, L);
    case M_ABS: return by_op<E, M_ABS>(op, fold, L);
    case M_ABS2: return by_op<E, M_ABS2>(op, fold, L);
    case M_DOT: return by_op<E, M_DOT>(op, fold, L);
  }
  set_error("reduction: map %d not instantiated", map);
  return PA_EINVAL;
}
static pa_status dispatch(int dtype, int map, int op, bool fold, const Launch& L) {
  switch (dtype) {
    case D_F64: return by_map<double>(map, op, fold, L);
    case D_F32: return by_map<float>(map, op, fold, L);
    case D_C64: return by_map<c64>(map, op, fold, L);
    case D_C32: return by_map<c32>(map, op, fold, L);
    case D_I32: return by_map<int32_t>(map, op, fold, L);
    case D_I64: return by_map<long long>(map, op, fold, L);
  }
  set_error("reduction: dtype %d not instantiated", dtype);
  return PA_EINVAL;
}

static int dtype_size(int dtype) {
  switch (dtype) {
    case D_F64: case D_C32: case D_I64: return 8;
    case D_F32: case D_I32: return 4;
    case D_C64: return 16;
  }
  return 0;
}

// the state serving a call: the communicator's, or the device's one-rank state (made here)
static pa_status state_of(Comm* comm, const ReduceWindow& w, void* stream, ReduceState** out) {
  if (comm) {
    *out = *w.state;  // made with the communicator
    return PA_OK;
  }
  int dev = 0;
  CU(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(g_local_mu);
  ReduceState*& s0 = g_local_states[dev];
  if (!s0) RC(make_state(1, (cudaStream_t)stream, true, &s0));
  *out = s0;
  return PA_OK;
}

static void set_pred(RArgs* g, int dtype, int map, int op, const void* pred_value, int es) {
  g->pred = op >> 4;
  if (pred_value) {
    int vs = (map == M_ID) ? es : (dtype == D_C64 ? 8 : dtype == D_C32 ? 4 : es);  // the mapped value
    memcpy(g->ref, pred_value, (size_t)vs);
  }
}

pa_status reduce(Comm* comm, int dtype, int map, int op, const void* pred_value, i64 n,
                 const void* a, const void* b, void* result, void* stream) {
  ReduceWindow w;
  if (comm) {
    pa_status s = comm_reduce_window(comm, &w);
    if (s != PA_OK) return s;
  }
  const int P = w.nranks;
  if (P > 1 && !w.flags && !w.nccl) {
    set_error("reduction: the communicator has neither a flag window nor NCCL");
    return PA_ESTATE;
  }
  ReduceState* st = nullptr;
  RC(state_of(comm, w, stream, &st));
  std::lock_guard<std::mutex> serial(st->mu);
  const bool flags = P > 1 && w.flags;
  if (flags && !st->tables_ready) {
    set_error("reduction: the flag window's tables were not uploaded (pa_comm_flags_import)");
    return PA_ESTATE;
  }

  Launch L;
  memset(&L, 0, sizeof L);
  RArgs& g = L.g;
  const int es = dtype_size(dtype);
  const int V = 16 / es;
  // 16-byte units: from the first 16-byte boundary of `a` that is a whole number of elements in
  const uintptr_t pa_ = (uintptr_t)a, pb = (uintptr_t)b;
  const i64 head_bytes = (i64)((16 - (pa_ & 15)) & 15);
  const bool vec = n > 0 && head_bytes % es == 0;
  g.head = vec ? std::min<i64>(head_bytes / es, n) : 0;
  g.nunits = (n - g.head) / V;
  g.tail = n - g.head - g.nunits * V;
  g.vec_a = vec;
  g.vec_b = vec && map == M_DOT && ((pb - pa_) & 15) == 0;
  // the CTA count depends on n and the device only; the split into head, units and tail (and so
  // the summation order) also on the base address modulo 16
  const i64 want = (n + (i64)V * RT * RU - 1) / ((i64)V * RT * RU);
  g.G = (int)std::max<i64>(1, std::min<i64>(want, st->G_max));
  g.chunk = (g.nunits + g.G - 1) / g.G;
  g.a = a;
  g.b = map == M_DOT ? b : a;
  set_pred(&g, dtype, map, op, pred_value, es);
  g.ticket = st->ticket;
  g.part = st->part;
  g.result = result;
  g.nranks = P;
  g.rank = w.rank;
  g.mode = P == 1 ? C_LOCAL : flags ? C_FLAGS : C_GATHER;
  if (flags) {
    g.seq = ++st->seq;
    g.local_words = w.local_words;
    g.word_stride = w.word_stride;
    g.remote_words = (ull* const*)st->tables;
    g.peer_slots = (unsigned char* const*)(st->tables + P);
    g.local_slots = w.local_slots;
    g.timeout_ns = w.timeout_ns;
    g.err = w.err;
  }
  g.partial_out = st->gather;
  L.stream = (cudaStream_t)stream;
  L.gathered = st->gather + 16;
  L.nranks = P;

  CU(cudaStreamWaitEvent(L.stream, st->done, 0));
  pa_status s = dispatch(dtype, map, op, false, L);
  if (s != PA_OK) return s;
  if (g.mode == C_GATHER) {
    s = comm_allgather(comm, st->gather, st->gather + 16, 16, stream);
    if (s != PA_OK) return s;
    s = dispatch(dtype, map, op, true, L);
    if (s != PA_OK) return s;
  }
  CU(cudaEventRecord(st->done, L.stream));
  return PA_OK;
}

// the combine's arguments for a call on a communicator with a flag window; the group is every rank
// until the caller narrows it (keep_grid)
static void combine_args(const ReduceWindow& w, ReduceState* st, GroupCombine* cb) {
  const int P = w.nranks;
  cb->nranks = P;
  cb->rank = w.rank;
  cb->seq = ++st->seq;  // one sequence with pa_reduce: the parity sets alternate across all calls
  cb->local_words = w.local_words;
  cb->word_stride = w.word_stride;
  cb->remote_words = (ull* const*)st->tables;
  cb->areas = (unsigned char* const*)(st->tables + 2 * P);
  cb->area_off = (size_t)(cb->seq & 1) * REDUCE_AREA_BYTES;
  cb->timeout_ns = w.timeout_ns;
  cb->err = w.err;
}

static i64 pow2_ceil(i64 x) {
  i64 p = 1;
  while (p < x) p <<= 1;
  return p;
}

pa_status reduce_dims(Comm* comm, int dtype, int map, int op, const void* pred_value,
                      const DimsGeom& geo, const void* a, const void* b, void* result, void* stream) {
  ReduceWindow w;
  if (comm) RC(comm_reduce_window(comm, &w));
  const int P = w.nranks;
  if (P > 1 && !w.flags) {
    set_error("pa_reduce_dims: the combine runs through the communicator's flag window, and this "
              "communicator has none (NCCL without the window, or the nccl_fences tunable)");
    return PA_ESTATE;
  }
  ReduceState* st = nullptr;
  RC(state_of(comm, w, stream, &st));
  std::lock_guard<std::mutex> serial(st->mu);
  if (P > 1 && !st->tables_ready) {
    set_error("reduction: the flag window's tables were not uploaded (pa_comm_flags_import)");
    return PA_ESTATE;
  }
  const cudaStream_t cs = (cudaStream_t)stream;
  if (!st->dtickets) {  // stream-ordered: the first call does not synchronise the host either
    CU(cudaMallocAsync((void**)&st->dtickets, (size_t)(st->G_max + 1) * sizeof(unsigned), cs));
    CU(cudaMemsetAsync(st->dtickets, 0, (size_t)(st->G_max + 1) * sizeof(unsigned), cs));
    CU(cudaMallocAsync((void**)&st->dpart, (size_t)st->G_max * RT * 16, cs));
  }

  DArgs d;
  memset(&d, 0, sizeof d);
  const int es = dtype_size(dtype), V = 16 / es;
  // runs: extent-1 dims dropped, neighbours of the same class merged
  bool rred[PA_MAX_DIMS];
  i64 rext[PA_MAX_DIMS], rstr[PA_MAX_DIMS], stride = 1, nred = 1;
  int nruns = 0;
  d.nout = 1;
  for (int i = 0; i < geo.nd; ++i) {
    (geo.red[i] ? nred : d.nout) *= geo.ext[i];
    if (geo.ext[i] != 1) {
      if (nruns > 0 && rred[nruns - 1] == geo.red[i]) {
        rext[nruns - 1] *= geo.ext[i];
      } else {
        rred[nruns] = geo.red[i];
        rext[nruns] = geo.ext[i];
        rstr[nruns++] = stride;
      }
    }
    stride *= geo.ext[i];
  }
  // the row regime: the fastest run is reduced and at least 64 bytes long
  const bool row = nruns > 0 && rred[0] && rext[0] * es >= 64;
  const i64 L = row ? rext[0] : 1;
  for (int i = row ? 1 : 0; i < nruns; ++i) {
    if (rred[i]) {
      d.re[d.nr] = rext[i];
      d.rs[d.nr++] = rstr[i];
    } else {
      d.ke[d.nk] = rext[i];
      d.ks[d.nk++] = rstr[i];
    }
  }
  d.nrows = nred / L;
  d.vec = row && (uintptr_t)a % 16 == 0 && (map != M_DOT || (uintptr_t)b % 16 == 0) &&
          (L * es) % 16 == 0;
  d.lu = d.vec ? L / V : L;
  // teams: along the row's units first, then fewer outputs per CTA when there are few outputs
  int Wi = row ? (int)std::min<i64>(32, pow2_ceil(d.lu)) : 1, Wr = 1, Oc = RT / Wi;
  while (Oc > 1 && Oc / 2 >= d.nout) {
    Oc /= 2;
    if (row && d.nrows < 2 * (i64)Wr && d.lu > Wi) Wi *= 2;
    else Wr *= 2;
  }
  d.Wi = Wi;
  d.Wr = Wr;
  d.Oc = Oc;
  d.tiles = std::max<i64>(1, (d.nout + Oc - 1) / Oc);
  // splits: only when the tiles leave SMs idle and each member keeps >= 64 items; depends on the
  // geometry and the device only
  i64 S = 1;
  if (d.nout > 0 && d.tiles < st->G_max)
    S = std::max<i64>(1, std::min<i64>(st->G_max / d.tiles, d.nrows * d.lu / ((i64)Wi * Wr * 64)));
  const i64 Sr = std::min<i64>(S, std::max<i64>(1, d.nrows / Wr));
  const i64 Si = std::max<i64>(1, std::min<i64>(S / Sr, d.lu / Wi));
  d.Sr = (int)Sr;
  d.S = (int)(Sr * Si);
  d.rchunk = std::max<i64>(1, (d.nrows + Sr - 1) / Sr);
  d.uchunk = std::max<i64>(1, (d.lu + Si - 1) / Si);
  d.a = a;
  d.b = map == M_DOT ? b : a;
  RArgs pr;
  memset(&pr, 0, sizeof pr);
  set_pred(&pr, dtype, map, op, pred_value, es);
  d.pred = pr.pred;
  memcpy(d.ref, pr.ref, 16);
  d.tickets = st->dtickets;
  d.part = st->dpart;
  d.result = result;
  if (P > 1) {
    combine_args(w, st, &d.cb);
    d.cb.topo_M = geo.topo_M;
    for (int i = 0; i < geo.topo_M; ++i) {
      d.cb.topo_dims[i] = (int)geo.topo_dims[i];
      d.cb.coords[i] = (int)geo.coords[i];
    }
    d.cb.keep_grid = geo.keep_grid;
  }
  d.cb.nranks = P;
  d.cb.rank = w.rank;

  Launch Ln;
  memset(&Ln, 0, sizeof Ln);
  Ln.stream = cs;
  Ln.d = &d;
  CU(cudaStreamWaitEvent(cs, st->done, 0));
  RC(dispatch(dtype, map, op, false, Ln));
  CU(cudaEventRecord(st->done, cs));
  return PA_OK;
}

// ---- pa_shell_spectrum ---------------------------------------------------------------------------
// the spectra's partials hold at least `need` doubles (stream-ordered: after the previous
// reduction on this state, which may still read them)
static pa_status grow_spart(ReduceState* st, size_t need, cudaStream_t cs) {
  if (st->spart_n >= need) return PA_OK;
  if (st->spart) CU(cudaFreeAsync(st->spart, cs));
  st->spart = nullptr;
  st->spart_n = 0;
  CU(cudaMallocAsync((void**)&st->spart, need * sizeof(double), cs));
  st->spart_n = need;
  return PA_OK;
}

template <class E, int M> static pa_status run_spectrum(const SArgs& g, size_t smem, cudaStream_t s) {
  CU(cudaFuncSetAttribute(k_spectrum<E, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_spectrum<E, M><<<g.G, ST, smem, s>>>(g);
  count_launch();
  CU(cudaGetLastError());
  return PA_OK;
}
template <class E, int M> static pa_status spectrum_occupancy(size_t smem, int* occ) {
  CU(cudaFuncSetAttribute(k_spectrum<E, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, k_spectrum<E, M>, ST, smem));
  return PA_OK;
}

pa_status shell_spectrum(Comm* comm, int dtype, int map, const SpecGeom& sg, const void* a,
                         const void* b, void* result, void* stream) {
  ReduceWindow w;
  if (comm) RC(comm_reduce_window(comm, &w));
  const int P = w.nranks;
  if (P > 1 && !w.flags) {
    set_error("pa_shell_spectrum: the combine runs through the communicator's flag window, and this "
              "communicator has none (NCCL without the window, or the nccl_fences tunable)");
    return PA_ESTATE;
  }
  ReduceState* st = nullptr;
  RC(state_of(comm, w, stream, &st));
  std::lock_guard<std::mutex> serial(st->mu);
  if (P > 1 && !st->tables_ready) {
    set_error("reduction: the flag window's tables were not uploaded (pa_comm_flags_import)");
    return PA_ESTATE;
  }
  const cudaStream_t cs = (cudaStream_t)stream;
  const bool wide = dtype == D_C64, dot = map == M_DOT;
  const size_t smem = (size_t)SW * sg.nbins * sizeof(double);
  int occ = 0;
  RC(wide ? (dot ? spectrum_occupancy<c64, M_DOT>(smem, &occ) : spectrum_occupancy<c64, M_ABS2>(smem, &occ))
         : (dot ? spectrum_occupancy<c32, M_DOT>(smem, &occ) : spectrum_occupancy<c32, M_ABS2>(smem, &occ)));

  SArgs g;
  memset(&g, 0, sizeof g);
  const int es = wide ? 16 : 8, V = 16 / es;
  const i64 n = sg.n;
  // k_reduce's split into head, 16-byte units and tail
  const uintptr_t pa_ = (uintptr_t)a, pb = (uintptr_t)b;
  const i64 head_bytes = (i64)((16 - (pa_ & 15)) & 15);
  const bool vec = n > 0 && head_bytes % es == 0;
  g.head = vec ? std::min<i64>(head_bytes / es, n) : 0;
  g.nunits = (n - g.head) / V;
  g.tail = n - g.head - g.nunits * V;
  g.vec_a = vec;
  g.vec_b = vec && dot && ((pb - pa_) & 15) == 0;
  // the CTA count depends on n, nbins and the device only
  const int sms = st->G_max / R_CTAS_PER_SM;
  const i64 want = (n + (i64)V * ST * RU - 1) / ((i64)V * ST * RU);
  g.G = (int)std::max<i64>(1, std::min<i64>(want, (i64)sms * std::max(1, std::min(occ, S_CTAS_PER_SM))));
  g.chunk = (g.nunits + g.G - 1) / g.G;
  g.a = a;
  g.b = dot ? b : a;
  g.N = sg.N;
  i64 delta = (i64)ST * V;
  for (int m = 0; m < sg.N; ++m) {
    g.ext[m] = (int)sg.ext[m];
    g.lo[m] = (int)sg.lo[m];
    g.ng[m] = (int)sg.ng[m];
    g.s[m] = sg.s[m];
    g.lpos[m] = sg.lpos[m];
    if (n > 0) {
      g.step[m] = (int)(delta % sg.ext[m]);
      delta /= sg.ext[m];
    }
  }
  g.r2c = sg.r2c;
  g.rfft_n = sg.rfft_n;
  g.width = sg.width;
  g.nbins = sg.nbins;
  g.result = result;
  if (P > 1) combine_args(w, st, &g.cb);
  g.cb.nranks = P;
  g.cb.rank = w.rank;

  CU(cudaStreamWaitEvent(cs, st->done, 0));
  // workspace, stream-ordered (after the previous reduction on this state, which may still use it)
  if (!st->sticket) {
    CU(cudaMallocAsync((void**)&st->sticket, sizeof(unsigned), cs));
    CU(cudaMemsetAsync(st->sticket, 0, sizeof(unsigned), cs));
  }
  RC(grow_spart(st, (size_t)g.G * sg.nbins, cs));
  g.ticket = st->sticket;
  g.part = st->spart;
  RC(wide ? (dot ? run_spectrum<c64, M_DOT>(g, smem, cs) : run_spectrum<c64, M_ABS2>(g, smem, cs))
         : (dot ? run_spectrum<c32, M_DOT>(g, smem, cs) : run_spectrum<c32, M_ABS2>(g, smem, cs)));
  CU(cudaEventRecord(st->done, cs));
  return PA_OK;
}

// ---- pa_shell_spectrum_dims ------------------------------------------------------------------------
template <class E, int M> static pa_status run_spectrum_dims(const SDArgs& g, size_t smem, cudaStream_t s) {
  CU(cudaFuncSetAttribute(k_spectrum_dims<E, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_spectrum_dims<E, M><<<(unsigned)(g.tiles * g.S), ST, smem, s>>>(g);
  count_launch();
  CU(cudaGetLastError());
  return PA_OK;
}
template <class E, int M> static pa_status spectrum_dims_occupancy(size_t smem, int* occ) {
  CU(cudaFuncSetAttribute(k_spectrum_dims<E, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, k_spectrum_dims<E, M>, ST, smem));
  return PA_OK;
}

pa_status shell_spectrum_dims(Comm* comm, int dtype, int map, const SpecDimsGeom& geo,
                              const void* a, const void* b, void* result, void* stream) {
  const SpecGeom& sg = geo.sp;
  const DimsGeom& dg = geo.dg;
  ReduceWindow w;
  if (comm) RC(comm_reduce_window(comm, &w));
  const int P = w.nranks;
  if (P > 1 && !w.flags) {
    set_error("pa_shell_spectrum_dims: the combine runs through the communicator's flag window, and "
              "this communicator has none (NCCL without the window, or the nccl_fences tunable)");
    return PA_ESTATE;
  }
  ReduceState* st = nullptr;
  RC(state_of(comm, w, stream, &st));
  std::lock_guard<std::mutex> serial(st->mu);
  if (P > 1 && !st->tables_ready) {
    set_error("reduction: the flag window's tables were not uploaded (pa_comm_flags_import)");
    return PA_ESTATE;
  }
  const cudaStream_t cs = (cudaStream_t)stream;
  const bool wide = dtype == D_C64, dot = map == M_DOT;
  const int es = wide ? 16 : 8;

  SDArgs g;
  memset(&g, 0, sizeof g);
  g.nd = dg.nd;
  g.N = sg.N;
  g.nout = geo.nout;
  g.nslab = 1;
  i64 stride = 1;
  int fastest = -1;  // the fastest memory dim of extent > 1
  for (int m = 0; m < dg.nd; ++m) {
    g.kept[m] = !dg.red[m];
    g.ext[m] = (int)dg.ext[m];
    g.str[m] = stride;
    stride *= dg.ext[m];
    if (dg.red[m]) g.nslab *= dg.ext[m];
    if (fastest < 0 && dg.ext[m] > 1) fastest = m;
  }
  for (int m = 0; m < sg.N; ++m) {
    g.lo[m] = (int)sg.lo[m];
    g.ng[m] = (int)sg.ng[m];
    g.s[m] = sg.s[m];
    g.lpos[m] = sg.lpos[m];
  }
  g.mask = geo.bin_mask;
  g.r2c = sg.r2c;
  g.rfft_n = sg.rfft_n;
  g.width = sg.width;
  g.nbins = sg.nbins;
  // tiles of Kc outputs: Kc > 1 only when the fastest memory dim is kept (the lanes' loads are then
  // consecutive elements), as long as the warp histograms fit SD_SMEM
  int Kc = 1;
  if (fastest >= 0 && g.kept[fastest]) {
    Kc = SD_KC;
    while (Kc > 1 && (Kc / 2 >= dg.ext[fastest] || (size_t)SW * Kc * sg.nbins * 8 > SD_SMEM)) Kc /= 2;
  }
  g.Kc = Kc;
  g.Rw = 32 / Kc;
  const size_t smem = (size_t)SW * Kc * sg.nbins * sizeof(double);
  int occ = 0;
  RC(wide ? (dot ? spectrum_dims_occupancy<c64, M_DOT>(smem, &occ) : spectrum_dims_occupancy<c64, M_ABS2>(smem, &occ))
         : (dot ? spectrum_dims_occupancy<c32, M_DOT>(smem, &occ) : spectrum_dims_occupancy<c32, M_ABS2>(smem, &occ)));
  g.tiles = std::max<i64>(1, (g.nout + Kc - 1) / Kc);
  // splits of the slab: only when the tiles leave resident CTAs idle and each split keeps at least
  // RU steps per warp; depends on the geometry, nbins and the device only
  const int sms = st->G_max / R_CTAS_PER_SM;
  const i64 G = (i64)sms * std::max(1, std::min(occ, S_CTAS_PER_SM));
  i64 S = 1;
  if (g.nout > 0 && g.tiles < G)
    S = std::max<i64>(1, std::min<i64>(G / g.tiles, g.nslab / ((i64)g.Rw * SW * RU)));
  g.jchunk = std::max<i64>(1, (g.nslab + S - 1) / S);
  g.S = (int)S;
  i64 delta = (i64)g.Rw * SW;
  for (int m = 0; m < dg.nd; ++m)
    if (dg.red[m] && g.nslab > 0) {
      g.sstep[m] = (int)(delta % dg.ext[m]);
      delta /= dg.ext[m];
    }
  const uintptr_t pa_ = (uintptr_t)a, pb = (uintptr_t)b;
  g.vec = (pa_ % es == 0) && (!dot || pb % es == 0);
  g.a = a;
  g.b = dot ? b : a;
  g.result = result;
  if (P > 1) {
    combine_args(w, st, &g.cb);
    g.cb.topo_M = dg.topo_M;
    for (int i = 0; i < dg.topo_M; ++i) {
      g.cb.topo_dims[i] = (int)dg.topo_dims[i];
      g.cb.coords[i] = (int)dg.coords[i];
    }
    g.cb.keep_grid = dg.keep_grid;
  }
  g.cb.nranks = P;
  g.cb.rank = w.rank;

  CU(cudaStreamWaitEvent(cs, st->done, 0));
  if (!st->sdtickets) {  // (S > 1 only with fewer tiles than G <= G_max)
    CU(cudaMallocAsync((void**)&st->sdtickets, (size_t)(st->G_max + 1) * sizeof(unsigned), cs));
    CU(cudaMemsetAsync(st->sdtickets, 0, (size_t)(st->G_max + 1) * sizeof(unsigned), cs));
  }
  if (S > 1) RC(grow_spart(st, (size_t)g.tiles * S * Kc * sg.nbins, cs));
  g.tickets = st->sdtickets;
  g.part = st->spart;
  RC(wide ? (dot ? run_spectrum_dims<c64, M_DOT>(g, smem, cs) : run_spectrum_dims<c64, M_ABS2>(g, smem, cs))
         : (dot ? run_spectrum_dims<c32, M_DOT>(g, smem, cs) : run_spectrum_dims<c32, M_ABS2>(g, smem, cs)));
  CU(cudaEventRecord(st->done, cs));
  return PA_OK;
}

}  // namespace pa
