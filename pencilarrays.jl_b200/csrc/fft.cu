// Fused unpack + batched 1-d FFT (SURVEY.md §8(f2)).
//
// In a PencilFFTs-style transform every transposition is followed by a 1-d FFT
// along the dimension that has just become local and -- thanks to the pencil's
// permutation -- contiguous (reference docs/src/Pencils.md:210-214;
// docs/src/Transpositions.md:7-9).  Unfused that is two HBM round trips: the
// unpack (copy_permuted!, Transpositions.jl:585-664) writes the permuted array,
// the FFT reads and rewrites it.  This kernel does both in one:
//
//   * a CTA owns C = 8 consecutive destination LINES (same outer coordinates,
//     8 consecutive values of the source-contiguous dim; 4 for 1024-point lines);
//   * it gathers them from EVERY block of the transposition -- the blocks the
//     peers sent (dense in recv_buf, wire layout of :380-416) and the self block
//     straight out of `src` -- with 128-byte (8 x ComplexF64) coalesced loads,
//     writing them transposed into shared memory (padded: fft_core.hpp);
//   * runs the mixed-radix (2/4/8) decimation-in-frequency passes in shared memory,
//     butterflies in registers; for 1024-point lines the first pass (radix 16) runs on
//     the values as they arrive from HBM -- a thread's loads are exactly one
//     butterfly's inputs -- before they ever touch shared memory;
//   * stores each transformed line with fully contiguous 128-bit stores.
//
// HBM traffic: 2 * s * n bytes for n elements, the same as the plain unpack.
// ComplexF64 lines of 8 ... 1024 points (power of two); anything else is refused
// (PA_EINVAL) and the caller transposes and transforms separately.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <mutex>
#include <vector>

// twiddles: one table lookup per butterfly, the other powers by squaring / products (the
// lookups share the load/store path with shared memory, the kernel's limiter)
#ifndef PA_FFT_TWIDDLE_LOOKUPS
#define PA_FFT_TWIDDLE_LOOKUPS 1
#endif
#include "fft_core.hpp"
#include "pa_internal.hpp"

namespace pa {

using pa_fft::cplx;

constexpr int FFT_MAXB = 8;   // blocks gathered by one launch (ranks of a grid line on one box)
constexpr int FFT_MAXO = PA_MAX_DIMS - 2;
constexpr int FFT_THREADS = 256;
// lines per CTA: 8 (128-byte gathers); 4 for 1024-point lines so that three CTAs still
// share an SM's shared memory (75 KB each)
constexpr int fft_lines(int logL) { return logL >= 10 ? 4 : 8; }

struct FftBlock {
  const char* src;  // block origin
  int y0, ey;       // destination line range [y0, y0 + ey) this block fills
  long long ssy;    // source byte stride of the line dim
  long long ssx;    // source byte stride between consecutive columns (= lines)
  long long so[FFT_MAXO];
};
struct FftParams {
  int nb;
  FftBlock blk[FFT_MAXB];
  char* dst;
  long long ex;   // columns (source-contiguous dim)
  long long dsx;  // destination byte stride of a column step (= one line)
  int no;
  long long oe[FFT_MAXO], dso[FFT_MAXO];
  int L, logL, sign, pitch;
  int linear;  // the lines are contiguous in the source too (no transposition): consecutive
               // threads then walk along a line instead of across the columns
  const cplx* tw;
  unsigned tiles_x;
};

struct SmLine {
  cplx* p;
  __device__ __forceinline__ cplx get(int i) const { return p[pa_fft::pad_index(i)]; }
  __device__ __forceinline__ void put(int i, cplx v) { p[pa_fft::pad_index(i)] = v; }
};

// radix of the pass that starts at sub-length 2^LOGM (the odd bits go first: radices_of)
template <int LOGM>
struct PassRadix {
  static constexpr int LOGR = (LOGM % 3 == 0) ? 3 : (LOGM % 3);
};

template <int LOGL, int LOGM, int C, class Tw>
__device__ __forceinline__ void fft_passes(cplx* sm, int pitch, int ncol, int sign, const Tw& tw) {
  if constexpr (LOGM > 0) {
    constexpr int LOGR = PassRadix<LOGM>::LOGR;
    constexpr int R = 1 << LOGR, L = 1 << LOGL, M = 1 << LOGM;
    constexpr int PER_LINE = L / R;
    constexpr int TOTAL = C * PER_LINE;
#pragma unroll
    for (int w0 = 0; w0 < TOTAL; w0 += FFT_THREADS) {
      const int w = w0 + (int)threadIdx.x;
      const int c = w / PER_LINE, u = w % PER_LINE;
      if (w < TOTAL && c < ncol) {
        SmLine x{sm + c * pitch};
        pa_fft::butterfly<R>(x, u, L, M, sign, tw);
      }
    }
    __syncthreads();
    fft_passes<LOGL, LOGM - LOGR, C>(sm, pitch, ncol, sign, tw);
  }
}

// storage position of output frequency k (fft_position_of with compile-time radices)
template <int LOGL, int LOGM>
__device__ __forceinline__ int fft_pos(int k) {
  if constexpr (LOGM == 0) {
    return 0;
  } else {
    constexpr int LOGR = PassRadix<LOGM>::LOGR;
    return ((k & ((1 << LOGR) - 1)) << (LOGM - LOGR)) + fft_pos<LOGL, LOGM - LOGR>(k >> LOGR);
  }
}

template <int LOGL, int C>
__global__ void __launch_bounds__(FFT_THREADS) k_unpack_fft(const __grid_constant__ FftParams p) {
  constexpr int L = 1 << LOGL;
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cplx* sm = reinterpret_cast<cplx*>(fft_smem);
  const int t = threadIdx.x;
  unsigned long long bid = blockIdx.x;
  const long long x0 = (long long)(bid % p.tiles_x) * C;
  bid /= p.tiles_x;
  long long so_off[FFT_MAXB];
#pragma unroll
  for (int b = 0; b < FFT_MAXB; ++b) so_off[b] = 0;
  long long d_off = 0;
#pragma unroll 1
  for (int i = 0; i < p.no; ++i) {
    const long long k = (long long)(bid % (unsigned long long)p.oe[i]);
    bid /= (unsigned long long)p.oe[i];
    d_off += k * p.dso[i];
#pragma unroll
    for (int b = 0; b < FFT_MAXB; ++b)
      if (b < p.nb) so_off[b] += k * p.blk[b].so[i];
  }
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;

  // ---- gather (+ first pass): C threads read C consecutive columns (C x 16 B) of one
  //      source row.  A thread owns the rows r, r + RS, r + 2 RS, ... of its column: exactly
  //      the inputs of one butterfly of a first pass of radix R1 = L / RS -- so that pass runs
  //      on the values as they arrive from HBM, before they ever touch shared memory ----
  constexpr int RS = FFT_THREADS / C;  // rows per sweep
  constexpr int LOGRS = (C == 8) ? 5 : 6;
  static_assert((1 << LOGRS) == RS, "rows per sweep");
  // (only for 1024-point lines, where shared memory bounds the CTAs per SM; for 512-point
  //  lines the radix-16 butterfly's registers would cost the third resident CTA)
  constexpr int LOGR1 = (C == 4 && LOGL > LOGRS) ? (LOGL - LOGRS) : 0;
  static_assert(LOGR1 == 0 || LOGL - LOGR1 == LOGRS, "first-pass stride must equal the sweep");
  const cplx* twp = p.tw;
  auto tw = [twp](int i) {
    const double2 w = __ldg(reinterpret_cast<const double2*>(twp) + i);
    return cplx{w.x, w.y};
  };
  {
    // transposing gather: C consecutive threads read C consecutive columns of one source row;
    // linear gather (lines contiguous in the source): consecutive threads read along a line
    const int c = p.linear ? t / RS : t % C, r = p.linear ? t % RS : t / C;
    cplx* line = sm + c * pitch;
    if constexpr (LOGR1 > 0) {
      constexpr int R1 = 1 << LOGR1;
      if (c < ncol) {
        double2 v[R1];
#pragma unroll
        for (int q = 0; q < R1; ++q) {
          const int y = r + q * RS;
          const char* s = nullptr;
#pragma unroll
          for (int b = 0; b < FFT_MAXB; ++b)
            if (b < p.nb && y >= p.blk[b].y0 && y < p.blk[b].y0 + p.blk[b].ey)
              s = p.blk[b].src + so_off[b] + (long long)(y - p.blk[b].y0) * p.blk[b].ssy +
                  (x0 + c) * p.blk[b].ssx;
          v[q] = __ldcs(reinterpret_cast<const double2*>(s));
        }
        cplx a[R1];
#pragma unroll
        for (int q = 0; q < R1; ++q) a[q] = cplx{v[q].x, v[q].y};
        pa_fft::butterfly_regs<R1>(a, r, L, L, p.sign, tw);
#pragma unroll
        for (int q = 0; q < R1; ++q) line[pa_fft::pad_index(r + q * RS)] = a[q];
      }
    } else {
      constexpr int U = 8;
#pragma unroll
      for (int b = 0; b < FFT_MAXB; ++b) {
        if (b < p.nb) {
          const FftBlock& B = p.blk[b];
          const char* s = B.src + so_off[b] + (x0 + c) * B.ssx;
          const int ey = B.ey, y0 = B.y0;
          const long long ssy = B.ssy;
          for (int y = r; y < ey; y += U * RS) {
            double2 v[U];
#pragma unroll
            for (int k = 0; k < U; ++k) {
              const int yy = y + k * RS;
              if (c < ncol && yy < ey) v[k] = __ldcs(reinterpret_cast<const double2*>(s + (long long)yy * ssy));
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
              const int yy = y + k * RS;
              if (c < ncol && yy < ey) line[pa_fft::pad_index(y0 + yy)] = cplx{v[k].x, v[k].y};
            }
          }
        }
      }
    }
  }
  __syncthreads();

  // ---- remaining passes in shared memory (radices and strides are compile-time constants) ----
  fft_passes<LOGL, LOGL - LOGR1, C>(sm, pitch, ncol, p.sign, tw);

  // ---- store: natural order, every line one contiguous run ----
  char* d = p.dst + x0 * p.dsx + d_off;
  for (int c = 0; c < ncol; ++c) {
    const cplx* line = sm + c * pitch;
    double2* out = reinterpret_cast<double2*>(d + c * p.dsx);
#pragma unroll
    for (int k0 = 0; k0 < L; k0 += FFT_THREADS) {
      const int k = k0 + t;
      if (k < L) {
        // position of frequency k: first-pass digit, then the digits of the later passes
        const int pos = ((k & ((1 << LOGR1) - 1)) << (LOGL - LOGR1)) +
                        fft_pos<LOGL, LOGL - LOGR1>(k >> LOGR1);
        const cplx v = line[pa_fft::pad_index(pos)];
        __stcs(out + k, make_double2(v.x, v.y));
      }
    }
  }
}

// ---- real lines (rfft_ / brfft_, DESIGN §3c): N = 2L reals <-> N/2 + 1 complex bins ----
// The lines are dense and consecutive on both sides (the transform axis is the first memory dim
// of both arrays, the other dims are the same), so a launch is a flat batch of `nlines` lines.
struct RfftParams {
  const char* src;
  char* dst;
  long long nlines;
  long long src_line, dst_line;  // byte strides of consecutive lines
  int pitch;
  const cplx* tw;  // W_N^k, k < N: the post- / pre-pass reads entry k, the L-point passes entry 2i
};

template <int LOGL, int C, bool FWD>
__global__ void __launch_bounds__(FFT_THREADS) k_rfft(const __grid_constant__ RfftParams p) {
  constexpr int L = 1 << LOGL;
  constexpr int RS = FFT_THREADS / C;  // threads per line
  constexpr int P = L / 2 + 1;         // pairs (k, L - k) per line
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cplx* sm = reinterpret_cast<cplx*>(fft_smem);
  const int t = threadIdx.x;
  const long long l0 = (long long)blockIdx.x * C;
  const int ncol = (int)((p.nlines - l0) < C ? (p.nlines - l0) : C);
  const int pitch = p.pitch;
  const cplx* twp = p.tw;
  auto twN = [twp](int k) {
    const double2 w = __ldg(reinterpret_cast<const double2*>(twp) + k);
    return cplx{w.x, w.y};
  };
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const double2 w = __ldg(reinterpret_cast<const double2*>(twp) + 2 * i);
    return cplx{w.x, w.y};
  };

  // ---- load (linear gather): consecutive threads walk along a line with 128-bit loads.
  //      Forward: the N reals ARE the complex line z[n] = x[2n] + i x[2n+1]; backward: N/2+1 bins ----
  {
    constexpr int NIN = FWD ? L : L + 1;
    constexpr int U = (NIN + RS - 1) / RS;
    const int c = t / RS, r = t % RS;
    if (c < ncol) {
      const double2* s = reinterpret_cast<const double2*>(p.src + (l0 + c) * p.src_line);
      cplx* line = sm + c * pitch;
      double2 v[U];
#pragma unroll
      for (int q = 0; q < U; ++q)
        if (r + q * RS < NIN) v[q] = __ldcs(s + r + q * RS);
#pragma unroll
      for (int q = 0; q < U; ++q)
        if (r + q * RS < NIN) line[pa_fft::pad_index(r + q * RS)] = cplx{v[q].x, v[q].y};
    }
  }
  __syncthreads();

  if constexpr (!FWD) {
    // ---- pre-pass in place: a thread owns the slots k and L - k of its pair ----
#pragma unroll
    for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
      const int w = w0 + t, c = w / P, k = w % P;
      if (w < C * P && c < ncol) {
        cplx* line = sm + c * pitch;
        cplx zk, zl;
        pa_fft::brfft_pre_pair(k, line[pa_fft::pad_index(k)], line[pa_fft::pad_index(L - k)], twN(k),
                               &zk, &zl);
        line[pa_fft::pad_index(k)] = zk;
        if (k > 0) line[pa_fft::pad_index(L - k)] = zl;
      }
    }
    __syncthreads();
  }

  fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, FWD ? -1 : 1, twL);

  if constexpr (FWD) {
    // ---- post-pass + store: N/2 + 1 bins per line, one contiguous run ----
#pragma unroll
    for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
      const int w = w0 + t, c = w / P, k = w % P;
      if (w < C * P && c < ncol) {
        const cplx* line = sm + c * pitch;
        cplx xk, xl;
        pa_fft::rfft_post_pair(line[pa_fft::pad_index(fft_pos<LOGL, LOGL>(k & (L - 1)))],
                               line[pa_fft::pad_index(fft_pos<LOGL, LOGL>((L - k) & (L - 1)))], twN(k),
                               &xk, &xl);
        double2* out = reinterpret_cast<double2*>(p.dst + (l0 + c) * p.dst_line);
        __stcs(out + k, make_double2(xk.x, xk.y));
        if (k != L - k) __stcs(out + (L - k), make_double2(xl.x, xl.y));
      }
    }
  } else {
    // ---- store: z[n] = x[2n] + i x[2n+1], the N reals of a line as L 128-bit stores ----
#pragma unroll
    for (int w0 = 0; w0 < C * L; w0 += FFT_THREADS) {
      const int w = w0 + t, c = w >> LOGL, n = w & (L - 1);
      if (c < ncol) {
        const cplx v = sm[c * pitch + pa_fft::pad_index(fft_pos<LOGL, LOGL>(n))];
        __stcs(reinterpret_cast<double2*>(p.dst + (l0 + c) * p.dst_line) + n, make_double2(v.x, v.y));
      }
    }
  }
}

// forward twiddle table W_L^k per (device, L), computed once in extended precision
static const cplx* twiddles(int L) {
  static std::mutex mu;
  static std::map<std::pair<int, int>, cplx*> cache;
  std::lock_guard<std::mutex> lock(mu);
  int dev = 0;
  cudaGetDevice(&dev);
  auto key = std::make_pair(dev, L);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  std::vector<cplx> h(L);
  for (int k = 0; k < L; ++k) {
    const long double a = -2.0L * 3.141592653589793238462643383279502884L * k / L;
    h[k] = cplx{(double)cosl(a), (double)sinl(a)};
  }
  cplx* d = nullptr;
  if (cudaMalloc((void**)&d, sizeof(cplx) * L) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.data(), sizeof(cplx) * L, cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
  cache[key] = d;
  return d;
}

// Launch geometry of the fused kernel from the blocks of one rank (`blocks[i]` moves block i
// from `srcs[i]` -- recv_buf, or the src parent for the fused self block -- into `dst`;
// together they must tile the destination box), and every check of it.  srcs / dst may be
// NULL: plan_fft_check runs this on the blocks a peer would see, without arrays.  *grid = 0:
// nothing to do on this rank.
static pa_status fft_geometry(int nb, const BlockCopy* const* blocks, const void* const* srcs,
                              void* dst, FftParams& p, int* C_out, unsigned long long* grid_out) {
  memset(&p, 0, sizeof p);
  *grid_out = 0;
  // the line dim: destination stride 1 (and extent > 1) in some block
  int jy = -1;
  for (int b = 0; b < nb && jy < 0; ++b)
    for (int i = 0; i < blocks[b]->nd_raw; ++i)
      if (blocks[b]->raw[i].e > 1 && blocks[b]->raw[i].ds == 1) {
        jy = i;
        break;
      }
  // (every block one row long -- as many ranks as points: the dim of destination stride 1
  //  along which the blocks lie side by side)
  for (int i = 0; jy < 0 && nb > 0 && i < blocks[0]->nd_raw; ++i) {
    i64 rows = 0;
    bool unit = true;
    for (int b = 0; b < nb; ++b)
      if (blocks[b]->count > 0) {
        unit = unit && blocks[b]->nd_raw == blocks[0]->nd_raw && blocks[b]->raw[i].ds == 1;
        rows += blocks[b]->raw[i].e;
      }
    if (unit && rows > 1) jy = i;
  }
  if (jy < 0) {
    set_error("fused FFT: the destination has no contiguous dimension longer than 1");
    return PA_EINVAL;
  }
  // jy == 0: the transform axis is contiguous in the source too -- no transposition along it
  // (a local copy / permutation of the outer dims, or an in-place transform): the "columns"
  // are then the next dim, and only a single block (the whole local array) is supported
  const bool linear = (jy == 0);
  int jx = 0;  // the column dim: consecutive lines of a CTA
  if (linear) {
    int nonempty = 0;
    for (int b = 0; b < nb; ++b) nonempty += blocks[b]->count > 0;
    if (nonempty > 1) {
      set_error("fused FFT: the transform axis is contiguous in the source and the destination is "
                "assembled from several blocks: transform after the transposition instead");
      return PA_EINVAL;
    }
    jx = -1;
    for (int b = 0; b < nb && jx < 0; ++b)
      for (int i = 1; i < blocks[b]->nd_raw; ++i)
        if (blocks[b]->raw[i].e > 1) {
          jx = i;
          break;
        }
  }
  i64 min_doff = -1;
  const BlockCopy* ref = nullptr;
  for (int b = 0; b < nb; ++b) {
    const BlockCopy& B = *blocks[b];
    if (B.count == 0) continue;
    if (B.elsize != 16) {
      set_error("fused FFT: ComplexF64 (16-byte) elements only");
      return PA_EINVAL;
    }
    if (B.raw[0].ss != 1) {
      set_error("fused FFT: unexpected source layout");
      return PA_EINVAL;
    }
    if (linear && B.raw[0].ds != 1) {
      set_error("fused FFT: unexpected destination layout");
      return PA_EINVAL;
    }
    if (!ref) ref = &B;
    if (B.nd_raw != ref->nd_raw) {
      set_error("fused FFT: the blocks do not share their line set");
      return PA_EINVAL;
    }
    for (int i = 0; i < B.nd_raw; ++i)
      if (i != jy && (B.raw[i].e != ref->raw[i].e || B.raw[i].ds != ref->raw[i].ds)) {
        set_error("fused FFT: the blocks do not share their line set");
        return PA_EINVAL;
      }
    if (min_doff < 0 || B.dst_off < min_doff) min_doff = B.dst_off;
  }
  if (!ref) return PA_OK;  // nothing to do on this rank (*grid = 0)
  i64 L = 0;
  for (int b = 0; b < nb; ++b) {
    const BlockCopy& B = *blocks[b];
    if (B.count == 0) continue;
    if (p.nb >= FFT_MAXB) {
      set_error("fused FFT: more than %d blocks", FFT_MAXB);
      return PA_EINVAL;
    }
    FftBlock& F = p.blk[p.nb++];
    F.src = srcs ? (const char*)srcs[b] + B.src_off * 16 : nullptr;
    F.y0 = (int)(B.dst_off - min_doff);
    F.ey = (int)B.raw[jy].e;
    F.ssy = B.raw[jy].ss * 16;
    F.ssx = jx >= 0 ? B.raw[jx].ss * 16 : 16;
    int o = 0;
    for (int i = 1; i < B.nd_raw; ++i)
      if (i != jy && i != jx && B.raw[i].e > 1) F.so[o++] = B.raw[i].ss * 16;
    L += B.raw[jy].e;
  }
  int logL = 0;
  while ((1LL << logL) < L) ++logL;
  if ((1LL << logL) != L || L < 8 || L > 1024) {
    set_error("fused FFT: line length %lld is not a power of two in 8..1024", (long long)L);
    return PA_EINVAL;
  }
  // the blocks must tile [0, L) without gaps
  {
    std::vector<std::pair<int, int>> seg;
    for (int b = 0; b < p.nb; ++b) seg.push_back({p.blk[b].y0, p.blk[b].ey});
    std::sort(seg.begin(), seg.end());
    int pos = 0;
    for (auto& s : seg) {
      if (s.first != pos) {
        set_error("fused FFT: the blocks do not tile the transform axis");
        return PA_EINVAL;
      }
      pos += s.second;
    }
  }
  p.dst = dst ? (char*)dst + min_doff * 16 : nullptr;
  p.linear = linear ? 1 : 0;
  p.ex = jx >= 0 ? ref->raw[jx].e : 1;
  p.dsx = jx >= 0 ? ref->raw[jx].ds * 16 : 16;
  p.no = 0;
  for (int i = 1; i < ref->nd_raw; ++i)
    if (i != jy && i != jx && ref->raw[i].e > 1) {
      if (p.no >= FFT_MAXO) {
        set_error("fused FFT: more than %d outer dims", FFT_MAXO);
        return PA_EINVAL;
      }
      p.oe[p.no] = ref->raw[i].e;
      p.dso[p.no] = ref->raw[i].ds * 16;
      ++p.no;
    }
  p.L = (int)L;
  p.logL = logL;
  p.pitch = pa_fft::padded_pitch((int)L);
  // tunable "fft_lines" = 4: 4 lines per CTA also for 256- / 512-point lines (64-byte gathers,
  // first pass of radix 4 / 8 in registers, half the shared memory per CTA)
  const int C = (g_tun.fft_lines == 4 && logL >= 8) ? 4 : fft_lines(logL);
  p.tiles_x = (unsigned)((p.ex + C - 1) / C);
  unsigned long long grid = p.tiles_x;
  for (int i = 0; i < p.no; ++i) grid *= (unsigned long long)p.oe[i];
  if (grid > 0x7fffffffULL) {
    set_error("fused FFT: too many lines for one launch");
    return PA_EINVAL;
  }
  *C_out = C;
  *grid_out = grid;
  return PA_OK;
}

pa_status unpack_fft(int nb, const BlockCopy* const* blocks, const void* const* srcs, void* dst,
                     int sign, void* stream) {
  // (pa_transpose has already asked plan_fft_check, for every rank of the line, before it
  //  enqueued anything: these checks only guard direct callers)
  FftParams p;
  int C = 0;
  unsigned long long grid = 0;
  pa_status s = fft_geometry(nb, blocks, srcs, dst, p, &C, &grid);
  if (s != PA_OK || grid == 0) return s;
  const int logL = p.logL;
  p.sign = sign < 0 ? -1 : 1;
  p.tw = twiddles(p.L);
  if (!p.tw) {
    set_error("fused FFT: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const size_t smem = sizeof(cplx) * (size_t)C * p.pitch;
  cudaError_t e = cudaSuccess;
  auto launch = [&](auto kern) {
    // shared memory is the scarce resource: ask for the largest carve-out so that
    // several CTAs (gather of one, butterflies of another) overlap on an SM
    static bool configured = false;  // one static per instantiation of this lambda's closure type
    (void)configured;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    cudaGetLastError();
    kern<<<(unsigned)grid, FFT_THREADS, smem, (cudaStream_t)stream>>>(p);
    e = cudaGetLastError();
  };
  switch (logL) {
    case 3: launch(k_unpack_fft<3, 8>); break;
    case 4: launch(k_unpack_fft<4, 8>); break;
    case 5: launch(k_unpack_fft<5, 8>); break;
    case 6: launch(k_unpack_fft<6, 8>); break;
    case 7: launch(k_unpack_fft<7, 8>); break;
    case 8: if (C == 4) launch(k_unpack_fft<8, 4>); else launch(k_unpack_fft<8, 8>); break;
    case 9: if (C == 4) launch(k_unpack_fft<9, 4>); else launch(k_unpack_fft<9, 8>); break;
    default: launch(k_unpack_fft<10, 4>); break;
  }
  if (e != cudaSuccess) {
    set_error("fused FFT kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

// Can pa_transpose fuse the FFT into this plan's unpack?  Every rank of a grid line must
// get the same answer: a rank that refused before the exchange while its peers went ahead
// would leave them waiting on flags it never sets.  So the answer depends on the global
// geometry only: the blocks that EVERY rank of the line would gather -- each rank's plan
// rebuilt from the pencils with that rank's coordinates -- with the self block read from src
// and staged through recv_buf alike.  Cached per plan (and per value of tunable fft_lines).
pa_status plan_fft_check(Plan* P) {
  if (P->fft_check_lines == g_tun.fft_lines) {
    if (P->fft_check != PA_OK) set_error("%s", P->fft_check_err.c_str());
    return P->fft_check;
  }
  auto verdict = [&](pa_status s) {
    P->fft_check = s;
    P->fft_check_err = s == PA_OK ? std::string() : std::string(last_error());
    P->fft_check_lines = g_tun.fft_lines;
    return s;
  };
  if (P->elsize != 16) {
    set_error("fused FFT: ComplexF64 (16-byte) elements only");
    return verdict(PA_EINVAL);
  }
  FftParams p;
  int C = 0;
  unsigned long long grid = 0;
  if (P->dim < 0 || P->nproc == 1) {
    const BlockCopy* b = &P->self_fused;
    return verdict(fft_geometry(1, &b, nullptr, nullptr, p, &C, &grid));
  }
  for (int n = 0; n < P->nproc; ++n) {
    std::unique_ptr<Plan> hold;
    const Plan* Q = P;
    if (n != P->self_index) {
      auto topo = std::make_shared<Topology>(*P->pin->topo);
      topo->coords[P->dim] = n;
      topo->rank = topo->rank_of(topo->coords);
      auto pin = std::make_shared<Pencil>(*P->pin);
      auto pout = std::make_shared<Pencil>(*P->pout);
      pin->topo = topo;
      pout->topo = topo;
      Plan* q = nullptr;
      pa_status s = build_plan(pin, pout, P->n_extra, P->extra, P->elsize, P->method, &q);
      if (s != PA_OK) return verdict(s);
      hold.reset(q);
      Q = q;
    }
    for (int staged_self = 0; staged_self < 2; ++staged_self) {
      std::vector<const BlockCopy*> bl;
      for (int k = 0; k < Q->nproc; ++k)
        bl.push_back(k == Q->self_index && !staged_self ? &Q->self_fused : &Q->peers[k].unpack);
      pa_status s = fft_geometry(Q->nproc, bl.data(), nullptr, nullptr, p, &C, &grid);
      if (s != PA_OK) {
        if (n != P->self_index) {
          const std::string why = last_error();
          set_error("%s (on rank %d of the grid line)", why.c_str(), n + 1);
        }
        return verdict(s);
      }
    }
  }
  return verdict(PA_OK);
}

pa_status rfft_lines(int N, bool forward, i64 nlines, const void* src, void* dst, void* stream) {
  const int L = N / 2;
  int logL = 0;
  while ((1 << logL) < L) ++logL;
  if ((1 << logL) != L || logL < 3 || logL > 10) {
    set_error("rfft: line length %d is not a power of two in 16..2048", N);
    return PA_EINVAL;
  }
  if (nlines == 0) return PA_OK;
  RfftParams p;
  p.src = (const char*)src;
  p.dst = (char*)dst;
  p.nlines = nlines;
  p.src_line = forward ? 8LL * N : 16LL * (L + 1);
  p.dst_line = forward ? 16LL * (L + 1) : 8LL * N;
  p.pitch = pa_fft::padded_pitch(forward ? L : L + 1);  // backward stages all N/2 + 1 bins
  p.tw = twiddles(N);
  if (!p.tw) {
    set_error("rfft: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const int C = fft_lines(logL);
  const long long grid = (nlines + C - 1) / C;
  if (grid > 0x7fffffffLL) {
    set_error("rfft: too many lines for one launch");
    return PA_EINVAL;
  }
  const size_t smem = sizeof(cplx) * (size_t)C * p.pitch;
  cudaError_t e = cudaSuccess;
  auto launch = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    cudaGetLastError();
    kern<<<(unsigned)grid, FFT_THREADS, smem, (cudaStream_t)stream>>>(p);
    e = cudaGetLastError();
  };
  auto launch_dir = [&](auto fwd_kern, auto bwd_kern) { forward ? launch(fwd_kern) : launch(bwd_kern); };
  switch (logL) {
    case 3: launch_dir(k_rfft<3, 8, true>, k_rfft<3, 8, false>); break;
    case 4: launch_dir(k_rfft<4, 8, true>, k_rfft<4, 8, false>); break;
    case 5: launch_dir(k_rfft<5, 8, true>, k_rfft<5, 8, false>); break;
    case 6: launch_dir(k_rfft<6, 8, true>, k_rfft<6, 8, false>); break;
    case 7: launch_dir(k_rfft<7, 8, true>, k_rfft<7, 8, false>); break;
    case 8: launch_dir(k_rfft<8, 8, true>, k_rfft<8, 8, false>); break;
    case 9: launch_dir(k_rfft<9, 8, true>, k_rfft<9, 8, false>); break;
    default: launch_dir(k_rfft<10, 4, true>, k_rfft<10, 4, false>); break;
  }
  if (e != cudaSuccess) {
    set_error("rfft kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

}  // namespace pa
