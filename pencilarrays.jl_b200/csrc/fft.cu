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
//
// Single precision (PA_FFT_F32, DESIGN §3d): the same kernels instantiated for float --
// ComplexF32 elements, fp32 arithmetic, an fp32 twiddle table rounded from the same
// long-double values -- with 16 lines per CTA (128-byte gathers again), 8 for 1024 points.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

// twiddles: one table lookup per butterfly, the other powers by squaring / products (the
// lookups share the load/store path with shared memory, the kernel's limiter)
#ifndef PA_FFT_TWIDDLE_LOOKUPS
#define PA_FFT_TWIDDLE_LOOKUPS 1
#endif
#include "fft_core.hpp"
#include "flags.cuh"
#include "pa_internal.hpp"

namespace pa {

using pa_fft::cplx;
using pa_fft::cplx_t;

// the 64-bit (float2) or 128-bit (double2) vector of one complex element
template <class T>
struct Vec2;
template <>
struct Vec2<double> {
  using type = double2;
};
template <>
struct Vec2<float> {
  using type = float2;
};
__device__ __forceinline__ double2 vec2(double x, double y) { return make_double2(x, y); }
__device__ __forceinline__ float2 vec2(float x, float y) { return make_float2(x, y); }

constexpr int FFT_MAXB = 8;   // blocks gathered by one launch (ranks of a grid line on one box)
constexpr int FFT_MAXO = PA_MAX_DIMS - 2;
constexpr int FFT_THREADS = 256;
// lines per CTA: 8 (128-byte gathers); 4 for 1024-point lines so that three CTAs still
// share an SM's shared memory (75 KB each)
constexpr int fft_lines(int logL) { return logL >= 10 ? 4 : 8; }
// single precision: twice as many lines in the same shared memory -- 16 (128-byte gathers of
// 8-byte elements) up to 512 points, 8 for 1024 points
constexpr int fft_lines_f32(int logL) { return logL >= 10 ? 8 : 16; }

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
  const void* tw;  // twiddle table of the kernel's precision (cplx or cplxf)
  unsigned tiles_x;
  // k_unpack_r2r only (after the fields the other kernels read, which keep their offsets)
  const void* tw4;  // W_4N^k, as R2rParams::tw4
  int sine;         // DST (RODFT10 / RODFT01) instead of DCT
};

template <class T>
struct SmLine {
  cplx_t<T>* p;
  __device__ __forceinline__ cplx_t<T> get(int i) const { return p[pa_fft::pad_index(i)]; }
  __device__ __forceinline__ void put(int i, cplx_t<T> v) { p[pa_fft::pad_index(i)] = v; }
};

// radix of the pass that starts at sub-length 2^LOGM (the odd bits go first: radices_of)
template <int LOGM>
struct PassRadix {
  static constexpr int LOGR = (LOGM % 3 == 0) ? 3 : (LOGM % 3);
};

template <int LOGL, int LOGM, int C, class T, class Tw>
__device__ __forceinline__ void fft_passes(cplx_t<T>* sm, int pitch, int ncol, int sign, const Tw& tw) {
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
        SmLine<T> x{sm + c * pitch};
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

// The gather of every block's rows of one line into shared memory (thread (c, r) owns column
// c and the rows r, r + RS, ... of every block).  Any total row count: the blocks tile it.
template <int C, class T>
__device__ __forceinline__ void gather_rows(const FftParams& p, const long long* so_off, long long x0,
                                            int c, int r, int ncol, cplx_t<T>* line) {
  using V = typename Vec2<T>::type;
  constexpr int RS = FFT_THREADS / C;
  constexpr int U = 8;
#pragma unroll
  for (int b = 0; b < FFT_MAXB; ++b) {
    if (b < p.nb) {
      const FftBlock& B = p.blk[b];
      const char* s = B.src + so_off[b] + (x0 + c) * B.ssx;
      const int ey = B.ey, y0 = B.y0;
      const long long ssy = B.ssy;
      for (int y = r; y < ey; y += U * RS) {
        V v[U];
#pragma unroll
        for (int k = 0; k < U; ++k) {
          const int yy = y + k * RS;
          if (c < ncol && yy < ey) v[k] = __ldcs(reinterpret_cast<const V*>(s + (long long)yy * ssy));
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
          const int yy = y + k * RS;
          if (c < ncol && yy < ey) line[pa_fft::pad_index(y0 + yy)] = cplx_t<T>{v[k].x, v[k].y};
        }
      }
    }
  }
}

// Where real n of a line goes in a shared-memory line of N = 2L reals (viewed as T: part i & 1
// of complex slot i / 2 is entry 2 pad_index(i / 2) + (i & 1)) -- the maps k_rfft's and k_r2r's
// loads apply, one real at a time, so a slot may be filled from two different blocks.
enum class RealMap {
  rfft,  // identity: z[n] = x[2n] + i x[2n+1]
  dct2,  // Makhoul: v[m] = x[2m], v[N-1-m] = x[2m+1] (DST-II: -x[2m+1])
  dct3,  // slot j holds (X[j], X[N-j]), j = 0 ... L (DST-III: X reversed)
};

template <RealMap MAP, int LOGL, class T>
__device__ __forceinline__ void put_real(T* line, int n, T x, bool sine) {
  constexpr int L = 1 << LOGL, N = 2 * L;
  if constexpr (MAP == RealMap::rfft) {
    line[2 * pa_fft::pad_index(n >> 1) + (n & 1)] = x;
  } else if constexpr (MAP == RealMap::dct2) {
    const int i = (n & 1) ? N - 1 - (n >> 1) : (n >> 1);
    line[2 * pa_fft::pad_index(i >> 1) + (i & 1)] = ((n & 1) && sine) ? -x : x;
  } else {
    const int j = sine ? N - 1 - n : n;
    if (j <= L) line[2 * pa_fft::pad_index(j)] = x;
    if (j >= L) line[2 * pa_fft::pad_index(N - j) + 1] = x;
  }
}

// gather_rows for real elements (8-byte Float64, 4-byte Float32): every block's rows of one line,
// each real handed to put(n, x) with its position n along the line.  A block may start or end
// at an odd position, so nothing here assumes pairs.
template <int C, class T, class Put>
__device__ __forceinline__ void gather_real_rows(const FftParams& p, const long long* so_off, long long x0,
                                                 int c, int r, int ncol, const Put& put) {
  constexpr int RS = FFT_THREADS / C;
  constexpr int U = 8;
#pragma unroll
  for (int b = 0; b < FFT_MAXB; ++b) {
    if (b < p.nb) {
      const FftBlock& B = p.blk[b];
      const char* s = B.src + so_off[b] + (x0 + c) * B.ssx;
      const int ey = B.ey, y0 = B.y0;
      const long long ssy = B.ssy;
      for (int y = r; y < ey; y += U * RS) {
        T v[U];
#pragma unroll
        for (int k = 0; k < U; ++k) {
          const int yy = y + k * RS;
          if (c < ncol && yy < ey) v[k] = __ldcs(reinterpret_cast<const T*>(s + (long long)yy * ssy));
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
          const int yy = y + k * RS;
          if (c < ncol && yy < ey) put(y0 + yy, v[k]);
        }
      }
    }
  }
}

// CTA -> (first column x0, byte offsets of the outer coordinates in every block and in dst)
__device__ __forceinline__ long long cta_offsets(const FftParams& p, int C, long long* so_off,
                                                 long long* d_off) {
  unsigned long long bid = blockIdx.x;
  const long long x0 = (long long)(bid % p.tiles_x) * C;
  bid /= p.tiles_x;
#pragma unroll
  for (int b = 0; b < FFT_MAXB; ++b) so_off[b] = 0;
  *d_off = 0;
#pragma unroll 1
  for (int i = 0; i < p.no; ++i) {
    const long long k = (long long)(bid % (unsigned long long)p.oe[i]);
    bid /= (unsigned long long)p.oe[i];
    *d_off += k * p.dso[i];
#pragma unroll
    for (int b = 0; b < FFT_MAXB; ++b)
      if (b < p.nb) so_off[b] += k * p.blk[b].so[i];
  }
  return x0;
}

// The first pass of a CTA of C lines that runs in registers on the gathered values: radix
// 2^LOGR1 (0: none).  A thread owns the rows r, r + RS, r + 2 RS, ... of its line: exactly the
// inputs of one butterfly of a first pass of radix R1 = L / RS.  (Only for 1024-point lines,
// where shared memory bounds the CTAs per SM; for 512-point lines the radix-16 butterfly's
// registers would cost the third resident CTA.  Single precision holds 8 1024-point lines: a
// sweep of 32 rows would need a radix-32 pass, which does not exist, so every pass runs in
// shared memory there)
template <int LOGL, int C, class T>
struct FftCtaShape {
  static constexpr int RS = FFT_THREADS / C;  // rows per sweep
  static constexpr int LOGRS = (C == 16) ? 4 : (C == 8) ? 5 : 6;
  static_assert((1 << LOGRS) == RS, "rows per sweep");
  static constexpr int LOGR1 = (sizeof(T) == 8 && C == 4 && LOGL > LOGRS) ? (LOGL - LOGRS) : 0;
  static_assert(LOGR1 == 0 || LOGL - LOGR1 == LOGRS, "first-pass stride must equal the sweep");
  static_assert(LOGR1 <= 4, "the register first pass is at most radix 16");
};

// The load and the passes of one CTA of the complex FFT (k_unpack_fft, k_get_fft, k_fft_put): the
// C lines gathered from every block of p into shared memory (+ the register first pass), then the
// remaining passes.  Output frequency k of line c is then at fft_out_pos<LOGL, LOGR1>(k).
template <int LOGL, int C, class T>
__device__ __forceinline__ void fft_cta_lines(const FftParams& p, const long long* so_off, long long x0,
                                              int ncol, cplx_t<T>* sm) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  const int t = threadIdx.x;
  const int pitch = p.pitch;

  // ---- gather (+ first pass): C threads read C consecutive columns (C x sizeof(cx)) of one
  //      source row; the first pass (FftCtaShape) runs on the values as they arrive from HBM,
  //      before they ever touch shared memory ----
  constexpr int RS = FftCtaShape<LOGL, C, T>::RS;
  constexpr int LOGR1 = FftCtaShape<LOGL, C, T>::LOGR1;
  const V* twp = reinterpret_cast<const V*>(p.tw);
  auto tw = [twp](int i) {
    const V w = __ldg(twp + i);
    return cx{w.x, w.y};
  };
  {
    // transposing gather: C consecutive threads read C consecutive columns of one source row;
    // linear gather (lines contiguous in the source): consecutive threads read along a line
    const int c = p.linear ? t / RS : t % C, r = p.linear ? t % RS : t / C;
    cx* line = sm + c * pitch;
    if constexpr (LOGR1 > 0) {
      constexpr int R1 = 1 << LOGR1;
      if (c < ncol) {
        V v[R1];
#pragma unroll
        for (int q = 0; q < R1; ++q) {
          const int y = r + q * RS;
          const char* s = nullptr;
#pragma unroll
          for (int b = 0; b < FFT_MAXB; ++b)
            if (b < p.nb && y >= p.blk[b].y0 && y < p.blk[b].y0 + p.blk[b].ey)
              s = p.blk[b].src + so_off[b] + (long long)(y - p.blk[b].y0) * p.blk[b].ssy +
                  (x0 + c) * p.blk[b].ssx;
          v[q] = __ldcs(reinterpret_cast<const V*>(s));
        }
        cx a[R1];
#pragma unroll
        for (int q = 0; q < R1; ++q) a[q] = cx{v[q].x, v[q].y};
        pa_fft::butterfly_regs<R1>(a, r, L, L, p.sign, tw);
#pragma unroll
        for (int q = 0; q < R1; ++q) line[pa_fft::pad_index(r + q * RS)] = a[q];
      }
    } else {
      gather_rows<C, T>(p, so_off, x0, c, r, ncol, line);
    }
  }
  __syncthreads();

  // ---- remaining passes in shared memory (radices and strides are compile-time constants) ----
  fft_passes<LOGL, LOGL - LOGR1, C>(sm, pitch, ncol, p.sign, tw);
}

// storage position of output frequency k after fft_cta_lines: first-pass digit, then the digits
// of the later passes
template <int LOGL, int LOGR1>
__device__ __forceinline__ int fft_out_pos(int k) {
  return ((k & ((1 << LOGR1) - 1)) << (LOGL - LOGR1)) + fft_pos<LOGL, LOGL - LOGR1>(k >> LOGR1);
}

// One CTA of the fused unpack + FFT: gather its C lines from every block, transform, store.
template <int LOGL, int C, class T>
__device__ __forceinline__ void unpack_fft_cta(const FftParams& p) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const int t = threadIdx.x;
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;
  constexpr int LOGR1 = FftCtaShape<LOGL, C, T>::LOGR1;

  fft_cta_lines<LOGL, C, T>(p, so_off, x0, ncol, sm);

  // ---- store: natural order, every line one contiguous run ----
  char* d = p.dst + x0 * p.dsx + d_off;
  for (int c = 0; c < ncol; ++c) {
    const cx* line = sm + c * pitch;
    V* out = reinterpret_cast<V*>(d + c * p.dsx);
#pragma unroll
    for (int k0 = 0; k0 < L; k0 += FFT_THREADS) {
      const int k = k0 + t;
      if (k < L) {
        // position of frequency k: first-pass digit, then the digits of the later passes
        const int pos = ((k & ((1 << LOGR1) - 1)) << (LOGL - LOGR1)) +
                        fft_pos<LOGL, LOGL - LOGR1>(k >> LOGR1);
        const cx v = line[pa_fft::pad_index(pos)];
        __stcs(out + k, vec2(v.x, v.y));
      }
    }
  }
}

template <int LOGL, int C, class T>
__global__ void __launch_bounds__(FFT_THREADS) k_unpack_fft(const __grid_constant__ FftParams p) {
  unpack_fft_cta<LOGL, C, T>(p);
}

// ---- one-sided fused unpack + FFT (PeerGet, DESIGN §3h) ----
// The same CTA as k_unpack_fft, its remote blocks read straight out of the peers' src arrays
// through their peer mappings, bracketed by k_multi's window protocol: the first CTAs tell every
// peer READY ("my src is final and may be read"), and every CTA waits for READY from every peer
// before its first remote load (each line gathers from every block).  The CTA that finishes last
// tells every peer DONE ("I have finished reading your src"); the wait for the peers' DONE only
// guards the reuse of my src, so it is not in the kernel (get flavour: mf.wait_done is ignored).
// Empty flag sets: the plain gather from the mapped arrays (pa_get_all_fft, or a launch that
// standalone flag kernels bracket).
struct FftGetParams {
  FftParams p;
  MultiFlags mf;
};
static_assert(sizeof(FftGetParams) <= 4096, "FftParams + MultiFlags must fit the kernel parameters");

// (a register cap instead of __launch_bounds__(FFT_THREADS): under the launch bound ptxas
//  spills 4 bytes in the 64- and 128-point double-precision instantiations, as it does in
//  k_unpack_fft; with the cap no instantiation spills)
template <int LOGL, int C, class T>
__global__ void __maxnreg__(128) k_get_fft(const __grid_constant__ FftGetParams gp) {
  const MultiFlags& mf = gp.mf;
  if (mf.ready.n > 0) {
    if ((int)threadIdx.x < mf.ready.n) {
      if (blockIdx.x < 8) flag_signal(mf.ready.remote[threadIdx.x], mf.ready.seq[threadIdx.x]);
      flag_wait(mf.ready.local[threadIdx.x], mf.ready.seq[threadIdx.x], mf.timeout_ns, mf.err);
    }
    __syncthreads();
  }
  unpack_fft_cta<LOGL, C, T>(gp.p);
  if (mf.done.n > 0) {
    // every load of this CTA has been consumed (its lines are in shared memory or stored);
    // the last CTA to get here closes the window.  (No static shared memory: the 1024-point
    // instantiations fill three CTAs per SM with their dynamic shared memory alone)
    __syncthreads();
    int last = 0;
    if (threadIdx.x == 0) {
      __threadfence_system();
      last = atomicAdd(mf.counter, 1u) == gridDim.x - 1;
      if (last) {
        *mf.counter = 0;  // ready for the next launch (stream-ordered after this one)
        __threadfence_system();
      }
    }
    if (__syncthreads_or(last) && (int)threadIdx.x < mf.done.n)
      flag_signal(mf.done.remote[threadIdx.x], mf.done.seq[threadIdx.x]);
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
  const void* tw;  // W_N^k, k < N: the post- / pre-pass reads entry k, the L-point passes entry 2i
};

// The forward half of k_rfft after its load (k_unpack_rfft runs it after its gather): the L-point
// passes on the C shared-memory lines z[n] = x[2n] + i x[2n+1], then the post-pass and the store
// of the N/2 + 1 bins of line c at out(c).  tw = W_N.
template <int LOGL, int C, class T, class Out>
__device__ __forceinline__ void rfft_forward_tail(cplx_t<T>* sm, int pitch, int ncol, int t,
                                                  const typename Vec2<T>::type* twp, const Out& out) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  auto twN = [twp](int k) {
    const V w = __ldg(twp + k);
    return cx{w.x, w.y};
  };
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const V w = __ldg(twp + 2 * i);
    return cx{w.x, w.y};
  };
  fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, -1, twL);

  // ---- post-pass + store: N/2 + 1 bins per line, one contiguous run ----
#pragma unroll
  for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
    const int w = w0 + t, c = w / P, k = w % P;
    if (w < C * P && c < ncol) {
      const cx* line = sm + c * pitch;
      cx xk, xl;
      pa_fft::rfft_post_pair(line[pa_fft::pad_index(fft_pos<LOGL, LOGL>(k & (L - 1)))],
                             line[pa_fft::pad_index(fft_pos<LOGL, LOGL>((L - k) & (L - 1)))], twN(k),
                             &xk, &xl);
      V* o = reinterpret_cast<V*>(out(c));
      __stcs(o + k, vec2(xk.x, xk.y));
      if (k != L - k) __stcs(o + (L - k), vec2(xl.x, xl.y));
    }
  }
}

// The load of k_rfft (k_rfft_put loads its lines with it too), linear: consecutive threads walk
// along a line, one element per load, the RS threads of line c reading it from src(c).
// Forward: the N reals ARE the complex line z[n] = x[2n] + i x[2n+1]; backward: N/2+1 bins.
template <int LOGL, int C, bool FWD, class T, class Src>
__device__ __forceinline__ void rfft_load(cplx_t<T>* sm, int pitch, int ncol, int t, const Src& src) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  constexpr int RS = FFT_THREADS / C;
  constexpr int NIN = FWD ? L : L + 1;
  constexpr int U = (NIN + RS - 1) / RS;
  const int c = t / RS, r = t % RS;
  if (c < ncol) {
    const V* s = src(c);
    cx* line = sm + c * pitch;
    V v[U];
#pragma unroll
    for (int q = 0; q < U; ++q)
      if (r + q * RS < NIN) v[q] = __ldcs(s + r + q * RS);
#pragma unroll
    for (int q = 0; q < U; ++q)
      if (r + q * RS < NIN) line[pa_fft::pad_index(r + q * RS)] = cx{v[q].x, v[q].y};
  }
}

// Single precision: complex lines are 8 (N/2 + 1) bytes, an odd multiple of 8, so every other
// line starts only 8-byte aligned; every access is one 8-byte element (float2) on both sides.
template <int LOGL, int C, bool FWD, class T>
__global__ void __launch_bounds__(FFT_THREADS) k_rfft(const __grid_constant__ RfftParams p) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const int t = threadIdx.x;
  const long long l0 = (long long)blockIdx.x * C;
  const int ncol = (int)((p.nlines - l0) < C ? (p.nlines - l0) : C);
  const int pitch = p.pitch;
  const V* twp = reinterpret_cast<const V*>(p.tw);
  auto twN = [twp](int k) {
    const V w = __ldg(twp + k);
    return cx{w.x, w.y};
  };
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const V w = __ldg(twp + 2 * i);
    return cx{w.x, w.y};
  };

  // ---- load (linear gather): consecutive threads walk along a line, one element per load ----
  rfft_load<LOGL, C, FWD, T>(sm, pitch, ncol, t, [&p, l0](int c) {
    return reinterpret_cast<const V*>(p.src + (l0 + c) * p.src_line);
  });
  __syncthreads();

  if constexpr (FWD) {
    rfft_forward_tail<LOGL, C, T>(sm, pitch, ncol, t, twp,
                                  [&p, l0](int c) { return p.dst + (l0 + c) * p.dst_line; });
  } else {
    // ---- pre-pass in place: a thread owns the slots k and L - k of its pair ----
#pragma unroll
    for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
      const int w = w0 + t, c = w / P, k = w % P;
      if (w < C * P && c < ncol) {
        cx* line = sm + c * pitch;
        cx zk, zl;
        pa_fft::brfft_pre_pair(k, line[pa_fft::pad_index(k)], line[pa_fft::pad_index(L - k)], twN(k),
                               &zk, &zl);
        line[pa_fft::pad_index(k)] = zk;
        if (k > 0) line[pa_fft::pad_index(L - k)] = zl;
      }
    }
    __syncthreads();

    fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, 1, twL);

    // ---- store: z[n] = x[2n] + i x[2n+1], the N reals of a line as L pair stores ----
#pragma unroll
    for (int w0 = 0; w0 < C * L; w0 += FFT_THREADS) {
      const int w = w0 + t, c = w >> LOGL, n = w & (L - 1);
      if (c < ncol) {
        const cx v = sm[c * pitch + pa_fft::pad_index(fft_pos<LOGL, LOGL>(n))];
        __stcs(reinterpret_cast<V*>(p.dst + (l0 + c) * p.dst_line) + n, vec2(v.x, v.y));
      }
    }
  }
}

// ---- fused unpack + complex-to-real line transform (pa_transpose_brfft, DESIGN §3e) ----
// The gather of k_unpack_fft (the N/2 + 1 = L + 1 bins of each line from every block), then the
// backward half of k_rfft on the shared-memory lines: its pre-pass, its L-point passes and its
// store of the N reals.  p.dst / p.dsx / p.dso address the REAL destination (fft_geometry
// converts them); p.L = N / 2; p.tw = W_N.  Same lines per CTA as k_rfft for that N.
template <int LOGL, int C, class T>
__global__ void __launch_bounds__(FFT_THREADS) k_unpack_brfft(const __grid_constant__ FftParams p) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  constexpr int RS = FFT_THREADS / C;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const int t = threadIdx.x;
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;
  const V* twp = reinterpret_cast<const V*>(p.tw);
  auto twN = [twp](int k) {
    const V w = __ldg(twp + k);
    return cx{w.x, w.y};
  };
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const V w = __ldg(twp + 2 * i);
    return cx{w.x, w.y};
  };

  // ---- gather: transposing, or linear (lines contiguous in the source) ----
  {
    const int c = p.linear ? t / RS : t % C, r = p.linear ? t % RS : t / C;
    gather_rows<C, T>(p, so_off, x0, c, r, ncol, sm + c * pitch);
  }
  __syncthreads();

  // ---- pre-pass in place (k_rfft<..., false>): a thread owns the slots k and L - k ----
#pragma unroll 1
  for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
    const int w = w0 + t, c = w / P, k = w % P;
    if (w < C * P && c < ncol) {
      cx* line = sm + c * pitch;
      cx zk, zl;
      pa_fft::brfft_pre_pair(k, line[pa_fft::pad_index(k)], line[pa_fft::pad_index(L - k)], twN(k), &zk,
                             &zl);
      line[pa_fft::pad_index(k)] = zk;
      if (k > 0) line[pa_fft::pad_index(L - k)] = zl;
    }
  }
  __syncthreads();

  fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, 1, twL);

  // ---- store: z[n] = x[2n] + i x[2n+1], the N reals of a line as L pair stores ----
  char* d = p.dst + x0 * p.dsx + d_off;
#pragma unroll
  for (int w0 = 0; w0 < C * L; w0 += FFT_THREADS) {
    const int w = w0 + t, c = w >> LOGL, n = w & (L - 1);
    if (c < ncol) {
      const cx v = sm[c * pitch + pa_fft::pad_index(fft_pos<LOGL, LOGL>(n))];
      __stcs(reinterpret_cast<V*>(d + c * p.dsx) + n, vec2(v.x, v.y));
    }
  }
}

// ---- real-to-real lines (r2r_, DESIGN §3f): DCT-II / DCT-III of N = 2L reals through the
// real-line path of k_rfft (Makhoul's reordering, fft_core.hpp); DST-II / DST-III are sign and
// order changes of those in the load and the store.  Source and destination lines are both N
// dense reals; every line of a CTA is in shared memory before any store, so src == dst is safe.
struct R2rParams {
  const char* src;
  char* dst;
  long long nlines;
  long long line;   // byte stride of consecutive lines (N reals), both sides
  int pitch;
  int sine;         // DST (RODFT10 / RODFT01) instead of DCT (REDFT10 / REDFT01)
  const void* tw;   // W_N^k, k < N: the rfft table
  const void* tw4;  // W_4N^k: w_k = exp(-i pi k / 2N), k <= N/2
};

// The DCT-III pre-pass of the 01 kinds in place (r2r_tail, k_r2r_put): a thread owns the slots k
// and L - k of its pair.  tw = W_N, tw4 = W_4N.
template <int LOGL, int C, class T>
__device__ __forceinline__ void r2r_pre(cplx_t<T>* sm, int pitch, int ncol, int t,
                                        const typename Vec2<T>::type* twp,
                                        const typename Vec2<T>::type* tw4p) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  auto twN = [twp](int k) {
    const V w = __ldg(twp + k);
    return cx{w.x, w.y};
  };
  auto w4 = [tw4p](int k) {  // w_k = W_4N^k
    const V w = __ldg(tw4p + k);
    return cx{w.x, w.y};
  };
#pragma unroll
  for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
    const int w = w0 + t, c = w / P, k = w % P;
    if (w < C * P && c < ncol) {
      cx* line = sm + c * pitch;
      const cx vk = pa_fft::dct3_pre_pair(line[pa_fft::pad_index(k)], w4(k));
      const cx vl = pa_fft::dct3_pre_pair(line[pa_fft::pad_index(L - k)], w4(L - k));
      cx zk, zl;
      pa_fft::brfft_pre_pair(k, vk, vl, twN(k), &zk, &zl);
      line[pa_fft::pad_index(k)] = zk;
      if (k > 0) line[pa_fft::pad_index(L - k)] = zl;
    }
  }
  __syncthreads();
}

// k_r2r after its load (k_unpack_r2r runs it after its gather): the DCT-III pre-pass for the 01
// kinds, the L-point passes, and the DCT-II post-pass and store (10 kinds) or the store of the N
// reals (01 kinds) of line c at out(c).  tw = W_N, tw4 = W_4N.
template <int LOGL, int C, bool FWD, class T, class Out>
__device__ __forceinline__ void r2r_tail(cplx_t<T>* sm, int pitch, int ncol, int t, bool sine,
                                         const typename Vec2<T>::type* twp,
                                         const typename Vec2<T>::type* tw4p, const Out& out) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL, N = 2 * L;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  auto twN = [twp](int k) {
    const V w = __ldg(twp + k);
    return cx{w.x, w.y};
  };
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const V w = __ldg(twp + 2 * i);
    return cx{w.x, w.y};
  };
  auto w4 = [tw4p](int k) {  // w_k = W_4N^k
    const V w = __ldg(tw4p + k);
    return cx{w.x, w.y};
  };

  if constexpr (!FWD) r2r_pre<LOGL, C, T>(sm, pitch, ncol, t, twp, tw4p);

  fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, FWD ? -1 : 1, twL);

  if constexpr (FWD) {
    // ---- post-pass + store: the pair k yields V[k] and V[L-k], hence Y[k], Y[N-k], Y[L-k] and
    //      Y[L+k]; each of the N outputs is stored once.  DST-II stores Y[j] at N-1-j ----
#pragma unroll
    for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
      const int w = w0 + t, c = w / P, k = w % P;
      if (w < C * P && c < ncol) {
        const cx* line = sm + c * pitch;
        cx vk, vl;
        pa_fft::rfft_post_pair(line[pa_fft::pad_index(fft_pos<LOGL, LOGL>(k & (L - 1)))],
                               line[pa_fft::pad_index(fft_pos<LOGL, LOGL>((L - k) & (L - 1)))], twN(k),
                               &vk, &vl);
        T yk, ynk, yl, ynl;
        pa_fft::dct2_post_pair(vk, w4(k), &yk, &ynk);      // Y[k], Y[N-k]
        pa_fft::dct2_post_pair(vl, w4(L - k), &yl, &ynl);  // Y[L-k], Y[L+k]
        T* o = reinterpret_cast<T*>(out(c));
        auto put = [o, sine](int j, T y) { __stcs(o + (sine ? N - 1 - j : j), y); };
        put(k, yk);
        if (k > 0 && k < L / 2) put(N - k, ynk);
        if (k < L / 2) put(L - k, yl);
        if (k > 0) put(L + k, ynl);
      }
    }
  } else {
    // ---- store: x[2m] = v[m], x[2m+1] = v[N-1-m] as L pair stores; DST-III: times (-1)^n ----
#pragma unroll
    for (int w0 = 0; w0 < C * L; w0 += FFT_THREADS) {
      const int w = w0 + t, c = w >> LOGL, m = w & (L - 1);
      if (c < ncol) {
        const T* line = reinterpret_cast<const T*>(sm + c * pitch);
        const int i = N - 1 - m;
        const T a = line[2 * pa_fft::pad_index(fft_pos<LOGL, LOGL>(m >> 1)) + (m & 1)];
        const T b = line[2 * pa_fft::pad_index(fft_pos<LOGL, LOGL>(i >> 1)) + (i & 1)];
        __stcs(reinterpret_cast<V*>(out(c)) + m, vec2(a, sine ? -b : b));
      }
    }
  }
}

// The load of k_r2r (k_r2r_put loads its lines with it too), linear as k_rfft's: the reals
// (x[2m], x[2m+1]) of a line, one element per load, the RS threads of line c reading it from
// src(c), reordered on their way into shared memory
template <int LOGL, int C, bool FWD, class T, class Src>
__device__ __forceinline__ void r2r_load(cplx_t<T>* sm, int pitch, int ncol, int t, bool sine,
                                         const Src& src) {
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL, N = 2 * L;
  constexpr int RS = FFT_THREADS / C;  // threads per line
  constexpr int U = (L + RS - 1) / RS;
  const int c = t / RS, r = t % RS;
  if (c < ncol) {
    const V* s = src(c);
    T* line = reinterpret_cast<T*>(sm + c * pitch);
    V v[U];
#pragma unroll
    for (int q = 0; q < U; ++q)
      if (r + q * RS < L) v[q] = __ldcs(s + r + q * RS);
#pragma unroll
    for (int q = 0; q < U; ++q) {
      const int m = r + q * RS;
      if (m < L) {
        if constexpr (FWD) {
          // DCT-II: v[m] = x[2m], v[N-1-m] = x[2m+1], v[i] the part i & 1 of complex slot i / 2.
          // DST-II transforms (-1)^n x[n]
          line[2 * pa_fft::pad_index(m >> 1) + (m & 1)] = v[q].x;
          line[2 * pa_fft::pad_index((N - 1 - m) >> 1) + ((N - 1 - m) & 1)] = sine ? -v[q].y : v[q].y;
        } else {
          // DCT-III: slot j holds (X[j], X[N-j]), j = 0 ... L, as brfft_pre_pair's pairs do.
          // DST-III transforms X reversed: X[2m] is then entry N-1-2m
          const int ja = sine ? N - 1 - 2 * m : 2 * m, jb = sine ? N - 2 - 2 * m : 2 * m + 1;
          if (ja <= L) line[2 * pa_fft::pad_index(ja)] = v[q].x;
          if (ja >= L) line[2 * pa_fft::pad_index(N - ja) + 1] = v[q].x;
          if (jb <= L) line[2 * pa_fft::pad_index(jb)] = v[q].y;
          if (jb >= L) line[2 * pa_fft::pad_index(N - jb) + 1] = v[q].y;
        }
      }
    }
    if (!FWD && r == 0) line[1] = T(0);  // X[N] := 0 (slot 0)
  }
}

template <int LOGL, int C, bool FWD, class T>
__global__ void __launch_bounds__(FFT_THREADS) k_r2r(const __grid_constant__ R2rParams p) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const int t = threadIdx.x;
  const long long l0 = (long long)blockIdx.x * C;
  const int ncol = (int)((p.nlines - l0) < C ? (p.nlines - l0) : C);
  const int pitch = p.pitch;
  const bool sine = p.sine != 0;
  const V* twp = reinterpret_cast<const V*>(p.tw);
  const V* tw4p = reinterpret_cast<const V*>(p.tw4);

  // ---- load (linear gather, as k_rfft), reordered on its way into shared memory ----
  r2r_load<LOGL, C, FWD, T>(sm, pitch, ncol, t, sine, [&p, l0](int c) {
    return reinterpret_cast<const V*>(p.src + (l0 + c) * p.line);
  });
  __syncthreads();

  r2r_tail<LOGL, C, FWD, T>(sm, pitch, ncol, t, sine, twp, tw4p,
                            [&p, l0](int c) { return p.dst + (l0 + c) * p.line; });
}

// ---- fused unpack + real line transforms (pa_transpose_r2r / pa_transpose_rfft, DESIGN §3g) ----
// The blocks of a transposition of REAL arrays tile lines of N reals.  A CTA gathers C lines with
// gather_real_rows, placing every real where k_r2r's / k_rfft's load would, then runs their
// post-load stages (r2r_tail / rfft_forward_tail) on the shared-memory lines: the same
// fft_core.hpp calls in the same order on the same tables, so the output equals the unfused
// r2r_(transpose_(...)) / rfft_(transpose_(...)) bit for bit.  p.L = N / 2; p.tw = W_N.
// r2r: p.tw4 = W_4N, p.sine; dst / dsx / dso address the real destination.
// rfft: dst / dsx / dso address the COMPLEX destination of N/2 + 1 bins per line (fft_geometry
// converts them).  Same lines per CTA and pitch as k_r2r / k_rfft for that N.
template <int LOGL, int C, bool FWD, class T>
__global__ void __launch_bounds__(FFT_THREADS) k_unpack_r2r(const __grid_constant__ FftParams p) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int RS = FFT_THREADS / C;
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const int t = threadIdx.x;
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;
  const bool sine = p.sine != 0;

  // ---- gather: transposing, or linear (lines contiguous in the source) ----
  {
    const int c = p.linear ? t / RS : t % C, r = p.linear ? t % RS : t / C;
    T* line = reinterpret_cast<T*>(sm + c * pitch);
    gather_real_rows<C, T>(p, so_off, x0, c, r, ncol, [line, sine](int n, T x) {
      put_real<FWD ? RealMap::dct2 : RealMap::dct3, LOGL>(line, n, x, sine);
    });
    if (!FWD && r == 0 && c < ncol) line[1] = T(0);  // X[N] := 0 (slot 0)
  }
  __syncthreads();

  char* d = p.dst + x0 * p.dsx + d_off;
  r2r_tail<LOGL, C, FWD, T>(sm, pitch, ncol, t, sine, reinterpret_cast<const V*>(p.tw),
                            reinterpret_cast<const V*>(p.tw4),
                            [&p, d](int c) { return d + c * p.dsx; });
}

template <int LOGL, int C, class T>
__global__ void __launch_bounds__(FFT_THREADS) k_unpack_rfft(const __grid_constant__ FftParams p) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int RS = FFT_THREADS / C;
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const int t = threadIdx.x;
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;

  {
    const int c = p.linear ? t / RS : t % C, r = p.linear ? t % RS : t / C;
    T* line = reinterpret_cast<T*>(sm + c * pitch);
    gather_real_rows<C, T>(p, so_off, x0, c, r, ncol,
                           [line](int n, T x) { put_real<RealMap::rfft, LOGL>(line, n, x, false); });
  }
  __syncthreads();

  char* d = p.dst + x0 * p.dsx + d_off;
  rfft_forward_tail<LOGL, C, T>(sm, pitch, ncol, t, reinterpret_cast<const V*>(p.tw),
                                [&p, d](int c) { return d + c * p.dsx; });
}

// ---- send-side fused transform + put (pa_fft_put / pa_rfft_put, DESIGN §3i) ----
// The mirror of k_get_fft: the dim a PencilFFTs leg transforms first is the first memory dim of
// its src, local and contiguous.  A CTA loads C whole source lines with the linear load of fft_
// (k_rfft's for r2c), runs the same passes in shared memory, and stores every output bin straight
// into the block that owns it: the self block into the local dst, every other block into its
// peer's dst through the peer mapping.  So dst = transpose(fft_(src)) (transpose(rfft_(src))) byte
// for byte, with one read of src and one write of dst.
//   Window protocol (k_multi's, with the put flavour's wait for the peers' DONE): the first CTAs
// signal READY at the start, every CTA waits for READY from every peer only after its transform,
// before its first store -- the load and the passes never touch peer memory, so the wait hides
// behind them -- and the CTA that finishes last signals DONE and waits for the peers' DONE (only
// then has every peer's store into my dst landed).  Empty flag sets: the plain kernel
// (pa_put_all_fft / pa_put_all_rfft, or a launch that standalone flag kernels bracket).
struct FftPutBlock {
  char* dst;        // the block's origin in its destination array (dst, or a peer's as mapped here)
  int y0, ey;       // the bins [y0, y0 + ey) of every line that this block receives
  long long dsy;    // destination byte stride of a bin step
  long long dsx;    // destination byte stride of a column step (consecutive lines of a CTA)
  long long dso[FFT_MAXO];
};
struct FftPutParams {
  FftParams p;  // the load: ONE linear block, the whole source lines (p.dst / p.dsx / p.dso unused)
  int nb;
  int across;   // the columns have destination stride 1: C consecutive threads store one bin of
                // C consecutive lines (128 bytes); else consecutive threads walk along a line
  FftPutBlock blk[FFT_MAXB];
  MultiFlags mf;
};
static_assert(sizeof(FftPutParams) <= 4096, "FftPutParams must fit the kernel parameters");

__device__ __forceinline__ void put_ready_signal(const MultiFlags& mf) {
  if (mf.ready.n > 0 && blockIdx.x < 8 && (int)threadIdx.x < mf.ready.n)
    flag_signal(mf.ready.remote[threadIdx.x], mf.ready.seq[threadIdx.x]);
}
__device__ __forceinline__ void put_ready_wait(const MultiFlags& mf) {
  if (mf.ready.n > 0) {
    if ((int)threadIdx.x < mf.ready.n)
      flag_wait(mf.ready.local[threadIdx.x], mf.ready.seq[threadIdx.x], mf.timeout_ns, mf.err);
    __syncthreads();
  }
}
__device__ __forceinline__ void put_done(const MultiFlags& mf) {
  if (mf.done.n > 0) {
    // every store of this CTA has been issued; the last CTA to get here closes the window.  (No
    // static shared memory, as in k_get_fft)
    __syncthreads();
    int last = 0;
    if (threadIdx.x == 0) {
      __threadfence_system();
      last = atomicAdd(mf.counter, 1u) == gridDim.x - 1;
      if (last) {
        *mf.counter = 0;  // ready for the next launch (stream-ordered after this one)
        __threadfence_system();
      }
    }
    if (__syncthreads_or(last) && (int)threadIdx.x < mf.done.n) {
      flag_signal(mf.done.remote[threadIdx.x], mf.done.seq[threadIdx.x]);
      if (mf.wait_done) flag_wait(mf.done.local[threadIdx.x], mf.done.seq[threadIdx.x], mf.timeout_ns, mf.err);
    }
  }
}

// The destination of element k (a bin; k_r2r_put / k_brfft_put: a real) of the CTA's line c: the
// block that owns it, at its CTA origin `base` (every block is tried with a compile-time index, so
// `base` stays in registers)
template <class E>
__device__ __forceinline__ E* put_at(const FftPutParams& pp, char* const* base, int c, int k) {
  char* o = nullptr;
#pragma unroll
  for (int b = 0; b < FFT_MAXB; ++b)
    if (b < pp.nb && k >= pp.blk[b].y0 && k < pp.blk[b].y0 + pp.blk[b].ey)
      o = base[b] + (long long)(k - pp.blk[b].y0) * pp.blk[b].dsy + c * pp.blk[b].dsx;
  return reinterpret_cast<E*>(o);
}
template <class T>
__device__ __forceinline__ typename Vec2<T>::type* put_target(const FftPutParams& pp, char* const* base,
                                                              int c, int k) {
  return put_at<typename Vec2<T>::type>(pp, base, c, k);
}

// Every block's origin for this CTA's first line: its outer offsets (from the CTA index, as
// cta_offsets) and the first column x0
__device__ __forceinline__ void put_bases(const FftPutParams& pp, long long x0, char** base) {
  long long off[FFT_MAXB];
#pragma unroll
  for (int b = 0; b < FFT_MAXB; ++b) off[b] = 0;
  unsigned long long bid = blockIdx.x / pp.p.tiles_x;
#pragma unroll 1
  for (int i = 0; i < pp.p.no; ++i) {
    const long long k = (long long)(bid % (unsigned long long)pp.p.oe[i]);
    bid /= (unsigned long long)pp.p.oe[i];
#pragma unroll
    for (int b = 0; b < FFT_MAXB; ++b)
      if (b < pp.nb) off[b] += k * pp.blk[b].dso[i];
  }
#pragma unroll
  for (int b = 0; b < FFT_MAXB; ++b) base[b] = pp.blk[b].dst + off[b] + x0 * pp.blk[b].dsx;
}

// (a register cap as k_get_fft's)
template <int LOGL, int C, class T>
__global__ void __maxnreg__(128) k_fft_put(const __grid_constant__ FftPutParams pp) {
  using cx = cplx_t<T>;
  constexpr int L = 1 << LOGL;
  constexpr int LOGR1 = FftCtaShape<LOGL, C, T>::LOGR1;
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const FftParams& p = pp.p;
  const int t = threadIdx.x;
  put_ready_signal(pp.mf);
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  fft_cta_lines<LOGL, C, T>(p, so_off, x0, ncol, sm);
  put_ready_wait(pp.mf);

  // ---- store: bin k of line c into the block that owns k ----
  char* base[FFT_MAXB];
  put_bases(pp, x0, base);
  const bool across = pp.across != 0;
  for (int w0 = 0; w0 < C * L; w0 += FFT_THREADS) {
    const int w = w0 + t;
    const int c = across ? (w & (C - 1)) : (w >> LOGL), k = across ? (w / C) : (w & (L - 1));
    if (w < C * L && c < ncol) {
      const cx v = sm[c * p.pitch + pa_fft::pad_index(fft_out_pos<LOGL, LOGR1>(k))];
      __stcs(put_target<T>(pp, base, c, k), vec2(v.x, v.y));
    }
  }
  put_done(pp.mf);
}

// r2c: k_rfft's load (forward) and its passes, then rfft_post_pair on the pairs (k, L - k), the
// N/2 + 1 = L + 1 bins of a line stored into the blocks that own them.  p.L = N / 2, p.tw = W_N.
template <int LOGL, int C, class T>
__global__ void __maxnreg__(128) k_rfft_put(const __grid_constant__ FftPutParams pp) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const FftParams& p = pp.p;
  const int t = threadIdx.x;
  put_ready_signal(pp.mf);
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;
  rfft_load<LOGL, C, true, T>(sm, pitch, ncol, t, [&p, &so_off, x0](int c) {
    return reinterpret_cast<const V*>(p.blk[0].src + so_off[0] + (x0 + c) * p.blk[0].ssx);
  });
  __syncthreads();
  const V* twp = reinterpret_cast<const V*>(p.tw);
  auto twN = [twp](int k) {
    const V w = __ldg(twp + k);
    return cx{w.x, w.y};
  };
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const V w = __ldg(twp + 2 * i);
    return cx{w.x, w.y};
  };
  fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, -1, twL);
  put_ready_wait(pp.mf);

  // ---- post-pass + store: the pair k yields bins k and L - k ----
  char* base[FFT_MAXB];
  put_bases(pp, x0, base);
  const bool across = pp.across != 0;
  for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
    const int w = w0 + t;
    const int c = across ? (w & (C - 1)) : (w / P), k = across ? (w / C) : (w % P);
    if (w < C * P && c < ncol) {
      const cx* line = sm + c * pitch;
      cx xk, xl;
      pa_fft::rfft_post_pair(line[pa_fft::pad_index(fft_pos<LOGL, LOGL>(k & (L - 1)))],
                             line[pa_fft::pad_index(fft_pos<LOGL, LOGL>((L - k) & (L - 1)))], twN(k),
                             &xk, &xl);
      __stcs(put_target<T>(pp, base, c, k), vec2(xk.x, xk.y));
      if (k != L - k) __stcs(put_target<T>(pp, base, c, L - k), vec2(xl.x, xl.y));
    }
  }
  put_done(pp.mf);
}

// ---- send-side fused real line transforms + put (pa_r2r_put / pa_brfft_put, DESIGN §3j) ----
// The plan moves REAL elements: N reals per line, the blocks tiling [0, N) at any boundary (32
// reals over 3 ranks: 11 / 11 / 10), so every real is stored alone -- a pair (x[2m], x[2m+1]) may
// straddle two blocks, and a block that starts at an odd real is only element-aligned.  The
// across-lines pattern stores one real of C consecutive lines from C consecutive threads; the
// along-the-line pattern one real per thread, consecutive threads on consecutive reals.

// r2r: k_r2r's load (r2r_load), the DCT-III pre-pass (01 kinds), the L-point passes, then the
// DCT-II post-pass (10 kinds) or the read-out of the N reals, every real stored into the block
// that owns it.  p.L = N / 2, p.tw = W_N, p.tw4 = W_4N, p.sine.  Same lines per CTA and pitch as
// k_r2r for that N and direction.
template <int LOGL, int C, bool FWD, class T>
__global__ void __maxnreg__(128) k_r2r_put(const __grid_constant__ FftPutParams pp) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL, N = 2 * L;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const FftParams& p = pp.p;
  const int t = threadIdx.x;
  put_ready_signal(pp.mf);
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;
  const bool sine = p.sine != 0;
  const V* twp = reinterpret_cast<const V*>(p.tw);
  const V* tw4p = reinterpret_cast<const V*>(p.tw4);
  r2r_load<LOGL, C, FWD, T>(sm, pitch, ncol, t, sine, [&p, &so_off, x0](int c) {
    return reinterpret_cast<const V*>(p.blk[0].src + so_off[0] + (x0 + c) * p.blk[0].ssx);
  });
  __syncthreads();
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const V w = __ldg(twp + 2 * i);
    return cx{w.x, w.y};
  };
  if constexpr (!FWD) r2r_pre<LOGL, C, T>(sm, pitch, ncol, t, twp, tw4p);
  fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, FWD ? -1 : 1, twL);
  put_ready_wait(pp.mf);

  char* base[FFT_MAXB];
  put_bases(pp, x0, base);
  const bool across = pp.across != 0;
  if constexpr (FWD) {
    // ---- post-pass + store: the pair k yields Y[k], Y[N-k], Y[L-k] and Y[L+k] (r2r_tail's);
    //      DST-II stores Y[j] at N-1-j ----
    auto twN = [twp](int k) {
      const V w = __ldg(twp + k);
      return cx{w.x, w.y};
    };
    auto w4 = [tw4p](int k) {  // w_k = W_4N^k
      const V w = __ldg(tw4p + k);
      return cx{w.x, w.y};
    };
    for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
      const int w = w0 + t;
      const int c = across ? (w & (C - 1)) : (w / P), k = across ? (w / C) : (w % P);
      if (w < C * P && c < ncol) {
        const cx* line = sm + c * pitch;
        cx vk, vl;
        pa_fft::rfft_post_pair(line[pa_fft::pad_index(fft_pos<LOGL, LOGL>(k & (L - 1)))],
                               line[pa_fft::pad_index(fft_pos<LOGL, LOGL>((L - k) & (L - 1)))], twN(k),
                               &vk, &vl);
        T yk, ynk, yl, ynl;
        pa_fft::dct2_post_pair(vk, w4(k), &yk, &ynk);      // Y[k], Y[N-k]
        pa_fft::dct2_post_pair(vl, w4(L - k), &yl, &ynl);  // Y[L-k], Y[L+k]
        auto put = [&](int j, T y) { __stcs(put_at<T>(pp, base, c, sine ? N - 1 - j : j), y); };
        put(k, yk);
        if (k > 0 && k < L / 2) put(N - k, ynk);
        if (k < L / 2) put(L - k, yl);
        if (k > 0) put(L + k, ynl);
      }
    }
  } else {
    // ---- store: x[2m] = v[m], x[2m+1] = v[N-1-m]; DST-III: times (-1)^n ----
    for (int w0 = 0; w0 < C * N; w0 += FFT_THREADS) {
      const int w = w0 + t;
      const int c = across ? (w & (C - 1)) : (w >> (LOGL + 1)), n = across ? (w / C) : (w & (N - 1));
      if (w < C * N && c < ncol) {
        const T* line = reinterpret_cast<const T*>(sm + c * pitch);
        const int i = (n & 1) ? N - 1 - (n >> 1) : (n >> 1);
        const T v = line[2 * pa_fft::pad_index(fft_pos<LOGL, LOGL>(i >> 1)) + (i & 1)];
        __stcs(put_at<T>(pp, base, c, n), (sine && (n & 1)) ? -v : v);
      }
    }
  }
  put_done(pp.mf);
}

// c2r: k_rfft's backward load (rfft_load, the N/2 + 1 bins), its pre-pass and its L-point passes,
// then the N reals z[n] = x[2n] + i x[2n+1] of a line stored into the blocks that own them.  The
// source is the complex counterpart of the plan's real one; p.L = N / 2, p.tw = W_N.
template <int LOGL, int C, class T>
__global__ void __maxnreg__(128) k_brfft_put(const __grid_constant__ FftPutParams pp) {
  using cx = cplx_t<T>;
  using V = typename Vec2<T>::type;
  constexpr int L = 1 << LOGL, N = 2 * L;
  constexpr int P = L / 2 + 1;  // pairs (k, L - k) per line
  extern __shared__ __align__(16) unsigned char fft_smem[];
  cx* sm = reinterpret_cast<cx*>(fft_smem);
  const FftParams& p = pp.p;
  const int t = threadIdx.x;
  put_ready_signal(pp.mf);
  long long so_off[FFT_MAXB], d_off;
  const long long x0 = cta_offsets(p, C, so_off, &d_off);
  const int ncol = (int)((p.ex - x0) < C ? (p.ex - x0) : C);
  const int pitch = p.pitch;
  rfft_load<LOGL, C, false, T>(sm, pitch, ncol, t, [&p, &so_off, x0](int c) {
    return reinterpret_cast<const V*>(p.blk[0].src + so_off[0] + (x0 + c) * p.blk[0].ssx);
  });
  __syncthreads();
  const V* twp = reinterpret_cast<const V*>(p.tw);
  auto twN = [twp](int k) {
    const V w = __ldg(twp + k);
    return cx{w.x, w.y};
  };
  auto twL = [twp](int i) {  // W_L^i = W_N^(2i)
    const V w = __ldg(twp + 2 * i);
    return cx{w.x, w.y};
  };
  // ---- pre-pass in place (k_rfft<..., false>): a thread owns the slots k and L - k ----
#pragma unroll
  for (int w0 = 0; w0 < C * P; w0 += FFT_THREADS) {
    const int w = w0 + t, c = w / P, k = w % P;
    if (w < C * P && c < ncol) {
      cx* line = sm + c * pitch;
      cx zk, zl;
      pa_fft::brfft_pre_pair(k, line[pa_fft::pad_index(k)], line[pa_fft::pad_index(L - k)], twN(k),
                             &zk, &zl);
      line[pa_fft::pad_index(k)] = zk;
      if (k > 0) line[pa_fft::pad_index(L - k)] = zl;
    }
  }
  __syncthreads();
  fft_passes<LOGL, LOGL, C>(sm, pitch, ncol, 1, twL);
  put_ready_wait(pp.mf);

  // ---- store: real n of line c is part n & 1 of complex slot n / 2 ----
  char* base[FFT_MAXB];
  put_bases(pp, x0, base);
  const bool across = pp.across != 0;
  for (int w0 = 0; w0 < C * N; w0 += FFT_THREADS) {
    const int w = w0 + t;
    const int c = across ? (w & (C - 1)) : (w >> (LOGL + 1)), n = across ? (w / C) : (w & (N - 1));
    if (w < C * N && c < ncol) {
      const T* line = reinterpret_cast<const T*>(sm + c * pitch);
      __stcs(put_at<T>(pp, base, c, n), line[2 * pa_fft::pad_index(fft_pos<LOGL, LOGL>(n >> 1)) + (n & 1)]);
    }
  }
  put_done(pp.mf);
}

// forward twiddle table W_L^k per (device, L, precision), computed once in extended precision
// and rounded once to double (cplx) or float (cplxf)
template <class T>
static std::vector<cplx_t<T>> twiddle_values(int L) {
  std::vector<cplx_t<T>> h(L);
  for (int k = 0; k < L; ++k) {
    const long double a = -2.0L * 3.141592653589793238462643383279502884L * k / L;
    h[k] = cplx_t<T>{(T)cosl(a), (T)sinl(a)};
  }
  return h;
}

static const void* twiddles(int L, bool f32) {
  static std::mutex mu;
  static std::map<std::tuple<int, int, bool>, void*> cache;
  std::lock_guard<std::mutex> lock(mu);
  int dev = 0;
  cudaGetDevice(&dev);
  auto key = std::make_tuple(dev, L, f32);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  auto upload = [&](const void* h, size_t bytes) -> void* {
    void* d = nullptr;
    if (cudaMalloc(&d, bytes) != cudaSuccess) return nullptr;
    if (cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
    return d;
  };
  void* d = nullptr;
  if (f32) {
    const auto h = twiddle_values<float>(L);
    d = upload(h.data(), sizeof(h[0]) * L);
  } else {
    const auto h = twiddle_values<double>(L);
    d = upload(h.data(), sizeof(h[0]) * L);
  }
  if (d) cache[key] = d;
  return d;
}

// Launch geometry of the fused kernel from the blocks of one rank (`blocks[i]` moves block i
// from `srcs[i]` -- recv_buf, or the src parent for the fused self block -- into `dst`;
// together they must tile the destination box), and every check of it.  srcs / dst may be
// NULL: plan_fft_check runs this on the blocks a peer would see, without arrays.  *grid = 0:
// nothing to do on this rank.  f32: ComplexF32 elements (PA_FFT_F32), else ComplexF64.
// brfft (k_unpack_brfft): the lines are M = N/2 + 1 bins, and `dst` is the REAL array of N
// reals per line in place of the complex one the blocks describe (DESIGN §3e).
// r2r / rfft (k_unpack_r2r / k_unpack_rfft): the elements are reals (Float64, or Float32 with
// f32) and the lines N reals; rfft: `dst` is the COMPLEX array of N/2 + 1 bins per line in place
// of the real one the blocks describe (DESIGN §3g).
static pa_status fft_geometry(int nb, const BlockCopy* const* blocks, const void* const* srcs,
                              void* dst, bool f32, FusedMode mode, FftParams& p, int* C_out,
                              unsigned long long* grid_out) {
  const bool brfft = mode == FusedMode::brfft;
  const bool real = mode == FusedMode::r2r || mode == FusedMode::rfft;  // real source elements
  const i64 es = real ? (f32 ? 4 : 8) : (f32 ? 8 : 16);  // element bytes
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
    if (B.elsize != es) {
      if (real)
        set_error(f32 ? "fused real transform: PA_FFT_F32 takes Float32 (4-byte) elements only"
                      : "fused real transform: Float64 (8-byte) elements only");
      else
        set_error(f32 ? "fused FFT: PA_FFT_F32 takes ComplexF32 (8-byte) elements only"
                      : "fused FFT: ComplexF64 (16-byte) elements only");
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
    F.src = srcs ? (const char*)srcs[b] + B.src_off * es : nullptr;
    F.y0 = (int)(B.dst_off - min_doff);
    F.ey = (int)B.raw[jy].e;
    F.ssy = B.raw[jy].ss * es;
    F.ssx = jx >= 0 ? B.raw[jx].ss * es : es;
    int o = 0;
    for (int i = 1; i < B.nd_raw; ++i)
      if (i != jy && i != jx && B.raw[i].e > 1) F.so[o++] = B.raw[i].ss * es;
    L += B.raw[jy].e;
  }
  const i64 M = L;  // rows per line (brfft: bins; r2r / rfft: reals)
  if (brfft) L = M - 1;  // the N/2-point complex FFT of a real line of N = 2 (M - 1)
  if (real) L = M / 2;   // the N/2-point complex FFT of a real line of N = M
  int logL = 0;
  while ((1LL << logL) < L) ++logL;
  if ((1LL << logL) != L || L < 8 || L > 1024 || (real && 2 * L != M)) {
    if (brfft)
      set_error("fused brfft: %lld bins per line are not N/2+1 with N a power of two in 16..2048",
                (long long)M);
    else if (real)
      set_error("fused real transform: line length N = %lld is not a power of two in 16..2048",
                (long long)M);
    else
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
  p.dst = dst ? (char*)dst + min_doff * es : nullptr;
  p.linear = linear ? 1 : 0;
  p.ex = jx >= 0 ? ref->raw[jx].e : 1;
  p.dsx = jx >= 0 ? ref->raw[jx].ds * es : es;
  p.no = 0;
  for (int i = 1; i < ref->nd_raw; ++i)
    if (i != jy && i != jx && ref->raw[i].e > 1) {
      if (p.no >= FFT_MAXO) {
        set_error("fused FFT: more than %d outer dims", FFT_MAXO);
        return PA_EINVAL;
      }
      p.oe[p.no] = ref->raw[i].e;
      p.dso[p.no] = ref->raw[i].ds * es;
      ++p.no;
    }
  p.L = (int)L;
  p.logL = logL;
  p.pitch = real ? 0 : pa_fft::padded_pitch((int)M);  // r2r / rfft: the launcher's, by direction
  if (brfft) {
    // The line dim is the destination's first memory dim (stride 1) and whole (the blocks tile
    // [0, M)), so every other destination offset and stride is a multiple of M elements: line k
    // of the complex array starts at k M complex elements, and at k N reals in the real array
    // of the same shape otherwise.  Only dims of extent > 1 are addressed.
    const i64 N = 2 * L, rs = es / 2;
    auto to_real = [&](long long off, long long* out) {
      if (off % M != 0) {
        set_error("fused brfft: a destination stride or offset is not a multiple of the %lld bins "
                  "of a line", (long long)M);
        return false;
      }
      *out = off / M * N * rs;
      return true;
    };
    long long v = 0;
    if (!to_real(min_doff, &v)) return PA_EINVAL;
    p.dst = dst ? (char*)dst + v : nullptr;
    p.dsx = N * rs;
    if (jx >= 0 && p.ex > 1 && !to_real(ref->raw[jx].ds, &p.dsx)) return PA_EINVAL;
    for (int o = 0; o < p.no; ++o)
      if (!to_real(p.dso[o] / es, &p.dso[o])) return PA_EINVAL;
  }
  if (mode == FusedMode::rfft) {
    // brfft's rescale the other way round: line k of the real array starts at k N reals, and at
    // k M complex bins in the complex array of the same shape otherwise
    const i64 N = M, Mc = L + 1, cs = 2 * es;
    auto to_cplx = [&](long long off, long long* out) {
      if (off % N != 0) {
        set_error("fused rfft: a destination stride or offset is not a multiple of the %lld reals "
                  "of a line", (long long)N);
        return false;
      }
      *out = off / N * Mc * cs;
      return true;
    };
    long long v = 0;
    if (!to_cplx(min_doff, &v)) return PA_EINVAL;
    p.dst = dst ? (char*)dst + v : nullptr;
    p.dsx = Mc * cs;
    if (jx >= 0 && p.ex > 1 && !to_cplx(ref->raw[jx].ds, &p.dsx)) return PA_EINVAL;
    for (int o = 0; o < p.no; ++o)
      if (!to_cplx(p.dso[o] / es, &p.dso[o])) return PA_EINVAL;
  }
  // tunable "fft_lines" = 4: 4 lines per CTA also for 256- / 512-point lines (64-byte gathers,
  // first pass of radix 4 / 8 in registers, half the shared memory per CTA); double precision
  // only -- single precision always takes fft_lines_f32.  brfft, r2r, rfft: the lines per CTA of
  // k_rfft
  const int C = f32 ? fft_lines_f32(logL)
                    : ((mode == FusedMode::fft && g_tun.fft_lines == 4 && logL >= 8) ? 4 : fft_lines(logL));
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
                     int sign, bool f32, void* stream) {
  // (pa_transpose has already asked plan_fft_check, for every rank of the line, before it
  //  enqueued anything: these checks only guard direct callers)
  FftParams p;
  int C = 0;
  unsigned long long grid = 0;
  pa_status s = fft_geometry(nb, blocks, srcs, dst, f32, FusedMode::fft, p, &C, &grid);
  if (s != PA_OK || grid == 0) return s;
  const int logL = p.logL;
  p.sign = sign < 0 ? -1 : 1;
  p.tw = twiddles(p.L, f32);
  if (!p.tw) {
    set_error("fused FFT: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const size_t smem = (f32 ? sizeof(pa_fft::cplxf) : sizeof(cplx)) * (size_t)C * p.pitch;
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
  if (f32) {
    switch (logL) {
      case 3: launch(k_unpack_fft<3, 16, float>); break;
      case 4: launch(k_unpack_fft<4, 16, float>); break;
      case 5: launch(k_unpack_fft<5, 16, float>); break;
      case 6: launch(k_unpack_fft<6, 16, float>); break;
      case 7: launch(k_unpack_fft<7, 16, float>); break;
      case 8: launch(k_unpack_fft<8, 16, float>); break;
      case 9: launch(k_unpack_fft<9, 16, float>); break;
      default: launch(k_unpack_fft<10, 8, float>); break;
    }
  } else {
    switch (logL) {
      case 3: launch(k_unpack_fft<3, 8, double>); break;
      case 4: launch(k_unpack_fft<4, 8, double>); break;
      case 5: launch(k_unpack_fft<5, 8, double>); break;
      case 6: launch(k_unpack_fft<6, 8, double>); break;
      case 7: launch(k_unpack_fft<7, 8, double>); break;
      case 8: if (C == 4) launch(k_unpack_fft<8, 4, double>); else launch(k_unpack_fft<8, 8, double>); break;
      case 9: if (C == 4) launch(k_unpack_fft<9, 4, double>); else launch(k_unpack_fft<9, 8, double>); break;
      default: launch(k_unpack_fft<10, 4, double>); break;
    }
  }
  if (e != cudaSuccess) {
    set_error("fused FFT kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

pa_status get_fft(int nb, const BlockCopy* const* blocks, const void* const* srcs, void* dst, int sign,
                  bool f32, const MultiFlags* mf, void* stream, bool* launched) {
  // (pa_transpose and pa_get_all_fft have already asked plan_fft_check)
  *launched = false;
  FftGetParams gp;
  int C = 0;
  unsigned long long grid = 0;
  pa_status s = fft_geometry(nb, blocks, srcs, dst, f32, FusedMode::fft, gp.p, &C, &grid);
  if (s != PA_OK || grid == 0) return s;
  FftParams& p = gp.p;
  memset(&gp.mf, 0, sizeof gp.mf);
  if (mf) gp.mf = *mf;
  const int logL = p.logL;
  p.sign = sign < 0 ? -1 : 1;
  p.tw = twiddles(p.L, f32);
  if (!p.tw) {
    set_error("fused FFT: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const size_t smem = (f32 ? sizeof(pa_fft::cplxf) : sizeof(cplx)) * (size_t)C * p.pitch;
  cudaError_t e = cudaSuccess;
  auto launch = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    cudaGetLastError();
    kern<<<(unsigned)grid, FFT_THREADS, smem, (cudaStream_t)stream>>>(gp);
    e = cudaGetLastError();
  };
  if (f32) {
    switch (logL) {
      case 3: launch(k_get_fft<3, 16, float>); break;
      case 4: launch(k_get_fft<4, 16, float>); break;
      case 5: launch(k_get_fft<5, 16, float>); break;
      case 6: launch(k_get_fft<6, 16, float>); break;
      case 7: launch(k_get_fft<7, 16, float>); break;
      case 8: launch(k_get_fft<8, 16, float>); break;
      case 9: launch(k_get_fft<9, 16, float>); break;
      default: launch(k_get_fft<10, 8, float>); break;
    }
  } else {
    switch (logL) {
      case 3: launch(k_get_fft<3, 8, double>); break;
      case 4: launch(k_get_fft<4, 8, double>); break;
      case 5: launch(k_get_fft<5, 8, double>); break;
      case 6: launch(k_get_fft<6, 8, double>); break;
      case 7: launch(k_get_fft<7, 8, double>); break;
      case 8: if (C == 4) launch(k_get_fft<8, 4, double>); else launch(k_get_fft<8, 8, double>); break;
      case 9: if (C == 4) launch(k_get_fft<9, 4, double>); else launch(k_get_fft<9, 8, double>); break;
      default: launch(k_get_fft<10, 4, double>); break;
    }
  }
  if (e != cudaSuccess) {
    set_error("one-sided fused FFT kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  *launched = true;
  return PA_OK;
}

// Launch geometry of k_fft_put / k_rfft_put from the blocks of one rank -- the mirror of
// fft_geometry on the source side.  `blocks[i]` moves a box of the local `src` into `dsts[i]`
// (the local dst for the self block, a peer's dst as mapped here otherwise); together they must
// tile the source lines.  The line dim is the source dim of stride 1 (raw dim 0); the blocks
// must tile [0, M) along it (M = L points; rfft: M = N/2 + 1 bins) and share every other dim,
// whose destination strides may differ (the peers' arrays have their own layouts).  The column
// dim is the destination's stride-1 dim when that is not the line dim.  src / dsts may be NULL:
// plan_fft_put_check runs this without arrays.  *grid = 0: this rank has no source lines.
// rfft: the plan is the COMPLEX plan of M bins per line, and `src` the REAL array of N reals per
// line that replaces its source (same layout otherwise): the source offsets and strides, multiples
// of M, are rescaled to N reals -- brfft's destination rescale, mirrored.
// r2r / brfft: the plan is the REAL plan of M = N reals per line (the blocks may split it at any
// real).  r2r: `src` is its source.  brfft: `src` is the COMPLEX array of N/2 + 1 bins per line
// that replaces it, the source offsets and strides rescaled from N reals to N/2 + 1 bins.  Both
// require those offsets and strides to be multiples of N, so one verdict serves both.
static pa_status put_fft_geometry(int nb, const BlockCopy* const* blocks, const void* src,
                                  void* const* dsts, bool f32, PutMode mode, FftPutParams& pp, int* C_out,
                                  unsigned long long* grid_out) {
  const bool rfft = mode == PutMode::rfft;
  const bool real = mode == PutMode::r2r || mode == PutMode::brfft;  // the plan moves reals
  const char* what = real ? "fused real transform + put" : rfft ? "fused rfft + put" : "fused FFT + put";
  const i64 es = real ? (f32 ? 4 : 8) : (f32 ? 8 : 16);  // the plan's element bytes
  memset(&pp, 0, sizeof pp);
  *grid_out = 0;
  const BlockCopy* ref = nullptr;
  i64 min_soff = -1;
  for (int b = 0; b < nb; ++b) {
    const BlockCopy& B = *blocks[b];
    if (B.count == 0) continue;
    if (B.elsize != es) {
      if (real)
        set_error(f32 ? "%s: PA_FFT_F32 takes Float32 (4-byte) elements only"
                      : "%s: Float64 (8-byte) elements only", what);
      else
        set_error(f32 ? "%s: PA_FFT_F32 takes ComplexF32 (8-byte) elements only"
                      : "%s: ComplexF64 (16-byte) elements only", what);
      return PA_EINVAL;
    }
    if (B.raw[0].ss != 1) {
      set_error("%s: unexpected source layout", what);
      return PA_EINVAL;
    }
    if (!ref) ref = &B;
    if (B.nd_raw != ref->nd_raw) {
      set_error("%s: the blocks do not share their line set", what);
      return PA_EINVAL;
    }
    for (int i = 1; i < B.nd_raw; ++i)
      if (B.raw[i].e != ref->raw[i].e || B.raw[i].ss != ref->raw[i].ss) {
        set_error("%s: the blocks do not share their line set", what);
        return PA_EINVAL;
      }
    if (min_soff < 0 || B.src_off < min_soff) min_soff = B.src_off;
  }
  if (!ref) return PA_OK;  // no source lines on this rank (*grid = 0)
  i64 M = 0;
  for (int b = 0; b < nb; ++b) {
    const BlockCopy& B = *blocks[b];
    if (B.count == 0) continue;
    if (pp.nb >= FFT_MAXB) {
      set_error("%s: more than %d blocks", what, FFT_MAXB);
      return PA_EINVAL;
    }
    FftPutBlock& F = pp.blk[pp.nb++];
    F.dst = dsts && dsts[b] ? (char*)dsts[b] + B.dst_off * es : nullptr;
    F.y0 = (int)(B.src_off - min_soff);
    F.ey = (int)B.raw[0].e;
    F.dsy = B.raw[0].ds * es;
    M += B.raw[0].e;
  }
  // rfft: the N/2-point complex FFT of a real line of N = 2 (M - 1); r2r / brfft: of N = M reals
  const i64 L = rfft ? M - 1 : real ? M / 2 : M;
  int logL = 0;
  while ((1LL << logL) < L) ++logL;
  if ((1LL << logL) != L || L < 8 || L > 1024 || (real && 2 * L != M)) {
    if (rfft)
      set_error("%s: %lld bins per line are not N/2+1 with N a power of two in 16..2048", what,
                (long long)M);
    else if (real)
      set_error("%s: line length N = %lld is not a power of two in 16..2048", what, (long long)M);
    else
      set_error("%s: line length %lld is not a power of two in 8..1024", what, (long long)L);
    return PA_EINVAL;
  }
  {
    std::vector<std::pair<int, int>> seg;
    for (int b = 0; b < pp.nb; ++b) seg.push_back({pp.blk[b].y0, pp.blk[b].ey});
    std::sort(seg.begin(), seg.end());
    int pos = 0;
    for (auto& s : seg) {
      if (s.first != pos) {
        set_error("%s: the blocks do not tile the transform axis", what);
        return PA_EINVAL;
      }
      pos += s.second;
    }
  }
  // the column dim: the destination's stride-1 dim (in every block) when the line dim is not it;
  // otherwise (or when no such dim is longer than 1) the next dim longer than 1
  int jx = -1;
  bool across = false;
  if (ref->raw[0].ds != 1)
    for (int i = 1; i < ref->nd_raw && jx < 0; ++i) {
      if (ref->raw[i].e <= 1) continue;
      bool unit = true;
      for (int b = 0; b < nb; ++b)
        if (blocks[b]->count > 0) unit = unit && blocks[b]->raw[i].ds == 1;
      if (unit) jx = i, across = true;
    }
  for (int i = 1; i < ref->nd_raw && jx < 0; ++i)
    if (ref->raw[i].e > 1) jx = i;
  // source offsets and strides: complex elements, or (rfft) multiples of M bins that become
  // multiples of N reals, or (r2r / brfft) multiples of N reals that stay reals (r2r) or become
  // multiples of N/2 + 1 bins (brfft)
  const i64 N = 2 * L, rs = real ? es : es / 2, Mc = L + 1;
  auto src_bytes = [&](long long off, long long* out) {
    if (!rfft && !real) {
      *out = off * es;
      return true;
    }
    if (off % M != 0) {
      if (rfft)
        set_error("%s: a source stride or offset is not a multiple of the %lld bins of a line", what,
                  (long long)M);
      else
        set_error("%s: a source stride or offset is not a multiple of the %lld reals of a line", what,
                  (long long)M);
      return false;
    }
    *out = rfft ? off / M * N * rs : mode == PutMode::brfft ? off / M * Mc * 2 * rs : off * rs;
    return true;
  };
  FftParams& p = pp.p;
  FftBlock& S = p.blk[0];
  p.nb = 1;
  long long v = 0;
  if (!src_bytes(min_soff, &v)) return PA_EINVAL;
  S.src = src ? (const char*)src + v : nullptr;
  S.y0 = 0;
  S.ey = (int)L;
  S.ssy = (rfft || real) ? 2 * rs : es;
  S.ssx = mode == PutMode::brfft ? Mc * 2 * rs : (rfft || real) ? N * rs : L * es;
  if (jx >= 0 && !src_bytes(ref->raw[jx].ss, &S.ssx)) return PA_EINVAL;
  for (int i = 1; i < ref->nd_raw; ++i)
    if (i != jx && ref->raw[i].e > 1) {
      if (p.no >= FFT_MAXO) {
        set_error("%s: more than %d outer dims", what, FFT_MAXO);
        return PA_EINVAL;
      }
      if (!src_bytes(ref->raw[i].ss, &S.so[p.no])) return PA_EINVAL;
      p.oe[p.no] = ref->raw[i].e;
      int o = 0;
      for (int b = 0; b < nb; ++b)
        if (blocks[b]->count > 0) pp.blk[o++].dso[p.no] = blocks[b]->raw[i].ds * es;
      ++p.no;
    }
  {
    int o = 0;
    for (int b = 0; b < nb; ++b)
      if (blocks[b]->count > 0) pp.blk[o++].dsx = jx >= 0 ? blocks[b]->raw[jx].ds * es : 0;
  }
  pp.across = across ? 1 : 0;
  p.linear = 1;
  p.ex = jx >= 0 ? ref->raw[jx].e : 1;
  p.L = (int)L;
  p.logL = logL;
  // fft_ / k_rfft (forward) / k_r2r (10 kinds): L points per shared line; k_rfft (backward) and
  // k_r2r (01 kinds) stage the L + 1 slots, which put_fft sets
  p.pitch = pa_fft::padded_pitch((int)L);
  // the lines per CTA of fft_ (tunable fft_lines included) / of k_rfft and k_r2r
  const int C = f32 ? fft_lines_f32(logL)
                    : ((mode == PutMode::fft && g_tun.fft_lines == 4 && logL >= 8) ? 4 : fft_lines(logL));
  p.tiles_x = (unsigned)((p.ex + C - 1) / C);
  unsigned long long grid = p.tiles_x;
  for (int i = 0; i < p.no; ++i) grid *= (unsigned long long)p.oe[i];
  if (grid > 0x7fffffffULL) {
    set_error("%s: too many lines for one launch", what);
    return PA_EINVAL;
  }
  *C_out = C;
  *grid_out = grid;
  return PA_OK;
}

pa_status put_fft(int nb, const BlockCopy* const* blocks, const void* src, void* const* dsts, int sign,
                  PutMode mode, int r2r_kind, bool f32, const MultiFlags* mf, void* stream, bool* launched) {
  // (the entry points have already asked plan_fft_put_check / plan_rfft_put_check /
  //  plan_real_put_check)
  *launched = false;
  FftPutParams pp;
  int C = 0;
  unsigned long long grid = 0;
  pa_status s = put_fft_geometry(nb, blocks, src, dsts, f32, mode, pp, &C, &grid);
  if (s != PA_OK || grid == 0) return s;
  if (mf) pp.mf = *mf;
  FftParams& p = pp.p;
  const int logL = p.logL;
  const bool rfft = mode == PutMode::rfft;
  // r2r: the 10 kinds run k_r2r's forward path, the 01 kinds its backward one
  const bool r2r_fwd = r2r_kind == PA_REDFT10 || r2r_kind == PA_RODFT10;
  p.sign = rfft ? -1 : (sign < 0 ? -1 : 1);
  p.tw = twiddles(mode == PutMode::fft ? p.L : 2 * p.L, f32);
  if (mode == PutMode::r2r) {
    p.sine = (r2r_kind == PA_RODFT10 || r2r_kind == PA_RODFT01) ? 1 : 0;
    p.tw4 = twiddles(8 * p.L, f32);
  }
  // k_rfft (backward) and k_r2r (01 kinds) stage the pairs of slots 0..L
  if (mode == PutMode::brfft || (mode == PutMode::r2r && !r2r_fwd)) p.pitch = pa_fft::padded_pitch(p.L + 1);
  if (!p.tw || (mode == PutMode::r2r && !p.tw4)) {
    set_error("fused put: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const size_t smem = (f32 ? sizeof(pa_fft::cplxf) : sizeof(cplx)) * (size_t)C * p.pitch;
  cudaError_t e = cudaSuccess;
  auto launch = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    cudaGetLastError();
    kern<<<(unsigned)grid, FFT_THREADS, smem, (cudaStream_t)stream>>>(pp);
    e = cudaGetLastError();
  };
  // the kernels of one line length and lines per CTA, by mode (and r2r direction)
#define PUT_KERNELS(LG, CC, T)                                                                   \
  switch (mode) {                                                                                \
    case PutMode::fft: launch(k_fft_put<LG, CC, T>); break;                                      \
    case PutMode::rfft: launch(k_rfft_put<LG, CC, T>); break;                                    \
    case PutMode::r2r:                                                                           \
      r2r_fwd ? launch(k_r2r_put<LG, CC, true, T>) : launch(k_r2r_put<LG, CC, false, T>);        \
      break;                                                                                     \
    case PutMode::brfft: launch(k_brfft_put<LG, CC, T>); break;                                  \
  }
  if (f32) {
    switch (logL) {
      case 3: PUT_KERNELS(3, 16, float) break;
      case 4: PUT_KERNELS(4, 16, float) break;
      case 5: PUT_KERNELS(5, 16, float) break;
      case 6: PUT_KERNELS(6, 16, float) break;
      case 7: PUT_KERNELS(7, 16, float) break;
      case 8: PUT_KERNELS(8, 16, float) break;
      case 9: PUT_KERNELS(9, 16, float) break;
      default: PUT_KERNELS(10, 8, float) break;
    }
  } else {
    switch (logL) {
      case 3: PUT_KERNELS(3, 8, double) break;
      case 4: PUT_KERNELS(4, 8, double) break;
      case 5: PUT_KERNELS(5, 8, double) break;
      case 6: PUT_KERNELS(6, 8, double) break;
      case 7: PUT_KERNELS(7, 8, double) break;
      case 8:
        if (C == 4) launch(k_fft_put<8, 4, double>);  // (tunable fft_lines = 4: the complex FFT only)
        else PUT_KERNELS(8, 8, double)
        break;
      case 9:
        if (C == 4) launch(k_fft_put<9, 4, double>);
        else PUT_KERNELS(9, 8, double)
        break;
      default: PUT_KERNELS(10, 4, double) break;
    }
  }
#undef PUT_KERNELS
  if (e != cudaSuccess) {
    set_error("fused put kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  *launched = true;
  return PA_OK;
}

pa_status unpack_brfft(int nb, const BlockCopy* const* blocks, const void* const* srcs, void* dst,
                       bool f32, void* stream) {
  // (pa_transpose_brfft has already asked plan_brfft_check for every rank of the line)
  FftParams p;
  int C = 0;
  unsigned long long grid = 0;
  pa_status s = fft_geometry(nb, blocks, srcs, dst, f32, FusedMode::brfft, p, &C, &grid);
  if (s != PA_OK || grid == 0) return s;
  const int logL = p.logL;
  p.sign = 1;
  p.tw = twiddles(2 * p.L, f32);
  if (!p.tw) {
    set_error("fused brfft: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const size_t smem = (f32 ? sizeof(pa_fft::cplxf) : sizeof(cplx)) * (size_t)C * p.pitch;
  cudaError_t e = cudaSuccess;
  auto launch = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    cudaGetLastError();
    kern<<<(unsigned)grid, FFT_THREADS, smem, (cudaStream_t)stream>>>(p);
    e = cudaGetLastError();
  };
  if (f32) {
    switch (logL) {
      case 3: launch(k_unpack_brfft<3, 16, float>); break;
      case 4: launch(k_unpack_brfft<4, 16, float>); break;
      case 5: launch(k_unpack_brfft<5, 16, float>); break;
      case 6: launch(k_unpack_brfft<6, 16, float>); break;
      case 7: launch(k_unpack_brfft<7, 16, float>); break;
      case 8: launch(k_unpack_brfft<8, 16, float>); break;
      case 9: launch(k_unpack_brfft<9, 16, float>); break;
      default: launch(k_unpack_brfft<10, 8, float>); break;
    }
  } else {
    switch (logL) {
      case 3: launch(k_unpack_brfft<3, 8, double>); break;
      case 4: launch(k_unpack_brfft<4, 8, double>); break;
      case 5: launch(k_unpack_brfft<5, 8, double>); break;
      case 6: launch(k_unpack_brfft<6, 8, double>); break;
      case 7: launch(k_unpack_brfft<7, 8, double>); break;
      case 8: launch(k_unpack_brfft<8, 8, double>); break;
      case 9: launch(k_unpack_brfft<9, 8, double>); break;
      default: launch(k_unpack_brfft<10, 4, double>); break;
    }
  }
  if (e != cudaSuccess) {
    set_error("fused brfft kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

// kind: FFTW's REDFT10 (DCT-II), REDFT01 (DCT-III), RODFT10 (DST-II) or RODFT01 (DST-III)
pa_status unpack_r2r(int nb, const BlockCopy* const* blocks, const void* const* srcs, void* dst,
                     int kind, bool f32, void* stream) {
  // (pa_transpose_r2r has already asked plan_real_check for every rank of the line)
  const bool forward = kind == PA_REDFT10 || kind == PA_RODFT10;
  FftParams p;
  int C = 0;
  unsigned long long grid = 0;
  pa_status s = fft_geometry(nb, blocks, srcs, dst, f32, FusedMode::r2r, p, &C, &grid);
  if (s != PA_OK || grid == 0) return s;
  const int logL = p.logL, N = 2 * p.L;
  p.pitch = pa_fft::padded_pitch(forward ? p.L : p.L + 1);  // as r2r_lines
  p.sine = (kind == PA_RODFT10 || kind == PA_RODFT01) ? 1 : 0;
  p.tw = twiddles(N, f32);
  p.tw4 = twiddles(4 * N, f32);
  if (!p.tw || !p.tw4) {
    set_error("fused r2r: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const size_t smem = (f32 ? sizeof(pa_fft::cplxf) : sizeof(cplx)) * (size_t)C * p.pitch;
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
  if (f32) {
    switch (logL) {
      case 3: launch_dir(k_unpack_r2r<3, 16, true, float>, k_unpack_r2r<3, 16, false, float>); break;
      case 4: launch_dir(k_unpack_r2r<4, 16, true, float>, k_unpack_r2r<4, 16, false, float>); break;
      case 5: launch_dir(k_unpack_r2r<5, 16, true, float>, k_unpack_r2r<5, 16, false, float>); break;
      case 6: launch_dir(k_unpack_r2r<6, 16, true, float>, k_unpack_r2r<6, 16, false, float>); break;
      case 7: launch_dir(k_unpack_r2r<7, 16, true, float>, k_unpack_r2r<7, 16, false, float>); break;
      case 8: launch_dir(k_unpack_r2r<8, 16, true, float>, k_unpack_r2r<8, 16, false, float>); break;
      case 9: launch_dir(k_unpack_r2r<9, 16, true, float>, k_unpack_r2r<9, 16, false, float>); break;
      default: launch_dir(k_unpack_r2r<10, 8, true, float>, k_unpack_r2r<10, 8, false, float>); break;
    }
  } else {
    switch (logL) {
      case 3: launch_dir(k_unpack_r2r<3, 8, true, double>, k_unpack_r2r<3, 8, false, double>); break;
      case 4: launch_dir(k_unpack_r2r<4, 8, true, double>, k_unpack_r2r<4, 8, false, double>); break;
      case 5: launch_dir(k_unpack_r2r<5, 8, true, double>, k_unpack_r2r<5, 8, false, double>); break;
      case 6: launch_dir(k_unpack_r2r<6, 8, true, double>, k_unpack_r2r<6, 8, false, double>); break;
      case 7: launch_dir(k_unpack_r2r<7, 8, true, double>, k_unpack_r2r<7, 8, false, double>); break;
      case 8: launch_dir(k_unpack_r2r<8, 8, true, double>, k_unpack_r2r<8, 8, false, double>); break;
      case 9: launch_dir(k_unpack_r2r<9, 8, true, double>, k_unpack_r2r<9, 8, false, double>); break;
      default: launch_dir(k_unpack_r2r<10, 4, true, double>, k_unpack_r2r<10, 4, false, double>); break;
    }
  }
  if (e != cudaSuccess) {
    set_error("fused r2r kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

pa_status unpack_rfft(int nb, const BlockCopy* const* blocks, const void* const* srcs, void* dst,
                      bool f32, void* stream) {
  // (pa_transpose_rfft has already asked plan_real_check for every rank of the line)
  FftParams p;
  int C = 0;
  unsigned long long grid = 0;
  pa_status s = fft_geometry(nb, blocks, srcs, dst, f32, FusedMode::rfft, p, &C, &grid);
  if (s != PA_OK || grid == 0) return s;
  const int logL = p.logL;
  p.pitch = pa_fft::padded_pitch(p.L);  // as rfft_lines, forward
  p.tw = twiddles(2 * p.L, f32);
  if (!p.tw) {
    set_error("fused rfft: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const size_t smem = (f32 ? sizeof(pa_fft::cplxf) : sizeof(cplx)) * (size_t)C * p.pitch;
  cudaError_t e = cudaSuccess;
  auto launch = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    cudaGetLastError();
    kern<<<(unsigned)grid, FFT_THREADS, smem, (cudaStream_t)stream>>>(p);
    e = cudaGetLastError();
  };
  if (f32) {
    switch (logL) {
      case 3: launch(k_unpack_rfft<3, 16, float>); break;
      case 4: launch(k_unpack_rfft<4, 16, float>); break;
      case 5: launch(k_unpack_rfft<5, 16, float>); break;
      case 6: launch(k_unpack_rfft<6, 16, float>); break;
      case 7: launch(k_unpack_rfft<7, 16, float>); break;
      case 8: launch(k_unpack_rfft<8, 16, float>); break;
      case 9: launch(k_unpack_rfft<9, 16, float>); break;
      default: launch(k_unpack_rfft<10, 8, float>); break;
    }
  } else {
    switch (logL) {
      case 3: launch(k_unpack_rfft<3, 8, double>); break;
      case 4: launch(k_unpack_rfft<4, 8, double>); break;
      case 5: launch(k_unpack_rfft<5, 8, double>); break;
      case 6: launch(k_unpack_rfft<6, 8, double>); break;
      case 7: launch(k_unpack_rfft<7, 8, double>); break;
      case 8: launch(k_unpack_rfft<8, 8, double>); break;
      case 9: launch(k_unpack_rfft<9, 8, double>); break;
      default: launch(k_unpack_rfft<10, 4, double>); break;
    }
  }
  if (e != cudaSuccess) {
    set_error("fused rfft kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

// Can pa_transpose fuse the FFT (brfft: pa_transpose_brfft the complex-to-real transform) into
// this plan's unpack?  Every rank of a grid line must get the same answer: a rank that refused
// before the exchange while its peers went ahead would leave them waiting on flags it never
// sets.  So the answer depends on the global geometry only: the blocks that EVERY rank of the
// line would gather -- each rank's plan rebuilt from the pencils with that rank's coordinates --
// with the self block read from src and staged through recv_buf alike.  A PeerGet plan may also
// run the complex FFT one-sided (k_get_fft): its blocks are then the peers' get blocks, read from
// their src arrays, and the self block from src, so that configuration is checked as well.
// The plan rank n of P's grid line holds: P itself for this rank, else rebuilt from the pencils
// with that rank's coordinates (owned by `hold`).
static pa_status line_plan(Plan* P, int n, std::unique_ptr<Plan>& hold, const Plan** Q) {
  *Q = P;
  if (n == P->self_index) return PA_OK;
  auto topo = std::make_shared<Topology>(*P->pin->topo);
  topo->coords[P->dim] = n;
  topo->rank = topo->rank_of(topo->coords);
  auto pin = std::make_shared<Pencil>(*P->pin);
  auto pout = std::make_shared<Pencil>(*P->pout);
  pin->topo = topo;
  pout->topo = topo;
  Plan* q = nullptr;
  pa_status s = build_plan(pin, pout, P->n_extra, P->extra, P->elsize, P->method, &q);
  if (s != PA_OK) return s;
  hold.reset(q);
  *Q = q;
  return PA_OK;
}

static pa_status fused_check(Plan* P, bool f32, FusedMode mode) {
  if (mode == FusedMode::r2r || mode == FusedMode::rfft) {
    if (P->elsize != (f32 ? 4 : 8)) {
      set_error(f32 ? "fused real transform: PA_FFT_F32 takes Float32 (4-byte) elements only"
                    : "fused real transform: Float64 (8-byte) elements only");
      return PA_EINVAL;
    }
  } else if (!f32 && P->elsize != 16) {
    set_error("fused FFT: ComplexF64 (16-byte) elements only");
    return PA_EINVAL;
  } else if (f32 && P->elsize != 8) {
    set_error("fused FFT: PA_FFT_F32 takes ComplexF32 (8-byte) elements only");
    return PA_EINVAL;
  }
  FftParams p;
  int C = 0;
  unsigned long long grid = 0;
  if (P->dim < 0 || P->nproc == 1) {
    const BlockCopy* b = &P->self_fused;
    return fft_geometry(1, &b, nullptr, nullptr, f32, mode, p, &C, &grid);
  }
  for (int n = 0; n < P->nproc; ++n) {
    std::unique_ptr<Plan> hold;
    const Plan* Q = nullptr;
    {
      pa_status s = line_plan(P, n, hold, &Q);
      if (s != PA_OK) return s;
    }
    // 0: self block from src, 1: self block staged through recv_buf, 2: one-sided get
    const int configs = (mode == FusedMode::fft && P->method == PA_PEER_GET) ? 3 : 2;
    for (int cfg = 0; cfg < configs; ++cfg) {
      std::vector<const BlockCopy*> bl;
      for (int k = 0; k < Q->nproc; ++k)
        bl.push_back(k == Q->self_index && cfg != 1 ? &Q->self_fused
                                                    : cfg == 2 ? &Q->peers[k].get : &Q->peers[k].unpack);
      pa_status s = fft_geometry(Q->nproc, bl.data(), nullptr, nullptr, f32, mode, p, &C, &grid);
      if (s != PA_OK) {
        if (n != P->self_index) {
          const std::string why = last_error();
          set_error("%s (on rank %d of the grid line)", why.c_str(), n + 1);
        }
        return s;
      }
    }
  }
  return PA_OK;
}

// Cached per plan, per precision (f32: ComplexF32) and per value of tunable fft_lines.
pa_status plan_fft_check(Plan* P, bool f32) {
  const int q = f32 ? 1 : 0;
  if (P->fft_check_lines[q] != g_tun.fft_lines) {
    P->fft_check[q] = fused_check(P, f32, FusedMode::fft);
    P->fft_check_err[q] = P->fft_check[q] == PA_OK ? std::string() : std::string(last_error());
    P->fft_check_lines[q] = g_tun.fft_lines;
  } else if (P->fft_check[q] != PA_OK) {
    set_error("%s", P->fft_check_err[q].c_str());
  }
  return P->fft_check[q];
}

// Cached per plan and per precision, apart from plan_fft_check's verdicts (the lines per CTA of
// the brfft kernel do not depend on tunable fft_lines).
pa_status plan_brfft_check(Plan* P, bool f32) {
  const int q = f32 ? 1 : 0;
  if (!P->brfft_checked[q]) {
    if (P->dim >= 0 && P->nproc > 1 && (P->method == PA_PEER_PUT || P->method == PA_PEER_GET)) {
      // (src and the real dst never alias, so these methods never fall back to a staged schedule)
      set_error("fused brfft: the one-sided methods have no unpack pass to fuse with; use "
                "PointToPoint / Alltoallv");
      P->brfft_check[q] = PA_EINVAL;
    } else {
      P->brfft_check[q] = fused_check(P, f32, FusedMode::brfft);
    }
    P->brfft_check_err[q] = P->brfft_check[q] == PA_OK ? std::string() : std::string(last_error());
    P->brfft_checked[q] = true;
  } else if (P->brfft_check[q] != PA_OK) {
    set_error("%s", P->brfft_check_err[q].c_str());
  }
  return P->brfft_check[q];
}

// Can pa_transpose_r2r / pa_transpose_rfft run on this real plan?  Both kernels gather the same
// blocks (N reals per line), so one verdict answers for both: the rfft geometry, which checks
// everything the r2r geometry does plus the rescale of the destination to N/2 + 1 bins per line.
// Cached per plan and per precision, apart from the fft and brfft verdicts.
pa_status plan_real_check(Plan* P, bool f32) {
  const int q = f32 ? 1 : 0;
  if (!P->real_checked[q]) {
    if (P->dim >= 0 && P->nproc > 1 && (P->method == PA_PEER_PUT || P->method == PA_PEER_GET)) {
      // (src and dst never overlap, so these methods never fall back to a staged schedule)
      set_error("fused real transform: the one-sided methods have no unpack pass to fuse with; "
                "use PointToPoint / Alltoallv");
      P->real_check[q] = PA_EINVAL;
    } else {
      P->real_check[q] = fused_check(P, f32, FusedMode::rfft);
    }
    P->real_check_err[q] = P->real_check[q] == PA_OK ? std::string() : std::string(last_error());
    P->real_checked[q] = true;
  } else if (P->real_check[q] != PA_OK) {
    set_error("%s", P->real_check_err[q].c_str());
  }
  return P->real_check[q];
}

// Can pa_fft_put (rfft: pa_rfft_put; brfft: pa_r2r_put and pa_brfft_put) run on this plan?  The
// send-side kernel runs on PeerPut plans and on local transposes (no exchange, or a line of one
// rank) of any method.  As fused_check, every rank of the grid line gets the same answer: its plan
// is rebuilt and its blocks -- the self block and the put blocks -- checked.
static pa_status put_check(Plan* P, bool f32, PutMode mode) {
  const bool real = mode == PutMode::r2r || mode == PutMode::brfft;
  const char* what = real ? "fused real transform + put"
                          : mode == PutMode::rfft ? "fused rfft + put" : "fused FFT + put";
  if (real && P->elsize != (f32 ? 4 : 8)) {
    set_error(f32 ? "%s: PA_FFT_F32 takes a Float32 (elsize 4) plan"
                  : "%s: a Float64 (elsize 8) plan, or PA_FFT_F32 for Float32", what);
    return PA_EINVAL;
  }
  if (!real && P->elsize != (f32 ? 8 : 16)) {
    set_error(f32 ? "%s: PA_FFT_F32 takes a ComplexF32 (elsize 8) plan"
                  : "%s: a ComplexF64 (elsize 16) plan, or PA_FFT_F32 for ComplexF32", what);
    return PA_EINVAL;
  }
  const Pencil& Pi = *P->pin;
  for (int i = 0; i < Pi.topo->M; ++i)
    if (Pi.decomp[i] == Pi.perm[0]) {
      set_error("%s: the transform axis (logical dim %d, the first memory dim of src) is decomposed",
                what, Pi.perm[0] + 1);
      return PA_EINVAL;
    }
  FftPutParams pp;
  int C = 0;
  unsigned long long grid = 0;
  if (P->dim < 0 || P->nproc == 1) {
    const BlockCopy* b = &P->self_fused;
    return put_fft_geometry(1, &b, nullptr, nullptr, f32, mode, pp, &C, &grid);
  }
  if (P->method != PA_PEER_PUT) {
    if (real)
      set_error("%s: the send-side fusion needs PeerPut (or a local transposition); with "
                "PointToPoint, Alltoallv or PeerGet transform src first and fuse the next transform "
                "into the receive side (pa_transpose_r2r, pa_transpose_rfft, pa_transpose_brfft)", what);
    else
      set_error("%s: the send-side fusion needs PeerPut (or a local transposition); with "
                "PointToPoint, Alltoallv or PeerGet transform src first and fuse the next transform "
                "into the receive side (pa_transpose with PA_FFT_FORWARD / PA_FFT_BACKWARD)", what);
    return PA_EINVAL;
  }
  for (int n = 0; n < P->nproc; ++n) {
    std::unique_ptr<Plan> hold;
    const Plan* Q = nullptr;
    pa_status s = line_plan(P, n, hold, &Q);
    if (s != PA_OK) return s;
    std::vector<const BlockCopy*> bl;
    for (int k = 0; k < Q->nproc; ++k)
      bl.push_back(k == Q->self_index ? &Q->self_fused : &Q->peers[k].put);
    s = put_fft_geometry(Q->nproc, bl.data(), nullptr, nullptr, f32, mode, pp, &C, &grid);
    if (s != PA_OK) {
      if (n != P->self_index) {
        const std::string why = last_error();
        set_error("%s (on rank %d of the grid line)", why.c_str(), n + 1);
      }
      return s;
    }
  }
  return PA_OK;
}

// Cached per plan, per precision and (lines per CTA of fft_) per value of tunable fft_lines, apart
// from every other verdict.
pa_status plan_fft_put_check(Plan* P, bool f32) {
  const int q = f32 ? 1 : 0;
  if (P->fft_put_check_lines[q] != g_tun.fft_lines) {
    P->fft_put_check[q] = put_check(P, f32, PutMode::fft);
    P->fft_put_check_err[q] = P->fft_put_check[q] == PA_OK ? std::string() : std::string(last_error());
    P->fft_put_check_lines[q] = g_tun.fft_lines;
  } else if (P->fft_put_check[q] != PA_OK) {
    set_error("%s", P->fft_put_check_err[q].c_str());
  }
  return P->fft_put_check[q];
}

// Cached per plan and per precision, apart from every other verdict.
pa_status plan_rfft_put_check(Plan* P, bool f32) {
  const int q = f32 ? 1 : 0;
  if (!P->rfft_put_checked[q]) {
    P->rfft_put_check[q] = put_check(P, f32, PutMode::rfft);
    P->rfft_put_check_err[q] = P->rfft_put_check[q] == PA_OK ? std::string() : std::string(last_error());
    P->rfft_put_checked[q] = true;
  } else if (P->rfft_put_check[q] != PA_OK) {
    set_error("%s", P->rfft_put_check_err[q].c_str());
  }
  return P->rfft_put_check[q];
}

// One verdict for pa_r2r_put and pa_brfft_put (the brfft geometry checks all that r2r's does, and
// its rescale); cached per plan and per precision, apart from every other verdict.
pa_status plan_real_put_check(Plan* P, bool f32) {
  const int q = f32 ? 1 : 0;
  if (!P->real_put_checked[q]) {
    P->real_put_check[q] = put_check(P, f32, PutMode::brfft);
    P->real_put_check_err[q] = P->real_put_check[q] == PA_OK ? std::string() : std::string(last_error());
    P->real_put_checked[q] = true;
  } else if (P->real_put_check[q] != PA_OK) {
    set_error("%s", P->real_put_check_err[q].c_str());
  }
  return P->real_put_check[q];
}

pa_status rfft_lines(int N, bool forward, bool f32, i64 nlines, const void* src, void* dst,
                     void* stream) {
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
  const long long rs = f32 ? 4 : 8, cs = 2 * rs;  // bytes of a real / a complex element
  p.src_line = forward ? rs * N : cs * (L + 1);
  p.dst_line = forward ? cs * (L + 1) : rs * N;
  p.pitch = pa_fft::padded_pitch(forward ? L : L + 1);  // backward stages all N/2 + 1 bins
  p.tw = twiddles(N, f32);
  if (!p.tw) {
    set_error("rfft: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const int C = f32 ? fft_lines_f32(logL) : fft_lines(logL);
  const long long grid = (nlines + C - 1) / C;
  if (grid > 0x7fffffffLL) {
    set_error("rfft: too many lines for one launch");
    return PA_EINVAL;
  }
  const size_t smem = (size_t)cs * C * p.pitch;
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
  if (f32) {
    switch (logL) {
      case 3: launch_dir(k_rfft<3, 16, true, float>, k_rfft<3, 16, false, float>); break;
      case 4: launch_dir(k_rfft<4, 16, true, float>, k_rfft<4, 16, false, float>); break;
      case 5: launch_dir(k_rfft<5, 16, true, float>, k_rfft<5, 16, false, float>); break;
      case 6: launch_dir(k_rfft<6, 16, true, float>, k_rfft<6, 16, false, float>); break;
      case 7: launch_dir(k_rfft<7, 16, true, float>, k_rfft<7, 16, false, float>); break;
      case 8: launch_dir(k_rfft<8, 16, true, float>, k_rfft<8, 16, false, float>); break;
      case 9: launch_dir(k_rfft<9, 16, true, float>, k_rfft<9, 16, false, float>); break;
      default: launch_dir(k_rfft<10, 8, true, float>, k_rfft<10, 8, false, float>); break;
    }
  } else {
    switch (logL) {
      case 3: launch_dir(k_rfft<3, 8, true, double>, k_rfft<3, 8, false, double>); break;
      case 4: launch_dir(k_rfft<4, 8, true, double>, k_rfft<4, 8, false, double>); break;
      case 5: launch_dir(k_rfft<5, 8, true, double>, k_rfft<5, 8, false, double>); break;
      case 6: launch_dir(k_rfft<6, 8, true, double>, k_rfft<6, 8, false, double>); break;
      case 7: launch_dir(k_rfft<7, 8, true, double>, k_rfft<7, 8, false, double>); break;
      case 8: launch_dir(k_rfft<8, 8, true, double>, k_rfft<8, 8, false, double>); break;
      case 9: launch_dir(k_rfft<9, 8, true, double>, k_rfft<9, 8, false, double>); break;
      default: launch_dir(k_rfft<10, 4, true, double>, k_rfft<10, 4, false, double>); break;
    }
  }
  if (e != cudaSuccess) {
    set_error("rfft kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

pa_status r2r_lines(int N, bool forward, bool sine, bool f32, i64 nlines, const void* src, void* dst,
                    void* stream) {
  const int L = N / 2;
  int logL = 0;
  while ((1 << logL) < L) ++logL;
  if ((1 << logL) != L || logL < 3 || logL > 10) {
    set_error("r2r: line length %d is not a power of two in 16..2048", N);
    return PA_EINVAL;
  }
  if (nlines == 0) return PA_OK;
  R2rParams p;
  p.src = (const char*)src;
  p.dst = (char*)dst;
  p.nlines = nlines;
  const long long rs = f32 ? 4 : 8, cs = 2 * rs;  // bytes of a real / a complex element
  p.line = rs * N;
  p.pitch = pa_fft::padded_pitch(forward ? L : L + 1);  // backward stages the pairs of slots 0..L
  p.sine = sine ? 1 : 0;
  p.tw = twiddles(N, f32);
  p.tw4 = twiddles(4 * N, f32);
  if (!p.tw || !p.tw4) {
    set_error("r2r: twiddle table allocation failed");
    cudaGetLastError();
    return PA_ENOMEM;
  }
  const int C = f32 ? fft_lines_f32(logL) : fft_lines(logL);
  const long long grid = (nlines + C - 1) / C;
  if (grid > 0x7fffffffLL) {
    set_error("r2r: too many lines for one launch");
    return PA_EINVAL;
  }
  const size_t smem = (size_t)cs * C * p.pitch;
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
  if (f32) {
    switch (logL) {
      case 3: launch_dir(k_r2r<3, 16, true, float>, k_r2r<3, 16, false, float>); break;
      case 4: launch_dir(k_r2r<4, 16, true, float>, k_r2r<4, 16, false, float>); break;
      case 5: launch_dir(k_r2r<5, 16, true, float>, k_r2r<5, 16, false, float>); break;
      case 6: launch_dir(k_r2r<6, 16, true, float>, k_r2r<6, 16, false, float>); break;
      case 7: launch_dir(k_r2r<7, 16, true, float>, k_r2r<7, 16, false, float>); break;
      case 8: launch_dir(k_r2r<8, 16, true, float>, k_r2r<8, 16, false, float>); break;
      case 9: launch_dir(k_r2r<9, 16, true, float>, k_r2r<9, 16, false, float>); break;
      default: launch_dir(k_r2r<10, 8, true, float>, k_r2r<10, 8, false, float>); break;
    }
  } else {
    switch (logL) {
      case 3: launch_dir(k_r2r<3, 8, true, double>, k_r2r<3, 8, false, double>); break;
      case 4: launch_dir(k_r2r<4, 8, true, double>, k_r2r<4, 8, false, double>); break;
      case 5: launch_dir(k_r2r<5, 8, true, double>, k_r2r<5, 8, false, double>); break;
      case 6: launch_dir(k_r2r<6, 8, true, double>, k_r2r<6, 8, false, double>); break;
      case 7: launch_dir(k_r2r<7, 8, true, double>, k_r2r<7, 8, false, double>); break;
      case 8: launch_dir(k_r2r<8, 8, true, double>, k_r2r<8, 8, false, double>); break;
      case 9: launch_dir(k_r2r<9, 8, true, double>, k_r2r<9, 8, false, double>); break;
      default: launch_dir(k_r2r<10, 4, true, double>, k_r2r<10, 4, false, double>); break;
    }
  }
  if (e != cudaSuccess) {
    set_error("r2r kernel launch failed: %s", cudaGetErrorString(e));
    return PA_ECUDA;
  }
  count_launch();
  return PA_OK;
}

}  // namespace pa
