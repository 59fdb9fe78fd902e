// sm_90a kernels of the transpose! hot path.
//
// Every data movement of the path -- K1 pack (copy_range!,
// Transpositions.jl:552-583), K2 unpack+permute (copy_permuted! ->
// _permutedims!, :585-664), K3 fused self block / permute_local! (:235-270),
// and the one-sided K1-put / K2-get variants whose other side is a peer GPU's
// memory over NVLink -- is one primitive: an N-d strided box copy
//     dst[sum k_i ds_i] = src[sum k_i ss_i],  k in box,
// canonicalised on the host (plan.cpp) into tile dims X (source-fastest),
// Y (destination-fastest, or the next dim) and up to 6 outer dims.
//
// Three tile bodies, all bandwidth-bound pure byte movers (bit-exact by construction):
//   RowsBody<VT,ULOG>     X contiguous on both sides: vectorised row copy, 2^ULOG
//                         accesses in flight per thread (8 x 128-bit, or 16 narrower
//                         ones when a side is not 16-byte aligned), streaming hints.
//   TransBody<S,TBQ,SE,DE> X contiguous in src, Y contiguous in dst: 512-byte
//                         coalesced 128-bit loads, VxV register micro-transpose,
//                         padded (conflict-free) shared tile in 16-byte items,
//                         512-byte coalesced 128-bit stores.  SE / DE: that side
//                         is only element-aligned (odd extents: the N/2+1 grids of
//                         real-to-complex transforms) and is accessed element-wise,
//                         still coalesced, while the other side keeps its 128-bit
//                         accesses and the shared tile keeps its 16-byte items.
//   ScalarBody<ET>        any strides (tiny boxes, split elements): 32x32 element
//                         tile through padded shared memory.
// Each body runs under three kernels: k_box<B,false> one tile per CTA (HBM-bound
// local work: the grid is the whole problem), k_box<B,true> a capped grid whose
// CTAs stride over the tiles (NVLink-bound remote work: a few CTAs per SM saturate
// the links and the rest of the SM stays available to concurrent local kernels),
// and k_multi<B>: ONE launch over the blocks of every peer of a grid line, tiles
// interleaved round-robin so that all destination links are driven at once, with
// the window protocol (ready / done flags over NVLink) folded into its prologue
// and epilogue.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>

#include "flags.cuh"
#include "pa_internal.hpp"

namespace pa {

Tunables g_tun;
static std::atomic<i64> g_launches{0};
i64 launch_count() { return g_launches.load(); }
void count_launch() { g_launches.fetch_add(1); }

constexpr int MAXO = PA_MAX_DIMS - 1;
typedef unsigned long long ull;

struct KParams {
  const char* src;  // offset to the box origin
  char* dst;
  long long ex, ey;                  // tile-dim extents (rows: ex in vectors)
  long long sx_s, sx_d, sy_s, sy_d;  // byte strides of X and Y
  unsigned tiles_x, tiles_y;
  ull total;  // tiles in the launch
  int no;     // outer dims
  long long oe[MAXO], os[MAXO], od[MAXO];
  int lx_log2, ux_log2;  // rows thread/unroll shape
  int y_fastest;         // tile order: consecutive CTAs walk along Y (destination rows) first
};

__device__ __forceinline__ void decode_tile(const KParams& p, ull bid, unsigned& tx, unsigned& ty,
                                            const char*& s, char*& d) {
  if (p.y_fastest) {
    ty = (unsigned)(bid % p.tiles_y);
    bid /= p.tiles_y;
    tx = (unsigned)(bid % p.tiles_x);
    bid /= p.tiles_x;
  } else {
    tx = (unsigned)(bid % p.tiles_x);
    bid /= p.tiles_x;
    ty = (unsigned)(bid % p.tiles_y);
    bid /= p.tiles_y;
  }
  s = p.src;
  d = p.dst;
#pragma unroll 1
  for (int i = 0; i < p.no; ++i) {
    long long k = (long long)(bid % (ull)p.oe[i]);
    bid /= (ull)p.oe[i];
    s += k * p.os[i];
    d += k * p.od[i];
  }
}

// streaming (evict-first) accesses: every byte is touched exactly once
template <typename T>
__device__ __forceinline__ T ld_stream(const char* p) {
  return __ldcs(reinterpret_cast<const T*>(p));
}
template <typename T>
__device__ __forceinline__ void st_stream(char* p, const T& v) {
  __stcs(reinterpret_cast<T*>(p), v);
}
// 1- and 2-byte flavours have no __ldcs overload for the unsigned short/char we use
template <>
__device__ __forceinline__ uint16_t ld_stream<uint16_t>(const char* p) {
  return *reinterpret_cast<const uint16_t*>(p);
}
template <>
__device__ __forceinline__ void st_stream<uint16_t>(char* p, const uint16_t& v) {
  *reinterpret_cast<uint16_t*>(p) = v;
}
template <>
__device__ __forceinline__ uint8_t ld_stream<uint8_t>(const char* p) {
  return *reinterpret_cast<const uint8_t*>(p);
}
template <>
__device__ __forceinline__ void st_stream<uint8_t>(char* p, const uint8_t& v) {
  *reinterpret_cast<uint8_t*>(p) = v;
}

// programmatic dependent launch: a kernel launched with the stream-serialisation
// attribute may be scheduled while its predecessor drains; it must not touch
// global memory before `wait`, and lets ITS successor in once every CTA is running
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ---------------------------------------------------------------------------
// Rows: runs contiguous on both sides.
// 256 threads as LX x LY, each thread moves U = 2^ULOG vectors laid out UX x UY.
template <typename VT, int ULOG>
struct RowsBody {
  static constexpr int SMEM_ITEMS = 0;
  static constexpr bool SYNC = false;
  static __device__ __forceinline__ void run(const KParams& p, ull bid, uint4*) {
    constexpr int W = sizeof(VT);
    constexpr int U = 1 << ULOG;
    const int lxl = p.lx_log2, uxl = p.ux_log2;
    const int LX = 1 << lxl, LY = 256 >> lxl;
    const int lx = threadIdx.x & (LX - 1), ly = threadIdx.x >> lxl;
    unsigned tx, ty;
    const char* s;
    char* d;
    decode_tile(p, bid, tx, ty, s, d);
    const long long xv0 = (long long)tx * ((long long)LX << uxl) + lx;
    const long long y0 = (long long)ty * ((long long)LY << (ULOG - uxl)) + ly;
    VT v[U];
    long long so[U], dof[U];
    bool ok[U];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int ux = i & ((1 << uxl) - 1), uy = i >> uxl;
      const long long xv = xv0 + (long long)ux * LX, y = y0 + (long long)uy * LY;
      ok[i] = (xv < p.ex) && (y < p.ey);
      so[i] = y * p.sy_s + xv * W;
      dof[i] = y * p.sy_d + xv * W;
    }
#pragma unroll
    for (int i = 0; i < U; ++i)
      if (ok[i]) v[i] = ld_stream<VT>(s + so[i]);
#pragma unroll
    for (int i = 0; i < U; ++i)
      if (ok[i]) st_stream<VT>(d + dof[i], v[i]);
  }
};

// ---------------------------------------------------------------------------
// Rows as a pure DMA pipeline (TMA bulk copies, SASS UBLKCP).  One elected
// thread per CTA drives a ring of STAGES shared-memory buffers: cp.async.bulk
// global->shared completing on an mbarrier, then cp.async.bulk shared->global
// in a bulk group; the CTA strides over (row, chunk) units.  No registers or
// LSU slots are spent on the payload (tunable "bulk_rows").
constexpr int BULK_STAGES = 4;
constexpr int BULK_CHUNK = 16384;  // bytes per stage

__device__ __forceinline__ unsigned smem_u32(const void* p) {
  return (unsigned)__cvta_generic_to_shared(p);
}

__global__ void __launch_bounds__(32) k_rows_bulk(const __grid_constant__ KParams p) {
  extern __shared__ __align__(128) char bulk_smem[];
  __shared__ __align__(8) ull full[BULK_STAGES];
  if (threadIdx.x != 0) return;  // a single thread owns the whole pipeline
  const unsigned chunk = (unsigned)p.lx_log2;  // bytes per unit (<= BULK_CHUNK), multiple of 16
  const long long run = p.ex;                  // bytes per row
  for (int s = 0; s < BULK_STAGES; ++s)
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&full[s])));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

  auto unit = [&](ull bid, const char*& s, char*& d, unsigned& bytes) {
    unsigned tx, ty;
    decode_tile(p, bid, tx, ty, s, d);
    const long long x = (long long)tx * chunk;
    s += (long long)ty * p.sy_s + x;
    d += (long long)ty * p.sy_d + x;
    bytes = (unsigned)((run - x) < (long long)chunk ? (run - x) : (long long)chunk);
  };
  auto load = [&](int st, ull bid) {
    const char* s;
    char* d;
    unsigned bytes;
    unit(bid, s, d, bytes);
    const unsigned bar = smem_u32(&full[st]);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(bulk_smem + st * BULK_CHUNK)),
        "l"(s), "r"(bytes), "r"(bar)
        : "memory");
  };

  ull next_load = blockIdx.x;
  int ls = 0;
  for (int i = 0; i < BULK_STAGES && next_load < p.total; ++i) {
    load(ls, next_load);
    next_load += gridDim.x;
    ls = (ls + 1) % BULK_STAGES;
  }
  int ss = 0, prev = -1;
  unsigned parity = 0;
  for (ull bid = blockIdx.x; bid < p.total; bid += gridDim.x) {
    const unsigned bar = smem_u32(&full[ss]);
    unsigned done = 0;
    while (!done) {
      asm volatile(
          "{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\n\t"
          "selp.u32 %0, 1, 0, q;\n\t}"
          : "=r"(done)
          : "r"(bar), "r"(parity)
          : "memory");
    }
    const char* s;
    char* d;
    unsigned bytes;
    unit(bid, s, d, bytes);
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(d),
                 "r"(smem_u32(bulk_smem + ss * BULK_CHUNK)), "r"(bytes)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    if (prev >= 0 && next_load < p.total) {
      // the PREVIOUS stage may be refilled once its store has finished READING it
      // (all but the newest bulk group done reading)
      asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      load(prev, next_load);
      next_load += gridDim.x;
    }
    prev = ss;
    ss = (ss + 1) % BULK_STAGES;
    if (ss == 0) parity ^= 1;
  }
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ---------------------------------------------------------------------------
// Transpose: element size S in {4,8,16}, V = 16/S elements per 16-byte item.
// Tile: TA = 32*V elements along X (512 B of source row), TB = TBQ*V elements
// along Y (TBQ*16 B of destination row).
template <int S>
struct Elem;
template <>
struct Elem<4> {
  typedef uint32_t T;
};
template <>
struct Elem<8> {
  typedef uint2 T;
};
template <>
struct Elem<16> {
  typedef uint4 T;
};

template <int S>
__device__ __forceinline__ uint4 gather_col(const uint4 (&r)[16 / S], int c);
template <>
__device__ __forceinline__ uint4 gather_col<16>(const uint4 (&r)[1], int) {
  return r[0];
}
template <>
__device__ __forceinline__ uint4 gather_col<8>(const uint4 (&r)[2], int c) {
  return c == 0 ? make_uint4(r[0].x, r[0].y, r[1].x, r[1].y)
                : make_uint4(r[0].z, r[0].w, r[1].z, r[1].w);
}
__device__ __forceinline__ unsigned comp(const uint4& v, int c) {
  return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w;
}
template <>
__device__ __forceinline__ uint4 gather_col<4>(const uint4 (&r)[4], int c) {
  return make_uint4(comp(r[0], c), comp(r[1], c), comp(r[2], c), comp(r[3], c));
}
// V elements (consecutive along Y) <-> one 16-byte item
__device__ __forceinline__ uint4 pack_item(const uint32_t (&e)[4]) {
  return make_uint4(e[0], e[1], e[2], e[3]);
}
__device__ __forceinline__ uint4 pack_item(const uint2 (&e)[2]) {
  return make_uint4(e[0].x, e[0].y, e[1].x, e[1].y);
}
__device__ __forceinline__ uint4 pack_item(const uint4 (&e)[1]) { return e[0]; }
__device__ __forceinline__ void unpack_item(const uint4& v, uint32_t (&e)[4]) {
  e[0] = v.x, e[1] = v.y, e[2] = v.z, e[3] = v.w;
}
__device__ __forceinline__ void unpack_item(const uint4& v, uint2 (&e)[2]) {
  e[0] = make_uint2(v.x, v.y), e[1] = make_uint2(v.z, v.w);
}
__device__ __forceinline__ void unpack_item(const uint4& v, uint4 (&e)[1]) { e[0] = v; }

template <int S, int TBQ, bool SE, bool DE>
struct TransBody {
  static constexpr int V = 16 / S;
  static constexpr int TA = 32 * V;
  static constexpr int TB = TBQ * V;
  static constexpr int PITCH = TBQ + 1;  // odd pitch in 16-byte items: conflict-free both phases
  static constexpr int QI = TBQ / 8;
  static constexpr int SMEM_ITEMS = TA * PITCH;
  static constexpr bool SYNC = true;
  typedef typename Elem<S>::T ET;

  static __device__ __forceinline__ void run(const KParams& p, ull bid, uint4* sm) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned tx, ty;
    const char* s;
    char* d;
    decode_tile(p, bid, tx, ty, s, d);
    const long long x0 = (long long)tx * TA, y0 = (long long)ty * TB;

    if constexpr (!SE) {
      // 16-byte loads: lane -> V consecutive x, V rows per thread and pass
      const long long xl = x0 + lane * V;
      const bool xok = xl < p.ex;
      uint4 r[QI][V];
#pragma unroll
      for (int qi = 0; qi < QI; ++qi) {
#pragma unroll
        for (int rr = 0; rr < V; ++rr) {
          const long long y = y0 + (long long)(warp + 8 * qi) * V + rr;
          r[qi][rr] = (xok && y < p.ey) ? ld_stream<uint4>(s + y * p.sy_s + xl * S)
                                        : make_uint4(0u, 0u, 0u, 0u);
        }
      }
#pragma unroll
      for (int qi = 0; qi < QI; ++qi) {
        const int q = warp + 8 * qi;
#pragma unroll
        for (int c = 0; c < V; ++c) sm[(c * 32 + lane) * PITCH + q] = gather_col<S>(r[qi], c);
      }
    } else {
      // element loads (the source rows are only S-byte aligned): lane -> x, V columns
      // 32 apart and V rows per thread and pass -- same bytes in flight as above
      ET r[QI][V][V];
#pragma unroll
      for (int qi = 0; qi < QI; ++qi) {
#pragma unroll
        for (int c = 0; c < V; ++c) {
          const long long x = x0 + c * 32 + lane;
#pragma unroll
          for (int rr = 0; rr < V; ++rr) {
            const long long y = y0 + (long long)(warp + 8 * qi) * V + rr;
            if (x < p.ex && y < p.ey)
              r[qi][c][rr] = ld_stream<ET>(s + y * p.sy_s + x * S);
            else
              r[qi][c][rr] = ET();
          }
        }
      }
#pragma unroll
      for (int qi = 0; qi < QI; ++qi) {
        const int q = warp + 8 * qi;
#pragma unroll
        for (int c = 0; c < V; ++c) sm[(c * 32 + lane) * PITCH + q] = pack_item(r[qi][c]);
      }
    }
    __syncthreads();
    if constexpr (!DE) {
      constexpr int IT = TA * TBQ / 256;
#pragma unroll
      for (int k = 0; k < IT; ++k) {
        const int idx = threadIdx.x + 256 * k;
        const int xr = idx / TBQ, qq = idx % TBQ;
        const long long x = SE ? x0 + xr : x0 + (long long)(xr & 31) * V + (xr >> 5);
        const long long y = y0 + (long long)qq * V;
        if (x < p.ex && y < p.ey) st_stream<uint4>(d + x * p.sx_d + y * S, sm[xr * PITCH + qq]);
      }
    } else {
      // element stores (the destination rows are only S-byte aligned): consecutive lanes
      // take consecutive ELEMENTS of a destination row -- shared memory read as S-byte
      // words of the 16-byte items, conflict-free, 32 x S bytes contiguous per warp store
      const ET* sme = reinterpret_cast<const ET*>(sm);
      constexpr int ITE = TA * TB / 256;
#pragma unroll 8
      for (int k = 0; k < ITE; ++k) {
        const int idx = threadIdx.x + 256 * k;
        const int xr = idx / TB, ye = idx % TB;
        const long long x = SE ? x0 + xr : x0 + (long long)(xr & 31) * V + (xr >> 5);
        const long long y = y0 + ye;
        if (x < p.ex && y < p.ey)
          st_stream<ET>(d + x * p.sx_d + y * S, sme[(xr * PITCH + ye / V) * V + (ye % V)]);
      }
    }
  }
};

// ---------------------------------------------------------------------------
// Scalar: general strides, element-wise accesses.
template <typename ET>
struct ScalarBody {
  static constexpr int SMEM_ITEMS = (32 * 33 * sizeof(ET) + 15) / 16;
  static constexpr bool SYNC = true;
  static __device__ __forceinline__ void run(const KParams& p, ull bid, uint4* smraw) {
    ET(*sm)[33] = reinterpret_cast<ET(*)[33]>(smraw);
    const int a = threadIdx.x & 31, b = threadIdx.x >> 5;
    unsigned tx, ty;
    const char* s;
    char* d;
    decode_tile(p, bid, tx, ty, s, d);
    const long long x0 = (long long)tx * 32, y0 = (long long)ty * 32;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long x = x0 + a, y = y0 + b + 8 * k;
      if (x < p.ex && y < p.ey)
        sm[b + 8 * k][a] = *reinterpret_cast<const ET*>(s + x * p.sx_s + y * p.sy_s);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long x = x0 + b + 8 * k, y = y0 + a;
      if (x < p.ex && y < p.ey)
        *reinterpret_cast<ET*>(d + x * p.sx_d + y * p.sy_d) = sm[a][b + 8 * k];
    }
  }
};

// ---------------------------------------------------------------------------
template <class B, bool LOOP>
__global__ void __launch_bounds__(256) k_box(const __grid_constant__ KParams p) {
  __shared__ uint4 sm[B::SMEM_ITEMS > 0 ? B::SMEM_ITEMS : 1];
  pdl_enter();
  if constexpr (LOOP) {
    for (ull bid = blockIdx.x; bid < p.total; bid += gridDim.x) {
      B::run(p, bid, sm);
      if (B::SYNC) __syncthreads();  // the shared tile is reused by the next iteration
    }
  } else {
    B::run(p, blockIdx.x, sm);
  }
}

// ---- flag words over NVLink (flag_signal / flag_wait: flags.cuh) ----------------
struct FlagKernelParams {
  int n;
  ull* remote[64];
  ull* local[64];
  ull seq[64];
  int do_signal, do_wait;
  ull timeout_ns;
  int* err;
};
__global__ void k_flags(const __grid_constant__ FlagKernelParams fp) {
  const int t = threadIdx.x;
  if (t >= fp.n) return;
  if (fp.do_signal) flag_signal(fp.remote[t], fp.seq[t]);
  if (fp.do_wait) flag_wait(fp.local[t], fp.seq[t], fp.timeout_ns, fp.err);
}

pa_status launch_flags(int n, ull* const* remote, ull* const* local, const ull* seq, bool do_signal,
                       bool do_wait, ull timeout_ns, int* err, void* stream) {
  // every signal of the line is sent before the first wait (no batch may wait
  // for a signal a later batch would send)
  for (int pass = 0; pass < 2; ++pass) {
    const bool sig = pass == 0 && do_signal, wt = pass == 1 && do_wait;
    if (!sig && !wt) continue;
    for (int base = 0; base < n; base += 64) {
      FlagKernelParams fp;
      memset(&fp, 0, sizeof fp);
      fp.n = std::min(64, n - base);
      for (int i = 0; i < fp.n; ++i) {
        fp.remote[i] = remote ? remote[base + i] : nullptr;
        fp.local[i] = local ? local[base + i] : nullptr;
        fp.seq[i] = seq[base + i];
      }
      fp.do_signal = sig;
      fp.do_wait = wt;
      fp.timeout_ns = timeout_ns;
      fp.err = err;
      cudaGetLastError();  // (clear: only this launch is being checked)
      k_flags<<<1, 64, 0, (cudaStream_t)stream>>>(fp);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) {
        set_error("flag kernel launch failed: %s", cudaGetErrorString(e));
        return PA_ECUDA;
      }
      count_launch();
    }
  }
  return PA_OK;
}

// ---- one launch over the blocks of every peer ------------------------------------
struct MultiParams {
  int nb;
  ull max_total;  // max over the blocks' tile counts
  KParams kp[FLAG_INLINE_MAX];
  MultiFlags mf;
};

template <class B>
__global__ void __launch_bounds__(256) k_multi(const __grid_constant__ MultiParams mp) {
  __shared__ uint4 sm[B::SMEM_ITEMS > 0 ? B::SMEM_ITEMS : 1];
  __shared__ int s_last;
  const MultiFlags& mf = mp.mf;
  if (mf.ready.n > 0) {
    // window open: tell every peer that the memory it is about to touch on my
    // side is ready (sent by the first CTAs, which are resident in any schedule),
    // and wait for the same promise from the peers whose memory I touch
    if ((int)threadIdx.x < mf.ready.n) {
      if (blockIdx.x < 8) flag_signal(mf.ready.remote[threadIdx.x], mf.ready.seq[threadIdx.x]);
      flag_wait(mf.ready.local[threadIdx.x], mf.ready.seq[threadIdx.x], mf.timeout_ns, mf.err);
    }
    __syncthreads();
  }
  const ull span = (ull)mp.nb * mp.max_total;
  for (ull g = blockIdx.x; g < span; g += gridDim.x) {
    const int b = (int)(g % (ull)mp.nb);
    const ull t = g / (ull)mp.nb;
    if (t < mp.kp[b].total) {  // uniform over the CTA
      B::run(mp.kp[b], t, sm);
      if (B::SYNC) __syncthreads();
    }
  }
  if (mf.done.n > 0) {
    // window close: the CTA that finishes last tells every peer that all my
    // accesses to its memory are complete (and, for puts, waits for the same
    // from them: only then is my own array complete)
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      const unsigned old = atomicAdd(mf.counter, 1u);
      s_last = (old == gridDim.x - 1);
      if (s_last) {
        *mf.counter = 0;  // ready for the next launch (stream-ordered after this one)
        __threadfence_system();
      }
    }
    __syncthreads();
    if (s_last && (int)threadIdx.x < mf.done.n) {
      flag_signal(mf.done.remote[threadIdx.x], mf.done.seq[threadIdx.x]);
      if (mf.wait_done)
        flag_wait(mf.done.local[threadIdx.x], mf.done.seq[threadIdx.x], mf.timeout_ns, mf.err);
    }
  }
}

// ---------------------------------------------------------------------------
static int pow2_of_ptr(const void* a) {
  uintptr_t v = (uintptr_t)a;
  int al = 1;
  while (al < 16 && (v % (2 * al)) == 0) al *= 2;
  return al;
}
static int ceil_log2(long long x) {
  int l = 0;
  while ((1LL << l) < x) ++l;
  return l;
}
static long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

static int sm_count() {
  static int n = [] {
    int dev = 0, v = 132;
    if (cudaGetDevice(&dev) == cudaSuccess)
      cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v > 0 ? v : 132;
  }();
  return n;
}

// which kernel a block runs under
enum Family { F_ROWS = 1, F_TRANS = 2, F_SCALAR = 3, F_BULK = 4 };
struct Sel {
  int fam = 0;
  int w = 0;    // rows: access width; trans / scalar: element size
  int tbq = 0;  // trans
  bool se = false, de = false;
  bool operator==(const Sel& o) const {
    return fam == o.fam && w == o.w && tbq == o.tbq && se == o.se && de == o.de;
  }
};

template <class B>
struct Tag {
  typedef B Body;
};

// calls f(Tag<Body>{}) for the body `sel` names
template <class F>
static pa_status dispatch(const Sel& sel, F&& f) {
  if (sel.fam == F_ROWS) {
    switch (sel.w) {
      case 16: return f(Tag<RowsBody<uint4, 3>>{});
      case 8: return f(Tag<RowsBody<uint2, 4>>{});
      case 4: return f(Tag<RowsBody<uint32_t, 4>>{});
      case 2: return f(Tag<RowsBody<uint16_t, 4>>{});
      default: return f(Tag<RowsBody<uint8_t, 4>>{});
    }
  }
  if (sel.fam == F_TRANS) {
    if (sel.w == 16) {
      if (sel.tbq == 16) return f(Tag<TransBody<16, 16, false, false>>{});
      return f(Tag<TransBody<16, 32, false, false>>{});
    }
#define PA_SEDE(S_, Q_)                                                           \
  (sel.se ? (sel.de ? f(Tag<TransBody<S_, Q_, true, true>>{})                     \
                    : f(Tag<TransBody<S_, Q_, true, false>>{}))                   \
          : (sel.de ? f(Tag<TransBody<S_, Q_, false, true>>{})                    \
                    : f(Tag<TransBody<S_, Q_, false, false>>{})))
    if (sel.w == 8) {
      if (sel.tbq == 16) return PA_SEDE(8, 16);
      return PA_SEDE(8, 32);
    }
    return PA_SEDE(4, 16);
#undef PA_SEDE
  }
  switch (sel.w) {
    case 16: return f(Tag<ScalarBody<uint4>>{});
    case 8: return f(Tag<ScalarBody<uint2>>{});
    case 4: return f(Tag<ScalarBody<uint32_t>>{});
    case 2: return f(Tag<ScalarBody<uint16_t>>{});
    case 1: return f(Tag<ScalarBody<uint8_t>>{});
  }
  set_error("unsupported element word size %d", sel.w);
  return PA_EINVAL;
}

// fills the launch parameters of one block and names its kernel
static pa_status prepare(const BlockCopy& b, const void* src, void* dst, KParams& p, Sel& sel,
                         int* vec_used) {
  if (!src || !dst) {
    set_error("null array pointer");
    return PA_EINVAL;
  }
  const long long S = b.elsize;
  const char* s = (const char*)src + b.src_off * S;
  char* d = (char*)dst + b.dst_off * S;
  const int spal = pow2_of_ptr(s), dpal = pow2_of_ptr(d);
  if (std::min(spal, dpal) < (S > 16 ? 16 : S)) {
    set_error("array pointers must be aligned to the element word size (%lld)", S);
    return PA_EINVAL;
  }
  memset(&p, 0, sizeof p);
  p.src = s;
  p.dst = d;
  const Dim X = b.d[0];
  const Dim Y = b.nd > 1 ? b.d[1] : Dim{1, 0, 0};
  p.ex = X.e;
  p.ey = Y.e;
  p.sx_s = X.ss * S;
  p.sx_d = X.ds * S;
  p.sy_s = Y.ss * S;
  p.sy_d = Y.ds * S;
  p.no = b.nd > 2 ? b.nd - 2 : 0;
  if (p.no > MAXO) {
    set_error("internal error: too many outer dims");
    return PA_EINVAL;
  }
  for (int i = 0; i < p.no; ++i) {
    p.oe[i] = b.d[i + 2].e;
    p.os[i] = b.d[i + 2].ss * S;
    p.od[i] = b.d[i + 2].ds * S;
  }
  const int sal = std::min(b.src_align, spal), dal = std::min(b.dst_align, dpal);

  if (b.klass == KC_ROWS) {
    const int W = std::min(sal, dal);
    const long long exv = X.e * S / W;
    p.ex = exv;
    const int ulog = W == 16 ? 3 : 4;
    int lxl = std::min(8, ceil_log2(exv));
    const long long LX = 1LL << lxl, LY = 256 >> lxl;
    int uxl = std::min(ulog, ceil_log2(cdiv(exv, LX)));
    p.lx_log2 = lxl;
    p.ux_log2 = uxl;
    p.tiles_x = (unsigned)cdiv(exv, LX << uxl);
    p.tiles_y = (unsigned)cdiv(Y.e, LY << (ulog - uxl));
    sel.fam = F_ROWS;
    sel.w = W;
    if (vec_used) *vec_used = W;
  } else if (b.klass == KC_TRANSPOSE && (S == 4 || S == 8 || S == 16)) {
    // destination-run length of a tile = TBQ*16 B.  256 B (TBQ = 16) by default: more,
    // smaller tiles -> shorter tail, fewer DRAM pages open per tile; tunable
    // "transpose_tbq" = 32 selects 512-B runs
    int tbq = g_tun.transpose_tbq == 32 && S != 4 ? 32 : 16;
    const int V = 16 / (int)S;
    p.tiles_x = (unsigned)cdiv(X.e, 32 * V);
    p.tiles_y = (unsigned)cdiv(Y.e, tbq * V);
    sel.fam = F_TRANS;
    sel.w = (int)S;
    sel.tbq = tbq;
    // Tile order.  Consecutive CTAs should complete the SHORT rows first: when the
    // destination rows are much shorter than the source rows (few tiles along Y, many
    // along X -- typically a 2-d transpose left after merging dims) walking along Y
    // first fills whole destination rows (full DRAM pages) instead of 256-byte pieces
    // of thousands of them (the r2c-shaped grids of bench.py).  Tunable
    // "transpose_y_fastest": -1 = this rule (default), 0 / 1 = forced.
    p.y_fastest = g_tun.transpose_y_fastest >= 0 ? g_tun.transpose_y_fastest
                                                 : (2ull * p.tiles_y <= (unsigned long long)p.tiles_x);
    sel.se = S < 16 && sal < 16;
    sel.de = S < 16 && dal < 16;
    if (vec_used) *vec_used = (sel.se || sel.de) ? (int)S : 16;
  } else {
    p.tiles_x = (unsigned)cdiv(X.e, 32);
    p.tiles_y = (unsigned)cdiv(Y.e, 32);
    sel.fam = F_SCALAR;
    sel.w = (int)S;
    if (vec_used) *vec_used = (int)S;
  }
  ull tiles = (ull)p.tiles_x * p.tiles_y;
  for (int i = 0; i < p.no; ++i) tiles *= (ull)p.oe[i];
  p.total = tiles;
  return PA_OK;
}

static pa_status launch_err(cudaError_t e) {
  set_error("kernel launch failed: %s", cudaGetErrorString(e));
  return e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? PA_ENOGPU : PA_ECUDA;
}

static pa_status launch_bulk(const BlockCopy& b, KParams& p, cudaStream_t st, int max_ctas) {
  static bool attr_set[64] = {false};  // the attribute is per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaFuncSetAttribute(k_rows_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         BULK_STAGES * BULK_CHUNK);
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const long long S = b.elsize;
  const long long run = b.d[0].e * S;
  const long long chunk = std::min<long long>(BULK_CHUNK, run);
  p.ex = run;
  p.lx_log2 = (int)chunk;
  p.tiles_x = (unsigned)cdiv(run, chunk);
  p.tiles_y = (unsigned)(b.nd > 1 ? b.d[1].e : 1);
  ull units = (ull)p.tiles_x * p.tiles_y;
  for (int i = 0; i < p.no; ++i) units *= (ull)p.oe[i];
  p.total = units;
  long long ctas = max_ctas > 0 ? max_ctas : (max_ctas < 0 ? -max_ctas : 3) * (long long)sm_count();
  if ((ull)ctas > units) ctas = (long long)units;
  cudaGetLastError();
  k_rows_bulk<<<(unsigned)ctas, 32, BULK_STAGES * BULK_CHUNK, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return launch_err(e);
  count_launch();
  return PA_OK;
}

// max_ctas: 0 = one tile per CTA; > 0 = capped, tile-striding grid;
//           < 0 = -max_ctas CTAs per SM (resolved against the device here)
pa_status launch_block(const BlockCopy& b, const void* src, void* dst, void* stream, int* vec_used,
                       int max_ctas, bool pdl) {
  if (vec_used) *vec_used = 0;
  if (b.klass == KC_EMPTY) return PA_OK;
  KParams p;
  Sel sel;
  pa_status rc = prepare(b, src, dst, p, sel, vec_used);
  if (rc != PA_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (p.total == 0) return PA_OK;
  if (sel.fam == F_ROWS && g_tun.bulk_rows && sel.w == 16) {
    if (vec_used) *vec_used = 16;
    return launch_bulk(b, p, st, max_ctas);
  }
  if (max_ctas < 0) max_ctas = -max_ctas * sm_count();
  // grids are limited to 2^31-1 CTAs: anything larger strides over its tiles
  if (p.total > 0x7fffffffULL && (max_ctas <= 0 || max_ctas > 0x7fffffff))
    max_ctas = 64 * sm_count();
  const bool loop = max_ctas > 0 && p.total > (ull)max_ctas;
  const unsigned grid = loop ? (unsigned)max_ctas : (unsigned)p.total;
  pdl = pdl && g_tun.pdl;
  return dispatch(sel, [&](auto tag) -> pa_status {
    typedef typename decltype(tag)::Body B;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    cudaError_t e = loop ? cudaLaunchKernelEx(&cfg, k_box<B, true>, p)
                         : cudaLaunchKernelEx(&cfg, k_box<B, false>, p);
    if (e != cudaSuccess) return launch_err(e);
    count_launch();
    return PA_OK;
  });
}

pa_status launch_multi(int nb, const BlockCopy* const* blocks, const void* const* srcs,
                       void* const* dsts, void* stream, int max_ctas, const MultiFlags* mf) {
  if (nb > FLAG_INLINE_MAX) return PA_EINCOMPAT;
  MultiParams mp;
  memset(&mp, 0, sizeof mp);
  Sel sel0;
  bool have = false;
  for (int i = 0; i < nb; ++i) {
    if (blocks[i]->klass == KC_EMPTY) continue;
    KParams p;
    Sel sel;
    pa_status rc = prepare(*blocks[i], srcs[i], dsts[i], p, sel, nullptr);
    if (rc != PA_OK) return rc;
    if (p.total == 0) continue;
    if (p.total > 0x7fffffffULL) return PA_EINCOMPAT;
    if (have && !(sel == sel0)) return PA_EINCOMPAT;  // caller falls back to per-block launches
    sel0 = sel;
    have = true;
    mp.kp[mp.nb++] = p;
    mp.max_total = std::max(mp.max_total, p.total);
  }
  if (mf) mp.mf = *mf;
  if (!have) {
    if (!mf || (mf->ready.n == 0 && mf->done.n == 0)) return PA_OK;
    // nothing to move, but the protocol still has to be spoken
    sel0.fam = F_ROWS;
    sel0.w = 16;
    mp.nb = 0;
    mp.max_total = 0;
  }
  if (max_ctas < 0) max_ctas = -max_ctas * sm_count();
  const ull span = (ull)mp.nb * mp.max_total;
  ull grid = span;
  if (max_ctas > 0 && grid > (ull)max_ctas) grid = (ull)max_ctas;
  if (grid > (ull)64 * sm_count()) grid = (ull)64 * sm_count();
  if (grid == 0) grid = 1;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch(sel0, [&](auto tag) -> pa_status {
    typedef typename decltype(tag)::Body B;
    cudaGetLastError();
    k_multi<B><<<(unsigned)grid, 256, 0, st>>>(mp);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return launch_err(e);
    count_launch();
    return PA_OK;
  });
}

int device_count() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

}  // namespace pa
