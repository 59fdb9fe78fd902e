// Internal structures of libpa_b200: geometry, plan, kernel descriptors.
// Everything here is host-side integer arithmetic; indices are 0-BASED and
// ranges half-open [lo, hi) internally (the C ABI converts from/to Julia's
// 1-based inclusive convention).
#pragma once
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/pa_b200.h"

namespace pa {

using i64 = int64_t;

// ---- error plumbing --------------------------------------------------------
void set_error(const char* fmt, ...);
const char* last_error();

// return a failed status to the caller
#define RC(call)                    \
  do {                              \
    pa_status rc_ = (call);         \
    if (rc_ != PA_OK) return rc_;   \
  } while (0)

// ---- MPITopology (MPITopologies.jl:72-119) ---------------------------------
struct Topology {
  int M = 0;
  i64 dims[PA_MAX_TOPO] = {0};
  int rank = 0;
  int size = 1;
  i64 coords[PA_MAX_TOPO] = {0};  // 0-based coords of `rank`

  // rank <-> coords, row-major (last coordinate fastest):
  // MPI_Cart_create(reorder=false), MPITopologies.jl:125-131,208-226
  void coords_of(int r, i64* c) const;
  int rank_of(const i64* c) const;
  bool same_as(const Topology& o) const;
};

// ---- staging arenas shared by a pencil family (Pencils.jl:185-189,265-270) -
struct Buffers {
  void* send = nullptr;
  i64 send_cap = 0;
  void* recv = nullptr;
  i64 recv_cap = 0;
  void* comm_done_event = nullptr;    // cudaEvent_t of the last exchange using them
  void* unpack_done_event = nullptr;  // cudaEvent_t of the last unpack that READ recv (or wrote it locally)
  unsigned long long generation = 0;  // bumped whenever an arena is (re)allocated: stale peer windows are refused
  // NCCL user-buffer registration (tunable "nccl_register"): arenas come from
  // ncclMemAlloc and are registered with the communicator so that ncclSend /
  // ncclRecv can go zero-copy over NVLink instead of through NCCL's staging FIFO
  bool send_nccl = false, recv_nccl = false;  // allocated with ncclMemAlloc
  void* reg_comm = nullptr;                   // ncclComm_t the arenas are registered with
  void* reg_send = nullptr;                   // registration handles
  void* reg_recv = nullptr;
  void* reg_send_ptr = nullptr;               // the pointers that were registered
  void* reg_recv_ptr = nullptr;
  ~Buffers();
  pa_status reserve(i64 send_bytes, i64 recv_bytes);
};

// ---- Pencil (Pencils.jl:151-272) -------------------------------------------
struct Pencil {
  std::shared_ptr<Topology> topo;
  int N = 0;
  i64 size_global[PA_MAX_DIMS] = {0};
  int decomp[PA_MAX_TOPO] = {0};  // 0-based array dim decomposed by grid dim i
  int perm[PA_MAX_DIMS] = {0};    // 0-based; memory dim i holds logical dim perm[i]
  bool perm_identity = true;
  std::shared_ptr<Buffers> bufs;

  // axes_all[coords] in logical order (data_ranges.jl:4-9,30-45)
  void range_of(const i64* coords, i64* lo, i64* hi) const;
  void range_local(i64* lo, i64* hi) const { range_of(topo->coords, lo, hi); }
};

// block partition rule, 0-based half-open restatement of
// local_data_range(p, P, N) = (N(p-1))÷P + 1 : (N p)÷P   (data_ranges.jl:4-9)
inline void local_data_range(i64 p0, i64 P, i64 N, i64* lo, i64* hi) {
  *lo = (N * p0) / P;
  *hi = (N * (p0 + 1)) / P;
}

// ---- strided box copy: the one primitive all kernels implement -------------
struct Dim {
  i64 e;   // extent (elements)
  i64 ss;  // source stride (elements)
  i64 ds;  // destination stride (elements)
};

enum KernelClass { KC_EMPTY = 0, KC_ROWS = 1, KC_TRANSPOSE = 2, KC_TILE_SCALAR = 3 };

// Canonical, launch-ready description of `dst[off_d + sum k_i ds_i] =
// src[off_s + sum k_i ss_i]` for k in the box.  dims[0] = X (smallest source
// stride), dims[1] = Y (the tile's second dim), the rest are outer dims.
struct BlockCopy {
  // as given (source memory order), kept for pa_plan_get_block; one spare slot for
  // the innermost word pseudo-dimension of non-power-of-two element sizes
  int nd_raw = 0;
  Dim raw[PA_MAX_DIMS + 1];
  i64 src_off = 0, dst_off = 0;  // elements
  int elsize = 0;
  i64 count = 0;                 // elements in the box

  // canonical form
  int nd = 0;
  Dim d[PA_MAX_DIMS + 1];
  int klass = KC_EMPTY;
  int stride_align = 16;  // largest power of two (<=16) dividing every byte stride / run length
  int src_align = 16;     // same, source side only (row starts / run lengths of the loads)
  int dst_align = 16;     // same, destination side only
  bool contiguous_both = false;  // whole block is one contiguous run on both sides
};

void canonicalize(BlockCopy& b);
// sub-block [c0, c1) of the OUTERMOST raw dim with extent > 1 (chunked pipelining of
// a peer block: the chunk is a contiguous sub-range of the dense side); returns the
// element offset of the chunk inside the dense side through *dense_off, its length
// through *dense_cnt
BlockCopy sub_block(const BlockCopy& b, int part, int nparts, bool dense_is_dst, i64* dense_off,
                    i64* dense_cnt);

// launch on `stream`; src/dst are array base pointers (offsets come from b)
// max_ctas > 0 caps the grid (CTAs then stride over the tiles): used for the
// NVLink-bound remote kernels so that they leave SMs to concurrent local work.
pa_status launch_block(const BlockCopy& b, const void* src, void* dst, void* stream,
                       int* vec_used, int max_ctas = 0, bool pdl = false);

// Flag words of the one-sided protocols (NVLink signals between the ranks of a
// grid line): a set of (peer's word for me, my word for the peer, sequence number).
constexpr int FLAG_INLINE_MAX = 8;  // peers handled inside one multi-peer launch (one NVSwitch box: <= 7)
struct FlagSet {
  int n;
  unsigned long long* remote[FLAG_INLINE_MAX];
  unsigned long long* local[FLAG_INLINE_MAX];
  unsigned long long seq[FLAG_INLINE_MAX];
};
struct MultiFlags {
  FlagSet ready;  // prologue: signal + wait ("the other side of every block may be touched")
  FlagSet done;   // epilogue: the last CTA signals ("all my blocks have landed / been read")
  int wait_done;           // the last CTA also waits for every peer's `done` before exiting
  unsigned int* counter;   // device word counting finished CTAs (reset by the last one)
  unsigned long long timeout_ns;
  int* err;
};
// ONE launch executing up to FLAG_INLINE_MAX box copies of the same kernel flavour,
// tiles interleaved round-robin over the blocks so that every destination link is
// driven at once; optional in-kernel ready/done protocol (mf may be NULL).
// Returns PA_EINCOMPAT (without launching) when the blocks need different kernels.
pa_status launch_multi(int nb, const BlockCopy* const* blocks, const void* const* srcs,
                       void* const* dsts, void* stream, int max_ctas, const MultiFlags* mf);

// run-time tunables (pa_set_tunable)
struct Tunables {
  int remote_ctas = -4;   // grid cap of put/get kernels: n > 0 CTAs, n < 0 = |n| per SM, 0 = uncapped
                          // (a few CTAs per SM drive the links; the rest stay free for local work)
  int box_copy_ctas = 0;  // grid cap applied to pa_box_copy (benchmarks)
  int transpose_y_fastest = -1;  // transpose tile order: 1 = consecutive CTAs along the destination rows,
                                 // 0 = along the source rows, -1 = along the side with fewer tiles (kernels.cu)
  int transpose_tbq = 0;  // 16-byte items per destination run of a transpose tile: 0 / 16 = 256-byte runs
                          // (default: best or tied on every measured shape), 32 = 512-byte runs
  long long small_block_bytes = 256ll << 20;  // (kept for ABI compatibility of pa_set_tunable; unused)
  int bulk_rows = 0;     // 1: row copies run as the TMA bulk-copy pipeline (k_rows_bulk)
  int nccl_register = 1;  // staging arenas from ncclMemAlloc + ncclCommRegister (registered NCCL p2p:
                          // exchange 637 -> 673 GB/s at N=2); falls back to cudaMalloc when unavailable
  int nccl_fences = 0;   // 1: one-sided paths fence with NCCL groups even when the flag window exists
  int oneside_self_ctas = 0;  // grid cap of the self block (K3) while the one-sided puts / gets run
                              // beside it (0 = uncapped, < 0 per SM): trades K3 speed for NVLink rate
  int fft_lines = 0;     // fused unpack+FFT: 4 = four lines per CTA for 256/512-point lines too (default 8)
  int multi_put = 1;     // 1: one launch interleaving every peer's tiles (+ in-kernel flags) on the one-sided paths
  int p2p_chunks = 1;    // staged schedules: sub-blocks per peer block (pack-chunk -> send-chunk -> unpack-chunk)
  int self_first = 0;    // staged schedules: 1 = self block first and beside the packs (round-1 order)
  int staged_ctas = 0;   // grid cap of pack/unpack kernels while an exchange is in flight (0 = uncapped, <0 per SM)
  int ipc_exchange = 0;  // 1: staged schedules move the blocks with this library's own NVLink copy kernels
                         //    (peer-mapped recv_buf + flag signals) even when an NCCL communicator exists
  long long fence_timeout_ms = 60000;  // a flag wait longer than this sets the error word and traps
  int pdl = 1;           // programmatic dependent launch between the back-to-back kernels of a chain
  int nccl_ctas = 0;     // > 0: ncclCommInitRankConfig min/maxCTAs
  long long host_chunk_bytes = 64ll << 20;  // pa_transpose_host: bytes per pipelined chunk
  int host_slots = 2;    // pa_host_chain: device staging sets = submits that may be in flight (2..4)
};
extern Tunables g_tun;

// ---- Transposition plan (Transpositions.jl:69-119, 281-343) ----------------
struct Peer {
  int world_rank = -1;
  bool is_self = false;
  i64 send_off = 0, send_cnt = 0;  // elements
  i64 recv_off = 0, recv_cnt = 0;  // elements
  BlockCopy pack;    // K1: src parent box -> contiguous @ (send_off | recv_off)
  BlockCopy unpack;  // K2: contiguous @ recv_off -> dest parent box
  BlockCopy put;     // K1-put: src parent box -> the PEER's dest parent (its layout), no staging
  BlockCopy get;     // K2-get: the PEER's src parent box (its layout) -> dest parent box
  i64 remote_recv_off = 0;  // elements: where MY block starts inside the PEER's recv_buf
};

struct TransposeState;  // streams/events, defined in transpose.cpp

// one cached answer of plan_check: valid while `key` is the tunable it depends on (-1: not asked)
struct Verdict {
  int key = -1;
  pa_status status = PA_OK;
  std::string err;  // last_error() of a refusal
};

struct Plan {
  std::shared_ptr<Pencil> pin, pout;
  int n_extra = 0;
  i64 extra[PA_MAX_DIMS] = {0};
  i64 prod_extra = 1;
  int elsize = 0;
  int method = PA_POINT_TO_POINT;
  int dim = -1;  // grid dim of the exchange (0-based), -1 = local only
  int nproc = 1;
  int self_index = 0;  // 0-based
  bool same_perm = false;
  i64 length_in = 0, length_out = 0, length_self = 0;
  i64 send_elems = 0, recv_elems = 0;
  std::vector<Peer> peers;
  BlockCopy self_fused;  // K3: src parent -> dest parent (self block or local permute)
  TransposeState* st = nullptr;
  // PeerPut windows: local dest base pointer -> peer-mapped dest base pointers
  // (indexed by position in the grid line; nullptr for self)
  std::map<const void*, std::vector<void*>> windows;
  // windows on the peers' recv_buf arenas (own-kernel exchange of the staged schedules)
  std::vector<void*> recv_windows;
  unsigned long long recv_windows_gen = 0;  // generation of MY arenas when they were registered
  // host-transpose staging
  void* h_src_dev = nullptr;
  void* h_dst_dev = nullptr;
  i64 h_src_cap = 0, h_dst_cap = 0;
  // cached answers of plan_check, [question][0: Float64 / ComplexF64, 1: PA_FFT_F32]
  Verdict verdicts[6][2];
  ~Plan();
};

pa_status build_plan(std::shared_ptr<Pencil> pin, std::shared_ptr<Pencil> pout, int n_extra,
                     const i64* extra, int elsize, int method, Plan** out);

// ---- communicator ----------------------------------------------------------
struct Comm;
pa_status comm_unique_id(void* id128);
pa_status comm_init(const void* id128, int nranks, int rank, Comm** out);
pa_status comm_init_local(int nranks, int rank, Comm** out);  // no NCCL: flag window + peer mappings only
void comm_destroy(Comm* c);
pa_status comm_flags_export(Comm* c, void* handle64, i64* offset);
pa_status comm_flags_import(Comm* c, int rank, const void* handle64, i64 offset);

// What a reduction (reduce.cu) needs of a communicator.  The flag window carries the combine: the
// words of kind FK_REDUCE and, behind all the words, two sets (the parity of the call) of one
// 16-byte slot per source rank.
constexpr int REDUCE_SLOT_BYTES = 16;
struct ReduceState;  // workspace + serialising event of the reductions on one communicator
struct ReduceWindow {
  int nranks = 1, rank = 0;
  bool flags = false;   // the flag window is mapped everywhere and not overridden by nccl_fences
  bool nccl = false;    // an NCCL communicator exists (the fallback when !flags)
  unsigned long long* local_words = nullptr;      // word from rank r: local_words[r * word_stride]
  int word_stride = 0;
  unsigned char* local_slots = nullptr;           // slot [parity][r] at (parity * nranks + r) * 16
  int* err = nullptr;
  unsigned long long timeout_ns = 0;
  ReduceState** state = nullptr;  // owned by the communicator
};
pa_status comm_reduce_window(Comm* c, ReduceWindow* w);
int comm_size(const Comm* c);
// ncclAllGather of `bytes` per rank (the reductions' fallback without a flag window)
pa_status comm_allgather(Comm* c, const void* send, void* recv, size_t bytes, void* stream);
// a communicator's reduction state, made with the communicator (synchronous); its window tables
// uploaded once the flag window is mapped everywhere
pa_status reduce_state_create(int nranks, ReduceState** out);
pa_status reduce_state_set_tables(ReduceState* s, int nranks, unsigned long long* const* remote_words,
                                  unsigned char* const* peer_slots);
void reduce_state_destroy(ReduceState* s);
// the reduction itself (reduce.cu); every argument has been checked.  comm NULL: one rank
pa_status reduce(Comm* comm, int dtype, int map, int op, const void* pred_value, i64 n,
                 const void* a, const void* b, void* result, void* stream);

// What a fused line kernel computes: from the lines it gathers on the receive side of a
// transposition (unpack_fused, get_fft) or from the source lines it loads on the send side
// (put_fft).  A plan moves the elements of one side; the array on the other side of the transform
// may have the other element type.
enum class FusedMode {
  fft,    // the complex FFT: complex arrays on both sides
  rfft,   // N reals -> N/2 + 1 complex bins
  r2r,    // N reals -> N reals, a DCT / DST
  brfft,  // N/2 + 1 complex bins -> N reals
};
enum class Side { unpack, put };
// What a fused line kernel computes, and on which side of the exchange.  The entry points decode
// it from their flags (and r2r's kind) and check it once; below them flags carry the schedule bits
// only (PA_WAITALL, PA_NO_OVERLAP, PA_STAGE_SELF).
struct LineOp {
  Side side;       // unpack: unpack_fused / get_fft; put: put_fft
  FusedMode mode;
  int sign;        // fft only: -1 forward, +1 backward (0 otherwise: no kernel reads it)
  int r2r_kind;    // r2r only: PA_REDFT10 / PA_REDFT01 / PA_RODFT10 / PA_RODFT01
  bool f32;        // PA_FFT_F32: single precision
};
// the plan moves reals: the destination's on the receive side, the source's on the send side
inline bool unpack_moves_reals(FusedMode m) { return m == FusedMode::r2r || m == FusedMode::rfft; }
inline bool put_moves_reals(FusedMode m) { return m == FusedMode::r2r || m == FusedMode::brfft; }

// FFTW's r2r kinds: PA_REDFT10 (DCT-II) and PA_RODFT10 (DST-II) run forward, PA_REDFT01 (DCT-III)
// and PA_RODFT01 (DST-III) backward; the RODFT kinds are the sine transforms
inline bool r2r_forward(int kind) { return kind == PA_REDFT10 || kind == PA_RODFT10; }
inline bool r2r_sine(int kind) { return kind == PA_RODFT10 || kind == PA_RODFT01; }

// dst = transpose(src); op (NULL: none) fuses a line transform into it: op->side unpack, dst =
// T(transpose(src)) through the fused unpack; put, dst = transpose(T(src)) on the caller's stream
// (local plans) or PeerPut's one-sided schedule.  Every argument has been checked.
pa_status transpose(Plan* plan, Comm* comm, const void* src, void* dst, unsigned flags,
                    void* stream, const LineOp* op = nullptr);
// pa_transpose's fused FFT (capi.cpp): the PA_FFT_* bits of flags decoded into *op and checked
// (the plan's verdict, the alias rule); *fused = false when flags hold none
pa_status transpose_fft_op(Plan* plan, unsigned flags, const void* src, const void* dst, LineOp* op,
                           bool* fused);
pa_status wait_sends(Plan* plan, void* stream);
pa_status permute_local(Plan* plan, const void* src, void* dst, void* scratch, void* stream);
pa_status transpose_host(Plan* plan, Comm* comm, const void* hsrc, void* hdst, unsigned flags);
pa_status plan_timings(Plan* plan, pa_timings* t);
pa_status plan_enable_timing(Plan* plan, int on);
void destroy_state(TransposeState* st);

// CUDA IPC plumbing of the PeerPut method (one-sided puts over NVLink)
pa_status ipc_export(const void* devptr, void* handle64, i64* offset);
pa_status ipc_import(const void* handle64, i64 offset, void** mapped);
pa_status ipc_release_handle(const void* handle64);
pa_status plan_set_window(Plan* plan, const void* local_dst, int n0, void* peer_dst);
pa_status plan_set_recv_window(Plan* plan, int n0, void* peer_recv_buf);

// host pipelines (pa_host_chain_*)
struct HostChain;
pa_status host_chain_create(int n, Plan* const* plans, Comm* comm, HostChain** out);
void host_chain_destroy(HostChain* c);
pa_status host_chain_submit(HostChain* c, const void* hsrc, void* hdst, i64* ticket);
pa_status host_chain_wait(HostChain* c, i64 ticket);
pa_status host_chain_buffer(HostChain* c, int slot, int which, void** p, i64* bytes);
pa_status host_chain_time_begin(HostChain* c);
pa_status host_chain_time_end(HostChain* c, float* ms);

// fused unpack + line transform op along the destination's contiguous dim (fft.cu, k_unpack_fft /
// k_unpack_rfft / k_unpack_r2r / k_unpack_brfft): the blocks together tile the destination box;
// srcs[i] = base pointer blocks[i] reads from.  The plan's elements: fft ComplexF64, rfft / r2r
// Float64, brfft ComplexF64, or their single-precision counterparts with op.f32.  rfft: `dst` is
// the complex array of N/2 + 1 bins per line that replaces the real destination (same layout
// otherwise); brfft: `dst` is the real array of N reals per line that replaces the complex one
pa_status unpack_fused(int nb, const BlockCopy* const* blocks, const void* const* srcs, void* dst,
                       const LineOp& op, void* stream);
// the complex FFT's kernel one-sided (fft.cu, k_get_fft): srcs[i] are the peers' src arrays as
// mapped here (the self block's: the local src), read in place, and `mf` (NULL: none) the window
// protocol spoken inside the launch.  *launched = false: this rank has no destination lines and
// nothing was launched -- the caller then speaks the protocol with flag kernels
pa_status get_fft(int nb, const BlockCopy* const* blocks, const void* const* srcs, void* dst,
                  const LineOp& op, const MultiFlags* mf, void* stream, bool* launched);
// send-side fused transform + put (fft.cu, k_fft_put / k_rfft_put / k_r2r_put / k_brfft_put): the
// transform along the first memory dim of the local `src`, every output element stored into the
// block that owns it.  blocks[i] / dsts[i]: the self block (self_fused) into the local dst, the put
// block of every other rank into that rank's dst as mapped here.  `mf` (NULL: none): the window
// protocol spoken inside the launch.  *launched = false: this rank has no source lines and nothing
// was launched -- the caller then speaks the protocol with flag kernels
pa_status put_fft(int nb, const BlockCopy* const* blocks, const void* src, void* const* dsts,
                  const LineOp& op, const MultiFlags* mf, void* stream, bool* launched);
// Can the fused kernel of `mode` run on this plan, on the receive side (unpack_fused; the complex
// FFT of a PeerGet plan: get_fft too) or on the send side (put_fft: PeerPut plans and local
// transposes only)?  The same answer on every rank of the grid line (global geometry only);
// PA_EINVAL + last_error otherwise.  Cached per plan, side, transform and precision; r2r shares
// the answer of rfft (receive side) or brfft (send side).  No device call.
pa_status plan_check(Plan* plan, Side side, FusedMode mode, bool f32);
// real-line transforms (fft.cu): `nlines` dense, consecutive lines of N reals (src when forward,
// dst when backward) <-> N/2 + 1 complex bins; N a power of two in 16..2048.  f32: Float32 <->
// ComplexF32, else Float64 <-> ComplexF64
pa_status rfft_lines(int N, bool forward, bool f32, i64 nlines, const void* src, void* dst,
                     void* stream);
// real-to-real line transforms (fft.cu, k_r2r): `nlines` dense, consecutive lines of N reals on
// both sides (src == dst allowed).  forward: DCT-II (sine: DST-II), else DCT-III (sine: DST-III),
// unnormalised as FFTW's REDFT10 / RODFT10 / REDFT01 / RODFT01; N a power of two in 16..2048.
// f32: Float32, else Float64
pa_status r2r_lines(int N, bool forward, bool sine, bool f32, i64 nlines, const void* src, void* dst,
                    void* stream);

// standalone flag step on `stream`: signal the n remote words (monotonic max,
// release at system scope) and/or wait for the n local words to reach seq
pa_status launch_flags(int n, unsigned long long* const* remote, unsigned long long* const* local,
                       const unsigned long long* seq, bool do_signal, bool do_wait,
                       unsigned long long timeout_ns, int* err, void* stream);

// PencilIO binary layout (io.cpp)
pa_status io_sizes(const Pencil& P, int n_extra, const i64* extra, int elsize, int chunks,
                   i64* global_bytes, i64* local_bytes, i64* nruns, i64* run_bytes, i64* first_offset);
pa_status io_run_offset(const Pencil& P, int n_extra, const i64* extra, int elsize, int chunks, i64 run,
                        i64* file_offset);
pa_status io_transfer(const Pencil& P, int n_extra, const i64* extra, int elsize, int chunks, void* dev,
                      const char* path, i64 offset, bool write);

int device_count();
pa_status set_device(int dev);
i64 launch_count();
void count_launch();

}  // namespace pa

struct pa_topology { std::shared_ptr<pa::Topology> p; };
struct pa_pencil { std::shared_ptr<pa::Pencil> p; };
struct pa_plan { pa::Plan* p; };
struct pa_comm { pa::Comm* p; };
struct pa_host_chain { pa::HostChain* p; };
