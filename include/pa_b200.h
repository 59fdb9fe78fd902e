/*
 * pa_b200.h -- C ABI of the H100-native global-transposition hot path.
 *
 * This is the drop-in boundary for the `transpose!` path of PencilArrays.jl
 * (reference: src/Transpositions/Transpositions.jl).  The reference has no
 * FFI of its own: its seam is Julia multiple dispatch on the array type
 * carried by a `Pencil` (Pencils.jl:282-304).  A device array type plugs in
 * by providing the "generic" methods `copy_range!` (Transpositions.jl:568-583),
 * `_viewreshape` (:615-623), `_permutedims!` (:648-664) and the transport
 * pair `transpose_send_other!` / `MPI.Alltoallv!` / `MPI.Waitany`
 * (:462-484, :422, :513).  Each entry point below names the reference
 * function it replaces.  `INTEGRATION.md` shows the Julia `ccall` stubs.
 *
 * Conventions
 *  - plain C: opaque handles, `int64_t` sizes, `void*` device pointers,
 *    `void*` for `cudaStream_t`; no torch / C++ types cross this boundary;
 *  - dimension indices, permutations, ranges and peer indices are 1-BASED and
 *    ranges are inclusive, exactly as the Julia reference passes them;
 *  - every function returns a `pa_status`; nothing throws across the ABI.
 *    The Julia veneer maps PA_EINVAL / PA_EINCOMPAT to `ArgumentError` and
 *    PA_EDIM to `DimensionMismatch` (Transpositions.jl:99-103,181-198;
 *    arrays.jl:108-114);
 *  - there is NO CPU fallback: every data-path call fails with PA_ENOGPU /
 *    PA_ECUDA when no device is usable.
 */
#ifndef PA_B200_H
#define PA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PA_MAX_DIMS 8        /* spatial + extra dims of one array           */
#define PA_MAX_TOPO 7        /* dims of the process grid (M < N)            */
#define PA_UNIQUE_ID_BYTES 128

typedef enum pa_status {
  PA_OK = 0,
  PA_EINVAL = 1,     /* bad argument                      -> ArgumentError      */
  PA_EINCOMPAT = 2,  /* pencils not transposable          -> ArgumentError      */
  PA_EDIM = 3,       /* array does not match its pencil   -> DimensionMismatch  */
  PA_ECUDA = 4,      /* CUDA runtime error (see pa_last_error)                  */
  PA_ENCCL = 5,      /* NCCL error / NCCL library not loadable                  */
  PA_ENOMEM = 6,     /* device or host allocation failed                        */
  PA_ESTATE = 7,     /* call sequence error (e.g. comm missing for Nproc > 1)   */
  PA_ENOGPU = 8      /* no CUDA device: the data path has no CPU fallback       */
} pa_status;

typedef enum pa_method {
  PA_POINT_TO_POINT = 0, /* Transpositions.PointToPoint  (Transpositions.jl:18) */
  PA_ALLTOALLV = 1,      /* Transpositions.Alltoallv     (Transpositions.jl:19) */
  PA_PEER_PUT = 2,       /* GPU extension (no reference counterpart): one-sided puts.
                            The pack kernel of each remote block stores straight into
                            the destination rank's `dest` array over NVLink (peer-mapped
                            memory): no send_buf, no recv_buf, no unpack pass.  Needs
                            pa_plan_set_window for `dest`; falls back to PointToPoint
                            when src and dest alias.                                   */
  PA_PEER_GET = 3        /* same, pull flavour: the unpack kernel of each remote block
                            LOADS straight out of the source rank's `src` array over
                            NVLink and stores permuted into the local `dest`.  Needs
                            pa_plan_set_window for `src`.                              */
} pa_method;

/* flags of pa_transpose */
#define PA_WAITALL   1u  /* transpose!(t; waitall=true)   (Transpositions.jl:170-176) */
#define PA_NO_OVERLAP 2u /* run pack -> exchange -> unpack strictly in sequence      */
#define PA_STAGE_SELF 4u /* self block through recv_buf like the reference (:393-403)
                            instead of the fused src->dest kernel                    */
/* Fused neighbour step (SURVEY §8 f2): the unpack of ALL blocks and a 1-d complex FFT
 * along the destination's contiguous dimension (the one that has just become local:
 * the reason the pencil is permuted, docs/src/Pencils.md:210-214) run as ONE kernel --
 * `dst` receives fft(transposed array) (forward: exp(-2*pi*i*jk/n); backward: the
 * unnormalised inverse, as FFTW / PencilFFTs).  ComplexF64 (or ComplexF32 with
 * PA_FFT_F32), power-of-two lines of 8..1024 points, staged methods, PA_PEER_GET or local
 * transposes, src and dst not aliased;
 * PA_EINVAL otherwise (transpose, then transform, separately; PA_PEER_PUT has no pass to
 * fuse with).  On a PA_PEER_GET plan the fused step is ONE kernel per rank that gathers every
 * line straight out of the peers' src arrays (and the local src), transforms and stores it,
 * with the window protocol inside the launch; without PA_WAITALL only the wait that guards
 * the reuse of src is deferred to pa_wait, as for the plain PeerGet.  A plan between
 * IDENTICAL pencils with src == dst is the plain in-place transform along the
 * contiguous dim -- the first step of a PencilFFTs-style 3-d transform, whose other
 * two steps are the fused transposes.                                               */
#define PA_FFT_FORWARD  8u
#define PA_FFT_BACKWARD 16u
/* Single precision, with PA_FFT_FORWARD / PA_FFT_BACKWARD only: on pa_transpose the
 * elements are ComplexF32 (the plan's elsize must be 8; elsize 16 is PA_EINVAL), on
 * pa_rfft the pair is Float32 <-> ComplexF32.  Storage and arithmetic are fp32.  The
 * element size alone never selects it: without this flag an elsize-8 plan is refused
 * for a fused FFT as before.                                                         */
#define PA_FFT_F32      32u

typedef struct pa_topology pa_topology; /* MPITopology   (MPITopologies.jl:72-119) */
typedef struct pa_pencil pa_pencil;     /* Pencil        (Pencils.jl:151-272)      */
typedef struct pa_plan pa_plan;         /* Transposition (Transpositions.jl:69-119)*/
typedef struct pa_comm pa_comm;         /* communicator standing in for
                                           topology.comm / subcomms               */
typedef struct pa_host_chain pa_host_chain; /* asynchronous upload -> transpose!... ->
                                           download pipeline for host arrays      */

/* ---- library ------------------------------------------------------------- */
const char* pa_version(void);
const char* pa_strerror(pa_status s);
/* detail text of the last failure on the calling thread ("" if none) */
const char* pa_last_error(void);
/* number of CUDA kernels this library has launched in this process */
int64_t pa_launch_count(void);
/* number of visible CUDA devices (0 on a CPU-only box); never fails */
int pa_device_count(void);
/* run-time tunables: "remote_ctas" = grid cap of the PeerPut/PeerGet kernels
 * (they are NVLink-bound; a capped, tile-striding grid leaves SMs to the local
 * kernels running beside them; n > 0 = n CTAs, n < 0 = |n| CTAs per SM (default
 * -4), 0 = uncapped), "box_copy_ctas" = same cap for pa_box_copy (benchmarks),
 * "nccl_fences" = 1: one-sided methods fence with NCCL groups, "nccl_register"
 * (default 1; 0 = plain cudaMalloc arenas): staging arenas from ncclMemAlloc +
 * ncclCommRegister, "bulk_rows" = 1: row copies as the TMA bulk-copy pipeline,
 * "transpose_tbq" (0/16 = 256-byte destination runs per tile, the default; 32 = 512),
 * "transpose_y_fastest" (-1 = consecutive CTAs walk along the side with fewer tiles,
 * the default; 0 / 1 = forced along source / destination rows), "small_block_bytes"
 * (accepted, unused since round 2),
 * "multi_put" (default 1): the one-sided methods issue ONE launch over all peers'
 * blocks with the window protocol inside the kernel, "p2p_chunks" (default 1):
 * sub-blocks per peer block flowing pack -> exchange -> unpack independently
 * (must be equal on all ranks), "staged_ctas": grid cap of pack/unpack kernels
 * while an exchange is in flight, "ipc_exchange" = 1: the staged methods move the
 * blocks with this library's own NVLink copy kernels instead of ncclSend/ncclRecv,
 * "fence_timeout_ms" (default 60000): a flag wait longer than this records the
 * failure and traps, "pdl" (default 1): programmatic dependent launch between
 * back-to-back local kernels, "nccl_ctas": ncclCommInitRankConfig min/maxCTAs,
 * "host_chunk_bytes": bytes per pipelined cut of the host paths, "host_slots" (2..4):
 * device staging sets = submits a pa_host_chain keeps in flight, "self_first" = 1:
 * staged schedules run the self block first and beside the packs (round-1 order;
 * default: remote packs first and alone), "oneside_self_ctas": grid cap of the self
 * block while the one-sided puts run beside it (default 0 = uncapped, measured best),
 * "fft_lines" = 4: the fused unpack+FFT uses four lines per CTA for 256/512-point
 * lines too (default eight, measured faster).                                     */
pa_status pa_set_tunable(const char* name, int64_t value);
/* bind the calling thread to a device (one process per GPU: LOCAL_RANK).  All
 * handles created afterwards (streams, staging arenas, communicator) live there. */
pa_status pa_set_device(int device);

/* ---- MPITopology ---------------------------------------------------------
 * Row-major rank grid, identical to MPI_Cart_create(reorder=false)
 * (MPITopologies.jl:125-131,208-226): the LAST coordinate varies fastest.   */
pa_status pa_dims_create(int nprocs, int M, int64_t* dims /* out[M] */);
        /* balanced, non-increasing factorisation: MPI_Dims_create analogue
           (MPITopologies.jl:138-144)                                        */
pa_status pa_topology_create(int M, const int64_t* dims, int world_rank,
                             pa_topology** out);
void pa_topology_destroy(pa_topology* t);
pa_status pa_topology_info(const pa_topology* t, int* M, int64_t* dims /*[M]*/,
                           int* world_rank, int* world_size,
                           int64_t* coords_local /*[M], 1-based*/);
pa_status pa_topology_rank_of(const pa_topology* t,
                              const int64_t* coords /*1-based*/, int* rank);
/* world ranks of the grid line through the local coords along grid dim R
 * (1-based) -- `subcomm_ranks[R]` + `get_remote_indices`
 * (Transpositions.jl:293-299,539-549)                                       */
pa_status pa_topology_line(const pa_topology* t, int R, int* ranks /*[dims[R]]*/);

/* ---- Pencil -------------------------------------------------------------- */
/* `share_with` != NULL reproduces Pencil(p; decomp_dims, permute): the new
 * pencil shares send_buf / recv_buf with `share_with` (Pencils.jl:257-271). */
pa_status pa_pencil_create(pa_topology* topo, int N, const int64_t* size_global,
                           const int* decomp_dims /*[M], 1-based*/,
                           const int* perm /*[N], 1-based; NULL = NoPermutation*/,
                           pa_pencil* share_with, pa_pencil** out);
void pa_pencil_destroy(pa_pencil* p);
/* range_local / range_remote (Pencils.jl:472-497): `coords` NULL = local rank;
 * memory_order != 0 applies the pencil's permutation. lo/hi 1-based inclusive
 * (hi = lo - 1 for an empty range).                                          */
pa_status pa_pencil_range(const pa_pencil* p, const int64_t* coords,
                          int memory_order, int64_t* lo, int64_t* hi);
pa_status pa_pencil_size_local(const pa_pencil* p, int memory_order,
                               int64_t* dims /*[N]*/);
/* staging arenas living in the pencil family (Pencils.jl:185-189).  Device
 * pointers; capacity in bytes; grow-only (Transpositions.jl:313-317).       */
pa_status pa_pencil_buffers(const pa_pencil* p, void** send_buf,
                            int64_t* send_cap, void** recv_buf,
                            int64_t* recv_cap);
pa_status pa_pencil_reserve(pa_pencil* p, int64_t send_bytes, int64_t recv_bytes);

/* ---- Transposition plan --------------------------------------------------
 * Transposition(dest, src; method) (Transpositions.jl:93-118): compatibility
 * checks (assert_compatible, :181-198), `dim` discovery (:110), per-peer
 * ranges/offsets (transpose_send!, :380-416; transpose_recv!, :516-524), all
 * reduced once to kernel launch descriptors.                                */
pa_status pa_plan_create(pa_pencil* pin, pa_pencil* pout, int n_extra,
                         const int64_t* extra_dims, int elsize, pa_method method,
                         pa_plan** out);
void pa_plan_destroy(pa_plan* plan);

typedef struct pa_plan_info {
  int dim;            /* grid dim of the exchange, 1-based; 0 = `nothing` (local) */
  int nproc;          /* topology.dims[dim]  (1 when dim == 0)                  */
  int self_index;     /* my index in the grid line, 1-based                      */
  int same_perm;      /* local path: plain copy! (Transpositions.jl:226-227)     */
  int elsize;
  int method;
  int64_t length_in;       /* length(Ai), elements incl. extra dims             */
  int64_t length_out;      /* length(Ao)                                        */
  int64_t length_self;     /* Transpositions.jl:302-305                         */
  int64_t send_bytes;      /* sizeof(T) * length_send       (:308,313)          */
  int64_t recv_bytes;      /* sizeof(T) * length_recv_total (:309,316)          */
} pa_plan_info;
pa_status pa_plan_get_info(const pa_plan* plan, pa_plan_info* info);

typedef struct pa_peer_info {
  int world_rank;        /* rank of peer n in the world communicator            */
  int is_self;
  int64_t send_offset;   /* bytes into send_buf (self: unused, 0)               */
  int64_t send_count;    /* bytes                                               */
  int64_t recv_offset;   /* bytes into recv_buf; self block sits at the tail
                            (Transpositions.jl:393-403)                         */
  int64_t recv_count;    /* bytes                                               */
  int64_t remote_recv_offset; /* bytes into the PEER's recv_buf where this rank's block
                            lands (= that peer's recv_offset for me): the address the
                            own-kernel exchange stores to (pa_plan_set_recv_window)  */
} pa_peer_info;
pa_status pa_plan_get_peer(const pa_plan* plan, int n /*1-based*/, pa_peer_info* info);

/* Strided-copy descriptor of one block as the kernels see it, exported so
 * tests can compare the C++ plan with the oracle's independent derivation.
 * op: 0 = pack (src parent -> contiguous), 1 = unpack (contiguous -> dest
 * parent), 2 = fused self/local (src parent -> dest parent), 3 = put (src
 * parent -> peer n's dest parent, in the peer's layout; self: empty), 4 = get
 * (peer n's src parent, in its layout -> dest parent).
 * Dims are listed in the source's memory order incl. merged extra dims;
 * strides and offsets in elements.                                           */
typedef struct pa_block_desc {
  int nd;
  int64_t extent[PA_MAX_DIMS];
  int64_t src_stride[PA_MAX_DIMS];
  int64_t dst_stride[PA_MAX_DIMS];
  int64_t src_offset;
  int64_t dst_offset;
  int kernel_class;   /* 0 empty, 1 row copy, 2 tiled transpose, 3 generic scalar,
                         4 contiguous memcpy                                     */
  int vec_bytes;      /* access width chosen for this block                      */
} pa_block_desc;
pa_status pa_plan_get_block(const pa_plan* plan, int op, int n /*1-based*/,
                            pa_block_desc* desc);
/* sub-block `part` (0-based) of `nparts` of a pack (op 0) / unpack (op 1) block as the
 * chunked PointToPoint schedule cuts it (tunable "p2p_chunks"): a sub-range of the
 * block's outermost dimension, i.e. one contiguous piece of the wire block --
 * [*wire_offset, *wire_offset + *wire_bytes) bytes into send_buf / recv_buf.     */
pa_status pa_plan_get_chunk(const pa_plan* plan, int op, int n, int part, int nparts,
                            pa_block_desc* desc, int64_t* wire_offset, int64_t* wire_bytes);

/* ---- kernels (enqueue on `stream`; asynchronous) -------------------------
 * K1 pack: copy_range! (Transpositions.jl:552-583).  `buf` is the base of
 * send_buf (remote peer) or recv_buf (self) -- offsets come from the plan.  */
pa_status pa_pack(pa_plan* plan, int n, const void* src, void* buf, void* stream);
/* K2 unpack: copy_permuted! -> _viewreshape -> _permutedims! (:585-664)     */
pa_status pa_unpack(pa_plan* plan, int n, const void* recv_buf, void* dst, void* stream);
/* K3 fused self block: src parent -> permuted dest parent in one pass
 * (replaces :393-403 followed by :527-529 for the local block)              */
pa_status pa_copy_self(pa_plan* plan, const void* src, void* dst, void* stream);
/* K1-put: block for peer n read from `src` and stored, already permuted, into
 * `peer_dst` = peer n's dest parent array (any pointer this device can write:
 * an IPC/peer mapping, a symmetric heap, or -- for tests -- local memory).
 * Replaces :406-412 + the peer's :527-529 for that block in one pass.         */
pa_status pa_put(pa_plan* plan, int n, const void* src, void* peer_dst, void* stream);
/* K2-get: the block peer n holds for this rank, loaded from `peer_src` = peer
 * n's src parent array (its layout) and stored permuted into `dst`.           */
pa_status pa_get(pa_plan* plan, int n, const void* peer_src, void* dst, void* stream);
/* K1-put / K2-get of EVERY remote block in ONE launch (the kernel the one-sided
 * methods run, here without the window protocol): `peers[n-1]` = peer n's dest
 * (put) / src (get) parent array, the self entry is ignored.  Tiles of the blocks
 * are interleaved round-robin so that all destination links are driven at once.
 * `max_ctas`: grid cap (0 = tunable "remote_ctas").  Falls back to one launch per
 * block when the blocks need different kernel flavours.                        */
pa_status pa_put_all(pa_plan* plan, const void* src, void* const* peers, int max_ctas,
                     void* stream);
pa_status pa_get_all(pa_plan* plan, void* const* peers, void* dst, int max_ctas, void* stream);
/* K2-get of every remote block, the self block and the 1-d FFT along dst's contiguous dim in ONE
 * launch: the kernel a PA_PEER_GET pa_transpose with PA_FFT_FORWARD / PA_FFT_BACKWARD runs, here
 * without the window protocol.  dst = fft(transpose(...)) gathered from `src` (this rank's src
 * parent, for the self block) and `peers[n-1]` = peer n's src parent array (its layout, as
 * mapped here; the self entry is ignored).  flags: PA_FFT_FORWARD or PA_FFT_BACKWARD, optionally
 * with PA_FFT_F32 (ComplexF32, elsize-8 plan); anything else is PA_EINVAL.  The plan's
 * pa_plan_fft_check_ex verdict is asked first; NULL pointers are allowed only for empty blocks /
 * arrays, arrays element-aligned (dst 16 bytes), src and dst not overlapping.  Every refusal
 * happens on the host before anything is enqueued; without a device PA_ENOGPU after those
 * checks.  The result equals the staged fused transpose byte for byte.                        */
pa_status pa_get_all_fft(pa_plan* plan, const void* src, void* const* peers, void* dst,
                         unsigned flags, void* stream);
/* transpose_impl!(::Nothing) / permute_local! (:213-270).  `scratch` must hold
 * length_out elements when src and dst alias, may be NULL otherwise.        */
pa_status pa_permute_local(pa_plan* plan, const void* src, void* dst,
                           void* scratch, void* stream);
/* raw N-d strided copy used by all of the above (bench / tests)             */
pa_status pa_box_copy(int nd, const int64_t* extent, const int64_t* src_stride,
                      const int64_t* dst_stride, int elsize, const void* src,
                      void* dst, void* stream, pa_block_desc* chosen /*NULL ok*/);

/* ---- communicator --------------------------------------------------------
 * Stands in for MPI.COMM_WORLD + MPI_Cart_sub sub-communicators
 * (MPITopologies.jl:244-251): one NCCL communicator over all ranks, peers of
 * a grid line addressed by world rank.  Bootstrap: rank 0 calls
 * pa_comm_unique_id and distributes the 128 bytes by any side channel.      */
pa_status pa_comm_unique_id(void* id128);
pa_status pa_comm_init_rank(const void* id128, int nranks, int rank, pa_comm** out);
/* NCCL-free communicator: ranks talk only through peer-mapped memory (CUDA IPC) and
 * the flag window below, which is then mandatory.  Serves PA_PEER_PUT / PA_PEER_GET
 * as they are and the staged methods through the library's own NVLink copy kernels
 * (pa_plan_set_recv_window).  Unlike NCCL it also allows several ranks on ONE device
 * (test rigs; a single-GPU box can exercise the whole multi-rank path).          */
pa_status pa_comm_init_local(int nranks, int rank, pa_comm** out);
void pa_comm_destroy(pa_comm* c);
/* Flag window: each rank exports a small device buffer (a few 64-bit words per
 * source rank) and imports everybody else's.  Words only increase (signals are
 * red.max.release.sys over NVLink, waits are ld.acquire.sys polls with the
 * "fence_timeout_ms" time-out): window-open / window-close of PA_PEER_PUT /
 * PA_PEER_GET ride inside the transfer kernel, block arrival of the own-kernel
 * exchange is one word per peer.  Without it (NCCL communicators only) the
 * one-sided methods fence with NCCL send/recv groups.                          */
pa_status pa_comm_flags_export(pa_comm* c, void* handle64, int64_t* offset);
pa_status pa_comm_flags_import(pa_comm* c, int rank, const void* handle64, int64_t offset);

/* ---- PeerPut windows (PA_PEER_PUT) -----------------------------------------
 * The analogue of a collective MPI_Win_create over `dest`: every rank exports
 * an IPC handle of its `dest` array, hands it to the peers of its grid line by
 * any side channel (the host mirror uses the same channel as the NCCL id), and
 * registers the mapped peer pointers with the plan.                          */
#define PA_IPC_HANDLE_BYTES 64
/* handle of the device allocation containing `devptr` + byte offset of devptr in it */
pa_status pa_ipc_export(const void* devptr, void* handle64, int64_t* offset);
/* map a peer's allocation (one mapping per handle, reference-counted) and return
 * base + offset; every successful import is paired with one pa_ipc_release     */
pa_status pa_ipc_import(const void* handle64, int64_t offset, void** mapped);
/* drop one reference; the mapping is closed (cudaIpcCloseMemHandle) with the last */
pa_status pa_ipc_release(const void* handle64);
/* `peer_dst` = peer n's (1-based index in the grid line) dest array as mapped here;
 * `local_dst` = this rank's dest array the window belongs to                   */
pa_status pa_plan_set_window(pa_plan* plan, const void* local_dst, int n, void* peer_dst);
/* own-kernel exchange of the staged methods (NCCL-free communicator, or tunable
 * "ipc_exchange"): `peer_recv_buf` = peer n's recv_buf arena (pa_pencil_buffers
 * after pa_pencil_reserve, exported with pa_ipc_export) as mapped here.  Must be
 * renewed when the arenas are reallocated (PA_ESTATE otherwise).                */
pa_status pa_plan_set_recv_window(pa_plan* plan, int n, void* peer_recv_buf);

/* ---- transpose! ----------------------------------------------------------
 * transpose!(t; waitall) (Transpositions.jl:170-179) for device arrays.
 * Ordered after prior work on `stream`; on return, later work on `stream`
 * sees `dst` complete.  Without PA_WAITALL the send side (send_buf reuse) is
 * only guaranteed after pa_wait -- MPI.Waitall(t) (:127-130).
 * `comm` may be NULL when nproc == 1.                                        */
pa_status pa_transpose(pa_plan* plan, pa_comm* comm, const void* src, void* dst,
                       unsigned flags, void* stream);
pa_status pa_wait(pa_plan* plan, void* stream);
/* Can pa_transpose fuse PA_FFT_FORWARD / PA_FFT_BACKWARD into this plan?  PA_OK, or
 * PA_EINVAL with the reason in pa_last_error.  The answer depends on the global geometry
 * only (element size, line length, the blocks every rank of the grid line gathers), so it
 * is the same on every rank of the line: a caller may pick the fused or the separate
 * transpose + transform up front.  pa_transpose asks the same question before it enqueues
 * anything, and a refused fused transpose launches nothing.  Host-only; no device needed. */
pa_status pa_plan_fft_check(const pa_plan* plan);
/* same question for the precision in `flags` (the pa_transpose flags of the fused call;
 * only PA_FFT_F32 matters): PA_FFT_F32 set asks about ComplexF32, unset about
 * ComplexF64 like pa_plan_fft_check.  Each precision's verdict is cached on its own. */
pa_status pa_plan_fft_check_ex(const pa_plan* plan, unsigned flags);
/* same, with HOST arrays: H2D of `src`, transpose!, D2H of `dst`; blocks until
 * `host_dst` is valid.  Device staging is owned by the plan.  A purely local
 * transposition (nproc == 1 or dim == nothing) is cut along the source's outermost
 * dimension and pipelined on three streams: upload(c+1) || kernel(c) ||
 * download(c-1) (the download joins when that dimension is outermost in `dst` too).
 * Pinning the host arrays (cudaHostRegister / pinned allocation) is the caller's job. */
pa_status pa_transpose_host(pa_plan* plan, pa_comm* comm, const void* host_src,
                            void* host_dst, unsigned flags);

/* ---- real-to-complex line transforms ----------------------------------------
 * Step 1 of a PencilFFTs real-input plan (rfft along the first, local dimension; the
 * two complex steps are the fused transposes above), and its inverse.  `real` has global
 * size (..., N, ...), `cplx` the same with N/2+1 along the transform axis = the first
 * MEMORY-order dimension (perm[1]) of both, which must not be decomposed; same topology
 * object, decomposition and permutation (Pencil(p; size_global) builds such a pencil).
 *   PA_FFT_FORWARD:  src = real Float64 array, dst = ComplexF64 array, dst = rfft(src)
 *   PA_FFT_BACKWARD: src = ComplexF64, dst = Float64, dst = N * irfft(src, N) -- unnormalised
 *                    like FFTW's brfft; the imaginary parts of bins 0 and N/2 are ignored and
 *                    `src` is left unmodified.
 *   either | PA_FFT_F32: the same with Float32 / ComplexF32 arrays and fp32 arithmetic.
 * N: power of two in 16..2048.  One kernel per call, local to the rank (no communication);
 * extra dims are batched.  Arrays dense (parent layout), 16-byte aligned, not overlapping;
 * NULL allowed where the local array is empty.  Ordered on `stream` like pa_transpose.
 * PA_EINCOMPAT: pencils not related as above; PA_EINVAL: other bad arguments.          */
pa_status pa_rfft(const pa_pencil* real, const pa_pencil* cplx, int n_extra,
                  const int64_t* extra_dims, unsigned flags, const void* src, void* dst,
                  void* stream);

/* ---- real-to-real line transforms ------------------------------------------------
 * The DCT / DST of PencilFFTs' Transforms.R2R (walls: Neumann through DCT-II/III, Dirichlet
 * through DST-II/III) along the first MEMORY-order dimension (perm[1]) of a real array on
 * `pencil`, which must not be decomposed.  src and dst have the same shape; N points per line,
 * n, k = 0 ... N-1, unnormalised as FFTW defines them (scipy.fft.dct / dst types 2 and 3):
 *   PA_REDFT10  DCT-II    Y[k] = 2 sum_n x[n] cos(pi (2n+1) k / 2N)
 *   PA_REDFT01  DCT-III   Y[k] = x[0] + 2 sum_{n>=1} x[n] cos(pi n (2k+1) / 2N)
 *   PA_RODFT10  DST-II    Y[k] = 2 sum_n x[n] sin(pi (2n+1) (k+1) / 2N)
 *   PA_RODFT01  DST-III   Y[k] = (-1)^k x[N-1] + 2 sum_{n<N-1} x[n] sin(pi (n+1) (2k+1) / 2N)
 * so that REDFT01(REDFT10(x)) = RODFT01(RODFT10(x)) = 2N x.  The kind values are FFTW's
 * fftw_r2r_kind values.  flags: 0 (Float64) or PA_FFT_F32 (Float32, fp32 arithmetic).
 * N: power of two in 16..2048.  One kernel per call, local to the rank; extra dims are batched.
 * Arrays dense (parent layout), 16-byte aligned; src == dst (in place) is allowed, any other
 * overlap is not; NULL allowed where the local array is empty.  Ordered on `stream` like
 * pa_transpose.  Every refusal happens before anything is enqueued.  PA_EINCOMPAT: the
 * transform axis is decomposed; PA_EINVAL: other bad arguments.                          */
#define PA_REDFT01 4
#define PA_REDFT10 5
#define PA_RODFT01 8
#define PA_RODFT10 9
pa_status pa_r2r(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims, int kind,
                 unsigned flags, const void* src, void* dst, void* stream);

/* ---- fused transpose + complex-to-real line transform ---------------------------
 * The last step of a PencilFFTs real-input backward transform in one kernel per rank after
 * the exchange: dst = brfft(transpose(src)), with no complex x-pencil array in between.
 * `plan` is the ordinary complex plan y-pencil -> x-pencil (ComplexF64, elsize 16; with
 * PA_FFT_F32 ComplexF32, elsize 8); `real` is the real counterpart of the plan's output pencil,
 * related to it as `real` and `cplx` of pa_rfft (same topology object, decomposition and
 * permutation; N along perm[1], N/2+1 in the output pencil; that axis not decomposed).
 *   src: the y-pencil ComplexF64 (ComplexF32) array of the plan, left unmodified;
 *   dst: the Float64 (Float32) array on `real`, = N * irfft(transpose(src), N) along perm[1],
 *        unnormalised like FFTW's brfft; the imaginary parts of bins 0 and N/2 are ignored.
 * N: power of two in 16..2048.  flags: any of PA_WAITALL, PA_NO_OVERLAP, PA_STAGE_SELF and
 * PA_FFT_F32 -- the direction is implied, any other bit is PA_EINVAL.  Ordering, waitall,
 * pa_wait, NULL pointers for empty local arrays and the staged methods behave as for
 * pa_transpose with a fused FFT; PA_PEER_PUT / PA_PEER_GET are refused.  src and dst must not
 * overlap, dst 16-byte aligned.  Every refusal (PA_EINCOMPAT: pencils not related as above;
 * PA_EINVAL: other bad arguments, or a geometry pa_plan_brfft_check refuses) happens before
 * anything is enqueued, and a refused geometry is refused on every rank of the grid line.   */
pa_status pa_transpose_brfft(pa_plan* plan, pa_comm* comm, const pa_pencil* real,
                             const void* src, void* dst, unsigned flags, void* stream);
/* Can pa_transpose_brfft run on this plan?  pa_plan_fft_check_ex's question for the fused
 * complex-to-real transform (line length N/2+1, at most 8 blocks per line, the destination
 * strides, and a staged method: PA_PEER_PUT / PA_PEER_GET are refused when the plan exchanges
 * data): the same answer on every rank of the grid line.  Only PA_FFT_F32 of `flags`
 * matters.  Cached per plan and precision, apart from pa_plan_fft_check's verdicts.
 * Host-only; no device needed.                                                            */
pa_status pa_plan_brfft_check(const pa_plan* plan, unsigned flags);

/* ---- fused transpose + real line transforms ----------------------------------------
 * A transposition of REAL arrays and a line transform along the dimension it makes local, in
 * one kernel per rank after the exchange: the steps of a wall-bounded PencilFFTs transform
 * (DCT / DST along some dims, RFFT / FFT along the others) without the array in between.
 * `plan` is an ordinary real plan (Float64, elsize 8; with PA_FFT_F32 Float32, elsize 4); the
 * transform runs along the first memory dim of its output pencil (not decomposed: PA_EINCOMPAT),
 * N points, N a power of two in 16..2048.  src: the input-pencil array of the plan, left unmodified.
 *
 * pa_transpose_r2r: dst = r2r(transpose(src), kind), the plan's output-pencil array of the same
 *   element type; kind PA_REDFT10, PA_REDFT01, PA_RODFT10 or PA_RODFT01, as pa_r2r.
 * pa_transpose_rfft: dst = rfft(transpose(src)), the ComplexF64 (ComplexF32) array on `cplx`, the
 *   complex counterpart of the plan's output pencil related to it as `cplx` to `real` in pa_rfft
 *   (N/2+1 points along perm[1]).
 *
 * Both equal the unfused pa_transpose + pa_r2r / pa_rfft bit for bit.  flags: any of
 * PA_WAITALL, PA_NO_OVERLAP, PA_STAGE_SELF and PA_FFT_F32 -- the direction is implied, any other
 * bit is PA_EINVAL; a kind other than the four is PA_EINVAL.  Ordering, waitall, pa_wait, NULL
 * pointers for empty local arrays and the staged methods behave as for pa_transpose_brfft;
 * PA_PEER_PUT / PA_PEER_GET are refused.  src and dst must not overlap, dst 16-byte aligned.
 * Every refusal (PA_EINCOMPAT: pencils not related as above; PA_EINVAL: other bad arguments, or
 * a geometry pa_plan_real_check refuses) happens before anything is enqueued, and a refused
 * geometry is refused on every rank of the grid line.                                     */
pa_status pa_transpose_r2r(pa_plan* plan, pa_comm* comm, int kind, const void* src, void* dst,
                           unsigned flags, void* stream);
pa_status pa_transpose_rfft(pa_plan* plan, pa_comm* comm, const pa_pencil* cplx, const void* src,
                            void* dst, unsigned flags, void* stream);
/* Can pa_transpose_r2r / pa_transpose_rfft run on this plan?  One answer for both (their
 * exchange is the same, N reals per line): line length N, at most 8 blocks per line, the
 * destination strides, and a staged method (PA_PEER_PUT / PA_PEER_GET are refused when the plan
 * exchanges data): the same answer on every rank of the grid line.  Only PA_FFT_F32 of `flags`
 * matters.  Cached per plan and precision, apart from the pa_plan_fft_check_ex and
 * pa_plan_brfft_check verdicts.  Host-only; no device needed.                             */
pa_status pa_plan_real_check(const pa_plan* plan, unsigned flags);

/* ---- send-side fused transform + transposition (PA_PEER_PUT) -------------------------
 * dst = transpose(T(src)), T along the FIRST memory dim of the plan's input pencil (not
 * decomposed), in ONE kernel per rank: it loads whole local source lines, transforms them in
 * shared memory and stores every output bin into the block that owns it -- the self block into
 * dst, every other block straight into its rank's dst through the PeerPut window (pa_plan_set_window).
 * The window protocol runs inside the launch (standalone flag kernels around it when tunable
 * multi_put = 0 or the line has more than 8 peers; NCCL line barriers under nccl_fences); a rank
 * without source lines launches no transform but still takes part in the protocol.  Events and
 * PA_WAITALL behave as for the plain PeerPut transposition.  Local plans (no exchange, or a grid
 * line of one rank) of any method run the kernel on `stream` alone.  Other methods that exchange
 * data are refused: there the receive-side fusion (pa_transpose with PA_FFT_*, pa_transpose_rfft)
 * covers the chain.  The result equals the unfused pair under the same tunables byte for byte.
 *
 * pa_fft_put: T is the complex FFT (PA_FFT_FORWARD, or the unnormalised PA_FFT_BACKWARD) of a
 *   ComplexF64 plan (with PA_FFT_F32 ComplexF32, elsize 8), L a power of two in 8..1024;
 *   dst equals fft_ on a copy of src followed by pa_transpose.
 * pa_rfft_put: T is the r2c transform of pa_rfft; `plan` is the COMPLEX plan from the N/2+1-bin
 *   counterpart of `real` (related to it as `cplx` to `real` in pa_rfft) to dst's pencil; src is the
 *   Float64 (Float32 with PA_FFT_F32) array on `real`, N a power of two in 16..2048; dst equals
 *   pa_rfft followed by pa_transpose of the complex array.
 *
 * flags: pa_fft_put exactly one of PA_FFT_FORWARD / PA_FFT_BACKWARD, optionally with PA_FFT_F32
 * and PA_WAITALL; pa_rfft_put any of PA_FFT_F32 and PA_WAITALL (the direction is implied).  Any
 * other bit (PA_STAGE_SELF included: there is no staged schedule) is PA_EINVAL.  src and dst must
 * not overlap, NULL only when empty, aligned to the complex element.  Every refusal (PA_EINVAL; a
 * `real` not related to the plan's input pencil: PA_EINCOMPAT) happens on the host before anything
 * is enqueued, and a refused geometry is refused on every rank of the grid line; without a device
 * PA_ENOGPU after those checks.                                                            */
pa_status pa_fft_put(pa_plan* plan, pa_comm* comm, const void* src, void* dst, unsigned flags,
                     void* stream);
pa_status pa_rfft_put(pa_plan* plan, pa_comm* comm, const pa_pencil* real, const void* src, void* dst,
                      unsigned flags, void* stream);
/* The same kernels without the window protocol (the counterparts of pa_get_all_fft): the self
 * block into `dst`, the block of peer n into `peers[n-1]` (its dst parent array, as mapped here;
 * the self entry is ignored).  flags: pa_put_all_fft PA_FFT_FORWARD or PA_FFT_BACKWARD, optionally
 * with PA_FFT_F32; pa_put_all_rfft 0 or PA_FFT_F32.  The plan must exchange data; checks as above. */
pa_status pa_put_all_fft(pa_plan* plan, const void* src, void* const* peers, void* dst, unsigned flags,
                         void* stream);
pa_status pa_put_all_rfft(pa_plan* plan, const pa_pencil* real, const void* src, void* const* peers,
                          void* dst, unsigned flags, void* stream);
/* Can pa_fft_put (pa_rfft_put) run on this plan?  Element size, line length, at most 8 blocks per
 * line that tile it and share every other dim, and PA_PEER_PUT when the plan exchanges data: the
 * same answer on every rank of the grid line (each rank's plan is rebuilt).  Only PA_FFT_F32 of
 * `flags` matters.  Cached per plan and precision, apart from every other verdict.  Host-only.  */
pa_status pa_plan_fft_put_check(const pa_plan* plan, unsigned flags);
pa_status pa_plan_rfft_put_check(const pa_plan* plan, unsigned flags);
/* The wall-bounded legs of the same send-side fusion (DESIGN §3j).  `plan` is a REAL plan (Float64,
 * elsize 8; Float32, elsize 4 with PA_FFT_F32) that moves N reals per line along the first memory
 * dim of its input pencil, N a power of two in 16..2048; the blocks may split a line at any real.
 * pa_r2r_put: T is pa_r2r's transform of `kind` (PA_REDFT10, PA_REDFT01, PA_RODFT10 or PA_RODFT01)
 *   on the real src; dst equals pa_r2r on a copy of src followed by pa_transpose.
 * pa_brfft_put: T is the c2r transform of pa_brfft; src is the ComplexF64 (ComplexF32) array on
 *   `cplx`, the N/2+1-bin counterpart of the plan's input pencil (related to it as `cplx` to `real`
 *   in pa_rfft); dst equals pa_brfft followed by pa_transpose of the real array.
 * flags: any of PA_FFT_F32 and PA_WAITALL (the direction is implied); every other bit, PA_STAGE_SELF
 * included, is PA_EINVAL, as is any other kind.  src (aligned to 2 reals) and dst (aligned to the
 * real) must not overlap, NULL only when empty.  Schedule, protocol, events, refusals on the host
 * (a `cplx` not related to the plan's input pencil: PA_EINCOMPAT) and PA_ENOGPU as for pa_fft_put. */
pa_status pa_r2r_put(pa_plan* plan, pa_comm* comm, int kind, const void* src, void* dst, unsigned flags,
                     void* stream);
pa_status pa_brfft_put(pa_plan* plan, pa_comm* comm, const pa_pencil* cplx, const void* src, void* dst,
                       unsigned flags, void* stream);
/* Their kernels without the window protocol, as pa_put_all_fft: the self block into `dst`, the
 * block of peer n into `peers[n-1]`.  flags: 0 or PA_FFT_F32.  The plan must exchange data.      */
pa_status pa_put_all_r2r(pa_plan* plan, int kind, const void* src, void* const* peers, void* dst,
                         unsigned flags, void* stream);
pa_status pa_put_all_brfft(pa_plan* plan, const pa_pencil* cplx, const void* src, void* const* peers,
                           void* dst, unsigned flags, void* stream);
/* Can pa_r2r_put and pa_brfft_put run on this real plan?  One verdict for both, with the rules of
 * pa_plan_fft_put_check (line length N, at most 8 blocks, PA_PEER_PUT when the plan exchanges data,
 * the same answer on every rank of the grid line).  Only PA_FFT_F32 of `flags` matters.  Cached per
 * plan and precision, apart from every other verdict.  Host-only.                                 */
pa_status pa_plan_real_put_check(const pa_plan* plan, unsigned flags);

/* ---- distributed reductions (reductions.jl:10-38) -------------------------------------
 * mapreduce(f, op, u[, v]) over the parent arrays of PencilArrays (extra dims included), combined
 * across every rank of the communicator: each rank gets the same global result, as a 0-d device
 * value at `result`.  ONE kernel per rank and call: a streaming pass over the local array and the
 * combine through the communicator's flag window (DESIGN §3k); ordered after prior work on
 * `stream`, and the host is not synchronised.  Julia's semantics:
 *   maps   PA_MAP_IDENTITY, PA_MAP_ABS (complex: hypot(re, im)), PA_MAP_ABS2 (integers wrap),
 *          PA_MAP_DOT = real(x * conj(y)) of two arrays a, b (the same expression as abs2 when
 *          a == b: mapreduce(dot, +, u, u) == sum(abs2, u) bit for bit);
 *   ops    PA_OP_SUM, PA_OP_MAX, PA_OP_MIN (a NaN anywhere gives NaN; max(-0.0, 0.0) == 0.0),
 *          PA_OP_ANY / PA_OP_ALL or-ed with one PA_PRED_*: the predicate of the mapped value,
 *          against *pred_value (one value of the mapped type: the element type under
 *          identity, the real type under abs / abs2 / dot) for the comparisons;
 *   result pa_reduce_result_type: sum of Int32 gives Int64, abs / abs2 / dot of complex values
 *          give the real type, any / all give Bool (one byte), otherwise the element type.
 * Float32 / ComplexF32 sums accumulate in fp64; the result is deterministic (the same bits on
 * every rank and for every call on the same data and grid).  Refused with PA_EINVAL: an unknown or
 * invalid (dtype, map, op) -- max / min of complex values under identity, an ordered comparison of
 * complex values --, `b` given for a one-array map or missing for PA_MAP_DOT, NULL pointers for a
 * non-empty local array, arrays not aligned to their real component, a NULL `result` or one
 * not aligned to the whole result type (16 bytes for ComplexF64, 8 for ComplexF32), a missing
 * pred_value for a comparison, maximum / minimum of a globally empty array;
 * PA_EINCOMPAT: the topology's rank count is not the communicator's, or comm == NULL with more
 * than one rank.  Every refusal happens on the host before anything is enqueued; without a device
 * PA_ENOGPU after those checks.  Reductions on one communicator are serialised in issue order.   */
typedef enum pa_dtype {
  PA_FLOAT64 = 0, PA_FLOAT32 = 1, PA_COMPLEXF64 = 2, PA_COMPLEXF32 = 3, PA_INT32 = 4, PA_INT64 = 5,
  PA_BOOL = 6 /* result type of any / all only */
} pa_dtype;
typedef enum pa_reduce_map { PA_MAP_IDENTITY = 0, PA_MAP_ABS = 1, PA_MAP_ABS2 = 2, PA_MAP_DOT = 3 } pa_reduce_map;
typedef enum pa_reduce_op { PA_OP_SUM = 0, PA_OP_MAX = 1, PA_OP_MIN = 2, PA_OP_ANY = 3, PA_OP_ALL = 4 } pa_reduce_op;
#define PA_PRED_EQ       (1 << 4)  /* ==(value) */
#define PA_PRED_NE       (2 << 4)  /* !=(value) */
#define PA_PRED_LT       (3 << 4)  /* <(value)  */
#define PA_PRED_LE       (4 << 4)  /* <=(value) */
#define PA_PRED_GT       (5 << 4)  /* >(value)  */
#define PA_PRED_GE       (6 << 4)  /* >=(value) */
#define PA_PRED_ISNAN    (7 << 4)
#define PA_PRED_ISFINITE (8 << 4)
pa_status pa_reduce(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims, pa_comm* comm,
                    int dtype, int map, int op, const void* pred_value, const void* a,
                    const void* b, void* result, void* stream);
/* the result's pa_dtype of pa_reduce(dtype, map, op); PA_EINVAL (with the reason) for the
 * combinations pa_reduce refuses.  Host-only.                                                  */
pa_status pa_reduce_result_type(int dtype, int map, int op, int* result_dtype);

/* mapreduce(f, op, u[, v]; dims): the reduction of pa_reduce (same maps, ops, predicates, result
 * types and rules) over the logical dims `dims` only (n_dims of them, 1-based: 1..N the pencil's
 * spatial dims, N+1..N+n_extra its extra dims; any order; no duplicates).  Each rank gets, at
 * `result`, a dense array laid out like its parent array (memory order, extra dims last) with extent
 * 1 along every reduced dim and its local extent along every kept dim: entry I holds the reduction
 * over the GLOBAL ranges of the reduced dims at this rank's global index I of the kept dims.  A rank
 * combines with the ranks whose grid coordinates agree with its own on every grid dim that
 * decomposes a kept dim, folding their partials in rank order; every member gets the same bits.
 * `dims` covering every dim is pa_reduce.  ONE kernel per rank and call (DESIGN §3l), ordered on
 * `stream`, collective over the communicator (ranks with an empty array or result take part), the
 * host is not synchronised.  Refused with PA_EINVAL, checked in this order (error texts start with
 * "pa_reduce_dims:"): a NULL pencil; an invalid (dtype, map, op) as pa_reduce_result_type decides
 * it; bad extra dims; bad `dims` (none, NULL, out of 1..N+n_extra, or one given twice); then
 * pa_reduce's array checks in its order -- `b` given or missing, NULL arrays for a non-empty local
 * array, alignment, `result` (which may be NULL when the local result is empty), a comparison
 * without pred_value --; max / min over a globally empty reduced range (a sum gives zeros); with
 * more than one rank, a local result larger than the flag window's partial area (524288 elements
 * on the rank with the most), decided from the global geometry.  PA_EINCOMPAT: the topology and the
 * communicator disagree on the rank count, as in pa_reduce.  Then without a device PA_ENOGPU.
 * PA_ESTATE: more than one rank on a communicator without a flag window (NCCL alone, or the
 * nccl_fences tunable).
 * pa_reduce and pa_reduce_dims on one communicator share one serialisation, in issue order.      */
pa_status pa_reduce_dims(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims,
                         pa_comm* comm, int dtype, int map, int op, const void* pred_value,
                         const void* a, const void* b, int n_dims, const int* dims, void* result,
                         void* stream);

/* Shell-binned spectrum of complex PencilArrays whose spatial dims are the modes of an unnormalised
 * DFT: E(b) = sum over the modes k with bin(|k|) == b of w(k) * f(x), f = abs2 of `a`
 * (PA_MAP_ABS2) or real(a * conj(b)) (PA_MAP_DOT, a co-spectrum); extra dims (vector components)
 * add into the same bins.  `result` receives nbins values of pa_reduce_result_type(dtype, map,
 * PA_OP_SUM) (Float64 / Float32): the GLOBAL spectrum, the same bits on every rank.  Geometry
 * (reduce_core.hpp, DESIGN §3m), along logical dim d of global extent N_d at global 0-based index i:
 *   wavenumber  n = i if i < (N_d + 1) / 2 else i - N_d (numpy's fftfreq order); along the r2c dim
 *               (rfft_dim, 1-based; 0: none) n = i, that dim holding M = rfft_n / 2 + 1 bins of a
 *               real length rfft_n (0: the default 2 (M - 1); any rfft_n with rfft_n / 2 + 1 == M);
 *   weight      w = 2 along the r2c dim except at i = 0 and (rfft_n even) i = rfft_n / 2, else 1;
 *   bin         k_d = scales[d - 1] * n_d (scales NULL: all 1), q = k_1 * k_1 + k_2 * k_2 + ... in
 *               logical-dim order, b = floor(sqrt(q) / width + 0.5), each operation one correctly
 *               rounded fp64 operation (NumPy's elementwise result bit for bit); modes with
 *               b >= nbins are dropped.
 * Contributions are computed as pa_reduce computes the map and summed in fp64 (Float32 results
 * rounded once), a NaN poisons its own bin only; the order of every sum depends on the geometry, the
 * arguments, the device and the base addresses modulo 16 only.  ONE kernel per rank and call,
 * ordered on `stream`, collective over the communicator (ranks owning nothing take part), the host
 * is not synchronised; shares pa_reduce's serialisation.  nbins is at most PA_SPECTRUM_MAX_BINS:
 * each of a CTA's four warps keeps a histogram of nbins doubles in shared memory (128 KiB at the
 * cap).  Refused on the host, in this order, identically on every rank (error texts start with
 * "pa_shell_spectrum:"), PA_EINVAL: a NULL pencil; dtype not complex or map not PA_MAP_ABS2 /
 * PA_MAP_DOT; `b` given for PA_MAP_ABS2 or missing for PA_MAP_DOT (NULL arrays are fine where the
 * local array is empty); bad extra dims; rfft_dim outside
 * 0..N; rfft_n inconsistent with the r2c dim's extent (or given without one); a scale or the width
 * not finite and positive; nbins outside 1..PA_SPECTRUM_MAX_BINS; NULL arrays for a non-empty local
 * array; arrays not aligned to their real component; a NULL `result` or one not aligned to the
 * result type.  PA_EINCOMPAT: the topology's rank count is not the communicator's (or comm == NULL
 * with more than one rank).  Then without a device PA_ENOGPU.  PA_ESTATE: more than one rank on a
 * communicator without a flag window.                                                             */
#define PA_SPECTRUM_MAX_BINS 4096
pa_status pa_shell_spectrum(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims,
                            pa_comm* comm, int dtype, int map, const void* a, const void* b,
                            int rfft_dim, int64_t rfft_n, const double* scales, double width,
                            int nbins, void* result, void* stream);
/* The default nbins of pa_shell_spectrum: the bin of the extreme mode (the largest |wavenumber|
 * along every dim) plus one, from the same geometry functions; it may exceed
 * PA_SPECTRUM_MAX_BINS, which pa_shell_spectrum then refuses.  Refused like pa_shell_spectrum (a
 * NULL pencil, then its rfft_dim / rfft_n / scales / width checks), or when the bin does not fit an
 * int.  Host-only.                                                                                 */
pa_status pa_shell_spectrum_nbins(const pa_pencil* pencil, int rfft_dim, int64_t rfft_n,
                                  const double* scales, double width, int* nbins);

/* The spectrum of pa_shell_spectrum over chosen dims, each logical dim given one role (DESIGN §3n):
 *   bin dims   bin_dims[0 .. n_bin-1]: 1-based SPATIAL dims (at least one, no repeats); |k| is formed
 *              from these only (q summed over them in logical-dim order, every operation one
 *              correctly rounded fp64 operation as in pa_shell_spectrum);
 *   kept dims  keep_dims[0 .. n_keep-1]: 1-based logical dims (1..N spatial, N+1..N+n_extra extra),
 *              none of them a bin dim, no repeats (n_keep 0: none); each rank gets its local range;
 *   every other dim, spatial or extra, is summed into the bins.
 * The wavenumbers, weights and bins are pa_shell_spectrum's, whatever role the r2c dim has: along a
 * kept r2c dim index i holds modes i and -i together (weight 2 in the interior), so the sum over
 * the bins and over the kept indices of every rank is Parseval's total.  scales: one per spatial
 * dim (all checked, only the bin dims' used).  `result` receives, as pa_reduce_result_type(dtype,
 * map, PA_OP_SUM) values, result[b + nbins * o]: o the column-major index over the local extents of
 * the kept dims in the parent's memory order (extra dims last), as in pa_reduce_dims' result.  A
 * rank combines with the ranks whose grid coordinates agree with its own on every grid dim that
 * decomposes a kept dim, folding their partials in rank order; every member gets the same bits
 * (with no kept dim decomposed: every rank).  Every spatial dim binned and nothing kept is
 * pa_shell_spectrum, bit for bit.  ONE kernel per rank and call, ordered on `stream`, collective
 * over the communicator (ranks owning nothing take part), the host is not synchronised; shares
 * pa_reduce's serialisation.  Refused on the host, in this order, identically on every rank (error
 * texts start with "pa_shell_spectrum_dims:"), PA_EINVAL: a NULL pencil; dtype not complex or map
 * not PA_MAP_ABS2 / PA_MAP_DOT; `b` given for PA_MAP_ABS2 or missing for PA_MAP_DOT; bad extra
 * dims; bad bin dims (none, NULL, outside 1..N, or one given twice); bad kept dims (n_keep < 0, NULL
 * with n_keep > 0, outside 1..N+n_extra, given twice, or a bin dim); rfft_dim outside 0..N; rfft_n
 * inconsistent with the r2c dim; a scale or the width not finite and positive; nbins outside
 * 1..PA_SPECTRUM_MAX_BINS; NULL arrays for a non-empty local array; arrays not aligned to their
 * real component; `result` NULL (allowed when the local result is empty) or not aligned to the
 * result type; with more than one rank, nbins x the kept outputs of the rank with the most above
 * the flag window's partial area (524288 accumulators), decided from the global geometry.
 * PA_EINCOMPAT: the topology's rank count is not the communicator's (or comm == NULL with more than
 * one rank).  Then without a device PA_ENOGPU.  PA_ESTATE: more than one rank on a communicator
 * without a flag window.                                                                          */
pa_status pa_shell_spectrum_dims(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims,
                                 pa_comm* comm, int dtype, int map, const void* a, const void* b,
                                 int rfft_dim, int64_t rfft_n, const double* scales, double width,
                                 int nbins, int n_bin, const int* bin_dims, int n_keep,
                                 const int* keep_dims, void* result, void* stream);
/* The default nbins of pa_shell_spectrum_dims: the bin of the extreme mode over the bin dims plus
 * one.  Refused (texts start with "pa_shell_spectrum_dims:") for a NULL pencil, bad bin dims, then
 * pa_shell_spectrum_nbins' checks.  Host-only.                                                    */
pa_status pa_shell_spectrum_dims_nbins(const pa_pencil* pencil, int rfft_dim, int64_t rfft_n,
                                       const double* scales, double width, int n_bin,
                                       const int* bin_dims, int* nbins);

/* ---- host chains -----------------------------------------------------------
 * A sequence of transpositions applied to HOST arrays (plan i+1 consumes what
 * plan i produces): one submit = upload of `host_src`, every transpose! on the
 * device, download into `host_dst`.  Submits return immediately and are double-
 * buffered on the device: the download of one overlaps the upload of the next
 * (PCIe is full duplex).  pa_host_chain_wait(ticket) blocks until that submit's
 * `host_dst` is valid (ticket < 0: all).  The host arrays must stay untouched /
 * alive until then.  For the one-sided methods the device buffers the plans will
 * see are exposed through pa_host_chain_buffer(slot 0..1, which 0..1) so that
 * windows can be registered on them (plan i of a submit in slot s reads buffer
 * (s, i % 2) and writes buffer (s, 1 - i % 2)).                                  */
pa_status pa_host_chain_create(int n, pa_plan* const* plans, pa_comm* comm,
                               pa_host_chain** out);
void pa_host_chain_destroy(pa_host_chain* c);
pa_status pa_host_chain_submit(pa_host_chain* c, const void* host_src, void* host_dst,
                               int64_t* ticket /* out, may be NULL */);
pa_status pa_host_chain_wait(pa_host_chain* c, int64_t ticket);
pa_status pa_host_chain_buffer(pa_host_chain* c, int slot, int which, void** devptr,
                               int64_t* bytes);
/* CUDA-event bracket around a run of submits (device-side timing of the pipeline):
 * begin marks the upload stream now, end waits for everything submitted so far and
 * returns the milliseconds between the two.                                      */
pa_status pa_host_chain_time_begin(pa_host_chain* c);
pa_status pa_host_chain_time_end(pa_host_chain* c, float* ms);

/* ---- PencilIO binary layout (SURVEY 8 f4) ---------------------------------------
 * Device arrays <-> the raw binary files of the reference's MPIIODriver
 * (src/PencilIO/mpi_io.jl), byte for byte:
 *   chunks == 0  the dataset is the GLOBAL array in the pencil's memory order, dims
 *                (perm * size_global..., extra_dims...), column-major; this rank owns
 *                the sub-box range_local(x, MemoryOrder()) (:372-380) -- files can be
 *                read back with any other decomposition;
 *   chunks != 0  the ranks' parent arrays one after the other in column-major order of
 *                the process-grid coordinates (:382-424).
 * `offset` = byte offset of the dataset in the file (MPIFile position, :159-164).
 * Every rank calls these for its own part (no collective: ranks pwrite / pread
 * disjoint byte ranges of the same file); the device array moves through a double-
 * buffered pinned staging area on a stream of the library's own.  Each call first waits
 * for ALL device work queued so far in the process, on any stream (cudaDeviceSynchronize:
 * a kernel may still be writing the array that is about to be written, or reading the one
 * about to be read), and returns once the transfer is complete, so work queued afterwards
 * on any stream sees the read data.  The JSON sidecar (:194-211) is written by the host
 * veneer (Julia: the reference's own add_metadata; Python mirror: pencilio.py).     */
pa_status pa_io_sizes(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                      int chunks, int64_t* global_bytes, int64_t* local_bytes, int64_t* nruns,
                      int64_t* run_bytes, int64_t* first_offset);
/* the local array is `nruns` runs of `run_bytes` bytes, contiguous in the array and in the
 * file; run r of the array starts `*file_offset` bytes into the dataset               */
pa_status pa_io_run_offset(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                           int chunks, int64_t run, int64_t* file_offset);
pa_status pa_io_write(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                      int chunks, const void* dev_array, const char* path, int64_t offset);
pa_status pa_io_read(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                     int chunks, void* dev_array, const char* path, int64_t offset);

/* CUDA-event timings (ms) of the last pa_transpose on this plan, named after
 * the reference's TimerOutputs sections (Transpositions.jl:172-175,326,336).
 * Blocks until that transpose has finished.                                  */
typedef struct pa_timings {
  float total_ms;        /* "transpose!"    */
  float pack_ms;         /* "pack data"     */
  float exchange_ms;     /* Isend/Irecv or "MPI.Alltoallv!" */
  float unpack_ms;       /* "unpack data"   */
} pa_timings;
pa_status pa_plan_timings(pa_plan* plan, pa_timings* t);
pa_status pa_plan_enable_timing(pa_plan* plan, int on);

#ifdef __cplusplus
}
#endif
#endif /* PA_B200_H */
