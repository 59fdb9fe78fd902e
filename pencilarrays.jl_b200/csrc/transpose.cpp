// transpose! driver: streams, events and the exchange.
//
// Reference flow (Transpositions.jl:281-343): pack every block
// (transpose_send!, :345-430) posting Isend/Irecv per peer as soon as its
// block is packed (:406-412) or one Alltoallv after all packs (:418-427); then
// unpack blocks as they arrive (transpose_recv!, :486-533), self block first.
//
// GPU restatement: three CUDA streams (pack / comm / unpack) joined by
// events.  PointToPoint = one {send, recv} pair per exchange step, enqueued the
// moment that step's pack finishes, unpack gated on that step's receive -- so
// pack(k+1), exchange(k) and unpack(k-1) overlap; every peer block can be cut
// into sub-blocks that flow through the three stages independently (tunable
// "p2p_chunks").  Steps follow a rotation (send to me+k, receive from me-k)
// instead of the reference's identical 1..Nproc order on every rank: over
// NVSwitch all peers are equidistant and the rotation keeps every link busy.
// Alltoallv = one group holding every peer's send and receive.
//
// Two transports carry the staged schedules:
//   NCCL   grouped ncclSend/ncclRecv on the comm stream (the default whenever
//          the communicator owns an NCCL communicator);
//   IPC    this library's own copy kernels storing send_buf blocks straight into
//          the peer's recv_buf through a CUDA-IPC mapping, completion signalled
//          with flag words over NVLink.  The only transport of an NCCL-free
//          communicator (pa_comm_init_local: several processes may then share
//          one GPU, which NCCL refuses), selectable with tunable "ipc_exchange".
// The one-sided methods (PeerPut / PeerGet) skip staging altogether: ONE kernel
// launch covers the blocks of all peers, with the window-open / window-close
// protocol folded into its prologue / epilogue (kernels.cu, k_multi).
// NCCL is loaded with dlopen so that the library itself has no link-time
// dependency and picks up the libnccl already mapped by the host process.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstdlib>
#include <mutex>
#include <set>

#include "pa_internal.hpp"

namespace pa {

typedef unsigned long long ull;
constexpr size_t IPC_BLOCK = 2u << 20;

#define CU(call)                                                                  \
  do {                                                                            \
    cudaError_t e_ = (call);                                                      \
    if (e_ != cudaSuccess) {                                                      \
      cudaGetLastError(); /* do not leave it for an unrelated later check */      \
      set_error("%s failed: %s", #call, cudaGetErrorString(e_));                  \
      return (e_ == cudaErrorNoDevice || e_ == cudaErrorInsufficientDriver)       \
                 ? PA_ENOGPU                                                      \
                 : (e_ == cudaErrorMemoryAllocation ? PA_ENOMEM : PA_ECUDA);      \
    }                                                                             \
  } while (0)

pa_status set_device(int dev) {
  CU(cudaSetDevice(dev));
  return PA_OK;
}

// ---- CUDA IPC: windows of the one-sided methods -----------------------------------
typedef int (*cuMemGetAddressRange_fn)(unsigned long long*, size_t*, unsigned long long);

static cuMemGetAddressRange_fn addr_range_fn() {
  static cuMemGetAddressRange_fn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return (cuMemGetAddressRange_fn)f;
  }();
  return fn;
}

pa_status ipc_export(const void* devptr, void* handle64, i64* offset) {
  static_assert(sizeof(cudaIpcMemHandle_t) == PA_IPC_HANDLE_BYTES, "ipc handle size");
  if (device_count() == 0) {
    set_error("no CUDA device");
    return PA_ENOGPU;
  }
  CU(cudaFree(nullptr));  // make sure this runtime instance has its context
  cuMemGetAddressRange_fn fn = addr_range_fn();
  unsigned long long base = 0;
  size_t size = 0;
  if (!fn || fn(&base, &size, (unsigned long long)(uintptr_t)devptr) != 0) {
    set_error("cuMemGetAddressRange failed for %p (not a device allocation?)", devptr);
    return PA_ECUDA;
  }
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, (void*)(uintptr_t)base));
  memcpy(handle64, &h, sizeof h);
  *offset = (i64)((unsigned long long)(uintptr_t)devptr - base);
  return PA_OK;
}

// one mapping per peer allocation, reference-counted: pa_ipc_import takes a
// reference, pa_ipc_release drops it and closes the mapping with the last one
struct IpcEntry {
  void* base = nullptr;
  int refs = 0;
};
static std::mutex g_ipc_mu;
static std::map<std::string, IpcEntry> g_ipc_cache;

pa_status ipc_import(const void* handle64, i64 offset, void** mapped) {
  std::lock_guard<std::mutex> lock(g_ipc_mu);
  std::string key((const char*)handle64, PA_IPC_HANDLE_BYTES);
  IpcEntry& e = g_ipc_cache[key];
  if (!e.base) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof h);
    void* base = nullptr;
    cudaError_t err = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
    if (err != cudaSuccess) {
      g_ipc_cache.erase(key);
      set_error("cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(err));
      cudaGetLastError();
      return PA_ECUDA;
    }
    e.base = base;
  }
  ++e.refs;
  *mapped = (char*)e.base + offset;
  return PA_OK;
}

pa_status ipc_release_handle(const void* handle64) {
  std::lock_guard<std::mutex> lock(g_ipc_mu);
  std::string key((const char*)handle64, PA_IPC_HANDLE_BYTES);
  auto it = g_ipc_cache.find(key);
  if (it == g_ipc_cache.end()) return PA_OK;
  if (--it->second.refs <= 0) {
    // nothing may still be running against the mapping
    cudaDeviceSynchronize();
    cudaIpcCloseMemHandle(it->second.base);
    cudaGetLastError();
    g_ipc_cache.erase(it);
  }
  return PA_OK;
}

pa_status plan_set_window(Plan* P, const void* local_dst, int n0, void* peer_dst) {
  if (P->dim < 0 || n0 < 0 || n0 >= P->nproc) {
    set_error("window peer index out of range");
    return PA_EINVAL;
  }
  std::vector<void*>& v = P->windows[local_dst];
  v.resize(P->nproc, nullptr);
  v[n0] = peer_dst;
  return PA_OK;
}

pa_status plan_set_recv_window(Plan* P, int n0, void* peer_recv_buf) {
  if (P->dim < 0 || n0 < 0 || n0 >= P->nproc) {
    set_error("window peer index out of range");
    return PA_EINVAL;
  }
  P->recv_windows.resize(P->nproc, nullptr);
  P->recv_windows[n0] = peer_recv_buf;
  P->recv_windows_gen = P->pout->bufs->generation;
  return PA_OK;
}

// ---- NCCL via dlopen ---------------------------------------------------------
struct NcclApi {
  void* h = nullptr;
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommInitRankConfig) CommInitRankConfig = nullptr;  // optional
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclSend) Send = nullptr;
  decltype(&ncclRecv) Recv = nullptr;
  decltype(&ncclGroupStart) GroupStart = nullptr;
  decltype(&ncclGroupEnd) GroupEnd = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  decltype(&ncclGetVersion) GetVersion = nullptr;
  decltype(&ncclMemAlloc) MemAlloc = nullptr;        // optional (user-buffer registration)
  decltype(&ncclMemFree) MemFree = nullptr;
  decltype(&ncclCommRegister) CommRegister = nullptr;
  decltype(&ncclCommDeregister) CommDeregister = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  bool ok = false;
};

static NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.h) break;
    }
    if (!api.h) return;
#define LOAD(sym) api.sym = (decltype(api.sym))dlsym(api.h, "nccl" #sym)
    LOAD(GetUniqueId);
    LOAD(CommInitRank);
    LOAD(CommInitRankConfig);
    LOAD(CommDestroy);
    LOAD(Send);
    LOAD(Recv);
    LOAD(GroupStart);
    LOAD(GroupEnd);
    LOAD(GetErrorString);
    LOAD(GetVersion);
    LOAD(MemAlloc);
    LOAD(MemFree);
    LOAD(CommRegister);
    LOAD(CommDeregister);
    LOAD(AllGather);
#undef LOAD
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.Send && api.Recv &&
             api.GroupStart && api.GroupEnd && api.GetErrorString;
  });
  return api;
}

#define NC(call)                                                       \
  do {                                                                 \
    ncclResult_t r_ = (call);                                          \
    if (r_ != ncclSuccess) {                                           \
      set_error("%s failed: %s", #call, nccl().GetErrorString(r_));    \
      return PA_ENCCL;                                                 \
    }                                                                  \
  } while (0)

// ---- communicator -------------------------------------------------------------
// Flag window: PA_FLAG_WORDS 64-bit words per source rank, written by that rank
// over NVLink (monotonic max, release.sys) and polled locally (acquire.sys).
enum FlagKind { FK_READY = 0, FK_DONE = 1, FK_DATA = 2, FK_REDUCE = 3, FK_KINDS = 4 };

struct Comm {
  ncclComm_t comm = nullptr;  // nullptr: NCCL-free communicator (pa_comm_init_local)
  int nranks = 0, rank = 0, device = 0;
  ull* flags = nullptr;                  // my words: [source rank][kind]
  std::vector<ull*> peer_flags;          // peers' windows as mapped here
  std::vector<ull> seq_tx[FK_KINDS];     // signals sent to each rank so far, per kind
  std::vector<ull> seq_rx[FK_KINDS];     // signals consumed from each rank so far
  int* fence_err = nullptr;              // mapped pinned host word set on time-out
  bool flags_ready = false;
  std::vector<std::string> imported;     // handles of the peers' flag windows (released on destroy)
  ReduceState* reduce = nullptr;         // the reductions' workspace and event (reduce.cu)
};

// the window: the words [source rank][kind], then the reductions' slots [parity][source rank]
static size_t reduce_slots_offset(int nranks) {
  return (sizeof(ull) * (size_t)nranks * FK_KINDS + 15) / 16 * 16;
}
static size_t window_bytes(int nranks) {
  return reduce_slots_offset(nranks) + 2 * (size_t)nranks * REDUCE_SLOT_BYTES;
}

static ull* remote_word(Comm* c, int peer_rank, int kind) {
  return c->peer_flags[peer_rank] + (size_t)c->rank * FK_KINDS + kind;
}
static ull* local_word(Comm* c, int peer_rank, int kind) {
  return c->flags + (size_t)peer_rank * FK_KINDS + kind;
}
static ull timeout_ns() { return (ull)std::max<long long>(0, g_tun.fence_timeout_ms) * 1000000ull; }

static pa_status check_fence_err(Comm* c) {
  if (c && c->fence_err && *(volatile int*)c->fence_err) {
    set_error("an NVLink flag wait timed out: a peer rank is gone (the CUDA context is lost)");
    return PA_ECUDA;
  }
  return PA_OK;
}

pa_status comm_unique_id(void* id128) {
  static_assert(sizeof(ncclUniqueId) <= PA_UNIQUE_ID_BYTES, "unique id size");
  if (!nccl().ok) {
    set_error("libnccl.so.2 could not be loaded");
    return PA_ENCCL;
  }
  ncclUniqueId id;
  NC(nccl().GetUniqueId(&id));
  memset(id128, 0, PA_UNIQUE_ID_BYTES);
  memcpy(id128, &id, sizeof id);
  return PA_OK;
}

static std::mutex g_live_mu;
static std::set<void*> g_live_comms;  // NCCL communicators that may still hold registrations

static bool any_live_nccl() {
  std::lock_guard<std::mutex> lock(g_live_mu);
  return !g_live_comms.empty();
}

pa_status comm_init(const void* id128, int nranks, int rank, Comm** out) {
  if (!nccl().ok) {
    set_error("libnccl.so.2 could not be loaded");
    return PA_ENCCL;
  }
  if (device_count() == 0) {
    set_error("no CUDA device");
    return PA_ENOGPU;
  }
  std::unique_ptr<Comm> c(new Comm);
  c->nranks = nranks;
  c->rank = rank;
  CU(cudaGetDevice(&c->device));
  ncclUniqueId id;
  memcpy(&id, id128, sizeof id);
  if (g_tun.nccl_ctas > 0 && nccl().CommInitRankConfig) {
    ncclConfig_t cfg = NCCL_CONFIG_INITIALIZER;
    cfg.minCTAs = g_tun.nccl_ctas;
    cfg.maxCTAs = g_tun.nccl_ctas;
    NC(nccl().CommInitRankConfig(&c->comm, nranks, id, rank, &cfg));
  } else {
    NC(nccl().CommInitRank(&c->comm, nranks, id, rank));
  }
  {
    std::lock_guard<std::mutex> lock(g_live_mu);
    g_live_comms.insert((void*)c->comm);
  }
  pa_status rs = reduce_state_create(nranks, &c->reduce);
  if (rs != PA_OK) {
    comm_destroy(c.release());
    return rs;
  }
  *out = c.release();
  return PA_OK;
}

pa_status comm_init_local(int nranks, int rank, Comm** out) {
  if (device_count() == 0) {
    set_error("no CUDA device");
    return PA_ENOGPU;
  }
  std::unique_ptr<Comm> c(new Comm);
  c->nranks = nranks;
  c->rank = rank;
  CU(cudaGetDevice(&c->device));
  RC(reduce_state_create(nranks, &c->reduce));
  *out = c.release();
  return PA_OK;
}

void comm_destroy(Comm* c) {
  if (!c) return;
  if (c->comm) {
    {
      std::lock_guard<std::mutex> lock(g_live_mu);
      g_live_comms.erase((void*)c->comm);
    }
    if (nccl().ok) nccl().CommDestroy(c->comm);
  }
  reduce_state_destroy(c->reduce);
  for (const std::string& h : c->imported) ipc_release_handle(h.data());
  if (c->flags) cudaFree(c->flags);
  if (c->fence_err) cudaFreeHost(c->fence_err);
  delete c;
}

// flag window: allocate + export (the collective exchange is the caller's job)
pa_status comm_flags_export(Comm* c, void* handle64, i64* offset) {
  if (!c->flags) {
    // (a whole 2 MiB block of its own: small cudaMalloc allocations share a block, and
    //  a block can be opened only once per importing process)
    const size_t bytes = std::max<size_t>(window_bytes(c->nranks), IPC_BLOCK);
    CU(cudaMalloc((void**)&c->flags, bytes));
    CU(cudaMemset(c->flags, 0, bytes));
    CU(cudaHostAlloc((void**)&c->fence_err, sizeof(int), cudaHostAllocMapped));
    *c->fence_err = 0;
    CU(cudaDeviceSynchronize());
    c->peer_flags.assign(c->nranks, nullptr);
    for (int k = 0; k < FK_KINDS; ++k) {
      c->seq_tx[k].assign(c->nranks, 0);
      c->seq_rx[k].assign(c->nranks, 0);
    }
  }
  return ipc_export(c->flags, handle64, offset);
}

pa_status comm_flags_import(Comm* c, int rank, const void* handle64, i64 offset) {
  if (!c->flags || rank < 0 || rank >= c->nranks) {
    set_error("flag window: export first / rank out of range");
    return PA_ESTATE;
  }
  if (rank == c->rank) return PA_OK;
  void* p = nullptr;
  RC(ipc_import(handle64, offset, &p));
  c->imported.emplace_back((const char*)handle64, PA_IPC_HANDLE_BYTES);
  c->peer_flags[rank] = (ull*)p;
  bool all = true;
  for (int r = 0; r < c->nranks; ++r)
    if (r != c->rank && !c->peer_flags[r]) all = false;
  c->flags_ready = all;
  if (all && c->nranks > 1) {  // the reductions' peer words and slots (reduce.cu)
    const size_t so = reduce_slots_offset(c->nranks);
    std::vector<ull*> words(c->nranks, nullptr);
    std::vector<unsigned char*> slots(c->nranks, nullptr);
    for (int r = 0; r < c->nranks; ++r)
      if (r != c->rank) {
        words[r] = remote_word(c, r, FK_REDUCE);
        slots[r] = (unsigned char*)c->peer_flags[r] + so;
      }
    RC(reduce_state_set_tables(c->reduce, c->nranks, words.data(), slots.data()));
  }
  return PA_OK;
}

int comm_size(const Comm* c) { return c->nranks; }

pa_status comm_reduce_window(Comm* c, ReduceWindow* w) {
  RC(check_fence_err(c));
  w->nranks = c->nranks;
  w->rank = c->rank;
  w->flags = c->flags_ready && !g_tun.nccl_fences;
  w->nccl = c->comm != nullptr;
  w->state = &c->reduce;
  w->err = c->fence_err;
  w->timeout_ns = timeout_ns();
  if (!w->flags) return PA_OK;
  const size_t so = reduce_slots_offset(c->nranks);
  w->local_words = c->flags + FK_REDUCE;
  w->word_stride = FK_KINDS;
  w->local_slots = (unsigned char*)c->flags + so;
  return PA_OK;
}

pa_status comm_allgather(Comm* c, const void* send, void* recv, size_t bytes, void* stream) {
  if (!c->comm || !nccl().AllGather) {
    set_error("reduction: the communicator has neither a flag window nor ncclAllGather");
    return PA_ESTATE;
  }
  NC(nccl().AllGather(send, recv, bytes, ncclUint8, c->comm, (cudaStream_t)stream));
  return PA_OK;
}

// ---- staging arenas ----------------------------------------------------------
static void buffers_deregister(Buffers& b) {
  if (!b.reg_comm) return;
  bool live;
  {
    std::lock_guard<std::mutex> lock(g_live_mu);
    live = g_live_comms.count(b.reg_comm) != 0;
  }
  if (live && nccl().CommDeregister) {
    if (b.reg_send) nccl().CommDeregister((ncclComm_t)b.reg_comm, b.reg_send);
    if (b.reg_recv) nccl().CommDeregister((ncclComm_t)b.reg_comm, b.reg_recv);
  }
  b.reg_comm = b.reg_send = b.reg_recv = b.reg_send_ptr = b.reg_recv_ptr = nullptr;
}

static void free_arena(void* p, bool from_nccl) {
  if (!p) return;
  if (from_nccl && nccl().MemFree) nccl().MemFree(p);
  else cudaFree(p);
}

Buffers::~Buffers() {
  buffers_deregister(*this);
  free_arena(send, send_nccl);
  free_arena(recv, recv_nccl);
  if (comm_done_event) cudaEventDestroy((cudaEvent_t)comm_done_event);
  if (unpack_done_event) cudaEventDestroy((cudaEvent_t)unpack_done_event);
}

// grow-only, like resize! on the pencil's UInt8 vectors (Transpositions.jl:313-317)
pa_status Buffers::reserve(i64 send_bytes, i64 recv_bytes) {
  auto grow = [this](void*& p, i64& cap, bool& from_nccl, i64 need) -> pa_status {
    // (an arena from ncclMemAlloc is VMM memory: it cannot be exported with CUDA IPC,
    //  so the own-kernel exchange replaces it by a plain allocation)
    const bool wrong_kind = p && from_nccl && g_tun.ipc_exchange;
    if (need <= cap && !wrong_kind) return PA_OK;
    need = std::max(need, cap);
    // a previous exchange may still be reading/writing the old arena
    CU(cudaDeviceSynchronize());
    buffers_deregister(*this);
    free_arena(p, from_nccl);
    p = nullptr;
    cap = 0;
    // whole 2 MiB blocks: the arena may be exported over CUDA IPC, and allocations that
    // share a block cannot be opened separately by a peer
    i64 n = (need + (i64)IPC_BLOCK - 1) / (i64)IPC_BLOCK * (i64)IPC_BLOCK;
    from_nccl = false;
    // ncclMemAlloc only pays off (and NCCL is only touched at all) when an NCCL
    // communicator exists to register the arena with
    if (g_tun.nccl_register && !g_tun.ipc_exchange && any_live_nccl() && nccl().ok && nccl().MemAlloc &&
        nccl().MemFree && nccl().MemAlloc(&p, (size_t)n) == ncclSuccess && p) {
      from_nccl = true;
    } else {
      p = nullptr;
      cudaGetLastError();
      CU(cudaMalloc(&p, (size_t)n));
    }
    cap = n;
    ++generation;
    return PA_OK;
  };
  RC(grow(send, send_cap, send_nccl, send_bytes));
  return grow(recv, recv_cap, recv_nccl, recv_bytes);
}

// register the arenas with `comm` (no-op unless tunable nccl_register and ncclMemAlloc'ed arenas)
static void buffers_register(Buffers& b, ncclComm_t comm) {
  if (!g_tun.nccl_register || !nccl().CommRegister) return;
  if (b.reg_comm == (void*)comm && b.reg_send_ptr == b.send && b.reg_recv_ptr == b.recv) return;
  buffers_deregister(b);
  b.reg_comm = (void*)comm;
  if (b.send && b.send_nccl &&
      nccl().CommRegister(comm, b.send, (size_t)b.send_cap, &b.reg_send) != ncclSuccess)
    b.reg_send = nullptr;
  if (b.recv && b.recv_nccl &&
      nccl().CommRegister(comm, b.recv, (size_t)b.recv_cap, &b.reg_recv) != ncclSuccess)
    b.reg_recv = nullptr;
  b.reg_send_ptr = b.send;
  b.reg_recv_ptr = b.recv;
}

static pa_status buffer_events(Buffers& B, cudaEvent_t* comm_ev, cudaEvent_t* unpack_ev) {
  if (!B.comm_done_event) {
    cudaEvent_t e;
    CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    B.comm_done_event = e;
  }
  if (!B.unpack_done_event) {
    cudaEvent_t e;
    CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    B.unpack_done_event = e;
  }
  *comm_ev = (cudaEvent_t)B.comm_done_event;
  *unpack_ev = (cudaEvent_t)B.unpack_done_event;
  return PA_OK;
}

// A one-rank use of the recv arena on the caller's stream (the nproc == 1 staged self block,
// the aliased local permutation's scratch): it starts after the last exchange into the arena
// and the last unpack out of it, whatever stream those ran on ...
static pa_status arena_acquire(Buffers& B, cudaStream_t user) {
  cudaEvent_t comm_ev, unpack_ev;
  RC(buffer_events(B, &comm_ev, &unpack_ev));
  CU(cudaStreamWaitEvent(user, comm_ev, 0));
  CU(cudaStreamWaitEvent(user, unpack_ev, 0));
  return PA_OK;
}

// ... and the next user of the arena waits for it: both events move past its last read (the
// caller's stream already waited for their previous records, so the chain stays transitive)
static pa_status arena_release(Buffers& B, cudaStream_t user) {
  CU(cudaEventRecord((cudaEvent_t)B.comm_done_event, user));
  CU(cudaEventRecord((cudaEvent_t)B.unpack_done_event, user));
  return PA_OK;
}

// ---- per-plan stream/event state --------------------------------------------
struct TransposeState {
  cudaStream_t pack_s = nullptr, comm_s = nullptr, unpack_s = nullptr;
  cudaStream_t host_s = nullptr, h2d_s = nullptr, d2h_s = nullptr;
  cudaEvent_t ev_start = nullptr, ev_allpacked = nullptr, ev_comm_done = nullptr,
              ev_unpack_done = nullptr, ev_self_done = nullptr;
  std::vector<cudaEvent_t> ev_packed, ev_recvd;  // [step * chunks + chunk]
  std::vector<cudaEvent_t> ev_host;              // host pipeline (per chunk: upload, kernel)
  bool timing = false;
  bool timed_once = false;
  cudaEvent_t t[8] = {nullptr};  // 0 start,1 pack_end,2 comm0,3 comm1,4 unpack0,5 unpack1,6 end
  bool sends_pending = false;
  Comm* pending_comm = nullptr;
  char* tok = nullptr;  // 4-byte tokens of the NCCL line barrier: [0] sent, [1+n] received from n
  unsigned int* counter = nullptr;  // finished-CTA counter of the multi-peer launches
  // sub-blocks of the peers' pack / unpack descriptors for the current chunk count
  int chunks = 0;
  std::vector<std::vector<BlockCopy>> pack_c, unpack_c;
};

void destroy_state(TransposeState* st) {
  if (!st) return;
  for (cudaStream_t s : {st->pack_s, st->comm_s, st->unpack_s, st->host_s, st->h2d_s, st->d2h_s})
    if (s) cudaStreamDestroy(s);
  for (cudaEvent_t e : {st->ev_start, st->ev_allpacked, st->ev_comm_done, st->ev_unpack_done,
                        st->ev_self_done})
    if (e) cudaEventDestroy(e);
  for (auto e : st->ev_packed) cudaEventDestroy(e);
  for (auto e : st->ev_recvd) cudaEventDestroy(e);
  for (auto e : st->ev_host) cudaEventDestroy(e);
  for (auto e : st->t)
    if (e) cudaEventDestroy(e);
  if (st->tok) cudaFree(st->tok);
  if (st->counter) cudaFree(st->counter);
  delete st;
}

Plan::~Plan() {
  destroy_state(st);
  if (h_src_dev) cudaFree(h_src_dev);
  if (h_dst_dev) cudaFree(h_dst_dev);
}

static pa_status ensure_state(Plan* P) {
  if (P->st) return PA_OK;
  if (device_count() == 0) {
    set_error("no CUDA device: the transpose! path has no CPU fallback");
    return PA_ENOGPU;
  }
  std::unique_ptr<TransposeState> st(new TransposeState);
  int lo = 0, hi = 0;
  CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  CU(cudaStreamCreateWithPriority(&st->pack_s, cudaStreamNonBlocking, lo));
  CU(cudaStreamCreateWithPriority(&st->comm_s, cudaStreamNonBlocking, hi));  // exchange first
  CU(cudaStreamCreateWithPriority(&st->unpack_s, cudaStreamNonBlocking, lo));
  CU(cudaStreamCreateWithFlags(&st->host_s, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&st->h2d_s, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&st->d2h_s, cudaStreamNonBlocking));
  for (cudaEvent_t* e : {&st->ev_start, &st->ev_allpacked, &st->ev_comm_done, &st->ev_unpack_done,
                         &st->ev_self_done})
    CU(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  for (int i = 0; i < 7; ++i) CU(cudaEventCreate(&st->t[i]));
  CU(cudaMalloc((void**)&st->tok, 4 * (size_t)(P->nproc + 1)));
  CU(cudaMemset(st->tok, 0, 4 * (size_t)(P->nproc + 1)));
  CU(cudaMalloc((void**)&st->counter, sizeof(unsigned int)));
  CU(cudaMemset(st->counter, 0, sizeof(unsigned int)));
  CU(cudaDeviceSynchronize());
  P->st = st.release();
  return PA_OK;
}

static pa_status ensure_events(std::vector<cudaEvent_t>& v, size_t n) {
  while (v.size() < n) {
    cudaEvent_t e;
    CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    v.push_back(e);
  }
  return PA_OK;
}

// sub-blocks of every peer's pack / unpack descriptor for `chunks` pieces
static void ensure_chunks(Plan* P, int chunks) {
  TransposeState& S = *P->st;
  if (S.chunks == chunks) return;
  S.pack_c.assign(P->nproc, {});
  S.unpack_c.assign(P->nproc, {});
  for (int n = 0; n < P->nproc; ++n) {
    if (n == P->self_index) continue;
    for (int c = 0; c < chunks; ++c) {
      S.pack_c[n].push_back(sub_block(P->peers[n].pack, c, chunks, true, nullptr, nullptr));
      S.unpack_c[n].push_back(sub_block(P->peers[n].unpack, c, chunks, false, nullptr, nullptr));
    }
  }
  S.chunks = chunks;
}

pa_status plan_enable_timing(Plan* P, int on) {
  RC(ensure_state(P));
  P->st->timing = on != 0;
  return PA_OK;
}

pa_status plan_timings(Plan* P, pa_timings* out) {
  memset(out, 0, sizeof *out);
  if (!P->st || !P->st->timed_once) {
    set_error("no timed transpose! has run on this plan (pa_plan_enable_timing first)");
    return PA_ESTATE;
  }
  TransposeState& S = *P->st;
  CU(cudaEventSynchronize(S.t[6]));
  CU(cudaEventElapsedTime(&out->total_ms, S.t[0], S.t[6]));
  if (P->dim >= 0 && P->nproc > 1) {
    CU(cudaEventElapsedTime(&out->pack_ms, S.t[0], S.t[1]));
    CU(cudaEventElapsedTime(&out->exchange_ms, S.t[2], S.t[3]));
    CU(cudaEventElapsedTime(&out->unpack_ms, S.t[4], S.t[5]));
  }
  return PA_OK;
}

static bool ranges_overlap(const void* a, i64 na, const void* b, i64 nb) {
  const char* pa_ = (const char*)a;
  const char* pb = (const char*)b;
  return pa_ < pb + nb && pb < pa_ + na;
}

// transpose_impl!(::Nothing) (Transpositions.jl:213-270)
static pa_status local_transpose(Plan* P, const void* src, void* dst, void* scratch,
                                 cudaStream_t st) {
  const i64 bytes = P->length_out * P->elsize;
  if (P->same_perm) {
    if (src == dst) return PA_OK;  // copy!(uo, ui) onto itself
    return launch_block(P->self_fused, src, dst, st, nullptr, 0, true);
  }
  const bool inplace = ranges_overlap(src, bytes, dst, bytes);  // Base.mightalias (:249)
  if (!inplace) return launch_block(P->self_fused, src, dst, st, nullptr, 0, true);
  if (!scratch) {
    set_error("aliased local permutation needs a scratch buffer");
    return PA_EINVAL;
  }
  // permute into the temporary, then copy! to the output (:251-263)
  RC(launch_block(P->self_fused, src, scratch, st, nullptr, 0, true));
  CU(cudaMemcpyAsync(dst, scratch, (size_t)bytes, cudaMemcpyDeviceToDevice, st));
  return PA_OK;
}

pa_status permute_local(Plan* P, const void* src, void* dst, void* scratch, void* stream) {
  if (P->dim >= 0) {
    set_error("plan needs an exchange (dim = %d); use pa_transpose", P->dim + 1);
    return PA_ESTATE;
  }
  if (device_count() == 0) {
    set_error("no CUDA device");
    return PA_ENOGPU;
  }
  return local_transpose(P, src, dst, scratch, (cudaStream_t)stream);
}

// one dense run of `bytes` as a box copy (the IPC transport's block mover)
static BlockCopy contiguous_block(i64 bytes, const void* src, const void* dst) {
  BlockCopy b;
  int w = 16;
  const uintptr_t bits = (uintptr_t)bytes | (uintptr_t)src | (uintptr_t)dst;
  while (w > 1 && bits % w) w /= 2;
  b.elsize = w;
  b.nd_raw = 1;
  b.raw[0] = Dim{bytes / w, 1, 1};
  canonicalize(b);
  return b;
}

// ---- the one-sided methods --------------------------------------------------------

// PeerPut: each remote block is read from `src` and stored, already permuted,
// into the destination rank's `dest` through its peer mapping.  PeerGet is the
// pull flavour (window on `src`).  Protocol per transposition and pair of ranks:
// READY ("my side of the window may be touched": my dest may be overwritten /
// my src is final) before the first remote access, DONE ("all my accesses to
// your memory are complete") after the last.
// op on the receive side (PeerGet only, the complex FFT): the fused gather + FFT (k_get_fft)
// replaces the get kernel and the self block -- ONE kernel reads every line from the peers' src and
// the local src, transforms and stores it; the protocol around it is the same.
// op on the send side (PeerPut only): the send-side fused transform (k_fft_put, k_rfft_put,
// k_r2r_put, k_brfft_put) replaces the put kernel and the self block -- ONE kernel loads every
// local source line, transforms it and stores its outputs into the local dst and the peers' dst.
static pa_status one_sided(Plan* P, Comm* comm, const void* src, void* dst, unsigned flags,
                           const LineOp* op, cudaStream_t user) {
  TransposeState& S = *P->st;
  const int nproc = P->nproc, me = P->self_index;
  const bool get = P->method == PA_PEER_GET;
  const bool fft = op != nullptr;  // one fused kernel replaces the blocks
  const bool timing = S.timing;
  // (a rank none of whose peers owns anything has no window to register: nothing will be
  //  put / got, but it still speaks the protocol)
  auto w = P->windows.find(get ? src : (const void*)dst);
  const std::vector<void*> no_window(nproc, nullptr);
  const std::vector<void*>& win = (w == P->windows.end()) ? no_window : w->second;
  for (int n = 0; n < nproc; ++n)
    if (n != me && (get ? P->peers[n].recv_cnt : P->peers[n].send_cnt) > 0 &&
        ((int)win.size() <= n || !win[n])) {
      set_error("one-sided transpose: `%s` has no registered window for peer %d (pa_plan_set_window)",
                get ? "src" : "dest", n + 1);
      return PA_ESTATE;
    }
  RC(check_fence_err(comm));

  if (!fft) {
    // self block: fused K3 on the low-priority stream, beside the remote kernels
    if (timing) CU(cudaEventRecord(S.t[4], S.unpack_s));
    RC(launch_block(P->self_fused, src, dst, S.unpack_s, nullptr, g_tun.oneside_self_ctas));
    CU(cudaEventRecord(S.ev_unpack_done, S.unpack_s));
    if (timing) CU(cudaEventRecord(S.t[5], S.unpack_s));
  }
  if (timing) CU(cudaEventRecord(S.t[2], S.comm_s));
  if (timing && fft) CU(cudaEventRecord(S.t[4], S.comm_s));

  const bool use_flags = comm->flags_ready && !g_tun.nccl_fences;
  if (!use_flags && !comm->comm) {
    set_error("one-sided transpose: the communicator has neither a flag window nor NCCL");
    return PA_ESTATE;
  }

  // blocks in rotation order (me+k): every rank starts on a different peer
  std::vector<const BlockCopy*> blocks;
  std::vector<const void*> srcs;
  std::vector<void*> dsts;
  std::vector<int> peer_rank;
  for (int k = 1; k < nproc; ++k) {
    const int to = (me + k) % nproc, from = (me - k + nproc) % nproc;
    const int n = get ? from : to;
    blocks.push_back(get ? &P->peers[n].get : &P->peers[n].put);
    srcs.push_back(get ? (const void*)win[n] : src);
    dsts.push_back(get ? dst : win[n]);
    peer_rank.push_back(P->peers[n].world_rank);
  }
  const int np = nproc - 1;
  // fft: every get block and the self block in one kernel, `mf` spoken inside it (NULL: none);
  // *launched = false on a rank without destination lines
  // (send: the self block and every put block, stored into dst / the peers' dst)
  std::vector<const BlockCopy*> fb;
  std::vector<const void*> fs;
  std::vector<void*> fd;
  for (int n = 0; fft && n < nproc; ++n) {
    fb.push_back(n == me ? &P->self_fused : get ? &P->peers[n].get : &P->peers[n].put);
    fs.push_back(n == me ? src : (const void*)win[n]);
    fd.push_back(n == me ? dst : win[n]);
  }
  auto fused = [&](const MultiFlags* mf, bool* launched) {
    if (op->side == Side::put) return put_fft(nproc, fb.data(), src, fd.data(), *op, mf, S.comm_s, launched);
    return get_fft(nproc, fb.data(), fs.data(), dst, *op, mf, S.comm_s, launched);
  };
  bool launched = false;

  if (use_flags) {
    std::vector<ull*> rr(np), rl(np), dr(np), dl(np);
    std::vector<ull> rs(np), ds(np);
    for (int i = 0; i < np; ++i) {
      const int wr = peer_rank[i];
      rr[i] = remote_word(comm, wr, FK_READY);
      rl[i] = local_word(comm, wr, FK_READY);
      rs[i] = ++comm->seq_tx[FK_READY][wr];
      dr[i] = remote_word(comm, wr, FK_DONE);
      dl[i] = local_word(comm, wr, FK_DONE);
      ds[i] = ++comm->seq_tx[FK_DONE][wr];
    }
    pa_status rc = PA_EINCOMPAT;
    if (g_tun.multi_put && np <= FLAG_INLINE_MAX) {
      MultiFlags mf;
      memset(&mf, 0, sizeof mf);
      mf.ready.n = mf.done.n = np;
      for (int i = 0; i < np; ++i) {
        mf.ready.remote[i] = rr[i], mf.ready.local[i] = rl[i], mf.ready.seq[i] = rs[i];
        mf.done.remote[i] = dr[i], mf.done.local[i] = dl[i], mf.done.seq[i] = ds[i];
      }
      mf.wait_done = get ? 0 : 1;  // put: my dest is complete when every peer is done
      mf.counter = S.counter;
      mf.timeout_ns = timeout_ns();
      mf.err = comm->fence_err;
      if (fft) {
        RC(fused(&mf, &launched));
        // (no destination lines on this rank -- send: no source lines -- yet its peers still
        //  read its src / store into its dst, so the flag kernels below speak the protocol
        //  without a kernel between them)
        rc = launched ? PA_OK : PA_EINCOMPAT;
      } else {
        rc = launch_multi(np, blocks.data(), srcs.data(), dsts.data(), S.comm_s, g_tun.remote_ctas,
                          &mf);
      }
      if (rc != PA_OK && rc != PA_EINCOMPAT) return rc;
      if (rc == PA_OK) {
        CU(cudaEventRecord(S.ev_allpacked, S.comm_s));
        if (timing) CU(cudaEventRecord(S.t[1], S.comm_s));
        if (get)  // the wait for the peers' DONE only guards the reuse of src
          RC(launch_flags(np, nullptr, dl.data(), ds.data(), false, true, timeout_ns(),
                          comm->fence_err, S.comm_s));
      }
    }
    if (rc == PA_EINCOMPAT) {
      // blocks of different kernel flavours (or too many peers): same protocol,
      // spoken by standalone flag kernels around per-block launches
      RC(launch_flags(np, rr.data(), rl.data(), rs.data(), true, true, timeout_ns(),
                      comm->fence_err, S.comm_s));
      if (fft)
        RC(fused(nullptr, &launched));
      else
        for (int i = 0; i < np; ++i)
          RC(launch_block(*blocks[i], srcs[i], dsts[i], S.comm_s, nullptr, g_tun.remote_ctas));
      CU(cudaEventRecord(S.ev_allpacked, S.comm_s));
      if (timing) CU(cudaEventRecord(S.t[1], S.comm_s));
      RC(launch_flags(np, dr.data(), dl.data(), ds.data(), true, true, timeout_ns(),
                      comm->fence_err, S.comm_s));
    }
  } else {
    // NCCL fences: two tiny grouped send/recv rounds among the line's ranks
    auto line_barrier = [&]() -> pa_status {
      NC(nccl().GroupStart());
      for (int k = 1; k < nproc; ++k) {
        const int to = (me + k) % nproc, from = (me - k + nproc) % nproc;
        NC(nccl().Send(S.tok, 4, ncclUint8, P->peers[to].world_rank, comm->comm, S.comm_s));
        NC(nccl().Recv(S.tok + 4 * (1 + from), 4, ncclUint8, P->peers[from].world_rank, comm->comm,
                       S.comm_s));
      }
      NC(nccl().GroupEnd());
      return PA_OK;
    };
    RC(line_barrier());
    if (fft)
      RC(fused(nullptr, &launched));
    else
      for (int i = 0; i < np; ++i)
        RC(launch_block(*blocks[i], srcs[i], dsts[i], S.comm_s, nullptr, g_tun.remote_ctas));
    CU(cudaEventRecord(S.ev_allpacked, S.comm_s));
    if (timing) CU(cudaEventRecord(S.t[1], S.comm_s));
    RC(line_barrier());
  }
  if (fft) {
    // get: dst is complete once the fused kernel is (ev_allpacked); the DONE steps behind it on
    // the comm stream only guard the reuse of src.  send: the local part of dst is complete then,
    // the peers' parts at ev_comm_done, which the caller's stream waits for below
    CU(cudaStreamWaitEvent(S.unpack_s, S.ev_allpacked, 0));
    CU(cudaEventRecord(S.ev_unpack_done, S.unpack_s));
    if (timing) CU(cudaEventRecord(S.t[5], S.unpack_s));
  }
  CU(cudaEventRecord(S.ev_comm_done, S.comm_s));
  if (timing) CU(cudaEventRecord(S.t[3], S.comm_s));
  CU(cudaStreamWaitEvent(user, S.ev_allpacked, 0));
  CU(cudaStreamWaitEvent(user, S.ev_unpack_done, 0));
  // put: dest is complete only after the closing step (peers' stores have landed);
  // get: dest is complete once my loads are done, the closing step only guards
  //      the reuse of `src` -- exactly MPI.Waitall(t)'s role (:127-130).
  S.sends_pending = true;
  S.pending_comm = comm;
  if (!get || (flags & PA_WAITALL)) {
    CU(cudaStreamWaitEvent(user, S.ev_comm_done, 0));
    S.sends_pending = false;
  }
  return PA_OK;
}

// ---- the staged schedules (PointToPoint / Alltoallv) --------------------------------
// op (NULL: none): the fused unpack (receive side) that replaces the unpacks and the self block
static pa_status staged(Plan* P, Comm* comm, const void* src, void* dst, unsigned flags,
                        const LineOp* op, bool stage_self, cudaStream_t user, cudaEvent_t buf_ev,
                        cudaEvent_t buf_unpack_ev) {
  TransposeState& S = *P->st;
  Buffers& B = *P->pout->bufs;
  const int nproc = P->nproc, me = P->self_index;
  const bool overlap = !(flags & PA_NO_OVERLAP);
  const bool timing = S.timing;
  const i64 ES = P->elsize;
  char* sbuf = (char*)B.send;
  char* rbuf = (char*)B.recv;
  const Peer& self = P->peers[me];
  const bool ipc = !comm->comm || g_tun.ipc_exchange;
  const bool p2p = P->method != PA_ALLTOALLV;  // one-sided methods with aliased arrays run as PointToPoint
  const int C = p2p ? std::max(1, std::min(g_tun.p2p_chunks, 64)) : 1;
  const int cap = g_tun.staged_ctas;
  ensure_chunks(P, C);
  RC(ensure_events(S.ev_packed, (size_t)nproc * C));
  RC(ensure_events(S.ev_recvd, (size_t)nproc * C));

  if (ipc) {
    if (!comm->flags_ready) {
      set_error("staged transpose over peer memory: the communicator has no flag window");
      return PA_ESTATE;
    }
    if ((int)P->recv_windows.size() != nproc || P->recv_windows_gen != B.generation) {
      set_error("staged transpose over peer memory: the peers' recv_buf windows are missing or "
                "stale (pa_plan_set_recv_window after pa_pencil_reserve)");
      return PA_ESTATE;
    }
    for (int n = 0; n < nproc; ++n)
      if (n != me && P->peers[n].send_cnt > 0 && !P->recv_windows[n]) {
        set_error("staged transpose over peer memory: recv_buf window of peer %d is missing",
                  n + 1);
        return PA_ESTATE;
      }
    RC(check_fence_err(comm));
  }

  // ---- 1. pack ---------------------------------------------------------------
  // The remote blocks go first and alone: the exchange is the critical path, every
  // microsecond the first send waits for HBM is lost.  The self block follows on the
  // same stream (fused K3: src -> dest in one pass) and fills the HBM time the
  // NVLink-bound exchange leaves idle.  tunable "self_first" = 1 restores the
  // reference's order (self block packed first, :393-403).
  const bool fused = op != nullptr;
  const bool self_first = stage_self || g_tun.self_first;
  if (stage_self) {
    RC(launch_block(self.pack, src, rbuf, S.pack_s, nullptr));  // tail of recv_buf (:393-403)
  } else if (fused) {
    // (the fused unpack+FFT kernel gathers the self block straight out of src)
  } else if (self_first) {
    RC(launch_block(P->self_fused, src, dst, S.unpack_s, nullptr));  // K3, one pass
  }
  for (int k = 1; k < nproc; ++k) {
    const int to = (me + k) % nproc;
    for (int c = 0; c < C; ++c) {
      RC(launch_block(S.pack_c[to][c], src, sbuf, S.pack_s, nullptr, cap));
      CU(cudaEventRecord(S.ev_packed[k * C + c], S.pack_s));
    }
  }
  CU(cudaEventRecord(S.ev_allpacked, S.pack_s));
  if (timing) CU(cudaEventRecord(S.t[1], S.pack_s));
  if (!self_first && !fused) RC(launch_block(P->self_fused, src, dst, S.pack_s, nullptr, cap));
  CU(cudaEventRecord(S.ev_self_done, S.pack_s));

  // ---- 2. exchange -------------------------------------------------------------
  const int np = nproc - 1;
  std::vector<int> to_of(nproc), from_of(nproc);
  for (int k = 1; k < nproc; ++k) {
    to_of[k] = (me + k) % nproc;
    from_of[k] = (me - k + nproc) % nproc;
  }
  // byte range of chunk c of a pack (dense destination) / unpack (dense source) descriptor
  auto send_range = [&](int to, int c, i64* off, i64* len) {
    const BlockCopy& b = S.pack_c[to][c];
    *off = b.dst_off * b.elsize;
    *len = b.count * b.elsize;
  };
  auto recv_range = [&](int from, int c, i64* off, i64* len) {
    const BlockCopy& b = S.unpack_c[from][c];
    *off = b.src_off * b.elsize;
    *len = b.count * b.elsize;
  };

  if (ipc) {
    // window open: every peer's recv_buf may be overwritten (its previous unpack
    // has finished: the peer signals from its comm stream, behind its arena events)
    std::vector<ull*> rr(np), rl(np);
    std::vector<ull> rs(np);
    for (int k = 1; k < nproc; ++k) {
      const int wr = P->peers[to_of[k]].world_rank;
      rr[k - 1] = remote_word(comm, wr, FK_READY);
      rl[k - 1] = local_word(comm, wr, FK_READY);
      rs[k - 1] = ++comm->seq_tx[FK_READY][wr];
    }
    RC(launch_flags(np, rr.data(), rl.data(), rs.data(), true, true, timeout_ns(), comm->fence_err,
                    S.comm_s));
  }

  auto nccl_pair = [&](int to, int from, int c) -> pa_status {
    i64 so, sl, ro, rl;
    send_range(to, c, &so, &sl);
    recv_range(from, c, &ro, &rl);
    if (sl > 0)
      NC(nccl().Send(sbuf + so, (size_t)sl, ncclUint8, P->peers[to].world_rank, comm->comm,
                     S.comm_s));
    if (rl > 0)
      NC(nccl().Recv(rbuf + ro, (size_t)rl, ncclUint8, P->peers[from].world_rank, comm->comm,
                     S.comm_s));
    return PA_OK;
  };
  // IPC: my chunk stored into the peer's recv_buf, where the peer expects it
  auto ipc_copy = [&](int to, int c) -> pa_status {
    i64 so, sl;
    send_range(to, c, &so, &sl);
    if (sl <= 0) return PA_OK;
    const Peer& pt = P->peers[to];
    char* rdst = (char*)P->recv_windows[to] + pt.remote_recv_off * ES + (so - pt.send_off * ES);
    return launch_block(contiguous_block(sl, sbuf + so, rdst), sbuf + so, rdst, S.comm_s, nullptr,
                        g_tun.remote_ctas);
  };
  auto data_signal = [&](int to) -> pa_status {
    const int wr = P->peers[to].world_rank;
    ull* r = remote_word(comm, wr, FK_DATA);
    ull s = ++comm->seq_tx[FK_DATA][wr];
    return launch_flags(1, &r, nullptr, &s, true, false, timeout_ns(), comm->fence_err, S.comm_s);
  };
  auto data_wait = [&](int from, cudaStream_t st) -> pa_status {
    const int wr = P->peers[from].world_rank;
    ull* l = local_word(comm, wr, FK_DATA);
    ull s = ++comm->seq_rx[FK_DATA][wr];
    return launch_flags(1, nullptr, &l, &s, false, true, timeout_ns(), comm->fence_err, st);
  };

  if (p2p) {
    for (int k = 1; k < nproc; ++k) {
      const int to = to_of[k], from = from_of[k];
      for (int c = 0; c < C; ++c) {
        CU(cudaStreamWaitEvent(S.comm_s, overlap ? S.ev_packed[k * C + c] : S.ev_allpacked, 0));
        if (timing && k == 1 && c == 0) CU(cudaEventRecord(S.t[2], S.comm_s));
        if (!ipc) {
          NC(nccl().GroupStart());
          pa_status rc = nccl_pair(to, from, c);
          NC(nccl().GroupEnd());
          RC(rc);
          CU(cudaEventRecord(S.ev_recvd[k * C + c], S.comm_s));
        } else {
          i64 so, sl;
          send_range(to, c, &so, &sl);
          if (sl > 0) {
            RC(ipc_copy(to, c));
            RC(data_signal(to));
          }
        }
      }
    }
    if (ipc && (!overlap || fused)) {
      // sequential phases: every block has landed before the first unpack
      for (int k = 1; k < nproc; ++k)
        for (int c = 0; c < C; ++c) {
          i64 ro, rl;
          recv_range(from_of[k], c, &ro, &rl);
          if (rl > 0) RC(data_wait(from_of[k], S.comm_s));
        }
    }
  } else {
    // one collective-like step after all packs (MPI.Alltoallv!, :418-427)
    CU(cudaStreamWaitEvent(S.comm_s, S.ev_allpacked, 0));
    if (timing) CU(cudaEventRecord(S.t[2], S.comm_s));
    if (!ipc) {
      NC(nccl().GroupStart());
      pa_status rc = PA_OK;
      for (int k = 1; k < nproc && rc == PA_OK; ++k) rc = nccl_pair(to_of[k], from_of[k], 0);
      NC(nccl().GroupEnd());
      RC(rc);
    } else {
      // all blocks in one interleaved launch when they share a kernel flavour
      std::vector<BlockCopy> cb;
      std::vector<const BlockCopy*> bp;
      std::vector<const void*> ss;
      std::vector<void*> dd;
      cb.reserve(np);
      for (int k = 1; k < nproc; ++k) {
        i64 so, sl;
        send_range(to_of[k], 0, &so, &sl);
        if (sl <= 0) continue;
        const Peer& pt = P->peers[to_of[k]];
        char* rdst = (char*)P->recv_windows[to_of[k]] + pt.remote_recv_off * ES;
        cb.push_back(contiguous_block(sl, sbuf + so, rdst));
        ss.push_back(sbuf + so);
        dd.push_back(rdst);
      }
      for (auto& b : cb) bp.push_back(&b);
      pa_status rc = PA_EINCOMPAT;
      if (g_tun.multi_put && !bp.empty())
        rc = launch_multi((int)bp.size(), bp.data(), ss.data(), dd.data(), S.comm_s,
                          g_tun.remote_ctas, nullptr);
      if (rc == PA_EINCOMPAT)
        for (size_t i = 0; i < bp.size(); ++i)
          RC(launch_block(*bp[i], ss[i], dd[i], S.comm_s, nullptr, g_tun.remote_ctas));
      else
        RC(rc);
      for (int k = 1; k < nproc; ++k)
        if (P->peers[to_of[k]].send_cnt > 0) RC(data_signal(to_of[k]));
      for (int k = 1; k < nproc; ++k)
        if (P->peers[from_of[k]].recv_cnt > 0) RC(data_wait(from_of[k], S.comm_s));
    }
  }
  CU(cudaEventRecord(S.ev_comm_done, S.comm_s));
  CU(cudaEventRecord(buf_ev, S.comm_s));
  if (timing) CU(cudaEventRecord(S.t[3], S.comm_s));

  // ---- 3. unpack ------------------------------------------------------------
  // With aliased src/dest no unpack may start before every block is packed:
  // the reference finishes transpose_send! before transpose_recv! (:326-340).
  if (stage_self) CU(cudaStreamWaitEvent(S.unpack_s, S.ev_allpacked, 0));
  if (timing) CU(cudaEventRecord(S.t[4], S.unpack_s));
  if (fused) {
    // ONE kernel: gather every block (remote ones from recv_buf, the self block from src
    // or from the tail of recv_buf), transform along the now-local contiguous dim, store
    CU(cudaStreamWaitEvent(S.unpack_s, S.ev_comm_done, 0));
    std::vector<const BlockCopy*> bl;
    std::vector<const void*> sp;
    for (int n = 0; n < nproc; ++n) {
      const bool fused_self = (n == me) && !stage_self;
      bl.push_back(fused_self ? &P->self_fused : &P->peers[n].unpack);
      sp.push_back(fused_self ? src : (const void*)rbuf);
    }
    RC(unpack_fused(nproc, bl.data(), sp.data(), dst, *op, S.unpack_s));
  } else if (stage_self) {
    RC(launch_block(self.unpack, rbuf, dst, S.unpack_s, nullptr));  // local data first (:511)
  }
  if (fused) {
    // (nothing else to unpack)
  } else if (p2p && overlap) {
    for (int k = 1; k < nproc; ++k) {
      const int from = from_of[k];
      for (int c = 0; c < C; ++c) {
        i64 ro, rl;
        recv_range(from, c, &ro, &rl);
        if (rl <= 0) continue;
        if (ipc)
          RC(data_wait(from, S.unpack_s));
        else
          CU(cudaStreamWaitEvent(S.unpack_s, S.ev_recvd[k * C + c], 0));
        RC(launch_block(S.unpack_c[from][c], rbuf, dst, S.unpack_s, nullptr, cap));
      }
    }
  } else {
    CU(cudaStreamWaitEvent(S.unpack_s, S.ev_comm_done, 0));
    if (timing && !stage_self) CU(cudaEventRecord(S.t[4], S.unpack_s));
    for (int n = 0; n < nproc; ++n) {  // n = 1..Nproc in order (:508-509)
      if (n == me) continue;
      for (int c = 0; c < C; ++c) RC(launch_block(S.unpack_c[n][c], rbuf, dst, S.unpack_s, nullptr));
    }
  }
  CU(cudaEventRecord(S.ev_unpack_done, S.unpack_s));
  CU(cudaEventRecord(buf_unpack_ev, S.unpack_s));
  if (timing) CU(cudaEventRecord(S.t[5], S.unpack_s));

  // ---- join -----------------------------------------------------------------
  CU(cudaStreamWaitEvent(user, S.ev_self_done, 0));    // src may be reused by the caller
  CU(cudaStreamWaitEvent(user, S.ev_unpack_done, 0));  // dst complete
  S.sends_pending = true;
  S.pending_comm = comm;
  if (flags & PA_WAITALL) {
    CU(cudaStreamWaitEvent(user, S.ev_comm_done, 0));  // MPI.Waitall(t) (:174-176)
    S.sends_pending = false;
  }
  return PA_OK;
}

pa_status transpose(Plan* P, Comm* comm, const void* src, void* dst, unsigned flags,
                    void* stream, const LineOp* op) {
  RC(ensure_state(P));
  TransposeState& S = *P->st;
  cudaStream_t user = (cudaStream_t)stream;
  const i64 ES = P->elsize;
  const bool timing = S.timing;
  if (timing) CU(cudaEventRecord(S.t[0], user));
  auto timed_end = [&]() -> pa_status {
    if (timing) {
      CU(cudaEventRecord(S.t[6], user));
      S.timed_once = true;
    }
    return PA_OK;
  };

  if (op && (P->dim < 0 || P->nproc == 1)) {
    // one block, the whole local array: src -> T(permuted dest) / permuted T(src), one kernel on the
    // caller's stream
    const BlockCopy* b = &P->self_fused;
    if (op->side == Side::put) {
      bool launched = false;
      RC(put_fft(1, &b, src, &dst, *op, nullptr, user, &launched));
    } else {
      if (P->length_out == 0) return PA_OK;
      RC(unpack_fused(1, &b, &src, dst, *op, user));
    }
    return timed_end();
  }

  if (P->dim < 0) {
    void* scratch = nullptr;
    const i64 bytes = P->length_out * ES;
    if (bytes == 0) return PA_OK;
    const bool staged_local = !P->same_perm && ranges_overlap(src, bytes, dst, bytes);
    if (staged_local) {
      Buffers& Bi = *P->pin->bufs;
      RC(Bi.reserve(0, std::max<i64>(1, bytes)));  // reuses Pi.recv_buf (:255)
      scratch = Bi.recv;
      RC(arena_acquire(Bi, user));
    }
    RC(local_transpose(P, src, dst, scratch, user));
    if (staged_local) RC(arena_release(*P->pin->bufs, user));
    return timed_end();
  }

  const int nproc = P->nproc, me = P->self_index;
  if (nproc > 1 && !comm) {
    set_error("this transposition exchanges data among %d ranks: a communicator is required",
              nproc);
    return PA_ESTATE;
  }
  Buffers& B = *P->pout->bufs;  // Po.send_buf / Po.recv_buf (:313-317)
  // (same base pointer counts even when one side is empty on this rank: every rank of
  //  an in-place transpose must take the same schedule.  The real-line modes and the send side
  //  have refused aliased arrays at their entry points)
  const bool may_alias = !op || (op->side == Side::unpack && op->mode == FusedMode::fft);
  const bool aliased = may_alias && src && dst &&
      (src == dst || ranges_overlap(src, P->length_in * ES, dst, P->length_out * ES));
  const bool stage_self = aliased || (flags & PA_STAGE_SELF);
  const bool one = (P->method == PA_PEER_PUT || P->method == PA_PEER_GET) && !stage_self && nproc > 1;
  // (PeerGet runs the complex FFT one-sided, k_get_fft; a put has nothing to fuse with, and the
  //  real-line modes have been refused for both methods by their plan checks.  The send side runs
  //  on PeerPut plans only: their verdict)
  if (op && op->side == Side::unpack && one && (P->method == PA_PEER_PUT || op->mode != FusedMode::fft)) {
    set_error("fused FFT: the one-sided methods have no unpack pass to fuse with; use "
              "PointToPoint / Alltoallv");
    return PA_EINVAL;
  }
  if (!one) {
    // (one-sided puts/gets need no staging arenas)
    i64 need_send = nproc > 1 ? std::max<i64>(1, P->send_elems * ES) : 0;
    i64 need_recv = (nproc > 1 || stage_self) ? std::max<i64>(1, P->recv_elems * ES) : 0;
    RC(B.reserve(need_send, need_recv));
    if (comm && comm->comm && nproc > 1 && !g_tun.ipc_exchange) buffers_register(B, comm->comm);
  }
  const Peer& self = P->peers[me];

  if (nproc == 1) {
    // only the self block: no exchange, everything on the caller's stream
    if (stage_self) {
      char* rbuf = (char*)B.recv;
      RC(arena_acquire(B, user));
      RC(launch_block(self.pack, src, rbuf, user, nullptr, 0, true));
      RC(launch_block(self.unpack, rbuf, dst, user, nullptr, 0, true));
      RC(arena_release(B, user));
    } else {
      RC(launch_block(P->self_fused, src, dst, user, nullptr, 0, true));
    }
    return timed_end();
  }

  cudaEvent_t buf_ev, buf_unpack_ev;
  RC(buffer_events(B, &buf_ev, &buf_unpack_ev));
  // fork: the three streams start after the caller's prior work, after the
  // previous exchange that used these (shared) arenas and after the previous
  // unpack that was still reading recv_buf
  CU(cudaEventRecord(S.ev_start, user));
  for (cudaStream_t s : {S.pack_s, S.comm_s, S.unpack_s}) {
    CU(cudaStreamWaitEvent(s, S.ev_start, 0));
    CU(cudaStreamWaitEvent(s, buf_ev, 0));
    CU(cudaStreamWaitEvent(s, buf_unpack_ev, 0));
  }
  if (one)
    RC(one_sided(P, comm, src, dst, flags, op, user));
  else
    RC(staged(P, comm, src, dst, flags, op, stage_self, user, buf_ev, buf_unpack_ev));
  return timed_end();
}

// MPI.Waitall(t::Transposition) (Transpositions.jl:127-130)
pa_status wait_sends(Plan* P, void* stream) {
  if (!P->st) return PA_OK;
  RC(check_fence_err(P->st->pending_comm));
  if (!P->st->sends_pending) return PA_OK;
  CU(cudaStreamWaitEvent((cudaStream_t)stream, P->st->ev_comm_done, 0));
  P->st->sends_pending = false;
  return PA_OK;
}

// ---- host arrays -------------------------------------------------------------------
// Cuts of a purely local transposition (one kernel: nproc == 1 or dim == nothing)
// along the source's outermost dimension: each cut is a contiguous range of the
// source, so upload(c+1) || kernel(c) || download(c-1) pipeline on three streams;
// the download joins in only when the same dimension is outermost in the
// destination too (the cut is then contiguous there as well).
struct HostCuts {
  bool ok = false, dst_contiguous = false;
  std::vector<BlockCopy> blk;
  std::vector<i64> s_off, s_len, d_off, d_len;  // bytes
};

static HostCuts make_cuts(const Plan* P, i64 target_bytes) {
  HostCuts hc;
  if (!(P->dim < 0 || P->nproc == 1)) return hc;
  const BlockCopy& b = P->self_fused;
  if (b.count == 0) return hc;
  int j = -1;
  for (int i = b.nd_raw - 1; i >= 0; --i)
    if (b.raw[i].e > 1) {
      j = i;
      break;
    }
  if (j < 0) return hc;
  const i64 e = b.raw[j].e, W = b.elsize;
  if (b.raw[j].ss * e != b.count) return hc;  // not outermost in the source (cannot happen)
  hc.dst_contiguous = (b.raw[j].ds * e == b.count);
  const i64 total = b.count * W;
  i64 n = std::max<i64>(1, std::min<i64>(e, (total + target_bytes - 1) / std::max<i64>(1, target_bytes)));
  n = std::min<i64>(n, 256);
  for (i64 c = 0; c < n; ++c) {
    i64 so = 0, sc = 0;
    BlockCopy sb = sub_block(b, (int)c, (int)n, false, &so, &sc);
    hc.s_off.push_back(so * W);
    hc.s_len.push_back(sc * W);
    const i64 c0 = e * c / n, c1 = e * (c + 1) / n;
    hc.d_off.push_back(c0 * b.raw[j].ds * W);
    hc.d_len.push_back((c1 - c0) * b.raw[j].ds * W);
    hc.blk.push_back(sb);
  }
  hc.ok = true;
  return hc;
}

static pa_status grow_dev(void** p, i64* cap, i64 need) {
  if (need <= *cap) return PA_OK;
  if (*p) {
    CU(cudaDeviceSynchronize());
    CU(cudaFree(*p));
    *p = nullptr;
    *cap = 0;
  }
  CU(cudaMalloc(p, (size_t)std::max<i64>(need, 1)));
  *cap = need;
  return PA_OK;
}

// upload (+ first transposition) of one host array: H2D in cuts on `h2d`, the
// kernel of each cut on `ks` as soon as its cut has arrived
static pa_status upload_and_transpose(Plan* P, const HostCuts& hc, const void* hsrc, void* dsrc,
                                      void* ddst, cudaStream_t h2d, cudaStream_t ks,
                                      std::vector<cudaEvent_t>& evs) {
  const size_t n = hc.blk.size();
  RC(ensure_events(evs, 2 * n));
  for (size_t c = 0; c < n; ++c) {
    CU(cudaMemcpyAsync((char*)dsrc + hc.s_off[c], (const char*)hsrc + hc.s_off[c],
                       (size_t)hc.s_len[c], cudaMemcpyHostToDevice, h2d));
    CU(cudaEventRecord(evs[2 * c], h2d));
    CU(cudaStreamWaitEvent(ks, evs[2 * c], 0));
    RC(launch_block(hc.blk[c], dsrc, ddst, ks, nullptr, 0, true));
    CU(cudaEventRecord(evs[2 * c + 1], ks));
  }
  return PA_OK;
}

pa_status transpose_host(Plan* P, Comm* comm, const void* hsrc, void* hdst, unsigned flags) {
  RC(ensure_state(P));
  TransposeState& S = *P->st;
  const i64 nin = P->length_in * P->elsize, nout = P->length_out * P->elsize;
  RC(grow_dev(&P->h_src_dev, &P->h_src_cap, nin));
  RC(grow_dev(&P->h_dst_dev, &P->h_dst_cap, nout));
  if ((nin > 0 && !hsrc) || (nout > 0 && !hdst)) {
    set_error("pa_transpose_host: null host array");
    return PA_EINVAL;
  }
  const HostCuts hc = make_cuts(P, g_tun.host_chunk_bytes);
  if (hc.ok && hc.blk.size() > 1) {
    // upload(c+1) || kernel(c) || download(c-1)
    RC(upload_and_transpose(P, hc, hsrc, P->h_src_dev, P->h_dst_dev, S.h2d_s, S.host_s, S.ev_host));
    if (hc.dst_contiguous) {
      for (size_t c = 0; c < hc.blk.size(); ++c) {
        CU(cudaStreamWaitEvent(S.d2h_s, S.ev_host[2 * c + 1], 0));
        CU(cudaMemcpyAsync((char*)hdst + hc.d_off[c], (char*)P->h_dst_dev + hc.d_off[c],
                           (size_t)hc.d_len[c], cudaMemcpyDeviceToHost, S.d2h_s));
      }
    } else {
      CU(cudaStreamWaitEvent(S.d2h_s, S.ev_host[2 * hc.blk.size() - 1], 0));
      CU(cudaMemcpyAsync(hdst, P->h_dst_dev, (size_t)nout, cudaMemcpyDeviceToHost, S.d2h_s));
    }
    CU(cudaStreamSynchronize(S.d2h_s));
    return PA_OK;
  }
  cudaStream_t s = S.host_s;
  // (PA_FFT_* pass through to the one-call path only: the cuts above run plain copies)
  LineOp op;
  bool fused = false;
  RC(transpose_fft_op(P, flags, P->h_src_dev, P->h_dst_dev, &op, &fused));
  if (nin > 0) CU(cudaMemcpyAsync(P->h_src_dev, hsrc, (size_t)nin, cudaMemcpyHostToDevice, s));
  RC(transpose(P, comm, P->h_src_dev, P->h_dst_dev, flags | PA_WAITALL, s, fused ? &op : nullptr));
  if (nout > 0) CU(cudaMemcpyAsync(hdst, P->h_dst_dev, (size_t)nout, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return PA_OK;
}

// ---- host chains: upload -> transpose! ... transpose! -> download, asynchronous ------
// What a caller holding host arrays does around a sequence of transpositions
// (a PencilFFTs-style plan on `Array`s): one submit uploads the input, runs the
// chain on the device and downloads the result.  Submits are asynchronous and
// double-buffered on the device, so the download of one overlaps the upload of
// the next (PCIe is full duplex); inside a submit the first / last transposition
// is cut as in pa_transpose_host when it is purely local.
struct HostChain {
  std::vector<Plan*> plans;
  Comm* comm = nullptr;
  static constexpr int MAX_SLOTS = 4;
  int SLOTS = 2;  // device staging sets: submits that may be in flight at once (tunable "host_slots")
  void* buf[MAX_SLOTS][2] = {{nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}};
  i64 cap = 0;
  cudaStream_t h2d_s = nullptr, ks = nullptr, d2h_s = nullptr;
  cudaEvent_t ev_up[MAX_SLOTS] = {nullptr}, ev_k[MAX_SLOTS] = {nullptr}, ev_out[MAX_SLOTS] = {nullptr};
  std::vector<cudaEvent_t> evs[MAX_SLOTS], evs_last[MAX_SLOTS];
  cudaEvent_t t_mark = nullptr, t_end = nullptr;  // device-side timing of a run of submits
  HostCuts first, last;
  i64 submitted = 0;
  i64 ticket_of[MAX_SLOTS] = {-1, -1, -1, -1};
};

void host_chain_destroy(HostChain* c) {
  if (!c) return;
  cudaDeviceSynchronize();
  for (int s = 0; s < HostChain::MAX_SLOTS; ++s) {
    for (int k = 0; k < 2; ++k)
      if (c->buf[s][k]) cudaFree(c->buf[s][k]);
    for (cudaEvent_t e : {c->ev_up[s], c->ev_k[s], c->ev_out[s]})
      if (e) cudaEventDestroy(e);
    for (auto e : c->evs[s]) cudaEventDestroy(e);
    for (auto e : c->evs_last[s]) cudaEventDestroy(e);
  }
  for (cudaStream_t s : {c->h2d_s, c->ks, c->d2h_s})
    if (s) cudaStreamDestroy(s);
  for (cudaEvent_t e : {c->t_mark, c->t_end})
    if (e) cudaEventDestroy(e);
  delete c;
}

// CUDA-event bracket around a run of submits: begin = "the upload stream reaches
// this point", end = "the download stream has delivered everything submitted so far"
pa_status host_chain_time_begin(HostChain* c) {
  if (!c->t_mark) CU(cudaEventCreate(&c->t_mark));
  if (!c->t_end) CU(cudaEventCreate(&c->t_end));
  CU(cudaEventRecord(c->t_mark, c->h2d_s));
  return PA_OK;
}

pa_status host_chain_time_end(HostChain* c, float* ms) {
  if (!c->t_mark || !c->t_end) {
    set_error("pa_host_chain_time_end without pa_host_chain_time_begin");
    return PA_ESTATE;
  }
  CU(cudaEventRecord(c->t_end, c->d2h_s));
  CU(cudaEventSynchronize(c->t_end));
  CU(cudaEventElapsedTime(ms, c->t_mark, c->t_end));
  return PA_OK;
}

pa_status host_chain_create(int n, Plan* const* plans, Comm* comm, HostChain** out) {
  if (device_count() == 0) {
    set_error("no CUDA device: the transpose! path has no CPU fallback");
    return PA_ENOGPU;
  }
  std::unique_ptr<HostChain> c(new HostChain);
  for (int i = 0; i < n; ++i) {
    if (!plans[i]) return PA_EINVAL;
    if (i > 0 && (plans[i]->length_in != plans[i - 1]->length_out ||
                  plans[i]->elsize != plans[i - 1]->elsize)) {
      set_error("host chain: plan %d does not consume what plan %d produces", i + 1, i);
      return PA_EINCOMPAT;
    }
    c->plans.push_back(plans[i]);
    c->cap = std::max<i64>(c->cap, std::max(plans[i]->length_in, plans[i]->length_out) *
                                       (i64)plans[i]->elsize);
  }
  c->comm = comm;
  c->cap = std::max<i64>(c->cap, 1);
  c->SLOTS = std::max(2, std::min(g_tun.host_slots, (int)HostChain::MAX_SLOTS));
  auto fail = [&](pa_status s) {
    host_chain_destroy(c.release());
    return s;
  };
  for (int s = 0; s < c->SLOTS; ++s)
    for (int k = 0; k < 2; ++k)
      if (cudaMalloc(&c->buf[s][k], (size_t)c->cap) != cudaSuccess) {
        set_error("host chain: device staging allocation failed");
        cudaGetLastError();
        return fail(PA_ENOMEM);
      }
  for (cudaStream_t* s : {&c->h2d_s, &c->ks, &c->d2h_s})
    if (cudaStreamCreateWithFlags(s, cudaStreamNonBlocking) != cudaSuccess) return fail(PA_ECUDA);
  for (int s = 0; s < c->SLOTS; ++s)
    for (cudaEvent_t* e : {&c->ev_up[s], &c->ev_k[s], &c->ev_out[s]})
      if (cudaEventCreateWithFlags(e, cudaEventDisableTiming) != cudaSuccess) return fail(PA_ECUDA);
  c->first = make_cuts(c->plans.front(), g_tun.host_chunk_bytes);
  c->last = make_cuts(c->plans.back(), g_tun.host_chunk_bytes);
  if (!c->last.dst_contiguous) c->last.ok = false;
  *out = c.release();
  return PA_OK;
}

pa_status host_chain_buffer(HostChain* c, int slot, int which, void** p, i64* bytes) {
  if (slot < 0 || slot >= HostChain::MAX_SLOTS || which < 0 || which > 1) return PA_EINVAL;
  if (slot >= c->SLOTS) {
    if (p) *p = nullptr;
    if (bytes) *bytes = 0;
    return PA_OK;
  }
  if (p) *p = c->buf[slot][which];
  if (bytes) *bytes = c->cap;
  return PA_OK;
}

pa_status host_chain_submit(HostChain* c, const void* hsrc, void* hdst, i64* ticket) {
  const int n = (int)c->plans.size();
  const int slot = (int)(c->submitted % c->SLOTS);
  Plan* P0 = c->plans.front();
  Plan* Pl = c->plans.back();
  const i64 nin = P0->length_in * P0->elsize, nout = Pl->length_out * Pl->elsize;
  if ((nin > 0 && !hsrc) || (nout > 0 && !hdst)) {
    set_error("pa_host_chain_submit: null host array");
    return PA_EINVAL;
  }
  void* a = c->buf[slot][0];
  void* b = c->buf[slot][1];
  // this slot's previous result must have left the device
  CU(cudaStreamWaitEvent(c->h2d_s, c->ev_out[slot], 0));
  CU(cudaStreamWaitEvent(c->ks, c->ev_out[slot], 0));
  int i0 = 0;
  const bool cut_first = c->first.ok && c->first.blk.size() > 1 && !(n == 1 && !c->last.ok);
  if (cut_first) {
    RC(upload_and_transpose(P0, c->first, hsrc, a, b, c->h2d_s, c->ks, c->evs[slot]));
    std::swap(a, b);
    i0 = 1;
  } else {
    if (nin > 0) CU(cudaMemcpyAsync(a, hsrc, (size_t)nin, cudaMemcpyHostToDevice, c->h2d_s));
    CU(cudaEventRecord(c->ev_up[slot], c->h2d_s));
    CU(cudaStreamWaitEvent(c->ks, c->ev_up[slot], 0));
  }
  const bool cut_last = c->last.ok && c->last.blk.size() > 1 && !(n == 1 && cut_first);
  const int i1 = cut_last ? n - 1 : n;
  for (int i = i0; i < i1; ++i) {
    RC(transpose(c->plans[i], c->comm, a, b, PA_WAITALL, c->ks));
    std::swap(a, b);
  }
  if (n == 1 && cut_first) {
    // single purely local plan: the kernels of the cuts already ran; download per cut
    // when contiguous in the destination, else in one piece
    const HostCuts& hc = c->first;
    if (hc.dst_contiguous) {
      for (size_t k = 0; k < hc.blk.size(); ++k) {
        CU(cudaStreamWaitEvent(c->d2h_s, c->evs[slot][2 * k + 1], 0));
        CU(cudaMemcpyAsync((char*)hdst + hc.d_off[k], (char*)a + hc.d_off[k], (size_t)hc.d_len[k],
                           cudaMemcpyDeviceToHost, c->d2h_s));
      }
    } else {
      CU(cudaEventRecord(c->ev_k[slot], c->ks));
      CU(cudaStreamWaitEvent(c->d2h_s, c->ev_k[slot], 0));
      if (nout > 0) CU(cudaMemcpyAsync(hdst, a, (size_t)nout, cudaMemcpyDeviceToHost, c->d2h_s));
    }
  } else if (cut_last) {
    const HostCuts& hc = c->last;
    RC(ensure_events(c->evs_last[slot], hc.blk.size()));
    for (size_t k = 0; k < hc.blk.size(); ++k) {
      RC(launch_block(hc.blk[k], a, b, c->ks, nullptr, 0, true));
      CU(cudaEventRecord(c->evs_last[slot][k], c->ks));
      CU(cudaStreamWaitEvent(c->d2h_s, c->evs_last[slot][k], 0));
      CU(cudaMemcpyAsync((char*)hdst + hc.d_off[k], (char*)b + hc.d_off[k], (size_t)hc.d_len[k],
                         cudaMemcpyDeviceToHost, c->d2h_s));
    }
  } else {
    CU(cudaEventRecord(c->ev_k[slot], c->ks));
    CU(cudaStreamWaitEvent(c->d2h_s, c->ev_k[slot], 0));
    if (nout > 0) CU(cudaMemcpyAsync(hdst, a, (size_t)nout, cudaMemcpyDeviceToHost, c->d2h_s));
  }
  CU(cudaEventRecord(c->ev_out[slot], c->d2h_s));
  c->ticket_of[slot] = c->submitted;
  if (ticket) *ticket = c->submitted;
  ++c->submitted;
  return PA_OK;
}

pa_status host_chain_wait(HostChain* c, i64 ticket) {
  for (int s = 0; s < c->SLOTS; ++s) {
    if (c->ticket_of[s] < 0) continue;
    if (ticket >= 0 && c->ticket_of[s] > ticket) continue;  // a later submit: not asked for
    CU(cudaEventSynchronize(c->ev_out[s]));
  }
  return PA_OK;
}

}  // namespace pa
