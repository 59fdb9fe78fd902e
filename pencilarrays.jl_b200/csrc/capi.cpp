// extern "C" surface of libpa_b200 (see include/pa_b200.h).  Converts between
// the reference's 1-based / inclusive conventions and the 0-based internals.
#include <algorithm>
#include <new>
#include <vector>

#include "pa_internal.hpp"
#include "reduce_core.hpp"

using namespace pa;

#define GUARD(expr)                    \
  try {                                \
    expr                               \
  } catch (const std::bad_alloc&) {    \
    set_error("out of host memory");   \
    return PA_ENOMEM;                  \
  } catch (...) {                      \
    set_error("unexpected exception"); \
    return PA_EINVAL;                  \
  }

extern "C" {

const char* pa_version(void) { return "pa_b200 0.2.0 (sm_90a)"; }

const char* pa_strerror(pa_status s) {
  switch (s) {
    case PA_OK: return "success";
    case PA_EINVAL: return "invalid argument";
    case PA_EINCOMPAT: return "pencil configurations are not compatible for transposition";
    case PA_EDIM: return "array dimensions do not match the pencil";
    case PA_ECUDA: return "CUDA error";
    case PA_ENCCL: return "NCCL error";
    case PA_ENOMEM: return "out of memory";
    case PA_ESTATE: return "invalid call sequence";
    case PA_ENOGPU: return "no CUDA device (there is no CPU fallback)";
  }
  return "unknown status";
}

const char* pa_last_error(void) { return last_error(); }
int64_t pa_launch_count(void) { return launch_count(); }
int pa_device_count(void) { return device_count(); }
pa_status pa_set_device(int device) {
  if (device_count() == 0) {
    set_error("no CUDA device");
    return PA_ENOGPU;
  }
  return set_device(device);
}

pa_status pa_set_tunable(const char* name, int64_t value) {
  if (!name) return PA_EINVAL;
  if (!strcmp(name, "remote_ctas")) g_tun.remote_ctas = (int)value;
  else if (!strcmp(name, "box_copy_ctas")) g_tun.box_copy_ctas = (int)value;
  else if (!strcmp(name, "nccl_fences")) g_tun.nccl_fences = (int)value;
  else if (!strcmp(name, "bulk_rows")) g_tun.bulk_rows = (int)value;
  else if (!strcmp(name, "nccl_register")) g_tun.nccl_register = (int)value;
  else if (!strcmp(name, "transpose_tbq")) g_tun.transpose_tbq = (int)value;
  else if (!strcmp(name, "small_block_bytes")) g_tun.small_block_bytes = value;
  else if (!strcmp(name, "transpose_y_fastest")) g_tun.transpose_y_fastest = (int)value;
  else if (!strcmp(name, "multi_put")) g_tun.multi_put = (int)value;
  else if (!strcmp(name, "fft_lines")) g_tun.fft_lines = (int)value;
  else if (!strcmp(name, "oneside_self_ctas")) g_tun.oneside_self_ctas = (int)value;
  else if (!strcmp(name, "p2p_chunks")) g_tun.p2p_chunks = (int)value;
  else if (!strcmp(name, "staged_ctas")) g_tun.staged_ctas = (int)value;
  else if (!strcmp(name, "self_first")) g_tun.self_first = (int)value;
  else if (!strcmp(name, "ipc_exchange")) g_tun.ipc_exchange = (int)value;
  else if (!strcmp(name, "fence_timeout_ms")) g_tun.fence_timeout_ms = value;
  else if (!strcmp(name, "pdl")) g_tun.pdl = (int)value;
  else if (!strcmp(name, "nccl_ctas")) g_tun.nccl_ctas = (int)value;
  else if (!strcmp(name, "host_chunk_bytes")) g_tun.host_chunk_bytes = value;
  else if (!strcmp(name, "host_slots")) g_tun.host_slots = (int)value;
  else {
    set_error("unknown tunable '%s'", name);
    return PA_EINVAL;
  }
  return PA_OK;
}

// ---- topology -----------------------------------------------------------------
pa_status pa_dims_create(int nprocs, int M, int64_t* dims) {
  if (nprocs < 1 || M < 1 || M > PA_MAX_TOPO || !dims) {
    set_error("pa_dims_create: bad arguments");
    return PA_EINVAL;
  }
  // balanced factorisation: hand the prime factors, largest first, to the
  // currently smallest dimension; report in non-increasing order
  for (int i = 0; i < M; ++i) dims[i] = 1;
  int64_t primes[64];
  int np = 0;
  int n = nprocs;
  for (int f = 2; (int64_t)f * f <= n; ++f)
    while (n % f == 0) {
      primes[np++] = f;
      n /= f;
    }
  if (n > 1) primes[np++] = n;
  for (int k = np - 1; k >= 0; --k) {
    int j = 0;
    for (int i = 1; i < M; ++i)
      if (dims[i] < dims[j]) j = i;
    dims[j] *= primes[k];
  }
  std::sort(dims, dims + M, [](int64_t a, int64_t b) { return a > b; });
  return PA_OK;
}

pa_status pa_topology_create(int M, const int64_t* dims, int world_rank, pa_topology** out) {
  GUARD({
    if (M < 1 || M > PA_MAX_TOPO || !dims || !out) {
      set_error("topology must have 1..%d dimensions", PA_MAX_TOPO);
      return PA_EINVAL;
    }
    auto t = std::make_shared<Topology>();
    t->M = M;
    int64_t size = 1;
    for (int i = 0; i < M; ++i) {
      if (dims[i] < 1) {
        set_error("process grid dimensions must be >= 1");
        return PA_EINVAL;
      }
      t->dims[i] = dims[i];
      size *= dims[i];
    }
    if (world_rank < 0 || world_rank >= size) {
      set_error("rank %d outside of a %lld-process grid", world_rank, (long long)size);
      return PA_EINVAL;
    }
    t->size = (int)size;
    t->rank = world_rank;
    t->coords_of(world_rank, t->coords);
    *out = new pa_topology{t};
    return PA_OK;
  })
}

void pa_topology_destroy(pa_topology* t) { delete t; }

pa_status pa_topology_info(const pa_topology* t, int* M, int64_t* dims, int* world_rank,
                           int* world_size, int64_t* coords_local) {
  if (!t) return PA_EINVAL;
  const Topology& T = *t->p;
  if (M) *M = T.M;
  if (world_rank) *world_rank = T.rank;
  if (world_size) *world_size = T.size;
  for (int i = 0; i < T.M; ++i) {
    if (dims) dims[i] = T.dims[i];
    if (coords_local) coords_local[i] = T.coords[i] + 1;
  }
  return PA_OK;
}

pa_status pa_topology_rank_of(const pa_topology* t, const int64_t* coords, int* rank) {
  if (!t || !coords || !rank) return PA_EINVAL;
  const Topology& T = *t->p;
  int64_t c[PA_MAX_TOPO];
  for (int i = 0; i < T.M; ++i) {
    if (coords[i] < 1 || coords[i] > T.dims[i]) {
      set_error("coordinate %d out of range", i + 1);
      return PA_EINVAL;
    }
    c[i] = coords[i] - 1;
  }
  *rank = T.rank_of(c);
  return PA_OK;
}

pa_status pa_topology_line(const pa_topology* t, int R, int* ranks) {
  if (!t || !ranks) return PA_EINVAL;
  const Topology& T = *t->p;
  if (R < 1 || R > T.M) {
    set_error("grid dimension %d out of range 1:%d", R, T.M);
    return PA_EINVAL;
  }
  int64_t c[PA_MAX_TOPO];
  for (int i = 0; i < T.M; ++i) c[i] = T.coords[i];
  for (int64_t n = 0; n < T.dims[R - 1]; ++n) {
    c[R - 1] = n;
    ranks[n] = T.rank_of(c);
  }
  return PA_OK;
}

// ---- pencil -------------------------------------------------------------------
pa_status pa_pencil_create(pa_topology* topo, int N, const int64_t* size_global,
                           const int* decomp_dims, const int* perm, pa_pencil* share_with,
                           pa_pencil** out) {
  GUARD({
    if (!topo || !size_global || !decomp_dims || !out) return PA_EINVAL;
    const int M = topo->p->M;
    if (N < 1 || N > PA_MAX_DIMS) {
      set_error("number of dimensions must be in 1:%d", PA_MAX_DIMS);
      return PA_EINVAL;
    }
    // _check_selected_dimensions (Pencils.jl:397-412)
    if (M > N) {
      set_error("number of decomposed dimensions `M` cannot be larger than N = %d (got M = %d)", N,
                M);
      return PA_EINVAL;
    }
    auto p = std::make_shared<Pencil>();
    p->topo = topo->p;
    p->N = N;
    for (int d = 0; d < N; ++d) {
      if (size_global[d] < 0) {
        set_error("negative global size");
        return PA_EINVAL;
      }
      p->size_global[d] = size_global[d];
    }
    for (int i = 0; i < M; ++i) {
      if (decomp_dims[i] < 1 || decomp_dims[i] > N) {
        set_error("dimensions must be in 1:%d", N);
        return PA_EINVAL;
      }
      for (int j = 0; j < i; ++j)
        if (decomp_dims[j] == decomp_dims[i]) {
          set_error("dimensions may not be repeated");
          return PA_EINVAL;
        }
      p->decomp[i] = decomp_dims[i] - 1;
    }
    bool seen[PA_MAX_DIMS] = {false};
    p->perm_identity = true;
    for (int d = 0; d < N; ++d) {
      int v = perm ? perm[d] : d + 1;
      if (v < 1 || v > N || seen[v - 1]) {  // check_permutation (Pencils.jl:384-387)
        set_error("invalid permutation of dimensions");
        return PA_EINVAL;
      }
      seen[v - 1] = true;
      p->perm[d] = v - 1;
      if (v - 1 != d) p->perm_identity = false;
    }
    p->bufs = share_with ? share_with->p->bufs : std::make_shared<Buffers>();
    *out = new pa_pencil{p};
    return PA_OK;
  })
}

void pa_pencil_destroy(pa_pencil* p) { delete p; }

pa_status pa_pencil_range(const pa_pencil* p, const int64_t* coords, int memory_order, int64_t* lo,
                          int64_t* hi) {
  if (!p || !lo || !hi) return PA_EINVAL;
  const Pencil& P = *p->p;
  int64_t c[PA_MAX_TOPO], l[PA_MAX_DIMS], h[PA_MAX_DIMS];
  for (int i = 0; i < P.topo->M; ++i) {
    if (coords) {
      if (coords[i] < 1 || coords[i] > P.topo->dims[i]) {
        set_error("coordinate %d out of range", i + 1);
        return PA_EINVAL;
      }
      c[i] = coords[i] - 1;
    } else {
      c[i] = P.topo->coords[i];
    }
  }
  P.range_of(c, l, h);
  for (int m = 0; m < P.N; ++m) {
    int d = memory_order ? P.perm[m] : m;  // (perm * t)[m] = t[perm[m]]
    lo[m] = l[d] + 1;
    hi[m] = h[d];
  }
  return PA_OK;
}

pa_status pa_pencil_size_local(const pa_pencil* p, int memory_order, int64_t* dims) {
  if (!p || !dims) return PA_EINVAL;
  int64_t lo[PA_MAX_DIMS], hi[PA_MAX_DIMS];
  pa_status s = pa_pencil_range(p, nullptr, memory_order, lo, hi);
  if (s != PA_OK) return s;
  for (int d = 0; d < p->p->N; ++d) dims[d] = hi[d] - lo[d] + 1;
  return PA_OK;
}

pa_status pa_pencil_buffers(const pa_pencil* p, void** send_buf, int64_t* send_cap,
                            void** recv_buf, int64_t* recv_cap) {
  if (!p) return PA_EINVAL;
  const Buffers& b = *p->p->bufs;
  if (send_buf) *send_buf = b.send;
  if (send_cap) *send_cap = b.send_cap;
  if (recv_buf) *recv_buf = b.recv;
  if (recv_cap) *recv_cap = b.recv_cap;
  return PA_OK;
}

pa_status pa_pencil_reserve(pa_pencil* p, int64_t send_bytes, int64_t recv_bytes) {
  if (!p) return PA_EINVAL;
  if (device_count() == 0) {
    set_error("no CUDA device");
    return PA_ENOGPU;
  }
  return p->p->bufs->reserve(send_bytes, recv_bytes);
}

// ---- plan ---------------------------------------------------------------------
pa_status pa_plan_create(pa_pencil* pin, pa_pencil* pout, int n_extra, const int64_t* extra_dims,
                         int elsize, pa_method method, pa_plan** out) {
  GUARD({
    if (!pin || !pout || !out || (n_extra > 0 && !extra_dims)) return PA_EINVAL;
    Plan* P = nullptr;
    pa_status s = build_plan(pin->p, pout->p, n_extra, extra_dims, elsize, (int)method, &P);
    if (s != PA_OK) return s;
    *out = new pa_plan{P};
    return PA_OK;
  })
}

void pa_plan_destroy(pa_plan* plan) {
  if (!plan) return;
  delete plan->p;
  delete plan;
}

pa_status pa_plan_get_info(const pa_plan* plan, pa_plan_info* info) {
  if (!plan || !info) return PA_EINVAL;
  const Plan& P = *plan->p;
  info->dim = P.dim + 1;
  info->nproc = P.nproc;
  info->self_index = P.self_index + 1;
  info->same_perm = P.same_perm;
  info->elsize = P.elsize;
  info->method = P.method;
  info->length_in = P.length_in;
  info->length_out = P.length_out;
  info->length_self = P.length_self;
  info->send_bytes = P.send_elems * P.elsize;
  info->recv_bytes = P.recv_elems * P.elsize;
  return PA_OK;
}

pa_status pa_plan_get_peer(const pa_plan* plan, int n, pa_peer_info* info) {
  if (!plan || !info) return PA_EINVAL;
  const Plan& P = *plan->p;
  if (P.dim < 0 || n < 1 || n > P.nproc) {
    set_error("peer index %d out of range", n);
    return PA_EINVAL;
  }
  const Peer& pr = P.peers[n - 1];
  const int64_t S = P.elsize;
  info->world_rank = pr.world_rank;
  info->is_self = pr.is_self;
  info->send_offset = pr.send_off * S;
  info->send_count = pr.send_cnt * S;
  info->recv_offset = pr.recv_off * S;
  info->recv_count = pr.recv_cnt * S;
  info->remote_recv_offset = pr.remote_recv_off * S;
  return PA_OK;
}

static void export_block(const BlockCopy& b, pa_block_desc* d) {
  memset(d, 0, sizeof *d);
  d->nd = b.nd_raw;
  for (int i = 0; i < b.nd_raw; ++i) {
    d->extent[i] = b.raw[i].e;
    d->src_stride[i] = b.raw[i].ss;
    d->dst_stride[i] = b.raw[i].ds;
  }
  d->src_offset = b.src_off;
  d->dst_offset = b.dst_off;
  d->kernel_class = b.klass;
  d->vec_bytes = b.stride_align;
}

pa_status pa_plan_get_block(const pa_plan* plan, int op, int n, pa_block_desc* desc) {
  if (!plan || !desc) return PA_EINVAL;
  const Plan& P = *plan->p;
  if (op == 2) {
    export_block(P.self_fused, desc);
    return PA_OK;
  }
  if (P.dim < 0 || n < 1 || n > P.nproc || op < 0 || op > 4) {
    set_error("bad block selector (op=%d, n=%d)", op, n);
    return PA_EINVAL;
  }
  const Peer& pr = P.peers[n - 1];
  export_block(op == 0 ? pr.pack : op == 1 ? pr.unpack : op == 3 ? pr.put : pr.get, desc);
  return PA_OK;
}

pa_status pa_plan_get_chunk(const pa_plan* plan, int op, int n, int part, int nparts,
                            pa_block_desc* desc, int64_t* wire_offset, int64_t* wire_bytes) {
  if (!plan || !desc) return PA_EINVAL;
  const Plan& P = *plan->p;
  if (P.dim < 0 || n < 1 || n > P.nproc || op < 0 || op > 1 || nparts < 1 || part < 0 ||
      part >= nparts) {
    set_error("bad chunk selector (op=%d, n=%d, part=%d/%d)", op, n, part, nparts);
    return PA_EINVAL;
  }
  const Peer& pr = P.peers[n - 1];
  const BlockCopy c = sub_block(op == 0 ? pr.pack : pr.unpack, part, nparts, op == 0, nullptr, nullptr);
  export_block(c, desc);
  if (wire_offset) *wire_offset = (op == 0 ? c.dst_off : c.src_off) * c.elsize;
  if (wire_bytes) *wire_bytes = c.count * c.elsize;
  return PA_OK;
}

// ---- kernels --------------------------------------------------------------------
static pa_status need_gpu() {
  if (device_count() == 0) {
    set_error("no CUDA device: the transpose! path has no CPU fallback");
    return PA_ENOGPU;
  }
  return PA_OK;
}

pa_status pa_pack(pa_plan* plan, int n, const void* src, void* buf, void* stream) {
  if (!plan) return PA_EINVAL;
  Plan& P = *plan->p;
  if (P.dim < 0 || n < 1 || n > P.nproc) {
    set_error("peer index %d out of range", n);
    return PA_EINVAL;
  }
  pa_status s = need_gpu();
  if (s != PA_OK) return s;
  return launch_block(P.peers[n - 1].pack, src, buf, stream, nullptr);
}

pa_status pa_unpack(pa_plan* plan, int n, const void* recv_buf, void* dst, void* stream) {
  if (!plan) return PA_EINVAL;
  Plan& P = *plan->p;
  if (P.dim < 0 || n < 1 || n > P.nproc) {
    set_error("peer index %d out of range", n);
    return PA_EINVAL;
  }
  pa_status s = need_gpu();
  if (s != PA_OK) return s;
  return launch_block(P.peers[n - 1].unpack, recv_buf, dst, stream, nullptr);
}

pa_status pa_put(pa_plan* plan, int n, const void* src, void* peer_dst, void* stream) {
  if (!plan) return PA_EINVAL;
  Plan& P = *plan->p;
  if (P.dim < 0 || n < 1 || n > P.nproc || P.peers[n - 1].is_self) {
    set_error("pa_put: peer index %d out of range (or self)", n);
    return PA_EINVAL;
  }
  pa_status s = need_gpu();
  if (s != PA_OK) return s;
  return launch_block(P.peers[n - 1].put, src, peer_dst, stream, nullptr);
}

pa_status pa_get(pa_plan* plan, int n, const void* peer_src, void* dst, void* stream) {
  if (!plan) return PA_EINVAL;
  Plan& P = *plan->p;
  if (P.dim < 0 || n < 1 || n > P.nproc || P.peers[n - 1].is_self) {
    set_error("pa_get: peer index %d out of range (or self)", n);
    return PA_EINVAL;
  }
  pa_status s = need_gpu();
  if (s != PA_OK) return s;
  return launch_block(P.peers[n - 1].get, peer_src, dst, stream, nullptr);
}

static pa_status all_blocks(pa_plan* plan, bool get, const void* local, void* const* peers,
                            int max_ctas, void* stream) {
  if (!plan || !peers) return PA_EINVAL;
  Plan& P = *plan->p;
  if (P.dim < 0) {
    set_error("plan has no exchange");
    return PA_EINVAL;
  }
  pa_status s = need_gpu();
  if (s != PA_OK) return s;
  std::vector<const BlockCopy*> blocks;
  std::vector<const void*> srcs;
  std::vector<void*> dsts;
  for (int k = 1; k < P.nproc; ++k) {
    const int n = get ? (P.self_index - k + P.nproc) % P.nproc : (P.self_index + k) % P.nproc;
    const BlockCopy& b = get ? P.peers[n].get : P.peers[n].put;
    if (b.klass == KC_EMPTY) continue;
    blocks.push_back(&b);
    srcs.push_back(get ? (const void*)peers[n] : local);
    dsts.push_back(get ? (void*)local : peers[n]);
  }
  if (blocks.empty()) return PA_OK;
  if (max_ctas == 0) max_ctas = g_tun.remote_ctas;
  s = launch_multi((int)blocks.size(), blocks.data(), srcs.data(), dsts.data(), stream, max_ctas,
                   nullptr);
  if (s != PA_EINCOMPAT) return s;
  for (size_t i = 0; i < blocks.size(); ++i) {
    s = launch_block(*blocks[i], srcs[i], dsts[i], stream, nullptr, max_ctas);
    if (s != PA_OK) return s;
  }
  return PA_OK;
}

pa_status pa_put_all(pa_plan* plan, const void* src, void* const* peers, int max_ctas,
                     void* stream) {
  GUARD({ return all_blocks(plan, false, src, peers, max_ctas, stream); })
}

pa_status pa_get_all(pa_plan* plan, void* const* peers, void* dst, int max_ctas, void* stream) {
  GUARD({ return all_blocks(plan, true, dst, peers, max_ctas, stream); })
}

// src / dst of the local arrays: NULL only when empty, not overlapping, dst 16-byte aligned
static pa_status fused_pointers(const char* who, const void* src, i64 src_bytes, const void* dst,
                                i64 dst_bytes) {
  if ((!src && src_bytes > 0) || (!dst && dst_bytes > 0)) {
    set_error("%s: null array pointer for a non-empty local array", who);
    return PA_EINVAL;
  }
  const uintptr_t a = (uintptr_t)src, b = (uintptr_t)dst;
  if (src_bytes > 0 && dst_bytes > 0 && a < b + (uintptr_t)dst_bytes && b < a + (uintptr_t)src_bytes) {
    set_error("%s: src and dst overlap", who);
    return PA_EINVAL;
  }
  if (dst_bytes > 0 && (b & 15)) {
    set_error("%s: dst must be 16-byte aligned", who);
    return PA_EINVAL;
  }
  return PA_OK;
}

pa_status pa_copy_self(pa_plan* plan, const void* src, void* dst, void* stream) {
  if (!plan) return PA_EINVAL;
  pa_status s = need_gpu();
  if (s != PA_OK) return s;
  return launch_block(plan->p->self_fused, src, dst, stream, nullptr);
}

pa_status pa_permute_local(pa_plan* plan, const void* src, void* dst, void* scratch,
                           void* stream) {
  if (!plan) return PA_EINVAL;
  return permute_local(plan->p, src, dst, scratch, stream);
}

pa_status pa_box_copy(int nd, const int64_t* extent, const int64_t* src_stride,
                      const int64_t* dst_stride, int elsize, const void* src, void* dst,
                      void* stream, pa_block_desc* chosen) {
  if (nd < 0 || nd > PA_MAX_DIMS || (nd > 0 && (!extent || !src_stride || !dst_stride))) {
    set_error("pa_box_copy: 0..%d dimensions", PA_MAX_DIMS);
    return PA_EINVAL;
  }
  if (elsize != 1 && elsize != 2 && elsize != 4 && elsize != 8 && elsize != 16) {
    set_error("pa_box_copy: element size must be 1, 2, 4, 8 or 16");
    return PA_EINVAL;
  }
  BlockCopy b;
  b.elsize = elsize;
  b.nd_raw = nd;
  for (int i = 0; i < nd; ++i) {
    if (extent[i] < 0 || src_stride[i] < 0 || dst_stride[i] < 0) {
      set_error("pa_box_copy: negative extent or stride");
      return PA_EINVAL;
    }
    b.raw[i] = Dim{extent[i], src_stride[i], dst_stride[i]};
  }
  canonicalize(b);
  int vec = 0;
  pa_status s = PA_OK;
  if (src || dst) {
    s = need_gpu();
    if (s != PA_OK) return s;
    s = launch_block(b, src, dst, stream, &vec, g_tun.box_copy_ctas);
  }
  if (chosen) {
    export_block(b, chosen);
    if (vec) chosen->vec_bytes = vec;
  }
  return s;
}

// ---- communicator ----------------------------------------------------------------
pa_status pa_comm_unique_id(void* id128) {
  if (!id128) return PA_EINVAL;
  return comm_unique_id(id128);
}

pa_status pa_comm_init_rank(const void* id128, int nranks, int rank, pa_comm** out) {
  GUARD({
    if (!id128 || !out || nranks < 1 || rank < 0 || rank >= nranks) return PA_EINVAL;
    Comm* c = nullptr;
    pa_status s = comm_init(id128, nranks, rank, &c);
    if (s != PA_OK) return s;
    *out = new pa_comm{c};
    return PA_OK;
  })
}

pa_status pa_comm_init_local(int nranks, int rank, pa_comm** out) {
  GUARD({
    if (!out || nranks < 1 || rank < 0 || rank >= nranks) return PA_EINVAL;
    Comm* c = nullptr;
    pa_status s = comm_init_local(nranks, rank, &c);
    if (s != PA_OK) return s;
    *out = new pa_comm{c};
    return PA_OK;
  })
}

pa_status pa_comm_flags_export(pa_comm* c, void* handle64, int64_t* offset) {
  if (!c || !handle64 || !offset) return PA_EINVAL;
  return comm_flags_export(c->p, handle64, offset);
}

pa_status pa_comm_flags_import(pa_comm* c, int rank, const void* handle64, int64_t offset) {
  GUARD({
    if (!c || !handle64) return PA_EINVAL;
    return comm_flags_import(c->p, rank, handle64, offset);
  })
}

void pa_comm_destroy(pa_comm* c) {
  if (!c) return;
  comm_destroy(c->p);
  delete c;
}

// ---- PeerPut windows ---------------------------------------------------------------
pa_status pa_ipc_export(const void* devptr, void* handle64, int64_t* offset) {
  if (!devptr || !handle64 || !offset) return PA_EINVAL;
  return ipc_export(devptr, handle64, offset);
}

pa_status pa_ipc_import(const void* handle64, int64_t offset, void** mapped) {
  GUARD({
    if (!handle64 || !mapped) return PA_EINVAL;
    return ipc_import(handle64, offset, mapped);
  })
}

pa_status pa_ipc_release(const void* handle64) {
  GUARD({
    if (!handle64) return PA_EINVAL;
    return ipc_release_handle(handle64);
  })
}

pa_status pa_plan_set_window(pa_plan* plan, const void* local_dst, int n, void* peer_dst) {
  GUARD({
    // local_dst may be NULL: a rank that owns nothing of `dest` still puts into its peers
    if (!plan) return PA_EINVAL;
    return plan_set_window(plan->p, local_dst, n - 1, peer_dst);
  })
}

pa_status pa_plan_set_recv_window(pa_plan* plan, int n, void* peer_recv_buf) {
  GUARD({
    if (!plan) return PA_EINVAL;
    return plan_set_recv_window(plan->p, n - 1, peer_recv_buf);
  })
}

// pa_plan_*check*: plan_check's answer for the fused kernel of `mode` on `side`
static pa_status plan_verdict(const char* who, const pa_plan* plan, Side side, FusedMode mode, bool f32) {
  GUARD({
    if (!plan) {
      set_error("%s: null plan", who);
      return PA_EINVAL;
    }
    return plan_check(plan->p, side, mode, f32);
  })
}

pa_status pa_plan_fft_check(const pa_plan* plan) {
  return plan_verdict("pa_plan_fft_check", plan, Side::unpack, FusedMode::fft, false);
}

pa_status pa_plan_fft_check_ex(const pa_plan* plan, unsigned flags) {
  return plan_verdict("pa_plan_fft_check_ex", plan, Side::unpack, FusedMode::fft, (flags & PA_FFT_F32) != 0);
}

pa_status pa_wait(pa_plan* plan, void* stream) {
  if (!plan) return PA_EINVAL;
  return wait_sends(plan->p, stream);
}

pa_status pa_transpose_host(pa_plan* plan, pa_comm* comm, const void* host_src, void* host_dst,
                            unsigned flags) {
  GUARD({
    if (!plan) return PA_EINVAL;
    return transpose_host(plan->p, comm ? comm->p : nullptr, host_src, host_dst, flags);
  })
}

// ---- line transforms along the first memory dimension (pa_rfft, pa_r2r) ---------------
// The checks they share; `who` prefixes the messages.
// The transform axis is perm[1], the logical dim of the first memory dim; it must be local.
static pa_status line_axis(const char* who, const Pencil& R, int* ax_out) {
  const int ax = R.perm[0];
  for (int i = 0; i < R.topo->M; ++i)
    if (R.decomp[i] == ax) {
      set_error("%s: the transform axis (logical dim %d) is decomposed", who, ax + 1);
      return PA_EINCOMPAT;
    }
  *ax_out = ax;
  return PA_OK;
}

// lines of the local array: its extents off the axis times the extra dims
static pa_status line_count(const char* who, const Pencil& R, int ax, int n_extra,
                            const int64_t* extra_dims, i64* nlines_out) {
  if (n_extra < 0 || (n_extra > 0 && !extra_dims) || R.N + n_extra > PA_MAX_DIMS) {
    set_error("%s: %d extra dims on a %d-d pencil (at most %d dims in all)", who, n_extra, R.N,
              PA_MAX_DIMS);
    return PA_EINVAL;
  }
  i64 lo[PA_MAX_DIMS], hi[PA_MAX_DIMS];
  R.range_local(lo, hi);
  i64 nlines = 1;
  for (int d = 0; d < R.N; ++d)
    if (d != ax) nlines *= hi[d] - lo[d];
  for (int i = 0; i < n_extra; ++i) {
    if (extra_dims[i] < 0) {
      set_error("%s: negative extra dim", who);
      return PA_EINVAL;
    }
    nlines *= extra_dims[i];
  }
  *nlines_out = nlines;
  return PA_OK;
}

// src / dst of a non-empty local array: not NULL, not overlapping (in_place: src == dst is
// allowed, any other overlap is not), 16-byte aligned
static pa_status line_pointers(const char* who, const void* src, i64 src_bytes, const void* dst,
                               i64 dst_bytes, bool in_place) {
  if (!src || !dst) {
    set_error("%s: null array pointer for a non-empty local array", who);
    return PA_EINVAL;
  }
  const uintptr_t s = (uintptr_t)src, d = (uintptr_t)dst;
  if (!(in_place && s == d) && s < d + (uintptr_t)dst_bytes && d < s + (uintptr_t)src_bytes) {
    set_error("%s: src and dst overlap", who);
    return PA_EINVAL;
  }
  if ((s | d) & 15) {
    set_error("%s: src and dst must be 16-byte aligned", who);
    return PA_EINVAL;
  }
  return PA_OK;
}

// ---- real-to-complex line transforms ------------------------------------------------
// Every check runs on the host before any device call.  `who` prefixes the messages; with
// check_ptrs false the caller checks src / dst itself (pa_transpose_brfft: src is not on `cplx`).
static pa_status rfft_checks(const char* who, const pa_pencil* real, const pa_pencil* cplx,
                             int n_extra, const int64_t* extra_dims, unsigned flags,
                             const void* src, const void* dst, bool check_ptrs, int* N_out,
                             i64* nlines_out) {
  if (!real || !cplx) {
    set_error("%s: null pencil", who);
    return PA_EINVAL;
  }
  const Pencil& R = *real->p;
  const Pencil& Cp = *cplx->p;
  if (R.topo != Cp.topo || R.N != Cp.N) {
    set_error("%s: the pencils must share their topology and number of dimensions", who);
    return PA_EINCOMPAT;
  }
  const int M = R.topo->M;
  for (int i = 0; i < M; ++i)
    if (R.decomp[i] != Cp.decomp[i]) {
      set_error("%s: the pencils have different decompositions", who);
      return PA_EINCOMPAT;
    }
  for (int d = 0; d < R.N; ++d)
    if (R.perm[d] != Cp.perm[d]) {
      set_error("%s: the pencils have different permutations", who);
      return PA_EINCOMPAT;
    }
  int ax = 0;  // logical dim of the first memory dim: the transform axis
  pa_status s = line_axis(who, R, &ax);
  if (s != PA_OK) return s;
  for (int d = 0; d < R.N; ++d)
    if (d != ax && R.size_global[d] != Cp.size_global[d]) {
      set_error("%s: global sizes differ along dim %d", who, d + 1);
      return PA_EINCOMPAT;
    }
  const i64 N = R.size_global[ax];
  if (Cp.size_global[ax] != N / 2 + 1) {
    set_error("%s: the complex pencil has %lld points along the transform axis, expected "
              "N/2+1 = %lld", who, (long long)Cp.size_global[ax], (long long)(N / 2 + 1));
    return PA_EINCOMPAT;
  }
  const unsigned dir = flags & ~PA_FFT_F32;
  if (dir != PA_FFT_FORWARD && dir != PA_FFT_BACKWARD) {
    set_error("%s: flags must be exactly PA_FFT_FORWARD or PA_FFT_BACKWARD, optionally "
              "with PA_FFT_F32", who);
    return PA_EINVAL;
  }
  if (N < 16 || N > 2048 || (N & (N - 1))) {
    set_error("%s: N = %lld is not a power of two in 16..2048", who, (long long)N);
    return PA_EINVAL;
  }
  i64 nlines = 0;
  s = line_count(who, R, ax, n_extra, extra_dims, &nlines);
  if (s != PA_OK) return s;
  const bool fwd = dir == PA_FFT_FORWARD;
  const i64 rs = (flags & PA_FFT_F32) ? 4 : 8;  // bytes of a real element; a complex one is 2 rs
  const i64 real_bytes = nlines * N * rs, cplx_bytes = nlines * (N / 2 + 1) * 2 * rs;
  const i64 src_bytes = fwd ? real_bytes : cplx_bytes, dst_bytes = fwd ? cplx_bytes : real_bytes;
  if (check_ptrs && nlines > 0) {
    s = line_pointers(who, src, src_bytes, dst, dst_bytes, false);
    if (s != PA_OK) return s;
  }
  *N_out = (int)N;
  *nlines_out = nlines;
  return PA_OK;
}

pa_status pa_rfft(const pa_pencil* real, const pa_pencil* cplx, int n_extra,
                  const int64_t* extra_dims, unsigned flags, const void* src, void* dst,
                  void* stream) {
  GUARD({
    int N = 0;
    i64 nlines = 0;
    pa_status s =
        rfft_checks("pa_rfft", real, cplx, n_extra, extra_dims, flags, src, dst, true, &N, &nlines);
    if (s != PA_OK) return s;
    s = need_gpu();
    if (s != PA_OK) return s;
    return rfft_lines(N, (flags & ~PA_FFT_F32) == PA_FFT_FORWARD, (flags & PA_FFT_F32) != 0, nlines,
                      src, dst, stream);
  })
}

// ---- real-to-real line transforms (DCT-II/III, DST-II/III) ----------------------------
// kind: FFTW's REDFT10 (DCT-II), REDFT01 (DCT-III), RODFT10 (DST-II) or RODFT01 (DST-III)
static pa_status r2r_kind_check(const char* who, int kind) {
  if (kind != PA_REDFT10 && kind != PA_REDFT01 && kind != PA_RODFT10 && kind != PA_RODFT01) {
    set_error("%s: kind %d is not PA_REDFT10, PA_REDFT01, PA_RODFT10 or PA_RODFT01", who, kind);
    return PA_EINVAL;
  }
  return PA_OK;
}

// The checks in pa_rfft's order, all on the host before any device call.
static pa_status r2r(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims, int kind,
                     unsigned flags, const void* src, void* dst, void* stream) {
  const char* who = "pa_r2r";
  if (!pencil) {
    set_error("%s: null pencil", who);
    return PA_EINVAL;
  }
  const Pencil& R = *pencil->p;
  int ax = 0;
  pa_status s = line_axis(who, R, &ax);
  if (s != PA_OK) return s;
  s = r2r_kind_check(who, kind);
  if (s != PA_OK) return s;
  if (flags & ~PA_FFT_F32) {
    set_error("%s: flags must be 0 or PA_FFT_F32", who);
    return PA_EINVAL;
  }
  const i64 N = R.size_global[ax];
  if (N < 16 || N > 2048 || (N & (N - 1))) {
    set_error("%s: N = %lld is not a power of two in 16..2048", who, (long long)N);
    return PA_EINVAL;
  }
  i64 nlines = 0;
  s = line_count(who, R, ax, n_extra, extra_dims, &nlines);
  if (s != PA_OK) return s;
  const bool f32 = (flags & PA_FFT_F32) != 0;
  const i64 bytes = nlines * N * (f32 ? 4 : 8);
  if (nlines > 0) {
    s = line_pointers(who, src, bytes, dst, bytes, true);
    if (s != PA_OK) return s;
  }
  s = need_gpu();
  if (s != PA_OK) return s;
  return r2r_lines((int)N, r2r_forward(kind), r2r_sine(kind), f32, nlines, src, dst, stream);
}

pa_status pa_r2r(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims, int kind,
                 unsigned flags, const void* src, void* dst, void* stream) {
  GUARD({ return r2r(pencil, n_extra, extra_dims, kind, flags, src, dst, stream); })
}

// ---- fused transpose + line transform -----------------------------------------------------
// Every entry point of a fused line transform is one (side, mode); `all`: the launch without the
// window protocol (pa_get_all_fft, pa_put_all_*).
static const char* line_op_name(Side side, FusedMode mode, bool all) {
  switch (mode) {
    case FusedMode::fft:
      if (side == Side::unpack) return all ? "pa_get_all_fft" : "pa_transpose";
      return all ? "pa_put_all_fft" : "pa_fft_put";
    case FusedMode::rfft:
      if (side == Side::unpack) return "pa_transpose_rfft";
      return all ? "pa_put_all_rfft" : "pa_rfft_put";
    case FusedMode::r2r:
      if (side == Side::unpack) return "pa_transpose_r2r";
      return all ? "pa_put_all_r2r" : "pa_r2r_put";
    case FusedMode::brfft: break;
  }
  if (side == Side::unpack) return "pa_transpose_brfft";
  return all ? "pa_put_all_brfft" : "pa_brfft_put";
}

// The LineOp an entry point's flags (and r2r's kind) ask for, or its refusal.  The flags besides
// PA_FFT_F32:
// - pa_transpose: PA_FFT_FORWARD or PA_FFT_BACKWARD (both: forward), PA_FFT_F32 only with one;
// - pa_transpose_brfft / _r2r / _rfft: the direction is implied; any of PA_WAITALL,
//   PA_NO_OVERLAP and PA_STAGE_SELF;
// - pa_get_all_fft and the send side: never PA_STAGE_SELF; fft exactly one direction, the other
//   modes none; PA_WAITALL except for the launches without the window protocol.
static pa_status line_op(Side side, FusedMode mode, bool all, unsigned flags, int kind, LineOp* op) {
  const char* who = line_op_name(side, mode, all);
  const bool fft = mode == FusedMode::fft;
  if (side == Side::put && (flags & PA_STAGE_SELF)) {
    set_error("%s: PA_STAGE_SELF does not apply: the send-side fusion stores the self block "
              "straight into dst", who);
    return PA_EINVAL;
  }
  if (side == Side::put || all) {
    const unsigned dir = flags & ~(all ? PA_FFT_F32 : PA_FFT_F32 | PA_WAITALL);
    if (fft ? (dir != PA_FFT_FORWARD && dir != PA_FFT_BACKWARD) : dir != 0) {
      if (fft)
        set_error("%s: flags must be exactly PA_FFT_FORWARD or PA_FFT_BACKWARD, optionally with %s", who,
                  all ? "PA_FFT_F32" : "PA_FFT_F32 and PA_WAITALL");
      else
        set_error("%s: flags may combine %s only (the direction is implied)", who,
                  all ? "PA_FFT_F32" : "PA_WAITALL and PA_FFT_F32");
      return PA_EINVAL;
    }
  } else if (!fft) {
    if (flags & ~(PA_WAITALL | PA_NO_OVERLAP | PA_STAGE_SELF | PA_FFT_F32)) {
      set_error("%s: flags may combine PA_WAITALL, PA_NO_OVERLAP, PA_STAGE_SELF and PA_FFT_F32 only "
                "(the direction is implied)", who);
      return PA_EINVAL;
    }
  } else if ((flags & PA_FFT_F32) && !(flags & (PA_FFT_FORWARD | PA_FFT_BACKWARD))) {
    set_error("pa_transpose: PA_FFT_F32 without PA_FFT_FORWARD / PA_FFT_BACKWARD");
    return PA_EINVAL;
  }
  const bool r2r = mode == FusedMode::r2r;
  if (r2r) RC(r2r_kind_check(who, kind));
  *op = LineOp{side, mode, !fft ? 0 : (flags & PA_FFT_FORWARD) ? -1 : 1, r2r ? kind : 0,
               (flags & PA_FFT_F32) != 0};
  return PA_OK;
}

// The plan's elements: reals (Float64; Float32 with PA_FFT_F32) or complex ones
static pa_status plan_elsize(const char* who, const Plan& P, bool real, bool f32) {
  if (P.elsize == (real ? 4 : 8) * (f32 ? 1 : 2)) return PA_OK;
  const char* t32 = real ? "Float32" : "ComplexF32";
  if (f32)
    set_error("%s: PA_FFT_F32 takes a %s (elsize %d) plan", who, t32, real ? 4 : 8);
  else
    set_error("%s: a %s (elsize %d) plan, or PA_FFT_F32 for %s", who, real ? "Float64" : "ComplexF64",
              real ? 8 : 16, t32);
  return PA_EINVAL;
}

// The per-rank table of a launch over every block of the grid line without the window protocol:
// this rank's self block with `local` (get: src, put: dst), peer n's get / put block with peers[n],
// its array as mapped here.  A non-empty block needs an array aligned to the plan's element.
static pa_status peer_table(const char* who, const Plan& P, bool get, const void* local,
                            void* const* peers, std::vector<const BlockCopy*>* blocks,
                            std::vector<void*>* arrays) {
  for (int n = 0; n < P.nproc; ++n) {
    const bool self = n == P.self_index;
    const BlockCopy& b = self ? P.self_fused : get ? P.peers[n].get : P.peers[n].put;
    void* p = self ? (void*)local : (peers ? peers[n] : nullptr);
    if (b.count > 0 && !p) {
      if (self)
        set_error("%s: null %s for a non-empty self block", who, get ? "src" : "dst");
      else
        set_error("%s: null peer array for a non-empty block (peer %d)", who, n + 1);
      return PA_EINVAL;
    }
    if (b.count > 0 && ((uintptr_t)p % P.elsize)) {
      set_error("%s: arrays must be aligned to the %lld-byte element", who, (long long)P.elsize);
      return PA_EINVAL;
    }
    blocks->push_back(&b);
    arrays->push_back(p);
  }
  return PA_OK;
}

// pa_transpose and the receive-side fused transforms (pa_transpose_brfft, _r2r, _rfft).  Every
// check runs on the host before any device call.  `pen`: brfft the real pencil of dst, rfft the
// complex one, against the plan's output pencil as pa_rfft relates them; r2r: `kind`.
static pa_status transpose_unpack(pa_plan* plan, pa_comm* comm, const pa_pencil* pen, int kind,
                                  const void* src, void* dst, unsigned flags, void* stream,
                                  FusedMode mode) {
  const char* who = line_op_name(Side::unpack, mode, false);
  if (!plan) {
    set_error("%s: null plan", who);
    return PA_EINVAL;
  }
  Plan& P = *plan->p;
  Comm* c = comm ? comm->p : nullptr;
  LineOp op;
  if (mode == FusedMode::fft) {
    // a rank may own nothing (more processes than points, Pencils.jl:193-218): its empty arrays
    // have no storage, yet it takes part in the exchange
    if ((!src && P.length_in > 0) || (!dst && P.length_out > 0)) {
      set_error("pa_transpose: null array pointer");
      return PA_EINVAL;
    }
    bool fused = false;
    RC(transpose_fft_op(&P, flags, src, dst, &op, &fused));
    return transpose(&P, c, src, dst, flags, stream, fused ? &op : nullptr);
  }
  RC(line_op(Side::unpack, mode, false, flags, kind, &op));
  RC(plan_elsize(who, P, unpack_moves_reals(mode), op.f32));
  const i64 es = P.elsize;
  i64 dst_bytes = P.length_out * es;
  if (mode == FusedMode::r2r) {
    int ax = 0;  // the transform axis, the output pencil's first memory dim, must be whole (as pa_r2r)
    RC(line_axis(who, *P.pout, &ax));
  } else {
    // dst on `pen`, the other side of the transform from the plan's output pencil
    const bool rfft = mode == FusedMode::rfft;
    const pa_pencil out{P.pout};
    int N = 0;
    i64 nlines = 0;
    RC(rfft_checks(who, rfft ? &out : pen, rfft ? pen : &out, P.n_extra, P.extra,
                   (rfft ? PA_FFT_FORWARD : PA_FFT_BACKWARD) | (op.f32 ? PA_FFT_F32 : 0u), nullptr,
                   nullptr, false, &N, &nlines));
    const i64 rs = op.f32 ? 4 : 8;  // bytes of a real
    dst_bytes = rfft ? nlines * (N / 2 + 1) * 2 * rs : nlines * N * rs;
  }
  RC(fused_pointers(who, src, P.length_in * es, dst, dst_bytes));
  // the same verdict on every rank of the grid line: a refusal launches nothing anywhere
  RC(plan_check(&P, Side::unpack, mode, op.f32));
  RC(need_gpu());
  return transpose(&P, c, src, dst, flags, stream, &op);
}

pa_status pa_transpose(pa_plan* plan, pa_comm* comm, const void* src, void* dst, unsigned flags,
                       void* stream) {
  GUARD({ return transpose_unpack(plan, comm, nullptr, 0, src, dst, flags, stream, FusedMode::fft); })
}

pa_status pa_transpose_brfft(pa_plan* plan, pa_comm* comm, const pa_pencil* real, const void* src,
                             void* dst, unsigned flags, void* stream) {
  GUARD({ return transpose_unpack(plan, comm, real, 0, src, dst, flags, stream, FusedMode::brfft); })
}

pa_status pa_transpose_r2r(pa_plan* plan, pa_comm* comm, int kind, const void* src, void* dst,
                           unsigned flags, void* stream) {
  GUARD({ return transpose_unpack(plan, comm, nullptr, kind, src, dst, flags, stream, FusedMode::r2r); })
}

pa_status pa_transpose_rfft(pa_plan* plan, pa_comm* comm, const pa_pencil* cplx, const void* src,
                            void* dst, unsigned flags, void* stream) {
  GUARD({ return transpose_unpack(plan, comm, cplx, 0, src, dst, flags, stream, FusedMode::rfft); })
}

pa_status pa_plan_brfft_check(const pa_plan* plan, unsigned flags) {
  return plan_verdict("pa_plan_brfft_check", plan, Side::unpack, FusedMode::brfft, (flags & PA_FFT_F32) != 0);
}

pa_status pa_plan_real_check(const pa_plan* plan, unsigned flags) {
  return plan_verdict("pa_plan_real_check", plan, Side::unpack, FusedMode::r2r, (flags & PA_FFT_F32) != 0);
}

// The one-sided fused gather + FFT without the window protocol.  Every check runs on the host
// before any device call.
static pa_status get_all_fft(pa_plan* plan, const void* src, void* const* peers, void* dst,
                             unsigned flags, void* stream) {
  const char* who = "pa_get_all_fft";
  if (!plan) {
    set_error("%s: null plan", who);
    return PA_EINVAL;
  }
  Plan& P = *plan->p;
  if (P.dim < 0) {
    set_error("%s: plan has no exchange", who);
    return PA_EINVAL;
  }
  LineOp op;
  RC(line_op(Side::unpack, FusedMode::fft, true, flags, 0, &op));
  // the verdict pa_transpose asks (for a PeerGet plan it covers this gather)
  RC(plan_check(&P, Side::unpack, FusedMode::fft, op.f32));
  std::vector<const BlockCopy*> blocks;
  std::vector<void*> srcs;
  RC(peer_table(who, P, true, src, peers, &blocks, &srcs));
  RC(fused_pointers(who, src, P.length_in * P.elsize, dst, P.length_out * P.elsize));
  RC(need_gpu());
  bool launched = false;
  return get_fft(P.nproc, blocks.data(), srcs.data(), dst, op, nullptr, stream, &launched);
}

pa_status pa_get_all_fft(pa_plan* plan, const void* src, void* const* peers, void* dst, unsigned flags,
                         void* stream) {
  GUARD({ return get_all_fft(plan, src, peers, dst, flags, stream); })
}

// ---- send-side fused transform + put (pa_fft_put, pa_rfft_put, pa_r2r_put, pa_brfft_put and
//      their pa_put_all_*) ------------------------------------------------------------------------
// The checks they share, all on the host: the plan's verdict, then (rfft, brfft) `pen` against the
// plan's INPUT pencil as pa_rfft relates them (rfft: `pen` is the real pencil of src; brfft: the
// complex one), then src / dst (NULL only when empty, not overlapping, aligned: fft / rfft to the
// complex element; r2r / brfft src to a pair of reals or a complex element, dst to the real).
static pa_status put_args(const char* who, Plan& P, const pa_pencil* pen, const void* src,
                          const void* dst, const LineOp& op) {
  const FusedMode mode = op.mode;
  const bool rfft = mode == FusedMode::rfft, real = put_moves_reals(mode);
  RC(plan_check(&P, Side::put, mode, op.f32));
  const i64 es = P.elsize;
  i64 src_bytes = P.length_in * es;
  if (rfft || mode == FusedMode::brfft) {
    const pa_pencil in{P.pin};
    int N = 0;
    i64 nlines = 0;
    RC(rfft_checks(who, rfft ? pen : &in, rfft ? &in : pen, P.n_extra, P.extra,
                   PA_FFT_FORWARD | (op.f32 ? PA_FFT_F32 : 0u), nullptr, nullptr, false, &N, &nlines));
    src_bytes = rfft ? nlines * N * (es / 2) : nlines * (N / 2 + 1) * 2 * es;
  }
  const i64 dst_bytes = P.length_out * es;
  if ((!src && src_bytes > 0) || (!dst && dst_bytes > 0)) {
    set_error("%s: null array pointer for a non-empty local array", who);
    return PA_EINVAL;
  }
  const uintptr_t a = (uintptr_t)src, b = (uintptr_t)dst;
  if (src_bytes > 0 && dst_bytes > 0 && a < b + (uintptr_t)dst_bytes && b < a + (uintptr_t)src_bytes) {
    set_error("%s: src and dst overlap (the send-side fusion has no staged schedule: transform in "
              "place with %s, then transpose)", who,
              mode == FusedMode::fft ? "fft_" : rfft ? "rfft_" : mode == FusedMode::r2r ? "r2r_" : "brfft_");
    return PA_EINVAL;
  }
  if (real) {
    // (the load reads pairs of reals / complex elements; every real is stored alone)
    if ((src_bytes > 0 && a % (2 * es)) || (dst_bytes > 0 && b % es)) {
      set_error("%s: src must be aligned to %lld bytes and dst to the %lld-byte real", who,
                (long long)(2 * es), (long long)es);
      return PA_EINVAL;
    }
    return PA_OK;
  }
  if ((src_bytes > 0 && a % es) || (dst_bytes > 0 && b % es)) {
    set_error("%s: src and dst must be aligned to the %lld-byte complex element", who, (long long)es);
    return PA_EINVAL;
  }
  return PA_OK;
}

// all = false: dst = transpose(T(src)) through transpose(), PeerPut's one-sided schedule for a plan
// with an exchange.  all = true: the fused kernel without the window protocol, the self block into
// `dst`, the put block of peer n into peers[n - 1] (its dst, as mapped here; the self entry is
// ignored).
static pa_status put_fused(pa_plan* plan, pa_comm* comm, const pa_pencil* pen, int kind, const void* src,
                           void* const* peers, void* dst, unsigned flags, void* stream, FusedMode mode,
                           bool all) {
  const char* who = line_op_name(Side::put, mode, all);
  if (!plan) {
    set_error("%s: null plan", who);
    return PA_EINVAL;
  }
  Plan& P = *plan->p;
  if (all && P.dim < 0) {
    set_error("%s: plan has no exchange", who);
    return PA_EINVAL;
  }
  LineOp op;
  RC(line_op(Side::put, mode, all, flags, kind, &op));
  RC(put_args(who, P, pen, src, dst, op));
  if (!all) {
    RC(need_gpu());
    return transpose(&P, comm ? comm->p : nullptr, src, dst, flags, stream, &op);
  }
  std::vector<const BlockCopy*> blocks;
  std::vector<void*> dsts;
  RC(peer_table(who, P, false, dst, peers, &blocks, &dsts));
  RC(need_gpu());
  bool launched = false;
  return put_fft(P.nproc, blocks.data(), src, dsts.data(), op, nullptr, stream, &launched);
}

pa_status pa_fft_put(pa_plan* plan, pa_comm* comm, const void* src, void* dst, unsigned flags,
                     void* stream) {
  GUARD({ return put_fused(plan, comm, nullptr, 0, src, nullptr, dst, flags, stream, FusedMode::fft, false); })
}

pa_status pa_rfft_put(pa_plan* plan, pa_comm* comm, const pa_pencil* real, const void* src, void* dst,
                      unsigned flags, void* stream) {
  GUARD({ return put_fused(plan, comm, real, 0, src, nullptr, dst, flags, stream, FusedMode::rfft, false); })
}

pa_status pa_r2r_put(pa_plan* plan, pa_comm* comm, int kind, const void* src, void* dst, unsigned flags,
                     void* stream) {
  GUARD({ return put_fused(plan, comm, nullptr, kind, src, nullptr, dst, flags, stream, FusedMode::r2r, false); })
}

pa_status pa_brfft_put(pa_plan* plan, pa_comm* comm, const pa_pencil* cplx, const void* src, void* dst,
                       unsigned flags, void* stream) {
  GUARD({ return put_fused(plan, comm, cplx, 0, src, nullptr, dst, flags, stream, FusedMode::brfft, false); })
}

pa_status pa_put_all_fft(pa_plan* plan, const void* src, void* const* peers, void* dst, unsigned flags,
                         void* stream) {
  GUARD({ return put_fused(plan, nullptr, nullptr, 0, src, peers, dst, flags, stream, FusedMode::fft, true); })
}

pa_status pa_put_all_rfft(pa_plan* plan, const pa_pencil* real, const void* src, void* const* peers,
                          void* dst, unsigned flags, void* stream) {
  GUARD({ return put_fused(plan, nullptr, real, 0, src, peers, dst, flags, stream, FusedMode::rfft, true); })
}

pa_status pa_put_all_r2r(pa_plan* plan, int kind, const void* src, void* const* peers, void* dst,
                         unsigned flags, void* stream) {
  GUARD({ return put_fused(plan, nullptr, nullptr, kind, src, peers, dst, flags, stream, FusedMode::r2r, true); })
}

pa_status pa_put_all_brfft(pa_plan* plan, const pa_pencil* cplx, const void* src, void* const* peers,
                           void* dst, unsigned flags, void* stream) {
  GUARD({ return put_fused(plan, nullptr, cplx, 0, src, peers, dst, flags, stream, FusedMode::brfft, true); })
}

pa_status pa_plan_real_put_check(const pa_plan* plan, unsigned flags) {
  return plan_verdict("pa_plan_real_put_check", plan, Side::put, FusedMode::r2r, (flags & PA_FFT_F32) != 0);
}

pa_status pa_plan_fft_put_check(const pa_plan* plan, unsigned flags) {
  return plan_verdict("pa_plan_fft_put_check", plan, Side::put, FusedMode::fft, (flags & PA_FFT_F32) != 0);
}

pa_status pa_plan_rfft_put_check(const pa_plan* plan, unsigned flags) {
  return plan_verdict("pa_plan_rfft_put_check", plan, Side::put, FusedMode::rfft, (flags & PA_FFT_F32) != 0);
}

pa_status pa_host_chain_create(int n, pa_plan* const* plans, pa_comm* comm, pa_host_chain** out) {
  GUARD({
    if (n < 1 || n > 64 || !plans || !out) {
      set_error("pa_host_chain_create: 1..64 plans");
      return PA_EINVAL;
    }
    Plan* ps[64];
    for (int i = 0; i < n; ++i) {
      if (!plans[i]) return PA_EINVAL;
      ps[i] = plans[i]->p;
    }
    HostChain* c = nullptr;
    pa_status s = host_chain_create(n, ps, comm ? comm->p : nullptr, &c);
    if (s != PA_OK) return s;
    *out = new pa_host_chain{c};
    return PA_OK;
  })
}

void pa_host_chain_destroy(pa_host_chain* c) {
  if (!c) return;
  host_chain_destroy(c->p);
  delete c;
}

pa_status pa_host_chain_submit(pa_host_chain* c, const void* host_src, void* host_dst,
                               int64_t* ticket) {
  GUARD({
    if (!c) return PA_EINVAL;
    return host_chain_submit(c->p, host_src, host_dst, ticket);
  })
}

pa_status pa_host_chain_wait(pa_host_chain* c, int64_t ticket) {
  if (!c) return PA_EINVAL;
  return host_chain_wait(c->p, ticket);
}

pa_status pa_host_chain_time_begin(pa_host_chain* c) {
  if (!c) return PA_EINVAL;
  return host_chain_time_begin(c->p);
}

pa_status pa_host_chain_time_end(pa_host_chain* c, float* ms) {
  if (!c || !ms) return PA_EINVAL;
  return host_chain_time_end(c->p, ms);
}

pa_status pa_host_chain_buffer(pa_host_chain* c, int slot, int which, void** devptr,
                               int64_t* bytes) {
  if (!c) return PA_EINVAL;
  return host_chain_buffer(c->p, slot, which, devptr, bytes);
}

// ---- PencilIO binary layout --------------------------------------------------------
pa_status pa_io_sizes(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                      int chunks, int64_t* global_bytes, int64_t* local_bytes, int64_t* nruns,
                      int64_t* run_bytes, int64_t* first_offset) {
  GUARD({
    if (!p || (n_extra > 0 && !extra_dims)) return PA_EINVAL;
    return io_sizes(*p->p, n_extra, extra_dims, elsize, chunks, global_bytes, local_bytes, nruns,
                    run_bytes, first_offset);
  })
}

pa_status pa_io_run_offset(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                           int chunks, int64_t run, int64_t* file_offset) {
  GUARD({
    if (!p || !file_offset || (n_extra > 0 && !extra_dims)) return PA_EINVAL;
    return io_run_offset(*p->p, n_extra, extra_dims, elsize, chunks, run, file_offset);
  })
}

pa_status pa_io_write(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                      int chunks, const void* dev_array, const char* path, int64_t offset) {
  GUARD({
    if (!p || !path || offset < 0 || (n_extra > 0 && !extra_dims)) return PA_EINVAL;
    return io_transfer(*p->p, n_extra, extra_dims, elsize, chunks, (void*)dev_array, path, offset, true);
  })
}

pa_status pa_io_read(const pa_pencil* p, int n_extra, const int64_t* extra_dims, int elsize,
                     int chunks, void* dev_array, const char* path, int64_t offset) {
  GUARD({
    if (!p || !path || offset < 0 || (n_extra > 0 && !extra_dims)) return PA_EINVAL;
    return io_transfer(*p->p, n_extra, extra_dims, elsize, chunks, dev_array, path, offset, false);
  })
}

// ---- distributed reductions -----------------------------------------------------------------
pa_status pa_reduce_result_type(int dtype, int map, int op, int* result_dtype) {
  const char* why = "";
  const int r = red::result_dtype(dtype, map, op, &why);
  if (r < 0) {
    set_error("pa_reduce: dtype %d, map %d, op %d: %s", dtype, map, op, why);
    return PA_EINVAL;
  }
  if (result_dtype) *result_dtype = r;
  return PA_OK;
}

static int elem_bytes(int dtype) {  // element size of a pa_dtype
  static const int sz[] = {8, 4, 16, 8, 4, 8, 1};
  return dtype >= 0 && dtype <= PA_BOOL ? sz[dtype] : 0;
}
static int component_bytes(int dtype) {  // the alignment an array of dtype needs
  return dtype == PA_COMPLEXF64 ? 8 : dtype == PA_COMPLEXF32 ? 4 : elem_bytes(dtype);
}

// Every check in the order of pa_b200.h, on the host before any device call.
static pa_status reduce_checks(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims,
                               pa_comm* comm, int dtype, int map, int op, const void* pred_value,
                               const void* a, const void* b, void* result, i64* n_local) {
  const char* who = "pa_reduce";
  if (!pencil) {
    set_error("%s: null pencil", who);
    return PA_EINVAL;
  }
  int rt = 0;
  pa_status s = pa_reduce_result_type(dtype, map, op, &rt);
  if (s != PA_OK) return s;
  const Pencil& Pn = *pencil->p;
  if (n_extra < 0 || (n_extra > 0 && !extra_dims) || Pn.N + n_extra > PA_MAX_DIMS) {
    set_error("%s: %d extra dims on a %d-d pencil (at most %d dims in all)", who, n_extra, Pn.N,
              PA_MAX_DIMS);
    return PA_EINVAL;
  }
  i64 lo[PA_MAX_DIMS], hi[PA_MAX_DIMS];
  Pn.range_local(lo, hi);
  i64 n = 1, nglobal = 1;
  for (int d = 0; d < Pn.N; ++d) {
    n *= hi[d] - lo[d];
    nglobal *= Pn.size_global[d];
  }
  for (int i = 0; i < n_extra; ++i) {
    if (extra_dims[i] < 0) {
      set_error("%s: negative extra dim", who);
      return PA_EINVAL;
    }
    n *= extra_dims[i];
    nglobal *= extra_dims[i];
  }
  if (map == PA_MAP_DOT ? (n > 0 && !b) : b != nullptr) {
    set_error(map == PA_MAP_DOT ? "%s: PA_MAP_DOT reduces two arrays: `b` is missing"
                                : "%s: a second array `b` goes with PA_MAP_DOT only", who);
    return PA_EINVAL;
  }
  const uintptr_t al = (uintptr_t)component_bytes(dtype);
  if (n > 0 && (!a || (map == PA_MAP_DOT && !b))) {
    set_error("%s: null array pointer for a non-empty local array", who);
    return PA_EINVAL;
  }
  if (((uintptr_t)a | (uintptr_t)b) % al) {
    set_error("%s: arrays must be aligned to %d bytes (their real component)", who, (int)al);
    return PA_EINVAL;
  }
  // (the kernels store the result whole: 16-byte stores for ComplexF64, 8-byte for ComplexF32)
  const uintptr_t ral = (uintptr_t)elem_bytes(rt);
  if (!result || (uintptr_t)result % ral) {
    set_error("%s: `result` must be a device pointer aligned to %d bytes", who, (int)ral);
    return PA_EINVAL;
  }
  const int p = op >> 4;
  if (p >= (PA_PRED_EQ >> 4) && p <= (PA_PRED_GE >> 4) && !pred_value) {
    set_error("%s: the comparison needs pred_value", who);
    return PA_EINVAL;
  }
  const int base = op & 15;
  if (nglobal == 0 && (base == PA_OP_MAX || base == PA_OP_MIN)) {
    set_error("%s: reducing over an empty collection is not allowed (maximum / minimum of an "
              "empty array)", who);
    return PA_EINVAL;
  }
  const int nranks = Pn.topo->size;
  if (comm ? comm_size(comm->p) != nranks : nranks > 1) {
    set_error(comm ? "%s: the topology has %d ranks, the communicator %d"
                   : "%s: a topology of %d ranks needs a communicator", who, nranks,
              comm ? comm_size(comm->p) : 0);
    return PA_EINCOMPAT;
  }
  *n_local = n;
  return PA_OK;
}

pa_status pa_reduce(const pa_pencil* pencil, int n_extra, const int64_t* extra_dims, pa_comm* comm,
                    int dtype, int map, int op, const void* pred_value, const void* a,
                    const void* b, void* result, void* stream) {
  GUARD({
    i64 n = 0;
    pa_status s = reduce_checks(pencil, n_extra, extra_dims, comm, dtype, map, op, pred_value, a, b,
                                result, &n);
    if (s != PA_OK) return s;
    s = need_gpu();
    if (s != PA_OK) return s;
    return reduce(comm ? comm->p : nullptr, dtype, map, op, pred_value, n, a, b, result, stream);
  })
}

pa_status pa_plan_timings(pa_plan* plan, pa_timings* t) {
  if (!plan || !t) return PA_EINVAL;
  return plan_timings(plan->p, t);
}

pa_status pa_plan_enable_timing(pa_plan* plan, int on) {
  if (!plan) return PA_EINVAL;
  return plan_enable_timing(plan->p, on);
}

}  // extern "C"

pa_status pa::transpose_fft_op(Plan* P, unsigned flags, const void* src, const void* dst, LineOp* op,
                               bool* fused) {
  *fused = (flags & (PA_FFT_FORWARD | PA_FFT_BACKWARD | PA_FFT_F32)) != 0;
  if (!*fused) return PA_OK;
  RC(line_op(Side::unpack, FusedMode::fft, false, flags, 0, op));
  // a fused FFT this plan cannot run is refused before anything is enqueued -- and on every
  // rank of the line alike (the peers of a refusing rank must not start the exchange)
  RC(plan_check(P, Side::unpack, FusedMode::fft, op->f32));
  // src and dst may not alias -- except for the plain in-place transform along the contiguous
  // dim (same pencil on both sides, src == dst): a CTA reads its lines completely before it
  // writes them back
  const uintptr_t a = (uintptr_t)src, b = (uintptr_t)dst;
  const bool in_place = src && src == dst && P->dim < 0 && P->same_perm;
  if (!in_place && src && dst &&
      (a == b || (a < b + (uintptr_t)(P->length_out * P->elsize) &&
                  b < a + (uintptr_t)(P->length_in * P->elsize)))) {
    set_error("fused FFT: src and dst must not alias (in place only between identical pencils)");
    return PA_EINVAL;
  }
  return PA_OK;
}
