// PencilIO binary layout (SURVEY.md §8 f4): device arrays <-> the raw binary files of
// the reference's MPIIODriver (reference src/PencilIO/mpi_io.jl).
//
// Layout written by the reference and reproduced here byte for byte:
//  * discontiguous (chunks = false, the default; :372-380 `create_discontiguous_datatype`
//    with MemoryOrder): the dataset is the GLOBAL array in the pencil's MEMORY order --
//    dims (perm * size_global..., extra_dims...), column-major -- each rank owning the
//    sub-box `range_local(x, MemoryOrder())`; readable with any other decomposition;
//  * chunks = true (:382-424): the ranks' parent arrays one after the other, ordered by
//    the column-major linear index of their coordinates in the process grid
//    (`mpi_io_offset`, :412-424).
// The JSON sidecar (:194-211) is the host mirror's business (it is plain metadata).
//
// No MPI is needed on one box: every rank opens the same file and pwrite()s / pread()s
// its own runs -- what MPI-IO's "native" data representation does underneath.  The
// device array moves through a double-buffered pinned staging area: the device->host
// copy of piece k+1 overlaps the file writes of piece k.
#include <cuda_runtime.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <vector>

#include "pa_internal.hpp"

namespace pa {

namespace {

struct IoLayout {
  i64 local_bytes = 0, global_bytes = 0;
  i64 run_bytes = 0;   // contiguous run shared by file and local array
  i64 nruns = 0;
  int nd = 0;          // dims above the run
  i64 ext[PA_MAX_DIMS + 1] = {0}, fstride[PA_MAX_DIMS + 1] = {0};  // per outer dim: local extent, file byte stride
  i64 file_base = 0;   // byte offset of the rank's first element inside the dataset
};

// rank-local sub-box of the global memory-order array, cut into the longest runs that are
// contiguous on both sides
pa_status make_layout(const Pencil& P, int n_extra, const i64* extra, int elsize, bool chunks,
                      IoLayout& L) {
  if (n_extra < 0 || P.N + n_extra > PA_MAX_DIMS || elsize <= 0) {
    set_error("pa_io: bad extra dims / element size");
    return PA_EINVAL;
  }
  i64 lo[PA_MAX_DIMS], hi[PA_MAX_DIMS];
  P.range_local(lo, hi);
  const int D = P.N + n_extra;
  i64 g[PA_MAX_DIMS], l[PA_MAX_DIMS], o[PA_MAX_DIMS];
  for (int m = 0; m < P.N; ++m) {  // memory dim m holds logical dim perm[m]
    const int d = P.perm[m];
    g[m] = P.size_global[d];
    l[m] = hi[d] - lo[d];
    o[m] = lo[d];
  }
  for (int j = 0; j < n_extra; ++j) {
    g[P.N + j] = l[P.N + j] = extra[j];
    o[P.N + j] = 0;
  }
  L.local_bytes = L.global_bytes = elsize;
  for (int i = 0; i < D; ++i) {
    L.local_bytes *= l[i];
    L.global_bytes *= g[i];
  }
  if (chunks) {
    // the whole parent array is one run; its place follows the ranks that precede this
    // one in column-major order of the grid coordinates (:412-424)
    const Topology& T = *P.topo;
    i64 mine = 0, mul = 1;
    for (int i = 0; i < T.M; ++i) {
      mine += T.coords[i] * mul;
      mul *= T.dims[i];
    }
    i64 before = 0;
    for (i64 n = 0; n < mine; ++n) {
      i64 c[PA_MAX_TOPO], r = n;
      for (int i = 0; i < T.M; ++i) {
        c[i] = r % T.dims[i];
        r /= T.dims[i];
      }
      i64 rlo[PA_MAX_DIMS], rhi[PA_MAX_DIMS];
      P.range_of(c, rlo, rhi);
      i64 cnt = 1;
      for (int d = 0; d < P.N; ++d) cnt *= rhi[d] - rlo[d];
      for (int j = 0; j < n_extra; ++j) cnt *= extra[j];
      before += cnt;
    }
    L.file_base = before * elsize;
    L.run_bytes = L.local_bytes;
    L.nruns = L.local_bytes > 0 ? 1 : 0;
    L.nd = 0;
    return PA_OK;
  }
  // longest prefix of dims the rank owns completely, plus the first partial one
  int p = 0;
  i64 run = elsize, gstride = elsize;
  while (p < D && l[p] == g[p]) {
    run *= l[p];
    gstride *= g[p];
    ++p;
  }
  L.file_base = 0;
  if (p < D) {
    run *= l[p];
    L.file_base += o[p] * gstride;
    gstride *= g[p];
    ++p;
  }
  L.run_bytes = run;
  L.nruns = 1;
  L.nd = 0;
  for (int i = p; i < D; ++i) {
    L.ext[L.nd] = l[i];
    L.fstride[L.nd] = gstride;
    L.file_base += o[i] * gstride;
    L.nruns *= l[i];
    gstride *= g[i];
    ++L.nd;
  }
  if (L.local_bytes == 0) L.nruns = 0;
  return PA_OK;
}

i64 file_offset_of_run(const IoLayout& L, i64 r) {
  i64 off = L.file_base;
  for (int i = 0; i < L.nd; ++i) {
    off += (r % L.ext[i]) * L.fstride[i];
    r /= L.ext[i];
  }
  return off;
}

bool full_io(int fd, char* buf, i64 n, i64 off, bool write) {
  while (n > 0) {
    const ssize_t k = write ? pwrite(fd, buf, (size_t)n, (off_t)off) : pread(fd, buf, (size_t)n, (off_t)off);
    if (k < 0) {
      if (errno == EINTR) continue;
      return false;
    }
    if (k == 0) return false;  // short file
    buf += k;
    n -= k;
    off += k;
  }
  return true;
}

}  // namespace

pa_status io_sizes(const Pencil& P, int n_extra, const i64* extra, int elsize, int chunks,
                   i64* global_bytes, i64* local_bytes, i64* nruns, i64* run_bytes, i64* first_offset) {
  IoLayout L;
  pa_status s = make_layout(P, n_extra, extra, elsize, chunks != 0, L);
  if (s != PA_OK) return s;
  if (global_bytes) *global_bytes = L.global_bytes;
  if (local_bytes) *local_bytes = L.local_bytes;
  if (nruns) *nruns = L.nruns;
  if (run_bytes) *run_bytes = L.run_bytes;
  if (first_offset) *first_offset = L.file_base;
  return PA_OK;
}

pa_status io_run_offset(const Pencil& P, int n_extra, const i64* extra, int elsize, int chunks, i64 run,
                        i64* file_offset) {
  IoLayout L;
  pa_status s = make_layout(P, n_extra, extra, elsize, chunks != 0, L);
  if (s != PA_OK) return s;
  if (run < 0 || run >= L.nruns) {
    set_error("pa_io: run index out of range");
    return PA_EINVAL;
  }
  *file_offset = file_offset_of_run(L, run);
  return PA_OK;
}

pa_status io_transfer(const Pencil& P, int n_extra, const i64* extra, int elsize, int chunks, void* dev,
                      const char* path, i64 offset, bool write) {
  if (device_count() == 0) {
    set_error("no CUDA device: PencilArray storage lives in device memory");
    return PA_ENOGPU;
  }
  IoLayout L;
  pa_status s = make_layout(P, n_extra, extra, elsize, chunks != 0, L);
  if (s != PA_OK) return s;
  if (L.local_bytes > 0 && !dev) {
    set_error("pa_io: null device array");
    return PA_EINVAL;
  }
  const int fd = write ? open(path, O_WRONLY | O_CREAT, 0644) : open(path, O_RDONLY);
  if (fd < 0) {
    set_error("pa_io: cannot open '%s': %s", path, strerror(errno));
    return PA_EINVAL;
  }
  if (!write) {
    struct stat st;
    if (fstat(fd, &st) != 0 || (i64)st.st_size < offset + L.global_bytes) {
      close(fd);
      set_error("pa_io: file '%s' is smaller than the dataset (%lld bytes at offset %lld)", path,
                (long long)L.global_bytes, (long long)offset);
      return PA_EINVAL;
    }
  }
  if (L.nruns == 0) {
    close(fd);
    return PA_OK;
  }
  // Work queued on any stream of the process may still write the array (before a write) or
  // read it (before a read), and the copies below run on a stream of their own: wait for all
  // of it.  Both calls block until the transfer is done anyway.
  const cudaError_t prior = cudaDeviceSynchronize();
  if (prior != cudaSuccess) {
    close(fd);
    cudaGetLastError();
    set_error("pa_io: prior device work failed: %s", cudaGetErrorString(prior));
    return PA_ECUDA;
  }
  // pieces of whole runs, about 32 MiB each, through two pinned buffers
  const i64 target = 32ll << 20;
  const i64 runs_per_piece = std::max<i64>(1, std::min<i64>(L.nruns, target / std::max<i64>(1, L.run_bytes)));
  const i64 piece_cap = L.run_bytes <= target ? runs_per_piece * L.run_bytes : target;
  char* host[2] = {nullptr, nullptr};
  cudaStream_t st = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  pa_status rc = PA_OK;
  auto cleanup = [&]() {
    for (int i = 0; i < 2; ++i) {
      if (host[i]) cudaFreeHost(host[i]);
      if (ev[i]) cudaEventDestroy(ev[i]);
    }
    if (st) cudaStreamDestroy(st);
    close(fd);
    cudaGetLastError();
  };
  if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMallocHost((void**)&host[0], (size_t)piece_cap) != cudaSuccess ||
      cudaMallocHost((void**)&host[1], (size_t)piece_cap) != cudaSuccess ||
      cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming) != cudaSuccess) {
    cleanup();
    set_error("pa_io: staging allocation failed");
    return PA_ENOMEM;
  }
  // list of pieces: (first local byte, bytes); a run longer than a piece is split
  struct Piece {
    i64 local, bytes;
  };
  std::vector<Piece> pieces;
  if (L.run_bytes <= target) {
    for (i64 r = 0; r < L.nruns; r += runs_per_piece)
      pieces.push_back({r * L.run_bytes, std::min(runs_per_piece, L.nruns - r) * L.run_bytes});
  } else {
    for (i64 r = 0; r < L.nruns; ++r)
      for (i64 b = 0; b < L.run_bytes; b += target)
        pieces.push_back({r * L.run_bytes + b, std::min(target, L.run_bytes - b)});
  }
  auto file_io = [&](const Piece& pc, char* buf) -> bool {
    // the piece covers whole runs, or a part of one run
    i64 done = 0;
    while (done < pc.bytes) {
      const i64 lb = pc.local + done;
      const i64 r = lb / L.run_bytes, within = lb % L.run_bytes;
      const i64 n = std::min(pc.bytes - done, L.run_bytes - within);
      if (!full_io(fd, buf + done, n, offset + file_offset_of_run(L, r) + within, write)) return false;
      done += n;
    }
    return true;
  };
  const size_t np = pieces.size();
  if (write) {
    // D2H(k+1) || pwrite(k)
    cudaMemcpyAsync(host[0], (char*)dev + pieces[0].local, (size_t)pieces[0].bytes, cudaMemcpyDeviceToHost, st);
    cudaEventRecord(ev[0], st);
    for (size_t k = 0; k < np && rc == PA_OK; ++k) {
      if (k + 1 < np) {
        cudaMemcpyAsync(host[(k + 1) & 1], (char*)dev + pieces[k + 1].local, (size_t)pieces[k + 1].bytes,
                        cudaMemcpyDeviceToHost, st);
        cudaEventRecord(ev[(k + 1) & 1], st);
      }
      if (cudaEventSynchronize(ev[k & 1]) != cudaSuccess) {
        set_error("pa_io: device -> host copy failed");
        rc = PA_ECUDA;
      } else if (!file_io(pieces[k], host[k & 1])) {
        set_error("pa_io: write to '%s' failed: %s", path, strerror(errno));
        rc = PA_EINVAL;
      }
    }
  } else {
    // pread(k+1) || H2D(k)
    for (size_t k = 0; k < np && rc == PA_OK; ++k) {
      if (k >= 2 && cudaEventSynchronize(ev[k & 1]) != cudaSuccess) {  // buffer free again?
        set_error("pa_io: host -> device copy failed");
        rc = PA_ECUDA;
        break;
      }
      if (!file_io(pieces[k], host[k & 1])) {
        set_error("pa_io: read from '%s' failed: %s", path, errno ? strerror(errno) : "short file");
        rc = PA_EINVAL;
        break;
      }
      cudaMemcpyAsync((char*)dev + pieces[k].local, host[k & 1], (size_t)pieces[k].bytes,
                      cudaMemcpyHostToDevice, st);
      cudaEventRecord(ev[k & 1], st);
    }
  }
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == PA_OK) {
    set_error("pa_io: copy failed");
    rc = PA_ECUDA;
  }
  cleanup();
  return rc;
}

}  // namespace pa
