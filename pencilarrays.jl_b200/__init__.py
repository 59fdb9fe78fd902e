"""H100-native implementation of the PencilArrays.jl global-transposition path.

Host-side mirror (Python; Julia is not available in this image -- the Julia
veneer over the same C ABI is in ``julia/B200PencilArrays.jl``) of the
reference's ``Pencil`` / ``PencilArray`` / ``Transpositions`` interface.  All
data movement runs in hand-written sm_90a CUDA kernels inside
``libpa_b200.so``; importing this package without that library fails.

The directory name contains a dot, so import it through the repo-root shim:

    import pencilarrays_b200 as pa
"""
from . import _lib
from ._lib import (lib, check, PencilError, ArgumentError, DimensionMismatch, DeviceError,
                   PA_WAITALL, PA_NO_OVERLAP, PA_STAGE_SELF)
from .comm import Comm, COMM_SELF, comm_world
from .permutations import (Permutation, NoPermutation, AbstractPermutation, inv, append,
                           isidentity, isperm)
from .pencils import (MPITopology, Pencil, MemoryOrder, LogicalOrder, topology, decomposition,
                      permutation, range_local, range_remote, size_global, length_local,
                      length_global, to_local, get_comm, coords_local, default_decomposition)
from .arrays import (PencilArray, ManyPencilArray, parent, pencil, extra_dims, ndims_extra,
                     size_local, similar)
from . import transpositions as Transpositions
from .transpositions import (Transposition, transpose_, transpose_bang, Waitall, PointToPoint,
                             Alltoallv, PeerPut, PeerGet, HostChain, transpose_host_, set_tunable, fft_,
                             rfft_, brfft_, r2r_)


from . import reductions
from .reductions import mapreduce, sum, maximum, minimum, any, all, abs2, realdot
from .reductions import shell_spectrum, spectrum_nbins


from . import pencilio as PencilIO
from .pencilio import MPIIODriver, MPIFile, open_, read_, sizeof_global


def launch_count() -> int:
    """Number of CUDA kernels libpa_b200 has launched in this process."""
    return int(lib.pa_launch_count())


def device_count() -> int:
    return int(lib.pa_device_count())


__version__ = lib.pa_version().decode()
