"""ctypes binding of libpa_b200.so (the C ABI in include/pa_b200.h).

This is the same kind of stub the Julia veneer uses via ``ccall`` (see
INTEGRATION.md); nothing here computes anything.  The library is mandatory:
importing the package fails loudly if it has not been built -- there is no
Python/NumPy fallback for the data path.
"""
from __future__ import annotations

import ctypes as C
import os

PA_MAX_DIMS = 8
PA_MAX_TOPO = 7
PA_UNIQUE_ID_BYTES = 128

PA_OK, PA_EINVAL, PA_EINCOMPAT, PA_EDIM, PA_ECUDA, PA_ENCCL, PA_ENOMEM, PA_ESTATE, PA_ENOGPU = range(9)

PA_POINT_TO_POINT = 0
PA_ALLTOALLV = 1
PA_PEER_PUT = 2
PA_PEER_GET = 3
PA_IPC_HANDLE_BYTES = 64

PA_WAITALL = 1
PA_NO_OVERLAP = 2
PA_STAGE_SELF = 4
PA_FFT_FORWARD = 8
PA_FFT_BACKWARD = 16
PA_FFT_F32 = 32

# real-to-real kinds (pa_r2r), FFTW's fftw_r2r_kind values
PA_REDFT01 = 4
PA_REDFT10 = 5
PA_RODFT01 = 8
PA_RODFT10 = 9

# distributed reductions (pa_reduce): element types, maps, ops and the predicates of any / all
PA_FLOAT64, PA_FLOAT32, PA_COMPLEXF64, PA_COMPLEXF32, PA_INT32, PA_INT64, PA_BOOL = range(7)
PA_MAP_IDENTITY, PA_MAP_ABS, PA_MAP_ABS2, PA_MAP_DOT = range(4)
PA_OP_SUM, PA_OP_MAX, PA_OP_MIN, PA_OP_ANY, PA_OP_ALL = range(5)
PA_SPECTRUM_MAX_BINS = 4096
(PA_PRED_EQ, PA_PRED_NE, PA_PRED_LT, PA_PRED_LE, PA_PRED_GT, PA_PRED_GE, PA_PRED_ISNAN,
 PA_PRED_ISFINITE) = (k << 4 for k in range(1, 9))

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpa_b200.so")


class PlanInfo(C.Structure):
    _fields_ = [
        ("dim", C.c_int), ("nproc", C.c_int), ("self_index", C.c_int), ("same_perm", C.c_int),
        ("elsize", C.c_int), ("method", C.c_int),
        ("length_in", C.c_int64), ("length_out", C.c_int64), ("length_self", C.c_int64),
        ("send_bytes", C.c_int64), ("recv_bytes", C.c_int64),
    ]


class PeerInfo(C.Structure):
    _fields_ = [
        ("world_rank", C.c_int), ("is_self", C.c_int),
        ("send_offset", C.c_int64), ("send_count", C.c_int64),
        ("recv_offset", C.c_int64), ("recv_count", C.c_int64),
        ("remote_recv_offset", C.c_int64),
    ]


class BlockDesc(C.Structure):
    _fields_ = [
        ("nd", C.c_int),
        ("extent", C.c_int64 * PA_MAX_DIMS),
        ("src_stride", C.c_int64 * PA_MAX_DIMS),
        ("dst_stride", C.c_int64 * PA_MAX_DIMS),
        ("src_offset", C.c_int64), ("dst_offset", C.c_int64),
        ("kernel_class", C.c_int), ("vec_bytes", C.c_int),
    ]


class Timings(C.Structure):
    _fields_ = [("total_ms", C.c_float), ("pack_ms", C.c_float),
                ("exchange_ms", C.c_float), ("unpack_ms", C.c_float)]


# every symbol include/pa_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
_I64P = C.POINTER(C.c_int64)
_IP = C.POINTER(C.c_int)
SIGNATURES = {
    "pa_version": (C.c_char_p, []),
    "pa_strerror": (C.c_char_p, [C.c_int]),
    "pa_last_error": (C.c_char_p, []),
    "pa_launch_count": (C.c_int64, []),
    "pa_device_count": (C.c_int, []),
    "pa_set_device": (C.c_int, [C.c_int]),
    "pa_set_tunable": (C.c_int, [C.c_char_p, C.c_int64]),
    "pa_dims_create": (C.c_int, [C.c_int, C.c_int, _I64P]),
    "pa_topology_create": (C.c_int, [C.c_int, _I64P, C.c_int, C.POINTER(_P)]),
    "pa_topology_destroy": (None, [_P]),
    "pa_topology_info": (C.c_int, [_P, _IP, _I64P, _IP, _IP, _I64P]),
    "pa_topology_rank_of": (C.c_int, [_P, _I64P, _IP]),
    "pa_topology_line": (C.c_int, [_P, C.c_int, _IP]),
    "pa_pencil_create": (C.c_int, [_P, C.c_int, _I64P, _IP, _IP, _P, C.POINTER(_P)]),
    "pa_pencil_destroy": (None, [_P]),
    "pa_pencil_range": (C.c_int, [_P, _I64P, C.c_int, _I64P, _I64P]),
    "pa_pencil_size_local": (C.c_int, [_P, C.c_int, _I64P]),
    "pa_pencil_buffers": (C.c_int, [_P, C.POINTER(_P), _I64P, C.POINTER(_P), _I64P]),
    "pa_pencil_reserve": (C.c_int, [_P, C.c_int64, C.c_int64]),
    "pa_plan_create": (C.c_int, [_P, _P, C.c_int, _I64P, C.c_int, C.c_int, C.POINTER(_P)]),
    "pa_plan_destroy": (None, [_P]),
    "pa_plan_get_info": (C.c_int, [_P, C.POINTER(PlanInfo)]),
    "pa_plan_get_peer": (C.c_int, [_P, C.c_int, C.POINTER(PeerInfo)]),
    "pa_plan_get_block": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(BlockDesc)]),
    "pa_plan_get_chunk": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(BlockDesc),
                                    _I64P, _I64P]),
    "pa_pack": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "pa_unpack": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "pa_put": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "pa_get": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "pa_put_all": (C.c_int, [_P, _P, C.POINTER(_P), C.c_int, _P]),
    "pa_get_all": (C.c_int, [_P, C.POINTER(_P), _P, C.c_int, _P]),
    "pa_get_all_fft": (C.c_int, [_P, _P, C.POINTER(_P), _P, C.c_uint, _P]),
    "pa_copy_self": (C.c_int, [_P, _P, _P, _P]),
    "pa_permute_local": (C.c_int, [_P, _P, _P, _P, _P]),
    "pa_box_copy": (C.c_int, [C.c_int, _I64P, _I64P, _I64P, C.c_int, _P, _P, _P,
                              C.POINTER(BlockDesc)]),
    "pa_comm_unique_id": (C.c_int, [_P]),
    "pa_comm_init_rank": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(_P)]),
    "pa_comm_init_local": (C.c_int, [C.c_int, C.c_int, C.POINTER(_P)]),
    "pa_comm_destroy": (None, [_P]),
    "pa_comm_flags_export": (C.c_int, [_P, _P, _I64P]),
    "pa_comm_flags_import": (C.c_int, [_P, C.c_int, _P, C.c_int64]),
    "pa_ipc_export": (C.c_int, [_P, _P, _I64P]),
    "pa_ipc_import": (C.c_int, [_P, C.c_int64, C.POINTER(_P)]),
    "pa_ipc_release": (C.c_int, [_P]),
    "pa_plan_set_window": (C.c_int, [_P, _P, C.c_int, _P]),
    "pa_plan_set_recv_window": (C.c_int, [_P, C.c_int, _P]),
    "pa_transpose": (C.c_int, [_P, _P, _P, _P, C.c_uint, _P]),
    "pa_wait": (C.c_int, [_P, _P]),
    "pa_plan_fft_check": (C.c_int, [_P]),
    "pa_plan_fft_check_ex": (C.c_int, [_P, C.c_uint]),
    "pa_transpose_host": (C.c_int, [_P, _P, _P, _P, C.c_uint]),
    "pa_rfft": (C.c_int, [_P, _P, C.c_int, _I64P, C.c_uint, _P, _P, _P]),
    "pa_r2r": (C.c_int, [_P, C.c_int, _I64P, C.c_int, C.c_uint, _P, _P, _P]),
    "pa_transpose_brfft": (C.c_int, [_P, _P, _P, _P, _P, C.c_uint, _P]),
    "pa_plan_brfft_check": (C.c_int, [_P, C.c_uint]),
    "pa_transpose_r2r": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_uint, _P]),
    "pa_transpose_rfft": (C.c_int, [_P, _P, _P, _P, _P, C.c_uint, _P]),
    "pa_plan_real_check": (C.c_int, [_P, C.c_uint]),
    "pa_fft_put": (C.c_int, [_P, _P, _P, _P, C.c_uint, _P]),
    "pa_rfft_put": (C.c_int, [_P, _P, _P, _P, _P, C.c_uint, _P]),
    "pa_put_all_fft": (C.c_int, [_P, _P, C.POINTER(_P), _P, C.c_uint, _P]),
    "pa_put_all_rfft": (C.c_int, [_P, _P, _P, C.POINTER(_P), _P, C.c_uint, _P]),
    "pa_plan_fft_put_check": (C.c_int, [_P, C.c_uint]),
    "pa_plan_rfft_put_check": (C.c_int, [_P, C.c_uint]),
    "pa_r2r_put": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_uint, _P]),
    "pa_brfft_put": (C.c_int, [_P, _P, _P, _P, _P, C.c_uint, _P]),
    "pa_put_all_r2r": (C.c_int, [_P, C.c_int, _P, C.POINTER(_P), _P, C.c_uint, _P]),
    "pa_put_all_brfft": (C.c_int, [_P, _P, _P, C.POINTER(_P), _P, C.c_uint, _P]),
    "pa_plan_real_put_check": (C.c_int, [_P, C.c_uint]),
    "pa_host_chain_create": (C.c_int, [C.c_int, C.POINTER(_P), _P, C.POINTER(_P)]),
    "pa_host_chain_destroy": (None, [_P]),
    "pa_host_chain_submit": (C.c_int, [_P, _P, _P, _I64P]),
    "pa_host_chain_wait": (C.c_int, [_P, C.c_int64]),
    "pa_host_chain_time_begin": (C.c_int, [_P]),
    "pa_host_chain_time_end": (C.c_int, [_P, C.POINTER(C.c_float)]),
    "pa_host_chain_buffer": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(_P), _I64P]),
    "pa_io_sizes": (C.c_int, [_P, C.c_int, _I64P, C.c_int, C.c_int, _I64P, _I64P, _I64P, _I64P, _I64P]),
    "pa_io_run_offset": (C.c_int, [_P, C.c_int, _I64P, C.c_int, C.c_int, C.c_int64, _I64P]),
    "pa_io_write": (C.c_int, [_P, C.c_int, _I64P, C.c_int, C.c_int, _P, C.c_char_p, C.c_int64]),
    "pa_io_read": (C.c_int, [_P, C.c_int, _I64P, C.c_int, C.c_int, _P, C.c_char_p, C.c_int64]),
    "pa_reduce": (C.c_int, [_P, C.c_int, _I64P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "pa_reduce_result_type": (C.c_int, [C.c_int, C.c_int, C.c_int, _IP]),
    "pa_reduce_dims": (C.c_int, [_P, C.c_int, _I64P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P,
                                 C.c_int, _IP, _P, _P]),
    "pa_shell_spectrum": (C.c_int, [_P, C.c_int, _I64P, _P, C.c_int, C.c_int, _P, _P, C.c_int,
                                    C.c_int64, _P, C.c_double, C.c_int, _P, _P]),
    "pa_shell_spectrum_nbins": (C.c_int, [_P, C.c_int, C.c_int64, _P, C.c_double, _IP]),
    "pa_shell_spectrum_dims": (C.c_int, [_P, C.c_int, _I64P, _P, C.c_int, C.c_int, _P, _P, C.c_int,
                                         C.c_int64, _P, C.c_double, C.c_int, C.c_int, _IP, C.c_int,
                                         _IP, _P, _P]),
    "pa_shell_spectrum_dims_nbins": (C.c_int, [_P, C.c_int, C.c_int64, _P, C.c_double, C.c_int, _IP,
                                               _IP]),
    "pa_plan_timings": (C.c_int, [_P, C.POINTER(Timings)]),
    "pa_plan_enable_timing": (C.c_int, [_P, C.c_int]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (or `make -C pencilarrays.jl_b200/csrc`). The transpose! path has no "
            "CPU/Python fallback.")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


class PencilError(Exception):
    """Base class of errors raised for a non-zero ``pa_status``."""

    def __init__(self, status, detail):
        self.status = status
        super().__init__(f"{lib.pa_strerror(status).decode()}: {detail}" if detail
                         else lib.pa_strerror(status).decode())


class ArgumentError(PencilError, ValueError):
    """Julia ``ArgumentError`` (PA_EINVAL / PA_EINCOMPAT)."""


class DimensionMismatch(PencilError, ValueError):
    """Julia ``DimensionMismatch`` (PA_EDIM)."""


class DeviceError(PencilError, RuntimeError):
    """CUDA / NCCL / device-availability failures."""


def check(status: int) -> None:
    if status == PA_OK:
        return
    detail = lib.pa_last_error().decode()
    if status in (PA_EINVAL, PA_EINCOMPAT):
        raise ArgumentError(status, detail)
    if status == PA_EDIM:
        raise DimensionMismatch(status, detail)
    raise DeviceError(status, detail)


def i64arr(vals):
    vals = list(vals)
    return (C.c_int64 * max(1, len(vals)))(*vals)


def intarr(vals):
    vals = list(vals)
    return (C.c_int * max(1, len(vals)))(*vals)
