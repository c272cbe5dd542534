"""ctypes binding of the C ABI in include/matrel.h (the same entry points a JNI shim would bind).

The shared library is built in-tree by ``__graft_entry__.build()`` (``matrel_b200/libmatrel_b200.so``).
If it is missing, importing this module raises: there is no Python / CPU fallback for the
operators.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmatrel_b200.so")

MR_OK, MR_EINVAL, MR_EDIM, MR_ENOMEM, MR_ECUDA, MR_ENOTSUP, MR_ENOTFOUND, MR_ENCCL = range(8)


class MatrelError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(msg)
        self.code = code


class IllegalArgumentException(MatrelError, ValueError):
    """`require` failure of the reference (message starts with 'requirement failed: ')."""


class UnsupportedOperation(MatrelError):
    pass


class CudaError(MatrelError):
    pass


class mr_block_desc(C.Structure):
    _fields_ = [
        ("type", C.c_uint8),
        ("numRows", C.c_int32),
        ("numCols", C.c_int32),
        ("colPtrs", C.POINTER(C.c_int32)),
        ("rowIndices", C.POINTER(C.c_int32)),
        ("values", C.POINTER(C.c_double)),
        ("isTransposed", C.c_uint8),
        ("colPtrsLen", C.c_int64),
        ("rowIndicesLen", C.c_int64),
        ("valuesLen", C.c_int64),
    ]


class mr_options(C.Structure):
    _fields_ = [
        ("device", C.c_int32),
        ("compat_bugs", C.c_int32),
        ("gemm_algo", C.c_int32),
        ("ozaki_slices", C.c_int32),
        ("stream", C.c_void_p),
    ]


class mr_stats(C.Structure):
    _fields_ = [
        ("kernel_launches", C.c_int64),
        ("gemm_launches", C.c_int64),
        ("h2d_bytes", C.c_int64),
        ("d2h_bytes", C.c_int64),
        ("last_gemm_ms", C.c_double),
        ("gemm_ms_total", C.c_double),
        ("last_gemm_flops", C.c_int64),
        ("tc_gemm_ms_total", C.c_double),
        ("tc_gemm_launches", C.c_int64),
        ("tc_int8_ops", C.c_int64),
        ("p2p_bytes", C.c_int64),
        ("tc_moduli", C.c_int64),
    ]


class mr_grid_layout(C.Structure):
    _fields_ = [
        ("nrows", C.c_int64),
        ("ncols", C.c_int64),
        ("blkSize", C.c_int32),
        ("pr", C.c_int32),
        ("pc", C.c_int32),
        ("r", C.c_int32),
        ("c", C.c_int32),
    ]


_P = C.c_void_p
_PP = C.POINTER(C.c_void_p)
_i32, _i64, _f64 = C.c_int32, C.c_int64, C.c_double
_BIN = [_P, _i64, _i64, _P, _i64, _i64, _i32, _PP]

# name -> argtypes; every symbol include/matrel.h declares (tests/test_abi_cpu.py checks the two agree)
SIGNATURES = {
    "mr_init": [C.POINTER(mr_options), _PP],
    "mr_shutdown": [_P],
    "mr_set_stream": [_P, _P],
    "mr_set_option": [_P, C.c_char_p, _i64],
    "mr_sync": [_P],
    "mr_wait_ingest": [_P],
    "mr_wait_ingest_on": [_P, _P],
    "mr_matrix_create": [_P, _PP],
    "mr_matrix_free": [_P],
    "mr_matrix_put_block": [_P, _i32, _i32, C.POINTER(mr_block_desc)],
    "mr_matrix_put_blocks": [_P, _i64, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(mr_block_desc)],
    "mr_matrix_wait_ingest": [_P],
    "mr_matrix_put_block_device": [_P, _i32, _i32, _i32, _i32, _P, C.c_uint8],
    "mr_matrix_put_blocks_device": [_P, _i64, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32),
                                    C.POINTER(C.c_void_p), C.POINTER(C.c_uint8)],
    "mr_matrix_num_blocks": [_P, C.POINTER(_i64)],
    "mr_matrix_has_block": [_P, _i32, _i32, C.POINTER(_i32)],
    "mr_matrix_block_ids": [_P, C.POINTER(_i32), C.POINTER(_i32), _i64],
    "mr_matrix_get_block": [_P, _i32, _i32, C.POINTER(mr_block_desc)],
    "mr_matrix_block_device_ptr": [_P, _i32, _i32, _PP],
    "mr_matrix_rand": [_P, _i64, _i64, _i32, _i64, _PP],
    "mr_matrix_sprand": [_P, _i64, _i64, _i32, _f64, _i64, C.c_uint8, _PP],
    "mr_matrix_rand_partition": [_P, _i64, _i64, _i32, _i64, _i32, _i32, _i32, _i32, _P, _i64, _PP],
    "mr_matrix_multiply": _BIN,
    "mr_transpose": [_P, _PP],
    "mr_add_element": _BIN,
    "mr_multiply_element": _BIN,
    "mr_divide_element": _BIN,
    "mr_add_scalar": [_P, _f64, _PP],
    "mr_multiply_scalar": [_P, _f64, _PP],
    "mr_power": [_P, _f64, _PP],
    "mr_rank_one_update": _BIN,
    "mr_materialize": [_P, _PP],
    "mr_vec": [_P, _i64, _i64, _i32, _PP],
    "mr_project": [_P, _i64, _i64, _i32, _i32, _i64, _PP],
    "mr_selection": [_P, _i64, _i64, _i32, _i64, _i64, _PP],
    "mr_row_sum": [_P, _i64, _i64, _PP],
    "mr_col_sum": [_P, _i64, _i64, _PP],
    "mr_sum": [_P, _i64, _i64, _PP],
    "mr_trace": [_P, _i64, _i64, _PP],
    "mr_row_partition": [_i32, _i32, _i32, C.POINTER(_i32)],
    "mr_column_partition": [_i32, _i32, _i32, C.POINTER(_i32)],
    "mr_index_partition": [_i32, _i32, C.POINTER(_i32)],
    "mr_gen_block_cyclic": [_i64, _i64, _i32, C.POINTER(_i32)],
    "mr_block_cyclic_partition": [C.POINTER(_i32), _i32, _i32, C.POINTER(_i32)],
    "mr_block_cyclic_num_partitions": [C.POINTER(_i32), C.POINTER(_i32)],
    "mr_partition_id": [_i32, C.POINTER(_i32), _i32, _i32, C.POINTER(_i32)],
    "mr_matrix_create_sharded": [_P, C.POINTER(mr_grid_layout), _PP],
    "mr_matrix_adopt_sharded": [_P, C.POINTER(mr_grid_layout), _P, C.c_uint8, _PP],
    "mr_matrix_layout": [_P, C.POINTER(mr_grid_layout)],
    "mr_matrix_slab": [_P, _PP, C.POINTER(_i64)],
    "mr_ipc_export": [_P, _P, C.POINTER(_i64)],
    "mr_ipc_open": [_P, _P, _i64, _PP],
    "mr_ipc_close_all": [_P],
    "mr_memcpy_d2h": [_P, _P, _P, _i64],
    "mr_grid_multiply": [_P, _P, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), _i32, _PP],
    "mr_grid_multiply_gated": [_P, _P, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), _i32, C.POINTER(C.c_void_p), _PP],
    "mr_grid_multiply_rows": [_P, _i64, _i64, _P, C.POINTER(C.c_void_p), _PP],
    "mr_matrix_filter_blocks": [_P, _i32, _i32, _i32, _i32, _PP],
    "mr_init_grid": [C.POINTER(mr_options), _i32, _PP],
    "mr_grid_shutdown": [_P],
    "mr_grid_info": [_P, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32)],
    "mr_grid_context": [_P, _i32, _PP],
    "mr_grid_sync": [_P],
    "mr_dmatrix_create": [_P, _i64, _i64, _i32, _PP],
    "mr_dmatrix_rand": [_P, _i64, _i64, _i32, _i64, _PP],
    "mr_dmatrix_free": [_P],
    "mr_dmatrix_dims": [_P, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i32)],
    "mr_dmatrix_owner": [_P, _i32, _i32, C.POINTER(_i32)],
    "mr_dmatrix_part": [_P, _i32, _PP],
    "mr_dmatrix_put_block": [_P, _i32, _i32, C.POINTER(mr_block_desc)],
    "mr_dmatrix_get_block": [_P, _i32, _i32, C.POINTER(mr_block_desc)],
    "mr_dmatrix_has_block": [_P, _i32, _i32, C.POINTER(_i32)],
    "mr_dmatrix_num_blocks": [_P, C.POINTER(_i64)],
    "mr_dmatrix_multiply": [_P, _P, _PP],
    "mr_dmatrix_elementwise": [_i32, _P, _P, _PP],
    "mr_dmatrix_reduce_scalar": [_P, _i32, C.POINTER(_f64)],
    "mr_dmatrix_repartition": [_P, _i32, _i32, _PP],
    "mr_dmatrix_transpose": [_P, _PP],
    "mr_dmatrix_scalar": [_i32, _P, _f64, _PP],
    "mr_dmatrix_axis_sum": [_P, _i32, _PP],
    "mr_dmatrix_project": [_P, _i32, _i64, _PP],
    "mr_dmatrix_selection": [_P, _i64, _i64, _PP],
    "mr_get_stats": [_P, C.POINTER(mr_stats)],
    "mr_reset_stats": [_P],
}
_STR_FUNCS = ("mr_last_error", "mr_version")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(nvcc, sm_90a). matrel_b200 has no CPU fallback.")

lib = C.CDLL(LIB_PATH)
for _name, _args in SIGNATURES.items():
    _f = getattr(lib, _name)
    _f.argtypes = _args
    _f.restype = C.c_int32
for _name in _STR_FUNCS:
    _f = getattr(lib, _name)
    _f.argtypes = []
    _f.restype = C.c_char_p


def last_error() -> str:
    return lib.mr_last_error().decode("utf-8", "replace")


def check(status: int) -> None:
    if status == MR_OK:
        return
    msg = last_error()
    if status in (MR_EINVAL, MR_EDIM):
        raise IllegalArgumentException(status, msg)
    if status == MR_ENOTSUP:
        raise UnsupportedOperation(status, msg)
    if status == MR_ECUDA:
        raise CudaError(status, msg)
    if status == MR_ENOMEM:
        raise MemoryError(msg)
    if status == MR_ENOTFOUND:
        raise KeyError(msg)
    raise MatrelError(status, msg)
