"""ctypes binding of libb200sparse.so (the C ABI declared in include/b200sparse.h).

Plays the part of the reference's cffi/opcode glue (sparse/config.py:21-152: Library subclass,
`SparseOpCode` enum import) -- here there are no opcodes, just C functions.  There is NO CPU
fallback: if the shared library cannot be loaded (or built) this module raises at import.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from . import _build

c_i32 = ctypes.c_int
c_i64 = ctypes.c_int64
c_vp = ctypes.c_void_p

OK, EINVAL, ECUDA, EUNSUPPORTED, ENOMEM = 0, 1, 2, 3, 4
F32, F64 = 0, 1
I32, I64 = 0, 1

# name -> (restype, argtypes); every symbol include/b200sparse.h declares
SIGNATURES = {
    "b2s_version": (c_i32, []),
    "b2s_last_error": (ctypes.c_char_p, []),
    "b2s_device_info": (c_i32, [c_i32, c_vp]),
    "b2s_ws_bytes": (c_i64, []),
    "b2s_spmv_plan_tiles": (c_i64, [c_i32, c_i64, c_i64]),
    "b2s_spmv_plan_bytes": (c_i64, [c_i32, c_i64, c_i64]),
    "b2s_spmv_plan_create": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
                                     ctypes.POINTER(c_vp)]),
    "b2s_spmv_plan_create_ex": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
                                        ctypes.POINTER(c_vp), c_i32]),
    "b2s_spmv_plan_destroy": (c_i32, [c_vp]),
    "b2s_spmv_plan_info": (c_i32, [c_vp, c_vp]),
    "b2s_spmv_plan_pack_bytes": (c_i64, [c_vp]),
    "b2s_spmv_plan_pack": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmv_plan_pack_coded": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmv_plan_set_packed": (c_i32, [c_vp, c_i32]),
    "b2s_spmv_plan_templates_bytes": (c_i64, [c_vp]),
    "b2s_spmv_plan_templates": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmv_csr": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmm_csr": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp,
                             c_i64, c_vp]),
    "b2s_spmm_set_kernel": (c_i32, [c_i32]),
    "b2s_spmv_plan_chunks": (c_i32, [c_vp, c_vp, c_i32, ctypes.POINTER(c_i32)]),
    "b2s_spmv_csr_tiles": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                   c_i64, c_i64, c_vp]),
    "b2s_spmv_csr_fused": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                   c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmv_csr_add": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmv_csr_host": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                  c_vp, c_vp]),
    "b2s_spmv_csr_dot": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                 c_vp, c_vp, c_vp, c_vp]),
    "b2s_axpby": (c_i32, [c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_vp]),
    "b2s_dot": (c_i32, [c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_nrm2": (c_i32, [c_i32, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "b2s_cg_update_xr": (c_i32, [c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_csr_diagonal": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spgemm_row_work": (c_i32, [c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spgemm_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "b2s_spgemm_dense_bytes": (c_i64, [c_i32, c_i64, c_i64]),
    "b2s_spgemm_csr_symbolic": (c_i32, [c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spgemm_csr_numeric": (c_i32, [c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                       c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "b2s_peer_header_bytes": (c_i64, []),
    "b2s_ipc_alloc": (c_i32, [c_i64, ctypes.POINTER(c_vp)]),
    "b2s_ipc_free": (c_i32, [c_vp]),
    "b2s_peer_allreduce": (c_i32, [c_i32, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp]),
    "b2s_peer_halo_exchange": (c_i32, [c_i32, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp, c_i32, c_vp, c_vp]),
    "b2s_peer_push": (c_i32, [c_i32, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp, c_i32, c_vp, c_i32, c_vp]),
    "b2s_peer_push_wait": (c_i32, [c_i32, c_i32, c_vp, c_i32, c_vp, c_vp]),
    "b2s_peer_header_offset": (c_i64, [c_i32, c_i32]),
    "b2s_peer_check": (c_i32, [c_vp, c_vp, c_vp]),
    "b2s_ipc_export": (c_i32, [c_vp, c_vp]),
    "b2s_ipc_open": (c_i32, [c_vp, ctypes.POINTER(c_vp)]),
    "b2s_ipc_close": (c_i32, [c_vp]),
    "b2s_copy": (c_i32, [c_i32, c_i64, c_vp, c_vp, c_vp]),
    "b2s_convert_scratch_bytes": (c_i64, [c_i64, c_i32]),
    "b2s_coo_to_csr": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_csr_transpose": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_csr_sort_rows": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_csr_binop_scratch_bytes": (c_i64, [c_i64]),
    "b2s_csr_binop_symbolic": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                       c_vp]),
    "b2s_csr_binop_numeric": (c_i32, [c_i32, c_i32, c_i32, c_i32, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                      c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_csr_scale": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp,
                              c_vp]),
    "b2s_sddmm_csr": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp,
                              c_i64, c_vp, c_vp]),
    "b2s_tropical_spmv_csr": (c_i32, [c_i32, c_i32, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_i64,
                                      c_vp]),
    "b2s_csr_reduce_rows": (c_i32, [c_i32, c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i32, c_vp,
                                    c_vp]),
    "b2s_csr_select_scratch_bytes": (c_i64, [c_i64]),
    "b2s_csr_select": (c_i32, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp,
                               c_i64, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp]),
    "b2s_csr_lookup": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp,
                               c_vp, c_vp]),
    "b2s_csr_kron": (c_i32, [c_i32, c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i32, c_i32, c_i64,
                             c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_csr_blocks_scratch_bytes": (c_i64, [c_i64]),
    "b2s_csr_blocks": (c_i32, [c_i32, c_i32, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmv_csc": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmm_csc": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp,
                             c_i64, c_vp]),
    "b2s_spmv_dia": (c_i32, [c_i32, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_spmm_dia": (c_i32, [c_i32, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp]),
    "b2s_dia_scratch_bytes": (c_i64, [c_i64, c_i64]),
    "b2s_dia_to_csr": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                               c_vp, c_vp, c_i64, c_vp, c_vp]),
    "b2s_csr_to_dia": (c_i32, [c_i32, c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp,
                               c_vp, c_i64, c_vp, c_vp]),
    "b2s_random_table_slots": (c_i64, [c_i64]),
    "b2s_random_sample": (c_i32, [c_i32, c_i64, c_i64, c_i64, ctypes.c_uint64, c_vp, c_i64, c_vp, c_vp, c_vp,
                                  ctypes.POINTER(c_i64), c_vp]),
    "b2s_random_complement": (c_i32, [c_i32, c_i32, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2s_random_values": (c_i32, [c_i32, c_i32, c_i64, ctypes.c_uint64, c_vp, c_vp]),
    "b2s_comm_nccl_version": (c_i32, []),
    "b2s_comm_unique_id": (c_i32, [c_vp]),
    "b2s_comm_init": (c_i32, [c_i32, c_i32, c_vp, ctypes.POINTER(c_vp)]),
    "b2s_comm_destroy": (c_i32, [c_vp]),
    "b2s_allgather_x": (c_i32, [c_i32, c_i32, c_vp, c_i64, c_vp, c_vp]),
    "b2s_allreduce_scalars": (c_i32, [c_vp, c_vp, c_i32, c_vp]),
    "b2s_probe_gather": (c_i32, [c_i32, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "b2s_device_l2_fetch_granularity": (c_i32, [c_i32, ctypes.POINTER(c_i64)]),
    # tuning hooks (not in the public header)
    "b2s_spmv_set_config": (c_i32, [c_i32, c_i32]),
    "b2s_spmv_get_config": (c_i32, []),
    "b2s_spmv_num_configs": (c_i32, []),
    "b2s_spmv_plan_set_kernel": (c_i32, [c_vp, c_i32]),
    "b2s_spmv_plan_set_flavor": (c_i32, [c_vp, c_i32]),
    "b2s_spmv_set_template_config": (c_i32, [c_i32, c_i32, c_i32]),
}


class FuseDesc(ctypes.Structure):
    """b2s_fuse_desc of include/b200sparse.h (the exchange fused into b2s_spmv_csr_fused)."""

    _fields_ = [
        ("nranges", ctypes.c_int32), ("n_free", ctypes.c_int32),
        ("ranges", c_i64 * 12),
        ("n_flags", ctypes.c_int32), ("n_sends", ctypes.c_int32), ("n_acks", ctypes.c_int32),
        ("accumulate", ctypes.c_int32),
        ("flag", c_vp * 8),
        ("send_src", c_vp * 4), ("send_dst", c_vp * 4), ("send_count", c_i64 * 4),
        ("send_flag", c_vp * 4), ("send_ack", c_vp * 4),
        ("ack_out", c_vp * 8),
        ("epoch_ctr", c_vp), ("ticket", c_vp),
        ("epoch_add", ctypes.c_int32), ("epoch_bump", ctypes.c_int32),
        ("expect", ctypes.c_uint64),
        ("error", c_vp),
    ]


# b2s_block_desc of include/b200sparse.h (one block of b2s_csr_blocks), as a numpy record so a table of many blocks
# is filled column by column
BLOCK_DESC = np.dtype([("indptr", np.uint64), ("indices", np.uint64), ("vals", np.uint64), ("it", np.int32),
                       ("pt", np.int32), ("nrows", np.int64), ("ncols", np.int64), ("nnz", np.int64),
                       ("row_block", np.int64), ("row_off", np.int64), ("col_off", np.int64)])


class B200SparseError(RuntimeError):
    pass


def _load() -> ctypes.CDLL:
    path = _build.LIB_PATH
    if not os.path.exists(path) or (_build.needs_build() and _build.shutil.which("nvcc")):
        try:
            _build.build()
        except Exception as exc:  # pragma: no cover - environment dependent
            if not os.path.exists(path):
                raise ImportError(
                    "legate.sparse_b200: libb200sparse.so is missing and could not be built "
                    f"({exc}). There is no CPU fallback."
                ) from exc
    try:
        lib = ctypes.CDLL(path)
    except OSError as exc:
        raise ImportError(f"legate.sparse_b200: cannot load {path}: {exc}. There is no CPU fallback.") from exc
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = ABI mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
LIB_PATH = _build.LIB_PATH


def last_error() -> str:
    return lib.b2s_last_error().decode("utf-8", "replace")


def check(rc: int, what: str = "") -> None:
    if rc != OK:
        names = {EINVAL: "EINVAL", ECUDA: "ECUDA", EUNSUPPORTED: "EUNSUPPORTED", ENOMEM: "ENOMEM"}
        raise B200SparseError(f"{what or 'libb200sparse'} failed [{names.get(rc, rc)}]: {last_error()}")
