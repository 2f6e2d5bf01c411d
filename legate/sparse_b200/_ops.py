"""Leaf-op launchers: torch device tensors in, C-ABI calls out.

This is the layer that corresponds to the reference's "task builders" (free functions
`spmv` sparse/csr.py:863-968, `cg_axpby` sparse/linalg.py:479-496, `spgemm_csr_csr_csr`
sparse/csr.py:1317-1490): they marshal stores into a task launch; here they marshal device
pointers into libb200sparse.so.  Everything runs on the caller's current CUDA stream.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .runtime import idx_code, ptr, runtime, torch_dtype, vt_code

L = _lib.lib


def _stream():
    return runtime.stream_ptr()


def _chk_dev(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            runtime.require_cuda("legate.sparse_b200 kernel launch")
            raise RuntimeError("operand is not a CUDA tensor; legate.sparse_b200 has no CPU fallback")


# ---- SpMV -----------------------------------------------------------------------------------------
class SpmvPlan:
    """Host handle + device buffer of a b2s SpMV plan (see include/b200sparse.h)."""

    def __init__(self, handle: int, buf: torch.Tensor, pack_buf: torch.Tensor | None = None):
        self.handle = handle
        self.buf = buf
        # the packed structure (b2s_spmv_plan_pack / _pack_coded), read by every launch with this plan: it lives as long
        # as the plan, and is never rewritten (a captured launch may still read it)
        self.pack_buf = pack_buf
        # the row templates (b2s_spmv_plan_templates): same lifetime rule as pack_buf
        self.tpl_buf = None
        self._info()

    def _info(self):
        out = (_lib.c_i64 * 4)()
        _lib.check(L.b2s_spmv_plan_info(self.handle, out), "b2s_spmv_plan_info")
        self.config, self.rowgroup, self.uniform, self.scattered = int(out[0]), bool(out[1] & 1), bool(out[1] & 2), bool(out[1] & 4)
        self.short_rows, self.tma, self.packed = bool(out[1] & 8), bool(out[1] & 16), bool(out[1] & 32)
        self.coded, self.ndict = bool(out[1] & 64), int(out[1] >> 8) & 31
        self.templated, self.ntemplates = bool(out[1] & 128), int(out[1] >> 16) & 255
        self.tiles, self.lines_per_warp = int(out[2]), out[3] / 1000.0

    @property
    def chunks(self):
        """Row chunks for pipelined host<->device products: list of (tile_lo, tile_hi, row_lo, row_hi, col_lo, col_hi);
        empty when the plan is too small or not a TMA tile plan."""
        if getattr(self, "_chunks", None) is None:
            out = (_lib.c_i64 * (6 * 16))()
            n = ctypes.c_int(0)
            _lib.check(L.b2s_spmv_plan_chunks(self.handle, out, 16, ctypes.byref(n)), "b2s_spmv_plan_chunks")
            self._chunks = [tuple(int(out[6 * c + k]) for k in range(6)) for c in range(n.value)]
        return self._chunks

    def set_kernel(self, rowgroup: bool):
        _lib.check(L.b2s_spmv_plan_set_kernel(self.handle, int(bool(rowgroup))), "b2s_spmv_plan_set_kernel")
        self._info()

    def set_flavor(self, flavor: int):
        """tools / tests: 0 generic, 1 uniform rows, 2 short rows (one lane per row)."""
        _lib.check(L.b2s_spmv_plan_set_flavor(self.handle, int(flavor)), "b2s_spmv_plan_set_flavor")
        self._info()

    def set_packed(self, mode):
        """tools / tests: 0 / False = stream the CSR arrays, 1 / True = the packed structure and the values, 2 = the
        packed structure with coded values (the plan must have been packed / coded), 3 = row templates for whole-matrix
        products (the plan must have them)."""
        _lib.check(L.b2s_spmv_plan_set_packed(self.handle, int(mode)), "b2s_spmv_plan_set_packed")
        self._info()

    @property
    def kernel_name(self) -> str:
        """The kernel this plan launches, for the bench line (derived from the plan, not a literal)."""
        if self.rowgroup:
            return "b2s::spmv_rowgroup_kernel"
        fl = "short-rows(one lane per row)" if self.short_rows else ("uniform-rows" if self.uniform else "generic")
        if self.packed:
            fl += ", packed u16 columns/row offsets"
        if self.coded:
            fl += f", coded values ({self.ndict} distinct)"
        tiles = f"b2s::spmv_{'tma' if self.tma else 'tile'}_kernel cfg {self.config} [{fl}]"
        if self.templated:
            # whole-matrix products; tile ranges, fused exchanges and y += A x keep the tile kernel
            return f"b2s::spmv_template_kernel [{self.ntemplates} row templates, uint8 code per 32-row group, ids of mixed groups; tiles: {tiles}]"
        return tiles

    # bytes of the TemplateTable at the head of tpl_buf (spmv_common.cuh)
    TPL_TABLE_BYTES = 32 * 8 * 8 + 32 * 8 + 32 * 8 * 4 + 32 * 4

    def template_sections(self, nrows):
        """tools / tests: (ids, codes) -- uint8 views of tpl_buf's per-row template ids and per-32-row-group codes
        (0xFF for a group whose rows hold more than one template)."""
        r16 = lambda b: (b + 15) // 16 * 16  # noqa: E731
        ngroups = (nrows + 31) // 32
        ids_off, codes_off = self.TPL_TABLE_BYTES, self.TPL_TABLE_BYTES + r16(nrows)
        raw = self.tpl_buf.view(torch.uint8)
        assert raw.numel() == codes_off + r16(ngroups), (raw.numel(), nrows)
        return raw[ids_off:ids_off + nrows], raw[codes_off:codes_off + ngroups]

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            try:
                L.b2s_spmv_plan_destroy(h)
            except Exception:
                pass


def _plan_handle(plan):
    return None if plan is None else plan.handle


def spmv_plan(indptr: torch.Tensor, indices: torch.Tensor, shape, nnz: int, vdtype, tma_only: bool = False) -> SpmvPlan:
    """Build the SpMV plan for a CSR structure (tile boundaries + kernel choice).  `tma_only`: the plan must use the
    TMA tile kernel (needed by spmv_add / spmv_fused).  When the library reports that the structure qualifies (short
    rows, every tile's columns within 65536 of each other) the plan is packed: its launches stream uint16 columns and
    row offsets instead of `indices` / `indptr`, so the plan is only valid while those arrays are unchanged.  See
    spmv_plan_code for coding the values as well."""
    _chk_dev(indptr, indices)
    vt = vt_code(vdtype)
    nrows, ncols = shape
    nbytes = int(L.b2s_spmv_plan_bytes(vt, nrows, nnz))
    buf = torch.empty(max(nbytes, 16) // 4, dtype=torch.int32, device=indptr.device)
    out = _lib.c_vp()
    _lib.check(L.b2s_spmv_plan_create_ex(vt, idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols, nnz,
                                         ptr(indptr), ptr(indices), ptr(buf), _stream(), ctypes.byref(out),
                                         1 if tma_only else 0), "b2s_spmv_plan_create")
    handle = int(out.value)
    pack_buf = None
    pbytes = int(L.b2s_spmv_plan_pack_bytes(handle))
    if pbytes > 0:
        pack_buf = torch.empty(pbytes // 4, dtype=torch.int32, device=indptr.device)
        rc = L.b2s_spmv_plan_pack(handle, ptr(indptr), ptr(indices), ptr(pack_buf), _stream())
        if rc != _lib.OK:
            L.b2s_spmv_plan_destroy(handle)
            _lib.check(rc, "b2s_spmv_plan_pack")
    plan = SpmvPlan(handle, buf, pack_buf)
    plan.nnz = nnz
    return plan


def spmv_plan_code(plan: SpmvPlan, indptr: torch.Tensor, indices: torch.Tensor, data: torch.Tensor) -> SpmvPlan:
    """Code the values of a packed plan that no launch has used yet: when `data` holds at most 16 distinct values (bit
    patterns) and every tile's column window leaves room for their codes in the uint16 column words, the pack buffer
    is rewritten with the codes, and launches with this `data` stream no values at all -- so the plan is then also only
    valid while `data` is unchanged.  Otherwise the plan stays packed with streamed values.  A plan without a pack
    buffer is returned as it is."""
    if getattr(plan, "pack_buf", None) is None:
        return plan
    _chk_dev(data)
    assert data.is_contiguous() and data.shape[0] == plan.nnz
    _lib.check(L.b2s_spmv_plan_pack_coded(plan.handle, ptr(indptr), ptr(indices), ptr(data), ptr(plan.pack_buf),
                                          _stream()), "b2s_spmv_plan_pack_coded")
    plan._info()
    return plan


def spmv_plan_templates(plan: SpmvPlan, indptr: torch.Tensor, indices: torch.Tensor, data: torch.Tensor) -> SpmvPlan:
    """Give a plan that no launch has used yet row templates when the matrix qualifies (rows of at most 8 entries, at
    most 32 distinct (length, column - row, value bits) signatures -- structured-grid stencils): whole-matrix products
    with this `data` then read one uint8 code per 32-row group (and the per-row ids of groups that mix templates)
    instead of the matrix, so the plan is also only valid while `data` is unchanged.  Otherwise, or for a plan that cannot use them, the plan is returned as it was."""
    if getattr(plan, "handle", None) is None:
        return plan
    nbytes = int(L.b2s_spmv_plan_templates_bytes(plan.handle))
    if nbytes <= 0:
        return plan
    _chk_dev(data)
    assert data.is_contiguous() and data.shape[0] == plan.nnz
    buf = torch.empty(nbytes // 4, dtype=torch.int32, device=indptr.device)
    _lib.check(L.b2s_spmv_plan_templates(plan.handle, ptr(indptr), ptr(indices), ptr(data), ptr(buf), _stream()),
               "b2s_spmv_plan_templates")
    plan._info()
    if plan.ntemplates:
        plan.tpl_buf = buf
    return plan


def spmv(indptr, indices, data, x, y, shape, plan=None):
    """y = A @ x (replaces task CSR_SPMV_ROW_SPLIT, sparse/csr.py:928-968)."""
    _chk_dev(indptr, indices, data, x, y)
    nrows, ncols = shape
    nnz = data.shape[0]
    assert x.dtype == data.dtype == y.dtype and x.is_contiguous() and y.is_contiguous()
    assert x.shape[0] == ncols and y.shape[0] == nrows
    _lib.check(L.b2s_spmv_csr(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                              nnz, ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y), _plan_handle(plan), _stream()),
               "b2s_spmv_csr")
    return y


def spmm(indptr, indices, data, X, Y, shape):
    """Y = A @ X for row-major dense X (ncols, k), Y (nrows, k) (replaces task SPMM_CSR_DENSE, sparse/csr.py:1151-1205).
    Rows of X / Y may be strided (leading dimension = stride(0)); the k entries of a row must be contiguous."""
    _chk_dev(indptr, indices, data, X, Y)
    nrows, ncols = shape
    assert X.dtype == data.dtype == Y.dtype and X.ndim == 2 and Y.ndim == 2
    k = X.shape[1]
    assert X.shape[0] == ncols and tuple(Y.shape) == (nrows, k)
    assert k <= 1 or (X.stride(1) == 1 and Y.stride(1) == 1)
    ldx = X.stride(0) if X.shape[0] > 1 else max(k, 1)
    ldy = Y.stride(0) if Y.shape[0] > 1 else max(k, 1)
    _lib.check(L.b2s_spmm_csr(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                              data.shape[0], k, ptr(indptr), ptr(indices), ptr(data), ptr(X), ldx, ptr(Y), ldy,
                              _stream()), "b2s_spmm_csr")
    return Y


def spmv_csc(indptr, indices, data, x, y, shape):
    """y = A @ x for a CSC matrix A of `shape` (indptr over columns, indices = rows) through b2s_spmv_csc (replaces task
    CSC_SPMV, sparse/csc.py:523-553).  y is overwritten; the launch neither syncs nor allocates."""
    _chk_dev(indptr, indices, data, x, y)
    nrows, ncols = shape
    assert x.dtype == data.dtype == y.dtype and x.is_contiguous() and y.is_contiguous()
    assert x.shape[0] == ncols and y.shape[0] == nrows and indptr.shape[0] == ncols + 1
    _lib.check(L.b2s_spmv_csc(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                              int(data.shape[0]), ptr(indptr), ptr(indices.contiguous()), ptr(data.contiguous()), ptr(x),
                              ptr(y), _stream()), "b2s_spmv_csc")
    return y


def spmm_csc(indptr, indices, data, X, Y, shape):
    """Y = A @ X for a CSC matrix A and row-major dense X (ncols, k), Y (nrows, k) through b2s_spmm_csc (replaces task
    CSC_SPMM, sparse/csc.py:630-680).  Rows of X / Y may be strided; the k entries of a row must be contiguous."""
    _chk_dev(indptr, indices, data, X, Y)
    nrows, ncols = shape
    assert X.dtype == data.dtype == Y.dtype and X.ndim == 2 and Y.ndim == 2
    k = X.shape[1]
    assert X.shape[0] == ncols and tuple(Y.shape) == (nrows, k) and indptr.shape[0] == ncols + 1
    assert k <= 1 or ((ncols == 0 or X.stride(1) == 1) and (nrows == 0 or Y.stride(1) == 1))
    ldx = X.stride(0) if X.shape[0] > 1 else max(k, 1)
    ldy = Y.stride(0) if Y.shape[0] > 1 else max(k, 1)
    _lib.check(L.b2s_spmm_csc(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                              int(data.shape[0]), k, ptr(indptr), ptr(indices.contiguous()), ptr(data.contiguous()),
                              ptr(X), ldx, ptr(Y), ldy, _stream()), "b2s_spmm_csc")
    return Y


def spmv_dia(offsets, data, x, y, shape):
    """y = A @ x for a DIA matrix A of `shape` (int64 device `offsets`, contiguous `data` of ndiag x L) through
    b2s_spmv_dia.  y is overwritten; the launch neither syncs nor allocates."""
    _chk_dev(offsets, data, x, y)
    nrows, ncols = shape
    assert x.dtype == data.dtype == y.dtype and x.is_contiguous() and y.is_contiguous() and data.is_contiguous()
    assert offsets.dtype == torch.int64 and data.ndim == 2 and offsets.shape[0] == data.shape[0]
    assert x.shape[0] == ncols and y.shape[0] == nrows
    ndiag, Ld = data.shape
    _lib.check(L.b2s_spmv_dia(vt_code(data.dtype), nrows, ncols, ndiag, Ld, ptr(offsets), ptr(data), ptr(x), ptr(y),
                              _stream()), "b2s_spmv_dia")
    return y


def spmm_dia(offsets, data, X, Y, shape):
    """Y = A @ X for a DIA matrix A and row-major dense X (ncols, k), Y (nrows, k) through b2s_spmm_dia.  Rows of X / Y
    may be strided; the k entries of a row must be contiguous."""
    _chk_dev(offsets, data, X, Y)
    nrows, ncols = shape
    assert X.dtype == data.dtype == Y.dtype and X.ndim == 2 and Y.ndim == 2 and data.is_contiguous()
    assert offsets.dtype == torch.int64 and data.ndim == 2 and offsets.shape[0] == data.shape[0]
    k = X.shape[1]
    assert X.shape[0] == ncols and tuple(Y.shape) == (nrows, k)
    assert k <= 1 or ((ncols == 0 or X.stride(1) == 1) and (nrows == 0 or Y.stride(1) == 1))
    ldx = X.stride(0) if X.shape[0] > 1 else max(k, 1)
    ldy = Y.stride(0) if Y.shape[0] > 1 else max(k, 1)
    ndiag, Ld = data.shape
    _lib.check(L.b2s_spmm_dia(vt_code(data.dtype), nrows, ncols, ndiag, Ld, k, ptr(offsets), ptr(data), ptr(X), ldx,
                              ptr(Y), ldy, _stream()), "b2s_spmm_dia")
    return Y


def dia_to_csr(offsets, order, data, shape, ptr_dtype, idx_dtype):
    """CSR arrays (indptr, indices, vals) of a DIA matrix through b2s_dia_to_csr: in-band entries with data != 0, each
    row's columns ascending (`order` sorts `offsets`).  Reads the nnz back to allocate the result."""
    _chk_dev(offsets, order, data)
    nrows, ncols = shape
    ndiag, Ld = data.shape
    dev = data.device
    vt, it, pt = vt_code(data.dtype), idx_code(idx_dtype), idx_code(ptr_dtype)
    indptr = torch.empty(nrows + 1, dtype=ptr_dtype, device=dev)
    scratch = torch.empty(max(int(L.b2s_dia_scratch_bytes(nrows, ncols)), 1), dtype=torch.uint8, device=dev)
    nnz = _lib.c_i64(0)
    args = (vt, it, pt, nrows, ncols, ndiag, Ld, ptr(offsets), ptr(order), ptr(data))
    _lib.check(L.b2s_dia_to_csr(*args, 0, ptr(indptr), None, None, ptr(scratch), scratch.numel(), ctypes.byref(nnz),
                                _stream()), "b2s_dia_to_csr")
    indices = torch.empty(nnz.value, dtype=idx_dtype, device=dev)
    vals = torch.empty(nnz.value, dtype=data.dtype, device=dev)
    if nnz.value:
            _lib.check(L.b2s_dia_to_csr(*args, nnz.value, ptr(indptr), ptr(indices), ptr(vals), None, 0, None, _stream()),
                   "b2s_dia_to_csr")
    return indptr, indices, vals


def csr_to_dia(indptr, indices, data, shape, allocate):
    """(offsets, data) of the DIA form of a CSR matrix with no repeated (row, column) through b2s_csr_to_dia.  The
    diagonal count and L = largest column + 1 are read back and passed to `allocate(ndiag, L)`, which may raise before
    anything of that size is allocated; it returns nothing."""
    _chk_dev(indptr, indices, data)
    nrows, ncols = shape
    nnz = int(data.shape[0])
    dev = data.device
    vt, it, pt = vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype)
    scratch = torch.empty(max(int(L.b2s_dia_scratch_bytes(nrows, ncols)), 1), dtype=torch.uint8, device=dev)
    got = (_lib.c_i64 * 2)()
    args = (vt, it, pt, nrows, ncols, nnz, ptr(indptr), ptr(indices), ptr(data))
    _lib.check(L.b2s_csr_to_dia(*args, 0, 0, None, None, ptr(scratch), scratch.numel(), got, _stream()),
               "b2s_csr_to_dia")
    ndiag, Ld = int(got[0]), int(got[1])
    allocate(ndiag, Ld)
    offsets = torch.empty(ndiag, dtype=torch.int64, device=dev)
    out = torch.empty((ndiag, Ld), dtype=data.dtype, device=dev)
    if ndiag:
            _lib.check(L.b2s_csr_to_dia(*args, ndiag, Ld, ptr(offsets), ptr(out), ptr(scratch), scratch.numel(), None,
                                    _stream()), "b2s_csr_to_dia")
    return offsets, out


def spmv_tiles(indptr, indices, data, x, y, shape, plan, tile_lo: int, tile_hi: int):
    """Rows of tiles [tile_lo, tile_hi) of y = A @ x (x must be valid on that chunk's column window)."""
    _chk_dev(indptr, indices, data, x, y)
    nrows, ncols = shape
    _lib.check(L.b2s_spmv_csr_tiles(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                                    data.shape[0], ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y),
                                    _plan_handle(plan), tile_lo, tile_hi, _stream()), "b2s_spmv_csr_tiles")
    return y


def spmv_host(indptr, indices, data, x_host_ptr: int, y_host_ptr: int, x_dev, y_dev, shape, plan):
    """y_host = A @ x_host through the pipelined C entry point (returns when y_host is complete)."""
    _chk_dev(indptr, indices, data, x_dev, y_dev)
    nrows, ncols = shape
    _lib.check(L.b2s_spmv_csr_host(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                                   data.shape[0], ptr(indptr), ptr(indices), ptr(data), x_host_ptr, y_host_ptr,
                                   ptr(x_dev), ptr(y_dev), _plan_handle(plan), _stream()), "b2s_spmv_csr_host")


def spmv_dot(indptr, indices, data, x, y, w, out, shape, plan):
    """y = A @ x and out[0] = w . y in one launch."""
    _chk_dev(indptr, indices, data, x, y, w, out)
    nrows, ncols = shape
    nnz = data.shape[0]
    assert x.dtype == data.dtype == y.dtype == w.dtype == out.dtype
    assert w.shape[0] == nrows and w.is_contiguous()
    ws = runtime.workspace()
    _lib.check(L.b2s_spmv_csr_dot(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows,
                                  ncols, nnz, ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y), ptr(w),
                                  ptr(out), _plan_handle(plan), ptr(ws), _stream()), "b2s_spmv_csr_dot")
    return y


# ---- CG vector kernels --------------------------------------------------------------------------------
def axpby(y, x, a, b, isalpha=True, negate=False):
    _chk_dev(y, x, a, b)
    assert y.dtype == x.dtype == a.dtype == b.dtype and y.shape == x.shape
    assert y.is_contiguous() and x.is_contiguous()
    _lib.check(L.b2s_axpby(vt_code(y.dtype), y.numel(), ptr(y), ptr(x), ptr(a), ptr(b), int(bool(isalpha)),
                           int(bool(negate)), _stream()), "b2s_axpby")
    return y


def dot(x, y, out=None):
    _chk_dev(x, y)
    assert x.dtype == y.dtype and x.shape == y.shape and x.is_contiguous() and y.is_contiguous()
    if out is None:
        out = torch.empty(1, dtype=x.dtype, device=x.device)
    _lib.check(L.b2s_dot(vt_code(x.dtype), x.numel(), ptr(x), ptr(y), ptr(out), ptr(runtime.workspace()), _stream()),
               "b2s_dot")
    return out


def nrm2(x, out=None):
    _chk_dev(x)
    assert x.is_contiguous()
    if out is None:
        out = torch.empty(1, dtype=x.dtype, device=x.device)
    _lib.check(L.b2s_nrm2(vt_code(x.dtype), x.numel(), ptr(x), ptr(out), ptr(runtime.workspace()), _stream()),
               "b2s_nrm2")
    return out


def cg_update_xr(x, r, p, q, rho, pq, rr_out):
    _chk_dev(x, r, p, q, rho, pq, rr_out)
    assert x.dtype == r.dtype == p.dtype == q.dtype == rho.dtype == pq.dtype == rr_out.dtype
    _lib.check(L.b2s_cg_update_xr(vt_code(x.dtype), x.numel(), ptr(x), ptr(r), ptr(p), ptr(q), ptr(rho), ptr(pq),
                                  ptr(rr_out), ptr(runtime.workspace()), _stream()), "b2s_cg_update_xr")
    return rr_out


def csr_diagonal(indptr, indices, data, nrows: int):
    _chk_dev(indptr, indices, data)
    out = torch.empty(nrows, dtype=data.dtype, device=data.device)
    _lib.check(L.b2s_csr_diagonal(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows,
                                  ptr(indptr), ptr(indices), ptr(data), ptr(out), _stream()), "b2s_csr_diagonal")
    return out


def copy(dst, src_ptr: int, n: int):
    """dst[:n] = *(src_ptr) -- src may be a peer-mapped (IPC) pointer."""
    _chk_dev(dst)
    _lib.check(L.b2s_copy(vt_code(dst.dtype), n, ptr(dst), src_ptr, _stream()), "b2s_copy")
    return dst


# ---- SpGEMM --------------------------------------------------------------------------------------------
def spgemm(a_indptr, a_indices, a_data, b_indptr, b_indices, b_data, shape_a, shape_b):
    """C = A @ B (replaces SPGEMM_CSR_CSR_CSR_GPU + scan_local_results_and_scale_pos,
    sparse/csr.py:1322-1389, 827-859). Returns (c_indptr int64, c_indices int32, c_data, info)."""
    _chk_dev(a_indptr, a_indices, a_data, b_indptr, b_indices, b_data)
    m, k = shape_a
    k2, n = shape_b
    assert k == k2
    assert a_indices.dtype == torch.int32 and b_indices.dtype == torch.int32, "SpGEMM needs int32 column indices"
    assert a_indptr.dtype == b_indptr.dtype and a_data.dtype == b_data.dtype
    dev = a_data.device
    pt = idx_code(a_indptr.dtype)
    vt = vt_code(a_data.dtype)
    st = _stream()
    scratch = torch.empty(int(L.b2s_spgemm_scratch_bytes(m, n)), dtype=torch.uint8, device=dev)
    c_indptr = torch.empty(m + 1, dtype=torch.int64, device=dev)
    info = (_lib.c_i64 * 3)()
    _lib.check(L.b2s_spgemm_csr_symbolic(pt, m, k, n, ptr(a_indptr), ptr(a_indices), ptr(b_indptr), ptr(b_indices),
                                         ptr(c_indptr), info, ptr(scratch), st), "b2s_spgemm_csr_symbolic")
    nnz, products, dense_rows = int(info[0]), int(info[1]), int(info[2])
    c_indices = torch.empty(nnz, dtype=torch.int32, device=dev)
    c_data = torch.empty(nnz, dtype=a_data.dtype, device=dev)
    dense_bytes = int(L.b2s_spgemm_dense_bytes(vt, n, dense_rows))
    dense = torch.empty(dense_bytes, dtype=torch.uint8, device=dev) if dense_bytes else None
    _lib.check(L.b2s_spgemm_csr_numeric(vt, pt, m, k, n, ptr(a_indptr), ptr(a_indices), ptr(a_data), ptr(b_indptr),
                                        ptr(b_indices), ptr(b_data), ptr(c_indptr), ptr(c_indices), ptr(c_data),
                                        ptr(scratch), ptr(dense), dense_bytes, st), "b2s_spgemm_csr_numeric")
    return c_indptr, c_indices, c_data, {"nnz": nnz, "products": products, "dense_rows": dense_rows}


# ---- assembly -------------------------------------------------------------------------------------------------
def coo_to_csr(rows, cols, vals, nrows: int, ptr_dtype, idx_dtype):
    """COO triplets (device tensors) -> canonical CSR arrays (indptr, indices, vals) through b2s_coo_to_csr."""
    _chk_dev(rows, cols, vals)
    nnz = int(vals.shape[0])
    rows, cols = rows.to(idx_dtype).contiguous(), cols.to(idx_dtype).contiguous()
    vals = vals.contiguous()
    dev = vals.device
    indptr = torch.empty(nrows + 1, dtype=ptr_dtype, device=dev)
    indices = torch.empty(nnz, dtype=idx_dtype, device=dev)
    out_vals = torch.empty(nnz, dtype=vals.dtype, device=dev)
    pt = idx_code(ptr_dtype)
    scratch = torch.empty(int(L.b2s_convert_scratch_bytes(nrows, pt)), dtype=torch.uint8, device=dev)
    bad = _lib.c_i64(0)
    _lib.check(L.b2s_coo_to_csr(vt_code(vals.dtype), idx_code(idx_dtype), pt, nrows, nnz, ptr(rows), ptr(cols), ptr(vals),
                                ptr(indptr), ptr(indices), ptr(out_vals), ptr(scratch), ctypes.byref(bad), _stream()),
               "b2s_coo_to_csr")
    if bad.value:
        raise ValueError(f"{bad.value} triplets have a row index outside [0, {nrows})")
    return indptr, indices, out_vals


def csr_transpose(indptr, indices, data, shape):
    """CSR arrays of the transpose (same index widths) through b2s_csr_transpose."""
    _chk_dev(indptr, indices, data)
    nrows, ncols = shape
    nnz = int(data.shape[0])
    dev = data.device
    t_indptr = torch.empty(ncols + 1, dtype=indptr.dtype, device=dev)
    t_indices = torch.empty(nnz, dtype=indices.dtype, device=dev)
    t_vals = torch.empty(nnz, dtype=data.dtype, device=dev)
    pt = idx_code(indptr.dtype)
    scratch = torch.empty(int(L.b2s_convert_scratch_bytes(ncols, pt)), dtype=torch.uint8, device=dev)
    _lib.check(L.b2s_csr_transpose(vt_code(data.dtype), idx_code(indices.dtype), pt, nrows, ncols, nnz, ptr(indptr),
                                   ptr(indices.contiguous()), ptr(data.contiguous()), ptr(t_indptr), ptr(t_indices),
                                   ptr(t_vals), ptr(scratch), _stream()), "b2s_csr_transpose")
    return t_indptr, t_indices, t_vals


def csr_sort_rows(indptr, indices, data):
    """Sort every row of (indptr, indices, data) by column IN PLACE through b2s_csr_sort_rows; returns (indices, data)."""
    _chk_dev(indptr, indices, data)
    assert indices.is_contiguous() and data.is_contiguous()
    nrows = indptr.shape[0] - 1
    pt = idx_code(indptr.dtype)
    scratch = torch.empty(int(L.b2s_convert_scratch_bytes(nrows, pt)), dtype=torch.uint8, device=data.device)
    _lib.check(L.b2s_csr_sort_rows(vt_code(data.dtype), idx_code(indices.dtype), pt, nrows, int(data.shape[0]),
                                   ptr(indptr), ptr(indices), ptr(data), ptr(scratch), _stream()), "b2s_csr_sort_rows")
    return indices, data


# ---- elementwise ------------------------------------------------------------------------------------------------
EW_OPS = {"add": 0, "sub": 1, "mul": 2}       # B2S_EW_ADD / _SUB / _MUL
SCALE_MODES = {"rows": 0, "cols": 1, "dense": 2}   # B2S_SCALE_ROWS / _COLS / _DENSE


def csr_binop(op: str, a_indptr, a_indices, a_data, b_indptr, b_indices, b_data, shape):
    """C = A op B for two CSR matrices of one shape (op: "add" / "sub" / "mul") through the two passes of
    b2s_csr_binop_symbolic / _numeric (replaces the reference's add(), sparse/csr.py:972-1030, and mult(), :1033-1099).
    Returns (c_indptr int64, c_indices, c_data, info), info = {nnz, a_unsorted, b_unsorted}.  When a row of A or B has
    decreasing columns the numeric pass does not run and c_indices / c_data are None."""
    _chk_dev(a_indptr, a_indices, a_data, b_indptr, b_indices, b_data)
    assert a_indptr.dtype == b_indptr.dtype and a_indices.dtype == b_indices.dtype and a_data.dtype == b_data.dtype
    a_indices, a_data, b_indices, b_data = (t.contiguous() for t in (a_indices, a_data, b_indices, b_data))
    m, n = shape
    dev = a_data.device
    it, pt = idx_code(a_indices.dtype), idx_code(a_indptr.dtype)
    st = _stream()
    code = EW_OPS[op]
    scratch = torch.empty(int(L.b2s_csr_binop_scratch_bytes(m)), dtype=torch.uint8, device=dev)
    c_indptr = torch.empty(m + 1, dtype=torch.int64, device=dev)
    out = (_lib.c_i64 * 3)()
    _lib.check(L.b2s_csr_binop_symbolic(code, it, pt, m, n, ptr(a_indptr), ptr(a_indices), ptr(b_indptr),
                                        ptr(b_indices), ptr(c_indptr), out, ptr(scratch), st), "b2s_csr_binop_symbolic")
    info = {"nnz": int(out[0]), "a_unsorted": bool(out[1]), "b_unsorted": bool(out[2])}
    if info["a_unsorted"] or info["b_unsorted"]:
        return c_indptr, None, None, info
    c_indices = torch.empty(info["nnz"], dtype=a_indices.dtype, device=dev)
    c_data = torch.empty(info["nnz"], dtype=a_data.dtype, device=dev)
    _lib.check(L.b2s_csr_binop_numeric(code, vt_code(a_data.dtype), it, pt, m, n, ptr(a_indptr), ptr(a_indices),
                                       ptr(a_data), ptr(b_indptr), ptr(b_indices), ptr(b_data), ptr(c_indptr),
                                       ptr(c_indices), ptr(c_data), ptr(scratch), st), "b2s_csr_binop_numeric")
    return c_indptr, c_indices, c_data, info


def csr_scale(indptr, indices, data, d, mode: str, shape):
    """New values data[p] * D with A's structure through b2s_csr_scale; D (contiguous, data's dtype) holds one factor per
    row (mode "rows"), per column ("cols") or is the row-major dense (m, n) operand ("dense")."""
    _chk_dev(indptr, indices, data, d)
    assert d.dtype == data.dtype and d.is_contiguous()
    m, n = shape
    out = torch.empty_like(data)
    _lib.check(L.b2s_csr_scale(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), m, n,
                               int(data.shape[0]), SCALE_MODES[mode], ptr(indptr), ptr(indices.contiguous()),
                               ptr(data.contiguous()), ptr(d), n, ptr(out), _stream()), "b2s_csr_scale")
    return out


def sddmm(indptr, indices, data, C, Dt, out=None):
    """out[p] = data[p] * dot(C[i], Dt[j]) for every stored entry p = (i, j) through b2s_sddmm_csr (replaces task
    CSR_SDDMM, sparse/csr.py:1243-1314).  C is (nrows, k), Dt is D transposed, (ncols, k); rows of either may be strided,
    the k entries of a row must be contiguous.  `out` (data's shape and dtype) may be preallocated, e.g. for graph
    capture; the launch neither syncs nor allocates."""
    _chk_dev(indptr, indices, data, C, Dt, out)
    nrows, k = C.shape
    ncols = Dt.shape[0]
    assert C.dtype == Dt.dtype == data.dtype and C.ndim == 2 and Dt.ndim == 2 and Dt.shape[1] == k
    assert indptr.shape[0] == nrows + 1
    assert k <= 1 or ((nrows == 0 or C.stride(1) == 1) and (ncols == 0 or Dt.stride(1) == 1))
    ldc = C.stride(0) if nrows > 1 else max(k, 1)
    ldd = Dt.stride(0) if ncols > 1 else max(k, 1)
    if out is None:
        out = torch.empty(data.shape, dtype=data.dtype, device=data.device)
    assert out.dtype == data.dtype and out.shape == data.shape and out.is_contiguous()
    _lib.check(L.b2s_sddmm_csr(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                               int(data.shape[0]), k, ptr(indptr), ptr(indices.contiguous()), ptr(data.contiguous()),
                               ptr(C), ldc, ptr(Dt), ldd, ptr(out), _stream()), "b2s_sddmm_csr")
    return out


def tropical_spmv(indptr, indices, x, y=None):
    """y[i] = lexicographic max of 0 and x[j] over the stored entries (i, j) through b2s_tropical_spmv_csr (replaces
    task CSR_SPMV_ROW_SPLIT_TROPICAL_SEMIRING, sparse/csr.py:365-424).  x is (ncols, F) int64 and y (nrows, F) int64;
    rows of either may be strided, the F fields of a row must be contiguous, and y must not overlap x.  `y` may be
    preallocated, e.g. for graph capture; the launch neither syncs nor allocates."""
    _chk_dev(indptr, indices, x, y)
    nrows = indptr.shape[0] - 1
    ncols, nf = x.shape
    assert x.dtype == torch.int64 and (nf <= 1 or ncols == 0 or x.stride(1) == 1)
    if y is None:
        y = torch.empty((nrows, nf), dtype=torch.int64, device=x.device)
    assert y.dtype == torch.int64 and tuple(y.shape) == (nrows, nf) and (nf <= 1 or nrows == 0 or y.stride(1) == 1)
    ldx = x.stride(0) if ncols > 1 else max(nf, 1)
    ldy = y.stride(0) if nrows > 1 else max(nf, 1)
    _lib.check(L.b2s_tropical_spmv_csr(idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                                       int(indices.shape[0]), nf, ptr(indptr), ptr(indices.contiguous()), ptr(x), ldx,
                                       ptr(y), ldy, _stream()), "b2s_tropical_spmv_csr")
    return y


REDUCE_OPS = {"sum": 0, "max": 1, "min": 2, "argmax": 3, "argmin": 4, "count_nonzero": 5}   # B2S_REDUCE_*


def csr_reduce_rows(op: str, indptr, indices, data, ncols: int, explicit: bool = False, out=None):
    """out[i] = reduction `op` over row i through b2s_csr_reduce_rows (op: "sum", "max", "min", "argmax", "argmin",
    "count_nonzero"; see include/b200sparse.h for the implicit-zero, NaN and input rules).  `out` is data's dtype for
    sum / max / min and int64 otherwise; it may be preallocated, e.g. for graph capture: the launch neither syncs nor
    allocates.  `indices` may be None except for argmax / argmin."""
    _chk_dev(indptr, indices, data, out)
    code = REDUCE_OPS[op]
    nrows = indptr.shape[0] - 1
    odt = data.dtype if op in ("sum", "max", "min") else torch.int64
    if out is None:
        out = torch.empty(nrows, dtype=odt, device=data.device)
    assert out.dtype == odt and tuple(out.shape) == (nrows,) and out.is_contiguous()
    assert indptr.is_contiguous()
    it = idx_code(indices.dtype) if indices is not None else _lib.I32
    _lib.check(L.b2s_csr_reduce_rows(code, vt_code(data.dtype), it, idx_code(indptr.dtype), nrows, int(ncols),
                                     int(data.shape[0]), ptr(indptr),
                                     ptr(indices.contiguous()) if indices is not None else None,
                                     ptr(data.contiguous()), int(bool(explicit)), ptr(out), _stream()),
               "b2s_csr_reduce_rows")
    return out


def csr_column_map(cols, ncols: int):
    """The column map of a column selection through b2s_coo_to_csr: (col_ptr, col_pos, bad), an int64 CSR matrix from
    source column to the output positions (ascending) that request it, and the number of requested columns outside
    [-ncols, ncols).  `cols` is an int64 device tensor; negative entries count from the end.  Syncs once."""
    _chk_dev(cols)
    k = int(cols.shape[0])
    dev = cols.device
    cols = torch.where(cols < 0, cols + ncols, cols).contiguous()
    pos = torch.arange(k, dtype=torch.int64, device=dev)
    dummy = torch.zeros(k, dtype=torch.float32, device=dev)      # b2s_coo_to_csr moves values; these are not read back
    col_ptr = torch.empty(ncols + 1, dtype=torch.int64, device=dev)
    col_pos = torch.empty(k, dtype=torch.int64, device=dev)
    out_vals = torch.empty(k, dtype=torch.float32, device=dev)
    scratch = torch.empty(int(L.b2s_convert_scratch_bytes(ncols, _lib.I64)), dtype=torch.uint8, device=dev)
    bad = _lib.c_i64(0)
    _lib.check(L.b2s_coo_to_csr(_lib.F32, _lib.I64, _lib.I64, ncols, k, ptr(cols), ptr(pos), ptr(dummy), ptr(col_ptr),
                                ptr(col_pos), ptr(out_vals), ptr(scratch), ctypes.byref(bad), _stream()),
               "b2s_coo_to_csr")
    return col_ptr, col_pos, int(bad.value)


def csr_select(indptr, indices, data, shape, nrows_out: int, rows=None, row_start: int = 0, row_step: int = 1,
               col_map=None, ncols_out=None, out_index_dtype=torch.int32):
    """Rows and columns of a CSR matrix through the two passes of b2s_csr_select.  Output row t is source row rows[t]
    (an int64 device tensor; negatives count from the end) or row_start + t * row_step; col_map = (col_ptr, col_pos) of
    `csr_column_map`, or None for every column.  Returns (indptr int64, indices of out_index_dtype, data, bad): with
    bad > 0 row indices outside the matrix, indices and data are None.  Syncs once."""
    _chk_dev(indptr, indices, data, rows)
    nrows, ncols = shape
    dev = data.device
    indices, data = indices.contiguous(), data.contiguous()
    col_ptr, col_pos = col_map if col_map is not None else (None, None)
    if col_map is None:
        ncols_out = ncols
    if rows is not None:
        rows = rows.contiguous()
    vw = data.element_size()
    it, pt, ot = idx_code(indices.dtype), idx_code(indptr.dtype), idx_code(out_index_dtype)
    st = _stream()
    scratch = torch.empty(int(L.b2s_csr_select_scratch_bytes(nrows_out)), dtype=torch.uint8, device=dev)
    out_ptr = torch.empty(nrows_out + 1, dtype=torch.int64, device=dev)
    info = (_lib.c_i64 * 4)()
    args = (nrows, ncols, int(data.shape[0]), ptr(indptr), ptr(indices), ptr(data), nrows_out, ptr(rows), row_start,
            row_step, ptr(col_ptr), ptr(col_pos), ncols_out, ptr(out_ptr))
    _lib.check(L.b2s_csr_select(0, vw, it, pt, ot, *args, None, None, 0, ptr(scratch), info, st), "b2s_csr_select")
    nnz_out, bad = int(info[0]), int(info[1])
    if bad:
        return out_ptr, None, None, bad
    out_idx = torch.empty(nnz_out, dtype=out_index_dtype, device=dev)
    out_val = torch.empty(nnz_out, dtype=data.dtype, device=dev)
    _lib.check(L.b2s_csr_select(1, vw, it, pt, ot, *args, ptr(out_idx), ptr(out_val), nnz_out, ptr(scratch), None, st),
               "b2s_csr_select")
    return out_ptr, out_idx, out_val, 0


def csr_lookup(indptr, indices, data, shape, ri, ci):
    """out[w] = A[ri[w], ci[w]] (int64 device tensors; negatives count from the end) through b2s_csr_lookup: the sum of
    the stored entries there in stored order, or 0.  Returns (out, bad) with bad a one-element int64 device tensor
    counting the pairs outside the matrix; nothing syncs."""
    _chk_dev(indptr, indices, data, ri, ci)
    nrows, ncols = shape
    k = int(ri.shape[0])
    ri, ci, indices, data = ri.contiguous(), ci.contiguous(), indices.contiguous(), data.contiguous()
    out = torch.empty(k, dtype=data.dtype, device=data.device)
    bad = torch.zeros(1, dtype=torch.int64, device=data.device)
    _lib.check(L.b2s_csr_lookup(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                                int(data.shape[0]), ptr(indptr), ptr(indices), ptr(data), k, ptr(ri), ptr(ci), ptr(out),
                                ptr(bad), _stream()),
               "b2s_csr_lookup")
    return out, bad


def csr_kron(a_indptr, a_indices, a_data, a_shape, b_indptr, b_indices, b_data, b_shape, out_index_dtype):
    """kron(A, B) through b2s_csr_kron: (indptr int64, indices of out_index_dtype, data).  Each operand is read in its
    own index widths; A and B share a value dtype (float32 / float64).  Nothing syncs."""
    _chk_dev(a_indptr, a_indices, a_data, b_indptr, b_indices, b_data)
    assert a_data.dtype == b_data.dtype
    (am, an), (bm, bn) = a_shape, b_shape
    a_indices, a_data, b_indices, b_data = (t.contiguous() for t in (a_indices, a_data, b_indices, b_data))
    annz, bnnz = int(a_data.shape[0]), int(b_data.shape[0])
    dev = a_data.device
    out_ptr = torch.empty(am * bm + 1, dtype=torch.int64, device=dev)
    out_idx = torch.empty(annz * bnnz, dtype=out_index_dtype, device=dev)
    out_val = torch.empty(annz * bnnz, dtype=a_data.dtype, device=dev)
    _lib.check(L.b2s_csr_kron(vt_code(a_data.dtype), idx_code(out_index_dtype), idx_code(a_indices.dtype),
                              idx_code(a_indptr.dtype), am, an, annz, ptr(a_indptr), ptr(a_indices), ptr(a_data),
                              idx_code(b_indices.dtype), idx_code(b_indptr.dtype), bm, bn, bnnz, ptr(b_indptr),
                              ptr(b_indices), ptr(b_data), ptr(out_ptr), ptr(out_idx), ptr(out_val), _stream()),
               "b2s_csr_kron")
    return out_ptr, out_idx, out_val


def csr_blocks(blocks, shape, nnz: int, dtype, out_index_dtype):
    """bmat through b2s_csr_blocks: `blocks` lists (row_block, row_off, col_off, indptr, indices, data, (m, n)) for the
    blocks with stored entries, in block-row order and left to right; their data share `dtype`, of 4, 8 or 16 bytes.
    Returns (indptr int64, indices of out_index_dtype, data).  Uploads the block table; nothing syncs."""
    nrows, ncols = shape
    dev = runtime.device
    table = np.zeros(len(blocks), dtype=_lib.BLOCK_DESC)
    if blocks:
        rb, ro, co, ip, ix, dv, shp = zip(*blocks)
        _chk_dev(*ip, *ix, *dv)
        ix = [t.contiguous() for t in ix]
        dv = [t.contiguous() for t in dv]
        table["indptr"] = [t.data_ptr() for t in ip]
        table["indices"] = [t.data_ptr() for t in ix]
        table["vals"] = [t.data_ptr() for t in dv]
        table["it"] = [idx_code(t.dtype) for t in ix]
        table["pt"] = [idx_code(t.dtype) for t in ip]
        table["nrows"], table["ncols"] = zip(*shp)
        table["nnz"] = [t.shape[0] for t in dv]
        table["row_block"], table["row_off"], table["col_off"] = rb, ro, co
    out_ptr = torch.empty(nrows + 1, dtype=torch.int64, device=dev)
    out_idx = torch.empty(nnz, dtype=out_index_dtype, device=dev)
    out_val = torch.empty(nnz, dtype=dtype, device=dev)
    scratch = torch.empty(int(L.b2s_csr_blocks_scratch_bytes(len(blocks))), dtype=torch.uint8, device=dev)
    _lib.check(L.b2s_csr_blocks(out_val.element_size(), idx_code(out_index_dtype), nrows, ncols, nnz, len(blocks),
                                table.ctypes.data, ptr(out_ptr), ptr(out_idx), ptr(out_val), ptr(scratch), _stream()),
               "b2s_csr_blocks")
    return out_ptr, out_idx, out_val


def random_csr(shape, k: int, seed: int, idx_dtype, ptr_dtype, dtype, data=None):
    """The canonical CSR arrays (indptr, indices, data) of a uniform random k-subset of the m x n positions, and the
    number of sampling rounds, through csrc/random.cu: b2s_random_sample of s = min(k, mn - k) positions,
    b2s_coo_to_csr of them and, when k > mn - k, b2s_random_complement of that zero set.  The values are
    b2s_random_values of `seed` in `dtype` (float32, float64, complex64 or complex128), or `data`, a device tensor of k
    values already in canonical order.  Every buffer is allocated before the first launch, so a sample that does not
    fit raises MemoryError (or torch's out-of-memory error) instead of failing in a kernel.  The sampler syncs once per
    round, the assembly once."""
    m, n = shape
    mn = m * n
    complement = k > mn - k
    s = mn - k if complement else k
    dev = runtime.device
    slots = int(L.b2s_random_table_slots(s))
    sptr_dtype = torch.int64 if complement else ptr_dtype   # the zero set's row pointers feed the complement kernel
    tdt = torch_dtype(dtype)
    isz, psz, vsz = (torch.empty(0, dtype=t).element_size() for t in (idx_dtype, sptr_dtype, tdt))
    need = 8 * slots + 3 * s * isz + (m + 1) * psz + int(L.b2s_convert_scratch_bytes(m, idx_code(sptr_dtype)))
    need += (8 * (m + 1) + k * isz if complement else 0) + (k * vsz if data is None else 0)
    # free device memory plus what torch's caching allocator holds unused, which it hands out before asking CUDA
    free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    if slots == 0 or need > free:
        raise MemoryError(f"a random {m} x {n} matrix with {k} stored entries needs {need} bytes of device memory to "
                          f"sample; {free} are free")
    table = torch.empty(slots, dtype=torch.int64, device=dev)
    rows, cols = (torch.empty(s, dtype=idx_dtype, device=dev) for _ in range(2))
    counters = torch.empty(2, dtype=torch.int64, device=dev)
    sptr = torch.empty(m + 1, dtype=sptr_dtype, device=dev)
    sidx = torch.empty(s, dtype=idx_dtype, device=dev)
    scratch = torch.empty(int(L.b2s_convert_scratch_bytes(m, idx_code(sptr_dtype))), dtype=torch.uint8, device=dev)
    if complement:
        indptr, indices = torch.empty(m + 1, dtype=ptr_dtype, device=dev), torch.empty(k, dtype=idx_dtype, device=dev)
    else:
        indptr, indices = sptr, sidx
    generate = data is None
    if generate:
        data = torch.empty(k, dtype=tdt, device=dev)
    # b2s_coo_to_csr moves a value per triplet; nothing reads them here, so they live in the table, which is no longer
    # needed once the sample is drawn (slots >= 2s: room for two float32 arrays of s)
    moved = table.view(torch.float32)
    it, st = idx_code(idx_dtype), _stream()
    rounds = _lib.c_i64(0)
    _lib.check(L.b2s_random_sample(it, m, n, s, seed, ptr(table), slots, ptr(rows), ptr(cols), ptr(counters),
                                   ctypes.byref(rounds), st), "b2s_random_sample")
    bad = _lib.c_i64(0)
    _lib.check(L.b2s_coo_to_csr(_lib.F32, it, idx_code(sptr_dtype), m, s, ptr(rows), ptr(cols), ptr(moved[:s]),
                                ptr(sptr), ptr(sidx), ptr(moved[s:2 * s]), ptr(scratch), ctypes.byref(bad), st),
               "b2s_coo_to_csr")
    if complement:
        _lib.check(L.b2s_random_complement(it, idx_code(ptr_dtype), m, n, k, ptr(sptr), ptr(sidx), ptr(indptr),
                                           ptr(indices), st), "b2s_random_complement")
    if generate:
        vt = _lib.F32 if tdt in (torch.float32, torch.complex64) else _lib.F64
        _lib.check(L.b2s_random_values(vt, int(tdt.is_complex), k, seed, ptr(data), st), "b2s_random_values")
    return indptr, indices, data, int(rounds.value)


def spgemm_row_work(a_indptr, a_indices, b_indptr) -> torch.Tensor:
    """Products per row of A @ B (int64 device tensor of len m): the chunk planner's measure of work / output size."""
    _chk_dev(a_indptr, a_indices, b_indptr)
    assert a_indices.dtype == torch.int32 and a_indptr.dtype == b_indptr.dtype
    m = a_indptr.shape[0] - 1
    out = torch.empty(max(m, 1), dtype=torch.int64, device=a_indptr.device)
    _lib.check(L.b2s_spgemm_row_work(idx_code(a_indptr.dtype), m, ptr(a_indptr), ptr(a_indices), ptr(b_indptr), ptr(out),
                                     _stream()), "b2s_spgemm_row_work")
    return out[:m]


# ---- CUDA IPC / NVLink peer exchange -----------------------------------------------------------------------
def ipc_alloc(nbytes: int) -> int:
    out = _lib.c_vp()
    _lib.check(L.b2s_ipc_alloc(int(nbytes), ctypes.byref(out)), "b2s_ipc_alloc")
    return int(out.value)


def ipc_free(p: int) -> None:
    _lib.check(L.b2s_ipc_free(p), "b2s_ipc_free")


def ipc_export(p) -> bytes:
    if isinstance(p, torch.Tensor):
        _chk_dev(p)
        p = ptr(p)
    buf = ctypes.create_string_buffer(64)
    _lib.check(L.b2s_ipc_export(p, buf), "b2s_ipc_export")
    return buf.raw


def peer_allreduce(t: torch.Tensor, rank: int, peers) -> torch.Tensor:
    _chk_dev(t)
    n = len(peers)
    arr = (_lib.c_vp * n)(*peers)
    _lib.check(L.b2s_peer_allreduce(vt_code(t.dtype), rank, n, arr, ptr(t), t.numel(), _stream()), "b2s_peer_allreduce")
    return t


def peer_halo_exchange(x_local: torch.Tensor, rank: int, peers, sends, recv_peers) -> None:
    """sends: list of (peer, src_elem_off, dst_elem_off, count)."""
    _chk_dev(x_local)
    n = len(peers)
    arr = (_lib.c_vp * n)(*peers)
    flat = [int(v) for s in sends for v in s]
    desc = (_lib.c_i64 * max(len(flat), 1))(*flat)
    rp = (ctypes.c_int32 * max(len(recv_peers), 1))(*recv_peers)
    _lib.check(L.b2s_peer_halo_exchange(vt_code(x_local.dtype), rank, n, arr, ptr(x_local), len(sends), desc,
                                        len(recv_peers), rp, _stream()), "b2s_peer_halo_exchange")


def peer_push(x_local: torch.Tensor, rank: int, peers, sends, recv_peers, ctas_per_send: int = 8) -> None:
    """Fused-protocol push (no wait kernel): slices of x_local go to the peers' x buffers, `ctas_per_send` CTAs each;
    the arrival flags are consumed inside later `spmv_fused` launches."""
    _chk_dev(x_local)
    n = len(peers)
    arr = (_lib.c_vp * n)(*peers)
    flat = [int(v) for s in sends for v in s]
    desc = (_lib.c_i64 * max(len(flat), 1))(*flat)
    rp = (ctypes.c_int32 * max(len(recv_peers), 1))(*recv_peers)
    _lib.check(L.b2s_peer_push(vt_code(x_local.dtype), rank, n, arr, ptr(x_local), len(sends), desc,
                               len(recv_peers), rp, int(ctas_per_send), _stream()), "b2s_peer_push")


def peer_push_wait(rank: int, peers, recv_peers) -> None:
    """Wait on the current stream for the slices `recv_peers` pushed (b2s_peer_push) in the current exchange."""
    n = len(peers)
    arr = (_lib.c_vp * n)(*peers)
    rp = (ctypes.c_int32 * max(len(recv_peers), 1))(*recv_peers)
    _lib.check(L.b2s_peer_push_wait(rank, n, arr, len(recv_peers), rp, _stream()), "b2s_peer_push_wait")


def fuse_desc(ranges, n_free=None, flags=(), sends=(), acks=(), epoch_ctr=0, ticket=0, epoch_add=1, epoch_bump=1,
              expect=0, error=0, accumulate=False) -> "_lib.FuseDesc":
    """Build a b2s_fuse_desc.  ranges: [(tile_lo, tile_hi)]; flags: local arrival-word addresses;
    sends: [(src_ptr, dst_ptr, count, remote_flag_ptr, local_ack_ptr)]; acks: remote ack-word addresses."""
    d = _lib.FuseDesc()
    ranges = list(ranges)
    d.nranges = len(ranges)
    d.n_free = len(ranges) if n_free is None else int(n_free)
    for i, (lo, hi) in enumerate(ranges):
        d.ranges[2 * i], d.ranges[2 * i + 1] = int(lo), int(hi)
    d.n_flags, d.n_sends, d.n_acks = len(flags), len(sends), len(acks)
    d.accumulate = int(bool(accumulate))
    for i, f in enumerate(flags):
        d.flag[i] = int(f)
    for i, (src, dst, cnt, rflag, lack) in enumerate(sends):
        d.send_src[i], d.send_dst[i], d.send_count[i] = int(src), int(dst), int(cnt)
        d.send_flag[i], d.send_ack[i] = int(rflag), int(lack)
    for i, a in enumerate(acks):
        d.ack_out[i] = int(a)
    d.epoch_ctr = int(epoch_ctr) or None
    d.ticket = int(ticket) or None
    d.epoch_add, d.epoch_bump = int(epoch_add), int(epoch_bump)
    d.expect = int(expect)
    d.error = int(error) or None
    return d


def spmv_fused(indptr, indices, data, x, y, shape, plan, desc, w=None, dot_out=None):
    """y = A @ x (or y += with desc.accumulate) with the x exchange fused into the kernel; optional fused w . y."""
    _chk_dev(indptr, indices, data, x, y, w, dot_out)
    nrows, ncols = shape
    ws = ptr(runtime.workspace()) if w is not None else None
    _lib.check(L.b2s_spmv_csr_fused(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                                    data.shape[0], ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y),
                                    ptr(w) if w is not None else None, ptr(dot_out) if dot_out is not None else None,
                                    _plan_handle(plan), ws, ctypes.byref(desc), _stream()), "b2s_spmv_csr_fused")
    return y


def spmv_add(indptr, indices, data, x, y, shape, plan):
    """y += A @ x (TMA tile plans)."""
    _chk_dev(indptr, indices, data, x, y)
    nrows, ncols = shape
    _lib.check(L.b2s_spmv_csr_add(vt_code(data.dtype), idx_code(indices.dtype), idx_code(indptr.dtype), nrows, ncols,
                                  data.shape[0], ptr(indptr), ptr(indices), ptr(data), ptr(x), ptr(y),
                                  _plan_handle(plan), _stream()), "b2s_spmv_csr_add")
    return y


def peer_check(own_ptr: int) -> int:
    out = _lib.c_i64(0)
    _lib.check(L.b2s_peer_check(own_ptr, _stream(), ctypes.byref(out)), "b2s_peer_check")
    return int(out.value)


def ipc_open(handle: bytes) -> int:
    out = _lib.c_vp()
    _lib.check(L.b2s_ipc_open(handle, ctypes.byref(out)), "b2s_ipc_open")
    return int(out.value)


def ipc_close(p: int) -> None:
    _lib.check(L.b2s_ipc_close(p), "b2s_ipc_close")
