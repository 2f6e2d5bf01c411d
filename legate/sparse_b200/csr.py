"""`csr_array` -- the scipy.sparse-compatible CSR matrix of the hot path.

Mirrors the public surface of the reference class (sparse/csr.py:98-262 constructor forms,
:304-322 astype/copy, :426-440 to_scipy_sparse_csr, :442-582 dot, :799 __matmul__), but the
three Legate stores `pos`/`crd`/`vals` become three device tensors in plain scipy layout:

    indptr  int32 (int64 when nnz >= 2^31)   -- reference: Rect<1> pos, 16 B/row
    indices int32 (int64 when ncols >= 2^31) -- reference: int64 crd
    data    float32 / float64

so a 5-point Laplacian row costs 5*12 + 4 bytes instead of 5*16 + 16.  Dense vectors are either
numpy arrays (host; copied to the device and back around the kernel) or torch CUDA tensors
(device resident; the role cuNumeric ndarrays play in the reference).  Compute always happens in
libb200sparse.so; there is no CPU path.
"""
from __future__ import annotations

import os
import warnings

import numpy as np
import scipy.sparse
import torch

from . import _ops
from ._dense import check_out, deliver, dense_dot, dense_rows, direct_out
from .runtime import (
    SUPPORTED_VALUE_DTYPES,
    numpy_dtype,
    runtime,
    to_device,
    to_host,
    torch_dtype,
)

_INT32_MAX = 2**31 - 1


def _force_wide() -> bool:
    # testing knob: keep 64-bit indices/indptr (exercises the int64 kernel instantiations)
    return os.environ.get("B2S_INDEX_WIDTH", "") == "64"


def _indptr_dtype(nnz: int) -> torch.dtype:
    """Row-pointer dtype of a CSR matrix with `nnz` stored entries: int32 only below 2^31 - 1 entries, the bound the
    kernels' entry points accept an int32 indptr for."""
    return torch.int32 if nnz < _INT32_MAX and not _force_wide() else torch.int64


def _index_dtype(largest: int) -> torch.dtype:
    """Column-index dtype for indices up to `largest`."""
    return torch.int32 if largest <= _INT32_MAX and not _force_wide() else torch.int64


def _entry_rows(indptr: torch.Tensor) -> torch.Tensor:
    """The int64 row of every stored entry of a CSR matrix with row pointers `indptr`."""
    ptr = indptr.to(torch.int64)
    return torch.repeat_interleave(ptr[1:] - ptr[:-1])


def cast_to_common_type(*args):
    """numpy.result_type promotion of the operands (reference sparse/utils.py:134-140)."""
    dts = [numpy_dtype(a.dtype) for a in args]
    common = np.result_type(*dts)
    return tuple(a.astype(common, copy=False) if numpy_dtype(a.dtype) != common else a for a in args)


class csr_array:
    """CSR matrix resident on one GPU (or, with no GPU visible, on the host for format logic)."""

    ndim = 2
    format = "csr"
    __array_priority__ = 10.1  # like scipy.sparse: `ndarray @ A` defers to A.__rmatmul__

    def __init__(self, arg, shape=None, dtype=None, copy=False):
        from .module import is_sparse_matrix

        self._cache = {}
        if isinstance(arg, torch.Tensor) and arg.ndim == 2:
            arg = to_host(arg)
        if isinstance(arg, np.ndarray):
            # dense -> CSR: nonzero test is `!= 0`, columns ascending
            # (src/sparse/array/conv/dense_to_csr.cc:32-38,53-62)
            assert arg.ndim == 2
            shape = arg.shape
            mask = arg != 0
            counts = mask.sum(axis=1).astype(np.int64)
            indptr = np.zeros(shape[0] + 1, dtype=np.int64)
            np.cumsum(counts, out=indptr[1:])
            rows, cols = np.nonzero(mask)
            self._set_arrays(indptr, cols, arg[rows, cols])
        elif isinstance(arg, (scipy.sparse.csr_array, scipy.sparse.csr_matrix)):
            shape = arg.shape
            self._set_arrays(arg.indptr, arg.indices, arg.data, copy=True)
        elif isinstance(arg, tuple):
            if copy:
                raise NotImplementedError
            if shape is None:
                raise AssertionError("Cannot infer shape in this case.")
            if len(arg) == 2:
                # (data, (row, col)) goes through COO (reference csr.py:174-185)
                from .coo import coo_array

                data, (row, col) = arg
                res = coo_array((data, (row, col)), shape=shape).tocsr()
                self._indptr, self._indices, self._data = res._indptr, res._indices, res._data
                shape = res.shape
            elif len(arg) == 3:
                data, indices, indptr = arg
                assert indptr.shape[0] == shape[0] + 1
                self._set_arrays(indptr, indices, data)
            else:
                raise AssertionError
        elif is_sparse_matrix(arg):
            csr = arg.tocsr()
            if copy:
                csr = csr.copy()
            self._indptr, self._indices, self._data = csr._indptr, csr._indices, csr._data
            shape = csr.shape
        elif scipy.sparse.issparse(arg):
            s = arg.tocsr()
            shape = s.shape
            self._set_arrays(s.indptr, s.indices, s.data, copy=True)
        else:
            raise NotImplementedError

        assert shape is not None
        self.shape = tuple(int(i) for i in shape)
        assert self._indptr.shape[0] == self.shape[0] + 1
        if dtype is not None and numpy_dtype(dtype) != numpy_dtype(self._data.dtype):
            self._data = self._data.to(torch_dtype(dtype))
        self.dtype = numpy_dtype(self._data.dtype)

    # -- storage ------------------------------------------------------------------------------------
    def _set_arrays(self, indptr, indices, data, copy=False):
        self._indptr = to_device(indptr, dtype=_indptr_dtype(int(data.shape[0])), copy=copy)
        if not isinstance(indices, torch.Tensor):
            indices = np.asarray(indices)
        self._indices = to_device(indices, dtype=_index_dtype(int(indices.max()) if len(indices) else 0), copy=copy)
        self._data = to_device(data, copy=copy)

    # reference exposes `.data` / `.indices` as device arrays (csr.py:264-287); `.indptr` is added
    # because the layout here is plain scipy CSR.
    @property
    def data(self):
        return self._data

    @data.setter
    def data(self, value):
        self._data = to_device(value)
        self.dtype = numpy_dtype(self._data.dtype)
        self._cache.clear()

    @property
    def indices(self):
        return self._indices

    @indices.setter
    def indices(self, value):
        self._indices = to_device(value)
        self._cache.clear()

    @property
    def indptr(self):
        return self._indptr

    @property
    def nnz(self) -> int:
        return int(self._data.shape[0])

    @property
    def device(self):
        return self._data.device

    @classmethod
    def _from_parts(cls, indptr, indices, data, shape):
        obj = cls.__new__(cls)
        obj._cache = {}
        obj._indptr, obj._indices, obj._data = indptr, indices, data
        obj.shape = tuple(int(i) for i in shape)
        obj.dtype = numpy_dtype(data.dtype)
        return obj

    @classmethod
    def make_empty(cls, shape, dtype):
        dev = runtime.device
        return cls._from_parts(
            torch.zeros(shape[0] + 1, dtype=torch.int32, device=dev),
            torch.zeros(0, dtype=torch.int32, device=dev),
            torch.zeros(0, dtype=torch_dtype(dtype), device=dev),
            shape,
        )

    # -- conversions ----------------------------------------------------------------------------------
    def astype(self, dtype, casting="unsafe", copy=True):
        dtype = np.dtype(dtype)
        if not copy and dtype == self.dtype:
            return self
        data = self._data.to(torch_dtype(dtype), copy=copy)
        indptr = self._indptr.clone() if copy else self._indptr
        indices = self._indices.clone() if copy else self._indices
        return csr_array._from_parts(indptr, indices, data, self.shape)

    def copy(self):
        return csr_array._from_parts(self._indptr.clone(), self._indices.clone(), self._data.clone(), self.shape)

    def conj(self, copy=True):
        if self.dtype.kind == "c":
            return csr_array._from_parts(self._indptr, self._indices, self._data.conj().resolve_conj(), self.shape)
        return self.copy() if copy else self   # real: the identity

    def tocsr(self, copy=False):
        return self.copy() if copy else self

    def tocsc(self, copy=False):
        """The CSC form: a csc_array holding the CSR transpose (`transpose`), so new arrays whatever `copy` says."""
        from .csc import csc_array

        return csc_array(self)

    def todia(self, copy=False):
        """The DIA form (b2s_csr_to_dia on the GPU), as scipy's `todia`: new arrays whatever `copy` says."""
        from .dia import _csr_to_dia

        return _csr_to_dia(self)

    def tocoo(self, copy=False):
        from .coo import coo_array

        rows = _entry_rows(self._indptr)
        return coo_array((self._data.clone() if copy else self._data, (rows, self._indices)), shape=self.shape)

    def to_scipy_sparse_csr(self):
        return scipy.sparse.csr_array(
            (to_host(self._data), to_host(self._indices), to_host(self._indptr)), shape=self.shape, dtype=self.dtype
        )

    def todense(self, order=None, out=None):
        if order is not None:
            raise NotImplementedError
        res = self.to_scipy_sparse_csr().toarray()
        if out is not None:
            out[...] = res
            return out
        return res

    toarray = todense

    def transpose(self, copy=False):
        """CSR of the transpose (construction path: the reference reaches it through CSC aliasing,
        csc.py:317-324).  Counting sort by column with plain tensor ops on the device."""
        nrows, ncols = self.shape
        dev = self.device
        if (self._data.is_cuda and self._data.dtype in (torch.float32, torch.float64)
                and (self._indices.dtype == torch.int64 or nrows <= _INT32_MAX)):
            # the library's own kernels (b2s_csr_transpose, csrc/convert.cu): counting sort by column + per-row sort
            t_ptr, t_idx, t_val = _ops.csr_transpose(self._indptr, self._indices, self._data, self.shape)
            return csr_array._from_parts(t_ptr, t_idx, t_val, (ncols, nrows))
        rows = _entry_rows(self._indptr)
        cols = self._indices.to(torch.int64)
        order = torch.argsort(cols * max(nrows, 1) + rows)
        t_counts = torch.bincount(cols, minlength=ncols)
        t_indptr = torch.zeros(ncols + 1, dtype=torch.int64, device=dev)
        torch.cumsum(t_counts, 0, out=t_indptr[1:])
        return csr_array._from_parts(t_indptr.to(_indptr_dtype(self.nnz)), rows[order].to(_index_dtype(nrows)),
                                     self._data[order], (ncols, nrows))

    T = property(transpose)

    def diagonal(self, k=0):
        """Main diagonal as a device vector (reference csr.py:629-649; only k = 0 there too)."""
        if k != 0:
            raise NotImplementedError
        rows, cols = self.shape
        if self._data.is_cuda:
            d = _ops.csr_diagonal(self._indptr, self._indices, self._data, rows)
            return d[: min(rows, cols)]
        return to_device(self.to_scipy_sparse_csr().diagonal())

    # -- what is derived from the arrays, cached -------------------------------------------------------
    def _stamp(self):
        """Pointer and version counter of indptr, indices and data.  An in-place edit of any of them changes it;
        assigning a new array does not always (a new tensor may reuse a freed one's address and version), so every
        assignment clears `_cache` as well."""
        p, i, d = self._indptr, self._indices, self._data
        return p.data_ptr(), p._version, i.data_ptr(), i._version, d.data_ptr(), d._version

    def _derived(self, kind, extra, build):
        """The derivative `kind` of the arrays (SpMV plan, promoted copy, transpose, ...) for the parameters `extra`:
        `build()` runs again whenever `self._stamp()` or `extra` differs from the cached one.  One slot per kind, so a
        caller switching parameters on one matrix does not pile up device buffers.  `dia_array` caches the same way,
        against its own stamp."""
        stamp = self._stamp()
        hit = self._cache.get(kind)
        if hit is None or hit[0] != stamp or hit[1] != extra:
            hit = self._cache[kind] = (stamp, extra, build())
        return hit[2]

    # -- the hot path -----------------------------------------------------------------------------------
    def _get_plan(self, tma_only: bool = False):
        """Tile plan for the SpMV kernel, built once per structure and cached (the reference caches
        its image partitions per store the same way, sparse/partition.py:96-120).  `tma_only`: the plan must
        launch the TMA tile kernel (accumulating / exchange-fused products); sticky once requested.  A packed plan
        holds its own copy of the structure, and a coded one of the values, so an in-place edit builds a new plan --
        a new one, never a rewrite of the old pack buffer, which a captured graph may still read."""
        from . import _lib

        tma_only = bool(tma_only or getattr(self, "_plan_tma_only", False))
        self._plan_tma_only = tma_only

        def build():
            plan = _ops.spmv_plan(self._indptr, self._indices, self.shape, self.nnz, self.dtype, tma_only=tma_only)
            if self._data.is_contiguous():
                plan = _ops.spmv_plan_code(plan, self._indptr, self._indices, self._data)
                plan = _ops.spmv_plan_templates(plan, self._indptr, self._indices, self._data)
            return plan

        return self._derived("plan", (int(_lib.lib.b2s_spmv_get_config()), tma_only), build)

    # -- column-split SpMV (reference csr.py:869-927 / spmv.cu:125-153: x partitioned, y reduced) -------------------
    @staticmethod
    def _col_block_bytes() -> int:
        """One block's slice of x: what stays L2-resident next to the matrix stream (a third of L2)."""
        return runtime.l2_bytes() // 3

    def _col_split(self, nblocks=None):
        """[(column block, plan)]: block q holds the entries whose column lies in [q*T, (q+1)*T), global column ids
        kept, so `y = sum_q A_q x` with every block gathering from ONE slice of x.  Built once per structure / values
        and cached.  The reference's column-split SpMV partitions x the same way and reduces the partial y with ADD."""
        n = self.shape[1]
        if nblocks is None:
            # scattered columns: one block per third of L2 of x (each block's slice stays in L2); otherwise the split is
            # only the partitioning the caller asked for -- two blocks (more blocks of a one-entry-per-row operator such
            # as GMG's restriction only add launches)
            scattered = bool(getattr(self._get_plan(), "scattered", False))
            nblocks = max(2, min(16, -(-n * self.dtype.itemsize // self._col_block_bytes()))) if scattered else 2
        nblocks = max(1, min(int(nblocks), max(n, 1)))

        def build():
            T = -(-n // nblocks)
            blocks = _column_blocks(self, [(q * T, min((q + 1) * T, n)) for q in range(nblocks)])
            return [(B, B._get_plan(tma_only=True)) for B in blocks if B is not None]

        return self._derived("colsplit", nblocks, build)

    def _dot_col_split(self, xd, y, nblocks=None):
        """y = A @ xd as a sum over column blocks: the first block writes y, the others accumulate (b2s_spmv_csr_add)."""
        blocks = self._col_split(nblocks)
        if not blocks:
            y.zero_()
            return y
        first = True
        for B, pl in blocks:
            if first:
                _ops.spmv(B._indptr, B._indices, B._data, xd, y, B.shape, plan=pl)
                first = False
            else:
                _ops.spmv_add(B._indptr, B._indices, B._data, xd, y, B.shape, pl)
        return y

    def _wants_col_split(self, plan) -> bool:
        """Scattered columns and an x larger than L2 can hold next to the matrix stream: gathers from one slice of x at a
        time hit L2, the unsplit product misses it.  "Larger" is more than 3/8 of L2.  Only when the blocks keep a few
        entries per row."""
        if os.environ.get("B2S_COL_SPLIT", "auto") == "0":
            return False
        xbytes = self.shape[1] * self.dtype.itemsize
        if not getattr(plan, "scattered", False) or xbytes <= 3 * runtime.l2_bytes() // 8:
            return False
        nblocks = -(-xbytes // self._col_block_bytes())
        if self.nnz < 4 * nblocks * max(self.shape[0], 1):
            return False
        if "colsplit" in self._cache:
            return True
        # the blocks are a second copy of the matrix (+ one indptr per block, + transient masks while they are cut):
        # only when that fits comfortably in what the device has free
        need = self.nnz * (self.dtype.itemsize + 4 + 9) + nblocks * (self.shape[0] + 1) * 16
        try:
            free, _total = torch.cuda.mem_get_info(self.device)
        except Exception:  # pragma: no cover - no usable device query: keep the unsplit product
            return False
        return need < 0.6 * free

    def _promoted(self, common):
        """A cast to the resolved dtype of (A, x) -- reference cast_to_common_type, csr.py:493 -- cached
        so a mixed-dtype SpMV does not re-cast the matrix on every call."""
        if self.dtype == common:
            return self
        return self._derived(("promoted", common), None, lambda: self.astype(common, copy=False))

    def _dot_host_pipelined(self, x: np.ndarray, out, plan):
        """y = A @ x for HOST vectors, software-pipelined over the plan's row chunks.

        Chunk c only reads x inside its column window (plan.chunks; the reference's MinMaxImagePartition idea
        applied to row chunks of one GPU), so its tiles can run as soon as x[:col_hi_c] has arrived, while the
        rest of x is still crossing PCIe and while y of earlier chunks is already on its way back.  For a
        banded matrix the product then costs about max(H2D, D2H) instead of H2D + kernel + D2H.  Pinned host
        arrays give true overlap; pageable ones still work (the copies just serialise)."""
        dev = self.device
        tdt = torch_dtype(self.dtype)
        st = self.__dict__.setdefault("_pipe", {})
        if st.get("key") != (self.shape, self.dtype):
            st.clear()
            st.update(key=(self.shape, self.dtype), xd=torch.empty(self.shape[1], dtype=tdt, device=dev),
                      yd=torch.empty(self.shape[0], dtype=tdt, device=dev))
        if out is None:
            out = np.empty(self.shape[0], dtype=self.dtype)
        _ops.spmv_host(self._indptr, self._indices, self._data, x.ctypes.data, out.ctypes.data, st["xd"], st["yd"],
                       self.shape, plan)
        return out

    # -- complex operands ------------------------------------------------------------------------------
    def _real_expansion(self, rdt):
        """Real (2m x 2n) CSR matrix E with E @ interleave(re x, im x) = interleave(re (A x), im (A x)): every
        complex entry a at (r, c) becomes the block [[re a, -im a], [im a, re a]] at rows 2r, 2r+1 / columns
        2c, 2c+1.  Built once per matrix with tensor ops and cached, so a complex SpMV is ONE launch of the real
        SpMV kernel on interleaved (re, im) storage -- which is exactly how complex vectors sit in memory."""
        return self._derived("expansion", np.dtype(rdt), lambda: self._make_real_expansion(rdt))

    def _make_real_expansion(self, rdt):
        m, n = self.shape
        dev = self.device
        nnz = self.nnz
        tdt = torch_dtype(rdt)
        ptr64 = self._indptr.to(torch.int64)
        lens = ptr64[1:] - ptr64[:-1]
        rows = _entry_rows(ptr64)
        q = torch.arange(nnz, dtype=torch.int64, device=dev) - ptr64[rows]      # position inside its row
        top = 4 * ptr64[rows] + 2 * q                                           # slot of (2r, 2c)
        bot = top + 2 * lens[rows]                                              # slot of (2r+1, 2c)
        cols = self._indices.to(torch.int64)
        data = self._data.to(torch.complex128 if np.dtype(rdt) == np.float64 else torch.complex64)
        re, im = data.real.to(tdt), data.imag.to(tdt)
        e_idx = torch.empty(4 * nnz, dtype=torch.int64, device=dev)
        e_val = torch.empty(4 * nnz, dtype=tdt, device=dev)
        e_idx[top], e_idx[top + 1], e_idx[bot], e_idx[bot + 1] = 2 * cols, 2 * cols + 1, 2 * cols, 2 * cols + 1
        e_val[top], e_val[top + 1], e_val[bot], e_val[bot + 1] = re, -im, im, re
        e_ptr = torch.empty(2 * m + 1, dtype=torch.int64, device=dev)
        e_ptr[0:2 * m:2] = 4 * ptr64[:-1]
        e_ptr[1:2 * m:2] = 4 * ptr64[:-1] + 2 * lens
        e_ptr[2 * m] = 4 * nnz
        return csr_array._from_parts(e_ptr.to(_indptr_dtype(4 * nnz)), e_idx.to(_index_dtype(2 * n)), e_val,
                                     (2 * m, 2 * n))

    def _dot_complex(self, x, out):
        """A @ x for a complex A (the reference dispatches its SpMV / SpMM tasks over complex64/128 too,
        src/sparse/util/dispatch.h).  No complex kernels: the real SpMV / SpMM of A's real expansion
        (`_real_expansion`) on the (re, im)-interleaved view of x."""
        m, n = self.shape
        common = np.result_type(self.dtype, numpy_dtype(x.dtype))
        rshape = (m,) if x.ndim == 1 else (m, x.shape[1])
        check_out(out, rshape, common)
        runtime.require_cuda("csr_array.dot")
        X = to_device(x, dtype=common)
        k = 1 if X.ndim == 1 else X.shape[1]
        Xr = torch.view_as_real(X.reshape(n, k))                                  # (n, k, 2) real view
        E = self._real_expansion(np.dtype(np.float32) if common == np.complex64 else np.dtype(np.float64))
        if k == 1:
            yr = torch.empty(2 * m, dtype=Xr.dtype, device=Xr.device)
            _ops.spmv(E._indptr, E._indices, E._data, Xr.reshape(2 * n), yr, E.shape, plan=E._get_plan())
            Y = torch.view_as_complex(yr.reshape(m, 1, 2))
        else:
            Xe = Xr.permute(0, 2, 1).reshape(2 * n, k).contiguous()           # rows: re x_0, im x_0, re x_1, ...
            Ye = torch.empty((2 * m, k), dtype=Xr.dtype, device=Xr.device)
            _ops.spmm(E._indptr, E._indices, E._data, Xe, Ye, E.shape)
            Y = torch.view_as_complex(Ye.reshape(m, 2, k).permute(0, 2, 1).contiguous())
        return deliver(Y.reshape(rshape), out, isinstance(x, torch.Tensor) and x.is_cuda, False)

    def dot(self, other, out=None, spmv_domain_part=False):
        """`A.dot(x)` / `A @ B`; see reference sparse/csr.py:442-582.

        * x 1-D or (n,1), numpy or torch CUDA tensor -> SpMV; result has x's array kind.
        * other dense 2-D (n,k) -> SpMM, dense (m,k) result of the same array kind.
        * other a csr_array -> SpGEMM (CSR x CSR -> CSR).
        `spmv_domain_part=True` (column-split SpMV, csr.py:869-927, spmv.cu:125-153): x is partitioned into column
        blocks, every block's partial product is reduced into y by the accumulating kernel (`_dot_col_split`); the
        same path is taken by itself when the columns are scattered and x exceeds L2 (`_wants_col_split`).
        """
        from .module import is_sparse_matrix

        if isinstance(other, csr_array):
            if out is not None:
                raise ValueError("Cannot provide out for CSRxCSR matmul.")
            assert self.shape[1] == other.shape[0]
            return spgemm_csr_csr_csr(*cast_to_common_type(self, other))
        densified = is_sparse_matrix(other) or scipy.sparse.issparse(other)
        if densified:
            from .csc import csc_array

            from .dia import dia_array

            if isinstance(other, (csc_array, dia_array)):
                # CSR x CSC and CSR x DIA are SpGEMM with the cached CSR form, not a dense product
                return self.dot(other.tocsr(), out=out)
            other = np.asarray(other.todense())
        x = other if isinstance(other, (np.ndarray, torch.Tensor)) else np.asarray(other)
        res = self._dot_dense(x, out, spmv_domain_part)
        if densified:
            return csr_array(np.asarray(to_host(res)).reshape(self.shape[0], -1))
        return res

    def _dot_dense(self, x, out, spmv_domain_part):
        """A @ x for a dense x: `dense_dot` with this class's launchers, after the checks the reference makes and the
        software-pipelined product of host vectors (`_dot_host_pipelined`), which has to see x before it moves."""
        m, n = self.shape
        if x.ndim not in (1, 2):
            raise NotImplementedError("csr_array.dot: operand must be a vector, a dense 2-D array or a csr_array")
        rshape = (m,) if x.ndim == 1 else (m, x.shape[1])
        assert x.shape[0] == n
        assert out is None or tuple(out.shape) == rshape
        common = np.result_type(self.dtype, numpy_dtype(x.dtype))
        if (x.ndim == 1 or x.shape[1] == 1) and common.kind != "c":
            if isinstance(x, torch.Tensor) and not x.reshape(-1).is_contiguous():
                warnings.warn(
                    "CSR SpMV creating an implicit copy due to transformed x vector.",
                    category=RuntimeWarning,
                    stacklevel=3,
                )
            assert out is None or x.ndim == 1 or not spmv_domain_part
            if (isinstance(x, np.ndarray) and x.dtype == common and common in SUPPORTED_VALUE_DTYPES
                    and x.reshape(-1).flags.c_contiguous
                    and (out is None or (isinstance(out, np.ndarray) and out.flags.c_contiguous))
                    and not spmv_domain_part and os.environ.get("B2S_PIPELINE", "1") != "0"):
                check_out(out, rshape, common)
                runtime.require_cuda("csr_array.dot")
                A = self._promoted(common)
                plan = A._get_plan()
                if plan.chunks:
                    # host vectors: stream x in / y out chunk by chunk, overlapping both PCIe directions with the kernel
                    y = A._dot_host_pipelined(x.reshape(-1), None if out is None else out.reshape(-1), plan)
                    return out if out is not None else y.reshape(rshape)

        def spmv(dt, xd, y):
            A = self._promoted(dt)
            plan = A._get_plan()
            if spmv_domain_part or A._wants_col_split(plan):
                A._dot_col_split(xd, y)      # x partitioned by columns, partial products reduced into y
            else:
                _ops.spmv(A._indptr, A._indices, A._data, xd, y, A.shape, plan=plan)

        def spmm(dt, X, Y):
            A = self._promoted(dt)
            _ops.spmm(A._indptr, A._indices, A._data, X, Y, A.shape)

        return dense_dot(x, out, self.dtype, self.shape, "csr_array.dot", spmv, spmm, self._dot_complex)

    def matvec(self, other):
        return self @ other

    def __matmul__(self, other):
        return self.dot(other)

    def __rmatmul__(self, other):
        """dense (i, m) @ A (m, n) -> dense (i, n)  (reference csr.py:801-822, rspmm csr.py:1208-1262).
        Computed as (A^T @ other^T)^T with the row-major SpMM kernel; A^T is built once and cached."""
        if not isinstance(other, (np.ndarray, torch.Tensor)):
            other = np.asarray(other)
        if other.ndim != 2:
            raise NotImplementedError
        assert other.shape[1] == self.shape[0]
        At = self._derived("transpose", None, self.transpose)
        if isinstance(other, torch.Tensor):
            return At.dot(other.t().contiguous()).t().contiguous()
        return np.ascontiguousarray(At.dot(np.ascontiguousarray(other.T)).T)

    def __mul__(self, other):
        if np.isscalar(other):
            return csr_array._from_parts(self._indptr, self._indices, self._data * other, self.shape)
        return self.multiply(other)   # elementwise, as the reference's __mul__ (csr.py:1033-1148)

    __rmul__ = __mul__

    def __neg__(self):
        return self * -1

    # -- elementwise arithmetic (reference csr.py:760-776 __add__ / add, 1033-1148 mult / mult_dense) ------------------
    def _binop(self, other, op: str, reverse: bool = False):
        """self op other (other op self when `reverse`) for a sparse `other`; None when `other` is not sparse."""
        B = _as_sparse_operand(other)
        if B is None:
            return None
        if B.shape != self.shape:
            raise ValueError(f"inconsistent shapes {self.shape} and {B.shape}")
        A, B = cast_to_common_type(self, B)
        if A.dtype not in SUPPORTED_VALUE_DTYPES:
            raise NotImplementedError(f"sparse {op} for dtype {A.dtype} is not implemented (float32/float64 kernels only)")
        return _csr_binop(B, A, op) if reverse else _csr_binop(A, B, op)

    def _dense_binop(self, other, op: str, reverse: bool = False):
        """self op other for a dense `other`: the dense result, in other's array kind (reference: todense() + other)."""
        common = np.result_type(self.dtype, numpy_dtype(other.dtype))
        if common.kind == "c":
            raise NotImplementedError("complex elementwise operations are not implemented")
        if isinstance(other, torch.Tensor):
            D = torch.zeros(self.shape, dtype=torch_dtype(common), device=other.device)
            rows = _entry_rows(self._indptr)
            D.index_put_((rows.to(other.device), self._indices.to(device=other.device, dtype=torch.int64)),
                         self._data.to(device=other.device, dtype=D.dtype), accumulate=True)
        else:
            D = self.todense().astype(common, copy=False)
        if op == "add":
            return D + other
        return other - D if reverse else D - other

    def _scalar_binop(self, other, op: str, reverse: bool = False):
        if other != 0:
            raise NotImplementedError(f"{'adding' if op == 'add' else 'subtracting'} a nonzero scalar to a sparse matrix "
                                      "is not supported")
        return -self if (reverse and op == "sub") else self.copy()

    def _arith(self, other, op: str, reverse: bool = False):
        if np.isscalar(other):
            return self._scalar_binop(other, op, reverse)
        C = self._binop(other, op, reverse)
        if C is not None:
            return C
        if isinstance(other, (np.ndarray, torch.Tensor)):
            return self._dense_binop(other, op, reverse)
        return NotImplemented

    def __add__(self, other):
        return self._arith(other, "add")

    def __radd__(self, other):
        return self._arith(other, "add", reverse=True)

    def __sub__(self, other):
        return self._arith(other, "sub")

    def __rsub__(self, other):
        return self._arith(other, "sub", reverse=True)

    def multiply(self, other):
        """Elementwise product.  Sparse `other`: the intersection of the two structures.  Dense `other` of shape (m, n),
        (m, 1), (1, n) or (n,): A's structure, each value times its entry of `other` (broadcast along rows / columns)."""
        if np.isscalar(other):
            return self * other
        C = self._binop(other, "mul")
        if C is not None:
            return C
        D = other if isinstance(other, torch.Tensor) else np.asarray(other)
        if D.ndim == 0:
            return self * D.item()
        m, n = self.shape
        shape = tuple(D.shape)
        if shape == (m, n):
            mode = "dense"
        elif shape == (m, 1):
            mode = "rows"
        elif shape in ((1, n), (n,)):
            mode = "cols"
        else:
            raise ValueError(f"inconsistent shapes {self.shape} and {shape}")
        common = np.result_type(self.dtype, numpy_dtype(D.dtype))
        if common not in SUPPORTED_VALUE_DTYPES:
            raise NotImplementedError(f"multiply for dtype {common} is not implemented (float32/float64 kernels only)")
        runtime.require_cuda("csr_array.multiply")
        A = self.astype(common, copy=False)
        Dd = to_device(D, dtype=common).reshape(-1)
        data = _ops.csr_scale(A._indptr, A._indices, A._data, Dd, mode, self.shape)
        return csr_array._from_parts(A._indptr, A._indices, data, self.shape)

    def sddmm(self, C, D):
        """Sampled dense-dense product (reference csr.py:688-705): a new csr_array with A's structure (it shares A's
        indptr and indices) whose value at each stored entry (i, j) is A[i, j] * (C @ D)[i, j], for C (m, k) and D (k, n)
        given as numpy arrays or torch tensors.  Every stored entry is computed on its own: repeated columns, unsorted
        rows and explicit zeros are kept, and k = 0 gives A.data * 0.  The dtype is np.result_type(A, C, D).

        The kernel reads D transposed, an (n, k) array with contiguous rows.  When D.T already has unit inner stride
        (D = K.T for a row-major (n, k) K, or a Fortran-ordered D) it is used as it is; otherwise D is copied once into
        that layout, which costs a read and a write of n * k values (comparable to the product itself when k is large
        and A has few entries per column).  C is copied only when its rows are not unit-stride."""
        Cx = C if isinstance(C, (np.ndarray, torch.Tensor)) else np.asarray(C)
        Dx = D if isinstance(D, (np.ndarray, torch.Tensor)) else np.asarray(D)
        if Cx.ndim != 2 or Dx.ndim != 2:
            raise ValueError(f"sddmm needs 2-D dense operands, got {Cx.ndim}-D and {Dx.ndim}-D")
        m, n = self.shape
        if Cx.shape[0] != m or Dx.shape[1] != n or Cx.shape[1] != Dx.shape[0]:
            raise ValueError(f"inconsistent shapes {self.shape}, {tuple(Cx.shape)} and {tuple(Dx.shape)} for sddmm")
        common = np.result_type(self.dtype, numpy_dtype(Cx.dtype), numpy_dtype(Dx.dtype))
        if common.kind == "c":
            raise NotImplementedError("complex sddmm is not implemented")
        if common not in SUPPORTED_VALUE_DTYPES:
            raise NotImplementedError(f"sddmm for dtype {common} is not implemented (float32/float64 kernels only)")
        runtime.require_cuda("csr_array.sddmm")
        A = self._promoted(common)
        Cd = dense_rows(Cx, common)
        Dt = dense_rows(Dx.T, common)
        out = _ops.sddmm(A._indptr, A._indices, A._data, Cd, Dt)
        return csr_array._from_parts(A._indptr, A._indices, out, self.shape)

    def tropical_spmv(self, other, out=None):
        """Lexicographic-max product (reference csr.py:365-424, kernel tropical_spmv.cu:26-56): for x of shape (n, F),
        row i of the (m, F) int64 result is the lexicographic maximum of the zero vector and of x[j, :] over every
        stored entry (i, j).  Fields compare as signed int64, field 0 the most significant.  Only A's structure counts:
        its values and dtype are ignored, and explicit zeros and repeated columns are edges like any other.  An empty
        row, or one whose neighbours are all lexicographically negative, gives zeros.  The result is exact.

        x must be 2-D with n rows (else ValueError).  The reference leaves dtype checks open; here any integer dtype is
        accepted and cast to int64 (uint64 values above 2^63 - 1 wrap), and float, complex and bool raise TypeError.
        The result has x's array kind, as in `dot`: a numpy x gives numpy, a torch CUDA x a torch CUDA tensor, used
        without a copy when it is int64 with unit-stride rows.  `out` may be a numpy array or a torch tensor of shape
        (m, F) and dtype int64 (else ValueError), and must not overlap x (ValueError): the kernel reads x rows while
        other rows of the result are written.  Every argument is checked before a device is touched."""
        x = other if isinstance(other, (np.ndarray, torch.Tensor)) else np.asarray(other)
        if x.ndim != 2:
            raise ValueError(f"tropical_spmv needs a 2-D operand, got {x.ndim}-D")
        m, n = self.shape
        if x.shape[0] != n:
            raise ValueError(f"inconsistent shapes {self.shape} and {tuple(x.shape)} for tropical_spmv")
        if not _is_integer_dtype(x.dtype):
            raise TypeError(f"tropical_spmv needs an integer operand, got {x.dtype}")
        nf = int(x.shape[1])
        if out is not None:
            int64_out = ((isinstance(out, np.ndarray) and out.dtype == np.int64)
                         or (isinstance(out, torch.Tensor) and out.dtype == torch.int64))
            if not int64_out or tuple(out.shape) != (m, nf):
                raise ValueError(f"out must be an int64 numpy array or torch tensor of shape {(m, nf)}")
            if _overlaps(out, x):
                raise ValueError("out overlaps the operand of tropical_spmv")
        runtime.require_cuda("csr_array.tropical_spmv")
        direct = direct_out(out, (m, nf))
        y = _ops.tropical_spmv(self._indptr, self._indices, dense_rows(x, np.int64), out if direct else None)
        return deliver(y, out, isinstance(x, torch.Tensor) and x.is_cuda, direct)

    # -- reductions (scipy csr_array sum / mean / max / min / argmax / argmin / count_nonzero; csrc/reduce.cu) ----------
    def _canonical(self):
        """(indptr, indices, data) of A with sorted rows and repeated columns summed -- what `A.toarray()` sees, explicit
        zeros kept.  Built once per stamp from a sorted clone when a row is unsorted; the merge of repeated columns runs
        the row-sum kernel over the runs of equal columns.  Without either, it is A's own arrays (no copy)."""
        return self._derived("canonical", None, lambda: _canonical_parts(self, rows_sorted=False))

    def _canonical_t(self):
        """The canonical form of the cached transpose (the one `X @ A` uses): its rows, A's columns, are sorted already."""
        At = self._derived("transpose", None, self.transpose)
        return self._derived("canonical_t", None, lambda: _canonical_parts(At, rows_sorted=True))

    def _check_reduction(self, axis, what):
        """`axis` as None, 0 or 1, after the checks that need no device: ValueError for any other axis,
        NotImplementedError for data other than float32 / float64."""
        if axis is not None:
            if isinstance(axis, (bool, np.bool_)) or not isinstance(axis, (int, np.integer)) or not -2 <= axis <= 1:
                raise ValueError(f"axis {axis!r} out of range for a 2-D sparse array (None, 0, 1, -2 or -1)")
            axis = int(axis) % 2
        if self.dtype not in SUPPORTED_VALUE_DTYPES:
            raise NotImplementedError(f"csr_array.{what} for dtype {self.dtype} is not implemented (float32/float64 only)")
        return axis

    def _reduce_axis(self, op, axis, explicit=False):
        """1-D device tensor: `op` over every row (axis 1) or column (axis 0).  Sums read A (or its transpose) as it
        is; the other reductions read the canonical form."""
        m, n = self.shape
        if self.nnz == 0:       # every row or column is empty: no transpose to build
            ptr_ = torch.zeros(self.shape[1 - axis] + 1, dtype=torch.int32, device=self.device)
            return _ops.csr_reduce_rows(op, ptr_, self._indices, self._data, n if axis == 1 else m, explicit)
        if op == "sum":
            B = self if axis == 1 else self._derived("transpose", None, self.transpose)
            ptr_, idx, dat = B._indptr, B._indices, B._data
        else:
            ptr_, idx, dat = self._canonical() if axis == 1 else self._canonical_t()
        return _ops.csr_reduce_rows(op, ptr_, idx if op in ("argmax", "argmin") else None, dat, n if axis == 1 else m,
                                    explicit)

    def sum(self, axis=None, dtype=None, out=None):
        """Sum of all entries (axis None: a numpy scalar), of every column (axis 0: a length-n CUDA tensor) or of every
        row (axis 1: length m).  Rows are summed by the kernel in fp64 in an order fixed by their length, then rounded
        once to `dtype` (default: the data's); float32 data with dtype float64 is summed from a cached float64 copy.
        axis None is the sum of the stored values (fp64, one sync).  `out`: a numpy array or torch tensor of the
        result's shape and dtype.  A column reduction builds a transposed copy of A once and keeps it in A's cache (the
        one `X @ A` uses) until A's arrays change."""
        axis = self._check_reduction(axis, "sum")
        rdt = self._reduction_dtype(dtype, "sum")
        _check_reduction_out(out, () if axis is None else (self.shape[1 - axis],), rdt)
        runtime.require_cuda("csr_array.sum")
        A = self._promoted(rdt) if rdt.itemsize > self.dtype.itemsize else self
        if axis is None:
            return _deliver_scalar(rdt.type(float(A._data.sum(dtype=torch.float64))), out)
        v = A._reduce_axis("sum", axis)
        return deliver(v.to(torch_dtype(rdt)), out, True, False)

    def mean(self, axis=None, dtype=None, out=None):
        """`sum(axis, dtype)` divided by shape[axis] (by m * n for axis None); same result kinds and `out` as sum."""
        axis = self._check_reduction(axis, "mean")
        rdt = self._reduction_dtype(dtype, "mean")
        _check_reduction_out(out, () if axis is None else (self.shape[1 - axis],), rdt)
        count = self.shape[0] * self.shape[1] if axis is None else self.shape[axis]
        s = self.sum(axis=axis, dtype=rdt)
        if axis is None:
            with np.errstate(invalid="ignore", divide="ignore"):
                return _deliver_scalar(rdt.type(np.true_divide(s, rdt.type(count))), out)
        return deliver(s / count, out, True, False)

    def _reduction_dtype(self, dtype, what):
        rdt = self.dtype if dtype is None else np.dtype(dtype)
        if rdt not in SUPPORTED_VALUE_DTYPES:
            raise NotImplementedError(f"csr_array.{what} with dtype {rdt} is not implemented (float32/float64 only)")
        return rdt

    def _extreme(self, op, axis, out, explicit):
        axis = self._check_reduction(axis, op)
        if out is not None:
            raise ValueError("Sparse min/max does not support an 'out' parameter.")
        m, n = self.shape
        if (m * n == 0) if axis is None else self.shape[axis] == 0:
            raise ValueError("zero-size array to reduction operation")
        runtime.require_cuda(f"csr_array.{op}")
        if axis is not None:
            return self._reduce_axis(op, axis, explicit)
        ptr_, _, dat = self._canonical()
        rows = _ops.csr_reduce_rows(op, ptr_, None, dat, n, explicit)
        if explicit:
            # an empty row has no stored value to offer; a matrix without any gives 0, as scipy does
            rows = torch.cat([rows[ptr_[1:] > ptr_[:-1]], rows.new_zeros(1 if dat.shape[0] == 0 else 0)])
        return self.dtype.type((rows.max() if op == "max" else rows.min()).item())

    def max(self, axis=None, out=None, *, explicit=False):
        """Largest entry of A (axis None: a numpy scalar), of every column (axis 0: a length-n CUDA tensor of A's dtype)
        or of every row (axis 1: length m).  Implicit zeros count unless `explicit`; a NaN anywhere in a row makes that
        row's result NaN.  Differences from scipy: along an axis the result is the dense vector, not a sparse 1-D
        coo_array (a tensor's `.data` is the tensor itself, so `B.max(axis=0).data[B.indices]` works on both), and
        csr_matrix, an alias of csr_array here, also returns 1-D rather than an (m, 1) matrix.  `out` is not supported
        (ValueError), nor is a reduction over a zero-length axis.  A column reduction builds a transposed copy of A
        once and keeps it in A's cache (with its canonical form) until A's arrays change."""
        return self._extreme("max", axis, out, explicit)

    def min(self, axis=None, out=None, *, explicit=False):
        """Smallest entry; see `max`."""
        return self._extreme("min", axis, out, explicit)

    def _arg(self, op, axis, out, explicit):
        axis = self._check_reduction(axis, op)
        if out is not None:
            raise ValueError(f"Sparse {op} does not support an 'out' parameter.")
        m, n = self.shape
        if axis is None and m * n == 0:
            raise ValueError(f"Cannot apply {op} to an empty matrix.")
        if axis is not None and self.shape[axis] == 0:
            raise ValueError(f"Cannot apply {op} along a zero-sized dimension.")
        if axis is None and explicit and self.nnz == 0:
            raise ValueError(f"Cannot apply {op} to zero matrix when explicit=True.")
        runtime.require_cuda(f"csr_array.{op}")
        if axis is not None:
            return self._reduce_axis(op, axis, explicit)
        ptr_, idx, dat = self._canonical()
        ext = "max" if op == "argmax" else "min"
        vals = _ops.csr_reduce_rows(ext, ptr_, None, dat, n, explicit)
        cols = _ops.csr_reduce_rows(op, ptr_, idx, dat, n, explicit)
        # the first row (C order) holding a NaN, else the first row attaining the extreme; with `explicit`, empty rows
        # have no candidate
        keep = ptr_[1:] > ptr_[:-1] if explicit else torch.ones(m, dtype=torch.bool, device=vals.device)
        rid = torch.arange(m, device=vals.device)
        nan = keep & torch.isnan(vals)
        ok = keep & ~nan
        fill = torch.tensor(float("-inf") if ext == "max" else float("inf"), dtype=vals.dtype, device=vals.device)
        masked = torch.where(ok, vals, fill)
        g = masked.max() if ext == "max" else masked.min()
        first_nan = torch.where(nan, rid, m).min()
        first_hit = torch.where(ok & (vals == g), rid, m).min()
        i = torch.where(first_nan < m, first_nan, first_hit)
        return int((i * n + cols[i]).item())

    def argmax(self, axis=None, out=None, *, explicit=False):
        """Position of the first largest entry: for axis None the flat index i * n + j in C order (a Python int), along
        an axis an int64 CUDA tensor of column (axis 1) or row (axis 0) indices.  Implicit zeros count unless `explicit`
        (the first missing position stands for them).  NaN: the first NaN wins, numpy's rule on the dense row; scipy
        1.18 instead returns the first implicit zero of a row that holds both.  With `explicit` and axis None the result
        is still the flat index, where scipy 1.18 returns the position in its canonical data array.  `out` is not
        supported (ValueError);
        an empty matrix or a zero-length axis, and `explicit` on a matrix without stored entries (axis None), raise
        ValueError.  A column reduction keeps a transposed copy of A in A's cache, as `max` does."""
        return self._arg("argmax", axis, out, explicit)

    def argmin(self, axis=None, out=None, *, explicit=False):
        """Position of the first smallest entry; see `argmax`."""
        return self._arg("argmin", axis, out, explicit)

    def count_nonzero(self, axis=None):
        """Number of nonzero entries of A after repeated columns are summed (axis None: a Python int), or of every column
        (axis 0) / row (axis 1) as an int64 CUDA tensor.  Explicit zeros do not count; NaN does.  A column count keeps a
        transposed copy of A in A's cache, as `max` does."""
        axis = self._check_reduction(axis, "count_nonzero")
        runtime.require_cuda("csr_array.count_nonzero")
        if axis is None:
            return int((self._canonical()[2] != 0).sum().item())
        return self._reduce_axis("count_nonzero", axis)

    def __abs__(self):
        """|A| with A's structure: shares A's indptr and indices."""
        return csr_array._from_parts(self._indptr, self._indices, self._data.abs(), self.shape)

    def power(self, n, dtype=None):
        """Elementwise power of the stored values (reference csr.py:351-360), as a new csr_array sharing A's indptr and
        indices; the values are cast to `dtype` first when it is given.  n must be a nonzero scalar
        (NotImplementedError otherwise: n = 0 would make every implicit zero a one)."""
        if not np.isscalar(n):
            raise NotImplementedError("Input is not a scalar")
        if n == 0:
            raise NotImplementedError("zero power is not supported as it would densify the matrix")
        data = self._data if dtype is None else self._data.to(torch_dtype(dtype))
        return csr_array._from_parts(self._indptr, self._indices, data**n, self.shape)

    def eliminate_zeros(self):
        """Remove the explicitly stored zeros (either sign), in place."""
        keep = self._data != 0
        if bool(keep.all()):
            return
        kept = torch.zeros(self.nnz + 1, dtype=torch.int64, device=keep.device)
        torch.cumsum(keep.to(torch.int64), 0, out=kept[1:])
        self._indptr = kept[self._indptr.to(torch.int64)].to(self._indptr.dtype)
        self._indices = self._indices[keep]
        self._data = self._data[keep]
        self._cache.clear()

    @property
    def has_sorted_indices(self) -> bool:
        """True when the columns of every row are non-decreasing."""
        nnz = self.nnz
        if nnz < 2:
            return True
        drop = self._indices[1:] < self._indices[:-1]
        starts = self._indptr[1:-1].to(torch.int64)
        starts = starts[(starts > 0) & (starts < nnz)]
        drop[starts - 1] = False        # the first entry of a row is not compared with the previous row's last
        return not bool(drop.any())

    def sort_indices(self):
        """Sort the columns of every row, in place (new index / value arrays: other matrices sharing them keep theirs)."""
        if self.has_sorted_indices:
            return
        self._indices, self._data = _ops.csr_sort_rows(self._indptr, self._indices.clone(), self._data.clone())
        self._cache.clear()

    # -- indexing (scipy csr_matrix semantics; csrc/index.cu) ----------------------------------------------------------
    def __getitem__(self, key):
        """scipy-style indexing on the device.

        * `A[i, j]`, two integers: the numpy scalar sum of the entries stored at (i, j), added in stored order, or 0.
        * `A[I, J]`, two 1-D index arrays of one length k: the k element values, numpy for host indices and a CUDA tensor
          for CUDA indices, as `dot` returns.
        * `A[r]`, `A[r, :]`, `A[:, c]`, `A[r, c]`, `A[..., c]` with r and c each an int, a slice (any step), a 1-D integer
          array (any order, repeats, negatives) or a 1-D boolean mask, not both arrays; and `A[np.ix_(I, J)]`: a new
          csr_array of the outer selection.  As in scipy's csr_matrix (csr_matrix is an alias of csr_array here), an
          integer keeps its axis with length 1; scipy's csr_array would return a 1-D coo_array, a type this library
          does not have.
        Entries keep the source row's stored order; an entry whose column is requested r times appears r times, output
        columns ascending; duplicates and explicit zeros are kept.  The result holds new arrays; A is not modified.
        Index arrays may be lists, numpy arrays or tensors on either side.  Out-of-range indices, a mask of the wrong
        length, too many indices and None raise IndexError, as do float index arrays (scipy truncates them; numpy
        refuses them).  Other 2-D index arrays raise NotImplementedError, and so do lookups on data other than
        float32 / float64 (selections move values of any 4-, 8- or 16-byte type).  A selection syncs once (twice with
        a column selection: the column map is built first); CUDA row and column indices are checked on the device."""
        kind, R, C = _index_key(key, self.shape)
        if kind in ("element", "points"):
            if self.dtype not in SUPPORTED_VALUE_DTYPES:
                raise NotImplementedError(f"element lookup for dtype {self.dtype} is not implemented (float32/float64 only)")
            runtime.require_cuda("csr_array.__getitem__")
            dev = self.device
            on_device = kind == "points" and any(isinstance(a, torch.Tensor) for a in (R, C))
            ri, ci = (_index_tensor(np.asarray([a]) if kind == "element" else a, dev) for a in (R, C))
            out, bad = _ops.csr_lookup(self._indptr, self._indices, self._data, self.shape, ri, ci)
            if on_device:
                if int(bad.item()):
                    raise IndexError(f"{int(bad.item())} index pairs out of range for shape {self.shape}")
                return out
            res = to_host(out)
            return self.dtype.type(res[0]) if kind == "element" else res
        if self._data.element_size() not in (4, 8, 16):
            raise NotImplementedError(f"selection for dtype {self.dtype} is not implemented (4-, 8- or 16-byte values)")
        runtime.require_cuda("csr_array.__getitem__")
        return self._select(R, C)

    def _select(self, R, C):
        """The outer selection of `_index_key`'s row and column selections (each ("slice", start, step, count) or
        ("array", int64 indices))."""
        m, n = self.shape
        dev = self.device
        rows, start, step = None, 0, 1
        if R[0] == "slice":
            start, step, nout = R[1], R[2], R[3]
        else:
            rows = _index_tensor(R[1], dev)
            nout = int(rows.shape[0])
        col_map, ncols_out = None, n
        if C != ("slice", 0, 1, n):
            if C[0] == "slice":
                cols = torch.arange(C[1], C[1] + C[2] * C[3], C[2], dtype=torch.int64, device=dev)
            else:
                cols = _index_tensor(C[1], dev)
            ncols_out = int(cols.shape[0])
            col_ptr, col_pos, bad = _ops.csr_column_map(cols, n)
            if bad:
                raise IndexError(f"{bad} column indices out of range for {n} columns")
            col_map = (col_ptr, col_pos)
        ptr_, idx, dat, bad = _ops.csr_select(self._indptr, self._indices, self._data, self.shape, nout, rows, start,
                                              step, col_map, ncols_out, _index_dtype(ncols_out - 1))
        if bad:
            raise IndexError(f"{bad} row indices out of range for {m} rows")
        return csr_array._from_parts(ptr_.to(_indptr_dtype(int(idx.shape[0]))), idx, dat, (nout, ncols_out))

    def balance(self):
        """No-op on a single device; kept for API parity (reference base.py:198-282 re-tiles the rows by
        nnz; the multi-GPU row plan lives in dist.py)."""
        return None

    def __repr__(self):
        return (f"<{self.shape[0]}x{self.shape[1]} legate.sparse_b200 csr_array, {self.nnz} stored elements, "
                f"dtype {self.dtype}, device {self.device}>")

    def __str__(self):
        return repr(self)


csr_matrix = csr_array


def spgemm_csr_csr_csr(A: csr_array, B: csr_array) -> csr_array:
    """C = A @ B (reference builder sparse/csr.py:1317-1490). Rows of C are sorted by column."""
    runtime.require_cuda("spgemm_csr_csr_csr")
    if A.dtype not in SUPPORTED_VALUE_DTYPES:
        raise NotImplementedError(f"SpGEMM for dtype {A.dtype} is not implemented")
    a_idx, b_idx = A._indices, B._indices
    if a_idx.dtype != torch.int32 or b_idx.dtype != torch.int32:
        if max(A.shape[1], B.shape[1]) > _INT32_MAX:
            raise NotImplementedError("SpGEMM needs column counts < 2^31")
        a_idx, b_idx = a_idx.to(torch.int32), b_idx.to(torch.int32)
    a_ptr, b_ptr = A._indptr, B._indptr
    if a_ptr.dtype != b_ptr.dtype:
        a_ptr, b_ptr = a_ptr.to(torch.int64), b_ptr.to(torch.int64)
    c_ptr, c_idx, c_val, info = _ops.spgemm(a_ptr, a_idx, A._data, b_ptr, b_idx, B._data, A.shape, B.shape)
    C = csr_array._from_parts(c_ptr.to(_indptr_dtype(info["nnz"])), c_idx.to(_index_dtype(B.shape[1] - 1)), c_val,
                              (A.shape[0], B.shape[1]))
    C.spgemm_info = info
    return C


def _column_blocks(A: csr_array, ranges) -> list:
    """[block or None per (lo, hi) in `ranges`]: block q holds the entries of A whose column lies in [lo_q, hi_q), with
    global column ids and A's shape kept, or is None when there are none."""
    idx = A._indices
    nrows = A.shape[0]
    rows = _entry_rows(A._indptr)
    blocks = []
    for lo, hi in ranges:
        mask = (idx >= lo) & (idx < hi)
        nnz = int(mask.sum())
        if nnz == 0:
            blocks.append(None)
            continue
        ip = torch.zeros(nrows + 1, dtype=torch.int64, device=idx.device)
        torch.cumsum(torch.bincount(rows[mask], minlength=nrows), 0, out=ip[1:])
        blocks.append(csr_array._from_parts(ip.to(_indptr_dtype(nnz)), idx[mask].contiguous(),
                                            A._data[mask].contiguous(), A.shape))
    return blocks


def _canonical_parts(A: csr_array, rows_sorted: bool):
    """(indptr, indices, data) of A with every row sorted and each run of a repeated column summed into its first entry
    (row-sum kernel over the runs).  A's own arrays are never written: a sort works on clones, and a matrix already in
    that form is returned as it is."""
    indptr, indices, data = A._indptr, A._indices, A._data
    if not rows_sorted and not A.has_sorted_indices:
        indices, data = _ops.csr_sort_rows(indptr, indices.clone(), data.contiguous().clone())
    nnz = int(data.shape[0])
    if nnz < 2:
        return indptr, indices, data
    same = indices[1:] == indices[:-1]
    starts = indptr[1:-1].to(torch.int64)
    starts = starts[(starts > 0) & (starts < nnz)]
    same[starts - 1] = False        # a row's first entry starts a run whatever the previous row ends with
    if not bool(same.any()):
        return indptr, indices, data
    head = torch.ones(nnz, dtype=torch.bool, device=data.device)
    head[1:] = ~same
    heads = torch.nonzero(head).reshape(-1)
    run_ptr = torch.cat([heads, heads.new_full((1,), nnz)])
    merged = _ops.csr_reduce_rows("sum", run_ptr, None, data, A.shape[1])
    runs_before = torch.zeros(nnz + 1, dtype=torch.int64, device=data.device)
    torch.cumsum(head.to(torch.int64), 0, out=runs_before[1:])
    return runs_before[indptr.to(torch.int64)].to(indptr.dtype), indices[heads], merged


def _axis_index(x, n: int):
    """One axis of an index key, for an axis of length n: ("int", i) with 0 <= i < n, ("slice", start, step, count), or
    ("array", indices) -- an int64 numpy array wrapped into [0, n), or an int64 CUDA tensor left as given (the kernels
    wrap and check it).  Masks become the positions of their True entries."""
    if isinstance(x, (bool, np.bool_)):
        raise IndexError("a boolean scalar is not a valid index")
    if isinstance(x, (int, np.integer)):
        i = int(x)
        if not -n <= i < n:
            raise IndexError(f"index ({i}) out of range for an axis of length {n}")
        return ("int", i + n if i < 0 else i)
    if isinstance(x, slice):
        start, stop, step = x.indices(n)        # ValueError for a zero step, as scipy
        count = len(range(start, stop, step))
        return ("slice", start if count else 0, step, count)
    if isinstance(x, torch.Tensor) and x.is_cuda:
        if x.ndim == 0:
            return _axis_index(x.item(), n)
        if x.ndim != 1:
            raise NotImplementedError("index arrays must be 1-D, or the pair np.ix_ makes")
        if x.dtype == torch.bool:
            if x.shape[0] != n:
                raise IndexError(f"boolean index of length {x.shape[0]} for an axis of length {n}")
            return ("array", torch.nonzero(x).reshape(-1))
        if not _is_integer_dtype(x.dtype):
            raise IndexError(f"arrays used as indices must be of integer (or boolean) type, got {x.dtype}")
        return ("array", x.to(torch.int64))
    a = x.numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    if a.ndim == 0:
        if a.dtype.kind in "iu":
            return _axis_index(int(a), n)
        raise IndexError(f"only integers, slices, ellipsis and integer or boolean arrays are valid indices, got {x!r}")
    if a.ndim != 1:
        raise NotImplementedError("index arrays must be 1-D, or the pair np.ix_ makes")
    if a.size == 0 and a.dtype.kind == "f":
        a = a.astype(np.int64)               # [] is an empty index
    if a.dtype.kind == "b":
        if a.size != n:
            raise IndexError(f"boolean index of length {a.size} for an axis of length {n}")
        return ("array", np.flatnonzero(a).astype(np.int64))
    if a.dtype.kind not in "iu":
        raise IndexError(f"arrays used as indices must be of integer (or boolean) type, got {a.dtype}")
    a = a.astype(np.int64)
    if a.size and (a.min() < -n or a.max() >= n):
        bad = a[(a < -n) | (a >= n)][0]
        raise IndexError(f"index ({bad}) out of range for an axis of length {n}")
    return ("array", np.where(a < 0, a + n, a))


def _ndim(x):
    return x.ndim if isinstance(x, (np.ndarray, torch.Tensor)) else np.ndim(x) if isinstance(x, list) else 0


def _index_key(key, shape):
    """The host half of `csr_array.__getitem__`, touching no device: ("element", i, j) for two integers, ("points", I,
    J) for two 1-D index arrays of one length, or ("outer", R, C) with R and C each ("slice", start, step, count) or
    ("array", indices) (an integer becomes a slice of one).  Raises what scipy raises for a malformed key (see
    `csr_array.__getitem__`)."""
    m, n = shape
    parts = list(key) if isinstance(key, tuple) else [key]
    if len(parts) == 2 and all(_ndim(p) == 2 for p in parts):
        r, c = (p if isinstance(p, (np.ndarray, torch.Tensor)) else np.asarray(p) for p in parts)
        if r.shape[1] == 1 and c.shape[0] == 1:                  # np.ix_(I, J)
            R, C = _axis_index(r.reshape(-1), m), _axis_index(c.reshape(-1), n)
            return ("outer", R, C)
        raise NotImplementedError("2-D index arrays other than the pair np.ix_ makes are not supported")
    if any(p is None for p in parts):
        raise IndexError("None (newaxis) is not supported in sparse indexing")
    ell = [k for k, p in enumerate(parts) if p is Ellipsis]
    if len(ell) > 1:
        raise IndexError("an index can only have a single ellipsis ('...')")
    if ell:
        k = ell[0]
        fill = 2 - (len(parts) - 1)
        if fill < 0:
            raise IndexError("too many indices for a 2-D sparse array")
        parts = parts[:k] + [slice(None)] * fill + parts[k + 1:]
    if len(parts) > 2:
        raise IndexError("too many indices for a 2-D sparse array")
    parts += [slice(None)] * (2 - len(parts))
    R, C = _axis_index(parts[0], m), _axis_index(parts[1], n)
    if R[0] == "int" and C[0] == "int":
        return ("element", R[1], C[1])
    if R[0] == "array" and C[0] == "array":
        if R[1].shape[0] != C[1].shape[0]:
            raise IndexError(f"shape mismatch: index arrays of lengths {R[1].shape[0]} and {C[1].shape[0]}")
        return ("points", R[1], C[1])
    as_sel = lambda s: ("slice", s[1], 1, 1) if s[0] == "int" else s  # noqa: E731
    return ("outer", as_sel(R), as_sel(C))


def _index_tensor(a, device) -> torch.Tensor:
    """An int64 index array (numpy or tensor) as a contiguous int64 tensor on `device`."""
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=torch.int64).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(device)


def _check_reduction_out(out, shape, dtype):
    if out is None:
        return
    if isinstance(out, np.ndarray):
        ok = out.dtype == dtype
    elif isinstance(out, torch.Tensor):
        ok = out.dtype == torch_dtype(dtype)
    else:
        ok = False
    if not ok or tuple(out.shape) != tuple(shape):
        raise ValueError(f"out must be a numpy array or torch tensor of shape {tuple(shape)} and dtype {dtype}")


def _deliver_scalar(value, out):
    if out is None:
        return value
    if isinstance(out, torch.Tensor):
        out.fill_(float(value))
    else:
        out[...] = value
    return out


def _is_integer_dtype(dt) -> bool:
    if isinstance(dt, torch.dtype):
        return not (dt.is_floating_point or dt.is_complex or dt == torch.bool)
    return np.dtype(dt).kind in "iu"


def _overlaps(a, b) -> bool:
    """True when the memory ranges of two arrays intersect: numpy arrays and CPU tensors in host memory, or tensors on
    one device."""
    def span(t):
        if isinstance(t, np.ndarray):
            if t.size == 0:
                return None
            lo, hi = np.lib.array_utils.byte_bounds(t)
            return "cpu", lo, hi
        if t.numel() == 0:
            return None
        lo = t.data_ptr()
        return str(t.device), lo, lo + (sum((s - 1) * st for s, st in zip(t.shape, t.stride())) + 1) * t.element_size()

    sa, sb = span(a), span(b)
    return sa is not None and sb is not None and sa[0] == sb[0] and sa[1] < sb[2] and sb[1] < sa[2]


def _as_sparse_operand(other):
    """`other` as a csr_array when it is a sparse matrix (csr_array, coo_array, what diags() returns, scipy.sparse),
    else None."""
    if isinstance(other, csr_array):
        return other
    if scipy.sparse.issparse(other):
        return csr_array(other)
    if hasattr(other, "tocsr") and not isinstance(other, (np.ndarray, torch.Tensor)):
        csr = other.tocsr()
        if isinstance(csr, csr_array):
            return csr
    return None


def _csr_binop(A: csr_array, B: csr_array, op: str) -> csr_array:
    """C = A op B (op "add" / "sub" / "mul") for operands of one shape and dtype: the row merge of csrc/elementwise.cu.
    Operands with a decreasing row are merged from sorted copies; their own arrays are left as they are."""
    runtime.require_cuda(f"csr_array {op}")
    a_ptr, b_ptr, a_idx, b_idx = A._indptr, B._indptr, A._indices, B._indices
    if a_ptr.dtype != b_ptr.dtype:
        a_ptr, b_ptr = a_ptr.to(torch.int64), b_ptr.to(torch.int64)
    if a_idx.dtype != b_idx.dtype:
        a_idx, b_idx = a_idx.to(torch.int64), b_idx.to(torch.int64)
    a_val, b_val = A._data, B._data
    c_ptr, c_idx, c_val, info = _ops.csr_binop(op, a_ptr, a_idx, a_val, b_ptr, b_idx, b_val, A.shape)
    if c_idx is None:
        if info["a_unsorted"]:
            a_idx, a_val = _ops.csr_sort_rows(a_ptr, a_idx.clone(), a_val.clone())
        if info["b_unsorted"]:
            b_idx, b_val = _ops.csr_sort_rows(b_ptr, b_idx.clone(), b_val.clone())
        c_ptr, c_idx, c_val, info = _ops.csr_binop(op, a_ptr, a_idx, a_val, b_ptr, b_idx, b_val, A.shape)
        assert c_idx is not None, "row sort left a decreasing row"
    if c_idx.dtype == torch.int64 or _force_wide():     # an int32 result keeps its width
        c_idx = c_idx.to(_index_dtype(A.shape[1] - 1))
    return csr_array._from_parts(c_ptr.to(_indptr_dtype(info["nnz"])), c_idx, c_val, A.shape)


def spgemm_chunked(A: csr_array, B: csr_array, max_products: int = 1 << 31, keep: bool = False, on_chunk=None):
    """C = A @ B computed in ROW CHUNKS of A so that the output of one chunk fits a memory budget -- how BASELINE
    config 5 (R-MAT scale 22 squared: nnz(C) is hundreds of GB) runs on one 80 GB GPU.

    A cheap pass counts the products of every row (`b2s_spgemm_row_work`, an upper bound of the row's nnz); rows are
    cut greedily into ranges of <= `max_products` products (a single heavier row is its own chunk); each range is a
    CSR matrix in its own right (indptr slice rebased, contiguous indices / vals slice) and goes through the two-pass
    SpGEMM of `spgemm_csr_csr_csr`.  A chunk of C is handed to `on_chunk(row_lo, row_hi, C_chunk)` and dropped, or
    kept and concatenated when `keep` (only if everything fits).  The reference sizes its output with a blocking
    `int(nnz)` and a single allocation (sparse/csr.py:1442); it cannot run this case on one GPU either.

    Returns (C or None, stats) with stats = {chunks, products, nnz, rows_per_chunk, checksum (sum of all values,
    fp64), max_chunk_nnz}."""
    runtime.require_cuda("spgemm_chunked")
    assert A.shape[1] == B.shape[0]
    m = A.shape[0]
    a_idx = A._indices if A._indices.dtype == torch.int32 else A._indices.to(torch.int32)
    a_ptr, b_ptr = A._indptr, B._indptr
    if a_ptr.dtype != b_ptr.dtype:
        a_ptr, b_ptr = a_ptr.to(torch.int64), b_ptr.to(torch.int64)
    work = _ops.spgemm_row_work(a_ptr, a_idx, b_ptr)
    cum = torch.cumsum(work, 0).cpu().numpy() if m else np.zeros(0, dtype=np.int64)
    cuts = [0]
    while cuts[-1] < m:
        base = int(cum[cuts[-1] - 1]) if cuts[-1] > 0 else 0
        nxt = int(np.searchsorted(cum, base + int(max_products), side="right"))
        cuts.append(min(max(nxt, cuts[-1] + 1), m))
    del work
    parts = []
    stats = {"chunks": 0, "products": int(cum[-1]) if m else 0, "nnz": 0, "checksum": 0.0, "max_chunk_nnz": 0,
             "rows_per_chunk": []}
    ip_host = A._indptr.cpu().numpy() if m else np.zeros(1, dtype=np.int64)
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        klo, khi = int(ip_host[lo]), int(ip_host[hi])
        Ac = csr_array._from_parts((A._indptr[lo : hi + 1] - klo).contiguous(), A._indices[klo:khi], A._data[klo:khi],
                                   (hi - lo, A.shape[1]))
        Cc = spgemm_csr_csr_csr(Ac, B)
        stats["chunks"] += 1
        stats["nnz"] += Cc.nnz
        stats["max_chunk_nnz"] = max(stats["max_chunk_nnz"], Cc.nnz)
        stats["rows_per_chunk"].append(hi - lo)
        stats["checksum"] += float(Cc._data.sum(dtype=torch.float64)) if Cc.nnz else 0.0
        if on_chunk is not None:
            on_chunk(lo, hi, Cc)
        if keep:
            parts.append(Cc)
        del Cc, Ac
    C = None
    if keep:
        ptrs, off = [torch.zeros(1, dtype=torch.int64, device=A.device)], 0
        for P_ in parts:
            ptrs.append(P_._indptr[1:].to(torch.int64) + off)
            off += P_.nnz
        indptr = torch.cat(ptrs).to(_indptr_dtype(off))
        C = csr_array._from_parts(indptr, torch.cat([P_._indices for P_ in parts]) if parts else A._indices[:0],
                                  torch.cat([P_._data for P_ in parts]) if parts else A._data[:0], (m, B.shape[1]))
    return C, stats
