"""`dia_array` -- diagonal-format matrices (reference sparse/dia.py).

A DIA matrix A (m x n) stores ndiag diagonals: `offsets` k_d and an ndiag x L array `data`, column-aligned as in scipy,
so entry (r, r + k_d) is data[d, r + k_d], stored when 0 <= r < m and 0 <= r + k_d < min(n, L).  `data` is a device
tensor; the offsets live on the host (`_offsets`), where every shape computation reads them without touching the
device, and go to the device as int64 once per stamp of `data`.

Products with a dense operand run the row-owned kernels of csrc/dia.cu (b2s_spmv_dia, b2s_spmm_dia): each output row
sums its diagonals in stored order, with no atomics and no plan, so two calls give identical results.  `A.tocsr()` is
the device conversion (b2s_dia_to_csr), cached, and carries its own SpMV plan; sparse products, elementwise arithmetic
with sparse or dense operands, SDDMM and the reductions are the CSR operations of that cached form.  Scalar products,
negation and `abs` act on `data` and stay DIA, as in scipy.
"""
from __future__ import annotations

import warnings

import numpy as np
import scipy.sparse
import torch

from . import _ops
from .csr import _dense_rows, _index_dtype, _indptr_dtype, csr_array
from .runtime import SUPPORTED_VALUE_DTYPES, numpy_dtype, runtime, to_device, to_host, torch_dtype

_DIA_WARN_DIAGONALS = 100   # scipy's coo.todia warns above this many diagonals


class dia_array:
    """DIA matrix resident on one GPU (or, with no GPU visible, on the host for format logic)."""

    ndim = 2
    format = "dia"
    __array_priority__ = 10.1  # like scipy.sparse: `ndarray @ A` defers to A.__rmatmul__

    def __init__(self, arg, shape=None, dtype=None, copy=False):
        from .coo import coo_array
        from .csc import csc_array

        if isinstance(arg, torch.Tensor) and arg.ndim == 2:
            arg = to_host(arg)
        if isinstance(arg, dia_array):
            data, offsets, shape_ = arg._data.clone() if copy else arg._data, arg._offsets, arg.shape
        elif isinstance(arg, (csr_array, csc_array, coo_array)):
            A = arg.todia()
            data, offsets, shape_ = A._data, A._offsets, A.shape
        elif scipy.sparse.issparse(arg):
            A = arg.todia()
            data, offsets, shape_ = A.data, A.offsets, A.shape
        elif isinstance(arg, tuple) and len(arg) == 2 and all(np.isscalar(s) for s in arg):
            shape_ = arg   # an empty (M, N) matrix
            data, offsets = np.zeros((0, 0), dtype=np.float64 if dtype is None else dtype), np.zeros(0, np.int64)
        elif isinstance(arg, tuple):
            try:
                data, offsets = arg
            except Exception as e:
                raise ValueError("unrecognized form for dia_array constructor") from e
            if shape is None:
                raise ValueError("expected a shape argument")
            shape_ = shape
            if not isinstance(data, torch.Tensor):
                data = np.atleast_2d(np.array(data, copy=copy or None))
            elif data.ndim < 2:
                data = data.reshape(1, -1)
            elif copy:
                data = data.clone()
            offsets = np.atleast_1d(np.asarray(to_host(offsets)))
        else:
            a = np.asarray(arg)
            if a.ndim != 2:
                raise ValueError(f"DIA arrays don't support {a.ndim}D input. Use 2D")
            A = scipy.sparse.coo_array(a).todia()
            data, offsets, shape_ = A.data, A.offsets, A.shape
        if offsets.ndim != 1:
            raise ValueError("offsets array must have rank 1")
        if data.ndim != 2:
            raise ValueError("data array must have rank 2")
        if data.shape[0] != len(offsets):
            raise ValueError(f"number of diagonals ({data.shape[0]}) does not match the number of offsets "
                             f"({len(offsets)})")
        offsets = np.asarray(offsets).astype(np.int64)
        if len(np.unique(offsets)) != len(offsets):
            raise ValueError("offset array contains duplicate values")
        if shape is not None and tuple(int(s) for s in shape) != tuple(int(s) for s in shape_):
            raise ValueError(f"shape {tuple(shape)} does not match the operand's {tuple(shape_)}")
        data = to_device(data)
        if dtype is not None and numpy_dtype(dtype) != numpy_dtype(data.dtype):
            data = data.to(torch_dtype(dtype))
        self._init(data, offsets, shape_)

    def _init(self, data, offsets, shape):
        self._data = data.contiguous()
        self._offsets = offsets
        self.shape = tuple(int(s) for s in shape)
        self._cache = {}

    @classmethod
    def _from_parts(cls, data: torch.Tensor, offsets: np.ndarray, shape) -> "dia_array":
        """A dia_array of device `data` and host int64 `offsets`, unchecked (offsets may repeat: `diags` sums them
        through `tocsr`)."""
        obj = cls.__new__(cls)
        obj._init(data, np.asarray(offsets, dtype=np.int64), shape)
        return obj

    # -- storage ----------------------------------------------------------------------------------------------------
    @property
    def data(self):
        return self._data

    @data.setter
    def data(self, value):
        value = to_device(value)
        if value.ndim != 2 or value.shape[0] != len(self._offsets):
            raise ValueError(f"data must be 2-D with {len(self._offsets)} rows, got shape {tuple(value.shape)}")
        self._data = value
        self._cache.clear()

    @property
    def offsets(self):
        """The offsets as a new int64 device tensor: editing it does not change the matrix."""
        return to_device(self._offsets, copy=True)

    @property
    def dtype(self):
        return numpy_dtype(self._data.dtype)

    @property
    def device(self):
        return self._data.device

    @property
    def nnz(self) -> int:
        """Stored positions, explicit zeros included: scipy's `_getnnz`, bounded by L = data.shape[1]."""
        M, N = self.shape
        L = min(int(self._data.shape[1]), N)
        return sum(max(min(M + k, L) - max(k, 0), 0) for k in self._offsets.tolist())

    def count_nonzero(self, axis=None):
        if axis is not None:
            raise NotImplementedError("count_nonzero over an axis is not implemented for DIA format")
        return self.tocsr().nnz

    # -- what is derived from the arrays, cached ---------------------------------------------------------------------
    def _stamp(self):
        """Pointer and version counter of `data`: an in-place edit changes it, and assigning `data` clears `_cache`.
        The offsets never change after construction."""
        return self._data.data_ptr(), self._data._version

    def _derived(self, kind, extra, build):
        """As `csr_array._derived`: `build()` runs again whenever the stamp or `extra` differs from the cached one."""
        stamp = self._stamp()
        hit = self._cache.get(kind)
        if hit is None or hit[0] != stamp or hit[1] != extra:
            hit = self._cache[kind] = (stamp, extra, build())
        return hit[2]

    def _in_band(self):
        """(offsets, data) restricted to the diagonals that meet the band -- -m < k < min(n, L) -- with the offsets as
        an int64 device tensor.  Offsets out of band, however large, never reach a kernel."""
        def build():
            m, n = self.shape
            lim = min(n, int(self._data.shape[1]))
            keep = (self._offsets > -m) & (self._offsets < lim)
            data = self._data if keep.all() else self._data[torch.from_numpy(keep).to(self._data.device)]
            return to_device(self._offsets[keep]), data.contiguous()
        return self._derived("in_band", None, build)

    def _promoted(self, common) -> "dia_array":
        return self._derived(("promoted", common), None, lambda: self.astype(common, copy=False))

    # -- conversions ------------------------------------------------------------------------------------------------
    def copy(self):
        return dia_array._from_parts(self._data.clone(), self._offsets.copy(), self.shape)

    def astype(self, dtype, casting="unsafe", copy=True):
        dtype = np.dtype(dtype)
        if not copy and dtype == self.dtype:
            return self
        return dia_array._from_parts(self._data.to(torch_dtype(dtype), copy=copy), self._offsets.copy(), self.shape)

    def conj(self, copy=True):
        if self.dtype.kind == "c":
            return dia_array._from_parts(self._data.conj().resolve_conj(), self._offsets.copy(), self.shape)
        return self.copy() if copy else self

    def todia(self, copy=False):
        return self.copy() if copy else self

    def tocsr(self, copy=False):
        """The CSR form, zeros dropped and columns sorted (b2s_dia_to_csr for float32 / float64 on the GPU, tensor
        operations otherwise).  Built once per stamp of `data` and shared between calls (it also carries its own SpMV
        plan); `copy=True` gives arrays of your own."""
        A = self._derived("csr", None, self._tocsr)
        return A.copy() if copy else A

    def _tocsr(self) -> csr_array:
        offsets, data = self._in_band()
        if runtime.has_cuda and data.is_cuda and data.dtype in (torch.float32, torch.float64):
            m, n = self.shape
            order = torch.sort(offsets, stable=True).indices
            idx_dt = _index_dtype(n - 1)
            indptr, indices, vals = _ops.dia_to_csr(offsets, order, data, self.shape, _indptr_dtype(self.nnz), idx_dt)
            nnz = int(vals.shape[0])
            if idx_dt == torch.int64:   # the width the largest column present needs, as the tensor route gives
                indices = indices.to(_index_dtype(int(indices.max()) if nnz else 0))
            return csr_array._from_parts(indptr.to(_indptr_dtype(nnz)), indices, vals, self.shape)
        return self._tocsr_tensor_ops()

    def _tocsr_tensor_ops(self) -> csr_array:
        """The CSR form for other dtypes, or with no GPU: the arrays b2s_dia_to_csr gives, through tensor operations
        over the diagonals in ascending offset order."""
        m, n = self.shape
        offsets, data = self._in_band()
        order = torch.sort(offsets, stable=True).indices
        lim = min(n, int(data.shape[1]))
        dev = data.device
        rows_l, cols_l, vals_l = [], [], []
        for d, k in zip(order.tolist(), offsets[order].tolist()):
            j = torch.arange(max(k, 0), min(m + k, lim), dtype=torch.int64, device=dev)
            v = data[d, j]
            keep = v != 0
            rows_l.append(j[keep] - k)
            cols_l.append(j[keep])
            vals_l.append(v[keep])
        if rows_l:
            rows, cols, vals = torch.cat(rows_l), torch.cat(cols_l), torch.cat(vals_l)
        else:
            rows = cols = torch.zeros(0, dtype=torch.int64, device=dev)
            vals = torch.zeros(0, dtype=data.dtype, device=dev)
        rank = torch.sort(rows, stable=True).indices
        rows, cols, vals = rows[rank], cols[rank], vals[rank]
        nnz = int(vals.shape[0])
        indptr = torch.zeros(m + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.bincount(rows, minlength=m), 0, out=indptr[1:])
        return csr_array._from_parts(indptr.to(_indptr_dtype(nnz)),
                                     cols.to(_index_dtype(int(cols.max()) if nnz else 0)), vals.contiguous(),
                                     self.shape)

    def tocsc(self, copy=False):
        from .csc import csc_array

        return csc_array(self.tocsr())

    def tocoo(self, copy=False):
        return self.tocsr().tocoo(copy=True)

    def to_scipy_sparse_dia(self):
        """The scipy dia_array on the host.  Diagonals outside the band hold nothing and are left out, so offsets
        beyond scipy's index width cannot wrap around."""
        offsets, data = self._in_band()
        return scipy.sparse.dia_array((to_host(data), to_host(offsets)), shape=self.shape)

    def todense(self, order=None, out=None):
        if order is not None:
            raise NotImplementedError
        res = self.to_scipy_sparse_dia().toarray()
        if out is not None:
            out[...] = res
            return out
        return res

    toarray = todense

    def asformat(self, format, copy=False):
        if format in (None, "dia"):
            return self.copy() if copy else self
        if format == "csr":
            return self.tocsr(copy=copy)
        if format == "csc":
            return self.tocsc(copy=copy)
        if format == "coo":
            return self.tocoo(copy=copy)
        raise NotImplementedError(f"format {format!r}")

    def transpose(self, copy=False):
        """Aᵀ as a dia_array: offsets negated, each diagonal re-aligned to the columns of Aᵀ (L = m), as scipy does;
        positions out of band are zero.  (scipy 1.18.1 wraps its index around when L > max(m, n) and returns a
        different matrix there; this is the transpose in every case.)"""
        m, n = self.shape
        ndiag, L = self._data.shape
        lim = min(n, L)
        dev = self._data.device
        k = torch.from_numpy(np.clip(self._offsets, -m, lim)).to(dev)   # clipped: no overflow, and out of band stays out
        j = torch.arange(m, dtype=torch.int64, device=dev)[None, :] + k[:, None]
        valid = (j >= 0) & (j < lim)
        data = torch.gather(self._data, 1, j.clamp(0, max(L - 1, 0))) if L else self._data.new_zeros((ndiag, m))
        data = torch.where(valid, data, torch.zeros((), dtype=data.dtype, device=dev))
        return dia_array._from_parts(data.contiguous(), -self._offsets, (n, m))

    T = property(transpose)

    def diagonal(self, k=0):
        """Diagonal k as a device vector: a slice of `data`, zero-padded past L, empty when k is outside the matrix."""
        rows, cols = self.shape
        if k <= -rows or k >= cols:
            return self._data.new_zeros(0)
        first, last = max(0, k), min(rows + k, cols)
        out = self._data.new_zeros(last - first)
        idx = np.nonzero(self._offsets == k)[0]
        if idx.size:
            seg = self._data[int(idx[0]), first:last]
            out[: seg.shape[0]] = seg
        return out

    # -- products -----------------------------------------------------------------------------------------------------
    def dot(self, other, out=None):
        """`A.dot(x)` / `A @ B`.

        * x 1-D or (n, 1), numpy or torch CUDA tensor: y = A x on b2s_spmv_dia, with x's array kind and shape.
        * dense (n, k): Y = A X on b2s_spmm_dia, (m, k) of the same array kind.
        * a sparse matrix: the CSR SpGEMM of `tocsr()` with it, a csr_array.
        `out` (numpy or torch, the result's shape and resolved dtype) receives the result.  The resolved dtype is
        np.result_type of A and x; float32 and float64 run the kernels, a complex operand runs the real SpMM on the
        (re, im)-interleaved view (a complex A runs the complex CSR path of `tocsr()`), and anything else raises
        NotImplementedError."""
        from .csc import _check_out, _deliver

        B = _as_csr_operand(other)
        if B is not None:
            if out is not None:
                raise ValueError("Cannot provide out for sparse matmul.")
            if B.shape[0] != self.shape[1]:
                raise ValueError(f"dimension mismatch: {self.shape} @ {B.shape}")
            return self.tocsr().dot(B)
        x = other if isinstance(other, (np.ndarray, torch.Tensor)) else np.asarray(other)
        if x.ndim not in (1, 2):
            raise NotImplementedError("dia_array.dot: operand must be a vector, a dense 2-D array or a sparse matrix")
        if x.shape[0] != self.shape[1]:
            raise ValueError(f"dimension mismatch: {self.shape} @ {tuple(x.shape)}")
        common = np.result_type(self.dtype, numpy_dtype(x.dtype))
        if common.kind == "c":
            if self.dtype.kind == "c":
                return self.tocsr().dot(x, out=out)
            return self._dot_complex(x, out, common)
        vector = x.ndim == 1 or x.shape[1] == 1
        if common not in SUPPORTED_VALUE_DTYPES:
            raise NotImplementedError(f"{'SpMV' if vector else 'SpMM'} for resolved dtype {common} is not implemented "
                                      "(float32/float64 kernels only)")
        m, n = self.shape
        rshape = (m,) if x.ndim == 1 else (m, x.shape[1])
        _check_out(out, rshape, common)
        runtime.require_cuda("dia_array.dot")
        on_device = isinstance(x, torch.Tensor) and x.is_cuda
        offsets, data = self._promoted(common)._in_band()
        if vector:
            xd = to_device(x.reshape(-1), dtype=common)
            direct = isinstance(out, torch.Tensor) and out.is_cuda and out.is_contiguous()
            y = out.reshape(-1) if direct else torch.empty(m, dtype=torch_dtype(common), device=data.device)
            _ops.spmv_dia(offsets, data, xd, y, self.shape)
            res = y.reshape(rshape)
        else:
            X = _dense_rows(x, common)
            k = X.shape[1]
            direct = (isinstance(out, torch.Tensor) and out.is_cuda and (k <= 1 or out.stride(1) == 1)
                      and (m <= 1 or out.stride(0) >= k))
            res = out if direct else torch.empty((m, k), dtype=torch_dtype(common), device=data.device)
            _ops.spmm_dia(offsets, data, X, res, self.shape)
        return _deliver(res, out, on_device, direct)

    def _dot_complex(self, x, out, common):
        """A real A times a complex operand: the real SpMM of A on the (re, im)-interleaved view of x (twice the
        columns), which is how complex arrays sit in memory."""
        from .csc import _check_out, _deliver

        m, n = self.shape
        rdt = np.dtype(np.float32) if common == np.complex64 else np.dtype(np.float64)
        rshape = (m,) if x.ndim == 1 else (m, x.shape[1])
        _check_out(out, rshape, common)
        runtime.require_cuda("dia_array.dot")
        on_device = isinstance(x, torch.Tensor) and x.is_cuda
        X = to_device(x, dtype=common)
        k = 1 if X.ndim == 1 else X.shape[1]
        Xr = torch.view_as_real(X.reshape(n, k)).reshape(n, 2 * k)
        offsets, data = self._promoted(rdt)._in_band()
        Yr = torch.empty((m, 2 * k), dtype=Xr.dtype, device=Xr.device)
        _ops.spmm_dia(offsets, data, Xr, Yr, self.shape)
        return _deliver(torch.view_as_complex(Yr.reshape(m, k, 2)).reshape(rshape), out, on_device, False)

    def matvec(self, other):
        return self @ other

    def __matmul__(self, other):
        return self.dot(other)

    def __rmatmul__(self, other):
        """x @ A = (Aᵀ x)ᵀ: the DIA product of the cached transpose."""
        x = other if isinstance(other, (np.ndarray, torch.Tensor)) else np.asarray(other)
        At = self._derived("transpose", None, self.transpose)
        if x.ndim == 1:
            return At.dot(x)
        if x.ndim != 2:
            raise NotImplementedError
        if x.shape[1] != self.shape[0]:
            raise ValueError(f"dimension mismatch: {tuple(x.shape)} @ {self.shape}")
        if isinstance(x, torch.Tensor):
            return At.dot(x.t()).t().contiguous()
        return np.ascontiguousarray(At.dot(x.T).T)

    # -- elementwise: scalars act on data; everything else is the CSR operation of tocsr() ----------------------------
    def _arith(self, other, op: str, reverse: bool = False):
        if isinstance(other, dia_array):
            other = other.tocsr()
        return self.tocsr()._arith(other, op, reverse)

    def __add__(self, other):
        return self._arith(other, "add")

    def __radd__(self, other):
        return self._arith(other, "add", reverse=True)

    def __sub__(self, other):
        return self._arith(other, "sub")

    def __rsub__(self, other):
        return self._arith(other, "sub", reverse=True)

    def multiply(self, other):
        if np.isscalar(other):
            return self * other
        return self.tocsr().multiply(other.tocsr() if isinstance(other, dia_array) else other)

    def __mul__(self, other):
        if np.isscalar(other):
            return dia_array._from_parts(self._data * other, self._offsets.copy(), self.shape)
        return self.multiply(other)

    __rmul__ = __mul__

    def __neg__(self):
        return dia_array._from_parts(-self._data, self._offsets.copy(), self.shape)

    def __abs__(self):
        return dia_array._from_parts(self._data.abs(), self._offsets.copy(), self.shape)

    def sddmm(self, C, D):
        return self.tocsr().sddmm(C, D)

    def sum(self, axis=None, dtype=None, out=None):
        return self.tocsr().sum(axis=axis, dtype=dtype, out=out)

    def mean(self, axis=None, dtype=None, out=None):
        return self.tocsr().mean(axis=axis, dtype=dtype, out=out)

    def max(self, axis=None, out=None, *, explicit=False):
        return self.tocsr().max(axis=axis, out=out, explicit=explicit)

    def min(self, axis=None, out=None, *, explicit=False):
        return self.tocsr().min(axis=axis, out=out, explicit=explicit)

    def __repr__(self):
        return (f"<{self.shape[0]}x{self.shape[1]} legate.sparse_b200 dia_array, {self.nnz} stored elements "
                f"({len(self._offsets)} diagonals), dtype {self.dtype}, device {self.device}>")

    def __str__(self):
        return repr(self)


dia_matrix = dia_array


def _as_csr_operand(other):
    """`other` as a csr_array when it is a sparse matrix of this library or of scipy, else None."""
    from .module import is_sparse_matrix

    if isinstance(other, csr_array):
        return other
    if is_sparse_matrix(other) or scipy.sparse.issparse(other):
        return csr_array(other)
    return None


def _csr_to_dia(A: csr_array) -> dia_array:
    """The DIA form of a CSR matrix, as scipy's `todia`: offsets ascending, repeated entries summed, explicit zeros
    kept, L = largest column + 1, and a SparseEfficiencyWarning above 100 diagonals.  ValueError, before anything of
    that size is allocated, when the ndiag x L result cannot fit in device memory."""
    m, n = A.shape
    itemsize = np.dtype(A.dtype).itemsize

    def check(ndiag, L):
        if ndiag > _DIA_WARN_DIAGONALS:
            warnings.warn(f"Constructing a DIA matrix with {ndiag} diagonals is inefficient",
                          scipy.sparse.SparseEfficiencyWarning, stacklevel=4)
        need = ndiag * L * itemsize
        free = torch.cuda.mem_get_info(A.device)[0] if A.device.type == "cuda" else None
        if need >= 2**63 or (free is not None and need > free):
            raise ValueError(f"the DIA form of this {m} x {n} matrix has {ndiag} diagonals of length {L}: {need} bytes, "
                             f"more than the device's {free} free bytes")

    if runtime.has_cuda and A._data.is_cuda and A._data.dtype in (torch.float32, torch.float64):
        offsets, out = _ops.csr_to_dia(*A._canonical(), A.shape, check)
        return dia_array._from_parts(out, to_host(offsets).astype(np.int64), A.shape)
    # other dtypes, or no GPU: tensor operations, repeated entries summed by an accumulating scatter
    indptr, indices, data = A._indptr, A._indices, A._data
    rows = torch.repeat_interleave(indptr[1:].to(torch.int64) - indptr[:-1].to(torch.int64))
    cols = indices.to(torch.int64)
    diag = cols - rows
    offsets, slot = torch.unique(diag, sorted=True, return_inverse=True)
    ndiag, L = int(offsets.shape[0]), int(cols.max()) + 1 if cols.numel() else 0
    check(ndiag, L)
    out = torch.zeros((ndiag, L), dtype=data.dtype, device=data.device)
    out.index_put_((slot, cols), data, accumulate=True)
    return dia_array._from_parts(out, to_host(offsets).astype(np.int64), A.shape)
