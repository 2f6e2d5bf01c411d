"""`csc_array` -- compressed-column matrices (reference sparse/csc.py).

A CSC matrix A (m x n) has the same three arrays as the CSR matrix of its transpose: indptr over the n columns, row
ids in `indices`, values in `data`.  So a `csc_array` holds that `csr_array` of Aᵀ, `_T`, and nothing else: the arrays,
the cache stamp, the promoted copies and the SpMV plan all live there, and the CSC layout does not leak out of this
class.  `A.T` is `_T` itself, free, as in scipy and the reference.

Products with a dense operand run the scatter kernels of csrc/csc.cu (b2s_spmv_csc, b2s_spmm_csc): every stored entry
adds its product into the output with an atomic, so a row that receives three or more terms may differ in the last bits
between calls.  The deterministic alternatives are `A.tocsr() @ x` (the tuned CSR SpMV, its plan cached with the CSR
copy) and `x @ A`, which is the CSR product of `_T`.  Sparse products, elementwise arithmetic, SDDMM and the reductions
are the CSR operations of `_T`, with operands and axes transposed.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse
import torch

from . import _ops
from .coo import coo_array
from .csr import _dense_rows, csr_array
from .dia import dia_array
from .runtime import SUPPORTED_VALUE_DTYPES, numpy_dtype, runtime, to_device, to_host, torch_dtype


def _swap_axis(axis):
    """The axis of Aᵀ that a reduction of A over `axis` runs on; anything that is not 0, 1, -2 or -1 is passed on
    unchanged, for `csr_array` to reject."""
    if isinstance(axis, (int, np.integer)) and not isinstance(axis, (bool, np.bool_)) and -2 <= axis <= 1:
        return 1 - int(axis) % 2
    return axis


class csc_array:
    """CSC matrix resident on one GPU (or, with no GPU visible, on the host for format logic)."""

    ndim = 2
    format = "csc"
    __array_priority__ = 10.1  # like scipy.sparse: `ndarray @ A` defers to A.__rmatmul__

    def __init__(self, arg, shape=None, dtype=None, copy=False):
        if isinstance(arg, torch.Tensor) and arg.ndim == 2:
            arg = to_host(arg)
        if isinstance(arg, np.ndarray):
            if arg.ndim != 2:
                raise ValueError(f"a dense operand must be 2-D, got {arg.ndim}-D")
            T = csr_array(arg.T)
        elif isinstance(arg, csc_array):
            T = arg._T.copy() if copy else arg._T
        elif isinstance(arg, csr_array):
            T = arg.transpose()
        elif isinstance(arg, coo_array):
            T = arg.transpose().tocsr()
        elif isinstance(arg, dia_array):
            T = arg.tocsr().transpose()
        elif isinstance(arg, tuple):
            if shape is None:
                raise AssertionError("Cannot infer shape in this case.")
            m, n = (int(s) for s in shape)
            if len(arg) == 2:
                data, (row, col) = arg
                T = coo_array((data, (col, row)), shape=(n, m)).tocsr()
            elif len(arg) == 3:
                data, indices, indptr = arg
                T = csr_array((data, indices, indptr), shape=(n, m))
                if copy:
                    T = T.copy()
            else:
                raise AssertionError
        elif scipy.sparse.issparse(arg):
            s = arg.tocsc()   # a scipy CSC keeps its arrays; csr_array copies them to the device
            T = csr_array(scipy.sparse.csr_array((s.data, s.indices, s.indptr), shape=(s.shape[1], s.shape[0])))
        else:
            raise NotImplementedError(f"csc_array from {type(arg).__name__}")
        if shape is not None and tuple(int(s) for s in shape) != (T.shape[1], T.shape[0]):
            raise ValueError(f"shape {tuple(shape)} does not match the operand's {(T.shape[1], T.shape[0])}")
        if dtype is not None and numpy_dtype(dtype) != T.dtype:
            T = T.astype(dtype, copy=False)
        self._T = T

    @classmethod
    def _wrap(cls, T: csr_array) -> "csc_array":
        """The CSC matrix whose transpose is the CSR matrix T (no copy)."""
        obj = cls.__new__(cls)
        obj._T = T
        return obj

    # -- storage: the arrays of the transpose ----------------------------------------------------------------------
    @property
    def data(self):
        return self._T.data

    @data.setter
    def data(self, value):
        self._T.data = value

    @property
    def indices(self):
        return self._T.indices

    @property
    def indptr(self):
        return self._T.indptr

    @property
    def nnz(self) -> int:
        return self._T.nnz

    @property
    def shape(self):
        return (self._T.shape[1], self._T.shape[0])

    @property
    def dtype(self):
        return self._T.dtype

    @property
    def device(self):
        return self._T.device

    # -- conversions --------------------------------------------------------------------------------------------------
    def tocsc(self, copy=False):
        return self.copy() if copy else self

    def copy(self):
        return csc_array._wrap(self._T.copy())

    def astype(self, dtype, casting="unsafe", copy=True):
        return csc_array._wrap(self._T.astype(dtype, casting=casting, copy=copy))

    def conj(self, copy=True):
        return csc_array._wrap(self._T.conj(copy=copy))

    def tocsr(self, copy=False):
        """The CSR form: `b2s_csr_transpose` of the stored arrays, sorted and on the device.  Built once per stamp of the
        arrays and shared between calls (it also carries its own SpMV plan); `copy=True` gives arrays of your own."""
        A = self._T._derived("transpose", None, self._T.transpose)
        return A.copy() if copy else A

    def tocoo(self, copy=False):
        return self._T.tocoo(copy=copy).transpose()

    def todia(self, copy=False):
        """The DIA form: that of `tocsr()` (b2s_csr_to_dia), new arrays whatever `copy` says."""
        return self.tocsr().todia()

    def to_scipy_sparse_csc(self):
        return scipy.sparse.csc_array((to_host(self.data), to_host(self.indices), to_host(self.indptr)),
                                      shape=self.shape, dtype=self.dtype)

    def todense(self, order=None, out=None):
        if order is not None:
            raise NotImplementedError
        res = self.to_scipy_sparse_csc().toarray()
        if out is not None:
            out[...] = res
            return out
        return res

    toarray = todense

    def asformat(self, format, copy=False):
        if format in (None, "csc"):
            return self.copy() if copy else self
        if format == "csr":
            return self.tocsr(copy=copy)
        if format == "coo":
            return self.tocoo(copy=copy)
        if format == "dia":
            return self.todia(copy=copy)
        raise NotImplementedError(f"format {format!r}")

    def transpose(self, copy=False):
        """Aᵀ as a csr_array: the stored arrays themselves (a copy with `copy`)."""
        return self._T.copy() if copy else self._T

    T = property(transpose)

    def diagonal(self, k=0):
        return self._T.diagonal(k)

    # -- products -----------------------------------------------------------------------------------------------------
    def dot(self, other, out=None):
        """`A.dot(x)` / `A @ B`.

        * x 1-D or (n, 1), numpy or torch CUDA tensor: y = A x on b2s_spmv_csc, with x's array kind and shape.
        * dense (n, k): Y = A X on b2s_spmm_csc, (m, k) of the same array kind.
        * a sparse matrix: a csc_array, the CSR SpGEMM (AB)ᵀ = BᵀAᵀ of the stored transposes.
        `out` (numpy or torch, the result's shape and resolved dtype) receives the result.  The resolved dtype is
        np.result_type of A and x; float32 and float64 run the kernels, complex operands run the real SpMM on the
        (re, im)-interleaved view (a complex A runs the complex CSR path of `tocsr()`), and anything else raises
        NotImplementedError."""
        B = _as_csc_operand(other)
        if B is not None:
            if out is not None:
                raise ValueError("Cannot provide out for sparse matmul.")
            if B.shape[0] != self.shape[1]:
                raise ValueError(f"dimension mismatch: {self.shape} @ {B.shape}")
            return csc_array._wrap(B._T.dot(self._T))
        x = other if isinstance(other, (np.ndarray, torch.Tensor)) else np.asarray(other)
        if x.ndim not in (1, 2):
            raise NotImplementedError("csc_array.dot: operand must be a vector, a dense 2-D array or a sparse matrix")
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
        runtime.require_cuda("csc_array.dot")
        on_device = isinstance(x, torch.Tensor) and x.is_cuda
        S = self._T._promoted(common)
        if vector:
            xd = to_device(x.reshape(-1), dtype=common)
            direct = isinstance(out, torch.Tensor) and out.is_cuda and out.is_contiguous()
            y = out.reshape(-1) if direct else torch.empty(m, dtype=torch_dtype(common), device=S.device)
            _ops.spmv_csc(S._indptr, S._indices, S._data, xd, y, self.shape)
            res = y.reshape(rshape)
        else:
            X = _dense_rows(x, common)
            k = X.shape[1]
            direct = (isinstance(out, torch.Tensor) and out.is_cuda and (k <= 1 or out.stride(1) == 1)
                      and (m <= 1 or out.stride(0) >= k))
            res = out if direct else torch.empty((m, k), dtype=torch_dtype(common), device=S.device)
            _ops.spmm_csc(S._indptr, S._indices, S._data, X, res, self.shape)
        return _deliver(res, out, on_device, direct)

    def _dot_complex(self, x, out, common):
        """A real A times a complex operand: the real SpMM of A on the (re, im)-interleaved view of x (twice the
        columns), which is how complex arrays sit in memory."""
        m, n = self.shape
        rdt = np.dtype(np.float32) if common == np.complex64 else np.dtype(np.float64)
        rshape = (m,) if x.ndim == 1 else (m, x.shape[1])
        _check_out(out, rshape, common)
        runtime.require_cuda("csc_array.dot")
        on_device = isinstance(x, torch.Tensor) and x.is_cuda
        X = to_device(x, dtype=common)
        k = 1 if X.ndim == 1 else X.shape[1]
        Xr = torch.view_as_real(X.reshape(n, k)).reshape(n, 2 * k)
        S = self._T._promoted(rdt)
        Yr = torch.empty((m, 2 * k), dtype=Xr.dtype, device=Xr.device)
        _ops.spmm_csc(S._indptr, S._indices, S._data, Xr, Yr, self.shape)
        return _deliver(torch.view_as_complex(Yr.reshape(m, k, 2)).reshape(rshape), out, on_device, False)

    def matvec(self, other):
        return self @ other

    def __matmul__(self, other):
        return self.dot(other)

    def __rmatmul__(self, other):
        """x @ A = (Aᵀ x)ᵀ: the CSR SpMV / SpMM of the stored transpose, deterministic and with its cached plan."""
        x = other if isinstance(other, (np.ndarray, torch.Tensor)) else np.asarray(other)
        if x.ndim == 1:
            return self._T.dot(x)
        if x.ndim != 2:
            raise NotImplementedError
        if x.shape[1] != self.shape[0]:
            raise ValueError(f"dimension mismatch: {tuple(x.shape)} @ {self.shape}")
        if isinstance(x, torch.Tensor):
            return self._T.dot(x.t().contiguous()).t().contiguous()
        return np.ascontiguousarray(self._T.dot(np.ascontiguousarray(x.T)).T)

    # -- elementwise: the CSR operations of the transposes -------------------------------------------------------------
    def _arith(self, other, op: str, reverse: bool = False):
        if np.isscalar(other):
            return csc_array._wrap(self._T._arith(other, op, reverse))
        B = _as_csc_operand(other)
        if B is not None:
            if B.shape != self.shape:
                raise ValueError(f"inconsistent shapes {self.shape} and {B.shape}")
            return csc_array._wrap(self._T._arith(B._T, op, reverse))
        if isinstance(other, (np.ndarray, torch.Tensor)):
            return self.tocsr()._arith(other, op, reverse)   # dense result
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
        """Elementwise product: with a sparse operand the intersection of the structures (a csc_array), with a dense one
        `tocsr().multiply(other)`."""
        if np.isscalar(other):
            return self * other
        B = _as_csc_operand(other)
        if B is not None:
            if B.shape != self.shape:
                raise ValueError(f"inconsistent shapes {self.shape} and {B.shape}")
            return csc_array._wrap(self._T.multiply(B._T))
        return self.tocsr().multiply(other)

    def __mul__(self, other):
        if np.isscalar(other):
            return csc_array._wrap(self._T * other)
        return self.multiply(other)

    __rmul__ = __mul__

    def __neg__(self):
        return csc_array._wrap(-self._T)

    def __abs__(self):
        return csc_array._wrap(abs(self._T))

    def power(self, n, dtype=None):
        return csc_array._wrap(self._T.power(n, dtype=dtype))

    def eliminate_zeros(self):
        self._T.eliminate_zeros()

    def sort_indices(self):
        """Sort the rows of every column, in place."""
        self._T.sort_indices()

    @property
    def has_sorted_indices(self) -> bool:
        return self._T.has_sorted_indices

    def sddmm(self, C, D):
        """A ⊙ (C @ D) on A's stored entries, for C (m, k) and D (k, n): the CSR SDDMM of Aᵀ with Dᵀ and Cᵀ.  The result
        shares A's indptr and indices; see `csr_array.sddmm`."""
        Cx = C if isinstance(C, (np.ndarray, torch.Tensor)) else np.asarray(C)
        Dx = D if isinstance(D, (np.ndarray, torch.Tensor)) else np.asarray(D)
        if Cx.ndim != 2 or Dx.ndim != 2:
            raise ValueError(f"sddmm needs 2-D dense operands, got {Cx.ndim}-D and {Dx.ndim}-D")
        m, n = self.shape
        if Cx.shape[0] != m or Dx.shape[1] != n or Cx.shape[1] != Dx.shape[0]:
            raise ValueError(f"inconsistent shapes {self.shape}, {tuple(Cx.shape)} and {tuple(Dx.shape)} for sddmm")
        return csc_array._wrap(self._T.sddmm(Dx.T, Cx.T))

    # -- reductions: the CSR reductions of Aᵀ over the other axis ------------------------------------------------------
    def sum(self, axis=None, dtype=None, out=None):
        return self._T.sum(axis=_swap_axis(axis), dtype=dtype, out=out)

    def mean(self, axis=None, dtype=None, out=None):
        return self._T.mean(axis=_swap_axis(axis), dtype=dtype, out=out)

    def max(self, axis=None, out=None, *, explicit=False):
        return self._T.max(axis=_swap_axis(axis), out=out, explicit=explicit)

    def min(self, axis=None, out=None, *, explicit=False):
        return self._T.min(axis=_swap_axis(axis), out=out, explicit=explicit)

    def count_nonzero(self, axis=None):
        return self._T.count_nonzero(axis=_swap_axis(axis))

    def __repr__(self):
        return (f"<{self.shape[0]}x{self.shape[1]} legate.sparse_b200 csc_array, {self.nnz} stored elements, "
                f"dtype {self.dtype}, device {self.device}>")

    def __str__(self):
        return repr(self)


csc_matrix = csc_array


def _as_csc_operand(other):
    """`other` as a csc_array when it is a sparse matrix (csc_array, csr_array, coo_array, what diags() returns,
    scipy.sparse), else None."""
    if isinstance(other, csc_array):
        return other
    if isinstance(other, (csr_array, coo_array)) or scipy.sparse.issparse(other):
        return csc_array(other)
    if hasattr(other, "tocsc") and not isinstance(other, (np.ndarray, torch.Tensor)):
        csc = other.tocsc()
        if isinstance(csc, csc_array):
            return csc
    return None


def _check_out(out, shape, dtype):
    if out is None:
        return
    odt = numpy_dtype(out.dtype)
    if odt != dtype:
        raise ValueError(f"Output type {odt} is not consistent with resolved dtype {dtype}")
    if tuple(out.shape) != tuple(shape):
        raise ValueError(f"out has shape {tuple(out.shape)}, the result {tuple(shape)}")


def _deliver(res, out, on_device, direct):
    """The device result `res` in the caller's array kind: `out` when given (written unless the kernel wrote it
    directly), else a CUDA tensor for a CUDA operand and numpy otherwise."""
    if out is None:
        return res if on_device else to_host(res)
    if not direct:
        if isinstance(out, torch.Tensor):
            out.copy_(res)
        else:
            out[...] = to_host(res)
    return out
