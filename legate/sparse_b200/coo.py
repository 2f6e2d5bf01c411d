"""Minimal `coo_array`: the container `mmread` returns and the (data,(row,col)) constructor path.

The reference converts COO -> CSR with a distributed sort-by-key over NCCL (sparse/coo.py:233-347,
src/sparse/sort/sort.cu) followed by sorted-coordinates -> counts -> pos (sorted_coords_to_counts.cu,
base.py:30-48).  That is matrix assembly, the step before the SpMV/CG/SpGEMM hot path.  Here:

* host triplets (numpy, what `mmread` produces): a host-side stable sort on (row, col);
* device triplets (CUDA tensors): the same result without leaving the GPU -- one stable 64-bit key sort
  (row * ncols + col), a bincount and a prefix sum, all tensor ops on the current stream (no kernel of this
  library is involved; a multi-GPU sample sort is not implemented).

Duplicates are assumed absent in both (coo.py:73-76).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse
import torch

from .runtime import numpy_dtype, to_host


def _torch_dtype(dt):
    from .runtime import torch_dtype

    return torch_dtype(dt)


class coo_array:
    ndim = 2
    format = "coo"

    def __init__(self, arg, shape=None, dtype=None):
        self._dev = None
        if (isinstance(arg, tuple) and len(arg) == 2 and isinstance(arg[0], torch.Tensor) and arg[0].is_cuda
                and all(isinstance(t, torch.Tensor) and t.is_cuda for t in arg[1])):
            # device triplets stay on the device; the host copies below are made lazily (properties)
            data, (row, col) = arg
            if dtype is not None:
                data = data.to(_torch_dtype(dtype))
            self._dev = (data.reshape(-1), row.reshape(-1).to(torch.int64), col.reshape(-1).to(torch.int64))
            if shape is None:
                shape = (int(self._dev[1].max()) + 1, int(self._dev[2].max()) + 1)
            self._vals = self._i = self._j = None
            self.shape = tuple(int(s) for s in shape)
            self.dtype = numpy_dtype(data.dtype)
            return
        if isinstance(arg, tuple) and len(arg) == 2:
            data, (row, col) = arg
            self._vals = np.asarray(to_host(data))
            self._i = np.asarray(to_host(row)).astype(np.int64, copy=False)
            self._j = np.asarray(to_host(col)).astype(np.int64, copy=False)
            if shape is None:
                shape = (int(self._i.max()) + 1, int(self._j.max()) + 1)
        elif scipy.sparse.issparse(arg):
            c = arg.tocoo()
            self._vals, self._i, self._j = c.data, c.row.astype(np.int64), c.col.astype(np.int64)
            shape = c.shape
        else:
            raise NotImplementedError
        if dtype is not None:
            self._vals = self._vals.astype(dtype)
        self.shape = tuple(int(s) for s in shape)
        self.dtype = numpy_dtype(self._vals.dtype)

    def _host(self):
        if self._vals is None:
            self._vals, self._i, self._j = (to_host(t) for t in self._dev)
        return self._vals, self._i, self._j

    @property
    def nnz(self):
        return int(self._dev[0].shape[0]) if self._dev is not None else int(self._vals.shape[0])

    @property
    def row(self):
        return self._host()[1]

    @property
    def col(self):
        return self._host()[2]

    @property
    def data(self):
        return self._host()[0]

    def astype(self, dtype, casting="unsafe", copy=True):
        if self._dev is not None:
            return coo_array((self._dev[0].to(_torch_dtype(dtype)), (self._dev[1], self._dev[2])), shape=self.shape)
        return coo_array((self._vals.astype(dtype, casting=casting, copy=copy), (self._i, self._j)), shape=self.shape)

    def tocoo(self, copy=False):
        return self

    def _tocsr_device(self):
        """Assembly on the GPU by the library's own kernels (b2s_coo_to_csr, csrc/convert.cu): counting sort of the
        triplets by row, scan of the row counts (nnz_to_pos, reference base.py:30-48), per-row bitonic sort by column.
        Real float32/float64 values; other dtypes (complex) take the tensor-op route below."""
        from .csr import _index_dtype, _indptr_dtype, csr_array

        vals, rows, cols = self._dev
        m, n = self.shape
        ptr_dt = _indptr_dtype(vals.shape[0])
        idx_dt = _index_dtype(max(m, n))
        if vals.dtype in (torch.float32, torch.float64) and vals.is_cuda:
            from . import _ops

            indptr, indices, data = _ops.coo_to_csr(rows, cols, vals, m, ptr_dt, idx_dt)
            return csr_array._from_parts(indptr, indices, data, self.shape)
        if m * n < 2 ** 62:
            order = torch.sort(rows * n + cols, stable=True).indices
        else:  # the fused key would overflow: two stable passes, minor key first
            order = torch.sort(cols, stable=True).indices
            order = order[torch.sort(rows[order], stable=True).indices]
        rows, cols, vals = rows[order], cols[order], vals[order]
        indptr = torch.zeros(m + 1, dtype=torch.int64, device=vals.device)
        torch.cumsum(torch.bincount(rows, minlength=m), 0, out=indptr[1:])  # nnz_to_pos, reference base.py:30-48
        return csr_array._from_parts(indptr.to(ptr_dt), cols.to(idx_dt), vals.contiguous(), self.shape)

    def tocsr(self, copy=False):
        from .csr import csr_array

        if self._dev is not None:
            return self._tocsr_device()
        order = np.lexsort((self._j, self._i))  # sort by (row, col), stable
        rows, cols, vals = self._i[order], self._j[order], self._vals[order]
        counts = np.bincount(rows, minlength=self.shape[0]).astype(np.int64)
        indptr = np.zeros(self.shape[0] + 1, dtype=np.int64)
        np.cumsum(counts, out=indptr[1:])  # nnz_to_pos, reference base.py:30-48
        return csr_array((vals, cols, indptr), shape=self.shape)

    def tocsc(self, copy=False):
        from .csc import csc_array

        return csc_array(self)

    def todia(self, copy=False):
        """The DIA form of `tocsr()` (b2s_csr_to_dia on the GPU), as scipy's `todia`: repeated entries summed."""
        return self.tocsr().todia()

    def todense(self):
        vals, i, j = self._host()
        out = np.zeros(self.shape, dtype=self.dtype)
        np.add.at(out, (i, j), vals)
        return out

    toarray = todense

    def transpose(self, copy=False):
        if self._dev is not None:
            return coo_array((self._dev[0], (self._dev[2], self._dev[1])), shape=(self.shape[1], self.shape[0]))
        return coo_array((self._vals, (self._j, self._i)), shape=(self.shape[1], self.shape[0]))

    T = property(transpose)

    # products go through CSR, as in the reference (coo.py:467-477: `self.tocsr() @ other`)
    def dot(self, other, out=None):
        return self.tocsr().dot(other, out=out)

    def __matmul__(self, other):
        return self.dot(other)

    def __rmatmul__(self, other):
        return self.tocsr().__rmatmul__(other)

    def __mul__(self, other):
        if not np.isscalar(other):
            raise NotImplementedError
        if self._dev is not None:
            return coo_array((self._dev[0] * other, (self._dev[1], self._dev[2])), shape=self.shape)
        return coo_array((self._vals * other, (self._i, self._j)), shape=self.shape)

    __rmul__ = __mul__

    def asformat(self, format, copy=False):
        if format in (None, "coo"):
            return self
        if format == "csr":
            return self.tocsr()
        if format == "csc":
            return self.tocsc()
        if format == "dia":
            return self.todia()
        raise NotImplementedError(f"format {format!r}")
