"""Synthetic matrices of BASELINE.json's configs, assembled directly as `csr_array`s on the device.

Construction only (not the hot path): plain torch tensor ops.  Each generator can emit a ROW SHARD
[row_lo, row_hi) of the global matrix so a multi-GPU run never materialises the whole matrix on one
rank (the reference's examples build on CPUs then repartition; pde.py:48-196).
"""
from __future__ import annotations

import numpy as np
import torch

from .csr import _indptr_dtype, csr_array
from .runtime import runtime, torch_dtype


def _finish(indptr64, indices, data, shape, nnz):
    return csr_array._from_parts(indptr64.to(_indptr_dtype(nnz)), indices, data, shape)


def laplacian_5pt(n1: int, n2: int, dtype=np.float64, row_lo: int = 0, row_hi: int | None = None,
                  a: float | None = None, g: float | None = None) -> csr_array:
    """The operator of examples/pde.py:124-163 on an n1 x n2 interior grid (n1 = nx-2 fastest):
    offsets [-n1,-1,0,1,n1] with values [g,a,c,a,g], c = -2a-2g, the +-1 couplings removed at grid-row
    boundaries.  Defaults a = 1/dx^2, g = 1/dy^2 with dx = 1/(n1+1), dy = 1/(n2+1)."""
    dev = runtime.device
    N = n1 * n2
    row_hi = N if row_hi is None else row_hi
    a = float((n1 + 1) ** 2) if a is None else a
    g = float((n2 + 1) ** 2) if g is None else g
    c = -2.0 * a - 2.0 * g
    i = torch.arange(row_lo, row_hi, dtype=torch.int64, device=dev)
    rem = i % n1
    valid = torch.stack([i >= n1, rem != 0, torch.ones_like(i, dtype=torch.bool), rem != n1 - 1, i < N - n1], dim=1)
    cols = torch.stack([i - n1, i - 1, i, i + 1, i + n1], dim=1)
    vals = torch.tensor([g, a, c, a, g], dtype=torch_dtype(dtype), device=dev).repeat(i.shape[0], 1)
    counts = valid.sum(dim=1)
    indptr = torch.zeros(i.shape[0] + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=indptr[1:])
    indices = cols[valid].to(torch.int32)
    data = vals[valid]
    return _finish(indptr, indices, data, (row_hi - row_lo, N), int(indptr[-1]))


def banded(n: int, nnz_per_row: int = 11, dtype=np.float64, row_lo: int = 0, row_hi: int | None = None) -> csr_array:
    """examples/dot_microbenchmark.py:24-30: diags([1]*k, [-k//2..k//2], shape=(n,n), format='csr')."""
    dev = runtime.device
    row_hi = n if row_hi is None else row_hi
    i = torch.arange(row_lo, row_hi, dtype=torch.int64, device=dev)
    offs = torch.arange(nnz_per_row, dtype=torch.int64, device=dev) - (nnz_per_row // 2)
    cols = i[:, None] + offs[None, :]
    valid = (cols >= 0) & (cols < n)
    counts = valid.sum(dim=1)
    indptr = torch.zeros(i.shape[0] + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=indptr[1:])
    indices = cols[valid].to(torch.int32)
    data = torch.ones(indices.shape[0], dtype=torch_dtype(dtype), device=dev)
    return _finish(indptr, indices, data, (row_hi - row_lo, n), int(indptr[-1]))


def random_fixed(nrows: int, ncols: int, nnz_per_row: int = 32, dtype=np.float32, seed: int = 1234,
                 window: int | None = None, row_offset: int = 0, chunk: int = 1 << 20) -> csr_array:
    """BASELINE config 4: exactly `nnz_per_row` entries per row, uniform random columns (sorted within
    the row; rare duplicate columns are kept as separate entries -- their products add), N(0,1) values.
    `window` restricts row r's columns to [r - window/2, r + window/2) (clipped) -- a banded-random
    variant whose x working set stays cache resident."""
    dev = runtime.device
    gen = torch.Generator(device=dev).manual_seed(seed)
    idx_parts = []
    for lo in range(0, nrows, chunk):
        hi = min(nrows, lo + chunk)
        if window is None:
            c = torch.randint(0, ncols, (hi - lo, nnz_per_row), device=dev, generator=gen, dtype=torch.int64)
        else:
            centre = torch.arange(lo, hi, device=dev, dtype=torch.int64)[:, None] + row_offset
            base = (centre - window // 2).clamp_(0, max(ncols - window, 0))
            c = base + torch.randint(0, min(window, ncols), (hi - lo, nnz_per_row), device=dev, generator=gen,
                                     dtype=torch.int64)
        c, _ = torch.sort(c, dim=1)
        idx_parts.append(c.to(torch.int32).reshape(-1))
    indices = torch.cat(idx_parts)
    del idx_parts
    nnz = nrows * nnz_per_row
    data = torch.randn(nnz, device=dev, generator=gen, dtype=torch_dtype(dtype))
    indptr = torch.arange(0, nnz + 1, nnz_per_row, dtype=torch.int64, device=dev)
    return _finish(indptr, indices, data, (nrows, ncols), nnz)


def rmat(scale: int, edge_factor: int = 16, seed: int = 42, dtype=np.float64,
         abcd=(0.57, 0.19, 0.19, 0.05)) -> csr_array:
    """BASELINE config 5: R-MAT graph, 2^scale vertices, duplicates summed, values 1.0 before summing."""
    dev = runtime.device
    n = 1 << scale
    m = edge_factor * n
    gen = torch.Generator(device=dev).manual_seed(seed)
    a, b, c, _ = abcd
    rows = torch.zeros(m, dtype=torch.int64, device=dev)
    cols = torch.zeros(m, dtype=torch.int64, device=dev)
    for bit in range(scale):
        r = torch.rand(m, device=dev, generator=gen, dtype=torch.float64)
        right = ((r >= a) & (r < a + b)) | (r >= a + b + c)
        down = r >= a + b
        rows |= down.to(torch.int64) << bit
        cols |= right.to(torch.int64) << bit
    key = rows * n + cols
    key, counts = torch.unique(key, sorted=True, return_counts=True)
    rows, cols = key // n, key % n
    data = counts.to(torch_dtype(dtype))
    rc = torch.bincount(rows, minlength=n)
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(rc, 0, out=indptr[1:])
    return _finish(indptr, cols.to(torch.int32), data, (n, n), int(key.shape[0]))
