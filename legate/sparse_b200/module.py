"""Construction: `diags`, `eye`, `identity`, `is_sparse_matrix`, and assembly from blocks: `kron`, `kronsum`, `bmat`,
`hstack`, `vstack`, `block_diag`.

`diags`, `spdiags`, `eye` and `identity` follow the reference (sparse/module.py:96-246, sparse/dia.py:175-249): the
diagonals are laid out on the host as scipy lays them out and uploaded as a `dia_array`; their CSR and CSC forms are
its device conversion, which drops entries equal to zero (the `data != 0` mask of dia.py:236).

The block functions run on the device (csrc/construct.cu, DESIGN section 3.13): shapes, dtypes and the block table are
worked out on the host from the operands' shapes alone, and two kernels write the result without reading anything back.
They keep every stored entry -- stored order, explicit zeros, repeated columns -- and sum nothing, except `kronsum`,
which adds its two Kronecker products with the sparse add (a sum that cancels to zero stays stored).  Unlike scipy,
which returns BSR or COO by default, they return a `csr_array` for `format=None` and `"csr"`, and `result.tocoo()` for
`"coo"`; this library has no BSR type and no COO compute path, and other formats raise NotImplementedError.

`random`, `rand` and `random_array` sample uniform random sparse matrices on the device (csrc/random.cu, DESIGN section
3.16) from one 64-bit seed drawn from the caller's generator.
"""
from __future__ import annotations

import functools
import numbers
from itertools import accumulate

import numpy as np
import scipy.sparse
import torch

from . import _ops
from .coo import coo_array
from .csc import csc_array
from .csr import _csr_binop, _index_dtype, _indptr_dtype, csr_array
from .dia import dia_array
from .runtime import SUPPORTED_VALUE_DTYPES, runtime, to_device, to_host, torch_dtype


def is_sparse_matrix(o) -> bool:
    return isinstance(o, (csr_array, csc_array, coo_array, dia_array))


def _dia_data(diagonals, offsets, shape, dtype) -> np.ndarray:
    """The ndiag x L data array of `diagonals` at `offsets`, laid out as scipy.sparse.diags_array lays it out: diagonal
    k starts at column max(k, 0), and L is scipy's bound over the offsets."""
    m, n = shape
    L = max([0] + [min(m + k, n - k) + max(0, k) for k in offsets])
    data = np.zeros((len(offsets), L), dtype=dtype)
    for j, (d, k) in enumerate(zip(diagonals, offsets)):
        length = min(m + min(k, 0), n - max(k, 0))
        if length <= 0:
            continue
        d = np.asarray(d)
        if d.ndim == 0:
            d = np.full(length, d)
        if d.shape[0] < length:
            raise ValueError(f"Diagonal length (index {k}: {d.shape[0]} at offset {k}) does not agree with "
                             f"array size ({m}, {n}).")
        data[j, max(k, 0):max(k, 0) + length] = d[:length]
    return data


def diags(diagonals, offsets=0, shape=None, format=None, dtype=None):
    """scipy.sparse.diags signature (reference sparse/module.py:96-218).  Returns a dia_array (format None or "dia")
    whose data and offsets are those of scipy.sparse.diags_array, or its tocsr() / tocsc() ("csr", "csc"), which drop
    entries equal to zero.  Repeated offsets are accepted and give repeated entries in the CSR form."""
    if np.isscalar(offsets):
        if len(diagonals) == 0 or np.isscalar(diagonals[0]):
            diagonals = [np.atleast_1d(diagonals)]
        offsets = [offsets]
    else:
        diagonals = [np.atleast_1d(d) for d in diagonals]
    offsets = [int(o) for o in np.atleast_1d(offsets)]
    if len(diagonals) != len(offsets):
        raise ValueError("Different number of diagonals and offsets.")
    if shape is None:
        m = len(diagonals[0]) + abs(offsets[0])
        shape = (m, m)
    if dtype is None:
        dtype = np.result_type(*[np.asarray(d).dtype for d in diagonals])
    m, n = (int(s) for s in shape)
    full = []
    for d, k in zip(diagonals, offsets):
        length = min(m + min(k, 0), n - max(k, 0))
        if length < 0:
            raise ValueError(f"Offset {k} (index) out of bounds")
        d = np.asarray(d)
        if d.shape[0] == 1 and length != 1:
            d = np.full(length, d[0])  # scalar broadcast, as scipy
        full.append(d)
    A = dia_array._from_parts(to_device(_dia_data(full, offsets, (m, n), np.dtype(dtype))), offsets, (m, n))
    if format in (None, "dia"):
        return A
    if format == "csr":
        return A.tocsr()
    if format == "csc":
        return A.tocsc()
    raise NotImplementedError(f"diags(format={format!r})")


def spdiags(data, diags, m=None, n=None, format=None):
    """scipy.sparse.spdiags: the matrix with the rows of `data` on the diagonals `diags`, as
    dia_array((data, diags), shape=(m, n)).asformat(format); (m, n) may be given as one tuple in m, and both default
    to len(data[0])."""
    if m is None and n is None:
        m = n = len(data[0])
    elif n is None:
        m, n = m
    return dia_array((data, diags), shape=(m, n)).asformat(format)


def eye(m, n=None, k=0, dtype=np.float64, format=None):
    """Reference sparse/module.py:221-246: a CSR identity-like matrix, or for format="dia" the dia_array scipy builds
    (one diagonal of ones)."""
    if n is None:
        n = m
    m, n = int(m), int(n)
    if format == "dia":
        return diags([np.ones(max(0, min(m + k, n)), dtype=dtype)], [k], shape=(m, n), dtype=dtype)
    length = max(0, min(m + min(k, 0), n - max(k, 0)))   # a diagonal outside the matrix gives an empty one
    data = _dia_data([np.ones(length, dtype=dtype)], [k], (m, n), np.dtype(dtype))
    return dia_array._from_parts(to_device(data), [k], (m, n)).tocsr()


def identity(n, dtype=np.float64, format=None):
    return eye(n, n, dtype=dtype, format=format)


# ---- assembly from blocks (csrc/construct.cu) ---------------------------------------------------------------------------
_INT64_MAX = 2**63 - 1


def _as_csr(x) -> csr_array:
    """An operand as a csr_array: a csr_array as it is; a coo_array, a scipy sparse matrix or what `diags` returns
    through its CSR; a dense numpy array or torch tensor through `csr_array(dense)`, which drops zeros (a 1-D array is one
    row, as scipy reads it)."""
    if isinstance(x, csr_array):
        return x
    if isinstance(x, coo_array):
        return x.tocsr()
    if scipy.sparse.issparse(x):
        return csr_array(x)
    if isinstance(x, torch.Tensor):
        x = to_host(x)
    if not isinstance(x, np.ndarray) and hasattr(x, "tocsr"):
        return _as_csr(x.tocsr())
    a = np.atleast_2d(np.asarray(x))
    if a.ndim != 2:
        raise NotImplementedError(f"a {a.ndim}-D operand cannot be a block")
    return csr_array(a)


def _is_csr(x) -> bool:
    """scipy's test for its CSR stacking path: a sparse matrix in CSR format"""
    return isinstance(x, csr_array) or (scipy.sparse.issparse(x) and x.format == "csr")


def _check_result(shape, nnz, format, what):
    """The host checks every assembly makes before it allocates: the result fits int64 indices, and the format is one
    this library returns."""
    if max(shape[0], shape[1], nnz) >= _INT64_MAX:
        raise ValueError(f"{what}: a {shape[0]} x {shape[1]} result with {nnz} stored entries does not fit in int64")
    if format not in (None, "csr", "coo"):
        raise NotImplementedError(f"{what}(format={format!r}): only 'csr' (the default) and 'coo' results are built")


def _finish(C: csr_array, format):
    return C.tocoo() if format == "coo" else C


def kron(A, B, format=None):
    """Kronecker product of A (m x n) and B (p x q), scipy.sparse.kron on the device (reference sparse/module.py).

    Output row i * p + r holds, for each stored entry (j, a) of row i of A in stored order, row r of B in stored order,
    with columns j * q + c and values a * b.  Stored order, explicit zeros and repeated columns are kept, so canonical
    operands give a canonical result, equal to scipy's bit for bit.  The dtype is np.result_type of the operands,
    float32 or float64 (others raise NotImplementedError); only an operand of another dtype is cast.  Returns a
    csr_array (format None / "csr") or its tocoo() ("coo")."""
    A, B = _as_csr(A), _as_csr(B)
    shape = (A.shape[0] * B.shape[0], A.shape[1] * B.shape[1])
    nnz = A.nnz * B.nnz
    _check_result(shape, nnz, format, "kron")
    dtype = np.result_type(A.dtype, B.dtype)
    if dtype not in SUPPORTED_VALUE_DTYPES:
        raise NotImplementedError(f"kron for dtype {dtype} is not implemented (float32/float64 kernels only)")
    runtime.require_cuda("kron")
    A, B = A.astype(dtype, copy=False), B.astype(dtype, copy=False)
    ptr, idx, val = _ops.csr_kron(A._indptr, A._indices, A._data, A.shape, B._indptr, B._indices, B._data, B.shape,
                                  _index_dtype(shape[1] - 1))
    return _finish(csr_array._from_parts(ptr.to(_indptr_dtype(nnz)), idx, val, shape), format)


def _identity(n: int, dtype) -> csr_array:
    ar = torch.arange(n + 1, dtype=torch.int64, device=runtime.device)
    return csr_array._from_parts(ar.to(_indptr_dtype(n)), ar[:n].to(_index_dtype(n - 1)),
                                 torch.ones(n, dtype=torch_dtype(dtype), device=runtime.device), (n, n))


def kronsum(A, B, format=None):
    """Kronecker sum of square A (m x m) and B (n x n): kron(I_n, A) + kron(B, I_m), scipy's definition.  The two
    products come from `kron` and are added by the sparse add (csrc/elementwise.cu), which keeps entries that cancel to
    zero where scipy drops them.  Raises ValueError for a non-square operand, as scipy does."""
    A, B = _as_csr(A), _as_csr(B)
    if A.shape[0] != A.shape[1]:
        raise ValueError("A is not square")
    if B.shape[0] != B.shape[1]:
        raise ValueError("B is not square")
    m, n = A.shape[0], B.shape[0]
    _check_result((m * n, m * n), n * A.nnz + m * B.nnz, format, "kronsum")
    dtype = np.result_type(A.dtype, B.dtype)
    if dtype not in SUPPORTED_VALUE_DTYPES:
        raise NotImplementedError(f"kronsum for dtype {dtype} is not implemented (float32/float64 kernels only)")
    runtime.require_cuda("kronsum")
    C = _csr_binop(kron(_identity(n, dtype), A), kron(B, _identity(m, dtype)), "add")
    return _finish(C, format)


def _assemble(placed, shape, dtype, format, what):
    """The csr_array of the blocks `placed` = [(block row, row offset, column offset, csr_array)], in block-row order
    and left to right within a block row, through b2s_csr_blocks."""
    nnz = sum(A.nnz for _, _, _, A in placed)
    _check_result(shape, nnz, format, what)
    dtype = np.dtype(dtype)
    if dtype.itemsize not in (4, 8, 16) or dtype.kind not in "fciu":
        raise NotImplementedError(f"{what} for dtype {dtype} is not implemented (4-, 8- or 16-byte values)")
    runtime.require_cuda(what)
    tdt = torch_dtype(dtype)
    blocks = [(I, ro, co, A._indptr, A._indices, A._data if A._data.dtype == tdt else A._data.to(tdt), A.shape)
              for I, ro, co, A in placed if A.nnz]
    ptr, idx, val = _ops.csr_blocks(blocks, shape, nnz, tdt, _index_dtype(shape[1] - 1))
    return _finish(csr_array._from_parts(ptr.to(_indptr_dtype(nnz)), idx, val, shape), format)


def _result_dtype(mats, dtype):
    if dtype is not None:
        return np.dtype(dtype)
    return np.result_type(*[A.dtype for A in mats]) if mats else np.dtype(np.float64)


def bmat(blocks, format=None, dtype=None):
    """A sparse matrix from a 2-D grid of blocks (None: an all-zero block), scipy.sparse.bmat on the device.

    Output row r of block row I is the concatenation, over the block columns in order, of row r of each block, its
    columns shifted by the width of the blocks to its left.  Entries keep their stored order; nothing is summed or
    pruned.  Shapes are checked as scipy 1.18.1 checks them: when every block is a CSR matrix and format is None or
    "csr", scipy stacks each block row horizontally and the rows vertically, so the blocks of a row must share a height
    and the rows a total width; otherwise every block row has one height and every block column one width, a block
    with no rows or columns leaving its row's or column's size open.  The dtype is np.result_type of the blocks (or
    `dtype`), of 4, 8 or 16 bytes; only blocks of another dtype are cast.  Returns a csr_array (format None / "csr")
    or its tocoo() ("coo")."""
    grid = np.asarray(blocks, dtype="object")
    if grid.ndim != 2:
        raise ValueError("blocks must be 2-D, and some must be sparse")
    M, N = grid.shape
    placed = []
    if format in (None, "csr") and all(_is_csr(b) for b in grid.flat):
        if N == 0:
            raise IndexError(f"index 0 is out of bounds for axis 1 with size {N}")
        if M == 0:
            raise ValueError("need at least one array to concatenate")
        rows = [[_as_csr(b) for b in grid[I]] for I in range(M)]
        for row in rows:
            heights = {A.shape[0] for A in row}
            if len(heights) > 1:
                raise ValueError(f"Mismatching dimensions along axis 0: {heights}")
        widths = [sum(A.shape[1] for A in row) for row in rows]
        if any(w != widths[0] for w in widths):
            raise ValueError("incompatible dimensions for axis 1")
        r = 0
        for I, row in enumerate(rows):
            c = 0
            for A in row:
                placed.append((I, r, c, A))
                c += A.shape[1]
            r += row[0].shape[0]
        shape = (r, widths[0])
    else:
        brow, bcol = [0] * M, [0] * N
        mats = {}
        for i in range(M):
            for j in range(N):
                if grid[i, j] is None:
                    continue
                A = mats[i, j] = _as_csr(grid[i, j])
                if brow[i] == 0:
                    brow[i] = A.shape[0]
                elif brow[i] != A.shape[0]:
                    raise ValueError(f"blocks[{i},:] has incompatible row dimensions. Got blocks[{i},{j}].shape[0] == "
                                     f"{A.shape[0]}, expected {brow[i]}.")
                if bcol[j] == 0:
                    bcol[j] = A.shape[1]
                elif bcol[j] != A.shape[1]:
                    raise ValueError(f"blocks[:,{j}] has incompatible column dimensions. Got blocks[{i},{j}].shape[1] "
                                     f"== {A.shape[1]}, expected {bcol[j]}.")
        roff, coff = [0, *accumulate(brow)], [0, *accumulate(bcol)]
        placed = [(i, roff[i], coff[j], A) for (i, j), A in mats.items()]
        shape = (roff[-1], coff[-1])
    return _assemble(placed, shape, _result_dtype([A for *_, A in placed], dtype), format, "bmat")


def hstack(blocks, format=None, dtype=None):
    """Blocks side by side: bmat([blocks]), as scipy.sparse.hstack."""
    return bmat([np.asarray(blocks, dtype="object")], format=format, dtype=dtype)


def vstack(blocks, format=None, dtype=None):
    """Blocks one above the other: bmat([[b] for b in blocks]), as scipy.sparse.vstack."""
    return bmat([[b] for b in np.asarray(blocks, dtype="object")], format=format, dtype=dtype)


def block_diag(mats, format=None, dtype=None):
    """A block-diagonal matrix of `mats`, scipy.sparse.block_diag on the device: blocks as bmat takes them, and scalars
    (and lists) as dense arrays of at least two dimensions, so a scalar is a 1 x 1 block.  Dense blocks drop their
    zeros (scipy keeps the zeros of dense ndarray blocks as stored entries)."""
    placed = []
    r = c = 0
    for k, a in enumerate(mats):
        if isinstance(a, (list, numbers.Number)):
            A = csr_array(np.atleast_2d(a))
        elif isinstance(a, (np.ndarray, torch.Tensor)):
            if a.ndim != 2:  # scipy unpacks a dense block's shape into (rows, columns)
                raise ValueError(f"a dense block must be 2-D, got shape {tuple(a.shape)}")
            A = _as_csr(a)
        else:
            A = _as_csr(a)
        placed.append((k, r, c, A))
        r += A.shape[0]
        c += A.shape[1]
    if not placed:
        raise ValueError("need at least one array to concatenate")
    return _assemble(placed, (r, c), _result_dtype([A for *_, A in placed], dtype), format, "block_diag")


# ---- random sparse matrices (csrc/random.cu) --------------------------------------------------------------------------
_RANDOM_DTYPES = tuple(np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))


def _check_random_state(seed):
    """scipy's check_random_state: None -> numpy's global RandomState, an int -> a new RandomState, a Generator or
    RandomState as it is."""
    if seed is None or seed is np.random:
        return np.random.mtrand._rand
    if isinstance(seed, (numbers.Integral, np.integer)):
        return np.random.RandomState(seed)
    if isinstance(seed, (np.random.RandomState, np.random.Generator)):
        return seed
    raise ValueError(f"'{seed}' cannot be used to seed a numpy.random.RandomState instance")


def _scipy_rng(position=None):
    """Resolve `rng` / `random_state` into one generator as scipy 1.18.1 does (its _transition_to_rng): a keyword `rng`
    through numpy.random.default_rng, a `random_state` keyword or the argument at `position` as check_random_state
    reads it; the resolved generator reaches the function as `rng`."""
    def decorate(fun):
        @functools.wraps(fun)
        def wrapper(*args, **kwargs):
            positional = position is not None and len(args) > position
            if ("random_state" in kwargs) + ("rng" in kwargs) + positional > 1:
                raise TypeError(f"{fun.__name__}() got multiple values for argument now known as `rng`. Specify one of "
                                "`rng` or `random_state`.")
            if "rng" in kwargs:
                kwargs["rng"] = np.random.default_rng(kwargs["rng"])
            elif positional:
                args = (*args[:position], _check_random_state(args[position]), *args[position + 1:])
            else:
                kwargs["rng"] = _check_random_state(kwargs.pop("random_state", None))
            return fun(*args, **kwargs)
        return wrapper
    return decorate


def _random(shape, density, format, dtype, rng, data_sampler, what):
    """The one implementation of random, rand and random_array.  Checks as scipy does, draws one 64-bit seed from `rng`,
    calls `data_sampler(size=k)` once if given, then samples and assembles on the device (`_ops.random_csr`)."""
    if not 0 <= density <= 1:
        raise ValueError("density expected to be 0 <= density <= 1")
    if len(shape) != 2:
        raise NotImplementedError(f"{what}: a {len(shape)}-D shape; only 2-D random matrices are implemented")
    m, n = (int(s) for s in shape)
    if m < 0 or n < 0:
        raise ValueError("'shape' elements cannot be negative")
    mn = m * n
    if mn > _INT64_MAX:
        raise NotImplementedError(f"{what}: {m} x {n} positions do not fit in int64")
    k = int(round(density * mn))
    if format not in ("coo", "csr", "csc", "dia"):
        raise NotImplementedError(f"{what}(format={format!r}): 'coo', 'csr', 'csc' and 'dia' are implemented")
    dtype = np.dtype(np.float64 if dtype is None else dtype)
    if dtype not in _RANDOM_DTYPES:
        raise NotImplementedError(f"{what} for dtype {dtype} is not implemented (float32, float64, complex64 and "
                                  "complex128 are)")
    if isinstance(rng, np.random.Generator):
        seed = int(rng.integers(0, 2**64, dtype=np.uint64))
    else:
        seed = int(rng.randint(0, 2**64, dtype=np.uint64))
    vals = None
    if data_sampler is not None:
        vals = np.asarray(data_sampler(size=k)).astype(dtype, copy=False)
        if vals.shape != (k,):
            raise ValueError(f"{what}: the data sampler returned {vals.shape} values for {k} stored entries")
    runtime.require_cuda(what)
    ptr, idx, data, _ = _ops.random_csr((m, n), k, seed, _index_dtype(max(m, n)), _indptr_dtype(k), dtype,
                                        None if vals is None else to_device(vals))
    A = csr_array._from_parts(ptr, idx, data, (m, n))
    if format == "csr":
        return A
    if format == "coo":
        return A.tocoo()
    if format == "dia":
        return A.todia()
    # csc: b2s_csr_transpose, which takes real values only; complex values follow their entries' positions, moved as
    # float64 bit patterns (denormals).  This relies on the transpose moving values without arithmetic, as
    # include/b200sparse.h states; the complex CSC test of tests/test_gpu_random.py fails if it ever flushes them.
    cplx = dtype.kind == "c"
    moved = torch.arange(k, dtype=torch.int64, device=data.device).view(torch.float64) if cplx else data
    t_ptr, t_idx, t_val = _ops.csr_transpose(ptr, idx, moved, (m, n))
    t_data = data[t_val.view(torch.int64)] if cplx else t_val
    return csc_array._wrap(csr_array._from_parts(t_ptr, t_idx, t_data, (n, m)))


@_scipy_rng(position=5)
def random(m, n, density=0.01, format="coo", dtype=None, rng=None, data_rvs=None, *, random_state=None):
    """A random m x n sparse matrix with exactly k = int(round(density * m * n)) stored entries at a uniform random
    k-subset of the positions, scipy.sparse.random's signature, sampled on the device.

    The values are uniform on [0, 1) (complex dtypes: real and imaginary parts each), or `data_rvs(k)`, called once
    and cast to `dtype`, in canonical order.  float32, float64 (the default), complex64 and complex128.  `rng` and
    `random_state` are resolved as scipy resolves them, and exactly one 64-bit seed is drawn from the result; everything
    after that runs on the device, so one seed gives bit-identical arrays on every run and in every format ("coo", the
    default, in row-major order, "csr", "csc", "dia").  It is not the matrix scipy draws for that seed.  The reference's
    positional order (..., dtype, random_state, data_rvs) works unchanged."""
    return _random((m, n), density, format, dtype, rng, None if data_rvs is None else (lambda size: data_rvs(size)),
                   "random")


@_scipy_rng(position=5)
def rand(m, n, density=0.01, format="coo", dtype=None, rng=None, *, random_state=None):
    """`random` with uniform [0, 1) values, scipy.sparse.rand's signature."""
    return _random((m, n), density, format, dtype, rng, None, "rand")


@_scipy_rng()
def random_array(shape, *, density=0.01, format="coo", dtype=None, rng=None, data_sampler=None, random_state=None):
    """`random` with scipy.sparse.random_array's signature: a 2-D `shape`, and `data_sampler(size=k)` for the values."""
    return _random(tuple(shape), density, format, dtype, rng, data_sampler, "random_array")
