"""Host-side checks of the csr_array reductions (csrc/reduce.cu through `_ops.csr_reduce_rows`).

`reduce_oracle` restates the kernel's per-row rules with numpy: sums in fp64, MAX / MIN with the implicit zero of a row
shorter than ncols, ARG* with the first missing column standing for the implicit zeros, NaN first.  It is pinned to
numpy on `toarray()` (and to scipy for `explicit=True`) on the MatrixMarket fixtures and on hand-built rows.  The argument
checks need no device, nor do the C entry point's own checks.  The `-m gpu` file is rehearsed through
tests/dryrun_cpu.py with `_ops.csr_reduce_rows` swapped for the oracle."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, ROOT, mtx_path

OPS = ["sum", "max", "min", "argmax", "argmin", "count_nonzero"]


def reduce_oracle(indptr, indices, data, ncols, op, explicit=False):
    """Per-row `op` of a CSR matrix.  sum accepts any rows; the other ops need rows without repeated columns, and
    argmax / argmin strictly ascending ones (the kernel's input contract)."""
    indptr = np.asarray(indptr).astype(np.int64)
    indices = np.asarray(indices).astype(np.int64)
    data = np.asarray(data)
    m = indptr.size - 1
    lens = np.diff(indptr)
    rows = np.repeat(np.arange(m), lens)
    full = (not explicit) & (lens < ncols)            # rows with implicit zeros that count
    if op == "sum":
        out = np.zeros(m, dtype=np.float64)
        np.add.at(out, rows, data.astype(np.float64))
        return out.astype(data.dtype)
    if op == "count_nonzero":
        return np.bincount(rows, weights=data != 0, minlength=m).astype(np.int64)
    nonempty = lens > 0
    starts = indptr[:-1][nonempty]
    if op in ("max", "min"):
        f = np.maximum if op == "max" else np.minimum
        out = np.zeros(m, dtype=data.dtype)
        if data.size:
            out[nonempty] = f.reduceat(data, starts)                 # NaN propagates
        return np.where(full & nonempty, f(out, 0), out).astype(data.dtype)
    out = np.zeros(m, dtype=np.int64)
    if data.size == 0:
        return out
    nan = np.isnan(data)
    key = -data if op == "argmax" else data
    order = np.lexsort((indices, np.where(nan, 0, key), ~nan, rows))  # per row: NaN first, then the extreme, then column
    first = order[np.r_[0, np.flatnonzero(np.diff(rows[order])) + 1]]
    bcol, bval, bnan = indices[first], data[first], nan[first]
    pos = np.arange(data.size) - indptr[rows]
    miss = np.minimum(np.minimum.reduceat(np.where(indices != pos, pos, np.iinfo(np.int64).max), starts), lens[nonempty])
    better = bval > 0 if op == "argmax" else bval < 0
    implicit = np.where(better, bcol, np.where(bval == 0, np.minimum(miss, bcol), miss))
    out[nonempty] = np.where(bnan, bcol, np.where(full[nonempty], implicit, bcol))
    return out


def _dryrun_reduce(op, indptr, indices, data, ncols, explicit=False, out=None):
    """`_ops.csr_reduce_rows` for the CPU dry run of the GPU test file."""
    idx = np.zeros(data.shape[0], dtype=np.int64) if indices is None else indices.numpy()
    v = torch.from_numpy(np.ascontiguousarray(reduce_oracle(indptr.numpy(), idx, data.numpy(), ncols, op, explicit)))
    if out is None:
        return v
    out.copy_(v)
    return out


def _dryrun_sort_rows(indptr, indices, data):
    """`_ops.csr_sort_rows` for the CPU dry run: the rows sorted by column, in place."""
    ptr = indptr.numpy().astype(np.int64)
    for i in range(ptr.size - 1):
        lo, hi = ptr[i], ptr[i + 1]
        o = np.argsort(indices[lo:hi].numpy(), kind="stable")
        indices[lo:hi] = indices[lo:hi][o].clone()
        data[lo:hi] = data[lo:hi][o].clone()
    return indices, data


def _dense_reduce(D, op, axis):
    """numpy's answer on the dense matrix."""
    if op == "count_nonzero":
        return np.count_nonzero(D, axis=axis)
    return getattr(D, op)(axis=axis)


def _canonical(S):
    S = sp.csr_array(S, copy=True)
    S.sum_duplicates()
    return S


def _rows(S, op, explicit=False):
    return reduce_oracle(S.indptr, S.indices, S.data, S.shape[1], op, explicit)


@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("op", OPS)
def test_oracle_matches_numpy_on_fixtures(name, op):
    S = _canonical(scipy.io.mmread(mtx_path(name)))
    D = S.toarray()
    for axis, M in ((1, S), (0, _canonical(S.T))):
        got, want = _rows(M, op), _dense_reduce(D, op, axis)
        if op == "sum":
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
        else:
            assert np.array_equal(got, want), (axis, got, want)
    if op in ("max", "min", "argmax", "argmin"):
        want = getattr(S, op)(axis=1, explicit=True)
        want = want.toarray() if hasattr(want, "toarray") else want
        assert np.array_equal(_rows(S, op, explicit=True), want)


def _hand_matrix():
    """Rows (n = 6): empty; full; all negative with holes; all positive with holes; stored zeros before and after the
    first missing column; NaN with holes; NaN in a full row; +-0 and +-inf; a single -inf; only stored zeros."""
    inf, nan = np.inf, np.nan
    rows = [
        [],
        [(0, 1.0), (1, -2.0), (2, 3.0), (3, 3.0), (4, -7.0), (5, 0.5)],
        [(0, -1.0), (1, -4.0), (3, -2.0)],
        [(1, 2.0), (2, 5.0), (5, 5.0)],
        [(0, 0.0), (1, -3.0), (3, 0.0)],
        [(0, -1.0), (2, 0.0), (4, 0.0)],
        [(0, 2.0), (3, nan), (4, 9.0)],
        [(0, 1.0), (1, nan), (2, 3.0), (3, nan), (4, 1.0), (5, 0.0)],
        [(0, -0.0), (1, 0.0), (2, inf), (4, -inf)],
        [(3, -inf)],
        [(1, 0.0), (2, -0.0)],
        [(0, -5.0), (1, -5.0), (2, -5.0), (3, -5.0), (4, -5.0), (5, -5.0)],
    ]
    indptr = np.r_[0, np.cumsum([len(r) for r in rows])]
    indices = np.array([c for r in rows for c, _ in r], dtype=np.int64)
    data = np.array([v for r in rows for _, v in r], dtype=np.float64)
    return sp.csr_array((data, indices, indptr), shape=(len(rows), 6))


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_hand_rows(op, dtype):
    S = _hand_matrix().astype(dtype)
    D = S.toarray()
    with np.errstate(invalid="ignore"):
        want = _dense_reduce(D, op, 1)
    got = _rows(S, op)
    assert got.dtype == (dtype if op in ("sum", "max", "min") else np.int64)
    if op in ("sum", "max", "min"):
        np.testing.assert_array_equal(got, want.astype(dtype))       # NaN == NaN here; -0 == +0
    else:
        assert np.array_equal(got, want), (got, want)


@pytest.mark.parametrize("op", ["max", "min", "argmax", "argmin"])
def test_hand_rows_explicit(op):
    S = _hand_matrix()
    got = _rows(S, op, explicit=True)
    nan_rows = np.isnan(S.toarray()).any(axis=1)
    want = getattr(S, op)(axis=1, explicit=True)
    want = want.toarray() if hasattr(want, "toarray") else want
    # scipy agrees wherever the row has no NaN; NaN rows follow numpy over the stored values
    assert np.array_equal(got[~nan_rows], want[~nan_rows])
    for i in np.flatnonzero(nan_rows):
        stored = S.data[S.indptr[i]:S.indptr[i + 1]]
        k = int(getattr(np, op)(stored)) if op.startswith("arg") else None
        if op.startswith("arg"):
            assert got[i] == S.indices[S.indptr[i] + k]
        else:
            assert np.isnan(got[i])


def test_scipy_nan_difference_is_as_documented():
    # a row holding a NaN and implicit zeros: numpy (and this library) answers the NaN, scipy 1.18 the first zero
    S = sp.csr_array(np.array([[3.0, np.nan, 0.0]]))
    assert _rows(S, "argmax")[0] == 1 == np.argmax(S.toarray()[0])


def test_duplicates_and_unsorted_rows_sum_as_toarray():
    rng = np.random.default_rng(0)
    indptr = np.r_[0, np.cumsum(rng.integers(0, 12, 300))]
    indices = rng.integers(0, 7, indptr[-1])
    data = rng.integers(-3, 4, indptr[-1]).astype(np.float64)
    S = sp.csr_array((data, indices, indptr), shape=(300, 7))
    D = S.toarray()
    assert np.array_equal(_rows(S, "sum"), D.sum(axis=1))           # sums need no canonical form
    C = _canonical(S)
    for op in OPS:
        assert np.array_equal(_rows(C, op), _dense_reduce(D, op, 1)), op


def _host_only(monkeypatch):
    from legate.sparse_b200.runtime import Runtime

    monkeypatch.setattr(Runtime, "has_cuda", property(lambda self: False))


def test_argument_errors_need_no_device(monkeypatch):
    _host_only(monkeypatch)
    A = csr_array(sp.random_array((5, 6), density=0.5, format="csr", rng=np.random.default_rng(0)))
    reducers = [A.sum, A.mean, A.max, A.min, A.argmax, A.argmin, A.count_nonzero]
    for f in reducers:
        for axis in (2, -3, 1.0, "0", (0, 1), True):
            with pytest.raises(ValueError):
                f(axis=axis)
    for f in (A.max, A.min, A.argmax, A.argmin):
        with pytest.raises(ValueError):
            f(axis=1, out=np.zeros(5))
    for f in (A.sum, A.mean):
        for out in (np.zeros(6), np.zeros(5, dtype=np.float32), torch.zeros(5, dtype=torch.float32), [0.0] * 5,
                    np.zeros((5, 1))):
            with pytest.raises(ValueError):
                f(axis=1, out=out)
        with pytest.raises(NotImplementedError):
            f(dtype=np.int64)
    # empty shapes
    for shape in ((0, 4), (4, 0), (0, 0)):
        E = csr_array(sp.csr_array(shape))
        for f in (E.max, E.min, E.argmax, E.argmin):
            with pytest.raises(ValueError):
                f()
    for f in (csr_array(sp.csr_array((4, 0))).max, csr_array(sp.csr_array((4, 0))).argmin):
        with pytest.raises(ValueError):
            f(axis=1)
    for f in (csr_array(sp.csr_array((0, 4))).min, csr_array(sp.csr_array((0, 4))).argmax):
        with pytest.raises(ValueError):
            f(axis=0)
    with pytest.raises(ValueError):
        csr_array(sp.csr_array((3, 4))).argmax(explicit=True)
    # data types other than float32 / float64
    for dt in (np.complex64, np.int32, np.int64, bool):
        Z = csr_array(sp.csr_array(np.eye(3, dtype=dt)))
        for f in (Z.sum, Z.mean, Z.max, Z.min, Z.argmax, Z.argmin, Z.count_nonzero):
            with pytest.raises(NotImplementedError):
                f(axis=1)
    # power: scalars only, and not 0 (both before any device)
    with pytest.raises(NotImplementedError):
        A.power(np.array([1, 2]))
    with pytest.raises(NotImplementedError):
        A.power(0)
    # valid arguments reach the device check
    for f in reducers:
        with pytest.raises(RuntimeError, match="no CUDA device"):
            f(axis=0)


def test_abs_and_power_share_the_structure():
    S = sp.random_array((5, 6), density=0.5, format="csr", rng=np.random.default_rng(0))
    S.data -= 0.5
    A = csr_array(S)
    B = abs(A)
    assert B.indptr is A.indptr and B.indices is A.indices
    assert torch.equal(B.data, A.data.abs())
    P = A.power(3, dtype=np.float32)
    assert P.indptr is A.indptr and P.indices is A.indices and P.dtype == np.float32
    assert torch.allclose(P.data, A.data.to(torch.float32) ** 3)


def test_abi_rejects_bad_arguments():
    from legate.sparse_b200 import _lib

    L = _lib.lib
    buf = (ctypes.c_int64 * 64)()
    obuf = (ctypes.c_int64 * 64)()
    pb, po = ctypes.addressof(buf), ctypes.addressof(obuf)

    def call(op=0, vt=_lib.F64, it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4, indptr=pb, indices=pb + 64, vals=pb + 128,
             out=po):
        rc = L.b2s_csr_reduce_rows(op, vt, it, pt, m, n, nnz, indptr, indices, vals, 0, out, None)
        return rc, _lib.last_error()

    cases = [
        (dict(op=6), "bad reduction code 6"),
        (dict(op=-1), "bad reduction code -1"),
        (dict(vt=2), "bad value type code 2"),
        (dict(it=5), "bad index type code 5"),
        (dict(pt=9), "bad indptr type code 9"),
        (dict(m=-1), "negative dimension"),
        (dict(n=-1), "negative dimension"),
        (dict(nnz=-1), "negative dimension"),
        (dict(m=2**31 - 1), "nrows >= 2^31-1 is not supported"),
        (dict(nnz=2**31 - 1), "int32 indptr cannot address nnz >= 2^31-1"),
        (dict(indptr=None), "indptr is NULL"),
        (dict(out=None), "out is NULL"),
        (dict(vals=None), "vals NULL with nnz > 0"),
        (dict(op=3, indices=None), "indices NULL with nnz > 0"),
        (dict(op=4, indices=None), "indices NULL with nnz > 0"),
        (dict(n=0), "nnz > 0 in a matrix with no columns"),
        (dict(out=pb + 128), "out overlaps vals"),
        (dict(out=pb + 128 + 8 * 3), "out overlaps vals"),           # vals' last fp64 value
        (dict(out=pb + 64, op=3), "out overlaps indices"),
        (dict(out=pb + 64 - 8 * 4 + 4, op=5), "out overlaps indices"),  # int64 counts ending 4 bytes into indices
        (dict(out=pb), "out overlaps indptr"),
    ]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc == _lib.EINVAL and msg in err, (kw, err)
    # indices may be NULL for the other ops (the call then fails only on the host pointers at launch, so it is not
    # made here); nothing to compute needs no pointer at all
    assert call(m=0, indptr=None, indices=None, vals=None, out=None)[0] == _lib.OK
    # an int64 indptr may address 2^31 - 1 entries and more
    assert "int32 indptr" not in call(pt=_lib.I64, nnz=2**31 - 1, out=None)[1]


def test_gpu_file_passes_the_cpu_dry_run():
    script = (
        "import sys, pytest\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import dryrun_cpu\n"
        "dryrun_cpu.install()\n"
        "from legate.sparse_b200 import _ops\n"
        "import test_reduce_host\n"
        "_ops.csr_reduce_rows = test_reduce_host._dryrun_reduce\n"
        "_ops.csr_sort_rows = test_reduce_host._dryrun_sort_rows\n"
        "sys.exit(pytest.main(['-m', 'gpu', '-q', '-p', 'no:cacheprovider', sys.argv[1], '-k', sys.argv[2]]))\n"
    )
    # the graph test needs a device; the full-size cases and the example runs are minutes of numpy here
    r = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "tests", "test_gpu_reduce.py"),
                        "not graph and not full_size and not amg and not million"], capture_output=True, text=True,
                       timeout=900, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
