"""Host-side checks of csr_array indexing (csrc/index.cu through `_ops.csr_column_map`, `_ops.csr_select` and
`_ops.csr_lookup`).

`select_oracle` restates the kernels' entry-order rule with numpy: output row t is the source row rows[t], its entries
in stored order, each written once per requested position of its column, positions ascending.  It is pinned to scipy on
the MatrixMarket fixtures and on hand-built rows with repeated and unsorted columns and explicit zeros.  The key
normaliser `_index_key` is pinned to scipy's shapes and errors, the C entry points' own checks are called through
ctypes, and the `-m gpu` file is rehearsed through tests/dryrun_cpu.py with the three `_ops` wrappers swapped for the
restatement."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200.csr import _index_key, csr_array

from conftest import MTX_FILES, ROOT, mtx_path


def select_oracle(indptr, indices, data, rows, cols, ncols):
    """(indptr, indices, data) of the outer selection: rows an int64 array (negatives count from the end), cols an
    int64 array or None for every column."""
    indptr = np.asarray(indptr).astype(np.int64)
    indices = np.asarray(indices).astype(np.int64)
    data = np.asarray(data)
    rows = np.asarray(rows, dtype=np.int64).reshape(-1)
    rows = np.where(rows < 0, rows + indptr.size - 1, rows)
    lens = indptr[rows + 1] - indptr[rows]
    ptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    src = (np.repeat(indptr[rows] - ptr[:-1], lens) + np.arange(ptr[-1])).astype(np.int64)
    if cols is None:
        return ptr, indices[src], data[src]
    cols = np.asarray(cols, dtype=np.int64).reshape(-1)
    cols = np.where(cols < 0, cols + ncols, cols)
    mptr = np.r_[0, np.cumsum(np.bincount(cols, minlength=ncols))].astype(np.int64)
    mpos = np.argsort(cols, kind="stable").astype(np.int64)          # positions of every column, ascending
    c = indices[src]
    mult = mptr[c + 1] - mptr[c]
    first = np.r_[0, np.cumsum(mult)][:-1].astype(np.int64)
    slot = np.repeat(mptr[c], mult) + np.arange(int(mult.sum())) - np.repeat(first, mult)
    out_ptr = np.r_[0, np.cumsum(np.bincount(np.repeat(np.arange(rows.size), lens), weights=mult,
                                             minlength=rows.size))].astype(np.int64)
    return out_ptr, mpos[slot.astype(np.int64)], data[np.repeat(src, mult)]


def lookup_oracle(indptr, indices, data, shape, ri, ci):
    """A[ri[w], ci[w]]: the matches added in stored order, from the first one; 0 when there is none."""
    m, n = shape
    out = np.zeros(len(ri), dtype=np.asarray(data).dtype)
    for w, (i, j) in enumerate(zip(np.asarray(ri), np.asarray(ci))):
        i, j = int(i) % m, int(j) % n
        acc = None
        for p in range(int(indptr[i]), int(indptr[i + 1])):
            if int(indices[p]) == j:
                acc = data[p] if acc is None else acc + data[p]
        out[w] = 0 if acc is None else acc
    return out


def _canonical_equal(ptr, idx, val, shape, S):
    """True when (ptr, idx, val) and scipy's S are the same matrix with every entry kept (duplicates are compared as a
    multiset of (row, column, value))."""
    rows = np.repeat(np.arange(shape[0]), np.diff(ptr))
    a = sorted(zip(rows.tolist(), np.asarray(idx).tolist(), np.asarray(val).tolist()))
    C = S.tocsr() if hasattr(S, "tocsr") else S
    rs = np.repeat(np.arange(C.shape[0]), np.diff(C.indptr))
    b = sorted(zip(rs.tolist(), C.indices.tolist(), C.data.tolist()))
    return tuple(shape) == tuple(C.shape) and a == b


def _sel(S, key):
    """select_oracle for a key `_index_key` classifies as an outer selection."""
    kind, R, C = _index_key(key, S.shape)
    assert kind == "outer"
    rows = np.arange(R[1], R[1] + R[2] * R[3], R[2]) if R[0] == "slice" else R[1]
    if C == ("slice", 0, 1, S.shape[1]):
        cols = None
    else:
        cols = np.arange(C[1], C[1] + C[2] * C[3], C[2]) if C[0] == "slice" else C[1]
    ncols_out = S.shape[1] if cols is None else len(cols)
    return select_oracle(S.indptr, S.indices, S.data, rows, cols, S.shape[1]), (len(rows), ncols_out)


def _keys(m, n, seed=0):
    """Outer-selection keys: every kind of row and column index, and np.ix_."""
    rng = np.random.default_rng(seed)
    p, q = rng.permutation(m), rng.permutation(n)
    return [
        3 % m, -1, slice(None), slice(1, None, 2), slice(None, None, -3), list(p[: m // 2]),
        (slice(None), list(q)), (slice(None), q[: n // 3]), (slice(2, -1), slice(None, None, -1)),
        (list(p), 1), (0, q[:4]), (rng.random(m) < 0.5, slice(None)), (slice(None), rng.random(n) < 0.5),
        (Ellipsis, -2), (1, Ellipsis), np.ix_(p[:7], q[:5]), np.ix_(p, p[:0] if m != n else p),
        (slice(None), [0, 0, 1, 1, 0]), ([-1, -2, 0, -1], slice(None)), (slice(None), []), ([], slice(None)),
    ]


@pytest.mark.parametrize("name", MTX_FILES)
def test_oracle_matches_scipy_on_fixtures(name):
    S = sp.csr_matrix(scipy.io.mmread(mtx_path(name)))
    m, n = S.shape
    for key in _keys(m, n):
        if isinstance(key, tuple) and len(key) == 2 and isinstance(key[0], np.ndarray) and key[0].ndim == 2 \
                and key[1].size == 0:
            continue
        (ptr, idx, val), shape = _sel(S, key)
        W = S[key]
        cols = key[1] if isinstance(key, tuple) and len(key) == 2 else None
        unique = cols is None or not isinstance(cols, (list, np.ndarray)) or len(set(np.asarray(cols).ravel().tolist()
                                                                                    )) == np.asarray(cols).size
        assert tuple(W.shape) == shape, (key, W.shape, shape)
        if unique:
            assert np.array_equal(ptr, W.indptr) and np.array_equal(idx, W.indices), key
            assert np.array_equal(val, W.data), key
        else:
            assert _canonical_equal(ptr, idx, val, shape, W), key


def _hand():
    """Rows (n = 6) with repeated and unsorted columns, explicit zeros and an empty row."""
    rows = [
        [(4, 1.0), (1, 2.0), (4, 3.0), (0, 0.0)],
        [],
        [(5, -1.0), (5, 0.0), (2, 7.0)],
        [(0, 1.5), (1, 2.5), (2, 3.5), (3, 4.5), (4, 5.5), (5, 6.5)],
        [(3, 0.0)],
    ]
    indptr = np.r_[0, np.cumsum([len(r) for r in rows])]
    indices = np.array([c for r in rows for c, _ in r], dtype=np.int64)
    data = np.array([v for r in rows for _, v in r])
    return sp.csr_matrix((data, indices, indptr), shape=(len(rows), 6))


def test_entry_order_rule_on_hand_rows():
    S = _hand()
    # unique columns, any order: scipy's arrays exactly
    for cols in ([5, 4, 3, 2, 1, 0], [4, 0], [1, 3, 5], [-1, 0]):
        (ptr, idx, val), shape = _sel(S, (slice(None), cols))
        W = S[:, cols]
        assert np.array_equal(ptr, W.indptr) and np.array_equal(idx, W.indices) and np.array_equal(val, W.data)
    # repeated columns: every kept entry once per position, positions ascending, in stored order
    ptr, idx, val = select_oracle(S.indptr, S.indices, S.data, [0], [4, 1, 4], 6)
    assert ptr.tolist() == [0, 5]
    assert idx.tolist() == [0, 2, 1, 0, 2] and val.tolist() == [1.0, 1.0, 2.0, 3.0, 3.0]
    assert _canonical_equal(ptr, idx, val, (1, 3), S[[0]][:, [4, 1, 4]])
    # duplicates and explicit zeros of A are kept, rows repeat
    ptr, idx, val = select_oracle(S.indptr, S.indices, S.data, [2, 2, 1], None, 6)
    assert ptr.tolist() == [0, 3, 6, 6] and idx.tolist() == [5, 5, 2] * 2 and val.tolist() == [-1.0, 0.0, 7.0] * 2


def test_lookup_oracle_matches_scipy():
    S = _hand()
    rng = np.random.default_rng(0)
    ri, ci = rng.integers(-5, 5, 200), rng.integers(-6, 6, 200)
    assert np.array_equal(lookup_oracle(S.indptr, S.indices, S.data, S.shape, ri, ci), np.asarray(S[ri, ci]).ravel())
    for name in MTX_FILES:
        F = sp.csr_matrix(scipy.io.mmread(mtx_path(name)))
        ri, ci = rng.integers(0, F.shape[0], 300), rng.integers(0, F.shape[1], 300)
        assert np.array_equal(lookup_oracle(F.indptr, F.indices, F.data, F.shape, ri, ci), np.asarray(F[ri, ci]).ravel())


def _scipy_outcome(S, key):
    try:
        r = S[key]
    except Exception as exc:  # noqa: BLE001
        return type(exc)
    return ("scalar",) if np.isscalar(r) or np.ndim(r) == 0 else tuple(np.shape(r))


def _our_outcome(shape, key):
    try:
        kind, R, C = _index_key(key, shape)
    except Exception as exc:  # noqa: BLE001
        return type(exc)
    if kind == "element":
        return ("scalar",)
    if kind == "points":
        return (1, len(R))                                   # csr_matrix returns a (1, k) matrix; this library 1-D k
    size = lambda s: s[3] if s[0] == "slice" else len(s[1])  # noqa: E731
    return (size(R), size(C))


def test_key_normaliser_against_scipy():
    S = sp.csr_matrix(np.arange(1.0, 31.0).reshape(5, 6))
    p = np.array([4, 0, 2])
    cases = _keys(5, 6) + [
        (2, 3), (-1, -6), (np.int64(1), np.int32(2)), (p, [1, 2, 3]), (np.array([True, False, True, False, True]),
                                                                           np.array([0, 1, 2])),
        (5, 0), (0, 6), (-6, 0), ([5], slice(None)), (slice(None), [-7]), (np.zeros(4, bool), slice(None)),
        (slice(None), np.zeros(7, bool)), (1, 2, 3), (Ellipsis, Ellipsis),
        (p, [1, 2]), (slice(None, None, 0), 1),
    ]
    for key in cases:
        want, got = _scipy_outcome(S, key), _our_outcome(S.shape, key)
        assert got == want, (key, got, want)


def test_key_normaliser_differences_are_as_documented():
    # float index arrays raise IndexError here (numpy's rule), and so does None (scipy's csr_matrix adds an axis of
    # length 1, which a 2-D sparse result cannot keep apart from a row); 2-D arrays other than np.ix_ are not supported
    for key in ((np.array([0.0, 1.0]), slice(None)), (slice(None), [1.5]), 1.0, (0, 2.0), (None, 1), (1, None)):
        with pytest.raises(IndexError):
            _index_key(key, (5, 6))
    for key in (np.zeros((2, 2), np.int64), (np.zeros((2, 3), np.int64), np.zeros((2, 3), np.int64))):
        with pytest.raises(NotImplementedError):
            _index_key(key, (5, 6))
    # an int keeps its axis (csr_matrix), and a slice is never materialised
    assert _index_key(3, (5, 6)) == ("outer", ("slice", 3, 1, 1), ("slice", 0, 1, 6))
    assert _index_key((slice(None, None, -2), 0), (5, 6)) == ("outer", ("slice", 4, -2, 3), ("slice", 0, 1, 1))
    # host arrays are wrapped and checked on the host; CPU tensors are host arrays
    kind, R, C = _index_key((torch.tensor([-1, 0]), [True, False, True, False, False, False]), (5, 6))
    assert kind == "points" and R.tolist() == [4, 0] and C.tolist() == [0, 2]


def _host_only(monkeypatch):
    from legate.sparse_b200.runtime import Runtime

    monkeypatch.setattr(Runtime, "has_cuda", property(lambda self: False))


def test_errors_need_no_device(monkeypatch):
    _host_only(monkeypatch)
    A = csr_array(sp.random_array((5, 6), density=0.5, format="csr", rng=np.random.default_rng(0)))
    for key in ((5, 0), (0, [6]), ([1, 2], [1]), (None,), (1, 2, 3), (np.zeros(4, bool),), ([0.5],)):
        with pytest.raises(IndexError):
            A[key]
    with pytest.raises(NotImplementedError):
        A[np.zeros((2, 2), np.int64)]
    Z = csr_array(sp.csr_array(np.eye(3, dtype=np.complex128)))
    with pytest.raises(NotImplementedError):
        Z[0, 0]
    with pytest.raises(TypeError):
        A[0, 0] = 1.0
    for key in ((1, 2), (slice(None), [0, 1]), ([0, 1], [2, 3])):
        with pytest.raises(RuntimeError, match="no CUDA device"):
            A[key]
    with pytest.raises(RuntimeError, match="no CUDA device"):
        Z[:, [0]]                                             # complex selections only move values


def test_abi_rejects_bad_arguments():
    from legate.sparse_b200 import _lib

    L = _lib.lib
    buf = (ctypes.c_int64 * 256)()
    pb = ctypes.addressof(buf)
    info = (ctypes.c_int64 * 4)()
    # inputs at pb .. pb + 8 * 64, outputs after
    op, oi, ov, sc = pb + 8 * 100, pb + 8 * 140, pb + 8 * 180, pb + 8 * 220

    def select(pass_=0, vw=8, it=_lib.I32, pt=_lib.I32, ot=_lib.I32, m=4, n=4, nnz=4, indptr=pb, indices=pb + 64,
               vals=pb + 128, nout=2, rows=pb + 256, cptr=None, cpos=None, ncols_out=4, out_ptr=op, out_idx=oi,
               out_val=ov, nnz_out=4, scratch=sc, inf=info):
        rc = L.b2s_csr_select(pass_, vw, it, pt, ot, m, n, nnz, indptr, indices, vals, nout, rows, 0, 1, cptr, cpos,
                              ncols_out, out_ptr, out_idx, out_val, nnz_out, scratch, inf, None)
        return rc, _lib.last_error()

    cases = [
        (dict(pass_=2), "bad pass 2"),
        (dict(vw=2), "bad value width 2"),
        (dict(it=3), "bad index type code 3"),
        (dict(pt=3), "bad indptr type code 3"),
        (dict(ot=3), "bad output index type code 3"),
        (dict(m=-1), "negative dimension"),
        (dict(nout=-1), "negative dimension"),
        (dict(nnz=2**31 - 1), "int32 indptr cannot address"),
        (dict(ncols_out=2**31 + 1, cptr=pb + 400, cpos=pb + 400), "int32 output indices cannot hold"),
        (dict(ncols_out=3), "without a column map every column is kept"),
        (dict(out_ptr=None), "out_indptr is NULL"),
        (dict(scratch=None), "scratch is NULL"),
        (dict(inf=None), "info_host is NULL"),
        (dict(indptr=None), "indptr is NULL"),
        (dict(indices=None), "indices NULL with nnz > 0"),
        (dict(pass_=1, vals=None), "vals NULL with nnz > 0"),
        (dict(pass_=1, out_idx=None), "out_indices/out_vals NULL"),
        (dict(pass_=1, cptr=pb + 400, cpos=None, ncols_out=3), "col_pos NULL with a column map"),
        (dict(out_ptr=pb + 8), "out_indptr overlaps indptr"),
        (dict(out_ptr=pb + 256), "out_indptr overlaps rows"),
        (dict(pass_=1, out_idx=pb + 64), "out_indices overlaps indices"),
        (dict(pass_=1, out_val=pb + 128 + 24), "out_vals overlaps vals"),
        (dict(pass_=1, out_val=oi), "out_indices overlaps out_vals"),
        (dict(pass_=1, out_idx=op + 8), "out_indptr overlaps out_indices"),
    ]
    for kw, msg in cases:
        rc, err = select(**kw)
        assert rc == _lib.EINVAL and msg in err, (kw, err)

    def lookup(vt=_lib.F64, it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4, k=2, ri=pb + 256, ci=pb + 272, out=op,
               bad=oi):
        rc = L.b2s_csr_lookup(vt, it, pt, m, n, nnz, pb, pb + 64, pb + 128, k, ri, ci, out, bad, None)
        return rc, _lib.last_error()

    cases = [
        (dict(vt=2), "bad value type code 2"),
        (dict(it=2), "bad index type code 2"),
        (dict(k=-1), "negative dimension"),
        (dict(ri=None), "row/column index arrays NULL"),
        (dict(out=None), "out is NULL"),
        (dict(bad=None), "bad is NULL"),
        (dict(out=pb + 128), "out overlaps vals"),
        (dict(out=pb + 264), "out overlaps row indices"),
        (dict(out=oi - 8), "out overlaps bad"),
    ]
    for kw, msg in cases:
        rc, err = lookup(**kw)
        assert rc == _lib.EINVAL and msg in err, (kw, err)
    assert lookup(k=0, ri=None, out=None)[0] == _lib.OK
    assert L.b2s_csr_select_scratch_bytes(-1) == 0 and L.b2s_csr_select_scratch_bytes(10) >= 256 + 80


# ---- the CPU dry run of tests/test_gpu_index.py: the three _ops wrappers restated -------------------------------------
def _dryrun_column_map(cols, ncols):
    c = cols.numpy().astype(np.int64)
    bad = int(((c < -ncols) | (c >= ncols)).sum())
    c = np.where(c < 0, c + ncols, c)
    ok = c[(c >= 0) & (c < ncols)]
    mptr = np.r_[0, np.cumsum(np.bincount(ok, minlength=ncols))].astype(np.int64)
    return torch.from_numpy(mptr), torch.from_numpy(np.argsort(c, kind="stable").astype(np.int64)), bad


def _dryrun_select(indptr, indices, data, shape, nrows_out, rows=None, row_start=0, row_step=1, col_map=None,
                   ncols_out=None, out_index_dtype=torch.int32):
    nrows, ncols = shape
    r = (np.arange(row_start, row_start + row_step * nrows_out, row_step) if rows is None
         else rows.numpy().astype(np.int64))
    bad = int(((r < -nrows) | (r >= nrows)).sum())
    if bad:
        return torch.zeros(nrows_out + 1, dtype=torch.int64), None, None, bad
    cols = None
    if col_map is not None:
        mptr, mpos = (t.numpy() for t in col_map)
        cols = np.empty(mpos.size, dtype=np.int64)
        cols[mpos] = np.repeat(np.arange(ncols), np.diff(mptr))
    ptr, idx, val = select_oracle(indptr.numpy(), indices.numpy(), data.numpy(), r, cols, ncols)
    return (torch.from_numpy(ptr), torch.from_numpy(idx).to(out_index_dtype), torch.from_numpy(np.ascontiguousarray(val)),
            0)


def _dryrun_lookup(indptr, indices, data, shape, ri, ci):
    m, n = shape
    i, j = ri.numpy().astype(np.int64), ci.numpy().astype(np.int64)
    ok = (i >= -m) & (i < m) & (j >= -n) & (j < n)
    out = np.zeros(i.size, dtype=data.numpy().dtype)
    out[ok] = lookup_oracle(indptr.numpy(), indices.numpy(), data.numpy(), shape, i[ok], j[ok])
    return torch.from_numpy(out), torch.tensor([int((~ok).sum())])


def test_gpu_file_passes_the_cpu_dry_run():
    script = (
        "import sys, pytest\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import dryrun_cpu\n"
        "dryrun_cpu.install()\n"
        "from legate.sparse_b200 import _ops\n"
        "import test_index_host\n"
        "_ops.csr_column_map = test_index_host._dryrun_column_map\n"
        "_ops.csr_select = test_index_host._dryrun_select\n"
        "_ops.csr_lookup = test_index_host._dryrun_lookup\n"
        "sys.exit(pytest.main(['-m', 'gpu', '-q', '-p', 'no:cacheprovider', sys.argv[1], '-k', sys.argv[2]]))\n"
    )
    # the full-size cases and the million-entry row are minutes of numpy here
    r = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "tests", "test_gpu_index.py"),
                        "not full_size and not million"], capture_output=True, text=True, timeout=900, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
