"""Host-side checks of `csc_array` (legate/sparse_b200/csc.py) and of the CSC products' C entry points
(csrc/csc.cu).

`csc_spmv` and `csc_spmm` restate the products in numpy (every stored entry (i, j) of column j adds vals * x[j] into
row i) and are pinned to scipy.  Construction, conversions and the `diags(...).tocsc()` path run on the host, as they do
without a GPU, and the entry points' argument checks are called through ctypes in a subprocess that sees no CUDA
device.  The `-m gpu` file is rehearsed through tests/dryrun_cpu.py with the `_ops` wrappers it needs swapped for the
restatements below."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200.csc import csc_array
from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, ROOT, mtx_path


def csc_spmv(indptr, indices, data, shape, x):
    """y = A x for the CSC matrix (indptr, indices, data) of `shape`, in np.result_type(data, x)."""
    m, n = shape
    dt = np.result_type(np.asarray(data).dtype, np.asarray(x).dtype)
    cols = np.repeat(np.arange(n), np.diff(np.asarray(indptr, dtype=np.int64)))
    y = np.zeros(m, dtype=dt)
    np.add.at(y, np.asarray(indices, dtype=np.int64), np.asarray(data, dtype=dt) * np.asarray(x, dtype=dt)[cols])
    return y


def csc_spmm(indptr, indices, data, shape, X):
    """Y = A X for a dense (n, k) X."""
    m, n = shape
    X = np.asarray(X)
    dt = np.result_type(np.asarray(data).dtype, X.dtype)
    cols = np.repeat(np.arange(n), np.diff(np.asarray(indptr, dtype=np.int64)))
    Y = np.zeros((m, X.shape[1]), dtype=dt)
    np.add.at(Y, np.asarray(indices, dtype=np.int64), np.asarray(data, dtype=dt)[:, None] * X.astype(dt)[cols])
    return Y


def _dryrun_spmv_csc(indptr, indices, data, x, y, shape):
    """`_ops.spmv_csc` for the CPU dry run of the GPU test file."""
    y.copy_(torch.from_numpy(csc_spmv(indptr.numpy(), indices.numpy(), data.numpy(), shape, x.numpy())))
    return y


def _dryrun_spmm_csc(indptr, indices, data, X, Y, shape):
    """`_ops.spmm_csc` for the CPU dry run of the GPU test file."""
    Y.copy_(torch.from_numpy(csc_spmm(indptr.numpy(), indices.numpy(), data.numpy(), shape, X.numpy())))
    return Y


def _dryrun_binop(op, a_indptr, a_indices, a_data, b_indptr, b_indices, b_data, shape):
    """`_ops.csr_binop` for the CPU dry run: scipy's canonical result."""
    A = sp.csr_array((a_data.numpy(), a_indices.numpy(), a_indptr.numpy()), shape=shape)
    B = sp.csr_array((b_data.numpy(), b_indices.numpy(), b_indptr.numpy()), shape=shape)
    C = sp.csr_array(A + B if op == "add" else A - B if op == "sub" else A.multiply(B))
    C.sort_indices()
    return (torch.from_numpy(C.indptr.astype(np.int64)), torch.from_numpy(C.indices.astype(np.int64)).to(a_indices.dtype),
            torch.from_numpy(C.data), {"nnz": C.nnz, "a_unsorted": False, "b_unsorted": False})


@pytest.fixture(autouse=True)
def _host_only(monkeypatch):
    """The host side as it runs without a GPU, also where one is visible: arrays stay on the host."""
    from legate.sparse_b200.runtime import Runtime

    monkeypatch.setattr(Runtime, "has_cuda", property(lambda self: False))


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _same_as_scipy(A, ref):
    """A (a csc_array) equals the scipy CSC `ref` in shape, dtype and values, and in its arrays once both are sorted."""
    assert isinstance(A, csc_array) and A.format == "csc" and A.ndim == 2
    assert A.shape == ref.shape and A.dtype == ref.dtype and A.nnz == ref.nnz
    assert np.array_equal(A.todense(), ref.toarray())
    A.sort_indices()
    ref = ref.copy()
    ref.sort_indices()
    assert np.array_equal(_np(A.indptr), ref.indptr) and np.array_equal(_np(A.indices), ref.indices)
    assert np.array_equal(_np(A.data), ref.data)


# ---- the numpy restatements --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MTX_FILES)
def test_restatements_match_scipy(name):
    S = sp.csc_array(scipy.io.mmread(mtx_path(name))).astype(np.float64)
    rng = np.random.default_rng(0)
    x = rng.standard_normal(S.shape[1])
    assert np.allclose(csc_spmv(S.indptr, S.indices, S.data, S.shape, x), S @ x, rtol=1e-12, atol=1e-12)
    for k in (0, 1, 3, 33):
        X = rng.standard_normal((S.shape[1], k))
        assert np.allclose(csc_spmm(S.indptr, S.indices, S.data, S.shape, X), S @ X, rtol=1e-12, atol=1e-12)


def test_restatements_sum_repeated_rows():
    # column 0: rows 2, 0, 2 (unsorted, repeated); column 1 empty; column 2: row 1
    indptr, indices, data = np.array([0, 3, 3, 4]), np.array([2, 0, 2, 1]), np.array([1.0, 2.0, 3.0, 4.0])
    S = sp.csc_array((data, indices, indptr), shape=(3, 3))
    x = np.array([1.0, 10.0, 100.0])
    assert np.array_equal(csc_spmv(indptr, indices, data, (3, 3), x), [2.0, 400.0, 4.0])
    assert np.array_equal(csc_spmv(indptr, indices, data, (3, 3), x), S @ x)
    assert np.array_equal(csc_spmm(indptr, indices, data, (3, 3), np.stack([x, -x], 1)), S @ np.stack([x, -x], 1))


# ---- construction ----------------------------------------------------------------------------------------------
def test_construction_from_every_input():
    rng = np.random.default_rng(1)
    ref = sp.random_array((7, 9), density=0.4, format="csc", rng=rng)
    D = ref.toarray()
    _same_as_scipy(csc_array(D), sp.csc_array(D))
    _same_as_scipy(csc_array(torch.from_numpy(D)), sp.csc_array(D))
    _same_as_scipy(csc_array(ref), ref)
    _same_as_scipy(csc_array(sp.csc_matrix(ref)), ref)
    for other in (ref.tocsr(), ref.tocoo(), sp.csr_matrix(ref), ref.todia()):
        _same_as_scipy(csc_array(other), ref)
    _same_as_scipy(csc_array((ref.data, ref.indices, ref.indptr), shape=ref.shape), ref)
    coo = ref.tocoo()
    _same_as_scipy(csc_array((coo.data, (coo.row, coo.col)), shape=ref.shape), sp.csc_array(coo))
    _same_as_scipy(csc_array(csr_array(ref.tocsr())), ref)
    _same_as_scipy(csc_array(sparse.coo_array(coo)), ref)
    _same_as_scipy(csc_array(ref, dtype=np.float32), ref.astype(np.float32))
    _same_as_scipy(csc_array(csc_array(ref), copy=True), ref)
    _same_as_scipy(sparse.csc_matrix(ref), ref)
    assert sparse.csc_matrix is sparse.csc_array is csc_array
    import sparse as alias

    assert alias.csc_array is csc_array and alias.csc_matrix is csc_array
    with pytest.raises(ValueError):
        csc_array(ref, shape=(9, 7))
    with pytest.raises(AssertionError):
        csc_array((ref.data, ref.indices, ref.indptr))
    with pytest.raises(NotImplementedError):
        csc_array("not a matrix")


def test_scipy_csc_keeps_unsorted_and_repeated_rows():
    indptr, indices, data = np.array([0, 3, 3, 4]), np.array([2, 0, 2, 1]), np.array([1.0, 2.0, 3.0, 4.0])
    S = sp.csc_array((data, indices, indptr), shape=(3, 3))
    A = csc_array(S)
    assert np.array_equal(_np(A.indices), indices) and np.array_equal(_np(A.data), data)
    assert not A.has_sorted_indices
    assert np.array_equal(A.toarray(), S.toarray())


def test_copies_do_not_share_arrays():
    S = sp.random_array((5, 6), density=0.5, format="csc", rng=np.random.default_rng(2))
    A = csc_array(S)
    B = A.copy()
    B.data[:] = 0
    assert np.array_equal(A.toarray(), S.toarray())
    C = A.astype(np.float32)
    assert C.dtype == np.float32 and A.dtype == np.float64
    assert A.tocsc() is A and A.tocsc(copy=True) is not A
    assert A.conj(copy=False).toarray().dtype == np.float64


# ---- conversions ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MTX_FILES)
def test_round_trips_on_fixtures(name):
    S = sp.csc_array(scipy.io.mmread(mtx_path(name))).astype(np.float64)
    A = csc_array(S)
    D = S.toarray()
    R = A.tocsr()
    assert isinstance(R, csr_array) and R is A.tocsr() and np.array_equal(R.toarray(), D)
    ref = S.tocsr()
    ref.sort_indices()
    assert np.array_equal(_np(R.indptr), ref.indptr) and np.array_equal(_np(R.indices), ref.indices)
    assert np.array_equal(A.tocsr(copy=True).toarray(), D)
    assert np.array_equal(A.tocoo().toarray(), D) and A.tocoo().shape == S.shape
    T = A.T
    assert isinstance(T, csr_array) and T is A.transpose() and np.array_equal(T.toarray(), D.T)
    assert np.array_equal(A.transpose(copy=True).toarray(), D.T)
    assert np.array_equal(csr_array(S.tocsr()).tocsc().toarray(), D)
    coo = sparse.io.mmread(mtx_path(name))
    assert np.array_equal(coo.tocsc().toarray(), sp.csc_array(scipy.io.mmread(mtx_path(name))).toarray())
    assert isinstance(coo.asformat("csc"), csc_array)
    assert isinstance(A.asformat("csr"), csr_array) and A.asformat("csc") is A
    sc = A.to_scipy_sparse_csc()
    assert isinstance(sc, sp.csc_array) and np.array_equal(sc.toarray(), D)
    assert np.array_equal(_np(A.diagonal()), S.diagonal())
    assert np.array_equal(csr_array(A).toarray(), D)
    assert sparse.is_sparse_matrix(A)


def test_diags_tocsc_gives_the_transpose_as_before():
    """`diags(...).tocsc().T` (examples/pde.py, gmg.py) is the csr_array `diags(..., format="csr").T`, array for
    array, and `.tocsr()` / `.todense()` are the matrix itself."""
    nx = 9
    a = 64.0
    diag_a = a * np.ones((nx - 2) ** 2 - 1)
    diag_a[nx - 3 :: nx - 2] = 0.0
    diag_g = a * np.ones((nx - 2) * (nx - 3))
    diag_c = -4 * a * np.ones((nx - 2) ** 2)
    args = ([diag_g, diag_a, diag_c, diag_a, diag_g], [-(nx - 2), -1, 0, 1, nx - 2])
    M = sparse.diags(*args, dtype=np.float64, format="csr")
    old_T = M.T
    for C in (sparse.diags(*args, dtype=np.float64).tocsc(), sparse.diags(*args, dtype=np.float64, format="csc")):
        assert isinstance(C, csc_array)
        T = C.T
        assert isinstance(T, csr_array)
        for got, want in ((T, old_T), (C.tocsr(), M)):
            assert got.shape == want.shape
            for f in ("indptr", "indices", "data"):
                g, w = getattr(got, f), getattr(want, f)
                assert g.dtype == w.dtype and torch.equal(g, w), f
        assert np.array_equal(C.todense(), M.todense())


# ---- no device -----------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    A = csc_array(sp.csc_array(scipy.io.mmread(mtx_path("test.mtx"))))
    for f in (lambda: A @ np.ones(5), lambda: A @ np.ones((5, 3)), lambda: A @ (np.ones(5) * 1j), lambda: A @ A):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            f()


def test_argument_errors_need_no_device():
    A = csc_array(sp.random_array((5, 6), density=0.5, format="csc", rng=np.random.default_rng(3)))
    with pytest.raises(ValueError):
        A @ np.ones(5)
    with pytest.raises(ValueError):
        A @ np.ones((4, 2))
    with pytest.raises(ValueError):
        A.dot(np.ones(6), out=np.empty(5, dtype=np.float32))
    with pytest.raises(ValueError):
        A.dot(np.ones(6), out=np.empty(4))
    with pytest.raises(NotImplementedError):
        A.astype(np.int64) @ np.ones(6, dtype=np.int64)
    with pytest.raises(NotImplementedError):
        A @ np.ones((6, 2, 2))
    with pytest.raises(ValueError):
        A @ csc_array(np.ones((5, 5)))
    with pytest.raises(ValueError):
        A + csc_array(np.ones((6, 5)))
    with pytest.raises(ValueError):
        A.sddmm(np.ones((5, 2)), np.ones((3, 6)))
    with pytest.raises(ValueError):
        A.sum(axis=2)


# ---- the C entry points' checks ---------------------------------------------------------------------------------
def _abi_failures():
    """Every rejected argument set of b2s_spmv_csc / b2s_spmm_csc, as 'name(kw): what happened' lines."""
    from legate.sparse_b200 import _lib

    L = _lib.lib
    buf = (ctypes.c_int64 * 2048)()
    base = ctypes.addressof(buf)

    def p(i):  # one 256-byte slot per array, so no two arguments overlap unless a case says so
        return base + 256 * i

    def spmv(vt=_lib.F64, it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4, x=p(3), y=p(4)):
        return L.b2s_spmv_csc(vt, it, pt, m, n, nnz, p(0), p(1), p(2), x, y, None)

    def spmm(vt=_lib.F64, it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4, k=2, X=p(3), ldx=2, Y=p(5), ldy=2):
        return L.b2s_spmm_csc(vt, it, pt, m, n, nnz, k, p(0), p(1), p(2), X, ldx, Y, ldy, None)

    common = [
        (dict(vt=7), "bad value type code 7"),
        (dict(it=5), "bad index type code 5"),
        (dict(pt=9), "bad indptr type code 9"),
        (dict(m=-1), "negative dimension"),
        (dict(n=-1), "negative dimension"),
        (dict(nnz=-1), "negative dimension"),
        (dict(nnz=2**31 - 1), "int32 indptr cannot address nnz >= 2^31-1"),
    ]
    cases = [("b2s_spmv_csc", spmv, kw, msg) for kw, msg in common]
    cases += [("b2s_spmm_csc", spmm, kw, msg) for kw, msg in common]
    cases += [
        ("b2s_spmv_csc", spmv, dict(y=p(3) + 8), "y overlaps x"),
        ("b2s_spmv_csc", spmv, dict(y=p(0)), "y overlaps indptr"),
        ("b2s_spmm_csc", spmm, dict(k=-1), "negative dimension"),
        ("b2s_spmm_csc", spmm, dict(Y=p(3) + 16), "Y overlaps X"),
        ("b2s_spmm_csc", spmm, dict(ldx=1), "leading dimensions (1, 2) smaller than k = 2"),
        ("b2s_spmm_csc", spmm, dict(ldy=1), "leading dimensions (2, 1) smaller than k = 2"),
    ]
    out = []
    for name, call, kw, msg in cases:
        rc = call(**kw)
        err = _lib.last_error()
        if rc != _lib.EINVAL or msg not in err:
            out.append(f"{name}({kw}): rc {rc}, {err!r}, expected EINVAL and {msg!r}")
    # an int64 indptr addresses 2^31 - 1 entries and more; nothing to compute needs no pointer at all
    if "int32 indptr" in (spmv(pt=_lib.I64, nnz=2**31 - 1), _lib.last_error())[1]:
        out.append("b2s_spmv_csc rejected an int64 indptr with nnz = 2^31-1")
    if spmv(m=0, n=0, nnz=0, x=None, y=None) != _lib.OK:
        out.append(f"b2s_spmv_csc of a 0 x 0 matrix: {_lib.last_error()!r}")
    if spmm(m=3, n=0, nnz=0, k=0, X=None, Y=None) != _lib.OK:
        out.append(f"b2s_spmm_csc with k = 0: {_lib.last_error()!r}")
    return out


def test_abi_rejects_bad_arguments():
    script = (
        "import sys\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import test_csc_host as t\n"
        "print('\\n'.join(t._abi_failures()))\n"
    )
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.strip() == "", r.stdout


def test_gpu_file_passes_the_cpu_dry_run():
    script = (
        "import sys, pytest\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import dryrun_cpu\n"
        "dryrun_cpu.install()\n"
        "from legate.sparse_b200 import _ops\n"
        "import test_csc_host, test_reduce_host, test_sddmm_host\n"
        "_ops.spmv_csc = test_csc_host._dryrun_spmv_csc\n"
        "_ops.spmm_csc = test_csc_host._dryrun_spmm_csc\n"
        "_ops.csr_binop = test_csc_host._dryrun_binop\n"
        "_ops.csr_reduce_rows = test_reduce_host._dryrun_reduce\n"
        "_ops.csr_sort_rows = test_reduce_host._dryrun_sort_rows\n"
        "_ops.sddmm = test_sddmm_host._dryrun_sddmm\n"
        "sys.exit(pytest.main(['-m', 'gpu', '-q', '-p', 'no:cacheprovider', sys.argv[1], '-k', sys.argv[2]]))\n"
    )
    # the 10M-row Laplacian is minutes of numpy here; CG's fused kernels have no stand-in
    r = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "tests", "test_gpu_csc.py"),
                        "not large_laplacian and not cg"], capture_output=True, text=True, timeout=900, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
