"""`csc_array` on the device: the scatter products of csrc/csc.cu (b2s_spmv_csc, b2s_spmm_csc) against scipy and
against exact references, and the surface delegated to the stored CSR transpose.

Floating-point atomics add a row's terms in an unspecified order, so products of general data are held to a bound of
the usual form |y - ref| <= c * u * (|A| |x|) and products of integer-valued data must be exact."""
import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import gallery, linalg
from legate.sparse_b200.csc import csc_array
from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, mtx_path, sample_spd

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
PAIRINGS = [(torch.int32, torch.int32), (torch.int32, torch.int64), (torch.int64, torch.int32),
            (torch.int64, torch.int64)]


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _fixture(name, dtype):
    return sp.csc_array(scipy.io.mmread(mtx_path(name))).astype(dtype)


def _close(got, S, x, dtype):
    """got against scipy's S @ x in float64, within 4 * (max column count + 2) units of roundoff of |S| |x|."""
    got = _np(got)
    assert got.dtype == np.dtype(dtype)
    S64 = S.astype(np.float64)
    ref = S64 @ np.asarray(x, dtype=np.float64)
    mag = abs(S64) @ np.abs(np.asarray(x, dtype=np.float64))
    u = np.finfo(dtype).eps
    terms = max(int(np.diff(S.tocsr().indptr).max()) if S.nnz else 0, 1) + 2
    assert got.shape == ref.shape
    assert np.all(np.abs(got - ref) <= 4 * terms * u * mag + 1e-300), np.max(np.abs(got - ref))


def _csc(indptr, indices, data, shape, it=torch.int32, pt=torch.int32):
    """A csc_array of `shape` with the given arrays at explicit index / indptr widths."""
    m, n = shape
    T = csr_array._from_parts(torch.as_tensor(np.asarray(indptr), dtype=pt).cuda(),
                              torch.as_tensor(np.asarray(indices), dtype=it).cuda(),
                              torch.as_tensor(np.asarray(data)).cuda(), (n, m))
    return csc_array._wrap(T)


def _exact_spmv(indptr, indices, data, shape, x):
    """Integer y = A x of a CSC matrix, summed in int64."""
    m, n = shape
    cols = np.repeat(np.arange(n), np.diff(np.asarray(indptr, dtype=np.int64)))
    y = np.zeros(m, dtype=np.int64)
    np.add.at(y, np.asarray(indices, dtype=np.int64), np.asarray(data, dtype=np.int64) * np.asarray(x)[cols])
    return y


def _exact_spmm(indptr, indices, data, shape, X):
    m, n = shape
    cols = np.repeat(np.arange(n), np.diff(np.asarray(indptr, dtype=np.int64)))
    Y = np.zeros((m, X.shape[1]), dtype=np.int64)
    np.add.at(Y, np.asarray(indices, dtype=np.int64), np.asarray(data, dtype=np.int64)[:, None] * X[cols])
    return Y


# ---- SpMV and SpMM against scipy ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_spmv_matches_scipy(name, dtype):
    S = _fixture(name, dtype)
    A = csc_array(S)
    m, n = S.shape
    x = np.random.default_rng(0).standard_normal(n).astype(dtype)
    y = A @ x
    assert isinstance(y, np.ndarray) and y.shape == (m,)
    _close(y, S, x, dtype)
    y2 = A.dot(x[:, None])
    assert y2.shape == (m, 1)
    _close(y2[:, 0], S, x, dtype)
    xt = torch.from_numpy(x).cuda()
    yt = A @ xt
    assert isinstance(yt, torch.Tensor) and yt.is_cuda
    _close(yt, S, x, dtype)
    out = np.empty(m, dtype=dtype)
    assert A.dot(x, out=out) is out
    _close(out, S, x, dtype)
    outd = torch.empty(m, dtype=yt.dtype, device="cuda")
    assert A.dot(xt, out=outd) is outd
    _close(outd, S, x, dtype)
    out2 = torch.empty((m, 1), dtype=yt.dtype, device="cuda")
    assert A.matvec(xt[:, None]).shape == (m, 1)
    A.dot(xt[:, None], out=out2)
    _close(out2[:, 0], S, x, dtype)


@pytest.mark.parametrize("name", MTX_FILES)
def test_mixed_dtypes_promote(name):
    S = _fixture(name, np.float32)
    A = csc_array(S)
    x64 = np.random.default_rng(1).standard_normal(S.shape[1])
    y = A @ x64
    _close(y, S.astype(np.float64), x64, np.float64)
    B = csc_array(S.astype(np.float64))
    x32 = x64.astype(np.float32)
    _close(B @ x32, S.astype(np.float64), x32, np.float64)
    with pytest.raises(ValueError):
        A.dot(x64, out=np.empty(S.shape[0], dtype=np.float32))
    with pytest.raises(NotImplementedError):
        A.astype(np.int64) @ np.ones(S.shape[1], dtype=np.int64)


@pytest.mark.parametrize("k", [0, 1, 3, 32, 33, 100])
@pytest.mark.parametrize("dtype", DTYPES)
def test_spmm_matches_scipy(k, dtype):
    rng = np.random.default_rng(k)
    for name in MTX_FILES:
        S = _fixture(name, dtype)
        A = csc_array(S)
        m, n = S.shape
        X = rng.standard_normal((n, k)).astype(dtype)
        Y = A @ X
        assert isinstance(Y, np.ndarray) and Y.shape == (m, k)
        for j in range(k):
            _close(Y[:, j], S, X[:, j], dtype)
        # strided rows, Fortran order, CUDA out
        Xs = torch.zeros((n, k + 5), dtype=torch.from_numpy(X).dtype, device="cuda")
        Xs[:, :k] = torch.from_numpy(X).cuda()
        Yt = A @ Xs[:, :k]
        assert isinstance(Yt, torch.Tensor) and tuple(Yt.shape) == (m, k)
        Yf = A @ np.asfortranarray(X)
        Yft = A @ torch.from_numpy(np.asfortranarray(X)).cuda().t().contiguous().t()
        out = torch.full((m, k), 7.0, dtype=Yt.dtype, device="cuda")
        assert A.dot(Xs[:, :k], out=out) is out
        outn = np.full((m, k), 7.0, dtype=dtype)
        A.dot(X, out=outn)
        for got in (Yt, Yf, Yft, out, outn):
            got = _np(got)
            for j in range(k):
                _close(got[:, j], S, X[:, j], dtype)


# ---- exact products on integer-valued data ------------------------------------------------------------------------
def _integer_cases():
    rng = np.random.default_rng(7)
    cases = []
    # unsorted and repeated rows within a column, empty columns (first, middle, last)
    indptr = np.array([0, 0, 4, 4, 4, 7, 9, 9])
    indices = np.array([3, 0, 3, 1, 2, 2, 0, 4, 0])
    data = rng.integers(-5, 6, indices.size).astype(np.float64)
    cases.append((indptr, indices, data, (5, 7)))
    # many empty columns inside one warp run (more than 32 columns end inside a 32-entry chunk)
    n = 300
    counts = np.zeros(n, dtype=np.int64)
    counts[rng.choice(n, 40, replace=False)] = rng.integers(1, 4, 40)
    indptr = np.concatenate([[0], np.cumsum(counts)])
    indices = rng.integers(0, 50, int(indptr[-1]))
    cases.append((indptr, indices, rng.integers(-3, 4, indices.size).astype(np.float64), (50, n)))
    # random, 10^5 columns, many runs
    S = sp.random_array((2000, 100000), density=2e-3, format="csc", rng=rng)
    cases.append((S.indptr, S.indices, rng.integers(-9, 10, S.nnz).astype(np.float64), S.shape))
    # nnz = 0, and empty shapes
    cases.append((np.zeros(6, dtype=np.int64), np.zeros(0, dtype=np.int64), np.zeros(0), (4, 5)))
    cases.append((np.zeros(6, dtype=np.int64), np.zeros(0, dtype=np.int64), np.zeros(0), (0, 5)))
    cases.append((np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int64), np.zeros(0), (4, 0)))
    return cases


@pytest.mark.parametrize("it,pt", PAIRINGS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_exact_on_integer_data(it, pt, dtype):
    rng = np.random.default_rng(11)
    for indptr, indices, data, shape in _integer_cases():
        A = _csc(indptr, indices, data.astype(dtype), shape, it, pt)
        m, n = shape
        x = rng.integers(-4, 5, n)
        y = A @ x.astype(dtype)
        assert y.dtype == np.dtype(dtype) and y.shape == (m,)
        assert np.array_equal(y, _exact_spmv(indptr, indices, data, shape, x).astype(dtype))
        for k in (1, 3, 33):
            X = rng.integers(-4, 5, (n, k))
            Y = A @ X.astype(dtype)
            assert np.array_equal(Y, _exact_spmm(indptr, indices, data, shape, X).astype(dtype))


@pytest.mark.parametrize("it,pt", PAIRINGS)
def test_one_column_holds_every_entry(it, pt):
    """A 1M x 3 matrix whose middle column holds all 10^6 entries (rows shuffled, some repeated): spread over
    thousands of warps, added up exactly."""
    rng = np.random.default_rng(3)
    m = 1 << 20
    rows = rng.permutation(m)
    rows[::97] = rows[5]                        # repeated rows
    indptr = np.array([0, 0, m, m])
    data = rng.integers(-3, 4, m).astype(np.float64)
    A = _csc(indptr, rows, data, (m, 3), it, pt)
    x = np.array([5.0, -2.0, 9.0])
    assert np.array_equal(A @ x, _exact_spmv(indptr, rows, data, (m, 3), x.astype(np.int64)).astype(np.float64))
    X = rng.integers(-2, 3, (3, 5))
    assert np.array_equal(A @ X.astype(np.float64), _exact_spmm(indptr, rows, data, (m, 3), X).astype(np.float64))


def test_large_laplacian_matches_the_csr_plan():
    """The 10M-row 5-point Laplacian is symmetric, so its CSC arrays are its CSR arrays: the scatter product and the
    tuned CSR plan read the same bytes and agree to fp64 rounding."""
    A = gallery.laplacian_5pt(3163, 3163, np.float64)
    C = csc_array._wrap(A)
    x = torch.rand(A.shape[1], dtype=torch.float64, device="cuda")
    y_csr = A @ x
    y_csc = C @ x
    ref_mag = torch.abs(A.data).max() * 5 * torch.abs(x).max()
    assert float(torch.max(torch.abs(y_csr - y_csc))) <= 16 * np.finfo(np.float64).eps * float(ref_mag)


# ---- complex -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MTX_FILES)
def test_complex_operands_and_matrices(name):
    rng = np.random.default_rng(5)
    for rdt, cdt in ((np.float32, np.complex64), (np.float64, np.complex128)):
        S = _fixture(name, rdt)
        A = csc_array(S)
        m, n = S.shape
        tol = dict(rtol=1e-4, atol=1e-4) if rdt == np.float32 else dict(rtol=1e-11, atol=1e-11)
        z = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(cdt)
        y = A @ z
        assert y.dtype == cdt and np.allclose(y, S @ z, **tol)
        Z = (rng.standard_normal((n, 3)) + 1j * rng.standard_normal((n, 3))).astype(cdt)
        assert np.allclose(_np(A @ torch.from_numpy(Z).cuda()), S @ Z, **tol)
        Sc = (S + 1j * S.multiply(S)).astype(cdt)
        Ac = csc_array(Sc)
        assert np.allclose(Ac @ z, Sc @ z, **tol)
        assert np.allclose(Ac @ np.real(z), Sc @ np.real(z), **tol)


# ---- the rest of the surface ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MTX_FILES)
def test_left_products_and_sparse_products(name):
    rng = np.random.default_rng(9)
    S = _fixture(name, np.float64)
    A = csc_array(S)
    m, n = S.shape
    x = rng.standard_normal(m)
    assert np.allclose(x @ A, x @ S, rtol=1e-12, atol=1e-12)
    X = rng.standard_normal((4, m))
    assert np.allclose(X @ A, X @ S, rtol=1e-12, atol=1e-12)
    Yt = A.__rmatmul__(torch.from_numpy(X).cuda())
    assert isinstance(Yt, torch.Tensor) and np.allclose(_np(Yt), X @ S, rtol=1e-12, atol=1e-12)
    St = S.T.tocsc()
    B = csc_array(St)
    C = A @ B
    assert isinstance(C, csc_array) and np.allclose(C.toarray(), (S @ St).toarray(), rtol=1e-12, atol=1e-12)
    R = sparse.csr_array(sp.csr_array(St))
    D = A @ R
    assert isinstance(D, csc_array) and np.allclose(D.toarray(), (S @ St).toarray(), rtol=1e-12, atol=1e-12)
    E = R @ A
    assert isinstance(E, csr_array) and np.allclose(E.toarray(), (St @ S).toarray(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", MTX_FILES)
def test_delegated_elementwise_sddmm_and_reductions(name):
    rng = np.random.default_rng(13)
    S = _fixture(name, np.float64)
    S2 = sp.csc_array(sp.random_array(S.shape, density=0.3, format="csc", rng=rng))
    A, B = csc_array(S), csc_array(S2)
    for got, ref in ((A + B, S + S2), (A - B, S - S2), (A.multiply(B), S.multiply(S2)), (A * B, S.multiply(S2)),
                     (A + sparse.csr_array(sp.csr_array(S2)), S + S2), (A * 2.5, S * 2.5), (-A, -S),
                     (abs(A), abs(S)), (A.power(2), S.power(2))):
        assert isinstance(got, csc_array)
        assert np.allclose(got.toarray(), ref.toarray(), rtol=1e-12, atol=1e-12)
    m, n = S.shape
    Cd, Dd = rng.standard_normal((m, 3)), rng.standard_normal((3, n))
    Q = A.sddmm(Cd, Dd)
    assert isinstance(Q, csc_array) and np.allclose(Q.toarray(), S.multiply(Cd @ Dd).toarray(), rtol=1e-12, atol=1e-12)
    D = S.toarray()
    for axis in (None, 0, 1, -1):
        assert np.allclose(_np(A.sum(axis=axis)), D.sum(axis=axis), rtol=1e-12, atol=1e-12)
        assert np.allclose(_np(A.mean(axis=axis)), D.mean(axis=axis), rtol=1e-12, atol=1e-12)
        assert np.array_equal(_np(A.max(axis=axis)), D.max(axis=axis))
        assert np.array_equal(_np(A.min(axis=axis)), D.min(axis=axis))
        assert np.array_equal(_np(A.count_nonzero(axis=axis)), np.count_nonzero(D, axis=axis))
    assert np.array_equal(_np(A.diagonal()), S.diagonal())


def test_conversions_on_the_device():
    S = _fixture("Ragusa18.mtx", np.float64)
    A = csc_array(S)
    R = A.tocsr()
    assert R is A.tocsr() and isinstance(R, csr_array)
    ref = S.tocsr()
    ref.sort_indices()
    assert np.array_equal(_np(R.indptr), ref.indptr) and np.array_equal(_np(R.indices), ref.indices)
    assert np.array_equal(_np(R.data), ref.data)
    assert np.array_equal(A.tocoo().toarray(), S.toarray())
    assert np.array_equal(sparse.csr_array(sp.csr_array(S)).tocsc().toarray(), S.toarray())
    x = np.random.default_rng(2).standard_normal(S.shape[1])
    assert np.allclose(A.tocsr() @ x, S @ x, rtol=1e-12, atol=1e-12)


def test_cg_on_a_csc_matrix():
    Ad, xs = sample_spd(400, 0.05, 17)
    b = Ad @ xs
    A_csr = sparse.csr_array(Ad)
    A_csc = sparse.csc_array(Ad)
    x1, it1 = linalg.cg(A_csr, b, tol=1e-10)
    x2, it2 = linalg.cg(A_csc, b, tol=1e-10)
    r1, r2 = np.linalg.norm(b - Ad @ x1), np.linalg.norm(b - Ad @ x2)
    assert r2 <= 1e-8 * np.linalg.norm(b) and r1 <= 1e-8 * np.linalg.norm(b)
    assert abs(it1 - it2) <= 25 and np.allclose(x1, x2, rtol=1e-8, atol=1e-10)
