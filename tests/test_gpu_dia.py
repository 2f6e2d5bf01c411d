"""`dia_array` on the device: the row-owned products of csrc/dia.cu (b2s_spmv_dia, b2s_spmm_dia) against scipy and
against exact references, the two conversions (b2s_dia_to_csr, b2s_csr_to_dia), and the surface delegated to the
cached CSR form.

Each row sums its diagonals in stored order, so products of general data are held to |y - ref| <= c * u * (|A| |x|)
against scipy in float64, products of integer-valued data must be exact, and two calls must agree bit for bit."""
import warnings

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import linalg
from legate.sparse_b200.dia import dia_array

from conftest import MTX_FILES, mtx_path

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _close(got, S, x, dtype):
    """got against scipy's S @ x in float64, within 4 * (diagonals + 2) units of roundoff of |S| |x|."""
    got = _np(got)
    assert got.dtype == np.dtype(dtype)
    S64 = sp.csr_array(S).astype(np.float64)
    xx = np.asarray(x, dtype=np.float64)
    ref, mag = S64 @ xx, abs(S64) @ np.abs(xx)
    u = np.finfo(dtype).eps
    terms = max(int(np.diff(S64.indptr).max()) if S64.nnz else 0, 1) + 2
    assert got.shape == ref.shape
    assert np.all(np.abs(got - ref) <= 4 * terms * u * mag + 1e-300), np.max(np.abs(got - ref))


def _quiet_todia(S):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
        return S.todia()


# square and rectangular both ways, L < n and L > n, unsorted offsets, offsets out of band, no diagonals
SHAPES = [((300, 300), [0, 1, -1, 5, -7], 300), ((200, 350), [3, -2, 0, 120, -150], 350),
          ((350, 200), [-100, 7, 0, -349, 199], 200), ((257, 257), [2, 0, -1], 100), ((257, 257), [1, 0, -3], 600),
          ((100, 100), [0, 2**62, -(2**62), 100, -100, 3], 100), ((64, 80), [], 80), ((0, 5), [0, 1], 5),
          ((5, 0), [0], 0), ((1, 1), [0], 1), ((1000, 1000), list(range(-300, 301, 2)), 1000)]


def _scipy(data, offsets, shape):
    """scipy's dia_array of the same matrix: scipy stores offsets at its index width, so the diagonals at +-2^62 (which
    hold nothing) are left out of it."""
    offsets = np.asarray(offsets, dtype=np.int64)
    keep = np.abs(offsets) < 2**31
    return sp.dia_array((np.asarray(data)[keep], offsets[keep]), shape=shape)


def _random(rng, shape, offsets, L, dtype):
    """(scipy's matrix, ours) with the same random diagonals"""
    data = rng.standard_normal((len(offsets), L)).astype(dtype)
    return _scipy(data, offsets, shape), dia_array((data, offsets), shape=shape)


# ---- SpMV and SpMM against scipy ---------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(SHAPES)))
@pytest.mark.parametrize("dtype", DTYPES)
def test_spmv_matches_scipy_on_banded_matrices(case, dtype):
    shape, offsets, L = SHAPES[case]
    rng = np.random.default_rng(case)
    S, A = _random(rng, shape, offsets, L, dtype)
    m, n = shape
    x = rng.standard_normal(n).astype(dtype)
    y = A @ x
    assert isinstance(y, np.ndarray) and y.shape == (m,)
    _close(y, S, x, dtype)
    xt = torch.from_numpy(x).cuda()
    yt = A @ xt
    assert isinstance(yt, torch.Tensor) and yt.is_cuda
    _close(yt, S, x, dtype)
    assert A.dot(x[:, None]).shape == (m, 1)
    _close(A.dot(x[:, None])[:, 0], S, x, dtype)
    out = np.empty(m, dtype=dtype)
    assert A.dot(x, out=out) is out
    _close(out, S, x, dtype)
    outd = torch.empty(m, dtype=yt.dtype, device="cuda")
    assert A.dot(xt, out=outd) is outd
    _close(outd, S, x, dtype)
    out2 = torch.empty((m, 1), dtype=yt.dtype, device="cuda")
    A.dot(xt[:, None], out=out2)
    _close(out2[:, 0], S, x, dtype)
    assert torch.equal(A @ xt, A @ xt)   # same bits on every call


@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_products_match_scipy_on_fixtures(name, dtype):
    S = _quiet_todia(sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(dtype))
    A = dia_array(S)
    rng = np.random.default_rng(1)
    x = rng.standard_normal(S.shape[1]).astype(dtype)
    _close(A @ x, S, x, dtype)
    X = rng.standard_normal((S.shape[1], 5)).astype(dtype)
    got = A @ X
    for j in range(5):
        _close(got[:, j], S, X[:, j], dtype)


@pytest.mark.parametrize("k", [0, 1, 3, 32, 33, 100])
@pytest.mark.parametrize("dtype", DTYPES)
def test_spmm_matches_scipy(k, dtype):
    rng = np.random.default_rng(k)
    for case in (0, 1, 2, 4, 5):
        shape, offsets, L = SHAPES[case]
        S, A = _random(rng, shape, offsets, L, dtype)
        m, n = shape
        X = rng.standard_normal((n, k)).astype(dtype)
        Y = A @ X
        assert isinstance(Y, np.ndarray) and Y.shape == (m, k)
        for j in range(k):
            _close(Y[:, j], S, X[:, j], dtype)
        Xt = torch.from_numpy(X).cuda()
        ref = A @ Xt
        assert ref.is_cuda and torch.equal(ref.cpu(), torch.from_numpy(Y))
        # strided rows and Fortran order give the same bits
        wide = torch.zeros((n, k + 7), dtype=Xt.dtype, device="cuda")
        wide[:, :k] = Xt
        assert torch.equal(A @ wide[:, :k], ref)
        assert torch.equal(A @ Xt.t().contiguous().t(), ref)
        np.testing.assert_array_equal(A @ np.asfortranarray(X), Y)
        out = torch.empty((m, k + 3), dtype=Xt.dtype, device="cuda")[:, :k]
        assert A.dot(Xt, out=out) is out and torch.equal(out, ref)
        outh = np.empty((m, k), dtype=dtype)
        assert A.dot(X, out=outh) is outh
        np.testing.assert_array_equal(outh, Y)


@pytest.mark.parametrize("dtype", DTYPES)
def test_exact_on_integer_data(dtype):
    rng = np.random.default_rng(7)
    for shape, offsets, L in SHAPES:
        data = rng.integers(-8, 9, (len(offsets), L)).astype(dtype)
        S = _scipy(data.astype(np.int64), offsets, shape)
        A = dia_array((data, offsets), shape=shape)
        x = rng.integers(-8, 9, shape[1])
        np.testing.assert_array_equal(A @ x.astype(dtype), (S @ x).astype(dtype))
        X = rng.integers(-8, 9, (shape[1], 3))
        np.testing.assert_array_equal(A @ X.astype(dtype), (S @ X).astype(dtype))


def test_mixed_dtypes_promote():
    S, A = _random(np.random.default_rng(2), (50, 60), [0, 3, -4], 60, np.float32)
    x64 = np.random.default_rng(3).standard_normal(60)
    _close(A @ x64, S.astype(np.float64), x64, np.float64)
    with pytest.raises(ValueError):
        A.dot(x64, out=np.empty(50, dtype=np.float32))
    with pytest.raises(NotImplementedError):
        A.astype(np.int64) @ np.ones(60, dtype=np.int64)


# ---- transposed and complex products --------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [0, 1, 2, 3, 4, 5])
def test_left_and_transposed_products(case):
    shape, offsets, L = SHAPES[case]
    rng = np.random.default_rng(10 + case)
    S, A = _random(rng, shape, offsets, L, np.float64)
    D = S.toarray()
    x = rng.standard_normal(shape[0])
    np.testing.assert_allclose(x @ A, x @ D, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(A.T @ x, D.T @ x, rtol=1e-12, atol=1e-12)
    X = rng.standard_normal((4, shape[0]))
    np.testing.assert_allclose(X @ A, X @ D, rtol=1e-12, atol=1e-12)
    Xt = torch.from_numpy(X).cuda()
    got = Xt @ A
    assert isinstance(got, torch.Tensor) and got.is_cuda
    np.testing.assert_allclose(_np(got), X @ D, rtol=1e-12, atol=1e-12)
    # A @ sparse is the CSR SpGEMM of tocsr()
    B = sp.random_array((shape[1], 9), density=0.2, rng=rng, format="csr")
    C = A @ sparse.csr_array(B)
    np.testing.assert_allclose(C.todense(), D @ B.toarray(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose((A @ B).todense(), D @ B.toarray(), rtol=1e-12, atol=1e-12)


def test_complex_operands_and_matrices():
    rng = np.random.default_rng(11)
    S, A = _random(rng, (120, 90), [0, 1, -5, 30], 90, np.float64)
    D = S.toarray()
    z = rng.standard_normal(90) + 1j * rng.standard_normal(90)
    np.testing.assert_allclose(A @ z, D @ z, rtol=1e-12, atol=1e-12)
    Z = rng.standard_normal((90, 3)) + 1j * rng.standard_normal((90, 3))
    np.testing.assert_allclose(A @ Z, D @ Z, rtol=1e-12, atol=1e-12)
    Zt = torch.from_numpy(Z.astype(np.complex64)).cuda()
    np.testing.assert_allclose(_np(A.astype(np.float32) @ Zt), D @ Z, rtol=1e-4, atol=1e-4)
    Ac = dia_array((S.data * (1 + 2j), S.offsets), shape=S.shape)
    np.testing.assert_allclose(Ac @ z, (D * (1 + 2j)) @ z, rtol=1e-12, atol=1e-12)


# ---- conversions --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_dia_to_csr_matches_the_tensor_route(dtype):
    rng = np.random.default_rng(12)
    for shape, offsets, L in SHAPES:
        data = rng.standard_normal((len(offsets), L)).astype(dtype)
        if data.size:
            data[rng.random(data.shape) < 0.2] = 0.0
            data[rng.random(data.shape) < 0.05] = -0.0
            data[rng.random(data.shape) < 0.05] = np.nan
            data[0] = 0.0    # an all-zero diagonal
        A = dia_array((data, offsets), shape=shape)
        C, R = A.tocsr(), A._tocsr_tensor_ops()
        assert C.indptr.dtype == R.indptr.dtype and C.indices.dtype == R.indices.dtype
        assert torch.equal(C.indptr.cpu(), R.indptr.cpu()) and torch.equal(C.indices.cpu(), R.indices.cpu())
        np.testing.assert_array_equal(_np(C.data), _np(R.data))
        assert C.data.dtype == (torch.float64 if dtype == np.float64 else torch.float32)
    # diags gives the arrays of the old host route: int32 widths, zeros dropped
    C = sparse.diags([[1.0, 0.0, 2.0], [-0.0, np.nan]], [0, 1], format="csr")
    assert C.indptr.dtype == torch.int32 and C.indices.dtype == torch.int32
    assert _np(C.indptr).tolist() == [0, 1, 2, 3] and _np(C.indices).tolist() == [0, 2, 2]


@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_csr_to_dia_matches_scipy(name, dtype):
    S = sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
        R = S.todia()
        A = sparse.csr_array(S).todia()
    np.testing.assert_array_equal(_np(A.offsets), R.offsets)
    np.testing.assert_array_equal(_np(A.data), R.data)


def test_csr_to_dia_sums_repeated_entries_and_warns():
    rows, cols = np.array([0, 0, 2, 3, 3]), np.array([1, 1, 0, 3, 3])
    vals = np.array([1.0, 2.0, 4.0, 1.0, -1.0])
    A = sparse.coo_array((torch.from_numpy(vals).cuda(), (torch.from_numpy(rows).cuda(), torch.from_numpy(cols).cuda())),
                         shape=(4, 4)).todia()
    R = sp.coo_array((vals, (rows, cols)), shape=(4, 4)).todia()
    np.testing.assert_array_equal(_np(A.offsets), R.offsets)
    np.testing.assert_array_equal(_np(A.data), R.data)
    n = 300
    W = sp.csr_array((np.ones(n), (np.arange(n), np.random.default_rng(0).permutation(n))), shape=(n, n))
    with pytest.warns(sp.SparseEfficiencyWarning):
        B = sparse.csr_array(W).todia()
    with pytest.warns(sp.SparseEfficiencyWarning):
        R = W.todia()
    np.testing.assert_array_equal(_np(B.offsets), R.offsets)


def test_csr_to_dia_too_large_raises_before_allocating():
    n = 1 << 20
    rng = np.random.default_rng(13)
    W = sp.random_array((n, n), density=4.0 / n, rng=rng, format="csr")
    A = sparse.csr_array(W)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
        with pytest.raises(ValueError, match="free bytes"):
            A.todia()
    assert torch.cuda.max_memory_allocated() < before + (1 << 33)


# ---- large matrices -------------------------------------------------------------------------------------------------
def test_large_laplacian_matches_csr():
    nx = ny = 3163   # about 10M rows
    n = nx * ny
    main = np.full(n, 4.0)
    side = -np.ones(n - 1)
    side[np.arange(1, n) % nx == 0] = 0.0
    A = sparse.diags([main, side, side, -np.ones(n - nx), -np.ones(n - nx)], [0, 1, -1, nx, -nx])
    assert isinstance(A, dia_array)
    x = torch.from_numpy(np.random.default_rng(14).standard_normal(n)).cuda()
    y, ref = A @ x, A.tocsr() @ x
    torch.testing.assert_close(y, ref, rtol=1e-13, atol=1e-12)
    assert torch.equal(A @ x, y)


def test_large_int64_element_offsets():
    L = (1 << 29) + 1000
    need = 5 * L * 4 * 2 + L * 4 * 2
    if torch.cuda.mem_get_info()[0] < need + (2 << 30):
        pytest.skip("not enough free device memory for 5 fp32 diagonals of 2^29 + 1000")
    data = torch.ones((5, L), dtype=torch.float32, device="cuda")
    data[4] = 2.0
    A = dia_array((data, [-2, -1, 0, 1, 2]), shape=(L, L))
    x = torch.ones(L, dtype=torch.float32, device="cuda")
    y = A @ x
    assert float(y[L // 2]) == 6.0 and float(y[-1]) == 3.0 and float(y[0]) == 4.0
    assert float(y[-3]) == 6.0 and float(y[-2]) == 4.0
    del data, x, y


# ---- in-place edits, solvers, delegated surface -----------------------------------------------------------------------
def test_in_place_edit_is_seen_by_the_next_product():
    S, A = _random(np.random.default_rng(15), (64, 64), [0, 1, -1], 64, np.float64)
    x = np.ones(64)
    y0 = A @ x
    A.data[1, 5] += 1.0
    y1 = A @ x
    assert y1[4] == y0[4] + 1.0
    C = A.tocsr()
    A.data.mul_(2.0)
    np.testing.assert_allclose(A @ x, 2 * y1, rtol=1e-15)
    assert A.tocsr() is not C


def test_solvers_agree_with_the_csr_form():
    n = 400
    A = sparse.diags([np.full(n, 4.0), -np.ones(n - 1), -np.ones(n - 1), -0.5 * np.ones(n - 20)], [0, 1, -1, 20])
    S = sparse.diags([np.full(n, 4.0), -np.ones(n - 1), -np.ones(n - 1)], [0, 1, -1])
    b = np.random.default_rng(16).standard_normal(n)
    x1, _ = linalg.cg(S, b, tol=1e-10)
    x2, _ = linalg.cg(S.tocsr(), b, tol=1e-10)
    np.testing.assert_allclose(x1, x2, rtol=1e-8, atol=1e-10)
    g1, _ = linalg.gmres(A, b, tol=1e-10)
    g2, _ = linalg.gmres(A.tocsr(), b, tol=1e-10)
    np.testing.assert_allclose(g1, g2, rtol=1e-8, atol=1e-10)
    l1 = linalg.lsqr(A, b)[0]
    l2 = linalg.lsqr(A.tocsr(), b)[0]
    np.testing.assert_allclose(l1, l2, rtol=1e-8, atol=1e-10)


def test_delegated_surface_agrees_with_tocsr():
    rng = np.random.default_rng(17)
    S, A = _random(rng, (40, 50), [0, 2, -3], 50, np.float64)
    C = A.tocsr()
    B = sparse.csr_array(sp.random_array((40, 50), density=0.2, rng=rng, format="csr"))
    D = rng.standard_normal((40, 50))
    for got, ref in ((A + B, C + B), (A - B, C - B), (A + A, C + C), (A.multiply(B), C.multiply(B)),
                     (A.multiply(A), C.multiply(C))):
        np.testing.assert_array_equal(got.todense(), ref.todense())
    np.testing.assert_array_equal(_np(A + D), _np(C + D))
    for axis in (None, 0, 1):
        np.testing.assert_array_equal(_np(A.sum(axis=axis)), _np(C.sum(axis=axis)))
        np.testing.assert_array_equal(_np(A.mean(axis=axis)), _np(C.mean(axis=axis)))
        np.testing.assert_array_equal(_np(A.max(axis=axis)), _np(C.max(axis=axis)))
        np.testing.assert_array_equal(_np(A.min(axis=axis)), _np(C.min(axis=axis)))
    X, Y = rng.standard_normal((40, 4)), rng.standard_normal((4, 50))
    np.testing.assert_array_equal(_np(A.sddmm(X, Y).data), _np(C.sddmm(X, Y).data))
    np.testing.assert_array_equal((A * 2.0).todense(), 2.0 * S.toarray())
    np.testing.assert_array_equal((-A).todense(), -S.toarray())
    np.testing.assert_array_equal(abs(A).todense(), abs(S).toarray())
    assert A.count_nonzero() == S.count_nonzero()
    np.testing.assert_array_equal(A.tocsc().todense(), S.toarray())
    assert (sparse.csr_array(B.T.to_scipy_sparse_csr()) @ A).shape == (50, 50)
    import sparse as alias

    x = np.ones(3)
    np.testing.assert_array_equal(alias.diags([[1.0, 2.0, 3.0], [4.0, 5.0]], [0, 1]) @ x,
                                  sp.diags_array([[1.0, 2.0, 3.0], [4.0, 5.0]], offsets=[0, 1]) @ x)
    np.testing.assert_array_equal(alias.eye(4, format="dia") @ np.arange(4.0), np.arange(4.0))
