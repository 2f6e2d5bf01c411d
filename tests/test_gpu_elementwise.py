"""Sparse + sparse, sparse - sparse and elementwise products of `csr_array` (csrc/elementwise.cu) against scipy.

Canonical inputs: C's structure is the union (add / subtract) or intersection (multiply) of the two patterns, with
explicit zeros kept; after `eliminate_zeros()` the arrays are bit-for-bit scipy's, because every value is one rounding
of the same operands.  Non-canonical inputs (unsorted rows, repeated columns) are compared to a tolerance, and the
caller's arrays must come back untouched."""
import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import gallery
from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, mtx_path

pytestmark = pytest.mark.gpu

OPS = {"add": lambda x, y: x + y, "sub": lambda x, y: x - y, "mul": lambda x, y: x.multiply(y)}


def _fixture(name):
    return sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(np.float64)


def _random_like(S, seed, density=0.3):
    m, n = S.shape
    return sp.random_array((m, n), density=density, format="csr", dtype=np.float64, rng=np.random.default_rng(seed))


def _pattern(S):
    P = S.copy()
    P.data = np.ones_like(P.data)
    return P


def _bits(x):
    x = np.asarray(x)
    return x.view(np.uint32 if x.dtype == np.float32 else np.uint64)


def _same_values(x, y):
    """Bitwise equal, except that NaNs only need to sit at the same places (the GPU does not keep NaN payloads)."""
    x, y = np.asarray(x), np.asarray(y)
    if x.dtype != y.dtype or x.shape != y.shape:
        return False
    nx, ny = np.isnan(x), np.isnan(y)
    return np.array_equal(nx, ny) and np.array_equal(_bits(x[~nx]), _bits(y[~ny]))


def _host(C):
    return C.indptr.cpu().numpy(), C.indices.cpu().numpy(), C.data.cpu().numpy()


def _restrict(R, P):
    """The entries of R inside the pattern P.  scipy's multiply visits the union of the two patterns and keeps
    NaN * (absent entry) = NaN; the product here is defined on the intersection, as the reference's mult()."""
    R, P = R.tocoo(), P.tocoo()
    n = R.shape[1]
    keep = np.isin(R.row.astype(np.int64) * n + R.col, P.row.astype(np.int64) * n + P.col)
    return sp.csr_array((R.data[keep], (R.row[keep], R.col[keep])), shape=R.shape)


def _check(As, Bs, op):
    """C = A op B through csr_array: structure first, then the pruned form bitwise against scipy."""
    A, B = csr_array(As), csr_array(Bs)
    C = OPS[op](A, B)
    assert isinstance(C, csr_array) and C.shape == As.shape
    P = OPS["mul" if op == "mul" else "add"](_pattern(As), _pattern(Bs))
    P = sp.csr_array(P)
    P.sort_indices()
    ptr, idx, _ = _host(C)
    assert np.array_equal(ptr, P.indptr) and np.array_equal(idx, P.indices)
    assert C.has_sorted_indices
    C.eliminate_zeros()
    R = sp.csr_array(OPS[op](As, Bs))
    if op == "mul":
        R = _restrict(R, P)
    R.sort_indices()
    ptr, idx, val = _host(C)
    assert np.array_equal(ptr, R.indptr) and np.array_equal(idx, R.indices)
    assert _same_values(val, R.data.astype(val.dtype))
    assert val.dtype == np.result_type(As.dtype, Bs.dtype)
    return C


@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("op", sorted(OPS))
def test_fixtures(name, op):
    S = _fixture(name)
    if S.shape[0] == S.shape[1]:
        _check(S, sp.csr_array(S.T), op)
    _check(S, _random_like(S, 7), op)
    _check(S, S, op)


@pytest.mark.parametrize("dts", [(np.float64, np.float64), (np.float32, np.float32), (np.float32, np.float64)])
@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("op", sorted(OPS))
def test_dtypes_and_widths(dts, wide, op, monkeypatch):
    if wide:
        monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    rng = np.random.default_rng(11)
    As = sp.random_array((300, 200), density=0.05, format="csr", dtype=np.float64, rng=rng).astype(dts[0])
    Bs = sp.random_array((300, 200), density=0.08, format="csr", dtype=np.float64, rng=rng).astype(dts[1])
    C = _check(As, Bs, op)
    want = torch.int64 if wide else torch.int32
    assert C.indptr.dtype == want and C.indices.dtype == want


def _with_rows(m, n, lengths, seed):
    """Random CSR matrix whose row r has lengths[r] distinct sorted columns."""
    rng = np.random.default_rng(seed)
    cols = [np.sort(rng.choice(n, size=k, replace=False)) for k in lengths]
    indptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    indices = np.concatenate(cols).astype(np.int64) if cols else np.zeros(0, np.int64)
    data = rng.standard_normal(indices.shape[0])
    return sp.csr_array((data, indices, indptr), shape=(m, n))


@pytest.mark.parametrize("op", sorted(OPS))
def test_shapes_and_bins(op):
    rng = np.random.default_rng(3)
    m, n = 700, 9000
    la = rng.integers(0, 12, size=m)
    lb = rng.integers(0, 12, size=m)
    la[rng.random(m) < 0.2] = 0                       # empty rows
    la[5], lb[5] = 40, 30                             # a warp row
    la[6], lb[6] = 6000, 2500                         # longer than every warp row: a CTA row
    la[300:428] = 20                                  # a tile whose short rows need two staging rounds
    lb[300:428] = 12
    As, Bs = _with_rows(m, n, la, 1), _with_rows(m, n, lb, 2)
    _check(As, Bs, op)
    _check(As, As, op)
    _check(As[:, :4000], Bs[:, 5000:], op)            # rectangular, different column ranges
    Z = sp.csr_array((m, n), dtype=np.float64)
    _check(Z, Z, op)                                  # nnz = 0
    _check(As, Z, op)
    _check(sp.csr_array((0, 5)), sp.csr_array((0, 5)), op)


@pytest.mark.parametrize("op", sorted(OPS))
def test_signed_zeros_and_nans(op):
    rng = np.random.default_rng(5)
    As = sp.random_array((200, 150), density=0.1, format="csr", dtype=np.float64, rng=rng)
    Bs = sp.random_array((200, 150), density=0.1, format="csr", dtype=np.float64, rng=rng)
    k = As.data.shape[0]
    As.data[: k // 4] = -0.0
    As.data[k // 4 : k // 3] = 0.0
    As.data[k // 3 : k // 3 + 5] = np.nan
    Bs.data[::7] = -Bs.data[::7]
    Bs.data[::11] = -0.0
    _check(As, Bs, op)
    _check(As, As, op)
    _check(Bs, As, op)


def _messy(m, n, seed):
    """(data, indices, indptr) with shuffled rows and repeated columns, and the scipy matrix they stand for."""
    rng = np.random.default_rng(seed)
    rows = []
    for r in range(m):
        k = int(rng.integers(0, 9)) if r != 3 else 3000
        c = rng.integers(0, n, size=k)
        if k > 2:
            c[1] = c[0]
        rows.append(rng.permutation(c))
    indptr = np.concatenate([[0], np.cumsum([len(c) for c in rows])]).astype(np.int32)
    indices = np.concatenate(rows).astype(np.int32)
    data = rng.standard_normal(indices.shape[0])
    S = sp.csr_array((data.copy(), indices.copy(), indptr.copy()), shape=(m, n))
    return (data, indices, indptr), S


@pytest.mark.parametrize("op", sorted(OPS))
def test_noncanonical_inputs(op):
    m, n = 400, 5000
    (da, ia, pa), Sa = _messy(m, n, 1)
    (db, ib, pb), Sb = _messy(m, n, 2)
    A = csr_array((torch.from_numpy(da).cuda(), torch.from_numpy(ia).cuda(), torch.from_numpy(pa).cuda()), shape=(m, n))
    B = csr_array((torch.from_numpy(db).cuda(), torch.from_numpy(ib).cuda(), torch.from_numpy(pb).cuda()), shape=(m, n))
    assert not A.has_sorted_indices and not B.has_sorted_indices
    before = [t.clone() for t in (A.indptr, A.indices, A.data, B.indptr, B.indices, B.data)]
    C = OPS[op](A, B)
    for t0, t in zip(before, (A.indptr, A.indices, A.data, B.indptr, B.indices, B.data)):
        assert torch.equal(t0, t)
    assert C.has_sorted_indices
    ptr, idx = C.indptr.cpu().numpy(), C.indices.cpu().numpy()
    for r in range(m):
        assert np.all(np.diff(idx[ptr[r]:ptr[r + 1]]) > 0)
    ref = OPS[op](Sa, Sb)
    np.testing.assert_allclose(C.todense(), ref.toarray(), rtol=1e-12, atol=1e-12)
    # sort_indices sorts in place and leaves the values with their columns
    A.sort_indices()
    assert A.has_sorted_indices
    np.testing.assert_allclose(A.todense(), Sa.toarray(), rtol=1e-12, atol=1e-12)


@pytest.fixture(scope="module")
def l5():
    return gallery.laplacian_5pt(3162, 3162, np.float64)


def test_l5_full_size(l5):
    A = l5
    C = A + A
    assert torch.equal(C.indptr, A.indptr) and torch.equal(C.indices, A.indices)
    assert torch.equal((2 * A.data).view(torch.int64), C.data.view(torch.int64))
    del C
    D = A - A
    assert D.nnz == A.nnz
    D.eliminate_zeros()
    assert D.nnz == 0 and int(D.indptr[-1]) == 0
    del D
    sigma = 0.375
    S = A - sigma * sparse.eye(A.shape[0])
    rows = torch.repeat_interleave(torch.arange(A.shape[0], device="cuda"),
                                   (A.indptr[1:] - A.indptr[:-1]).to(torch.int64))
    want = torch.where(A.indices.to(torch.int64) == rows, A.data - sigma, A.data)
    assert torch.equal(S.indptr, A.indptr) and torch.equal(S.indices, A.indices)
    assert torch.equal(S.data.view(torch.int64), want.view(torch.int64))


def test_l5_fp32_multiply(l5):
    A = l5.astype(np.float32)
    C = A.multiply(A)
    assert torch.equal(C.indices, A.indices)
    assert torch.equal(C.data.view(torch.int32), (A.data * A.data).view(torch.int32))


@pytest.mark.parametrize("kind", ["numpy", "torch"])
def test_dense_operands(kind):
    rng = np.random.default_rng(9)
    m, n = 120, 90
    As = sp.random_array((m, n), density=0.1, format="csr", dtype=np.float64, rng=rng)
    A = csr_array(As)
    conv = (lambda x: x) if kind == "numpy" else (lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda())
    back = (lambda x: np.asarray(x)) if kind == "numpy" else (lambda x: x.cpu().numpy())
    for D in (rng.standard_normal((m, 1)), rng.standard_normal((1, n)), rng.standard_normal(n),
              rng.standard_normal((m, n))):
        C = A.multiply(conv(D))
        assert isinstance(C, csr_array)
        assert torch.equal(C.indptr, A.indptr) and torch.equal(C.indices, A.indices)
        assert np.array_equal(C.todense(), np.asarray(As.multiply(D).toarray() if sp.issparse(As.multiply(D))
                                                      else As.multiply(D)))
        assert np.array_equal((A * conv(D)).todense(), C.todense())
    D = rng.standard_normal((m, n))
    for got, want in ((A + conv(D), As.toarray() + D), (conv(D) + A, D + As.toarray()),
                      (A - conv(D), As.toarray() - D), (conv(D) - A, D - As.toarray())):
        assert isinstance(got, np.ndarray if kind == "numpy" else torch.Tensor)
        assert np.array_equal(back(got), want)
    D32 = conv(rng.standard_normal((m, n)).astype(np.float32))
    assert A.multiply(D32).dtype == np.float64          # promotion


def test_operand_kinds_and_scalars():
    rng = np.random.default_rng(4)
    As = sp.random_array((80, 80), density=0.1, format="csr", dtype=np.float64, rng=rng)
    Bs = sp.random_array((80, 80), density=0.1, format="csr", dtype=np.float64, rng=rng)
    A = csr_array(As)
    ref = (As + Bs).toarray()
    for B in (Bs, sp.coo_array(Bs), sparse.coo_array(Bs.tocoo()), csr_array(Bs)):
        assert np.array_equal((A + B).todense(), ref)
        assert np.array_equal((B + A).todense(), (Bs + As).toarray())
        assert np.array_equal((A - B).todense(), (As - Bs).toarray())
        assert np.array_equal((B - A).todense(), (Bs - As).toarray())
    d = rng.standard_normal(80)
    Dg = sparse.diags([d, d[:79]], [0, 1], shape=(80, 80))
    Ds = sp.diags_array([d, d[:79]], offsets=[0, 1], shape=(80, 80))
    assert np.array_equal((A + Dg).todense(), (As + Ds).toarray())
    assert np.array_equal(A.multiply(Dg).todense(), As.multiply(Ds).toarray())
    assert np.array_equal((A + 0).todense(), As.toarray()) and (A + 0) is not A
    assert np.array_equal(sum([A, A, A]).todense(), (As + As + As).toarray())
    with pytest.raises(NotImplementedError):
        A + 1.5
    with pytest.raises(NotImplementedError):
        A - 2


def test_errors():
    A = csr_array(sp.random_array((10, 12), density=0.3, format="csr", dtype=np.float64, rng=np.random.default_rng(1)))
    B = csr_array(sp.random_array((12, 10), density=0.3, format="csr", dtype=np.float64, rng=np.random.default_rng(2)))
    for f in (lambda: A + B, lambda: A - B, lambda: A.multiply(B), lambda: A.multiply(np.ones((3, 3)))):
        with pytest.raises(ValueError):
            f()
    Z = sp.random_array((10, 12), density=0.3, format="csr", dtype=np.complex128, rng=np.random.default_rng(3))
    for f in (lambda: A + Z, lambda: A - Z, lambda: A.multiply(Z), lambda: A.multiply(np.ones((10, 12), np.complex128))):
        with pytest.raises(NotImplementedError):
            f()


def test_eliminate_zeros_drops_plan():
    A = gallery.laplacian_5pt(40, 40, np.float64)
    x = torch.rand(A.shape[1], dtype=torch.float64, device="cuda")
    D = A - sparse.diags([A.diagonal().cpu().numpy()], [0], shape=A.shape)
    assert D.nnz == A.nnz
    D @ x                                             # builds a plan for the structure with explicit zeros
    D.eliminate_zeros()
    assert D.nnz == A.nnz - A.shape[0]
    Ds = A.to_scipy_sparse_csr()
    Ds.setdiag(0)
    Ds.eliminate_zeros()
    assert np.array_equal(D.indptr.cpu().numpy(), Ds.indptr) and np.array_equal(D.indices.cpu().numpy(), Ds.indices)
    torch.testing.assert_close(D @ x, torch.from_numpy(Ds @ x.cpu().numpy()).cuda(), rtol=1e-13, atol=1e-13)
