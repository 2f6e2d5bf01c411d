"""kron, kronsum, bmat, hstack, vstack and block_diag (csrc/construct.cu) on the device: bit for bit against the host
restatement in test_construct_host.py, and against scipy's format="csr" result on canonical inputs."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import gallery
from legate.sparse_b200.csr import csr_array

from test_construct_host import _parts, assert_same_csr, bmat_oracle, kron_oracle

pytestmark = pytest.mark.gpu

DTYPES_ALL = [np.float32, np.float64, np.complex64, np.complex128]


def _rand(m, n, density, dtype, seed):
    S = sp.random(m, n, density=density, format="csr", random_state=seed, dtype=np.float64)
    S.data[:] = np.random.default_rng(seed).standard_normal(S.nnz)
    if np.dtype(dtype).kind == "c":
        S = (S + 1j * S).astype(dtype)
    return S.astype(dtype)


def _same(C, ref):
    """C (a csr_array) equals the (indptr, indices, data) `ref` in indptr, indices and data bytes"""
    p, i, v = ref
    assert np.array_equal(C.indptr.cpu().numpy().astype(np.int64), p)
    assert np.array_equal(C.indices.cpu().numpy().astype(np.int64), i)
    d = C.data.cpu().numpy()
    assert d.dtype == np.asarray(v).dtype and d.tobytes() == np.asarray(v).tobytes()


def _wide(S):
    """the library operand of S with int64 indices and indptr"""
    return csr_array._from_parts(torch.from_numpy(S.indptr.astype(np.int64)).cuda(),
                                 torch.from_numpy(S.indices.astype(np.int64)).cuda(), torch.from_numpy(S.data).cuda(),
                                 S.shape)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_kron_matches_oracle_and_scipy(dtype):
    A, B = _rand(40, 30, 0.1, dtype, 1), _rand(17, 23, 0.2, dtype, 2)
    C = sparse.kron(csr_array(A), csr_array(B))
    _same(C, kron_oracle(_parts(A), _parts(B)))
    assert_same_csr((C.indptr.cpu(), C.indices.cpu(), C.data.cpu().numpy()), sp.kron(A, B, format="csr"))
    assert C.has_sorted_indices
    # mixed operand widths, dense operands and a mixed dtype
    D = np.roll(A.toarray(), 1)
    C2 = sparse.kron(_wide(A), torch.from_numpy(D))
    _same(C2, kron_oracle(_parts(A), _parts(sp.csr_array(D))))
    C3 = sparse.kron(csr_array(A.astype(np.float32)), csr_array(B.astype(np.float64)))
    assert C3.dtype == np.float64


def test_kron_keeps_stored_order_duplicates_and_zeros():
    p, i, v = np.array([0, 3, 3, 5]), np.array([2, 0, 2, 1, 0]), np.array([1.0, 0.0, 3.0, -0.0, 5.0])
    A = sp.csr_array((v, i, p), shape=(3, 3))
    B = sp.csr_array((np.array([2.0, 0.5, 0.0]), np.array([1, 0, 1]), np.array([0, 2, 3])), shape=(2, 2))
    C = sparse.kron(csr_array(A), csr_array(B))
    _same(C, kron_oracle(_parts(A), _parts(B)))
    assert C.nnz == A.nnz * B.nnz


def test_kron_long_rows_and_wide_columns(monkeypatch):
    # one output row of 2^20 entries: 512 emit CTAs
    a, b = np.arange(1, 1025, dtype=np.float64)[None, :], np.linspace(-1, 1, 1024)[None, :]
    A, B = sp.csr_array(a), sp.csr_array(b)
    C = sparse.kron(csr_array(A), csr_array(B))
    _same(C, kron_oracle(_parts(A), _parts(B)))
    # 2^32 output columns with few entries: int64 output indices
    A = sp.csr_array((np.array([1.0, 2.0, 3.0]), np.array([0, 7, 2**20 - 1]), np.array([0, 3])), shape=(1, 2**20))
    B = sp.csr_array((np.array([-1.0, 4.0]), np.array([5, 2**12 - 1]), np.array([0, 2])), shape=(1, 2**12))
    C = sparse.kron(csr_array(A), csr_array(B))
    assert C.shape == (1, 2**32) and C.indices.dtype == torch.int64
    _same(C, kron_oracle(_parts(A), _parts(B)))
    # B2S_INDEX_WIDTH=64 keeps the wide instantiations
    monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    A, B = _rand(30, 20, 0.2, np.float64, 3), _rand(9, 11, 0.3, np.float64, 4)
    C = sparse.kron(csr_array(A), csr_array(B))
    assert C.indices.dtype == torch.int64 and C.indptr.dtype == torch.int64
    _same(C, kron_oracle(_parts(A), _parts(B)))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_kronsum_matches_scipy(dtype):
    A, B = _rand(12, 12, 0.3, dtype, 5), _rand(7, 7, 0.4, dtype, 6)
    C = sparse.kronsum(csr_array(A), csr_array(B))
    S = sp.kronsum(A, B, format="csr")
    C.eliminate_zeros()
    S.eliminate_zeros()
    S.sort_indices()
    assert_same_csr((C.indptr.cpu(), C.indices.cpu(), C.data.cpu().numpy()), S)
    with pytest.raises(NotImplementedError):
        sparse.kronsum(csr_array(A.astype(np.complex64)), csr_array(B))


def _tridiag(n, s):
    return sparse.diags([s * np.ones(n - 1), -2 * s * np.ones(n), s * np.ones(n - 1)], [-1, 0, 1], format="csr")


@pytest.mark.parametrize("n1,n2", [(5, 7), (3162, 3162)])
def test_kronsum_of_tridiagonals_is_the_5_point_laplacian(n1, n2):
    a, g = float((n1 + 1) ** 2), float((n2 + 1) ** 2)
    C = sparse.kronsum(_tridiag(n1, a), _tridiag(n2, g))
    L = gallery.laplacian_5pt(n1, n2, np.float64)
    for x, y in ((C.indptr, L.indptr), (C.indices, L.indices)):
        assert torch.equal(x.to(torch.int64), y.to(torch.int64))
    assert torch.equal(C.data.view(torch.int64), L.data.view(torch.int64))


def _grid_parts(grid):
    heights = [next(b.shape[0] for b in row if b is not None) for row in grid]
    widths = [next(row[j].shape[1] for row in grid if row[j] is not None) for j in range(len(grid[0]))]
    ro, co = np.r_[0, np.cumsum(heights)], np.r_[0, np.cumsum(widths)]
    placed = [(int(ro[i]), int(co[j]), _parts(b)) for i, row in enumerate(grid) for j, b in enumerate(row)
              if b is not None]
    return placed, (int(ro[-1]), int(co[-1]))


@pytest.mark.parametrize("dtype", DTYPES_ALL)
def test_bmat_stacking_and_block_diag_match_oracle_and_scipy(dtype):
    A, B, E = _rand(50, 40, 0.1, dtype, 7), _rand(50, 25, 0.2, dtype, 8), _rand(30, 25, 0.0, dtype, 9)
    Z = sp.csr_array((0, 40), dtype=dtype)
    grid = [[A, B], [None, E], [Z, None]]
    C = sparse.bmat([[None if b is None else csr_array(b) for b in row] for row in grid])
    placed, shape = _grid_parts(grid)
    _same(C, bmat_oracle(placed, shape))
    S = sp.bmat(grid, format="csr")
    S.sort_indices()
    assert_same_csr((C.indptr.cpu(), C.indices.cpu(), C.data.cpu().numpy()), S)
    assert C.has_sorted_indices
    H = sparse.hstack([csr_array(A), _wide(B)])
    _same(H, bmat_oracle(*_grid_parts([[A, B]])))
    V = sparse.vstack([csr_array(B), csr_array(E)])
    _same(V, bmat_oracle(*_grid_parts([[B], [E]])))
    D = sparse.block_diag([csr_array(A), _wide(B), E])
    placed = [(0, 0, _parts(A)), (50, 40, _parts(B)), (100, 65, _parts(E))]
    _same(D, bmat_oracle(placed, (130, 90)))
    assert D.dtype == np.dtype(dtype)


def test_bmat_casts_to_the_result_dtype_and_coo_round_trips():
    A, B = _rand(20, 20, 0.2, np.float32, 10), _rand(20, 10, 0.2, np.float64, 11)
    C = sparse.hstack([csr_array(A), csr_array(B)])
    assert C.dtype == np.float64
    _same(C, bmat_oracle(*_grid_parts([[A.astype(np.float64), B]])))
    C = sparse.hstack([csr_array(A), csr_array(B)], dtype=np.complex128)
    assert C.dtype == np.complex128
    K = sparse.kron(csr_array(A), csr_array(B), format="coo")
    assert isinstance(K, sparse.coo_array)
    assert np.array_equal(K.todense(), sp.kron(A, B).toarray().astype(np.float64))
    Bc = sparse.block_diag([csr_array(A), 2.0, [[1.0, 0.0], [0.0, 3.0]]], format="coo")
    assert np.array_equal(Bc.tocsr().todense(), sp.block_diag([A, 2.0, [[1.0, 0.0], [0.0, 3.0]]]).toarray())


def test_long_rows_span_many_emit_ctas_and_index_width_64(monkeypatch):
    rng = np.random.default_rng(12)
    rows = [sp.csr_array(rng.standard_normal((2, 1 << 18))) for _ in range(3)]
    C = sparse.hstack([csr_array(r) for r in rows])
    _same(C, bmat_oracle(*_grid_parts([rows])))
    monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    A, B = _rand(40, 30, 0.2, np.float64, 13), _rand(40, 20, 0.2, np.float64, 14)
    C = sparse.bmat([[csr_array(A), None], [None, csr_array(B)]])
    assert C.indices.dtype == torch.int64 and C.indptr.dtype == torch.int64
    _same(C, bmat_oracle(*_grid_parts([[A, None], [None, B]])))


def test_block_diag_of_ten_thousand_blocks():
    rng = np.random.default_rng(15)
    mats = [sp.csr_array(rng.standard_normal((1 + k % 5, 1 + k % 3)) * (rng.random((1 + k % 5, 1 + k % 3)) < 0.7))
            for k in range(10_000)]
    C = sparse.block_diag([csr_array(M) for M in mats])
    placed, r, c = [], 0, 0
    for M in mats:
        placed.append((r, c, _parts(M)))
        r, c = r + M.shape[0], c + M.shape[1]
    _same(C, bmat_oracle(placed, (r, c)))
    assert_same_csr((C.indptr.cpu(), C.indices.cpu(), C.data.cpu().numpy()), sp.block_diag(mats, format="csr"))


def test_alias_exports():
    import sparse as alias

    A = _rand(6, 6, 0.5, np.float64, 16)
    for name in ("kron", "kronsum", "bmat", "hstack", "vstack", "block_diag"):
        assert getattr(alias, name) is getattr(sparse, name)
    assert np.array_equal(alias.kron(csr_array(A), csr_array(A)).todense(), sp.kron(A, A).toarray())
