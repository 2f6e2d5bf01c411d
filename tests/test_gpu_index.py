"""csr_array indexing (csrc/index.cu) against scipy and the host restatement in test_index_host.py: bit for bit against
the restatement, and against scipy where requested columns are unique (in canonical form otherwise)."""
import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200 import gallery
from legate.sparse_b200.csr import _index_key, csr_array

from conftest import MTX_FILES, mtx_path
from test_index_host import _canonical_equal, _keys, _sel, lookup_oracle, select_oracle

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _parts(B):
    return _np(B.indptr).astype(np.int64), _np(B.indices).astype(np.int64), _np(B.data)


def _same(B, want):
    ptr, idx, val = _parts(B)
    wp, wi, wv = want
    assert np.array_equal(ptr, wp) and np.array_equal(idx, wi), (ptr, wp, idx, wi)
    assert val.dtype == np.asarray(wv).dtype and np.array_equal(val.view(np.uint8), np.asarray(wv).view(np.uint8))


def _unique_cols(key):
    cols = key[1] if isinstance(key, tuple) and len(key) == 2 else None
    if cols is None or not isinstance(cols, (list, np.ndarray)):
        return True
    a = np.asarray(cols).ravel()
    return a.dtype == bool or len(set(a.tolist())) == a.size


def _check_key(A, S, key):
    B = A[key]
    want, shape = _sel(S, key)
    assert B.shape == shape
    _same(B, want)
    W = sp.csr_matrix(S)[key]
    if _unique_cols(key):
        assert np.array_equal(_np(B.indices), W.indices) and np.array_equal(_np(B.data), W.data)
    else:
        assert _canonical_equal(*_parts(B), B.shape, W)
    assert B.indptr.dtype == (torch.int32 if B.nnz < 2**31 - 1 else torch.int64)


@pytest.mark.parametrize("name", MTX_FILES)
def test_fixtures_every_key(name):
    S = sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(np.float64)
    A = csr_array(S)
    m, n = S.shape
    for key in _keys(m, n):
        _check_key(A, S, key)
    # elements and pointwise pairs
    rng = np.random.default_rng(1)
    ri, ci = rng.integers(-m, m, 500), rng.integers(-n, n, 500)
    want = lookup_oracle(S.indptr, S.indices, S.data, S.shape, ri, ci)
    got = A[ri, ci]
    assert isinstance(got, np.ndarray) and np.array_equal(got, want)
    assert np.array_equal(got, np.asarray(sp.csr_matrix(S)[ri, ci]).ravel())
    gd = A[torch.from_numpy(ri).cuda(), torch.from_numpy(ci).cuda()]
    assert isinstance(gd, torch.Tensor) and gd.is_cuda and np.array_equal(_np(gd), want)
    assert np.array_equal(A[list(ri[:5]), list(ci[:5])], want[:5])
    for i, j in zip(ri[:20], ci[:20]):
        v = A[int(i), int(j)]
        assert isinstance(v, np.float64) and v == S[int(i), int(j)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64, np.complex128])
def test_value_types(dtype):
    S = sp.random_array((300, 200), density=0.05, format="csr", rng=np.random.default_rng(2)).astype(dtype)
    if np.dtype(dtype).kind == "c":
        S.data = S.data + 1j * np.random.default_rng(3).standard_normal(S.nnz)
    A = csr_array(S)
    p = np.random.default_rng(4).permutation(300)
    for key in (p, (slice(None), p[:150] % 200), np.ix_(p[:100], p[:100] % 200), (slice(5, 250, 3), [7, 7, 3])):
        _check_key(A, S, key)
    if np.dtype(dtype).kind != "c":
        assert A[3, 4] == S[3, 4]


@pytest.mark.parametrize("pt", [torch.int32, torch.int64])
@pytest.mark.parametrize("it", [torch.int32, torch.int64])
def test_index_widths_bitwise(it, pt, monkeypatch):
    lens = np.r_[np.random.default_rng(0).integers(0, 40, 2000), [500, 0, 33, 5000, 4096, 4097]]
    rng = np.random.default_rng(1)
    n = 6000
    indptr = np.r_[0, np.cumsum(lens)]
    S = sp.csr_array((rng.standard_normal(indptr[-1]), rng.integers(0, n, indptr[-1]), indptr), shape=(len(lens), n))
    A = csr_array(S)
    B = csr_array._from_parts(A.indptr.to(pt), A.indices.to(it), A.data, A.shape)
    p, q = rng.permutation(len(lens)), rng.integers(0, n, 3000)
    keys = [p, (slice(None), q), np.ix_(p[:1000], q), (slice(None, None, -1), slice(None, None, 2))]
    for key in keys:
        want = A[key]
        got = B[key]
        assert torch.equal(got.indptr, want.indptr) and torch.equal(got.indices, want.indices)
        assert torch.equal(got.data, want.data)
    assert np.array_equal(B[p[:50], q[:50]], A[p[:50], q[:50]])
    monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    for key in keys:
        W = B[key]
        assert W.indptr.dtype == W.indices.dtype == torch.int64
        _same(W, tuple(x for x in _parts(A[key])))


def test_bin_boundaries_and_repeats():
    # rows on both sides of the lane (32) and warp (4096) limits, under a column map with repeated columns
    pattern = [0, 1, 31, 32, 33, 4095, 4096, 4097, 9000, 2]
    lens = np.array(pattern * 3)
    n = 9001
    rng = np.random.default_rng(5)
    indptr = np.r_[0, np.cumsum(lens)]
    S = sp.csr_array((rng.integers(-9, 10, indptr[-1]).astype(np.float64), rng.integers(0, n, indptr[-1]), indptr),
                     shape=(len(lens), n))
    A = csr_array(S)
    cols = np.r_[rng.integers(0, n, 4000), [0, 0, 0, 5, 5]]
    for key in ((slice(None), cols), (slice(None, None, -1), cols[::-1]), np.ix_([3, 3, -1, 7, 8, 8], cols),
                (slice(None), slice(None, None, -1)), (slice(None), np.r_[np.arange(n), np.arange(n)])):
        _check_key(A, S, key)


def test_million_entry_row():
    n = (1 << 20) + 77
    rng = np.random.default_rng(6)
    cols = rng.integers(0, n, n + 11)
    S = sp.csr_array((rng.standard_normal(n + 11), cols, [0, 0, n + 11, n + 11]), shape=(3, n))
    A = csr_array(S)
    for key in ([1, 1, 0], (slice(None), rng.permutation(n)), (1, rng.integers(0, n, 5000))):
        B = A[key]
        want, shape = _sel(S, key)
        _same(B, want)


def test_empty_and_degenerate():
    for shape in ((0, 5), (5, 0), (0, 0)):
        A = csr_array(sp.csr_array(shape))
        B = A[:, :]
        assert B.shape == shape and B.nnz == 0
        assert A[[], :].shape == (0, shape[1])
        assert A[:, []].shape == (shape[0], 0)
    S = sp.csr_array(np.array([[0.0, 1.0], [0.0, 0.0], [2.0, 0.0]]))
    A = csr_array(S)
    assert A[1].nnz == 0 and A[1].shape == (1, 2)
    assert A[[], []].shape == (0,)
    assert A[2:0, :].shape == (0, 2)
    assert A[:, 5:].shape == (3, 0)


def test_out_of_range_raises():
    A = csr_array(sp.random_array((6, 7), density=0.5, format="csr", rng=np.random.default_rng(7)))
    dev = torch.device("cuda")
    for key in ((6, 0), (0, -8), ([0, 6], slice(None)), (slice(None), [7]), ([1], [9]),
                (torch.tensor([0, 6], device=dev), slice(None)), (torch.tensor([-7], device=dev), slice(None)),
                (slice(None), torch.tensor([7], device=dev)), (slice(None), torch.tensor([-8], device=dev)),
                (torch.tensor([0, 1], device=dev), torch.tensor([0, 7], device=dev)),
                (torch.tensor([6], device=dev), torch.tensor([0], device=dev)),
                (torch.ones(5, dtype=torch.bool, device=dev), slice(None))):
        with pytest.raises(IndexError):
            A[key]


def test_cuda_and_list_indices_match_numpy():
    S = sp.random_array((50, 40), density=0.2, format="csr", rng=np.random.default_rng(8))
    A = csr_array(S)
    rng = np.random.default_rng(9)
    r, c = rng.integers(-50, 50, 30), rng.integers(-40, 40, 25)
    mask = rng.random(40) < 0.5
    want = A[np.ix_(r, c)]
    for key in ((torch.from_numpy(r).cuda(), slice(None)), (slice(None), torch.from_numpy(c).cuda()),
                (list(r), slice(None)), (slice(None), list(c)), (slice(None), torch.from_numpy(mask).cuda()),
                (torch.from_numpy(r).cuda().reshape(-1, 1), torch.from_numpy(c).cuda().reshape(1, -1))):
        host = tuple(k.cpu().numpy() if isinstance(k, torch.Tensor) else k for k in key)
        _same(A[key], _parts(A[host]))
    _same(A[torch.from_numpy(r).cuda()][:, torch.from_numpy(c).cuda()], _parts(want))
    _same(A[np.ix_(r, c)], select_oracle(S.indptr, S.indices, S.data, r, c, 40))


def test_arrays_and_stamp_unchanged_and_repeatable():
    A = gallery.rmat(14)
    stamp, cached = A._stamp(), set(A._cache)
    keep = tuple(t.clone() for t in (A.indptr, A.indices, A.data))
    p = torch.from_numpy(np.random.default_rng(12).permutation(A.shape[0])).cuda()
    B1 = A[p][:, p]
    B2 = A[p][:, p]
    assert torch.equal(B1.indptr, B2.indptr) and torch.equal(B1.indices, B2.indices) and torch.equal(B1.data, B2.data)
    assert A._stamp() == stamp and set(A._cache) == cached
    for t, k in zip((A.indptr, A.indices, A.data), keep):
        assert torch.equal(t, k)
    B1.data.zero_()
    assert torch.equal(A.data, keep[2])


def test_full_size_laplacian_symmetric_permutation():
    A = gallery.laplacian_5pt(3162, 3162, np.float64)
    n = A.shape[0]
    rng = np.random.default_rng(10)
    p = rng.permutation(n)
    q = np.argsort(p)
    B = A[np.ix_(p, p)]
    S = A.to_scipy_sparse_csr()
    W = S[np.ix_(p, p)]
    assert np.array_equal(_np(B.indptr), W.indptr) and np.array_equal(_np(B.indices), W.indices)
    assert np.array_equal(_np(B.data), W.data)
    C = B[np.ix_(q, q)]
    assert torch.equal(C.indptr, A.indptr) and torch.equal(C.indices, A.indices) and torch.equal(C.data, A.data)


def test_full_size_rmat_half_mask():
    A = gallery.rmat(20)
    rng = np.random.default_rng(11)
    mask = rng.random(A.shape[0]) < 0.5
    S = A.to_scipy_sparse_csr()
    for key in (mask, (slice(None), mask), np.ix_(mask.nonzero()[0], mask.nonzero()[0])):
        B = A[key]
        W = S[key]
        assert np.array_equal(_np(B.indptr), W.indptr) and np.array_equal(_np(B.indices), W.indices)
        assert np.array_equal(_np(B.data), W.data)
    ri, ci = rng.integers(0, A.shape[0], 1 << 20), rng.integers(0, A.shape[1], 1 << 20)
    got = A[torch.from_numpy(ri).cuda(), torch.from_numpy(ci).cuda()]
    assert np.array_equal(_np(got), np.asarray(S[ri, ci]).ravel())
