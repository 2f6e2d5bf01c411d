"""csr_array sum / mean / max / min / argmax / argmin / count_nonzero (csrc/reduce.cu) against scipy, numpy on
`toarray()` and the host restatement in test_reduce_host.py; abs and power against scipy; and the AMG example's
strength of connection with theta > 0 against the same script on scipy."""
import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200 import _ops, gallery
from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, mtx_path
from test_gpu_amg import parse, run
from test_reduce_host import reduce_oracle

pytestmark = pytest.mark.gpu

AXES = [None, 0, 1, -1, -2]
EXTREMES = ["max", "min", "argmax", "argmin"]


def _np(x):
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    if hasattr(x, "toarray"):
        return x.toarray()
    return np.asarray(x)


def _scipy(S, op, axis, explicit=False):
    if op in ("argmax", "argmin") and axis is None and explicit:
        # scipy 1.18 returns the position in its canonical data here; this library the flat index i * n + j
        C = S.tocoo()
        C.sum_duplicates()
        k = getattr(S, op)(explicit=True)
        return np.asarray(int(C.row[k]) * S.shape[1] + int(C.col[k]))
    if op in EXTREMES:
        return _np(getattr(S, op)(axis=axis, explicit=explicit))
    if op == "count_nonzero":
        return _np(S.count_nonzero(axis=axis))
    return _np(getattr(S, op)(axis=axis))


def _check(got, want, op, dtype):
    got = _np(got)
    assert got.shape == want.shape, (got.shape, want.shape)
    if op in ("sum", "mean"):
        tol = 1e-5 if dtype == np.float32 else 1e-12
        np.testing.assert_allclose(got, want, rtol=tol, atol=tol)
    else:
        np.testing.assert_array_equal(got, want)


def _random(m, n, lens=None, seed=0, lo=-3, hi=4, dups=True, dtype=np.float64):
    """A csr_array with the given row lengths (random otherwise), unsorted columns (repeating when `dups`) and small
    integer values, so that sums in any order are exact; with its scipy twin."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 2 * n if dups else n, m) if lens is None else np.asarray(lens)
    if dups:
        indices = rng.integers(0, n, int(lens.sum()))
    else:
        indices = np.concatenate([rng.permutation(n)[:k] for k in lens]) if m else np.zeros(0, dtype=np.int64)
    indptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    data = rng.integers(lo, hi, int(indptr[-1])).astype(dtype)
    S = sp.csr_array((data, indices, indptr), shape=(m, n))
    return csr_array(S), S


@pytest.mark.parametrize("explicit", [False, True])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", ["sum", "mean", "count_nonzero"] + EXTREMES)
@pytest.mark.parametrize("name", MTX_FILES)
def test_fixtures_against_scipy(name, op, dtype, explicit):
    if explicit and op not in EXTREMES:
        return                                   # `explicit` only exists for the extremes
    S = sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(dtype)
    A = csr_array(S)
    kw = {"explicit": explicit} if op in EXTREMES else {}
    for axis in AXES:
        got = getattr(A, op)(axis=axis, **kw)
        if axis is None:
            assert np.isscalar(got)
            if op in ("argmax", "argmin", "count_nonzero"):
                assert type(got) is int
        else:
            assert isinstance(got, torch.Tensor) and got.is_cuda and got.ndim == 1
            assert got.dtype == (torch.int64 if op in ("argmax", "argmin", "count_nonzero") else A.data.dtype)
        _check(got, _scipy(S, op, axis, explicit), op, dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_nan_rows_follow_numpy(dtype):
    S = sp.csr_array(scipy.io.mmread(mtx_path("Ragusa18.mtx"))).astype(dtype)
    S.data[::7] = np.nan
    A = csr_array(S)
    D = S.toarray()
    with np.errstate(invalid="ignore"):
        for axis in (None, 0, 1):
            for op in EXTREMES:
                _check(getattr(A, op)(axis=axis), np.asarray(getattr(D, op)(axis=axis)), op, dtype)
            np.testing.assert_allclose(_np(A.sum(axis=axis)), D.sum(axis=axis), rtol=1e-5)


def test_sum_dtype_and_out():
    S = sp.csr_array(scipy.io.mmread(mtx_path("GlossGT.mtx"))).astype(np.float32)
    A = csr_array(S)
    D = S.toarray().astype(np.float64)
    for axis in (None, 0, 1):
        got = A.sum(axis=axis, dtype=np.float64)
        assert (got.dtype == np.float64) if axis is None else (got.dtype == torch.float64)
        np.testing.assert_allclose(_np(got), D.sum(axis=axis), rtol=1e-12)
        got = A.mean(axis=axis, dtype=np.float64)
        np.testing.assert_allclose(_np(got), D.mean(axis=axis), rtol=1e-12)
    for axis, shape in ((0, S.shape[1]), (1, S.shape[0])):
        out_t = torch.zeros(shape, dtype=torch.float32, device="cuda")
        assert A.sum(axis=axis, out=out_t) is out_t
        np.testing.assert_allclose(_np(out_t), D.sum(axis=axis), rtol=1e-5)
        out_n = np.zeros(shape, dtype=np.float64)
        assert A.mean(axis=axis, dtype=np.float64, out=out_n) is out_n
        np.testing.assert_allclose(out_n, D.mean(axis=axis), rtol=1e-12)
    out0 = np.zeros((), dtype=np.float32)
    assert A.sum(out=out0) is out0
    np.testing.assert_allclose(out0, D.sum(), rtol=1e-5)


@pytest.mark.parametrize("pt", [torch.int32, torch.int64])
@pytest.mark.parametrize("it", [torch.int32, torch.int64])
def test_index_widths_bitwise(it, pt, monkeypatch):
    lens = np.r_[np.random.default_rng(0).integers(0, 40, 3000), [500, 0, 33, 900]]
    A, S = _random(len(lens), 900, lens=lens, seed=1, dups=False)
    A.data.copy_(torch.randn(A.nnz, dtype=torch.float64, device="cuda"))   # sums that round
    B = csr_array._from_parts(A.indptr.to(pt), A.indices.to(it), A.data, A.shape)
    monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    W = csr_array(A.to_scipy_sparse_csr())
    assert W.indptr.dtype == W.indices.dtype == torch.int64
    for op in ["sum", "count_nonzero"] + EXTREMES:
        for axis in (0, 1):
            want = getattr(A, op)(axis=axis)
            assert torch.equal(getattr(B, op)(axis=axis), want), (op, axis)
            assert torch.equal(getattr(W, op)(axis=axis), want), (op, axis)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_row_lengths_around_the_warp_threshold(dtype):
    pattern = [0, 1, 31, 32, 33, 5000, 2, 0, 64, 31, 32, 33, 3, 0, 1, 4096, 6000, 6000]
    lens = np.array((pattern * 40)[:611])
    A, S = _random(len(lens), 6001, lens=lens, seed=2, lo=-1000, hi=1000, dups=False, dtype=dtype)
    S.sort_indices()
    for op in ["sum", "count_nonzero"] + EXTREMES:
        for explicit in ((False, True) if op in EXTREMES else (False,)):
            kw = {"explicit": explicit} if op in EXTREMES else {}
            want = reduce_oracle(S.indptr, S.indices, S.data, S.shape[1], op, explicit)
            _check(getattr(A, op)(axis=1, **kw), want, op, dtype)
    # random real values: the long-row sums are still within rounding of the fp64 truth
    R = csr_array._from_parts(A.indptr, A.indices, torch.randn(A.nnz, dtype=A.data.dtype, device="cuda"), A.shape)
    np.testing.assert_allclose(_np(R.sum(axis=1)), R.to_scipy_sparse_csr().astype(np.float64).sum(axis=1),
                               rtol=1e-5 if dtype == np.float32 else 1e-12, atol=1e-4)


def test_million_entry_row():
    n = (1 << 20) + 77
    rng = np.random.default_rng(3)
    data = rng.integers(-9, 10, n - 5).astype(np.float64)
    cols = np.sort(rng.choice(n, n - 5, replace=False))
    S = sp.csr_array((data, cols, [0, n - 5]), shape=(1, n))
    A = csr_array(S)
    D = S.toarray()
    for op in ["sum", "count_nonzero"] + EXTREMES:
        _check(getattr(A, op)(axis=1), np.atleast_1d(_scipy(S, op, 1)), op, np.float64)
        _check(np.asarray(getattr(A, op)()), np.asarray(getattr(np, op)(D) if op != "sum" else D.sum()), op,
               np.float64)


def test_one_column_and_empty_shapes():
    A, S = _random(500, 1, lens=np.random.default_rng(4).integers(0, 2, 500), seed=4, dups=False)
    for op in ["sum", "count_nonzero"] + EXTREMES:
        for axis in (None, 0, 1):
            _check(getattr(A, op)(axis=axis), _scipy(S, op, axis), op, np.float64)
    for shape in ((0, 5), (5, 0), (0, 0)):
        E = csr_array(sp.csr_array(shape))
        for axis in (0, 1):
            length = shape[1 - axis]
            assert torch.equal(E.sum(axis=axis), torch.zeros(length, dtype=torch.float64, device="cuda"))
            assert torch.equal(E.count_nonzero(axis=axis), torch.zeros(length, dtype=torch.int64, device="cuda"))
            if shape[axis] > 0:
                assert E.max(axis=axis).shape == (0,) and E.argmin(axis=axis).shape == (0,)
        assert E.sum() == 0 and E.count_nonzero() == 0


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_duplicates_and_unsorted_rows(dtype):
    A, S = _random(700, 40, seed=5, dtype=dtype)
    assert not A.has_sorted_indices
    D = S.toarray()
    before = [(t.data_ptr(), t._version, t.clone()) for t in (A.indptr, A.indices, A.data)]
    for op in ["sum", "count_nonzero"] + EXTREMES:
        for axis in (None, 0, 1):
            _check(getattr(A, op)(axis=axis), np.asarray(_np(getattr(np, op)(D, axis=axis)) if op != "sum"
                                                         else D.sum(axis=axis)), op, dtype)
    for t, (p, v, c) in zip((A.indptr, A.indices, A.data), before):
        assert t.data_ptr() == p and t._version == v and torch.equal(t, c)
    # a second call reuses the canonical form; an in-place edit of data or indices builds a fresh one
    canon = A._cache["canonical"][2]
    A.max(axis=1)
    assert A._cache["canonical"][2] is canon
    A.data.mul_(-1)
    _check(A.max(axis=1), (-D).max(axis=1), "max", dtype)
    _check(A.argmin(axis=0), (-D).argmin(axis=0), "argmin", dtype)
    A.indices.copy_((A.indices + 1) % 40)
    S2 = sp.csr_array((_np(A.data), _np(A.indices), _np(A.indptr)), shape=A.shape)
    D2 = S2.toarray()
    _check(A.argmax(axis=1), D2.argmax(axis=1), "argmax", dtype)
    _check(A.count_nonzero(axis=0), np.count_nonzero(D2, axis=0), "count_nonzero", dtype)
    _check(A.sum(axis=0), D2.sum(axis=0), "sum", dtype)


def test_real_values_with_duplicates():
    A, S = _random(300, 25, seed=6)
    A.data.copy_(torch.randn(A.nnz, dtype=torch.float64, device="cuda"))
    D = A.toarray()
    for axis in (0, 1):
        np.testing.assert_allclose(_np(A.max(axis=axis)), D.max(axis=axis), rtol=1e-14, atol=1e-14)
        np.testing.assert_allclose(_np(A.sum(axis=axis)), D.sum(axis=axis), rtol=1e-12, atol=1e-12)


def test_full_size_laplacian():
    A = gallery.laplacian_5pt(3162, 3162, np.float64)
    S = A.to_scipy_sparse_csr()
    for op in ("sum", "max", "argmax", "count_nonzero"):
        for axis in (0, 1):
            _check(getattr(A, op)(axis=axis), _scipy(S, op, axis), op, np.float64)
    F = A.astype(np.float32)
    np.testing.assert_allclose(_np(F.sum(axis=1)), S.sum(axis=1), rtol=1e-5, atol=1e-2)


def test_full_size_rmat():
    A = gallery.rmat(20)
    S = A.to_scipy_sparse_csr()
    for op in ("sum", "max", "min", "argmax", "argmin", "count_nonzero"):
        for axis in (0, 1):
            _check(getattr(A, op)(axis=axis), _scipy(S, op, axis), op, np.float64)
    _check(A.max(), S.max(), "max", np.float64)
    assert A.argmax() == S.argmax()


def test_repeatable():
    A = gallery.rmat(14)
    A.data.copy_(torch.randn(A.nnz, dtype=torch.float64, device="cuda"))
    for op in ("sum", "max", "argmin", "count_nonzero"):
        for axis in (0, 1):
            assert torch.equal(getattr(A, op)(axis=axis), getattr(A, op)(axis=axis))


def test_graph_capture():
    A = gallery.rmat(12)
    A.data.copy_(torch.randn(A.nnz, dtype=torch.float64, device="cuda"))
    ptr_, idx, dat = A._canonical()
    outs = {op: torch.empty(A.shape[0], dtype=torch.float64 if op in ("sum", "max") else torch.int64, device="cuda")
            for op in ("sum", "max", "argmax")}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for op, o in outs.items():
            _ops.csr_reduce_rows(op, ptr_, idx, dat, A.shape[1], out=o)   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for op, o in outs.items():
            _ops.csr_reduce_rows(op, ptr_, idx, dat, A.shape[1], out=o)
    dat.copy_(torch.randn(dat.shape[0], dtype=torch.float64, device="cuda"))
    for o in outs.values():
        o.fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    for op, o in outs.items():
        assert torch.equal(o, _ops.csr_reduce_rows(op, ptr_, idx, dat, A.shape[1])), op


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_abs_and_power(dtype):
    S = sp.csr_array(scipy.io.mmread(mtx_path("cage4.mtx"))).astype(dtype)
    S.data -= 0.3
    A = csr_array(S)
    np.testing.assert_array_equal(abs(A).toarray(), abs(S).toarray())
    for n, dt in ((2, None), (3, np.float64), (0.5, None), (-1, np.float64)):
        with np.errstate(invalid="ignore"):
            want = S.power(n, dtype=dt).toarray()
        got = A.power(n, dtype=dt)
        assert got.dtype == want.dtype
        np.testing.assert_allclose(got.toarray(), want, rtol=1e-6)


@pytest.mark.parametrize("nodes", [64, 100])
def test_amg_example_with_theta_matches_scipy(nodes):
    lg, state_g, ig, rg, tol = parse(run("-nodes", str(nodes), "-t", "1e-10", "--theta", "0.25"))
    ls, state_s, is_, rs, tol_s = parse(run("-nodes", str(nodes), "-t", "1e-10", "--theta", "0.25",
                                            "--package", "scipy"))
    assert len(lg) == len(ls) > 1
    assert [lvl[:2] for lvl in lg] == [lvl[:2] for lvl in ls]       # same levels, same unknowns per level
    assert state_g == state_s == "Converged" and rg < tol and rs < tol
    assert ig == -(-is_ // 5) * 5 or abs(ig - is_) <= 5
