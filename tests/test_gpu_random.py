"""`random`, `rand` and `random_array` on the device (csrc/random.cu), against the numpy restatement of
tests/test_random_host.py: the same seed gives the same indptr, indices and data bytes.  Also: several sampling rounds,
one matrix in every format, row, column and subset statistics, custom value samplers, a 10^7-entry sample, and the
reference's way of building a CG test matrix."""
import functools
import math

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.stats as stats
import torch

from test_random_host import SUBSET_CHI2_MAX, oracle_structure, oracle_values, subset_chi2

import legate.sparse_b200 as sparse
from legate.sparse_b200 import _ops
from legate.sparse_b200.csr import _index_dtype, _indptr_dtype

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64, np.complex64, np.complex128]


def device_seed(s):
    """the 64-bit seed `rng=s` hands to the device: one draw of default_rng(s)"""
    return int(np.random.default_rng(s).integers(0, 2**64, dtype=np.uint64))


@functools.lru_cache(maxsize=None)
def structure(shape, density, s):
    return oracle_structure(shape, density, device_seed(s))


def oracle(shape, density, s, dtype):
    """(indptr, indices, data, rounds) of the restatement for rng=s"""
    ptr, idx, rounds = structure(shape, density, s)
    return ptr, idx, oracle_values(idx.size, device_seed(s), dtype), rounds


def assert_bits(A, shape, density, s, dtype):
    ptr, idx, data, _ = oracle(shape, density, s, np.dtype(dtype))
    assert A.shape == shape and A.dtype == np.dtype(dtype)
    assert A.indptr.dtype == _indptr_dtype(idx.size) and A.indices.dtype == _index_dtype(max(shape))
    assert np.array_equal(A.indptr.cpu().numpy(), ptr)
    assert np.array_equal(A.indices.cpu().numpy(), idx)
    assert A.data.cpu().numpy().tobytes() == data.tobytes()


def _densities(shape):
    mn = math.prod(shape)
    return [0.0, 1e-4, 0.01, 0.3, 0.5, 0.9, 1.0] + ([0.5 + 1 / mn] if mn > 2 else [])


@pytest.mark.parametrize("s", [0, 12345])
@pytest.mark.parametrize("shape", [(0, 5), (5, 0), (1, 1), (1, 1000), (1000, 1), (300, 700), (2000, 2000)])
def test_bit_identical_to_restatement(shape, s):
    for density in _densities(shape):
        for dt in DTYPES:
            assert_bits(sparse.random_array(shape, density=density, format="csr", dtype=dt, rng=s), shape, density, s,
                        dt)


@pytest.mark.parametrize("shape", [(3, 2049), (40, 5000), (2, 9001)])
def test_bit_identical_on_long_complement_rows(shape):
    """rows of more than 2048 columns on the complement path: one CTA per row, eight warps on column spans that end
    inside a 32-column chunk"""
    mn = math.prod(shape)
    for density in (0.5 + 1 / mn, 0.9, 1.0):
        for dt in (np.float32, np.complex128):
            assert_bits(sparse.random_array(shape, density=density, format="csr", dtype=dt, rng=7), shape, density, 7,
                        dt)


def test_bit_identical_with_64_bit_indices(monkeypatch):
    monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    for shape, density in (((300, 700), 0.02), ((300, 700), 0.8), ((40, 5000), 0.9), ((2, 9001), 0.5 + 1 / 18002)):
        A = sparse.random(*shape, density, format="csr", dtype=np.float64, rng=4)
        assert A.indptr.dtype == A.indices.dtype == torch.int64
        assert_bits(A, shape, density, 4, np.float64)


def test_bit_identical_with_more_than_2_31_columns():
    shape = (3, 2**31 + 10)
    A = sparse.random(*shape, 5e-9, format="csr", dtype=np.float32, rng=6)
    assert A.nnz == round(5e-9 * shape[0] * shape[1]) and A.indices.dtype == torch.int64
    assert_bits(A, shape, 5e-9, 6, np.float32)


def test_several_rounds():
    k = 64 * 64 // 2
    ptr, idx, data, rounds = _ops.random_csr((64, 64), k, device_seed(1), torch.int32, torch.int32, np.float64)
    want = oracle((64, 64), 0.5, 1, np.dtype(np.float64))
    assert rounds >= 2 and rounds == want[3]
    assert np.array_equal(idx.cpu().numpy(), want[1]) and data.cpu().numpy().tobytes() == want[2].tobytes()


@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
@pytest.mark.parametrize("density", [0.05, 0.7])
def test_every_format_is_one_matrix(dtype, density):
    mats = {f: sparse.random(120, 90, density, format=f, dtype=dtype, rng=3) for f in ("coo", "csr", "csc", "dia")}
    dense = mats["csr"].toarray()
    assert np.count_nonzero(dense) == round(density * 120 * 90)
    for f, A in mats.items():
        assert A.format == f and np.array_equal(A.toarray(), dense), f
    C = mats["csc"]
    want = sp.csc_array(dense)   # canonical: each column's rows ascending
    assert np.array_equal(C.indptr.cpu().numpy(), want.indptr) and np.array_equal(C.indices.cpu().numpy(), want.indices)
    assert np.array_equal(C.data.cpu().numpy(), want.data)
    coo = mats["coo"]
    order = np.lexsort((coo.col, coo.row))
    assert np.array_equal(order, np.arange(coo.nnz))   # row-major canonical order


def count_chi2(counts, k, N):
    """chi-square of per-row (or per-column) counts of a uniform k-subset of N positions, with the multivariate
    hypergeometric's finite-population factor (N - 1) / (N - k): about chi2(len(counts) - 1)"""
    e = k / counts.size
    return float(((counts - e) ** 2).sum() / e * (N - 1) / (N - k))


def assert_counts_uniform(A):
    m, n = A.shape
    csr = A.to_scipy_sparse_csr()
    for counts in (np.diff(csr.indptr), np.bincount(csr.indices, minlength=n)):
        p = stats.chi2.sf(count_chi2(counts, csr.nnz, m * n), counts.size - 1)
        assert 1e-4 < p < 1 - 1e-4, p


def test_row_and_column_counts():
    assert_counts_uniform(sparse.random(2000, 2000, 0.01, format="csr", rng=10))
    assert_counts_uniform(sparse.random(300, 300, 0.8, format="csr", rng=11))   # the complement path


def test_uniform_over_subsets():
    def sample(seed):
        A = sparse.random_array((2, 3), density=1 / 3, format="csr", rng=seed)
        return np.repeat(np.arange(2), np.diff(A.indptr.cpu().numpy())) * 3 + A.indices.cpu().numpy()

    assert subset_chi2(sample) < SUBSET_CHI2_MAX


def test_custom_sampler():
    calls = []

    def sampler(size):
        calls.append(size)
        return np.arange(size, dtype=float)

    A = sparse.random_array((400, 300), density=0.6, format="csr", dtype=np.float32, rng=2, data_sampler=sampler)
    k = round(0.6 * 400 * 300)
    assert calls == [k] and A.dtype == np.float32
    assert np.array_equal(A.data.cpu().numpy(), np.arange(k, dtype=np.float32))
    assert np.array_equal(A.indices.cpu().numpy(), oracle((400, 300), 0.6, 2, np.dtype(np.float32))[1])
    B = sparse.random(50, 40, 0.1, format="csc", dtype=np.complex64, rng=2, data_rvs=lambda n: np.arange(n) * 1j)
    dense = B.toarray()
    assert np.array_equal(np.sort(dense[dense != 0].imag), np.arange(1, 200, dtype=np.float32))


def _sorted_unique_rows(A):
    ptr = A.indptr.to(torch.int64)
    idx = A.indices.to(torch.int64)
    rows = torch.repeat_interleave(torch.arange(A.shape[0], device=idx.device), ptr[1:] - ptr[:-1])
    same_row = rows[1:] == rows[:-1]
    return bool(((idx[1:] > idx[:-1]) | ~same_row).all())


def test_large_sample():
    m = n = 10**6
    A = sparse.random(m, n, 1e-5, format="csr", dtype=np.float32, rng=99)
    B = sparse.random(m, n, 1e-5, format="csr", dtype=np.float32, rng=99)
    assert A.nnz == 10**7 and int(A.indptr[-1]) == 10**7 and _sorted_unique_rows(A)
    assert int(A.indices.min()) >= 0 and int(A.indices.max()) < n
    assert all(torch.equal(a, b) for a, b in ((A.indptr, B.indptr), (A.indices, B.indices), (A.data, B.data)))


def test_drop_in_cg_matrix():
    """sparse.random builds the SPD test matrix of the reference's CG tests (0.5 (S + S^T) + N I), which cg solves"""
    import sparse as alias

    N = 1000
    S = alias.random(N, N, 0.01, format="csr", random_state=1)
    assert S.nnz == 10**4
    Sd = S.toarray()
    A = alias.csr_array(0.5 * (Sd + Sd.T) + N * np.eye(N))
    b = np.random.default_rng(0).random(N)
    x, iters = alias.linalg.cg(A, b, tol=1e-10)
    assert np.linalg.norm(A.toarray() @ x - b) <= 1e-8 * np.linalg.norm(b)
