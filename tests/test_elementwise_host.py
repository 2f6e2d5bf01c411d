"""Host-side checks of the elementwise operations of `csr_array`.

`row_merge` restates, on the host, the row merge the GPU kernels run (csrc/elementwise.cu; the reference's add() and
mult(), sparse/csr.py:972-1099): per row, repeated columns of one operand summed in stored order, then the union (add,
subtract) or intersection (multiply) of the column keys, no entry dropped for being zero.  It is pinned to scipy on
the MatrixMarket fixtures and on seeded random matrices.  The argument checks and `eliminate_zeros` /
`has_sorted_indices` need no device."""
import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, mtx_path


def row_merge(A, B, op):
    """C = A op B (op "add" / "sub" / "mul") for scipy CSR operands with non-decreasing rows; symbolic structure."""
    m, _ = A.shape
    dt = np.result_type(A.dtype, B.dtype)
    ptr, idx, val = [0], [], []
    for r in range(m):
        rows = []
        for S in (A, B):
            keys, sums = [], []
            for p in range(S.indptr[r], S.indptr[r + 1]):
                c, v = int(S.indices[p]), dt.type(S.data[p])
                if keys and keys[-1] == c:
                    sums[-1] = dt.type(sums[-1] + v)
                else:
                    keys.append(c)
                    sums.append(v)
            rows.append(dict(zip(keys, sums)))
        a, b = rows
        keys = sorted(set(a) & set(b)) if op == "mul" else sorted(set(a) | set(b))
        for k in keys:
            if op == "mul":
                v = a[k] * b[k]
            elif k in a and k in b:
                v = a[k] + b[k] if op == "add" else a[k] - b[k]
            elif k in a:
                v = a[k]
            else:
                v = b[k] if op == "add" else -b[k]
            idx.append(k)
            val.append(v)
        ptr.append(len(idx))
    return np.array(ptr), np.array(idx, dtype=np.int64), np.array(val, dtype=dt)


def _pruned(ptr, idx, val, shape):
    C = sp.csr_array((val, idx, ptr), shape=shape)
    C.eliminate_zeros()
    return C


def _scipy(A, B, op):
    return sp.csr_array(A + B if op == "add" else A - B if op == "sub" else A.multiply(B))


@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("op", ["add", "sub", "mul"])
def test_row_merge_matches_scipy_on_fixtures(name, op):
    S = sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(np.float64)
    others = [S, sp.random_array(S.shape, density=0.2, format="csr", rng=np.random.default_rng(1))]
    if S.shape[0] == S.shape[1]:
        others.append(sp.csr_array(S.T))
    for B in others:
        B = sp.csr_array(B)
        B.sort_indices()
        ptr, idx, val = row_merge(S, B, op)
        P = _scipy(abs(S).astype(bool).astype(np.float64), abs(B).astype(bool).astype(np.float64),
                   "mul" if op == "mul" else "add")
        P.sort_indices()
        assert np.array_equal(ptr, P.indptr) and np.array_equal(idx, P.indices)
        C, R = _pruned(ptr, idx, val, S.shape), _scipy(S, B, op)
        R.sort_indices()
        assert np.array_equal(C.indptr, R.indptr) and np.array_equal(C.indices, R.indices)
        assert np.array_equal(C.data, R.data)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("op", ["add", "sub", "mul"])
def test_row_merge_matches_scipy_random(seed, op):
    rng = np.random.default_rng(seed)
    m, n = int(rng.integers(1, 60)), int(rng.integers(1, 60))
    A = sp.random_array((m, n), density=0.2, format="csr", rng=rng).astype(np.float32)
    B = sp.random_array((m, n), density=0.3, format="csr", rng=rng)
    ptr, idx, val = row_merge(A, B, op)
    C, R = _pruned(ptr, idx, val, (m, n)), _scipy(A, B, op)
    R.sort_indices()
    assert val.dtype == np.float64
    assert np.array_equal(C.indptr, R.indptr) and np.array_equal(C.indices, R.indices)
    assert np.array_equal(C.data, R.data)


def test_row_merge_sums_repeated_columns():
    # row 0 of A holds column 2 twice; the structure keeps A's explicit zero at column 0 in A - B
    A = sp.csr_array((np.array([1.0, 2.0, 3.0]), np.array([0, 2, 2]), np.array([0, 3])), shape=(1, 4))
    B = sp.csr_array((np.array([1.0, 4.0]), np.array([0, 3]), np.array([0, 2])), shape=(1, 4))
    ptr, idx, val = row_merge(A, B, "sub")
    assert list(idx) == [0, 2, 3] and list(val) == [0.0, 5.0, -4.0]
    ptr, idx, val = row_merge(A, B, "mul")
    assert list(idx) == [0] and list(val) == [1.0]


def _host_csr(S):
    return csr_array(sp.csr_array(S))


def test_argument_errors_need_no_device():
    A = _host_csr(sp.random_array((5, 6), density=0.5, format="csr", rng=np.random.default_rng(0)))
    B = _host_csr(sp.random_array((6, 5), density=0.5, format="csr", rng=np.random.default_rng(1)))
    for f in (lambda: A + B, lambda: A - B, lambda: A.multiply(B), lambda: A.multiply(np.ones((2, 2)))):
        with pytest.raises(ValueError):
            f()
    Z = sp.random_array((5, 6), density=0.5, format="csr", dtype=np.complex128, rng=np.random.default_rng(2))
    for f in (lambda: A + Z, lambda: A - Z, lambda: A.multiply(Z)):
        with pytest.raises(NotImplementedError):
            f()
    for f in (lambda: A + 1.0, lambda: 2 - A):
        with pytest.raises(NotImplementedError):
            f()


def test_eliminate_zeros_and_sorted_flag_on_host():
    data = torch.tensor([0.0, 1.0, -0.0, 2.0, 0.0, float("nan")], dtype=torch.float64)
    indices = torch.tensor([3, 1, 0, 2, 5, 4], dtype=torch.int32)
    indptr = torch.tensor([0, 2, 2, 6], dtype=torch.int32)
    A = csr_array((data, indices, indptr), shape=(3, 6))
    assert not A.has_sorted_indices                   # row 0 is 3, 1
    A.eliminate_zeros()
    assert A.indptr.tolist() == [0, 1, 1, 3] and A.indices.tolist() == [1, 2, 4]
    assert A.has_sorted_indices and np.isnan(A.data[2].item())
    B = csr_array((torch.tensor([1.0, 2.0]), torch.tensor([4, 0], dtype=torch.int32),
                   torch.tensor([0, 1, 2], dtype=torch.int32)), shape=(2, 5))
    assert B.has_sorted_indices                       # the decrease is across rows
