"""Everything csr_array derives from indptr / indices / data (SpMV plan, promoted copy, transpose, real expansion of
complex values, column blocks) follows every kind of edit of the three arrays: in-place edits of any of them and
assignment of a new index array.  The GPU cases compare each product against scipy on the edited arrays; the host
cases check the caches and the index-width rule without a device."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import gallery, linalg

M, N = 120, 150
ROW = 5          # the row every edit touches

EDITS = ["indices_inplace", "indptr_inplace", "indices_assigned", "data_inplace"]


@pytest.fixture
def host_only(monkeypatch):
    """Arrays stay on the host, also where a GPU is visible."""
    from legate.sparse_b200.runtime import Runtime

    monkeypatch.setattr(Runtime, "has_cuda", property(lambda self: False))


def _random_csr(dtype, seed=11):
    rng = np.random.default_rng(seed)
    S = sp.random(M, N, density=0.08, random_state=rng, format="csr")
    S.sort_indices()
    vals = rng.standard_normal(S.nnz)
    if np.dtype(dtype).kind == "c":
        vals = vals + 1j * rng.standard_normal(S.nnz)
    ip, ix = S.indptr.astype(np.int64), S.indices.astype(np.int64)
    assert ip[ROW + 1] > ip[ROW] and ip[ROW + 1] - ip[ROW] < N
    return ip, ix, vals.astype(dtype)


def _edit(edit, A, ip, ix, dv):
    """Apply `edit` to A's arrays and the same change to the host copies (ip, ix, dv)."""
    lo, hi = ip[ROW], ip[ROW + 1]
    if edit == "indices_inplace":
        col = next(c for c in range(N) if c not in ix[lo:hi])
        A.indices[lo] = col
        ix[lo] = col
    elif edit == "indptr_inplace":
        A.indptr[ROW + 1] -= 1              # the last entry of ROW becomes the first of ROW + 1
        ip[ROW + 1] -= 1
    elif edit == "indices_assigned":
        ix[:] = (ix + 1) % N
        A.indices = torch.from_numpy(ix.astype(np.int32)).to(A.indices.device)
    elif edit == "data_inplace":
        A.data[lo] = 7
        dv[lo] = 7
    else:
        raise AssertionError(edit)


def _products(product, A, rng):
    """(what A computes, what scipy computes from the host arrays, tolerance) for one derivative."""
    if product == "plain":
        x = rng.random(N).astype(np.float32)
        return (lambda: (A @ torch.from_numpy(x).cuda()).cpu().numpy(), lambda S: S @ x.astype(np.float64),
                dict(rtol=1e-4, atol=1e-4))
    if product == "promoted":                       # float32 A, float64 x: through A's promoted copy
        x = rng.random(N)
        return lambda: A @ x, lambda S: S.astype(np.float64) @ x, dict(rtol=1e-12, atol=1e-12)
    if product == "transpose":                      # X @ A: through A's transpose
        X = rng.random((4, M)).astype(np.float32)
        return lambda: X @ A, lambda S: X.astype(np.float64) @ S.toarray(), dict(rtol=1e-4, atol=1e-4)
    if product == "complex":                        # complex A: through A's real expansion
        z = rng.random(N) + 1j * rng.random(N)
        return lambda: A @ z, lambda S: S @ z, dict(rtol=1e-12, atol=1e-12)
    if product == "column_split":                   # through A's column blocks
        x = rng.random(N).astype(np.float32)
        return (lambda: A.dot(torch.from_numpy(x).cuda(), spmv_domain_part=True).cpu().numpy(),
                lambda S: S @ x.astype(np.float64), dict(rtol=1e-4, atol=1e-4))
    raise AssertionError(product)


@pytest.mark.gpu
@pytest.mark.parametrize("edit", EDITS)
@pytest.mark.parametrize("product", ["plain", "promoted", "transpose", "complex", "column_split"])
def test_derived_products_follow_edits(product, edit):
    ip, ix, dv = _random_csr(np.complex128 if product == "complex" else np.float32)
    A = sparse.csr_array((dv, ix, ip), shape=(M, N))
    got, ref, tol = _products(product, A, np.random.default_rng(12))
    np.testing.assert_allclose(got(), ref(sp.csr_array((dv, ix, ip), shape=(M, N))), **tol)   # builds the derivative
    _edit(edit, A, ip, ix, dv)
    np.testing.assert_allclose(got(), ref(sp.csr_array((dv, ix, ip), shape=(M, N))), **tol)


def _cg_with_midrun_index_edit():
    A = gallery.laplacian_5pt(200, 150, np.float64)
    assert A._get_plan().templated or A._get_plan().packed
    k = int(A.indptr[A.shape[0] // 2])          # first entry of an interior row: column i - n1; i - n1 + 1 is free
    calls = []

    def callback(x):
        calls.append(1)
        if len(calls) == 5:
            A.indices[k] += 1

    b = torch.ones(A.shape[0], dtype=torch.float64, device="cuda")
    x, iters = linalg.cg(A, b, tol=0, maxiter=20, callback=callback)
    assert iters == 20
    return x


@pytest.mark.gpu
def test_cg_graphs_follow_an_index_edit_from_the_callback(monkeypatch):
    """The captured CG iterations replay the plan of the structure at capture: an in-place edit of A.indices from the
    callback must send the loop back to eager launches, exactly like a run without graphs."""
    monkeypatch.setenv("B2S_CG_GRAPH", "1")
    x_graphs = _cg_with_midrun_index_edit()
    monkeypatch.setenv("B2S_CG_GRAPH", "0")
    x_eager = _cg_with_midrun_index_edit()
    scale = float(x_eager.abs().max())
    torch.testing.assert_close(x_graphs, x_eager, rtol=1e-12, atol=1e-12 * scale)


# -- host only ------------------------------------------------------------------------------------------------------


def _real_expansion_dense(S):
    D = S.toarray()
    E = np.zeros((2 * D.shape[0], 2 * D.shape[1]))
    E[0::2, 0::2], E[0::2, 1::2], E[1::2, 0::2], E[1::2, 1::2] = D.real, -D.imag, D.imag, D.real
    return E


@pytest.mark.parametrize("edit", EDITS)
def test_real_expansion_follows_edits(host_only, edit):
    ip, ix, dv = _random_csr(np.complex128)
    A = sparse.csr_array((dv, ix, ip), shape=(M, N))
    E0 = A._real_expansion(np.float64)
    assert A._real_expansion(np.float64) is E0
    _edit(edit, A, ip, ix, dv)
    E1 = A._real_expansion(np.float64)
    assert E1 is not E0
    np.testing.assert_array_equal(E1.todense(), _real_expansion_dense(sp.csr_array((dv, ix, ip), shape=(M, N))))


def test_promoted_copy_follows_index_assignment(host_only):
    ip, ix, dv = _random_csr(np.float32)
    B = sparse.csr_array((dv, ix, ip), shape=(M, N))
    f64 = np.dtype(np.float64)
    P0 = B._promoted(f64)
    assert B._promoted(f64) is P0
    _edit("indices_assigned", B, ip, ix, dv)
    P1 = B._promoted(f64)
    assert P1.indices is B.indices
    np.testing.assert_array_equal(P1.todense(), sp.csr_array((dv.astype(np.float64), ix, ip), shape=(M, N)).toarray())


@pytest.mark.parametrize("wide", [False, True])
def test_index_width_rule(host_only, monkeypatch, wide):
    """int32 row pointers below 2^31 - 1 entries (the bound every kernel entry point checks), int32 indices up to
    2^31 - 1; B2S_INDEX_WIDTH=64 forces both wide, for matrices from the gallery too."""
    from legate.sparse_b200.csr import _index_dtype, _indptr_dtype

    if wide:
        monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    else:
        monkeypatch.delenv("B2S_INDEX_WIDTH", raising=False)
    narrow = torch.int64 if wide else torch.int32
    assert _indptr_dtype(2**31 - 2) == narrow and _indptr_dtype(2**31 - 1) == torch.int64
    assert _index_dtype(2**31 - 1) == narrow and _index_dtype(2**31) == torch.int64
    assert gallery.laplacian_5pt(4, 4, np.float64).indptr.dtype == narrow
    assert sparse.csr_array(sp.eye(4, format="csr")).indptr.dtype == narrow
