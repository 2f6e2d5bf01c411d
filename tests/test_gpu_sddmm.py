"""`csr_array.sddmm` and `_ops.sddmm` (csrc/sddmm.cu) against a float64 host reference.

Each value is held to |out_p - ref_p| <= 2 (k + 2) u |a_p| sum_t |C_it D_tj|, u the unit roundoff of the result dtype:
the kernel sums each dot product in its own fixed order, so it is not bitwise the reference's, but it is bitwise
repeatable and the same for every index width."""
import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200 import _ops, gallery
from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, mtx_path

pytestmark = pytest.mark.gpu

KS = [0, 1, 2, 3, 4, 8, 16, 17, 32, 64, 100, 256, 1000, 4096]


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _check(A_ptr, A_idx, A_val, C, D, got, dtype):
    """got (the result's values) against float64 numpy, within the bound of the module docstring."""
    ptr, idx = _np(A_ptr).astype(np.int64), _np(A_idx).astype(np.int64)
    a, C, D = _np(A_val).astype(np.float64), _np(C).astype(np.float64), _np(D).astype(np.float64)
    got = _np(got)
    assert got.dtype == np.dtype(dtype) and got.shape == a.shape
    rows = np.repeat(np.arange(ptr.size - 1), np.diff(ptr))
    k = C.shape[1]
    ref = np.zeros(a.size)
    mag = np.zeros(a.size)
    for t0 in range(0, k, 256):          # in panels: rows x k gathers of C and D stay small
        Cp, Dp = C[rows, t0:t0 + 256], D[t0:t0 + 256, idx].T
        ref += np.einsum("ij,ij->i", Cp, Dp)
        mag += np.einsum("ij,ij->i", np.abs(Cp), np.abs(Dp))
    ref *= a
    u = np.finfo(dtype).eps / 2
    bound = 2 * (k + 2) * u * np.abs(a) * mag
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    assert np.all(np.abs(got[fin].astype(np.float64) - ref[fin]) <= bound[fin]), \
        float(np.max(np.abs(got[fin] - ref[fin]) - bound[fin]))


def _fixture(name, dtype):
    return sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(dtype)


def _operands(m, n, k, dtype, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((m, k)).astype(dtype), rng.standard_normal((k, n)).astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", MTX_FILES)
def test_fixtures(name, k, dtype):
    S = _fixture(name, dtype)
    A = csr_array(S)
    C, D = _operands(S.shape[0], S.shape[1], k, dtype, seed=k)
    R = A.sddmm(C, D)
    assert isinstance(R, csr_array) and R.shape == A.shape and R.dtype == np.dtype(dtype)
    assert R.indptr is A.indptr and R.indices is A.indices
    assert R.data.is_cuda
    _check(S.indptr, S.indices, S.data, C, D, R.data, dtype)


def test_zero_k_keeps_nan_and_inf():
    S = _fixture("karate.mtx", np.float64)
    S.data[0], S.data[1] = np.nan, np.inf
    R = csr_array(S).sddmm(np.zeros((S.shape[0], 0)), np.zeros((0, S.shape[1])))
    v = _np(R.data)
    assert np.isnan(v[0]) and np.isnan(v[1]) and np.array_equal(v[2:], np.zeros(v.size - 2))


def test_dtype_promotion():
    S = _fixture("GlossGT.mtx", np.float32)
    A = csr_array(S)
    C, D = _operands(S.shape[0], S.shape[1], 16, np.float64, seed=3)
    R = A.sddmm(C, D.astype(np.float32))
    assert R.dtype == np.float64 and R.data.dtype == torch.float64
    _check(S.indptr, S.indices, S.data, C, D.astype(np.float32), R.data, np.float64)
    assert A.dtype == np.float32 and A.data.dtype == torch.float32


@pytest.mark.parametrize("k", [3, 16, 64])
def test_index_widths_are_bitwise_equal(k, monkeypatch):
    S = sp.random_array((3000, 2000), density=0.01, format="csr", rng=np.random.default_rng(7))
    A = csr_array(S)
    assert A.indptr.dtype == torch.int32 and A.indices.dtype == torch.int32
    C, D = _operands(3000, 2000, k, np.float64, seed=k)
    base = _np(A.sddmm(C, D).data)
    _check(S.indptr, S.indices, S.data, C, D, base, np.float64)
    for it in (torch.int32, torch.int64):
        for pt in (torch.int32, torch.int64):
            B = csr_array._from_parts(A.indptr.to(pt), A.indices.to(it), A.data, A.shape)
            assert np.array_equal(_np(B.sddmm(C, D).data).view(np.uint64), base.view(np.uint64)), (it, pt)
    monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    W = csr_array(S)
    assert W.indptr.dtype == torch.int64 and W.indices.dtype == torch.int64
    assert np.array_equal(_np(W.sddmm(C, D).data).view(np.uint64), base.view(np.uint64))


def _structure_cases():
    rng = np.random.default_rng(11)
    out = {}
    # empty rows between short ones
    S = sp.random_array((5000, 300), density=0.02, format="csr", rng=rng)
    keep = np.ones(5000, dtype=bool)
    keep[rng.choice(5000, 2500, replace=False)] = False
    out["empty_rows"] = sp.csr_array(sp.diags_array(keep.astype(float)) @ S)
    out["empty_matrix"] = sp.csr_array((0, 0))
    out["no_entries"] = sp.csr_array((7, 9))
    # one row of 200 000 entries among empty rows: every tile but the ends lies inside it
    n = 200_000
    long_row = sp.csr_array((rng.standard_normal(n), np.arange(n), np.r_[np.zeros(1501, int), np.full(1500, n)]),
                            shape=(3000, n))
    out["long_row"] = long_row
    # rows of ~37 entries: tile boundaries (every 1024 entries) fall inside rows
    out["boundary_inside_row"] = sp.random_array((400, 500), density=37 / 500, format="csr", rng=rng)
    # a few entries spread over 10^5 rows: one tile spans more rows than it can stage
    r = np.sort(rng.choice(100_000, 300, replace=False))
    out["sparse_rows"] = sp.csr_array((rng.standard_normal(300), (r, rng.integers(0, 50, 300))), shape=(100_000, 50))
    return out


@pytest.mark.parametrize("case", ["empty_rows", "empty_matrix", "no_entries", "long_row", "boundary_inside_row",
                                  "sparse_rows"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_tile_boundaries(case, dtype):
    S = _structure_cases()[case].astype(dtype)
    k = 8
    A = csr_array(S)
    C, D = _operands(S.shape[0], S.shape[1], k, dtype, seed=5)
    R = A.sddmm(C, D)
    assert R.nnz == S.nnz and R.shape == S.shape
    _check(S.indptr, S.indices, S.data, C, D, R.data, dtype)


@pytest.mark.parametrize("k", [5, 32])
def test_unsorted_rows_and_repeated_columns(k):
    rng = np.random.default_rng(2)
    m, n = 300, 40
    lens = rng.integers(0, 30, m)
    indptr = np.r_[0, np.cumsum(lens)]
    indices = rng.integers(0, n, indptr[-1]).astype(np.int32)   # unsorted, with repeats
    data = rng.standard_normal(indptr[-1])
    A = csr_array((torch.tensor(data), torch.tensor(indices), torch.tensor(indptr, dtype=torch.int32)), shape=(m, n))
    before = [t.clone() for t in (A.indptr, A.indices, A.data)]
    C, D = _operands(m, n, k, np.float64, seed=9)
    R = A.sddmm(C, D)
    for t, b in zip((A.indptr, A.indices, A.data), before):
        assert torch.equal(t, b)
    assert torch.equal(R.indices, A.indices) and torch.equal(R.indptr, A.indptr)
    _check(indptr, indices, data, C, D, R.data, np.float64)


def test_d_layouts(monkeypatch):
    S = _fixture("Ragusa18.mtx", np.float32)
    A = csr_array(S)
    m, n = S.shape
    k = 32
    seen = []
    real = _ops.sddmm

    def spy(indptr, indices, data, C, Dt, out=None):
        seen.append((C.data_ptr(), Dt.data_ptr()))
        return real(indptr, indices, data, C, Dt, out)

    monkeypatch.setattr(_ops, "sddmm", spy)
    g = torch.Generator().manual_seed(0)
    K = torch.randn(n, k, generator=g).cuda()          # D = K.T: D transposed is K itself
    Cd = torch.randn(m, k, generator=g).cuda()
    R = A.sddmm(Cd, K.T)
    assert seen[-1] == (Cd.data_ptr(), K.data_ptr())
    _check(S.indptr, S.indices, S.data, Cd, K.T, R.data, np.float32)
    Drow = K.T.contiguous()                              # row-major D: one transposed copy
    R2 = A.sddmm(Cd, Drow)
    assert seen[-1][1] not in (Drow.data_ptr(), K.data_ptr())
    assert torch.equal(R2.data, R.data)
    Df = np.asfortranarray(_np(Drow))                    # Fortran-ordered numpy D: D.T is C-ordered
    assert torch.equal(A.sddmm(_np(Cd), Df).data, R.data)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_unaligned_strided_operands(dtype):
    S = _fixture("GlossGT.mtx", dtype)
    A = csr_array(S)
    m, n = S.shape
    k = 13                                              # not a multiple of either pack width
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    g = torch.Generator().manual_seed(1)
    Cbig = torch.randn(m, k + 6, generator=g, dtype=tdt).cuda()
    Dbig = torch.randn(n, k + 4, generator=g, dtype=tdt).cuda()
    C, Dt = Cbig[:, 1:1 + k], Dbig[:, 3:3 + k]          # ld > k, odd element offsets
    assert C.stride(0) == k + 6 and Dt.stride(0) == k + 4
    v = _ops.sddmm(A.indptr, A.indices, A.data, C, Dt)
    _check(S.indptr, S.indices, S.data, C, Dt.T, v, dtype)
    R = A.sddmm(C, Dt.T)
    assert torch.equal(R.data, v)
    # the same at a pack-aligned k, through the 16-byte path, still with ld > k
    k2 = 16
    C2, Dt2 = Cbig[:, :k2], Dbig[:, :k2]
    _check(S.indptr, S.indices, S.data, C2, Dt2.T, _ops.sddmm(A.indptr, A.indices, A.data, C2, Dt2), dtype)


@pytest.mark.parametrize("kind", ["numpy", "torch_cpu", "torch_cuda", "mixed"])
def test_operand_kinds(kind):
    S = _fixture("cage4.mtx", np.float64)
    A = csr_array(S)
    C, D = _operands(S.shape[0], S.shape[1], 8, np.float64, seed=4)
    if kind == "torch_cpu":
        Cx, Dx = torch.from_numpy(C), torch.from_numpy(D)
    elif kind == "torch_cuda":
        Cx, Dx = torch.from_numpy(C).cuda(), torch.from_numpy(D).cuda()
    elif kind == "mixed":
        Cx, Dx = torch.from_numpy(C).cuda(), D
    else:
        Cx, Dx = C, D
    R = A.sddmm(Cx, Dx)
    assert R.data.is_cuda
    _check(S.indptr, S.indices, S.data, C, D, R.data, np.float64)


def test_repeatable():
    S = sp.random_array((2000, 1500), density=0.02, format="csr", rng=np.random.default_rng(3))
    A = csr_array(S)
    C, D = _operands(2000, 1500, 100, np.float64, seed=8)
    v1, v2 = _np(A.sddmm(C, D).data), _np(A.sddmm(C, D).data)
    assert np.array_equal(v1.view(np.uint64), v2.view(np.uint64))


def test_graph_capture():
    S = _fixture("GlossGT.mtx", np.float64)
    A = csr_array(S)
    m, n = S.shape
    k = 16
    g = torch.Generator().manual_seed(2)
    C = torch.randn(m, k, generator=g, dtype=torch.float64).cuda()
    K = torch.randn(n, k, generator=g, dtype=torch.float64).cuda()
    out = torch.empty_like(A.data)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _ops.sddmm(A.indptr, A.indices, A.data, C, K, out)        # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _ops.sddmm(A.indptr, A.indices, A.data, C, K, out)
    C.mul_(-2.0).add_(1.0)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    _check(S.indptr, S.indices, S.data, C, K.T, out, np.float64)


def test_full_size_laplacian_row_sample():
    A = gallery.laplacian_5pt(3162, 3162, np.float64)
    m, n = A.shape
    k = 16
    g = torch.Generator(device="cuda").manual_seed(0)
    C = torch.randn(m, k, generator=g, dtype=torch.float64, device="cuda")
    K = torch.randn(n, k, generator=g, dtype=torch.float64, device="cuda")
    R = A.sddmm(C, K.T)
    rows = np.sort(np.random.default_rng(0).choice(m, 4000, replace=False))
    ptr = _np(A.indptr).astype(np.int64)
    idx, val, got = _np(A.indices), _np(A.data), _np(R.data)
    sel = np.concatenate([np.arange(ptr[r], ptr[r + 1]) for r in rows])
    sub_ptr = np.r_[0, np.cumsum(ptr[rows + 1] - ptr[rows])]
    _check(sub_ptr, idx[sel], val[sel], _np(C)[rows], _np(K).T, got[sel], np.float64)
