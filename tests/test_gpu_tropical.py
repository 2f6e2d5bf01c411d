"""`csr_array.tropical_spmv` and `_ops.tropical_spmv` (csrc/tropical.cu) against the host restatement of the reference
kernel in test_tropical_host.py.  The product is exact integer maxima, so every comparison is bitwise."""
import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200 import _ops, gallery
from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, mtx_path
from test_tropical_host import _values, tropical_oracle

pytestmark = pytest.mark.gpu

FIELDS = [0, 1, 2, 3, 4, 5, 9]


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _ref(A, x):
    return tropical_oracle(_np(A.indptr), _np(A.indices), _np(x))


def _assert_same(got, want):
    got = _np(got)
    assert got.dtype == np.int64 and got.shape == want.shape
    assert np.array_equal(got, want)


def _from_lengths(lens, n, seed):
    """A csr_array with the given row lengths and random (unsorted, repeating) columns in [0, n)."""
    rng = np.random.default_rng(seed)
    indptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    indices = rng.integers(0, n, int(indptr[-1]))
    data = rng.standard_normal(int(indptr[-1]))
    return csr_array(sp.csr_array((data, indices, indptr), shape=(len(lens), n)))


@pytest.mark.parametrize("nf", FIELDS)
@pytest.mark.parametrize("name", MTX_FILES)
def test_fixtures(name, nf):
    S = sp.csr_array(scipy.io.mmread(mtx_path(name)))
    A = csr_array(S)
    x = _values(S.shape[1], nf, seed=nf)
    y = A.tropical_spmv(x)
    assert isinstance(y, np.ndarray)
    _assert_same(y, tropical_oracle(S.indptr, S.indices, x))


@pytest.mark.parametrize("nf", [1, 2, 3, 4, 5])
def test_index_widths(nf):
    lens = np.r_[np.random.default_rng(0).integers(0, 40, 3000), [500, 0, 33]]
    A = _from_lengths(lens, 2000, seed=1)
    x = torch.from_numpy(_values(2000, nf, seed=2, lo=-50, hi=50)).cuda()
    want = _ref(A, x)
    for it in (torch.int32, torch.int64):
        for pt in (torch.int32, torch.int64):
            B = csr_array._from_parts(A.indptr.to(pt), A.indices.to(it), A.data, A.shape)
            _assert_same(B.tropical_spmv(x), want)


@pytest.mark.parametrize("nf", [1, 2, 3, 4, 6])
def test_short_and_long_rows_in_one_warp(nf):
    # every warp of 32 rows mixes lengths around the warp-wide threshold with empty and very long rows
    pattern = [0, 1, 31, 32, 33, 5000, 2, 0, 64, 31, 32, 33, 3, 0, 1, 4096]
    lens = np.array((pattern * 40)[:611])                      # 611 rows: the last warp is partial
    A = _from_lengths(lens, 3001, seed=nf)
    x = _values(3001, nf, seed=nf + 10, lo=-1000, hi=1000)
    _assert_same(A.tropical_spmv(x), _ref(A, x))
    # one long row alone, and a warp of long rows only
    for lens in ([100_000], [40] * 32, [0] * 31 + [70_000]):
        B = _from_lengths(np.array(lens), 777, seed=3)
        _assert_same(B.tropical_spmv(x[:777]), _ref(B, x[:777]))


@pytest.mark.parametrize("shape", [(1, 1), (33, 7), (31, 65), (1000, 3), (5, 100_001)])
@pytest.mark.parametrize("nf", [1, 2, 3])
def test_sizes_off_the_warp(shape, nf):
    m, n = shape
    S = sp.random_array(shape, density=min(1.0, 20 / n), format="csr", rng=np.random.default_rng(m + n))
    A = csr_array(S)
    x = _values(n, nf, seed=m)
    _assert_same(A.tropical_spmv(x), tropical_oracle(S.indptr, S.indices, x))


@pytest.mark.parametrize("nf", [0, 2])
def test_empty_cases(nf):
    for shape in ((0, 0), (0, 5), (5, 0), (40, 9)):
        A = csr_array(sp.csr_array(shape))
        x = np.ones((shape[1], nf), dtype=np.int64)
        y = A.tropical_spmv(x)
        _assert_same(y, np.zeros((shape[0], nf), dtype=np.int64))
        xt = torch.ones((shape[1], nf), dtype=torch.int64, device="cuda")
        out = torch.full((shape[0], nf), 7, dtype=torch.int64, device="cuda")
        assert A.tropical_spmv(xt, out=out) is out
        _assert_same(out, np.zeros((shape[0], nf), dtype=np.int64))


@pytest.mark.parametrize("nf", [1, 2, 3, 4, 5])
def test_strided_unaligned_operands(nf):
    S = sp.csr_array(scipy.io.mmread(mtx_path("GlossGT.mtx")))
    A = csr_array(S)
    m, n = S.shape
    base = torch.from_numpy(_values(n, nf + 3, seed=nf)).cuda()
    want = tropical_oracle(S.indptr, S.indices, _np(base[:, 1:1 + nf]))
    x = base[:, 1:1 + nf]                                      # ld > F, odd element offset: no 16-byte loads
    assert x.stride(0) == nf + 3
    ybig = torch.full((m, nf + 5), -9, dtype=torch.int64, device="cuda")
    out = ybig[:, 3:3 + nf]
    assert A.tropical_spmv(x, out=out) is out
    _assert_same(out, want)
    assert torch.all(ybig[:, :3] == -9) and torch.all(ybig[:, 3 + nf:] == -9)
    # the same through _ops directly, and from an aligned base with an even row stride (the 16-byte path for F = 2)
    _assert_same(_ops.tropical_spmv(A.indptr, A.indices, x), want)
    x2 = torch.zeros((n, nf + 2 + nf % 2), dtype=torch.int64, device="cuda")[:, :nf]
    x2.copy_(x)
    _assert_same(_ops.tropical_spmv(A.indptr, A.indices, x2), want)
    # a transposed (column-strided) x is copied to unit-stride rows
    xt = base[:, 1:1 + nf].T.contiguous().T
    _assert_same(A.tropical_spmv(xt), want)


@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.uint8, np.uint16, np.uint32, np.uint64])
def test_integer_dtypes_are_cast(dtype):
    S = sp.csr_array(scipy.io.mmread(mtx_path("Ragusa18.mtx")))
    A = csr_array(S)
    info = np.iinfo(dtype)
    x = np.random.default_rng(4).integers(max(info.min, -100), min(info.max, 100), (S.shape[1], 3)).astype(dtype)
    want = tropical_oracle(S.indptr, S.indices, x.astype(np.int64))
    _assert_same(A.tropical_spmv(x), want)
    if dtype in (np.int8, np.int16, np.int32, np.uint8):
        _assert_same(A.tropical_spmv(torch.from_numpy(x).cuda()), want)


@pytest.mark.parametrize("kind", ["numpy", "torch_cpu", "torch_cuda", "list"])
@pytest.mark.parametrize("out_kind", [None, "numpy", "torch_cpu", "torch_cuda"])
def test_operand_kinds(kind, out_kind, monkeypatch):
    S = sp.csr_array(scipy.io.mmread(mtx_path("cage4.mtx")))
    A = csr_array(S)
    m, n = S.shape
    x = _values(n, 3, seed=5)
    want = tropical_oracle(S.indptr, S.indices, x)
    xx = {"numpy": x, "torch_cpu": torch.from_numpy(x), "torch_cuda": torch.from_numpy(x).cuda(),
          "list": x.tolist()}[kind]
    out = {None: None, "numpy": np.zeros((m, 3), dtype=np.int64), "torch_cpu": torch.zeros((m, 3), dtype=torch.int64),
           "torch_cuda": torch.zeros((m, 3), dtype=torch.int64, device="cuda")}[out_kind]
    seen = []
    real = _ops.tropical_spmv

    def spy(indptr, indices, xd, y=None):
        seen.append((xd.data_ptr(), None if y is None else y.data_ptr()))
        return real(indptr, indices, xd, y)

    monkeypatch.setattr(_ops, "tropical_spmv", spy)
    y = A.tropical_spmv(xx, out=out)
    if out is not None:
        assert y is out
    elif isinstance(xx, torch.Tensor) and xx.is_cuda:
        assert isinstance(y, torch.Tensor) and y.is_cuda
    else:
        assert isinstance(y, np.ndarray)
    _assert_same(y, want)
    if kind == "torch_cuda":
        assert seen[-1][0] == xx.data_ptr()                    # int64 CUDA x with unit-stride rows: no copy
    if out_kind == "torch_cuda":
        assert seen[-1][1] == out.data_ptr()                   # written in place


def test_out_overlapping_x_is_refused():
    S = sp.csr_array(scipy.io.mmread(mtx_path("karate.mtx")))
    A = csr_array(S)
    buf = torch.zeros((S.shape[0], 4), dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        A.tropical_spmv(buf[:, :2], out=buf[:, 2:])
    with pytest.raises(ValueError):
        A.tropical_spmv(buf, out=buf)


def test_repeatable():
    A = gallery.rmat(14)
    x = torch.from_numpy(_values(A.shape[1], 3, seed=6, lo=0, hi=5)).cuda()
    y1, y2 = A.tropical_spmv(x), A.tropical_spmv(x)
    assert torch.equal(y1, y2)
    _assert_same(y1, _ref(A, x))


def test_graph_capture():
    A = gallery.rmat(12)
    n = A.shape[1]
    x = torch.from_numpy(_values(n, 3, seed=7)).cuda()
    y = torch.empty((A.shape[0], 3), dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _ops.tropical_spmv(A.indptr, A.indices, x, y)           # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _ops.tropical_spmv(A.indptr, A.indices, x, y)
    x.copy_(torch.from_numpy(_values(n, 3, seed=8)))
    y.fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    _assert_same(y, _ref(A, x))


@pytest.mark.parametrize("nf", [1, 3])
def test_full_size_laplacian_rows(nf):
    # the host restatement of all 10M rows takes about a minute; it checks the first and last 100 000 rows and a
    # seeded sample between them
    A = gallery.laplacian_5pt(3162, 3162, np.float64)
    m, n = A.shape
    x = torch.randint(-2**40, 2**40, (n, nf), dtype=torch.int64, device="cuda")
    y = _np(A.tropical_spmv(x))
    rows = np.unique(np.r_[np.arange(100_000), np.arange(m - 100_000, m),
                           np.random.default_rng(0).choice(m, 20_000, replace=False)])
    ptr = _np(A.indptr).astype(np.int64)
    sel = np.concatenate([np.arange(ptr[r], ptr[r + 1]) for r in rows])
    sub_ptr = np.r_[0, np.cumsum(ptr[rows + 1] - ptr[rows])]
    _assert_same(y[rows], tropical_oracle(sub_ptr, _np(A.indices)[sel], _np(x)))


def test_full_size_rmat():
    A = gallery.rmat(20)
    x = torch.randint(-3, 4, (A.shape[1], 3), dtype=torch.int64, device="cuda")
    _assert_same(A.tropical_spmv(x), _ref(A, x))
