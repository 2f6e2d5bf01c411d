"""Dense-operand products of `csr_array`, `csc_array` and `dia_array` (legate/sparse_b200/_dense.py) through one table.

The three classes are built from one scipy matrix and multiplied by the same operands: 1-D, (n, 1) and (n, k) for
k in {0, 1, 3, 33}; numpy arrays, CUDA tensors, column-strided and Fortran-ordered arrays and zero-stride `expand`
tensors; real and complex dtypes.  Every `out` kind is tried: none, contiguous and strided numpy arrays, contiguous CUDA
tensors, CUDA tensors whose rows overlap, and a wrong dtype or shape.  The data is integer-valued, so every product is
exact and is compared with scipy bit for bit, together with the result's array kind, shape and dtype."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200.runtime import torch_dtype

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:CSR SpMV creating an implicit copy")]

M, N = 37, 29
# (matrix dtype, operand dtype)
DTYPES = [(np.float32, np.float32), (np.float32, np.float64), (np.float32, np.complex64), (np.float32, np.complex128),
          (np.float64, np.float32), (np.float64, np.float64), (np.float64, np.complex64), (np.float64, np.complex128),
          (np.complex128, np.float64), (np.complex64, np.complex64)]
WIDTHS = [None, 0, 1, 3, 33]   # None: a 1-D operand; k: an (n, k) operand
OPERANDS = ["numpy", "cuda", "strided", "fortran", "expand"]
OUTS = ["none", "numpy", "numpy_strided", "cuda", "cuda_overlapping", "wrong_dtype", "wrong_shape"]


def _scipy_matrix(dtype):
    rng = np.random.default_rng(7)
    S = sp.random_array((M, N), density=0.25, format="csr", rng=rng)
    S.data = rng.integers(-4, 5, S.nnz).astype(np.float64)
    if np.dtype(dtype).kind == "c":
        S = S + 1j * sp.csr_array((rng.integers(-4, 5, S.nnz).astype(np.float64), S.indices, S.indptr), shape=S.shape)
    return S.astype(dtype)


def _matrices(dtype):
    S = _scipy_matrix(dtype)
    return S, {"csr": sparse.csr_array(S), "csc": sparse.csc_array(S.tocsc()), "dia": sparse.dia_array(S)}


def _values(width, dtype, kind):
    """The integer-valued operand's values as a numpy array of `dtype`; `expand` repeats one row (or one value)."""
    rng = np.random.default_rng(11)
    shape = (N,) if width is None else (N, width)
    v = rng.integers(-3, 4, shape).astype(np.float64)
    if np.dtype(dtype).kind == "c":
        v = v + 1j * rng.integers(-3, 4, shape)
    if kind == "expand":
        v = np.broadcast_to(v[:1], shape).copy()
    return v.astype(dtype)


def _operand(v, kind):
    """`v` in the layout `kind`; None when the layout does not apply to v's rank."""
    if kind == "numpy":
        return v.copy()
    if kind == "cuda":
        return torch.from_numpy(v.copy()).cuda()
    if kind == "strided":            # every other element (1-D) or column (2-D) of a wider CUDA tensor
        wide = np.zeros(v.shape[:-1] + (2 * v.shape[-1],), dtype=v.dtype)
        wide[..., ::2] = v
        return torch.from_numpy(wide).cuda()[..., ::2]
    if kind == "fortran":
        return np.asfortranarray(v) if v.ndim == 2 else None
    if kind == "expand":             # zero-stride rows: every row is the same memory
        t = torch.from_numpy(v[:1].copy()).cuda()
        return t.expand(*v.shape)
    raise AssertionError(kind)


def _out(kind, shape, dtype):
    """An `out` of the kind `kind` for a result of `shape` and `dtype`, filled with 99 where it has to be overwritten;
    None when the kind does not apply to the shape."""
    tdt = torch_dtype(dtype)
    if kind == "none":
        return None
    if kind == "numpy":
        return np.full(shape, 99, dtype=dtype)
    if kind == "numpy_strided":
        return np.full(shape[:-1] + (2 * shape[-1],), 99, dtype=dtype)[..., ::2] if shape[-1] else None
    if kind == "cuda":
        return torch.full(shape, 99, dtype=tdt, device="cuda")
    if kind == "cuda_overlapping":   # row i starts where row i - 1 ends: the last column of one row is the next's first
        if len(shape) == 1 or shape[1] < 3:
            return None
        m, k = shape
        return torch.zeros(m * (k - 1) + 1, dtype=tdt, device="cuda").as_strided(shape, (k - 1, 1))
    if kind == "wrong_dtype":
        return np.zeros(shape, dtype=np.float32 if np.dtype(dtype) != np.float32 else np.float64)
    if kind == "wrong_shape":
        return np.zeros((shape[0] + 1,) + shape[1:], dtype=dtype)
    raise AssertionError(kind)


def _np(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _expected_error(fmt, out_kind, matrix_dtype):
    """The exception each class raises for a wrong `out`: csr asserts the shape (as the reference does), csc and dia
    raise ValueError unless A is complex (their complex matrices run the product of `tocsr()`)."""
    if out_kind == "wrong_dtype":
        return ValueError
    if out_kind == "wrong_shape":
        return AssertionError if fmt == "csr" or np.dtype(matrix_dtype).kind == "c" else ValueError
    return None


@pytest.mark.parametrize("width", WIDTHS, ids=lambda w: "1d" if w is None else f"k{w}")
@pytest.mark.parametrize("mdt,xdt", DTYPES, ids=lambda d: np.dtype(d).name)
def test_dense_operand_table(mdt, xdt, width):
    if width == 0 and np.dtype(mdt).kind == "c":
        pytest.skip("the real-expansion product of a complex matrix does not take an (n, 0) operand")
    S, mats = _matrices(mdt)
    common = np.result_type(mdt, xdt)
    rshape = (M,) if width is None else (M, width)
    for op_kind in OPERANDS:
        v = _values(width, xdt, op_kind)
        ref = S.toarray().astype(common) @ v.astype(common)
        for out_kind in OUTS:
            for fmt, A in mats.items():
                x = _operand(v, op_kind)
                out = _out(out_kind, rshape, common)
                if x is None or (out is None and out_kind != "none"):
                    continue
                what = f"{fmt} {op_kind} x, {out_kind} out"
                err = _expected_error(fmt, out_kind, mdt)
                if err is not None:
                    with pytest.raises(err):
                        A.dot(x, out=out)
                    continue
                got = A.dot(x, out=out)
                if out is not None:
                    assert got is out, what
                if out_kind == "cuda_overlapping":
                    # the columns no other row shares hold the product; the shared ones hold one of the two rows'
                    assert np.array_equal(_np(got)[:, 1:-1], ref[:, 1:-1]), what
                    continue
                if out is None:   # x's array kind
                    assert isinstance(got, torch.Tensor if isinstance(x, torch.Tensor) else np.ndarray), what
                    assert not isinstance(got, torch.Tensor) or got.is_cuda, what
                assert tuple(got.shape) == rshape and _np(got).dtype == common, what
                assert np.array_equal(_np(got), ref), what


@pytest.mark.parametrize("fmt", ["csr", "csc", "dia"])
def test_operand_errors(fmt):
    _, mats = _matrices(np.float64)
    A = mats[fmt]
    with pytest.raises(AssertionError if fmt == "csr" else ValueError):
        A.dot(np.ones(N + 1))
    with pytest.raises(AssertionError if fmt == "csr" else ValueError):
        A.dot(torch.ones((N - 1, 3), dtype=torch.float64, device="cuda"))
    with pytest.raises(NotImplementedError):
        A.dot(np.ones((N, 2, 2)))
    with pytest.raises(NotImplementedError, match="SpMV for resolved dtype int64"):
        A.astype(np.int64).dot(np.ones(N, dtype=np.int64))
    with pytest.raises(NotImplementedError, match="SpMM for resolved dtype int64"):
        A.astype(np.int64).dot(torch.ones((N, 3), dtype=torch.int64, device="cuda"))
