"""Host-side checks of `dia_array` (legate/sparse_b200/dia.py), `diags` / `spdiags` / `eye(format="dia")`, and of
the DIA C entry points (csrc/dia.cu).

`dia_spmv` restates the product in numpy (row r of diagonal d adds data[d, r + k] * x[r + k] into y[r], for the
in-band positions) and is pinned to scipy.  Construction and conversions run on the host, as they do without a GPU, and
the entry points' argument checks are called through ctypes in a subprocess that sees no CUDA device."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200.dia import dia_array

from conftest import MTX_FILES, ROOT, mtx_path


def dia_spmv(data, offsets, shape, x):
    """y = A x for the DIA matrix (data, offsets) of `shape`, diagonals summed in stored order."""
    m, n = shape
    data = np.asarray(data)
    x = np.asarray(x)
    dt = np.result_type(data.dtype, x.dtype)
    lim = min(n, data.shape[1])
    y = np.zeros((m,) + x.shape[1:], dtype=dt)
    for d, k in enumerate(np.asarray(offsets).tolist()):
        j = np.arange(max(k, 0), max(min(m + k, lim), max(k, 0)))
        y[j - k] += (data[d, j].astype(dt) * x[j].astype(dt).T).T
    return y


def _dryrun_spmv_dia(offsets, data, x, y, shape):
    """`_ops.spmv_dia` for the CPU dry run of the GPU test file."""
    y.copy_(torch.from_numpy(dia_spmv(data.numpy(), offsets.numpy(), shape, x.numpy())))
    return y


def _dryrun_spmm_dia(offsets, data, X, Y, shape):
    """`_ops.spmm_dia` for the CPU dry run of the GPU test file."""
    Y.copy_(torch.from_numpy(dia_spmv(data.numpy(), offsets.numpy(), shape, X.contiguous().numpy())))
    return Y


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _random_dia(rng, shape, offsets, L, dtype=np.float64):
    return sp.dia_array((rng.standard_normal((len(offsets), L)).astype(dtype), np.asarray(offsets)), shape=shape)


CASES = [((7, 7), [0, 1, -1], 7), ((5, 9), [-2, 0, 3, 8], 9), ((9, 5), [4, -8, 0], 5), ((6, 6), [2, -1, 0], 4),
         ((6, 6), [1, 0, -3], 10), ((4, 4), [0, 7, -9], 4), ((3, 5), [], 5), ((0, 4), [0, 1], 4)]


@pytest.mark.parametrize("shape,offsets,L", CASES)
def test_restatement_matches_scipy(shape, offsets, L):
    rng = np.random.default_rng(0)
    S = _random_dia(rng, shape, offsets, L)
    x = rng.standard_normal(shape[1])
    np.testing.assert_allclose(dia_spmv(S.data, S.offsets, shape, x), S @ x, rtol=1e-13, atol=1e-13)
    X = rng.standard_normal((shape[1], 3))
    np.testing.assert_allclose(dia_spmv(S.data, S.offsets, shape, X), S @ X, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("shape,offsets,L", CASES)
def test_attributes_and_conversions_match_scipy(shape, offsets, L):
    rng = np.random.default_rng(1)
    S = _random_dia(rng, shape, offsets, L)
    S.data[S.data < -1.0] = 0.0   # stored zeros: counted by nnz, not by count_nonzero, dropped by the conversions
    A = dia_array((S.data, S.offsets), shape=shape)
    assert A.shape == S.shape and A.dtype == S.dtype and A.ndim == 2 and A.format == "dia"
    assert A.nnz == S.nnz
    assert A.count_nonzero() == S.count_nonzero()
    for k in range(-shape[0] - 1, shape[1] + 2):
        np.testing.assert_array_equal(_np(A.diagonal(k)), S.diagonal(k))
    dense = S.toarray()
    np.testing.assert_array_equal(A.todense(), dense)
    np.testing.assert_array_equal(A.toarray(), dense)
    np.testing.assert_array_equal(A.T.todense(), dense.T)
    assert A.T.shape == S.T.shape
    np.testing.assert_array_equal(A.tocoo().todense(), S.tocoo().toarray())
    C = A.tocsr()
    R = S.tocsr()
    R.sort_indices()
    np.testing.assert_array_equal(_np(C.indptr), R.indptr)
    np.testing.assert_array_equal(_np(C.indices), R.indices)
    np.testing.assert_array_equal(_np(C.data), R.data)
    np.testing.assert_array_equal(A.tocsc().todense(), dense)
    np.testing.assert_array_equal(A.asformat("csc").todense(), dense)
    assert A.todia() is A and A.asformat("dia") is A
    np.testing.assert_array_equal(A.to_scipy_sparse_dia().toarray(), dense)


def test_transpose_matches_scipy_in_band():
    rng = np.random.default_rng(2)
    for shape, offsets, L in CASES:
        S = _random_dia(rng, shape, offsets, L)
        T, R = dia_array(S).T, S.T
        np.testing.assert_array_equal(_np(T.offsets), R.offsets)
        np.testing.assert_array_equal(T.todense(), S.toarray().T)
        assert T.nnz == R.nnz
        if L <= max(shape):   # scipy 1.18.1 re-aligns a longer data array with a wrap-around index
            np.testing.assert_array_equal(T.todense(), R.toarray())


def test_construction_from_every_input():
    rng = np.random.default_rng(3)
    S = _random_dia(rng, (6, 8), [-1, 0, 2], 8)
    dense = S.toarray()
    forms = [dia_array((S.data, S.offsets), shape=S.shape), dia_array((torch.from_numpy(S.data), S.offsets),
                                                                      shape=S.shape),
             dia_array(S), dia_array(sp.csr_array(S)), dia_array(dense), dia_array(torch.from_numpy(dense)),
             dia_array(sparse.csr_array(sp.csr_array(S))), dia_array(sparse.csc_array(sp.csc_array(S))),
             dia_array(sparse.coo_array(sp.coo_array(S))), dia_array(dia_array(S)), dia_array(dia_array(S), copy=True),
             sparse.dia_matrix(S)]
    for A in forms:
        assert isinstance(A, dia_array) and A.shape == S.shape
        np.testing.assert_array_equal(A.todense(), dense)
    A = dia_array(S, dtype=np.float32)
    assert A.dtype == np.float32
    np.testing.assert_array_equal(A.todense(), dense.astype(np.float32))
    # the CSR, CSC and COO conversions give scipy's todia: offsets ascending, L = largest column + 1
    R = sp.csr_array(S).todia()
    for A in (sparse.csr_array(sp.csr_array(S)).todia(), sparse.csc_array(sp.csc_array(S)).todia(),
              sparse.coo_array(sp.coo_array(S)).todia(), sparse.coo_array(sp.coo_array(S)).asformat("dia"),
              sparse.csc_array(sp.csc_array(S)).asformat("dia")):
        np.testing.assert_array_equal(_np(A.offsets), R.offsets)
        np.testing.assert_array_equal(_np(A.data), R.data)
    # and the CSR and CSC constructors take a dia_array
    np.testing.assert_array_equal(sparse.csr_array(dia_array(S)).todense(), dense)
    np.testing.assert_array_equal(sparse.csc_array(dia_array(S)).todense(), dense)
    assert sparse.is_sparse_matrix(dia_array(S))
    # an empty (M, N) matrix
    E = dia_array((3, 4))
    assert E.shape == (3, 4) and E.nnz == 0
    np.testing.assert_array_equal(E.todense(), np.zeros((3, 4)))


def test_repeated_entries_are_summed_by_todia():
    C = sparse.coo_array((np.array([1.0, 2.0, 4.0]), (np.array([0, 0, 2]), np.array([1, 1, 0]))), shape=(3, 3))
    A = C.todia()
    R = sp.coo_array((np.array([1.0, 2.0, 4.0]), (np.array([0, 0, 2]), np.array([1, 1, 0]))), shape=(3, 3)).todia()
    np.testing.assert_array_equal(_np(A.offsets), R.offsets)
    np.testing.assert_array_equal(_np(A.data), R.data)


def test_constructor_errors_match_scipy():
    good = np.ones((2, 3))
    bad = [
        (lambda c: c((good, np.array([[0, 1]])), shape=(3, 3)), "offsets array must have rank 1"),
        (lambda c: c((np.ones((2, 3, 1)), [0, 1]), shape=(3, 3)), "data array must have rank 2"),
        (lambda c: c((good, [0, 1, 2]), shape=(3, 3)), "number of diagonals (2) does not match the number of offsets"),
        (lambda c: c((good, [1, 1]), shape=(3, 3)), "offset array contains duplicate values"),
        (lambda c: c((good, [0, 1])), "expected a shape argument"),
    ]
    for make, msg in bad:
        with pytest.raises(ValueError) as ref:
            make(sp.dia_array)
        assert msg in str(ref.value)
        with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)")):
            make(dia_array)
    with pytest.raises(ValueError, match="Use 2D"):
        dia_array(np.ones(3))


def test_reference_spdiags_example():
    # reference tests/integration/test_dia.py
    data = np.array([[1, 2, 3, 4], [1, 2, 3, 4], [1, 2, 3, 4]])
    diags = np.array([0, -1, 2])
    A = sparse.spdiags(data, diags, 4, 4)
    assert isinstance(A, dia_array)
    np.testing.assert_array_equal(A.todense(), sp.spdiags(data, diags, 4, 4).toarray())
    np.testing.assert_array_equal(sparse.spdiags(data, diags, (4, 4)).todense(), A.todense())
    np.testing.assert_array_equal(sparse.spdiags(data, diags).todense(), A.todense())
    np.testing.assert_array_equal(sparse.spdiags(data, diags, 4, 4, format="csr").todense(), A.todense())


@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("k", [-1, 0, 1])
def test_reference_eye_cases(m, n, k):
    # reference tests/integration/test_dia.py: eye(m, n, k, format="dia") .diagonal and .tocoo()
    A = sparse.eye(m, n, k, format="dia")
    S = sp.eye_array(m, n, k=k, format="dia")
    assert isinstance(A, dia_array)
    np.testing.assert_array_equal(_np(A.diagonal(k)), S.diagonal(k))
    np.testing.assert_array_equal(A.tocoo().todense(), S.tocoo().toarray())
    np.testing.assert_array_equal(_np(A.data), S.data)


def test_eye_and_identity_keep_their_other_formats():
    for f in (None, "csr", "csc", "coo"):
        A = sparse.eye(5, 4, 1, format=f)
        assert isinstance(A, sparse.csr_array)
        np.testing.assert_array_equal(A.todense(), np.eye(5, 4, 1))
    assert isinstance(sparse.identity(3, format="dia"), dia_array)
    assert isinstance(sparse.identity(3), sparse.csr_array)
    assert sparse.eye(3, k=5).nnz == 0    # a diagonal outside the matrix: an empty matrix, as before


def test_diags_returns_scipy_diags_array():
    rng = np.random.default_rng(4)
    cases = [
        (([1.0, 2.0, 3.0], [4.0, 5.0]), [0, 1], None),
        (([1.0, 2.0, 3.0, 4.0], [5.0, 6.0, 7.0], [8.0]), [0, -1, 3], (4, 4)),
        ((rng.standard_normal(5), rng.standard_normal(5)), [0, 2], (5, 7)),
        ((rng.standard_normal(4), [2.0]), [-1, 1], (6, 4)),
    ]
    for diagonals, offsets, shape in cases:
        A = sparse.diags(diagonals, offsets, shape=shape)
        S = sp.diags_array(diagonals, offsets=offsets, shape=shape)
        assert isinstance(A, dia_array) and A.shape == S.shape and A.dtype == S.dtype
        np.testing.assert_array_equal(_np(A.offsets), S.offsets)
        np.testing.assert_array_equal(A.todense(), S.toarray())
        np.testing.assert_array_equal(_np(A.data)[:, :S.data.shape[1]], S.data)
        assert isinstance(sparse.diags(diagonals, offsets, shape=shape, format="dia"), dia_array)


def test_out_of_band_offsets_contribute_nothing():
    A = dia_array((np.ones((3, 4)), [2**62, -(2**62), 0]), shape=(4, 4))
    np.testing.assert_array_equal(A.todense(), np.eye(4))
    assert A.nnz == 4 and A.count_nonzero() == 4
    np.testing.assert_array_equal(A.tocsr().todense(), np.eye(4))
    np.testing.assert_array_equal(A.T.todense(), np.eye(4))
    offsets, data = A._in_band()
    assert _np(offsets).tolist() == [0] and tuple(data.shape) == (1, 4)


def test_offsets_property_is_a_copy_and_data_edits_are_seen():
    A = dia_array((np.arange(1.0, 5.0).reshape(1, 4), [0]), shape=(4, 4))
    o = A.offsets
    o += 1
    assert _np(A.offsets).tolist() == [0]
    C1 = A.tocsr()
    A.data[0, 0] = 0.0                 # in place: the cached CSR form is rebuilt
    assert A.tocsr() is not C1 and A.tocsr().nnz == 3
    A.data = np.full((1, 4), 2.0)
    np.testing.assert_array_equal(A.todense(), 2 * np.eye(4))


def test_scalar_operations_stay_dia():
    S = _random_dia(np.random.default_rng(5), (5, 5), [0, 1], 5)
    A = dia_array(S)
    for got, ref in ((A * 3.0, S * 3.0), (3.0 * A, 3.0 * S), (-A, -S), (abs(A), abs(S))):
        assert isinstance(got, dia_array)
        np.testing.assert_array_equal(got.todense(), ref.toarray())
    assert A.copy().data is not A.data
    assert A.astype(np.float32).dtype == np.float32 and A.conj(copy=False) is A


def test_diags_tocsr_arrays_on_the_host():
    """Without a GPU the CSR form comes from tensor operations: zeros dropped, columns sorted, the narrowest widths."""
    A = sparse.diags([[1.0, 0.0, 2.0], [-0.0, np.nan]], [0, 1], format="csr")
    assert A.indptr.dtype == torch.int32 and A.indices.dtype == torch.int32
    assert _np(A.indptr).tolist() == [0, 1, 2, 3] and _np(A.indices).tolist() == [0, 2, 2]
    assert np.isnan(_np(A.data)[1])


def _fallback_failures():
    """The products that must raise the no-CPU-fallback error when no GPU is visible, as lines saying which did not."""
    A = sparse.diags([[1.0, 2.0, 3.0], [4.0, 5.0]], [0, 1])
    out = []
    for what, f in (("A @ x", lambda: A @ np.ones(3)), ("A @ X", lambda: A @ np.ones((3, 2))),
                    ("A @ z", lambda: A @ (np.ones(3) * 1j)), ("x @ A", lambda: np.ones(3) @ A)):
        try:
            f()
            out.append(f"{what} did not raise")
        except RuntimeError as e:
            if "no CPU fallback" not in str(e):
                out.append(f"{what}: {e}")
    return out


def test_no_cpu_fallback():
    script = (
        "import sys\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import test_dia_host as t\n"
        "print('\\n'.join(t._fallback_failures()))\n"
    )
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.strip() == "", r.stdout


def test_argument_errors_need_no_device():
    A = sparse.diags([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]], [0, 1], shape=(3, 4))
    with pytest.raises(ValueError):
        A @ np.ones(3)
    with pytest.raises(ValueError):
        A.dot(np.ones(4), out=np.empty(3, dtype=np.float32))
    with pytest.raises(ValueError):
        A.dot(np.ones(4), out=np.empty(4))
    with pytest.raises(NotImplementedError):
        A.astype(np.int64) @ np.ones(4, dtype=np.int64)
    with pytest.raises(NotImplementedError):
        A @ np.ones((4, 2, 2))
    with pytest.raises(NotImplementedError):
        sparse.block_diag([A, A], format="dia")


# ---- the C entry points' checks ---------------------------------------------------------------------------------
def _abi_failures():
    """Every rejected argument set of the four DIA entry points, as 'name(kw): what happened' lines."""
    from legate.sparse_b200 import _lib

    L = _lib.lib
    buf = (ctypes.c_int64 * 4096)()
    base = ctypes.addressof(buf)
    n64 = ctypes.c_int64(0)
    got = (ctypes.c_int64 * 2)()

    def p(i):  # one 256-byte slot per array, so no two arguments overlap unless a case says so
        return base + 256 * i

    def spmv(vt=_lib.F64, m=4, n=4, nd=2, Ld=4, x=p(3), y=p(4)):
        return L.b2s_spmv_dia(vt, m, n, nd, Ld, p(0), p(1), x, y, None)

    def spmm(vt=_lib.F64, m=4, n=4, nd=2, Ld=4, k=2, X=p(3), ldx=2, Y=p(5), ldy=2):
        return L.b2s_spmm_dia(vt, m, n, nd, Ld, k, p(0), p(1), X, ldx, Y, ldy, None)

    def to_csr(vt=_lib.F64, it=_lib.I32, pt=_lib.I32, m=4, n=4, nd=2, Ld=4, nnz=4, indptr=p(4), idx=p(6), val=p(7),
               scratch=p(9), sb=256):
        return L.b2s_dia_to_csr(vt, it, pt, m, n, nd, Ld, p(0), p(2), p(1), nnz, indptr, idx, val, scratch, sb,
                                ctypes.byref(n64), None)

    def to_dia(vt=_lib.F64, it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4, nd=2, Ld=4, offs=p(6), data=p(7),
               scratch=p(9), sb=2048):
        return L.b2s_csr_to_dia(vt, it, pt, m, n, nnz, p(0), p(1), p(2), nd, Ld, offs, data, scratch, sb, got, None)

    dia_common = [
        (dict(vt=7), "bad value type code 7"),
        (dict(m=-1), "negative dimension"),
        (dict(n=-1), "negative dimension"),
        (dict(nd=-1), "negative dimension"),
        (dict(Ld=-1), "negative dimension"),
        (dict(nd=2**40, Ld=2**40), "overflows int64"),
    ]
    cases = [(f, call, kw, msg) for f, call in (("b2s_spmv_dia", spmv), ("b2s_spmm_dia", spmm),
                                               ("b2s_dia_to_csr", to_csr)) for kw, msg in dia_common]
    cases += [("b2s_csr_to_dia", to_dia, kw, msg) for kw, msg in dia_common[:3]]
    cases += [("b2s_csr_to_dia", to_dia, kw, msg) for kw, msg in dia_common[3:]]
    cases += [
        ("b2s_spmv_dia", spmv, dict(y=p(3) + 8), "y overlaps x"),
        ("b2s_spmv_dia", spmv, dict(y=p(1)), "y overlaps data"),
        ("b2s_spmv_dia", spmv, dict(y=p(0)), "y overlaps offsets"),
        ("b2s_spmm_dia", spmm, dict(k=-1), "negative dimension"),
        ("b2s_spmm_dia", spmm, dict(Y=p(3) + 16), "Y overlaps X"),
        ("b2s_spmm_dia", spmm, dict(ldx=1), "leading dimensions (1, 2) smaller than k = 2"),
        ("b2s_spmm_dia", spmm, dict(ldy=1), "leading dimensions (2, 1) smaller than k = 2"),
        ("b2s_dia_to_csr", to_csr, dict(it=5), "bad index type code 5"),
        ("b2s_dia_to_csr", to_csr, dict(pt=9), "bad indptr type code 9"),
        ("b2s_dia_to_csr", to_csr, dict(nnz=2**31 - 1), "int32 indptr cannot address nnz >= 2^31-1"),
        ("b2s_dia_to_csr", to_csr, dict(indptr=p(1)), "indptr overlaps an input"),
        ("b2s_dia_to_csr", to_csr, dict(idx=p(7)), "indices/vals overlap another array"),
        ("b2s_dia_to_csr", to_csr, dict(idx=None, val=None, sb=8), "scratch needs"),
        ("b2s_csr_to_dia", to_dia, dict(it=5), "bad index type code 5"),
        ("b2s_csr_to_dia", to_dia, dict(pt=9), "bad indptr type code 9"),
        ("b2s_csr_to_dia", to_dia, dict(nnz=-1), "negative dimension"),
        ("b2s_csr_to_dia", to_dia, dict(nnz=2**31 - 1), "int32 indptr cannot address nnz >= 2^31-1"),
        ("b2s_csr_to_dia", to_dia, dict(sb=8), "scratch needs"),
        ("b2s_csr_to_dia", to_dia, dict(scratch=p(1)), "scratch overlaps an input"),
        ("b2s_csr_to_dia", to_dia, dict(data=p(6) + 8), "offsets/data overlap another array"),
    ]
    out = []
    for name, call, kw, msg in cases:
        rc = call(**kw)
        err = _lib.last_error()
        if rc != _lib.EINVAL or msg not in err:
            out.append(f"{name}({kw}): rc {rc}, {err!r}, expected EINVAL and {msg!r}")
    # nothing to compute needs no pointer at all
    if L.b2s_spmv_dia(_lib.F64, 0, 0, 0, 0, None, None, None, None, None) != _lib.OK:
        out.append(f"b2s_spmv_dia of a 0 x 0 matrix: {_lib.last_error()!r}")
    if spmm(m=3, n=0, nd=0, Ld=0, k=0, X=None, Y=None) != _lib.OK:
        out.append(f"b2s_spmm_dia with k = 0: {_lib.last_error()!r}")
    if L.b2s_dia_scratch_bytes(-1, 4) != 0 or L.b2s_dia_scratch_bytes(4, 4) < 8 * 7:
        out.append("b2s_dia_scratch_bytes")
    return out


def test_abi_rejects_bad_arguments():
    script = (
        "import sys\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import test_dia_host as t\n"
        "print('\\n'.join(t._abi_failures()))\n"
    )
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.strip() == "", r.stdout


@pytest.mark.parametrize("name", MTX_FILES)
def test_fixtures_round_trip(name):
    S = sp.csr_array(scipy.io.mmread(mtx_path(name)))
    if S.shape[0] + S.shape[1] > 4000:
        pytest.skip("a DIA form of this fixture is large")
    with np.errstate(all="ignore"), __import__("warnings").catch_warnings():
        __import__("warnings").simplefilter("ignore")
        R = S.todia()
        A = sparse.csr_array(S).todia()
    np.testing.assert_array_equal(_np(A.offsets), R.offsets)
    np.testing.assert_array_equal(_np(A.data), R.data)
    np.testing.assert_array_equal(A.todense(), S.toarray())


def test_gpu_file_passes_the_cpu_dry_run():
    script = (
        "import sys, pytest\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import dryrun_cpu\n"
        "dryrun_cpu.install()\n"
        "from legate.sparse_b200 import _ops\n"
        "import test_csc_host, test_dia_host, test_reduce_host, test_sddmm_host\n"
        "_ops.spmv_dia = test_dia_host._dryrun_spmv_dia\n"
        "_ops.spmm_dia = test_dia_host._dryrun_spmm_dia\n"
        "_ops.csr_binop = test_csc_host._dryrun_binop\n"
        "_ops.csr_reduce_rows = test_reduce_host._dryrun_reduce\n"
        "_ops.csr_sort_rows = test_reduce_host._dryrun_sort_rows\n"
        "_ops.sddmm = test_sddmm_host._dryrun_sddmm\n"
        "sys.exit(pytest.main(['-m', 'gpu', '-q', '-p', 'no:cacheprovider', sys.argv[1], '-k', sys.argv[2]]))\n"
    )
    # the 10M-row matrices are minutes of numpy here; the solvers' fused kernels have no stand-in
    r = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "tests", "test_gpu_dia.py"),
                        "not large and not solvers and not too_large"], capture_output=True, text=True, timeout=900,
                       cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
