"""Host-side checks of `csr_array.sddmm` (the sampled dense-dense product of csrc/sddmm.cu).

`sddmm_oracle` restates, on the host, the reference's CPU body (src/sparse/array/csr/sddmm.cc:37-46): every stored
entry p = (i, j) on its own, out[p] = A.data[p] * sum_t C[i, t] * D[t, j], the sum taken in t order in the result
dtype.  It is pinned to scipy's `S.multiply(C @ D)` on the MatrixMarket fixtures (the reference test's cases) and to
hand-computed values on a matrix with a repeated column, an unsorted row and an explicit zero.  The argument checks
need no device, nor do the C entry point's own checks.  The `-m gpu` file is rehearsed through tests/dryrun_cpu.py
with `_ops.sddmm` swapped for the oracle."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from legate.sparse_b200.csr import csr_array

from conftest import MTX_FILES, ROOT, mtx_path


def sddmm_oracle(indptr, indices, data, C, D):
    """Values of A ⊙ (C @ D) on A's stored entries, in np.result_type(data, C, D)."""
    indptr, indices = np.asarray(indptr).astype(np.int64), np.asarray(indices).astype(np.int64)
    dt = np.result_type(np.asarray(data).dtype, np.asarray(C).dtype, np.asarray(D).dtype)
    a, C, D = np.asarray(data, dtype=dt), np.asarray(C, dtype=dt), np.asarray(D, dtype=dt)
    rows = np.repeat(np.arange(indptr.size - 1), np.diff(indptr))
    dot = np.zeros(a.size, dtype=dt)
    for t in range(C.shape[1]):
        dot = dot + C[rows, t] * D[t, indices]
    return a * dot


def _dryrun_sddmm(indptr, indices, data, C, Dt, out=None):
    """`_ops.sddmm` for the CPU dry run of the GPU test file."""
    v = torch.from_numpy(np.ascontiguousarray(sddmm_oracle(indptr.numpy(), indices.numpy(), data.numpy(), C.numpy(),
                                                           Dt.numpy().T)))
    if out is None:
        return v
    out.copy_(v)
    return out


@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("k", [2, 4, 8, 16])
def test_oracle_matches_scipy_on_fixtures(name, k):
    S = sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(np.float64)
    rng = np.random.default_rng(k)
    C = rng.standard_normal((S.shape[0], k))
    D = rng.standard_normal((k, S.shape[1]))
    R = sp.csr_array(S.multiply(C @ D))
    R.sort_indices()
    got = sp.csr_array((sddmm_oracle(S.indptr, S.indices, S.data, C, D), S.indices, S.indptr), shape=S.shape)
    got.sort_indices()
    assert np.array_equal(got.indptr, R.indptr) and np.array_equal(got.indices, R.indices)
    assert np.allclose(got.data, R.data, rtol=1e-12, atol=1e-12)


def test_oracle_keeps_every_stored_entry():
    # row 0: column 2 twice; row 1 unsorted (3, 0); row 2: an explicit zero and a NaN-free entry; row 3 empty
    data = np.array([1.0, 2.0, 3.0, -1.0, 0.0, 4.0])
    indices = np.array([2, 2, 1, 3, 0, 1])
    indptr = np.array([0, 3, 5, 6, 6])
    C = np.arange(8.0).reshape(4, 2)
    D = np.arange(10.0).reshape(2, 5) - 3.0
    P = C @ D
    rows = [0, 0, 0, 1, 1, 2]
    want = np.array([data[p] * P[rows[p], indices[p]] for p in range(6)])
    got = sddmm_oracle(indptr, indices, data, C, D)
    assert np.array_equal(got, want) and got[4] == 0.0
    zero_k = sddmm_oracle(indptr, indices, np.array([np.nan, 1, 2, 3, np.inf, 5]), np.zeros((4, 0)), np.zeros((0, 5)))
    assert np.isnan(zero_k[0]) and np.isnan(zero_k[4]) and np.array_equal(zero_k[[1, 2, 3, 5]], np.zeros(4))


def test_argument_errors_need_no_device():
    A = csr_array(sp.random_array((5, 6), density=0.5, format="csr", rng=np.random.default_rng(0)))
    C, D = np.ones((5, 3)), np.ones((3, 6))
    for c, d in ((np.ones((4, 3)), D), (C, np.ones((3, 5))), (C, np.ones((2, 6))), (np.ones(5), D), (C, np.ones((3, 6, 1)))):
        with pytest.raises(ValueError):
            A.sddmm(c, d)
    with pytest.raises(NotImplementedError):
        A.sddmm(C.astype(np.complex128), D)
    Z = csr_array(sp.random_array((5, 6), density=0.5, format="csr", dtype=np.complex64, rng=np.random.default_rng(1)))
    with pytest.raises(NotImplementedError):
        Z.sddmm(C, D)
    with pytest.raises(NotImplementedError):
        A.astype(np.int64).sddmm(C.astype(np.int64), torch.ones((3, 6), dtype=torch.int64))


def test_abi_rejects_bad_arguments():
    from legate.sparse_b200 import _lib

    L = _lib.lib
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)

    def call(vt=_lib.F64, it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4, k=2, indptr=p, indices=p, vals=p, C=p, ldc=2, Dt=p,
             ldd=2, out=p):
        rc = L.b2s_sddmm_csr(vt, it, pt, m, n, nnz, k, indptr, indices, vals, C, ldc, Dt, ldd, out, None)
        return rc, _lib.last_error()

    cases = [
        (dict(vt=7), "bad value type code 7"),
        (dict(it=5), "bad index type code 5"),
        (dict(pt=9), "bad indptr type code 9"),
        (dict(k=-1), "negative dimension"),
        (dict(ldc=1), "leading dimensions (1, 2) smaller than k = 2"),
        (dict(ldd=1), "leading dimensions (2, 1) smaller than k = 2"),
        (dict(nnz=2**31), "int32 indptr cannot address nnz >= 2^31-1"),
        (dict(indptr=None), "indptr is NULL"),
        (dict(indices=None), "indices/vals NULL with nnz > 0"),
        (dict(vals=None), "indices/vals NULL with nnz > 0"),
        (dict(C=None), "C/Dt NULL with k > 0"),
        (dict(Dt=None), "C/Dt NULL with k > 0"),
        (dict(out=None), "out is NULL"),
        (dict(m=0), "nnz > 0 in a matrix with no rows or no columns"),
    ]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc == _lib.EINVAL and msg in err, (kw, err)
    # nothing to compute: no pointer is needed
    assert call(nnz=0, indptr=None, indices=None, vals=None, C=None, Dt=None, out=None)[0] == _lib.OK


def test_gpu_file_passes_the_cpu_dry_run():
    script = (
        "import sys, pytest\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import dryrun_cpu\n"
        "dryrun_cpu.install()\n"
        "from legate.sparse_b200 import _ops\n"
        "import test_sddmm_host\n"
        "_ops.sddmm = test_sddmm_host._dryrun_sddmm\n"
        "sys.exit(pytest.main(['-m', 'gpu', '-q', '-p', 'no:cacheprovider', sys.argv[1], '-k', sys.argv[2]]))\n"
    )
    # the graph test needs a device; the full-size case is minutes of numpy here
    r = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "tests", "test_gpu_sddmm.py"),
                        "not graph and not full_size"], capture_output=True, text=True, timeout=900, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
