"""Host-side checks of `csr_array.tropical_spmv` (the lexicographic-max product of csrc/tropical.cu).

`tropical_oracle` restates the reference kernel (src/sparse/array/csr/tropical_spmv.cu:26-56) with numpy: y[i] is the
lexicographic maximum of the zero vector and of x[j] over the stored entries (i, j), fields compared as signed int64
with field 0 the most significant.  It is pinned to `literal`, a per-row Python loop written the way the reference
kernel is (start from zero, replace only when a neighbour is strictly greater), on the MatrixMarket fixtures and on
hand-computed cases.  The argument checks need no device, nor do the C entry point's own checks.  The `-m gpu` file is
rehearsed through tests/dryrun_cpu.py with `_ops.tropical_spmv` swapped for the oracle."""
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


def tropical_oracle(indptr, indices, x):
    """(m, F) int64: per row, the lexicographic max of 0 and x[indices[p]] over the row's entries p."""
    indptr, indices = np.asarray(indptr).astype(np.int64), np.asarray(indices).astype(np.int64)
    x = np.asarray(x).astype(np.int64)
    m, nf = indptr.size - 1, x.shape[1]
    y = np.zeros((m, nf), dtype=np.int64)
    if nf == 0 or indices.size == 0:
        return y
    rows = np.repeat(np.arange(m), np.diff(indptr))
    vals = x[indices]
    # sort the entries by (row, field 0, field 1, ...): the last entry of each row is that row's maximum
    order = np.lexsort(tuple(vals[:, f] for f in range(nf - 1, -1, -1)) + (rows,))
    last = order[np.r_[np.flatnonzero(np.diff(rows[order])), order.size - 1]]
    best = vals[last]
    # floor at zero: keep a maximum only when its first nonzero field is positive
    nz = best != 0
    first = np.argmax(nz, axis=1)
    positive = nz.any(axis=1) & (best[np.arange(best.shape[0]), first] > 0)
    y[rows[last[positive]]] = best[positive]
    return y


def literal(indptr, indices, x):
    """The reference kernel's loop, one row at a time, in Python integers."""
    x = np.asarray(x).astype(np.int64)
    m, nf = len(indptr) - 1, x.shape[1]
    y = np.zeros((m, nf), dtype=np.int64)
    for i in range(m):
        cur = [0] * nf
        for p in range(int(indptr[i]), int(indptr[i + 1])):
            cand = [int(v) for v in x[int(indices[p])]]
            if cand > cur:                       # Python list order is lexicographic
                cur = cand
        y[i] = cur
    return y


def _dryrun_tropical(indptr, indices, x, y=None):
    """`_ops.tropical_spmv` for the CPU dry run of the GPU test file."""
    v = torch.from_numpy(tropical_oracle(indptr.numpy(), indices.numpy(), x.numpy()))
    if y is None:
        return v
    y.copy_(v)
    return y


def _values(n, nf, seed, lo=-3, hi=4):
    """Small integers (ties and negatives are common), with int64 extremes mixed in."""
    rng = np.random.default_rng(seed)
    x = rng.integers(lo, hi, (n, nf), dtype=np.int64)
    ext = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0, 1], dtype=np.int64)
    mask = rng.random((n, nf)) < 0.05
    x[mask] = rng.choice(ext, int(mask.sum()))
    return x


@pytest.mark.parametrize("name", MTX_FILES)
@pytest.mark.parametrize("nf", [0, 1, 2, 3, 5])
def test_oracle_matches_literal_loop_on_fixtures(name, nf):
    S = sp.csr_array(scipy.io.mmread(mtx_path(name)))
    x = _values(S.shape[1], nf, seed=nf)
    got = tropical_oracle(S.indptr, S.indices, x)
    assert got.dtype == np.int64 and got.shape == (S.shape[0], nf)
    assert np.array_equal(got, literal(S.indptr, S.indices, x))


def test_hand_computed_cases():
    # row 0: column 2 twice and column 1 (unsorted); row 1: only negative neighbours; row 2: an explicit-zero entry
    # pointing at the largest row; row 3 empty; row 4: a tie in field 0 decided by field 1; row 5: ties throughout
    x = np.array([[0, 0], [1, -5], [1, -7], [-1, 100], [3, 1], [3, 2], [-2, 0]], dtype=np.int64)
    indptr = np.array([0, 3, 5, 6, 6, 8, 10])
    indices = np.array([2, 2, 1, 3, 6, 5, 4, 5, 1, 1])
    data = np.array([1.0, 1.0, 1.0, 2.0, 2.0, 0.0, 1.0, 1.0, 1.0, 1.0])   # values never matter
    want = np.array([[1, -5], [0, 0], [3, 2], [0, 0], [3, 2], [1, -5]], dtype=np.int64)
    assert np.array_equal(tropical_oracle(indptr, indices, x), want)
    assert np.array_equal(literal(indptr, indices, x), want)
    # field 0 zero, field 1 negative: below the zero vector, so the floor wins
    assert np.array_equal(tropical_oracle([0, 1], [0], np.array([[0, -1]])), [[0, 0]])
    assert np.array_equal(tropical_oracle([0, 1], [0], np.array([[0, 0, 1]])), [[0, 0, 1]])
    # the extremes of int64 compare as signed
    big = np.array([[np.iinfo(np.int64).max], [np.iinfo(np.int64).min]])
    assert np.array_equal(tropical_oracle([0, 2, 3], [0, 1, 1], big), [[np.iinfo(np.int64).max], [0]])
    # values and explicit zeros play no part: a csr_array keeps the structure exactly
    A = csr_array((torch.tensor(data), torch.tensor(indices, dtype=torch.int32),
                   torch.tensor(indptr, dtype=torch.int32)), shape=(6, 7))
    assert A.nnz == 10


def test_argument_errors_need_no_device():
    A = csr_array(sp.random_array((5, 6), density=0.5, format="csr", rng=np.random.default_rng(0)))
    x = np.ones((6, 3), dtype=np.int64)
    for bad in (np.ones(6, dtype=np.int64), np.ones((6, 3, 1), dtype=np.int64), np.ones((5, 3), dtype=np.int64),
                torch.ones((7, 2), dtype=torch.int64)):
        with pytest.raises(ValueError):
            A.tropical_spmv(bad)
    for bad in (x.astype(np.float64), x.astype(np.complex128), x.astype(bool), torch.ones((6, 3)),
                torch.ones((6, 3), dtype=torch.bool), torch.ones((6, 3), dtype=torch.complex64)):
        with pytest.raises(TypeError):
            A.tropical_spmv(bad)
    for out in (np.zeros((5, 2), dtype=np.int64), np.zeros((5, 3), dtype=np.int32), np.zeros((5, 3)),
                torch.zeros((5, 3), dtype=torch.int32), [[0] * 3] * 5, np.zeros(15, dtype=np.int64)):
        with pytest.raises(ValueError):
            A.tropical_spmv(x, out=out)
    # out overlapping x: the same buffer, a view of it, or a CPU tensor sharing it
    S = csr_array(sp.random_array((6, 6), density=0.5, format="csr", rng=np.random.default_rng(1)))
    buf = np.zeros((6, 6), dtype=np.int64)
    for xx, out in ((buf[:, :3], buf[:, :3]), (buf[:, :3], buf[:, 3:]), (buf[:, ::2], buf[:, 1::2]),
                    (torch.from_numpy(buf[:, :3]), buf[:, 2:5])):
        with pytest.raises(ValueError):
            S.tropical_spmv(xx, out=out)
    t = torch.zeros((6, 6), dtype=torch.int64)
    with pytest.raises(ValueError):
        S.tropical_spmv(t[:, :3], out=t[:, 3:])
    # a complex matrix is fine: only the structure counts (the call reaches the device check, or runs)
    Z = csr_array(sp.random_array((5, 6), density=0.5, format="csr", dtype=np.complex64, rng=np.random.default_rng(2)))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CUDA device"):
            Z.tropical_spmv(x)


def test_abi_rejects_bad_arguments():
    from legate.sparse_b200 import _lib

    L = _lib.lib
    xbuf = (ctypes.c_int64 * 64)()
    ybuf = (ctypes.c_int64 * 64)()
    px, py = ctypes.addressof(xbuf), ctypes.addressof(ybuf)

    def call(it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4, nf=2, indptr=px, indices=px, x=px, ldx=2, y=py, ldy=2):
        rc = L.b2s_tropical_spmv_csr(it, pt, m, n, nnz, nf, indptr, indices, x, ldx, y, ldy, None)
        return rc, _lib.last_error()

    cases = [
        (dict(it=5), "bad index type code 5"),
        (dict(pt=9), "bad indptr type code 9"),
        (dict(m=-1), "negative dimension"),
        (dict(n=-1), "negative dimension"),
        (dict(nnz=-1), "negative dimension"),
        (dict(nf=-1), "negative dimension"),
        (dict(ldx=1), "leading dimensions (1, 2) smaller than nfields = 2"),
        (dict(ldy=1), "leading dimensions (2, 1) smaller than nfields = 2"),
        (dict(nnz=2**31), "int32 indptr cannot address nnz >= 2^31-1"),
        (dict(indptr=None), "indptr is NULL"),
        (dict(y=None), "y is NULL"),
        (dict(indices=None), "indices/x NULL with nnz > 0"),
        (dict(x=None), "indices/x NULL with nnz > 0"),
        (dict(n=0), "nnz > 0 in a matrix with no columns"),
        (dict(y=px), "x and y overlap"),
        (dict(y=px + 8 * 7), "x and y overlap"),          # x spans 8 int64 (4 rows of 2), y starts at x's last one
    ]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc == _lib.EINVAL and msg in err, (kw, err)
    # nothing to compute: no pointer is needed
    assert call(m=0, indptr=None, indices=None, x=None, y=None)[0] == _lib.OK
    assert call(nf=0, ldx=0, ldy=0, indptr=None, indices=None, x=None, y=None)[0] == _lib.OK


def test_gpu_file_passes_the_cpu_dry_run():
    script = (
        "import sys, pytest\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import dryrun_cpu\n"
        "dryrun_cpu.install()\n"
        "from legate.sparse_b200 import _ops\n"
        "import test_tropical_host\n"
        "_ops.tropical_spmv = test_tropical_host._dryrun_tropical\n"
        "sys.exit(pytest.main(['-m', 'gpu', '-q', '-p', 'no:cacheprovider', sys.argv[1], '-k', sys.argv[2]]))\n"
    )
    # the graph test needs a device; the full-size cases are minutes of numpy here
    r = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "tests", "test_gpu_tropical.py"),
                        "not graph and not full_size"], capture_output=True, text=True, timeout=900, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
