"""Host-side checks of the dense-operand products of `csr_array`, `csc_array` and `dia_array`
(legate/sparse_b200/_dense.py).

Argument errors come before the device is needed, so they are checked here with no GPU, class by class: csr keeps the
reference's AssertionError for a wrong leading dimension or `out` shape, csc and dia raise ValueError.  The helpers that
choose operand and output layouts and deliver results are checked on host tensors.  The `-m gpu` file is rehearsed
through tests/dryrun_cpu.py with the CSC and DIA launchers swapped for their numpy restatements."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200._dense import deliver, dense_rows, direct_out

from conftest import ROOT

M, N = 5, 6


@pytest.fixture(autouse=True)
def _host_only(monkeypatch):
    """The host side as it runs without a GPU, also where one is visible: arrays stay on the host."""
    from legate.sparse_b200.runtime import Runtime

    monkeypatch.setattr(Runtime, "has_cuda", property(lambda self: False))


def _matrix(fmt, dtype=np.float64):
    S = sp.random_array((M, N), density=0.5, format="csr", rng=np.random.default_rng(3)).astype(dtype)
    return {"csr": sparse.csr_array, "csc": lambda S: sparse.csc_array(S.tocsc()), "dia": sparse.dia_array}[fmt](S)


@pytest.mark.parametrize("fmt", ["csr", "csc", "dia"])
def test_argument_errors_come_before_the_device(fmt):
    A = _matrix(fmt)
    csr = fmt == "csr"
    for x in (np.ones(N + 1), np.ones((N - 1, 1)), np.ones((N - 1, 3))):
        with pytest.raises(AssertionError) if csr else pytest.raises(ValueError, match=r"dimension mismatch: \(5, 6\)"):
            A.dot(x)
    for x, out in ((np.ones(N), np.empty(M + 1)), (np.ones((N, 1)), np.empty(M)), (np.ones((N, 3)), np.empty((M, 2))),
                   (np.ones(N) * 1j, np.empty(M + 1, dtype=np.complex128))):
        with pytest.raises(AssertionError) if csr else pytest.raises(ValueError, match="out has shape"):
            A.dot(x, out=out)
    for x, out in ((np.ones(N), np.empty(M, dtype=np.float32)), (np.ones((N, 3)), np.empty((M, 3), dtype=np.float32))):
        with pytest.raises(ValueError, match="^Output type float32 is not consistent with resolved dtype float64$"):
            A.dot(x, out=out)
    with pytest.raises(ValueError, match="^Output type float64 is not consistent with resolved dtype complex128$"):
        A.dot(np.ones(N) * 1j, out=np.empty(M))
    with pytest.raises(NotImplementedError, match=f"^{fmt}_array.dot: operand must be a vector, a dense 2-D array"):
        A.dot(np.ones((N, 2, 2)))
    with pytest.raises(NotImplementedError, match=f"^{fmt}_array.dot: operand must be a vector, a dense 2-D array"):
        A.dot(np.ones((N + 1, 2, 2)))   # a 3-D operand is refused whatever its length
    B = A.astype(np.int64)
    with pytest.raises(NotImplementedError, match=r"^SpMV for resolved dtype int64 is not implemented \(float32/float64"):
        B.dot(np.ones(N, dtype=np.int64))
    with pytest.raises(NotImplementedError, match=r"^SpMV for resolved dtype int64 is not implemented \(float32/float64"):
        B.dot(np.ones((N, 1), dtype=np.int64))
    with pytest.raises(NotImplementedError, match=r"^SpMM for resolved dtype int64 is not implemented \(float32/float64"):
        B.dot(np.ones((N, 3), dtype=np.int64))
    for x in (np.ones(N), np.ones((N, 3)), np.ones(N) * 1j, torch.ones(N, dtype=torch.float32)):
        with pytest.raises(RuntimeError, match=f"{fmt}_array.dot: no CUDA device is visible"):
            A.dot(x)


def test_deliver_returns_the_callers_array_kind():
    res = torch.arange(6, dtype=torch.float64).reshape(3, 2)
    got = deliver(res, None, False, False)
    assert isinstance(got, np.ndarray) and np.array_equal(got, res.numpy())
    assert deliver(res, None, True, False) is res
    for out in (np.zeros((3, 2)), np.zeros((3, 4))[:, ::2], np.zeros((2, 3)).T, torch.zeros(3, 2),
                torch.zeros(3, 4)[:, ::2]):
        assert deliver(res, out, False, False) is out
        assert np.array_equal(np.asarray(out), res.numpy())
    written = torch.full((3, 2), 7.0)
    assert deliver(res, written, True, True) is written and bool((written == 7).all())   # the kernel wrote it


def test_layout_rules():
    assert not direct_out(None, (3,)) and not direct_out(np.zeros(3), (3,)) and not direct_out(torch.zeros(3), (3,))
    t = torch.zeros(4, 5)
    assert dense_rows(t, np.float64).data_ptr() != t.data_ptr()          # a new dtype is a new tensor
    t = torch.zeros(4, 5, dtype=torch.float64)
    assert dense_rows(t, np.float64) is t
    assert dense_rows(t[:, :3], np.float64).data_ptr() == t.data_ptr()  # padded rows are used as they are
    for a in (t[:, ::2], t.T, torch.zeros(1, 5, dtype=torch.float64).expand(4, 5),
              t.as_strided((4, 3), (1, 1))):
        d = dense_rows(a, np.float64)
        assert d.is_contiguous() and torch.equal(d, a)
    d = dense_rows(np.asfortranarray(np.ones((4, 3))), np.float64)
    assert d.is_contiguous()


def test_gpu_file_passes_the_cpu_dry_run():
    script = (
        "import sys, pytest\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import dryrun_cpu\n"
        "dryrun_cpu.install()\n"
        "from legate.sparse_b200 import _ops\n"
        "import test_csc_host, test_dia_host\n"
        "_ops.spmv_csc = test_csc_host._dryrun_spmv_csc\n"
        "_ops.spmm_csc = test_csc_host._dryrun_spmm_csc\n"
        "_ops.spmv_dia = test_dia_host._dryrun_spmv_dia\n"
        "_ops.spmm_dia = test_dia_host._dryrun_spmm_dia\n"
        "sys.exit(pytest.main(['-m', 'gpu', '-q', '-p', 'no:cacheprovider', sys.argv[1]]))\n"
    )
    r = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "tests", "test_gpu_dense_products.py")],
                       capture_output=True, text=True, timeout=900, cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
