"""The CSR operand contract of the C ABI, checked at every entry point that takes an index and an indptr type code.

include/b200sparse.h (Conventions) states it once: `it` and `pt` are B2S_I32 or B2S_I64, nrows, ncols and nnz are not
negative, and an int32 indptr cannot address nnz >= 2^31-1.  Each entry point below must reject a violation with
B2S_EINVAL and the same message.  Pointers are host addresses of a small ctypes buffer, so the calls run in a
subprocess that sees no CUDA device: a call that got past its checks would then fail on its first CUDA call instead of
handing host memory to a kernel."""
import ctypes
import os
import subprocess
import sys

from conftest import ROOT

INT32_LIMIT = 2**31 - 1


def _entries():
    """name -> (call(it, pt, m, n, nnz), takes ncols, takes nnz).  Every argument other than the operand's is valid."""
    from legate.sparse_b200 import _lib

    L = _lib.lib
    buf = (ctypes.c_int64 * 2048)()
    base = ctypes.addressof(buf)

    def p(i):  # one 128-byte slot per array, so no two arguments overlap
        return base + 128 * i

    F64, I32 = _lib.F64, _lib.I32
    plan = ctypes.c_void_p()
    return {
        "b2s_spmv_csr": (lambda it, pt, m, n, nnz: L.b2s_spmv_csr(
            F64, it, pt, m, n, nnz, p(0), p(1), p(2), p(3), p(4), None, None), True, True),
        "b2s_spmv_plan_create": (lambda it, pt, m, n, nnz: L.b2s_spmv_plan_create(
            F64, it, pt, m, n, nnz, p(0), p(1), p(2), None, ctypes.byref(plan)), True, True),
        "b2s_spmm_csr": (lambda it, pt, m, n, nnz: L.b2s_spmm_csr(
            F64, it, pt, m, n, nnz, 2, p(0), p(1), p(2), p(3), 2, p(4), 2, None), True, True),
        "b2s_sddmm_csr": (lambda it, pt, m, n, nnz: L.b2s_sddmm_csr(
            F64, it, pt, m, n, nnz, 2, p(0), p(1), p(2), p(3), 2, p(4), 2, p(5), None), True, True),
        "b2s_tropical_spmv_csr": (lambda it, pt, m, n, nnz: L.b2s_tropical_spmv_csr(
            it, pt, m, n, nnz, 2, p(0), p(1), p(2), 2, p(3), 2, None), True, True),
        "b2s_csr_reduce_rows": (lambda it, pt, m, n, nnz: L.b2s_csr_reduce_rows(
            0, F64, it, pt, m, n, nnz, p(0), p(1), p(2), 0, p(3), None), True, True),
        "b2s_csr_select": (lambda it, pt, m, n, nnz: L.b2s_csr_select(
            0, 8, it, pt, I32, m, n, nnz, p(0), p(1), p(2), 2, p(3), 0, 1, None, None, n, p(4), p(5), p(6), 4,
            p(7), p(8), None), True, True),
        "b2s_csr_lookup": (lambda it, pt, m, n, nnz: L.b2s_csr_lookup(
            F64, it, pt, m, n, nnz, p(0), p(1), p(2), 2, p(3), p(4), p(5), p(6), None), True, True),
        "b2s_coo_to_csr": (lambda it, pt, m, n, nnz: L.b2s_coo_to_csr(
            F64, it, pt, m, nnz, p(0), p(1), p(2), p(3), p(4), p(5), p(6), p(7), None), False, True),
        "b2s_csr_transpose": (lambda it, pt, m, n, nnz: L.b2s_csr_transpose(
            F64, it, pt, m, n, nnz, p(0), p(1), p(2), p(3), p(4), p(5), p(6), None), True, True),
        "b2s_csr_sort_rows": (lambda it, pt, m, n, nnz: L.b2s_csr_sort_rows(
            F64, it, pt, m, nnz, p(0), p(1), p(2), p(3), None), False, True),
        "b2s_csr_binop_symbolic": (lambda it, pt, m, n, nnz: L.b2s_csr_binop_symbolic(
            0, it, pt, m, n, p(0), p(1), p(2), p(3), p(4), p(5), p(6), None), True, False),
        "b2s_csr_binop_numeric": (lambda it, pt, m, n, nnz: L.b2s_csr_binop_numeric(
            0, F64, it, pt, m, n, p(0), p(1), p(2), p(3), p(4), p(5), p(6), p(7), p(8), p(9), None), True, False),
        "b2s_csr_scale": (lambda it, pt, m, n, nnz: L.b2s_csr_scale(
            F64, it, pt, m, n, nnz, 0, p(0), p(1), p(2), p(3), n, p(4), None), True, True),
        "b2s_csr_diagonal": (lambda it, pt, m, n, nnz: L.b2s_csr_diagonal(
            F64, it, pt, m, p(0), p(1), p(2), p(3), None), False, False),
    }


def _cases(takes_ncols, takes_nnz):
    """(arguments that break the contract once, the message every entry point gives)"""
    from legate.sparse_b200 import _lib

    ok = dict(it=_lib.I32, pt=_lib.I32, m=4, n=4, nnz=4)
    cases = [
        (dict(ok, it=5), "bad index type code 5"),
        (dict(ok, pt=9), "bad indptr type code 9"),
        (dict(ok, m=-1), "negative dimension"),
    ]
    if takes_ncols:
        cases.append((dict(ok, n=-1), "negative dimension"))
    if takes_nnz:
        cases.append((dict(ok, nnz=-1), "negative dimension"))
        cases.append((dict(ok, nnz=INT32_LIMIT), "int32 indptr cannot address nnz >= 2^31-1"))
    return cases


def _failures():
    from legate.sparse_b200 import _lib

    out = []
    for name, (call, takes_ncols, takes_nnz) in _entries().items():
        for kw, msg in _cases(takes_ncols, takes_nnz):
            rc = call(**kw)
            err = _lib.last_error()
            if rc != _lib.EINVAL or msg not in err:
                out.append(f"{name}({kw}): rc {rc}, {err!r}, expected EINVAL and {msg!r}")
    return out


def test_every_entry_point_checks_the_csr_operand_alike():
    script = (
        "import sys\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import test_abi_csr_checks_host as t\n"
        "print('\\n'.join(t._failures()))\n"
    )
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.strip() == "", r.stdout
