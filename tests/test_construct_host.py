"""Host-side checks of assembly from blocks: kron, kronsum, bmat, hstack, vstack, block_diag (csrc/construct.cu through
`_ops.csr_kron` and `_ops.csr_blocks`).

`kron_oracle` and `bmat_oracle` restate with numpy the entry order the kernels write: kron's output row i * p + r holds,
for each stored entry of row i of A in stored order, row r of B in stored order; bmat's output row is the concatenation,
left to right, of the rows of the blocks beside it.  Both are pinned to scipy 1.18.1: structure and bytes on canonical
inputs, dense values on inputs with unsorted rows, duplicates, explicit zeros, empty rows and empty matrices (scipy sums
duplicates there, the library keeps them).  The shape errors are pinned to scipy's (ValueError exactly where scipy
raises one), and the C entry points' CSR operand contract is checked as tests/test_abi_csr_checks_host.py checks the
others."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp

from conftest import MTX_FILES, ROOT, mtx_path

import legate.sparse_b200 as sparse
from legate.sparse_b200.csr import csr_array


@pytest.fixture(autouse=True)
def _host_only(monkeypatch):
    """Operands stay on the host, also where a GPU is visible: every call that passes its checks then stops at the
    missing device."""
    from legate.sparse_b200.runtime import Runtime

    monkeypatch.setattr(Runtime, "has_cuda", property(lambda self: False))


def _parts(M):
    """(indptr, indices, data, shape) of a scipy or library CSR matrix, numpy arrays"""
    if isinstance(M, csr_array):
        M = M.to_scipy_sparse_csr()
    return np.asarray(M.indptr), np.asarray(M.indices), np.asarray(M.data), tuple(M.shape)


def kron_oracle(a, b):
    """(indptr int64, indices int64, data) of kron(A, B) for A, B given as `_parts`"""
    ap, ai, av, (am, an) = a
    bp, bi, bv, (bm, bn) = b
    ap, ai, bp, bi = (np.asarray(x, dtype=np.int64) for x in (ap, ai, bp, bi))
    la, lb = np.diff(ap), np.diff(bp)
    t = np.arange(am * bm, dtype=np.int64)
    i, r = t // max(bm, 1), t % max(bm, 1)
    lens = la[i] * lb[r] if t.size else np.zeros(0, dtype=np.int64)
    ptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    te = np.repeat(t, lens)
    off = np.arange(ptr[-1], dtype=np.int64) - ptr[te]
    ie, re = te // max(bm, 1), te % max(bm, 1)
    ea = ap[ie] + off // np.maximum(lb[re], 1)
    eb = bp[re] + off % np.maximum(lb[re], 1)
    return ptr, ai[ea] * bn + bi[eb], av[ea] * bv[eb]


def bmat_oracle(placed, shape):
    """(indptr int64, indices int64, data) of the blocks placed = [(row offset, column offset, parts)], listed by block
    row and left to right: each output row concatenates the rows of its blocks in that order"""
    rows, cols, vals = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)], []
    for roff, coff, (p, i, v, _) in placed:
        p = np.asarray(p, dtype=np.int64)
        rows.append(np.repeat(np.arange(p.size - 1, dtype=np.int64), np.diff(p)) + roff)
        cols.append(np.asarray(i, dtype=np.int64) + coff)
        vals.append(np.asarray(v))
    R, C = np.concatenate(rows), np.concatenate(cols)
    V = np.concatenate(vals) if vals else np.zeros(0)
    order = np.argsort(R, kind="stable")
    ptr = np.r_[0, np.cumsum(np.bincount(R, minlength=shape[0]))].astype(np.int64)
    return ptr, C[order], V[order]


def grid_placed(grid):
    """`bmat_oracle`'s placement of a grid of scipy matrices / None (every block row and column has a non-None block)"""
    heights = [next(b.shape[0] for b in row if b is not None) for row in grid]
    widths = [next(row[j].shape[1] for row in grid if row[j] is not None) for j in range(len(grid[0]))]
    ro, co = np.r_[0, np.cumsum(heights)], np.r_[0, np.cumsum(widths)]
    placed = [(int(ro[i]), int(co[j]), _parts(b)) for i, row in enumerate(grid) for j, b in enumerate(row)
              if b is not None]
    return placed, (int(ro[-1]), int(co[-1]))


def assert_same_csr(ours, S):
    """structure and data bytes of (indptr, indices, data) equal to the scipy CSR matrix S"""
    p, i, v = ours
    assert np.array_equal(np.asarray(p, np.int64), np.asarray(S.indptr, np.int64))
    assert np.array_equal(np.asarray(i, np.int64), np.asarray(S.indices, np.int64))
    assert np.asarray(v).dtype == S.data.dtype and np.asarray(v).tobytes() == S.data.tobytes()


def dense_of(parts):
    p, i, v, shape = parts if len(parts) == 4 else (*parts, None)
    return sp.csr_array((v, i, p), shape=shape).toarray()


def _mtx(name):
    return sp.csr_array(scipy.io.mmread(mtx_path(name))).astype(np.float64)


@pytest.mark.parametrize("name", MTX_FILES)
def test_kron_oracle_matches_scipy_on_fixtures(name):
    A = _mtx(name)
    A.sum_duplicates()
    B = sp.csr_array(np.roll(A.toarray(), 1))   # the reference's test_kron operand
    S = sp.kron(A, B, format="csr")
    assert_same_csr(kron_oracle(_parts(A), _parts(B)), S)
    small = sp.csr_array(np.array([[1.5, 0, -2], [0, 0, 0], [4, 0.25, 0]]))
    assert_same_csr(kron_oracle(_parts(small), _parts(A)), sp.kron(small, A, format="csr"))


@pytest.mark.parametrize("name", MTX_FILES)
def test_bmat_oracle_matches_scipy_on_fixtures(name):
    A = _mtx(name)
    A.sum_duplicates()
    B = sp.csr_array(np.roll(A.toarray(), 1, axis=1))
    grid = [[A, None, B], [None, B, A]]
    placed, shape = grid_placed(grid)
    assert_same_csr(bmat_oracle(placed, shape), sp.bmat(grid, format="csr"))
    placed, shape = grid_placed([[A, B]])
    assert_same_csr(bmat_oracle(placed, shape), sp.hstack([A, B], format="csr"))
    placed, shape = grid_placed([[A], [B]])
    assert_same_csr(bmat_oracle(placed, shape), sp.vstack([A, B], format="csr"))
    placed = [(0, 0, _parts(A)), (A.shape[0], A.shape[1], _parts(B))]
    shape = (A.shape[0] + B.shape[0], A.shape[1] + B.shape[1])
    assert_same_csr(bmat_oracle(placed, shape), sp.block_diag([A, B], format="csr"))


def _awkward():
    """CSR matrices scipy would not produce: unsorted rows, repeated columns, explicit zeros, empty rows, no entries"""
    unsorted = ((np.array([0, 3, 3, 5]), np.array([2, 0, 1, 1, 0]), np.array([1.0, 2.0, 3.0, 4.0, 5.0])), (3, 3))
    dups = ((np.array([0, 2, 2, 4]), np.array([1, 1, 0, 0]), np.array([0.5, 0.25, 0.0, -1.0])), (3, 2))
    zeros = ((np.array([0, 0, 2]), np.array([3, 0]), np.array([0.0, -0.0])), (2, 4))
    empty = ((np.zeros(3, np.int64), np.zeros(0, np.int64), np.zeros(0)), (2, 5))
    nothing = ((np.zeros(1, np.int64), np.zeros(0, np.int64), np.zeros(0)), (0, 0))
    return [(p, i, v, shape) for (p, i, v), shape in (unsorted, dups, zeros, empty, nothing)]


def test_oracles_match_scipy_values_on_awkward_inputs():
    mats = _awkward()
    for a in mats:
        for b in mats:
            Sa, Sb = (sp.csr_array((x[2], x[1], x[0]), shape=x[3]) for x in (a, b))
            p, i, v = kron_oracle(a, b)
            shape = (a[3][0] * b[3][0], a[3][1] * b[3][1])
            assert np.array_equal(dense_of((p, i, v, shape)), sp.kron(Sa, Sb).toarray())
            assert p[-1] == Sa.nnz * Sb.nnz    # nothing pruned
    a, b = mats[0], mats[1]
    Sa, Sb = (sp.csr_array((x[2], x[1], x[0]), shape=x[3]) for x in (a, b))
    d = (np.array([0, 2, 3]), np.array([1, 1, 0]), np.array([0.0, 3.0, -2.0]), (2, 2))
    placed = [(0, 0, a), (0, 3, b), (3, 3, d)]
    shape = (5, 5)
    p, i, v = bmat_oracle(placed, shape)
    ref = sp.bmat([[Sa, Sb], [None, sp.csr_array((d[2], d[1], d[0]), shape=d[3])]]).toarray()
    assert np.array_equal(dense_of((p, i, v, shape)), ref)
    # the row of a block keeps its stored order: unsorted columns stay unsorted, duplicates stay apart
    assert list(i[p[0]:p[1]]) == [2, 0, 1, 4, 4]


def _pair(shape, kind, seed):
    """(scipy operand, library operand) of one shape; kind "csr" or "coo" (scipy's stacking paths differ by kind)"""
    S = sp.random(shape[0], shape[1], density=0.5, format="csr", random_state=seed)
    if kind == "coo":
        return S.tocoo(), sparse.coo_array(S.tocoo())
    return S, csr_array(S)


def _grid(spec, kind):
    s, o = [], []
    for i, row in enumerate(spec):
        sr, orow = [], []
        for j, shape in enumerate(row):
            a, b = (None, None) if shape is None else _pair(shape, kind, 7 * i + j)
            sr.append(a)
            orow.append(b)
        s.append(sr)
        o.append(orow)
    return s, o


BMAT_SPECS = [
    [[(2, 3), (3, 3)]],                                  # heights differ in a block row
    [[(2, 3), (2, 4)], [(2, 2), (2, 5)]],                # column widths differ, row widths agree
    [[(2, 3), None], [None, (3, 3)]],
    [[(2, 3), None], [(3, 3), None]],
    [[(2, 3), (3, 1)], [None, None]],
    [[(0, 3), (3, 1)]],                                  # a block with no rows before a taller one
    [[(3, 3), (0, 1)]],                                  # ... and after it
    [[(3, 0), (3, 2)], [(1, 4), (1, 2)]],                # a block with no columns
    [[(2, 2)], [(2, 3)]],                                # widths differ in a block column
    [[(2, 2), None], [None, None]],                      # a block row and a block column of None
]


def _raises(f):
    try:
        f()
    except ValueError:
        return "ValueError"
    except Exception as e:  # noqa: BLE001 -- any other outcome counts as "no ValueError"
        return type(e).__name__
    return None


@pytest.mark.parametrize("kind", ["csr", "coo"])
@pytest.mark.parametrize("spec", BMAT_SPECS, ids=range(len(BMAT_SPECS)))
def test_bmat_raises_value_error_where_scipy_does(spec, kind):
    S, O = _grid(spec, kind)
    for fmt in (None, "csr", "coo"):
        ref = _raises(lambda: sp.bmat(S, format=fmt))
        got = _raises(lambda: sparse.bmat(O, format=fmt))
        assert (ref == "ValueError") == (got == "ValueError"), (fmt, ref, got)
        if got != "ValueError":
            assert got == "RuntimeError"        # past the checks: stops at the missing device, no CPU fallback


def test_stacking_raises_value_error_where_scipy_does():
    (a, A), (b, B), (c, C) = _pair((2, 3), "csr", 1), _pair((3, 3), "csr", 2), _pair((2, 4), "csr", 3)
    cases = [
        (lambda: sp.hstack([a, b]), lambda: sparse.hstack([A, B])),
        (lambda: sp.hstack([a, c]), lambda: sparse.hstack([A, C])),
        (lambda: sp.vstack([a, b]), lambda: sparse.vstack([A, B])),
        (lambda: sp.vstack([a, c]), lambda: sparse.vstack([A, C])),
        (lambda: sp.vstack([a.tocoo(), c]), lambda: sparse.vstack([A.tocoo(), C])),
        (lambda: sp.vstack([]), lambda: sparse.vstack([])),
        (lambda: sp.hstack([]), lambda: sparse.hstack([])),
        (lambda: sp.bmat([a, b]), lambda: sparse.bmat([A, B])),                      # not 2-D
        (lambda: sp.bmat([[a, b], [a]]), lambda: sparse.bmat([[A, B], [A]])),        # ragged
        (lambda: sp.bmat([[[a]]]), lambda: sparse.bmat([[[A]]])),                    # 3-D
        (lambda: sp.kronsum(a, b), lambda: sparse.kronsum(A, B)),                    # A not square
        (lambda: sp.kronsum(b, a), lambda: sparse.kronsum(B, A)),                    # B not square
        (lambda: sp.kronsum(b, b), lambda: sparse.kronsum(B, B)),
        (lambda: sp.kron(a, c), lambda: sparse.kron(A, C)),
        (lambda: sp.block_diag([a, b, 2.5]), lambda: sparse.block_diag([A, B, 2.5])),
        (lambda: sp.block_diag([a, np.ones(3)]), lambda: sparse.block_diag([A, np.ones(3)])),
        (lambda: sp.block_diag([a, [[1, 0], [0, 2]]]), lambda: sparse.block_diag([A, [[1, 0], [0, 2]]])),
        (lambda: sp.block_diag([]), lambda: sparse.block_diag([])),
    ]
    for k, (ref, ours) in enumerate(cases):
        r, g = _raises(ref), _raises(ours)
        assert (r == "ValueError") == (g == "ValueError"), (k, r, g)


def test_results_beyond_int64_raise_value_error_before_allocating():
    import torch

    z = torch.zeros(2, dtype=torch.int32)
    huge = csr_array._from_parts(z, torch.zeros(0, dtype=torch.int32), torch.zeros(0), (2**40, 2**40))
    with pytest.raises(ValueError, match="does not fit in int64"):
        sparse.kron(huge, huge)
    with pytest.raises(ValueError, match="does not fit in int64"):
        sparse.kronsum(huge, huge)
    with pytest.raises(ValueError, match="does not fit in int64"):
        sparse.block_diag([huge] * 2**24)


def test_unsupported_formats_and_dtypes():
    (a, A) = _pair((3, 3), "csr", 4)
    for f in (lambda: sparse.kron(A, A, format="bsr"), lambda: sparse.bmat([[A]], format="csc"),
              lambda: sparse.block_diag([A], format="dia")):
        with pytest.raises(NotImplementedError):
            f()
    with pytest.raises(NotImplementedError, match="float32/float64"):
        sparse.kron(A.astype(np.complex128), A)
    with pytest.raises(NotImplementedError, match="4-, 8- or 16-byte"):
        sparse.hstack([A.astype(np.int16), A.astype(np.int16)])


def test_alias_package_exports_the_assembly_functions():
    import sparse as alias

    for name in ("kron", "kronsum", "bmat", "hstack", "vstack", "block_diag"):
        assert getattr(alias, name) is getattr(sparse, name)


# ---- the CSR operand contract of b2s_csr_kron and b2s_csr_blocks ------------------------------------------------------
def _entries():
    """name -> (call(it, pt, m, n, nnz), takes ncols, takes nnz), as test_abi_csr_checks_host._entries: every argument
    other than the broken operand's is valid"""
    from legate.sparse_b200 import _lib

    L = _lib.lib
    buf = (ctypes.c_int64 * 2048)()
    base = ctypes.addressof(buf)

    def p(i):
        return base + 128 * i

    F64, I32 = _lib.F64, _lib.I32

    def blocks(it, pt, m, n, nnz):
        d = np.zeros(1, dtype=_lib.BLOCK_DESC)
        d["indptr"], d["indices"], d["vals"] = p(0), p(1), p(2)
        d["it"], d["pt"], d["nrows"], d["ncols"], d["nnz"] = it, pt, m, n, nnz
        return L.b2s_csr_blocks(8, I32, 4, 4, 4, 1, d.ctypes.data, p(3), p(4), p(5), p(6), None)

    return {
        "b2s_csr_kron(A)": (lambda it, pt, m, n, nnz: L.b2s_csr_kron(
            F64, I32, it, pt, m, n, nnz, p(0), p(1), p(2), I32, I32, 4, 4, 4, p(3), p(4), p(5), p(6), p(7), p(8),
            None), True, True),
        "b2s_csr_kron(B)": (lambda it, pt, m, n, nnz: L.b2s_csr_kron(
            F64, I32, I32, I32, 4, 4, 4, p(0), p(1), p(2), it, pt, m, n, nnz, p(3), p(4), p(5), p(6), p(7), p(8),
            None), True, True),
        "b2s_csr_blocks": (blocks, True, True),
    }


def _failures():
    from legate.sparse_b200 import _lib
    from test_abi_csr_checks_host import _cases

    out = []
    for name, (call, takes_ncols, takes_nnz) in _entries().items():
        for kw, msg in _cases(takes_ncols, takes_nnz):
            rc = call(**kw)
            err = _lib.last_error()
            if rc != _lib.EINVAL or msg not in err:
                out.append(f"{name}({kw}): rc {rc}, {err!r}, expected EINVAL and {msg!r}")
    return out


def test_assembly_entry_points_check_the_csr_operand_alike():
    script = (
        "import sys\n"
        f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
        "import test_construct_host as t\n"
        "print('\\n'.join(t._failures()))\n"
    )
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.strip() == "", r.stdout
