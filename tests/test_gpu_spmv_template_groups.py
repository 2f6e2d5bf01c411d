"""Group codes of the row-template kernel.  The template buffer holds one code per 32-row group next to the per-row
ids: the template every row of the group shares, or 0xFF when the group mixes templates, and the kernel reads the
per-row ids of mixed groups only.  These cases put grid-row boundaries at every position within a group (5-point
Laplacians with n1 in {31, 32, 33, 64, 3162}), put the last group's end one short of, at and one past multiples of 32
and 64, make every group mixed, leave a single template, take the longer-row instantiation (3-D 7-point stencil),
and run each at R = 1 and 2 and 128 and 256 threads.  y must be bit-for-bit the y of the same plan with the CSR arrays
streamed; the fused dot is compared to a tolerance.  The codes read back from the buffer must equal a numpy
restatement from the ids."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import _lib, _ops, gallery

SHAPES = [(1, 256), (2, 256), (1, 128), (2, 128)]


def _same(a, b):
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    return a.shape == b.shape and bool(((a.view(it) == b.view(it)) | (torch.isnan(a) & torch.isnan(b))).all())


def _codes_from_ids(ids):
    """numpy restatement: per group of 32 rows (the last one ragged) its rows' common id, else 0xFF."""
    n = ids.shape[0]
    ng = (n + 31) // 32
    pad = np.concatenate([ids, np.repeat(ids[-1:], ng * 32 - n)]).reshape(ng, 32)
    return np.where((pad == pad[:, :1]).all(axis=1), pad[:, 0], 0xFF).astype(np.uint8)


def _plan(A):
    dt = np.dtype(str(A.data.dtype).split(".")[1])
    plan = _ops.spmv_plan(A.indptr, A.indices, A.shape, A.nnz, dt)
    plan = _ops.spmv_plan_code(plan, A.indptr, A.indices, A.data)
    if plan.tma and not plan.short_rows:
        # a matrix whose tiles are mostly uniform runs the uniform-row kernel and gets no templates; the one-lane-per-row
        # kernel, which the templates reproduce bit for bit, runs it as well
        plan.set_flavor(2)
    plan = _ops.spmv_plan_templates(plan, A.indptr, A.indices, A.data)
    assert plan.templated, plan.kernel_name
    return plan


def _check(A, expect_mixed=None):
    """Codes against the ids, then y and the fused dot at every kernel shape against the streamed CSR arrays."""
    n = A.shape[0]
    dt = A.data.dtype
    plan = _plan(A)
    ids, codes = plan.template_sections(n)
    ids, codes = ids.cpu().numpy(), codes.cpu().numpy()
    assert codes.shape == ((n + 31) // 32,)
    assert ids.max() < plan.ntemplates
    want = _codes_from_ids(ids)
    assert np.array_equal(codes, want), (n, np.flatnonzero(codes != want)[:8])
    if expect_mixed is not None:
        assert np.array_equal(np.flatnonzero(codes == 0xFF), expect_mixed), n
    g = torch.Generator("cuda").manual_seed(n)
    x = torch.rand(A.shape[1], dtype=dt, device="cuda", generator=g) - 0.5
    w = torch.rand(n, dtype=dt, device="cuda", generator=g) - 0.5

    def run():
        y = _ops.spmv(A.indptr, A.indices, A.data, x, torch.full((n,), 7.0, dtype=dt, device="cuda"), A.shape, plan=plan)
        yd = torch.full((n,), 7.0, dtype=dt, device="cuda")
        out = torch.zeros(1, dtype=dt, device="cuda")
        _ops.spmv_dot(A.indptr, A.indices, A.data, x, yd, w, out, A.shape, plan)
        return y, yd, out

    plan.set_packed(0)
    y0, _, out0 = run()
    plan.set_packed(3)
    tol = 1e-4 if dt == torch.float32 else 1e-11
    L = _lib.lib
    for rows, threads in SHAPES:
        try:
            _lib.check(L.b2s_spmv_set_template_config(rows, threads, 0), "b2s_spmv_set_template_config")
            y, yd, out = run()
        finally:
            L.b2s_spmv_set_template_config(0, 0, 0)
        assert _same(y, y0) and _same(yd, y0), (n, rows, threads)
        assert torch.allclose(out, out0, rtol=tol, atol=tol * float(y0.abs().sum())), (n, float(out), float(out0))
    return codes


def _band(n, dtype, period):
    """A 1-D 3-point operator with every `period`-th sub-diagonal entry left out, so the rows just below those holes
    take a different template from their neighbours."""
    sub = np.full(n - 1, -1.0)
    sub[::period] = 0.0
    S = sp.csr_array(sp.diags([sub, np.full(n, 2.0), np.full(n - 1, -1.0)], [-1, 0, 1], format="csr", dtype=dtype))
    S.eliminate_zeros()
    S.sort_indices()
    return sparse.csr_array(S)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n1,n2", [(31, 45), (32, 45), (33, 45), (64, 45), (3162, 3162)])
def test_laplacian_grid_rows_at_every_group_position(n1, n2, dtype):
    codes = _check(gallery.laplacian_5pt(n1, n2, dtype))
    if n1 == 3162:
        # the benchmark's grid: 3,360 of its 312,446 groups hold a grid-row boundary or the edges of the first or last
        # grid row
        assert codes.shape[0] == 312446 and int((codes == 0xFF).sum()) == 3360


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_nrows_around_multiples_of_32_and_64(dtype):
    for base in (64, 128, 32 * 1001, 64 * 1001):
        for n in (base - 1, base, base + 1):
            _check(_band(n, dtype, 45))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_every_group_mixed(dtype):
    """Diagonal entries alternate between two values, so every group of two rows or more is mixed (n = 97 and 20001
    end in a one-row group)."""
    for n in (95, 96, 97, 20001):
        d = np.where(np.arange(n) % 2 == 0, 4.0, 5.0)
        S = sp.csr_array(sp.diags([np.full(n - 1, -1.0), d, np.full(n - 1, -1.0)], [-1, 0, 1], format="csr",
                                  dtype=dtype))
        S.sort_indices()
        _check(sparse.csr_array(S), expect_mixed=np.arange((n + 30) // 32))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_single_template(dtype):
    """A constant diagonal: one template, no mixed group."""
    for n in (63, 64, 65, 10001):
        S = sp.csr_array(sp.diags([np.full(n, 3.0)], [0], format="csr", dtype=dtype))
        codes = _check(sparse.csr_array(S), expect_mixed=np.array([], dtype=np.int64))
        assert (codes == 0).all()


def _stencil7(nx, ny, nz, dtype):
    N = nx * ny * nz
    i = np.arange(N)
    ix, iy, iz = i % nx, (i // nx) % ny, i // (nx * ny)
    rows, cols = [i], [i]
    vals = [np.full(N, 6.0)]
    for off, ok in ((1, ix < nx - 1), (-1, ix > 0), (nx, iy < ny - 1), (-nx, iy > 0), (nx * ny, iz < nz - 1),
                    (-nx * ny, iz > 0)):
        rows.append(i[ok]), cols.append(i[ok] + off), vals.append(np.full(ok.sum(), -1.0))
    S = sp.csr_array((np.concatenate(vals).astype(dtype), (np.concatenate(rows), np.concatenate(cols))), shape=(N, N))
    S.sort_indices()
    return sparse.csr_array(S)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_stencil7_longer_rows(dtype):
    """Rows of up to 7 entries run the kTplLen instantiation; nx = 40 leaves uniform groups inside each x-line."""
    for nx, ny, nz in ((40, 5, 7), (33, 9, 11), (64, 16, 16)):
        _check(_stencil7(nx, ny, nz, dtype))
