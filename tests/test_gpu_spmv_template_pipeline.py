"""Edges of the row-template kernel's software pipeline.  Each warp walks the chunks c, c + S, c + 2S, ... (S = warps in
the grid) and keeps the ids and x gathers of the next chunks in flight while it sums the current one, so these sizes
put the pipeline's prologue, its last steps and its loads past the last chunk to work: fewer chunks than one resident
wave of warps (most warps have none), exactly one wave (one chunk each), one wave plus one chunk (one warp has two),
nrows one short of, equal to and one past a multiple of 32 R, the longer rows of a 3-D 7-point stencil, and the fused
dot.  y must be bit-for-bit the y of the same plan with the CSR arrays streamed; the dot is compared to a tolerance."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import _lib, _ops


def _same(a, b):
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    return a.shape == b.shape and bool(((a.view(it) == b.view(it)) | (torch.isnan(a) & torch.isnan(b))).all())


def _wave_chunks(ctas):
    """Chunks one resident wave of 256-thread CTAs takes at `ctas` CTAs per SM (8 warps each)."""
    return torch.cuda.get_device_properties(0).multi_processor_count * ctas * 8


def _sizes(rows_per_lane):
    """nrows around the chunk boundaries and the wave boundaries of every launch bound the kernel is built with (8, 6, 5
    or 4 CTAs per SM).  The smallest matrices are two chunks long: fp32 plans of a single chunk are not templated."""
    c = 32 * rows_per_lane
    out = {2 * c - 1, 2 * c, 2 * c + 1, 3 * c + 1}
    for ctas in (8, 6, 5, 4):
        w = _wave_chunks(ctas)
        out |= {c * (w // 2), c * w - 1, c * w, c * w + 1, c * (w + 1), c * (2 * w) + 1}
    return sorted(out)


def _check(A, rows_per_lane=1):
    dt = A.data.dtype
    plan = _ops.spmv_plan(A.indptr, A.indices, A.shape, A.nnz, np.dtype(str(dt).split(".")[1]))
    plan = _ops.spmv_plan_code(plan, A.indptr, A.indices, A.data)
    plan = _ops.spmv_plan_templates(plan, A.indptr, A.indices, A.data)
    assert plan.templated, plan.kernel_name
    n = A.shape[0]
    g = torch.Generator("cuda").manual_seed(n)
    x = torch.rand(A.shape[1], dtype=dt, device="cuda", generator=g) - 0.5
    w = torch.rand(n, dtype=dt, device="cuda", generator=g) - 0.5

    def run():
        y = _ops.spmv(A.indptr, A.indices, A.data, x, torch.full((n,), 7.0, dtype=dt, device="cuda"), A.shape, plan=plan)
        yd = torch.full((n,), 7.0, dtype=dt, device="cuda")
        out = torch.zeros(1, dtype=dt, device="cuda")
        _ops.spmv_dot(A.indptr, A.indices, A.data, x, yd, w, out, A.shape, plan)
        return y, yd, out

    L = _lib.lib
    try:
        _lib.check(L.b2s_spmv_set_template_config(rows_per_lane, 256, 0), "b2s_spmv_set_template_config")
        y, yd, out = run()
    finally:
        L.b2s_spmv_set_template_config(0, 0, 0)
    plan.set_packed(0)
    y0, _, out0 = run()
    assert _same(y, y0) and _same(yd, y0), (n, rows_per_lane)
    tol = 1e-4 if dt == torch.float32 else 1e-11
    assert torch.allclose(out, out0, rtol=tol, atol=tol * float(y0.abs().sum())), (n, float(out), float(out0))


def _band(n, dtype):
    """A 1-D 3-point operator with every fifth sub-diagonal entry left out: its row lengths vary inside every tile, so
    the plan takes the one-lane-per-row kernel that templates stand in for at every size (a plain tridiagonal matrix's
    tiles can be uniform, and a plan with enough uniform tiles has no templates)."""
    sub = np.full(n - 1, -1.0)
    sub[::5] = 0.0
    S = sp.csr_array(sp.diags([sub, np.full(n, 2.0), np.full(n - 1, -1.0)], [-1, 0, 1], format="csr", dtype=dtype))
    S.eliminate_zeros()
    S.sort_indices()
    return sparse.csr_array(S)


@pytest.mark.gpu
@pytest.mark.parametrize("rows_per_lane", [1, 2])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_chunk_and_wave_edges(dtype, rows_per_lane):
    for n in _sizes(rows_per_lane):
        _check(_band(n, dtype), rows_per_lane)


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
def test_long_rows_at_wave_edges(dtype):
    """Rows of up to 7 entries run the kTplLen instantiation (6 CTAs per SM): nrows = 16 nx, so the last chunk is
    ragged whenever nx is odd."""
    w = _wave_chunks(6)
    for nx in (3, w // 2 + 1, 2 * w - 1, 2 * w, 2 * w + 1, 4 * w + 3):
        A = _stencil7(nx, 4, 4, dtype)
        assert A.shape[0] == 16 * nx
        _check(A)
