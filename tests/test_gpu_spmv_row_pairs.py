"""Packed tiles of rows with at most 5 entries and more rows than the kernel's 128 consumer lanes take two rows per lane
in one round of gathers.  The rows are summed exactly as one lane per row sums them, so every product must be
bit-for-bit the one the CSR-streaming kernel computes on the same plan -- y, y += A x, the y of the fused dot and tile
ranges -- whatever mix of row lengths (4-entry tiles, 5-entry tiles, empty rows) a tile holds.  The dot itself is a grid
reduction whose grouping follows the launch's grid, which differs between kernels of different shared-memory size, so
across kernels it is compared to a tolerance."""
import numpy as np
import pytest
import torch

from legate.sparse_b200 import _ops, gallery


def _same(a, b):
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    return a.shape == b.shape and torch.equal(a.view(it), b.view(it))


def _x(n, dt, seed=3):
    return torch.rand(n, dtype=dt, device="cuda", generator=torch.Generator("cuda").manual_seed(seed)) - 0.5


def _entry_points(d_ptr, d_idx, d_val, d_x, shape, plan):
    nrows = shape[0]
    dev, dt = d_val.device, d_val.dtype
    y = _ops.spmv(d_ptr, d_idx, d_val, d_x, torch.full((nrows,), 7.0, dtype=dt, device=dev), shape, plan=plan)
    y0 = torch.from_numpy(np.random.default_rng(5).standard_normal(nrows)).to(dev, dt)
    ya = _ops.spmv_add(d_ptr, d_idx, d_val, d_x, y0.clone(), shape, plan)
    w = torch.from_numpy(np.random.default_rng(6).standard_normal(nrows)).to(dev, dt)
    yd = torch.empty(nrows, dtype=dt, device=dev)
    out = torch.zeros(1, dtype=dt, device=dev)
    _ops.spmv_dot(d_ptr, d_idx, d_val, d_x, yd, w, out, shape, plan)
    nt = plan.tiles
    cuts = sorted({0, nt // 3, nt // 2, nt})
    yt = torch.full((nrows,), 7.0, dtype=dt, device=dev)
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        _ops.spmv_tiles(d_ptr, d_idx, d_val, d_x, yt, shape, plan, lo, hi)
    return [y, ya, torch.cat([yd, out]), yt]


def _check(d_ptr, d_idx, d_val, shape):
    dt = np.dtype(str(d_val.dtype).split(".")[1])
    plan = _ops.spmv_plan(d_ptr, d_idx, shape, int(d_val.shape[0]), dt)
    plan = _ops.spmv_plan_code(plan, d_ptr, d_idx, d_val)
    assert plan.packed and plan.short_rows, plan.kernel_name
    x = _x(shape[1], d_val.dtype)
    plan.set_packed(0)
    ref = _entry_points(d_ptr, d_idx, d_val, x, shape, plan)
    for mode in ([2, 1] if plan.coded else [1]):
        plan.set_packed(mode)
        got = _entry_points(d_ptr, d_idx, d_val, x, shape, plan)
        n = shape[0]
        for i, (g, r) in enumerate(zip(got, ref)):
            assert _same(g[:n], r[:n]), (mode, i, plan.kernel_name)
        tol = 1e-5 if d_val.dtype == torch.float32 else 1e-12
        assert torch.allclose(got[2][n:], ref[2][n:], rtol=tol, atol=0), (mode, plan.kernel_name)


def _rows(lens, rng, nvals=None, dtype=np.float64):
    """CSR with the given row lengths, columns in a short band after the row, sorted within each row."""
    nrows = len(lens)
    indptr = np.zeros(nrows + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    r = np.repeat(np.arange(nrows), lens)
    pos = np.arange(indptr[-1]) - indptr[r]
    cols = np.minimum(r + 3 * pos, nrows - 1)
    vals = (rng.integers(0, nvals, r.shape[0]) - 1.5 if nvals else rng.standard_normal(r.shape[0])).astype(dtype)
    return (torch.from_numpy(indptr).cuda(), torch.from_numpy(cols.astype(np.int32)).cuda(),
            torch.from_numpy(vals).cuda(), (nrows, nrows))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [300, 3162])
def test_laplacian_row_pairs_match_csr(n, dtype):
    A = gallery.laplacian_5pt(n, n, dtype)
    _check(A.indptr, A.indices, A.data, A.shape)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("maxlen", [4, 5])
@pytest.mark.parametrize("coded", [True, False])
def test_mixed_short_rows_match_csr(maxlen, coded, dtype):
    """Rows of maxlen - 1 or maxlen entries with scattered and runs of empty rows, coded and streamed values (fp64 tiles
    then hold 170-260 rows: two per lane)."""
    rng = np.random.default_rng(maxlen)
    lens = rng.integers(maxlen - 1, maxlen + 1, 200000)
    lens[rng.integers(0, 200000, 2000)] = 0
    lens[1000:1500] = 0
    _check(*_rows(lens, rng, nvals=3 if coded else None, dtype=dtype))


@pytest.mark.gpu
def test_signed_zero_sums_keep_their_sign():
    """Rows whose products are all -0.0: the padded zero terms act exactly as in the one-row-per-lane walk."""
    rng = np.random.default_rng(9)
    lens = np.full(100000, 4)
    lens[::7] = 5
    d_ptr, d_idx, d_val, shape = _rows(lens, rng, nvals=2)
    d_val = torch.where(d_val > 0, torch.full_like(d_val, -0.0), torch.full_like(d_val, 2.0))
    _check(d_ptr, d_idx, d_val, shape)
