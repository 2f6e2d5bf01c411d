"""Coded values in the packed SpMV structure (b2s_spmv_plan_pack_coded): when the values take at most 16 distinct bit
patterns, the spare high bits of the uint16 column words carry each value's index in a dictionary and the kernel
streams no values.  The same values enter the same FMAs in the same order, so every product must be bit-for-bit the one
the CSR-streaming kernel computes -- through every single-GPU entry point of the short-row kernel -- and a plan must
never outlive the values it coded."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import _lib, _ops, gallery


def _same(a, b):
    """Bit-for-bit equality (NaN == NaN when the bits agree)."""
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    return a.shape == b.shape and torch.equal(a.view(it), b.view(it))


def _modes(run, plan):
    """run() with coded values (mode 2), then with the CSR arrays (mode 0); the plan is left coded."""
    plan.set_packed(2)
    assert plan.packed and plan.coded, plan.kernel_name
    a = run()
    plan.set_packed(0)
    assert not plan.packed and not plan.coded
    b = run()
    plan.set_packed(2)
    return a, b


def _check_entry_points(d_ptr, d_idx, d_val, d_x, shape, plan):
    """Coded vs CSR arrays through b2s_spmv_csr, _add, _dot and _tiles: bit-for-bit equal.  Returns the coded y."""
    nrows = shape[0]
    dev = d_val.device
    dt = d_val.dtype

    def plain():
        y = torch.full((nrows,), 7.0, dtype=dt, device=dev)
        return _ops.spmv(d_ptr, d_idx, d_val, d_x, y, shape, plan=plan)

    yc, yu = _modes(plain, plan)
    assert _same(yc, yu)

    y0 = torch.from_numpy(np.random.default_rng(5).standard_normal(nrows)).to(dev, dt)

    def add():
        return _ops.spmv_add(d_ptr, d_idx, d_val, d_x, y0.clone(), shape, plan)

    ac, au = _modes(add, plan)
    assert _same(ac, au)

    w = torch.from_numpy(np.random.default_rng(6).standard_normal(nrows)).to(dev, dt)

    def dot():
        y = torch.empty(nrows, dtype=dt, device=dev)
        out = torch.zeros(1, dtype=dt, device=dev)
        _ops.spmv_dot(d_ptr, d_idx, d_val, d_x, y, w, out, shape, plan)
        return torch.cat([y, out])

    dc, du = _modes(dot, plan)
    assert _same(dc, du) and _same(dc[:nrows], yc)

    nt = plan.tiles
    cuts = sorted({0, nt // 3, nt // 2, nt})

    def tiles():
        y = torch.full((nrows,), 7.0, dtype=dt, device=dev)
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            _ops.spmv_tiles(d_ptr, d_idx, d_val, d_x, y, shape, plan, lo, hi)
        return y

    tc, tu = _modes(tiles, plan)
    assert _same(tc, tu) and _same(tc, yc)
    return yc


def _coded_plan(d_ptr, d_idx, d_val, shape):
    plan = _ops.spmv_plan(d_ptr, d_idx, shape, int(d_val.shape[0]), np.dtype(str(d_val.dtype).split(".")[1]))
    return _ops.spmv_plan_code(plan, d_ptr, d_idx, d_val)


def _x(n, dt, seed=3):
    return torch.rand(n, dtype=dt, device="cuda", generator=torch.Generator("cuda").manual_seed(seed)) - 0.5


def _band5(nrows, values, rng):
    """5 entries per row on columns r-2..r+2 (clipped), values drawn from `values` (numpy, host)."""
    r = np.repeat(np.arange(nrows), 5)
    c = r + np.tile(np.arange(-2, 3), nrows)
    keep = (c >= 0) & (c < nrows)
    r, c = r[keep], c[keep]
    indptr = np.zeros(nrows + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=nrows), out=indptr[1:])
    vals = np.asarray(values)[rng.integers(0, len(values), c.shape[0])]
    vals[: len(values)] = values          # every value occurs
    return indptr, c.astype(np.int64), vals


def _tile_windows(plan, indptr, indices):
    """(first row, last row + 1, smallest column, largest column) of every non-empty tile of a plan."""
    e = plan.buf[: 4 * (plan.tiles + 1)].view(-1, 4).cpu().numpy().astype(np.int64)
    k = (e[:, 0] & 0xFFFFFFFF) | (e[:, 1] << 32)
    r = e[:, 2]
    out = []
    for t in range(plan.tiles):
        if r[t + 1] > r[t] and k[t + 1] > k[t]:
            cols = indices[k[t] : k[t + 1]]
            out.append((int(r[t]), int(r[t + 1]), int(cols.min()), int(cols.max())))
    return out


def _dev(indptr, indices, vals, idt=torch.int32):
    return (torch.from_numpy(indptr).to("cuda", idt), torch.from_numpy(indices).to("cuda", idt),
            torch.from_numpy(vals).cuda())


@pytest.mark.gpu
@pytest.mark.parametrize("n", [300, 3162])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_coded_laplacian(n, dtype):
    A = gallery.laplacian_5pt(n, n, dtype)
    plan = A._get_plan()
    assert plan.coded and plan.ndict == 2, plan.kernel_name
    assert "coded values (2 distinct)" in plan.kernel_name
    x = _x(A.shape[1], A.data.dtype)
    yc = _check_entry_points(A.indptr, A.indices, A.data, x, A.shape, plan)
    if n == 300:
        s = sp.csr_matrix((A.data.cpu().numpy(), A.indices.cpu().numpy(), A.indptr.cpu().numpy()), shape=A.shape)
        xs = x.cpu().numpy().astype(np.float64)
        tol = 1e-4 if dtype == np.float32 else 1e-10
        assert np.allclose(yc.cpu().numpy(), s @ xs, rtol=tol, atol=tol * abs(s).max())


@pytest.mark.gpu
@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
def test_coded_laplacian_a_ne_g_and_index_widths(idt):
    """a != g (3 distinct values, as the per-rank shards have), int32 and int64 indices / indptr."""
    A = gallery.laplacian_5pt(300, 200, np.float64, a=3.0, g=5.0)
    d_ptr, d_idx = A.indptr.to(idt), A.indices.to(idt)
    plan = _coded_plan(d_ptr, d_idx, A.data, A.shape)
    assert plan.coded and plan.ndict == 3, plan.kernel_name
    _check_entry_points(d_ptr, d_idx, A.data, _x(A.shape[1], torch.float64), A.shape, plan)


@pytest.mark.gpu
def test_coded_banded_single_value():
    """One distinct value: no code bits (vb = 0), every word decodes to dict[0]."""
    A = gallery.banded(100000, 11, np.float64)
    plan = A._get_plan()
    assert plan.coded and plan.ndict == 1, plan.kernel_name
    _check_entry_points(A.indptr, A.indices, A.data, _x(A.shape[1], torch.float64), A.shape, plan)


@pytest.mark.gpu
def test_coded_gmg_poisson_with_explicit_zeros():
    """GMG's poisson2d: 4 on the diagonal, -1 to the neighbours and explicit zeros at the grid-row ends."""
    n = 400
    N = n * n
    side = np.full(N - 1, -1.0)
    side[n - 1 :: n] = 0.0
    far = np.full(N - n, -1.0)
    # the triplets of the five diagonals by hand (scipy's conversions would drop the explicit zeros)
    rows, cols, vals = [], [], []
    for off, d in ((-n, far), (-1, side), (0, np.full(N, 4.0)), (1, side), (n, far)):
        r = np.arange(len(d)) + max(-off, 0)
        rows.append(r), cols.append(r + off), vals.append(d)
    rows, cols, vals = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
    order = np.lexsort((cols, rows))
    rows, cols, vals = rows[order], cols[order], vals[order]
    indptr = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=N), out=indptr[1:])
    assert (vals == 0.0).any()
    d_ptr, d_idx, d_val = _dev(indptr, cols.astype(np.int64), vals)
    plan = _coded_plan(d_ptr, d_idx, d_val, (N, N))
    assert plan.coded and plan.ndict == 3, plan.kernel_name
    _check_entry_points(d_ptr, d_idx, d_val, _x(N, torch.float64), (N, N), plan)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_16_values_are_coded_17_are_not(dtype):
    rng = np.random.default_rng(11)
    for nv in (16, 17):
        values = (np.arange(nv) * 0.37 - 2.0).astype(dtype)
        indptr, indices, vals = _band5(50000, values, rng)
        d_ptr, d_idx, d_val = _dev(indptr, indices, vals)
        plan = _coded_plan(d_ptr, d_idx, d_val, (50000, 50000))
        x = _x(50000, d_val.dtype)
        if nv == 16:
            assert plan.coded and plan.ndict == 16, plan.kernel_name
            _check_entry_points(d_ptr, d_idx, d_val, x, (50000, 50000), plan)
        else:
            assert plan.packed and not plan.coded, plan.kernel_name
            with pytest.raises(_lib.B200SparseError):
                plan.set_packed(2)
            y = lambda: _ops.spmv(d_ptr, d_idx, d_val, x, torch.empty_like(x), (50000, 50000), plan=plan)  # noqa: E731
            yp = y()
            plan.set_packed(0)
            assert _same(yp, y())


@pytest.mark.gpu
@pytest.mark.parametrize("nv,vb", [(2, 1), (16, 4)])
def test_window_limit_of_the_code_bits(nv, vb):
    """A tile whose columns span exactly 2^(16 - vb) - 1 keeps coded values; one more column and the plan stays
    packed with streamed values."""
    rng = np.random.default_rng(nv)
    nrows = 60000
    values = np.linspace(-1.0, 1.0, nv)
    indptr, indices, vals = _band5(nrows, values, rng)
    d_ptr, d_idx, d_val = _dev(indptr, indices, vals)
    probe = _ops.spmv_plan(d_ptr, d_idx, (nrows, nrows), int(indptr[-1]), np.float64)
    r0, r1, lo, hi = _tile_windows(probe, indptr, indices)[3]
    limit = 1 << (16 - vb)
    for span, coded in ((limit - 1, True), (limit, False)):
        idx = indices.copy()
        idx[indptr[r1] - 1] = lo + span        # the last entry of the tile's last row
        assert lo + span < nrows
        d_idx2 = torch.from_numpy(idx).to("cuda", torch.int32)
        plan = _coded_plan(d_ptr, d_idx2, d_val, (nrows, nrows))
        assert max(h - l for _, _, l, h in _tile_windows(plan, indptr, idx)) == span
        assert plan.packed and plan.coded == coded, (span, plan.kernel_name)
        x = _x(nrows, torch.float64)
        if coded:
            _check_entry_points(d_ptr, d_idx2, d_val, x, (nrows, nrows), plan)
        else:
            yp = _ops.spmv(d_ptr, d_idx2, d_val, x, torch.empty_like(x), (nrows, nrows), plan=plan)
            plan.set_packed(0)
            assert _same(yp, _ops.spmv(d_ptr, d_idx2, d_val, x, torch.empty_like(x), (nrows, nrows), plan=plan))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_signed_zeros_inf_and_nan_are_distinct_codes(dtype):
    values = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.5, -2.25], dtype=dtype)
    rng = np.random.default_rng(2)
    indptr, indices, vals = _band5(40000, values, rng)
    d_ptr, d_idx, d_val = _dev(indptr, indices, vals)
    plan = _coded_plan(d_ptr, d_idx, d_val, (40000, 40000))
    assert plan.coded and plan.ndict == 7, plan.kernel_name   # -0.0 and +0.0 apart
    yc = _check_entry_points(d_ptr, d_idx, d_val, _x(40000, d_val.dtype), (40000, 40000), plan)
    assert torch.isnan(yc).any() and torch.isinf(yc).any()


@pytest.mark.gpu
@pytest.mark.parametrize("new", ["same_count", "more_than_16", "fewer"])
def test_inplace_data_edit_rebuilds_the_coded_plan(new):
    A = gallery.laplacian_5pt(300, 300, np.float64)
    x = _x(A.shape[1], torch.float64)
    y0 = A @ x
    plan0 = A._get_plan()
    assert plan0.coded
    ptr_before = A.data.data_ptr()
    nnz = A.nnz
    if new == "same_count":
        A.data[:] = torch.where(A.data > 0, torch.full_like(A.data, 2.5), torch.full_like(A.data, -10.0))
    elif new == "more_than_16":
        A.data[:] = torch.arange(nnz, dtype=torch.float64, device="cuda") % 23 - 11.0
    else:
        A.data[:] = 1.0
    assert A.data.data_ptr() == ptr_before
    y1 = A @ x
    assert not _same(y0, y1)
    B = sparse.csr_array((A.data.clone(), A.indices.clone(), A.indptr.clone()), shape=A.shape)
    ref_plan = B._get_plan()
    ref_plan.set_packed(0)
    assert _same(y1, B @ x)
    plan1 = A._get_plan()
    assert plan1 is not plan0
    assert plan1.coded == (new != "more_than_16"), plan1.kernel_name


@pytest.mark.gpu
def test_launch_with_other_values_streams_them():
    """A coded plan launched with a different `data` tensor: the launch streams that tensor's values."""
    A = gallery.laplacian_5pt(300, 300, np.float64)
    plan = A._get_plan()
    assert plan.coded
    other = torch.rand(A.nnz, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(9))
    x = _x(A.shape[1], torch.float64)

    def run(vals):
        return _ops.spmv(A.indptr, A.indices, vals, x, torch.empty_like(x), A.shape, plan=plan)

    yo = run(other)
    plan.set_packed(0)
    assert _same(yo, run(other))
    plan.set_packed(2)
    assert not _same(run(other), run(A.data))


def test_coded_entry_points_reject_bad_handles():
    """Without a plan: packing with codes and switching modes report EINVAL instead of touching memory."""
    L = _lib.lib
    assert L.b2s_spmv_plan_pack_coded(None, None, None, None, None, None) == _lib.EINVAL
    assert L.b2s_spmv_plan_set_packed(None, 2) == _lib.EINVAL
    bogus = ctypes.create_string_buffer(256)
    assert L.b2s_spmv_plan_pack_coded(ctypes.addressof(bogus), None, None, None, None, None) == _lib.EINVAL
