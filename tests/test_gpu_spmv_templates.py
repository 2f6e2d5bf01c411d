"""Row templates (b2s_spmv_plan_templates): a matrix whose rows have at most 8 entries and at most 32 distinct
signatures (length, column - row of each entry, value bits) is held as one uint8 template id per row, and whole-matrix
products read only the ids, x and y.  Each row is summed exactly as the one-lane-per-row CSR kernel sums it, so y must
be bit-for-bit the y of the same plan with the CSR arrays streamed (mode 0) -- up to which of two NaNs survives when
both meet in one FMA, see _same; the fused dot is a grid reduction over a
different grid, so it is compared to a tolerance.  Matrices that do not qualify keep the coded / packed / CSR kernels."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from legate.sparse_b200 import _lib, _ops, gallery


def _same(a, b):
    """Bit-for-bit equality, signed zeros included.  NaNs only have to be NaN in both: where two different NaNs meet in
    one FMA (x holds a NaN and an earlier inf - inf made the sum the default NaN), which one propagates is left open by
    IEEE 754 and follows the operand order the compiler picked for that FMA, which differs between kernels."""
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    same_bits = a.view(it) == b.view(it)
    return a.shape == b.shape and bool((same_bits | (torch.isnan(a) & torch.isnan(b))).all())


def _x(n, dt, seed=3):
    return torch.rand(n, dtype=dt, device="cuda", generator=torch.Generator("cuda").manual_seed(seed)) - 0.5


def _signatures(indptr, indices, vals):
    """numpy restatement of the rule: the number of distinct (length, column - row..., value bits...) rows, or None
    when a row has more than 8 entries."""
    indptr, indices = np.asarray(indptr, dtype=np.int64), np.asarray(indices, dtype=np.int64)
    bits = np.asarray(vals).view(np.int32 if np.asarray(vals).dtype == np.float32 else np.int64).astype(np.int64)
    n = indptr.shape[0] - 1
    lens = np.diff(indptr)
    if n and lens.max() > 8:
        return None
    M = np.zeros((n, 17), dtype=np.int64)
    M[:, 0] = lens
    r = np.repeat(np.arange(n), lens)
    pos = np.arange(indptr[-1]) - indptr[r]
    M[r, 1 + pos] = indices - r
    M[r, 9 + pos] = bits
    return int(np.unique(M, axis=0).shape[0])


def _plan(d_ptr, d_idx, d_val, shape):
    dt = np.dtype(str(d_val.dtype).split(".")[1])
    plan = _ops.spmv_plan(d_ptr, d_idx, shape, int(d_val.shape[0]), dt)
    plan = _ops.spmv_plan_code(plan, d_ptr, d_idx, d_val)
    return _ops.spmv_plan_templates(plan, d_ptr, d_idx, d_val)


def _products(d_ptr, d_idx, d_val, x, shape, plan):
    nrows = shape[0]
    dev, dt = d_val.device, d_val.dtype
    y = _ops.spmv(d_ptr, d_idx, d_val, x, torch.full((nrows,), 7.0, dtype=dt, device=dev), shape, plan=plan)
    w = torch.from_numpy(np.random.default_rng(6).standard_normal(nrows)).to(dev, dt)
    yd = torch.full((nrows,), 7.0, dtype=dt, device=dev)
    out = torch.zeros(1, dtype=dt, device=dev)
    _ops.spmv_dot(d_ptr, d_idx, d_val, x, yd, w, out, shape, plan)
    return y, yd, out


def _check(d_ptr, d_idx, d_val, shape, ntemplates, x=None):
    """Templates vs the CSR arrays on the same plan; the other entry points of a templated plan as well."""
    plan = _plan(d_ptr, d_idx, d_val, shape)
    assert plan.templated and plan.ntemplates == ntemplates, plan.kernel_name
    assert "b2s::spmv_template_kernel" in plan.kernel_name
    if x is None:
        x = _x(shape[1], d_val.dtype)
    y, yd, out = _products(d_ptr, d_idx, d_val, x, shape, plan)
    # the tile-range entry point keeps the tile kernel on a templated plan
    nt = plan.tiles
    yt = torch.full_like(y, 7.0)
    for lo, hi in zip([0, nt // 2], [nt // 2, nt]):
        _ops.spmv_tiles(d_ptr, d_idx, d_val, x, yt, shape, plan, lo, hi)
    plan.set_packed(0)
    assert not plan.templated
    y0, yd0, out0 = _products(d_ptr, d_idx, d_val, x, shape, plan)
    assert _same(y, y0) and _same(yd, y0) and _same(yt, y0), plan.kernel_name
    tol = 1e-4 if d_val.dtype == torch.float32 else 1e-11
    assert torch.allclose(out, out0, rtol=tol, atol=0) or (torch.isnan(out).all() and torch.isnan(out0).all())
    plan.set_packed(3)
    assert plan.templated
    return plan, y


def _from_host(indptr, indices, vals, idt=torch.int32):
    return (torch.from_numpy(np.asarray(indptr)).to("cuda", idt), torch.from_numpy(np.asarray(indices)).to("cuda", idt),
            torch.from_numpy(np.asarray(vals)).cuda())


def _csr_from_triplets(rows, cols, vals, n):
    order = np.lexsort((cols, rows))
    rows, cols, vals = rows[order], cols[order], vals[order]
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=indptr[1:])
    return indptr, cols.astype(np.int64), vals


def _host(A):
    return A.indptr.cpu().numpy(), A.indices.cpu().numpy(), A.data.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [300, 3162])
def test_laplacian_templates_match_csr(n, dtype):
    A = gallery.laplacian_5pt(n, n, dtype)
    if n == 300:
        assert _signatures(*_host(A)) == 9
    plan, _ = _check(A.indptr, A.indices, A.data, A.shape, 9)
    assert A._get_plan().templated


@pytest.mark.gpu
def test_pde_operator_and_its_cg():
    """pde.py's 4094 x 4094 operator, and a CG solve on a templated plan (the fused-dot entry point)."""
    A = gallery.laplacian_5pt(4094, 4094, np.float64)
    _check(A.indptr, A.indices, A.data, A.shape, 9)
    from legate.sparse_b200 import linalg

    B = gallery.laplacian_5pt(200, 150, np.float64)
    assert B._get_plan().templated
    b = np.ones(B.shape[0])
    xs, iters = linalg.cg(B, b, tol=1e-10)
    ip, ix, dv = _host(B)
    S = sp.csr_matrix((dv, ix, ip), shape=B.shape)
    xs = xs.cpu().numpy() if isinstance(xs, torch.Tensor) else np.asarray(xs)
    assert iters > 0 and np.linalg.norm(b - S @ xs) <= 1e-6 * np.linalg.norm(b)


@pytest.mark.gpu
def test_gmg_poisson_with_explicit_zeros():
    n = 400
    N = n * n
    side = np.full(N - 1, -1.0)
    side[n - 1 :: n] = 0.0
    far = np.full(N - n, -1.0)
    rows, cols, vals = [], [], []
    for off, d in ((-n, far), (-1, side), (0, np.full(N, 4.0)), (1, side), (n, far)):
        r = np.arange(len(d)) + max(-off, 0)
        rows.append(r), cols.append(r + off), vals.append(d)
    indptr, indices, vals = _csr_from_triplets(np.concatenate(rows), np.concatenate(cols), np.concatenate(vals), N)
    assert (vals == 0.0).any()
    k = _signatures(indptr, indices, vals)
    assert k == 9
    x = _x(N, torch.float64)
    x[::17] = float("inf")          # explicit zeros times inf: NaN in both kernels
    _check(*_from_host(indptr, indices, vals), (N, N), k, x=x)


@pytest.mark.gpu
def test_stencil7_3d_has_27_templates():
    nx, ny, nz = 40, 30, 20
    N = nx * ny * nz
    i = np.arange(N)
    ix, iy, iz = i % nx, (i // nx) % ny, i // (nx * ny)
    rows, cols, vals = [i], [i], [np.full(N, 6.0)]
    for off, ok in ((1, ix < nx - 1), (-1, ix > 0), (nx, iy < ny - 1), (-nx, iy > 0), (nx * ny, iz < nz - 1),
                    (-nx * ny, iz > 0)):
        rows.append(i[ok]), cols.append(i[ok] + off), vals.append(np.full(ok.sum(), -1.0))
    indptr, indices, vals = _csr_from_triplets(np.concatenate(rows), np.concatenate(cols), np.concatenate(vals), N)
    assert _signatures(indptr, indices, vals) == 27
    for dt in (np.float32, np.float64):
        _check(*_from_host(indptr, indices, vals.astype(dt)), (N, N), 27)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_signed_zero_nan_inf_in_x(dtype):
    A = gallery.laplacian_5pt(300, 300, dtype)
    x = _x(A.shape[1], A.data.dtype)
    x[::5] = -0.0
    x[::7] = 0.0
    x[3::101] = float("nan")
    x[5::103] = float("inf")
    x[6::107] = -float("inf")
    _, y = _check(A.indptr, A.indices, A.data, A.shape, 9, x=x)
    assert torch.isnan(y).any()


@pytest.mark.gpu
def test_negative_zero_products_keep_their_sum_sign():
    """Rows whose products are all -0.0 (values -0.0 and 2.0, x >= 0): the sum is +0.0 in both kernels."""
    A = gallery.laplacian_5pt(300, 300, np.float64, a=-0.0, g=2.0)
    x = torch.zeros(A.shape[1], dtype=torch.float64, device="cuda")
    x[::3] = 1.0
    ip, ix, dv = _host(A)
    _check(A.indptr, A.indices, A.data, A.shape, _signatures(ip, ix, dv), x=x)


@pytest.mark.gpu
def test_int64_indices():
    A = gallery.laplacian_5pt(300, 200, np.float64, a=3.0, g=5.0)
    _check(A.indptr.to(torch.int64), A.indices.to(torch.int64), A.data, A.shape, 9)
    _check(A.indptr.to(torch.int64), A.indices, A.data, A.shape, 9)


@pytest.mark.gpu
@pytest.mark.parametrize("rows_per_lane,threads,streaming", [(1, 128, 1), (2, 128, 1), (2, 256, 0)])
def test_kernel_shapes_and_ragged_chunks(rows_per_lane, threads, streaming):
    """nrows not a multiple of a warp's 32 R rows; every shape the tuning hook offers computes the same y."""
    A = gallery.laplacian_5pt(301, 97, np.float64)
    assert A.shape[0] % 64 != 0
    L = _lib.lib
    try:
        _lib.check(L.b2s_spmv_set_template_config(rows_per_lane, threads, streaming), "b2s_spmv_set_template_config")
        _check(A.indptr, A.indices, A.data, A.shape, 9)
    finally:
        L.b2s_spmv_set_template_config(0, 0, 0)


@pytest.mark.gpu
def test_empty_rows():
    rng = np.random.default_rng(4)
    n = 100003
    lens = rng.integers(2, 4, n)
    lens[rng.integers(0, n, 3000)] = 0
    lens[500:900] = 0
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    r = np.repeat(np.arange(n), lens)
    pos = np.arange(indptr[-1]) - indptr[r]
    cols = np.minimum(r + 2 * pos, n - 1)
    vals = np.where(pos == 0, 2.0, -1.0)
    k = _signatures(indptr, cols, vals)
    assert k is not None and k <= 32
    _check(*_from_host(indptr, cols, vals), (n, n), k)


@pytest.mark.gpu
def test_32_signatures_qualify_33_do_not():
    n = 200000
    for nsig, want in ((32, True), (33, False)):
        rows = np.repeat(np.arange(n), 3)
        offs = np.tile(np.array([-1, 0, 1]), n)
        cols = np.clip(rows + offs, 0, n - 1)
        vals = np.tile(np.array([-1.0, 2.0, -1.0]), n)
        vals[1::3] = 2.0 + (np.arange(n) % (nsig - 2))      # interior rows: nsig - 2 diagonals, + 2 boundary rows
        keep = (rows + offs >= 0) & (rows + offs < n)
        indptr, indices, v = _csr_from_triplets(rows[keep], cols[keep], vals[keep], n)
        k = _signatures(indptr, indices, v)
        assert k == nsig
        d = _from_host(indptr, indices, v)
        plan = _plan(*d, (n, n))
        assert plan.templated == want and plan.ntemplates == (nsig if want else 0), plan.kernel_name
        if want:
            _check(*d, (n, n), nsig)
        else:
            assert plan.packed and "template" not in plan.kernel_name, plan.kernel_name
            with pytest.raises(_lib.B200SparseError):
                plan.set_packed(3)


@pytest.mark.gpu
def test_long_rows_and_scattered_matrices_fall_back():
    """A row of 9 entries, the 11-per-row band and R32 (32 random columns per row) keep their kernels."""
    n = 50000
    rows = np.repeat(np.arange(n), 3)
    cols = np.clip(rows + np.tile(np.array([-1, 0, 1]), n), 0, n - 1)
    rows, cols = np.concatenate([rows, np.full(6, 100)]), np.concatenate([cols, np.arange(110, 116)])
    indptr, indices, vals = _csr_from_triplets(rows, cols, np.ones(rows.shape[0]), n)
    assert np.diff(indptr).max() == 9
    plan = _plan(*_from_host(indptr, indices, vals), (n, n))
    assert not plan.templated and plan.ntemplates == 0 and "template" not in plan.kernel_name
    assert plan.coded, plan.kernel_name
    B = gallery.banded(100000, 11, np.float64)
    pb = B._get_plan()
    assert not pb.templated and pb.coded and "template" not in pb.kernel_name, pb.kernel_name
    R = gallery.random_fixed(100000, 100000, 32, np.float32)
    pr = R._get_plan()
    assert not pr.templated and "template" not in pr.kernel_name, pr.kernel_name


@pytest.mark.gpu
def test_launch_with_other_values_keeps_the_tile_kernel():
    A = gallery.laplacian_5pt(300, 300, np.float64)
    plan = A._get_plan()
    assert plan.templated
    other = torch.rand(A.nnz, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(9))
    x = _x(A.shape[1], torch.float64)

    def run(vals):
        return _ops.spmv(A.indptr, A.indices, vals, x, torch.empty_like(x), A.shape, plan=plan)

    yo = run(other)
    ya = run(A.data)
    plan.set_packed(0)
    assert _same(yo, run(other)) and _same(ya, run(A.data))
    plan.set_packed(3)
    assert not _same(yo, ya)


@pytest.mark.gpu
def test_inplace_data_edit_builds_a_new_plan():
    A = gallery.laplacian_5pt(300, 300, np.float64)
    x = _x(A.shape[1], torch.float64)
    y0 = A @ x
    plan0 = A._get_plan()
    assert plan0.templated
    A.data[:] = torch.where(A.data > 0, torch.full_like(A.data, 2.5), torch.full_like(A.data, -10.0))
    y1 = A @ x
    plan1 = A._get_plan()
    assert plan1 is not plan0 and plan1.templated
    assert not _same(y0, y1)
    B = sparse.csr_array((A.data.clone(), A.indices.clone(), A.indptr.clone()), shape=A.shape)
    B._get_plan().set_packed(0)
    assert _same(y1, B @ x)


def test_template_entry_points_reject_bad_handles():
    L = _lib.lib
    assert L.b2s_spmv_plan_templates_bytes(None) == 0
    assert L.b2s_spmv_plan_templates(None, None, None, None, None, None) == _lib.EINVAL
    assert L.b2s_spmv_plan_set_packed(None, 3) == _lib.EINVAL
    bogus = ctypes.create_string_buffer(256)
    assert L.b2s_spmv_plan_templates_bytes(ctypes.addressof(bogus)) == 0
    assert L.b2s_spmv_plan_templates(ctypes.addressof(bogus), None, None, None, None, None) == _lib.EINVAL
    assert L.b2s_spmv_set_template_config(4, 0, 0) == _lib.EINVAL
    assert L.b2s_spmv_set_template_config(0, 0, 0) == _lib.OK
