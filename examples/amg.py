#!/usr/bin/env python
"""Smoothed-aggregation algebraic-multigrid-preconditioned CG on a rotated anisotropic diffusion problem -- the workload
of the reference's examples/amg.py (a V-cycle as the preconditioner M of linalg.cg).

The matrix is diffusion2D(N, epsilon=0.1, theta=pi/4): the 9-point finite-difference stencil of the reference, built
with `diags` from 9 offsets, with the stencil entries that cross the grid boundary dropped as the reference's
stencil_grid drops them.  Per level, as in the reference:
  * strength of connection: with theta = 0 (the reference default, `--theta 0`) the matrix itself; with theta > 0 the
    reference's filter: B = |A|, drop the entries with B_ij < theta * sqrt(B_ii * B_jj), then scale every entry by the
    largest of its column, B.max(axis=0) (the column reduction of csr_array; scipy's sparse column maximum, densified,
    with `--package scipy`);
  * aggregation by a distance-2 maximal independent set, MIS(2), found by repeated lexicographic-max products
    `C.tropical_spmv(x, out=z)` over (state, random priority, node id) triples, then one aggregate per MIS node
    (mis_aggregate);
  * when a level's aggregation would keep more than 90% of its unknowns, coarsening has stalled and that level is the
    coarsest (it only happens with theta > 0, once the coarse operators are dense);
  * the tentative prolongator T from fit_candidates (column sums by bincount), the smoothed prolongator
    P = T - (omega / rho) D^-1 A T with rho the spectral radius of D^-1 A by power iteration, R = P^T and
    A_c = R A P (two SpGEMMs), down to at most `max_coarse` unknowns, where a dense solve finishes the cycle.
A V-cycle is: pre-smooth, residual, restrict, recurse, prolong, correct, post-smooth (weighted Jacobi).

With `--package scipy` the same script runs on the host.  scipy has no tropical product, so the script brings a
vectorised one with the same rule as the library's: each row starts at the zero vector, so an empty row, or one whose
neighbours are all lexicographically negative, gives zeros.  The reference's scipy fallback takes the plain maximum
over the neighbours and omits that floor.  Every random value (MIS priorities, power-iteration start vectors) comes from
one seeded numpy generator on the host, so both packages build the same aggregates.

    python examples/amg.py -nodes 512 [--theta 0.25] [--package scipy]
"""
import argparse

import numpy as np

from common import select_package

ap = argparse.ArgumentParser()
ap.add_argument("-nodes", type=int, default=64, help="grid is nodes x nodes")
ap.add_argument("-m", "--maxiter", type=int, default=1000)
ap.add_argument("-t", "--tol", type=float, default=1e-8, help="CG stops when |r| < tol * |b|")
ap.add_argument("--max-coarse", type=int, default=10)
ap.add_argument("--seed", type=int, default=123)
ap.add_argument("--theta", type=float, default=0.0, help="strength-of-connection threshold (0 keeps every coupling)")
ap.add_argument("--package", default="b200")
args = ap.parse_args()

name, timer, xp, sparse, linalg, on_device = select_package()
rng = np.random.default_rng(args.seed)

if on_device:
    import torch

    def dev(a):
        return torch.as_tensor(a).cuda()

    def norm(v):
        return float(torch.linalg.norm(v))

    def vdot(a, b):
        return float(torch.dot(a, b))

    def tropical(C, x, out):
        C.tropical_spmv(x, out=out)

    def dense_solver(A):
        Ad = dev(A.toarray())
        return lambda b: torch.linalg.solve(Ad, b)

    def transpose(P):
        return P.T

    def entry_rows(B):
        return torch.repeat_interleave(torch.diff(B.indptr.long()))

    def column_max(B):
        return B.max(axis=0)
else:

    def dev(a):
        return np.asarray(a)

    def norm(v):
        return float(np.linalg.norm(v))

    def vdot(a, b):
        return float(np.dot(a, b))

    def tropical(C, x, out):
        """out[i] = lexicographic max of 0 and x[j] over the stored entries (i, j) of C (vectorised)."""
        m, nf = out.shape
        out[...] = 0
        rows = np.repeat(np.arange(m), np.diff(C.indptr))
        vals = x[C.indices]
        order = np.lexsort(tuple(vals[:, f] for f in range(nf - 1, -1, -1)) + (rows,))
        if order.size == 0:
            return
        last = order[np.r_[np.flatnonzero(np.diff(rows[order])), order.size - 1]]
        best = vals[last]
        nz = best != 0
        first = np.argmax(nz, axis=1)
        positive = nz.any(axis=1) & (best[np.arange(best.shape[0]), first] > 0)
        out[rows[last[positive]]] = best[positive]

    def dense_solver(A):
        Ad = A.toarray()
        return lambda b: np.linalg.solve(Ad, b)

    def transpose(P):
        return P.T.tocsr()

    def entry_rows(B):
        return np.repeat(np.arange(B.shape[0]), np.diff(B.indptr))

    def column_max(B):
        return B.max(axis=0).toarray().ravel()


def count(mask):
    return int(mask.sum())


def int_zeros(shape):
    return dev(np.zeros(shape, dtype=np.int64))


def diffusion2d(N, epsilon=0.1, theta=np.pi / 4):
    """The reference's diffusion2D: a rotated anisotropic 9-point stencil on an N x N grid, row-major numbering."""
    eps, C, S = float(epsilon), np.cos(theta), np.sin(theta)
    CS, CC, SS = C * S, C**2, S**2
    a = (-1 * eps - 1) * CC + (-1 * eps - 1) * SS + (3 * eps - 3) * CS
    b = (2 * eps - 4) * CC + (-4 * eps + 2) * SS
    c = (-1 * eps - 1) * CC + (-1 * eps - 1) * SS + (-3 * eps + 3) * CS
    d = (-4 * eps + 2) * CC + (2 * eps - 4) * SS
    e = (8 * eps + 8) * CC + (8 * eps + 8) * SS
    stencil = np.array([[a, b, c], [d, e, d], [c, b, a]]) / 6.0
    nv = N * N
    gi, gj = np.divmod(np.arange(nv), N)                     # grid coordinates of each column
    diagonals, offsets = [], []
    for di in (-1, 0, 1):
        for dj in (-1, 0, 1):
            col = np.full(nv, stencil[di + 1, dj + 1])
            # stencil_grid zeroes the couplings that cross the boundary, indexed by column
            col[(gi < di) | (gi >= N + di) | (gj < dj) | (gj >= N + dj)] = 0.0
            off = di * N + dj
            diagonals.append(col[off:] if off >= 0 else col[: nv + off])
            offsets.append(off)
    A = sparse.diags(diagonals, offsets, shape=(nv, nv), format="csr")
    A.eliminate_zeros()                                       # the dropped couplings are not edges of the graph
    return A


def strength(A, theta=0.0):
    """Strength of connection; theta = 0 (the reference default) keeps every coupling.  A stored zero couples nothing,
    and scipy prunes the zeros its products cancel to while this library keeps them, so the graph leaves them out
    (a no-op for a matrix without stored zeros).  theta > 0 follows the reference: |A| without its weak couplings,
    B_ij < theta * sqrt(B_ii * B_jj) (stored zeros among them), each entry divided by its column's maximum."""
    if theta > 0:
        B = abs(A)
        D = B.diagonal()
        rows, cols = entry_rows(B), B.indices
        B.data *= B.data >= theta * (D[rows] * D[cols]) ** 0.5
        B.eliminate_zeros()
        B.data /= column_max(B)[B.indices]
        return B
    if count(A.data == 0) == 0:
        return A
    C = A.copy()
    C.eliminate_zeros()
    return C


def maximal_independent_set(C, k):
    """Nodes of a distance-k maximal independent set of C's graph (the reference's maximal_independent_set).  Each node
    carries (state, priority, id): state 1 undecided, 2 in the set, 0 out.  A k-fold lexicographic-max product finds,
    for each node, the largest triple within distance k: an undecided node that is its own maximum joins the set, and
    an undecided node that sees a member leaves."""
    N = C.shape[0]
    prio = rng.integers(0, np.iinfo(np.int64).max, size=N)
    x = dev(np.stack([np.ones(N, dtype=np.int64), prio, np.arange(N, dtype=np.int64)], axis=1))
    y, z = int_zeros((N, 3)), int_zeros((N, 3))
    ids = dev(np.arange(N, dtype=np.int64))
    active = N
    while True:
        tropical(C, x, z)
        for _ in range(1, k):
            y, z = z, y
            tropical(C, y, z)
        undecided = x[:, 0] == 1
        mis = undecided & (z[:, 2] == ids)
        x[mis, 0] = 2
        out = (x[:, 0] == 1) & (z[:, 0] == 2)
        x[out, 0] = 0
        active -= count(mis) + count(out)
        if active == 0:
            break
        assert 0 < active < N
    return x[:, 0] == 2


def mis_aggregate(C):
    """Aggregate index of every node (the reference's mis_aggregate): each MIS(2) node roots an aggregate.  Two roots
    are at least 3 steps apart, so a root's neighbours join that root, and a node two steps away joins the
    largest-indexed root its neighbours joined."""
    roots = maximal_independent_set(C, 2)
    N = C.shape[0]
    n_coarse = count(roots)
    x, y, z = int_zeros((N, 2)), int_zeros((N, 2)), int_zeros((N, 2))
    x[roots, 0] = 2
    x[roots, 1] = dev(np.arange(n_coarse, dtype=np.int64))
    tropical(C, x, y)
    y[:, 0] += x[:, 0]
    tropical(C, y, z)
    return z[:, 1], n_coarse


def fit_candidates(agg, n_coarse, B):
    """Tentative prolongator T (one entry per row, in the aggregate's column) and the coarse candidates, as the
    reference's fit_candidates: values B^2 scaled by the square root of their column sums (a bincount)."""
    N = agg.shape[0]
    q = B * B
    if on_device:
        R = torch.sqrt(torch.bincount(agg, weights=q, minlength=n_coarse))
        T = sparse.coo_array((q / R[agg], (dev(np.arange(N)), agg)), shape=(N, n_coarse)).tocsr()
    else:
        R = np.sqrt(np.bincount(agg, weights=q, minlength=n_coarse))
        T = sparse.coo_array((q / R[agg], (np.arange(N), agg)), shape=(N, n_coarse)).tocsr()
    return T, R


def spectral_radius(A, iters=15):
    x = dev(rng.random(A.shape[0]))
    for _ in range(iters):
        x = x / norm(x)
        x, y = A @ x, x
    return vdot(x, y) / norm(y)


def smooth_prolongator(A, T, D, omega=4.0 / 3.0):
    """P = T - (omega / rho) D^-1 A T."""
    Dinv = 1.0 / D
    DinvA = A.multiply(Dinv.reshape(-1, 1)).tocsr()
    rho = spectral_radius(DinvA)
    return T - (DinvA * (omega / rho)) @ T, rho


class Level:
    def __init__(self, A, B):
        self.A, self.B = A, B
        self.R = self.P = self.D = None
        self.rho = None

    def pre(self, b, omega=4.0 / 3.0):
        return (omega / self.rho) * b / self.D

    def post(self, x, b, omega=4.0 / 3.0):
        return x + (omega / self.rho) * (b - self.A @ x) / self.D


def build_hierarchy(A, max_coarse):
    levels = [Level(A, dev(np.ones(A.shape[0])))]
    while levels[-1].A.shape[0] > max_coarse:
        L = levels[-1]
        L.D = L.A.diagonal()
        agg, n_coarse = mis_aggregate(strength(L.A, args.theta))
        if n_coarse > 0.9 * L.A.shape[0]:
            # coarsening has stalled (theta > 0 can filter a dense coarse level down to isolated nodes): this level
            # becomes the coarsest and is solved directly
            L.D = None
            break
        T, B_coarse = fit_candidates(agg, n_coarse, L.B)
        L.P, L.rho = smooth_prolongator(L.A, T, L.D)
        L.R = transpose(L.P)
        levels.append(Level(L.R @ L.A @ L.P, B_coarse))
    return levels, dense_solver(levels[-1].A)


def cycle(levels, solve, lvl, b):
    L = levels[lvl]
    x = L.pre(b)
    coarse_b = L.R @ (b - L.A @ x)
    coarse_x = solve(coarse_b) if lvl == len(levels) - 2 else cycle(levels, solve, lvl + 1, coarse_b)
    x = x + L.P @ coarse_x
    return L.post(x, b)


A = diffusion2d(args.nodes)
N = A.shape[0]
b = xp.ones(N)
timer.start()
levels, solve = build_hierarchy(A, args.max_coarse)
build_ms = timer.stop()
print(f"AMG hierarchy: {len(levels)} levels" + (f", strength of connection theta = {args.theta:g}" if args.theta else ""))
print("  level   unknowns   nonzeros")
for i, L in enumerate(levels):
    print(f"{i:>7d} {L.A.shape[0]:>10d} {L.A.nnz:>10d}")
print(f"AMG build time: {build_ms:.3f} ms")

if len(levels) > 1:
    def precondition(r):
        return cycle(levels, solve, 0, r)
else:
    def precondition(r):
        return solve(r)

tol = args.tol * norm(b)
M = linalg.LinearOperator(A.shape, matvec=precondition, dtype=np.float64)
timer.start()
if name == "b200":
    x, iters = linalg.cg(A, b, x0=xp.zeros(N), tol=tol, maxiter=args.maxiter, M=M, conv_test_iters=5)
else:
    it = [0]

    def counter(_):
        it[0] += 1

    x, info = linalg.cg(A, b, x0=np.zeros(N), rtol=0.0, atol=tol, maxiter=args.maxiter, M=M, callback=counter)
    iters = it[0]
solve_ms = timer.stop()
res = norm(b - A @ x)
print(f"Solve time: {solve_ms:.3f} ms")
print(f"Iterations / sec: {iters / (solve_ms / 1e3):.3f}")
state = "Converged" if res < tol else "Stopped"
print(f"{state} after {iters} iterations, |b - Ax| = {res:.3e} (tolerance {tol:.3e})")
