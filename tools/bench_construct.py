"""Timing of assembly from blocks (csrc/construct.cu) next to a streaming probe, device and torch baselines and scipy.

    python tools/bench_construct.py [--launches 5] [--reps 3] [--no-scipy] [--out DIR]

One process, one GPU, fp64.  Workloads: kronsum of two tridiagonals to the 5-point Laplacian on a 3162 x 3162 grid
(10M rows); the 3-D 7-point operator on a 215^3 grid through nested kronsum; vstack of the two row halves and hstack of
the two column halves of that Laplacian; block_diag of 10^5 dense 8 x 8 blocks (already csr_arrays on the device).
Per call: the whole call (CUDA events around `--launches` calls, median of `--reps` rounds, after a warm-up call; it
includes the host checks, the allocations and, for kronsum, both products and the add); the bytes it must move, from
shapes (every operand array read once, the result's arrays written once); that against a read-only streaming probe
(torch.sum over 1.6 GB of fp64) in the same run.  Baselines: gallery.laplacian_5pt on the device for the Laplacian, a
torch composite (torch.cat with shifted row pointers and columns) for vstack and block_diag, and one scipy call on the
host (host arrays prepared beforehand).  The card's name, power limit and maximum SM clock are printed with the
numbers; `--out` writes JSON.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import legate.sparse_b200 as sparse  # noqa: E402
from legate.sparse_b200 import gallery  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_elementwise import timed  # noqa: E402
from bench_tropical import card  # noqa: E402


def median_time(fn, launches, reps):
    fn()
    torch.cuda.synchronize()
    return float(np.median([timed(fn, launches) for _ in range(reps)]))


def nbytes(*mats):
    """bytes of the indptr, indices and data arrays of csr_arrays"""
    return sum(t.numel() * t.element_size() for M in mats for t in (M.indptr, M.indices, M.data))


def tridiag(n, s):
    return sparse.diags([s * np.ones(n - 1), -2 * s * np.ones(n), s * np.ones(n - 1)], [-1, 0, 1], format="csr")


def torch_stack_rows(mats, col_offsets):
    """vstack / block_diag with torch ops: row pointers shifted by the entries above, columns by the offsets"""
    ptrs, base = [torch.zeros(1, dtype=torch.int64, device="cuda")], 0
    for M in mats:
        ptrs.append(M.indptr[1:].to(torch.int64) + base)
        base += M.nnz
    idx = torch.cat([M.indices.to(torch.int64) + c for M, c in zip(mats, col_offsets)])
    return torch.cat(ptrs), idx, torch.cat([M.data for M in mats])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-scipy", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, power, clock = card()

    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    ceiling = probe.numel() * 8 / median_time(lambda: probe.sum(), 20, args.reps)
    del probe

    n = 3162
    a, g = float((n + 1) ** 2), float((n + 1) ** 2)
    T1, T2 = tridiag(n, a), tridiag(n, g)
    L = gallery.laplacian_5pt(n, n, np.float64)
    N = L.shape[0]
    top, bottom = L[: N // 2], L[N // 2:]
    left, right = L[:, : N // 2], L[:, N // 2:]
    m = 215
    T3 = tridiag(m, 1.0)
    P2 = sparse.kronsum(T3, T3)
    rng = np.random.default_rng(0)
    blocks = [sparse.csr_array(rng.standard_normal((8, 8))) for _ in range(100_000)]

    cases = []

    def case(label, fn, operands, baselines=(), host=None):
        out = fn()
        torch.cuda.synchronize()
        t = median_time(fn, args.launches, args.reps)
        moved = nbytes(*operands) + nbytes(out)
        row = {"case": label, "shape": list(out.shape), "nnz": out.nnz, "us": t * 1e6, "bytes": moved,
               "GBps": moved / t / 1e9, "frac_of_probe": moved / t / ceiling}
        for bname, bfn in baselines:
            row[f"{bname}_us"] = median_time(bfn, args.launches, args.reps) * 1e6
        if host is not None and not args.no_scipy:
            h0 = time.perf_counter()
            host()
            row["scipy_host_us"] = (time.perf_counter() - h0) * 1e6
        cases.append(row)
        del out

    host_t = (T1.to_scipy_sparse_csr(), T2.to_scipy_sparse_csr())
    case("kronsum -> 5-point Laplacian 3162^2", lambda: sparse.kronsum(T1, T2), [T1, T2],
         [("gallery_laplacian_5pt", lambda: gallery.laplacian_5pt(n, n, np.float64))],
         lambda: sp.kronsum(*host_t, format="csr"))
    host_3 = (P2.to_scipy_sparse_csr(), T3.to_scipy_sparse_csr())
    case("nested kronsum -> 7-point 215^3", lambda: sparse.kronsum(P2, T3), [P2, T3], (),
         lambda: sp.kronsum(*host_3, format="csr"))
    host_v = (top.to_scipy_sparse_csr(), bottom.to_scipy_sparse_csr())
    case("vstack of two L5 row halves", lambda: sparse.vstack([top, bottom]), [top, bottom],
         [("torch_cat", lambda: torch_stack_rows([top, bottom], [0, 0]))],
         lambda: sp.vstack(host_v, format="csr"))
    host_h = (left.to_scipy_sparse_csr(), right.to_scipy_sparse_csr())
    case("hstack of two L5 column halves", lambda: sparse.hstack([left, right]), [left, right], (),
         lambda: sp.hstack(host_h, format="csr"))
    offs = [8 * k for k in range(len(blocks))]
    host_b = [B.to_scipy_sparse_csr() for B in blocks]
    case("block_diag of 1e5 dense 8x8", lambda: sparse.block_diag(blocks), blocks,
         [("torch_cat", lambda: torch_stack_rows(blocks, offs))], lambda: sp.block_diag(host_b, format="csr"))

    print(f"# {name}, power limit {power}, max SM clock {clock}")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for r in cases:
        extra = "".join(f", {k[:-3]} {v:.0f} us" for k, v in r.items() if k.endswith("_us") and k != "us")
        print(f"{r['case']:<38} {r['us']:>10.0f} us  {r['bytes'] / 1e6:>9.1f} MB  {r['GBps']:>7.1f} GB/s "
              f"({r['frac_of_probe']:.2f} of probe){extra}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_construct.json"), "w") as f:
            json.dump({"card": name, "power_limit": power, "max_sm_clock": clock, "probe_Bps": ceiling,
                       "cases": cases}, f, indent=1)


if __name__ == "__main__":
    main()
