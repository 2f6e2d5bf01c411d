"""Timing of csr_array indexing (csrc/index.cu) next to a streaming probe, a torch composite and scipy on the host.

    python tools/bench_index.py [--launches 5] [--reps 3] [--no-scipy] [--out DIR]

One process, one GPU.  Matrices: the 5-point Laplacian on a 3162 x 3162 grid (10M rows, fp64) and R-MAT scale 20 (fp64).
Cases: a contiguous row slice (the middle half), a random row permutation, a column permutation, a symmetric
permutation A[ix_(p, p)], a half row mask, repeated columns (every column twice) and 1M random element lookups.  Per
case: the whole `A[key]` call (CUDA events around `--launches` calls, median of `--reps` rounds; it includes the map
build, the one readback and the allocations); the bytes it must move, from shapes (the selected source entries read,
the output written, the indptr reads and writes); that against a read-only streaming probe (torch.sum over 1.6 GB of
fp64) in the same run; a torch composite of the same selection (repeat_interleave / index_select / cumsum, the way
`_column_blocks` cuts blocks; lookups have none) and scipy on the host (one call, host arrays prepared beforehand).
The card's name, power limit and maximum SM clock (nvidia-smi) are printed with the numbers; `--out` writes JSON.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from legate.sparse_b200 import gallery  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_elementwise import timed  # noqa: E402
from bench_tropical import card  # noqa: E402


def median_time(fn, launches, reps):
    fn()
    torch.cuda.synchronize()
    return float(np.median([timed(fn, launches) for _ in range(reps)]))


def torch_rows(A, rows):
    """Row selection with torch ops: output indptr by cumsum of the lengths, source positions by repeat_interleave."""
    ptr = A.indptr.to(torch.int64)
    lens = (ptr[1:] - ptr[:-1]).index_select(0, rows)
    out_ptr = torch.zeros(rows.numel() + 1, dtype=torch.int64, device=ptr.device)
    torch.cumsum(lens, 0, out=out_ptr[1:])
    start = torch.repeat_interleave(ptr.index_select(0, rows) - out_ptr[:-1], lens)
    src = start + torch.arange(start.numel(), device=ptr.device)
    return out_ptr, A.indices.index_select(0, src), A.data.index_select(0, src)


def torch_cols(A, cols, ncols):
    """Column selection with torch ops for unique or repeated `cols`: a dense map from column to its first position and
    multiplicity, every kept entry repeated by its multiplicity (positions of a repeated column are first + k * n, as
    for `tile`)."""
    dev = A.data.device
    mult = torch.bincount(cols, minlength=ncols)
    first = torch.full((ncols,), -1, dtype=torch.int64, device=dev)
    first.scatter_reduce_(0, cols, torch.arange(cols.numel(), device=dev), "amin", include_self=False)
    c = A.indices.to(torch.int64)
    m = mult.index_select(0, c)
    keep = torch.repeat_interleave(torch.arange(c.numel(), device=dev), m)
    ptr = A.indptr.to(torch.int64)
    row_m = torch.zeros(A.shape[0], dtype=torch.int64, device=dev).index_add_(
        0, torch.repeat_interleave(torch.arange(A.shape[0], device=dev), ptr[1:] - ptr[:-1]), m)
    out_ptr = torch.zeros(A.shape[0] + 1, dtype=torch.int64, device=dev)
    torch.cumsum(row_m, 0, out=out_ptr[1:])
    return out_ptr, first.index_select(0, c.index_select(0, keep)), A.data.index_select(0, keep)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-scipy", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_index.py measures on the GPU; there is no CPU path"
    name, power, sm_clock = card()
    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    ceiling = probe.numel() * 8 / median_time(lambda: probe.sum(), 20, args.reps)
    del probe
    rng = np.random.default_rng(0)
    rows_out = []
    for mname, make in (("l5_10M_f64", lambda: gallery.laplacian_5pt(3162, 3162, np.float64)),
                        ("rmat20_f64", lambda: gallery.rmat(20))):
        A = make()
        m, n = A.shape
        dev = A.data.device
        S = None if args.no_scipy else A.to_scipy_sparse_csr()
        p_np = rng.permutation(m)
        p = torch.from_numpy(p_np).to(dev)
        q = torch.from_numpy(rng.permutation(n)).to(dev)
        mask = rng.random(m) < 0.5
        twice = torch.arange(2 * n, device=dev) % n
        ri, ci = rng.integers(0, m, 1 << 20), rng.integers(0, n, 1 << 20)
        rid, cid = torch.from_numpy(ri).to(dev), torch.from_numpy(ci).to(dev)
        cases = [
            ("row slice", (slice(m // 4, 3 * m // 4), slice(None)), lambda: torch_rows(A, torch.arange(
                m // 4, 3 * m // 4, device=dev)), (slice(m // 4, 3 * m // 4), slice(None))),
            ("row permutation", (p, slice(None)), lambda: torch_rows(A, p), (p_np, slice(None))),
            ("column permutation", (slice(None), q), lambda: torch_cols(A, q, n), (slice(None), q.cpu().numpy())),
            ("symmetric permutation", np.ix_(p_np, p_np), None, np.ix_(p_np, p_np)),
            ("half row mask", (torch.from_numpy(mask).to(dev), slice(None)), lambda: torch_rows(
                A, torch.from_numpy(np.flatnonzero(mask)).to(dev)), (mask, slice(None))),
            ("repeated columns", (slice(None), twice), lambda: torch_cols(A, twice, n), (slice(None), twice.cpu().numpy())),
            ("1M lookups", (rid, cid), None, (ri, ci)),
        ]
        for cname, key, composite, host_key in cases:
            B = A[key]
            t = median_time(lambda: A[key], args.launches, args.reps)
            if isinstance(B, torch.Tensor):
                nbytes = 2 * B.numel() * 8 + B.numel() * B.element_size()             # (i, j) pairs in, values out
            else:
                nbytes = (B.nnz * (B.data.element_size() + A.indices.element_size())    # selected entries read
                          + B.nnz * (B.data.element_size() + B.indices.element_size())  # output written
                          + (B.shape[0] + 1) * 8 * 3)                                 # indptr reads, writes, scan
            base = None if composite is None else median_time(composite, args.launches, args.reps)
            t_scipy = None
            if S is not None:
                t0 = time.perf_counter()
                S[host_key]
                t_scipy = time.perf_counter() - t0
            rows_out.append({"matrix": mname, "case": cname, "call_us": t * 1e6, "bytes": nbytes,
                             "frac_of_probe": nbytes / t / ceiling, "torch_us": None if base is None else base * 1e6,
                             "scipy_ms": None if t_scipy is None else t_scipy * 1e3})
            del B
        del A, S
        torch.cuda.empty_cache()
    print(f"# {name}, power limit {power}, max SM clock {sm_clock}")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for r in rows_out:
        tb = f"  torch {r['torch_us']:9.1f} us" if r["torch_us"] is not None else "  torch        -"
        sc = f"  scipy {r['scipy_ms']:9.1f} ms" if r["scipy_ms"] is not None else ""
        print(f"{r['matrix']:11s} {r['case']:22s} call {r['call_us']:9.1f} us  {r['bytes'] / 1e6:8.1f} MB "
              f"({r['frac_of_probe']:.2f} of probe){tb}{sc}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_index.json"), "w") as f:
            json.dump({"card": name, "power_limit": power, "max_sm_clock": sm_clock, "launches": args.launches,
                       "reps": args.reps, "probe_tbs": ceiling / 1e12, "cases": rows_out}, f, indent=1)


if __name__ == "__main__":
    main()
