"""Timing of sparse.random (csrc/random.cu) next to a streaming probe, a torch composite and scipy.

    python tools/bench_random.py [--reps 3] [--no-scipy] [--no-torch] [--out DIR]

One process, one GPU.  Workloads: a 10^7 x 10^7 fp32 matrix with 32 entries per row on average (3.2e8 entries, the
size of the project's SpMV benchmarks); a 10^6 x 10^6 fp64 matrix at density 10^-4 (10^8 entries); a 2e4 x 2e4 fp64
matrix at density 0.7, which samples the 1.2e8 zeros and emits their complement.  Per workload: the whole call
`sparse.random(..., format="csr")` (CUDA events around one call, median of `--reps`, after a warm-up call; it includes
the host checks, the allocations and the per-round readbacks); the number of sampling rounds; the bytes of the result
and the bytes the call moves as modelled from shapes (`model_bytes`), the latter as a rate against a read-only
streaming probe (torch.sum over 1.6 GB of fp64) in the same run.  Baselines: a torch composite on the device with the
same complement rule (torch.randint of the shortfall and torch.unique of everything drawn, until enough positions are
distinct; above density 1/2 these are the zeros and a boolean mask gives the rest), and scipy.sparse.random_array
once on the host at the middle size.  The card's name, power limit and maximum SM
clock are printed with the numbers; `--out` writes JSON.
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
from legate.sparse_b200 import _ops  # noqa: E402
from legate.sparse_b200.csr import _index_dtype, _indptr_dtype  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_elementwise import timed  # noqa: E402
from bench_tropical import card  # noqa: E402

WORKLOADS = [  # (label, m, n, density, dtype, scipy)
    ("1e7 x 1e7, 32 per row, fp32", 10**7, 10**7, 32 / 10**7, np.float32, False),
    ("1e6 x 1e6, density 1e-4, fp64", 10**6, 10**6, 1e-4, np.float64, True),
    ("2e4 x 2e4, density 0.7 (complement), fp64", 2 * 10**4, 2 * 10**4, 0.7, np.float64, False),
]


def model_bytes(m, n, k, isz, psz, vsz):
    """Device traffic of one call, from shapes, as the kernels are written (s = min(k, mn - k) sampled positions,
    slots the table's capacity, 32-byte sectors): the table memset, one sector read and written per insert, the
    (row, column) triplets written; the assembly's count (triplet rows read), fill (triplets and their moved 4-byte
    values read, indices and values written) and row sort (indices and values read and written once more); the row
    pointers written and scanned (about four passes); the complement (zero columns read, k indices written); the values
    written.  Collisions, rejected draws and the readbacks are left out, so this is a floor for the algorithm."""
    mn = m * n
    s = min(k, mn - k)
    slots = 2
    while slots < 2 * s:
        slots *= 2
    b = 8 * slots + 2 * 32 * s + 2 * isz * s                 # table, inserts, triplets
    b += isz * s + (2 * isz + 4) * s + (isz + 4) * s           # count, fill
    b += 2 * (isz + 4) * s + 4 * (m + 1) * psz                 # row sort, row pointers
    if k > mn - k:
        b += isz * s + isz * k + (m + 1) * psz                  # complement
    return b + vsz * k


def median_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    return float(np.median([timed(fn, 1) for _ in range(reps)]))


def torch_composite(m, n, k, dtype, gen):
    """canonical CSR arrays of a uniform k-subset with torch ops, with the sampler's complement rule: draw the shortfall
    of s = min(k, mn - k) with randint and keep the distinct positions (torch.unique sorts them), until s are distinct
    (each round draws only the shortfall, so there are never more); when k > mn - k those are the zeros, and the
    result is the positions a boolean mask over all mn leaves set"""
    mn = m * n
    s = min(k, mn - k)
    pos = torch.empty(0, dtype=torch.int64, device="cuda")
    while pos.numel() < s:
        draw = torch.randint(0, mn, (s - pos.numel(),), dtype=torch.int64, device="cuda", generator=gen)
        pos = torch.unique(torch.cat([pos, draw]))
    if s < k:
        keep = torch.ones(mn, dtype=torch.bool, device="cuda")
        keep[pos] = False
        pos = keep.nonzero().squeeze(1)
    rows, cols = pos // n, pos % n
    indptr = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(torch.bincount(rows, minlength=m), 0, out=indptr[1:])
    return indptr, cols, torch.rand(k, dtype=dtype, device="cuda", generator=gen)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-scipy", action="store_true")
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, power, clock = card()

    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    ceiling = probe.numel() * 8 / median_time(lambda: probe.sum(), args.reps)
    del probe

    cases = []
    for label, m, n, density, dtype, with_scipy in WORKLOADS:
        k = int(round(density * m * n))
        seed = np.random.default_rng(0)
        fn = lambda: sparse.random(m, n, density, format="csr", dtype=dtype, rng=seed)  # noqa: E731
        A = fn()
        assert A.nnz == k
        del A
        t = median_time(fn, args.reps)
        _, _, _, rounds = _ops.random_csr((m, n), k, 1, _index_dtype(max(m, n)), _indptr_dtype(k), dtype)
        isz, psz, vsz = _index_dtype(max(m, n)).itemsize, _indptr_dtype(k).itemsize, np.dtype(dtype).itemsize
        out_bytes = (m + 1) * psz + k * (isz + vsz)
        moved = model_bytes(m, n, k, isz, psz, vsz)
        row = {"case": label, "shape": [m, n], "nnz": k, "rounds": rounds, "ms": t * 1e3, "result_bytes": out_bytes,
               "model_bytes": moved, "GBps": moved / t / 1e9, "frac_of_probe": moved / t / ceiling}
        torch.cuda.empty_cache()
        if not args.no_torch:
            gen = torch.Generator(device="cuda").manual_seed(0)
            tdt = torch.float32 if dtype == np.float32 else torch.float64
            row["torch_composite_ms"] = median_time(lambda: torch_composite(m, n, k, tdt, gen), args.reps) * 1e3
            torch.cuda.empty_cache()
        if with_scipy and not args.no_scipy:
            h0 = time.perf_counter()
            sp.random_array((m, n), density=density, format="csr", dtype=dtype, rng=0)
            row["scipy_host_ms"] = (time.perf_counter() - h0) * 1e3
        cases.append(row)
        print(row, flush=True)

    print(f"# {name}, power limit {power}, max SM clock {clock}")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for r in cases:
        extra = "".join(f", {k[:-3]} {v:.1f} ms" for k, v in r.items() if k.endswith("_ms") and k != "ms")
        print(f"{r['case']:<44} {r['ms']:>9.1f} ms  rounds {r['rounds']}  {r['result_bytes'] / 1e9:>6.2f} GB result  "
              f"{r['model_bytes'] / 1e9:>6.2f} GB modelled, {r['GBps']:>7.1f} GB/s ({r['frac_of_probe']:.2f} of probe)"
              f"{extra}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_random.json"), "w") as f:
            json.dump({"card": name, "power_limit": power, "max_sm_clock": clock, "probe_Bps": ceiling,
                       "cases": cases}, f, indent=1)


if __name__ == "__main__":
    main()
