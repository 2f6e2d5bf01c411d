"""Timing of the CSC scatter products `A @ x` / `A @ X` of a `csc_array` (csrc/csc.cu) next to the CSR route.

    python tools/bench_csc.py [--launches 50] [--reps 3] [--out DIR]

One process, one GPU.  Workloads:
  * L5: the 5-point Laplacian on a 3163 x 3163 grid (10M rows), fp64.  It is symmetric, so its CSC arrays are its CSR
    arrays and the scatter kernel reads the same bytes as the tuned CSR plan.
  * R32: 10M x 10M with 32 uniformly random columns per row (gallery.random_fixed), fp32, as a csc_array: the rows of
    each column are scattered, the worst case for the atomics.
  * RMAT21T: the transpose of R-MAT scale 21 (its CSR arrays read as CSC), fp64: power-law columns test the balancing.
  * SpMM: the 11-per-row band at 4M rows, fp64, k = 32.
Per workload: the kernel alone (`_ops.spmv_csc` / `_ops.spmm_csc` into a preallocated output, CUDA events around
`--launches` calls, median of `--reps` rounds); the bytes it must move, nnz*(value + index) + (ncols+1)*indptr + x + y
(X and Y for SpMM), and the nnz (nnz*k) atomics it issues; `A.tocsr() @ x` with a warm plan (the CSR SpMV / SpMM); and
the one-shot costs from a cold CSR cache: `A.tocsr()` plus its plan plus one product, against one public `A @ x`
(host clock around a device synchronise).  Each scatter output is checked against the CSR product.  The card's name
and power limit are read in the same run and printed with the numbers; `--out` also writes them as JSON.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from legate.sparse_b200 import _ops, gallery  # noqa: E402
from legate.sparse_b200.csc import csc_array  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_elementwise import card, timed  # noqa: E402


def workloads():
    """(name, make() -> csc_array, k or None for SpMV)"""
    yield "L5_fp64", lambda: csc_array._wrap(gallery.laplacian_5pt(3163, 3163, np.float64)), None
    yield "R32_fp32", lambda: csc_array(gallery.random_fixed(10_000_000, 10_000_000, 32, np.float32)), None
    yield "RMAT21T_fp64", lambda: csc_array._wrap(gallery.rmat(21, dtype=np.float64)), None
    yield "band11_4M_fp64_k32", lambda: csc_array._wrap(gallery.banded(4_000_000, 11, np.float64)), 32


def power_limit():
    _, limit = card()
    if limit is not None:
        return limit
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def one_shot(fn, reps):
    vals = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        vals.append(time.perf_counter() - t0)
    return float(np.median(vals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_csc.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)

    rows = {}
    for name, make, k in workloads():
        A = make()
        T = A.T                                  # the stored arrays: CSR of the transpose
        m, n = A.shape
        tdt = T.data.dtype
        g = torch.Generator(device="cuda").manual_seed(0)
        shape_in = (n,) if k is None else (n, k)
        x = torch.rand(shape_in, generator=g, dtype=tdt, device="cuda")
        y = torch.empty((m,) if k is None else (m, k), dtype=tdt, device="cuda")

        if k is None:
            def kernel():
                _ops.spmv_csc(T.indptr, T.indices, T.data, x, y, A.shape)
        else:
            def kernel():
                _ops.spmm_csc(T.indptr, T.indices, T.data, x, y, A.shape)

        kernel()
        R = A.tocsr()
        y_csr = R @ x                            # builds R's plan (SpMV)
        torch.cuda.synchronize()
        max_rel = float((y - y_csr).abs().max()) / max(float(y_csr.abs().max()), 1e-300)
        out_csr = torch.empty_like(y)
        t_k, t_csr = [], []
        for _ in range(args.reps):
            t_k.append(timed(kernel, args.launches))
            t_csr.append(timed(lambda: R.dot(x, out=out_csr), args.launches))
        tk, tc = float(np.median(t_k)), float(np.median(t_csr))

        def cold_csr():
            T._cache.pop("transpose", None)      # drop the cached CSR form (and with it its plan)
            A.tocsr() @ x

        t_cold_csr = one_shot(cold_csr, args.reps)
        t_cold_csc = one_shot(lambda: A @ x, args.reps)
        sv, si, sp_ = T.data.element_size(), T.indices.element_size(), T.indptr.element_size()
        kk = 1 if k is None else k
        nbytes = A.nnz * (sv + si) + (n + 1) * sp_ + n * kk * sv + m * kk * sv
        rows[name] = {"m": m, "n": n, "nnz": A.nnz, "k": k, "dtype": str(A.dtype), "kernel_us": tk * 1e6,
                      "bytes": nbytes, "gbs": nbytes / tk / 1e9, "atomics": A.nnz * kk,
                      "atomics_per_ns": A.nnz * kk / tk / 1e9, "csr_warm_us": tc * 1e6,
                      "one_shot_tocsr_plan_product_ms": t_cold_csr * 1e3, "one_shot_csc_product_ms": t_cold_csc * 1e3,
                      "max_rel_diff_vs_csr": max_rel}
        del A, T, R, x, y, y_csr, out_csr
        torch.cuda.empty_cache()

    gpu, limit = torch.cuda.get_device_name(), power_limit()
    print(f"# {gpu}, power limit {limit} W; {args.launches} launches x {args.reps} rounds per kernel time")
    for name, r in rows.items():
        print(f"{name:20s} nnz {r['nnz']:>10d}  scatter {r['kernel_us']:9.1f} us  {r['gbs']:7.1f} GB/s  "
              f"{r['atomics_per_ns']:6.2f} atomics/ns  |  tocsr() @ x warm {r['csr_warm_us']:9.1f} us  |  one shot: "
              f"tocsr + plan + product {r['one_shot_tocsr_plan_product_ms']:8.2f} ms, A @ x "
              f"{r['one_shot_csc_product_ms']:8.2f} ms  |  max rel diff {r['max_rel_diff_vs_csr']:.1e}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_csc.json"), "w") as f:
            json.dump({"gpu": gpu, "power_limit_w": limit, "launches": args.launches, "reps": args.reps,
                       "workloads": rows}, f, indent=1)
    bad = [n for n, r in rows.items() if not r["max_rel_diff_vs_csr"] <= (1e-4 if r["dtype"] == "float32" else 1e-10)]
    if bad:
        raise SystemExit(f"scatter products differ from the CSR products: {bad}")


if __name__ == "__main__":
    main()
