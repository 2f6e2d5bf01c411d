"""Timing of the DIA products `A @ x` / `A @ X` of a `dia_array` (csrc/dia.cu) next to the CSR route.

    python tools/bench_dia.py [--launches 50] [--reps 3] [--out DIR]

One process, one GPU.  Workloads:
  * L5: the 5-point Laplacian on a 3163 x 3163 grid (10M rows) built by `diags`, fp64: constant coefficients, which
    the warm CSR plan codes as row templates and so streams no values at all.
  * V7: the 7-point stencil on a 215^3 grid (9.94M rows) with random coefficients, fp64: CSR must stream every value
    and its column index, DIA only the value.
  * band11: 11 random diagonals at 4M rows, fp32 and fp64.
  * band11 SpMM: the fp64 band with k = 32.
Per workload: the kernel alone (`_ops.spmv_dia` / `_ops.spmm_dia` into a preallocated output, CUDA events around
`--launches` calls, median of `--reps` rounds); the bytes its model says it must move, sum over diagonals of the in-band
length * value + (n + m) * value (times k for X and Y in SpMM), and the GB/s they imply; `A.tocsr() @ x` with a warm
plan; the one-shot costs from a cold cache (host clock around a device synchronise): `A.tocsr()` plus its plan plus one
product, against one public `A @ x`; and the DIA -> CSR conversion, b2s_dia_to_csr against the tensor-operation route.
Each DIA output is checked against the CSR product.  The card's name and power limit are read in the same run and
printed with the numbers; `--out` also writes them as JSON.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import legate.sparse_b200 as sparse  # noqa: E402
from legate.sparse_b200 import _ops  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_csc import one_shot, power_limit  # noqa: E402
from bench_elementwise import timed  # noqa: E402


def laplacian_5pt(nx, dtype):
    n = nx * nx
    side = -np.ones(n - 1, dtype=dtype)
    side[np.arange(1, n) % nx == 0] = 0
    return sparse.diags([np.full(n, 4, dtype=dtype), side, side, -np.ones(n - nx, dtype=dtype),
                         -np.ones(n - nx, dtype=dtype)], [0, 1, -1, nx, -nx])


def variable_7pt(nx, dtype, seed=0):
    n, rng = nx ** 3, np.random.default_rng(seed)
    offsets = [0, 1, -1, nx, -nx, nx * nx, -nx * nx]
    return sparse.diags([rng.random(n - abs(k)).astype(dtype) + (6 if k == 0 else 0) for k in offsets], offsets)


def band(n, width, dtype, seed=1):
    rng = np.random.default_rng(seed)
    offsets = list(range(-(width // 2), width // 2 + 1))
    return sparse.diags([rng.random(n - abs(k)).astype(dtype) for k in offsets], offsets)


def workloads():
    """(name, make() -> dia_array, k or None for SpMV)"""
    yield "L5_fp64", lambda: laplacian_5pt(3163, np.float64), None
    yield "V7_fp64", lambda: variable_7pt(215, np.float64), None
    yield "band11_4M_fp32", lambda: band(4_000_000, 11, np.float32), None
    yield "band11_4M_fp64", lambda: band(4_000_000, 11, np.float64), None
    yield "band11_4M_fp64_k32", lambda: band(4_000_000, 11, np.float64), 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dia.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)

    rows = {}
    for name, make, k in workloads():
        A = make()
        m, n = A.shape
        offsets, data = A._in_band()
        tdt = data.dtype
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.rand((n,) if k is None else (n, k), generator=g, dtype=tdt, device="cuda")
        y = torch.empty((m,) if k is None else (m, k), dtype=tdt, device="cuda")

        if k is None:
            def kernel():
                _ops.spmv_dia(offsets, data, x, y, A.shape)
        else:
            def kernel():
                _ops.spmm_dia(offsets, data, x, y, A.shape)

        kernel()
        R = A.tocsr()
        y_csr = R @ x                            # builds R's plan
        torch.cuda.synchronize()
        max_rel = float((y - y_csr).abs().max()) / max(float(y_csr.abs().max()), 1e-300)
        out_csr = torch.empty_like(y)
        t_k, t_csr = [], []
        for _ in range(args.reps):
            t_k.append(timed(kernel, args.launches))
            t_csr.append(timed(lambda: R.dot(x, out=out_csr), args.launches))
        tk, tc = float(np.median(t_k)), float(np.median(t_csr))

        def cold_csr():
            A._cache.clear()                     # drop the cached CSR form (and with it its plan)
            A.tocsr() @ x

        def cold_dia():
            A._cache.clear()
            A @ x

        def convert_kernel():
            A._cache.clear()
            A.tocsr()

        t_cold_csr = one_shot(cold_csr, args.reps)
        t_cold_dia = one_shot(cold_dia, args.reps)
        t_conv = one_shot(convert_kernel, args.reps)
        t_conv_ops = one_shot(A._tocsr_tensor_ops, args.reps)
        sv, kk = data.element_size(), 1 if k is None else k
        nbytes = A.nnz * sv + (n + m) * kk * sv
        rows[name] = {"m": m, "n": n, "ndiag": int(data.shape[0]), "nnz": A.nnz, "k": k, "dtype": str(A.dtype),
                      "kernel_us": tk * 1e6, "model_bytes": nbytes, "gbs": nbytes / tk / 1e9, "csr_warm_us": tc * 1e6,
                      "one_shot_tocsr_plan_product_ms": t_cold_csr * 1e3, "one_shot_dia_product_ms": t_cold_dia * 1e3,
                      "dia_to_csr_kernel_ms": t_conv * 1e3, "dia_to_csr_tensor_ops_ms": t_conv_ops * 1e3,
                      "max_rel_diff_vs_csr": max_rel}
        del A, R, x, y, y_csr, out_csr, offsets, data
        torch.cuda.empty_cache()

    gpu, limit = torch.cuda.get_device_name(), power_limit()
    print(f"# {gpu}, power limit {limit} W; {args.launches} launches x {args.reps} rounds per kernel time")
    for name, r in rows.items():
        print(f"{name:20s} nnz {r['nnz']:>10d}  DIA {r['kernel_us']:9.1f} us  {r['gbs']:7.1f} GB/s of model bytes  |  "
              f"tocsr() @ x warm {r['csr_warm_us']:9.1f} us  |  one shot: tocsr + plan + product "
              f"{r['one_shot_tocsr_plan_product_ms']:8.2f} ms, A @ x {r['one_shot_dia_product_ms']:8.2f} ms  |  "
              f"DIA -> CSR {r['dia_to_csr_kernel_ms']:8.2f} ms (tensor ops {r['dia_to_csr_tensor_ops_ms']:8.2f} ms)"
              f"  |  max rel diff {r['max_rel_diff_vs_csr']:.1e}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_dia.json"), "w") as f:
            json.dump({"gpu": gpu, "power_limit_w": limit, "launches": args.launches, "reps": args.reps,
                       "workloads": rows}, f, indent=1)
    bad = [n for n, r in rows.items() if not r["max_rel_diff_vs_csr"] <= (1e-5 if r["dtype"] == "float32" else 1e-12)]
    if bad:
        raise SystemExit(f"DIA products differ from the CSR products: {bad}")


if __name__ == "__main__":
    main()
