"""Timing of the sampled dense-dense product `A.sddmm(C, D)` (csrc/sddmm.cu) next to a streaming ceiling.

    python tools/bench_sddmm.py [--launches 20] [--reps 3] [--out DIR]

One process, one GPU.  Cases (matrix, dtype, k):
  * the 5-point Laplacian on a 3162 x 3162 grid (10M rows), fp32 and fp64, k = 16 and 64: short rows, a packed lane
    group of 4 or 16 lanes (k = 16 fp32 / fp64) up to full warps;
  * the 11-per-row band at 4M rows (the SpMM benchmark's shape), fp64, k = 32;
  * R-MAT scale 20, fp32, k = 32: power-law rows, where a row-balanced kernel would idle;
  * 32 uniformly random columns per row on 2^20 x 2^20, fp32, k = 32: scattered gathers of D transposed.
Per case: the kernel alone (`_ops.sddmm` into a preallocated output, CUDA events around `--launches` calls), the
algorithmic HBM bytes nnz*(si + 2 sv) + (m+1)*sp + m*k*sv + n*k*sv set against a read-only streaming probe (torch.sum
over 1.6 GB of fp64), the gathered bytes nnz*k*sv, and one public `A.sddmm(C, D)` call with D given pre-transposed
(D = K.T, no copy) and row-major (one transposed copy).  torch.sparse.sampled_addmm on the same operands is timed
beside it when this torch build runs it; it samples C @ D on A's pattern without scaling by A's values, so its work is
comparable, not identical.  A row sample of every output is checked against float64 on the host.  The card's name and
power limit are printed with the numbers; `--out` also writes them as JSON.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from legate.sparse_b200 import _ops, gallery  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_elementwise import card, timed  # noqa: E402


def cases():
    yield "l5_fp32_k16", lambda: gallery.laplacian_5pt(3162, 3162, np.float32), 16
    yield "l5_fp32_k64", lambda: gallery.laplacian_5pt(3162, 3162, np.float32), 64
    yield "l5_fp64_k16", lambda: gallery.laplacian_5pt(3162, 3162, np.float64), 16
    yield "l5_fp64_k64", lambda: gallery.laplacian_5pt(3162, 3162, np.float64), 64
    yield "banded11_4M_fp64_k32", lambda: gallery.banded(4_000_000, 11, np.float64), 32
    yield "rmat20_fp32_k32", lambda: gallery.rmat(20, dtype=np.float32), 32
    yield "random32_2^20_fp32_k32", lambda: gallery.random_fixed(2**20, 2**20, 32, np.float32), 32


def check_rows(A, C, K, vals, nrows=256):
    """Largest |error| / bound over a seeded row sample, against float64 on the host (bound as in the tests)."""
    m = A.shape[0]
    rows = np.sort(np.random.default_rng(0).choice(m, min(nrows, m), replace=False))
    ptr = A.indptr.cpu().numpy().astype(np.int64)
    sel = np.concatenate([np.arange(ptr[r], ptr[r + 1]) for r in rows])
    rr = np.repeat(rows, ptr[rows + 1] - ptr[rows])
    cols = A.indices.cpu().numpy().astype(np.int64)[sel]
    a = A.data.cpu().numpy().astype(np.float64)[sel]
    Cr = C[torch.as_tensor(rr, device=C.device)].double().cpu().numpy()
    Kr = K[torch.as_tensor(cols, device=K.device)].double().cpu().numpy()
    ref = a * np.einsum("ij,ij->i", Cr, Kr)
    bound = 2 * (C.shape[1] + 2) * np.finfo(A.dtype).eps / 2 * np.abs(a) * np.einsum("ij,ij->i", np.abs(Cr), np.abs(Kr))
    err = np.abs(vals.cpu().numpy().astype(np.float64)[sel] - ref)
    return float(np.max(err / np.maximum(bound, np.finfo(np.float64).tiny))) if sel.size else 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sddmm.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)

    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    probe.sum()
    ceiling = probe.numel() * 8 / float(np.median([timed(lambda: probe.sum(), 20) for _ in range(args.reps)]))
    del probe
    torch.cuda.empty_cache()

    rows = {}
    for name, make, k in cases():
        A = make()
        m, n = A.shape
        tdt = A.data.dtype
        g = torch.Generator(device="cuda").manual_seed(0)
        C = torch.randn(m, k, generator=g, dtype=tdt, device="cuda")
        K = torch.randn(n, k, generator=g, dtype=tdt, device="cuda")     # D = K.T
        Drow = K.T.contiguous()                                           # the same D, row-major
        out = torch.empty_like(A.data)

        def kernel():
            _ops.sddmm(A.indptr, A.indices, A.data, C, K, out)

        kernel()
        torch.cuda.synchronize()
        max_err = check_rows(A, C, K, out)
        t_kernel, t_pre, t_row = [], [], []
        for _ in range(args.reps):
            t_kernel.append(timed(kernel, args.launches))
            t_pre.append(timed(lambda: A.sddmm(C, K.T), args.launches))
            t_row.append(timed(lambda: A.sddmm(C, Drow), args.launches))
        tk, tp, tr = (float(np.median(t)) for t in (t_kernel, t_pre, t_row))
        sp_, si, sv = A.indptr.element_size(), A.indices.element_size(), A.data.element_size()
        hbm = A.nnz * (si + 2 * sv) + (m + 1) * sp_ + m * k * sv + n * k * sv
        gathered = A.nnz * k * sv
        row = {"m": m, "n": n, "nnz": A.nnz, "k": k, "dtype": str(A.dtype), "kernel_us": tk * 1e6,
               "hbm_bytes": hbm, "hbm_frac_of_probe": hbm / tk / ceiling, "gathered_bytes": gathered,
               "gathered_tbs": gathered / tk / 1e12, "call_pretransposed_us": tp * 1e6, "call_row_major_us": tr * 1e6,
               "max_err_over_bound": max_err}
        try:
            T = torch.sparse_csr_tensor(A.indptr.to(torch.int64), A.indices.to(torch.int64), A.data, A.shape)

            def ref():
                return torch.sparse.sampled_addmm(T, C, K.T, beta=0.0, alpha=1.0)

            ref()
            row["torch_sampled_addmm_us"] = float(np.median([timed(ref, args.launches) for _ in range(args.reps)])) * 1e6
            del T
        except Exception as exc:   # not every torch build runs it for every dtype / size
            row["torch_sampled_addmm_us"] = f"not run: {type(exc).__name__}"
        rows[name] = row
        del A, C, K, Drow, out
        torch.cuda.empty_cache()

    gpu, limit = card()
    print(f"# {gpu}, power limit {limit} W; {args.launches} calls x {args.reps} rounds per case")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for name, r in rows.items():
        tt = r["torch_sampled_addmm_us"]
        tt = f"{tt:.1f} us" if isinstance(tt, float) else tt
        print(f"{name:24s} nnz {r['nnz']:>10d}  kernel {r['kernel_us']:8.1f} us ({r['hbm_frac_of_probe']:.2f} of probe, "
              f"gathers {r['gathered_tbs']:.2f} TB/s)  call D=K.T {r['call_pretransposed_us']:8.1f} us  "
              f"call D row-major {r['call_row_major_us']:8.1f} us  torch sampled_addmm {tt}  "
              f"err/bound {r['max_err_over_bound']:.2f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sddmm.json"), "w") as f:
            json.dump({"gpu": gpu, "power_limit_w": limit, "launches": args.launches, "reps": args.reps,
                       "probe_tbs": ceiling / 1e12, "cases": rows}, f, indent=1)
    bad = [n for n, r in rows.items() if not r["max_err_over_bound"] <= 1.0]
    if bad:
        raise SystemExit(f"outputs outside the error bound: {bad}")


if __name__ == "__main__":
    main()
