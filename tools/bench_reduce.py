"""Timing of the csr_array row / column reductions (csrc/reduce.cu) next to a streaming probe and torch / SpMV baselines.

    python tools/bench_reduce.py [--launches 20] [--reps 5] [--out DIR]

One process, one GPU.  Matrices: the 5-point Laplacian on a 3162 x 3162 grid (10M rows) in fp64 and fp32, and R-MAT
scale 20 (fp64).  Ops: sum, max, argmax and count_nonzero, along rows (axis 1) and columns (axis 0).
Per case: the kernel alone (`_ops.csr_reduce_rows` into a preallocated output on the arrays it reads -- A for row sums,
the canonical form otherwise, the transpose / its canonical form for columns; CUDA events around `--launches` calls,
median of `--reps` rounds); the bytes from shapes, (m+1)*sp + nnz*sv (+ nnz*si for argmax) + m*so, set against a
read-only streaming probe (torch.sum over 1.6 GB of fp64) in the same run; and one baseline per direction:
  * rows: `torch.segment_reduce` over the values with the row lengths (sum / max; argmax and count have none), and for
    sum also `A @ ones` through the library's SpMV with its plan built beforehand (not timed);
  * columns: `torch.scatter_reduce` of the values into the columns (sum / amax; count as a sum of `data != 0`).
The one-time costs of a column reduction -- building the transpose and its canonical form -- are timed separately.
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
from legate.sparse_b200 import _ops, gallery  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_elementwise import timed  # noqa: E402
from bench_tropical import card  # noqa: E402

OPS = ["sum", "max", "argmax", "count_nonzero"]


def matrices():
    yield "l5_10M_f64", lambda: gallery.laplacian_5pt(3162, 3162, np.float64)
    yield "l5_10M_f32", lambda: gallery.laplacian_5pt(3162, 3162, np.float32)
    yield "rmat20_f64", lambda: gallery.rmat(20)


def median_time(fn, launches, reps):
    fn()
    torch.cuda.synchronize()
    return float(np.median([timed(fn, launches) for _ in range(reps)]))


def once(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_reduce.py measures on the GPU; there is no CPU path"
    name, power, sm_clock = card()
    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    ceiling = probe.numel() * 8 / median_time(lambda: probe.sum(), 20, args.reps)
    del probe
    rows = []
    for mname, make in matrices():
        A = make()
        m, n = A.shape
        dev = A.data.device
        _, t_transpose = once(lambda: A._derived("transpose", None, A.transpose))
        _, t_canon = once(A._canonical)
        _, t_canon_t = once(A._canonical_t)
        plan = A._get_plan()
        ones = torch.ones(n, dtype=A.data.dtype, device=dev)
        y = torch.empty(m, dtype=A.data.dtype, device=dev)
        lengths = (A.indptr[1:] - A.indptr[:-1]).to(torch.int64)
        cols = A.indices.to(torch.int64)
        for axis in (1, 0):
            if axis == 1:
                src = {"sum": (A.indptr, A.indices, A.data)}
                canon = A._canonical()
            else:
                At = A._derived("transpose", None, A.transpose)
                src = {"sum": (At.indptr, At.indices, At.data)}
                canon = A._canonical_t()
            nout = m if axis == 1 else n
            for op in OPS:
                ptr_, idx, dat = src.get(op, canon)
                odt = dat.dtype if op in ("sum", "max") else torch.int64
                out = torch.empty(nout, dtype=odt, device=dev)
                arg = op == "argmax"
                t = median_time(lambda: _ops.csr_reduce_rows(op, ptr_, idx if arg else None, dat, n if axis == 1 else m,
                                                             out=out), args.launches, args.reps)
                nbytes = (ptr_.numel() * ptr_.element_size() + dat.numel() * dat.element_size()
                          + (idx.numel() * idx.element_size() if arg else 0) + nout * out.element_size())
                base, base_name = None, None
                if axis == 1 and op in ("sum", "max"):
                    red = "sum" if op == "sum" else "max"
                    base = median_time(lambda: torch.segment_reduce(A.data, red, lengths=lengths), args.launches,
                                       args.reps)
                    base_name = f"segment_reduce({red})"
                if axis == 0 and op in ("sum", "max", "count_nonzero"):
                    red = "amax" if op == "max" else "sum"
                    vals = (A.data != 0).to(torch.int64) if op == "count_nonzero" else A.data
                    init = torch.zeros(n, dtype=vals.dtype, device=dev)
                    base = median_time(lambda: init.scatter_reduce(0, cols, vals, red, include_self=False),
                                       args.launches, args.reps)
                    base_name = f"scatter_reduce({red})"
                row = {"matrix": mname, "op": op, "axis": axis, "kernel_us": t * 1e6, "bytes": nbytes,
                       "frac_of_probe": nbytes / t / ceiling, "baseline": base_name,
                       "baseline_us": None if base is None else base * 1e6}
                if axis == 1 and op == "sum":
                    row["spmv_ones_us"] = median_time(
                        lambda: _ops.spmv(A.indptr, A.indices, A.data, ones, y, A.shape, plan=plan),
                        args.launches, args.reps) * 1e6
                rows.append(row)
        rows.append({"matrix": mname, "build_transpose_ms": t_transpose * 1e3, "build_canonical_ms": t_canon * 1e3,
                     "build_canonical_t_ms": t_canon_t * 1e3})
        del A
        torch.cuda.empty_cache()
    print(f"# {name}, power limit {power}, max SM clock {sm_clock}")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for r in rows:
        if "op" not in r:
            print(f"{r['matrix']:12s} one-time: transpose {r['build_transpose_ms']:.2f} ms, canonical "
                  f"{r['build_canonical_ms']:.2f} ms, canonical of the transpose {r['build_canonical_t_ms']:.2f} ms")
            continue
        extra = f"  A @ ones {r['spmv_ones_us']:8.1f} us" if "spmv_ones_us" in r else ""
        base = f"  {r['baseline']} {r['baseline_us']:9.1f} us" if r["baseline"] else ""
        print(f"{r['matrix']:12s} {r['op']:14s} axis {r['axis']}  kernel {r['kernel_us']:8.1f} us  "
              f"{r['bytes'] / 1e6:8.1f} MB ({r['frac_of_probe']:.2f} of probe){base}{extra}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_reduce.json"), "w") as f:
            json.dump({"card": name, "power_limit": power, "max_sm_clock": sm_clock, "launches": args.launches,
                       "reps": args.reps, "probe_tbs": ceiling / 1e12, "cases": rows}, f, indent=1)


if __name__ == "__main__":
    main()
