"""Timing of the lexicographic-max product `A.tropical_spmv(x)` (csrc/tropical.cu) next to a streaming ceiling, a torch
composite and the fp64 SpMV on the same structure.

    python tools/bench_tropical.py [--launches 20] [--reps 5] [--out DIR]

One process, one GPU.  Cases (matrix, F):
  * the 5-point Laplacian on a 3162 x 3162 grid (10M rows), F = 1, 2, 3: short rows of 3-5 entries;
  * the 9-point diffusion operator of examples/amg.py on the same grid, F = 3: the AMG fine level's MIS(2) product;
  * R-MAT scale 20, F = 3: power-law rows, the long ones finished one warp per row;
  * 32 uniformly random columns per row on 2^20 x 2^20, F = 2: scattered gathers of x rows.
Per case: the kernel alone (`_ops.tropical_spmv` into a preallocated output, CUDA events around `--launches` calls,
median of `--reps` rounds); the algorithmic bytes nnz*si + (m+1)*sp + n*F*8 + m*F*8 set against a read-only streaming
probe (torch.sum over 1.6 GB of fp64) in the same run; a torch composite of F masked `scatter_reduce(amax)` passes (each
pass keeps, per row, the entries that tie the maximum of the fields before it; the entries' row ids are precomputed and
not timed); and the fp64 SpMV `A @ x` on the same structure, for context.  The kernel's output is compared bitwise
with the composite's.  The card's name, power limit and maximum SM clock (nvidia-smi) are printed with the numbers;
`--out` also writes them as JSON.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import legate.sparse_b200 as sparse  # noqa: E402
from legate.sparse_b200 import _ops, gallery  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_elementwise import timed  # noqa: E402


def card():
    """(name, power limit, max SM clock) as nvidia-smi reports them."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        line = r.stdout.strip().splitlines()[torch.cuda.current_device()]
        return tuple(v.strip() for v in line.split(","))
    except Exception as exc:   # no nvidia-smi: the name from torch, the rest unknown
        return torch.cuda.get_device_name(), f"unknown ({type(exc).__name__})", "unknown"


def diffusion9(N):
    """The structure of examples/amg.py's diffusion2D(N): 9 offsets, couplings across the grid boundary dropped."""
    nv = N * N
    gi, gj = np.divmod(np.arange(nv), N)
    diagonals, offsets = [], []
    for di in (-1, 0, 1):
        for dj in (-1, 0, 1):
            col = np.ones(nv)
            col[(gi < di) | (gi >= N + di) | (gj < dj) | (gj >= N + dj)] = 0.0
            off = di * N + dj
            diagonals.append(col[off:] if off >= 0 else col[: nv + off])
            offsets.append(off)
    return sparse.diags(diagonals, offsets, shape=(nv, nv), format="csr")


def cases():
    yield "l5_10M_F1", lambda: gallery.laplacian_5pt(3162, 3162, np.float64), 1
    yield "l5_10M_F2", lambda: gallery.laplacian_5pt(3162, 3162, np.float64), 2
    yield "l5_10M_F3", lambda: gallery.laplacian_5pt(3162, 3162, np.float64), 3
    yield "diffusion9_3162^2_F3", lambda: diffusion9(3162), 3
    yield "rmat20_F3", lambda: gallery.rmat(20), 3
    yield "random32_2^20_F2", lambda: gallery.random_fixed(2**20, 2**20, 32, np.float64), 2


class Composite:
    """Lexicographic max of 0 and x[j] per row with torch ops: F masked scatter_reduce(amax) passes, then the floor."""

    def __init__(self, A):
        m = A.shape[0]
        counts = (A.indptr[1:] - A.indptr[:-1]).to(torch.int64)
        self.rows = torch.repeat_interleave(torch.arange(m, device="cuda"), counts)
        self.cols = A.indices.to(torch.int64)
        self.m = m

    def __call__(self, x):
        nf = x.shape[1]
        low = torch.iinfo(torch.int64).min
        y = torch.empty((self.m, nf), dtype=torch.int64, device="cuda")
        live = torch.ones_like(self.rows, dtype=torch.bool)
        for f in range(nf):
            v = x[self.cols, f]
            best = torch.full((self.m,), low, dtype=torch.int64, device="cuda")
            best.scatter_reduce_(0, self.rows, torch.where(live, v, low), "amax")
            live &= v == best[self.rows]
            y[:, f] = best
        # floor at zero: keep a row only when its first nonzero field is positive (empty rows hold `low`: negative)
        nz = y != 0
        first = torch.argmax(nz.to(torch.int8), dim=1)
        keep = nz.any(dim=1) & (y.gather(1, first[:, None])[:, 0] > 0)
        return torch.where(keep[:, None], y, 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tropical.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)

    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    probe.sum()
    ceiling = probe.numel() * 8 / float(np.median([timed(lambda: probe.sum(), 20) for _ in range(args.reps)]))
    del probe
    torch.cuda.empty_cache()

    rows = {}
    for name, make, nf in cases():
        A = make()
        m, n = A.shape
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randint(-2**40, 2**40, (n, nf), generator=g, dtype=torch.int64, device="cuda")
        y = torch.empty((m, nf), dtype=torch.int64, device="cuda")

        def kernel():
            _ops.tropical_spmv(A.indptr, A.indices, x, y)

        comp = Composite(A)
        kernel()
        same = bool(torch.equal(y, comp(x)))
        Af = A.astype(np.float64, copy=False)
        xf = torch.rand(n, dtype=torch.float64, device="cuda")
        yf = torch.empty(m, dtype=torch.float64, device="cuda")
        Af.dot(xf, out=yf)                                               # plan built outside the timing
        t_k, t_c, t_s = [], [], []
        for _ in range(args.reps):
            t_k.append(timed(kernel, args.launches))
            t_c.append(timed(lambda: comp(x), max(1, args.launches // 4)))
            t_s.append(timed(lambda: Af.dot(xf, out=yf), args.launches))
        tk, tc, ts = (float(np.median(t)) for t in (t_k, t_c, t_s))
        sp_, si = A.indptr.element_size(), A.indices.element_size()
        nbytes = A.nnz * si + (m + 1) * sp_ + n * nf * 8 + m * nf * 8
        counts = (A.indptr[1:] - A.indptr[:-1])
        rows[name] = {"m": m, "n": n, "nnz": A.nnz, "F": nf, "long_rows": int((counts > 32).sum()),
                      "kernel_us": tk * 1e6, "bytes": nbytes, "frac_of_probe": nbytes / tk / ceiling,
                      "composite_us": tc * 1e6, "spmv_fp64_us": ts * 1e6, "bitwise_equal_to_composite": same}
        del A, Af, x, y, xf, yf, comp
        torch.cuda.empty_cache()

    gpu, limit, clock = card()
    print(f"# {gpu}, power limit {limit}, max SM clock {clock}; {args.launches} calls x {args.reps} rounds per case")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for name, r in rows.items():
        print(f"{name:22s} nnz {r['nnz']:>10d} long rows {r['long_rows']:>6d}  kernel {r['kernel_us']:8.1f} us "
              f"({r['frac_of_probe']:.2f} of probe)  torch composite {r['composite_us']:9.1f} us "
              f"({r['composite_us'] / r['kernel_us']:.1f}x)  fp64 SpMV {r['spmv_fp64_us']:7.1f} us  "
              f"equal {r['bitwise_equal_to_composite']}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_tropical.json"), "w") as f:
            json.dump({"gpu": gpu, "power_limit": limit, "max_sm_clock": clock, "launches": args.launches,
                       "reps": args.reps, "probe_tbs": ceiling / 1e12, "cases": rows}, f, indent=1)
    bad = [n for n, r in rows.items() if not r["bitwise_equal_to_composite"]]
    if bad:
        raise SystemExit(f"kernel and composite differ: {bad}")


if __name__ == "__main__":
    main()
