"""Kernel-level A/B/C of the SpMV structure encodings -- row templates, coded values, packed structure, CSR arrays -- next
to a streaming ceiling.

    python tools/bench_packed.py [--launches 200] [--reps 5] [--out DIR]

One process, one GPU.  The cases run in alternation, round after round (so drift on a shared machine hits all of them
alike), each timed with CUDA events around `--launches` back-to-back launches:
  * the 5-point Laplacian on a 3162 x 3162 grid (the benchmark's operator) in fp64, with coded values, packed with
    streamed values, and unpacked (the plan hook b2s_spmv_plan_set_packed switches the same plan), and in fp32;
  * an 11-per-row band of 10M rows, fp64, the same three ways;
  * a read-only streaming probe: torch.sum over 1.6 GB of fp64 -- the bandwidth this card sustains at its power limit.
Per case: median / min / max time per launch, the CSR-equivalent rate (the bytes CSR SpMV needs, what bench.py
counts), the bytes the launched kernel actually moves (from the plan's tile shapes) and that rate as a fraction of the
probe.  The card's name and power limit are printed with the numbers.  `--out` also writes them as JSON.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from legate.sparse_b200 import _ops, gallery  # noqa: E402


def card():
    name, limit = torch.cuda.get_device_name(), None
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        limit = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        pass
    return name, limit


def csr_bytes(A):
    sv, si, sp = A.data.element_size(), A.indices.element_size(), A.indptr.element_size()
    n, m = A.shape
    return A.nnz * (sv + si) + (n + 1) * sp + m * sv + n * sv


def moved_bytes(A, plan, mode):
    """Bytes one launch streams: per tile the plan entry, and either the staged 16-byte groups of indices / indptr or
    the packed uint16 slices plus the tile base; values (none when coded: mode 2), x once and y once.  Row templates
    (mode 3): one id byte per row, x once and y once."""
    sv, si, sp = A.data.element_size(), A.indices.element_size(), A.indptr.element_size()
    n, m = A.shape
    if mode == 3:
        return n + m * sv + n * sv
    e = plan.buf[: 4 * (plan.tiles + 1)].view(-1, 4).cpu().numpy().astype(np.int64)
    k = (e[:, 0] & 0xFFFFFFFF) | (e[:, 1] << 32)
    r = e[:, 2]
    t = np.arange(plan.tiles)
    k0, k1, r0, r1 = k[:-1], k[1:], r[:-1], r[1:]
    live = r1 > r0
    if mode:
        c = ((k1 + 7) & ~7) - (k0 & ~7)
        q = ((r1 + 1 + 8 * t + 7) & ~7) - ((r0 + 8 * t) & ~7)
        struct = int(((c + q) * 2 + 8)[live].sum())
    else:
        struct = int(((k1 - (k0 & ~3)) * si)[live].sum() + ((((r1 + 1 + 3) & ~3) - (r0 & ~3)) * sp)[live].sum())
    return (0 if mode == 2 else A.nnz * sv) + struct + 16 * plan.tiles + m * sv + n * sv


def time_per_launch(fn, launches):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e-3 / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_packed.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)

    mats = {
        "l5_fp64": gallery.laplacian_5pt(3162, 3162, np.float64),
        "l5_fp32": gallery.laplacian_5pt(3162, 3162, np.float32),
        "banded11_fp64": gallery.banded(10_000_000, 11, np.float64),
    }
    cases = {}
    for name, A in mats.items():
        plan = A._get_plan()
        x = torch.rand(A.shape[1], dtype=A.data.dtype, device="cuda")
        y = torch.empty(A.shape[0], dtype=A.data.dtype, device="cuda")

        def run(A=A, plan=plan, x=x, y=y):
            _ops.spmv(A.indptr, A.indices, A.data, x, y, A.shape, plan=plan)

        modes = [2, 1, 0] if plan.coded else [1, 0] if plan.packed else [0]
        for mode in ([3] if plan.templated else []) + modes:
            cases[f"{name}_{('csr', 'packed', 'coded', 'templates')[mode]}"] = dict(
                run=run, plan=plan, mode=mode, csr=csr_bytes(A), moved=moved_bytes(A, plan, mode),
                flops=2 * A.nnz, kernel=None)
    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    cases["probe_sum_fp64_1.6GB"] = dict(run=lambda: probe.sum(), plan=None, mode=0, csr=None,
                                         moved=probe.numel() * 8, flops=None, kernel="torch.sum")

    def select(c):
        plan = c["plan"]
        if plan is None:
            return
        if plan.pack_buf is not None:
            plan.set_packed(c["mode"])
        c["kernel"] = plan.kernel_name

    for c in cases.values():       # warm-up: module load, first-touch of every buffer
        select(c)
        for _ in range(10):
            c["run"]()
    torch.cuda.synchronize()
    times = {n: [] for n in cases}
    for _ in range(args.reps):
        for n, c in cases.items():
            select(c)
            c["run"]()
            times[n].append(time_per_launch(c["run"], args.launches))

    name, limit = card()
    ceiling = float(np.median([cases["probe_sum_fp64_1.6GB"]["moved"] / t for t in times["probe_sum_fp64_1.6GB"]]))
    rows = {}
    print(f"# {name}, power limit {limit} W; {args.launches} launches x {args.reps} alternating rounds per case")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for n, c in cases.items():
        ts = sorted(times[n])
        t = float(np.median(ts))
        row = {"us_median": t * 1e6, "us_min": ts[0] * 1e6, "us_max": ts[-1] * 1e6, "kernel": c["kernel"],
               "moved_bytes": c["moved"], "moved_tbs": c["moved"] / t / 1e12, "moved_frac_of_probe": c["moved"] / t / ceiling}
        if c["csr"] is not None:
            row.update(csr_bytes=c["csr"], csr_equiv_tbs=c["csr"] / t / 1e12, gflops=c["flops"] / t / 1e9)
        rows[n] = row
        extra = f" csr-equiv {row['csr_equiv_tbs']:.3f} TB/s  {row['gflops']:.1f} GFLOP/s" if c["csr"] is not None else ""
        print(f"{n:24s} {t * 1e6:8.1f} us [{ts[0] * 1e6:.1f}..{ts[-1] * 1e6:.1f}]  moved {c['moved'] / 1e6:7.1f} MB "
              f"{row['moved_tbs']:.3f} TB/s = {row['moved_frac_of_probe']:.3f} of probe{extra}  {c['kernel']}")
    for m in mats:
        if f"{m}_packed" in rows:
            print(f"# {m}: csr / packed time = {rows[f'{m}_csr']['us_median'] / rows[f'{m}_packed']['us_median']:.3f}")
        if f"{m}_coded" in rows:
            print(f"# {m}: packed / coded time = {rows[f'{m}_packed']['us_median'] / rows[f'{m}_coded']['us_median']:.3f}, "
                  f"csr / coded = {rows[f'{m}_csr']['us_median'] / rows[f'{m}_coded']['us_median']:.3f}")
        if f"{m}_templates" in rows and f"{m}_coded" in rows:
            print(f"# {m}: coded / templates time = "
                  f"{rows[f'{m}_coded']['us_median'] / rows[f'{m}_templates']['us_median']:.3f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_packed.json"), "w") as f:
            json.dump({"gpu": name, "power_limit_w": limit, "launches": args.launches, "reps": args.reps,
                       "probe_tbs": ceiling / 1e12, "cases": rows}, f, indent=1)


if __name__ == "__main__":
    main()
