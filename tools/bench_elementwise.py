"""Timing of sparse + / - sparse (the row merge of csrc/elementwise.cu) next to a streaming ceiling.

    python tools/bench_elementwise.py [--launches 10] [--reps 3] [--out DIR]

One process, one GPU.  Cases:
  * the 5-point Laplacian on a 3162 x 3162 grid (10M rows, the benchmark's operator), fp64 and fp32: A + A,
    A - sigma * I and A + B with B the 11-per-row band of the same size;
  * the 11-per-row band at 4M rows: B + B.
Per case: the time of one `A + B` call (allocation of C included), and the symbolic and numeric passes alone (each
timed with CUDA events around `--launches` calls on preallocated buffers; the symbolic pass ends with its one host
sync).  Bytes moved per pass are computed from the shapes, and set against a read-only streaming probe (torch.sum over
1.6 GB of fp64).  torch's own sparse-CSR addition on the device is timed beside ours when this torch build runs it.
The card's name and power limit are printed with the numbers.  `--out` also writes them as JSON.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import legate.sparse_b200 as sparse  # noqa: E402
from legate.sparse_b200 import _lib, gallery  # noqa: E402
from legate.sparse_b200.runtime import idx_code, ptr, runtime, vt_code  # noqa: E402

L = _lib.lib


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


def timed(fn, launches):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e-3 / launches


class Passes:
    """The two passes of C = A + B on preallocated buffers (what _ops.csr_binop runs, minus the allocations)."""

    def __init__(self, A, B):
        self.A, self.B = A, B
        m, n = A.shape
        dev = A.data.device
        self.scratch = torch.empty(int(L.b2s_csr_binop_scratch_bytes(m)), dtype=torch.uint8, device=dev)
        self.c_ptr = torch.empty(m + 1, dtype=torch.int64, device=dev)
        self.info = (_lib.c_i64 * 3)()
        self.symbolic()
        self.nnz = int(self.info[0])
        self.c_idx = torch.empty(self.nnz, dtype=A.indices.dtype, device=dev)
        self.c_val = torch.empty(self.nnz, dtype=A.data.dtype, device=dev)

    def symbolic(self):
        A, B = self.A, self.B
        _lib.check(L.b2s_csr_binop_symbolic(0, idx_code(A.indices.dtype), idx_code(A.indptr.dtype), A.shape[0], A.shape[1],
                                            ptr(A.indptr), ptr(A.indices), ptr(B.indptr), ptr(B.indices), ptr(self.c_ptr),
                                            self.info, ptr(self.scratch), runtime.stream_ptr()), "symbolic")

    def numeric(self):
        A, B = self.A, self.B
        _lib.check(L.b2s_csr_binop_numeric(0, vt_code(A.data.dtype), idx_code(A.indices.dtype), idx_code(A.indptr.dtype),
                                           A.shape[0], A.shape[1], ptr(A.indptr), ptr(A.indices), ptr(A.data),
                                           ptr(B.indptr), ptr(B.indices), ptr(B.data), ptr(self.c_ptr), ptr(self.c_idx),
                                           ptr(self.c_val), ptr(self.scratch), runtime.stream_ptr()), "numeric")

    def bytes(self):
        """(symbolic, numeric) bytes: both indptr and indices read, c_indptr written and scanned (read + write) /
        both indptr, c_indptr and every entry of A and B read, every entry of C written."""
        A, B = self.A, self.B
        m = A.shape[0]
        sp, si, sv = A.indptr.element_size(), A.indices.element_size(), A.data.element_size()
        nin = A.nnz + B.nnz
        sym = 2 * (m + 1) * sp + nin * si + 3 * (m + 1) * 8
        num = 2 * (m + 1) * sp + (m + 1) * 8 + nin * (si + sv) + self.nnz * (si + sv)
        return sym, num


def torch_csr(A):
    return torch.sparse_csr_tensor(A.indptr.to(torch.int64), A.indices.to(torch.int64), A.data, A.shape)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_elementwise.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)

    cases = {}
    for dt, tag in ((np.float64, "fp64"), (np.float32, "fp32")):
        A = gallery.laplacian_5pt(3162, 3162, dt)
        n = A.shape[0]
        S = 0.5 * sparse.eye(n, dtype=dt)
        Bd = gallery.banded(n, 11, dt)
        cases[f"l5_{tag} A+A"] = (A, A)
        cases[f"l5_{tag} A-sigma*I"] = (A, S)
        cases[f"l5_{tag} A+banded11"] = (A, Bd)
    Bb = gallery.banded(4_000_000, 11, np.float64)
    cases["banded11_4M_fp64 B+B"] = (Bb, Bb)
    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB

    rows = {}
    t_probe = []
    for _ in range(args.reps):
        t_probe.append(timed(lambda: probe.sum(), 20))
    ceiling = probe.numel() * 8 / float(np.median(t_probe))
    for name, (A, B) in cases.items():
        sub = "-sigma" in name
        ps = Passes(A, -1.0 * B if sub else B)   # the subtraction's merge is the addition's with -b: same bytes
        ps.numeric()

        def call(A=A, B=B, sub=sub):
            return A - B if sub else A + B

        call()
        t_sym, t_num, t_call = [], [], []
        for _ in range(args.reps):
            t_sym.append(timed(ps.symbolic, args.launches))
            t_num.append(timed(ps.numeric, args.launches))
            t_call.append(timed(call, args.launches))
        b_sym, b_num = ps.bytes()
        ts, tn, tc = (float(np.median(t)) for t in (t_sym, t_num, t_call))
        row = {"nnz_a": A.nnz, "nnz_b": B.nnz, "nnz_c": ps.nnz, "call_us": tc * 1e6, "symbolic_us": ts * 1e6,
               "numeric_us": tn * 1e6, "symbolic_bytes": b_sym, "numeric_bytes": b_num,
               "symbolic_frac_of_probe": b_sym / ts / ceiling, "numeric_frac_of_probe": b_num / tn / ceiling}
        try:
            ta, tb = torch_csr(A), torch_csr(B)
            fn = (lambda: ta - tb) if sub else (lambda: ta + tb)
            fn()
            row["torch_csr_us"] = float(np.median([timed(fn, args.launches) for _ in range(args.reps)])) * 1e6
        except Exception as exc:   # not every torch build adds sparse CSR tensors on the device
            row["torch_csr_us"] = f"not run: {type(exc).__name__}"
        rows[name] = row
        del ps
        torch.cuda.empty_cache()

    gpu, limit = card()
    print(f"# {gpu}, power limit {limit} W; {args.launches} calls x {args.reps} rounds per case")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    for name, r in rows.items():
        tt = r["torch_csr_us"]
        tt = f"{tt:.1f} us" if isinstance(tt, float) else tt
        print(f"{name:26s} nnz(C) {r['nnz_c']:>10d}  call {r['call_us']:8.1f} us  symbolic {r['symbolic_us']:7.1f} us "
              f"({r['symbolic_frac_of_probe']:.2f} of probe)  numeric {r['numeric_us']:7.1f} us "
              f"({r['numeric_frac_of_probe']:.2f} of probe)  torch CSR add {tt}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_elementwise.json"), "w") as f:
            json.dump({"gpu": gpu, "power_limit_w": limit, "launches": args.launches, "reps": args.reps,
                       "probe_tbs": ceiling / 1e12, "cases": rows}, f, indent=1)


if __name__ == "__main__":
    main()
