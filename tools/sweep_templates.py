"""Row-template SpMV kernel: shape sweep, plan-build cost and host dispatch cost on the benchmark's operator.

    python tools/sweep_templates.py [--launches 200] [--reps 5] [--out DIR]

One process, one GPU.
  * Sweep: the 5-point Laplacian on a 3162 x 3162 grid (fp64 and fp32), one plan, the kernel shape switched with the
    tuning hook b2s_spmv_set_template_config -- rows per lane R in {1, 2}, 128 / 256 threads per CTA, plain or
    evict-first y stores -- next to the coded tile kernel of the same plan (b2s_spmv_plan_set_packed 2), in alternating
    rounds of `--launches` back-to-back launches timed with CUDA events.  As a control, the same kernel on a 1-D 3-point
    Laplacian with as many rows, whose x reuse stays in L1 / L2 by construction.
  * Plan build: wall time of plan creation, value coding and template detection (each ends in a host sync), median of 3.
  * Host dispatch: host time per dist_csr_array.dot enqueue at world size 1 (1,000 calls back to back, no sync inside),
    next to the device time per call.
  * Pipeline sweep: tools/sweep_templates_kernels.cu, compiled into a temporary directory, builds the kernel at every
    pipeline depth D in {1, 2, 3} and launch bound of 4, 5, 6 or 8 CTAs of 256 threads per SM, at R in {1, 2}; each is
    timed on fp64 and fp32 L5 (and at R = 1 on the fp64 control) with its registers and spill bytes from ptxas.
  * Copy ceiling: y.copy_(x) on as many fp64 elements as L5 has rows plus a read of one byte per row (two torch
    launches), timed like the kernels.
  * Native ceiling: one launch of a streaming kernel on the template kernel's grid (one resident wave of 256-thread CTAs,
    32-element chunks per warp) that copies as many fp64 elements as L5 has rows and reads m more bytes: at m = nrows
    (one id per row) and at m = the fp64 L5 plan's code and mixed-group id bytes -- the template kernel's traffic with no
    gathers and nothing to wait for.
Moved bytes of the template kernel: one code byte per 32-row group, 32 id bytes per mixed group, x and y once, the
table per CTA (from L2).  The card's name and power limit are printed with the numbers.
"""
import ctypes
import re
import subprocess
import tempfile
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import legate.sparse_b200 as sparse  # noqa: E402
from legate.sparse_b200 import _lib, _ops, gallery  # noqa: E402
from legate.sparse_b200 import dist as bd  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_packed import card, time_per_launch  # noqa: E402


def build_sweep_lib(tmp):
    """The sweep's kernels as a shared object under tmp, and {(value, R, D, MINB): (registers, spill bytes)}."""
    here = os.path.dirname(os.path.abspath(__file__))
    so = os.path.join(tmp, "libsweep_templates.so")
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
           "-Xptxas", "-v", "-I", os.path.join(os.path.dirname(here), "include"),
           os.path.join(here, "sweep_templates_kernels.cu"), _lib.lib._name, "-o", so]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    regs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"(?:Compiling entry function '|Function properties for )(_Z\w+)", line)
        if m:
            k = re.search(r"spmv_template_kernelI([fd])Li5ELi(\d)ELi256ELi(\d)ELi(\d)ELb0E", m.group(1))
            cur = ("fp64" if k.group(1) == "d" else "fp32",) + tuple(int(g) for g in k.groups()[1:]) if k else None
            continue
        if cur is None:
            continue
        if (m := re.search(r"(\d+) bytes spill stores", line)):
            regs.setdefault(cur, [0, 0])[1] = int(m.group(1))
        if (m := re.search(r"Used (\d+) registers", line)):
            regs.setdefault(cur, [0, 0])[0] = int(m.group(1))
    lib = ctypes.CDLL(so)
    lib.sweep_template_launch.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int] + \
        [ctypes.c_void_p] * 3
    lib.sweep_stream_ceiling.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]
    return lib, regs


def set_shape(rows, threads, streaming):
    _lib.check(_lib.lib.b2s_spmv_set_template_config(rows, threads, streaming), "b2s_spmv_set_template_config")


def plan_build_ms(A):
    out = {}
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        plan = _ops.spmv_plan(A.indptr, A.indices, A.shape, A.nnz, A.dtype)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        plan = _ops.spmv_plan_code(plan, A.indptr, A.indices, A.data)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        plan = _ops.spmv_plan_templates(plan, A.indptr, A.indices, A.data)
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        for k, v in (("create", t1 - t0), ("code", t2 - t1), ("templates", t3 - t2)):
            out.setdefault(k, []).append(v * 1e3)
    return {k: float(np.median(v)) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sweep_templates.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    n = 3162 * 3162
    mats = {
        "l5_fp64": gallery.laplacian_5pt(3162, 3162, np.float64),
        "l5_fp32": gallery.laplacian_5pt(3162, 3162, np.float32),
        "l3_1d_fp64": sparse.diags([-1.0, 2.0, -1.0], [-1, 0, 1], shape=(n, n), format="csr", dtype=np.float64),
    }
    shapes = [(r, t, s) for r in (1, 2) for t in (128, 256) for s in (0, 1)]
    tmp = tempfile.mkdtemp(prefix="sweep_templates_")
    sweep, regs = build_sweep_lib(tmp)
    cases = {}
    id_bytes = {}
    for name, A in mats.items():
        plan = A._get_plan()
        assert plan.templated, (name, plan.kernel_name)
        x = torch.rand(A.shape[1], dtype=A.data.dtype, device="cuda")
        y = torch.empty(A.shape[0], dtype=A.data.dtype, device="cuda")

        def run(A=A, plan=plan, x=x, y=y):
            _ops.spmv(A.indptr, A.indices, A.data, x, y, A.shape, plan=plan)

        sv = A.data.element_size()
        _, codes = plan.template_sections(A.shape[0])
        mixed = int((codes == 0xFF).sum())
        id_bytes[name] = dict(groups=codes.numel(), mixed=mixed, bytes=codes.numel() + 32 * mixed)
        moved = id_bytes[name]["bytes"] + A.shape[0] * sv + A.shape[1] * sv
        for shp in shapes if name != "l3_1d_fp64" else [(0, 0, 0)]:
            cases[f"{name}_tpl_R{shp[0]}_T{shp[1]}_{'cs' if shp[2] else 'st'}"] = dict(
                run=run, plan=plan, mode=3, shape=shp, moved=moved, flops=2 * A.nnz)
        vt = name.split("_")[-1]
        for (v, r, d, m), (nreg, spill) in sorted(regs.items()):
            if v != vt or (name == "l3_1d_fp64" and r != 1):
                continue

            def run_pipe(plan=plan, x=x, y=y, A=A, key=(v, r, d, m)):
                _lib.check(sweep.sweep_template_launch(int(key[0] == "fp64"), key[2], key[3], key[1],
                                                       plan.tpl_buf.data_ptr(), A.shape[0], 5, x.data_ptr(),
                                                       y.data_ptr(), torch.cuda.current_stream().cuda_stream),
                           "sweep_template_launch")
            cases[f"{name}_pipe_R{r}_D{d}_M{m}"] = dict(run=run_pipe, plan=plan, mode=3, shape=(0, 0, 0), moved=moved,
                                                        flops=2 * A.nnz, regs=nreg, spill=spill)
        if plan.coded:
            cases[f"{name}_coded"] = dict(run=run, plan=plan, mode=2, shape=(0, 0, 0), moved=None, flops=2 * A.nnz)

    def select(c):
        c["plan"].set_packed(c["mode"])
        set_shape(*c["shape"])

    for c in cases.values():
        select(c)
        for _ in range(10):
            c["run"]()
    torch.cuda.synchronize()
    times = {k: [] for k in cases}
    for _ in range(args.reps):
        for k, c in cases.items():
            select(c)
            c["run"]()
            times[k].append(time_per_launch(c["run"], args.launches))
    set_shape(0, 0, 0)
    for c in cases.values():
        c["plan"].set_packed(3)

    probe = torch.rand(200_000_000, dtype=torch.float64, device="cuda")   # 1.6 GB
    probe.sum()
    pt = [time_per_launch(lambda: probe.sum(), 50) for _ in range(3)]
    ceiling = probe.numel() * 8 / float(np.median(pt))
    del probe
    # copy ceiling of the fp64 L5 template traffic: x read, y written, one byte per row read
    xc = torch.rand(n, dtype=torch.float64, device="cuda")
    yc = torch.empty_like(xc)
    idc = torch.zeros(n // 8, dtype=torch.int64, device="cuda")   # n bytes

    def copy_and_ids():
        yc.copy_(xc)
        idc.sum()
    copy_and_ids()
    ct = [time_per_launch(copy_and_ids, args.launches) for _ in range(args.reps)]
    copy_bytes = n * 8 * 2 + idc.numel() * 8
    copy_ceiling = copy_bytes / float(np.median(ct))
    # the native ceiling, one launch on the template kernel's grid, at the parent's and this kernel's id traffic
    sink = torch.zeros(4, dtype=torch.int32, device="cuda")
    native = {}
    for label, m in (("one id per row", n), ("group codes", id_bytes["l5_fp64"]["bytes"])):
        mb = torch.zeros((m + 15) // 16 * 16, dtype=torch.uint8, device="cuda")

        def stream(mb=mb):
            _lib.check(sweep.sweep_stream_ceiling(n, xc.data_ptr(), yc.data_ptr(), mb.data_ptr(), mb.numel(),
                                                  sink.data_ptr(), torch.cuda.current_stream().cuda_stream),
                       "sweep_stream_ceiling")
        stream()
        nt = float(np.median([time_per_launch(stream, args.launches) for _ in range(args.reps)]))
        native[label] = dict(m_bytes=mb.numel(), us=nt * 1e6, moved_bytes=n * 16 + mb.numel(),
                             tbs=(n * 16 + mb.numel()) / nt / 1e12)
        del mb
    del xc, yc, idc

    gname, limit = card()
    print(f"# {gname}, power limit {limit} W; {args.launches} launches x {args.reps} alternating rounds per case")
    print(f"# streaming ceiling (probe) {ceiling / 1e12:.3f} TB/s")
    print(f"# copy ceiling: y.copy_(x) on {n} fp64 + {n} bytes read: {float(np.median(ct)) * 1e6:.1f} us, "
          f"{copy_bytes / 1e6:.1f} MB, {copy_ceiling / 1e12:.3f} TB/s")
    for label, v in native.items():
        print(f"# native ceiling ({label}): copy of {n} fp64 + {v['m_bytes'] / 1e6:.2f} MB read, one launch: "
              f"{v['us']:.1f} us, {v['moved_bytes'] / 1e6:.1f} MB, {v['tbs']:.3f} TB/s")
    for name, v in id_bytes.items():
        print(f"# {name}: {v['groups']} groups, {v['mixed']} mixed ({100 * v['mixed'] / v['groups']:.2f} %), "
              f"{v['bytes'] / 1e6:.2f} MB of codes and ids")
    native_tbs = native["group codes"]["tbs"] * 1e12
    rows = {}
    for k, c in cases.items():
        ts = sorted(times[k])
        t = float(np.median(ts))
        row = {"us_median": t * 1e6, "us_min": ts[0] * 1e6, "us_max": ts[-1] * 1e6, "gflops": c["flops"] / t / 1e9}
        if c["moved"]:
            row.update(moved_bytes=c["moved"], moved_tbs=c["moved"] / t / 1e12, moved_frac_of_probe=c["moved"] / t / ceiling,
                       moved_frac_of_copy=c["moved"] / t / copy_ceiling, moved_frac_of_native=c["moved"] / t / native_tbs)
        if "regs" in c:
            row.update(registers=c["regs"], spill_bytes=c["spill"])
        rows[k] = row
        mv = f"  moved {c['moved'] / 1e6:6.1f} MB {row['moved_tbs']:.3f} TB/s = {row['moved_frac_of_probe']:.3f} of probe" \
             f", {row['moved_frac_of_copy']:.3f} of copy, {row['moved_frac_of_native']:.3f} of native" \
            if c["moved"] else ""
        if "regs" in c:
            mv += f"  [{c['regs']} regs, {c['spill']} B spilled]"
        print(f"{k:28s} {t * 1e6:8.1f} us [{ts[0] * 1e6:.1f}..{ts[-1] * 1e6:.1f}]  {row['gflops']:7.1f} GFLOP/s{mv}")

    build = {name: plan_build_ms(A) for name, A in mats.items() if name != "l3_1d_fp64"}
    for name, b in build.items():
        print(f"# plan build {name}: create {b['create']:.2f} ms, code {b['code']:.2f} ms, templates {b['templates']:.2f} ms")

    # host dispatch of dist_csr_array.dot at world size 1 (the call bench.py times)
    local = mats["l5_fp64"]
    D = bd.dist_csr_array(local, local.shape, rank=0, nranks=1)
    x_full = D.new_full_vector(np.float64)
    D.local_view(x_full).copy_(torch.rand(local.shape[0], dtype=torch.float64, device="cuda"))
    y = torch.empty(local.shape[0], dtype=torch.float64, device="cuda")
    for _ in range(20):
        D.dot(x_full, out=y)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    t0 = time.perf_counter()
    for _ in range(1000):
        D.dot(x_full, out=y)
    host_us = (time.perf_counter() - t0) * 1e3
    e.record()
    torch.cuda.synchronize()
    dev_us = s.elapsed_time(e)
    print(f"# dist_csr_array.dot world 1: host {host_us:.2f} us per enqueue, device {dev_us:.2f} us per call "
          f"(1000 calls; {D.local._get_plan().kernel_name})")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sweep_templates.json"), "w") as f:
            json.dump({"gpu": gname, "power_limit_w": limit, "launches": args.launches, "reps": args.reps,
                       "probe_tbs": ceiling / 1e12,
                       "copy_ceiling_tbs": copy_ceiling / 1e12, "copy_ceiling_us": float(np.median(ct)) * 1e6,
                       "native_ceiling": native, "template_id_bytes": id_bytes, "cases": rows, "plan_build_ms": build,
                       "dot_host_us_per_enqueue": host_us, "dot_device_us_per_call": dev_us}, f, indent=1)


if __name__ == "__main__":
    main()
