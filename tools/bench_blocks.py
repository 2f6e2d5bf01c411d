"""1-GPU experiment behind the column-blocked all-gather SpMV (dist._fused_setup 'blocks'): the R32 shard of rank 0 of a
P-rank run (10M/P rows x 10M columns, 32 per row), split into P column blocks; per-block accumulating SpMV under each
kernel flavour / tile config vs the unsplit shard.  Says which path the blocks should take.
    python tools/bench_blocks.py [P ...]"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from legate.sparse_b200 import _lib, _ops, gallery  # noqa: E402
from legate.sparse_b200.csr import _column_blocks  # noqa: E402


def time_fn(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for s, e in ev:
        s.record(); fn(); e.record()
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) for s, e in ev)
    return ts[len(ts) // 2] * 1e3


def blocks_of(A, P):
    n = A.shape[1]
    T = (n + P - 1) // P
    return _column_blocks(A, [(q * T, min((q + 1) * T, n)) for q in range(P)])


def l2_gran(set_bytes=0):
    import ctypes
    cur = ctypes.c_int64(0)
    _lib.check(_lib.lib.b2s_device_l2_fetch_granularity(set_bytes, ctypes.byref(cur)))
    return cur.value


def gran_sweep(P):
    """--l2gran: the weak-scaled shard (x = 40 MB * P) unsplit and in column blocks under each L2 fetch granularity."""
    n = 10_000_000 * P
    rows = 10_000_000
    A = gallery.random_fixed(rows, n, 32, np.float32, seed=1234)
    x = torch.rand(n, dtype=torch.float32, device="cuda")
    y = torch.zeros(rows, dtype=torch.float32, device="cuda")
    plan = A._get_plan()
    blocks = blocks_of(A, P)
    plans = [B._get_plan(tma_only=True) for B in blocks]
    print(f"l2 fetch granularity at start: {l2_gran()} bytes", flush=True)
    for g in (128, 64, 32, 128):
        got = l2_gran(g)
        t_un = time_fn(lambda: _ops.spmv(A.indptr, A.indices, A.data, x, y, A.shape, plan=plan), reps=10)
        tot = 0.0
        for B, pl in zip(blocks, plans):
            tot += time_fn(lambda: _ops.spmv_add(B.indptr, B.indices, B.data, x, y, B.shape, pl), reps=10)
        print(f"P={P} weak, l2 fetch granularity set {g} -> {got}: unsplit {t_un:8.1f} us ({plan.kernel_name}), "
              f"{P} blocks {tot:8.1f} us ({plans[0].kernel_name})", flush=True)


def main():
    if "--l2gran" in sys.argv:
        for P in [int(a) for a in sys.argv[1:] if not a.startswith("--")] or [8]:
            gran_sweep(P)
        return
    weak = "--weak" in sys.argv          # 10M rows per shard, 10M*P columns (weak scaling) instead of 10M/P rows x 10M
    one = "--one-block" in sys.argv      # profile mode: only block 1, default plan, 3 launches (target of ncu)
    Ps = [int(a) for a in sys.argv[1:] if not a.startswith("--")] or [2, 4, 8]
    nblk = [int(a.split("=")[1]) for a in sys.argv[1:] if a.startswith("--nblocks=")]   # column blocks != ranks
    cfgs = [int(c) for a in sys.argv[1:] if a.startswith("--cfgs=") for c in a.split("=")[1].split(",")]
    flavors = [None, 0, 1, 2] if "--all-flavors" in sys.argv or not weak else [None]
    for P in Ps:
        n = 10_000_000 * (P if weak else 1)
        rows = 10_000_000 if weak else n // P
        A = gallery.random_fixed(rows, n, 32, np.float32, seed=1234)
        x = torch.rand(n, dtype=torch.float32, device="cuda")
        y = torch.zeros(rows, dtype=torch.float32, device="cuda")
        plan = A._get_plan()
        t_unsplit = 0.0 if one else time_fn(lambda: _ops.spmv(A.indptr, A.indices, A.data, x, y, A.shape, plan=plan))
        print(f"P={P} shard {rows} rows: unsplit {plan.kernel_name}: {t_unsplit:8.1f} us", flush=True)
        Q = nblk[0] if nblk else P
        blocks = blocks_of(A, Q)
        if one:
            B = blocks[1]
            pl = B._get_plan(tma_only=True)
            for _ in range(3):
                _ops.spmv_add(B.indptr, B.indices, B.data, x, y, B.shape, pl)
            torch.cuda.synchronize()
            print("profiled", pl.kernel_name, B.nnz, flush=True)
            return
        for cfg in (cfgs or ((-1, 8) if weak else (-1, 5, 8, 3, 0))):
            _lib.check(_lib.lib.b2s_spmv_set_config(cfg, 0))
            for flavor in flavors:
                tot, names = 0.0, set()
                for B in blocks:
                    pl = B._get_plan(tma_only=True)     # a new config builds a new plan
                    if flavor is not None:
                        pl.set_flavor(flavor)
                    names.add(pl.kernel_name)
                    tot += time_fn(lambda: _ops.spmv_add(B.indptr, B.indices, B.data, x, y, B.shape, pl), reps=10)
                print(f"   cfg {cfg:2d} flavor {str(flavor):4s}: sum over {Q} blocks {tot:8.1f} us   ({sorted(names)[0]})", flush=True)
        _lib.check(_lib.lib.b2s_spmv_set_config(-1, 0))
        del A, blocks, x, y
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
