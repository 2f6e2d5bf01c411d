"""Multi-GPU: 1-D row-block sharding of CSR matrices and vectors, one process per GPU.

Replaces the reference's partitioning layer (sparse/partition.py, sparse/csr.py:238-246, spmv()
:930-968) and Legion's implicit copies with an explicit static plan:

* rows   : rank p owns rows [p*T, min((p+1)*T, N)), T = ceil(N/P)            (csr.py:242-245)
* nnz    : the contiguous indices/vals slice [indptr[p*T], indptr[(p+1)*T))   (CompressedImagePartition,
           partition.py:56-128) with indptr rebased to 0
* x      : each shard reads x only inside its column window [min col, max col] (MinMaxImagePartition,
           partition.py:139-208).  Before an SpMV every rank fills that window of its full-length x
           buffer: either by an all-gather of the T-padded shards (dense/random matrices) or by point-to-
           point pieces of exactly the window (stencil/banded matrices: two halo messages).
* scalars: CG dot products are all-reduced (sum) as 1-element device tensors; they never visit the host
           between convergence checks (linalg.py:539-555 keeps them in futures).  On GPUs of one box the
           reduction is the one-shot NVLink peer-memory kernel of csrc/peer.cu (PeerComm), NCCL otherwise.
* SpGEMM : B all-gathered once, C row-sharded (`spgemm`); rows can also be cut nnz-balanced
           (`RowBlockPlan.balanced`, the reference's `balance()`).

Plumbing goes through `torch.distributed` (NCCL on GPUs; gloo on CPU for the host-logic tests) and CUDA IPC for
the peer buffers.  The local compute is always the C-ABI kernels via `_ops`.
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.distributed as dist

from . import _ops
from .csr import _column_blocks, _indptr_dtype, csr_array
from .runtime import numpy_dtype, runtime, to_device, to_host, torch_dtype


def init_process_group(backend: str | None = None) -> None:
    """Initialise torch.distributed from the torchrun environment (RANK/WORLD_SIZE/LOCAL_RANK/MASTER_*)
    and bind this process to its GPU.  The reference does the equivalent at import when more than one GPU is
    present (sparse/runtime.py:84-87)."""
    if dist.is_initialized():
        return
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29512")
    kwargs = {}
    if backend == "nccl":
        kwargs["device_id"] = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group(backend=backend, **kwargs)


def world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


class RowBlockPlan:
    """Static 1-D row-block partition of N rows over P ranks.

    Default: equal row tiles, T = ceil(N/P) (reference sparse/csr.py:238-246).  `balanced()` instead cuts the
    rows so every rank holds about nnz/P nonzeros -- the reference's `csr_array.balance()` (sparse/base.py:198-282:
    equal nnz tiles, preimage to rows, made disjoint), which matters for power-law matrices."""

    def __init__(self, nrows: int, nranks: int, bounds=None):
        self.nrows = int(nrows)
        self.nranks = int(nranks)
        if bounds is None:
            t = (self.nrows + self.nranks - 1) // self.nranks if self.nranks > 0 else 0
            bounds = [min(r * t, self.nrows) for r in range(self.nranks + 1)]
            self.uniform = True
            self.tile = t
        else:
            bounds = [int(b) for b in bounds]
            assert len(bounds) == self.nranks + 1 and bounds[0] == 0 and bounds[-1] == self.nrows
            assert all(b1 >= b0 for b0, b1 in zip(bounds, bounds[1:]))
            self.uniform = False
            self.tile = max([b1 - b0 for b0, b1 in zip(bounds, bounds[1:])] + [0])
        self.bounds = bounds

    @classmethod
    def balanced(cls, indptr, nranks: int):
        """Row cuts at the first row whose starting nonzero reaches k*nnz/P."""
        ip = np.asarray(to_host(indptr)).astype(np.int64)
        nrows, nnz = ip.shape[0] - 1, int(ip[-1])
        targets = [(k * nnz) // nranks for k in range(1, nranks)]
        cuts = [int(np.searchsorted(ip, t, side="left")) for t in targets]
        bounds = [0] + [min(max(c, 0), nrows) for c in cuts] + [nrows]
        for k in range(1, len(bounds)):
            bounds[k] = max(bounds[k], bounds[k - 1])
        return cls(nrows, nranks, bounds)

    def rows(self, rank: int):
        return self.bounds[rank], self.bounds[rank + 1]

    def owner(self, row: int) -> int:
        return max(0, min(int(np.searchsorted(self.bounds, row, side="right")) - 1, self.nranks - 1))

    @property
    def padded(self) -> int:
        return max(self.tile * self.nranks, self.nrows)


def _intersect(a_lo, a_hi, b_lo, b_hi):
    lo, hi = max(a_lo, b_lo), min(a_hi, b_hi)
    return (lo, hi) if hi > lo else None


class _RawCudaBuffer:
    """Zero-copy view of a raw device allocation as a torch tensor (via __cuda_array_interface__)."""

    def __init__(self, ptr: int, nelems: int, np_dtype):
        self.__cuda_array_interface__ = {
            "shape": (int(nelems),),
            "typestr": np.dtype(np_dtype).str,
            "data": (int(ptr), False),
            "version": 3,
            "strides": None,
        }


class PeerComm:
    """NVLink peer-memory communicator of one box: every rank allocates one IPC-shareable buffer
    [header | x vector], maps the other ranks' buffers, and then exchanges halos / all-reduces scalars with
    plain remote stores + epoch flags (csrc/peer.cu) instead of NCCL calls.  Collective constructor."""

    def __init__(self, x_elems: int, np_dtype, rank: int, nranks: int, group=None):
        from . import _lib

        self.rank, self.nranks = rank, nranks
        self.dtype = np.dtype(np_dtype)
        self.header = int(_lib.lib.b2s_peer_header_bytes())
        self.x_elems = int(x_elems)
        nbytes = self.header + (self.x_elems + 8) * self.dtype.itemsize
        # Every rank takes part in every collective below even if one of its own steps fails (`ok` is agreed on by
        # the caller with an all-reduce, which is also the barrier that orders the mappings before first use).
        self.ok = True
        self.own, self.peers, self._opened = 0, [], []
        self.x_base = self._keep = None
        handle = None
        try:
            self.own = _ops.ipc_alloc(nbytes)
            handle = _ops.ipc_export(self.own)
        except Exception:
            self.ok = False
        handles = [None] * nranks
        dist.all_gather_object(handles, handle, group=group)
        if self.ok and all(h is not None for h in handles):
            try:
                for q in range(nranks):
                    if q == rank:
                        self.peers.append(self.own)
                    else:
                        p = _ops.ipc_open(handles[q])
                        self._opened.append(p)
                        self.peers.append(p)
                self._keep = _RawCudaBuffer(self.own + self.header, self.x_elems + 8, self.dtype)
                self.x_base = torch.as_tensor(self._keep, device=runtime.device)
            except Exception:
                self.ok = False
        else:
            self.ok = False

    def allreduce(self, t: torch.Tensor) -> torch.Tensor:
        return _ops.peer_allreduce(t, self.rank, self.peers)

    # addresses of the fused-protocol words (PeerHeader::fuse_*, csrc/peer.cu) in my header or in a peer's
    def _word(self, which: int, idx: int = 0, peer: int | None = None) -> int:
        from . import _lib

        base = self.own if peer is None else self.peers[peer]
        return base + int(_lib.lib.b2s_peer_header_offset(which, idx))

    def flag_local(self, src: int) -> int:        # written by `src` when its slice has landed here
        return self._word(0, src)

    def flag_remote(self, dst: int) -> int:       # my arrival word in dst's header
        return self._word(0, self.rank, dst)

    def ack_local(self, dst: int) -> int:         # written by `dst` when it has consumed my previous slice
        return self._word(2, dst)

    def ack_remote(self, src: int) -> int:        # my acknowledgement word in src's header
        return self._word(2, self.rank, src)

    @property
    def epoch_ctr(self) -> int:
        return self._word(3)

    @property
    def ticket(self) -> int:
        return self._word(4)

    @property
    def error_word(self) -> int:
        return self._word(1)

    def x_remote(self, peer: int, elem: int) -> int:
        """Device address (peer-mapped) of element `elem` of `peer`'s full-length x vector."""
        return self.peers[peer] + self.header + (self.peer_x_off[peer] + elem) * self.dtype.itemsize

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self):
        if _ops.peer_check(self.own):
            raise RuntimeError("NVLink peer exchange timed out waiting for another rank (PeerHeader.error set)")

    def close(self):
        for p in self._opened:
            try:
                _ops.ipc_close(p)
            except Exception:
                pass
        self._opened = []
        if self.own:
            self.x_base = None
            self._keep = None
            try:
                _ops.ipc_free(self.own)
            except Exception:
                pass
            self.own = 0


class dist_csr_array:
    """A row shard of a global square-or-rectangular CSR matrix.

    `local` holds rows [row_lo, row_hi) with GLOBAL column ids.  Vectors are sharded the same way
    (ncols is partitioned by the same plan as nrows for the square matrices of the hot path; for
    rectangular ones x is partitioned by its own RowBlockPlan over ncols)."""

    def __init__(self, local: csr_array, global_shape, rank=None, nranks=None, group=None, row_plan=None):
        r, w = world()
        self.rank = r if rank is None else rank
        self.nranks = w if nranks is None else nranks
        self.group = group
        self.local = local
        self.shape = tuple(int(s) for s in global_shape)
        self.dtype = local.dtype
        self.row_plan = RowBlockPlan(self.shape[0], self.nranks) if row_plan is None else row_plan
        # vectors are sharded like the rows when the matrix is square (CG); otherwise by equal tiles of ncols
        self.col_plan = self.row_plan if self.shape[0] == self.shape[1] else RowBlockPlan(self.shape[1], self.nranks)
        self.row_lo, self.row_hi = self.row_plan.rows(self.rank)
        assert local.shape == (self.row_hi - self.row_lo, self.shape[1]), (local.shape, self.shape)
        self._xbuf = {}
        self._build_exchange()

    # -- construction -------------------------------------------------------------------------------
    @classmethod
    def from_global(cls, A, rank=None, nranks=None, balanced=False):
        """Slice this rank's shard out of a replicated global matrix (scipy CSR or csr_array). Used by
        tests and small problems; large runs assemble shards directly (gallery.*(row_lo=, row_hi=))."""
        import scipy.sparse as sp

        r, w = world()
        rank = r if rank is None else rank
        nranks = w if nranks is None else nranks
        S = A.to_scipy_sparse_csr() if isinstance(A, csr_array) else sp.csr_array(A)
        plan = RowBlockPlan.balanced(S.indptr, nranks) if balanced else RowBlockPlan(S.shape[0], nranks)
        lo, hi = plan.rows(rank)
        klo, khi = int(S.indptr[lo]), int(S.indptr[hi])
        local = csr_array((S.data[klo:khi], S.indices[klo:khi], S.indptr[lo : hi + 1] - klo),
                          shape=(hi - lo, S.shape[1]))
        return cls(local, S.shape, rank=rank, nranks=nranks, row_plan=plan)

    @classmethod
    def from_triplets(cls, data, row, col, shape, rank=None, nranks=None, group=None):
        """Assemble the row shards from COO triplets scattered over the ranks in any order (each rank passes the
        triplets it happens to hold, global row / column ids).  The reference does this with a distributed
        sort-by-key over NCCL followed by counts -> pos (sparse/coo.py:233-347, src/sparse/sort/sort.cu,
        base.py:30-48).  Here the splitters are known -- the row blocks of the partition -- so one exchange
        routes every triplet to the owner of its row (counts all-gathered, then grouped point-to-point
        send/recv of the three arrays) and each rank sorts what it received by (row, col) on its own device
        (`coo_array.tocsr`).  Duplicates are assumed absent, as in the reference."""
        from .coo import coo_array

        r, w = world()
        rank = r if rank is None else rank
        nranks = w if nranks is None else nranks
        shape = tuple(int(s) for s in shape)
        plan = RowBlockPlan(shape[0], nranks)
        dev = runtime.device
        vals = to_device(data).reshape(-1)
        rows = to_device(row).reshape(-1).to(torch.int64)
        cols = to_device(col).reshape(-1).to(torch.int64)
        dest = torch.clamp(rows // max(plan.tile, 1), max=nranks - 1)
        order = torch.sort(dest, stable=True).indices
        vals, rows, cols = vals[order], rows[order], cols[order]
        send_counts = torch.bincount(dest, minlength=nranks).to(torch.int64)
        if nranks > 1:
            all_counts = torch.empty(nranks * nranks, dtype=torch.int64, device=dev)
            dist.all_gather_into_tensor(all_counts, send_counts, group=group)
            all_counts = all_counts.reshape(nranks, nranks).cpu()      # [sender, receiver]
            recv_counts = [int(all_counts[q, rank]) for q in range(nranks)]
            send_off = np.concatenate([[0], np.cumsum(send_counts.cpu().numpy())])
            pieces = {}
            for name, arr in (("vals", vals), ("rows", rows), ("cols", cols)):
                recv = [torch.empty(c, dtype=arr.dtype, device=dev) for c in recv_counts]
                ops = []
                for q in range(nranks):
                    if q == rank:
                        recv[q] = arr[send_off[q]:send_off[q + 1]]
                        continue
                    if recv_counts[q]:
                        ops.append(dist.P2POp(dist.irecv, recv[q], q, group=group))
                    if send_off[q + 1] > send_off[q]:
                        ops.append(dist.P2POp(dist.isend, arr[send_off[q]:send_off[q + 1]].contiguous(), q, group=group))
                if ops:
                    for req in dist.batch_isend_irecv(ops):
                        req.wait()
                pieces[name] = torch.cat(recv)
            vals, rows, cols = pieces["vals"], pieces["rows"], pieces["cols"]
        lo, hi = plan.rows(rank)
        local = coo_array((vals, (rows - lo, cols)), shape=(hi - lo, shape[1])).tocsr()
        return cls(local, shape, rank=rank, nranks=nranks, group=group, row_plan=plan)

    # -- exchange plan --------------------------------------------------------------------------------
    def _build_exchange(self):
        """Column window of this shard + who sends what to whom."""
        idx = self.local.indices
        if idx.numel():
            lo, hi = int(idx.min()), int(idx.max()) + 1
        else:
            lo, hi = 0, 0
        self.window = (lo, hi)
        wins = [None] * self.nranks
        if self.nranks > 1:
            dist.all_gather_object(wins, (lo, hi), group=self.group)
        else:
            wins[0] = (lo, hi)
        self.windows = wins
        my_lo, my_hi = self.col_plan.rows(self.rank)
        self.my_cols = (my_lo, my_hi)
        # pieces of MY x rows that peer q reads; pieces of q's x rows that I read
        self.sends = []
        self.recvs = []
        for q in range(self.nranks):
            if q == self.rank:
                continue
            s = _intersect(*wins[q], my_lo, my_hi) if wins[q][1] > wins[q][0] else None
            if s:
                self.sends.append((q, s[0], s[1]))
            qlo, qhi = self.col_plan.rows(q)
            r = _intersect(lo, hi, qlo, qhi) if hi > lo else None
            if r:
                self.recvs.append((q, r[0], r[1]))
        need = sum(b - a for _, a, b in self.recvs)
        total_need = need
        if self.nranks > 1:
            t = torch.tensor([need], dtype=torch.int64, device=self._comm_device())
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
            total_need = int(t.item())
        mode = os.environ.get("B2S_EXCHANGE", "auto")
        if mode == "auto":
            # all-gather moves (P-1)*T elements into every rank; use p2p windows when they are much smaller
            mode = "p2p" if total_need * 4 < (self.nranks - 1) * self.col_plan.tile else "allgather"
        if not self.col_plan.uniform and mode == "allgather":
            mode = "p2p"  # the in-place all-gather needs equal shards; uneven (balanced) plans exchange windows
        self.exchange_mode = mode if self.nranks > 1 else "none"
        self.recv_elems = need
        # NVLink peer-memory path (csrc/peer.cu), for ranks that are CUDA devices of ONE box (CUDA IPC):
        #   B2S_PEER=1 (default)   CG scalars are all-reduced by the one-shot peer kernel, and the x exchange is
        #                          FUSED into the SpMV kernel: a halo is pushed / awaited by the SpMV launch itself
        #                          (`_fused_halo`), an all-gather becomes b2s_peer_push + one column block per
        #                          source rank, each waiting in-kernel for its own slice (`_fused_blocks`).
        #                          Device-side epochs: the whole step replays from a CUDA graph.
        #   B2S_PEER_FUSED=0       keep the peer all-reduce but exchange x with NCCL (the round-1 path)
        #   B2S_PEER_HALO=1        explicit `exchange()` calls push halos with peer kernels instead of NCCL p2p
        self._peer = {}
        self._fused = {}
        peer_ok = self.nranks > 1 and runtime.has_cuda and self.nranks <= 16
        if peer_ok:
            import socket

            hosts = [None] * self.nranks
            dist.all_gather_object(hosts, socket.gethostname(), group=self.group)
            peer_ok = len(set(hosts)) == 1       # CUDA IPC maps memory of GPUs in the same box only
        self.use_peer = peer_ok and os.environ.get("B2S_PEER", "1") != "0"
        self.use_peer_halo = self.use_peer and os.environ.get("B2S_PEER_HALO", "0") == "1"
        self.use_fused = self.use_peer and os.environ.get("B2S_PEER_FUSED", "1") != "0"
        blocks_min = os.environ.get("B2S_BLOCKS_MIN_BYTES")   # read once, at construction; default 3/8 of L2
        self._blocks_min = None if blocks_min is None else int(blocks_min)

    def _comm_device(self):
        return runtime.device

    # -- vectors ----------------------------------------------------------------------------------------
    def _peer_comm(self, np_dtype):
        key = np.dtype(np_dtype)
        pc = self._peer.get(key)
        if pc is None:
            n = max(self.col_plan.padded, 1)
            pc = PeerComm(n, key, self.rank, self.nranks, self.group)
            ok = 1 if pc.ok else 0   # no peer access between some pair of GPUs, IPC refused, out of memory ...
            flag = torch.tensor([ok], dtype=torch.int32, device=self._comm_device())
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
            if int(flag.item()) == 0:      # some rank failed: everybody falls back to NCCL, consistently
                if pc is not None:
                    pc.close()
                self.use_peer = self.use_peer_halo = self.use_fused = False
                return None
            per16 = 16 // key.itemsize
            pc.x_off = (-self.my_cols[0]) % per16  # own slice starts 16-byte aligned
            offs = [None] * self.nranks
            dist.all_gather_object(offs, pc.x_off, group=self.group)
            pc.peer_x_off = offs
            pc.x_full = pc.x_base[pc.x_off : pc.x_off + n]
            self._peer[key] = pc
        return pc

    def new_full_vector(self, dtype=None) -> torch.Tensor:
        """Full-length x buffer (padded to P*T so the all-gather lands in place).  The buffer is offset
        inside its allocation so that this rank's own slice starts 16-byte aligned (the vector kernels
        then take their 128-bit path on the shard views).  With the peer path enabled the buffer lives in
        this rank's IPC allocation (one per dtype, reused) so neighbours can push their halo pieces into it."""
        np_dt = numpy_dtype(self.dtype if dtype is None else dtype)
        if self.use_peer_halo or self.use_fused:
            pc = self._peer_comm(np_dt)
            if pc is not None:
                pc.x_full.zero_()
                return pc.x_full
        dt = torch_dtype(np_dt)
        n = max(self.col_plan.padded, 1)
        base = torch.zeros(n + 4, dtype=dt, device=runtime.device)
        per16 = 16 // base.element_size()
        off = (-self.my_cols[0]) % per16
        return base[off : off + n]

    def local_view(self, full: torch.Tensor) -> torch.Tensor:
        lo, hi = self.my_cols
        return full[lo:hi]

    def scatter_vector(self, v_global) -> torch.Tensor:
        """This rank's shard of a replicated global vector (as a view into a fresh full buffer)."""
        full = self.new_full_vector(numpy_dtype(v_global.dtype) if hasattr(v_global, "dtype") else None)
        lo, hi = self.my_cols
        full[lo:hi] = to_device(v_global[lo:hi], dtype=numpy_dtype(full.dtype))
        return full

    def exchange(self, full: torch.Tensor) -> None:
        """Make full[window] valid on every rank, given that full[my_cols] is valid."""
        if self.exchange_mode == "none":
            return
        if self.exchange_mode == "allgather":
            assert self.col_plan.uniform
            T = self.col_plan.tile
            src = full[self.rank * T : (self.rank + 1) * T]
            dist.all_gather_into_tensor(full, src, group=self.group)
            return
        pc = self._peer.get(numpy_dtype(full.dtype)) if self.use_peer_halo else None
        if pc is not None and full.data_ptr() == pc.x_full.data_ptr():
            sends = [(q, a, pc.peer_x_off[q] + a, b - a) for q, a, b in self.sends]
            _ops.peer_halo_exchange(full, self.rank, pc.peers, sends, [q for q, _, _ in self.recvs])
            return
        ops = []
        for q, a, b in self.recvs:
            ops.append(dist.P2POp(dist.irecv, full[a:b], q, group=self.group))
        for q, a, b in self.sends:
            ops.append(dist.P2POp(dist.isend, full[a:b], q, group=self.group))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()

    # -- SpMV ---------------------------------------------------------------------------------------------
    def _overlap_schedule(self, plan=None):
        """Split an SpMV plan of the local shard into runs of tiles that only read locally owned x (can run while
        the halo is still in flight) and runs that touch remote columns (must wait for the exchange).  Uses the
        plan's row chunks and their column windows; None when the plan is not chunked."""
        plan = self.local._get_plan() if plan is None else plan
        cache = self.__dict__.setdefault("_scheds", {})
        key = id(plan)
        if key not in cache:
            lo, hi = self.my_cols
            interior, boundary = [], []
            for tile_lo, tile_hi, _, _, col_lo, col_hi in plan.chunks:
                if tile_hi <= tile_lo:
                    continue
                inside = col_hi <= col_lo or (col_lo >= lo and col_hi <= hi)
                runs = interior if inside else boundary
                if runs and runs[-1][1] == tile_lo:
                    runs[-1][1] = tile_hi
                else:
                    runs.append([tile_lo, tile_hi])
            cache[key] = (interior, boundary) if plan.chunks and interior else ()
        return cache[key] or None

    def _agree(self, ok: bool) -> bool:
        """True iff `ok` on every rank (the fused protocols deadlock unless all ranks take the same path)."""
        if self.nranks == 1:
            return bool(ok)
        t = torch.tensor([1 if ok else 0], dtype=torch.int32, device=self._comm_device())
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
        return bool(int(t.item()))

    def _fused_setup(self, A: csr_array, x_full: torch.Tensor):
        """One-time (collective) setup of the fused exchange for products of `A` (the local shard or a promoted copy
        of it) with the peer-resident vector `x_full`.  Returns a dict describing the path, or None (NCCL path).

        halo   (exchange_mode p2p): ONE launch per product -- `b2s_spmv_csr_fused` pushes this rank's boundary
               slices into the neighbours' x buffers, computes the interior tiles, and waits for the neighbours'
               slices only before its boundary tiles.
        blocks (exchange_mode allgather): the shard is cut at plan time into one CSR block per source rank (the
               columns that rank owns; the reference gets the same effect from Legion's image partitions,
               sparse/csr.py:930-968).  `b2s_peer_push` sends this rank's slice to everybody on a side stream while
               the own-column block is multiplied; each remote block is one accumulating launch that waits
               in-kernel for the arrival flag of ITS source only, so products start as slices land."""
        key = (id(A), x_full.data_ptr())
        if key in self._fused:
            return self._fused[key]
        info = None
        np_dt = numpy_dtype(x_full.dtype)
        pc = self._peer.get(np_dt) if self.use_fused else None
        usable = (pc is not None and x_full.is_cuda and x_full.data_ptr() == pc.x_full.data_ptr()
                  and A.dtype == np_dt and self.exchange_mode in ("p2p", "allgather"))
        item = np.dtype(np_dt).itemsize
        if self.exchange_mode == "p2p":
            plan = A._get_plan() if usable else None
            sched = self._overlap_schedule(plan) if usable and plan.tma else None
            if sched is not None and len(sched[0]) + len(sched[1]) > 6:
                sched = None
            ok = bool(usable and plan.tma and len(self.sends) <= 4 and len(self.recvs) <= 8)
            if self._agree(ok):
                if sched is None:      # plan too small to be chunked: every tile waits for the halo (no overlap)
                    ranges, n_free = [(0, plan.tiles)], (0 if self.recvs else 1)
                else:
                    ranges, n_free = [tuple(r) for r in sched[0] + sched[1]], len(sched[0])
                sends = [(x_full.data_ptr() + a * item, pc.x_remote(q, a), b - a, pc.flag_remote(q), pc.ack_local(q))
                         for q, a, b in self.sends]
                flags = [pc.flag_local(q) for q, _, _ in self.recvs]
                acks = [pc.ack_remote(q) for q, _, _ in self.recvs]
                dbg = os.environ.get("B2S_FUSE_DEBUG", "")   # timing experiments only (results are then WRONG)
                if dbg == "order-only":      # same tile order, no exchange at all
                    sends, flags, acks = [], [], []
                elif dbg == "no-wait":       # push + acks, but nobody waits for arrival
                    flags = []
                desc = _ops.fuse_desc(ranges, n_free, flags=flags, sends=sends, acks=acks, epoch_ctr=pc.epoch_ctr,
                                      ticket=pc.ticket, epoch_add=1, epoch_bump=1, error=pc.error_word)
                info = {"mode": "halo", "desc": desc, "pc": pc}
        elif self.exchange_mode == "allgather":
            ok = bool(usable and self.col_plan.uniform)
            # Column blocks pay per-block launch / row-pointer / y read-modify-write overheads (tools/bench_blocks.py
            # measures them on an R32 shard), so they are used only when the gathered x would NOT stay L2-resident next
            # to the matrix stream (more than 3/8 of L2; each block then gathers from one L2-sized slice).
            # Otherwise ("gather"): push, wait for every slice, one product of the unsplit shard.
            blocks_min = self._blocks_min if self._blocks_min is not None else 3 * runtime.l2_bytes() // 8
            want_blocks = self.shape[1] * item > blocks_min
            lo, hi = self.my_cols
            if ok and not want_blocks:
                ok = self._agree(True)
                if ok:
                    sends = [(q, lo, pc.peer_x_off[q] + lo, hi - lo) for q in range(self.nranks) if q != self.rank and hi > lo]
                    slice_bytes = (hi - lo) * item
                    info = {"mode": "gather", "sends": sends, "pc": pc,
                            "recv_peers": [q for q in range(self.nranks) if q != self.rank],
                            "cps": 16 if slice_bytes >= (1 << 22) else (4 if slice_bytes >= (1 << 18) else 1)}
            elif self._agree(ok):
                blocks = self._column_blocks(A)
                sends = [(q, lo, pc.peer_x_off[q] + lo, hi - lo) for q in range(self.nranks) if q != self.rank and hi > lo]
                recv_peers = [q for q in range(self.nranks) if q != self.rank]
                descs = {}
                for q, Bq in blocks.items():
                    if q == self.rank or Bq is None:
                        continue
                    pl = Bq._get_plan(tma_only=True)
                    if not pl.tma:
                        raise RuntimeError("column block without a TMA tile plan")
                    descs[q] = _ops.fuse_desc([(0, pl.tiles)], 0, flags=[pc.flag_local(q)], epoch_ctr=pc.epoch_ctr,
                                              ticket=pc.ticket, epoch_add=0, epoch_bump=0, error=pc.error_word,
                                              accumulate=True)
                slice_bytes = (hi - lo) * item
                info = {"mode": "blocks", "blocks": blocks, "descs": descs, "sends": sends, "recv_peers": recv_peers,
                        "pc": pc, "cps": 16 if slice_bytes >= (1 << 22) else (4 if slice_bytes >= (1 << 18) else 1),
                        "order": [(self.rank + d) % self.nranks for d in range(1, self.nranks)]}
        self._fused[key] = info
        return info

    def _column_blocks(self, A: csr_array):
        """{q: CSR of the entries of A whose column is owned by rank q (global column ids kept), or None if empty}, cut
        once per state of A's arrays and cached with A's other derivatives."""
        ranges = tuple(self.col_plan.rows(q) for q in range(self.nranks))
        return A._derived("rank_blocks", ranges, lambda: dict(enumerate(_column_blocks(A, ranges))))

    def _dot_fused(self, info, A, x_full, out, w=None, dot_out=None):
        # the plan is looked up per launch, not kept in `info`: a coded plan holds the values, so an in-place edit of
        # A.data must reach the launch through a new plan (same structure: the same tiles the descriptors name)
        xin = x_full[: A.shape[1]]
        if info["mode"] == "halo":
            _ops.spmv_fused(A.indptr, A.indices, A.data, xin, out, A.shape, A._get_plan(), info["desc"], w=w, dot_out=dot_out)
            return out
        pc = info["pc"]
        if info["mode"] == "gather":
            # every tile of an unsplit shard needs every slice: push, wait for all arrivals, multiply
            _ops.peer_push(x_full, self.rank, pc.peers, info["sends"], info["recv_peers"], info["cps"])
            _ops.peer_push_wait(self.rank, pc.peers, info["recv_peers"])
            if w is not None:
                _ops.spmv_dot(A.indptr, A.indices, A.data, xin, out, w, dot_out, A.shape, A._get_plan())
            else:
                _ops.spmv(A.indptr, A.indices, A.data, xin, out, A.shape, plan=A._get_plan())
            return out
        # the column blocks hold copies of the values: after an edit of A.data they are cut again (same structure, so
        # the same tiles the descriptors name)
        info["blocks"] = self._column_blocks(A)
        cur = torch.cuda.current_stream()
        if getattr(self, "_comm_stream", None) is None:
            self._comm_stream = torch.cuda.Stream()
        cs = self._comm_stream
        cs.wait_stream(cur)
        with torch.cuda.stream(cs):
            _ops.peer_push(x_full, self.rank, pc.peers, info["sends"], info["recv_peers"], info["cps"])
            pushed = cs.record_event()
        own = info["blocks"].get(self.rank)
        if own is None:
            out.zero_()
        else:
            _ops.spmv(own.indptr, own.indices, own.data, xin, out, own.shape, plan=own._get_plan())
        cur.wait_event(pushed)   # the epoch counter the block launches read is the one this push advanced
        for q in info["order"]:
            Bq = info["blocks"].get(q)
            if Bq is not None:
                _ops.spmv_fused(Bq.indptr, Bq.indices, Bq.data, xin, out, Bq.shape, Bq._get_plan(), info["descs"][q])
        if w is not None:
            _ops.dot(w, out, out=dot_out)
        return out

    def dot(self, x_full: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """y_local = A_local @ x.  `x_full` is a full-length buffer whose my_cols slice is current.

        Default on the GPUs of one box: the exchange is fused into the SpMV launch(es) (`_fused_setup`).  Otherwise
        (B2S_PEER_FUSED=0, gloo, several hosts) x is exchanged with NCCL first -- optionally on a side stream while the
        tiles that read only local columns run (B2S_OVERLAP=1)."""
        A = self.local
        if out is None:
            out = torch.empty(A.shape[0], dtype=x_full.dtype, device=x_full.device)
        xin = x_full if x_full.shape[0] == A.shape[1] else x_full[: A.shape[1]]
        if self.use_fused and x_full.is_cuda and self.exchange_mode != "none":
            info = self._fused_setup(A, x_full)
            if info is not None:
                return self._dot_fused(info, A, x_full, out)
        plan = A._get_plan()
        sched = None
        if (self.exchange_mode == "p2p" and x_full.is_cuda and A.dtype == numpy_dtype(x_full.dtype)
                and os.environ.get("B2S_OVERLAP", "0") == "1"):
            sched = self._overlap_schedule()
        if sched is None:
            self.exchange(x_full)
            _ops.spmv(A.indptr, A.indices, A.data, xin, out, A.shape, plan=plan)
            return out
        interior, boundary = sched
        cur = torch.cuda.current_stream()
        if getattr(self, "_comm_stream", None) is None:
            self._comm_stream = torch.cuda.Stream()
        cs = self._comm_stream
        cs.wait_stream(cur)
        with torch.cuda.stream(cs):
            self.exchange(x_full)
            done = cs.record_event()
        for tile_lo, tile_hi in interior:
            _ops.spmv_tiles(A.indptr, A.indices, A.data, xin, out, A.shape, plan, tile_lo, tile_hi)
        cur.wait_event(done)
        for tile_lo, tile_hi in boundary:
            _ops.spmv_tiles(A.indptr, A.indices, A.data, xin, out, A.shape, plan, tile_lo, tile_hi)
        return out

    def spmv_dot(self, Ad: csr_array, x_full, out, w, dot_out):
        """q = A p and dot_out = all-reduced p.q for the CG loop (`Ad` = the local shard, possibly promoted): the x
        exchange, the product and the local inner product are one launch on the fused halo path."""
        info = None
        if self.use_fused and x_full.is_cuda and self.exchange_mode != "none":
            info = self._fused_setup(Ad, x_full)
        if info is not None:
            self._dot_fused(info, Ad, x_full, out, w=w, dot_out=dot_out)
        else:
            self.exchange(x_full)
            _ops.spmv_dot(Ad._indptr, Ad._indices, Ad._data, x_full[: Ad.shape[1]], out, w, dot_out, Ad.shape, Ad._get_plan())
        self.allreduce(dot_out)
        return out

    def dot_graphed(self, x_full: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
        """`dot` replayed from a CUDA graph (captured on first use for this (x_full, out) pair): the exchange
        (fused launches with device-side epochs, NCCL send/recv or peer kernels), the stream fork/join and the tile
        launches cost one graph launch on the host instead of the Python/NCCL call overhead per product, which is
        what bounds a SpMV step of a few hundred microseconds otherwise."""
        from .linalg import _try_capture

        key = (x_full.data_ptr(), out.data_ptr(), os.environ.get("B2S_OVERLAP", "0"))
        cache = self.__dict__.setdefault("_dot_graphs", {})
        # a graph replays the launches of the plan it was captured with (which may hold coded values of local.data):
        # it is only valid while that plan is the current one, and keeps it -- and its pack buffer -- alive
        plan = self.local._get_plan()
        hit = cache.get(key)
        g = hit[0] if hit is not None and hit[1] is plan else None
        if g is None:
            self.dot(x_full, out=out)  # eager warm-up: plans, schedules, communicators, kernel attributes
            torch.cuda.synchronize()
            g = _try_capture(lambda: self.dot(x_full, out=out)) or False
            cache[key] = (g, plan)
        if g:
            g.replay()
        else:
            self.dot(x_full, out=out)
        return out

    # -- SpMM ---------------------------------------------------------------------------------------------
    def new_full_matrix(self, k: int, dtype=None) -> torch.Tensor:
        """(ncols padded to P*T, k) row-major buffer for a dense operand sharded by rows like the vectors."""
        dt = torch_dtype(numpy_dtype(self.dtype if dtype is None else dtype))
        return torch.zeros((max(self.col_plan.padded, 1), int(k)), dtype=dt, device=runtime.device)

    def spmm(self, X_full: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """Y_local (local rows, k) = A_local @ X (reference spmm(), csr.py:1151-1205: rows of A tiled, the image
        of `crd` into the rows of the dense operand decides what each shard needs).  `X_full` is a full-height
        buffer whose rows [my_cols) are current; the rows of this shard's column window are fetched with the same
        exchange plan as the SpMV vector (all-gather or point-to-point halo, k values per exchanged row)."""
        A = self.local
        assert X_full.ndim == 2 and X_full.is_contiguous()
        if out is None:
            out = torch.empty((A.shape[0], X_full.shape[1]), dtype=X_full.dtype, device=X_full.device)
        self.exchange(X_full)
        _ops.spmm(A.indptr, A.indices, A.data, X_full[: A.shape[1]], out, A.shape)
        return out

    def matmat_global(self, X_global):
        """Convenience for tests: replicated dense X in, replicated Y out (numpy)."""
        X_global = np.asarray(X_global, dtype=self.dtype)
        full = self.new_full_matrix(X_global.shape[1])
        lo, hi = self.my_cols
        full[lo:hi] = to_device(X_global[lo:hi], dtype=self.dtype)
        Y = self.spmm(full)
        cols = [gather_vector(Y[:, j].contiguous(), self.row_plan, self.rank, self.group) for j in range(Y.shape[1])]
        return np.stack(cols, axis=1) if cols else np.zeros((self.shape[0], 0), dtype=self.dtype)

    def dot_fused(self, x_full, out, w, dot_out):
        """y_local = A_local @ x and dot_out = all-reduced sum_i w_i y_i."""
        self.exchange(x_full)
        A = self.local
        _ops.spmv_dot(A.indptr, A.indices, A.data, x_full[: A.shape[1]], out, w, dot_out, A.shape, A._get_plan())
        allreduce_scalar(dot_out, self.group)
        return out

    # -- exchange / all-reduce interface used by linalg._cg_fused_loop -------------------------------------------
    def new_p(self, n, like):
        full = self.new_full_vector(numpy_dtype(like.dtype))
        return full, self.local_view(full)

    def allreduce(self, t):
        if self.use_peer and t.is_cuda and t.numel() <= 4:
            # any of this shard's peer communicators will do: the scalar mailboxes do not depend on the x dtype
            pc = next(iter(self._peer.values())) if self._peer else self._peer_comm(self.dtype)
            if pc is not None:
                return pc.allreduce(t)
        return allreduce_scalar(t, self.group)

    def check_peer(self):
        for pc in self._peer.values():
            pc.check()

    def close(self):
        self.__dict__.pop("_dot_graphs", None)   # captured graphs reference the buffers freed below
        self._fused = {}
        for pc in self._peer.values():
            pc.close()
        self._peer = {}

    def as_linear_operator(self):
        """This shard as a `linalg.LinearOperator` on row-sharded vectors: matvec(x_local) -> y_local exchanges the
        halo / all-gathers x, and the `allreduce` it carries makes the Krylov solvers of linalg (cgs, bicgstab, gmres,
        eigsh; cg has its own fused loop, `dist.cg`) sum their inner products over the ranks.  No rmatvec: the
        transpose of a row-sharded matrix is column-sharded."""
        from .linalg import LinearOperator

        shard = self

        class _ShardOperator(LinearOperator):
            def __init__(self):
                assert shard.shape[0] == shard.shape[1], "row-sharded solvers need a square matrix"
                lo, hi = shard.my_cols
                super().__init__(shard.dtype, (shard.local.shape[0], hi - lo))
                self.global_shape = shard.shape
                self._full = {}

            def _matvec(self, x, out=None):
                key = numpy_dtype(x.dtype)
                full = self._full.get(key)
                if full is None:
                    full = self._full[key] = shard.new_full_vector(key)
                shard.local_view(full).copy_(x.reshape(-1))
                return shard.dot(full, out=out)

            def allreduce(self, t):
                return shard.allreduce(t)

        return _ShardOperator()

    def matvec_global(self, x_global):
        """Convenience for tests: replicated x in, replicated y out (numpy)."""
        full = self.scatter_vector(np.asarray(x_global, dtype=self.dtype))
        y = self.dot(full)
        return gather_vector(y, self.row_plan, self.rank, self.group)


def _allgather_varlen(t: torch.Tensor, group=None):
    """All-gather 1-D tensors of different lengths; returns the list of per-rank tensors."""
    world = dist.get_world_size(group)
    sizes = [None] * world
    dist.all_gather_object(sizes, int(t.shape[0]), group=group)
    m = max(max(sizes), 1)
    pad = torch.zeros(m, dtype=t.dtype, device=t.device)
    pad[: t.shape[0]] = t
    out = torch.empty(m * world, dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    return [out[q * m : q * m + sizes[q]] for q in range(world)]


def gather_matrix(A: "dist_csr_array") -> csr_array:
    """Replicate a row-sharded matrix on every rank (all-gather of indptr / indices / data shards)."""
    if A.nranks == 1:
        return A.local
    loc = A.local
    counts = (loc.indptr[1:] - loc.indptr[:-1]).to(torch.int64)
    all_counts = torch.cat(_allgather_varlen(counts, A.group))
    indptr = torch.zeros(all_counts.shape[0] + 1, dtype=torch.int64, device=all_counts.device)
    torch.cumsum(all_counts, 0, out=indptr[1:])
    indices = torch.cat(_allgather_varlen(loc.indices, A.group))
    data = torch.cat(_allgather_varlen(loc.data, A.group))
    return csr_array._from_parts(indptr.to(_indptr_dtype(int(indptr[-1]))), indices, data, A.shape)


def spgemm(A: "dist_csr_array", B: "dist_csr_array") -> "dist_csr_array":
    """C = A @ B for row-sharded operands: B is replicated (all-gather once), every rank multiplies its
    rows of A, and C comes back row-sharded with the same row plan as A -- the partitioning of the
    reference's GPU branch (sparse/csr.py:1322-1389: rows of the left operand tiled, the right operand
    gathered by image, per-GPU local CSR).  `C.nnz_offset` is this shard's position in the global nnz
    order (exclusive scan of the per-rank nnz; the reference does that scan on the host,
    scan_local_results_and_scale_pos csr.py:827-859)."""
    assert A.shape[1] == B.shape[0]
    Bfull = gather_matrix(B)
    Cl = A.local @ Bfull
    C = dist_csr_array(Cl, (A.shape[0], B.shape[1]), rank=A.rank, nranks=A.nranks, group=A.group,
                       row_plan=A.row_plan)
    nnzs = [None] * A.nranks
    if A.nranks > 1:
        dist.all_gather_object(nnzs, Cl.nnz, group=A.group)
    else:
        nnzs[0] = Cl.nnz
    C.nnz_offset = int(sum(nnzs[: A.rank]))
    C.global_nnz = int(sum(nnzs))
    return C


def allreduce_scalar(t: torch.Tensor, group=None) -> torch.Tensor:
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def gather_vector(v_local: torch.Tensor, plan: RowBlockPlan, rank: int, group=None) -> np.ndarray:
    """All ranks receive the concatenated global vector (host numpy)."""
    if plan.nranks == 1:
        return to_host(v_local)
    T = max(plan.tile, 1)
    pad = torch.zeros(T, dtype=v_local.dtype, device=v_local.device)
    pad[: v_local.shape[0]] = v_local
    full = torch.empty(T * plan.nranks, dtype=v_local.dtype, device=v_local.device)
    dist.all_gather_into_tensor(full, pad, group=group)
    if plan.uniform:
        return to_host(full[: plan.nrows])
    return to_host(torch.cat([full[q * T : q * T + (plan.bounds[q + 1] - plan.bounds[q])] for q in range(plan.nranks)]))


def cg(A: dist_csr_array, b_local, x0_local=None, tol=1e-08, maxiter=None, callback=None, conv_test_iters=25):
    """Row-sharded conjugate gradient: the fused loop of linalg._cg_fused_loop with the SpMV input exchanged
    per iteration and the two inner products all-reduced.  Same semantics as linalg.cg (absolute tol,
    test every conv_test_iters, returns (x_local, iters)); every rank returns its shard of x."""
    from .linalg import _cg_fused_loop

    assert A.shape[0] == A.shape[1]
    n_global = A.shape[0]
    if maxiter is None:
        maxiter = n_global * 10
    dt = np.result_type(np.float64 if x0_local is None else numpy_dtype(x0_local.dtype), numpy_dtype(b_local.dtype),
                        A.local.dtype)   # never narrow the matrix (reference: r = b - A x in the promoted type)
    Al = A.local if A.local.dtype == dt else A.local._promoted(dt)  # same structure, promoted values
    b = to_device(b_local, dtype=dt).reshape(-1)
    n = b.shape[0]
    x = torch.zeros(n, dtype=b.dtype, device=b.device) if x0_local is None else to_device(x0_local, dtype=dt, copy=True)
    out = _cg_fused_loop(Al, A, b, x, tol, maxiter, callback, conv_test_iters, True)
    A.check_peer()
    return out
