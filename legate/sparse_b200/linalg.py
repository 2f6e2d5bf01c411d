"""`linalg`: LinearOperator family, `cg_axpby` and the conjugate-gradient solver.

Public surface and semantics follow the reference (sparse/linalg.py:128-352 LinearOperator,
:357-414 _CustomLinearOperator, :420-432 _SparseMatrixLinearOperator, :437-459 IdentityOperator,
:462-466 make_linear_operator, :479-496 cg_axpby, :499-565 cg):

* `tol` is an ABSOLUTE threshold on ||r||_2, tested only every `conv_test_iters` iterations
  (and at `maxiter-1`), `atol` must be None, default `maxiter = 10 n`, returns `(x, iters)`.
* the scalars rho, rho1, pq never visit the host: they live in 1-element device arrays and the
  divisions rho/pq, rho/rho1 happen inside the kernels (reference: Legion futures + AXPBY task).

Two code paths produce the same iterates:
  - generic : any LinearOperator A / preconditioner M, one kernel per reference op;
  - fused   : A is a `csr_array`, M is None -> 3 launches per iteration
              (SpMV+p.q | x,r update + r.r | p update) instead of 7, and the Identity copy z = r
              (2 vector passes) disappears.  Selected automatically; `B2S_CG_FUSED=0` disables it.
"""
from __future__ import annotations

import inspect
import os
import warnings

import numpy as np
import torch

from . import _ops
from .csr import csr_array
from .runtime import is_device_array, numpy_dtype, runtime, to_device, to_host, torch_dtype


def _zeros(n, dtype=np.float64):
    return torch.zeros(n, dtype=torch_dtype(dtype), device=runtime.device)


class LinearOperator:
    """Common interface for matrix-vector products (scipy.sparse.linalg.LinearOperator subset).

    Subclasses implement `_matvec(x, out=None)`; `LinearOperator(shape, matvec=...)` builds a
    `_CustomLinearOperator`.  Vectors are device tensors inside the solvers.
    """

    ndim = 2

    def __new__(cls, *args, **kwargs):
        if cls is LinearOperator:
            return super().__new__(_CustomLinearOperator)
        obj = super().__new__(cls)
        if type(obj)._matvec == LinearOperator._matvec:
            warnings.warn(
                "LinearOperator subclass should implement at least one of _matvec and _matmat.",
                category=RuntimeWarning,
                stacklevel=2,
            )
        return obj

    def __init__(self, dtype, shape):
        if dtype is not None:
            dtype = np.dtype(dtype)
        self.dtype = dtype
        self.shape = tuple(shape)

    def _init_dtype(self):
        if self.dtype is None:
            v = _zeros(self.shape[-1])
            self.dtype = numpy_dtype(self.matvec(v).dtype)

    def _matvec(self, x, out=None):
        raise NotImplementedError

    def matvec(self, x, out=None):
        M, N = self.shape
        if tuple(x.shape) != (N,) and tuple(x.shape) != (N, 1):
            raise ValueError("dimension mismatch")
        y = self._matvec(x, out=out)
        if x.ndim == 1:
            y = y.reshape(M)
        elif x.ndim == 2:
            y = y.reshape(M, 1)
        else:
            raise ValueError("invalid shape returned by user-defined matvec()")
        return y

    def _rmatvec(self, x, out=None):
        raise NotImplementedError

    def rmatvec(self, x, out=None):
        M, N = self.shape
        if tuple(x.shape) != (M,) and tuple(x.shape) != (M, 1):
            raise ValueError("dimension mismatch")
        y = self._rmatvec(x, out=out)
        return y.reshape(N) if x.ndim == 1 else y.reshape(N, 1)

    def __matmul__(self, x):
        return self.matvec(x)

    def __repr__(self):
        M, N = self.shape
        dt = "unspecified dtype" if self.dtype is None else f"dtype={self.dtype}"
        return f"<{M}x{N} {self.__class__.__name__} with {dt}>"


class _CustomLinearOperator(LinearOperator):
    """Linear operator defined in terms of user-specified callables."""

    def __init__(self, shape, matvec, rmatvec=None, matmat=None, dtype=None, rmatmat=None):
        super().__init__(dtype, shape)
        self.args = ()
        self.__matvec_impl = matvec
        self.__rmatvec_impl = rmatvec
        # does the user's callable take an out= parameter? (reference linalg.py:407-414)
        self._matvec_has_out = self._has_out(matvec)
        self._rmatvec_has_out = self._has_out(rmatvec)
        self._init_dtype()

    def _matvec(self, x, out=None):
        if self._matvec_has_out:
            return self.__matvec_impl(x, out=out)
        if out is None:
            return self.__matvec_impl(x)
        out[:] = self.__matvec_impl(x)
        return out

    def _rmatvec(self, x, out=None):
        func = self.__rmatvec_impl
        if func is None:
            raise NotImplementedError("rmatvec is not defined")
        if self._rmatvec_has_out:
            return func(x, out=out)
        if out is None:
            return func(x)
        out[:] = func(x)
        return out

    @staticmethod
    def _has_out(o):
        if o is None:
            return False
        return "out" in inspect.signature(o).parameters


class _SparseMatrixLinearOperator(LinearOperator):
    def __init__(self, A):
        self.A = A
        self.AH = None
        super().__init__(A.dtype, A.shape)

    def _matvec(self, x, out=None):
        return self.A.dot(x, out=out)

    def _rmatvec(self, x, out=None):
        if self.AH is None:
            self.AH = self.A.T.conj(copy=False)
        return self.AH.dot(x, out=out)


class IdentityOperator(LinearOperator):
    def __init__(self, shape, dtype=None):
        super().__init__(dtype, shape)

    def _matvec(self, x, out=None):
        if out is not None:
            out[:] = x
            return out
        # copy so callers never alias their input (reference linalg.py:446-449)
        return x.clone() if isinstance(x, torch.Tensor) else x.copy()

    _rmatvec = _matvec


def make_linear_operator(A):
    if isinstance(A, LinearOperator):
        return A
    if hasattr(A, "as_linear_operator"):  # a row shard of a distributed matrix (dist.dist_csr_array)
        return A.as_linear_operator()
    return _SparseMatrixLinearOperator(A)


def cg_axpby(y, x, a, b, isalpha=True, negate=False):
    """y = alpha*x + y (isalpha) or y = x + beta*y, with alpha|beta = a/b (negated if `negate`).

    a, b are 1-element device arrays; the division happens on the device
    (reference sparse/linalg.py:479-496 -> AXPBY task, src/sparse/linalg/axpby.cu:25-43).
    """
    return _ops.axpby(y, x, a, b, isalpha=isalpha, negate=negate)


def _as_scalar_array(v, dtype):
    if isinstance(v, torch.Tensor):
        return v.reshape(1).to(torch_dtype(dtype))
    return torch.full((1,), float(v), dtype=torch_dtype(dtype), device=runtime.device)


def _use_fused(A, M) -> bool:
    return isinstance(A, csr_array) and M is None and os.environ.get("B2S_CG_FUSED", "1") != "0"


def cg(A, b, x0=None, tol=1e-08, maxiter=None, M=None, callback=None, atol=None, conv_test_iters=25):
    """Conjugate gradient, reference semantics (sparse/linalg.py:499-565). Returns (x, iters).

    b / x0 may be numpy arrays (then x is returned as numpy) or CUDA tensors (x returned on device).
    """
    assert len(b.shape) == 1 or (len(b.shape) == 2 and b.shape[1] == 1)
    assert len(A.shape) == 2 and A.shape[0] == A.shape[1]
    assert atol is None, "atol is not supported."
    runtime.require_cuda("linalg.cg")

    n = b.shape[0]
    if maxiter is None:
        maxiter = n * 10
    on_device = is_device_array(b) and b.is_cuda
    # the reference allocates x, p with np.zeros(n) -> float64 (linalg.py:526-527)
    work_dtype = np.float64 if x0 is None else numpy_dtype(x0.dtype)
    if work_dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
        work_dtype = np.float64
    wide = [work_dtype, numpy_dtype(b.dtype)]
    if isinstance(A, csr_array) and np.dtype(A.dtype) in (np.dtype(np.float32), np.dtype(np.float64)):
        wide.append(A.dtype)   # r = b - A x is computed in the promoted type (reference linalg.py:532): never narrow A
    bd = to_device(b, dtype=np.result_type(*wide)).reshape(-1)
    work_dtype = numpy_dtype(bd.dtype)
    x = _zeros(n, work_dtype) if x0 is None else to_device(x0, dtype=work_dtype, copy=True).reshape(-1)

    if _use_fused(A, M):
        x, iters = _cg_fused(A, bd, x, tol, maxiter, callback, conv_test_iters, on_device)
    else:
        x, iters = _cg_generic(A, bd, x, tol, maxiter, M, callback, conv_test_iters, on_device)
    return (x if on_device else to_host(x)), iters


def _cg_generic(A, b, x, tol, maxiter, M, callback, conv_test_iters, on_device):
    """Op-for-op the reference loop: copy z=M r, dot, axpby, SpMV, dot, axpby, axpby (+ norm/25)."""
    n = b.shape[0]
    dt = numpy_dtype(b.dtype)
    A = make_linear_operator(A)
    M = IdentityOperator(A.shape, dtype=A.dtype) if M is None else make_linear_operator(M)
    p = _zeros(n, dt)
    r = b - A.matvec(x)
    iters = 0
    rho = _as_scalar_array(0.0, dt)
    z = None
    q = None
    while iters < maxiter:
        z = M.matvec(r, out=z)
        rho1 = rho
        rho = _ops.dot(r, z)
        if iters == 0:
            p[:] = z
        else:
            cg_axpby(p, z, rho, rho1, isalpha=False, negate=False)
        q = A.matvec(p, out=q)
        pq = _ops.dot(p, q)
        cg_axpby(x, p, rho, pq, isalpha=True, negate=False)
        cg_axpby(r, q, rho, pq, isalpha=True, negate=True)
        iters += 1
        if callback is not None:
            callback(x if on_device else to_host(x))
        if (iters % conv_test_iters == 0 or iters == (maxiter - 1)) and float(_ops.nrm2(r)[0]) < tol:
            break
    return x, iters


class _LocalComm:
    """Single-GPU stand-in for the exchange/all-reduce interface of dist.dist_csr_array."""

    def new_p(self, n, like):
        p = torch.empty(n, dtype=like.dtype, device=like.device)
        return p, p

    def exchange(self, p_full):
        return None

    def allreduce(self, t):
        return t

    def dot(self, x_full, out=None, A=None):
        _ops.spmv(A._indptr, A._indices, A._data, x_full[: A.shape[1]], out, A.shape, plan=A._get_plan())
        return out

    def spmv_dot(self, A, x_full, out, w, dot_out):
        _ops.spmv_dot(A._indptr, A._indices, A._data, x_full[: A.shape[1]], out, w, dot_out, A.shape, A._get_plan())
        return out


def _cg_fused(A: csr_array, b, x, tol, maxiter, callback, conv_test_iters, on_device):
    dt = numpy_dtype(b.dtype)
    Ad = A._promoted(dt) if A.dtype != dt else A      # dt >= A.dtype by construction (see cg): a widening cast
    return _cg_fused_loop(Ad, _LocalComm(), b, x, tol, maxiter, callback, conv_test_iters, on_device)


def _cg_fused_loop(Ad: csr_array, comm, b, x, tol, maxiter, callback, conv_test_iters, on_device):
    """Fused CG recurrence, 3 kernel launches per iteration (+ exchange / 2 scalar all-reduces when sharded).

    With M = I: z = r, rho = r.r.  Per iteration
        p = r + (rho/rho_prev) p              (b2s_axpby, isalpha=False)            [skipped at k = 0: p = r]
        [x-window exchange of p]
        q = A p ; pq = p.q                    (b2s_spmv_csr_dot)                    [all-reduce pq]
        x += (rho/pq) p ; r -= (rho/pq) q ; rr = r.r   (b2s_cg_update_xr)           [all-reduce rr]
        rho_prev <- rho ; rho <- rr
    ||r|| for the convergence test is sqrt(rho) -- no extra pass.  All scalars stay on the device; the host
    reads one of them every `conv_test_iters` iterations (reference cadence, linalg.py:559-563).

    Iterations k >= 1 are identical, so they are captured once in a CUDA graph and replayed (removes the
    per-launch CPU cost, which dominates once the per-GPU shard is small); `B2S_CG_GRAPH=0` disables it.
    """
    n = b.shape[0]
    plan = Ad._get_plan()
    shape = Ad.shape
    q = torch.empty(n, dtype=b.dtype, device=b.device)
    p_full, p = comm.new_p(n, b)
    xin = p_full[: shape[1]]

    # r = b - A x
    p.copy_(x)
    comm.spmv_dot(Ad, p_full, q, p, torch.empty(1, dtype=b.dtype, device=b.device))   # q = A x (the dot is discarded)
    r = b - q
    # rho_k = r_k . r_k lives in slot k % 3 of `scal`: iteration k reads rho_k and rho_{k-1} and writes rho_{k+1}, so the
    # roles rotate with period 3 and no scalar is ever copied (three captured graphs, one per k % 3, instead of one
    # graph plus two one-element copy kernels per iteration)
    scal = torch.zeros(3, dtype=b.dtype, device=b.device)
    slot = [scal[i : i + 1] for i in range(3)]
    _ops.dot(r, r, out=slot[0])
    comm.allreduce(slot[0])
    pq = torch.empty(1, dtype=b.dtype, device=b.device)

    def tail_of_iteration(k):
        comm.spmv_dot(Ad, p_full, q, p, pq)      # exchange of p (fused into the launch when sharded) + product + p.q
        _ops.cg_update_xr(x, r, p, q, slot[k % 3], pq, slot[(k + 1) % 3])
        comm.allreduce(slot[(k + 1) % 3])

    def generic_iteration(k):
        cg_axpby(p, r, slot[k % 3], slot[(k - 1) % 3], isalpha=False, negate=False)
        tail_of_iteration(k)

    def converged(iters):
        return (iters % conv_test_iters == 0 or iters == (maxiter - 1)) and float(slot[iters % 3][0]) ** 0.5 < tol

    iters = 0
    if maxiter <= 0:
        return x, iters
    # iteration 0: p = r (no alias: p is updated in place later, reference linalg.py:541-544)
    p.copy_(r)
    tail_of_iteration(0)
    iters = 1
    if callback is not None:
        callback(x if on_device else to_host(x))
    if converged(iters):
        return x, iters

    graphs = None
    if os.environ.get("B2S_CG_GRAPH", "1") != "0" and maxiter - iters >= 6 and b.is_cuda:
        graphs = [_try_capture(lambda k=k: generic_iteration(k)) for k in (3, 1, 2)]   # index = k % 3
        if any(g is None for g in graphs):
            graphs = None
    # the graphs replay the launches of the plan current at capture, which holds its own copy of the structure and
    # codes the values of that point: an edit of Ad's arrays (from the callback) sends the loop back to eager launches,
    # which re-plan
    stamp = Ad._stamp()
    while iters < maxiter:
        if graphs is not None and Ad._stamp() != stamp:
            graphs = None
        if graphs is not None:
            graphs[iters % 3].replay()
        else:
            generic_iteration(iters)
        iters += 1
        if callback is not None:
            callback(x if on_device else to_host(x))
        if converged(iters):
            break
    return x, iters


def _try_capture(fn):
    """Capture `fn` (kernel launches on the current stream) into a CUDA graph; None if capture fails.

    The iteration is idempotent-unsafe (it updates x, r, p in place), so it cannot be 'warmed up' by simply
    running it; all kernels and workspaces it uses were already exercised by iteration 0 and the setup SpMV.
    """
    cur = torch.cuda.current_stream()
    try:
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            runtime.workspace()  # allocate the reduction workspace of the capture stream before capturing
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        # capture_begin/end directly: the torch.cuda.graph() context manager also runs gc.collect() and
        # torch.cuda.empty_cache(), which costs seconds when gigabytes of assembly temporaries are cached
        with torch.cuda.stream(side):
            g.capture_begin()
            try:
                fn()
            finally:
                g.capture_end()
        cur.wait_stream(side)
        torch.cuda.synchronize()
        return g
    except Exception as exc:  # pragma: no cover - depends on driver / NCCL capture support
        warnings.warn(f"CUDA graph capture of the CG iteration failed ({exc}); running eagerly", RuntimeWarning)
        try:
            torch.cuda.synchronize()
        except Exception:
            pass
        return None


__all__ = [
    "LinearOperator",
    "IdentityOperator",
    "make_linear_operator",
    "cg_axpby",
    "cg",
    "cgs",
    "bicg",
    "bicgstab",
    "gmres",
    "lsqr",
    "eigsh",
]


# the other Krylov solvers of the reference module (linalg.py:570-1569) live in krylov.py
from .krylov import bicg, bicgstab, cgs, eigsh, gmres, lsqr  # noqa: E402,F401
