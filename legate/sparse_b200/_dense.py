"""Dense operands and results of the sparse-times-dense products (`csr_array.dot`, `csc_array.dot`, `dia_array.dot`).

Which dense operands and outputs a kernel takes as they are, which it gets copies of, and how the result comes back in
the caller's array kind is decided here, once; a format supplies only its kernel launches (`dense_dot`).
"""
from __future__ import annotations

import numpy as np
import torch

from .runtime import SUPPORTED_VALUE_DTYPES, numpy_dtype, runtime, to_device, to_host, torch_dtype


def dense_rows(a, dtype):
    """A 2-D operand as a device tensor of `dtype` whose rows are unit-stride and do not overlap (the row stride may be
    larger than a row): a tensor already in that form is used without a copy."""
    if not isinstance(a, torch.Tensor):
        return to_device(a, dtype=dtype)   # numpy: C-ordered (a view when it already is) and copied to the device
    t = a.to(device=runtime.device, dtype=torch_dtype(dtype))
    rows, k = t.shape
    if (k > 1 and t.stride(1) != 1) or (rows > 1 and t.stride(0) < k):
        t = t.contiguous()
    return t


def check_out(out, shape, dtype):
    """ValueError unless `out` is None or has the result's `shape` and resolved `dtype`."""
    if out is None:
        return
    odt = numpy_dtype(out.dtype)
    if odt != dtype:
        raise ValueError(f"Output type {odt} is not consistent with resolved dtype {dtype}")
    if tuple(out.shape) != tuple(shape):
        raise ValueError(f"out has shape {tuple(out.shape)}, the result {tuple(shape)}")


def direct_out(out, shape) -> bool:
    """True when `out` is a CUDA tensor a kernel writing a result of `shape` may write as it is: contiguous for a
    vector; for an (m, k) result, unit-stride rows (k > 1) that do not overlap (m > 1)."""
    if not (isinstance(out, torch.Tensor) and out.is_cuda):
        return False
    if len(shape) == 1:
        return out.is_contiguous()
    m, k = shape
    return (k <= 1 or out.stride(1) == 1) and (m <= 1 or out.stride(0) >= k)


def deliver(res, out, on_device, direct):
    """The device result `res` in the caller's array kind: `out` when given (written unless the kernel wrote it
    directly), else a CUDA tensor for a CUDA operand and numpy otherwise."""
    if out is None:
        return res if on_device else to_host(res)
    if not direct:
        if isinstance(out, torch.Tensor):
            out.copy_(res)
        elif out.flags.c_contiguous:
            torch.from_numpy(out).copy_(res)   # D2H straight into the caller's (pinned) buffer
        else:
            out[...] = to_host(res)
    return out


def dense_dot(x, out, dtype, shape, name, spmv, spmm, complex_matrix):
    """A @ x for a dense x (numpy array or torch tensor) and a matrix A of `shape` and `dtype`, given A's launchers:

    * `spmv(dt, xd, y)` writes y = A xd for contiguous device vectors of the real dtype dt;
    * `spmm(dt, X, Y)` writes Y = A X for (n, k) / (m, k) device arrays of dt with unit-stride rows (`dense_rows`);
    * `complex_matrix(x, out)` returns the whole product when A itself is complex.

    A 1-D or (n, 1) x is a SpMV, any other 2-D x a SpMM; the result has x's shape ((m,), (m, 1) or (m, k)) and array
    kind, or is `out`.  The resolved dtype is np.result_type(A, x): float32 and float64 run the launchers, a complex x
    with a real A runs the real SpMM on the (re, im)-interleaved view of x (twice the columns, which is how complex
    arrays sit in memory), and anything else raises NotImplementedError.  `out` is checked before `runtime.require_cuda`
    and written in place: by the kernel when `direct_out` allows, else by a copy."""
    if x.ndim not in (1, 2):
        raise NotImplementedError(f"{name}: operand must be a vector, a dense 2-D array or a sparse matrix")
    m, n = shape
    if x.shape[0] != n:
        raise ValueError(f"dimension mismatch: {tuple(shape)} @ {tuple(x.shape)}")
    common = np.result_type(dtype, numpy_dtype(x.dtype))
    if common.kind == "c" and dtype.kind == "c":
        return complex_matrix(x, out)
    vector = x.ndim == 1 or x.shape[1] == 1
    if common.kind != "c" and common not in SUPPORTED_VALUE_DTYPES:
        raise NotImplementedError(f"{'SpMV' if vector else 'SpMM'} for resolved dtype {common} is not implemented "
                                  "(float32/float64 kernels only)")
    rshape = (m,) if x.ndim == 1 else (m, x.shape[1])
    check_out(out, rshape, common)
    runtime.require_cuda(name)
    on_device = isinstance(x, torch.Tensor) and x.is_cuda
    if common.kind == "c":
        k = 1 if x.ndim == 1 else x.shape[1]
        Xr = torch.view_as_real(to_device(x, dtype=common).reshape(n, k)).reshape(n, 2 * k)
        Yr = torch.empty((m, 2 * k), dtype=Xr.dtype, device=Xr.device)
        spmm(np.dtype(np.float32) if common == np.complex64 else np.dtype(np.float64), Xr, Yr)
        return deliver(torch.view_as_complex(Yr.reshape(m, k, 2)).reshape(rshape), out, on_device, False)
    if vector:
        xd = to_device(x.reshape(-1), dtype=common)
        direct = direct_out(out, (m,))
        y = out.reshape(-1) if direct else torch.empty(m, dtype=torch_dtype(common), device=xd.device)
        spmv(common, xd, y)
        res = y.reshape(rshape)
    else:
        X = dense_rows(x, common)
        direct = direct_out(out, rshape)
        res = out if direct else torch.empty(rshape, dtype=torch_dtype(common), device=X.device)
        spmm(common, X, res)
    return deliver(res, out, on_device, direct)
