"""legate.sparse_b200 -- H100-native (sm_90a) drop-in for the legate.sparse hot path.

Same scipy.sparse-style surface as the reference package (sparse/__init__.py:21-31) for the one
path this project accelerates: `csr_array`/`csr_matrix` construction, `A @ x` / `A.dot(x)` (CSR
SpMV), `A @ B` (CSR x CSR SpGEMM) and `linalg.cg` with its axpby/dot/norm inner loop -- all executed by
hand-written sm_90a kernels in libb200sparse.so (no cuSPARSE, no Legion, no CPU fallback).
"""
from . import _lib  # noqa: F401  (loads libb200sparse.so; raises if it is missing)
from .coo import coo_array  # noqa: F401
from .csc import csc_array, csc_matrix  # noqa: F401
from .csr import csr_array, csr_matrix, spgemm_csr_csr_csr  # noqa: F401
from .dia import dia_array, dia_matrix  # noqa: F401
from .module import (  # noqa: F401
    block_diag, bmat, diags, eye, hstack, identity, is_sparse_matrix, kron, kronsum, rand, random, random_array,
    spdiags, vstack,
)
from .runtime import runtime  # noqa: F401
from . import io, linalg  # noqa: F401

coo_matrix = coo_array

__version__ = "0.1.0"
