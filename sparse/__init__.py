"""Drop-in alias: `import sparse` / `import sparse.linalg as linalg` / `import sparse.io` resolve to
legate.sparse_b200, so a script written against the reference package runs unchanged for the hot path
(CSR construction, SpMV, SpGEMM, CG).  Everything lives in legate/sparse_b200; nothing is implemented here."""
from legate.sparse_b200 import *  # noqa: F401,F403
from legate.sparse_b200 import (  # noqa: F401
    block_diag,
    bmat,
    coo_array,
    coo_matrix,
    csc_array,
    csc_matrix,
    csr_array,
    csr_matrix,
    dia_array,
    dia_matrix,
    diags,
    eye,
    hstack,
    identity,
    io,
    is_sparse_matrix,
    kron,
    kronsum,
    linalg,
    rand,
    random,
    random_array,
    runtime,
    spdiags,
    vstack,
)


class SparseArray:
    """Placeholder only.  scipy's array-API helper looks up `sys.modules["sparse"].SparseArray` (the pydata/sparse
    base class) whenever a module called `sparse` is loaded; without this name every scipy.sparse.linalg solver
    raises AttributeError once this alias package has been imported.  Nothing derives from it."""
