"""CSR x CSR SpGEMM (csrc/spgemm.cu) at the limits of every row class, in fp32 and fp64, with 32- and 64-bit row pointers.

The symbolic pass bins rows by product count: <= 32 products go to the warp kernel with a 64-slot hash table, <= 128 to
the warp kernel with 256 slots, <= 1024 to the CTA kernel with 2048 slots, <= 8192 to the CTA kernel with 16384 slots,
and larger rows to the dense kernel (global bitmaps, six sub-classes by size).  The numeric pass bins rows by exact nnz,
with the dense kernel beyond 1024 entries unless B2S_SPGEMM_DENSE_MIN raises that limit.  Each case below is built so
that its rows land in stated classes, and is checked against exact references:

* integer values (|a|, |b| <= 8, every partial sum below 2^24): indptr, indices and values equal the product in int64,
  whatever order the atomics add in;
* random values: |c - ref| <= 2 k u (|A||B|) against scipy's fp64 product, k the number of products behind the entry
  and u the unit roundoff of the value type;
* structure: the product of the two patterns in int64, so cancellation zeros are kept.

References run on the columns B stores only and are mapped back, so matrices with 2^31 - 2 columns cost no more than
their entries.  tests/test_spgemm_host.py checks the case builders and the references without a GPU."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import legate.sparse_b200 as sparse
from conftest import ROOT

pytestmark = pytest.mark.gpu

TYPES = [np.float32, np.float64]
WIDTHS = ["32", "64"]

# csrc/spgemm.cu: the symbolic pass's largest shared-memory class, the numeric pass's default one, and the hash tables
SYMBOLIC_CLS3 = 8192
NUMERIC_CLS3 = 1024
HASH_MUL = 2654435761
TABLE_BITS = {64: 6, 256: 8, 2048: 11, 16384: 14}
TABLE_ROWS = {64: 32, 256: 128, 2048: 1024, 16384: 8192}     # most distinct columns a row of the table's class has
TABLE_CLASSES = {64: (1, 1), 256: (2, 2), 2048: (3, 3), 16384: (4, 10)}   # (symbolic, numeric) class of such a row
UNIT_ROUNDOFF = {np.float32: 2.0**-24, np.float64: 2.0**-53}


# ---- restatements of the kernel's row classes and hash -------------------------------------------------------------
def classify(v, cls3):
    """classify() of csrc/spgemm.cu on an array of row sizes: 0 empty, 1 warp / 64 slots, 2 warp / 256, 3 CTA / 2048,
    4 CTA / 16384 (only when `cls3` > 1024), 5..10 dense, from 5 (more than 2^23) down to 10 (at most 2^15)."""
    v = np.asarray(v, dtype=np.int64)
    table = np.select([v == 0, v <= 32, v <= 128, v <= 1024], [0, 1, 2, 3], 4)
    dense = 10 - sum((v > (1 << t)).astype(np.int64) for t in (15, 17, 19, 21, 23))
    return np.where((v <= cls3) | (v <= 1024), table, dense)


def hash_col(c, bits):
    """hash_col() of csrc/spgemm.cu: (c * 2654435761 mod 2^32) >> (32 - bits)."""
    return ((np.asarray(c, dtype=np.uint64) * np.uint64(HASH_MUL)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - bits)


@functools.lru_cache(maxsize=None)
def colliding_columns(count, bits):
    """The `count` smallest columns that hash_col sends to slot 0 of a table of 2^bits slots."""
    found, lo, step = [], 0, 1 << 22
    while sum(len(f) for f in found) < count:
        c = np.arange(lo, lo + step, dtype=np.int64)
        found.append(c[hash_col(c, bits) == 0])
        lo += step
    return np.concatenate(found)[:count]


# ---- case builders: scipy CSR pairs with integer values, rows kept exactly as built ------------------------------
def int_values(rng, n):
    """n integers in [-8, 8] without 0."""
    return rng.integers(1, 9, n) * rng.choice(np.array([-1, 1]), n)


def csr_from_rows(rows, ncols, rng):
    """CSR whose row i stores the columns rows[i] in the given order (duplicates kept), with int_values."""
    indptr = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=indptr[1:])
    indices = np.concatenate([np.asarray(r, dtype=np.int64) for r in rows] + [np.zeros(0, dtype=np.int64)])
    return sp.csr_array((int_values(rng, len(indices)), indices, indptr), shape=(len(rows), ncols))


def own_b_rows(lengths_per_a_row, rng):
    """A references, per row, B rows of its own with the given lengths; every B row's columns are disjoint from every
    other's, so a row's nnz equals its product count.  Columns are scattered over [0, n) and sorted within a row."""
    n = int(sum(int(np.sum(ls)) for ls in lengths_per_a_row))
    perm = rng.permutation(n)
    a_rows, b_rows, col = [], [], 0
    for lens in lengths_per_a_row:
        a_rows.append(np.arange(len(b_rows), len(b_rows) + len(lens)))
        for L in lens:
            b_rows.append(np.sort(perm[col:col + int(L)]))
            col += int(L)
    return csr_from_rows(a_rows, len(b_rows), rng), csr_from_rows(b_rows, n, rng)


# product count of each row -> (symbolic class, numeric class); nnz == product count
LIMIT_ROWS = {0: (0, 0), 1: (1, 1), 31: (1, 1), 32: (1, 1), 33: (2, 2), 127: (2, 2), 128: (2, 2), 129: (3, 3),
              1023: (3, 3), 1024: (3, 3), 1025: (4, 10), 8191: (4, 10), 8192: (4, 10), 8193: (10, 10),
              2**15 - 1: (10, 10), 2**15 + 1: (9, 9), 2**17 - 1: (9, 9), 2**17 + 1: (8, 8)}


def case_class_limits(rng):
    """One row per product count of LIMIT_ROWS, spread over min(p, 37) B rows."""
    lengths = []
    for p in LIMIT_ROWS:
        q = min(p, 37)
        ls = np.full(q, p // q if q else 0)
        ls[: p - int(ls.sum())] += 1
        lengths.append(ls)
    A, B = own_b_rows(lengths, rng)
    return A, B, dict(enumerate(LIMIT_ROWS.values()))


# (distinct columns, B rows that repeat them) -> (symbolic class by d * r products, numeric class by d entries)
DISAGREE_ROWS = {(32, 20): (3, 1), (33, 20): (3, 2), (128, 20): (4, 2), (129, 20): (4, 3), (1024, 20): (10, 3),
                 (1025, 20): (10, 10), (5, 20000): (9, 1)}


def case_passes_disagree(rng):
    """Rows whose distinct-column count sits at a numeric limit while their product count is far higher: each row
    references r B rows that hold the same d columns, each in its own order, so the two passes bin it differently."""
    n = sum(d for d, _ in DISAGREE_ROWS)
    perm = rng.permutation(n)
    a_rows, b_rows, col = [], [], 0
    for d, r in DISAGREE_ROWS:
        cols = perm[col:col + d]
        col += d
        a_rows.append(np.arange(len(b_rows), len(b_rows) + r))
        b_rows += [rng.permutation(cols) for _ in range(r)]
    return csr_from_rows(a_rows, len(b_rows), rng), csr_from_rows(b_rows, n, rng), dict(enumerate(DISAGREE_ROWS.values()))


def case_collisions(table, rng):
    """Row 0 holds as many distinct columns as the table's class admits, all hashed to slot 0, spread over four B rows
    (products == nnz, so both passes pick the table by the same count); row 1 holds half of them."""
    d = TABLE_ROWS[table]
    cols = rng.permutation(colliding_columns(d, TABLE_BITS[table]))
    b_rows = [np.sort(part) for part in np.array_split(cols, 4)]
    A = csr_from_rows([np.arange(4), np.array([1, 3])], 4, rng)
    B = csr_from_rows(b_rows, int(cols.max()) + 1, rng)
    return A, B, {0: TABLE_CLASSES[table], 1: TABLE_CLASSES[table]}


# A rows longer than one round of the warp (32 entries), the 128-thread CTA and the 256-thread CTA and dense kernels,
# referencing empty B rows: (entries, B-row lengths to draw from, entries forced empty, (symbolic, numeric) class)
OWNER_ROWS = [
    (70, [0, 0, 0, 1], [0, 31, *range(32, 64), 64], (1, 1)),
    (100, [0, 1, 1, 2], [0, 31, 32, 63, 64, 95, 96, 99], (2, 2)),
    (300, [0, 0, 1, 2, 3, 4], [0, 127, 128, 255, 256, 299, *range(140, 180)], (3, 3)),
    (600, [0, 0, 1, 1, 2, 5, 9], [0, 255, 256, 511, 512, 599, *range(300, 340)], (4, 10)),
    (700, [0, 0, 1, 8, 24, 40, 64], [0, 255, 256, 511, 512, 699, *range(300, 340)], (10, 10)),
]


def case_owner_search(rng):
    """The owner search of the flattened expansion (largest t with excl_t <= p) has to skip empty B rows: at a round's
    first and last lane, in whole rounds of them, and between the U = 4 / U = 8 products a thread takes at once
    (lengths of 0 and 1 next to each other)."""
    lengths = []
    for entries, draw, empty, _ in OWNER_ROWS:
        ls = rng.choice(np.array(draw), entries)
        ls[np.array(empty)] = 0
        lengths.append(ls)
    A, B = own_b_rows(lengths, rng)
    return A, B, {i: row[3] for i, row in enumerate(OWNER_ROWS)}


def case_malformed(rng):
    """Unsorted rows, duplicate (row, column) entries, explicit zeros, empty rows in A and B, one B row referenced by
    every non-empty A row, and a row whose products cancel exactly (A row 50 = 3 * (B row 11 - B row 12), equal rows)."""
    m, k, n = 300, 400, 500
    b_rows = [rng.choice(n, int(rng.integers(0, 13)), replace=False) for _ in range(k)]
    for i in (0, 3, 5, 199, 200, 399):
        b_rows[i] = np.zeros(0, dtype=np.int64)
    b_rows[7] = rng.choice(n, 50, replace=False)
    b_rows[11] = rng.choice(n, 30, replace=False)
    for i in rng.choice(k, 40, replace=False):
        if len(b_rows[i]):
            b_rows[i] = np.concatenate([b_rows[i], b_rows[i][:2]])
    b_rows[12] = b_rows[11]
    B = csr_from_rows(b_rows, n, rng)
    B.data[rng.random(B.nnz) < 0.1] = 0
    s11, s12 = slice(B.indptr[11], B.indptr[12]), slice(B.indptr[12], B.indptr[13])
    B.data[s12] = B.data[s11]
    a_rows = [np.concatenate([rng.choice(k, int(rng.integers(0, 16)), replace=False), [7]]) for _ in range(m)]
    for i in rng.choice(m, 30, replace=False):
        a_rows[i] = np.concatenate([a_rows[i], a_rows[i][:3]])
    for i in (0, *range(10, 20), m - 1):
        a_rows[i] = np.zeros(0, dtype=np.int64)
    a_rows[50] = np.array([12, 11])
    A = csr_from_rows(a_rows, k, rng)
    A.data[rng.random(A.nnz) < 0.1] = 0
    A.data[A.indptr[50]:A.indptr[51]] = [-3, 3]
    return A, B, {}


def case_degenerate(shape_a, n, a_per_row, b_per_row, classes, rng):
    """A of shape_a with a_per_row entries per row (in random order), B with n columns and b_per_row per row."""
    m, k = shape_a
    A = csr_from_rows([rng.choice(k, min(k, a_per_row), replace=False) for _ in range(m)], k, rng)
    B = csr_from_rows([rng.choice(n, min(n, b_per_row), replace=False) for _ in range(k)], n, rng)
    return A, B, classes


CASES = {
    "class_limits": case_class_limits,
    "passes_disagree": case_passes_disagree,
    **{f"collide{t}": functools.partial(case_collisions, t) for t in TABLE_BITS},
    "owner_search": case_owner_search,
    "malformed": case_malformed,
    "m0": functools.partial(case_degenerate, (0, 5), 4, 2, 2, {}),
    "k0": functools.partial(case_degenerate, (3, 0), 4, 2, 2, {0: (0, 0)}),
    "n0": functools.partial(case_degenerate, (3, 5), 0, 2, 2, {0: (0, 0)}),
    "n1": functools.partial(case_degenerate, (50, 40), 1, 5, 1, {0: (1, 1)}),
    "a_without_entries": functools.partial(case_degenerate, (20, 30), 40, 0, 4, {0: (0, 0)}),
    "hub_row": functools.partial(case_degenerate, (1, 3000), 500, 3000, 3, {0: (10, 3)}),
}


@functools.lru_cache(maxsize=None)
def case(name):
    """(A, B, {row: (symbolic class, numeric class)}) of CASES[name], seeded by the name.  The arrays are read-only:
    scipy sorts and merges a matrix's entries in place in some operations (abs, astype), which would quietly turn the
    malformed operands into canonical ones."""
    A, B, classes = CASES[name](np.random.default_rng(sum(name.encode())))
    for a in (A.data, A.indices, A.indptr, B.data, B.indices, B.indptr):
        a.flags.writeable = False
    return A, B, classes


# ---- references ----------------------------------------------------------------------------------------------------
def compact_product(A, B):
    """(indptr, indices, data) of A @ B with rows sorted by column, computed by scipy on the columns B stores only (its
    product allocates work arrays as long as B's column count) and mapped back.  scipy leaves out entries that sum to
    zero; `on_pattern` puts them back."""
    cols, inv = np.unique(np.asarray(B.indices, dtype=np.int64), return_inverse=True)
    Bc = sp.csr_array((B.data, inv.reshape(-1), B.indptr), shape=(B.shape[0], max(len(cols), 1)))
    C = sp.csr_array(A @ Bc)
    C.sort_indices()
    return C.indptr.astype(np.int64), cols[C.indices].astype(np.int64), C.data


def with_data(S, data):
    """S's rows exactly as stored (duplicates and explicit zeros included) with the values `data`."""
    return sp.csr_array((data, S.indices, S.indptr), shape=S.shape)


def pattern(S):
    """S with every stored entry replaced by an int64 one."""
    return with_data(S, np.ones(S.nnz, dtype=np.int64))


def on_pattern(P, V):
    """The values of the product V at the positions of the pattern product P (0 where V has no entry)."""
    def keys(t):
        rows = np.repeat(np.arange(len(t[0]) - 1, dtype=np.int64), np.diff(t[0]))
        return rows * (1 << 32) + t[1]

    pk, vk = keys(P), keys(V)
    pos = np.searchsorted(pk, vk)
    assert np.array_equal(pk[pos], vk), "the product has an entry outside the pattern product"
    out = np.zeros(len(pk), dtype=V[2].dtype)
    out[pos] = V[2]
    return out


@functools.lru_cache(maxsize=None)
def exact_reference(name):
    """(P, values): P = (indptr, indices, k) is the pattern product (k = products behind each entry); values the int64
    product on P's positions."""
    A, B, _ = case(name)
    P = compact_product(pattern(A), pattern(B))
    return P, on_pattern(P, compact_product(A, B))


def random_valued(S, dtype, rng):
    """S with standard-normal values of `dtype` (explicit zeros stay zero)."""
    return with_data(S, np.where(S.data == 0, 0, rng.standard_normal(S.nnz)).astype(dtype))


def error_bound(P, A, B, dtype):
    """(fp64 reference, bound) on P's positions: |c - ref| <= 2 k u (|A||B|)."""
    A64, B64 = with_data(A, A.data.astype(np.float64)), with_data(B, B.data.astype(np.float64))
    ref = on_pattern(P, compact_product(A64, B64))
    absab = on_pattern(P, compact_product(with_data(A, np.abs(A64.data)), with_data(B, np.abs(B64.data))))
    return ref, 2.0 * P[2] * UNIT_ROUNDOFF[dtype] * absab


# ---- running on the GPU ------------------------------------------------------------------------------------------
def to_gpu(S, dtype):
    """sparse.csr_array of S's arrays as stored, values in `dtype`; index widths follow B2S_INDEX_WIDTH."""
    return sparse.csr_array((S.data.astype(dtype), np.array(S.indices), np.array(S.indptr)), shape=S.shape)


def gpu_product(A, B, dtype):
    """A @ B on the GPU; under B2S_INDEX_WIDTH=64 both operands carry int64 row pointers, so the kernels run their
    P = int64_t instantiations."""
    GA, GB = to_gpu(A, dtype), to_gpu(B, dtype)
    want = torch.int64 if os.environ.get("B2S_INDEX_WIDTH") == "64" else torch.int32
    assert GA.indptr.dtype == GB.indptr.dtype == want
    C = GA @ GB
    assert C.indptr.dtype == want and C.shape == (A.shape[0], B.shape[1])
    return C


def row_sums(P):
    """Products behind each row of the pattern product P."""
    cs = np.concatenate([[0], np.cumsum(P[2])])
    return cs[P[0][1:]] - cs[P[0][:-1]]


def row_classes(P, dense_min=NUMERIC_CLS3):
    """(symbolic class, numeric class) of every row of the product whose pattern product is P, as an (m, 2) array."""
    return np.stack([classify(row_sums(P), SYMBOLIC_CLS3), classify(np.diff(P[0]), dense_min)], axis=1)


def triple(C):
    return (C.indptr.cpu().numpy().astype(np.int64), C.indices.cpu().numpy().astype(np.int64),
            C.data.cpu().numpy())


def assert_structure(C, P):
    cp, ci, _ = triple(C)
    assert np.array_equal(cp, P[0]), f"indptr differs from row {int(np.argmax(cp != P[0])) - 1}"
    assert np.array_equal(ci, P[1]), f"indices differ from entry {int(np.argmax(ci != P[1]))}"


def assert_exact(C, P, values, dtype):
    assert_structure(C, P)
    cv = triple(C)[2]
    assert cv.dtype == dtype
    bad = np.flatnonzero(cv != values)
    assert bad.size == 0, f"{bad.size} values differ, first at entry {bad[0]}: {cv[bad[0]]} != {values[bad[0]]}"


def assert_info(C, P, products, dense_min=NUMERIC_CLS3):
    nnz = np.diff(P[0])
    assert C.spgemm_info["nnz"] == len(P[1])
    assert C.spgemm_info["products"] == products
    assert C.spgemm_info["dense_rows"] == int((nnz > dense_min).sum())


def check_exact(name, dtype, dense_min=NUMERIC_CLS3):
    A, B, _ = case(name)
    P, values = exact_reference(name)
    C = gpu_product(A, B, dtype)
    assert_exact(C, P, values, dtype)
    assert_info(C, P, int(P[2].sum()), dense_min)
    return C


def _use_width(monkeypatch, width):
    if width == "64":
        monkeypatch.setenv("B2S_INDEX_WIDTH", "64")
    else:
        monkeypatch.delenv("B2S_INDEX_WIDTH", raising=False)


# ---- tests -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("width", WIDTHS)
def test_integer_values_are_exact(name, dtype, width, monkeypatch):
    """Every case on integer data: structure, values and the products / dense-row counts exact; the rows sit in the
    classes the case claims for them."""
    _use_width(monkeypatch, width)
    _, _, classes = case(name)
    P, _ = exact_reference(name)
    rows = sorted(classes)
    assert [list(classes[r]) for r in rows] == row_classes(P)[rows].tolist()
    check_exact(name, dtype)


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("dtype", TYPES)
def test_random_values_within_the_forward_error_bound(name, dtype, monkeypatch):
    """Every case on standard-normal data: the structure exact, every value within 2 k u (|A||B|) of the fp64 product."""
    _use_width(monkeypatch, "32")
    A, B, _ = case(name)
    P, _ = exact_reference(name)
    rng = np.random.default_rng(7)
    A, B = random_valued(A, dtype, rng), random_valued(B, dtype, rng)
    ref, bound = error_bound(P, A, B, dtype)
    C = gpu_product(A, B, dtype)
    assert_structure(C, P)
    err = np.abs(triple(C)[2].astype(np.float64) - ref)
    bad = np.flatnonzero(err > bound)
    assert bad.size == 0, f"{bad.size} entries beyond the bound, first at {bad[0]}: error {err[bad[0]]}, bound {bound[bad[0]]}"


def test_warp_rows_repeat_bit_for_bit(monkeypatch):
    """Rows the numeric pass gives the warp kernel are summed without atomics: two products agree bit for bit there,
    even where one row adds 20000 products per entry."""
    _use_width(monkeypatch, "32")
    A, B, classes = case("passes_disagree")
    rng = np.random.default_rng(3)
    A, B = random_valued(A, np.float64, rng), random_valued(B, np.float64, rng)
    C1, C2 = gpu_product(A, B, np.float64), gpu_product(A, B, np.float64)
    ptr = triple(C1)[0]
    warp = [r for r, (_, num) in classes.items() if num in (1, 2)]
    assert len(warp) == 4
    for r in warp:
        assert torch.equal(C1.data[ptr[r]:ptr[r + 1]], C2.data[ptr[r]:ptr[r + 1]]), f"row {r}"


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("n", [100_003, 1 << 23, (1 << 23) + 1])
@pytest.mark.parametrize("l1_global", [False, True])
def test_dense_rows_reach_both_column_edges(n, l1_global, dtype, width, monkeypatch):
    """Dense rows touching columns 0 and n - 1 and level-0 / level-1 word edges, at n = 2^23 (the largest level-1
    bitmap that fits shared memory), 2^23 + 1 and a column count that is not a multiple of 32; with the level-1
    bitmap where the kernel puts it and forced into global memory."""
    _use_width(monkeypatch, width)
    if l1_global:
        monkeypatch.setenv("B2S_SPGEMM_L1_GLOBAL", "1")
    rng = np.random.default_rng(n)
    edges = np.array([0, 31, 32, 1023, 1024, n - 1025, n - 33, n - 32, n - 2, n - 1])
    b_rows = [np.sort(rng.choice(n, 300, replace=False)) for _ in range(40)]
    b_rows[0] = np.union1d(b_rows[0], edges)
    b_rows[39] = np.union1d(b_rows[39], [n - 1])
    A = csr_from_rows([np.arange(40), np.array([0, 5, 9, 20, 39]), [], [39]], 40, rng)
    B = csr_from_rows(b_rows, n, rng)
    P = compact_product(pattern(A), pattern(B))
    values = on_pattern(P, compact_product(A, B))
    assert row_classes(P).tolist() == [[10, 10], [4, 10], [0, 0], [3, 3]]
    C = gpu_product(A, B, dtype)
    assert_exact(C, P, values, dtype)
    assert_info(C, P, int(P[2].sum()))
    assert P[1][P[0][1] - 1] == n - 1 and P[1][0] == 0


def test_wide_rule_gives_64_bit_result_indices(monkeypatch):
    """Under B2S_INDEX_WIDTH=64 the product's indices are int64 like its indptr, as kron / bmat give them."""
    _use_width(monkeypatch, "64")
    A, B, _ = case("malformed")
    C = gpu_product(A, B, np.float64)
    assert C.indptr.dtype == C.indices.dtype == torch.int64
    P, values = exact_reference("malformed")
    assert_exact(C, P, values, np.float64)
    _use_width(monkeypatch, "32")
    assert gpu_product(A, B, np.float64).indices.dtype == torch.int32


def test_bitmap_scratch_is_bounded():
    """The dense kernel's bitmap slots (about n/8 bytes each, 4 per SM) stay within 1 GiB: at the column counts of the
    benchmark's products every slot is kept, and 2^31 - 2 columns need less than 1 GiB of scratch."""
    from legate.sparse_b200._ops import L

    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def slot_bytes(n):
        w0 = (n + 31) // 32
        return (4 * (w0 + (w0 + 31) // 32) + 255) // 256 * 256

    for n in (10**6, 1 << 22):
        assert L.b2s_spgemm_scratch_bytes(1, n) - L.b2s_spgemm_scratch_bytes(1, 0) == 4 * sms * slot_bytes(n)
    assert 0 < L.b2s_spgemm_scratch_bytes(3, 2**31 - 2) < 1 << 30


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("width", WIDTHS)
def test_wide_b_with_three_entries(dtype, width, monkeypatch):
    """B with 2^31 - 2 columns (the most the entry points accept) and a product of 3 entries at columns 0 and n - 1:
    correct, and less than 1 GiB of device memory in all."""
    _use_width(monkeypatch, width)
    n = 2**31 - 2
    A = sp.csr_array((np.array([1, 2, 3]), np.array([0, 2, 1]), np.array([0, 2, 3])), shape=(2, 3))
    B = sp.csr_array((np.array([4, 5, 6]), np.array([0, n - 1, n - 1]), np.array([0, 2, 3, 3])), shape=(3, n))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    C = gpu_product(A, B, dtype)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < 1 << 30
    cp, ci, cv = triple(C)
    assert cp.tolist() == [0, 2, 3] and ci.tolist() == [0, n - 1, n - 1] and cv.tolist() == [4, 5, 18]
    assert C.spgemm_info == {"nnz": 3, "products": 3, "dense_rows": 0}


def test_dense_row_at_2_28_columns(monkeypatch):
    """One dense row (in both passes) of a B with 2^28 + 3 columns, in fp32: about 1 GiB of accumulators and a level-1
    bitmap in global memory."""
    _use_width(monkeypatch, "32")
    n = (1 << 28) + 3
    if torch.cuda.mem_get_info()[0] < 4 << 30:
        pytest.skip("not enough free device memory for the fp32 dense accumulator of one row of 2^28 + 3 columns")
    rng = np.random.default_rng(28)
    b_rows = [rng.choice(n, 1000, replace=False) for _ in range(10)]
    b_rows[0] = np.union1d(b_rows[0], [0, n - 1])
    A = csr_from_rows([np.arange(10)], 10, rng)
    B = csr_from_rows(b_rows, n, rng)
    P = compact_product(pattern(A), pattern(B))
    assert row_classes(P).tolist() == [[10, 10]]
    C = gpu_product(A, B, np.float32)
    assert_exact(C, P, on_pattern(P, compact_product(A, B)), np.float32)
    assert_info(C, P, int(P[2].sum()))
    assert P[1][0] == 0 and P[1][-1] == n - 1


def dense_min_child():
    """Body of test_numeric_16384_slot_table, run with B2S_SPGEMM_DENSE_MIN=8192 set before the first product: rows of
    1025..8192 entries take the numeric 16384-slot table instead of the dense kernel."""
    assert os.environ["B2S_SPGEMM_DENSE_MIN"] == "8192"
    for name in ("class_limits", "collide16384", "owner_search"):
        for width in WIDTHS:
            os.environ["B2S_INDEX_WIDTH"] = "64" if width == "64" else ""
            for dtype in TYPES:
                check_exact(name, dtype, dense_min=8192)
    print("dense-min child ok")


def test_numeric_16384_slot_table():
    """B2S_SPGEMM_DENSE_MIN is read once per process, so the numeric 16384-slot table is tested in a child process."""
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n" \
           "import test_gpu_spgemm_classes as t; t.dense_min_child()"
    env = dict(os.environ, B2S_SPGEMM_DENSE_MIN="8192")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0 and "dense-min child ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("budget", ["one_row", "below_heaviest", "total"])
def test_chunked_driver(budget, monkeypatch):
    """csr.spgemm_chunked on the class-limits matrix: chunks are greedy ranges within the budget, a row heavier than the
    budget is a chunk of its own, and the concatenated product equals the unchunked one bit for bit."""
    from legate.sparse_b200.csr import spgemm_chunked

    _use_width(monkeypatch, "32")
    A, B, _ = case("class_limits")
    row_work = row_sums(exact_reference("class_limits")[0])
    limit = {"one_row": 1025, "below_heaviest": 1000, "total": int(row_work.sum())}[budget]
    GA, GB = to_gpu(A, np.float64), to_gpu(B, np.float64)
    seen = []
    C, st = spgemm_chunked(GA, GB, max_products=limit, keep=True, on_chunk=lambda lo, hi, Cc: seen.append((lo, hi)))
    assert seen[0][0] == 0 and seen[-1][1] == A.shape[0] and all(a[1] == b[0] for a, b in zip(seen, seen[1:]))
    for lo, hi in seen:
        w = int(row_work[lo:hi].sum())
        assert w <= limit or hi - lo == 1
        assert hi == A.shape[0] or w + row_work[hi] > limit          # greedy: the next row would not have fitted
    if budget == "below_heaviest":
        assert (int(np.argmax(row_work)), int(np.argmax(row_work)) + 1) in seen
    if budget == "total":
        assert len(seen) == 1
    full = GA @ GB
    assert st["products"] == int(row_work.sum()) and st["nnz"] == full.nnz
    assert torch.equal(C.indptr.to(torch.int64), full.indptr.to(torch.int64))
    assert torch.equal(C.indices, full.indices) and torch.equal(C.data, full.data)
    P, values = exact_reference("class_limits")
    assert_exact(C, P, values, np.float64)
