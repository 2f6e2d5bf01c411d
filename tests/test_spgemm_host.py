"""Host-side checks of the SpGEMM case builders and references of tests/test_gpu_spgemm_classes.py: the numpy
restatements of the kernel's row classes and hash, the classes each case claims for its rows, the slot the collision
columns share, the 2^24 bound that keeps the integer cases exact in fp32, and the compacted-column reference."""
import numpy as np
import pytest
import scipy.sparse as sp

from test_gpu_spgemm_classes import (CASES, LIMIT_ROWS, NUMERIC_CLS3, SYMBOLIC_CLS3, TABLE_BITS, TABLE_ROWS, case,
                                     classify, compact_product, exact_reference, hash_col, on_pattern, pattern,
                                     random_valued, row_classes, with_data)


def classify_scalar(v, cls3):
    """classify() of csrc/spgemm.cu, statement for statement."""
    if v <= cls3 or v <= 1024:
        return 0 if v == 0 else (1 if v <= 32 else (2 if v <= 128 else (3 if v <= 1024 else 4)))
    sub, t = 5, 1 << 15
    while sub > 0 and v > t:
        sub -= 1
        t <<= 2
    return 5 + sub


@pytest.mark.parametrize("cls3", [NUMERIC_CLS3, 4096, SYMBOLIC_CLS3])
def test_classify_restatement(cls3):
    edges = [0, 1, 31, 32, 33, 127, 128, 129, 1023, 1024, 1025, 4095, 4096, 4097, 8191, 8192, 8193]
    edges += [(1 << t) + d for t in (15, 17, 19, 21, 23, 25) for d in (-1, 0, 1)]
    v = np.array(edges + list(np.random.default_rng(0).integers(0, 1 << 26, 2000)))
    assert classify(v, cls3).tolist() == [classify_scalar(int(x), cls3) for x in v]
    assert [(int(classify(p, SYMBOLIC_CLS3)), int(classify(p, NUMERIC_CLS3))) for p in LIMIT_ROWS] == \
        list(LIMIT_ROWS.values())


@pytest.mark.parametrize("name", [n for n in CASES if case(n)[2]])
def test_cases_put_their_rows_in_the_claimed_classes(name):
    _, _, classes = case(name)
    P, _ = exact_reference(name)
    rows = sorted(classes)
    assert [list(classes[r]) for r in rows] == row_classes(P)[rows].tolist()


def test_class_limit_rows_have_nnz_equal_to_products():
    P, _ = exact_reference("class_limits")
    assert np.diff(P[0]).tolist() == list(LIMIT_ROWS) and np.all(P[2] == 1)


def test_owner_search_rows_span_rounds_with_empty_b_rows():
    A, B, _ = case("owner_search")
    lens = np.diff(B.indptr)[A.indices]
    rows = [lens[A.indptr[i]:A.indptr[i + 1]] for i in range(A.shape[0])]
    assert [len(r) for r in rows] == [70, 100, 300, 600, 700]
    for r, rnd in zip(rows, (32, 32, 128, 256, 256)):
        assert r[0] == 0 and r[rnd - 1] == 0 and r[rnd] == 0 and r[-1] == 0
        assert np.any((r[:-1] == 0) & (r[1:] == 1)) and np.any((r[:-1] == 1) & (r[1:] == 0))
    assert not rows[0][32:64].any()        # a whole warp round of empty B rows


@pytest.mark.parametrize("table", list(TABLE_BITS))
def test_collision_columns_share_one_slot(table):
    A, B, _ = case(f"collide{table}")
    cols = B.indices[B.indptr[0]:B.indptr[4]].astype(np.int64)
    bits = TABLE_BITS[table]
    assert len(np.unique(cols)) == len(cols) == TABLE_ROWS[table]
    assert np.all(hash_col(cols, bits) == 0)
    assert [(int(c) * 2654435761 % 2**32) >> (32 - bits) for c in cols[:50]] == [0] * min(50, len(cols))
    P, _ = exact_reference(f"collide{table}")
    assert np.diff(P[0]).tolist() == [TABLE_ROWS[table], TABLE_ROWS[table] // 2]


@pytest.mark.parametrize("name", list(CASES))
def test_integer_cases_stay_below_2_24_in_every_partial_sum(name):
    """Every partial sum of an entry is at most (|A||B|)_ij in magnitude; below 2^24 fp32 adds it exactly."""
    A, B, _ = case(name)
    assert np.abs(A.data).max(initial=0) <= 8 and np.abs(B.data).max(initial=0) <= 8
    assert np.all(A.data == np.round(A.data)) and np.all(B.data == np.round(B.data))
    absab = compact_product(with_data(A, np.abs(A.data)), with_data(B, np.abs(B.data)))[2]
    assert absab.max(initial=0) < 2**24


def test_malformed_case_is_malformed():
    A, B, _ = case("malformed")
    for S in (A, B):
        rows = [S.indices[S.indptr[i]:S.indptr[i + 1]] for i in range(S.shape[0])]
        assert any(np.any(np.diff(r) < 0) for r in rows) and any(len(np.unique(r)) < len(r) for r in rows)
        assert np.any(S.data == 0) and np.any(np.diff(S.indptr) == 0)
    assert np.sum(A.indices == 7) > 250
    P, values = exact_reference("malformed")
    assert P[0][51] > P[0][50] and not values[P[0][50]:P[0][51]].any()     # exact cancellation, entries kept


SMALL = [((7, 9), 11, 0.3), ((0, 4), 5, 0.5), ((4, 0), 3, 0.5), ((5, 6), 0, 0.5), ((30, 40), 1, 0.2), ((20, 30), 50, 0.0)]


@pytest.mark.parametrize("shape_a,n,density", SMALL)
def test_compacted_reference_matches_scipy(shape_a, n, density):
    rng = np.random.default_rng(5)
    m, k = shape_a
    A = sp.random(m, k, density=density, random_state=rng, format="csr")
    B = sp.random(k, n, density=0.3, random_state=rng, format="csr")
    ptr, idx, val = compact_product(A, B)
    S = sp.csr_array(A @ B)
    S.sort_indices()
    assert np.array_equal(ptr, S.indptr) and np.array_equal(idx, S.indices) and np.allclose(val, S.data, rtol=1e-15)
    D = A.toarray() @ B.toarray()
    rows = np.repeat(np.arange(m), np.diff(ptr))
    dense = np.zeros((m, n))
    dense[rows, idx] = val
    assert np.allclose(dense, D, rtol=1e-14, atol=0)


@pytest.mark.parametrize("name", ["malformed", "hub_row", "n1", "collide64", "k0"])
def test_references_match_dense_products(name):
    """On non-canonical operands too (unsorted rows, duplicates, explicit zeros): the pattern product counts the
    products behind each entry, and the exact and random-valued references agree with dense numpy products."""
    A, B, _ = case(name)
    P, values = exact_reference(name)
    rows = np.repeat(np.arange(A.shape[0]), np.diff(P[0]))
    dense = np.zeros((A.shape[0], B.shape[1]), dtype=np.int64)
    dense[rows, P[1]] = values
    assert np.array_equal(dense, A.toarray() @ B.toarray())
    counts = np.zeros_like(dense)
    counts[rows, P[1]] = P[2]
    assert np.array_equal(counts, pattern(A).toarray() @ pattern(B).toarray())
    R = random_valued(A, np.float32, np.random.default_rng(1))
    assert np.array_equal(R.indices, A.indices) and np.array_equal(R.data == 0, A.data == 0)
    R64, B64 = with_data(R, R.data.astype(np.float64)), with_data(B, B.data.astype(np.float64))
    dense_r = np.zeros(dense.shape)
    dense_r[rows, P[1]] = on_pattern(P, compact_product(R64, B64))
    assert np.allclose(dense_r, R64.toarray() @ B64.toarray(), rtol=1e-12, atol=1e-12)
