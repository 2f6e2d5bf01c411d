"""Host-side checks of `random`, `rand` and `random_array` (csrc/random.cu through `_ops.random_csr`).

`random_oracle` restates the whole device sampler with numpy: Philox4x64-10 on uint64 arrays, Lemire's multiply-high
with rejection, the rounds as set unions, the complement, canonical order and the values.  Its block function is pinned
to numpy.random.Philox, which implements the same generator, and the GPU tests (tests/test_gpu_random.py) compare the
device arrays with it byte for byte.  Here the restatement itself is checked: exact counts, no duplicates, sorted
rows, the complement path, and uniformity over subsets.  Argument handling is pinned to scipy 1.18.1."""
import math

import numpy as np
import pytest
import scipy.sparse as sp

import legate.sparse_b200 as sparse
from legate.sparse_b200 import module


@pytest.fixture(autouse=True)
def _host_only(monkeypatch):
    """Operands stay on the host, also where a GPU is visible: every call that passes its checks then stops at the
    missing device."""
    from legate.sparse_b200.runtime import Runtime

    monkeypatch.setattr(Runtime, "has_cuda", property(lambda self: False))


# ---- the restatement --------------------------------------------------------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)
_PHILOX_M = (np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157))
_PHILOX_W = (np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B))


def _mulhi(a, b):
    """high 64 bits of the 128-bit products a * b (uint64 arrays), from 32-bit halves"""
    a, b = np.broadcast_arrays(np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64))
    s32 = np.uint64(32)
    al, ah, bl, bh = a & _M32, a >> s32, b & _M32, b >> s32
    ll, lh, hl, hh = al * bl, al * bh, ah * bl, ah * bh
    mid = (ll >> s32) + (lh & _M32) + (hl & _M32)
    return hh + (lh >> s32) + (hl >> s32) + (mid >> s32)


def philox4x64_10(key, ctr):
    """The Philox4x64-10 blocks of `key` = (k0, k1) at counters `ctr` = (c0, c1, c2, c3), each a uint64 scalar or
    array: four uint64 arrays, words 0..3."""
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    c = [np.array(x, dtype=np.uint64, ndmin=1) for x in np.broadcast_arrays(*[np.asarray(x, dtype=np.uint64)
                                                                                for x in ctr])]
    for r in range(10):
        if r:
            with np.errstate(over="ignore"):   # the key schedule wraps mod 2^64
                k0, k1 = k0 + _PHILOX_W[0], k1 + _PHILOX_W[1]
        hi0, lo0 = _mulhi(_PHILOX_M[0], c[0]), _PHILOX_M[0] * c[0]
        hi1, lo1 = _mulhi(_PHILOX_M[1], c[2]), _PHILOX_M[1] * c[2]
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return c


def _draws(seed, rnd, need, mn):
    """draws 0..need-1 of round `rnd`: positions in [0, mn), each retried with attempt a + 1 while Lemire rejects it"""
    out = np.empty(need, dtype=np.uint64)
    pending = np.arange(need, dtype=np.uint64)
    umn = np.uint64(mn)
    reject_below = np.uint64((2**64 - mn) % mn)
    a = 0
    while pending.size:
        w0 = philox4x64_10((seed, 0), (pending, rnd, a, 0))[0]
        ok = w0 * umn >= reject_below
        out[pending[ok].astype(np.int64)] = _mulhi(w0[ok], umn)
        pending = pending[~ok]
        a += 1
    return out


def random_oracle(shape, density, seed, dtype):
    """(indptr, indices, data, rounds) of the device sampler for `shape`, `density`, the 64-bit `seed` and `dtype`:
    int64 indptr and indices, data in `dtype`"""
    indptr, indices, rounds = oracle_structure(shape, density, seed)
    return indptr, indices, oracle_values(indices.size, seed, dtype), rounds


def oracle_structure(shape, density, seed):
    """(indptr, indices, rounds) of `random_oracle`"""
    m, n = shape
    mn = m * n
    k = int(round(density * mn))
    complement = k > mn - k
    s = mn - k if complement else k
    taken = np.zeros(0, dtype=np.uint64)
    rounds = 0
    while taken.size < s:
        taken = np.union1d(taken, _draws(seed, rounds, s - taken.size, mn))
        rounds += 1
    pos = np.setdiff1d(np.arange(mn, dtype=np.uint64), taken) if complement else taken
    pos = pos.astype(np.int64)
    rows, cols = pos // max(n, 1), pos % max(n, 1)
    indptr = np.zeros(m + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=m), out=indptr[1:])
    return indptr, cols, rounds


def oracle_values(k, seed, dtype):
    """the k values of `random_oracle`, in canonical order"""
    w = philox4x64_10((seed, 1), (np.arange(k, dtype=np.uint64), 0, 0, 0)) if k else [np.zeros(0, np.uint64)] * 2
    dtype = np.dtype(dtype)
    if dtype in (np.float32, np.complex64):
        part = [(x >> np.uint64(40)).astype(np.float32) * np.float32(2.0**-24) for x in w[:2]]
    else:
        part = [(x >> np.uint64(11)).astype(np.float64) * 2.0**-53 for x in w[:2]]
    data = np.empty(k, dtype=dtype)
    data.real = part[0]
    if dtype.kind == "c":
        data.imag = part[1]
    return data


def _philox_numpy(key, ctr):
    """numpy.random.Philox's block at counter `ctr`: numpy adds one to its counter (with carry) before each block"""
    c = (sum(int(x) << (64 * i) for i, x in enumerate(ctr)) - 1) % 2**256
    bg = np.random.Philox(key=np.array(key, dtype=np.uint64),
                          counter=np.array([(c >> (64 * i)) & (2**64 - 1) for i in range(4)], dtype=np.uint64))
    return bg.random_raw(4)


@pytest.mark.parametrize("key, ctr", [((0, 0), (0, 0, 0, 0)), ((123, 0), (5, 7, 0, 0)), ((2**64 - 1, 1), (3, 0, 1, 0)),
                                      ((0xDEADBEEF, 0), (2**64 - 1, 2**64 - 1, 9, 2**63)), ((77, 1), (1, 2, 3, 4))])
def test_philox_block_matches_numpy(key, ctr):
    assert np.array_equal(np.concatenate(philox4x64_10(key, ctr)), _philox_numpy(key, ctr))


def test_philox_is_vectorised_per_counter():
    ctrs = np.arange(5, dtype=np.uint64) * np.uint64(0x1234567)
    words = philox4x64_10((9, 0), (ctrs, 2, 0, 0))
    for j, c in enumerate(ctrs):
        assert [w[j] for w in words] == list(_philox_numpy((9, 0), (c, 2, 0, 0)))


def test_lemire_mapping_is_multiply_high():
    """a draw maps to floor(w0 * mn / 2^64), unless its low word falls in the biased band"""
    for mn in (1, 6, 1000, 2**40 + 3, 2**63 - 1):
        p = _draws(11, 0, 64, mn)
        assert (p < np.uint64(mn)).all()
        w0 = philox4x64_10((11, 0), (np.arange(64, dtype=np.uint64), 0, 0, 0))[0]
        accepted = [int(x) * mn % 2**64 >= (2**64 - mn) % mn for x in w0]
        for j in np.flatnonzero(accepted):
            assert int(p[j]) == int(w0[j]) * mn >> 64


def _check_canonical(indptr, indices, shape, k):
    m, n = shape
    assert indptr[0] == 0 and indptr[-1] == k and indices.size == k and (np.diff(indptr) >= 0).all()
    assert ((indices >= 0) & (indices < max(n, 1))).all()
    for i in range(m):
        row = indices[indptr[i]:indptr[i + 1]]
        assert (np.diff(row) > 0).all()   # sorted, so no repeated position


@pytest.mark.parametrize("shape", [(0, 5), (5, 0), (1, 1), (1, 100), (100, 1), (30, 70), (64, 64)])
@pytest.mark.parametrize("density", [0.0, 1e-3, 0.01, 0.3, 0.5, 0.9, 1.0])
def test_oracle_exact_count_sorted_unique(shape, density):
    k = int(round(density * math.prod(shape)))
    indptr, indices, data, _ = random_oracle(shape, density, 42, np.float64)
    _check_canonical(indptr, indices, shape, k)
    assert data.shape == (k,) and ((data >= 0) & (data < 1)).all()


@pytest.mark.parametrize("shape", [(7, 9), (30, 70), (64, 64)])
def test_oracle_complement_path(shape):
    """densities 0.5 (k = mn - k samples the entries), 0.5 + 1/mn, 0.9 and 1.0 (the zeros, then their complement)"""
    mn = math.prod(shape)
    for density in (0.5, 0.5 + 1 / mn, 0.9, 1.0):
        k = int(round(density * mn))
        indptr, indices, _, rounds = random_oracle(shape, density, 3, np.float32)
        _check_canonical(indptr, indices, shape, k)
        if density == 1.0:
            assert rounds == 0 and np.array_equal(indices, np.tile(np.arange(shape[1]), shape[0]))


def test_oracle_values_follow_the_formula():
    _, _, d32, _ = random_oracle((10, 10), 0.3, 5, np.float32)
    _, _, d64, _ = random_oracle((10, 10), 0.3, 5, np.float64)
    _, _, z128, _ = random_oracle((10, 10), 0.3, 5, np.complex128)
    _, _, z64, _ = random_oracle((10, 10), 0.3, 5, np.complex64)
    assert d32.dtype == np.float32 and np.array_equal(z64.real, d32) and np.array_equal(z128.real, d64)
    w = philox4x64_10((5, 1), (np.arange(30, dtype=np.uint64), 0, 0, 0))
    assert np.array_equal(d64, (w[0] >> np.uint64(11)).astype(np.float64) / 2.0**53)
    assert np.array_equal(z128.imag, (w[1] >> np.uint64(11)).astype(np.float64) / 2.0**53)
    assert np.array_equal(d32, ((w[0] >> np.uint64(40)).astype(np.float64) / 2.0**24).astype(np.float32))


SUBSET_SEEDS = 3000
SUBSET_CHI2_MAX = 40.0   # chi-square, 14 degrees of freedom: P(X > 40) is about 2.6e-4


def subset_chi2(sample):
    """chi-square of the 15 two-element subsets of a 2 x 3 matrix over SUBSET_SEEDS calls of sample(seed), which
    returns the sorted row-major positions of a density-1/3 sample"""
    counts = {}
    for seed in range(SUBSET_SEEDS):
        key = tuple(int(p) for p in sample(seed))
        assert len(key) == 2 and key[0] < key[1]
        counts[key] = counts.get(key, 0) + 1
    assert len(counts) == 15
    expected = SUBSET_SEEDS / 15
    return sum((c - expected) ** 2 / expected for c in counts.values())


def test_oracle_uniform_over_subsets():
    def sample(seed):
        indptr, indices, _, _ = random_oracle((2, 3), 1 / 3, seed, np.float64)
        return np.repeat(np.arange(2), np.diff(indptr)) * 3 + indices

    assert subset_chi2(sample) < SUBSET_CHI2_MAX


# ---- argument handling, pinned to scipy 1.18.1 -------------------------------------------------------------------------
CALLS = {
    "random": lambda shape, **kw: sparse.random(shape[0], shape[1], **kw),
    "rand": lambda shape, **kw: sparse.rand(shape[0], shape[1], **kw),
    "random_array": lambda shape, **kw: sparse.random_array(shape, **kw),
}
SCIPY_CALLS = {
    "random": lambda shape, **kw: sp.random(shape[0], shape[1], **kw),
    "rand": lambda shape, **kw: sp.rand(shape[0], shape[1], **kw),
    "random_array": lambda shape, **kw: sp.random_array(shape, **kw),
}


def _raises(f):
    try:
        f()
    except Exception as e:  # noqa: BLE001
        return type(e), str(e)
    return None, None


@pytest.mark.parametrize("name", CALLS)
@pytest.mark.parametrize("density", [-0.1, 1.5, float("nan")])
def test_density_errors_as_scipy(name, density):
    theirs = _raises(lambda: SCIPY_CALLS[name]((4, 5), density=density, rng=1))
    ours = _raises(lambda: CALLS[name]((4, 5), density=density, rng=1))
    assert theirs[0] is ValueError and ours[0] is ValueError
    if not math.isnan(density):
        assert ours[1] == theirs[1] == "density expected to be 0 <= density <= 1"


@pytest.mark.parametrize("name", CALLS)
@pytest.mark.parametrize("shape", [(-1, 5), (5, -1), (-2, -3), (0, -1)])
def test_negative_shape_errors_as_scipy(name, shape):
    theirs = _raises(lambda: SCIPY_CALLS[name](shape, density=0.5, rng=1))
    ours = _raises(lambda: CALLS[name](shape, density=0.5, rng=1))
    assert theirs[0] is ValueError and ours[0] is ValueError


@pytest.mark.parametrize("name", CALLS)
def test_unsupported_formats_and_dtypes(name):
    for fmt in ("bsr", "lil", "dok", "nonsense", None):
        with pytest.raises(NotImplementedError, match="format"):
            CALLS[name]((4, 5), density=0.5, format=fmt, rng=1)
    for dt in (np.int32, np.int64, np.bool_, np.float16, np.uint8):
        with pytest.raises(NotImplementedError, match="float32, float64, complex64 and complex128"):
            CALLS[name]((4, 5), density=0.5, dtype=dt, rng=1)


def test_shapes_beyond_int64_and_not_2d():
    with pytest.raises(NotImplementedError, match="int64"):
        sparse.random(2**32, 2**32, 0.0)
    for shape in ((5,), (2, 3, 4)):
        with pytest.raises(NotImplementedError, match="2-D"):
            sparse.random_array(shape, density=0.1)


def test_sampler_of_the_wrong_length():
    with pytest.raises(ValueError, match="data sampler"):
        sparse.random_array((10, 10), density=0.2, rng=0, data_sampler=lambda size: np.zeros(size + 1))
    with pytest.raises(ValueError, match="data sampler"):
        sparse.random(10, 10, 0.2, rng=0, data_rvs=lambda size: np.zeros((size, 2)))


def test_sampler_called_once_before_the_device():
    calls = []

    def sampler(size):
        calls.append(size)
        return np.ones(size)

    with pytest.raises(RuntimeError, match="no CUDA device"):
        sparse.random_array((10, 10), density=0.25, rng=0, data_sampler=sampler)
    assert calls == [25]


def test_stops_at_the_missing_device_after_its_checks():
    for call in (lambda: sparse.random(10, 10, 0.5, format="csr"), lambda: sparse.rand(3, 4, 1.0, format="csc"),
                 lambda: sparse.random_array((0, 0), format="dia", dtype=np.complex64)):
        with pytest.raises(RuntimeError, match="no CUDA device"):
            call()


def test_generator_advanced_by_one_draw():
    g, copy = np.random.default_rng(2024), np.random.default_rng(2024)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        sparse.random(50, 50, 0.1, rng=g)
    copy.bit_generator.random_raw()
    assert g.bit_generator.state == copy.bit_generator.state
    r, rcopy = np.random.RandomState(7), np.random.RandomState(7)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        sparse.random_array((50, 50), density=0.1, random_state=r)
    rcopy.randint(0, 2**64, dtype=np.uint64)
    assert all(np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b
               for a, b in zip(r.get_state(), rcopy.get_state()))


@pytest.fixture
def seeds(monkeypatch):
    """the 64-bit seed each call hands to the device, recorded instead of launching"""
    got = []

    def fake(shape, k, seed, *args):
        got.append(seed)
        raise _Launched

    monkeypatch.setattr(module.runtime, "require_cuda", lambda what: None)
    monkeypatch.setattr(module._ops, "random_csr", fake)
    return got


class _Launched(Exception):
    pass


def test_seed_resolution_as_scipy(seeds):
    """rng= goes through default_rng; random_state= and the sixth positional argument through check_random_state"""
    calls = [
        (lambda: sparse.random(6, 6, 0.5, rng=5), np.random.default_rng(5).integers(0, 2**64, dtype=np.uint64)),
        (lambda: sparse.random(6, 6, 0.5, random_state=5), np.random.RandomState(5).randint(0, 2**64, dtype=np.uint64)),
        (lambda: sparse.random(6, 6, 0.5, "csr", None, 5), np.random.RandomState(5).randint(0, 2**64, dtype=np.uint64)),
        (lambda: sparse.rand(6, 6, 0.5, "csr", np.float32, np.random.default_rng(8)),
         np.random.default_rng(8).integers(0, 2**64, dtype=np.uint64)),
        (lambda: sparse.random_array((6, 6), rng=9), np.random.default_rng(9).integers(0, 2**64, dtype=np.uint64)),
        (lambda: sparse.random_array((6, 6), random_state=9),
         np.random.RandomState(9).randint(0, 2**64, dtype=np.uint64)),
    ]
    for call, want in calls:
        with pytest.raises(_Launched):
            call()
        assert seeds[-1] == int(want)
    with pytest.raises(TypeError, match="multiple values"):
        sparse.random(6, 6, 0.5, rng=1, random_state=1)
    with pytest.raises(TypeError, match="multiple values"):
        sparse.random(6, 6, 0.5, "coo", None, 1, rng=1)
    with pytest.raises(ValueError, match="cannot be used to seed"):
        sparse.random(6, 6, 0.5, random_state="seed")


def test_reference_positional_order(seeds):
    """random(m, n, density, format, dtype, random_state, data_rvs): the reference's order works unchanged"""
    calls = []
    with pytest.raises(_Launched):
        sparse.random(4, 4, 0.5, "csr", np.float64, 3, lambda size: calls.append(size) or np.zeros(size))
    assert calls == [8] and seeds[-1] == int(np.random.RandomState(3).randint(0, 2**64, dtype=np.uint64))


def test_exported_from_both_namespaces():
    import sparse as alias

    for name in ("random", "rand", "random_array"):
        assert getattr(alias, name) is getattr(sparse, name) is getattr(module, name)
