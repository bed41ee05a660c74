"""The counter-based generator of the sampling loop (sat_sample_loop): a numpy copy of it equals the library's host
function sat_sample_uniform bit for bit, and its variates look uniform and independent.  No GPU needed."""
import numpy as np
import pytest

M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(z):
    z = np.asarray(z, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def sample_uniform(seed, row, step, word):
    """u(seed, row, step, word) = (bits + 0.5) * 2^-32 (include/sat_b200.h, sat_linear.cuh); broadcasts over arrays."""
    with np.errstate(over="ignore"):
        row = np.asarray(row, np.int64).astype(np.uint64)
        step = np.asarray(step, np.int64).astype(np.uint64) & np.uint64(0xFFFFFFFF)
        z = splitmix64(np.uint64(seed) ^ splitmix64((row << np.uint64(32)) | step))
        k0 = (z & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        k1 = (z >> np.uint64(32)).astype(np.uint32)
        x = np.asarray(word, np.int64).astype(np.uint32) ^ k0
        x ^= x >> np.uint32(16)
        x = x * np.uint32(0x7FEB352D)
        x ^= x >> np.uint32(15)
        x = x + k1
        x = x * np.uint32(0x846CA68B)
        x ^= x >> np.uint32(16)
    return (x.astype(np.float64) + 0.5) * 2.0 ** -32


def gumbel(u):
    return -np.log(-np.log(u))


@pytest.fixture(scope="module")
def lib(built_lib):
    import sat_b200
    return sat_b200.load_library()


def test_numpy_copy_matches_the_library(lib):
    seeds = [0, 1, 7, 0x9E3779B97F4A7C15, int(M64)]
    rows = [0, 1, 5, 63, 64, 65535, 65536, 70001, 2 ** 31 - 1]
    steps = [0, 1, 19, 29, 1000]
    words = [0, 1, 2, 127, 128, 4999, 9999, 65535, 65536, 99999, 2 ** 31 - 1]
    for s in seeds:
        for r in rows:
            for t in steps:
                got = np.array([lib.sat_sample_uniform(s, r, t, w) for w in words])
                exp = sample_uniform(s, r, t, np.array(words))
                assert np.array_equal(got, exp), (s, r, t)


def test_uniform_strictly_inside_the_unit_interval():
    u = sample_uniform(12345, np.arange(64)[:, None, None], np.arange(20)[None, :, None], np.arange(1000)[None, None, :])
    assert u.min() > 0.0 and u.max() < 1.0
    g = gumbel(u)
    assert np.isfinite(g).all()
    # the extreme values of a 32-bit variate: 0.5 * 2^-32 and 1 - 0.5 * 2^-32
    lo, hi = 0.5 * 2.0 ** -32, 1.0 - 0.5 * 2.0 ** -32
    assert np.isfinite(gumbel(np.array([lo, hi]))).all()
    assert gumbel(np.array([hi]))[0] > 22.0   # (a 24-bit variate stops near 16.6)


def test_kolmogorov_smirnov():
    from scipy import stats
    u = sample_uniform(2024, np.arange(128)[:, None, None], np.arange(8)[None, :, None],
                       np.arange(1000)[None, None, :]).ravel()
    assert u.size >= 10 ** 6
    assert stats.kstest(u, "uniform").pvalue > 1e-3
    # and the Gumbel noise built from it
    assert stats.kstest(gumbel(u[:200000]), "gumbel_r").pvalue > 1e-3


def test_neighbouring_counters_uncorrelated():
    n = 200000
    base = sample_uniform(99, 3, 4, np.arange(n))
    for other in (sample_uniform(99, 3, 4, np.arange(1, n + 1)),   # next word
                  sample_uniform(99, 4, 4, np.arange(n)),          # next row
                  sample_uniform(99, 3, 5, np.arange(n)),          # next step
                  sample_uniform(100, 3, 4, np.arange(n))):        # next seed
        c = np.corrcoef(base, other)[0, 1]
        assert abs(c) < 5.0 / np.sqrt(n), c
    # lag-1 along the word axis of many rows
    u = sample_uniform(5, np.arange(256)[:, None], 0, np.arange(1024)[None, :])
    c = np.corrcoef(u[:, :-1].ravel(), u[:, 1:].ravel())[0, 1]
    assert abs(c) < 5.0 / np.sqrt(u.size), c
