"""The fp64 reference of filtered sampling (sample_filter_ref.py) against a brute-force sort, on boundary ties and on the
filters' limits.  No GPU needed."""
import numpy as np
import pytest

from sample_filter_ref import filtered_draw, kept_words


def brute_force(x, tau, top_k, top_p):
    """the kept words by the definition: a full sort by (x desc, index asc), the first k, then a running sum"""
    V = len(x)
    order = sorted(range(V), key=lambda i: (-x[i], i))
    S = order[:top_k] if 0 < top_k < V else order
    if top_p >= 1.0:
        return S
    z = np.array([x[i] / tau for i in S])
    q = np.exp(z - z.max())
    q /= q.sum()
    acc = 0.0
    for j, i in enumerate(S):
        acc += q[j]
        if acc >= top_p:
            return S[:j + 1]
    return S


@pytest.mark.parametrize("top_k,top_p", [(1, 1.0), (5, 1.0), (50, 1.0), (0, 0.5), (0, 0.9), (50, 0.8), (20, 0.3)])
@pytest.mark.parametrize("tau", [0.7, 1.0, 1.5])
def test_reference_against_a_full_sort(top_k, top_p, tau):
    rng = np.random.default_rng(int(100 * tau) + top_k)
    for _ in range(20):
        x = rng.normal(0.0, 2.0, 300)
        got = list(kept_words(x, tau, top_k, top_p))
        exp = brute_force(list(x), tau, top_k, top_p)
        if top_p < 1.0:   # (a cumulative sum can sit a rounding error from p: compare away from it)
            z = np.sort(x)[::-1][:top_k if top_k else None] / tau
            c = np.cumsum(np.exp(z - z[0]))
            c /= c[-1]
            if np.abs(c - top_p).min() < 1e-12:
                continue
        assert got == exp


def test_ties_at_the_top_k_boundary_go_to_the_lower_index():
    x = np.zeros(40)
    x[[3, 9, 17, 30]] = 2.0      # four words tie for ranks 1..4
    x[[1, 2]] = 5.0
    assert list(kept_words(x, 1.0, 4, 1.0)) == [1, 2, 3, 9]
    assert list(kept_words(x, 1.0, 5, 1.0)) == [1, 2, 3, 9, 17]
    # the rest of the row (36 words at 0) ties too
    assert list(kept_words(x, 1.0, 8, 1.0)) == [1, 2, 3, 9, 17, 30, 0, 4]


def test_ties_at_the_nucleus_boundary_go_to_the_lower_index():
    V = 10
    x = np.full(V, -np.inf)
    x[[7, 2, 5, 8]] = 0.0        # four words of 1/4 each
    assert list(kept_words(x, 1.0, 0, 0.5)) == [2, 5]
    assert list(kept_words(x, 1.0, 0, 0.51)) == [2, 5, 7]
    assert list(kept_words(x, 1.0, 0, 0.25)) == [2]
    assert list(kept_words(x, 1.0, 0, 1e-9)) == [2]
    assert list(kept_words(x, 1.0, 3, 0.9)) == [2, 5, 7]     # renormalised over the top 3: 2/3 < 0.9 <= 1


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
def test_filters_off_keep_every_word(tau):
    rng = np.random.default_rng(7)
    x = rng.normal(0.0, 3.0, 257)
    for k in (0, 257, 258, 10 ** 6):
        assert sorted(kept_words(x, tau, k, 1.0)) == list(range(257))
    pert = x / tau + rng.gumbel(size=257)
    w, _ = filtered_draw(x, tau, 0, 1.0, pert)
    assert w == int(np.argmax(pert))


def test_k1_is_the_argmax():
    rng = np.random.default_rng(3)
    for _ in range(50):
        x = np.round(rng.normal(0.0, 1.0, 100), 1)   # (with ties)
        assert list(kept_words(x, 1.0, 1, 1.0)) == [int(np.argmax(x))]
        pert = x + rng.gumbel(size=100)
        assert filtered_draw(x, 1.0, 1, 0.9, pert)[0] == int(np.argmax(x))


def test_the_draw_is_the_unfiltered_draw_when_that_is_kept():
    rng = np.random.default_rng(11)
    same = 0
    for _ in range(200):
        x = rng.normal(0.0, 2.0, 200)
        pert = x / 0.8 + rng.gumbel(size=200)
        w0 = int(np.argmax(pert))
        keep = set(kept_words(x, 0.8, 20, 0.9))
        w, _ = filtered_draw(x, 0.8, 20, 0.9, pert)
        assert w in keep
        if w0 in keep:
            assert w == w0
            same += 1
    assert same > 100


def test_near_boundary_steps_are_undecidable_only_when_the_draw_depends_on_them():
    x = np.array([3.0, 1.0, 1.0 - 1e-7, -2.0])
    pert = np.array([0.0, 1.0, 5.0, -1.0])   # the word at rank 3 wins if the near tie lets it in
    assert filtered_draw(x, 1.0, 2, 1.0, pert) == (1, False)
    pert = np.array([9.0, 1.0, 5.0, -1.0])   # the top word wins either way
    assert filtered_draw(x, 1.0, 2, 1.0, pert) == (0, True)
