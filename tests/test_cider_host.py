"""The fp64 CIDEr-D reference (cider_ref.py) on hand-computed cases, the padding helper of sat_b200.CiderD, and the
device form of the SCST advantage arithmetic (captions.scst_advantages_torch) against the host one."""
import math

import numpy as np
import pytest

import cider_ref as CR

V, EOS = 100, 2


def score(cand, refs, corpus, eos=EOS, vocab=V):
    df, N = CR.doc_freq(corpus, eos, vocab)
    return CR.scores([[cand]], [refs], df, N, eos, vocab)[0][0]


def test_rows_end_after_eos_and_before_padding_or_out_of_range_ids():
    assert CR.cut([5, 6, 2, 7, 8], EOS, V) == [5, 6, 2]
    assert CR.cut([5, -1, 7], EOS, V) == [5]
    assert CR.cut([5, 6, V, 7], EOS, V) == [5, 6]
    assert CR.cut([0, 0, 0], EOS, V) == [0, 0, 0]
    assert CR.cut([-1, 5], EOS, V) == []
    assert CR.cut([2, 5], EOS, V) == [2]


def test_identical_caption_and_single_reference_scores_ten():
    cap = [5, 6, 7, 8, 9, 2]
    corpus = [[cap], [[11, 12, 13]]]          # N = 2, every df of the caption's n-grams is 1
    df, _ = CR.doc_freq(corpus, EOS, V)
    assert all(df[g] == 1 for g in CR.ngrams(cap))
    assert abs(score(cap, [cap], corpus) - 10.0) < 1e-12


def test_bigram_length_penalty():
    """every n-gram weight is log N (counts 1, df <= 1): s_n = |h_n & r_n| / sqrt(|h_n| |r_n|), and the penalty
    uses the bigram counts 3 and 5"""
    h, r = [21, 22, 23, 24], [21, 22, 23, 24, 25, 26]
    corpus = [[r], [[40, 41]]]
    s = 4 / math.sqrt(24) + 3 / math.sqrt(15) + 2 / math.sqrt(8) + 1 / math.sqrt(3)
    expect = 10.0 * math.exp(-(3 - 5) ** 2 / 72.0) * s / 4.0
    assert abs(score(h, [r], corpus) - expect) < 1e-12
    # the same n-gram overlap at equal bigram counts has no penalty: a caption scores 10 only at its own length
    assert abs(score(r, [r], corpus) - 10.0) < 1e-12


def test_clipping_of_repeated_ngrams():
    """h = 7 7 7 against r = 7 8: the unigram (7) has weight 3a in h and a in r; min(3a, a) * a = a^2"""
    h, r = [7, 7, 7], [7, 8]
    corpus = [[r], [[40, 41]]]
    s1 = 1.0 / (3.0 * math.sqrt(2.0))      # a^2 / (|v_1(h)| = 3a) / (|v_1(r)| = sqrt(2) a)
    expect = 10.0 * math.exp(-(2 - 1) ** 2 / 72.0) * s1 / 4.0
    assert abs(score(h, [r], corpus) - expect) < 1e-12
    unclipped = 10.0 * math.exp(-1 / 72.0) * (1 / math.sqrt(2.0)) / 4.0
    assert score(h, [r], corpus) < unclipped


def test_ngram_absent_from_the_corpus_has_the_largest_weight():
    corpus = [[[4]], [[4]], [[9]]]            # N = 3, df(4) = 2, df(5) = df(4 5) = 0
    df, N = CR.doc_freq(corpus, EOS, V)
    v, norms, length = CR.vec([4, 5], df, N)
    b, c = math.log(3) - math.log(2), math.log(3)
    assert v[1] == pytest.approx({(4,): b, (5,): c}, abs=1e-15) and v[2] == pytest.approx({(4, 5): c}, abs=1e-15)
    assert length == 1 and norms[2] == 0 and norms[3] == 0
    expect = 10.0 * math.exp(-1 / 72.0) * (b / math.sqrt(b * b + c * c)) / 4.0
    assert abs(score([4, 5], [[4]], corpus) - expect) < 1e-12


def test_eos_only_candidate():
    corpus = [[[2]], [[9]]]
    assert abs(score([2, 5, 6], [[2, 7]], corpus) - 2.5) < 1e-12      # one unigram on each side, both cut to [2]
    assert score([2], [[9, 2]], corpus) > 0
    assert score([-1, 2], [[2]], corpus) == 0.0                         # an empty candidate scores 0


def test_image_without_references_scores_zero():
    corpus = [[[5, 6, 2]], [[9]]]
    assert score([5, 6, 2], [[-1, -1, -1], [-1, 5, 6]], corpus) == 0.0
    assert score([5, 6, 2], [], corpus) == 0.0


def test_empty_references_do_not_count():
    corpus = [[[5, 6, 7, 8, 2]], [[9]]]
    cap = [5, 6, 7, 8, 2]
    assert abs(score(cap, [cap, [-1, -1], [V + 1, 5]], corpus) - 10.0) < 1e-12


def test_pad_ragged_references():
    from sat_b200.cider import pad
    p = pad([[[5, 6, 2], [7]], [], [[8, 9, 10, 11]]])
    assert p.dtype == np.int32 and p.shape == (3, 2, 4)
    np.testing.assert_array_equal(p[0], [[5, 6, 2, -1], [7, -1, -1, -1]])
    assert (p[1] == -1).all() and list(p[2, 0]) == [8, 9, 10, 11] and (p[2, 1] == -1).all()
    a = np.arange(24).reshape(2, 3, 4)
    assert pad(a).dtype == np.int32 and (pad(a) == a).all()
    with pytest.raises(ValueError):
        pad(np.zeros((2, 3), np.int32))


@pytest.mark.parametrize("baseline,width", [("greedy", 5), ("mean", 4)])
def test_device_advantages_mirror_the_host_arithmetic(baseline, width):
    import torch
    from sat_b200.captions import scst_advantages, scst_advantages_torch
    r = np.random.RandomState(0).uniform(0, 3, (6, width)).astype(np.float32)
    K = 4
    a, rs, rb = scst_advantages(r.astype(np.float64), K, baseline)
    ta, trs, trb = scst_advantages_torch(torch.from_numpy(r), K, baseline)
    assert ta.dtype == torch.float64 and trs.dim() == 0 and trb.dim() == 0
    np.testing.assert_allclose(ta.numpy(), a, rtol=0, atol=1e-15)
    assert abs(float(trs) - rs) < 1e-15 and abs(float(trb) - rb) < 1e-15
