"""captions.write_attention_maps: the .npz of per-word maps opens without pickle and keeps the caption's words."""
import numpy as np
import pytest

from sat_b200.captions import Vocabulary, write_attention_maps
from sat_b200.model import CaptionData

WORDS = ["<start>", "a", ".", "dog", "on", "the", "grass", "'s", ","]


@pytest.mark.parametrize("L", [196, 49, 30])
def test_write_attention_maps_round_trip(tmp_path, L):
    voc = Vocabulary(words=WORDS)
    rng = np.random.RandomState(L)
    sents = [[1, 3, 4, 5, 6, 2], [1, 3, 7, 8, 2, 6, 6]]   # the second continues past its first '.'
    caps = []
    for s in sents:
        a = rng.uniform(size=(len(s), L)).astype(np.float32)
        a /= a.sum(1, keepdims=True)
        p = rng.uniform(0.1, 1.0, len(s)).astype(np.float32)
        caps.append(CaptionData(s, float(np.prod(p.astype(np.float64))), True, a, p))
    path = write_attention_maps(str(tmp_path / "maps.npz"), ["x.jpg", "y.jpg"], caps, voc)
    with np.load(path, allow_pickle=False) as f:
        assert list(f["image_files"]) == ["x.jpg", "y.jpg"]
        side = int(round(L ** 0.5))
        for i, (s, cd) in enumerate(zip(sents, caps)):
            n = s.index(2) + 1
            assert list(f["img%d_word_ids" % i]) == s[:n]
            words = list(f["img%d_words" % i])
            assert words == [WORDS[w] for w in s[:n]]
            assert voc.get_sentence(s) == voc.get_sentence(list(f["img%d_word_ids" % i]))
            al = f["img%d_alphas" % i]
            assert al.shape == ((n, side, side) if side * side == L else (n, L))
            np.testing.assert_array_equal(al.reshape(n, L), cd.alphas[:n])
            np.testing.assert_array_equal(f["img%d_word_probs" % i], cd.word_probs[:n])
            assert float(f["img%d_score" % i]) == cd.score


def test_caption_data_defaults_unchanged():
    cd = CaptionData([1, 2], 0.5, True)
    assert cd.alphas is None and cd.word_probs is None
    assert repr(cd) == "CaptionData(score=0.5, sentence=[1, 2])"
    with pytest.raises(ValueError):
        write_attention_maps("unused.npz", ["x"], [cd], Vocabulary(words=WORDS))
