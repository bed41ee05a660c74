"""Caption assembly after beam search: word ids -> sentence, and the result files of the reference's
eval / test loops (SURVEY.md §8 f2).

  Vocabulary.load / get_sentence    utils/vocabulary.py:53-63, 72-80 (the csv written by Vocabulary.save)
  assemble_captions                 the per-image part of base_model.py:82-92 / 135-143: best caption + its score
  write_eval_results                base_model.py:109-111: json list of {"image_id", "caption"} (COCO result format)
  write_test_results                base_model.py:157-160: csv with columns image_files, caption, prob

Only the text side is mirrored: the reference also renders every image with its caption through matplotlib
(base_model.py:94-107, 145-155); image files are out of scope here (features are precomputed).  `beam_results` is what
CaptionGenerator.beam_search returns: per image, the captions sorted by descending score.
"""
import csv
import json
import string


class Vocabulary(object):
    """The word table of the reference (utils/vocabulary.py): `words[i]` is the word of id i; id 0 is '<start>' and
    '.' ends a sentence (id 2 in the shipped data/vocabulary.csv)."""

    def __init__(self, size=None, save_file=None, words=None):
        self.words = list(words) if words is not None else []
        self.word2idx = {w: i for i, w in enumerate(self.words)}
        self.size = size if size is not None else (len(self.words) or None)
        if save_file is not None:
            self.load(save_file)

    def load(self, save_file):
        """utils/vocabulary.py:72-80: the csv has the columns (index), frequency, index, word."""
        with open(save_file, newline="") as f:
            rows = list(csv.DictReader(f))
        rows.sort(key=lambda r: int(r["index"]))
        self.words = [r["word"] for r in rows]
        self.word2idx = {w: i for i, w in enumerate(self.words)}
        if self.size is None or self.size > len(self.words):
            self.size = len(self.words)
        return self

    @property
    def eos_id(self):
        """id of '.', the word that completes a caption in beam search (base_model.py:229)"""
        return self.word2idx["."]

    def get_sentence(self, idxs):
        """utils/vocabulary.py:53-63: words up to and including the first '.', a '.' appended if the last word is not
        one, joined with spaces except before punctuation and before tokens that start with an apostrophe."""
        words = [self.words[i] for i in idxs]
        if not words or words[-1] != ".":
            words.append(".")
        length = words.index(".") + 1
        words = words[:length]
        return "".join(" " + w if not w.startswith("'") and w not in string.punctuation else w for w in words).strip()


def assemble_captions(beam_results, vocabulary, fake_count=0):
    """Best caption and its score for every real image of a batch (base_model.py:82-92; the last batch of the reference
    is padded with `fake_count` copies, dataset.py:51-54, which are dropped here the same way)."""
    n = len(beam_results) - int(fake_count)
    captions, scores = [], []
    for caps in beam_results[:n]:
        best = caps[0]                                   # sorted by descending score (base_model.py:236-238)
        captions.append(vocabulary.get_sentence(best.sentence))
        scores.append(best.score)
    return captions, scores


def write_eval_results(path, image_ids, captions):
    """base_model.py:87-88, 109-111: [{"image_id": id, "caption": text}, ...] as json (what COCO.loadRes reads)."""
    results = [{"image_id": int(i), "caption": c} for i, c in zip(image_ids, captions)]
    with open(path, "w") as f:
        json.dump(results, f)
    return results


def write_test_results(path, image_files, captions, scores):
    """base_model.py:157-160: pandas.DataFrame({'image_files', 'caption', 'prob'}).to_csv(path) — a leading unnamed
    index column, then the columns in the order pandas keeps them (insertion order)."""
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["", "image_files", "caption", "prob"])
        for i, (a, c, p) in enumerate(zip(image_files, captions, scores)):
            w.writerow([i, a, c, repr(float(p))])
    return path


def write_attention_maps(path, image_files, captions, vocabulary):
    """One .npz (readable with np.load(..., allow_pickle=False)) with, for image i and its caption `captions[i]` (a
    CaptionData from beam_search(with_attention=True)):
      image_files                       [n] str
      img<i>_word_ids / img<i>_words    the caption's word ids and words, tokenised as Vocabulary.get_sentence does
                                        (up to and including the first '.')
      img<i>_score, img<i>_word_probs   the caption's score and the probability of each of those words
      img<i>_alphas                     where the model looked for each word: [len, sqrt(L), sqrt(L)] when L is a
                                        square (14 x 14 for VGG conv5_3, 7 x 7 for ResNet res5c), else [len, L]"""
    import numpy as np
    out = {"image_files": np.asarray([str(f) for f in image_files])}
    for i, cd in enumerate(captions):
        if cd.alphas is None or cd.word_probs is None:
            raise ValueError("caption %d carries no maps: use beam_search(..., with_attention=True)" % i)
        ids = [int(w) for w in cd.sentence]
        if "." in (vocabulary.words[w] for w in ids):
            ids = ids[:[vocabulary.words[w] for w in ids].index(".") + 1]
        n = len(ids)
        alphas = np.asarray(cd.alphas, np.float32)[:n]
        L = alphas.shape[1]
        side = int(round(L ** 0.5))
        if side * side == L:
            alphas = alphas.reshape(n, side, side)
        out["img%d_word_ids" % i] = np.asarray(ids, np.int32)
        out["img%d_words" % i] = np.asarray([vocabulary.words[w] for w in ids], dtype=str)
        out["img%d_score" % i] = np.float64(cd.score)
        out["img%d_word_probs" % i] = np.asarray(cd.word_probs, np.float32)[:n]
        out["img%d_alphas" % i] = alphas
    np.savez(path, **out)
    return path


def cut_after_eos(tokens, eos_id):
    """Word ids of one caption up to and including the first eos_id (all of them if there is none)."""
    ids = [int(w) for w in tokens]
    return ids[:ids.index(int(eos_id)) + 1] if int(eos_id) in ids else ids


def scst_advantages(rewards, num_samples, baseline="greedy"):
    """Self-critical advantages of K sampled captions per image (pure host arithmetic, float64).

    rewards: [n, K + 1] for baseline "greedy" (column K is the reward of the image's greedy caption), [n, K] for
    baseline "mean" (each sample's baseline is the mean reward of the image's OTHER K - 1 samples, so K >= 2).
    Returns (advantages [n, K] = sample reward - baseline, mean sample reward, mean baseline reward)."""
    import numpy as np
    K = int(num_samples)
    r = np.asarray(rewards, dtype=np.float64)
    if K < 1:
        raise ValueError("num_samples must be >= 1")
    if baseline == "greedy":
        if r.ndim != 2 or r.shape[1] != K + 1:
            raise ValueError("baseline 'greedy': rewards must be [n, %d] (K samples, then the greedy caption), got %s"
                             % (K + 1, r.shape))
        samples = r[:, :K]
        base = np.broadcast_to(r[:, K:], samples.shape)
    elif baseline == "mean":
        if K < 2:
            raise ValueError("baseline 'mean' (leave-one-out) needs num_samples >= 2")
        if r.ndim != 2 or r.shape[1] != K:
            raise ValueError("baseline 'mean': rewards must be [n, %d], got %s" % (K, r.shape))
        samples = r
        base = (r.sum(axis=1, keepdims=True) - r) / (K - 1)
    else:
        raise ValueError("baseline must be 'greedy' or 'mean', got %r" % (baseline,))
    return samples - base, float(samples.mean()), float(base.mean())


def scst_advantages_torch(rewards, num_samples, baseline="greedy"):
    """scst_advantages with torch ops on a rewards tensor (e.g. CIDEr-D scores on the device), in float64 like it and
    without reading anything back: (advantages [n, K] float64, mean sample reward, mean baseline reward), the two
    means as 0-dim tensors on the rewards' device.  The caller has validated baseline and K."""
    K = int(num_samples)
    r = rewards.double()
    if baseline == "greedy":
        samples = r[:, :K]
        base = r[:, K:K + 1].expand(-1, K)
    else:
        samples = r
        base = (r.sum(dim=1, keepdim=True) - r) / (K - 1)
    return samples - base, samples.mean(), base.mean()
