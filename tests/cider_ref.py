"""fp64 reference of CIDEr-D on word-id captions (sat_cider_create / sat_cider_d), written from the definition.

A row ends after its first eos_id (the eos word counts), or before its first id < 0 (padding) or >= V.  For n = 1..4:
  v_n(c)[g] = count_c(g) * (log N - log max(1, df(g)))        ||v_n(c)|| = sqrt(sum_g v_n(c)[g]^2)
  l(c)      = the number of bigrams of c (the "length" of coco-caption's cider_scorer.py and of CiderD)
  s_n(h, r) = sum over the distinct g of h of min(v_n(h)[g], v_n(r)[g]) * v_n(r)[g], divided by ||v_n(h)|| ||v_n(r)||
              when both are non-zero, times exp(-(l(h) - l(r))^2 / (2 * 6^2))
  CIDEr-D(h, R) = 10 * (1 / |R|) sum_r (1 / 4) sum_n s_n(h, r)   (0 when the image has no non-empty reference)
df(g): the number of corpus images whose references, taken together, contain g; N: the corpus's number of images."""
import math
from collections import Counter

SIGMA = 6.0


def cut(row, eos_id, V):
    """the words of one row"""
    out = []
    for w in row:
        w = int(w)
        if w < 0 or w >= V:
            break
        out.append(w)
        if w == eos_id:
            break
    return out


def ngrams(words):
    """Counter of the contiguous n-grams (tuples), n = 1..4"""
    c = Counter()
    for n in range(1, 5):
        for i in range(len(words) - n + 1):
            c[tuple(words[i:i + n])] += 1
    return c


def image_refs(refs, eos_id, V):
    """the non-empty references of one image (rows of word ids, -1 padded or ragged)"""
    return [r for r in (cut(row, eos_id, V) for row in refs) if r]


def doc_freq(corpus, eos_id, V):
    """(df Counter over n-gram tuples, N) of a corpus: corpus[i] = the reference rows of image i"""
    df = Counter()
    for refs in corpus:
        seen = set()
        for r in image_refs(refs, eos_id, V):
            seen.update(ngrams(r))
        df.update(seen)
    return df, len(corpus)


def vec(words, df, N):
    """(v: n -> {g: weight}, norms [4], length = number of bigrams)"""
    v = {n: {} for n in range(1, 5)}
    for g, cnt in ngrams(words).items():
        v[len(g)][g] = cnt * (math.log(N) - math.log(max(1.0, df.get(g, 0))))
    norms = [math.sqrt(sum(x * x for x in v[n].values())) for n in range(1, 5)]
    return v, norms, max(0, len(words) - 1)


def sim(h, r):
    """[s_1 .. s_4] of two vec() results"""
    (vh, nh, lh), (vr, nr, lr) = h, r
    pen = math.exp(-float(lh - lr) ** 2 / (2 * SIGMA ** 2))
    out = []
    for n in range(1, 5):
        val = sum(min(x, vr[n].get(g, 0.0)) * vr[n].get(g, 0.0) for g, x in vh[n].items())
        if nh[n - 1] != 0 and nr[n - 1] != 0:
            val /= nh[n - 1] * nr[n - 1]
        out.append(val * pen)
    return out


def cider_d(words, refs, df, N):
    """CIDEr-D of one caption (word list) against a list of non-empty reference word lists"""
    if not refs:
        return 0.0
    h = vec(words, df, N)
    return 10.0 * sum(sum(sim(h, vec(r, df, N))) for r in refs) / len(refs) / 4.0


def scores(candidates, references, df, N, eos_id, V):
    """[n][C] list of CIDEr-D: candidates[i] = the candidate rows of image i, references[i] = its reference rows"""
    out = []
    for cands, refs in zip(candidates, references):
        rr = image_refs(refs, eos_id, V)
        out.append([cider_d(cut(c, eos_id, V), rr, df, N) for c in cands])
    return out
