"""fp64 numpy reference of filtered sampling (sat_sample_loop_filtered): temperature, then top-k, then top-p, then the
Gumbel arg-max of sat_sample_loop over the kept words.

Row r at step t, raw logits x: words rank by (x desc, index asc); top_k keeps the first k of them (0 or k >= V: all);
top_p keeps the shortest prefix of those whose softmax(x / tau), renormalised over them, sums to p or more (1: all);
the word is argmax over the kept words of x / tau + g(seed, r, t, word)."""
import numpy as np

from oracle import ref_step as R
from test_sample_rng import gumbel, sample_uniform

NEAR_GAP = 1e-4    # logit gap at a filter boundary, relative to the row's range
NEAR_MASS = 1e-4   # cumulative mass this close to p


def ranked(x):
    """word indices in rank order: x descending, then index ascending"""
    x = np.asarray(x, np.float64)
    return np.lexsort((np.arange(x.size), -x))


def kept_count(xs, tau, top_k, top_p):
    """(n, s, c): the filters keep the first n words of the ranked row xs (x sorted in rank order); s = size of the
    top-k set; c = cumulative renormalised mass over it (None without a nucleus)."""
    V = xs.size
    s = top_k if 0 < top_k < V else V
    if top_p >= 1.0:
        return s, s, None
    z = xs[:s] / tau
    c = np.cumsum(np.exp(z - z[0]))
    c /= c[-1]
    n = min(int(np.searchsorted(c, top_p, side="left")) + 1, s)
    return n, s, c


def kept_words(x, tau, top_k, top_p):
    """indices of the kept words of one row, in rank order"""
    order = ranked(x)
    n, _, _ = kept_count(np.asarray(x, np.float64)[order], tau, top_k, top_p)
    return order[:n]


def draw(pert, words):
    """argmax of pert over `words` (ties to the lower index)"""
    words = np.sort(np.asarray(words))
    return int(words[np.argmax(pert[words])])


def filtered_draw(x, tau, top_k, top_p, pert):
    """(word, decidable) for one row: pert = x / tau + g.  Undecidable when the draw changes as a word near a filter
    boundary (logit gap at the last kept word below NEAR_GAP x range, or cumulative mass within NEAR_MASS of p) is
    added to or removed from the kept set, or when the top-2 perturbed margin inside the kept set is below NEAR_GAP x
    the perturbed range."""
    x = np.asarray(x, np.float64)
    V = x.size
    order = ranked(x)
    xs = x[order]
    n, s, c = kept_count(xs, tau, top_k, top_p)
    kept = order[:n]
    w = draw(pert, kept)
    span = xs[0] - xs[-1]
    # a near tie across the boundary of the kept prefix (the k-th word when the nucleus keeps all k words; at the
    # nucleus boundary, fp32 logits may rank two nearly equal words the other way)
    near = n < V and xs[n - 1] - xs[n] < NEAR_GAP * span
    if c is not None:
        near = near or abs(c[n - 1] - top_p) < NEAR_MASS or (n >= 2 and abs(c[n - 2] - top_p) < NEAR_MASS)
    ok = True
    if near:
        if n < V and draw(pert, order[:n + 1]) != w:
            ok = False
        if n > 1 and draw(pert, order[:n - 1]) != w:
            ok = False
    if n >= 2:
        top2 = np.sort(pert[kept])[-2:]
        ok = ok and top2[1] - top2[0] >= NEAR_GAP * (pert.max() - pert.min())
    return w, ok


def oracle_sample_filtered(ocfg, w, ctx, K, T, tau, seed, top_k, top_p):
    """tokens [n*K, T], word probabilities [n*K, T] (softmax at temperature 1 over the whole vocabulary) and, per row,
    its first undecidable step (T if none); the reference feeds its own draws to the next step."""
    n = ctx.shape[0]
    B, V = n * K, ocfg.vocabulary_size
    cx = np.repeat(ctx, K, axis=0).astype(np.float64)
    t1 = R.HoistedStepper(ocfg, w, cx, np.float64).t1
    c, h = R.initialize(ocfg, w, cx, np.float64)
    word = np.zeros(B, np.int32)
    toks, probs = np.zeros((B, T), np.int32), np.zeros((B, T))
    first_bad = np.full(B, T)
    rows = np.arange(B)
    for t in range(T):
        r = R.decode_step(ocfg, w, cx, word, c, h, np.float64, t1)
        c, h = r["memory"], r["output"]
        logits = r["logits"]
        pert = logits / tau + gumbel(sample_uniform(seed, rows[:, None], t, np.arange(V)[None, :]))
        for b in range(B):
            wd, ok = filtered_draw(logits[b], tau, top_k, top_p, pert[b])
            toks[b, t] = wd
            if not ok and first_bad[b] == T:
                first_bad[b] = t
        probs[:, t] = r["probs"][rows, toks[:, t]]
        word = toks[:, t].copy()
    return toks, probs, first_bad
