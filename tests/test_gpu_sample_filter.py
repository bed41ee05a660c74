"""Top-k / nucleus sampling (sat_sample_loop_filtered, CaptionGenerator.sample(top_k=, top_p=)) against the fp64
reference of sample_filter_ref.py, driven autoregressively with the numpy copy of the generator.  Rows are compared
up to their first undecidable step (a draw that a near-boundary word or a near perturbed tie could change)."""
import numpy as np
import pytest

from _util import SMALL, assert_close, make_pair
from oracle import ref_step as R
from sample_filter_ref import kept_words, oracle_sample_filtered, ranked

pytestmark = pytest.mark.gpu

REF_DEFAULT = dict(max_caption_length=6)   # the reference default graph: L=196, D=512, H=512, V=5000
FILTERS = [(1, 1.0), (5, 1.0), (50, 1.0), (0, 0.5), (0, 0.9), (50, 0.8)]


def compare(tokens, wprobs, ref, min_full=0.9, name=""):
    toks, probs, first_bad = ref
    B, T = toks.shape
    tokens, wprobs = tokens.reshape(B, T), wprobs.reshape(B, T)
    assert (first_bad == T).mean() >= min_full, (name, (first_bad == T).mean())
    mask = np.arange(T)[None, :] < first_bad[:, None]
    np.testing.assert_array_equal(np.where(mask, tokens, -1), np.where(mask, toks, -1), err_msg=name)
    assert_close(np.where(mask, wprobs, 0.0), np.where(mask, probs, 0.0), "word_probs " + name)


def dims_for(kind, layers):
    d = dict(SMALL) if kind == "small" else dict(REF_DEFAULT)
    d["num_attend_layers"] = d["num_decode_layers"] = layers
    return d


def run(m, ctx, K, T, tau, seed, top_k, top_p, want_word_probs=True):
    import torch
    t, p = m.sample_device(ctx, K, T, tau, seed, want_word_probs=want_word_probs, top_k=top_k, top_p=top_p)
    torch.cuda.synchronize()
    return t.cpu().numpy().copy(), (p.cpu().numpy().copy() if p is not None else None)


def lib_call(m, ctx, n, K, T, tau, seed, tok, wp=None, top_k=0, top_p=1.0, filtered=True):
    if filtered:
        return m.lib.sat_sample_loop_filtered(m._h, m._p(ctx), n, K, T, tau, top_k, top_p, seed, m._p(tok), m._p(wp),
                                              m._st())
    return m.lib.sat_sample_loop(m._h, m._p(ctx), n, K, T, tau, seed, m._p(tok), m._p(wp), m._st())


@pytest.mark.parametrize("top_k,top_p", FILTERS)
@pytest.mark.parametrize("tau", [0.7, 1.0, 1.5])
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("kind", ["small", "ref"])
def test_filtered_sample_vs_reference(kind, layers, K, tau, top_k, top_p):
    import torch
    n = 64 // K   # (64 rows: the share of rows the reference can decide over all T is not at the mercy of a few near ties)
    ocfg, w, m = make_pair(n * K, **dims_for(kind, layers))
    T = ocfg.max_caption_length
    ctx = R.synth_contexts(ocfg, n)
    seed = 2000 + 17 * K + int(10 * tau) + top_k
    ref = oracle_sample_filtered(ocfg, w, ctx, K, T, tau, seed, top_k, top_p)
    name = "%s/%d K=%d tau=%g k=%d p=%g" % (kind, layers, K, tau, top_k, top_p)
    for _ in range(3):   # eager, capture, replay
        tokens, wprobs = run(m, torch.from_numpy(ctx).cuda(), K, T, tau, seed, top_k, top_p)
        assert tokens.shape == (n, K, T) and wprobs.shape == (n, K, T)
        compare(tokens, wprobs, ref, name=name)


@pytest.mark.parametrize("V,n,K,T", [(10000, 16, 4, 3), (10000, 48, 4, 3), (30001, 8, 2, 3)])
def test_vocabulary_shapes(V, n, K, T):
    """V=10000 at 64 rows (cached row) and 192 rows; V=30001: the row is not a multiple of 4 and is read from global
    memory"""
    import torch
    ocfg, w, m = make_pair(n * K, vocabulary_size=V, max_caption_length=T)
    ctx = R.synth_contexts(ocfg, n)
    for top_k, top_p, tau in ((50, 1.0, 1.0), (0, 0.9, 1.0), (50, 0.8, 0.7)):
        seed = 300 + top_k + int(10 * top_p)
        ref = oracle_sample_filtered(ocfg, w, ctx, K, T, tau, seed, top_k, top_p)
        for _ in range(3):
            tokens, wprobs = run(m, torch.from_numpy(ctx).cuda(), K, T, tau, seed, top_k, top_p)
            compare(tokens, wprobs, ref, name="V=%d rows=%d k=%d p=%g" % (V, n * K, top_k, top_p))


def test_filters_off_is_plain_sampling():
    import torch
    n, K, T = 4, 4, 6
    ocfg, w, m = make_pair(n * K, vocabulary_size=1000, max_caption_length=T)
    ctx = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    for filtered in (False, True, True, True):   # the filtered entry: eager, capture, replay of sat_sample_loop's graph
        tok = torch.zeros(n * K * T, dtype=torch.int32, device="cuda")
        wp = torch.zeros(n * K * T, dtype=torch.float32, device="cuda")
        assert lib_call(m, ctx, n, K, T, 0.9, 77, tok, wp, filtered=filtered) == 0
        torch.cuda.synchronize()
        if not filtered:
            t0, p0 = tok.cpu().numpy(), wp.cpu().numpy()
        else:
            assert np.array_equal(tok.cpu().numpy(), t0) and np.array_equal(wp.cpu().numpy(), p0)
    t1, p1 = run(m, ctx, K, T, 0.9, 77, 0, 1.0)
    assert np.array_equal(t1.ravel(), t0) and np.array_equal(p1.ravel(), p0)


def test_k1_is_greedy():
    """top_k = 1 keeps the arg-max: each row repeats the greedy loop up to its first step whose greedy top-2 margin is
    0.05 or less, and the word probabilities are those of the greedy loop"""
    import torch
    n, T = 16, 6
    ocfg, w, m = make_pair(n, **dict(REF_DEFAULT))
    ctx = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    g = m.decode_loop(ctx, T, want_logits=True, want_word_probs=True)
    greedy, logits, gprobs = [np.asarray(x.cpu().numpy() if hasattr(x, "cpu") else x)
                              for x in (g["tokens"], g["logits"], g["word_probs"])]
    top2 = np.sort(logits, axis=2)[:, :, -2:]
    small = (top2[:, :, 1] - top2[:, :, 0]).T <= 0.05
    upto = np.where(small.any(1), small.argmax(1), T)
    mask = np.arange(T)[None, :] < upto[:, None]
    assert mask.sum() >= n
    for tau in (0.7, 1.5):
        tokens, wprobs = run(m, ctx, 1, T, tau, 3, 1, 1.0)
        np.testing.assert_array_equal(np.where(mask, tokens[:, 0], -1), np.where(mask, greedy, -1))
        np.testing.assert_allclose(np.where(mask, wprobs[:, 0], 0.0), np.where(mask, gprobs, 0.0), atol=1e-3)


@pytest.mark.parametrize("top_k,top_p", [(20, 1.0), (0, 0.9), (50, 0.8)])
@pytest.mark.parametrize("tau", [0.7, 1.5])
def test_first_word_distribution(top_k, top_p, tau):
    """V=300, T=1: 128 rows of one image (32 copies x 4 samples) x 100 seeds against the renormalised filtered
    softmax(logits / tau); no draw outside the kept words"""
    import torch
    from scipy import stats
    ocfg, w, m = make_pair(128, **dict(SMALL))
    V = ocfg.vocabulary_size
    ctx1 = R.synth_contexts(ocfg, 1)
    ctx = torch.from_numpy(np.repeat(ctx1, 32, axis=0)).cuda()
    counts = np.zeros(V)
    for s in range(100):
        tokens, _ = run(m, ctx, 4, 1, tau, 7000 + s, top_k, top_p, want_word_probs=False)
        counts += np.bincount(tokens.ravel(), minlength=V)
    c, h = R.initialize(ocfg, w, ctx1.astype(np.float64), np.float64)
    logits = R.decode_step(ocfg, w, ctx1, np.zeros(1, np.int32), c, h, np.float64)["logits"][0]
    kept = kept_words(logits, tau, top_k, top_p)
    order = ranked(logits)
    allowed = set(int(i) for i in kept)
    n = len(kept)
    if n < V and logits[order[n - 1]] - logits[order[n]] < 1e-4 * np.ptp(logits):
        allowed.add(int(order[n]))   # (a near tie across the boundary)
    outside = [i for i in np.flatnonzero(counts) if int(i) not in allowed]
    assert not outside, outside
    p = np.zeros(V)
    p[kept] = np.exp((logits[kept] - logits.max()) / tau)
    p /= p.sum()
    exp = p * counts.sum()
    big = exp >= 5
    obs = np.append(counts[big], counts[~big].sum())
    ex = np.append(exp[big], exp[~big].sum())
    if ex[-1] < 5:   # fold a small pooled bin into the largest one
        obs[np.argmax(ex[:-1])] += obs[-1]; ex[np.argmax(ex[:-1])] += ex[-1]
        obs, ex = obs[:-1], ex[:-1]
    if len(ex) > 1:
        assert stats.chisquare(obs, ex).pvalue > 1e-3


def test_graph_replay_follows_new_filters():
    import torch
    n, K, T = 16, 4, 6
    ocfg, w, m = make_pair(n * K, **dict(SMALL))
    ctx_np = R.synth_contexts(ocfg, n)
    ctx = torch.from_numpy(ctx_np).cuda()
    outs = [run(m, ctx, K, T, 1.0, 11, 5, 1.0)[0] for _ in range(3)]   # eager, capture, replay
    assert all(np.array_equal(outs[0], o) for o in outs[1:])
    for top_k, top_p, seed, tau in ((5, 1.0, 12, 1.0), (0, 0.9, 12, 1.0), (50, 0.8, 13, 1.0), (50, 0.8, 13, 0.5),
                                    (1, 0.5, 14, 1.5)):
        tokens, wprobs = run(m, ctx, K, T, tau, seed, top_k, top_p)   # replays of the same graph
        compare(tokens, wprobs, oracle_sample_filtered(ocfg, w, ctx_np, K, T, tau, seed, top_k, top_p),
                name="replay k=%d p=%g seed=%d tau=%g" % (top_k, top_p, seed, tau))


def test_launch_layouts_agree():
    import torch
    n, K, T, tau, seed = 16, 4, 5, 1.0, 4242
    ocfg, w, m = make_pair(n * K, max_caption_length=T)
    ctx0 = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    ref = oracle_sample_filtered(ocfg, w, ctx0.cpu().numpy(), K, T, tau, seed, 50, 0.9)
    layouts = [dict(overlap=o, graphs=g, pdl=p, pa=a) for o in (0, 1, 2) for g in (0, 1) for p in (0, 1) for a in (0, 1)]
    first, keep = None, []
    ok = ref[2] == T
    for lay in layouts:
        for k, v in lay.items():
            m.set_option(k, v)
        ctx = ctx0.clone()
        keep.append(ctx)
        for _ in range(3):
            tokens, wprobs = run(m, ctx, K, T, tau, seed, 50, 0.9)
            compare(tokens, wprobs, ref, name=str(lay))
            first = tokens if first is None else first
            np.testing.assert_array_equal(tokens.reshape(n * K, T)[ok], first.reshape(n * K, T)[ok], err_msg=str(lay))


def test_invalid_arguments_launch_nothing():
    import torch
    ocfg, w, m = make_pair(8, **dict(SMALL))
    ctx = torch.from_numpy(R.synth_contexts(ocfg, 2)).cuda()
    tok = torch.zeros(8 * 6, dtype=torch.int32, device="cuda")

    def call(c=ctx, n=2, K=2, T=3, tau=1.0, t=tok, top_k=5, top_p=0.9):
        return lib_call(m, c, n, K, T, tau, 1, t, None, top_k, top_p)
    assert call() == 0
    m.stream.synchronize()
    before = m.info("launches")
    for kw in (dict(top_k=-1), dict(top_p=0.0), dict(top_p=-0.5), dict(top_p=1.5), dict(top_p=float("nan")),
               dict(top_p=float("inf")), dict(top_k=-1, top_p=1.0), dict(top_k=0, top_p=0.0),
               dict(tau=0.0), dict(tau=-1.0), dict(tau=float("inf")), dict(tau=float("nan")), dict(K=0), dict(K=-1),
               dict(n=3, K=3), dict(n=0), dict(T=0), dict(c=None), dict(t=None)):
        assert call(**kw) == -1, kw
    assert m.info("launches") == before
    assert call(n=1, K=5) == -4   # (more than 4 rows per image: SAT_ERR_UNSUPPORTED, nothing launched)
    assert m.info("launches") == before


def test_facade_sample():
    import torch
    n, K, T, seed = 3, 6, 6, 123
    ocfg, w, m = make_pair(n * K, **dict(SMALL))
    ctx = R.synth_contexts(ocfg, n)
    ctx_t = torch.from_numpy(ctx).cuda()
    t6, p6 = run(m, ctx_t, 6, T, 1.2, seed, 20, 0.9)
    t4, p4 = run(m, ctx_t, 4, T, 1.2, seed, 20, 0.9)
    t2, p2 = run(m, ctx_t, 2, T, 1.2, (seed + 0x9E3779B97F4A7C15) % 2 ** 64, 20, 0.9)
    assert np.array_equal(t6[:, :4], t4) and np.array_equal(t6[:, 4:], t2)
    assert np.array_equal(p6[:, :4], p4) and np.array_equal(p6[:, 4:], p2)
    a = m.sample(ctx, num_samples=K, temperature=1.2, seed=seed, eos_id=-1, top_k=20, top_p=0.9)
    b = m.sample(ctx_t, num_samples=K, temperature=1.2, seed=seed, eos_id=-1, top_k=20, top_p=0.9)
    assert [[c.sentence for c in x] for x in a] == [[list(map(int, t6[k, j])) for j in range(K)] for k in range(n)]
    assert [[(c.sentence, c.score) for c in x] for x in a] == [[(c.sentence, c.score) for c in x] for x in b]
    plain = m.sample(ctx, num_samples=K, temperature=1.2, seed=seed, eos_id=-1)
    assert [[c.sentence for c in x] for x in plain] != [[c.sentence for c in x] for x in a]


def test_filtered_sampling_leaves_plain_sampling_and_the_greedy_loop_alone():
    import torch
    n, K, T = 8, 4, 5
    ocfg, w, m = make_pair(n * K, max_caption_length=T)
    ctx = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    ctx_big = torch.from_numpy(R.synth_contexts(ocfg, n * K, seed=7)).cuda()
    for _ in range(3):   # eager, capture, replay
        for c in (ctx, ctx_big):
            t0, l0 = m.decode_loop(c, T, want_logits=True)
            t0, l0 = t0.clone(), l0.clone()
            s0 = run(m, ctx, K, T, 1.0, 5, 0, 1.0)
            run(m, ctx, K, T, 1.0, 5, 50, 0.9)
            t1, l1 = m.decode_loop(c, T, want_logits=True)
            s1 = run(m, ctx, K, T, 1.0, 5, 0, 1.0)
            assert torch.equal(t0, t1) and torch.equal(l0, l1)
            assert np.array_equal(s0[0], s1[0]) and np.array_equal(s0[1], s1[1])
