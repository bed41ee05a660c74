"""Sampled captions (sat_sample_loop / CaptionGenerator.sample) against the fp64 oracle driven autoregressively with the
numpy copy of the generator: the draw of row r at step t is argmax(logits / temperature + g(seed, r, t, word))."""
import numpy as np
import pytest

from _util import SMALL, assert_close, make_pair
from oracle import ref_step as R
from test_sample_rng import gumbel, sample_uniform

pytestmark = pytest.mark.gpu

REF_DEFAULT = dict(max_caption_length=6)   # the reference default graph: L=196, D=512, H=512, V=5000


def oracle_sample(ocfg, w, ctx, K, T, tau, seed):
    """tokens [n*K, T], word probabilities [n*K, T] (softmax at temperature 1) and, per row, the first step whose
    perturbed top-2 margin is below 1e-4 x (max - min) of the perturbed logits (T if none): beyond it the fp32 and fp64
    draws may part, so rows are compared up to there."""
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
        pert = r["logits"] / tau + gumbel(sample_uniform(seed, rows[:, None], t, np.arange(V)[None, :]))
        wd = pert.argmax(1).astype(np.int32)
        top2 = np.partition(pert, V - 2, axis=1)[:, -2:]
        margin = top2[:, 1] - top2[:, 0]
        bad = margin < 1e-4 * (pert.max(1) - pert.min(1))
        first_bad = np.where((first_bad == T) & bad, t, first_bad)
        toks[:, t], probs[:, t] = wd, r["probs"][rows, wd]
        word = wd
    return toks, probs, first_bad


def compare(tokens, wprobs, ref, min_full=0.9, name=""):
    toks, probs, first_bad = ref
    B, T = toks.shape
    tokens, wprobs = tokens.reshape(B, T), wprobs.reshape(B, T)
    assert (first_bad == T).mean() >= min_full, (first_bad == T).mean()
    mask = np.arange(T)[None, :] < first_bad[:, None]
    np.testing.assert_array_equal(np.where(mask, tokens, -1), np.where(mask, toks, -1), err_msg=name)
    assert_close(np.where(mask, wprobs, 0.0), np.where(mask, probs, 0.0), "word_probs " + name)


def dims_for(kind, layers):
    d = dict(SMALL) if kind == "small" else dict(REF_DEFAULT)
    d["num_attend_layers"] = d["num_decode_layers"] = layers
    return d


def run(m, ctx, K, T, tau, seed):
    import torch
    t, p = m.sample_device(ctx, K, T, tau, seed)
    torch.cuda.synchronize()
    return t.cpu().numpy(), p.cpu().numpy()


@pytest.mark.parametrize("tau", [0.7, 1.0, 1.5])
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("kind", ["small", "ref"])
def test_sample_vs_oracle(kind, layers, K, tau):
    import torch
    n = 32 // K   # (32 rows: the share of rows the oracle can decide over all T is not at the mercy of one near tie)
    ocfg, w, m = make_pair(n * K, **dims_for(kind, layers))
    T = ocfg.max_caption_length
    ctx = R.synth_contexts(ocfg, n)
    seed = 1000 + 17 * K + int(10 * tau)
    ref = oracle_sample(ocfg, w, ctx, K, T, tau, seed)
    for _ in range(3):   # eager, capture, replay
        tokens, wprobs = run(m, torch.from_numpy(ctx).cuda(), K, T, tau, seed)
        assert tokens.shape == (n, K, T) and wprobs.shape == (n, K, T)
        compare(tokens, wprobs, ref, name="%s/%d K=%d tau=%g" % (kind, layers, K, tau))


def rows_kernel_launches(m, f):
    """(result of f(), launches of the per-row vocabulary kernel it made): f's first call is eager, so option "profile"
    records every launch"""
    m.set_option("profile", 1)
    r = f()
    n = m.info("prof_n_rows")
    m.set_option("profile", 0)
    return r, n


def test_both_vocabulary_paths():
    """16 images x 4 at V=10000: fused sampling in the vocabulary layer; 48 x 4 (192 rows): that layer does not fit one
    wave and the row kernel draws.  The first 16 images are the same in both calls.  Without word probabilities the
    draws are the same."""
    import torch
    ocfg, w, m = make_pair(192, vocabulary_size=10000, max_caption_length=3)
    T, K, tau, seed = 3, 4, 1.0, 77
    ctx = R.synth_contexts(ocfg, 48)
    ref = oracle_sample(ocfg, w, ctx, K, T, tau, seed)
    c16, c48 = torch.from_numpy(ctx[:16]).cuda(), torch.from_numpy(ctx).cuda()
    (a_t, a_p), n_a = rows_kernel_launches(m, lambda: run(m, c16, K, T, tau, seed))
    (b_t, b_p), n_b = rows_kernel_launches(m, lambda: run(m, c48, K, T, tau, seed))
    assert n_a == 0 and n_b == T, (n_a, n_b)
    compare(b_t, b_p, ref, name="row kernel")
    ref16 = tuple(x[:64] for x in ref)
    compare(a_t, a_p, ref16, name="fused")
    ok = ref16[2] == T
    np.testing.assert_array_equal(a_t.reshape(64, T)[ok], b_t.reshape(192, T)[:64][ok])
    for c, t in ((c16, a_t), (c48, b_t)):
        for _ in range(3):   # eager, capture, replay
            tokens, wprobs = m.sample_device(c, K, T, tau, seed, want_word_probs=False)
            assert wprobs is None and np.array_equal(tokens.cpu().numpy(), t)


def test_fused_sampling_over_two_row_tiles():
    """V=300 at 192 rows: the vocabulary layer still fits one wave with two row tiles, so the draw of the second tile
    keys on its global row index."""
    import torch
    ocfg, w, m = make_pair(192, **dict(SMALL))
    T, K, tau, seed = ocfg.max_caption_length, 4, 1.0, 31
    ctx = R.synth_contexts(ocfg, 48)
    ref = oracle_sample(ocfg, w, ctx, K, T, tau, seed)
    (tokens, wprobs), n_rows = rows_kernel_launches(m, lambda: run(m, torch.from_numpy(ctx).cuda(), K, T, tau, seed))
    assert n_rows == 0
    compare(tokens, wprobs, ref, name="two row tiles")


def test_more_than_four_samples():
    """the library draws at most 4 rows per image in one call (SAT_ERR_UNSUPPORTED beyond, nothing launched); the
    facade draws more in groups of 4, group c with seed + c * 0x9E3779B97F4A7C15"""
    import torch
    n, T, seed = 3, 6, 123
    ocfg, w, m = make_pair(n * 6, **dict(SMALL))
    ctx = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    tok = torch.zeros(n * 6 * T, dtype=torch.int32, device="cuda")
    before = m.info("launches")
    assert m.lib.sat_sample_loop(m._h, m._p(ctx), n, 5, T, 1.0, 1, m._p(tok), None, m._st()) == -4
    assert m.info("launches") == before
    t6, p6 = [x.cpu().numpy() for x in m.sample_device(ctx, 6, T, 1.0, seed)]
    assert t6.shape == (n, 6, T) and p6.shape == (n, 6, T)
    t4, p4 = [x.cpu().numpy() for x in m.sample_device(ctx, 4, T, 1.0, seed)]
    t2, p2 = [x.cpu().numpy() for x in m.sample_device(ctx, 2, T, 1.0, (seed + 0x9E3779B97F4A7C15) % 2 ** 64)]
    assert np.array_equal(t6[:, :4], t4) and np.array_equal(t6[:, 4:], t2)
    assert np.array_equal(p6[:, :4], p4) and np.array_equal(p6[:, 4:], p2)
    assert not np.array_equal(t6[:, 4:], t6[:, :2])
    caps = m.sample(ctx.cpu().numpy(), num_samples=6, seed=seed, eos_id=-1)
    assert [[c.sentence for c in x] for x in caps] == [[list(map(int, t6[k, j])) for j in range(6)] for k in range(n)]


def test_launch_layouts_agree():
    import torch
    n, K, T, tau, seed = 4, 4, 5, 1.0, 4242
    ocfg, w, m = make_pair(n * K, max_caption_length=T)
    ctx0 = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    ref = oracle_sample(ocfg, w, ctx0.cpu().numpy(), K, T, tau, seed)
    layouts = [dict(overlap=o, graphs=g, pdl=p, pa=a) for o in (0, 1, 2) for g in (0, 1) for p in (0, 1) for a in (0, 1)]
    first, keep = None, []
    ok = ref[2] == T
    for lay in layouts:
        for k, v in lay.items():
            m.set_option(k, v)
        ctx = ctx0.clone()
        keep.append(ctx)
        for _ in range(3):
            tokens, wprobs = run(m, ctx, K, T, tau, seed)
            compare(tokens, wprobs, ref, name=str(lay))
            first = tokens if first is None else first
            np.testing.assert_array_equal(tokens.reshape(n * K, T)[ok], first.reshape(n * K, T)[ok], err_msg=str(lay))


def test_graph_replay_takes_a_new_seed():
    import torch
    n, K, T, tau = 4, 4, 6, 1.0
    ocfg, w, m = make_pair(n * K, **dict(SMALL))
    ctx_np = R.synth_contexts(ocfg, n)
    ctx = torch.from_numpy(ctx_np).cuda()
    outs = [run(m, ctx, K, T, tau, 11)[0] for _ in range(3)]   # eager, capture, replay
    assert all(np.array_equal(outs[0], o) for o in outs[1:])
    tokens, wprobs = run(m, ctx, K, T, tau, 12)                   # a replay of the same graph with another seed
    compare(tokens, wprobs, oracle_sample(ocfg, w, ctx_np, K, T, tau, 12), name="second seed")
    assert not np.array_equal(tokens, outs[0])
    tokens, wprobs = run(m, ctx, K, T, 0.5, 12)                   # and another temperature
    compare(tokens, wprobs, oracle_sample(ocfg, w, ctx_np, K, T, 0.5, 12), name="second temperature")


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
def test_first_word_distribution(tau):
    """V=300, T=1: 128 rows of one image (32 copies x 4 samples) x 100 seeds against softmax(logits / tau)."""
    import torch
    from scipy import stats
    dims = dict(SMALL)
    ocfg, w, m = make_pair(128, **dims)
    ctx1 = R.synth_contexts(ocfg, 1)
    ctx = torch.from_numpy(np.repeat(ctx1, 32, axis=0)).cuda()
    counts = np.zeros(ocfg.vocabulary_size)
    for s in range(100):
        tokens, _ = run(m, ctx, 4, 1, tau, 5000 + s)
        counts += np.bincount(tokens.ravel(), minlength=ocfg.vocabulary_size)
    c, h = R.initialize(ocfg, w, ctx1.astype(np.float64), np.float64)
    logits = R.decode_step(ocfg, w, ctx1, np.zeros(1, np.int32), c, h, np.float64)["logits"][0]
    p = np.exp((logits - logits.max()) / tau)
    p /= p.sum()
    exp = p * counts.sum()
    big = exp >= 5
    obs = np.append(counts[big], counts[~big].sum())
    ex = np.append(exp[big], exp[~big].sum())
    if ex[-1] < 5:   # fold a small pooled bin into the largest one
        obs[np.argmax(ex[:-1])] += obs[-1]; ex[np.argmax(ex[:-1])] += ex[-1]
        obs, ex = obs[:-1], ex[:-1]
    assert stats.chisquare(obs, ex).pvalue > 1e-3


def test_low_temperature_is_greedy():
    """tau = 1e-3 scales the noise (|g| < 23) below 0.025 logits: each row repeats the greedy loop up to its first
    step whose greedy top-2 margin is 0.05 or less."""
    import torch
    n, T = 16, 6
    ocfg, w, m = make_pair(n, **dict(REF_DEFAULT))
    ctx = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    greedy, logits = m.decode_loop(ctx, T, want_logits=True)
    greedy, logits = greedy.cpu().numpy(), logits.cpu().numpy()   # [B,T], [T,B,V]
    top2 = np.sort(logits, axis=2)[:, :, -2:]
    small = (top2[:, :, 1] - top2[:, :, 0]).T <= 0.05             # [B,T]
    upto = np.where(small.any(1), small.argmax(1), T)
    mask = np.arange(T)[None, :] < upto[:, None]
    assert mask.sum() >= n
    tokens, _ = run(m, ctx, 1, T, 1e-3, 3)
    np.testing.assert_array_equal(np.where(mask, tokens[:, 0], -1), np.where(mask, greedy, -1))


def test_sampling_leaves_the_greedy_loop_alone():
    import torch
    n, K, T = 8, 4, 5
    ocfg, w, m = make_pair(n * K, max_caption_length=T)
    ctx = torch.from_numpy(R.synth_contexts(ocfg, n)).cuda()
    ctx_big = torch.from_numpy(R.synth_contexts(ocfg, n * K, seed=7)).cuda()
    for _ in range(3):   # eager, capture, replay
        for c in (ctx, ctx_big):
            t0, l0 = m.decode_loop(c, T, want_logits=True)
            t0, l0 = t0.clone(), l0.clone()
            m.sample_device(ctx, K, T, 1.0, 5)
            t1, l1 = m.decode_loop(c, T, want_logits=True)
            assert torch.equal(t0, t1) and torch.equal(l0, l1)


def test_invalid_arguments_launch_nothing():
    import torch
    ocfg, w, m = make_pair(8, **dict(SMALL))
    ctx = torch.from_numpy(R.synth_contexts(ocfg, 2)).cuda()
    tok = torch.zeros(8 * 6, dtype=torch.int32, device="cuda")
    L = m.lib

    def call(c=ctx, n=2, K=2, T=3, tau=1.0, t=tok):
        return L.sat_sample_loop(m._h, m._p(c), n, K, T, tau, 1, m._p(t), None, m._st())
    assert call() == 0
    m.stream.synchronize()
    before = m.info("launches")
    for kw in (dict(tau=0.0), dict(tau=-1.0), dict(tau=float("inf")), dict(tau=float("nan")), dict(K=0), dict(K=-1),
               dict(n=3, K=3), dict(n=0), dict(T=0), dict(c=None), dict(t=None)):
        assert call(**kw) == -1, kw
    assert m.info("launches") == before


def test_facade_sample():
    import torch
    n, K = 3, 4
    ocfg, w, m = make_pair(n * K, **dict(SMALL))
    T = ocfg.max_caption_length
    ctx = R.synth_contexts(ocfg, n)
    tokens, _ = run(m, torch.from_numpy(ctx).cuda(), K, T, 1.5, 9)
    vals, cnt = np.unique(tokens[:, :, 1:], return_counts=True)
    eos = int(vals[np.argmax(cnt)])   # a word most captions meet
    a = m.sample(ctx, num_samples=K, temperature=1.5, seed=9, eos_id=eos)
    b = m.sample(torch.from_numpy(ctx).cuda(), num_samples=K, temperature=1.5, seed=9, eos_id=eos)
    assert len(a) == n and all(len(x) == K for x in a)
    assert any(c.complete for x in a for c in x)
    for k in range(n):
        for j in range(K):
            ca, cb = a[k][j], b[k][j]
            assert ca.sentence == cb.sentence and ca.score == cb.score
            row = [int(x) for x in tokens[k, j]]
            if eos in row:
                assert ca.complete and ca.sentence == row[:row.index(eos) + 1]
            else:
                assert not ca.complete and ca.sentence == row
            s = 1.0
            for x in ca.word_probs:
                s *= float(x)
            assert s == ca.score and len(ca.word_probs) == len(ca.sentence)
    # seed=None: successive calls differ; a fresh instance repeats the sequence
    _, _, m2 = make_pair(n * K, **dict(SMALL))
    s1 = [c.sentence for x in m.sample(ctx, K, eos_id=-1) for c in x]
    s2 = [c.sentence for x in m.sample(ctx, K, eos_id=-1) for c in x]
    r1 = [c.sentence for x in m2.sample(ctx, K, eos_id=-1) for c in x]
    assert s1 != s2 and s1 == r1
