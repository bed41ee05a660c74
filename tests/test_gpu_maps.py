"""Per-word attention maps and word probabilities from the device loop (sat_decode_loop_maps) and the device beam search
(sat_beam_search_maps) against the oracle, and the guarantee that asking for them changes nothing else."""
import numpy as np
import pytest

from _util import SMALL, assert_close, make_pair
from oracle import ref_step as R

pytestmark = pytest.mark.gpu

REF_DEFAULT = dict(max_caption_length=6)   # the reference default graph (config 1): L=196, D=512, H=512, V=5000


def dims_for(kind, layers):
    d = dict(SMALL) if kind == "small" else dict(REF_DEFAULT)
    d["num_attend_layers"] = d["num_decode_layers"] = layers
    return d


def oracle_maps(ocfg, w, ctx, T, forced=None):
    toks, steps = R.decode_loop(ocfg, w, ctx, T, forced, np.float64)
    alphas = np.stack([s["alpha"] for s in steps], 1)                       # [B,T,L]
    fed = toks if forced is None else forced
    probs = np.stack([steps[t]["probs"][np.arange(ctx.shape[0]), fed[:, t]] for t in range(T)], 1)
    return toks, alphas, probs


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("kind", ["small", "ref"])
def test_loop_maps_vs_oracle(kind, layers):
    B = 4
    ocfg, w, m = make_pair(B, **dims_for(kind, layers))
    T = ocfg.max_caption_length
    ctx = R.synth_contexts(ocfg, B)
    r = m.decode_loop(ctx, T, want_alphas=True, want_word_probs=True)
    toks, alphas, probs = oracle_maps(ocfg, w, ctx, T)
    np.testing.assert_array_equal(r["tokens"], toks)
    assert r["alphas"].shape == (B, T, ocfg.num_ctx) and r["word_probs"].shape == (B, T)
    assert_close(r["alphas"], alphas, "alphas")
    assert_close(r["word_probs"], probs, "word_probs")
    np.testing.assert_allclose(r["alphas"].sum(-1), 1.0, atol=1e-5)
    spread = np.abs(r["alphas"] - r["alphas"][:, :1]).max()
    if layers == 2:   # the map does not depend on the state (header of sat_b200.h)
        assert spread <= 1e-5, spread
    else:
        assert spread > 1e-4, spread


@pytest.mark.parametrize("kind", ["small", "ref"])
def test_teacher_forced_word_probs(kind):
    B = 4
    ocfg, w, m = make_pair(B, **dims_for(kind, 2))
    T = ocfg.max_caption_length
    ctx = R.synth_contexts(ocfg, B)
    forced = np.random.RandomState(4).randint(0, ocfg.vocabulary_size, (B, T)).astype(np.int32)
    _, _, probs = oracle_maps(ocfg, w, ctx, T, forced)
    r = m.decode_loop(ctx, T, forced_words=forced, want_word_probs=True)
    assert_close(r["word_probs"], probs, "forced word_probs")
    # a forced word outside [0, V) gets probability 0 (in the last column: it is never fed to another step)
    forced[0, T - 1], forced[1, T - 1] = -3, ocfg.vocabulary_size + 7
    r = m.decode_loop(ctx, T, forced_words=forced, want_word_probs=True)
    assert r["word_probs"][0, T - 1] == 0.0 and r["word_probs"][1, T - 1] == 0.0
    assert_close(r["word_probs"][2:], probs[2:], "forced word_probs")


def test_teacher_forced_matches_training_cross_entropy():
    TD = dict(num_ctx=9, dim_ctx=64, dim_embedding=32, num_lstm_units=32, dim_initalize_layer=16,
              dim_attend_layer=24, dim_decode_layer=40, vocabulary_size=50, max_caption_length=5)
    B = 4
    ocfg, w, m = make_pair(B, seed=3, **TD)
    T = ocfg.max_caption_length
    rng = np.random.RandomState(3)
    ctx = R.synth_contexts(ocfg, B, 3)
    sent = rng.randint(1, ocfg.vocabulary_size, (B, T)).astype(np.int32)
    lens = rng.randint(2, T + 1, B)
    masks = (np.arange(T)[None, :] < lens[:, None]).astype(np.float32)
    m.train_setup(B, T, weights=w)
    m.sync_inference_weights()
    ce_train = float(m.train_forward_backward(ctx, sent, masks, seed=0).cpu().numpy()[0])
    p = m.decode_loop(ctx, T, forced_words=sent, want_word_probs=True)["word_probs"].astype(np.float64)
    ce_loop = -(np.log(p) * masks).sum() / masks.sum()
    assert abs(ce_loop - ce_train) <= 1e-4 * abs(ce_train), (ce_loop, ce_train)


@pytest.mark.parametrize("B", [64, 192])
def test_both_vocabulary_paths(B):
    """B=64: fused arg-max of the vocabulary layer; B=192 at V=10000: the grid does not fit one wave (row kernel)."""
    ocfg, w, m = make_pair(B, vocabulary_size=10000, max_caption_length=3)
    T = 3
    ctx = R.synth_contexts(ocfg, B)
    forced = np.random.RandomState(1).randint(0, 10000, (B, T)).astype(np.int32)
    for fw in (None, forced):
        r = m.decode_loop(ctx, T, forced_words=fw, want_word_probs=True)
        _, _, probs = oracle_maps(ocfg, w, ctx, T, fw)
        assert_close(r["word_probs"], probs, "word_probs B=%d forced=%s" % (B, fw is not None))


LAYOUTS = [dict(overlap=o, graphs=g, pdl=p, pa=a, xbatch=0) for o in (0, 1, 2) for g in (0, 1) for p in (0, 1)
           for a in (0, 1)] + [dict(overlap=2, graphs=g, pdl=1, pa=1, xbatch=1) for g in (0, 1)]


def test_no_behaviour_change_across_layouts():
    import torch
    B, T = 16, 5
    ocfg, w, m = make_pair(B, max_caption_length=T)
    ctx0 = torch.from_numpy(R.synth_contexts(ocfg, B)).cuda()
    forced = torch.from_numpy(np.random.RandomState(2).randint(0, 5000, (B, T)).astype(np.int32)).cuda()
    first, keep = {}, []
    for lay in LAYOUTS:
        for k, v in lay.items():
            m.set_option(k, v)
        ctx = ctx0.clone()   # a new contexts buffer: new graph keys, so every layout is captured afresh
        keep.append(ctx)
        torch.cuda.synchronize()   # ("xbatch": the contexts are complete when the loop is called)
        for fw in (None, forced):
            for _ in range(3):   # eager, capture, replay (graphs on)
                t0, l0 = m.decode_loop(ctx, T, forced_words=fw, want_logits=True)
                t0, l0 = t0.clone(), l0.clone()
                r = m.decode_loop(ctx, T, forced_words=fw, want_logits=True, want_alphas=True, want_word_probs=True)
                assert torch.equal(t0, r["tokens"]), lay
                assert torch.equal(l0, r["logits"]), lay
                ref = first.setdefault(fw is None, {k: v.cpu().numpy() for k, v in r.items()})
                assert_close(r["alphas"].cpu().numpy(), ref["alphas"], "alphas %s" % lay)
                assert_close(r["word_probs"].cpu().numpy(), ref["word_probs"], "word_probs %s" % lay)


def test_graph_keys_follow_the_map_buffers():
    import torch
    B, T = 8, 4
    ocfg, w, m = make_pair(B, max_caption_length=T)
    ctx_np = R.synth_contexts(ocfg, B)
    ctx = torch.from_numpy(ctx_np).cuda()
    _, alphas, probs = oracle_maps(ocfg, w, ctx_np, T)
    L = ocfg.num_ctx
    bufs = [(torch.zeros(T, B, L, device="cuda"), torch.zeros(B, T, device="cuda")) for _ in range(2)]
    tokens = torch.zeros(B, T, dtype=torch.int32, device="cuda")

    def run(maps):
        a, p = maps if maps else (None, None)
        for x in (maps or ()):
            x.fill_(-1.0)
        m._sync_in()
        m._check(m.lib.sat_decode_loop_maps(m._h, m._p(ctx), B, T, None, m._p(tokens), None, m._p(a), m._p(p), m._st()))
        m.stream.synchronize()
        if maps:
            assert_close(a.transpose(0, 1).cpu().numpy(), alphas, "alphas")
            assert_close(p.cpu().numpy(), probs, "word_probs")
    for _ in range(2):   # (second round: every key is replayed from its graph)
        run(bufs[0]); run(None); run(bufs[1]); run(bufs[0])
        untouched = bufs[1][0].clone()
        run(bufs[0])
        assert torch.equal(bufs[1][0], untouched)


def caption_maps(ocfg, w, ctx, items, hoist=False):
    """Expected maps of beam-search captions from the oracle: a beam's state at step t is that of the model run along
    its own prefix, so the alpha and the probability of word t of caption (image k, sentence s) are those of step t of a
    loop teacher-forced with s.  items: [(k, s)]; returns [(alphas [len, L], probs [len])] in fp64."""
    if not items:
        return []
    rows = np.array([k for k, _ in items])
    cx = ctx[rows].astype(np.float64)
    n, T = len(items), max(len(sn) for _, sn in items)
    forced = np.zeros((n, T), np.int32)
    for i, (_, sn) in enumerate(items):
        forced[i, :len(sn)] = sn
    t1 = R.HoistedStepper(ocfg, w, cx, np.float64).t1 if hoist else None
    c, h = R.initialize(ocfg, w, cx, np.float64)
    word = np.zeros(n, np.int32)
    alphas, probs = [], []
    for t in range(T):
        r = R.decode_step(ocfg, w, cx, word, c, h, np.float64, t1)
        c, h = r["memory"], r["output"]
        alphas.append(r["alpha"])
        probs.append(r["probs"][np.arange(n), forced[:, t]])
        word = forced[:, t]
    alphas, probs = np.stack(alphas, 1), np.stack(probs, 1)
    return [(alphas[i, :len(sn)], probs[i, :len(sn)]) for i, (_, sn) in enumerate(items)]


def beam_compare(ocfg, w, ctx, got, ref, images=None, hoist=False):
    """captions equal to the oracle's beam search; their maps equal the oracle's teacher-forced ones; score == the fp64
    product of the word probabilities in step order; images: the indices of got / ref to check (default all)."""
    images = range(len(got)) if images is None else images
    items = []
    for k in images:
        assert len(got[k]) == len(ref[k]), k
        for g, e in zip(got[k], ref[k]):
            assert g.sentence == [int(x) for x in e.sentence], k
            n = len(g.sentence)
            assert g.alphas.shape == (n, ocfg.num_ctx) and g.word_probs.shape == (n,)
            s = 1.0
            for x in g.word_probs:
                s *= float(x)
            assert s == g.score, (s, g.score)
            items.append((k, g.sentence))
    exp = caption_maps(ocfg, w, ctx, items, hoist)
    got_caps = [g for k in images for g in got[k]]
    for (k, _), g, (ea, ep) in zip(items, got_caps, exp):
        assert_close(g.alphas, ea, "beam alphas image %d" % k)
        assert_close(g.word_probs, ep, "beam word_probs image %d" % k)


@pytest.mark.parametrize("beam", [1, 3, 4])
def test_beam_maps_small(beam):
    from test_gpu_beam import pick_eos
    dims = dict(SMALL)
    dims["max_caption_length"] = 8
    ocfg, w, m = make_pair(5, beam=beam, **dims)
    ctx = R.synth_contexts(ocfg, 5)
    eos = pick_eos(ocfg, w, ctx)
    ref = R.beam_search(ocfg, w, ctx, eos_id=eos, dtype=np.float64)
    for _ in range(3):   # eager, capture, replay
        got = m.beam_search(ctx, eos_id=eos, with_attention=True)
        beam_compare(ocfg, w, ctx, got, ref)
    assert any(c.complete for caps in got for c in caps)
    if beam > 1:   # captions of several lengths (one beam may complete every image at the same step)
        assert len({len(c.sentence) for caps in got for c in caps}) > 1
    plain = m.beam_search(ctx, eos_id=eos)
    for a, b in zip(plain, got):
        assert [(c.sentence, c.score) for c in a] == [(c.sentence, c.score) for c in b]
    # zero past the length, on the raw device outputs
    sent, lens, scores, nres, comp, al, wp = [t.cpu().numpy() for t in
                                              m.beam_device(__import__("torch").from_numpy(ctx).cuda(), beam, 8, eos, True)]
    for k in range(5):
        for j in range(beam):
            assert not al[k, j, lens[k, j]:].any() and not wp[k, j, lens[k, j]:].any()
    if beam == 1:
        r = m.decode_loop(ctx, 8, want_alphas=True)
        ref_nc = m.beam_search(ctx, eos_id=-1, with_attention=True)
        for k in range(5):
            assert_close(ref_nc[k][0].alphas, r["alphas"][k], "beam-1 vs greedy alphas")


def test_beam_graph_keys():
    import torch
    dims = dict(SMALL)
    ocfg, w, m = make_pair(3, beam=3, **dims)
    T = ocfg.max_caption_length
    ctx_np = R.synth_contexts(ocfg, 3)
    ctx = torch.from_numpy(ctx_np).cuda()
    ref = R.beam_search(ocfg, w, ctx_np, eos_id=-1, dtype=np.float64)
    exp = iter(caption_maps(ocfg, w, ctx_np, [(k, c.sentence) for k in range(3) for c in ref[k]]))
    ref_alpha = [[next(exp)[0] for _ in ref[k]] for k in range(3)]
    L = ocfg.num_ctx
    sets = [(torch.zeros(3, 3, T, L, device="cuda"), torch.zeros(3, 3, T, device="cuda")) for _ in range(2)]
    ts = m.beam_device(ctx, 3, T, -1)

    def run(maps):
        a, p = maps if maps else (None, None)
        for x in (maps or ()):
            x.fill_(-1.0)
        m._sync_in()
        m._check(m.lib.sat_beam_search_maps(m._h, m._p(ctx), 3, 3, T, -1, *[m._p(t) for t in ts[:5]], m._p(a), m._p(p),
                                            m._st()))
        m.stream.synchronize()
        if maps:
            for k in range(3):
                for j in range(len(ref[k])):
                    assert_close(a[k, j].cpu().numpy(), ref_alpha[k][j], "beam alphas")
    for _ in range(2):
        run(sets[0]); run(None); run(sets[1]); run(sets[0])


def test_beam_maps_config5():
    """config 5 (128 images x beam 3, T=30, L=196, H=1024, V=10000), on the decidable images of test_config5_as_stated."""
    from test_gpu_beam import pick_eos_fast
    ocfg, w, m = make_pair(128, beam=3, num_lstm_units=1024, vocabulary_size=10000, max_caption_length=30)
    ctx = R.synth_contexts(ocfg, 128)
    stepper = R.HoistedStepper(ocfg, w, ctx, np.float64)
    eos = pick_eos_fast(ocfg, w, ctx[:8])
    ref = R.beam_search(ocfg, w, ctx, eos_id=eos, dtype=np.float64, step_fn=stepper.step, fast_topk=True)
    rng = np.random.RandomState(5)

    def noisy(cx, lw, lm, lo):
        mem, out, probs = stepper.step(cx, lw, lm, lo)
        return mem, out, probs * (1.0 + 3e-5 * rng.standard_normal(probs.shape))
    ref2 = R.beam_search(ocfg, w, ctx, eos_id=eos, dtype=np.float64, step_fn=noisy, fast_topk=True)
    got = m.beam_search(ctx, eos_id=eos, with_attention=True)
    decidable = [k for k in range(128)
                 if len(ref[k]) == len(ref2[k]) and all(a.sentence == b.sentence for a, b in zip(ref[k], ref2[k]))]
    assert len(decidable) >= 115, len(decidable)
    beam_compare(ocfg, w, ctx, got, ref, decidable, hoist=True)
