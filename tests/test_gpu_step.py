"""Parity of the CUDA decode path with the oracle (and the committed golden vectors), through the
reference-shaped facade, which calls the C ABI."""
import os

import numpy as np
import pytest

from _util import SMALL, TOL, assert_close, make_pair, rel_err
from oracle import ref_step as R

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("tag,layers", [("2layer", 2), ("1layer", 1)])
def test_golden_step_and_loop(tag, layers):
    import sat_b200
    z = np.load(os.path.join(GOLD, "step_%s.npz" % tag))
    cfg = sat_b200.Config(batch_size=3, beam_size=1, num_attend_layers=layers, num_decode_layers=layers,
                          num_initalize_layers=layers, **SMALL)
    m = sat_b200.CaptionGenerator(cfg)
    assert m.set_weights({k[2:]: z[k] for k in z.files if k.startswith("w:")}) == 0
    r = m.decode_step(z["ctx"], z["last_word"], z["last_memory"], z["last_output"], extras=True)
    for k in ("memory", "output", "probs", "logits", "alpha"):
        assert_close(r[k], z["step_" + k], "%s/%s" % (tag, k))
    c0, h0 = m.initialize(z["ctx"])
    assert_close(c0, z["c0"], "c0")
    assert_close(h0, z["h0"], "h0")
    toks, logits = m.decode_loop(z["ctx"], 6, z["forced"], want_logits=True)
    assert_close(logits, z["loop_logits"], "loop logits")
    assert (toks == z["tokens"]).all()


@pytest.mark.parametrize("layers", [2, 1])
def test_config1_reference_default_graph(layers):
    """BASELINE config 1: B=4, L=196, D=512, H=512, V=5000 (the reference's default graph)."""
    ocfg, w, m = make_pair(4, num_attend_layers=layers, num_decode_layers=layers, num_initalize_layers=layers)
    ctx = R.synth_contexts(ocfg, 4)
    rng = np.random.RandomState(0)
    lw = rng.randint(0, 5000, 4).astype(np.int32)
    c = rng.uniform(-0.5, 0.5, (4, 512)).astype(np.float32)
    h = rng.uniform(-0.5, 0.5, (4, 512)).astype(np.float32)
    ref = R.decode_step(ocfg, w, ctx, lw, c, h, np.float64)
    got = m.decode_step(ctx, lw, c, h, extras=True)
    for k in ("memory", "output", "probs", "logits", "alpha"):
        assert_close(got[k], ref[k], k)
    # host-buffer form (what a sess.run caller sees) returns the same three tensors
    mem, out, probs = m.decode_step(ctx, lw, c, h)
    assert_close(mem, ref["memory"], "memory(host)")
    assert_close(probs, ref["probs"], "probs(host)")
    np.testing.assert_allclose(probs.sum(1), 1.0, rtol=1e-4)
    # fp32 oracle is inside the same budget (both fp32 sides bounded by the fp64 truth)
    ref32 = R.decode_step(ocfg, w, ctx, lw, c, h, np.float32)
    assert rel_err(ref32["logits"], ref["logits"]) < 1e-4


def test_n1_alpha_invariant_under_hidden_state_on_gpu():
    ocfg, w, m = make_pair(4)
    ctx = R.synth_contexts(ocfg, 4)
    rng = np.random.RandomState(1)
    lw = np.zeros(4, np.int32)
    c = rng.uniform(-0.5, 0.5, (4, 512)).astype(np.float32)
    a1 = m.decode_step(ctx, lw, c, rng.uniform(-0.5, 0.5, (4, 512)).astype(np.float32), extras=True)["alpha"]
    a2 = m.decode_step(ctx, lw, c, rng.uniform(-2, 2, (4, 512)).astype(np.float32), extras=True)["alpha"]
    assert np.abs(a1 - a2).max() < 1e-6
    np.testing.assert_allclose(a1.sum(1), 1.0, rtol=1e-5)


def test_config2_twenty_teacher_forced_steps():
    """BASELINE config 2: B=64, L=196, D=512, H=1024, V=10000, T=20 — error growth through the recurrence."""
    ocfg, w, m = make_pair(64, num_lstm_units=1024, vocabulary_size=10000)
    ctx = R.synth_contexts(ocfg, 64)
    rng = np.random.RandomState(2)
    forced = rng.randint(1, 10000, (64, 20)).astype(np.int32)
    toks_ref, steps = R.decode_loop(ocfg, w, ctx, 20, forced, np.float32)
    toks, logits = m.decode_loop(ctx, 20, forced, want_logits=True)
    for t in (0, 9, 19):
        assert_close(logits[t], steps[t]["logits"], "logits step %d" % t)
    # argmax agrees wherever the reference's top-1 margin is not a numerical tie
    for t in range(20):
        lg = steps[t]["logits"]
        top2 = np.sort(lg, axis=1)[:, -2:]
        clear = (top2[:, 1] - top2[:, 0]) > 2 * TOL * np.abs(lg).max()
        assert (toks[clear, t] == toks_ref[clear, t]).all()
    # greedy loop twice (second call replays the CUDA graph) is bit-identical
    g1 = m.decode_loop(ctx, 20)
    g2 = m.decode_loop(ctx, 20)
    g3 = m.decode_loop(ctx, 20)
    assert (g1 == g2).all() and (g2 == g3).all()


def test_config3_wide_features_three_steps():
    """BASELINE config 3 shapes (D=2048, H=1536) at L=49 (what the reference's ResNet path yields) and B=32."""
    ocfg, w, m = make_pair(32, num_ctx=49, dim_ctx=2048, num_lstm_units=1536, vocabulary_size=10000)
    ctx = R.synth_contexts(ocfg, 32)
    _, steps = R.decode_loop(ocfg, w, ctx, 3, None, np.float32)
    _, logits = m.decode_loop(ctx, 3, None, want_logits=True)
    assert_close(logits[2], steps[2]["logits"], "logits step 2")


def test_hoisted_and_per_step_projection_agree():
    ocfg, w, m = make_pair(4)
    ctx = R.synth_contexts(ocfg, 4)
    a = m.decode_loop(ctx, 5, None, want_logits=True)[1]
    m.set_option("hoist", 0)          # recompute attend/fc_1a every step, like model.py:259-262
    b = m.decode_loop(ctx, 5, None, want_logits=True)[1]
    m.set_option("hoist", 1)
    assert np.array_equal(a, b)


@pytest.mark.parametrize("B", [4, 64])
def test_one_pass_prologue_matches_the_three_launch_prologue(B):
    """SURVEY section 8 row f3: the mean over the L locations (model.py:240) is taken by the same pass that packs the
    conv features for the context projection (attend/fc_1a).  Same summation order and the same bf16 split as the
    separate kernels: initial state, projection and every token after it are bit-identical."""
    ocfg, w, m = make_pair(B, num_ctx=196, dim_ctx=512, dim_attend_layer=128, dim_embedding=64, num_lstm_units=64,
                           dim_initalize_layer=64, dim_decode_layer=64, vocabulary_size=200, max_caption_length=4)
    ctx = R.synth_contexts(ocfg, B, seed=3)
    out = {}
    for one in (1, 0):
        m.set_option("prologue1", one)
        c0, h0 = m.initialize(ctx)
        toks, logits = m.decode_loop(ctx, 4, None, want_logits=True)
        out[one] = (np.asarray(c0).copy(), np.asarray(h0).copy(), toks.copy(), logits.copy())
    m.set_option("prologue1", 1)
    for a, b in zip(out[1], out[0]):
        assert np.array_equal(a, b)
    ref_c, ref_h = R.initialize(ocfg, w, ctx, np.float64)
    assert_close(out[1][0], ref_c, "initial memory")
    assert_close(out[1][1], ref_h, "initial output")


def test_packed_activation_and_prepass_paths_agree():
    """Operands packed by their producer kernels (default) vs the cooperative pre-pass vs per-stage producer
    warps: the same bf16 hi/lo split feeds the same MMAs.  The two conversion paths agree bit for bit; the packed path
    issues the same MMAs in the same order, so it agrees with them to fp32 round-off."""
    ocfg, w, m = make_pair(4)
    ctx = R.synth_contexts(ocfg, 4)
    toks = {}
    m.set_option("overlap", 0)      # same attention grid in the three runs (its split-L merge order is grid dependent)
    for name, opts in (("pa", dict(pa=1, xpack=1)), ("prepass", dict(pa=0, xpack=1)), ("warps", dict(pa=0, xpack=0))):
        for k, v in opts.items():
            m.set_option(k, v)
        toks[name] = m.decode_loop(ctx, 6, None, want_logits=True)
    m.set_option("pa", 1); m.set_option("xpack", 1); m.set_option("overlap", 2)
    assert np.array_equal(toks["prepass"][0], toks["warps"][0])
    assert np.array_equal(toks["prepass"][1], toks["warps"][1])
    for t in range(6):
        assert_close(toks["pa"][1][t], toks["warps"][1][t], "packed vs converted operands, step %d" % t, tol=2e-5)


def test_loop_layouts_agree_and_pipelined_host_api():
    """The launch layouts of the greedy loop (in-order, two streams, chained on programmatic dependent launch)
    choose the same words; the pipelined host API returns what the synchronous call returns, batch by batch."""
    import torch
    ocfg, w, m = make_pair(64, num_lstm_units=1024, vocabulary_size=10000)
    rng = np.random.RandomState(5)
    batches = [R.synth_contexts(ocfg, 64) * np.float32(0.5 + 0.25 * i) for i in range(4)]
    ref = [m.decode_loop(b, 20) for b in batches]                      # default layout, synchronous host call
    for overlap, pdl, graphs in ((0, 0, 1), (0, 1, 1), (1, 1, 1), (2, 1, 0), (1, 0, 0)):
        m.set_option("overlap", overlap); m.set_option("pdl", pdl); m.set_option("graphs", graphs)
        for rep in range(2):
            got = m.decode_loop(batches[1], 20)
            assert np.array_equal(got, ref[1]), (overlap, pdl, graphs, rep)
    m.set_option("overlap", 2); m.set_option("pdl", 1); m.set_option("graphs", 1)
    # cross-batch overlap: the prologue of batch i+1 runs on its own stream under the decode steps of batch i
    dev = [torch.from_numpy(b).cuda() for b in batches]
    torch.cuda.synchronize()                                           # "xbatch" wants complete inputs
    for graphs in (0, 1):
        m.set_option("graphs", graphs); m.set_option("xbatch", 1)
        outs = [m.loop_device(dev[i % 4], 20)[0].clone() for i in range(10)]
        torch.cuda.synchronize()
        for i, o in enumerate(outs):
            assert np.array_equal(o.cpu().numpy(), ref[i % 4]), (graphs, i)
        m.set_option("xbatch", 0)
        assert np.array_equal(m.decode_step(batches[0], np.zeros(64, np.int32), np.zeros((64, 1024), np.float32),
                                            np.zeros((64, 1024), np.float32))[2].shape, (64, 10000))
    m.set_option("graphs", 1)
    host = [torch.from_numpy(b).pin_memory() for b in batches]
    toks = [torch.empty(64, 20, dtype=torch.int32).pin_memory() for _ in range(2)]
    out = []
    for rep in range(2):                                               # second round replays the captured graphs
        for i, hb in enumerate(host):
            m.loop_host_submit(hb, 20, toks[i & 1], i & 1)
            if i >= 1:
                out.append(m.loop_host_wait((i - 1) & 1).numpy().copy())
        out.append(m.loop_host_wait((len(host) - 1) & 1).numpy().copy())
    for i, o in enumerate(out):
        assert np.array_equal(o, ref[i % 4]), i
    with pytest.raises(Exception):
        m.loop_host_wait(0)                                            # nothing in flight


def test_reference_checkpoint_import(tmp_path):
    """SURVEY §8 f1: the reference saves / loads a pickled {tf_variable_name + ':0': ndarray} dict
    (base_model.py:242-278) that also holds global_step and the optimizer slots.  load() takes that file as is."""
    ocfg, w, m = make_pair(4)
    ctx = R.synth_contexts(ocfg, 4)
    want = m.decode_loop(ctx, 5, None, want_logits=True)[1]
    import sat_b200
    cfg = m.config
    m2 = sat_b200.CaptionGenerator(cfg)
    ckpt = {k + ":0": v for k, v in w.items()}
    ckpt["global_step:0"] = np.int64(12345)
    ckpt["optimizer/beta1_power:0"] = np.float32(0.5)
    ckpt["OptimizeLoss/lstm/lstm_cell/kernel/Adam:0"] = np.zeros_like(w["lstm/lstm_cell/kernel"])
    path = str(tmp_path / "289999.npy")
    np.save(path, ckpt)
    assert m2.load(None, path) == len(w)                 # every decoder variable found, extras ignored
    got = m2.decode_loop(ctx, 5, None, want_logits=True)[1]
    assert np.array_equal(got, want)
    del ckpt["decode/fc_2/bias:0"]
    np.save(path, ckpt)
    m3 = sat_b200.CaptionGenerator(cfg)
    assert m3.load(None, path) == len(w) - 1             # like the reference: counts what it could assign ...
    with pytest.raises(sat_b200.SatError) as e:          # ... but a missing variable is an error at first use
        m3.decode_loop(ctx, 2)
    assert "decode/fc_2/bias" in str(e.value)


def test_error_behaviour():
    import sat_b200
    cfg = sat_b200.Config(batch_size=2, beam_size=1, **SMALL)
    m = sat_b200.CaptionGenerator(cfg)
    ctx = np.zeros((2, 49, 64), np.float32)
    with pytest.raises(sat_b200.SatError) as e:           # weights never loaded
        m.decode_step(ctx, np.zeros(2, np.int32), np.zeros((2, 64), np.float32), np.zeros((2, 64), np.float32))
    assert "never set" in str(e.value)
    ocfg = R.OracleConfig(batch_size=2, **SMALL)
    w = R.init_weights(ocfg)
    with pytest.raises(ValueError):                       # wrong shape, like TF's assign
        m.set_weights({"lstm/lstm_cell/kernel": np.zeros((5, 5), np.float32)})
    assert m.set_weights(w) == 0
    big = np.zeros((3, 49, 64), np.float32)               # batch larger than the static graph batch
    with pytest.raises(sat_b200.SatError):
        m.decode_step(big, np.zeros(3, np.int32), np.zeros((3, 64), np.float32), np.zeros((3, 64), np.float32))


def test_replayed_loop_then_step_on_other_contexts():
    """A replayed decode-loop graph re-projects ITS contexts into the hoisted T1 on the device; a later single step on
    the contexts of an earlier prepare() must notice and project again (round-1 advisor finding: the host-side record
    was only updated on eager runs)."""
    import torch
    ocfg, w, m = make_pair(4, beam=3)
    ctx_a = torch.from_numpy(R.synth_contexts(ocfg, 4, seed=11)).cuda()
    ctx_b_np = R.synth_contexts(ocfg, 4, seed=12)
    ctx_b = torch.from_numpy(ctx_b_np).cuda()
    rng = np.random.RandomState(4)
    lw = rng.randint(0, 5000, 4).astype(np.int32)
    c = rng.uniform(-0.5, 0.5, (4, 512)).astype(np.float32)
    h = rng.uniform(-0.5, 0.5, (4, 512)).astype(np.float32)
    ref = R.decode_step(ocfg, w, ctx_b_np, lw, c, h, np.float64)
    to = lambda a, dt: torch.from_numpy(a).cuda().to(dt)
    for loops in (1, 2, 3, 4):                       # eager, capture, replay, replay
        m.prepare(ctx_b, want_state=False)
        for _ in range(loops):
            m.loop_device(ctx_a, 5)
        got = m.decode_step(ctx_b, to(lw, torch.int32), to(c, torch.float32), to(h, torch.float32),
                            contexts_changed=False, extras=True)
        torch.cuda.synchronize()
        assert_close(got["alpha"].cpu().numpy(), ref["alpha"], "alpha after %d loops" % loops)
        assert_close(got["logits"].cpu().numpy(), ref["logits"], "logits after %d loops" % loops)
    # beam search replays behave the same way
    for loops in (1, 3):
        m.prepare(ctx_b, want_state=False)
        for _ in range(loops):
            m.beam_device(ctx_a, 3, 4, 2)
        got = m.decode_step(ctx_b, to(lw, torch.int32), to(c, torch.float32), to(h, torch.float32),
                            contexts_changed=False, extras=True)
        torch.cuda.synchronize()
        assert_close(got["alpha"].cpu().numpy(), ref["alpha"], "alpha after %d beam searches" % loops)


@pytest.mark.parametrize("shape", ["config2"])
def test_chained_launch_agrees_with_the_per_layer_launches(shape):
    """sat_chain.cu (LSTM -> fc_1 || q -> vocabulary layer as phases of one persistent launch) against one launch per
    layer: the same MMAs on the same operands; the chained launch sums even and odd K blocks in two accumulators, so the
    results agree to fp32 round-off (not bit for bit), teacher forced and greedy, eager and replayed."""
    B, T, dims = 64, 20, dict(num_lstm_units=1024, vocabulary_size=10000)   # (the opt-in path serves 64-row tiles only)
    ocfg, w, m = make_pair(B, **dims)
    ctx = R.synth_contexts(ocfg, B)
    rng = np.random.RandomState(8)
    forced = rng.randint(1, ocfg.vocabulary_size, (B, T)).astype(np.int32)
    out = {}
    for chain in (1, 0):
        m.set_option("chain", chain)
        greedy = [m.decode_loop(ctx, T) for _ in range(3)]           # eager, capture, replay
        assert all(np.array_equal(greedy[0], g) for g in greedy[1:]), chain
        out[chain] = (greedy[0],) + m.decode_loop(ctx, T, forced, want_logits=True)
    m.set_option("chain", 0)
    for t in range(T):
        assert_close(out[1][2][t], out[0][2][t], "logits step %d, chained vs per-layer" % t, tol=2e-5)
    lg = out[0][2]
    top2 = np.sort(lg, axis=2)[:, :, -2:]
    clear = (top2[:, :, 1] - top2[:, :, 0]) > 1e-4 * np.abs(lg).max()           # [T, B]
    assert (out[1][1].T[clear] == out[0][1].T[clear]).all()
    same_greedy = (out[1][0] == out[0][0]).all(axis=1).mean()
    assert same_greedy >= 0.9, same_greedy        # (a numerical tie may send a greedy caption down another path)
    # and against the oracle, through the chained path
    _, steps = R.decode_loop(ocfg, w, ctx, T, forced, np.float32)
    assert_close(out[1][2][T - 1], steps[T - 1]["logits"], "logits of the last step (chained launch)")


def test_config3_as_stated():
    """BASELINE config 3 exactly as stated: B=256, L=196, D=2048, H=1536, V=10000 — the att_fused_kernel grid that fills the GPU
    with two row tiles per dense layer that bench.py --workload 3 times.  Three greedy steps, logits of each step."""
    ocfg, w, m = make_pair(256, num_ctx=196, dim_ctx=2048, num_lstm_units=1536, vocabulary_size=10000)
    ctx = R.synth_contexts(ocfg, 256)
    toks_ref, steps = R.decode_loop(ocfg, w, ctx, 3, None, np.float32)
    toks, logits = m.decode_loop(ctx, 3, None, want_logits=True)
    for t in range(3):
        assert_close(logits[t], steps[t]["logits"], "logits step %d" % t)
        lg = steps[t]["logits"]
        top2 = np.sort(lg, axis=1)[:, -2:]
        clear = (top2[:, 1] - top2[:, 0]) > 2 * TOL * np.abs(lg).max()
        assert (toks[clear, t] == toks_ref[clear, t]).all()
        if not (toks[:, t] == toks_ref[:, t]).all():
            break          # a numerical tie sent the two greedy loops down different paths: later steps differ by design
    # single step at the same shape: alpha, context-dependent state and probabilities
    rng = np.random.RandomState(3)
    lw = rng.randint(0, 10000, 256).astype(np.int32)
    c = rng.uniform(-0.5, 0.5, (256, 1536)).astype(np.float32)
    hh = rng.uniform(-0.5, 0.5, (256, 1536)).astype(np.float32)
    ref = R.decode_step(ocfg, w, ctx, lw, c, hh, np.float32)
    got = m.decode_step(ctx, lw, c, hh, extras=True)
    for k in ("memory", "output", "probs", "logits", "alpha"):
        assert_close(got[k], ref[k], "config 3 step / " + k)


def test_real_conv5_3_features():
    """SURVEY §8 f3: the decoder on REAL conv5_3 features (tests/golden/vgg_conv5_3.npz: the 14 images the reference ships,
    through its own VGG16 weights: 94 % zeros, values up to ~290 — far from the relu(N(0,1)) of the other tests, the tanh
    layers saturate) against the oracle: single step, initialize, and a teacher-forced loop with real caption ids."""
    z = np.load(os.path.join(GOLD, "vgg_conv5_3.npz"))
    ctx = z["feats"].astype(np.float32)[:12]
    sent = z["sentences"][:12, :8].astype(np.int32)
    ocfg, w, m = make_pair(12, max_caption_length=8)
    c0r, h0r = R.initialize(ocfg, w, ctx, np.float64)
    c0, h0 = m.initialize(ctx)
    assert_close(c0, c0r, "c0 (real features)")
    assert_close(h0, h0r, "h0 (real features)")
    rng = np.random.RandomState(6)
    lw = sent[:, 0]
    c = rng.uniform(-0.5, 0.5, (12, 512)).astype(np.float32)
    h = rng.uniform(-0.5, 0.5, (12, 512)).astype(np.float32)
    ref = R.decode_step(ocfg, w, ctx, lw, c, h, np.float64)
    got = m.decode_step(ctx, lw, c, h, extras=True)
    for k in ("memory", "output", "probs", "logits", "alpha"):
        assert_close(got[k], ref[k], k + " (real features)")
    _, steps = R.decode_loop(ocfg, w, ctx, 8, sent, np.float32)
    _, logits = m.decode_loop(ctx, 8, sent, want_logits=True)
    for t in (0, 3, 7):
        assert_close(logits[t], steps[t]["logits"], "loop logits step %d (real features)" % t)
