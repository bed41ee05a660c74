"""The decode loop's attention beside the vocabulary layer.

Inside the single-stream loop (overlap = 2) the attention of step t+1 is launched, without waiting for the vocabulary
layer of step t, on the SMs that layer leaves idle (#SMs - 79 at V = 10000: 53 on an H100), also when that is fewer
than the images and CTA row ranges cross image boundaries.  These tests check, at the config-2 shape (L = 196,
D = 512, H = 1024, V = 10000):
  * the plan: every batch size, including those with more images than idle SMs, runs beside the vocabulary layer;
  * the timeline: the attention's first CTA starts before the vocabulary layer's last CTA ends;
  * the values: tokens, logits, alphas and word probabilities of the greedy, maps and sampling loops against the fp64
    oracle fed the same words, and against the in-order layout (overlap = 0);
  * reproducibility: eager call, captured graph and replays, and the two "xbatch" buffer sets, bit for bit;
  * the self-resetting counters: a loop after a loop of another batch size gives what a fresh handle gives."""
import numpy as np
import pytest

from _util import TOL, assert_close, make_pair
from oracle import ref_step as R

pytestmark = pytest.mark.gpu

BENCH = dict(num_lstm_units=1024, vocabulary_size=10000)
T = 3


def oracle_fed(ocfg, w, ctx, tokens):
    """fp64 oracle logits / alphas / word probabilities with the words the device loop chose fed back in."""
    _, steps = R.decode_loop(ocfg, w, ctx, tokens.shape[1], tokens, np.float64)
    logits = np.stack([s["logits"] for s in steps], 1)
    alphas = np.stack([s["alpha"] for s in steps], 1)
    probs = np.stack([steps[t]["probs"][np.arange(ctx.shape[0]), tokens[:, t]] for t in range(tokens.shape[1])], 1)
    return logits, alphas, probs


def check_choice(tokens, logits_ref, what):
    """Every token is the arg-max of the reference logits wherever the top-2 margin exceeds the parity bar."""
    bar = TOL * np.abs(logits_ref).max()
    top2 = np.sort(logits_ref, -1)[..., -2:]
    clear = top2[..., 1] - top2[..., 0] > bar
    best = logits_ref.argmax(-1)
    assert clear.mean() > 0.5, what
    assert np.array_equal(tokens[clear], best[clear]), what


def loop_grid(n_img, sms, L=196, vocab_tiles=79):
    """att_plan's grid on the SMs the vocabulary layer leaves (loop_enqueue_chain's budget)."""
    budget = sms - vocab_tiles
    if budget < sms // 4:
        budget = sms
    grid = min(n_img * L, budget)
    if n_img <= budget:
        k = min(budget // n_img, L)
        if k >= 1 and n_img * k >= 0.8 * grid:
            grid = n_img * k
    return grid


def planned_beside(m, n_img):
    grid = m.info("att_loop_grid")
    assert m.info("att_loop_beside") == 1, n_img
    assert grid == loop_grid(n_img, m.info("num_sms")), (n_img, grid)


@pytest.mark.parametrize("B", [1, 53, 54, 63, 64])
def test_greedy_loop_beside_vocabulary(B):
    ocfg, w, m = make_pair(B, max_caption_length=T, **BENCH)
    try:
        ctx = R.synth_contexts(ocfg, B, seed=B)
        r = m.decode_loop(ctx, T, want_logits=True, want_alphas=True, want_word_probs=True)
        planned_beside(m, B)
        logits, alphas, probs = oracle_fed(ocfg, w, ctx, r["tokens"])
        got = r["logits"].transpose(1, 0, 2)                  # [T, B, V] -> [B, T, V]
        assert_close(got, logits, "logits B=%d" % B)
        assert_close(r["alphas"], alphas, "alphas B=%d" % B)
        assert_close(r["word_probs"], probs, "word_probs B=%d" % B)
        check_choice(r["tokens"], logits, "tokens B=%d" % B)
        # the in-order layout computes the same
        m.set_option("overlap", 0)
        s = m.decode_loop(ctx, T, want_logits=True, want_alphas=True, want_word_probs=True)
        assert_close(r["logits"], s["logits"], "logits vs overlap=0, B=%d" % B)
        assert_close(r["word_probs"], s["word_probs"], "word_probs vs overlap=0, B=%d" % B)
        assert_close(r["alphas"], s["alphas"], "alphas vs overlap=0, B=%d" % B)
        check_choice(r["tokens"], s["logits"].transpose(1, 0, 2).astype(np.float64), "tokens vs overlap=0, B=%d" % B)
        # teacher forcing takes the same launch
        m.set_option("overlap", 2)
        forced = np.random.RandomState(B).randint(0, ocfg.vocabulary_size, (B, T)).astype(np.int32)
        f = m.decode_loop(ctx, T, forced_words=forced, want_logits=True, want_word_probs=True)
        planned_beside(m, B)
        logits_f, _, probs_f = oracle_fed(ocfg, w, ctx, forced)
        assert_close(f["logits"].transpose(1, 0, 2), logits_f, "forced logits B=%d" % B)
        assert_close(f["word_probs"], probs_f, "forced word_probs B=%d" % B)
    finally:
        m.close()


class _DeviceWords:
    """A device buffer the library owns, seen by torch as int64 words (__cuda_array_interface__)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="<i8", data=(ptr, False), strides=None, version=3)


def test_attention_starts_before_vocabulary_ends():
    import torch
    B = 64
    ocfg, w, m = make_pair(B, max_caption_length=6, **BENCH)
    try:
        ctx = torch.from_numpy(R.synth_contexts(ocfg, B)).cuda()
        m.set_option("graphs", 0)
        for _ in range(2):
            m.loop_device(ctx, 6)
        torch.cuda.synchronize()
        m.set_option("trace", 3)
        m.loop_device(ctx, 6)
        torch.cuda.synchronize()
        n = m.info("tl_count")
        host = torch.as_tensor(_DeviceWords(m.info("trace_ptr"), 4 * n), device="cuda").cpu().numpy()
        names = []
        for i in range(n):
            m.info("tl_tag_%d" % i)
            names.append(m.lib.sat_last_error().decode().strip())
        m.set_option("trace", 0)
        pairs = [(i, i + 1) for i in range(n - 1) if names[i].startswith("dec2") and names[i + 1].startswith("attention")]
        assert len(pairs) == 5, names
        for v, a in pairs:
            vocab_end, att_start = int(host[4 * v + 1]), int(host[4 * a])
            assert att_start < vocab_end, (names[v], names[a], att_start, vocab_end)
    finally:
        m.close()


def test_replays_and_xbatch_slots_bit_identical():
    import torch
    B = 64
    ocfg, w, m = make_pair(B, max_caption_length=4, **BENCH)
    try:
        ctx = torch.from_numpy(R.synth_contexts(ocfg, B)).cuda()
        m.set_option("graphs", 0)
        m.set_option("xbatch", 1)
        torch.cuda.synchronize()
        t0, l0 = (x.clone() for x in m.decode_loop(ctx, 4, want_logits=True))   # eager, buffer set 0
        m.set_option("graphs", 1)
        for i in range(5):   # sets 1, 0, 1, 0, 1: each set's graph captured, then replayed
            t, l = m.decode_loop(ctx, 4, want_logits=True)
            assert torch.equal(t, t0) and torch.equal(l, l0), i
        planned_beside(m, B)
    finally:
        m.close()


def test_counters_reset_between_batch_sizes():
    import torch
    ocfg, w, m = make_pair(64, max_caption_length=T, **BENCH)
    _, _, fresh = make_pair(17, max_caption_length=T, max_batch=64, **BENCH)
    try:
        ctx = torch.from_numpy(R.synth_contexts(ocfg, 64)).cuda()
        first = [x.clone() for x in m.decode_loop(ctx, T, want_logits=True)]
        small = [x.clone() for x in m.decode_loop(ctx[:17].contiguous(), T, want_logits=True)]
        ref = fresh.decode_loop(ctx[:17].contiguous(), T, want_logits=True)
        assert all(torch.equal(a, b) for a, b in zip(small, ref))
        again = m.decode_loop(ctx, T, want_logits=True)
        assert all(torch.equal(a, b) for a, b in zip(first, again))
    finally:
        m.close()
        fresh.close()


@pytest.mark.parametrize("n,G", [(64, 1), (16, 4)])
def test_sampling_beside_vocabulary(n, G):
    import torch
    ocfg, w, m = make_pair(64, max_caption_length=T, **BENCH)
    try:
        ctx = torch.from_numpy(R.synth_contexts(ocfg, n, seed=5)).cuda()
        tok, wp = (x.clone() for x in m.sample_device(ctx, G, T, seed=11))
        planned_beside(m, n)
        tok2, wp2 = m.sample_device(ctx, G, T, seed=11)
        assert torch.equal(tok, tok2) and torch.equal(wp, wp2)   # reproducible run to run
        # the words drawn, fed to the fp64 oracle (row r of image r // G), give the same word probabilities
        rows = tok.reshape(n * G, T).cpu().numpy()
        octx = np.repeat(ctx.cpu().numpy(), G, 0).astype(np.float64)
        _, _, probs = oracle_fed(ocfg, w, octx, rows)
        assert_close(wp.reshape(n * G, T).cpu().numpy(), probs, "sampled word_probs %dx%d" % (n, G))
        # the in-order layout draws the same words from (almost) the same probabilities
        m.set_option("overlap", 0)
        tok0, wp0 = m.sample_device(ctx, G, T, seed=11)
        same = (tok0 == tok).all(-1).reshape(-1).cpu().numpy()
        assert same.mean() >= 0.95, same.mean()
        assert_close(wp.reshape(n * G, T).cpu().numpy()[same], wp0.reshape(n * G, T).cpu().numpy()[same],
                     "sampled word_probs vs overlap=0")
    finally:
        m.close()
