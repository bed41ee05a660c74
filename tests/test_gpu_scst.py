"""Grouped, row-weighted training step (sat_train_forward_backward_grouped) and self-critical training
(CaptionGenerator.scst_step) against the autograd oracle (grouped_train_ref.py on top of oracle/train_ref.py)."""
import numpy as np
import pytest

from _util import make_pair
from oracle import ref_step as R
from oracle import train_ref as TR
from test_gpu_train import TC_DIMS, TDIMS, grad_check

import grouped_train_ref as GR

pytestmark = pytest.mark.gpu


def gsetup(n_img, G, seed=3, dims=TDIMS, max_batch=None):
    ocfg, w, m = make_pair(n_img * G, seed=seed, max_batch=max_batch, **dims)
    T = ocfg.max_caption_length
    rng = np.random.RandomState(seed)
    ctx = R.synth_contexts(ocfg, n_img, seed)
    rows = n_img * G
    sent = rng.randint(1, ocfg.vocabulary_size, (rows, T)).astype(np.int32)
    masks = (np.arange(T)[None, :] < rng.randint(1, T + 1, rows)[:, None]).astype(np.float32)
    rw = rng.uniform(-1.5, 2.0, rows).astype(np.float32)
    rw[::3] = 0.0
    rw[1] = -abs(rw[1]) - 0.5                       # zero and negative weights present
    m.train_setup(n_img, T, weights=w, group=G)
    return ocfg, w, m, ctx, sent, masks, rw


def check_losses(losses, ref_l):
    ce, acc, att, reg = [float(x) for x in losses]
    assert abs(ce - ref_l["cross_entropy_loss"]) < 1e-4 * abs(ref_l["cross_entropy_loss"])
    assert abs(att - ref_l["attention_loss"]) < 1e-4 * ref_l["attention_loss"] + 1e-9
    assert abs(reg - ref_l["reg_loss"]) < 1e-4 * ref_l["reg_loss"]
    assert abs(acc - ref_l["accuracy"]) < 1e-6


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("seed", [0, 77])
@pytest.mark.parametrize("G", [1, 2, 3, 5])
def test_grouped_step_matches_autograd(G, seed, weighted):
    ocfg, w, m, ctx, sent, masks, rw = gsetup(2, G)
    rw = rw if weighted else None
    ref_l, ref_g = GR.loss_and_grads(ocfg, w, ctx, sent, masks, seed if seed else None, reg_in_grad=False, group=G,
                                     row_weights=rw)
    losses = m.train_forward_backward(ctx, sent, masks, seed=seed, group=G, row_weights=rw).cpu().numpy()
    check_losses(losses, ref_l)
    grad_check(m, ref_g, 2e-4, floor_rel=1e-3)


@pytest.mark.parametrize("seed", [0, 13])
@pytest.mark.parametrize("layers", [(1, 2, 2), (1, 1, 1), (2, 2, 1)])
def test_grouped_step_one_layer_variants(layers, seed):
    la, ld, li = layers
    dims = dict(TDIMS, num_attend_layers=la, num_decode_layers=ld, num_initalize_layers=li)
    ocfg, w, m, ctx, sent, masks, rw = gsetup(2, 3, seed=5, dims=dims)
    ref_l, ref_g = GR.loss_and_grads(ocfg, w, ctx, sent, masks, seed if seed else None, reg_in_grad=False, group=3,
                                     row_weights=rw)
    losses = m.train_forward_backward(ctx, sent, masks, seed=seed, group=3, row_weights=rw).cpu().numpy()
    check_losses(losses, ref_l)
    grad_check(m, ref_g, 2e-4, floor_rel=1e-3)


@pytest.mark.parametrize("seed", [0, 31])
@pytest.mark.parametrize("G", [2, 5])
def test_grouped_step_tensor_core_shapes(G, seed):
    """n_img * L = 128: attend/fc_1a (forward and weight gradient) on the wgmma kernel over image rows; train_tc 1 and 0."""
    ocfg, w, m, ctx, sent, masks, rw = gsetup(4, G, seed=11, dims=TC_DIMS)
    ref_l, ref_g = GR.loss_and_grads(ocfg, w, ctx, sent, masks, seed if seed else None, reg_in_grad=False, group=G,
                                     row_weights=rw)
    for tc in (1, 0):
        m.set_option("train_tc", tc)
        losses = m.train_forward_backward(ctx, sent, masks, seed=seed, group=G, row_weights=rw).cpu().numpy()
        check_losses(losses, ref_l)
        grad_check(m, ref_g, 2e-4, floor_rel=1e-3)
    m.set_option("train_tc", 1)


@pytest.mark.parametrize("dims,B,seed", [(TDIMS, 4, 77), (TC_DIMS, 16, 31)])
def test_group_one_runs_the_ungrouped_step(dims, B, seed):
    """group 1 and NULL weights: the grouped entry launches exactly the kernels of sat_train_forward_backward (as a
    multiset: the attend/fc_1a products run on a second stream, so their interleaving in time varies) and gives the same
    losses and gradients.  (Bit equality cannot be asked of two calls: the step sums
    losses and several gradients with float atomics, whose order varies from call to call.)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    ocfg, w, m, ctx, sent, masks, _ = gsetup(B, 1, seed=11, dims=dims)
    ctx, masks = (torch.from_numpy(x).cuda() for x in (ctx, masks))

    def kernels(f):   # (a fresh sentences buffer: a new graph key, so the call runs eagerly)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = f(torch.from_numpy(sent).cuda()).clone()
            torch.cuda.synchronize()
            # a capture can stop before the records of its last kernels are delivered (they then arrive with the next
            # capture): a marker kernel on the step's stream, after its work, keeps the step's records inside this one
            with torch.cuda.stream(m.stream):
                torch.cuda._sleep(20000)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emset" not in e.name
                 and "spin_kernel" not in e.name]
        return out, m.grads.clone(), names
    dsum = masks.sum(dtype=torch.float64).reshape(1)   # (both through the device mask sum)
    a, ga, ka = kernels(lambda s: m.train_forward_backward(ctx, s, masks, seed=seed, global_mask_sum=dsum))
    b, gb, kb = kernels(lambda s: m._train_forward_backward_grouped(ctx, s, masks, seed, dsum, None, None))
    assert len(ka) > 50 and sorted(ka) == sorted(kb)
    assert torch.allclose(a, b, rtol=1e-6, atol=0)
    assert float((ga - gb).abs().max()) <= 1e-6 * float(ga.abs().max())


@pytest.mark.parametrize("dims,n_img", [(TDIMS, 2), (TC_DIMS, 4)])
def test_sharing_equals_replicated_contexts(dims, n_img):
    G = 5
    ocfg, w, m, ctx, sent, masks, rw = gsetup(n_img, G, seed=4, dims=dims)
    m.train_forward_backward(ctx, sent, masks, seed=0, group=G, row_weights=rw)
    g_shared = m.grads.detach().cpu().numpy().copy()
    m.train_setup(n_img * G, ocfg.max_caption_length, weights=w)
    m.train_forward_backward(np.repeat(ctx, G, axis=0), sent, masks, seed=0, row_weights=rw)
    g_rep = m.grads.detach().cpu().numpy()
    assert np.abs(g_shared - g_rep).max() <= 1e-5 * np.abs(g_rep).max()


def test_caption_masks():
    import torch
    eos, T = 2, 6
    toks = np.array([[2, 5, 2, 7, 7, 7],      # eos at t = 0
                     [4, 5, 2, 2, 9, 1],      # mid-caption, then repeated
                     [4, 5, 6, 7, 8, 9],      # absent
                     [4, 5, 6, 7, 8, 2]], np.int32)
    ref = np.zeros(toks.shape, np.float32)
    for r, row in enumerate(toks):
        hit = np.flatnonzero(row == eos)
        ref[r, :(hit[0] + 1 if hit.size else T)] = 1
    ocfg, w, m = make_pair(4, **TDIMS)
    tk = torch.from_numpy(toks).cuda()
    mk = torch.full(toks.shape, -1.0, device="cuda")
    s = torch.zeros(1, dtype=torch.float64, device="cuda")
    assert m.lib.sat_caption_masks(m._p(tk), 4, T, eos, m._p(mk), m._p(s), None) == 0
    assert m.lib.sat_caption_masks(m._p(tk), 4, T, eos, m._p(mk), None, None) == 0
    torch.cuda.synchronize()
    np.testing.assert_array_equal(mk.cpu().numpy(), ref)
    assert float(s) == ref.sum()
    assert m.lib.sat_caption_masks(None, 4, T, eos, m._p(mk), None, None) == -1
    assert m.lib.sat_caption_masks(m._p(tk), 4, 0, eos, m._p(mk), None, None) == -1


def test_on_policy_identity():
    """seed = 0 and unit weights: the step's summed cross entropy on sampled captions is the sampler's own
    sum of -log p(word) over the kept words."""
    import torch
    n, K = 3, 4
    ocfg, w, m, ctx, _, _, _ = gsetup(n, K, seed=6, dims=dict(TDIMS, max_caption_length=6))
    T = ocfg.max_caption_length
    c = torch.from_numpy(ctx).cuda()
    m.sync_inference_weights(sync=False)
    tokens, wp = m.sample_device(c, K, T, 1.0, seed=123)
    torch.cuda.synchronize()
    sent = tokens.reshape(n * K, T).clone()
    mk = torch.empty(n * K, T, device="cuda")
    msum = torch.zeros(1, dtype=torch.float64, device="cuda")
    assert m.lib.sat_caption_masks(m._p(sent), n * K, T, 2, m._p(mk), m._p(msum), None) == 0
    torch.cuda.synchronize()
    losses = m.train_forward_backward(c, sent, mk, seed=0, global_mask_sum=msum, group=K,
                                      row_weights=torch.ones(n * K, device="cuda")).cpu().numpy()
    mks = mk.cpu().numpy()
    expect = float((-np.log(wp.reshape(n * K, T).cpu().numpy().astype(np.float64)) * mks).sum())
    assert abs(float(losses[0]) * float(msum) - expect) < 1e-4 * expect


def test_graph_replay_reads_new_row_weights():
    import torch
    ocfg, w, m, ctx, sent, masks, rw = gsetup(2, 3, seed=8)
    c, s, mk = (torch.from_numpy(x).cuda() for x in (ctx, sent, masks))   # (stable addresses: graphs replay)
    buf = torch.from_numpy(rw).cuda()
    for _ in range(3):   # eager, captured, replayed
        m.train_forward_backward(c, s, mk, seed=5, group=3, row_weights=buf)
    g_a = m.grads.clone()
    rw2 = (-2.0 * rw + 0.25).astype(np.float32)
    buf.copy_(torch.from_numpy(rw2))
    m.train_forward_backward(c, s, mk, seed=5, group=3, row_weights=buf)       # replayed graph, new values
    g_b = m.grads.clone()
    other = torch.from_numpy(rw).cuda()                                               # a different buffer
    m.train_forward_backward(c, s, mk, seed=5, group=3, row_weights=other)
    g_c = m.grads.clone()
    _, ref_b = GR.loss_and_grads(ocfg, w, ctx, sent, masks, 5, reg_in_grad=False, group=3, row_weights=rw2)
    m.grads.copy_(g_b)
    grad_check(m, ref_b, 2e-4, floor_rel=1e-3)
    assert (g_b - g_a).abs().max() > 0
    assert (g_c - g_a).abs().max() <= 1e-5 * g_a.abs().max()


def test_data_parallel_image_shards_sum_to_global_gradient():
    G, n_img = 3, 4
    ocfg, w, m, ctx, sent, masks, rw = gsetup(n_img, G, seed=9)
    _, ref_g = GR.loss_and_grads(ocfg, w, ctx, sent, masks, None, reg_in_grad=False, group=G, row_weights=rw)
    msum = float(masks.sum())
    m.train_setup(2, ocfg.max_caption_length, weights=w, group=G)      # a "rank" holds half of the images
    tot = None
    for lo in (0, 2):
        r = slice(lo * G, (lo + 2) * G)
        m.train_forward_backward(ctx[lo:lo + 2], sent[r], masks[r], 0, msum, n_img * G, group=G, row_weights=rw[r])
        g = m.grads.clone()
        tot = g if tot is None else tot + g
    m.grads.copy_(tot)
    grad_check(m, ref_g, 2e-4, floor_rel=1e-3)


@pytest.mark.parametrize("baseline", ["greedy", "mean"])
def test_scst_step_matches_the_oracle_update(baseline):
    import torch
    n, K = 2, 5
    ocfg, w, m, ctx, _, _, _ = gsetup(n, K, seed=12, dims=dict(TDIMS, max_caption_length=6), max_batch=n * 4)
    T = ocfg.max_caption_length
    seen = []

    def reward(caps):   # deterministic: fraction of even word ids, plus a length term
        seen.append(caps)
        return np.array([[np.mean([wd % 2 == 0 for wd in c]) + 0.1 * len(c) for c in img] for img in caps])

    c = torch.from_numpy(ctx).cuda()
    out = m.scst_step(c, reward, num_samples=K, baseline=baseline, seed=0, sample_seed=99)
    caps = seen[0]
    assert len(caps) == n and all(len(img) == K + (baseline == "greedy") for img in caps)
    sent = m._buf("scst_sent", (n * K, T), torch.int32).cpu().numpy()
    for i in range(n):
        for k in range(K):
            assert caps[i][k] == [int(x) for x in sent[i * K + k][:len(caps[i][k])]]
    from sat_b200.captions import scst_advantages
    adv, rs, rb = scst_advantages(reward(caps), K, baseline)
    assert out["sample_reward"] == pytest.approx(rs) and out["baseline_reward"] == pytest.approx(rb)
    masks = np.zeros((n * K, T), np.float32)
    for r in range(n * K):
        hit = np.flatnonzero(sent[r] == 2)
        masks[r, :(hit[0] + 1 if hit.size else T)] = 1
    w64 = {k: v.astype(np.float64) for k, v in w.items()}
    _, g = GR.loss_and_grads(ocfg, w64, ctx, sent, masks, None, reg_in_grad=True, group=K, row_weights=adv.reshape(-1))
    zeros = lambda: {k: np.zeros_like(v) for k, v in w64.items()}
    new_w, _, _, norm = TR.clip_and_adam(w64, g, zeros(), zeros(), 1, lr=m.config.initial_learning_rate, clip=5.0)
    assert abs(out["gradient_norm"] - norm) < 2e-4 * norm
    got = {k: v.detach().cpu().numpy() for k, v in m.train_state_dict("params").items()}
    for k in w64:
        np.testing.assert_allclose(got[k].reshape(w64[k].shape), new_w[k], rtol=0, atol=3e-6, err_msg=k)


def test_scst_step_rejects_invalid_input():
    import torch
    ocfg, w, m, ctx, _, _, _ = gsetup(4, 1, max_batch=8)
    c = torch.from_numpy(ctx).cuda()
    with pytest.raises(ValueError):
        m.scst_step(c, lambda caps: None, num_samples=1, baseline="mean")
    m.train_setup(4, ocfg.max_caption_length, weights=w, group=5)
    with pytest.raises(ValueError, match="max_batch"):             # 4 images x 4 samples per call > 8 rows
        m.scst_step(c, lambda caps: None, num_samples=5)


def test_invalid_grouped_calls_enqueue_nothing():
    import torch
    ocfg, w, m, ctx, sent, masks, rw = gsetup(2, 3)
    T = ocfg.max_caption_length
    c, s, mk = (torch.from_numpy(x).cuda() for x in (ctx, sent, masks))
    wt = torch.from_numpy(rw).cuda()
    gsum = torch.tensor([float(masks.sum())], dtype=torch.float64, device="cuda")
    losses = torch.full((4,), 7.0, device="cuda")
    L = m.lib

    def call(n=2, G=3, T=T, ctx=c, sent=s, mk=mk, wt=wt, gs=gsum, out=losses, params=m.params):
        return L.sat_train_forward_backward_grouped(m._h, m._p(params), m._p(m.grads), m._p(ctx), n, G, m._p(sent), m._p(mk),
                                                    m._p(wt), T, 0, m._p(gs), 6, m._p(out), m._st())
    m.grads.fill_(3.0)
    torch.cuda.synchronize()
    for kw in (dict(G=0), dict(G=-2), dict(n=1, G=6), dict(n=3), dict(G=2), dict(T=T - 1), dict(ctx=None), dict(sent=None),
               dict(mk=None), dict(gs=None), dict(out=None), dict(params=None)):
        assert call(**kw) == -1, kw
    m.stream.synchronize()
    assert bool((losses == 7.0).all()) and bool((m.grads == 3.0).all())
    assert call(wt=None) == 0          # NULL weights are valid
