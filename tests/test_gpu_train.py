"""Training step on the GPU (sat_train.cu) against the autograd oracle (oracle/train_ref.py): losses, every
gradient, clip + Adam, and the data-parallel shard identity — with dropout off and with injected masks."""
import numpy as np
import pytest

from _util import make_pair
from oracle import ref_step as R
from oracle import train_ref as TR

pytestmark = pytest.mark.gpu

TDIMS = dict(num_ctx=9, dim_ctx=64, dim_embedding=32, num_lstm_units=32, dim_initalize_layer=16,
             dim_attend_layer=24, dim_decode_layer=40, vocabulary_size=50, max_caption_length=5)


def setup(B=4, seed=3, dims=TDIMS):
    ocfg, w, m = make_pair(B, seed=seed, **dims)
    T = ocfg.max_caption_length
    rng = np.random.RandomState(seed)
    ctx = R.synth_contexts(ocfg, B, seed)
    sent = rng.randint(1, ocfg.vocabulary_size, (B, T)).astype(np.int32)
    lens = rng.randint(2, T + 1, B)
    masks = (np.arange(T)[None, :] < lens[:, None]).astype(np.float32)
    m.train_setup(B, T, weights=w)
    return ocfg, w, m, ctx, sent, masks


def grad_check(m, ref_g, tol, floor_rel=1e-4):
    got = {k: v.detach().cpu().numpy() for k, v in m.train_state_dict("grads").items()}
    worst = 0.0
    # some gradients are mathematically zero (dropout off: the 2-layer scorer does not depend on the state
    # branch, SURVEY.md N1): compare those against the size of a typical gradient, not against round-off
    floor = floor_rel * max(np.abs(g).max() for g in ref_g.values())
    for k, g in ref_g.items():
        scale = max(np.abs(g).max(), floor)
        err = np.abs(got[k].reshape(g.shape) - g).max() / scale
        worst = max(worst, err)
        assert err < tol, "%s: gradient max-norm relative error %.3e" % (k, err)
    return worst


@pytest.mark.parametrize("seed", [0, 77])
def test_losses_and_gradients_match_autograd(seed):
    ocfg, w, m, ctx, sent, masks = setup()
    ref_l, ref_g = TR.loss_and_grads(ocfg, w, ctx, sent, masks, seed if seed else None, reg_in_grad=False)
    losses = m.train_forward_backward(ctx, sent, masks, seed=seed).cpu().numpy()
    ce, acc, att, reg = [float(x) for x in losses]
    assert abs(ce - ref_l["cross_entropy_loss"]) < 1e-4 * ref_l["cross_entropy_loss"]
    assert abs(att - ref_l["attention_loss"]) < 1e-4 * ref_l["attention_loss"] + 1e-9
    assert abs(reg - ref_l["reg_loss"]) < 1e-4 * ref_l["reg_loss"]
    assert abs(acc - ref_l["accuracy"]) < 1e-6
    grad_check(m, ref_g, 2e-4)


TC_DIMS = dict(num_ctx=32, dim_ctx=128, dim_embedding=64, num_lstm_units=64, dim_initalize_layer=16,
               dim_attend_layer=128, dim_decode_layer=64, vocabulary_size=72, max_caption_length=4)


@pytest.mark.parametrize("seed", [0, 31])
def test_tensor_core_attend_projection_in_training(seed):
    """Shapes at which attend/fc_1a (forward and weight gradient; dim_ctx, dim_attend_layer and B*L multiples of 128)
    and every batch-row product (forward, and dx where the output width is a multiple of 64) run on the wgmma dense
    kernel: same parity bars, and agreement with the CUDA-core path."""
    # B = 16, T = 4: T*B = 64 rows, so the weight gradients of the batch-row layers are also taken as ONE stacked
    # product per layer after the time loop
    ocfg, w, m, ctx, sent, masks = setup(B=16, seed=11, dims=TC_DIMS)
    ref_l, ref_g = TR.loss_and_grads(ocfg, w, ctx, sent, masks, seed if seed else None, reg_in_grad=False)
    res = {}
    for tc in (1, 0):
        m.set_option("train_tc", tc)
        losses = m.train_forward_backward(ctx, sent, masks, seed=seed).cpu().numpy()
        ce, acc, att, reg = [float(x) for x in losses]
        assert abs(ce - ref_l["cross_entropy_loss"]) < 1e-4 * ref_l["cross_entropy_loss"], tc
        assert abs(att - ref_l["attention_loss"]) < 1e-4 * ref_l["attention_loss"] + 1e-9, tc
        grad_check(m, ref_g, 2e-4)
        res[tc] = {k: v.detach().cpu().numpy().copy() for k, v in m.train_state_dict("grads").items()}
    m.set_option("train_tc", 1)
    g1, g0 = res[1]["attend/fc_1a/kernel"], res[0]["attend/fc_1a/kernel"]
    assert np.abs(g1 - g0).max() <= 1e-4 * np.abs(g0).max()
    assert np.abs(g1 - g0).max() > 0          # the two paths really differ (bf16x3 tensor cores vs fp32 FMA)


def test_adam_update_matches_tf_semantics():
    ocfg, w, m, ctx, sent, masks = setup(seed=5)
    w64 = {k: v.astype(np.float64) for k, v in w.items()}
    mm = {k: np.zeros_like(v) for k, v in w64.items()}
    vv = {k: np.zeros_like(v) for k, v in w64.items()}
    for step in (1, 2, 3):
        _, g = TR.loss_and_grads(ocfg, w64, ctx, sent, masks, 100 + step, reg_in_grad=True)
        # exaggerate the gradient so that the global-norm clip is active on step 2
        w64, mm, vv, norm = TR.clip_and_adam(w64, g, mm, vv, step, lr=1e-4, clip=5.0 if step != 2 else 1e-3)
        m.config.clip_gradients = 5.0 if step != 2 else 1e-3
        out = m.train_step(ctx, sent, masks, seed=100 + step)
        assert abs(out["gradient_norm"] - norm) < 2e-4 * norm
        got = {k: v.detach().cpu().numpy() for k, v in m.train_state_dict("params").items()}
        for k in w64:
            # parameters move by ~lr per step: compare the UPDATE, not the value
            np.testing.assert_allclose(got[k].reshape(w64[k].shape), w64[k], rtol=0, atol=3e-6)
    m.config.clip_gradients = 5.0


def test_data_parallel_shards_sum_to_global_gradient():
    ocfg, w, m, ctx, sent, masks = setup(B=4, seed=9)
    _, ref_g = TR.loss_and_grads(ocfg, w, ctx, sent, masks, None, reg_in_grad=False)
    msum = float(masks.sum())
    m.train_setup(2, ocfg.max_caption_length, weights=w)          # a "rank" holds half of the batch
    tot = None
    for lo in (0, 2):
        m.train_forward_backward(ctx[lo:lo + 2], sent[lo:lo + 2], masks[lo:lo + 2], 0, msum, 4)
        g = m.grads.clone()
        tot = g if tot is None else tot + g                        # what the NCCL all-reduce computes
    m.grads.copy_(tot)
    grad_check(m, ref_g, 2e-4)


def test_training_reduces_the_loss_and_feeds_the_decoder():
    ocfg, w, m, ctx, sent, masks = setup(seed=11)
    m.config.initial_learning_rate = 3e-3
    first = m.train_step(ctx, sent, masks, seed=1)["total_loss"]
    for it in range(2, 40):
        last = m.train_step(ctx, sent, masks, seed=it)["total_loss"]
    assert last < 0.75 * first   # (every step draws new dropout masks: the two losses are noisy samples)
    assert m.sync_inference_weights() == 0                          # trained weights drive the decode kernels
    toks = m.decode_loop(ctx, ocfg.max_caption_length)
    assert toks.shape == (4, ocfg.max_caption_length)


def test_mask_sum_from_device_memory():
    """sat_train_forward_backward_dsum: the whole-batch mask sum as a device scalar gives the same step."""
    import torch
    ocfg, w, m, ctx, sent, masks = setup(seed=5)
    a = m.train_forward_backward(ctx, sent, masks, seed=9, global_mask_sum=float(masks.sum()) * 2, global_batch=8).cpu().numpy().copy()
    ga = m.grads.detach().cpu().numpy().copy()
    dsum = torch.tensor([float(masks.sum()) * 2], dtype=torch.float64, device=m.device)
    b = m.train_forward_backward(ctx, sent, masks, seed=9, global_mask_sum=dsum, global_batch=8).cpu().numpy()
    assert np.allclose(a, b, rtol=1e-6, atol=0)
    assert np.allclose(ga, m.grads.detach().cpu().numpy(), rtol=1e-5, atol=1e-9)


def test_reference_shapes_one_step():
    """default reference graph (L=196, D=512, H=512, V=5000), B=8, T=4: losses against the oracle forward."""
    dims = dict(max_caption_length=4)
    ocfg, w, m, ctx, sent, masks = setup(B=8, seed=2, dims=dims)
    dm = [TR.step_masks(ocfg, 5, t, 8) for t in range(4)]
    ref = R.train_forward(ocfg, w, ctx, sent, masks, np.float32, dm, TR.init_masks(ocfg, 5, 8))
    ce, acc, att, reg = [float(x) for x in m.train_forward_backward(ctx, sent, masks, seed=5).cpu().numpy()]
    assert abs(ce - ref["cross_entropy_loss"]) < 1e-3 * ref["cross_entropy_loss"]
    assert abs(att - ref["attention_loss"]) < 1e-3 * ref["attention_loss"]
    assert abs(reg - ref["reg_loss"]) < 1e-3 * ref["reg_loss"]
    g = m.grads
    assert bool(g.isfinite().all()) and float(g.abs().max()) > 0


@pytest.mark.parametrize("seed", [0, 21])
def test_config4_widths_every_gradient(seed):
    """BASELINE config 4 per-GPU shapes (B=64, L=196, D=512, H=1024, V=10000; T=4 keeps the fp64 autograd oracle to
    seconds): losses and EVERY gradient against the oracle at the widths bench.py --workload 4 times, dropout off
    and with injected masks — the shapes at which every product of the step runs on the wgmma dense kernel
    (attend/fc_1a forward + weight gradient, the batch-row layers, the stacked weight gradients with T*B = 256 rows,
    the ragged K = V input gradient of the vocabulary layer)."""
    import warnings
    dims = dict(num_lstm_units=1024, vocabulary_size=10000, max_caption_length=4)
    ocfg, w, m, ctx, sent, masks = setup(B=64, seed=13, dims=dims)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref_l, ref_g = TR.loss_and_grads(ocfg, w, ctx, sent, masks, seed if seed else None, reg_in_grad=False)
    losses = m.train_forward_backward(ctx, sent, masks, seed=seed).cpu().numpy()
    ce, acc, att, reg = [float(x) for x in losses]
    assert abs(ce - ref_l["cross_entropy_loss"]) < 1e-4 * ref_l["cross_entropy_loss"]
    assert abs(att - ref_l["attention_loss"]) < 1e-4 * ref_l["attention_loss"] + 1e-9
    assert abs(reg - ref_l["reg_loss"]) < 1e-4 * ref_l["reg_loss"]
    assert abs(acc - ref_l["accuracy"]) < 1e-6
    # (dropout off: d/d attend/fc_1b is mathematically zero, SURVEY.md N1; at these widths its fp32 round-off is 2e-8 of
    # the largest gradient, so the "typical gradient" floor for such tensors is 1e-3 of the largest one here)
    worst = grad_check(m, ref_g, 2e-4, floor_rel=1e-3 if seed == 0 else 1e-4)
    assert worst > 0
    assert m.info("train_bad_ids") == 0


def test_out_of_vocabulary_ids_are_counted_not_dereferenced():
    """TF's embedding_lookup / sparse softmax raise on ids outside [0, V); here such an id reads as a zero row, adds no
    gradient, is reported by sat_get_info("train_bad_ids"), and every gradient stays finite."""
    ocfg, w, m, ctx, sent, masks = setup(seed=6)
    bad = sent.copy()
    bad[1, 1] = ocfg.vocabulary_size + 7
    bad[2, 0] = -3
    m.train_forward_backward(ctx, bad, masks, seed=0)
    assert m.info("train_bad_ids") >= 2
    assert bool(m.grads.isfinite().all())
    m.train_forward_backward(ctx, sent, masks, seed=0)
    assert m.info("train_bad_ids") == 0


@pytest.mark.parametrize("kind,extra", [("RMSProp", dict(momentum=0.9, centered=True)), ("RMSProp", dict(momentum=0.0, centered=False)),
                                        ("Momentum", dict(momentum=0.9, use_nesterov=True)),
                                        ("Momentum", dict(momentum=0.5, use_nesterov=False)), ("SGD", dict())])
def test_other_optimizers_match_tf_semantics(kind, extra):
    """model.py:486-503: RMSProp (centered or not, rms slot starting at one), Momentum (Nesterov or not), SGD — behind the
    same global-norm clip as Adam, three steps against the fp64 restatement of the TF 1.x update rules."""
    ocfg, w, m, ctx, sent, masks = setup(seed=5)
    m.config.optimizer = kind
    m.config.initial_learning_rate = 1e-2
    for k, v in extra.items():
        setattr(m.config, k, v)
    m.train_setup(4, ocfg.max_caption_length, weights=w)
    w64 = {k: v.astype(np.float64) for k, v in w.items()}
    zeros = lambda: {k: np.zeros_like(v) for k, v in w64.items()}
    slots = {"RMSProp": [{k: np.ones_like(v) for k, v in w64.items()}, zeros(), zeros()], "Momentum": [zeros()], "SGD": []}[kind]
    for step in (1, 2, 3):
        _, g = TR.loss_and_grads(ocfg, w64, ctx, sent, masks, 100 + step, reg_in_grad=True)
        clip = 5.0 if step != 2 else 1e-3                      # the clip is active on step 2
        w64, slots, norm = TR.apply_optimizer(kind, w64, g, slots, step, lr=1e-2, clip=clip, eps=m.config.epsilon,
                                              decay=m.config.decay, momentum=m.config.momentum, centered=m.config.centered,
                                              use_nesterov=m.config.use_nesterov)
        m.config.clip_gradients = clip
        out = m.train_step(ctx, sent, masks, seed=100 + step)
        assert abs(out["gradient_norm"] - norm) < 2e-4 * norm
        got = {k: v.detach().cpu().numpy() for k, v in m.train_state_dict("params").items()}
        for k in w64:
            upd = np.abs(w64[k] - w[k].astype(np.float64)).max()
            np.testing.assert_allclose(got[k].reshape(w64[k].shape), w64[k], rtol=0, atol=max(2e-3 * upd, 3e-6), err_msg=k)
    m.config.clip_gradients = 5.0


def test_save_in_the_reference_format_and_resume(tmp_path):
    """base_model.py:242-255: {tf variable name + ':0': array} incl. global_step and the Adam slots under their TF names;
    the file resumes training bit for bit and loads into the decode path like a reference checkpoint."""
    import sat_b200
    ocfg, w, m, ctx, sent, masks = setup(seed=8)
    for it in range(3):
        m.train_step(ctx, sent, masks, seed=10 + it)
    path = m.save(str(tmp_path))
    assert path.endswith("3.npy") and (tmp_path / "config.pickle").exists()
    data = np.load(path, allow_pickle=True, encoding="latin1").item()
    assert int(data["global_step:0"]) == 3
    for k in ("word_embedding/weights:0", "lstm/lstm_cell/kernel:0", "optimizer/OptimizeLoss/lstm/lstm_cell/kernel/Adam:0",
              "optimizer/OptimizeLoss/decode/fc_2/bias/Adam_1:0", "optimizer/OptimizeLoss/beta1_power:0"):
        assert k in data, k
    assert data["lstm/lstm_cell/kernel:0"].shape == w["lstm/lstm_cell/kernel"].shape
    assert len([k for k in data if k.startswith("optimizer/OptimizeLoss/") and k.endswith("/Adam:0")]) == 20
    nxt = m.train_step(ctx, sent, masks, seed=99)
    after = m.params.clone()
    # resume in a fresh model
    m2 = sat_b200.CaptionGenerator(m.config)
    m2.train_setup(4, ocfg.max_caption_length)
    assert m2.train_restore(path) == 60 and m2.global_step == 3           # 20 variables + 2 x 20 Adam slots
    nxt2 = m2.train_step(ctx, sent, masks, seed=99)
    assert nxt2["global_step"] == 4 and abs(nxt2["total_loss"] - nxt["total_loss"]) < 1e-6 * abs(nxt["total_loss"])
    assert bool((m2.params == after).all())
    # and as an inference checkpoint (base_model.py:257-278 assigns by name, ignoring what it does not know)
    m3 = sat_b200.CaptionGenerator(m.config)
    assert m3.load(None, path) == 20
    assert m3.decode_loop(ctx, ocfg.max_caption_length).shape == (4, ocfg.max_caption_length)


@pytest.mark.parametrize("layers", [(1, 1, 1), (1, 2, 2), (2, 1, 2), (2, 2, 1)])
@pytest.mark.parametrize("seed", [0, 13])
def test_one_layer_variants_of_attend_decode_initialize(layers, seed):
    """config.py:15-19 lets each of initialize / attend / decode have one layer instead of two (model.py:362-371,
    401-414, 442-447; different variable names and, for attend, no biases and no hidden layer).  Same bars as the
    shipped graph: losses to 1e-4, every gradient to 2e-4, with dropout off and on; and one optimizer step."""
    la, ld, li = layers
    dims = dict(TDIMS, num_attend_layers=la, num_decode_layers=ld, num_initalize_layers=li)
    ocfg, w, m, ctx, sent, masks = setup(B=4, seed=5, dims=dims)
    names = set(m.train_state_dict("grads"))
    assert names == set(w), names ^ set(w)
    ref_l, ref_g = TR.loss_and_grads(ocfg, w, ctx, sent, masks, seed if seed else None, reg_in_grad=False)
    losses = m.train_forward_backward(ctx, sent, masks, seed=seed).cpu().numpy()
    ce, acc, att, reg = [float(x) for x in losses]
    assert abs(ce - ref_l["cross_entropy_loss"]) < 1e-4 * ref_l["cross_entropy_loss"]
    assert abs(att - ref_l["attention_loss"]) < 1e-4 * ref_l["attention_loss"] + 1e-9
    assert abs(reg - ref_l["reg_loss"]) < 1e-4 * ref_l["reg_loss"]
    grad_check(m, ref_g, 2e-4, floor_rel=1e-3)
    # clip + Adam on top (reg gradient included), against the oracle's update of every variable
    w64 = {k: v.astype(np.float64) for k, v in w.items()}
    _, g = TR.loss_and_grads(ocfg, w64, ctx, sent, masks, 100, reg_in_grad=True)
    zeros = lambda: {k: np.zeros_like(v) for k, v in w64.items()}
    new_w, _, _, norm = TR.clip_and_adam(w64, g, zeros(), zeros(), 1, lr=1e-4, clip=5.0)
    out = m.train_step(ctx, sent, masks, seed=100)
    assert abs(out["gradient_norm"] - norm) < 2e-4 * norm
    got = {k: v.detach().cpu().numpy() for k, v in m.train_state_dict("params").items()}
    for k in w64:
        np.testing.assert_allclose(got[k].reshape(w64[k].shape), new_w[k], rtol=0, atol=3e-6)
    # the trained variables drive the decode kernels of the same handle
    assert m.sync_inference_weights() == 0
    assert m.decode_loop(ctx, ocfg.max_caption_length).shape == (4, ocfg.max_caption_length)
