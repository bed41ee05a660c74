"""Host side of self-critical training: the grouped / row-weighted training oracle (grouped_train_ref.py) against the
ungrouped one (oracle/train_ref.py), and the advantage (baseline) arithmetic of CaptionGenerator.scst_step."""
import numpy as np
import pytest

from oracle import ref_step as R
from oracle import train_ref as TR

import grouped_train_ref as GR


def small_cfg(layers=(2, 2, 2)):
    la, ld, li = layers
    return R.OracleConfig(num_ctx=9, dim_ctx=16, dim_embedding=8, num_lstm_units=16, dim_initalize_layer=8,
                          dim_attend_layer=8, dim_decode_layer=16, vocabulary_size=30, batch_size=3,
                          max_caption_length=4, num_attend_layers=la, num_decode_layers=ld, num_initalize_layers=li)


def data(cfg, n_img, group, seed=0):
    rng = np.random.RandomState(seed)
    w = R.init_weights(cfg, seed)
    ctx = R.synth_contexts(cfg, n_img, seed)
    rows, T = n_img * group, cfg.max_caption_length
    sent = rng.randint(1, cfg.vocabulary_size, (rows, T)).astype(np.int32)
    masks = (np.arange(T)[None, :] < rng.randint(1, T + 1, rows)[:, None]).astype(np.float32)
    return w, ctx, sent, masks


@pytest.mark.parametrize("seed", [None, 5])
def test_group_one_equals_the_ungrouped_oracle(seed):
    cfg = small_cfg()
    w, ctx, sent, masks = data(cfg, 3, 1)
    a_l, a_g = TR.loss_and_grads(cfg, w, ctx, sent, masks, seed, reg_in_grad=False)
    b_l, b_g = GR.loss_and_grads(cfg, w, ctx, sent, masks, seed, reg_in_grad=False, group=1)
    assert a_l == b_l
    for k in a_g:
        assert np.array_equal(a_g[k], b_g[k]), k
    c_l, c_g = GR.loss_and_grads(cfg, w, ctx, sent, masks, seed, reg_in_grad=False, group=1, row_weights=np.ones(3))
    for k in a_l:
        assert abs(a_l[k] - c_l[k]) <= 1e-13 * max(1.0, abs(a_l[k])), k
    for k in a_g:
        np.testing.assert_allclose(c_g[k], a_g[k], rtol=1e-12, atol=1e-16, err_msg=k)


@pytest.mark.parametrize("layers", [(2, 2, 2), (1, 2, 1)])
def test_grouped_oracle_equals_replicated_contexts_without_dropout(layers):
    cfg = small_cfg(layers)
    n_img, G = 2, 3
    w, ctx, sent, masks = data(cfg, n_img, G, seed=1)
    a_l, a_g = GR.loss_and_grads(cfg, w, ctx, sent, masks, None, reg_in_grad=False, group=G)
    b_l, b_g = TR.loss_and_grads(cfg, w, np.repeat(ctx, G, axis=0), sent, masks, None, reg_in_grad=False)
    for k in a_l:
        assert abs(a_l[k] - b_l[k]) <= 1e-12 * max(1.0, abs(b_l[k])), k
    for k in a_g:
        np.testing.assert_allclose(a_g[k], b_g[k], rtol=1e-10, atol=1e-14, err_msg=k)


@pytest.mark.parametrize("seed", [None, 7])
def test_row_weights_scale_each_rows_cross_entropy_only(seed):
    """Weighted cross entropy = sum_r w_r x (the cross entropy of row r alone, over the whole-batch mask sum)."""
    cfg = small_cfg()
    w, ctx, sent, masks = data(cfg, 3, 1, seed=2)
    rw = np.array([0.5, -1.25, 0.0])
    msum = float(masks.sum())
    base, _ = TR.loss_and_grads(cfg, w, ctx, sent, masks, seed, reg_in_grad=False)
    got, _ = GR.loss_and_grads(cfg, w, ctx, sent, masks, seed, reg_in_grad=False, row_weights=rw)
    per_row = []
    for r in range(3):
        only = masks * (np.arange(3) == r)[:, None]
        per_row.append(TR.loss_and_grads(cfg, w, ctx, sent, only, seed, msum, reg_in_grad=False)[0]["cross_entropy_loss"])
    assert abs(got["cross_entropy_loss"] - float(np.dot(rw, per_row))) < 1e-12
    assert got["accuracy"] == base["accuracy"] and got["attention_loss"] == base["attention_loss"]


def test_image_level_masks_are_shared_by_the_rows_of_an_image():
    cfg = small_cfg()
    n_img, G, L = 2, 3, cfg.num_ctx
    init, step = GR._grouped_masks(G, L)
    im, ref = init(cfg, 9, n_img * G), TR.init_masks(cfg, 9, n_img)
    for k in ref:
        np.testing.assert_array_equal(im[k], np.repeat(ref[k], G, axis=0))
    dm, rows = step(cfg, 9, 2, n_img * G), TR.step_masks(cfg, 9, 2, n_img * G)
    np.testing.assert_array_equal(dm["att_ctx"].reshape(n_img * G, L, -1),
                                  np.repeat(rows["att_ctx"][:n_img * L].reshape(n_img, L, -1), G, axis=0))
    for k in ("att_out", "att_mid", "lstm_in", "dec_in"):   # row-level masks: as drawn for the rows
        np.testing.assert_array_equal(dm[k], rows[k])
    w, ctx, sent, masks = data(cfg, n_img, G, seed=3)
    a_l, _ = GR.loss_and_grads(cfg, w, ctx, sent, masks, 9, reg_in_grad=False, group=G)
    b_l, _ = TR.loss_and_grads(cfg, w, np.repeat(ctx, G, axis=0), sent, masks, 9, reg_in_grad=False)
    assert np.isfinite(a_l["total_loss"]) and a_l["cross_entropy_loss"] != b_l["cross_entropy_loss"]


def test_advantages_greedy_baseline():
    from sat_b200.captions import scst_advantages
    r = np.array([[1.0, 2.0, 0.5, 1.5], [0.0, 0.0, 3.0, 1.0]])
    adv, ms, mb = scst_advantages(r, 3, "greedy")
    np.testing.assert_array_equal(adv, [[-0.5, 0.5, -1.0], [-1.0, -1.0, 2.0]])
    assert ms == pytest.approx(6.5 / 6) and mb == pytest.approx(1.25)


def test_advantages_leave_one_out_mean():
    from sat_b200.captions import scst_advantages
    r = np.array([[1.0, 2.0, 4.0], [3.0, 3.0, 3.0]])
    adv, ms, mb = scst_advantages(r, 3, "mean")
    np.testing.assert_allclose(adv, [[1.0 - 3.0, 2.0 - 2.5, 4.0 - 1.5], [0.0, 0.0, 0.0]])
    np.testing.assert_allclose(adv.sum(axis=1), 0.0, atol=1e-12)   # leave-one-out: zero-sum per image
    assert ms == pytest.approx(16 / 6)
    assert mb == pytest.approx(np.mean([3.0, 2.5, 1.5, 3.0, 3.0, 3.0]))


def test_advantages_reject_bad_input():
    from sat_b200.captions import scst_advantages
    with pytest.raises(ValueError):
        scst_advantages(np.zeros((2, 1)), 1, "mean")          # leave-one-out needs K >= 2
    with pytest.raises(ValueError):
        scst_advantages(np.zeros((2, 3)), 3, "greedy")        # the greedy column is missing
    with pytest.raises(ValueError):
        scst_advantages(np.zeros((2, 4)), 3, "mean")
    with pytest.raises(ValueError):
        scst_advantages(np.zeros((2, 3)), 3, "max")


def test_cut_after_eos():
    from sat_b200.captions import cut_after_eos
    assert cut_after_eos([4, 2, 5, 2], 2) == [4, 2]
    assert cut_after_eos(np.array([2, 7]), 2) == [2]
    assert cut_after_eos([4, 5], 2) == [4, 5]
