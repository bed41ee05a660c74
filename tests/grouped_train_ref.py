"""Autograd oracle of the grouped, row-weighted training step (sat_train_forward_backward_grouped), built on
oracle/train_ref.forward_torch without changing it.

rows = n_img * group; row r is a caption of image r // group and contexts are [n_img, L, D].  What depends on the image
alone (context mean, initialize, attend fc_a / fc_1a) uses masks drawn for n_img rows (att_ctx: the first n_img * L rows
of the step's mask, the generator being flat-indexed); every other mask is drawn per row.  This is forward_torch run
on the contexts replicated to the rows, with each image-level mask replicated likewise: the two are the same function
of the weights, so the gradients agree.

Row weights w_r scale the cross entropy only: loss = sum_r w_r sum_t m_rt CE_rt / msum + attention loss (+ reg), with
accuracy and the attention loss taken on the unweighted masks.  forward_torch's cross entropy with masks m_rt * w_r and
the normaliser msum given explicitly is exactly that first term, so the loss is the sum of two forward passes.
"""
from unittest import mock

import numpy as np

from oracle import train_ref as TR


def _grouped_masks(group, L):
    init_masks, step_masks = TR.init_masks, TR.step_masks

    def init(cfg, seed, rows):
        return {k: np.repeat(v, group, axis=0) for k, v in init_masks(cfg, seed, rows // group).items()}

    def step(cfg, seed, t, rows):
        dm = step_masks(cfg, seed, t, rows)
        ni = rows // group
        img = dm["att_ctx"][:ni * L].reshape(ni, L, -1)
        dm["att_ctx"] = np.repeat(img, group, axis=0).reshape(rows * L, -1)
        return dm
    return init, step


def forward_torch(cfg, w, contexts, sentences, masks, seed=None, global_mask_sum=None, global_batch=None, group=1,
                  row_weights=None):
    """Losses of the grouped, row-weighted step as torch float64 scalars (keys of train_ref.forward_torch)."""
    G = int(group)
    rows = np.shape(sentences)[0]
    assert rows % G == 0 and np.shape(contexts)[0] == rows // G
    ctx = np.repeat(np.asarray(contexts), G, axis=0)
    mk = np.asarray(masks, np.float64)
    msum = float(mk.sum()) if global_mask_sum is None else float(global_mask_sum)
    init, step = _grouped_masks(G, cfg.num_ctx)
    with mock.patch.object(TR, "init_masks", init), mock.patch.object(TR, "step_masks", step):
        out = TR.forward_torch(cfg, w, ctx, sentences, mk, seed, msum, global_batch)
        if row_weights is not None:
            wm = mk * np.asarray(row_weights, np.float64).reshape(rows, 1)
            ce = TR.forward_torch(cfg, w, ctx, sentences, wm, seed, msum, global_batch)["cross_entropy_loss"]
            out = dict(out, cross_entropy_loss=ce, total_loss=ce + out["attention_loss"] + out["reg_loss"])
    return out


def loss_and_grads(cfg, weights_np, contexts, sentences, masks, seed=None, global_mask_sum=None, global_batch=None,
                   reg_in_grad=True, group=1, row_weights=None):
    """train_ref.loss_and_grads for the grouped, row-weighted step."""
    import torch
    w = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in weights_np.items()}
    out = forward_torch(cfg, w, contexts, sentences, masks, seed, global_mask_sum, global_batch, group, row_weights)
    loss = out["total_loss"] if reg_in_grad else out["cross_entropy_loss"] + out["attention_loss"]
    grads = torch.autograd.grad(loss, [w[k] for k in w], allow_unused=True)
    g = {k: (np.zeros_like(weights_np[k], dtype=np.float64) if gi is None else gi.numpy()) for k, gi in zip(w, grads)}
    return {k: float(v.detach()) for k, v in out.items()}, g
