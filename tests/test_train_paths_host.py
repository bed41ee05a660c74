"""Host-only checks behind tests/test_gpu_train_paths.py: the kernel plan of the training step on hand-worked shapes,
the reduction of profiled kernel names, and that the gradient comparison rejects plausible kernel bugs (emulated in
fp64 with the autograd oracle on the CPU)."""
from unittest import mock

import numpy as np
import pytest

import grouped_train_ref as GR
from oracle import ref_step as R
from oracle import train_ref as TR
from test_gpu_train import TC_DIMS, TDIMS, grad_check
from train_plan import kernel_key, plan_diff, train_plan

GROUP_SHAPE = dict(num_ctx=196, dim_ctx=128, dim_attend_layer=128, dim_embedding=64, num_lstm_units=64,
                   dim_decode_layer=64, vocabulary_size=1000, max_caption_length=4)
C4 = dict(num_lstm_units=1024, vocabulary_size=10000, max_caption_length=4)


def lin(k):
    return {n: v for n, v in k.items() if n.startswith("lin_mma")}


def test_plan_ragged_vocabulary():
    # K = [64, 256, 256, 64], N = [128, 256, 64, 100]: fc_2 forward on wgmma, its dx (N = 100) and the stacked
    # path's d td on sgemm (V % 8 != 0: no ragged-K wgmma operand), T*B = 64 rows stacked
    f, k = train_plan(dict(TC_DIMS, vocabulary_size=100), 16, 1, 4)
    assert f["tc_ok"] and f["tc_rt"] == 16 and f["fwd"] == [True] * 4 and f["dx"] == [True, True, True, False]
    assert f["tc_vk"] == 0 and f["tc_stack"] and not f["dec_all"]
    # per step: fc_1a fwd (NT 8) + dW (8); q, lstm, fc_1, fc_2 fwd (1); fc_1, lstm, fc_1b dx (1); then 4 stacked dW (8)
    assert lin(k) == {"lin_mma_kernel<8>": 2 * 4 + 4, "lin_mma_kernel<1>": 7 * 4}
    assert k["ce_kernel<false>"] == 4 and k["dropout_steps_kernel"] == 0
    # d td = dlogits W2^T per step (M 16, N 64, K 100: no split), the rest of sgemm_kernel<false,true> is initialize
    assert k["sgemm_kernel<false,true>"] == 4 + 2 and k["sgemm_kernel<true,false>"] == 4


def test_plan_padded_dec_all_tile():
    f, k = train_plan(TC_DIMS, 48, 1, 4)                 # T*B = 192: one full 128-row tile and a padded one
    assert f["tc_rt"] == 48 and f["tc_vk"] == 128 and f["tc_stack"] and f["dec_all"]
    assert f["all_rt"] == 128 and f["all_rows"] == 256
    # dec_all: 2 forward + 2 backward products on 128-row tiles; fc_1a 2 per step and 4 stacked
    assert lin(k) == {"lin_mma_kernel<8>": 2 * 4 + 4 + 4, "lin_mma_kernel<3>": 4 * 4}
    assert k["ce_kernel<false>"] == 1 and k["dropout_steps_kernel"] == 1


def test_plan_rows_not_a_multiple_of_16():
    f, k = train_plan(TC_DIMS, 20, 1, 4)                 # tc_rt 32; T*B = 80: per-step weight gradients
    assert f["tc_rt"] == 32 and all(f["fwd"]) and not f["tc_stack"] and not f["dec_all"] and f["tc_vk"] == 128
    assert lin(k) == {"lin_mma_kernel<8>": 2 * 4, "lin_mma_kernel<2>": 8 * 4}
    assert k["sgemm_kernel<true,false>"] == 4 * 4 + 4     # the four layers' weight gradients per step + initialize


def test_plan_more_than_128_rows():
    f, k = train_plan(GROUP_SHAPE, 32, 5, 4, weighted=True)
    assert f["tc_ok"] and f["tc_rt"] == 160 and not any(f["fwd"]) and f["tc_vk"] == 0 and not f["tc_stack"]
    assert f["side_f"] and f["side_b"]
    # 132 SMs: ceil(528 / 32) = 17 row chunks, at most ceil(196 / 16) = 13; 16 rows each
    assert f["ab_chunks"] == 13 and f["ab_rows"] == 16 and f["att_bwd_ctas"] == 13 * 32
    assert lin(k) == {"lin_mma_kernel<8>": 2 * 4}         # attend/fc_1a only
    assert k["sgemm_kernel<false,true>+splitk"] == 4      # decode fc_2 dx: M 160, N 64, K = V = 1000 in 7 chunks
    assert k["att_bwd_grouped_kernel"] == 4 and k["ce_kernel<true>"] == 4 and k["expand_rows_kernel"] == 2
    assert k["pack_rows_kernel"] == 4 and "dropout_pack_kernel" not in k   # (the contexts of attend/fc_1a only)


@pytest.mark.parametrize("dims,n_img,G,chunks", [(TDIMS, 2, 8, 1), (TDIMS, 2, 17, 1), (TC_DIMS, 4, 9, 2), (TC_DIMS, 4, 16, 2)])
def test_plan_wide_groups(dims, n_img, G, chunks):
    f, k = train_plan(dims, n_img, G, dims["max_caption_length"], weighted=True)
    assert f["ab_chunks"] == chunks and k["att_bwd_grouped_kernel"] == dims["max_caption_length"]
    assert "att_bwd_fused_kernel" not in k and k["group_sum_kernel"] == 2


def test_plan_config4_on_cuda_cores():
    f, k = train_plan(C4, 64, 1, 4, train_tc=0)
    assert f["tc_ok"] and not f["side_f"] and not f["dec_all"]
    assert not any(n.startswith(("lin_mma", "pack_rows", "repack", "dropout_pack", "tanh_bwd_pack")) for n in k)
    # every forward product on the 64 batch rows (K >= 512, fewer tiles than SMs) splits K over a zeroed output: q,
    # LSTM, fc_1 and fc_2 per step and the four initialize layers; attend/fc_1a (B*L = 12544 rows) does not
    assert k["sgemm_kernel<false,false>+splitk"] == 4 * 4 + 4 and k["sgemm_kernel<false,false>"] == 4
    # attend/fc_1a's weight gradient (K = B*L) splits K over the accumulated gradient
    assert k["sgemm_kernel<true,false>+splitk"] >= 4 and k["sgemm_kernel<false,true>+splitk"] >= 4


def test_plan_switches():
    base = train_plan(TC_DIMS, 16, 1, 4)[1]
    assert base["softmax_context_fwd4_kernel"] == 4 and base["att_bwd_fused_kernel"] == 4 and base["dropout_steps_kernel"] == 1
    for env in ({"SAT_TRAIN_PDL": "0"}, {"SAT_TRAIN_SIDE": "0"}, {"SAT_TRAIN_SIDE": "2"}, {"SAT_TRAIN_SIDE": "3"}):
        assert train_plan(TC_DIMS, 16, 1, 4, env=env)[1] == base, env
    f, k = train_plan(TC_DIMS, 16, 1, 4, env={"SAT_TRAIN_SIDE": "0"})
    assert not f["side_f"] and not f["side_b"]
    f, k = train_plan(TC_DIMS, 16, 1, 4, env={"SAT_TRAIN_SIDE": "3"})
    assert not f["side_f"] and f["side_b"]
    k = train_plan(TC_DIMS, 16, 1, 4, env={"SAT_TRAIN_FUSE_SOFTMAX": "0"})[1]
    assert k["softmax_rows_kernel"] == k["context_fwd4_kernel"] == k["softmax_bwd_kernel"] == 4
    assert "softmax_context_fwd4_kernel" not in k
    k = train_plan(TC_DIMS, 16, 1, 4, env={"SAT_TRAIN_FUSE_SOFTMAX": "2"})[1]
    assert k["softmax_context_fwd4_kernel"] == 4 and k["softmax_bwd_kernel"] == 4
    f, k = train_plan(TC_DIMS, 16, 1, 4, env={"SAT_TRAIN_ATTBWD_WAVE": "1"})
    assert k["att_bwd_fused_wave_kernel"] == 4 and "att_bwd_fused_kernel" not in k and f["ab_chunks"] is None
    f, k = train_plan(TC_DIMS, 16, 1, 4, env={"SAT_TRAIN_DEC_ALL": "0"})
    assert not f["dec_all"] and k["ce_kernel<false>"] == 4 and "dropout_steps_kernel" not in k
    k = train_plan(TC_DIMS, 16, 1, 4, env={"SAT_TRAIN_FUSE_PACK": "0"})[1]
    assert "dropout_pack_kernel" not in k and "tanh_bwd_pack_kernel" not in k
    assert k["pack_rows_kernel"] > base["pack_rows_kernel"]
    # TDIMS: only the LSTM layer (K 128, N 128) is on wgmma, no stacked gradients: DEC_ALL has nothing to switch
    f, k = train_plan(TDIMS, 4, 1, 5, env={"SAT_TRAIN_DEC_ALL": "0"})
    assert f["fwd"] == [False, True, True, False] and not f["tc_stack"] and k == train_plan(TDIMS, 4, 1, 5)[1]


def test_kernel_names():
    assert kernel_key("void (anonymous namespace)::sgemm_kernel<false, true>(int, int, int, float const*)", (1, 2, 7)) == \
        "sgemm_kernel<false,true>+splitk"
    assert kernel_key("void (anonymous namespace)::sgemm_kernel<true, false>(int)", (4, 4, 1)) == "sgemm_kernel<true,false>"
    assert kernel_key("_ZN12_GLOBAL__N_112sgemm_kernelILb1ELb0EEEviiiPKfiS2_iPfiii") == "sgemm_kernel<true,false>"
    assert kernel_key("void sat::lin_mma_kernel<3, false, false>(sat::LinLaunch)") == "lin_mma_kernel<3>"
    assert kernel_key("_ZN3sat14lin_mma_kernelILi2ELb0ELb0EEEvNS_9LinLaunchE") == "lin_mma_kernel<2>"
    assert kernel_key("void (anonymous namespace)::ce_kernel<true>(float const*)") == "ce_kernel<true>"
    # a name inside another must not match it
    assert kernel_key("void (anonymous namespace)::drop_tanh_bwd_kernel(float*)") == "drop_tanh_bwd_kernel"
    assert kernel_key("_ZN12_GLOBAL__N_120drop_tanh_bwd_kernelEPfPKfmPKyyfm") == "drop_tanh_bwd_kernel"
    assert kernel_key("void (anonymous namespace)::softmax_context_fwd4_kernel(float*)") == "softmax_context_fwd4_kernel"
    assert kernel_key("void (anonymous namespace)::att_bwd_fused_wave_kernel(float*)") == "att_bwd_fused_wave_kernel"
    assert kernel_key("void at::native::vectorized_elementwise_kernel<4>(int)") is None
    assert kernel_key("spin_kernel") is None
    rec = [("void (anonymous namespace)::sgemm_kernel<false, true>(int)", (1, 2, 7)), ("mean_L_kernel", None)]
    assert plan_diff({"sgemm_kernel<false,true>+splitk": 1, "mean_L_kernel": 1}, rec) == ""
    assert plan_diff({"sgemm_kernel<false,true>": 1, "mean_L_kernel": 1}, rec) != ""
    assert plan_diff({"sgemm_kernel<false,true>": 1, "mean_L_kernel": 1}, [(rec[0][0], None), rec[1]]) == ""


# ============================================================================================ the comparator
G_WIDE, N_WIDE, SEED = 9, 2, 5


class Grads(object):
    def __init__(self, g):
        self.g = g

    def train_state_dict(self, which):
        import torch
        return {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in self.g.items()}


@pytest.fixture(scope="module")
def wide():
    ocfg = R.OracleConfig(batch_size=N_WIDE * G_WIDE, **TDIMS)
    w = R.init_weights(ocfg, seed=3)
    rng = np.random.RandomState(3)
    rows, T = N_WIDE * G_WIDE, ocfg.max_caption_length
    ctx = R.synth_contexts(ocfg, N_WIDE, 3)
    sent = rng.randint(1, ocfg.vocabulary_size, (rows, T)).astype(np.int32)
    masks = (np.arange(T)[None, :] < rng.randint(1, T + 1, rows)[:, None]).astype(np.float32)
    rw = rng.uniform(-1.5, 2.0, rows).astype(np.float32)
    args = (ocfg, w, ctx, sent, masks, SEED)
    _, ref = GR.loss_and_grads(*args, reg_in_grad=False, group=G_WIDE, row_weights=rw)
    return args, rw, ref


def test_comparator_accepts_the_oracle(wide):
    args, rw, ref = wide
    assert grad_check(Grads(ref), ref, 2e-4, floor_rel=1e-3) == 0.0


def test_comparator_rejects_lost_later_tile_rows(wide):
    """A grouped scorer backward that drops the rows of its second tile: rows 8 and later of each image add nothing to
    attend/fc_1a (their T1 is detached)."""
    import torch
    args, rw, ref = wide
    ocfg = args[0]
    L, rows = ocfg.num_ctx, N_WIDE * G_WIDE
    tanh = torch.tanh
    late = torch.from_numpy((np.arange(rows) % G_WIDE >= 8).repeat(L))[:, None]

    def t1_tanh(x):   # T1 = tanh(drop(ctx) W1a + b1a) is the only tanh over rows * L rows
        y = tanh(x)
        return torch.where(late, y.detach(), y) if x.shape[0] == rows * L else y
    with mock.patch.object(torch, "tanh", t1_tanh):
        _, bad = GR.loss_and_grads(*args, reg_in_grad=False, group=G_WIDE, row_weights=rw)
    assert np.abs(bad["attend/fc_1a/kernel"] - ref["attend/fc_1a/kernel"]).max() > 0
    with pytest.raises(AssertionError, match="fc_1a"):
        grad_check(Grads(bad), ref, 2e-4, floor_rel=1e-3)


def test_comparator_rejects_a_shifted_att_mid_mask(wide):
    """The att_mid dropout mask of step t drawn from step t + 1's stream."""
    args, rw, ref = wide
    step_masks = TR.step_masks

    def shifted(cfg, seed, t, B):
        dm = step_masks(cfg, seed, t, B)
        dm["att_mid"] = step_masks(cfg, seed, t + 1, B)["att_mid"]
        return dm
    with mock.patch.object(TR, "step_masks", shifted):
        _, bad = GR.loss_and_grads(*args, reg_in_grad=False, group=G_WIDE, row_weights=rw)
    with pytest.raises(AssertionError):
        grad_check(Grads(bad), ref, 2e-4, floor_rel=1e-3)
