"""CPU checks of the reference, the comparator and the plan restatement of test_gpu_decode_layers.py: the comparator
accepts a kernel that computes the split-precision product exactly as described, and rejects the faults it exists to
catch."""
import numpy as np
import pytest

from oracle import ref_step as R
from test_gpu_decode_layers import (DENSE_BAR, LOOPS, LSTM_BAR, LSTM_SHAPES, PROB_BAR, ROWS_NT, SPLITS, bf16_product,
                                    bf16_rne, dense_error, fused_argmax, instance, lstm_emulated, lstm_errors,
                                    lstm_plan, lstm_reference, row_tile_for, softmax64, split_bf16, split_product,
                                    tie_pairs, token_mismatches, vocab_emulated, vocab_reference, word_prob_error,
                                    x_mode)

SMS_H100 = 132      # SMs of an H100 SXM


def _lstm_case(H=64, rows=24, seed=0, scale_cp=2.0):
    cfg = R.OracleConfig(batch_size=rows, beam_size=1, num_ctx=4, dim_ctx=64, dim_embedding=32, num_lstm_units=H,
                         vocabulary_size=300)
    w = R.init_weights(cfg, seed=seed)
    rng = np.random.RandomState(seed)
    ctx = np.maximum(rng.standard_normal((rows, 64)), 0).astype(np.float32)
    lw = rng.randint(0, 300, rows)
    cp = rng.uniform(-scale_cp, scale_cp, (rows, H)).astype(np.float32)
    hp = rng.uniform(-1, 1, (rows, H)).astype(np.float32)
    return cfg, w, (ctx, lw, cp, hp)


def _lstm_err(cfg, w, args, **fault):
    c, h = lstm_emulated(cfg, w, *args, **fault)
    return max(lstm_errors(c.astype(np.float32), h.astype(np.float32), lstm_reference(cfg, w, *args)))


def test_comparator_accepts_the_emulated_lstm():
    cfg, w, args = _lstm_case()
    assert _lstm_err(cfg, w, args) <= LSTM_BAR / 4


@pytest.mark.parametrize("fault", [dict(product=bf16_product), dict(order=(2, 1, 0, 3)), dict(order=(0, 3, 2, 1)),
                                   dict(unit_shift=1), dict(forget_bias=0.0), dict(forget_bias=2.0)],
                         ids=["bf16-only", "i-f-swapped", "j-o-swapped", "interleave-off-by-one", "no-forget-bias",
                              "forget-bias-doubled"])
def test_comparator_rejects_a_faulty_lstm(fault):
    cfg, w, args = _lstm_case()
    assert _lstm_err(cfg, w, args, **fault) > LSTM_BAR


def _vocab_case(layers, V=301, rows=16, seed=0):
    cfg = R.OracleConfig(batch_size=rows, beam_size=1, num_ctx=4, dim_ctx=64, dim_embedding=32, num_lstm_units=64,
                         dim_decode_layer=64, num_decode_layers=layers, vocabulary_size=V)
    w = R.init_weights(cfg, seed=seed)
    rng = np.random.RandomState(seed)
    h = rng.uniform(-1, 1, (rows, 64)).astype(np.float32)
    ctx = np.maximum(rng.standard_normal((rows, 64)), 0).astype(np.float32)
    return cfg, w, (h, ctx, rng.randint(0, V, rows))


@pytest.mark.parametrize("layers", [2, 1])
def test_comparator_accepts_the_emulated_decode(layers):
    cfg, w, args = _vocab_case(layers)
    ref = vocab_reference(cfg, w, *args)
    assert dense_error(vocab_emulated(cfg, w, *args).astype(np.float32), ref["logits"], ref["scale"]) <= DENSE_BAR / 4


@pytest.mark.parametrize("layers", [2, 1])
def test_comparator_rejects_a_bf16_only_decode(layers):
    cfg, w, args = _vocab_case(layers)
    ref = vocab_reference(cfg, w, *args)
    assert dense_error(vocab_emulated(cfg, w, *args, product=bf16_product), ref["logits"], ref["scale"]) > DENSE_BAR


def test_emulation_is_the_split_product():
    """split_product equals x @ (whi + wlo) minus the xlo * wlo term; and hi + lo keeps 16 bits of every value."""
    rng = np.random.RandomState(1)
    x = rng.uniform(-1, 1, (5, 70)).astype(np.float32)
    w = rng.uniform(-0.08, 0.08, (70, 9)).astype(np.float32)
    xh, xl = split_bf16(x)
    wh, wl = split_bf16(w)
    assert np.allclose(split_product(x, w), (xh + xl) @ (wh + wl) - xl @ wl, rtol=0, atol=1e-15)
    assert (np.abs(xh + xl - x) <= np.abs(x) * 2.0 ** -16).all()
    assert bf16_rne(np.float32([1 + 2 ** -8, 1 + 3 * 2 ** -8, -1 - 2 ** -8])).tolist() == [1.0, 1 + 2 ** -6, -1.0]


def test_comparator_rejects_a_tie_to_the_larger_index():
    logits = np.random.RandomState(2).standard_normal((2, 3, 300)).astype(np.float32)
    logits[:, :, [40, 200]] = 9.0
    tokens = np.full((3, 2), 40)
    assert token_mismatches(tokens, logits) == []
    assert len(token_mismatches(np.full((3, 2), 200), logits)) == 6


@pytest.mark.parametrize("V", [300, 5000])
def test_comparator_rejects_a_probability_without_the_last_word(V):
    """A word probability whose softmax sum dropped the last valid word of the partial last tile."""
    logits = np.random.RandomState(V).standard_normal((2, 4, V)).astype(np.float32)
    fed = np.random.RandomState(1).randint(0, V - 1, (4, 2))
    sm = softmax64(logits)
    good = sm[np.arange(2)[None, :], np.arange(4)[:, None], fed]
    assert word_prob_error(good.astype(np.float32), logits, fed) < 1e-6
    bad = good / (1.0 - sm[..., V - 1].T)
    assert word_prob_error(bad.astype(np.float32), logits, fed) > PROB_BAR


def test_plan_restatement():
    """The shapes of the split cases land on the factors they claim on 132 SMs (the H100 SXM)."""
    cfgs = {k: R.OracleConfig(**dict(dict(num_ctx=4, dim_ctx=64, dim_embedding=32, num_lstm_units=64), **d))
            for k, d in LSTM_SHAPES.items()}
    for key, rows, splits in SPLITS:
        assert lstm_plan(cfgs[key], rows, SMS_H100)["splits"] == splits, (key, rows)
    assert all(lstm_plan(cfgs["small"], r, SMS_H100)["splits"] == 1 for r in ROWS_NT)
    assert [row_tile_for(r) // 16 for r in ROWS_NT] == [1, 2, 3, 4, 5, 6, 7, 8, 8, 5, 7, 8]
    assert lstm_plan(cfgs["w2"], 64, SMS_H100)["grid"] == 128 and lstm_plan(cfgs["wide"], 1, SMS_H100)["grid"] == 16
    assert x_mode(lstm_plan(cfgs["w2"], 384, SMS_H100), SMS_H100) == 1
    loop = lambda layers, V: R.OracleConfig(num_decode_layers=layers, vocabulary_size=V, dim_decode_layer=64)
    assert [fused_argmax(loop(l, v), b, SMS_H100) for l, v, b, _ in LOOPS] == [True, True, True, False, False]
    assert tie_pairs(5000)[4:] == [("tiles", 11, 1035), ("0 and V-1", 0, 4999), ("last tile", 4992, 4999)]
    assert instance("void sat::lin_mma_kernel<4, false, false>(sat::LinLaunch)") == "lin_mma_kernel<4,false,false>"
    assert instance("_ZN3sat14lin_mma_kernelILi8ELb1ELb0EEEvNS_9LinLaunchE") == "lin_mma_kernel<8,true,false>"
    assert instance("_ZN3sat19rows_softmax_kernelILb1ELb0EEEvNS_10RowsParamsE") == "rows_softmax_kernel<true,false>"
    assert instance("void at::native::spin_kernel(long)") is None
