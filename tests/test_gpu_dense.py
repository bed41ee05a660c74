"""wgmma dense kernel (split-precision bf16x3, split-K) against fp64 numpy, through the C ABI."""
import ctypes as C

import numpy as np
import pytest

from _util import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    import sat_b200
    cfg = sat_b200.Config(batch_size=4, beam_size=1, num_ctx=49, dim_ctx=64, dim_embedding=32, num_lstm_units=64,
                          dim_initalize_layer=32, dim_attend_layer=32, dim_decode_layer=64, vocabulary_size=300)
    return sat_b200.CaptionGenerator(cfg)


def run_dense(model, rows, K, n_out, act, splits, seed=0):
    import torch
    rng = np.random.RandomState(seed)
    x = rng.uniform(-1, 1, (rows, K)).astype(np.float32)
    w = rng.uniform(-0.08, 0.08, (K, n_out)).astype(np.float32)
    b = rng.uniform(-0.08, 0.08, (n_out,)).astype(np.float32)
    xd, wd, bd = (torch.from_numpy(a).cuda() for a in (x, w, b))
    y = torch.full((rows, n_out), float("nan"), device="cuda")
    torch.cuda.synchronize()
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = model.lib.sat_dense_fwd(model._h, p(xd), p(wd), p(bd), p(y), rows, K, n_out, act, splits, model._st())
    assert rc == 0, model.lib.sat_last_error()
    torch.cuda.synchronize()
    ref = x.astype(np.float64) @ w.astype(np.float64) + b
    if act:
        ref = np.tanh(ref)
    return rel_err(y.cpu().numpy(), ref)


@pytest.mark.parametrize("rows,K,n_out,act,splits", [
    (4, 64, 128, 0, 1),        # one tile, one k-block, direct epilogue
    (4, 128, 128, 0, 2),       # split-K rendezvous
    (64, 2048, 4096, 0, 0),    # LSTM-sized, heuristic splits
    (64, 1024, 10000, 0, 0),   # vocabulary GEMM: partial last tile
    (64, 1024, 512, 1, 0),     # attend fc_1b + tanh
    (3, 72, 50, 1, 1),         # ragged K (zero padded k-block) and ragged n_out
    (200, 512, 512, 1, 1),     # two activation-row tiles of N = 112
    (384, 2048, 1024, 1, 0),   # three activation-row tiles (beam-search batch)
    (784, 512, 512, 1, 1),     # context projection (4 images x 196 locations)
])
def test_dense_umma_matches_fp64(model, rows, K, n_out, act, splits):
    model.set_option("gemm", 1)
    err = run_dense(model, rows, K, n_out, act, splits)
    # split-precision bf16x3 keeps ~16 mantissa bits: far inside the 1e-3 budget
    assert err < 1e-4, err


def test_dense_cuda_core_bringup_kernel_agrees(model):
    model.set_option("gemm", 0)
    try:
        assert run_dense(model, 64, 1024, 640, 1, 1) < 1e-4
    finally:
        model.set_option("gemm", 1)


def test_dense_is_deterministic(model):
    import torch
    errs = {run_dense(model, 64, 2048, 1024, 1, 0, seed=3) for _ in range(3)}
    assert len(errs) == 1
