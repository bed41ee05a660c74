"""L2 policies of the dense weight streams are hints: they change no result."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_l2_policy_does_not_change_results():
    """Tokens and logits of the bench.py workload-2 loop (graphed) are bit-identical under the default policy and under
    one explicit policy for every weight stream."""
    import torch
    import sat_b200
    B, L, D, H, V, T = 64, 196, 512, 1024, 10000, 20
    cfg = sat_b200.Config(batch_size=B, beam_size=1, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V,
                          max_caption_length=T)
    m = sat_b200.CaptionGenerator(cfg)
    wg = torch.Generator().manual_seed(1234)
    assert m.set_weights({n: torch.rand(*s, generator=wg) * 0.16 - 0.08
                          for n, s in sat_b200.weight_shapes(cfg).items()}) == 0
    ctx = torch.relu(torch.randn(B, L, D, generator=torch.Generator().manual_seed(1234))).cuda()
    out = {}
    for l2w in (-1, 1, 2, 3):
        m.set_option("l2_w", l2w)
        for _ in range(3):   # eager run, capture, replay
            tok, lg = m.loop_device(ctx, T, want_logits=True)
        torch.cuda.synchronize()
        out[l2w] = (tok.cpu().numpy().copy(), lg.cpu().numpy().copy())
    for l2w in (1, 2, 3):
        np.testing.assert_array_equal(out[l2w][0], out[-1][0])
        np.testing.assert_array_equal(out[l2w][1], out[-1][1])
    m.close()
