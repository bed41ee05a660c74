"""Time the config-2 decode loop under different library options (one process, same weights).
    python tools/sweep.py > sweep.log
"""
import itertools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sat_b200

B, L, D, H, V, T = 64, 196, 512, 1024, 10000, 20
cfg = sat_b200.Config(batch_size=B, beam_size=1, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V,
                      max_caption_length=T)
m = sat_b200.CaptionGenerator(cfg)
g = torch.Generator().manual_seed(1)
m.set_weights({n: torch.rand(*s, generator=g) * 0.16 - 0.08 for n, s in sat_b200.weight_shapes(cfg).items()})
pool = [torch.relu(torch.randn(B, L, D, generator=g)).cuda() for _ in range(6)]


def timeit(n=30):
    for i in range(14):
        m.loop_device(pool[i % 6], T)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(m.stream):
        a.record(m.stream)
        for i in range(n):
            m.loop_device(pool[i % 6], T)
        b.record(m.stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


base = dict(overlap=1, att_sms=0, pa=1, graphs=1, pdl=1)
variants = [dict(), dict(overlap=2), dict(overlap=0), dict(overlap=2, att_sms=132), dict(graphs=0), dict(graphs=0, overlap=2), dict(graphs=0, overlap=0), dict(pdl=0)]
ref = {}
for v in variants:
    o = dict(base)
    o.update(v)
    for k, val in o.items():
        m.set_option(k, val)
    ms = timeit()
    tok, lg = m.loop_device(pool[0], T, want_logits=True)
    torch.cuda.synchronize()
    key = (o["overlap"], o["att_sms"])
    if key not in ref:
        ref[key] = (tok.clone(), lg.clone())
    same = bool((tok == ref[key][0]).all()) and bool((lg == ref[key][1]).all())
    tsame = bool((tok == ref[(1, 0)][0]).all())
    print("options %-64s  %.3f ms/loop  %.1f us/step  %.0f tok/s  bit-identical to first run of this layout: %s; tokens == base: %s"
          % (o, ms, ms * 1e3 / T, B * T / ms * 1e3, same, tsame), flush=True)
