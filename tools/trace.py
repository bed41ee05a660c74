"""In-kernel timelines (globaltimer stamps) of the attention and dense kernels at config 2.
    python tools/trace.py > trace.log
"""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sat_b200

B, L, D, H, V, T = 64, 196, 512, 1024, 10000, 20
cfg = sat_b200.Config(batch_size=B, beam_size=1, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V,
                      max_caption_length=T)
m = sat_b200.CaptionGenerator(cfg)
g = torch.Generator().manual_seed(1)
m.set_weights({n: torch.rand(*s, generator=g) * 0.16 - 0.08 for n, s in sat_b200.weight_shapes(cfg).items()})
ctx = torch.relu(torch.randn(B, L, D, generator=g)).cuda()
hstate = (torch.rand(B, H, generator=g) - 0.5).cuda()
cstate = (torch.rand(B, H, generator=g) - 0.5).cuda()
lw = torch.zeros(B, dtype=torch.int32).cuda()
flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
m.prepare(ctx, want_state=False)
p = lambda t: C.c_void_p(t.data_ptr())
alpha = torch.empty(B, L, device="cuda"); z = torch.empty(B, D, device="cuda")
c2 = torch.empty_like(cstate); h2 = torch.empty_like(hstate); logits = torch.empty(B, V, device="cuda")


def read_trace(n):
    import cuda.bindings.runtime as cr
    torch.cuda.synchronize()
    host = np.zeros(1024 * 16, np.int64)
    err, = cr.cudaMemcpy(host.ctypes.data, m.info("trace_ptr"), host.nbytes, cr.cudaMemcpyKind.cudaMemcpyDeviceToHost)
    assert int(err) == 0, err
    return host.reshape(1024, 16)[:n]


def show(name, tr, labels):
    tr = tr[tr[:, 0] > 0]
    t0 = tr[:, 0].min()
    if name.startswith("attention"):
        print("  [thread 0 blocked on data: pass 1 %.2f us, pass 2 %.2f us (mean, at 1.965 GHz)]"
              % (tr[:, 8].mean() / 1965.0, tr[:, 9].mean() / 1965.0))
        print("  [thread 0 cycles->us: pass-1 loads+FMA %.2f, reduce %.2f, store+arrive %.2f; pass-2 compute+arrive %.2f]"
              % tuple(tr[:, k].mean() / 1965.0 for k in (10, 11, 12, 13)))
        tr = tr.copy(); tr[:, 8:14] = 0
    print("== %s  (us after the first CTA started; mean / max over %d CTAs)" % (name, len(tr)))
    for i, lab in enumerate(labels):
        col = tr[:, i]
        ok = col > 0
        if ok.any():
            v = (col[ok] - t0) / 1e3
            print("  %-34s mean %7.2f  min %7.2f  max %7.2f   (n=%d)" % (lab, v.mean(), v.min(), v.max(), ok.sum()))


def run(kind, fn, grid, labels, trace_mode, cold):
    for rep in range(3):
        if cold:
            flush.zero_()
        m.set_option("trace", trace_mode)
        m.set_option("trace_at", 0)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    show(kind + (" cold-L2" if cold else " warm-L2"), read_trace(grid), labels)
    m.set_option("trace", 0)


att_labels = ["start", "consumers ready", "first T1 chunk landed", "pass-1 done (seg 0)", "first ctx chunk landed",
              "pass-2 done (seg 0)", "published (seg 0)", "end"]
lin_labels = ["start", "producers start", "pack done -> arrive", "TMA thread: barrier passed", "MMA: first W stage",
              "MMA: first X stage", "MMA: all issued", "epilogue: accumulator ready", "partials written",
              "rendezvous passed", "end"]

def step_traced(k):
    """one full decode step through step_impl (packed-activation path); stamp the k-th dense launch"""
    def fn():
        m.set_option("trace_at", k)
        m.step_device(ctx, lw, cstate, hstate, want=())
    return fn


with torch.cuda.stream(m.stream):
    m.step_device(ctx, lw, cstate, hstate, want=())     # allocate everything once
    torch.cuda.synchronize()
    if "--dense" in sys.argv:
        # dense launches of one step: 0 = state branch q, 1 = LSTM, 2 = decode fc_1, 3 = decode fc_2
        for k, (name, grid) in enumerate([("step: att state (q)", 64), ("step: LSTM [packed operands]", 128),
                                          ("step: decode fc_1 [packed operands]", 128), ("step: decode fc_2 [packed]", 79)]):
            run(name, step_traced(k), grid, lin_labels, 1, False)
    for sms in (0, 64):
        m.set_option("att_sms", sms)
        for cold in (True, False):
            run("attention att_sms=%d" % sms, lambda: m.lib.sat_attention_fwd(m._h, p(ctx), p(hstate), p(alpha), p(z), B, 1, m._st()), m.info("num_sms"),
                att_labels, 2, cold)
