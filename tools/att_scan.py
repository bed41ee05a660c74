"""Attention kernel time vs number of CTAs (cold L2), config 2.   python tools/att_scan.py"""
import ctypes as C, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sat_b200
B, L, D, H, V, T = 64, 196, 512, 1024, 10000, 20
cfg = sat_b200.Config(batch_size=B, beam_size=1, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V, max_caption_length=T)
m = sat_b200.CaptionGenerator(cfg)
g = torch.Generator().manual_seed(1)
m.set_weights({n: torch.rand(*s, generator=g) * 0.16 - 0.08 for n, s in sat_b200.weight_shapes(cfg).items()})
ctx = torch.relu(torch.randn(B, L, D, generator=g)).cuda()
hs = (torch.rand(B, H, generator=g) - 0.5).cuda()
alpha = torch.empty(B, L, device="cuda"); z = torch.empty(B, D, device="cuda")
flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
m.prepare(ctx, want_state=False)
p = lambda t: C.c_void_p(t.data_ptr())
for occ, sms in ((8, 132), (16, 132), (8, 64), (16, 64)):
    for cold in (True, False):
        m.set_option("att_warps", occ)
        m.set_option("att_sms", sms)
        m.set_option("profile", 0)
        with torch.cuda.stream(m.stream):
            for i in range(13):
                if i == 3:
                    torch.cuda.synchronize(); m.set_option("profile", 1)
                if cold:
                    flush.zero_()
                m.lib.sat_attention_fwd(m._h, p(ctx), p(hs), p(alpha), p(z), B, 1, m._st())
        torch.cuda.synchronize()
        us = m.info("prof_ns_att") / max(1, m.info("prof_n_att")) / 1e3
        print("warps %d att_sms %3d  %s  %.2f us/launch (events)  -> %.0f GB/s" % (occ, sms, "cold" if cold else "warm", us, 51.69e6 / us / 1e3), flush=True)
