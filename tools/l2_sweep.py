"""L2 eviction-policy sweep of the workload-2 greedy loop (bench.py: B=64, L=196, D=512, H=1024, V=10000, T=20).

    python tools/l2_sweep.py [--steps 20] [--rounds 5]

Policies (option values, see l2_policy in sat_common.cuh): 1 = evict_first, 2 = evict_last, 3 = evict_normal.
`l2_w` is the hint of every dense weight stream of a step, `l2_vocab` overrides it for the vocabulary layer
(-1: the library's default, evict_first for the weights of the decode step).  The settings alternate within each
round; graphs on, cross-batch overlap on, contexts rotating over six device batches, as in bench.py.  Prints ms per loop (median and range over the rounds) and the card's name and
power limit.  If "all evict_first" and "all evict_last" time the same, no weight is reused from L2 across steps.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sat_b200  # noqa: E402

SETTINGS = [   # (label, l2_w, l2_vocab); (-1, -1) = the library's default
    ("default", -1, -1),
    ("all evict_first", 1, 1),
    ("all evict_last", 2, 2),
    ("all evict_normal", 3, 3),
    ("weights evict_last, vocab evict_first", 2, 1),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    B, L, D, H, V, T = 64, 196, 512, 1024, 10000, 20
    cfg = sat_b200.Config(batch_size=B, beam_size=1, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V,
                          max_caption_length=T)
    m = sat_b200.CaptionGenerator(cfg)
    wg = torch.Generator().manual_seed(1234)
    m.set_weights({n: torch.rand(*s, generator=wg) * 0.16 - 0.08 for n, s in sat_b200.weight_shapes(cfg).items()})
    g = torch.Generator().manual_seed(1)
    pool = [torch.relu(torch.randn(B, L, D, generator=g)).cuda() for _ in range(6)]
    m.set_option("xbatch", 1)

    def timeit():
        for i in range(14):   # eager run, capture, one replay per pool entry
            m.loop_device(pool[i % 6], T)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(m.stream):
            a.record(m.stream)
            for i in range(args.steps):
                m.loop_device(pool[i % 6], T)
            b.record(m.stream)
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps

    res = {lab: [] for lab, _, _ in SETTINGS}
    for _ in range(args.rounds):
        for lab, w, v in SETTINGS:
            m.set_option("l2_w", w)      # (an option change drops the captured graphs)
            m.set_option("l2_vocab", v)
            res[lab].append(timeit())
    out = {"gpu": card, "workload": "bench.py workload 2, graphed loop", "rounds": args.rounds, "steps": args.steps,
           "settings": []}
    for lab, w, v in SETTINGS:
        x = sorted(res[lab])
        out["settings"].append({"setting": lab, "l2_w": w, "l2_vocab": v, "ms_per_loop_median": x[len(x) // 2],
                                "ms_per_loop_min": x[0], "ms_per_loop_max": x[-1],
                                "us_per_step_median": x[len(x) // 2] * 1e3 / T})
        print("%-40s %.3f ms/loop  [%.3f, %.3f]  %.1f us/step" % (lab, x[len(x) // 2], x[0], x[-1], x[len(x) // 2] * 1e3 / T),
              flush=True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
