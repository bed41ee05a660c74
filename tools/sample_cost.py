"""Cost of sampling (sat_sample_loop) against the greedy loop on an H100.

    python tools/sample_cost.py [--steps 20] [--warmup 5] [--rounds 5] [--no-trace]

At the workload-2 model shape of bench.py (L=196, D=512, H=1024, V=10000, T=20), in one process, alternating rounds of
`steps` graphed calls each (contexts resident on the device):
  (a) greedy: the decode loop at 64 images;
  (a') greedy_probs: the same with the word probabilities (sat_decode_loop_maps, no attention maps);
  (b) sample_64x1: sampling, 64 images x 1 caption, with word probabilities;
  (b') sample_64x1_noprobs: the same without them (the draw alone);
  (c) sample_16x4: sampling, 16 images x 4 captions (the 4 rows of an image share its contexts), with word probabilities;
  (d) beam_16x4: beam search, 16 images x beam 4, for comparison;
  (e) sample_64x1_topk50, sample_64x1_topp09, sample_16x4_topp09: filtered sampling (sat_sample_loop_filtered) with
      top_k = 50 or top_p = 0.9, with word probabilities.  The vocabulary layer writes the logits and the filtered
      per-row kernel draws, one step at a time.
Then, in a block of its own (the option change drops the captured graphs), (f) sample_64x1_overlap0: plain sampling
forced into that per-step layout (option "overlap" = 0).  So (f) - (b) is the cost of the layout and (e) - (f) that of
writing the logits and running the filter kernel.
So (b') - (a) is the cost of the Gumbel draw, (a') - (a) that of the softmax partials of the word probabilities.
Then (unless --no-trace) one eager loop of (a), (a'), (b), (b'), (e) and (f) with in-kernel timeline stamps (option
"trace" = 3): the mean time from first CTA start to last CTA end of each kernel family per step ("filter": the filtered
per-row kernel).
Prints one JSON line: the card's name and power limit, the median ms per call of each leg and the per-family times.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS  # noqa: E402


def family_times(m, f):
    """mean first-start -> last-end (us) per kernel family over one eager call of f (trace = 3)."""
    import numpy as np
    import torch
    import cuda.bindings.runtime as cr
    m.set_option("graphs", 0)
    for _ in range(2):
        f()
    torch.cuda.synchronize()
    m.set_option("trace", 3)
    f()
    torch.cuda.synchronize()
    n = m.info("tl_count")
    host = np.zeros(1024 * 16, np.uint64)
    cr.cudaMemcpy(host.ctypes.data, m.info("trace_ptr"), host.nbytes, cr.cudaMemcpyKind.cudaMemcpyDeviceToHost)
    fam = {}
    for i in range(n):
        m.info("tl_tag_%d" % i)
        name = m.lib.sat_last_error().decode().split("/")[0]
        fam.setdefault(name, []).append((int(host[4 * i + 1]) - int(host[4 * i])) / 1e3)
    m.set_option("trace", 0)
    m.set_option("graphs", 1)
    return {k: {"n": len(v), "mean_us": sum(v) / len(v)} for k, v in fam.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-trace", action="store_true")
    args = ap.parse_args()
    import torch
    import sat_b200
    if not torch.cuda.is_available():
        raise SystemExit("sample_cost.py needs an H100: no CUDA device visible")
    torch.cuda.set_device(0)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:   # (the numbers are still reported; the card is then unnamed)
        card = "unknown (%s)" % e
    wl = WORKLOADS[2]
    B, L, D, H, V, T = (wl[k] for k in "BLDHVT")
    cfg = sat_b200.Config(batch_size=B, beam_size=4, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V,
                          max_caption_length=T)
    m = sat_b200.CaptionGenerator(cfg, max_batch=B)
    wg = torch.Generator(device="cpu").manual_seed(1234)
    assert m.set_weights({n: (torch.rand(*s, generator=wg) * 0.16 - 0.08)
                          for n, s in sat_b200.weight_shapes(cfg).items()}) == 0
    g = torch.Generator(device="cpu").manual_seed(1234)
    ctx = torch.relu(torch.randn(B, L, D, generator=g)).cuda()
    ctx16 = ctx[:16].contiguous()
    torch.cuda.synchronize()
    seeds = iter(range(1, 1 << 30))
    calls = {
        "greedy": lambda: m.loop_device(ctx, T),
        "greedy_probs": lambda: m.loop_maps_device(ctx, T, want_alphas=False, want_word_probs=True),
        "sample_64x1": lambda: m.sample_device(ctx, 1, T, 1.0, next(seeds)),
        "sample_64x1_noprobs": lambda: m.sample_device(ctx, 1, T, 1.0, next(seeds), want_word_probs=False),
        "sample_16x4": lambda: m.sample_device(ctx16, 4, T, 1.0, next(seeds)),
        "beam_16x4": lambda: m.beam_device(ctx16, 4, T, 2),
        "sample_64x1_topk50": lambda: m.sample_device(ctx, 1, T, 1.0, next(seeds), top_k=50),
        "sample_64x1_topp09": lambda: m.sample_device(ctx, 1, T, 1.0, next(seeds), top_p=0.9),
        "sample_16x4_topp09": lambda: m.sample_device(ctx16, 4, T, 1.0, next(seeds), top_p=0.9),
    }
    st = m.stream

    def timed(legs):
        for f in legs.values():
            for _ in range(max(args.warmup, 3)):   # eager run, capture, replays
                f()
        torch.cuda.synchronize()
        ms = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, f in legs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(st):
                    e0.record(st)
                    for _ in range(args.steps):
                        f()
                    e1.record(st)
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1) / args.steps)
        return ms

    ms = timed(calls)
    overlap0 = {"sample_64x1_overlap0": calls["sample_64x1"]}
    m.set_option("overlap", 0)
    ms.update(timed(overlap0))
    m.set_option("overlap", 2)
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    out = {"metric": "sample_cost", "gpu": card, "shape": dict(L=L, D=D, H=H, V=V, T=T), "steps": args.steps,
           "rounds": args.rounds, "ms_per_call": med,
           "vs_greedy_pct": {k: 100.0 * (v / med["greedy"] - 1.0) for k, v in med.items()}, "ms_per_call_rounds": ms}
    if not args.no_trace:
        out["trace_us"] = {k: family_times(m, calls[k])
                           for k in ("greedy", "greedy_probs", "sample_64x1", "sample_64x1_noprobs",
                                     "sample_64x1_topk50", "sample_64x1_topp09", "sample_16x4_topp09")}
        m.set_option("overlap", 0)
        out["trace_us"]["sample_64x1_overlap0"] = family_times(m, overlap0["sample_64x1_overlap0"])
        m.set_option("overlap", 2)
    m.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
