"""Cost of the per-word maps (sat_decode_loop_maps / sat_beam_search_maps) on an H100.

    python tools/maps_cost.py [--steps 20] [--warmup 5] [--rounds 5]

In one process, alternating A/B rounds of `steps` calls each (graphs on, contexts resident on the device):
  - the workload-2 greedy loop of bench.py (B=64, T=20, V=10000) with alphas and word probabilities against the plain loop;
  - the workload-5 beam search (128 images x beam 3, T=30) with maps against the plain beam search.
Prints one JSON line: the card's name and power limit, and per workload the median ms per call of either form and the
overhead in per cent.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import sat_b200
    if not torch.cuda.is_available():
        raise SystemExit("maps_cost.py needs an H100: no CUDA device visible")
    torch.cuda.set_device(0)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:   # (the numbers are still reported; the card is then unnamed)
        card = "unknown (%s)" % e
    out = {"metric": "maps_overhead", "gpu": card, "steps": args.steps, "rounds": args.rounds, "legs": {}}
    for wid in (2, 5):
        wl = WORKLOADS[wid]
        B, L, D, H, V, T = (wl[k] for k in "BLDHVT")
        beam = wl.get("beam", 1)
        cfg = sat_b200.Config(batch_size=B, beam_size=beam, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V,
                              max_caption_length=T)
        model = sat_b200.CaptionGenerator(cfg)
        wg = torch.Generator(device="cpu").manual_seed(1234)
        assert model.set_weights({n: (torch.rand(*s, generator=wg) * 0.16 - 0.08)
                                  for n, s in sat_b200.weight_shapes(cfg).items()}) == 0
        g = torch.Generator(device="cpu").manual_seed(1234)
        ctx = torch.relu(torch.randn(B, L, D, generator=g)).cuda()
        torch.cuda.synchronize()
        if beam > 1:
            calls = {"plain": lambda: model.beam_device(ctx, beam, T, 2),
                     "maps": lambda: model.beam_device(ctx, beam, T, 2, with_attention=True)}
        else:
            calls = {"plain": lambda: model.loop_device(ctx, T),
                     "maps": lambda: model.loop_maps_device(ctx, T)}
        for f in calls.values():
            for _ in range(max(args.warmup, 3)):   # eager run, capture, replays
                f()
        torch.cuda.synchronize()
        ms = {k: [] for k in calls}
        st = model.stream
        for _ in range(args.rounds):
            for k, f in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(st):
                    e0.record(st)
                    for _ in range(args.steps):
                        f()
                    e1.record(st)
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1) / args.steps)
        med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
        out["legs"]["workload%d" % wid] = {
            "name": wl["name"], "ms_per_call_plain": med["plain"], "ms_per_call_maps": med["maps"],
            "overhead_pct": 100.0 * (med["maps"] / med["plain"] - 1.0), "ms_per_call_rounds": ms}
        model.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
