"""Cost of self-critical training on an H100: the grouped training step against the replicated one, and a whole
CaptionGenerator.scst_step.

    python tools/scst_cost.py [--steps 10] [--warmup 3] [--rounds 5] [--no-profile]

At the workload-2 model shape of bench.py (L=196, D=512, H=1024, V=10000, T=20), 64 images x 5 samples, dropout on,
alternating rounds of `steps` graphed forward+backward calls each:
  (a) xe_64: the cross-entropy step at 64 rows;
  (b) xe_320_replicated: the cross-entropy step at 320 rows, contexts replicated 5 times ([320, L, D]);
  (c) grouped_64x5: the grouped, row-weighted step, 64 images x 5 rows sharing their contexts ([64, L, D]);
  (d) scst_step: refresh of the decode weights, sampling 5 captions per image, the greedy baseline, a trivial numpy
      reward, caption masks + grouped step + optimizer; timed whole and part by part (host wall clock, synchronised).
Also the device memory each training state takes (mem_get_info around train_setup: the library's stashes plus the
flat parameter / gradient / Adam buffers, which are the same for every leg) and, unless --no-profile, the CUDA kernel
time per kernel name of one eager call of (b) and (c) (torch.profiler).
Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import WORKLOADS  # noqa: E402


def kernel_table(f):
    """{kernel name: total ms} of the CUDA kernels of one call of f."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            out[e.key[:60]] = round(out.get(e.key[:60], 0.0) + t / 1e3, 3)
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:25])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    import sat_b200
    if not torch.cuda.is_available():
        raise SystemExit("scst_cost.py needs an H100: no CUDA device visible")
    torch.cuda.set_device(0)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:   # (the numbers are still reported; the card is then unnamed)
        card = "unknown (%s)" % e
    wl = WORKLOADS[2]
    n, L, D, H, V, T = (wl[k] for k in "BLDHVT")
    K = 5
    rows = n * K
    cfg = sat_b200.Config(batch_size=n, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V, max_caption_length=T)
    g = torch.Generator(device="cpu").manual_seed(1234)
    ctx = torch.relu(torch.randn(n, L, D, generator=g)).cuda()
    ctx_rep = ctx.repeat_interleave(K, dim=0).contiguous()
    sent = torch.randint(1, V, (rows, T), generator=g, dtype=torch.int32).cuda()
    lens = torch.randint(8, T + 1, (rows,), generator=g)
    masks = (torch.arange(T)[None, :] < lens[:, None]).float().cuda()
    rw = (torch.rand(rows, generator=g) * 2 - 1).cuda()

    def model(batch, group=1):
        m = sat_b200.CaptionGenerator(cfg, max_batch=rows)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        m.train_setup(batch, T, group=group)
        torch.cuda.synchronize()
        return m, (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 20

    ma, mem_a = model(n)
    mb, mem_b = model(rows)
    mc, mem_c = model(n, K)
    seeds = iter(range(1, 1 << 30))
    legs = {
        "xe_64": (ma, lambda: ma.train_forward_backward(ctx, sent[:n], masks[:n], seed=next(seeds))),
        "xe_320_replicated": (mb, lambda: mb.train_forward_backward(ctx_rep, sent, masks, seed=next(seeds))),
        "grouped_64x5": (mc, lambda: mc.train_forward_backward(ctx, sent, masks, seed=next(seeds), group=K, row_weights=rw)),
    }
    for _, f in legs.values():
        for _ in range(max(args.warmup, 3)):   # eager run, capture, replays
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in legs}
    parts = {k: [] for k in ("whole", "refresh", "sampling", "greedy", "reward", "train")}

    def reward(caps):   # trivial: caption length
        return np.array([[float(len(c)) for c in img] for img in caps])

    def scst_parts():
        """the stages of scst_step one by one, each synchronised: wall ms per stage"""
        out = {}

        def stage(name, f):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = f()
            torch.cuda.synchronize()
            out[name] = (time.perf_counter() - t0) * 1e3
            return r
        stage("refresh", lambda: mc.sync_inference_weights(sync=False))
        tok = stage("sampling", lambda: mc.sample_device(ctx, K, T, 1.0, next(seeds), want_word_probs=False)[0])
        gt = stage("greedy", lambda: mc.loop_device(ctx, T)[0])

        def rew():
            from sat_b200.captions import cut_after_eos, scst_advantages
            tk, gk = tok.cpu().numpy(), gt.cpu().numpy()
            caps = [[cut_after_eos(tk[i, k], cfg.eos_id) for k in range(K)] + [cut_after_eos(gk[i], cfg.eos_id)]
                    for i in range(n)]
            return scst_advantages(reward(caps), K, "greedy")
        stage("reward", rew)

        def train():
            mc.train_forward_backward(ctx, sent, masks, seed=next(seeds), group=K, row_weights=rw)
            mc.train_apply()
        stage("train", train)
        return out

    for _ in range(2):
        mc.scst_step(ctx, reward, num_samples=K, seed=next(seeds))
        scst_parts()
    st = {k: m.stream for k, (m, _) in legs.items()}
    for _ in range(args.rounds):
        for k, (m, f) in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(st[k]):
                e0.record(st[k])
                for _ in range(args.steps):
                    f()
                e1.record(st[k])
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / args.steps)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mc.scst_step(ctx, reward, num_samples=K, seed=next(seeds))
        parts["whole"].append((time.perf_counter() - t0) * 1e3)
        for k, v in scst_parts().items():
            parts[k].append(v)
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    out = {"metric": "scst_cost", "gpu": card, "shape": dict(n_img=n, samples=K, L=L, D=D, H=H, V=V, T=T), "dropout": True,
           "steps": args.steps, "rounds": args.rounds, "fwd_bwd_ms": med,
           "grouped_vs_replicated_pct": 100.0 * (med["grouped_64x5"] / med["xe_320_replicated"] - 1.0),
           "scst_step_ms": {k: sorted(v)[len(v) // 2] for k, v in parts.items()},
           "train_state_mib": {"xe_64": round(mem_a, 1), "xe_320_replicated": round(mem_b, 1), "grouped_64x5": round(mem_c, 1)},
           "fwd_bwd_ms_rounds": ms}
    if not args.no_profile:   # one eager call each (fresh sentence buffers: a new graph key runs eagerly first)
        s2, s3 = sent.clone(), sent.clone()
        out["kernels_ms"] = {
            "xe_320_replicated": kernel_table(lambda: mb.train_forward_backward(ctx_rep, s2, masks, seed=7)),
            "grouped_64x5": kernel_table(lambda: mc.train_forward_backward(ctx, s3, masks, seed=7, group=K, row_weights=rw)),
        }
    for m, _ in legs.values():
        m.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
