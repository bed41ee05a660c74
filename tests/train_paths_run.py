"""Calls of the training step for tests/test_gpu_train_paths.py, and the child process that runs them under a
SAT_TRAIN_* environment switch (the switches are read once per process).

    python train_paths_run.py OUT.npz     runs SWITCH_SHAPES, each eager under the profiler and then replayed from its
                                          captured graph, and writes losses, gradients and kernel records to OUT.npz.
The library must already be built: the child only loads it."""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)

from test_gpu_train import TC_DIMS, TDIMS  # noqa: E402

MARKERS = 32   # marker kernels before and after a profiled call
SWITCH_SEED = 31
# (name, dims, n_img, G): the shapes every switch setting runs (grouped ones with row weights)
SWITCH_SHAPES = [("tdims_b4", TDIMS, 4, 1), ("tc_b16", TC_DIMS, 16, 1), ("tc_4x5", TC_DIMS, 4, 5)]


def gpu_setup(dims, n_img, G, seed=3):
    """(ocfg, w, m, host inputs, device inputs) of a step on n_img images x G rows: gsetup's data, with row weights
    for G > 1, and a device mask sum."""
    import torch
    from test_gpu_scst import gsetup
    ocfg, w, m, ctx, sent, masks, rw = gsetup(n_img, G, seed=seed, dims=dims)
    rw = rw if G > 1 else None
    host = dict(ctx=ctx, sent=sent, masks=masks, rw=rw)
    dev = dict(ctx=torch.from_numpy(ctx).cuda(), sent=torch.from_numpy(sent).cuda(), masks=torch.from_numpy(masks).cuda(),
               rw=None if rw is None else torch.from_numpy(rw).cuda(),
               gsum=torch.tensor([float(masks.astype(np.float64).sum())], dtype=torch.float64, device="cuda"))
    torch.cuda.synchronize()
    return ocfg, w, m, host, dev


def step(m, dev, seed, sent=None):
    """One call of the step through the library's entry point (no torch kernels of its own): _dsum for one row per
    image without weights, _grouped otherwise.  Returns the status."""
    n_img, G = m._train_group
    B, T = m._train_BT
    s = dev["sent"] if sent is None else sent
    P = m._p
    if G == 1 and dev["rw"] is None:
        return m.lib.sat_train_forward_backward_dsum(m._h, P(m.params), P(m.grads), P(dev["ctx"]), P(s), P(dev["masks"]), B, T,
                                                     int(seed), P(dev["gsum"]), B, P(m._train_losses), m._st())
    return m.lib.sat_train_forward_backward_grouped(m._h, P(m.params), P(m.grads), P(dev["ctx"]), n_img, G, P(s), P(dev["masks"]),
                                                    P(dev["rw"]), T, int(seed), P(dev["gsum"]), B, P(m._train_losses), m._st())


def results(m):
    """(losses [4], {variable: gradient}) of the last step, as numpy."""
    m.stream.synchronize()
    return (m._train_losses.cpu().numpy().copy(),
            {k: v.detach().cpu().numpy().copy() for k, v in m.train_state_dict("grads").items()})


def kernel_records(prof):
    """(name, grid (x, y, z) or None) of every kernel of a profile, in start order."""
    import json
    import tempfile
    import torch
    fd, path = tempfile.mkstemp(suffix=".json")
    os.close(fd)
    try:
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    finally:
        os.unlink(path)
    ks = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0))
    out = [(e.get("name", ""), tuple(e["args"]["grid"]) if e.get("args", {}).get("grid") else None) for e in ks]
    if out:
        return out
    return [(e.name, None) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def eager_profiled(m, dev, seed):
    """One eager call under the profiler: (kernel records without the markers, losses, gradients).

    A capture can lose the records of the kernels at either end of its window (tests/test_gpu_decode_layers.py,
    captured()): the call runs between two runs of marker kernels on its stream, and a capture that lacks a marker
    before the call's first kernel or after its last is repeated after a growing pause.  Every attempt passes a fresh
    copy of the sentences (a new graph key), so every attempt runs eagerly."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    def markers():
        with torch.cuda.stream(m.stream):
            for _ in range(MARKERS):
                torch.cuda._sleep(1000)
    for pause in (0, 0.05, 0.2, 0.5, 1.0):
        time.sleep(pause)
        sent = dev["sent"].clone()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            markers()
            rc = step(m, dev, seed, sent)
            torch.cuda.synchronize()
            markers()
            torch.cuda.synchronize()
        assert rc == 0, m.lib.sat_last_error()
        rec = kernel_records(prof)
        mk = [i for i, (n, _) in enumerate(rec) if "spin_kernel" in n]
        work = [i for i, (n, _) in enumerate(rec) if "spin_kernel" not in n]
        if work and mk and mk[0] < work[0] and mk[-1] > work[-1]:
            break
    losses, grads = results(m)
    return [r for r in rec if "spin_kernel" not in r[0]], losses, grads


def eager_captured_replayed(m, dev, seed):
    """Three calls on the same buffers (eager, captured + launched, replayed): [(losses, gradients)] of each."""
    out = []
    for _ in range(3):
        assert step(m, dev, seed) == 0, m.lib.sat_last_error()
        out.append(results(m))
    return out


def main(path):
    import torch
    torch.cuda.set_device(0)
    save = {}
    for name, dims, n_img, G in SWITCH_SHAPES:
        ocfg, w, m, host, dev = gpu_setup(dims, n_img, G)
        rec, losses, grads = eager_profiled(m, dev, SWITCH_SEED)
        save[name + "/kernels"] = np.array([n for n, _ in rec])
        save[name + "/grids"] = np.array([g if g is not None else (-1, -1, -1) for _, g in rec], np.int64).reshape(-1, 3)
        runs = [(losses, grads)] + eager_captured_replayed(m, dev, SWITCH_SEED)[1:]
        for tag, (l, g) in zip(("eager", "captured", "replayed"), runs):
            save["%s/%s/losses" % (name, tag)] = l
            for k, v in g.items():
                save["%s/%s/grad/%s" % (name, tag, k)] = v
        m.close()
    np.savez(path, **save)


if __name__ == "__main__":
    main(sys.argv[1])
