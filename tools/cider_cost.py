"""Cost of CIDEr-D on the device (sat_cider_create / sat_cider_d) and of the self-critical step with it, on an H100.

    python tools/cider_cost.py [--launches 200] [--rounds 5] [--images 113287]

Corpus: a synthetic COCO-sized training set, `images` x 5 references of 8-16 words and eos (T_ref = 20), the words drawn
from a Zipf-like law over V = 10000 (p(w) ~ 1 / (w + 10)).  Batch: the workload-2 shape of bench.py (L=196, D=512,
H=1024, V=10000, T=20), 64 images x (5 samples + 1 greedy) candidates x 5 references.  Reports:
  create_s            sat_cider_create on the corpus (host build of the document-frequency table + upload), wall clock;
  kernel_us           sat_cider_d at 64 x 6 x 5, CUDA events over `launches` back-to-back launches (queued behind a
                      sleep kernel, so launch overhead is hidden);
  host_scorer_ms      the fp64 Python reference scorer of tests/cider_ref.py on the same inputs, on the CPU of the GPU
                      host (reference vectors recomputed per candidate; document frequencies looked up in a sorted
                      numpy table);
  scst_step_ms        a whole CaptionGenerator.scst_step (64 images x 5 samples, greedy baseline, dropout on) with the
                      CiderD reward ("device") and with a host reward_fn computing the same CIDEr-D with that scorer
                      ("host"), alternated, median of `rounds`.
Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import WORKLOADS  # noqa: E402


def synthetic_refs(rng, n, R, T_ref, V, eos):
    import numpy as np
    p = 1.0 / (np.arange(V) + 10.0)
    p[[0, eos]] = 0.0
    p /= p.sum()
    words = rng.choice(V, size=(n, R, T_ref), p=p).astype(np.int32)
    lens = rng.integers(8, 17, size=(n, R))
    pos = np.arange(T_ref)[None, None, :]
    words[pos == lens[..., None]] = eos
    words[pos > lens[..., None]] = -1
    return words


def pack(words):
    """n-gram keys of the device table: four 16-bit fields of (word + 1), the first word on top"""
    k = 0
    for m, w in enumerate(words):
        k |= (int(w) + 1) << (48 - 16 * m)
    return k


def doc_freq_table(corpus, eos):
    """(sorted keys, df) of a corpus [n, R, T_ref] whose rows are `words, eos, -1 ...` (numpy, for the host scorer)"""
    import numpy as np
    n, R, T = corpus.shape
    w = corpus.astype(np.uint64) + np.uint64(1)
    valid = corpus >= 0                                   # (every row ends with eos, then padding)
    img = np.broadcast_to(np.arange(n)[:, None, None], corpus.shape)
    keys, imgs = [], []
    for g in range(1, 5):
        k = np.zeros((n, R, T - g + 1), np.uint64)
        ok = np.ones((n, R, T - g + 1), bool)
        for m in range(g):
            k |= w[:, :, m:T - g + 1 + m] << np.uint64(48 - 16 * m)
            ok &= valid[:, :, m:T - g + 1 + m]
        keys.append(k[ok])
        imgs.append(img[:, :, :T - g + 1][ok])
    keys, imgs = np.concatenate(keys), np.concatenate(imgs)
    order = np.lexsort((imgs, keys))
    keys, imgs = keys[order], imgs[order]
    first = np.ones(keys.size, bool)
    first[1:] = (keys[1:] != keys[:-1]) | (imgs[1:] != imgs[:-1])
    return np.unique(keys[first], return_counts=True)


class PackedDF(object):
    """df.get(ngram tuple, 0) over the sorted numpy table (what cider_ref.vec asks of a df mapping)"""

    def __init__(self, keys, counts):
        self.keys, self.counts = keys, counts

    def get(self, g, default=0):
        import numpy as np
        k = np.uint64(pack(g))
        i = int(np.searchsorted(self.keys, k))
        return int(self.counts[i]) if i < self.keys.size and self.keys[i] == k else default


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--images", type=int, default=113287)
    args = ap.parse_args()
    import numpy as np
    import torch
    import sat_b200
    import cider_ref as CR
    if not torch.cuda.is_available():
        raise SystemExit("cider_cost.py needs an H100: no CUDA device visible")
    torch.cuda.set_device(0)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:   # (the numbers are still reported; the card is then unnamed)
        card = "unknown (%s)" % e
    wl = WORKLOADS[2]
    n, L, D, H, V, T = (wl[k] for k in "BLDHVT")
    K, R, T_ref, eos = 5, 5, 20, 2
    rng = np.random.default_rng(0)
    corpus = synthetic_refs(rng, args.images, R, T_ref, V, eos)
    refs = corpus[:n]
    cand = synthetic_refs(rng, n, K + 1, T, V, eos)

    t0 = time.perf_counter()
    cider = sat_b200.CiderD(corpus, eos, V)
    create_s = time.perf_counter() - t0

    c_d, r_d = torch.from_numpy(cand).cuda(), torch.from_numpy(refs).cuda()
    out = torch.empty(n, K + 1, device="cuda")
    lib, p = cider.lib, (lambda t: C.c_void_p(t.data_ptr()))
    st = torch.cuda.current_stream()
    launch = lambda: lib.sat_cider_d(cider._c, p(c_d), n, K + 1, T, p(r_d), R, T_ref, p(out),
                                     C.c_void_p(st.cuda_stream))
    for _ in range(10):
        assert launch() == 0
    torch.cuda.synchronize()
    kern = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(50_000_000)
        e0.record()
        for _ in range(args.launches):
            launch()
        e1.record()
        torch.cuda.synchronize()
        kern.append(e0.elapsed_time(e1) * 1e3 / args.launches)
    dev_scores = out.cpu().numpy()

    t0 = time.perf_counter()
    keys, counts = doc_freq_table(corpus, eos)
    df_table_s = time.perf_counter() - t0
    df, N = PackedDF(keys, counts), args.images
    host = []
    for _ in range(3):
        t0 = time.perf_counter()
        ref_scores = np.array(CR.scores(cand, refs, df, N, eos, V))
        host.append((time.perf_counter() - t0) * 1e3)
    max_err = float(np.abs(dev_scores - ref_scores).max())

    cfg = sat_b200.Config(batch_size=n, num_ctx=L, dim_ctx=D, num_lstm_units=H, vocabulary_size=V, max_caption_length=T)
    m = sat_b200.CaptionGenerator(cfg, max_batch=n * 4)
    m.train_setup(n, T, group=K)
    g = torch.Generator(device="cpu").manual_seed(1234)
    ctx = torch.relu(torch.randn(n, L, D, generator=g)).cuda()
    img_refs = [CR.image_refs(refs[i], eos, V) for i in range(n)]

    def host_reward(caps):
        return np.array([[CR.cider_d(CR.cut(c, eos, V), img_refs[i], df, N) for c in img] for i, img in enumerate(caps)])
    legs = {"device": lambda: m.scst_step(ctx, cider, num_samples=K, references=r_d),
            "host": lambda: m.scst_step(ctx, host_reward, num_samples=K)}
    for f in legs.values():
        for _ in range(2):
            f()
    ms = {k: [] for k in legs}
    for _ in range(args.rounds):
        for k, f in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1e3)
    med = lambda v: sorted(v)[len(v) // 2]
    res = {"metric": "cider_cost", "gpu": card,
           "shape": dict(n_img=n, candidates=K + 1, refs=R, T=T, T_ref=T_ref, V=V, corpus_images=args.images),
           "table_distinct_ngrams": int(keys.size), "create_s": round(create_s, 3),
           "kernel_us": round(med(kern), 2), "kernel_us_rounds": [round(x, 2) for x in kern],
           "host_scorer_ms_gpu_host_cpu": round(med(host), 1), "host_df_table_s": round(df_table_s, 2),
           "max_abs_diff_vs_host_scorer": max_err,
           "scst_step_ms": {k: round(med(v), 2) for k, v in ms.items()}, "scst_step_ms_rounds": ms}
    m.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
