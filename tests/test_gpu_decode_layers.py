"""The decode step's dense layers on lin_mma_kernel (csrc/sat_linear.cu), called as the decode step calls them, against
fp64: the LSTM layer (sat_lstm_fwd), the decode layers (sat_vocab_gemm), and the vocabulary layer's word choice and
word probabilities inside the decode loop (sat_decode_loop_maps: the fused arg-max of lin_mma_kernel, or the per-row
kernel of csrc/sat_rows.cu when the layer does not fit one wave or the decode has one layer).

References: oracle.ref_step.lstm_cell on concat(context, emb[last_word]) and h_prev, oracle.ref_step.decode on
concat(h, context, emb[last_word]) and oracle.ref_step.decode_loop, all in float64.  Each case identifies the
launches it ran (kernel instance and grid) from the CUDA activity of torch.profiler and fails if it cannot.

Comparison.  The kernel's product is Whi*Xhi + Wlo*Xhi + Whi*Xlo with W and X split into bf16 hi + lo, summed in fp32
(`split_product` restates it in fp64).  Its rounding error grows with the magnitude of the terms, so each error is
relative to the terms of the element:
  * dense outputs: |y - ref| / max(1, sum_k |x_k w_kn| + |b_n|); through two layers (decode fc_1 -> tanh -> fc_2) the
    first layer's scale is carried through tanh' and |fc_2| (`vocab_reference`);
  * LSTM c and h: |y - ref| / (max(1, largest gate scale of the unit) * max(1, |c_prev|)), the gate scale being the
    dense scale of the gate's pre-activation (+1 for the forget bias);
  * loop logits: as the decode layers, against the oracle's loop fed the same words (the error of the attention and
    LSTM layers before them is inside LOOP_BAR, not in the scale);
  * word probabilities: |p - ref| / ref, ref = the fp64 softmax of the logits the same launch returned.
A NaN anywhere (every output is prefilled with NaN, tokens with -1) fails.  Word choices have no tolerance: a token
is the first index of the maximum of the logits the same launch returned, and engineered exact ties (two vocabulary
columns of zero weights and the same bias) must go to the smaller index.

Worst normalised errors over the module on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit):
    LSTM epilogue, lin_mma_kernel<NT,false,false> for NT = 1..8, split factor 1   c 1.15e-6   h 6.3e-7
    LSTM epilogue, split factors 2, 4 and 8                                       c 5.8e-7    h 4.1e-7
    decode fc_1 -> tanh -> fc_2 (sat_vocab_gemm, NT = 1, 7, 8)                    7.4e-7
    decode/fc on the three-segment concat (NT = 1, 7, 8)                          3.9e-6
    loop logits against the oracle: fused arg-max path 6.1e-7, per-row kernel path 2.3e-6
    word probabilities: fused arg-max path 3.3e-7, per-row kernel path 2.9e-7
Bars: LSTM_BAR = 1e-5, DENSE_BAR = 3e-5, LOOP_BAR = 2e-5 and PROB_BAR = 3e-6, about 8x the worst of each.  The
module's GPU cases take ~10 s there; two runs gave the same figures.
"""
import json
import math
import os
import re
import tempfile
import time

import numpy as np
import pytest

from _util import TOL, make_pair, rel_err
from oracle import ref_step as R

LSTM_BAR = 1e-5
DENSE_BAR = 3e-5
LOOP_BAR = 2e-5
PROB_BAR = 3e-6

pytestmark = pytest.mark.gpu


# ============================================================================================ reference and comparator
def bf16_rne(x):
    """float32 -> the nearest bfloat16 (ties to even), as float32 (__float2bfloat16_rn)."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def split_bf16(x):
    """(hi, lo) in float64: hi = bf16(x), lo = bf16(x - hi) (x - hi is exact in fp32), as split_bf16x8 packs them."""
    x = np.asarray(x, np.float32)
    hi = bf16_rne(x)
    return hi.astype(np.float64), bf16_rne(x - hi).astype(np.float64)


def split_product(x, w):
    """fp64 value of the kernel's split-precision product x @ w = Whi*Xhi + Wlo*Xhi + Whi*Xlo."""
    xh, xl = split_bf16(x)
    wh, wl = split_bf16(w)
    return xh @ wh + xh @ wl + xl @ wh


def bf16_product(x, w):
    """x @ w with both operands rounded to bf16 (the lo terms dropped): a kernel that lost its split precision."""
    return split_bf16(x)[0] @ split_bf16(w)[0]


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def lstm_inputs(w, ctx, last_word, h_prev):
    emb = w["word_embedding/weights"].astype(np.float64)
    x = np.concatenate([np.asarray(ctx, np.float64), emb[np.asarray(last_word)]], 1)
    return x, np.concatenate([x, np.asarray(h_prev, np.float64)], 1)


def lstm_reference(cfg, w, ctx, last_word, c_prev, h_prev):
    """fp64 c, h [rows, H] of oracle.ref_step.lstm_cell and the error scale of every (row, unit)."""
    H = cfg.num_lstm_units
    x, xin = lstm_inputs(w, ctx, last_word, h_prev)
    cp = np.asarray(c_prev, np.float64)
    c, h = R.lstm_cell(cfg, w, x, cp, np.asarray(h_prev, np.float64))
    S = np.abs(xin) @ np.abs(w["lstm/lstm_cell/kernel"].astype(np.float64)) + \
        np.abs(w["lstm/lstm_cell/bias"].astype(np.float64))
    S[:, 2 * H:3 * H] += 1.0                                   # forget bias
    scale = np.maximum(1.0, S.reshape(-1, 4, H).max(1)) * np.maximum(1.0, np.abs(cp))
    return dict(c=c, h=h, scale=scale)


def lstm_emulated(cfg, w, ctx, last_word, c_prev, h_prev, product=split_product, order=(0, 1, 2, 3),
                  forget_bias=1.0, unit_shift=0):
    """An LSTM layer computed the kernel's way (product = split_product), or with one of the faults the comparator
    must catch: another product, gates read in another order (i, j, f, o positions), another forget bias, or the
    gates of unit u + unit_shift (an interleave p = unit * 4 + gate off by whole units)."""
    H = cfg.num_lstm_units
    _, xin = lstm_inputs(w, ctx, last_word, h_prev)
    g = product(xin, w["lstm/lstm_cell/kernel"]) + w["lstm/lstm_cell/bias"].astype(np.float64)
    g = g.reshape(-1, 4, H)
    g = np.roll(g, -unit_shift, axis=2)
    i, j, f, o = (g[:, k] for k in order)
    c = _sigmoid(f + forget_bias) * np.asarray(c_prev, np.float64) + _sigmoid(i) * np.tanh(j)
    return c, _sigmoid(o) * np.tanh(c)


def lstm_errors(c, h, ref):
    """(c error, h error) normalised as in the module docstring; inf for a NaN."""
    out = []
    for got, name in ((c, "c"), (h, "h")):
        g = np.asarray(got, np.float64)
        out.append(math.inf if not np.isfinite(g).all() else float((np.abs(g - ref[name]) / ref["scale"]).max()))
    return tuple(out)


def decode_input(w, h, ctx, last_word):
    emb = w["word_embedding/weights"].astype(np.float64)
    return np.concatenate([np.asarray(h, np.float64), np.asarray(ctx, np.float64), emb[np.asarray(last_word)]], 1)


def vocab_scale(cfg, w, x):
    """Error scale of every logit of decode(x): the dense scale of the last layer, plus (2 layers) the first layer's
    scale carried through tanh' and |fc_2|."""
    if cfg.num_decode_layers == 1:
        return np.abs(x) @ np.abs(w["decode/fc/kernel"].astype(np.float64)) + np.abs(w["decode/fc/bias"].astype(np.float64))
    w1, b1 = w["decode/fc_1/kernel"].astype(np.float64), w["decode/fc_1/bias"].astype(np.float64)
    w2, b2 = np.abs(w["decode/fc_2/kernel"].astype(np.float64)), np.abs(w["decode/fc_2/bias"].astype(np.float64))
    t = np.tanh(x @ w1 + b1)
    s1 = np.maximum(1.0, np.abs(x) @ np.abs(w1) + np.abs(b1))
    return np.abs(t) @ w2 + b2 + (s1 * (1.0 - t * t)) @ w2


def vocab_reference(cfg, w, h, ctx, last_word):
    """fp64 logits [rows, V] of oracle.ref_step.decode and their error scale."""
    x = decode_input(w, h, ctx, last_word)
    return dict(logits=R.decode(cfg, w, x), scale=vocab_scale(cfg, w, x))


def vocab_emulated(cfg, w, h, ctx, last_word, product=split_product):
    """decode() computed the kernel's way: the fc_1 output is stored in fp32 between the two launches."""
    x = decode_input(w, h, ctx, last_word).astype(np.float32)
    if cfg.num_decode_layers == 1:
        return product(x, w["decode/fc/kernel"]) + w["decode/fc/bias"]
    t = np.tanh(product(x, w["decode/fc_1/kernel"]) + w["decode/fc_1/bias"]).astype(np.float32)
    return product(t, w["decode/fc_2/kernel"]) + w["decode/fc_2/bias"]


def dense_error(y, ref, scale):
    y = np.asarray(y, np.float64)
    return math.inf if not np.isfinite(y).all() else float((np.abs(y - ref) / np.maximum(1.0, scale)).max())


def token_mismatches(tokens, logits):
    """(row, step) pairs whose token is not the first index of the maximum of that step's logits [T, B, V]."""
    return [tuple(x) for x in np.argwhere(np.asarray(tokens) != np.argmax(logits, -1).T)]


def softmax64(logits):
    l = np.asarray(logits, np.float64)
    e = np.exp(l - l.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def word_prob_error(word_probs, logits, fed):
    """max relative error of word_probs [B, T] against the fp64 softmax of the returned logits [T, B, V] at the
    words fed [B, T]."""
    p = np.asarray(word_probs, np.float64)
    if not np.isfinite(p).all():
        return math.inf
    sm = softmax64(logits)
    B, T = p.shape
    ref = sm[np.arange(T)[None, :], np.arange(B)[:, None], fed]
    return float((np.abs(p - ref) / ref).max())


# worst error per (kernel instance, what) over the module's cases, printed at the end (pytest -s)
WORST = {}


def note(key, err, what=""):
    WORST[key] = max(WORST.get(key, 0.0), err)
    print("%-48s %-40s %.3e" % (key, what, err))


# ========================================================================================== plan and kernels restated
def row_tile_for(rows):
    """Row tile of a launch (sat_api.cu row_tile_for): rows split evenly into tiles of at most 128, rounded to 16."""
    nrt = -(-rows // 128)
    per = -(-rows // nrt)
    return -(-per // 16) * 16


def plan(K, n_out, rows, sms, force_splits=0, group=1):
    """The grid plan() chooses: split-K factor from its cost model (K blocks + ~4 per CTA, +1 for a split)."""
    kb, nt, rt = -(-K // 64), -(-n_out // 128), row_tile_for(rows)
    nrt = -(-rows // rt)
    tiles, budget = nt * nrt, sms // group
    best = 1
    if force_splits > 0:
        while best * 2 <= force_splits and best * 2 <= 8 and best * 2 <= kb:
            best *= 2
    else:
        bc = 1e30
        s = 1
        while s <= 8 and s <= kb:
            c = -(-tiles * s // budget) * (-(-kb // s) + 4.0) + (1.0 if s > 1 else 0.0)
            if c < bc - 1e-9:
                bc, best = c, s
            s *= 2
    return dict(kb=kb, n_tiles=nt, row_tile=rt, n_row_tiles=nrt, splits=best, grid=tiles * best)


def x_mode(p, sms, xpack=1):
    """How an unpacked operand reaches the MMAs: 1 = cooperative pre-pass (one wave, no split), 0 = producer warps."""
    return 1 if xpack and p["splits"] == 1 and p["grid"] <= sms else 0


def lin(rows, wp=False):
    return "lin_mma_kernel<%d,%s,false>" % (row_tile_for(rows) // 16, "true" if wp else "false")


def lstm_plan(cfg, rows, sms):
    H = cfg.num_lstm_units
    return plan(cfg.dim_ctx + cfg.dim_embedding + H, 4 * H, rows, sms)


def vocab_plans(cfg, rows, sms):
    """[(what, plan)] of sat_vocab_gemm's launches: decode fc_1 (tanh) then fc_2, or decode/fc."""
    K = cfg.num_lstm_units + cfg.dim_ctx + cfg.dim_embedding
    if cfg.num_decode_layers == 1:
        return [("decode/fc", plan(K, cfg.vocabulary_size, rows, sms))]
    return [("decode/fc_1", plan(K, cfg.dim_decode_layer, rows, sms)),
            ("decode/fc_2", plan(cfg.dim_decode_layer, cfg.vocabulary_size, rows, sms))]


def fused_argmax(cfg, B, sms):
    """The loop picks words inside the vocabulary layer (2-layer decode, one wave of un-split CTAs); otherwise the
    per-row kernel does."""
    p = plan(cfg.dim_decode_layer, cfg.vocabulary_size, B, sms, force_splits=1)
    return cfg.num_decode_layers == 2 and p["grid"] <= sms


_KERNELS = [re.compile(r"(lin_mma_kernel)<(\d+),(true|false),(true|false)>"),
            re.compile(r"(rows_softmax_kernel)<(true|false),(true|false)>"),
            re.compile(r"(lin_mma_kernel)ILi(\d+)ELb([01])ELb([01])EE"),       # mangled
            re.compile(r"(rows_softmax_kernel)ILb([01])ELb([01])EE")]
_BOOL = {"0": "false", "1": "true"}


def instance(name):
    """'lin_mma_kernel<4,false,false>' / 'rows_softmax_kernel<true,false>' for a (de)mangled kernel name, else None."""
    n = name.replace(" ", "")
    for rx in _KERNELS:
        m = rx.search(n)
        if m:
            args = list(m.groups()[1:])
            first = 1 if m.group(1) == "lin_mma_kernel" else 0     # (NT is a number, the rest are bools)
            return "%s<%s>" % (m.group(1), ",".join(args[:first] + [_BOOL.get(a, a) for a in args[first:]]))
    return None


class Capture(list):
    """[(instance, grid)] of the dense-layer and per-row kernels of one call, in launch order (grid: CTAs, or None
    when the profiler did not record it), with every GPU activity name of the capture (for failure messages)."""
    def __init__(self, records):
        records = list(records)
        super().__init__((instance(n), g) for n, g in records if instance(n))
        self.names = sorted({n for n, _ in records})

    def where(self, prefix):
        return [x for x in self if x[0].startswith(prefix)]


def _kernel_records(prof):
    """(name, CTAs) of every kernel of a capture.  The grid comes from the trace's kernel events; without them, the
    names of the profiler's CUDA events and no grid."""
    import torch
    fd, path = tempfile.mkstemp(suffix=".json")
    os.close(fd)
    try:
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    finally:
        os.unlink(path)
    ks = [e for e in events if e.get("cat") == "kernel"]
    ks.sort(key=lambda e: e.get("ts", 0))
    out = []
    for e in ks:
        g = e.get("args", {}).get("grid")
        out.append((e.get("name", ""), int(np.prod(g)) if g else None))
    if out:
        return out
    return [(e.name, None) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def ran(cap, want):
    """The capture's launches are `want` [(instance, CTAs)] (a grid the profiler did not record is not compared)."""
    got = [(i, g) for i, g in cap]
    ok = len(got) == len(want) and all(gi == wi and (gg is None or gg == wg) for (gi, gg), (wi, wg) in zip(got, want))
    assert ok, "expected launches %s, captured %s; all GPU activities: %s" % (want, got, cap.names)
    return "%s grid %s" % (want[-1][0], "/".join(str(g) for _, g in got))


# ================================================================================================== GPU plumbing
_MODELS = {}
MARKERS = 32               # marker kernels before and after each captured call
INCOMPLETE_CAPTURES = []   # (markers seen, activity names) of captures that were repeated
GRIDS = {"recorded": 0, "missing": 0}


@pytest.fixture(scope="module", autouse=True)
def _module_report():
    t0 = time.time()
    yield
    for m in _MODELS.values():
        m[2].close()
    _MODELS.clear()
    if WORST:
        print("\nworst normalised errors (kernel instance / path, output):")
        for k in sorted(WORST):
            print("  %-60s %.3e" % (k, WORST[k]))
        print("launch grids recorded by the profiler: %(recorded)d, missing: %(missing)d" % GRIDS)
        print("calls repeated for an incomplete capture: %d %s" % (len(INCOMPLETE_CAPTURES), INCOMPLETE_CAPTURES[:5]))
        print("module time %.1f s" % (time.time() - t0))


def shared_model(key, rows=384, **dims):
    """(cfg, weights, model) cached per shape; a test that changes weights restores them."""
    if key not in _MODELS:
        d = dict(num_ctx=4, dim_ctx=64, dim_embedding=32, num_lstm_units=64, dim_initalize_layer=32,
                 dim_attend_layer=32, dim_decode_layer=64, vocabulary_size=300, max_caption_length=4)
        d.update(dims)
        cfg, w, m = make_pair(rows, max_batch=rows, **d)
        m.set_option("graphs", 0)   # every call enqueues its kernels (a replayed graph would hide them from a capture)
        _MODELS[key] = (cfg, w, m)
    return _MODELS[key]


LSTM_SHAPES = {   # model key -> dims (the decode layers are small: these models serve the LSTM cases)
    "small": dict(),                                                  # K = 160 (3 K blocks), 4H = 256 (2 tiles)
    "w2": dict(dim_ctx=512, dim_embedding=512, num_lstm_units=1024),  # workload 2: K = 2048 (32 blocks), 32 tiles
    "wide": dict(dim_ctx=2048, dim_embedding=64, num_lstm_units=64),  # K = 2176 (34 blocks), 2 tiles
    "h96": dict(num_lstm_units=96),                                   # 4H = 384: 3 tiles, H % 64 != 0
}


def lstm_model(key):
    return shared_model("lstm-" + key, **LSTM_SHAPES[key])


def num_sms():
    return lstm_model("small")[2].info("num_sms")


def captured(m, call, outputs):
    """Run call() (returns a status) under the profiler on outputs refilled with (tensor, fill value) first; returns
    (outputs as numpy, Capture).

    A capture can lose the records of the kernels at either end of its window: they arrive with the next capture, or
    not at all.  After other test modules had run in the same process, this emptied most captures of a single short
    launch (five times in a row, even with a 1 s host pause at both ends of the window) and cut steps off captures of
    decode loops.  So the call runs between two runs of MARKERS short marker kernels (torch.cuda._sleep) on its
    stream, and a capture that lacks a marker before the call's first kernel or after its last is repeated after a
    growing pause, at most five times.  The outputs of every attempt must be bit-identical."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    def markers():
        with torch.cuda.stream(m.stream):
            for _ in range(MARKERS):
                torch.cuda._sleep(1000)

    snaps = []
    for pause in (0, 0.05, 0.2, 0.5, 1.0):
        time.sleep(pause)
        for t, fill in outputs:
            t.fill_(fill)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            markers()
            rc = call()
            torch.cuda.synchronize()
            markers()
            torch.cuda.synchronize()
        assert rc == 0, m.lib.sat_last_error()
        records = _kernel_records(prof)
        cap = Capture(records)
        snaps.append([t.cpu().numpy() for t, _ in outputs])
        mk = [i for i, (n, _) in enumerate(records) if "spin_kernel" in n]
        work = [i for i, (n, _) in enumerate(records) if "spin_kernel" not in n]
        if work and mk and mk[0] < work[0] and mk[-1] > work[-1]:
            break
        INCOMPLETE_CAPTURES.append((len(mk), cap.names))
    for s in snaps[1:]:
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(s, snaps[0]))
    for _, g in cap:
        GRIDS["recorded" if g is not None else "missing"] += 1
    return snaps[-1], cap


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def lstm_gpu(m, ctx, last_word, c_prev, h_prev):
    """One sat_lstm_fwd call: (c, h, Capture)."""
    import torch
    rows, H = c_prev.shape
    x = [dev(ctx), dev(np.asarray(last_word, np.int32)), dev(c_prev), dev(h_prev)]
    mem, out = torch.empty(rows, H, device="cuda"), torch.empty(rows, H, device="cuda")
    (c, h), cap = captured(m, lambda: m.lib.sat_lstm_fwd(m._h, *[m._p(t) for t in x], m._p(mem), m._p(out), rows,
                                                         m._st()), [(mem, float("nan")), (out, float("nan"))])
    return c, h, cap


def lstm_inputs_random(cfg, rows, seed):
    rng = np.random.RandomState(seed)
    H = cfg.num_lstm_units
    ctx = np.maximum(rng.standard_normal((rows, cfg.dim_ctx)), 0).astype(np.float32)
    lw = rng.randint(0, cfg.vocabulary_size, rows).astype(np.int32)
    cp = rng.uniform(-2, 2, (rows, H)).astype(np.float32)
    hp = rng.uniform(-1, 1, (rows, H)).astype(np.float32)
    return ctx, lw, cp, hp


def run_lstm(key, rows, xpack=1, seed=0, inputs=None, what=""):
    cfg, w, m = lstm_model(key)
    sms = m.info("num_sms")
    p = lstm_plan(cfg, rows, sms)
    want = lin(rows)
    ctx, lw, cp, hp = inputs or lstm_inputs_random(cfg, rows, seed)
    m.set_option("xpack", xpack)
    try:
        c, h, cap = lstm_gpu(m, ctx, lw, cp, hp)
    finally:
        m.set_option("xpack", 1)
    desc = ran(cap, [(want, p["grid"])])
    ec, eh = lstm_errors(c, h, lstm_reference(cfg, w, ctx, lw, cp, hp))
    tag = "%s lstm x_mode %d splits %d" % (want, x_mode(p, sms, xpack), p["splits"])
    note(tag + " c", ec, "%s rows %d %s" % (key, rows, what))
    note(tag + " h", eh, desc)
    assert ec <= LSTM_BAR and eh <= LSTM_BAR, "%s rows %d: c %.3e h %.3e > %.1e" % (key, rows, ec, eh, LSTM_BAR)
    return c, h, p


# ======================================================================================== 1. the LSTM layer
ROWS_NT = [1, 17, 33, 49, 65, 81, 97, 113, 128, 129, 200, 384]   # NT = 1..8, then 2 and 3 row tiles


@pytest.mark.parametrize("rows", ROWS_NT)
def test_lstm_every_row_tile(rows):
    """K = 160 (3 K blocks, no split): both activation paths, which must agree bit for bit."""
    c1, h1, p = run_lstm("small", rows, xpack=1, seed=rows)
    assert p["splits"] == 1
    c0, h0, _ = run_lstm("small", rows, xpack=0, seed=rows)
    assert np.array_equal(c1, c0) and np.array_equal(h1, h0)


# (model, rows, split factor): rows > 16 per CTA (c_prev read directly after the two prefetched rows) with and
# without a split; fewer rows than CTAs of a cluster
SPLITS = [("w2", 1, 4), ("w2", 64, 4), ("w2", 128, 4), ("w2", 129, 2), ("w2", 200, 2), ("w2", 384, 1),
          ("wide", 1, 8), ("wide", 16, 8), ("wide", 100, 8), ("h96", 5, 1), ("h96", 130, 1)]


@pytest.mark.parametrize("key,rows,splits", SPLITS, ids=["%s-rows%d-splits%d" % s for s in SPLITS])
def test_lstm_split_plans(key, rows, splits):
    cfg = lstm_model(key)[0]
    assert lstm_plan(cfg, rows, num_sms())["splits"] == splits
    c1, h1, _ = run_lstm(key, rows, seed=100 + rows)
    if splits == 1:
        c0, h0, _ = run_lstm(key, rows, xpack=0, seed=100 + rows)
        assert np.array_equal(c1, c0) and np.array_equal(h1, h0)


def test_lstm_units_multiple_of_32():
    """A tile holds the 4 gates of 32 units, so no tile has padding units: the handle refuses other widths."""
    with pytest.raises(Exception, match="multiples of 32"):
        make_pair(4, num_ctx=4, dim_ctx=64, dim_embedding=32, num_lstm_units=40, dim_initalize_layer=32,
                  dim_attend_layer=32, dim_decode_layer=64, vocabulary_size=300)


def _set(m, w, names):
    assert m.set_weights({n: w[n] for n in names}) == 0


@pytest.mark.parametrize("rows", [49, 200])
def test_lstm_saturating_inputs(rows):
    """Gate pre-activations around +-20 (bias +-20) and c_prev = +-50: the fast sigmoid / tanh stay inside the bar."""
    cfg, w, m = lstm_model("small")
    keep = w["lstm/lstm_cell/bias"]
    rng = np.random.RandomState(7)
    try:
        w["lstm/lstm_cell/bias"] = (20.0 * rng.choice([-1.0, 1.0], keep.shape)).astype(np.float32)
        _set(m, w, ["lstm/lstm_cell/bias"])
        ctx, lw, cp, hp = lstm_inputs_random(cfg, rows, 8)
        cp = (50.0 * rng.choice([-1.0, 1.0], cp.shape)).astype(np.float32)
        for xpack in (1, 0):
            run_lstm("small", rows, xpack, inputs=(ctx, lw, cp, hp), what="saturating")
    finally:
        w["lstm/lstm_cell/bias"] = keep
        _set(m, w, ["lstm/lstm_cell/bias"])


@pytest.mark.parametrize("gate", [None, 0, 1, 2, 3])
def test_lstm_forget_bias_and_gate_order(gate):
    """Zero LSTM kernel: with zero bias c = sigmoid(1) * c_prev and h = 0.5 * tanh(c); then bias only on gate i, j, f
    or o (TF column gate * H + unit, a different value per unit), which moves c or h as that gate alone can."""
    cfg, w, m = lstm_model("small")
    H = cfg.num_lstm_units
    names = ["lstm/lstm_cell/kernel", "lstm/lstm_cell/bias"]
    keep = {n: w[n] for n in names}
    try:
        w[names[0]] = np.zeros_like(keep[names[0]])
        b = np.zeros_like(keep[names[1]])
        if gate is not None:
            b[gate * H:(gate + 1) * H] = np.linspace(-2.0, 2.5, H)
        w[names[1]] = b
        _set(m, w, names)
        rows = 33
        ctx, lw, cp, hp = lstm_inputs_random(cfg, rows, 9)
        c, h, _ = run_lstm("small", rows, inputs=(ctx, lw, cp, hp), what="bias on gate %s" % gate)
        if gate is None:
            c_cf = _sigmoid(1.0) * cp.astype(np.float64)
            ref = dict(c=c_cf, h=0.5 * np.tanh(c_cf), scale=np.maximum(1.0, np.abs(cp.astype(np.float64))))
            assert max(lstm_errors(c, h, ref)) <= LSTM_BAR
    finally:
        w.update(keep)
        _set(m, w, names)


# ======================================================================================== 2. the decode layers
VOCAB = [(layers, V) for layers in (2, 1) for V in (100, 300, 301, 5000, 10000)]


def vocab_model(layers, V):
    return shared_model("vocab-%d-%d" % (layers, V), num_decode_layers=layers, vocabulary_size=V)


@pytest.mark.parametrize("rows", [5, 200, 384])
@pytest.mark.parametrize("layers,V", VOCAB, ids=["%dlayer-V%d" % v for v in VOCAB])
def test_vocab_gemm(layers, V, rows):
    """sat_vocab_gemm: decode fc_1 (bias + tanh) then fc_2 (bias), or decode/fc on the three-segment concat
    (h, context, emb[last_word]); V < 128 (one partial tile), V % 4 != 0 (scalar stores), 1 to 3 row tiles."""
    import torch
    cfg, w, m = vocab_model(layers, V)
    sms = m.info("num_sms")
    rng = np.random.RandomState(rows + V)
    h = rng.uniform(-1, 1, (rows, cfg.num_lstm_units)).astype(np.float32)
    ctx = np.maximum(rng.standard_normal((rows, cfg.dim_ctx)), 0).astype(np.float32)
    lw = rng.randint(0, V, rows).astype(np.int32)
    x = [dev(h), dev(ctx), dev(lw)]
    logits = torch.empty(rows, V, device="cuda")
    (y,), cap = captured(m, lambda: m.lib.sat_vocab_gemm(m._h, *[m._p(t) for t in x], m._p(logits), rows, m._st()),
                         [(logits, float("nan"))])
    plans = vocab_plans(cfg, rows, sms)
    desc = ran(cap, [(lin(rows), p["grid"]) for _, p in plans])
    ref = vocab_reference(cfg, w, h, ctx, lw)
    e = dense_error(y, ref["logits"], ref["scale"])
    note("%s %s" % (lin(rows), "bias+tanh -> bias" if layers == 2 else "bias (3 segments)"), e,
         "V %d rows %d x_mode %s %s" % (V, rows, "/".join(str(x_mode(p, sms)) for _, p in plans), desc))
    assert e <= DENSE_BAR, "V %d rows %d: %.3e > %.1e" % (V, rows, e, DENSE_BAR)


# ======================================================================================== 3. words chosen in the loop
LOOP_DIMS = dict(num_ctx=9, dim_ctx=64, dim_embedding=64, num_lstm_units=64, dim_decode_layer=64)   # packed operands
T_LOOP = 2


def loop_model(layers, V, B):
    return shared_model("loop-%d-%d-%d" % (layers, V, B), rows=B, num_decode_layers=layers, vocabulary_size=V,
                        max_caption_length=T_LOOP, **LOOP_DIMS)


def loop_gpu(m, ctx_d, B, V, forced=None, wp=True):
    """sat_decode_loop_maps over T_LOOP steps: (tokens [B,T], logits [T,B,V], word_probs [B,T] or None, Capture)."""
    import torch
    T = T_LOOP
    tokens = torch.empty(B, T, dtype=torch.int32, device="cuda")
    logits = torch.empty(T, B, V, device="cuda")
    probs = torch.empty(B, T, device="cuda") if wp else None
    fw = None if forced is None else dev(np.asarray(forced, np.int32))
    outs = [(tokens, -1), (logits, float("nan"))] + ([(probs, float("nan"))] if wp else [])
    res, cap = captured(m, lambda: m.lib.sat_decode_loop_maps(m._h, m._p(ctx_d), B, T, m._p(fw), m._p(tokens),
                                                               m._p(logits), None, m._p(probs), m._st()), outs)
    return res[0], res[1], (res[2] if wp else None), cap


def check_path(cap, cfg, B, sms, wp):
    """Which kernel picked the words: 'fused' (no per-row kernel; the word-probability instance with wp) or 'rows'."""
    V = cfg.vocabulary_size
    rows = cap.where("rows_softmax_kernel")
    wp_inst = [x for x in cap.where("lin_mma_kernel") if ",true," in x[0]]
    if fused_argmax(cfg, B, sms):
        # (without word probabilities the vocabulary layer runs the plain instance: it is told apart by its grid)
        p = plan(cfg.dim_decode_layer, V, B, sms, force_splits=1)
        vocab = [x for x in cap if x[0] == lin(B, wp) and x[1] == p["grid"]]
        grids = all(g is not None for _, g in cap)
        assert not rows and (bool(wp_inst) == wp) and (not grids or len(vocab) == T_LOOP), \
            "expected the fused arg-max (%s x %d); captured %s; all: %s" % (lin(B, wp), T_LOOP, list(cap), cap.names)
        return "fused", lin(B, wp)
    want = "rows_softmax_kernel<%s,false>" % ("true" if V % 4 == 0 else "false")
    assert [x[0] for x in rows] == [want] * T_LOOP and not wp_inst and all(g in (None, B) for _, g in rows), \
        "expected %s x %d; captured %s; all: %s" % (want, T_LOOP, list(cap), cap.names)
    return "rows", want


def loop_oracle(cfg, w, ctx, fed):
    """fp64 logits [T, B, V] of the oracle's loop fed the words `fed` [B, T], and their error scales."""
    toks, steps = R.decode_loop(cfg, w, ctx, T_LOOP, fed, np.float64)
    emb = w["word_embedding/weights"].astype(np.float64)
    words = np.concatenate([np.zeros((ctx.shape[0], 1), np.int64), np.asarray(fed)[:, :-1]], 1)
    scales = [vocab_scale(cfg, w, np.concatenate([s["output"], s["context"], emb[words[:, t]]], 1))
              for t, s in enumerate(steps)]
    return np.stack([s["logits"] for s in steps]), np.stack(scales)


def run_loop(cfg, w, m, B, forced=None, wp=True, seed=0, what="", oracle=True):
    sms = m.info("num_sms")
    ctx = R.synth_contexts(cfg, B, seed=seed)
    tokens, logits, probs, cap = loop_gpu(m, dev(ctx), B, cfg.vocabulary_size, forced, wp)
    path, inst = check_path(cap, cfg, B, sms, wp)
    assert np.isfinite(logits).all()
    assert token_mismatches(tokens, logits) == [], what
    fed = tokens if forced is None else np.asarray(forced)
    key = "%s %s (%s)" % (path, inst, "word probs" if wp else "no word probs")
    if wp:
        e = word_prob_error(probs, logits, fed)
        note(key + " word prob", e, "%dlayer V %d B %d %s" % (cfg.num_decode_layers, cfg.vocabulary_size, B, what))
        assert e <= PROB_BAR, "%s: word probability error %.3e > %.1e" % (what, e, PROB_BAR)
    if oracle:
        ref, scale = loop_oracle(cfg, w, ctx, fed)
        e = dense_error(logits, ref, scale)
        note(key + " loop logits", e, what)
        assert e <= LOOP_BAR, "%s: logits error %.3e > %.1e" % (what, e, LOOP_BAR)
        if wp:
            sm = softmax64(ref)
            exp = sm[np.arange(T_LOOP)[None, :], np.arange(B)[:, None], fed]
            assert rel_err(probs, exp) <= TOL
    return tokens, logits, probs, path


# (decode layers, V, B, options): fused with packed operands, fused with pa = 0 (operands converted in the launch),
# a second row tile (rows 128.. have their own candidates in am_key), the per-row kernel (cached and uncached rows)
LOOPS = [(2, 300, 8, {}), (2, 300, 8, dict(pa=0)), (2, 5000, 200, {}), (2, 10000, 200, {}), (1, 301, 8, {})]
LOOP_IDS = ["%dlayer-V%d-B%d%s" % (l, v, b, "-pa0" if o else "") for l, v, b, o in LOOPS]


def with_options(m, opts, fn):
    for k, v in opts.items():
        m.set_option(k, v)
    try:
        return fn()
    finally:
        for k in opts:
            m.set_option(k, 1)


@pytest.mark.parametrize("layers,V,B,opts", LOOPS, ids=LOOP_IDS)
def test_loop_words_and_probabilities(layers, V, B, opts):
    """Greedy and teacher-forced, with and without word probabilities: every token is the first maximum of the logits
    the launch returned, every word probability the fp64 softmax of them, the logits match the oracle fed the same
    words.  Forced words include 0, 127, 128, the first word of the last tile and V - 1 (the forced word's logit is
    kept by the tile that owns it)."""
    cfg, w, m = loop_model(layers, V, B)
    last = (V - 1) // 128 * 128
    edges = np.array([0, 127, 128, last, V - 1])
    forced = np.random.RandomState(V + B).randint(0, V, (B, T_LOOP)).astype(np.int32)
    forced[:, 0] = edges[np.arange(B) % 5]
    forced[:, 1] = edges[(np.arange(B) + 2) % 5]
    for fw in (None, forced):
        for wp in (True, False):
            with_options(m, opts, lambda: run_loop(cfg, w, m, B, fw, wp, seed=B,
                                                   what="%s%s" % ("forced" if fw is not None else "greedy", opts or "")))


# tie placements (j1, j2) for a vocabulary of V words; the vocabulary layer's scan: 4 threads per row of a 128-word
# tile, each over 32 words as 8 float4 (x, y into one chain, z, w into the other)
def tie_pairs(V):
    last = (V - 1) // 128 * 128
    return [("float4", 4, 5), ("float4 chains", 5, 6), ("thread", 9, 17), ("shuffle", 10, 42),
            ("tiles", 11, 11 + 128 * min(8, last // 128)), ("0 and V-1", 0, V - 1), ("last tile", last, V - 1)]


@pytest.mark.parametrize("layers,V,B,opts", LOOPS, ids=LOOP_IDS)
def test_loop_exact_ties(layers, V, B, opts):
    """Vocabulary columns j1 < j2 with zero weights and the same bias +8 (every other logit is far below): both logits
    are exactly 8 in every row and step, and the word must be j1.  Their embedding rows are made very different, so
    the next step (checked against the oracle fed the chosen word) fails if the layer handed on j2's row."""
    cfg, w, m = loop_model(layers, V, B)
    kn, bn = ("decode/fc_2/kernel", "decode/fc_2/bias") if layers == 2 else ("decode/fc/kernel", "decode/fc/bias")
    en = "word_embedding/weights"
    keep = {n: w[n] for n in (kn, bn, en)}
    try:
        for what, j1, j2 in tie_pairs(V):
            w[kn], w[bn], w[en] = keep[kn].copy(), keep[bn].copy(), keep[en].copy()
            w[kn][:, [j1, j2]] = 0.0
            w[bn][[j1, j2]] = 8.0
            w[en][j1], w[en][j2] = 0.5, -0.5
            _set(m, w, [kn, bn, en])
            for wp in (True, False):
                tokens, logits, _, path = with_options(m, opts, lambda: run_loop(
                    cfg, w, m, B, None, wp, seed=3, what="tie %s (%d, %d)" % (what, j1, j2)))
                assert (logits[:, :, j1] == 8.0).all() and (logits[:, :, j2] == 8.0).all()
                assert (logits.max(-1) == 8.0).all()
                assert (tokens == j1).all(), "tie %s (%d, %d) on the %s path picked %s" % (
                    what, j1, j2, path, sorted(set(tokens.ravel().tolist())))
    finally:
        w.update(keep)
        _set(m, w, list(keep))


@pytest.mark.parametrize("layers,V,B,opts", LOOPS, ids=LOOP_IDS)
def test_loop_all_equal_logits(layers, V, B, opts):
    """Zero vocabulary kernel and bias: every logit is exactly 0, the word is 0 and its probability 1/V."""
    cfg, w, m = loop_model(layers, V, B)
    names = ["decode/fc_2/kernel", "decode/fc_2/bias"] if layers == 2 else ["decode/fc/kernel", "decode/fc/bias"]
    keep = {n: w[n] for n in names}
    try:
        for n in names:
            w[n] = np.zeros_like(keep[n])
        _set(m, w, names)
        tokens, logits, probs, _ = with_options(m, opts, lambda: run_loop(cfg, w, m, B, None, True, what="all equal",
                                                                          oracle=False))
        assert (logits == 0).all() and (tokens == 0).all()
        assert np.abs(probs.astype(np.float64) * V - 1.0).max() <= 4 * 2.0 ** -24
    finally:
        w.update(keep)
        _set(m, w, names)
