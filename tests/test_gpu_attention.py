"""The fused attention kernels (csrc/sat_attention.cu) called directly through sat_attention_fwd, against fp64.

Every kernel instance the library can launch (att_wpc_kernel<G>, att_fused_kernel<G, RV, OCC, NW>), every pass-2
branch of the fused kernel (vec2 / vec1 / scalar, chosen by D against NT = 32 * NW threads), the grid plans of
att_plan (k CTAs per image, one CTA per image, CTA row ranges across image boundaries, fewer rows than SMs, reduced
SM budgets) and the location counts where chunking and padding change are compared element by element with an fp64
restatement of the same operation:
    alpha = oracle.ref_step.attend(cfg, w, repeat(ctx, G), h, float64),   z = einsum("bl,bld->bd", alpha, ctx_rows)
Each case identifies the kernel it ran from the CUDA activity of torch.profiler and fails if it cannot.

Comparison (`errors`): the logits are dot products whose rounding error grows with the magnitude of their terms, so
both bars are relative to s = max(1, logit scale of the row), the largest sum of |terms| over the row's locations:
  * alpha: |a - ref| / (ref * s) per element; values whose reference is below 2^-122 (they underflow in fp32) only
    have to stay within 2^-122 of it;
  * z:     |z - ref| / (max|ctx| of the image * s) per element.
A NaN anywhere (the outputs are prefilled with NaN, so a row or location the kernel never writes) fails.

Worst normalised errors over the whole sweep on an H100 SXM 80 GB (132 SMs, 400 W power limit), per instance family
(the results are deterministic: two runs gave the same figures):
    att_wpc_kernel<1..4>            alpha 1.9e-6   z 5.9e-8
    att_fused_kernel<G, 4, 1, 8>    alpha 1.9e-6   z 8.0e-8
    att_fused_kernel<G, 0, 1, 8>    alpha 2.5e-6   z 6.2e-7
    att_fused_kernel<1, RV, 2, 8>   alpha 8.1e-7   z 4.2e-8
    att_fused_kernel<1, RV, 1, 16>  alpha 1.9e-6   z 7.0e-8
Bars: ALPHA_BAR = 2e-5 and Z_BAR = 5e-6, about 8x the worst of each.  The module's GPU cases take ~26 s there.
"""
import ctypes as C
import math
import os
import re
import time

import numpy as np
import pytest

from _util import TOL, make_pair, rel_err
from oracle import ref_step as R

ALPHA_BAR = 2e-5
Z_BAR = 5e-6
TINY = 2.0 ** -122      # alpha below this underflows (or loses its relative precision) in fp32

SMALL = dict(dim_embedding=32, num_lstm_units=64, dim_initalize_layer=32, dim_decode_layer=64, vocabulary_size=300,
             max_caption_length=6)
DEFAULT_OPTIONS = dict(att_wpc=1, att_occ=1, att_warps=8, att_sms=0, att_reuse_q=0)


# ============================================================================================ reference and comparator
def reference(cfg, w, ctx, h, G):
    """fp64 alpha [rows, L], z [rows, D], the logit scale of every row and max|ctx| of every row's image."""
    NI, L, D = ctx.shape
    ctx_rows = np.repeat(ctx.astype(np.float64), G, 0)
    h = np.asarray(h, np.float64)
    if cfg.num_attend_layers == 2:
        t1 = R._dense(ctx.astype(np.float64).reshape(NI * L, D), w, "attend/fc_1a", np.tanh)
        t1_rows = np.repeat(t1.reshape(NI, L, -1), G, 0).reshape(NI * G * L, -1)
        alpha = R.attend(cfg, w, ctx_rows, h, np.float64, None, t1_rows)
        q = R._dense(h, w, "attend/fc_1b", np.tanh)
        t = np.abs(t1_rows.reshape(NI * G, L, -1) + q[:, None, :])
        scale = (t @ np.abs(w["attend/fc_2/kernel"].astype(np.float64))).reshape(NI * G, L).max(1)
    else:
        alpha = R.attend(cfg, w, ctx_rows, h, np.float64)
        fa = np.abs(w["attend/fc_a/kernel"].astype(np.float64))
        fb = np.abs(w["attend/fc_b/kernel"].astype(np.float64))
        scale = ((np.abs(ctx_rows) @ fa)[..., 0] + np.abs(h) @ fb).max(1)
    z = np.einsum("bl,bld->bd", alpha, ctx_rows)
    cmax = np.repeat(np.abs(ctx).max(axis=(1, 2)).astype(np.float64), G)
    return dict(alpha=alpha, z=z, scale=scale, cmax=cmax)


def errors(alpha, z, ref):
    """(alpha error, z error) normalised as in the module docstring; inf for a NaN or an underflow outside the floor."""
    s = np.maximum(1.0, ref["scale"])[:, None]
    ea = 0.0
    if alpha is not None:
        a, ra = np.asarray(alpha, np.float64), ref["alpha"]
        d = np.abs(a - ra)
        small = ra < TINY
        if not np.isfinite(a).all() or (d[small] > TINY).any():
            ea = math.inf
        elif (~small).any():
            ea = float((d / (np.where(small, 1.0, ra) * s))[~small].max())
    zz = np.asarray(z, np.float64)
    ez = math.inf if not np.isfinite(zz).all() else float((np.abs(zz - ref["z"]) / (ref["cmax"][:, None] * s)).max())
    return ea, ez


# worst (alpha, z) error per kernel instance over the module's cases, printed at the end (pytest -s)
WORST = {}


def check(alpha, z, ref, kernel, what=""):
    ea, ez = errors(alpha, z, ref)
    w = WORST.setdefault(kernel, [0.0, 0.0])
    w[0], w[1] = max(w[0], ea), max(w[1], ez)
    print("%-34s %-44s alpha %.3e  z %.3e" % (kernel, what, ea, ez))
    assert ea <= ALPHA_BAR, "%s %s: alpha error %.3e > %.1e" % (kernel, what, ea, ALPHA_BAR)
    assert ez <= Z_BAR, "%s %s: z error %.3e > %.1e" % (kernel, what, ez, Z_BAR)


# ========================================================================================== plan and kernel restated
def plan_grid(NI, L, sms):
    """CTAs of att_plan's grid rule: one per SM (at most one per row), or k per image when that keeps >= 80 %."""
    grid = min(NI * L, sms)
    if NI <= sms:
        k = min(sms // NI, L)
        if k >= 1 and NI * k >= 0.8 * grid:
            grid = NI * k
    return grid


def cta_segments(NI, L, grid):
    """[(cta, image, first row, end row)] of every image segment of every CTA's row range."""
    NR, out = NI * L, []
    for c in range(grid):
        r, r_end = NR * c // grid, NR * (c + 1) // grid
        while r < r_end:
            img = r // L
            s1 = min(r_end, (img + 1) * L)
            out.append((c, img, r, s1))
            r = s1
    return out


def regime(NI, L, sms):
    """'cross': some CTA's rows span two images; 'whole': one CTA per image; 'split': k >= 2 CTAs per image."""
    grid = plan_grid(NI, L, sms)
    segs = cta_segments(NI, L, grid)
    if len(segs) > grid:
        return "cross"
    return "whole" if grid == NI else "split"


def expected_kernel(layers, D, A, G, att_wpc=1, att_occ=1, att_warps=8):
    """The instance att_plan / att_launch choose (RL = the width of the rows pass 1 streams)."""
    RL = A if layers == 2 else D
    occ2 = att_occ == 2 and G == 1
    if att_wpc and RL == 512 and D == 512 and not occ2:
        return "att_wpc_kernel<%d>" % G
    nw = 16 if (att_warps == 16 and G == 1 and not occ2) else 8
    return "att_fused_kernel<%d,%d,%d,%d>" % (G, 4 if RL == 512 else 0, 2 if occ2 else 1, nw)


def pass2_branch(D, nw):
    nt = 32 * nw
    return "vec2" if D % (2 * nt) == 0 else ("vec1" if D % nt == 0 else "scalar")


_DEMANGLED = re.compile(r"att_(?:fused|wpc)_kernel<[0-9,]+>")
_MANGLED = re.compile(r"att_(fused|wpc)_kernelI((?:Li\d+E)+)E")


def attention_kernels(names):
    """Names of the attention kernels among kernel names, as 'att_fused_kernel<1,4,1,8>'."""
    found = set()
    for name in names:
        name = name.replace("(int)", "").replace(" ", "")
        found.update(_DEMANGLED.findall(name))
        for kind, args in _MANGLED.findall(name):
            found.add("att_%s_kernel<%s>" % (kind, ",".join(re.findall(r"Li(\d+)E", args))))
    return found


class Kernels(set):
    """The attention kernels of one call, with every GPU activity name of its capture (for failure messages)."""
    def __init__(self, names):
        names = list(names)
        super().__init__(attention_kernels(names))
        self.names = sorted(set(names))


# ================================================================================================== GPU plumbing
_MODELS = {}
INCOMPLETE_CAPTURES = []   # activity names of captures without an attention kernel (the call was repeated)


@pytest.fixture(scope="module", autouse=True)
def _module_report():
    yield
    for m in _MODELS.values():
        m[2].close()
    _MODELS.clear()
    if WORST:
        print("\nworst normalised errors per kernel instance (alpha, z):")
        for k in sorted(WORST):
            print("  %-34s %.3e  %.3e" % (k, WORST[k][0], WORST[k][1]))
        print("calls repeated for a capture without an attention kernel: %d %s" % (len(INCOMPLETE_CAPTURES),
                                                                                   INCOMPLETE_CAPTURES))


def shared_model(layers, L, D, A, rows):
    """(cfg, weights, model) with the small H / E / V of this file; cached per shape, not to be modified."""
    key = (layers, L, D, A, rows)
    if key not in _MODELS:
        _MODELS[key] = own_model(layers, L, D, A, rows)
    return _MODELS[key]


def own_model(layers, L, D, A, rows, seed=1234):
    return make_pair(rows, max_batch=rows, seed=seed, num_ctx=L, dim_ctx=D, dim_attend_layer=A,
                     num_attend_layers=layers, **SMALL)


def set_options(m, **opts):
    for k, v in dict(DEFAULT_OPTIONS, **opts).items():
        m.set_option(k, v)


def inputs(cfg, NI, G, seed=0):
    """relu(N(0,1)) contexts [NI, L, D] and a different state h in (-1, 1) for every row."""
    ctx = R.synth_contexts(cfg, NI, seed=seed)
    h = np.random.RandomState(seed + 7).uniform(-1, 1, (NI * G, cfg.num_lstm_units)).astype(np.float32)
    return ctx, h


def attend_gpu(m, ctx, h, G, with_alpha=True, prepare=True):
    """One sat_attention_fwd call on NaN-prefilled outputs: (alpha or None, z, Kernels of the call).

    A capture can stop before the records of its last kernels are delivered (they then arrive with the next capture).
    So the capture ends with a marker kernel (torch.cuda._sleep's spin_kernel) launched on the call's stream after
    the call has completed.  A capture can also come back empty, occasionally a few in a row.  A capture that holds no
    attention kernel says nothing about which kernel ran: the call is made again after a growing pause, at most five
    times.  The outputs of every attempt must be bit-identical, so a call that launched nothing (NaN outputs) still
    fails."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    NI, L, D = ctx.shape
    ctx_d = torch.from_numpy(np.ascontiguousarray(ctx)).cuda() if isinstance(ctx, np.ndarray) else ctx
    h_d = torch.from_numpy(np.ascontiguousarray(h)).cuda() if isinstance(h, np.ndarray) else h
    torch.cuda.synchronize()
    if prepare:
        # the 2-layer projection is cached by contexts pointer and n_img: a reused address must be prepared again
        assert m.lib.sat_prepare_contexts(m._h, m._p(ctx_d), NI, None, None, m._st()) == 0, m.lib.sat_last_error()
        torch.cuda.synchronize()
    outs = []
    for pause in (0, 0.05, 0.2, 0.5, 1.0):
        time.sleep(pause)
        alpha = torch.full((NI * G, L), float("nan"), device="cuda") if with_alpha else None
        z = torch.full((NI * G, D), float("nan"), device="cuda")
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rc = m.lib.sat_attention_fwd(m._h, m._p(ctx_d), m._p(h_d), m._p(alpha), m._p(z), NI, G, m._st())
            torch.cuda.synchronize()
            with torch.cuda.stream(m.stream):
                torch.cuda._sleep(20000)
            torch.cuda.synchronize()
        assert rc == 0, m.lib.sat_last_error()
        ks = Kernels(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
        outs.append(((None if alpha is None else alpha.cpu().numpy()), z.cpu().numpy(), ks))
        if ks:
            break
        INCOMPLETE_CAPTURES.append(ks.names)
    for a, z, _ in outs[1:]:
        assert np.array_equal(z, outs[0][1]) and (a is None or np.array_equal(a, outs[0][0]))
    return outs[-1]


def ran(kernels, want):
    assert kernels == {want}, "expected %s to run; attention kernels seen: %s; all GPU activities of the capture: %s" % (
        want, sorted(kernels) or "none", kernels.names)


def run_case(layers, L, D, A, NI, G, opts=None, seed=0, fp32=False, what=""):
    """Shared model, random inputs, one call; checks the kernel and the errors."""
    opts = opts or {}
    cfg, w, m = shared_model(layers, L, D, A, NI * G)
    want = expected_kernel(layers, D, A, G, **{k: v for k, v in opts.items() if k != "att_sms"})
    ctx, h = inputs(cfg, NI, G, seed)
    set_options(m, **opts)
    try:
        alpha, z, ks = attend_gpu(m, ctx, h, G)
    finally:
        set_options(m)
    ref = reference(cfg, w, ctx, h, G)
    check(alpha, z, ref, want, what)
    ran(ks, want)
    if fp32:   # the fp32 oracle is well inside the project's max-norm bar of the fp64 truth, and so is the kernel
        a32 = R.attend(cfg, w, np.repeat(ctx, G, 0), h, np.float32)
        assert rel_err(a32, ref["alpha"]) < 1e-4
        assert rel_err(alpha, a32) <= TOL
    return want, alpha, z


def num_sms():
    return shared_model(2, 49, 64, 32, 4)[2].info("num_sms")


# ======================================================================================== every instance
# (instance, scorer layers, L, D, A, G, options)
INSTANCES = []
for _G, _L in ((1, 196), (2, 49), (3, 255), (4, 8)):
    INSTANCES += [("att_wpc_kernel<%d>" % _G, 2, _L, 512, 512, _G, {}),
                  ("att_wpc_kernel<%d>" % _G, 1, _L, 512, 512, _G, {})]
# RV = 4: rows of 512 floats in registers; D = A = 512 only with the warp-per-chunk kernel off; config-3 widths with G > 1
for _G, _L, _D in ((1, 196, 512), (2, 49, 256), (3, 9, 1024), (4, 7, 2048)):
    INSTANCES.append(("att_fused_kernel<%d,4,1,8>" % _G, 2, _L, _D, 512, _G, dict(att_wpc=0)))
    INSTANCES.append(("att_fused_kernel<%d,4,1,8>" % _G, 1, _L, 512, 8, _G, dict(att_wpc=0)))
for _G, _L, _D, _A, _D1 in ((1, 49, 64, 32, 64), (2, 255, 288, 24, 96), (3, 256, 768, 520, 2016), (4, 2, 2048, 40, 32)):
    INSTANCES.append(("att_fused_kernel<%d,0,1,8>" % _G, 2, _L, _D, _A, _G, {}))
    INSTANCES.append(("att_fused_kernel<%d,0,1,8>" % _G, 1, _L, _D1, 8, _G, {}))
INSTANCES += [
    ("att_fused_kernel<1,4,2,8>", 2, 196, 512, 512, 1, dict(att_occ=2)),
    ("att_fused_kernel<1,4,2,8>", 1, 49, 512, 8, 1, dict(att_occ=2)),
    ("att_fused_kernel<1,0,2,8>", 2, 49, 64, 32, 1, dict(att_occ=2)),
    ("att_fused_kernel<1,0,2,8>", 1, 255, 96, 8, 1, dict(att_occ=2)),
    ("att_fused_kernel<1,4,1,16>", 2, 196, 512, 512, 1, dict(att_warps=16, att_wpc=0)),
    ("att_fused_kernel<1,4,1,16>", 1, 9, 512, 8, 1, dict(att_warps=16, att_wpc=0)),
    ("att_fused_kernel<1,0,1,16>", 2, 49, 800, 520, 1, dict(att_warps=16)),
    ("att_fused_kernel<1,0,1,16>", 1, 256, 1536, 8, 1, dict(att_warps=16)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("instance,layers,L,D,A,G,opts", INSTANCES,
                         ids=["%s-%dlayer-L%d-D%d" % (i[0], i[1], i[2], i[3]) for i in INSTANCES])
def test_every_instance(instance, layers, L, D, A, G, opts):
    """Each instance at NI = 3 with the default plan (k CTAs per image) and with an SM budget that makes CTA row
    ranges cross image boundaries; the second call also checks that the first left the merge counters at zero."""
    assert expected_kernel(layers, D, A, G, **opts) == instance
    NI = 3
    occ = 2 if opts.get("att_occ") == 2 else 1
    sms = num_sms()
    assert regime(NI, L, sms * occ) in ("split", "whole")
    run_case(layers, L, D, A, NI, G, opts, fp32=True, what="default plan")
    if L > 1:
        budget = next(b for b in range(NI + 1, 4 * NI * L) if regime(NI, L, b * occ) == "cross")
        run_case(layers, L, D, A, NI, G, dict(opts, att_sms=budget), seed=1, what="att_sms=%d (cross)" % budget)


# ======================================================================================== pass-2 branches
# (consumer warps, D, branch): NT = 256 / 512 threads own the context features of a row
BRANCHES = ([(8, d, "scalar") for d in (32, 288, 2016)] + [(8, d, "vec1") for d in (256, 768, 1792)] +
            [(8, d, "vec2") for d in (512, 1024, 1536, 2048)] +
            [(16, d, "scalar") for d in (96, 800)] + [(16, d, "vec1") for d in (512, 1536)] +
            [(16, d, "vec2") for d in (1024, 2048)])


@pytest.mark.gpu
@pytest.mark.parametrize("layers", [2, 1])
@pytest.mark.parametrize("nw,D,branch", BRANCHES, ids=["NW%d-D%d-%s" % b for b in BRANCHES])
def test_pass2_branch(nw, D, branch, layers):
    """The fused kernel's context pass at every branch: scalar with one slot, a partial second slot and a partial
    eighth slot; vec1; vec2 (D = 1536 with 8 warps: vec2 on chunks of 5 rows, whose weights are not float4-aligned).
    The 2-layer rows have A = 24 or 520 (not multiples of 32); G = 3 with 8 warps, G = 1 with 16."""
    assert pass2_branch(D, nw) == branch
    G = 1 if nw == 16 else 3
    A = 24 if D % 64 else 520
    L = 49 if D <= 1024 else 9
    run_case(layers, L, D, A, 2, G, dict(att_wpc=0, att_warps=nw), what=branch)


# ======================================================================================== locations
@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2, 7, 8, 9, 49, 196, 255, 256])
@pytest.mark.parametrize("kernel", ["wpc", "fused"])
def test_locations(kernel, L):
    """Below and at one 8-row warp-per-chunk chunk, padded Lp (L % 4 != 0, the float4 weight reads of vec2), and the
    256 maximum.  wpc: 1-layer, D = 512, G = 2; fused: 2-layer, D = 512 (vec2), A = 24, G = 3."""
    if kernel == "wpc":
        run_case(1, L, 512, 8, 2, 2, what="L=%d" % L)
    else:
        run_case(2, L, 512, 24, 2, 3, what="L=%d" % L)


# ======================================================================================== grid regimes
def pick_ni(sms, L, which):
    """NI for a grid regime, from the grid rule.  Below #SMs the rows of a CTA cross image boundaries whenever
    NI * floor(#SMs / NI) < 0.8 * #SMs; on 132 SMs: cross_k3 = 34, cross_k2 = 45, cross_k1 = 67, cross_last = 105."""
    below = [n for n in range(1, sms) if regime(n, L, sms) == "cross"]
    return {"k1": 1, "k2": 2, "khalf": sms // 2,
            "cross_k3": min(below),
            "cross_k2": min(n for n in below if sms // n == 2),
            "cross_k1": min(n for n in below if sms // n == 1),
            "cross_last": max(below),
            "whole": sms, "over": sms + 1, "over2": 2 * sms + 5}[which]


REGIMES = [("k1", "split"), ("k2", "split"), ("khalf", "split"), ("cross_k3", "cross"), ("cross_k2", "cross"),
           ("cross_k1", "cross"), ("cross_last", "cross"), ("whole", "whole"), ("over", "cross"), ("over2", "cross")]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["wpc", "fused"])
@pytest.mark.parametrize("which,kind", REGIMES, ids=[r[0] for r in REGIMES])
def test_grid_regime(which, kind, kernel):
    """L = 49, 1-layer scorer (every row its own alpha); G = 2 except beyond 2 x #SMs images (G = 1, max_batch rows).
    wpc: D = 512; fused: D = 64 (scalar pass 2)."""
    sms = num_sms()
    NI = pick_ni(sms, 49, which)
    assert regime(NI, 49, sms) == kind
    G = 1 if which == "over2" else 2
    run_case(1, 49, 512 if kernel == "wpc" else 64, 8, NI, G, what="NI=%d %s" % (NI, kind))


@pytest.mark.gpu
def test_fewer_rows_than_sms():
    """NI * L < #SMs: one location per CTA, every image merged from L partials."""
    sms = num_sms()
    assert 3 * 7 < sms and plan_grid(3, 7, sms) == 21
    run_case(1, 7, 512, 8, 3, 2, what="NI*L < #SMs")
    run_case(2, 7, 64, 32, 3, 2, what="NI*L < #SMs")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["wpc", "fused"])
@pytest.mark.parametrize("budget", ["1", "2", "7", "sms-1"])
def test_sm_budget(budget, kernel):
    """att_sms: one CTA for all images, two, 7 (rows across images) and #SMs - 1; NI = 4, L = 49, G = 2.
    wpc: 1-layer D = 512; fused: 2-layer D = 288, A = 24."""
    b = num_sms() - 1 if budget == "sms-1" else int(budget)
    if kernel == "wpc":
        run_case(1, 49, 512, 8, 4, 2, dict(att_sms=b), what="att_sms=%d" % b)
    else:
        run_case(2, 49, 288, 24, 4, 2, dict(att_sms=b), what="att_sms=%d" % b)


@pytest.mark.gpu
def test_bench_configuration():
    """What bench.py times: the config-2 shape, att_sms = the grid of the attention launches inside a greedy loop,
    then att_reuse_q = 1 (the kernel alone, on the state branch of the call before)."""
    import torch
    cfg, w, m = make_pair(64, num_lstm_units=1024, vocabulary_size=10000)
    try:
        ctx, h = inputs(cfg, 64, 1, seed=3)
        m.decode_loop(ctx, 3)
        grid = m.info("att_loop_grid")
        assert 0 < grid <= m.info("num_sms")
        ctx_d = torch.from_numpy(ctx).cuda()
        ref = reference(cfg, w, ctx, h, 1)
        set_options(m, att_sms=grid)
        a1, z1, ks = attend_gpu(m, ctx_d, h, 1)
        ran(ks, "att_wpc_kernel<1>")
        check(a1, z1, ref, "att_wpc_kernel<1>", "bench: att_sms=%d" % grid)
        set_options(m, att_sms=grid, att_reuse_q=1)
        a2, z2, ks = attend_gpu(m, ctx_d, h, 1, prepare=False)
        ran(ks, "att_wpc_kernel<1>")
        assert np.array_equal(a1, a2) and np.array_equal(z1, z2)
    finally:
        set_options(m)
        m.close()


# ======================================================================================== values
@pytest.mark.gpu
@pytest.mark.parametrize("layers,L,D,A,G,opts", [(2, 49, 512, 512, 2, {}), (1, 255, 256, 8, 3, {}),
                                                (2, 196, 64, 24, 1, dict(att_warps=16)), (1, 256, 512, 8, 4, {})])
def test_uniform(layers, L, D, A, G, opts):
    """Zero attend/fc_2 (2-layer) or fc_a and fc_b (1-layer): alpha = 1/L and z = the mean context."""
    NI = 3
    cfg, w, m = own_model(layers, L, D, A, NI * G)
    try:
        names = ["attend/fc_2/kernel"] if layers == 2 else ["attend/fc_a/kernel", "attend/fc_b/kernel"]
        for n in names:
            w[n] = np.zeros_like(w[n])
        assert m.set_weights({n: w[n] for n in names}) == 0
        ctx, h = inputs(cfg, NI, G)
        set_options(m, **opts)
        alpha, z, ks = attend_gpu(m, ctx, h, G)
        want = expected_kernel(layers, D, A, G, **opts)
        ran(ks, want)
        ref = reference(cfg, w, ctx, h, G)
        assert np.allclose(ref["alpha"], 1.0 / L, rtol=1e-14, atol=0)
        assert np.allclose(ref["z"], np.repeat(ctx.astype(np.float64).mean(1), G, 0), rtol=1e-12, atol=1e-12)
        check(alpha, z, ref, want, "uniform")
    finally:
        m.close()


def hot_locations(NI, L, grid, chunk, per_image):
    """Per image, at most `per_image` locations: 0, L - 1, the first and last location of every CTA segment (the
    k-split boundaries floor(L*c/k) in the split regime), then, evenly spread over the rest of the budget, the
    chunk starts (multiples of `chunk` from a segment's start) with their predecessors."""
    ends = [{0, L - 1} for _ in range(NI)]
    inner = [set() for _ in range(NI)]
    for _, img, s0, s1 in cta_segments(NI, L, grid):
        a, b = s0 - img * L, s1 - img * L
        ends[img].update((a, b - 1))
        for x in range(a + chunk, b, chunk):
            inner[img].update((x - 1, x))
    hot = []
    for e, i in zip(ends, inner):
        e, i = sorted(e), sorted(i - e)
        n = max(0, per_image - len(e))
        hot.append(e[:per_image] + [i[j] for j in np.linspace(0, len(i) - 1, min(n, len(i))).astype(int)])
    return hot


@pytest.mark.gpu
@pytest.mark.parametrize("D,NI,G,L,opts,kind", [
    (512, 4, 4, 196, {}, "split"),                         # wpc, k = 33 CTAs per image
    (512, 4, 4, 256, dict(att_wpc=0), "split"),             # fused RV = 4, k = 33
    (64, "cross_k2", 1, 49, {}, "cross"),                   # fused RV = 0, rows across images
    (512, "cross_k2", 1, 196, {}, "cross"),                 # wpc, rows across images, 8-row chunks
])
def test_one_hot(D, NI, G, L, opts, kind):
    """1-layer: each row has one location whose logit is ~50 above the rest (column of attend/fc_b selected by a
    one-hot part of the row's state), placed in turn at up to 17 * G hot locations of its image: every segment
    boundary, and chunk boundaries.  alpha is ~1 there and z is that location's context."""
    sms = num_sms()
    if isinstance(NI, str):
        NI = pick_ni(sms, L, NI)
    assert regime(NI, L, sms) == kind
    rows = NI * G
    cfg, w, m = own_model(1, L, D, 8, rows)
    H = cfg.num_lstm_units
    assert rows <= H - 8
    try:
        want = expected_kernel(1, D, 8, G, **opts)
        chunk = 8 if want.startswith("att_wpc") else max(1, 32768 // (4 * D))
        hot = hot_locations(NI, L, plan_grid(NI, L, sms), chunk, 17 * G)
        ctx, h = inputs(cfg, NI, G, seed=5)
        h[:, :rows] = np.eye(rows, dtype=np.float32)
        base = w["attend/fc_b/kernel"].copy()
        base[:rows] = 0
        calls = max(-(-len(s) // G) for s in hot)
        for j in range(calls):
            pos = np.array([hot[r // G][(j * G + r % G) % len(hot[r // G])] for r in range(rows)])
            w["attend/fc_b/kernel"] = base.copy()
            w["attend/fc_b/kernel"][np.arange(rows), pos] = 50.0
            assert m.set_weights({"attend/fc_b/kernel": w["attend/fc_b/kernel"]}) == 0
            set_options(m, **opts)
            alpha, z, ks = attend_gpu(m, ctx, h, G)
            ran(ks, want)
            ref = reference(cfg, w, ctx, h, G)
            check(alpha, z, ref, want, "one-hot call %d" % j)
            assert (alpha[np.arange(rows), pos] > 1 - 1e-6).all()
            hot_ctx = ctx[np.arange(rows) // G, pos].astype(np.float64)
            assert (np.abs(z - hot_ctx).max(1) <= Z_BAR * ref["cmax"] * np.maximum(1, ref["scale"])).all()
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("D,A,NI,G,opts", [(512, 512, 3, 2, {}), (64, 32, 45, 1, {}), (256, 520, 5, 3, {}),
                                          (512, 512, 1, 1, dict(att_occ=2))])
def test_wide_logit_range(D, A, NI, G, opts):
    """2-layer with attend/fc_2 scaled so that a row's logits span several hundred: the segment maxima and the
    exp(m_c - M) merge must neither overflow nor lose the winning segments."""
    L = 196
    cfg, w, m = own_model(2, L, D, A, NI * G)
    try:
        ctx, h = inputs(cfg, NI, G, seed=9)
        lg = np.log(reference(cfg, w, ctx, h, G)["alpha"])          # logits up to a per-row constant
        w["attend/fc_2/kernel"] = w["attend/fc_2/kernel"] * np.float32(400 / (lg.max(1) - lg.min(1)).min())
        assert m.set_weights({"attend/fc_2/kernel": w["attend/fc_2/kernel"]}) == 0
        ref = reference(cfg, w, ctx, h, G)
        lg = np.log(ref["alpha"])
        assert (lg.max(1) - lg.min(1) > 390).all()
        set_options(m, **opts)
        alpha, z, ks = attend_gpu(m, ctx, h, G)
        want = expected_kernel(2, D, A, G, **opts)
        ran(ks, want)
        check(alpha, z, ref, want, "wide logits")
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("D,NI,G,opts", [(512, 3, 2, {}), (64, 45, 1, {}), (512, 2, 1, dict(att_wpc=0, att_warps=16))])
def test_shift_invariance(D, NI, G, opts):
    """1-layer with every column of attend/fc_b the same vector: h . fc_b adds one value per row (up to +-1e3) at
    every location, which the softmax removes: alpha and z equal those of the unshifted scorer (fc_b = 0)."""
    L = 49
    cfg, w, m = own_model(1, L, D, 8, NI * G)
    try:
        ctx, h = inputs(cfg, NI, G, seed=11)
        want = expected_kernel(1, D, 8, G, **opts)
        set_options(m, **opts)
        w["attend/fc_b/kernel"] = np.zeros_like(w["attend/fc_b/kernel"])
        assert m.set_weights({"attend/fc_b/kernel": w["attend/fc_b/kernel"]}) == 0
        a0, z0, ks = attend_gpu(m, ctx, h, G)
        ran(ks, want)
        ref = reference(cfg, w, ctx, h, G)
        check(a0, z0, ref, want, "unshifted")
        v = np.random.RandomState(2).uniform(-0.08, 0.08, cfg.num_lstm_units)
        v *= 1e3 / np.abs(h.astype(np.float64) @ v).max()
        w["attend/fc_b/kernel"] = np.repeat(v[:, None], L, 1).astype(np.float32)
        assert m.set_weights({"attend/fc_b/kernel": w["attend/fc_b/kernel"]}) == 0
        a1, z1, ks = attend_gpu(m, ctx, h, G)
        ran(ks, want)
        shifted = reference(cfg, w, ctx, h, G)
        assert np.abs(shifted["scale"]).max() > 900
        assert np.allclose(shifted["alpha"], ref["alpha"], rtol=1e-9, atol=0)
        check(a1, z1, shifted, want, "shifted +-1e3")
        # and against the kernel's own unshifted result, with the bars of the shifted rows
        check(a1, z1, dict(ref, alpha=a0.astype(np.float64), z=z0.astype(np.float64), scale=shifted["scale"]),
              want, "shifted vs unshifted")
    finally:
        set_options(m)
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("layers", [2, 1])
@pytest.mark.parametrize("wpc", [1, 0])
def test_vgg_features(wpc, layers):
    """The real conv5_3 features of tests/golden (14 images, 196 x 512, sparse with a long tail), G = 2."""
    feats = np.load(os.path.join(os.path.dirname(__file__), "golden", "vgg_conv5_3.npz"))["feats"].astype(np.float32)
    NI, L, D = feats.shape
    G = 2
    cfg, w, m = shared_model(layers, L, D, 512, NI * G)
    h = np.random.RandomState(4).uniform(-1, 1, (NI * G, cfg.num_lstm_units)).astype(np.float32)
    set_options(m, att_wpc=wpc)
    try:
        alpha, z, ks = attend_gpu(m, feats, h, G)
    finally:
        set_options(m)
    want = expected_kernel(layers, D, 512, G, att_wpc=wpc)
    ran(ks, want)
    check(alpha, z, reference(cfg, w, feats, h, G), want, "conv5_3 features")


# ======================================================================================== behaviour around the call
CALL_KERNELS = {"wpc": (1, 512, 8), "fused": (1, 288, 8)}


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["wpc", "fused"])
def test_repeatable_and_plan_changes(kernel):
    """Three calls with one plan are bit-identical (the merge order is fixed); calls alternating between plans
    (att_sms 0 -> 7 -> 0: k CTAs per image, then rows across images) each match the reference, so the merge
    counters reset themselves in both; alpha = NULL gives the same z."""
    import torch
    layers, D, A = CALL_KERNELS[kernel]
    NI, G, L = 4, 2, 49
    cfg, w, m = shared_model(layers, L, D, A, NI * G)
    sms = num_sms()
    assert regime(NI, L, sms) == "split" and regime(NI, L, 7) == "cross"
    ctx, h = inputs(cfg, NI, G, seed=13)
    ctx_d, h_d = torch.from_numpy(ctx).cuda(), torch.from_numpy(h).cuda()
    ref = reference(cfg, w, ctx, h, G)
    want = expected_kernel(layers, D, A, G)
    outs = []
    try:
        for sms_opt in (0, 0, 0, 7, 0, 7, 0):
            set_options(m, att_sms=sms_opt)
            alpha, z, ks = attend_gpu(m, ctx_d, h_d, G)
            ran(ks, want)
            check(alpha, z, ref, want, "att_sms=%d" % sms_opt)
            outs.append((sms_opt, alpha, z))
        first = outs[0]
        for sms_opt, alpha, z in outs:
            if sms_opt == 0:
                assert np.array_equal(alpha, first[1]) and np.array_equal(z, first[2])
        assert np.array_equal(outs[3][1], outs[5][1]) and np.array_equal(outs[3][2], outs[5][2])
        set_options(m)
        _, z_only, ks = attend_gpu(m, ctx_d, h_d, G, with_alpha=False)
        ran(ks, want)
        assert np.array_equal(z_only, first[2])
    finally:
        set_options(m)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["wpc", "fused"])
def test_reuse_q(kernel):
    """att_reuse_q = 1 (what bench.py times): the call keeps the state branch of the call before, so with the 1-layer
    scorer a second call with a different h returns the first call's results bit for bit."""
    import torch
    layers, D, A = CALL_KERNELS[kernel]
    NI, G, L = 3, 2, 49
    cfg, w, m = shared_model(layers, L, D, A, NI * G)
    ctx, h1 = inputs(cfg, NI, G, seed=17)
    h2 = np.random.RandomState(18).uniform(-1, 1, h1.shape).astype(np.float32)
    ref1, ref2 = reference(cfg, w, ctx, h1, G), reference(cfg, w, ctx, h2, G)
    assert np.abs(ref1["alpha"] - ref2["alpha"]).max() > 1e-3
    want = expected_kernel(layers, D, A, G)
    ctx_d = torch.from_numpy(ctx).cuda()
    try:
        set_options(m)
        a1, z1, ks = attend_gpu(m, ctx_d, h1, G)
        ran(ks, want)
        check(a1, z1, ref1, want, "reuse_q: first call")
        set_options(m, att_reuse_q=1)
        a2, z2, ks = attend_gpu(m, ctx_d, h2, G, prepare=False)
        ran(ks, want)
        assert np.array_equal(a1, a2) and np.array_equal(z1, z2)
        set_options(m)
        a3, z3, _ = attend_gpu(m, ctx_d, h2, G, prepare=False)
        check(a3, z3, ref2, want, "reuse_q off again")
    finally:
        set_options(m)


@pytest.mark.gpu
def test_invalid_calls_leave_outputs_untouched():
    """Errors return their code and enqueue no attention kernel: the NaN-filled outputs stay NaN."""
    import torch
    NI, L, D = 2, 49, 64
    cfg, w, m = shared_model(1, L, D, 8, 6)
    ctx, h = inputs(cfg, NI, 3)
    ctx_d, h_d = torch.from_numpy(ctx).cuda(), torch.from_numpy(h).cuda()
    alpha = torch.full((6, L), float("nan"), device="cuda")
    z = torch.full((6, D), float("nan"), device="cuda")
    P = m._p
    nul = C.c_void_p(0)
    cases = [
        ("group 0", (P(ctx_d), P(h_d), P(alpha), P(z), NI, 0), -1),
        ("group 5", (P(ctx_d), P(h_d), P(alpha), P(z), 1, 5), -4),
        ("n_img 0", (P(ctx_d), P(h_d), P(alpha), P(z), 0, 1), -1),
        ("n_img * group > max rows", (P(ctx_d), P(h_d), P(alpha), P(z), 4, 2), -1),
        ("null contexts", (nul, P(h_d), P(alpha), P(z), NI, 3), -1),
        ("null state", (P(ctx_d), nul, P(alpha), P(z), NI, 3), -1),
        ("null context vector", (P(ctx_d), P(h_d), P(alpha), nul, NI, 3), -1),
    ]
    torch.cuda.synchronize()
    for what, args, code in cases:
        rc = m.lib.sat_attention_fwd(m._h, *args, m._st())
        torch.cuda.synchronize()
        assert rc == code, "%s: returned %d, expected %d" % (what, rc, code)
        assert torch.isnan(alpha).all() and torch.isnan(z).all(), what
    a, zz, ks = attend_gpu(m, ctx, h, 3)
    want = expected_kernel(1, D, 8, 3)
    ran(ks, want)
    check(a, zz, reference(cfg, w, ctx, h, 3), want, "after the invalid calls")


# ======================================================================================== the comparator itself (CPU)
def _mutation_case(seed=0):
    """1-layer, NI = 3 images x G = 2 rows, L = 49, D = 64: fp64 reference and its fp32 rounding ("a perfect
    kernel"), plus the k = 4 split boundaries floor(L * c / k)."""
    cfg = R.OracleConfig(batch_size=6, beam_size=1, num_ctx=49, dim_ctx=64, num_attend_layers=1, **SMALL)
    w = R.init_weights(cfg, seed=seed)
    ctx = R.synth_contexts(cfg, 3, seed=seed)
    h = np.random.RandomState(seed).uniform(-1, 1, (6, cfg.num_lstm_units)).astype(np.float32)
    ref = reference(cfg, w, ctx, h, 2)
    bounds = [49 * c // 4 for c in range(5)]
    return ref, np.repeat(ctx.astype(np.float64), 2, 0), bounds


def _rejected(alpha, z, ref):
    ea, ez = errors(alpha, z, ref)
    return ea > ALPHA_BAR or ez > Z_BAR


def test_comparator_accepts_the_rounded_reference():
    ref, _, _ = _mutation_case()
    ea, ez = errors(ref["alpha"].astype(np.float32), ref["z"].astype(np.float32), ref)
    assert ea < 1e-7 and ez < 1e-7


def test_comparator_rejects_a_dropped_location():
    """The smallest weight of one row set to 0 and the row renormalised: far below the max-norm bar of _util."""
    ref, ctx_rows, _ = _mutation_case()
    a = ref["alpha"].copy()
    l = int(a[3].argmin())
    a[3, l] = 0
    a[3] /= a[3].sum()
    z = np.einsum("bl,bld->bd", a, ctx_rows)
    assert _rejected(a.astype(np.float32), z.astype(np.float32), ref)
    assert _rejected(a.astype(np.float32), ref["z"].astype(np.float32), ref)       # alpha alone
    assert _rejected(ref["alpha"].astype(np.float32), z.astype(np.float32), ref)   # z alone


@pytest.mark.parametrize("c", [0, 1, 2, 3])
@pytest.mark.parametrize("f", [math.exp(0.5), math.exp(-0.5)])
def test_comparator_rejects_a_misscaled_partial(f, c):
    """Segment c of a 4-way split merged with its (sum, partial context) scaled by e^+-0.5: every alpha of the row
    is off by the wrong total, z by the segment's share."""
    ref, ctx_rows, b = _mutation_case()
    a, z = ref["alpha"].copy(), ref["z"].copy()
    seg = slice(b[c], b[c + 1])
    mass = a[1, seg].sum()
    S = 1 + (f - 1) * mass
    z[1] = (z[1] + (f - 1) * a[1, seg] @ ctx_rows[1, seg]) / S
    a[1] /= S
    assert _rejected(a.astype(np.float32), z.astype(np.float32), ref)
    # alpha alone (a kernel that merged z right but the sum wrong) is rejected too
    assert _rejected(a.astype(np.float32), ref["z"].astype(np.float32), ref)


@pytest.mark.parametrize("c", [1, 2, 3])
def test_comparator_rejects_an_off_by_one_segment(c):
    """The segment starting at boundary c reads its weights one location early (alpha[l] = alpha[l - 1])."""
    ref, ctx_rows, b = _mutation_case()
    a = ref["alpha"].copy()
    a[4, b[c]:b[c + 1]] = ref["alpha"][4, b[c] - 1:b[c + 1] - 1]
    z = np.einsum("bl,bld->bd", a, ctx_rows)
    assert _rejected(a.astype(np.float32), z.astype(np.float32), ref)
    assert _rejected(ref["alpha"].astype(np.float32), z.astype(np.float32), ref)   # z alone


def test_comparator_rejects_swapped_rows():
    """1-layer: the two rows of image 1 exchanged (a kernel that mixes up img * G + g)."""
    ref, _, _ = _mutation_case()
    a, z = ref["alpha"].copy(), ref["z"].copy()
    a[[2, 3]], z[[2, 3]] = a[[3, 2]], z[[3, 2]]
    assert _rejected(a.astype(np.float32), z.astype(np.float32), ref)
    assert _rejected(ref["alpha"].astype(np.float32), z.astype(np.float32), ref)   # z alone


def test_comparator_rejects_unwritten_outputs():
    ref, _, _ = _mutation_case()
    a, z = ref["alpha"].astype(np.float32), ref["z"].astype(np.float32)
    a[5, 48] = np.nan
    z[0, 0] = np.nan
    assert errors(a, ref["z"], ref)[0] == math.inf and errors(ref["alpha"], z, ref)[1] == math.inf


def test_plan_restatement():
    """The grid rule restated here gives the regimes the GPU cases claim (132 SMs, the H100 SXM)."""
    assert [pick_ni(132, 49, k) for k in ("cross_k3", "cross_k2", "cross_k1", "cross_last")] == [34, 45, 67, 105]
    assert [n for n in range(1, 132) if regime(n, 7, 132) == "cross"] == [34, 35] + list(range(45, 53)) + list(range(67, 106))
    assert regime(66, 49, 132) == "split" and plan_grid(66, 49, 132) == 132
    assert regime(132, 49, 132) == "whole" and regime(133, 49, 132) == "cross"
    assert plan_grid(3, 7, 132) == 21 and regime(269, 49, 132) == "cross"
    assert [s[2] for s in cta_segments(1, 49, 4)] == [0, 12, 24, 36]
    assert expected_kernel(2, 512, 512, 2, att_occ=2) == "att_wpc_kernel<2>"
    assert expected_kernel(2, 512, 512, 1, att_occ=2, att_warps=16) == "att_fused_kernel<1,4,2,8>"
    assert pass2_branch(1536, 8) == "vec2" and pass2_branch(1536, 16) == "vec1"
