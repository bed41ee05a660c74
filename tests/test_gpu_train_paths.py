"""Every launch path of the training step (csrc/sat_train.cu) against the autograd oracle: the SAT_TRAIN_* environment
switches, groups wider than one tile of the grouped scorer backward, the tensor-core plan's edges (ragged vocabulary,
padded row tiles, more than 128 rows, CUDA cores at config-4 widths) and graph capture and replay.

Every eager call is profiled and its kernel multiset must equal the plan of tests/train_plan.py (the selection rules of
sat_train_init_grouped and train_enqueue restated), so a case that silently took another path fails.  Losses are
compared with the oracle to 1e-4 and every gradient to 2e-4 (max-norm relative per tensor, grad_check), the bars of
test_gpu_train.py.  A switch runs in a child process (tests/train_paths_run.py; the library reads each switch once
per process) whose results must also agree with the default path of this process, and a replayed graph must agree
with the eager call.  Both agreement bars compare the same tensor-core choices in another summation or float-atomic
order: AGREE_BAR (a switch's eager, captured and replayed calls vs the default path; its replay vs its eager call)
and REPLAY_BAR (replay vs eager on the default path), max |a - b| over the oracle tensor's largest value, per tensor
and for the losses.

Worst errors over the module on an H100 80GB HBM3 (SXM, 132 SMs, 400 W power limit); the module took 177 to 196 s there.
Where two runs differed, both are given (the order of float atomics varies from call to call):
    against the oracle (gradient: grad_check; losses: relative)        gradient   losses
      ragged vocabulary (V = 100)                                      1.7e-5     1.8e-7
      padded dec_all tile (T*B = 192)                                  1.3e-5     1.5e-7
      rows not a multiple of 16 (B = 20)                               1.3e-5     8.5e-8
      more than 128 rows, grouped (32 x 5)                             7.4e-6     3.9e-7
      wide groups (G = 8, 9, 16, 17), TDIMS / TC_DIMS                  7.3e-6 / 2.2e-5   4.3e-7 / 8.2e-7
      config-4 widths on CUDA cores                                    1.6e-5     1.5e-7
      graph replay, config-4 widths B = 32 T = 6 (every call)          2.1e-5     7.6e-7
      graph replay, TC_DIMS 4 x 5 (every call)                         2.2e-5     4.1e-6
      every switch, every call                                         1.0e-5     2.9e-7
    agreement with the default path (eager, captured and replayed calls of the child)
      SAT_TRAIN_PDL=0 3.4e-7 / 4.3e-7     DEC_ALL=0 3.4e-7 / 3.8e-7     SIDE=0 3.4e-7 / 3.1e-7
      SIDE=2 4.3e-7 / 3.4e-7     SIDE=3 3.4e-7 / 3.1e-7     FUSE_SOFTMAX=0 3.4e-7 / 2.9e-7
      FUSE_SOFTMAX=2 3.4e-7 / 2.9e-7     FUSE_PACK=0 5.1e-7 / 3.1e-7     ATTBWD_WAVE=1 3.1e-6 / 2.2e-6
    replay vs eager: config-4 widths 7.8e-6 / 7.9e-6, TC_DIMS 4 x 5 2.3e-6 / 4.7e-6; within a switch's child at most
      4.3e-7 (SAT_TRAIN_ATTBWD_WAVE=1: 3.1e-6)
The bars below are about 8x the worst of each.
"""
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import pytest

import grouped_train_ref as GR
import train_paths_run as RUN
from test_gpu_scst import check_losses
from test_gpu_train import TC_DIMS, TDIMS, grad_check
from train_plan import plan_diff, train_plan

pytestmark = pytest.mark.gpu

AGREE_BAR = {"SAT_TRAIN_PDL=0": 4e-6, "SAT_TRAIN_DEC_ALL=0": 3e-6, "SAT_TRAIN_SIDE=0": 3e-6, "SAT_TRAIN_SIDE=2": 4e-6,
             "SAT_TRAIN_SIDE=3": 3e-6, "SAT_TRAIN_FUSE_SOFTMAX=0": 3e-6, "SAT_TRAIN_FUSE_SOFTMAX=2": 4e-6,
             "SAT_TRAIN_FUSE_PACK=0": 4e-6, "SAT_TRAIN_ATTBWD_WAVE=1": 2.5e-5}
REPLAY_BAR = {"config4_b32_t6": 6e-5, "tc_grouped_4x5": 4e-5}
GRAD_BAR = 2e-4
FLOOR = 1e-3            # "typical gradient" floor of grad_check for mathematically zero gradients (dropout off)

SWITCHES = [("SAT_TRAIN_PDL", "0"), ("SAT_TRAIN_DEC_ALL", "0"), ("SAT_TRAIN_SIDE", "0"), ("SAT_TRAIN_SIDE", "2"),
            ("SAT_TRAIN_SIDE", "3"), ("SAT_TRAIN_FUSE_SOFTMAX", "0"), ("SAT_TRAIN_FUSE_SOFTMAX", "2"),
            ("SAT_TRAIN_FUSE_PACK", "0"), ("SAT_TRAIN_ATTBWD_WAVE", "1")]
C4 = dict(num_lstm_units=1024, vocabulary_size=10000)       # config-4 widths (L 196, D 512, A 512 by default)
GROUP_SHAPE = dict(num_ctx=196, dim_ctx=128, dim_attend_layer=128, dim_embedding=64, num_lstm_units=64,
                   dim_decode_layer=64, vocabulary_size=1000, max_caption_length=4)

_ORACLE = {}
_DEFAULT = {}
WORST = {}


def note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), float(v))


@pytest.fixture(scope="module", autouse=True)
def _module_report():
    t0 = time.time()
    yield
    print("\nworst errors (oracle: grad_check / losses relative; agreement: max |a - b| / max |oracle|):")
    for k in sorted(WORST):
        print("  %-56s %.3e" % (k, WORST[k]))
    print("module time %.1f s" % (time.time() - t0))


def oracle(key, ocfg, w, host, seed, G):
    """(losses, gradients) of the fp64 oracle, cached per (shape, seed, data) within the module."""
    k = (key, seed)
    if k not in _ORACLE:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            _ORACLE[k] = GR.loss_and_grads(ocfg, w, host["ctx"], host["sent"], host["masks"], seed if seed else None,
                                           reg_in_grad=False, group=G, row_weights=host["rw"])
    return _ORACLE[k]


class Grads(object):
    """grad_check's view of gradients held on the host."""
    def __init__(self, g):
        self.g = g

    def train_state_dict(self, which):
        import torch
        return {k: torch.from_numpy(v) for k, v in self.g.items()}


def check_oracle(tag, losses, grads, ref):
    ref_l, ref_g = ref
    check_losses(losses, ref_l)
    for i, name in ((0, "cross_entropy_loss"), (2, "attention_loss")):
        note("oracle %s: loss" % tag, abs(float(losses[i]) - ref_l[name]) / max(abs(ref_l[name]), 1e-30))
    note("oracle %s: gradient" % tag, grad_check(Grads(grads), ref_g, GRAD_BAR, floor_rel=FLOOR))


def agreement(a, b, ref):
    """Largest max |a - b| / max |oracle| over the losses and every gradient of two calls."""
    (la, ga), (lb, gb), (ref_l, ref_g) = a, b, ref
    worst = max(abs(float(la[i]) - float(lb[i])) / max(abs(ref_l[n]), 1e-30) for i, n in ((0, "cross_entropy_loss"),
                                                                                          (2, "attention_loss")))
    floor = FLOOR * max(np.abs(g).max() for g in ref_g.values())
    for k, g in ref_g.items():
        worst = max(worst, float(np.abs(ga[k].reshape(g.shape) - gb[k].reshape(g.shape)).max()) / max(np.abs(g).max(), floor))
    return worst


def num_sms(m):
    return m.info("num_sms")


def eager_case(tag, key, dims, n_img, G, seed, train_tc=1, data_seed=3):
    """One eager call: kernels against the plan, losses and gradients against the oracle."""
    ocfg, w, m, host, dev = RUN.gpu_setup(dims, n_img, G, seed=data_seed)
    T = ocfg.max_caption_length
    m.set_option("train_tc", train_tc)
    ref = oracle(key, ocfg, w, host, seed, G)
    rec, losses, grads = RUN.eager_profiled(m, dev, seed)
    fields, launches = train_plan(dims, n_img, G, T, train_tc, env={}, sms=num_sms(m), weighted=G > 1)
    diff = plan_diff(launches, rec)
    assert not diff, "%s: kernels differ from the plan %s: %s" % (tag, fields, diff)
    check_oracle(tag, losses, grads, ref)
    m.close()
    return fields, launches, rec, (losses, grads), ref


# ============================================================================================ shape cases
SHAPES = {   # name: (dims, n_img, G)
    "ragged_vocabulary": (dict(TC_DIMS, vocabulary_size=100), 16, 1),
    "padded_dec_all_tile": (TC_DIMS, 48, 1),
    "rows_not_multiple_of_16": (TC_DIMS, 20, 1),
    "more_than_128_rows": (GROUP_SHAPE, 32, 5),
}


@pytest.mark.parametrize("seed", [0, 31])
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_tensor_core_plan_edges(name, seed):
    dims, n_img, G = SHAPES[name]
    f, k, rec, _, _ = eager_case(name, (name, n_img, G), dims, n_img, G, seed)
    # what each shape is here to reach (the plan and the capture already agree on every launch)
    if name == "ragged_vocabulary":
        assert f["tc_stack"] and f["tc_vk"] == 0 and not f["dec_all"] and f["fwd"][3] and not f["dx"][3]
        assert k["lin_mma_kernel<1>"] > 0 and k["sgemm_kernel<false,true>"] >= 4     # fc_2 on wgmma, dtd via sgemm
    elif name == "padded_dec_all_tile":
        assert f["dec_all"] and f["all_rt"] == 128 and f["all_rows"] == 256 and f["tc_rt"] == 48
    elif name == "rows_not_multiple_of_16":
        assert f["tc_rt"] == 32 and not f["tc_stack"] and k["lin_mma_kernel<2>"] > 0
    else:
        assert f["tc_ok"] and f["tc_rt"] == 160 and not any(f["fwd"]) and f["ab_chunks"] > 1
        assert k["sgemm_kernel<false,true>+splitk"] > 0 and k["att_bwd_grouped_kernel"] == 4
        assert set(n for n in k if n.startswith("lin_mma")) == {"lin_mma_kernel<8>"}   # attend/fc_1a only


@pytest.mark.parametrize("seed", [0, 31])
@pytest.mark.parametrize("G", [8, 9, 16, 17])
@pytest.mark.parametrize("dims_name,n_img", [("TDIMS", 2), ("TC_DIMS", 4)])
def test_wide_groups(dims_name, n_img, G, seed):
    """More rows per image than one tile (8 rows) of att_bwd_grouped_kernel: the later tiles add to d temp, and are
    full (G = 16) or partial (9, 17)."""
    dims = dict(TDIMS=TDIMS, TC_DIMS=TC_DIMS)[dims_name]
    f, k, _, _, _ = eager_case("wide_groups %s" % dims_name, ("wide", dims_name, n_img, G), dims, n_img, G, seed)
    assert k["att_bwd_grouped_kernel"] == dims["max_caption_length"]


@pytest.mark.parametrize("seed", [0, 21])
def test_config4_widths_on_cuda_cores(seed):
    """train_tc = 0 at the config-4 widths: every product on sgemm_kernel, with split K on zeroed and on accumulated
    outputs."""
    dims = dict(C4, max_caption_length=4)
    f, k, _, _, _ = eager_case("config4_cuda_cores", ("c4", 64), dims, 64, 1, seed, train_tc=0, data_seed=13)
    assert not any(n.startswith(("lin_mma", "pack_rows", "repack")) for n in k)
    for inst in ("sgemm_kernel<false,false>+splitk", "sgemm_kernel<true,false>+splitk", "sgemm_kernel<false,true>+splitk"):
        assert k[inst] > 0, inst


# ============================================================================================ graph replay
@pytest.mark.parametrize("case", ["config4_b32_t6", "tc_grouped_4x5"])
def test_graph_replay_matches_the_oracle(case):
    """Eager, captured and replayed calls on the same buffers, each against the oracle; the replay against the eager
    call; then new contexts and sentences in the same buffers, replayed, against the oracle of the new values."""
    import torch
    seed = 7
    dims, n_img, G = (dict(C4, max_caption_length=6), 32, 1) if case == "config4_b32_t6" else (TC_DIMS, 4, 5)
    ocfg, w, m, host, dev = RUN.gpu_setup(dims, n_img, G, seed=5)
    fields, _ = train_plan(dims, n_img, G, ocfg.max_caption_length, sms=num_sms(m), weighted=G > 1)
    assert fields["side_f"] and fields["side_b"]
    if case == "config4_b32_t6":
        assert fields["dec_all"] and fields["all_rows"] == 256
    ref = oracle(("replay", case), ocfg, w, host, seed, G)
    runs = RUN.eager_captured_replayed(m, dev, seed)
    for tag, r in zip(("eager", "captured", "replayed"), runs):
        check_oracle("replay %s %s" % (case, tag), r[0], r[1], ref)
    for r in runs[1:]:
        e = agreement(runs[0], r, ref)
        note("replay vs eager: %s" % case, e)
        assert e <= REPLAY_BAR[case], e
    # new values in the same buffers: the graph reads them
    rng = np.random.RandomState(99)
    host2 = dict(host, ctx=(host["ctx"][::-1] * 0.5 + 0.1).astype(np.float32).copy(),
                 sent=rng.randint(1, ocfg.vocabulary_size, host["sent"].shape).astype(np.int32))
    dev["ctx"].copy_(torch.from_numpy(host2["ctx"]))
    dev["sent"].copy_(torch.from_numpy(host2["sent"]))
    assert RUN.step(m, dev, seed) == 0
    losses, grads = RUN.results(m)
    check_oracle("replay %s new inputs" % case, losses, grads, oracle(("replay2", case), ocfg, w, host2, seed, G))
    m.close()


# ============================================================================================ switches
def default_runs():
    """The switch shapes on the default path of this process (eager): [(name, ocfg, w, host, plan fields, run)]."""
    if not _DEFAULT:
        for name, dims, n_img, G in RUN.SWITCH_SHAPES:
            f, k, rec, run, ref = eager_case("default " + name, ("switch", name), dims, n_img, G, RUN.SWITCH_SEED)
            _DEFAULT[name] = (dims, n_img, G, run, ref)
    return _DEFAULT


@pytest.mark.parametrize("var,value", SWITCHES)
def test_switch_agrees_with_the_default_path(var, value, tmp_path, built_lib):
    defaults = default_runs()
    out = tmp_path / "switch.npz"
    env = {k: v for k, v in os.environ.items() if not k.startswith("SAT_TRAIN_")}
    env[var] = value
    # (the child only loads the library built_lib built; on a timeout, run() kills it and waits for it)
    proc = subprocess.run([sys.executable, os.path.join(RUN.HERE, "train_paths_run.py"), str(out)], env=env,
                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-4000:]
    data = np.load(out)
    tag = "%s=%s" % (var, value)
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for name, (dims, n_img, G, default, ref) in defaults.items():
        T = dims["max_caption_length"]
        fields, launches = train_plan(dims, n_img, G, T, env={var: value}, sms=sms, weighted=G > 1)
        rec = [(str(n), None if g[0] < 0 else tuple(int(x) for x in g))
               for n, g in zip(data[name + "/kernels"], data[name + "/grids"])]
        diff = plan_diff(launches, rec)
        assert not diff, "%s %s: kernels differ from the plan %s: %s" % (tag, name, fields, diff)
        runs = {}
        for call in ("eager", "captured", "replayed"):
            pre = "%s/%s/grad/" % (name, call)
            grads = {k[len(pre):]: data[k] for k in data.files if k.startswith(pre)}
            runs[call] = (data["%s/%s/losses" % (name, call)], grads)
            check_oracle("switch %s" % tag, runs[call][0], grads, ref)
        e = max(agreement(default, runs[c], ref) for c in runs)
        note("agreement %s" % tag, e)
        assert e <= AGREE_BAR[tag], "%s %s: %.3e" % (tag, name, e)
        e = max(agreement(runs["eager"], runs[c], ref) for c in ("captured", "replayed"))
        note("replay vs eager: switch %s" % tag, e)
        assert e <= AGREE_BAR[tag], "%s %s replay: %.3e" % (tag, name, e)


# ============================================================================================ alignment
def test_misaligned_buffers_are_refused_and_enqueue_nothing():
    """params, grads and contexts one float off a 16-byte boundary: SAT_ERR_INVALID from every training entry point,
    with nothing enqueued (the step reads these buffers with 16-byte vector loads)."""
    import torch
    ocfg, w, m, host, dev = RUN.gpu_setup(TC_DIMS, 4, 3)
    n_img, G = m._train_group
    B, T = m._train_BT
    L, P = m.lib, m._p

    def off(t):   # the same values one float later: a view whose address is 4 bytes past a 16-byte boundary
        buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
        v = buf[1:1 + t.numel()].view_as(t)
        v.copy_(t)
        return v
    losses = torch.full((4,), 7.0, device="cuda")
    gsum = dev["gsum"]

    def variants(ctx):   # (params, grads, contexts) with exactly one of them off
        bad_g = off(m.grads)
        return [(off(m.params), m.grads, ctx), (m.params, bad_g, ctx), (m.params, m.grads, off(ctx))], bad_g
    cases, bad_g = variants(dev["ctx"])
    m.grads.fill_(3.0)
    bad_g.fill_(3.0)
    torch.cuda.synchronize()
    for pp, gg, cc in cases:
        assert L.sat_train_forward_backward_grouped(m._h, P(pp), P(gg), P(cc), n_img, G, P(dev["sent"]), P(dev["masks"]),
                                                    P(dev["rw"]), T, 0, P(gsum), B, P(losses), m._st()) == -1
        assert b"aligned" in L.sat_last_error()
    m.stream.synchronize()
    assert bool((losses == 7.0).all()) and bool((m.grads == 3.0).all()) and bool((bad_g == 3.0).all())
    # the ungrouped entry points, on a state of B rows with the contexts replicated
    m.train_setup(B, T, weights=w)
    cases, bad_g = variants(torch.from_numpy(np.repeat(host["ctx"], G, axis=0)).cuda())
    m.grads.fill_(3.0)
    bad_g.fill_(3.0)
    torch.cuda.synchronize()
    for pp, gg, cc in cases:
        assert L.sat_train_forward_backward(m._h, P(pp), P(gg), P(cc), P(dev["sent"]), P(dev["masks"]), B, T, 0,
                                            float(host["masks"].sum()), B, P(losses), m._st()) == -1
        assert L.sat_train_forward_backward_dsum(m._h, P(pp), P(gg), P(cc), P(dev["sent"]), P(dev["masks"]), B, T, 0,
                                                 P(gsum), B, P(losses), m._st()) == -1
    m.stream.synchronize()
    assert bool((losses == 7.0).all()) and bool((m.grads == 3.0).all()) and bool((bad_g == 3.0).all())
    # and the same buffers aligned run
    assert L.sat_train_forward_backward_dsum(m._h, P(m.params), P(m.grads), P(cases[0][2]), P(dev["sent"]), P(dev["masks"]),
                                             B, T, 0, P(gsum), B, P(losses), m._st()) == 0
    m.stream.synchronize()
    assert bool((losses != 7.0).any())
    m.close()
