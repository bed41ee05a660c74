"""Which kernels one call of the training step launches: the selection rules of sat_train_init_grouped and
train_enqueue (csrc/sat_train.cu) restated in Python, and the kernel names of a profiler capture reduced to the names
the plan uses.

The plan covers the shipped graph (two attend, decode and initialize layers) called through an entry point that reads
the mask sum from device memory (sat_train_forward_backward_dsum or _grouped), with 16-byte aligned buffers.  It
returns the launch multiset of every kernel of the step (not the memsets and copies), with two refinements: a
sgemm_kernel launch that splits K over gridDim.z is named "sgemm_kernel<TA,TB>+splitk", and a lin_mma_kernel launch
is named by its row tile in 16-row MMA widths, "lin_mma_kernel<NT>"."""
import math
import re
from collections import Counter

from oracle import ref_step as R

K_MAX_ROW_TILE = 128      # sat_linear.cuh kMaxRowTile
K_AB_CT = 64              # sat_train.cu kAbCT: float4 columns per CTA of the scorer backward
K_SM_L = 1024             # sat_train.cu kSmL: the fused softmax + context kernel holds L weights in shared memory
NUM_REGULARISED = 10      # embedding + the nine dense kernels of the shipped graph (sumsq_kernel launches)

# every kernel train_forward_backward can launch for the shipped graph (base names; the anonymous namespace and
# sat:: are stripped)
KERNELS = (
    "sgemm_kernel", "dropout2d_kernel", "bias_act_kernel", "drop_tanh_bwd_kernel", "tanh_bwd_kernel", "colsum_kernel",
    "concat3_drop_kernel", "dropout_pack_kernel", "tanh_bwd_pack_kernel", "dropout_steps_kernel", "split3_drop_kernel",
    "copy2d_kernel", "gather_rows_kernel", "scatter_add_rows_kernel", "att_temp_kernel", "att_logits_kernel",
    "att_bwd_fused_kernel", "att_bwd_fused_wave_kernel", "att_bwd_grouped_kernel", "expand_rows_kernel",
    "group_sum_kernel", "rowdot_kernel", "softmax_rows_kernel", "softmax_bwd_kernel", "context_fwd_kernel",
    "context_fwd4_kernel", "softmax_context_fwd4_kernel", "context_bwd_kernel", "att_dtemp_kernel", "segsum_kernel",
    "lstm_fwd_kernel", "lstm_bwd_kernel", "ce_kernel", "coverage_loss_kernel", "mean_L_kernel", "sumsq_kernel",
    "reciprocal_kernel", "lin_mma_kernel", "repack_weight_kernel", "repack_bias_kernel", "pack_rows_kernel")
_KNOWN = frozenset(KERNELS)
_BOOL = {"0": "false", "1": "true"}


def _ceil(a, b):
    return (a + b - 1) // b


def _atoi(v, default):
    """C atoi of an environment value (unset: default)."""
    if v is None:
        return default
    m = re.match(r"\s*([+-]?\d+)", v)
    return int(m.group(1)) if m else 0


def train_plan(dims, n_img, G, T, train_tc=1, env=None, sms=132, weighted=False):
    """(fields, launches): the decisions of sat_train_init_grouped / train_enqueue for n_img images of G caption rows
    and T steps, and the Counter of kernel launches of one call.  dims: OracleConfig field names; env: the SAT_TRAIN_*
    environment of the process; sms: the device's SM count; weighted: row weights passed."""
    c = R.OracleConfig(batch_size=n_img * G, **dims)
    assert (c.num_attend_layers, c.num_decode_layers, c.num_initalize_layers) == (2, 2, 2), "the shipped graph only"
    L, D, E, H, A = c.num_ctx, c.dim_ctx, c.dim_embedding, c.num_lstm_units, c.dim_attend_layer
    Dd, I, V = c.dim_decode_layer, c.dim_initalize_layer, c.vocabulary_size
    env = {} if env is None else env
    B, NI = n_img * G, n_img
    BLi, XL, XD, TB = NI * L, D + E + H, H + D + E, T * B
    f = {}
    # ---- sat_train_init_grouped
    f["tc_ok"] = D % 128 == 0 and A % 128 == 0 and BLi % 128 == 0
    f["tc_rt"] = _ceil(B, 16) * 16
    Ks, Ns = [H, XL, XD, Dd], [A, 4 * H, Dd, V]
    f["fwd"] = [K % 64 == 0 and f["tc_rt"] <= K_MAX_ROW_TILE for K in Ks]
    f["dx"] = [f["fwd"][i] and Ns[i] % 64 == 0 for i in range(4)]
    f["tc_vk"] = _ceil(V, 64) * 64 if f["fwd"][3] and V % 8 == 0 else 0
    f["tc_stack"] = TB % 64 == 0 and all(f["fwd"][i] and (i == 3 or f["dx"][i]) for i in range(4))
    f["all_rt"] = f["all_rows"] = None
    if f["tc_stack"]:
        f["all_rt"] = 128 if TB >= 128 else TB
        f["all_rows"] = _ceil(TB, f["all_rt"]) * f["all_rt"]
    # ---- train_enqueue
    pdl = env.get("SAT_TRAIN_PDL", "x")[:1] != "0"
    fuse_pack = env.get("SAT_TRAIN_FUSE_PACK", "x")[:1] != "0"
    dec_all_env = env.get("SAT_TRAIN_DEC_ALL", "x")[:1] != "0"
    side_env = _atoi(env.get("SAT_TRAIN_SIDE"), 1)
    fuse_env = _atoi(env.get("SAT_TRAIN_FUSE_SOFTMAX"), 1)
    wave = env.get("SAT_TRAIN_ATTBWD_WAVE", "")[:1] == "1"
    tc, tcb = f["tc_ok"] and bool(train_tc), bool(train_tc)
    tcv = tcb and f["tc_vk"] > 0
    stack = tcb and f["tc_stack"]
    f["dec_all"] = stack and tcv and dec_all_env
    f["att_fused"] = A % 4 == 0
    side_any = tc and f["att_fused"] and side_env != 0          # (the side stream exists whenever tc_ok)
    f["side_f"], f["side_b"] = side_any and side_env != 3, side_any and side_env != 2
    f["fuse_softmax_fwd"] = D % 4 == 0 and L <= K_SM_L and fuse_env != 0
    f["fuse_softmax_bwd"] = f["att_fused"] and fuse_env == 1
    gx = _ceil(A // 4, K_AB_CT)
    ab = _ceil(sms * 4, NI * gx)
    ab = max(1, min(ab, _ceil(L, 16)))
    f["ab_rows"] = _ceil(L, ab)
    f["ab_chunks"] = _ceil(L, f["ab_rows"])
    if wave:          # (row chunks from the occupancy of the 64-register build: known on the device only)
        f["ab_rows"] = f["ab_chunks"] = None
    f["att_bwd_ctas"] = None if wave else gx * f["ab_chunks"] * (B if G == 1 else NI)
    f["pdl"] = pdl
    pk_fwd = [tcb and fuse_pack and f["fwd"][i] for i in range(4)]
    pk_dx = [tcb and fuse_pack and f["dx"][i] for i in range(4)]
    tc_fwd = [tcb and f["fwd"][i] for i in range(4)]
    tc_dx = [tcb and f["dx"][i] for i in range(4)]
    dec_all, rt = f["dec_all"], f["tc_rt"]

    k = Counter()

    def add(name, n=1):
        k[name] += n

    def mma(row_tile):
        add("lin_mma_kernel<%d>" % (row_tile // 16))

    def sgemm(ta, tb, M, N, K, ldc, acc):
        tiles, z = _ceil(N, 128) * _ceil(M, 128), 1
        if tiles < sms and K >= 512:
            z = max(1, min(_ceil(2 * sms, tiles), K // 128))
            kchunk = _ceil(_ceil(K, z), 8) * 8
            z = _ceil(K, kchunk)
            if z > 1 and not acc and ldc != N:
                z = 1
        add("sgemm_kernel<%s,%s>%s" % ("true" if ta else "false", "true" if tb else "false", "+splitk" if z > 1 else ""))

    def dense_fwd(rows, K, N):           # (every layer of the shipped graph has a bias: bias_act_kernel follows)
        sgemm(False, False, rows, N, K, N, False)
        add("bias_act_kernel")

    def dense_bwd(rows, K, N, dx):
        sgemm(True, False, K, N, rows, N, True)
        add("colsum_kernel")
        if dx:
            sgemm(False, True, rows, K, N, K, False)

    def pack_mma(row_tile):
        add("pack_rows_kernel")
        mma(row_tile)

    ce = "ce_kernel<%s>" % ("true" if weighted else "false")
    add("reciprocal_kernel")
    # initialize, per image
    add("mean_L_kernel")
    add("dropout2d_kernel", 3)
    for _ in range(2):
        dense_fwd(NI, D, I)
        dense_fwd(NI, I, H)
    if G > 1:
        add("expand_rows_kernel", 2)
    if tc:
        add("repack_weight_kernel")
        add("repack_bias_kernel")
    for i in range(4):
        if tc_fwd[i]:
            add("repack_weight_kernel")
            add("repack_bias_kernel")
        if tc_dx[i]:
            add("pack_rows_kernel")
    if tcv:
        add("pack_rows_kernel")
    # forward through time
    for t in range(T):
        if tc:                                               # (main or side stream)
            pack_mma(128)
        else:
            add("dropout2d_kernel")
            dense_fwd(BLi, D, A)
        if pk_fwd[0]:
            add("dropout_pack_kernel")
            mma(rt)
        else:
            add("dropout2d_kernel")
            if tc_fwd[0]:
                pack_mma(rt)
            else:
                dense_fwd(B, H, A)
        if f["att_fused"]:
            add("att_logits_kernel")
        else:
            add("att_temp_kernel")
            add("rowdot_kernel")
            if G > 1:
                add("expand_rows_kernel")
        if f["fuse_softmax_fwd"]:
            add("softmax_context_fwd4_kernel")
        else:
            add("softmax_rows_kernel")
            add("context_fwd4_kernel" if D % 4 == 0 else "context_fwd_kernel")
        if t == 0:
            add("gather_rows_kernel")
        add("concat3_drop_kernel")
        if pk_fwd[1]:
            mma(rt)
        elif tc_fwd[1]:
            pack_mma(rt)
        else:
            sgemm(False, False, B, 4 * H, XL, 4 * H, False)
        add("lstm_fwd_kernel")
        if dec_all:
            continue
        add("concat3_drop_kernel")
        for i, (K, N) in ((2, (XD, Dd)), (3, (Dd, V))):
            if tc_fwd[i]:
                pack_mma(rt)
            else:
                dense_fwd(B, K, N)
            if i == 2:
                add("dropout2d_kernel")
        add(ce)
    if dec_all:
        add("concat3_drop_kernel")
        pack_mma(f["all_rt"])
        add("dropout_steps_kernel")
        pack_mma(f["all_rt"])
        add(ce)
    add("coverage_loss_kernel")
    add("sumsq_kernel", NUM_REGULARISED)
    # backward through time
    if dec_all:
        pack_mma(f["all_rt"])
        add("drop_tanh_bwd_kernel")
        pack_mma(f["all_rt"])
    for t in range(T):
        if not dec_all:
            if tcv:
                pack_mma(rt)
            if stack:
                if not tcv:
                    sgemm(False, True, B, Dd, V, Dd, False)
            else:
                dense_bwd(B, Dd, V, dx=not tcv)
            add("drop_tanh_bwd_kernel")
            if tc_dx[2]:
                pack_mma(rt)
                if not stack:
                    dense_bwd(B, XD, Dd, dx=False)
            else:
                dense_bwd(B, XD, Dd, dx=True)
        add("split3_drop_kernel")
        add("lstm_bwd_kernel")
        if tc_dx[1]:
            if pk_dx[1]:
                mma(rt)
            else:
                pack_mma(rt)
            if not stack:
                dense_bwd(B, XL, 4 * H, dx=False)
        else:
            dense_bwd(B, XL, 4 * H, dx=True)
        add("split3_drop_kernel")
        add("context_bwd_kernel")
        if not f["fuse_softmax_bwd"]:
            add("softmax_bwd_kernel")
        if f["att_fused"]:
            add("att_bwd_grouped_kernel" if G > 1 else ("att_bwd_fused_wave_kernel" if wave else "att_bwd_fused_kernel"))
        else:
            for n in ("att_temp_kernel", "colsum_kernel", "att_dtemp_kernel", "segsum_kernel", "tanh_bwd_kernel"):
                add(n)
            if G > 1:
                add("group_sum_kernel")
        if tc:
            add("repack_weight_kernel", 2)
            mma(128)
            if not f["att_fused"]:
                add("colsum_kernel")
        else:
            add("dropout2d_kernel")
            dense_bwd(BLi, D, A, dx=False)
        if tc_dx[0]:
            if pk_dx[0]:
                add("tanh_bwd_pack_kernel")
                mma(rt)
            else:
                add("tanh_bwd_kernel")
                pack_mma(rt)
            if not stack:
                dense_bwd(B, H, A, dx=False)
        else:
            add("tanh_bwd_kernel")
            dense_bwd(B, H, A, dx=True)
        add("dropout2d_kernel")
    add("scatter_add_rows_kernel")
    if stack:
        for _ in range(4):
            add("repack_weight_kernel", 2)
            mma(128)
            add("colsum_kernel")
    # initialize backward
    add("copy2d_kernel")
    if G > 1:
        add("group_sum_kernel", 2)
    for _ in range(2):
        dense_bwd(NI, I, H, dx=True)
        add("drop_tanh_bwd_kernel")
        dense_bwd(NI, D, I, dx=False)
    return f, k


def kernel_key(name, grid=None):
    """The plan's name of a profiled kernel ("sgemm_kernel<false,true>+splitk", "lin_mma_kernel<2>", "ce_kernel<true>",
    or a base name), or None for a kernel that is not one of the training step's.  Demangled or mangled names;
    grid: (x, y, z) of the launch, when the profiler recorded it."""
    base, args = None, []
    if name.startswith("_Z"):
        name = name.replace("12_GLOBAL__N_1", "")   # (the anonymous namespace: its trailing 1 runs into the next length)
        for m in re.finditer(r"(\d+)(?=[A-Za-z_])", name):
            n, s = int(m.group(1)), m.end()
            if name[s:s + n] in _KNOWN:
                base, rest = name[s:s + n], name[s + n:]
                if rest.startswith("I"):
                    args = [("%s" % v) if kind == "i" else _BOOL[v] for kind, v in re.findall(r"L([bi])(\d+)E", rest.split("EE")[0] + "E")]
                break
    else:
        flat = name.replace(" ", "")
        for m in re.finditer(r"([A-Za-z_]\w*)(<[^<>]*>)?", flat):
            if m.group(1) in _KNOWN:
                base = m.group(1)
                args = m.group(2)[1:-1].split(",") if m.group(2) else []
                break
    if base is None:
        return None
    if base == "lin_mma_kernel":
        return "lin_mma_kernel<%s>" % args[0]
    if base in ("sgemm_kernel", "ce_kernel"):
        split = base == "sgemm_kernel" and grid is not None and len(grid) > 2 and grid[2] > 1
        return "%s<%s>%s" % (base, ",".join(args), "+splitk" if split else "")
    return base


def _merge_splits(c):
    out = Counter()
    for k, v in c.items():
        out[k.replace("+splitk", "")] += v
    return out


def plan_diff(launches, records):
    """'' if the kernels of `records` [(name, grid or None)] are the plan's launches, else what differs.  Where the
    profiler gave no grid for some sgemm_kernel launch, the split-K refinement is compared on neither side."""
    got = Counter()
    grids_known = all(g is not None for n, g in records if kernel_key(n) and kernel_key(n).startswith("sgemm"))
    for n, g in records:
        key = kernel_key(n, g)
        if key:
            got[key] += 1
    want = Counter(launches)
    if not grids_known:
        got, want = _merge_splits(got), _merge_splits(want)
    if got == want:
        return ""
    missing, extra = want - got, got - want
    return "missing %s; unexpected %s" % (dict(sorted(missing.items())), dict(sorted(extra.items())))
