"""CaptionGenerator — the reference's model/driver call surface for the decode path
(model.py:190-356 build_rnn, base_model.py:163-240 beam_search, :257-278 load) on top of
libsat_b200.so.

Mapping to the reference (SURVEY.md §8b):
  CaptionGenerator(config)                         main.py:48,61,69
  .load(sess, model_file) / .set_weights(dict)     base_model.py:257-278
  .initialize(contexts) -> (memory, output)        sess.run([initial_memory, initial_output]) base_model.py:168-170
  .decode_step(contexts, last_word, last_memory, last_output) -> (memory, output, probs)
                                                   sess.run([memory, output, probs], ...)     base_model.py:207-212
  .beam_search(contexts, ...) -> per image list of CaptionData(sentence, score)
                                                   base_model.py:163-240
  .decode_loop(contexts, T, forced_words)          the unrolled loop of model.py:258-312 (greedy / teacher forced)
  .sample(contexts, num_samples, temperature)      the same loop with each word drawn from softmax(logits / temperature)
The one intentional deviation: precomputed contexts (conv features) take the place of
image files, because the CNN is out of scope.  `sess` arguments are accepted and ignored.

numpy in -> numpy out goes through the *_host C entry points (host<->device copies
inside the call, like a sess.run).  torch CUDA tensors in -> torch CUDA tensors out stays
on the device and is asynchronous on `self.stream`.
"""
import ctypes as C

import numpy as np

from .lib import OPTIMIZER_KINDS, Dims, Optimizer, check, load_library


def weight_shapes(config):
    """TF variable names (without ':0') and shapes of the decoder, as tf.layers.dense /
    LSTMCell / get_variable create them (utils/nn.py:96-105, model.py:219-230)."""
    D, E, H, V = config.dim_ctx, config.dim_embedding, config.num_lstm_units, config.vocabulary_size
    A, Dd, I, L = (config.dim_attend_layer, config.dim_decode_layer, config.dim_initalize_layer,
                   config.num_ctx)
    s = {"word_embedding/weights": (V, E)}
    if config.num_initalize_layers == 1:
        for n in ("a", "b"):
            s["initialize/fc_%s/kernel" % n] = (D, H)
            s["initialize/fc_%s/bias" % n] = (H,)
    else:
        for n in ("a", "b"):
            s["initialize/fc_%s1/kernel" % n] = (D, I)
            s["initialize/fc_%s1/bias" % n] = (I,)
            s["initialize/fc_%s2/kernel" % n] = (I, H)
            s["initialize/fc_%s2/bias" % n] = (H,)
    if config.num_attend_layers == 1:
        s["attend/fc_a/kernel"] = (D, 1)
        s["attend/fc_b/kernel"] = (H, L)
    else:
        s["attend/fc_1a/kernel"] = (D, A)
        s["attend/fc_1a/bias"] = (A,)
        s["attend/fc_1b/kernel"] = (H, A)
        s["attend/fc_1b/bias"] = (A,)
        s["attend/fc_2/kernel"] = (A, 1)
    s["lstm/lstm_cell/kernel"] = (D + E + H, 4 * H)
    s["lstm/lstm_cell/bias"] = (4 * H,)
    if config.num_decode_layers == 1:
        s["decode/fc/kernel"] = (H + D + E, V)
        s["decode/fc/bias"] = (V,)
    else:
        s["decode/fc_1/kernel"] = (H + D + E, Dd)
        s["decode/fc_1/bias"] = (Dd,)
        s["decode/fc_2/kernel"] = (Dd, V)
        s["decode/fc_2/bias"] = (V,)
    return s


class CaptionData(object):
    """utils/misc.py:38-60 (memory/output are not returned to the host).  With beam_search(with_attention=True):
    alphas [len, L] (where the model looked for each word) and word_probs [len] (score = their product)."""
    __slots__ = ("sentence", "score", "complete", "alphas", "word_probs")

    def __init__(self, sentence, score, complete, alphas=None, word_probs=None):
        self.sentence, self.score, self.complete = sentence, score, complete
        self.alphas, self.word_probs = alphas, word_probs

    def __repr__(self):
        return "CaptionData(score=%.6g, sentence=%s)" % (self.score, self.sentence)


class CaptionGenerator(object):
    def __init__(self, config, max_batch=None, device=None):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("sat_b200 needs an NVIDIA H100 (sm_90a): no CUDA device visible, no CPU path")
        self.torch = torch
        self.config = config
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.lib = load_library()
        beam = max(1, int(getattr(config, "beam_size", 1)))
        if max_batch is None:
            max_batch = int(config.batch_size) * beam
        self.max_batch = int(max_batch)
        d = Dims(self.max_batch, config.num_ctx, config.dim_ctx, config.num_lstm_units, config.dim_embedding,
                 config.dim_attend_layer, config.dim_decode_layer, config.dim_initalize_layer,
                 config.vocabulary_size, config.num_attend_layers, config.num_decode_layers,
                 config.num_initalize_layers, config.max_caption_length, beam)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            check(self.lib, self.lib.sat_create(C.byref(d), C.byref(self._h)))
            # high priority: with cross-batch overlap ("xbatch") the decode steps must win SMs over the prologue of
            # the next batch, which the library runs on a default-priority stream of its own
            self.stream = torch.cuda.Stream(self.device, priority=-1)
        self._shapes = weight_shapes(config)
        self._keep = {}
        self._sample_calls = 0   # seeds of sample(seed=None): a fresh instance repeats its sequence

    # ------------------------------------------------------------------ plumbing
    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None and self._h.value:
                self.lib.sat_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    close = __del__

    def _st(self):
        return C.c_void_p(self.stream.cuda_stream)

    def _check(self, rc):
        check(self.lib, rc)

    def set_option(self, key, value):
        self._check(self.lib.sat_set_option(self._h, key.encode(), int(value)))

    def info(self, key):
        v = C.c_int64()
        self._check(self.lib.sat_get_info(self._h, key.encode(), C.byref(v)))
        return v.value

    @staticmethod
    def _p(t):
        return C.c_void_p(0 if t is None else t.data_ptr())

    def _dev(self, x, dtype):
        """torch CUDA tensor (contiguous, right dtype) from numpy / torch input."""
        torch = self.torch
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        return x.to(device=self.device, dtype=dtype).contiguous()

    def _buf(self, name, shape, dtype):
        """Persistent device buffer (stable address, so loop/beam CUDA graphs are replayed, not rebuilt).
        The returned tensor is overwritten by the next call of the same kind."""
        key = (name, tuple(shape), dtype)
        t = self._keep.get(key)
        if t is None:
            t = self.torch.empty(*shape, dtype=dtype, device=self.device)
            self._keep[key] = t
        return t

    def _sync_in(self):
        # make work queued on the caller's current stream visible to ours
        self.stream.wait_stream(self.torch.cuda.current_stream(self.device))

    def _sync_out(self):
        self.torch.cuda.current_stream(self.device).wait_stream(self.stream)

    # ------------------------------------------------------------------ weights
    def variable_names(self):
        return list(self._shapes)

    def set_weights(self, weights, sync=True):
        """weights: {tf_variable_name[:0]: ndarray/tensor} in the reference layouts.  sync=False skips the final host
        synchronisation: only for CUDA tensors that outlive the queued repack (e.g. views of the training parameters)."""
        torch = self.torch
        given = {(k[:-2] if k.endswith(":0") else k): v for k, v in weights.items()}
        keep = []
        for name, shp in self._shapes.items():
            if name not in given:
                continue
            w = self._dev(given[name], torch.float32)
            got = tuple(w.shape)
            # like tf.assign: the shape must match.  The only tolerated differences are a vector given as a
            # one-row / one-column matrix or the reverse (biases [n] vs [1,n]; attend/fc_2, fc_a [n,1] vs [n]).
            vec_ok = (len(shp) == 1 or 1 in shp) and sorted(d for d in got if d != 1) == sorted(d for d in shp if d != 1)
            if got != tuple(shp) and not vec_ok:
                raise ValueError("%s: expected shape %s, got %s" % (name, shp, got))
            rows, cols = (shp[0], shp[1]) if len(shp) == 2 else (1, shp[0])
            self._sync_in()                     # (the upload / cast above ran on the caller's stream: a stream wait, no host sync)
            self._check(self.lib.sat_set_weight(self._h, name.encode(), self._p(w), rows, cols, self._st()))
            keep.append(w)                      # the repack is asynchronous: the source lives until the stream is past it
        if keep and sync:
            self.stream.synchronize()           # ONE synchronisation per call (it was one per variable)
        return self.lib.sat_weights_missing(self._h)

    def load(self, sess=None, model_file=None):
        """base_model.py:257-278: np.load of the pickled {var.name: ndarray} dict."""
        data = np.load(model_file, encoding="latin1", allow_pickle=True).item()
        missing = self.set_weights(data)
        return len(self._shapes) - missing

    # ------------------------------------------------------------------ training step (base_model.py:39-68)
    def train_setup(self, batch_size, num_steps=None, weights=None, group=1):
        """Allocate the flat parameter / gradient / Adam buffers for training with `batch_size` images per
        process and `num_steps` unrolled time steps (config.max_caption_length).  `weights`: initial values
        (dict of TF variable names); default U(-s, s) kernels and zero biases like the reference
        (utils/nn.py:29-31).  The reference's trainable set (model.py:225: embedding, dense layers, LSTM).
        group > 1: `group` captions per image (batch_size * group rows, row r of image r // group) with the image's
        contexts shared by its rows (sat_train_init_grouped): train_forward_backward(..., group=group), scst_step."""
        torch = self.torch
        cfg = self.config
        T = int(num_steps or cfg.max_caption_length)
        group = int(group)
        if group == 1:
            self._check(self.lib.sat_train_init(self._h, int(batch_size), T, float(cfg.fc_drop_rate),
                                                float(cfg.lstm_drop_rate), float(cfg.attention_loss_factor),
                                                float(cfg.fc_kernel_regularizer_scale)))
        else:
            self._check(self.lib.sat_train_init_grouped(self._h, int(batch_size), group, T, float(cfg.fc_drop_rate),
                                                        float(cfg.lstm_drop_rate), float(cfg.attention_loss_factor),
                                                        float(cfg.fc_kernel_regularizer_scale)))
        self._train_BT = (int(batch_size) * group, T)
        self._train_group = (int(batch_size), group)
        n = self.lib.sat_train_num_vars(self._h)
        self._train_vars = []
        total = C.c_int64()
        for i in range(n):
            name, off, rows, cols, reg = C.c_char_p(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
            self._check(self.lib.sat_train_var(self._h, i, C.byref(name), C.byref(off), C.byref(rows), C.byref(cols),
                                               C.byref(reg), C.byref(total)))
            self._train_vars.append((name.value.decode(), off.value, rows.value, cols.value, bool(reg.value)))
        self.params = torch.zeros(total.value, device=self.device)
        # gradients + an 8-float tail in ONE buffer: the data-parallel step all-reduces it as a whole, so the loss sums
        # and the next batch's mask sum travel inside the gradient collective (tail: ce, accuracy, attention,
        # mask sum of the next batch)
        self._flat = torch.zeros(total.value + 8, device=self.device)
        self.grads = self._flat[:total.value]
        self._tail = self._flat[total.value:]
        from .parallel import StepCollective
        self._dp = StepCollective(self._flat, total.value)
        # optimizer slots (model.py:479-503): Adam m, v; RMSProp rms (starts at ONE like TF's), mg (centered), momentum;
        # Momentum accumulator; SGD none
        kind = getattr(cfg, "optimizer", "Adam")
        if kind not in OPTIMIZER_KINDS:
            raise ValueError("config.optimizer %r: expected one of %s" % (kind, sorted(OPTIMIZER_KINDS)))
        nslots = {"Adam": 2, "RMSProp": 3, "Momentum": 1, "SGD": 0}[kind]
        self.opt_slots = [torch.zeros_like(self.params) for _ in range(nslots)]
        if kind == "RMSProp":
            self._check(self.lib.sat_train_fill(self._h, self._p(self.opt_slots[0]), 1.0, self.params.numel(), self._st()))
            torch.cuda.synchronize(self.device)
        self.adam_m, self.adam_v = (self.opt_slots + [None, None])[:2] if kind == "Adam" else (None, None)
        self._train_losses = torch.zeros(4, device=self.device)
        self._train_norm = torch.zeros(1, device=self.device)
        self.global_step = 0
        if weights is None:
            g = torch.Generator(device="cpu").manual_seed(0)
            sc = cfg.fc_kernel_initializer_scale
            weights = {nm: (torch.zeros(r * c) if nm.endswith("/bias") else torch.rand(r * c, generator=g) * 2 * sc - sc)
                       for nm, _, r, c, _ in self._train_vars}
        self.train_load(weights)
        return self

    def _var_view(self, buf, name):
        for nm, off, r, c, _ in self._train_vars:
            if nm == name:
                shp = self._shapes[nm]
                return buf[off:off + r * c].view(*shp)
        raise KeyError(name)

    def train_load(self, weights):
        given = {(k[:-2] if k.endswith(":0") else k): v for k, v in weights.items()}
        for nm, off, r, c, _ in self._train_vars:
            if nm in given:
                self.params[off:off + r * c].copy_(self._dev(given[nm], self.torch.float32).reshape(-1))

    def train_state_dict(self, which="params"):
        """{tf variable name: tensor view} of the parameters ('params'), gradients ('grads') or Adam slots."""
        buf = dict(params=self.params, grads=self.grads, m=self.adam_m, v=self.adam_v)[which]
        return {nm: self._var_view(buf, nm) for nm, *_ in self._train_vars}

    def sync_inference_weights(self, sync=True):
        """Repack the trained parameters for the decode kernels (so beam_search / decode_step use them).  sync=False:
        no host synchronisation (the sources are views of the persistent self.params, which outlive the queued repack);
        the decode calls that follow on the same stream see the new weights."""
        return self.set_weights(self.train_state_dict("params"), sync=sync)

    def train_forward_backward(self, contexts, sentences, masks, seed=None, global_mask_sum=None, global_batch=None,
                               group=1, row_weights=None):
        """Forward + backward of one batch shard; fills self.grads (no regulariser term) and returns the device
        tensor of the four losses (cross_entropy, accuracy, attention, reg).  seed: see _step_seed.
        group > 1 (the group of train_setup): contexts [n_img, L, D] are shared by the `group` caption rows of each
        image (sentences / masks [n_img * group, T]).  row_weights [rows] (or None = 1) multiply each row's cross entropy
        and its gradient (sat_train_forward_backward_grouped)."""
        seed = self._step_seed(seed)
        torch = self.torch
        B, T = self._train_BT
        n_img, G = getattr(self, "_train_group", (B, 1))
        if int(group) != G:
            raise ValueError("group=%d, but train_setup was called with group=%d" % (int(group), G))
        if G > 1 or row_weights is not None:
            return self._train_forward_backward_grouped(contexts, sentences, masks, seed, global_mask_sum, global_batch,
                                                        row_weights)
        ctx = self._dev(contexts, torch.float32)
        sent = self._dev(sentences, torch.int32)
        mk = self._dev(masks, torch.float32)
        assert tuple(sent.shape) == (B, T) and tuple(mk.shape) == (B, T) and ctx.shape[0] == B
        gb = B if global_batch is None else int(global_batch)
        if isinstance(global_mask_sum, torch.Tensor):    # device scalar (float64 [1]): no host round trip
            gsum = global_mask_sum
            assert gsum.is_cuda and gsum.dtype == torch.float64 and gsum.numel() == 1
            self._sync_in()
            self._check(self.lib.sat_train_forward_backward_dsum(self._h, self._p(self.params), self._p(self.grads), self._p(ctx),
                                                                 self._p(sent), self._p(mk), B, T, int(seed), self._p(gsum), gb,
                                                                 self._p(self._train_losses), self._st()))
            self._sync_out()
            self._keep["train_in"] = (ctx, sent, mk, gsum)
            return self._train_losses
        gms = self._mask_sum(masks, mk) if global_mask_sum is None else float(global_mask_sum)
        self._sync_in()
        self._check(self.lib.sat_train_forward_backward(self._h, self._p(self.params), self._p(self.grads), self._p(ctx),
                                                        self._p(sent), self._p(mk), B, T, int(seed), gms, gb,
                                                        self._p(self._train_losses), self._st()))
        self._sync_out()
        self._keep["train_in"] = (ctx, sent, mk)
        return self._train_losses

    def _train_forward_backward_grouped(self, contexts, sentences, masks, seed, global_mask_sum, global_batch, row_weights):
        torch = self.torch
        B, T = self._train_BT
        n_img, G = self._train_group
        ctx = self._dev(contexts, torch.float32)
        sent = self._dev(sentences, torch.int32)
        mk = self._dev(masks, torch.float32)
        if tuple(sent.shape) != (B, T) or tuple(mk.shape) != (B, T) or ctx.shape[0] != n_img:
            raise ValueError("grouped step: contexts [%d, L, D] and sentences / masks [%d, %d] expected, got %s, %s, %s"
                             % (n_img, B, T, tuple(ctx.shape), tuple(sent.shape), tuple(mk.shape)))
        w = None if row_weights is None else self._dev(row_weights, torch.float32).reshape(-1)
        if w is not None and w.numel() != B:
            raise ValueError("row_weights: %d values for %d rows" % (w.numel(), B))
        gb = B if global_batch is None else int(global_batch)
        if isinstance(global_mask_sum, torch.Tensor):
            gsum = global_mask_sum
            assert gsum.is_cuda and gsum.dtype == torch.float64 and gsum.numel() == 1
        else:   # (the grouped entry reads the sum from device memory)
            v = self._mask_sum(masks, mk) if global_mask_sum is None else float(global_mask_sum)
            gsum = self._buf("train_msum", (1,), torch.float64)
            gsum.fill_(v)
        self._sync_in()
        self._check(self.lib.sat_train_forward_backward_grouped(self._h, self._p(self.params), self._p(self.grads), self._p(ctx),
                                                                n_img, G, self._p(sent), self._p(mk), self._p(w), T, int(seed),
                                                                self._p(gsum), gb, self._p(self._train_losses), self._st()))
        self._sync_out()
        self._keep["train_in"] = (ctx, sent, mk, w, gsum)
        return self._train_losses

    def _mask_sum(self, masks, mk):
        """Sum of the caption masks as a host float without stalling the device when it can be avoided: host arrays are
        summed on the host; a device tensor is summed once and remembered until it is modified."""
        torch = self.torch
        if isinstance(masks, np.ndarray):
            return float(masks.astype(np.float64).sum())
        if isinstance(masks, torch.Tensor) and not masks.is_cuda:
            return float(masks.double().sum())
        key = (mk.data_ptr(), mk._version, tuple(mk.shape))
        hit = self._keep.get("mask_sum")
        if hit is None or hit[0] != key:
            hit = (key, float(mk.sum().item()))
            self._keep["mask_sum"] = hit
        return hit[1]

    def learning_rate(self, step=None):
        """The staircase-decayed rate of model.py:466-476 at global step `step` (what the reference writes to its
        "learning_rate" summary): initial * factor ** floor(step / num_steps_per_decay)."""
        cfg = self.config
        step = self.global_step if step is None else int(step)
        f = float(getattr(cfg, "learning_rate_decay_factor", 1.0))
        if f >= 1.0:
            return float(cfg.initial_learning_rate)
        return float(cfg.initial_learning_rate) * f ** (step // int(cfg.num_steps_per_decay))

    def train_apply(self):
        """Regulariser gradient + global-norm clip + the configured optimizer (model.py:479-503) on self.grads (already
        summed over ranks).  See Config.apply_learning_rate_decay for which rate the optimizer gets."""
        cfg = self.config
        lr = self.learning_rate(self.global_step) if getattr(cfg, "apply_learning_rate_decay", False) \
            else float(cfg.initial_learning_rate)
        self.global_step += 1
        o = Optimizer(OPTIMIZER_KINDS[getattr(cfg, "optimizer", "Adam")], lr, float(cfg.beta1), float(cfg.beta2),
                      float(cfg.epsilon), float(getattr(cfg, "decay", 0.9)), float(getattr(cfg, "momentum", 0.0)),
                      int(bool(getattr(cfg, "centered", True))), int(bool(getattr(cfg, "use_nesterov", True))),
                      float(cfg.clip_gradients))
        slots = [self._p(t) for t in self.opt_slots] + [C.c_void_p(0)] * 3
        self._sync_in()
        self._check(self.lib.sat_train_apply_opt(self._h, self._p(self.params), self._p(self.grads), slots[0], slots[1],
                                                 slots[2], self.global_step, C.byref(o), self._p(self._train_norm), self._st()))
        self._sync_out()
        return self._train_norm

    # TF names of the optimizer slot variables, in slot order (graph fixture: optimizer/OptimizeLoss/<var>/Adam, .../Adam_1)
    _SLOT_SUFFIX = {"Adam": ["Adam", "Adam_1"], "RMSProp": ["RMSProp", "RMSProp_1", "RMSProp_2"], "Momentum": ["Momentum"],
                    "SGD": []}

    def save(self, save_dir=None):
        """base_model.py:242-255: np.save of {variable name + ':0': ndarray} over the global variables (the decoder's 20
        trainable tensors, global_step, the optimizer slots under their TF names, beta powers for Adam) to
        <save_dir>/<global_step>.npy, plus config.pickle with the step.  The file loads back through load() here and
        through the reference's own load() (which assigns by variable name)."""
        import copy
        import os
        import pickle
        cfg = self.config
        kind = getattr(cfg, "optimizer", "Adam")
        d = save_dir or getattr(cfg, "save_dir", "./models/")
        os.makedirs(d, exist_ok=True)
        self.torch.cuda.synchronize(self.device)
        data = {nm + ":0": self._var_view(self.params, nm).detach().cpu().numpy().copy() for nm, *_ in self._train_vars}
        data["global_step:0"] = np.int32(self.global_step)
        for slot, suffix in zip(self.opt_slots, self._SLOT_SUFFIX[kind]):
            for nm, *_ in self._train_vars:
                data["optimizer/OptimizeLoss/%s/%s:0" % (nm, suffix)] = self._var_view(slot, nm).detach().cpu().numpy().copy()
        if kind == "Adam":
            data["optimizer/OptimizeLoss/beta1_power:0"] = np.float32(float(cfg.beta1) ** (self.global_step + 1))
            data["optimizer/OptimizeLoss/beta2_power:0"] = np.float32(float(cfg.beta2) ** (self.global_step + 1))
        path = os.path.join(d, "%d.npy" % self.global_step)
        np.save(path, data, allow_pickle=True)
        cfg_ = copy.copy(cfg)
        cfg_.global_step = self.global_step
        with open(os.path.join(d, "config.pickle"), "wb") as f:
            pickle.dump(cfg_, f)
        return path

    def train_restore(self, model_file):
        """Resume training from a file written by save() (or by the reference: same keys): parameters, optimizer slots
        and global_step.  Returns the number of tensors restored."""
        data = np.load(model_file, encoding="latin1", allow_pickle=True).item()
        kind = getattr(self.config, "optimizer", "Adam")
        n = 0
        for nm, off, r, c, _ in self._train_vars:
            if nm + ":0" in data:
                self.params[off:off + r * c].copy_(self._dev(data[nm + ":0"], self.torch.float32).reshape(-1)); n += 1
            for slot, suffix in zip(self.opt_slots, self._SLOT_SUFFIX[kind]):
                k = "optimizer/OptimizeLoss/%s/%s:0" % (nm, suffix)
                if k in data:
                    slot[off:off + r * c].copy_(self._dev(data[k], self.torch.float32).reshape(-1)); n += 1
        if "global_step:0" in data:
            self.global_step = int(data["global_step:0"])
        return n

    def _step_seed(self, seed):
        """Dropout seed of the next optimisation step.  None (default): fresh masks every step, derived from the
        step counter and `config.dropout_seed` (the reference draws new unseeded masks every step with
        fc_drop_rate / lstm_drop_rate, model.py:231-236, nn.py:111-114); an explicit 0 switches dropout OFF (the C ABI's
        convention); any other value is used as given."""
        if seed is None:
            base = int(getattr(self.config, "dropout_seed", 0x5A17B200)) & 0xFFFFFFFF
            return ((base << 20) ^ (self.global_step + 1)) or 1
        return int(seed)

    def allreduce_gradients(self):
        """Sum the flat gradient buffer (with its scalar tail) over the ranks (what StepCollective.reduce does inside
        train_step; kept for callers that drive sat_train_forward_backward / train_apply themselves)."""
        import torch.distributed as dist
        dist.all_reduce(self._flat)

    def _shard_forward_backward(self, mk, seed, next_masks, fb):
        """The data-parallel protocol of one step around fb(seed, global_mask_sum, global_batch) -> losses [4] (device).
        Single process: fb gets the step's seed, None (the local mask sum) and the row count."""
        import torch.distributed as dist
        torch = self.torch
        B, T = self._train_BT
        world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
        if world > 1:
            # ONE collective per step: the flat buffer [gradients | ce, accuracy, attention sums | mask sum of the NEXT
            # batch].  The whole-batch mask sum (model.py:316-318 divides by it, so it is needed BEFORE the backward
            # pass) of this batch therefore arrived with the previous step's collective; only the first step of a run —
            # or a batch whose masks were not announced (`next_masks`) — pays a separate 8-byte all-reduce.  Everything
            # stays on the device and in stream order: the host can queue step i+1 while step i runs.
            nxt = mk if next_masks is None else self._dev(next_masks, torch.float32)
            gsum = self._dp.global_mask_sum(mk)
            seed = self._step_seed(seed)
            seed = seed + 0x1000003 * dist.get_rank() if seed else 0   # rank-offset mask streams (0 stays "off")
            losses = fb(seed, gsum, B * world)
            return torch.cat([self._dp.reduce(losses, nxt, announced=next_masks is not None), losses[3:4]])   # the single collective of the step
        return fb(self._step_seed(seed), None, B)

    def scst_step(self, contexts, reward_fn, num_samples=5, baseline="greedy", temperature=1.0, seed=None,
                  sample_seed=None, sync=True, references=None):
        """One self-critical (SCST) policy-gradient step on a shard of images.

          1. the decode weights are refreshed from the training parameters (no host synchronisation);
          2. num_samples = K captions per image are drawn (sample_device, sample_seed);
          3. baseline "greedy": the greedy caption of each image is decoded as well;
          4. reward_fn(captions) is called once: captions[i] is the list of image i's word-id lists, each cut after its
             first eos_id: the K samples, then the greedy caption for baseline "greedy".  It returns rewards [n, K + 1]
             ("greedy") or [n, K] ("mean");
          5. advantages = sample reward - baseline: the greedy caption's reward, or for "mean" the mean reward of the
             image's other K - 1 samples (captions.scst_advantages);
          6. the caption masks and their sum are built on the device (sat_caption_masks);
          7. the grouped step with the advantages as row weights minimises sum_r A_r sum_t m_rt (-log p(w_rt)) / sum m
             (plus the attention loss), with the image's contexts shared by its K rows; seed: the training dropout
             (see _step_seed; 0 = off, which makes the step exactly on-policy: sampling runs without dropout);
          8. train_apply (clip + optimizer).
        Needs train_setup(n_img, group=num_samples).  With torch.distributed initialised, the mask sum of the whole
        batch and the gradient sum travel in train_step's single collective.  Returns the losses, the mean sample
        reward, the mean baseline reward and the gradient norm (sync=False: the losses [4] and the squared gradient
        norm [1] as device tensors, the rewards as floats).
        Built-in reward: reward_fn = a CiderD instance and references = this batch's reference captions [n, R, T_ref]
        (device or host, -1 padded; R <= 8, T_ref <= 64).  Steps 4-5 then run on the device, in stream order: the K
        samples and the greedy caption of each image are scored by sat_cider_d, and the advantages follow from the
        scores in float64 (captions.scst_advantages_torch) into the row weights.  Nothing waits for the host, so with
        sync=False the call returns once the step is queued, and the sample and baseline rewards are 0-dim float64
        device tensors instead of floats."""
        from .captions import cut_after_eos, scst_advantages, scst_advantages_torch
        from .cider import CiderD
        torch = self.torch
        device_reward = isinstance(reward_fn, CiderD)
        if device_reward and references is None:
            raise ValueError("scst_step with a CiderD reward needs this batch's references [n, R, T_ref]")
        cfg = self.config
        K = int(num_samples)
        if baseline not in ("greedy", "mean"):
            raise ValueError("baseline must be 'greedy' or 'mean', got %r" % (baseline,))
        if K < 1 or (baseline == "mean" and K < 2):
            raise ValueError("num_samples=%d: at least 1 (baseline 'greedy') or 2 (baseline 'mean')" % K)
        ctx = self._dev(contexts, torch.float32)
        n = int(ctx.shape[0])
        if getattr(self, "_train_group", None) != (n, K):
            raise ValueError("scst_step on %d images x %d samples needs train_setup(%d, group=%d)" % (n, K, n, K))
        rows = n * min(K, self.SAMPLE_GROUP)
        if rows > self.max_batch:
            raise ValueError("sampling %d images x %d captions per call needs max_batch >= %d (the handle has %d)"
                             % (n, min(K, self.SAMPLE_GROUP), rows, self.max_batch))
        B, T = self._train_BT
        eos = int(cfg.eos_id)
        self.sync_inference_weights(sync=False)
        tokens, _ = self.sample_device(ctx, K, T, temperature, sample_seed, want_word_probs=False)
        sent = self._buf("scst_sent", (B, T), torch.int32)
        with torch.cuda.stream(self.stream):
            sent.copy_(tokens.reshape(B, T))
        greedy = self.loop_device(ctx, T)[0] if baseline == "greedy" else None
        w = self._buf("scst_w", (B,), torch.float32)
        if device_reward:
            with torch.cuda.stream(self.stream):
                cand = tokens if greedy is None else torch.cat([tokens, greedy[:, None, :]], 1)
            rewards = reward_fn.scores(cand, references, stream=self.stream)
            with torch.cuda.stream(self.stream):
                adv, r_sample, r_base = scst_advantages_torch(rewards, K, baseline)
                w.copy_(adv.reshape(-1))
        else:
            self.stream.synchronize()
            toks = sent.cpu().numpy().reshape(n, K, T)
            gt = greedy.cpu().numpy() if greedy is not None else None
            caps = [[cut_after_eos(toks[i, k], eos) for k in range(K)] + ([cut_after_eos(gt[i], eos)] if gt is not None else [])
                    for i in range(n)]
            adv, r_sample, r_base = scst_advantages(reward_fn(caps), K, baseline)
            w.copy_(torch.from_numpy(np.ascontiguousarray(adv.reshape(-1), dtype=np.float32)))
        mk = self._buf("scst_masks", (B, T), torch.float32)
        msum = self._buf("scst_msum", (1,), torch.float64)
        self._sync_in()
        self._check(self.lib.sat_caption_masks(self._p(sent), B, T, eos, self._p(mk), self._p(msum), self._st()))
        self._sync_out()
        torch.autograd.graph.increment_version(mk)   # (written in place by the library: new masks for StepCollective)
        losses = self._shard_forward_backward(
            mk, seed, None,
            lambda sd, gsum, gb: self.train_forward_backward(ctx, sent, mk, sd, msum if gsum is None else gsum, gb,
                                                             group=K, row_weights=w))
        norm2 = self.train_apply()
        if not sync:
            return dict(losses=losses, gradient_norm2=norm2, sample_reward=r_sample, baseline_reward=r_base)
        ce, acc, att, reg = [float(x) for x in losses.tolist()]
        return dict(cross_entropy_loss=ce, accuracy=acc, attention_loss=att, reg_loss=reg, total_loss=ce + att + reg,
                    sample_reward=float(r_sample), baseline_reward=float(r_base), gradient_norm=float(norm2.item()) ** 0.5,
                    global_step=self.global_step)

    def train_step(self, contexts, sentences, masks, seed=None, sync=True, next_masks=None):
        """One optimisation step (the sess.run(opt_op) of base_model.py:57-60) on this process's shard; with
        torch.distributed initialised the gradients are summed over the ranks by ONE all-reduce of the flat
        buffer (NCCL) and the losses are normalised by the global batch.  sync=False returns the device tensors
        (losses [4], squared gradient norm [1]) without reading them back, so that the host can queue the next step
        while this one runs (the reference reads its summary every step; a training loop rarely needs to).
        seed: see _step_seed (None = new dropout masks every step, 0 = dropout off).
        next_masks (data parallel): the masks the NEXT call will be given, if the input pipeline already has them: their
        sum then rides in this step's gradient collective and the next step starts without a collective of its own
        (a promise — only the shape is checked; default: the same masks tensor is expected again)."""
        torch = self.torch
        mk = self._dev(masks, torch.float32)
        losses = self._shard_forward_backward(
            mk, seed, next_masks,
            lambda sd, gsum, gb: self.train_forward_backward(contexts, sentences, mk, sd,
                                                             self._mask_sum(masks, mk) if gsum is None else gsum, gb,
                                                             group=self._train_group[1]))
        norm2 = self.train_apply()
        if not sync:
            return losses, norm2
        ce, acc, att, reg = [float(x) for x in losses.tolist()]
        bad = self.info("train_bad_ids")
        if bad:    # (TF's embedding_lookup / sparse softmax raise InvalidArgumentError on such ids)
            raise ValueError("%d word ids outside [0, %d) in `sentences`" % (bad, self.config.vocabulary_size))
        return dict(cross_entropy_loss=ce, accuracy=acc, attention_loss=att, reg_loss=reg, total_loss=ce + att + reg,
                    gradient_norm=float(norm2.item()) ** 0.5, learning_rate=self.learning_rate(self.global_step - 1),
                    global_step=self.global_step)

    # ------------------------------------------------------------------ device API
    def prepare(self, contexts, want_state=True):
        """Project the contexts once per image batch and run `initialize`.  contexts: CUDA tensor
        [B, L, D].  Returns (initial_memory, initial_output) CUDA tensors [B, H]."""
        torch = self.torch
        B = contexts.shape[0]
        c0 = torch.empty(B, self.config.num_lstm_units, device=self.device) if want_state else None
        h0 = torch.empty_like(c0) if want_state else None
        self._sync_in()
        self._check(self.lib.sat_prepare_contexts(self._h, self._p(contexts), B, self._p(c0), self._p(h0), self._st()))
        self._sync_out()
        self._keep["ctx"] = contexts
        return c0, h0

    def step_device(self, contexts, last_word, last_memory, last_output, want=("probs",)):
        torch = self.torch
        cfg = self.config
        B = contexts.shape[0]
        mem = torch.empty(B, cfg.num_lstm_units, device=self.device)
        out = torch.empty_like(mem)
        logits = torch.empty(B, cfg.vocabulary_size, device=self.device) if "logits" in want else None
        probs = torch.empty(B, cfg.vocabulary_size, device=self.device) if "probs" in want else None
        alpha = torch.empty(B, cfg.num_ctx, device=self.device) if "alpha" in want else None
        self._sync_in()
        self._check(self.lib.sat_decode_step(self._h, self._p(contexts), self._p(last_word), self._p(last_memory),
                                             self._p(last_output), self._p(mem), self._p(out), self._p(logits),
                                             self._p(probs), self._p(alpha), B, self._st()))
        self._sync_out()
        return dict(memory=mem, output=out, logits=logits, probs=probs, alpha=alpha)

    def loop_device(self, contexts, num_steps, forced_words=None, want_logits=False):
        torch = self.torch
        B = contexts.shape[0]
        tokens = self._buf("tokens", (B, num_steps), torch.int32)
        logits = (self._buf("loop_logits", (num_steps, B, self.config.vocabulary_size), torch.float32)
                  if want_logits else None)
        self._sync_in()
        self._check(self.lib.sat_decode_loop(self._h, self._p(contexts), B, num_steps, self._p(forced_words),
                                             self._p(tokens), self._p(logits), self._st()))
        self._sync_out()
        self._keep["loop"] = (contexts, forced_words, tokens, logits)
        return tokens, logits

    def loop_maps_device(self, contexts, num_steps, forced_words=None, want_logits=False, want_alphas=True,
                         want_word_probs=True):
        """sat_decode_loop_maps: tokens [B,T], logits [T,B,V] or None, alphas [T,B,L] or None, word_probs [B,T] or None
        (persistent buffers, overwritten by the next call of the same kind)."""
        torch = self.torch
        cfg = self.config
        B, T = contexts.shape[0], num_steps
        tokens = self._buf("tokens", (B, T), torch.int32)
        logits = self._buf("loop_logits", (T, B, cfg.vocabulary_size), torch.float32) if want_logits else None
        alphas = self._buf("loop_alphas", (T, B, cfg.num_ctx), torch.float32) if want_alphas else None
        wprobs = self._buf("loop_word_probs", (B, T), torch.float32) if want_word_probs else None
        self._sync_in()
        self._check(self.lib.sat_decode_loop_maps(self._h, self._p(contexts), B, T, self._p(forced_words),
                                                  self._p(tokens), self._p(logits), self._p(alphas), self._p(wprobs),
                                                  self._st()))
        self._sync_out()
        self._keep["loop"] = (contexts, forced_words, tokens, logits, alphas, wprobs)
        return tokens, logits, alphas, wprobs

    def loop_host_submit(self, contexts_host, num_steps, tokens_host, slot, forced_words_host=None):
        """Pipelined host-buffer greedy loop (sat_decode_loop_host_submit): upload on a copy stream, decode,
        download; returns at once.  Pair with loop_host_wait(slot).  Host tensors should be pinned."""
        B = contexts_host.shape[0]
        self._check(self.lib.sat_decode_loop_host_submit(self._h, self._p(contexts_host), B, num_steps,
                                                         self._p(forced_words_host), self._p(tokens_host), slot,
                                                         self._st()))
        self._keep["pipe%d" % slot] = (contexts_host, tokens_host, forced_words_host)

    def loop_host_wait(self, slot):
        self._check(self.lib.sat_decode_loop_host_wait(self._h, slot))
        return self._keep.pop("pipe%d" % slot)[1]

    def beam_device(self, contexts, beam_size, num_steps, eos_id, with_attention=False):
        """sat_beam_search (with_attention: sat_beam_search_maps, and alphas [n,beam,T,L], word_probs [n,beam,T]
        are appended to the returned tuple)."""
        torch = self.torch
        n = contexts.shape[0]
        sent = self._buf("b_sent", (n, beam_size, num_steps), torch.int32)
        lens = self._buf("b_lens", (n, beam_size), torch.int32)
        scores = self._buf("b_scores", (n, beam_size), torch.float64)
        nres = self._buf("b_nres", (n,), torch.int32)
        comp = self._buf("b_comp", (n,), torch.int32)
        self._sync_in()
        if with_attention:
            alphas = self._buf("b_alphas", (n, beam_size, num_steps, self.config.num_ctx), torch.float32)
            wprobs = self._buf("b_word_probs", (n, beam_size, num_steps), torch.float32)
            self._check(self.lib.sat_beam_search_maps(self._h, self._p(contexts), n, beam_size, num_steps, eos_id,
                                                      self._p(sent), self._p(lens), self._p(scores), self._p(nres),
                                                      self._p(comp), self._p(alphas), self._p(wprobs), self._st()))
            self._sync_out()
            self._keep["beam"] = (contexts, sent, lens, scores, nres, comp, alphas, wprobs)
            return sent, lens, scores, nres, comp, alphas, wprobs
        self._check(self.lib.sat_beam_search(self._h, self._p(contexts), n, beam_size, num_steps, eos_id,
                                             self._p(sent), self._p(lens), self._p(scores), self._p(nres),
                                             self._p(comp), self._st()))
        self._sync_out()
        self._keep["beam"] = (contexts, sent, lens, scores, nres, comp)
        return sent, lens, scores, nres, comp

    def _sample_seed(self, seed):
        """seed=None: the next seed of this instance's counter (successive calls differ, a fresh instance repeats)."""
        if seed is not None:
            return int(seed) & 0xFFFFFFFFFFFFFFFF
        self._sample_calls += 1
        return (self._sample_calls * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF

    # rows of one image per sat_sample_loop call (the attention kernels share an image's contexts between at most 4)
    SAMPLE_GROUP = 4

    def sample_device(self, contexts, num_samples, num_steps, temperature=1.0, seed=None, want_word_probs=True,
                      top_k=0, top_p=1.0):
        """sat_sample_loop: num_samples captions per image drawn from softmax(logits / temperature).  contexts: CUDA
        tensor [n, L, D].  Returns tokens [n, K, T] int32 and word_probs [n, K, T] (softmax(logits)[word] at
        temperature 1) or None (persistent buffers, overwritten by the next call of the same kind).
        More than SAMPLE_GROUP samples are drawn in groups of SAMPLE_GROUP per image: group c (samples 4c .. 4c+3) is
        a library call with seed + c * 0x9E3779B97F4A7C15 (mod 2^64), so group 0 is what a call with K <= 4 draws.
        top_k (0: off) / top_p (1: off): draw only among the top_k most probable words, and among the smallest set of
        those whose probability mass reaches top_p (sat_sample_loop_filtered); word_probs keep their meaning."""
        torch = self.torch
        n, K, T = contexts.shape[0], int(num_samples), int(num_steps)
        if K < 1:
            raise ValueError("num_samples must be >= 1")
        top_k, top_p = int(top_k), float(top_p)
        filtered = top_k != 0 or top_p != 1.0
        seed = self._sample_seed(seed)
        G = self.SAMPLE_GROUP
        parts = []
        self._sync_in()
        for c in range((K + G - 1) // G):
            kc = min(G, K - c * G)
            tokens = self._buf("s_tokens%d" % c, (n, kc, T), torch.int32)
            wprobs = self._buf("s_word_probs%d" % c, (n, kc, T), torch.float32) if want_word_probs else None
            sc = (seed + c * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
            if filtered:
                self._check(self.lib.sat_sample_loop_filtered(self._h, self._p(contexts), n, kc, T, float(temperature),
                                                              top_k, top_p, sc, self._p(tokens), self._p(wprobs),
                                                              self._st()))
            else:
                self._check(self.lib.sat_sample_loop(self._h, self._p(contexts), n, kc, T, float(temperature), sc,
                                                     self._p(tokens), self._p(wprobs), self._st()))
            parts.append((tokens, wprobs))
        if len(parts) > 1:   # (on our stream: the concatenation is ordered after every group)
            with torch.cuda.stream(self.stream):
                tokens = torch.cat([t for t, _ in parts], 1)
                wprobs = torch.cat([p for _, p in parts], 1) if want_word_probs else None
        else:
            tokens, wprobs = parts[0]
        self._sync_out()
        self._keep["sample"] = (contexts, tokens, wprobs, parts)
        return tokens, wprobs

    def sample(self, contexts, num_samples=1, temperature=1.0, seed=None, num_steps=None, eos_id=None, top_k=0,
               top_p=1.0):
        """Sampled captions: per image, num_samples CaptionData drawn word by word from softmax(logits / temperature).
        sentence: the words up to and including the first eos_id (default config.eos_id), or all num_steps words;
        complete: whether the caption reached eos_id; word_probs: the model's probability (temperature 1) of each of
        those words; score: their fp64 product (beam search's convention).  seed: a given seed reproduces the call bit
        for bit; None draws the next seed of this instance.  top_k / top_p: see sample_device (0 / 1: off).
        contexts: numpy or torch."""
        cfg = self.config
        T = int(num_steps or cfg.max_caption_length)
        eos = int(cfg.eos_id if eos_id is None else eos_id)
        ctx = self._dev(contexts, self.torch.float32)
        tokens, wprobs = self.sample_device(ctx, num_samples, T, temperature, seed, top_k=top_k, top_p=top_p)
        self.torch.cuda.synchronize(self.device)
        tokens, wprobs = tokens.cpu().numpy(), wprobs.cpu().numpy()
        results = []
        for k in range(tokens.shape[0]):
            caps = []
            for j in range(tokens.shape[1]):
                row = tokens[k, j]
                hit = np.flatnonzero(row == eos)
                ln = int(hit[0]) + 1 if hit.size else T
                wp = wprobs[k, j, :ln].copy()
                score = 1.0
                for x in wp:
                    score *= float(x)
                caps.append(CaptionData([int(w) for w in row[:ln]], score, bool(hit.size), word_probs=wp))
            results.append(caps)
        return results

    # ------------------------------------------------------------------ reference-shaped API
    def initialize(self, contexts, sess=None):
        """(initial_memory, initial_output) for a batch of contexts (base_model.py:168-170)."""
        is_np = isinstance(contexts, np.ndarray)
        ctx = self._dev(contexts, self.torch.float32)
        c0, h0 = self.prepare(ctx)
        if is_np:
            self.torch.cuda.synchronize(self.device)
            return c0.cpu().numpy(), h0.cpu().numpy()
        return c0, h0

    def decode_step(self, contexts, last_word, last_memory, last_output, sess=None, contexts_changed=True,
                    extras=False):
        """One sess.run([memory, output, probs], feed_dict=...) (base_model.py:207-212).

        numpy inputs: host path; `contexts_changed=False` tells the library the contexts are
        the ones of the previous call (the reference re-feeds them every call).
        torch CUDA inputs: device path.  `extras=True` also returns logits and alpha."""
        cfg = self.config
        if isinstance(contexts, np.ndarray) and not extras:
            B = contexts.shape[0]
            ctx = np.ascontiguousarray(contexts, np.float32)
            lw = np.ascontiguousarray(last_word, np.int32)
            lm = np.ascontiguousarray(last_memory, np.float32)
            lo = np.ascontiguousarray(last_output, np.float32)
            mem = np.empty((B, cfg.num_lstm_units), np.float32)
            out = np.empty_like(mem)
            probs = np.empty((B, cfg.vocabulary_size), np.float32)
            vp = lambda a: a.ctypes.data_as(C.c_void_p)
            self._check(self.lib.sat_decode_step_host(self._h, vp(ctx), 1 if contexts_changed else 0, vp(lw), vp(lm),
                                                      vp(lo), vp(mem), vp(out), vp(probs), B, self._st()))
            return mem, out, probs
        is_np = isinstance(contexts, np.ndarray)
        torch = self.torch
        ctx = self._dev(contexts, torch.float32)
        if contexts_changed or self._keep.get("ctx") is not ctx:
            self.prepare(ctx, want_state=False)
        r = self.step_device(ctx, self._dev(last_word, torch.int32), self._dev(last_memory, torch.float32),
                             self._dev(last_output, torch.float32),
                             want=("probs", "logits", "alpha") if extras else ("probs",))
        if is_np:
            torch.cuda.synchronize(self.device)
            r = {k: (v.cpu().numpy() if v is not None else None) for k, v in r.items()}
        if extras:
            return r
        return r["memory"], r["output"], r["probs"]

    def decode_loop(self, contexts, num_steps=None, forced_words=None, want_logits=False, want_alphas=False,
                    want_word_probs=False):
        """initialize + num_steps decode steps without host round trips; returns tokens [B,T]
        (argmax of every step, model.py:289) and optionally logits [T,B,V].

        want_alphas / want_word_probs: return a dict instead, with "tokens", "alphas" [B,T,L] (the attention map of
        the word emitted at step t) and/or "word_probs" [B,T] (probability of the word fed to step t+1: the argmax, or
        forced_words[:, t] when teacher forced, which scores a given caption), and "logits" [T,B,V] if want_logits."""
        cfg = self.config
        T = int(num_steps or cfg.max_caption_length)
        if want_alphas or want_word_probs:
            is_np = isinstance(contexts, np.ndarray)
            torch = self.torch
            ctx = self._dev(contexts, torch.float32)
            fw = None if forced_words is None else self._dev(forced_words, torch.int32)
            tokens, logits, alphas, wprobs = self.loop_maps_device(ctx, T, fw, want_logits, want_alphas, want_word_probs)
            r = dict(tokens=tokens)
            if want_logits:
                r["logits"] = logits
            if want_alphas:
                r["alphas"] = alphas.transpose(0, 1).contiguous()   # (a copy: the [T,B,L] buffer is reused)
            if want_word_probs:
                r["word_probs"] = wprobs
            if is_np:
                torch.cuda.synchronize(self.device)
                return {k: v.cpu().numpy() for k, v in r.items()}
            return r
        if isinstance(contexts, np.ndarray) and not want_logits:
            B = contexts.shape[0]
            ctx = np.ascontiguousarray(contexts, np.float32)
            fw = None if forced_words is None else np.ascontiguousarray(forced_words, np.int32)
            tokens = np.empty((B, T), np.int32)
            vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
            self._check(self.lib.sat_decode_loop_host(self._h, vp(ctx), B, T, vp(fw), vp(tokens), self._st()))
            return tokens
        is_np = isinstance(contexts, np.ndarray)
        torch = self.torch
        ctx = self._dev(contexts, torch.float32)
        fw = None if forced_words is None else self._dev(forced_words, torch.int32)
        tokens, logits = self.loop_device(ctx, T, fw, want_logits)
        if is_np:
            torch.cuda.synchronize(self.device)
            tokens = tokens.cpu().numpy()
            logits = logits.cpu().numpy() if logits is not None else None
        return (tokens, logits) if want_logits else tokens

    def beam_search(self, contexts, sess=None, vocabulary=None, eos_id=None, beam_size=None, num_steps=None,
                    with_attention=False):
        """base_model.py:163-240.  Returns, per image, the captions sorted by descending score
        (complete captions if any were completed, else the partial ones).  with_attention: every CaptionData also
        carries alphas [len, L] and word_probs [len] (runs on the device whatever the input)."""
        cfg = self.config
        beam = int(beam_size or cfg.beam_size)
        T = int(num_steps or cfg.max_caption_length)
        eos = int(cfg.eos_id if eos_id is None else eos_id)
        n = contexts.shape[0]
        maps = None
        if with_attention:
            ts = self.beam_device(self._dev(contexts, self.torch.float32), beam, T, eos, with_attention=True)
            self.torch.cuda.synchronize(self.device)
            sent, lens, scores, nres, comp, alphas, wprobs = [t.cpu().numpy() for t in ts]
            maps = (alphas, wprobs)
        elif isinstance(contexts, np.ndarray):
            ctx = np.ascontiguousarray(contexts, np.float32)
            sent = np.empty((n, beam, T), np.int32)
            lens = np.empty((n, beam), np.int32)
            scores = np.empty((n, beam), np.float64)
            nres = np.empty((n,), np.int32)
            comp = np.empty((n,), np.int32)
            vp = lambda a: a.ctypes.data_as(C.c_void_p)
            self._check(self.lib.sat_beam_search_host(self._h, vp(ctx), n, beam, T, eos, vp(sent), vp(lens),
                                                      vp(scores), vp(nres), vp(comp), self._st()))
        else:
            ts = self.beam_device(contexts, beam, T, eos)
            self.torch.cuda.synchronize(self.device)
            sent, lens, scores, nres, comp = [t.cpu().numpy() for t in ts]
        results = []
        for k in range(n):
            caps = []
            for j in range(int(nres[k])):
                ln = int(lens[k, j])
                cd = CaptionData([int(w) for w in sent[k, j, :ln]], float(scores[k, j]), bool(comp[k]))
                if maps is not None:
                    cd.alphas, cd.word_probs = maps[0][k, j, :ln].copy(), maps[1][k, j, :ln].copy()
                caps.append(cd)
            results.append(caps)
        return results
