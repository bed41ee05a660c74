"""ctypes binding of libsat_b200.so (include/sat_b200.h).  Fails loudly if the library is
missing: there is no fallback path."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class SatError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("sat_b200 error %d: %s" % (code, msg))
        self.code = code


class Optimizer(C.Structure):
    """sat_optimizer of include/sat_b200.h"""
    _fields_ = [("kind", C.c_int32), ("learning_rate", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("epsilon", C.c_float), ("decay", C.c_float), ("momentum", C.c_float), ("centered", C.c_int32),
                ("use_nesterov", C.c_int32), ("clip_gradients", C.c_float)]


OPTIMIZER_KINDS = {"Adam": 0, "RMSProp": 1, "Momentum": 2, "SGD": 3}


class Dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "max_batch", "num_ctx", "dim_ctx", "num_lstm_units", "dim_embedding", "dim_attend_layer",
        "dim_decode_layer", "dim_initalize_layer", "vocabulary_size", "num_attend_layers",
        "num_decode_layers", "num_initalize_layers", "max_caption_length", "max_beam")]


def library_path():
    return os.path.join(_HERE, "libsat_b200.so")


_P, _I, _L = C.c_void_p, C.c_int32, C.c_int64
# name -> (restype, argtypes); every symbol declared in include/sat_b200.h
SIGNATURES = {
    "sat_create": (C.c_int, [C.POINTER(Dims), C.POINTER(_P)]),
    "sat_destroy": (None, [_P]),
    "sat_last_error": (C.c_char_p, []),
    "sat_version": (C.c_int, []),
    "sat_set_option": (C.c_int, [_P, C.c_char_p, _L]),
    "sat_get_info": (C.c_int, [_P, C.c_char_p, C.POINTER(_L)]),
    "sat_set_weight": (C.c_int, [_P, C.c_char_p, _P, _L, _L, _P]),
    "sat_weights_missing": (C.c_int, [_P]),
    "sat_prepare_contexts": (C.c_int, [_P, _P, _I, _P, _P, _P]),
    "sat_decode_step": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "sat_decode_loop": (C.c_int, [_P, _P, _I, _I, _P, _P, _P, _P]),
    "sat_beam_search": (C.c_int, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "sat_decode_loop_maps": (C.c_int, [_P, _P, _I, _I, _P, _P, _P, _P, _P, _P]),
    "sat_beam_search_maps": (C.c_int, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "sat_sample_loop": (C.c_int, [_P, _P, _I, _I, _I, C.c_float, C.c_uint64, _P, _P, _P]),
    "sat_sample_loop_filtered": (C.c_int, [_P, _P, _I, _I, _I, C.c_float, _I, C.c_float, C.c_uint64, _P, _P, _P]),
    "sat_sample_uniform": (C.c_double, [C.c_uint64, _L, _I, _I]),
    "sat_decode_step_host": (C.c_int, [_P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _P]),
    "sat_decode_loop_host": (C.c_int, [_P, _P, _I, _I, _P, _P, _P]),
    "sat_beam_search_host": (C.c_int, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "sat_decode_loop_host_submit": (C.c_int, [_P, _P, _I, _I, _P, _P, _I, _P]),
    "sat_decode_loop_host_wait": (C.c_int, [_P, _I]),
    "sat_attention_fwd": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _P]),
    "sat_lstm_fwd": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "sat_vocab_gemm": (C.c_int, [_P, _P, _P, _P, _P, _I, _P]),
    "sat_dense_fwd": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "sat_train_init": (C.c_int, [_P, _I, _I, C.c_float, C.c_float, C.c_float, C.c_float]),
    "sat_train_num_vars": (C.c_int, [_P]),
    "sat_train_rng_uniform": (C.c_float, [C.c_uint64, C.c_uint64, C.c_uint64]),
    "sat_train_var": (C.c_int, [_P, _I, C.POINTER(C.c_char_p), C.POINTER(_L), C.POINTER(_L), C.POINTER(_L),
                                C.POINTER(_I), C.POINTER(_L)]),
    "sat_train_forward_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, _I, _I, C.c_uint64, C.c_double, _I, _P, _P]),
    "sat_train_forward_backward_dsum": (C.c_int, [_P, _P, _P, _P, _P, _P, _I, _I, C.c_uint64, _P, _I, _P, _P]),
    "sat_train_init_grouped": (C.c_int, [_P, _I, _I, _I, C.c_float, C.c_float, C.c_float, C.c_float]),
    "sat_train_forward_backward_grouped": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _P, _P, _I, C.c_uint64, _P, _I, _P, _P]),
    "sat_caption_masks": (C.c_int, [_P, _I, _I, _I, _P, _P, _P]),
    "sat_cider_create": (C.c_int, [_P, _L, _I, _I, _I, _I, C.POINTER(_P)]),
    "sat_cider_destroy": (None, [_P]),
    "sat_cider_d": (C.c_int, [_P, _P, _I, _I, _I, _P, _I, _I, _P, _P]),
    "sat_train_apply": (C.c_int, [_P, _P, _P, _P, _P, _L, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, _P,
                                  _P]),
    "sat_train_apply_opt": (C.c_int, [_P, _P, _P, _P, _P, _P, _L, C.POINTER(Optimizer), _P, _P]),
    "sat_train_fill": (C.c_int, [_P, _P, C.c_float, _L, _P]),
}


def load_library(path=None):
    """dlopen libsat_b200.so and declare every entry point.  Raises if it is not built."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    p = path or library_path()
    if not os.path.exists(p):
        raise RuntimeError(
            "libsat_b200.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `python show-attend-and-tell_b200/build.py`; sat_b200 has no CPU/eager fallback." % p)
    lib = C.CDLL(p)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _LIB = lib
    return lib


def check(lib, rc):
    if rc != 0:
        msg = lib.sat_last_error()
        raise SatError(rc, msg.decode() if msg else "?")
