"""The C-ABI library builds without a GPU, loads, and exports every symbol include/sat_b200.h declares.
No compute call is made here (there is no GPU in the build container)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "sat_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sat_[a-z_0-9]+)\s*\(", src)))


def test_header_declares_the_expected_entry_points():
    syms = declared_symbols()
    for must in ("sat_create", "sat_destroy", "sat_last_error", "sat_set_weight", "sat_prepare_contexts",
                 "sat_decode_step", "sat_decode_loop", "sat_beam_search", "sat_attention_fwd", "sat_lstm_fwd",
                 "sat_vocab_gemm"):
        assert must in syms


def test_library_builds_loads_and_exports_every_declared_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    for s in declared_symbols():
        assert hasattr(lib, s), "missing export %s" % s


def test_python_binding_covers_the_header(built_lib):
    import sat_b200
    from sat_b200 import lib as L
    assert sorted(L.SIGNATURES) == declared_symbols()
    assert sat_b200.load_library().sat_version() >= 100
    assert sat_b200.library_path() == built_lib


def test_create_fails_loudly_without_a_gpu(built_lib):
    import torch
    if torch.cuda.is_available():
        return
    import sat_b200
    from sat_b200.lib import Dims
    lib = sat_b200.load_library()
    d = Dims(4, 196, 512, 512, 512, 512, 1024, 512, 5000, 2, 2, 2, 20, 3)
    h = ctypes.c_void_p()
    rc = lib.sat_create(ctypes.byref(d), ctypes.byref(h))
    assert rc != 0 and not h.value
    assert b"CUDA" in lib.sat_last_error() or b"device" in lib.sat_last_error()
    try:
        sat_b200.CaptionGenerator(sat_b200.Config())
        raise AssertionError("CaptionGenerator must not construct without a GPU")
    except RuntimeError as e:
        assert "no CPU path" in str(e) or "CUDA" in str(e)


def test_sass_contains_wgmma_and_tma(built_lib):
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        return
    sass = subprocess.run([cuobjdump, "-sass", built_lib], stdout=subprocess.PIPE, text=True).stdout
    assert "arch = sm_90a" in sass
    assert "HGMMA" in sass        # wgmma.mma_async
    assert "UBLKCP" in sass       # cp.async.bulk (TMA) feeds both the dense and the attention kernels
    assert "HMMA." not in sass    # no legacy mma.sync path
