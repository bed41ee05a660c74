"""sat_b200 — H100-native soft-attention LSTM decode path of show-attend-and-tell.

Host side (Python) of the reference's CaptionGenerator call surface (model.py,
base_model.py) over the C ABI of libsat_b200.so (include/sat_b200.h).  PyTorch tensors
are used as device-buffer containers only; all arithmetic runs in the hand-written
sm_90a kernels under csrc/.  There is no CPU fallback: importing works anywhere, but
creating a CaptionGenerator without the built library or without an H100 raises.
"""
from .config import Config  # noqa: F401
from .lib import SatError, load_library, library_path  # noqa: F401
from .model import CaptionGenerator, weight_shapes  # noqa: F401
from .captions import Vocabulary, assemble_captions, write_eval_results, write_test_results  # noqa: F401
from .cider import CiderD  # noqa: F401

__all__ = ["Config", "CaptionGenerator", "SatError", "load_library", "library_path", "weight_shapes", "Vocabulary",
           "assemble_captions", "write_eval_results", "write_test_results", "CiderD"]
