"""CIDEr-D on the device (sat_cider_create / sat_cider_d of include/sat_b200.h): the reward of self-critical training
(CaptionGenerator.scst_step(contexts, CiderD(...), references=...)) and a validation metric on word ids.

    cider = CiderD(train_references, eos_id, vocabulary_size)    # document frequencies of a reference corpus
    scores = cider.scores(candidates [n, C, T], references [n, R, T_ref])   # device float32 [n, C]

Rows are word ids; a row ends after its first eos_id, or before its first id < 0 (padding) or >= vocabulary_size.
coco-caption's numbers (its tokenizer drops punctuation): strip '.' from the ids and pass an eos_id that never occurs.
"""
import ctypes as C

import numpy as np

from .lib import check, load_library


def pad(references):
    """int32 array [n, R, T_ref] padded with -1 from a ragged list (image -> list of word-id lists) or an array."""
    if isinstance(references, (list, tuple)):
        n = len(references)
        R = max([len(refs) for refs in references] + [1])
        T = max([len(r) for refs in references for r in refs] + [1])
        out = np.full((n, R, T), -1, np.int32)
        for i, refs in enumerate(references):
            for j, r in enumerate(refs):
                out[i, j, :len(r)] = np.asarray(r, np.int64)
        return out
    out = np.ascontiguousarray(np.asarray(references), np.int32)
    if out.ndim != 3:
        raise ValueError("references: [n, R, T_ref] expected, got shape %s" % (out.shape,))
    return out


class CiderD(object):
    """CIDEr-D scorer with the document frequencies of a reference corpus (`references`: ragged list or [N, R, T_ref]
    array, one entry per image; N = the number of images), kept on the CUDA device current at construction.
    Self-critical training builds it from the training references; coco-caption's convention builds it from the
    evaluated set's own references."""

    def __init__(self, references, eos_id, vocabulary_size):
        import torch
        self.torch = torch
        self.lib = load_library()
        self.eos_id, self.vocabulary_size = int(eos_id), int(vocabulary_size)
        refs = pad(references)
        self.device = torch.device("cuda", torch.cuda.current_device())
        self._c = C.c_void_p()
        check(self.lib, self.lib.sat_cider_create(refs.ctypes.data_as(C.c_void_p), refs.shape[0], refs.shape[1],
                                                  refs.shape[2], self.eos_id, self.vocabulary_size, C.byref(self._c)))

    def __del__(self):
        try:
            if getattr(self, "_c", None) is not None and self._c.value:
                self.lib.sat_cider_destroy(self._c)
                self._c = C.c_void_p()
        except Exception:
            pass

    close = __del__

    def _dev(self, x):
        torch = self.torch
        if not isinstance(x, torch.Tensor):
            x = torch.from_numpy(pad(x))
        return x.to(device=self.device, dtype=torch.int32).contiguous()

    def scores(self, candidates, references, stream=None):
        """CIDEr-D of candidates [n, C, T] against references [n, R, T_ref] (torch tensors, numpy arrays or ragged
        lists; -1 pads): a float32 device tensor [n, C], computed on `stream` (default: the current stream) and
        ordered there like any other work on it.  Limits: R <= 8, T and T_ref <= 64."""
        torch = self.torch
        st = torch.cuda.current_stream(self.device) if stream is None else stream
        with torch.cuda.device(self.device), torch.cuda.stream(st):
            cand, refs = self._dev(candidates), self._dev(references)
            if cand.dim() != 3 or refs.dim() != 3 or cand.shape[0] != refs.shape[0]:
                raise ValueError("candidates [n, C, T] and references [n, R, T_ref] expected, got %s and %s"
                                 % (tuple(cand.shape), tuple(refs.shape)))
            n, nc, T = cand.shape
            out = torch.empty(n, nc, dtype=torch.float32, device=self.device)
            p = lambda t: C.c_void_p(t.data_ptr())
            check(self.lib, self.lib.sat_cider_d(self._c, p(cand), n, nc, T, p(refs), refs.shape[1], refs.shape[2],
                                                 p(out), C.c_void_p(st.cuda_stream)))
        return out
