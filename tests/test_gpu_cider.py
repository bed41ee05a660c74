"""CIDEr-D on the device (sat_cider_create / sat_cider_d, sat_b200.CiderD) against the fp64 reference of cider_ref.py,
and CaptionGenerator.scst_step with the built-in reward against the same step with a host reward."""
import ctypes as C

import numpy as np
import pytest

import cider_ref as CR
from test_gpu_scst import gsetup
from test_gpu_train import TDIMS

pytestmark = pytest.mark.gpu


def random_rows(rng, shape, V, eos, lo=0):
    """rows of word ids in [lo, V) with eos now and then, word 0, repeated words, ids >= V and -1 padding"""
    out = np.full(shape, -1, np.int64)
    T = shape[-1]
    for idx in np.ndindex(*shape[:-1]):
        L = rng.randint(1, T + 1)
        row = rng.randint(lo, V, L)
        if rng.rand() < 0.3:
            row[rng.randint(L)] = eos
        if rng.rand() < 0.2:
            row[rng.randint(L)] = 0
        if L > 2 and rng.rand() < 0.3:
            i = rng.randint(L - 1)
            row[i + 1] = row[i]
        if rng.rand() < 0.1:
            row[rng.randint(L)] = V + rng.randint(3)
        if rng.rand() < 0.1:
            row[rng.randint(L)] = -1
        out[idx][:L] = row
    return out.astype(np.int32)


def case(seed, n, R, T, T_ref, V, C_=6, lo=0):
    rng = np.random.RandomState(seed)
    eos = min(2, V - 1)
    refs = random_rows(rng, (n, R, T_ref), V, eos, lo)
    for i in range(n):                     # 1..R references per image, and one image without any
        refs[i, rng.randint(1, R + 1):] = -1
    refs[n - 1] = -1
    cand = random_rows(rng, (n, C_, T), V, eos, lo)
    for i in range(n):                     # candidates equal to one of the image's references
        k = min(T, T_ref)
        cand[i, 0, :] = -1
        cand[i, 0, :k] = refs[i, 0, :k]
    corpus = np.concatenate([refs, random_rows(rng, (2 * n, R, T_ref), V, eos, lo)])
    return eos, refs, cand, corpus


def check_against_reference(cider, cand, refs, corpus, eos, V):
    import torch
    got = cider.scores(torch.from_numpy(cand).cuda(), torch.from_numpy(refs).cuda()).cpu().numpy().astype(np.float64)
    df, N = CR.doc_freq(corpus, eos, V)
    ref = np.array(CR.scores(cand, refs, df, N, eos, V))
    err = np.abs(got - ref) / np.maximum(1.0, np.abs(ref))
    assert err.max() <= 1e-5, (err.max(), np.unravel_index(err.argmax(), err.shape))
    return got, ref


@pytest.mark.parametrize("seed,R,T,T_ref,V", [
    (0, 1, 1, 5, 12), (1, 5, 20, 16, 12), (2, 7, 64, 64, 30), (3, 8, 33, 64, 7), (4, 3, 7, 2, 2), (5, 6, 12, 24, 5000),
    (6, 4, 40, 9, 9)])
def test_cider_d_matches_the_fp64_reference(seed, R, T, T_ref, V):
    import sat_b200
    eos, refs, cand, corpus = case(seed, 9, R, T, T_ref, V)
    cider = sat_b200.CiderD(corpus, eos, V)
    got, ref = check_against_reference(cider, cand, refs, corpus, eos, V)
    assert (got[-1] == 0).all()                        # the image without references
    assert ref.max() > 0.5


def test_largest_word_ids_and_ragged_input():
    """V = 65535: word 65534 fills a 16-bit key field with ones (a 4-gram of it is the all-ones key)"""
    import sat_b200
    V = 65535
    eos, refs, cand, corpus = case(7, 6, 5, 20, 20, V, lo=V - 6)
    refs[0, 1, :5] = V - 1
    cand[0, 1, :6] = V - 1
    cider = sat_b200.CiderD(corpus, eos, V)
    got, ref = check_against_reference(cider, cand, refs, corpus, eos, V)
    ragged = [[[int(w) for w in CR.cut(row, eos, V)] for row in img] for img in refs]
    assert np.array_equal(cider.scores(cand, ragged).cpu().numpy(), got.astype(np.float32))


def test_scores_are_bitwise_reproducible_and_stream_ordered():
    import sat_b200
    import torch
    eos, refs, cand, corpus = case(8, 64, 5, 20, 20, 50)
    cider = sat_b200.CiderD(corpus, eos, 50)
    c, r = torch.from_numpy(cand).cuda(), torch.from_numpy(refs).cuda()
    a = cider.scores(c, r)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    b = cider.scores(c, r, stream=s)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_invalid_arguments_enqueue_nothing():
    import sat_b200
    import torch
    lib = sat_b200.load_library()
    V, eos = 20, 2
    refs = np.random.RandomState(0).randint(0, V, (3, 9, 65)).astype(np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    h = C.c_void_p()
    for args in ((None, 3, 5, 10), (vp(refs), 0, 5, 10), (vp(refs), 3, 0, 10), (vp(refs), 3, 5, 0)):
        assert lib.sat_cider_create(*args, eos, V, C.byref(h)) == -1 and not h.value
    for bad_v in (1, 0, 65536):
        assert lib.sat_cider_create(vp(refs), 3, 5, 10, eos, bad_v, C.byref(h)) == -1 and not h.value
    cider = sat_b200.CiderD(refs[:, :5, :20], eos, V)
    cd = torch.from_numpy(refs).cuda()
    out = torch.full((3, 4), 7.0, device="cuda")
    p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())

    def call(c=cider._c, cand=cd, n=3, nc=4, T=20, refs=cd, R=5, T_ref=20, scores=out):
        return lib.sat_cider_d(c, p(cand), n, nc, T, p(refs), R, T_ref, p(scores), None)
    torch.cuda.synchronize()
    for kw in (dict(c=None), dict(cand=None), dict(refs=None), dict(scores=None), dict(n=-1), dict(nc=0), dict(T=0),
               dict(R=0), dict(T_ref=0)):
        assert call(**kw) == -1, kw
    for kw in (dict(R=9), dict(T=65), dict(T_ref=65)):
        assert call(**kw) == -4, kw
    assert call(n=0) == 0
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    with pytest.raises(sat_b200.SatError):
        cider.scores(cd[:, :, :20], cd[:, :9, :20])
    assert call() == 0
    torch.cuda.synchronize()
    assert bool((out != 7.0).any())


def scst_case(baseline, n=2, K=5):
    """a fresh model and reference captions built from what the sampler will draw (same weights and sample seed), so
    that rewards, hence advantages, differ from caption to caption"""
    import sat_b200
    import torch
    ocfg, w, m, ctx, _, _, _ = gsetup(n, K, seed=12, dims=dict(TDIMS, max_caption_length=6), max_batch=n * 4)
    T, V, eos = ocfg.max_caption_length, ocfg.vocabulary_size, int(m.config.eos_id)
    c = torch.from_numpy(ctx).cuda()
    m.sync_inference_weights()
    toks = m.sample_device(c, K, T, 1.0, seed=99, want_word_probs=False)[0].cpu().numpy()
    rng = np.random.RandomState(5)
    refs = np.full((n, 4, T), -1, np.int32)
    for i in range(n):
        refs[i, 0] = toks[i, 0]
        refs[i, 1, :4] = toks[i, 1, :4]
        refs[i, 2, :3] = toks[i, 2, 2:5]
        refs[i, 3] = rng.randint(0, V, T)
    corpus = np.concatenate([refs, rng.randint(0, V, (6, 4, T)).astype(np.int32)])
    return m, c, refs, corpus, sat_b200.CiderD(corpus, eos, V), eos, V


@pytest.mark.parametrize("baseline", ["greedy", "mean"])
def test_scst_step_with_cider_matches_a_host_reward(baseline):
    import torch
    n, K = 2, 5
    m, c, refs, corpus, cider, eos, V = scst_case(baseline, n, K)
    out_d = m.scst_step(c, cider, num_samples=K, baseline=baseline, seed=0, sample_seed=99,
                        references=torch.from_numpy(refs).cuda())
    w_d = m._buf("scst_w", (n * K,), torch.float32).cpu().numpy()
    p_d = m.params.cpu().numpy()

    m2, c2, refs2, corpus2, _, _, _ = scst_case(baseline, n, K)
    assert np.array_equal(refs, refs2)
    df, N = CR.doc_freq(corpus, eos, V)

    def reward(caps):
        return np.array([[CR.cider_d(CR.cut(cap, eos, V), CR.image_refs(refs[i], eos, V), df, N) for cap in img]
                         for i, img in enumerate(caps)])
    out_h = m2.scst_step(c2, reward, num_samples=K, baseline=baseline, seed=0, sample_seed=99)
    w_h = m2._buf("scst_w", (n * K,), torch.float32).cpu().numpy()
    assert np.abs(w_h).max() > 0.1
    np.testing.assert_allclose(w_d, w_h, rtol=0, atol=1e-5)
    for k in ("sample_reward", "baseline_reward"):
        assert isinstance(out_d[k], float) and out_d[k] == pytest.approx(out_h[k], abs=1e-5)
    np.testing.assert_allclose(p_d, m2.params.cpu().numpy(), rtol=0, atol=3e-6)


def test_scst_step_with_cider_never_waits_for_the_host():
    import torch
    n, K = 2, 5
    m, c, refs, corpus, cider, eos, V = scst_case("greedy", n, K)
    r = torch.from_numpy(refs).cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for s in (1, 2):
            out = m.scst_step(c, cider, num_samples=K, sample_seed=s, sync=False, references=r)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert isinstance(out["sample_reward"], torch.Tensor) and out["sample_reward"].is_cuda
    torch.cuda.synchronize()
    assert np.isfinite(float(out["sample_reward"])) and np.isfinite(float(out["losses"][0]))
    with pytest.raises(ValueError, match="references"):
        m.scst_step(c, cider, num_samples=K)
