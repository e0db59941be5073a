"""Launch counting: b200_ctx_launch_count is counted where the library launches kernels, in b200::launch
(csrc/common.cuh), on the counter the running entry point binds (CtxScope in api.cu).

CPU: no kernel is launched anywhere else in csrc/, and no hand-kept tally of launches is left.
GPU: for each entry point, the count's delta over one call equals the number of kernels torch.profiler records for
that call.  Memcpy and memset operations are not kernels and are counted by neither.  Every input is built, and every
cache the ops wrapper keeps is filled, by a warm-up call before the profiled one.
"""
import collections
import os
import time

import numpy as np
import pytest
import torch

from pyannote_audio_b200 import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pyannote_audio_b200", "csrc")
CHUNK = 160000


def test_kernels_are_launched_only_through_launch():
    hits = []
    for name in sorted(os.listdir(CSRC)):
        with open(os.path.join(CSRC, name)) as f:
            for i, line in enumerate(f, 1):
                for token in ("<<<", "cudaLaunchKernel", "cudaLaunchCooperativeKernel", "launches +="):
                    if token in line:
                        hits.append((name, i, token))
    assert sorted((name, token) for name, _, token in hits) == [("common.cuh", "<<<"),
                                                                 ("common.cuh", "cudaLaunchCooperativeKernel")]
    with open(os.path.join(CSRC, "common.cuh")) as f:
        lines = f.read().split("\n")
    first = next(i for i, line in enumerate(lines, 1) if line.startswith("int launch("))
    last = next(i for i, line in enumerate(lines, 1) if i > first and line == "}")
    assert all(first < i < last for _, i, _ in hits)


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _kernels(ctx, call):
    """(launch count delta, names of the kernels the profiler records) of one call of `call`, after a warm-up call."""
    from torch.profiler import ProfilerActivity, profile

    call()
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # The profiler keeps only device activity that it places inside its capture window, on a clock converted from
        # the GPU's.  Idle margins on both sides keep the first and the last kernel of the call inside the window.
        time.sleep(0.1)
        call()
        torch.cuda.synchronize()
        time.sleep(0.1)
    counted = ctx.launch_count - n0
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
    return counted, kernels


def _assert_counted(ctx, call):
    counted, kernels = _kernels(ctx, call)
    assert kernels
    assert counted == len(kernels), (counted, len(kernels), sorted(collections.Counter(kernels).items()))


class _Options:
    """set_option for the duration of a `with` block, restoring the given defaults afterwards."""

    def __init__(self, ctx, options, defaults):
        self.ctx, self.options, self.defaults = ctx, options, defaults

    def __enter__(self):
        for k, v in self.options.items():
            self.ctx.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.options:
            self.ctx.set_option(k, self.defaults[k])


def _context():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyannote_audio_b200 import ops

    return ops.Context(torch.device("cuda:0"))


def _wav(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * 0.1).cuda()


@pytest.fixture(scope="module")
def seg_ctx():
    c = _context()
    c.load_segmentation(syn.make_segmentation_state_dict(0))
    return c


SEG_DEFAULTS = {"seg_gemm_impl": 1, "seg_conv_impl": 1, "seg_rec_impl": 1, "seg_max_batch": 2112}
SEG_IMPLS = {
    "default": {},
    "fp32": {"seg_gemm_impl": 0, "seg_conv_impl": 0, "seg_rec_impl": 0},
    "reference": {"seg_conv_impl": 2, "seg_rec_impl": 2},
}


@pytest.mark.gpu
@pytest.mark.parametrize("impl", sorted(SEG_IMPLS))
@pytest.mark.parametrize("window,n", [(CHUNK, 1), (CHUNK, 5), (480000, 2)])
def test_seg_forward(seg_ctx, impl, window, n):
    # seg_max_batch 3: five 10 s windows run as two sub-batches, two 30 s windows (the part_reduce path) as two
    wav = _wav(window + 1600 * (n - 1) + 5, 40 + n)
    off = 5 + np.arange(n, dtype=np.int64) * 1600
    valid = np.full(n, window, dtype=np.int32)
    with _Options(seg_ctx, dict(SEG_IMPLS[impl], seg_max_batch=3), SEG_DEFAULTS):
        _assert_counted(seg_ctx, lambda: seg_ctx.seg_forward(wav, off, valid, return_logp=True, window=window))


@pytest.mark.gpu
def test_sincnet_forward(seg_ctx):
    wav = _wav(CHUNK + 3200, 7)
    _assert_counted(seg_ctx, lambda: seg_ctx.sincnet_forward(wav, [0, 1600, 3200], [CHUNK, CHUNK, CHUNK - 7]))


@pytest.mark.gpu
@pytest.mark.parametrize("layer", [-1, 3])
def test_ssl_forward(layer):
    c = _context()
    c.load_sseriouss(syn.make_sseriouss_state_dict(5, wav2vec_layer=layer, num_classes=7), wav2vec_layer=layer)
    wav = _wav(2 * CHUNK, 50)
    _assert_counted(c, lambda: c.ssl_forward(wav, [0, 16000, CHUNK], [CHUNK, CHUNK, CHUNK], return_logp=True))


@pytest.fixture(scope="module")
def emb_ctx():
    c = _context()
    c.load_embedding(syn.make_embedding_state_dict(1))
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("conv_impl", [0, 1, 2])
def test_emb_forward_and_trunk(emb_ctx, conv_impl):
    n = 3
    wav = _wav(CHUNK + 16000 * (n - 1), 60)
    off = np.arange(n, dtype=np.int64) * 16000
    valid = np.array([CHUNK, CHUNK, CHUNK - 999], dtype=np.int32)
    masks = (torch.rand((n, 3, 589), generator=torch.Generator().manual_seed(61)) > 0.3).to(torch.uint8).cuda()
    fbank = torch.randn((n, 998, 80), generator=torch.Generator().manual_seed(62)).cuda()
    with _Options(emb_ctx, {"conv_impl": conv_impl}, {"conv_impl": 1}):
        _assert_counted(emb_ctx, lambda: emb_ctx.emb_forward(wav, off, valid, masks))
        _assert_counted(emb_ctx, lambda: emb_ctx.emb_trunk(fbank))


@pytest.mark.gpu
def test_bottleneck_emb_forward_and_trunk():
    c = _context()
    c.load_embedding(syn.make_bottleneck_state_dict(152, 3))
    wav = _wav(CHUNK + 16000, 63)
    masks = torch.ones((2, 3, 589), dtype=torch.uint8).cuda()
    fbank = torch.randn((2, 998, 80), generator=torch.Generator().manual_seed(64)).cuda()
    _assert_counted(c, lambda: c.emb_forward(wav, [0, 16000], [CHUNK, CHUNK], masks))
    _assert_counted(c, lambda: c.emb_trunk(fbank))


@pytest.mark.gpu
@pytest.mark.parametrize("num_samples", [CHUNK, 700000])   # 125 and 547 trunk frames: either side of kPoolSlice = 512
def test_emb_forward_utt(emb_ctx, num_samples):
    wav = _wav(num_samples + 8000, 65)
    weights = torch.rand((2, 3, 300), generator=torch.Generator().manual_seed(66)).cuda()
    _assert_counted(emb_ctx, lambda: emb_ctx.emb_forward_utt(wav, [0, 8000], num_samples))
    _assert_counted(emb_ctx, lambda: emb_ctx.emb_forward_utt(wav, [0, 8000], num_samples, weights=weights))


@pytest.mark.gpu
def test_emb_fbank_embedding_and_stats_pool(emb_ctx):
    wav = _wav(CHUNK + 1600, 67)
    frames = torch.randn((2, 256, 10, 125), generator=torch.Generator().manual_seed(68)).cuda()
    seq = torch.randn((2, 40, 100), generator=torch.Generator().manual_seed(69)).cuda()
    _assert_counted(emb_ctx, lambda: emb_ctx.emb_fbank(wav, [0, 1600], [CHUNK, CHUNK - 5]))
    _assert_counted(emb_ctx, lambda: emb_ctx.emb_forward_embedding(frames))
    _assert_counted(emb_ctx, lambda: emb_ctx.stats_pool(seq))


@pytest.mark.gpu
def test_xvec_forward():
    c = _context()
    c.load_xvector(syn.make_xvector_state_dict(3))
    wav = _wav(3 * 32000, 70)
    _assert_counted(c, lambda: c.xvec_forward(wav, [0, 17, 32000], 48000))


@pytest.fixture(scope="module")
def ctx():
    return _context()


def _f64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("normalize", [0, 1, 2])
def test_linkage(ctx, normalize):
    rng = np.random.default_rng(normalize)
    ro = [0, 1, 41, 41, 106]                                  # a 1-row problem, 40 rows, an empty one, 65 rows
    x = _f64(rng.standard_normal((ro[-1], 16)))
    _assert_counted(ctx, lambda: ctx.linkage_centroid_batched(x, ro, normalize=normalize))
    with _Options(ctx, {"linkage_grid_min": 50}, {"linkage_grid_min": 32769}):   # 65 rows on the whole-GPU path
        _assert_counted(ctx, lambda: ctx.linkage_centroid_batched(x, ro, normalize=normalize))


@pytest.mark.gpu
def test_clustering_ops(ctx):
    from pyannote_audio_b200.ops import C, _ptr

    rng = np.random.default_rng(5)
    plda = syn.make_plda(2)
    ns, Ss, D = np.array([30, 12], dtype=np.int32), np.array([3, 2], dtype=np.int32), 128
    fea = _f64(rng.standard_normal((int(ns.sum()), D)))
    phi = _f64(np.abs(rng.standard_normal(D)) + 0.1)
    gamma0 = np.concatenate([rng.dirichlet(np.ones(s), n).reshape(-1) for n, s in zip(ns, Ss)])
    gamma, pi = _f64(gamma0), _f64(np.zeros(int(Ss.sum())))

    def vbx():   # the ABI call itself: Context.vbx_batched clones gamma0 with a torch kernel first
        gamma.copy_(torch.from_numpy(gamma0))
        ctx._call("b200_vbx_batched", _ptr(fea), _ptr(phi), ns.ctypes.data, Ss.ctypes.data, len(ns), D,
                  C.c_double(0.07), C.c_double(0.8), 20, C.c_double(1e-4), _ptr(gamma), _ptr(pi), None)

    x = _f64(rng.standard_normal((20, 256)))
    plda_args = [_f64(plda[k]) for k in ("mean1", "mean2", "lda", "mu")] + [_f64(plda["tr"].T)]
    q = _f64(rng.random((20, 4)))
    kept = torch.tensor([0, 2, 3], dtype=torch.int32).cuda()
    soft = _f64(rng.random((6, 3, 4)))
    _assert_counted(ctx, vbx)
    _assert_counted(ctx, lambda: ctx.plda_transform(x, *plda_args))
    _assert_counted(ctx, lambda: ctx.weighted_centroids(q, kept, x))
    _assert_counted(ctx, lambda: ctx.cdist_cosine(x, x[:4]))
    _assert_counted(ctx, lambda: ctx.assign(soft, constrained=True))
    _assert_counted(ctx, lambda: ctx.assign(soft, constrained=False))


@pytest.mark.gpu
def test_post_processing_ops(ctx):
    rng = np.random.default_rng(6)
    C_, F = 8, 589
    sf = np.arange(C_, dtype=np.int32) * 59
    num_frames = int(sf[-1]) + F
    cls = torch.from_numpy(rng.integers(0, 7, (C_, F), dtype=np.uint8)).cuda()
    seg = torch.from_numpy(rng.integers(0, 2, (C_, F, 3), dtype=np.uint8)).cuda()
    hard = torch.from_numpy(rng.integers(-2, 4, (C_, 3), dtype=np.int8)).cuda()
    count = torch.from_numpy(rng.integers(0, 3, num_frames, dtype=np.uint8)).cuda()
    scores = torch.from_numpy(rng.random((C_, F, 3), dtype=np.float32)).cuda()
    discrete = torch.from_numpy(rng.integers(0, 2, (num_frames, 4), dtype=np.uint8)).cuda()
    _assert_counted(ctx, lambda: ctx.powerset_to_multilabel(cls))
    _assert_counted(ctx, lambda: ctx.powerset_speech(cls))
    _assert_counted(ctx, lambda: ctx.speaker_count(seg, sf, num_frames))
    _assert_counted(ctx, lambda: ctx.reconstruct(seg, hard, sf, num_frames, count, 4))
    _assert_counted(ctx, lambda: ctx.reconstruct(seg, hard, sf, num_frames, count, 40))
    _assert_counted(ctx, lambda: ctx.aggregate(scores, sf, num_frames, hamming=True, warm_up=(0.5, 0.5)))
    _assert_counted(ctx, lambda: ctx.frame_transitions(discrete))
    _assert_counted(ctx, lambda: ctx.clean_frames(seg))


@pytest.mark.gpu
def test_audio_ingest(ctx):
    g = torch.Generator().manual_seed(7)
    pcm = (torch.randn((44100, 2), generator=g) * 3000).to(torch.int16).cuda()
    _assert_counted(ctx, lambda: ctx.audio_ingest(pcm, 44100, 16000))
    _assert_counted(ctx, lambda: ctx.audio_ingest(pcm, 44100, 16000, channel=1))
