"""SincNet front end: the persistent, weight-resident sinc / Conv1d kernels (seg_conv_impl = 1) against the per-tile
wgmma kernels (seg_conv_impl = 2).  Both sum each output's products in ascending K steps, lo*hi then hi*lo then
hi*hi, and pool, add the bias and sum the InstanceNorm partials in the same order, so every output is bit-identical
and the launch counts are equal.

Cases: 10 s windows at 1, 3, 133, 2112 and 2113 windows (two sub-batches at the default seg_max_batch); windows of
1261 samples (the shortest), of lengths whose last tile is partial at each of the three stages, and longer than 15.4 s
(more than 128 stage-0 tiles: the partial sums go through part_reduce); windows whose valid samples end before the
window does; a 10-minute conversation; XVectorSincNet embeddings.
"""
import numpy as np
import pytest
import torch

from pyannote_audio_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

CHUNK = 160000


@pytest.fixture(scope="module")
def ctx():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyannote_audio_b200 import ops

    c = ops.Context(torch.device("cuda:0"))
    c.load_segmentation(syn.make_segmentation_state_dict(0))
    return c


def _both(ctx, run):
    """(persistent outputs, per-tile outputs) as lists of numpy arrays, and the two launch counts."""
    out, launches = {}, {}
    try:
        for impl in (2, 1):
            ctx.set_option("seg_conv_impl", impl)
            n0 = ctx.launch_count
            res = run()
            res = res if isinstance(res, tuple) else (res,)
            out[impl] = [r.cpu().numpy() for r in res]
            launches[impl] = ctx.launch_count - n0
    finally:
        ctx.set_option("seg_conv_impl", 1)
    return out[1], out[2], launches[1], launches[2]


def _assert_same(new, ref, n_new, n_ref):
    assert len(new) == len(ref)
    for a, b in zip(new, ref):
        assert a.shape == b.shape and a.dtype == b.dtype
        f = b.astype(np.float64)
        assert np.abs(f[np.isfinite(f)]).max() > 0
        assert a.tobytes() == b.tobytes()
    assert n_new == n_ref


def _wav(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * 0.1).cuda()


@pytest.mark.parametrize("nb", [1, 3, 133, 2112, 2113])
def test_sincnet_forward_matches_per_tile(ctx, nb):
    step = 1600
    wav = _wav(step * (nb - 1) + CHUNK + 3, 500 + nb)
    off = 3 + np.arange(nb, dtype=np.int64) * step
    valid = np.full(nb, CHUNK, dtype=np.int32)
    _assert_same(*_both(ctx, lambda: ctx.sincnet_forward(wav, off, valid)))


def _stage_tiles(window):
    p0 = (1 + (window - 251) // 10) // 3
    p1 = (p0 - 4) // 3
    return p0, p1, (p1 - 4) // 3


# 1261: the shortest window; 20000 / 30000 / 34000: partial last tiles (pool0, pool1, pool2 % 64 != 0) with full
# ones elsewhere; 160001; 300000 and 480000: 157 and 250 stage-0 tiles, more than part_reduce's group of 128
@pytest.mark.parametrize("window", [1261, 20000, 30000, 34000, 160001, 300000, 480000])
def test_seg_forward_any_window_matches_per_tile(ctx, window):
    assert all(p % 64 for p in _stage_tiles(window)) or window == 1261
    nb = 3
    wav = _wav(window * nb + 11, window)
    off = np.array([0, 11, window * (nb - 1) + 11], dtype=np.int64)
    valid = np.full(nb, window, dtype=np.int32)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.seg_forward(wav, off, valid, return_logp=True, window=window))
    assert ref[1].shape[:2] == ref[0].shape
    _assert_same(new, ref, n_new, n_ref)


def test_short_valid_chunks_match_per_tile(ctx):
    nb = 7
    wav = _wav(CHUNK * 4, 77)
    off = np.arange(nb, dtype=np.int64) * 16000
    valid = np.array([CHUNK, 1, 1000, 1920 * 10 + 7, 77777, 159999, CHUNK - 16000 * 6 - 5], dtype=np.int32)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.seg_forward(wav, off, valid, return_logp=True))
    _assert_same(new, ref, n_new, n_ref)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.sincnet_forward(wav, off, valid))
    _assert_same(new, ref, n_new, n_ref)


def test_ten_minute_conversation_matches_per_tile(ctx):
    wav = syn.make_conversation(600.0, seed=21)[0].contiguous().cuda()
    off = np.arange(0, wav.numel() - CHUNK + 1, 16000, dtype=np.int64)
    valid = np.minimum(CHUNK, wav.numel() - off).astype(np.int32)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.seg_forward(wav, off, valid, return_logp=True))
    assert ref[0].shape == (len(off), 589)
    _assert_same(new, ref, n_new, n_ref)


def test_xvector_embeddings_match_per_tile():
    from pyannote_audio_b200 import ops

    c = ops.Context(torch.device("cuda:0"))
    c.load_xvector(syn.make_xvector_state_dict(3))
    for n in (36817, 160000):          # 4771 samples (one TDNN frame) pool to NaN without weights
        wav = _wav(3 * n + 5, n)
        _assert_same(*_both(c, lambda: c.xvec_forward(wav, [0, 5, 2 * n + 5], n)))
