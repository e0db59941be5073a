"""Trunk layer 3: the chunk-row kernel computes two output rows per unit for C_in = C_out = 128 (conv_impl = 1),
against the per-tap wgmma kernel (conv_impl = 2).  Both sum each output's products in the (tap, channel chunk,
16-channel step) order, so the results are bit-identical, and each conv is still one launch.

The 10 s batches put row pairs of one segment on different CTAs and walk the persistent loop's tail (one segment, an
odd handful, one embedding sub-batch and one segment more).  The any-length path covers fbank widths T0 whose layer-3
width (about T0 / 4) ends just below and just beyond one and two 128-pixel column tiles.  The bottleneck trunk runs
the same kernel on the conv2 of its layer-3 blocks.  With 80 mel bands layer 3 always has 20 rows, so the masked
second row of an odd row count is not reachable through the library's entry points.
"""
import numpy as np
import pytest
import torch

from pyannote_audio_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def _context(state_dict):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyannote_audio_b200 import ops

    c = ops.Context(torch.device("cuda:0"))
    c.load_embedding(state_dict)
    return c


@pytest.fixture(scope="module")
def ctx():
    return _context(syn.make_embedding_state_dict(5))


def _both(ctx, run):
    out, launches = {}, {}
    try:
        for impl in (2, 1):
            ctx.set_option("conv_impl", impl)
            n0 = ctx.launch_count
            out[impl] = run().cpu().numpy()
            launches[impl] = ctx.launch_count - n0
    finally:
        ctx.set_option("conv_impl", 1)
    return out[1], out[2], launches[1], launches[2]


def _fbank(batch, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((batch, 998, 80), generator=g) * 2.0 + 0.5).cuda()


@pytest.mark.parametrize("batch", [1, 3, 264, 265])
def test_trunk_layer3_pairs_match_per_tap(ctx, batch):
    fb = _fbank(batch, 3000 + batch)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.emb_trunk(fb))
    assert new.shape == (batch, 256, 10, 125)
    assert np.abs(ref).max() > 0
    assert np.array_equal(new, ref)
    calls = -(-batch // 264)                      # emb_trunk sub-batches of emb_max_batch = 264 segments
    assert n_ref - n_new == 3 * calls             # only the fused layer-1 blocks launch fewer kernels


# layer-3 width W3 = (T0 - 1) // 4 + 1 for T0 > 1: 127, 128, 129, 255, 256, 257 pixels
@pytest.mark.parametrize("t0", [505, 509, 513, 1017, 1021, 1025])
def test_utterance_layer3_pairs_match_per_tap(ctx, t0):
    batch = 2
    n = 400 + 160 * (t0 - 1)                 # T0 = 1 + (n - 400) // 160 fbank frames
    g = torch.Generator().manual_seed(t0 * 10 + 3)
    wav = (torch.randn(batch * n + 9, generator=g) * 0.1).cuda()
    off = [9 + i * n for i in range(batch)]
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.emb_forward_utt(wav, off, n))
    assert new.shape == (batch, 1, 256)
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)
    assert n_ref - n_new == 3


def test_bottleneck_trunk_layer3_pairs_match_per_tap():
    c = _context(syn.make_bottleneck_state_dict(152, 2))
    fb = _fbank(2, 1520)
    new, ref, n_new, n_ref = _both(c, lambda: c.emb_trunk(fb))
    assert new.shape == (2, 1024, 10, 125)
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)
    assert n_new == n_ref
