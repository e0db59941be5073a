"""Trunk convolutions: the persistent chunk-row kernel of layers 3 and 4 (conv_impl = 1) against the per-tap wgmma
kernel (conv_impl = 2).  Both sum each output's products in the (tap, channel chunk, 16-channel step) order, so the
results are bit-identical.

The 10 s batches cover one segment and an odd handful (fewer output tiles than CTAs), exactly one embedding
sub-batch and one more segment than that.  The any-length path covers fbank widths T0 whose layer-3 (about T0 / 4)
and layer-4 (about T0 / 8) rows end just below, at and just beyond the 128-pixel column tile and its 136-pixel box,
plus many column tiles.  The bottleneck trunk runs the same kernel on the conv2 of its layer-3 and layer-4 blocks.
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
    return _context(syn.make_embedding_state_dict(1))


def _both(ctx, run):
    out = {}
    try:
        for impl in (2, 1):
            ctx.set_option("conv_impl", impl)
            out[impl] = run().cpu().numpy()
    finally:
        ctx.set_option("conv_impl", 1)
    return out[1], out[2]


def _fbank(batch, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((batch, 998, 80), generator=g) * 2.0 + 0.5).cuda()


@pytest.mark.parametrize("batch", [1, 2, 3, 264, 265])
def test_trunk_chunk_row_kernel_matches_per_tap(ctx, batch):
    fb = _fbank(batch, 2000 + batch)
    new, ref = _both(ctx, lambda: ctx.emb_trunk(fb))
    assert new.shape == (batch, 256, 10, 125)
    assert np.abs(ref).max() > 0
    assert np.array_equal(new, ref)


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("t0", [9, 512, 513, 544, 545, 1024, 1025, 1088, 1089, 4097])
def test_utterance_chunk_row_kernel_matches_per_tap(ctx, batch, t0):
    n = 400 + 160 * (t0 - 1)                 # T0 = 1 + (n - 400) // 160 fbank frames
    g = torch.Generator().manual_seed(t0 * 10 + batch + 1)
    wav = (torch.randn(batch * n + 7, generator=g) * 0.1).cuda()
    off = [7 + i * n for i in range(batch)]
    new, ref = _both(ctx, lambda: ctx.emb_forward_utt(wav, off, n))
    assert new.shape == (batch, 1, 256)
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)


def test_bottleneck_trunk_chunk_row_kernel_matches_per_tap():
    c = _context(syn.make_bottleneck_state_dict(152, 1))
    fb = _fbank(3, 152)
    new, ref = _both(c, lambda: c.emb_trunk(fb))
    assert new.shape == (3, 1024, 10, 125)
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)
