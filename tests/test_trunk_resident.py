"""Trunk convolutions: the persistent row kernel of layers 1 and 2 (conv_impl = 1) against the per-tap wgmma kernel
(conv_impl = 2) for every conv.  Both sum each output's products in the same order, so the results are bit-identical.

The 10 s batches cover one segment and an odd handful (short bands so that every SM has work), exactly one embedding
sub-batch (full-height bands) and one more segment than that.  The any-length path covers fbank widths T0 around the
128-pixel column tile and its 136-pixel box: a single strip of one or a few pixels, partial last strips and many
strips.  At the narrowest widths the embedding is NaN (see below), so those cases check the launch and the NaN
pattern only.
"""
import numpy as np
import pytest
import torch

from pyannote_audio_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyannote_audio_b200 import ops

    c = ops.Context(torch.device("cuda:0"))
    c.load_embedding(syn.make_embedding_state_dict(1))
    return c


def _both(ctx, run):
    out = {}
    try:
        for impl in (2, 1):
            ctx.set_option("conv_impl", impl)
            out[impl] = run().cpu().numpy()
    finally:
        ctx.set_option("conv_impl", 1)
    return out[1], out[2]


@pytest.mark.parametrize("batch", [1, 3, 264, 265])
def test_trunk_row_kernel_matches_per_tap(ctx, batch):
    g = torch.Generator().manual_seed(1000 + batch)
    fb = (torch.randn((batch, 998, 80), generator=g) * 2.0 + 0.5).cuda()
    new, ref = _both(ctx, lambda: ctx.emb_trunk(fb))
    assert new.shape == (batch, 256, 10, 125)
    assert np.abs(ref).max() > 0
    assert np.array_equal(new, ref)


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("t0", [1, 2, 3, 127, 128, 129, 136, 998, 4097])
def test_utterance_row_kernel_matches_per_tap(ctx, batch, t0):
    n = 400 + 160 * (t0 - 1)                 # T0 = 1 + (n - 400) // 160 fbank frames
    g = torch.Generator().manual_seed(t0 * 10 + batch)
    wav = (torch.randn(batch * n + 7, generator=g) * 0.1).cuda()
    off = [7 + i * n for i in range(batch)]
    new, ref = _both(ctx, lambda: ctx.emb_forward_utt(wav, off, n))
    assert new.shape == (batch, 1, 256)
    # below T0 = 9 the trunk leaves one frame and the std (correction 1) of the pooling is NaN in both
    if t0 >= 9:
        assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref, equal_nan=True)
