"""Trunk layer 1: each stride-1 BasicBlock as one fused kernel (conv_impl = 1) against two per-tap wgmma convs per
block (conv_impl = 2).  The fused kernel keeps the intermediate activation in shared memory but rounds it to fp16 as
the unfused path stores it, and sums each output's products in the same order, so the results are bit-identical.

The 10 s batches cover short bands (one segment, an odd handful), full-height bands (one embedding sub-batch) and a
remainder sub-batch.  The any-length path covers fbank widths T0 around the fused kernel's 126-column strip and its
136-pixel box: a single strip of one or a few columns, strips that end exactly at or just past the image, and many
strips.  Below T0 = 9 the embedding is NaN (the std of one trunk frame), so those cases check the NaN pattern only.
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
    c.load_embedding(syn.make_embedding_state_dict(3))
    return c


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
    return out[1], out[2], launches[2] - launches[1]


@pytest.mark.parametrize("batch", [1, 3, 264, 265])
def test_trunk_fused_block_matches_per_tap(ctx, batch):
    g = torch.Generator().manual_seed(2000 + batch)
    fb = (torch.randn((batch, 998, 80), generator=g) * 2.0 + 0.5).cuda()
    new, ref, saved = _both(ctx, lambda: ctx.emb_trunk(fb))
    assert new.shape == (batch, 256, 10, 125)
    assert np.abs(ref).max() > 0
    assert np.array_equal(new, ref)
    calls = -(-batch // 264)                      # emb_trunk sub-batches of emb_max_batch = 264 segments
    assert saved == 3 * calls                     # the three layer-1 blocks: one launch each instead of two


@pytest.mark.parametrize("t0", [1, 2, 3, 125, 126, 127, 128, 129, 252, 253, 998, 4097])
def test_utterance_fused_block_matches_per_tap(ctx, t0):
    batch = 2
    n = 400 + 160 * (t0 - 1)                 # T0 = 1 + (n - 400) // 160 fbank frames
    g = torch.Generator().manual_seed(t0 * 10 + 7)
    wav = (torch.randn(batch * n + 5, generator=g) * 0.1).cuda()
    off = [5 + i * n for i in range(batch)]
    new, ref, _ = _both(ctx, lambda: ctx.emb_forward_utt(wav, off, n))
    assert new.shape == (batch, 1, 256)
    if t0 >= 9:
        assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref, equal_nan=True)


def test_chunk_embeddings_with_masks_fused_block_matches_per_tap(ctx):
    g = torch.Generator().manual_seed(11)
    wav = (torch.randn(16000 * 39 + 8000, generator=g) * 0.1).cuda()
    off = np.arange(0, 16000 * 31, 16000, dtype=np.int64)          # 10 s chunks every second, the last one short
    valid = np.minimum(160000, wav.numel() - off).astype(np.int32)
    masks = (torch.rand((len(off), 3, 589), generator=g) < 0.5).to(torch.uint8)
    masks[0, 2] = 0
    masks = masks.cuda()
    new, ref, _ = _both(ctx, lambda: ctx.emb_forward(wav, off, valid, masks))
    assert new.shape == (len(off), 3, 256)
    assert np.isfinite(ref[:, :2]).all() and np.abs(ref[:, :2]).max() > 0
    assert np.array_equal(new, ref, equal_nan=True)
