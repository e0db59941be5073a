"""Trunk layer 2: the row kernel's epilogue stages the residual row in shared memory by TMA and writes the output row
with one TMA store (conv_impl = 1), against the per-tap wgmma kernel (conv_impl = 2).  The arithmetic is the same
(+bias, +residual, ReLU, fp16), so the results are bit-identical, and the launch counts do not change.

The 10 s batches give short bands (1 and 3 segments), full-height bands (264) and a remainder sub-batch (265).  The
any-length path covers fbank widths T0 whose layer-2 width (T0 - 1) // 2 + 1 is 1, 127, 128, 129, 256 and 257 pixels:
stores clipped at W_out and residual columns beyond it zero-filled.  The bottleneck trunk runs the row kernel without a
residual (the conv2 of its layers 1 and 2, 32 and 64 channels), the store-only epilogue.
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
    return _context(syn.make_embedding_state_dict(6))


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
def test_trunk_row_epilogue_matches_per_tap(ctx, batch):
    fb = _fbank(batch, 4000 + batch)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.emb_trunk(fb))
    assert new.shape == (batch, 256, 10, 125)
    assert np.abs(ref).max() > 0
    assert np.array_equal(new, ref)
    calls = -(-batch // 264)                      # emb_trunk sub-batches of emb_max_batch = 264 segments
    assert n_ref - n_new == 3 * calls             # only the fused layer-1 blocks launch fewer kernels


# layer-2 width W2 = (T0 - 1) // 2 + 1: 1, 127, 128, 129, 256, 257 pixels
@pytest.mark.parametrize("t0", [1, 253, 255, 257, 511, 513])
def test_utterance_row_epilogue_matches_per_tap(ctx, t0):
    batch = 2
    n = 400 + 160 * (t0 - 1)                 # T0 = 1 + (n - 400) // 160 fbank frames
    g = torch.Generator().manual_seed(t0 * 10 + 4)
    wav = (torch.randn(batch * n + 7, generator=g) * 0.1).cuda()
    off = [7 + i * n for i in range(batch)]
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.emb_forward_utt(wav, off, n))
    assert new.shape == (batch, 1, 256)
    if t0 >= 9:                              # shorter inputs pool to NaN statistics on both paths
        assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref, equal_nan=True)
    assert n_ref - n_new == 3


def test_chunk_embeddings_with_masks_row_epilogue_matches_per_tap(ctx):
    g = torch.Generator().manual_seed(12)
    wav = (torch.randn(16000 * 39 + 8000, generator=g) * 0.1).cuda()
    off = np.arange(0, 16000 * 31, 16000, dtype=np.int64)          # 10 s chunks every second, the last one short
    valid = np.minimum(160000, wav.numel() - off).astype(np.int32)
    masks = (torch.rand((len(off), 3, 589), generator=g) < 0.5).to(torch.uint8)
    masks[0, 2] = 0
    masks = masks.cuda()
    new, ref, _, _ = _both(ctx, lambda: ctx.emb_forward(wav, off, valid, masks))
    assert new.shape == (len(off), 3, 256)
    assert np.isfinite(ref[:, :2]).all() and np.abs(ref[:, :2]).max() > 0
    assert np.array_equal(new, ref, equal_nan=True)


def test_bottleneck_trunk_store_only_epilogue_matches_per_tap():
    c = _context(syn.make_bottleneck_state_dict(152, 3))
    fb = _fbank(3, 1521)
    new, ref, n_new, n_ref = _both(c, lambda: c.emb_trunk(fb))
    assert new.shape == (3, 1024, 10, 125)
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(new, ref)
    assert n_new == n_ref
