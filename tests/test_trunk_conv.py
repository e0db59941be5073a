"""Trunk convolutions: the wgmma kernels (conv_impl = 1) against the fp32 CUDA-core twin (conv_impl = 0).

The batch sizes cover one segment, an odd handful, exactly one embedding sub-batch (264) and one more segment than
that (two sub-batches).  The input is random non-zero fbank of the real shape, so every zero-padded border pixel and
the last partial 128-pixel strip of each layer (998, 499, 250 and 125 are not multiples of 128) carry data.
Tolerance as in test_gpu_parity.test_embedding_parity.
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


@pytest.mark.parametrize("batch", [1, 3, 264, 265])
def test_trunk_tensor_cores_match_cuda_cores(ctx, batch):
    g = torch.Generator().manual_seed(batch)
    fb = (torch.randn((batch, 998, 80), generator=g) * 2.0 + 0.5).cuda()
    out = {}
    try:
        for impl in (0, 1):
            ctx.set_option("conv_impl", impl)
            out[impl] = ctx.emb_trunk(fb).cpu().numpy()
    finally:
        ctx.set_option("conv_impl", 1)
    assert out[1].shape == (batch, 256, 10, 125)
    assert np.isfinite(out[1]).all()
    scale = np.abs(out[0]).max()
    assert scale > 0
    assert np.abs(out[1] - out[0]).max() <= 2e-2 * scale
    # each segment on its own: a wrong tile or strip shows as one segment far off while the batch maximum still passes
    err = np.abs(out[1] - out[0]).reshape(batch, -1).max(1) / np.abs(out[0]).reshape(batch, -1).max(1)
    assert err.max() <= 2e-2, f"worst segment {int(err.argmax())}: relative error {err.max()}"
