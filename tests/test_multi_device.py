"""Two library contexts on two devices of one process.  The shared-memory opt-in of a kernel
(cudaFuncAttributeMaxDynamicSharedMemorySize) belongs to the kernel as loaded in one device's context, so every kernel
that needs more than 48 KB must be opted in on each device it runs on: the split-precision GEMMs, the SincNet layers
(wgmma and fp32), the wgmma LSTM recurrence and the centroid linkage.  Both devices run the same seeded inputs and
must give bit-identical outputs."""
import numpy as np
import pytest
import torch

from pyannote_audio_b200 import ops
from pyannote_audio_b200.core import Problem, Resolution, Specifications
from pyannote_audio_b200.testing import synthetic as syn

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible CUDA devices")]

OFF = np.array([0, 160000, 80000], dtype=np.int64)
VALID = np.array([160000, 160000, 120000], dtype=np.int32)


def _run(ctx):
    dev = ctx.device
    wav = torch.cat([syn.make_conversation(10.0, seed=s) for s in (5, 6)], dim=1).reshape(-1).contiguous().to(dev)
    out = {}
    ctx.load_segmentation(syn.make_segmentation_state_dict(0))
    out["powerset"], out["logp"] = ctx.seg_forward(wav, OFF, VALID, return_logp=True)
    ctx.set_option("seg_conv_impl", 0)                    # the fp32 CUDA-core SincNet layers
    out["powerset, fp32 sincnet"] = ctx.seg_forward(wav, OFF, VALID)
    ctx.set_option("seg_conv_impl", 1)
    specs = Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, 10.0,
                           classes=[f"label#{i}" for i in range(4)])
    ctx.load_segmentation(syn.make_segmentation_state_dict(0, num_classes=4), specs)
    out["sigmoid"] = ctx.seg_forward(wav, OFF, VALID)
    ctx.load_embedding(syn.make_embedding_state_dict(1))
    masks = torch.rand((len(OFF), ops.SPEAKERS, ops.FRAMES), generator=torch.Generator().manual_seed(0)) > 0.3
    out["resnet34"] = ctx.emb_forward(wav, OFF, VALID, masks.to(torch.uint8).to(dev))
    ctx.load_xvector(syn.make_xvector_state_dict(3))
    out["xvector"] = ctx.xvec_forward(wav, [0, 48000], 64000)
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((700, 256))).to(dev)
    out["linkage"] = ctx.linkage_centroid_batched(x, [0, 200, 700])
    torch.cuda.synchronize(dev)
    return {k: v.cpu().numpy() for k, v in out.items()}


def test_two_devices_in_one_process_give_identical_outputs():
    ctxs = [ops.Context("cuda:0"), ops.Context("cuda:1")]
    try:
        first, second = (_run(c) for c in ctxs)
    finally:
        for c in ctxs:
            c.close()
    assert first.keys() == second.keys()
    for k in first:
        assert np.array_equal(first[k], second[k]), k
