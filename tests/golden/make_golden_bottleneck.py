"""Generates tests/golden/reference_bottleneck_vectors.npz by EXECUTING the reference's own resnet.py where it lies
under /root/reference (oracle/ref_loader.py) -- run once in the build container:

    PYTHONPATH=. python tests/golden/make_golden_bottleneck.py

For each of ResNet152 / 221 / 293 (Bottleneck blocks, two_emb_layer=False) with make_bottleneck_state_dict weights:
the embedding of a (2, 120, 80) fbank batch with and without binary weights, and the reference's sorted state-dict
keys.  Nothing here is needed at test time; the committed .npz is.
"""
import os

import numpy as np
import torch

from oracle import ref_loader
from pyannote_audio_b200.testing import synthetic as syn

ref = ref_loader.load_all()["resnet"]
out = {}
g = torch.Generator().manual_seed(2930)
fb = torch.randn(2, 120, 80, generator=g)
wts = (torch.rand(2, 15, generator=g) > 0.3).float()
out["fbank"], out["weights"] = fb.numpy(), wts.numpy()
with torch.no_grad():
    for depth in (152, 221, 293):
        net = getattr(ref, f"ResNet{depth}")(feat_dim=80, embed_dim=256, two_emb_layer=False)
        sd = {k[len("resnet."):]: v for k, v in syn.make_bottleneck_state_dict(depth, 1).items()}
        net.load_state_dict(sd, strict=True)
        net.eval()
        out[f"emb_{depth}"] = net(fb.clone(), weights=wts)[1].numpy()
        out[f"emb_noweights_{depth}"] = net(fb.clone())[1].numpy()
        out[f"keys_{depth}"] = np.array(sorted(net.state_dict().keys()))

path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_bottleneck_vectors.npz")
np.savez_compressed(path, **out)
print("wrote", path, {k: v.shape for k, v in out.items()})
