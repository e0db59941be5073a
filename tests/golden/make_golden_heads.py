"""Generates tests/golden/reference_heads_vectors.npz by EXECUTING the reference's own
models/segmentation/PyanNet.py and utils/powerset.py where they lie under the reference checkout -- run once in the
build container:

    PYTHONPATH=. python tests/golden/make_golden_heads.py

The import stubs of make_golden_apply.py load sincnet.py and PyanNet.py; its `Model` stand-in gets the activation rule
of core/model.py:271-300 (sigmoid for binary and multi-label problems, log-softmax for mono-label ones), and
PyanNet.build() makes the classifier of `dimension` outputs from the specifications.  With
make_segmentation_state_dict(0, num_classes=K) weights the generator records, for a binary head (K = 1), multi-label
heads of 4 and 32 labels and a powerset head of 4 speakers with at most 2 per frame (K = 11), the outputs at 1261,
80000 and 160000 samples; the reference's Powerset mappings for (3, 2), (4, 2), (4, 3) and (2, 1); each head's
`dimension`; and the sorted state-dict keys.  Nothing here is needed at test time; the committed .npz is.
"""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_apply as A  # noqa: E402
import make_golden_pipeline as G  # noqa: E402

from pyannote_audio_b200.testing import synthetic as syn  # noqa: E402

# name -> (problem, labels, powerset max per frame or None)
HEADS = {"binary": ("BINARY_CLASSIFICATION", 1, None), "multilabel": ("MULTI_LABEL_CLASSIFICATION", 4, None),
         "wide": ("MULTI_LABEL_CLASSIFICATION", 32, None), "powerset42": ("MONO_LABEL_CLASSIFICATION", 4, 2)}
LENGTHS = {"min": (1261, 2), "5s": (80000, 2), "10s": (160000, 1)}      # samples, batch
SEEDS = (41, 42)


def audio(n, batch):
    return torch.cat([syn.make_conversation(n / 16000, seed=s)[None] for s in SEEDS[:batch]])[..., :n]


def default_activation(self):
    if self.specifications.problem in ("BINARY_CLASSIFICATION", "MULTI_LABEL_CLASSIFICATION"):
        return torch.nn.Sigmoid()
    return torch.nn.LogSoftmax(dim=-1)


def main():
    G.load_reference()
    A.Model.default_activation = default_activation
    mods = A.load_models(None)
    powerset = G.load("pyannote.audio.utils.powerset", "utils/powerset.py")
    out = {}
    for n, m in ((3, 2), (4, 2), (4, 3), (2, 1)):
        out[f"mapping_{n}_{m}"] = powerset.Powerset(n, m).mapping.numpy().astype(np.uint8)
    with torch.no_grad():
        for name, (problem, labels, max_per_frame) in HEADS.items():
            classes = [f"label#{i}" for i in range(labels)]
            k = powerset.Powerset(labels, max_per_frame).num_powerset_classes if max_per_frame else labels
            net = mods["pyannet"].PyanNet(lstm={"num_layers": 4})
            net.specifications = types.SimpleNamespace(problem=problem, classes=classes,
                                                       powerset=max_per_frame is not None, num_powerset_classes=k)
            net.build()
            net.load_state_dict(syn.make_segmentation_state_dict(0, num_classes=k), strict=True)
            net.eval()
            out[f"dimension_{name}"] = np.array(net.dimension, dtype=np.int64)
            if name == "binary":
                out["keys"] = np.array(sorted(net.state_dict().keys()))
            for tag, (samples, batch) in LENGTHS.items():
                out[f"{name}_{tag}"] = net(audio(samples, batch)).numpy()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_heads_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
