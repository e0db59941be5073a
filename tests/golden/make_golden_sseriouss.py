"""Generates tests/golden/reference_sseriouss_vectors.npz by EXECUTING the reference's
models/segmentation/SSeRiouSS.py where it lies under the reference checkout, with the real torchaudio -- run once in
the build container:

    PYTHONPATH=. python tests/golden/make_golden_sseriouss.py

The import stubs of make_golden_pipeline.py / make_golden_apply.py (pyannote.core stand-in, the `Model` stand-in) load
SSeRiouSS.py.  torchaudio.pipelines.WAVLM_BASE.get_model would download the pretrained weights; it is replaced by
torchaudio.models.wavlm_model(**WAVLM_BASE._params), a randomly initialised WavLM Base, whose weights are then
overwritten with make_sseriouss_state_dict(5, ...) through the reference module's own load_state_dict(strict=True).
Recorded: for a powerset head of 3 speakers (7 classes) with the layer average (wav2vec_layer -1) and a 4-label
sigmoid head on layer 6, the outputs at 400, 80000 and 160000 samples; the receptive field (size of 1 and 2 frames,
centre of frame 0); and the sorted state-dict keys with wav2vec_layer -1 and 3.  Nothing here is needed at test time;
the committed .npz is.
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

CASES = {"powerset_avg": (-1, "MONO_LABEL_CLASSIFICATION", 7), "sigmoid_layer6": (6, "MULTI_LABEL_CLASSIFICATION", 4)}
LENGTHS = {"min": (400, 2), "5s": (80000, 1), "10s": (160000, 1)}      # samples, batch
SEEDS = (41, 42)


def audio(n, batch):
    return torch.cat([syn.make_conversation(max(n, 16000) / 16000, seed=s) for s in SEEDS[:batch]])[..., :n]


def default_activation(self):
    if self.specifications.problem in ("BINARY_CLASSIFICATION", "MULTI_LABEL_CLASSIFICATION"):
        return torch.nn.Sigmoid()
    return torch.nn.LogSoftmax(dim=-1)


def main():
    import torchaudio

    G.load_reference()
    A.Model.default_activation = default_activation
    A.load_models(None)
    task = sys.modules["pyannote.audio.core.task"]
    if not hasattr(task, "Task"):
        task.Task = object
    bundle = torchaudio.pipelines.WAVLM_BASE
    bundle.get_model = lambda *a, **k: torchaudio.models.wavlm_model(**bundle._params)   # no download
    mod = G.load("pyannote.audio.models.segmentation.SSeRiouSS", "models/segmentation/SSeRiouSS.py")
    out = {}
    with torch.no_grad():
        for case, (layer, problem, k) in CASES.items():
            net = mod.SSeRiouSS(wav2vec="WAVLM_BASE", wav2vec_layer=layer, lstm={"num_layers": 4})
            net.specifications = types.SimpleNamespace(problem=problem, classes=[f"c{i}" for i in range(k)],
                                                       powerset=problem == "MONO_LABEL_CLASSIFICATION",
                                                       num_powerset_classes=k)
            net.build()
            net.load_state_dict(syn.make_sseriouss_state_dict(5, wav2vec_layer=layer, num_classes=k), strict=True)
            net.eval()
            for length, (n, batch) in LENGTHS.items():
                out[f"{case}_{length}"] = net(audio(n, batch)[:, None]).numpy().astype(np.float32)
            if case == "powerset_avg":
                out["receptive_field"] = np.array([net.receptive_field_size(1), net.receptive_field_size(2),
                                                   net.receptive_field_center(0)], dtype=np.int64)
        for layer in (-1, 3):
            net = mod.SSeRiouSS(wav2vec="WAVLM_BASE", wav2vec_layer=layer)
            net.specifications = types.SimpleNamespace(problem="MONO_LABEL_CLASSIFICATION", classes=["a", "b", "c"],
                                                       powerset=True, num_powerset_classes=7)
            net.build()
            out[f"keys_layer{layer}"] = np.array(sorted(net.state_dict().keys()))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_sseriouss_vectors.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
