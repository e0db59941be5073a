"""Generates tests/golden/reference_xvector_mfcc_vectors.npz by EXECUTING the reference's own
models/embedding/xvector.py where it lies under the reference checkout -- run once in the build container:

    PYTHONPATH=. python tests/golden/make_golden_xvector_mfcc.py

The module is loaded as make_golden_xvector.py loads it; XVectorMFCC's front end is torchaudio's MFCC.  With
make_xvector_mfcc_state_dict(5) weights the generator records XVectorMFCC embeddings at 2800 samples, an odd length
and 10 s, without weights, with 2-D soft weights and with 3-D weights of another frame count; num_frames /
receptive-field figures at several lengths; that 2799 samples raise and 2800 do not; and the sorted state-dict keys.
Nothing here is needed at test time; the committed .npz is.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_apply as A  # noqa: E402
import make_golden_pipeline as G  # noqa: E402

from pyannote_audio_b200.testing import synthetic as syn  # noqa: E402

LENGTHS = (("min", 2800), ("odd", 36817), ("10s", 160000))


def main():
    G.load_reference()
    A.load_models(None)
    task = sys.modules.get("pyannote.audio.core.task") or G.stub("pyannote.audio.core.task")
    if not hasattr(task, "Task"):
        task.Task = type("Task", (), {})
    xv = G.load("pyannote.audio.models.embedding.xvector", "models/embedding/xvector.py")
    torch.manual_seed(0)
    net = xv.XVectorMFCC()
    net.load_state_dict(syn.make_xvector_mfcc_state_dict(5), strict=True)
    net.eval()
    out = {"keys": np.array(sorted(net.state_dict().keys()))}
    g = torch.Generator().manual_seed(2800)
    with torch.no_grad():
        for name, n in LENGTHS:
            wav = torch.cat([syn.make_conversation(n / 16000, seed=s)[None] for s in (11, 12)])[..., :n]
            T = net.num_frames(n)
            w2 = torch.rand(2, T, generator=g)
            w3 = torch.rand(2, 3, T + 7, generator=g) * (torch.rand(2, 3, T + 7, generator=g) > 0.3)
            out[f"w2_{name}"], out[f"w3_{name}"] = w2.numpy(), w3.numpy()   # the audio is regenerated from its seeds
            out[f"emb_{name}"] = net(wav).numpy()
            out[f"emb_w2_{name}"] = net(wav, weights=w2).numpy()
            out[f"emb_w3_{name}"] = net(wav, weights=w3).numpy()
        lengths = np.array([2800, 2999, 3000, 16000, 36817, 160000, 480000], dtype=np.int64)
        out["lengths"] = lengths
        out["num_frames"] = np.array([net.num_frames(int(n)) for n in lengths], dtype=np.int64)
        out["rf_size"] = np.array([net.receptive_field_size(k) for k in (1, 2, 10)], dtype=np.int64)
        out["rf_center"] = np.array([net.receptive_field_center(k) for k in (0, 1, 10)], dtype=np.int64)
        raised = []
        for n in (2799, 2800):
            try:
                net(torch.zeros(1, 1, n))
                raised.append(0)
            except RuntimeError:
                raised.append(1)
        out["raises_2799_2800"] = np.array(raised, dtype=np.int64)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_xvector_mfcc_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
