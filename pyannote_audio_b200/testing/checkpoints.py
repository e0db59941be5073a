"""Test fixture: a Lightning-format ``pytorch_model.bin`` laid out as the reference writes it
(/root/reference/src/pyannote/audio/core/model.py:244-256), built without lightning / pyannote.audio."""
import torch

from . import synthetic as syn


def reference_style_checkpoint(kind):
    """``kind``: "seg" (PyanNet, community-1 head), "seg_multilabel" (PyanNet with a 4-label sigmoid head,
    permutation_invariant=False), "seg_binary" (a 1-class sigmoid ["speech"] head), "seg_powerset42" (a powerset
    head of 4 speakers with at most 2 per frame, 11 classes), "emb" (WeSpeakerResNet34), "emb293"
    (WeSpeakerResNet293), "xvec" (XVectorSincNet), "xvec_mfcc" (XVectorMFCC) or "sseriouss" (SSeRiouSS on WavLM Base, 4-label sigmoid head).  A Lightning-format pytorch_model.bin as the reference writes it (model.py:244-256): state_dict +
    hyper_parameters + checkpoint["pyannote.audio"] whose `specifications` is pickled under the REFERENCE's module
    path pyannote.audio.core.task (registered here only while pickling, then removed again)."""
    import dataclasses
    import enum
    import io
    import sys
    import types

    names = ("pyannote", "pyannote.audio", "pyannote.audio.core", "pyannote.audio.core.task")
    saved = {n: sys.modules.get(n) for n in names}
    mods = {n: types.ModuleType(n) for n in names}
    sys.modules.update(mods)
    try:
        class Problem(enum.Enum):
            BINARY_CLASSIFICATION = 0
            MONO_LABEL_CLASSIFICATION = 1
            MULTI_LABEL_CLASSIFICATION = 2
            REPRESENTATION = 3
            REGRESSION = 4

        class Resolution(enum.Enum):
            FRAME = 1
            CHUNK = 2

        @dataclasses.dataclass
        class Specifications:
            problem: Problem
            resolution: Resolution
            duration: float
            min_duration: float = None
            warm_up: tuple = (0.0, 0.0)
            classes: list = None
            powerset_max_classes: int = None
            permutation_invariant: bool = False

        for c in (Problem, Resolution, Specifications):
            c.__module__, c.__qualname__ = "pyannote.audio.core.task", c.__name__
            setattr(mods["pyannote.audio.core.task"], c.__name__, c)
        heads = {"seg": (7, Specifications(Problem.MONO_LABEL_CLASSIFICATION, Resolution.FRAME, 10.0,
                                           classes=["speaker#1", "speaker#2", "speaker#3"], powerset_max_classes=2,
                                           permutation_invariant=True)),
                 "seg_multilabel": (4, Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, 5.0,
                                                      classes=["speech", "music", "noise", "laughter"])),
                 "seg_binary": (1, Specifications(Problem.BINARY_CLASSIFICATION, Resolution.FRAME, 5.0,
                                                  classes=["speech"])),
                 "seg_powerset42": (11, Specifications(Problem.MONO_LABEL_CLASSIFICATION, Resolution.FRAME, 10.0,
                                                       classes=[f"speaker#{i}" for i in range(1, 5)],
                                                       powerset_max_classes=2, permutation_invariant=True))}
        if kind in heads:
            num_classes, specs = heads[kind]
            ck = {"state_dict": syn.make_segmentation_state_dict(0, num_classes=num_classes),
                  "hyper_parameters": {"sincnet": {"stride": 10}, "linear": {"hidden_size": 128, "num_layers": 2},
                                       "lstm": {"hidden_size": 128, "num_layers": 4, "bidirectional": True,
                                                "monolithic": True, "dropout": 0.0},
                                       "sample_rate": 16000, "num_channels": 1},
                  "pyannote.audio": {"versions": {"pyannote.audio": "4.0.0"},
                                     "architecture": {"module": "pyannote.audio.models.segmentation.PyanNet",
                                                      "class": "PyanNet"},
                                     "specifications": specs}}
        elif kind == "emb293":
            ck = {"state_dict": syn.make_bottleneck_state_dict(293, 1),
                  "hyper_parameters": {"sample_rate": 16000, "num_channels": 1, "num_mel_bins": 80,
                                       "frame_length": 25, "frame_shift": 10, "dither": 0.0,
                                       "window_type": "hamming", "use_energy": False},
                  "pyannote.audio": {"versions": {"pyannote.audio": "4.0.0"},
                                     "architecture": {"module": "pyannote.audio.models.embedding.wespeaker",
                                                      "class": "WeSpeakerResNet293"},
                                     "specifications": Specifications(Problem.REPRESENTATION, Resolution.CHUNK, 10.0)}}
        elif kind == "sseriouss":
            # a WavLM Base SSeRiouSS with a 4-label sigmoid head, layer average, the pre-parametrization weight-norm
            # spelling of the positional conv (weight_g / weight_v)
            ck = {"state_dict": syn.make_sseriouss_state_dict(5, num_classes=4, pos_weight_norm="weight_g"),
                  "hyper_parameters": {"wav2vec": "WAVLM_BASE", "wav2vec_frozen": False, "wav2vec_layer": -1,
                                       "lstm": {"hidden_size": 128, "num_layers": 4, "bidirectional": True,
                                                "monolithic": True, "dropout": 0.0, "batch_first": True},
                                       "linear": {"hidden_size": 128, "num_layers": 2},
                                       "sample_rate": 16000, "num_channels": 1},
                  "pyannote.audio": {"versions": {"pyannote.audio": "4.0.0"},
                                     "architecture": {"module": "pyannote.audio.models.segmentation.SSeRiouSS",
                                                      "class": "SSeRiouSS"},
                                     "specifications": Specifications(
                                         Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, 5.0,
                                         classes=["speech", "music", "noise", "laughter"])}}
        elif kind == "xvec":
            ck = {"state_dict": syn.make_xvector_state_dict(3),
                  "hyper_parameters": {"sincnet": {"stride": 10, "sample_rate": 16000}, "dimension": 512,
                                       "sample_rate": 16000, "num_channels": 1},
                  "pyannote.audio": {"versions": {"pyannote.audio": "4.0.0"},
                                     "architecture": {"module": "pyannote.audio.models.embedding.xvector",
                                                      "class": "XVectorSincNet"},
                                     "specifications": Specifications(Problem.REPRESENTATION, Resolution.CHUNK, 3.0)}}
        elif kind == "xvec_mfcc":
            ck = {"state_dict": syn.make_xvector_mfcc_state_dict(5),
                  "hyper_parameters": {"mfcc": {"n_mfcc": 40, "dct_type": 2, "norm": "ortho", "log_mels": False,
                                                "sample_rate": 16000},
                                       "dimension": 512, "sample_rate": 16000, "num_channels": 1},
                  "pyannote.audio": {"versions": {"pyannote.audio": "4.0.0"},
                                     "architecture": {"module": "pyannote.audio.models.embedding.xvector",
                                                      "class": "XVectorMFCC"},
                                     "specifications": Specifications(Problem.REPRESENTATION, Resolution.CHUNK, 3.0)}}
        else:
            ck = {"state_dict": syn.make_embedding_state_dict(1),
                  "hyper_parameters": {"sample_rate": 16000, "num_channels": 1, "num_mel_bins": 80,
                                       "frame_length": 25, "frame_shift": 10, "dither": 0.0,
                                       "window_type": "hamming", "use_energy": False},
                  "pyannote.audio": {"versions": {"pyannote.audio": "4.0.0"},
                                     "architecture": {"module": "pyannote.audio.models.embedding.wespeaker",
                                                      "class": "WeSpeakerResNet34"},
                                     "specifications": Specifications(Problem.REPRESENTATION, Resolution.CHUNK, 10.0)}}
        ck["pytorch-lightning_version"] = "2.6.1"
        buf = io.BytesIO()
        torch.save(ck, buf)
        return buf.getvalue(), ck["state_dict"]
    finally:
        for n in names:
            if saved[n] is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = saved[n]
