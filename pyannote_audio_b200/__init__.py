"""pyannote_audio_b200 -- H100-native (sm_90a) implementation of pyannote.audio's community-1 diarization hot path.

Public surface mirrors the reference for this path only:
  Inference, Model classes (PyanNet, SSeRiouSS, WeSpeakerResNet34 / 152 / 221 / 293, XVectorSincNet,
  XVectorMFCC), SpeakerDiarization (+ DiarizeOutput), SpeakerEmbedding,
  VoiceActivityDetection, MultiLabelSegmentation, VBxClustering,
  AgglomerativeClustering, PLDA, Audio, and the pyannote.core value types they exchange.
All compute goes through libb200diar.so (C ABI in include/b200diar.h); there is no CPU fallback.
"""
from .core import (Annotation, Problem, Resolution, Segment, SlidingWindow, SlidingWindowFeature,  # noqa: F401
                   Specifications)

__version__ = "0.1.0"

_LAZY = {
    "Audio": "audio", "Inference": "inference", "BaseInference": "inference", "Model": "models", "PyanNet": "models",
    "WeSpeakerResNet34": "models", "WeSpeakerResNet152": "models", "WeSpeakerResNet221": "models",
    "WeSpeakerResNet293": "models", "BaseWeSpeakerResNet": "models", "XVectorSincNet": "models", "XVectorMFCC": "models",
    "BaseXVector": "models", "SSeRiouSS": "models",
    "SpeakerDiarization": "pipeline", "DiarizeOutput": "pipeline",
    "PretrainedSpeakerEmbedding": "pipeline", "VBxClustering": "clustering",
    "AgglomerativeClustering": "clustering", "PLDA": "clustering", "VoiceActivityDetection": "vad",
    "MultiLabelSegmentation": "multilabel",
    "Binarize": "signal", "Pipeline": "loading", "SpeakerEmbedding": "speaker_verification",
}


def __getattr__(name):
    if name == "synthetic":        # fixtures live in pyannote_audio_b200.testing; old import path kept as an alias
        import importlib

        return importlib.import_module(".testing.synthetic", __name__)
    if name in _LAZY:
        import importlib

        return getattr(importlib.import_module(f".{_LAZY[name]}", __name__), name)
    raise AttributeError(name)
