"""Generic multi-label segmentation pipeline (mirror of /root/reference/src/pyannote/audio/pipelines/multilabel.py):
PyanNet with a sigmoid head slid over the file, the scores overlap-added on the device (b200_aggregate), then hysteresis
thresholding of each label with its own onset / offset (vectorised signal.Binarize)."""
from __future__ import annotations

from typing import Callable, Mapping, Optional, Union

import torch

from .audio import AudioFile
from .core import Annotation, SlidingWindowFeature
from .inference import Inference
from .models import PyanNet, SSeRiouSS
from .signal import Binarize


class MultiLabelSegmentation:
    """``segmentation``: a multi-label PyanNet, or a checkpoint path / {"checkpoint": ...} entry.  Hyper-parameters:
    per label ``thresholds[label]`` = {onset, offset, min_duration_on, min_duration_off}; with ``share_min_duration``
    the two durations are the pipeline's ``min_duration_on`` / ``min_duration_off`` instead.  Until instantiated,
    onset = offset = 0.5 and the durations are 0."""

    def __init__(self, segmentation: Union[PyanNet, SSeRiouSS, Mapping, str, None] = None, fscore: bool = False,
                 share_min_duration: bool = False, token=None, cache_dir=None, device: Optional[torch.device] = None,
                 **inference_kwargs):
        from .loading import get_model, is_checkpoint_spec

        if segmentation is None:
            raise ValueError("MultiLabelSegmentation pipeline must be provided with a `segmentation` model.")
        self.segmentation, self.fscore, self.share_min_duration = segmentation, fscore, share_min_duration
        model = get_model(segmentation, token=token, cache_dir=cache_dir) if is_checkpoint_spec(segmentation) \
            else segmentation
        if not isinstance(model, (PyanNet, SSeRiouSS)):
            raise ValueError("`segmentation` must be a PyanNet instance or a local checkpoint (no hub access here)")
        device = device or torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        model.to(device)
        self._classes = list(model.specifications.classes)
        self._segmentation = Inference(model, **inference_kwargs)
        if self.share_min_duration:
            self.min_duration_on = self.min_duration_off = 0.0
            self.thresholds = {label: {"onset": 0.5, "offset": 0.5} for label in self._classes}
        else:
            self.thresholds = {label: {"onset": 0.5, "offset": 0.5, "min_duration_on": 0.0, "min_duration_off": 0.0}
                               for label in self._classes}
        self.initialize()

    def classes(self):
        return self._classes

    def default_parameters(self):
        raise NotImplementedError()

    def instantiate(self, params: dict):
        """pyannote.pipeline's nested parameters: {"thresholds": {label: {"onset": ..., ...}}, "min_duration_on": ...,
        "min_duration_off": ...} (the last two with ``share_min_duration``)."""
        for label, values in (params.get("thresholds") or {}).items():
            if label not in self.thresholds:
                raise ValueError(f"unknown label '{label}' (the model's classes are {self._classes})")
            for k, v in values.items():
                if k not in self.thresholds[label]:
                    raise ValueError(f"unknown hyper-parameter thresholds.{label}.{k}")
                self.thresholds[label][k] = float(v)
        if self.share_min_duration:
            for k in ("min_duration_on", "min_duration_off"):
                if k in params:
                    setattr(self, k, float(params[k]))
        self.initialize()
        return self

    def initialize(self):
        def durations(label):
            if self.share_min_duration:
                return self.min_duration_on, self.min_duration_off
            return self.thresholds[label]["min_duration_on"], self.thresholds[label]["min_duration_off"]

        self._binarize = {label: Binarize(onset=self.thresholds[label]["onset"], offset=self.thresholds[label]["offset"],
                                          min_duration_on=durations(label)[0], min_duration_off=durations(label)[1])
                          for label in self._classes}

    def apply(self, file: AudioFile, hook: Optional[Callable] = None) -> Annotation:
        file = self._segmentation.model.audio.validate_file(file)
        user_hook = hook
        hook = (lambda *a, **k: user_hook(*a, file=file, **k)) if user_hook is not None else (lambda *a, **k: None)
        segmentations: SlidingWindowFeature = self._segmentation(file, hook=lambda **k: hook("segmentation", None, **k))
        hook("segmentation", segmentations)
        detection = Annotation(uri=file.get("uri"))
        for i, label in enumerate(self._classes):
            scores = SlidingWindowFeature(segmentations.data[:, i: i + 1], segmentations.sliding_window)
            for segment, track, _ in self._binarize[label](scores).itertracks(yield_label=True):
                detection.add(segment, track, label)
        return detection

    __call__ = apply

    def get_direction(self):
        return "maximize" if self.fscore else "minimize"
