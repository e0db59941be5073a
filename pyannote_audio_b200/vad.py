"""Voice activity detection pipeline (mirror of /root/reference/src/pyannote/audio/pipelines/
voice_activity_detection.py:66-204) reusing the diarization kernels: PyanNet sliding window -> speech score per
frame (max over the speakers of the powerset multilabel, or the maximum of a sigmoid head's scores, fused into its
classifier) -> Hamming-windowed overlap-add on the device (b200_aggregate) -> Binarize."""
from __future__ import annotations

from typing import Callable, Mapping, Optional, Union

import numpy as np
import torch

from .audio import AudioFile
from .core import Annotation, Segment, SlidingWindow, SlidingWindowFeature
from .inference import Inference, chunk_layout
from .models import PyanNet, SSeRiouSS
from .signal import Binarize


class VoiceActivityDetection:
    def __init__(self, segmentation: Union[PyanNet, SSeRiouSS, Mapping, str, None] = None, fscore: bool = False, token=None,
                 cache_dir=None, device: Optional[torch.device] = None, **inference_kwargs):
        from .loading import get_model, is_checkpoint_spec

        self.segmentation_id = segmentation if isinstance(segmentation, str) else None   # default_parameters' key
        if is_checkpoint_spec(segmentation):               # path / {"checkpoint": ...} from Pipeline.from_pretrained
            segmentation = get_model(segmentation, token=token, cache_dir=cache_dir)
        if isinstance(segmentation, Mapping):
            model = PyanNet()
            model.load_state_dict(segmentation)
            segmentation = model
        if not isinstance(segmentation, (PyanNet, SSeRiouSS)):
            raise ValueError("`segmentation` must be a PyanNet instance or its state dict (no hub access here)")
        self.segmentation, self.fscore = segmentation, fscore
        device = device or torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        segmentation.to(device)
        inference_kwargs["pre_aggregation_hook"] = lambda scores: np.max(scores, axis=-1, keepdims=True)
        self._segmentation = Inference(segmentation, **inference_kwargs)
        # powerset model: thresholds are fixed (voice_activity_detection.py:117-118); a sigmoid (multi-label or
        # binary) model has onset / offset hyper-parameters, 0.5 until instantiated
        self.powerset = segmentation.specifications.powerset
        self.onset = self.offset = 0.5
        self.min_duration_on = self.min_duration_off = 0.0
        self.initialize()

    def default_parameters(self):
        """voice_activity_detection.py:129-145: tuned values of pyannote/segmentation (DIHARD 3 development set) and
        pyannote/segmentation-3.0.0; a powerset model passed as an instance or state dict keeps its fixed thresholds."""
        if self.segmentation_id == "pyannote/segmentation":
            return {"onset": 0.767, "offset": 0.377, "min_duration_on": 0.136, "min_duration_off": 0.067}
        if self.segmentation_id == "pyannote/segmentation-3.0.0" or (self.segmentation_id is None and self.powerset):
            return {"min_duration_on": 0.0, "min_duration_off": 0.0}
        raise NotImplementedError()

    def instantiate(self, params: dict):
        for k in ("onset", "offset", "min_duration_on", "min_duration_off"):
            if k in params:
                setattr(self, k, float(params[k]))
        self.initialize()
        return self

    def classes(self):
        return ["SPEECH"]

    def initialize(self):
        self._binarize = Binarize(onset=self.onset, offset=self.offset, min_duration_on=self.min_duration_on,
                                  min_duration_off=self.min_duration_off)

    def speech_scores(self, file: AudioFile, hook: Optional[Callable] = None) -> SlidingWindowFeature:
        """Aggregated speech score per frame, (num_frames, 1) float32: what `self._segmentation(file)` returns in the
        reference (Inference with the max-over-speakers pre-aggregation hook), computed without leaving the device
        between the network and the overlap-add."""
        inf = self._segmentation
        waveform, sample_rate = inf.model.audio(file)
        specs = inf.model.specifications
        if self.powerset:
            cls, _, off, _ = inf.slide_device(waveform, sample_rate)              # (C,F) u8, F frames per window
            speech = inf.model._ctx().powerset_speech(cls, len(specs.classes), specs.powerset_max_classes)
        else:                                                                       # max of the sigmoid scores
            speech, _, off, _ = inf.slide_device(waveform, sample_rate, reduce_max=True)
        if hook is not None:
            hook(completed=len(off), total=len(off))                                # speech: (C,F,1) f32 on device
        chunks_sw = SlidingWindow(start=0.0, duration=inf.duration, step=inf.step)
        agg = inf.aggregate_device(SlidingWindowFeature(speech, chunks_sw), inf.model.receptive_field,
                                   warm_up=inf.warm_up, hamming=True, missing=0.0)
        num_samples = waveform.shape[1]
        _, _, _, has_last = chunk_layout(num_samples, inf.model.audio.get_num_samples(inf.duration),
                                         round(inf.step * sample_rate))
        if has_last:
            agg.data = agg.crop(Segment(0.0, num_samples / sample_rate), mode="loose")
        return agg

    def apply(self, file: AudioFile, hook: Optional[Callable] = None) -> Annotation:
        file = self._segmentation.model.audio.validate_file(file)
        user_hook = hook
        hook = (lambda *a, **k: user_hook(*a, file=file, **k)) if user_hook is not None else (lambda *a, **k: None)
        segmentations = self.speech_scores(file, hook=lambda **k: hook("segmentation", None, **k))
        hook("segmentation", segmentations)
        speech = self._binarize(segmentations)
        speech.uri = file.get("uri")
        return speech.rename_labels({label: "SPEECH" for label in speech.labels()})

    __call__ = apply
