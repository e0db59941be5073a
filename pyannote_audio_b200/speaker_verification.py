"""Speaker embedding pipeline (mirror of /root/reference/src/pyannote/audio/pipelines/speaker_verification.py:781-856):
one embedding per file, which is assumed to hold a single speaker, optionally pooled with voice activity weights."""
from __future__ import annotations

from typing import Mapping, Optional, Union

import numpy as np
import torch

from .audio import AudioFile
from .models import BaseWeSpeakerResNet, BaseXVector, PyanNet, WeSpeakerResNet34


class SpeakerEmbedding:
    """``apply(file)`` -> (1, dimension) ndarray.  Without ``segmentation`` the statistics pooling runs over the whole
    file; with it, frames are weighted by the cubed aggregated speech score of the voice activity detection
    (max over the speakers of the segmentation model), interpolated onto the model's frames."""

    def __init__(self, embedding: Union[BaseWeSpeakerResNet, BaseXVector, Mapping, str, None] = None,
                 segmentation: Union[PyanNet, Mapping, str, None] = None, token=None, cache_dir=None,
                 device: Optional[torch.device] = None):
        from .loading import get_model, is_checkpoint_spec

        if is_checkpoint_spec(embedding):                  # path / {"checkpoint": ...} from Pipeline.from_pretrained
            embedding = get_model(embedding, token=token, cache_dir=cache_dir)
        if isinstance(embedding, Mapping):
            model = WeSpeakerResNet34()
            model.load_state_dict(embedding)
            embedding = model
        if not isinstance(embedding, (BaseWeSpeakerResNet, BaseXVector)):
            raise ValueError("`embedding` must be a WeSpeaker ResNet, XVectorSincNet or XVectorMFCC instance, a ResNet34 "
                             "state dict or a local checkpoint (no hub access here)")
        device = device or torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.embedding = embedding
        self.segmentation = segmentation
        self.embedding_model_ = embedding.to(device).eval()
        self._vad = None
        if segmentation is not None:
            from .vad import VoiceActivityDetection

            # the reference's Inference(segmentation, pre_aggregation_hook=max over speakers)
            self._vad = VoiceActivityDetection(segmentation=segmentation, token=token, cache_dir=cache_dir,
                                               device=device)

    def instantiate(self, params: dict):
        return self

    def speech_weights(self, file: AudioFile) -> np.ndarray:
        """(num_frames,) float32 pooling weights: aggregated speech scores, NaN set to 0, cubed."""
        weights = np.array(self._vad.speech_scores(file).data[:, 0], dtype=np.float32)
        weights[np.isnan(weights)] = 0.0
        return weights ** 3

    def apply(self, file: AudioFile) -> np.ndarray:
        model = self.embedding_model_
        waveform, _ = model.audio(file)
        if self._vad is None:
            with torch.inference_mode():
                return model(waveform[None]).cpu().numpy()
        weights = torch.from_numpy(self.speech_weights(file))[None].to(model.device)
        wav = waveform[0].to(device=model.device, dtype=torch.float32).contiguous()
        if wav.numel() < model.min_num_samples:
            raise ValueError(f"{type(model).__name__} needs at least {model.min_num_samples} samples, got "
                             f"{wav.numel()}")
        # soft weights: the model's utterance entry (WeSpeaker's forward keeps the binary-mask contract)
        return model.forward_utterances(wav, np.zeros(1, dtype=np.int64), wav.numel(),
                                        weights=weights)[:, 0].cpu().numpy()

    __call__ = apply
