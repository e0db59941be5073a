"""Speaker embedding pipeline (mirror of /root/reference/src/pyannote/audio/pipelines/speaker_verification.py:781-856):
one embedding per file, which is assumed to hold a single speaker, optionally pooled with voice activity weights."""
from __future__ import annotations

from typing import Mapping, Optional, Union

import numpy as np
import torch

from .audio import AudioFile
from .models import BaseWeSpeakerResNet, PyanNet, WeSpeakerResNet34


class SpeakerEmbedding:
    """``apply(file)`` -> (1, 256) ndarray.  Without ``segmentation`` the statistics pooling runs over the whole file;
    with it, frames are weighted by the cubed aggregated speech score of the voice activity detection
    (max over the speakers of the segmentation model), interpolated onto the trunk frames."""

    def __init__(self, embedding: Union[BaseWeSpeakerResNet, Mapping, str, None] = None,
                 segmentation: Union[PyanNet, Mapping, str, None] = None, token=None, cache_dir=None,
                 device: Optional[torch.device] = None):
        from .loading import get_model, is_checkpoint_spec

        if is_checkpoint_spec(embedding):                  # path / {"checkpoint": ...} from Pipeline.from_pretrained
            embedding = get_model(embedding, token=token, cache_dir=cache_dir)
        if isinstance(embedding, Mapping):
            model = WeSpeakerResNet34()
            model.load_state_dict(embedding)
            embedding = model
        if not isinstance(embedding, BaseWeSpeakerResNet):
            raise ValueError("`embedding` must be a WeSpeaker ResNet instance, a ResNet34 state dict or a local checkpoint "
                             "(no hub access here)")
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
        ctx = model._ctx()
        wav = waveform[0].to(device=ctx.device, dtype=torch.float32).contiguous()
        if wav.numel() < 400:
            raise ValueError(f"WeSpeaker needs at least 400 samples (one 25 ms fbank frame), got {wav.numel()}")
        # soft weights: straight to the library (forward itself keeps the binary-mask contract)
        return ctx.emb_forward_utt(wav, np.zeros(1, dtype=np.int64), wav.numel(), weights=weights)[:, 0].cpu().numpy()

    __call__ = apply
