"""Sliding-window inference (mirror of /root/reference/src/pyannote/audio/core/inference.py).

Same constructor, attributes, exceptions and static helpers (``aggregate`` / ``trim``) as the reference's
``Inference``; what changes is underneath ``slide``: the waveform is copied to the device ONCE, all chunks are
addressed in place (no unfold copy, no per-batch H2D/D2H), PyanNet + its head (powerset argmax, or sigmoid scores)
run in libb200diar.so, and the result comes back in one D2H copy per file.
"""
from __future__ import annotations

import warnings
from typing import Callable, List, Optional, Text, Tuple, Union

import numpy as np
import torch

from . import ops
from .audio import AudioFile
from .core import Resolution, Segment, SlidingWindow, SlidingWindowFeature, Specifications
from .models import Model


class BaseInference:
    pass


def chunk_layout(num_samples: int, window_size: int, step_size: int):
    """Chunk offsets / valid lengths exactly as Inference.slide cuts them (inference.py:261-278)."""
    if num_samples >= window_size:
        num_chunks = (num_samples - window_size) // step_size + 1
    else:
        num_chunks = 0
    has_last_chunk = (num_samples < window_size) or (num_samples - window_size) % step_size > 0
    total = num_chunks + int(has_last_chunk)
    off = np.arange(total, dtype=np.int64) * step_size
    valid = np.minimum(window_size, num_samples - off).astype(np.int32)
    return off, valid, num_chunks, has_last_chunk


def _host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


class Inference(BaseInference):
    def __init__(self, model: Model, window: Text = "sliding", duration: Optional[float] = None,
                 step: Optional[float] = None, pre_aggregation_hook: Callable[[np.ndarray], np.ndarray] = None,
                 skip_aggregation: bool = False, skip_conversion: bool = False,
                 device: Optional[torch.device] = None, batch_size: int = 32):
        self.model = model
        if device is None:
            device = self.model.device
        self.device = device
        self.model.eval()
        self.model.to(self.device)
        specifications: Specifications = self.model.specifications

        if window not in ["sliding", "whole"]:
            raise ValueError('`window` must be "sliding" or "whole".')
        if window == "whole" and any(s.resolution == Resolution.FRAME for s in specifications):
            warnings.warn('Using "whole" `window` inference with a frame-based model might lead to bad results '
                          'and huge memory consumption: it is recommended to set `window` to "sliding".')
        self.window = window

        training_duration = next(iter(specifications)).duration
        duration = duration or training_duration
        if training_duration != duration:
            warnings.warn(f"Model was trained with {training_duration:g}s chunks, and you requested "
                          f"{duration:g}s chunks for inference: this might lead to suboptimal results.")
        self.duration = duration

        self.skip_conversion = skip_conversion
        # the powerset -> multilabel conversion (utils/powerset.py) is fused into the CUDA path
        self.conversion = "powerset" if (specifications.powerset and not skip_conversion) else "identity"

        self.skip_aggregation = skip_aggregation
        self.pre_aggregation_hook = pre_aggregation_hook
        self.warm_up = next(iter(specifications)).warm_up
        step = step or (0.1 * self.duration if self.warm_up[0] == 0.0 else self.warm_up[0])
        if step > self.duration:
            raise ValueError(f"Step between consecutive chunks is set to {step:g}s, while chunks are "
                             f"only {self.duration:g}s long, leading to gaps between consecutive chunks. "
                             f"Either decrease step or increase duration.")
        self.step = step
        self.batch_size = batch_size

    def to(self, device: torch.device) -> "Inference":
        if not isinstance(device, torch.device):
            raise TypeError(f"`device` must be an instance of `torch.device`, got `{type(device).__name__}`")
        self.model.to(device)
        self.device = device
        return self

    # ---- forward ------------------------------------------------------------------------------------
    def infer(self, chunks: torch.Tensor) -> np.ndarray:
        """(batch, channel, sample) chunks -> (batch, frames, speakers) multilabel {0,1} of a powerset model, else the
        model's output: (batch, frames, K) log-probabilities or sigmoid scores."""
        try:
            logp = self.model(chunks)
        except MemoryError:
            raise MemoryError(f"batch_size ({self.batch_size: d}) is probably too large. "
                              f"Try with a smaller value until memory error disappears.")
        if self.conversion == "identity":
            return logp.cpu().numpy()
        cls = torch.argmax(logp, dim=-1).to(torch.uint8).contiguous()
        return self._to_multilabel(cls).cpu().numpy().astype(np.float32)

    def _to_multilabel(self, cls: torch.Tensor) -> torch.Tensor:
        specs = self.model.specifications
        return self.model._ctx().powerset_to_multilabel(cls, len(specs.classes), specs.powerset_max_classes)

    def slide_device(self, waveform: torch.Tensor, sample_rate: int, return_logp: bool = False,
                     reduce_max: bool = False):
        """Device-resident result of the sliding window: (output, wav_dev, off, valid), F frames per window of
        ``duration``.  The output of a log-softmax head is classes (C,F) u8, or with ``return_logp`` the pair
        (classes, log-probabilities (C,F,K) f32); that of a sigmoid head is its scores (C,F,K) f32, or with
        ``reduce_max`` their per-frame maximum (C,F,1)."""
        window_size = self.model.audio.get_num_samples(self.duration)
        step_size = round(self.step * sample_rate)
        self.model.check_window(window_size)
        _, num_samples = waveform.shape
        off, valid, num_chunks, has_last = chunk_layout(num_samples, window_size, step_size)
        ctx = self.model._ctx()
        # one H2D copy per file; every chunk window must be addressable -> allocate up to the last chunk's end
        total = int(off[-1]) + window_size
        wav_dev = torch.zeros(total, dtype=torch.float32, device=ctx.device)
        src = waveform[0]
        if src.device.type == "cpu" and not src.is_pinned() and src.numel() > (1 << 22):
            src = src.contiguous()
        wav_dev[:num_samples].copy_(src, non_blocking=True)
        try:
            cls = self.model.forward_chunks(wav_dev, off, valid, return_logp=return_logp, window=window_size,
                                            reduce_max=reduce_max)
        except MemoryError:
            raise MemoryError(f"batch_size ({self.batch_size: d}) is probably too large. "
                              f"Try with a smaller value until memory error disappears.")
        return cls, wav_dev, off, valid

    def slide(self, waveform: torch.Tensor, sample_rate: int, hook: Optional[Callable] = None):
        if self.model.specifications.resolution == Resolution.CHUNK:      # embedding models
            return self._slide_embedding(waveform, sample_rate, hook=hook)
        specs = self.model.specifications
        sigmoid = ops.seg_activation(specs) == ops.SEG_SIGMOID
        out, _, off, _ = self.slide_device(waveform, sample_rate,
                                           return_logp=not sigmoid and self.conversion != "powerset")
        total = len(off)
        if hook is not None:
            hook(completed=0, total=total)
        if self.conversion == "powerset":
            outputs = self._to_multilabel(out).cpu().numpy().astype(np.float32)
        elif sigmoid:                           # multi-label / binary scores: aggregated on the device as they are
            outputs = out
        else:                                   # skip_conversion=True: raw log-probabilities (:130-141)
            outputs = out[1].cpu().numpy()
        if hook is not None:
            hook(completed=total, total=total)
        frames = self.model.receptive_field
        chunks_sw = SlidingWindow(start=0.0, duration=self.duration, step=self.step)
        if self.skip_aggregation or specs.resolution == Resolution.CHUNK or \
                (specs.permutation_invariant and self.pre_aggregation_hook is None):
            return SlidingWindowFeature(_host(outputs), chunks_sw)
        if self.pre_aggregation_hook is not None:
            outputs = np.asarray(self.pre_aggregation_hook(_host(outputs)))
        aggregated = self.aggregate_device(SlidingWindowFeature(outputs, chunks_sw), frames,
                                           warm_up=self.warm_up, hamming=True, missing=0.0)
        _, num_samples = waveform.shape
        _, _, _, has_last = chunk_layout(num_samples, self.model.audio.get_num_samples(self.duration),
                                         round(self.step * sample_rate))
        if has_last:
            aggregated.data = aggregated.crop(Segment(0.0, num_samples / sample_rate), mode="loose")
        return aggregated

    def _slide_embedding(self, waveform: torch.Tensor, sample_rate: int, hook: Optional[Callable] = None):
        """One embedding per window (inference.py:261-313 for a Resolution.CHUNK model): the chunks are cut as the
        reference cuts them, the last one zero-padded to the full window, and all of them (they have one length) go
        through one library call over a resident copy of the file -> SlidingWindowFeature (chunks, dimension)."""
        window_size = self.model.audio.get_num_samples(self.duration)
        step_size = round(self.step * sample_rate)
        _, num_samples = waveform.shape
        off, _, _, _ = chunk_layout(num_samples, window_size, step_size)
        total = len(off)
        if hook is not None:
            hook(completed=0, total=total)
        ctx = self.model._ctx()
        wav_dev = torch.zeros(int(off[-1]) + window_size, dtype=torch.float32, device=ctx.device)
        wav_dev[:num_samples].copy_(waveform[0])
        try:
            emb = self.model.forward_utterances(wav_dev, off, window_size)
        except MemoryError:
            raise MemoryError(f"batch_size ({self.batch_size: d}) is probably too large. "
                              f"Try with a smaller value until memory error disappears.")
        outputs = emb[:, 0].cpu().numpy()
        if hook is not None:
            hook(completed=total, total=total)
        return SlidingWindowFeature(outputs, SlidingWindow(start=0.0, duration=self.duration, step=self.step))

    def __call__(self, file: AudioFile, hook: Optional[Callable] = None):
        waveform, sample_rate = self.model.audio(file)
        if self.window == "sliding":
            return self.slide(waveform, sample_rate, hook=hook)
        out = self.infer(waveform[None])
        return out[0]

    def crop(self, file: AudioFile, chunk: Union[Segment, List[Segment]], hook: Optional[Callable] = None):
        if self.window == "sliding":
            if not isinstance(chunk, Segment):
                start = min(c.start for c in chunk)
                end = max(c.end for c in chunk)
                chunk = Segment(start=start, end=end)
            waveform, sample_rate = self.model.audio.crop(file, chunk)
            outputs = self.slide(waveform, sample_rate, hook=hook)
            shifted = SlidingWindow(start=chunk.start, duration=outputs.sliding_window.duration,
                                    step=outputs.sliding_window.step)
            return SlidingWindowFeature(outputs.data, shifted)
        if isinstance(chunk, Segment):
            waveform, sample_rate = self.model.audio.crop(file, chunk)
        else:
            waveform = torch.cat([self.model.audio.crop(file, c)[0] for c in chunk], dim=1)
        return self.infer(waveform[None])[0]

    def aggregate_device(self, scores: SlidingWindowFeature, frames: SlidingWindow,
                         warm_up: Tuple[float, float] = (0.0, 0.0), epsilon: float = 1e-12, hamming: bool = False,
                         missing: float = np.nan, skip_average: bool = False) -> SlidingWindowFeature:
        """Inference.aggregate on the device (b200_aggregate): same arguments, bit-identical result.  ``scores.data``
        may be a host array or a device tensor of shape (chunks, frames, classes)."""
        ctx = self.model._ctx()
        data = scores.data
        if not isinstance(data, torch.Tensor):
            data = torch.from_numpy(np.ascontiguousarray(data, dtype=np.float32))
        data = data.to(device=ctx.device, dtype=torch.float32)
        chunks = scores.sliding_window
        num_chunks, nfpc, _ = data.shape
        fr = SlidingWindow(start=chunks.start, duration=frames.duration, step=frames.step)
        sf = fr.closest_frames(chunks.start + np.arange(num_chunks) * chunks.step + 0.5 * fr.duration).astype(np.int32)
        num_frames = fr.closest_frame(
            chunks.start + chunks.duration + (num_chunks - 1) * chunks.step + 0.5 * fr.duration) + 1
        out = ctx.aggregate(data, sf, num_frames, hamming=hamming, warm_up=warm_up, chunk_duration=chunks.duration,
                            epsilon=epsilon, missing=missing, skip_average=skip_average)
        return SlidingWindowFeature(out.cpu().numpy(), fr)

    # ---- static helpers, called by name from the diarization mixin (diarization.py:175-176, 241) ---------
    @staticmethod
    def aggregate(scores: SlidingWindowFeature, frames: SlidingWindow, warm_up: Tuple[float, float] = (0.0, 0.0),
                  epsilon: float = 1e-12, hamming: bool = False, missing: float = np.nan,
                  skip_average: bool = False) -> SlidingWindowFeature:
        """Generic float overlap-add (inference.py:498-620).  The pipeline's integer special cases
        (speaker counting, clustered reconstruction) run on the device instead (ops.speaker_count /
        ops.reconstruct); this host version serves the aggregated (non skip_aggregation) API."""
        num_chunks, nfpc, num_classes = scores.data.shape
        chunks = scores.sliding_window
        frames = SlidingWindow(start=chunks.start, duration=frames.duration, step=frames.step)
        hamming_window = np.hamming(nfpc).reshape(-1, 1) if hamming else np.ones((nfpc, 1))
        warm_up_window = np.ones((nfpc, 1))
        warm_up_left = round(warm_up[0] / chunks.duration * nfpc)
        warm_up_window[:warm_up_left] = epsilon
        warm_up_right = round(warm_up[1] / chunks.duration * nfpc)
        warm_up_window[nfpc - warm_up_right:] = epsilon
        num_frames = frames.closest_frame(
            chunks.start + chunks.duration + (num_chunks - 1) * chunks.step + 0.5 * frames.duration) + 1
        agg = np.zeros((num_frames, num_classes), dtype=np.float32)
        cnt = np.zeros((num_frames, num_classes), dtype=np.float32)
        msk = np.zeros((num_frames, num_classes), dtype=np.float32)
        for c in range(num_chunks):
            score = scores.data[c]
            mask = 1 - np.isnan(score)
            score = np.nan_to_num(score, copy=True, nan=0.0)
            sf = frames.closest_frame(chunks.start + c * chunks.step + 0.5 * frames.duration)
            agg[sf:sf + nfpc] += score * mask * hamming_window * warm_up_window       # the reference's operand order
            cnt[sf:sf + nfpc] += mask * hamming_window * warm_up_window
            msk[sf:sf + nfpc] = np.maximum(msk[sf:sf + nfpc], mask)
        average = agg if skip_average else agg / np.maximum(cnt, epsilon)
        average[msk == 0.0] = missing
        return SlidingWindowFeature(average, frames)

    @staticmethod
    def trim(scores: SlidingWindowFeature, warm_up: Tuple[float, float] = (0.1, 0.1)) -> SlidingWindowFeature:
        assert scores.data.ndim == 3, \
            "Inference.trim expects (num_chunks, num_frames, num_classes)-shaped `scores`"
        _, num_frames, _ = scores.data.shape
        chunks = scores.sliding_window
        left = round(num_frames * warm_up[0])
        right = round(num_frames * warm_up[1])
        num_frames_step = round(num_frames * chunks.step / chunks.duration)
        if num_frames - left - right < num_frames_step:
            warnings.warn(f"Total `warm_up` is so large ({sum(warm_up) * 100:g}% of each chunk) "
                          f"that resulting trimmed scores does not cover a whole step ({chunks.step:g}s)")
        new_data = scores.data[:, left: num_frames - right]
        new_chunks = SlidingWindow(start=chunks.start + warm_up[0] * chunks.duration, step=chunks.step,
                                   duration=(1 - warm_up[0] - warm_up[1]) * chunks.duration)
        return SlidingWindowFeature(new_data, new_chunks)
