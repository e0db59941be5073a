"""Speaker diarization pipeline (mirror of /root/reference/src/pyannote/audio/pipelines/speaker_diarization.py).

Same constructor arguments, ``apply`` signature, hook protocol and ``DiarizeOutput`` as the reference's
``SpeakerDiarization``; plus the reference's own optional extension point ``apply_batch(files)``
(core/pipeline.py:497-508) which is where multi-file batching and multi-GPU sharding plug in.

Data flow per batch of files (everything between the H2D of the waveforms and the D2H of the discrete diarization
stays on the device):
  waveforms --H2D--> [PyanNet sliding window] -> powerset classes (C,589) u8 -> multilabel (C,589,3) u8
     -> speaker count (F,) u8 -> masks (C,3,589) -> [WeSpeaker trunk once per chunk + 3 masked poolings] -> (C,3,256)
     -> [filter -> centroid linkage -> (host: dendrogram cut) -> PLDA -> VBx -> cosine cdist -> 3xK assignment]
     -> [clustered overlap-add + top-count selection] -> discrete diarization (F,K) u8 --D2H--> run-length -> Annotation
"""
from __future__ import annotations

import math
import textwrap
import os
import sys
import time
import warnings
from dataclasses import dataclass
from typing import Any, Callable, Iterator, Mapping, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import ops
from .audio import Audio, AudioFile
from .clustering import PLDA, AgglomerativeClustering, VBxClustering
from .core import Annotation, SlidingWindow, SlidingWindowFeature
from .inference import Inference, chunk_layout
from .models import BaseWeSpeakerResNet, BaseXVector, PyanNet, WeSpeakerResNet34, get_context


def set_num_speakers(num_speakers=None, min_speakers=None, max_speakers=None):
    """pipelines/utils/diarization.py:34-69."""
    min_speakers = num_speakers or min_speakers or 1
    max_speakers = num_speakers or max_speakers or np.inf
    if min_speakers > max_speakers:
        raise ValueError(f"min_speakers must be smaller than (or equal to) max_speakers "
                         f"(here: min_speakers={min_speakers:g} and max_speakers={max_speakers:g}).")
    if min_speakers == max_speakers:
        num_speakers = min_speakers
    return num_speakers, min_speakers, max_speakers


@dataclass
class DiarizeOutput:
    speaker_diarization: Annotation
    exclusive_speaker_diarization: Annotation
    speaker_embeddings: Optional[np.ndarray] = None

    def serialize(self) -> dict:
        def rows(a):
            return [{"start": round(s.start, 3), "end": round(s.end, 3), "speaker": lab}
                    for s, _, lab in a.itertracks(yield_label=True)]

        return {"diarization": rows(self.speaker_diarization),
                "exclusive_diarization": rows(self.exclusive_speaker_diarization)}


class PretrainedSpeakerEmbedding:
    """pipelines/speaker_verification.py:622-716 (PyannoteAudioPretrainedSpeakerEmbedding) over the CUDA model."""

    def __init__(self, embedding: Union[BaseWeSpeakerResNet, BaseXVector], device: Optional[torch.device] = None):
        self.embedding = embedding
        self.model_ = embedding
        self.model_.eval()
        self.device = device or self.model_.device
        if self.device.type == "cuda":
            self.model_.to(self.device)

    def to(self, device: torch.device):
        if not isinstance(device, torch.device):
            raise TypeError(f"`device` must be an instance of `torch.device`, got `{type(device).__name__}`")
        self.model_.to(device)
        self.device = device
        return self

    @property
    def sample_rate(self) -> int:
        return self.model_.audio.sample_rate

    @property
    def dimension(self) -> int:
        return self.model_.dimension

    @property
    def metric(self) -> str:
        return "cosine"

    @property
    def min_num_samples(self) -> int:
        # the shortest input the model accepts (speaker_verification.py:688-702 finds it by bisection on exceptions):
        # 400 for the WeSpeaker ResNets, 4771 for XVectorSincNet, 2800 for XVectorMFCC
        return self.model_.min_num_samples

    def __call__(self, waveforms: torch.Tensor, masks: Optional[torch.Tensor] = None) -> np.ndarray:
        return self.model_(waveforms, weights=masks).cpu().numpy()


def _sparse_true(x: np.ndarray) -> np.ndarray:
    """Flat indices of the True entries of a (mostly False) bool array: scan 8 flags per uint64 word, then only the
    few non-zero words (np.nonzero on the 2-D array costs 0.35 ms for a 10-minute file, this 0.03 ms)."""
    flat = np.ascontiguousarray(x).ravel()
    pad = (-flat.size) % 8
    if pad:
        flat = np.concatenate([flat, np.zeros(pad, dtype=bool)])
    words = np.flatnonzero(flat.view(np.uint64))
    if words.size == 0:
        return np.zeros(0, dtype=np.int64)
    sub_w, sub_b = np.nonzero(flat.reshape(-1, 8)[words])
    return words[sub_w] * 8 + sub_b


def binarize_frames(discrete: Optional[np.ndarray], frames: SlidingWindow, min_duration_off: float = 0.0,
                    uri: Optional[str] = None, events=None) -> Tuple[Annotation, np.ndarray]:
    """to_annotation (diarization.py:188-218) / Binarize(onset=offset=0.5) (utils/signal.py:254-318), vectorised.

    A region switched on at frame a and off at frame b is [middle(a), middle(b)]; a region still active at the last
    frame n-1 closes at middle(n-1).  Returns the Annotation (integer labels) and the (n_segments, 3) int array of
    (start_frame, end_frame, label), both in Annotation.itertracks() order: by (start, end), then speaker column.
    ``events`` = (n, on, off) with the sorted flat indices k * (n + 1) + f found on the device
    (ops.Context.frame_transitions) replaces the host scan of ``discrete``.
    """
    if events is not None:
        n, on, off = events
        if n < 2:
            return Annotation(uri=uri), np.zeros((0, 3), dtype=np.int64)
    else:
        n, K = discrete.shape
        if n < 2 or K == 0:
            return Annotation(uri=uri), np.zeros((0, 3), dtype=np.int64)
        act = np.zeros((K, n + 2), dtype=bool)                 # speaker-major and contiguous
        act[:, 1:-1] = discrete.T > 0
        on = _sparse_true(act[:, 1:] & ~act[:, :-1])
        off = _sparse_true(act[:, :-1] & ~act[:, 1:])
    # grouped by k, ascending t; the i-th offset closes the i-th onset
    on_k, on_t = np.divmod(on, n + 1)
    off_k, off_t = np.divmod(off, n + 1)
    off_t = np.minimum(off_t, n - 1)                           # still active at the end -> last frame
    keep = off_t > on_t         # an onset at the very last frame is an empty Segment: Annotation.__setitem__ drops it
    if not keep.all():
        on_k, on_t, off_t = on_k[keep], on_t[keep], off_t[keep]
    order = np.lexsort((on_k, off_t, on_t))                    # sort by (start, end, k)
    rows = np.stack([on_t[order], off_t[order], on_k[order]], axis=1).astype(np.int64)
    # timestamps = frames[i].middle computed like pyannote.core: start_i = start + i*step; 0.5*(start_i + (start_i+dur))
    s0 = frames.start + rows[:, 0] * frames.step
    s1 = frames.start + rows[:, 1] * frames.step
    starts = 0.5 * (s0 + (s0 + frames.duration))
    ends = 0.5 * (s1 + (s1 + frames.duration))
    ann = Annotation.from_rows(starts, ends, rows[:, 2], uri=uri)
    if min_duration_off > 0.0:
        ann = ann.support(collar=min_duration_off)
    return ann, rows


def require_10s_window(window_size: int):
    """Speaker diarization runs on 10 s segmentation windows only: the embedding masks and the speaker counting /
    reconstruction kernels are laid out for 589 frames per chunk."""
    if int(window_size) != ops.CHUNK:
        raise ValueError(f"speaker diarization needs 10 s ({ops.CHUNK}-sample) segmentation windows, got "
                         f"{int(window_size)} samples: use Inference or VoiceActivityDetection for other durations")


def require_community_head(specifications):
    """Speaker diarization runs on the community-1 head only: a powerset of 3 speakers with at most 2 per frame (the
    embedding masks, speaker counting and reconstruction kernels take 3 binary local speakers)."""
    if not specifications.powerset or (len(specifications.classes), specifications.powerset_max_classes) != (3, 2):
        raise ValueError("speaker diarization needs the community-1 segmentation head (a powerset of 3 speakers with "
                         "at most 2 per frame): use Inference, VoiceActivityDetection or MultiLabelSegmentation for "
                         "other heads")


class SpeakerDiarization:
    def __init__(self, legacy: bool = False, segmentation: Union[PyanNet, Mapping, None] = None,
                 segmentation_step: float = 0.1, embedding: Union[BaseWeSpeakerResNet, Mapping, None] = None,
                 embedding_exclude_overlap: bool = False, plda: Union[PLDA, Mapping, None] = None,
                 clustering: str = "VBxClustering", embedding_batch_size: int = 1, segmentation_batch_size: int = 1,
                 der_variant: Optional[dict] = None, token=None, cache_dir=None,
                 device: Optional[torch.device] = None):
        self.legacy = legacy
        device = device or torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.device = device
        # paths / {"checkpoint": ..., "subfolder": ...} entries as Pipeline.from_pretrained hands them over
        # (pipelines/utils/getter.py get_model / get_plda); instances and state dicts pass through untouched
        from .loading import get_model, get_plda, is_checkpoint_spec

        if is_checkpoint_spec(segmentation):
            segmentation = get_model(segmentation, token=token, cache_dir=cache_dir)
        if is_checkpoint_spec(embedding):
            embedding = get_model(embedding, token=token, cache_dir=cache_dir)
        if is_checkpoint_spec(plda):
            plda = get_plda(plda, token=token, cache_dir=cache_dir)
        if isinstance(segmentation, Mapping):
            model = PyanNet()
            model.load_state_dict(segmentation)
            segmentation = model
        if isinstance(embedding, Mapping):
            model = WeSpeakerResNet34()
            model.load_state_dict(embedding)
            embedding = model
        if not isinstance(segmentation, PyanNet) or not isinstance(embedding, BaseWeSpeakerResNet):
            raise ValueError("`segmentation` / `embedding` must be PyanNet / WeSpeaker ResNet instances or their "
                             "state dicts (no network access here: pretrained hub checkpoints cannot be fetched)")
        self.segmentation_model = segmentation
        self.segmentation_step = segmentation_step
        self.embedding = embedding
        self.embedding_batch_size = embedding_batch_size
        self.embedding_exclude_overlap = embedding_exclude_overlap
        self.klustering = clustering
        self.der_variant = der_variant or {"collar": 0.0, "skip_overlap": False}
        self._plda = PLDA(plda) if isinstance(plda, Mapping) else plda
        duration = segmentation.specifications.duration
        require_community_head(segmentation.specifications)
        require_10s_window(segmentation.audio.get_num_samples(duration))
        segmentation.to(device)
        embedding.to(device)
        self._segmentation = Inference(segmentation, duration=duration, step=self.segmentation_step * duration,
                                       skip_aggregation=True, batch_size=segmentation_batch_size)
        self._embedding = PretrainedSpeakerEmbedding(embedding, device=device)
        self._audio = Audio(sample_rate=self._embedding.sample_rate, mono="downmix")
        if clustering == "VBxClustering":
            if self._plda is None:
                raise ValueError("VBxClustering needs a PLDA model")
            self.clustering = VBxClustering(self._plda, metric=self._embedding.metric, device=device)
        elif clustering == "AgglomerativeClustering":
            self.clustering = AgglomerativeClustering(metric=self._embedding.metric, device=device)
        else:
            raise ValueError("clustering must be one of [AgglomerativeClustering, VBxClustering]")
        self._expects_num_speakers = self.clustering.expects_num_clusters
        self.min_duration_off = 0.0
        self.d2h_bytes = 0        # bytes copied device -> host by the last apply/apply_batch (bench.py reports it)
        self.instantiate(self.default_parameters())

    # ---- pyannote.pipeline-style parameter plumbing -------------------------------------------------------
    @property
    def segmentation_batch_size(self) -> int:
        return self._segmentation.batch_size

    @segmentation_batch_size.setter
    def segmentation_batch_size(self, batch_size: int):
        self._segmentation.batch_size = batch_size

    def default_parameters(self):
        if self.klustering == "VBxClustering":
            return {"segmentation": {"min_duration_off": 0.0}, "clustering": {"threshold": 0.6, "Fa": 0.07, "Fb": 0.8}}
        return {"segmentation": {"min_duration_off": 0.0},
                "clustering": {"method": "centroid", "min_cluster_size": 12, "threshold": 0.7045654963945799}}

    def instantiate(self, params: dict):
        self.min_duration_off = float(params.get("segmentation", {}).get("min_duration_off", 0.0))
        self.clustering.instantiate(params.get("clustering", {}))
        return self

    def to(self, device: torch.device):
        if not isinstance(device, torch.device):
            raise TypeError(f"`device` must be an instance of `torch.device`, got `{type(device).__name__}`")
        self._segmentation.to(device)
        self._embedding.to(device)
        self.clustering.device = device
        self.device = device
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device if isinstance(device, int) else torch.cuda.current_device()))

    def classes(self):
        speaker = 0
        while True:
            yield f"SPEAKER_{speaker:02d}"
            speaker += 1

    @staticmethod
    def setup_hook(file, hook: Optional[Callable] = None) -> Callable:
        def noop(*args, **kwargs):
            return

        return (lambda *a, **k: hook(*a, file=file, **k)) if hook is not None else noop

    # ---- stages ---------------------------------------------------------------------------------------------
    def _frames(self) -> SlidingWindow:
        return self._segmentation.model.receptive_field

    def _grid(self, num_chunks: int):
        """Global frame grid of a file: per-chunk start frames and total frame count (inference.py:532-571, 596)."""
        frames = self._frames()
        duration, step = self._segmentation.duration, self._segmentation.step
        fr = SlidingWindow(start=0.0, duration=frames.duration, step=frames.step)
        sf = fr.closest_frames(np.arange(num_chunks) * step + 0.5 * fr.duration).astype(np.int32)
        num_frames = fr.closest_frame(0.0 + duration + (num_chunks - 1) * step + 0.5 * fr.duration) + 1
        return sf, int(num_frames), fr

    def get_segmentations(self, file, hook=None) -> SlidingWindowFeature:
        if hook is not None:
            import functools

            hook = functools.partial(hook, "segmentation", None)
        return self._segmentation(file, hook=hook)

    def speaker_count(self, binarized: SlidingWindowFeature, frames: SlidingWindow,
                      warm_up: Tuple[float, float] = (0.0, 0.0)) -> SlidingWindowFeature:
        """diarization.py:150-185 on the device (warm_up must be (0, 0), as the pipeline calls it)."""
        if tuple(warm_up) != (0.0, 0.0):
            raise NotImplementedError("device speaker counting implements warm_up=(0.0, 0.0)")
        ctx = get_context(self.device)
        seg = torch.from_numpy(np.nan_to_num(binarized.data).astype(np.uint8)).to(ctx.device)
        sf, F, fr = self._grid(seg.shape[0])
        count = ctx.speaker_count(seg, sf, F).cpu().numpy()[:, None]
        return SlidingWindowFeature(count, fr)

    def _masks(self, seg: torch.Tensor) -> torch.Tensor:
        """(C,589,3) u8 -> StatsPool masks (C,3,589) u8 (speaker_diarization.py:375-423)."""
        if self.embedding_exclude_overlap:
            num_frames = seg.shape[1]
            num_samples = self._segmentation.duration * self._embedding.sample_rate
            min_num_frames = math.ceil(num_frames * self._embedding.min_num_samples / num_samples)
            clean = seg * (seg.sum(dim=2, keepdim=True) < 2).to(seg.dtype)
            use_clean = clean.sum(dim=1, keepdim=True) > min_num_frames
            seg = torch.where(use_clean, clean, seg)
        return seg.permute(0, 2, 1).contiguous()

    def get_embeddings(self, file, binary_segmentations: SlidingWindowFeature, exclude_overlap: bool = False,
                       hook: Optional[Callable] = None) -> np.ndarray:
        """(C,3,256) float32 embeddings; reference loop speaker_diarization.py:332-478."""
        self._require_10s_window()
        ctx = get_context(self.device)
        waveform, sr = self._audio(file)
        seg = torch.from_numpy(np.nan_to_num(binary_segmentations.data).astype(np.uint8)).to(ctx.device)
        off, valid, _, _ = chunk_layout(waveform.shape[1], ops.CHUNK, round(self._segmentation.step * sr))
        wav_dev = torch.zeros(int(off[-1]) + ops.CHUNK, dtype=torch.float32, device=ctx.device)
        wav_dev[: waveform.shape[1]] = waveform[0].to(ctx.device)
        prev = self.embedding_exclude_overlap
        self.embedding_exclude_overlap = exclude_overlap
        try:
            emb = self.embedding.forward_chunks(wav_dev, off, valid, self._masks(seg))
        finally:
            self.embedding_exclude_overlap = prev
        if hook is not None:
            hook("embeddings", None, total=1, completed=1)
        return emb.cpu().numpy()

    def reconstruct(self, segmentations: SlidingWindowFeature, hard_clusters: np.ndarray,
                    count: SlidingWindowFeature) -> SlidingWindowFeature:
        """speaker_diarization.py:480-528 + to_diarization (diarization.py:221-268) on the device."""
        ctx = get_context(self.device)
        seg = torch.from_numpy(np.nan_to_num(segmentations.data).astype(np.uint8)).to(ctx.device)
        sf, F, fr = self._grid(seg.shape[0])
        cnt = torch.from_numpy(np.asarray(count.data).reshape(-1).astype(np.uint8)).to(ctx.device)
        K = int(np.max(hard_clusters)) + 1
        Kout = max(K, int(cnt.max().item()), 1)
        d = ctx.reconstruct(seg, hard_clusters, sf, F, cnt, Kout)
        return SlidingWindowFeature(d.cpu().numpy().astype(np.float64), fr)

    def to_annotation(self, discrete: SlidingWindowFeature, min_duration_on: float = 0.0,
                      min_duration_off: float = 0.0) -> Annotation:
        ann, _ = binarize_frames(np.asarray(discrete.data), discrete.sliding_window, min_duration_off)
        return ann

    # ---- apply ---------------------------------------------------------------------------------------------------
    def apply(self, file: AudioFile, num_speakers: Optional[int] = None, min_speakers: Optional[int] = None,
              max_speakers: Optional[int] = None, hook: Optional[Callable] = None, **kwargs):
        if len(kwargs) > 0:
            warnings.warn(f"Ignoring unexpected keyword arguments: {', '.join(list(kwargs.keys()))}")
        for _, output in self.apply_batch([file], num_speakers=num_speakers, min_speakers=min_speakers,
                                          max_speakers=max_speakers, hook=hook):
            return output

    def __call__(self, file, **kwargs):
        if isinstance(file, (list, tuple)):
            return [out for _, out in self.apply_batch(list(file), **kwargs)]
        return self.apply(file, **kwargs)

    def apply_batch(self, files: Sequence[AudioFile], num_speakers: Optional[int] = None,
                    min_speakers: Optional[int] = None, max_speakers: Optional[int] = None,
                    hook: Optional[Callable] = None, progress=None,
                    return_artifacts: bool = False) -> Iterator[Tuple[Mapping, Any]]:
        """Batched entry point: segmentation and embedding of ALL files run as two device passes over one resident
        buffer; clustering / reconstruction then run per file."""
        resident = self.upload(files)
        yield from self.run_resident(resident, num_speakers=num_speakers, min_speakers=min_speakers,
                                     max_speakers=max_speakers, hook=hook, return_artifacts=return_artifacts)

    def _require_10s_window(self):
        inf = self._segmentation
        require_community_head(inf.model.specifications)
        require_10s_window(inf.model.audio.get_num_samples(inf.duration))

    def upload(self, files: Sequence[AudioFile]) -> dict:
        """H2D: one device buffer for all files, every chunk window addressable (zero padded tails)."""
        self._require_10s_window()
        ctx = get_context(self.device)
        files = [self._audio.validate_file(f) for f in files]
        step_size = round(self._segmentation.step * self._embedding.sample_rate)
        raws, layouts, base = [], [], 0
        for f in files:
            raw, sr, channel = self._audio.raw(f)
            T = self._audio.num_samples_out(raw, sr)
            off, valid, _, _ = chunk_layout(T, ops.CHUNK, step_size)
            layouts.append((base, off, valid, T))
            raws.append((raw, sr, channel))
            base += int(off[-1]) + ops.CHUNK
        wav_dev = torch.zeros(base, dtype=torch.float32, device=ctx.device)
        for (b0, off, valid, T), (raw, sr, channel) in zip(layouts, raws):
            if self._audio.needs_ingest(raw, sr, channel):
                # multi-channel / other sample rate / int16 PCM: raw samples cross PCIe once, downmix + polyphase
                # resampling run on the device (b200_audio_ingest; reference core/io.py:223-265 does this on the CPU)
                self._audio.ingest(ctx, raw, sr, channel, out=wav_dev[b0: b0 + T])
            else:
                wav_dev[b0: b0 + T].copy_(raw[0], non_blocking=True)
        return dict(files=files, wav=wav_dev, layouts=layouts,
                    off=np.concatenate([b0 + off for b0, off, _, _ in layouts]),
                    valid=np.concatenate([valid for _, _, valid, _ in layouts]),
                    bounds=np.cumsum([0] + [len(l[1]) for l in layouts]))

    def run_resident(self, resident: dict, num_speakers: Optional[int] = None, min_speakers: Optional[int] = None,
                     max_speakers: Optional[int] = None, hook: Optional[Callable] = None,
                     return_artifacts: bool = False) -> Iterator[Tuple[Mapping, Any]]:
        num_speakers, min_speakers, max_speakers = set_num_speakers(num_speakers, min_speakers, max_speakers)
        if self._expects_num_speakers and num_speakers is None:
            raise ValueError(f"num_speakers must be provided when using {self.klustering} clustering")
        ctx = get_context(self.device)
        self.d2h_bytes = 0
        wav_dev, all_off, all_valid, bounds = resident["wav"], resident["off"], resident["valid"], resident["bounds"]
        # ---- device passes over all files at once ------------------------------------------------------------
        self._timer = _StageTimer(ctx.device)
        self._timer.start()
        cls = self._segmentation.model.forward_chunks(wav_dev, all_off, all_valid)        # (C,589) u8
        seg = ctx.powerset_to_multilabel(cls)                                              # (C,589,3) u8
        self._timer.mark("segmentation")
        emb = self.embedding.forward_chunks(wav_dev, all_off, all_valid, self._masks(seg))  # (C,3,256) f32
        self._timer.mark("embedding")
        # ---- clustering + reconstruction, batched across files -------------------------------------------------
        outs = self._finish_files(ctx, resident["files"], seg, emb, bounds, num_speakers, min_speakers, max_speakers,
                                  hook, return_artifacts, classes=cls)
        self._timer.report()
        for file, out in zip(resident["files"], outs):
            yield file, out

    def _finish_file(self, ctx, file, seg, emb, num_speakers, min_speakers, max_speakers, hook, return_artifacts):
        if not hasattr(self, "_timer"):
            self._timer = _StageTimer(ctx.device)
        return self._finish_files(ctx, [file], seg, emb, [0, seg.shape[0]], num_speakers, min_speakers, max_speakers,
                                  hook, return_artifacts)[0]

    def _finish_files(self, ctx, files, seg, emb, bounds, num_speakers, min_speakers, max_speakers, hook,
                      return_artifacts, classes=None):
        tm = self._timer
        F = len(files)
        chunks_sw = SlidingWindow(start=0.0, duration=self._segmentation.duration, step=self._segmentation.step)
        # hooks receive real SlidingWindowFeature / ndarray artifacts (copied device -> host only when a hook was given)
        # plus the reference's progress calls hook(name, None, total=, completed=) (speaker_diarization.py:439-459,
        # inference.py:287-320); the device passes over all files have already run when they fire
        hooks = [self.setup_hook(f, hook) for f in files] if hook is not None else None
        grids, counts = [], []
        for fi in range(F):
            c0, c1 = int(bounds[fi]), int(bounds[fi + 1])
            sf, nF, fr = self._grid(c1 - c0)
            grids.append((sf, nF, fr))
            sfile = seg[c0:c1]
            counts.append(ctx.speaker_count(sfile, sf, nF))
            if hooks is not None:
                hooks[fi]("segmentation", None, total=c1 - c0, completed=0)
                hooks[fi]("segmentation", None, total=c1 - c0, completed=c1 - c0)
                hooks[fi]("segmentation", SlidingWindowFeature(sfile.cpu().numpy().astype(np.float32), chunks_sw))
                hooks[fi]("speaker_counting", SlidingWindowFeature(counts[-1].cpu().numpy()[:, None], fr))
        count_max = torch.stack([c.max() for c in counts]).cpu().numpy().astype(np.int64)        # sync
        tm.mark("speaker_count")
        silent = [int(m) == 0 for m in count_max]
        if hooks is not None:
            for fi in range(F):
                if not silent[fi]:
                    hooks[fi]("embeddings", None, total=1, completed=0)
                    hooks[fi]("embeddings", None, total=1, completed=1)
                    hooks[fi]("embeddings", emb[int(bounds[fi]): int(bounds[fi + 1])].cpu().numpy())
        if isinstance(self.clustering, VBxClustering):
            results = self.clustering.cluster_batch(emb, seg, bounds, num_clusters=num_speakers,
                                                    min_clusters=min_speakers, max_clusters=max_speakers, skip=silent)
        else:
            results = []
            for fi in range(F):
                if silent[fi]:
                    results.append(None)
                    continue
                c0, c1 = int(bounds[fi]), int(bounds[fi + 1])
                h, s_, c = self.clustering(embeddings=emb[c0:c1], segmentations=seg[c0:c1], num_clusters=num_speakers,
                                           min_clusters=min_speakers, max_clusters=max_speakers)
                results.append(dict(hard=torch.from_numpy(h.astype(np.int8)).to(ctx.device),
                                    centroids=torch.from_numpy(c).to(ctx.device),
                                    active=seg[c0:c1].sum(dim=1) > 0))
        tm.mark("clustering")
        pending = []
        for fi in range(F):
            if silent[fi]:
                pending.append(None)
                continue
            c0, c1 = int(bounds[fi]), int(bounds[fi + 1])
            sf, nF, fr = grids[fi]
            r = results[fi]
            count = counts[fi]
            if np.isfinite(max_speakers):
                count = torch.clamp(count, max=int(max_speakers))
            hard = torch.where(r["active"], r["hard"], torch.full_like(r["hard"], -2))     # inactive -> -2
            K = int(r["centroids"].shape[0])
            Kout = max(K, 3)        # columns beyond max(K, max count) stay all-zero and are trimmed on the host
            discrete = ctx.reconstruct(seg[c0:c1], hard, sf, nF, count, Kout)
            exclusive = ctx.reconstruct(seg[c0:c1], hard, sf, nF, torch.clamp(count, max=1), Kout)
            pending.append((discrete, exclusive, hard, r["centroids"], K))
        tm.mark("reconstruct")
        outs = []
        d2h_s = 0.0
        _prof = None
        if os.environ.get("B200_TIMING") == "3":           # host-side diagnostics of the annotation loop
            import cProfile
            _prof = cProfile.Profile()
            _prof.enable()
        # run-length encoding: onsets / offsets are found on the device and only those events cross PCIe, in ONE
        # device -> host copy for all files (plus one for the centroids); the full (frames, clusters) matrices are
        # materialised on the host only for hooks / artifacts that look at them
        _t0 = time.perf_counter()
        live = [fi for fi in range(F) if not silent[fi]]
        events = ctx.frame_transitions_many([m for fi in live for m in pending[fi][:2]])
        self.d2h_bytes += ctx.last_transfer_bytes
        cents_host = {}
        if live:
            allc = torch.cat([pending[fi][3].reshape(-1, pending[fi][3].shape[-1]) for fi in live]).cpu().numpy()
            self.d2h_bytes += allc.nbytes + 8 * len(live)
            pos = 0
            for fi in live:
                k = int(pending[fi][3].shape[0])
                cents_host[fi] = allc[pos: pos + k]
                pos += k
        events = {fi: (events[2 * i], events[2 * i + 1]) for i, fi in enumerate(live)}
        d2h_s += time.perf_counter() - _t0
        for fi, file in enumerate(files):
            uri = file.get("uri", None)
            artifacts = None
            if return_artifacts:
                c0, c1 = int(bounds[fi]), int(bounds[fi + 1])
                artifacts = dict(segmentations=seg[c0:c1], count=counts[fi], embeddings=emb[c0:c1])
                if classes is not None:
                    artifacts["classes"] = classes[c0:c1]          # powerset class ids (C,589) u8
            if silent[fi]:
                output = DiarizeOutput(Annotation(uri=uri), Annotation(uri=uri),
                                       np.zeros((0, self._embedding.dimension)))
                output = output.speaker_diarization if self.legacy else output
                outs.append((output, artifacts) if return_artifacts else output)
                continue
            discrete, exclusive, hard, centroids, K = pending[fi]
            _, nF, fr = grids[fi]
            ev_d, ev_x = events[fi]
            centroids = cents_host[fi]
            cmax = int(count_max[fi]) if not np.isfinite(max_speakers) else min(int(count_max[fi]), int(max_speakers))
            kd, kx = max(K, cmax), max(K, min(cmax, 1))
            if K < min_speakers or K > max_speakers:
                warnings.warn(textwrap.dedent(f"""
                    The detected number of speakers ({K}) for {uri} is outside
                    the given bounds [{min_speakers}, {max_speakers}]. This can happen if the
                    given audio file is too short to contain {min_speakers} or more speakers.
                    Try to lower the desired minimal number of speakers.
                    """))
            if hooks is not None:
                hooks[fi]("discrete_diarization",
                          SlidingWindowFeature(discrete.cpu().numpy()[:, :kd].astype(np.float64), fr))
            diarization, rows = binarize_frames(None, fr, self.min_duration_off, uri=uri, events=(nF,) + ev_d)
            exclusive_diarization, xrows = binarize_frames(None, fr, self.min_duration_off, uri=uri,
                                                           events=(nF,) + ev_x)
            labels_int = diarization.labels()
            mapping = {label: expected for label, expected in zip(labels_int, self.classes())}
            diarization = diarization.rename_labels(mapping)
            exclusive_diarization = exclusive_diarization.rename_labels(mapping)
            if len(labels_int) > centroids.shape[0]:
                centroids = np.pad(centroids, ((0, len(labels_int) - centroids.shape[0]), (0, 0)))
            inverse = {label: index for index, label in mapping.items()}
            centroids = centroids[[inverse[l] for l in diarization.labels()]] if len(labels_int) else centroids[:0]
            output = DiarizeOutput(diarization, exclusive_diarization, centroids)
            if return_artifacts:
                artifacts.update(hard_clusters=hard.cpu().numpy(), discrete=discrete.cpu().numpy()[:, :kd],
                                 exclusive=exclusive.cpu().numpy()[:, :kx], segments=rows, exclusive_segments=xrows,
                                 centroids=centroids)
                outs.append(((output.speaker_diarization if self.legacy else output), artifacts))
            else:
                outs.append(output.speaker_diarization if self.legacy else output)
        if _prof is not None:
            import pstats
            _prof.disable()
            pstats.Stats(_prof, stream=sys.stderr).sort_stats("tottime").print_stats(12)
        tm.mark("d2h+annotation")
        if os.environ.get("B200_TIMING") == "2":
            print(f"[b200 annotation] d2h={d2h_s * 1e3:.1f}ms of the d2h+annotation stage", file=sys.stderr)
        return outs


class _StageTimer:
    """Opt-in (B200_TIMING=1) wall-clock breakdown of the per-file stages, with a device sync at every mark."""

    def __init__(self, device):
        import os

        self.on = bool(os.environ.get("B200_TIMING"))
        self.device, self.acc, self.t = device, {}, None

    def start(self):
        if self.on:
            torch.cuda.synchronize(self.device)
            import time

            self.t = time.perf_counter()

    def mark(self, name):
        if self.on:
            import time

            torch.cuda.synchronize(self.device)
            now = time.perf_counter()
            self.acc[name] = self.acc.get(name, 0.0) + (now - self.t)
            self.t = now

    def report(self):
        if self.on and self.acc:
            import sys

            tot = sum(self.acc.values())
            print("[b200 timing] " + ", ".join(f"{k}={v * 1e3:.1f}ms" for k, v in self.acc.items())
                  + f", total={tot * 1e3:.1f}ms", file=sys.stderr, flush=True)
