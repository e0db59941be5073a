"""Model-level seam: ``PyanNet``, the WeSpeaker ResNets (``WeSpeakerResNet34`` and the bottleneck
``WeSpeakerResNet152`` / ``221`` / ``293``), ``XVectorSincNet`` and ``XVectorMFCC`` with the reference's state-dict keys and
``forward`` contract, computing through libb200diar.so (no torch ops on the forward path, no CPU fallback).

Reference interfaces mirrored (paths relative to /root/reference/src/pyannote/audio):
  core/model.py:69-183 (Model: specifications, audio, receptive_field, device)
  models/segmentation/PyanNet.py:92-240 (ctor hyper-parameters, num_frames, receptive field, forward)
  models/embedding/wespeaker/__init__.py:41-466 (forward / forward_frames / forward_embedding / dimension)
  models/embedding/xvector.py:42-349 (XVectorMFCC, XVectorSincNet)
  models/segmentation/SSeRiouSS.py (SSeRiouSS on WavLM Base; module tree of torchaudio's wavlm_model)
"""
from __future__ import annotations

import itertools
import math
from functools import cached_property
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .audio import Audio
from .core import Problem, Resolution, SlidingWindow, Specifications

_CONTEXTS: Dict[int, "ops.Context"] = {}
_MODEL_IDS = itertools.count(1)


def get_context(device) -> "ops.Context":
    """One library context per CUDA device, shared by all models placed on it."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(
            f"pyannote_audio_b200 models only run on CUDA (H100 / sm_90a) devices, not on '{device}': move the "
            f"model with .to(torch.device('cuda'))")
    index = device.index if device.index is not None else torch.cuda.current_device()
    if index not in _CONTEXTS:
        _CONTEXTS[index] = ops.Context(torch.device("cuda", index))
    return _CONTEXTS[index]


def _conv1d_num_frames(n, k, s, p=0, d=1):
    return 1 + (n + 2 * p - d * (k - 1) - 1) // s


class Model(nn.Module):
    """Subset of pyannote.audio.core.model.Model that inference relies on."""

    def __init__(self, sample_rate: int = 16000, num_channels: int = 1):
        super().__init__()
        self.hparams = type("HParams", (), {})()
        self.hparams.sample_rate = sample_rate
        self.hparams.num_channels = num_channels
        self.audio = Audio(sample_rate=sample_rate, mono="downmix")
        self.register_buffer("_dummy", torch.zeros(0), persistent=False)      # device tracker, not in state_dict
        # The library context of a device holds ONE set of segmentation and ONE set of embedding weights.  Each model
        # stamps the slot it uploads into with (its unique id, its weight version); a forward re-uploads whenever the
        # slot carries another stamp, so several models on one GPU and load_state_dict() after a forward stay correct.
        self._model_id = next(_MODEL_IDS)
        self._weights_version = 0
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._bump_weights())

    _SLOT = ""          # "seg" | "emb" | "xvec" | "xvec_mfcc" | "ssl": the context slot this model family uploads into

    def _bump_weights(self):
        self._weights_version += 1

    @property
    def device(self) -> torch.device:
        return self._dummy.device

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        self._bump_weights()              # weights may have moved / changed dtype: re-upload lazily
        return out

    def _ctx(self) -> "ops.Context":
        ctx = get_context(self.device)
        stamp = (self._model_id, self._weights_version)
        if ctx.owners.get(self._SLOT) != stamp:
            self._upload(ctx)
            ctx.owners[self._SLOT] = stamp
        return ctx

    def _upload(self, ctx):
        raise NotImplementedError

    # ---- checkpoints (core/model.py:497-655 without lightning / the HF hub) -----------------------------------
    @classmethod
    def from_pretrained(cls, checkpoint, map_location=None, strict: bool = True, subfolder: Optional[str] = None,
                        revision: Optional[str] = None, token=None, cache_dir=None, **kwargs) -> "Model":
        """Load a pyannote.audio (Lightning-format) checkpoint: a local ``pytorch_model.bin``, a directory holding
        one (optionally under ``subfolder``), or an ``io.BytesIO``.  The file is read with plain ``torch.load``;
        the pickled ``pyannote.audio.core.task`` objects (Specifications / Problem / Resolution) are mapped onto this
        package's mirrors, so neither lightning nor pyannote.audio needs to be importable.  The checkpoint names its
        own architecture (``checkpoint["pyannote.audio"]["architecture"]``); ``kwargs`` override saved
        hyper-parameters like the reference.  Hub identifiers cannot be resolved offline and raise."""
        import io
        import os
        from pathlib import Path

        if isinstance(checkpoint, io.BytesIO) or os.path.isfile(checkpoint):
            if revision is not None:
                raise ValueError("Revisions cannot be used with local checkpoints.")
            path = checkpoint
        elif os.path.isdir(checkpoint):
            if revision is not None:
                raise ValueError("Revisions cannot be used with local checkpoints.")
            path = Path(checkpoint) / subfolder / "pytorch_model.bin" if subfolder else \
                Path(checkpoint) / "pytorch_model.bin"
        else:
            if "@" in str(checkpoint):
                raise ValueError("Revisions must be passed with `revision` keyword argument.")
            raise ValueError(f"'{checkpoint}' is not a local checkpoint; Hugging Face hub identifiers cannot be "
                             f"downloaded here (no network): pass the path of a downloaded pytorch_model.bin")
        if map_location is None:
            map_location = "cpu"
        loaded = torch.load(path, map_location=map_location, weights_only=False, pickle_module=_checkpoint_pickle)
        meta = loaded["pyannote.audio"]
        class_name = meta["architecture"]["class"]
        klass = {"PyanNet": PyanNet, "WeSpeakerResNet34": WeSpeakerResNet34, "WeSpeakerResNet152": WeSpeakerResNet152,
                 "WeSpeakerResNet221": WeSpeakerResNet221, "WeSpeakerResNet293": WeSpeakerResNet293,
                 "XVectorSincNet": XVectorSincNet, "XVectorMFCC": XVectorMFCC, "SSeRiouSS": SSeRiouSS}.get(class_name)
        if klass is None:
            raise NotImplementedError(f"architecture {meta['architecture']['module']}.{class_name} has no CUDA "
                                      f"implementation (PyanNet, SSeRiouSS, WeSpeakerResNet34 / 152 / 221 / 293, "
                                      f"XVectorSincNet and XVectorMFCC have one)")
        if cls not in (Model, klass) and not issubclass(klass, cls):
            raise ValueError(f"checkpoint holds a {class_name}, not a {cls.__name__}")
        hparams = dict(loaded.get("hyper_parameters", {}))
        hparams.update(kwargs)
        hparams = {k: v for k, v in hparams.items() if k in klass._HPARAMS}
        model = klass(**hparams)
        specs = meta.get("specifications", None)
        if specs is not None:
            if isinstance(specs, (tuple, list)):
                raise NotImplementedError("multi-task checkpoints are not supported")
            model.specifications = specs
        sd = loaded["state_dict"]
        own = set(model.state_dict().keys())
        if not strict:
            sd = {k: v for k, v in sd.items() if k in own}
        model.load_state_dict(sd, strict=strict)
        model.eval()
        return model

    @cached_property
    def receptive_field(self) -> SlidingWindow:
        size = self.receptive_field_size(num_frames=1)
        step = self.receptive_field_size(num_frames=2) - size
        start = self.receptive_field_center(frame=0) - (size - 1) / 2
        sr = self.hparams.sample_rate
        return SlidingWindow(start=start / sr, duration=size / sr, step=step / sr)


class _CheckpointUnpickler(__import__("pickle").Unpickler):
    """Resolves the reference's pickled task types to this package's mirrors (core.py)."""

    _MAP = {("pyannote.audio.core.task", "Specifications"): Specifications,
            ("pyannote.audio.core.task", "Problem"): Problem,
            ("pyannote.audio.core.task", "Resolution"): Resolution}

    def find_class(self, module, name):
        hit = self._MAP.get((module, name))
        if hit is not None:
            return hit
        if module.split(".")[0] in ("lightning", "pytorch_lightning", "lightning_fabric"):
            # e.g. AttributeDict for hyper_parameters: a plain dict subclass is enough
            return dict
        return super().find_class(module, name)


class _checkpoint_pickle:
    """``pickle_module`` for torch.load: the stdlib pickle with the class mapping above."""

    import pickle as _p

    Unpickler = _CheckpointUnpickler
    Pickler = _p.Pickler
    load = staticmethod(lambda f, **kw: _CheckpointUnpickler(f, **kw).load())
    loads = staticmethod(_p.loads)
    dump = staticmethod(_p.dump)
    dumps = staticmethod(_p.dumps)
    HIGHEST_PROTOCOL = _p.HIGHEST_PROTOCOL
    __name__ = "pickle"


def _mel_sinc_init(n_filters=80, sample_rate=16000.0, min_low_hz=50, min_band_hz=50):
    def to_mel(hz):
        return 2595 * np.log10(1 + hz / 700)

    def to_hz(mel):
        return 700 * (10 ** (mel / 2595) - 1)

    mel = np.linspace(to_mel(30), to_mel(sample_rate / 2 - (min_low_hz + min_band_hz)),
                      n_filters // 2 + 1, dtype="float32")
    hz = to_hz(mel)
    return torch.from_numpy(hz[:-1]).view(-1, 1), torch.from_numpy(np.diff(hz)).view(-1, 1)


def sinc_buffers(kernel_size=251, sample_rate=16000.0):
    half = kernel_size // 2
    window_ = torch.from_numpy(np.hamming(kernel_size)[:half]).float()
    n_ = 2 * np.pi * (torch.arange(-half, 0.0).view(1, -1) / sample_rate)
    return window_, n_


class _ParamSincFB(nn.Module):
    def __init__(self):
        super().__init__()
        low, band = _mel_sinc_init()
        self.low_hz_ = nn.Parameter(low, requires_grad=False)
        self.band_hz_ = nn.Parameter(band, requires_grad=False)
        window_, n_ = sinc_buffers()
        self.register_buffer("window_", window_)
        self.register_buffer("n_", n_)


class _Encoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.filterbank = _ParamSincFB()


class _SincNetParams(nn.Module):
    """Parameter container with the key names of models/blocks/sincnet.py:41-79."""

    def __init__(self):
        super().__init__()
        self.wav_norm1d = nn.InstanceNorm1d(1, affine=True)
        self.conv1d = nn.ModuleList([_Encoder(), nn.Conv1d(80, 60, 5), nn.Conv1d(60, 60, 5)])
        self.norm1d = nn.ModuleList([nn.InstanceNorm1d(80, affine=True), nn.InstanceNorm1d(60, affine=True),
                                     nn.InstanceNorm1d(60, affine=True)])


class _SegmentationModel(Model):
    """A front end, then the head PyanNet and SSeRiouSS share: 1-4 BiLSTM layers of 128, 2 linear layers of 128 and a
    classifier of 1 to 32 classes, log-softmax for powerset / mono-label problems, sigmoid for binary and multi-label
    problems (core/model.py:271-300).  A subclass holds its front-end modules and defines KERNEL / STRIDE (the front
    end's convolutions), num_frames and check_window; its _SLOT ("seg" | "ssl") names its ops.Context head."""

    def _head_hparams(self, lstm: Optional[dict], linear: Optional[dict]):
        """(lstm, linear) hyper-parameters with the defaults filled in; a head shape without a kernel is refused."""
        lstm_hp = {"hidden_size": 128, "num_layers": 4, "bidirectional": True, "monolithic": True, "dropout": 0.0}
        lstm_hp.update(lstm or {})
        linear_hp = {"hidden_size": 128, "num_layers": 2}
        linear_hp.update(linear or {})
        if (lstm_hp["hidden_size"], lstm_hp["bidirectional"], lstm_hp["monolithic"]) != (128, True, True) or \
                not (1 <= lstm_hp["num_layers"] <= 4) or (linear_hp["hidden_size"], linear_hp["num_layers"]) != (128, 2):
            raise NotImplementedError(f"the CUDA kernels implement {type(self).__name__} with the community-1 head "
                                      f"shape only: 1-4 monolithic bidirectional LSTM layers of 128, 2 linear layers "
                                      f"of 128")
        return lstm_hp, linear_hp

    def _build_head(self, in_features: int, duration: float):
        """The head's modules after the front end's (the state-dict order): lstm on ``in_features`` inputs, linear,
        and the classifier of community-1's powerset specifications."""
        self.lstm = nn.LSTM(in_features, hidden_size=128, num_layers=self.hparams.lstm["num_layers"],
                            bidirectional=True, batch_first=True)
        self.linear = nn.ModuleList([nn.Linear(256, 128), nn.Linear(128, 128)])
        self.specifications = Specifications(problem=Problem.MONO_LABEL_CLASSIFICATION, resolution=Resolution.FRAME,
                                             duration=duration, warm_up=(0.0, 0.0),
                                             classes=["speaker#1", "speaker#2", "speaker#3"], powerset_max_classes=2,
                                             permutation_invariant=True)

    @property
    def specifications(self) -> Specifications:
        return self._specifications

    @specifications.setter
    def specifications(self, specifications: Specifications):
        """As the reference's Model.specifications setter followed by PyanNet.build (core/model.py:131-146,
        PyanNet.py:152-161): the classifier becomes a fresh Linear(128, dimension).  Heads without a kernel (more than
        32 classes, or a problem that is not a classification) are refused here, before any device work."""
        if isinstance(specifications, (tuple, list)):
            raise ValueError(f"{type(self).__name__} does not support multi-tasking.")
        if not isinstance(specifications, Specifications):
            raise ValueError("Only regular specifications or tuple of specifications are supported.")
        ops.seg_activation(specifications)
        dimension = specifications.num_powerset_classes if specifications.powerset else len(specifications.classes)
        ops.check_seg_classes(dimension)
        self._specifications = specifications
        self.classifier = nn.Linear(128, dimension).to(self._dummy.device)
        for p in self.parameters():
            p.requires_grad_(False)
        self._bump_weights()

    @property
    def dimension(self) -> int:
        specs = self.specifications
        return specs.num_powerset_classes if specs.powerset else len(specs.classes)

    def receptive_field_size(self, num_frames: int = 1) -> int:
        rf = num_frames
        for k, s in reversed(list(zip(self.KERNEL, self.STRIDE))):
            rf = 1 + (k - 1) + (rf - 1) * s
        return rf

    def receptive_field_center(self, frame: int = 0) -> int:
        c = frame
        for k, s in reversed(list(zip(self.KERNEL, self.STRIDE))):
            c = c * s + (k - 1) // 2
        return c

    def forward_chunks(self, wav: torch.Tensor, chunk_off, chunk_valid, return_logp: bool = False, out=None,
                       window: int = ops.CHUNK, reduce_max: bool = False):
        """Hot-path entry: windows of ``window`` samples addressed inside one resident device waveform (no unfold
        copy) -> classes (chunks, num_frames(window)) uint8 for a log-softmax head, sigmoid scores
        (chunks, num_frames(window), dimension) float32 (or their per-frame maximum with ``reduce_max``) for a
        sigmoid head (ops.Context.seg_forward / ssl_forward)."""
        self.check_window(window)
        ctx_forward = getattr(self._ctx(), self._SLOT + "_forward")           # seg_forward | ssl_forward
        return ctx_forward(wav, chunk_off, chunk_valid, return_logp=return_logp, out=out, window=window,
                           reduce_max=reduce_max)

    def forward(self, waveforms: torch.Tensor) -> torch.Tensor:
        """waveforms (batch, channel, samples), samples at least check_window's minimum -> (batch,
        num_frames(samples), dimension): log-probabilities of a log-softmax head, sigmoid scores of a sigmoid head."""
        b, c, s = waveforms.shape
        if c != 1:
            raise ValueError(f"{type(self).__name__} kernels expect mono waveforms, got {c} channels")
        flat = waveforms.to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
        off = np.arange(b, dtype=np.int64) * s
        valid = np.full(b, s, dtype=np.int32)
        if ops.seg_activation(self.specifications) == ops.SEG_SIGMOID:
            return self.forward_chunks(flat, off, valid, window=s)
        _, logp = self.forward_chunks(flat, off, valid, return_logp=True, window=s)
        return logp


class PyanNet(_SegmentationModel):
    """SincNet > LSTM > Feed forward > Classifier, community-1 trunk (1-4 BiLSTM layers of 128, 2x128 linear) with
    any head of 1 to 32 classes: log-softmax for powerset / mono-label problems, sigmoid for binary and multi-label
    problems (core/model.py:271-300)."""

    _SLOT = "seg"
    _HPARAMS = ("sincnet", "lstm", "linear", "sample_rate", "num_channels")
    KERNEL = [251, 3, 5, 3, 5, 3]
    STRIDE = [10, 3, 1, 3, 1, 3]

    def __init__(self, sincnet: Optional[dict] = None, lstm: Optional[dict] = None, linear: Optional[dict] = None,
                 sample_rate: int = 16000, num_channels: int = 1, duration: float = 10.0):
        super().__init__(sample_rate=sample_rate, num_channels=num_channels)
        if sample_rate != 16000:
            raise NotImplementedError("SincNet only supports 16kHz audio for now.")
        sinc_hp = {"stride": 10}
        sinc_hp.update(sincnet or {})
        if sinc_hp["stride"] != 10:
            raise NotImplementedError("the CUDA kernels implement the community-1 PyanNet shape only: SincNet stride 10")
        lstm_hp, linear_hp = self._head_hparams(lstm, linear)
        self.hparams.sincnet, self.hparams.lstm, self.hparams.linear = sinc_hp, lstm_hp, linear_hp
        self.sincnet = _SincNetParams()
        self._build_head(60, duration)

    def num_frames(self, num_samples: int) -> int:
        n = num_samples
        for k, s in zip(self.KERNEL, self.STRIDE):
            n = _conv1d_num_frames(n, k, s)
        return n

    def check_window(self, num_samples: int):
        """Refuses windows too short for the kernels (Inference checks its window with this)."""
        ops.check_seg_window(num_samples)

    def _upload(self, ctx):
        ctx.load_segmentation(self.state_dict(), self.specifications)


class _BasicBlockParams(nn.Module):
    def __init__(self, in_planes, planes, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes, 3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=stride, bias=False),
                                          nn.BatchNorm2d(planes))


class _ResNet34Params(nn.Module):
    """Parameter container with the key names of models/embedding/wespeaker/resnet.py:233-252."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(1, 32, 3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(32)
        in_planes = 32
        for li, (planes, n, stride) in enumerate(((32, 3, 1), (64, 4, 2), (128, 6, 2), (256, 3, 2)), start=1):
            blocks = []
            for s in [stride] + [1] * (n - 1):
                blocks.append(_BasicBlockParams(in_planes, planes, s))
                in_planes = planes
            setattr(self, f"layer{li}", nn.Sequential(*blocks))
        self.seg_1 = nn.Linear(5120, 256)


class _BottleneckParams(nn.Module):
    """A Bottleneck block (resnet.py:148-176): 1x1 in -> p, 3x3 p -> p with the stride, 1x1 p -> 4p."""

    def __init__(self, in_planes, planes, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, 4 * planes, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(4 * planes)
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != 4 * planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, 4 * planes, 1, stride=stride, bias=False),
                                          nn.BatchNorm2d(4 * planes))


class _BottleneckResNetParams(nn.Module):
    """Parameter container with the key names of the bottleneck ResNet (resnet.py:214-252, 477-508), two_emb_layer
    False: 1024 trunk channels, seg_1 20480 -> 256."""

    def __init__(self, num_blocks):
        super().__init__()
        self.conv1 = nn.Conv2d(1, 32, 3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(32)
        in_planes = 32
        for li, (planes, n, stride) in enumerate(zip((32, 64, 128, 256), num_blocks, (1, 2, 2, 2)), start=1):
            blocks = []
            for s in [stride] + [1] * (n - 1):
                blocks.append(_BottleneckParams(in_planes, planes, s))
                in_planes = 4 * planes
            setattr(self, f"layer{li}", nn.Sequential(*blocks))
        self.seg_1 = nn.Linear(20480, 256)


class BaseWeSpeakerResNet(Model):
    """What the WeSpeaker ResNets share (wespeaker/__init__.py:41-322): the fbank, the frame arithmetic, TSTP pooling
    and the 256-dimensional embedding.  Subclasses build ``resnet``, the parameter container of their trunk, in
    ``_make_resnet``."""

    _SLOT = "emb"
    _HPARAMS = ("sample_rate", "num_channels", "num_mel_bins", "frame_length", "frame_shift", "dither",
                "window_type", "use_energy")

    def __init__(self, sample_rate: int = 16000, num_channels: int = 1, num_mel_bins: int = 80,
                 frame_length: int = 25, frame_shift: int = 10, dither: float = 0.0, window_type: str = "hamming",
                 use_energy: bool = False):
        super().__init__(sample_rate=sample_rate, num_channels=num_channels)
        if (sample_rate, num_mel_bins, frame_length, frame_shift, dither, window_type, use_energy) != \
                (16000, 80, 25, 10, 0.0, "hamming", False):
            raise NotImplementedError("the fbank kernel implements the community-1 configuration only "
                                      "(16 kHz, 80 mel bins, 25/10 ms hamming frames, no dither, no energy)")
        self.resnet = self._make_resnet()
        self.specifications = Specifications(problem=Problem.REPRESENTATION, resolution=Resolution.CHUNK, duration=10.0)
        self.eval()
        for p in self.parameters():
            p.requires_grad_(False)

    def _make_resnet(self) -> nn.Module:
        raise NotImplementedError

    @property
    def dimension(self) -> int:
        return 256

    # smallest input for which kaldi.fbank yields a frame (speaker_verification.py:688-702 finds it by bisection on
    # exceptions; with a 400-sample analysis window the bisection converges to 400)
    min_num_samples = 400

    def _upload(self, ctx):
        ctx.load_embedding(self.state_dict())

    def forward_utterances(self, wav: torch.Tensor, off, num_samples: int, weights: Optional[torch.Tensor] = None):
        """Embeddings of utterances of one length inside one device waveform (ops.Context.emb_forward_utt):
        soft (n, Tw) / (n, S, Tw) weights or None -> (n, max(S, 1), 256)."""
        return self._ctx().emb_forward_utt(wav, off, num_samples, weights=weights)

    def num_frames(self, num_samples: int) -> int:
        n = _conv1d_num_frames(num_samples, 400, 160)
        for s in (1, 2, 2, 2):
            n = _conv1d_num_frames(n, 3, s, p=1)
        return n

    def forward_chunks(self, wav: torch.Tensor, chunk_off, chunk_valid, masks: torch.Tensor, out=None,
                       peers=None) -> torch.Tensor:
        """Hot-path entry: (num_chunks, 3, 589) uint8 masks -> (num_chunks, 3, 256) embeddings, one trunk pass."""
        return self._ctx().emb_forward(wav, chunk_off, chunk_valid, masks, out=out, peers=peers)

    def _flat(self, waveforms):
        b, c, s = waveforms.shape
        if c != 1 or s != ops.CHUNK:
            raise ValueError(f"WeSpeaker kernels expect mono {ops.CHUNK}-sample (10 s @ 16 kHz) chunks, got {c}x{s}")
        ctx = self._ctx()
        flat = waveforms.to(device=ctx.device, dtype=torch.float32).reshape(-1).contiguous()
        return ctx, flat, np.arange(b, dtype=np.int64) * s, np.full(b, s, dtype=np.int32)

    def compute_fbank(self, waveforms: torch.Tensor) -> torch.Tensor:
        ctx, flat, off, valid = self._flat(waveforms)
        return ctx.emb_fbank(flat, off, valid)

    def forward_frames(self, waveforms: torch.Tensor) -> torch.Tensor:
        return self._ctx().emb_trunk(self.compute_fbank(waveforms))

    def forward(self, waveforms: torch.Tensor, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        """waveforms (batch, 1, samples) with samples >= 400, weights (batch, frames) or (batch, speakers<=3, frames) in
        {0,1}.  10 s chunks take the diarization path (weights over the 589 segmentation frames); other lengths
        interpolate any number of weight frames onto the trunk frames."""
        b, c, s = waveforms.shape
        if c != 1:
            raise ValueError(f"WeSpeaker kernels expect mono waveforms, got {c} channels")
        if s < 400:
            raise ValueError(f"WeSpeaker needs at least 400 samples (one 25 ms fbank frame), got {s}")
        if s != ops.CHUNK:
            return self._forward_utt(waveforms, weights)
        ctx, flat, off, valid = self._flat(waveforms)
        b = len(off)
        if weights is None:
            w = torch.ones((b, 1, ops.FRAMES), dtype=torch.float32)
            squeeze = True
        else:
            squeeze = weights.dim() == 2
            w = weights.unsqueeze(1) if squeeze else weights
        if w.shape[-1] != ops.FRAMES or w.shape[1] > 3:
            raise ValueError("weights must have 589 frames and at most 3 speakers")
        if not bool(((w == 0) | (w == 1)).all()):
            raise ValueError("the masked statistics pooling kernel takes binary (0/1) weights")
        masks = torch.zeros((b, 3, ops.FRAMES), dtype=torch.uint8, device=ctx.device)
        masks[:, : w.shape[1]] = w.to(ctx.device).to(torch.uint8)
        emb = ctx.emb_forward(flat, off, valid, masks)[:, : w.shape[1]]
        return emb[:, 0] if squeeze else emb

    def _forward_utt(self, waveforms: torch.Tensor, weights: Optional[torch.Tensor]) -> torch.Tensor:
        b, _, s = waveforms.shape
        squeeze = weights is None or weights.dim() == 2
        if weights is not None:
            w = weights.unsqueeze(1) if weights.dim() == 2 else weights
            if w.dim() != 3 or w.shape[0] != b or w.shape[1] > 3 or w.shape[2] < 1:
                raise ValueError("weights must be (batch, frames) or (batch, speakers<=3, frames)")
            if not bool(((w == 0) | (w == 1)).all()):
                raise ValueError("the masked statistics pooling kernel takes binary (0/1) weights")
            weights = w
        ctx = self._ctx()
        flat = waveforms.to(device=ctx.device, dtype=torch.float32).reshape(-1).contiguous()
        emb = ctx.emb_forward_utt(flat, np.arange(b, dtype=np.int64) * s, s, weights=weights)
        return emb[:, 0] if squeeze else emb

    def forward_embedding(self, frames: torch.Tensor, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Frame-wise features (batch, C, 10, frames) -> (batch, 256), or (batch, speakers, 256) for
        (batch, speakers, frames) weights; C = 256 for ResNet34 and 1024 for the bottleneck ResNets.  Any number of
        frames, any real weights, any number of speakers."""
        emb = self._ctx().emb_forward_embedding(frames, weights=weights)
        return emb if weights is not None and weights.dim() == 3 else emb[:, 0]


class WeSpeakerResNet34(BaseWeSpeakerResNet):
    def _make_resnet(self):
        return _ResNet34Params()


class _BottleneckWeSpeakerResNet(BaseWeSpeakerResNet):
    NUM_BLOCKS = ()             # Bottleneck blocks per layer

    def _make_resnet(self):
        return _BottleneckResNetParams(self.NUM_BLOCKS)


class WeSpeakerResNet152(_BottleneckWeSpeakerResNet):
    NUM_BLOCKS = (3, 8, 36, 3)


class WeSpeakerResNet221(_BottleneckWeSpeakerResNet):
    NUM_BLOCKS = (6, 16, 48, 3)


class WeSpeakerResNet293(_BottleneckWeSpeakerResNet):
    NUM_BLOCKS = (10, 20, 64, 3)


class BaseXVector(Model):
    """What XVectorSincNet and XVectorMFCC share behind their front ends (xvector.py): five dilated TDNN layers (Conv1d
    -> LeakyReLU -> BatchNorm1d), StatsPool and a Linear to ``dimension``.  A subclass adds its front end's modules,
    ``_SLOT``, ``_HPARAMS``, ``min_num_samples``, the front end's frame arithmetic and ``forward_utterances``."""

    KERNEL = [5, 3, 3, 1, 1]
    DILATION = [1, 2, 3, 1, 1]
    min_num_samples = 0

    def _build_tdnn(self, in_channel: int, dimension: int):
        layers = []
        for (_, out_channel, k, d) in ops.XVEC_TDNN:
            layers += [nn.Conv1d(in_channel, out_channel, k, dilation=d), nn.LeakyReLU(), nn.BatchNorm1d(out_channel)]
            in_channel = out_channel
        self.tdnns = nn.ModuleList(layers)
        self.embedding = nn.Linear(2 * in_channel, int(dimension))
        self.specifications = Specifications(problem=Problem.REPRESENTATION, resolution=Resolution.CHUNK, duration=10.0)
        self.eval()
        for p in self.parameters():
            p.requires_grad_(False)

    @property
    def dimension(self) -> int:
        return self.hparams.dimension

    def _tdnn_num_frames(self, n: int) -> int:
        for k, d in zip(self.KERNEL, self.DILATION):
            n = _conv1d_num_frames(n, k, 1, d=d)
        return n

    def _tdnn_receptive_field_size(self, num_frames: int) -> int:
        rf = num_frames
        for k, d in reversed(list(zip(self.KERNEL, self.DILATION))):
            rf = 1 + (k - 1) * d + (rf - 1)
        return rf

    def _tdnn_receptive_field_center(self, frame: int) -> int:
        c = frame
        for k, d in reversed(list(zip(self.KERNEL, self.DILATION))):
            c = c + (1 + (k - 1) * d - 1) // 2
        return c

    def forward(self, waveforms: torch.Tensor, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        """waveforms (batch, 1, samples) with samples >= min_num_samples, weights None, (batch, frames) or
        (batch, speakers, frames) of any real values -> (batch, dimension) or (batch, speakers, dimension)."""
        name = type(self).__name__
        b, c, s = waveforms.shape
        if c != 1:
            raise ValueError(f"{name} kernels expect mono waveforms, got {c} channels")
        if s < self.min_num_samples:
            raise ValueError(f"{name} needs at least {self.min_num_samples} samples, got {s}")
        if weights is not None and (weights.dim() not in (2, 3) or weights.shape[0] != b or weights.shape[-1] < 1):
            raise ValueError("weights must be (batch, frames) or (batch, speakers, frames)")
        ctx = self._ctx()
        flat = waveforms.to(device=ctx.device, dtype=torch.float32).reshape(-1).contiguous()
        emb = self.forward_utterances(flat, np.arange(b, dtype=np.int64) * s, s, weights=weights)
        return emb if weights is not None and weights.dim() == 3 else emb[:, 0]


class XVectorSincNet(BaseXVector):
    """x-vector on the SincNet front end (xvector.py:205-349; the architecture of pyannote/embedding): SincNet, five
    dilated TDNN layers (Conv1d -> LeakyReLU -> BatchNorm1d), StatsPool and a Linear to ``dimension``."""

    _SLOT = "xvec"
    _HPARAMS = ("sincnet", "dimension", "sample_rate", "num_channels")
    min_num_samples = ops.XVEC_MIN_SAMPLES

    def __init__(self, sample_rate: int = 16000, num_channels: int = 1, sincnet: Optional[dict] = None,
                 dimension: int = 512):
        super().__init__(sample_rate=sample_rate, num_channels=num_channels)
        sinc_hp = {"stride": 10}
        sinc_hp.update(sincnet or {})
        sinc_hp["sample_rate"] = sample_rate
        if sample_rate != 16000 or sinc_hp["stride"] != 10 or num_channels != 1 or int(dimension) < 1:
            raise NotImplementedError("the CUDA kernels implement XVectorSincNet on mono 16 kHz audio with SincNet "
                                      "stride 10 and a positive embedding dimension only")
        self.hparams.sincnet, self.hparams.dimension = sinc_hp, int(dimension)
        self.sincnet = _SincNetParams()
        self._build_tdnn(60, dimension)

    def num_frames(self, num_samples: int) -> int:
        n = num_samples
        for k, s in zip(PyanNet.KERNEL, PyanNet.STRIDE):
            n = _conv1d_num_frames(n, k, s)
        return self._tdnn_num_frames(n)

    def receptive_field_size(self, num_frames: int = 1) -> int:
        rf = self._tdnn_receptive_field_size(num_frames)
        for k, s in reversed(list(zip(PyanNet.KERNEL, PyanNet.STRIDE))):
            rf = 1 + (k - 1) + (rf - 1) * s
        return rf

    def receptive_field_center(self, frame: int = 0) -> int:
        c = self._tdnn_receptive_field_center(frame)
        for k, s in reversed(list(zip(PyanNet.KERNEL, PyanNet.STRIDE))):
            c = c * s + (k - 1) // 2
        return c

    def _upload(self, ctx):
        ctx.load_xvector(self.state_dict())

    def forward_utterances(self, wav: torch.Tensor, off, num_samples: int, weights: Optional[torch.Tensor] = None):
        """Embeddings of utterances of one length inside one device waveform (ops.Context.xvec_forward): soft
        (n, Tw) / (n, S, Tw) weights or None -> (n, max(S, 1), dimension)."""
        return self._ctx().xvec_forward(wav, off, num_samples, weights=weights)


# torchaudio.transforms.MFCC's defaults at 16 kHz: the only MFCC configuration the kernels implement
MFCC_DEFAULTS = {"n_mfcc": 40, "dct_type": 2, "norm": "ortho", "log_mels": False}
MFCC_N_FFT, MFCC_HOP, MFCC_N_MELS = 400, 200, 128


def mfcc_buffers(sample_rate: int = 16000) -> "OrderedDict[str, torch.Tensor]":
    """The three buffers of torchaudio's default MFCC under the reference's keys (without the ``mfcc.`` prefix),
    restated without torchaudio: dct_mat = torchaudio.functional.create_dct(40, 128, "ortho"), the periodic Hann
    window of 400 samples and fb = melscale_fbanks(201, 0, sample_rate / 2, 128, sample_rate, norm=None,
    mel_scale="htk")."""
    from collections import OrderedDict

    n_mels, n_mfcc, n_freqs = MFCC_N_MELS, MFCC_DEFAULTS["n_mfcc"], MFCC_N_FFT // 2 + 1
    n = torch.arange(float(n_mels))
    k = torch.arange(float(n_mfcc)).unsqueeze(1)
    dct = torch.cos(math.pi / float(n_mels) * (n + 0.5) * k)
    dct[0] *= 1.0 / math.sqrt(2.0)
    dct *= math.sqrt(2.0 / float(n_mels))
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_max = 2595.0 * math.log10(1.0 + (sample_rate / 2) / 700.0)
    m_pts = torch.linspace(0.0, m_max, n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    fb = torch.max(torch.zeros(1), torch.min(down, up))
    return OrderedDict([("dct_mat", dct.t().contiguous()),
                        ("MelSpectrogram.spectrogram.window", torch.hann_window(MFCC_N_FFT)),
                        ("MelSpectrogram.mel_scale.fb", fb)])


class _MfccParams(nn.Module):
    """Holds torchaudio MFCC's buffers under the reference's state-dict keys (``mfcc.dct_mat``,
    ``mfcc.MelSpectrogram.spectrogram.window``, ``mfcc.MelSpectrogram.mel_scale.fb``); the kernels use the loaded
    values."""

    def __init__(self, sample_rate: int = 16000):
        super().__init__()
        buf = mfcc_buffers(sample_rate)
        self.register_buffer("dct_mat", buf["dct_mat"])
        self.MelSpectrogram = nn.Module()
        self.MelSpectrogram.spectrogram = nn.Module()
        self.MelSpectrogram.spectrogram.register_buffer("window", buf["MelSpectrogram.spectrogram.window"])
        self.MelSpectrogram.mel_scale = nn.Module()
        self.MelSpectrogram.mel_scale.register_buffer("fb", buf["MelSpectrogram.mel_scale.fb"])


class XVectorMFCC(BaseXVector):
    """x-vector on torchaudio's MFCC (xvector.py:42-202): 40 MFCC per 200-sample hop, five dilated TDNN layers
    (Conv1d -> LeakyReLU -> BatchNorm1d), StatsPool and a Linear to ``dimension``."""

    _SLOT = "xvec_mfcc"
    _HPARAMS = ("mfcc", "dimension", "sample_rate", "num_channels")
    min_num_samples = ops.XVEC_MFCC_MIN_SAMPLES

    def __init__(self, sample_rate: int = 16000, num_channels: int = 1, mfcc: Optional[dict] = None,
                 dimension: int = 512):
        super().__init__(sample_rate=sample_rate, num_channels=num_channels)
        mfcc_hp = dict(MFCC_DEFAULTS)
        mfcc_hp.update(mfcc or {})
        if not mfcc_hp.get("melkwargs", True):
            del mfcc_hp["melkwargs"]                       # melkwargs None / {}: torchaudio's defaults
        mfcc_hp["sample_rate"] = sample_rate
        if sample_rate != 16000 or num_channels != 1 or int(dimension) < 1 or \
                mfcc_hp != dict(MFCC_DEFAULTS, sample_rate=sample_rate):
            raise NotImplementedError(f"the CUDA kernels implement XVectorMFCC on mono 16 kHz audio with torchaudio's "
                                      f"default MFCC ({MFCC_DEFAULTS}, no melkwargs) and a positive embedding "
                                      f"dimension only, got sample_rate={sample_rate}, num_channels={num_channels}, "
                                      f"mfcc={mfcc}")
        self.hparams.mfcc, self.hparams.dimension = mfcc_hp, int(dimension)
        self.mfcc = _MfccParams(sample_rate)
        self._build_tdnn(MFCC_DEFAULTS["n_mfcc"], dimension)

    def num_frames(self, num_samples: int) -> int:
        return self._tdnn_num_frames(1 + num_samples // MFCC_HOP)          # center=True

    def receptive_field_size(self, num_frames: int = 1) -> int:
        return MFCC_N_FFT + (self._tdnn_receptive_field_size(num_frames) - 1) * MFCC_HOP

    def receptive_field_center(self, frame: int = 0) -> int:
        return self._tdnn_receptive_field_center(frame) * MFCC_HOP

    def _upload(self, ctx):
        ctx.load_xvector_mfcc(self.state_dict())

    def forward_utterances(self, wav: torch.Tensor, off, num_samples: int, weights: Optional[torch.Tensor] = None):
        """Embeddings of utterances of one length inside one device waveform (ops.Context.xvec_mfcc_forward): soft
        (n, Tw) / (n, S, Tw) weights or None -> (n, max(S, 1), dimension)."""
        return self._ctx().xvec_mfcc_forward(wav, off, num_samples, weights=weights)

    def mfcc_features(self, waveforms: torch.Tensor) -> torch.Tensor:
        """The MFCC front end alone: (batch, 1, samples) -> (batch, 40, 1 + samples // 200), torchaudio's layout."""
        b, c, s = waveforms.shape
        if c != 1:
            raise ValueError(f"XVectorMFCC kernels expect mono waveforms, got {c} channels")
        ctx = self._ctx()
        flat = waveforms.to(device=ctx.device, dtype=torch.float32).reshape(-1).contiguous()
        return ctx.mfcc_features(flat, np.arange(b, dtype=np.int64) * s, s).transpose(1, 2)


# ---- SSeRiouSS ----------------------------------------------------------------------------------------------------
# torchaudio.pipelines.WAVLM_BASE._params (== WAVLM_BASE_PLUS._params): the only front-end configuration the kernels
# implement.  The package does not import torchaudio; the table is written out here.
WAVLM_BASE_PARAMS = {
    "extractor_mode": "group_norm", "extractor_conv_bias": False,
    "extractor_conv_layer_config": [(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2,
    "encoder_embed_dim": 768, "encoder_pos_conv_kernel": 128, "encoder_pos_conv_groups": 16,
    "encoder_num_layers": 12, "encoder_num_heads": 12, "encoder_max_distance": 800, "encoder_num_buckets": 320,
    "encoder_ff_interm_features": 3072, "encoder_layer_norm_first": False,
}
SSL_BUNDLES = ("WAVLM_BASE", "WAVLM_BASE_PLUS")


class _ConvLayerParams(nn.Module):
    def __init__(self, cin, k, s, norm):
        super().__init__()
        self.conv = nn.Conv1d(cin, 512, k, stride=s, bias=False)
        if norm:
            self.layer_norm = nn.GroupNorm(512, 512)


class _FeatureExtractorParams(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv_layers = nn.ModuleList(
            [_ConvLayerParams(1 if i == 0 else 512, k, s, i == 0)
             for i, (_, k, s) in enumerate(WAVLM_BASE_PARAMS["extractor_conv_layer_config"])])


class _WeightNormParams(nn.Module):
    """torch.nn.utils.parametrizations.weight_norm(dim=2) of the positional conv: original0 = g, original1 = v."""

    def __init__(self):
        super().__init__()
        self.original0 = nn.Parameter(torch.ones(1, 1, 128))
        self.original1 = nn.Parameter(torch.randn(768, 48, 128) * 0.02)


class _PosConvParams(nn.Module):
    """pos_conv_embed.conv with the parametrization's key names.  Checkpoints saved with the older
    torch.nn.utils.weight_norm spell the pair ``weight_g`` / ``weight_v``; they are renamed on load."""

    def __init__(self):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(768))
        self.parametrizations = nn.Module()
        self.parametrizations.weight = _WeightNormParams()
        self._register_load_state_dict_pre_hook(self._rename_weight_norm)

    @staticmethod
    def _rename_weight_norm(state_dict, prefix, *args):
        for old, new in (("weight_g", "parametrizations.weight.original0"),
                         ("weight_v", "parametrizations.weight.original1")):
            if prefix + old in state_dict:
                state_dict[prefix + new] = state_dict.pop(prefix + old)


class _WavLMAttentionParams(nn.Module):
    def __init__(self, first):
        super().__init__()
        if first:
            self.rel_attn_embed = nn.Embedding(320, 12)
        self.attention = nn.MultiheadAttention(768, 12, batch_first=True)
        self.gru_rel_pos_linear = nn.Linear(64, 8)
        self.gru_rel_pos_const = nn.Parameter(torch.ones(1, 12, 1, 1))


class _FeedForwardParams(nn.Module):
    def __init__(self):
        super().__init__()
        self.intermediate_dense = nn.Linear(768, 3072)
        self.output_dense = nn.Linear(3072, 768)


class _EncoderLayerParams(nn.Module):
    def __init__(self, first):
        super().__init__()
        self.attention = _WavLMAttentionParams(first)
        self.layer_norm = nn.LayerNorm(768)
        self.feed_forward = _FeedForwardParams()
        self.final_layer_norm = nn.LayerNorm(768)


class _WavLMParams(nn.Module):
    """Parameter container with the key names of torchaudio's wavlm_model(**WAVLM_BASE._params)."""

    def __init__(self):
        super().__init__()
        self.feature_extractor = _FeatureExtractorParams()
        self.encoder = nn.Module()
        self.encoder.feature_projection = nn.Module()
        self.encoder.feature_projection.layer_norm = nn.LayerNorm(512)
        self.encoder.feature_projection.projection = nn.Linear(512, 768)
        self.encoder.transformer = nn.Module()
        self.encoder.transformer.pos_conv_embed = nn.Module()
        self.encoder.transformer.pos_conv_embed.conv = _PosConvParams()
        self.encoder.transformer.layer_norm = nn.LayerNorm(768)
        self.encoder.transformer.layers = nn.ModuleList([_EncoderLayerParams(i == 0) for i in range(12)])


class SSeRiouSS(_SegmentationModel):
    """WavLM Base > LSTM > Feed forward > Classifier (models/segmentation/SSeRiouSS.py) with ``wav2vec`` one of
    "WAVLM_BASE" / "WAVLM_BASE_PLUS", the PyanNet LSTM / linear shape (1-4 BiLSTM layers of 128, 2 linear layers of
    128) and any head PyanNet accepts.  ``wav2vec_layer`` < 0 averages the 12 layer outputs with
    softmax(``wav2vec_weights``); 1 .. 12 takes that layer's output.  ``wav2vec_frozen`` and dropout only concern
    training and change nothing here."""

    _SLOT = "ssl"
    _HPARAMS = ("wav2vec", "wav2vec_frozen", "wav2vec_layer", "lstm", "linear", "sample_rate", "num_channels")
    KERNEL = [k for (_, k, _) in WAVLM_BASE_PARAMS["extractor_conv_layer_config"]]
    STRIDE = [s for (_, _, s) in WAVLM_BASE_PARAMS["extractor_conv_layer_config"]]
    min_num_samples = ops.SSL_MIN_SAMPLES

    def __init__(self, wav2vec=None, wav2vec_frozen: bool = False, wav2vec_layer: int = -1,
                 lstm: Optional[dict] = None, linear: Optional[dict] = None, sample_rate: int = 16000,
                 num_channels: int = 1, duration: float = 10.0):
        super().__init__(sample_rate=sample_rate, num_channels=num_channels)
        wav2vec = "WAVLM_BASE" if wav2vec is None else wav2vec
        if not isinstance(wav2vec, str) or wav2vec not in SSL_BUNDLES:
            raise NotImplementedError(f"SSeRiouSS has CUDA kernels for the WavLM Base front end only "
                                      f"(wav2vec = {' / '.join(SSL_BUNDLES)}), not for {wav2vec!r}")
        if sample_rate != 16000:
            raise ValueError(f"Expected 16000Hz, found {sample_rate}Hz.")
        wav2vec_layer = int(wav2vec_layer)
        if not (wav2vec_layer < 0 or 1 <= wav2vec_layer <= 12):
            raise ValueError(f"`wav2vec_layer` must be negative or between 1 and 12, got {wav2vec_layer}")
        lstm_hp, linear_hp = self._head_hparams(lstm, linear)
        self.hparams.wav2vec, self.hparams.wav2vec_frozen = wav2vec, bool(wav2vec_frozen)
        self.hparams.wav2vec_layer, self.hparams.lstm, self.hparams.linear = wav2vec_layer, lstm_hp, linear_hp
        self.wav2vec = _WavLMParams()
        if wav2vec_layer < 0:
            self.wav2vec_weights = nn.Parameter(torch.ones(12))
        self._build_head(768, duration)

    def num_frames(self, num_samples: int) -> int:
        return ops.ssl_num_frames(num_samples)

    def check_window(self, num_samples: int):
        """Refuses windows shorter than one WavLM frame (400 samples)."""
        ops.check_ssl_window(num_samples)

    def _upload(self, ctx):
        ctx.load_sseriouss(self.state_dict(), self.specifications, self.hparams.wav2vec_layer)
