"""Thin Python layer over the C ABI: one ``Context`` per device, torch tensors for device memory and streams.

Nothing here computes on the CPU: every op forwards raw device pointers to libb200diar.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Mapping, Optional, Sequence

import numpy as np
import torch

from . import _lib

CHUNK = 160000
FRAMES = 589
SPEAKERS = 3
CLASSES = 7
SEG_MAX_CLASSES = 32       # largest classifier head of the segmentation kernels (and largest powerset)
SEG_LOGSOFTMAX, SEG_SIGMOID = 0, 1
EMB_DIM = 256
SEG_MIN_SAMPLES = 1261     # shortest PyanNet window: 2 output frames (one frame cannot be instance-normalised)
XVEC_MIN_SAMPLES = 4771    # shortest XVectorSincNet input: 15 SincNet frames, one frame after the TDNN layers
XVEC_MFCC_MIN_SAMPLES = 2800   # shortest XVectorMFCC input: 15 MFCC frames
XVEC_TDNN = ((60, 512, 5, 1), (512, 512, 3, 2), (512, 512, 3, 3), (512, 512, 1, 1), (512, 1500, 1, 1))


def seg_num_frames(num_samples: int) -> int:
    """PyanNet output frames of a window (models/segmentation/PyanNet.py num_frames): sinc conv (251, stride 10),
    MaxPool 3, Conv1d 5, MaxPool 3, Conv1d 5, MaxPool 3.  589 for 160000 samples."""
    n = 1 + (int(num_samples) - 251) // 10
    return ((n // 3 - 4) // 3 - 4) // 3


def check_seg_window(num_samples: int):
    if int(num_samples) < SEG_MIN_SAMPLES:
        raise ValueError(f"PyanNet needs windows of at least {SEG_MIN_SAMPLES} samples (2 output frames), got "
                         f"{int(num_samples)}")


SSL_MIN_SAMPLES = 400      # shortest SSeRiouSS window: one WavLM frame (receptive field 400 samples, step 320)
SSL_LAYERS = 12
SSL_REL_SPAN = 1023        # relative offsets beyond +-1023 frames share the (saturated) bucket of +-1023


def ssl_num_frames(num_samples: int) -> int:
    """WavLM Base feature-extractor frames of a window: conv (10, 5), 4 x conv (3, 2), 2 x conv (2, 2).  499 for
    160000 samples, 1 for 400."""
    n = 1 + (int(num_samples) - 10) // 5
    for k in (3, 3, 3, 3, 2, 2):
        n = 1 + (n - k) // 2
    return n


def check_ssl_window(num_samples: int):
    if int(num_samples) < SSL_MIN_SAMPLES:
        raise ValueError(f"SSeRiouSS needs windows of at least {SSL_MIN_SAMPLES} samples (one WavLM frame), got "
                         f"{int(num_samples)}")


def wavlm_relative_buckets(num_buckets: int = 320, max_distance: int = 800) -> torch.Tensor:
    """int32 bucket of every relative offset d = key - query in [-1023, 1023] (index d + 1023), with the torch ops
    of WavLM's bidirectional bucketing (torchaudio wavlm_attention.py), so that the float ``log`` rounds alike."""
    d = torch.arange(-SSL_REL_SPAN, SSL_REL_SPAN + 1, dtype=torch.long)
    half = num_buckets // 2
    buckets = (d > 0).to(torch.long) * half
    a = torch.abs(d)
    max_exact = half // 2
    large = max_exact + (torch.log(a.float() / max_exact) / np.log(max_distance / max_exact)
                         * (half - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, half - 1))
    buckets = buckets + torch.where(a < max_exact, a, large)
    # the kernels clamp longer offsets to +-1023: the buckets must already be saturated there
    if int(buckets[0]) != half - 1 or int(buckets[-1]) != num_buckets - 1:
        raise AssertionError("relative position buckets are not saturated at +-1023 frames")
    return buckets.to(torch.int32).contiguous()


def check_seg_classes(num_classes: int):
    if not 1 <= int(num_classes) <= SEG_MAX_CLASSES:
        raise NotImplementedError(f"a PyanNet classifier of {int(num_classes)} classes has no CUDA kernel: the "
                                  f"segmentation heads have 1 to {SEG_MAX_CLASSES} classes")


def powerset_mapping(num_speakers: int, max_per_frame: int) -> np.ndarray:
    """(K, num_speakers) uint8 mapping of utils/powerset.py (build_mapping): set size 0 .. max_per_frame,
    itertools.combinations within each size.  Raises ValueError outside the kernels' range (K <= 32)."""
    from itertools import combinations
    from math import comb

    n, m = int(num_speakers), int(max_per_frame)
    if not 1 <= m <= n <= 32:
        raise ValueError(f"powerset of {n} speakers with at most {m} per frame: need 1 <= max_per_frame <= "
                         f"speakers <= 32")
    k = sum(comb(n, i) for i in range(m + 1))
    if k > SEG_MAX_CLASSES:
        raise ValueError(f"powerset of {n} speakers with at most {m} per frame has {k} classes; at most "
                         f"{SEG_MAX_CLASSES} are supported")
    rows = [[1 if j in s else 0 for j in range(n)] for size in range(m + 1) for s in combinations(range(n), size)]
    return np.array(rows, dtype=np.uint8)


def seg_activation(specifications) -> int:
    """Activation of a PyanNet head (core/model.py:271-300): sigmoid for binary and multi-label problems, log-softmax
    for mono-label (powerset) problems."""
    from .core import Problem

    if specifications.problem in (Problem.BINARY_CLASSIFICATION, Problem.MULTI_LABEL_CLASSIFICATION):
        return SEG_SIGMOID
    if specifications.problem == Problem.MONO_LABEL_CLASSIFICATION:
        return SEG_LOGSOFTMAX
    raise NotImplementedError(f"PyanNet heads for {specifications.problem} have no CUDA kernel")


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _fp(t: torch.Tensor):
    return C.cast(C.c_void_p(t.data_ptr()), _lib.c_float_p)


def _stream(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def sinc_filter_bank(low_hz_: torch.Tensor, band_hz_: torch.Tensor, window_: Optional[torch.Tensor] = None,
                     n_: Optional[torch.Tensor] = None, sample_rate: float = 16000.0, min_low_hz: float = 50.0,
                     min_band_hz: float = 50.0, kernel_size: int = 251) -> torch.Tensor:
    """Realise the (80,251) ParamSincFB filter bank from its parameters (done once at load, the weights are frozen).

    Same arithmetic, same op order as asteroid_filterbanks.ParamSincFB.filters() (call site
    /root/reference/src/pyannote/audio/models/blocks/sincnet.py:58-69), in torch fp32 on the CPU.
    """
    half = kernel_size // 2
    low_hz_ = low_hz_.detach().float().cpu()
    band_hz_ = band_hz_.detach().float().cpu()
    if window_ is None:
        window_ = torch.from_numpy(np.hamming(kernel_size)[:half]).float()
    if n_ is None:
        n_ = 2 * np.pi * (torch.arange(-half, 0.0).view(1, -1) / sample_rate)
    window_, n_ = window_.float().cpu(), n_.float().cpu()
    low = min_low_hz + torch.abs(low_hz_)
    high = torch.clamp(low + min_band_hz + torch.abs(band_hz_), min_low_hz, sample_rate / 2)
    band = (high - low)[:, 0]
    ft_low, ft_high = torch.matmul(low, n_), torch.matmul(high, n_)
    cos_left = ((torch.sin(ft_high) - torch.sin(ft_low)) / (n_ / 2)) * window_
    cos = torch.cat([cos_left, 2 * band.view(-1, 1), torch.flip(cos_left, dims=[1])], dim=1)
    sin_left = ((torch.cos(ft_low) - torch.cos(ft_high)) / (n_ / 2)) * window_
    sin = torch.cat([sin_left, torch.zeros_like(band.view(-1, 1)), -torch.flip(sin_left, dims=[1])], dim=1)
    bank = torch.cat([cos / (2 * band[:, None]), sin / (2 * band[:, None])], dim=0)
    return bank.contiguous()


def _state_dict_reader(sd: Mapping[str, torch.Tensor]):
    """``f(name)`` -> float pointer to a contiguous float32 CPU copy of ``sd[name]``.  The copies (and whatever else
    goes into ``f.keep``) stay alive as long as ``f``, i.e. until the loader that reads them has returned."""
    keep = []

    def f(name):
        t = sd[name].detach().to(torch.float32).cpu().contiguous()
        keep.append(t)
        return _fp(t)

    f.keep = keep
    return f


def _head_of(sd: Mapping[str, torch.Tensor], specifications) -> tuple:
    """(classes, activation) of a PyanNet or SSeRiouSS head: ``classifier.weight``'s K rows (1 .. 32), and the
    activation of ``specifications`` (sigmoid for binary / multi-label problems), log-softmax without them."""
    num_classes = int(sd["classifier.weight"].shape[0])
    check_seg_classes(num_classes)
    return num_classes, SEG_LOGSOFTMAX if specifications is None else seg_activation(specifications)


def _fill_head(w, sd: Mapping[str, torch.Tensor], f):
    """The ``lstm.*``, ``linear.*`` and ``classifier.*`` fields that SegWeights (PyanNet) and SslWeights (SSeRiouSS)
    share; the LSTM depth comes from the keys."""
    layers = 0
    while f"lstm.weight_ih_l{layers}" in sd:
        layers += 1
    w.lstm_layers = layers
    for layer in range(layers):
        for d, suffix in enumerate(("", "_reverse")):
            w.lstm_w_ih[layer * 2 + d] = f(f"lstm.weight_ih_l{layer}{suffix}")
            w.lstm_w_hh[layer * 2 + d] = f(f"lstm.weight_hh_l{layer}{suffix}")
            w.lstm_b_ih[layer * 2 + d] = f(f"lstm.bias_ih_l{layer}{suffix}")
            w.lstm_b_hh[layer * 2 + d] = f(f"lstm.bias_hh_l{layer}{suffix}")
    for i in range(2):
        w.linear_weight[i] = f(f"linear.{i}.weight")
        w.linear_bias[i] = f(f"linear.{i}.bias")
    w.classifier_weight = f("classifier.weight")
    w.classifier_bias = f("classifier.bias")


def _fill_sincnet(w, sd: Mapping[str, torch.Tensor], f):
    """The ``sincnet.*`` fields that SegWeights (PyanNet) and XvecWeights (XVectorSincNet) share."""
    w.wav_norm_weight = float(sd["sincnet.wav_norm1d.weight"].reshape(-1)[0])
    w.wav_norm_bias = float(sd["sincnet.wav_norm1d.bias"].reshape(-1)[0])
    p = "sincnet.conv1d.0.filterbank."
    bank = sinc_filter_bank(sd[p + "low_hz_"], sd[p + "band_hz_"], sd.get(p + "window_"), sd.get(p + "n_"))
    f.keep.append(bank)
    w.sinc_filters = _fp(bank)
    for i in range(3):
        w.norm_weight[i] = f(f"sincnet.norm1d.{i}.weight")
        w.norm_bias[i] = f(f"sincnet.norm1d.{i}.bias")
    for i in range(2):
        w.conv_weight[i] = f(f"sincnet.conv1d.{i + 1}.weight")
        w.conv_bias[i] = f(f"sincnet.conv1d.{i + 1}.bias")


def _fill_tdnn(w, sd: Mapping[str, torch.Tensor], f, cin0: int) -> int:
    """The ``tdnns.*`` and ``embedding.*`` fields that XvecWeights and XvecMfccWeights share (tdnns.0 has ``cin0``
    input channels); returns the embedding dimension."""
    for layer, (cin, cout, k, _) in enumerate(XVEC_TDNN):
        cin = cin0 if layer == 0 else cin
        conv, bn = f"tdnns.{3 * layer}", f"tdnns.{3 * layer + 2}"
        if tuple(sd[conv + ".weight"].shape) != (cout, cin, k):
            raise ValueError(f"{conv}.weight has shape {tuple(sd[conv + '.weight'].shape)}, expected "
                             f"{(cout, cin, k)}")
        w.tdnn_weight[layer] = f(conv + ".weight")
        w.tdnn_bias[layer] = f(conv + ".bias")
        w.bn_weight[layer] = f(bn + ".weight")
        w.bn_bias[layer] = f(bn + ".bias")
        w.bn_mean[layer] = f(bn + ".running_mean")
        w.bn_var[layer] = f(bn + ".running_var")
    dim, k_in = sd["embedding.weight"].shape
    if k_in != 3000:
        raise ValueError(f"embedding.weight has {k_in} inputs, expected 3000")
    w.dimension = int(dim)
    w.embedding_weight = f("embedding.weight")
    w.embedding_bias = f("embedding.bias")
    return int(dim)


def fold_weight_norm(sd: Mapping[str, torch.Tensor], prefix: str) -> torch.Tensor:
    """The plain fp32 weight of a conv under weight norm over dim 2 (torch.nn.utils.parametrizations.weight_norm, or
    the older torch.nn.utils.weight_norm): ``prefix + parametrizations.weight.original0 / original1`` or
    ``prefix + weight_g / weight_v``, folded with torch's own kernel."""
    if prefix + "parametrizations.weight.original0" in sd:
        g, v = sd[prefix + "parametrizations.weight.original0"], sd[prefix + "parametrizations.weight.original1"]
    else:
        g, v = sd[prefix + "weight_g"], sd[prefix + "weight_v"]
    g, v = g.detach().float().cpu(), v.detach().float().cpu()
    return torch._weight_norm(v, g, 2).contiguous()


def _norm_mode(normalize) -> int:
    """False/0: rows as given; True/1: fp64 L2 normalisation; "float32"/2: numpy's float32 normalisation of rows that
    hold float32 values (what the reference does to float32 embeddings before scipy's linkage)."""
    if normalize in ("float32", 2):
        return 2
    return int(bool(normalize))


class Context:
    """Owns a ``b200_ctx`` (weights + workspaces) on one CUDA device."""

    def __init__(self, device: torch.device | int | str = "cuda:0"):
        self.lib = _lib.load()
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.B200Error(f"pyannote_audio_b200 runs on CUDA (sm_90a) devices only, got '{device}'")
        if not torch.cuda.is_available():
            raise _lib.B200Error("no CUDA device is visible: pyannote_audio_b200 has no CPU fallback")
        self.device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
        torch.cuda.init()
        h = C.c_void_p()
        _lib.check(self.lib.b200_ctx_create(C.byref(h), self.device.index))
        self._h = h
        # PyanNet ("seg") and SSeRiouSS ("ssl") slots: the slots whose last load succeeded, and per slot the
        # (classes, activation) of the last head the library accepted.  A refused load keeps that entry: the library
        # checks a head before it releases the resident one, so it may go on running the previous head.
        self._loaded = set()
        self._heads = {}
        self._lstm_layers = {}    # slot -> BiLSTM layers of the head the library accepted last
        self._options = {}        # options set through set_option, by key
        self.emb_loaded = False
        self.emb_channels = 256   # trunk output channels of the loaded embedding model: 256 (ResNet34) or 1024
        self.emb_blocks = []      # (C_in, C_out, stride) of each block of the loaded trunk, in order
        self.xvec_loaded = False
        self.xvec_dimension = 512
        self.xvec_mfcc_loaded = False
        self.xvec_mfcc_dimension = 512
        # slot ("seg" | "emb" | "xvec" | "xvec_mfcc" | "ssl") -> stamp of the model whose weights are resident
        self.owners = {}
        # A/B knob for scripts (like B200_CONV_IMPL / B200_EMB_MAX_BATCH / B200_SEG_MAX_BATCH, which the library
        # reads itself): B200_OPTIONS="key=value,..."
        # is applied through b200_ctx_set_option, so unknown keys / bad values fail loudly
        import os

        for kv in filter(None, os.environ.get("B200_OPTIONS", "").split(",")):
            key, value = kv.split("=")
            self.set_option(key.strip(), int(value))

    def close(self):
        if getattr(self, "_h", None):
            self.lib.b200_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def seg_loaded(self) -> bool:
        return "seg" in self._loaded

    @property
    def ssl_loaded(self) -> bool:
        return "ssl" in self._loaded

    def set_option(self, key: str, value: int):
        _lib.check(self.lib.b200_ctx_set_option(self._h, key.encode(), int(value)))
        self._options[key] = int(value)

    @property
    def launch_count(self) -> int:
        return int(self.lib.b200_ctx_launch_count(self._h))

    def timer(self, name: str):
        """(accumulated device ms, units) of a profiled region ("trunk" | "seg"); needs set_option("profile", 1)."""
        ms, units = C.c_double(0.0), C.c_int64(0)
        _lib.check(self.lib.b200_ctx_timer(self._h, name.encode(), C.byref(ms), C.byref(units)))
        return float(ms.value), int(units.value)

    def _call(self, name: str, *args):
        """``b200_<name>(ctx, *args, stream)`` with this ctx's device selected and its current stream; a failure
        raises (ValueError, MemoryError or B200Error)."""
        with torch.cuda.device(self.device):
            _lib.check(getattr(self.lib, name)(self._h, *args, _stream(self.device)))

    # ---- weights ---------------------------------------------------------------------------------
    def load_segmentation(self, sd: Mapping[str, torch.Tensor], specifications=None):
        """PyanNet weights.  The head has ``classifier.weight``'s K rows (1 .. 32); its activation comes from
        ``specifications`` (sigmoid for binary / multi-label problems), log-softmax without them."""
        head = _head_of(sd, specifications)
        f = _state_dict_reader(sd)
        w = _lib.SegWeights()
        _fill_sincnet(w, sd, f)
        _fill_head(w, sd, f)
        self._load_head("seg", "b200_seg_load_head", w, head)

    def load_embedding(self, sd: Mapping[str, torch.Tensor]):
        f = _state_dict_reader(sd)

        def conv_bn(dst, conv, bn):
            dst.conv_weight = f(conv + ".weight")
            dst.bn_weight = f(bn + ".weight")
            dst.bn_bias = f(bn + ".bias")
            dst.bn_mean = f(bn + ".running_mean")
            dst.bn_var = f(bn + ".running_var")

        if "resnet.layer1.0.conv3.weight" in sd:
            return self._load_bottleneck(sd, f, conv_bn)
        w = _lib.EmbWeights()
        conv_bn(w.stem, "resnet.conv1", "resnet.bn1")
        bi, blocks = 0, []
        for li, n in enumerate((3, 4, 6, 3), start=1):
            for i in range(n):
                p = f"resnet.layer{li}.{i}"
                blocks.append((blocks[-1][1] if blocks else 32, 32 << (li - 1), 2 if i == 0 and li > 1 else 1))
                conv_bn(w.block_conv1[bi], p + ".conv1", p + ".bn1")
                conv_bn(w.block_conv2[bi], p + ".conv2", p + ".bn2")
                if p + ".shortcut.0.weight" in sd:
                    conv_bn(w.block_shortcut[bi], p + ".shortcut.0", p + ".shortcut.1")
                bi += 1
        w.seg1_weight = f("resnet.seg_1.weight")
        w.seg1_bias = f("resnet.seg_1.bias")
        self.owners.pop("emb", None)
        self.emb_loaded = False
        _lib.check(self.lib.b200_emb_load(self._h, C.byref(w)))
        self.emb_loaded, self.emb_channels, self.emb_blocks = True, 256, blocks

    def load_xvector(self, sd: Mapping[str, torch.Tensor]):
        """XVectorSincNet weights (models/embedding/xvector.py:205-252) into the ctx's own slot."""
        f = _state_dict_reader(sd)
        w = _lib.XvecWeights()
        _fill_sincnet(w, sd, f)
        dim = _fill_tdnn(w, sd, f, 60)
        self.owners.pop("xvec", None)
        self.xvec_loaded = False
        _lib.check(self.lib.b200_xvec_load(self._h, C.byref(w)))
        self.xvec_loaded, self.xvec_dimension = True, dim

    def load_xvector_mfcc(self, sd: Mapping[str, torch.Tensor]):
        """XVectorMFCC weights (models/embedding/xvector.py:42-89) into the ctx's own slot: the TDNN stack and Linear,
        and the MFCC buffers as loaded."""
        f = _state_dict_reader(sd)
        w = _lib.XvecMfccWeights()
        for field, key, shape in (("dct_mat", "mfcc.dct_mat", (128, 40)),
                                  ("window", "mfcc.MelSpectrogram.spectrogram.window", (400,)),
                                  ("mel_fb", "mfcc.MelSpectrogram.mel_scale.fb", (201, 128))):
            if tuple(sd[key].shape) != shape:
                raise ValueError(f"{key} has shape {tuple(sd[key].shape)}, expected {shape}")
            setattr(w, field, f(key))
        dim = _fill_tdnn(w, sd, f, 40)
        self.owners.pop("xvec_mfcc", None)
        self.xvec_mfcc_loaded = False
        _lib.check(self.lib.b200_xvec_mfcc_load(self._h, C.byref(w)))
        self.xvec_mfcc_loaded, self.xvec_mfcc_dimension = True, dim

    def load_sseriouss(self, sd: Mapping[str, torch.Tensor], specifications=None, wav2vec_layer: int = -1):
        """SSeRiouSS weights (models/segmentation/SSeRiouSS.py on WavLM Base) into the ctx's own slot.  ``sd`` uses
        the module's keys; the positional conv's weight norm is folded here (either spelling).  The LSTM reads the
        softmax(wav2vec_weights)-weighted average of the 12 layer outputs for ``wav2vec_layer`` < 0, else the output
        of layer ``wav2vec_layer`` (1 .. 12), and then only that many layers run."""
        head = _head_of(sd, specifications)
        f = _state_dict_reader(sd)
        w = _lib.SslWeights()
        fe, enc = "wav2vec.feature_extractor.conv_layers.", "wav2vec.encoder."
        w.conv0_weight = f(fe + "0.conv.weight")
        w.conv0_norm_weight = f(fe + "0.layer_norm.weight")
        w.conv0_norm_bias = f(fe + "0.layer_norm.bias")
        for i in range(6):
            w.conv_weight[i] = f(f"{fe}{i + 1}.conv.weight")
        w.proj_norm_weight = f(enc + "feature_projection.layer_norm.weight")
        w.proj_norm_bias = f(enc + "feature_projection.layer_norm.bias")
        w.proj_weight = f(enc + "feature_projection.projection.weight")
        w.proj_bias = f(enc + "feature_projection.projection.bias")
        tr = enc + "transformer."
        pos = fold_weight_norm(sd, tr + "pos_conv_embed.conv.")
        f.keep.append(pos)
        w.pos_conv_weight = _fp(pos)
        w.pos_conv_bias = f(tr + "pos_conv_embed.conv.bias")
        w.encoder_norm_weight = f(tr + "layer_norm.weight")
        w.encoder_norm_bias = f(tr + "layer_norm.bias")
        w.rel_attn_embed = f(tr + "layers.0.attention.rel_attn_embed.weight")
        buckets = wavlm_relative_buckets()
        f.keep.append(buckets)
        w.rel_bucket = C.cast(C.c_void_p(buckets.data_ptr()), C.POINTER(C.c_int32))
        if wav2vec_layer < 0:
            num_layers = SSL_LAYERS
            lw = torch.softmax(sd["wav2vec_weights"].detach().float().cpu(), dim=0).contiguous()
            f.keep.append(lw)
            w.layer_weights = _fp(lw)
        else:
            num_layers = int(wav2vec_layer)
            if not 1 <= num_layers <= SSL_LAYERS:
                raise ValueError(f"wav2vec_layer must be negative or between 1 and {SSL_LAYERS}, got {num_layers}")
        w.num_layers = num_layers
        names = {"in_proj_weight": "attention.attention.in_proj_weight",
                 "in_proj_bias": "attention.attention.in_proj_bias",
                 "out_proj_weight": "attention.attention.out_proj.weight",
                 "out_proj_bias": "attention.attention.out_proj.bias",
                 "gru_weight": "attention.gru_rel_pos_linear.weight", "gru_bias": "attention.gru_rel_pos_linear.bias",
                 "gru_const": "attention.gru_rel_pos_const",
                 "layer_norm_weight": "layer_norm.weight", "layer_norm_bias": "layer_norm.bias",
                 "ff1_weight": "feed_forward.intermediate_dense.weight",
                 "ff1_bias": "feed_forward.intermediate_dense.bias",
                 "ff2_weight": "feed_forward.output_dense.weight", "ff2_bias": "feed_forward.output_dense.bias",
                 "final_layer_norm_weight": "final_layer_norm.weight",
                 "final_layer_norm_bias": "final_layer_norm.bias"}
        for layer in range(num_layers):
            for field, key in names.items():
                setattr(w.layer[layer], field, f(f"{tr}layers.{layer}.{key}"))
        _fill_head(w, sd, f)
        self._load_head("ssl", "b200_ssl_load", w, head)

    def _load_head(self, slot: str, entry: str, w, head):
        """``entry``(ctx, w, classes, activation) into ``slot`` ("seg" | "ssl"), ``head`` = (classes, activation)."""
        self.owners.pop(slot, None)           # whoever uploaded before no longer owns the slot
        self._loaded.discard(slot)
        _lib.check(getattr(self.lib, entry)(self._h, C.byref(w), *head))
        self._loaded.add(slot)
        self._heads[slot] = head
        self._lstm_layers[slot] = int(w.lstm_layers)

    def _load_bottleneck(self, sd, f, conv_bn):
        """WeSpeakerResNet152 / 221 / 293 (Bottleneck blocks, resnet.py:148-212): the block counts come from the keys."""
        counts = []
        for li in range(1, 5):
            n = 0
            while f"resnet.layer{li}.{n}.conv1.weight" in sd:
                n += 1
            counts.append(n)
        total = sum(counts)
        arrays = [(_lib.ConvBN * total)() for _ in range(4)]
        conv1, conv2, conv3, shortcut = arrays
        bi, blocks = 0, []
        for li, n in enumerate(counts, start=1):
            for i in range(n):
                p = f"resnet.layer{li}.{i}"
                blocks.append((blocks[-1][1] if blocks else 32, 128 << (li - 1), 2 if i == 0 and li > 1 else 1))
                conv_bn(conv1[bi], p + ".conv1", p + ".bn1")
                conv_bn(conv2[bi], p + ".conv2", p + ".bn2")
                conv_bn(conv3[bi], p + ".conv3", p + ".bn3")
                if p + ".shortcut.0.weight" in sd:
                    conv_bn(shortcut[bi], p + ".shortcut.0", p + ".shortcut.1")
                bi += 1
        w = _lib.EmbBottleneckWeights()
        for li, n in enumerate(counts):
            w.num_blocks[li] = n
        conv_bn(w.stem, "resnet.conv1", "resnet.bn1")
        w.block_conv1, w.block_conv2, w.block_conv3, w.block_shortcut = arrays
        w.seg1_weight = f("resnet.seg_1.weight")
        w.seg1_bias = f("resnet.seg_1.bias")
        self.owners.pop("emb", None)
        self.emb_loaded = False
        _lib.check(self.lib.b200_emb_load_bottleneck(self._h, C.byref(w)))
        self.emb_loaded, self.emb_channels, self.emb_blocks = True, 1024, blocks

    # ---- helpers ---------------------------------------------------------------------------------
    def _check_waveform(self, wav: torch.Tensor):
        if wav.device != self.device or wav.dtype != torch.float32 or not wav.is_contiguous():
            raise ValueError(f"waveform must be a contiguous float32 tensor on {self.device}")

    def _chunks(self, wav: torch.Tensor, chunk_off, chunk_valid):
        self._check_waveform(wav)
        off = np.ascontiguousarray(chunk_off, dtype=np.int64)
        valid = np.ascontiguousarray(chunk_valid, dtype=np.int32)
        if off.shape != valid.shape or off.ndim != 1:
            raise ValueError("chunk_off / chunk_valid must be 1-D and of equal length")
        if len(off) and int((off + valid).max()) > wav.numel():
            raise ValueError("a chunk reads past the end of the waveform buffer")
        return off, valid

    def _utterances(self, wav: torch.Tensor, off, num_samples: int, min_samples: int, too_short: str):
        """Utterance i = wav[off[i] : off[i] + num_samples] -> (host int64 offsets, n, num_samples); ``too_short`` is
        the error message (formatted with num_samples) for utterances shorter than ``min_samples``."""
        self._check_waveform(wav)
        off = np.ascontiguousarray(off, dtype=np.int64).reshape(-1)
        n, num_samples = len(off), int(num_samples)
        if num_samples < min_samples:
            raise ValueError(too_short.format(num_samples))
        if n and (int(off.min()) < 0 or int(off.max()) + num_samples > wav.numel()):
            raise ValueError("an utterance reads outside the waveform buffer")
        return off, n, num_samples

    # ---- segmentation ----------------------------------------------------------------------------
    def _out(self, out: Optional[torch.Tensor], shape, dtype) -> torch.Tensor:
        """Caller-provided output (e.g. this rank's slice of a collective's buffer) or a fresh tensor."""
        if out is None:
            return torch.empty(shape, dtype=dtype, device=self.device)
        if tuple(out.shape) != tuple(shape) or out.dtype != dtype or out.device != self.device or \
                not out.is_contiguous():
            raise ValueError(f"`out` must be a contiguous {dtype} tensor of shape {tuple(shape)} on {self.device}")
        return out

    def seg_forward(self, wav, chunk_off, chunk_valid, return_logp=False, out: Optional[torch.Tensor] = None,
                    window: int = CHUNK, reduce_max: bool = False):
        """PyanNet on windows of ``window`` samples (>= 1261): window i = wav[off[i] : off[i] + window], of which the
        first valid[i] samples are real (zeros after); F = seg_num_frames(window), K the loaded head's classes.
        Log-softmax head -> classes (n, F) uint8 (+ log-probabilities (n, F, K)).  Sigmoid head -> scores (n, F, K)
        float32, or with ``reduce_max`` their per-frame maximum (n, F, 1) computed in the same kernel."""
        return self._head_forward("seg", wav, chunk_off, chunk_valid, return_logp, out, window, reduce_max)

    def ssl_forward(self, wav, chunk_off, chunk_valid, return_logp=False, out: Optional[torch.Tensor] = None,
                    window: int = CHUNK, reduce_max: bool = False):
        """SSeRiouSS on windows of ``window`` samples (>= 400), arguments and outputs as in seg_forward with
        F = ssl_num_frames(window) frames per window."""
        return self._head_forward("ssl", wav, chunk_off, chunk_valid, return_logp, out, window, reduce_max)

    # per slot: the window check, frames per window, the model's name in messages and its entry points' prefix
    _HEAD_SLOTS = {"seg": (check_seg_window, seg_num_frames, "segmentation", "b200_seg"),
                   "ssl": (check_ssl_window, ssl_num_frames, "SSeRiouSS", "b200_ssl")}

    def _head_forward(self, slot, wav, chunk_off, chunk_valid, return_logp, out, window, reduce_max):
        """seg_forward / ssl_forward on the head resident in ``slot``.  A slot the library never accepted a head for
        takes the log-softmax path, where the library reports the missing weights."""
        check_window, num_frames, name, prefix = self._HEAD_SLOTS[slot]
        check_window(window)
        window = int(window)
        off, valid = self._chunks(wav, chunk_off, chunk_valid)
        n = len(off)
        F = num_frames(window)
        K, activation = self._heads.get(slot, (CLASSES, SEG_LOGSOFTMAX))
        if activation == SEG_SIGMOID:
            if return_logp:
                raise ValueError(f"the loaded {name} head is a sigmoid head: it has scores, not log-probabilities")
            scores = self._out(out, (n, F, 1 if reduce_max else K), torch.float32)
            self._call(prefix + "_forward_scores", _ptr(wav), off.ctypes.data, valid.ctypes.data, n, window,
                       None if reduce_max else _ptr(scores), _ptr(scores) if reduce_max else None)
            return scores
        if reduce_max:
            raise ValueError("reduce_max needs a sigmoid segmentation head (use powerset_speech for a powerset head)")
        cls = self._out(out, (n, F), torch.uint8)
        logp = torch.empty((n, F, K), dtype=torch.float32, device=self.device) if return_logp else None
        self._call(prefix + "_forward_window", _ptr(wav), off.ctypes.data, valid.ctypes.data, n, window, _ptr(cls),
                   _ptr(logp))
        return (cls, logp) if return_logp else cls

    def sincnet_forward(self, wav, chunk_off, chunk_valid):
        off, valid = self._chunks(wav, chunk_off, chunk_valid)
        n = len(off)
        out = torch.empty((n, FRAMES, 60), dtype=torch.float32, device=self.device)
        self._call("b200_sincnet_forward", _ptr(wav), off.ctypes.data, valid.ctypes.data, n, _ptr(out))
        return out

    def ssl_features(self, wav, chunk_off, chunk_valid, window: int = CHUNK):
        """The loaded SSeRiouSS's WavLM Base front end alone, windows as in ssl_forward -> (n, F, 768) float32, the
        LSTM input of ssl_forward (the weighted layer average, or the output of layer wav2vec_layer)."""
        check_ssl_window(window)
        window = int(window)
        off, valid = self._chunks(wav, chunk_off, chunk_valid)
        n = len(off)
        out = torch.empty((n, ssl_num_frames(window), 768), dtype=torch.float32, device=self.device)
        self._call("b200_ssl_features", _ptr(wav), off.ctypes.data, valid.ctypes.data, n, window, _ptr(out))
        return out

    def seg_stages(self, wav, chunk_off, chunk_valid, window: int = CHUNK) -> dict:
        """The loaded PyanNet on windows as seg_forward runs them (same kernels, under the ctx's seg_*_impl options),
        returning every intermediate: "af_wav" (n, 2), "P0" (n, 80, pool0), "af0" (n, 80, 2), "P1" (n, 60, pool1),
        "af1", "P2" (n, 60, F), "af2", "x0" (n, F, 64), and the head's tensors as seg_head_stages returns them.  The
        affines are (scale, shift) pairs.  The windows must fit one sub-batch (ValueError otherwise)."""
        check_seg_window(window)
        window = int(window)
        off, valid = self._chunks(wav, chunk_off, chunk_valid)
        n = len(off)
        sinc_len = 1 + (window - 251) // 10
        pool0 = sinc_len // 3
        pool1 = (pool0 - 4) // 3
        pool2 = (pool1 - 4) // 3
        f32 = dict(dtype=torch.float32, device=self.device)
        out = {"af_wav": torch.empty((n, 2), **f32), "P0": torch.empty((n, 80, pool0), **f32),
               "af0": torch.empty((n, 80, 2), **f32), "P1": torch.empty((n, 60, pool1), **f32),
               "af1": torch.empty((n, 60, 2), **f32), "P2": torch.empty((n, 60, pool2), **f32),
               "af2": torch.empty((n, 60, 2), **f32), "x0": torch.empty((n, pool2, 64), **f32)}
        cap = self._head_capture("seg", n, pool2, out)
        for name in ("af_wav", "P0", "af0", "P1", "af1", "P2", "af2", "x0"):
            setattr(cap, name, out[name].data_ptr())
        self._call("b200_seg_stages", _ptr(wav), off.ctypes.data, valid.ctypes.data, n, window, C.byref(cap))
        return out

    def seg_head_stages(self, model: str, x0: torch.Tensor) -> dict:
        """The segmentation head of the loaded ``model`` ("seg": PyanNet, x0 (n, T, 64); "ssl": SSeRiouSS, x0
        (n, T, 768)) on any input, T >= 1, as the forward runs it, returning "gx" (per LSTM layer (n, T, 1024): input
        projection plus both biases, column dir * 512 + unit * 4 + gate), "y" (per layer (n, T, 256) float32 under
        seg_gemm_impl 0, else a (hi, lo) pair of float16 tensors), "z1" (n, T, 128) likewise, "z2" (n, T, 128) and the
        classifier's outputs: "cls" (n, T) uint8 and "logp" (n, T, K), or "scores" (n, T, K) and "max_scores" (n, T)."""
        k0 = {"seg": 64, "ssl": 768}.get(model)
        if k0 is None:
            raise ValueError(f"model must be 'seg' (PyanNet) or 'ssl' (SSeRiouSS), got {model!r}")
        if x0.dim() != 3 or x0.shape[2] != k0 or x0.shape[1] < 1:
            raise ValueError(f"x0 must have shape (n, T >= 1, {k0}), got {tuple(x0.shape)}")
        x0 = x0.to(device=self.device, dtype=torch.float32).contiguous()
        n, T = int(x0.shape[0]), int(x0.shape[1])
        out = {}
        cap = self._head_capture(model, n, T, out)
        self._call("b200_seg_head_stages", 0 if model == "seg" else 1, _ptr(x0), n, T, C.byref(cap))
        return out

    def _head_capture(self, slot: str, n: int, T: int, out: dict) -> "_lib.SegCapture":
        """A capture of every head tensor of ``slot``'s loaded head for n sequences of T frames, allocated into
        ``out``."""
        K, activation = self._heads.get(slot, (CLASSES, SEG_LOGSOFTMAX))
        layers = self._lstm_layers.get(slot, 4)
        split = self._options.get("seg_gemm_impl", 1) != 0
        f32 = dict(dtype=torch.float32, device=self.device)
        f16 = dict(dtype=torch.float16, device=self.device)
        cap = _lib.SegCapture()
        out["gx"], out["y"] = [], []
        for layer in range(layers):
            out["gx"].append(torch.empty((n, T, 1024), **f32))
            cap.gx[layer] = out["gx"][-1].data_ptr()
            if split:
                hi, lo = torch.empty((n, T, 256), **f16), torch.empty((n, T, 256), **f16)
                cap.y_hi[layer], cap.y_lo[layer] = hi.data_ptr(), lo.data_ptr()
                out["y"].append((hi, lo))
            else:
                out["y"].append(torch.empty((n, T, 256), **f32))
                cap.y[layer] = out["y"][-1].data_ptr()
        if split:
            out["z1"] = (torch.empty((n, T, 128), **f16), torch.empty((n, T, 128), **f16))
            cap.z1_hi, cap.z1_lo = out["z1"][0].data_ptr(), out["z1"][1].data_ptr()
        else:
            out["z1"] = torch.empty((n, T, 128), **f32)
            cap.z1 = out["z1"].data_ptr()
        out["z2"] = torch.empty((n, T, 128), **f32)
        cap.z2 = out["z2"].data_ptr()
        if activation == SEG_SIGMOID:
            out["scores"], out["max_scores"] = torch.empty((n, T, K), **f32), torch.empty((n, T), **f32)
            cap.scores, cap.max_scores = out["scores"].data_ptr(), out["max_scores"].data_ptr()
        else:
            out["cls"], out["logp"] = torch.empty((n, T), dtype=torch.uint8, device=self.device), \
                torch.empty((n, T, K), **f32)
            cap.cls, cap.logp = out["cls"].data_ptr(), out["logp"].data_ptr()
        return cap

    def powerset_to_multilabel(self, cls: torch.Tensor, num_speakers: int = SPEAKERS, max_per_frame: int = 2):
        """(…) uint8 powerset classes of ``num_speakers`` speakers with at most ``max_per_frame`` per frame ->
        (…, num_speakers) uint8 multilabel (Powerset.to_multilabel, hard)."""
        k = len(powerset_mapping(num_speakers, max_per_frame))
        cls = cls.contiguous()
        out = torch.empty(tuple(cls.shape) + (int(num_speakers),), dtype=torch.uint8, device=self.device)
        self._call("b200_powerset_to_multilabel_generic", _ptr(cls), cls.numel(), k, int(num_speakers),
                   int(max_per_frame), _ptr(out))
        return out

    # ---- embeddings ------------------------------------------------------------------------------
    def emb_forward(self, wav, chunk_off, chunk_valid, masks: torch.Tensor, out: Optional[torch.Tensor] = None,
                    peers: Optional[Sequence[int]] = None):
        """``peers``: raw device addresses of this rank's (n,3,256) float32 slot inside other GPUs' gather buffers
        (peer-mapped memory); the final GEMM's epilogue then pushes the embeddings there (fused all-gather)."""
        off, valid = self._chunks(wav, chunk_off, chunk_valid)
        n = len(off)
        if tuple(masks.shape) != (n, SPEAKERS, FRAMES) or masks.dtype != torch.uint8 or not masks.is_contiguous():
            raise ValueError(f"masks must be a contiguous uint8 tensor of shape ({n}, 3, 589)")
        emb = self._out(out, (n, SPEAKERS, EMB_DIM), torch.float32)
        args = (_ptr(wav), off.ctypes.data, valid.ctypes.data, n, _ptr(masks), _ptr(emb))
        if peers:
            arr = (C.c_void_p * len(peers))(*[C.c_void_p(int(a)) for a in peers])
            self._call("b200_emb_forward_push", *args, arr, len(peers))
        else:
            self._call("b200_emb_forward", *args)
        return emb

    def _pool_weights(self, weights: Optional[torch.Tensor], n: int):
        """(n, Tw) or (n, S, Tw) fp32 pooling weights on this device -> (tensor or None, S, Tw)."""
        if weights is None:
            return None, 1, 0
        if weights.dim() == 2:
            weights = weights.unsqueeze(1)
        if weights.dim() != 3 or weights.shape[0] != n or weights.shape[1] < 1 or weights.shape[2] < 1:
            raise ValueError(f"weights must have shape ({n}, frames) or ({n}, speakers, frames), got "
                             f"{tuple(weights.shape)}")
        weights = weights.to(device=self.device, dtype=torch.float32).contiguous()
        return weights, int(weights.shape[1]), int(weights.shape[2])

    def emb_forward_utt(self, wav, off, num_samples: int, weights: Optional[torch.Tensor] = None,
                        out: Optional[torch.Tensor] = None):
        """Embeddings of utterances of one length: utterance i = wav[off[i] : off[i] + num_samples] (any length >= 400
        samples).  ``weights``: None or (n, Tw) / (n, S, Tw) soft pooling weights (any Tw, interpolated onto the
        trunk frames) -> (n, max(S, 1), 256) float32."""
        off, n, num_samples = self._utterances(wav, off, num_samples, 400,
                                               "utterances of {} samples are shorter than one 400-sample fbank frame")
        w, S, Tw = self._pool_weights(weights, n)
        emb = self._out(out, (n, S, EMB_DIM), torch.float32)
        self._call("b200_emb_forward_utt", _ptr(wav), off.ctypes.data, num_samples, n, _ptr(w),
                   S if w is not None else 0, Tw, _ptr(emb))
        return emb

    def xvec_forward(self, wav, off, num_samples: int, weights: Optional[torch.Tensor] = None,
                     out: Optional[torch.Tensor] = None):
        """XVectorSincNet embeddings of utterances of one length: utterance i = wav[off[i] : off[i] + num_samples]
        (>= 4771 samples).  ``weights``: None or (n, Tw) / (n, S, Tw) pooling weights of any real values (any Tw,
        nearest-interpolated onto the TDNN frames) -> (n, max(S, 1), dimension) float32."""
        return self._xvec_run("b200_xvec_forward", "XVectorSincNet", XVEC_MIN_SAMPLES, self.xvec_dimension, wav, off,
                              num_samples, weights, out)

    def xvec_mfcc_forward(self, wav, off, num_samples: int, weights: Optional[torch.Tensor] = None,
                          out: Optional[torch.Tensor] = None):
        """XVectorMFCC embeddings, as xvec_forward (>= 2800 samples)."""
        return self._xvec_run("b200_xvec_mfcc_forward", "XVectorMFCC", XVEC_MFCC_MIN_SAMPLES, self.xvec_mfcc_dimension,
                              wav, off, num_samples, weights, out)

    def _xvec_run(self, entry: str, name: str, min_samples: int, dim: int, wav, off, num_samples: int, weights, out):
        off, n, num_samples = self._utterances(wav, off, num_samples, min_samples,
                                               f"{name} needs at least {min_samples} samples, got {{}}")
        w, S, Tw = self._pool_weights(weights, n)
        emb = self._out(out, (n, S, dim), torch.float32)
        self._call(entry, _ptr(wav), off.ctypes.data, num_samples, n, _ptr(w), S if w is not None else 0, Tw,
                   _ptr(emb))
        return emb

    def mfcc_features(self, wav, off, num_samples: int) -> torch.Tensor:
        """The loaded XVectorMFCC's front end alone on utterances of one length (> 200 samples) -> (n, frames, 40)
        float32 MFCC, frames = 1 + num_samples // 200."""
        off, n, num_samples = self._utterances(wav, off, num_samples, 201,
                                               "the MFCC front end needs more than 200 samples, got {}")
        out = torch.empty((n, 1 + num_samples // 200, 40), dtype=torch.float32, device=self.device)
        self._call("b200_xvec_mfcc_features", _ptr(wav), off.ctypes.data, num_samples, n, _ptr(out))
        return out

    def emb_forward_embedding(self, frames: torch.Tensor, weights: Optional[torch.Tensor] = None):
        """ResNet.forward_embedding on frames (B, C, 10, T) -> (B, max(S, 1), 256) float32, C the trunk channels of
        the loaded model (256 for ResNet34, 1024 for the bottleneck ResNets); weights as in emb_forward_utt."""
        c = self.emb_channels
        if frames.dim() != 4 or tuple(frames.shape[1:3]) != (c, 10) or frames.shape[3] < 1:
            raise ValueError(f"frames must have shape (batch, {c}, 10, frames), got {tuple(frames.shape)}")
        frames = frames.to(device=self.device, dtype=torch.float32).contiguous()
        B, T = int(frames.shape[0]), int(frames.shape[3])
        w, S, Tw = self._pool_weights(weights, B)
        emb = torch.empty((B, S, EMB_DIM), dtype=torch.float32, device=self.device)
        self._call("b200_emb_forward_embedding", _ptr(frames), B, T, _ptr(w), S if w is not None else 0, Tw, _ptr(emb))
        return emb

    def push(self, src: torch.Tensor, peers: Sequence[int]):
        """P2P copy of a contiguous device tensor to raw peer addresses (same layout), on the current stream."""
        if not peers or src.numel() == 0:
            return
        arr = (C.c_void_p * len(peers))(*[C.c_void_p(int(a)) for a in peers])
        self._call("b200_push", _ptr(src), src.numel() * src.element_size(), arr, len(peers))

    def emb_fbank(self, wav, chunk_off, chunk_valid):
        off, valid = self._chunks(wav, chunk_off, chunk_valid)
        n = len(off)
        fb = torch.empty((n, 998, 80), dtype=torch.float32, device=self.device)
        self._call("b200_emb_fbank", _ptr(wav), off.ctypes.data, valid.ctypes.data, n, _ptr(fb))
        return fb

    def emb_trunk(self, fbank: torch.Tensor):
        n = fbank.shape[0]
        fbank = fbank.contiguous()
        out = torch.empty((n, self.emb_channels, 10, 125), dtype=torch.float32, device=self.device)
        self._call("b200_emb_trunk", _ptr(fbank), n, _ptr(out))
        return out

    def emb_trunk_stage(self, stage: int, x: torch.Tensor, fmean: Optional[torch.Tensor] = None):
        """One stage of the loaded trunk on B segments of width W, as emb_trunk runs it under the ctx's conv_impl.
        Stage 0 is the stem: fp32 fbank (B, W, 80) minus ``fmean`` (B, 80; zeros when None) -> NHWC float16
        (B, 80, W, 32).  Stage k >= 1 is block k - 1: NHWC float16 (B, H, W, C_in) -> (B, H', W', C_out)."""
        if not 0 <= stage <= len(self.emb_blocks):
            raise ValueError(f"stage {stage}: the trunk has stages 0 .. {len(self.emb_blocks)}")
        if x.dim() != (3 if stage == 0 else 4):
            raise ValueError(f"stage {stage} takes a {3 if stage == 0 else 4}-d tensor, got shape {tuple(x.shape)}")
        B, W = x.shape[0], x.shape[-2 if stage else 1]
        if stage == 0:
            shape, dtype, (H, C_out, s) = (B, W, 80), torch.float32, (80, 32, 1)
            fmean = torch.zeros((B, 80)) if fmean is None else fmean
            if tuple(fmean.shape) != (B, 80):
                raise ValueError(f"fmean has shape {tuple(fmean.shape)}, expected {(B, 80)}")
            fmean = fmean.to(device=self.device, dtype=torch.float32).contiguous()
        else:
            C_in, C_out, s = self.emb_blocks[stage - 1]
            H = 80 >> sum(b[2] == 2 for b in self.emb_blocks[:stage - 1])
            shape, dtype = (B, H, W, C_in), torch.float16
        if tuple(x.shape) != shape or x.dtype != dtype:
            raise ValueError(f"stage {stage} takes {dtype} of shape {shape}, got {x.dtype} {tuple(x.shape)}")
        x = x.to(device=self.device).contiguous()
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        out = torch.empty((B, Ho, Wo, C_out), dtype=torch.float16, device=self.device)
        self._call("b200_emb_trunk_stage", int(stage), _ptr(x), _ptr(fmean if stage == 0 else None), B, W, _ptr(out))
        return out

    def stats_pool(self, seq: torch.Tensor, weights: Optional[torch.Tensor] = None):
        B, F, T = seq.shape
        seq = seq.contiguous().float()
        squeeze = False
        if weights is None:
            S, Tw = 1, T
            squeeze = True
        else:
            if weights.dim() == 2:
                weights = weights.unsqueeze(1)
                squeeze = True
            weights = weights.contiguous().float()
            S, Tw = weights.shape[1], weights.shape[2]
        out = torch.empty((B, S, 2 * F), dtype=torch.float32, device=self.device)
        self._call("b200_stats_pool", _ptr(seq), _ptr(weights), _ptr(out), B, F, T, S, Tw)
        return out.squeeze(1) if squeeze else out

    # ---- overlap-add / reconstruction ----------------------------------------------------------------
    def start_frames(self, start_frame) -> torch.Tensor:
        """Device copy of the per-chunk start frames (cached per distinct array)."""
        if isinstance(start_frame, torch.Tensor):
            return start_frame
        sf = np.ascontiguousarray(start_frame, dtype=np.int32)
        if len(sf) > 1 and not bool((np.diff(sf) >= 0).all()):
            raise ValueError("start_frame must be non-decreasing")
        key = (len(sf), int(sf[0]) if len(sf) else 0, int(sf[-1]) if len(sf) else 0)
        cache = self.__dict__.setdefault("_sf_cache", {})
        hit = cache.get(key)
        if hit is None or not np.array_equal(hit[0], sf):
            hit = (sf, torch.from_numpy(sf).to(self.device))
            if len(cache) > 64:
                cache.clear()
            cache[key] = hit
        return hit[1]

    def speaker_count(self, seg: torch.Tensor, start_frame, num_frames: int):
        sf = self.start_frames(start_frame)
        count = torch.empty((num_frames,), dtype=torch.uint8, device=self.device)
        self._call("b200_speaker_count", _ptr(seg), _ptr(sf), sf.numel(), num_frames, _ptr(count))
        return count

    def reconstruct(self, seg: torch.Tensor, hard_clusters, start_frame, num_frames: int, count: torch.Tensor,
                    num_clusters_out: int):
        sf = self.start_frames(start_frame)
        if not isinstance(hard_clusters, torch.Tensor):
            hard_clusters = torch.from_numpy(np.ascontiguousarray(hard_clusters, dtype=np.int8)).to(self.device)
        hc = hard_clusters.to(torch.int8).contiguous()
        out = torch.empty((num_frames, num_clusters_out), dtype=torch.uint8, device=self.device)
        self._call("b200_reconstruct", _ptr(seg), _ptr(hc), _ptr(sf), sf.numel(), num_frames, _ptr(count),
                   num_clusters_out, _ptr(out))
        return out

    def frame_transitions(self, discrete: torch.Tensor, cap: int = 4096):
        """discrete (F, K) u8 on the device -> sorted flat event indices k * (F + 1) + f of onsets and offsets
        (host int64 arrays).  One kernel + one 32 KB D2H instead of shipping and scanning the whole matrix."""
        return self.frame_transitions_many([discrete], cap)[0]

    def frame_transitions_many(self, matrices: Sequence[torch.Tensor], cap: int = 4096):
        """frame_transitions of several (F_i, K_i) matrices with ONE device -> host copy (and one synchronisation)
        for all of them: every matrix gets a row [n_on, n_off, on[cap], off[cap]] of one int32 buffer.  A row whose
        event count exceeds ``cap`` is redone alone with a larger buffer."""
        m = len(matrices)
        self.last_transfer_bytes = 0
        if m == 0:
            return []
        mats = [d.contiguous() for d in matrices]
        buf = torch.empty((m, 2 + 2 * cap), dtype=torch.int32, device=self.device)
        for i, d in enumerate(mats):
            self._call("b200_frame_transitions", _ptr(d), int(d.shape[0]), int(d.shape[1]), cap, _ptr(buf[i]))
        host = buf.cpu().numpy()
        self.last_transfer_bytes = host.nbytes
        out = []
        for i, d in enumerate(mats):
            row, c = host[i], cap
            n_on, n_off = int(row[0]), int(row[1])
            while max(n_on, n_off) > c:                       # rare: more events than slots -> this matrix again
                c = 1 << int(max(n_on, n_off) - 1).bit_length()
                big = torch.empty((2 + 2 * c,), dtype=torch.int32, device=self.device)
                self._call("b200_frame_transitions", _ptr(d), int(d.shape[0]), int(d.shape[1]), c, _ptr(big))
                row = big.cpu().numpy()
                self.last_transfer_bytes += row.nbytes
                n_on, n_off = int(row[0]), int(row[1])
            on = np.sort(row[2: 2 + n_on].astype(np.int64))
            off = np.sort(row[2 + c: 2 + c + n_off].astype(np.int64))
            out.append((on, off))
        return out

    # ---- audio ingest ------------------------------------------------------------------------------
    def audio_ingest(self, pcm: torch.Tensor, sample_rate: int, target_rate: Optional[int] = None,
                     channel: Optional[int] = None, downmix: bool = True, out: Optional[torch.Tensor] = None):
        """Raw decoded audio on the device -> float32 mono waveform (frames_out,) at ``target_rate``.

        ``pcm``: int16 (frames, channels) interleaved PCM, or float32 (channels, frames) like the reference's
        in-memory files.  ``channel`` selects one channel, otherwise channels are averaged (mono="downmix").
        (core/io.py:223-265: downmix, then torchaudio.functional.resample.)"""
        if pcm.device != self.device or not pcm.is_contiguous() or pcm.dim() != 2:
            raise ValueError(f"pcm must be a contiguous 2-D tensor on {self.device}")
        if pcm.dtype == torch.int16:
            fmt, (frames, channels) = 0, pcm.shape
        elif pcm.dtype == torch.float32:
            fmt, (channels, frames) = 1, pcm.shape
        else:
            raise ValueError("pcm must be int16 (frames, channels) or float32 (channels, frames)")
        if channel is None and not downmix and channels > 1:
            raise ValueError("multi-channel audio needs `channel` or downmix=True")
        target_rate = int(target_rate or sample_rate)
        n = int(self.lib.b200_audio_num_frames(int(frames), int(sample_rate), target_rate))
        if out is None:
            out = torch.empty((n,), dtype=torch.float32, device=self.device)
        elif out.dtype != torch.float32 or out.device != self.device or not out.is_contiguous() or out.numel() < n:
            raise ValueError(f"`out` must be a contiguous float32 tensor with at least {n} elements on {self.device}")
        self._call("b200_audio_ingest", _ptr(pcm), fmt, int(channels), int(frames), int(sample_rate), target_rate,
                   -1 if channel is None else int(channel), _ptr(out), out.numel())
        return out[:n]

    # ---- generic overlap-add (Inference.aggregate) ---------------------------------------------------
    def _window(self, key, build):
        cache = self.__dict__.setdefault("_win_cache", {})
        if key not in cache:
            cache[key] = torch.from_numpy(np.ascontiguousarray(build(), dtype=np.float64)).to(self.device)
        return cache[key]

    def aggregate(self, scores: torch.Tensor, start_frame, num_frames: int, hamming: bool = False,
                  warm_up=(0.0, 0.0), chunk_duration: float = 10.0, epsilon: float = 1e-12,
                  missing: float = float("nan"), skip_average: bool = False) -> torch.Tensor:
        """scores (C, F, K) float32 device (NaN = missing; any F frames per chunk) -> (num_frames, K) float32 device,
        bit-identical to Inference.aggregate's numpy arithmetic (core/inference.py:498-620)."""
        if scores.dtype != torch.float32 or scores.device != self.device or scores.dim() != 3 or \
                scores.shape[1] < 1:
            raise ValueError(f"scores must be a float32 (chunks, frames, classes) tensor on {self.device}")
        scores = scores.contiguous()
        F = int(scores.shape[1])
        sf = self.start_frames(start_frame)
        ham = self._window(("hamming", F), lambda: np.hamming(F)) if hamming else None
        wl = round(warm_up[0] / chunk_duration * F)
        wr = round(warm_up[1] / chunk_duration * F)
        warm = None
        if wl or wr:
            def build():
                w = np.ones(F)
                w[:wl] = epsilon
                w[F - wr:] = epsilon
                return w
            warm = self._window(("warm", F, wl, wr, epsilon), build)
        out = torch.empty((num_frames, scores.shape[2]), dtype=torch.float32, device=self.device)
        self._call("b200_aggregate_window", _ptr(scores), _ptr(sf), sf.numel(), int(num_frames), F,
                   int(scores.shape[2]), _ptr(ham), _ptr(warm), int(skip_average), float(missing),
                   float(np.float32(epsilon)), _ptr(out))
        return out

    def powerset_speech(self, cls: torch.Tensor, num_speakers: int = SPEAKERS, max_per_frame: int = 2) -> torch.Tensor:
        """(…) uint8 powerset classes -> (…, 1) float32 speech indicator (max over the speakers of the multilabel)."""
        k = len(powerset_mapping(num_speakers, max_per_frame))
        cls = cls.contiguous()
        out = torch.empty(tuple(cls.shape) + (1,), dtype=torch.float32, device=self.device)
        self._call("b200_powerset_speech_generic", _ptr(cls), cls.numel(), k, int(num_speakers), int(max_per_frame),
                   _ptr(out))
        return out

    def clean_frames(self, seg: torch.Tensor):
        n = seg.shape[0]
        clean = torch.empty((n, SPEAKERS), dtype=torch.int32, device=self.device)
        active = torch.empty((n, SPEAKERS), dtype=torch.uint8, device=self.device)
        self._call("b200_clean_frames", _ptr(seg), n, _ptr(clean), _ptr(active))
        return clean, active

    # ---- clustering (fp64) -------------------------------------------------------------------------------
    def plda_transform(self, x: torch.Tensor, mean1, mean2, lda, mu, trT) -> torch.Tensor:
        """PLDA.__call__ on the device: x (n, Din) float64 -> (n, L) float64 (core/plda.py:50-63)."""
        x, lda, trT = x.contiguous(), lda.contiguous(), trT.contiguous()
        n, din = x.shape
        dout, L = trT.shape
        fea = torch.empty((n, L), dtype=torch.float64, device=self.device)
        self._call("b200_plda_transform", _ptr(x), n, din, dout, L, _ptr(mean1), _ptr(mean2), _ptr(lda), _ptr(mu),
                   _ptr(trT), _ptr(fea))
        return fea

    def weighted_centroids(self, q: torch.Tensor, kept: torch.Tensor, train: torch.Tensor) -> torch.Tensor:
        """(W.T @ train) / W.sum(0).T with W = q[:, kept] (clustering.py:620-621): q (n,S), train (n,dim) float64."""
        q, train = q.contiguous(), train.contiguous()
        kept = kept.to(device=self.device, dtype=torch.int32).contiguous()
        out = torch.empty((kept.numel(), train.shape[1]), dtype=torch.float64, device=self.device)
        self._call("b200_weighted_centroids", _ptr(q), q.shape[0], q.shape[1], _ptr(kept), kept.numel(), _ptr(train),
                   train.shape[1], _ptr(out))
        return out

    def _linkage_check(self, name: str, *args):
        """``_call`` of a linkage entry point.  A file above 32 768 observations allocates its packed distances
        outside torch's caching allocator, so memory torch holds cached (e.g. from the segmentation and embedding of
        that same file) cannot serve it: on an allocation failure the cache is returned to the device and the call
        made once more."""
        try:
            self._call(name, *args)
        except MemoryError:
            torch.cuda.empty_cache()
            self._call(name, *args)

    def linkage_centroid(self, x: torch.Tensor, normalize=True) -> torch.Tensor:
        """x (n, dim) float64 on device -> Z (n-1, 4) float64 on device (scipy linkage format)."""
        n, dim = x.shape
        x = x.contiguous()
        Z = torch.empty((n - 1, 4), dtype=torch.float64, device=self.device)
        self._linkage_check("b200_linkage_centroid", _ptr(x), n, dim, _norm_mode(normalize), _ptr(Z))
        return Z

    def linkage_centroid_batched(self, x: torch.Tensor, row_offsets, normalize=True) -> torch.Tensor:
        """x (sum n_f, dim) f64; row_offsets host int array (F+1,) -> concatenated Z ((sum max(n_f-1,0)), 4) f64."""
        x = x.contiguous()
        ro = np.ascontiguousarray(row_offsets, dtype=np.int32)
        nz = int(np.maximum(np.diff(ro) - 1, 0).sum())
        Z = torch.empty((nz, 4), dtype=torch.float64, device=self.device)
        self._linkage_check("b200_linkage_centroid_batched", _ptr(x), ro.ctypes.data, len(ro) - 1, x.shape[1],
                            _norm_mode(normalize), _ptr(Z))
        return Z

    def cdist_cosine(self, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        a, b = a.contiguous(), b.contiguous()
        m, dim = a.shape
        k = b.shape[0]
        d = torch.empty((m, k), dtype=torch.float64, device=self.device)
        self._call("b200_cdist_cosine", _ptr(a), m, _ptr(b), k, dim, _ptr(d))
        return d

    def vbx(self, fea: torch.Tensor, phi: torch.Tensor, gamma0: torch.Tensor, Fa: float, Fb: float,
            max_iters: int = 20, epsilon: float = 1e-4):
        fea, phi = fea.contiguous(), phi.contiguous()
        gamma = gamma0.contiguous().clone()
        n, D = fea.shape
        S = gamma.shape[1]
        pi = torch.empty((S,), dtype=torch.float64, device=self.device)
        iters = C.c_int32(0)
        self._call("b200_vbx", _ptr(fea), _ptr(phi), n, D, S, C.c_double(Fa), C.c_double(Fb), max_iters,
                   C.c_double(epsilon), _ptr(gamma), _ptr(pi), C.byref(iters))
        return gamma, pi, int(iters.value)

    def vbx_batched(self, fea: torch.Tensor, phi: torch.Tensor, gamma0: torch.Tensor, n, S, Fa: float, Fb: float,
                    max_iters: int = 20, epsilon: float = 1e-4, want_iters: bool = False):
        """fea (sum n_f, D); gamma0 flat concatenation of the per-problem (n_f, S_f) initial responsibilities."""
        fea, phi = fea.contiguous(), phi.contiguous()
        gamma = gamma0.contiguous().clone()
        n = np.ascontiguousarray(n, dtype=np.int32)
        S = np.ascontiguousarray(S, dtype=np.int32)
        pi = torch.empty((int(S.sum()),), dtype=torch.float64, device=self.device)
        iters = np.zeros(len(n), dtype=np.int32)
        self._call("b200_vbx_batched", _ptr(fea), _ptr(phi), n.ctypes.data, S.ctypes.data, len(n), fea.shape[1],
                   C.c_double(Fa), C.c_double(Fb), max_iters, C.c_double(epsilon), _ptr(gamma), _ptr(pi),
                   iters.ctypes.data if want_iters else None)
        return gamma, pi, iters

    def assign(self, soft: torch.Tensor, constrained: bool = True) -> torch.Tensor:
        soft = soft.contiguous()
        c, s, k = soft.shape
        assert s == SPEAKERS
        hard = torch.empty((c, s), dtype=torch.int8, device=self.device)
        self._call("b200_assign", _ptr(soft), c, k, int(constrained), _ptr(hard))
        return hard


def fcluster_distance(Z: np.ndarray, t: float) -> np.ndarray:
    """Host tree cut, 1-based labels like scipy.cluster.hierarchy.fcluster(Z, t, 'distance')."""
    Z = np.ascontiguousarray(Z, dtype=np.float64)
    n = Z.shape[0] + 1
    T = np.zeros(n, dtype=np.int32)
    _lib.check(_lib.load().b200_fcluster_distance(Z.ctypes.data, n, C.c_double(float(t)), T.ctypes.data))
    return T


def linkage_bytes(row_offsets, dim: int) -> int:
    """Device bytes ``linkage_centroid_batched`` needs for these problems (host only, no device): the workspace it grows
    to plus the per-call packed distances of its largest problem above 32 768 observations."""
    ro = np.ascontiguousarray(row_offsets, dtype=np.int32)
    nbytes = int(_lib.load().b200_linkage_bytes(ro.ctypes.data, len(ro) - 1, int(dim)))
    if nbytes <= 0:
        _lib.check(nbytes)
    return nbytes
