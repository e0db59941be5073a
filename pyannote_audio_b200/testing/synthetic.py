"""Deterministic synthetic weights, PLDA and audio for parity tests and benchmarks.

No pretrained community-1 checkpoint exists offline, so every test/bench uses seeded random weights
with the *reference's state-dict key names and shapes* (real checkpoints drop in unchanged):

* segmentation: ``PyanNet`` (SincNet + 4-layer BiLSTM(128) + 2xLinear(128) + Linear(7));
  keys as in /root/reference/src/pyannote/audio/models/segmentation/PyanNet.py:92-161 and
  models/blocks/sincnet.py:41-79 (module tree: tutorials/training_a_model.ipynb:1001-1016)
* embedding: ``WeSpeakerResNet34``; keys as in models/embedding/wespeaker/resnet.py:233-252; the bottleneck
  ``WeSpeakerResNet152`` / ``221`` / ``293`` (resnet.py:148-212) with ``make_bottleneck_state_dict``
* x-vector: ``XVectorSincNet`` with ``make_xvector_state_dict``; keys as in models/embedding/xvector.py:205-252
* x-vector on MFCC: ``XVectorMFCC`` with ``make_xvector_mfcc_state_dict``; keys as in models/embedding/xvector.py:42-89
* PLDA: ``xvec_transform.npz{mean1,mean2,lda}`` + ``plda.npz{mu,tr,psi}`` (utils/vbx.py:195-199)

Audio: a synthetic multi-speaker "conversation" (harmonic sources, 3-6 Hz amplitude modulation,
Markov turn-taking with some overlap, -30 dB noise floor), float32 mono 16 kHz in [-1, 1].
"""

from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch

SAMPLE_RATE = 16000

# ----------------------------------------------------------------------------------------
# segmentation state dict
# ----------------------------------------------------------------------------------------


def _uniform(gen, shape, bound):
    return (torch.rand(shape, generator=gen, dtype=torch.float32) * 2 - 1) * bound


from ..models import _mel_sinc_init, sinc_buffers  # noqa: E402,F401  (ParamSincFB default initialisation)


def make_segmentation_state_dict(seed: int = 0, lstm_layers: int = 4, num_classes: int = 7,
                                 logit_scale: float = 6.0, ih_gain: float = 4.0, hh_gain: float = 1.5,
                                 lin_gain: float = 3.0,
                                 fitted_classifier: bool = True) -> "OrderedDict[str, torch.Tensor]":
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    sd["sincnet.wav_norm1d.weight"] = 1.0 + 0.1 * torch.randn(1, generator=g)
    sd["sincnet.wav_norm1d.bias"] = 0.05 * torch.randn(1, generator=g)
    low, band = _mel_sinc_init()
    # jitter the learnable cut-offs a little so they are not the textbook initialisation
    sd["sincnet.conv1d.0.filterbank.low_hz_"] = low * (1.0 + 0.05 * torch.randn(low.shape, generator=g))
    sd["sincnet.conv1d.0.filterbank.band_hz_"] = band * (1.0 + 0.05 * torch.randn(band.shape, generator=g))
    window_, n_ = sinc_buffers()
    sd["sincnet.conv1d.0.filterbank.window_"] = window_
    sd["sincnet.conv1d.0.filterbank.n_"] = n_
    for i, (cin, cout) in zip((1, 2), ((80, 60), (60, 60))):
        bound = 1.0 / math.sqrt(cin * 5)
        sd[f"sincnet.conv1d.{i}.weight"] = _uniform(g, (cout, cin, 5), bound)
        sd[f"sincnet.conv1d.{i}.bias"] = _uniform(g, (cout,), bound)
    for i, c in enumerate((80, 60, 60)):
        sd[f"sincnet.norm1d.{i}.weight"] = 1.0 + 0.2 * torch.randn(c, generator=g)
        sd[f"sincnet.norm1d.{i}.bias"] = 0.2 * torch.randn(c, generator=g)
    H = 128
    bound = 1.0 / math.sqrt(H)
    for layer in range(lstm_layers):
        isz = 60 if layer == 0 else 2 * H
        for suffix in ("", "_reverse"):
            sd[f"lstm.weight_ih_l{layer}{suffix}"] = _uniform(g, (4 * H, isz), bound) * ih_gain
            sd[f"lstm.weight_hh_l{layer}{suffix}"] = _uniform(g, (4 * H, H), bound) * hh_gain
            sd[f"lstm.bias_ih_l{layer}{suffix}"] = _uniform(g, (4 * H,), bound)
            sd[f"lstm.bias_hh_l{layer}{suffix}"] = _uniform(g, (4 * H,), bound)
    sd["linear.0.weight"] = _uniform(g, (128, 256), 1.0 / math.sqrt(256)) * lin_gain
    sd["linear.0.bias"] = _uniform(g, (128,), 1.0 / math.sqrt(256))
    sd["linear.1.weight"] = _uniform(g, (128, 128), 1.0 / math.sqrt(128)) * lin_gain
    sd["linear.1.bias"] = _uniform(g, (128,), 1.0 / math.sqrt(128))
    sd["classifier.weight"] = _uniform(g, (num_classes, 128), 1.0 / math.sqrt(128)) * logit_scale
    sd["classifier.bias"] = _uniform(g, (num_classes,), 1.0 / math.sqrt(128))
    if fitted_classifier and seed == 0 and lstm_layers == 4 and num_classes == 7:
        # last layer fitted in closed form on synthetic conversations so that segmentations are not
        # degenerate (generator: tests/golden/make_synthetic_classifier.py)
        import os

        path = os.path.join(os.path.dirname(__file__), "data", "synthetic_classifier_seed0.npz")
        if os.path.exists(path):
            z = np.load(path)
            sd["classifier.weight"] = torch.from_numpy(z["weight"]).clone()
            sd["classifier.bias"] = torch.from_numpy(z["bias"]).clone()
    return sd


# ----------------------------------------------------------------------------------------
# embedding state dict
# ----------------------------------------------------------------------------------------


def _bn(sd, prefix, c, g):
    sd[prefix + ".weight"] = 0.8 + 0.4 * torch.rand(c, generator=g)
    sd[prefix + ".bias"] = 0.1 * torch.randn(c, generator=g)
    sd[prefix + ".running_mean"] = 0.1 * torch.randn(c, generator=g)
    sd[prefix + ".running_var"] = 0.5 + torch.rand(c, generator=g)
    sd[prefix + ".num_batches_tracked"] = torch.tensor(1000, dtype=torch.long)


def _conv(sd, name, cout, cin, k, g, gain=1.1):
    fan_in = cin * k * k
    sd[name] = torch.randn(cout, cin, k, k, generator=g) * (gain / math.sqrt(fan_in))


def make_embedding_state_dict(seed: int = 1, centered: bool = True) -> "OrderedDict[str, torch.Tensor]":
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    _conv(sd, "resnet.conv1.weight", 32, 1, 3, g)
    _bn(sd, "resnet.bn1", 32, g)
    in_planes = 32
    for li, (planes, n, stride) in enumerate(((32, 3, 1), (64, 4, 2), (128, 6, 2), (256, 3, 2)), start=1):
        for bi in range(n):
            s = stride if bi == 0 else 1
            p = f"resnet.layer{li}.{bi}"
            _conv(sd, p + ".conv1.weight", planes, in_planes, 3, g)
            _bn(sd, p + ".bn1", planes, g)
            _conv(sd, p + ".conv2.weight", planes, planes, 3, g, gain=0.5)
            _bn(sd, p + ".bn2", planes, g)
            if s != 1 or in_planes != planes:
                _conv(sd, p + ".shortcut.0.weight", planes, in_planes, 1, g, gain=0.8)
                _bn(sd, p + ".shortcut.1", planes, g)
            in_planes = planes
    sd["resnet.seg_1.weight"] = torch.randn(256, 5120, generator=g) / math.sqrt(5120)
    sd["resnet.seg_1.bias"] = 0.01 * torch.randn(256, generator=g)
    if centered and seed == 1:
        # bias calibrated so that embeddings of synthetic conversations are roughly zero-mean (otherwise all
        # cosines are > 0.95 and clustering is trivial); generator: tests/golden/make_synthetic_classifier.py
        import os

        path = os.path.join(os.path.dirname(__file__), "data", "synthetic_embedding_bias_seed1.npz")
        if os.path.exists(path):
            sd["resnet.seg_1.bias"] = torch.from_numpy(np.load(path)["bias"]).clone()
    return sd


BOTTLENECK_BLOCKS = {152: (3, 8, 36, 3), 221: (6, 16, 48, 3), 293: (10, 20, 64, 3)}


def make_bottleneck_state_dict(depth: int = 293, seed: int = 1) -> "OrderedDict[str, torch.Tensor]":
    """WeSpeakerResNet152 / 221 / 293 weights with the keys of the reference's bottleneck ResNet (resnet.py:148-212,
    214-252, two_emb_layer=False).  Trained bottleneck ResNets end each residual branch on a small BatchNorm scale;
    drawing bn3.weight around 0.1 (not the 0.8-1.2 of the other BatchNorms) keeps the residual stream in a realistic
    range through the 100 blocks of ResNet293 instead of growing with depth, which the fp16 trunk could not hold."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    _conv(sd, "resnet.conv1.weight", 32, 1, 3, g)
    _bn(sd, "resnet.bn1", 32, g)
    in_planes = 32
    for li, (planes, n, stride) in enumerate(zip((32, 64, 128, 256), BOTTLENECK_BLOCKS[depth], (1, 2, 2, 2)),
                                             start=1):
        for bi in range(n):
            s = stride if bi == 0 else 1
            p = f"resnet.layer{li}.{bi}"
            _conv(sd, p + ".conv1.weight", planes, in_planes, 1, g)
            _bn(sd, p + ".bn1", planes, g)
            _conv(sd, p + ".conv2.weight", planes, planes, 3, g)
            _bn(sd, p + ".bn2", planes, g)
            _conv(sd, p + ".conv3.weight", 4 * planes, planes, 1, g)
            _bn(sd, p + ".bn3", 4 * planes, g)
            sd[p + ".bn3.weight"] = 0.05 + 0.1 * torch.rand(4 * planes, generator=g)
            if s != 1 or in_planes != 4 * planes:
                _conv(sd, p + ".shortcut.0.weight", 4 * planes, in_planes, 1, g, gain=0.8)
                _bn(sd, p + ".shortcut.1", 4 * planes, g)
            in_planes = 4 * planes
    sd["resnet.seg_1.weight"] = torch.randn(256, 20480, generator=g) / math.sqrt(20480)
    sd["resnet.seg_1.bias"] = 0.01 * torch.randn(256, generator=g)
    return sd


XVECTOR_TDNN = ((60, 512, 5), (512, 512, 3), (512, 512, 3), (512, 512, 1), (512, 1500, 1))


def make_xvector_state_dict(seed: int = 3, dimension: int = 512) -> "OrderedDict[str, torch.Tensor]":
    """XVectorSincNet weights with the reference's keys (xvector.py:205-252): the SincNet front end drawn like
    make_segmentation_state_dict's, then per TDNN layer a Conv1d of gain 1.5 / sqrt(fan_in) and a BatchNorm1d whose
    running statistics are those of a LeakyReLU of a zero-mean input of standard deviation ~1.5 (mean ~0.6, variance
    ~0.8), so that every layer's output stays O(1) on synthetic speech; the Linear 3000 -> dimension has unit gain."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict((k, v) for k, v in make_segmentation_state_dict(seed, fitted_classifier=False).items()
                     if k.startswith("sincnet."))
    return _xvector_tdnn(sd, g, 60, 1.0, dimension)


def make_xvector_mfcc_state_dict(seed: int = 5, dimension: int = 512) -> "OrderedDict[str, torch.Tensor]":
    """XVectorMFCC weights with the reference's keys (xvector.py:42-89): torchaudio's default MFCC buffers
    (models.mfcc_buffers) and the TDNN stack and Linear drawn as in make_xvector_state_dict, except that the first
    Conv1d's gain is 1/30 of it: MFCC coefficients are tens of units (c0 around -130 and reaching the hundreds on
    synthetic speech, RMS ~28 over all 40), where SincNet's features are O(1)."""
    from ..models import mfcc_buffers

    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict(("mfcc." + k, v) for k, v in mfcc_buffers().items())
    return _xvector_tdnn(sd, g, 40, 1.0 / 30.0, dimension)


def _xvector_tdnn(sd, g, cin0: int, gain0: float, dimension: int):
    """The ``tdnns.*`` and ``embedding.*`` entries of make_xvector_state_dict / make_xvector_mfcc_state_dict: tdnns.0
    has ``cin0`` inputs and ``gain0`` times the other layers' gain."""
    for layer, (cin, cout, k) in enumerate(XVECTOR_TDNN):
        cin, gain = (cin0, gain0) if layer == 0 else (cin, 1.0)
        conv, bn = f"tdnns.{3 * layer}", f"tdnns.{3 * layer + 2}"
        sd[conv + ".weight"] = torch.randn(cout, cin, k, generator=g) * (gain * 1.5 / math.sqrt(cin * k))
        sd[conv + ".bias"] = 0.05 * torch.randn(cout, generator=g)
        sd[bn + ".weight"] = 0.8 + 0.4 * torch.rand(cout, generator=g)
        sd[bn + ".bias"] = 0.1 * torch.randn(cout, generator=g)
        sd[bn + ".running_mean"] = 0.6 * (1.0 + 0.2 * torch.randn(cout, generator=g))
        sd[bn + ".running_var"] = 0.8 * (0.75 + 0.5 * torch.rand(cout, generator=g))
        sd[bn + ".num_batches_tracked"] = torch.tensor(1000, dtype=torch.long)
    sd["embedding.weight"] = torch.randn(dimension, 3000, generator=g) / math.sqrt(3000)
    sd["embedding.bias"] = 0.01 * torch.randn(dimension, generator=g)
    return sd


# ----------------------------------------------------------------------------------------
# PLDA
# ----------------------------------------------------------------------------------------


def make_sseriouss_state_dict(seed: int = 5, wav2vec_layer: int = -1, lstm_layers: int = 4, num_classes: int = 7,
                              pos_weight_norm: str = "parametrizations",
                              logit_scale: float = 4.0) -> "OrderedDict[str, torch.Tensor]":
    """SSeRiouSS on WavLM Base (models/segmentation/SSeRiouSS.py, torchaudio wavlm_model(**WAVLM_BASE._params)):
    seeded weights under the module's keys.  Gains keep every activation O(1) through the conv stack and the 12
    post-LN layers (no fp16 under- or overflow), and the relative position bias and layer weights are far from uniform
    so that each part of the network shows in the output.  ``wav2vec_layer`` >= 1 drops ``wav2vec_weights`` (the
    reference builds it only for the layer average); ``pos_weight_norm`` = "parametrizations" (current torch) or
    "weight_g" (torch.nn.utils.weight_norm spelling of older checkpoints)."""
    g = torch.Generator().manual_seed(seed)

    def normal(shape, std):
        return torch.randn(shape, generator=g, dtype=torch.float32) * std

    def affine(prefix, c):
        sd[prefix + ".weight"] = 1.0 + 0.1 * torch.randn(c, generator=g)
        sd[prefix + ".bias"] = 0.05 * torch.randn(c, generator=g)

    def linear(prefix, cout, cin, gain=1.0):
        sd[prefix + ".weight"] = normal((cout, cin), gain / math.sqrt(cin))
        sd[prefix + ".bias"] = normal((cout,), 0.02)

    sd = OrderedDict()
    fe, tr = "wav2vec.feature_extractor.conv_layers.", "wav2vec.encoder.transformer."
    sd[fe + "0.conv.weight"] = normal((512, 1, 10), 1.0 / math.sqrt(10))
    affine(fe + "0.layer_norm", 512)
    for i, k in enumerate((3, 3, 3, 3, 2, 2), start=1):
        sd[f"{fe}{i}.conv.weight"] = normal((512, 512, k), 1.8 / math.sqrt(512 * k))
    affine("wav2vec.encoder.feature_projection.layer_norm", 512)
    linear("wav2vec.encoder.feature_projection.projection", 768, 512)
    pc = tr + "pos_conv_embed.conv."
    g_, v_ = 2.0 + 0.2 * torch.randn((1, 1, 128), generator=g), normal((768, 48, 128), 1.0)
    if pos_weight_norm == "parametrizations":
        sd[pc + "parametrizations.weight.original0"], sd[pc + "parametrizations.weight.original1"] = g_, v_
    else:
        sd[pc + "weight_g"], sd[pc + "weight_v"] = g_, v_
    sd[pc + "bias"] = normal((768,), 0.05)
    affine(tr + "layer_norm", 768)
    for layer in range(12):
        p = f"{tr}layers.{layer}."
        if layer == 0:
            sd[p + "attention.rel_attn_embed.weight"] = normal((320, 12), 1.5)
        sd[p + "attention.attention.in_proj_weight"] = normal((2304, 768), 1.5 / math.sqrt(768))
        sd[p + "attention.attention.in_proj_bias"] = normal((2304,), 0.02)
        linear(p + "attention.attention.out_proj", 768, 768)
        linear(p + "attention.gru_rel_pos_linear", 8, 64, gain=0.5)
        sd[p + "attention.gru_rel_pos_const"] = 1.0 + 0.2 * torch.randn((1, 12, 1, 1), generator=g)
        affine(p + "layer_norm", 768)
        linear(p + "feed_forward.intermediate_dense", 3072, 768)
        linear(p + "feed_forward.output_dense", 768, 3072)
        affine(p + "final_layer_norm", 768)
    if wav2vec_layer < 0:
        sd["wav2vec_weights"] = normal((12,), 1.0)
    for layer in range(lstm_layers):
        cin = 768 if layer == 0 else 256
        for suffix in ("", "_reverse"):
            sd[f"lstm.weight_ih_l{layer}{suffix}"] = normal((512, cin), 2.0 / math.sqrt(cin))
            sd[f"lstm.weight_hh_l{layer}{suffix}"] = normal((512, 128), 1.0 / math.sqrt(128))
            sd[f"lstm.bias_ih_l{layer}{suffix}"] = normal((512,), 0.1)
            sd[f"lstm.bias_hh_l{layer}{suffix}"] = normal((512,), 0.1)
    linear("linear.0", 128, 256, gain=2.0)
    linear("linear.1", 128, 128, gain=2.0)
    linear("classifier", num_classes, 128, gain=logit_scale)
    return sd


def make_plda(seed: int = 2, dim: int = 256, lda_dim: int = 128):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((dim, dim)))
    lda = q[:, :lda_dim] * (1.0 + 0.1 * rng.standard_normal((1, lda_dim)))
    mean1 = 0.05 * rng.standard_normal(dim)
    mean2 = 0.05 * rng.standard_normal(lda_dim)
    mu = 0.05 * rng.standard_normal(lda_dim)
    tr = np.eye(lda_dim) + 0.05 * rng.standard_normal((lda_dim, lda_dim))
    psi = np.sort(np.exp(rng.uniform(np.log(0.05), np.log(20.0), lda_dim)))[::-1].copy()
    return dict(mean1=mean1, mean2=mean2, lda=lda, mu=mu, tr=tr, psi=psi)


# ----------------------------------------------------------------------------------------
# audio
# ----------------------------------------------------------------------------------------


def make_conversation(duration_s: float, seed: int = 1234, num_speakers: int = 3,
                      sample_rate: int = SAMPLE_RATE, return_turns: bool = False):
    """(1, T) float32 synthetic conversation in [-1, 1] (+ list of (start_s, end_s, speaker) turns)."""
    rng = np.random.default_rng(seed)
    T = int(round(duration_s * sample_rate))
    out = np.zeros(T, dtype=np.float32)
    t_all = np.arange(T, dtype=np.float64) / sample_rate
    spk = []
    for _ in range(num_speakers):
        f0 = rng.uniform(80, 250)
        nh = int(rng.integers(10, 21))
        env = np.exp(-0.5 * ((np.arange(1, nh + 1) * f0 - rng.uniform(300, 2500)) / rng.uniform(400, 1500)) ** 2)
        env = env / env.sum() + 0.02
        spk.append(dict(f0=f0, amps=env, phases=rng.uniform(0, 2 * np.pi, nh), am=rng.uniform(3, 6),
                        vib=rng.uniform(0.002, 0.01)))
    # turn taking: alternate speakers with 0.5-5 s turns, ~8% overlap, some silences
    t = 0.0
    turns = []
    cur = int(rng.integers(num_speakers))
    while t < duration_s:
        turn = float(rng.uniform(0.5, 5.0))
        if rng.uniform() < 0.15:
            t += float(rng.uniform(0.2, 1.5))      # silence
        a, b = t, min(duration_s, t + turn)
        i0, i1 = int(a * sample_rate), int(b * sample_rate)
        if i1 > i0:
            turns.append((a, b, cur))
            s = spk[cur]
            tt = t_all[i0:i1]
            sig = np.zeros(i1 - i0)
            f0 = s["f0"] * (1.0 + s["vib"] * np.sin(2 * np.pi * 5.0 * tt))
            ph = 2 * np.pi * np.cumsum(f0) / sample_rate
            for h, (amp, p0) in enumerate(zip(s["amps"], s["phases"]), start=1):
                if h * s["f0"] < sample_rate / 2 - 200:
                    sig += amp * np.sin(h * ph + p0)
            am = 0.6 + 0.4 * np.sin(2 * np.pi * s["am"] * tt + rng.uniform(0, 2 * np.pi))
            ramp = np.minimum(1.0, np.minimum(np.arange(i1 - i0), np.arange(i1 - i0)[::-1]) / (0.02 * sample_rate))
            out[i0:i1] += (0.35 * sig * am * ramp).astype(np.float32)
        if b >= duration_s:
            break
        overlap = turn * (rng.uniform(0.0, 0.16))
        t = b - overlap
        nxt = int(rng.integers(num_speakers - 1))
        cur = nxt if nxt < cur else nxt + 1
    out += (10 ** (-30 / 20)) * rng.standard_normal(T).astype(np.float32) * 0.3
    peak = np.max(np.abs(out)) + 1e-9
    out = np.clip(out / max(1.0, peak / 0.95), -1.0, 1.0)
    wav = torch.from_numpy(out.astype(np.float32))[None]
    return (wav, turns) if return_turns else wav
