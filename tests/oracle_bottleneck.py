"""Oracle (TEST INFRASTRUCTURE): CPU / fp32 torch restatement of the bottleneck WeSpeaker ResNets
(WeSpeakerResNet152 / 221 / 293: models/embedding/wespeaker/resnet.py:148-212, 214-252, 477-508 and
wespeaker/__init__.py:375-466, two_emb_layer=False), next to ``oracle.nets.WeSpeakerResNet34``.

It reuses the fbank and the statistics pooling of ``oracle.nets`` (repository root on the import path) and has the
reference's state-dict keys.  It lives with the tests because the product package never imports the oracle.  Pinned against the reference's own resnet.py by tests/golden/make_golden_bottleneck.py
and tests/test_wespeaker_deep.py.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import nets

from pyannote_audio_b200.testing.synthetic import BOTTLENECK_BLOCKS


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, in_planes, planes, stride=1):
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

    def forward(self, x):
        out = F.relu(self.bn1(self.conv1(x)))
        out = F.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(out)) + self.shortcut(x)
        return F.relu(out)


class BottleneckResNet(nn.Module):
    """Stem 3x3 1 -> 32, layers of Bottlenecks with planes 32 / 64 / 128 / 256 and strides 1 / 2 / 2 / 2, TSTP
    statistics pooling of the 1024 x 10 trunk channels, seg_1 20480 -> 256."""

    def __init__(self, num_blocks, feat_dim=80, embed_dim=256, m_channels=32):
        super().__init__()
        self.in_planes = m_channels
        self.conv1 = nn.Conv2d(1, m_channels, 3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(m_channels)
        self.layer1 = self._make_layer(m_channels, num_blocks[0], 1)
        self.layer2 = self._make_layer(m_channels * 2, num_blocks[1], 2)
        self.layer3 = self._make_layer(m_channels * 4, num_blocks[2], 2)
        self.layer4 = self._make_layer(m_channels * 8, num_blocks[3], 2)
        self.seg_1 = nn.Linear(int(feat_dim / 8) * m_channels * 8 * 4 * 2, embed_dim)

    def _make_layer(self, planes, n, stride):
        layers = []
        for s in [stride] + [1] * (n - 1):
            layers.append(Bottleneck(self.in_planes, planes, s))
            self.in_planes = 4 * planes
        return nn.Sequential(*layers)

    def blocks(self):
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            yield from layer

    def forward_frames(self, fbank, trace=None):
        """(B, T, 80) -> (B, 1024, 10, T'); ``trace``: a list that receives every block's output."""
        out = F.relu(self.bn1(self.conv1(fbank.permute(0, 2, 1).unsqueeze(1))))
        for block in self.blocks():
            out = block(out)
            if trace is not None:
                trace.append(out)
        return out

    def forward_embedding(self, frames, weights=None):
        b, c, f, t = frames.shape
        return self.seg_1(nets.stats_pool(frames.reshape(b, c * f, t), weights=weights))

    def forward(self, fbank, weights=None):
        return self.forward_embedding(self.forward_frames(fbank), weights=weights)


class WeSpeakerBottleneck(nn.Module):
    """WeSpeakerResNet152 / 221 / 293 with the interface of ``oracle.nets.WeSpeakerResNet34``."""

    def __init__(self, depth: int):
        super().__init__()
        self.resnet = BottleneckResNet(BOTTLENECK_BLOCKS[depth])

    compute_fbank = staticmethod(nets.WeSpeakerResNet34.compute_fbank)

    def forward(self, waveforms, weights=None):
        return self.resnet(self.compute_fbank(waveforms), weights=weights)

    def forward_frames(self, waveforms):
        return self.resnet.forward_frames(self.compute_fbank(waveforms))

    def forward_embedding(self, frames, weights=None):
        return self.resnet.forward_embedding(frames, weights=weights)
