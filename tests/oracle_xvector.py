"""Oracle (TEST INFRASTRUCTURE): CPU / fp32 torch restatement of XVectorSincNet (models/embedding/xvector.py:205-349)
built from ``oracle.nets.SincNet`` and ``oracle.nets.stats_pool`` plus torch Conv1d / LeakyReLU / BatchNorm1d / Linear,
with the reference's state-dict keys.  It lives with the tests because the product package never imports the oracle.
Pinned against the reference's own xvector.py by tests/golden/make_golden_xvector.py and tests/test_xvector.py.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from oracle import nets

KERNEL = [5, 3, 3, 1, 1]
DILATION = [1, 2, 3, 1, 1]
CHANNELS = [512, 512, 512, 512, 1500]


class XVectorSincNet(nn.Module):
    def __init__(self, dimension: int = 512):
        super().__init__()
        self.sincnet = nets.SincNet(stride=10)
        self.tdnns = nn.ModuleList()
        cin = 60
        for cout, k, d in zip(CHANNELS, KERNEL, DILATION):
            self.tdnns.extend([nn.Conv1d(cin, cout, k, dilation=d), nn.LeakyReLU(), nn.BatchNorm1d(cout)])
            cin = cout
        self.embedding = nn.Linear(2 * cin, dimension)

    def frames(self, waveforms):
        """(B, 1, samples) -> the last TDNN layer's output (B, 1500, T), and every layer's output on the way."""
        out = self.sincnet(waveforms)
        per_layer = []
        for i, m in enumerate(self.tdnns):
            out = m(out)
            if i % 3 == 2:
                per_layer.append(out)
        return out, per_layer

    def forward(self, waveforms, weights=None):
        out, _ = self.frames(waveforms)
        return self.embedding(nets.stats_pool(out, weights=weights))


def num_frames(num_samples: int) -> int:
    return nets.multi_conv_num_frames(nets.sincnet_num_frames(num_samples), KERNEL, [1] * 5, [0] * 5, DILATION)


def receptive_field_size(num_frames: int = 1) -> int:
    rf = nets.multi_conv_receptive_field_size(num_frames, KERNEL, [1] * 5, [0] * 5, DILATION)
    return nets.multi_conv_receptive_field_size(rf, nets.SINCNET_K, nets.SINCNET_S, nets.SINCNET_P, nets.SINCNET_D)


def receptive_field_center(frame: int = 0) -> int:
    c = nets.multi_conv_receptive_field_center(frame, KERNEL, [1] * 5, [0] * 5, DILATION)
    return nets.multi_conv_receptive_field_center(c, nets.SINCNET_K, nets.SINCNET_S, nets.SINCNET_P, nets.SINCNET_D)
