"""Oracle (TEST INFRASTRUCTURE): CPU / fp32 torch restatement of XVectorMFCC (models/embedding/xvector.py:42-202):
torchaudio's MFCC with its defaults (the reference's own front end) followed by the TDNN stack, StatsPool and Linear of
``oracle_xvector.XVectorSincNet``, with the reference's state-dict keys.  Pinned against the reference's own xvector.py
by tests/golden/make_golden_xvector_mfcc.py and tests/test_xvector_mfcc.py.
"""
from __future__ import annotations

import torch.nn as nn
import torchaudio

from oracle import nets
from oracle_xvector import CHANNELS, DILATION, KERNEL


class XVectorMFCC(nn.Module):
    def __init__(self, dimension: int = 512):
        super().__init__()
        self.mfcc = torchaudio.transforms.MFCC(sample_rate=16000, n_mfcc=40, dct_type=2, norm="ortho", log_mels=False)
        self.tdnns = nn.ModuleList()
        cin = 40
        for cout, k, d in zip(CHANNELS, KERNEL, DILATION):
            self.tdnns.extend([nn.Conv1d(cin, cout, k, dilation=d), nn.LeakyReLU(), nn.BatchNorm1d(cout)])
            cin = cout
        self.embedding = nn.Linear(2 * cin, dimension)

    def frames(self, waveforms):
        """(B, 1, samples) -> the last TDNN layer's output (B, 1500, T), and every layer's output on the way."""
        out = self.mfcc(waveforms).squeeze(dim=1)
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
    return nets.multi_conv_num_frames(1 + num_samples // 200, KERNEL, [1] * 5, [0] * 5, DILATION)


def receptive_field_size(num_frames: int = 1) -> int:
    return 400 + (nets.multi_conv_receptive_field_size(num_frames, KERNEL, [1] * 5, [0] * 5, DILATION) - 1) * 200


def receptive_field_center(frame: int = 0) -> int:
    return nets.multi_conv_receptive_field_center(frame, KERNEL, [1] * 5, [0] * 5, DILATION) * 200
