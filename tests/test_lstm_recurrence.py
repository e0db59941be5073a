"""BiLSTM recurrence: the two-warpgroup, Gx-pipelined kernel (seg_rec_impl = 1) against the one-warpgroup kernel
(seg_rec_impl = 2).  Both give every (sequence, unit, gate) column the same 24 split-precision products (K steps 0..7;
lo*hi, hi*lo, hi*hi) in the same order onto the same Gx, and run the same gate and cell arithmetic, so log-probabilities,
classes and scores are bit-identical and the launch counts are equal.

Cases: seg_forward on 10 s windows at 1, 63, 64, 65, 756, 2112 and 2113 windows (partial 64-sequence tiles, a second
sub-batch at the default seg_max_batch); windows of other lengths (other step counts T); a multi-label sigmoid head;
SSeRiouSS, whose LSTM head goes through the same recurrence.
"""
import numpy as np
import pytest
import torch

from pyannote_audio_b200 import synthetic as syn
from pyannote_audio_b200.core import Problem, Resolution, Specifications
from pyannote_audio_b200.models import PyanNet, SSeRiouSS

pytestmark = pytest.mark.gpu

CHUNK = 160000


@pytest.fixture(scope="module")
def ctx():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyannote_audio_b200 import ops

    c = ops.Context(torch.device("cuda:0"))
    c.load_segmentation(syn.make_segmentation_state_dict(0))
    return c


def _both(ctx, run):
    """(pipelined outputs, reference outputs) as lists of numpy arrays, and the two launch counts."""
    out, launches = {}, {}
    try:
        for impl in (2, 1):
            ctx.set_option("seg_rec_impl", impl)
            n0 = ctx.launch_count
            res = run()
            torch.cuda.synchronize()
            res = res if isinstance(res, tuple) else (res,)
            out[impl] = [r.cpu().numpy() for r in res]
            launches[impl] = ctx.launch_count - n0
    finally:
        ctx.set_option("seg_rec_impl", 1)
    return out[1], out[2], launches[1], launches[2]


def _assert_same(new, ref, n_new, n_ref):
    assert len(new) == len(ref)
    for a, b in zip(new, ref):
        assert a.shape == b.shape and a.dtype == b.dtype
        f = b.astype(np.float64)
        assert np.abs(f[np.isfinite(f)]).max() > 0
        assert a.tobytes() == b.tobytes()
    assert n_new == n_ref


def _wav(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * 0.1).cuda()


@pytest.mark.parametrize("nb", [1, 63, 64, 65, 756, 2112, 2113])
def test_seg_forward_matches_one_warpgroup(ctx, nb):
    step = 1600
    wav = _wav(step * (nb - 1) + CHUNK + 5, 900 + nb)
    off = 5 + np.arange(nb, dtype=np.int64) * step
    valid = np.full(nb, CHUNK, dtype=np.int32)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.seg_forward(wav, off, valid, return_logp=True))
    assert ref[1].shape == (nb, 589, 7)
    _assert_same(new, ref, n_new, n_ref)


# 1261: the shortest window (one step); 48000 and 160001: other step counts; 480000: 1771 steps
@pytest.mark.parametrize("window", [1261, 48000, 160001, 480000])
def test_seg_forward_any_window_matches_one_warpgroup(ctx, window):
    nb = 67
    wav = _wav(window + 333 * (nb - 1) + 7, window)
    off = 7 + np.arange(nb, dtype=np.int64) * 333
    valid = np.full(nb, window, dtype=np.int32)
    new, ref, n_new, n_ref = _both(ctx, lambda: ctx.seg_forward(wav, off, valid, return_logp=True, window=window))
    _assert_same(new, ref, n_new, n_ref)


def test_sigmoid_head_matches_one_warpgroup():
    k = 4
    m = PyanNet()
    m.specifications = Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, 5.0,
                                      classes=[f"label#{i}" for i in range(k)])
    m.load_state_dict(syn.make_segmentation_state_dict(0, num_classes=m.dimension))
    m = m.to(torch.device("cuda:0"))
    wav = torch.stack([_wav(80000, 31 + i) for i in range(70)])[:, None]
    _assert_same(*_both(m._ctx(), lambda: m(wav)))


def test_sseriouss_matches_one_warpgroup():
    m = SSeRiouSS(wav2vec_layer=-1)
    m.specifications = Specifications(Problem.MONO_LABEL_CLASSIFICATION, Resolution.FRAME, 10.0,
                                      classes=["speaker#1", "speaker#2", "speaker#3"], powerset_max_classes=2,
                                      permutation_invariant=True)
    m.load_state_dict(syn.make_sseriouss_state_dict(5, wav2vec_layer=-1, num_classes=7))
    m = m.eval().to(torch.device("cuda:0"))
    wav = torch.stack([_wav(CHUNK, 61 + i) for i in range(3)])[:, None]
    _assert_same(*_both(m._ctx(), lambda: m(wav)))
