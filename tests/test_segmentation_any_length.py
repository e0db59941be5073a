"""Segmentation of audio of any length: PyanNet.forward, Inference (window="whole", crop, sliding with any duration)
and VoiceActivityDetection with any window, against the fp32 oracle run on the GPU with TF32 off (reference:
models/segmentation/PyanNet.py:223-240, models/blocks/sincnet.py:163-184, core/inference.py:182-373, 498-620,
pipelines/voice_activity_detection.py:95-127).

"Agrees" means: log-probabilities within 3e-4, and class ids equal to the oracle's argmax wherever the oracle's top-2
log-probability margin is at least LOW_MARGIN (below it an argmax flip is fp32 summation-order noise)."""
import numpy as np
import pytest
import torch

from oracle import nets, pipeline as P
from pyannote_audio_b200 import ops, synthetic as syn
from pyannote_audio_b200.models import PyanNet

SR = 16000
LOW_MARGIN = 1e-4          # top-2 log-probability margin under which an argmax flip is fp32 reordering noise
ATOL = 3e-4
FP32_TWINS = ("seg_conv_impl", "seg_gemm_impl", "seg_rec_impl")


# ---- host-only ------------------------------------------------------------------------------------------------
def test_num_frames_matches_the_oracle():
    for n in list(range(1261, 1400)) + [16000, 48000, 159999, 160000, 160001, 480000, 1000000, 57600000]:
        assert ops.seg_num_frames(n) == nets.sincnet_num_frames(n) == PyanNet().num_frames(n)
    assert ops.seg_num_frames(1261) == 2 and ops.seg_num_frames(1260) == 1


def test_too_short_windows_raise_before_any_device_work():
    seg = PyanNet()                                        # on the CPU: a device call would fail differently
    with pytest.raises(ValueError, match="1261"):
        seg(torch.zeros(1, 1, 1260))
    with pytest.raises(ValueError, match="1261"):
        seg.forward_chunks(torch.zeros(2000), [0], [1000], window=1000)
    from pyannote_audio_b200.inference import Inference

    with pytest.warns(UserWarning):
        inf = Inference(seg, duration=0.07, step=0.01)     # 1120 samples
    with pytest.raises(ValueError, match="1261"):
        inf.slide_device(torch.zeros(1, 16000), SR)


def test_diarization_rejects_other_windows_before_any_device_work():
    from pyannote_audio_b200.models import WeSpeakerResNet34
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    seg = PyanNet(duration=5.0)
    with pytest.raises(ValueError, match="10 s"):
        SpeakerDiarization(segmentation=seg, embedding=WeSpeakerResNet34(), clustering="AgglomerativeClustering")


# ---- GPU ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def seg(dev):
    m = PyanNet()
    m.load_state_dict(syn.make_segmentation_state_dict(0))
    return m.to(dev)


@pytest.fixture(scope="module")
def oseg(dev):
    m = nets.PyanNet()
    m.load_state_dict(syn.make_segmentation_state_dict(0))
    return m.to(dev).eval()


@pytest.fixture(autouse=True)
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


@pytest.fixture(scope="module")
def long_wav():
    return syn.make_conversation(66.0, seed=5)


class fp32_twins:
    """Context: run the SincNet convs, the GEMMs and the recurrence on their fp32 CUDA-core twins."""

    def __init__(self, ctx):
        self.ctx = ctx

    def __enter__(self):
        for k in FP32_TWINS:
            self.ctx.set_option(k, 0)

    def __exit__(self, *exc):
        for k in FP32_TWINS:
            self.ctx.set_option(k, 1)


def _oracle(oseg, wav):
    with torch.inference_mode():
        return oseg(wav.cuda()).cpu().numpy()


def _low_margin(ref_logp):
    top2 = np.sort(ref_logp, axis=-1)
    return (top2[..., -1] - top2[..., -2]) < LOW_MARGIN


def _assert_agrees(name, logp, ref):
    assert logp.shape == ref.shape, (name, logp.shape, ref.shape)
    err = float(np.abs(logp - ref).max())
    mism = logp.argmax(-1) != ref.argmax(-1)
    low = _low_margin(ref)
    print(f"[any-length] {name}: {ref.shape[0]}x{ref.shape[1]} frames, max |dlogp| {err:.2e}, "
          f"{int(mism.sum())} class mismatches ({int((mism & low).sum())} low-margin)")
    assert err <= ATOL, (name, err)
    assert not (mism & ~low).any(), name


def _classes_agree(cls, ref_logp):
    """Class ids vs the oracle: equal wherever the oracle's margin is clear; returns the oracle's ids with the
    low-margin frames taken from ``cls`` (the reference input of a bit-exact aggregation check)."""
    ref_cls = ref_logp.argmax(-1)
    low = _low_margin(ref_logp)
    assert not ((cls != ref_cls) & ~low).any()
    return np.where(low, cls, ref_cls)


def _multilabel(cls):
    return nets.powerset_mapping(3, 2).numpy()[cls].astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1261, 1271, 16000, 48000, 159999, 160001, 480000, 1000000])
@pytest.mark.parametrize("batch", [1, 3])
def test_forward_any_length_matches_oracle(seg, oseg, long_wav, N, batch):
    rng = np.random.default_rng(N + batch)
    starts = rng.integers(0, long_wav.shape[1] - N, size=batch)
    wav = torch.stack([long_wav[:, s: s + N] for s in starts])                         # (batch, 1, N)
    F = seg.num_frames(N)
    ref = _oracle(oseg, wav)
    got = seg(wav).cpu().numpy()
    assert got.shape == (batch, F, 7)
    _assert_agrees(f"N={N} B={batch}", got, ref)
    with fp32_twins(seg._ctx()):
        twin = seg(wav).cpu().numpy()
    _assert_agrees(f"N={N} B={batch} fp32 twins", twin, ref)
    _assert_agrees(f"N={N} B={batch} fp32 twins vs default", twin, got)


@pytest.mark.gpu
def test_forward_ten_minute_conversation(seg, oseg):
    wav = syn.make_conversation(600.0, seed=23)[None]                                 # (1, 1, 9.6 M)
    ref = _oracle(oseg, wav)
    assert ref.shape[1] == seg.num_frames(wav.shape[-1]) > 35000
    _assert_agrees("10 min", seg(wav).cpu().numpy(), ref)
    with fp32_twins(seg._ctx()):
        twin = seg(wav).cpu().numpy()
    _assert_agrees("10 min fp32 twins", twin, ref)


@pytest.mark.gpu
def test_window_path_reproduces_the_10s_path_bit_for_bit(seg, dev):
    from pyannote_audio_b200 import _lib
    from pyannote_audio_b200.inference import chunk_layout

    ctx = seg._ctx()
    wav = syn.make_conversation(31.3, seed=17)[0].to(dev)
    off, valid, _, _ = chunk_layout(wav.numel(), 160000, 16000)
    buf = torch.zeros(int(off[-1]) + 160000, device=dev)
    buf[: wav.numel()] = wav
    assert valid[-1] < 160000                                                         # a padded last chunk
    n = len(off)
    cls = torch.empty((n, 589), dtype=torch.uint8, device=dev)
    logp = torch.empty((n, 589, 7), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(ctx.lib.b200_seg_forward(ctx._h, ops._ptr(buf), off.ctypes.data, valid.ctypes.data, n,
                                            ops._ptr(cls), ops._ptr(logp), ops._stream(dev)))
    got_cls, got_logp = ctx.seg_forward(buf, off, valid, return_logp=True, window=160000)
    assert torch.equal(got_cls, cls) and torch.equal(got_logp, logp)


@pytest.mark.gpu
def test_limits_and_sub_batches(seg, dev, long_wav):
    ctx = seg._ctx()
    wav = long_wav[0].to(dev).contiguous()
    with pytest.raises(ValueError, match="1261"):
        ctx.seg_forward(wav, [0], [1260], window=1260)
    with pytest.raises(ValueError):
        ctx.seg_forward(wav, [0], [48001], window=48000)                                # valid > window
    # many short windows, then three 1 M-sample windows (several wav_stats slices, two-level InstanceNorm sums)
    for N, n, small in ((48000, 20, 1), (1000000, 3, 7)):
        off = np.linspace(0, wav.numel() - N, n).astype(np.int64)
        valid = np.full(n, N, dtype=np.int32)
        valid[-1] = N - 777                                                             # a padded window
        try:
            ref = ctx.seg_forward(wav, off, valid, return_logp=True, window=N)
            ctx.set_option("seg_max_batch", small)          # 160000 / 1 120 000 samples: 3 / 1 windows per sub-batch
            got = ctx.seg_forward(wav, off, valid, return_logp=True, window=N)
            assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
            if N > 160000:
                ctx.set_option("seg_max_batch", 6)          # 960 000 samples < one window
                with pytest.raises(ValueError, match="seg_max_batch to at least 7"):
                    ctx.seg_forward(wav, off, valid, window=N)
        finally:
            ctx.set_option("seg_max_batch", 2112)


def _file(seconds, seed):
    return {"waveform": syn.make_conversation(seconds, seed=seed), "sample_rate": SR}


@pytest.mark.gpu
def test_inference_whole_and_crop(seg, oseg):
    from pyannote_audio_b200.core import Segment
    from pyannote_audio_b200.inference import Inference

    file = _file(66.0, 9)
    with pytest.warns(UserWarning):                        # "whole" with a frame-based model, as the reference warns
        whole = Inference(seg, window="whole")
    out = whole(file)
    ref = _oracle(oseg, file["waveform"][None])[0]
    assert out.shape == (seg.num_frames(file["waveform"].shape[1]), 3) and out.dtype == np.float32
    cls = _classes_agree(_ml_to_cls(out), ref)
    assert np.array_equal(out, _multilabel(cls))
    excerpt = Segment(2.0, 19.5)
    out = whole.crop(file, excerpt)
    wav, _ = seg.audio.crop(file, excerpt)
    ref = _oracle(oseg, wav[None])[0]
    assert out.shape == (seg.num_frames(wav.shape[1]), 3)
    _classes_agree(_ml_to_cls(out), ref)


def _ml_to_cls(ml):
    """multilabel rows -> powerset class ids (the mapping is one-to-one)."""
    mapping = nets.powerset_mapping(3, 2).numpy()
    return (ml[..., None, :] == mapping).all(-1).argmax(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("duration,step", [(5.0, 0.5), (2.0, 0.2)])
def test_inference_sliding_any_duration(seg, oseg, duration, step):
    from pyannote_audio_b200.inference import Inference

    file = _file(23.33, 31)                                # leaves a padded last chunk for both steps
    W, S = int(duration * SR), int(step * SR)
    chunks = P.chunk_waveform(file["waveform"], window_size=W, step_size=S)
    ref = _oracle(oseg, chunks)                                                        # (C, F, 7)
    with pytest.warns(UserWarning):                        # trained on 10 s chunks, as the reference warns
        raw = Inference(seg, duration=duration, step=step, skip_aggregation=True)
    out = raw(file)
    sw = out.sliding_window
    assert (sw.start, sw.duration, sw.step) == (0.0, duration, step)
    assert out.data.shape == (chunks.shape[0], seg.num_frames(W), 3)
    cls = _classes_agree(_ml_to_cls(out.data), ref)
    assert np.array_equal(out.data, _multilabel(cls))
    # aggregated (a pre-aggregation hook makes a permutation-invariant model's output aggregate, as in the reference)
    with pytest.warns(UserWarning):
        agg_inf = Inference(seg, duration=duration, step=step, pre_aggregation_hook=lambda s: s)
    agg = agg_inf(file)
    frames = P.SW(*nets.sincnet_receptive_field())
    num_samples = file["waveform"].shape[1]
    expected = P.aggregate(P.SWF(_multilabel(cls), P.SW(0.0, duration, step)), frames, hamming=True, missing=0.0)
    expected = expected.crop_loose((0.0, num_samples / SR))
    assert np.array_equal(agg.data, expected.data)
    # the device overlap-add is bit-identical to Inference.aggregate (host numpy) on the same classes
    from pyannote_audio_b200.core import Segment, SlidingWindowFeature

    host = Inference.aggregate(SlidingWindowFeature(out.data, sw), seg.receptive_field, hamming=True, missing=0.0)
    host = host.crop(Segment(0.0, num_samples / SR), mode="loose")
    assert np.array_equal(agg.data, host)


@pytest.mark.gpu
def test_voice_activity_detection_any_window(seg, oseg):
    from pyannote_audio_b200.vad import VoiceActivityDetection

    file = _file(47.77, 12)
    with pytest.warns(UserWarning):
        vad = VoiceActivityDetection(seg, duration=5.0, step=0.5)
    scores = vad.speech_scores(file)
    W, S = 5 * SR, SR // 2
    chunks = P.chunk_waveform(file["waveform"], window_size=W, step_size=S)
    cls = _classes_agree(seg.forward_chunks(*_resident(seg, file, W, S), window=W).cpu().numpy(),
                         _oracle(oseg, chunks))
    speech = _multilabel(cls).max(-1, keepdims=True)
    frames = P.SW(*nets.sincnet_receptive_field())
    ref = P.aggregate(P.SWF(speech, P.SW(0.0, 5.0, 0.5)), frames, hamming=True, missing=0.0)
    ref = ref.crop_loose((0.0, file["waveform"].shape[1] / SR))
    assert np.array_equal(scores.data, ref.data)
    assert 0.0 < scores.data.mean() < 1.0
    ann = vad(file)
    got = [(s.start, s.end) for s, _ in ann.itertracks()]
    want = [(a, b) for a, b, _ in P.binarize_scores(ref)]
    assert len(got) == len(want) > 0
    np.testing.assert_allclose(np.array(got), np.array(want), rtol=0, atol=1e-9)


def _resident(seg, file, W, S):
    """(device waveform, offsets, valid lengths) of Inference.slide's windows."""
    from pyannote_audio_b200.inference import chunk_layout

    wav = file["waveform"]
    off, valid, _, _ = chunk_layout(wav.shape[1], W, S)
    buf = torch.zeros(int(off[-1]) + W, device=seg.device)
    buf[: wav.shape[1]] = wav[0].to(seg.device)
    return buf, off, valid


@pytest.mark.gpu
def test_diarization_rejects_an_inference_with_another_window(seg, dev):
    from pyannote_audio_b200.inference import Inference
    from pyannote_audio_b200.models import WeSpeakerResNet34
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    emb = WeSpeakerResNet34()
    emb.load_state_dict(syn.make_embedding_state_dict(1))
    pipe = SpeakerDiarization(segmentation=seg, embedding=emb, clustering="AgglomerativeClustering", device=dev)
    with pytest.warns(UserWarning):
        pipe._segmentation = Inference(seg, duration=5.0, step=0.5, skip_aggregation=True)
    with pytest.raises(ValueError, match="10 s"):
        pipe(_file(12.0, 3))
