"""PyanNet heads other than community-1's: sigmoid (binary and multi-label) heads of 1 to 32 classes, powerset heads of
any (speakers, max per frame) up to 32 classes, and what runs on them: Inference, VoiceActivityDetection and
MultiLabelSegmentation (reference: models/segmentation/PyanNet.py:141-161, 223-240, core/model.py:271-300,
utils/powerset.py, core/inference.py, pipelines/voice_activity_detection.py, pipelines/multilabel.py).

Golden vectors: tests/golden/make_golden_heads.py executes the reference's PyanNet.py and powerset.py.  On the GPU the
fp32 oracle (oracle.nets.PyanNet with the head's activation, TF32 off) is the reference for long inputs.  The weights
are synthetic (make_segmentation_state_dict(0, num_classes=K)): no trained multi-label or binary checkpoint is
available offline."""
import io
import os

import numpy as np
import pytest
import torch

from oracle import nets
from pyannote_audio_b200 import ops
from pyannote_audio_b200.core import Problem, Resolution, Segment, SlidingWindow, SlidingWindowFeature, Specifications
from pyannote_audio_b200.models import Model, PyanNet
from pyannote_audio_b200.testing import synthetic as syn
from pyannote_audio_b200.testing.checkpoints import reference_style_checkpoint

HERE = os.path.dirname(os.path.abspath(__file__))
SR = 16000
SCORE_ATOL = 1e-4
LOGP_ATOL = 3e-4
LOW_MARGIN = 1e-4          # top-2 log-probability margin under which an argmax flip is fp32 reordering noise
FP32_TWINS = ("seg_conv_impl", "seg_gemm_impl", "seg_rec_impl")
LENGTHS = {"min": (1261, 2), "5s": (80000, 2), "10s": (160000, 1)}      # as make_golden_heads.py
SEEDS = (41, 42)
GOLDEN_HEADS = {"binary": 1, "multilabel": 4, "wide": 32}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "reference_heads_vectors.npz"))


def _audio(n, batch):
    return torch.cat([syn.make_conversation(n / 16000, seed=s)[None] for s in SEEDS[:batch]])[..., :n]


def _specs(k, duration=5.0):
    """Multi-label specifications of k labels (binary for k = 1), permutation_invariant=False."""
    if k == 1:
        return Specifications(Problem.BINARY_CLASSIFICATION, Resolution.FRAME, duration, classes=["speech"])
    return Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, duration,
                          classes=[f"label#{i}" for i in range(k)])


def _powerset_specs(n, m, duration=10.0):
    return Specifications(Problem.MONO_LABEL_CLASSIFICATION, Resolution.FRAME, duration,
                          classes=[f"speaker#{i + 1}" for i in range(n)], powerset_max_classes=m,
                          permutation_invariant=True)


def _model(specs):
    m = PyanNet()
    m.specifications = specs
    m.load_state_dict(syn.make_segmentation_state_dict(0, num_classes=m.dimension))
    return m


def _oracle(k, sigmoid):
    m = nets.PyanNet(num_classes=k)
    if sigmoid:
        m.activation = torch.nn.Sigmoid()
    m.load_state_dict(syn.make_segmentation_state_dict(0, num_classes=k))
    return m.eval()


# ---- host-only ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,dimension,problem", [("seg", 7, Problem.MONO_LABEL_CLASSIFICATION),
                                                    ("seg_multilabel", 4, Problem.MULTI_LABEL_CLASSIFICATION),
                                                    ("seg_binary", 1, Problem.BINARY_CLASSIFICATION),
                                                    ("seg_powerset42", 11, Problem.MONO_LABEL_CLASSIFICATION)])
def test_checkpoints_of_every_head_load(kind, dimension, problem, golden):
    blob, sd = reference_style_checkpoint(kind)
    m = Model.from_pretrained(io.BytesIO(blob))
    assert isinstance(m, PyanNet) and m.specifications.problem is problem
    assert m.dimension == dimension and tuple(m.classifier.weight.shape) == (dimension, 128)
    assert torch.equal(m.classifier.weight, sd["classifier.weight"])
    assert sorted(m.state_dict().keys()) == list(golden["keys"])


def test_dimension_and_conversion_follow_the_specifications(golden):
    from pyannote_audio_b200.inference import Inference

    for name, k in GOLDEN_HEADS.items():
        m = _model(_specs(k))
        assert m.dimension == int(golden[f"dimension_{name}"]) == k
        inf = Inference(m)
        assert inf.conversion == "identity" and inf.duration == 5.0
    m = _model(_powerset_specs(4, 2))
    assert m.dimension == int(golden["dimension_powerset42"]) == 11
    assert Inference(m).conversion == "powerset"
    assert Inference(m, skip_conversion=True).conversion == "identity"
    # assigning specifications rebuilds the classifier, as the reference's build() does
    m.specifications = _specs(3)
    assert tuple(m.classifier.weight.shape) == (3, 128)


def test_heads_without_a_kernel_are_refused_before_device_work():
    m = PyanNet()                                          # on the CPU: a device call would fail differently
    with pytest.raises(NotImplementedError, match="32"):
        m.specifications = _specs(33)
    with pytest.raises(NotImplementedError, match="32"):
        m.specifications = _powerset_specs(6, 3)           # 42 classes
    with pytest.raises(NotImplementedError, match="REGRESSION"):
        m.specifications = Specifications(Problem.REGRESSION, Resolution.FRAME, 5.0, classes=["x"])
    assert m.dimension == 7 and tuple(m.classifier.weight.shape) == (7, 128)   # unchanged after a refusal
    with pytest.raises(ValueError, match="42 classes"):
        ops.powerset_mapping(6, 3)
    assert len(ops.powerset_mapping(31, 1)) == 32
    with pytest.raises(ValueError, match="max_per_frame"):
        ops.powerset_mapping(3, 4)
    with pytest.raises(NotImplementedError, match="trunk|community-1"):
        PyanNet(lstm={"hidden_size": 256})


def test_diarization_refuses_other_heads_before_device_work():
    from pyannote_audio_b200.models import WeSpeakerResNet34
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    for specs in (_powerset_specs(4, 2), _specs(3, duration=10.0), _powerset_specs(3, 3)):
        with pytest.raises(ValueError, match="community-1 segmentation head"):
            SpeakerDiarization(segmentation=_model(specs), embedding=WeSpeakerResNet34(),
                               clustering="AgglomerativeClustering")


def test_host_powerset_mapping_matches_the_reference(golden):
    for n, m in ((3, 2), (4, 2), (4, 3), (2, 1)):
        assert np.array_equal(ops.powerset_mapping(n, m), golden[f"mapping_{n}_{m}"])
    assert np.array_equal(ops.powerset_mapping(3, 2), nets.powerset_mapping(3, 2).numpy())


def test_oracle_matches_the_reference_heads(golden):
    """The GPU tests below use the oracle for long inputs: pin it against the reference's own PyanNet here."""
    with torch.inference_mode():
        for name, k in list(GOLDEN_HEADS.items()) + [("powerset42", 11)]:
            o = _oracle(k, sigmoid=name != "powerset42")
            for tag in ("min", "5s"):
                got = o(_audio(*LENGTHS[tag])).numpy()
                np.testing.assert_allclose(got, golden[f"{name}_{tag}"], rtol=0, atol=2e-5)


def test_vad_hyper_parameters(tmp_path, monkeypatch):
    from pyannote_audio_b200.vad import VoiceActivityDetection

    cpu = torch.device("cpu")
    vad = VoiceActivityDetection(_model(_powerset_specs(4, 2)), device=cpu)
    assert (vad.onset, vad.offset) == (0.5, 0.5)
    assert vad.default_parameters() == {"min_duration_on": 0.0, "min_duration_off": 0.0}
    vad = VoiceActivityDetection(_model(_specs(1)), device=cpu)
    with pytest.raises(NotImplementedError):
        vad.default_parameters()
    vad.instantiate({"onset": 0.7, "offset": 0.3, "min_duration_on": 0.1, "min_duration_off": 0.2})
    b = vad._binarize
    assert (b.onset, b.offset, b.min_duration_on, b.min_duration_off) == (0.7, 0.3, 0.1, 0.2)
    # a local copy of pyannote/segmentation gets the reference's tuned values (voice_activity_detection.py:131-138)
    blob, _ = reference_style_checkpoint("seg_binary")
    os.makedirs(tmp_path / "pyannote" / "segmentation")
    (tmp_path / "pyannote" / "segmentation" / "pytorch_model.bin").write_bytes(blob)
    monkeypatch.chdir(tmp_path)
    vad = VoiceActivityDetection("pyannote/segmentation", device=cpu)
    assert vad.default_parameters() == {"onset": 0.767, "offset": 0.377, "min_duration_on": 0.136,
                                        "min_duration_off": 0.067}


def test_multilabel_pipeline_parameters_and_loading(tmp_path):
    from pyannote_audio_b200.loading import Pipeline, _pipeline_class
    from pyannote_audio_b200.multilabel import MultiLabelSegmentation

    assert _pipeline_class("pyannote.audio.pipelines.MultiLabelSegmentation") is MultiLabelSegmentation
    cpu = torch.device("cpu")
    with pytest.raises(ValueError, match="must be provided"):
        MultiLabelSegmentation()
    pipe = MultiLabelSegmentation(_model(_specs(4)), device=cpu)
    assert pipe.classes() == [f"label#{i}" for i in range(4)]
    with pytest.raises(NotImplementedError):
        pipe.default_parameters()
    pipe.instantiate({"thresholds": {"label#2": {"onset": 0.8, "offset": 0.6, "min_duration_on": 0.5}}})
    b = pipe._binarize["label#2"]
    assert (b.onset, b.offset, b.min_duration_on, b.min_duration_off) == (0.8, 0.6, 0.5, 0.0)
    assert pipe._binarize["label#0"].onset == 0.5
    shared = MultiLabelSegmentation(_model(_specs(4)), share_min_duration=True, device=cpu)
    shared.instantiate({"min_duration_on": 0.25, "min_duration_off": 0.125,
                        "thresholds": {"label#1": {"onset": 0.9, "offset": 0.1}}})
    assert all(b.min_duration_on == 0.25 and b.min_duration_off == 0.125 for b in shared._binarize.values())
    with pytest.raises(ValueError, match="min_duration_on"):
        shared.instantiate({"thresholds": {"label#1": {"min_duration_on": 0.3}}})
    # Pipeline.from_pretrained on a local directory with a multi-label checkpoint
    blob, _ = reference_style_checkpoint("seg_multilabel")
    os.makedirs(tmp_path / "segmentation")
    (tmp_path / "segmentation" / "pytorch_model.bin").write_bytes(blob)
    (tmp_path / "config.yaml").write_text(
        "pipeline:\n  name: pyannote.audio.pipelines.MultiLabelSegmentation\n"
        "  params:\n    segmentation: $model/segmentation\n"
        "params:\n  thresholds:\n    music: {onset: 0.6, offset: 0.4, min_duration_on: 0.0, min_duration_off: 0.0}\n")
    pipe = Pipeline.from_pretrained(str(tmp_path), device=cpu)
    assert isinstance(pipe, MultiLabelSegmentation) and pipe.classes() == ["speech", "music", "noise", "laughter"]
    assert pipe._binarize["music"].onset == 0.6


# ---- GPU ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


class fp32_twins:
    def __init__(self, ctx):
        self.ctx = ctx

    def __enter__(self):
        for k in FP32_TWINS:
            self.ctx.set_option(k, 0)

    def __exit__(self, *exc):
        for k in FP32_TWINS:
            self.ctx.set_option(k, 1)


def _close(name, got, ref, atol=SCORE_ATOL):
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = float(np.abs(got - ref).max())
    print(f"[heads] {name}: {got.shape}, max |d| {err:.2e}")
    assert err <= atol, (name, err)


def _low_margin(ref_logp):
    top2 = np.sort(ref_logp, axis=-1)
    return (top2[..., -1] - top2[..., -2]) < LOW_MARGIN


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GOLDEN_HEADS))
def test_sigmoid_scores_match_the_reference(dev, golden, name):
    k = GOLDEN_HEADS[name]
    m = _model(_specs(k)).to(dev)
    for tag, (n, batch) in LENGTHS.items():
        wav = _audio(n, batch)
        got = m(wav).cpu().numpy()
        _close(f"K={k} {tag}", got, golden[f"{name}_{tag}"])
        with fp32_twins(m._ctx()):
            _close(f"K={k} {tag} fp32 twins", m(wav).cpu().numpy(), golden[f"{name}_{tag}"])
        # the fused maximum is the maximum of the very same scores
        ctx = m._ctx()
        flat = wav.to(dev).reshape(-1).contiguous()
        off, valid = np.arange(batch, dtype=np.int64) * n, np.full(batch, n, dtype=np.int32)
        mx = ctx.seg_forward(flat, off, valid, window=n, reduce_max=True).cpu().numpy()
        assert np.array_equal(mx, got.max(-1, keepdims=True))


@pytest.mark.gpu
def test_sigmoid_scores_on_a_30_minute_file(dev):
    """All heads share the trunk weights (make_segmentation_state_dict draws the classifier last), so the oracle runs
    the trunk once; cuDNN rejects this 106 k-frame sequence, torch's native CUDA LSTM runs it."""
    import torch.nn.functional as F

    wav = syn.make_conversation(1800.0, seed=29)[None]                                # (1, 1, 28.8 M)
    o = _oracle(7, sigmoid=False).to(dev)
    with torch.inference_mode(), torch.backends.cudnn.flags(enabled=False):
        z, _ = o.lstm(o.sincnet(wav.to(dev)).transpose(1, 2))
        for linear in o.linear:
            z = F.leaky_relu(linear(z))
    for k in (1, 4, 32):
        sd = syn.make_segmentation_state_dict(0, num_classes=k)
        with torch.inference_mode():
            ref = torch.sigmoid(F.linear(z, sd["classifier.weight"].to(dev), sd["classifier.bias"].to(dev)))
        ref = ref.cpu().numpy()
        m = _model(_specs(k)).to(dev)
        assert ref.shape == (1, m.num_frames(wav.shape[-1]), k)
        _close(f"30 min K={k}", m(wav).cpu().numpy(), ref)
        with fp32_twins(m._ctx()):
            _close(f"30 min K={k} fp32 twins", m(wav).cpu().numpy(), ref)


@pytest.mark.gpu
def test_powerset_42_head_and_generic_conversion(dev, golden):
    m = _model(_powerset_specs(4, 2)).to(dev)
    ctx = m._ctx()
    mapping = golden["mapping_4_2"]
    for tag, (n, batch) in LENGTHS.items():
        wav = _audio(n, batch)
        ref = golden[f"powerset42_{tag}"]
        for twins in (False, True):
            if twins:
                with fp32_twins(ctx):
                    got = m(wav).cpu().numpy()
            else:
                got = m(wav).cpu().numpy()
            _close(f"(4,2) {tag} twins={twins}", got, ref, atol=LOGP_ATOL)
            mism = got.argmax(-1) != ref.argmax(-1)
            assert not (mism & ~_low_margin(ref)).any()
        flat = wav.to(dev).reshape(-1).contiguous()
        off, valid = np.arange(batch, dtype=np.int64) * n, np.full(batch, n, dtype=np.int32)
        cls, logp = ctx.seg_forward(flat, off, valid, return_logp=True, window=n)
        assert torch.equal(cls, torch.argmax(logp, -1).to(torch.uint8))
        ml = ctx.powerset_to_multilabel(cls, 4, 2).cpu().numpy()
        assert np.array_equal(ml, mapping[cls.cpu().numpy()])
    # every class id (and out-of-range ids -> the empty set) for each golden mapping; the speech indicator
    for n, mm in ((3, 2), (4, 2), (4, 3), (2, 1)):
        mp = golden[f"mapping_{n}_{mm}"]
        ids = torch.arange(len(mp) + 3, dtype=torch.uint8, device=dev)
        want = np.concatenate([mp, np.zeros((3, n), np.uint8)])
        assert np.array_equal(ctx.powerset_to_multilabel(ids, n, mm).cpu().numpy(), want)
        assert np.array_equal(ctx.powerset_speech(ids, n, mm).cpu().numpy()[:, 0], want.max(-1).astype(np.float32))
    # the ABI checks (speakers, max per frame) against the class count, and the head kind of each forward
    from pyannote_audio_b200 import _lib

    ids = torch.zeros(4, dtype=torch.uint8, device=dev)
    out = torch.empty((4, 4), dtype=torch.uint8, device=dev)
    with pytest.raises(ValueError, match="has 11 classes, not 7"):
        _lib.check(ctx.lib.b200_powerset_to_multilabel_generic(ctx._h, ops._ptr(ids), 4, 7, 4, 2, ops._ptr(out),
                                                               ops._stream(dev)))
    with pytest.raises(ValueError, match="at most 32"):
        _lib.check(ctx.lib.b200_powerset_speech_generic(ctx._h, ops._ptr(ids), 4, 7, 8, 4, ops._ptr(out),
                                                        ops._stream(dev)))
    wav = _audio(16000, 1).to(dev).reshape(-1).contiguous()
    scores = torch.empty((1, ops.seg_num_frames(16000), 11), device=dev)
    with pytest.raises(ValueError, match="log-softmax"):
        _lib.check(ctx.lib.b200_seg_forward_scores(ctx._h, ops._ptr(wav), np.zeros(1, np.int64).ctypes.data,
                                                   np.full(1, 16000, np.int32).ctypes.data, 1, 16000,
                                                   ops._ptr(scores), None, ops._stream(dev)))
    s = _model(_specs(4)).to(dev)
    sctx = s._ctx()
    cls = torch.empty((1, ops.seg_num_frames(16000)), dtype=torch.uint8, device=dev)
    with pytest.raises(ValueError, match="sigmoid"):
        _lib.check(sctx.lib.b200_seg_forward_window(sctx._h, ops._ptr(wav), np.zeros(1, np.int64).ctypes.data,
                                                    np.full(1, 16000, np.int32).ctypes.data, 1, 16000, ops._ptr(cls),
                                                    None, ops._stream(dev)))
    with pytest.raises(NotImplementedError, match="33 classes"):
        big = dict(syn.make_segmentation_state_dict(0, num_classes=33))
        sctx.load_segmentation(big, _specs(4))


class _LoadWithSegLoad:
    """The ctx's library with b200_seg_load_head answered by the fixed-head b200_seg_load."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def b200_seg_load_head(self, h, w, num_classes, activation):
        assert (num_classes, activation) == (7, ops.SEG_LOGSOFTMAX)
        return self._lib.b200_seg_load(h, w)


@pytest.mark.gpu
def test_community_head_through_load_head_is_bit_identical(dev):
    from pyannote_audio_b200.inference import chunk_layout

    ctx = ops.Context(dev)
    sd = syn.make_segmentation_state_dict(0)
    wav = syn.make_conversation(41.0, seed=3)[0].to(dev)
    off, valid, _, _ = chunk_layout(wav.numel(), 160000, 16000)
    buf = torch.zeros(int(off[-1]) + 160000, device=dev)
    buf[: wav.numel()] = wav
    ctx.load_segmentation(sd)
    got = ctx.seg_forward(buf, off, valid, return_logp=True)
    lib = ctx.lib
    ctx.lib = _LoadWithSegLoad(lib)
    try:
        ctx.load_segmentation(sd)
    finally:
        ctx.lib = lib
    ref = ctx.seg_forward(buf, off, valid, return_logp=True)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    ctx.close()


def _file(seconds, seed):
    return {"waveform": syn.make_conversation(seconds, seed=seed), "sample_rate": SR, "uri": f"conv{seed}"}


def _oracle_chunks(k, file, duration, step, dev):
    """The oracle's per-chunk sigmoid scores of Inference.slide's chunks (the last one zero-padded)."""
    from oracle import pipeline as P

    W, S = int(duration * SR), int(step * SR)
    chunks = P.chunk_waveform(file["waveform"], window_size=W, step_size=S)
    o = _oracle(k, sigmoid=True).to(dev)
    with torch.inference_mode():
        return np.concatenate([o(chunks[i: i + 256].to(dev)).cpu().numpy() for i in range(0, len(chunks), 256)])


def _host_aggregate(scores, chunks_sw, frames, num_samples):
    """Inference.slide's aggregation on the host (core/inference.py:336-373): overlap-add, then the crop to the file
    when the last chunk was zero-padded."""
    from pyannote_audio_b200.inference import Inference, chunk_layout

    out = Inference.aggregate(SlidingWindowFeature(scores, chunks_sw), frames, hamming=True, missing=0.0)
    _, _, _, has_last = chunk_layout(num_samples, round(chunks_sw.duration * SR), round(chunks_sw.step * SR))
    return out.crop(Segment(0.0, num_samples / SR), mode="loose") if has_last else out.data


@pytest.mark.gpu
def test_sliding_inference_of_a_multilabel_head(dev):
    from pyannote_audio_b200.inference import Inference

    k = 4
    m = _model(_specs(k)).to(dev)
    file = _file(600.0, 7)
    num_samples = file["waveform"].shape[1]
    ref_chunks = _oracle_chunks(k, file, 5.0, 0.5, dev)
    raw = Inference(m, duration=5.0, step=0.5, skip_aggregation=True)(file)
    assert (raw.sliding_window.duration, raw.sliding_window.step) == (5.0, 0.5)
    _close("sliding 10 min per chunk", raw.data, ref_chunks)
    agg = Inference(m, duration=5.0, step=0.5)(file)          # permutation_invariant=False: aggregated
    chunks_sw = SlidingWindow(start=0.0, duration=5.0, step=0.5)

    def host(scores):
        return _host_aggregate(scores, chunks_sw, m.receptive_field, num_samples)

    assert np.array_equal(agg.data, host(raw.data))           # the device overlap-add is numpy's, bit for bit
    _close("sliding 10 min aggregated vs oracle", agg.data, host(ref_chunks))


@pytest.mark.gpu
def test_vad_and_multilabel_pipelines_with_sigmoid_heads(dev):
    from pyannote_audio_b200.inference import Inference
    from pyannote_audio_b200.multilabel import MultiLabelSegmentation
    from pyannote_audio_b200.signal import Binarize
    from pyannote_audio_b200.vad import VoiceActivityDetection

    file = _file(95.3, 11)
    num_samples = file["waveform"].shape[1]
    chunks_sw = SlidingWindow(start=0.0, duration=5.0, step=0.5)
    for k in (1, 4):
        m = _model(_specs(k)).to(dev)
        raw = Inference(m, skip_aggregation=True)(file).data                     # (C, F, k) per chunk
        ref_chunks = _oracle_chunks(k, file, 5.0, 0.5, dev)
        _close(f"K={k} chunks", raw, ref_chunks)

        def host(scores):
            return _host_aggregate(scores, chunks_sw, m.receptive_field, num_samples)

        vad = VoiceActivityDetection(m, device=dev)
        vad.instantiate({"onset": 0.6, "offset": 0.4, "min_duration_on": 0.1, "min_duration_off": 0.05})
        speech = vad.speech_scores(file)
        assert np.array_equal(speech.data, host(raw.max(-1, keepdims=True)))
        _close(f"VAD K={k} vs oracle", speech.data, host(ref_chunks.max(-1, keepdims=True)))
        want = Binarize(onset=0.6, offset=0.4, min_duration_on=0.1, min_duration_off=0.05)(
            SlidingWindowFeature(speech.data, speech.sliding_window))
        got = vad(file)
        assert [(s.start, s.end) for s, _ in got.itertracks()] == [(s.start, s.end) for s, _ in want.itertracks()]
        assert len(got) > 0 and set(got.labels()) == {"SPEECH"}
        for share in (False, True):
            pipe = MultiLabelSegmentation(m, share_min_duration=share, device=dev)
            params = {"thresholds": {lab: {"onset": 0.55 + 0.05 * i, "offset": 0.45 - 0.05 * i}
                                     for i, lab in enumerate(pipe.classes())}}
            for i, lab in enumerate(pipe.classes()):
                if share:
                    params.update(min_duration_on=0.05, min_duration_off=0.02)
                else:
                    params["thresholds"][lab].update(min_duration_on=0.1 * i, min_duration_off=0.05 * i)
            pipe.instantiate(params)
            calls = []
            ann = pipe(file, hook=lambda step, artefact, file=None, **kw: calls.append((step, artefact is None)))
            assert calls[-1] == ("segmentation", False) and ("segmentation", True) in calls
            agg = host(raw)
            expected = []
            for i, lab in enumerate(pipe.classes()):
                b = pipe._binarize[lab]
                one = Binarize(onset=b.onset, offset=b.offset, min_duration_on=b.min_duration_on,
                               min_duration_off=b.min_duration_off)(
                    SlidingWindowFeature(agg[:, i: i + 1], m.receptive_field))
                expected += [(s.start, s.end, lab) for s, _ in one.itertracks()]
            got = sorted((s.start, s.end, lab) for s, _, lab in ann.itertracks(yield_label=True))
            assert got == sorted(expected), (k, share)
            assert share or len(got) > 0, k


@pytest.mark.gpu
def test_community_and_multilabel_models_alternate_on_one_gpu(dev):
    a = PyanNet()
    a.load_state_dict(syn.make_segmentation_state_dict(0))
    a.to(dev)
    b = _model(_specs(4)).to(dev)
    wav = _audio(80000, 2)
    ra, rb = a(wav), b(wav)
    assert ra.shape[-1] == 7 and rb.shape[-1] == 4
    for _ in range(2):
        assert torch.equal(a(wav), ra)
        assert torch.equal(b(wav), rb)
    assert a._ctx() is b._ctx()
