"""SSeRiouSS (models/segmentation/SSeRiouSS.py) on the WavLM Base front end: model keys, loading and refusals on the
CPU; the CUDA forward, Inference, VoiceActivityDetection, MultiLabelSegmentation and residency next to PyanNet on the
GPU.

Golden vectors: tests/golden/make_golden_sseriouss.py executes the reference's SSeRiouSS.py with torchaudio's WavLM
Base and the synthetic weights (make_sseriouss_state_dict).  The fp32 oracle (tests/oracle_sseriouss.py) is pinned to
them here and is the reference of the GPU tests (run on the GPU with TF32 off)."""
import io
import os
import sys

import numpy as np
import pytest
import torch

from pyannote_audio_b200 import ops
from pyannote_audio_b200.core import Problem, Resolution, SlidingWindow, SlidingWindowFeature, Specifications
from pyannote_audio_b200.models import Model, PyanNet, SSeRiouSS
from pyannote_audio_b200.testing import synthetic as syn
from pyannote_audio_b200.testing.checkpoints import reference_style_checkpoint

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import oracle_sseriouss as oracle  # noqa: E402

SR = 16000
# against the fp32 oracle the fp16 (hi, lo) GEMMs and the reordered fp32 sums of 12 post-LN layers and 4 LSTM layers
# measured at most 2.4e-4 (log-probabilities) and 3.3e-4 (sigmoid scores) on an H100 80GB HBM3
LOGP_ATOL = 2e-3
SCORE_ATOL = 1e-3
LOW_MARGIN = 1e-2          # top-2 log-probability margin under which an argmax flip is accumulated rounding
# (name, wav2vec_layer, head): as make_golden_sseriouss.py
CASES = {"powerset_avg": (-1, "powerset"), "sigmoid_layer6": (6, "sigmoid")}
LENGTHS = {"min": (400, 2), "5s": (80000, 1), "10s": (160000, 1)}      # samples, batch
SEEDS = (41, 42)


def _audio(n, batch):
    return torch.cat([syn.make_conversation(max(n, SR) / SR, seed=s) for s in SEEDS[:batch]])[..., :n]


def _specs(head, duration=10.0):
    if head == "powerset":
        return Specifications(Problem.MONO_LABEL_CLASSIFICATION, Resolution.FRAME, duration,
                              classes=["speaker#1", "speaker#2", "speaker#3"], powerset_max_classes=2,
                              permutation_invariant=True)
    return Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, duration,
                          classes=["speech", "music", "noise", "laughter"])


def _state_dict(layer, head):
    return syn.make_sseriouss_state_dict(5, wav2vec_layer=layer, num_classes=7 if head == "powerset" else 4)


def _model(layer, head, duration=10.0):
    m = SSeRiouSS(wav2vec_layer=layer)
    m.specifications = _specs(head, duration)
    m.load_state_dict(_state_dict(layer, head))
    return m.eval()


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "reference_sseriouss_vectors.npz"))


# ---- CPU -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("length", ["min", "5s"])
def test_oracle_matches_the_reference(golden, case, length):
    layer, head = CASES[case]
    n, batch = LENGTHS[length]
    got = oracle.sseriouss(_state_dict(layer, head), _audio(n, batch), layer, sigmoid=head == "sigmoid").numpy()
    ref = golden[f"{case}_{length}"]
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, atol=1e-4, rtol=0)


def test_oracle_matches_torchaudio_wavlm():
    torchaudio = pytest.importorskip("torchaudio")
    sd = _state_dict(-1, "powerset")
    net = torchaudio.models.wavlm_model(**torchaudio.pipelines.WAVLM_BASE._params).eval()
    net.load_state_dict({k[len("wav2vec."):]: v for k, v in sd.items() if k.startswith("wav2vec.")})
    wav = _audio(24000, 2)
    with torch.no_grad():
        ref, _ = net.extract_features(wav)
        got = oracle.wavlm_layers(sd, wav)
    for a, b in zip(got, ref):
        torch.testing.assert_close(a, b, atol=1e-5, rtol=0)


def test_frame_arithmetic_matches_the_reference(golden):
    m = SSeRiouSS()
    for n in (400, 719, 720, 80000, 160000, 160001, 3_000_000):
        assert m.num_frames(n) == ops.ssl_num_frames(n) == 1 + (n - 400) // 320
    assert (m.receptive_field_size(1), m.receptive_field_size(2), m.receptive_field_center(0)) == \
        tuple(int(v) for v in golden["receptive_field"])
    for length, (n, _) in LENGTHS.items():
        assert m.num_frames(n) == golden[f"powerset_avg_{length}"].shape[1]


@pytest.mark.parametrize("spelling", ["parametrizations", "weight_g"])
@pytest.mark.parametrize("layer", [-1, 3])
def test_state_dict_keys_equal_the_reference_module(golden, spelling, layer):
    m = SSeRiouSS(wav2vec_layer=layer)
    keys = set(str(k) for k in golden[f"keys_layer{layer}"])
    assert set(m.state_dict()) == keys
    sd = syn.make_sseriouss_state_dict(7, wav2vec_layer=layer, pos_weight_norm=spelling)
    m.load_state_dict(sd, strict=True)
    pc = "wav2vec.encoder.transformer.pos_conv_embed.conv."
    ref = ops.fold_weight_norm(sd, pc)
    assert torch.equal(ops.fold_weight_norm(m.state_dict(), pc), ref)


def test_from_pretrained(tmp_path):
    data, sd = reference_style_checkpoint("sseriouss")
    (tmp_path / "pytorch_model.bin").write_bytes(data)
    for src in (str(tmp_path), io.BytesIO(data)):
        m = Model.from_pretrained(src)
        assert isinstance(m, SSeRiouSS) and m.dimension == 4 and m.hparams.wav2vec == "WAVLM_BASE"
        assert m.specifications.problem == Problem.MULTI_LABEL_CLASSIFICATION
        own = m.state_dict()
        assert torch.equal(own["wav2vec.encoder.transformer.pos_conv_embed.conv.parametrizations.weight.original1"],
                           sd["wav2vec.encoder.transformer.pos_conv_embed.conv.weight_v"])
        assert torch.equal(own["classifier.weight"], sd["classifier.weight"])
    assert isinstance(SSeRiouSS.from_pretrained(io.BytesIO(data)), SSeRiouSS)
    with pytest.raises(ValueError):
        PyanNet.from_pretrained(io.BytesIO(data))


def test_unsupported_configurations_and_short_windows_are_refused_before_device_work():
    for kw in ({"wav2vec": "WAVLM_LARGE"}, {"wav2vec": "WAV2VEC2_BASE"}, {"wav2vec": "HUBERT_BASE"},
               {"wav2vec": {"encoder_embed_dim": 768}}, {"wav2vec": "/some/checkpoint.pt"},
               {"lstm": {"hidden_size": 256}}, {"lstm": {"num_layers": 5}}, {"lstm": {"monolithic": False}},
               {"lstm": {"bidirectional": False}}, {"linear": {"num_layers": 3}}):
        with pytest.raises(NotImplementedError):
            SSeRiouSS(**kw)
    for layer in (0, 13):
        with pytest.raises(ValueError):
            SSeRiouSS(wav2vec_layer=layer)
    with pytest.raises(ValueError):
        SSeRiouSS(sample_rate=8000)
    m = SSeRiouSS()
    with pytest.raises(NotImplementedError):
        m.specifications = Specifications(Problem.MULTI_LABEL_CLASSIFICATION, Resolution.FRAME, 5.0,
                                          classes=[f"l{i}" for i in range(33)])
    with pytest.raises(ValueError, match="at least 400 samples"):
        m(torch.zeros(1, 1, 399))                   # the model is on the CPU: the check comes before any device
    from pyannote_audio_b200.inference import Inference

    inf = Inference(m, duration=0.02, step=0.01)
    with pytest.raises(ValueError, match="at least 400 samples"):
        inf.slide_device(torch.zeros(1, 16000), SR)
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    with pytest.raises(ValueError):
        SpeakerDiarization(segmentation=m)


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


def _compare(name, got, ref, head):
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = float(np.abs(got - ref).max())
    print(f"[sseriouss] {name}: {got.shape}, max |d| {err:.2e}")
    assert err <= (SCORE_ATOL if head == "sigmoid" else LOGP_ATOL), (name, err)
    if head == "powerset":
        top2 = np.sort(ref, axis=-1)
        low = (top2[..., -1] - top2[..., -2]) < LOW_MARGIN
        flips = (got.argmax(-1) != ref.argmax(-1)) & ~low
        assert not flips.any(), (name, int(flips.sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_forward_matches_the_oracle(dev, case):
    layer, head = CASES[case]
    m = _model(layer, head).to(dev)
    sd = _state_dict(layer, head)
    for length, (n, batch) in LENGTHS.items():
        wav = _audio(n, batch)
        got = m(wav[:, None].to(dev)).cpu().numpy()
        ref = oracle.sseriouss(sd, wav, layer, sigmoid=head == "sigmoid", device=dev).numpy()
        _compare(f"{case} {length}", got, ref, head)


@pytest.mark.gpu
def test_batch_invariance_across_sub_batches(dev):
    m = _model(-1, "powerset").to(dev)
    wav = _audio(160000, 2)
    wav = torch.cat([wav, wav.flip(-1)[:1]]).to(dev)          # 3 windows
    ctx = m._ctx()
    batched = m(wav[:, None]).cpu()
    alone = torch.cat([m(wav[i: i + 1, None]).cpu() for i in range(3)])
    assert torch.equal(batched, alone)
    ctx.set_option("ssl_max_batch", 1)                         # one 10 s window per sub-batch
    try:
        split = m(wav[:, None]).cpu()
        with pytest.raises(ValueError, match="ssl_max_batch"):
            m(torch.zeros(1, 1, 160001, device=dev))
    finally:
        ctx.set_option("ssl_max_batch", 32)
    assert torch.equal(batched, split)
    # a window longer than the default budget (32 x 10 s) is refused, naming the option
    with pytest.raises(ValueError, match="ssl_max_batch"):
        m(torch.zeros(1, 1, 32 * 160000 + 1, device=dev))


def _oracle_chunks(sd, layer, head, wav, window, step, dev):
    """The reference's sliding-window chunks (zero-padded last chunk) through the oracle -> (C, F, K)."""
    from pyannote_audio_b200.inference import chunk_layout

    n = wav.shape[-1]
    off, valid, _, _ = chunk_layout(n, window, step)
    padded = torch.zeros(int(off[-1]) + window)
    padded[:n] = wav
    chunks = torch.stack([padded[o: o + window] for o in off])
    outs = [oracle.sseriouss(sd, chunks[i: i + 32], layer, sigmoid=head == "sigmoid", device=dev)
            for i in range(0, len(chunks), 32)]
    return torch.cat(outs).numpy()


@pytest.mark.gpu
def test_pipelines_match_the_oracle(dev):
    from pyannote_audio_b200.inference import Inference
    from pyannote_audio_b200.multilabel import MultiLabelSegmentation
    from pyannote_audio_b200.signal import Binarize
    from pyannote_audio_b200.vad import VoiceActivityDetection

    layer, head = CASES["sigmoid_layer6"]
    sd = _state_dict(layer, head)
    m = _model(layer, head, duration=10.0).to(dev)
    wav = syn.make_conversation(185.3, seed=11)
    file = {"waveform": wav, "sample_rate": SR, "uri": "conversation"}
    raw = Inference(m, skip_aggregation=True)(file).data                          # 10 s windows, 1 s step
    ref = _oracle_chunks(sd, layer, head, wav[0], 160000, 16000, dev)
    _compare("sliding chunks", raw, ref, head)
    agg = Inference(m)(file)
    chunks_sw = SlidingWindow(start=0.0, duration=10.0, step=1.0)
    ref_agg = Inference.aggregate(SlidingWindowFeature(ref, chunks_sw), m.receptive_field, hamming=True,
                                  missing=0.0)
    n = len(agg.data)                          # Inference crops to the file, the padded last chunk reaches past it
    _compare("aggregated", agg.data[:n], ref_agg.data[:n], head)
    vad = VoiceActivityDetection(m, device=dev)
    vad.instantiate({"onset": 0.6, "offset": 0.4, "min_duration_on": 0.1, "min_duration_off": 0.05})
    speech = vad.speech_scores(file)
    ref_speech = Inference.aggregate(SlidingWindowFeature(ref.max(-1, keepdims=True), chunks_sw), m.receptive_field,
                                     hamming=True, missing=0.0)
    _compare("VAD speech scores", speech.data[:n], ref_speech.data[:n], head)
    got = vad(file)
    want = Binarize(onset=0.6, offset=0.4, min_duration_on=0.1, min_duration_off=0.05)(speech)
    assert [(s.start, s.end) for s, _ in got.itertracks()] == [(s.start, s.end) for s, _ in want.itertracks()]
    pipe = MultiLabelSegmentation(m, device=dev)
    pipe.instantiate({"thresholds": {lab: {"onset": 0.5, "offset": 0.5, "min_duration_on": 0.0,
                                           "min_duration_off": 0.0} for lab in pipe.classes()}})
    ann = pipe(file)
    expected = []
    for i, lab in enumerate(pipe.classes()):
        one = Binarize(onset=0.5, offset=0.5)(SlidingWindowFeature(agg.data[:, i: i + 1], agg.sliding_window))
        expected += [(s.start, s.end, lab) for s, _ in one.itertracks()]
    assert sorted((s.start, s.end, lab) for s, _, lab in ann.itertracks(yield_label=True)) == sorted(expected)
    # whole-window inference of a multi-minute file: one window of the whole file
    whole = Inference(m, window="whole")
    short = {"waveform": wav[:, : 150 * SR], "sample_rate": SR}
    got = whole(short)
    ref_whole = oracle.sseriouss(sd, wav[:, : 150 * SR], layer, sigmoid=True, device=dev).numpy()[0]
    _compare("whole 150 s window", got, ref_whole, head)


@pytest.mark.gpu
def test_pyannet_and_sseriouss_stay_resident_side_by_side(dev):
    p = PyanNet().to(dev)
    p.load_state_dict(syn.make_segmentation_state_dict(0))
    s = _model(-1, "powerset").to(dev)
    wav = _audio(160000, 2)[:, None].to(dev)
    a0 = p(wav).cpu()
    b0 = s(wav).cpu()
    ctx = p._ctx()
    assert ctx is s._ctx() and ctx.seg_loaded and ctx.ssl_loaded
    launches = ctx.launch_count
    a1 = p(wav).cpu()
    b1 = s(wav).cpu()
    a2 = p(wav).cpu()
    assert torch.equal(a0, a1) and torch.equal(a0, a2) and torch.equal(b0, b1)
    assert ctx.owners["seg"][0] == p._model_id and ctx.owners["ssl"][0] == s._model_id
    assert ctx.launch_count > launches
