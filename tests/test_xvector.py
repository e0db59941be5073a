"""XVectorSincNet (models/embedding/xvector.py:205-349), the architecture of pyannote/embedding.  CPU: the fp32 oracle
against the reference's own xvector.py (golden vectors), the state-dict keys, the frame arithmetic, checkpoint loading
and the activation range of the synthetic weights.  GPU: the CUDA path (SincNet, TDNN implicit GEMMs, pooling, Linear)
against the fp32 oracle run on the GPU with TF32 off, its batching invariances, and the pipelines on top of it."""
import os

import numpy as np
import pytest
import torch
import yaml

from oracle_xvector import XVectorSincNet as OracleXVector
from oracle_xvector import receptive_field_center, receptive_field_size
from pyannote_audio_b200 import synthetic as syn
from pyannote_audio_b200.testing.checkpoints import reference_style_checkpoint

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_xvector_vectors.npz")
LENGTHS = {"min": 4771, "odd": 36800, "10s": 160000}


def _cos_dist(a, b):
    return 1 - (a * b).sum(-1) / np.maximum(np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1), 1e-30)


def _wav(n, seeds=(11, 12)):
    """(len(seeds), 1, n) synthetic speech, as tests/golden/make_golden_xvector.py cuts it."""
    return torch.cat([syn.make_conversation(n / 16000, seed=s)[None] for s in seeds])[..., :n]


def _oracle(device="cpu"):
    m = OracleXVector()
    m.load_state_dict(syn.make_xvector_state_dict(3))
    return m.eval().to(device)


# ---- CPU ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(LENGTHS))
def test_oracle_matches_reference_module(name):
    golden = np.load(GOLDEN)
    net, wav = _oracle(), _wav(LENGTHS[name])
    w2, w3 = torch.from_numpy(golden[f"w2_{name}"]), torch.from_numpy(golden[f"w3_{name}"])
    with torch.inference_mode():
        got = {"emb": net(wav), "emb_w2": net(wav, weights=w2), "emb_w3": net(wav, weights=w3)}
    for key, value in got.items():
        # 4771 samples give one TDNN frame: the unweighted std (correction=1) is NaN there, as in the reference
        np.testing.assert_allclose(value.numpy(), golden[f"{key}_{name}"], rtol=0, atol=2e-5, equal_nan=True)


def test_state_dict_keys_are_the_reference_ones():
    from pyannote_audio_b200.models import XVectorSincNet

    ref_keys = list(np.load(GOLDEN)["keys"])
    assert sorted(XVectorSincNet().state_dict()) == ref_keys
    assert sorted(syn.make_xvector_state_dict(3)) == ref_keys
    assert sorted(OracleXVector().state_dict()) == ref_keys


def test_frame_arithmetic_is_the_reference_one():
    from pyannote_audio_b200.models import XVectorSincNet

    golden = np.load(GOLDEN)
    m = XVectorSincNet()
    assert [m.num_frames(int(n)) for n in golden["lengths"]] == list(golden["num_frames"])
    assert [m.receptive_field_size(k) for k in (1, 2, 10)] == list(golden["rf_size"])
    assert [receptive_field_size(k) for k in (1, 2, 10)] == list(golden["rf_size"])
    assert [m.receptive_field_center(k) for k in (0, 1, 10)] == list(golden["rf_center"])
    assert [receptive_field_center(k) for k in (0, 1, 10)] == list(golden["rf_center"])
    rf = m.receptive_field
    size, step = int(golden["rf_size"][0]), int(golden["rf_size"][1] - golden["rf_size"][0])
    assert (rf.duration, rf.step) == (size / 16000, step / 16000)
    assert rf.start == (int(golden["rf_center"][0]) - (size - 1) / 2) / 16000
    # the reference's conv raises at 4770 samples and not at 4771: the shortest input is 4771 samples
    assert list(golden["raises_4770_4771"]) == [1, 0]
    assert m.min_num_samples == 4771 and m.num_frames(4771) == 1


def test_from_pretrained_and_pipeline_config(tmp_path):
    from pyannote_audio_b200.loading import get_model, resolve_pipeline
    from pyannote_audio_b200.models import Model, WeSpeakerResNet34, XVectorSincNet
    from pyannote_audio_b200.speaker_verification import SpeakerEmbedding

    blob, sd = reference_style_checkpoint("xvec")
    path = tmp_path / "pytorch_model.bin"
    path.write_bytes(blob)
    for klass in (Model, XVectorSincNet):
        m = klass.from_pretrained(str(path))
        assert type(m) is XVectorSincNet and not m.training and m.dimension == 512
        assert m.specifications.duration == 3.0
        assert torch.equal(m.state_dict()["tdnns.12.weight"], sd["tdnns.12.weight"])
    with pytest.raises(ValueError, match="not a WeSpeakerResNet34"):
        WeSpeakerResNet34.from_pretrained(str(path))
    root = tmp_path / "embedding-pipeline"
    (root / "embedding").mkdir(parents=True)
    (root / "embedding" / "pytorch_model.bin").write_bytes(blob)
    config = {"version": "4.0.0", "pipeline": {"name": "pyannote.audio.pipelines.SpeakerEmbedding",
                                               "params": {"embedding": "$model/embedding"}}}
    (root / "config.yaml").write_text(yaml.dump(config))
    klass, params, _ = resolve_pipeline(root)
    assert klass is SpeakerEmbedding
    emb = get_model(params["embedding"])
    assert type(emb) is XVectorSincNet and emb.num_frames(160000) == 575


def test_unsupported_hyper_parameters_and_diarization_refuse():
    from pyannote_audio_b200.models import PyanNet, XVectorSincNet
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    with pytest.raises(NotImplementedError, match="stride 10"):
        XVectorSincNet(sincnet={"stride": 5})
    with pytest.raises(NotImplementedError, match="16 kHz"):
        XVectorSincNet(sample_rate=8000)
    # the diarization pipeline's fused chunk path and PLDA are specific to the 256-d WeSpeaker models
    with pytest.raises(ValueError, match="WeSpeaker"):
        SpeakerDiarization(segmentation=PyanNet(), embedding=XVectorSincNet())


def test_synthetic_weights_keep_activations_in_range():
    """Activation RMS after every TDNN layer within [0.1, 10] and max |x| < 1e3 (far below the fp16 limit the
    (hi, lo) activations between layers are stored in) on 10 s of synthetic speech."""
    with torch.inference_mode():
        _, per_layer = _oracle().frames(syn.make_conversation(10.0, seed=7)[None])
    assert len(per_layer) == 5
    rms = np.array([float(x.pow(2).mean().sqrt()) for x in per_layer])
    peak = max(float(x.abs().max()) for x in per_layer)
    assert rms.min() >= 0.1 and rms.max() <= 10 and peak < 1e3, (rms, peak)


# ---- GPU ------------------------------------------------------------------------------------------------
COS_BAR, ABS_BAR = 1e-5, 1e-4      # cosine distance, max |diff| relative to max |e|


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def model(dev):
    from pyannote_audio_b200.models import XVectorSincNet

    m = XVectorSincNet()
    m.load_state_dict(syn.make_xvector_state_dict(3))
    return m.to(dev)


@pytest.fixture(scope="module")
def oracle(dev):
    return _oracle(dev)


def _check(got, ref, what, abs_bar=ABS_BAR):
    got, ref = got.detach().cpu().double().numpy(), ref.detach().cpu().double().numpy()
    cos = float(np.nanmax(_cos_dist(got, ref)))
    rel = float(np.nanmax(np.abs(got - ref)) / np.nanmax(np.abs(ref)))
    print(f"{what}: cos dist {cos:.2e}, max|d|/max|e| {rel:.2e}")
    assert np.array_equal(np.isnan(got), np.isnan(ref)), what
    assert cos <= COS_BAR and rel <= abs_bar, (what, cos, rel)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4771, 36817, 160000, 30 * 60 * 16000])
def test_forward_matches_oracle(model, oracle, dev, n):
    b = 1 if n > 160000 else 3
    wav = _wav(n, seeds=tuple(range(20, 20 + b))).to(dev)
    T = model.num_frames(n)
    g = torch.Generator().manual_seed(n)
    weights = {"none": None,
               "binary": (torch.rand(b, T, generator=g) > 0.4).float(),
               "soft": torch.rand(b, T, generator=g),
               "3d": torch.rand(b, 3, T + 11, generator=g) * (torch.rand(b, 3, T + 11, generator=g) > 0.3)}
    with torch.inference_mode():
        for kind, w in weights.items():
            if n == 4771 and kind == "none":
                continue                      # one frame: std with correction=1 is NaN, checked below
            wd = None if w is None else w.to(dev)
            # One TDNN frame with a soft weight w: StatsPool's std is sqrt(w (x - mean)^2 / (v1 - w^2 / v1 + 1e-8))
            # with v1 = w + 1e-8, a ratio of two rounding residues of fp32 arithmetic in any implementation, so those
            # 1500 std inputs of the Linear are noise of ~1e-3 |x| and the embeddings differ by ~1e-4 max|e| (the
            # direction still agrees to a cosine distance of ~1e-8).  Every other case keeps the 1e-4 bar.
            bar = 1e-3 if n == 4771 and kind in ("soft", "3d") else ABS_BAR
            _check(model(wav, weights=wd), oracle(wav, weights=wd), f"{n} samples, {kind} weights", abs_bar=bar)
        if n == 4771:
            e = model(wav).cpu()
            assert torch.isnan(e).any(dim=-1).all()


@pytest.mark.gpu
def test_sub_batches_and_repeats_are_bit_identical(model, dev):
    from pyannote_audio_b200.models import get_context

    ctx = get_context(dev)
    wav = _wav(48000, seeds=tuple(range(40, 45))).to(dev)
    w = torch.rand(5, 2, 37, generator=torch.Generator().manual_seed(3)).to(dev)
    default = int(os.environ.get("B200_EMB_MAX_BATCH", 264))
    outs = []
    try:
        # a sub-batch holds emb_max_batch x 160000 samples: 1 -> 3 utterances of 48000 per sub-batch
        for mb in (1, 2, default):
            ctx.set_option("emb_max_batch", mb)
            outs.append(model(wav, weights=w))
    finally:
        ctx.set_option("emb_max_batch", default)
    assert all(torch.equal(outs[0], o) for o in outs[1:])
    assert torch.equal(model(wav, weights=w), model(wav, weights=w))


@pytest.mark.gpu
def test_inference_whole_and_sliding(model, oracle, dev):
    from pyannote_audio_b200.core import Segment
    from pyannote_audio_b200.inference import Inference

    wav = syn.make_conversation(64.3, seed=9)
    file = {"waveform": wav, "sample_rate": 16000}
    with torch.inference_mode():
        whole = Inference(model, window="whole")
        _check(torch.from_numpy(np.asarray(whole(file)))[None], oracle(wav[None].to(dev)), "whole file")
        crop = whole.crop(file, Segment(3.0, 17.5))
        _check(torch.from_numpy(np.asarray(crop))[None], oracle(wav[None, :, 48000:280000].to(dev)), "whole crop")
        out = Inference(model, window="sliding", duration=3.0, step=1.0)(file)
        n, win = wav.shape[1], 48000
        offs = list(range(0, n - win + 1, 16000))
        if (n - win) % 16000:
            offs.append(offs[-1] + 16000)              # the last chunk, zero-padded to the full window
        padded = torch.zeros(1, offs[-1] + win)
        padded[:, :n] = wav
        chunks = torch.stack([padded[:, o:o + win] for o in offs]).to(dev)
        assert out.data.shape == (len(offs), 512)
        _check(torch.from_numpy(out.data), oracle(chunks), "sliding 3 s / 1 s")


@pytest.mark.gpu
def test_pretrained_speaker_embedding_with_masks(model, oracle, dev):
    from pyannote_audio_b200.pipeline import PretrainedSpeakerEmbedding

    pse = PretrainedSpeakerEmbedding(model, device=dev)
    assert pse.min_num_samples == 4771 and pse.dimension == 512
    wav = _wav(80000, seeds=(1, 2, 3)).to(dev)
    masks = (torch.rand(3, 589, generator=torch.Generator().manual_seed(5)) > 0.3).float().to(dev)
    with torch.inference_mode():
        _check(torch.from_numpy(pse(wav, masks=masks)), oracle(wav, weights=masks), "PretrainedSpeakerEmbedding")


@pytest.mark.gpu
def test_speaker_embedding_pipeline(model, oracle, dev):
    from pyannote_audio_b200.models import PyanNet
    from pyannote_audio_b200.speaker_verification import SpeakerEmbedding

    wav = syn.make_conversation(21.7, seed=4)
    file = {"waveform": wav, "sample_rate": 16000}
    with torch.inference_mode():
        plain = SpeakerEmbedding(embedding=model, device=dev)(file)
        _check(torch.from_numpy(plain), oracle(wav[None].to(dev)), "SpeakerEmbedding")
        seg = PyanNet()
        seg.load_state_dict(syn.make_segmentation_state_dict(0), strict=False)
        pipe = SpeakerEmbedding(embedding=model, segmentation=seg, device=dev)
        weights = torch.from_numpy(pipe.speech_weights(file))[None].to(dev)
        _check(torch.from_numpy(pipe(file)), oracle(wav[None].to(dev), weights=weights), "SpeakerEmbedding + VAD")


@pytest.mark.gpu
def test_weight_slots_are_independent(model, dev):
    from pyannote_audio_b200.models import PyanNet, WeSpeakerResNet34, XVectorSincNet

    seg, emb = PyanNet(), WeSpeakerResNet34()
    seg.load_state_dict(syn.make_segmentation_state_dict(0), strict=False)
    emb.load_state_dict(syn.make_embedding_state_dict(1), strict=False)
    seg, emb = seg.to(dev), emb.to(dev)
    wav = _wav(160000, seeds=(6, 7)).to(dev)
    with torch.inference_mode():
        alone = [seg(wav), emb(wav), model(wav)]
        mixed = [model(wav), seg(wav), emb(wav), model(wav)]
        assert torch.equal(mixed[0], alone[2]) and torch.equal(mixed[3], alone[2])
        assert torch.equal(mixed[1], alone[0]) and torch.equal(mixed[2], alone[1])
        other = XVectorSincNet().to(dev)
        other.load_state_dict(syn.make_xvector_state_dict(3))
        base = other(wav)
        assert torch.equal(base, alone[2])
        other.load_state_dict(syn.make_xvector_state_dict(4))     # after a forward: the new weights are uploaded
        assert not torch.equal(other(wav), base)
        assert torch.equal(model(wav), alone[2])


@pytest.mark.gpu
def test_errors(model, dev):
    from pyannote_audio_b200.models import get_context

    with pytest.raises(ValueError, match="4771"):
        model(torch.zeros(1, 1, 4770, device=dev))
    with pytest.raises(ValueError, match="mono"):
        model(torch.zeros(1, 2, 16000, device=dev))
    ctx = get_context(dev)
    default = int(os.environ.get("B200_EMB_MAX_BATCH", 264))
    try:
        ctx.set_option("emb_max_batch", 1)
        with pytest.raises(ValueError, match="emb_max_batch to at least 2"):
            model(torch.zeros(1, 1, 200000, device=dev))
    finally:
        ctx.set_option("emb_max_batch", default)
