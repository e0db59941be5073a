"""XVectorMFCC (models/embedding/xvector.py:42-202): the x-vector TDNN stack behind torchaudio's MFCC.  CPU: the fp32
oracle against the reference's own xvector.py (golden vectors), the state-dict keys, the frame arithmetic, checkpoint
loading, the refused configurations and the activation range of the synthetic weights.  GPU: the CUDA path (MFCC front
end, TDNN implicit GEMMs, pooling, Linear) and the front end alone against the fp32 oracle run on the GPU with TF32 off,
the per-utterance top_db, and the pipelines on top of it."""
import os

import numpy as np
import pytest
import torch
import yaml

from oracle_xvector import XVectorSincNet as OracleXVectorSincNet
from oracle_xvector_mfcc import XVectorMFCC as OracleXVectorMFCC
from oracle_xvector_mfcc import num_frames, receptive_field_center, receptive_field_size
from pyannote_audio_b200 import synthetic as syn
from pyannote_audio_b200.testing.checkpoints import reference_style_checkpoint

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_xvector_mfcc_vectors.npz")
LENGTHS = {"min": 2800, "odd": 36817, "10s": 160000}


def _cos_dist(a, b):
    return 1 - (a * b).sum(-1) / np.maximum(np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1), 1e-30)


def _wav(n, seeds=(11, 12)):
    """(len(seeds), 1, n) synthetic speech, as tests/golden/make_golden_xvector_mfcc.py cuts it."""
    return torch.cat([syn.make_conversation(n / 16000, seed=s)[None] for s in seeds])[..., :n]


def _oracle(device="cpu"):
    m = OracleXVectorMFCC()
    m.load_state_dict(syn.make_xvector_mfcc_state_dict(5))
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
        # 2800 samples give one TDNN frame: the unweighted std (correction=1) is NaN there, as in the reference
        np.testing.assert_allclose(value.numpy(), golden[f"{key}_{name}"], rtol=0, atol=2e-5, equal_nan=True)


def test_state_dict_keys_and_buffers_are_the_reference_ones():
    import torchaudio

    from pyannote_audio_b200.models import XVectorMFCC

    ref_keys = list(np.load(GOLDEN)["keys"])
    assert sorted(XVectorMFCC().state_dict()) == ref_keys
    assert sorted(syn.make_xvector_mfcc_state_dict(5)) == ref_keys
    assert sorted(OracleXVectorMFCC().state_dict()) == ref_keys
    # the default buffers are torchaudio's, bit for bit
    ta = torchaudio.transforms.MFCC(sample_rate=16000, n_mfcc=40, dct_type=2, norm="ortho", log_mels=False)
    ours = XVectorMFCC().state_dict()
    for key, value in ta.state_dict().items():
        assert torch.equal(ours["mfcc." + key], value), key


def test_frame_arithmetic_is_the_reference_one():
    from pyannote_audio_b200.models import XVectorMFCC

    golden = np.load(GOLDEN)
    m = XVectorMFCC()
    assert [m.num_frames(int(n)) for n in golden["lengths"]] == list(golden["num_frames"])
    assert [num_frames(int(n)) for n in golden["lengths"]] == list(golden["num_frames"])
    assert [m.receptive_field_size(k) for k in (1, 2, 10)] == list(golden["rf_size"])
    assert [receptive_field_size(k) for k in (1, 2, 10)] == list(golden["rf_size"])
    assert [m.receptive_field_center(k) for k in (0, 1, 10)] == list(golden["rf_center"])
    assert [receptive_field_center(k) for k in (0, 1, 10)] == list(golden["rf_center"])
    rf = m.receptive_field
    size, step = int(golden["rf_size"][0]), int(golden["rf_size"][1] - golden["rf_size"][0])
    assert (rf.duration, rf.step) == (size / 16000, step / 16000)
    assert rf.start == (int(golden["rf_center"][0]) - (size - 1) / 2) / 16000
    # the reference's conv raises at 2799 samples and not at 2800: the shortest input is 2800 samples
    assert list(golden["raises_2799_2800"]) == [1, 0]
    assert m.min_num_samples == 2800 and m.num_frames(2800) == 1 and m.num_frames(160000) == 787


def test_from_pretrained_and_pipeline_config(tmp_path):
    from pyannote_audio_b200.loading import get_model, resolve_pipeline
    from pyannote_audio_b200.models import Model, XVectorMFCC, XVectorSincNet
    from pyannote_audio_b200.speaker_verification import SpeakerEmbedding

    blob, sd = reference_style_checkpoint("xvec_mfcc")
    path = tmp_path / "pytorch_model.bin"
    path.write_bytes(blob)
    for klass in (Model, XVectorMFCC):
        m = klass.from_pretrained(str(path))
        assert type(m) is XVectorMFCC and not m.training and m.dimension == 512
        assert m.specifications.duration == 3.0
        assert torch.equal(m.state_dict()["tdnns.0.weight"], sd["tdnns.0.weight"])
        assert torch.equal(m.state_dict()["mfcc.MelSpectrogram.mel_scale.fb"], sd["mfcc.MelSpectrogram.mel_scale.fb"])
    with pytest.raises(ValueError, match="not a XVectorSincNet"):
        XVectorSincNet.from_pretrained(str(path))
    root = tmp_path / "embedding-pipeline"
    (root / "embedding").mkdir(parents=True)
    (root / "embedding" / "pytorch_model.bin").write_bytes(blob)
    config = {"version": "4.0.0", "pipeline": {"name": "pyannote.audio.pipelines.SpeakerEmbedding",
                                               "params": {"embedding": "$model/embedding"}}}
    (root / "config.yaml").write_text(yaml.dump(config))
    klass, params, _ = resolve_pipeline(root)
    assert klass is SpeakerEmbedding
    emb = get_model(params["embedding"])
    assert type(emb) is XVectorMFCC and emb.num_frames(160000) == 787


@pytest.mark.parametrize("kwargs", [
    {"mfcc": {"n_mfcc": 20}}, {"mfcc": {"dct_type": 3}}, {"mfcc": {"norm": None}}, {"mfcc": {"log_mels": True}},
    {"mfcc": {"melkwargs": {"n_mels": 64}}}, {"sample_rate": 8000}, {"num_channels": 2}])
def test_unsupported_configurations_refuse_before_device_work(kwargs):
    from pyannote_audio_b200.models import XVectorMFCC

    with pytest.raises(NotImplementedError, match="default MFCC"):
        XVectorMFCC(**kwargs)


def test_defaults_spelled_out_are_accepted_and_diarization_refuses():
    from pyannote_audio_b200.models import PyanNet, XVectorMFCC
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    m = XVectorMFCC(mfcc={"n_mfcc": 40, "dct_type": 2, "norm": "ortho", "log_mels": False, "sample_rate": 16000,
                          "melkwargs": None})
    assert m.hparams.mfcc == {"n_mfcc": 40, "dct_type": 2, "norm": "ortho", "log_mels": False, "sample_rate": 16000}
    # the diarization pipeline's fused chunk path and PLDA are specific to the 256-d WeSpeaker models
    with pytest.raises(ValueError, match="WeSpeaker"):
        SpeakerDiarization(segmentation=PyanNet(), embedding=XVectorMFCC())


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
# Front end: max |diff| relative to the utterance's max |coefficient|.  Measured on an H100: at most 1.0e-4 (2800
# samples; 7e-5 at 36817 and 160000; 0 on silence).  The DFT runs on fp16 (hi, lo) operands (22 significant bits),
# whose error, ~1e-7 of a frame's energy, is a visible share of the filters that lie 60-80 dB below it in dB.
MFCC_BAR = 3e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def model(dev):
    from pyannote_audio_b200.models import XVectorMFCC

    m = XVectorMFCC()
    m.load_state_dict(syn.make_xvector_mfcc_state_dict(5))
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
@pytest.mark.parametrize("n", [2800, 36817, 160000, 30 * 60 * 16000])
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
            if n == 2800 and kind == "none":
                continue                      # one frame: std with correction=1 is NaN, checked below
            wd = None if w is None else w.to(dev)
            # One TDNN frame with a soft weight: StatsPool's std divides one fp32 rounding residue by another in any
            # implementation (see test_xvector.py), so that case has a 1e-3 bar.
            bar = 1e-3 if n == 2800 and kind in ("soft", "3d") else ABS_BAR
            _check(model(wav, weights=wd), oracle(wav, weights=wd), f"{n} samples, {kind} weights", abs_bar=bar)
        if n == 2800:
            assert torch.isnan(model(wav).cpu()).any(dim=-1).all()


def _check_mfcc(got, ref, what):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    rel = ((got - ref).abs().amax(dim=(1, 2)) / ref.abs().amax(dim=(1, 2))).max().item()
    print(f"{what}: max|d|/max|c| {rel:.2e}")
    assert rel <= MFCC_BAR, (what, rel)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2800, 36817, 160000])
def test_mfcc_front_end_matches_torchaudio(model, oracle, dev, n):
    """The front end alone on a batch of a normal, a 60 dB quieter (each clamped at its own max - 80 dB) and a
    half-silent utterance (its silent frames are -100 dB in every filter before the clamp)."""
    wav = _wav(n, seeds=(30, 31, 32))
    wav[1] *= 1e-3
    wav[2, :, n // 2:] = 0.0
    with torch.inference_mode():
        _check_mfcc(model.mfcc_features(wav.to(dev)), oracle.mfcc(wav.to(dev)).squeeze(1), f"MFCC of {n} samples")


@pytest.mark.gpu
def test_silent_utterance(model, oracle, dev):
    wav = torch.zeros(2, 1, 48000, device=dev)
    with torch.inference_mode():
        feats, ref = model.mfcc_features(wav), oracle.mfcc(wav).squeeze(1)
        # every filter at -100 dB: c0 = -100 * sqrt(128), the other coefficients -100 * sqrt(2 / 128) * sum of cosines
        _check_mfcc(feats, ref, "MFCC of silence")
        assert torch.equal(feats[:, :, :1].expand_as(feats), feats)
        _check(model(wav), oracle(wav), "silence")


@pytest.mark.gpu
def test_top_db_is_per_utterance(model, oracle, dev):
    """An utterance gives the same bits alone and inside a batch of louder and quieter ones (AmplitudeToDB's top_db
    reference is its own maximum), and sub-batch sizes do not change any bit."""
    from pyannote_audio_b200.models import get_context

    wav = _wav(48000, seeds=(40, 41, 42, 43, 44)).to(dev)
    wav[1] *= 1e-4
    wav[3] *= 30.0
    w = torch.rand(5, 2, 37, generator=torch.Generator().manual_seed(3)).to(dev)
    with torch.inference_mode():
        batch = model(wav, weights=w)
        for i in range(5):
            assert torch.equal(model(wav[i:i + 1], weights=w[i:i + 1]), batch[i:i + 1]), i
        _check(batch, oracle(wav, weights=w), "loud and quiet batch")
        ctx = get_context(dev)
        default = int(os.environ.get("B200_EMB_MAX_BATCH", 264))
        try:
            for mb in (1, 2):            # 3 and 6 utterances of 48000 samples per sub-batch
                ctx.set_option("emb_max_batch", mb)
                assert torch.equal(model(wav, weights=w), batch)
        finally:
            ctx.set_option("emb_max_batch", default)


@pytest.mark.gpu
def test_inference_whole_and_sliding(model, oracle, dev):
    from pyannote_audio_b200.inference import Inference

    wav = syn.make_conversation(64.3, seed=9)
    file = {"waveform": wav, "sample_rate": 16000}
    with torch.inference_mode():
        whole = Inference(model, window="whole")
        _check(torch.from_numpy(np.asarray(whole(file)))[None], oracle(wav[None].to(dev)), "whole file")
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
    assert pse.min_num_samples == 2800 and pse.dimension == 512
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
def test_both_xvector_models_stay_resident(model, dev):
    from pyannote_audio_b200.models import XVectorMFCC, XVectorSincNet

    sinc = XVectorSincNet()
    sinc.load_state_dict(syn.make_xvector_state_dict(3))
    sinc = sinc.to(dev)
    wav = _wav(160000, seeds=(6, 7)).to(dev)
    with torch.inference_mode():
        alone = [sinc(wav), model(wav)]
        mixed = [model(wav), sinc(wav), model(wav), sinc(wav)]
        assert torch.equal(mixed[0], alone[1]) and torch.equal(mixed[2], alone[1])
        assert torch.equal(mixed[1], alone[0]) and torch.equal(mixed[3], alone[0])
        other = XVectorMFCC().to(dev)
        other.load_state_dict(syn.make_xvector_mfcc_state_dict(5))
        base = other(wav)
        assert torch.equal(base, alone[1])
        other.load_state_dict(syn.make_xvector_mfcc_state_dict(6))     # after a forward: the new weights are uploaded
        assert not torch.equal(other(wav), base)
        assert torch.equal(model(wav), alone[1]) and torch.equal(sinc(wav), alone[0])
        # the SincNet model still matches its own oracle next to a resident XVectorMFCC
        ref = OracleXVectorSincNet()
        ref.load_state_dict(syn.make_xvector_state_dict(3))
        _check(sinc(wav), ref.eval().to(dev)(wav), "XVectorSincNet next to XVectorMFCC")


# The profiled call runs in a process of its own.  In a process that has kept an H100 busy for minutes, torch.profiler
# was seen to leave out of its trace the first kernels of a profiled call, or all of them: 13 launched and counted,
# 13, 6, 3, 0 or 13 recorded at different times of the same process.  A fresh process records every kernel, so the
# comparison below does not depend on where the test falls in a long suite.
_PROFILED_FORWARD = """
import json
import torch
from test_launch_count import _kernels
from pyannote_audio_b200 import synthetic as syn
from pyannote_audio_b200.models import XVectorMFCC

dev = torch.device("cuda:0")
m = XVectorMFCC()
m.load_state_dict(syn.make_xvector_mfcc_state_dict(5))
m = m.to(dev)
wav = torch.cat([syn.make_conversation(10.0, seed=s)[None] for s in (1, 2)]).to(dev)
w = torch.rand(2, 3, 50, generator=torch.Generator().manual_seed(1)).to(dev)
with torch.inference_mode():
    counted, kernels = _kernels(m._ctx(), lambda: m(wav, weights=w))
print(json.dumps({"counted": counted, "kernels": kernels}))
"""


@pytest.mark.gpu
def test_every_launch_is_counted(dev):
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests")]))
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", _PROFILED_FORWARD], cwd=root, env=env, capture_output=True,
                         text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-4000:]
    out = json.loads(run.stdout.strip().splitlines()[-1])
    counted, kernels = out["counted"], out["kernels"]
    assert counted == len(kernels) and counted > 0, (counted, kernels)
    # every sub-batch runs the rows, mel / dB and DCT kernels once
    per_kernel = [sum(name in k for k in kernels) for name in ("mfcc_rows_kernel", "mfcc_mel_db_kernel",
                                                               "mfcc_dct_kernel")]
    assert per_kernel[0] >= 1 and len(set(per_kernel)) == 1, (per_kernel, kernels)


@pytest.mark.gpu
def test_errors(model, dev):
    from pyannote_audio_b200.models import get_context

    with pytest.raises(ValueError, match="2800"):
        model(torch.zeros(1, 1, 2799, device=dev))
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
