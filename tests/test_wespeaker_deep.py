"""WeSpeakerResNet152 / 221 / 293: the bottleneck ResNets (models/embedding/wespeaker/resnet.py:148-212, 477-508,
wespeaker/__init__.py:375-466).  CPU: the fp32 oracle against the reference's own resnet.py (golden vectors), the
state-dict keys, checkpoint loading and the fp16 activation range of the synthetic weights.  GPU: the CUDA trunk
against the fp32 oracle run on the GPU with TF32 off (cosine distance <= 1e-3), its bit-exact reference paths, and the
pipelines on top of it."""
import os

import numpy as np
import pytest
import torch
import yaml

from oracle_bottleneck import WeSpeakerBottleneck
from pyannote_audio_b200 import synthetic as syn
from pyannote_audio_b200.testing.checkpoints import reference_style_checkpoint

DEPTHS = (152, 221, 293)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_bottleneck_vectors.npz")


def _cos_dist(a, b):
    return 1 - (a * b).sum(-1) / np.maximum(np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1), 1e-30)


def _model_class(depth):
    from pyannote_audio_b200 import models

    return getattr(models, f"WeSpeakerResNet{depth}")


def _oracle(depth):
    m = WeSpeakerBottleneck(depth)
    m.load_state_dict(syn.make_bottleneck_state_dict(depth, 1))
    return m.eval()


# ---- CPU ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("depth", DEPTHS)
def test_oracle_matches_reference_module(depth):
    golden = np.load(GOLDEN)
    net = _oracle(depth)
    fb, w = torch.from_numpy(golden["fbank"]), torch.from_numpy(golden["weights"])
    with torch.inference_mode():
        e = net.resnet(fb, weights=w)
        e0 = net.resnet(fb)
    np.testing.assert_allclose(e.numpy(), golden[f"emb_{depth}"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(e0.numpy(), golden[f"emb_noweights_{depth}"], rtol=0, atol=2e-5)


@pytest.mark.parametrize("depth", DEPTHS)
def test_state_dict_keys_are_the_reference_ones(depth):
    ref_keys = list(np.load(GOLDEN)[f"keys_{depth}"])
    own = sorted(k[len("resnet."):] for k in _model_class(depth)().state_dict())
    assert own == ref_keys
    assert sorted(k[len("resnet."):] for k in syn.make_bottleneck_state_dict(depth, 1)) == ref_keys
    assert sorted(k[len("resnet."):] for k in WeSpeakerBottleneck(depth).state_dict()) == ref_keys


def test_from_pretrained_and_community_directory_with_resnet293(tmp_path):
    from pyannote_audio_b200.loading import get_model, resolve_pipeline
    from pyannote_audio_b200.models import BaseWeSpeakerResNet, Model, WeSpeakerResNet34, WeSpeakerResNet293
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    blob, sd = reference_style_checkpoint("emb293")
    path = tmp_path / "pytorch_model.bin"
    path.write_bytes(blob)
    for klass in (Model, BaseWeSpeakerResNet, WeSpeakerResNet293):
        m = klass.from_pretrained(str(path))
        assert type(m) is WeSpeakerResNet293 and not m.training and m.dimension == 256
        assert torch.equal(m.state_dict()["resnet.layer3.63.conv3.weight"], sd["resnet.layer3.63.conv3.weight"])
    with pytest.raises(ValueError, match="not a WeSpeakerResNet34"):
        WeSpeakerResNet34.from_pretrained(str(path))
    root = tmp_path / "community-1"
    for sub, kind in (("segmentation", "seg"), ("embedding", "emb293")):
        (root / sub).mkdir(parents=True)
        (root / sub / "pytorch_model.bin").write_bytes(reference_style_checkpoint(kind)[0])
    config = {"version": "4.0.0",
              "pipeline": {"name": "pyannote.audio.pipelines.SpeakerDiarization",
                           "params": {"clustering": "VBxClustering", "segmentation": "$model/segmentation",
                                      "embedding": "$model/embedding", "plda": "$model/plda"}}}
    (root / "config.yaml").write_text(yaml.dump(config))
    klass, params, _ = resolve_pipeline(root)
    assert klass is SpeakerDiarization and params["embedding"]["subfolder"] == "embedding"
    emb = get_model(params["embedding"])
    assert type(emb) is WeSpeakerResNet293 and emb.num_frames(160000) == 125


@pytest.mark.parametrize("depth", DEPTHS)
def test_synthetic_weights_keep_the_fp16_range(depth):
    """Activation RMS after every block within [0.05, 50] and max |x| < 1e3 on 10 s of synthetic audio: the fp16
    trunk holds the residual stream of all the blocks."""
    net = _oracle(depth)
    trace = []
    with torch.inference_mode():
        net.resnet.forward_frames(net.compute_fbank(syn.make_conversation(10.0, seed=7)[None]), trace=trace)
    assert len(trace) == sum(syn.BOTTLENECK_BLOCKS[depth])
    rms = np.array([float(x.pow(2).mean().sqrt()) for x in trace])
    peak = max(float(x.abs().max()) for x in trace)
    assert rms.min() >= 0.05 and rms.max() <= 50 and peak < 1e3, (rms.min(), rms.max(), peak)


# ---- GPU ------------------------------------------------------------------------------------------------
EMB_MAX_BATCH = 16           # chunks per sub-batch in these tests: about 1 GB of bottleneck workspace


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ctx(dev):
    from pyannote_audio_b200.models import get_context

    c = get_context(dev)
    c.set_option("emb_max_batch", EMB_MAX_BATCH)
    yield c
    c.set_option("emb_max_batch", int(os.environ.get("B200_EMB_MAX_BATCH", 264)))
    c.set_option("conv_impl", 1)
    c.set_option("fbank_share", 1)


@pytest.fixture(autouse=True)
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


_MODELS = {}


def _pair(depth, dev):
    """(CUDA model, fp32 oracle on the GPU) of one depth, built once."""
    if depth not in _MODELS:
        m = _model_class(depth)()
        m.load_state_dict(syn.make_bottleneck_state_dict(depth, 1))
        _MODELS[depth] = (m.to(dev), _oracle(depth).to(dev))
    return _MODELS[depth]


def _run_oracle(oemb, wav, weights=None):
    with torch.inference_mode():
        return oemb(wav.cuda(), weights=None if weights is None else weights.cuda()).cpu().numpy()


def _binary(rng, shape):
    w = (rng.uniform(size=shape) < 0.5).astype(np.float32)
    w[..., 0] = 1.0
    return torch.from_numpy(w)


def _wavs(n, N, seed):
    wav = syn.make_conversation(n * N / 16000 + 0.1, seed=seed)[0]
    return torch.stack([wav[i * N:(i + 1) * N] for i in range(n)])[:, None]


@pytest.mark.gpu
@pytest.mark.parametrize("depth", DEPTHS)
def test_chunks_with_and_without_masks(ctx, dev, depth):
    emb, oemb = _pair(depth, dev)
    rng = np.random.default_rng(depth)
    for b in (1, 5):
        wav = _wavs(b, 160000, seed=depth + b)
        for S in (None, 1, 3):
            w = None if S is None else _binary(rng, (b, S, 589))
            got = emb(wav.to(dev), weights=None if w is None else w.to(dev)).cpu().numpy()
            ref = _run_oracle(oemb, wav, w)
            assert got.shape == ref.shape and np.isfinite(got).all()
            d = _cos_dist(got, ref).max()
            print(f"ResNet{depth} 10 s chunks b={b} S={S}: max cosine distance {d:.2e}")
            assert d <= 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("depth", DEPTHS)
def test_any_length(ctx, dev, depth):
    emb, oemb = _pair(depth, dev)
    lengths = [400, 16000, 160001, 480000] + ([1000000] if depth == 293 else [])
    worst = 0.0
    rng = np.random.default_rng(depth)
    for N in lengths:
        for b in (1, 3):
            wav = _wavs(b, N, seed=N % 1000 + b)
            got = emb(wav.to(dev)).cpu().numpy()
            ref = _run_oracle(oemb, wav)
            assert got.shape == (b, 256)
            if emb.num_frames(N) == 1:                     # std(correction=1) of one frame
                assert np.isnan(got).all() and np.isnan(ref).all()
            else:
                assert np.isfinite(got).all()
                worst = max(worst, float(_cos_dist(got, ref).max()))
            w = _binary(rng, (b, 3, 7 + N // 2000))
            got = emb(wav.to(dev), weights=w.to(dev)).cpu().numpy()
            ref = _run_oracle(oemb, wav, w)
            assert got.shape == (b, 3, 256) and np.isfinite(got).all()
            worst = max(worst, float(_cos_dist(got, ref).max()))
            assert worst <= 1e-3, (N, b, worst)
    print(f"ResNet{depth} any length: max cosine distance {worst:.2e}")
    if depth == 293:
        # soft weights with two speakers through forward_embedding on 1024-channel frames
        wav = _wavs(2, 160000, seed=3)
        with torch.inference_mode():
            frames = oemb.forward_frames(wav.cuda())
        assert tuple(frames.shape) == (2, 1024, 10, 125)
        w = torch.rand(2, 2, 589, generator=torch.Generator().manual_seed(0))
        got = emb.forward_embedding(frames, weights=w.to(dev)).cpu().numpy()
        with torch.inference_mode():
            ref = oemb.forward_embedding(frames, weights=w.cuda()).cpu().numpy()
        assert got.shape == (2, 2, 256) and np.isfinite(got).all()
        assert _cos_dist(got, ref).max() <= 1e-3
        with pytest.raises(ValueError, match="1024, 10"):
            emb.forward_embedding(torch.zeros(1, 256, 10, 5, device=dev))


@pytest.mark.gpu
@pytest.mark.parametrize("depth", DEPTHS)
def test_reference_paths_and_sub_batches(ctx, dev, depth):
    emb, oemb = _pair(depth, dev)
    emb._ctx()
    wav = syn.make_conversation(16.0, seed=11)
    buf = wav[0].to(dev).contiguous()
    off = np.arange(0, 6 * 16000 + 1, 16000, dtype=np.int64)
    valid = np.full(len(off), 160000, dtype=np.int32)
    fb = ctx.emb_fbank(buf, off, valid)
    frames = {}
    for impl in (0, 1, 2):
        ctx.set_option("conv_impl", impl)
        frames[impl] = ctx.emb_trunk(fb)
    ctx.set_option("conv_impl", 1)
    assert tuple(frames[1].shape) == (len(off), 1024, 10, 125) and torch.isfinite(frames[1]).all()
    assert torch.equal(frames[1], frames[2])
    a, b = frames[1].cpu().numpy(), frames[0].cpu().numpy()
    assert np.abs(a - b).max() <= 2e-2 * np.abs(b).max()
    with torch.inference_mode():
        ref = oemb.resnet.forward_frames(fb).cpu().numpy()
    assert np.abs(a - ref).max() / np.abs(ref).max() < 2e-2
    # sub-batch split and shared / private fbank frames: bit-identical embeddings
    masks = torch.from_numpy((np.random.default_rng(1).uniform(size=(len(off), 3, 589)) < 0.6).astype(np.uint8))
    masks = masks.to(dev)
    base = ctx.emb_forward(buf, off, valid, masks).clone()
    ctx.set_option("emb_max_batch", 4)
    small = ctx.emb_forward(buf, off, valid, masks).clone()
    utt_small = emb(_wavs(3, 480000, seed=2).to(dev)).clone()
    ctx.set_option("emb_max_batch", EMB_MAX_BATCH)
    utt = emb(_wavs(3, 480000, seed=2).to(dev))
    ctx.set_option("fbank_share", 0)
    private = ctx.emb_forward(buf, off, valid, masks).clone()
    ctx.set_option("fbank_share", 1)
    assert torch.equal(base, small) and torch.equal(base, private) and torch.equal(utt, utt_small)
    assert torch.isfinite(base).all()


@pytest.mark.gpu
def test_resnet34_after_resnet293_is_bit_identical(ctx, dev):
    from pyannote_audio_b200.models import WeSpeakerResNet34

    r34 = WeSpeakerResNet34()
    r34.load_state_dict(syn.make_embedding_state_dict(1))
    r34 = r34.to(dev)
    wav = _wavs(3, 160000, seed=4).to(dev)
    w = _binary(np.random.default_rng(2), (3, 3, 589)).to(dev)
    first = r34(wav, weights=w).clone()
    first_utt = r34(wav[..., :50000]).clone()
    emb293, _ = _pair(293, dev)
    assert torch.isfinite(emb293(wav, weights=w)).all()
    assert ctx.emb_channels == 1024
    assert torch.equal(r34(wav, weights=w), first) and torch.equal(r34(wav[..., :50000]), first_utt)
    assert ctx.emb_channels == 256


class _OracleOnGpu:
    """The oracle ResNet293 on the GPU behind the CPU interface oracle.pipeline.get_embeddings expects."""

    def __init__(self, m):
        self.m = m

    def forward_frames(self, wav):
        return self.m.forward_frames(wav.cuda())

    def forward_embedding(self, frames, weights=None):
        return self.m.forward_embedding(frames, weights=None if weights is None else weights.cuda()).cpu()


@pytest.mark.gpu
def test_speaker_diarization_with_resnet293(ctx, dev):
    from oracle import nets
    from pyannote_audio_b200.models import PyanNet
    from pyannote_audio_b200.pipeline import SpeakerDiarization
    from test_gpu_parity import _e2e_case

    emb, oemb = _pair(293, dev)
    seg = PyanNet()
    seg.load_state_dict(syn.make_segmentation_state_dict(0))
    pipeline = SpeakerDiarization(segmentation=seg, embedding=emb, plda=syn.make_plda(2), device=dev)
    oseg = nets.PyanNet()
    oseg.load_state_dict(syn.make_segmentation_state_dict(0))
    out, art = _e2e_case(pipeline, (oseg.eval(), _OracleOnGpu(oemb)), syn.make_conversation(180.0, seed=293),
                         "resnet293-180s")
    assert np.isfinite(art["embeddings"].cpu().numpy()).all()


@pytest.mark.gpu
def test_speaker_embedding_pipeline_with_resnet293(ctx, dev):
    from pyannote_audio_b200.models import PyanNet
    from pyannote_audio_b200.speaker_verification import SpeakerEmbedding

    emb, oemb = _pair(293, dev)
    wav = syn.make_conversation(40.0, seed=9)
    file = {"waveform": wav, "sample_rate": 16000}
    plain = SpeakerEmbedding(embedding=emb, device=dev)(file)
    assert plain.shape == (1, 256) and np.isfinite(plain).all()
    assert _cos_dist(plain, _run_oracle(oemb, wav[None])).max() <= 1e-3
    seg = PyanNet()
    seg.load_state_dict(syn.make_segmentation_state_dict(0))
    vad = SpeakerEmbedding(embedding=emb, segmentation=seg, device=dev)
    weights = vad.speech_weights(file)
    got = vad.apply(file)
    ref = _run_oracle(oemb, wav[None], torch.from_numpy(weights)[None])
    assert got.shape == (1, 256) and np.isfinite(got).all() and _cos_dist(got, ref).max() <= 1e-3
