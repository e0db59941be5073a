"""Speaker embeddings of audio of any length: WeSpeakerResNet34.forward / forward_embedding, Inference with an
embedding model (window="whole" and "sliding") and the SpeakerEmbedding pipeline, against the fp32 oracle run on the
GPU with TF32 off (reference: models/embedding/wespeaker/__init__.py:288-343, models/blocks/pooling.py:30-130,
core/inference.py:235-313, pipelines/speaker_verification.py:781-856)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nets, pipeline as P
from pyannote_audio_b200 import synthetic as syn

SR = 16000


def _cos_dist(a, b):
    return 1 - (a * b).sum(-1) / np.maximum(np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1), 1e-30)


def test_pipeline_name_resolves_to_speaker_embedding():
    from pyannote_audio_b200.loading import resolve_pipeline
    from pyannote_audio_b200.speaker_verification import SpeakerEmbedding

    klass, params, _ = resolve_pipeline({"pipeline": {"name": "pyannote.audio.pipelines.SpeakerEmbedding",
                                                      "params": {"embedding": "$model/embedding"}}})
    assert klass is SpeakerEmbedding and params["embedding"]["subfolder"] == "embedding"
    import pyannote_audio_b200

    assert pyannote_audio_b200.SpeakerEmbedding is SpeakerEmbedding


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def emb(dev):
    from pyannote_audio_b200.models import WeSpeakerResNet34

    m = WeSpeakerResNet34()
    m.load_state_dict(syn.make_embedding_state_dict(1))
    return m.to(dev)


@pytest.fixture(scope="module")
def oemb(dev):
    m = nets.WeSpeakerResNet34()
    m.load_state_dict(syn.make_embedding_state_dict(1))
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


def _oracle(oemb, wav, weights=None):
    with torch.inference_mode():
        return oemb(wav.cuda(), weights=None if weights is None else weights.cuda()).cpu().numpy()


def _binary(rng, shape):
    w = (rng.uniform(size=shape) < 0.5).astype(np.float32)
    w[..., 0] = 1.0                                        # no all-zero speaker
    return torch.from_numpy(w)


# ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N", [400, 1520, 1680, 16000, 48000, 160001, 1000000])
@pytest.mark.parametrize("batch", [1, 3])
def test_forward_any_length_matches_oracle(emb, oemb, long_wav, N, batch):
    rng = np.random.default_rng(N + batch)
    starts = rng.integers(0, long_wav.shape[1] - N, size=batch)
    wav = torch.stack([long_wav[:, s: s + N] for s in starts])                         # (batch, 1, N)
    T = emb.num_frames(N)
    got = emb(wav).cpu().numpy()
    ref = _oracle(oemb, wav)
    assert got.shape == (batch, 256)
    if T == 1:                                             # std(correction=1) of one frame
        assert np.isnan(got).all() and np.isnan(ref).all()
    else:
        assert _cos_dist(got, ref).max() <= 1e-3
    Tw = 7 + N // 2000                                     # weights over any number of frames
    for w in (_binary(rng, (batch, Tw)), _binary(rng, (batch, 3, Tw))):
        got = emb(wav, weights=w).cpu().numpy()
        ref = _oracle(oemb, wav, w)
        assert got.shape == ref.shape
        assert _cos_dist(got, ref).max() <= 1e-3
    with pytest.raises(ValueError):
        emb(wav, weights=torch.full((batch, Tw), 0.5))    # forward keeps the binary-mask contract


@pytest.mark.gpu
def test_forward_rejects_less_than_one_frame(emb):
    with pytest.raises(ValueError):
        emb(torch.zeros(1, 1, 399))


@pytest.mark.gpu
def test_utterance_path_reproduces_the_10s_path_bit_for_bit(emb, dev):
    """emb_forward_utt at 160000 samples with the binary masks of real chunks == emb_forward (diarization path)."""
    from pyannote_audio_b200.models import PyanNet

    seg = PyanNet()
    seg.load_state_dict(syn.make_segmentation_state_dict(0))
    seg.to(dev)
    wav = syn.make_conversation(31.0, seed=17)
    chunks = P.chunk_waveform(wav)[:6]
    flat = chunks.reshape(-1).to(dev).contiguous()
    off = np.arange(len(chunks), dtype=np.int64) * 160000
    valid = np.full(len(chunks), 160000, dtype=np.int32)
    cls = seg.forward_chunks(flat, off, valid)
    ctx = emb._ctx()
    masks = ctx.powerset_to_multilabel(cls).permute(0, 2, 1).contiguous()                # (C, 3, 589) u8
    assert 0 < int(masks.sum()) < masks.numel()
    ref = ctx.emb_forward(flat, off, valid, masks)
    got = ctx.emb_forward_utt(flat, off, 160000, weights=masks.float())
    assert torch.equal(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 2, 5])
@pytest.mark.parametrize("T,Tw", [(125, 589), (300, 77), (41000, 13001)])
def test_forward_embedding_soft_weights(emb, oemb, dev, S, T, Tw):
    g = torch.Generator(device="cpu").manual_seed(T + S)
    B = 2 if T < 1000 else 1
    frames = (torch.rand((B, 256, 10, T), generator=g) * 3.0).to(dev)
    w = torch.rand((B, S, Tw), generator=g).to(dev)
    got = emb.forward_embedding(frames, weights=w)
    with torch.inference_mode():
        wi = F.interpolate(w, size=T, mode="nearest")                                   # CUDA index map
        ref = oemb.forward_embedding(frames, weights=wi)
    assert tuple(got.shape) == (B, S, 256)
    err = (got - ref).abs().max().item()
    assert err <= 1e-4 * ref.abs().max().item(), err
    if S == 1:                                             # (batch, frames) weights -> (batch, 256)
        assert tuple(emb.forward_embedding(frames, weights=w[:, 0]).shape) == (B, 256)
        got = emb.forward_embedding(frames)                # no weights: mean and std(correction=1)
        with torch.inference_mode():
            ref = oemb.forward_embedding(frames)
        assert (got - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


@pytest.mark.gpu
def test_pooling_uses_the_cuda_nearest_index(emb, oemb, dev):
    """Find a (Tw, T) pair on which torch's CUDA F.interpolate(mode="nearest") index differs from t * Tw // T, and
    put all the weight on one source frame where they disagree: a wrong map moves the mean by O(1)."""
    found = None
    for T in (2049, 3001, 4093, 13490):
        for Tw in (123133, 204455, 99991, 77777):
            src = F.interpolate(torch.arange(Tw, dtype=torch.float32, device=dev)[None, None], size=T,
                                mode="nearest")[0, 0].long().cpu().numpy()
            diff = np.flatnonzero(src != np.arange(T) * Tw // T)
            if len(diff):
                found = (T, Tw, int(src[diff[0]]))
                break
        if found:
            break
    assert found is not None, "no (Tw, T) pair where the CUDA nearest index differs from the integer formula"
    T, Tw, k = found
    g = torch.Generator(device="cpu").manual_seed(3)
    frames = (torch.randn((1, 256, 10, T), generator=g) + 2.0).to(dev)
    w = torch.zeros((1, 1, Tw), device=dev)
    w[0, 0, k] = 1.0
    got = emb.forward_embedding(frames, weights=w)
    with torch.inference_mode():
        ref = oemb.forward_embedding(frames, weights=F.interpolate(w, size=T, mode="nearest"))
    assert (got - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


@pytest.mark.gpu
def test_sub_batches_do_not_change_results(emb, dev):
    ctx = emb._ctx()
    N = 60 * SR
    wav = torch.cat([syn.make_conversation(60.5, seed=40 + i)[0, :N] for i in range(5)]).to(dev).contiguous()
    off = np.arange(5, dtype=np.int64) * N
    try:
        ref = ctx.emb_forward_utt(wav, off, N)
        ctx.set_option("emb_max_batch", 7)                 # 6986 frames: one 5998-frame utterance per sub-batch
        got = ctx.emb_forward_utt(wav, off, N)
        assert torch.equal(got, ref)
        ctx.set_option("emb_max_batch", 4)                 # 3992 frames < 5998
        with pytest.raises(ValueError, match="emb_max_batch"):
            ctx.emb_forward_utt(wav, off, N)
    finally:
        ctx.set_option("emb_max_batch", 264)


@pytest.mark.gpu
def test_inference_whole_crop_and_sliding(emb, oemb):
    from pyannote_audio_b200.core import Segment, SlidingWindowFeature
    from pyannote_audio_b200.inference import Inference

    wav = syn.make_conversation(37.3, seed=8)
    file = {"waveform": wav, "sample_rate": SR}
    whole = Inference(emb, window="whole")
    e = whole(file)
    assert e.shape == (256,)
    assert _cos_dist(e, _oracle(oemb, wav[None])[0]) <= 1e-3
    seg = Segment(2.0, 19.5)
    c = whole.crop(file, seg)
    excerpt, _ = emb.audio.crop(file, seg)
    assert c.shape == (256,) and _cos_dist(c, _oracle(oemb, excerpt[None])[0]) <= 1e-3

    wav = wav[:, : int(12.5 * SR)]
    calls = []
    with pytest.warns(UserWarning):                        # trained on 10 s chunks, as the reference warns
        sliding = Inference(emb, window="sliding", duration=3.0, step=1.0)
    out = sliding({"waveform": wav, "sample_rate": SR}, hook=lambda **kw: calls.append(kw))
    assert isinstance(out, SlidingWindowFeature) and out.data.shape == (11, 256)
    sw = out.sliding_window
    assert (sw.start, sw.duration, sw.step) == (0.0, 3.0, 1.0)
    assert calls[0] == {"completed": 0, "total": 11} and calls[-1] == {"completed": 11, "total": 11}
    chunks = P.chunk_waveform(wav, window_size=3 * SR, step_size=SR)                 # padded tail chunk
    assert chunks.shape[0] == 11
    assert _cos_dist(out.data, _oracle(oemb, chunks)).max() <= 1e-3


@pytest.mark.gpu
def test_speaker_embedding_pipeline(emb, oemb, dev, tmp_path):
    from pyannote_audio_b200.loading import Pipeline
    from pyannote_audio_b200.models import PyanNet
    from pyannote_audio_b200.speaker_verification import SpeakerEmbedding
    from pyannote_audio_b200.testing.checkpoints import reference_style_checkpoint

    wav = syn.make_conversation(23.7, seed=61)
    file = {"waveform": wav, "sample_rate": SR}
    plain = SpeakerEmbedding(embedding=emb, device=dev)
    e = plain(file)
    assert isinstance(e, np.ndarray) and e.shape == (1, 256)
    assert np.array_equal(e, emb(wav[None]).cpu().numpy())

    seg = PyanNet()
    seg.load_state_dict(syn.make_segmentation_state_dict(0))
    vad = SpeakerEmbedding(embedding=emb, segmentation=seg, device=dev)
    weights = vad.speech_weights(file)
    assert weights.dtype == np.float32 and 0.0 < weights.max() <= 1.0 and not np.isnan(weights).any()
    assert ((weights > 0) & (weights < 1)).any()           # soft weights
    e = vad.apply(file)
    ref = _oracle(oemb, wav[None], torch.from_numpy(weights)[None])
    assert e.shape == (1, 256) and _cos_dist(e, ref).max() <= 1e-3
    assert _cos_dist(e, plain(file)).max() > 1e-6          # the weights took effect

    blob, _ = reference_style_checkpoint("emb")
    (tmp_path / "embedding").mkdir()
    (tmp_path / "embedding" / "pytorch_model.bin").write_bytes(blob)
    (tmp_path / "config.yaml").write_text("pipeline:\n  name: pyannote.audio.pipelines.SpeakerEmbedding\n"
                                          "  params:\n    embedding: $model/embedding\n")
    pipe = Pipeline.from_pretrained(tmp_path)
    assert isinstance(pipe, SpeakerEmbedding)
    assert np.array_equal(pipe(file), plain(file))         # same weights, no segmentation
