"""GPU tests of the reference-signature seams (pytest -m gpu): the calls a pyannote.audio user makes -- ``Inference``,
``Model.forward``, ``PretrainedSpeakerEmbedding.__call__``, the ``SpeakerDiarization`` stage methods, the clustering
classes, hooks -- against the CPU oracle.  Reference signatures (relative to /root/reference/src/pyannote/audio):
core/inference.py:182-215,375-496; models/segmentation/PyanNet.py:211-240; models/embedding/wespeaker/__init__.py:
324-343; pipelines/speaker_verification.py:704-716; pipelines/speaker_diarization.py:305-528;
pipelines/clustering.py:214-289,330-480,572-669; pipelines/utils/hook.py:37-203.
"""
import numpy as np
import pytest
import torch

from oracle import nets, pipeline as P
from pyannote_audio_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

FRAMES = P.SW(*nets.sincnet_receptive_field())
LOW_MARGIN = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def oracle_models():
    seg = nets.PyanNet()
    seg.load_state_dict(syn.make_segmentation_state_dict(0))
    emb = nets.WeSpeakerResNet34()
    emb.load_state_dict(syn.make_embedding_state_dict(1))
    return seg.eval(), emb.eval()


@pytest.fixture(scope="module")
def models(dev):
    from pyannote_audio_b200.models import PyanNet, WeSpeakerResNet34

    seg, emb = PyanNet(), WeSpeakerResNet34()
    seg.load_state_dict(syn.make_segmentation_state_dict(0))
    emb.load_state_dict(syn.make_embedding_state_dict(1))
    return seg.to(dev), emb.to(dev)


@pytest.fixture(scope="module")
def pipeline(dev, models):
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    return SpeakerDiarization(segmentation=models[0], embedding=models[1], plda=syn.make_plda(2), device=dev)


def _clear_margin(ref_logp):
    top2 = np.sort(ref_logp, axis=-1)
    return (top2[..., -1] - top2[..., -2]) >= LOW_MARGIN


def _cos_dist(a, b):
    return 1 - (a * b).sum(-1) / np.maximum(np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1), 1e-30)


# ---------------------------------------------------------------------------------------------------------
def test_model_forward_seams(models, oracle_models):
    seg, emb = models
    oseg, oemb = oracle_models
    wav = syn.make_conversation(14.0, seed=31)
    chunks = P.chunk_waveform(wav)[:4]                                   # (4,1,160000)
    with torch.inference_mode():
        ref_logp = oseg(chunks).numpy()
    logp = seg(chunks)                                                    # host tensor in, device tensor out
    assert logp.is_cuda and tuple(logp.shape) == (4, 589, 7)
    np.testing.assert_allclose(logp.cpu().numpy(), ref_logp, atol=2e-4, rtol=0)
    with pytest.raises(ValueError):
        seg(chunks[:, :, :1000])
    # WeSpeakerResNet34.forward(waveforms, weights): None, (batch, frames) and (batch, speakers, frames)
    rng = np.random.default_rng(5)
    w2 = (rng.uniform(size=(4, 589)) < 0.6).astype(np.float32)
    w3 = (rng.uniform(size=(4, 3, 589)) < 0.4).astype(np.float32)
    with torch.inference_mode():
        fr = oemb.forward_frames(chunks)
        ref_none = oemb.forward_embedding(fr).numpy()
        ref2 = oemb.forward_embedding(fr, weights=torch.from_numpy(w2)).numpy()
        ref3 = oemb.forward_embedding(fr, weights=torch.from_numpy(w3)).numpy()
    e_none, e2, e3 = emb(chunks), emb(chunks, weights=torch.from_numpy(w2)), emb(chunks, weights=torch.from_numpy(w3))
    assert tuple(e_none.shape) == (4, 256) and tuple(e2.shape) == (4, 256) and tuple(e3.shape) == (4, 3, 256)
    assert _cos_dist(e_none.cpu().numpy(), ref_none).max() <= 1e-3
    assert _cos_dist(e2.cpu().numpy(), ref2).max() <= 1e-3
    assert _cos_dist(e3.cpu().numpy(), ref3).max() <= 1e-3
    with pytest.raises(ValueError):
        emb(chunks, weights=torch.full((4, 589), 0.5))                    # binary masks only (documented limit)
    # forward_frames / compute_fbank (wespeaker/__init__.py:113-139,288-322)
    np.testing.assert_allclose(emb.compute_fbank(chunks).cpu().numpy(), oemb.compute_fbank(chunks).numpy(), atol=5e-3)
    got_fr = emb.forward_frames(chunks).cpu().numpy()
    assert np.abs(got_fr - fr.numpy()).max() <= 2e-2 * np.abs(fr.numpy()).max()


def test_two_models_share_a_device(dev, models, oracle_models):
    """ADVICE r1: weights live in one context slot per family; a second model with other weights must not be run
    with the first model's weights (and vice versa), and load_state_dict after a forward must take effect."""
    from pyannote_audio_b200.models import PyanNet

    seg_a, _ = models
    oseg, _ = oracle_models
    seg_b = PyanNet()
    seg_b.load_state_dict(syn.make_segmentation_state_dict(7))
    seg_b.to(dev)
    oseg_b = nets.PyanNet()
    oseg_b.load_state_dict(syn.make_segmentation_state_dict(7))
    chunks = P.chunk_waveform(syn.make_conversation(11.0, seed=3))[:2]
    with torch.inference_mode():
        ra, rb = oseg(chunks).numpy(), oseg_b.eval()(chunks).numpy()
    assert np.abs(ra - rb).max() > 1e-2                                   # the two nets really differ
    for _ in range(2):                                                    # interleaved calls
        np.testing.assert_allclose(seg_a(chunks).cpu().numpy(), ra, atol=2e-4, rtol=0)
        np.testing.assert_allclose(seg_b(chunks).cpu().numpy(), rb, atol=2e-4, rtol=0)
    seg_b.load_state_dict(syn.make_segmentation_state_dict(0))            # now the same weights as A
    np.testing.assert_allclose(seg_b(chunks).cpu().numpy(), ra, atol=2e-4, rtol=0)
    free0 = torch.cuda.mem_get_info(dev)[0]
    for _ in range(5):                                                    # re-uploads free the previous copy
        seg_b.load_state_dict(syn.make_segmentation_state_dict(7))
        seg_b(chunks)
        seg_a(chunks)
    assert free0 - torch.cuda.mem_get_info(dev)[0] < 64 << 20


def test_inference_seams(models, oracle_models):
    from pyannote_audio_b200.core import Segment
    from pyannote_audio_b200.inference import Inference

    seg, _ = models
    oseg, _ = oracle_models
    wav = syn.make_conversation(33.4, seed=41)                            # 25 chunks incl. a padded tail
    file = {"waveform": wav, "sample_rate": 16000}
    ref, ref_logp = P.slide(oseg, wav, return_logp=True)
    clear = _clear_margin(ref_logp)
    # __call__ with skip_aggregation (the pipeline's use, speaker_diarization.py:237-244)
    inf = Inference(seg, duration=10.0, step=1.0, skip_aggregation=True, batch_size=32)
    progress = []
    out = inf(file, hook=lambda completed=None, total=None: progress.append((completed, total)))
    assert out.data.shape == ref.data.shape == (25, 589, 3) and out.data.dtype == np.float32
    assert (out.sliding_window.start, out.sliding_window.duration, out.sliding_window.step) == (0.0, 10.0, 1.0)
    assert np.array_equal(out.data[clear], ref.data[clear])
    assert progress[0] == (0, 25) and progress[-1] == (25, 25)
    # infer(chunks) (inference.py:182-215): numpy (b,589,3) in {0,1}
    chunks = P.chunk_waveform(wav)
    got = inf.infer(chunks[:5])
    assert isinstance(got, np.ndarray) and got.shape == (5, 589, 3)
    assert np.array_equal(got[clear[:5]], ref.data[:5][clear[:5]])
    # skip_conversion=True: raw powerset log-probabilities (inference.py:130-141,210-215)
    raw = Inference(seg, duration=10.0, step=1.0, skip_aggregation=True, skip_conversion=True)
    lp = raw(file)
    assert lp.data.shape == (25, 589, 7)
    np.testing.assert_allclose(lp.data, ref_logp, atol=2e-4, rtol=0)
    np.testing.assert_allclose(raw.infer(chunks[:3]), ref_logp[:3], atol=2e-4, rtol=0)
    # aggregated output (hamming overlap-add, padded tail cropped; inference.py:349-369,498-620)
    agg = Inference(seg, duration=10.0, step=1.0, pre_aggregation_hook=lambda s: s)(file)
    oagg = P.aggregate(P.SWF(out.data, P.SW(0.0, 10.0, 1.0)), FRAMES, warm_up=(0.0, 0.0), hamming=True, missing=0.0)
    oagg = oagg.crop_loose((0.0, wav.shape[1] / 16000))
    assert agg.data.shape == oagg.data.shape
    np.testing.assert_allclose(agg.data, oagg.data, rtol=0, atol=1e-6)
    assert abs(agg.sliding_window.step - FRAMES.step) < 1e-12
    # crop(file, Segment) (inference.py:408-496): the window slides inside the excerpt, output shifted to its start
    focus = Segment(5.0, 27.5)
    sub = inf.crop(file, focus)
    s0, s1 = round(5.0 * 16000), round(27.5 * 16000)
    oref, olp = P.slide(oseg, wav[:, s0:s1], return_logp=True)
    assert sub.data.shape == oref.data.shape and sub.sliding_window.start == 5.0
    oc = _clear_margin(olp)
    assert np.array_equal(sub.data[oc], oref.data[oc])
    # window="whole" on a single 10 s excerpt
    whole = Inference(seg, window="whole", skip_aggregation=True)
    w = whole({"waveform": wav[:, :160000], "sample_rate": 16000})
    assert w.shape == (589, 3) and np.array_equal(w[clear[0]], ref.data[0][clear[0]])


def test_pipeline_stage_seams(pipeline, oracle_models):
    from pyannote_audio_b200.core import SlidingWindowFeature
    from pyannote_audio_b200.hooks import ArtifactHook, Hooks, TimingHook

    oseg, oemb = oracle_models
    wav = syn.make_conversation(41.0, seed=52)
    file = {"waveform": wav, "sample_rate": 16000, "uri": "seams"}
    ref, ref_logp = P.slide(oseg, wav, return_logp=True)
    clear = _clear_margin(ref_logp)
    seg = pipeline.get_segmentations(file)                                   # speaker_diarization.py:305-330
    assert isinstance(seg, SlidingWindowFeature) and seg.data.shape == ref.data.shape
    assert np.array_equal(seg.data[clear], ref.data[clear])
    if not np.array_equal(seg.data, ref.data):
        ref = P.SWF(seg.data, ref.sw)                                         # low-margin flip (reported by e2e tests)
    frames = pipeline._segmentation.model.receptive_field
    count = pipeline.speaker_count(seg, frames, warm_up=(0.0, 0.0))           # diarization.py:150-185
    ocount = P.speaker_count(ref, FRAMES, (0.0, 0.0))
    assert count.data.dtype == np.uint8 and np.array_equal(count.data, ocount.data)
    for excl in (False, True):                                               # speaker_diarization.py:332-478
        emb = pipeline.get_embeddings(file, seg, exclude_overlap=excl)
        oe = P.get_embeddings(oemb, wav, ref, exclude_overlap=excl, max_chunks=6)
        assert emb.shape == (ref.data.shape[0], 3, 256) and emb.dtype == np.float32
        ok = np.linalg.norm(oe, axis=-1) > 0
        assert _cos_dist(emb[:6], oe)[ok].max() <= 1e-3
    # PretrainedSpeakerEmbedding.__call__(waveforms, masks) -> np.ndarray (speaker_verification.py:704-716)
    chunks = P.chunk_waveform(wav)[:3]
    masks = torch.from_numpy(np.ascontiguousarray(ref.data[:3, :, 0]))
    e = pipeline._embedding(chunks, masks=masks)
    with torch.inference_mode():
        oe1 = oemb(chunks, weights=masks).numpy()
    assert isinstance(e, np.ndarray) and e.shape == (3, 256)
    ok = np.linalg.norm(oe1, axis=-1) > 0
    assert _cos_dist(e, oe1)[ok].max() <= 1e-3
    assert pipeline._embedding.dimension == 256 and pipeline._embedding.metric == "cosine"
    assert pipeline._embedding.sample_rate == 16000 and pipeline._embedding.min_num_samples == 400
    # clustering class call + reconstruct + to_annotation (clustering.py:572-669, speaker_diarization.py:480-528)
    hard, soft, centroids = pipeline.clustering(embeddings=emb, segmentations=seg)
    oh, osoft, oc = P.vbx_clustering(emb, ref.data, P.PLDA(**syn.make_plda(2)))
    assert np.array_equal(hard, oh)
    np.testing.assert_allclose(soft, osoft, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(centroids, oc, rtol=1e-9, atol=1e-12)
    inactive = np.sum(ref.data, axis=1) == 0
    hard = hard.copy()
    hard[inactive] = -2
    ocount.data = ocount.data.astype(np.int8)
    disc = pipeline.reconstruct(seg, hard, count)
    odisc = P.reconstruct(ref, hard, ocount)
    assert np.array_equal(disc.data[:, : odisc.data.shape[1]], odisc.data)
    ann = pipeline.to_annotation(disc, min_duration_on=0.0, min_duration_off=0.0)
    rows, times = P.binarize_to_segments(odisc)
    assert [(s.start, s.end, lab) for s, _, lab in ann.itertracks(yield_label=True)] == times
    # hooks: the four step names with real artifacts, progress calls, ArtifactHook / TimingHook / Hooks
    f2 = dict(file)
    with Hooks(ArtifactHook(), TimingHook()) as hook:
        out = pipeline(f2, hook=hook)
    assert set(f2["artifact"]) == {"segmentation", "speaker_counting", "embeddings", "discrete_diarization"}
    assert isinstance(f2["artifact"]["segmentation"], SlidingWindowFeature)
    assert np.array_equal(f2["artifact"]["segmentation"].data, seg.data)
    assert np.array_equal(np.asarray(f2["artifact"]["embeddings"]), pipeline.get_embeddings(file, seg))
    assert f2["artifact"]["discrete_diarization"].data.shape[0] == disc.data.shape[0]
    assert {"segmentation", "embeddings", "total"} <= set(f2["timing"])
    assert len(out.speaker_diarization.labels()) == out.speaker_embeddings.shape[0]


def test_clustering_class_seams(dev):
    """VBxClustering / AgglomerativeClustering called like the reference calls them, on synthetic embeddings with
    speaker structure, against the oracle (scipy + the reference's VBx)."""
    from pyannote_audio_b200.clustering import PLDA, AgglomerativeClustering, VBxClustering

    rng = np.random.default_rng(8)
    C = 120
    centers = rng.standard_normal((4, 256))
    who = rng.integers(0, 4, size=(C, 3))
    emb = (centers[who] + 0.35 * rng.standard_normal((C, 3, 256))).astype(np.float32)
    seg = np.zeros((C, 589, 3), dtype=np.float32)
    for c in range(C):                                                   # non-overlapping turns + some short / silent
        cuts = np.sort(rng.integers(0, 589, size=2))
        seg[c, : cuts[0], 0] = 1
        seg[c, cuts[0]: cuts[1], 1] = 1
        if c % 7:
            seg[c, cuts[1]:, 2] = 1
    plda_d = syn.make_plda(2)
    vbx = VBxClustering(PLDA(plda_d), device=dev)
    hard, soft, cent = vbx(embeddings=emb, segmentations=seg)
    oh, osoft, oc = P.vbx_clustering(emb, seg, P.PLDA(**plda_d))
    assert hard.dtype == np.int8 and np.array_equal(hard, oh)
    np.testing.assert_allclose(soft, osoft, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(cent, oc, rtol=1e-9, atol=1e-12)
    # forced speaker count -> KMeans fallback + plain argmax (clustering.py:626-642)
    hard_k, _, cent_k = vbx(embeddings=emb, segmentations=seg, num_clusters=2)
    oh_k, _, oc_k = P.vbx_clustering(emb, seg, P.PLDA(**plda_d), num_clusters=2, min_clusters=2, max_clusters=2)
    assert cent_k.shape == (2, 256) and np.array_equal(hard_k, oh_k)
    np.testing.assert_allclose(cent_k, oc_k, rtol=1e-5, atol=1e-6)      # the reference averages float32 rows here
    # AgglomerativeClustering (legacy 3.1 path): threshold cut, min_cluster_size reassignment, forced num_clusters
    ahc = AgglomerativeClustering(device=dev)
    for params, kw in (({"threshold": 0.9, "min_cluster_size": 12}, {}),
                       ({"threshold": 0.5, "min_cluster_size": 25}, {}),                 # many small clusters
                       ({"threshold": 0.9, "min_cluster_size": 12}, {"num_clusters": 3}),
                       ({"threshold": 1.4, "min_cluster_size": 5}, {"min_clusters": 2, "max_clusters": 6})):
        ahc.instantiate(dict(method="centroid", **params))
        h, s_, cc = ahc(embeddings=emb, segmentations=seg, **kw)
        rh, rs, rc = P.ahc_call(emb, seg, params["threshold"], params["min_cluster_size"], **kw)
        assert np.array_equal(h, rh), (params, kw)
        np.testing.assert_allclose(cc, rc, rtol=1e-5, atol=1e-6)        # reference: np.mean of float32 rows
        np.testing.assert_allclose(s_, rs, rtol=0, atol=1e-6)
        train, _, _ = P.filter_embeddings(emb, seg)
        assert np.array_equal(ahc.cluster(train, **{"min_clusters": kw.get("num_clusters") or kw.get("min_clusters", 1),
                                                    "max_clusters": kw.get("num_clusters") or kw.get("max_clusters"),
                                                    "num_clusters": kw.get("num_clusters")}),
                              P.ahc_cluster(train, threshold=params["threshold"],
                                            min_cluster_size=params["min_cluster_size"],
                                            min_clusters=kw.get("num_clusters") or kw.get("min_clusters", 1),
                                            max_clusters=kw.get("num_clusters") or kw.get("max_clusters"),
                                            num_clusters=kw.get("num_clusters")))
    with pytest.raises(NotImplementedError):
        AgglomerativeClustering(device=dev).instantiate({"method": "average"}).cluster(train)


def test_reconstruct_many_clusters(dev):
    """More than 32 clusters (ADVICE r1): generic kernel, same exact arithmetic as the oracle."""
    from pyannote_audio_b200.models import get_context

    ctx = get_context(dev)
    rng = np.random.default_rng(12)
    C = 30
    seg = (rng.uniform(size=(C, 589, 3)) < 0.4).astype(np.float32)
    swf = P.SWF(seg, P.SW(0.0, 10.0, 1.0))
    count = P.speaker_count(swf, FRAMES, (0.0, 0.0))
    sf = P.chunk_start_frames(C, FRAMES)
    F = len(count.data)
    for K in (33, 60, 127):
        hard = rng.integers(-1, K, size=(C, 3)).astype(np.int8)
        hard[hard == -1] = -2
        hard[0] = (K - 1, 0, 0)                                           # duplicates inside a chunk + the last cluster
        cnt = P.SWF(np.minimum(count.data, 3).astype(np.int8), count.sw)
        ref = P.reconstruct(swf, hard, cnt)
        d = ctx.reconstruct(torch.from_numpy(seg.astype(np.uint8)).to(dev), hard, sf, F,
                            torch.from_numpy(cnt.data[:, 0].astype(np.uint8)).to(dev), K)
        assert np.array_equal(d.cpu().numpy(), ref.data.astype(np.uint8))
    with pytest.raises(Exception):
        ctx.reconstruct(torch.from_numpy(seg.astype(np.uint8)).to(dev), hard, sf, F,
                        torch.from_numpy(cnt.data[:, 0].astype(np.uint8)).to(dev), 200)


def test_apply_sharded_single_rank(pipeline):
    """parallel.apply_sharded (one long file, chunk ranges per rank + all-gather) on a 1-rank NCCL group equals
    the plain pipeline; the 2-rank host logic is covered on CPU/gloo (tests/test_parallel_gloo.py)."""
    import torch.distributed as dist

    from pyannote_audio_b200.parallel import apply_sharded

    wav = syn.make_conversation(52.0, seed=61)
    file = {"waveform": wav, "sample_rate": 16000, "uri": "sharded"}
    ref = pipeline(file)
    created = False
    if not dist.is_initialized():
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29533", rank=0, world_size=1,
                                device_id=pipeline.device)
        created = True
    try:
        seen = []
        out = apply_sharded(pipeline, file, hook=lambda name, artifact, **k: seen.append(name))
    finally:
        if created:
            dist.destroy_process_group()
    a = [(s.start, s.end, lab) for s, _, lab in out.speaker_diarization.itertracks(yield_label=True)]
    b = [(s.start, s.end, lab) for s, _, lab in ref.speaker_diarization.itertracks(yield_label=True)]
    assert a == b and "discrete_diarization" in seen
    np.testing.assert_allclose(out.speaker_embeddings, ref.speaker_embeddings, rtol=1e-12)


def test_audio_ingest_on_device(dev, pipeline, tmp_path):
    """PCM -> float, downmix, resample to 16 kHz on the device (b200_audio_ingest) against
    the reference's host path (core/io.py:223-265: mean over channels, then torchaudio.functional.resample)."""
    import torchaudio.functional as AF
    from scipy.io import wavfile

    from pyannote_audio_b200.audio import Audio
    from pyannote_audio_b200.models import get_context

    ctx = get_context(dev)
    rng = np.random.default_rng(3)
    base = syn.make_conversation(6.3, seed=9)                                # (1, T) float32 @ 16 kHz
    for sr_in in (16000, 8000, 44100, 48000, 22050):
        T = int(round(6.3 * sr_in))
        t = np.arange(T) / sr_in
        stereo = np.stack([0.4 * np.sin(2 * np.pi * 220 * t) + 0.05 * rng.standard_normal(T),
                           0.3 * np.sin(2 * np.pi * 330 * t + 1.0)]).astype(np.float32)
        x = torch.from_numpy(stereo)
        ref = x.mean(dim=0, keepdim=True)
        if sr_in != 16000:
            ref = AF.resample(ref, sr_in, 16000)
        got = ctx.audio_ingest(x.to(dev), sr_in, 16000)
        assert got.shape[0] == ref.shape[1], (sr_in, got.shape, ref.shape)
        err = float((got.cpu() - ref[0]).abs().max())
        print(f"[parity] ingest {sr_in} -> 16000 Hz float32 stereo: max abs err {err:.2e}")
        assert err <= 1e-5        # float32 FIR of up to 475 taps, different summation order than the CPU conv1d
        one = ctx.audio_ingest(x.to(dev), sr_in, 16000, channel=1)          # io.py:232-233 channel selection
        ref1 = x[1:2] if sr_in == 16000 else AF.resample(x[1:2], sr_in, 16000)
        assert float((one.cpu() - ref1[0]).abs().max()) <= 1e-5
        # int16 interleaved PCM, as a WAV file holds it
        pcm = np.ascontiguousarray(np.clip(np.round(stereo.T * 32767.0), -32768, 32767).astype(np.int16))  # (frames, ch)
        reff = torch.from_numpy(pcm.T.astype(np.float32) / 32768.0).mean(dim=0, keepdim=True)
        if sr_in != 16000:
            reff = AF.resample(reff, sr_in, 16000)
        goti = ctx.audio_ingest(torch.from_numpy(pcm).to(dev), sr_in, 16000)
        assert float((goti.cpu() - reff[0]).abs().max()) <= 1e-5
    # same rate, mono: the kernel is the identity (bit-exact)
    same = ctx.audio_ingest(base.to(dev), 16000, 16000)
    assert torch.equal(same.cpu(), base[0])
    # through the pipeline: a 44.1 kHz stereo WAV file and the equivalent in-memory file give the same diarization
    # as the host-resampled mono waveform
    sr_in = 44100
    hi = AF.resample(syn.make_conversation(21.0, seed=19), 16000, sr_in)
    stereo = torch.cat([hi, 0.5 * hi], dim=0)
    pcm = np.ascontiguousarray(np.clip(np.round(stereo.numpy().T * 32767.0), -32768, 32767).astype(np.int16))
    path = tmp_path / "stereo44k.wav"
    wavfile.write(str(path), sr_in, pcm)
    audio = Audio(sample_rate=16000, mono="downmix")
    w_host, sr = audio(str(path))                                            # reference-style host path
    assert sr == 16000
    raw, sr_raw, ch = audio.raw(str(path))
    assert raw.dtype == torch.int16 and sr_raw == sr_in and audio.needs_ingest(raw, sr_raw)
    w_dev = audio.ingest(ctx, raw, sr_raw)
    assert w_dev.shape[0] == w_host.shape[1] == audio.num_samples_out(raw, sr_raw)
    assert float((w_dev.cpu() - w_host[0]).abs().max()) <= 1e-5
    out_file = pipeline(str(path))
    out_host = pipeline({"waveform": w_host, "sample_rate": 16000, "uri": "stereo44k"})
    a = [(s.start, s.end, lab) for s, _, lab in out_file.speaker_diarization.itertracks(yield_label=True)]
    b = [(s.start, s.end, lab) for s, _, lab in out_host.speaker_diarization.itertracks(yield_label=True)]
    assert a == b and out_file.speaker_diarization.uri == "stereo44k"


def test_aggregate_and_vad_on_device(dev, models, oracle_models):
    """Inference.aggregate on the device (bit-identical to numpy's arithmetic, NaN-aware,
    hamming / warm-up windows, skip_average) and the VoiceActivityDetection pipeline built on it."""
    from pyannote_audio_b200.inference import Inference
    from pyannote_audio_b200.core import SlidingWindow, SlidingWindowFeature
    from pyannote_audio_b200.vad import VoiceActivityDetection

    seg, _ = models
    oseg, _ = oracle_models
    rng = np.random.default_rng(21)
    inf = Inference(seg, duration=10.0, step=1.0, skip_aggregation=True)
    frames = SlidingWindow(start=FRAMES.start, duration=FRAMES.duration, step=FRAMES.step)
    for C, K, kw in ((1, 1, dict(hamming=True, missing=0.0)), (13, 3, dict(hamming=True, missing=0.0)),
                     (13, 3, dict(hamming=False, missing=np.nan, skip_average=True)),
                     (9, 2, dict(hamming=True, warm_up=(0.1, 0.05), missing=0.0))):
        data = rng.uniform(size=(C, 589, K)).astype(np.float32)
        data[rng.uniform(size=(C, 1, K)).repeat(589, 1) < 0.2] = np.nan          # whole (chunk, class) columns missing
        swf = SlidingWindowFeature(data, SlidingWindow(start=0.0, duration=10.0, step=1.0))
        got = inf.aggregate_device(swf, frames, **kw)
        ref = Inference.aggregate(swf, frames, **kw)                              # host numpy mirror of the reference
        oref = P.aggregate(P.SWF(data, P.SW(0.0, 10.0, 1.0)), FRAMES, **kw)
        assert got.data.shape == ref.data.shape == oref.data.shape
        assert np.array_equal(got.data, oref.data, equal_nan=True), (C, K, kw)
        assert np.array_equal(ref.data, oref.data, equal_nan=True)
    # VAD end to end
    wav = syn.make_conversation(47.3, seed=88)
    wav[:, 16000 * 20: 16000 * 24] = 0.0                                          # a real pause
    vad = VoiceActivityDetection(segmentation=seg, device=dev)
    scores = vad.speech_scores({"waveform": wav, "sample_rate": 16000})
    oscores = P.vad_scores(oseg, wav)
    _, ref_logp = P.slide(oseg, wav, return_logp=True)
    if _clear_margin(ref_logp).all():
        assert np.array_equal(scores.data, oscores.data)
    else:
        np.testing.assert_allclose(scores.data, oscores.data, atol=0.11)          # one low-margin frame of 10 chunks
    for params in ({}, {"min_duration_on": 0.3, "min_duration_off": 0.4}):
        vad.instantiate(params)
        seen = []
        speech = vad({"waveform": wav, "sample_rate": 16000, "uri": "vad"},
                     hook=lambda name, artifact, **k: seen.append(name))
        ref = P.binarize_scores(P.SWF(scores.data, oscores.sw), 0.5, 0.5, params.get("min_duration_on", 0.0),
                                params.get("min_duration_off", 0.0))
        got = [(s.start, s.end) for s, _, lab in speech.itertracks(yield_label=True)]
        assert got == [(a, b) for a, b, _ in ref] and set(speech.labels()) <= {"SPEECH"} and "segmentation" in seen
        assert speech.uri == "vad" and len(got) >= 1
