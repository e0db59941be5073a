"""GPU tests of multi-file batches against per-file results (pytest -m gpu).

``SpeakerDiarization.apply_batch`` / ``run_resident`` run all files of a batch through shared launches, and
``VBxClustering.cluster_batch`` clusters them together (one linkage launch, one VBx launch, host bookkeeping that
slices the results back per file).  Every file's result must be what the oracle computes for that file alone,
whatever else is in the batch and in whatever order.  Also: NaN embedding rows through the public clustering classes.
"""
import numpy as np
import pytest
import torch

from oracle import pipeline as P
from pyannote_audio_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

PLDA_SEED = 2


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def oplda():
    return P.PLDA(**syn.make_plda(PLDA_SEED))


@pytest.fixture(scope="module")
def vbx(dev):
    from pyannote_audio_b200.clustering import PLDA, VBxClustering

    return VBxClustering(PLDA(syn.make_plda(PLDA_SEED)), device=dev)


# ---------------------------------------------------------------------------------------------------------
# cluster_batch on constructed files
# ---------------------------------------------------------------------------------------------------------
def _turns(rng, C, keep_third=True):
    """Non-overlapping turns of the three local speakers per chunk, as in test_clustering_class_seams."""
    seg = np.zeros((C, 589, 3), dtype=np.float32)
    for c in range(C):
        cuts = np.sort(rng.integers(0, 589, size=2))
        seg[c, : cuts[0], 0] = 1
        seg[c, cuts[0]: cuts[1], 1] = 1
        if c % 7 and keep_third:
            seg[c, cuts[1]:, 2] = 1
    return seg


def _speakers(rng, C, k, spread=0.35):
    centers = rng.standard_normal((k, 256))
    return (centers[rng.integers(0, k, size=(C, 3))] + spread * rng.standard_normal((C, 3, 256))).astype(np.float32)


def _make_files(seed=40):
    """name -> (embeddings (C,3,256) f32, segmentation (C,589,3) f32, silent)."""
    rng = np.random.default_rng(seed)
    files = {}
    files["silent"] = (_speakers(rng, 12, 3), np.zeros((12, 589, 3), dtype=np.float32), True)
    overlap = np.ones((5, 589, 3), dtype=np.float32)                   # speech, but never one speaker alone
    files["n0"] = (_speakers(rng, 5, 2), overlap, False)
    seg = np.ones((4, 589, 3), dtype=np.float32)
    seg[0] = 0
    seg[0, :, 0] = 1                                                   # one clean (chunk, speaker)
    files["n1"] = (_speakers(rng, 4, 2), seg, False)
    seg = np.ones((3, 589, 3), dtype=np.float32)
    seg[1] = 0
    seg[1, :300, 0] = 1
    seg[1, 300:, 1] = 1                                                # two clean (chunk, speaker)
    files["n2"] = (_speakers(rng, 3, 2), seg, False)
    seg = np.zeros((30, 589, 3), dtype=np.float32)
    seg[:, :, 0] = 1
    seg[::4, 400:, 0] = 0
    files["single"] = (_speakers(rng, 30, 1), seg, False)
    files["many"] = (_speakers(rng, 70, 12, spread=0.25), _turns(rng, 70), False)   # > 8 AHC clusters
    emb = _speakers(rng, 40, 3)
    emb[[2, 9, 9, 17, 33], [0, 1, 2, 0, 2]] = np.nan                   # NaN embedding rows
    files["nan"] = (emb, _turns(rng, 40), False)
    files["plain"] = (_speakers(rng, 50, 3), _turns(rng, 50), False)
    files["plain4"] = (_speakers(rng, 90, 4), _turns(rng, 90), False)
    return files


def _run_batch(vbx, dev, files, names, **kw):
    embs = [files[n][0] for n in names]
    segs = [files[n][1] for n in names]
    bounds = np.cumsum([0] + [len(e) for e in embs])
    emb_all = torch.from_numpy(np.concatenate(embs)).to(dev)
    seg_all = torch.from_numpy(np.concatenate(segs).astype(np.uint8)).to(dev)
    return vbx.cluster_batch(emb_all, seg_all, bounds, skip=[files[n][2] for n in names], **kw)


def _check_file(r, name, emb, seg, silent, oplda, kmeans=False, **kw):
    if silent:
        assert r is None, name
        return
    oh, osoft, oc = P.vbx_clustering(emb, seg, oplda, **kw)
    hard, soft, cent = r["hard"].cpu().numpy(), r["soft"].cpu().numpy(), r["centroids"].cpu().numpy()
    assert hard.dtype == np.int8 and np.array_equal(hard, oh), name
    assert soft.shape == osoft.shape and cent.shape == oc.shape, name
    if kmeans:                                          # the reference averages float32 rows here
        np.testing.assert_allclose(cent, oc, rtol=1e-5, atol=1e-6, err_msg=name)
        np.testing.assert_allclose(soft, osoft, rtol=0, atol=1e-6, equal_nan=True, err_msg=name)
    else:
        np.testing.assert_allclose(cent, oc, rtol=1e-9, atol=1e-12, equal_nan=True, err_msg=name)
        np.testing.assert_allclose(soft, osoft, rtol=1e-9, atol=1e-12, equal_nan=True, err_msg=name)


NONTRIVIAL = ["many", "n2", "nan", "single", "plain", "plain4"]
MIXED = ["plain", "silent", "n0", "many", "n1", "nan", "n2", "single", "plain4"]


def test_cluster_batch_matches_per_file_oracle(dev, vbx, oplda):
    files = _make_files()
    # the filter gives the intended training-set sizes
    for name, want in (("n0", 0), ("n1", 1), ("n2", 2)):
        train, _, _ = P.filter_embeddings(files[name][0], files[name][1])
        assert len(train) == want, name
    ahc, _, _ = P.ahc_centroid_labels(P.filter_embeddings(*files["many"][:2])[0], 0.6)
    assert ahc.max() + 1 > 8, "the > 8 cluster file does not have more than 8 AHC clusters"
    for names in (NONTRIVIAL, NONTRIVIAL[::-1], MIXED, MIXED[::-1]):
        results = _run_batch(vbx, dev, files, names)
        assert len(results) == len(names)
        for name, r in zip(names, results):
            _check_file(r, name, *files[name], oplda)
        for name, r in zip(names, results):
            if r is not None and not r["trivial"]:       # the AHC cut and VBx of this file alone
                dbg_ref = P.vbx_clustering(*files[name][:2], oplda, return_debug=True)[3]
                assert np.array_equal(r["ahc"], dbg_ref["ahc"]), name
                np.testing.assert_allclose(r["q"].cpu().numpy(), dbg_ref["q"], rtol=1e-8, atol=1e-10, err_msg=name)


@pytest.mark.parametrize("kw", [dict(num_clusters=2, min_clusters=2, max_clusters=2), dict(min_clusters=5),
                                dict(max_clusters=2)])
def test_cluster_batch_forced_counts(dev, vbx, oplda, kw):
    """num / min / max clusters: the per-file KMeans fallback (clustering.py:626-642) where the VBx count is out of
    bounds, plain VBx elsewhere."""
    files = _make_files()
    names = [n for n in NONTRIVIAL if kw.get("min_clusters", 1) <= 2 or n != "n2"]
    results = _run_batch(vbx, dev, files, names, **kw)
    for name, r in zip(names, results):
        emb, seg, silent = files[name]
        auto = P.vbx_clustering(emb, seg, oplda)[2].shape[0]
        forced = auto < kw.get("min_clusters", 1) or auto > kw.get("max_clusters", np.inf) or \
            (kw.get("num_clusters") and kw["num_clusters"] != auto)
        _check_file(r, name, emb, seg, silent, oplda, kmeans=bool(forced), **kw)


# ---------------------------------------------------------------------------------------------------------
# NaN embeddings through the public classes
# ---------------------------------------------------------------------------------------------------------
def test_nan_embeddings_public_classes(dev, vbx, oplda):
    from pyannote_audio_b200.clustering import AgglomerativeClustering

    emb, seg, _ = _make_files()["nan"]
    hard, soft, cent = vbx(embeddings=emb, segmentations=seg)
    oh, osoft, oc = P.vbx_clustering(emb, seg, oplda)
    assert np.isnan(osoft).any()
    assert np.array_equal(hard, oh)
    np.testing.assert_allclose(soft, osoft, rtol=1e-9, atol=1e-12, equal_nan=True)
    np.testing.assert_allclose(cent, oc, rtol=1e-9, atol=1e-12)
    for constrained in (False, True):
        ahc = AgglomerativeClustering(constrained_assignment=constrained, device=dev)
        ahc.instantiate(dict(method="centroid", threshold=0.9, min_cluster_size=5))
        h, s_, c_ = ahc(embeddings=emb, segmentations=seg)
        rh, rs, rc = P.ahc_call(emb, seg, 0.9, 5, constrained=constrained)
        assert np.array_equal(h, rh), constrained
        np.testing.assert_allclose(c_, rc, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(s_, rs, rtol=0, atol=1e-6, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------
# apply_batch / run_resident end to end
# ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pipeline(dev):
    from pyannote_audio_b200.models import PyanNet, WeSpeakerResNet34
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    seg, emb = PyanNet(), WeSpeakerResNet34()
    seg.load_state_dict(syn.make_segmentation_state_dict(0), strict=False)
    emb.load_state_dict(syn.make_embedding_state_dict(1), strict=False)
    return SpeakerDiarization(segmentation=seg, embedding=emb, plda=syn.make_plda(PLDA_SEED), device=dev)


def _rows(x):
    return [tuple(int(v) for v in r) for r in x]


def _compare_with_oracle(art, out, ref):
    """Integer outputs of the CUDA pipeline against the oracle re-fed with the same segmentation and embeddings."""
    assert np.array_equal(art["count"].cpu().numpy(), ref.count.data[:, 0])
    assert np.array_equal(art["hard_clusters"], ref.hard_clusters)
    assert np.array_equal(art["discrete"][:, : ref.discrete.data.shape[1]], ref.discrete.data.astype(np.uint8))
    assert not art["discrete"][:, ref.discrete.data.shape[1]:].any()
    assert np.array_equal(art["exclusive"][:, : ref.exclusive.data.shape[1]], ref.exclusive.data.astype(np.uint8))
    assert _rows(art["segments"]) == _rows(ref.segments)
    assert _rows(art["exclusive_segments"]) == _rows(ref.exclusive_segments)
    got = [(s.start, s.end, lab) for s, _, lab in out.speaker_diarization.itertracks(yield_label=True)]
    assert got == ref.times
    gotx = [(s.start, s.end, lab) for s, _, lab in out.exclusive_speaker_diarization.itertracks(yield_label=True)]
    assert gotx == ref.exclusive_times


def _batch_files(tmp_path):
    import torchaudio.functional as AF
    from scipy.io import wavfile

    files = [{"waveform": torch.zeros(1, 16000 * 12), "sample_rate": 16000, "uri": "silence"},
             {"waveform": syn.make_conversation(3.0, seed=2), "sample_rate": 16000, "uri": "short"},
             {"waveform": syn.make_conversation(10.0, seed=3)[:, :160000], "sample_rate": 16000, "uri": "one-chunk"},
             {"waveform": syn.make_conversation(37.3, seed=11), "sample_rate": 16000, "uri": "ragged"},
             {"waveform": syn.make_conversation(75.0, seed=1234), "sample_rate": 16000, "uri": "e2e-75s"}]
    assert files[2]["waveform"].shape[1] == 160000
    hi = AF.resample(syn.make_conversation(21.0, seed=19), 16000, 44100)
    stereo = torch.cat([hi, 0.5 * hi], dim=0)
    pcm = np.ascontiguousarray(np.clip(np.round(stereo.numpy().T * 32767.0), -32768, 32767).astype(np.int16))
    path = tmp_path / "stereo44k.wav"
    wavfile.write(str(path), 44100, pcm)
    files.append({"audio": str(path), "uri": "stereo44k"})              # int16 stereo: device ingest
    return files


def _uri(f):
    return f["uri"]


def test_apply_batch_per_file(pipeline, tmp_path):
    files = _batch_files(tmp_path)
    plda = P.PLDA(**syn.make_plda(PLDA_SEED))
    alone = {}
    for f in files:
        (_, (out, art)), = list(pipeline.apply_batch([dict(f)], return_artifacts=True))
        alone[_uri(f)] = art
    for order in (files, files[::-1]):
        seen = {}
        hook = lambda step, artifact, file=None, **k: seen.setdefault(file["uri"], []).append((step, artifact is None))  # noqa: E731
        batch = list(pipeline.apply_batch([dict(f) for f in order], hook=hook, return_artifacts=True))
        assert [_uri(f) for f, _ in batch] == [_uri(f) for f in order]
        for f, (out, art) in batch:
            uri = _uri(f)
            a = alone[uri]
            seg = art["segmentations"].cpu().numpy()
            assert torch.equal(art["classes"], a["classes"]), f"{uri}: segmentation depends on the batch"
            assert np.array_equal(seg, a["segmentations"].cpu().numpy())
            names = [n for n, progress in seen[uri] if not progress]
            if int(art["count"].max()) == 0:              # no speech at all: skipped by the clustering
                assert len(out.speaker_diarization) == 0 and out.speaker_embeddings.shape == (0, 256)
                assert names == ["segmentation", "speaker_counting"], uri
                continue
            assert names == ["segmentation", "speaker_counting", "embeddings", "discrete_diarization"], uri
            # the embedding sub-batches (emb_max_batch) and the shared fbank frames differ between the batch and the
            # file alone; a chunk's arithmetic does not depend on them
            emb = art["embeddings"].cpu().numpy()
            assert np.array_equal(emb, a["embeddings"].cpu().numpy()), f"{uri}: embeddings depend on the batch"
            wav = f["waveform"] if "waveform" in f else None
            ref = P.apply(None, None, plda, wav, segmentations=P.SWF(seg.astype(np.float32), P.SW(0.0, 10.0, 1.0)),
                          embeddings=emb)
            _compare_with_oracle(art, out, ref)
            np.testing.assert_allclose(out.speaker_embeddings, ref.speaker_embeddings, rtol=1e-6, atol=1e-8)
