"""CPU: the oracle's pipeline-level restatements against vectors produced by EXECUTING the reference's own files
(core/inference.py, utils/signal.py, pipelines/utils/diarization.py, pipelines/clustering.py, core/plda.py,
pipelines/speaker_diarization.py) -- tests/golden/make_golden_pipeline.py, reference_pipeline_vectors.npz.
Integer / index results must be identical, float results equal to the last bit where the arithmetic is the same
sequence of numpy operations (aggregate) and to 1e-12 otherwise."""
import os

import numpy as np
import pytest

from oracle import nets, pipeline as P
from pyannote_audio_b200 import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FRAMES = P.SW(*nets.sincnet_receptive_field())
CHUNKS = P.SW(0.0, 10.0, 1.0)


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_pipeline_vectors.npz"))


def _sw(a):
    return P.SW(float(a[0]), float(a[1]), float(a[2]))


def test_receptive_field_of_the_generator_is_the_oracles():
    assert (FRAMES.start, FRAMES.duration, FRAMES.step) == (0.0, 0.0619375, 0.016875)


def test_aggregate_and_trim_match_reference_inference(ref):
    scores = ref["agg_scores"]
    for name, kw in (("plain", dict()), ("hamming", dict(hamming=True)), ("warm", dict(warm_up=(1.0, 1.5), hamming=True)),
                     ("skip", dict(skip_average=True, missing=0.0)), ("missing0", dict(missing=0.0))):
        got = P.aggregate(P.SWF(scores.copy(), CHUNKS), FRAMES, **kw)
        np.testing.assert_array_equal(got.data, ref[f"agg_{name}"], err_msg=name)     # NaNs in the same places too
        assert got.data.dtype == ref[f"agg_{name}"].dtype
        assert (got.sw.start, got.sw.duration, got.sw.step) == tuple(ref[f"agg_{name}_sw"])
    tr = P.trim(P.SWF(scores.copy(), CHUNKS), warm_up=(0.1, 0.05))
    assert tuple(tr.data.shape) == tuple(ref["trim_data_shape"])
    np.testing.assert_allclose([tr.sw.start, tr.sw.duration, tr.sw.step], ref["trim_sw"], rtol=0, atol=1e-15)


def test_speaker_count_reconstruct_and_annotation_match_reference(ref):
    binar = ref["bin_seg"].astype(np.float32)
    for name, wu in (("w0", (0.0, 0.0)), ("w1", (0.1, 0.1))):
        cnt = P.speaker_count(P.SWF(binar.copy(), CHUNKS), FRAMES, warm_up=wu)
        np.testing.assert_array_equal(cnt.data, ref[f"count_{name}"])
        assert cnt.data.dtype == np.uint8
        np.testing.assert_allclose([cnt.sw.start, cnt.sw.duration, cnt.sw.step], ref[f"count_{name}_sw"], atol=1e-15)
    count = P.speaker_count(P.SWF(binar.copy(), CHUNKS), FRAMES, warm_up=(0.0, 0.0))
    hard = ref["rec_hard"]
    for name, cmax in (("full", None), ("cap1", 1)):
        c = P.SWF(count.data.copy(), count.sw)
        if cmax is not None:
            c.data = np.minimum(c.data, cmax).astype(np.int8)
        # (the reference sorts with numpy's default argsort, the oracle with a stable one: identical here)
        disc = P.reconstruct(P.SWF(binar.copy(), CHUNKS), hard, c)
        want = ref[f"rec_{name}"]
        np.testing.assert_allclose([disc.sw.start, disc.sw.duration, disc.sw.step], ref[f"rec_{name}_sw"], atol=1e-15)
        # The reference picks the `count` most active clusters with numpy's DEFAULT argsort, whose order of equal
        # activations depends on the numpy build (x86-simd-sort on AVX-512 / AVX2 is not stable); the oracle fixes it
        # as "descending activation, then ascending cluster index".  So: identical wherever the
        # choice is unique, and on every other frame both picked the same NUMBER of clusters with the same activations.
        act = P.aggregate(P.clustered_segmentations(P.SWF(binar.copy(), CHUNKS), hard), c.sw, hamming=False,
                          missing=0.0, skip_average=True).data[: len(want)]
        assert disc.data.shape == want.shape
        differ = np.nonzero((disc.data != want).any(axis=1))[0]
        np.testing.assert_array_equal(disc.data.sum(axis=1), want.sum(axis=1))
        for t in differ:
            assert sorted(act[t][disc.data[t] > 0]) == sorted(act[t][want[t] > 0]), f"frame {t}: not a tie"
        assert len(differ) < 0.2 * len(want)                # random cluster labels: ties are frequent here
        print(f"[reconstruct {name}] {len(differ)} of {len(want)} frames differ from the reference's run, all of them ties")
        # Binarize of the reference's own matrix: the oracle's run-length encoding on the same input
        disc = P.SWF(want, disc.sw)
        rows, times = P.binarize_to_segments(disc)
        want = ref[f"ann_{name}"]
        assert len(times) == len(want)
        np.testing.assert_array_equal(np.array([t[2] for t in times], dtype=np.float64), want[:, 2])
        np.testing.assert_array_equal(np.array([[t[0], t[1]] for t in times]), want[:, :2])      # same float times


def test_binarize_hysteresis_matches_reference_signal(ref):
    got = P.binarize_scores(P.SWF(ref["binz_scores"], FRAMES), onset=0.6, offset=0.4)
    want = ref["binz_rows"]
    assert len(got) == len(want) and len(want) > 4
    np.testing.assert_array_equal(np.array(got, dtype=np.float64), want)


def test_set_num_speakers_matches_reference(ref):
    from pyannote_audio_b200.pipeline import set_num_speakers

    for args, want in zip(((None, None, None), (3, None, None), (None, 2, 5), (None, 4, 4)), ref["set_num_speakers"]):
        got = [np.nan if v is None else float(v) for v in set_num_speakers(*args)]
        np.testing.assert_array_equal(np.array(got), want)


def test_clustering_matches_reference_clustering(ref):
    seg, emb = ref["cl_seg"].astype(np.float32), ref["cl_emb"].astype(np.float64)
    train, ci, si = P.filter_embeddings(emb, seg)
    np.testing.assert_array_equal(ci, ref["cl_filter_chunk"])
    np.testing.assert_array_equal(si, ref["cl_filter_speaker"])
    np.testing.assert_array_equal(P.constrained_argmax(ref["carg_soft"].copy()), ref["carg_hard"])
    plda = P.PLDA(**syn.make_plda(2))
    for name, kw in (("auto", dict(num_clusters=None, min_clusters=1, max_clusters=np.inf)),
                     ("forced2", dict(num_clusters=2, min_clusters=2, max_clusters=2)),
                     ("max2", dict(num_clusters=None, min_clusters=1, max_clusters=2)),
                     ("min5", dict(num_clusters=None, min_clusters=5, max_clusters=np.inf))):
        hard, soft, cent = P.vbx_clustering(emb.copy(), seg.copy(), plda, threshold=0.6, Fa=0.07, Fb=0.8, **kw)
        np.testing.assert_array_equal(hard, ref[f"vbx_{name}_hard"], err_msg=name)
        assert cent.shape[0] == dict(auto=3, forced2=2, max2=2, min5=5)[name]      # 6 sessions -> 3 speakers; KMeans paths
        np.testing.assert_allclose(cent, ref[f"vbx_{name}_centroids"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(soft, ref[f"vbx_{name}_soft"], rtol=0, atol=1e-12)
    hard, soft, cent = P.vbx_clustering(ref["cl_emb"].copy(), seg.copy(), plda, threshold=0.6, Fa=0.07, Fb=0.8,
                                        num_clusters=None, min_clusters=1, max_clusters=np.inf)      # float32 embeddings
    np.testing.assert_array_equal(hard, ref["vbx_f32_hard"])
    np.testing.assert_allclose(cent, ref["vbx_f32_centroids"], rtol=0, atol=1e-6)
    assert cent.dtype == ref["vbx_f32_centroids"].dtype
    for name, kw in (("auto", dict()), ("forced3", dict(num_clusters=3)), ("min5", dict(min_clusters=5, max_clusters=20))):
        hard, soft, cent = P.ahc_call(emb.copy(), seg.copy(), threshold=0.7, min_cluster_size=4, method="centroid", **kw)
        np.testing.assert_array_equal(hard, ref[f"ahc_{name}_hard"], err_msg=name)
        np.testing.assert_allclose(cent, ref[f"ahc_{name}_centroids"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(soft, ref[f"ahc_{name}_soft"], rtol=0, atol=1e-12)
