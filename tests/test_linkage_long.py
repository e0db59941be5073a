"""Centroid linkage above 32 768 observations: the whole-GPU path over scipy's condensed distances.

* CPU: ``b200_linkage_bytes`` (the device bytes a linkage call needs) on both sides of the threshold;
* GPU: the whole-GPU path (forced with the ``linkage_grid_min`` option) against the one-CTA-per-problem kernel, bit for
  bit; against scipy's ``linkage(.., "centroid")`` / ``fcluster`` above the old 32 768 cap; mixed batches; and a
  recording of more than 32 768 kept embeddings through ``SpeakerDiarization`` (VBx and agglomerative) against the
  oracle fed with the pipeline's own segmentations and embeddings.
"""
import numpy as np
import pytest
import torch

from pyannote_audio_b200 import ops

GRID_MIN = 32769


# ---------------------------------------------------------------------------------------------------------
# CPU: the planner
# ---------------------------------------------------------------------------------------------------------
def _align(x, a=256):
    return (x + a - 1) // a * a


def _expected_bytes(sizes, dim):
    """The workspace of the batched kernel (dense matrices of the small problems, normalised rows, per-row state, job
    table) plus, with a problem above the threshold, the grid scratch and the packed distances of the largest one."""
    ntot, nf = sum(sizes), len(sizes)
    dense = sum(n * n for n in sizes if n < GRID_MIN)
    big = [n for n in sizes if n >= GRID_MIN]
    ws = _align(dense * 8) + _align(ntot * dim * 8) + (ntot + nf + 64) * 40 + nf * 24 + 8192
    if big:
        ws += 2 * 1024 * 16 + 256
    return ws + max((4 * n * (n - 1) for n in big), default=0)


@pytest.mark.parametrize("sizes,dim", [([2], 256), ([1000, 0, 1], 256), ([32768], 256), ([32769], 256),
                                       ([5, 40000, 300], 16), ([33000, 70000, 12], 8), ([0], 3)])
def test_linkage_bytes(sizes, dim):
    ro = np.concatenate([[0], np.cumsum(sizes)])
    assert ops.linkage_bytes(ro, dim) == _expected_bytes(sizes, dim)


def test_linkage_bytes_packed_size_is_64_bit():
    n = 70000
    got = ops.linkage_bytes([0, n], 256)
    packed = 4 * n * (n - 1)
    assert packed > 2 ** 34 and got >= packed
    assert got - packed == _expected_bytes([n], 256) - packed
    # the dense kernel's bytes at the threshold stay what they were: 8 n^2 in the workspace
    assert ops.linkage_bytes([0, 32768], 256) - ops.linkage_bytes([0, 2], 256) > 8 * 32768 ** 2 - 2 ** 27


def test_linkage_bytes_bad_arguments():
    from pyannote_audio_b200 import _lib

    lib = _lib.load()
    ro = np.array([0, 40, 30], dtype=np.int32)
    assert lib.b200_linkage_bytes(ro.ctypes.data, 2, 16) <= 0                 # decreasing offsets
    assert lib.b200_linkage_bytes(ro.ctypes.data, 0, 16) <= 0
    assert lib.b200_linkage_bytes(ro.ctypes.data, 1, 0) <= 0
    assert lib.b200_linkage_bytes(None, 1, 16) <= 0
    with pytest.raises(ValueError):
        ops.linkage_bytes([0, 40, 30], 16)


# ---------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ctx(dev):
    from pyannote_audio_b200.models import get_context

    return get_context(dev)


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _rows(rng, n, dim, dups=True):
    """Clustered rows holding float32 values; with ``dups`` exact duplicates (zero-distance ties) and
    near-duplicates."""
    centers = rng.standard_normal((9, dim))
    x = centers[rng.integers(0, 9, n)] + 0.5 * rng.standard_normal((n, dim))
    if dups and n >= 3:
        dup = rng.choice(n, size=max(1, n // 20), replace=False)
        x[dup] = x[rng.integers(0, n, size=dup.size)]
        near = rng.choice(n, size=max(1, n // 50), replace=False)
        x[near] = x[rng.integers(0, n, size=near.size)] * (1 + 1e-6 * rng.standard_normal((near.size, 1)))
    return x.astype(np.float32).astype(np.float64)


def _link(ctx, x, ro, normalize, grid_min):
    ctx.set_option("linkage_grid_min", grid_min)
    try:
        return ctx.linkage_centroid_batched(x, ro, normalize=normalize).cpu().numpy()
    finally:
        ctx.set_option("linkage_grid_min", GRID_MIN)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 256])
@pytest.mark.parametrize("n", [2, 3, 257, 4097, 20000, 32768])
def test_grid_path_matches_cta_kernel(ctx, dev, n, dim):
    rng = np.random.default_rng(n * 7 + dim)
    x = _t(_rows(rng, n, dim), dev)
    ro = [0, n]
    # the one-CTA kernel needs about 45 s at n = 32768, dim 256 on an H100: there only the pipeline's normalisation
    modes = ("float32",) if n * dim > 32768 * 16 else ("float32", True, False)
    for normalize in modes:
        Z_cta = _link(ctx, x, ro, normalize, GRID_MIN)
        Z_grid = _link(ctx, x, ro, normalize, 2)
        assert Z_grid.shape == (n - 1, 4)
        assert np.array_equal(Z_grid, Z_cta), f"n={n} dim={dim} normalize={normalize}"


def _same_partition(a, b):
    m = {}
    for x, y in zip(a, b):
        if m.setdefault(x, y) != y:
            return False
    return len(set(m.values())) == len(m)


@pytest.mark.gpu
@pytest.mark.parametrize("n,dim", [(33000, 8), (40000, 32)])
def test_grid_path_matches_scipy_above_old_cap(ctx, dev, n, dim):
    from scipy.cluster.hierarchy import fcluster, linkage

    rng = np.random.default_rng(n + dim)
    x = _rows(rng, n, dim, dups=(dim == 8))
    xn = x / np.linalg.norm(x, axis=1, keepdims=True)
    Z = ctx.linkage_centroid(_t(x, dev), normalize=True).cpu().numpy()
    ref = linkage(xn, "centroid", "euclidean")
    # scipy lists the merges sorted by height (centroid heights are not monotone); its distances may differ from the
    # device's in the last bit, as for the one-CTA kernel (test_clustering_kernels): heights to 1e-9, same partitions
    np.testing.assert_allclose(np.sort(Z[:, 2]), np.sort(ref[:, 2]), rtol=1e-9, atol=1e-12, err_msg=f"n={n}")
    assert np.array_equal(np.sort(Z[:, 3]), np.sort(ref[:, 3]))
    for t in (0.05, 0.2, 0.6):
        assert _same_partition(fcluster(ref, t, "distance"), ops.fcluster_distance(Z, t)), t


@pytest.mark.gpu
def test_mixed_batch_per_problem(ctx, dev):
    """One problem above the threshold between small ones, forward and reversed: each problem's Z rows are its solo
    run's."""
    rng = np.random.default_rng(5)
    sizes = [300, 2, 33500, 0, 4100, 17]
    xs = [_rows(rng, n, 16) if n else np.zeros((0, 16)) for n in sizes]
    alone = [ctx.linkage_centroid(_t(x, dev), normalize="float32").cpu().numpy() if len(x) >= 2 else None for x in xs]
    for order in (list(range(len(sizes))), list(range(len(sizes)))[::-1]):
        ro = np.concatenate([[0], np.cumsum([sizes[f] for f in order])]).astype(np.int32)
        Z = ctx.linkage_centroid_batched(_t(np.concatenate([xs[f] for f in order]), dev), ro,
                                         normalize="float32").cpu().numpy()
        z = 0
        for f in order:
            rows = max(sizes[f] - 1, 0)
            if rows:
                assert np.array_equal(Z[z: z + rows], alone[f]), f"n={sizes[f]}"
            z += rows
        assert z == len(Z)


# ---------------------------------------------------------------------------------------------------------
# GPU end to end: a recording of more than 32 768 kept embeddings
# ---------------------------------------------------------------------------------------------------------
PLDA_SEED = 2
HOURS = 5


@pytest.fixture(scope="module")
def long_wave():
    from pyannote_audio_b200 import synthetic as syn

    # three distinct synthetic hours, played in turn: the repeats add exact duplicate embeddings (ties)
    hours = [syn.make_conversation(3600.0, seed=500 + h) for h in range(3)]
    return torch.cat([hours[h % 3] for h in range(HOURS)], dim=1)


@pytest.fixture(scope="module")
def cached_scipy_linkage():
    """The oracle's VBx and AHC both run scipy's linkage on the same normalised float32 rows: compute it once."""
    from scipy.cluster import hierarchy

    from oracle import pipeline as P

    cache = {}

    def linkage(y, method="single", metric="euclidean", **kw):
        key = (np.asarray(y).tobytes(), np.asarray(y).shape, method, metric)
        if key not in cache:
            cache[key] = hierarchy.linkage(y, method=method, metric=metric, **kw)
        return cache[key].copy()

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(P, "linkage", linkage)
        yield cache


def _pipeline(dev, clustering):
    from pyannote_audio_b200 import synthetic as syn
    from pyannote_audio_b200.models import PyanNet, WeSpeakerResNet34
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    seg, emb = PyanNet(), WeSpeakerResNet34()
    seg.load_state_dict(syn.make_segmentation_state_dict(0), strict=False)
    emb.load_state_dict(syn.make_embedding_state_dict(1), strict=False)
    return SpeakerDiarization(segmentation=seg, embedding=emb, plda=syn.make_plda(PLDA_SEED), clustering=clustering,
                              device=dev)


def _tracks(annotation):
    return [(s.start, s.end, lab) for s, _, lab in annotation.itertracks(yield_label=True)]


@pytest.mark.gpu
@pytest.mark.parametrize("clustering", ["VBxClustering", "AgglomerativeClustering"])
def test_long_recording_end_to_end(dev, long_wave, cached_scipy_linkage, clustering):
    from oracle import pipeline as P
    from pyannote_audio_b200 import synthetic as syn

    pipe = _pipeline(dev, clustering)
    (_, (out, art)), = list(pipe.apply_batch([{"waveform": long_wave, "sample_rate": 16000, "uri": "long"}],
                                             return_artifacts=True))
    seg = art["segmentations"].cpu().numpy().astype(np.float32)
    emb = art["embeddings"].cpu().numpy()
    train, _, _ = P.filter_embeddings(emb, seg)
    n = train.shape[0]
    print(f"[linkage-long] {clustering}: {seg.shape[0]} chunks, {n} kept embeddings")
    assert n > 32768, f"only {n} kept embeddings: the whole-GPU linkage path is not exercised"
    sw = P.SWF(seg, P.SW(0.0, 10.0, 1.0))
    if clustering == "VBxClustering":
        ref = P.apply(None, None, P.PLDA(**syn.make_plda(PLDA_SEED)), long_wave, segmentations=sw, embeddings=emb)
        hard_ref, times_ref = ref.hard_clusters, ref.times
    else:
        params = pipe.default_parameters()["clustering"]
        hard_ref, _, _ = P.ahc_call(emb, seg, params["threshold"], params["min_cluster_size"])
        hard_ref = hard_ref.astype(np.int8)
        hard_ref[seg.sum(1) == 0] = -2
        count = P.speaker_count(sw, P.SW(*P.nets.sincnet_receptive_field()))
        count.data = count.data.astype(np.int8)
        _, times = P.binarize_to_segments(P.reconstruct(sw, hard_ref, count))
        labels = sorted({k for _, _, k in times})
        mapping = {k: f"SPEAKER_{i:02d}" for i, k in enumerate(labels)}
        times_ref = [(a, b, mapping[k]) for a, b, k in times]
    assert np.array_equal(art["hard_clusters"], hard_ref)
    assert _tracks(out.speaker_diarization) == times_ref
