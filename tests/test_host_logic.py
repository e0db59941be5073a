"""CPU: host-side logic of the product package (no GPU, no compute calls into the CUDA library)."""

import numpy as np
import pytest
import torch

from oracle import nets, pipeline as P
from pyannote_audio_b200 import synthetic as syn
from pyannote_audio_b200.core import Annotation, Segment, SlidingWindow, SlidingWindowFeature
from pyannote_audio_b200.inference import Inference, chunk_layout
from pyannote_audio_b200.models import PyanNet, WeSpeakerResNet34
from pyannote_audio_b200.pipeline import binarize_frames, set_num_speakers


@pytest.mark.parametrize("T", [480000, 160000, 159999, 100, 176000, 176001, 9600000])
def test_chunk_layout_matches_oracle_chunking(T):
    off, valid, num_chunks, has_last = chunk_layout(T, 160000, 16000)
    if T <= 200000:
        wav = torch.arange(T, dtype=torch.float32)[None]
        chunks = P.chunk_waveform(wav)
        assert chunks.shape[0] == len(off)
        for c in range(len(off)):
            ref = chunks[c, 0].numpy()
            got = np.zeros(160000, dtype=np.float32)
            got[: valid[c]] = wav[0, off[c]: off[c] + valid[c]].numpy()
            assert np.array_equal(ref, got)
    assert len(off) == num_chunks + int(has_last)
    # 30 s -> 21 chunks, 10 min -> 591
    if T == 480000:
        assert len(off) == 21
    if T == 9600000:
        assert len(off) == 591


def test_inference_ctor_validation():
    # mirrors /root/reference/tests/inference_test.py:51-76
    model = PyanNet()
    with pytest.warns(UserWarning):
        Inference(model, duration=5.0)
    with pytest.raises(ValueError):
        Inference(model, step=20.0)
    with pytest.raises(ValueError):
        Inference(model, window="hopping")
    with pytest.warns(UserWarning):
        Inference(model, window="whole")
    inf = Inference(model, skip_aggregation=True)
    assert inf.duration == 10.0 and inf.step == 1.0
    with pytest.raises(TypeError):
        inf.to("cuda")


def test_models_have_reference_state_dict_keys():
    seg_sd, emb_sd = syn.make_segmentation_state_dict(0), syn.make_embedding_state_dict(1)
    m = PyanNet()
    m.load_state_dict(seg_sd, strict=True)            # exactly the reference's keys: nothing missing, nothing extra
    e = WeSpeakerResNet34()
    e.load_state_dict(emb_sd, strict=True)
    # oracle modules take the very same dicts (same key names as the reference)
    nets.PyanNet().load_state_dict(seg_sd, strict=True)
    nets.WeSpeakerResNet34().load_state_dict(emb_sd, strict=True)
    assert m.num_frames(160000) == 589 and m.receptive_field_size(1) == 991 and m.receptive_field_center(0) == 495
    rf = m.receptive_field
    assert (rf.start, rf.duration, rf.step) == (0.0, 991 / 16000, 270 / 16000)
    assert e.num_frames(160000) == 125


def test_models_refuse_cpu_forward():
    m = PyanNet()
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 1, 160000))


def test_binarize_frames_matches_oracle():
    rng = np.random.default_rng(0)
    frames = SlidingWindow(start=0.0, duration=991 / 16000, step=270 / 16000)
    for trial in range(5):
        d = (rng.uniform(size=(400, 3)) < 0.5).astype(np.uint8)
        d[:, 2] = 0 if trial == 0 else d[:, 2]
        if trial == 1:
            d[-5:, 0] = 1
            d[0, 1] = 1
        ann, rows = binarize_frames(d, frames)
        ref_rows, ref_times = P.binarize_to_segments(P.SWF(d.astype(np.float64), P.SW(0.0, 991 / 16000, 270 / 16000)))
        assert [tuple(r) for r in rows] == ref_rows
        got = [(s.start, s.end, lab) for s, _, lab in ann.itertracks(yield_label=True)]
        assert got == ref_times
        # the same from precomputed onset / offset events (what ops.Context.frame_transitions returns)
        n, K = d.shape
        act = np.zeros((K, n + 2), dtype=bool)
        act[:, 1:-1] = d.T > 0
        on = np.flatnonzero(act[:, 1:] & ~act[:, :-1])
        off = np.flatnonzero(act[:, :-1] & ~act[:, 1:])
        ann2, rows2 = binarize_frames(None, frames, events=(n, on, off))
        assert np.array_equal(rows2, rows)
        assert [(s.start, s.end, lab) for s, _, lab in ann2.itertracks(yield_label=True)] == got


def test_sliding_window_arithmetic_matches_oracle():
    sw = SlidingWindow(start=0.0, duration=991 / 16000, step=270 / 16000)
    osw = P.SW(0.0, 991 / 16000, 270 / 16000)
    for t in [0.0, 0.03, 1.0, 59.0 * 270 / 16000, 10.03096875, 3600.0]:
        assert sw.closest_frame(t) == osw.closest_frame(t)
    ts = np.arange(4000) * 1.0 + 0.5 * sw.duration
    assert np.array_equal(sw.closest_frames(ts), np.array([osw.closest_frame(t) for t in ts]))
    data = np.zeros((100, 2))
    swf = SlidingWindowFeature(data, sw)
    e = swf.extent
    assert (e.start, e.end) == osw.range_to_segment(0, 100)
    assert swf.crop(e, return_data=True).shape[0] == 100


def test_annotation_and_set_num_speakers():
    a = Annotation(uri="x")
    a.add(Segment(1.0, 2.0), 0, 1)
    a.add(Segment(0.5, 0.7), 1, 0)
    a.add(Segment(2.1, 3.0), 2, 1)
    assert a.labels() == [0, 1]
    assert [s.start for s in a.itersegments()] == [0.5, 1.0, 2.1]
    b = a.rename_labels({0: "SPEAKER_00", 1: "SPEAKER_01"})
    assert b.labels() == ["SPEAKER_00", "SPEAKER_01"]
    assert len(a.support(collar=0.2)) == 2
    assert "SPEAKER x 1 0.500 0.200" in b.to_rttm()
    assert set_num_speakers(None, None, None) == (None, 1, np.inf)
    assert set_num_speakers(3, None, None) == (3, 3, 3)
    with pytest.raises(ValueError):
        set_num_speakers(None, 4, 2)


def test_fcluster_host_matches_scipy():
    from scipy.cluster.hierarchy import fcluster, linkage

    from pyannote_audio_b200 import ops

    rng = np.random.default_rng(0)
    for _ in range(100):
        n = int(rng.integers(2, 80))
        X = rng.standard_normal((n, 8))
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        Z = linkage(X, "centroid", "euclidean")
        t = float(rng.uniform(0.2, 1.5))
        assert np.array_equal(fcluster(Z, t, "distance"), ops.fcluster_distance(Z, t))


def test_sinc_filter_bank_matches_oracle():
    from pyannote_audio_b200.ops import sinc_filter_bank

    sd = syn.make_segmentation_state_dict(0)
    p = "sincnet.conv1d.0.filterbank."
    bank = sinc_filter_bank(sd[p + "low_hz_"], sd[p + "band_hz_"], sd[p + "window_"], sd[p + "n_"])
    fb = nets.ParamSincFB()
    fb.load_state_dict({k[len(p):]: v for k, v in sd.items() if k.startswith(p)})
    assert torch.equal(bank, fb.filters()[:, 0, :])
    # (anti)symmetry the CUDA kernel relies on
    assert torch.equal(bank[:40], torch.flip(bank[:40], dims=[1]))
    assert torch.equal(bank[40:], -torch.flip(bank[40:], dims=[1]))


def test_product_plda_setup_matches_oracle():
    from pyannote_audio_b200.clustering import PLDA

    arrays = syn.make_plda(2)
    a, b = PLDA(arrays), P.PLDA(**arrays)
    np.testing.assert_allclose(a.phi, b.phi, rtol=1e-12)
    np.testing.assert_allclose(a._plda_tr, b._tr, rtol=1e-12, atol=1e-14)


def test_oracle_not_imported_by_product():
    import pathlib
    import re

    root = pathlib.Path(__file__).resolve().parents[1] / "pyannote_audio_b200"
    for f in root.rglob("*.py"):
        src = f.read_text()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports the oracle"


def test_annotation_integer_labels_relabel_like_object_labels():
    """Bulk annotations keep integer labels (one table lookup to relabel); same result as the object-label path."""
    from pyannote_audio_b200.core import Annotation
    rng = np.random.default_rng(3)
    n = 500
    starts = np.sort(rng.uniform(0, 100, n))
    ends = starts + rng.uniform(0.1, 2.0, n)
    lab = rng.integers(0, 7, n)
    a_int = Annotation.from_rows(starts, ends, lab, uri="u")
    a_obj = Annotation.from_rows(starts, ends, [int(v) for v in lab], uri="u")
    assert a_int.labels() == a_obj.labels() == sorted(set(lab.tolist()))
    mapping = {k: f"SPEAKER_{i:02d}" for i, k in enumerate(a_int.labels())}
    r_int, r_obj = a_int.rename_labels(mapping), a_int.rename_labels(mapping)
    got = [(s.start, s.end, l) for s, _, l in r_int.itertracks(yield_label=True)]
    ref = [(s.start, s.end, mapping[int(l)]) for s, _, l in a_obj.itertracks(yield_label=True)]
    assert got == ref and r_int.labels() == sorted(mapping.values())
    assert len(r_obj) == n and r_int.to_rttm().count("SPEAKER u 1") == n


def test_sparse_true_matches_flatnonzero():
    from pyannote_audio_b200.pipeline import _sparse_true
    rng = np.random.default_rng(4)
    for _ in range(50):
        x = rng.uniform(size=(int(rng.integers(1, 6)), int(rng.integers(1, 400)))) < rng.uniform(0, 0.3)
        assert np.array_equal(_sparse_true(x), np.flatnonzero(x))
    assert _sparse_true(np.zeros((3, 17), dtype=bool)).size == 0


# ---- checkpoints (core/model.py:497-655, core/plda.py:65-135) without lightning -------------------------------------
from pyannote_audio_b200.testing.checkpoints import reference_style_checkpoint as _reference_style_checkpoint  # noqa: E402


def test_from_pretrained_reads_reference_checkpoints(tmp_path):
    import io

    from pyannote_audio_b200.core import Problem, Resolution, Specifications
    from pyannote_audio_b200.models import Model

    blob, sd = _reference_style_checkpoint("seg")
    assert "pyannote.audio.core.task" not in __import__("sys").modules        # nothing of the reference is importable
    m = Model.from_pretrained(io.BytesIO(blob))
    assert isinstance(m, PyanNet) and isinstance(m.specifications, Specifications)
    assert m.specifications.problem is Problem.MONO_LABEL_CLASSIFICATION and m.specifications.powerset
    assert m.specifications.resolution is Resolution.FRAME and m.specifications.num_powerset_classes == 7
    for k, v in sd.items():
        assert torch.equal(m.state_dict()[k], v), k
    # directory form (+ subfolder), class check, kwargs override, hub ids refused offline
    d = tmp_path / "ckpt" / "segmentation"
    d.mkdir(parents=True)
    (d / "pytorch_model.bin").write_bytes(blob)
    assert isinstance(PyanNet.from_pretrained(tmp_path / "ckpt", subfolder="segmentation"), PyanNet)
    with pytest.raises(ValueError):
        WeSpeakerResNet34.from_pretrained(d / "pytorch_model.bin")
    with pytest.raises(ValueError):
        Model.from_pretrained("pyannote/segmentation-3.0")
    with pytest.raises(ValueError):
        Model.from_pretrained(d / "pytorch_model.bin", revision="main")
    blob_e, sd_e = _reference_style_checkpoint("emb")
    e = Model.from_pretrained(io.BytesIO(blob_e))
    assert isinstance(e, WeSpeakerResNet34) and e.specifications.resolution is Resolution.CHUNK
    assert torch.equal(e.state_dict()["resnet.seg_1.weight"], sd_e["resnet.seg_1.weight"])
    # PLDA.from_pretrained: directory with xvec_transform.npz + plda.npz (plda.py:97-105)
    p = syn.make_plda(2)
    np.savez(tmp_path / "xvec_transform.npz", mean1=p["mean1"], mean2=p["mean2"], lda=p["lda"])
    np.savez(tmp_path / "plda.npz", mu=p["mu"], tr=p["tr"], psi=p["psi"])
    from pyannote_audio_b200.clustering import PLDA

    a, b = PLDA.from_pretrained(tmp_path), PLDA(p)
    assert np.array_equal(a.phi, b.phi) and np.array_equal(a._plda_tr, b._plda_tr)
    with pytest.raises(ValueError):
        PLDA.from_pretrained("pyannote/speaker-diarization-community-1")


def test_weight_ownership_stamps():
    """Two models of one family on the same device share one context slot: the stamp protocol re-uploads whenever
    the resident weights are not the caller's (ADVICE r1); load_state_dict and .to() invalidate."""
    a, b = PyanNet(), PyanNet()
    assert a._model_id != b._model_id
    v = a._weights_version
    a.load_state_dict(syn.make_segmentation_state_dict(0), strict=True)
    assert a._weights_version == v + 1
    a.to(torch.device("cpu"))
    assert a._weights_version == v + 2
    assert "_dummy" not in a.state_dict()


def test_binarize_drops_empty_segments_and_support_is_strict():
    from pyannote_audio_b200.core import Annotation, Segment, SlidingWindow
    from pyannote_audio_b200.pipeline import binarize_frames

    fr = SlidingWindow(start=0.0, duration=0.0619375, step=0.016875)
    d = np.zeros((10, 2), dtype=np.uint8)
    d[2:5, 0] = 1
    d[9, 1] = 1                                   # onset at the very last frame: Segment(t, t) is empty -> dropped
    ann, rows = binarize_frames(d, fr)
    assert rows.tolist() == [[2, 5, 0]] and ann.labels() == [0]
    swf = P.SWF(d.astype(np.float64), P.SW(fr.start, fr.duration, fr.step))
    assert [list(r) for r in P.binarize_to_segments(swf)[0]] == rows.tolist()
    # support(collar): merge when the gap is < collar (strict) or empty (<= 1e-6), per label in sorted label order
    ann = Annotation()
    for s, e, lab in ((0.0, 1.0, "b"), (1.5, 2.0, "b"), (2.2, 3.0, "b"), (0.0, 1.0, "a"), (1.0, 2.0, "a")):
        ann.add(Segment(s, e), "_", lab)
    got = [(s.start, s.end, lab) for s, _, lab in ann.support(collar=0.5).itertracks(yield_label=True)]
    assert got == [(0.0, 1.0, "b"), (0.0, 2.0, "a"), (1.5, 3.0, "b")]         # gap 0.5 is NOT < 0.5; gap 0.2 is
    assert got == P.support([(0.0, 1.0, "b"), (1.5, 2.0, "b"), (2.2, 3.0, "b"), (0.0, 1.0, "a"), (1.0, 2.0, "a")], 0.5)
    ann.add(Segment(5.0, 5.0), "_", "c")          # empty segments are never stored
    assert "c" not in ann.labels()


def test_annotation_rttm_and_summaries():
    """The pyannote.core conveniences downstream code relies on (reference CLI: speaker_diarization.write_rttm(rttm),
    /root/reference/src/pyannote/audio/__main__.py:705-706)."""
    import io

    from pyannote_audio_b200.core import Annotation, Segment

    a = Annotation(uri="file1")
    a[Segment(0.5, 2.0), 1] = "SPEAKER_00"
    a[Segment(0.0, 1.0), 0] = "SPEAKER_00"
    a[Segment(3.0, 4.25), 2] = "SPEAKER_01"
    expected = ("SPEAKER file1 1 0.000 1.000 <NA> <NA> SPEAKER_00 <NA> <NA>\n"
                "SPEAKER file1 1 0.500 1.500 <NA> <NA> SPEAKER_00 <NA> <NA>\n"
                "SPEAKER file1 1 3.000 1.250 <NA> <NA> SPEAKER_01 <NA> <NA>\n")
    assert a.to_rttm() == expected
    f = io.StringIO()
    a.write_rttm(f)
    assert f.getvalue() == expected
    assert a.label_duration("SPEAKER_00") == 2.0 and a.label_duration("SPEAKER_01") == 1.25
    assert a.chart() == [("SPEAKER_00", 2.0), ("SPEAKER_01", 1.25)]
    assert a.get_timeline() == [Segment(0.0, 1.0), Segment(0.5, 2.0), Segment(3.0, 4.25)]
    with pytest.raises(ValueError, match="URIs containing spaces"):
        Annotation(uri="a b").to_rttm()
    bad = Annotation(uri="ok")
    bad[Segment(0, 1), 0] = "two words"
    with pytest.raises(ValueError, match="labels containing spaces"):
        bad.to_rttm()


def test_hooks_store_artifacts_and_timing():
    """Mirror of the reference's hook protocol (pipelines/utils/hook.py:37-239): artifacts are deep-copied into the
    file mapping, progress calls (artifact None) are ignored by ArtifactHook and drive TimingHook."""
    from pyannote_audio_b200.hooks import ArtifactHook, Hooks, TimingHook

    file = {"uri": "f"}
    data = np.arange(6).reshape(2, 3)
    with Hooks(ArtifactHook("segmentation", "embeddings"), TimingHook()) as hook:
        hook("segmentation", None, file=file, total=4, completed=0)
        hook("segmentation", None, file=file, total=4, completed=4)
        hook("segmentation", data, file=file)
        hook("speaker_counting", data, file=file)                       # not in the requested list
        hook("embeddings", None, file=file, total=1, completed=0)
        hook("embeddings", None, file=file, total=1, completed=1)
        hook("embeddings", data * 2, file=file)
    data[0, 0] = 99                                                     # stored artifacts are copies
    assert set(file["artifact"]) == {"segmentation", "embeddings"}
    assert file["artifact"]["segmentation"][0, 0] == 0 and file["artifact"]["embeddings"][1, 2] == 10
    assert set(file["timing"]) == {"total", "segmentation", "embeddings"}
    assert all(v >= 0.0 for v in file["timing"].values())
    with ArtifactHook() as everything:                                  # no names: keep every artifact
        everything("discrete_diarization", data, file=file)
    assert "discrete_diarization" in file["artifact"]
