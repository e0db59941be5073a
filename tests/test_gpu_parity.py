"""GPU parity tests (pytest -m gpu): every check goes through the C ABI (pyannote_audio_b200.ops / the public API)
and compares against the CPU oracle on the same seeded inputs.  Tolerances:
  * integer / index outputs (classes, counts, discrete diarization, segment frame indices, partitions): bit-exact
  * segmentation log-probabilities (fp32 both sides, different summation order): 2e-4 absolute
  * embeddings (fp16 tensor-core trunk vs fp32 oracle): cosine distance <= 1e-3 (BASELINE.json north_star)
  * fp64 clustering arithmetic: 1e-9
"""
import numpy as np
import pytest
import torch

from oracle import nets, pipeline as P
from pyannote_audio_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

FRAMES = P.SW(*nets.sincnet_receptive_field())


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ctx(dev):
    from pyannote_audio_b200.models import get_context

    c = get_context(dev)
    c.load_segmentation(syn.make_segmentation_state_dict(0))
    c.load_embedding(syn.make_embedding_state_dict(1))
    return c


@pytest.fixture(scope="module")
def oracle_models():
    seg = nets.PyanNet()
    seg.load_state_dict(syn.make_segmentation_state_dict(0))
    emb = nets.WeSpeakerResNet34()
    emb.load_state_dict(syn.make_embedding_state_dict(1))
    return seg.eval(), emb.eval()


LOW_MARGIN = 1e-4          # top-2 log-probability margin under which an argmax flip is fp32 reordering noise


def _class_mismatches(cls, ref_logp):
    """(mismatch mask, low-margin mask) of CUDA class ids against the oracle's log-probabilities."""
    top2 = np.sort(ref_logp, axis=-1)
    low = (top2[..., -1] - top2[..., -2]) < LOW_MARGIN
    return cls != ref_logp.argmax(-1), low


def _report(name, mism, low):
    print(f"[parity] {name}: {mism.size} frames, {int(low.sum())} low-margin (< {LOW_MARGIN:g}), "
          f"{int(mism.sum())} class mismatches ({int((mism & low).sum())} of them low-margin)")


def _device_wave(wav, dev):
    from pyannote_audio_b200.inference import chunk_layout

    T = wav.shape[1]
    off, valid, _, _ = chunk_layout(T, 160000, 16000)
    buf = torch.zeros(int(off[-1]) + 160000, dtype=torch.float32, device=dev)
    buf[:T] = wav[0].to(dev)
    return buf, off, valid


def _diagnose_sincnet(ctx, buf, off, valid, first, ref):
    import subprocess

    def worst(a):
        d = np.abs(a - ref).reshape(a.shape[0], -1).max(axis=1)
        return f"max {d.max():.2e}, chunks over 2e-4: {np.nonzero(d > 2e-4)[0].tolist()}"

    print(f"[sincnet diagnosis] first call: {worst(first)}")
    for name, mode in (("tensor-core again", 1), ("fp32 CUDA-core twin", 0)):
        ctx.set_option("seg_conv_impl", mode)
        out = ctx.sincnet_forward(buf, off, valid).cpu().numpy()
        print(f"[sincnet diagnosis] {name}: {worst(out)}; equal to the first call: {np.array_equal(out, first)}")
    ctx.set_option("seg_conv_impl", 1)
    try:
        print("[sincnet diagnosis] " + subprocess.run(
            ["nvidia-smi", "--query-gpu=name,serial,uuid,clocks.sm,temperature.gpu,ecc.errors.uncorrected.volatile.total",
             "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip())
    except Exception as exc:                                # diagnostics only
        print(f"[sincnet diagnosis] nvidia-smi: {exc}")


# ---------------------------------------------------------------------------------------------------------
def test_stats_pool_known_answers_cuda(ctx, dev, golden):
    # /root/reference/tests/test_stats_pool.py:28-131, through b200_stats_pool
    r4 = lambda t: torch.round(t.cpu(), decimals=4)  # noqa: E731
    x = torch.tensor([[[2.0, 4.0], [2.0, 4.0]], [[1.0, 1.0], [1.0, 1.0]]], device=dev)
    assert torch.equal(r4(ctx.stats_pool(x)), torch.Tensor([[3.0, 3.0, 1.4142, 1.4142], [1.0, 1.0, 0.0, 0.0]]))
    w = torch.tensor([[0.5, 0.01], [0.2, 0.1]], device=dev)
    assert torch.equal(r4(ctx.stats_pool(x, w)), torch.Tensor([[2.0392, 2.0392, 1.4142, 1.4142], [1.0, 1.0, 0.0, 0.0]]))
    assert torch.equal(r4(ctx.stats_pool(x, torch.zeros(2, 2, device=dev))), torch.zeros(2, 4))
    # vectors produced by the reference's pooling.py (incl. nearest interpolation of 5 weights onto 11 frames)
    xs = torch.from_numpy(golden["sp_x"]).to(dev)
    np.testing.assert_allclose(ctx.stats_pool(xs).cpu().numpy(), golden["sp_y_none"], atol=2e-6)
    np.testing.assert_allclose(ctx.stats_pool(xs, torch.from_numpy(golden["sp_w2"]).to(dev)).cpu().numpy(),
                               golden["sp_y_w2"], atol=2e-6)
    np.testing.assert_allclose(ctx.stats_pool(xs, torch.from_numpy(golden["sp_w3"]).to(dev)).cpu().numpy(),
                               golden["sp_y_w3"], atol=2e-6)


def test_powerset_cuda(ctx, dev, golden):
    logits = torch.from_numpy(golden["ps_logits"])
    cls = logits.argmax(-1).to(torch.uint8).to(dev)
    assert np.array_equal(ctx.powerset_to_multilabel(cls).cpu().numpy(), golden["ps_multilabel"].astype(np.uint8))


def test_segmentation_parity(ctx, dev, oracle_models):
    seg_model, _ = oracle_models
    wav = syn.make_conversation(37.3, seed=11)           # ragged: padded tail chunk
    chunks = P.chunk_waveform(wav)
    buf, off, valid = _device_wave(wav, dev)
    assert len(off) == chunks.shape[0] and valid[-1] < 160000
    with torch.inference_mode():
        ref_sinc = seg_model.sincnet(chunks).transpose(1, 2).numpy()
        ref_logp = seg_model(chunks).numpy()
    sinc = ctx.sincnet_forward(buf, off, valid).cpu().numpy()
    if np.abs(sinc - ref_sinc).max() > 2e-4:
        # every kernel on this path is deterministic: say which implementation deviates and whether it repeats
        _diagnose_sincnet(ctx, buf, off, valid, sinc, ref_sinc)
    np.testing.assert_allclose(sinc, ref_sinc, atol=2e-4, rtol=0)
    cls, logp = ctx.seg_forward(buf, off, valid, return_logp=True)
    np.testing.assert_allclose(logp.cpu().numpy(), ref_logp, atol=2e-4, rtol=0)
    # bit-identical class decisions; frames whose oracle top-2 log-prob margin is below LOW_MARGIN (fp32
    # summation-order noise) are reported separately and are the ONLY place a
    # difference is tolerated
    mism, low = _class_mismatches(cls.cpu().numpy(), ref_logp)
    _report("segmentation_parity 37.3 s", mism, low)
    assert not (mism & ~low).any(), "class decision differs from the oracle on a frame with a clear margin"
    assert mism.sum() == 0 or mism.sum() <= low.sum()
    # a chunk computed inside a batch equals the same chunk computed alone (bitwise: deterministic kernels)
    alone = ctx.seg_forward(buf, off[5:6], valid[5:6])
    assert torch.equal(alone[0], cls[5])
    # split-fp16 tensor-core GEMMs (default) against the fp32 CUDA-core GEMMs: fp32-level agreement
    ctx.set_option("seg_gemm_impl", 0)
    cls0, logp0 = ctx.seg_forward(buf, off, valid, return_logp=True)
    ctx.set_option("seg_gemm_impl", 1)
    np.testing.assert_allclose(logp0.cpu().numpy(), ref_logp, atol=2e-4, rtol=0)
    assert float((logp0 - logp).abs().max()) < 1e-4
    assert float((cls0 != cls).float().mean()) < 1e-3
    # tensor-core SincNet layers (default) against the fp32 CUDA-core kernels
    ctx.set_option("seg_conv_impl", 0)
    sinc0 = ctx.sincnet_forward(buf, off, valid).cpu().numpy()
    cls2, logp2 = ctx.seg_forward(buf, off, valid, return_logp=True)
    ctx.set_option("seg_conv_impl", 1)
    np.testing.assert_allclose(sinc0, ref_sinc, atol=2e-4, rtol=0)
    np.testing.assert_allclose(sinc0, sinc, atol=1e-4, rtol=0)
    assert float((logp2 - logp).abs().max()) < 2e-4
    assert float((cls2 != cls).float().mean()) < 1e-3
    # tensor-core LSTM recurrence (default) against the fp32 CUDA-core cluster kernel
    ctx.set_option("seg_rec_impl", 0)
    cls1, logp1 = ctx.seg_forward(buf, off, valid, return_logp=True)
    ctx.set_option("seg_rec_impl", 1)
    np.testing.assert_allclose(logp1.cpu().numpy(), ref_logp, atol=2e-4, rtol=0)
    assert float((logp1 - logp).abs().max()) < 1e-4
    assert float((cls1 != cls).float().mean()) < 1e-3


def test_segmentation_edge_cases(ctx, dev, oracle_models):
    seg_model, _ = oracle_models
    for T in (100, 160000, 171234):                       # shorter than a chunk / exactly one / one + ragged tail
        wav = syn.make_conversation(T / 16000.0, seed=5)[:, :T]
        chunks = P.chunk_waveform(wav)
        buf, off, valid = _device_wave(wav, dev)
        assert chunks.shape[0] == len(off)
        with torch.inference_mode():
            ref = seg_model(chunks).numpy()
        _, logp = ctx.seg_forward(buf, off, valid, return_logp=True)
        np.testing.assert_allclose(logp.cpu().numpy(), ref, atol=3e-4, rtol=0)
    with pytest.raises(ValueError):
        ctx.seg_forward(buf, np.array([0], dtype=np.int64), np.array([160001], dtype=np.int32))
    assert ctx.seg_forward(buf, np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int32)).shape == (0, 589)


def test_embedding_parity(ctx, dev, oracle_models):
    _, emb_model = oracle_models
    wav = syn.make_conversation(13.7, seed=21)
    chunks = P.chunk_waveform(wav)
    buf, off, valid = _device_wave(wav, dev)
    n = chunks.shape[0]
    with torch.inference_mode():
        ref_fb = emb_model.compute_fbank(chunks)
        ref_frames = emb_model.resnet.forward_frames(ref_fb)
    fb = ctx.emb_fbank(buf, off, valid)
    np.testing.assert_allclose(fb.cpu().numpy(), ref_fb.numpy(), atol=5e-3, rtol=0)
    # trunk: tensor-core path and CUDA-core path against the fp32 oracle, and against each other
    out = {}
    for impl in (0, 1):                                   # CUDA cores, wgmma tensor cores (default)
        ctx.set_option("conv_impl", impl)
        out[impl] = ctx.emb_trunk(ref_fb.to(dev)).cpu().numpy()
        rel = np.abs(out[impl] - ref_frames.numpy()).max() / np.abs(ref_frames.numpy()).max()
        assert rel < 2e-2, f"impl {impl}: trunk relative error {rel}"
    ctx.set_option("conv_impl", 1)
    assert np.abs(out[1] - out[0]).max() <= 2e-2 * np.abs(out[0]).max()
    rng = np.random.default_rng(0)
    masks = (rng.uniform(size=(n, 3, 589)) < 0.5).astype(np.uint8)
    masks[0, 2] = 0                                        # all-zero weights (test_stats_pool.py:111-131 case)
    masks[1, 0] = 1
    with torch.inference_mode():
        ref = emb_model.forward_embedding(ref_frames, weights=torch.from_numpy(masks.astype(np.float32))).numpy()
    emb = ctx.emb_forward(buf, off, valid, torch.from_numpy(masks).to(dev)).cpu().numpy()
    cos = (emb * ref).sum(-1) / (np.linalg.norm(emb, axis=-1) * np.linalg.norm(ref, axis=-1))
    assert (1 - cos).max() <= 1e-3, f"cosine distance to oracle {1 - cos}"
    # pairwise cosine-distance matrix
    a, b = emb.reshape(-1, 256), ref.reshape(-1, 256)
    da = 1 - (a @ a.T) / np.outer(np.linalg.norm(a, axis=1), np.linalg.norm(a, axis=1))
    db = 1 - (b @ b.T) / np.outer(np.linalg.norm(b, axis=1), np.linalg.norm(b, axis=1))
    assert np.abs(da - db).max() <= 1e-3
    # shared fbank frames (default: overlapping hop-aligned full chunks compute their common frames once) against one
    # private run of 998 frames per chunk: the same samples through the same arithmetic -> bit-identical embeddings.
    # The list mixes full chunks, the short last chunk, an unaligned chunk and a repeated one, in two sub-batches.
    off2 = np.concatenate([off, [int(off[0]) + 37, int(off[1])]]).astype(np.int64)
    valid2 = np.concatenate([valid, [160000, 160000]]).astype(np.int32)
    masks2 = torch.from_numpy(np.concatenate([masks, masks[:2]])).to(dev)
    ctx.set_option("emb_max_batch", 4)
    shared = ctx.emb_forward(buf, off2, valid2, masks2).cpu().numpy()
    ctx.set_option("fbank_share", 0)
    private = ctx.emb_forward(buf, off2, valid2, masks2).cpu().numpy()
    ctx.set_option("fbank_share", 1)
    ctx.set_option("emb_max_batch", 264)                   # the library default
    assert np.array_equal(shared, private)
    np.testing.assert_allclose(shared[:n], emb, atol=1e-5, rtol=1e-5)     # other sub-batch split, same segments
    np.testing.assert_allclose(shared[n + 1], shared[1], atol=1e-5, rtol=1e-5)   # a repeated chunk: its own run


def test_post_processing_bit_exact(ctx, dev):
    rng = np.random.default_rng(1)
    for C, p in ((1, 0.5), (7, 0.3), (40, 0.3), (40, 0.02)):
        seg = (rng.uniform(size=(C, 589, 3)) < p).astype(np.float32)
        swf = P.SWF(seg, P.SW(0.0, 10.0, 1.0))
        ref_count = P.speaker_count(swf, FRAMES, (0.0, 0.0))
        sf = P.chunk_start_frames(C, FRAMES)
        F = len(ref_count.data)
        seg_dev = torch.from_numpy(seg.astype(np.uint8)).to(dev)
        count = ctx.speaker_count(seg_dev, sf, F)
        assert np.array_equal(count.cpu().numpy(), ref_count.data[:, 0])
        hard = rng.integers(-1, 5, size=(C, 3)).astype(np.int8)
        hard[hard == -1] = -2
        if hard.max() < 0:
            hard[0, 0] = 0
        for cap in (3, 1):
            cnt = P.SWF(np.minimum(ref_count.data, cap).astype(np.int8), ref_count.sw)
            ref_d = P.reconstruct(swf, hard, cnt)
            K = int(hard.max()) + 1
            Kout = max(K, int(cnt.data.max()), 1)
            d = ctx.reconstruct(seg_dev, hard, sf, F, torch.from_numpy(cnt.data[:, 0].astype(np.uint8)).to(dev), Kout)
            assert np.array_equal(d.cpu().numpy()[:, : ref_d.data.shape[1]], ref_d.data.astype(np.uint8))
            assert not d.cpu().numpy()[:, ref_d.data.shape[1]:].any()
            # device run-length events == host scan of the same matrix (also with a capacity that overflows once)
            dn = d.cpu().numpy()
            act = np.zeros((dn.shape[1], F + 2), dtype=bool)
            act[:, 1:-1] = dn.T > 0
            for ecap in (4096, 2):
                on, off = ctx.frame_transitions(d, cap=ecap)
                assert np.array_equal(on, np.flatnonzero(act[:, 1:] & ~act[:, :-1]))
                assert np.array_equal(off, np.flatnonzero(act[:, :-1] & ~act[:, 1:]))
        clean, active = ctx.clean_frames(seg_dev)
        single = seg.sum(2, keepdims=True) == 1
        assert np.array_equal(clean.cpu().numpy(), (seg * single).sum(1).astype(np.int32))
        assert np.array_equal(active.cpu().numpy() > 0, seg.sum(1) > 0)


def _same_partition(a, b):
    m = {}
    for x, y in zip(a, b):
        if m.setdefault(x, y) != y:
            return False
    return len(set(m.values())) == len(m)


def test_linkage_parity_with_scipy(ctx, dev):
    from scipy.cluster.hierarchy import fcluster, linkage

    from pyannote_audio_b200 import ops

    rng = np.random.default_rng(3)
    # issue-1525 vector of /root/reference/tests/test_clustering.py:6-29 (2 embeddings)
    e2 = np.array([[1.0, 1.0, 1.0, 1.0], [1.0, 2.0, 1.0, 2.0]])
    Z = ctx.linkage_centroid(torch.from_numpy(e2).to(dev), normalize=True).cpu().numpy()
    ref = linkage(e2 / np.linalg.norm(e2, axis=1, keepdims=True), "centroid", "euclidean")
    np.testing.assert_allclose(Z, ref, rtol=1e-12)
    for n, dim in ((3, 4), (50, 16), (300, 256), (1000, 256)):
        centers = rng.standard_normal((5, dim))
        X = centers[rng.integers(0, 5, n)] + 0.6 * rng.standard_normal((n, dim))
        Xn = X / np.linalg.norm(X, axis=1, keepdims=True)
        ref = linkage(Xn, "centroid", "euclidean")
        Z = ctx.linkage_centroid(torch.from_numpy(X).to(dev), normalize=True).cpu().numpy()
        np.testing.assert_allclose(np.sort(Z[:, 2]), np.sort(ref[:, 2]), rtol=1e-9, atol=1e-12)
        for t in (0.3, 0.6, 0.9, 1.2):
            assert _same_partition(fcluster(ref, t, "distance"), ops.fcluster_distance(Z, t))


def test_vbx_cdist_assign_parity(ctx, dev, golden):
    from scipy.optimize import linear_sum_assignment
    from scipy.spatial.distance import cdist
    from scipy.special import softmax

    fea, phi, ahc = golden["vbx_fea"], golden["vbx_phi"], golden["vbx_ahc"]
    q0 = np.zeros((len(ahc), ahc.max() + 1))
    q0[range(len(ahc)), ahc] = 1.0
    q0 = softmax(q0 * 7.0, axis=1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    gamma, pi, iters = ctx.vbx(t(fea), t(phi), t(q0), 0.07, 0.8, max_iters=20)
    np.testing.assert_allclose(gamma.cpu().numpy(), golden["vbx_gamma"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(pi.cpu().numpy(), golden["vbx_pi"], rtol=1e-8, atol=1e-10)
    assert 1 <= iters <= 20
    rng = np.random.default_rng(4)
    a, b = rng.standard_normal((37, 256)), rng.standard_normal((6, 256))
    np.testing.assert_allclose(ctx.cdist_cosine(t(a), t(b)).cpu().numpy(), cdist(a, b, "cosine"), rtol=1e-10, atol=1e-12)
    for K in (1, 2, 3, 6):
        soft = rng.standard_normal((50, 3, K))
        hard = ctx.assign(t(soft), constrained=True).cpu().numpy()
        for c in range(50):
            rows, cols = linear_sum_assignment(soft[c], maximize=True)
            ref = -2 * np.ones(3, dtype=np.int8)
            ref[rows] = cols
            assert np.array_equal(hard[c], ref)
        assert np.array_equal(ctx.assign(t(soft), constrained=False).cpu().numpy(), soft.argmax(-1))


@pytest.fixture(scope="module")
def pipeline(dev):
    from pyannote_audio_b200.models import PyanNet, WeSpeakerResNet34
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    seg, emb = PyanNet(), WeSpeakerResNet34()
    seg.load_state_dict(syn.make_segmentation_state_dict(0), strict=False)
    emb.load_state_dict(syn.make_embedding_state_dict(1), strict=False)
    return SpeakerDiarization(segmentation=seg, embedding=emb, plda=syn.make_plda(2), device=dev)


def _rows(x):
    return [tuple(int(v) for v in r) for r in x]


LOW_ASSIGN_MARGIN = 1e-3


def _low_margin_assignments(hard, ref):
    """Chunks whose speaker -> cluster assignment differs from the INDEPENDENT oracle run although the CUDA choice is
    within LOW_ASSIGN_MARGIN of the optimum under the oracle's own scores (2 - cosine distance to the centroids): a
    near-tie of the reference's constrained argmax that fp16-level embedding noise (relative 1e-3) decides either
    way -- the clustering counterpart of the low-margin frames of the segmentation.  Returns (differing chunks,
    those of them that are low-margin)."""
    soft = ref.soft_clusters
    differ = np.flatnonzero((np.asarray(hard) != ref.hard_clusters).any(axis=1))
    low = []
    if soft is None or np.asarray(hard).shape != ref.hard_clusters.shape:
        return differ, np.array(low, dtype=int)
    for c in differ:
        def objective(h):
            return sum(soft[c, s, k] for s, k in enumerate(h) if 0 <= k < soft.shape[2])
        if objective(ref.hard_clusters[c]) - objective(np.asarray(hard)[c]) < LOW_ASSIGN_MARGIN:
            low.append(c)
    return differ, np.array(low, dtype=int)


def _compare_with_oracle(art, out, ref, independent, own_embeddings=False):
    """Integer outputs of the CUDA pipeline against an oracle run (bit-exact)."""
    assert np.array_equal(art["count"].cpu().numpy(), ref.count.data[:, 0])
    if own_embeddings:
        # the oracle clusters ITS OWN fp32 embeddings: identical decisions except reported near-ties
        differ, low = _low_margin_assignments(art["hard_clusters"], ref)
        print(f"[parity] independent run: {len(differ)} chunk(s) with a different assignment, {len(low)} of them "
              f"within {LOW_ASSIGN_MARGIN} of the oracle's optimum")
        assert len(differ) == len(low), "cluster assignment differs from the independent oracle with a clear margin"
        if len(differ):
            return False                                  # downstream stages are checked against the re-fed oracle
    assert np.array_equal(art["hard_clusters"], ref.hard_clusters), ("independent" if independent else "re-fed")
    assert np.array_equal(art["discrete"][:, : ref.discrete.data.shape[1]], ref.discrete.data.astype(np.uint8))
    assert not art["discrete"][:, ref.discrete.data.shape[1]:].any()
    assert np.array_equal(art["exclusive"][:, : ref.exclusive.data.shape[1]], ref.exclusive.data.astype(np.uint8))
    assert _rows(art["segments"]) == _rows(ref.segments)                          # integer frame boundaries
    assert _rows(art["exclusive_segments"]) == _rows(ref.exclusive_segments)
    got = [(s.start, s.end, lab) for s, _, lab in out.speaker_diarization.itertracks(yield_label=True)]
    assert got == ref.times
    gotx = [(s.start, s.end, lab) for s, _, lab in out.exclusive_speaker_diarization.itertracks(yield_label=True)]
    assert gotx == ref.exclusive_times
    return True


def _e2e_case(pipeline, oracle_models, wav, name, exclude_overlap=False, min_duration_off=0.0, emb_oracle=True):
    """Runs one file through apply_batch and through the oracle.  The comparison is with the fully INDEPENDENT
    oracle run (its own segmentation, its own fp32 embeddings); only if a low-margin frame flipped (reported) the
    integer stages are compared with the oracle re-fed with the CUDA segmentation instead."""
    seg_model, emb_model = oracle_models
    plda = P.PLDA(**syn.make_plda(2))
    file = {"waveform": wav, "sample_rate": 16000, "uri": name}
    pipeline.embedding_exclude_overlap = exclude_overlap
    pipeline.min_duration_off = min_duration_off
    try:
        seen = []
        (_, (out, art)), = list(pipeline.apply_batch(
            [file], hook=lambda step, artifact, **k: seen.append((step, artifact is None)), return_artifacts=True))
    finally:
        pipeline.embedding_exclude_overlap = False
        pipeline.min_duration_off = 0.0
    names = [n for n, progress in seen if not progress]
    assert names == ["segmentation", "speaker_counting", "embeddings", "discrete_diarization"]
    assert ("segmentation", True) in seen and ("embeddings", True) in seen            # progress calls fire too
    ref_seg, ref_logp = P.slide(seg_model, wav, return_logp=True)
    seg = art["segmentations"].cpu().numpy().astype(np.float32)
    assert seg.shape == ref_seg.data.shape
    cls = art["classes"].cpu().numpy()
    mism, low = _class_mismatches(cls, ref_logp)
    _report(name, mism, low)
    assert not (mism & ~low).any()
    identical = not mism.any()
    assert identical == bool((seg == ref_seg.data).all())
    emb = art["embeddings"].cpu().numpy()
    if emb_oracle:
        ref = P.apply(seg_model, emb_model, plda, wav, segmentations=ref_seg if identical else P.SWF(seg, ref_seg.sw),
                      exclude_overlap=exclude_overlap, min_duration_off=min_duration_off)
        cos = (emb * ref.embeddings).sum(-1) / (np.linalg.norm(emb, axis=-1) * np.linalg.norm(ref.embeddings, axis=-1))
        assert (1 - cos).max() <= 1e-3, f"embedding cosine distance {np.nanmax(1 - cos)}"
        same = _compare_with_oracle(art, out, ref, independent=identical, own_embeddings=True)
        a, b = out.speaker_embeddings, ref.speaker_embeddings
        assert a.shape == b.shape or not same
        real = np.linalg.norm(b, axis=-1) > 0                # rows padded for labels without a centroid are all-zero
        if same:
            assert np.array_equal(real, np.linalg.norm(a, axis=-1) > 0)
        if same and real.any():
            ccos = (a * b).sum(-1)[real] / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))[real]
            assert (1 - ccos).max() <= 1e-3
    # and with the CUDA embeddings fed to the oracle's clustering: everything downstream is exact arithmetic
    ref2 = P.apply(seg_model, emb_model, plda, wav, segmentations=P.SWF(seg, ref_seg.sw), embeddings=emb,
                   exclude_overlap=exclude_overlap, min_duration_off=min_duration_off)
    _compare_with_oracle(art, out, ref2, independent=False)
    np.testing.assert_allclose(out.speaker_embeddings, ref2.speaker_embeddings, rtol=1e-6, atol=1e-8)
    return out, art


def test_pipeline_end_to_end_vs_oracle(pipeline, oracle_models):
    _e2e_case(pipeline, oracle_models, syn.make_conversation(75.0, seed=1234), "e2e-75s")


def test_pipeline_exclude_overlap_and_min_duration_off(pipeline, oracle_models):
    """embedding_exclude_overlap=True (the setting published pipelines ship with, speaker_diarization.py:375-391)
    and segmentation.min_duration_off > 0 (Binarize -> Annotation.support, utils/signal.py:307-310)."""
    wav = syn.make_conversation(48.0, seed=77)
    _e2e_case(pipeline, oracle_models, wav, "exclude-overlap", exclude_overlap=True)
    out, art = _e2e_case(pipeline, oracle_models, wav, "min-duration-off", min_duration_off=0.5)
    assert len(out.speaker_diarization) <= len(art["segments"])
    # the overlap-free masks differ from the plain ones on this file (otherwise the first case proves nothing)
    seg = art["segmentations"]
    assert bool((seg.sum(dim=2) > 1).any())


def test_bench_workload_file_vs_oracle(pipeline, oracle_models):
    """BASELINE.json configs[4]: one 10-minute file of the bench workload (bench.py seed 1000) through apply_batch;
    591 chunks of segmentation against the oracle, then clustering + reconstruction + segments exact with the CUDA
    embeddings fed to the oracle (its ResNet would need ~15 min of CPU for 1773 embeddings)."""
    wav = syn.make_conversation(600.0, seed=1000)
    _, art = _e2e_case(pipeline, oracle_models, wav, "bench-file-600s", emb_oracle=False)
    assert art["segmentations"].shape[0] == 591
    # a sample of the embeddings against the fp32 oracle (cosine <= 1e-3)
    _, emb_model = oracle_models
    seg = art["segmentations"].cpu().numpy().astype(np.float32)
    pick = [0, 137, 590]
    sub = P.SWF(seg, P.SW(0.0, 10.0, 1.0))
    masks = P.embedding_masks(sub)
    with torch.inference_mode():
        for c in pick:
            chunk = P.crop_pad(wav, float(c), float(c) + 10.0)[None]
            ref = emb_model.forward_embedding(emb_model.forward_frames(chunk), weights=torch.from_numpy(masks[c:c + 1]))
            got = art["embeddings"][c].cpu().numpy()
            r = ref[0].numpy()
            ok = np.linalg.norm(r, axis=-1) > 0
            cos = (got * r).sum(-1)[ok] / (np.linalg.norm(got, axis=-1) * np.linalg.norm(r, axis=-1))[ok]
            assert (1 - cos).max() <= 1e-3


def test_pipeline_edge_cases(pipeline):
    silence = {"waveform": torch.zeros(1, 16000 * 12), "sample_rate": 16000, "uri": "silence"}
    short = {"waveform": syn.make_conversation(3.0, seed=2), "sample_rate": 16000, "uri": "short"}
    outs = pipeline([silence, short])
    assert len(outs) == 2
    for o in outs:
        assert hasattr(o, "speaker_diarization") and isinstance(o.serialize(), dict)
    one = pipeline(short, num_speakers=1)
    assert len(one.speaker_diarization.labels()) <= 1


def test_cfg2_sincnet_frontend_1024_chunks(ctx, dev, oracle_models):
    """BASELINE.json configs[1]: SincNet + Conv1d front-end on a 1024-chunk batch against the oracle (full size)."""
    seg_model, _ = oracle_models
    wav = syn.make_conversation(10.0 + 1023.0, seed=2024)
    buf, off, valid = _device_wave(wav, dev)
    assert len(off) == 1024
    got = ctx.sincnet_forward(buf, off, valid)
    assert got.shape == (1024, 589, 60)
    chunks = P.chunk_waveform(wav)
    worst = 0.0
    with torch.inference_mode():
        for c0 in range(0, 1024, 64):
            ref = seg_model.sincnet(chunks[c0:c0 + 64]).transpose(1, 2)
            worst = max(worst, float((got[c0:c0 + 64].cpu() - ref).abs().max()))
    print(f"[parity] cfg2: 1024 chunks, max |sincnet - oracle| = {worst:.2e}")
    assert worst <= 2e-4
    assert torch.equal(got[100:108], ctx.sincnet_forward(buf, off[100:108], valid[100:108]))     # batch invariance


def test_cfg3_cfg4_one_hour_file_vs_oracle(pipeline, ctx, dev, oracle_models):
    """BASELINE.json configs[2] + configs[3] at full size.  One synthetic hour (3591 chunks, 10 773 embedding slots):
    * PyanNet sliding window: class ids of all 3591 x 589 frames against the oracle (bit-identical outside the
      reported low-margin set), speaker count on the 213 334-frame grid;
    * embeddings -> clean-frame filter -> centroid linkage at n > 4096 (the global-memory state path) -> fcluster ->
      PLDA -> VBx -> cosine cdist -> constrained assignment -> reconstruction -> segments, all bit-exact against the
      oracle (scipy linkage / fcluster / cdist / linear_sum_assignment, the reference's VBx) fed with the same
      embeddings; a sample of the embeddings and the full 10 773^2 cosine-distance matrix against the oracle."""
    from scipy.cluster.hierarchy import fcluster, linkage
    from scipy.spatial.distance import cdist

    from pyannote_audio_b200 import ops

    _, emb_model = oracle_models
    wav = syn.make_conversation(3600.0, seed=99)
    out, art = _e2e_case(pipeline, oracle_models, wav, "cfg3-one-hour", emb_oracle=False)
    assert art["segmentations"].shape == (3591, 589, 3) and art["count"].shape == (213334,)
    assert int(art["count"].max()) <= 2                                                          # powerset: <= 2
    emb = art["embeddings"]
    assert emb.shape == (3591, 3, 256) and bool(torch.isfinite(emb).all())
    # cfg4: cosine-distance matrix of the ~10k embeddings against scipy
    x = emb.reshape(-1, 256).double()
    d = ctx.cdist_cosine(x, x).cpu().numpy()
    xn = x.cpu().numpy()
    assert d.shape == (10773, 10773)
    for r0 in range(0, 10773, 2048):
        np.testing.assert_allclose(d[r0:r0 + 2048], cdist(xn[r0:r0 + 2048], xn, "cosine"), rtol=0, atol=1e-12)
    del d
    # cfg4: a sample of the embeddings against the fp32 oracle network (cosine <= 1e-3)
    seg = art["segmentations"].cpu().numpy().astype(np.float32)
    masks = P.embedding_masks(P.SWF(seg, P.SW(0.0, 10.0, 1.0)))
    pick = list(range(0, 3591, 449))
    with torch.inference_mode():
        chunks = torch.stack([P.crop_pad(wav, float(c), float(c) + 10.0) for c in pick])
        ref = emb_model.forward_embedding(emb_model.forward_frames(chunks), weights=torch.from_numpy(masks[pick])).numpy()
    got = emb[pick].cpu().numpy()
    ok = np.linalg.norm(ref, axis=-1) > 0
    cos = (got * ref).sum(-1)[ok] / (np.linalg.norm(got, axis=-1) * np.linalg.norm(ref, axis=-1))[ok]
    print(f"[parity] cfg4: {int(ok.sum())} sampled embeddings, max cosine distance to the fp32 oracle {float((1 - cos).max()):.2e}")
    assert (1 - cos).max() <= 1e-3
    # cfg4: the linkage itself at n > 4096 against scipy (heights + partitions at several thresholds)
    train, _, _ = P.filter_embeddings(emb.cpu().numpy(), seg)
    n = train.shape[0]
    assert n > 4096, f"only {n} training embeddings: the large-n linkage path is not exercised"
    tn = train.astype(np.float64)
    tn = tn / np.linalg.norm(tn, axis=1, keepdims=True)
    Zref = linkage(tn, "centroid", "euclidean")
    Z = ctx.linkage_centroid(torch.from_numpy(train.astype(np.float64)).to(dev), normalize=True).cpu().numpy()
    np.testing.assert_allclose(np.sort(Z[:, 2]), np.sort(Zref[:, 2]), rtol=1e-9, atol=1e-12)
    for t in (0.3, 0.6, 0.9):
        assert _same_partition(fcluster(Zref, t, "distance"), ops.fcluster_distance(Z, t))
    print(f"[parity] cfg4: linkage n={n} heights and partitions identical to scipy")
    # size-independent properties on top: idempotence and batch invariance at this size
    buf, off, valid = _device_wave(wav, dev)
    cls = art["classes"]
    assert torch.equal(cls[1000:1010], ctx.seg_forward(buf, off[1000:1010], valid[1000:1010]))
    m = art["segmentations"].permute(0, 2, 1).contiguous()
    assert torch.equal(ctx.emb_forward(buf, off[2000:2003], valid[2000:2003], m[2000:2003]), emb[2000:2003])
