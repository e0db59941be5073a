"""Oracle (TEST INFRASTRUCTURE): CPU restatement of the community-1 pipeline plumbing.

Follows (paths relative to /root/reference/src/pyannote/audio):

* ``slide``                 core/inference.py:217-373 (skip_aggregation branch :336-347)
* ``aggregate`` / ``trim``  core/inference.py:498-620 / :622-667
* ``speaker_count``         pipelines/utils/diarization.py:150-185
* ``to_diarization``        pipelines/utils/diarization.py:221-268
* ``binarize_to_segments``  utils/signal.py:254-318 (Binarize.__call__, onset=offset=0.5)
* ``get_embeddings``        pipelines/speaker_diarization.py:332-478 (+ core/io.py:384-414 crop/pad)
* ``reconstruct``           pipelines/speaker_diarization.py:480-528
* ``filter_embeddings`` / ``constrained_argmax`` / ``vbx_clustering`` / ``ahc_cluster``
                            pipelines/clustering.py:77-140, 572-669, 330-480
* ``VBx`` / ``cluster_vbx`` / ``vbx_setup`` / PLDA   utils/vbx.py:27-218, core/plda.py:33-63
* ``apply``                 pipelines/speaker_diarization.py:530-784

Pinning: aggregate / trim / speaker_count / to_diarization / reconstruct / binarize / filter_embeddings /
constrained_argmax / vbx_clustering / ahc_call are checked against outputs of the reference's own files executed by
path (tests/golden/make_golden_pipeline.py -> reference_pipeline_vectors.npz, tests/test_oracle_pipeline_golden.py);
get_embeddings and apply against the reference's SpeakerDiarization.get_embeddings / apply run on a synthetic
conversation (tests/golden/make_golden_apply.py -> reference_apply_vectors.npz, tests/test_oracle_apply_golden.py).

pyannote.core 6.0.1 (SlidingWindow.closest_frame / crop / range_to_segment, Segment.middle) is NOT
in the tree and not installed: restated from its published behaviour -- parity unpinned for the
frame arithmetic (cross-checked against the shape facts in tutorials/applying_a_model.ipynb).
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F
from scipy.cluster.hierarchy import fcluster, linkage
from scipy.linalg import eigh
from scipy.optimize import linear_sum_assignment
from scipy.spatial.distance import cdist
from scipy.special import logsumexp, softmax

from . import nets

# ----------------------------------------------------------------------------------------
# pyannote.core restatement (minimal)
# ----------------------------------------------------------------------------------------


@dataclass(frozen=True)
class SW:
    """SlidingWindow(start, duration, step)."""

    start: float = 0.0
    duration: float = 0.03
    step: float = 0.01

    def closest_frame(self, t: float) -> int:
        return int(np.rint((t - self.start - 0.5 * self.duration) / self.step))

    def segment(self, i: int):
        s = self.start + i * self.step
        return (s, s + self.duration)

    def middle(self, i: int) -> float:
        s, e = self.segment(i)
        return 0.5 * (s + e)

    def range_to_segment(self, i0: int, n: int):
        start = self.start + (i0 - 0.5) * self.step + 0.5 * self.duration
        end = start + n * self.step
        if i0 == 0:
            start = self.start
        return (start, end)

    def crop_loose(self, focus):
        i = int(np.ceil((focus[0] - self.duration - self.start) / self.step))
        j = int(np.floor((focus[1] - self.start) / self.step))
        return (i, j + 1)


@dataclass
class SWF:
    """SlidingWindowFeature(data, sliding_window)."""

    data: np.ndarray
    sw: SW

    def extent(self):
        return self.sw.range_to_segment(0, len(self.data))

    def crop_loose(self, focus):
        i, j = self.sw.crop_loose(focus)
        n = self.data.shape[0]
        if j < 0 or i >= n:
            return SWF(self.data[:0], self.sw)
        i0, j0 = max(i, 0), min(j, n)
        return SWF(self.data[i0:j0], SW(self.sw.segment(i0)[0], self.sw.duration, self.sw.step))


# ----------------------------------------------------------------------------------------
# Inference.slide / aggregate / trim
# ----------------------------------------------------------------------------------------

SAMPLE_RATE = 16000
DURATION = 10.0
STEP = 1.0


def chunk_waveform(waveform: torch.Tensor, window_size=160000, step_size=16000):
    """waveform (1,T) -> (C,1,window) incl. zero-padded tail chunk (inference.py:261-278)."""
    _, num_samples = waveform.shape
    chunks = []
    if num_samples >= window_size:
        full = waveform.unfold(1, window_size, step_size).permute(1, 0, 2)
        num_chunks = full.shape[0]
        chunks.append(full)
    else:
        num_chunks = 0
    has_last = (num_samples < window_size) or (num_samples - window_size) % step_size > 0
    if has_last:
        last = waveform[:, num_chunks * step_size:]
        last = F.pad(last, (0, window_size - last.shape[1]))
        chunks.append(last[None])
    return torch.cat(chunks, dim=0)


def slide(model: "nets.PyanNet", waveform: torch.Tensor, batch_size=32, return_logp=False):
    """Inference.slide with skip_aggregation=True -> SWF((C,589,3), SW(0,10,1))."""
    mapping = nets.powerset_mapping(3, 2)
    chunks = chunk_waveform(waveform)
    outs, logps = [], []
    with torch.inference_mode():
        for c in range(0, chunks.shape[0], batch_size):
            logp = model(chunks[c:c + batch_size])
            logps.append(logp)
            outs.append(nets.powerset_to_multilabel(logp, mapping).numpy())
    seg = SWF(np.vstack(outs), SW(0.0, DURATION, STEP))
    if return_logp:
        return seg, torch.cat(logps).numpy()
    return seg


def trim(scores: SWF, warm_up=(0.1, 0.1)) -> SWF:
    _, num_frames, _ = scores.data.shape
    left = round(num_frames * warm_up[0])
    right = round(num_frames * warm_up[1])
    new = scores.data[:, left:num_frames - right]
    sw = SW(scores.sw.start + warm_up[0] * scores.sw.duration, (1 - warm_up[0] - warm_up[1]) * scores.sw.duration,
            scores.sw.step)
    return SWF(new, sw)


def aggregate(scores: SWF, frames: SW, warm_up=(0.0, 0.0), epsilon=1e-12, hamming=False,
              missing=np.nan, skip_average=False) -> SWF:
    num_chunks, nfpc, num_classes = scores.data.shape
    chunks = scores.sw
    frames = SW(chunks.start, frames.duration, frames.step)
    hamming_window = np.hamming(nfpc).reshape(-1, 1) if hamming else np.ones((nfpc, 1))
    warm_up_window = np.ones((nfpc, 1))
    wl = round(warm_up[0] / chunks.duration * nfpc)
    warm_up_window[:wl] = epsilon
    wr = round(warm_up[1] / chunks.duration * nfpc)
    warm_up_window[nfpc - wr:] = epsilon
    num_frames = frames.closest_frame(
        chunks.start + chunks.duration + (num_chunks - 1) * chunks.step + 0.5 * frames.duration) + 1
    agg = np.zeros((num_frames, num_classes), dtype=np.float32)
    cnt = np.zeros((num_frames, num_classes), dtype=np.float32)
    msk = np.zeros((num_frames, num_classes), dtype=np.float32)
    for c in range(num_chunks):
        score = scores.data[c].copy()
        chunk_start = chunks.start + c * chunks.step
        mask = 1 - np.isnan(score)
        np.nan_to_num(score, copy=False, nan=0.0)
        sf = frames.closest_frame(chunk_start + 0.5 * frames.duration)
        agg[sf:sf + nfpc] += score * mask * hamming_window * warm_up_window
        cnt[sf:sf + nfpc] += mask * hamming_window * warm_up_window
        msk[sf:sf + nfpc] = np.maximum(msk[sf:sf + nfpc], mask)
    average = agg if skip_average else agg / np.maximum(cnt, epsilon)
    average[msk == 0.0] = missing
    return SWF(average, frames)


def chunk_start_frames(num_chunks: int, frames: SW, chunks: SW = SW(0.0, DURATION, STEP)):
    """Integer frame offset of every chunk on the global grid (inference.py:596)."""
    fr = SW(chunks.start, frames.duration, frames.step)
    return np.array([fr.closest_frame(chunks.start + c * chunks.step + 0.5 * fr.duration)
                     for c in range(num_chunks)], dtype=np.int64)


def speaker_count(binarized: SWF, frames: SW, warm_up=(0.0, 0.0)) -> SWF:
    trimmed = trim(binarized, warm_up)
    summed = SWF(np.sum(trimmed.data, axis=-1, keepdims=True), trimmed.sw)
    count = aggregate(summed, frames, hamming=False, missing=0.0, skip_average=False)
    count.data = np.rint(count.data).astype(np.uint8)
    return count


def to_diarization(segmentations: SWF, count: SWF, stable=True) -> SWF:
    activations = aggregate(segmentations, count.sw, hamming=False, missing=0.0, skip_average=True)
    _, num_speakers = activations.data.shape
    max_spf = int(np.max(count.data))
    if num_speakers < max_spf:
        activations.data = np.pad(activations.data, ((0, 0), (0, max_spf - num_speakers)))
    e1, e2 = activations.extent(), count.extent()
    extent = (max(e1[0], e2[0]), min(e1[1], e2[1]))
    activations = activations.crop_loose(extent)
    count = count.crop_loose(extent)
    # reference: np.argsort(-activations) (default introsort, ties unstable in principle);
    # the oracle pins ties as "descending value, then ascending cluster index".
    sorted_speakers = np.argsort(-activations.data, axis=-1, kind="stable" if stable else None)
    binary = np.zeros_like(activations.data)
    for t in range(min(len(count.data), len(binary))):
        c = int(count.data[t, 0])
        for i in range(c):
            binary[t, sorted_speakers[t, i]] = 1.0
    return SWF(binary, activations.sw)


def binarize_to_segments(discrete: SWF):
    """Binarize(onset=offset=0.5) -> list of (start_frame, end_frame, label) + float times.

    A region turned on at frame i and off at frame j is [middle(i), middle(j)]; a region still active at
    the last frame n-1 ends at middle(n-1) (signal.py:276-305).
    Returns rows sorted like Annotation.itertracks(): by (start, end), then label.
    """
    data = discrete.data
    n, K = data.shape
    rows = []
    for k in range(K):
        col = data[:, k]
        start = 0
        active = col[0] > 0.5
        t = 0
        for t in range(1, n):
            y = col[t]
            if active:
                if y < 0.5:
                    rows.append((start, t, k))
                    start = t
                    active = False
            else:
                if y > 0.5:
                    start = t
                    active = True
        if active and t > start:      # Segment(start, start) is empty: Annotation.__setitem__ ignores it
            rows.append((start, t, k))
    rows.sort(key=lambda r: (r[0], r[1], r[2]))
    times = [(discrete.sw.middle(a), discrete.sw.middle(b), k) for a, b, k in rows]
    return rows, times


def binarize_scores(scores: SWF, onset=0.5, offset=0.5, min_duration_on=0.0, min_duration_off=0.0):
    """Binarize.__call__ (utils/signal.py:254-318) restated literally for float scores (hysteresis thresholds),
    pad_onset = pad_offset = 0.  Returns [(start_s, end_s, class_index)] in itertracks order."""
    n, K = scores.data.shape
    ts = [scores.sw.middle(i) for i in range(n)]
    out = []
    for k in range(K):
        col = scores.data[:, k]
        start = ts[0]
        is_active = col[0] > onset
        t = ts[0]
        for t, y in zip(ts[1:], col[1:]):
            if is_active:
                if y < offset:
                    if t - start > 1e-6:
                        out.append((start, t, k))
                    start = t
                    is_active = False
            else:
                if y > onset:
                    start = t
                    is_active = True
        if is_active and t - start > 1e-6:
            out.append((start, t, k))
    out.sort(key=lambda r: (r[0], r[1], r[2]))
    if min_duration_off > 0.0:
        out = support(out, min_duration_off)
    if min_duration_on > 0:
        out = [r for r in out if r[1] - r[0] >= min_duration_on]
    return out


def vad_scores(seg_model, waveform: torch.Tensor, batch_size=32) -> SWF:
    """VoiceActivityDetection's `self._segmentation(file)` (pipelines/voice_activity_detection.py:111-115, 196-198):
    Inference with pre_aggregation_hook = max over speakers, Hamming aggregation, padded tail cropped
    (core/inference.py:349-369)."""
    seg = slide(seg_model, waveform, batch_size)
    speech = SWF(np.max(seg.data, axis=-1, keepdims=True), seg.sw)
    frames = SW(*nets.sincnet_receptive_field())
    agg = aggregate(speech, frames, warm_up=(0.0, 0.0), hamming=True, missing=0.0)
    num_samples = waveform.shape[1]
    if num_samples < 160000 or (num_samples - 160000) % 16000 > 0:
        agg = agg.crop_loose((0.0, num_samples / SAMPLE_RATE))
    return agg


def support(times, collar=0.0):
    """pyannote.core Annotation.support(collar) (called by Binarize when min_duration_off > 0, signal.py:307-310),
    restated from the published behaviour (parity unpinned, like the rest of pyannote.core): per label in sorted
    order, walk the label's segments by (start, end) and merge the next one into the current one when they touch /
    overlap (gap <= 1e-6, an "empty" Segment) or the gap is strictly shorter than ``collar``.
    ``times`` = [(start_s, end_s, label)]; returns the merged list in itertracks order (start, end, label)."""
    out = []
    for lab in sorted({k for _, _, k in times}):
        segs = sorted((a, b) for a, b, k in times if k == lab)
        cs, ce = segs[0]
        for a, b in segs[1:]:
            gap = a - ce
            if gap <= 1e-6 or gap < collar:
                ce = max(ce, b)
            else:
                out.append((cs, ce, lab))
                cs, ce = a, b
        out.append((cs, ce, lab))
    out.sort(key=lambda r: (r[0], r[1], r[2]))
    return out


# ----------------------------------------------------------------------------------------
# embeddings
# ----------------------------------------------------------------------------------------


def crop_pad(waveform: torch.Tensor, start: float, end: float, sr=SAMPLE_RATE):
    """Audio.crop(mode="pad"), in-memory branch (core/io.py:384-414)."""
    _, num_samples = waveform.shape
    s = round(start * sr)
    pad_start = max(0, -s)
    s = max(s, 0)
    e = round(end * sr)
    pad_end = max(e, num_samples) - num_samples
    e = min(e, num_samples)
    return F.pad(waveform[:, s:e], (pad_start, pad_end))


def embedding_masks(binary: SWF, exclude_overlap=False, min_num_samples=400):
    """(C,3,589) float32 masks actually fed to StatsPool (speaker_diarization.py:375-423)."""
    data = binary.data
    num_chunks, num_frames, _ = data.shape
    if exclude_overlap:
        num_samples = binary.sw.duration * SAMPLE_RATE
        min_num_frames = math.ceil(num_frames * min_num_samples / num_samples)
        clean = data * (1.0 * (np.sum(data, axis=2, keepdims=True) < 2))
    else:
        min_num_frames = -1
        clean = data
    masks = np.nan_to_num(data, nan=0.0).astype(np.float32)
    clean = np.nan_to_num(clean, nan=0.0).astype(np.float32)
    use_clean = clean.sum(axis=1) > min_num_frames          # (C,3)
    out = np.where(use_clean[:, None, :], clean, masks)      # (C,589,3)
    return np.ascontiguousarray(out.transpose(0, 2, 1))


def get_embeddings(model: "nets.WeSpeakerResNet34", waveform: torch.Tensor, binary: SWF,
                   exclude_overlap=False, batch_size=8, share_trunk=True, max_chunks=None):
    """(C,3,256) float32.  share_trunk=False reproduces the reference's 3 forwards per chunk."""
    masks = embedding_masks(binary, exclude_overlap)
    C = masks.shape[0] if max_chunks is None else min(max_chunks, masks.shape[0])
    out = np.zeros((C, 3, 256), dtype=np.float32)
    with torch.inference_mode():
        if share_trunk:
            for c0 in range(0, C, batch_size):
                cs = range(c0, min(C, c0 + batch_size))
                wav = torch.stack([crop_pad(waveform, binary.sw.start + c * binary.sw.step,
                                            binary.sw.start + c * binary.sw.step + binary.sw.duration) for c in cs])
                frames = model.forward_frames(wav)
                emb = model.forward_embedding(frames, weights=torch.from_numpy(masks[c0:c0 + len(cs)]))
                out[c0:c0 + len(cs)] = emb.numpy()
        else:
            items = [(c, s) for c in range(C) for s in range(3)]
            for i0 in range(0, len(items), batch_size):
                sel = items[i0:i0 + batch_size]
                wav = torch.stack([crop_pad(waveform, binary.sw.start + c * binary.sw.step,
                                            binary.sw.start + c * binary.sw.step + binary.sw.duration) for c, _ in sel])
                w = torch.from_numpy(np.stack([masks[c, s] for c, s in sel]))
                emb = model(wav, weights=w).numpy()
                for (c, s), e in zip(sel, emb):
                    out[c, s] = e
    return out


# ----------------------------------------------------------------------------------------
# PLDA / VBx
# ----------------------------------------------------------------------------------------


def l2_norm(x):
    if x.ndim == 1:
        return x / np.linalg.norm(x)
    return x / np.linalg.norm(x, axis=1, ord=2)[:, np.newaxis]


class PLDA:
    """core/plda.py:33-63 over utils/vbx.py:181-218, fed with in-memory arrays instead of npz paths."""

    def __init__(self, mean1, mean2, lda, mu, tr, psi, lda_dimension=128):
        W = np.linalg.inv(tr.T.dot(tr))
        B = np.linalg.inv((tr.T / psi).dot(tr))
        acvar, wccn = eigh(B, W)
        self._psi = acvar[::-1]
        self._tr = wccn.T[::-1]
        self.mean1, self.mean2, self.lda, self.mu = mean1, mean2, lda, mu
        self.lda_dimension = lda_dimension

    @property
    def phi(self):
        return self._psi[: self.lda_dimension]

    def xvec_tf(self, x):
        lda = self.lda
        return np.sqrt(lda.shape[1]) * l2_norm(
            lda.T.dot(np.sqrt(lda.shape[0]) * l2_norm(x - self.mean1).T).T - self.mean2)

    def plda_tf(self, x0):
        return (x0 - self.mu).dot(self._tr.T)[:, : self.lda_dimension]

    def __call__(self, embeddings):
        return self.plda_tf(self.xvec_tf(embeddings))


def VBx(X, Phi, Fa=1.0, Fb=1.0, pi=10, gamma=None, maxIters=10, epsilon=1e-4):
    """utils/vbx.py:27-137 (GMM update branch)."""
    D = X.shape[1]
    if type(pi) is int:
        pi = np.ones(pi) / pi
    G = -0.5 * (np.sum(X ** 2, axis=1, keepdims=True) + D * np.log(2 * np.pi))
    V = np.sqrt(Phi)
    rho = X * V
    Li = []
    for ii in range(maxIters):
        invL = 1.0 / (1 + Fa / Fb * gamma.sum(axis=0, keepdims=True).T * Phi)
        alpha = Fa / Fb * invL * gamma.T.dot(rho)
        log_p_ = Fa * (rho.dot(alpha.T) - 0.5 * (invL + alpha ** 2).dot(Phi) + G)
        eps = 1e-8
        lpi = np.log(pi + eps)
        log_p_x = logsumexp(log_p_ + lpi, axis=-1)
        log_pX_ = np.sum(log_p_x, axis=0)
        gamma = np.exp(log_p_ + lpi - log_p_x[:, None])
        pi = np.sum(gamma, axis=0)
        pi = pi / pi.sum()
        ELBO = log_pX_ + Fb * 0.5 * np.sum(np.log(invL) - invL - alpha ** 2 + 1)
        Li.append([ELBO])
        if ii > 0 and ELBO - Li[-2][0] < epsilon:
            break
    return gamma, pi, Li


def cluster_vbx(ahc_init, fea, Phi, Fa, Fb, maxIters=20, init_smoothing=7.0):
    qinit = np.zeros((len(ahc_init), ahc_init.max() + 1))
    qinit[range(len(ahc_init)), ahc_init.astype(int)] = 1.0
    qinit = qinit if init_smoothing < 0 else softmax(qinit * init_smoothing, axis=1)
    gamma, pi, _ = VBx(fea, Phi, Fa=Fa, Fb=Fb, pi=qinit.shape[1], gamma=qinit, maxIters=maxIters)
    return gamma, pi


# ----------------------------------------------------------------------------------------
# clustering
# ----------------------------------------------------------------------------------------


def filter_embeddings(embeddings, seg_data, min_active_ratio=0.2):
    _, num_frames, _ = seg_data.shape
    single = (np.sum(seg_data, axis=2, keepdims=True) == 1)
    num_clean = np.sum(seg_data * single, axis=1)
    active = num_clean >= min_active_ratio * num_frames
    valid = ~np.any(np.isnan(embeddings), axis=2)
    chunk_idx, speaker_idx = np.where(active * valid)
    return embeddings[chunk_idx, speaker_idx], chunk_idx, speaker_idx


def constrained_argmax(soft):
    soft = np.nan_to_num(soft, nan=np.nanmin(soft))
    num_chunks, num_speakers, _ = soft.shape
    hard = -2 * np.ones((num_chunks, num_speakers), dtype=np.int8)
    for c, cost in enumerate(soft):
        speakers, clusters = linear_sum_assignment(cost, maximize=True)
        for s, k in zip(speakers, clusters):
            hard[c, s] = k
    return hard


def ahc_centroid_labels(train_embeddings, threshold):
    normed = train_embeddings / np.linalg.norm(train_embeddings, axis=1, keepdims=True)
    dendrogram = linkage(normed, method="centroid", metric="euclidean")
    ahc = fcluster(dendrogram, threshold, criterion="distance") - 1
    _, ahc = np.unique(ahc, return_inverse=True)
    return ahc, dendrogram, normed


def vbx_clustering(embeddings, seg_data, plda: PLDA, threshold=0.6, Fa=0.07, Fb=0.8,
                   num_clusters=None, min_clusters=None, max_clusters=None, return_debug=False):
    """VBxClustering.__call__ (pipelines/clustering.py:572-669); KMeans fallback (:626-642)."""
    min_clusters = min_clusters if min_clusters is not None else 1
    max_clusters = max_clusters if max_clusters is not None else np.inf
    constrained = True
    train, _, _ = filter_embeddings(embeddings, seg_data)
    num_chunks, num_speakers, dimension = embeddings.shape
    if train.shape[0] < 2:
        hard = np.zeros((num_chunks, num_speakers), dtype=np.int8)
        soft = np.ones((num_chunks, num_speakers, 1))
        centroids = np.mean(train, axis=0, keepdims=True)
        return (hard, soft, centroids, {}) if return_debug else (hard, soft, centroids)
    ahc, dendrogram, normed = ahc_centroid_labels(train, threshold)
    fea = plda(train)
    q, sp = cluster_vbx(ahc, fea, plda.phi, Fa=Fa, Fb=Fb, maxIters=20)
    W = q[:, sp > 1e-7]
    centroids = W.T @ train.reshape(-1, dimension) / W.sum(0, keepdims=True).T
    auto_num, _ = centroids.shape
    if auto_num < min_clusters:
        num_clusters = min_clusters
    elif auto_num > max_clusters:
        num_clusters = max_clusters
    if num_clusters and num_clusters != auto_num:
        from sklearn.cluster import KMeans

        constrained = False
        km = KMeans(n_clusters=num_clusters, n_init=3, random_state=42, copy_x=False).fit_predict(normed)
        centroids = np.vstack([np.mean(train[km == k], axis=0) for k in range(num_clusters)])
    e2k = cdist(embeddings.reshape(-1, dimension), centroids, metric="cosine").reshape(
        num_chunks, num_speakers, -1)
    soft = 2 - e2k
    if constrained:
        const = soft.min() - 1.0
        soft[seg_data.sum(1) == 0] = const
        hard = constrained_argmax(soft)
    else:
        hard = np.argmax(soft, axis=2)
    hard = hard.reshape(num_chunks, num_speakers)
    if return_debug:
        return hard, soft, centroids, dict(ahc=ahc, dendrogram=dendrogram, fea=fea, q=q, sp=sp, train=train)
    return hard, soft, centroids


def ahc_cluster(embeddings, method="centroid", threshold=0.0, min_cluster_size=0,
                min_clusters=1, max_clusters=None, num_clusters=None, metric="cosine"):
    """AgglomerativeClustering.cluster (pipelines/clustering.py:330-480), legacy 3.1 path."""
    embeddings = np.array(embeddings)          # a copy in the caller's dtype: the reference normalises IN PLACE, i.e.
    num_embeddings, _ = embeddings.shape       # in float32 when called through BaseClustering.__call__ (:371-373)
    max_clusters = max_clusters if max_clusters is not None else num_embeddings
    min_cluster_size = min(min_cluster_size, max(1, round(0.1 * num_embeddings)))
    if num_embeddings == 1:
        return np.zeros((1,), dtype=np.uint8)
    if metric == "cosine" and method in ["centroid", "median", "ward"]:
        with np.errstate(divide="ignore", invalid="ignore"):
            embeddings /= np.linalg.norm(embeddings, axis=-1, keepdims=True)
        dendrogram = linkage(embeddings, method=method, metric="euclidean")
    else:
        dendrogram = linkage(embeddings, method=method, metric=metric)
    clusters = fcluster(dendrogram, threshold, criterion="distance") - 1
    uniq, counts = np.unique(clusters, return_counts=True)
    large = uniq[counts >= min_cluster_size]
    num_large = len(large)
    if num_large < min_clusters:
        num_clusters = min_clusters
    elif num_large > max_clusters:
        num_clusters = max_clusters
    if num_clusters is not None and num_large != num_clusters:
        _d = np.copy(dendrogram)
        _d[:, 2] = np.arange(num_embeddings - 1)
        best_iteration = num_embeddings - 1
        best_num_large = 1
        for iteration in np.argsort(np.abs(dendrogram[:, 2] - threshold)):
            if _d[iteration, 3] < min_cluster_size:
                continue
            clusters = fcluster(_d, iteration, criterion="distance") - 1
            uniq, counts = np.unique(clusters, return_counts=True)
            large = uniq[counts >= min_cluster_size]
            num_large = len(large)
            if abs(num_large - num_clusters) < abs(best_num_large - num_clusters):
                best_iteration = iteration
                best_num_large = num_large
            if num_large == num_clusters:
                break
        if best_num_large != num_clusters:
            clusters = fcluster(_d, best_iteration, criterion="distance") - 1
            uniq, counts = np.unique(clusters, return_counts=True)
            large = uniq[counts >= min_cluster_size]
            num_large = len(large)
    if num_large == 0:
        clusters[:] = 0
        return clusters
    small = uniq[counts < min_cluster_size]
    if len(small) == 0:
        return clusters
    large_c = np.vstack([np.mean(embeddings[clusters == k], axis=0) for k in large])
    small_c = np.vstack([np.mean(embeddings[clusters == k], axis=0) for k in small])
    d = cdist(large_c, small_c, metric=metric)
    for sk, lk in enumerate(np.argmin(d, axis=0)):
        clusters[clusters == small[sk]] = large[lk]
    _, clusters = np.unique(clusters, return_inverse=True)
    return clusters


def set_num_clusters(num_embeddings, num_clusters=None, min_clusters=None, max_clusters=None):
    """BaseClustering.set_num_clusters (pipelines/clustering.py:54-75)."""
    min_clusters = num_clusters or min_clusters or 1
    min_clusters = max(1, min(num_embeddings, min_clusters))
    max_clusters = num_clusters or max_clusters or num_embeddings
    max_clusters = max(1, min(num_embeddings, max_clusters))
    if min_clusters > max_clusters:
        raise ValueError("min_clusters must be smaller than (or equal to) max_clusters")
    if min_clusters == max_clusters:
        num_clusters = min_clusters
    return num_clusters, min_clusters, max_clusters


def ahc_call(embeddings, seg_data, threshold, min_cluster_size, method="centroid", num_clusters=None,
             min_clusters=None, max_clusters=None, constrained=False):
    """AgglomerativeClustering via BaseClustering.__call__ (pipelines/clustering.py:214-289) +
    assign_embeddings (:142-212): filter -> cluster -> centroids = mean of train embeddings per cluster ->
    cosine cdist -> (constrained) argmax.  Returns (hard, soft, centroids)."""
    train, chunk_idx, speaker_idx = filter_embeddings(embeddings, seg_data)
    num_chunks, num_speakers, dimension = embeddings.shape
    num_clusters, min_clusters, max_clusters = set_num_clusters(train.shape[0], num_clusters, min_clusters,
                                                                max_clusters)
    if max_clusters < 2:
        return (np.zeros((num_chunks, num_speakers), dtype=np.int8), np.ones((num_chunks, num_speakers, 1)),
                np.mean(train, axis=0, keepdims=True))
    train_clusters = ahc_cluster(train, method=method, threshold=threshold, min_cluster_size=min_cluster_size,
                                 min_clusters=min_clusters, max_clusters=max_clusters, num_clusters=num_clusters)
    K = int(np.max(train_clusters)) + 1
    centroids = np.vstack([np.mean(train[train_clusters == k], axis=0) for k in range(K)])
    e2k = cdist(embeddings.reshape(-1, dimension), centroids, metric="cosine").reshape(num_chunks, num_speakers, -1)
    soft = 2 - e2k
    hard = constrained_argmax(soft) if constrained else np.argmax(soft, axis=2)
    return hard, soft, centroids


# ----------------------------------------------------------------------------------------
# reconstruct + apply
# ----------------------------------------------------------------------------------------


def clustered_segmentations(segmentations: SWF, hard_clusters) -> SWF:
    """speaker_diarization.py:480-520: per chunk, the activity of a cluster is the max over its local speakers."""
    num_chunks, num_frames, _ = segmentations.data.shape
    num_clusters = int(np.max(hard_clusters)) + 1
    clustered = np.nan * np.zeros((num_chunks, num_frames, num_clusters))
    for c in range(num_chunks):
        cluster = hard_clusters[c]
        seg = segmentations.data[c]
        for k in np.unique(cluster):
            if k == -2:
                continue
            clustered[c, :, k] = np.max(seg[:, cluster == k], axis=1)
    return SWF(clustered, segmentations.sw)


def reconstruct(segmentations: SWF, hard_clusters, count: SWF) -> SWF:
    return to_diarization(clustered_segmentations(segmentations, hard_clusters), count)


@dataclass
class OracleOutput:
    segmentations: SWF = None
    count: SWF = None
    embeddings: np.ndarray = None
    hard_clusters: np.ndarray = None
    soft_clusters: np.ndarray = None                        # (chunks, speakers, clusters) scores behind hard_clusters
    centroids: np.ndarray = None
    discrete: SWF = None
    exclusive: SWF = None
    segments: list = field(default_factory=list)           # (start_frame, end_frame, label_index)
    exclusive_segments: list = field(default_factory=list)
    times: list = field(default_factory=list)               # (start_s, end_s, "SPEAKER_xx")
    exclusive_times: list = field(default_factory=list)
    labels: list = field(default_factory=list)
    speaker_embeddings: np.ndarray = None


def apply(seg_model, emb_model, plda: PLDA, waveform: torch.Tensor, threshold=0.6, Fa=0.07, Fb=0.8,
          num_speakers=None, min_speakers=None, max_speakers=None, seg_batch=32, emb_batch=8,
          share_trunk=True, segmentations: SWF = None, embeddings=None, exclude_overlap=False,
          min_duration_off=0.0) -> OracleOutput:
    """SpeakerDiarization.apply (pipelines/speaker_diarization.py:530-784), powerset + VBx branch."""
    min_speakers = num_speakers or min_speakers or 1
    max_speakers = num_speakers or max_speakers or np.inf
    if min_speakers == max_speakers:
        num_speakers = min_speakers
    out = OracleOutput()
    frames = SW(*nets.sincnet_receptive_field())
    seg = segmentations if segmentations is not None else slide(seg_model, waveform, seg_batch)
    out.segmentations = seg
    count = speaker_count(seg, frames, warm_up=(0.0, 0.0))
    out.count = SWF(count.data.copy(), count.sw)
    if np.nanmax(count.data) == 0.0:
        out.speaker_embeddings = np.zeros((0, 256))
        return out
    emb = embeddings if embeddings is not None else get_embeddings(
        emb_model, waveform, seg, exclude_overlap=exclude_overlap, batch_size=emb_batch, share_trunk=share_trunk)
    out.embeddings = emb
    hard, soft, centroids = vbx_clustering(emb, seg.data, plda, threshold, Fa, Fb, num_clusters=num_speakers,
                                           min_clusters=min_speakers, max_clusters=max_speakers)
    out.soft_clusters = soft
    count.data = np.minimum(count.data, max_speakers).astype(np.int8)
    inactive = np.sum(seg.data, axis=1) == 0
    hard = hard.copy()
    hard[inactive] = -2
    out.hard_clusters = hard
    out.discrete = reconstruct(seg, hard, count)
    out.segments, times = binarize_to_segments(out.discrete)
    count.data = np.minimum(count.data, 1).astype(np.int8)
    out.exclusive = reconstruct(seg, hard, count)
    out.exclusive_segments, xtimes = binarize_to_segments(out.exclusive)
    if min_duration_off > 0.0:
        times, xtimes = support(times, min_duration_off), support(xtimes, min_duration_off)
    labels = sorted({k for _, _, k in out.segments})
    mapping = {k: f"SPEAKER_{i:02d}" for i, k in enumerate(labels)}
    out.labels = [mapping[k] for k in labels]
    out.times = [(a, b, mapping[k]) for a, b, k in times]
    out.exclusive_times = [(a, b, mapping.get(k, k)) for a, b, k in xtimes]
    if len(labels) > centroids.shape[0]:
        centroids = np.pad(centroids, ((0, len(labels) - centroids.shape[0]), (0, 0)))
    out.centroids = centroids
    out.speaker_embeddings = centroids[labels] if len(labels) else centroids[:0]
    return out
