"""Clustering stage (mirror of /root/reference/src/pyannote/audio/pipelines/clustering.py, core/plda.py, utils/vbx.py).

Same classes / call signatures as the reference (``VBxClustering``, ``AgglomerativeClustering``, ``PLDA``); the
arithmetic runs in fp64 on the device through libb200diar.so: clean-frame filter, centroid linkage, PLDA transform
(plain fp64 matmuls), VBx iterations, cosine cdist and the constrained 3xK assignment.  Only the dendrogram cut
(``fcluster``, a tree walk over (n-1) rows) and the rarely used KMeans fallback stay on the host.
"""
from __future__ import annotations

from pathlib import Path
from typing import Optional, Union

import numpy as np
import torch

from . import ops
from .core import SlidingWindowFeature
from .models import get_context


class PLDA:
    """core/plda.py:33-63 over utils/vbx.py:181-218.  The one-off setup (matrix inverses + generalised eigh) runs on
    the host in float64 exactly like the reference; the per-file transform runs on the device."""

    def __init__(self, transform_npz: Union[str, Path, dict], plda_npz: Union[str, Path, dict, None] = None,
                 lda_dimension: int = 128):
        from scipy.linalg import eigh

        x = transform_npz if isinstance(transform_npz, dict) else np.load(transform_npz)
        p = x if plda_npz is None else (plda_npz if isinstance(plda_npz, dict) else np.load(plda_npz))
        self.mean1, self.mean2, self.lda = (np.asarray(x[k], dtype=np.float64) for k in ("mean1", "mean2", "lda"))
        mu, tr, psi = (np.asarray(p[k], dtype=np.float64) for k in ("mu", "tr", "psi"))
        W = np.linalg.inv(tr.T.dot(tr))
        B = np.linalg.inv((tr.T / psi).dot(tr))
        acvar, wccn = eigh(B, W)
        self._plda_psi = acvar[::-1].copy()
        self._plda_tr = wccn.T[::-1].copy()
        self._plda_mu = mu
        self.lda_dimension = lda_dimension
        self._dev = {}

    @classmethod
    def from_pretrained(cls, checkpoint, subfolder: Optional[str] = None, revision: Optional[str] = None, token=None,
                        cache_dir=None, **kwargs) -> "PLDA":
        """core/plda.py:65-135 for local checkpoints: a directory holding ``xvec_transform.npz`` and ``plda.npz``
        (optionally under ``subfolder``).  Hub identifiers cannot be downloaded here (no network)."""
        import os

        if not os.path.isdir(checkpoint):
            if "@" in str(checkpoint):
                raise ValueError("Revisions must be passed with `revision` keyword argument.")
            raise ValueError(f"'{checkpoint}' is not a local directory; Hugging Face hub identifiers cannot be "
                             f"downloaded here (no network)")
        if revision is not None:
            raise ValueError("Revisions cannot be used with local checkpoints.")
        base = Path(checkpoint) / subfolder if subfolder else Path(checkpoint)
        return cls(base / "xvec_transform.npz", base / "plda.npz", **kwargs)

    @property
    def phi(self) -> np.ndarray:
        return self._plda_psi[: self.lda_dimension]

    def _consts(self, device):
        key = str(device)
        if key not in self._dev:
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)  # noqa: E731
            self._dev[key] = dict(mean1=t(self.mean1), mean2=t(self.mean2), lda=t(self.lda), mu=t(self._plda_mu),
                                  trT=t(self._plda_tr.T[:, : self.lda_dimension]), phi=t(self.phi))
        return self._dev[key]

    def transform(self, x: torch.Tensor) -> torch.Tensor:
        """(n, 256) float64 device tensor -> (n, lda_dimension) (vbx.py:211-217), one kernel (b200_plda_transform)."""
        c = self._consts(x.device)
        return get_context(x.device).plda_transform(x.double(), c["mean1"], c["mean2"], c["lda"], c["mu"], c["trT"])

    def __call__(self, embeddings) -> np.ndarray:
        if isinstance(embeddings, torch.Tensor):
            return self.transform(embeddings.double())
        dev = torch.device("cuda", torch.cuda.current_device())
        return self.transform(torch.from_numpy(np.asarray(embeddings, dtype=np.float64)).to(dev)).cpu().numpy()


def _seg_tensor(segmentations, ctx) -> torch.Tensor:
    """(C,589,3) uint8 device tensor from a SlidingWindowFeature / ndarray / tensor of {0,1}."""
    data = segmentations.data if isinstance(segmentations, SlidingWindowFeature) else segmentations
    if isinstance(data, torch.Tensor):
        return data.to(device=ctx.device, dtype=torch.uint8).contiguous()
    return torch.from_numpy(np.nan_to_num(np.asarray(data), nan=0.0).astype(np.uint8)).to(ctx.device).contiguous()


class BaseClustering:
    def __init__(self, metric: str = "cosine", constrained_assignment: bool = False, device=None):
        if metric != "cosine":
            raise NotImplementedError("the device clustering path implements the cosine metric (community-1)")
        self.metric = metric
        self.constrained_assignment = constrained_assignment
        self.device = device

    def _ctx(self, like=None):
        if isinstance(like, torch.Tensor) and like.is_cuda:
            return get_context(like.device)
        return get_context(self.device if self.device is not None else torch.device("cuda", torch.cuda.current_device()))

    def set_num_clusters(self, num_embeddings: int, num_clusters=None, min_clusters=None, max_clusters=None):
        min_clusters = num_clusters or min_clusters or 1
        min_clusters = max(1, min(num_embeddings, min_clusters))
        max_clusters = num_clusters or max_clusters or num_embeddings
        max_clusters = max(1, min(num_embeddings, max_clusters))
        if min_clusters > max_clusters:
            raise ValueError(f"min_clusters must be smaller than (or equal to) max_clusters "
                             f"(here: min_clusters={min_clusters:g} and max_clusters={max_clusters:g}).")
        if min_clusters == max_clusters:
            num_clusters = min_clusters
        return num_clusters, min_clusters, max_clusters

    def filter_embeddings(self, embeddings, segmentations, min_active_ratio: float = 0.2):
        """clustering.py:77-125 -> (train (n,256) f64 device, chunk_idx, speaker_idx, active (C,3) bool device)."""
        ctx = self._ctx(embeddings)
        seg = _seg_tensor(segmentations, ctx)
        emb = embeddings if isinstance(embeddings, torch.Tensor) else torch.from_numpy(np.asarray(embeddings))
        emb = emb.to(ctx.device)
        num_frames = seg.shape[1]
        clean, active = ctx.clean_frames(seg)
        keep = (clean.double() >= min_active_ratio * num_frames) & ~torch.isnan(emb).any(dim=2)
        chunk_idx, speaker_idx = torch.nonzero(keep, as_tuple=True)
        return emb[chunk_idx, speaker_idx].double(), chunk_idx, speaker_idx, active.bool()

    def constrained_argmax(self, soft_clusters) -> np.ndarray:
        ctx = self._ctx(soft_clusters)
        soft = soft_clusters if isinstance(soft_clusters, torch.Tensor) else torch.from_numpy(soft_clusters)
        soft = torch.nan_to_num(soft.to(ctx.device).double(), nan=float(torch.nan_to_num(soft, nan=np.inf).min()))
        return ctx.assign(soft, constrained=True).cpu().numpy()

    def _assign(self, ctx, emb64, centroids, active, constrained):
        """``active`` (C,3) bool: VBx gives inactive speakers the score ``soft.min() - 1`` before the constrained
        assignment (clustering.py:655-663); None: scores as computed (assign_embeddings, :142-212)."""
        C = emb64.shape[0]
        K = centroids.shape[0]
        e2k = ctx.cdist_cosine(emb64.reshape(-1, emb64.shape[-1]), centroids).reshape(C, ops.SPEAKERS, K)
        soft = 2 - e2k
        if not constrained:
            return ctx.assign(soft, constrained=False), soft
        # with a NaN embedding row (filter_embeddings drops it from training, but it is still assigned) `const` is NaN
        # too and so are the inactive rows; constrained_argmax (:127-132) gives the solver NaN replaced by the
        # nan-minimum, and the caller gets `soft` with its NaN
        if active is not None:
            const = soft.min() - 1.0
            soft = torch.where(active[:, :, None], soft, const)
        nanmin = torch.nan_to_num(soft, nan=float("inf")).min()
        hard = ctx.assign(torch.where(torch.isnan(soft), nanmin, soft), constrained=True)
        return hard, soft


class _Tick:
    """B200_TIMING=2: synchronising wall-clock split of cluster_batch (diagnostics only)."""

    def __init__(self, dev):
        import os, time
        self.on = os.environ.get("B200_TIMING") == "2"
        self.dev, self.t, self.acc, self._time = dev, None, {}, time
        if self.on:
            torch.cuda.synchronize(dev)
            self.t = time.perf_counter()

    def __call__(self, name):
        if not self.on:
            return
        torch.cuda.synchronize(self.dev)
        now = self._time.perf_counter()
        self.acc[name] = self.acc.get(name, 0.0) + (now - self.t) * 1e3
        self.t = now

    def report(self):
        if self.on:
            import sys
            print("[b200 clustering] " + ", ".join(f"{k}={v:.1f}ms" for k, v in self.acc.items()), file=sys.stderr)


class VBxClustering(BaseClustering):
    expects_num_clusters: bool = False

    def __init__(self, plda: PLDA, metric: str = "cosine", constrained_assignment: bool = True, device=None):
        super().__init__(metric=metric, constrained_assignment=constrained_assignment, device=device)
        self.plda = plda
        self.threshold, self.Fa, self.Fb = 0.6, 0.07, 0.8

    def instantiate(self, params: dict):
        for k in ("threshold", "Fa", "Fb"):
            if k in params:
                setattr(self, k, float(params[k]))
        return self

    def cluster_batch(self, emb_all: torch.Tensor, seg_all: torch.Tensor, bounds, num_clusters=None,
                      min_clusters=None, max_clusters=None, skip=None):
        """VBx clustering of several files at once (clustering.py:572-669 per file).

        emb_all (Ctot,3,256) f32 and seg_all (Ctot,589,3) u8 are device tensors holding the files back to back,
        ``bounds`` the chunk boundaries (F+1,).  Device work is batched across files (one linkage launch, one VBx
        launch, ...); host work is the dendrogram cut per file.  Returns a list of dicts with device tensors:
        hard (C,3) int8, soft (C,3,K) f64, centroids (K,256) f64, active (C,3) bool (+ debug entries).
        """
        ctx = self._ctx(emb_all)
        dev = ctx.device
        tick = _Tick(dev)
        min_clusters = min_clusters if min_clusters is not None else 1
        max_clusters = max_clusters if max_clusters is not None else np.inf
        F = len(bounds) - 1
        skip = skip if skip is not None else [False] * F
        num_frames = seg_all.shape[1]
        dim = emb_all.shape[-1]
        clean, active_all = ctx.clean_frames(seg_all)
        keep = (clean.double() >= 0.2 * num_frames) & ~torch.isnan(emb_all).any(dim=2)          # (Ctot,3)
        flat_idx = torch.nonzero(keep.reshape(-1)).reshape(-1)                                    # row-major = np.where
        csum = torch.cumsum(keep.sum(dim=1), dim=0)
        bnd = torch.as_tensor(np.asarray(bounds[1:], dtype=np.int64) - 1, device=dev)
        ends = csum[bnd].cpu().numpy().astype(np.int64)                                           # sync: train counts
        row_off = np.concatenate([[0], ends]).astype(np.int32)
        n_f = np.diff(row_off)
        train_all = emb_all.reshape(-1, dim)[flat_idx].double()
        emb64_all = emb_all.double()
        active_all = active_all.bool()
        tick("filter")
        results = [None] * F
        todo = []
        for f in range(F):
            c0, c1 = int(bounds[f]), int(bounds[f + 1])
            if skip[f]:
                continue
            if n_f[f] < 2:
                tr = train_all[row_off[f]: row_off[f + 1]]
                results[f] = dict(hard=torch.zeros((c1 - c0, ops.SPEAKERS), dtype=torch.int8, device=dev),
                                  soft=torch.ones((c1 - c0, ops.SPEAKERS, 1), dtype=torch.float64, device=dev),
                                  centroids=tr.mean(dim=0, keepdim=True), active=active_all[c0:c1], trivial=True)
            else:
                todo.append(f)
        if not todo:
            return results
        # ---- AHC: one batched linkage launch, dendrogram cut on the host ------------------------------------
        lro_n = np.where(np.isin(np.arange(F), todo), n_f, 0)           # problems not in `todo` get n = 0
        sub_off = np.concatenate([[0], np.cumsum(lro_n)]).astype(np.int32)
        if len(todo) == F and not any(skip):
            x_link, link_off = train_all, row_off
        else:
            x_link = torch.cat([train_all[row_off[f]: row_off[f + 1]] for f in todo])
            link_off = sub_off
        # embeddings are float32 network outputs: normalise them exactly as numpy does on float32 (clustering.py:597-599)
        Z_all = ctx.linkage_centroid_batched(x_link, link_off, normalize="float32").cpu().numpy()   # sync
        tick("linkage")
        ahcs, S_f, zpos = {}, {}, 0
        for f in todo:
            n = int(n_f[f])
            Z = Z_all[zpos: zpos + n - 1]
            zpos += n - 1
            ahc = ops.fcluster_distance(Z, self.threshold) - 1
            _, ahc = np.unique(ahc, return_inverse=True)
            ahcs[f], S_f[f] = ahc, int(ahc.max()) + 1
            results[f] = dict(dendrogram=Z, ahc=ahc)
        tick("fcluster(host)")
        # ---- VBx: PLDA transform of all rows, initial responsibilities built on the host, one launch ----------
        fea = self.plda.transform(x_link)
        hot_blocks = []
        for f in todo:
            n, S = int(n_f[f]), S_f[f]
            # softmax(7 * one_hot) (vbx.py:142-144) has two distinct values per row
            tot = 1.0 + (S - 1) * np.exp(-7.0)
            g = np.full((n, S), np.exp(-7.0) / tot)
            g[np.arange(n), ahcs[f]] = 1.0 / tot
            hot_blocks.append(g.reshape(-1))
        gamma0 = torch.from_numpy(np.concatenate(hot_blocks)).to(dev)
        tick("plda+gamma0")
        phi = self.plda._consts(dev)["phi"]
        n_list = [int(n_f[f]) for f in todo]
        S_list = [S_f[f] for f in todo]
        gamma, pi, _ = ctx.vbx_batched(fea, phi, gamma0, n_list, S_list, self.Fa, self.Fb, max_iters=20)
        pi_host = pi.cpu().numpy()                                                                 # sync
        tick("vbx")
        # speakers that survive VBx (clustering.py:619: sp > 1e-7), for all files in ONE host -> device copy
        kept_lists, spos = [], 0
        for S in S_list:
            kept_lists.append(np.nonzero(pi_host[spos: spos + S] > 1e-7)[0].astype(np.int32))
            spos += S
        kept_all = torch.from_numpy(np.concatenate(kept_lists)).to(dev)
        gpos = spos = rpos = kpos = 0
        for j, (f, n, S) in enumerate(zip(todo, n_list, S_list)):
            c0, c1 = int(bounds[f]), int(bounds[f + 1])
            q = gamma[gpos: gpos + n * S].reshape(n, S)
            sp = pi_host[spos: spos + S]
            train = x_link[rpos: rpos + n]
            gpos, spos, rpos = gpos + n * S, spos + S, rpos + n
            kept = kept_all[kpos: kpos + len(kept_lists[j])]
            kpos += len(kept_lists[j])
            centroids = ctx.weighted_centroids(q, kept, train)
            constrained = self.constrained_assignment
            auto_num = centroids.shape[0]
            nc = num_clusters
            if auto_num < min_clusters:
                nc = min_clusters
            elif auto_num > max_clusters:
                nc = max_clusters
            if nc and nc != auto_num:
                from sklearn.cluster import KMeans

                constrained = False
                tr = train.cpu().numpy().astype(np.float32)       # the float32 rows the reference works on (:629-642)
                normed = tr / np.linalg.norm(tr, axis=1, keepdims=True)
                km = KMeans(n_clusters=int(nc), n_init=3, random_state=42, copy_x=False).fit_predict(normed)
                centroids = torch.from_numpy(np.vstack([np.mean(tr[km == k], axis=0)
                                                        for k in range(int(nc))]).astype(np.float64)).to(dev)
            hard, soft = self._assign(ctx, emb64_all[c0:c1], centroids.contiguous(), active_all[c0:c1], constrained)
            results[f].update(hard=hard, soft=soft, centroids=centroids, active=active_all[c0:c1], q=q, sp=sp,
                              train=train, fea=fea[rpos - n: rpos], trivial=False)
        tick("centroids+assign")
        tick.report()
        return results

    def __call__(self, embeddings, segmentations=None, num_clusters=None, min_clusters=None, max_clusters=None,
                 return_debug: bool = False, **kwargs):
        """clustering.py:572-669.  Returns (hard_clusters (C,3) int8, soft_clusters (C,3,K) f64, centroids (K,256))."""
        ctx = self._ctx(embeddings)
        emb = embeddings if isinstance(embeddings, torch.Tensor) else torch.from_numpy(np.asarray(embeddings))
        emb = emb.to(ctx.device).float().contiguous()
        seg = _seg_tensor(segmentations, ctx)
        r = self.cluster_batch(emb, seg, [0, emb.shape[0]], num_clusters, min_clusters, max_clusters)[0]
        out = (r["hard"].cpu().numpy(), r["soft"].cpu().numpy(), r["centroids"].cpu().numpy())
        if return_debug:
            dbg = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in r.items()
                   if k in ("ahc", "dendrogram", "q", "sp", "fea", "train", "active")}
            return out + (dbg,)
        return out


class AgglomerativeClustering(BaseClustering):
    """Legacy (3.1) clustering, clustering.py:293-480.  ``method="centroid"`` runs on the device."""

    expects_num_clusters: bool = False

    def __init__(self, metric: str = "cosine", constrained_assignment: bool = False, device=None):
        super().__init__(metric=metric, constrained_assignment=constrained_assignment, device=device)
        self.method, self.threshold, self.min_cluster_size = "centroid", 0.7, 12

    def instantiate(self, params: dict):
        for k in ("method", "threshold", "min_cluster_size"):
            if k in params:
                setattr(self, k, params[k])
        return self

    def cluster(self, embeddings: np.ndarray, min_clusters: int = 1, max_clusters: Optional[int] = None,
                num_clusters: Optional[int] = None) -> np.ndarray:
        if self.method != "centroid":
            raise NotImplementedError("device linkage implements method='centroid' (the pyannote default)")
        ctx = self._ctx()
        embeddings = np.array(embeddings)                   # copy; the reference normalises in the caller's dtype
        if embeddings.dtype not in (np.float32, np.float64):
            embeddings = embeddings.astype(np.float64)
        f32 = embeddings.dtype == np.float32
        num_embeddings, _ = embeddings.shape
        max_clusters = max_clusters if max_clusters is not None else num_embeddings
        min_cluster_size = min(self.min_cluster_size, max(1, round(0.1 * num_embeddings)))
        if num_embeddings == 1:
            return np.zeros((1,), dtype=np.uint8)
        x = torch.from_numpy(embeddings.astype(np.float64)).to(ctx.device)
        dendrogram = ctx.linkage_centroid(x, normalize="float32" if f32 else True).cpu().numpy()
        with np.errstate(divide="ignore", invalid="ignore"):
            embeddings /= np.linalg.norm(embeddings, axis=-1, keepdims=True)
        clusters = ops.fcluster_distance(dendrogram, self.threshold) - 1
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
            best_iteration, best_num_large = num_embeddings - 1, 1
            for iteration in np.argsort(np.abs(dendrogram[:, 2] - self.threshold)):
                if _d[iteration, 3] < min_cluster_size:
                    continue
                clusters = ops.fcluster_distance(_d, iteration) - 1
                uniq, counts = np.unique(clusters, return_counts=True)
                large = uniq[counts >= min_cluster_size]
                num_large = len(large)
                if abs(num_large - num_clusters) < abs(best_num_large - num_clusters):
                    best_iteration, best_num_large = iteration, num_large
                if num_large == num_clusters:
                    break
            if best_num_large != num_clusters:
                clusters = ops.fcluster_distance(_d, best_iteration) - 1
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
        d = ctx.cdist_cosine(torch.from_numpy(large_c.astype(np.float64)).to(ctx.device),
                             torch.from_numpy(small_c.astype(np.float64)).to(ctx.device))
        for sk, lk in enumerate(torch.argmin(d, dim=0).cpu().numpy()):
            clusters[clusters == small[sk]] = large[lk]
        _, clusters = np.unique(clusters, return_inverse=True)
        return clusters

    def __call__(self, embeddings, segmentations=None, num_clusters=None, min_clusters=None, max_clusters=None,
                 **kwargs):
        """BaseClustering.__call__ (clustering.py:214-289) + assign_embeddings (:142-212)."""
        ctx = self._ctx(embeddings)
        train, chunk_idx, speaker_idx, active = self.filter_embeddings(embeddings, segmentations)
        emb = embeddings if isinstance(embeddings, torch.Tensor) else torch.from_numpy(np.asarray(embeddings))
        emb64 = emb.to(ctx.device).double()
        num_chunks, num_speakers, _ = emb64.shape
        num_embeddings = train.shape[0]
        num_clusters, min_clusters, max_clusters = self.set_num_clusters(num_embeddings, num_clusters, min_clusters,
                                                                         max_clusters)
        if max_clusters < 2:
            hard = np.zeros((num_chunks, num_speakers), dtype=np.int8)
            soft = np.ones((num_chunks, num_speakers, 1))
            return hard, soft, train.mean(dim=0, keepdim=True).cpu().numpy()
        train32 = train.cpu().numpy().astype(np.float32)     # exact: the rows are float32 network outputs
        train_clusters = self.cluster(train32, min_clusters=min_clusters, max_clusters=max_clusters,
                                      num_clusters=num_clusters)
        K = int(train_clusters.max()) + 1
        # centroids = float32 means of the float32 rows, like assign_embeddings (clustering.py:182-188)
        centroids = torch.from_numpy(np.vstack([np.mean(train32[train_clusters == k], axis=0)
                                                for k in range(K)]).astype(np.float64)).to(ctx.device)
        hard, soft = self._assign(ctx, emb64, centroids.contiguous(), None, self.constrained_assignment)
        return hard.cpu().numpy(), soft.cpu().numpy(), centroids.cpu().numpy()
