"""Multi-GPU sharding of the hot path (one process per GPU, torch.distributed; NCCL on GPUs, gloo in CPU tests).

The reference has no inference-time parallelism at all; the path shards naturally:
  * many files  -> ``ChunkPool``: the chunks of all files form one global pool, every rank runs PyanNet + WeSpeaker on
    its share and writes the results straight into its slice of ONE packed buffer, a single in-place NCCL all-gather
    replicates (embeddings (C,3,256) f32 | powerset classes (C,589) u8) on every GPU, then file g is clustered /
    reconstructed on rank g mod N (hook point core/pipeline.py:497-508).  File-level sharding
    without any collective stays available (bench.py --parallelism files);
  * one long file -> ``apply_sharded``: contiguous chunk ranges per rank (chunk c only needs samples
    [c*step, c*step+160000)), the same all-gather, clustering replicated.
"""
from __future__ import annotations

from typing import Callable, List, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced split of n chunks: first (n % world) ranks get one extra."""
    base, extra = divmod(n, world)
    a = rank * base + min(rank, extra)
    return a, a + base + (1 if rank < extra else 0)


def shard_files(n: int, rank: int, world: int) -> List[int]:
    return list(range(rank, n, world))


def all_gather_rows(local: torch.Tensor, counts: Sequence[int], group=None) -> torch.Tensor:
    """All-gather of row blocks with per-rank row counts known to everyone (derived from shard_range)."""
    world = dist.get_world_size(group)
    mx = max(counts)
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([o[:c] for o, c in zip(out, counts)], dim=0)


def sharded_forward(num_chunks: int, seg_fn: Callable[[int, int], torch.Tensor],
                    emb_fn: Callable[[int, int, torch.Tensor], torch.Tensor], group=None):
    """Runs seg_fn / emb_fn on this rank's chunk range and all-gathers the results.

    seg_fn(a, b) -> (b-a, 589) uint8 powerset classes; emb_fn(a, b, classes) -> (b-a, 3, 256) float32.
    Returns (classes (C,589) u8, embeddings (C,3,256) f32) identical on every rank.
    """
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    counts = [shard_range(num_chunks, r, world)[1] - shard_range(num_chunks, r, world)[0] for r in range(world)]
    a, b = shard_range(num_chunks, rank, world)
    cls = seg_fn(a, b)
    emb = emb_fn(a, b, cls)
    return all_gather_rows(cls.contiguous(), counts, group), all_gather_rows(emb.contiguous(), counts, group)


class ChunkPool:
    """Global chunk pool over many files with one all-gather before clustering (BASELINE.json configs[4]).

    Every rank holds its own files (their chunks are its share of the pool: the heavy per-chunk work never crosses
    NVLink), but clustering ownership is global round-robin (file g -> rank g mod N), which is what balances the
    per-file stage when files differ in length.  One packed buffer [world][emb bytes | class bytes] lives on each
    GPU; the network kernels write their outputs directly into this rank's slice (no staging copy) and
    ``all_gather_into_tensor`` runs in place on it.
    """

    EMB_BYTES = 3 * 256 * 4
    CLS_BYTES = 589

    def __init__(self, pipeline, group=None, collective: str = "nccl"):
        """``collective``: "nccl" = one in-place ncclAllGather of the packed buffer; "p2p" = no collective call at
        all: the pool buffer lives in symmetric memory (every GPU maps every peer's buffer over NVLink), the final
        Linear GEMM of the embedding network pushes its output tiles to all peers from its epilogue
        (b200_emb_forward_push), the powerset classes follow with a P2P copy kernel, and a symmetric-memory barrier
        publishes the stores.  Falls back to "nccl" when symmetric memory cannot be set up."""
        self.pipeline, self.group = pipeline, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.collective = collective if self.world > 1 else "nccl"
        self.last_collective = dict(bytes_sent=0, bytes_received=0, ms=None)
        self._events = None
        self._symm = None          # (buffer, handle) of the symmetric pool

    # ---- planning: per-file chunk counts of every rank (tiny object all-gather, once per batch of files) ----------
    def plan(self, layouts, uris):
        mine = [(u, int(len(l[1])), int(l[3])) for u, l in zip(uris, layouts)]
        everyone = [None] * self.world
        dist.all_gather_object(everyone, mine, group=self.group)
        files, counts = [], []
        for r, lst in enumerate(everyone):
            counts.append(sum(c for _, c, _ in lst))
            pos = 0
            for uri, c, T in lst:
                files.append(dict(uri=uri, rank=r, start=pos, chunks=c, num_samples=T))
                pos += c
        cmax = max(counts) if counts else 0
        blk = -(-(cmax * (self.EMB_BYTES + self.CLS_BYTES)) // 16) * 16
        return dict(files=files, counts=counts, cmax=cmax, blk=blk)

    def views(self, buf, plan, r):
        """(embeddings (C_r,3,256) f32, classes (C_r,589) u8) views of rank r's block of the packed buffer."""
        c, base = plan["counts"][r], r * plan["blk"]
        emb = buf[base: base + c * self.EMB_BYTES].view(torch.float32).view(c, 3, 256)
        o = base + plan["cmax"] * self.EMB_BYTES
        cls = buf[o: o + c * self.CLS_BYTES].view(c, self.CLS_BYTES)
        return emb, cls

    def upload(self, files):
        resident = self.pipeline.upload(files)
        resident["plan"] = self.plan(resident["layouts"], [f.get("uri") for f in resident["files"]])
        return resident

    def apply_batch(self, files, **kwargs):
        yield from self.run_resident(self.upload(files), **kwargs)

    def run_resident(self, resident, num_speakers=None, min_speakers=None, max_speakers=None, hook=None,
                     return_artifacts=False):
        from .models import get_context
        from .pipeline import set_num_speakers

        pipe, plan = self.pipeline, resident["plan"]
        ctx = get_context(pipe.device)
        num_speakers, min_speakers, max_speakers = set_num_speakers(num_speakers, min_speakers, max_speakers)
        pipe.d2h_bytes = 0
        buf, hdl = self._pool_buffer(resident, plan, ctx)
        emb_mine, cls_mine = self.views(buf, plan, self.rank)
        # ---- this rank's share of the pool: outputs land in its slice of the collective's buffer ----------------
        pipe._segmentation.model.forward_chunks(resident["wav"], resident["off"], resident["valid"], out=cls_mine)
        seg_mine = ctx.powerset_to_multilabel(cls_mine)
        if hdl is None:
            pipe.embedding.forward_chunks(resident["wav"], resident["off"], resident["valid"], pipe._masks(seg_mine),
                                          out=emb_mine)
            self.exchange(buf, plan)
        else:
            # fused: the embedding GEMM's epilogue stores every tile into all peers' copies of this rank's slot
            peers = [r for r in range(self.world) if r != self.rank]
            emb_off = emb_mine.data_ptr() - buf.data_ptr()
            cls_off = cls_mine.data_ptr() - buf.data_ptr()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            pipe.embedding.forward_chunks(resident["wav"], resident["off"], resident["valid"], pipe._masks(seg_mine),
                                          out=emb_mine, peers=[int(hdl.buffer_ptrs[r]) + emb_off for r in peers])
            e0.record()
            ctx.push(cls_mine, [int(hdl.buffer_ptrs[r]) + cls_off for r in peers])
            hdl.barrier(channel=0)                         # all ranks' pushes have landed and are visible
            e1.record()
            self._events = (e0, e1)
            self.last_collective = dict(bytes_sent=int(plan["counts"][self.rank] * (self.EMB_BYTES + self.CLS_BYTES)
                                                       * (self.world - 1)),
                                        bytes_received=int(sum(plan["counts"][r] for r in peers)
                                                           * (self.EMB_BYTES + self.CLS_BYTES)))
        got = self.owned_inputs(buf, plan)
        if got is None:
            return
        emb, cls, bounds, owned = got
        seg = ctx.powerset_to_multilabel(cls)
        metas = [dict(uri=plan["files"][g]["uri"], global_index=g, computed_on=plan["files"][g]["rank"])
                 for g in owned]
        from .pipeline import _StageTimer

        pipe._timer = _StageTimer(ctx.device)
        pipe._timer.start()
        outs = pipe._finish_files(ctx, metas, seg, emb, bounds, num_speakers, min_speakers, max_speakers, hook,
                                  return_artifacts, classes=cls)
        for meta, out in zip(metas, outs):
            yield meta, out

    def _pool_buffer(self, resident, plan, ctx):
        """The packed pool buffer: a plain device tensor (nccl) or a symmetric-memory allocation + handle (p2p)."""
        nbytes = self.world * plan["blk"]
        if self.collective == "p2p":
            if self._symm is None or self._symm[0].numel() != nbytes:
                try:
                    import torch.distributed._symmetric_memory as symm_mem

                    grp = self.group if self.group is not None else dist.group.WORLD
                    t = symm_mem.empty(nbytes, dtype=torch.uint8, device=ctx.device)
                    hdl = symm_mem.rendezvous(t, group=grp)
                    t.zero_()
                    torch.cuda.synchronize(ctx.device)
                    dist.barrier(group=self.group)
                    self._symm = (t, hdl)
                except Exception as exc:           # symmetric memory unavailable: same data path through NCCL
                    import warnings

                    warnings.warn(f"symmetric memory unavailable ({exc}); ChunkPool falls back to ncclAllGather")
                    self.collective = "nccl"
            if self.collective == "p2p":
                return self._symm
        buf = resident.get("pool")
        if buf is None or buf.numel() != nbytes:
            buf = resident["pool"] = torch.zeros(nbytes, dtype=torch.uint8, device=ctx.device)
        return buf, None

    def exchange(self, buf, plan):
        """The one exchange step of the path: in-place all-gather of the packed per-rank blocks."""
        mine = buf[self.rank * plan["blk"]: (self.rank + 1) * plan["blk"]]
        timed = buf.is_cuda
        if timed:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        if self.world > 1:
            src = mine if buf.is_cuda else mine.clone()        # NCCL: in place; gloo (CPU tests) wants no aliasing
            dist.all_gather_into_tensor(buf, src, group=self.group)
        if timed:
            e1.record()
            self._events = (e0, e1)
        self.last_collective = dict(bytes_sent=int(plan["blk"]), bytes_received=int(plan["blk"] * (self.world - 1)))

    def owned_inputs(self, buf, plan):
        """Inputs of the per-file stage for the files this rank owns (file g -> rank g mod world): embeddings and
        classes of those files back to back, chunk bounds, global file indices."""
        owned = [g for g in range(len(plan["files"])) if g % self.world == self.rank]
        if not owned:
            return None
        embs, clss, bounds = [], [], [0]
        views = {r: self.views(buf, plan, r) for r in {plan["files"][g]["rank"] for g in owned}}
        for g in owned:
            f = plan["files"][g]
            e, c = views[f["rank"]]
            embs.append(e[f["start"]: f["start"] + f["chunks"]])
            clss.append(c[f["start"]: f["start"] + f["chunks"]])
            bounds.append(bounds[-1] + f["chunks"])
        return torch.cat(embs).contiguous(), torch.cat(clss).contiguous(), bounds, owned

    def collective_ms(self):
        """Device time of the last all-gather (CUDA events on the launching stream; call after a synchronize)."""
        if self._events is None:
            return None
        return float(self._events[0].elapsed_time(self._events[1]))


def apply_sharded(pipeline, file, group=None, **kwargs):
    """SpeakerDiarization over ONE long file with its chunks sharded across the ranks of `group`.

    Every rank holds the (host) waveform, uploads only the sample range its chunks touch, runs PyanNet + WeSpeaker on
    them, all-gathers (NCCL over NVLink) classes + embeddings, and rank-locally finishes clustering / reconstruction
    (cheap, replicated) so that every rank returns the same DiarizeOutput.
    """
    from . import ops
    from .inference import chunk_layout
    from .models import get_context

    pipeline._require_10s_window()
    ctx = get_context(pipeline.device)
    file = pipeline._audio.validate_file(file)
    wav, sr = pipeline._audio(file)
    off, valid, _, _ = chunk_layout(wav.shape[1], ops.CHUNK, round(pipeline._segmentation.step * sr))
    C = len(off)
    state = {}

    def seg_fn(a, b):
        lo, hi = int(off[a]), int(off[b - 1]) + ops.CHUNK
        buf = torch.zeros(hi - lo, dtype=torch.float32, device=ctx.device)
        n = max(0, min(hi, wav.shape[1]) - lo)
        buf[:n].copy_(wav[0, lo: lo + n])
        state.update(buf=buf, off=off[a:b] - lo, valid=valid[a:b])
        return pipeline._segmentation.model.forward_chunks(buf, state["off"], state["valid"])

    def emb_fn(a, b, cls):
        seg = ctx.powerset_to_multilabel(cls)
        return pipeline.embedding.forward_chunks(state["buf"], state["off"], state["valid"], pipeline._masks(seg))

    cls, emb = sharded_forward(C, seg_fn, emb_fn, group)
    seg = ctx.powerset_to_multilabel(cls)
    from .pipeline import set_num_speakers

    ns, mn, mx = set_num_speakers(kwargs.get("num_speakers"), kwargs.get("min_speakers"), kwargs.get("max_speakers"))
    return pipeline._finish_file(ctx, file, seg, emb, ns, mn, mx, kwargs.get("hook"), False)
