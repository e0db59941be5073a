"""Centroid linkage of long recordings: the one-CTA kernel against the whole-GPU path, and one long file end to end.

    python scripts/linkage_long_perf.py [--hours 5] [--out linkage_long_perf.json]

* the linkage alone (b200_linkage_centroid, normalisation + distances + merges) at n = 8192, 32768, 50000 and 65536
  rows of dim 256, normalised as the pipeline normalises them (float32 rows); n <= 32768 run on both paths in
  alternation (the option ``linkage_grid_min``);
* one synthetic multi-hour recording through SpeakerDiarization with B200_TIMING=1 (the stage split); 5 h give
  about 36 000 kept embeddings, above the 32 768 where the whole-GPU path starts, and the script checks that;
* the card's name and power limit, queried in the same run.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def time_linkage(ctx, x, grid_min, reps):
    ctx.set_option("linkage_grid_min", grid_min)
    ms = []
    try:
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            ctx.linkage_centroid(x, normalize="float32")
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
    finally:
        ctx.set_option("linkage_grid_min", 32769)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hours", type=float, default=5.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", type=int, nargs="+", default=[8192, 32768, 50000, 65536])
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()

    from pyannote_audio_b200 import synthetic as syn
    from pyannote_audio_b200.models import PyanNet, WeSpeakerResNet34, get_context
    from pyannote_audio_b200.pipeline import SpeakerDiarization

    dev = torch.device("cuda:0")
    ctx = get_context(dev)
    res = {"card": card(), "linkage_ms": {}}
    ctx.linkage_centroid(torch.ones((2, 256), dtype=torch.float64, device=dev))        # load the module
    print(f"card: {res['card']}", flush=True)
    rng = np.random.default_rng(0)
    centers = rng.standard_normal((40, 256))
    for n in args.sizes:
        x = centers[rng.integers(0, 40, n)] + 0.5 * rng.standard_normal((n, 256))
        x = torch.from_numpy(x.astype(np.float32).astype(np.float64)).to(dev)
        paths = [("cta", 32769), ("grid", 2)] if n <= 32768 else [("grid", 32769)]
        for name, _ in paths:
            res["linkage_ms"][f"{n}/{name}"] = []
        for _ in range(args.reps):                         # alternate the paths
            for name, gmin in paths:
                t = time_linkage(ctx, x, gmin, 1)
                res["linkage_ms"][f"{n}/{name}"] += t
                print(f"linkage n={n} dim=256 {name}: {t[0]:.0f} ms", flush=True)
        del x
        torch.cuda.empty_cache()

    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    if args.no_e2e:
        return
    # one long recording end to end, with the stage split: distinct synthetic hours until the kept embeddings pass
    # the whole-GPU threshold (about 7 200 per hour with these seeded weights)
    seg, emb = PyanNet(), WeSpeakerResNet34()
    seg.load_state_dict(syn.make_segmentation_state_dict(0), strict=False)
    emb.load_state_dict(syn.make_embedding_state_dict(1), strict=False)
    pipe = SpeakerDiarization(segmentation=seg, embedding=emb, plda=syn.make_plda(2), device=dev)
    list(pipe.apply_batch([{"waveform": syn.make_conversation(60.0, seed=1), "sample_rate": 16000, "uri": "warm"}]))
    pieces = int(np.ceil(args.hours))
    wav = torch.cat([syn.make_conversation(3600.0 * args.hours / pieces, seed=700 + h) for h in range(pieces)], dim=1)
    os.environ["B200_TIMING"] = "1"
    split = io.StringIO()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stderr(split):
        (_, (out, art)), = list(pipe.apply_batch([{"waveform": wav, "sample_rate": 16000, "uri": "long"}],
                                                 return_artifacts=True))
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    del os.environ["B200_TIMING"]
    from oracle import pipeline as P

    n = len(P.filter_embeddings(art["embeddings"].cpu().numpy(),
                                art["segmentations"].cpu().numpy().astype(np.float32))[0])
    stages = [line for line in split.getvalue().splitlines() if line.startswith("[b200 timing]")]
    res["e2e"] = {"hours": args.hours, "chunks": int(art["segmentations"].shape[0]), "kept_embeddings": n,
                  "wall_s": wall, "speakers": len(out.speaker_diarization.labels()), "stage_split": stages}
    print(f"e2e: {json.dumps(res['e2e'])}", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    assert n > 32768, f"only {n} kept embeddings: the file was clustered on the one-CTA kernel; raise --hours"

if __name__ == "__main__":
    main()
