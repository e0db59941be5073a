"""Per-kernel profile of the segmentation network (PyanNet): time, executed TFLOP/s and model bytes/s of every kernel of
one `ctx.seg_forward` call on 10 s windows.

    python scripts/seg_profile.py                  # the library in this tree (needs a GPU)
    python scripts/seg_profile.py --root OTHER     # another tree's build
    python scripts/seg_profile.py --model-only     # the FLOP / byte model alone (no GPU)

`ctx.seg_forward` runs on a full sub-batch (--batch, the library's seg_max_batch of 2112 windows) and on --tail
windows (bench.py's step of 12 x 10 min = 7092 windows = 3 x 2112 + 756), after warm-up, under torch.profiler with
CUDA activities.  A call's kernels run from `wav_stats_kernel` to the classifier.

FLOP / byte model, per call of NB windows of W samples (computed from the shapes, not measured):
  FLOP  = as executed: the split-precision kernels run three products (lo*hi, hi*lo, hi*hi) per multiply-add, and the
          SincNet layers compute whole 192-position tiles (64 pooled outputs, N padded to 80 / 64 channels)
  bytes = each kernel's global inputs and outputs once (fp32 activations, fp16 (hi, lo) pairs where a kernel reads or
          writes them); weights and InstanceNorm partial sums other than the finalize kernels' are left out
"""
import argparse
import os
import re
import subprocess
import sys

SINC_K, SINC_STRIDE, TILE_P = 251, 10, 64
CHUNK = 160000
HIDDEN, LAYERS = 128, 4


def geom(W):
    """(pool0, pool1, pool2, tiles0, tiles1, tiles2) of a window of W samples (seg.cuh seg_geom)."""
    pool0 = (1 + (W - SINC_K) // SINC_STRIDE) // 3
    pool1 = (pool0 - 4) // 3
    pool2 = (pool1 - 4) // 3
    return pool0, pool1, pool2, *(-(-p // TILE_P) for p in (pool0, pool1, pool2))


def model(NB, W=CHUNK, classes=7):
    """[(label, FLOP, bytes)] of one seg_forward call in launch order (the GPU path's defaults)."""
    p0, p1, p2, t0, t1, t2 = geom(W)
    T = p2
    M = NB * T
    f4 = 4
    rows = [("wav stats", 3.0 * NB * W, NB * W * f4)]
    rows.append(("sinc", 6.0 * NB * t0 * 192 * 80 * 256, NB * W * f4 + NB * 80 * p0 * f4))
    rows.append(("IN finalize 0", 10.0 * NB * 80 * t0, NB * 80 * t0 * 16))
    rows.append(("conv1", 6.0 * NB * t1 * 192 * 64 * 400, NB * 80 * p0 * f4 + NB * 60 * p1 * f4))
    rows.append(("IN finalize 1", 10.0 * NB * 60 * t1, NB * 60 * t1 * 16))
    rows.append(("conv2", 6.0 * NB * t2 * 192 * 64 * 320, NB * 60 * p1 * f4 + NB * 60 * p2 * f4))
    rows.append(("IN finalize 2", 10.0 * NB * 60 * t2, NB * 60 * t2 * 16))
    rows.append(("apply/transpose", 3.0 * NB * 60 * T, NB * 60 * T * f4 + M * 64 * f4))
    rows.append(("split", 2.0 * M * 64, M * 64 * f4 + M * 64 * 4))
    for l in range(LAYERS):
        K = 64 if l == 0 else 2 * HIDDEN
        rows.append((f"input proj l{l}", 6.0 * M * 1024 * K, M * K * 4 + M * 1024 * f4))
        rows.append((f"recurrence l{l}", 6.0 * M * 2 * 4 * HIDDEN * HIDDEN, M * 1024 * f4 + M * 2 * HIDDEN * 4))
    rows.append(("linear 1", 6.0 * M * 128 * 256, M * 256 * 4 + M * 128 * 4))
    rows.append(("linear 2", 6.0 * M * 128 * 128, M * 128 * 4 + M * 128 * f4))
    rows.append(("classifier", 2.0 * M * classes * 128, M * 128 * f4 + M * (1 + 4 * classes)))
    return rows


FRONT_END = {"wav stats", "wav finalize", "sinc", "IN finalize 0", "conv1", "IN finalize 1", "conv2", "IN finalize 2",
             "apply/transpose"}


def label_call(names):
    """Labels of one call's kernel names, in launch order (names: demangled kernel names from the profiler)."""
    out, layer, gemms, recs = [], -1, 0, 0
    for n in names:
        if "wav_stats" in n:
            lab = "wav stats"
        elif "wav_finalize" in n:
            lab = "wav finalize"
        elif re.search(r"sinc_conv_\w+_kernel<0,|sinc_pool_kernel", n):
            lab, layer = "sinc", 0
        elif re.search(r"sinc_conv_\w+_kernel<80,|conv5_pool_kernel<80>", n):
            lab, layer = "conv1", 1
        elif re.search(r"sinc_conv_\w+_kernel<60,|conv5_pool_kernel<60>", n):
            lab, layer = "conv2", 2
        elif "in_finalize" in n or "part_reduce" in n:
            lab = f"IN finalize {layer}" if "in_finalize" in n else f"IN reduce {layer}"
        elif "in_apply_transpose" in n:
            lab = "apply/transpose"
        elif "split_f16" in n:
            lab = "split"
        elif "gemm" in n.lower():
            lab = f"input proj l{gemms}" if gemms < LAYERS else f"linear {gemms - LAYERS + 1}"
            gemms += 1
        elif "rec" in n.lower() or "lstm" in n.lower():
            lab = f"recurrence l{recs}"
            recs += 1
        elif "classifier" in n or "head" in n.lower():
            lab = "classifier"
        else:
            lab = n.split("(")[0][-40:]
        out.append(lab)
    return out


def print_model(NB):
    print(f"model of one seg_forward call, {NB} x 10 s windows:")
    print(f"{'kernel':<18} {'GFLOP':>9} {'MB':>9}")
    for lab, f, b in model(NB):
        print(f"{lab:<18} {f / 1e9:9.1f} {b / 1e6:9.1f}")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        return out.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def profile_calls(ctx, wav, off, valid, iters):
    """{label: mean us} and the label order of `iters` profiled seg_forward calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(2):
        ctx.seg_forward(wav, off, valid)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            ctx.seg_forward(wav, off, valid)
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                  and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()),
                 key=lambda e: e.time_range.start)
    calls, cur = [], None
    for e in evs:
        if "wav_stats" in e.name:
            cur = []
            calls.append(cur)
        if cur is not None:
            cur.append((e.name, e.time_range.end - e.time_range.start))
    if not calls:
        raise SystemExit("found no seg_forward call (no wav_stats_kernel in the trace)")
    labels = label_call([n for n, _ in calls[0]])
    us = {}
    for c in calls:
        if len(c) != len(labels):
            raise SystemExit(f"calls launched {len(c)} and {len(labels)} kernels")
        for lab, (_, t) in zip(label_call([n for n, _ in c]), c):
            us[lab] = us.get(lab, 0.0) + t / len(calls)
    return us, labels


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="tree whose built library is timed (default: this one)")
    ap.add_argument("--batch", type=int, default=2112, help="windows of a full sub-batch (seg_max_batch: 2112)")
    ap.add_argument("--tail", type=int, default=756, help="windows of bench.py's last sub-batch per step (756)")
    ap.add_argument("--iters", type=int, default=5, help="profiled calls per size")
    ap.add_argument("--model-only", action="store_true", help="print the FLOP / byte model and exit (no GPU needed)")
    args = ap.parse_args()

    print_model(args.batch)
    if args.model_only:
        return

    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np
    import torch

    from pyannote_audio_b200 import ops, synthetic as syn

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: only --model-only runs without a GPU")
    dev = torch.device("cuda:0")
    ctx = ops.Context(dev)
    ctx.load_segmentation(syn.make_segmentation_state_dict(0))
    g = torch.Generator().manual_seed(0)
    n_max = max(args.batch, args.tail)
    step = 16000                                        # 10 s windows every second, as the pipeline's sliding window
    wav = (torch.randn(step * (n_max - 1) + CHUNK, generator=g) * 0.1).to(dev)
    info = gpu_info()
    print(f"\nGPU: {info}   (name, power limit, SM clock now, max SM clock)")
    print(f"root {os.path.abspath(args.root)}, mean of {args.iters} calls per size")
    per_size = {}
    for nb in (args.batch, args.tail):
        off = np.arange(nb, dtype=np.int64) * step
        valid = np.full(nb, CHUNK, dtype=np.int32)
        us, labels = profile_calls(ctx, wav, off, valid, args.iters)
        per_size[nb] = us
        mdl = {lab: (f, b) for lab, f, b in model(nb)}
        total = sum(us.values())
        front = sum(t for lab, t in us.items() if lab in FRONT_END)
        print(f"\nseg_forward on {nb} x 10 s windows: {total / 1e3:.3f} ms of kernels, SincNet front end "
              f"{front / 1e3:.3f} ms ({100 * front / total:.1f} %)")
        print(f"{'kernel':<18} {'us':>9} {'share':>6} {'TFLOP/s':>8} {'GB/s':>7}")
        for lab in labels:
            t = us[lab]
            f, b = mdl.get(lab, (0.0, 0.0))
            sec = t * 1e-6
            print(f"{lab:<18} {t:9.1f} {100 * t / total:5.1f}% {f / sec / 1e12:8.1f} {b / sec / 1e9:7.0f}")
    if len(per_size) == 2:
        full, tail = (per_size[n] for n in (args.batch, args.tail))
        per_step = {lab: 3 * full[lab] + tail.get(lab, 0.0) for lab in full}
        tot = sum(per_step.values())
        front = sum(t for lab, t in per_step.items() if lab in FRONT_END)
        print(f"\nper bench.py step (3 x {args.batch} + {args.tail} windows): {tot / 1e3:.1f} ms of segmentation kernels, "
              f"SincNet front end {front / 1e3:.1f} ms ({100 * front / tot:.1f} %): "
              + ", ".join(f"{lab} {per_step[lab] / 1e3:.1f}" for lab in ("sinc", "conv1", "conv2")) + " ms")


if __name__ == "__main__":
    main()
