"""Per-conv profile of a WeSpeaker trunk: time, TFLOP/s, operand fill and unique HBM traffic of each trunk conv.

    python scripts/trunk_profile.py                  # the library in this tree (needs a GPU), ResNet34
    python scripts/trunk_profile.py --model resnet293   # a bottleneck trunk (resnet152 | resnet221 | resnet293)
    python scripts/trunk_profile.py --root OTHER --plan pairs  # another tree's build, with its launch plan
    python scripts/trunk_profile.py --model-only     # the byte model alone (no GPU)

`ctx.emb_trunk` runs on --batch segments (the library's embedding sub-batch) under torch.profiler with CUDA
activities, after warm-up.  The trunk convs are the kernel launches between the stem (`conv1_kernel`) and
`frames_to_nchw`, in the order of trunk_convs() below.

Byte model, per segment (computed from the shapes, not measured):
  fill  = bytes TMA moves from L2 into shared memory for the operands, for the launch plan of conv_forward:
          per-tap : every (tap, channel chunk) stages a 128-pixel activation box and one weight tile (per 256-channel
                    column tile for C_out > 256)
          reuse   : stride-1 3x3 convs with one channel chunk and C_out <= 64 (layers 1 and 2) stage one 136-pixel
                    activation box per kh for the three kw taps, and every weight tile; the other convs stay per-tap
          resident: the stride-1 3x3 convs with one channel chunk and C_in = C_out (layers 1 and 2) stage each input
                    row of a band of output rows once as a 136-pixel box (plus two halo rows per band) and their nine
                    weight taps once per CTA (--sms CTAs per SM count as in conv_forward); the other convs stay per-tap
          rows    : resident for layers 1 and 2; the stride-1 3x3 convs with C_in = C_out = 128 / 256 (layers 3 and 4)
                    stage each of the three input rows of an output tile once per channel chunk as a 136-pixel box,
                    and every weight tile; the other convs stay per-tap
          fused   : rows, except that each stride-1 BasicBlock of layer 1 is one launch (block_row_kernel): it stages
                    each input row of a band once (plus four halo rows per band) as a 136-pixel box per 126-column
                    strip, and both convs' weights once per CTA; the intermediate activation stays on chip
          pairs   : fused, except that the stride-1 3x3 convs with C_in = C_out = 128 (layer 3) compute two output rows
                    per unit: four input rows per channel chunk as 136-pixel boxes, and every weight tile once for
                    both rows
          epilogue: pairs, except that the resident convs with a residual (conv_row_kernel: layer 2's conv2) also
                    stage each output row's residual, 128 pixels, into shared memory for the epilogue
  HBM   = input + output (+ residual) activations once, and the weights once per launch shared by --batch segments;
          a fused block reads its input once and writes its output once
"""
import argparse
import os
import statistics
import subprocess
import sys

TILE_M = 128
HALO = 8
STRIP_W = TILE_M - 2         # output columns per strip of block_row_kernel


BOTTLENECK_BLOCKS = {"resnet152": (3, 8, 36, 3), "resnet221": (6, 16, 48, 3), "resnet293": (10, 20, 64, 3)}


def trunk_convs(model="resnet34"):
    """(layer, name, C_in, C_out, ksize, stride, H_in, W_in, has_residual) of the trunk convs in launch order (35 for
    ResNet34; conv1, conv2, shortcut, conv3 per Bottleneck, api.cu bottleneck_run)."""
    convs = []
    H, W, C = 80, 998, 32
    if model != "resnet34":
        for li, (p, blocks, stride) in enumerate(zip((32, 64, 128, 256), BOTTLENECK_BLOCKS[model], (1, 2, 2, 2)),
                                                 start=1):
            for bi in range(blocks):
                s = stride if bi == 0 else 1
                Ho, Wo = (H + 2 - 3) // s + 1, (W + 2 - 3) // s + 1
                convs.append((li, f"layer{li}.{bi}.conv1", C, p, 1, 1, H, W, False))
                convs.append((li, f"layer{li}.{bi}.conv2", p, p, 3, s, H, W, False))
                if s != 1 or C != 4 * p:
                    convs.append((li, f"layer{li}.{bi}.shortcut", C, 4 * p, 1, s, H, W, False))
                convs.append((li, f"layer{li}.{bi}.conv3", p, 4 * p, 1, 1, Ho, Wo, True))
                H, W, C = Ho, Wo, 4 * p
        return convs
    for li, (cout, blocks, stride) in enumerate(((32, 3, 1), (64, 4, 2), (128, 6, 2), (256, 3, 2)), start=1):
        for bi in range(blocks):
            s = stride if bi == 0 else 1
            Ho, Wo = (H + 2 - 3) // s + 1, (W + 2 - 3) // s + 1
            convs.append((li, f"layer{li}.{bi}.conv1", C, cout, 3, s, H, W, False))
            if s != 1 or C != cout:
                convs.append((li, f"layer{li}.{bi}.shortcut", C, cout, 1, s, H, W, False))
            convs.append((li, f"layer{li}.{bi}.conv2", cout, cout, 3, 1, Ho, Wo, True))
            H, W, C = Ho, Wo, cout
    return convs


def resident_plan(cout, ho, tiles_w, batch, sms):
    """(CTAs, output rows per band, bands) of conv_row_kernel, as conv_forward chooses them."""
    ctas = (2 if cout == 32 else 1) * sms
    strips = batch * tiles_w
    band = -(-ho // min(ho, -(-ctas // strips)))
    return min(ctas, strips * -(-ho // band)), band, -(-ho // band)


def launches(model, plan):
    """The trunk's kernel launches in order: lists of the trunk_convs() entries each one computes (two for a fused
    block, conv1 and conv2)."""
    convs = trunk_convs(model)
    out = []
    for c in convs:
        fuse = (plan in ("fused", "pairs", "epilogue") and model == "resnet34" and c[0] == 1 and c[1].endswith(".conv2") and out and
                out[-1][0][1].endswith(".conv1") and out[-1][0][5] == 1)
        if fuse:
            out[-1].append(c)
        else:
            out.append([c])
    return out


def fused_model(c1, c2, batch, sms=132):
    """(GFLOP, fill MB, unique HBM MB) per segment of a fused block (block_row_kernel: two CTAs per SM)."""
    _, _, cin, cout, k, _, H, W, _ = c1
    strips = -(-W // STRIP_W)
    ctas = 2 * sms
    band = -(-H // min(H, -(-ctas // (batch * strips))))
    bands = -(-H // band)
    ctas = min(ctas, batch * strips * bands)
    fill = strips * (H + 4 * bands) * (TILE_M + HALO) * cin * 2 + ctas * 2 * k * k * cin * cout * 2 / batch
    hbm = H * W * cin * 2 + H * W * cout * 2 + 2 * k * k * cin * cout * 2 / batch
    return 2 * 2.0 * H * W * cout * cin * k * k / 1e9, fill / 1e6, hbm / 1e6


def launch_model(convs, plan, batch, sms=132):
    if len(convs) == 2:
        return fused_model(*convs, batch, sms)
    return conv_model(convs[0], plan, batch, sms)


def conv_model(c, plan, batch, sms=132):
    """(GFLOP, fill MB, unique HBM MB) per segment of one conv."""
    _, _, cin, cout, k, s, H, W, res = c
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    ck = 64 if cin >= 64 else 32
    chunks = cin // ck
    n_tile = min(cout, 256)
    tiles = Ho * -(-Wo // TILE_M) * (cout // n_tile)
    b_tile = n_tile * ck * 2
    reuse = k == 3 and s == 1 and ((plan == "reuse" and cin == ck and cout <= 64) or
                                   (plan in ("rows", "fused", "pairs", "epilogue") and cin == cout and
                                    cout in (128, 256)))
    if plan in ("resident", "rows", "fused", "pairs", "epilogue") and k == 3 and s == 1 and cin == ck and cout == cin:
        tiles_w = -(-Wo // TILE_M)
        ctas, _, bands = resident_plan(cout, Ho, tiles_w, batch, sms)
        fill = tiles_w * (Ho + 2 * bands) * (TILE_M + HALO) * ck * 2 + ctas * k * k * b_tile / batch
        if plan == "epilogue" and res:
            fill += tiles_w * Ho * TILE_M * cout * 2
    elif reuse:
        rows = 2 if plan in ("pairs", "epilogue") and cout == 128 else 1   # output rows per unit
        units = -(-Ho // rows) * -(-Wo // TILE_M)
        fill = units * ((rows + k - 1) * chunks * (TILE_M + HALO) * ck * 2 + k * k * chunks * b_tile)
    else:
        fill = tiles * k * k * chunks * (TILE_M * ck * 2 + b_tile)
    act_out = Ho * Wo * cout * 2
    hbm = H * W * cin * 2 + act_out * (2 if res else 1) + k * k * cin * cout * 2 / batch
    return 2.0 * Ho * Wo * cout * cin * k * k / 1e9, fill / 1e6, hbm / 1e6


def print_model(plan, batch, sms, model="resnet34"):
    rows = [(cs, *launch_model(cs, plan, batch, sms)) for cs in launches(model, plan)]
    print(f"byte model of {model} ({plan} plan), per segment:")
    print(f"{'layer':>6} {'convs':>5} {'launches':>8} {'GFLOP':>7} {'fill MB':>8} {'HBM MB':>7} {'FLOP/fill B':>11} "
          f"{'FLOP/HBM B':>10}")
    tot = [0, 0, 0.0, 0.0, 0.0]
    for li in (1, 2, 3, 4):
        sel = [r for r in rows if r[0][0][0] == li]
        nc = sum(len(r[0]) for r in sel)
        g, f, h = (sum(r[i] for r in sel) for i in (1, 2, 3))
        tot = [tot[0] + nc, tot[1] + len(sel), tot[2] + g, tot[3] + f, tot[4] + h]
        print(f"{li:>6} {nc:>5} {len(sel):>8} {g:7.2f} {f:8.1f} {h:7.1f} {g * 1e3 / f:11.0f} {g * 1e3 / h:10.0f}")
    print(f"{'total':>6} {tot[0]:>5} {tot[1]:>8} {tot[2]:7.2f} {tot[3]:8.1f} {tot[4]:7.1f} {tot[2] * 1e3 / tot[3]:11.0f} "
          f"{tot[2] * 1e3 / tot[4]:10.0f}")
    return rows


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        return out.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="tree whose built library is timed (default: this one)")
    ap.add_argument("--plan", choices=["epilogue", "pairs", "fused", "rows", "resident", "reuse", "per-tap"],
                    default="epilogue",
                    help="launch plan of the timed library for the byte model (pairs: a library whose layer 2 convs "
                         "read the residual from global memory; fused: one whose layer 3 convs "
                         "compute one output row per unit; rows: one whose layer 1 blocks "
                         "run as two conv launches each; resident: one whose layer 3 and "
                         "4 convs stage one box per tap; reuse: one whose layer 1 and 2 convs stage one box per kh; "
                         "per-tap: one box per tap everywhere)")
    ap.add_argument("--sms", type=int, default=132, help="SMs of the GPU for the resident plan (H100 SXM: 132)")
    ap.add_argument("--batch", type=int, default=264, help="segments per emb_trunk call (library sub-batch: 264)")
    ap.add_argument("--iters", type=int, default=5, help="profiled emb_trunk calls")
    ap.add_argument("--model-only", action="store_true", help="print the byte model and exit (no GPU needed)")
    ap.add_argument("--model", choices=["resnet34", *BOTTLENECK_BLOCKS], default="resnet34",
                    help="trunk to profile (synthetic weights)")
    args = ap.parse_args()

    rows = print_model(args.plan, args.batch, args.sms, args.model)
    if args.model_only:
        return

    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from torch.profiler import ProfilerActivity, profile

    from pyannote_audio_b200 import ops, synthetic as syn

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: only --model-only runs without a GPU")
    dev = torch.device("cuda:0")
    ctx = ops.Context(dev)
    ctx.load_embedding(syn.make_embedding_state_dict(1) if args.model == "resnet34" else
                       syn.make_bottleneck_state_dict(int(args.model[len("resnet"):]), 1))
    g = torch.Generator().manual_seed(0)
    fb = (torch.randn((args.batch, 998, 80), generator=g) * 2.0).to(dev)
    for _ in range(3):
        ctx.emb_trunk(fb)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            ctx.emb_trunk(fb)
        torch.cuda.synchronize()
    info = gpu_info()

    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    runs, cur = [], None
    for e in evs:
        if "conv1_kernel" in e.name:
            cur = []
        elif "frames_to_nchw" in e.name:
            if cur is not None:
                runs.append(cur)
            cur = None
        elif cur is not None and ("conv" in e.name or "block_row_kernel" in e.name):
            cur.append(e.time_range.end - e.time_range.start)        # us
    n = len(rows)
    runs = [r for r in runs if len(r) == n]
    if not runs:
        raise SystemExit(f"found no emb_trunk call with {n} trunk launches between conv1_kernel and frames_to_nchw")
    us = [sum(r[i] for r in runs) / len(runs) for i in range(n)]

    print(f"\nGPU: {info}   (name, power limit, SM clock now, max SM clock)")
    print(f"root {os.path.abspath(args.root)}, {args.batch} segments per call, mean of {len(runs)} calls\n")
    print(f"{'conv':<20} {'Cin>Cout':>9} {'k/s':>4} {'HxW in':>8} {'us':>8} {'TFLOP/s':>8} {'fill GB/s':>9} {'HBM GB/s':>9}")
    tot_us = 0.0
    per_layer = {}
    for (cs, gf, fmb, hmb), t in zip(rows, us):
        c = cs[0]
        _, name, cin, cout, k, s, H, W, _ = c
        if len(cs) == 2:
            name = name.rsplit(".", 1)[0] + " (fused)"
        sec = t * 1e-6
        tot_us += t
        L = per_layer.setdefault(c[0], [0.0, 0.0, 0.0, 0.0])
        L[0] += t; L[1] += gf; L[2] += fmb; L[3] += hmb
        print(f"{name:<20} {f'{cin}>{cout}':>9} {f'{k}/{s}':>4} {f'{H}x{W}':>8} {t:8.1f} "
              f"{gf * args.batch / sec / 1e3:8.1f} {fmb * args.batch / sec / 1e3:9.0f} {hmb * args.batch / sec / 1e3:9.0f}")
    print()
    for li, (t, gf, fmb, hmb) in sorted(per_layer.items()):
        sec = t * 1e-6
        print(f"layer{li}: {t / 1e3:7.3f} ms  {gf * args.batch / sec / 1e3:6.1f} TFLOP/s  "
              f"fill {fmb * args.batch / sec / 1e3:6.0f} GB/s  HBM {hmb * args.batch / sec / 1e3:6.0f} GB/s")
    print(f"trunk convs: {tot_us / 1e3:.3f} ms per call of {args.batch} segments "
          f"({tot_us / args.batch:.1f} us per segment)")
    # what the residual costs: median time of the single-launch stride-1 3x3 convs with a residual (BasicBlock conv2)
    # over the median of those without one (conv1), per layer
    for li in sorted(per_layer):
        t = {True: [], False: []}
        for (cs, *_), t_us in zip(rows, us):
            c = cs[0]
            if len(cs) == 1 and c[0] == li and c[4] == 3 and c[5] == 1:
                t[c[8]].append(t_us)
        if t[True] and t[False]:
            print(f"layer{li} conv2/conv1: {statistics.median(t[True]) / statistics.median(t[False]):.3f} "
                  f"({statistics.median(t[True]):.1f} / {statistics.median(t[False]):.1f} us, medians)")


if __name__ == "__main__":
    main()
